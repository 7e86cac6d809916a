// nr_soft_frag.cu -- soft fragments (nr_b200_soft_fragments / nr_b200_soft_fragments_backward, include/nr_b200.h): for
// every pixel the K nearest faces within reach, by (zp, f), with their depth zp, perspective-correct barycentrics l'_k and
// signed squared distance, for shading and blending in PyTorch.
//
// The host checks, the workspace and the binning (setup, scan, depth records; unsorted: the selection does not depend on
// the list order) are nr_soft_rgb.cu's (nr_internal.h); the face staging, the barycentrics and the distance test are
// nr_soft_rgb.cuh's and nr_soft.cuh's; the chain from l'_k and zp into the vertices is k_soft_attr_bwd's (a copy,
// soft_lprime_chain, as nr_soft_attr.cu copies it from k_soft_uv_bwd).  New kernels:
//   k_soft_frag_fwd<K, kCap>  one CTA per (tile, item), stage_rgb's rounds; per pixel a fully unrolled compare-and-shift
//                             insertion of (zp, f) into kCap register slots (kCap = 4, 8, 16 or 32, the smallest >= K: a
//                             dynamically indexed register array would spill); after the traversal the <= K winners are
//                             re-evaluated from their global records (bit-identical to the staged copies) and written,
//                             four slots at a time, as 16-byte vectors when K % 4 == 0
//   k_soft_frag_bwd           one CTA per (tile, item) over the saved pix_to_face (no lists, no key width): every
//                             fragment's 9 vertex partials are merged per face in a shared-memory hash table, which is
//                             flushed with one set of global atomics per face (against one set per fragment: DESIGN.md 4s)
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <string.h>

#include "nr_b200.h"
#include "nr_internal.h"
#include "nr_soft.cuh"
#include "nr_soft_rgb.cuh"

namespace {

constexpr int kMaxK = 32;

struct SoftFragParams {
    SoftRgbParams r;         // the soft RGB's binning (its colour, alpha and softmax fields unused)
    long long* p2f;          // [B,S,S,K]
    float* zbuf;             // [B,S,S,K]
    float* bary;             // [B,S,S,K,3]
    float* dists;            // [B,S,S,K]
    const long long* ip2f;   // backward: the forward's pix_to_face
    const float* g_zbuf;     // backward: [B,S,S,K] or nullptr
    const float* g_bary;     // backward: [B,S,S,K,3] or nullptr
    const float* g_dists;    // backward: [B,S,S,K] or nullptr
    int K;
    bool vec;                // K % 4 == 0 and every output 16-byte aligned
};

// l'_k = l_k (zp / z_k) (nr_soft_attr.cu)
__device__ __forceinline__ void lprime(const SoftBary& bc, const float4& z, float lp[3]) {
    lp[0] = __fmul_rn(bc.l[0], __fdiv_rn(bc.zp, z.x));
    lp[1] = __fmul_rn(bc.l[1], __fdiv_rn(bc.zp, z.y));
    lp[2] = __fmul_rn(bc.l[2], __fdiv_rn(bc.zp, z.z));
}

// The backward from l'_k = l_k r_k, r_k = zp / z_k, and zp of a (pixel, face): nr_soft_attr.cu's soft_lprime_chain,
// copied (sharing it changed the instruction schedule of the kernel it came from, DESIGN.md 4r).  Gt_k = d loss / d l'_k,
// dzp = d loss / d zp so far; on through l_k, zp and z_k, the lh clamp (held) and the edge functions c_e of the face
// record `rec` at pixel (px, py) into v[2m], v[2m + 1] (x, y of vertex m) and v[6 + m] (its z).
__device__ __forceinline__ void soft_lprime_chain(const SoftBary& bc, const float4& z, const float4* rec, float px, float py,
                                                  const float Gt_k[3], float dzp, float* v) {
    const float zz[3] = {z.x, z.y, z.z};
    float dl[3], dz[3];
#pragma unroll
    for (int a = 0; a < 3; a++) {
        const float r = __fdiv_rn(bc.zp, zz[a]);
        const float Gt = Gt_k[a];
        dl[a] = __fmul_rn(Gt, r);
        dzp = __fmaf_rn(Gt, __fdiv_rn(bc.l[a], zz[a]), dzp);
        dz[a] = -__fmul_rn(__fmul_rn(Gt, bc.l[a]), __fdiv_rn(r, zz[a]));
    }
    // zp = 1 / Q, Q = sum_k l_k / z_k
    const float dQ = -__fmul_rn(__fmul_rn(bc.zp, bc.zp), dzp);
    float sl = 0.0f;
#pragma unroll
    for (int a = 0; a < 3; a++) {
        dl[a] = __fmaf_rn(dQ, __frcp_rn(zz[a]), dl[a]);
        dz[a] = __fsub_rn(dz[a], __fmul_rn(dQ, __fdiv_rn(__fdiv_rn(bc.l[a], zz[a]), zz[a])));
        v[6 + a] = dz[a];
        sl = __fmaf_rn(bc.l[a], dl[a], sl);
    }
    // l = lh / s, lh = clamp(lam, 0, 1), lam_m = c_{m+1} / A
    float dlam[3], sg = 0.0f;
#pragma unroll
    for (int a = 0; a < 3; a++) {
        const bool in = bc.lam[a] >= 0.0f && bc.lam[a] <= 1.0f;
        dlam[a] = in ? __fdiv_rn(__fsub_rn(dl[a], sl), bc.s) : 0.0f;
        sg = __fmaf_rn(dlam[a], bc.lam[a], sg);
    }
    // c_e = (b - a) x (p - a) of edge e = (v_e, v_e+1): d c / d a = (by - py, px - bx), d c / d b = (py - ay, ax - px)
#pragma unroll
    for (int e = 0; e < 3; e++) {
        const float dc = __fdiv_rn(__fsub_rn(dlam[e == 0 ? 2 : e - 1], sg), z.w);
        const float4 ed = rec[e];
        const float dx = __fsub_rn(px, ed.x), dy = __fsub_rn(py, ed.y);
        const int nb = e == 2 ? 0 : e + 1;
        v[2 * e] = __fmaf_rn(dc, __fsub_rn(ed.w, dy), v[2 * e]);
        v[2 * e + 1] = __fmaf_rn(dc, __fsub_rn(dx, ed.z), v[2 * e + 1]);
        v[2 * nb] = __fmaf_rn(dc, dy, v[2 * nb]);
        v[2 * nb + 1] = __fmaf_rn(dc, -dx, v[2 * nb + 1]);
    }
}

// One (pixel, face) re-evaluated from the face's global records: false when it is not a candidate (never for a face the
// forward selected: the records and the pixel are the ones it tested).  dist = +-d^2 (- outside; soft_eval's d^2, the
// expression it minimised, so exactly sigma x_j before the scaling by 1 / sigma).
struct Frag {
    SoftBary bc;
    float4 z;
    float x, t, qx, qy, dist;
    int k;
};
__device__ __forceinline__ bool frag_eval(const SoftParams& s, const float4* rec, const float4& z, float px, float py, Frag& o) {
    float c[3];
    if (!soft_eval(rec, px, py, s.inv_sigma, s.cut, o.x, o.k, o.t, o.qx, o.qy, c)) return false;
    if (z.w == 0.0f) return false;
    o.z = z;
    o.bc = soft_bary(c, z);
    const float d2 = __fmaf_rn(o.qx, o.qx, o.qy * o.qy);
    o.dist = signbit(o.x) ? -d2 : d2;
    return isfinite(o.bc.zp);
}

// ------------------------------------------------------------------------------------------------ k_soft_frag_fwd
// (zp, f) < (zq, g): the selection order (f >= 0 of a candidate always beats the empty slot {+inf, INT_MAX})
__device__ __forceinline__ bool frag_less(float za, int fa, float zb, int fb) { return za < zb || (za == zb && fa < fb); }

template <typename K, int kCap>
__global__ void __launch_bounds__(kThreads) k_soft_frag_fwd(const __grid_constant__ SoftFragParams P) {
    __shared__ float4 s_rec[kThreads * 4];
    __shared__ float4 s_z[kThreads];
    __shared__ int s_face[kThreads];
    __shared__ int s_wn[kWarps];
    const SoftRgbParams& p = P.r;
    const int tile = blockIdx.x, b = blockIdx.y;
    const int tx = tile % p.s.ntx, ty = tile / p.s.ntx;
    const int col = tx * kTile + (threadIdx.x % kTile), row = ty * kTile + (threadIdx.x / kTile);
    const int S = p.s.S, Kq = P.K;
    const float px = soft_centre(col, S), py = soft_centre(S - 1 - row, S);
    const size_t seg = (size_t)b * (p.s.ntiles + 1);
    const int n_tile = p.s.cnt[seg + tile], n_all = n_tile + p.s.cnt[seg + p.s.ntiles];
    float sz[kCap];
    int sf[kCap];
#pragma unroll
    for (int i = 0; i < kCap; i++) { sz[i] = INFINITY; sf[i] = 0x7FFFFFFF; }
    for (int next = 0; next < n_all; next += kThreads) {
        const int n = stage_rgb<K>(p, b, tile, tx, ty, n_tile, n_all, next, s_rec, s_z, s_face, s_wn);
        for (int j = 0; j < n; j++) {
            float x, t, qx, qy, c[3];
            int k;
            if (!soft_eval(s_rec + 4 * j, px, py, p.s.inv_sigma, p.s.cut, x, k, t, qx, qy, c)) continue;
            const float4 z = s_z[j];
            if (z.w == 0.0f) continue;  // a zero-area face is not a fragment
            float cz = soft_bary(c, z).zp;
            if (!isfinite(cz)) continue;
            int cf = s_face[j];
            if (!frag_less(cz, cf, sz[kCap - 1], sf[kCap - 1])) continue;
            // compare and shift: the candidate sinks to its place, every larger slot moves one down
#pragma unroll
            for (int i = 0; i < kCap; i++) {
                const bool lt = frag_less(cz, cf, sz[i], sf[i]);
                const float tz = sz[i];
                const int tf = sf[i];
                sz[i] = lt ? cz : tz; sf[i] = lt ? cf : tf;
                cz = lt ? tz : cz; cf = lt ? tf : cf;
            }
        }
        __syncthreads();
    }
    if (row >= S || col >= S) return;
    const size_t pix = ((size_t)b * S + row) * S + col, o = pix * (size_t)Kq;
    const SoftParams& s = p.s;
    // four slots at a time: re-evaluate the winners, then store (16-byte vectors when K % 4 == 0)
#pragma unroll
    for (int g = 0; g < kCap; g += 4) {
        if (g >= Kq) break;
        long long id4[4];
        float z4[4], d4[4], l12[12];
#pragma unroll
        for (int q = 0; q < 4; q++) {
            const int i = g + q;
            id4[q] = -1; z4[q] = -1.0f; d4[q] = -1.0f;
            l12[3 * q] = -1.0f; l12[3 * q + 1] = -1.0f; l12[3 * q + 2] = -1.0f;
            if (i < Kq && sf[i] != 0x7FFFFFFF) {
                const size_t fid = (size_t)b * s.F + sf[i];
                Frag fr;
                if (frag_eval(s, s.rec + fid * 4, __ldg(p.zrec + fid), px, py, fr)) {
                    float lp[3];
                    lprime(fr.bc, fr.z, lp);
                    id4[q] = sf[i]; z4[q] = fr.bc.zp; d4[q] = fr.dist;
                    l12[3 * q] = lp[0]; l12[3 * q + 1] = lp[1]; l12[3 * q + 2] = lp[2];
                }
            }
        }
        if (P.vec) {
            __stcs((longlong2*)(P.p2f + o + g), make_longlong2(id4[0], id4[1]));
            __stcs((longlong2*)(P.p2f + o + g + 2), make_longlong2(id4[2], id4[3]));
            __stcs((float4*)(P.zbuf + o + g), make_float4(z4[0], z4[1], z4[2], z4[3]));
            __stcs((float4*)(P.dists + o + g), make_float4(d4[0], d4[1], d4[2], d4[3]));
            float4* bv = (float4*)(P.bary + 3 * (o + g));
            __stcs(bv, make_float4(l12[0], l12[1], l12[2], l12[3]));
            __stcs(bv + 1, make_float4(l12[4], l12[5], l12[6], l12[7]));
            __stcs(bv + 2, make_float4(l12[8], l12[9], l12[10], l12[11]));
        } else {
#pragma unroll
            for (int q = 0; q < 4; q++) {
                const int i = g + q;
                if (i >= Kq) break;
                __stcs(P.p2f + o + i, id4[q]);
                __stcs(P.zbuf + o + i, z4[q]);
                __stcs(P.dists + o + i, d4[q]);
                float* bq = P.bary + 3 * (o + i);
                __stcs(bq, l12[3 * q]); __stcs(bq + 1, l12[3 * q + 1]); __stcs(bq + 2, l12[3 * q + 2]);
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------ k_soft_frag_bwd
constexpr int kFragPartials = 9;    // per face: (x, y) of 3 vertices, z of 3 vertices
constexpr int kTable = 1024;        // hash slots per CTA (a tile's distinct faces; a full table sends straight to global)

__device__ __forceinline__ void send_global(const SoftParams& s, int b, int f, const float* v) {
#pragma unroll
    for (int m = 0; m < 3; m++) {
        if (v[2 * m] == 0.0f && v[2 * m + 1] == 0.0f && v[6 + m] == 0.0f) continue;
        float* gv = nr::face_grad_vertex(s.dst, b, f, m);
        if (gv) { atomicAdd(gv, v[2 * m]); atomicAdd(gv + 1, v[2 * m + 1]); atomicAdd(gv + 2, v[6 + m]); }
    }
}

__global__ void __launch_bounds__(kThreads) k_soft_frag_bwd(const __grid_constant__ SoftFragParams P) {
    __shared__ int s_key[kTable];
    __shared__ float s_acc[kTable * kFragPartials];
    const SoftParams& s = P.r.s;
    const int tile = blockIdx.x, b = blockIdx.y;
    const int tx = tile % s.ntx, ty = tile / s.ntx;
    const int col = tx * kTile + (threadIdx.x % kTile), row = ty * kTile + (threadIdx.x / kTile);
    const int S = s.S, Kq = P.K;
    for (int i = threadIdx.x; i < kTable; i += kThreads) s_key[i] = -1;
    for (int i = threadIdx.x; i < kTable * kFragPartials; i += kThreads) s_acc[i] = 0.0f;
    __syncthreads();
    if (row < S && col < S) {
        const float px = soft_centre(col, S), py = soft_centre(S - 1 - row, S);
        const size_t o = (((size_t)b * S + row) * S + col) * (size_t)Kq;
        for (int i = 0; i < Kq; i++) {
            const long long f = P.ip2f[o + i];
            if (f < 0) break;  // the slots fill front to back
            if (f >= s.F) continue;
            const float gz = P.g_zbuf ? P.g_zbuf[o + i] : 0.0f, gd = P.g_dists ? P.g_dists[o + i] : 0.0f;
            float Gt[3] = {0.0f, 0.0f, 0.0f};
            if (P.g_bary) {
                const float* gb = P.g_bary + 3 * (o + i);
                Gt[0] = gb[0]; Gt[1] = gb[1]; Gt[2] = gb[2];
            }
            if (gz == 0.0f && gd == 0.0f && Gt[0] == 0.0f && Gt[1] == 0.0f && Gt[2] == 0.0f) continue;
            const size_t fid = (size_t)b * s.F + f;
            const float4* rec = s.rec + fid * 4;
            Frag fr;
            if (!frag_eval(s, rec, __ldg(P.r.zrec + fid), px, py, fr)) continue;
            float v[kFragPartials];
#pragma unroll
            for (int m = 0; m < kFragPartials; m++) v[m] = 0.0f;
            soft_lprime_chain(fr.bc, fr.z, rec, px, py, Gt, gz, v);
            // dists = +-d^2: d(d^2)/da = -2 (1 - t)(p - q), d(d^2)/db = -2 t (p - q) for the nearest edge (a, b)
            const float sd = gd * (signbit(fr.x) ? 2.0f : -2.0f);
            const float wa = sd * (1.0f - fr.t), wb = sd * fr.t;
#pragma unroll
            for (int m = 0; m < 3; m++) {
                const bool is_a = m == fr.k, is_b = m == (fr.k == 2 ? 0 : fr.k + 1);
                const float wm = is_a ? wa : (is_b ? wb : 0.0f);
                v[2 * m] = __fmaf_rn(wm, fr.qx, v[2 * m]);
                v[2 * m + 1] = __fmaf_rn(wm, fr.qy, v[2 * m + 1]);
            }
#if defined(NR_B200_TUNING) && defined(NR_SOFT_FRAG_GLOBAL_ATOMICS)
            // the measured alternative (DESIGN.md 4s): one set of global atomics per fragment
            send_global(s, b, (int)f, v);
#else
            // the face's slot: linear probing from a multiplicative hash; a full table sends this fragment to global memory
            int slot = -1;
            unsigned h = ((unsigned)f * 2654435761u) >> 22;  // 10 bits: kTable
            for (int probe = 0; probe < kTable; probe++, h = (h + 1) & (kTable - 1)) {
                const int cur = atomicCAS(&s_key[h], -1, (int)f);
                if (cur == -1 || cur == (int)f) { slot = (int)h; break; }
            }
            if (slot < 0) {
                send_global(s, b, (int)f, v);
            } else {
                float* a = s_acc + slot * kFragPartials;
#pragma unroll
                for (int m = 0; m < kFragPartials; m++)
                    if (v[m] != 0.0f) atomicAdd(a + m, v[m]);
            }
#endif
        }
    }
    __syncthreads();
    // one set of global atomics per face of the tile: thread (table slot, vertex)
    for (int i = threadIdx.x; i < kTable * 3; i += kThreads) {
        const int j = i / 3, m = i % 3;
        const int f = s_key[j];
        if (f < 0) continue;
        const float* a = s_acc + j * kFragPartials;
        const float gx = a[2 * m], gy = a[2 * m + 1], gz = a[6 + m];
        if (gx == 0.0f && gy == 0.0f && gz == 0.0f) continue;
        float* gv = nr::face_grad_vertex(s.dst, b, f, m);
        if (gv) { atomicAdd(gv, gx); atomicAdd(gv + 1, gy); atomicAdd(gv + 2, gz); }
    }
}

constexpr uint32_t kSoftFragFlags = NR_FACES_INDEXED | NR_INDICES_SHARED | NR_GRAD_ACCUMULATE;

// the host checks of both entry points; fills `p` and `L`
int soft_frag_setup(const nr_b200_soft_rgb_args* a, const nr_b200_soft_frag_args* fa, bool backward, SoftFragParams* p,
                    SoftRgbLayout* L) {
    nr_internal::launch_count() = 0;
    if (!a || a->struct_size != sizeof(nr_b200_soft_rgb_args) || !fa || fa->struct_size != sizeof(nr_b200_soft_frag_args))
        return NR_ERR_INVALID_ARG;
    const int K = fa->faces_per_pixel;
    if (K < 1 || K > kMaxK) return NR_ERR_INVALID_ARG;
    if (!fa->pix_to_face || (!backward && (!fa->zbuf || !fa->bary || !fa->dists))) return NR_ERR_INVALID_ARG;
    // the soft RGB's colour, alpha and softmax buffers have no meaning here
    if (a->textures || a->face_light || a->rgb || a->alpha || a->state || a->grad_rgb || a->grad_alpha || a->grad_textures ||
        a->grad_face_light)
        return NR_ERR_INVALID_ARG;
    memset(p, 0, sizeof(*p));
    int rc = nr_internal::soft_rgb_check(a, kSoftFragFlags, nr_internal::kSoftFragments, backward, &p->r);
    if (rc != NR_OK) return rc;
    p->K = K;
    if (backward) {
        p->ip2f = (const long long*)fa->pix_to_face;
        p->g_zbuf = fa->grad_zbuf; p->g_bary = fa->grad_bary; p->g_dists = fa->grad_dists;
    } else {
        p->p2f = (long long*)fa->pix_to_face;
        p->zbuf = fa->zbuf; p->bary = fa->bary; p->dists = fa->dists;
        const uintptr_t al = (uintptr_t)fa->pix_to_face | (uintptr_t)fa->zbuf | (uintptr_t)fa->bary | (uintptr_t)fa->dists;
        p->vec = K % 4 == 0 && (al & 15) == 0;
    }
    return nr_internal::soft_rgb_workspace(a, &p->r, L);
}

template <typename K>
void soft_frag_fwd_launch(const SoftFragParams& p, cudaStream_t s) {
    nr_internal::LaunchScope ls("k_soft_frag_fwd", s);
    const dim3 grid((unsigned)p.r.s.ntiles, (unsigned)p.r.s.B);
    if (p.K <= 4) k_soft_frag_fwd<K, 4><<<grid, kThreads, 0, s>>>(p);
    else if (p.K <= 8) k_soft_frag_fwd<K, 8><<<grid, kThreads, 0, s>>>(p);
    else if (p.K <= 16) k_soft_frag_fwd<K, 16><<<grid, kThreads, 0, s>>>(p);
    else k_soft_frag_fwd<K, 32><<<grid, kThreads, 0, s>>>(p);
}

}  // namespace

extern "C" int nr_b200_soft_fragments(const nr_b200_soft_rgb_args* args, const nr_b200_soft_frag_args* frag,
                                      void* cuda_stream) {
    SoftFragParams p;
    SoftRgbLayout L;
    const int rc = soft_frag_setup(args, frag, false, &p, &L);
    if (rc != NR_OK) return rc;
    cudaStream_t s = (cudaStream_t)cuda_stream;
    if (nr_internal::soft_rgb_bin(&p.r, &L, false, s) != NR_OK) return NR_ERR_CUDA;
    if (L.wide) soft_frag_fwd_launch<unsigned long long>(p, s);
    else soft_frag_fwd_launch<uint32_t>(p, s);
    return cudaGetLastError() == cudaSuccess ? NR_OK : NR_ERR_CUDA;
}

extern "C" int nr_b200_soft_fragments_backward(const nr_b200_soft_rgb_args* args, const nr_b200_soft_frag_args* frag,
                                               void* cuda_stream) {
    SoftFragParams p;
    SoftRgbLayout L;
    const int rc = soft_frag_setup(args, frag, true, &p, &L);
    if (rc != NR_OK) return rc;
    const nr_b200_soft_rgb_args* a = args;
    const bool indexed = (a->flags & NR_FACES_INDEXED) != 0;
    cudaStream_t s = (cudaStream_t)cuda_stream;
    if (!(a->flags & NR_GRAD_ACCUMULATE)) {
        nr_internal::prof_begin("memset_grads", s);
        const cudaError_t e = indexed ? cudaMemsetAsync(a->grad_vertices, 0, (size_t)p.r.s.B * a->num_vertices * 3 * sizeof(float), s)
                                      : cudaMemsetAsync(a->grad_faces, 0, (size_t)p.r.s.B * p.r.s.F * 9 * sizeof(float), s);
        nr_internal::prof_end(s);
        if (e != cudaSuccess) return NR_ERR_CUDA;
    }
    if (!frag->grad_zbuf && !frag->grad_bary && !frag->grad_dists)
        return cudaGetLastError() == cudaSuccess ? NR_OK : NR_ERR_CUDA;
    // the records and depth records of the binning; its lists are not read
    if (nr_internal::soft_rgb_bin(&p.r, &L, false, s) != NR_OK) return NR_ERR_CUDA;
    {
        nr_internal::LaunchScope ls("k_soft_frag_bwd", s);
        k_soft_frag_bwd<<<dim3((unsigned)p.r.s.ntiles, (unsigned)p.r.s.B), kThreads, 0, s>>>(p);
    }
    return cudaGetLastError() == cudaSuccess ? NR_OK : NR_ERR_CUDA;
}
