// nr_attr.cu -- attribute interpolation (nr_b200_interpolate / nr_b200_interpolate_backward, include/nr_b200.h).
//
// Renders C arbitrary channels, given per face corner or per vertex, into planar images through the maps an ordinary
// forward call already wrote (face_index_map, weight_map), with the winner's own vertex depths:
//
//   k_interp        one thread per API pixel (one pooled 2x2 quad with anti-aliasing).  zp and the perspective weights
//                   l_k are recomputed with the forward's expressions (nr_math.cuh), the attribute rows are gathered
//                   through L1 (neighbouring lanes mostly show the same face) and every channel is one coalesced,
//                   streaming store of a plane.
//   k_interp_grad   one thread per raster pixel, as k_depth_grad.  d loss / d attributes = l_k g_c is reduced with the
//                   CHANNELS across the lanes: the warp walks its runs of lanes that show the same face, lane c sums
//                   l_k(p) g_c(p) over the run's pixels p (the weights and the pixel's plane offset arrive by 4
//                   shuffles per pixel and 32 channels) and issues one atomic per corner and channel -- a warp's 32
//                   atomics hit one contiguous row of the corner / vertex, so the L2 sees a few requests per run, and no
//                   3C floats per pixel ever pass through shuffles.  The optional interior vertex gradient loops over
//                   the channels per pixel (no shuffles), leaving 9 floats that go through k_depth_grad's segmented
//                   run reduction before one set of atomics per run.
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include "nr_b200.h"
#include "nr_internal.h"
#include "nr_math.cuh"

namespace {

struct AttrParams {
    nr::FaceSrc src;
    nr::FaceGrad dst;      // grad_faces / grad_vertices of the vertex gradient (kVGrad only)
    const int32_t* fim;    // [B,S,S]
    const float* wmap;     // [B,3,S,S]
    const float* attr;     // [.,F,3,C] or [.,Nv,C]
    float* out;            // [B,C,H,W]
    const float* g;        // [B,C,H,W]
    float* gattr;          // layout of attr, or nullptr
    size_t attr_bstride;   // floats per item in attr / gattr (0 = shared)
    int S, C, Nv;
    int aa;
};

// first float of the attribute row of corner k of face f (item b): the corner slot, or the vertex slot face_indices[f,k];
// -1 for an index outside [0, Nv)
template <bool kPV>
__device__ __forceinline__ long long attr_row(const AttrParams& p, int b, int f, int k) {
    const size_t base = (size_t)b * p.attr_bstride;
    if (!kPV) return (long long)(base + ((size_t)f * 3 + k) * (size_t)p.C);
    const int i = __ldg(p.src.idx + (size_t)b * p.src.idx_bstride + (size_t)f * 3 + k);
    return (unsigned)i < (unsigned)p.Nv ? (long long)(base + (size_t)i * (size_t)p.C) : -1;
}

__device__ __forceinline__ float ld_or0(const float* a, long long row, int c) { return row >= 0 ? __ldg(a + row + c) : 0.0f; }

// out_c = fma(l2, a_2c, fma(l1, a_1c, l0 a_0c)): the chain of nr::corner_light_at
__device__ __forceinline__ float interp(const float l[3], float a0, float a1, float a2) {
    return __fmaf_rn(l[2], a2, __fmaf_rn(l[1], a1, __fmul_rn(l[0], a0)));
}

// ------------------------------------------------------------------------------------------------------- k_interp
template <bool kAA, bool kPV, bool kIdx>
__global__ void __launch_bounds__(256) k_interp(const __grid_constant__ AttrParams p) {
    const int S = p.S, H = kAA ? (S >> 1) : S;
    const size_t plane = (size_t)S * S, oplane = (size_t)H * H;
    const size_t o = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int b = blockIdx.y;
    if (o >= oplane) return;
    const int orow = (int)(o / H), ocol = (int)(o % H);
    constexpr int kQ = kAA ? 4 : 1;  // raster pixels of the API pixel: TL, TR, BL, BR
    float lam[kQ][3];
    long long row[kQ][3];
    bool cov[kQ];
#pragma unroll
    for (int q = 0; q < kQ; q++) {
        const int r = kAA ? 2 * orow + (q >> 1) : orow, c = kAA ? 2 * ocol + (q & 1) : ocol;
        const size_t i = (size_t)r * S + c;
        const int fn = __ldg(p.fim + (size_t)b * plane + i);
        cov[q] = fn >= 0;
#pragma unroll
        for (int k = 0; k < 3; k++) { lam[q][k] = 0.0f; row[q][k] = -1; }
        if (fn >= 0) {
            const float* wm = p.wmap + (size_t)b * 3 * plane + i;
            const float w[3] = {__ldg(wm), __ldg(wm + plane), __ldg(wm + 2 * plane)};
            const float z0 = __ldg(nr::face_vertex_t<kIdx>(p.src, b, fn, 0) + 2);
            const float z1 = __ldg(nr::face_vertex_t<kIdx>(p.src, b, fn, 1) + 2);
            const float z2 = __ldg(nr::face_vertex_t<kIdx>(p.src, b, fn, 2) + 2);
            nr::perspective_weights(w, nr::pixel_depth(w, z0, z1, z2), z0, z1, z2, lam[q]);
#pragma unroll
            for (int k = 0; k < 3; k++) row[q][k] = attr_row<kPV>(p, b, fn, k);
        }
    }
    float* out = p.out + (size_t)b * p.C * oplane + o;
    for (int c = 0; c < p.C; c++) {
        float s = 0.0f;
#pragma unroll
        for (int q = 0; q < kQ; q++) {
            const float v = cov[q] ? interp(lam[q], ld_or0(p.attr, row[q][0], c), ld_or0(p.attr, row[q][1], c),
                                             ld_or0(p.attr, row[q][2], c))
                                   : 0.0f;
            if (kAA) s += v; else s = v;  // the forward's pooling order, then * 0.25
        }
        __stcs(out + (size_t)c * oplane, kAA ? s * 0.25f : s);
    }
}

// -------------------------------------------------------------------------------------------------- k_interp_grad
template <bool kPV, bool kIdx, bool kVGrad>
__global__ void __launch_bounds__(256) k_interp_grad(const __grid_constant__ AttrParams p) {
    const int S = p.S, C = p.C;
    const size_t plane = (size_t)S * S;
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int b = blockIdx.y;
    const int lane = threadIdx.x & 31;
    const int fn = (i < plane) ? __ldg(p.fim + (size_t)b * plane + i) : -1;
    if (!__any_sync(0xffffffffu, fn >= 0)) return;  // warp-uniform
    const bool aa = p.aa != 0;
    const int H = aa ? (S >> 1) : S;
    const size_t gplane = (size_t)H * H;
    const float gscale = aa ? 0.25f : 1.0f;  // the pooling backward: each raster pixel gets g / 4 (load_grad)
    const float* gb = p.g + (size_t)b * C * gplane;
    float lam[3] = {0.0f, 0.0f, 0.0f};
    uint32_t goff = 0;  // the pixel's offset within a plane of the upstream gradient (S <= 32767)
    float vg[kVGrad ? 9 : 1];
#pragma unroll
    for (int k = 0; k < (kVGrad ? 9 : 1); k++) vg[k] = 0.0f;
    if (fn >= 0) {
        const int r = (int)(i / S), c = (int)(i % S);
        goff = aa ? (uint32_t)(r >> 1) * (uint32_t)H + (uint32_t)(c >> 1) : (uint32_t)i;
        const float* wm = p.wmap + (size_t)b * 3 * plane + i;
        const float w[3] = {__ldg(wm), __ldg(wm + plane), __ldg(wm + 2 * plane)};
        if constexpr (kVGrad) {
            float v[9];
            nr::load_face(p.src, b, fn, v);
            const float z[3] = {v[2], v[5], v[8]};
            const float zp = nr::pixel_depth(w, z[0], z[1], z[2]);
            nr::perspective_weights(w, zp, z[0], z[1], z[2], lam);
            const float fS = (float)S;
            float inv[9];
            nr::face_inverse(nr::to_pixel(v[0], fS), nr::to_pixel(v[1], fS), nr::to_pixel(v[3], fS), nr::to_pixel(v[4], fS),
                             nr::to_pixel(v[6], fS), nr::to_pixel(v[7], fS), inv);
            // d l_k / d(x, y) in raster pixels (nr::mip_lod): zp (q_k - l_k sum_j q_j), q_k = inv[3k (+1)] / z_k
            float qx[3], qy[3];
#pragma unroll
            for (int k = 0; k < 3; k++) { qx[k] = __fdiv_rn(inv[3 * k], z[k]); qy[k] = __fdiv_rn(inv[3 * k + 1], z[k]); }
            const float sx = (qx[0] + qx[1]) + qx[2], sy = (qy[0] + qy[1]) + qy[2];
            const float lx1 = zp * (qx[1] - lam[1] * sx), lx2 = zp * (qx[2] - lam[2] * sx);
            const float ly1 = zp * (qy[1] - lam[1] * sy), ly2 = zp * (qy[2] - lam[2] * sy);
            const long long a0r = attr_row<kPV>(p, b, fn, 0), a1r = attr_row<kPV>(p, b, fn, 1), a2r = attr_row<kPV>(p, b, fn, 2);
            // D_k = sum_c g_c (a_kc - a_0c) (differences against corner 0, as mip_lod), P_m = sum_c g_c (out_c - a_mc)
            float D1 = 0.0f, D2 = 0.0f, P0 = 0.0f, P1 = 0.0f, P2 = 0.0f;
            for (int ch = 0; ch < C; ch++) {
                const float g = __ldg(gb + (size_t)ch * gplane + goff) * gscale;
                const float a0 = ld_or0(p.attr, a0r, ch), a1 = ld_or0(p.attr, a1r, ch), a2 = ld_or0(p.attr, a2r, ch);
                const float o = interp(lam, a0, a1, a2);
                D1 += g * (a1 - a0); D2 += g * (a2 - a0);
                P0 += g * (o - a0); P1 += g * (o - a1); P2 += g * (o - a2);
            }
            const float Gx = D1 * lx1 + D2 * lx2, Gy = D1 * ly1 + D2 * ly2;
            const float half_s = fS * 0.5f;
            const float P[3] = {P0, P1, P2};
#pragma unroll
            for (int m = 0; m < 3; m++) {
                vg[3 * m] = -w[m] * Gx * half_s;
                vg[3 * m + 1] = -w[m] * Gy * half_s;
                vg[3 * m + 2] = __fdiv_rn(lam[m], z[m]) * P[m];
            }
        } else {
            const float z0 = __ldg(nr::face_vertex_t<kIdx>(p.src, b, fn, 0) + 2);
            const float z1 = __ldg(nr::face_vertex_t<kIdx>(p.src, b, fn, 1) + 2);
            const float z2 = __ldg(nr::face_vertex_t<kIdx>(p.src, b, fn, 2) + 2);
            nr::perspective_weights(w, nr::pixel_depth(w, z0, z1, z2), z0, z1, z2, lam);
        }
    }
    // runs of neighbouring lanes that show the same face (a warp = 32 consecutive pixels of a row)
    const int fn_prev = __shfl_up_sync(0xffffffffu, fn, 1);
    const uint32_t heads = __ballot_sync(0xffffffffu, lane == 0 || fn != fn_prev);
    if (p.gattr) {
        // d loss / d attributes, channels across lanes: per run, lane c accumulates sum_p l_k(p) g_c(p) for c = c0 + lane
        uint32_t todo = heads & __ballot_sync(0xffffffffu, fn >= 0);
        while (todo) {  // warp-uniform
            const int h = __ffs(todo) - 1;
            todo &= todo - 1u;
            const uint32_t later = heads & ~((2u << h) - 1u);
            const int e = later ? __ffs(later) - 2 : 31;
            const int f = __shfl_sync(0xffffffffu, fn, h);
            const long long r0 = attr_row<kPV>(p, b, f, 0), r1 = attr_row<kPV>(p, b, f, 1), r2 = attr_row<kPV>(p, b, f, 2);
            for (int c0 = 0; c0 < C; c0 += 32) {
                const int ch = c0 + lane;
                const float* gc = gb + (size_t)(ch < C ? ch : 0) * gplane;
                float acc0 = 0.0f, acc1 = 0.0f, acc2 = 0.0f;
                for (int q = h; q <= e; q++) {
                    const float l0 = __shfl_sync(0xffffffffu, lam[0], q), l1 = __shfl_sync(0xffffffffu, lam[1], q),
                                l2 = __shfl_sync(0xffffffffu, lam[2], q);
                    const uint32_t go = __shfl_sync(0xffffffffu, goff, q);
                    if (ch < C) {
                        const float g = __ldg(gc + go) * gscale;
                        acc0 += l0 * g; acc1 += l1 * g; acc2 += l2 * g;
                    }
                }
                if (ch < C) {
                    if (r0 >= 0) atomicAdd(p.gattr + r0 + ch, acc0);
                    if (r1 >= 0) atomicAdd(p.gattr + r1 + ch, acc1);
                    if (r2 >= 0) atomicAdd(p.gattr + r2 + ch, acc2);
                }
            }
        }
    }
    if constexpr (kVGrad) {
        // the 9 floats of k_depth_grad's segmented run reduction, then one set of atomics per run
        const uint32_t later = heads & ~((2u << lane) - 1u);
        const int run_end = (lane == 31 || later == 0) ? 31 : (__ffs(later) - 2);
#pragma unroll
        for (int off = 1; off < 32; off <<= 1) {
            const bool take = lane + off <= run_end;
#pragma unroll
            for (int k = 0; k < 9; k++) {
                const float t = __shfl_down_sync(0xffffffffu, vg[k], off);
                if (take) vg[k] += t;
            }
        }
        if (fn >= 0 && ((heads >> lane) & 1u)) {
#pragma unroll
            for (int k = 0; k < 3; k++) {
                float* gv = nr::face_grad_vertex_t<kIdx>(p.dst, b, fn, k);
                if (gv) { atomicAdd(gv, vg[3 * k]); atomicAdd(gv + 1, vg[3 * k + 1]); atomicAdd(gv + 2, vg[3 * k + 2]); }
            }
        }
    }
}

template <bool kAA>
void launch_interp(const AttrParams& p, bool pv, bool idx, dim3 grid, cudaStream_t s) {
    nr_internal::LaunchScope ls("k_interp", s);
    if (pv) k_interp<kAA, true, true><<<grid, 256, 0, s>>>(p);
    else if (idx) k_interp<kAA, false, true><<<grid, 256, 0, s>>>(p);
    else k_interp<kAA, false, false><<<grid, 256, 0, s>>>(p);
}

template <bool kVGrad>
void launch_interp_grad(const AttrParams& p, bool pv, bool idx, dim3 grid, cudaStream_t s) {
    nr_internal::LaunchScope ls("k_interp_grad", s);
    if (pv) k_interp_grad<true, true, kVGrad><<<grid, 256, 0, s>>>(p);
    else if (idx) k_interp_grad<false, true, kVGrad><<<grid, 256, 0, s>>>(p);
    else k_interp_grad<false, false, kVGrad><<<grid, 256, 0, s>>>(p);
}

// the host checks of both entry points; fills `p` (and the attribute row count per item) on success
int interp_setup(const nr_b200_interpolate_args* args, bool backward, AttrParams* p, size_t* attr_rows) {
    nr_internal::launch_count() = 0;
    if (!args || args->struct_size != sizeof(nr_b200_interpolate_args)) return NR_ERR_INVALID_ARG;
    const nr_b200_interpolate_args* a = args;
    const uint32_t flags = a->flags;
    const int B = a->batch_size, F = a->num_faces, S = a->raster_size, C = a->channels;
    if (B <= 0 || F <= 0 || S <= 0 || C < 1) return NR_ERR_INVALID_ARG;
    if (!a->face_index_map || !a->weight_map || !a->attributes) return NR_ERR_INVALID_ARG;
    const bool indexed = (flags & NR_FACES_INDEXED) != 0, pv = (flags & NR_ATTR_PER_VERTEX) != 0;
    if (pv && !indexed) return NR_ERR_INVALID_ARG;
    if ((flags & NR_ANTI_ALIASING) && (S & 1)) return NR_ERR_INVALID_ARG;
    // grid.y = B; 32-bit plane offsets of the upstream gradient
    if (S > 32767 || B > 65535) return NR_ERR_INVALID_ARG;
    memset(p, 0, sizeof(*p));
    if (!nr_internal::make_face_src(flags, a->faces, a->vertices, a->face_indices, F, a->num_vertices, &p->src))
        return NR_ERR_INVALID_ARG;
    if (!backward && !a->out) return NR_ERR_INVALID_ARG;
    if (backward) {
        if (indexed ? a->grad_faces != nullptr : a->grad_vertices != nullptr) return NR_ERR_INVALID_ARG;
        const bool vgrad = indexed ? a->grad_vertices != nullptr : a->grad_faces != nullptr;
        if (vgrad && !nr_internal::make_face_grad(flags, a->grad_faces, a->grad_vertices, a->face_indices, F, a->num_vertices, &p->dst))
            return NR_ERR_INVALID_ARG;
    }
    *attr_rows = pv ? (size_t)a->num_vertices : (size_t)F * 3;
    p->fim = a->face_index_map; p->wmap = a->weight_map; p->attr = a->attributes; p->out = a->out;
    p->g = a->grad_out; p->gattr = a->grad_attributes;
    p->attr_bstride = (flags & NR_ATTR_SHARED) ? 0 : *attr_rows * (size_t)C;
    p->S = S; p->C = C; p->Nv = a->num_vertices;
    p->aa = (flags & NR_ANTI_ALIASING) ? 1 : 0;
    return NR_OK;
}

}  // namespace

extern "C" int nr_b200_interpolate(const nr_b200_interpolate_args* args, void* cuda_stream) {
    AttrParams p;
    size_t rows = 0;
    const int rc = interp_setup(args, false, &p, &rows);
    if (rc != NR_OK) return rc;
    const int H = p.aa ? p.S / 2 : p.S;
    const dim3 grid((unsigned)(((size_t)H * H + 255) / 256), args->batch_size);
    cudaStream_t s = (cudaStream_t)cuda_stream;
    const bool pv = (args->flags & NR_ATTR_PER_VERTEX) != 0, idx = (args->flags & NR_FACES_INDEXED) != 0;
    if (p.aa) launch_interp<true>(p, pv, idx, grid, s);
    else launch_interp<false>(p, pv, idx, grid, s);
    return cudaGetLastError() == cudaSuccess ? NR_OK : NR_ERR_CUDA;
}

extern "C" int nr_b200_interpolate_backward(const nr_b200_interpolate_args* args, void* cuda_stream) {
    AttrParams p;
    size_t rows = 0;
    const int rc = interp_setup(args, true, &p, &rows);
    if (rc != NR_OK) return rc;
    const nr_b200_interpolate_args* a = args;
    const int B = a->batch_size, F = a->num_faces;
    const bool indexed = (a->flags & NR_FACES_INDEXED) != 0, pv = (a->flags & NR_ATTR_PER_VERTEX) != 0;
    const bool vgrad = indexed ? a->grad_vertices != nullptr : a->grad_faces != nullptr;
    cudaStream_t s = (cudaStream_t)cuda_stream;
    if (!(a->flags & NR_GRAD_ACCUMULATE)) {
        nr_internal::prof_begin("memset_grads", s);
        const size_t items = (a->flags & NR_ATTR_SHARED) ? 1 : (size_t)B;
        if (p.gattr && cudaMemsetAsync(p.gattr, 0, items * rows * (size_t)a->channels * sizeof(float), s) != cudaSuccess)
            return NR_ERR_CUDA;
        if (vgrad) {
            const cudaError_t e = indexed ? cudaMemsetAsync(a->grad_vertices, 0, (size_t)B * a->num_vertices * 3 * sizeof(float), s)
                                          : cudaMemsetAsync(a->grad_faces, 0, (size_t)B * F * 9 * sizeof(float), s);
            if (e != cudaSuccess) return NR_ERR_CUDA;
        }
        nr_internal::prof_end(s);
    }
    if (!a->grad_out || (!p.gattr && !vgrad)) return cudaGetLastError() == cudaSuccess ? NR_OK : NR_ERR_CUDA;
    const dim3 grid((unsigned)(((size_t)p.S * p.S + 255) / 256), B);
    if (vgrad) launch_interp_grad<true>(p, pv, indexed, grid, s);
    else launch_interp_grad<false>(p, pv, indexed, grid, s);
    return cudaGetLastError() == cudaSuccess ? NR_OK : NR_ERR_CUDA;
}
