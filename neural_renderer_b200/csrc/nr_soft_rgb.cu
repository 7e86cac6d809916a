// nr_soft_rgb.cu -- soft RGB (nr_b200_soft_rgb / nr_b200_soft_rgb_backward, include/nr_b200.h): SoftRas colour
// aggregation over every face within reach, on the tile binning of the soft silhouettes (nr_soft.cuh).
//
// nr_b200_soft_rgb / nr_b200_soft_rgb_backward reuse k_soft_setup, k_strip_scan and soft_eval, and add:
//   k_soft_rgb_keys   the forward only: every list entry gets its item's sentinel key (past every segment of the item)
//   k_soft_rgb_fill   one thread per face with a tile box: the depth record {z0, z1, z2, A} and one composite key
//                     (segment << fbits) | f per tile it counted into (atomic cursors, so in arbitrary order)
//   soft_rgb_sort     the forward only: cub::DeviceRadixSort::SortKeys over the whole list; the sentinels keep each
//                     item's entries inside its own list range, so the offsets of k_strip_scan stay valid
//   k_soft_rgb_fwd    one CTA per (tile, item): faces staged in list order (block-wide scan of the box-test ballot), a
//                     running-max softmax per pixel in that order -- the forward is bit-for-bit repeatable
//   k_soft_rgb_bwd    the same traversal of the unsorted lists: 12 partials per face (x, y, z of three vertices, three
//                     light channels) reduced over the warp and the CTA; the 8-tap texture scatters of a warp merged in a
//                     per-warp shared-memory cube when ts^3 3 <= kWarpCube, then flushed to global memory
// The forward traversal is nr_soft_rgb.cuh's, with the cube sampler below.  The host checks, the workspace layout and
// the binning are shared with nr_soft_uv.cu through nr_internal.h.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <string.h>

#include <cub/device/device_radix_sort.cuh>

#include "nr_b200.h"
#include "nr_internal.h"
#include "nr_soft.cuh"
#include "nr_soft_rgb.cuh"
#include "nr_texture.cuh"

namespace {

constexpr int kWarpCube = 384;   // floats of a warp's texture-gradient cube (ts <= 5)

template <typename K>
__global__ void __launch_bounds__(256) k_soft_rgb_keys(const __grid_constant__ SoftRgbParams p) {
    const long long per_item = (long long)p.s.F * kWideTiles, n = per_item * p.s.B;
    K* keys = (K*)p.keys;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const long long b = i / per_item;
        keys[i] = ((K)((b + 1) * (p.s.ntiles + 1)) << p.fbits) - 1;
    }
}

template <typename K>
__global__ void __launch_bounds__(256) k_soft_rgb_fill(const __grid_constant__ SoftRgbParams p) {
    const int b = blockIdx.y;
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= p.s.F) return;
    const size_t id = (size_t)b * p.s.F + f;
    const uint2 bb = __ldg(p.s.box + id);
    const int tx0 = lo16(bb.x), tx1 = hi16(bb.x), ty0 = lo16(bb.y), ty1 = hi16(bb.y);
    if (tx0 > tx1) return;
    float v[9];
    nr::load_face(p.s.src, b, f, v);
    // plain products: a face whose vertices are exactly collinear in x, y (or coincide) gets exactly A = 0
    const float A = __fsub_rn(__fmul_rn(__fsub_rn(v[3], v[0]), __fsub_rn(v[7], v[1])),
                              __fmul_rn(__fsub_rn(v[4], v[1]), __fsub_rn(v[6], v[0])));
    p.zrec[id] = make_float4(v[2], v[5], v[8], A);
    const int nt1 = p.s.ntiles + 1;
    int* seg = p.s.cursor + (size_t)b * nt1;
    const int* segoff = p.s.off + (size_t)b * nt1;
    K* keys = (K*)p.keys;
    const int w = tx1 - tx0 + 1, n = w * (ty1 - ty0 + 1);
    for (int i = 0; i < (n > kWideTiles ? 1 : n); i++) {
        const int t = n > kWideTiles ? p.s.ntiles : (ty0 + i / w) * p.s.ntx + tx0 + i % w;
        const int pos = atomicAdd(seg + t, 1);
        keys[segoff[t] + pos] = ((K)((size_t)b * nt1 + t) << p.fbits) | (K)f;
    }
}

// the forward colour of the per-face cubes: the trilinear sample at texture_coords(l, zp, z)
struct CubeSampler {
    __device__ __forceinline__ void color(const SoftRgbParams& p, int b, int f, const SoftBary& bc, const float4& z,
                                          const float4*, float& r, float& g, float& bl) const {
        const int ts = p.ts;
        const nr::TexCoord tc = nr::texture_coords(bc.l, bc.zp, z.x, z.y, z.z, ts, p.tex.tex_cmp, p.tex.tex_val);
        const float* cube = p.tex.tex + p.tex.cube_off(b, f, ts);
        if (p.light) nr::cube_blend<true, true>(cube, tc, ts, false, p.light + ((size_t)b * p.s.F + f) * 3, r, g, bl);
        else nr::cube_blend<false, true>(cube, tc, ts, false, nullptr, r, g, bl);
    }
};

// ------------------------------------------------------------------------------------------------ k_soft_rgb_fwd
template <typename K>
__global__ void __launch_bounds__(kThreads) k_soft_rgb_fwd(const __grid_constant__ SoftRgbParams p) {
    __shared__ float4 s_rec[kThreads * 4];
    __shared__ float4 s_z[kThreads];
    __shared__ int s_face[kThreads];
    __shared__ int s_wn[kWarps];
    soft_rgb_fwd_body<K>(p, CubeSampler{}, s_rec, s_z, s_face, s_wn);
}

// ------------------------------------------------------------------------------------------------ k_soft_rgb_bwd
constexpr int kRgbPartials = 12;  // per face: (x, y) of 3 vertices, z of 3 vertices, 3 light channels

template <typename K>
__global__ void __launch_bounds__(kThreads) k_soft_rgb_bwd(const __grid_constant__ SoftRgbParams p) {
    __shared__ float4 s_rec[kThreads * 4];
    __shared__ float4 s_z[kThreads];
    __shared__ int s_face[kThreads];
    __shared__ float s_acc[kThreads * kRgbPartials];
    __shared__ float s_cube[kWarps * kWarpCube];
    __shared__ int s_wn[kWarps];
    const int tile = blockIdx.x, b = blockIdx.y;
    const int tx = tile % p.s.ntx, ty = tile / p.s.ntx;
    const int col = tx * kTile + (threadIdx.x % kTile), row = ty * kTile + (threadIdx.x / kTile);
    const int S = p.s.S, ts = p.ts, lane = threadIdx.x & 31;
    const float px = soft_centre(col, S), py = soft_centre(S - 1 - row, S);
    const size_t seg = (size_t)b * (p.s.ntiles + 1);
    const int n_tile = p.s.cnt[seg + tile], n_all = n_tile + p.s.cnt[seg + p.s.ntiles];
    if (n_all == 0) return;  // CTA-uniform
    const int n3 = ts * ts * ts * 3;
    const bool warp_cube = p.grad_tex != nullptr && n3 <= kWarpCube;
    float* my_cube = s_cube + (threadIdx.x >> 5) * kWarpCube;
    float ga = 0.0f, gr[3] = {0.0f, 0.0f, 0.0f}, out[3] = {0.0f, 0.0f, 0.0f}, Z = 1.0f, zref = 0.0f;
    if (row < S && col < S) {
        const size_t plane = (size_t)S * S, o = (size_t)row * S + col;
        if (p.s.g) ga = __ldg(p.s.g + b * plane + o) * (1.0f - __ldg(p.s.alpha + b * plane + o));
        if (p.g_rgb) {
#pragma unroll
            for (int c = 0; c < 3; c++) {
                gr[c] = __ldg(p.g_rgb + ((size_t)b * 3 + c) * plane + o);
                out[c] = __ldg(p.rgb + ((size_t)b * 3 + c) * plane + o);
            }
        }
        Z = __ldg(p.state + (size_t)b * 2 * plane + o);
        zref = __ldg(p.state + (size_t)b * 2 * plane + plane + o);
    }
    const float iZ = __frcp_rn(Z);
    const bool want_rgb = gr[0] != 0.0f || gr[1] != 0.0f || gr[2] != 0.0f;
    const bool active = ga != 0.0f || want_rgb;
    // h = g . (C - rgb) / Z = (g . C) / Z - (g . rgb) / Z
    const float g_out = __fmul_rn(__fmaf_rn(gr[2], out[2], __fmaf_rn(gr[1], out[1], __fmul_rn(gr[0], out[0]))), iZ);
    for (int i = threadIdx.x; i < kThreads * kRgbPartials; i += kThreads) s_acc[i] = 0.0f;
    for (int i = threadIdx.x; i < kWarps * kWarpCube; i += kThreads) s_cube[i] = 0.0f;
    for (int next = 0; next < n_all; next += kThreads) {
        const int n = stage_rgb<K>(p, b, tile, tx, ty, n_tile, n_all, next, s_rec, s_z, s_face, s_wn);
        for (int j = 0; j < n; j++) {
            float x = 0.0f, t = 0.0f, qx = 0.0f, qy = 0.0f, c[3];
            int k = 0;
            const bool hit = active && soft_eval(s_rec + 4 * j, px, py, p.s.inv_sigma, p.s.cut, x, k, t, qx, qy, c);
            if (!__any_sync(0xffffffffu, hit)) continue;  // warp-uniform
            const int f = s_face[j];
            float v[kRgbPartials];
#pragma unroll
            for (int m = 0; m < kRgbPartials; m++) v[m] = 0.0f;
            bool tex_hit = false;
            nr::TexCoord tc;
            float gl[3] = {0.0f, 0.0f, 0.0f};  // d loss / d tap = gl_c * corner weight
            if (hit) {
                const float D = soft_sigmoid(x);
                float gx = __fmul_rn(ga, D);  // d loss / d x_j
                const float4 z = s_z[j];
                if (want_rgb && z.w != 0.0f) {
                    const SoftBary bc = soft_bary(c, z);
                    const float w = __fmul_rn(D, expf(__fmul_rn(__fsub_rn(zref, bc.zp), p.inv_fg)));
                    if (w != 0.0f) {
                        const float zz[3] = {z.x, z.y, z.z};
                        tc = nr::texture_coords(bc.l, bc.zp, z.x, z.y, z.z, ts, p.tex.tex_cmp, p.tex.tex_val);
                        float su[3], dt[3][3], L[3] = {1.0f, 1.0f, 1.0f};
                        nr::cube_blend_axis_grad(p.tex.tex + p.tex.cube_off(b, f, ts), tc, ts, false, su, dt);
                        if (p.light) {
                            const float* lt = p.light + ((size_t)b * p.s.F + f) * 3;
                            L[0] = __ldg(lt); L[1] = __ldg(lt + 1); L[2] = __ldg(lt + 2);
                        }
                        const float gC = __fmaf_rn(gr[2], __fmul_rn(su[2], L[2]),
                                                   __fmaf_rn(gr[1], __fmul_rn(su[1], L[1]), __fmul_rn(gr[0], __fmul_rn(su[0], L[0]))));
                        const float h = __fsub_rn(__fmul_rn(gC, iZ), g_out);
                        gx = __fmaf_rn(__fmul_rn(w, 1.0f - D), h, gx);
                        float dzp = -__fmul_rn(__fmul_rn(w, h), p.inv_fg);  // d loss / d zp through the weight
                        const float wz = __fmul_rn(w, iZ);
#pragma unroll
                        for (int ch = 0; ch < 3; ch++) {
                            const float gCc = __fmul_rn(wz, gr[ch]);  // d loss / d C_c
                            v[9 + ch] = __fmul_rn(gCc, su[ch]);
                            gl[ch] = __fmul_rn(gCc, L[ch]);
                        }
                        tex_hit = p.grad_tex != nullptr;
                        // texture coordinates t_k = l_k (ts - 1) zp / z_k, gated by their clamp; the cell held fixed
                        const float fts1 = (float)(ts - 1);
                        float dl[3], dz[3];
#pragma unroll
                        for (int a = 0; a < 3; a++) {
                            const float r = __fdiv_rn(bc.zp, zz[a]);
                            const float tk = __fmul_rn(__fmul_rn(bc.l[a], fts1), r);
                            const bool in = tk >= 0.0f && tk <= p.tex.tex_cmp;
                            const float Gt = in ? __fmul_rn(__fmaf_rn(gl[2], dt[a][2], __fmaf_rn(gl[1], dt[a][1], __fmul_rn(gl[0], dt[a][0]))), fts1) : 0.0f;
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
                        const float4* r = s_rec + 4 * j;
#pragma unroll
                        for (int e = 0; e < 3; e++) {
                            const float dc = __fdiv_rn(__fsub_rn(dlam[e == 0 ? 2 : e - 1], sg), z.w);
                            const float4 ed = r[e];
                            const float dx = __fsub_rn(px, ed.x), dy = __fsub_rn(py, ed.y);
                            const int nb = e == 2 ? 0 : e + 1;
                            v[2 * e] = __fmaf_rn(dc, __fsub_rn(ed.w, dy), v[2 * e]);
                            v[2 * e + 1] = __fmaf_rn(dc, __fsub_rn(dx, ed.z), v[2 * e + 1]);
                            v[2 * nb] = __fmaf_rn(dc, dy, v[2 * nb]);
                            v[2 * nb + 1] = __fmaf_rn(dc, -dx, v[2 * nb + 1]);
                        }
                    }
                }
                // d x / d(d^2) = +-1/sigma; d(d^2)/da = -2 (1 - t)(p - q), d(d^2)/db = -2 t (p - q) for edge (a, b)
                const float s = gx * (x >= 0.0f ? -2.0f : 2.0f) * p.s.inv_sigma;
                const float wa = s * (1.0f - t), wb = s * t;
#pragma unroll
                for (int m = 0; m < 3; m++) {
                    const bool is_a = m == k, is_b = m == (k == 2 ? 0 : k + 1);
                    const float wm = is_a ? wa : (is_b ? wb : 0.0f);
                    v[2 * m] = __fmaf_rn(wm, qx, v[2 * m]);
                    v[2 * m + 1] = __fmaf_rn(wm, qy, v[2 * m + 1]);
                }
            }
            // the texture taps: merged per warp in shared memory, or straight to global memory past the budget
            const bool any_tex = __any_sync(0xffffffffu, tex_hit);
            if (any_tex) {
                float* gcube = p.grad_tex + p.tex.cube_off(b, f, ts);
                if (tex_hit) {
#pragma unroll
                    for (int pn = 0; pn < 8; pn++) {
                        const float cw = nr::corner_weight(tc, pn);
                        const int ci = nr::corner_index(tc, pn, ts) * 3;
#pragma unroll
                        for (int ch = 0; ch < 3; ch++) {
                            const float gt = __fmul_rn(gl[ch], cw);
                            if (gt == 0.0f) continue;
                            if (warp_cube) atomicAdd(my_cube + ci + ch, gt);
                            else atomicAdd(gcube + ci + ch, gt);
                        }
                    }
                }
                if (warp_cube) {
                    __syncwarp();
                    for (int e = lane; e < n3; e += 32) {
                        const float gv = my_cube[e];
                        if (gv != 0.0f) { atomicAdd(gcube + e, gv); my_cube[e] = 0.0f; }
                    }
                    __syncwarp();
                }
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1)
#pragma unroll
                for (int m = 0; m < kRgbPartials; m++) v[m] += __shfl_xor_sync(0xffffffffu, v[m], o);
            if (lane < kRgbPartials) {
                float mine = v[0];
#pragma unroll
                for (int m = 1; m < kRgbPartials; m++) if (lane == m) mine = v[m];
                if (mine != 0.0f) atomicAdd(&s_acc[j * kRgbPartials + lane], mine);
            }
        }
        __syncthreads();
        // one set of global atomics per face of the round: thread (face slot, vertex or light)
        for (int i = threadIdx.x; i < n * 4; i += kThreads) {
            const int j = i / 4, m = i % 4;
            float* a = s_acc + j * kRgbPartials;
            if (m < 3) {
                const float gx = a[2 * m], gy = a[2 * m + 1], gz = a[6 + m];
                a[2 * m] = 0.0f; a[2 * m + 1] = 0.0f; a[6 + m] = 0.0f;
                if (gx == 0.0f && gy == 0.0f && gz == 0.0f) continue;
                float* gv = nr::face_grad_vertex(p.s.dst, b, s_face[j], m);
                if (gv) { atomicAdd(gv, gx); atomicAdd(gv + 1, gy); atomicAdd(gv + 2, gz); }
            } else {
                const float l0 = a[9], l1 = a[10], l2 = a[11];
                a[9] = 0.0f; a[10] = 0.0f; a[11] = 0.0f;
                if (!p.grad_light || (l0 == 0.0f && l1 == 0.0f && l2 == 0.0f)) continue;
                float* gl = p.grad_light + ((size_t)b * p.s.F + s_face[j]) * 3;
                atomicAdd(gl, l0); atomicAdd(gl + 1, l1); atomicAdd(gl + 2, l2);
            }
        }
        __syncthreads();
    }
}

template <typename K>
bool sort_temp_bytes(size_t n, int end_bit, size_t* bytes) {
    *bytes = 0;
    return cub::DeviceRadixSort::SortKeys(nullptr, *bytes, (const K*)nullptr, (K*)nullptr, (int)n, 0, end_bit) == cudaSuccess;
}

// false: sizes the kernels cannot index, or CUB could not size its scratch (it asks the current device)
bool soft_rgb_layout(int B, int F, int S, SoftRgbLayout* L) {
    if (!soft_sizes_ok(B, F, S)) return false;
    L->s = soft_layout(B, F, S);
    const size_t nt1 = (size_t)tiles_per_axis(S) * tiles_per_axis(S) + 1, cap = (size_t)B * F * kWideTiles;
    L->fbits = 1;
    while (((size_t)1 << L->fbits) <= (size_t)F) L->fbits++;              // f <= 2^fbits - 2 < the sentinel's low bits
    const unsigned long long max_key = ((unsigned long long)(B * nt1) << L->fbits) - 1;  // the last item's sentinel
    L->end_bit = 1;
    while (L->end_bit < 64 && (max_key >> L->end_bit) != 0) L->end_bit++;
    L->wide = L->end_bit > 32;
    const size_t ksz = L->wide ? 8 : 4;
    if (!(L->wide ? sort_temp_bytes<unsigned long long>(cap, L->end_bit, &L->temp_bytes)
                  : sort_temp_bytes<uint32_t>(cap, L->end_bit, &L->temp_bytes)))
        return false;
    // the silhouettes' int lists are not used: the keys take their place
    L->zrec = L->s.list;
    L->keys = L->zrec + align256((size_t)B * F * sizeof(float4));
    L->keys_out = L->keys + align256(cap * ksz);
    L->temp = L->keys_out + align256(cap * ksz);
    L->total = L->temp + align256(L->temp_bytes);
    return true;
}

constexpr uint32_t kSoftRgbFlags = NR_FACES_INDEXED | NR_INDICES_SHARED | NR_TEX_SHARED | NR_GRAD_ACCUMULATE;

// the silhouettes' setup and scan, then the depth records and keys (the forward: sentinels first, sorted after)
template <typename K>
int bin_faces_rgb(SoftRgbParams& p, const SoftRgbLayout& L, bool sort, cudaStream_t s) {
    const SoftParams& q = p.s;
    nr_internal::prof_begin("memset_soft_bins", s);
    if (cudaMemsetAsync(q.cnt, 0, 2 * (size_t)q.B * (q.ntiles + 1) * sizeof(int), s) != cudaSuccess) return NR_ERR_CUDA;
    nr_internal::prof_end(s);
    const dim3 grid((unsigned)((q.F + 255) / 256), (unsigned)q.B);
    {
        nr_internal::LaunchScope ls("k_soft_setup", s);
        k_soft_setup<false><<<grid, 256, 0, s>>>(q);
    }
    nr_internal::strip_scan(q.cnt, q.off, q.ntiles + 1, (long long)q.F * kWideTiles, q.B, s);
    const size_t cap = (size_t)q.B * q.F * kWideTiles;
    if (sort) {
        nr_internal::LaunchScope ls("k_soft_rgb_keys", s);
        const size_t blocks = (cap + 255) / 256;
        k_soft_rgb_keys<K><<<(unsigned)(blocks < (1u << 20) ? blocks : (1u << 20)), 256, 0, s>>>(p);
    }
    {
        nr_internal::LaunchScope ls("k_soft_rgb_fill", s);
        k_soft_rgb_fill<K><<<grid, 256, 0, s>>>(p);
    }
    if (sort) {
        nr_internal::LaunchScope ls("soft_rgb_sort", s);
        char* ws = (char*)p.keys - L.keys;
        size_t temp = L.temp_bytes;
        if (cub::DeviceRadixSort::SortKeys(ws + L.temp, temp, (const K*)p.keys, (K*)(ws + L.keys_out), (int)cap, 0, L.end_bit,
                                           s) != cudaSuccess)
            return NR_ERR_CUDA;
        p.keys = ws + L.keys_out;
    }
    return NR_OK;
}

template <typename K>
int soft_rgb_forward(SoftRgbParams& p, const SoftRgbLayout& L, cudaStream_t s) {
    if (nr_internal::soft_rgb_bin(&p, &L, true, s) != NR_OK) return NR_ERR_CUDA;
    nr_internal::LaunchScope ls("k_soft_rgb_fwd", s);
    k_soft_rgb_fwd<K><<<dim3((unsigned)p.s.ntiles, (unsigned)p.s.B), kThreads, 0, s>>>(p);
    return NR_OK;
}

template <typename K>
int soft_rgb_backward(SoftRgbParams& p, const SoftRgbLayout& L, cudaStream_t s) {
    if (nr_internal::soft_rgb_bin(&p, &L, false, s) != NR_OK) return NR_ERR_CUDA;
    nr_internal::LaunchScope ls("k_soft_rgb_bwd", s);
    k_soft_rgb_bwd<K><<<dim3((unsigned)p.s.ntiles, (unsigned)p.s.B), kThreads, 0, s>>>(p);
    return NR_OK;
}

}  // namespace

namespace nr_internal {

int soft_rgb_check(const nr_b200_soft_rgb_args* a, uint32_t allowed, SoftColourSource src, bool backward, void* params) {
    SoftRgbParams* p = (SoftRgbParams*)params;
    const bool cubes = src == kSoftCubes, colour = src != kSoftAttributes && src != kSoftFragments;
    const bool softmax = src != kSoftFragments;
    if (!a || a->struct_size != sizeof(nr_b200_soft_rgb_args)) return NR_ERR_INVALID_ARG;
    const uint32_t flags = a->flags;
    if (flags & ~allowed) return NR_ERR_INVALID_ARG;
    const int B = a->batch_size, F = a->num_faces, S = a->image_size, ts = a->texture_size;
    if (!soft_sizes_ok(B, F, S)) return NR_ERR_INVALID_ARG;
    const float sigma = a->sigma, gamma = a->gamma;
    if (!isfinite(sigma) || !(sigma > 0.0f) || (softmax && (!isfinite(gamma) || !(gamma > 0.0f)))) return NR_ERR_INVALID_ARG;
    if (!(a->near_ < a->far_) || !isfinite(a->far_ - a->near_) || (cubes && !isfinite(a->eps))) return NR_ERR_INVALID_ARG;
    memset(p, 0, sizeof(*p));
    if (!make_face_src(flags, a->faces, a->vertices, a->face_indices, F, a->num_vertices, &p->s.src))
        return NR_ERR_INVALID_ARG;
    if ((colour && !a->textures) || (cubes && (ts < 2 || (long long)ts * ts * ts * 3 > 0x7FFFFFFFll))) return NR_ERR_INVALID_ARG;
    if ((colour && !a->rgb) || (softmax && (!a->alpha || !a->state))) return NR_ERR_INVALID_ARG;
    if (backward) {
        const bool indexed = (flags & NR_FACES_INDEXED) != 0;
        if (indexed ? a->grad_faces != nullptr : a->grad_vertices != nullptr) return NR_ERR_INVALID_ARG;
        if (!make_face_grad(flags, a->grad_faces, a->grad_vertices, a->face_indices, F, a->num_vertices, &p->s.dst))
            return NR_ERR_INVALID_ARG;
    }
    SoftParams& s = p->s;
    s.alpha = a->alpha; s.g = a->grad_alpha;
    s.B = B; s.F = F; s.S = S;
    s.ntx = tiles_per_axis(S); s.ntiles = s.ntx * s.ntx;
    const double cut = (double)sigma * log((1.0 - NR_SOFT_EPS) / NR_SOFT_EPS);
    s.inv_sigma = (float)(1.0 / (double)sigma);
    s.cut = (float)cut;
    s.reach = (float)(sqrt(cut) * S * 0.5) + 1.0f;
    s.near_ = a->near_; s.far_ = a->far_;
    if (cubes) {
        p->tex.tex = a->textures;
        p->tex.cube_bstride = (flags & NR_TEX_SHARED) ? 0 : (size_t)F;
        const double tmax = (double)(ts - 1) - a->eps;
        p->tex.tex_cmp = float_le(tmax);
        p->tex.tex_val = (float)tmax;
        p->ts = ts;
    }
    p->light = a->face_light;
    p->rgb = a->rgb; p->state = a->state; p->g_rgb = a->grad_rgb;
    p->grad_tex = a->grad_textures; p->grad_light = a->grad_face_light;
    for (int c = 0; c < 3; c++) p->bg[c] = a->background[c];
    const double fn = (double)a->far_ - (double)a->near_;
    p->zp_bg = (float)((double)a->far_ - NR_SOFT_BG_DEPTH * fn);
    p->inv_fg = softmax ? (float)(1.0 / (fn * (double)gamma)) : 0.0f;
    return NR_OK;
}

int soft_rgb_workspace(const nr_b200_soft_rgb_args* a, void* params, void* layout) {
    SoftRgbParams* p = (SoftRgbParams*)params;
    SoftRgbLayout* L = (SoftRgbLayout*)layout;
    if (!a->workspace || ((uintptr_t)a->workspace & 15)) return NR_ERR_WORKSPACE;
    if (!soft_rgb_layout(p->s.B, p->s.F, p->s.S, L)) return NR_ERR_CUDA;
    if (a->workspace_bytes < L->total) return NR_ERR_WORKSPACE;
    char* ws = (char*)a->workspace;
    SoftParams& s = p->s;
    s.rec = (float4*)(ws + L->s.rec); s.box = (uint2*)(ws + L->s.box);
    s.cnt = (int*)(ws + L->s.cnt); s.cursor = (int*)(ws + L->s.cursor); s.off = (int*)(ws + L->s.off);
    p->zrec = (float4*)(ws + L->zrec);
    p->keys = ws + L->keys;
    p->fbits = L->fbits;
    return NR_OK;
}

int soft_rgb_bin(void* params, const void* layout, bool sort, cudaStream_t s) {
    SoftRgbParams& p = *(SoftRgbParams*)params;
    const SoftRgbLayout& L = *(const SoftRgbLayout*)layout;
    return L.wide ? bin_faces_rgb<unsigned long long>(p, L, sort, s) : bin_faces_rgb<uint32_t>(p, L, sort, s);
}

}  // namespace nr_internal

namespace {

// the host checks of both soft RGB entry points; fills `p` and `L` on success
int soft_rgb_setup(const nr_b200_soft_rgb_args* a, bool backward, SoftRgbParams* p, SoftRgbLayout* L) {
    nr_internal::launch_count() = 0;
    const int rc = nr_internal::soft_rgb_check(a, kSoftRgbFlags, nr_internal::kSoftCubes, backward, p);
    return rc != NR_OK ? rc : nr_internal::soft_rgb_workspace(a, p, L);
}

}  // namespace

extern "C" size_t nr_b200_soft_rgb_workspace_bytes(int32_t B, int32_t F, int32_t S, uint32_t flags) {
    SoftRgbLayout L;
    if ((flags & ~kSoftRgbFlags) || !soft_rgb_layout(B, F, S, &L)) return 0;
    return L.total;
}

extern "C" int nr_b200_soft_rgb(const nr_b200_soft_rgb_args* args, void* cuda_stream) {
    SoftRgbParams p;
    SoftRgbLayout L;
    const int rc = soft_rgb_setup(args, false, &p, &L);
    if (rc != NR_OK) return rc;
    cudaStream_t s = (cudaStream_t)cuda_stream;
    if ((L.wide ? soft_rgb_forward<unsigned long long>(p, L, s) : soft_rgb_forward<uint32_t>(p, L, s)) != NR_OK)
        return NR_ERR_CUDA;
    return cudaGetLastError() == cudaSuccess ? NR_OK : NR_ERR_CUDA;
}

extern "C" int nr_b200_soft_rgb_backward(const nr_b200_soft_rgb_args* args, void* cuda_stream) {
    SoftRgbParams p;
    SoftRgbLayout L;
    const int rc = soft_rgb_setup(args, true, &p, &L);
    if (rc != NR_OK) return rc;
    const nr_b200_soft_rgb_args* a = args;
    const bool indexed = (a->flags & NR_FACES_INDEXED) != 0;
    cudaStream_t s = (cudaStream_t)cuda_stream;
    if (!(a->flags & NR_GRAD_ACCUMULATE)) {
        nr_internal::prof_begin("memset_grads", s);
        cudaError_t e = indexed ? cudaMemsetAsync(a->grad_vertices, 0, (size_t)p.s.B * a->num_vertices * 3 * sizeof(float), s)
                                : cudaMemsetAsync(a->grad_faces, 0, (size_t)p.s.B * p.s.F * 9 * sizeof(float), s);
        const size_t cube = (size_t)p.ts * p.ts * p.ts * 3;
        const size_t tex_items = (a->flags & NR_TEX_SHARED) ? 1 : (size_t)p.s.B;
        if (e == cudaSuccess && a->grad_textures)
            e = cudaMemsetAsync(a->grad_textures, 0, tex_items * p.s.F * cube * sizeof(float), s);
        if (e == cudaSuccess && a->grad_face_light)
            e = cudaMemsetAsync(a->grad_face_light, 0, (size_t)p.s.B * p.s.F * 3 * sizeof(float), s);
        nr_internal::prof_end(s);
        if (e != cudaSuccess) return NR_ERR_CUDA;
    }
    if (!a->grad_alpha && !a->grad_rgb) return cudaGetLastError() == cudaSuccess ? NR_OK : NR_ERR_CUDA;
    if ((L.wide ? soft_rgb_backward<unsigned long long>(p, L, s) : soft_rgb_backward<uint32_t>(p, L, s)) != NR_OK)
        return NR_ERR_CUDA;
    return cudaGetLastError() == cudaSuccess ? NR_OK : NR_ERR_CUDA;
}

