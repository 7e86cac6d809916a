// nr_soft_attr.cu -- soft attribute images (nr_b200_soft_attributes / nr_b200_soft_attributes_backward,
// include/nr_b200.h): the soft RGB's aggregation with a C-channel colour A_jc = sum_k l'_k a_kc interpolated from
// per-corner or per-vertex attributes (per-vertex colours, soft depth, normals, features).
//
// The host checks, the workspace and the binning (keys, sort) are nr_soft_rgb.cu's (nr_internal.h), on the parameter
// fill and the binning start (setup, scan) of nr_soft.cuh; the gradient zero-fill is nr_internal.h's; the face staging, the barycentrics and the sigmoid are nr_soft_rgb.cuh's; the chain from l'_k into the vertices is
// k_soft_uv_bwd's (a copy, soft_lprime_chain).  New kernels, each for 32- and 64-bit keys and
// for channel blocks of kCB = 4 or 16:
//   k_soft_attr_fwd<K, kCB>  the traversal of k_soft_rgb_fwd with kCB numerators per pixel in registers; grid.z runs the
//                            channel blocks of a C > kCB call, each re-traversing in the same order (every channel's
//                            arithmetic is its own, so a channel comes out the same in any block); block 0 writes alpha
//                            and state
//   k_soft_attr_bwd<K, kCB>  the soft RGB backward with the attributes' chain: 9 vertex partials per face reduced over the
//                            warp and the CTA as k_soft_rgb_bwd; d loss / d attributes with the CHANNELS across the lanes:
//                            per (warp, face) the contributing lanes broadcast l'_k w / Z and their pixel by shuffle, lane
//                            c sums l'_k (w / Z) g_c(p) over them (g read through L1) and issues one atomic per corner and
//                            channel (against a per-lane scatter of 3C atomics per pixel: up to 2.4x faster at C 16, up
//                            to 15 % slower at C 1; DESIGN.md 4r)
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <string.h>

#include "nr_b200.h"
#include "nr_internal.h"
#include "nr_soft.cuh"
#include "nr_soft_rgb.cuh"

namespace {

constexpr uint32_t kNoRow = 0xFFFFFFFFu;  // a per-vertex corner whose index is outside [0, Nv): reads zeros, no gradient
constexpr int kMaxChannelBlocks = 65535;  // grid.z

struct SoftAttrParams {
    SoftRgbParams r;          // the soft RGB's binning, alpha, state and softmax constants (its colour fields unused)
    const float* attr;        // [.,F,3,C] or [.,Nv,C]
    const float* bg;          // [C] or nullptr (zeros)
    float* out;               // [B,C,S,S]
    const float* g_out;       // [B,C,S,S] or nullptr
    float* gattr;             // layout of attr, or nullptr
    const int32_t* idx;       // face_indices (NR_ATTR_PER_VERTEX), else nullptr
    long long idx_bstride;    // 3F, or 0 with NR_INDICES_SHARED
    uint32_t attr_bstride;    // floats per item of attr (0 = shared)
    int C, Nv;
};

// the first float of the attribute rows of the staged faces' corners (32-bit: the host refuses more), after stage_rgb
__device__ __forceinline__ void stage_rows(const SoftAttrParams& P, int b, int n, const int* s_face, uint32_t* s_row) {
    const int j = threadIdx.x;
    if (j < n) {
        const int f = s_face[j];
        const uint32_t base = (uint32_t)b * P.attr_bstride, C = (uint32_t)P.C;
#pragma unroll
        for (int k = 0; k < 3; k++) {
            uint32_t row;
            if (P.idx == nullptr) {
                row = base + ((uint32_t)f * 3u + (uint32_t)k) * C;
            } else {
                const int i = __ldg(P.idx + (size_t)b * P.idx_bstride + (size_t)f * 3 + k);
                row = (unsigned)i < (unsigned)P.Nv ? base + (uint32_t)i * C : kNoRow;
            }
            s_row[j * 3 + k] = row;
        }
    }
    __syncthreads();
}

__device__ __forceinline__ float attr_at(const float* a, uint32_t row, int c) {
    return row == kNoRow ? 0.0f : __ldg(a + row + (uint32_t)c);
}

// A_c = fma(l'_2, a_2c, fma(l'_1, a_1c, l'_0 a_0c)) (include/nr_b200.h)
__device__ __forceinline__ float attr_blend(const float lp[3], const float* a, const uint32_t row[3], int c) {
    return __fmaf_rn(lp[2], attr_at(a, row[2], c), __fmaf_rn(lp[1], attr_at(a, row[1], c), __fmul_rn(lp[0], attr_at(a, row[0], c))));
}

// l'_k = l_k (zp / z_k)
__device__ __forceinline__ void lprime(const SoftBary& bc, const float4& z, float lp[3]) {
    lp[0] = __fmul_rn(bc.l[0], __fdiv_rn(bc.zp, z.x));
    lp[1] = __fmul_rn(bc.l[1], __fdiv_rn(bc.zp, z.y));
    lp[2] = __fmul_rn(bc.l[2], __fdiv_rn(bc.zp, z.z));
}

// The backward from the perspective-correct weights l'_k = l_k r_k, r_k = zp / z_k, of a contributing (pixel, face):
// with Gt_k = d loss / d l'_k and dzp = d loss / d zp so far (through the weight), on through l_k, zp and z_k, the lh
// clamp (held) and the edge functions c_e of the face record `rec` at pixel (px, py) into v[2m], v[2m + 1] (x, y of
// vertex m) and v[6 + m] (its z).  The expressions of k_soft_uv_bwd's chain from gu u_k + gv v_k, which keeps its own
// copy: calling a shared function from it changed that kernel's instruction schedule (DESIGN.md 4r).
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

// ------------------------------------------------------------------------------------------------ k_soft_attr_fwd
// soft_rgb_fwd_body with a C-vector colour: the same staging, order, alpha, softmax and state
// (the explicit minimum of one CTA per SM: with the default, ptxas gives kCB = 4 40 registers and a 16-byte spill)
template <typename K, int kCB>
__global__ void __launch_bounds__(kThreads, 1) k_soft_attr_fwd(const __grid_constant__ SoftAttrParams P) {
    __shared__ float4 s_rec[kThreads * 4];
    __shared__ float4 s_z[kThreads];
    __shared__ int s_face[kThreads];
    __shared__ uint32_t s_row[kThreads * 3];
    __shared__ int s_wn[kWarps];
    const SoftRgbParams& p = P.r;
    const int tile = blockIdx.x, b = blockIdx.y, c0 = blockIdx.z * kCB;
    const int nc = min(kCB, P.C - c0);
    const int tx = tile % p.s.ntx, ty = tile / p.s.ntx;
    const int col = tx * kTile + (threadIdx.x % kTile), row = ty * kTile + (threadIdx.x / kTile);
    const int S = p.s.S;
    const float px = soft_centre(col, S), py = soft_centre(S - 1 - row, S);
    const size_t seg = (size_t)b * (p.s.ntiles + 1);
    const int n_tile = p.s.cnt[seg + tile], n_all = n_tile + p.s.cnt[seg + p.s.ntiles];
    const unsigned long long cap = (unsigned long long)(kTermCap * kFix);
    unsigned long long acc = 0;  // alpha exactly as k_soft_fwd
    // running-max softmax: zref = the smallest depth so far (the background level first), Z and N relative to it
    float zref = p.zp_bg, Z = 1.0f, N[kCB];
#pragma unroll
    for (int q = 0; q < kCB; q++) N[q] = (q < nc && P.bg) ? __ldg(P.bg + c0 + q) : 0.0f;
    for (int next = 0; next < n_all; next += kThreads) {
        const int n = stage_rgb<K>(p, b, tile, tx, ty, n_tile, n_all, next, s_rec, s_z, s_face, s_wn);
        stage_rows(P, b, n, s_face, s_row);
        for (int j = 0; j < n; j++) {
            float x, t, qx, qy, c[3];
            int k;
            if (!soft_eval(s_rec + 4 * j, px, py, p.s.inv_sigma, p.s.cut, x, k, t, qx, qy, c)) continue;
            const float sp = fmaxf(x, 0.0f) + log1pf(expf(-fabsf(x)));
            acc += (unsigned long long)__float2ll_rn(fminf(sp, kTermCap) * kFix);
            acc = acc < cap ? acc : cap;
            const float4 z = s_z[j];
            if (z.w == 0.0f) continue;  // a zero-area face: alpha only
            const SoftBary bc = soft_bary(c, z);
            const float D = soft_sigmoid(x);
            float w;
            if (bc.zp < zref) {
                const float sc = expf(__fmul_rn(__fsub_rn(bc.zp, zref), p.inv_fg));
                Z = __fmul_rn(Z, sc);
#pragma unroll
                for (int q = 0; q < kCB; q++) N[q] = __fmul_rn(N[q], sc);
                zref = bc.zp;
                w = D;
            } else {
                w = __fmul_rn(D, expf(__fmul_rn(__fsub_rn(zref, bc.zp), p.inv_fg)));
                if (w == 0.0f) continue;  // its attributes are not read
            }
            float lp[3];
            lprime(bc, z, lp);
            const uint32_t rows[3] = {s_row[3 * j], s_row[3 * j + 1], s_row[3 * j + 2]};
            Z = __fadd_rn(Z, w);
#pragma unroll
            for (int q = 0; q < kCB; q++)
                if (q < nc) N[q] = __fmaf_rn(w, attr_blend(lp, P.attr, rows, c0 + q), N[q]);
        }
        __syncthreads();
    }
    if (row < S && col < S) {
        const size_t plane = (size_t)S * S, o = (size_t)row * S + col;
        if (blockIdx.z == 0) {
            const float lam = __ull2float_rn(acc) * (1.0f / kFix);
            __stcs(p.s.alpha + b * plane + o, -expm1f(-lam));
            float* st = p.state + (size_t)b * 2 * plane + o;
            __stcs(st, Z);
            __stcs(st + plane, zref);
        }
        float* out = P.out + ((size_t)b * P.C + c0) * plane + o;
#pragma unroll
        for (int q = 0; q < kCB; q++)
            if (q < nc) __stcs(out + q * plane, __fdiv_rn(N[q], Z));
    }
}

// ------------------------------------------------------------------------------------------------ k_soft_attr_bwd
constexpr int kAttrPartials = 9;  // per face: (x, y) of 3 vertices, z of 3 vertices

template <typename K, int kCB>
__global__ void __launch_bounds__(kThreads) k_soft_attr_bwd(const __grid_constant__ SoftAttrParams P) {
    __shared__ float4 s_rec[kThreads * 4];
    __shared__ float4 s_z[kThreads];
    __shared__ int s_face[kThreads];
    __shared__ uint32_t s_row[kThreads * 3];
    __shared__ float s_acc[kThreads * kAttrPartials];
    __shared__ int s_wn[kWarps];
    const SoftRgbParams& p = P.r;
    const int tile = blockIdx.x, b = blockIdx.y;
    const int tx = tile % p.s.ntx, ty = tile / p.s.ntx;
    const int col = tx * kTile + (threadIdx.x % kTile), row = ty * kTile + (threadIdx.x / kTile);
    const int S = p.s.S, C = P.C, lane = threadIdx.x & 31;
    const float px = soft_centre(col, S), py = soft_centre(S - 1 - row, S);
    const size_t seg = (size_t)b * (p.s.ntiles + 1);
    const int n_tile = p.s.cnt[seg + tile], n_all = n_tile + p.s.cnt[seg + p.s.ntiles];
    if (n_all == 0) return;  // CTA-uniform
    const size_t plane = (size_t)S * S;
    const bool in_image = row < S && col < S;
    const uint32_t o = in_image ? (uint32_t)row * (uint32_t)S + (uint32_t)col : 0u;  // S <= 32767
    const float* gb = P.g_out ? P.g_out + (size_t)b * C * plane : nullptr;
    float ga = 0.0f, g[kCB], Z = 1.0f, zref = 0.0f, gdot = 0.0f;  // gdot = sum_c g_c out_c
    bool want = false;
#pragma unroll
    for (int q = 0; q < kCB; q++) g[q] = 0.0f;
    if (in_image) {
        if (p.s.g) ga = __ldg(p.s.g + b * plane + o) * (1.0f - __ldg(p.s.alpha + b * plane + o));
        if (gb) {
            const float* ob = P.out + (size_t)b * C * plane + o;
#pragma unroll
            for (int q = 0; q < kCB; q++) {
                if (q < C) {
                    g[q] = __ldg(gb + q * plane + o);
                    want = want || g[q] != 0.0f;
                    gdot = __fmaf_rn(g[q], __ldg(ob + q * plane), gdot);
                }
            }
            for (int ch = kCB; ch < C; ch++) {
                const float gc = __ldg(gb + ch * plane + o);
                want = want || gc != 0.0f;
                gdot = __fmaf_rn(gc, __ldg(ob + ch * plane), gdot);
            }
        }
        Z = __ldg(p.state + (size_t)b * 2 * plane + o);
        zref = __ldg(p.state + (size_t)b * 2 * plane + plane + o);
    }
    const float iZ = __frcp_rn(Z);
    const bool active = ga != 0.0f || want;
    // H = g . (A - out) / Z = (g . A) / Z - (g . out) / Z
    const float g_out = __fmul_rn(gdot, iZ);
    for (int i = threadIdx.x; i < kThreads * kAttrPartials; i += kThreads) s_acc[i] = 0.0f;
    for (int next = 0; next < n_all; next += kThreads) {
        const int n = stage_rgb<K>(p, b, tile, tx, ty, n_tile, n_all, next, s_rec, s_z, s_face, s_wn);
        stage_rows(P, b, n, s_face, s_row);
        for (int j = 0; j < n; j++) {
            float x = 0.0f, t = 0.0f, qx = 0.0f, qy = 0.0f, c[3];
            int k = 0;
            const bool hit = active && soft_eval(s_rec + 4 * j, px, py, p.s.inv_sigma, p.s.cut, x, k, t, qx, qy, c);
            if (!__any_sync(0xffffffffu, hit)) continue;  // warp-uniform
            const uint32_t rows[3] = {s_row[3 * j], s_row[3 * j + 1], s_row[3 * j + 2]};
            float v[kAttrPartials];
#pragma unroll
            for (int m = 0; m < kAttrPartials; m++) v[m] = 0.0f;
            bool attr_hit = false;
            float sa[3] = {0.0f, 0.0f, 0.0f};  // l'_k w / Z: d loss / d a_kc = sa_k g_c
            if (hit) {
                const float D = soft_sigmoid(x);
                float gx = __fmul_rn(ga, D);  // d loss / d x_j
                const float4 z = s_z[j];
                if (want && z.w != 0.0f) {
                    const SoftBary bc = soft_bary(c, z);
                    const float w = __fmul_rn(D, expf(__fmul_rn(__fsub_rn(zref, bc.zp), p.inv_fg)));
                    if (w != 0.0f) {
                        float lp[3];
                        lprime(bc, z, lp);
                        // G_k = sum_c g_c a_kc: g . A = sum_k l'_k G_k, d loss / d l'_k = (w / Z) G_k
                        float G[3] = {0.0f, 0.0f, 0.0f};
#pragma unroll
                        for (int q = 0; q < kCB; q++) {
                            if (q < C) {
#pragma unroll
                                for (int a = 0; a < 3; a++) G[a] = __fmaf_rn(g[q], attr_at(P.attr, rows[a], q), G[a]);
                            }
                        }
                        for (int ch = kCB; ch < C; ch++) {
                            const float gc = __ldg(gb + ch * plane + o);
#pragma unroll
                            for (int a = 0; a < 3; a++) G[a] = __fmaf_rn(gc, attr_at(P.attr, rows[a], ch), G[a]);
                        }
                        const float gA = __fmaf_rn(lp[2], G[2], __fmaf_rn(lp[1], G[1], __fmul_rn(lp[0], G[0])));
                        const float h = __fsub_rn(__fmul_rn(gA, iZ), g_out);
                        gx = __fmaf_rn(__fmul_rn(w, 1.0f - D), h, gx);
                        const float dzp = -__fmul_rn(__fmul_rn(w, h), p.inv_fg);  // d loss / d zp through the weight
                        const float wz = __fmul_rn(w, iZ);
                        const float Gt[3] = {__fmul_rn(wz, G[0]), __fmul_rn(wz, G[1]), __fmul_rn(wz, G[2])};
                        soft_lprime_chain(bc, z, s_rec + 4 * j, px, py, Gt, dzp, v);
                        if (P.gattr) {
                            attr_hit = true;
#pragma unroll
                            for (int a = 0; a < 3; a++) sa[a] = __fmul_rn(lp[a], wz);
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
#if defined(NR_B200_TUNING) && defined(NR_SOFT_ATTR_LANE_SCATTER)
            // the measured alternative (DESIGN.md 4r): every contributing lane sends its own 3C products
            if (attr_hit) {
                for (int ch = 0; ch < C; ch++) {
                    const float gq = __ldg(gb + ch * plane + o);
#pragma unroll
                    for (int a = 0; a < 3; a++)
                        if (rows[a] != kNoRow && gq != 0.0f) atomicAdd(P.gattr + rows[a] + ch, __fmul_rn(sa[a], gq));
                }
            }
            const uint32_t hits = 0u;
#else
            const uint32_t hits = __ballot_sync(0xffffffffu, attr_hit);
#endif
            // d loss / d attributes, channels across the lanes: lane c sums sa_k(p) g_c(p) over the contributing lanes
            if (hits) {  // warp-uniform
                for (int cb = 0; cb < C; cb += 32) {
                    const int ch = cb + lane;
                    const float* gc = gb + (size_t)(ch < C ? ch : 0) * plane;
                    float a0 = 0.0f, a1 = 0.0f, a2 = 0.0f;
                    uint32_t todo = hits;
                    while (todo) {  // warp-uniform
                        const int q = __ffs(todo) - 1;
                        todo &= todo - 1u;
                        const float s0 = __shfl_sync(0xffffffffu, sa[0], q), s1 = __shfl_sync(0xffffffffu, sa[1], q),
                                    s2 = __shfl_sync(0xffffffffu, sa[2], q);
                        const uint32_t oq = __shfl_sync(0xffffffffu, o, q);
                        if (ch < C) {
                            const float gq = __ldg(gc + oq);
                            a0 = __fmaf_rn(s0, gq, a0); a1 = __fmaf_rn(s1, gq, a1); a2 = __fmaf_rn(s2, gq, a2);
                        }
                    }
                    if (ch < C) {
                        if (rows[0] != kNoRow && a0 != 0.0f) atomicAdd(P.gattr + rows[0] + ch, a0);
                        if (rows[1] != kNoRow && a1 != 0.0f) atomicAdd(P.gattr + rows[1] + ch, a1);
                        if (rows[2] != kNoRow && a2 != 0.0f) atomicAdd(P.gattr + rows[2] + ch, a2);
                    }
                }
            }
#pragma unroll
            for (int off = 16; off > 0; off >>= 1)
#pragma unroll
                for (int m = 0; m < kAttrPartials; m++) v[m] += __shfl_xor_sync(0xffffffffu, v[m], off);
            if (lane < kAttrPartials) {
                float mine = v[0];
#pragma unroll
                for (int m = 1; m < kAttrPartials; m++) if (lane == m) mine = v[m];
                if (mine != 0.0f) atomicAdd(&s_acc[j * kAttrPartials + lane], mine);
            }
        }
        __syncthreads();
        // one set of global atomics per face of the round: thread (face slot, vertex)
        for (int i = threadIdx.x; i < n * 3; i += kThreads) {
            const int j = i / 3, m = i % 3;
            float* a = s_acc + j * kAttrPartials;
            const float gx = a[2 * m], gy = a[2 * m + 1], gz = a[6 + m];
            a[2 * m] = 0.0f; a[2 * m + 1] = 0.0f; a[6 + m] = 0.0f;
            if (gx == 0.0f && gy == 0.0f && gz == 0.0f) continue;
            float* gv = nr::face_grad_vertex(p.s.dst, b, s_face[j], m);
            if (gv) { atomicAdd(gv, gx); atomicAdd(gv + 1, gy); atomicAdd(gv + 2, gz); }
        }
        __syncthreads();
    }
}

constexpr uint32_t kSoftAttrFlags = NR_FACES_INDEXED | NR_INDICES_SHARED | NR_ATTR_PER_VERTEX | NR_ATTR_SHARED |
                                    NR_GRAD_ACCUMULATE;
constexpr int kSmallBlock = 4, kLargeBlock = 16;

// the host checks of both entry points; fills `p`, `L` and the floats of the attribute set
int soft_attr_setup(const nr_b200_soft_rgb_args* a, const nr_b200_soft_attr_args* at, bool backward, SoftAttrParams* p,
                    SoftRgbLayout* L, size_t* attr_floats) {
    nr_internal::launch_count() = 0;
    if (!a || a->struct_size != sizeof(nr_b200_soft_rgb_args) || !at || at->struct_size != sizeof(nr_b200_soft_attr_args))
        return NR_ERR_INVALID_ARG;
    const uint32_t flags = a->flags;
    const bool per_vertex = (flags & NR_ATTR_PER_VERTEX) != 0;
    if (at->channels < 1 || !at->attributes || !at->out) return NR_ERR_INVALID_ARG;
    if (per_vertex && !(flags & NR_FACES_INDEXED)) return NR_ERR_INVALID_ARG;
    // the soft RGB's colour buffers have no meaning here
    if (a->textures || a->face_light || a->rgb || a->grad_rgb || a->grad_textures || a->grad_face_light)
        return NR_ERR_INVALID_ARG;
    memset(p, 0, sizeof(*p));
    int rc = nr_internal::soft_rgb_check(a, kSoftAttrFlags, nr_internal::kSoftAttributes, backward, &p->r);
    if (rc != NR_OK) return rc;
    const int B = a->batch_size, F = a->num_faces, C = at->channels;
    const size_t rows = per_vertex ? (size_t)a->num_vertices : (size_t)F * 3;
    const size_t per_item = rows * (size_t)C, items = (flags & NR_ATTR_SHARED) ? 1 : (size_t)B;
    *attr_floats = items * per_item;
    // 32-bit attribute offsets in the kernels; the forward's channel blocks on grid.z
    if (*attr_floats > 0x7FFFFFFFull || (C + kLargeBlock - 1) / kLargeBlock > kMaxChannelBlocks) return NR_ERR_UNSUPPORTED;
    p->attr = at->attributes;
    p->bg = at->background;
    p->out = at->out;
    p->g_out = backward ? at->grad_out : nullptr;
    p->gattr = backward ? at->grad_attributes : nullptr;
    if (per_vertex) {
        p->idx = a->face_indices;
        p->idx_bstride = (flags & NR_INDICES_SHARED) ? 0 : (long long)F * 3;
    }
    p->attr_bstride = (flags & NR_ATTR_SHARED) ? 0u : (uint32_t)per_item;
    p->C = C;
    p->Nv = a->num_vertices;
    return nr_internal::soft_rgb_workspace(a, &p->r, L);
}

template <typename K, int kCB>
void soft_attr_launch(const SoftAttrParams& p, bool backward, cudaStream_t s) {
    if (backward) {
        nr_internal::LaunchScope ls("k_soft_attr_bwd", s);
        k_soft_attr_bwd<K, kCB><<<dim3((unsigned)p.r.s.ntiles, (unsigned)p.r.s.B), kThreads, 0, s>>>(p);
    } else {
        nr_internal::LaunchScope ls("k_soft_attr_fwd", s);
        const dim3 grid((unsigned)p.r.s.ntiles, (unsigned)p.r.s.B, (unsigned)((p.C + kCB - 1) / kCB));
        k_soft_attr_fwd<K, kCB><<<grid, kThreads, 0, s>>>(p);
    }
}

template <typename K>
void soft_attr_launch(const SoftAttrParams& p, bool backward, cudaStream_t s) {
    if (p.C <= kSmallBlock) soft_attr_launch<K, kSmallBlock>(p, backward, s);
    else soft_attr_launch<K, kLargeBlock>(p, backward, s);
}

// the binning (sorted for the forward), then the traversal
int soft_attr_run(SoftAttrParams& p, const SoftRgbLayout& L, bool backward, cudaStream_t s) {
    if (nr_internal::soft_rgb_bin(&p.r, &L, !backward, s) != NR_OK) return NR_ERR_CUDA;
    if (L.wide) soft_attr_launch<unsigned long long>(p, backward, s);
    else soft_attr_launch<uint32_t>(p, backward, s);
    return cudaGetLastError() == cudaSuccess ? NR_OK : NR_ERR_CUDA;
}

}  // namespace

extern "C" int nr_b200_soft_attributes(const nr_b200_soft_rgb_args* args, const nr_b200_soft_attr_args* attr,
                                       void* cuda_stream) {
    SoftAttrParams p;
    SoftRgbLayout L;
    size_t attr_floats;
    const int rc = soft_attr_setup(args, attr, false, &p, &L, &attr_floats);
    if (rc != NR_OK) return rc;
    return soft_attr_run(p, L, false, (cudaStream_t)cuda_stream);
}

extern "C" int nr_b200_soft_attributes_backward(const nr_b200_soft_rgb_args* args, const nr_b200_soft_attr_args* attr,
                                                void* cuda_stream) {
    SoftAttrParams p;
    SoftRgbLayout L;
    size_t attr_floats;
    const int rc = soft_attr_setup(args, attr, true, &p, &L, &attr_floats);
    if (rc != NR_OK) return rc;
    const nr_b200_soft_rgb_args* a = args;
    cudaStream_t s = (cudaStream_t)cuda_stream;
    if (!(a->flags & NR_GRAD_ACCUMULATE) &&
        nr_internal::zero_grads({nr_internal::geometry_grad(a), {p.gattr, attr_floats * sizeof(float)}}, s) != cudaSuccess)
        return NR_ERR_CUDA;
    if (!a->grad_alpha && !attr->grad_out) return cudaGetLastError() == cudaSuccess ? NR_OK : NR_ERR_CUDA;
    return soft_attr_run(p, L, true, s);
}
