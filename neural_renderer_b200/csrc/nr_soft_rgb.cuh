// nr_soft_rgb.cuh -- what the soft RGB units share: the parameter record and workspace layout, the face staging, the
// barycentrics and the forward traversal of a (tile, item), parameterised by the sampler that gives a contributing
// (pixel, face) its colour C_j: nr_soft_rgb.cu samples per-face cubes, nr_soft_uv.cu texture images and mip pyramids
// through face_uvs.  A sampler provides color(p, b, f, bc, z, rec, r, g, bl) (rec = the face's edge record).
// Everything is in an anonymous namespace: each translation unit compiles its own copy of what it uses.
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "nr_b200.h"
#include "nr_internal.h"
#include "nr_soft.cuh"
#include "nr_texture.cuh"

namespace {

constexpr int kWarps = kThreads / 32;

struct SoftRgbParams {
    SoftParams s;          // the silhouettes' binning and alpha (s.g = grad_alpha)
    float4* zrec;          // [B*F] {z0, z1, z2, A}: vertex depths and the doubled signed area
    void* keys;            // [B*F*kWideTiles] composite keys (uint32_t or uint64_t)
    nr::Texture tex;       // cubes [Bt,F,ts,ts,ts,3], or the image / pyramid and face_uvs (nr_soft_uv.cu)
    const float* light;    // [B,F,3] face_light or nullptr
    float* rgb;            // [B,3,S,S]
    float* state;          // [B,2,S,S]: Z, zref
    const float* g_rgb;    // [B,3,S,S] or nullptr
    float* grad_tex;       // like tex, or nullptr
    float* grad_light;     // [B,F,3] or nullptr
    int ts, fbits;
    float bg[3];
    float zp_bg;           // far - NR_SOFT_BG_DEPTH (far - near): the depth of the background level
    float inv_fg;          // 1 / ((far - near) gamma)
};

// soft RGB workspace = the silhouettes' records, boxes, counters, cursors and offsets | depth records | keys | sorted
// keys | CUB scratch.  The keys are 32-bit when (B (ntiles + 1)) << fbits fits, else 64-bit.
struct SoftRgbLayout {
    SoftLayout s;
    size_t zrec, keys, keys_out, temp, temp_bytes, total;
    int fbits, end_bit;
    bool wide;
};

// Stages the next <= kThreads faces of the tile in list order (its own list, then the wide list with a box test): the
// slots come from a block-wide scan of the ballots, so slot order is list order.  Returns how many were staged.
template <typename K>
__device__ __forceinline__ int stage_rgb(const SoftRgbParams& p, int b, int tile, int tx, int ty, int n_tile, int n_all,
                                         int next, float4* s_rec, float4* s_z, int* s_face, int* s_wn) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int i = next + tid;
    const size_t seg = (size_t)b * (p.s.ntiles + 1);
    const K* keys = (const K*)p.keys;
    const K mask = ((K)1 << p.fbits) - 1;
    int f = -1;
    if (i < n_tile) {
        f = (int)(keys[p.s.off[seg + tile] + i] & mask);
    } else if (i < n_all) {
        f = (int)(keys[p.s.off[seg + p.s.ntiles] + (i - n_tile)] & mask);
        const uint2 bb = __ldg(p.s.box + (size_t)b * p.s.F + f);
        if (tx < lo16(bb.x) || tx > hi16(bb.x) || ty < lo16(bb.y) || ty > hi16(bb.y)) f = -1;
    }
    const unsigned m = __ballot_sync(0xffffffffu, f >= 0);
    if (lane == 0) s_wn[warp] = __popc(m);
    __syncthreads();
    int base = 0, n = 0;
#pragma unroll
    for (int w = 0; w < kWarps; w++) {
        const int c = s_wn[w];
        base += w < warp ? c : 0;
        n += c;
    }
    if (f >= 0) {
        const int slot = base + __popc(m & ((1u << lane) - 1u));
        const size_t id = (size_t)b * p.s.F + f;
        const float4* r = p.s.rec + id * 4;
#pragma unroll
        for (int k = 0; k < 4; k++) s_rec[slot * 4 + k] = __ldg(r + k);
        s_z[slot] = __ldg(p.zrec + id);
        s_face[slot] = f;
    }
    __syncthreads();
    return n;
}

// the soft RGB barycentrics of a pixel (include/nr_b200.h): lam_k = c_{k+1} / A, clamped to [0, 1] (lh), renormalised
// (l = lh / s), and the perspective-correct depth zp = 1 / sum_k l_k / z_k
struct SoftBary {
    float lam[3], l[3], s, zp;
};
__device__ __forceinline__ SoftBary soft_bary(const float c[3], const float4& z) {
    SoftBary o;
    const float zz[3] = {z.x, z.y, z.z};
    float lh[3];
#pragma unroll
    for (int k = 0; k < 3; k++) {
        o.lam[k] = __fdiv_rn(c[k == 2 ? 0 : k + 1], z.w);
        lh[k] = fminf(fmaxf(o.lam[k], 0.0f), 1.0f);
    }
    o.s = __fadd_rn(__fadd_rn(lh[0], lh[1]), lh[2]);
    float q = 0.0f;
#pragma unroll
    for (int k = 0; k < 3; k++) {
        o.l[k] = __fdiv_rn(lh[k], o.s);
        q = __fadd_rn(q, __fdiv_rn(o.l[k], zz[k]));
    }
    o.zp = __frcp_rn(q);
    return o;
}

__device__ __forceinline__ float soft_sigmoid(float x) {
    const float e = expf(-fabsf(x));
    return x >= 0.0f ? __frcp_rn(1.0f + e) : __fdiv_rn(e, 1.0f + e);
}

// ------------------------------------------------------------------------------------------------ forward traversal
// one CTA per (tile, item): faces staged in list order, a running-max softmax per pixel in that order
template <typename K, class Smp>
__device__ __forceinline__ void soft_rgb_fwd_body(const SoftRgbParams& p, const Smp& smp, float4* s_rec, float4* s_z,
                                                  int* s_face, int* s_wn) {
    const int tile = blockIdx.x, b = blockIdx.y;
    const int tx = tile % p.s.ntx, ty = tile / p.s.ntx;
    const int col = tx * kTile + (threadIdx.x % kTile), row = ty * kTile + (threadIdx.x / kTile);
    const int S = p.s.S;
    const float px = soft_centre(col, S), py = soft_centre(S - 1 - row, S);
    const size_t seg = (size_t)b * (p.s.ntiles + 1);
    const int n_tile = p.s.cnt[seg + tile], n_all = n_tile + p.s.cnt[seg + p.s.ntiles];
    const unsigned long long cap = (unsigned long long)(kTermCap * kFix);
    unsigned long long acc = 0;  // alpha exactly as k_soft_fwd
    // running-max softmax: zref = the smallest depth so far (the background level first), Z and N relative to it
    float zref = p.zp_bg, Z = 1.0f, N0 = p.bg[0], N1 = p.bg[1], N2 = p.bg[2];
    for (int next = 0; next < n_all; next += kThreads) {
        const int n = stage_rgb<K>(p, b, tile, tx, ty, n_tile, n_all, next, s_rec, s_z, s_face, s_wn);
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
                Z = __fmul_rn(Z, sc); N0 = __fmul_rn(N0, sc); N1 = __fmul_rn(N1, sc); N2 = __fmul_rn(N2, sc);
                zref = bc.zp;
                w = D;
            } else {
                w = __fmul_rn(D, expf(__fmul_rn(__fsub_rn(zref, bc.zp), p.inv_fg)));
                if (w == 0.0f) continue;  // its texels are not read
            }
            const int f = s_face[j];
            float r, g, bl;
            smp.color(p, b, f, bc, z, s_rec + 4 * j, r, g, bl);
            Z = __fadd_rn(Z, w);
            N0 = __fmaf_rn(w, r, N0); N1 = __fmaf_rn(w, g, N1); N2 = __fmaf_rn(w, bl, N2);
        }
        __syncthreads();
    }
    if (row < S && col < S) {
        const size_t plane = (size_t)S * S, o = (size_t)row * S + col;
        const float lam = __ull2float_rn(acc) * (1.0f / kFix);
        __stcs(p.s.alpha + b * plane + o, -expm1f(-lam));
        float* rgb = p.rgb + (size_t)b * 3 * plane + o;
        __stcs(rgb, __fdiv_rn(N0, Z));
        __stcs(rgb + plane, __fdiv_rn(N1, Z));
        __stcs(rgb + 2 * plane, __fdiv_rn(N2, Z));
        float* st = p.state + (size_t)b * 2 * plane + o;
        __stcs(st, Z);
        __stcs(st + plane, zref);
    }
}

}  // namespace
