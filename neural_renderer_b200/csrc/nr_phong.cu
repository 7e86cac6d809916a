// nr_phong.cu -- the Phong-shading gradients of nr_b200_backward_phong, nr_b200_backward_lights, nr_b200_backward_sh,
// nr_b200_backward_normal_map and nr_b200_backward_specular_map (include/nr_b200.h, nr_b200_phong_args,
// nr_b200_lights_args, nr_b200_sh_args, nr_b200_normal_map_args, nr_b200_specular_map_args).
//
//   k_phong_grad<kTex, kIdx, kLights, kSH, kNM, kSM>   one thread per raster pixel, modelled on k_interior_grad.  The winner's perspective weights
//                   l_k and the unlit sample s are recomputed with the forward's device helpers (the depth map gives zp;
//                   per-face cubes read the sampler depths NR_TEX_Z_BATCH0 selects), nr::phong_at evaluates the forward's
//                   expression and nr::phong_grad its derivative.  The 18 corner floats l_k (d loss / d n, d loss / d p) go
//                   through k_depth_grad's segmented run reduction (runs of neighbouring lanes that show the same face)
//                   before one set of atomics per run; the 16 parameter floats are summed over the warp, then over the CTA
//                   in shared memory, before 16 atomics per CTA.  kTex: 0 = per-face cubes, 1 = bilinear image,
//                   2 = trilinear pyramid.  Anti-aliasing and fill_back are runtime flags.  kLights / kSH split the
//                   call's light mode (nr_shading.cuh) by register layout: kLightPhong = neither, kLightPhongSet =
//                   kLights, kLightPhongSH = kSH with kLights when NL > 0.
//                   kLights (a light set, NL > 0): after light 0 the pixel keeps its d loss / d nh, d vh and d p
//                   accumulators across the loop over the lights (nr::phong_light_grad); each light's 10 record floats
//                   are summed over the warp into shared memory, and after the loop over the CTA before 10 atomics per
//                   light per CTA, so no NL x 10 register array exists.
//                   kSH (an SH environment): with kLights, after the loop over the lights d E / d nh joins the
//                   d loss / d nh accumulator before the normalisation chain; without, d E / d nh goes through that chain
//                   on its own and is added to light 0's normal gradient.  The 27 floats Y_k g_c s_c are summed over the
//                   warp one at a time into shared memory, then over the CTA before 27 atomics per CTA
//                   (sh_grad_reduce), so no 27-float register array exists.
//                   kNM (kLightPhongNM, a tangent-space normal map; kTex 1 / 2): the expression is evaluated with the
//                   mapped normal n' (nr::nm_pixel_normal), so the chains above end in g' = d loss / d n'.  Then
//                   nm_grad_tail samples the map and builds the frame again and sends gm to the map's four taps (two
//                   6-float rows by vector reductions, as k_image_grad); the 9 tangent floats l_k gt and the 6 UV floats l_k (gu, gv) widen the run reduction to 33.
//                   The launcher takes kLights (NL > 0), kSH, kNM and kSM from which inputs the record holds.
//                   kSM (kLightPhongSM, a specular map; kTex 1 / 2; kNM = a normal map given too): the map's sample
//                   (ks, sigma') at the pixel's uv enters the expression and its derivative as K' = ks K, K'_j = ks K_j and
//                   sigma' (the sq argument of the nr_math.cuh helpers).  Per pixel gq_c = K_c g_c h + sum_j K_jc g_c a_j h_j
//                   is split off the K and K_j gradients (which keep ks_c times theirs) and gq_3 = d loss / d sigma' off
//                   params' slot 12, which receives 0; sm_grad_tail samples the map again and sends gq to its four taps (one
//                   16-byte vector reduction each) and l_k (gu, gv) to the UV floats of the run reduction (24, or shared with
//                   the normal map's six in 33).  Both map tails and the corner floats are written by pixel_grad_tail,
//                   after light 0 alone or after the loop over the lights.
//
// It belongs to the texture half of the backward: the texture-gradient kernels (K6, k_image_grad) only need the pixel's
// L_c, and keeping the 34 gradient floats out of them keeps their register budgets (DESIGN.md section 4g).
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include "nr_b200.h"
#include "nr_internal.h"
#include "nr_math.cuh"
#include "nr_phong.h"

namespace {

struct PhongParams {
    nr::FaceSrc src;
    const int32_t* fim;     // [B,S,S]
    const float* wmap;      // [B,3,S,S]
    const float* dmap;      // [B,S,S]
    const float* g;         // grad_rgb [B,3,H,W] (API layout)
    float* grad_cs;         // the layouts of corner_shading, params, lights (kLights) and sh (kSH), or nullptr
    float* grad_prm;
    float* grad_lts;
    float* grad_sh;
    int S, F, ts;
    int aa, fill_back, z_batch0;
    nr::Texture tex;
    nr::Shading shading;  // corner_shading, params, lights, sh and the maps
    float* grad_nm;       // kNM: the layouts of normal_map, corner_tangents and face_uvs, or nullptr
    float* grad_tg;
    float* grad_uvs;
    float* grad_sm;       // kSM: the layout of specular_map, or nullptr
};

// kNM, once g' = d loss / d n' of the pixel is known: the map's sample (with its uv derivative) and the frame again, the
// same loads and arithmetic as nm_pixel_normal; gn = g' on entry, d loss / d n (of the interpolated normal) on return.
// d loss / d m goes to the map's four taps (tap weight x gm) by vector reductions; cgx[0..8] = l_k gt (corner-major) and
// cgx[9..14] = l_k (gu, gv) for the stored face's UV corners (a fill_back copy's corner k is corner 2 - k).
__device__ __forceinline__ void nm_grad_tail(const PhongParams& p, int b, int fn, const float lam[3], float u, float v, bool rev,
                                             float gn[3], float* cgx) {
    const nr::Shading& s = p.shading;
    const nr::UvTaps t = nr::uv_taps(u, v, s.Hm, s.Wm);
    float m[3], du[3], dv[3], np[3];
    nr::nm_sample<true>(s.nm + s.nm_off(b), s.Hm, s.Wm, t, m, du, dv);
    nr::NmFrame F;
    nr::nm_normal(s.cs + s.cs_off(b, fn), s.tg + s.tg_off(b, fn), lam, m, F, np);
    float gm[3], gt[3], gi[3];
    nr::nm_normal_grad(F, m, gn, gm, gt, gi);
#pragma unroll
    for (int k = 0; k < 3; k++) gn[k] = gi[k];
    if (p.grad_nm) {  // uniform: per tap row the horizontal pair (x0, x1) = 6 consecutive floats, by vector reductions
        const uint32_t row3 = (uint32_t)s.Wm * 3u, c0 = (uint32_t)t.x0 * 3u;
        float* q0 = p.grad_nm + s.nm_off(b) + (uint32_t)t.r0 * row3 + c0;
        float* q1 = p.grad_nm + s.nm_off(b) + (uint32_t)t.r1 * row3 + c0;
        float v0[6], v1[6];
#pragma unroll
        for (int k = 0; k < 3; k++) {
            v0[k] = __fmul_rn(t.w00, gm[k]); v0[3 + k] = __fmul_rn(t.w10, gm[k]);
            v1[k] = __fmul_rn(t.w01, gm[k]); v1[3 + k] = __fmul_rn(t.w11, gm[k]);
        }
        if (t.x1 != t.x0) {
            nr::red_add_6(q0, v0);
            nr::red_add_6(q1, v1);
        } else {  // a clamped column (x1 = x0, weight 0 on x1): both taps are one texel
#pragma unroll
            for (int k = 0; k < 3; k++) {
                atomicAdd(q0 + k, __fadd_rn(v0[k], v0[3 + k]));
                atomicAdd(q1 + k, __fadd_rn(v1[k], v1[3 + k]));
            }
        }
    }
#pragma unroll
    for (int k = 0; k < 3; k++)
#pragma unroll
        for (int j = 0; j < 3; j++) cgx[3 * k + j] = __fmul_rn(lam[k], gt[j]);
    const float gu = __fmaf_rn(gm[2], du[2], __fmaf_rn(gm[1], du[1], __fmul_rn(gm[0], du[0])));
    const float gv = __fmaf_rn(gm[2], dv[2], __fmaf_rn(gm[1], dv[1], __fmul_rn(gm[0], dv[0])));
    const float s0 = rev ? lam[2] : lam[0], s2 = rev ? lam[0] : lam[2];
    cgx[9] = __fmul_rn(s0, gu); cgx[10] = __fmul_rn(s0, gv);
    cgx[11] = __fmul_rn(lam[1], gu); cgx[12] = __fmul_rn(lam[1], gv);
    cgx[13] = __fmul_rn(s2, gu); cgx[14] = __fmul_rn(s2, gv);
}

// kSM, once gq = d loss / d (ks, sigma') of the pixel is known: the map's uv derivative at the same taps, tap weight x gq to
// the four taps of grad_sm (a clamped column, x1 = x0, merges its two taps first), and l_k (gu, gv) added into cuv[0..5]
// for the stored face's UV corners (a fill_back copy's corner k is corner 2 - k)
__device__ __forceinline__ void sm_grad_tail(const PhongParams& p, int b, const float lam[3], float u, float v, bool rev,
                                             const float gq[4], float* cuv) {
    const nr::Shading& s = p.shading;
    const nr::UvTaps t = nr::uv_taps(u, v, s.Hq, s.Wq);
    float q[4], du[4], dv[4];
    nr::sm_sample<true>(s.sm + s.sm_off(b), s.Hq, s.Wq, t, q, du, dv);
    if (p.grad_sm) {  // uniform
        float* g0 = p.grad_sm + s.sm_off(b) + ((uint32_t)t.r0 * (uint32_t)s.Wq + (uint32_t)t.x0) * 4u;
        float* g1 = p.grad_sm + s.sm_off(b) + ((uint32_t)t.r1 * (uint32_t)s.Wq + (uint32_t)t.x0) * 4u;
        float v00[4], v10[4], v01[4], v11[4];
#pragma unroll
        for (int k = 0; k < 4; k++) {
            v00[k] = __fmul_rn(t.w00, gq[k]); v10[k] = __fmul_rn(t.w10, gq[k]);
            v01[k] = __fmul_rn(t.w01, gq[k]); v11[k] = __fmul_rn(t.w11, gq[k]);
        }
        if (t.x1 != t.x0) {
            nr::red_add_4(g0, v00); nr::red_add_4(g0 + 4, v10);
            nr::red_add_4(g1, v01); nr::red_add_4(g1 + 4, v11);
        } else {
#pragma unroll
            for (int k = 0; k < 4; k++) { v00[k] = __fadd_rn(v00[k], v10[k]); v01[k] = __fadd_rn(v01[k], v11[k]); }
            nr::red_add_4(g0, v00);
            nr::red_add_4(g1, v01);
        }
    }
    float gu = __fmul_rn(gq[0], du[0]), gv = __fmul_rn(gq[0], dv[0]);
#pragma unroll
    for (int k = 1; k < 4; k++) { gu = __fmaf_rn(gq[k], du[k], gu); gv = __fmaf_rn(gq[k], dv[k], gv); }
    const float s0 = rev ? lam[2] : lam[0], s2 = rev ? lam[0] : lam[2];
    cuv[0] = __fmaf_rn(s0, gu, cuv[0]); cuv[1] = __fmaf_rn(s0, gv, cuv[1]);
    cuv[2] = __fmaf_rn(lam[1], gu, cuv[2]); cuv[3] = __fmaf_rn(lam[1], gv, cuv[3]);
    cuv[4] = __fmaf_rn(s2, gu, cuv[4]); cuv[5] = __fmaf_rn(s2, gv, cuv[5]);
}

// where the maps' 6 UV floats start in the run reduction: after the 18 corner floats and kNM's 9 tangent floats
template <bool kNM>
constexpr int kUvAt = kNM ? 27 : 18;

// The per-pixel end of k_phong_grad once gn = d loss / d n (kNM: d loss / d n') and gp = d loss / d p are known: the map
// tails (kSM: d loss / d sigma' goes to the map as gq[3], not to params' slot 12), then the 18 corner floats of cg
template <bool kNM, bool kSM>
__device__ __forceinline__ void pixel_grad_tail(const PhongParams& p, int b, int fn, const float lam[3], float u, float v,
                                                bool rev, float gn[3], const float gp[3], float gq[4], float gprm[16],
                                                float* cg) {
    if constexpr (kNM) nm_grad_tail(p, b, fn, lam, u, v, rev, gn, cg + 18);
    if constexpr (kSM) {
        gq[3] = gprm[12];
        gprm[12] = 0.0f;
        sm_grad_tail(p, b, lam, u, v, rev, gq, cg + kUvAt<kNM>);
    }
#pragma unroll
    for (int k = 0; k < 3; k++)
#pragma unroll
        for (int j = 0; j < 3; j++) {
            cg[6 * k + j] = __fmul_rn(lam[k], gn[j]);
            cg[6 * k + 3 + j] = __fmul_rn(lam[k], gp[j]);
        }
}

// kSH: the 27 floats Y_k w_c of grad_sh summed over the warp one at a time into shared memory, then over the CTA before 27
// atomics into `o` (item b's [9,3] slot, or slot 0 with Bs = 1).  Every thread of the CTA calls it (0 off the mesh).
__device__ __forceinline__ void sh_grad_reduce(const float Y[9], const float ws[3], float* o, int lane, int warp) {
    __shared__ float s_sh[8][27];
#pragma unroll
    for (int t = 0; t < 27; t++) {
        float v = __fmul_rn(Y[t / 3], ws[t % 3]);
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
        if (lane == 0) s_sh[warp][t] = v;
    }
    __syncthreads();
    if (threadIdx.x < 27) {
        float v = 0.0f;
        const int nw = (int)(blockDim.x >> 5);
        for (int w = 0; w < nw; w++) v += s_sh[w][threadIdx.x];
        atomicAdd(o + threadIdx.x, v);
    }
}

template <int kTex, bool kIdx, bool kLights, bool kSH, bool kNM, bool kSM>
__global__ void __launch_bounds__(256) k_phong_grad(const __grid_constant__ PhongParams p) {
    static_assert(!(kNM || kSM) || kTex != 0, "the maps need NR_TEX_UV");
    constexpr int kCg = kNM ? 33 : kSM ? 24 : 18;  // the corner floats of the run reduction
    __shared__ float s_prm[8][16];
    const int S = p.S;
    const size_t plane = (size_t)S * S;
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int b = blockIdx.y;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int fn = (i < plane) ? __ldg(p.fim + (size_t)b * plane + i) : -1;
    if (!__syncthreads_or(fn >= 0)) return;  // CTA-uniform
    float cg[kCg], gprm[16];
#pragma unroll
    for (int k = 0; k < kCg; k++) cg[k] = 0.0f;
#pragma unroll
    for (int k = 0; k < 16; k++) gprm[k] = 0.0f;
    // kLights: what the loop over the lights needs of the covered pixel below
    nr::PhongEval xE;
    float xg[3], xs[3], xlam[3], xpos[3], xgn[3], xgp[3];
    // kSH without kLights: Y_k(nh) and g_c s_c of the covered pixel, 0 elsewhere
    float shY[9], shw[3];
    if constexpr (kSH && !kLights) {
#pragma unroll
        for (int k = 0; k < 9; k++) shY[k] = 0.0f;
#pragma unroll
        for (int k = 0; k < 3; k++) shw[k] = 0.0f;
    }
    float nmu = 0.0f, nmv = 0.0f;  // kNM / kSM: the pixel's uv, its UV face and whether it is a fill_back copy
    int nmtf = 0;
    bool nmrev = false;
    // kSM: the map's sample (ks, sigma') and d loss / d (ks, sigma') of the covered pixel
    float smq[4] = {0.0f, 0.0f, 0.0f, 0.0f}, gq[4] = {0.0f, 0.0f, 0.0f, 0.0f};
    const float* sq = kSM ? smq : nullptr;
    if (fn >= 0) {
        const int r = (int)(i / S), c = (int)(i % S);
        const bool aa = p.aa != 0;
        const int H = aa ? (S >> 1) : S;
        const size_t gplane = (size_t)H * H;
        const size_t goff = aa ? (size_t)(r >> 1) * H + (c >> 1) : i;
        const float gscale = aa ? 0.25f : 1.0f;  // the pooling backward
        const float* gb = p.g + (size_t)b * 3 * gplane + goff;
        const float g[3] = {__ldg(gb) * gscale, __ldg(gb + gplane) * gscale, __ldg(gb + 2 * gplane) * gscale};
        const float* wm = p.wmap + (size_t)b * 3 * plane + i;
        const float w[3] = {__ldg(wm), __ldg(wm + plane), __ldg(wm + 2 * plane)};
        const float zp = __ldg(p.dmap + (size_t)b * plane + i);
        float v[9];
        if constexpr (kTex == 2) {
            nr::load_face(p.src, b, fn, v);
        } else {
#pragma unroll
            for (int k = 0; k < 3; k++) v[3 * k + 2] = __ldg(nr::face_vertex_t<kIdx>(p.src, b, fn, k) + 2);
        }
        const float z[3] = {v[2], v[5], v[8]};
        float lam[3];
        nr::perspective_weights(w, zp, z[0], z[1], z[2], lam);
        bool rev;
        const int tf = nr::stored_face(p.fill_back, p.F, fn, rev);
        float s[3];  // the unlit sample, as the forward computes it
        float uv[6];  // kTex 1 / 2: the face's UV corners
        if constexpr (kTex == 0) {
            const int ts = p.ts;
            float zt[3] = {z[0], z[1], z[2]};  // the sampler's depths: item 0's with NR_TEX_Z_BATCH0
            if (p.z_batch0 && b != 0) {
#pragma unroll
                for (int k = 0; k < 3; k++) zt[k] = __ldg(nr::face_vertex_t<kIdx>(p.src, 0, fn, k) + 2);
            }
            const nr::TexCoord tc = nr::texture_coords(w, zp, zt[0], zt[1], zt[2], ts, p.tex.tex_cmp, p.tex.tex_val);
            nr::cube_blend<false, true>(p.tex.tex + p.tex.cube_off(b, tf, ts), tc, ts, rev, nullptr, s[0], s[1], s[2]);
        } else {
            float u, vv;
            nr::face_uvs(p.tex, b, tf, rev, uv);
            nr::pixel_uv(w, zp, z[0], z[1], z[2], uv, u, vv);
            const float* img = p.tex.tex + p.tex.img_off(b);
            if constexpr (kTex == 2) {
                const float fS = (float)S;
                float inv[9];
                nr::face_inverse(nr::to_pixel(v[0], fS), nr::to_pixel(v[1], fS), nr::to_pixel(v[3], fS), nr::to_pixel(v[4], fS),
                                 nr::to_pixel(v[6], fS), nr::to_pixel(v[7], fS), inv);
                const float lod = nr::mip_lod(inv, w, zp, z[0], z[1], z[2], uv, p.tex.Ht, p.tex.Wt, p.tex.mip.levels);
                nr::mip_blend<false>(img, p.tex.mip, nr::mip_levels(lod, p.tex.mip.levels), u, vv, 1.0f, 1.0f, 1.0f, s);
            } else {
                nr::uv_blend<false>(img, p.tex.Wt, nr::uv_taps(u, vv, p.tex.Ht, p.tex.Wt), 1.0f, 1.0f, 1.0f, s);
            }
        }
        const float* prm = p.shading.prm + p.shading.prm_off(b);
        nr::PhongEval E;
        if constexpr (kNM || kSM) {  // the mapped normal (or n) in E.n and the specular sample, then the rest of phong_at
            nr::pixel_uv(w, zp, z[0], z[1], z[2], uv, nmu, nmv);
            nmtf = tf; nmrev = rev;
            if constexpr (kNM) {
                float m[3];
                nr::NmFrame Fm;
                nr::nm_pixel_normal(p.shading, b, fn, lam, nmu, nmv, m, Fm, E);
            } else {
                nr::phong_normal(p.shading.cs + p.shading.cs_off(b, fn), lam, E.n);
            }
            if constexpr (kSM) nr::sm_pixel_sample(p.shading, b, nmu, nmv, smq);
            nr::phong_diffuse_n(prm, E);
            nr::phong_specular(p.shading.cs + p.shading.cs_off(b, fn), lam, prm, E, sq);
        } else {
            nr::phong_at(p.shading.cs + p.shading.cs_off(b, fn), lam, prm, E);
        }
        float gn[3], gp[3];
        nr::phong_grad(E, prm, g, s, gn, gp, gprm, sq);
        if constexpr (kSM) {  // g_c h: K_c's share to the map, ks_c's to K_c
#pragma unroll
            for (int k = 0; k < 3; k++) {
                gq[k] = __fmul_rn(__ldg(prm + 9 + k), gprm[9 + k]);
                gprm[9 + k] = __fmul_rn(smq[k], gprm[9 + k]);
            }
        }
        if constexpr (kLights) {  // the set's gradients read neither E.L nor the set's diffuse terms
            nr::phong_position(p.shading.cs + p.shading.cs_off(b, fn), lam, xpos);
            xE = E;
#pragma unroll
            for (int k = 0; k < 3; k++) {
                xg[k] = g[k]; xs[k] = s[k]; xlam[k] = lam[k]; xgn[k] = gn[k]; xgp[k] = gp[k];
            }
        } else {
            if constexpr (kSH) {  // no light set: d E / d nh through the normalisation chain on its own (it is linear)
                float gnh[3] = {0.0f, 0.0f, 0.0f}, t[3];
#pragma unroll
                for (int k = 0; k < 3; k++) shw[k] = __fmul_rn(g[k], s[k]);
                nr::sh_basis(E.nh, shY);
                nr::sh_grad_nh(p.shading.sh + p.shading.sh_off(b), E.nh, shw, gnh);
                nr::normalize_eps_grad(E.n, E.n_len, gnh, t);
#pragma unroll
                for (int k = 0; k < 3; k++) gn[k] = __fadd_rn(gn[k], t[k]);
            }
            pixel_grad_tail<kNM, kSM>(p, b, fn, lam, nmu, nmv, nmrev, gn, gp, gq, gprm, cg);
        }
    }
    if constexpr (kLights) {
        __shared__ float s_lt[8][nr_internal::kMaxLights * 10];  // per warp: each light's 10 record floats
        const float* lts = p.shading.lts + p.shading.lts_off(b);
        const float sigma = kSM ? smq[3] : __ldg(p.shading.prm + p.shading.prm_off(b) + 12);
        float gnh[3] = {0.0f, 0.0f, 0.0f}, gvh[3] = {0.0f, 0.0f, 0.0f}, gsig = 0.0f;
        for (int j = 0; j < p.shading.NL; j++) {  // uniform
            float gl[10];
#pragma unroll
            for (int k = 0; k < 10; k++) gl[k] = 0.0f;
            if (fn >= 0) {
                nr::phong_light_grad(lts + 12 * j, xE, xpos, sigma, xg, xs, gnh, gvh, xgp, gsig, gl, sq);
                if constexpr (kSM) {  // g_c a_j h_j: K_jc's share to the map, ks_c's to K_jc
#pragma unroll
                    for (int k = 0; k < 3; k++) {
                        gq[k] = __fmaf_rn(__ldg(lts + 12 * j + 3 + k), gl[3 + k], gq[k]);
                        gl[3 + k] = __fmul_rn(smq[k], gl[3 + k]);
                    }
                }
            }
            if (p.grad_lts) {  // uniform
#pragma unroll
                for (int off = 16; off > 0; off >>= 1)
#pragma unroll
                    for (int k = 0; k < 10; k++) gl[k] += __shfl_xor_sync(0xffffffffu, gl[k], off);
                if (lane == 0) {
#pragma unroll
                    for (int k = 0; k < 10; k++) s_lt[warp][10 * j + k] = gl[k];
                }
            }
        }
        if constexpr (kSH) {  // before the normalisation chain: d E / d nh joins gnh
            float Y[9], ws[3];             // Y_k(nh) and g_c s_c (d rgb_c / d L_c = s_c); 0 off the mesh
            if (fn >= 0) {
#pragma unroll
                for (int k = 0; k < 3; k++) ws[k] = __fmul_rn(xg[k], xs[k]);
                nr::sh_basis(xE.nh, Y);
                nr::sh_grad_nh(p.shading.sh + p.shading.sh_off(b), xE.nh, ws, gnh);
            } else {
#pragma unroll
                for (int k = 0; k < 9; k++) Y[k] = 0.0f;
#pragma unroll
                for (int k = 0; k < 3; k++) ws[k] = 0.0f;
            }
            if (p.grad_sh) sh_grad_reduce(Y, ws, p.grad_sh + p.shading.sh_off(b), lane, warp);  // uniform
        }
        if (fn >= 0) {
            nr::phong_lights_grad_end(xE, gnh, gvh, gsig, xgn, xgp, gprm);
            pixel_grad_tail<kNM, kSM>(p, b, fn, xlam, nmu, nmv, nmrev, xgn, xgp, gq, gprm, cg);
        }
        if (p.grad_lts) {  // uniform: the CTA's sum of each light's 10 floats, then 10 atomics per light
            __syncthreads();
            const int nw = (int)(blockDim.x >> 5);
            for (int t = threadIdx.x; t < 10 * p.shading.NL; t += blockDim.x) {
                float v = 0.0f;
                for (int w = 0; w < nw; w++) v += s_lt[w][t];
                atomicAdd(p.grad_lts + p.shading.lts_off(b) + (size_t)(t / 10) * 12 + t % 10, v);
            }
        }
    }
    if constexpr (kSH && !kLights) {
        if (p.grad_sh) sh_grad_reduce(shY, shw, p.grad_sh + p.shading.sh_off(b), lane, warp);  // uniform
    }
    if ((kNM || kSM) ? (p.grad_cs || p.grad_tg || p.grad_uvs) : p.grad_cs != nullptr) {  // uniform
        // the segmented run reduction of k_depth_grad over 18 (kNM: 33, kSM: 24) floats, then one set of atomics per run
        const int fn_prev = __shfl_up_sync(0xffffffffu, fn, 1);
        const uint32_t heads = __ballot_sync(0xffffffffu, lane == 0 || fn != fn_prev);
        const uint32_t later = heads & ~((2u << lane) - 1u);
        const int run_end = (lane == 31 || later == 0) ? 31 : (__ffs(later) - 2);
#pragma unroll
        for (int off = 1; off < 32; off <<= 1) {
            const bool take = lane + off <= run_end;
#pragma unroll
            for (int k = 0; k < kCg; k++) {
                const float t = __shfl_down_sync(0xffffffffu, cg[k], off);
                if (take) cg[k] += t;
            }
        }
        if (fn >= 0 && ((heads >> lane) & 1u)) {
            if (!(kNM || kSM) || p.grad_cs) {
                float* o = p.grad_cs + p.shading.cs_off(b, fn);
#pragma unroll
                for (int k = 0; k < 18; k++) atomicAdd(o + k, cg[k]);
            }
            if constexpr (kNM) {
                if (p.grad_tg) {
                    float* o = p.grad_tg + p.shading.tg_off(b, fn);
#pragma unroll
                    for (int k = 0; k < 3; k++)
#pragma unroll
                        for (int j = 0; j < 3; j++) atomicAdd(o + 4 * k + j, cg[18 + 3 * k + j]);
                }
            }
            if constexpr (kNM || kSM) {
                if (p.grad_uvs) {
                    float* o = p.grad_uvs + p.tex.uv_off(b, nmtf);
#pragma unroll
                    for (int k = 0; k < 6; k++) atomicAdd(o + k, cg[kUvAt<kNM> + k]);
                }
            }
        }
    }
    if (p.grad_prm) {  // uniform: warp sums, then the CTA's sum in shared memory, 16 atomics per CTA
#pragma unroll
        for (int off = 16; off > 0; off >>= 1)
#pragma unroll
            for (int k = 0; k < 16; k++) gprm[k] += __shfl_xor_sync(0xffffffffu, gprm[k], off);
        if (lane == 0) {
#pragma unroll
            for (int k = 0; k < 16; k++) s_prm[warp][k] = gprm[k];
        }
        __syncthreads();
        if (threadIdx.x < 16) {
            float t = 0.0f;
            const int nw = (int)(blockDim.x >> 5);
            for (int w = 0; w < nw; w++) t += s_prm[w][threadIdx.x];
            atomicAdd(p.grad_prm + p.shading.prm_off(b) + threadIdx.x, t);
        }
    }
}

}  // namespace

namespace nr_internal {

void launch_phong_grad(const PhongGradLaunch& L, cudaStream_t stream) {
    const nr_b200_backward_args* a = L.args;
    const uint32_t flags = a->flags;
    PhongParams p;
    memset(&p, 0, sizeof(p));
    p.src = L.src;
    p.fim = a->face_index_map; p.wmap = a->weight_map; p.dmap = a->depth_map; p.g = a->grad_rgb;
    p.grad_cs = L.grad.cs; p.grad_prm = L.grad.prm; p.grad_lts = L.grad.lts; p.grad_sh = L.grad.sh;
    p.S = a->raster_size; p.F = a->num_faces; p.ts = a->texture_size;
    p.aa = (flags & NR_ANTI_ALIASING) ? 1 : 0;
    p.fill_back = (flags & NR_TEX_FILL_BACK) ? 1 : 0;
    p.z_batch0 = (flags & NR_TEX_Z_BATCH0) ? 1 : 0;
    p.tex = L.tex;
    p.shading = L.shading;
    p.grad_nm = L.grad.nm; p.grad_tg = L.grad.tg; p.grad_uvs = L.grad.uvs; p.grad_sm = L.grad.sm;
    const bool idx = (flags & NR_FACES_INDEXED) != 0;
    const int tex = (flags & NR_TEX_MIPMAP) ? 2 : (flags & NR_TEX_UV) ? 1 : 0;
    const dim3 grid((unsigned)(((size_t)p.S * p.S + 255) / 256), a->batch_size);
    LaunchScope ls("k_phong_grad", stream);
    // the kernel's split of the light mode (3-7): a light set of NL > 0 lights, an SH environment, a normal map and a
    // specular map, each read from the record
    nr::dispatch_bool(p.shading.NL > 0, [&](auto kLights) {
        nr::dispatch_bool(p.shading.sh != nullptr, [&](auto kSH) {
            nr::dispatch_bool(idx, [&](auto kIdx) {
                nr::dispatch_bool(p.shading.nm != nullptr, [&](auto kNM) {
                    nr::dispatch_bool(p.shading.sm != nullptr, [&](auto kSM) {
                        if (tex == 2) k_phong_grad<2, kIdx, kLights, kSH, kNM, kSM><<<grid, 256, 0, stream>>>(p);
                        else if (tex == 1) k_phong_grad<1, kIdx, kLights, kSH, kNM, kSM><<<grid, 256, 0, stream>>>(p);
                        else if constexpr (!kNM && !kSM)  // the maps need NR_TEX_UV (checked on the host)
                            k_phong_grad<0, kIdx, kLights, kSH, false, false><<<grid, 256, 0, stream>>>(p);
                    });
                });
            });
        });
    });
}

}  // namespace nr_internal
