// nr_interior.cu -- the interior vertex gradient of the RGB image (NR_GRAD_INTERIOR, include/nr_b200.h).
//
// The textured or smooth-shaded colour of a covered pixel depends on the geometry through the perspective weights l_k:
// the texture is sampled at sum_k l_k uv_k (or at the cube coordinates (ts - 1) l_k) and smooth shading interpolates its
// corner light with them.  k_interior_grad forms G_k = d loss / d l_k for the renderer's own samplers and lights and
// chains it into grad_faces / grad_vertices exactly as attribute interpolation does (nr_attr.cu, k_interp_grad):
//
//   k_interior_grad<kTex, kLight, kIdx>   one thread per raster pixel.  The winner's depth zp and weights l_k are
//                   recomputed with the forward's expressions (zp == depth_map bit for bit, so the depth map is not read),
//                   the sampler's derivative comes from the nr_math.cuh helpers with the cell, the level of detail and the
//                   clamps held fixed, and the 9 floats per pixel go through k_depth_grad's segmented run reduction before
//                   one set of atomics per run.  kTex: 0 = per-face cubes, 1 = bilinear image, 2 = trilinear pyramid;
//                   kLight: kLightNone, kLightFace or kLightCorner (nr_shading.cuh).  Anti-aliasing and fill_back are
//                   runtime flags.
//
// It belongs to the faces half of nr_b200_backward and runs after K5 / K7 into the same (already zero-filled) output.
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include "nr_b200.h"
#include "nr_interior.h"
#include "nr_internal.h"
#include "nr_math.cuh"

namespace {

struct InteriorParams {
    nr::FaceSrc src;
    nr::FaceGrad dst;
    const int32_t* fim;     // [B,S,S]
    const float* wmap;      // [B,3,S,S]
    const float* g;         // grad_rgb [B,3,H,W] (API layout)
    int S, F, ts;
    int aa, fill_back;
    nr::Texture tex;
    nr::Shading shading;  // face_light (kLightFace) or corner_light (kLightCorner)
};

template <int kTex, int kLight, bool kIdx>
__global__ void __launch_bounds__(256) k_interior_grad(const __grid_constant__ InteriorParams p) {
    const int S = p.S;
    const size_t plane = (size_t)S * S;
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int b = blockIdx.y;
    const int lane = threadIdx.x & 31;
    const int fn = (i < plane) ? __ldg(p.fim + (size_t)b * plane + i) : -1;
    if (!__any_sync(0xffffffffu, fn >= 0)) return;  // warp-uniform
    float vg[9];
#pragma unroll
    for (int k = 0; k < 9; k++) vg[k] = 0.0f;
    if (fn >= 0) {
        const int r = (int)(i / S), c = (int)(i % S);
        const bool aa = p.aa != 0;
        const int H = aa ? (S >> 1) : S;
        const size_t gplane = (size_t)H * H;
        const size_t goff = aa ? (size_t)(r >> 1) * H + (c >> 1) : i;
        const float gscale = aa ? 0.25f : 1.0f;  // the pooling backward
        const float* gb = p.g + (size_t)b * 3 * gplane + goff;
        float g[3] = {__ldg(gb) * gscale, __ldg(gb + gplane) * gscale, __ldg(gb + 2 * gplane) * gscale};
        const float* wm = p.wmap + (size_t)b * 3 * plane + i;
        const float w[3] = {__ldg(wm), __ldg(wm + plane), __ldg(wm + 2 * plane)};
        float v[9];
#pragma unroll
        for (int k = 0; k < 3; k++) {
            const float* q = nr::face_vertex_t<kIdx>(p.src, b, fn, k);
            v[3 * k] = __ldg(q); v[3 * k + 1] = __ldg(q + 1); v[3 * k + 2] = __ldg(q + 2);
        }
        const float z[3] = {v[2], v[5], v[8]};
        const float zp = nr::pixel_depth(w, z[0], z[1], z[2]);
        float lam[3];
        nr::perspective_weights(w, zp, z[0], z[1], z[2], lam);
        const float fS = (float)S;
        float inv[9];
        nr::face_inverse(nr::to_pixel(v[0], fS), nr::to_pixel(v[1], fS), nr::to_pixel(v[3], fS), nr::to_pixel(v[4], fS),
                         nr::to_pixel(v[6], fS), nr::to_pixel(v[7], fS), inv);
        float lx[3], ly[3];
        nr::perspective_weight_grads(inv, z, zp, lam, lx, ly);
        // the light factor L_c of d rgb_c / d s_c
        float L[3], C[9];
        nr::pixel_light<kLight>(p.shading, b, p.F, fn, lam, 0.0f, 0.0f, L);  // no Phong mode, so no map reads the uv
        if constexpr (kLight == nr::kLightCorner) {
            const float* cp = p.shading.corner_light + p.shading.cl_off(b, p.F, fn);
#pragma unroll
            for (int k = 0; k < 9; k++) C[k] = __ldg(cp + k);
        }
        const float h[3] = {g[0] * L[0], g[1] * L[1], g[2] * L[2]};  // d loss / d unlit sample
        bool rev;
        const int tf = nr::stored_face(p.fill_back, p.F, fn, rev);
        float s[3];              // the unlit sample
        float D1, D2, P[3];      // the sampler's part of D_k = G_k - G_0 and P_m = sum_k l_k G_k - G_m
        if constexpr (kTex == 0) {
            const int ts = p.ts;
            const nr::TexCoord tc = nr::texture_coords(w, zp, z[0], z[1], z[2], ts, p.tex.tex_cmp, p.tex.tex_val);
            float dt[3][3];
            nr::cube_blend_axis_grad(p.tex.tex + p.tex.cube_off(b, tf, ts), tc, ts, rev, s, dt);
            const float fts1 = (float)(ts - 1);
            float G[3];
#pragma unroll
            for (int k = 0; k < 3; k++) {
                // the clamp gate of texture_coords on the unclamped coordinate (NaN -> 0)
                const float t = __fmul_rn(__fmul_rn(w[k], fts1), __fdiv_rn(zp, z[k]));
                const bool in = t >= 0.0f && t <= p.tex.tex_cmp;
                const float e = __fmaf_rn(h[2], dt[k][2], __fmaf_rn(h[1], dt[k][1], __fmul_rn(h[0], dt[k][0])));
                G[k] = in ? __fmul_rn(fts1, e) : 0.0f;
            }
            D1 = __fsub_rn(G[1], G[0]); D2 = __fsub_rn(G[2], G[0]);
            const float lg = __fmaf_rn(lam[2], G[2], __fmaf_rn(lam[1], G[1], __fmul_rn(lam[0], G[0])));
#pragma unroll
            for (int m = 0; m < 3; m++) P[m] = __fsub_rn(lg, G[m]);
        } else {
            constexpr bool kMip = kTex == 2;
            float uv[6], u, vv;
            nr::face_uvs(p.tex, b, tf, rev, uv);
            nr::pixel_uv(w, zp, z[0], z[1], z[2], uv, u, vv);
            // gu = sum_l a_l sum_c h_c Du_c^l (gv alike): d loss / d u with the light folded in (image_grad's kUvGrad sum)
            const nr::LevelPair lp = nr::level_pair<kMip>(p.tex, inv, w, zp, z[0], z[1], z[2], uv);
            const nr::UvTaps t0 = nr::uv_taps(u, vv, p.tex.level_h<kMip>(lp.l[0]), p.tex.level_w<kMip>(lp.l[0]));
            float gu, gv;
            nr::image_sample_grad<kMip>(p.tex, p.tex.tex + p.tex.img_off(b), lp, t0, u, vv, h, s, gu, gv);
            // G_k = gu u_k + gv v_k: differences of the UV corners (no fp32 cancellation for corners close together far
            // from 0), and sum_k l_k uv_k = the pixel's uv
            D1 = __fmaf_rn(gv, __fsub_rn(uv[3], uv[1]), __fmul_rn(gu, __fsub_rn(uv[2], uv[0])));
            D2 = __fmaf_rn(gv, __fsub_rn(uv[5], uv[1]), __fmul_rn(gu, __fsub_rn(uv[4], uv[0])));
#pragma unroll
            for (int m = 0; m < 3; m++) P[m] = __fmaf_rn(gv, __fsub_rn(vv, uv[2 * m + 1]), __fmul_rn(gu, __fsub_rn(u, uv[2 * m])));
        }
        if constexpr (kLight == nr::kLightCorner) {
            // smooth shading: d rgb_c / d l_k also holds C_kc s_c; with gs_c = g_c s_c the corner differences give
            // sum_c gs_c (C_kc - C_0c) and sum_c gs_c (L_c - C_mc)
            const float gs[3] = {g[0] * s[0], g[1] * s[1], g[2] * s[2]};
            float e1 = 0.0f, e2 = 0.0f;
#pragma unroll
            for (int ch = 0; ch < 3; ch++) {
                e1 = __fmaf_rn(gs[ch], __fsub_rn(C[3 + ch], C[ch]), e1);
                e2 = __fmaf_rn(gs[ch], __fsub_rn(C[6 + ch], C[ch]), e2);
            }
            D1 = __fadd_rn(D1, e1); D2 = __fadd_rn(D2, e2);
#pragma unroll
            for (int m = 0; m < 3; m++) {
                float e = 0.0f;
#pragma unroll
                for (int ch = 0; ch < 3; ch++) e = __fmaf_rn(gs[ch], __fsub_rn(L[ch], C[3 * m + ch]), e);
                P[m] = __fadd_rn(P[m], e);
            }
        }
        nr::perspective_vertex_grad(w, lam, z, lx, ly, D1, D2, P, __fmul_rn(fS, 0.5f), vg);
    }
    // the 9 floats of k_depth_grad's segmented run reduction (runs of neighbouring lanes that show the same face), then one
    // set of atomics per run
    const int fn_prev = __shfl_up_sync(0xffffffffu, fn, 1);
    const uint32_t heads = __ballot_sync(0xffffffffu, lane == 0 || fn != fn_prev);
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

}  // namespace

namespace nr_internal {

void launch_interior_grad(const InteriorLaunch& L, cudaStream_t stream) {
    const nr_b200_backward_args* a = L.args;
    const uint32_t flags = a->flags;
    InteriorParams p;
    memset(&p, 0, sizeof(p));
    p.src = L.src; p.dst = L.dst;
    p.fim = a->face_index_map; p.wmap = a->weight_map; p.g = a->grad_rgb;
    p.tex = L.tex;
    p.shading = L.shading;
    p.S = a->raster_size; p.F = a->num_faces; p.ts = a->texture_size;
    p.aa = (flags & NR_ANTI_ALIASING) ? 1 : 0;
    p.fill_back = (flags & NR_TEX_FILL_BACK) ? 1 : 0;
    const bool idx = (flags & NR_FACES_INDEXED) != 0;
    const int tex = (flags & NR_TEX_MIPMAP) ? 2 : (flags & NR_TEX_UV) ? 1 : 0;
    const dim3 grid((unsigned)(((size_t)p.S * p.S + 255) / 256), a->batch_size);
    LaunchScope ls("k_interior_grad", stream);
    nr::dispatch_light<nr::kLightNone, nr::kLightFace, nr::kLightCorner>(L.light, [&](auto kL) {
        nr::dispatch_bool(idx, [&](auto kIdx) {
            if (tex == 2) k_interior_grad<2, kL, kIdx><<<grid, 256, 0, stream>>>(p);
            else if (tex == 1) k_interior_grad<1, kL, kIdx><<<grid, 256, 0, stream>>>(p);
            else k_interior_grad<0, kL, kIdx><<<grid, 256, 0, stream>>>(p);
        });
    });
}

}  // namespace nr_internal
