// nr_texture.cuh -- what a pixel samples: per-face texture cubes, a texture image through face_uvs, or its mip pyramid,
// the counterpart of nr_geom.cuh's "where a face comes from" and nr_shading.cuh's "what lights the pixel".
//
// The host fills one nr::Texture from the ABI arguments (nr_internal::make_texture, nr_internal.h); every kernel that
// samples or differentiates a pixel's texels reads its inputs from that record.  The gradients (grad_textures,
// grad_face_uvs) stay in the kernels' own structs and share the record's offsets, as they have the same layouts.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include "nr_math.cuh"

namespace nr {

// The sampler inputs of one call; strides are 0 for a texture or UV set shared by every batch item.  The cube size ts
// is not in the record: like B, F and S it is one of the call's sizes (texture_size of the ABI) and the parameter structs
// keep it beside them.
struct Texture {
    const float* tex;       // cubes [Bt,F',ts,ts,ts,3], image [Bt,Ht,Wt,3] (NR_TEX_UV) or packed pyramid [Bt,P,3]
                            // (NR_TEX_MIPMAP); F' = F/2 stored faces with NR_TEX_FILL_BACK, else F
    size_t cube_bstride;    // cubes per item in tex
    const float* uvs;       // NR_TEX_UV: face_uvs [Bu,F',3,2]
    uint32_t uv_bstride;    // floats per item in uvs (32-bit, checked on the host)
    uint32_t img_bstride;   // floats per item in the image / pyramid (likewise)
    int Ht, Wt;             // level-0 size of the image
    MipTable mip;           // NR_TEX_MIPMAP: the pyramid's levels
    float tex_cmp, tex_val; // cubes: the clamp of texture_coords (largest float <= ts - 1 - eps, and ts - 1 - eps)

    // float offsets of item b's cube of stored face tf (ts texels per axis), of item b's image, and of face tf's UV corners
    __host__ __device__ __forceinline__ size_t cube_off(int b, int tf, int ts) const {
        return ((size_t)b * cube_bstride + tf) * (size_t)(ts * ts * ts) * 3;
    }
    __host__ __device__ __forceinline__ uint32_t img_off(int b) const { return (uint32_t)b * img_bstride; }
    __host__ __device__ __forceinline__ uint32_t uv_off(int b, int tf) const {
        return (uint32_t)b * uv_bstride + (uint32_t)tf * 6u;
    }
    // level l of the image (kMip: of the pyramid; the bilinear sampler has level 0 only)
    template <bool kMip>
    __device__ __forceinline__ int level_h(int l) const { return kMip ? mip.h[l] : Ht; }
    template <bool kMip>
    __device__ __forceinline__ int level_w(int l) const { return kMip ? mip.w[l] : Wt; }
    template <bool kMip>
    __device__ __forceinline__ uint32_t level_off(int l) const { return kMip ? mip.off[l] : 0u; }
};

// NR_TEX_FILL_BACK (fill_back = flags & NR_TEX_FILL_BACK): face fn >= F/2 is the reversed copy of face fn - F/2 and
// samples that stored face's cube with reversed axes, or its UV corners in reverse order.  Returns the stored face.
__device__ __forceinline__ int stored_face(bool fill_back, int F, int fn, bool& rev) {
    int tf = fn;
    rev = false;
    if (fill_back) {
        const int half = F >> 1;
        if (fn >= half) { tf = fn - half; rev = true; }
    }
    return tf;
}

// the UV corners of stored face tf of item b (rev: a fill_back copy's, reversed)
__device__ __forceinline__ void face_uvs(const Texture& t, int b, int tf, bool rev, float uv[6]) {
    load_face_uvs(t.uvs + t.uv_off(b, tf), rev, uv);
}

// rasterize.py:415-426: the 8-corner blend of cube `cube` at tc (rev: a fill_back copy's reversed axes), every texel
// times lt[0..2] first when kLit (face_light, rounded like the materialised product).  kLdg: the texels are read through
// the read-only cache; without it by plain loads, which also reach a cube k_resolve staged in shared memory.
template <bool kLit, bool kLdg>
__device__ __forceinline__ void cube_blend(const float* cube, const TexCoord& tc, int ts, bool rev, const float* lt, float& r,
                                           float& g, float& bl) {
    float l0 = 1.0f, l1 = 1.0f, l2 = 1.0f;
    if (kLit) {
        l0 = __ldg(lt); l1 = __ldg(lt + 1); l2 = __ldg(lt + 2);
    }
    r = g = bl = 0.0f;
#pragma unroll
    for (int pn = 0; pn < 8; pn++) {
        const float cw = corner_weight(tc, pn);
        const float* t = cube + (rev ? corner_index_rev(tc, pn, ts) : corner_index(tc, pn, ts)) * 3;
        float t0 = kLdg ? __ldg(t) : t[0], t1 = kLdg ? __ldg(t + 1) : t[1], t2 = kLdg ? __ldg(t + 2) : t[2];
        if (kLit) {
            t0 = __fmul_rn(t0, l0); t1 = __fmul_rn(t1, l1); t2 = __fmul_rn(t2, l2);
        }
        r = __fmaf_rn(cw, t0, r);
        g = __fmaf_rn(cw, t1, g);
        bl = __fmaf_rn(cw, t2, bl);
    }
}

// The levels an image sample reads and their weights a: the bilinear sampler reads level 0 with weight 1; the trilinear
// one (kMip) levels l0 and l1 of mip_levels at the pixel's level of detail, with weights 1 - f and f (n = 1 when f = 0).
struct LevelPair {
    int l[2];
    float a[2];
    int n;
};
template <bool kMip>
__device__ __forceinline__ LevelPair level_pair(const Texture& t, const float inv[9], const float w[3], float zp, float z0,
                                                float z1, float z2, const float uv[6]) {
    LevelPair L = {{0, 0}, {1.0f, 0.0f}, 1};
    if constexpr (kMip) {
        const MipLevels m = mip_levels(mip_lod(inv, w, zp, z0, z1, z2, uv, t.Ht, t.Wt, t.mip.levels), t.mip.levels);
        L.l[0] = m.l0; L.l[1] = m.l1;
        L.a[0] = __fsub_rn(1.0f, m.f); L.a[1] = m.f;
        L.n = m.f != 0.0f ? 2 : 1;
    }
    return L;
}

// The unlit image sample s at (u, v) over the levels of L (bit for bit uv_blend / mip_blend) and gu = sum_l a_l sum_c h_c
// du_c^l (gv alike), h = d loss / d s: the derivative of uv_blend_grad with cells and levels held fixed.  img = the
// item's image or pyramid, t0 = the taps of level L.l[0].
template <bool kMip>
__device__ __forceinline__ void image_sample_grad(const Texture& t, const float* img, const LevelPair& L, const UvTaps& t0,
                                                  float u, float v, const float h[3], float s[3], float& gu, float& gv) {
    gu = 0.0f; gv = 0.0f;
#pragma unroll
    for (int q = 0; q < 2; q++) {
        if (q >= L.n) break;
        const int Hl = t.level_h<kMip>(L.l[q]), Wl = t.level_w<kMip>(L.l[q]);
        const UvTaps tq = q == 0 ? t0 : uv_taps(u, v, Hl, Wl);
        float bl[3], du[3], dv[3];
        uv_blend_grad(img + t.level_off<kMip>(L.l[q]), Hl, Wl, tq, bl, du, dv);
#pragma unroll
        for (int k = 0; k < 3; k++) s[k] = q == 0 ? bl[k] : __fmaf_rn(L.a[1], bl[k], __fmul_rn(L.a[0], s[k]));  // mip_blend
        const float eu = __fmaf_rn(h[2], du[2], __fmaf_rn(h[1], du[1], __fmul_rn(h[0], du[0])));
        const float ev = __fmaf_rn(h[2], dv[2], __fmaf_rn(h[1], dv[1], __fmul_rn(h[0], dv[0])));
        gu = __fmaf_rn(L.a[q], eu, gu);
        gv = __fmaf_rn(L.a[q], ev, gv);
    }
}

}  // namespace nr
