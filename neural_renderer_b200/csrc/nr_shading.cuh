// nr_shading.cuh -- what lights a pixel: the light mode of a call and the shading inputs it reads, the counterpart of
// nr_geom.cuh's "where a face comes from".
//
// The host picks the mode and fills one nr::Shading from the ABI arguments (nr_internal::make_shading, nr_internal.h);
// every kernel that shades or differentiates a pixel is instantiated per mode and reads its inputs from that record.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

#include <type_traits>

#include "nr_math.cuh"

namespace nr {

// The light modes, in the order of their template parameter kLight.
constexpr int kLightNone = 0;      // unlit
constexpr int kLightFace = 1;      // face_light [B,F,3] multiplies every texel inside the samplers.  The backward
                                   // kernels have no mode-1 instantiation: their kLightNone variant serves unlit and
                                   // face_light calls alike and tests the face_light pointer at run time.
constexpr int kLightCorner = 2;    // corner_light [B,F,3,3] interpolated to the pixel multiplies the unlit sample
constexpr int kLightPhong = 3;     // Phong shading of the unlit sample (corner_shading, params)
constexpr int kLightPhongSet = 4;  // the same with a light set of NL > 0 lights
constexpr int kLightPhongSH = 5;   // the same with an SH environment, and a light set of NL >= 0 lights
constexpr int kLightPhongNM = 6;   // Phong through a tangent-space normal map (NR_TEX_UV only), with a light set of NL >= 0
                                   // lights and an optional SH environment (both uniform per launch, decided at run time)
constexpr int kLightPhongSM = 7;   // Phong through a specular map (NR_TEX_UV only), with a light set of NL >= 0 lights, an
                                   // optional SH environment and an optional normal map (all uniform, decided at run time)

// The shading inputs of one call; strides are 0 for a set shared by every batch item.
struct Shading {
    const float* face_light;    // [B,F,3] (kLightFace), or nullptr
    const float* corner_light;  // [B,F,3,3] (kLightCorner), or nullptr
    const float* cs;            // corner_shading [Bc,F,3,6] (the Phong modes)
    const float* prm;           // params [Bp,16]
    size_t cs_bstride;          // faces per item in cs (0 with Bc = 1)
    size_t prm_bstride;         // floats per item in prm (0 with Bp = 1)
    const float* lts;           // lights [Bl,NL,12] (kLightPhongSet, kLightPhongSH), or nullptr with NL = 0
    size_t lt_bstride;          // floats per item in lts (0 with Bl = 1)
    int NL;
    const float* sh;            // [Bs,9,3] (kLightPhongSH)
    size_t sh_bstride;          // floats per item in sh (0 with Bs = 1)
    const float* nm;            // normal map [Bm,Hm,Wm,3] (kLightPhongNM)
    const float* tg;            // corner tangents [Bt,F,3,4] (kLightPhongNM)
    uint32_t nm_bstride;        // floats per item in nm (0 with Bm = 1; 32-bit, checked on the host)
    size_t tg_bstride;          // faces per item in tg (0 with Bt = 1)
    int Hm, Wm;
    const float* sm;            // specular map [Bq,Hq,Wq,4] (kLightPhongSM)
    uint32_t sm_bstride;        // floats per item in sm (0 with Bq = 1; 32-bit, checked on the host)
    int Hq, Wq;

    // float offsets of item b's records (and of face fn's; F = faces per item of the [B,F,...] light tensors), shared
    // with the gradients of the same layout
    __host__ __device__ __forceinline__ size_t fl_off(int b, int F, int fn) const { return ((size_t)b * F + fn) * 3; }
    __host__ __device__ __forceinline__ size_t cl_off(int b, int F, int fn) const { return ((size_t)b * F + fn) * 9; }
    __host__ __device__ __forceinline__ size_t cs_off(int b, int fn) const { return ((size_t)b * cs_bstride + fn) * 18; }
    __host__ __device__ __forceinline__ size_t prm_off(int b) const { return (size_t)b * prm_bstride; }
    __host__ __device__ __forceinline__ size_t lts_off(int b) const { return (size_t)b * lt_bstride; }
    __host__ __device__ __forceinline__ size_t sh_off(int b) const { return (size_t)b * sh_bstride; }
    __host__ __device__ __forceinline__ uint32_t nm_off(int b) const { return (uint32_t)b * nm_bstride; }
    __host__ __device__ __forceinline__ size_t tg_off(int b, int fn) const { return ((size_t)b * tg_bstride + fn) * 12; }
    __host__ __device__ __forceinline__ uint32_t sm_off(int b) const { return (uint32_t)b * sm_bstride; }
};

// kLightPhongNM: the map's sample at the pixel's (u, v) and the frame of face fn's pixel, the mapped normal in E.n
// (nr::nm_normal); m and the frame are returned for the backward
__device__ __forceinline__ void nm_pixel_normal(const Shading& s, int b, int fn, const float l[3], float u, float v, float m[3],
                                                NmFrame& F, PhongEval& E) {
    float du[3], dv[3];
    nm_sample<false>(s.nm + s.nm_off(b), s.Hm, s.Wm, uv_taps(u, v, s.Hm, s.Wm), m, du, dv);
    nm_normal(s.cs + s.cs_off(b, fn), s.tg + s.tg_off(b, fn), l, m, F, E.n);
}
// kLightPhongSM: the specular map's sample sq = (ks, sigma') at the pixel's (u, v)
__device__ __forceinline__ void sm_pixel_sample(const Shading& s, int b, float u, float v, float sq[4]) {
    float du[4], dv[4];
    sm_sample<false>(s.sm + s.sm_off(b), s.Hq, s.Wq, uv_taps(u, v, s.Hq, s.Wq), sq, du, dv);
}

// What the Phong modes read besides corner_shading and params: modes 3-5 fix it at compile time, the maps' modes 6-7
// test the light set (NL >= 0), the SH environment and (mode 7) the normal map at run time, uniform per launch.
template <int kLight>
__device__ __forceinline__ bool reads_sh(const Shading& s) {
    return kLight == kLightPhongSH || (kLight >= kLightPhongNM && s.sh);
}
// E.n of a Phong mode's pixel (cs = face fn's corner_shading): the mapped normal n' at the pixel's (u, v), or the
// interpolated n
template <int kLight>
__device__ __forceinline__ void pixel_normal(const Shading& s, int b, int fn, const float* cs, const float l[3], float u, float v,
                                             PhongEval& E) {
    if (kLight == kLightPhongNM || (kLight == kLightPhongSM && s.nm)) {  // uniform
        NmFrame F;
        float m[3];
        nm_pixel_normal(s, b, fn, l, u, v, m, F, E);
    } else {
        phong_normal(cs, l, E.n);
    }
}

// L_c = d rgb_c / d s_c of face fn's pixel with perspective weights l (own vertex depths) and uv (u, v) (read by the
// normal map only): 1, face_light, the interpolated corner light, or the diffuse part of the Phong expression (with the
// set's diffuse terms, then E_c).  The specular map never enters L_c.
template <int kLight>
__device__ __forceinline__ void pixel_light(const Shading& s, int b, int F, int fn, const float l[3], float u, float v,
                                            float L[3]) {
    if constexpr (kLight == kLightNone) {
        L[0] = L[1] = L[2] = 1.0f;
    } else if constexpr (kLight == kLightFace) {
        const float* lp = s.face_light + s.fl_off(b, F, fn);
        L[0] = __ldg(lp); L[1] = __ldg(lp + 1); L[2] = __ldg(lp + 2);
    } else if constexpr (kLight == kLightCorner) {
        corner_light_at(s.corner_light + s.cl_off(b, F, fn), l, L);
    } else {
        const float* cs = s.cs + s.cs_off(b, fn);
        PhongEval E;
        if constexpr (kLight >= kLightPhongNM) {  // modes 3-5 form params' address before the normal, which their SASS keeps
            pixel_normal<kLight>(s, b, fn, cs, l, u, v, E);
            phong_diffuse_n(s.prm + s.prm_off(b), E);
        } else {
            phong_diffuse(cs, l, s.prm + s.prm_off(b), E);
        }
        if constexpr (kLight >= kLightPhongSet) {
            if (kLight < kLightPhongNM || s.NL > 0) {  // uniform
                float pos[3];
                phong_position(cs, l, pos);
                lights_diffuse_loop(s.lts + s.lts_off(b), s.NL, pos, E);
            }
        }
        if (reads_sh<kLight>(s)) sh_add_irradiance(s.sh + s.sh_off(b), E);  // uniform
        L[0] = E.L[0]; L[1] = E.L[1]; L[2] = E.L[2];
    }
}

// rgb of face fn's pixel from its unlit sample c (in place), perspective weights l and uv (u, v) (read by the maps
// only), for the modes that shade the sample after sampling (kLightCorner and the Phong modes; face_light is applied
// per texel by the samplers).  With NL = 0 and no environment phong_lights_rgb is phong_rgb, so a flat normal map and a
// constant (1, 1, 1, sigma) specular map render as modes 3-5 do, bit for bit.
template <int kLight>
__device__ __forceinline__ void shade(const Shading& s, int b, int F, int fn, const float l[3], float u, float v, float c[3]) {
    static_assert(kLight >= kLightCorner, "unlit and face_light samples are final");
    if constexpr (kLight == kLightCorner) {
        float L[3];
        corner_light_at(s.corner_light + s.cl_off(b, F, fn), l, L);
        c[0] = __fmul_rn(L[0], c[0]); c[1] = __fmul_rn(L[1], c[1]); c[2] = __fmul_rn(L[2], c[2]);
    } else {
        const float* prm = s.prm + s.prm_off(b);
        const float* lts = s.lts + s.lts_off(b);  // the set modes
        const float* cs = s.cs + s.cs_off(b, fn);
        float sq[4];  // kLightPhongSM: K' and sigma' come from the specular map
        const float* q = kLight == kLightPhongSM ? sq : nullptr;
        PhongEval E;
        pixel_normal<kLight>(s, b, fn, cs, l, u, v, E);
        if constexpr (kLight == kLightPhongSM) sm_pixel_sample(s, b, u, v, sq);
        phong_diffuse_n(prm, E);
        phong_specular(cs, l, prm, E, q);
        float rgb[3];
        if constexpr (kLight == kLightPhong) {
            phong_rgb(E, prm, c, rgb);
        } else {
            float pos[3];
            phong_position(cs, l, pos);
            lights_diffuse_loop(lts, s.NL, pos, E);
            if (reads_sh<kLight>(s)) sh_add_irradiance(s.sh + s.sh_off(b), E);  // uniform
            phong_lights_rgb(E, pos, prm, lts, s.NL, c, rgb, q);
        }
        c[0] = rgb[0]; c[1] = rgb[1]; c[2] = rgb[2];
    }
}

// Host-side dispatch of a run-time choice to a compile-time one.  dispatch_light<kModes...>(mode, fn) calls
// fn(std::integral_constant<int, M>{}) for the M of kModes equal to mode (the modes the launched kernel is instantiated
// for; the caller never passes another, the last listed one would take it) and returns what fn returns.
template <int kMode, int... kRest, class Fn>
inline auto dispatch_light(int mode, Fn&& fn) {
    if constexpr (sizeof...(kRest) > 0) {
        if (mode != kMode) return dispatch_light<kRest...>(mode, fn);
    }
    return fn(std::integral_constant<int, kMode>{});
}
// fn(std::true_type{}) or fn(std::false_type{})
template <class Fn>
inline auto dispatch_bool(bool v, Fn&& fn) {
    return v ? fn(std::true_type{}) : fn(std::false_type{});
}

}  // namespace nr
