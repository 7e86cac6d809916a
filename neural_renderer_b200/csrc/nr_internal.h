// nr_internal.h -- host-side helpers shared by the translation units of libnr_b200.so (not part of the ABI).
#pragma once
#include <cuda_runtime.h>

#include <math.h>

#include <atomic>

#include "nr_b200.h"
#include "nr_geom.cuh"
#include "nr_shading.cuh"
#include "nr_texture.cuh"

namespace nr_internal {
// kernels launched by the last forward/backward call on this thread (nr_b200_last_launch_count)
std::atomic<int>& launch_count();
// optional per-kernel CUDA-event timing on the launching stream (nr_b200_set_profiling / nr_b200_read_profile)
void prof_begin(const char* name, cudaStream_t stream);
void prof_end(cudaStream_t stream);

struct LaunchScope {
    cudaStream_t s;
    LaunchScope(const char* name, cudaStream_t stream) : s(stream) { prof_begin(name, s); }
    ~LaunchScope() { prof_end(s); launch_count()++; }
};

// Exclusive prefix sums of nseg segments of seg_len counters, segment i offset by i * seg_stride (k_strip_scan of
// nr_backward.cu, also the tile scan of the soft silhouettes)
void strip_scan(const int* cnt, int* off, int seg_len, long long seg_stride, int nseg, cudaStream_t stream);

// The soft RGB's host half (nr_soft_rgb.cu), shared by the cube and the texture-image units.  `params` / `layout` point
// to nr_soft_rgb.cuh's SoftRgbParams / SoftRgbLayout, which each unit compiles in its own anonymous namespace (as its
// kernels), so they pass by address.
//   soft_rgb_check      the NR_ERR_INVALID_ARG rules of nr_b200_soft_rgb(_backward) with `allowed` flags for the colour
//                       source `src`: kSoftImage skips texture_size and eps (the caller fills params->tex), kSoftAttributes
//                       also textures and rgb (nr_soft_attr.cu has its own colour buffers), kSoftFragments also gamma,
//                       alpha and state (nr_soft_frag.cu has no softmax); fills everything but the workspace
//   soft_rgb_workspace  NR_ERR_WORKSPACE / NR_ERR_CUDA: the layout (soft_rgb_layout) and the workspace pointers
//   soft_rgb_bin        the tile binning (bin_faces_rgb): setup, scan, depth records and keys, sorted when `sort`
enum SoftColourSource { kSoftCubes, kSoftImage, kSoftAttributes, kSoftFragments };
int soft_rgb_check(const nr_b200_soft_rgb_args* a, uint32_t allowed, SoftColourSource src, bool backward, void* params);
int soft_rgb_workspace(const nr_b200_soft_rgb_args* a, void* params, void* layout);
int soft_rgb_bin(void* params, const void* layout, bool sort, cudaStream_t stream);

// FaceSrc / FaceGrad of a call from its ABI arguments; false = missing pointers for the chosen geometry form
inline bool make_face_src(uint32_t flags, const float* faces, const float* vertices, const int32_t* indices, int F, int Nv,
                          nr::FaceSrc* s) {
    s->F = F; s->Nv = 0; s->faces = nullptr; s->vertices = nullptr; s->idx = nullptr; s->idx_bstride = 0;
    if (flags & NR_FACES_INDEXED) {
        if (!vertices || !indices || Nv <= 0) return false;
        s->vertices = vertices; s->idx = indices; s->Nv = Nv;
        s->idx_bstride = (flags & NR_INDICES_SHARED) ? 0 : (long long)F * 3;
        return true;
    }
    if (!faces) return false;
    s->faces = faces;
    return true;
}
inline bool make_face_grad(uint32_t flags, float* grad_faces, float* grad_vertices, const int32_t* indices, int F, int Nv,
                           nr::FaceGrad* g) {
    g->F = F; g->Nv = 0; g->grad_faces = nullptr; g->grad_vertices = nullptr; g->idx = nullptr; g->idx_bstride = 0;
    if (flags & NR_FACES_INDEXED) {
        if (!grad_vertices || !indices || Nv <= 0) return false;
        g->grad_vertices = grad_vertices; g->idx = indices; g->Nv = Nv;
        g->idx_bstride = (flags & NR_INDICES_SHARED) ? 0 : (long long)F * 3;
        return true;
    }
    if (!grad_faces) return false;
    g->grad_faces = grad_faces;
    return true;
}

// the checks every Phong entry point makes on its nr_b200_phong_args (the size first: only then are the fields read)
inline bool phong_args_ok(const nr_b200_phong_args* ph, int B) {
    return ph->struct_size == sizeof(nr_b200_phong_args) && ph->corner_shading && ph->params &&
           (ph->shading_batch == 1 || ph->shading_batch == B) && (ph->params_batch == 1 || ph->params_batch == B);
}

// the same for a light set (nr_b200_lights_args); NL = 0 needs no lights pointer
constexpr int kMaxLights = 8;
inline bool lights_args_ok(const nr_b200_lights_args* ls, int B) {
    return ls->struct_size == sizeof(nr_b200_lights_args) && ls->num_lights >= 0 && ls->num_lights <= kMaxLights &&
           (ls->lights || ls->num_lights == 0) && (ls->lights_batch == 1 || ls->lights_batch == B);
}

// the same for an SH environment (nr_b200_sh_args)
inline bool sh_args_ok(const nr_b200_sh_args* sh, int B) {
    return sh->struct_size == sizeof(nr_b200_sh_args) && sh->sh && (sh->sh_batch == 1 || sh->sh_batch == B);
}

// the same for a normal map (nr_b200_normal_map_args)
inline bool nm_args_ok(const nr_b200_normal_map_args* nm, int B) {
    return nm->struct_size == sizeof(nr_b200_normal_map_args) && nm->normal_map && nm->corner_tangents &&
           (nm->map_batch == 1 || nm->map_batch == B) && (nm->tangent_batch == 1 || nm->tangent_batch == B) &&
           nm->map_height >= 1 && nm->map_width >= 1;
}
// floats of one item's normal map (the kernels' offsets into it are 32-bit: the caller refuses more than 2^31 - 1 in all)
inline size_t nm_floats(const nr_b200_normal_map_args* nm) { return (size_t)nm->map_height * (size_t)nm->map_width * 3; }

// the same for a specular map (nr_b200_specular_map_args); its texels are read as aligned 16-byte vectors
inline bool sm_args_ok(const nr_b200_specular_map_args* sm, int B) {
    return sm->struct_size == sizeof(nr_b200_specular_map_args) && sm->specular_map &&
           ((uintptr_t)sm->specular_map & 15) == 0 && (sm->map_batch == 1 || sm->map_batch == B) && sm->map_height >= 1 &&
           sm->map_width >= 1;
}
// floats of one item's specular map (32-bit offsets in the kernels, as nm_floats)
inline size_t sm_floats(const nr_b200_specular_map_args* sm) { return (size_t)sm->map_height * (size_t)sm->map_width * 4; }

// The Phong inputs of a call as the ABI passes them, each NULL when absent (all NULL: no Phong shading).  Every Phong
// entry point is nr_b200_*_specular_map with its missing trailing structs NULL.
struct PhongCall {
    const nr_b200_phong_args* phong;
    const nr_b200_lights_args* lights;
    const nr_b200_sh_args* sh;
    const nr_b200_normal_map_args* nm;
    const nr_b200_specular_map_args* sm;
};

// What a Phong entry point returns for a NULL phong struct: nothing else is read and nothing is launched
inline int refuse_null_phong() {
    launch_count() = 0;
    return NR_ERR_INVALID_ARG;
}

// The light mode (nr_shading.cuh) and nr::Shading of a call from its ABI arguments, or -1 for a refused combination
// (NR_ERR_INVALID_ARG): corner_light only for RGB and instead of face_light; Phong only for RGB and instead of both; the
// Phong, light-set, SH, normal-map and specular-map structs pass their checks.  face_light is ignored without RGB, and a
// set of NL = 0 lights is the Phong call exactly.
inline int make_shading(bool rgb, const float* face_light, const float* corner_light, const PhongCall& c, int B, int F,
                        nr::Shading* s) {
    auto [phong, lights, sh, nm, sm] = c;
    *s = nr::Shading{};
    if (corner_light && (!rgb || face_light)) return -1;
    if (phong && (!rgb || face_light || corner_light || !phong_args_ok(phong, B))) return -1;
    if (lights && !lights_args_ok(lights, B)) return -1;
    if (sh && !sh_args_ok(sh, B)) return -1;
    if (nm && (!phong || !nm_args_ok(nm, B))) return -1;
    if (sm && (!phong || !sm_args_ok(sm, B))) return -1;
    if (lights && lights->num_lights == 0) lights = nullptr;
    s->face_light = rgb ? face_light : nullptr;
    s->corner_light = corner_light;
    if (phong) {
        s->cs = phong->corner_shading; s->prm = phong->params;
        s->cs_bstride = phong->shading_batch == 1 ? 0 : (size_t)F;
        s->prm_bstride = phong->params_batch == 1 ? 0 : 16;
    }
    if (lights) {
        s->lts = lights->lights; s->NL = lights->num_lights;
        s->lt_bstride = lights->lights_batch == 1 ? 0 : (size_t)lights->num_lights * 12;
    }
    if (sh) {
        s->sh = sh->sh;
        s->sh_bstride = sh->sh_batch == 1 ? 0 : 27;
    }
    if (nm) {
        s->nm = nm->normal_map; s->tg = nm->corner_tangents;
        s->nm_bstride = nm->map_batch == 1 ? 0u : (uint32_t)nm_floats(nm);
        s->tg_bstride = nm->tangent_batch == 1 ? 0 : (size_t)F;
        s->Hm = nm->map_height; s->Wm = nm->map_width;
    }
    if (sm) {
        s->sm = sm->specular_map;
        s->sm_bstride = sm->map_batch == 1 ? 0u : (uint32_t)sm_floats(sm);
        s->Hq = sm->map_height; s->Wq = sm->map_width;
        return nr::kLightPhongSM;
    }
    if (nm) return nr::kLightPhongNM;
    if (sh) return nr::kLightPhongSH;
    if (lights) return nr::kLightPhongSet;
    if (phong) return nr::kLightPhong;
    if (corner_light) return nr::kLightCorner;
    return s->face_light ? nr::kLightFace : nr::kLightNone;
}

inline float float_le(double d) {  // largest float <= d
    float f = (float)d;
    if ((double)f > d) f = nextafterf(f, -INFINITY);
    return f;
}

// The nr::Texture of a call from its ABI arguments (nr_b200_forward_args or nr_b200_backward_args), and the floats of
// its whole texel and face_uvs buffers (the sizes of their gradients).  Returns NR_ERR_INVALID_ARG for a refused
// combination: NR_TEX_UV without RGB, face_uvs or an image of at least 1 x 1; NR_TEX_MIPMAP without NR_TEX_UV; RGB cubes
// with ts < 2; RGB with NR_TEX_FILL_BACK and an odd F.  Returns NR_ERR_UNSUPPORTED when the image or UV offsets do not
// fit the kernels' 32 bits.  The caller returns NR_ERR_INVALID_ARG at once and NR_ERR_UNSUPPORTED after its own
// NR_ERR_INVALID_ARG rules.
template <class Args>
inline int make_texture(const Args* a, nr::Texture* t, size_t* tex_floats, size_t* uv_floats) {
    const uint32_t flags = a->flags;
    const bool rgb = (flags & NR_RETURN_RGB) != 0, uv = (flags & NR_TEX_UV) != 0, mip = (flags & NR_TEX_MIPMAP) != 0;
    const int B = a->batch_size, F = a->num_faces, ts = a->texture_size;
    *t = nr::Texture{};
    if (uv && (!rgb || !a->face_uvs || a->texture_height < 1 || a->texture_width < 1)) return NR_ERR_INVALID_ARG;
    if (mip && !uv) return NR_ERR_INVALID_ARG;
    if (rgb && !uv && ts < 2) return NR_ERR_INVALID_ARG;
    if (rgb && (flags & NR_TEX_FILL_BACK) && (F & 1)) return NR_ERR_INVALID_ARG;
    const size_t faces = (flags & NR_TEX_FILL_BACK) ? (size_t)F / 2 : (size_t)F;  // stored faces per item
    const size_t tex_items = (flags & NR_TEX_SHARED) ? 1 : (size_t)B, uv_items = (flags & NR_UV_SHARED) ? 1 : (size_t)B;
    t->tex = a->textures;
    t->cube_bstride = (flags & NR_TEX_SHARED) ? 0 : faces;
    const double tmax = (double)(ts - 1) - a->eps;
    t->tex_cmp = float_le(tmax);
    t->tex_val = (float)tmax;
    *uv_floats = 0;
    if (!uv) {
        *tex_floats = tex_items * faces * ts * ts * ts * 3;
        return NR_OK;
    }
    const size_t img_floats = mip ? nr::mip_table(a->texture_height, a->texture_width, &t->mip) * 3
                                  : (size_t)a->texture_height * (size_t)a->texture_width * 3;
    *tex_floats = tex_items * img_floats;
    *uv_floats = uv_items * faces * 6;
    if (*tex_floats > 0x7FFFFFFFull || *uv_floats > 0x7FFFFFFFull) return NR_ERR_UNSUPPORTED;
    t->uvs = a->face_uvs;
    t->uv_bstride = (flags & NR_UV_SHARED) ? 0u : (uint32_t)(faces * 6);
    t->img_bstride = (flags & NR_TEX_SHARED) ? 0u : (uint32_t)img_floats;
    t->Ht = a->texture_height; t->Wt = a->texture_width;
    return NR_OK;
}

// cudaFuncSetAttribute(MaxDynamicSharedMemorySize) is issued once per (kernel instantiation, device, size high-water
// mark) instead of on every launch: `slot` is a function-local static of the launching template.
struct SmemOptIn {
    static constexpr int kMaxDevices = 64;
    std::atomic<int> bytes[kMaxDevices];
    SmemOptIn() { for (auto& b : bytes) b.store(0, std::memory_order_relaxed); }
    template <typename Kernel>
    cudaError_t ensure(Kernel kernel, size_t need) {
        int dev = 0;
        cudaError_t e = cudaGetDevice(&dev);
        if (e != cudaSuccess) return e;
        if (dev < 0 || dev >= kMaxDevices) return cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)need);
        if ((int)need <= bytes[dev].load(std::memory_order_acquire)) return cudaSuccess;
        e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)need);
        if (e == cudaSuccess) bytes[dev].store((int)need, std::memory_order_release);
        return e;
    }
};
}  // namespace nr_internal
