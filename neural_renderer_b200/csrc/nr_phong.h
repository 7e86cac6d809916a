// nr_phong.h -- host interface of the Phong-gradient kernel (nr_phong.cu) for the Phong light modes of the backward (not part of the ABI).
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include "nr_b200.h"
#include "nr_geom.cuh"
#include "nr_math.cuh"
#include "nr_shading.cuh"

namespace nr_internal {

struct PhongGradLaunch {
    const nr_b200_backward_args* args;  // the checked call (flags, maps, grad_rgb, textures, face_uvs)
    nr::Shading shading;                // the call's Phong inputs (nr_internal::make_shading)
    int light;                          // its light mode: kLightPhong, kLightPhongSet, kLightPhongSH, kLightPhongNM or kLightPhongSM
    float* grad_cs;                     // d loss / d corner_shading, params, lights (NL > 0) and sh, or nullptr
    float* grad_prm;
    float* grad_lts;
    float* grad_sh;
    float* grad_nm;                     // kLightPhongNM: d loss / d normal_map, corner_tangents, and the map's term of
    float* grad_tg;                     // d loss / d face_uvs, or nullptr
    float* grad_uvs;
    float* grad_sm;                     // kLightPhongSM: d loss / d specular_map, or nullptr
    nr::FaceSrc src;
    size_t tex_bstride;       // floats per item in `textures` (0 = shared)
    uint32_t uv_bstride;      // floats per item in face_uvs (0 = shared)
    float tex_cmp, tex_val;   // the cube clamp thresholds of the forward
    const nr::MipTable* mip;  // NR_TEX_MIPMAP: the pyramid's level table, else nullptr
};

// one launch of k_phong_grad, adding into grad_corner_shading / grad_params (texture half); launch errors surface through
// the caller's cudaGetLastError
void launch_phong_grad(const PhongGradLaunch& L, cudaStream_t stream);

}  // namespace nr_internal
