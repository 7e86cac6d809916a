// nr_phong.h -- host interface of the Phong-gradient kernel (nr_phong.cu) for nr_b200_backward_phong (not part of the ABI).
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include "nr_b200.h"
#include "nr_geom.cuh"
#include "nr_math.cuh"

namespace nr_internal {

struct PhongGradLaunch {
    const nr_b200_backward_args* args;  // the checked call (flags, maps, grad_rgb, textures, face_uvs)
    const nr_b200_phong_args* phong;    // the checked Phong inputs and gradient outputs
    const nr_b200_lights_args* lights;  // the checked light set (NL > 0), or nullptr
    const nr_b200_sh_args* sh;          // the checked SH environment, or nullptr
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
