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

// what k_phong_grad writes, each in the layout of its input, or nullptr
struct PhongGrads {
    float *cs, *prm, *lts, *sh;  // d loss / d corner_shading, params, lights (NL > 0) and sh
    float *nm, *tg, *sm;         // d loss / d normal_map, corner_tangents and specular_map
    float* uvs;                  // with a map: the maps' term of d loss / d face_uvs
};

struct PhongGradLaunch {
    const nr_b200_backward_args* args;  // the checked call (flags, maps, grad_rgb, textures, face_uvs)
    nr::Shading shading;                // the call's Phong inputs (nr_internal::make_shading)
    PhongGrads grad;
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
