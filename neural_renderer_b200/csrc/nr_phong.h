// nr_phong.h -- host interface of the Phong-gradient kernel (nr_phong.cu) for the Phong light modes of the backward (not part of the ABI).
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include "nr_b200.h"
#include "nr_geom.cuh"
#include "nr_math.cuh"
#include "nr_shading.cuh"
#include "nr_texture.cuh"

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
    nr::Texture tex;                    // what the pixel samples (nr_internal::make_texture)
};

// one launch of k_phong_grad, adding into grad_corner_shading / grad_params (texture half); launch errors surface through
// the caller's cudaGetLastError
void launch_phong_grad(const PhongGradLaunch& L, cudaStream_t stream);

}  // namespace nr_internal
