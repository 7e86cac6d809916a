// nr_interior.h -- host interface of the NR_GRAD_INTERIOR kernel (nr_interior.cu) for nr_b200_backward (not part of the ABI).
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

struct InteriorLaunch {
    const nr_b200_backward_args* args;  // the checked call (flags, maps, grad_rgb, textures, face_uvs)
    nr::FaceSrc src;
    nr::FaceGrad dst;
    nr::Shading shading;        // the call's face_light or corner_light (nr_internal::make_shading)
    int light;                  // its light mode: kLightNone, kLightFace or kLightCorner
    nr::Texture tex;            // what the pixel samples (nr_internal::make_texture)
};

// one launch of k_interior_grad, adding d loss / d vertices through l_k into src / dst's gradient (faces half); launch
// errors surface through the caller's cudaGetLastError
void launch_interior_grad(const InteriorLaunch& L, cudaStream_t stream);

}  // namespace nr_internal
