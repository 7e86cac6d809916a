// nr_mip.cu -- mip pyramid of a texture image for trilinear sampling (NR_TEX_MIPMAP, include/nr_b200.h).
//
//   k_mip_build         one CTA per 32 x 32 texel tile of level 0 (per item): loads the tile into shared memory, copies
//                       it to level 0 of the pyramid and reduces it through levels 1..5 in shared memory.  A level-l+1
//                       texel only reads level-l texels of the same tile (its taps 2x, min(2x+1, W_l-1) stay inside),
//                       so the tiles are independent.
//   k_mip_build_coarse  levels 6.. (only when the image has more than 6 levels): one CTA per item walks the remaining
//                       levels through global memory (L2), a barrier between levels.  Two launches for any image size.
//   k_mip_collapse      the transpose of the build as a gather: every (level-0 texel, channel) walks up its ancestors
//                       (x >> l, y >> l) and sums their gradients times the product of m_x m_y / 4 over the steps,
//                       m = 2 where the edge clamp counts the child twice.  Each factor is a power of two, so the
//                       coefficients are exact; no atomics, deterministic.
// All sizes are in tap coordinates (x right, y up from the bottom row): level l row r holds y = H_l - 1 - r.
#include <cuda_runtime.h>
#include <stdint.h>

#include "nr_b200.h"
#include "nr_internal.h"
#include "nr_math.cuh"

namespace {

constexpr int kTileLog2 = 5;
constexpr int kTile = 1 << kTileLog2;  // level-0 texels per tile side; levels 1..kTileLog2 are reduced in the same CTA
constexpr int kCoarseThreads = 1024;

// texel (x, y) of level l+1 from the four level-l taps, in the order pinned in the header
__device__ __forceinline__ float mip_reduce(float a, float b, float c, float d) {
    return __fmul_rn(__fadd_rn(__fadd_rn(a, b), __fadd_rn(c, d)), 0.25f);
}

__global__ void __launch_bounds__(256) k_mip_build(const float* __restrict__ image, float* __restrict__ pyr, const nr::MipTable mt,
                                                   uint32_t pyr_floats, int tiles_x) {
    __shared__ float s_buf[2][kTile * kTile * 3];
    const int b = blockIdx.y;
    const int tx = (int)(blockIdx.x % (unsigned)tiles_x), ty = (int)(blockIdx.x / (unsigned)tiles_x);
    const int H = mt.h[0], W = mt.w[0];
    const float* img = image + (uint32_t)b * (uint32_t)(H * W * 3);  // < 2^31 (checked on the host)
    float* out = pyr + (uint32_t)b * pyr_floats;
    // level 0: 32 rows of 96 consecutive floats
    for (int e = threadIdx.x; e < kTile * kTile * 3; e += blockDim.x) {
        const int ly = e / (kTile * 3), rem = e - ly * (kTile * 3);
        const int gx = tx * kTile + rem / 3, gy = ty * kTile + ly;
        if (gx < W && gy < H) {
            const uint32_t o = ((uint32_t)(H - 1 - gy) * (uint32_t)W + (uint32_t)gx) * 3u + (uint32_t)(rem % 3);
            const float t = __ldg(img + o);
            out[o] = t;
            s_buf[0][e] = t;
        }
    }
    const int last = min(kTileLog2, mt.levels - 1);
    for (int j = 0; j < last; j++) {
        __syncthreads();
        const float* src = s_buf[j & 1];
        float* dst = s_buf[(j + 1) & 1];
        const int n = kTile >> (j + 1);
        const int Hs = mt.h[j], Ws = mt.w[j], Hd = mt.h[j + 1], Wd = mt.w[j + 1];
        const int bx_s = (tx * kTile) >> j, by_s = (ty * kTile) >> j;  // tile origin on the source level
        for (int e = threadIdx.x; e < n * n * 3; e += blockDim.x) {
            const int ly = e / (n * 3), rem = e - ly * (n * 3), lx = rem / 3, c = rem - lx * 3;
            const int gx = (bx_s >> 1) + lx, gy = (by_s >> 1) + ly;
            if (gx >= Wd || gy >= Hd) continue;
            const int x0 = 2 * lx, x1 = min(2 * gx + 1, Ws - 1) - bx_s;
            const int y0 = 2 * ly, y1 = min(2 * gy + 1, Hs - 1) - by_s;
            const float v = mip_reduce(src[(y0 * kTile + x0) * 3 + c], src[(y0 * kTile + x1) * 3 + c],
                                       src[(y1 * kTile + x0) * 3 + c], src[(y1 * kTile + x1) * 3 + c]);
            dst[(ly * kTile + lx) * 3 + c] = v;
            out[mt.off[j + 1] + ((uint32_t)(Hd - 1 - gy) * (uint32_t)Wd + (uint32_t)gx) * 3u + (uint32_t)c] = v;
        }
    }
}

__global__ void __launch_bounds__(kCoarseThreads) k_mip_build_coarse(float* __restrict__ pyr, const nr::MipTable mt, uint32_t pyr_floats) {
    float* out = pyr + (uint32_t)blockIdx.x * pyr_floats;
    for (int j = kTileLog2; j + 1 < mt.levels; j++) {
        const int Hs = mt.h[j], Ws = mt.w[j], Hd = mt.h[j + 1], Wd = mt.w[j + 1];
        const float* src = out + mt.off[j];  // written by k_mip_build or by this CTA before the barrier: plain loads
        float* dst = out + mt.off[j + 1];
        const int n = Hd * Wd * 3;
        for (int e = threadIdx.x; e < n; e += blockDim.x) {
            const int t = e / 3, c = e - t * 3;
            const int r = t / Wd, gx = t - r * Wd, gy = Hd - 1 - r;
            const int x0 = 2 * gx, x1 = min(2 * gx + 1, Ws - 1), y0 = 2 * gy, y1 = min(2 * gy + 1, Hs - 1);
            const int r0 = Hs - 1 - y0, r1 = Hs - 1 - y1;
            dst[e] = mip_reduce(src[(r0 * Ws + x0) * 3 + c], src[(r0 * Ws + x1) * 3 + c], src[(r1 * Ws + x0) * 3 + c],
                                src[(r1 * Ws + x1) * 3 + c]);
        }
        __syncthreads();
    }
}

__global__ void __launch_bounds__(256) k_mip_collapse(const float* __restrict__ gpyr, float* __restrict__ gimg, const nr::MipTable mt,
                                                      uint32_t pyr_floats, int accumulate) {
    const int H = mt.h[0], W = mt.w[0];
    const uint32_t n = (uint32_t)H * (uint32_t)W * 3u;
    const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n) return;
    const int b = blockIdx.y;
    const float* g = gpyr + (uint32_t)b * pyr_floats;
    const uint32_t t = e / 3u, c = e - t * 3u;
    int x = (int)(t % (uint32_t)W), y = H - 1 - (int)(t / (uint32_t)W);
    float acc = __ldg(g + e);
    float coef = 1.0f;
    for (int l = 1; l < mt.levels; l++) {
        const int mx = (x == mt.w[l - 1] - 1 && !(x & 1)) ? 2 : 1, my = (y == mt.h[l - 1] - 1 && !(y & 1)) ? 2 : 1;
        coef = __fmul_rn(coef, 0.25f * (float)(mx * my));  // a power of two: exact
        x >>= 1; y >>= 1;
        const uint32_t o = mt.off[l] + ((uint32_t)(mt.h[l] - 1 - y) * (uint32_t)mt.w[l] + (uint32_t)x) * 3u + c;
        acc = __fmaf_rn(coef, __ldg(g + o), acc);
    }
    float* dst = gimg + (uint32_t)b * n + e;
    *dst = accumulate ? __fadd_rn(*dst, acc) : acc;
}

// shared argument checks: sizes, 32-bit offsets of the whole batch of pyramids
int mip_check(int32_t Bt, int32_t Ht, int32_t Wt, nr::MipTable* mt, size_t* pyr_floats) {
    if (Bt < 1 || Ht < 1 || Wt < 1) return NR_ERR_INVALID_ARG;
    *pyr_floats = nr::mip_table(Ht, Wt, mt) * 3;
    if (Bt > 65535 || (size_t)Bt * *pyr_floats > 0x7FFFFFFFull) return NR_ERR_UNSUPPORTED;
    return NR_OK;
}

}  // namespace

extern "C" size_t nr_b200_mip_texels(int32_t Ht, int32_t Wt) { return nr::mip_table(Ht, Wt, nullptr); }

extern "C" int nr_b200_mip_build(const float* image, int32_t Bt, int32_t Ht, int32_t Wt, float* pyramid, void* cuda_stream) {
    nr_internal::launch_count() = 0;
    if (!image || !pyramid) return NR_ERR_INVALID_ARG;
    nr::MipTable mt;
    size_t pf = 0;
    const int rc = mip_check(Bt, Ht, Wt, &mt, &pf);
    if (rc != NR_OK) return rc;
    cudaStream_t stream = (cudaStream_t)cuda_stream;
    const int tiles_x = (Wt + kTile - 1) / kTile, tiles_y = (Ht + kTile - 1) / kTile;
    {
        nr_internal::LaunchScope ls("k_mip_build", stream);
        k_mip_build<<<dim3((unsigned)(tiles_x * tiles_y), (unsigned)Bt), 256, 0, stream>>>(image, pyramid, mt, (uint32_t)pf, tiles_x);
    }
    if (mt.levels > kTileLog2 + 1) {
        nr_internal::LaunchScope ls("k_mip_build", stream);
        k_mip_build_coarse<<<(unsigned)Bt, kCoarseThreads, 0, stream>>>(pyramid, mt, (uint32_t)pf);
    }
    return cudaGetLastError() == cudaSuccess ? NR_OK : NR_ERR_CUDA;
}

extern "C" int nr_b200_mip_collapse(const float* grad_pyramid, int32_t Bt, int32_t Ht, int32_t Wt, float* grad_image, uint32_t flags,
                                    void* cuda_stream) {
    nr_internal::launch_count() = 0;
    if (!grad_pyramid || !grad_image) return NR_ERR_INVALID_ARG;
    nr::MipTable mt;
    size_t pf = 0;
    const int rc = mip_check(Bt, Ht, Wt, &mt, &pf);
    if (rc != NR_OK) return rc;
    cudaStream_t stream = (cudaStream_t)cuda_stream;
    const size_t n = (size_t)Ht * Wt * 3;
    {
        nr_internal::LaunchScope ls("k_mip_collapse", stream);
        k_mip_collapse<<<dim3((unsigned)((n + 255) / 256), (unsigned)Bt), 256, 0, stream>>>(grad_pyramid, grad_image, mt, (uint32_t)pf,
                                                                                           (flags & NR_GRAD_ACCUMULATE) ? 1 : 0);
    }
    return cudaGetLastError() == cudaSuccess ? NR_OK : NR_ERR_CUDA;
}
