// nr_soft_blend.cu -- the soft blend of fragments (nr_b200_blend_fragments / nr_b200_blend_fragments_backward,
// include/nr_b200.h): SoftRas's depth softmax over the K slots of every pixel, with gradients into the per-slot colours,
// the depths and the signed distances.  Pixel-local streaming passes, no atomics, no workspace.
//
//   k_soft_blend_fwd<kStaged>  one thread per pixel, kPix consecutive pixels per CTA.  The weights of the K slots are
//                              computed once (blend_weights) into a shared [K][kPix] column, then the colours are
//                              reduced kCB channels at a time in slot order, and out is written planar (coalesced).
//   k_soft_blend_bwd<kStaged>  the same weights from the same device function, H_k accumulated over the channel blocks,
//                              and grad_colors, grad_zbuf and grad_dists written pixel-locally.
// kStaged: the CTA's contiguous ranges of pix_to_face (as a validity flag), zbuf, dists and colours are first copied into
// shared memory with coalesced loads (16-byte vectors when every address allows), padded by one word every 32 so that
// the per-thread reads at stride K and K C are free of bank conflicts; the backward's outputs are assembled there and
// written back coalesced.  Without staging every thread reads and writes its own slots in global memory.  Staging is
// used whenever the tile fits kStageBudget (DESIGN.md 4t has the measured comparison).
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <string.h>

#include "nr_b200.h"
#include "nr_internal.h"

namespace {

constexpr int kMaxK = 32;                  // the fragments' own cap
constexpr int kPix = 64;                   // pixels (threads) per CTA
constexpr int kCB = 4;                     // channels per block held in registers
constexpr size_t kStageBudget = 96 * 1024; // the largest staged tile (bytes of dynamic shared memory)

struct BlendParams {
    const long long* p2f;    // [N,K]  (N = B H W pixels)
    const float* zbuf;       // [N,K]
    const float* dists;      // [N,K]
    const float* col;        // [N,K,C]
    const float* bg;         // [C] or nullptr
    float* out;              // [B,C,HW]
    float* alpha;            // [B,HW] (forward)
    const float* g_out;      // backward: [B,C,HW] or nullptr
    const float* g_alpha;    // backward: [B,HW] or nullptr
    float* g_col;            // backward: [N,K,C] or nullptr
    float* g_zbuf;           // backward: [N,K] or nullptr
    float* g_dists;          // backward: [N,K] or nullptr
    long long npix, hw;
    int K, C;
    float inv_sigma;         // 1 / sigma
    float inv_fg;            // 1 / ((far - near) gamma)
    float zp_bg;             // far - NR_SOFT_BG_DEPTH (far - near)
    bool vec;                // every staged array 16-byte aligned (CTA ranges start at multiples of kPix pixels)
};

// a staged array of n words, padded by one word every 32
__host__ __device__ __forceinline__ int padi(int e) { return e + (e >> 5); }
__host__ __device__ __forceinline__ int padn(int n) { return n + (n >> 5) + 1; }

__device__ __forceinline__ float blend_sigmoid(float x) {
    const float e = expf(-fabsf(x));
    return x >= 0.0f ? __frcp_rn(1.0f + e) : __fdiv_rn(e, 1.0f + e);
}

// The inputs of one pixel, from global memory or from the CTA's staged tile.
struct Slots {
    const long long* p2f;
    const float *z, *d, *c;        // global: the pixel's own slots; staged: the tile
    const int* f;                  // staged validity flags
    int base, K, C;                // staged: the pixel's first word (tid K) and sizes
    bool staged;
    __device__ __forceinline__ bool valid(int k) const { return staged ? f[padi(base + k)] != 0 : __ldg(p2f + k) >= 0; }
    __device__ __forceinline__ float zb(int k) const { return staged ? z[padi(base + k)] : __ldg(z + k); }
    __device__ __forceinline__ float ds(int k) const { return staged ? d[padi(base + k)] : __ldg(d + k); }
    __device__ __forceinline__ float cl(int k, int ch) const {
        return staged ? c[padi((base + k) * C + ch)] : __ldg(c + (size_t)k * C + ch);
    }
};

// The weights of one pixel (include/nr_b200.h): zref = min(zp_bg, min over valid zbuf), w_k into s_w[k kPix] (0 for an
// invalid slot), D_k into s_D when given; returns the validity mask, Z = w_b + w_0 + w_1 + ... (slot order), w_b and
// lam = sum softplus(x_k) (slot order).  Forward and backward call this one function, so the backward's Z is the
// forward's.
__device__ __forceinline__ unsigned blend_weights(const BlendParams& P, const Slots& s, float* s_w, float* s_D, float& Z,
                                                  float& wb, float& lam) {
    const int K = P.K, tid = threadIdx.x;
    unsigned mask = 0;
    float zref = P.zp_bg;
    for (int k = 0; k < K; k++)
        if (s.valid(k)) {
            mask |= 1u << k;
            zref = fminf(zref, s.zb(k));
        }
    wb = expf(__fmul_rn(__fsub_rn(zref, P.zp_bg), P.inv_fg));
    Z = wb;
    lam = 0.0f;
    for (int k = 0; k < K; k++) {
        float w = 0.0f, D = 0.0f;
        if ((mask >> k) & 1u) {
            const float x = __fmul_rn(s.ds(k), P.inv_sigma);
            D = blend_sigmoid(x);
            w = __fmul_rn(D, expf(__fmul_rn(__fsub_rn(zref, s.zb(k)), P.inv_fg)));
            Z = __fadd_rn(Z, w);
            lam = __fadd_rn(lam, fmaxf(x, 0.0f) + log1pf(expf(-fabsf(x))));
        }
        s_w[k * kPix + tid] = w;
        if (s_D) s_D[k * kPix + tid] = D;
    }
    return mask;
}

// ------------------------------------------------------------------------------------------------ staging
// n words of src into the padded tile dst, coalesced (16-byte loads when vec); streaming: every input is read once
__device__ __forceinline__ void stage_in(float* dst, const float* src, int n, bool vec) {
    int e0 = 0;
    if (vec) {
        const int n4 = n >> 2;
        const float4* s4 = (const float4*)src;
#pragma unroll 4
        for (int i = threadIdx.x; i < n4; i += kPix) {
            const float4 v = __ldcs(s4 + i);
            const int e = padi(4 * i);  // the four words share one row of 32
            dst[e] = v.x; dst[e + 1] = v.y; dst[e + 2] = v.z; dst[e + 3] = v.w;
        }
        e0 = 4 * n4;
    }
#pragma unroll 4
    for (int e = e0 + threadIdx.x; e < n; e += kPix) dst[padi(e)] = __ldcs(src + e);
}

// pix_to_face [n] as validity flags
__device__ __forceinline__ void stage_flags(int* dst, const long long* src, int n, bool vec) {
    int e0 = 0;
    if (vec) {
        const int n2 = n >> 1;
        const longlong2* s2 = (const longlong2*)src;
#pragma unroll 4
        for (int i = threadIdx.x; i < n2; i += kPix) {
            const longlong2 v = __ldcs(s2 + i);
            const int e = padi(2 * i);
            dst[e] = v.x >= 0; dst[e + 1] = v.y >= 0;
        }
        e0 = 2 * n2;
    }
#pragma unroll 4
    for (int e = e0 + threadIdx.x; e < n; e += kPix) dst[padi(e)] = __ldcs(src + e) >= 0;
}

// the padded tile src [n] out to dst, coalesced (16-byte stores when vec)
__device__ __forceinline__ void stage_out(float* dst, const float* src, int n, bool vec) {
    int e0 = 0;
    if (vec) {
        const int n4 = n >> 2;
        float4* d4 = (float4*)dst;
#pragma unroll 4
        for (int i = threadIdx.x; i < n4; i += kPix) {
            const int e = padi(4 * i);
            __stcs(d4 + i, make_float4(src[e], src[e + 1], src[e + 2], src[e + 3]));
        }
        e0 = 4 * n4;
    }
#pragma unroll 4
    for (int e = e0 + threadIdx.x; e < n; e += kPix) __stcs(dst + e, src[padi(e)]);
}

// the shared-memory layout of a CTA: [K][kPix] columns (nw of them), then the staged tile
struct Smem {
    float *w, *D, *h, *z, *d, *c;
    int* f;
};
__device__ __forceinline__ Smem smem_layout(float* sm, int K, int C, int ncols, bool staged) {
    Smem m;
    const int col = K * kPix, t = padn(kPix * K);
    m.w = sm;
    m.D = ncols > 1 ? sm + col : nullptr;
    m.h = ncols > 2 ? sm + 2 * col : nullptr;
    float* s = sm + ncols * col;
    m.f = staged ? (int*)s : nullptr;
    m.z = staged ? s + t : nullptr;
    m.d = staged ? s + 2 * t : nullptr;
    m.c = staged ? s + 3 * t : nullptr;
    return m;
}

size_t smem_bytes(int K, int C, int ncols, bool staged) {
    size_t words = (size_t)ncols * K * kPix;
    if (staged) words += 3 * (size_t)padn(kPix * K) + (size_t)padn(kPix * K * C);
    return words * sizeof(float);
}

__device__ __forceinline__ Slots slots_of(const BlendParams& P, const Smem& m, long long pix, bool staged) {
    Slots s;
    s.K = P.K; s.C = P.C; s.staged = staged;
    s.f = m.f;
    if (staged) {
        s.p2f = nullptr;
        s.z = m.z; s.d = m.d; s.c = m.c;
        s.base = threadIdx.x * P.K;
    } else {
        const size_t o = (size_t)pix * P.K;
        s.p2f = P.p2f + o;
        s.z = P.zbuf + o; s.d = P.dists + o; s.c = P.col + o * P.C;
        s.base = 0;
    }
    return s;
}

// the CTA's first pixel, its pixel count and the staging of its inputs
template <bool kStaged>
__device__ __forceinline__ int stage_inputs(const BlendParams& P, const Smem& m, long long p0) {
    const int np = (int)min((long long)kPix, P.npix - p0);
    if (kStaged) {
        const int K = P.K, C = P.C;
        const size_t o = (size_t)p0 * K;
        stage_flags(m.f, P.p2f + o, np * K, P.vec);
        stage_in(m.z, P.zbuf + o, np * K, P.vec);
        stage_in(m.d, P.dists + o, np * K, P.vec);
        stage_in(m.c, P.col + o * C, np * K * C, P.vec);
        __syncthreads();
    }
    return np;
}

// ------------------------------------------------------------------------------------------------ k_soft_blend_fwd
template <bool kStaged>
__global__ void __launch_bounds__(kPix) k_soft_blend_fwd(const __grid_constant__ BlendParams P) {
    extern __shared__ float sm[];
    const Smem m = smem_layout(sm, P.K, P.C, 1, kStaged);
    const long long p0 = (long long)blockIdx.x * kPix;
    const int np = stage_inputs<kStaged>(P, m, p0);
    if ((int)threadIdx.x >= np) return;
    const long long pix = p0 + threadIdx.x;
    const Slots s = slots_of(P, m, pix, kStaged);
    float Z, wb, lam;
    const unsigned mask = blend_weights(P, s, m.w, nullptr, Z, wb, lam);
    const long long b = pix / P.hw, o = pix - b * P.hw;
    __stcs(P.alpha + pix, -expm1f(-lam));
    const int K = P.K, C = P.C;
    float* out = P.out + (size_t)b * C * P.hw + o;
    for (int c0 = 0; c0 < C; c0 += kCB) {
        float N[kCB];
#pragma unroll
        for (int i = 0; i < kCB; i++) N[i] = (c0 + i < C && P.bg) ? __fmul_rn(wb, __ldg(P.bg + c0 + i)) : 0.0f;
        for (int k = 0; k < K; k++) {
            if (!((mask >> k) & 1u)) continue;
            const float w = m.w[k * kPix + threadIdx.x];
#pragma unroll
            for (int i = 0; i < kCB; i++)
                if (c0 + i < C) N[i] = __fmaf_rn(w, s.cl(k, c0 + i), N[i]);
        }
#pragma unroll
        for (int i = 0; i < kCB; i++)
            if (c0 + i < C) __stcs(out + (size_t)(c0 + i) * P.hw, __fdiv_rn(N[i], Z));
    }
}

// ------------------------------------------------------------------------------------------------ k_soft_blend_bwd
template <bool kStaged>
__global__ void __launch_bounds__(kPix) k_soft_blend_bwd(const __grid_constant__ BlendParams P) {
    extern __shared__ float sm[];
    const Smem m = smem_layout(sm, P.K, P.C, 3, kStaged);
    const long long p0 = (long long)blockIdx.x * kPix;
    const int np = stage_inputs<kStaged>(P, m, p0);
    const int K = P.K, C = P.C, tid = threadIdx.x;
    if (tid < np) {
        const long long pix = p0 + tid;
        const Slots s = slots_of(P, m, pix, kStaged);
        float Z, wb, lam;
        const unsigned mask = blend_weights(P, s, m.w, m.D, Z, wb, lam);
        const long long b = pix / P.hw, o = pix - b * P.hw;
        for (int k = 0; k < K; k++) m.h[k * kPix + tid] = 0.0f;
        // staged: the gradients replace the pixel's own words of the tile (each word is read before it is written)
        float* gcol = kStaged ? m.c : (P.g_col ? P.g_col + (size_t)pix * K * C : nullptr);
        const bool want_col = P.g_col != nullptr;
        const float* outp = P.out + (size_t)b * C * P.hw + o;
        const float* gop = P.g_out ? P.g_out + (size_t)b * C * P.hw + o : nullptr;
        for (int c0 = 0; c0 < C; c0 += kCB) {
            float g[kCB], ov[kCB];
#pragma unroll
            for (int i = 0; i < kCB; i++) {
                const bool in = c0 + i < C;
                g[i] = (in && gop) ? __ldcs(gop + (size_t)(c0 + i) * P.hw) : 0.0f;
                ov[i] = in ? __ldcs(outp + (size_t)(c0 + i) * P.hw) : 0.0f;
            }
            for (int k = 0; k < K; k++) {
                const bool v = (mask >> k) & 1u;
                const float w = m.w[k * kPix + tid];
                float hk = 0.0f;
#pragma unroll
                for (int i = 0; i < kCB; i++) {
                    const int ch = c0 + i;
                    if (ch >= C) continue;
                    if (v) hk = __fmaf_rn(g[i], __fsub_rn(s.cl(k, ch), ov[i]), hk);
                    if (want_col) {
                        const float gc = v ? __fdiv_rn(__fmul_rn(w, g[i]), Z) : 0.0f;
                        if (kStaged) gcol[padi((tid * K + k) * C + ch)] = gc;
                        else __stcs(gcol + (size_t)k * C + ch, gc);
                    }
                }
                if (v) m.h[k * kPix + tid] = __fadd_rn(m.h[k * kPix + tid], hk);
            }
        }
        // 1 - alpha = exp(-lam) from the recomputed sum: the saved alpha rounds to 1 long before exp(-lam) underflows
        const float ga = P.g_alpha ? __ldcs(P.g_alpha + pix) : 0.0f;
        const float ta = __fmul_rn(expf(-lam), ga);
        for (int k = 0; k < K; k++) {
            float gd = 0.0f, gz = 0.0f;
            if ((mask >> k) & 1u) {
                const float w = m.w[k * kPix + tid], D = m.D[k * kPix + tid];
                const float H = __fdiv_rn(m.h[k * kPix + tid], Z);
                const float wH = __fmul_rn(w, H);
                gd = __fmul_rn(__fmaf_rn(ta, D, __fmul_rn(wH, 1.0f - D)), P.inv_sigma);
                gz = -__fmul_rn(wH, P.inv_fg);
            }
            if (kStaged) {
                m.z[padi(tid * K + k)] = gz;
                m.d[padi(tid * K + k)] = gd;
            } else {
                const size_t q = (size_t)pix * K + k;
                if (P.g_zbuf) __stcs(P.g_zbuf + q, gz);
                if (P.g_dists) __stcs(P.g_dists + q, gd);
            }
        }
    }
    if (kStaged) {
        __syncthreads();
        const size_t q = (size_t)p0 * K;
        if (P.g_zbuf) stage_out(P.g_zbuf + q, m.z, np * K, P.vec);
        if (P.g_dists) stage_out(P.g_dists + q, m.d, np * K, P.vec);
        if (P.g_col) stage_out(P.g_col + q * C, m.c, np * K * C, P.vec);
    }
}

// ------------------------------------------------------------------------------------------------ host
bool aligned(const void* p, uintptr_t a) { return ((uintptr_t)p & (a - 1)) == 0; }

// the host checks of both entry points; fills `p`
int blend_setup(const nr_b200_blend_args* a, bool backward, BlendParams* p) {
    nr_internal::launch_count() = 0;
    if (!a || a->struct_size != sizeof(nr_b200_blend_args)) return NR_ERR_INVALID_ARG;
    const long long B = a->batch_size, H = a->height, W = a->width, K = a->faces_per_pixel, C = a->channels;
    if (B < 1 || H < 1 || W < 1 || K < 1 || K > kMaxK || C < 1) return NR_ERR_INVALID_ARG;
    // every index is 64-bit; the grid has one CTA per kPix pixels
    const double n = (double)B * (double)H * (double)W;
    if (n * (double)K * (double)C > 4.0e18 || n / kPix > 2147483647.0) return NR_ERR_INVALID_ARG;
    const float sigma = a->sigma, gamma = a->gamma;
    if (!(isfinite(sigma) && sigma > 0.0f) || !(isfinite(gamma) && gamma > 0.0f)) return NR_ERR_INVALID_ARG;
    if (!isfinite(a->near_) || !isfinite(a->far_) || !(a->near_ < a->far_) || !isfinite(a->far_ - a->near_))
        return NR_ERR_INVALID_ARG;
    const double fn = (double)a->far_ - (double)a->near_;
    const double inv_sigma = 1.0 / (double)sigma, inv_fg = 1.0 / (fn * (double)gamma);
    if (!(inv_sigma < 3.0e38) || !(inv_fg < 3.0e38)) return NR_ERR_INVALID_ARG;  // finite in fp32
    if (!a->pix_to_face || !a->zbuf || !a->dists || !a->colors || !a->out || (!backward && !a->alpha))
        return NR_ERR_INVALID_ARG;
    if (backward && !a->grad_colors && !a->grad_zbuf && !a->grad_dists) return NR_ERR_INVALID_ARG;
    const void* f32[] = {a->zbuf, a->dists, a->colors, a->background, a->out, a->alpha, a->grad_out, a->grad_alpha,
                         a->grad_colors, a->grad_zbuf, a->grad_dists};
    if (!aligned(a->pix_to_face, 8)) return NR_ERR_INVALID_ARG;
    for (const void* q : f32)
        if (!aligned(q, 4)) return NR_ERR_INVALID_ARG;
    memset(p, 0, sizeof(*p));
    p->p2f = (const long long*)a->pix_to_face;
    p->zbuf = a->zbuf; p->dists = a->dists; p->col = a->colors; p->bg = a->background;
    p->out = a->out; p->alpha = a->alpha;
    p->npix = B * H * W; p->hw = H * W;
    p->K = (int)K; p->C = (int)C;
    p->inv_sigma = (float)inv_sigma;
    p->inv_fg = (float)inv_fg;
    p->zp_bg = (float)((double)a->far_ - NR_SOFT_BG_DEPTH * fn);
    bool al = aligned(a->pix_to_face, 16) && aligned(a->zbuf, 16) && aligned(a->dists, 16) && aligned(a->colors, 16);
    if (backward) {
        p->g_out = a->grad_out; p->g_alpha = a->grad_alpha;
        p->g_col = a->grad_colors; p->g_zbuf = a->grad_zbuf; p->g_dists = a->grad_dists;
        al = al && aligned(a->grad_colors, 16) && aligned(a->grad_zbuf, 16) && aligned(a->grad_dists, 16);
    }
    p->vec = al;
    return NR_OK;
}

// staged when the tile fits (and not in the per-thread experiment build)
bool use_staging(const BlendParams& p, int ncols) {
#if defined(NR_B200_TUNING) && defined(NR_SOFT_BLEND_PER_THREAD)
    (void)p; (void)ncols;
    return false;
#else
    return smem_bytes(p.K, p.C, ncols, true) <= kStageBudget;
#endif
}

template <typename Kern>
cudaError_t launch(Kern kern, const BlendParams& p, size_t smem, cudaStream_t s) {
    if (smem > 48 * 1024) {
        const cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
    }
    const unsigned grid = (unsigned)((p.npix + kPix - 1) / kPix);
    kern<<<grid, kPix, smem, s>>>(p);
    return cudaGetLastError();
}

}  // namespace

extern "C" int nr_b200_blend_fragments(const nr_b200_blend_args* args, void* cuda_stream) {
    BlendParams p;
    const int rc = blend_setup(args, false, &p);
    if (rc != NR_OK) return rc;
    cudaStream_t s = (cudaStream_t)cuda_stream;
    const bool st = use_staging(p, 1);
    nr_internal::LaunchScope ls("k_soft_blend_fwd", s);
    const cudaError_t e = st ? launch(k_soft_blend_fwd<true>, p, smem_bytes(p.K, p.C, 1, true), s)
                             : launch(k_soft_blend_fwd<false>, p, smem_bytes(p.K, p.C, 1, false), s);
    return e == cudaSuccess ? NR_OK : NR_ERR_CUDA;
}

extern "C" int nr_b200_blend_fragments_backward(const nr_b200_blend_args* args, void* cuda_stream) {
    BlendParams p;
    const int rc = blend_setup(args, true, &p);
    if (rc != NR_OK) return rc;
    cudaStream_t s = (cudaStream_t)cuda_stream;
    const bool st = use_staging(p, 3);
    nr_internal::LaunchScope ls("k_soft_blend_bwd", s);
    const cudaError_t e = st ? launch(k_soft_blend_bwd<true>, p, smem_bytes(p.K, p.C, 3, true), s)
                             : launch(k_soft_blend_bwd<false>, p, smem_bytes(p.K, p.C, 3, false), s);
    return e == cudaSuccess ? NR_OK : NR_ERR_CUDA;
}
