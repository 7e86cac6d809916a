// nr_soft_interp.cu -- the soft interpolation of fragments (nr_b200_interpolate_fragments /
// nr_b200_interpolate_fragments_backward, include/nr_b200.h): per-corner or per-vertex attributes interpolated at the K
// slots of every pixel, with gradients into the attributes and the barycentrics.  No workspace.
//
//   k_soft_interp_fwd<kPV, kV>  a streaming gather, kSlots consecutive slots per CTA.  The CTA first copies its slots'
//                               barycentrics (coalesced) and resolves every slot's three attribute rows (per corner, or
//                               through face_indices) into shared memory; then thread e of the CTA's ns C / kV outputs
//                               computes kV consecutive channels of one slot, so every store is coalesced (16-byte vectors
//                               when C % 4 == 0 and the addresses allow: kV = 4).  The attribute rows are gathered through
//                               L1 / L2 (neighbouring slots mostly show the same faces).
//   k_soft_interp_bwd<kPV>      one CTA per G groups of 32 consecutive pixels (G = ceil(kWarpsB / K), so that every warp
//                               has work at small K), one lane per pixel; warp w takes the tasks (group, slot k) = w,
//                               w + kWarpsB, ...  pix_to_face and bary are staged in shared memory with coalesced loads;
//                               grad_bary is summed per lane over the channels and written back from the tile coalesced.
//                               The attribute gradient is merged before it reaches L2 as k_interp_grad (nr_attr.cu) merges
//                               it: the warp walks its runs of neighbouring pixels whose slot k shows the same face, lane c
//                               sums l_m(p) g_c(p) over the run (the weights arrive by 3 shuffles per pixel and 32
//                               channels) and issues one atomic per corner and channel.  The experiment build
//                               NR_B200_TUNING + NR_SOFT_INTERP_GLOBAL_ATOMICS sends every slot's l_m g_c straight to
//                               global atomics instead (DESIGN.md 4u has the measured comparison).
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <string.h>

#include "nr_b200.h"
#include "nr_internal.h"

namespace {

constexpr int kMaxK = 32;               // the fragments' own cap
constexpr int kSlots = 256;             // forward: slots (and threads) per CTA
constexpr int kPixB = 32;               // backward: pixels per group, one per lane
constexpr int kWarpsB = 8;              // backward: warps per CTA
constexpr long long kMaxC = 1ll << 20;  // the forward's 32-bit output index within a CTA: kSlots C < 2^31

struct InterpParams {
    const long long* p2f;    // [N,K]  (N = B H W pixels)
    const float* bary;       // [N,K,3]
    const int32_t* idx;      // [.,F,3] (per vertex)
    const float* attr;       // [.,F,3,C] / [.,Nv,C]
    float* out;              // forward: [N,K,C]
    const float* g;          // backward: [N,K,C] or nullptr (zeros)
    float* gattr;            // backward: layout of attr, or nullptr
    float* gbary;            // backward: [N,K,3], or nullptr
    long long nslot, npix;   // N K, N
    long long hwk;           // slots per item (H W K)
    double inv_hwk;          // 1 / hwk
    size_t attr_bstride;     // floats per item in attr / gattr (0 = shared)
    size_t idx_bstride;      // ints per item in idx (0 = shared)
    int K, C, F, Nv;
    int G;                   // backward: pixel groups per CTA
    bool accumulate;         // NR_GRAD_ACCUMULATE: grad_bary += the sum
};

// first float of corner m's attribute row for face f of item b: the corner slot, or the vertex slot face_indices[f,m];
// -1 for an index outside [0, Nv)
template <bool kPV>
__device__ __forceinline__ long long attr_row(const InterpParams& P, long long b, long long f, int m) {
    const size_t base = (size_t)b * P.attr_bstride;
    if (!kPV) return (long long)(base + ((size_t)f * 3 + m) * (size_t)P.C);
    const int i = __ldg(P.idx + (size_t)b * P.idx_bstride + (size_t)f * 3 + m);
    return (unsigned)i < (unsigned)P.Nv ? (long long)(base + (size_t)i * (size_t)P.C) : -1;
}

__device__ __forceinline__ bool slot_valid(const InterpParams& P, long long f) {
    return (unsigned long long)f < (unsigned long long)P.F;
}

// x / n for 0 <= x < 2^50 and n >= 1, from the host's inv = 1 / n in double and one correction step (a 64-bit integer
// or a double division would be a called subroutine, with a stack frame)
__device__ __forceinline__ long long div_index(long long x, long long n, double inv) {
    long long q = (long long)__dmul_rz((double)x, inv);
    if (q * n > x) q--;
    else if ((q + 1) * n <= x) q++;
    return q;
}

__device__ __forceinline__ float ld_or0(const float* a, long long row, int c) { return row >= 0 ? __ldg(a + row + c) : 0.0f; }

// out_c = fma(l2, a_2c, fma(l1, a_1c, l0 a_0c)): the chain of nr_attr.cu's interp and nr_soft_attr.cu's attr_blend
__device__ __forceinline__ float interp(float l0, float l1, float l2, float a0, float a1, float a2) {
    return __fmaf_rn(l2, a2, __fmaf_rn(l1, a1, __fmul_rn(l0, a0)));
}

// ------------------------------------------------------------------------------------------------ k_soft_interp_fwd
template <bool kPV, int kV>
__global__ void __launch_bounds__(kSlots) k_soft_interp_fwd(const __grid_constant__ InterpParams P) {
    __shared__ long long s_row[3][kSlots];
    __shared__ float s_l[3 * kSlots];
    const long long s0 = (long long)blockIdx.x * kSlots;
    const int ns = (int)min((long long)kSlots, P.nslot - s0);
    const int t = threadIdx.x;
    for (int e = t; e < 3 * ns; e += kSlots) s_l[e] = __ldcs(P.bary + 3 * s0 + e);
    __syncthreads();
    if (t < ns) {
        const long long slot = s0 + t;
        const long long f = __ldcs(P.p2f + slot);
        if (slot_valid(P, f)) {
            const long long b = div_index(slot, P.hwk, P.inv_hwk);
#pragma unroll
            for (int m = 0; m < 3; m++) s_row[m][t] = attr_row<kPV>(P, b, f, m);
        } else {
            // an empty slot: no rows and zero weights (whatever bary holds there), so its output is exactly +0
#pragma unroll
            for (int m = 0; m < 3; m++) { s_row[m][t] = -1; s_l[3 * t + m] = 0.0f; }
        }
    }
    __syncthreads();
    const int CG = P.C / kV;
    float* out = P.out + (size_t)s0 * P.C;
    for (int e = t; e < ns * CG; e += kSlots) {
        const int s = e / CG, c = (e - s * CG) * kV;
        const long long r0 = s_row[0][s], r1 = s_row[1][s], r2 = s_row[2][s];
        const float l0 = s_l[3 * s], l1 = s_l[3 * s + 1], l2 = s_l[3 * s + 2];
        if constexpr (kV == 4) {
            const float4 z = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
            const float4 a0 = r0 >= 0 ? __ldg((const float4*)(P.attr + r0 + c)) : z;
            const float4 a1 = r1 >= 0 ? __ldg((const float4*)(P.attr + r1 + c)) : z;
            const float4 a2 = r2 >= 0 ? __ldg((const float4*)(P.attr + r2 + c)) : z;
            const float4 v = make_float4(interp(l0, l1, l2, a0.x, a1.x, a2.x), interp(l0, l1, l2, a0.y, a1.y, a2.y),
                                         interp(l0, l1, l2, a0.z, a1.z, a2.z), interp(l0, l1, l2, a0.w, a1.w, a2.w));
            *(float4*)(out + (size_t)e * 4) = v;
        } else {
            out[e] = interp(l0, l1, l2, ld_or0(P.attr, r0, c), ld_or0(P.attr, r1, c), ld_or0(P.attr, r2, c));
        }
    }
}

// ------------------------------------------------------------------------------------------------ k_soft_interp_bwd
// dynamic shared memory: pix_to_face [G kPixB K] (long long), then bary and grad_bary [G kPixB K 3] each
size_t bwd_smem_bytes(int K, int G) { return (size_t)G * kPixB * K * (sizeof(long long) + 6 * sizeof(float)); }

template <bool kPV>
__global__ void __launch_bounds__(kPixB * kWarpsB, 1) k_soft_interp_bwd(const __grid_constant__ InterpParams P) {
    extern __shared__ long long smb[];
    const int K = P.K, C = P.C;
    long long* s_f = smb;
    const int G = P.G;
    float* s_l = (float*)(smb + G * kPixB * K);
    float* s_gb = s_l + 3 * G * kPixB * K;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const long long p0 = (long long)blockIdx.x * (G * kPixB);
    const int np = (int)min((long long)(G * kPixB), P.npix - p0);
    const long long q0 = p0 * K;  // the CTA's first slot
    const int nq = np * K;
    for (int e = threadIdx.x; e < nq; e += kPixB * kWarpsB) s_f[e] = __ldcs(P.p2f + q0 + e);
    for (int e = threadIdx.x; e < 3 * nq; e += kPixB * kWarpsB) s_l[e] = __ldcs(P.bary + 3 * q0 + e);
    __syncthreads();
    for (int task = warp; task < G * K; task += kWarpsB) {  // warp-uniform
        const int grp = task / K, k = task - grp * K;
        const int pl = grp * kPixB + lane;                 // the lane's pixel within the tile
        const bool in = pl < np;
        const long long b = in ? div_index((p0 + pl) * K, P.hwk, P.inv_hwk) : 0;
        const int j = pl * K + k;                          // the lane's slot within the tile
        const long long f = in ? s_f[j] : -1;
        const bool valid = in && slot_valid(P, f);
        float l[3] = {0.0f, 0.0f, 0.0f};
        long long r[3] = {-1, -1, -1};
        if (valid) {
#pragma unroll
            for (int m = 0; m < 3; m++) { l[m] = s_l[3 * j + m]; r[m] = attr_row<kPV>(P, b, f, m); }
        }
        const float* g = (valid && P.g) ? P.g + (size_t)(q0 + j) * C : nullptr;
        if (P.gbary && in) {
            float s[3] = {0.0f, 0.0f, 0.0f};
            if (g) {
                const float g0 = __ldg(g);
#pragma unroll
                for (int m = 0; m < 3; m++) s[m] = __fmul_rn(g0, ld_or0(P.attr, r[m], 0));
                for (int c = 1; c < C; c++) {
                    const float gc = __ldg(g + c);
#pragma unroll
                    for (int m = 0; m < 3; m++) s[m] = __fmaf_rn(gc, ld_or0(P.attr, r[m], c), s[m]);
                }
            }
#pragma unroll
            for (int m = 0; m < 3; m++) s_gb[3 * j + m] = s[m];
        }
        if (P.gattr && P.g) {
#if defined(NR_B200_TUNING) && defined(NR_SOFT_INTERP_GLOBAL_ATOMICS)
            // the measured alternative (DESIGN.md 4u): every slot's l_m g_c straight to global atomics
            if (valid)
                for (int c = 0; c < C; c++) {
                    const float gc = __ldg(g + c);
#pragma unroll
                    for (int m = 0; m < 3; m++)
                        if (r[m] >= 0) atomicAdd(P.gattr + r[m] + c, __fmul_rn(l[m], gc));
                }
#else
            // runs of neighbouring lanes whose slot k shows the same face of the same item
            const long long key = valid ? b * P.F + f : -1;
            const long long kprev = __shfl_up_sync(0xffffffffu, key, 1);
            const uint32_t heads = __ballot_sync(0xffffffffu, lane == 0 || key != kprev);
            uint32_t todo = heads & __ballot_sync(0xffffffffu, valid);
            while (todo) {  // warp-uniform
                const int h = __ffs(todo) - 1;
                todo &= todo - 1u;
                const uint32_t later = heads & ~((2u << h) - 1u);
                const int e = later ? __ffs(later) - 2 : 31;
                const long long r0 = __shfl_sync(0xffffffffu, r[0], h), r1 = __shfl_sync(0xffffffffu, r[1], h),
                                r2 = __shfl_sync(0xffffffffu, r[2], h);
                for (int c0 = 0; c0 < C; c0 += 32) {
                    const int ch = c0 + lane;
                    float acc0 = 0.0f, acc1 = 0.0f, acc2 = 0.0f;
                    for (int q = h; q <= e; q++) {
                        const float l0 = __shfl_sync(0xffffffffu, l[0], q), l1 = __shfl_sync(0xffffffffu, l[1], q),
                                    l2 = __shfl_sync(0xffffffffu, l[2], q);
                        if (ch < C) {
                            const float gq = __ldg(P.g + (size_t)(q0 + (grp * kPixB + q) * K + k) * C + ch);
                            acc0 = __fmaf_rn(l0, gq, acc0);
                            acc1 = __fmaf_rn(l1, gq, acc1);
                            acc2 = __fmaf_rn(l2, gq, acc2);
                        }
                    }
                    if (ch < C) {
                        if (r0 >= 0) atomicAdd(P.gattr + r0 + ch, acc0);
                        if (r1 >= 0) atomicAdd(P.gattr + r1 + ch, acc1);
                        if (r2 >= 0) atomicAdd(P.gattr + r2 + ch, acc2);
                    }
                }
            }
#endif
        }
    }
    if (P.gbary) {
        __syncthreads();
        float* gb = P.gbary + 3 * q0;
        for (int e = threadIdx.x; e < 3 * nq; e += kPixB * kWarpsB)
            gb[e] = P.accumulate ? __fadd_rn(gb[e], s_gb[e]) : s_gb[e];
    }
}

// ------------------------------------------------------------------------------------------------ host
bool aligned(const void* p, uintptr_t a) { return ((uintptr_t)p & (a - 1)) == 0; }

constexpr uint32_t kFwdFlags = NR_ATTR_PER_VERTEX | NR_ATTR_SHARED | NR_INDICES_SHARED;

// the host checks of both entry points; fills `p` and the attribute set's float count `attr_floats`
int interp_setup(const nr_b200_frag_interp_args* a, bool backward, InterpParams* p, size_t* attr_floats) {
    nr_internal::launch_count() = 0;
    if (!a || a->struct_size != sizeof(nr_b200_frag_interp_args)) return NR_ERR_INVALID_ARG;
    const uint32_t flags = a->flags;
    if (flags & ~(kFwdFlags | (backward ? NR_GRAD_ACCUMULATE : 0u))) return NR_ERR_INVALID_ARG;
    const long long B = a->batch_size, H = a->height, W = a->width, K = a->faces_per_pixel, C = a->channels;
    const long long F = a->num_faces, Nv = a->num_vertices;
    const bool pv = (flags & NR_ATTR_PER_VERTEX) != 0, shared = (flags & NR_ATTR_SHARED) != 0;
    if (B < 1 || H < 1 || W < 1 || K < 1 || K > kMaxK || C < 1 || F < 1 || (pv && Nv < 1)) return NR_ERR_INVALID_ARG;
    if (pv && !a->face_indices) return NR_ERR_INVALID_ARG;
    if (!a->pix_to_face || !a->bary || !a->attributes || (!backward && !a->out)) return NR_ERR_INVALID_ARG;
    if (backward && !a->grad_attributes && !a->grad_bary) return NR_ERR_INVALID_ARG;
    if (!aligned(a->pix_to_face, 8)) return NR_ERR_INVALID_ARG;
    const void* f32[] = {a->bary, a->face_indices, a->attributes, a->out, a->grad_out, a->grad_attributes, a->grad_bary};
    for (const void* q : f32)
        if (!aligned(q, 4)) return NR_ERR_INVALID_ARG;
    // index width: 64-bit element offsets, one forward CTA per kSlots slots, one backward CTA per kPixB pixels
    const double npix = (double)B * (double)H * (double)W;
    const double rows = pv ? (double)Nv : 3.0 * (double)F;
    if (C > kMaxC || npix * (double)K * (double)C > 4.0e18 || (shared ? 1.0 : (double)B) * rows * (double)C > 4.0e18)
        return NR_ERR_INVALID_ARG;
    if (npix * (double)K / kSlots > 2147483647.0 || npix / kPixB > 2147483647.0) return NR_ERR_INVALID_ARG;
    memset(p, 0, sizeof(*p));
    p->p2f = (const long long*)a->pix_to_face;
    p->bary = a->bary;
    p->idx = pv ? a->face_indices : nullptr;
    p->attr = a->attributes;
    p->npix = B * H * W;
    p->nslot = p->npix * K;
    p->hwk = H * W * K;
    p->inv_hwk = 1.0 / (double)p->hwk;
    const size_t row_floats = (size_t)(pv ? Nv : 3 * F) * (size_t)C;
    p->attr_bstride = shared ? 0 : row_floats;
    p->idx_bstride = (flags & NR_INDICES_SHARED) ? 0 : (size_t)F * 3;
    p->K = (int)K; p->C = (int)C; p->F = (int)F; p->Nv = pv ? (int)Nv : 0;
    *attr_floats = (shared ? 1 : (size_t)B) * row_floats;
    if (backward) {
        p->g = a->grad_out; p->gattr = a->grad_attributes; p->gbary = a->grad_bary;
        p->accumulate = (flags & NR_GRAD_ACCUMULATE) != 0;
    } else {
        p->out = a->out;
    }
    return NR_OK;
}

}  // namespace

extern "C" int nr_b200_interpolate_fragments(const nr_b200_frag_interp_args* args, void* cuda_stream) {
    InterpParams p;
    size_t nattr = 0;
    const int rc = interp_setup(args, false, &p, &nattr);
    if (rc != NR_OK) return rc;
    cudaStream_t s = (cudaStream_t)cuda_stream;
    const bool pv = p.idx != nullptr;
    const bool vec = p.C % 4 == 0 && aligned(p.attr, 16) && aligned(p.out, 16);
    const unsigned grid = (unsigned)((p.nslot + kSlots - 1) / kSlots);
    {
        nr_internal::LaunchScope ls("k_soft_interp_fwd", s);
        if (pv) {
            if (vec) k_soft_interp_fwd<true, 4><<<grid, kSlots, 0, s>>>(p);
            else k_soft_interp_fwd<true, 1><<<grid, kSlots, 0, s>>>(p);
        } else {
            if (vec) k_soft_interp_fwd<false, 4><<<grid, kSlots, 0, s>>>(p);
            else k_soft_interp_fwd<false, 1><<<grid, kSlots, 0, s>>>(p);
        }
    }
    return cudaGetLastError() == cudaSuccess ? NR_OK : NR_ERR_CUDA;
}

extern "C" int nr_b200_interpolate_fragments_backward(const nr_b200_frag_interp_args* args, void* cuda_stream) {
    InterpParams p;
    size_t nattr = 0;
    const int rc = interp_setup(args, true, &p, &nattr);
    if (rc != NR_OK) return rc;
    cudaStream_t s = (cudaStream_t)cuda_stream;
    if (p.gattr && !p.accumulate && nr_internal::zero_grads({{p.gattr, nattr * sizeof(float)}}, s) != cudaSuccess)
        return NR_ERR_CUDA;
    // without an upstream gradient the attribute gradient stays as it is; grad_bary still gets its zeros
    if (!p.gbary && !p.g) return cudaGetLastError() == cudaSuccess ? NR_OK : NR_ERR_CUDA;
    p.G = p.K >= kWarpsB ? 1 : (kWarpsB + p.K - 1) / p.K;
    const unsigned grid = (unsigned)((p.npix + p.G * kPixB - 1) / (p.G * kPixB));
    const size_t smem = bwd_smem_bytes(p.K, p.G);
    {
        nr_internal::LaunchScope ls("k_soft_interp_bwd", s);
        if (p.idx) k_soft_interp_bwd<true><<<grid, kPixB * kWarpsB, smem, s>>>(p);
        else k_soft_interp_bwd<false><<<grid, kPixB * kWarpsB, smem, s>>>(p);
    }
    return cudaGetLastError() == cudaSuccess ? NR_OK : NR_ERR_CUDA;
}
