// nr_soft.cu -- soft silhouettes (nr_b200_soft_silhouettes / nr_b200_soft_silhouettes_backward, include/nr_b200.h).
//
// Every face gives every pixel within reach a probability D = sigmoid(+-d^2 / sigma) of the pixel's squared distance d^2
// to the face (SoftRas), and alpha = 1 - prod_j (1 - D_j).  Both passes walk 16 x 16 pixel tiles:
//
//   k_soft_setup    one thread per face: the participation test (every vertex depth in [near, far]), the face record
//                   (three edges {a, b - a, 1 / |b - a|^2}, 64 bytes) and the face's tile box -- its pixel box grown by the
//                   cut-off reach plus one pixel -- and counts the face into each tile it overlaps (global atomics).
//                   Faces spanning more than kWideTiles tiles are counted once, into the item's wide slot.
//   k_strip_scan    the backward's segment scan (nr_backward.cu), one segment per item: tile counters -> list offsets.
//   k_soft_fill     one thread per face: appends the face to the list of each tile it counted into (atomic cursors).
//   k_soft_fwd      one CTA per (tile, item), one thread per pixel.  The tile's list, then the wide list with a box
//                   test, are staged into shared memory 256 records at a time; every thread adds softplus(x_j) of its
//                   pixel into a 64-bit fixed-point sum, so the list order the atomic fill left does not reach alpha: the
//                   forward is bit-for-bit deterministic.  alpha = -expm1(-Lambda), one streaming store per pixel.
//   k_soft_bwd      the same traversal with g (1 - alpha) per pixel: each face's 6 xy partials are reduced over the
//                   warp (shuffles, only when a lane of the warp is within reach), then over the CTA (shared-memory
//                   adds), and leave the CTA as one set of global atomics per face and tile through nr::FaceGrad.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <string.h>

#include "nr_b200.h"
#include "nr_internal.h"
#include "nr_soft.cuh"

namespace {

// Stages the next <= kThreads faces of the tile (its own list, then the wide list with a box test) into shared memory;
// returns how many were staged.  `next` is the position in the concatenated list, advanced by kThreads.
__device__ __forceinline__ int stage_faces(const SoftParams& p, int b, int tile, int tx, int ty, int n_tile, int n_all,
                                           int next, float4* s_rec, int* s_face, int* s_n) {
    const int tid = threadIdx.x;
    if (tid == 0) *s_n = 0;
    __syncthreads();
    const int i = next + tid;
    const size_t seg = (size_t)b * (p.ntiles + 1);
    int f = -1;
    if (i < n_tile) {
        f = p.list[p.off[seg + tile] + i];
    } else if (i < n_all) {
        f = p.list[p.off[seg + p.ntiles] + (i - n_tile)];
        const uint2 bb = __ldg(p.box + (size_t)b * p.F + f);
        if (tx < lo16(bb.x) || tx > hi16(bb.x) || ty < lo16(bb.y) || ty > hi16(bb.y)) f = -1;
    }
    const unsigned m = __ballot_sync(0xffffffffu, f >= 0);
    int base = 0;
    if ((tid & 31) == 0 && m) base = atomicAdd(s_n, __popc(m));
    base = __shfl_sync(0xffffffffu, base, 0);
    if (f >= 0) {
        const int slot = base + __popc(m & ((1u << (tid & 31)) - 1u));
        const float4* r = p.rec + ((size_t)b * p.F + f) * 4;
#pragma unroll
        for (int k = 0; k < 4; k++) s_rec[slot * 4 + k] = __ldg(r + k);
        s_face[slot] = f;
    }
    __syncthreads();
    return *s_n;
}

// ------------------------------------------------------------------------------------------------ k_soft_fwd
__global__ void __launch_bounds__(kThreads) k_soft_fwd(const __grid_constant__ SoftParams p) {
    __shared__ float4 s_rec[kThreads * 4];
    __shared__ int s_face[kThreads];
    __shared__ int s_n;
    const int tile = blockIdx.x, b = blockIdx.y;
    const int tx = tile % p.ntx, ty = tile / p.ntx;
    const int col = tx * kTile + (threadIdx.x % kTile), row = ty * kTile + (threadIdx.x / kTile);
    const int S = p.S;
    const float px = soft_centre(col, S), py = soft_centre(S - 1 - row, S);
    const size_t seg = (size_t)b * (p.ntiles + 1);
    const int n_tile = p.cnt[seg + tile], n_all = n_tile + p.cnt[seg + p.ntiles];
    const unsigned long long cap = (unsigned long long)(kTermCap * kFix);
    unsigned long long acc = 0;  // Lambda in units of 2^-40: integer adds, so the order of the faces does not matter
    for (int next = 0; next < n_all; next += kThreads) {
        const int n = stage_faces(p, b, tile, tx, ty, n_tile, n_all, next, s_rec, s_face, &s_n);
        for (int j = 0; j < n; j++) {
            float x, t, qx, qy;
            int k;
            if (!soft_term(s_rec + 4 * j, px, py, p.inv_sigma, p.cut, x, k, t, qx, qy)) continue;
            const float sp = fmaxf(x, 0.0f) + log1pf(expf(-fabsf(x)));  // softplus(x) >= 0
            acc += (unsigned long long)__float2ll_rn(fminf(sp, kTermCap) * kFix);
            acc = acc < cap ? acc : cap;
        }
        __syncthreads();
    }
    if (row < S && col < S) {
        const float lam = __ull2float_rn(acc) * (1.0f / kFix);
        __stcs(p.alpha + (size_t)b * S * S + (size_t)row * S + col, -expm1f(-lam));
    }
}

// ------------------------------------------------------------------------------------------------ k_soft_bwd
__global__ void __launch_bounds__(kThreads) k_soft_bwd(const __grid_constant__ SoftParams p) {
    __shared__ float4 s_rec[kThreads * 4];
    __shared__ int s_face[kThreads];
    __shared__ float s_acc[kThreads * 6];
    __shared__ int s_n;
    const int tile = blockIdx.x, b = blockIdx.y;
    const int tx = tile % p.ntx, ty = tile / p.ntx;
    const int col = tx * kTile + (threadIdx.x % kTile), row = ty * kTile + (threadIdx.x / kTile);
    const int S = p.S, lane = threadIdx.x & 31;
    const float px = soft_centre(col, S), py = soft_centre(S - 1 - row, S);
    const size_t seg = (size_t)b * (p.ntiles + 1);
    const int n_tile = p.cnt[seg + tile], n_all = n_tile + p.cnt[seg + p.ntiles];
    if (n_all == 0) return;  // CTA-uniform
    float gp = 0.0f;  // d loss / d x_j = gp D_j with gp = g (1 - alpha) (-2 sign / sigma folded in below)
    if (row < S && col < S) {
        const size_t o = (size_t)b * S * S + (size_t)row * S + col;
        gp = __ldg(p.g + o) * (1.0f - __ldg(p.alpha + o));
    }
    for (int i = threadIdx.x; i < kThreads * 6; i += kThreads) s_acc[i] = 0.0f;
    for (int next = 0; next < n_all; next += kThreads) {
        const int n = stage_faces(p, b, tile, tx, ty, n_tile, n_all, next, s_rec, s_face, &s_n);
        for (int j = 0; j < n; j++) {
            float x = 0.0f, t = 0.0f, qx = 0.0f, qy = 0.0f;
            int k = 0;
            const bool hit = gp != 0.0f && soft_term(s_rec + 4 * j, px, py, p.inv_sigma, p.cut, x, k, t, qx, qy);
            if (!__any_sync(0xffffffffu, hit)) continue;  // warp-uniform
            float v[6] = {0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f};
            if (hit) {
                const float e = expf(-fabsf(x));
                const float D = x >= 0.0f ? __frcp_rn(1.0f + e) : __fdiv_rn(e, 1.0f + e);
                // d x / d(d^2) = +-1/sigma; d(d^2)/da = -2 (1 - t)(p - q), d(d^2)/db = -2 t (p - q) for edge (a, b)
                const float s = gp * D * (x >= 0.0f ? -2.0f : 2.0f) * p.inv_sigma;
                const float wa = s * (1.0f - t), wb = s * t;
#pragma unroll
                for (int m = 0; m < 3; m++) {
                    const bool is_a = m == k, is_b = m == (k == 2 ? 0 : k + 1);
                    v[2 * m] = is_a ? wa * qx : (is_b ? wb * qx : 0.0f);
                    v[2 * m + 1] = is_a ? wa * qy : (is_b ? wb * qy : 0.0f);
                }
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1)
#pragma unroll
                for (int m = 0; m < 6; m++) v[m] += __shfl_xor_sync(0xffffffffu, v[m], o);
            if (lane < 6) {
                float mine = v[0];
#pragma unroll
                for (int m = 1; m < 6; m++) if (lane == m) mine = v[m];
                atomicAdd(&s_acc[j * 6 + lane], mine);
            }
        }
        __syncthreads();
        // one set of global atomics per face of the round: thread (face slot, vertex)
        for (int i = threadIdx.x; i < n * 3; i += kThreads) {
            const int j = i / 3, m = i % 3;
            const float gx = s_acc[j * 6 + 2 * m], gy = s_acc[j * 6 + 2 * m + 1];
            s_acc[j * 6 + 2 * m] = 0.0f; s_acc[j * 6 + 2 * m + 1] = 0.0f;
            if (gx == 0.0f && gy == 0.0f) continue;
            float* gv = nr::face_grad_vertex(p.dst, b, s_face[j], m);
            if (gv) { atomicAdd(gv, gx); atomicAdd(gv + 1, gy); }
        }
        __syncthreads();
    }
}

// the host checks of both entry points; fills `p` on success (NR_ERR_WORKSPACE after every NR_ERR_INVALID_ARG rule)
int soft_setup(const nr_b200_soft_args* a, bool backward, SoftParams* p) {
    nr_internal::launch_count() = 0;
    if (!a || a->struct_size != sizeof(nr_b200_soft_args)) return NR_ERR_INVALID_ARG;
    if (!(a->near_ <= a->far_) || !a->alpha) return NR_ERR_INVALID_ARG;
    memset(p, 0, sizeof(*p));
    if (!fill_soft_params(a, backward, p)) return NR_ERR_INVALID_ARG;
    const SoftLayout L = soft_layout(p->B, p->F, p->S);
    if (!a->workspace || a->workspace_bytes < L.total || ((uintptr_t)a->workspace & 15)) return NR_ERR_WORKSPACE;
    char* ws = (char*)a->workspace;
    p->rec = (float4*)(ws + L.rec); p->box = (uint2*)(ws + L.box);
    p->cnt = (int*)(ws + L.cnt); p->cursor = (int*)(ws + L.cursor); p->off = (int*)(ws + L.off); p->list = (int*)(ws + L.list);
    return NR_OK;
}

// A template, as bin_prefix is: k_soft_setup<true> is then instantiated after k_soft_setup<false>, so the object lists
// its kernels in the order of earlier builds and its SASS compares with theirs line for line
template <typename = void>
void fill_lists(const SoftParams& p, cudaStream_t s) {
    nr_internal::LaunchScope ls("k_soft_fill", s);
    k_soft_setup<true><<<dim3((unsigned)((p.F + 255) / 256), (unsigned)p.B), 256, 0, s>>>(p);
}

// setup -> scan -> fill: the tile lists of every item
int bin_faces(const SoftParams& p, cudaStream_t s) {
    if (bin_prefix(p, s) != NR_OK) return NR_ERR_CUDA;
    fill_lists(p, s);
    return NR_OK;
}

}  // namespace

extern "C" size_t nr_b200_soft_workspace_bytes(int32_t B, int32_t F, int32_t S, float sigma, uint32_t flags) {
    (void)flags;
    if (!soft_sizes_ok(B, F, S) || !isfinite(sigma) || !(sigma > 0.0f)) return 0;
    return soft_layout(B, F, S).total;
}

extern "C" int nr_b200_soft_silhouettes(const nr_b200_soft_args* args, void* cuda_stream) {
    SoftParams p;
    const int rc = soft_setup(args, false, &p);
    if (rc != NR_OK) return rc;
    cudaStream_t s = (cudaStream_t)cuda_stream;
    if (bin_faces(p, s) != NR_OK) return NR_ERR_CUDA;
    {
        nr_internal::LaunchScope ls("k_soft_fwd", s);
        k_soft_fwd<<<dim3((unsigned)p.ntiles, (unsigned)p.B), kThreads, 0, s>>>(p);
    }
    return cudaGetLastError() == cudaSuccess ? NR_OK : NR_ERR_CUDA;
}

extern "C" int nr_b200_soft_silhouettes_backward(const nr_b200_soft_args* args, void* cuda_stream) {
    SoftParams p;
    const int rc = soft_setup(args, true, &p);
    if (rc != NR_OK) return rc;
    const nr_b200_soft_args* a = args;
    cudaStream_t s = (cudaStream_t)cuda_stream;
    if (!(a->flags & NR_GRAD_ACCUMULATE) && nr_internal::zero_grads({nr_internal::geometry_grad(a)}, s) != cudaSuccess)
        return NR_ERR_CUDA;
    if (!a->grad_alpha) return cudaGetLastError() == cudaSuccess ? NR_OK : NR_ERR_CUDA;
    if (bin_faces(p, s) != NR_OK) return NR_ERR_CUDA;
    {
        nr_internal::LaunchScope ls("k_soft_bwd", s);
        k_soft_bwd<<<dim3((unsigned)p.ntiles, (unsigned)p.B), kThreads, 0, s>>>(p);
    }
    return cudaGetLastError() == cudaSuccess ? NR_OK : NR_ERR_CUDA;
}
