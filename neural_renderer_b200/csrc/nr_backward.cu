// nr_backward.cu -- backward pass for sm_90a (H100).
//
// Replaces Rasterize.backward_gpu (reference neural_renderer/rasterize.py:849-889):
//
//   k_strip_bin       pre-pass of K5, two launches (count, fill): every front face is appended to the list of each W-line
//                     strip (per axis) that its pixel box overlaps.  The counting pass computes the boxes and counts per
//                     CTA in shared memory first; every CTA of the fill pass scans its item's counters itself.  Faces
//                     spanning more than kWideStrips strips go to one "wide" list per item / axis.  (Rasters with more
//                     than 2048 strips per axis use k_face_bbox + k_strip_bin_global + k_strip_scan instead.)
//   k_edge_scan       K5, the approximate-gradient image scan (rasterize.py:528-748).  The reference runs one thread
//                     per face that walks image columns / rows straight out of global memory.  Here a CTA owns a strip
//                     of W image lines (columns for axis 0, rows for axis 1) of one batch item and stages it once in
//                     shared memory as pixel PAIRS {A, g0 | g1, g2} with A = sum_c I_c * g_c (every scan walks
//                     contiguous shared memory; diff_grad = A - sum_c ref_c * g_c).  The strip's face list is expanded
//                     into (face, edge, line) tasks, counting-sorted by scan length and pulled by warps in batches of
//                     32: every lane sets up its own task and runs the short in-scan; the long out-scans are swept by
//                     4 lanes per task, two pixels per lane and step (fp32 pairs: two independent FMA chains).  Each task
//                     reproduces the reference's discrete decisions exactly (crossing pixel floor/ceil, the
//                     `face_index_map == fn` gates, the in-scan limit) and accumulates the same
//                     -relu(dI . dL/dI) / dist terms; only the summation order differs (fp32 atomics into grad_faces).
//                     Its CTAs also zero-fill grad_textures on the side when one call runs both halves of the pass.
//   k_texture_grad    K6 (rasterize.py:760-792): the 8 trilinear weights/indices are recomputed from the saved
//                     weight/depth maps with the forward expression tree instead of being stored (64 B/pixel in the
//                     reference) and scattered with vector float reductions (red.global.add.v2/v4.f32); applies the
//                     per-face light factor / fill_back cube sharing of the forward sampler and reduces d loss /
//                     d face_light per run of lanes; neighbouring lanes that blend the same eight texels merge their
//                     contributions with shuffles before the reductions.
//   k_image_grad      K6 for a texture image sampled through per-corner UVs (NR_TEX_UV): four bilinear taps per pixel,
//                     two 6-float horizontal pairs scattered the same way.  k_image_grad_mip: the trilinear variant
//                     (NR_TEX_MIPMAP), up to four pairs on two levels of the packed pyramid.
//   The texture-gradient kernels are instantiated per light mode (nr_shading.cuh) except kLightFace, which their
//   kLightNone variant serves with a run-time face_light pointer.
//   k_depth_grad      K7 (rasterize.py:805-847): analytic d zp / d(x, y, z) of the winning face, summed per run of
//                     neighbouring lanes that show the same face before the atomics.
//
// Upstream gradients arrive in API layout (planar, image orientation, pooled by 2x2 when anti-aliasing): the
// backward of rasterize_rgbad's transpose / flip / average pooling (rasterize.py:953-969) is folded into the loads.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include <type_traits>

#include "nr_b200.h"
#include "nr_bbox.cuh"
#include "nr_interior.h"
#include "nr_internal.h"
#include "nr_math.cuh"
#include "nr_phong.h"

#ifndef NR_ES_CTAS_PER_1024
#define NR_ES_CTAS_PER_1024 6   // k_edge_scan CTAs per SM at 128 threads (6 = 80 registers; 8 = 64 spills on sm_90 and was
                                // measured slower on H100 at raster 512: 2.93 vs 2.86 ms RGB, 3.44 vs 3.26 ms RGB + alpha)
#endif
#ifndef NR_ES_UNROLL
#define NR_ES_UNROLL 2          // steady-state out-scan steps per pointer bump
#endif
#ifndef NR_FILL_AT_END
#define NR_FILL_AT_END 0        // where an edge-scan CTA does its share of the grad_textures zero-fill: 0 = first, 1 = last
#endif
#ifndef NR_FILL_STREAMING
#define NR_FILL_STREAMING 1
#endif
#if NR_FILL_STREAMING
#define NR_FILL_STORE(ptr, v) __stcs(ptr, v)
#else
#define NR_FILL_STORE(ptr, v) (*(ptr) = (v))
#endif
#ifndef NR_TG_COMBINE
#define NR_TG_COMBINE 2         // shuffle steps that merge neighbouring lanes' contributions to the same texels (0: off)
#endif
#ifndef NR_TG_MIN_CTAS
#define NR_TG_MIN_CTAS 6
#endif
#ifndef NR_TGC_MIN_CTAS
#define NR_TGC_MIN_CTAS 3       // k_texture_grad with corner_light: spills at 4 CTAs (64 registers)
#endif
#ifndef NR_IG_MIN_CTAS
#define NR_IG_MIN_CTAS 4        // k_image_grad CTAs of 256 threads per SM (64 registers; see DESIGN.md section 4)
#endif
#ifndef NR_IGM_MIN_CTAS
#define NR_IGM_MIN_CTAS 3       // k_image_grad_mip (trilinear): chosen with -Xptxas -v, see DESIGN.md section 4c
#endif
#ifndef NR_IGU_MIN_CTAS
#define NR_IGU_MIN_CTAS 4       // k_image_grad with the face_uvs gradient: 56 registers, no spills (DESIGN.md section 4c)
#endif
#ifndef NR_IGMU_MIN_CTAS
#define NR_IGMU_MIN_CTAS 3      // k_image_grad_mip with the face_uvs gradient: 79 registers, no spills
#endif

namespace {

// Phase-ablation switches exist only in experiment builds (-DNR_B200_DEBUG_KNOBS); the product never drops a term.
#ifdef NR_B200_DEBUG_KNOBS
#define NR_SKIP(p, bit) (((p).debug_skip & (bit)) != 0)
#else
#define NR_SKIP(p, bit) false
#endif

// k_edge_scan<kMode, kT>: kT threads per CTA; 2*kT queued faces (<= 9-bit slot), 8*kT scan tasks (<= 12-bit rank) per round
constexpr int kEdgeScanThreadsDefault = 128;
constexpr int kEsUnroll = NR_ES_UNROLL;
constexpr int kMaxLines = 16;                 // W upper bound (4-bit line in a task word)
constexpr int kStripBytesDefault = 16 * 1024; // shared memory budget for the staged strip (NR_B200_STRIP_KB overrides)

struct BwdParams {
    nr::FaceSrc src;
    nr::FaceGrad dst;
    const int32_t* fim;
    const float* wmap;
    const float* dmap;
    const float* rgb;
    const float* g_rgb;
    const float* g_alpha;
    const float* g_depth;
    const uint2* bbox;
    const uint2* chunk_bbox;
    const int* strip_cnt;   // [B*2*(nstrips+1)]  faces per (item, axis, strip); slot nstrips = faces wider than kWideStrips
    const int* strip_off;   // exclusive prefix of strip_cnt
    const int* strip_list;  // face indices, grouped by (item, axis, strip)
    float* grad_textures;   // the layout of tex.tex
    float* grad_face_light;
    float* grad_corner_light;  // d loss / d corner_light (the kLightCorner variants), or nullptr
    int B, F, S, ts, nchunks;
    int W;          // lines per strip (power of two)
    int w_log2, nstrips;
    int len_shift;  // scan length >> len_shift -> one of 32 sort buckets
    int stage_fast; // even raster + 8-byte aligned maps: strips are staged with 8-byte loads
    int col_smem;   // the strip keeps the pixels' colours in shared memory (rasters up to kColSmemMaxS)
    float* zero_dst;          // 16-byte aligned buffer that the edge scan's CTAs zero-fill on the side (grad_textures), or nullptr
    unsigned long long zero_count;    // floats
    unsigned long long zero_per_cta;  // float4 per CTA
#ifdef NR_B200_DEBUG_KNOBS
    int debug_skip; // ablation knob of experiment builds (NR_B200_ES_SKIP): 1 = no in-scan, 2 = no out-scan, 4 = no task processing
#endif
    uint32_t flags;
    float eps, two_over_S;
    nr::Texture tex;  // what the pixel samples
    float* grad_uvs;  // d loss / d face_uvs (the layout of tex.uvs), or nullptr
    // what lights the pixel: face_light, corner_light or the Phong inputs of the call's light mode
    nr::Shading shading;
};

//@phase helpers: rcp / vector RED / load_grad (inlined)
// MUFU.RCP (about 1 ulp): the edge-scan terms are held to 1e-4 relative, not to bit-exactness
__device__ __forceinline__ float rcp_approx(float x) {
    float r;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}

using nr::red_add_v2;  // vector float reductions (nr_math.cuh)
using nr::red_add_v4;

// upstream gradient of raster pixel (row, col) of plane `pl` -- folds the 2x2 average-pooling backward
__device__ __forceinline__ float load_grad(const float* g, bool aa, int S, size_t img_plane_index, int row, int col) {
    if (!aa) return __ldg(g + img_plane_index * (size_t)S * S + (size_t)row * S + col);
    const int H = S >> 1;
    return 0.25f * __ldg(g + img_plane_index * (size_t)H * H + (size_t)(row >> 1) * H + (col >> 1));
}

// ------------------------------------------------------------------------------------------------ strip binning
// Every front face is appended to the list of each strip its pixel box overlaps, per axis (count -> scan -> fill), so a
// strip CTA reads exactly its faces instead of culling all F boxes.  Faces spanning more than kWideStrips strips go
// to one "wide" list per (item, axis) that every strip of that item/axis walks with a box test; this bounds the list
// storage at kWideStrips entries per face and axis.
constexpr int kWideStrips = 8;

constexpr int kBinSmemStrips = 2048;  // strips (+1 wide slot) per axis whose counters fit the CTA's shared memory

// One CTA = 256 consecutive faces of one item.  The faces are first counted per strip in SHARED memory (neighbouring
// faces hit the same few strips: native shared-memory integer atomics instead of contended global ones); the CTA then
// touches every non-empty global counter / cursor ONCE to publish its count (kFill = false) or to reserve its range of
// the list (kFill = true), and the faces are written at reserved base + local rank.
// The two launches also do what used to be launches of their own (4 small latency-bound kernels -> 2): the counting
// pass computes the faces' pixel boxes itself (k_face_bbox), and every CTA of the fill pass scans its item's 2 x
// (nstrips + 1) counters in shared memory (k_strip_scan) -- CTA 0 of an item leaves the offsets for the edge scan.
template <bool kFill>
__global__ void __launch_bounds__(256) k_strip_bin(const nr::FaceSrc src, uint2* __restrict__ bbox, int F, int S, int w_log2,
                                                   int nstrips, int* __restrict__ cnt, int* __restrict__ off,
                                                   int* __restrict__ cursor, int* __restrict__ list, long long seg_stride) {
    extern __shared__ int s_bin[];  // [2][nstrips + 1] local counts, then (fill) [2][nstrips + 1] offsets / reserved bases
    __shared__ int s_warp[8];
    const int b = blockIdx.y;
    const int tid = threadIdx.x, lane = tid & 31;
    const int f = blockIdx.x * blockDim.x + tid;
    const int nslots = 2 * (nstrips + 1);
    const size_t gbase = (size_t)b * nslots;
    int* s_cnt = s_bin;
    int* s_base = s_bin + nslots;
    for (int i = tid; i < nslots; i += blockDim.x) {
        s_cnt[i] = 0;
        if (kFill) s_base[i] = cnt[gbase + i];
    }
    __syncthreads();
    uint2 bb = make_uint2(pack16(1, 0), pack16(1, 0));
    if (f < F) {
        if (kFill) {
            bb = __ldg(bbox + (size_t)b * F + f);
        } else {
            const float *v0 = nr::face_vertex(src, b, f, 0), *v1 = nr::face_vertex(src, b, f, 1), *v2 = nr::face_vertex(src, b, f, 2);
            int xlo, xhi, ylo, yhi;
            if (face_pixel_box(__ldg(v0), __ldg(v0 + 1), __ldg(v1), __ldg(v1 + 1), __ldg(v2), __ldg(v2 + 1), S, xlo, xhi, ylo, yhi))
                bb = make_uint2(pack16(xlo, xhi), pack16(ylo, yhi));
            bbox[(size_t)b * F + f] = bb;
        }
    }
    if (kFill) {
        // exclusive scan of each axis' counters; segment (item, axis) owns list entries [seg * seg_stride, ...)
        for (int axis = 0; axis < 2; axis++) {
            int* a = s_base + axis * (nstrips + 1);
            const int n = nstrips + 1, K = (n + 255) >> 8;
            int sum = 0;
            for (int k = 0; k < K; k++) { const int i = tid * K + k; if (i < n) sum += a[i]; }
            int incl = sum;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const int t = __shfl_up_sync(0xffffffffu, incl, o);
                if (lane >= o) incl += t;
            }
            if (lane == 31) s_warp[tid >> 5] = incl;
            __syncthreads();
            int run = (int)(((long long)b * 2 + axis) * seg_stride) + incl - sum;
            for (int w = 0; w < (tid >> 5); w++) run += s_warp[w];
            for (int k = 0; k < K; k++) {
                const int i = tid * K + k;
                if (i < n) { const int v = a[i]; a[i] = run; run += v; }
            }
            __syncthreads();
        }
        if (blockIdx.x == 0)
            for (int i = tid; i < nslots; i += blockDim.x) off[gbase + i] = s_base[i];
    }
    const bool active = unpack_lo(bb.x) <= unpack_hi(bb.x);  // culled faces carry an empty box
    int slot0[2], nslot[2];
    int rank[2][kWideStrips];
#pragma unroll
    for (int axis = 0; axis < 2; axis++) {
        const uint32_t v = axis == 0 ? bb.x : bb.y;
        const int s_lo = unpack_lo(v) >> w_log2, s_hi = unpack_hi(v) >> w_log2;
        const bool wide = s_hi - s_lo + 1 > kWideStrips;
        slot0[axis] = axis * (nstrips + 1) + (wide ? nstrips : s_lo);
        nslot[axis] = active ? (wide ? 1 : s_hi - s_lo + 1) : 0;
#pragma unroll
        for (int k = 0; k < kWideStrips; k++) {
            rank[axis][k] = 0;
            if (k < nslot[axis]) rank[axis][k] = atomicAdd(&s_cnt[slot0[axis] + k], 1);
        }
    }
    __syncthreads();
    for (int i = tid; i < nslots; i += blockDim.x) {
        const int c = s_cnt[i];
        if (c == 0) continue;
        if (!kFill) atomicAdd(cnt + gbase + i, c);
        else s_base[i] += atomicAdd(cursor + gbase + i, c);
    }
    if (!kFill) return;
    __syncthreads();
#pragma unroll
    for (int axis = 0; axis < 2; axis++)
#pragma unroll
        for (int k = 0; k < kWideStrips; k++)
            if (k < nslot[axis]) list[s_base[slot0[axis] + k] + rank[axis][k]] = f;
}

// The same binning with global atomics only, for rasters with more strips than the shared-memory counters hold.
template <bool kFill>
__global__ void __launch_bounds__(256) k_strip_bin_global(const uint2* __restrict__ bbox, int F, int w_log2, int nstrips,
                                                          int* __restrict__ cnt, const int* __restrict__ off,
                                                          int* __restrict__ cursor, int* __restrict__ list) {
    const int b = blockIdx.y;
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= F) return;
    const uint2 bb = __ldg(bbox + (size_t)b * F + f);
    if (unpack_lo(bb.x) > unpack_hi(bb.x)) return;  // culled face
#pragma unroll
    for (int axis = 0; axis < 2; axis++) {
        const uint32_t v = axis == 0 ? bb.x : bb.y;
        const int s_lo = unpack_lo(v) >> w_log2, s_hi = unpack_hi(v) >> w_log2;
        const size_t base = ((size_t)b * 2 + axis) * (nstrips + 1);
        if (s_hi - s_lo + 1 > kWideStrips) {
            if (!kFill) atomicAdd(cnt + base + nstrips, 1);
            else list[off[base + nstrips] + atomicAdd(cursor + base + nstrips, 1)] = f;
        } else {
            for (int st = s_lo; st <= s_hi; st++) {
                if (!kFill) atomicAdd(cnt + base + st, 1);
                else list[off[base + st] + atomicAdd(cursor + base + st, 1)] = f;
            }
        }
    }
}

// Exclusive prefix sum of the nstrips + 1 counters of one (item, axis) segment; every segment owns a fixed region of
// the list storage (seg_stride entries: at most kWideStrips per face), so segments are scanned independently.
__global__ void __launch_bounds__(256) k_strip_scan(const int* __restrict__ cnt, int* __restrict__ off, int seg_len,
                                                    long long seg_stride) {
    __shared__ int warp_sum[8];
    __shared__ int carry;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const size_t seg = blockIdx.x;
    cnt += seg * seg_len;
    off += seg * seg_len;
    if (tid == 0) carry = 0;
    __syncthreads();
    for (int base = 0; base < seg_len; base += 256) {
        const int i = base + tid;
        const int v = i < seg_len ? cnt[i] : 0;
        int incl = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int t = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += t;
        }
        if (lane == 31) warp_sum[warp] = incl;
        __syncthreads();
        if (warp == 0) {
            const int w = lane < 8 ? warp_sum[lane] : 0;
            int wi = w;
#pragma unroll
            for (int o = 1; o < 8; o <<= 1) {
                const int t = __shfl_up_sync(0xffffffffu, wi, o);
                if (lane >= o) wi += t;
            }
            if (lane < 8) warp_sum[lane] = wi - w;  // exclusive
        }
        __syncthreads();
        const int c = carry;
        if (i < seg_len) off[i] = (int)(seg * seg_stride) + c + warp_sum[warp] + incl - v;
        __syncthreads();
        if (tid == 255) carry = c + warp_sum[warp] + incl;
        __syncthreads();
    }
}

// ------------------------------------------------------------------------------------------------ k_edge_scan
//@phase f32x2 pair helpers (the out-scan's math is attributed here)
// fp32 pairs: two pixels of a scan advance together.  sm_90 has no packed fp32 instructions, so each pair operation
// is two independent scalar FFMA / FMUL / FADD (two dependency chains per lane), rounded per element exactly like
// the packed fma.rn / mul.rn / add.rn forms.
struct f32x2 {
    float x, y;
};
__device__ __forceinline__ f32x2 pk(float a, float b) { return f32x2{a, b}; }
__device__ __forceinline__ void upk(f32x2 v, float& a, float& b) { a = v.x; b = v.y; }
__device__ __forceinline__ f32x2 fma2(f32x2 a, f32x2 b, f32x2 c) { return f32x2{__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y)}; }
__device__ __forceinline__ f32x2 add2(f32x2 a, f32x2 b) { return f32x2{__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)}; }
__device__ __forceinline__ f32x2 mul2(f32x2 a, f32x2 b) { return f32x2{__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)}; }

// Shared-memory strip.  Pixels of a line are stored as PAIRS (2*pp, 2*pp+1) so that one 16-byte load feeds the
// multiply-adds of both pixels (one f32x2 pair step):
//   P[pp] = {A_e, A_o, g0_e, g0_o}   A = sum_c I_c * g_c (+ alpha * g_alpha): the scan evaluates the reference's
//   Q[pp] = {g1_e, g1_o, g2_e, g2_o}     diff_grad = sum_c (I_c - ref_c) * g_c  as  A - sum_c ref_c * g_c
//   R[pp] = {ga_e, ga_o}             only when both rgb and alpha gradients exist (kMode == 3)
//   ci[i] = {I0, I1, I2, fim}        colours and face index per pixel: task set-up and the short in-scan only (kCol)
//   fs[i] = fim                      face index only (!kCol): larger rasters keep 20 instead of 32 bytes per pixel in
//                                    shared memory (more CTAs per SM at raster 512) and fetch the two
//                                    reference colours of a task from the global rgb map (L2 hits) when it is set up
// kMode: 1 = rgb, 2 = alpha only (g0 = g_alpha, I0 = alpha), 3 = rgb + alpha
//@phase prologue
template <int kMode, int kThreads, bool kIdx, bool kCol>
__global__ void __launch_bounds__(kThreads, NR_ES_CTAS_PER_1024 * 1024 / kThreads / 8) k_edge_scan(const __grid_constant__ BwdParams p) {
    constexpr int kFaceQueue = 2 * kThreads, kTaskCap = 8 * kThreads;
    static_assert(kFaceQueue <= 512 && kTaskCap <= 4096, "task word layout");
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int S = p.S, W = p.W;
    const int Sp = (S + 1) & ~1, npair = Sp >> 1;
    float4* P = reinterpret_cast<float4*>(smem_raw);
    float4* Q = P + (size_t)W * npair;
    float4* ci = Q + (size_t)W * npair;                  // kCol
    int* fs = reinterpret_cast<int*>(Q + (size_t)W * npair);  // !kCol (same place)
    float2* R = kCol ? reinterpret_cast<float2*>(ci + (size_t)W * Sp) : reinterpret_cast<float2*>(fs + (size_t)W * Sp);
    __shared__ int s_faceq[kFaceQueue];
    __shared__ uint32_t s_tmp[kTaskCap];     // unsorted tasks: q<<23 | e<<21 | line<<17 | bucket<<12 | rank
    __shared__ uint16_t s_sorted[kTaskCap];  // tasks ordered by descending scan length: q<<6 | e<<4 | line
    __shared__ int s_hist[32], s_off[32];
    __shared__ int s_nface, s_ntask, s_next;

    const int tid = threadIdx.x, lane = tid & 31;
    const int axis = blockIdx.y, b = blockIdx.z;
    const int l0 = blockIdx.x * W;
    // Side job: the zero-fill of grad_textures (246 MB of pure HBM writes at the headline shape, a memset of its
    // own) is spread over this kernel's CTAs -- the edge scan is issue-bound and leaves the DRAM mostly idle, so the
    // (streaming) stores ride
    // along; K6 runs after this kernel instead of before it.
    auto side_fill = [&]() {
        if (!p.zero_dst) return;
        const unsigned long long cta = blockIdx.x + (unsigned long long)gridDim.x * (blockIdx.y + (unsigned long long)gridDim.y * blockIdx.z);
        const unsigned long long n4 = p.zero_count >> 2;
        const unsigned long long lo = cta * p.zero_per_cta, hi = min(lo + p.zero_per_cta, n4);
        float4* d = reinterpret_cast<float4*>(p.zero_dst);
        for (unsigned long long i = lo + tid; i < hi; i += kThreads) NR_FILL_STORE(d + i, make_float4(0.0f, 0.0f, 0.0f, 0.0f));
        if (cta == 0 && tid < (int)(p.zero_count & 3)) p.zero_dst[(n4 << 2) + tid] = 0.0f;
    };
#if NR_FILL_AT_END == 0
    side_fill();
#endif
    const int nlines = min(W, S - l0);
    const bool aa = (p.flags & NR_ANTI_ALIASING) != 0;
    const size_t plane = (size_t)S * S;

    //@phase 1 stage strip
    // ---- 1. stage the strip (image orientation in global memory: raster row y is stored at row S-1-y).
    //         One thread per pixel PAIR of a line: 16-byte shared-memory stores, half the index arithmetic.
    struct Px { float A, g0, g1, g2, ga; float4 c; };
    auto load_px = [&](int line, int d1) {
        Px q;
        q.c = make_float4(0.f, 0.f, 0.f, __int_as_float(-1));
        q.A = q.g0 = q.g1 = q.g2 = q.ga = 0.f;
        if (d1 >= S || NR_SKIP(p, 8)) return q;  // the padding pixel of an odd raster size stays zero
        const int x = (axis == 0) ? l0 + line : d1, y = (axis == 0) ? d1 : l0 + line;
        const int row = S - 1 - y;
        const size_t o = (size_t)row * S + x;
        const int fi = __ldg(p.fim + (size_t)b * plane + o);
        q.c.w = __int_as_float(fi);
        const float alpha = fi >= 0 ? 1.0f : 0.0f;
        if (kMode == 2) {
            q.g0 = load_grad(p.g_alpha, aa, S, (size_t)b, row, x);
            q.c.x = alpha;
            q.A = alpha * q.g0;
        } else {
            const float* rm = p.rgb + (size_t)b * 3 * plane + o;
            q.c.x = __ldg(rm); q.c.y = __ldg(rm + plane); q.c.z = __ldg(rm + 2 * plane);
            q.g0 = load_grad(p.g_rgb, aa, S, (size_t)b * 3 + 0, row, x);
            q.g1 = load_grad(p.g_rgb, aa, S, (size_t)b * 3 + 1, row, x);
            q.g2 = load_grad(p.g_rgb, aa, S, (size_t)b * 3 + 2, row, x);
            float acc = 0.0f;
            if (kMode == 3) {
                q.ga = load_grad(p.g_alpha, aa, S, (size_t)b, row, x);
                acc = alpha * q.ga;
            }
            q.A = __fmaf_rn(q.c.z, q.g2, __fmaf_rn(q.c.y, q.g1, __fmaf_rn(q.c.x, q.g0, acc)));
        }
        return q;
    };
    // Fast path (two-line strips of an even raster, 8-byte aligned maps): a thread stages a 2 x 2 block of pixels (column
    // strips: two image rows x the strip's two columns; row strips: one pixel pair of a line) with ONE 8-byte load per
    // plane and image row instead of one 4-byte load per plane and pixel; with anti-aliasing the four pixels of a block
    // share one texel of the pooled upstream gradient.
    const bool stage_fast = p.stage_fast && nlines == 2 && W == 2;
    if (stage_fast) {
        const int H = S >> 1;
        const int32_t* fimb = p.fim + (size_t)b * plane;
        const float* rgbb = (kMode != 2) ? p.rgb + (size_t)b * 3 * plane : nullptr;
        auto pooled = [&](const float* g, size_t pl, int row, int col) {
            return 0.25f * __ldg(g + pl * (size_t)H * H + (size_t)(row >> 1) * H + (col >> 1));
        };
        struct Px2 { float A[2], g0[2], g1[2], g2[2], ga[2]; float4 c[2]; };
        // two horizontally adjacent pixels (row, x), (row, x + 1) of the image, x even
        auto load2 = [&](int row, int x) {
            Px2 q;
            const size_t o = (size_t)row * S + x;
            const int2 fi = __ldg(reinterpret_cast<const int2*>(fimb + o));
            const int f2[2] = {fi.x, fi.y};
            float g[4][2] = {{0.f, 0.f}, {0.f, 0.f}, {0.f, 0.f}, {0.f, 0.f}};  // g0 g1 g2 ga
            float col[3][2] = {{0.f, 0.f}, {0.f, 0.f}, {0.f, 0.f}};
            if (kMode != 2) {
#pragma unroll
                for (int c = 0; c < 3; c++) {
                    const float2 v = __ldg(reinterpret_cast<const float2*>(rgbb + (size_t)c * plane + o));
                    col[c][0] = v.x; col[c][1] = v.y;
                    if (aa) {
                        g[c][0] = g[c][1] = pooled(p.g_rgb, (size_t)b * 3 + c, row, x);
                    } else {
                        const float2 w = __ldg(reinterpret_cast<const float2*>(p.g_rgb + ((size_t)b * 3 + c) * plane + o));
                        g[c][0] = w.x; g[c][1] = w.y;
                    }
                }
            }
            if (kMode != 1) {
                if (aa) {
                    g[3][0] = g[3][1] = pooled(p.g_alpha, (size_t)b, row, x);
                } else {
                    const float2 w = __ldg(reinterpret_cast<const float2*>(p.g_alpha + (size_t)b * plane + o));
                    g[3][0] = w.x; g[3][1] = w.y;
                }
            }
#pragma unroll
            for (int k = 0; k < 2; k++) {
                const float alpha = f2[k] >= 0 ? 1.0f : 0.0f;
                if (kMode == 2) {
                    q.g0[k] = g[3][k]; q.g1[k] = q.g2[k] = q.ga[k] = 0.f;
                    q.c[k] = make_float4(alpha, 0.f, 0.f, __int_as_float(f2[k]));
                    q.A[k] = alpha * g[3][k];
                } else {
                    q.g0[k] = g[0][k]; q.g1[k] = g[1][k]; q.g2[k] = g[2][k]; q.ga[k] = g[3][k];
                    q.c[k] = make_float4(col[0][k], col[1][k], col[2][k], __int_as_float(f2[k]));
                    const float acc = (kMode == 3) ? alpha * g[3][k] : 0.0f;
                    q.A[k] = __fmaf_rn(col[2][k], g[2][k], __fmaf_rn(col[1][k], g[1][k], __fmaf_rn(col[0][k], g[0][k], acc)));
                }
            }
            return q;
        };
        auto put = [&](int line, int pp, const float A[2], const float g0[2], const float g1[2], const float g2[2], const float ga[2],
                       const float4& ce, const float4& co) {
            const size_t pi = (size_t)line * npair + pp;
            P[pi] = make_float4(A[0], A[1], g0[0], g0[1]);
            if (kMode != 2) Q[pi] = make_float4(g1[0], g1[1], g2[0], g2[1]);
            if (kMode == 3) R[pi] = make_float2(ga[0], ga[1]);
            if (kCol) {
                ci[(size_t)line * Sp + 2 * pp] = ce;
                ci[(size_t)line * Sp + 2 * pp + 1] = co;
            } else {
                *reinterpret_cast<int2*>(fs + (size_t)line * Sp + 2 * pp) = make_int2(__float_as_int(ce.w), __float_as_int(co.w));
            }
        };
        if (axis == 0) {
            // columns l0, l0 + 1; pair pp = raster rows y = 2pp, 2pp + 1 = image rows S-1-2pp and one above
            for (int pp = tid; pp < npair; pp += kThreads) {
                const int r0 = S - 1 - 2 * pp;
                const Px2 a = load2(r0, l0), c = load2(r0 - 1, l0);  // a: y = 2pp (lines 0, 1), c: y = 2pp + 1
#pragma unroll
                for (int line = 0; line < 2; line++) {
                    const float A[2] = {a.A[line], c.A[line]}, g0[2] = {a.g0[line], c.g0[line]}, g1[2] = {a.g1[line], c.g1[line]},
                                g2[2] = {a.g2[line], c.g2[line]}, ga[2] = {a.ga[line], c.ga[line]};
                    put(line, pp, A, g0, g1, g2, ga, a.c[line], c.c[line]);
                }
            }
        } else {
            // rows y = l0, l0 + 1; pair pp = columns 2pp, 2pp + 1 of one image row
            for (int i = tid; i < 2 * npair; i += kThreads) {
                const int line = i / npair, pp = i - line * npair;
                const Px2 a = load2(S - 1 - (l0 + line), 2 * pp);
                put(line, pp, a.A, a.g0, a.g1, a.g2, a.ga, a.c[0], a.c[1]);
            }
        }
    } else
    for (int i = tid; i < nlines * npair; i += kThreads) {
        int line, pp;
        if (axis == 0) { line = i % nlines; pp = i / nlines; }   // columns: d0 = x, d1 = y
        else           { line = i / npair;  pp = i % npair; }
        const Px e = load_px(line, 2 * pp), o = load_px(line, 2 * pp + 1);
        const size_t pi = (size_t)line * npair + pp;
        P[pi] = make_float4(e.A, o.A, e.g0, o.g0);
        if (kMode != 2) Q[pi] = make_float4(e.g1, o.g1, e.g2, o.g2);
        if (kMode == 3) R[pi] = make_float2(e.ga, o.ga);
        if (kCol) {
            ci[(size_t)line * Sp + 2 * pp] = e.c;
            ci[(size_t)line * Sp + 2 * pp + 1] = o.c;
        } else {
            *reinterpret_cast<int2*>(fs + (size_t)line * Sp + 2 * pp) = make_int2(__float_as_int(e.c.w), __float_as_int(o.c.w));
        }
    }
    if (tid < 32) s_hist[tid] = 0;
    if (tid == 0) { s_nface = 0; s_ntask = 0; s_next = 0; }
    __syncthreads();

    const uint2* bbox = p.bbox + (size_t)b * p.F;
    const float fS = (float)S;
    const int lhi = l0 + nlines - 1;
    // face index / {I0, I1, I2, fim} of pixel d1 of a line of the strip
    auto fim_at = [&](int line, int d1) -> int {
        return kCol ? __float_as_int(ci[(size_t)line * Sp + d1].w) : fs[(size_t)line * Sp + d1];
    };
    auto colour_at = [&](int line, int d1) -> float4 {
        if (kCol) return ci[(size_t)line * Sp + d1];
        const int fi = fs[(size_t)line * Sp + d1];
        float4 c = make_float4(fi >= 0 ? 1.0f : 0.0f, 0.0f, 0.0f, __int_as_float(fi));  // kMode 2: I0 = alpha
        if (kMode != 2) {
            const int x = (axis == 0) ? l0 + line : d1, y = (axis == 0) ? d1 : l0 + line;
            const float* rm = p.rgb + (size_t)b * 3 * plane + (size_t)(S - 1 - y) * S + x;
            c.x = __ldg(rm); c.y = __ldg(rm + plane); c.z = __ldg(rm + 2 * plane);
        }
        return c;
    };

    //@phase task_setup (inlined into 2b and 3)
    // Geometry of one (face, edge, line) scan, evaluated exactly as rasterize.py:545-609 / :662-672 does.
    struct Task {
        float d1_cross, k0, k1;  // dist_v = (d1 - d1_cross) * k_v  (k_v = ratio_v * 2 / S), +-eps
        bool has0, has1;         // vertex not exactly on this line (rasterize.py:648, :653)
        int dir, d1_in, d1_out;  // crossing pixel inside / outside the face
        int out_from, out_to;    // out-scan range (empty unless the inside pixel shows this face)
        int in_from, in_to;      // in-scan range
        int pi0, pi1;
        bool valid;
    };
    auto task_setup = [&](int f, int e, int line, Task& T) {
        const int pi0 = e, pi1 = (e + 1) % 3, pi2 = (e + 2) % 3;
        const float *v0 = nr::face_vertex_t<kIdx>(p.src, b, f, pi0), *v1 = nr::face_vertex_t<kIdx>(p.src, b, f, pi1);
        const int a = axis, c = 1 - axis;
        T.pi0 = pi0; T.pi1 = pi1;
        T.valid = false;
        T.out_from = 0; T.out_to = -1; T.in_from = 0; T.in_to = -1;
        const float p00 = nr::to_pixel(__ldg(v0 + a), fS), p10 = nr::to_pixel(__ldg(v1 + a), fS);
        // (int)max(ceil(min(p0,p1)), 0.) and (int)min(max(p0,p1), is - 1.): truncating conversions (NaN -> 0)
        const int d0_from = __float2int_rz(fmaxf(ceilf(fminf(p00, p10)), 0.0f));
        const int d0_to = __float2int_rz(fminf(fmaxf(p00, p10), (float)(S - 1)));
        const int d0 = l0 + line;
        if (d0 < d0_from || d0 > d0_to) return;  // most (face, edge, line) slots end here
        const float p01 = nr::to_pixel(__ldg(v0 + c), fS), p11 = nr::to_pixel(__ldg(v1 + c), fS);
        const bool lt = p00 < p10;
        T.dir = (axis == 0) ? (lt ? -1 : 1) : (lt ? 1 : -1);
        const float fd0 = (float)d0;
        const float slope = __fdiv_rn(__fsub_rn(p11, p01), __fsub_rn(p10, p00));
        T.d1_cross = __fmaf_rn(__fsub_rn(fd0, p00), slope, p01);
        T.d1_in = __float2int_rz(T.dir > 0 ? floorf(T.d1_cross) : ceilf(T.d1_cross));
        T.d1_out = T.d1_in + T.dir;
        if (T.d1_in < 0 || T.d1_in >= S || T.d1_out < 0 || T.d1_out >= S) return;
        T.valid = true;
        T.has0 = (p10 != fd0); T.has1 = (p00 != fd0);
        const float len = __fsub_rn(p10, p00);
        T.k0 = __fdiv_rn(len, __fsub_rn(p10, fd0)) * p.two_over_S;
        T.k1 = __fdiv_rn(len, __fsub_rn(fd0, p00)) * p.two_over_S;
        // out-scan: from the outside pixel to the image border, only if the inside pixel shows this face
        if (fim_at(line, T.d1_in) == f) {
            const int lim = (T.dir > 0) ? S - 1 : 0;
            T.out_from = max(min(T.d1_out, lim), 0);
            T.out_to = min(max(T.d1_out, lim), S - 1);
        }
        // in-scan: from the inside pixel to where this line leaves the face through one of the other two edges
        const float* v2 = nr::face_vertex_t<kIdx>(p.src, b, f, pi2);
        const float p20 = nr::to_pixel(__ldg(v2 + a), fS), p21 = nr::to_pixel(__ldg(v2 + c), fS);
        float ba, bb, ea, eb;
        if (__fmul_rn(__fsub_rn(fd0, p00), __fsub_rn(fd0, p20)) < 0.0f) { ba = p00; bb = p01; ea = p20; eb = p21; }
        else { ba = p20; bb = p21; ea = p10; eb = p11; }
        const float cross2 = __fmaf_rn(__fsub_rn(fd0, ba), __fdiv_rn(__fsub_rn(eb, bb), __fsub_rn(ea, ba)), bb);
        const int lim2 = __float2int_rz(T.dir > 0 ? ceilf(cross2) : floorf(cross2));
        T.in_from = max(min(T.d1_in, lim2), 0);
        T.in_to = min(max(T.d1_in, lim2), S - 1);
    };
    //@phase scalar visit (in-scan)
    // scalar visit (in-scan, and out-scans of the rare tasks with a vertex exactly on the line)
    auto visit = [&](const Task& T, int line, int d1, float r0, float r1, float r2, float ra, float& acc0, float& acc1) {
        const size_t pi = (size_t)line * npair + (d1 >> 1);
        const int h = d1 & 1;
        float dg = reinterpret_cast<const float*>(P + pi)[h];
        dg = __fmaf_rn(-r0, reinterpret_cast<const float*>(P + pi)[2 + h], dg);
        if (kMode != 2) {
            dg = __fmaf_rn(-r1, reinterpret_cast<const float*>(Q + pi)[h], dg);
            dg = __fmaf_rn(-r2, reinterpret_cast<const float*>(Q + pi)[2 + h], dg);
        }
        if (kMode == 3) dg = __fmaf_rn(-ra, reinterpret_cast<const float*>(R + pi)[h], dg);
        if (!(dg > 0.0f)) return;
        const float tt = __fsub_rn((float)d1, T.d1_cross);
        if (T.has0) {
            float dist = tt * T.k0;
            dist = (0.0f < dist) ? dist + p.eps : dist - p.eps;
            acc0 -= __fdividef(dg, dist);
        }
        if (T.has1) {
            float dist = tt * T.k1;
            dist = (0.0f < dist) ? dist + p.eps : dist - p.eps;
            acc1 -= __fdividef(dg, dist);
        }
    };

    //@phase 2a face lists
    const int len_shift = p.len_shift;  // scan length >> len_shift indexes 32 sort buckets
    // faces are queued until the next batch of kThreads could overflow the face queue or the task expansion
    const int cap_faces = min(kFaceQueue, kTaskCap / (3 * nlines));
    int nface = 0;  // uniform across the CTA
    const size_t cid = ((size_t)b * 2 + axis) * (p.nstrips + 1);
    const int n_own = __ldg(p.strip_cnt + cid + blockIdx.x), n_wide = __ldg(p.strip_cnt + cid + p.nstrips);
    const int* own = p.strip_list + __ldg(p.strip_off + cid + blockIdx.x);
    const int* wide = p.strip_list + __ldg(p.strip_off + cid + p.nstrips);
    const int ncand = n_own + n_wide;
    for (int base = 0; base < ncand && !NR_SKIP(p, 16); base += kThreads) {
        // ---- 2a. this strip's faces (binned by k_strip_bin) plus the item's wide faces that overlap it
        const int i = base + tid;
        const bool last = base + kThreads >= ncand;
        bool pass = false;
        int f = 0;
        if (i < n_own) {
            f = __ldg(own + i);
            pass = true;
        } else if (i < ncand) {
            f = __ldg(wide + (i - n_own));
            const uint2 bb = __ldg(bbox + f);
            const uint32_t v = (axis == 0) ? bb.x : bb.y;
            pass = !(unpack_lo(v) > lhi || unpack_hi(v) < l0);
        }
        const int cnt = __syncthreads_count(pass);
        if (cnt) {
            const uint32_t m = __ballot_sync(0xffffffffu, pass);
            if (m) {
                int pos = 0;
                if (lane == 0) pos = atomicAdd(&s_nface, __popc(m));
                pos = __shfl_sync(0xffffffffu, pos, 0);
                if (pass) s_faceq[pos + __popc(m & ((1u << lane) - 1u))] = f;
            }
            nface += cnt;
        }
        if (nface == 0 || (!last && nface + kThreads <= cap_faces)) continue;
        __syncthreads();

        // the queue may hold more faces than one expansion round can take (cap_faces < kThreads for wide strips)
        for (int q0 = 0; q0 < nface; q0 += cap_faces) {
            const int nq = min(cap_faces, nface - q0);
            //@phase 2b expand + sort
            // ---- 2b. expand (face, edge, line) slots; valid ones become tasks bucketed by scan length
            for (int i = tid; i < nq * 3; i += kThreads) {
                const int e = i % 3, q = q0 + i / 3;
                const int f = s_faceq[q];
                // lines of the strip that this edge spans (same truncating conversions as task_setup)
                const float p00 = nr::to_pixel(__ldg(nr::face_vertex_t<kIdx>(p.src, b, f, e) + axis), fS),
                            p10 = nr::to_pixel(__ldg(nr::face_vertex_t<kIdx>(p.src, b, f, (e + 1) % 3) + axis), fS);
                const int lo = max(__float2int_rz(fmaxf(ceilf(fminf(p00, p10)), 0.0f)), l0);
                const int hi = min(__float2int_rz(fminf(fmaxf(p00, p10), (float)(S - 1))), lhi);
                if (lo > hi) continue;
                // Only what decides whether the slot is a task and how long it runs: the crossing (rasterize.py:567-573,
                // slope hoisted out of the line loop) and the face_index_map gate of the out-scan (:604).  The full
                // geometry of a task is set up once, by the lane that runs it (phase 3).  (Without the gate in the sort
                // key the batches get uneven.)
                const float p01 = nr::to_pixel(__ldg(nr::face_vertex_t<kIdx>(p.src, b, f, e) + (1 - axis)), fS),
                            p11 = nr::to_pixel(__ldg(nr::face_vertex_t<kIdx>(p.src, b, f, (e + 1) % 3) + (1 - axis)), fS);
                const bool lt = p00 < p10;
                const int dir = (axis == 0) ? (lt ? -1 : 1) : (lt ? 1 : -1);
                const float slope = __fdiv_rn(__fsub_rn(p11, p01), __fsub_rn(p10, p00));
                for (int d0 = lo; d0 <= hi; d0++) {
                    const int line = d0 - l0;
                    const float d1_cross = __fmaf_rn(__fsub_rn((float)d0, p00), slope, p01);
                    const int d1_in = __float2int_rz(dir > 0 ? floorf(d1_cross) : ceilf(d1_cross));
                    const int d1_out = d1_in + dir;
                    if (d1_in < 0 || d1_in >= S || d1_out < 0 || d1_out >= S) continue;
                    const bool gate = fim_at(line, d1_in) == f;
                    // sort key: direction, then length -- a sub-pass of 8 out-scans then (almost always) runs one way,
                    // which lets the sweep use a compile-time stride (immediate address offsets, 4 steps per pointer bump)
                    const int L = (gate ? (dir > 0 ? S - 1 - d1_in : d1_in) : 0) + 8;
                    const int bucket = min(L >> len_shift, 15) + ((gate && dir > 0) ? 16 : 0);
                    const int rank = atomicAdd(&s_hist[bucket], 1);
                    const int t = atomicAdd(&s_ntask, 1);
                    s_tmp[t] = ((uint32_t)q << 23) | ((uint32_t)e << 21) | ((uint32_t)line << 17) | ((uint32_t)bucket << 12) | (uint32_t)rank;
                }
            }
            __syncthreads();
            const int ntask = s_ntask;
            if (tid < 32) {  // offsets: longest scans first
                const int h = s_hist[31 - lane];
                int incl = h;
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) {
                    const int v = __shfl_up_sync(0xffffffffu, incl, o);
                    if (lane >= o) incl += v;
                }
                s_off[31 - lane] = incl - h;
            }
            __syncthreads();
            for (int t = tid; t < ntask; t += kThreads) {
                const uint32_t e = s_tmp[t];
                const int bucket = (e >> 12) & 31, rank = e & 4095;
                s_sorted[s_off[bucket] + rank] = (uint16_t)(((e >> 23) << 6) | (((e >> 21) & 3) << 4) | ((e >> 17) & 15));
            }
            __syncthreads();

            //@phase 3 batches: set-up + in-scan
            // ---- 3. warps pull batches of 32 tasks of similar length.  Every lane sets up its own task and runs the
            //         short in-scan; the long out-scans are then swept by 4 lanes per task (8 tasks at a time), two
            //         pixels per lane and step (f32x2 pairs: two scalar FMA chains, 16-byte shared-memory loads).
            for (;;) {
                int t0 = 0;
                if (lane == 0) t0 = atomicAdd(&s_next, 32);
                t0 = __shfl_sync(0xffffffffu, t0, 0);
                if (t0 >= ntask || NR_SKIP(p, 4)) break;
                const int t = t0 + lane;
                Task T;
                T.valid = false; T.out_from = 0; T.out_to = -1; T.in_from = 0; T.in_to = -1;
                T.d1_cross = 0.f; T.k0 = 0.f; T.k1 = 0.f; T.has0 = T.has1 = true; T.dir = 1; T.d1_in = T.d1_out = 0; T.pi0 = T.pi1 = 0;
                int line = 0, fn = 0;
                if (t < ntask) {
                    const uint32_t tk = s_sorted[t];
                    line = tk & 15;
                    fn = s_faceq[tk >> 6];
                    task_setup(fn, (tk >> 4) & 3, line, T);
                }
                float acc0 = 0.0f, acc1 = 0.0f;  // this lane's own (scalar) contributions
                float c0 = 0.f, c1 = 0.f, c2 = 0.f, ca = 0.f;
                bool fast = false;
                if (T.valid) {
                    {   // in-scan (rasterize.py:662-730): reference colour = outside pixel, only pixels that show this face
                        const float4 cout = colour_at(line, T.d1_out);
                        const float ra = (kMode == 3) ? ((__float_as_int(cout.w) >= 0) ? 1.0f : 0.0f) : 0.0f;
                        for (int d1 = T.in_from; d1 <= T.in_to && !NR_SKIP(p, 1); d1++) {
                            if (fim_at(line, d1) != fn) continue;
                            visit(T, line, d1, cout.x, cout.y, cout.z, ra, acc0, acc1);
                        }
                    }
                    // out-scan (rasterize.py:604-659): reference colour = inside pixel
                    const float4 cin = colour_at(line, T.d1_in);
                    c0 = cin.x; c1 = cin.y; c2 = cin.z;
                    ca = (kMode == 3) ? ((__float_as_int(cin.w) >= 0) ? 1.0f : 0.0f) : 0.0f;
                    fast = T.has0 && T.has1;
                    if (!fast)
                        for (int d1 = T.out_from; d1 <= T.out_to; d1++) visit(T, line, d1, c0, c1, c2, ca, acc0, acc1);
                }
                //@phase 3 out-scan passes
                // along an out-scan (d1 - d1_cross) keeps the sign of dir, so the sign of eps is fixed per vertex
                const float fdir = (float)T.dir;
                const float e0 = (fdir * T.k0 > 0.0f) ? p.eps : -p.eps, e1 = (fdir * T.k1 > 0.0f) ? p.eps : -p.eps;
                const int my_from = (fast && !NR_SKIP(p, 2)) ? T.out_from : 1, my_to = (fast && !NR_SKIP(p, 2)) ? T.out_to : 0;

                const int qd = lane >> 2, j = lane & 3;  // 8 tasks per pass, 4 lanes (8 pixels per step) each
#pragma unroll 1
                for (int sub = 0; sub < 4; sub++) {
                    const int src = sub * 8 + qd;
                    const int o_from = __shfl_sync(0xffffffffu, my_from, src), o_to = __shfl_sync(0xffffffffu, my_to, src);
                    const int o_line = __shfl_sync(0xffffffffu, line, src);
                    const float o_dc = __shfl_sync(0xffffffffu, T.d1_cross, src);
                    const float o_k0 = __shfl_sync(0xffffffffu, T.k0, src), o_k1 = __shfl_sync(0xffffffffu, T.k1, src);
                    const float o_e0 = __shfl_sync(0xffffffffu, e0, src), o_e1 = __shfl_sync(0xffffffffu, e1, src);
                    const float o_c0 = __shfl_sync(0xffffffffu, c0, src), o_c1 = __shfl_sync(0xffffffffu, c1, src);
                    const float o_c2 = __shfl_sync(0xffffffffu, c2, src);
                    const float o_ca = (kMode == 3) ? __shfl_sync(0xffffffffu, ca, src) : 0.0f;
                    const int o_dir = __shfl_sync(0xffffffffu, T.dir, src);
                    const bool act = o_from <= o_to;
                    const uint32_t am = __ballot_sync(0xffffffffu, act);
                    if (am == 0) continue;
                    const uint32_t um = __ballot_sync(0xffffffffu, act && o_dir > 0);
                    f32x2 a0 = pk(0.f, 0.f), a1 = pk(0.f, 0.f);  // positive sums; the sign is applied at the hand-over
                    // An out-scan runs from the crossing to an image border, so only the pixel pair at the crossing end
                    // can hold a pixel outside [o_from, o_to] (the padding pixel of an odd raster size is staged as
                    // zeros).  Pairs are therefore walked FROM the crossing: the first step is peeled with the range
                    // gates, the steady-state loop carries none.  kDir = +-1: every out-scan of this sub-pass runs that
                    // way (compile-time stride); kDir = 0: mixed sub-pass at the boundary of the sort, run-time stride.
                    auto sweep = [&](auto dir_tag) {
                        constexpr int kDir = decltype(dir_tag)::value;
                        const int pa = o_from >> 1, npairs = (o_to >> 1) - pa + 1;
                        if (!(act && j < npairs)) return;
                        const bool up = kDir != 0 ? kDir > 0 : o_dir > 0;
                        const int dpp = kDir != 0 ? 4 * kDir : (up ? 4 : -4);
                        const float nc0 = -o_c0, nc1 = -o_c1, nc2 = -o_c2, nca = -o_ca;
                        const int pp = up ? pa + j : (o_to >> 1) - j;
                        const float4* Pp = P + (size_t)o_line * npair + pp;
                        const float4* Qp = Q + (size_t)o_line * npair + pp;
                        const float2* Rp = R + (size_t)o_line * npair + pp;
                        const float ta = __fsub_rn((float)(pp << 1), o_dc);  // d1 - d1_cross of the lane's first pixel
                        const f32x2 tt2 = pk(ta, ta + 1.0f);
                        // dist_v = (d1 - d1_cross) * k_v +- eps, advanced by +-8 pixels per step
                        f32x2 d0_2 = fma2(tt2, pk(o_k0, o_k0), pk(o_e0, o_e0)), d1_2 = fma2(tt2, pk(o_k1, o_k1), pk(o_e1, o_e1));
                        const float s8 = up ? 8.0f : -8.0f;
                        const f32x2 dk0 = pk(s8 * o_k0, s8 * o_k0), dk1 = pk(s8 * o_k1, s8 * o_k1);
                        auto diff_grad = [&](int off, float& dga, float& dgb) {
                            const float4 pv = Pp[off];
                            f32x2 dg2 = fma2(pk(nc0, nc0), pk(pv.z, pv.w), pk(pv.x, pv.y));
                            if (kMode != 2) {
                                const float4 qv = Qp[off];
                                dg2 = fma2(pk(nc1, nc1), pk(qv.x, qv.y), dg2);
                                dg2 = fma2(pk(nc2, nc2), pk(qv.z, qv.w), dg2);
                            }
                            if (kMode == 3) {
                                const float2 rv = Rp[off];
                                dg2 = fma2(pk(nca, nca), pk(rv.x, rv.y), dg2);
                            }
                            upk(dg2, dga, dgb);
                        };
                        auto accumulate = [&](float dga, float dgb) {
                            float qa, qb;
                            upk(mul2(d0_2, d1_2), qa, qb);
                            // one reciprocal serves both vertices: dg / d0 = dg * d1 / (d0 * d1)
                            const f32x2 t2 = mul2(pk(dga, dgb), pk(rcp_approx(qa), rcp_approx(qb)));
                            a0 = fma2(t2, d1_2, a0);
                            a1 = fma2(t2, d0_2, a1);
                            d0_2 = add2(d0_2, dk0);
                            d1_2 = add2(d1_2, dk1);
                        };
                        {   // first step: relu gate of rasterize.py:647 (max drops a NaN diff_grad) + range ends
                            float dga, dgb;
                            diff_grad(0, dga, dgb);
                            const int y0 = pp << 1;
                            dga = (y0 >= o_from) ? fmaxf(dga, 0.0f) : 0.0f;
                            dgb = (y0 + 1 <= o_to) ? fmaxf(dgb, 0.0f) : 0.0f;
                            accumulate(dga, dgb);
                        }
                        int rem = ((npairs - j + 3) >> 2) - 1;  // steps left for this lane
                        Pp += dpp; Qp += dpp; Rp += dpp;
#pragma unroll 1
                        for (; rem >= kEsUnroll; rem -= kEsUnroll) {
#pragma unroll
                            for (int k = 0; k < kEsUnroll; k++) {
                                float dga, dgb;
                                diff_grad(k * dpp, dga, dgb);
                                accumulate(fmaxf(dga, 0.0f), fmaxf(dgb, 0.0f));
                            }
                            Pp += kEsUnroll * dpp; Qp += kEsUnroll * dpp; Rp += kEsUnroll * dpp;
                        }
#pragma unroll 1
                        for (; rem > 0; rem--) {
                            float dga, dgb;
                            diff_grad(0, dga, dgb);
                            accumulate(fmaxf(dga, 0.0f), fmaxf(dgb, 0.0f));
                            Pp += dpp; Qp += dpp; Rp += dpp;
                        }
                    };
                    if (um == am) sweep(std::integral_constant<int, 1>{});
                    else if (um == 0) sweep(std::integral_constant<int, -1>{});
                    else sweep(std::integral_constant<int, 0>{});
                    float s0a, s0b, s1a, s1b;
                    upk(a0, s0a, s0b);
                    upk(a1, s1a, s1b);
                    float s0 = s0a + s0b, s1 = s1a + s1b;
#pragma unroll
                    for (int o = 1; o < 4; o <<= 1) {
                        s0 += __shfl_xor_sync(0xffffffffu, s0, o);
                        s1 += __shfl_xor_sync(0xffffffffu, s1, o);
                    }
                    // hand the totals to the lane that owns the task
                    const float r0 = __shfl_sync(0xffffffffu, s0, (lane & 7) << 2), r1 = __shfl_sync(0xffffffffu, s1, (lane & 7) << 2);
                    if ((lane >> 3) == sub) { acc0 -= r0; acc1 -= r1; }
                }
                if (acc0 != 0.0f) { float* g = nr::face_grad_vertex_t<kIdx>(p.dst, b, fn, T.pi0); if (g) atomicAdd(g + (1 - axis), acc0); }
                if (acc1 != 0.0f) { float* g = nr::face_grad_vertex_t<kIdx>(p.dst, b, fn, T.pi1); if (g) atomicAdd(g + (1 - axis), acc1); }
            }
            __syncthreads();
            if (tid < 32) s_hist[tid] = 0;
            if (tid == 0) { s_ntask = 0; s_next = 0; }
            __syncthreads();
        }
        if (tid == 0) s_nface = 0;
        nface = 0;
        __syncthreads();
    }
#if NR_FILL_AT_END == 1
    side_fill();
#endif
}

// ---------------------------------------------------------------------------------------- corner-light gradient
// d loss / d corner_light of one pixel from its unlit sample s, upstream gradient g and perspective weights l:
// [k][c] = l_k (g_c s_c), the face_light term g_c s_c spread over the corners
__device__ __forceinline__ void corner_light_grad(const float s[3], float g0, float g1, float g2, const float l[3], float (&gl)[9]) {
    const float gs[3] = {s[0] * g0, s[1] * g1, s[2] * g2};
#pragma unroll
    for (int k = 0; k < 3; k++)
#pragma unroll
        for (int c = 0; c < 3; c++) gl[3 * k + c] = l[k] * gs[c];
}

// warp-aggregated scatter of a light gradient into dst [B,F,N]: runs of neighbouring lanes that show the same face sum
// their N floats with a segmented shuffle and the run's first lane adds them -- the face_light tail of k_texture_grad /
// image_grad widened to N floats (the corner_light variants, N = 9; the face_light variants keep their own 3-float copy,
// whose SASS this form would change)
template <int N>
__device__ __forceinline__ void light_grad_scatter(float (&gl)[N], int fn, int lane, float* dst, int b, int F) {
    const int fn_prev = __shfl_up_sync(0xffffffffu, fn, 1);
    const uint32_t heads = __ballot_sync(0xffffffffu, lane == 0 || fn != fn_prev);
    const uint32_t later = heads & ~((2u << lane) - 1u);
    const int run_end = (lane == 31 || later == 0) ? 31 : (__ffs(later) - 2);
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
        const bool take = lane + off <= run_end;
        float t[N];
#pragma unroll
        for (int k = 0; k < N; k++) t[k] = __shfl_down_sync(0xffffffffu, gl[k], off);
        if (take) {
#pragma unroll
            for (int k = 0; k < N; k++) gl[k] += t[k];
        }
    }
    if (fn >= 0 && ((heads >> lane) & 1u)) {
        float* g = dst + ((size_t)b * F + fn) * N;
#pragma unroll
        for (int k = 0; k < N; k++) atomicAdd(g + k, gl[k]);
    }
}

// --------------------------------------------------------------------------------------------- k_texture_grad
// Neighbouring pixels of a face often blend the SAME eight texels (the same cell of the texture cube: 31 % of the
// covered pixels at the headline shape, 57 % at raster 512), and the L2 pays per reduction it receives.  Lanes of a warp
// that sit next to each other with the same (cube, cell) therefore add their 8 x 3 contributions together with
// kTgCombine shuffle steps first (runs of up to 2^kTgCombine lanes collapse into one lane's reductions).
//
// kLight (nr_shading.cuh): kLightNone serves unlit and face_light calls.  kCorner (kLightCorner): the pixel's light
// L_c = the corner factors interpolated with its perspective weights l_k (own vertex depths) takes face_light's place, and
// d loss / d corner_light = l_k g_c s_c goes through the same run reduction.  kPhong (the Phong modes): L_c = the diffuse
// part of the Phong expression at the pixel (nr::pixel_light) takes face_light's place; the Phong gradients themselves
// come from k_phong_grad (nr_phong.cu).
template <int kTgCombine, int kLight>
__global__ void __launch_bounds__(256, kTgCombine ? (kLight >= nr::kLightCorner ? NR_TGC_MIN_CTAS : 4) : NR_TG_MIN_CTAS) k_texture_grad(const __grid_constant__ BwdParams p) {
    constexpr bool kCorner = kLight == nr::kLightCorner, kPhong = kLight >= nr::kLightPhong;
    const int S = p.S;
    const size_t plane = (size_t)S * S;
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;  // pixel within the image (image orientation)
    const int b = blockIdx.y;
    const int lane = threadIdx.x & 31;
    const int fn = (i < plane) ? __ldg(p.fim + (size_t)b * plane + i) : -1;
    const bool want_light = !kPhong && (kCorner ? p.grad_corner_light : p.grad_face_light) != nullptr;  // uniform
    if (kTgCombine) {
        if (!want_light && !__any_sync(0xffffffffu, fn >= 0)) return;  // warp-uniform
    } else {
        if (fn < 0 && !want_light) return;
    }
    float gl0 = 0.0f, gl1 = 0.0f, gl2 = 0.0f;  // d loss / d face_light of this pixel
    float glc[kCorner ? 9 : 1];                // kCorner: d loss / d corner_light of this pixel
#pragma unroll
    for (int k = 0; k < (kCorner ? 9 : 1); k++) glc[k] = 0.0f;
    float val[4][6];                           // contributions to the four corner pairs (6 consecutive floats each)
    float* tp[4] = {nullptr, nullptr, nullptr, nullptr};
    long long key = -1 - (long long)lane;      // (cube, cell, orientation): equal keys <=> the same eight texels
#pragma unroll
    for (int pr = 0; pr < 4; pr++)
#pragma unroll
        for (int k = 0; k < 6; k++) val[pr][k] = 0.0f;
    if (fn >= 0) {
        const int row = (int)(i / S), col = (int)(i % S);
        const bool aa = (p.flags & NR_ANTI_ALIASING) != 0;
        float g0 = load_grad(p.g_rgb, aa, S, (size_t)b * 3 + 0, row, col);
        float g1 = load_grad(p.g_rgb, aa, S, (size_t)b * 3 + 1, row, col);
        float g2 = load_grad(p.g_rgb, aa, S, (size_t)b * 3 + 2, row, col);
        const float* wm = p.wmap + (size_t)b * 3 * plane + i;
        const float w[3] = {__ldg(wm), __ldg(wm + plane), __ldg(wm + 2 * plane)};
        const float zp = __ldg(p.dmap + (size_t)b * plane + i);
        const int zb = (p.flags & NR_TEX_Z_BATCH0) ? 0 : b;
        const int ts = p.ts;
        float z0, z1, z2;
        if (p.src.idx == nullptr) {
            const float* v = p.src.faces + ((size_t)zb * p.F + fn) * 9;
            z0 = __ldg(v + 2); z1 = __ldg(v + 5); z2 = __ldg(v + 8);
        } else {
            z0 = __ldg(nr::face_vertex_t<true>(p.src, zb, fn, 0) + 2);
            z1 = __ldg(nr::face_vertex_t<true>(p.src, zb, fn, 1) + 2);
            z2 = __ldg(nr::face_vertex_t<true>(p.src, zb, fn, 2) + 2);
        }
        const nr::TexCoord tc = nr::texture_coords(w, zp, z0, z1, z2, ts, p.tex.tex_cmp, p.tex.tex_val);
        float lam[3] = {0.0f, 0.0f, 0.0f}, L[3];  // kCorner / kPhong: perspective weights (own depths) and light of the pixel
        if constexpr (kCorner || kPhong) {  // l_k with the item's own depths (NR_TEX_Z_BATCH0 only moves the cube coordinates)
            float oz[3] = {z0, z1, z2};
            if (zb != b) {
#pragma unroll
                for (int k = 0; k < 3; k++) oz[k] = __ldg(nr::face_vertex(p.src, b, fn, k) + 2);
            }
            nr::perspective_weights(w, zp, oz[0], oz[1], oz[2], lam);
            nr::pixel_light<kLight>(p.shading, b, p.F, fn, lam, 0.0f, 0.0f, L);  // no uv: the cube modes have no map
        }
        // NR_TEX_FILL_BACK as nr::stored_face, written out: through the helper nvcc allocates this kernel's registers
        // differently (+8 instructions)
        int cube = fn, ncubes = p.F;
        bool rev = false;
        if (p.flags & NR_TEX_FILL_BACK) {
            ncubes = p.F >> 1;
            if (fn >= ncubes) { cube = fn - ncubes; rev = true; }
        }
        const size_t cube_off = p.tex.cube_off(b, cube, ts);
        if (want_light) {  // unlit sample (same blend as the forward pass) times the upstream gradient
            float r, g, bl;
            nr::cube_blend<false, true>(p.tex.tex + cube_off, tc, ts, rev, nullptr, r, g, bl);
            if constexpr (kCorner) {
                const float s3[3] = {r, g, bl};
                corner_light_grad(s3, g0, g1, g2, lam, glc);
            } else {
                gl0 = r * g0; gl1 = g * g1; gl2 = bl * g2;
            }
        }
        if constexpr (kCorner || kPhong) {  // d rgb / d texel = weight * interpolated light
            g0 *= L[0]; g1 *= L[1]; g2 *= L[2];
        } else if (p.shading.face_light) {  // d rgb / d texel = weight * light
            const float* lp = p.shading.face_light + p.shading.fl_off(b, p.F, fn);
            g0 *= __ldg(lp); g1 *= __ldg(lp + 1); g2 *= __ldg(lp + 2);
        }
        float* gt = p.grad_textures + cube_off;
        key = (((long long)(cube_off / 3) + nr::corner_index(tc, 0, ts)) << 1) | (rev ? 1 : 0);
        // The two corners that differ only along the fastest texture axis (axis 2; axis 0 of a reversed cube) are
        // neighbours in memory: 6 consecutive floats per corner pair.
#pragma unroll
        for (int pr = 0; pr < 4; pr++) {
            const int pn_lo = rev ? (pr << 1) : pr, pn_hi = rev ? (pn_lo | 1) : (pn_lo | 4);
            const float w_lo = nr::corner_weight(tc, pn_lo), w_hi = nr::corner_weight(tc, pn_hi);
            tp[pr] = gt + (rev ? nr::corner_index_rev(tc, pn_lo, ts) : nr::corner_index(tc, pn_lo, ts)) * 3;
            val[pr][0] = w_lo * g0; val[pr][1] = w_lo * g1; val[pr][2] = w_lo * g2;
            val[pr][3] = w_hi * g0; val[pr][4] = w_hi * g1; val[pr][5] = w_hi * g2;
        }
    }
    bool issue = fn >= 0;
    if (kTgCombine) {
        // runs of neighbouring lanes with the same key: after k steps lane l holds the sum over lanes l .. l + 2^k - 1 of
        // its run; every 2^kTgCombine-th lane of a run issues
        const long long key_prev = __shfl_up_sync(0xffffffffu, key, 1);
        const uint32_t heads = __ballot_sync(0xffffffffu, lane == 0 || key != key_prev);
        const uint32_t later = heads & ~((2u << lane) - 1u);
        const int run_end = (lane == 31 || later == 0) ? 31 : (__ffs(later) - 2);
        const int run_start = 31 - __clz(heads & ((2u << lane) - 1u));
        if (heads != 0xffffffffu) {  // warp-uniform: somebody has a neighbour to merge with
#pragma unroll
            for (int step = 0; step < kTgCombine; step++) {
                const int off = 1 << step;
                const bool take = lane + off <= run_end;
#pragma unroll
                for (int pr = 0; pr < 4; pr++)
#pragma unroll
                    for (int k = 0; k < 6; k++) {
                        const float t = __shfl_down_sync(0xffffffffu, val[pr][k], off);
                        if (take) val[pr][k] += t;
                    }
            }
            issue = issue && (((lane - run_start) & ((1 << kTgCombine) - 1)) == 0);
        }
    }
    if (issue) {
        // scattered with the widest vector reductions the alignment allows (red.global.add.v4/v2.f32, sm_90+): 2-4
        // requests per pair instead of 6
#pragma unroll
        for (int pr = 0; pr < 4; pr++) {
            float* t = tp[pr];
            const float v0 = val[pr][0], v1 = val[pr][1], v2 = val[pr][2], v3 = val[pr][3], v4 = val[pr][4], v5 = val[pr][5];
            switch ((reinterpret_cast<uintptr_t>(t) >> 2) & 3) {
                case 0: red_add_v4(t, v0, v1, v2, v3); red_add_v2(t + 4, v4, v5); break;
                case 2: red_add_v2(t, v0, v1); red_add_v4(t + 2, v2, v3, v4, v5); break;
                case 3: atomicAdd(t, v0); red_add_v4(t + 1, v1, v2, v3, v4); atomicAdd(t + 5, v5); break;
                // (padding the 4-byte-offset case to two aligned quads with +0 on either side -- 2 requests instead of 4
                // -- does not pay: the L2 pays per sector touched, not per request)
                default: atomicAdd(t, v0); red_add_v2(t + 1, v1, v2); red_add_v2(t + 3, v3, v4); atomicAdd(t + 5, v5); break;
            }
        }
    }
    if (!want_light) return;
    if constexpr (kCorner) {
        light_grad_scatter(glc, fn, lane, p.grad_corner_light, b, p.F);
        return;
    }
    // warp-aggregated scatter of the light gradient: runs of neighbouring lanes that show the same face
    const int fn_prev = __shfl_up_sync(0xffffffffu, fn, 1);
    const uint32_t heads = __ballot_sync(0xffffffffu, lane == 0 || fn != fn_prev);
    const uint32_t later = heads & ~((2u << lane) - 1u);
    const int run_end = (lane == 31 || later == 0) ? 31 : (__ffs(later) - 2);
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
        const bool take = lane + off <= run_end;
        const float t0 = __shfl_down_sync(0xffffffffu, gl0, off), t1 = __shfl_down_sync(0xffffffffu, gl1, off),
                    t2 = __shfl_down_sync(0xffffffffu, gl2, off);
        if (take) { gl0 += t0; gl1 += t1; gl2 += t2; }
    }
    if (fn >= 0 && ((heads >> lane) & 1u)) {
        float* gl = p.grad_face_light + ((size_t)b * p.F + fn) * 3;
        atomicAdd(gl, gl0); atomicAdd(gl + 1, gl1); atomicAdd(gl + 2, gl2);
    }
}

// ----------------------------------------------------------------------------------------------- k_image_grad
// NR_TEX_UV counterpart of K6, one thread per raster pixel in the same row-major map.  The pixel's uv and its four
// bilinear taps are recomputed from the saved weight / depth maps and the winner's own vertex depths with the forward's
// helpers (nr_math.cuh), and w_xy * light * grad_rgb goes to the taps: per tap row one horizontal pair = 6 consecutive
// floats, scattered with vector reductions by alignment as in K6.  A shared image receives from every item, so lanes
// next to each other that hit the same (image, cell) first merge their contributions (kTgCombine shuffle steps).
using nr::red_add_6;

// kMip (NR_TEX_MIPMAP): trilinear variant.  The pixel's level of detail is recomputed with the forward's nr::mip_lod from
// the K1 inverse of the same pixel-space vertices (face_inverse(to_pixel(...)), as k_depth_grad) and the saved weight /
// depth maps, so the taps and level weights are the forward's.  Up to four 6-float pairs (two rows on each of the two
// levels) go to the packed pyramid; lanes merge only when they hit the same cells on both levels.
//
// kUvGrad (grad_face_uvs given): the same pass also sends d loss / d face_uvs.  Per sampled level, nr::uv_blend_grad reads
// the four unlit taps once and returns d sample / d (u, v) per channel together with the unlit blend (which the light
// gradient then takes instead of reading the taps again); gu = sum_l a_l sum_c g_c light_c du_c (v alike, a_l = the level
// weight) goes to UV corner k as l_k (gu, gv), corners reversed back for a fill_back copy.  Runs of neighbouring lanes
// that show the same face sum their 6 floats with shuffles and the run's first lane adds them.
//
// kLight: as in k_texture_grad.  kCorner (kLightCorner): as in k_texture_grad, the interpolated light L_c replaces face_light (also in the face_uvs
// gradient) and the 9-float corner-light gradient goes through the run reduction.  kPhong: likewise with the Phong L_c.
template <int kTgCombine, bool kMip, bool kUvGrad, int kLight>
__device__ __forceinline__ void image_grad(const BwdParams& p) {
    constexpr bool kCorner = kLight == nr::kLightCorner, kPhong = kLight >= nr::kLightPhong;
    constexpr int kPairs = kMip ? 4 : 2;
    const int S = p.S;
    const size_t plane = (size_t)S * S;
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;  // pixel within the image (image orientation)
    const int b = blockIdx.y;
    const int lane = threadIdx.x & 31;
    const int fn = (i < plane) ? __ldg(p.fim + (size_t)b * plane + i) : -1;
    const bool want_light = !kPhong && (kCorner ? p.grad_corner_light : p.grad_face_light) != nullptr;  // uniform
    if (!want_light && !__any_sync(0xffffffffu, fn >= 0)) return;  // warp-uniform
    float gl0 = 0.0f, gl1 = 0.0f, gl2 = 0.0f;  // d loss / d face_light of this pixel
    float glc[kCorner ? 9 : 1];                // kCorner: d loss / d corner_light of this pixel
#pragma unroll
    for (int k = 0; k < (kCorner ? 9 : 1); k++) glc[k] = 0.0f;
    float val[kPairs][6];                      // tap row 0 / 1 (of level l0, then l1): taps (x0, x1) x 3 channels
    float* tp[kPairs];
    bool adjacent[kPairs / 2];                 // x1 == x0 + 1 (else both taps of a row are the same texel, weight 0 on x1)
    long long key = -1 - (long long)lane;      // (image, cell): equal keys <=> the same four texels
    long long key1 = -1;                       // kMip: the cell on level l1 (-1 when f == 0)
    float uvg[6] = {0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f};  // kUvGrad: d loss / d face_uvs, corners of the stored face
    uint32_t uv_at = 0;                        // kUvGrad: offset of the face's corners in face_uvs / grad_face_uvs
#pragma unroll
    for (int r = 0; r < kPairs; r++) {
        tp[r] = nullptr;
#pragma unroll
        for (int k = 0; k < 6; k++) val[r][k] = 0.0f;
    }
#pragma unroll
    for (int r = 0; r < kPairs / 2; r++) adjacent[r] = true;
    if (fn >= 0) {
        const int row = (int)(i / S), col = (int)(i % S);
        const bool aa = (p.flags & NR_ANTI_ALIASING) != 0;
        float g0 = load_grad(p.g_rgb, aa, S, (size_t)b * 3 + 0, row, col);
        float g1 = load_grad(p.g_rgb, aa, S, (size_t)b * 3 + 1, row, col);
        float g2 = load_grad(p.g_rgb, aa, S, (size_t)b * 3 + 2, row, col);
        const float* wm = p.wmap + (size_t)b * 3 * plane + i;
        const float w[3] = {__ldg(wm), __ldg(wm + plane), __ldg(wm + 2 * plane)};
        const float zp = __ldg(p.dmap + (size_t)b * plane + i);
        float z0, z1, z2;  // the item's own vertex depths, as in the forward sampler
        float inv[9];
        if constexpr (kMip) {
            float c[9];
            nr::load_face(p.src, b, fn, c);
            const float fS = (float)S;
            nr::face_inverse(nr::to_pixel(c[0], fS), nr::to_pixel(c[1], fS), nr::to_pixel(c[3], fS), nr::to_pixel(c[4], fS),
                             nr::to_pixel(c[6], fS), nr::to_pixel(c[7], fS), inv);
            z0 = c[2]; z1 = c[5]; z2 = c[8];
        } else if (p.src.idx == nullptr) {
            const float* v = p.src.faces + ((size_t)b * p.F + fn) * 9;
            z0 = __ldg(v + 2); z1 = __ldg(v + 5); z2 = __ldg(v + 8);
        } else {
            z0 = __ldg(nr::face_vertex_t<true>(p.src, b, fn, 0) + 2);
            z1 = __ldg(nr::face_vertex_t<true>(p.src, b, fn, 1) + 2);
            z2 = __ldg(nr::face_vertex_t<true>(p.src, b, fn, 2) + 2);
        }
        bool rev;
        const int uf = nr::stored_face(p.flags & NR_TEX_FILL_BACK, p.F, fn, rev);
        float uv[6], u, v;
        nr::face_uvs(p.tex, b, uf, rev, uv);
        nr::pixel_uv(w, zp, z0, z1, z2, uv, u, v);
        float lam[3] = {0.0f, 0.0f, 0.0f}, L[3];  // kCorner / kPhong: perspective weights and light of the pixel
        if constexpr (kCorner || kPhong) {
            nr::perspective_weights(w, zp, z0, z1, z2, lam);
            nr::pixel_light<kLight>(p.shading, b, p.F, fn, lam, u, v, L);
        }
        const uint32_t img_off = p.tex.img_off(b);
        const nr::LevelPair lp = nr::level_pair<kMip>(p.tex, inv, w, zp, z0, z1, z2, uv);
        const nr::UvTaps t0 = nr::uv_taps(u, v, p.tex.level_h<kMip>(lp.l[0]), p.tex.level_w<kMip>(lp.l[0]));
        if constexpr (kUvGrad) {
            float lt[3] = {1.0f, 1.0f, 1.0f};
            if constexpr (kCorner || kPhong) {
                lt[0] = L[0]; lt[1] = L[1]; lt[2] = L[2];
            } else if (p.shading.face_light) {
                const float* lp = p.shading.face_light + p.shading.fl_off(b, p.F, fn);
                lt[0] = __ldg(lp); lt[1] = __ldg(lp + 1); lt[2] = __ldg(lp + 2);
            }
            const float h[3] = {g0 * lt[0], g1 * lt[1], g2 * lt[2]};  // d loss / d unlit tap value, per unit weight
            float c[3], gu, gv;
            nr::image_sample_grad<kMip>(p.tex, p.tex.tex + img_off, lp, t0, u, v, h, c, gu, gv);
            if constexpr (kCorner) {
                if (want_light) corner_light_grad(c, g0, g1, g2, lam, glc);
            } else {
                if (want_light) { gl0 = c[0] * g0; gl1 = c[1] * g1; gl2 = c[2] * g2; }
            }
            // uv = sum_k l_k uv_k (pixel_uv); a fill_back copy's corner k is corner 2 - k of the stored face
            const float l0 = __fmul_rn(w[0], __fdiv_rn(zp, z0)), l1 = __fmul_rn(w[1], __fdiv_rn(zp, z1)),
                        l2 = __fmul_rn(w[2], __fdiv_rn(zp, z2));
            const float s0 = rev ? l2 : l0, s2 = rev ? l0 : l2;  // l of the stored face's corners 0 and 2
            uvg[0] = __fmul_rn(s0, gu); uvg[1] = __fmul_rn(s0, gv);
            uvg[2] = __fmul_rn(l1, gu); uvg[3] = __fmul_rn(l1, gv);
            uvg[4] = __fmul_rn(s2, gu); uvg[5] = __fmul_rn(s2, gv);
            uv_at = p.tex.uv_off(b, uf);
        }
        if (!kUvGrad && want_light) {  // unlit sample (same blend as the forward pass) times the upstream gradient
            float c[3];
            if constexpr (kMip) {
                nr::MipLevels m;
                m.l0 = lp.l[0]; m.l1 = lp.l[1]; m.f = lp.a[1];
                nr::mip_blend<false>(p.tex.tex + img_off, p.tex.mip, m, u, v, 1.0f, 1.0f, 1.0f, c);
            } else {
                nr::uv_blend<false>(p.tex.tex + img_off, p.tex.Wt, t0, 1.0f, 1.0f, 1.0f, c);
            }
            if constexpr (kCorner) corner_light_grad(c, g0, g1, g2, lam, glc);
            else { gl0 = c[0] * g0; gl1 = c[1] * g1; gl2 = c[2] * g2; }
        }
        if constexpr (kCorner || kPhong) {  // d rgb / d texel = weight * interpolated light
            g0 *= L[0]; g1 *= L[1]; g2 *= L[2];
        } else if (p.shading.face_light) {  // d rgb / d texel = weight * light
            const float* lp = p.shading.face_light + p.shading.fl_off(b, p.F, fn);
            g0 *= __ldg(lp); g1 *= __ldg(lp + 1); g2 *= __ldg(lp + 2);
        }
        float* gi = p.grad_textures + img_off;
#pragma unroll
        for (int q = 0; q < kPairs / 2; q++) {
            if (q >= lp.n) break;
            const int Hl = p.tex.level_h<kMip>(lp.l[q]), Wl = p.tex.level_w<kMip>(lp.l[q]);
            const uint32_t loff = p.tex.level_off<kMip>(lp.l[q]);
            const nr::UvTaps t = q == 0 ? t0 : nr::uv_taps(u, v, Hl, Wl);
            const uint32_t row3 = (uint32_t)Wl * 3u;
            tp[2 * q] = gi + loff + (uint32_t)t.r0 * row3 + (uint32_t)t.x0 * 3u;
            tp[2 * q + 1] = gi + loff + (uint32_t)t.r1 * row3 + (uint32_t)t.x0 * 3u;
            adjacent[q] = t.x1 != t.x0;
            const long long k = (long long)((img_off + loff) / 3u) + t.cell;
            if (q == 0) key = k; else key1 = k;
            const float h0 = kMip ? __fmul_rn(lp.a[q], g0) : g0, h1 = kMip ? __fmul_rn(lp.a[q], g1) : g1,
                        h2 = kMip ? __fmul_rn(lp.a[q], g2) : g2;
            float* v0 = val[2 * q];
            float* v1 = val[2 * q + 1];
            v0[0] = t.w00 * h0; v0[1] = t.w00 * h1; v0[2] = t.w00 * h2;
            v0[3] = t.w10 * h0; v0[4] = t.w10 * h1; v0[5] = t.w10 * h2;
            v1[0] = t.w01 * h0; v1[1] = t.w01 * h1; v1[2] = t.w01 * h2;
            v1[3] = t.w11 * h0; v1[4] = t.w11 * h1; v1[5] = t.w11 * h2;
        }
    }
    bool issue = fn >= 0;
    if (kTgCombine) {
        // runs of neighbouring lanes with the same key (segmented shuffle of k_texture_grad)
        const long long key_prev = __shfl_up_sync(0xffffffffu, key, 1);
        bool differs = key != key_prev;
        if constexpr (kMip) {
            const long long key1_prev = __shfl_up_sync(0xffffffffu, key1, 1);  // every lane takes part in the shuffle
            differs = differs || key1 != key1_prev;
        }
        const uint32_t heads = __ballot_sync(0xffffffffu, lane == 0 || differs);
        const uint32_t later = heads & ~((2u << lane) - 1u);
        const int run_end = (lane == 31 || later == 0) ? 31 : (__ffs(later) - 2);
        const int run_start = 31 - __clz(heads & ((2u << lane) - 1u));
        if (heads != 0xffffffffu) {  // warp-uniform: somebody has a neighbour to merge with
#pragma unroll
            for (int step = 0; step < kTgCombine; step++) {
                const int off = 1 << step;
                const bool take = lane + off <= run_end;
#pragma unroll
                for (int r = 0; r < kPairs; r++)
#pragma unroll
                    for (int k = 0; k < 6; k++) {
                        const float x = __shfl_down_sync(0xffffffffu, val[r][k], off);
                        if (take) val[r][k] += x;
                    }
            }
            issue = issue && (((lane - run_start) & ((1 << kTgCombine) - 1)) == 0);
        }
    }
    if (issue) {
#pragma unroll
        for (int r = 0; r < kPairs; r++) {
            if (kMip && tp[r] == nullptr) break;  // level l1 has no taps when f == 0
            if (adjacent[r >> 1]) {
                red_add_6(tp[r], val[r]);
            } else {
                float* q = tp[r];
                atomicAdd(q, val[r][0] + val[r][3]); atomicAdd(q + 1, val[r][1] + val[r][4]); atomicAdd(q + 2, val[r][2] + val[r][5]);
            }
        }
    }
    if constexpr (kUvGrad) {
        // warp-aggregated scatter of d loss / d face_uvs: runs of neighbouring lanes that show the same face (the same fn
        // is the same UV face with the same corner order)
        const int fn_prev = __shfl_up_sync(0xffffffffu, fn, 1);
        const uint32_t heads = __ballot_sync(0xffffffffu, lane == 0 || fn != fn_prev);
        const uint32_t later = heads & ~((2u << lane) - 1u);
        const int run_end = (lane == 31 || later == 0) ? 31 : (__ffs(later) - 2);
#pragma unroll
        for (int off = 1; off < 32; off <<= 1) {
            const bool take = lane + off <= run_end;
#pragma unroll
            for (int k = 0; k < 6; k++) {
                const float x = __shfl_down_sync(0xffffffffu, uvg[k], off);
                if (take) uvg[k] += x;
            }
        }
        if (fn >= 0 && ((heads >> lane) & 1u)) red_add_6(p.grad_uvs + uv_at, uvg);
    }
    if (!want_light) return;
    if constexpr (kCorner) {
        light_grad_scatter(glc, fn, lane, p.grad_corner_light, b, p.F);
        return;
    }
    // warp-aggregated scatter of the light gradient: runs of neighbouring lanes that show the same face
    const int fn_prev = __shfl_up_sync(0xffffffffu, fn, 1);
    const uint32_t heads = __ballot_sync(0xffffffffu, lane == 0 || fn != fn_prev);
    const uint32_t later = heads & ~((2u << lane) - 1u);
    const int run_end = (lane == 31 || later == 0) ? 31 : (__ffs(later) - 2);
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
        const bool take = lane + off <= run_end;
        const float t0 = __shfl_down_sync(0xffffffffu, gl0, off), t1 = __shfl_down_sync(0xffffffffu, gl1, off),
                    t2 = __shfl_down_sync(0xffffffffu, gl2, off);
        if (take) { gl0 += t0; gl1 += t1; gl2 += t2; }
    }
    if (fn >= 0 && ((heads >> lane) & 1u)) {
        float* gl = p.grad_face_light + ((size_t)b * p.F + fn) * 3;
        atomicAdd(gl, gl0); atomicAdd(gl + 1, gl1); atomicAdd(gl + 2, gl2);
    }
}

template <int kTgCombine, bool kUvGrad, int kLight>
__global__ void __launch_bounds__(256, kUvGrad ? NR_IGU_MIN_CTAS : NR_IG_MIN_CTAS) k_image_grad(const __grid_constant__ BwdParams p) {
    image_grad<kTgCombine, false, kUvGrad, kLight>(p);
}
template <int kTgCombine, bool kUvGrad, int kLight>
__global__ void __launch_bounds__(256, kUvGrad ? NR_IGMU_MIN_CTAS : NR_IGM_MIN_CTAS) k_image_grad_mip(const __grid_constant__ BwdParams p) {
    image_grad<kTgCombine, true, kUvGrad, kLight>(p);
}

// ----------------------------------------------------------------------------------------------- k_depth_grad
__global__ void __launch_bounds__(256) k_depth_grad(const __grid_constant__ BwdParams p) {
    const int S = p.S;
    const size_t plane = (size_t)S * S;
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int b = blockIdx.y;
    const int lane = threadIdx.x & 31;
    const int fn = (i < plane) ? __ldg(p.fim + (size_t)b * plane + i) : -1;
    float out[9];
#pragma unroll
    for (int k = 0; k < 9; k++) out[k] = 0.0f;
    if (fn >= 0) {
        const int row = (int)(i / S), col = (int)(i % S);
        const bool aa = (p.flags & NR_ANTI_ALIASING) != 0;
        const float g = load_grad(p.g_depth, aa, S, (size_t)b, row, col);
        float c[9];
        nr::load_face(p.src, b, fn, c);
        const float fS = (float)S;
        float inv[9];
        nr::face_inverse(nr::to_pixel(c[0], fS), nr::to_pixel(c[1], fS), nr::to_pixel(c[3], fS), nr::to_pixel(c[4], fS),
                         nr::to_pixel(c[6], fS), nr::to_pixel(c[7], fS), inv);
        const float* wm = p.wmap + (size_t)b * 3 * plane + i;
        const float w[3] = {__ldg(wm), __ldg(wm + plane), __ldg(wm + 2 * plane)};
        const float depth = __ldg(p.dmap + (size_t)b * plane + i);
        const float depth2 = depth * depth;
        const float z[3] = {c[2], c[5], c[8]};
        // rasterize.py:824-827  d zp / d z_k = w_k * zp^2 / z_k^2
#pragma unroll
        for (int k = 0; k < 3; k++) out[3 * k + 2] = __fdiv_rn((g * w[k]) * depth2, z[k] * z[k]);
        // rasterize.py:830-837  tmp_l = -sum_v inv[v][l] / z_v ;  d zp / d (x,y)_k = -g * tmp_l * w_k * zp^2 * is / 2
        float tmp[2];
#pragma unroll
        for (int l = 0; l < 2; l++)
            tmp[l] = ((0.0f - __fdiv_rn(inv[l], z[0])) - __fdiv_rn(inv[3 + l], z[1])) - __fdiv_rn(inv[6 + l], z[2]);
#pragma unroll
        for (int k = 0; k < 3; k++)
#pragma unroll
            for (int l = 0; l < 2; l++) out[3 * k + l] = (((((-g) * tmp[l]) * w[k]) * depth2) * fS) * 0.5f;
    }
    // Warp-aggregated scatter: a warp holds 32 consecutive pixels of a row, where a (convex) face shows as a run of
    // neighbouring lanes.  Each run is summed with a segmented shuffle reduction and its first lane issues the nine
    // atomics (the reference issues them per pixel, rasterize.py:826-837; fp32 atomics are unordered there too).
    const int fn_prev = __shfl_up_sync(0xffffffffu, fn, 1);
    const uint32_t heads = __ballot_sync(0xffffffffu, lane == 0 || fn != fn_prev);
    const uint32_t later = heads & ~((2u << lane) - 1u);  // run heads after this lane (2u << 31 wraps to 0: mask = all)
    const int run_end = (lane == 31 || later == 0) ? 31 : (__ffs(later) - 2);
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
        const bool take = lane + off <= run_end;
#pragma unroll
        for (int k = 0; k < 9; k++) {
            const float t = __shfl_down_sync(0xffffffffu, out[k], off);
            if (take) out[k] += t;
        }
    }
    if (fn >= 0 && ((heads >> lane) & 1u)) {
#pragma unroll
        for (int k = 0; k < 3; k++) {
            float* gf = nr::face_grad_vertex(p.dst, b, fn, k);
            if (gf) { atomicAdd(gf, out[3 * k]); atomicAdd(gf + 1, out[3 * k + 1]); atomicAdd(gf + 2, out[3 * k + 2]); }
        }
    }
}

template <int kMode, int kT, bool kIdx, bool kCol>
int launch_edge_scan_c(const BwdParams& p, int nstrips, size_t smem, cudaStream_t stream) {
    static nr_internal::SmemOptIn optin;
    if (optin.ensure(k_edge_scan<kMode, kT, kIdx, kCol>, smem) != cudaSuccess) return NR_ERR_CUDA;
    nr_internal::LaunchScope ls("k_edge_scan", stream);
    k_edge_scan<kMode, kT, kIdx, kCol><<<dim3(nstrips, 2, p.B), kT, smem, stream>>>(p);
    return NR_OK;
}
template <int kMode, int kT, bool kIdx>
int launch_edge_scan_i(const BwdParams& p, int nstrips, size_t smem, cudaStream_t stream) {
    return p.col_smem ? launch_edge_scan_c<kMode, kT, kIdx, true>(p, nstrips, smem, stream)
                      : launch_edge_scan_c<kMode, kT, kIdx, false>(p, nstrips, smem, stream);
}
template <int kMode, int kT>
int launch_edge_scan_t(const BwdParams& p, int nstrips, size_t smem, cudaStream_t stream) {
    return p.src.idx ? launch_edge_scan_i<kMode, kT, true>(p, nstrips, smem, stream)
                     : launch_edge_scan_i<kMode, kT, false>(p, nstrips, smem, stream);
}

template <int kMode>
int launch_edge_scan(const BwdParams& p, int nstrips, size_t smem, cudaStream_t stream) {
    int threads = kEdgeScanThreadsDefault;
#ifdef NR_B200_TUNING
    if (const char* env = getenv("NR_B200_ES_THREADS")) threads = atoi(env);
#endif
#ifdef NR_B200_TUNING
    if (threads == 256) return launch_edge_scan_t<kMode, 256>(p, nstrips, smem, stream);
#endif
    (void)threads;
    return launch_edge_scan_t<kMode, 128>(p, nstrips, smem, stream);
}

}  // namespace

void nr_internal::strip_scan(const int* cnt, int* off, int seg_len, long long seg_stride, int nseg, cudaStream_t stream) {
    nr_internal::LaunchScope ls("k_strip_scan", stream);
    k_strip_scan<<<nseg, 256, 0, stream>>>(cnt, off, seg_len, seg_stride);
}

namespace {
struct BinLayout {
    int W, w_log2, nstrips;
    size_t ncounters, off_cnt, off_off, off_cursor, off_list, total;
};
// strip width from the shared-memory budget; workspace = boxes | counters | offsets | cursors | lists
// Shared-memory bytes per staged pixel: pairs P, Q (16) [+ R (4)] plus either {colours, face index} (16) or, above
// kColSmemMaxS, the face index alone (4) -- see k_edge_scan.  [raster 512, 70 k faces, batch 32: 3.19 -> see DESIGN.md]
#ifndef NR_COL_SMEM_MAX_S
#define NR_COL_SMEM_MAX_S 256
#endif
constexpr int kColSmemMaxS = NR_COL_SMEM_MAX_S;
inline bool strip_keeps_colours(int S) { return S <= kColSmemMaxS; }
inline int strip_rec_bytes(int S, bool rgb_and_alpha) { return (strip_keeps_colours(S) ? 32 : 20) + (rgb_and_alpha ? 4 : 0); }

BinLayout bin_layout(int B, int F, int S, int rec_bytes) {
    BinLayout L{};
    size_t strip_bytes = kStripBytesDefault;
    bool strip_forced = false;
#ifdef NR_B200_TUNING
    if (const char* env = getenv("NR_B200_STRIP_KB")) { strip_bytes = (size_t)atoi(env) * 1024; strip_forced = true; }
#endif
    int W = kMaxLines;
    while (W > 1 && (size_t)W * ((S + 1) & ~1) * rec_bytes > strip_bytes) W >>= 1;
    // one-line strips pay the per-CTA front end (staging, face list, task sort) per line: two lines are worth twice
    // the shared memory up to 32 KB; beyond that the lost occupancy costs more
    if (W == 1 && !strip_forced && (size_t)2 * ((S + 1) & ~1) * rec_bytes <= 2 * (size_t)kStripBytesDefault) W = 2;
    L.W = W;
    L.w_log2 = 0;
    while ((1 << L.w_log2) < W) L.w_log2++;
    L.nstrips = (S + W - 1) / W;
    L.ncounters = (size_t)B * 2 * (L.nstrips + 1);
    L.off_cnt = bbox_workspace_bytes(B, F);
    L.off_off = L.off_cnt + nr_align_up(L.ncounters * sizeof(int), 256);
    L.off_cursor = L.off_off + nr_align_up(L.ncounters * sizeof(int), 256);
    L.off_list = L.off_cursor + nr_align_up(L.ncounters * sizeof(int), 256);
    L.total = L.off_list + nr_align_up((size_t)B * F * 2 * kWideStrips * sizeof(int), 256);
    return L;
}
}  // namespace

extern "C" size_t nr_b200_backward_workspace_bytes(int32_t B, int32_t F, int32_t S, int32_t ts, uint32_t flags) {
    (void)ts;
    if (B <= 0 || F <= 0 || S <= 0) return 16;
    const bool both = (flags & NR_RETURN_RGB) && (flags & NR_RETURN_ALPHA);
    return bin_layout(B, F, S, strip_rec_bytes(S, both)).total;
}

// nr_b200_backward (no corner_light, no Phong inputs), nr_b200_backward_corner_light (smooth shading) and the five Phong
// entry points
static int backward_impl(const nr_b200_backward_args* args, const float* corner_light, float* grad_corner_light,
                         const nr_internal::PhongCall& pc, void* cuda_stream) {
    nr_internal::launch_count() = 0;
    // Two layouts: the full struct, and the ABI-4 struct from before grad_face_uvs (which then reads as NULL).  Only the
    // caller's struct_size bytes are read.
    if (!args) return NR_ERR_INVALID_ARG;
    const uint32_t size = args->struct_size;
    if (size != sizeof(nr_b200_backward_args) && size != offsetof(nr_b200_backward_args, grad_face_uvs)) return NR_ERR_INVALID_ARG;
    nr_b200_backward_args args_copy;
    memset(&args_copy, 0, sizeof(args_copy));
    memcpy(&args_copy, args, size);
    const nr_b200_backward_args* a = &args_copy;
    const int B = a->batch_size, F = a->num_faces, S = a->raster_size, ts = a->texture_size;
    const uint32_t flags = a->flags;
    if (B <= 0 || F <= 0 || S <= 0) return NR_ERR_INVALID_ARG;
    if (!a->face_index_map || !a->weight_map || !a->depth_map) return NR_ERR_INVALID_ARG;
    // the two halves of the pass can be issued separately (NR_BWD_PART_*): textures first lets the caller start a
    // collective on grad_textures while the edge scan runs
    const bool part_tex = !(flags & NR_BWD_PART_FACES) || (flags & NR_BWD_PART_TEXTURES);
    const bool part_faces = !(flags & NR_BWD_PART_TEXTURES) || (flags & NR_BWD_PART_FACES);
    nr::FaceSrc src{};
    nr::FaceGrad dst{};
    if (!nr_internal::make_face_src(flags, a->faces, a->vertices, a->face_indices, F, a->num_vertices, &src)) return NR_ERR_INVALID_ARG;
    if (part_faces && !nr_internal::make_face_grad(flags, a->grad_faces, a->grad_vertices, a->face_indices, F, a->num_vertices, &dst))
        return NR_ERR_INVALID_ARG;
    const bool rgb = (flags & NR_RETURN_RGB) != 0, alpha = (flags & NR_RETURN_ALPHA) != 0, depth = (flags & NR_RETURN_DEPTH) != 0;
    const bool uv = (flags & NR_TEX_UV) != 0, mip = (flags & NR_TEX_MIPMAP) != 0;
    nr::Texture tex;
    size_t tex_floats, uv_floats;  // of grad_textures and grad_face_uvs
    const int tex_rc = nr_internal::make_texture(a, &tex, &tex_floats, &uv_floats);
    if (tex_rc == NR_ERR_INVALID_ARG) return tex_rc;
    // d loss / d face_uvs: only for the texture-image sampler, and it reads the image (pyramid).  It has the layout of
    // face_uvs, so make_texture's 32-bit UV offset check covers it.
    const bool uv_grad = a->grad_face_uvs != nullptr;
    if (uv_grad && (!uv || !rgb || !a->textures)) return NR_ERR_INVALID_ARG;
    if (rgb && !a->rgb_map) return NR_ERR_INVALID_ARG;
    if (rgb && part_tex && !a->grad_textures) return NR_ERR_INVALID_ARG;
    if (rgb && a->grad_face_light && !a->textures) return NR_ERR_INVALID_ARG;
    nr::Shading shading;
    const int light = nr_internal::make_shading(rgb, a->face_light, corner_light, pc, B, F, &shading);
    if (light < 0) return NR_ERR_INVALID_ARG;
    const nr_b200_phong_args* phong = pc.phong;
    const nr_b200_normal_map_args* nm = pc.nm;
    const nr_b200_specular_map_args* sm = pc.sm;
    if ((nm || sm) && !uv) return NR_ERR_INVALID_ARG;  // the maps are addressed by the pixel's uv
    // The Phong gradient outputs in ABI order, with their float counts.  A set of NL = 0 lights has a grad_lights of 0
    // floats: it needs the textures like every other, and is never written.
    const struct { float* ptr; size_t floats; } phong_out[] = {
        {phong ? phong->grad_corner_shading : nullptr, phong ? (size_t)phong->shading_batch * F * 18 : 0},
        {phong ? phong->grad_params : nullptr, phong ? (size_t)phong->params_batch * 16 : 0},
        {pc.lights ? pc.lights->grad_lights : nullptr, pc.lights ? (size_t)pc.lights->lights_batch * shading.NL * 12 : 0},
        {pc.sh ? pc.sh->grad_sh : nullptr, pc.sh ? (size_t)pc.sh->sh_batch * 27 : 0},
        {nm ? nm->grad_normal_map : nullptr, nm ? (size_t)nm->map_batch * nr_internal::nm_floats(nm) : 0},
        {nm ? nm->grad_corner_tangents : nullptr, nm ? (size_t)nm->tangent_batch * F * 12 : 0},
        {sm ? sm->grad_specular_map : nullptr, sm ? (size_t)sm->map_batch * nr_internal::sm_floats(sm) : 0},
    };
    // the shading gradients: grad_corner_light needs corner_light, and every one reads the (unlit) textures
    if (grad_corner_light && !corner_light) return NR_ERR_INVALID_ARG;
    // a normal or specular map also sends its own term into grad_face_uvs from the Phong-gradient kernel
    bool any_phong_out = false, phong_grads = (nm || sm) && uv_grad;
    for (const auto& o : phong_out) {
        any_phong_out |= o.ptr != nullptr;
        phong_grads |= o.ptr && o.floats;
    }
    if (!a->textures && (grad_corner_light || any_phong_out)) return NR_ERR_INVALID_ARG;
    // NR_GRAD_INTERIOR: the sampler's derivative reads the textures; the cubes of NR_TEX_Z_BATCH0 sample item b with the
    // depths of item 0, so their derivative would cross items (B = 1 is the plain sampler)
    const bool interior = (flags & NR_GRAD_INTERIOR) != 0;
    if (interior && phong) return NR_ERR_UNSUPPORTED;  // no vertex gradient through l_k of the Phong normal and position
    if (interior && (!rgb || !a->textures)) return NR_ERR_INVALID_ARG;
    if (interior && !uv && (flags & NR_TEX_Z_BATCH0) && B > 1) return NR_ERR_INVALID_ARG;
    if ((flags & NR_ANTI_ALIASING) && (S & 1)) return NR_ERR_INVALID_ARG;
    if (S > 32767 || B > 65535) return NR_ERR_UNSUPPORTED;
    if ((size_t)B * F * 2 * kWideStrips >= (size_t)0x7FFFFFFF) return NR_ERR_UNSUPPORTED;  // 32-bit list offsets
    if (tex_rc != NR_OK) return tex_rc;  // 32-bit image / UV offsets
    if (nm && nr_internal::nm_floats(nm) * (size_t)nm->map_batch > 0x7FFFFFFFull) return NR_ERR_UNSUPPORTED;  // 32-bit map offsets
    if (sm && nr_internal::sm_floats(sm) * (size_t)sm->map_batch > 0x7FFFFFFFull) return NR_ERR_UNSUPPORTED;
    const size_t need = nr_b200_backward_workspace_bytes(B, F, S, ts, flags);
    if (!a->workspace || a->workspace_bytes < need || ((uintptr_t)a->workspace & 15)) return NR_ERR_WORKSPACE;
    cudaStream_t stream = (cudaStream_t)cuda_stream;

    // When one call runs both halves, grad_textures is zero-filled by the CTAs of the edge scan (a side job of an
    // issue-bound kernel instead of a memset of its own) and K6 runs after the edge scan.  Separate halves (the caller wants
    // the texture gradient first, for a collective) and unaligned buffers keep the memset.
    const bool scan_will_run = part_faces && ((rgb && a->grad_rgb) || (alpha && a->grad_alpha));
    bool fill_in_scan = !(flags & NR_GRAD_ACCUMULATE) && part_tex && part_faces && rgb && a->grad_rgb && scan_will_run &&
                        (((uintptr_t)a->grad_textures & 15) == 0);
#ifdef NR_NO_FILL_IN_SCAN
    fill_in_scan = false;
#endif
    if (!(flags & NR_GRAD_ACCUMULATE)) {
        nr_internal::prof_begin("memset_grads", stream);
        if (part_faces) {
            const cudaError_t e = (flags & NR_FACES_INDEXED)
                ? cudaMemsetAsync(a->grad_vertices, 0, (size_t)B * a->num_vertices * 3 * sizeof(float), stream)
                : cudaMemsetAsync(a->grad_faces, 0, (size_t)B * F * 9 * sizeof(float), stream);
            if (e != cudaSuccess) return NR_ERR_CUDA;
        }
        if (part_tex && rgb && !fill_in_scan && cudaMemsetAsync(a->grad_textures, 0, tex_floats * sizeof(float), stream) != cudaSuccess)
            return NR_ERR_CUDA;
        if (part_tex && rgb && a->grad_face_light && cudaMemsetAsync(a->grad_face_light, 0, (size_t)B * F * 3 * sizeof(float), stream) != cudaSuccess)
            return NR_ERR_CUDA;
        if (part_tex && uv_grad && cudaMemsetAsync(a->grad_face_uvs, 0, uv_floats * sizeof(float), stream) != cudaSuccess)
            return NR_ERR_CUDA;
        if (part_tex && grad_corner_light &&
            cudaMemsetAsync(grad_corner_light, 0, (size_t)B * F * 9 * sizeof(float), stream) != cudaSuccess)
            return NR_ERR_CUDA;
        for (const auto& o : phong_out)
            if (part_tex && o.ptr && o.floats && cudaMemsetAsync(o.ptr, 0, o.floats * sizeof(float), stream) != cudaSuccess)
                return NR_ERR_CUDA;
        nr_internal::prof_end(stream);
    }

    BwdParams p{};
    p.src = src; p.dst = dst;
    p.tex = tex;
    p.fim = a->face_index_map; p.wmap = a->weight_map; p.dmap = a->depth_map; p.rgb = a->rgb_map;
    p.g_rgb = rgb ? a->grad_rgb : nullptr; p.g_alpha = alpha ? a->grad_alpha : nullptr; p.g_depth = depth ? a->grad_depth : nullptr;
    p.grad_textures = a->grad_textures;
    p.grad_face_light = rgb ? a->grad_face_light : nullptr;
    p.B = B; p.F = F; p.S = S; p.ts = ts;
    p.flags = flags;
    p.eps = (float)a->eps;
    p.two_over_S = 2.0f / (float)S;
    if (uv) p.grad_uvs = a->grad_face_uvs;
    p.grad_corner_light = grad_corner_light;
    p.shading = shading;
    const dim3 pgrid((unsigned)(((size_t)S * S + 255) / 256), B);
    auto launch_texture_grad = [&]() {
        nr_internal::LaunchScope ls(uv ? "k_image_grad" : "k_texture_grad", stream);
        // face_light is the kLightNone variant's run-time branch; L_c of a specular-map render is that of the same call
        // without the map
        const int tg_light = light == nr::kLightFace ? nr::kLightNone
                           : light != nr::kLightPhongSM ? light
                           : nm ? nr::kLightPhongNM : pc.sh ? nr::kLightPhongSH : shading.NL > 0 ? nr::kLightPhongSet : nr::kLightPhong;
        nr::dispatch_light<nr::kLightNone, nr::kLightCorner, nr::kLightPhong, nr::kLightPhongSet, nr::kLightPhongSH,
                           nr::kLightPhongNM>(tg_light, [&](auto kL) {
            if constexpr (kL != nr::kLightPhongNM) {  // a normal map needs NR_TEX_UV
                if (!uv) {
                    k_texture_grad<NR_TG_COMBINE, kL><<<pgrid, 256, 0, stream>>>(p);
                    return;
                }
            }
            nr::dispatch_bool(uv_grad, [&](auto kUvGrad) {
                if (mip) k_image_grad_mip<NR_TG_COMBINE, kUvGrad, kL><<<pgrid, 256, 0, stream>>>(p);
                else k_image_grad<NR_TG_COMBINE, kUvGrad, kL><<<pgrid, 256, 0, stream>>>(p);
            });
        });
    };
    // Phong: d loss / d corner_shading, params, lights, sh and the maps per pixel (nr_phong.cu), part of the texture half
    auto launch_phong_grad = [&]() {
        if (!phong_grads) return;
        auto written = [&](int k) { return phong_out[k].floats ? phong_out[k].ptr : nullptr; };
        nr_internal::PhongGradLaunch pl{};
        pl.args = a; pl.src = src; pl.shading = shading; pl.tex = tex;
        pl.grad = {written(0), written(1), written(2), written(3), written(4), written(5), written(6),
                   (nm || sm) ? a->grad_face_uvs : nullptr};
        nr_internal::launch_phong_grad(pl, stream);
    };
    // K6 first, unless its output buffer is zero-filled by the edge scan
    if (part_tex && rgb && p.g_rgb && !fill_in_scan) launch_texture_grad();
    if (part_tex && rgb && p.g_rgb) launch_phong_grad();
    if (!part_faces) return cudaGetLastError() == cudaSuccess ? NR_OK : NR_ERR_CUDA;

    // K5 runs when an rgb or alpha gradient exists (rasterize.py:523); without upstream gradients it contributes 0
    const bool need_scan = (rgb && p.g_rgb) || (alpha && p.g_alpha);
    if (need_scan) {
        uint2* bbox = (uint2*)a->workspace;
        uint2* cbox = (uint2*)((char*)a->workspace + nr_align_up((size_t)B * F * sizeof(uint2), 256));
        const bool use_rgb = rgb && p.g_rgb, use_alpha = alpha && p.g_alpha;
        const int rec_bytes = strip_rec_bytes(S, use_rgb && use_alpha);
        const BinLayout L = bin_layout(B, F, S, strip_rec_bytes(S, rgb && alpha));  // same strip width as the workspace query
        p.col_smem = strip_keeps_colours(S) ? 1 : 0;
        const int W = L.W;
        p.W = W; p.w_log2 = L.w_log2; p.nstrips = L.nstrips;
        p.len_shift = 3;
        p.stage_fast = ((S & 1) == 0) && ((((uintptr_t)a->face_index_map | (uintptr_t)a->rgb_map | (uintptr_t)a->grad_rgb | (uintptr_t)a->grad_alpha) & 7) == 0);
#ifdef NR_B200_DEBUG_KNOBS
        p.debug_skip = getenv("NR_B200_ES_SKIP") ? atoi(getenv("NR_B200_ES_SKIP")) : 0;
#endif
        while ((2 * S) >> p.len_shift > 32) p.len_shift++;
        const size_t smem = (size_t)W * ((S + 1) & ~1) * rec_bytes;
        if (smem > 160 * 1024) return NR_ERR_UNSUPPORTED;
        const int nstrips = L.nstrips;
        char* wsb = (char*)a->workspace;
        int* cnt = (int*)(wsb + L.off_cnt);
        int* off = (int*)(wsb + L.off_off);
        int* cursor = (int*)(wsb + L.off_cursor);
        int* list = (int*)(wsb + L.off_list);
        if (cudaMemsetAsync(cnt, 0, L.off_list - L.off_cnt, stream) != cudaSuccess) return NR_ERR_CUDA;  // counters, offsets, cursors
        {
            const dim3 g((F + 255) / 256, B);
            bool bin_smem = nstrips + 1 <= kBinSmemStrips;
#ifdef NR_B200_TUNING
            if (getenv("NR_B200_BIN_GLOBAL")) bin_smem = false;
#endif
            const size_t bin_bytes = (size_t)4 * (nstrips + 1) * sizeof(int);
            const long long seg_stride = (long long)F * kWideStrips;
            if (bin_smem) {
                static nr_internal::SmemOptIn optin_count, optin_fill;
                if (optin_count.ensure(k_strip_bin<false>, bin_bytes) != cudaSuccess || optin_fill.ensure(k_strip_bin<true>, bin_bytes) != cudaSuccess)
                    return NR_ERR_CUDA;
                {
                    nr_internal::LaunchScope ls("k_strip_bin", stream);
                    k_strip_bin<false><<<g, 256, bin_bytes, stream>>>(src, bbox, F, S, L.w_log2, nstrips, cnt, nullptr, nullptr, nullptr, seg_stride);
                }
                {
                    nr_internal::LaunchScope ls("k_strip_bin", stream);
                    k_strip_bin<true><<<g, 256, bin_bytes, stream>>>(src, bbox, F, S, L.w_log2, nstrips, cnt, off, cursor, list, seg_stride);
                }
            } else {
                const int nchunks = (F + kChunk - 1) / kChunk, ngroups = (F + kGroup - 1) / kGroup;
                {
                    nr_internal::LaunchScope ls("k_face_bbox", stream);
                    k_face_bbox<<<dim3(nchunks, B), kChunk, 0, stream>>>(src, F, S, ngroups, bbox, cbox);
                }
                {
                    nr_internal::LaunchScope ls("k_strip_bin", stream);
                    k_strip_bin_global<false><<<g, 256, 0, stream>>>(bbox, F, L.w_log2, nstrips, cnt, nullptr, nullptr, nullptr);
                }
                {
                    nr_internal::LaunchScope ls("k_strip_scan", stream);
                    k_strip_scan<<<B * 2, 256, 0, stream>>>(cnt, off, nstrips + 1, seg_stride);
                }
                {
                    nr_internal::LaunchScope ls("k_strip_bin", stream);
                    k_strip_bin_global<true><<<g, 256, 0, stream>>>(bbox, F, L.w_log2, nstrips, cnt, off, cursor, list);
                }
            }
        }
        p.bbox = bbox;
        p.strip_cnt = cnt; p.strip_off = off; p.strip_list = list;
        if (fill_in_scan) {
            const unsigned long long ncta = (unsigned long long)nstrips * 2 * B, n4 = tex_floats >> 2;
            p.zero_dst = a->grad_textures; p.zero_count = tex_floats; p.zero_per_cta = (n4 + ncta - 1) / ncta;
        }
        int rc;
        if (use_rgb && use_alpha) rc = launch_edge_scan<3>(p, nstrips, smem, stream);
        else if (use_rgb) rc = launch_edge_scan<1>(p, nstrips, smem, stream);
        else rc = launch_edge_scan<2>(p, nstrips, smem, stream);
        if (rc != NR_OK) return rc;
        p.zero_dst = nullptr;
        if (fill_in_scan) launch_texture_grad();
    }
    if (depth && p.g_depth) {
        nr_internal::LaunchScope ls("k_depth_grad", stream);
        k_depth_grad<<<pgrid, 256, 0, stream>>>(p);
    }
    if (interior && p.g_rgb) {  // the interior term of the rgb image (nr_interior.cu), into the same face / vertex gradient
        nr_internal::InteriorLaunch il{};
        il.args = a; il.src = src; il.dst = dst; il.shading = shading; il.tex = tex; il.light = light;
        nr_internal::launch_interior_grad(il, stream);
    }
    return cudaGetLastError() == cudaSuccess ? NR_OK : NR_ERR_CUDA;
}

extern "C" int nr_b200_backward(const nr_b200_backward_args* args, void* cuda_stream) {
    return backward_impl(args, nullptr, nullptr, {}, cuda_stream);
}

extern "C" int nr_b200_backward_corner_light(const nr_b200_backward_args* args, const float* corner_light,
                                             float* grad_corner_light, void* cuda_stream) {
    if (!corner_light) {
        nr_internal::launch_count() = 0;
        return NR_ERR_INVALID_ARG;
    }
    return backward_impl(args, corner_light, grad_corner_light, {}, cuda_stream);
}

extern "C" int nr_b200_backward_phong(const nr_b200_backward_args* args, const nr_b200_phong_args* phong, void* cuda_stream) {
    return phong ? backward_impl(args, nullptr, nullptr, {phong}, cuda_stream) : nr_internal::refuse_null_phong();
}

extern "C" int nr_b200_backward_lights(const nr_b200_backward_args* args, const nr_b200_phong_args* phong,
                                       const nr_b200_lights_args* lights, void* cuda_stream) {
    return phong ? backward_impl(args, nullptr, nullptr, {phong, lights}, cuda_stream) : nr_internal::refuse_null_phong();
}

extern "C" int nr_b200_backward_sh(const nr_b200_backward_args* args, const nr_b200_phong_args* phong,
                                   const nr_b200_lights_args* lights, const nr_b200_sh_args* sh, void* cuda_stream) {
    return phong ? backward_impl(args, nullptr, nullptr, {phong, lights, sh}, cuda_stream) : nr_internal::refuse_null_phong();
}

extern "C" int nr_b200_backward_normal_map(const nr_b200_backward_args* args, const nr_b200_phong_args* phong,
                                           const nr_b200_lights_args* lights, const nr_b200_sh_args* sh,
                                           const nr_b200_normal_map_args* nm, void* cuda_stream) {
    return phong ? backward_impl(args, nullptr, nullptr, {phong, lights, sh, nm}, cuda_stream) : nr_internal::refuse_null_phong();
}

extern "C" int nr_b200_backward_specular_map(const nr_b200_backward_args* args, const nr_b200_phong_args* phong,
                                             const nr_b200_lights_args* lights, const nr_b200_sh_args* sh,
                                             const nr_b200_normal_map_args* nm, const nr_b200_specular_map_args* sm,
                                             void* cuda_stream) {
    return phong ? backward_impl(args, nullptr, nullptr, {phong, lights, sh, nm, sm}, cuda_stream)
                 : nr_internal::refuse_null_phong();
}
