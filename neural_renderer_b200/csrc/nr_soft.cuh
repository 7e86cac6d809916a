// nr_soft.cuh -- what the soft silhouettes (nr_soft.cu) and the soft RGB (nr_soft_rgb.cu) share: the tile binning's
// parameters, the per-face setup / fill kernel k_soft_setup, the per-pixel distance test, the workspace layout, the
// host fill of the parameters and the start of the binning.
// Everything is in an anonymous namespace: each translation unit compiles its own copy of what it uses.
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "nr_b200.h"
#include "nr_internal.h"

namespace {

constexpr int kTile = 16;                   // tile side in pixels
constexpr int kThreads = kTile * kTile;     // one thread per pixel of the tile
constexpr int kWideTiles = 16;              // faces over more tiles go to the item's wide list (bounds the list storage)
constexpr float kFix = 1099511627776.0f;    // 2^40: fixed-point scale of Lambda
constexpr float kTermCap = 64.0f;           // softplus terms and Lambda saturate here: -expm1(-64) == 1.0f

struct SoftParams {
    nr::FaceSrc src;
    nr::FaceGrad dst;
    float4* rec;        // [B*F][4] face records: edge k = {ax, ay, ex, ey} in rec[k], rec[3] = {1/|e_0|^2, 1/|e_1|^2, 1/|e_2|^2, 0}
    uint2* box;         // [B*F] tile box {tx_lo | tx_hi << 16, ty_lo | ty_hi << 16}; lo > hi = takes no part
    int* cnt;           // [B*(ntiles+1)] faces per (item, tile); slot ntiles = the item's wide faces
    int* cursor;        // [B*(ntiles+1)] fill cursors
    int* off;           // [B*(ntiles+1)] list offsets (k_strip_scan)
    int* list;          // [B*F*kWideTiles] face indices grouped by (item, tile)
    float* alpha;       // [B,S,S]: written by the forward, read by the backward
    const float* g;     // [B,S,S] upstream gradient
    int B, F, S, ntx, ntiles;
    float inv_sigma;    // 1 / sigma
    float cut;          // sigma ln((1 - eps) / eps): an outside face contributes only when d^2 <= cut
    float reach;        // sqrt(cut) S / 2 + 1: the cut-off reach in pixels with one pixel of rounding guard
    float near_, far_;
};

__device__ __forceinline__ uint32_t pack16(int lo, int hi) { return ((uint32_t)lo & 0xFFFFu) | ((uint32_t)hi << 16); }
__device__ __forceinline__ int lo16(uint32_t v) { return (int)(short)(v & 0xFFFFu); }
__device__ __forceinline__ int hi16(uint32_t v) { return (int)(short)(v >> 16); }

// the pixel centre of the hard rasterizer (nr_forward.cu): NDC of raster column / row i
__device__ __forceinline__ float soft_centre(int i, int S) { return __fdiv_rn((float)(2 * i + 1 - S), (float)S); }

// ------------------------------------------------------------------------------------------------ k_soft_setup
template <bool kFill>
__global__ void __launch_bounds__(256) k_soft_setup(const __grid_constant__ SoftParams p) {
    const int b = blockIdx.y;
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= p.F) return;
    const size_t id = (size_t)b * p.F + f;
    uint2 bb;
    if (kFill) {
        bb = __ldg(p.box + id);
    } else {
        float v[9];
        nr::load_face(p.src, b, f, v);
        bool part = true;
#pragma unroll
        for (int k = 0; k < 3; k++) {
            part = part && v[3 * k + 2] >= p.near_ && v[3 * k + 2] <= p.far_;
            part = part && isfinite(v[3 * k]) && isfinite(v[3 * k + 1]);
        }
        const float S = (float)p.S, lim = (float)(p.S - 1);
        // column of x: (x S + S - 1) / 2; row of y: S - 1 - (y S + S - 1) / 2 (row 0 at the top)
        const float xmin = fminf(v[0], fminf(v[3], v[6])), xmax = fmaxf(v[0], fmaxf(v[3], v[6]));
        const float ymin = fminf(v[1], fminf(v[4], v[7])), ymax = fmaxf(v[1], fmaxf(v[4], v[7]));
        const float c0 = fmaxf(floorf(__fmaf_rn(xmin, S, lim) * 0.5f - p.reach), 0.0f);
        const float c1 = fminf(ceilf(__fmaf_rn(xmax, S, lim) * 0.5f + p.reach), lim);
        const float r0 = fmaxf(floorf(lim - __fmaf_rn(ymax, S, lim) * 0.5f - p.reach), 0.0f);
        const float r1 = fminf(ceilf(lim - __fmaf_rn(ymin, S, lim) * 0.5f + p.reach), lim);
        bb = make_uint2(pack16(1, 0), pack16(1, 0));
        if (part && c0 <= c1 && r0 <= r1) {
            bb = make_uint2(pack16((int)c0 / kTile, (int)c1 / kTile), pack16((int)r0 / kTile, (int)r1 / kTile));
            float4* r = p.rec + id * 4;
            float il[3];
#pragma unroll
            for (int k = 0; k < 3; k++) {
                const int n = k == 2 ? 0 : k + 1;
                const float ax = v[3 * k], ay = v[3 * k + 1];
                const float ex = __fsub_rn(v[3 * n], ax), ey = __fsub_rn(v[3 * n + 1], ay);
                const float l2 = __fmaf_rn(ex, ex, ey * ey);
                il[k] = l2 > 0.0f ? __frcp_rn(l2) : 0.0f;  // a zero-length edge: t = 0, the distance to its point
                r[k] = make_float4(ax, ay, ex, ey);
            }
            r[3] = make_float4(il[0], il[1], il[2], 0.0f);
        }
        p.box[id] = bb;
    }
    const int tx0 = lo16(bb.x), tx1 = hi16(bb.x), ty0 = lo16(bb.y), ty1 = hi16(bb.y);
    if (tx0 > tx1) return;
    int* seg = (kFill ? p.cursor : p.cnt) + (size_t)b * (p.ntiles + 1);
    const int* segoff = p.off + (size_t)b * (p.ntiles + 1);
    const int w = tx1 - tx0 + 1, n = w * (ty1 - ty0 + 1);
    for (int i = 0; i < (n > kWideTiles ? 1 : n); i++) {
        const int t = n > kWideTiles ? p.ntiles : (ty0 + i / w) * p.ntx + tx0 + i % w;
        const int pos = atomicAdd(seg + t, 1);
        if (kFill) p.list[segoff[t] + pos] = f;
    }
}

// ------------------------------------------------------------------------------------------------ per-pixel terms
// x_j of face record r at pixel p, or false when the face does not contribute (outside and beyond the cut-off).  With
// it: the nearest edge k, its segment parameter t and p - q (q the nearest point), for the backward, and the three edge
// functions c (the soft RGB's barycentrics).
__device__ __forceinline__ bool soft_eval(const float4* r, float px, float py, float inv_sigma, float cut, float& x,
                                          int& kb, float& tb, float& qxb, float& qyb, float c[3]) {
    const float il[3] = {r[3].x, r[3].y, r[3].z};
    float best = INFINITY;
    kb = 0; tb = 0.0f; qxb = 0.0f; qyb = 0.0f;
#pragma unroll
    for (int k = 0; k < 3; k++) {
        const float4 e = r[k];
        const float dx = __fsub_rn(px, e.x), dy = __fsub_rn(py, e.y);
        const float t = fminf(fmaxf(__fmaf_rn(dx, e.z, dy * e.w) * il[k], 0.0f), 1.0f);
        const float qx = __fmaf_rn(-t, e.z, dx), qy = __fmaf_rn(-t, e.w, dy);
        const float d2 = __fmaf_rn(qx, qx, qy * qy);
        c[k] = __fmaf_rn(e.z, dy, -(e.w * dx));  // edge function of edge k at p
        if (d2 < best) { best = d2; kb = k; tb = t; qxb = qx; qyb = qy; }
    }
    const bool inside = (c[0] > 0.0f && c[1] > 0.0f && c[2] > 0.0f) || (c[0] < 0.0f && c[1] < 0.0f && c[2] < 0.0f);
    if (!inside && best > cut) return false;
    const float a = best * inv_sigma;
    x = inside ? a : -a;
    return true;
}
__device__ __forceinline__ bool soft_term(const float4* r, float px, float py, float inv_sigma, float cut, float& x,
                                          int& kb, float& tb, float& qxb, float& qyb) {
    float c[3];
    return soft_eval(r, px, py, inv_sigma, cut, x, kb, tb, qxb, qyb, c);
}

// ------------------------------------------------------------------------------------------------ host
// workspace = face records | tile boxes | counters | cursors (one memset covers both) | offsets | lists
struct SoftLayout {
    size_t rec, box, cnt, cursor, off, list, total;
};

inline size_t align256(size_t x) { return (x + 255) / 256 * 256; }

inline int tiles_per_axis(int S) { return (S + kTile - 1) / kTile; }

// false: sizes the kernels cannot index (grid.y = B, grid.x = tiles, 16-bit tile boxes, 32-bit list offsets)
inline bool soft_sizes_ok(int B, int F, int S) {
    if (B <= 0 || F <= 0 || S <= 0) return false;
    if (B > 65535 || S > 32767) return false;
    return (long long)B * F * kWideTiles <= 0x7FFFFFFFll;
}

inline SoftLayout soft_layout(int B, int F, int S) {
    const size_t nt = (size_t)tiles_per_axis(S) * tiles_per_axis(S);
    const size_t nseg = (size_t)B * (nt + 1);
    SoftLayout L;
    L.rec = 0;
    L.box = L.rec + align256((size_t)B * F * 4 * sizeof(float4));
    L.cnt = L.box + align256((size_t)B * F * sizeof(uint2));
    L.cursor = L.cnt + nseg * sizeof(int);
    L.off = L.cnt + align256(2 * nseg * sizeof(int));
    L.list = L.off + align256(nseg * sizeof(int));
    L.total = L.list + align256((size_t)B * F * kWideTiles * sizeof(int));
    return L;
}

// The rules and fields of a zeroed SoftParams that nr_b200_soft_args and nr_b200_soft_rgb_args share: sizes the kernels
// can index, a finite sigma > 0, the geometry and (backward) its gradient in the same form -- the other form's gradient
// NULL -- and the tile grid, the cut-off, near / far, alpha and its gradient.  false = NR_ERR_INVALID_ARG; the caller
// sets the workspace pointers.
template <class Args>
inline bool fill_soft_params(const Args* a, bool backward, SoftParams* p) {
    const uint32_t flags = a->flags;
    const int B = a->batch_size, F = a->num_faces, S = a->image_size;
    const float sigma = a->sigma;
    if (!soft_sizes_ok(B, F, S) || !isfinite(sigma) || !(sigma > 0.0f)) return false;
    if (!nr_internal::make_face_src(flags, a->faces, a->vertices, a->face_indices, F, a->num_vertices, &p->src)) return false;
    if (backward) {
        const bool indexed = (flags & NR_FACES_INDEXED) != 0;
        if (indexed ? a->grad_faces != nullptr : a->grad_vertices != nullptr) return false;
        if (!nr_internal::make_face_grad(flags, a->grad_faces, a->grad_vertices, a->face_indices, F, a->num_vertices, &p->dst))
            return false;
    }
    p->alpha = a->alpha; p->g = a->grad_alpha;
    p->B = B; p->F = F; p->S = S;
    p->ntx = tiles_per_axis(S); p->ntiles = p->ntx * p->ntx;
    const double cut = (double)sigma * log((1.0 - NR_SOFT_EPS) / NR_SOFT_EPS);
    p->inv_sigma = (float)(1.0 / (double)sigma);
    p->cut = (float)cut;
    p->reach = (float)(sqrt(cut) * S * 0.5) + 1.0f;
    p->near_ = a->near_; p->far_ = a->far_;
    return true;
}

// The start of every tile binning: the counters zeroed, k_soft_setup (face records, tile boxes, counts) and the scan
// (list offsets).  A template so that only the units that call it instantiate k_soft_setup.
template <typename = void>
int bin_prefix(const SoftParams& p, cudaStream_t s) {
    nr_internal::prof_begin("memset_soft_bins", s);
    if (cudaMemsetAsync(p.cnt, 0, 2 * (size_t)p.B * (p.ntiles + 1) * sizeof(int), s) != cudaSuccess) return NR_ERR_CUDA;
    nr_internal::prof_end(s);
    {
        nr_internal::LaunchScope ls("k_soft_setup", s);
        k_soft_setup<false><<<dim3((unsigned)((p.F + 255) / 256), (unsigned)p.B), 256, 0, s>>>(p);
    }
    nr_internal::strip_scan(p.cnt, p.off, p.ntiles + 1, (long long)p.F * kWideTiles, p.B, s);
    return NR_OK;
}

}  // namespace
