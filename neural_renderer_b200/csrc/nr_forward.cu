// nr_forward.cu -- forward rasterization for sm_90a (H100).
//
// Replaces Rasterize.forward_gpu (reference neural_renderer/rasterize.py:467-513: K1 :242-277, K2 :281-359,
// K4 :372-438, alpha/background :440-465) and the transpose / flip / 2x2 pooling of rasterize_rgbad (:953-969).
//
// The reference tests every face against every pixel (B*S*S*F face tests).  Here the pass is FACE-parallel for
// coverage and PIXEL-parallel for shading, with a 64-bit z-buffer in the workspace (L2-resident at the headline shape)
// between the two:
//
//   cudaMemset       z-buffer = ~0 ("empty"), big-face counters = -1                                   (8 B / pixel)
//   k_raster_faces   one WARP per group of 32 consecutive faces, one face per lane:
//                      1. back-face / non-finite cull, conservative pixel box (nr_bbox.cuh), exact K1 inverse -- computed
//                         ONCE per face (not per tile) and written to a per-face record table {inv[9], z[3]} that the
//                         resolve pass reads back;
//                      2. row-span rasterization: for a fixed pixel row every edge test of the reference,
//                         r_k < (xp - x_k) * dy_k, is monotone in x, so the covered pixels of a row form one interval
//                         whose ends are found by binary search WITH THE REFERENCE'S OWN EXPRESSIONS (identical
//                         coverage, O(log width) tests per row).  Lanes = rows of the group's faces, flattened, 32 per pass;
//                      3. the pixels of the 32 spans are flattened again (prefix sum) and evaluated 32 fragments at a
//                         time: exact barycentric / perspective-depth expression, then ONE 64-bit reduction
//                         red.global.min.u64 on (ordered zp << 32 | face index) -- the lexicographic (zp, fn) minimum
//                         is the reference's strict `<` over ascending face index, whatever the arrival order.
//                    Faces whose box exceeds kBigArea pixels are not drawn here but appended to a per-item list.
//   k_raster_big     the listed big faces, by 64x64 screen tile (one CTA per tile, one warp per face at a time), the same
//                    row-span / fragment code clipped to the tile; exits at once when the list is empty.
//   k_resolve        one thread per pixel (per 2x2 quad when anti-aliasing): decode the winner, read its record,
//                    re-evaluate the weights with the same expression tree, sample the ts^3 texture (K4), composite the
//                    background and stream all maps out as planar, row-flipped (image orientation) coalesced rows; with
//                    anti-aliasing the thread also emits the pooled API pixel.  One variant per sampler, anti-aliasing and
//                    light mode (nr_shading.cuh: unlit, face_light, corner_light, Phong, Phong + light set, Phong + SH).
//
// Nothing depends on the screen being tiled: work is linear in the number of faces (a 1 M-face mesh costs 1 M lane
// set-ups, not 1 M box tests per tile) and in the number of covered pixels.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>

#include "nr_b200.h"
#include "nr_math.cuh"
#include "nr_internal.h"
#include "nr_bbox.cuh"

namespace {

constexpr int kFaceWarps = 8;          // warps (= 32-face groups) per CTA of k_raster_faces
constexpr int kXpTable = 2048;         // pixel-centre table in shared memory for rasters up to this size
#ifndef NR_BIG_AREA
#define NR_BIG_AREA 1024
#endif
constexpr int kBigArea = NR_BIG_AREA;  // big-face threshold up to raster 256, 4x above
constexpr int kBigTile = 64;           // screen tile of k_raster_big
constexpr int kRecWords = 12;          // {inv[9], z0, z1, z2}
constexpr int kOwnTable = 256;         // rows / fragments per pass whose owner lane is looked up instead of searched
#ifndef NR_FACES_MIN_CTAS
#define NR_FACES_MIN_CTAS 5
#endif
#ifndef NR_RESOLVE_MIN_CTAS
#define NR_RESOLVE_MIN_CTAS 6  // CTAs of 256 threads per SM the resolve pass is compiled for (40 registers: the pass is
                               // latency-bound on its dependent gathers; 8 CTAs = 32 registers spill on sm_90 and were
                               // measured slower on H100: 121 vs 114 us at the headline shape)
#endif
#ifndef NR_RESOLVE_MIP_MIN_CTAS
#define NR_RESOLVE_MIP_MIN_CTAS 4  // the trilinear variants (kTex == 3): 64 registers; at 5 or 6 CTAs (48 / 40 registers)
                                   // they spill (-Xptxas -v)
#endif
#ifndef NR_RESOLVE_SMOOTH_MIN_CTAS
#define NR_RESOLVE_SMOOTH_MIN_CTAS 6     // smooth-shaded (kLightCorner) cube / bilinear variants: 40 registers, no spills
#endif
#ifndef NR_RESOLVE_SMOOTH_AA_MIN_CTAS
#define NR_RESOLVE_SMOOTH_AA_MIN_CTAS 4  // the same with anti-aliasing: the cube variant spills at 5 CTAs (48 registers)
#endif
#ifndef NR_RESOLVE_PHONG_MIN_CTAS
#define NR_RESOLVE_PHONG_MIN_CTAS 4      // Phong-shaded (kLightPhong) variants, every sampler (DESIGN.md section 4g)
#endif
#ifndef NR_RESOLVE_LIGHTS_MIN_CTAS
#define NR_RESOLVE_LIGHTS_MIN_CTAS 4     // Phong with a light set (kLightPhongSet), every sampler (DESIGN.md section 4h)
#endif
#ifndef NR_RESOLVE_SH_MIN_CTAS
#define NR_RESOLVE_SH_MIN_CTAS 4         // Phong with an SH environment (kLightPhongSH), every sampler (DESIGN.md section 4i)
#endif
#ifndef NR_RESOLVE_NM_MIN_CTAS
#define NR_RESOLVE_NM_MIN_CTAS 4         // Phong through a normal map (kLightPhongNM), both image samplers (DESIGN.md section 4k)
#endif
#ifndef NR_RESOLVE_SM_MIN_CTAS
#define NR_RESOLVE_SM_MIN_CTAS 4         // Phong through a specular map (kLightPhongSM), both image samplers (DESIGN.md section 4l)
#endif
constexpr int kResolveTileW = 32, kResolveTileH = 8;  // API pixels per k_resolve CTA (256 threads, 8 x 4 per warp)
constexpr uint32_t kStageBytes = 32 * 1024;  // shared memory of a k_resolve CTA for staged texture cubes

struct FwdParams {
    nr::FaceSrc src;
    const float* bg_batch;
    unsigned long long* zbuf;  // [B,S,S] raster orientation (row = yi): ordered zp << 32 | face index, ~0 = empty
    float4* tab;               // [B,F,3] float4: {inv0..3}, {inv4..7}, {inv8, z0, z1, z2} of every drawn face
    int* big_cnt;              // [B] number of big faces - 1 (memset to 0xFF = -1)
    int* work_next;            // next (item, group) unit of k_raster_faces - 1 (memset to -1)
    int* any_big;              // -1 until some item has a big face
    int* big_list;             // [B,F]
    float4* z0tab;             // [F] {z0, z1, z2, -} of EVERY face of batch item 0 (NR_TEX_Z_BATCH0 with RGB), else nullptr
    int32_t* fim;
    float* wmap;
    float* dmap;
    float* rgb;
    float* alpha;
    float* out_rgb;
    float* out_alpha;
    float* out_depth;
    int B, F, S, ts, ngroups;
    int big_area;  // faces whose (clipped) pixel box is larger go through k_raster_big
    uint32_t flags;
    float near_lo, far_cmp, far_val;
    float bg[3];
    nr::Texture tex;  // what the pixel samples
    // what lights the pixel: face_light, corner_light or the Phong inputs of the call's light mode
    nr::Shading shading;
};

// rasterize.py:291-292  xp = (2 * xi + 1 - is) / is evaluated in double and rounded to float.  Both operands are
// integers below 2^24, so the correctly rounded fp32 quotient is the same number (a double rounding cannot land on a
// float midpoint: |n/S - midpoint| >= 2^-24 / S relative, far above the 2^-53 of the intermediate).
__device__ __forceinline__ float pixel_centre(int i, int S, float fS) { return __fdiv_rn((float)(2 * i + 1 - S), fS); }

struct PixelCentres {
    const float* table;  // shared memory, S entries, or nullptr
    int S;
    float fS;
    __device__ __forceinline__ float operator()(int i) const { return table ? table[i] : pixel_centre(i, S, fS); }
};

// Per-warp scratch of k_raster_faces / k_raster_big
struct __align__(16) WarpScratch {
    float4 rec[32][2];   // {x0, y0, x1, y1}, {x2, y2, box x (lo | hi << 16), box y}: sweep record of the lane's face
    float4 tab[32][3];   // {inv[9], z[3]} of the lane's face
    int rowpre[32];      // first row number of each lane's face
    int spanpre[32];     // first fragment number of each row span of the current pass
    uint8_t rowown[kOwnTable];   // owner lane of every row of the unit (when there are at most kOwnTable rows)
    uint8_t fragown[kOwnTable];  // owner lane of every fragment of the current pass (likewise)
};

//@phase row spans + fragments (shared by k_raster_faces and k_raster_big)
// Rows `r` in [0, nrows) of this warp's faces are distributed over the lanes (32 per pass).  rowpre[l] = first row of
// lane l's face (exclusive prefix of the box heights; faces without rows have height 0); face index = face_base + l.
__device__ __forceinline__ void raster_rows(const FwdParams& p, WarpScratch& ws, const PixelCentres& pc, int b, int nrows,
                                            int face_base, int lane, bool row_table) {
    unsigned long long* zb = p.zbuf + (size_t)b * p.S * p.S;
    for (int base = 0; base < nrows; base += 32) {
        const int r = base + lane;
        int lo = 1, hi = 0, own = 0, y = 0;
        if (r < nrows) {
            int a;
            if (row_table) {
                a = ws.rowown[r];
            } else {
                // owner = last lane whose first row is <= r (upper_bound - 1 over the non-decreasing prefix)
                a = 0;
                int bnd = 32;
#pragma unroll
                for (int it = 0; it < 5; it++) {
                    const int mid = (a + bnd) >> 1;
                    if (ws.rowpre[mid] <= r) a = mid; else bnd = mid;
                }
            }
            own = a;
            const float4 q0 = ws.rec[a][0], q1 = ws.rec[a][1];
            const float x0 = q0.x, y0 = q0.y, x1 = q0.z, y1 = q0.w, x2 = q1.x, y2 = q1.y;
            const uint32_t boxx = __float_as_uint(q1.z), boxy = __float_as_uint(q1.w);
            y = (int)(boxy & 0xFFFFu) + (r - ws.rowpre[a]);
            const float yp = pc(y);
            const float xk[3] = {x0, x1, x2};
            const float dyk[3] = {__fsub_rn(y1, y0), __fsub_rn(y2, y1), __fsub_rn(y0, y2)};
            const float rk[3] = {__fmul_rn(__fsub_rn(yp, y0), __fsub_rn(x1, x0)),
                                 __fmul_rn(__fsub_rn(yp, y1), __fsub_rn(x2, x1)),
                                 __fmul_rn(__fsub_rn(yp, y2), __fsub_rn(x0, x2))};
            const int lo0 = (int)(boxx & 0xFFFFu), hi0 = (int)(boxx >> 16);
            // out_k(x) = r_k < (xp(x) - x_k) * dy_k is non-decreasing in x for dy_k >= 0 (constant for dy_k == 0) and
            // non-increasing for dy_k < 0: per edge, the first x where out_k(x) != (dy_k < 0).  The three searches run
            // over the same interval in lockstep (three independent dependency chains instead of one long one).
            int a3[3] = {lo0, lo0, lo0}, b3[3] = {hi0 + 1, hi0 + 1, hi0 + 1};
            const bool neg[3] = {dyk[0] < 0.0f, dyk[1] < 0.0f, dyk[2] < 0.0f};
            while ((a3[0] < b3[0]) | (a3[1] < b3[1]) | (a3[2] < b3[2])) {
#pragma unroll
                for (int k = 0; k < 3; k++) {
                    if (a3[k] < b3[k]) {
                        const int mid = (a3[k] + b3[k]) >> 1;
                        const bool out = rk[k] < __fmul_rn(__fsub_rn(pc(mid), xk[k]), dyk[k]);
                        if (out != neg[k]) b3[k] = mid; else a3[k] = mid + 1;
                    }
                }
            }
            lo = lo0; hi = hi0;
#pragma unroll
            for (int k = 0; k < 3; k++) {
                if (neg[k]) lo = max(lo, a3[k]); else hi = min(hi, a3[k] - 1);
            }
        }
        // flatten the 32 spans into fragments
        const int n = max(hi - lo + 1, 0);
        int sincl = n;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int t = __shfl_up_sync(0xffffffffu, sincl, o);
            if (lane >= o) sincl += t;
        }
        const int nfrag = __shfl_sync(0xffffffffu, sincl, 31);
        ws.spanpre[lane] = sincl - n;
        const bool frag_table = nfrag <= kOwnTable;
        if (frag_table)
            for (int j = 0; j < n; j++) ws.fragown[sincl - n + j] = (uint8_t)lane;
        __syncwarp();
        for (int fb = 0; fb < nfrag; fb += 32) {
            const int i = fb + lane;
            int a = 0;
            if (frag_table) {
                if (i < nfrag) a = ws.fragown[i];
            } else {
                int bnd = 32;
#pragma unroll
                for (int it = 0; it < 5; it++) {
                    const int mid = (a + bnd) >> 1;
                    if (ws.spanpre[mid] <= i) a = mid; else bnd = mid;
                }
            }
            // all lanes take part in the shuffles; lanes past the end evaluate nothing
            const int o_own = __shfl_sync(0xffffffffu, own, a);
            const int o_y = __shfl_sync(0xffffffffu, y, a);
            const int o_lo = __shfl_sync(0xffffffffu, lo, a);
            if (i < nfrag) {
                const int x = o_lo + (i - ws.spanpre[a]);
                const float4 aa = ws.tab[o_own][0], bb = ws.tab[o_own][1], cc = ws.tab[o_own][2];
                const float inv[9] = {aa.x, aa.y, aa.z, aa.w, bb.x, bb.y, bb.z, bb.w, cc.x};
                float w[3];
                const float zp = nr::weights_and_depth(inv, (float)x, (float)o_y, cc.y, cc.z, cc.w, w);
                // rasterize.py:331 + :334 against the initial depth_min = far; NaN fails both (never wins)
                if (zp > p.near_lo && zp < p.far_cmp) {
                    const unsigned long long key =
                        ((unsigned long long)nr::float_to_ordered(zp) << 32) | (uint32_t)(face_base + o_own);
                    atomicMin(zb + (size_t)o_y * p.S + x, key);  // result unused: red.global.min.u64
                }
            }
        }
        __syncwarp();  // spanpre / fragown are rewritten by the next pass
    }
}

__device__ __forceinline__ void fill_centres(float* table, int S, int tid, int nthreads) {
    const float fS = (float)S;
    for (int i = tid; i < S; i += nthreads) table[i] = pixel_centre(i, S, fS);
}

// ------------------------------------------------------------------------------------------ k_raster_faces
//@phase k_raster_faces: cull + K1 + records
__global__ void __launch_bounds__(kFaceWarps * 32, NR_FACES_MIN_CTAS) k_raster_faces(const __grid_constant__ FwdParams p) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    WarpScratch* scratch = reinterpret_cast<WarpScratch*>(smem_raw);
    float* centres = reinterpret_cast<float*>(smem_raw + sizeof(WarpScratch) * kFaceWarps);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int S = p.S;
    const bool use_table = S <= kXpTable;
    if (use_table) {
        fill_centres(centres, S, tid, kFaceWarps * 32);
        __syncthreads();
    }
    const PixelCentres pc{use_table ? centres : nullptr, S, (float)S};
    WarpScratch& ws = scratch[warp];
    // Persistent warps pull (item, group) units from one counter: groups differ a lot in cost (all back faces: nothing;
    // a dense front patch: thousands of fragments), so a static assignment leaves most of the chip idle in the tail.
    const int nunits = p.B * p.ngroups;
    for (;;) {
        int u = 0;
        if (lane == 0) u = atomicAdd(p.work_next, 1) + 1;  // the counter starts at -1
        u = __shfl_sync(0xffffffffu, u, 0);
        if (u >= nunits) break;
        const int b = u / p.ngroups, g = u - b * p.ngroups;
        const int f = (g << 5) + lane;
        int h = 0;
        if (f < p.F) {
            float c[9];
            nr::load_face(p.src, b, f, c);
            // rasterize.py:389: the sampler of every item reads the vertex depths of item 0 -- of drawn and culled faces
            // alike -- so item 0's groups leave them in a compact table (one 16-byte load per pixel in k_resolve)
            if (b == 0 && p.z0tab) p.z0tab[f] = make_float4(c[2], c[5], c[8], 0.0f);
            int xlo, xhi, ylo, yhi;
            if (face_pixel_box<true>(c[0], c[1], c[3], c[4], c[6], c[7], S, xlo, xhi, ylo, yhi)) {
                const float fS = (float)S;
                float inv[9];
                nr::face_inverse(nr::to_pixel(c[0], fS), nr::to_pixel(c[1], fS), nr::to_pixel(c[3], fS), nr::to_pixel(c[4], fS),
                                 nr::to_pixel(c[6], fS), nr::to_pixel(c[7], fS), inv);
                const float4 t0 = make_float4(inv[0], inv[1], inv[2], inv[3]), t1 = make_float4(inv[4], inv[5], inv[6], inv[7]),
                             t2 = make_float4(inv[8], c[2], c[5], c[8]);
                float4* gt = p.tab + ((size_t)b * p.F + f) * 3;
                gt[0] = t0; gt[1] = t1; gt[2] = t2;
                if ((xhi - xlo + 1) * (yhi - ylo + 1) > p.big_area) {
                    const int slot = atomicAdd(p.big_cnt + b, 1) + 1;  // counters start at -1
                    p.big_list[(size_t)b * p.F + slot] = f;
                    if (slot == 0) *p.any_big = 0;
                } else {
                    h = yhi - ylo + 1;
                    ws.tab[lane][0] = t0; ws.tab[lane][1] = t1; ws.tab[lane][2] = t2;
                    ws.rec[lane][0] = make_float4(c[0], c[1], c[3], c[4]);
                    ws.rec[lane][1] = make_float4(c[6], c[7], __uint_as_float((uint32_t)xlo | ((uint32_t)xhi << 16)),
                                                  __uint_as_float((uint32_t)ylo | ((uint32_t)yhi << 16)));
                }
            }
        }
        int incl = h;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int t = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += t;
        }
        const int nrows = __shfl_sync(0xffffffffu, incl, 31);
        if (nrows == 0) continue;
        ws.rowpre[lane] = incl - h;
        const bool row_table = nrows <= kOwnTable;
        if (row_table)
            for (int j = 0; j < h; j++) ws.rowown[incl - h + j] = (uint8_t)lane;
        __syncwarp();
        raster_rows(p, ws, pc, b, nrows, g << 5, lane, row_table);
        __syncwarp();  // the scratch is rewritten by the next unit
    }
}

// -------------------------------------------------------------------------------------------- k_raster_big
//@phase k_raster_big
__global__ void __launch_bounds__(256) k_raster_big(const __grid_constant__ FwdParams p) {
    if (__ldg(p.any_big) < 0) return;  // no item has a big face: the common case costs one load
    extern __shared__ __align__(16) unsigned char smem_raw[];
    WarpScratch* scratch = reinterpret_cast<WarpScratch*>(smem_raw);
    float* centres = reinterpret_cast<float*>(smem_raw + sizeof(WarpScratch) * 8);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int S = p.S;
    const bool use_table = S <= kXpTable;
    if (use_table) {
        fill_centres(centres, S, tid, 256);
        __syncthreads();
    }
    const PixelCentres pc{use_table ? centres : nullptr, S, (float)S};
    const int tiles_x = (S + kBigTile - 1) / kBigTile;
    const int ntiles = tiles_x * tiles_x;
    WarpScratch& ws = scratch[warp];
    for (int unit = blockIdx.x; unit < ntiles * p.B; unit += gridDim.x) {
        const int b = unit / ntiles, tile = unit - b * ntiles;
        const int nbig = __ldg(p.big_cnt + b) + 1;
        if (nbig <= 0) continue;
        const int tx0 = (tile % tiles_x) * kBigTile, ty0 = (tile / tiles_x) * kBigTile;
        const int tx1 = min(tx0 + kBigTile, S) - 1, ty1 = min(ty0 + kBigTile, S) - 1;
        for (int i = warp; i < nbig; i += 8) {
            const int f = __ldg(p.big_list + (size_t)b * p.F + i);
            float c[9];
            nr::load_face(p.src, b, f, c);  // warp-uniform
            int xlo, xhi, ylo, yhi;
            if (!face_pixel_box<true>(c[0], c[1], c[3], c[4], c[6], c[7], S, xlo, xhi, ylo, yhi)) continue;
            xlo = max(xlo, tx0); xhi = min(xhi, tx1); ylo = max(ylo, ty0); yhi = min(yhi, ty1);
            if (xlo > xhi || ylo > yhi) continue;
            // the face sits in slot 0 of the warp's scratch; every lane rasterizes rows of that one face
            if (lane == 0) {
                const float4* gt = p.tab + ((size_t)b * p.F + f) * 3;
                ws.tab[0][0] = gt[0]; ws.tab[0][1] = gt[1]; ws.tab[0][2] = gt[2];
                ws.rec[0][0] = make_float4(c[0], c[1], c[3], c[4]);
                ws.rec[0][1] = make_float4(c[6], c[7], __uint_as_float((uint32_t)xlo | ((uint32_t)xhi << 16)),
                                           __uint_as_float((uint32_t)ylo | ((uint32_t)yhi << 16)));
            }
            const int h = yhi - ylo + 1;
            ws.rowpre[lane] = lane == 0 ? 0 : h;  // lane 0 owns rows [0, h); the other prefix entries lie past the end
            __syncwarp();
            raster_rows(p, ws, pc, b, h, f, lane, false);  // face_base + slot 0 = f
            __syncwarp();
        }
    }
}

// ------------------------------------------------------------------------------------------------ k_resolve
//@phase shade (resolve helper)
struct Shaded {
    int fim;
    float w0, w1, w2, depth, r, g, b, alpha;
};

// ---- bulk asynchronous copies (TMA engine, cp.async.bulk -> SASS UBLKCP) completing on a shared-memory mbarrier
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");  // visible to the async proxy
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_copy_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst_smem)),
                 "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    for (;;) {
        uint32_t done;
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.b32 %0, 1, 0, p;\n\t}"
                     : "=r"(done)
                     : "r"(smem_u32(bar)), "r"(parity)
                     : "memory");
        if (done) break;
        __nanosleep(64);  // do not burn issue slots of the warps that are still computing
    }
}

// geometry half of a pixel: winner's record -> weights (+ texture coordinates when drawing RGB)
struct PixelGeom {
    int fn, cube;
    bool rev;
    float zp, w[3];
};

// rasterize.py:389 -- the sampler's vertex depths come from batch item 0 (NR_TEX_Z_BATCH0: the table k_raster_faces
// left), else from the winner's record
__device__ __forceinline__ void sampler_depths(const FwdParams& p, int fn, const float4& cc, float& z0, float& z1, float& z2) {
    z0 = cc.y; z1 = cc.z; z2 = cc.w;
    if (p.z0tab) {
        const float4 z = __ldg(p.z0tab + fn);
        z0 = z.x; z1 = z.y; z2 = z.z;
    }
}

// face fn's face_light (kLightFace; nullptr in the other modes, whose samples are unlit)
template <int kLight>
__device__ __forceinline__ const float* face_light_of(const FwdParams& p, int b, int fn) {
    return kLight == nr::kLightFace ? p.shading.face_light + p.shading.fl_off(b, p.F, fn) : nullptr;
}

// one pixel, every texel straight from global memory (anti-aliased quads, texture sizes the bulk copy cannot stage);
// kUV: bilinear sample of the texture image at the pixel's perspective-correct UV instead of the ts^3 cube; kMip:
// trilinear sample of its mip pyramid at the pixel's level of detail.  kLight (nr_shading.cuh): kLightFace multiplies every
// texel by face_light, the later modes shade the unlit sample (nr::shade)
template <int kLight, bool kUV = false, bool kMip = false>
__device__ __forceinline__ Shaded shade_pixel(const FwdParams& p, int b, unsigned long long key, int xi, int yi, float bgr,
                                              float bgg, float bgb) {
    Shaded o;
    if (key == ~0ull) {
        o.fim = -1; o.w0 = o.w1 = o.w2 = 0.0f; o.depth = p.far_val; o.r = bgr; o.g = bgg; o.b = bgb; o.alpha = 0.0f;
        return o;
    }
    const int fn = (int)(uint32_t)(key & 0xFFFFFFFFull);
    const float zp = nr::ordered_to_float((uint32_t)(key >> 32));
    const float4* t4 = p.tab + ((size_t)b * p.F + fn) * 3;
    const float4 a = __ldg(t4), bb = __ldg(t4 + 1), cc = __ldg(t4 + 2);
    const float inv[9] = {a.x, a.y, a.z, a.w, bb.x, bb.y, bb.z, bb.w, cc.x};
    float w[3];
    nr::barycentric_weights(inv, (float)xi, (float)yi, w);
    o.fim = fn; o.w0 = w[0]; o.w1 = w[1]; o.w2 = w[2]; o.depth = zp; o.alpha = 1.0f;
    o.r = o.g = o.b = 0.0f;
    if (p.flags & NR_RETURN_RGB) {
        float u = 0.0f, v = 0.0f;  // kUV: the pixel's uv, where the maps of modes 6-7 are sampled too
        if constexpr (kUV) {
            // the winner's own vertex depths (no batch-0 quirk); fill_back copies read face fn - F/2's corners reversed
            bool rev;
            const int uf = nr::stored_face(p.flags & NR_TEX_FILL_BACK, p.F, fn, rev);
            float uv[6];
            nr::face_uvs(p.tex, b, uf, rev, uv);
            nr::pixel_uv(w, zp, cc.y, cc.z, cc.w, uv, u, v);
            float l0 = 1.0f, l1 = 1.0f, l2 = 1.0f;
            if (kLight == nr::kLightFace) {
                const float* lp = p.shading.face_light + p.shading.fl_off(b, p.F, fn);
                l0 = __ldg(lp); l1 = __ldg(lp + 1); l2 = __ldg(lp + 2);
            }
            float c[3];
            if constexpr (kMip) {
                const float lod = nr::mip_lod(inv, w, zp, cc.y, cc.z, cc.w, uv, p.tex.Ht, p.tex.Wt, p.tex.mip.levels);
                nr::mip_blend<kLight == nr::kLightFace>(p.tex.tex + p.tex.img_off(b), p.tex.mip,
                                                        nr::mip_levels(lod, p.tex.mip.levels), u, v, l0, l1, l2, c);
            } else {
                const nr::UvTaps t = nr::uv_taps(u, v, p.tex.Ht, p.tex.Wt);
                nr::uv_blend<kLight == nr::kLightFace>(p.tex.tex + p.tex.img_off(b), p.tex.Wt, t, l0, l1, l2, c);
            }
            o.r = c[0]; o.g = c[1]; o.b = c[2];
        } else {
            float z0, z1, z2;
            sampler_depths(p, fn, cc, z0, z1, z2);
            const int ts = p.ts;
            const nr::TexCoord tc = nr::texture_coords(w, zp, z0, z1, z2, ts, p.tex.tex_cmp, p.tex.tex_val);
            bool rev;
            const int cube = nr::stored_face(p.flags & NR_TEX_FILL_BACK, p.F, fn, rev);
            const float* tex = p.tex.tex + p.tex.cube_off(b, cube, ts);
            nr::cube_blend<kLight == nr::kLightFace, false>(tex, tc, ts, rev, face_light_of<kLight>(p, b, fn), o.r, o.g, o.b);
        }
        if constexpr (kLight >= nr::kLightCorner) {  // the light of the pixel's l_k (own depths) on the unlit sample
            float l[3], c[3] = {o.r, o.g, o.b};
            nr::perspective_weights(w, zp, cc.y, cc.z, cc.w, l);
            nr::shade<kLight>(p.shading, b, p.F, fn, l, u, v, c);
            o.r = c[0]; o.g = c[1]; o.b = c[2];
        }
    }
    return o;
}

// CTAs per SM each k_resolve variant is compiled for (the NR_RESOLVE_*_MIN_CTAS above)
constexpr int resolve_min_ctas(bool aa, int tex, int light) {
    if (light == nr::kLightPhongSM) return NR_RESOLVE_SM_MIN_CTAS;
    if (light == nr::kLightPhongNM) return NR_RESOLVE_NM_MIN_CTAS;
    if (light == nr::kLightPhongSH) return NR_RESOLVE_SH_MIN_CTAS;
    if (light == nr::kLightPhongSet) return NR_RESOLVE_LIGHTS_MIN_CTAS;
    if (light == nr::kLightPhong) return NR_RESOLVE_PHONG_MIN_CTAS;
    if (tex == 3) return NR_RESOLVE_MIP_MIN_CTAS;
    if (light == nr::kLightCorner) return aa ? NR_RESOLVE_SMOOTH_AA_MIN_CTAS : NR_RESOLVE_SMOOTH_MIN_CTAS;
    return aa ? 5 : NR_RESOLVE_MIN_CTAS;
}

//@phase resolve + stores
// grid = (column chunks, API rows, batch items): row / item are block-uniform, all offsets are 32-bit.
//
// kStage (opt-in NR_FWD_STAGE_TEXTURES; RGB, no anti-aliasing, cube size a multiple of 16 bytes): the CTA = 256
// consecutive pixels of one image row.
// Runs of neighbouring pixels that show the same texture cube are found with a ballot; the first pixel of every run
// issues ONE asynchronous bulk copy (cp.async.bulk, the TMA engine) of that face's whole ts^3 cube into shared memory,
// all copies of the CTA complete on one mbarrier, and while they are in flight every thread reads its winner's record
// and evaluates weights and texture coordinates.  The 24 texel reads of the trilinear blend then hit shared memory
// instead of being 24 dependent, uncoalesced global loads behind the record load.  Runs beyond the staging capacity
// (and the other kernel variants) sample global memory directly.  Measured on H100 at the headline shape: 183 us against
// 119 us for the direct gather (ts = 4; 92.5 vs 90.8 us at ts = 2) -- a whole 768-byte cube (ts = 4) is copied for the 8 texels a pixel blends, and the L1 data stage pays
// for the shared-memory writes of the copy plus the bank conflicts of the 24 scattered reads.  The direct gather is
// therefore the default.
//
// kTex == 2 (NR_TEX_UV): the direct variants with the texture-image sampler (shade_pixel<kLight, true>), same tile map.
// kTex == 3 (NR_TEX_UV | NR_TEX_MIPMAP): the same with the trilinear pyramid sampler (shade_pixel<kLight, true, true>).
template <bool kAA, int kTex, int kLight>
__global__ void __launch_bounds__(256, resolve_min_ctas(kAA, kTex, kLight)) k_resolve(const __grid_constant__ FwdParams p, int nslots) {
    constexpr bool kStage = kTex == 1;  // kTex: 0 = every texel straight from global memory, 1 = cubes staged with cp.async.bulk
    constexpr bool kUV = kTex >= 2;     //       2 = texture image through per-corner UVs, 3 = its mip pyramid
    constexpr bool kMip = kTex == 3;
    extern __shared__ __align__(16) unsigned char stage_raw[];
    __shared__ uint64_t s_bar;
    __shared__ int s_runs[8];
    const int b = blockIdx.z;
    const int S = p.S;
    const uint32_t plane = (uint32_t)S * (uint32_t)S;
    float bgr = p.bg[0], bgg = p.bg[1], bgb = p.bg[2];
    if (p.flags & NR_BG_PER_BATCH) {
        bgr = __ldg(p.bg_batch + 3 * b + 0); bgg = __ldg(p.bg_batch + 3 * b + 1); bgb = __ldg(p.bg_batch + 3 * b + 2);
    }
    const bool want_rgb = (p.flags & NR_RETURN_RGB) != 0;
    const unsigned long long* zb = p.zbuf + (size_t)b * plane;
    int32_t* fim = p.fim + (size_t)b * plane;
    float* dmap = p.dmap + (size_t)b * plane;
    float* wmap = p.wmap + (size_t)b * 3 * plane;
    float* rgb = want_rgb ? p.rgb + (size_t)b * 3 * plane : nullptr;
    float* alpha = p.alpha ? p.alpha + (size_t)b * plane : nullptr;
    // Thread -> pixel map of the direct variants: a CTA of 256 threads covers a 32 x 8 tile of API pixels and every WARP an
    // 8 x 4 block of it.  Faces are compact blobs (about 4 x 3 pixels at the headline shape), so a 2-D footprint meets a
    // third of the distinct faces a 32 x 1 row segment meets -- and the gathers of the pass (texels, records) cost one
    // L1 wavefront per request and distinct 128-byte line, i.e. per distinct face.  Stores and key loads become four
    // 32-byte row segments per warp instead of one 128-byte segment: whole sectors, same DRAM traffic.
    const int t_lane = threadIdx.x & 31, t_warp = threadIdx.x >> 5;
    const int col2 = blockIdx.x * kResolveTileW + (t_warp & 3) * 8 + (t_lane & 7);
    const int row2 = blockIdx.y * kResolveTileH + (t_warp >> 2) * 4 + (t_lane >> 3);
    // (Anti-aliased quads are 2-D footprints already and the texture / depth gradient kernels lose with it: those keep the
    // row-major map.)
    const bool tiled = !kStage && !kAA;
    const int col = tiled ? col2 : (int)(blockIdx.x * blockDim.x + threadIdx.x);
    if (!kAA && kStage) {
        const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
        const int row = blockIdx.y, yi = S - 1 - row;
        if (tid == 0) mbar_init(&s_bar, 1);
        const unsigned long long key = col < S ? __ldg(zb + (uint32_t)yi * S + col) : ~0ull;
        const bool covered = key != ~0ull;
        const int fn = (int)(uint32_t)(key & 0xFFFFFFFFull);
        bool rev = false;
        const int cube = covered ? nr::stored_face(p.flags & NR_TEX_FILL_BACK, p.F, fn, rev) : -1;
        const int left = __shfl_up_sync(0xffffffffu, cube, 1);
        const bool head = covered && (lane == 0 || cube != left);
        const uint32_t heads = __ballot_sync(0xffffffffu, head);
        if (lane == 0) s_runs[warp] = __popc(heads);
        __syncthreads();
        int base = 0, total = 0;
        const int nwarps = blockDim.x >> 5;
        for (int w = 0; w < nwarps; w++) {
            const int c = s_runs[w];
            if (w < warp) base += c;
            total += c;
        }
        const int ts = p.ts;
        const uint32_t cube_bytes = (uint32_t)(ts * ts * ts) * 12u;
        const int slot = base + __popc(heads & ((2u << lane) - 1u)) - 1;  // run of this pixel (2u << 31 wraps: all heads)
        const bool staged = covered && slot < nslots;
        if (tid == 0) mbar_arrive_expect_tx(&s_bar, (uint32_t)min(total, nslots) * cube_bytes);
        const float* gtex = p.tex.tex + p.tex.cube_off(b, covered ? cube : 0, ts);
        float* stex = reinterpret_cast<float*>(stage_raw) + (size_t)(staged ? slot : 0) * (cube_bytes >> 2);
        if (head && staged) bulk_copy_g2s(stex, gtex, cube_bytes, &s_bar);
        if (col >= S) return;
        const uint32_t o = (uint32_t)row * S + col;
        if (!covered) {
            fim[o] = -1;
            dmap[o] = p.far_val;
            wmap[o] = 0.0f; wmap[o + plane] = 0.0f; wmap[o + 2 * plane] = 0.0f;
            if (alpha) alpha[o] = 0.0f;
            rgb[o] = bgr; rgb[o + plane] = bgg; rgb[o + 2 * plane] = bgb;
            return;
        }
        // while the cubes are in flight: record -> weights -> texture coordinates
        const float zp = nr::ordered_to_float((uint32_t)(key >> 32));
        const float4* t4 = p.tab + ((size_t)b * p.F + fn) * 3;
        const float4 a = __ldg(t4), bb = __ldg(t4 + 1), cc = __ldg(t4 + 2);
        const float inv[9] = {a.x, a.y, a.z, a.w, bb.x, bb.y, bb.z, bb.w, cc.x};
        float w[3];
        nr::barycentric_weights(inv, (float)col, (float)yi, w);
        float z0, z1, z2;
        sampler_depths(p, fn, cc, z0, z1, z2);
        const nr::TexCoord tc = nr::texture_coords(w, zp, z0, z1, z2, ts, p.tex.tex_cmp, p.tex.tex_val);
        fim[o] = fn;
        dmap[o] = zp;
        wmap[o] = w[0]; wmap[o + plane] = w[1]; wmap[o + 2 * plane] = w[2];
        if (alpha) alpha[o] = 1.0f;
        float r, g, bl;
        if (staged) {
            mbar_wait(&s_bar, 0);
            nr::cube_blend<kLight == nr::kLightFace, false>(stex, tc, ts, rev, face_light_of<kLight>(p, b, fn), r, g, bl);
        } else {
            nr::cube_blend<kLight == nr::kLightFace, false>(gtex, tc, ts, rev, face_light_of<kLight>(p, b, fn), r, g, bl);
        }
        rgb[o] = r; rgb[o + plane] = g; rgb[o + 2 * plane] = bl;
    } else if (!kAA) {
        // thread = one pixel of the IMAGE (row 0 = top): raster row yi = S - 1 - row
        const int row = row2, yi = S - 1 - row;
        if (col >= S || row >= S) return;
        const Shaded s = shade_pixel<kLight, kUV, kMip>(p, b, __ldg(zb + (uint32_t)yi * S + col), col, yi, bgr, bgg, bgb);
        const uint32_t o = (uint32_t)row * S + col;
        // streaming stores: 134 MB of maps that nothing reads again before the backward pass should not push the
        // z-buffer, the face records and the texture cubes out of the L2
        __stcs(fim + o, s.fim);
        __stcs(dmap + o, s.depth);
        __stcs(wmap + o, s.w0); __stcs(wmap + o + plane, s.w1); __stcs(wmap + o + 2 * plane, s.w2);
        if (alpha) __stcs(alpha + o, s.alpha);
        if (want_rgb) { __stcs(rgb + o, s.r); __stcs(rgb + o + plane, s.g); __stcs(rgb + o + 2 * plane, s.b); }
    } else {
        // thread = one pooled API pixel = one 2x2 quad of the raster
        const int H = S >> 1;
        const uint32_t oplane = (uint32_t)H * (uint32_t)H;
        const int orow = blockIdx.y;
        if (col >= H) return;
        float sr = 0.f, sg = 0.f, sb = 0.f, sa = 0.f, sd = 0.f;
        // the four pixels are shaded one after the other (keeps the register footprint of a single pixel) in image
        // order: top-left, top-right, bottom-left, bottom-right
#pragma unroll 1
        for (int k = 0; k < 4; k++) {
            const int row = 2 * orow + (k >> 1), xi = 2 * col + (k & 1);
            const int yi = S - 1 - row;
            const Shaded s = shade_pixel<kLight, kUV, kMip>(p, b, __ldg(zb + (uint32_t)yi * S + xi), xi, yi, bgr, bgg, bgb);
            const uint32_t o = (uint32_t)row * S + xi;
            __stcs(fim + o, s.fim);
            __stcs(dmap + o, s.depth);
            __stcs(wmap + o, s.w0); __stcs(wmap + o + plane, s.w1); __stcs(wmap + o + 2 * plane, s.w2);
            if (alpha) __stcs(alpha + o, s.alpha);
            if (want_rgb) { __stcs(rgb + o, s.r); __stcs(rgb + o + plane, s.g); __stcs(rgb + o + 2 * plane, s.b); }
            sr += s.r; sg += s.g; sb += s.b; sa += s.alpha; sd += s.depth;
        }
        const uint32_t oo = (uint32_t)orow * H + col;
        if (want_rgb && p.out_rgb) {
            float* orgb = p.out_rgb + (size_t)b * 3 * oplane + oo;
            orgb[0] = sr * 0.25f; orgb[oplane] = sg * 0.25f; orgb[2 * oplane] = sb * 0.25f;
        }
        if (p.out_alpha) p.out_alpha[(size_t)b * oplane + oo] = sa * 0.25f;
        if (p.out_depth) p.out_depth[(size_t)b * oplane + oo] = sd * 0.25f;
    }
}

inline float float_ge(double d) {  // smallest float >= d
    float f = (float)d;
    if ((double)f < d) f = nextafterf(f, INFINITY);
    return f;
}

struct FwdLayout {
    size_t off_cnt, off_zbuf, off_tab, off_list, off_z0, total;
};
// workspace = big-face counters | z-buffer (one memset covers both) | face records | big-face lists
FwdLayout fwd_layout(int B, int F, int S) {
    FwdLayout L{};
    L.off_cnt = 0;  // [B] big-face counters, then work_next, any_big
    L.off_zbuf = nr_align_up((size_t)(B + 2) * sizeof(int), 256);
    L.off_tab = L.off_zbuf + nr_align_up((size_t)B * S * S * sizeof(unsigned long long), 256);
    L.off_list = L.off_tab + nr_align_up((size_t)B * F * kRecWords * sizeof(float), 256);
    L.off_z0 = L.off_list + nr_align_up((size_t)B * F * sizeof(int), 256);
    L.total = L.off_z0 + nr_align_up((size_t)F * sizeof(float4), 256);
    return L;
}

// one k_resolve launch (the shared-memory opt-in is a static of each instantiation)
template <bool kAA, int kTex, int kLight>
int launch_resolve(const FwdParams& p, dim3 grid, int bx, size_t smem, int nslots, cudaStream_t stream) {
    static nr_internal::SmemOptIn optin;
    if (optin.ensure(k_resolve<kAA, kTex, kLight>, smem) != cudaSuccess) return NR_ERR_CUDA;
    k_resolve<kAA, kTex, kLight><<<grid, bx, smem, stream>>>(p, nslots);
    return NR_OK;
}

}  // namespace

extern "C" size_t nr_b200_forward_workspace_bytes(int32_t B, int32_t F, int32_t S, int32_t ts, uint32_t flags) {
    (void)ts; (void)flags;
    if (B <= 0 || F <= 0 || S <= 0) return 16;
    return fwd_layout(B, F, S).total;
}

// nr_b200_forward (no Phong inputs) and the five Phong entry points
static int forward_impl(const nr_b200_forward_args* args, const nr_internal::PhongCall& pc, void* cuda_stream) {
    nr_internal::launch_count() = 0;
    // Two layouts: the full struct, and the ABI-4 struct from before corner_light (which then reads as NULL).  Only the
    // caller's struct_size bytes are read.
    if (!args) return NR_ERR_INVALID_ARG;
    const uint32_t size = args->struct_size;
    if (size != sizeof(nr_b200_forward_args) && size != offsetof(nr_b200_forward_args, corner_light)) return NR_ERR_INVALID_ARG;
    nr_b200_forward_args args_copy;
    memset(&args_copy, 0, sizeof(args_copy));
    memcpy(&args_copy, args, size);
    const nr_b200_forward_args* a = &args_copy;
    const int B = a->batch_size, F = a->num_faces, S = a->raster_size, ts = a->texture_size;
    const uint32_t flags = a->flags;
    if (B <= 0 || F <= 0 || S <= 0) return NR_ERR_INVALID_ARG;
    if (!(flags & (NR_RETURN_RGB | NR_RETURN_ALPHA | NR_RETURN_DEPTH))) return NR_ERR_INVALID_ARG;  // rasterize.py:25-27
    if (!a->face_index_map || !a->weight_map || !a->depth_map) return NR_ERR_INVALID_ARG;
    nr::FaceSrc src{};
    if (!nr_internal::make_face_src(flags, a->faces, a->vertices, a->face_indices, F, a->num_vertices, &src)) return NR_ERR_INVALID_ARG;
    const bool uv = (flags & NR_TEX_UV) != 0, mip = (flags & NR_TEX_MIPMAP) != 0;
    if ((flags & NR_RETURN_RGB) && (!a->textures || !a->rgb_map || ((flags & NR_BG_PER_BATCH) && !a->background_batch)))
        return NR_ERR_INVALID_ARG;
    nr::Texture tex;
    size_t tex_floats, uv_floats;
    const int tex_rc = nr_internal::make_texture(a, &tex, &tex_floats, &uv_floats);
    if (tex_rc == NR_ERR_INVALID_ARG) return tex_rc;
    nr::Shading shading;
    const int light = nr_internal::make_shading((flags & NR_RETURN_RGB) != 0, a->face_light, a->corner_light, pc, B, F, &shading);
    if (light < 0) return NR_ERR_INVALID_ARG;
    const nr_b200_normal_map_args* nm = pc.nm;
    const nr_b200_specular_map_args* sm = pc.sm;
    if ((nm || sm) && !uv) return NR_ERR_INVALID_ARG;  // the maps are addressed by the pixel's uv
    if ((flags & NR_ANTI_ALIASING) && (S & 1)) return NR_ERR_INVALID_ARG;
    if (S > 32767 || B > 65535) return NR_ERR_UNSUPPORTED;  // 32-bit pixel offsets; batch = grid.z of the resolve pass
    if (tex_rc != NR_OK) return tex_rc;  // 32-bit image / UV offsets
    if (nm && nr_internal::nm_floats(nm) * (size_t)nm->map_batch > 0x7FFFFFFFull) return NR_ERR_UNSUPPORTED;  // 32-bit map offsets
    if (sm && nr_internal::sm_floats(sm) * (size_t)sm->map_batch > 0x7FFFFFFFull) return NR_ERR_UNSUPPORTED;
    const size_t need = nr_b200_forward_workspace_bytes(B, F, S, ts, flags);
    if (!a->workspace || a->workspace_bytes < need || ((uintptr_t)a->workspace & 15)) return NR_ERR_WORKSPACE;
    cudaStream_t stream = (cudaStream_t)cuda_stream;
    const FwdLayout L = fwd_layout(B, F, S);
    char* wsb = (char*)a->workspace;

    FwdParams p{};
    p.src = src;
    p.tex = tex;
    p.bg_batch = a->background_batch;
    p.shading = shading;
    p.big_cnt = (int*)(wsb + L.off_cnt);
    p.work_next = p.big_cnt + B;
    p.any_big = p.big_cnt + B + 1;
    p.zbuf = (unsigned long long*)(wsb + L.off_zbuf);
    p.tab = (float4*)(wsb + L.off_tab);
    p.big_list = (int*)(wsb + L.off_list);
    p.z0tab = ((flags & NR_RETURN_RGB) && (flags & NR_TEX_Z_BATCH0) && !uv) ? (float4*)(wsb + L.off_z0) : nullptr;
    p.fim = a->face_index_map; p.wmap = a->weight_map; p.dmap = a->depth_map; p.rgb = a->rgb_map; p.alpha = a->alpha_map;
    p.out_rgb = a->out_rgb; p.out_alpha = a->out_alpha; p.out_depth = a->out_depth;
    p.B = B; p.F = F; p.S = S; p.ts = ts; p.ngroups = (F + 31) / 32;
    p.big_area = S > 256 ? 4 * kBigArea : kBigArea;
    // the background only colours the RGB image: without NR_RETURN_RGB, background_batch is neither checked above nor
    // read (it may be NULL), so the resolve pass must not see NR_BG_PER_BATCH either
    p.flags = (flags & NR_RETURN_RGB) ? flags : (flags & ~NR_BG_PER_BATCH);
    p.near_lo = nr_internal::float_le(a->near_);
    p.far_cmp = fminf(float_ge(a->far_), (float)a->far_);
    p.far_val = (float)a->far_;
    p.bg[0] = a->background[0]; p.bg[1] = a->background[1]; p.bg[2] = a->background[2];

    {   // z-buffer = "empty" (~0), big-face counters = -1: one fill
        nr_internal::prof_begin("memset_zbuf", stream);
        if (cudaMemsetAsync(wsb, 0xFF, L.off_tab, stream) != cudaSuccess) return NR_ERR_CUDA;
        nr_internal::prof_end(stream);
    }
    const size_t centres_bytes = S <= kXpTable ? (size_t)S * sizeof(float) : 0;
    int dev = 0, sms = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess)
        return NR_ERR_CUDA;
    {
        const size_t smem = sizeof(WarpScratch) * kFaceWarps + centres_bytes;
        static nr_internal::SmemOptIn optin;
        if (optin.ensure(k_raster_faces, smem) != cudaSuccess) return NR_ERR_CUDA;
        int per_sm = 0;
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_raster_faces, kFaceWarps * 32, smem) != cudaSuccess || per_sm < 1)
            per_sm = 1;
        const long long nunits = (long long)B * p.ngroups;
        const int grid = (int)std::min<long long>((nunits + kFaceWarps - 1) / kFaceWarps, (long long)sms * per_sm);
        nr_internal::LaunchScope ls("k_raster_faces", stream);
        k_raster_faces<<<grid, kFaceWarps * 32, smem, stream>>>(p);
    }
    {
        const size_t smem = sizeof(WarpScratch) * 8 + centres_bytes;
        static nr_internal::SmemOptIn optin;
        if (optin.ensure(k_raster_big, smem) != cudaSuccess) return NR_ERR_CUDA;
        const int tiles = (S + kBigTile - 1) / kBigTile;
        const int grid = (int)std::min<long long>((long long)tiles * tiles * B, (long long)sms * 4);
        nr_internal::LaunchScope ls("k_raster_big", stream);
        k_raster_big<<<grid, 256, smem, stream>>>(p);
    }
    {
        nr_internal::LaunchScope ls("k_resolve", stream);
        const int width = (flags & NR_ANTI_ALIASING) ? S / 2 : S;   // one thread per API pixel
        int bx = width >= 256 ? 256 : ((width + 31) / 32) * 32;     // staged variant: a CTA = one row segment
        dim3 grid((width + bx - 1) / bx, width, B);
        // Staging whole cubes with cp.async.bulk needs 16-byte aligned, 16-byte sized cubes; up to kStageBytes of
        // shared memory per CTA hold the cubes of the row's runs (the rest of the runs read global memory)
        const bool aa = (flags & NR_ANTI_ALIASING) != 0;
        const uint32_t cube_bytes = (flags & NR_RETURN_RGB) ? (uint32_t)(ts * ts * ts) * 12u : 0u;
        const bool stage = !uv && light <= nr::kLightFace && (flags & NR_FWD_STAGE_TEXTURES) && !aa && (flags & NR_RETURN_RGB) &&
                           (cube_bytes % 16u) == 0 && cube_bytes <= kStageBytes / 8 && ((uintptr_t)a->textures & 15) == 0;
        int nslots = 0;
        size_t smem = 0;
        if (stage) {
            nslots = (int)std::min<uint32_t>(kStageBytes / cube_bytes, (uint32_t)bx);
            smem = (size_t)nslots * cube_bytes;
        } else if (!aa) {  // direct variant: 32 x 8 pixel tiles
            bx = 256;
            grid = dim3((width + kResolveTileW - 1) / kResolveTileW, (width + kResolveTileH - 1) / kResolveTileH, B);
        }
        int rc;
        if (stage) {
            rc = nr::dispatch_light<nr::kLightNone, nr::kLightFace>(
                light, [&](auto kL) { return launch_resolve<false, 1, kL>(p, grid, bx, smem, nslots, stream); });
        } else {
            rc = nr::dispatch_bool(aa, [&](auto kAA) {
                return nr::dispatch_light<nr::kLightNone, nr::kLightFace, nr::kLightCorner, nr::kLightPhong, nr::kLightPhongSet,
                                          nr::kLightPhongSH, nr::kLightPhongNM, nr::kLightPhongSM>(light, [&](auto kL) {
                    if constexpr (kL >= nr::kLightPhongNM) {  // NR_TEX_UV only
                        return mip ? launch_resolve<kAA, 3, kL>(p, grid, bx, smem, nslots, stream)
                                   : launch_resolve<kAA, 2, kL>(p, grid, bx, smem, nslots, stream);
                    } else {
                        return mip  ? launch_resolve<kAA, 3, kL>(p, grid, bx, smem, nslots, stream)
                               : uv ? launch_resolve<kAA, 2, kL>(p, grid, bx, smem, nslots, stream)
                                    : launch_resolve<kAA, 0, kL>(p, grid, bx, smem, nslots, stream);
                    }
                });
            });
        }
        if (rc != NR_OK) return rc;
    }
    return cudaGetLastError() == cudaSuccess ? NR_OK : NR_ERR_CUDA;
}

extern "C" int nr_b200_forward(const nr_b200_forward_args* args, void* cuda_stream) {
    return forward_impl(args, {}, cuda_stream);
}

extern "C" int nr_b200_forward_phong(const nr_b200_forward_args* args, const nr_b200_phong_args* phong, void* cuda_stream) {
    return phong ? forward_impl(args, {phong}, cuda_stream) : nr_internal::refuse_null_phong();
}

extern "C" int nr_b200_forward_lights(const nr_b200_forward_args* args, const nr_b200_phong_args* phong,
                                      const nr_b200_lights_args* lights, void* cuda_stream) {
    return phong ? forward_impl(args, {phong, lights}, cuda_stream) : nr_internal::refuse_null_phong();
}

extern "C" int nr_b200_forward_sh(const nr_b200_forward_args* args, const nr_b200_phong_args* phong,
                                  const nr_b200_lights_args* lights, const nr_b200_sh_args* sh, void* cuda_stream) {
    return phong ? forward_impl(args, {phong, lights, sh}, cuda_stream) : nr_internal::refuse_null_phong();
}

extern "C" int nr_b200_forward_normal_map(const nr_b200_forward_args* args, const nr_b200_phong_args* phong,
                                          const nr_b200_lights_args* lights, const nr_b200_sh_args* sh,
                                          const nr_b200_normal_map_args* nm, void* cuda_stream) {
    return phong ? forward_impl(args, {phong, lights, sh, nm}, cuda_stream) : nr_internal::refuse_null_phong();
}

extern "C" int nr_b200_forward_specular_map(const nr_b200_forward_args* args, const nr_b200_phong_args* phong,
                                            const nr_b200_lights_args* lights, const nr_b200_sh_args* sh,
                                            const nr_b200_normal_map_args* nm, const nr_b200_specular_map_args* sm,
                                            void* cuda_stream) {
    return phong ? forward_impl(args, {phong, lights, sh, nm, sm}, cuda_stream) : nr_internal::refuse_null_phong();
}
