/*
 * nr_b200.h -- C ABI of the H100-native (sm_90a) differentiable mesh rasterizer.
 *
 * This is the drop-in boundary for the hot path of hiroharu-kato/neural_renderer:
 * the `Rasterize` function object (neural_renderer/rasterize.py:19-897) and the
 * post-processing owned by `rasterize_rgbad` (rasterize.py:945-969).  The
 * reference has no FFI of its own -- CuPy hands raw device pointers to
 * JIT-compiled kernels (`chainer.cuda.elementwise(...)(arrays)`,
 * rasterize.py:236, :277, :359, :435, :745, :789, :844) -- so the entry points
 * below are what a binding for that path would call instead:
 *
 *   nr_b200_forward    replaces Rasterize.forward_gpu   (rasterize.py:467-513: K1 :242, K2 :281, K4 :372,
 *                      alpha/background :440-465) fused with the transpose / vertical flip / 2x2 average
 *                      pooling of rasterize_rgbad (rasterize.py:953-969)
 *   nr_b200_backward   replaces Rasterize.backward_gpu  (rasterize.py:849-889: K5 :528, K6 :760, K7 :805)
 *                      fused with the backward of that same post-processing
 *
 * Conventions
 *   - plain C, no C++/torch types; every pointer is a DEVICE pointer owned by the caller (torch allocator,
 *     cudaMalloc, ...) unless it says "host"; the stream is a cudaStream_t passed as void*; launches are
 *     asynchronous on that stream; nothing is allocated behind the caller's back (scratch = explicit workspace);
 *   - return value 0 = NR_OK, negative = error (nr_b200_error_string); never throws, no global state, re-entrant;
 *   - all images are planar, row-major, in IMAGE orientation: row 0 is the TOP row (the reference's
 *     `[:, ::-1, :]` flip is folded in), i.e. raster row yi (NDC y up) is stored at row S-1-yi;
 *   - S = raster size = image_size, or 2*image_size with NR_ANTI_ALIASING (then the API images are the 2x2
 *     means, size S/2, and the raster-resolution maps are still written because the backward needs them);
 *   - float32 / int32 throughout, C-contiguous.
 */
#ifndef NR_B200_H_
#define NR_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define NR_B200_ABI_VERSION 4

#if defined(__GNUC__)
#define NR_B200_API __attribute__((visibility("default")))
#else
#define NR_B200_API
#endif

/* error codes */
#define NR_OK 0
#define NR_ERR_INVALID_ARG (-1)
#define NR_ERR_WORKSPACE (-2)
#define NR_ERR_CUDA (-3)
#define NR_ERR_UNSUPPORTED (-4)

/* flags */
#define NR_RETURN_RGB 1u      /* Rasterize(return_rgb=True): needs textures                                   */
#define NR_RETURN_ALPHA 2u    /* Rasterize(return_alpha=True)                                                   */
#define NR_RETURN_DEPTH 4u    /* Rasterize(return_depth=True)                                                   */
#define NR_ANTI_ALIASING 8u   /* rasterize_rgbad(anti_aliasing=True): raster_size = 2 * image_size            */
#define NR_BG_PER_BATCH 16u   /* background_color given as [B,3] (rasterize.py:464-465) in `background_batch`  */
#define NR_TEX_Z_BATCH0 32u   /* reproduce rasterize.py:389: the texture sampler reads vertex depths of batch  */
                              /* item 0 (reference-exact; clear it for per-item depths)                        */
#define NR_GRAD_ACCUMULATE 64u /* backward: add into grad_faces | grad_vertices, grad_textures, grad_face_light    */
                               /* instead of zero-filling them first (also for each call of a two-part backward) */
#define NR_TEX_FILL_BACK 0x400u /* Renderer.fill_back without materialising the doubled texture tensor            */
                                /* (renderer.py:78-80): F is even, faces [F/2, F) are the reversed copies of      */
                                /* [0, F/2); `textures` / `grad_textures` hold F/2 cubes and face f >= F/2 samples */
                                /* cube f - F/2 with its three texture axes reversed (permute(0,1,4,3,2,5))        */

/* ABI 3 */
#define NR_FACES_INDEXED 0x800u   /* geometry is `vertices` [B,Nv,3] + `face_indices` (vertices_to_faces.py:16-21 folded   */
                                  /* into the rasterizer): `faces` is ignored, no [B,F,3,3] tensor exists on either pass;   */
                                  /* the backward scatters d loss / d vertex straight into `grad_vertices`                  */
#define NR_INDICES_SHARED 0x1000u /* face_indices is [F,3] and serves every batch item (else [B,F,3])                       */
#define NR_TEX_SHARED 0x2000u     /* ONE set of texture cubes [F,ts,ts,ts,3] serves every batch item (a shared mesh seen   */
                                  /* from B viewpoints, mesh.py:29-34); grad_textures [F,...] is the sum over the items     */
#define NR_BWD_PART_TEXTURES 0x4000u /* backward: only the part that produces grad_textures / grad_face_light (K6)         */
#define NR_BWD_PART_FACES 0x8000u    /* backward: only the part that produces grad_faces / grad_vertices (K5, K7)           */
                                     /* neither bit = both parts; a caller that wants to start a collective on the texture   */
                                     /* gradient while the edge scan runs calls TEXTURES first, then FACES                   */

#define NR_FWD_STAGE_TEXTURES 0x10000u /* forward, RGB without anti-aliasing: stage the texture cubes of every pixel row in     */
                                       /* shared memory with bulk asynchronous copies (cp.async.bulk / TMA, one mbarrier per CTA)  */
                                       /* before sampling.  Same pixels; measured SLOWER than the direct gather on H100            */
                                       /* (DESIGN.md section 4), hence opt-in.  Ignored when the cube size is not a multiple of   */
                                       /* 16 bytes or `textures` is not 16-byte aligned.                                           */

/* ABI 4: UV-mapped texture image instead of per-face cubes.
 *   `textures` / `grad_textures` are the image [Bt,Ht,Wt,3] float32, HWC, row 0 = TOP row (as a PNG is read); Bt = B, or
 *   1 with NR_TEX_SHARED (one image for every item; its gradient is the sum over the items).  `face_uvs` holds the UV of
 *   every face corner, OBJ convention (v = 0 is the BOTTOM of the image).  texture_size is ignored.
 *   Covered pixel with winner weights w_k, depth zp and the winner's OWN vertex depths z_k (NR_TEX_Z_BATCH0 has no
 *   effect on this sampler):  l_k = w_k * (zp / z_k)  (div.rn),  uv = l_0 uv_0 + l_1 uv_1 + l_2 uv_2  (not renormalised).
 *   Addressing as nr_b200_bake_textures: u, v clamped into [0,1] (NaN -> 0), pos_x = u (Wt-1), pos_y = v (Ht-1); taps
 *   ix, ix+1 / iy, iy+1 (clamped into the image; tap row iy is image row Ht-1-iy); bilinear weights products of frac and
 *   1 - frac; fp32, round-to-nearest; clamp to edge only (no wrap; NR_TEX_MIPMAP below samples a mip pyramid
 *   trilinearly instead).  face_light multiplies every tap first.
 *   With NR_TEX_FILL_BACK face f >= F/2 uses the UV corners of face f - F/2 in reverse order (`face_uvs` holds F/2 faces).
 *   The backward fills grad_textures (the image gradient), grad_face_light and, when given, grad_face_uvs:
 *   d loss / d face_uvs (nr_b200_backward_args.grad_face_uvs).  For a covered raster pixel with the winner's UV corners
 *   uv_k (reversed for a fill_back copy, as above), l_k as above, fp32 uv = (u, v) and upstream rgb gradient g_c (the
 *   pooled gradient / 4 with NR_ANTI_ALIASING): per sampled level l with weight a_l (bilinear: level 0, a = 1; NR_TEX_MIPMAP:
 *   l0 with 1 - f and, only when f != 0, l1 with f) and the taps T_xy of that level's addressing (tap (x, y), y up, so T_01
 *   is image row r1), each times face_light:
 *     Dx_c = (W_l - 1) (wy0 (T10 - T00) + wy1 (T11 - T01)),   Dy_c = (H_l - 1) (wx0 (T01 - T00) + wx1 (T11 - T10)),
 *     gu = [0 <= u <= 1] sum_l a_l sum_c g_c Dx_c,   gv = [0 <= v <= 1] sum_l a_l sum_c g_c Dy_c   (NaN u / v: 0),
 *     grad_face_uvs[corner k] += (l_k gu, l_k gv)
 *   (a fill_back copy f >= F/2 adds into face f - F/2, its corner k being that face's corner 2 - k; with NR_UV_SHARED the
 *   sum over the items).  This is the derivative of the bilinear sample within the cell the forward picked: the level of
 *   detail, l_k and the clamp are held fixed, a 1-texel axis gets 0.  fp32, not bit-pinned (unordered atomics).
 *   No vertex gradient flows through l_k unless NR_GRAD_INTERIOR (below). */
#define NR_TEX_UV 0x20000u    /* sample a texture image through per-corner UVs (fields face_uvs / texture_height / _width) */
#define NR_UV_SHARED 0x40000u /* face_uvs is [F,3,2] and serves every batch item (else [B,F,3,2])                        */

/* Trilinear sampling through a mip pyramid (additive to ABI 4: a flag bit and three entry points, no struct field).
 *   Only together with NR_TEX_UV.  `textures` is then the PACKED PYRAMID [Bt,P,3]: level 0 (the image, Ht x Wt), then
 *   level 1, 2, ... in order, each HWC with row 0 = top; `grad_textures` is the gradient of that pyramid (collapse it into
 *   the image with nr_b200_mip_collapse); grad_face_uvs is the face_uvs gradient (NR_TEX_UV above, through both
 *   levels).  texture_height / texture_width stay the level-0 size.
 *   Level sizes: H_{l+1} = max(1, (H_l + 1) >> 1), the same for W, until both are 1: L = 1 + ceil(log2(max(Ht, Wt)))
 *   levels, P = sum_l H_l W_l texels (nr_b200_mip_texels).  A 1x1 image has one level (trilinear = bilinear).
 *   Building (nr_b200_mip_build), in tap coordinates (x right, y up from the bottom row, row r = H_l-1-y): texel (x, y)
 *   of level l+1 = ((a + b) + (c + d)) * 0.25 (fp32, round-to-nearest) with a, b = level-l taps (2x, 2y), (2x+1, 2y) and
 *   c, d = (2x, 2y+1), (2x+1, 2y+1), each clamped into level l (the edge texel of an odd or 1-texel axis counts twice).
 *   Level of detail per covered raster pixel (raster pixels; anti-aliasing pools on top): with the winner's K1 inverse
 *   inv[9], weights w, depth zp and own vertex depths z_k,  l_k = w_k zp / z_k,
 *   d l_k / dx = zp (inv[3k] / z_k - l_k sum_j inv[3j] / z_j)  (y: inv[3k+1]),  du/dx = sum_k u_k d l_k / dx (v, y alike;
 *   evaluated as sum_{k=1,2} (u_k - u_0) d l_k / dx, equal because sum_k d l_k / dx = 0, without the fp32 cancellation
 *   of UV corners that lie close together far from 0),
 *   rho^2 = max(((Wt-1) du/dx)^2 + ((Ht-1) dv/dx)^2, the same in y),  lod = 0.5 log2(rho^2) clamped into [0, L-1]
 *   (NaN and -inf -> 0).  The derivative ignores the [0,1] clamp of u, v and the clamping of the weights.
 *   Sample: l0 = floor(lod), l1 = min(l0+1, L-1), f = lod - l0; rgb = (1-f) bilinear_l0 + f bilinear_l1, each level with
 *   the NR_TEX_UV addressing at its own size; face_light multiplies every tap first; level l1 is not read when f == 0.
 *   The backward sends (1-f or f) * tap weight * light * grad_rgb to each tap of the pyramid and grad_face_light gets the
 *   unlit trilinear sample times the upstream gradient.  NO gradient flows through the LOD. */
#define NR_TEX_MIPMAP 0x80000u /* textures = packed mip pyramid of the image, sampled trilinearly (needs NR_TEX_UV)        */

/* Smooth (Gouraud) shading, additive to ABI 4: the field corner_light appended to nr_b200_forward_args, and the backward
 * entry point nr_b200_backward_corner_light, which takes the same corner_light (the backward struct is unchanged).
 *   corner_light [B,F,3,3] is an RGB light factor at each corner k of face f, corners in the face's own order (the order
 *   of `faces` / `face_indices`); as with face_light, F counts the fill_back copies as faces of their own.  Per item only.
 *   A non-NULL corner_light needs NR_RETURN_RGB and excludes face_light (else NR_ERR_INVALID_ARG).
 *   Covered raster pixel with winner weights w_k, depth zp and the winner's OWN vertex depths z_k (NR_TEX_Z_BATCH0 has no
 *   effect on this):  l_k = w_k * (zp / z_k)  (div.rn, the l_k of NR_TEX_UV), and per channel c
 *     L_c = fma(l_2, C_2c, fma(l_1, C_1c, l_0 * C_0c)),   rgb_c = L_c * s_c  (fp32, round-to-nearest)
 *   where s is the UNLIT sample exactly as the unlit path computes it (ts^3 cube, bilinear image or trilinear pyramid):
 *   the light multiplies after the blend, not per tap.  The background is not lit; anti-aliasing pools on top as before.
 *   NR_FWD_STAGE_TEXTURES is ignored with corner_light.
 *   Backward (nr_b200_backward_corner_light), texture half: grad_textures as without light, with d rgb_c / d s_c = L_c in place of face_light; grad_face_uvs
 *   likewise uses L_c; grad_corner_light[b,f,k,c] += l_k * g_c * s_c (zero-filled first unless NR_GRAD_ACCUMULATE; needs
 *   corner_light and `textures`).  No vertex gradient flows through l_k unless NR_GRAD_INTERIOR (below): without it
 *   grad_faces / grad_vertices are those of the unchanged edge scan (which reads the smooth-shaded rgb map) and depth
 *   gradient.  fp32 atomics, not bit-pinned. */

/* Interior vertex gradient of the RGB image, additive to ABI 4: one backward flag, honoured by nr_b200_backward and
 * nr_b200_backward_corner_light (no struct field, no entry point, no workspace).  Without it the face / vertex gradient is
 * the reference's (edge scan K5 + depth K7), bit for bit as before.  With it, the faces half (NR_BWD_PART_FACES) also adds
 * the derivative of the colour INSIDE each face through the perspective weights: K5 covers the coverage changes, this term
 * the colour changes at fixed coverage, so nothing is counted twice.
 *   Covered raster pixel: winner fn, saved weights w_k, the winner's OWN camera depths z_k (also for cubes), zp recomputed
 *   as the forward does, l_k = w_k (zp / z_k) (nr::perspective_weights), upstream g_c (the pooled gradient / 4 with
 *   NR_ANTI_ALIASING).  L_c = face_light_c, 1 when unlit, or the corner_light interpolant (smooth shading).  s_c = the unlit
 *   sample.  E_kc = d s_c / d l_k with the cell, the level of detail and the clamps held fixed:
 *     cubes:     E_kc = [0 <= t_k <= ts-1-eps] (ts-1) dS_c/dt_k, t_k the unclamped texture coordinate of the sampler, and
 *                dS_c/dt_k = sum over the 4 corner pairs along axis k of (T_hi - T_lo) times the other two axes' weights,
 *                in the cell the forward picked (addressing as the forward, reversed axes for a NR_TEX_FILL_BACK copy);
 *     bilinear:  E_kc = Du_c u_k + Dv_c v_k with Du, Dv the d sample / d (u, v) of NR_TEX_UV above (clamp gates in_u / in_v
 *                and the (W-1) / (H-1) scales included), uv_k the (for a fill_back copy reversed) UV corners;
 *     trilinear: sum_l a_l (Du_c^l u_k + Dv_c^l v_k) over the one or two levels the forward read (none through the LOD).
 *   G_k = sum_c g_c (L_c E_kc + [smooth] C_kc s_c) = d loss / d l_k, and the chain of nr_b200_interpolate_backward:
 *     D_k = G_k - G_0 (k = 1, 2; images and corner light from corner differences (uv_k - uv_0), (C_k - C_0)),
 *     Gx = D_1 lx_1 + D_2 lx_2, Gy alike (lx_k, ly_k = d l_k / d (x, y) in raster pixels, as there),
 *     P_m = sum_k l_k G_k - G_m (images: gu (u - u_m) + gv (v - v_m) with the pixel's uv; light: sum_c g_c s_c (L_c - C_mc)),
 *     grad x_m += -w_m Gx S/2,   grad y_m += -w_m Gy S/2,   grad z_m += (l_m / z_m) P_m,
 *   with the weights' clamp and renormalisation held fixed, as K7.  fp32 atomics, not bit-pinned.
 *   Needs NR_RETURN_RGB and `textures` (the image / pyramid for NR_TEX_UV); per-face cubes with NR_TEX_Z_BATCH0 at B > 1
 *   (whose sampler reads the depths of item 0, so the derivative would cross items) are refused: NR_ERR_INVALID_ARG
 *   before any launch.  It runs only when grad_rgb is given; the texture half and its outputs are unchanged.
 *   NR_GRAD_ACCUMULATE and the short struct layouts behave as without it. */
#define NR_GRAD_INTERIOR 0x400000u

typedef struct nr_b200_forward_args {
    uint32_t struct_size; /* sizeof(nr_b200_forward_args), or offsetof(.., corner_light) (see there) */
    uint32_t flags;
    int32_t batch_size;   /* B */
    int32_t num_faces;    /* F */
    int32_t raster_size;  /* S (already doubled when NR_ANTI_ALIASING) */
    int32_t texture_size; /* ts (>= 2) when NR_RETURN_RGB, else ignored */
    double near_;         /* reject zp <= near   (compared in double, like the pasted literal, rasterize.py:331) */
    double far_;          /* reject far <= zp; uncovered depth = (float)far (rasterize.py:296, :480)             */
    double eps;           /* texture-coordinate clamp `ts - 1 - eps` (rasterize.py:402)                          */
    float background[3];  /* uniform background colour (host values)                                             */
    float _pad0;
    const float *faces;            /* [B,F,3,3]  x,y in NDC [-1,1], z = camera depth                            */
    const float *textures;         /* [B,F,ts,ts,ts,3] ([F,...] with NR_TEX_SHARED) or NULL                     */
    const float *background_batch; /* [B,3] device, only with NR_BG_PER_BATCH; read only with NR_RETURN_RGB     */
    /* raster-resolution maps, saved for the backward pass (all required unless noted) */
    int32_t *face_index_map; /* [B,S,S]   -1 where empty                                                      */
    float *weight_map;       /* [B,3,S,S] barycentric weights of the winning face, 0 where empty              */
    float *depth_map;        /* [B,S,S]   zp, (float)far where empty; IS the depth image when !ANTI_ALIASING  */
    float *rgb_map;          /* [B,3,S,S] post-background colour; required with NR_RETURN_RGB; IS the rgb     */
                             /*           image when !ANTI_ALIASING                                           */
    float *alpha_map;        /* [B,S,S]   0/1; optional (NULL ok); IS the alpha image when !ANTI_ALIASING     */
    /* API images at S/2, only with NR_ANTI_ALIASING (each may be NULL if not wanted) */
    float *out_rgb;   /* [B,3,S/2,S/2] */
    float *out_alpha; /* [B,S/2,S/2]   */
    float *out_depth; /* [B,S/2,S/2]   */
    void *workspace; /* nr_b200_forward_workspace_bytes() bytes, 16-byte aligned */
    size_t workspace_bytes;
    /* ABI 2: per-face RGB light factor of lighting.py:29-52 applied at sample time -- every texel is multiplied by
     * face_light[b,f,:] before the trilinear blend, bit-identical to sampling the materialised `textures * light`
     * product (lighting.py:52).  NULL = unlit. */
    const float *face_light; /* [B,F,3] or NULL */
    /* ABI 3: indexed geometry, only with NR_FACES_INDEXED (then `faces` may be NULL).  Indices outside [0, Nv) read
     * a vertex of zeros, like nr_b200_vertices_to_faces. */
    const float *vertices;       /* [B,Nv,3] x,y in NDC, z = camera depth */
    const int32_t *face_indices; /* [B,F,3], or [F,3] with NR_INDICES_SHARED */
    int32_t num_vertices;        /* Nv */
    int32_t _pad1;
    /* ABI 4: texture image, only with NR_TEX_UV (then `textures` is the image [Bt,Ht,Wt,3]) */
    const float *face_uvs;  /* [B,F,3,2], or [F,3,2] with NR_UV_SHARED (F/2 faces with NR_TEX_FILL_BACK) */
    int32_t texture_height; /* Ht >= 1 */
    int32_t texture_width;  /* Wt >= 1 */
    /* ABI 4, appended: smooth shading (above).  struct_size may also be offsetof(nr_b200_forward_args, corner_light), the
     * layout before this field, which then reads as NULL.  Only struct_size bytes are read. */
    const float *corner_light; /* [B,F,3,3] or NULL */
} nr_b200_forward_args;

typedef struct nr_b200_backward_args {
    uint32_t struct_size; /* sizeof(nr_b200_backward_args), or offsetof(nr_b200_backward_args, grad_face_uvs): the ABI-4
                             layout before that field, which then reads as NULL.  Only struct_size bytes are read. */
    uint32_t flags; /* same flag set as the forward call that produced the maps */
    int32_t batch_size, num_faces, raster_size, texture_size;
    double eps; /* edge-distance epsilon (rasterize.py:650) and texture clamp epsilon -- the reference uses one value */
    const float *faces;    /* [B,F,3,3] as given to the forward call */
    const float *textures; /* may be NULL: only its shape matters for the backward pass */
    const int32_t *face_index_map; /* saved maps from nr_b200_forward */
    const float *weight_map;
    const float *depth_map;
    const float *rgb_map;
    /* upstream gradients in API layout (size S, or S/2 with NR_ANTI_ALIASING); NULL = zeros */
    const float *grad_rgb;   /* [B,3,H,W] */
    const float *grad_alpha; /* [B,H,W]   */
    const float *grad_depth; /* [B,H,W]   */
    float *grad_faces;    /* [B,F,3,3]                 */
    float *grad_textures; /* [B,F,ts,ts,ts,3] ([B,F/2,...] with NR_TEX_FILL_BACK, no B with NR_TEX_SHARED) or NULL */
    void *workspace;
    size_t workspace_bytes;
    /* ABI 2: lighting folded into the sampler.  grad_textures receives the gradient of the UNLIT textures
     * (weights scaled by face_light); grad_face_light [B,F,3] (may be NULL) receives sum over pixels of
     * grad_rgb * unlit sample and needs `textures`. */
    const float *face_light; /* [B,F,3] as given to the forward call, or NULL */
    float *grad_face_light;  /* [B,F,3] or NULL */
    /* ABI 3: indexed geometry as in the forward call; with NR_FACES_INDEXED the face gradient is reduced into
     * grad_vertices [B,Nv,3] (zero-filled first unless NR_GRAD_ACCUMULATE); grad_faces is then neither read nor written
     * and may be NULL. */
    const float *vertices;
    const int32_t *face_indices;
    float *grad_vertices; /* [B,Nv,3] */
    int32_t num_vertices;
    int32_t _pad1;
    /* ABI 4: as in the forward call; with NR_TEX_UV grad_textures is the image gradient [Bt,Ht,Wt,3] */
    const float *face_uvs;
    int32_t texture_height;
    int32_t texture_width;
    /* ABI 4, appended: d loss / d face_uvs [B,F',3,2], or [F',3,2] with NR_UV_SHARED (F' = F/2 with NR_TEX_FILL_BACK), or
     * NULL = not wanted.  Needs NR_TEX_UV, NR_RETURN_RGB and `textures`.  Part of the texture half
     * (NR_BWD_PART_TEXTURES): zero-filled first unless NR_GRAD_ACCUMULATE; stays zero without grad_rgb. */
    float *grad_face_uvs;
} nr_b200_backward_args;

/* Phong shading, additive to ABI 4: one struct (nr_b200_phong_args), two entry points (nr_b200_forward_phong /
 * nr_b200_backward_phong) and a glue pair (nr_b200_corner_shading / _backward).  Ambient + diffuse + specular evaluated at
 * every pixel from a normal and a position interpolated per pixel; the forward and backward structs are unchanged.
 *   corner_shading [Bc,F,3,6]: per face corner k (the face's own order; F counts fill_back copies, which the caller gives
 *   their corners with the normal negated) the shading normal N_k (3 floats), then the shading position P_k (3 floats).
 *   params [Bp,16] (device): A[3] ambient intensity * colour, D[3] directional intensity * colour, d[3] light direction
 *   (towards the light, not normalised, as for face_light), K[3] specular intensity * colour, sigma the shininess, e[3] the
 *   eye position in the frame of P and N.  Bc, Bp in {1, B}; 1 = one set for every item (its gradient is the sum over the
 *   items).
 *   Covered raster pixel with winner weights w_k, depth zp and the winner's OWN vertex depths z_k (NR_TEX_Z_BATCH0 has no
 *   effect on this), fp32, every fused multiply-add explicit:
 *     l_k = w_k (zp / z_k)   (the l_k of NR_TEX_UV),   n = sum_k l_k N_k,   p = sum_k l_k P_k   (the fma chain of corner_light)
 *     nh = n / (|n| + 1e-5),   dh = d / (|d| + 1e-5),   vh = (e - p) / (|e - p| + 1e-5)
 *     c = nh . d,   L_c = A_c + D_c max(c, 0)   (the diffuse term uses d as given, like face_light)
 *     r = 2 (nh . dh) nh - dh,   q = max(r . vh, 0),   h = [c > 0] [q > 0] q^sigma   (q^sigma = exp2(sigma log2 q))
 *     rgb_c = L_c s_c + K_c h
 *   with s the UNLIT sample exactly as the unlit path computes it (ts^3 cube, bilinear image or trilinear pyramid).  The
 *   background is not lit; anti-aliasing pools on top; silhouettes and depth ignore shading; NR_FWD_STAGE_TEXTURES is
 *   ignored.  Held to a float64 evaluation of the same expression, not bit-pinned.
 *   Backward (nr_b200_backward_phong), texture half (NR_BWD_PART_TEXTURES): grad_textures and grad_face_uvs as on the smooth
 *   path with the pixel's L_c in place of the corner interpolant (d rgb_c / d s_c = L_c);
 *   grad_corner_shading[f,k] += l_k (d loss / d n, d loss / d p); grad_params receives the exact derivative of the
 *   expression above (through nh with its 1e-5, dh, vh, q^sigma with ln q for sigma, A, D and K).  The masks [c > 0],
 *   [q > 0] and both max take subgradient 0 at their kinks.  Each gradient output may be NULL (not wanted) and is
 *   zero-filled first unless NR_GRAD_ACCUMULATE; without grad_rgb it stays zero.  fp32 atomics, not bit-pinned.
 *   Faces half unchanged: the edge scan reads the Phong rgb map, the depth gradient is unchanged, and no vertex gradient
 *   flows through l_k: NR_GRAD_INTERIOR with Phong is NR_ERR_UNSUPPORTED before any launch.
 *   Host rejections (NR_ERR_INVALID_ARG, before any launch): a NULL phong struct or a struct_size mismatch, a NULL
 *   corner_shading or params, Bc or Bp not in {1, B}, face_light or corner_light set, no NR_RETURN_RGB, and a backward
 *   that asks for grad_corner_shading or grad_params without `textures` (both need s). */
typedef struct nr_b200_phong_args {
    uint32_t struct_size;          /* sizeof(nr_b200_phong_args) */
    int32_t shading_batch;         /* Bc: 1 or B */
    int32_t params_batch;          /* Bp: 1 or B */
    int32_t _pad0;
    const float *corner_shading;   /* [Bc,F,3,6] */
    const float *params;           /* [Bp,16] */
    float *grad_corner_shading;    /* backward: [Bc,F,3,6] or NULL */
    float *grad_params;            /* backward: [Bp,16] or NULL */
} nr_b200_phong_args;

/* Light sets for Phong shading, additive to ABI 4: one struct (nr_b200_lights_args) and two entry points
 * (nr_b200_forward_lights / nr_b200_backward_lights).  NL extra lights, 0 <= NL <= 8, on top of the light that `params`
 * carries ("light 0"): NL = 0 is nr_b200_*_phong exactly (the same kernels), and params D = K = 0 leaves only the set.
 *   lights [Bl,NL,12] (device), Bl in {1, B} (1 = one set for every item, its gradient the sum over the items), per light j:
 *     0-2 D_j diffuse intensity * colour,  3-5 K_j specular intensity * colour,
 *     6-8 x_j: the direction towards the light (directional, not normalised) or the light's position (point), in the frame
 *         of P and e,  9 f_j falloff (point lights only),  10 kind: > 0.5 = point light, else directional,  11 reserved.
 *   Covered raster pixel: nh, p, vh, L_c and h of the Phong expression above, then for j = 0 .. NL-1 in order
 *     directional: c_j = nh . x_j,   lh_j = x_j / (|x_j| + 1e-5),   a_j = 1
 *     point:       u_j = x_j - p,  r_j = |u_j|,  lh_j = u_j / (r_j + 1e-5),  c_j = nh . lh_j,  a_j = 1 / (1 + f_j r_j^2)
 *     L_c = fma(D_jc, a_j max(c_j, 0), L_c)
 *     q_j = max((2 (nh . lh_j) nh - lh_j) . vh, 0),   h_j = [c_j > 0] [q_j > 0] q_j^sigma   (sigma of params)
 *   and rgb_c = fma(K_c, h, L_c s_c) (L_c now every light's diffuse term), then rgb_c = fma(K_jc, a_j h_j, rgb_c) for
 *   j = 0 .. NL-1 in order.  So a directional record with params D = K = 0 gives nr_b200_forward_phong with that light in
 *   params bit for bit.  Held to a float64 evaluation, not bit-pinned otherwise.
 *   Backward (nr_b200_backward_lights), texture half: grad_textures / grad_face_uvs with the pixel's full L_c;
 *   grad_corner_shading also through lh_j and a_j of the point lights (they depend on p); grad_params as for Phong;
 *   grad_lights [Bl,NL,12] the exact derivative in slots 0-9, 0 in slots 10-11.  Masks and max take subgradient 0.  Each
 *   gradient output may be NULL and is zero-filled first unless NR_GRAD_ACCUMULATE.  The faces half is unchanged;
 *   NR_GRAD_INTERIOR is NR_ERR_UNSUPPORTED, as for Phong.
 *   Host rejections (NR_ERR_INVALID_ARG, before any launch), besides those of nr_b200_*_phong: a struct_size mismatch,
 *   NL < 0 or NL > 8, lights NULL with NL > 0, Bl not in {1, B}, and grad_lights without `textures`.  A NULL `lights`
 *   struct is allowed: the call is then nr_b200_*_phong. */
typedef struct nr_b200_lights_args {
    uint32_t struct_size;  /* sizeof(nr_b200_lights_args) */
    int32_t lights_batch;  /* Bl: 1 or B */
    int32_t num_lights;    /* NL: 0 .. 8 */
    int32_t _pad0;
    const float *lights;   /* [Bl,NL,12] */
    float *grad_lights;    /* backward: [Bl,NL,12] or NULL */
} nr_b200_lights_args;

/* Environment lighting for Phong shading, additive to ABI 4: one struct (nr_b200_sh_args) and two entry points
 * (nr_b200_forward_sh / nr_b200_backward_sh).  Second-order real spherical harmonics (9 coefficients per channel) hold the
 * diffuse irradiance of a distant environment (Ramamoorthi & Hanrahan 2001).
 *   sh [Bs,9,3] (device), coefficient k = 0..8 major, channel minor; Bs in {1, B} (1 = one environment for every item, its
 *   gradient the sum over the items).  The coefficients are irradiance-ready: already convolved with the clamped cosine
 *   and divided by pi, so S = (1/C0, 0, ..., 0) gives E = 1 and a white albedo under a uniform environment of radiance r
 *   renders r.  Frame: that of corner_shading's normals (the frame of e and of the light positions).
 *   Covered raster pixel: nh = (x, y, z) = n / (|n| + 1e-5) of the Phong expression, as is (not renormalised, so |nh| is
 *   slightly below 1), fp32 with every fused multiply-add explicit:
 *     Y0 = C0,  Y1 = C1 y,  Y2 = C1 z,  Y3 = C1 x,  Y4 = C2 (x y),  Y5 = C2 (y z),  Y6 = C3 fma(3 z, z, -1),
 *     Y7 = C2 (x z),  Y8 = C4 fma(x, x, -(y y))
 *     C0 = 0.28209479 = 1/(2 sqrt(pi)),  C1 = 0.48860251 = sqrt(3/(4 pi)),  C2 = 1.09254843 = sqrt(15/(4 pi)),
 *     C3 = 0.31539157 = sqrt(5/(16 pi)),  C4 = 0.54627422 = sqrt(15/(16 pi))
 *     E_c = S[0][c] Y0, then E_c = fma(S[k][c], Y_k, E_c) for k = 1 .. 8 in order
 *   E_c is not clamped: an environment whose coefficients make it negative somewhere gives negative irradiance there, and
 *   that is passed through.  Order of terms: L_c of the light-set expression above (params' ambient + diffuse, then the
 *   set's diffuse terms in order), then L_c = L_c + E_c, then rgb_c = fma(K_c, h, L_c s_c) and the set's highlights as
 *   for nr_b200_forward_lights.  So S = 0 gives nr_b200_forward_lights (NL = 0: nr_b200_forward_phong) bit for bit.
 *   Backward (nr_b200_backward_sh), texture half: grad_textures / grad_face_uvs with the pixel's full L_c;
 *   grad_corner_shading also through d E / d nh (E does not depend on p); grad_params and grad_lights as without SH;
 *   grad_sh[k][c] += Y_k(nh) g_c s_c.  Each gradient output may be NULL and is zero-filled first unless
 *   NR_GRAD_ACCUMULATE.  The faces half is unchanged; NR_GRAD_INTERIOR is NR_ERR_UNSUPPORTED, as for Phong.
 *   Host rejections (NR_ERR_INVALID_ARG, before any launch), besides those of nr_b200_*_lights: a struct_size mismatch,
 *   Bs not in {1, B}, sh NULL, and grad_sh without `textures`.  A NULL `sh` struct is allowed: the call is then
 *   nr_b200_*_lights with the same `lights`. */
typedef struct nr_b200_sh_args {
    uint32_t struct_size;  /* sizeof(nr_b200_sh_args) = 24 */
    int32_t sh_batch;      /* Bs: 1 or B */
    const float *sh;       /* [Bs,9,3] */
    float *grad_sh;        /* backward: [Bs,9,3] or NULL */
} nr_b200_sh_args;

/* Tangent-space normal maps for Phong shading, additive to ABI 4: one struct (nr_b200_normal_map_args) and two entry
 * points (nr_b200_forward_normal_map / nr_b200_backward_normal_map).  The map perturbs the interpolated normal n of the
 * Phong expression before anything reads it, so params' light, the light set and the SH environment all see the detail.
 *   normal_map [Bm,Hm,Wm,3] (device), HWC, row 0 = top, holding DECODED tangent-space vectors m = (m_x, m_y, m_z) (not
 *   [0,1] colours; +y along +v, the OpenGL convention).  corner_tangents [Bt,F,3,4]: per drawn face and corner
 *   (T_k, w_k), the tangent and its handedness; F counts the fill_back copies, as corner_shading does (a copy gets
 *   (-T, -w), as its normal is -N).  Bm, Bt in {1, B} (1 = one set for every item, its gradient the sum over the items).
 *   Covered raster pixel, l_k = the perspective weights of the Phong expression, fp32 with every fma explicit:
 *     n = sum_k l_k N_k (as nr_b200_phong_args),  t = fma(l_2, T_2, fma(l_1, T_1, l_0 T_0)) per component
 *     sigma = ((w_0 + w_1) + w_2 < 0) ? -1 : 1   (a majority vote: exact for w in {+-1}, negated for fill_back copies)
 *     b_i = sigma (n_j t_k - n_k t_j)   ((i,j,k) cyclic; each product rounded, then subtracted; n and t as interpolated,
 *                                        not renormalised: the pixel-shader convention of MikkTSpace)
 *     m = the map sampled at the pixel's uv (NR_TEX_UV's uv, fill_back corners reversed) with NR_TEX_UV's bilinear
 *         addressing clamped at the map's own Hm x Wm, level 0 always (also when the albedo is trilinear), per channel
 *         as two horizontal lerps and one vertical one, lerp(a, b, f) = fma(f, b - a, a):
 *           top = lerp(t00, t10, wx1), bot = lerp(t01, t11, wx1), m = lerp(top, bot, wy1)
 *         (so a constant map returns its value exactly)
 *     n' = fma(m_z, n, fma(m_y, b, m_x t)) per component
 *   and the rest of the Phong / light-set / SH expression is unchanged with n' in place of n (nh = n' / (|n'| + 1e-5), c,
 *   L, r, q, h, every light of the set, E_c).  A map (0,0,1) everywhere gives n' = n, so the render equals
 *   nr_b200_forward_sh bit for bit.
 *   Backward, texture half: with g' = d loss / d n' (every light's and the environment's normal gradient through the
 *   normalisation), gm = (g'.t, g'.b, g'.n), gb = m_y g', gt = m_x g' + sigma (gb x n), gn = m_z g' + sigma (t x gb):
 *   grad_corner_shading[f,k][0:3] += l_k gn (the position part as without a map), grad_corner_tangents[f,k] +=
 *   (l_k gt, 0) (no gradient into w), grad_normal_map's four taps += tap weight * gm, and grad_face_uvs also receives the
 *   map's l_k (gu, gv) by NR_TEX_UV's formula with the map's taps, gm in place of g_c and the map's (Wm-1), (Hm-1) and
 *   clamp gates.  grad_textures / grad_face_uvs use the pixel's L_c with the mapped normal.  Each gradient output may
 *   be NULL and is zero-filled first unless NR_GRAD_ACCUMULATE.  The faces half is unchanged.
 *   Host rejections, before any launch: NR_ERR_INVALID_ARG for a struct_size mismatch, Bm or Bt not in {1, B}, a NULL
 *   normal_map or corner_tangents, Hm or Wm < 1, no NR_TEX_UV (the map is addressed by the UVs), grad_normal_map or
 *   grad_corner_tangents without `textures`, and those of nr_b200_*_sh; NR_ERR_UNSUPPORTED for a map beyond 32-bit
 *   offsets and for NR_GRAD_INTERIOR (as for every Phong mode).  A NULL struct is allowed: the call is then
 *   nr_b200_*_sh with the same lights and sh. */
typedef struct nr_b200_normal_map_args {
    uint32_t struct_size;            /* sizeof(nr_b200_normal_map_args) = 56 */
    int32_t map_batch;               /* Bm: 1 or B */
    int32_t tangent_batch;           /* Bt: 1 or B */
    int32_t map_height, map_width;   /* Hm, Wm >= 1 */
    int32_t _pad0;
    const float *normal_map;         /* [Bm,Hm,Wm,3] */
    const float *corner_tangents;    /* [Bt,F,3,4] */
    float *grad_normal_map;          /* backward: [Bm,Hm,Wm,3] or NULL */
    float *grad_corner_tangents;     /* backward: [Bt,F,3,4] or NULL (the w slots receive 0) */
} nr_b200_normal_map_args;

/* Specular maps for Phong shading, additive to ABI 4: one struct (nr_b200_specular_map_args) and two entry points
 * (nr_b200_forward_specular_map / nr_b200_backward_specular_map).  The map makes the specular colour and the shininess
 * vary over the surface; everything diffuse is unchanged.
 *   specular_map [Bq,Hq,Wq,4] (device, 16-byte aligned), HWC, row 0 = top, each texel (ks_r, ks_g, ks_b, sigma'),
 *   Bq in {1, B} (1 = one map for every item, its gradient the sum over the items).
 *   Covered raster pixel: (ks, sigma') = the map sampled at the pixel's uv exactly as nr_b200_normal_map_args samples its
 *   map (NR_TEX_UV's uv, fill_back corners reversed, taps clamped at the map's own Hq x Wq, level 0 always, per channel
 *   top = lerp(t00, t10, wx1), bot = lerp(t01, t11, wx1), q = lerp(top, bot, wy1), lerp(a, b, f) = fma(f, b - a, a), so
 *   a constant map returns its value exactly).  With K'_c = ks_c * K_c and K'_jc = ks_c * K_jc (each product rounded),
 *   the Phong / light-set / SH / normal-map expression is unchanged with K', K'_j and sigma' in place of K, K_j and
 *   params' sigma:  h = [c > 0][q > 0] q^sigma',  rgb_c = fma(K'_c, h, L_c s_c), then fma(K'_jc, a_j h_j, rgb_c) per
 *   light in order.  sigma' replaces params' shininess for params' light and for every light of the set, and is not
 *   clamped.  A constant map (1, 1, 1, sigma of params) renders bit for bit as the same call without the map, and L_c
 *   never reads the map.
 *   Backward, texture half: g' = the upstream gradient of each highlight as without the map; the normal, position,
 *   tangent, light and eye chains are evaluated with K' and sigma'.  grad_params[9+c] += g_c h ks_c, and grad_params[12]
 *   receives 0 from a pixel shaded through the map (sigma is not read there); grad_lights[j][3+c] += g_c a_j h_j ks_c.
 *   grad_specular_map's four taps += tap weight * gq with gq_c = g_c (K_c h + sum_j K_jc a_j h_j) for c < 3 and
 *   gq_3 = sum_c g_c (K'_c h ln q + sum_j K'_jc a_j h_j ln q_j); grad_face_uvs also receives the map's l_k (gu, gv) by
 *   NR_TEX_UV's formula with the map's taps, gq in place of g_c and the map's (Wq-1), (Hq-1) and clamp gates (with a
 *   normal map too, the two UV terms add).  Masks and max take subgradient 0.  Each gradient output may be NULL and
 *   is zero-filled first unless NR_GRAD_ACCUMULATE.  The faces half is unchanged.
 *   Host rejections, before any launch: NR_ERR_INVALID_ARG for a struct_size mismatch, Bq not in {1, B}, a NULL or
 *   not 16-byte aligned specular_map, Hq or Wq < 1, no NR_TEX_UV (the map is addressed by the UVs), grad_specular_map
 *   without `textures`, and those of nr_b200_*_normal_map; NR_ERR_UNSUPPORTED for a map beyond 32-bit offsets and for
 *   NR_GRAD_INTERIOR (as for every Phong mode).  A NULL struct is allowed: the call is then nr_b200_*_normal_map. */
typedef struct nr_b200_specular_map_args {
    uint32_t struct_size;            /* sizeof(nr_b200_specular_map_args) = 32 */
    int32_t map_batch;               /* Bq: 1 or B */
    int32_t map_height, map_width;   /* Hq, Wq >= 1 */
    const float *specular_map;       /* [Bq,Hq,Wq,4], 16-byte aligned */
    float *grad_specular_map;        /* backward: [Bq,Hq,Wq,4] or NULL (any 4-byte alignment) */
} nr_b200_specular_map_args;

/* Attribute interpolation, additive to ABI 4: two flag bits, one struct and two entry points.  Renders C >= 1 arbitrary
 * channels (normals, positions, UVs, labels, features) through the maps an ordinary forward call wrote (face_index_map,
 * weight_map; a silhouette-only forward suffices), with gradients into the attributes and, through the perspective
 * weights, into the vertices.
 *   Attributes are per corner [B,F,3,C] (corners in the face's own order), or with NR_ATTR_PER_VERTEX per vertex [B,Nv,C]
 *   (needs NR_FACES_INDEXED: corner k of face f reads vertex face_indices[f,k], an index outside [0, Nv) reads zeros, as
 *   the geometry does).  NR_ATTR_SHARED: one set [F,3,C] / [Nv,C] serves every item; its gradient is the sum over the
 *   items.  F counts the fill_back copies as faces of their own (give the copies their corners; no fill_back fold).
 *   Forward, covered raster pixel (fn = face_index_map >= 0) with saved weights w_k and the winner's OWN camera depths z_k
 *   (NR_TEX_Z_BATCH0 has no effect):
 *     zp = rcp.rn((w0/z0 + w1/z1) + w2/z2)  (div.rn; the expression of the forward, so zp == depth_map bit for bit),
 *     l_k = w_k * (zp / z_k)  (the l_k of NR_TEX_UV),   out_c = fma(l_2, a_2c, fma(l_1, a_1c, l_0 * a_0c))
 *   (the chain of corner_light: interpolating corner_light as a C = 3 corner attribute gives smooth shading's L_c bit for
 *   bit).  Uncovered pixels are 0.  `out` is planar [B,C,H,W] in image orientation; with NR_ANTI_ALIASING it is the 2x2
 *   mean, summed top-left, top-right, bottom-left, bottom-right, then * 0.25f (only the pooled image is written).
 *   Backward, covered raster pixel with upstream g_c (the pooled gradient / 4 with NR_ANTI_ALIASING):
 *     grad_attributes[corner k (or vertex face_indices[fn,k]), c] += l_k g_c;
 *     interior vertex gradient (grad_faces [B,F,3,3], or grad_vertices [B,Nv,3] with NR_FACES_INDEXED): inv = the K1 inverse
 *     of the winner's pixel-space vertices (face_inverse(to_pixel(.)), as the depth gradient K7 recomputes it),
 *       qx_k = inv[3k] / z_k,  sx = sum_k qx_k,  lx_k = zp (qx_k - l_k sx)  (= d l_k / dx in raster pixels; y alike with
 *       inv[3k+1]),  Gx = sum_c g_c sum_{k=1,2} (a_kc - a_0c) lx_k  (differences against corner 0: no fp32 cancellation
 *       for attributes close together far from 0; sum_k lx_k = 0),  Gy alike,
 *       Gz_m = (l_m / z_m) sum_c g_c (out_c - a_mc)  (out_c the raster-resolution interpolant),
 *       grad x_m += -w_m Gx S/2,   grad y_m += -w_m Gy S/2,   grad z_m += Gz_m.
 *     Derivation: the unclamped barycentrics a_k are affine in the pixel and d a_k / d x_m = -a_m inv[3k] (pixel units), so
 *     d l_k / d x_m = -w_m d l_k / dx_screen; l_k = (w_k / z_k) / sum_j (w_j / z_j) gives d l_k / d z_m = -delta_km l_k / z_k
 *     + l_k l_m / z_m; S/2 takes pixel to NDC units.  This is the derivative at the saved w: the clamp / renormalisation of
 *     the weights is held fixed, as in K7.  No edge or occlusion gradient flows from the attribute image: those come from
 *     the rasterizer's backward (K5) through the alpha image.
 *   Either gradient output may be NULL (not wanted); each is zero-filled first unless NR_GRAD_ACCUMULATE.  grad_out NULL =
 *   zeros.  fp32 atomics, not bit-pinned.
 *   Host rejections (NR_ERR_INVALID_ARG, before any launch): struct_size != sizeof(nr_b200_interpolate_args), B, F or S < 1,
 *   C < 1, a NULL face_index_map / weight_map / attributes (or `out` in the forward), missing geometry for the chosen form,
 *   NR_ATTR_PER_VERTEX without NR_FACES_INDEXED, an odd S with NR_ANTI_ALIASING, grad_vertices without / grad_faces with
 *   NR_FACES_INDEXED, and S > 32767 or B > 65535 (the kernels' grid and 32-bit plane offsets).  No workspace. */
#define NR_ATTR_PER_VERTEX 0x100000u /* attributes [B,Nv,C] per vertex (needs NR_FACES_INDEXED), else [B,F,3,C] per corner */
#define NR_ATTR_SHARED 0x200000u     /* one attribute set [F,3,C] / [Nv,C] for every item                                */

typedef struct nr_b200_interpolate_args {
    uint32_t struct_size; /* sizeof(nr_b200_interpolate_args) */
    uint32_t flags;       /* NR_ANTI_ALIASING as the forward call, NR_FACES_INDEXED / NR_INDICES_SHARED, NR_ATTR_*,
                             NR_GRAD_ACCUMULATE (backward) */
    int32_t batch_size;   /* B */
    int32_t num_faces;    /* F */
    int32_t raster_size;  /* S (doubled with NR_ANTI_ALIASING), as the forward call */
    int32_t channels;     /* C >= 1 */
    const float *faces;          /* [B,F,3,3] as given to the forward call, or NULL with NR_FACES_INDEXED */
    const float *vertices;       /* [B,Nv,3], NR_FACES_INDEXED only */
    const int32_t *face_indices; /* [B,F,3], or [F,3] with NR_INDICES_SHARED */
    int32_t num_vertices;        /* Nv */
    int32_t _pad0;
    const int32_t *face_index_map; /* [B,S,S] saved by nr_b200_forward */
    const float *weight_map;       /* [B,3,S,S] saved by nr_b200_forward */
    const float *attributes;       /* [B,F,3,C] / [B,Nv,C] (no B with NR_ATTR_SHARED) */
    float *out;                    /* forward: [B,C,H,W], H = S or S/2 */
    const float *grad_out;         /* backward: [B,C,H,W] or NULL (zeros) */
    float *grad_attributes;        /* backward: layout of attributes, or NULL */
    float *grad_faces;             /* backward: [B,F,3,3] or NULL; not with NR_FACES_INDEXED */
    float *grad_vertices;          /* backward: [B,Nv,3] or NULL; only with NR_FACES_INDEXED */
} nr_b200_interpolate_args;

/* Soft silhouettes (within ABI 4, additive): per-pixel coverage aggregated over every face within reach (SoftRas, Liu et
 * al. 2019), with gradients into the vertices from every face a pixel reaches -- not only from the edges a hard pixel
 * flips on.  Geometry as nr_b200_forward: faces [B,F,3,3], or vertices [B,Nv,3] + int32 face_indices [F,3] / [B,F,3]
 * with NR_FACES_INDEXED (an index outside [0, Nv) reads the zero vertex); NDC x, y and camera z.
 *   API pixel (r, c) of the S x S image (row 0 at the top, as the hard alpha): p = (x, y), x = (2c + 1 - S) / S,
 *   y = (2 (S-1-r) + 1 - S) / S (div.rn; the hard rasterizer's pixel centres).  Face j:
 *     takes part when every vertex depth satisfies near <= z <= far (fp32) and its x, y are finite; otherwise it is
 *     skipped entirely.  (A per-face test: the hard rasterizer tests the interpolated depth per pixel.)
 *     d_j^2 = min over its three edges (v_k, v_k+1) of the squared distance from p to the closed segment, NDC units
 *     (t = clamp(((p - a) . e) / |e|^2, 0, 1), |e| = 0 gives t = 0);  inside_j = p strictly inside by the edge-function
 *     signs, either winding (all three > 0 or all three < 0; a zero-area face has no inside);
 *     x_j = +d_j^2 / sigma inside, -d_j^2 / sigma outside (fp32, d^2 * (1 / sigma));  D_j = sigmoid(x_j).
 *     Cut-off: an outside face contributes only when d_j^2 <= sigma ln((1 - eps) / eps), i.e. D_j >= eps = NR_SOFT_EPS.
 *   alpha = 1 - prod_j (1 - D_j) = -expm1(Lambda), Lambda = -sum_j softplus(x_j), softplus(x) = max(x,0) + log1p(exp(-|x|)).
 *   The sum is taken in 64-bit fixed point (each term rounded to 2^-40, terms and sum saturated at 64, where alpha is
 *   1.0f): integer adds do not depend on the order the faces arrive in, so alpha is bit-for-bit deterministic.
 *   Winding does not matter, so pass each face once: a duplicated face (a fill_back copy) counts twice, 1 - (1 - D)^2.
 *   Backward: d alpha / d x_j = (1 - alpha) D_j (exact, no division, from the saved alpha); d x_j / d(x, y) of the two
 *   endpoints a, b of the nearest edge: +-(1/sigma) (-2 (1 - t)(p - q), -2 t (p - q)), q = a + t e the nearest point
 *   (the subgradient of the active edge and segment branch; the cut-off is held fixed).  Every gradient into z is 0.
 *   grad_faces [B,F,3,3] (materialised) or grad_vertices [B,Nv,3] (NR_FACES_INDEXED; shared indices reduce over the
 *   items' own vertices, out-of-range indices are skipped), zero-filled first unless NR_GRAD_ACCUMULATE; grad_alpha NULL
 *   = zeros.  fp32 atomics, not bit-pinned.
 *   sigma > 0 and finite; 1e-5 gives a reach of sqrt(sigma ln((1-eps)/eps)) S / 2, about 1.2 pixels at S = 256.
 *   Scratch: nr_b200_soft_workspace_bytes (both passes; the backward bins the faces again, nothing is kept between calls).
 *   Host rejections (NR_ERR_INVALID_ARG, before any launch): struct_size != sizeof(nr_b200_soft_args), B, F or S < 1, a
 *   non-finite or non-positive sigma, near > far (or NaN), missing geometry for the chosen form, a NULL alpha, in the
 *   backward a NULL gradient output for the form or grad_faces with / grad_vertices without NR_FACES_INDEXED, and
 *   B > 65535, S > 32767 or B F 16 > 2^31 - 1 (the grid, 16-bit tile boxes and 32-bit list offsets).  Then
 *   NR_ERR_WORKSPACE for a missing, short or unaligned workspace. */
#define NR_SOFT_EPS 1e-4

typedef struct nr_b200_soft_args {
    uint32_t struct_size; /* sizeof(nr_b200_soft_args) */
    uint32_t flags;       /* NR_FACES_INDEXED / NR_INDICES_SHARED, NR_GRAD_ACCUMULATE (backward) */
    int32_t batch_size;   /* B */
    int32_t num_faces;    /* F */
    int32_t image_size;   /* S */
    int32_t num_vertices; /* Nv (NR_FACES_INDEXED) */
    float sigma;          /* > 0 */
    float near_;          /* faces with a vertex depth outside [near, far] take no part */
    float far_;
    int32_t _pad0;
    const float *faces;          /* [B,F,3,3], or NULL with NR_FACES_INDEXED */
    const float *vertices;       /* [B,Nv,3], NR_FACES_INDEXED only */
    const int32_t *face_indices; /* [B,F,3], or [F,3] with NR_INDICES_SHARED */
    float *alpha;                /* [B,S,S]: written by the forward, read by the backward */
    const float *grad_alpha;     /* backward: [B,S,S] or NULL (zeros) */
    float *grad_faces;           /* backward: [B,F,3,3]; not with NR_FACES_INDEXED */
    float *grad_vertices;        /* backward: [B,Nv,3]; only with NR_FACES_INDEXED */
    void *workspace;             /* nr_b200_soft_workspace_bytes() bytes, 16-byte aligned */
    size_t workspace_bytes;
} nr_b200_soft_args;

/* Soft RGB (within ABI 4, additive): SoftRas colour aggregation over every face within reach, with gradients into the
 * vertices (x, y and z), the per-face texture cubes and the face light.  Geometry, pixel centres, the participation
 * test, d_j^2, inside_j, x_j, D_j, the cut-off and alpha are exactly those of the soft silhouettes above: alpha is
 * bit-identical to nr_b200_soft_silhouettes on the same inputs.  For each contributing (pixel, face j):
 *   A = (x1 - x0)(y2 - y0) - (y1 - y0)(x2 - x0), the doubled signed area (fp32, plain products: vertices exactly collinear
 *     in x, y give exactly 0).  A face with A == 0 counts towards alpha but not towards rgb.
 *   Screen barycentrics: with the edge functions c_k of the distance test (edge k from v_k to v_k+1,
 *     c_k = (v_k+1 - v_k) x (p - v_k)), lam_k = c_{k+1 mod 3} / A; clipped lh = clamp(lam, 0, 1), l = lh / sum lh.
 *   zp = 1 / sum_k l_k / z_k (perspective-correct depth).
 *   C_j = the trilinear cube sample of texture_coords(l, zp, z_0, z_1, z_2) with ts and the clamp from eps, as
 *     nr_b200_forward samples cubes (no fill_back reversal); with face_light every tap is multiplied by the face's light
 *     first.
 *   zn_j = (far - zp) / (far - near); the background sits at zn_b = NR_SOFT_BG_DEPTH.
 *   zmax = max(zn_b, max_j zn_j), w_j = D_j exp((zn_j - zmax) / gamma), w_b = exp((zn_b - zmax) / gamma),
 *   Z = sum_j w_j + w_b,  rgb = (sum_j w_j C_j + w_b background) / Z.
 * The exponents are taken from depth differences, (zref - zp_j) / ((far - near) gamma), zref = far - zmax (far - near),
 * not from differences of zn (whose fp32 rounding near far would dominate at a small gamma).  The forward takes the faces
 * of each pixel in a fixed order (the tile's faces, then the item's wide faces, each by ascending face index: the lists
 * are sorted) and accumulates a running-max softmax: zref starts at the background level far - NR_SOFT_BG_DEPTH (far -
 * near) with Z = 1 and the background colour, and a nearer face rescales Z and the sum by exp((zp - zref) / ((far -
 * near) gamma)).  A face whose weight against the running zref is exactly 0 in fp32 contributes nothing and its cube is
 * not read.  rgb is therefore bit-for-bit repeatable; under a permutation of the faces it is equal only within fp32
 * rounding.  state = {Z, zref} per pixel, written by the forward and read by the backward.
 * Backward: the exact derivative of the above with subgradients at the branches (the nearest edge and its segment, the
 * clamps of lh and of texture_coords, the cube cell and the cut-off held fixed; zref cancels and is held fixed).  With
 * g = grad_rgb at the pixel, the saved rgb and Z (no division by D_j):
 *   d L / d x_j  = (1 - alpha) D_j grad_alpha + w_j (1 - D_j) g . (C_j - rgb) / Z
 *   d L / d zn_j = (w_j / gamma) g . (C_j - rgb) / Z      (through zp into l (x, y) and the vertex depths z_k)
 *   d L / d C_j  = w_j g / Z   (into the 8 taps times the light: grad_textures; into grad_face_light by the unlit sample;
 *                               through the cube's axis derivative and texture_coords into l, zp and z_k)
 *   grad_faces / grad_vertices (as the silhouettes, now with z), grad_textures and grad_face_light are zero-filled first
 *   unless NR_GRAD_ACCUMULATE.  fp32 atomics, not bit-pinned.  grad_rgb / grad_alpha NULL = zeros.
 * Scratch: nr_b200_soft_rgb_workspace_bytes (both passes).  It includes the sort's scratch, which CUB sizes for the
 * current device: the query needs one (0 without one, as nr_b200_vertex_normals_workspace_bytes).
 * Host rejections (NR_ERR_INVALID_ARG, before any launch): every rejection of the silhouettes (struct_size !=
 * sizeof(nr_b200_soft_rgb_args)), a non-finite or non-positive gamma, near >= far (strict: the normalisation divides by
 * far - near) or a non-finite far - near or eps, ts < 2 or ts^3 3 > 2^31 - 1, NULL textures, rgb, alpha or state, and any flag outside
 * NR_FACES_INDEXED | NR_INDICES_SHARED | NR_TEX_SHARED | NR_GRAD_ACCUMULATE (NR_TEX_UV, NR_TEX_MIPMAP and
 * NR_TEX_FILL_BACK included).  Then NR_ERR_WORKSPACE for a missing, short or unaligned workspace. */
#define NR_SOFT_BG_DEPTH 1e-3

typedef struct nr_b200_soft_rgb_args {
    uint32_t struct_size; /* sizeof(nr_b200_soft_rgb_args) */
    uint32_t flags;       /* NR_FACES_INDEXED / NR_INDICES_SHARED, NR_TEX_SHARED, NR_GRAD_ACCUMULATE (backward) */
    int32_t batch_size;   /* B */
    int32_t num_faces;    /* F */
    int32_t image_size;   /* S */
    int32_t num_vertices; /* Nv (NR_FACES_INDEXED) */
    int32_t texture_size; /* ts >= 2 */
    float sigma;          /* > 0 */
    float gamma;          /* > 0: the depth softmax temperature (in units of zn) */
    float near_;          /* near < far; faces with a vertex depth outside [near, far] take no part */
    float far_;
    float eps;            /* texture_coords' clamp: t <= ts - 1 - eps */
    float background[3];  /* RGB of the background term */
    int32_t _pad0;
    const float *faces;          /* [B,F,3,3], or NULL with NR_FACES_INDEXED */
    const float *vertices;       /* [B,Nv,3], NR_FACES_INDEXED only */
    const int32_t *face_indices; /* [B,F,3], or [F,3] with NR_INDICES_SHARED */
    const float *textures;       /* [B,F,ts,ts,ts,3], or [F,ts,ts,ts,3] with NR_TEX_SHARED */
    const float *face_light;     /* [B,F,3] or NULL = unlit */
    float *rgb;                  /* [B,3,S,S]: written by the forward (row 0 at the top), read by the backward */
    float *alpha;                /* [B,S,S]: likewise */
    float *state;                /* [B,2,S,S]: {Z, zref}, likewise */
    const float *grad_rgb;       /* backward: [B,3,S,S] or NULL (zeros) */
    const float *grad_alpha;     /* backward: [B,S,S] or NULL (zeros) */
    float *grad_faces;           /* backward: [B,F,3,3]; not with NR_FACES_INDEXED */
    float *grad_vertices;        /* backward: [B,Nv,3]; only with NR_FACES_INDEXED */
    float *grad_textures;        /* backward: layout of textures, or NULL = not wanted */
    float *grad_face_light;      /* backward: [B,F,3], or NULL = not wanted */
    void *workspace;             /* nr_b200_soft_rgb_workspace_bytes() bytes, 16-byte aligned */
    size_t workspace_bytes;
} nr_b200_soft_rgb_args;

/* Soft RGB through a texture image (within ABI 4, additive): nr_b200_soft_rgb_uv / _backward take the soft RGB's
 * arguments and this struct.  Everything up to the clipped, renormalised barycentrics l and zp, the participation test,
 * D_j, the cut-off, alpha (bit-identical to nr_b200_soft_silhouettes), zero-area faces (alpha only), the softmax, the
 * background term and the running-max order are exactly those of nr_b200_soft_rgb above.  Only the colour C_j of a
 * contributing (pixel, face j) differs:
 *   l'_k = l_k (zp / z_k)  (div.rn, not renormalised: the l_k of NR_TEX_UV with l in place of w),
 *   uv = sum_k l'_k uv_k   with the face's own UV corners (the expression of NR_TEX_UV),
 *   NR_TEX_UV:              the bilinear sample of NR_TEX_UV at uv (clamp to [0, 1], NaN -> 0, row 0 = top), every tap
 *                           times face_light first;
 *   NR_TEX_UV|NR_TEX_MIPMAP: `textures` is the packed pyramid of nr_b200_mip_build, sampled as NR_TEX_MIPMAP with the level
 *                           of detail of NR_TEX_MIPMAP per (pixel, face) in image pixels, taking the face's screen-barycentric
 *                           derivatives in place of K1's inverse: with lam_k = c_{k+1} / A, d lam_k / d column =
 *                           -(2/S) e_{k+1,y} / A and d lam_k / d row = -(2/S) e_{k+1,x} / A (e_m = v_{m+1} - v_m), and
 *                           l in place of w.  Level l1 is not read when f = 0.  No gradient flows through the LOD.
 * Backward: the exact derivative of the above with the cells, the levels, the UV clamp (gated per axis), the nearest edge,
 * the lh clamp and the cut-off held fixed.  With h = w_j g / Z (d L / d C_j of nr_b200_soft_rgb) and s the unlit sample:
 *   grad_textures:  every tap of the image (pyramid: of the pyramid; collapse it with nr_b200_mip_collapse) gets
 *                   a_l * tap weight * light_c * h_c;
 *   grad_face_light: h_c s_c;
 *   (gu, gv) = d L / d uv as NR_TEX_UV's face_uvs gradient with h_c light_c; grad_face_uvs[k] += l'_k (gu, gv) (summed over
 *                   the items with NR_UV_SHARED);
 *   vertices:       d L / d l'_k = gu u_k + gv v_k, on through l, zp and z_k, then as nr_b200_soft_rgb into x, y and z.
 *   Every gradient output is zero-filled first unless NR_GRAD_ACCUMULATE.  fp32 atomics, not bit-pinned.
 * uv NULL runs exactly nr_b200_soft_rgb / nr_b200_soft_rgb_backward.  With uv: NR_TEX_UV is required; NR_UV_SHARED,
 * NR_TEX_MIPMAP, NR_TEX_SHARED (one image for every item), NR_FACES_INDEXED, NR_INDICES_SHARED and NR_GRAD_ACCUMULATE are
 * allowed; `textures` is the image [Bt,Ht,Wt,3] or the pyramid [Bt,P,3]; texture_size and eps are ignored.
 * Scratch: the cube call's, nr_b200_soft_rgb_workspace_bytes(B, F, S, flags & ~(NR_TEX_UV | NR_UV_SHARED | NR_TEX_MIPMAP)).
 * Host rejections before any launch: every rejection of nr_b200_soft_rgb that still applies, a struct_size of either
 * struct other than its sizeof, no NR_TEX_UV, NULL face_uvs, Ht or Wt < 1, NR_TEX_FILL_BACK, NR_GRAD_INTERIOR,
 * NR_RETURN_*, NR_ANTI_ALIASING or any unknown flag (NR_ERR_INVALID_ARG); then image or UV offsets beyond 32 bits
 * (NR_ERR_UNSUPPORTED); then the workspace as nr_b200_soft_rgb. */
typedef struct nr_b200_soft_uv_args {
    uint32_t struct_size;          /* sizeof(nr_b200_soft_uv_args) */
    int32_t texture_height;        /* Ht >= 1 (level 0) */
    int32_t texture_width;         /* Wt >= 1 */
    int32_t _pad0;
    const float *face_uvs;         /* [B,F,3,2], or [F,3,2] with NR_UV_SHARED */
    float *grad_face_uvs;          /* backward: layout of face_uvs, or NULL = not wanted */
} nr_b200_soft_uv_args;

/* Soft attribute images (within ABI 4, additive): nr_b200_soft_attributes / _backward take the soft RGB's arguments and
 * this struct, and render C >= 1 arbitrary channels (per-vertex colours, soft depth, normals, positions, features) through
 * the soft RGB's aggregation.  Geometry, pixel centres, the participation test, d_j^2, x_j, D_j, the cut-off, alpha
 * (bit-identical to nr_b200_soft_silhouettes), zero-area faces (alpha only), l, zp, the weights w_j, the background level
 * NR_SOFT_BG_DEPTH, the running-max softmax, its fixed face order and the rule that a face whose weight is exactly 0
 * contributes nothing are exactly those of nr_b200_soft_rgb above.  Only the colour of a contributing (pixel, face j)
 * differs: it is a C-vector A_j,
 *   l'_k = l_k * (zp / z_k)  (div.rn: the l'_k of nr_b200_soft_rgb_uv),
 *   A_jc = fma(l'_2, a_2c, fma(l'_1, a_1c, l'_0 * a_0c))  (the chain of nr_b200_interpolate), a_kc = corner k's attribute:
 *   per corner [B,F,3,C] (corners in the face's own order), or with NR_ATTR_PER_VERTEX per vertex [B,Nv,C] through
 *   face_indices (needs NR_FACES_INDEXED; an index outside [0, Nv) reads zeros).  NR_ATTR_SHARED: one set [F,3,C] /
 *   [Nv,C] for every item.
 *   out_c = (sum_j w_j A_jc + w_b bg_c) / Z, accumulated as the soft RGB's N_c (bg = background [C], or zeros when NULL).
 * Every channel's arithmetic is independent of the others: channel c of a C-channel call is bit-identical to a C = 1 call
 * with that channel alone.  state = {Z, zref} does not depend on the attributes: on the same geometry, sigma, gamma, near
 * and far it is bit-identical to nr_b200_soft_rgb's.  A camera-z attribute (a_k = z_k) gives A_j = zp up to rounding: a
 * soft depth map (its background is bg; far matches what the hard depth writes where nothing is covered).
 * Backward: the exact derivative with the branches of nr_b200_soft_rgb held (the nearest edge and segment, the lh clamp,
 * the cut-off, zref).  No gradient flows into the background.  With g_c = grad_out at the pixel, the saved out and Z, and
 * h_c = w_j g_c / Z:
 *   grad_attributes[corner k, or vertex face_indices[b,f,k], c] += l'_k h_c  (summed over the items with NR_ATTR_SHARED;
 *                   out-of-range indices are skipped);
 *   H = sum_c g_c (A_jc - out_c) / Z;   d L / d x_j = (1 - alpha) D_j grad_alpha + w_j (1 - D_j) H;
 *   d L / d zp_j through the weight = -w_j H / ((far - near) gamma);
 *   d L / d l'_k = sum_c h_c a_kc, on through l, zp, z_k and the edge functions into x, y and z exactly as
 *                   nr_b200_soft_rgb_uv continues gu u_k + gv v_k.
 *   grad_faces / grad_vertices and grad_attributes are zero-filled first unless NR_GRAD_ACCUMULATE.  fp32 atomics, not
 *   bit-pinned.  grad_out / grad_alpha NULL = zeros; grad_attributes NULL = not wanted.
 * From nr_b200_soft_rgb_args the calls read the geometry, sigma, gamma, near, far, alpha, state, grad_alpha,
 * grad_faces / grad_vertices and the workspace; texture_size, eps and background[3] are ignored, and textures,
 * face_light, rgb, grad_rgb, grad_textures and grad_face_light must be NULL.  Allowed flags: NR_FACES_INDEXED,
 * NR_INDICES_SHARED, NR_ATTR_PER_VERTEX, NR_ATTR_SHARED, NR_GRAD_ACCUMULATE.
 * Scratch: the soft RGB's, nr_b200_soft_rgb_workspace_bytes(B, F, S, flags & (NR_FACES_INDEXED | NR_INDICES_SHARED |
 * NR_GRAD_ACCUMULATE)).
 * Host rejections before any launch: NR_ERR_INVALID_ARG for a struct_size of either struct other than its sizeof, C < 1,
 * a NULL attributes or out, NR_ATTR_PER_VERTEX without NR_FACES_INDEXED, any other flag, a non-NULL rgb-only pointer
 * above, and every rejection of nr_b200_soft_rgb that still applies (NULL alpha or state included); then
 * NR_ERR_UNSUPPORTED when the attribute set (or its gradient) holds more than 2^31 - 1 floats (32-bit offsets); then the
 * workspace as nr_b200_soft_rgb. */
typedef struct nr_b200_soft_attr_args {
    uint32_t struct_size;          /* sizeof(nr_b200_soft_attr_args) */
    int32_t channels;              /* C >= 1 */
    const float *attributes;       /* [B,F,3,C] / [B,Nv,C] (no B with NR_ATTR_SHARED) */
    const float *background;       /* [C], or NULL = zeros */
    float *out;                    /* [B,C,S,S]: written by the forward (row 0 at the top), read by the backward */
    const float *grad_out;         /* backward: [B,C,S,S] or NULL (zeros) */
    float *grad_attributes;        /* backward: layout of attributes, or NULL = not wanted */
} nr_b200_soft_attr_args;

/* Soft fragments (within ABI 4, additive): nr_b200_soft_fragments / _backward take the soft RGB's arguments and this
 * struct, and return for every pixel the K nearest faces within reach (PyTorch3D's MeshRasterizer with faces_per_pixel =
 * K and a blur radius), to be shaded and blended by the caller.  Pixel centres, the participation test, d_j^2, inside_j,
 * x_j, the cut-off, A, the barycentrics lam, lh, l and zp, and l'_k = l_k (zp / z_k) (div.rn) are exactly those of
 * nr_b200_soft_rgb and nr_b200_soft_attributes above.
 *   Candidate: a (pixel, face j) is one when the face takes part, is within reach (inside, or d_j^2 within the cut-off),
 *     has A != 0 (a zero-area face is not a fragment, as it is not a colour of the soft RGB) and a finite fp32 zp.
 *   Selection: candidates are ordered by the key (zp, f) -- the fp32 zp first, the face index within the item second, a
 *     total order that does not depend on the order of the lists -- and the first n = min(K, #candidates) are kept.  The
 *     result is deterministic, and invariant under a permutation of the faces up to exact zp ties.  The first K1 slots
 *     of a call with K2 > K1 are the K1 call's.
 *   Outputs, slot k < n nearest first, row 0 at the top:
 *     pix_to_face [B,S,S,K] int64: the face index within its item, in [0, F) (not packed b F + f);
 *     zbuf        [B,S,S,K] float: zp;
 *     bary        [B,S,S,K,3] float: l'_0, l'_1, l'_2, clipped and renormalised exactly as the soft attributes
 *                 interpolate, so sum_k l'_k a_k is A_j of nr_b200_soft_attributes;
 *     dists       [B,S,S,K] float: +d_j^2 inside, -d_j^2 outside, in squared NDC units (the d_j^2 soft_eval minimises,
 *                 i.e. sigma x_j before the scaling by 1 / sigma), so sigmoid(dists / sigma) is SoftRas's D_j.  The sign
 *                 is the OPPOSITE of PyTorch3D's dists (negative inside there).
 *   Slots k >= n hold -1 in every field (bary: all three), as in PyTorch3D.
 * Backward: the exact derivative with the selection held fixed, and with it the nearest edge and its segment branch, the
 * lh clamp and the cut-off.  grad_zbuf, grad_bary and grad_dists (each NULL = zeros) flow into x, y and z of the
 * vertices; empty slots are ignored.  zbuf and bary go through the chain of nr_b200_soft_attributes_backward from l'_k
 * and zp (d L / d l'_k = grad_bary, d L / d zp = grad_zbuf); dists through d(+-d^2)/d(a, b) of the nearest edge (a, b),
 * sigma times the silhouettes' d x_j / d(a, b), and nothing into z.  grad_faces / grad_vertices are zero-filled first
 * unless NR_GRAD_ACCUMULATE; shared indices reduce over the items, out-of-range indices are skipped.  fp32 atomics, not
 * bit-pinned.  The backward reads pix_to_face (the forward's) and the upstream gradients; zbuf, bary and dists are not
 * read and may be NULL there.
 * From nr_b200_soft_rgb_args the calls read the geometry, sigma, near, far, grad_faces / grad_vertices and the
 * workspace; gamma, texture_size, eps and background[3] are ignored, and textures, face_light, rgb, alpha, state,
 * grad_rgb, grad_alpha, grad_textures and grad_face_light must be NULL.  Allowed flags: NR_FACES_INDEXED,
 * NR_INDICES_SHARED, NR_GRAD_ACCUMULATE.  1 <= K <= 32.
 * Scratch: the soft RGB's, nr_b200_soft_rgb_workspace_bytes(B, F, S, flags).
 * Host rejections before any launch: NR_ERR_INVALID_ARG for a struct_size of either struct other than its sizeof, K
 * outside [1, 32], a NULL pix_to_face (and, in the forward, a NULL zbuf, bary or dists), a non-NULL pointer of the list
 * above, any other flag, and every rejection of nr_b200_soft_rgb that still applies; then the workspace as
 * nr_b200_soft_rgb. */
typedef struct nr_b200_soft_frag_args {
    uint32_t struct_size;          /* sizeof(nr_b200_soft_frag_args) */
    int32_t faces_per_pixel;       /* K, 1 <= K <= 32 */
    int64_t *pix_to_face;          /* [B,S,S,K]: written by the forward, read by the backward */
    float *zbuf;                   /* [B,S,S,K]: forward */
    float *bary;                   /* [B,S,S,K,3]: forward */
    float *dists;                  /* [B,S,S,K]: forward */
    const float *grad_zbuf;        /* backward: [B,S,S,K] or NULL (zeros) */
    const float *grad_bary;        /* backward: [B,S,S,K,3] or NULL (zeros) */
    const float *grad_dists;       /* backward: [B,S,S,K] or NULL (zeros) */
} nr_b200_soft_frag_args;

/* ABI version of the loaded library (== NR_B200_ABI_VERSION it was built with). */
NR_B200_API int nr_b200_abi_version(void);
NR_B200_API const char *nr_b200_error_string(int code);

/* Scratch sizes (bytes).  Pure host arithmetic; safe to call without a GPU. */
NR_B200_API size_t nr_b200_forward_workspace_bytes(int32_t batch_size, int32_t num_faces, int32_t raster_size, int32_t texture_size,
                                       uint32_t flags);
NR_B200_API size_t nr_b200_backward_workspace_bytes(int32_t batch_size, int32_t num_faces, int32_t raster_size,
                                        int32_t texture_size, uint32_t flags);

NR_B200_API int nr_b200_forward(const nr_b200_forward_args *args, void *cuda_stream);
NR_B200_API int nr_b200_backward(const nr_b200_backward_args *args, void *cuda_stream);
/* The backward of a forward call that had corner_light (smooth shading, above): `args` as for nr_b200_backward (with
 * face_light NULL), corner_light [B,F,3,3] as given to the forward call (required), grad_corner_light [B,F,3,3] or NULL =
 * not wanted (part of the texture half, NR_BWD_PART_TEXTURES).  nr_b200_backward is this call with corner_light NULL. */
NR_B200_API int nr_b200_backward_corner_light(const nr_b200_backward_args *args, const float *corner_light,
                                              float *grad_corner_light, void *cuda_stream);
/* Phong shading (nr_b200_phong_args above).  The forward takes `args` with face_light and corner_light NULL and the
 * workspace of nr_b200_forward_workspace_bytes; the backward is that of such a forward, `args` as for nr_b200_backward (with
 * face_light NULL), the same `phong` corner_shading / params, and its grad_corner_shading / grad_params filled by the
 * texture half. */
NR_B200_API int nr_b200_forward_phong(const nr_b200_forward_args *args, const nr_b200_phong_args *phong, void *cuda_stream);
NR_B200_API int nr_b200_backward_phong(const nr_b200_backward_args *args, const nr_b200_phong_args *phong, void *cuda_stream);
/* Phong shading with a light set (nr_b200_lights_args above): the Phong calls with `lights` added; lights NULL or NL = 0
 * runs exactly nr_b200_forward_phong / nr_b200_backward_phong.  grad_lights is filled by the texture half. */
NR_B200_API int nr_b200_forward_lights(const nr_b200_forward_args *args, const nr_b200_phong_args *phong,
                                       const nr_b200_lights_args *lights, void *cuda_stream);
NR_B200_API int nr_b200_backward_lights(const nr_b200_backward_args *args, const nr_b200_phong_args *phong,
                                        const nr_b200_lights_args *lights, void *cuda_stream);
/* Phong shading with a light set and an SH environment (nr_b200_sh_args above): the light-set calls with `sh` added;
 * lights may be NULL (no set), and sh NULL runs exactly nr_b200_forward_lights / nr_b200_backward_lights.  grad_sh is
 * filled by the texture half. */
NR_B200_API int nr_b200_forward_sh(const nr_b200_forward_args *args, const nr_b200_phong_args *phong,
                                   const nr_b200_lights_args *lights, const nr_b200_sh_args *sh, void *cuda_stream);
NR_B200_API int nr_b200_backward_sh(const nr_b200_backward_args *args, const nr_b200_phong_args *phong,
                                    const nr_b200_lights_args *lights, const nr_b200_sh_args *sh, void *cuda_stream);
/* Phong shading through a tangent-space normal map (nr_b200_normal_map_args above): the SH calls with `nm` added; lights
 * and sh may be NULL, and nm NULL runs exactly nr_b200_forward_sh / nr_b200_backward_sh.  grad_normal_map and
 * grad_corner_tangents are filled by the texture half. */
NR_B200_API int nr_b200_forward_normal_map(const nr_b200_forward_args *args, const nr_b200_phong_args *phong,
                                           const nr_b200_lights_args *lights, const nr_b200_sh_args *sh,
                                           const nr_b200_normal_map_args *nm, void *cuda_stream);
NR_B200_API int nr_b200_backward_normal_map(const nr_b200_backward_args *args, const nr_b200_phong_args *phong,
                                            const nr_b200_lights_args *lights, const nr_b200_sh_args *sh,
                                            const nr_b200_normal_map_args *nm, void *cuda_stream);
/* Phong shading through a specular map (nr_b200_specular_map_args above): the normal-map calls with `sm` added; lights,
 * sh and nm may be NULL, and sm NULL runs exactly nr_b200_forward_normal_map / nr_b200_backward_normal_map.
 * grad_specular_map is filled by the texture half. */
NR_B200_API int nr_b200_forward_specular_map(const nr_b200_forward_args *args, const nr_b200_phong_args *phong,
                                             const nr_b200_lights_args *lights, const nr_b200_sh_args *sh,
                                             const nr_b200_normal_map_args *nm, const nr_b200_specular_map_args *sm,
                                             void *cuda_stream);
NR_B200_API int nr_b200_backward_specular_map(const nr_b200_backward_args *args, const nr_b200_phong_args *phong,
                                              const nr_b200_lights_args *lights, const nr_b200_sh_args *sh,
                                              const nr_b200_normal_map_args *nm, const nr_b200_specular_map_args *sm,
                                              void *cuda_stream);
/* Attribute interpolation (nr_b200_interpolate_args above): the image `out`, and its backward into grad_attributes and the
 * interior vertex gradient.  One kernel launch each (plus the zero-fill of the backward). */
NR_B200_API int nr_b200_interpolate(const nr_b200_interpolate_args *args, void *cuda_stream);
NR_B200_API int nr_b200_interpolate_backward(const nr_b200_interpolate_args *args, void *cuda_stream);
/* Soft silhouettes (nr_b200_soft_args above): alpha [B,S,S], and its backward into grad_faces / grad_vertices.  The
 * workspace size is pure host arithmetic (0 for sizes or a sigma the calls refuse); `flags` is accepted for the future. */
NR_B200_API size_t nr_b200_soft_workspace_bytes(int32_t batch_size, int32_t num_faces, int32_t image_size, float sigma,
                                                uint32_t flags);
NR_B200_API int nr_b200_soft_silhouettes(const nr_b200_soft_args *args, void *cuda_stream);
NR_B200_API int nr_b200_soft_silhouettes_backward(const nr_b200_soft_args *args, void *cuda_stream);
/* Soft RGB (nr_b200_soft_rgb_args above): rgb [B,3,S,S], alpha [B,S,S] and state, and the backward into the geometry,
 * grad_textures and grad_face_light.  The workspace size is 0 for sizes or flags the calls refuse, or without a device. */
NR_B200_API size_t nr_b200_soft_rgb_workspace_bytes(int32_t batch_size, int32_t num_faces, int32_t image_size, uint32_t flags);
NR_B200_API int nr_b200_soft_rgb(const nr_b200_soft_rgb_args *args, void *cuda_stream);
NR_B200_API int nr_b200_soft_rgb_backward(const nr_b200_soft_rgb_args *args, void *cuda_stream);
/* Soft RGB through a texture image (nr_b200_soft_uv_args above); uv NULL runs exactly the two calls above. */
NR_B200_API int nr_b200_soft_rgb_uv(const nr_b200_soft_rgb_args *args, const nr_b200_soft_uv_args *uv, void *cuda_stream);
NR_B200_API int nr_b200_soft_rgb_uv_backward(const nr_b200_soft_rgb_args *args, const nr_b200_soft_uv_args *uv,
                                             void *cuda_stream);
/* Soft attribute images (nr_b200_soft_attr_args above): out [B,C,S,S], alpha and state, and the backward into the
 * geometry and grad_attributes. */
NR_B200_API int nr_b200_soft_attributes(const nr_b200_soft_rgb_args *args, const nr_b200_soft_attr_args *attr,
                                        void *cuda_stream);
NR_B200_API int nr_b200_soft_attributes_backward(const nr_b200_soft_rgb_args *args, const nr_b200_soft_attr_args *attr,
                                                 void *cuda_stream);
/* Soft fragments (nr_b200_soft_frag_args above): pix_to_face, zbuf, bary and dists, and the backward into the
 * geometry. */
NR_B200_API int nr_b200_soft_fragments(const nr_b200_soft_rgb_args *args, const nr_b200_soft_frag_args *frag,
                                       void *cuda_stream);
NR_B200_API int nr_b200_soft_fragments_backward(const nr_b200_soft_rgb_args *args, const nr_b200_soft_frag_args *frag,
                                                void *cuda_stream);

/* vertices_to_faces (reference vertices_to_faces.py:4-21), the step either side of the rasterizer:
 *   forward   out_faces[b,f,k,:] = vertices[b, faces[b,f,k], :]           ([B,Nv,3] x [B,Nf,3] int32 -> [B,Nf,3,3])
 *   backward  grad_vertices[b, faces[b,f,k], :] += grad_faces[b,f,k,:]   (zero-filled first unless NR_GRAD_ACCUMULATE)
 * Out-of-range indices gather zeros / are skipped. */
NR_B200_API int nr_b200_vertices_to_faces(const float *vertices, const int32_t *faces, int32_t batch_size,
                                          int32_t num_vertices, int32_t num_faces, float *out_faces, void *cuda_stream);
NR_B200_API int nr_b200_vertices_to_faces_backward(const float *grad_faces, const int32_t *faces, int32_t batch_size,
                                                   int32_t num_vertices, int32_t num_faces, float *grad_vertices,
                                                   uint32_t flags, void *cuda_stream);

/* Camera pipeline of Renderer (reference look_at.py:30-44 / look.py:29-43, then perspective.py:10-18) as one
 * per-vertex kernel each way:
 *   d = vertices[b,v,:] - eye[b];   o = rot[b] * d   (rows of rot = camera x, y, z axes; rot NULL = identity,
 *   eye NULL = origin);   with NR_CAM_PERSPECTIVE:  out = (o.x / o.z / width[b], o.y / o.z / width[b], o.z)
 * rot [B,9], eye [B,3], width [B] are device arrays; with NR_CAM_SHARED they hold ONE camera used by every item.
 * The backward stores grad_vertices [B,Nv,3] (may be NULL; overwritten, with or without NR_GRAD_ACCUMULATE) and
 * accumulates, per camera, grad_rot [.,9], grad_eye [.,3], grad_width [.] (each may be NULL; zero-filled first unless
 * NR_GRAD_ACCUMULATE, which adds into them). */
#define NR_CAM_PERSPECTIVE 0x100u
#define NR_CAM_SHARED 0x200u
NR_B200_API int nr_b200_camera_transform(const float *vertices, const float *rot, const float *eye, const float *width,
                                         int32_t batch_size, int32_t num_vertices, uint32_t flags, float *out,
                                         void *cuda_stream);
NR_B200_API int nr_b200_camera_transform_backward(const float *vertices, const float *rot, const float *eye,
                                                  const float *width, const float *grad_out, int32_t batch_size,
                                                  int32_t num_vertices, uint32_t flags, float *grad_vertices,
                                                  float *grad_rot, float *grad_eye, float *grad_width, void *cuda_stream);

/* Per-face light factor of lighting.py:29-51, straight from vertices and face indices:
 *   n = normalize(cross(v0 - v1, v2 - v1))  (x / (|x| + 1e-5), like chainer.functions.normalize)
 *   face_light[b,f,:] = ambient + directional * max(n . direction, 0)
 * `faces` is [B,Nf,3] int32, or [Nf,3] with NR_INDICES_SHARED (ABI 3).
 * light_params [B,9] (or [1,9] with NR_CAM_SHARED) = {intensity_ambient * color_ambient (3),
 * intensity_directional * color_directional (3), direction (3)}, device memory.  The factor is consumed by
 * nr_b200_forward_args.face_light; the backward turns d loss / d face_light (nr_b200_backward_args.grad_face_light)
 * into d loss / d vertices (zero-filled first unless NR_GRAD_ACCUMULATE). */
NR_B200_API int nr_b200_face_lighting(const float *vertices, const int32_t *faces, const float *light_params,
                                      int32_t batch_size, int32_t num_vertices, int32_t num_faces, uint32_t flags,
                                      float *face_light, void *cuda_stream);
NR_B200_API int nr_b200_face_lighting_backward(const float *vertices, const int32_t *faces, const float *light_params,
                                               const float *grad_face_light, int32_t batch_size, int32_t num_vertices,
                                               int32_t num_faces, uint32_t flags, float *grad_vertices, void *cuda_stream);

/* Smooth shading glue (feeds nr_b200_forward_args.corner_light).
 * Vertex normals, area weighted, from vertices [B,Nv,3] and the index set `faces` [B,Nf,3] ([Nf,3] with NR_INDICES_SHARED):
 *   c_f = cross(v0 - v1, v2 - v1) (unnormalised, the face-normal direction of lighting.py:40-43; 0 for a face with an index
 *   outside [0, Nv)),  s_v = sum of c_f over every corner (f, k) with faces[f,k] == v, added in ascending (f, k) order,
 *   n_v = s_v / (|s_v| + 1e-5)  (an unreferenced vertex gets 0).  Pass the original faces, not a fill_back-doubled set
 *   (whose copies would cancel the sums).  The forward is deterministic (no float atomics): a stable radix sort of the
 *   corners by vertex, then one ordered gather per vertex, with scratch in the caller's workspace of
 *   nr_b200_vertex_normals_workspace_bytes (it asks the current device for the sort's tuning, so it needs a CUDA device;
 *   0 = unsupported sizes).  The same workspace serves the backward, which turns d loss / d vertex_normals into
 *   d loss / d vertices (zero-filled first unless NR_GRAD_ACCUMULATE; fp32 atomics).
 *   NR_ERR_UNSUPPORTED when (items of the index set) * (Nv + 1) or 3 Nf exceeds 2^31 - 1. */
NR_B200_API size_t nr_b200_vertex_normals_workspace_bytes(int32_t batch_size, int32_t num_vertices, int32_t num_faces,
                                                         uint32_t flags);
NR_B200_API int nr_b200_vertex_normals(const float *vertices, const int32_t *faces, int32_t batch_size, int32_t num_vertices,
                                       int32_t num_faces, uint32_t flags, float *vertex_normals, void *workspace,
                                       size_t workspace_bytes, void *cuda_stream);
NR_B200_API int nr_b200_vertex_normals_backward(const float *vertices, const int32_t *faces, const float *grad_vertex_normals,
                                                int32_t batch_size, int32_t num_vertices, int32_t num_faces, uint32_t flags,
                                                float *grad_vertices, void *workspace, size_t workspace_bytes,
                                                void *cuda_stream);
/* Per-corner Lambertian light from vertex normals [B,Nv,3], `faces` the index set the rasterizer receives ([B,Nf,3] or
 * [Nf,3] with NR_INDICES_SHARED) and light_params [B,9] ([1,9] with NR_CAM_SHARED, layout of nr_b200_face_lighting):
 *   corner_light[b,f,k,:] = ambient + directional * max(sgn * (n . direction), 0),   n = vertex_normals[b, faces[f,k]]
 *   (0 for an index outside [0, Nv)), dot as (n0 d0 + n1 d1) + n2 d2, sgn = -1 for the reversed copies f >= Nf/2 with
 *   NR_TEX_FILL_BACK (Nf even; their face normal is reversed, as in face_light), else 1.  The backward scatters
 *   d loss / d corner_light into grad_vertex_normals [B,Nv,3] (zero-filled first unless NR_GRAD_ACCUMULATE; atomics). */
NR_B200_API int nr_b200_corner_lighting(const float *vertex_normals, const int32_t *faces, const float *light_params,
                                        int32_t batch_size, int32_t num_vertices, int32_t num_faces, uint32_t flags,
                                        float *corner_light, void *cuda_stream);
NR_B200_API int nr_b200_corner_lighting_backward(const float *vertex_normals, const int32_t *faces, const float *light_params,
                                                 const float *grad_corner_light, int32_t batch_size, int32_t num_vertices,
                                                 int32_t num_faces, uint32_t flags, float *grad_vertex_normals,
                                                 void *cuda_stream);
/* Phong shading glue (feeds nr_b200_phong_args.corner_shading) from vertex normals [B,Nv,3], vertices [B,Nv,3] (the
 * positions P, in the frame of the eye) and the index set `faces` ([B,Nf,3] or [Nf,3] with NR_INDICES_SHARED):
 *   corner_shading[b,f,k,:] = (sgn n, v),   n = vertex_normals[b, faces[f,k]],  v = vertices[b, faces[f,k]]
 *   (both 0 for an index outside [0, Nv)), sgn = -1 for the reversed copies f >= Nf/2 with NR_TEX_FILL_BACK (Nf even), else 1.
 * The backward scatters d loss / d corner_shading [B,Nf,3,6] into grad_vertex_normals and grad_vertices [B,Nv,3] (either may
 * be NULL, not both; each zero-filled first unless NR_GRAD_ACCUMULATE; atomics). */
NR_B200_API int nr_b200_corner_shading(const float *vertex_normals, const float *vertices, const int32_t *faces,
                                       int32_t batch_size, int32_t num_vertices, int32_t num_faces, uint32_t flags,
                                       float *corner_shading, void *cuda_stream);
NR_B200_API int nr_b200_corner_shading_backward(const int32_t *faces, const float *grad_corner_shading, int32_t batch_size,
                                                int32_t num_vertices, int32_t num_faces, uint32_t flags,
                                                float *grad_vertex_normals, float *grad_vertices, void *cuda_stream);

/* Texture baking of load_obj (reference load_obj.py:88-137): every texel (a, b, c) of the ts^3 cube of face f is the
 * bilinear sample of `image` [H,W,3] (rows already flipped, load_obj.py:82) at the UV position with barycentric
 * coordinates (a, b, c) / (a + b + c) of `uv_faces` [F,3,2]; faces with is_update[f] == 0 (is_update may be NULL =
 * all faces) keep their cube.  Texel (0,0,0) becomes NaN exactly as in the reference (0/0).  `textures`
 * [F,ts,ts,ts,3] is updated in place. */
NR_B200_API int nr_b200_bake_textures(const float *image, const float *uv_faces, const int32_t *is_update,
                                      int32_t num_faces, int32_t texture_size, int32_t image_height,
                                      int32_t image_width, float *textures, void *cuda_stream);

/* Mip pyramid of a texture image for NR_TEX_MIPMAP (layout and arithmetic above).
 *   nr_b200_mip_texels    P for an Ht x Wt image (0 for sizes < 1).  Pure host arithmetic; safe without a GPU.
 *   nr_b200_mip_build     image [Bt,Ht,Wt,3] -> pyramid [Bt,P,3] (level 0 is a copy).  At most two kernel launches.
 *   nr_b200_mip_collapse  the exact transpose of the build: grad_pyramid [Bt,P,3] -> grad_image [Bt,Ht,Wt,3]; a child
 *                         texel receives m_x m_y / 4 of its parent's gradient (m = 2 where the edge clamp counts it
 *                         twice, else 1).  Writes grad_image, or adds into it with NR_GRAD_ACCUMULATE.  Deterministic
 *                         (one gather per level-0 texel, no atomics).
 * Null pointers and sizes < 1 give NR_ERR_INVALID_ARG, pyramids beyond 32-bit offsets NR_ERR_UNSUPPORTED, before any
 * launch. */
NR_B200_API size_t nr_b200_mip_texels(int32_t texture_height, int32_t texture_width);
NR_B200_API int nr_b200_mip_build(const float *image, int32_t batch_size, int32_t texture_height, int32_t texture_width,
                                  float *pyramid, void *cuda_stream);
NR_B200_API int nr_b200_mip_collapse(const float *grad_pyramid, int32_t batch_size, int32_t texture_height,
                                     int32_t texture_width, float *grad_image, uint32_t flags, void *cuda_stream);

/* Number of kernels the last forward/backward call on this thread launched (for launch accounting). */
NR_B200_API int nr_b200_last_launch_count(void);

/* Optional per-kernel timing: when enabled (per host thread) every kernel launch of forward/backward is bracketed
 * by CUDA events on the launching stream.  nr_b200_read_profile synchronises on them, writes up to max_entries
 * durations (milliseconds) to `ms` and the kernel names as a NUL-separated list to `names`, clears the record and
 * returns the number of entries.  Used by bench.py for the roofline of the dominant kernel; off by default. */
NR_B200_API void nr_b200_set_profiling(int enabled);
NR_B200_API int nr_b200_read_profile(char *names, size_t names_bytes, float *ms, int max_entries);

#ifdef __cplusplus
}
#endif
#endif /* NR_B200_H_ */
