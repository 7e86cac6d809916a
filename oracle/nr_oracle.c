/*
 * nr_oracle.c -- CPU restatement of the reference rasterizer hot path.
 *
 * TEST INFRASTRUCTURE ONLY.  This file is the parity oracle for the CUDA
 * product in neural_renderer_b200/; the product never links, imports or calls
 * it.  Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
 * --impl reference legs may use it, and only as the checker or as the timed
 * CPU baseline.
 *
 * It restates, in scalar fp32 C, what the reference's CuPy kernel strings
 * compute (hiroharu-kato/neural_renderer, neural_renderer/rasterize.py):
 *
 *   nro_face_inv      <- K1  rasterize.py:242-277
 *   nro_zbuffer       <- K2  rasterize.py:281-359   (safe per-pixel z-buffer)
 *   nro_texture       <- K4  rasterize.py:372-438
 *   nro_compose       <- forward_alpha_map_gpu / forward_background_gpu  :440-465
 *   nro_pixel_bwd     <- K5  rasterize.py:528-748
 *   nro_texture_bwd   <- K6  rasterize.py:760-792
 *   nro_depth_bwd     <- K7  rasterize.py:805-847
 *
 * Floating point: the reference is compiled by NVRTC with --fmad=true and no
 * fast-math.  The exact sequence of mul / add / fma / div.rn / rcp.rn that
 * results was read off the PTX *and SASS* of the reference strings (ptxas
 * contracts PTX mul+add pairs that carry no .rn; see DESIGN.md, "pinned
 * arithmetic") and is reproduced here with explicit fmaf(); everything
 * else is compiled with -ffp-contract=off so gcc cannot fuse on its own.
 * Where the reference promotes to double (literal `0.`, `1.`, `2.`, near, eps)
 * the same promotion is done here.
 *
 * Parity pinned: checked in tests/test_oracle_golden.py against the reference
 * test fixtures (Blender silhouette, test_depth.png, the two known-answer
 * gradient vectors of tests/test_rasterize_silhouettes.py) and, on the GPU,
 * against the reference kernels themselves compiled into oracle/_ref/.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#ifdef _OPENMP
#include <omp.h>
#endif

#define NRO_API __attribute__((visibility("default")))


/* float/double -> int conversions with CUDA semantics (cvt.rzi.s32: NaN -> 0, saturating). */
static inline int f2i_rz(float x) {
    if (x != x) return 0;
    if (x >= 2147483648.0f) return INT32_MAX;
    if (x <= -2147483648.0f) return INT32_MIN;
    return (int)x;
}
static inline int d2i_rz(double x) {
    if (x != x) return 0;
    if (x >= 2147483648.0) return INT32_MAX;
    if (x <= -2147483649.0) return INT32_MIN;
    return (int)x;
}

static inline int backside(const float *f) {
    /* rasterize.py:252, :306, :540 -- sub, sub, mul on each side, fp32 compare */
    return (f[7] - f[1]) * (f[3] - f[0]) < (f[4] - f[1]) * (f[6] - f[0]);
}

static inline float to_pixel(float c, int is) {
    /* 0.5 * (c * is + is - 1): fma(c, is, is) + (-1), then an exact halving (rasterize.py:258, :549) */
    float fis = (float)is;
    float t = fmaf(c, fis, fis);
    t = t + (-1.0f);
    return (float)(0.5 * (double)t);
}

/* ------------------------------------------------------------------ K1 ---- */
static void face_inv_one(const float *face, int is, float *inv /*9, zero-initialised by caller*/) {
    if (backside(face)) return;
    float p0x = to_pixel(face[0], is), p0y = to_pixel(face[1], is);
    float p1x = to_pixel(face[3], is), p1y = to_pixel(face[4], is);
    float p2x = to_pixel(face[6], is), p2y = to_pixel(face[7], is);
    float n[9];
    n[0] = p1y - p2y;
    n[1] = p2x - p1x;
    /* a*b - c*d: PTX has mul, mul, sub without .rn; ptxas contracts it to fma(a, b, -RN(c*d)) in SASS */
    n[2] = fmaf(p1x, p2y, -(p2x * p1y));
    n[3] = p2y - p0y;
    n[4] = p0x - p2x;
    n[5] = fmaf(p2x, p0y, -(p0x * p2y));
    n[6] = p0y - p1y;
    n[7] = p1x - p0x;
    n[8] = fmaf(p0x, p1y, -(p1x * p0y));
    /* p2x*(p0y-p1y) + p0x*(p1y-p2y) + p1x*(p2y-p0y)  ->  fma(p1x, d3, fma(p2x, d6, p0x*d0)) */
    float d = fmaf(p1x, n[3], fmaf(p2x, n[6], p0x * n[0]));
    for (int k = 0; k < 9; k++) inv[k] = n[k] / d;
}

NRO_API void nro_face_inv(const float *faces, int64_t n_faces_total, int is, float *faces_inv) {
    memset(faces_inv, 0, sizeof(float) * 9 * (size_t)n_faces_total);
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < n_faces_total; i++) face_inv_one(faces + 9 * i, is, faces_inv + 9 * i);
}

static inline float clamp01_d(float w) {
    /* min(max(w, 0.), 1.) evaluated in double; max/min return the non-NaN operand like PTX max.f64/min.f64 */
    double x = (double)w;
    x = fmax(x, 0.0);
    x = fmin(x, 1.0);
    return (float)x;
}

/* ------------------------------------------------------------------ K2 ---- */
/* Maps must be pre-initialised by the caller exactly like forward_gpu does (rasterize.py:478-496):
 * face_index_map = -1, weight_map = 0, depth_map = far, face_inv_map = 0. */
NRO_API void nro_zbuffer(const float *faces, const float *faces_inv, int bs, int nf, int is, double near_, double far_,
                         int *face_index_map, float *weight_map, float *depth_map, float *face_inv_map /*nullable*/) {
    const int64_t npix = (int64_t)bs * is * is;
#pragma omp parallel for schedule(dynamic, 256)
    for (int64_t i = 0; i < npix; i++) {
        const int bn = (int)(i / ((int64_t)is * is));
        const int pn = (int)(i % ((int64_t)is * is));
        const int yi = pn / is, xi = pn % is;
        const float yp = (float)((2. * yi + 1 - is) / is);
        const float xp = (float)((2. * xi + 1 - is) / is);
        const float fxi = (float)xi, fyi = (float)yi;
        const float *face = faces + (int64_t)bn * nf * 9 - 9;
        const float *finv = faces_inv + (int64_t)bn * nf * 9 - 9;
        float depth_min = (float)far_;
        int face_index_min = -1;
        float weight_min[3] = {0, 0, 0};
        const float *inv_min = NULL;
        for (int fn = 0; fn < nf; fn++) {
            face += 9;
            finv += 9;
            if (backside(face)) continue;
            if (((yp - face[1]) * (face[3] - face[0]) < (xp - face[0]) * (face[4] - face[1])) ||
                ((yp - face[4]) * (face[6] - face[3]) < (xp - face[3]) * (face[7] - face[4])) ||
                ((yp - face[7]) * (face[0] - face[6]) < (xp - face[6]) * (face[1] - face[7])))
                continue;
            float w[3];
            for (int k = 0; k < 3; k++) {
                /* inv0*xi + inv1*yi + inv2 -> fma(inv0, xi, inv1*yi) + inv2 */
                float t = fmaf(finv[3 * k + 0], fxi, finv[3 * k + 1] * fyi);
                w[k] = finv[3 * k + 2] + t;
            }
            float w_sum = 0;
            for (int k = 0; k < 3; k++) {
                w[k] = clamp01_d(w[k]);
                w_sum = w_sum + w[k];
            }
            for (int k = 0; k < 3; k++) w[k] = w[k] / w_sum;
            /* 1. / (float sum): double divide rounded to float == fp32 reciprocal (innocuous double rounding) */
            const float s = (w[0] / face[2] + w[1] / face[5]) + w[2] / face[8];
            const float zp = 1.0f / s;
            if ((double)zp <= near_ || far_ <= (double)zp) continue;
            if (zp < depth_min) {
                depth_min = zp;
                face_index_min = fn;
                weight_min[0] = w[0];
                weight_min[1] = w[1];
                weight_min[2] = w[2];
                inv_min = finv;
            }
        }
        if (0 <= face_index_min) {
            depth_map[i] = depth_min;
            face_index_map[i] = face_index_min;
            for (int k = 0; k < 3; k++) weight_map[3 * i + k] = weight_min[k];
            if (face_inv_map)
                for (int k = 0; k < 9; k++) face_inv_map[9 * i + k] = inv_min[k];
        }
    }
}

/* ------------------------------------------------------------------ K4 ---- */
/* tex_z_batch0 != 0 reproduces rasterize.py:389 (vertex depths fetched from batch item 0). */
NRO_API void nro_texture(const float *faces, const float *textures, const int *face_index_map, const float *weight_map,
                         const float *depth_map, int bs, int nf, int is, int ts, double eps, int tex_z_batch0,
                         float *rgb_map, int *sampling_index_map /*nullable*/, float *sampling_weight_map /*nullable*/) {
    const int64_t npix = (int64_t)bs * is * is;
    const double tmax = (double)(ts - 1) - eps; /* `ts - 1 - eps`: int - double */
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < npix; i++) {
        const int face_index = face_index_map[i];
        if (face_index < 0) continue;
        const int bn = (int)(i / ((int64_t)is * is));
        const float *face = faces + ((int64_t)(tex_z_batch0 ? 0 : bn) * nf + face_index) * 9;
        const float *texture = textures + ((int64_t)bn * nf + face_index) * ts * ts * ts * 3;
        const float *weight = weight_map + 3 * i;
        const float depth = depth_map[i];
        float tif[3];
        for (int k = 0; k < 3; k++) {
            float t = (weight[k] * (float)(ts - 1)) * (depth / face[3 * k + 2]);
            t = (float)fmax((double)t, 0.0);
            t = (float)fmin((double)t, tmax);
            tif[k] = t;
        }
        float px[3] = {0, 0, 0};
        for (int pn = 0; pn < 8; pn++) {
            float w = 1;
            int ti[3];
            for (int k = 0; k < 3; k++) {
                const int ik = f2i_rz(tif[k]);
                if (((pn >> k) % 2) == 0) {
                    w = w * (((float)ik - tif[k]) + 1.0f); /* 1 - (t - i), bit-identical */
                    ti[k] = ik;
                } else {
                    w = w * (tif[k] - (float)ik);
                    ti[k] = ik + 1;
                }
            }
            const int isc = ti[0] * ts * ts + ti[1] * ts + ti[2];
            for (int k = 0; k < 3; k++) px[k] = fmaf(w, texture[isc * 3 + k], px[k]);
            if (sampling_index_map) sampling_index_map[8 * i + pn] = isc;
            if (sampling_weight_map) sampling_weight_map[8 * i + pn] = w;
        }
        for (int k = 0; k < 3; k++) rgb_map[3 * i + k] = px[k];
    }
}

/* ---------------------------------------------------- alpha / background ---- */
NRO_API void nro_compose(const int *face_index_map, int bs, int is, const float *background /*3 or bs*3*/,
                         int bg_per_batch, float *rgb_map /*nullable*/, float *alpha_map /*nullable*/) {
    const int64_t npix = (int64_t)bs * is * is;
    for (int64_t i = 0; i < npix; i++) {
        const int bn = (int)(i / ((int64_t)is * is));
        const float mask = face_index_map[i] >= 0 ? 1.0f : 0.0f;
        if (alpha_map && mask != 0.0f) alpha_map[i] = 1.0f;
        if (rgb_map) {
            const float *bg = background + (bg_per_batch ? 3 * bn : 0);
            for (int k = 0; k < 3; k++) rgb_map[3 * i + k] = rgb_map[3 * i + k] * mask + (1.0f - mask) * bg[k];
        }
    }
}

/* ------------------------------------------------------------------ K5 ---- */
static inline float k5_dist(float ratio, int d1, float d1_cross, int is, double eps) {
    float dist = (float)((double)(ratio * ((float)d1 - d1_cross)) * 2. / is);
    dist = (0 < dist) ? (float)((double)dist + eps) : (float)((double)dist - eps);
    return dist;
}

#define K5_ADD(j, term)                               \
    do {                                              \
        const float t_ = (term);                      \
        if (sum_fp64) grad_face64[j] -= (double)t_;   \
        else grad_face[j] -= t_;                      \
    } while (0)
NRO_API void nro_pixel_bwd(const float *faces, const int *face_index_map, const float *rgb_map, const float *alpha_map,
                           const float *grad_rgb_map, const float *grad_alpha_map, int bs, int nf, int is, double eps,
                           int return_rgb, int return_alpha, int sum_fp64, float *grad_faces) {
    /* sum_fp64: each term is the reference's fp32 diff_grad / dist, but the nine sums are kept in double.  The
     * reference adds up to ~S terms per crossing pixel in fp32, one after the other; at rasters of 2048 its own
     * rounding reaches 4e-4 of the tensor maximum, so a product that sums in another order is compared with this. */
    if (!return_rgb && !return_alpha) return;
    const int64_t n = (int64_t)bs * nf;
#pragma omp parallel for schedule(dynamic, 16)
    for (int64_t i = 0; i < n; i++) {
        const int bn = (int)(i / nf), fn = (int)(i % nf);
        const float *face = faces + 9 * i;
        float grad_face[9] = {0};
        double grad_face64[9] = {0};
        if (backside(face)) continue; /* `return`: grad_faces[i] keeps its zero initialisation */
        const int64_t base = (int64_t)bn * is * is;
        for (int edge_num = 0; edge_num < 3; edge_num++) {
            int pi[3];
            float pp[3][2];
            for (int num = 0; num < 3; num++) pi[num] = (edge_num + num) % 3;
            for (int num = 0; num < 3; num++)
                for (int dim = 0; dim < 2; dim++) pp[num][dim] = to_pixel(face[3 * pi[num] + dim], is);
            for (int axis = 0; axis < 2; axis++) {
                float p[3][2];
                for (int num = 0; num < 3; num++)
                    for (int dim = 0; dim < 2; dim++) p[num][dim] = pp[num][(dim + axis) % 2];
                int direction;
                if (axis == 0) direction = (p[0][0] < p[1][0]) ? -1 : 1;
                else direction = (p[0][0] < p[1][0]) ? 1 : -1;
                /* int <- double: truncation, as cvt.rzi.s32.f64 */
                const int d0_from = d2i_rz(fmax((double)ceilf(fminf(p[0][0], p[1][0])), 0.));
                const int d0_to = d2i_rz(fmin((double)fmaxf(p[0][0], p[1][0]), is - 1.));
                const float slope = (p[1][1] - p[0][1]) / (p[1][0] - p[0][0]);
                for (int d0 = d0_from; d0 <= d0_to; d0++) {
                    const float fd0 = (float)d0;
                    const float d1_cross = fmaf(fd0 - p[0][0], slope, p[0][1]);
                    int d1_in = (0 < direction) ? f2i_rz(floorf(d1_cross)) : f2i_rz(ceilf(d1_cross));
                    int d1_out = d1_in + direction;
                    if (d1_in < 0 || is <= d1_in) continue;
                    if (d1_out < 0 || is <= d1_out) continue;
                    int64_t map_index_in, map_index_out;
                    if (axis == 0) {
                        map_index_in = base + (int64_t)d1_in * is + d0;
                        map_index_out = base + (int64_t)d1_out * is + d0;
                    } else {
                        map_index_in = base + (int64_t)d0 * is + d1_in;
                        map_index_out = base + (int64_t)d0 * is + d1_out;
                    }
                    float alpha_in = 0, alpha_out = 0;
                    const float *rgb_in = NULL, *rgb_out = NULL;
                    if (return_alpha) {
                        alpha_in = alpha_map[map_index_in];
                        alpha_out = alpha_map[map_index_out];
                    }
                    if (return_rgb) {
                        rgb_in = rgb_map + map_index_in * 3;
                        rgb_out = rgb_map + map_index_out * 3;
                    }
                    const int map_offset = (axis == 0) ? is : 1;
                    const float ratio0 = (p[1][0] - p[0][0]) / (p[1][0] - fd0); /* used only if p[1][0] != d0 */
                    const float ratio1 = (p[1][0] - p[0][0]) / (fd0 - p[0][0]); /* used only if p[0][0] != d0 */
                    /* out */
                    if (face_index_map[map_index_in] == fn) {
                        const int d1_limit = (0 < direction) ? is - 1 : 0;
                        int d1_from = d1_out < d1_limit ? d1_out : d1_limit;
                        if (d1_from < 0) d1_from = 0;
                        int d1_to = d1_out > d1_limit ? d1_out : d1_limit;
                        if (d1_to > is - 1) d1_to = is - 1;
                        int64_t mi = (axis == 0) ? base + (int64_t)d1_from * is + d0 : base + (int64_t)d0 * is + d1_from;
                        for (int d1 = d1_from; d1 <= d1_to; d1++, mi += map_offset) {
                            float diff_grad = 0;
                            if (return_alpha) diff_grad = fmaf(alpha_map[mi] - alpha_in, grad_alpha_map[mi], diff_grad);
                            if (return_rgb)
                                for (int k = 0; k < 3; k++)
                                    diff_grad = fmaf(rgb_map[mi * 3 + k] - rgb_in[k], grad_rgb_map[mi * 3 + k], diff_grad);
                            if (diff_grad <= 0) continue;
                            if (p[1][0] != fd0) {
                                float dist = k5_dist(ratio0, d1, d1_cross, is, eps);
                                K5_ADD(pi[0] * 3 + (1 - axis), diff_grad / dist);
                            }
                            if (p[0][0] != fd0) {
                                float dist = k5_dist(ratio1, d1, d1_cross, is, eps);
                                K5_ADD(pi[1] * 3 + (1 - axis), diff_grad / dist);
                            }
                        }
                    }
                    /* in */
                    {
                        float ba, bb, ea, eb; /* base / end of the opposite edge that this column leaves through */
                        if ((fd0 - p[0][0]) * (fd0 - p[2][0]) < 0) {
                            ba = p[0][0]; bb = p[0][1]; ea = p[2][0]; eb = p[2][1];
                        } else {
                            ba = p[2][0]; bb = p[2][1]; ea = p[1][0]; eb = p[1][1];
                        }
                        const float d0_cross2 = fmaf(fd0 - ba, (eb - bb) / (ea - ba), bb);
                        const int d1_limit = (0 < direction) ? f2i_rz(ceilf(d0_cross2)) : f2i_rz(floorf(d0_cross2));
                        int d1_from = d1_in < d1_limit ? d1_in : d1_limit;
                        if (d1_from < 0) d1_from = 0;
                        int d1_to = d1_in > d1_limit ? d1_in : d1_limit;
                        if (d1_to > is - 1) d1_to = is - 1;
                        int64_t mi = (axis == 0) ? base + (int64_t)d1_from * is + d0 : base + (int64_t)d0 * is + d1_from;
                        for (int d1 = d1_from; d1 <= d1_to; d1++, mi += map_offset) {
                            if (face_index_map[mi] != fn) continue;
                            float diff_grad = 0;
                            if (return_alpha) diff_grad = fmaf(alpha_map[mi] - alpha_out, grad_alpha_map[mi], diff_grad);
                            if (return_rgb)
                                for (int k = 0; k < 3; k++)
                                    diff_grad = fmaf(rgb_map[mi * 3 + k] - rgb_out[k], grad_rgb_map[mi * 3 + k], diff_grad);
                            if (diff_grad <= 0) continue;
                            if (p[1][0] != fd0) {
                                float dist = k5_dist(ratio0, d1, d1_cross, is, eps);
                                K5_ADD(pi[0] * 3 + (1 - axis), diff_grad / dist);
                            }
                            if (p[0][0] != fd0) {
                                float dist = k5_dist(ratio1, d1, d1_cross, is, eps);
                                K5_ADD(pi[1] * 3 + (1 - axis), diff_grad / dist);
                            }
                        }
                    }
                }
            }
        }
        for (int k = 0; k < 9; k++) grad_faces[i * 9 + k] = sum_fp64 ? (float)grad_face64[k] : grad_face[k];
    }
}

/* ------------------------------------------------------------------ K6 ---- */
/* The reference scatters with float atomics (order-nondeterministic); the oracle sums in pixel order.
 * Sampling indices / weights are recomputed (bit-identically to nro_texture) when the maps are not given. */
NRO_API void nro_texture_bwd(const int *face_index_map, const float *sampling_weight_map, const int *sampling_index_map,
                             const float *grad_rgb_map, int bs, int nf, int is, int ts, float *grad_textures) {
    const int64_t per = (int64_t)is * is;
    for (int64_t i = 0; i < (int64_t)bs * per; i++) {
        const int face_index = face_index_map[i];
        if (face_index < 0) continue;
        const int bn = (int)(i / per);
        float *gt = grad_textures + ((int64_t)bn * nf + face_index) * ts * ts * ts * 3;
        for (int pn = 0; pn < 8; pn++) {
            const float w = sampling_weight_map[8 * i + pn];
            const int isc = sampling_index_map[8 * i + pn];
            for (int k = 0; k < 3; k++) gt[isc * 3 + k] += w * grad_rgb_map[3 * i + k];
        }
    }
}

/* ------------------------------------------------------------------ K7 ---- */
NRO_API void nro_depth_bwd(const float *faces, const float *depth_map, const int *face_index_map,
                           const float *face_inv_map, const float *weight_map, const float *grad_depth_map, int bs,
                           int nf, int is, float *grad_faces) {
    const int64_t per = (int64_t)is * is;
    for (int64_t i = 0; i < (int64_t)bs * per; i++) {
        const int fn = face_index_map[i];
        if (fn < 0) continue;
        const int bn = (int)(i / per);
        const float *face = faces + ((int64_t)bn * nf + fn) * 9;
        const float depth = depth_map[i];
        const float depth2 = depth * depth;
        const float *finv = face_inv_map + 9 * i;
        const float *weight = weight_map + 3 * i;
        const float g = grad_depth_map[i];
        float *gf = grad_faces + ((int64_t)bn * nf + fn) * 9;
        for (int k = 0; k < 3; k++) {
            const float z_k = face[3 * k + 2];
            gf[3 * k + 2] += ((g * weight[k]) * depth2) / (z_k * z_k);
        }
        float tmp[3] = {0, 0, 0};
        for (int k = 0; k < 3; k++)
            for (int l = 0; l < 3; l++) tmp[k] = tmp[k] - finv[3 * l + k] / face[3 * l + 2];
        for (int k = 0; k < 3; k++)
            for (int l = 0; l < 2; l++) gf[3 * k + l] += (((((-g) * tmp[l]) * weight[k]) * depth2) * (float)is) * 0.5f;
    }
}

/* ---------------------------------------------------------------------------------------------------------------
 * Texture baking of load_obj (load_obj.py:88-137).  Same operation order as the reference build evaluates (dims via a
 * double division rounded to float, IEEE float divisions by (d0 + d1) + d2, pos = fma(f2, d2, fma(f0, d0, f1 * d1)) *
 * (size - 1), taps blended as an fma chain in source order).  Texel (0,0,0) is 0/0 = NaN like the reference.  The
 * reference reads one row / column past the image when a coordinate is exactly 1 (with weight 0); here those taps
 * are clamped into the image.  `image` [H,W,3] is already flipped (load_obj.py:82). */
NRO_API void nro_bake_textures(const float *image, const float *uv_faces, const int *is_update, int64_t nf, int ts, int H,
                               int W, float *textures) {
    const int t3 = ts * ts * ts;
    const int64_t n = nf * t3;
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < n; i++) {
        const int64_t fn = i / t3;
        if (is_update && is_update[fn] == 0) continue;
        const int r = (int)(i - fn * t3);
        const double den = (double)ts - 1.0;
        float d0 = (float)((double)((r / (ts * ts)) % ts) / den);
        float d1 = (float)((double)((r / ts) % ts) / den);
        float d2 = (float)((double)(r % ts) / den);
        const float sum = (d0 + d1) + d2;
        d0 = d0 / sum; d1 = d1 / sum; d2 = d2 / sum;
        const float *f = uv_faces + fn * 6;
        const float pos_x = fmaf(f[4], d2, fmaf(f[0], d0, f[2] * d1)) * (float)(W - 1);
        const float pos_y = fmaf(f[5], d2, fmaf(f[1], d0, f[3] * d1)) * (float)(H - 1);
        const int ix = f2i_rz(pos_x), iy = f2i_rz(pos_y), iy1 = f2i_rz(pos_y + 1.0f);
        const float wx1 = pos_x - (float)ix, wy1 = pos_y - (float)iy;
        const float wx0 = 1.0f - wx1, wy0 = 1.0f - wy1;
        const float w00 = wx0 * wy0, w01 = wx0 * wy1, w10 = wx1 * wy0, w11 = wx1 * wy1;
#define NRO_CLAMP(v, hi) ((v) < 0 ? 0 : ((v) > (hi) ? (hi) : (v)))
        const int cx0 = NRO_CLAMP(ix, W - 1), cx1 = NRO_CLAMP(ix + 1, W - 1);
        const int cy0 = NRO_CLAMP(iy, H - 1), cy1 = NRO_CLAMP(iy1, H - 1);
#undef NRO_CLAMP
        const float *p00 = image + ((int64_t)cy0 * W + cx0) * 3, *p01 = image + ((int64_t)cy1 * W + cx0) * 3;
        const float *p10 = image + ((int64_t)cy0 * W + cx1) * 3, *p11 = image + ((int64_t)cy1 * W + cx1) * 3;
        for (int k = 0; k < 3; k++) {
            float c = w00 * p00[k];
            c = fmaf(w01, p01[k], c);
            c = fmaf(w10, p10[k], c);
            c = fmaf(w11, p11[k], c);
            textures[i * 3 + k] = c;
        }
    }
}

NRO_API int nro_num_threads(void) {
#ifdef _OPENMP
    return omp_get_max_threads();
#else
    return 1;
#endif
}

NRO_API void nro_set_num_threads(int n) {
#ifdef _OPENMP
    if (n > 0) omp_set_num_threads(n);
#else
    (void)n;
#endif
}
