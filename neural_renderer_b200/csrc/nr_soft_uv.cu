// nr_soft_uv.cu -- soft RGB through a texture image (nr_b200_soft_rgb_uv / nr_b200_soft_rgb_uv_backward,
// include/nr_b200.h): the soft RGB of nr_soft_rgb.cu with C_j sampled bilinearly from an image, or trilinearly from its
// mip pyramid, at the perspective-correct UV of the face's own corners.
//
// The host checks, the workspace and the binning (setup, scan, keys, sort) are nr_soft_rgb.cu's (nr_internal.h); the
// forward traversal is nr_soft_rgb.cuh's with the image sampler below.  New kernels:
//   k_soft_uv_fwd<K, kMip>  soft_rgb_fwd_body with ImageSampler<kMip>
//   k_soft_uv_bwd<K, kMip>  the soft RGB backward with the image sampler's chain: 18 partials per face (x, y, z of three
//                           vertices, three light channels, u and v of three UV corners) reduced over the warp and the CTA;
//                           each lane sends its image taps to global memory as vector reductions (merging the taps of
//                           neighbouring lanes that hit the same cells, as image_grad does, measured slower: DESIGN.md 4q)
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <string.h>

#include "nr_b200.h"
#include "nr_internal.h"
#include "nr_soft.cuh"
#include "nr_soft_rgb.cuh"
#include "nr_texture.cuh"

namespace {

struct SoftUvParams {
    SoftRgbParams r;   // r.tex: the image or pyramid and face_uvs (nr_internal::make_texture)
    float* grad_uvs;   // like face_uvs, or nullptr
};

// The UV, uv = sum_k l'_k uv_k with l'_k = l_k zp / z_k (nr::pixel_uv), and the levels it samples.  The trilinear level
// of detail is mip_lod's with the face's screen-barycentric derivatives in place of K1's inverse: lam_k = c_{k+1} / A,
// c_m = e_m x (p - v_m), so d lam_k / d column = -(2/S) e_{k+1,y} / A and d lam_k / d row = -(2/S) e_{k+1,x} / A.
template <bool kMip>
__device__ __forceinline__ nr::LevelPair uv_point(const SoftRgbParams& p, int b, int f, const SoftBary& bc, const float4& z,
                                                  const float4* rec, float uv[6], float& u, float& v) {
    nr::face_uvs(p.tex, b, f, false, uv);
    nr::pixel_uv(bc.l, bc.zp, z.x, z.y, z.z, uv, u, v);
    float inv[9] = {0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f};
    if constexpr (kMip) {
        const float q = __fdiv_rn(-2.0f, __fmul_rn((float)p.s.S, z.w));
#pragma unroll
        for (int k = 0; k < 3; k++) {
            const float4 e = rec[k == 2 ? 0 : k + 1];
            inv[3 * k] = __fmul_rn(q, e.w);
            inv[3 * k + 1] = __fmul_rn(q, e.z);
        }
    }
    return nr::level_pair<kMip>(p.tex, inv, bc.l, bc.zp, z.x, z.y, z.z, uv);
}

// the forward colour: uv_blend (kMip: mip_blend) at the pixel's UV, every tap times face_light first
template <bool kMip>
struct ImageSampler {
    __device__ __forceinline__ void color(const SoftRgbParams& p, int b, int f, const SoftBary& bc, const float4& z,
                                          const float4* rec, float& r, float& g, float& bl) const {
        float uv[6], u, v, c[3];
        const nr::LevelPair lp = uv_point<kMip>(p, b, f, bc, z, rec, uv, u, v);
        const float* img = p.tex.tex + p.tex.img_off(b);
        float l0 = 1.0f, l1 = 1.0f, l2 = 1.0f;
        const bool lit = p.light != nullptr;
        if (lit) {
            const float* lt = p.light + ((size_t)b * p.s.F + f) * 3;
            l0 = __ldg(lt); l1 = __ldg(lt + 1); l2 = __ldg(lt + 2);
        }
        if constexpr (kMip) {
            nr::MipLevels m;
            m.l0 = lp.l[0]; m.l1 = lp.l[1]; m.f = lp.a[1];
            if (lit) nr::mip_blend<true>(img, p.tex.mip, m, u, v, l0, l1, l2, c);
            else nr::mip_blend<false>(img, p.tex.mip, m, u, v, l0, l1, l2, c);
        } else {
            const nr::UvTaps t = nr::uv_taps(u, v, p.tex.Ht, p.tex.Wt);
            if (lit) nr::uv_blend<true>(img, p.tex.Wt, t, l0, l1, l2, c);
            else nr::uv_blend<false>(img, p.tex.Wt, t, l0, l1, l2, c);
        }
        r = c[0]; g = c[1]; bl = c[2];
    }
};

// ------------------------------------------------------------------------------------------------ k_soft_uv_fwd
template <typename K, bool kMip>
__global__ void __launch_bounds__(kThreads) k_soft_uv_fwd(const __grid_constant__ SoftUvParams p) {
    __shared__ float4 s_rec[kThreads * 4];
    __shared__ float4 s_z[kThreads];
    __shared__ int s_face[kThreads];
    __shared__ int s_wn[kWarps];
    soft_rgb_fwd_body<K>(p.r, ImageSampler<kMip>{}, s_rec, s_z, s_face, s_wn);
}

// ------------------------------------------------------------------------------------------------ k_soft_uv_bwd
constexpr int kUvPartials = 18;  // per face: (x, y) of 3 vertices, z of 3 vertices, 3 light channels, (u, v) of 3 corners

template <typename K, bool kMip>
__global__ void __launch_bounds__(kThreads) k_soft_uv_bwd(const __grid_constant__ SoftUvParams P) {
    constexpr int kPairs = kMip ? 4 : 2;  // tap rows: two per sampled level
    __shared__ float4 s_rec[kThreads * 4];
    __shared__ float4 s_z[kThreads];
    __shared__ int s_face[kThreads];
    __shared__ float s_acc[kThreads * kUvPartials];
    __shared__ int s_wn[kWarps];
    const SoftRgbParams& p = P.r;
    const int tile = blockIdx.x, b = blockIdx.y;
    const int tx = tile % p.s.ntx, ty = tile / p.s.ntx;
    const int col = tx * kTile + (threadIdx.x % kTile), row = ty * kTile + (threadIdx.x / kTile);
    const int S = p.s.S, lane = threadIdx.x & 31;
    const float px = soft_centre(col, S), py = soft_centre(S - 1 - row, S);
    const size_t seg = (size_t)b * (p.s.ntiles + 1);
    const int n_tile = p.s.cnt[seg + tile], n_all = n_tile + p.s.cnt[seg + p.s.ntiles];
    if (n_all == 0) return;  // CTA-uniform
    const uint32_t img_off = p.tex.img_off(b);
    float ga = 0.0f, gr[3] = {0.0f, 0.0f, 0.0f}, out[3] = {0.0f, 0.0f, 0.0f}, Z = 1.0f, zref = 0.0f;
    if (row < S && col < S) {
        const size_t plane = (size_t)S * S, o = (size_t)row * S + col;
        if (p.s.g) ga = __ldg(p.s.g + b * plane + o) * (1.0f - __ldg(p.s.alpha + b * plane + o));
        if (p.g_rgb) {
#pragma unroll
            for (int c = 0; c < 3; c++) {
                gr[c] = __ldg(p.g_rgb + ((size_t)b * 3 + c) * plane + o);
                out[c] = __ldg(p.rgb + ((size_t)b * 3 + c) * plane + o);
            }
        }
        Z = __ldg(p.state + (size_t)b * 2 * plane + o);
        zref = __ldg(p.state + (size_t)b * 2 * plane + plane + o);
    }
    const float iZ = __frcp_rn(Z);
    const bool want_rgb = gr[0] != 0.0f || gr[1] != 0.0f || gr[2] != 0.0f;
    const bool active = ga != 0.0f || want_rgb;
    // h = g . (C - rgb) / Z = (g . C) / Z - (g . rgb) / Z
    const float g_out = __fmul_rn(__fmaf_rn(gr[2], out[2], __fmaf_rn(gr[1], out[1], __fmul_rn(gr[0], out[0]))), iZ);
    for (int i = threadIdx.x; i < kThreads * kUvPartials; i += kThreads) s_acc[i] = 0.0f;
    for (int next = 0; next < n_all; next += kThreads) {
        const int n = stage_rgb<K>(p, b, tile, tx, ty, n_tile, n_all, next, s_rec, s_z, s_face, s_wn);
        for (int j = 0; j < n; j++) {
            float x = 0.0f, t = 0.0f, qx = 0.0f, qy = 0.0f, c[3];
            int k = 0;
            const bool hit = active && soft_eval(s_rec + 4 * j, px, py, p.s.inv_sigma, p.s.cut, x, k, t, qx, qy, c);
            if (!__any_sync(0xffffffffu, hit)) continue;  // warp-uniform
            const int f = s_face[j];
            float v[kUvPartials];
#pragma unroll
            for (int m = 0; m < kUvPartials; m++) v[m] = 0.0f;
            bool tex_hit = false;
            float u = 0.0f, vv = 0.0f;
            nr::LevelPair lp = {{0, 0}, {1.0f, 0.0f}, 1};
            float gl[3] = {0.0f, 0.0f, 0.0f};  // d loss / d unlit sample_c = d loss / d C_c * light_c
            if (hit) {
                const float D = soft_sigmoid(x);
                float gx = __fmul_rn(ga, D);  // d loss / d x_j
                const float4 z = s_z[j];
                if (want_rgb && z.w != 0.0f) {
                    const SoftBary bc = soft_bary(c, z);
                    const float w = __fmul_rn(D, expf(__fmul_rn(__fsub_rn(zref, bc.zp), p.inv_fg)));
                    if (w != 0.0f) {
                        const float zz[3] = {z.x, z.y, z.z};
                        float L[3] = {1.0f, 1.0f, 1.0f};
                        if (p.light) {
                            const float* lt = p.light + ((size_t)b * p.s.F + f) * 3;
                            L[0] = __ldg(lt); L[1] = __ldg(lt + 1); L[2] = __ldg(lt + 2);
                        }
                        const float wz = __fmul_rn(w, iZ);
                        float gCc[3];  // d loss / d C_c
#pragma unroll
                        for (int ch = 0; ch < 3; ch++) {
                            gCc[ch] = __fmul_rn(wz, gr[ch]);
                            gl[ch] = __fmul_rn(gCc[ch], L[ch]);
                        }
                        float uv[6], su[3], gu, gv;
                        lp = uv_point<kMip>(p, b, f, bc, z, s_rec + 4 * j, uv, u, vv);
                        const nr::UvTaps t0 = nr::uv_taps(u, vv, p.tex.level_h<kMip>(lp.l[0]), p.tex.level_w<kMip>(lp.l[0]));
                        nr::image_sample_grad<kMip>(p.tex, p.tex.tex + img_off, lp, t0, u, vv, gl, su, gu, gv);
                        const float gC = __fmaf_rn(gr[2], __fmul_rn(su[2], L[2]),
                                                   __fmaf_rn(gr[1], __fmul_rn(su[1], L[1]), __fmul_rn(gr[0], __fmul_rn(su[0], L[0]))));
                        const float h = __fsub_rn(__fmul_rn(gC, iZ), g_out);
                        gx = __fmaf_rn(__fmul_rn(w, 1.0f - D), h, gx);
                        float dzp = -__fmul_rn(__fmul_rn(w, h), p.inv_fg);  // d loss / d zp through the weight
#pragma unroll
                        for (int ch = 0; ch < 3; ch++) v[9 + ch] = __fmul_rn(gCc[ch], su[ch]);
                        tex_hit = p.grad_tex != nullptr;
                        // uv = sum_a l'_a uv_a, l'_a = l_a r_a, r_a = zp / z_a: d loss / d uv_a = l'_a (gu, gv) and
                        // d loss / d l'_a = gu u_a + gv v_a, on through l_a, zp and z_a (the cells and the clamp held fixed)
                        float dl[3], dz[3];
#pragma unroll
                        for (int a = 0; a < 3; a++) {
                            const float r = __fdiv_rn(bc.zp, zz[a]);
                            const float lp_a = __fmul_rn(bc.l[a], r);
                            v[12 + 2 * a] = __fmul_rn(lp_a, gu);
                            v[13 + 2 * a] = __fmul_rn(lp_a, gv);
                            const float Gt = __fmaf_rn(gv, uv[2 * a + 1], __fmul_rn(gu, uv[2 * a]));
                            dl[a] = __fmul_rn(Gt, r);
                            dzp = __fmaf_rn(Gt, __fdiv_rn(bc.l[a], zz[a]), dzp);
                            dz[a] = -__fmul_rn(__fmul_rn(Gt, bc.l[a]), __fdiv_rn(r, zz[a]));
                        }
                        // zp = 1 / Q, Q = sum_k l_k / z_k
                        const float dQ = -__fmul_rn(__fmul_rn(bc.zp, bc.zp), dzp);
                        float sl = 0.0f;
#pragma unroll
                        for (int a = 0; a < 3; a++) {
                            dl[a] = __fmaf_rn(dQ, __frcp_rn(zz[a]), dl[a]);
                            dz[a] = __fsub_rn(dz[a], __fmul_rn(dQ, __fdiv_rn(__fdiv_rn(bc.l[a], zz[a]), zz[a])));
                            v[6 + a] = dz[a];
                            sl = __fmaf_rn(bc.l[a], dl[a], sl);
                        }
                        // l = lh / s, lh = clamp(lam, 0, 1), lam_m = c_{m+1} / A
                        float dlam[3], sg = 0.0f;
#pragma unroll
                        for (int a = 0; a < 3; a++) {
                            const bool in = bc.lam[a] >= 0.0f && bc.lam[a] <= 1.0f;
                            dlam[a] = in ? __fdiv_rn(__fsub_rn(dl[a], sl), bc.s) : 0.0f;
                            sg = __fmaf_rn(dlam[a], bc.lam[a], sg);
                        }
                        // c_e = (b - a) x (p - a) of edge e = (v_e, v_e+1): d c / d a = (by - py, px - bx), d c / d b = (py - ay, ax - px)
                        const float4* r = s_rec + 4 * j;
#pragma unroll
                        for (int e = 0; e < 3; e++) {
                            const float dc = __fdiv_rn(__fsub_rn(dlam[e == 0 ? 2 : e - 1], sg), z.w);
                            const float4 ed = r[e];
                            const float dx = __fsub_rn(px, ed.x), dy = __fsub_rn(py, ed.y);
                            const int nb = e == 2 ? 0 : e + 1;
                            v[2 * e] = __fmaf_rn(dc, __fsub_rn(ed.w, dy), v[2 * e]);
                            v[2 * e + 1] = __fmaf_rn(dc, __fsub_rn(dx, ed.z), v[2 * e + 1]);
                            v[2 * nb] = __fmaf_rn(dc, dy, v[2 * nb]);
                            v[2 * nb + 1] = __fmaf_rn(dc, -dx, v[2 * nb + 1]);
                        }
                    }
                }
                // d x / d(d^2) = +-1/sigma; d(d^2)/da = -2 (1 - t)(p - q), d(d^2)/db = -2 t (p - q) for edge (a, b)
                const float s = gx * (x >= 0.0f ? -2.0f : 2.0f) * p.s.inv_sigma;
                const float wa = s * (1.0f - t), wb = s * t;
#pragma unroll
                for (int m = 0; m < 3; m++) {
                    const bool is_a = m == k, is_b = m == (k == 2 ? 0 : k + 1);
                    const float wm = is_a ? wa : (is_b ? wb : 0.0f);
                    v[2 * m] = __fmaf_rn(wm, qx, v[2 * m]);
                    v[2 * m + 1] = __fmaf_rn(wm, qy, v[2 * m + 1]);
                }
            }
            // the image taps: a_l w_xy gl_c per tap, one horizontal pair (6 floats) per tap row and level
            if (__any_sync(0xffffffffu, tex_hit)) {
                float val[kPairs][6];
                float* tp[kPairs];
                bool adjacent[kPairs / 2];
#pragma unroll
                for (int q = 0; q < kPairs; q++) {
                    tp[q] = nullptr;
#pragma unroll
                    for (int e = 0; e < 6; e++) val[q][e] = 0.0f;
                }
#pragma unroll
                for (int q = 0; q < kPairs / 2; q++) adjacent[q] = true;
                if (tex_hit) {
                    float* gi = p.grad_tex + img_off;
#pragma unroll
                    for (int q = 0; q < kPairs / 2; q++) {
                        if (q >= lp.n) break;
                        const int Hl = p.tex.level_h<kMip>(lp.l[q]), Wl = p.tex.level_w<kMip>(lp.l[q]);
                        const uint32_t loff = p.tex.level_off<kMip>(lp.l[q]);
                        const nr::UvTaps tq = nr::uv_taps(u, vv, Hl, Wl);
                        const uint32_t row3 = (uint32_t)Wl * 3u;
                        tp[2 * q] = gi + loff + (uint32_t)tq.r0 * row3 + (uint32_t)tq.x0 * 3u;
                        tp[2 * q + 1] = gi + loff + (uint32_t)tq.r1 * row3 + (uint32_t)tq.x0 * 3u;
                        adjacent[q] = tq.x1 != tq.x0;
                        const float h0 = __fmul_rn(lp.a[q], gl[0]), h1 = __fmul_rn(lp.a[q], gl[1]), h2 = __fmul_rn(lp.a[q], gl[2]);
                        float* v0 = val[2 * q];
                        float* v1 = val[2 * q + 1];
                        v0[0] = tq.w00 * h0; v0[1] = tq.w00 * h1; v0[2] = tq.w00 * h2;
                        v0[3] = tq.w10 * h0; v0[4] = tq.w10 * h1; v0[5] = tq.w10 * h2;
                        v1[0] = tq.w01 * h0; v1[1] = tq.w01 * h1; v1[2] = tq.w01 * h2;
                        v1[3] = tq.w11 * h0; v1[4] = tq.w11 * h1; v1[5] = tq.w11 * h2;
                    }
                }
                if (tex_hit) {
#pragma unroll
                    for (int q = 0; q < kPairs; q++) {
                        if (tp[q] == nullptr) break;  // level l1 has no taps when f == 0
                        if (adjacent[q >> 1]) {
                            nr::red_add_6(tp[q], val[q]);
                        } else {
                            float* g = tp[q];
                            atomicAdd(g, val[q][0] + val[q][3]); atomicAdd(g + 1, val[q][1] + val[q][4]);
                            atomicAdd(g + 2, val[q][2] + val[q][5]);
                        }
                    }
                }
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1)
#pragma unroll
                for (int m = 0; m < kUvPartials; m++) v[m] += __shfl_xor_sync(0xffffffffu, v[m], o);
            if (lane < kUvPartials) {
                float mine = v[0];
#pragma unroll
                for (int m = 1; m < kUvPartials; m++) if (lane == m) mine = v[m];
                if (mine != 0.0f) atomicAdd(&s_acc[j * kUvPartials + lane], mine);
            }
        }
        __syncthreads();
        // one set of global atomics per face of the round: thread (face slot, vertex, light or UV corners)
        for (int i = threadIdx.x; i < n * 5; i += kThreads) {
            const int j = i / 5, m = i % 5;
            float* a = s_acc + j * kUvPartials;
            if (m < 3) {
                const float gx = a[2 * m], gy = a[2 * m + 1], gz = a[6 + m];
                a[2 * m] = 0.0f; a[2 * m + 1] = 0.0f; a[6 + m] = 0.0f;
                if (gx == 0.0f && gy == 0.0f && gz == 0.0f) continue;
                float* gv = nr::face_grad_vertex(p.s.dst, b, s_face[j], m);
                if (gv) { atomicAdd(gv, gx); atomicAdd(gv + 1, gy); atomicAdd(gv + 2, gz); }
            } else if (m == 3) {
                const float l0 = a[9], l1 = a[10], l2 = a[11];
                a[9] = 0.0f; a[10] = 0.0f; a[11] = 0.0f;
                if (!p.grad_light || (l0 == 0.0f && l1 == 0.0f && l2 == 0.0f)) continue;
                float* gl = p.grad_light + ((size_t)b * p.s.F + s_face[j]) * 3;
                atomicAdd(gl, l0); atomicAdd(gl + 1, l1); atomicAdd(gl + 2, l2);
            } else {
                float g[6];
                bool any = false;
#pragma unroll
                for (int e = 0; e < 6; e++) { g[e] = a[12 + e]; a[12 + e] = 0.0f; any = any || g[e] != 0.0f; }
                if (!P.grad_uvs || !any) continue;
                float* gu = P.grad_uvs + p.tex.uv_off(b, s_face[j]);
#pragma unroll
                for (int e = 0; e < 6; e++) atomicAdd(gu + e, g[e]);
            }
        }
        __syncthreads();
    }
}

constexpr uint32_t kSoftUvFlags = NR_FACES_INDEXED | NR_INDICES_SHARED | NR_TEX_SHARED | NR_GRAD_ACCUMULATE | NR_TEX_UV |
                                  NR_UV_SHARED | NR_TEX_MIPMAP;

// the fields of a texture-image call that nr_internal::make_texture reads (NR_RETURN_RGB added: the soft RGB is RGB)
struct UvTexArgs {
    uint32_t flags;
    int32_t batch_size, num_faces, texture_size;
    const float* textures;
    float eps;
    const float* face_uvs;
    int32_t texture_height, texture_width;
};

// the host checks of both entry points (uv non-NULL); fills `p`, `L` and the floats of the image / pyramid and UV buffers
int soft_uv_setup(const nr_b200_soft_rgb_args* a, const nr_b200_soft_uv_args* uv, bool backward, SoftUvParams* p,
                  SoftRgbLayout* L, size_t* tex_floats, size_t* uv_floats) {
    nr_internal::launch_count() = 0;
    if (!a || a->struct_size != sizeof(nr_b200_soft_rgb_args) || uv->struct_size != sizeof(nr_b200_soft_uv_args))
        return NR_ERR_INVALID_ARG;
    if (!(a->flags & NR_TEX_UV)) return NR_ERR_INVALID_ARG;
    memset(p, 0, sizeof(*p));
    int rc = nr_internal::soft_rgb_check(a, kSoftUvFlags, nr_internal::kSoftImage, backward, &p->r);
    if (rc != NR_OK) return rc;
    const UvTexArgs t = {a->flags | NR_RETURN_RGB, a->batch_size, a->num_faces, 0, a->textures, 0.0f, uv->face_uvs,
                         uv->texture_height, uv->texture_width};
    rc = nr_internal::make_texture(&t, &p->r.tex, tex_floats, uv_floats);  // NR_ERR_UNSUPPORTED after every invalid arg
    if (rc != NR_OK) return rc;
    p->grad_uvs = backward ? uv->grad_face_uvs : nullptr;
    return nr_internal::soft_rgb_workspace(a, &p->r, L);
}

template <typename K, bool kMip>
void soft_uv_launch(const SoftUvParams& p, bool backward, cudaStream_t s) {
    const dim3 grid((unsigned)p.r.s.ntiles, (unsigned)p.r.s.B);
    if (backward) {
        nr_internal::LaunchScope ls("k_soft_uv_bwd", s);
        k_soft_uv_bwd<K, kMip><<<grid, kThreads, 0, s>>>(p);
    } else {
        nr_internal::LaunchScope ls("k_soft_uv_fwd", s);
        k_soft_uv_fwd<K, kMip><<<grid, kThreads, 0, s>>>(p);
    }
}

// the binning (sorted for the forward), then the traversal
int soft_uv_run(SoftUvParams& p, const SoftRgbLayout& L, bool backward, cudaStream_t s) {
    if (nr_internal::soft_rgb_bin(&p.r, &L, !backward, s) != NR_OK) return NR_ERR_CUDA;
    const bool mip = p.r.tex.mip.levels > 0;
    if (L.wide) mip ? soft_uv_launch<unsigned long long, true>(p, backward, s) : soft_uv_launch<unsigned long long, false>(p, backward, s);
    else mip ? soft_uv_launch<uint32_t, true>(p, backward, s) : soft_uv_launch<uint32_t, false>(p, backward, s);
    return cudaGetLastError() == cudaSuccess ? NR_OK : NR_ERR_CUDA;
}

}  // namespace

extern "C" int nr_b200_soft_rgb_uv(const nr_b200_soft_rgb_args* args, const nr_b200_soft_uv_args* uv, void* cuda_stream) {
    if (!uv) return nr_b200_soft_rgb(args, cuda_stream);
    SoftUvParams p;
    SoftRgbLayout L;
    size_t tex_floats, uv_floats;
    const int rc = soft_uv_setup(args, uv, false, &p, &L, &tex_floats, &uv_floats);
    if (rc != NR_OK) return rc;
    return soft_uv_run(p, L, false, (cudaStream_t)cuda_stream);
}

extern "C" int nr_b200_soft_rgb_uv_backward(const nr_b200_soft_rgb_args* args, const nr_b200_soft_uv_args* uv,
                                            void* cuda_stream) {
    if (!uv) return nr_b200_soft_rgb_backward(args, cuda_stream);
    SoftUvParams p;
    SoftRgbLayout L;
    size_t tex_floats, uv_floats;
    const int rc = soft_uv_setup(args, uv, true, &p, &L, &tex_floats, &uv_floats);
    if (rc != NR_OK) return rc;
    const nr_b200_soft_rgb_args* a = args;
    cudaStream_t s = (cudaStream_t)cuda_stream;
    if (!(a->flags & NR_GRAD_ACCUMULATE) &&
        nr_internal::zero_grads({nr_internal::geometry_grad(a), {a->grad_textures, tex_floats * sizeof(float)},
                                 {a->grad_face_light, (size_t)p.r.s.B * p.r.s.F * 3 * sizeof(float)},
                                 {p.grad_uvs, uv_floats * sizeof(float)}},
                                s) != cudaSuccess)
        return NR_ERR_CUDA;
    if (!a->grad_alpha && !a->grad_rgb) return cudaGetLastError() == cudaSuccess ? NR_OK : NR_ERR_CUDA;
    return soft_uv_run(p, L, true, s);
}
