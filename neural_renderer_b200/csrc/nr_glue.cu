// nr_glue.cu -- the step either side of the rasterizer: vertices_to_faces (reference
// neural_renderer/vertices_to_faces.py:4-21) as a fused gather (forward) / scatter-add (backward).
//
// The reference forms d loss / d vertex through Chainer's generic get_item backward (a scatter-add of the
// [B,F,3,3] face gradients into [B*Nv,3]); here it is one pass of fp32 vector reductions into the vertex gradient,
// reading grad_faces exactly once (SURVEY.md section 8(f), rank 1).
//
// Camera pipeline (SURVEY.md section 8(f), rank 2): look_at / look (look_at.py:30-44, look.py:29-43: subtract the
// eye, rotate into the camera frame) and perspective (perspective.py:10-18: x / z / tan(angle)) as ONE per-vertex
// kernel each way; the backward also reduces the gradients of the 3x3 rotation, the eye and the width per batch
// item, so camera-pose optimisation (examples/example4.py) differentiates through it.
//
// Lighting (SURVEY.md section 8(f), rank 3): the per-face RGB factor of lighting.py:29-51 straight from vertices and
// face indices (no gathered [B,F,3,3] tensor), and its backward as a scatter-add into the vertex gradient.  The
// factor itself is applied inside the rasterizer's sampler (nr_b200_forward_args.face_light).
//
// Smooth shading (include/nr_b200.h): area-weighted vertex normals and the per-corner Lambertian light the rasterizer
// interpolates (nr_b200_forward_args.corner_light).  The normal sums are deterministic: the corners are stable-sorted by
// vertex (cub radix sort) and every vertex adds its corners' face normals in ascending (face, corner) order.
//
// Texture baking (SURVEY.md section 8(f), rank 4): the bilinear image -> per-face ts^3 cube resampling kernel of
// load_obj.py:88-137, operation for operation (including its NaN at texel (0,0,0), where the three barycentric
// coordinates are 0/0).
#include <cuda_runtime.h>
#include <stdint.h>

#include <cub/device/device_radix_sort.cuh>

#include "nr_b200.h"
#include "nr_internal.h"

namespace {

__global__ void __launch_bounds__(256) k_v2f_gather(const float* __restrict__ vertices, const int32_t* __restrict__ faces,
                                                    int Nv, long long n_corners_per_item, float* __restrict__ out) {
    const int b = blockIdx.y;
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;  // corner index within the item: f*3 + k
    if (i >= n_corners_per_item) return;
    const int idx = __ldg(faces + (size_t)b * n_corners_per_item + i);
    float x = 0.f, y = 0.f, z = 0.f;
    if ((unsigned)idx < (unsigned)Nv) {
        const float* v = vertices + ((size_t)b * Nv + idx) * 3;
        x = __ldg(v); y = __ldg(v + 1); z = __ldg(v + 2);
    }
    float* o = out + ((size_t)b * n_corners_per_item + i) * 3;
    o[0] = x; o[1] = y; o[2] = z;
}

__global__ void __launch_bounds__(256) k_v2f_scatter(const float* __restrict__ grad_faces, const int32_t* __restrict__ faces,
                                                     int Nv, long long n_corners_per_item, float* __restrict__ grad_vertices) {
    const int b = blockIdx.y;
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_corners_per_item) return;
    const int idx = __ldg(faces + (size_t)b * n_corners_per_item + i);
    if ((unsigned)idx >= (unsigned)Nv) return;
    const float* g = grad_faces + ((size_t)b * n_corners_per_item + i) * 3;
    const float gx = __ldg(g), gy = __ldg(g + 1), gz = __ldg(g + 2);
    if (gx == 0.f && gy == 0.f && gz == 0.f) return;  // back faces and unseen faces carry exact zeros
    float* v = grad_vertices + ((size_t)b * Nv + idx) * 3;
    atomicAdd(v, gx); atomicAdd(v + 1, gy); atomicAdd(v + 2, gz);
}


struct CamItem {
    float r[9], e[3], w;
};
__device__ __forceinline__ CamItem load_cam(const float* rot, const float* eye, const float* width, int item) {
    CamItem c;
#pragma unroll
    for (int k = 0; k < 9; k++) c.r[k] = rot ? __ldg(rot + (size_t)item * 9 + k) : ((k % 4 == 0) ? 1.0f : 0.0f);
#pragma unroll
    for (int k = 0; k < 3; k++) c.e[k] = eye ? __ldg(eye + (size_t)item * 3 + k) : 0.0f;
    c.w = width ? __ldg(width + item) : 1.0f;
    return c;
}

// out = perspective(rot * (v - eye)): one thread per vertex
__global__ void __launch_bounds__(256) k_camera_fwd(const float* __restrict__ vertices, const float* __restrict__ rot,
                                                    const float* __restrict__ eye, const float* __restrict__ width,
                                                    int Nv, uint32_t flags, float* __restrict__ out) {
    const int b = blockIdx.y;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= Nv) return;
    const CamItem c = load_cam(rot, eye, width, (flags & NR_CAM_SHARED) ? 0 : b);
    const float* v = vertices + ((size_t)b * Nv + i) * 3;
    const float d0 = __ldg(v) - c.e[0], d1 = __ldg(v + 1) - c.e[1], d2 = __ldg(v + 2) - c.e[2];
    float ox = fmaf(d2, c.r[2], fmaf(d1, c.r[1], d0 * c.r[0]));
    float oy = fmaf(d2, c.r[5], fmaf(d1, c.r[4], d0 * c.r[3]));
    const float oz = fmaf(d2, c.r[8], fmaf(d1, c.r[7], d0 * c.r[6]));
    if (flags & NR_CAM_PERSPECTIVE) {  // perspective.py:15-17: x / z / width
        ox = ox / oz / c.w;
        oy = oy / oz / c.w;
    }
    float* o = out + ((size_t)b * Nv + i) * 3;
    o[0] = ox; o[1] = oy; o[2] = oz;
}

// grad_vertices = rot^T * g_o with g_o the gradient in front of the perspective division; per-item reductions
// grad_rot[j][k] = sum_v g_o[j] * d[k], grad_eye = -sum_v grad_vertex, grad_width = -sum_v (gx*x + gy*y) / width
__global__ void __launch_bounds__(256) k_camera_bwd(const float* __restrict__ vertices, const float* __restrict__ rot,
                                                    const float* __restrict__ eye, const float* __restrict__ width,
                                                    const float* __restrict__ grad_out, int Nv, uint32_t flags,
                                                    float* __restrict__ grad_vertices, float* __restrict__ grad_rot,
                                                    float* __restrict__ grad_eye, float* __restrict__ grad_width) {
    const int b = blockIdx.y;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int item = (flags & NR_CAM_SHARED) ? 0 : b;
    const CamItem c = load_cam(rot, eye, width, item);
    float acc[13];
#pragma unroll
    for (int k = 0; k < 13; k++) acc[k] = 0.0f;
    if (i < Nv) {
        const float* v = vertices + ((size_t)b * Nv + i) * 3;
        const float* g = grad_out + ((size_t)b * Nv + i) * 3;
        const float d[3] = {__ldg(v) - c.e[0], __ldg(v + 1) - c.e[1], __ldg(v + 2) - c.e[2]};
        float go[3] = {__ldg(g), __ldg(g + 1), __ldg(g + 2)};
        if (flags & NR_CAM_PERSPECTIVE) {
            const float ox = fmaf(d[2], c.r[2], fmaf(d[1], c.r[1], d[0] * c.r[0]));
            const float oy = fmaf(d[2], c.r[5], fmaf(d[1], c.r[4], d[0] * c.r[3]));
            const float oz = fmaf(d[2], c.r[8], fmaf(d[1], c.r[7], d[0] * c.r[6]));
            const float x = ox / oz / c.w, y = oy / oz / c.w;
            const float s = go[0] * x + go[1] * y;
            acc[12] = -s / c.w;
            go[2] = go[2] - s / oz;
            go[0] = go[0] / oz / c.w;
            go[1] = go[1] / oz / c.w;
        }
        float gv[3];
#pragma unroll
        for (int k = 0; k < 3; k++) gv[k] = fmaf(go[2], c.r[6 + k], fmaf(go[1], c.r[3 + k], go[0] * c.r[k]));
        if (grad_vertices) {
            float* o = grad_vertices + ((size_t)b * Nv + i) * 3;
            o[0] = gv[0]; o[1] = gv[1]; o[2] = gv[2];
        }
#pragma unroll
        for (int j = 0; j < 3; j++)
#pragma unroll
            for (int k = 0; k < 3; k++) acc[3 * j + k] = go[j] * d[k];
#pragma unroll
        for (int k = 0; k < 3; k++) acc[9 + k] = -gv[k];
    }
    if (!(grad_rot || grad_eye || grad_width)) return;  // uniform
    // block reduction of the 13 camera terms, then one atomic per term and CTA
    __shared__ float red[8][13];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int k = 0; k < 13; k++) {
        float t = acc[k];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
        if (lane == 0) red[warp][k] = t;
    }
    __syncthreads();
    if (threadIdx.x < 13) {
        float t = 0.0f;
#pragma unroll
        for (int w = 0; w < 8; w++) t += red[w][threadIdx.x];
        const int k = threadIdx.x;
        if (k < 9) { if (grad_rot) atomicAdd(grad_rot + (size_t)item * 9 + k, t); }
        else if (k < 12) { if (grad_eye) atomicAdd(grad_eye + (size_t)item * 3 + (k - 9), t); }
        else if (grad_width && (flags & NR_CAM_PERSPECTIVE)) atomicAdd(grad_width + item, t);
    }
}


// light parameters of one item: {ambient rgb (intensity * colour), directional rgb (intensity * colour), direction}
struct LightItem {
    float amb[3], dir_rgb[3], dir[3];
};
__device__ __forceinline__ LightItem load_light(const float* params, int item) {
    LightItem L;
    const float* q = params + (size_t)item * 9;
#pragma unroll
    for (int k = 0; k < 3; k++) { L.amb[k] = __ldg(q + k); L.dir_rgb[k] = __ldg(q + 3 + k); L.dir[k] = __ldg(q + 6 + k); }
    return L;
}
struct FaceGeom {
    float a[3], b[3], c[3], len;  // a = v0 - v1, b = v2 - v1, c = a x b (lighting.py:40-43)
    int i0, i1, i2;
    bool ok;
};
__device__ __forceinline__ FaceGeom face_geom(const float* vertices, const int32_t* faces, int b, int Nv, int Nf, int f,
                                              uint32_t flags) {
    FaceGeom G;
    const int32_t* fi = faces + ((size_t)((flags & NR_INDICES_SHARED) ? 0 : b) * Nf + f) * 3;
    G.i0 = __ldg(fi); G.i1 = __ldg(fi + 1); G.i2 = __ldg(fi + 2);
    G.ok = (unsigned)G.i0 < (unsigned)Nv && (unsigned)G.i1 < (unsigned)Nv && (unsigned)G.i2 < (unsigned)Nv;
    float v[3][3] = {};
    if (G.ok) {
        const int idx[3] = {G.i0, G.i1, G.i2};
#pragma unroll
        for (int k = 0; k < 3; k++) {
            const float* p = vertices + ((size_t)b * Nv + idx[k]) * 3;
            v[k][0] = __ldg(p); v[k][1] = __ldg(p + 1); v[k][2] = __ldg(p + 2);
        }
    }
#pragma unroll
    for (int k = 0; k < 3; k++) { G.a[k] = v[0][k] - v[1][k]; G.b[k] = v[2][k] - v[1][k]; }
    G.c[0] = G.a[1] * G.b[2] - G.a[2] * G.b[1];
    G.c[1] = G.a[2] * G.b[0] - G.a[0] * G.b[2];
    G.c[2] = G.a[0] * G.b[1] - G.a[1] * G.b[0];
    G.len = sqrtf((G.c[0] * G.c[0] + G.c[1] * G.c[1]) + G.c[2] * G.c[2]);
    return G;
}

// light[b,f,:] = ambient + directional * relu(normal . direction), normal = c / (|c| + 1e-5)
__global__ void __launch_bounds__(256) k_face_light_fwd(const float* __restrict__ vertices, const int32_t* __restrict__ faces,
                                                        const float* __restrict__ params, int Nv, int Nf, uint32_t flags,
                                                        float* __restrict__ light) {
    const int b = blockIdx.y;
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= Nf) return;
    const LightItem L = load_light(params, (flags & NR_CAM_SHARED) ? 0 : b);
    const FaceGeom G = face_geom(vertices, faces, b, Nv, Nf, f, flags);
    const float inv = 1.0f / (G.len + 1e-5f);
    const float cosv = fmaxf((G.c[0] * inv * L.dir[0] + G.c[1] * inv * L.dir[1]) + G.c[2] * inv * L.dir[2], 0.0f);
    float* o = light + ((size_t)b * Nf + f) * 3;
#pragma unroll
    for (int k = 0; k < 3; k++) o[k] = L.amb[k] + L.dir_rgb[k] * cosv;
}

// d loss / d vertices from d loss / d light: through relu, the normalisation and the cross product
__global__ void __launch_bounds__(256) k_face_light_bwd(const float* __restrict__ vertices, const int32_t* __restrict__ faces,
                                                        const float* __restrict__ params, const float* __restrict__ grad_light,
                                                        int Nv, int Nf, uint32_t flags, float* __restrict__ grad_vertices) {
    const int b = blockIdx.y;
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= Nf) return;
    const LightItem L = load_light(params, (flags & NR_CAM_SHARED) ? 0 : b);
    const FaceGeom G = face_geom(vertices, faces, b, Nv, Nf, f, flags);
    if (!G.ok) return;
    const float inv = 1.0f / (G.len + 1e-5f);
    const float n[3] = {G.c[0] * inv, G.c[1] * inv, G.c[2] * inv};
    const float dot = (n[0] * L.dir[0] + n[1] * L.dir[1]) + n[2] * L.dir[2];
    if (!(dot > 0.0f)) return;  // relu
    const float* g = grad_light + ((size_t)b * Nf + f) * 3;
    const float gcos = (__ldg(g) * L.dir_rgb[0] + __ldg(g + 1) * L.dir_rgb[1]) + __ldg(g + 2) * L.dir_rgb[2];
    if (gcos == 0.0f) return;
    // n = c / (len + eps):  g_c = g_n / (len + eps) - c * (c . g_n) / (len * (len + eps)^2),  g_n = gcos * direction
    const float gn[3] = {gcos * L.dir[0], gcos * L.dir[1], gcos * L.dir[2]};
    const float cg = (G.c[0] * gn[0] + G.c[1] * gn[1]) + G.c[2] * gn[2];
    const float k2 = G.len > 0.0f ? cg * inv * inv / G.len : 0.0f;
    const float gc[3] = {gn[0] * inv - G.c[0] * k2, gn[1] * inv - G.c[1] * k2, gn[2] * inv - G.c[2] * k2};
    // c = a x b:  g_a = b x g_c,  g_b = g_c x a;  a = v0 - v1, b = v2 - v1
    const float ga[3] = {G.b[1] * gc[2] - G.b[2] * gc[1], G.b[2] * gc[0] - G.b[0] * gc[2], G.b[0] * gc[1] - G.b[1] * gc[0]};
    const float gb[3] = {gc[1] * G.a[2] - gc[2] * G.a[1], gc[2] * G.a[0] - gc[0] * G.a[2], gc[0] * G.a[1] - gc[1] * G.a[0]};
    float* g0 = grad_vertices + ((size_t)b * Nv + G.i0) * 3;
    float* g1 = grad_vertices + ((size_t)b * Nv + G.i1) * 3;
    float* g2 = grad_vertices + ((size_t)b * Nv + G.i2) * 3;
#pragma unroll
    for (int k = 0; k < 3; k++) {
        atomicAdd(g0 + k, ga[k]);
        atomicAdd(g2 + k, gb[k]);
        atomicAdd(g1 + k, -(ga[k] + gb[k]));
    }
}


// ------------------------------------------------------------------------------------------- smooth shading
// sort keys of the vertex-normal adjacency: corner i = f*3 + k of index-set item `item` -> key item * (Nv + 1) + vertex
// (Nv for an index outside [0, Nv): sorted past every vertex, never gathered), value = i
__global__ void __launch_bounds__(256) k_vn_keys(const int32_t* __restrict__ faces, int Nv, long long n_corners_per_item,
                                                 uint32_t* __restrict__ keys, int32_t* __restrict__ vals) {
    const int item = blockIdx.y;
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_corners_per_item) return;
    const size_t o = (size_t)item * n_corners_per_item + i;
    const int idx = __ldg(faces + o);
    keys[o] = (uint32_t)item * (uint32_t)(Nv + 1) + ((unsigned)idx < (unsigned)Nv ? (uint32_t)idx : (uint32_t)Nv);
    vals[o] = (int32_t)i;
}

__device__ __forceinline__ uint32_t lower_bound_u32(const uint32_t* a, uint32_t n, uint32_t key) {
    uint32_t lo = 0, hi = n;
    while (lo < hi) {
        const uint32_t mid = (lo + hi) >> 1;
        if (__ldg(a + mid) < key) lo = mid + 1; else hi = mid;
    }
    return lo;
}

// n_v = s_v / (|s_v| + 1e-5), s_v = sum of the face normals c_f (face_geom) of v's corners in the sorted (= ascending
// corner) order: one thread per vertex of every batch item
__global__ void __launch_bounds__(256) k_vn_gather(const float* __restrict__ vertices, const int32_t* __restrict__ faces,
                                                   const uint32_t* __restrict__ keys, const int32_t* __restrict__ vals,
                                                   uint32_t n_keys, int Nv, int Nf, uint32_t flags, float* __restrict__ normals) {
    const int b = blockIdx.y;
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= Nv) return;
    const uint32_t key = (uint32_t)((flags & NR_INDICES_SHARED) ? 0 : b) * (uint32_t)(Nv + 1) + (uint32_t)v;
    const uint32_t lo = lower_bound_u32(keys, n_keys, key), hi = lower_bound_u32(keys, n_keys, key + 1);
    float s0 = 0.0f, s1 = 0.0f, s2 = 0.0f;
    for (uint32_t j = lo; j < hi; j++) {
        const FaceGeom G = face_geom(vertices, faces, b, Nv, Nf, __ldg(vals + j) / 3, flags);
        s0 += G.c[0]; s1 += G.c[1]; s2 += G.c[2];
    }
    const float inv = 1.0f / (sqrtf((s0 * s0 + s1 * s1) + s2 * s2) + 1e-5f);
    float* o = normals + ((size_t)b * Nv + v) * 3;
    o[0] = s0 * inv; o[1] = s1 * inv; o[2] = s2 * inv;
}

// backward, step 1: s_v again, with atomics (the backward is not bit-pinned)
__global__ void __launch_bounds__(256) k_vn_sums(const float* __restrict__ vertices, const int32_t* __restrict__ faces, int Nv,
                                                 int Nf, uint32_t flags, float* __restrict__ sums) {
    const int b = blockIdx.y;
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= Nf) return;
    const FaceGeom G = face_geom(vertices, faces, b, Nv, Nf, f, flags);
    if (!G.ok) return;
    const int idx[3] = {G.i0, G.i1, G.i2};
#pragma unroll
    for (int k = 0; k < 3; k++) {
        float* q = sums + ((size_t)b * Nv + idx[k]) * 3;
        atomicAdd(q, G.c[0]); atomicAdd(q + 1, G.c[1]); atomicAdd(q + 2, G.c[2]);
    }
}

// step 2, per face: g_c = sum over its corners of d n / d s (at s_v) applied to d loss / d n_v, then through c = a x b
// as in k_face_light_bwd
__global__ void __launch_bounds__(256) k_vn_bwd(const float* __restrict__ vertices, const int32_t* __restrict__ faces,
                                                const float* __restrict__ sums, const float* __restrict__ grad_normals, int Nv,
                                                int Nf, uint32_t flags, float* __restrict__ grad_vertices) {
    const int b = blockIdx.y;
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= Nf) return;
    const FaceGeom G = face_geom(vertices, faces, b, Nv, Nf, f, flags);
    if (!G.ok) return;
    const int idx[3] = {G.i0, G.i1, G.i2};
    float gc[3] = {0.0f, 0.0f, 0.0f};
#pragma unroll
    for (int k = 0; k < 3; k++) {
        const float* q = sums + ((size_t)b * Nv + idx[k]) * 3;
        const float* g = grad_normals + ((size_t)b * Nv + idx[k]) * 3;
        const float sv[3] = {q[0], q[1], q[2]}, gn[3] = {__ldg(g), __ldg(g + 1), __ldg(g + 2)};
        // n = s / (len + eps):  g_s = g_n / (len + eps) - s (s . g_n) / (len (len + eps)^2)
        const float len = sqrtf((sv[0] * sv[0] + sv[1] * sv[1]) + sv[2] * sv[2]);
        const float inv = 1.0f / (len + 1e-5f);
        const float sg = (sv[0] * gn[0] + sv[1] * gn[1]) + sv[2] * gn[2];
        const float k2 = len > 0.0f ? sg * inv * inv / len : 0.0f;
#pragma unroll
        for (int j = 0; j < 3; j++) gc[j] += gn[j] * inv - sv[j] * k2;
    }
    const float ga[3] = {G.b[1] * gc[2] - G.b[2] * gc[1], G.b[2] * gc[0] - G.b[0] * gc[2], G.b[0] * gc[1] - G.b[1] * gc[0]};
    const float gb[3] = {gc[1] * G.a[2] - gc[2] * G.a[1], gc[2] * G.a[0] - gc[0] * G.a[2], gc[0] * G.a[1] - gc[1] * G.a[0]};
    float* g0 = grad_vertices + ((size_t)b * Nv + G.i0) * 3;
    float* g1 = grad_vertices + ((size_t)b * Nv + G.i1) * 3;
    float* g2 = grad_vertices + ((size_t)b * Nv + G.i2) * 3;
#pragma unroll
    for (int k = 0; k < 3; k++) {
        atomicAdd(g0 + k, ga[k]);
        atomicAdd(g2 + k, gb[k]);
        atomicAdd(g1 + k, -(ga[k] + gb[k]));
    }
}

// corner_light[b,f,k,:] = ambient + directional * max(sgn * (n . direction), 0), n = the corner's vertex normal
__global__ void __launch_bounds__(256) k_corner_light_fwd(const float* __restrict__ normals, const int32_t* __restrict__ faces,
                                                          const float* __restrict__ params, int Nv, int Nf, uint32_t flags,
                                                          float* __restrict__ light) {
    const int b = blockIdx.y;
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= Nf) return;
    const LightItem L = load_light(params, (flags & NR_CAM_SHARED) ? 0 : b);
    const int32_t* fi = faces + ((size_t)((flags & NR_INDICES_SHARED) ? 0 : b) * Nf + f) * 3;
    const bool rev = (flags & NR_TEX_FILL_BACK) && f >= (Nf >> 1);  // reversed copy: its face normal is -n
    float* o = light + ((size_t)b * Nf + f) * 9;
#pragma unroll
    for (int k = 0; k < 3; k++) {
        const int idx = __ldg(fi + k);
        float n[3] = {0.0f, 0.0f, 0.0f};
        if ((unsigned)idx < (unsigned)Nv) {
            const float* q = normals + ((size_t)b * Nv + idx) * 3;
            n[0] = __ldg(q); n[1] = __ldg(q + 1); n[2] = __ldg(q + 2);
        }
        const float dot = (n[0] * L.dir[0] + n[1] * L.dir[1]) + n[2] * L.dir[2];
        const float cosv = fmaxf(rev ? -dot : dot, 0.0f);
#pragma unroll
        for (int c = 0; c < 3; c++) o[3 * k + c] = L.amb[c] + L.dir_rgb[c] * cosv;
    }
}

__global__ void __launch_bounds__(256) k_corner_light_bwd(const float* __restrict__ normals, const int32_t* __restrict__ faces,
                                                          const float* __restrict__ params, const float* __restrict__ grad_light,
                                                          int Nv, int Nf, uint32_t flags, float* __restrict__ grad_normals) {
    const int b = blockIdx.y;
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= Nf) return;
    const LightItem L = load_light(params, (flags & NR_CAM_SHARED) ? 0 : b);
    const int32_t* fi = faces + ((size_t)((flags & NR_INDICES_SHARED) ? 0 : b) * Nf + f) * 3;
    const float sgn = ((flags & NR_TEX_FILL_BACK) && f >= (Nf >> 1)) ? -1.0f : 1.0f;
    const float* g = grad_light + ((size_t)b * Nf + f) * 9;
#pragma unroll
    for (int k = 0; k < 3; k++) {
        const int idx = __ldg(fi + k);
        if ((unsigned)idx >= (unsigned)Nv) continue;
        const float* q = normals + ((size_t)b * Nv + idx) * 3;
        const float dot = (__ldg(q) * L.dir[0] + __ldg(q + 1) * L.dir[1]) + __ldg(q + 2) * L.dir[2];
        if (!(sgn * dot > 0.0f)) continue;  // relu
        const float gcos = (__ldg(g + 3 * k) * L.dir_rgb[0] + __ldg(g + 3 * k + 1) * L.dir_rgb[1]) + __ldg(g + 3 * k + 2) * L.dir_rgb[2];
        if (gcos == 0.0f) continue;
        float* o = grad_normals + ((size_t)b * Nv + idx) * 3;
        atomicAdd(o, sgn * gcos * L.dir[0]); atomicAdd(o + 1, sgn * gcos * L.dir[1]); atomicAdd(o + 2, sgn * gcos * L.dir[2]);
    }
}

// corner_shading[b,f,k,:] = (sgn n, v) of the corner's vertex (zeros for an index outside [0, Nv)); sgn = -1 for the
// reversed copies f >= Nf/2 with NR_TEX_FILL_BACK
__global__ void __launch_bounds__(256) k_corner_shading_fwd(const float* __restrict__ normals, const float* __restrict__ vertices,
                                                            const int32_t* __restrict__ faces, int Nv, int Nf, uint32_t flags,
                                                            float* __restrict__ out) {
    const int b = blockIdx.y;
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= Nf) return;
    const int32_t* fi = faces + ((size_t)((flags & NR_INDICES_SHARED) ? 0 : b) * Nf + f) * 3;
    const float sgn = ((flags & NR_TEX_FILL_BACK) && f >= (Nf >> 1)) ? -1.0f : 1.0f;
    float* o = out + ((size_t)b * Nf + f) * 18;
#pragma unroll
    for (int k = 0; k < 3; k++) {
        const int idx = __ldg(fi + k);
        float n[3] = {0.0f, 0.0f, 0.0f}, v[3] = {0.0f, 0.0f, 0.0f};
        if ((unsigned)idx < (unsigned)Nv) {
            const float* qn = normals + ((size_t)b * Nv + idx) * 3;
            const float* qv = vertices + ((size_t)b * Nv + idx) * 3;
#pragma unroll
            for (int c = 0; c < 3; c++) { n[c] = sgn * __ldg(qn + c); v[c] = __ldg(qv + c); }
        }
#pragma unroll
        for (int c = 0; c < 3; c++) { o[6 * k + c] = n[c]; o[6 * k + 3 + c] = v[c]; }
    }
}

__global__ void __launch_bounds__(256) k_corner_shading_bwd(const int32_t* __restrict__ faces, const float* __restrict__ grad,
                                                            int Nv, int Nf, uint32_t flags, float* __restrict__ grad_normals,
                                                            float* __restrict__ grad_vertices) {
    const int b = blockIdx.y;
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= Nf) return;
    const int32_t* fi = faces + ((size_t)((flags & NR_INDICES_SHARED) ? 0 : b) * Nf + f) * 3;
    const float sgn = ((flags & NR_TEX_FILL_BACK) && f >= (Nf >> 1)) ? -1.0f : 1.0f;
    const float* g = grad + ((size_t)b * Nf + f) * 18;
#pragma unroll
    for (int k = 0; k < 3; k++) {
        const int idx = __ldg(fi + k);
        if ((unsigned)idx >= (unsigned)Nv) continue;
        if (grad_normals) {
            float* o = grad_normals + ((size_t)b * Nv + idx) * 3;
#pragma unroll
            for (int c = 0; c < 3; c++) atomicAdd(o + c, sgn * __ldg(g + 6 * k + c));
        }
        if (grad_vertices) {
            float* o = grad_vertices + ((size_t)b * Nv + idx) * 3;
#pragma unroll
            for (int c = 0; c < 3; c++) atomicAdd(o + c, __ldg(g + 6 * k + 3 + c));
        }
    }
}

struct VnLayout {
    size_t n;  // corners of the index set (items x 3 Nf)
    int end_bit;
    size_t off_keys_out, off_vals_in, off_vals_out, off_temp, temp_bytes, total;
};
inline size_t align256(size_t x) { return (x + 255) / 256 * 256; }
// workspace = sort keys in | keys out | values in | values out | cub scratch; the backward uses the first B Nv 3 floats
bool vn_layout(int B, int Nv, int Nf, uint32_t flags, VnLayout* L) {
    if (B <= 0 || Nv <= 0 || Nf <= 0 || B > 65535) return false;
    const long long items = (flags & NR_INDICES_SHARED) ? 1 : B;
    if (items * ((long long)Nv + 1) > 0x7FFFFFFFll || 3ll * Nf > 0x7FFFFFFFll || items * 3ll * Nf > 0x7FFFFFFFll) return false;
    L->n = (size_t)(items * 3ll * Nf);
    const uint32_t max_key = (uint32_t)(items * ((long long)Nv + 1) - 1);
    L->end_bit = 1;
    while (L->end_bit < 32 && (max_key >> L->end_bit) != 0) L->end_bit++;
    L->temp_bytes = 0;
    if (cub::DeviceRadixSort::SortPairs(nullptr, L->temp_bytes, (const uint32_t*)nullptr, (uint32_t*)nullptr,
                                        (const int32_t*)nullptr, (int32_t*)nullptr, (int)L->n, 0, L->end_bit) != cudaSuccess)
        return false;
    const size_t a = align256(L->n * 4);
    L->off_keys_out = a; L->off_vals_in = 2 * a; L->off_vals_out = 3 * a; L->off_temp = 4 * a;
    L->total = L->off_temp + align256(L->temp_bytes);
    const size_t bwd = align256((size_t)B * Nv * 3 * sizeof(float));
    if (bwd > L->total) L->total = bwd;
    return true;
}

// load_obj.py:97-131.  One thread per texel of every face.  Arithmetic as the reference build evaluates it (read from
// its SASS): dims = (float)((double)k / (ts - 1.)), normalised by IEEE division with sum = (d0 + d1) + d2;
// pos = fma(f2, d2, fma(f0, d0, f1 * d1)) * (size - 1); taps blended as fma chains in source order.
__global__ void __launch_bounds__(256) k_bake_textures(const float* __restrict__ image, const float* __restrict__ uv_faces,
                                                       const int32_t* __restrict__ is_update, long long n, int ts, int H,
                                                       int W, float* __restrict__ textures) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int t3 = ts * ts * ts;
    const long long fn = i / t3;
    if (is_update && __ldg(is_update + fn) == 0) return;
    const int r = (int)(i - fn * t3);
    const double den = (double)ts - 1.0;
    float d0 = (float)((double)((r / (ts * ts)) % ts) / den);
    float d1 = (float)((double)((r / ts) % ts) / den);
    float d2 = (float)((double)(r % ts) / den);
    const float sum = __fadd_rn(__fadd_rn(d0, d1), d2);
    d0 = __fdiv_rn(d0, sum); d1 = __fdiv_rn(d1, sum); d2 = __fdiv_rn(d2, sum);  // texel (0,0,0): 0/0 = NaN, as in the reference
    const float* f = uv_faces + fn * 6;
    const float f0x = __ldg(f), f0y = __ldg(f + 1), f1x = __ldg(f + 2), f1y = __ldg(f + 3), f2x = __ldg(f + 4), f2y = __ldg(f + 5);
    const float pos_x = __fmul_rn(__fmaf_rn(f2x, d2, __fmaf_rn(f0x, d0, __fmul_rn(f1x, d1))), (float)(W - 1));
    const float pos_y = __fmul_rn(__fmaf_rn(f2y, d2, __fmaf_rn(f0y, d0, __fmul_rn(f1y, d1))), (float)(H - 1));
    const int ix = __float2int_rz(pos_x), iy = __float2int_rz(pos_y), iy1 = __float2int_rz(__fadd_rn(pos_y, 1.0f));
    const float wx1 = __fsub_rn(pos_x, (float)ix), wy1 = __fsub_rn(pos_y, (float)iy);
    const float wx0 = __fsub_rn(1.0f, wx1), wy0 = __fsub_rn(1.0f, wy1);
    const float w00 = __fmul_rn(wx0, wy0), w01 = __fmul_rn(wx0, wy1), w10 = __fmul_rn(wx1, wy0), w11 = __fmul_rn(wx1, wy1);
    // the reference reads one row / column past the image when a coordinate is exactly 1 (weight 0 -- or, when the
    // float sum pos_y + 1 rounds up, weight ~1: undefined behaviour there); those taps are addressed in bounds here
    const int cx0 = min(max(ix, 0), W - 1), cx1 = min(max(ix + 1, 0), W - 1);
    const int cy0 = min(max(iy, 0), H - 1), cy1 = min(max(iy1, 0), H - 1);
    const float* p00 = image + ((size_t)cy0 * W + cx0) * 3;
    const float* p01 = image + ((size_t)cy1 * W + cx0) * 3;  // next row, same column
    const float* p10 = image + ((size_t)cy0 * W + cx1) * 3;  // same row, next column
    const float* p11 = image + ((size_t)cy1 * W + cx1) * 3;
    float* out = textures + i * 3;
#pragma unroll
    for (int k = 0; k < 3; k++) {
        float c = __fmul_rn(w00, __ldg(p00 + k));
        c = __fmaf_rn(w01, __ldg(p01 + k), c);
        c = __fmaf_rn(w10, __ldg(p10 + k), c);
        c = __fmaf_rn(w11, __ldg(p11 + k), c);
        out[k] = c;
    }
}

}  // namespace

extern "C" int nr_b200_vertices_to_faces(const float* vertices, const int32_t* faces, int32_t B, int32_t Nv, int32_t Nf,
                                         float* out_faces, void* cuda_stream) {
    nr_internal::launch_count() = 0;
    if (!vertices || !faces || !out_faces || B <= 0 || Nv <= 0 || Nf <= 0 || B > 65535) return NR_ERR_INVALID_ARG;
    cudaStream_t stream = (cudaStream_t)cuda_stream;
    const long long n = (long long)Nf * 3;
    {
        nr_internal::LaunchScope ls("k_v2f_gather", stream);
        k_v2f_gather<<<dim3((unsigned)((n + 255) / 256), B), 256, 0, stream>>>(vertices, faces, Nv, n, out_faces);
    }
    return cudaGetLastError() == cudaSuccess ? NR_OK : NR_ERR_CUDA;
}

extern "C" int nr_b200_vertices_to_faces_backward(const float* grad_faces, const int32_t* faces, int32_t B, int32_t Nv,
                                                  int32_t Nf, float* grad_vertices, uint32_t flags, void* cuda_stream) {
    nr_internal::launch_count() = 0;
    if (!grad_faces || !faces || !grad_vertices || B <= 0 || Nv <= 0 || Nf <= 0 || B > 65535) return NR_ERR_INVALID_ARG;
    cudaStream_t stream = (cudaStream_t)cuda_stream;
    if (!(flags & NR_GRAD_ACCUMULATE) &&
        cudaMemsetAsync(grad_vertices, 0, (size_t)B * Nv * 3 * sizeof(float), stream) != cudaSuccess)
        return NR_ERR_CUDA;
    const long long n = (long long)Nf * 3;
    {
        nr_internal::LaunchScope ls("k_v2f_scatter", stream);
        k_v2f_scatter<<<dim3((unsigned)((n + 255) / 256), B), 256, 0, stream>>>(grad_faces, faces, Nv, n, grad_vertices);
    }
    return cudaGetLastError() == cudaSuccess ? NR_OK : NR_ERR_CUDA;
}

extern "C" int nr_b200_camera_transform(const float* vertices, const float* rot, const float* eye, const float* width,
                                        int32_t B, int32_t Nv, uint32_t flags, float* out, void* cuda_stream) {
    nr_internal::launch_count() = 0;
    if (!vertices || !out || B <= 0 || Nv <= 0 || B > 65535) return NR_ERR_INVALID_ARG;
    if ((flags & NR_CAM_PERSPECTIVE) && !width) return NR_ERR_INVALID_ARG;
    cudaStream_t stream = (cudaStream_t)cuda_stream;
    {
        nr_internal::LaunchScope ls("k_camera_fwd", stream);
        k_camera_fwd<<<dim3((unsigned)((Nv + 255) / 256), B), 256, 0, stream>>>(vertices, rot, eye, width, Nv, flags, out);
    }
    return cudaGetLastError() == cudaSuccess ? NR_OK : NR_ERR_CUDA;
}

extern "C" int nr_b200_camera_transform_backward(const float* vertices, const float* rot, const float* eye,
                                                 const float* width, const float* grad_out, int32_t B, int32_t Nv,
                                                 uint32_t flags, float* grad_vertices, float* grad_rot, float* grad_eye,
                                                 float* grad_width, void* cuda_stream) {
    nr_internal::launch_count() = 0;
    if (!vertices || !grad_out || B <= 0 || Nv <= 0 || B > 65535) return NR_ERR_INVALID_ARG;
    if ((flags & NR_CAM_PERSPECTIVE) && !width) return NR_ERR_INVALID_ARG;
    cudaStream_t stream = (cudaStream_t)cuda_stream;
    const size_t items = (flags & NR_CAM_SHARED) ? 1 : (size_t)B;
    if (!(flags & NR_GRAD_ACCUMULATE)) {  // the camera terms are accumulated with atomics
        if (grad_rot && cudaMemsetAsync(grad_rot, 0, items * 9 * sizeof(float), stream) != cudaSuccess) return NR_ERR_CUDA;
        if (grad_eye && cudaMemsetAsync(grad_eye, 0, items * 3 * sizeof(float), stream) != cudaSuccess) return NR_ERR_CUDA;
        if (grad_width && cudaMemsetAsync(grad_width, 0, items * sizeof(float), stream) != cudaSuccess) return NR_ERR_CUDA;
    }
    {
        nr_internal::LaunchScope ls("k_camera_bwd", stream);
        k_camera_bwd<<<dim3((unsigned)((Nv + 255) / 256), B), 256, 0, stream>>>(vertices, rot, eye, width, grad_out, Nv, flags,
                                                                               grad_vertices, grad_rot, grad_eye, grad_width);
    }
    return cudaGetLastError() == cudaSuccess ? NR_OK : NR_ERR_CUDA;
}

extern "C" int nr_b200_face_lighting(const float* vertices, const int32_t* faces, const float* light_params, int32_t B,
                                     int32_t Nv, int32_t Nf, uint32_t flags, float* face_light, void* cuda_stream) {
    nr_internal::launch_count() = 0;
    if (!vertices || !faces || !light_params || !face_light || B <= 0 || Nv <= 0 || Nf <= 0 || B > 65535) return NR_ERR_INVALID_ARG;
    cudaStream_t stream = (cudaStream_t)cuda_stream;
    {
        nr_internal::LaunchScope ls("k_face_light_fwd", stream);
        k_face_light_fwd<<<dim3((unsigned)((Nf + 255) / 256), B), 256, 0, stream>>>(vertices, faces, light_params, Nv, Nf, flags,
                                                                                   face_light);
    }
    return cudaGetLastError() == cudaSuccess ? NR_OK : NR_ERR_CUDA;
}

extern "C" int nr_b200_face_lighting_backward(const float* vertices, const int32_t* faces, const float* light_params,
                                              const float* grad_face_light, int32_t B, int32_t Nv, int32_t Nf,
                                              uint32_t flags, float* grad_vertices, void* cuda_stream) {
    nr_internal::launch_count() = 0;
    if (!vertices || !faces || !light_params || !grad_face_light || !grad_vertices || B <= 0 || Nv <= 0 || Nf <= 0 || B > 65535)
        return NR_ERR_INVALID_ARG;
    cudaStream_t stream = (cudaStream_t)cuda_stream;
    if (!(flags & NR_GRAD_ACCUMULATE) &&
        cudaMemsetAsync(grad_vertices, 0, (size_t)B * Nv * 3 * sizeof(float), stream) != cudaSuccess)
        return NR_ERR_CUDA;
    {
        nr_internal::LaunchScope ls("k_face_light_bwd", stream);
        k_face_light_bwd<<<dim3((unsigned)((Nf + 255) / 256), B), 256, 0, stream>>>(vertices, faces, light_params, grad_face_light,
                                                                                   Nv, Nf, flags, grad_vertices);
    }
    return cudaGetLastError() == cudaSuccess ? NR_OK : NR_ERR_CUDA;
}

extern "C" size_t nr_b200_vertex_normals_workspace_bytes(int32_t B, int32_t Nv, int32_t Nf, uint32_t flags) {
    VnLayout L;
    return vn_layout(B, Nv, Nf, flags, &L) ? L.total : 0;
}

extern "C" int nr_b200_vertex_normals(const float* vertices, const int32_t* faces, int32_t B, int32_t Nv, int32_t Nf,
                                      uint32_t flags, float* normals, void* workspace, size_t workspace_bytes,
                                      void* cuda_stream) {
    nr_internal::launch_count() = 0;
    if (!vertices || !faces || !normals || B <= 0 || Nv <= 0 || Nf <= 0 || B > 65535) return NR_ERR_INVALID_ARG;
    VnLayout L;
    if (!vn_layout(B, Nv, Nf, flags, &L)) return NR_ERR_UNSUPPORTED;
    if (!workspace || workspace_bytes < L.total || ((uintptr_t)workspace & 15)) return NR_ERR_WORKSPACE;
    cudaStream_t stream = (cudaStream_t)cuda_stream;
    char* w = (char*)workspace;
    uint32_t* keys_in = (uint32_t*)w;
    uint32_t* keys_out = (uint32_t*)(w + L.off_keys_out);
    int32_t* vals_in = (int32_t*)(w + L.off_vals_in);
    int32_t* vals_out = (int32_t*)(w + L.off_vals_out);
    const int items = (flags & NR_INDICES_SHARED) ? 1 : B;
    const long long n = 3ll * Nf;
    {
        nr_internal::LaunchScope ls("k_vn_keys", stream);
        k_vn_keys<<<dim3((unsigned)((n + 255) / 256), items), 256, 0, stream>>>(faces, Nv, n, keys_in, vals_in);
    }
    {
        nr_internal::LaunchScope ls("vn_sort", stream);  // stable: equal vertices keep ascending corner order
        size_t temp = L.temp_bytes;
        if (cub::DeviceRadixSort::SortPairs(w + L.off_temp, temp, keys_in, keys_out, vals_in, vals_out, (int)L.n, 0, L.end_bit,
                                            stream) != cudaSuccess)
            return NR_ERR_CUDA;
    }
    {
        nr_internal::LaunchScope ls("k_vn_gather", stream);
        k_vn_gather<<<dim3((unsigned)((Nv + 255) / 256), B), 256, 0, stream>>>(vertices, faces, keys_out, vals_out, (uint32_t)L.n,
                                                                             Nv, Nf, flags, normals);
    }
    return cudaGetLastError() == cudaSuccess ? NR_OK : NR_ERR_CUDA;
}

extern "C" int nr_b200_vertex_normals_backward(const float* vertices, const int32_t* faces, const float* grad_normals, int32_t B,
                                               int32_t Nv, int32_t Nf, uint32_t flags, float* grad_vertices, void* workspace,
                                               size_t workspace_bytes, void* cuda_stream) {
    nr_internal::launch_count() = 0;
    if (!vertices || !faces || !grad_normals || !grad_vertices || B <= 0 || Nv <= 0 || Nf <= 0 || B > 65535)
        return NR_ERR_INVALID_ARG;
    VnLayout L;
    if (!vn_layout(B, Nv, Nf, flags, &L)) return NR_ERR_UNSUPPORTED;
    if (!workspace || workspace_bytes < L.total || ((uintptr_t)workspace & 15)) return NR_ERR_WORKSPACE;
    cudaStream_t stream = (cudaStream_t)cuda_stream;
    float* sums = (float*)workspace;
    if (cudaMemsetAsync(sums, 0, (size_t)B * Nv * 3 * sizeof(float), stream) != cudaSuccess) return NR_ERR_CUDA;
    if (!(flags & NR_GRAD_ACCUMULATE) &&
        cudaMemsetAsync(grad_vertices, 0, (size_t)B * Nv * 3 * sizeof(float), stream) != cudaSuccess)
        return NR_ERR_CUDA;
    const dim3 grid((unsigned)((Nf + 255) / 256), B);
    {
        nr_internal::LaunchScope ls("k_vn_sums", stream);
        k_vn_sums<<<grid, 256, 0, stream>>>(vertices, faces, Nv, Nf, flags, sums);
    }
    {
        nr_internal::LaunchScope ls("k_vn_bwd", stream);
        k_vn_bwd<<<grid, 256, 0, stream>>>(vertices, faces, sums, grad_normals, Nv, Nf, flags, grad_vertices);
    }
    return cudaGetLastError() == cudaSuccess ? NR_OK : NR_ERR_CUDA;
}

extern "C" int nr_b200_corner_lighting(const float* normals, const int32_t* faces, const float* light_params, int32_t B,
                                       int32_t Nv, int32_t Nf, uint32_t flags, float* corner_light, void* cuda_stream) {
    nr_internal::launch_count() = 0;
    if (!normals || !faces || !light_params || !corner_light || B <= 0 || Nv <= 0 || Nf <= 0 || B > 65535) return NR_ERR_INVALID_ARG;
    if ((flags & NR_TEX_FILL_BACK) && (Nf & 1)) return NR_ERR_INVALID_ARG;
    cudaStream_t stream = (cudaStream_t)cuda_stream;
    {
        nr_internal::LaunchScope ls("k_corner_light_fwd", stream);
        k_corner_light_fwd<<<dim3((unsigned)((Nf + 255) / 256), B), 256, 0, stream>>>(normals, faces, light_params, Nv, Nf, flags,
                                                                                     corner_light);
    }
    return cudaGetLastError() == cudaSuccess ? NR_OK : NR_ERR_CUDA;
}

extern "C" int nr_b200_corner_lighting_backward(const float* normals, const int32_t* faces, const float* light_params,
                                                const float* grad_corner_light, int32_t B, int32_t Nv, int32_t Nf,
                                                uint32_t flags, float* grad_normals, void* cuda_stream) {
    nr_internal::launch_count() = 0;
    if (!normals || !faces || !light_params || !grad_corner_light || !grad_normals || B <= 0 || Nv <= 0 || Nf <= 0 || B > 65535)
        return NR_ERR_INVALID_ARG;
    if ((flags & NR_TEX_FILL_BACK) && (Nf & 1)) return NR_ERR_INVALID_ARG;
    cudaStream_t stream = (cudaStream_t)cuda_stream;
    if (!(flags & NR_GRAD_ACCUMULATE) &&
        cudaMemsetAsync(grad_normals, 0, (size_t)B * Nv * 3 * sizeof(float), stream) != cudaSuccess)
        return NR_ERR_CUDA;
    {
        nr_internal::LaunchScope ls("k_corner_light_bwd", stream);
        k_corner_light_bwd<<<dim3((unsigned)((Nf + 255) / 256), B), 256, 0, stream>>>(normals, faces, light_params,
                                                                                     grad_corner_light, Nv, Nf, flags,
                                                                                     grad_normals);
    }
    return cudaGetLastError() == cudaSuccess ? NR_OK : NR_ERR_CUDA;
}

extern "C" int nr_b200_corner_shading(const float* normals, const float* vertices, const int32_t* faces, int32_t B, int32_t Nv,
                                      int32_t Nf, uint32_t flags, float* corner_shading, void* cuda_stream) {
    nr_internal::launch_count() = 0;
    if (!normals || !vertices || !faces || !corner_shading || B <= 0 || Nv <= 0 || Nf <= 0 || B > 65535) return NR_ERR_INVALID_ARG;
    if ((flags & NR_TEX_FILL_BACK) && (Nf & 1)) return NR_ERR_INVALID_ARG;
    cudaStream_t stream = (cudaStream_t)cuda_stream;
    {
        nr_internal::LaunchScope ls("k_corner_shading_fwd", stream);
        k_corner_shading_fwd<<<dim3((unsigned)((Nf + 255) / 256), B), 256, 0, stream>>>(normals, vertices, faces, Nv, Nf, flags,
                                                                                       corner_shading);
    }
    return cudaGetLastError() == cudaSuccess ? NR_OK : NR_ERR_CUDA;
}

extern "C" int nr_b200_corner_shading_backward(const int32_t* faces, const float* grad_corner_shading, int32_t B, int32_t Nv,
                                               int32_t Nf, uint32_t flags, float* grad_normals, float* grad_vertices,
                                               void* cuda_stream) {
    nr_internal::launch_count() = 0;
    if (!faces || !grad_corner_shading || (!grad_normals && !grad_vertices) || B <= 0 || Nv <= 0 || Nf <= 0 || B > 65535)
        return NR_ERR_INVALID_ARG;
    if ((flags & NR_TEX_FILL_BACK) && (Nf & 1)) return NR_ERR_INVALID_ARG;
    cudaStream_t stream = (cudaStream_t)cuda_stream;
    if (!(flags & NR_GRAD_ACCUMULATE)) {
        const size_t bytes = (size_t)B * Nv * 3 * sizeof(float);
        if (grad_normals && cudaMemsetAsync(grad_normals, 0, bytes, stream) != cudaSuccess) return NR_ERR_CUDA;
        if (grad_vertices && cudaMemsetAsync(grad_vertices, 0, bytes, stream) != cudaSuccess) return NR_ERR_CUDA;
    }
    {
        nr_internal::LaunchScope ls("k_corner_shading_bwd", stream);
        k_corner_shading_bwd<<<dim3((unsigned)((Nf + 255) / 256), B), 256, 0, stream>>>(faces, grad_corner_shading, Nv, Nf, flags,
                                                                                       grad_normals, grad_vertices);
    }
    return cudaGetLastError() == cudaSuccess ? NR_OK : NR_ERR_CUDA;
}

extern "C" int nr_b200_bake_textures(const float* image, const float* uv_faces, const int32_t* is_update, int32_t F,
                                     int32_t ts, int32_t H, int32_t W, float* textures, void* cuda_stream) {
    nr_internal::launch_count() = 0;
    if (!image || !uv_faces || !textures || F <= 0 || ts < 2 || H <= 0 || W <= 0) return NR_ERR_INVALID_ARG;
    cudaStream_t stream = (cudaStream_t)cuda_stream;
    const long long n = (long long)F * ts * ts * ts;
    {
        nr_internal::LaunchScope ls("k_bake_textures", stream);
        k_bake_textures<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(image, uv_faces, is_update, n, ts, H, W, textures);
    }
    return cudaGetLastError() == cudaSuccess ? NR_OK : NR_ERR_CUDA;
}
