"""numpy/ctypes front end of the CPU oracle (oracle/nr_oracle.c).

TEST INFRASTRUCTURE ONLY -- the product package (neural_renderer_b200) never
imports this module.  It restates, on the CPU, the reference's rasterizer hot
path and the thin array glue around it so that the reference's own golden
vectors can be replayed without Chainer/CuPy:

  OracleRasterize          <- Rasterize.forward_gpu / backward_gpu   rasterize.py:467-513, :849-889
  rasterize_rgbad & co.    <- rasterize.py:900-1060 (transpose, vertical flip, 2x2 average pooling)
  look_at / perspective / lighting / vertices_to_faces / Renderer-style helpers
                           <- look_at.py:7-46, perspective.py:5-19, lighting.py:8-52,
                              vertices_to_faces.py:4-21, renderer.py:35-107

All raw maps use the reference's internal conventions: NHWC, un-flipped
(row 0 = bottom of the image), face_index_map = -1 where empty.
"""
from __future__ import annotations

import ctypes
import math
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None

c_f = ctypes.POINTER(ctypes.c_float)
c_i = ctypes.POINTER(ctypes.c_int)


def build(force=False):
    """Compile oracle/nr_oracle.c into oracle/libnr_oracle.so (make)."""
    so = os.path.join(HERE, "libnr_oracle.so")
    src = os.path.join(HERE, "nr_oracle.c")
    if force or not os.path.exists(so) or os.path.getmtime(so) < os.path.getmtime(src):
        subprocess.run(["make", "-s", "-C", HERE] + (["-B"] if force else []), check=True)
    return so


def lib():
    global _LIB
    if _LIB is None:
        so = os.path.join(HERE, "libnr_oracle.so")
        if not os.path.exists(so) or (os.path.exists(os.path.join(HERE, "nr_oracle.c"))
                                      and os.path.getmtime(so) < os.path.getmtime(os.path.join(HERE, "nr_oracle.c"))):
            build()
        _LIB = ctypes.CDLL(so)
        _LIB.nro_num_threads.restype = ctypes.c_int
    return _LIB


def _fp(a):
    return None if a is None else a.ctypes.data_as(c_f)


def _ip(a):
    return None if a is None else a.ctypes.data_as(c_i)


def _f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def num_threads():
    return int(lib().nro_num_threads())


def set_num_threads(n):
    lib().nro_set_num_threads(int(n))


def bake_textures(image, uv_faces, is_update, texture_size, textures=None):
    """load_obj.py:88-137 on the CPU: bilinear image -> per-face cube resampling (image [H,W,3] already flipped)."""
    image = _f32(image)
    uv_faces = _f32(uv_faces)
    nf = uv_faces.shape[0]
    if textures is None:
        textures = np.full((nf, texture_size, texture_size, texture_size, 3), 0.5, dtype=np.float32)
    textures = np.ascontiguousarray(textures, dtype=np.float32)
    upd = None if is_update is None else np.ascontiguousarray(is_update, dtype=np.int32)
    lib().nro_bake_textures(_fp(image), _fp(uv_faces), _ip(upd), ctypes.c_int64(nf), int(texture_size), int(image.shape[0]),
                            int(image.shape[1]), _fp(textures))
    return textures


class OracleRasterize:
    """CPU restatement of the reference `Rasterize` function object (rasterize.py:19-897)."""

    def __init__(self, image_size, near, far, eps, background_color, return_rgb=False, return_alpha=False,
                 return_depth=False, tex_z_batch0=True):
        if not any((return_rgb, return_alpha, return_depth)):
            raise Exception("nothing to draw")  # rasterize.py:25-27
        self.image_size = int(image_size)
        self.near, self.far, self.eps = near, far, eps
        self.background_color = background_color
        self.return_rgb, self.return_alpha, self.return_depth = bool(return_rgb), bool(return_alpha), bool(return_depth)
        self.tex_z_batch0 = bool(tex_z_batch0)
        self.k5_sum_fp64 = False  # True: K5 keeps its sums in double (nr_oracle.c nro_pixel_bwd)

    # ---- forward (rasterize.py:467-513)
    def forward(self, faces, textures=None):
        L = lib()
        faces = _f32(faces)
        assert faces.ndim == 4 and faces.shape[2:] == (3, 3)
        bs, nf = faces.shape[:2]
        S = self.image_size
        self.faces = faces
        self.batch_size, self.num_faces = bs, nf
        self.face_index_map = np.full((bs, S, S), -1, np.int32)
        self.weight_map = np.zeros((bs, S, S, 3), np.float32)
        self.depth_map = np.zeros((bs, S, S), np.float32) + np.float32(self.far)
        self.face_inv_map = np.zeros((bs, S, S, 3, 3), np.float32) if self.return_depth else None
        self.alpha_map = np.zeros((bs, S, S), np.float32) if self.return_alpha else None
        self.rgb_map = None
        self.sampling_index_map = self.sampling_weight_map = None
        if self.return_rgb:
            textures = _f32(textures)
            assert textures.ndim == 6 and textures.shape[:2] == (bs, nf) and textures.shape[5] == 3
            ts = textures.shape[2]
            assert ts >= 2 and textures.shape[3] == ts and textures.shape[4] == ts
            self.textures, self.texture_size = textures, ts
            self.rgb_map = np.zeros((bs, S, S, 3), np.float32)
            self.sampling_index_map = np.zeros((bs, S, S, 8), np.int32)
            self.sampling_weight_map = np.zeros((bs, S, S, 8), np.float32)

        faces_inv = np.zeros_like(faces)
        L.nro_face_inv(_fp(faces), ctypes.c_int64(bs * nf), S, _fp(faces_inv))
        L.nro_zbuffer(_fp(faces), _fp(faces_inv), bs, nf, S, ctypes.c_double(self.near), ctypes.c_double(self.far),
                      _ip(self.face_index_map), _fp(self.weight_map), _fp(self.depth_map), _fp(self.face_inv_map))
        if self.return_rgb:
            L.nro_texture(_fp(faces), _fp(self.textures), _ip(self.face_index_map), _fp(self.weight_map),
                          _fp(self.depth_map), bs, nf, S, self.texture_size, ctypes.c_double(self.eps),
                          int(self.tex_z_batch0), _fp(self.rgb_map), _ip(self.sampling_index_map),
                          _fp(self.sampling_weight_map))
        bg = None
        per_batch = 0
        if self.return_rgb:
            bg = _f32(np.array(self.background_color, np.float32))
            per_batch = int(bg.ndim == 2)
        L.nro_compose(_ip(self.face_index_map), bs, S, _fp(bg), per_batch, _fp(self.rgb_map), _fp(self.alpha_map))
        rgb = self.rgb_map if self.return_rgb else None
        alpha = self.alpha_map.copy() if self.return_alpha else None
        depth = self.depth_map.copy() if self.return_depth else None
        return rgb, alpha, depth

    # ---- backward (rasterize.py:849-889)
    def backward(self, grad_rgb=None, grad_alpha=None, grad_depth=None):
        L = lib()
        bs, nf, S = self.batch_size, self.num_faces, self.image_size
        grad_faces = np.zeros_like(self.faces)
        grad_textures = np.zeros_like(self.textures) if self.return_rgb else None
        g_rgb = g_alpha = g_depth = None
        if self.return_rgb:
            g_rgb = _f32(grad_rgb) if grad_rgb is not None else np.zeros_like(self.rgb_map)
        if self.return_alpha:
            g_alpha = _f32(grad_alpha) if grad_alpha is not None else np.zeros_like(self.alpha_map)
        if self.return_depth:
            g_depth = _f32(grad_depth) if grad_depth is not None else np.zeros_like(self.depth_map)
        L.nro_pixel_bwd(_fp(self.faces), _ip(self.face_index_map), _fp(self.rgb_map), _fp(self.alpha_map), _fp(g_rgb),
                        _fp(g_alpha), bs, nf, S, ctypes.c_double(self.eps), int(self.return_rgb),
                        int(self.return_alpha), int(self.k5_sum_fp64), _fp(grad_faces))
        if self.return_rgb:
            L.nro_texture_bwd(_ip(self.face_index_map), _fp(self.sampling_weight_map), _ip(self.sampling_index_map),
                              _fp(g_rgb), bs, nf, S, self.texture_size, _fp(grad_textures))
        if self.return_depth:
            L.nro_depth_bwd(_fp(self.faces), _fp(self.depth_map), _ip(self.face_index_map), _fp(self.face_inv_map),
                            _fp(self.weight_map), _fp(g_depth), bs, nf, S, _fp(grad_faces))
        return grad_faces, grad_textures


def _avg_pool2(x):
    """2x2 mean over the last two axes (chainer.functions.average_pooling_2d(x, 2, 2), rasterize.py:962-969)."""
    return (x[..., 0::2, 0::2] + x[..., 0::2, 1::2] + x[..., 1::2, 0::2] + x[..., 1::2, 1::2]) * np.float32(0.25)


def _avg_pool2_bwd(g):
    out = np.repeat(np.repeat(g, 2, axis=-2), 2, axis=-1) * np.float32(0.25)
    return out


class RasterizeResult(dict):
    """dict {'rgb','alpha','depth'} (API layout) + .backward(grad_rgb, grad_alpha, grad_depth) -> (grad_faces, grad_textures)."""


def rasterize_rgbad(faces, textures=None, image_size=256, anti_aliasing=True, near=0.1, far=100, eps=1e-4,
                    background_color=(0, 0, 0), return_rgb=True, return_alpha=True, return_depth=True,
                    tex_z_batch0=True):
    """rasterize.py:900-977 on the CPU oracle."""
    S = image_size * 2 if anti_aliasing else image_size
    fn = OracleRasterize(S, near, far, eps, background_color, return_rgb, return_alpha, return_depth, tex_z_batch0)
    rgb, alpha, depth = fn.forward(faces, textures)
    if return_rgb:
        rgb = rgb.transpose(0, 3, 1, 2)[:, :, ::-1, :]
    if return_alpha:
        alpha = alpha[:, ::-1, :]
    if return_depth:
        depth = depth[:, ::-1, :]
    if anti_aliasing:
        if return_rgb:
            rgb = _avg_pool2(rgb)
        if return_alpha:
            alpha = _avg_pool2(alpha)
        if return_depth:
            depth = _avg_pool2(depth)
    res = RasterizeResult(rgb=np.ascontiguousarray(rgb) if return_rgb else None,
                          alpha=np.ascontiguousarray(alpha) if return_alpha else None,
                          depth=np.ascontiguousarray(depth) if return_depth else None)
    res.fn = fn

    def backward(grad_rgb=None, grad_alpha=None, grad_depth=None):
        def back(g, is_rgb):
            if g is None:
                return None
            g = _f32(g)
            if anti_aliasing:
                g = _avg_pool2_bwd(g)
            if is_rgb:
                g = g[:, :, ::-1, :].transpose(0, 2, 3, 1)
            else:
                g = g[:, ::-1, :]
            return np.ascontiguousarray(g)
        return fn.backward(back(grad_rgb, True), back(grad_alpha, False), back(grad_depth, False))

    res.backward = backward
    return res


def rasterize(faces, textures, image_size=256, anti_aliasing=True, near=0.1, far=100, eps=1e-4,
              background_color=(0, 0, 0)):
    return rasterize_rgbad(faces, textures, image_size, anti_aliasing, near, far, eps, background_color, True, False,
                           False)


def rasterize_silhouettes(faces, image_size=256, anti_aliasing=True, near=0.1, far=100, eps=1e-4):
    return rasterize_rgbad(faces, None, image_size, anti_aliasing, near, far, eps, None, False, True, False)


def rasterize_depth(faces, image_size=256, anti_aliasing=True, near=0.1, far=100, eps=1e-4):
    return rasterize_rgbad(faces, None, image_size, anti_aliasing, near, far, eps, None, False, False, True)


# --------------------------------------------------------------------------- glue (numpy, float32)

def _normalize(x, eps=1e-5):
    """chainer.functions.normalize: x / (||x||_2 + eps) along axis 1 (third-party; eps default 1e-5)."""
    n = np.sqrt((x * x).sum(axis=1, keepdims=True))
    return (x / (n + np.float32(eps))).astype(np.float32)


def vertices_to_faces(vertices, faces):
    """vertices_to_faces.py:4-21"""
    vertices = _f32(vertices)
    faces = np.asarray(faces)
    bs, nv = vertices.shape[:2]
    idx = faces.astype(np.int64) + (np.arange(bs, dtype=np.int64) * nv)[:, None, None]
    return vertices.reshape(bs * nv, 3)[idx]


def vertices_to_faces_bwd(grad_faces, faces, nv):
    bs = grad_faces.shape[0]
    idx = faces.astype(np.int64) + (np.arange(bs, dtype=np.int64) * nv)[:, None, None]
    out = np.zeros((bs * nv, 3), np.float32)
    np.add.at(out, idx.reshape(-1), grad_faces.reshape(-1, 3))
    return out.reshape(bs, nv, 3)


def look_at_matrix(eye, batch_size, at=None, up=None):
    eye = np.asarray(eye, np.float32)
    at = np.zeros(3, np.float32) if at is None else np.asarray(at, np.float32)
    up = np.array([0, 1, 0], np.float32) if up is None else np.asarray(up, np.float32)
    if eye.ndim == 1:
        eye = np.tile(eye[None], (batch_size, 1))
    if at.ndim == 1:
        at = np.tile(at[None], (batch_size, 1))
    if up.ndim == 1:
        up = np.tile(up[None], (batch_size, 1))
    z = _normalize(at - eye)
    x = _normalize(np.cross(up, z).astype(np.float32))
    y = _normalize(np.cross(z, x).astype(np.float32))
    r = np.stack([x, y, z], axis=1)  # [bs,3,3]
    return eye, r


def look_at(vertices, eye, at=None, up=None):
    """look_at.py:7-46: (v - eye) @ R^T"""
    vertices = _f32(vertices)
    eye, r = look_at_matrix(eye, vertices.shape[0], at, up)
    v = vertices - eye[:, None, :]
    return np.matmul(v, r.transpose(0, 2, 1)).astype(np.float32)


def look_at_bwd(grad, eye, batch_size, at=None, up=None):
    _, r = look_at_matrix(eye, batch_size, at, up)
    return np.matmul(grad, r).astype(np.float32)


def perspective(vertices, angle=30.):
    """perspective.py:5-19 (pi approximated by 3.1416 in the reference)."""
    vertices = _f32(vertices)
    a = np.float32(angle) / np.float32(180.) * np.float32(3.1416)
    width = np.float32(np.tan(a))
    z = vertices[:, :, 2]
    x = vertices[:, :, 0] / z / width
    y = vertices[:, :, 1] / z / width
    return np.stack([x, y, z], axis=2).astype(np.float32)


def perspective_bwd(grad, vertices, angle=30.):
    a = np.float32(angle) / np.float32(180.) * np.float32(3.1416)
    width = np.float32(np.tan(a))
    x, y, z = vertices[:, :, 0], vertices[:, :, 1], vertices[:, :, 2]
    gx = grad[:, :, 0] / z / width
    gy = grad[:, :, 1] / z / width
    gz = grad[:, :, 2] - grad[:, :, 0] * x / (z * z) / width - grad[:, :, 1] * y / (z * z) / width
    return np.stack([gx, gy, gz], axis=2).astype(np.float32)


def lighting(faces, textures, intensity_ambient=0.5, intensity_directional=0.5, color_ambient=(1, 1, 1),
             color_directional=(1, 1, 1), direction=(0, 1, 0)):
    """lighting.py:8-52"""
    faces, textures = _f32(faces), _f32(textures)
    bs, nf = faces.shape[:2]
    ca = np.broadcast_to(np.asarray(color_ambient, np.float32).reshape(-1, 3), (bs, 3))
    cd = np.broadcast_to(np.asarray(color_directional, np.float32).reshape(-1, 3), (bs, 3))
    di = np.broadcast_to(np.asarray(direction, np.float32).reshape(-1, 3), (bs, 3))
    light = np.zeros((bs, nf, 3), np.float32)
    if intensity_ambient != 0:
        light = light + np.float32(intensity_ambient) * ca[:, None, :]
    if intensity_directional != 0:
        f = faces.reshape(bs * nf, 3, 3)
        v10 = f[:, 0] - f[:, 1]
        v12 = f[:, 2] - f[:, 1]
        normals = _normalize(np.cross(v10, v12).astype(np.float32)).reshape(bs, nf, 3)
        cos = np.maximum((normals * di[:, None, :]).sum(axis=2), 0)
        light = light + np.float32(intensity_directional) * cd[:, None, :] * cos[:, :, None]
    return (textures * light[:, :, None, None, None, :]).astype(np.float32)


def get_points_from_angles(distance, elevation, azimuth, degrees=True):
    """get_points_from_angles.py:6-24 (scalar form)"""
    if degrees:
        elevation, azimuth = math.radians(elevation), math.radians(azimuth)
    return (distance * math.cos(elevation) * math.sin(azimuth), distance * math.sin(elevation),
            -distance * math.cos(elevation) * math.cos(azimuth))


class Renderer:
    """numpy restatement of renderer.py:8-107 on top of the CPU oracle (forward; backward for vertices through the
    rasterizer's edge gradients, vertices_to_faces, perspective and look_at -- lighting's vertex path is not
    differentiated here)."""

    def __init__(self):
        self.image_size = 256
        self.anti_aliasing = True
        self.background_color = [0, 0, 0]
        self.fill_back = True
        self.perspective = True
        self.viewing_angle = 30
        self.eye = [0, 0, -(1. / math.tan(math.radians(self.viewing_angle)) + 1)]
        self.camera_mode = 'look_at'
        self.camera_direction = [0, 0, 1]
        self.near = 0.1
        self.far = 100
        self.light_intensity_ambient = 0.5
        self.light_intensity_directional = 0.5
        self.light_color_ambient = [1, 1, 1]
        self.light_color_directional = [1, 1, 1]
        self.light_direction = [0, 1, 0]
        self.rasterizer_eps = 1e-3

    def _camera(self, vertices):
        self._v_in = _f32(vertices)
        v = self._v_in
        if self.camera_mode == 'look_at':
            v = look_at(v, self.eye)
        elif self.camera_mode == 'look':
            raise NotImplementedError("oracle glue implements look_at and 'none' only")
        self._v_cam = v
        if self.perspective:
            v = perspective(v, angle=self.viewing_angle)
        return v

    def _camera_bwd(self, grad_v):
        if self.perspective:
            grad_v = perspective_bwd(grad_v, self._v_cam, self.viewing_angle)
        if self.camera_mode == 'look_at':
            grad_v = look_at_bwd(grad_v, self.eye, grad_v.shape[0])
        return grad_v

    def _fill(self, faces):
        faces = np.asarray(faces)
        if self.fill_back:
            faces = np.concatenate((faces, faces[:, :, ::-1]), axis=1)
        return faces

    def _wrap(self, res, faces_idx, nv):
        def backward_vertices(**grads):
            gf, gt = res.backward(**grads)
            gv = vertices_to_faces_bwd(gf, faces_idx, nv)
            return self._camera_bwd(gv), gt
        res.backward_vertices = backward_vertices
        return res

    def render_silhouettes(self, vertices, faces):
        fidx = self._fill(faces)
        v = self._camera(vertices)
        f = vertices_to_faces(v, fidx)
        return self._wrap(rasterize_silhouettes(f, self.image_size, self.anti_aliasing), fidx, v.shape[1])

    def render_depth(self, vertices, faces):
        fidx = self._fill(faces)
        v = self._camera(vertices)
        f = vertices_to_faces(v, fidx)
        return self._wrap(rasterize_depth(f, self.image_size, self.anti_aliasing), fidx, v.shape[1])

    def render(self, vertices, faces, textures):
        faces = np.asarray(faces)
        textures = _f32(textures)
        if self.fill_back:
            faces = np.concatenate((faces, faces[:, :, ::-1]), axis=1)
            textures = np.concatenate((textures, textures.transpose(0, 1, 4, 3, 2, 5)), axis=1)
        faces_lighting = vertices_to_faces(vertices, faces)
        textures = lighting(faces_lighting, textures, self.light_intensity_ambient, self.light_intensity_directional,
                            self.light_color_ambient, self.light_color_directional, self.light_direction)
        v = self._camera(vertices)
        f = vertices_to_faces(v, faces)
        res = rasterize(f, textures, self.image_size, self.anti_aliasing, self.near, self.far, self.rasterizer_eps,
                        self.background_color)
        return self._wrap(res, faces, v.shape[1])


def load_obj(filename_obj, normalization=True):
    """Plain-numpy OBJ reader for fixtures (vertices `v`, faces `f`, fan triangulation), load_obj.py:147-192."""
    vertices, faces = [], []
    with open(filename_obj) as f:
        for line in f:
            tok = line.split()
            if not tok:
                continue
            if tok[0] == 'v':
                vertices.append([float(v) for v in tok[1:4]])
            elif tok[0] == 'f':
                vs = [int(t.split('/')[0]) for t in tok[1:]]
                for i in range(len(vs) - 2):
                    faces.append((vs[0], vs[i + 1], vs[i + 2]))
    vertices = np.array(vertices, np.float32)
    faces = np.array(faces, np.int32) - 1
    if normalization:
        vertices -= vertices.min(0)[None, :]
        vertices /= np.abs(vertices).max()
        vertices *= 2
        vertices -= vertices.max(0)[None, :] / 2
    return vertices, faces
