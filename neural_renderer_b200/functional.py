"""The steps either side of the rasterizer (SURVEY.md section 8(f)), each mirroring the reference function of the same
name.  On CUDA float32 tensors the camera pipeline, the per-face light factor and vertices_to_faces run as fused
kernels behind the C ABI (csrc/nr_glue.cu); the plain torch formulation below them serves CPU tensors and is the
test oracle of those kernels.  `Renderer` goes one step further and hands vertices + indices to the rasterizer itself
(NR_FACES_INDEXED), so vertices_to_faces does not run at all on its path.

  cross                   cross.py:6-59
  get_points_from_angles  get_points_from_angles.py:6-24
  look_at                 look_at.py:7-46
  look                    look.py:7-45
  perspective             perspective.py:5-19   (pi is 3.1416 there, kept)
  lighting                lighting.py:8-52
  vertices_to_faces       vertices_to_faces.py:4-21

Not in the reference: smooth (Gouraud) shading -- `vertex_normals` (area weighted) and `corner_light`, the Lambertian
light of lighting.py evaluated at every face corner with its vertex normal, which the rasterizer interpolates across the
face (rasterize(..., corner_light=...)).
"""
from __future__ import annotations

import math

import torch


def _normalize(x, eps=1e-5):
    # chainer.functions.normalize (third-party, unpinned): x / (||x||_2 + eps) along axis 1
    return x / (x.norm(dim=1, keepdim=True) + eps)


def cross(a, b):
    """Row-wise 3-vector cross product of [N,3] arrays."""
    if a.dim() != 2 or b.dim() != 2 or a.shape[1] != 3 or b.shape[1] != 3 or a.shape[0] != b.shape[0]:
        raise ValueError("cross expects two [N,3] tensors")
    return torch.linalg.cross(a, b, dim=1)


def get_points_from_angles(distance, elevation, azimuth, degrees=True):
    if isinstance(distance, (float, int)):
        if degrees:
            elevation = math.radians(elevation)
            azimuth = math.radians(azimuth)
        return (
            distance * math.cos(elevation) * math.sin(azimuth),
            distance * math.sin(elevation),
            -distance * math.cos(elevation) * math.cos(azimuth))
    distance = torch.as_tensor(distance)
    elevation = torch.as_tensor(elevation, dtype=distance.dtype, device=distance.device)
    azimuth = torch.as_tensor(azimuth, dtype=distance.dtype, device=distance.device)
    if degrees:
        elevation = torch.deg2rad(elevation)
        azimuth = torch.deg2rad(azimuth)
    return torch.stack([
        distance * torch.cos(elevation) * torch.sin(azimuth),
        distance * torch.sin(elevation),
        -distance * torch.cos(elevation) * torch.cos(azimuth),
    ]).t()


def _as_vec(v, like):
    if isinstance(v, torch.Tensor):
        return v.to(device=like.device, dtype=like.dtype)
    return torch.tensor(v, dtype=like.dtype, device=like.device)


class _CameraTransform(torch.autograd.Function):
    """out = perspective(rot @ (vertices - eye)) as one CUDA kernel each way (nr_b200_camera_transform*).

    rot [C,3,3] / eye [C,3] / width [C] with C == batch or C == 1 (one camera for every item); rot or eye may be
    None (identity / origin); width None = no perspective division."""

    @staticmethod
    def forward(ctx, vertices, rot, eye, width):
        import ctypes
        from . import _lib
        lib = _lib.load()
        v = vertices.detach().contiguous()
        bs, nv = v.shape[:2]
        cams = [t.shape[0] for t in (rot, eye, width) if t is not None]
        shared = all(c == 1 for c in cams) and bs != 1
        if any(c != (1 if shared else bs) for c in cams):
            raise ValueError("camera arrays must hold one item per batch entry or exactly one")
        flags = (_lib.NR_CAM_SHARED if shared else 0) | (_lib.NR_CAM_PERSPECTIVE if width is not None else 0)
        r = None if rot is None else rot.detach().to(torch.float32).contiguous()
        e = None if eye is None else eye.detach().to(torch.float32).contiguous()
        w = None if width is None else width.detach().to(torch.float32).contiguous()
        out = torch.empty_like(v)
        ptr = lambda t: None if t is None else t.data_ptr()
        with torch.cuda.device(v.device):
            stream = ctypes.c_void_p(torch.cuda.current_stream(v.device).cuda_stream)
            _lib.check(lib.nr_b200_camera_transform(v.data_ptr(), ptr(r), ptr(e), ptr(w), bs, nv, flags, out.data_ptr(), stream))
        ctx.save_for_backward(v, r, e, w)
        ctx.flags = flags
        return out

    @staticmethod
    def backward(ctx, grad_out):
        import ctypes
        from . import _lib
        lib = _lib.load()
        v, r, e, w = ctx.saved_tensors
        g = grad_out.detach().to(torch.float32).contiguous()
        bs, nv = v.shape[:2]
        need_v, need_r, need_e, need_w = ctx.needs_input_grad
        gv = torch.empty_like(v) if need_v else None
        gr = torch.empty_like(r) if (need_r and r is not None) else None
        ge = torch.empty_like(e) if (need_e and e is not None) else None
        gw = torch.empty_like(w) if (need_w and w is not None) else None
        ptr = lambda t: None if t is None else t.data_ptr()
        with torch.cuda.device(v.device):
            stream = ctypes.c_void_p(torch.cuda.current_stream(v.device).cuda_stream)
            _lib.check(lib.nr_b200_camera_transform_backward(v.data_ptr(), ptr(r), ptr(e), ptr(w), g.data_ptr(), bs, nv,
                                                             ctx.flags, ptr(gv), ptr(gr), ptr(ge), ptr(gw), stream))
        return gv, gr, ge, gw


def _fused_camera_ok(vertices):
    return vertices.is_cuda and vertices.dtype == torch.float32 and vertices.shape[0] <= 65535


_CAMERA_CACHE = {}  # small device constants (camera frames, tan(angle), light parameters) keyed by their host values


def _cache_put(key, value):
    if len(_CAMERA_CACHE) >= 256:  # bounded: a caller that animates the camera / light with Python floats must not leak
        _CAMERA_CACHE.clear()
    _CAMERA_CACHE[key] = value
    return value


def _host_camera(kind, eye, aux, up, device):
    """Rotation / eye of a camera given as plain Python numbers: evaluated once on the host in float32 with the same
    operation order as the tensor path, cached per (camera, device) -- zero device work per call."""
    import numpy as np
    key = (kind, tuple(float(x) for x in eye), tuple(float(x) for x in aux), tuple(float(x) for x in up), str(device))
    hit = _CAMERA_CACHE.get(key)
    if hit is not None:
        return hit
    f32 = np.float32

    def normalize(x):
        return x / (np.sqrt((x * x).sum(dtype=f32), dtype=f32) + f32(1e-5))
    e = np.asarray(key[1], dtype=f32)
    a = np.asarray(key[2], dtype=f32)
    u = np.asarray(key[3], dtype=f32)
    z_axis = normalize((a - e) if kind == "look_at" else a)
    x_axis = normalize(np.cross(u, z_axis).astype(f32))
    y_axis = normalize(np.cross(z_axis, x_axis).astype(f32))
    rot = torch.from_numpy(np.stack((x_axis, y_axis, z_axis))[None].astype(f32)).to(device)
    eye_t = torch.from_numpy(e[None]).to(device)
    return _cache_put(key, (rot, eye_t))


def _is_plain(*vals):
    return all(v is None or not isinstance(v, torch.Tensor) for v in vals)


def _camera_frame(kind, vertices, eye, aux, up):
    """(rot [C,3,3], eye [C,3]) of look_at (aux = at) / look (aux = direction); C = 1 or batch."""
    batch_size = vertices.shape[0]
    aux_default = [0, 0, 0] if kind == "look_at" else [0, 0, 1]
    if _is_plain(eye, aux, up) and _fused_camera_ok(vertices):
        import numpy as np
        eye_np = np.asarray(eye, dtype=np.float64)
        if eye_np.ndim == 1:
            return _host_camera(kind, eye_np, aux_default if aux is None else aux, [0, 1, 0] if up is None else up,
                                vertices.device)
    aux = _as_vec(aux_default if aux is None else aux, vertices)
    up = _as_vec([0, 1, 0] if up is None else up, vertices)
    eye = _as_vec(eye, vertices)
    if eye.dim() == 1:
        eye = eye[None, :]
    if aux.dim() == 1:
        aux = aux[None, :]
    if up.dim() == 1:
        up = up[None, :]
    n = max(eye.shape[0], aux.shape[0], up.shape[0])
    z_axis = _normalize((aux - eye) if kind == "look_at" else aux)
    if z_axis.shape[0] != n:
        z_axis = z_axis.expand(n, 3)
    x_axis = _normalize(cross(up.expand(n, 3), z_axis))
    y_axis = _normalize(cross(z_axis, x_axis))
    rot = torch.stack((x_axis, y_axis, z_axis), dim=1)  # [C,3,3]
    if n not in (1, batch_size):
        raise ValueError("camera batch does not match the vertices")
    return rot, (eye if eye.shape[0] == n else eye.expand(n, 3))


def _perspective_width(vertices, angle):
    """tan(angle / 180 * 3.1416) as a [C] tensor (perspective.py:12-14; pi is 3.1416 there, kept)."""
    if isinstance(angle, (float, int)):
        key = ("width", float(angle), str(vertices.device), str(vertices.dtype))
        hit = _CAMERA_CACHE.get(key)
        if hit is None:
            a = torch.tensor(float(angle), dtype=vertices.dtype, device=vertices.device) / 180. * 3.1416
            hit = _cache_put(key, torch.tan(a)[None])
        return hit
    angle = angle / 180. * 3.1416
    angle = angle[None] if angle.dim() == 0 else angle
    return torch.tan(angle)


def camera_transform(vertices, eye, camera_mode="look_at", camera_direction=None, perspective=True, viewing_angle=30.,
                     at=None, up=None):
    """Renderer's camera pipeline (renderer.py:41-50): look_at / look, then perspective -- one fused kernel each way on
    CUDA float32 vertices, the reference's op-by-op formulation otherwise."""
    assert vertices.dim() == 3
    if not _fused_camera_ok(vertices):
        if camera_mode == "look_at":
            vertices = look_at(vertices, eye, at, up)
        elif camera_mode == "look":
            vertices = look(vertices, eye, camera_direction, up)
        return perspective_(vertices, viewing_angle) if perspective else vertices
    rot = eye_t = None
    if camera_mode == "look_at":
        rot, eye_t = _camera_frame("look_at", vertices, eye, at, up)
    elif camera_mode == "look":
        rot, eye_t = _camera_frame("look", vertices, eye, camera_direction, up)
    width = _perspective_width(vertices, viewing_angle) if perspective else None
    if rot is None and width is None:
        return vertices
    if rot is not None and width is not None and rot.shape[0] != width.shape[0]:
        n = max(rot.shape[0], width.shape[0])
        rot, eye_t, width = rot.expand(n, 3, 3), eye_t.expand(n, 3), width.expand(n)
    return _CameraTransform.apply(vertices, rot, eye_t, width)


def look_at(vertices, eye, at=None, up=None):
    """"Look at" transformation of vertices [B,Nv,3]."""
    if vertices.dim() == 3 and _fused_camera_ok(vertices):
        rot, eye_t = _camera_frame("look_at", vertices, eye, at, up)
        return _CameraTransform.apply(vertices, rot, eye_t, None)
    assert vertices.dim() == 3
    batch_size = vertices.shape[0]
    at = _as_vec([0, 0, 0] if at is None else at, vertices)
    up = _as_vec([0, 1, 0] if up is None else up, vertices)
    eye = _as_vec(eye, vertices)
    if eye.dim() == 1:
        eye = eye[None, :].expand(batch_size, 3)
    if at.dim() == 1:
        at = at[None, :].expand(batch_size, 3)
    if up.dim() == 1:
        up = up[None, :].expand(batch_size, 3)
    z_axis = _normalize(at - eye)
    x_axis = _normalize(cross(up, z_axis))
    y_axis = _normalize(cross(z_axis, x_axis))
    r = torch.stack((x_axis, y_axis, z_axis), dim=1)  # [bs,3,3]
    if r.shape[0] != vertices.shape[0]:
        r = r.expand(vertices.shape[0], 3, 3)
    vertices = vertices - eye[:, None, :]
    return torch.matmul(vertices, r.transpose(1, 2))


def look(vertices, eye, direction=None, up=None):
    """"Look" transformation of vertices [B,Nv,3] (camera at `eye` looking along `direction`)."""
    if vertices.dim() == 3 and _fused_camera_ok(vertices):
        rot, eye_t = _camera_frame("look", vertices, eye, direction, up)
        return _CameraTransform.apply(vertices, rot, eye_t, None)
    assert vertices.dim() == 3
    direction = _as_vec([0, 0, 1] if direction is None else direction, vertices)
    up = _as_vec([0, 1, 0] if up is None else up, vertices)
    eye = _as_vec(eye, vertices)
    if eye.dim() == 1:
        eye = eye[None, :]
    if direction.dim() == 1:
        direction = direction[None, :]
    if up.dim() == 1:
        up = up[None, :]
    z_axis = _normalize(direction)
    x_axis = _normalize(cross(up, z_axis))
    y_axis = _normalize(cross(z_axis, x_axis))
    r = torch.stack((x_axis, y_axis, z_axis), dim=1)
    if r.shape[0] != vertices.shape[0]:
        r = r.expand(vertices.shape[0], 3, 3)
    vertices = vertices - eye[:, None, :]
    return torch.matmul(vertices, r.transpose(1, 2))


def perspective(vertices, angle=30.):
    assert vertices.dim() == 3
    if _fused_camera_ok(vertices):
        return _CameraTransform.apply(vertices, None, None, _perspective_width(vertices, angle))
    if isinstance(angle, (float, int)):
        angle = torch.tensor(float(angle), dtype=vertices.dtype, device=vertices.device)
    angle = angle / 180. * 3.1416
    angle = angle[None].expand(vertices.shape[0]) if angle.dim() == 0 else angle
    width = torch.tan(angle)[:, None]
    z = vertices[:, :, 2]
    x = vertices[:, :, 0] / z / width
    y = vertices[:, :, 1] / z / width
    return torch.stack((x, y, z), dim=2)


perspective_ = perspective


def face_light(faces, intensity_ambient=0.5, intensity_directional=0.5, color_ambient=(1, 1, 1),
               color_directional=(1, 1, 1), direction=(0, 1, 0)):
    """Per-face RGB light factor [B,F,3] of lighting.py:29-51 (ambient + Lambertian directional)."""
    bs, nf = faces.shape[:2]
    color_ambient = _as_vec(color_ambient, faces)
    color_directional = _as_vec(color_directional, faces)
    direction = _as_vec(direction, faces)
    if color_ambient.dim() == 1:
        color_ambient = color_ambient[None, :].expand(bs, 3)
    if color_directional.dim() == 1:
        color_directional = color_directional[None, :].expand(bs, 3)
    if direction.dim() == 1:
        direction = direction[None, :].expand(bs, 3)
    light = torch.zeros((bs, nf, 3), dtype=faces.dtype, device=faces.device)
    if intensity_ambient != 0:
        light = light + intensity_ambient * color_ambient[:, None, :]
    if intensity_directional != 0:
        f = faces.reshape(bs * nf, 3, 3)
        v10 = f[:, 0] - f[:, 1]
        v12 = f[:, 2] - f[:, 1]
        normals = _normalize(cross(v10, v12)).reshape(bs, nf, 3)
        cos = torch.relu((normals * direction[:, None, :]).sum(dim=2))
        light = light + intensity_directional * color_directional[:, None, :] * cos[:, :, None]
    return light


class _FaceLighting(torch.autograd.Function):
    """face_light [B,F,3] straight from vertices and face indices (nr_b200_face_lighting*); params [C,9], C in {1, B}."""

    @staticmethod
    def forward(ctx, vertices, faces_i32, params):
        import ctypes
        from . import _lib
        lib = _lib.load()
        v = vertices.detach().contiguous()
        bs, nv = v.shape[:2]
        nf = faces_i32.shape[1]
        flags = _lib.NR_CAM_SHARED if (params.shape[0] == 1 and bs != 1) else 0
        if faces_i32.shape[0] == 1 and bs != 1:
            flags |= _lib.NR_INDICES_SHARED  # one index set for every batch item
        out = torch.empty((bs, nf, 3), dtype=torch.float32, device=v.device)
        with torch.cuda.device(v.device):
            stream = ctypes.c_void_p(torch.cuda.current_stream(v.device).cuda_stream)
            _lib.check(lib.nr_b200_face_lighting(v.data_ptr(), faces_i32.data_ptr(), params.data_ptr(), bs, nv, nf, flags,
                                                 out.data_ptr(), stream))
        ctx.save_for_backward(v, faces_i32, params)
        ctx.flags = flags
        return out

    @staticmethod
    def backward(ctx, grad_light):
        import ctypes
        from . import _lib
        lib = _lib.load()
        v, faces_i32, params = ctx.saved_tensors
        g = grad_light.detach().to(torch.float32).contiguous()
        bs, nv = v.shape[:2]
        grad_v = torch.empty_like(v)
        with torch.cuda.device(v.device):
            stream = ctypes.c_void_p(torch.cuda.current_stream(v.device).cuda_stream)
            _lib.check(lib.nr_b200_face_lighting_backward(v.data_ptr(), faces_i32.data_ptr(), params.data_ptr(), g.data_ptr(), bs,
                                                          nv, faces_i32.shape[1], ctx.flags, grad_v.data_ptr(), stream))
        return grad_v, None, None


def face_light_from_vertices(vertices, faces, intensity_ambient=0.5, intensity_directional=0.5, color_ambient=(1, 1, 1),
                             color_directional=(1, 1, 1), direction=(0, 1, 0)):
    """`face_light(vertices_to_faces(vertices, faces), ...)` without the gathered tensor: one kernel each way on CUDA."""
    plain = _is_plain(intensity_ambient, intensity_directional, color_ambient, color_directional, direction)
    if not (plain and _fused_camera_ok(vertices) and faces.is_cuda):
        return face_light(vertices_to_faces(vertices, faces), intensity_ambient, intensity_directional, color_ambient,
                          color_directional, direction)
    import numpy as np
    ca, cd, d = (np.asarray(x, dtype=np.float32) for x in (color_ambient, color_directional, direction))
    if ca.ndim != 1 or cd.ndim != 1 or d.ndim != 1:
        return face_light(vertices_to_faces(vertices, faces), intensity_ambient, intensity_directional, color_ambient,
                          color_directional, direction)
    key = ("light", float(intensity_ambient), float(intensity_directional), tuple(ca.tolist()), tuple(cd.tolist()),
           tuple(d.tolist()), str(vertices.device))
    params = _CAMERA_CACHE.get(key)
    if params is None:
        row = np.concatenate([np.float32(intensity_ambient) * ca, np.float32(intensity_directional) * cd, d]).astype(np.float32)
        params = _cache_put(key, torch.from_numpy(row[None]).to(vertices.device))
    if faces.dim() == 3 and faces.shape[0] > 1 and faces.stride(0) == 0:
        faces = faces[:1]  # expanded shared index set: keep it shared
    return _FaceLighting.apply(vertices, faces.to(torch.int32).contiguous(), params)


def lighting(faces, textures, intensity_ambient=0.5, intensity_directional=0.5, color_ambient=(1, 1, 1),
             color_directional=(1, 1, 1), direction=(0, 1, 0)):
    light = face_light(faces, intensity_ambient, intensity_directional, color_ambient, color_directional, direction)
    return textures * light[:, :, None, None, None, :]  # lighting.py:52


class _VerticesToFaces(torch.autograd.Function):
    """CUDA gather (forward) / scatter-add (backward) behind the C ABI (nr_b200_vertices_to_faces*)."""

    @staticmethod
    def forward(ctx, vertices, faces_i32):
        import ctypes
        from . import _lib
        lib = _lib.load()
        v = vertices.detach().contiguous()
        bs, nv = v.shape[:2]
        nf = faces_i32.shape[1]
        out = torch.empty((bs, nf, 3, 3), dtype=torch.float32, device=v.device)
        with torch.cuda.device(v.device):
            stream = ctypes.c_void_p(torch.cuda.current_stream(v.device).cuda_stream)
            _lib.check(lib.nr_b200_vertices_to_faces(v.data_ptr(), faces_i32.data_ptr(), bs, nv, nf, out.data_ptr(), stream))
        ctx.save_for_backward(faces_i32)
        ctx.nv = nv
        return out

    @staticmethod
    def backward(ctx, grad_out):
        import ctypes
        from . import _lib
        lib = _lib.load()
        faces_i32, = ctx.saved_tensors
        g = grad_out.detach().to(torch.float32).contiguous()
        bs, nf = g.shape[:2]
        grad_v = torch.empty((bs, ctx.nv, 3), dtype=torch.float32, device=g.device)
        with torch.cuda.device(g.device):
            stream = ctypes.c_void_p(torch.cuda.current_stream(g.device).cuda_stream)
            _lib.check(lib.nr_b200_vertices_to_faces_backward(g.data_ptr(), faces_i32.data_ptr(), bs, ctx.nv, nf,
                                                              grad_v.data_ptr(), 0, stream))
        return grad_v, None


def vertices_to_faces(vertices, faces):
    """[B,Nv,3] x [B,Nf,3] int -> [B,Nf,3,3]"""
    assert vertices.dim() == 3
    assert faces.dim() == 3
    assert vertices.shape[0] == faces.shape[0]
    assert vertices.shape[2] == 3
    assert faces.shape[2] == 3
    bs, nv = vertices.shape[:2]
    if vertices.is_cuda and faces.is_cuda and vertices.dtype == torch.float32 and bs <= 65535:
        return _VerticesToFaces.apply(vertices, faces.to(torch.int32).contiguous())
    idx = faces.long() + (torch.arange(bs, device=faces.device, dtype=torch.long) * nv)[:, None, None]
    return vertices.reshape(bs * nv, 3)[idx]


def _light_params(intensity_ambient, intensity_directional, color_ambient, color_directional, direction, device):
    """light_params [1,9] of the CUDA light kernels (cached per value), or None for tensor-valued / batched parameters."""
    if not _is_plain(intensity_ambient, intensity_directional, color_ambient, color_directional, direction):
        return None
    import numpy as np
    ca, cd, d = (np.asarray(x, dtype=np.float32) for x in (color_ambient, color_directional, direction))
    if ca.ndim != 1 or cd.ndim != 1 or d.ndim != 1:
        return None
    key = ("light", float(intensity_ambient), float(intensity_directional), tuple(ca.tolist()), tuple(cd.tolist()),
           tuple(d.tolist()), str(device))
    params = _CAMERA_CACHE.get(key)
    if params is None:
        row = np.concatenate([np.float32(intensity_ambient) * ca, np.float32(intensity_directional) * cd, d]).astype(np.float32)
        params = _cache_put(key, torch.from_numpy(row[None]).to(device))
    return params


def _index_set(faces, batch_size):
    """faces [F,3] / [1|B,F,3] (an expanded shared set stays shared) -> (int32 [1|B,F,3], shared)"""
    if faces.dim() == 2:
        faces = faces[None]
    if faces.shape[0] > 1 and faces.stride(0) == 0:
        faces = faces[:1]
    if faces.shape[0] not in (1, batch_size):
        raise ValueError("faces must have shape [num faces, 3] or [batch size, num faces, 3]")
    return faces.to(torch.int32).contiguous(), faces.shape[0] == 1 and batch_size != 1


def _gather_vertices(values, faces):
    """values [B,Nv,3], faces [1|B,F,3] -> [B,F,3,3] (zeros for indices outside [0, Nv)) and the in-range mask [B,F,3]"""
    bs, nv = values.shape[:2]
    idx = faces.long().expand(bs, -1, -1)
    ok = (idx >= 0) & (idx < nv)
    flat = (idx.clamp(0, nv - 1) + (torch.arange(bs, device=values.device) * nv)[:, None, None])
    return values.reshape(bs * nv, 3)[flat] * ok[..., None].to(values.dtype), ok


def _vertex_normals_torch(vertices, faces):
    bs, nv = vertices.shape[:2]
    faces = faces[None] if faces.dim() == 2 else faces
    v, ok = _gather_vertices(vertices, faces)
    face_ok = ok.all(dim=2)
    c = torch.linalg.cross(v[:, :, 0] - v[:, :, 1], v[:, :, 2] - v[:, :, 1], dim=2) * face_ok[..., None].to(v.dtype)
    idx = faces.long().expand(bs, -1, -1)
    corner_ok = (idx >= 0) & (idx < nv)
    target = (idx.clamp(0, nv - 1) + (torch.arange(bs, device=vertices.device) * nv)[:, None, None])
    contrib = c[:, :, None, :].expand(-1, -1, 3, -1) * corner_ok[..., None].to(c.dtype)
    s = torch.zeros((bs * nv, 3), dtype=vertices.dtype, device=vertices.device)
    s = s.index_add(0, target.reshape(-1), contrib.reshape(-1, 3)).reshape(bs, nv, 3)
    return s / (s.norm(dim=2, keepdim=True) + 1e-5)


class _VertexNormals(torch.autograd.Function):
    """vertex normals [B,Nv,3] from vertices and an index set (nr_b200_vertex_normals*); faces_i32 [1|B,F,3]."""

    @staticmethod
    def forward(ctx, vertices, faces_i32, shared):
        import ctypes
        from . import _lib
        lib = _lib.load()
        v = vertices.detach().contiguous()
        bs, nv = v.shape[:2]
        nf = faces_i32.shape[1]
        flags = _lib.NR_INDICES_SHARED if shared else 0
        out = torch.empty_like(v)
        with torch.cuda.device(v.device):
            ws_bytes = lib.nr_b200_vertex_normals_workspace_bytes(bs, nv, nf, flags)
            if ws_bytes == 0:
                raise RuntimeError("nr_b200: vertex normals of this size are not supported")
            ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=v.device)
            stream = ctypes.c_void_p(torch.cuda.current_stream(v.device).cuda_stream)
            _lib.check(lib.nr_b200_vertex_normals(v.data_ptr(), faces_i32.data_ptr(), bs, nv, nf, flags, out.data_ptr(),
                                                  ws.data_ptr(), ws_bytes, stream))
        ctx.save_for_backward(v, faces_i32)
        ctx.flags = flags
        return out

    @staticmethod
    def backward(ctx, grad_normals):
        import ctypes
        from . import _lib
        lib = _lib.load()
        v, faces_i32 = ctx.saved_tensors
        g = grad_normals.detach().to(torch.float32).contiguous()
        bs, nv = v.shape[:2]
        nf = faces_i32.shape[1]
        grad_v = torch.empty_like(v)
        with torch.cuda.device(v.device):
            ws_bytes = lib.nr_b200_vertex_normals_workspace_bytes(bs, nv, nf, ctx.flags)
            ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=v.device)
            stream = ctypes.c_void_p(torch.cuda.current_stream(v.device).cuda_stream)
            _lib.check(lib.nr_b200_vertex_normals_backward(v.data_ptr(), faces_i32.data_ptr(), g.data_ptr(), bs, nv, nf,
                                                           ctx.flags, grad_v.data_ptr(), ws.data_ptr(), ws_bytes, stream))
        return grad_v, None, None


def vertex_normals(vertices, faces):
    """Area-weighted vertex normals [B,Nv,3] of vertices [B,Nv,3] and faces [F,3] / [1|B,F,3] (integer indices):
    s_v = sum of cross(v0 - v1, v2 - v1) over the faces at v (the face-normal direction of `face_light`), n_v = s_v /
    (|s_v| + 1e-5).  A face with an index outside [0, Nv) contributes nothing; an unreferenced vertex gets 0.  Pass the
    original faces, not the fill_back-doubled set.  One deterministic CUDA kernel pair for CUDA float32 tensors."""
    assert vertices.dim() == 3 and vertices.shape[2] == 3
    if _fused_camera_ok(vertices) and faces.is_cuda:
        faces_i32, shared = _index_set(faces, vertices.shape[0])
        return _VertexNormals.apply(vertices, faces_i32, shared)
    return _vertex_normals_torch(vertices, faces)


def _corner_light_torch(vertex_normals, faces, intensity_ambient, intensity_directional, color_ambient, color_directional,
                        direction, fill_back):
    bs, nv = vertex_normals.shape[:2]
    faces = faces[None] if faces.dim() == 2 else faces
    nf = faces.shape[1]
    color_ambient, color_directional, direction = (_as_vec(x, vertex_normals) for x in (color_ambient, color_directional,
                                                                                        direction))
    color_ambient, color_directional, direction = (x[None, :].expand(bs, 3) if x.dim() == 1 else x
                                                   for x in (color_ambient, color_directional, direction))
    n, _ = _gather_vertices(vertex_normals, faces)  # [B,F,3 corners,3]
    light = torch.zeros((bs, nf, 3, 3), dtype=vertex_normals.dtype, device=vertex_normals.device)
    if intensity_ambient != 0:
        light = light + (intensity_ambient * color_ambient)[:, None, None, :]
    if intensity_directional != 0:
        dot = (n * direction[:, None, None, :]).sum(dim=3)
        if fill_back:
            sign = torch.ones(nf, dtype=dot.dtype, device=dot.device)
            sign[nf // 2:] = -1
            dot = dot * sign[None, :, None]
        light = light + (intensity_directional * color_directional)[:, None, None, :] * torch.relu(dot)[..., None]
    return light


class _CornerLighting(torch.autograd.Function):
    """corner_light [B,F,3,3] from vertex normals (nr_b200_corner_lighting*); params [1,9]."""

    @staticmethod
    def forward(ctx, normals, faces_i32, params, flags):
        import ctypes
        from . import _lib
        lib = _lib.load()
        n = normals.detach().to(torch.float32).contiguous()
        bs, nv = n.shape[:2]
        nf = faces_i32.shape[1]
        out = torch.empty((bs, nf, 3, 3), dtype=torch.float32, device=n.device)
        with torch.cuda.device(n.device):
            stream = ctypes.c_void_p(torch.cuda.current_stream(n.device).cuda_stream)
            _lib.check(lib.nr_b200_corner_lighting(n.data_ptr(), faces_i32.data_ptr(), params.data_ptr(), bs, nv, nf, flags,
                                                   out.data_ptr(), stream))
        ctx.save_for_backward(n, faces_i32, params)
        ctx.flags = flags
        return out

    @staticmethod
    def backward(ctx, grad_light):
        import ctypes
        from . import _lib
        lib = _lib.load()
        n, faces_i32, params = ctx.saved_tensors
        g = grad_light.detach().to(torch.float32).contiguous()
        bs, nv = n.shape[:2]
        grad_n = torch.empty_like(n)
        with torch.cuda.device(n.device):
            stream = ctypes.c_void_p(torch.cuda.current_stream(n.device).cuda_stream)
            _lib.check(lib.nr_b200_corner_lighting_backward(n.data_ptr(), faces_i32.data_ptr(), params.data_ptr(), g.data_ptr(),
                                                            bs, nv, faces_i32.shape[1], ctx.flags, grad_n.data_ptr(), stream))
        return grad_n, None, None, None


def corner_light(vertex_normals, faces, intensity_ambient=0.5, intensity_directional=0.5, color_ambient=(1, 1, 1),
                 color_directional=(1, 1, 1), direction=(0, 1, 0), fill_back=False):
    """Per-corner RGB light factor [B,F,3,3] for rasterize(..., corner_light=...): the Lambertian light of `face_light`
    with the normal of each corner's vertex, ambient + directional * relu(n . direction).  `faces` [F,3] / [1|B,F,3] is
    the index set the rasterizer receives; with fill_back=True faces [F/2, F) are the reversed copies and use -n.  An
    index outside [0, Nv) gets n = 0.  No gradient flows into the light parameters.  One CUDA kernel pair for CUDA float32
    tensors with plain-number light parameters, the torch formulation otherwise."""
    assert vertex_normals.dim() == 3 and vertex_normals.shape[2] == 3
    nf = faces.shape[-2]
    if fill_back and nf % 2:
        raise ValueError("fill_back needs an even number of faces (front faces, then their reversed copies)")
    params = _light_params(intensity_ambient, intensity_directional, color_ambient, color_directional, direction,
                           vertex_normals.device) if (_fused_camera_ok(vertex_normals) and faces.is_cuda) else None
    if params is None:
        return _corner_light_torch(vertex_normals, faces, intensity_ambient, intensity_directional, color_ambient,
                                   color_directional, direction, fill_back)
    from . import _lib
    faces_i32, shared = _index_set(faces, vertex_normals.shape[0])
    flags = (_lib.NR_CAM_SHARED if vertex_normals.shape[0] != 1 else 0) | (_lib.NR_INDICES_SHARED if shared else 0) | \
        (_lib.NR_TEX_FILL_BACK if fill_back else 0)
    return _CornerLighting.apply(vertex_normals, faces_i32, params, flags)


def _corner_shading_torch(vertex_normals, vertices, faces, fill_back):
    faces = faces[None] if faces.dim() == 2 else faces
    nf = faces.shape[1]
    n, _ = _gather_vertices(vertex_normals, faces)  # [B,F,3 corners,3], zeros for an out-of-range index
    p, _ = _gather_vertices(vertices, faces)
    if fill_back:
        sign = torch.ones(nf, dtype=n.dtype, device=n.device)
        sign[nf // 2:] = -1
        n = n * sign[None, :, None, None]
    return torch.cat((n, p), dim=3)


class _CornerShading(torch.autograd.Function):
    """corner_shading [B,F,3,6] from vertex normals and vertices (nr_b200_corner_shading*); faces_i32 [1|B,F,3]."""

    @staticmethod
    def forward(ctx, normals, vertices, faces_i32, flags):
        import ctypes
        from . import _lib
        lib = _lib.load()
        n = normals.detach().to(torch.float32).contiguous()
        v = vertices.detach().to(torch.float32).contiguous()
        bs, nv = n.shape[:2]
        nf = faces_i32.shape[1]
        out = torch.empty((bs, nf, 3, 6), dtype=torch.float32, device=n.device)
        with torch.cuda.device(n.device):
            stream = ctypes.c_void_p(torch.cuda.current_stream(n.device).cuda_stream)
            _lib.check(lib.nr_b200_corner_shading(n.data_ptr(), v.data_ptr(), faces_i32.data_ptr(), bs, nv, nf, flags,
                                                  out.data_ptr(), stream))
        ctx.save_for_backward(faces_i32)
        ctx.flags, ctx.bs, ctx.nv = flags, bs, nv
        return out

    @staticmethod
    def backward(ctx, grad):
        import ctypes
        from . import _lib
        lib = _lib.load()
        faces_i32, = ctx.saved_tensors
        want_n, want_v = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        if not (want_n or want_v):
            return None, None, None, None
        g = grad.detach().to(torch.float32).contiguous()
        grad_n = torch.empty((ctx.bs, ctx.nv, 3), dtype=torch.float32, device=g.device) if want_n else None
        grad_v = torch.empty((ctx.bs, ctx.nv, 3), dtype=torch.float32, device=g.device) if want_v else None
        ptr = lambda t: None if t is None else t.data_ptr()
        with torch.cuda.device(g.device):
            stream = ctypes.c_void_p(torch.cuda.current_stream(g.device).cuda_stream)
            _lib.check(lib.nr_b200_corner_shading_backward(faces_i32.data_ptr(), g.data_ptr(), ctx.bs, ctx.nv,
                                                           faces_i32.shape[1], ctx.flags, ptr(grad_n), ptr(grad_v), stream))
        return grad_n, grad_v, None, None


def corner_shading(vertex_normals, vertices, faces, fill_back=False):
    """Per-corner shading normal and position [B,F,3,6] for rasterize(..., corner_shading=...) (Phong shading): corner k of
    face f holds (n, v) of vertex faces[f,k], n from `vertex_normals` [B,Nv,3] and v from `vertices` [B,Nv,3] (the positions
    in the frame of the eye of F.phong_params).  `faces` [F,3] / [1|B,F,3] is the index set the rasterizer receives; with
    fill_back=True faces [F/2, F) are the reversed copies and get -n.  An index outside [0, Nv) gives zeros.  One CUDA
    kernel pair for CUDA float32 tensors, the torch formulation otherwise; both inputs receive gradients."""
    assert vertex_normals.dim() == 3 and vertex_normals.shape[2] == 3
    assert tuple(vertices.shape) == tuple(vertex_normals.shape)
    nf = faces.shape[-2]
    if fill_back and nf % 2:
        raise ValueError("fill_back needs an even number of faces (front faces, then their reversed copies)")
    if not (_fused_camera_ok(vertex_normals) and _fused_camera_ok(vertices) and faces.is_cuda):
        return _corner_shading_torch(vertex_normals, vertices, faces, fill_back)
    from . import _lib
    faces_i32, shared = _index_set(faces, vertex_normals.shape[0])
    flags = (_lib.NR_INDICES_SHARED if shared else 0) | (_lib.NR_TEX_FILL_BACK if fill_back else 0)
    return _CornerShading.apply(vertex_normals, vertices, faces_i32, flags)


def phong_params(intensity_ambient=0.5, intensity_directional=0.5, intensity_specular=0.2, color_ambient=(1, 1, 1),
                 color_directional=(1, 1, 1), color_specular=(1, 1, 1), direction=(0, 1, 0), shininess=64.0, eye=(0, 0, 0),
                 device=None):
    """Phong parameters [1|B,16] for rasterize(..., shading_params=...): {ambient intensity * colour (3), directional
    intensity * colour (3), light direction (3, towards the light, not normalised), specular intensity * colour (3),
    shininess, eye position (3)}.  Built with torch ops, so tensor-valued arguments (intensities and shininess scalar or
    [B], colours, direction and eye [3] or [B,3]) receive gradients.  `device`: where plain numbers go (default: the device
    of the first tensor argument, else the CPU)."""
    args = (intensity_ambient, intensity_directional, intensity_specular, color_ambient, color_directional, color_specular,
            direction, shininess, eye)
    if device is None:
        device = next((a.device for a in args if isinstance(a, torch.Tensor)), torch.device('cpu'))
    key = None
    if _is_plain(*args):  # plain numbers: one cached device tensor per value (no host copy per call, CUDA-graph safe)
        import numpy as np
        key = ("phong",) + tuple(tuple(np.asarray(a, dtype=np.float64).reshape(-1).tolist()) for a in args) + (str(device),)
        if key in _CAMERA_CACHE:
            return _CAMERA_CACHE[key]

    def as_t(x, cols):
        t = x.to(device=device, dtype=torch.float32) if isinstance(x, torch.Tensor) else \
            torch.tensor(x, dtype=torch.float32, device=device)
        return t.reshape(-1, cols) if t.dim() <= 1 else t

    A = as_t(intensity_ambient, 1) * as_t(color_ambient, 3)
    D = as_t(intensity_directional, 1) * as_t(color_directional, 3)
    K = as_t(intensity_specular, 1) * as_t(color_specular, 3)
    parts = [A, D, as_t(direction, 3), K, as_t(shininess, 1), as_t(eye, 3)]
    n = max(p.shape[0] for p in parts)
    if any(p.shape[0] not in (1, n) for p in parts):
        raise ValueError("Phong parameters must hold one entry or one per batch item")
    out = torch.cat([p.expand(n, -1) for p in parts], dim=1)
    return out if key is None else _cache_put(key, out)


def _light_record(kind, x, intensity, color, intensity_specular, color_specular, falloff, device):
    args = (x, intensity, color, intensity_specular, color_specular, falloff)
    if device is None:
        device = next((a.device for a in args if isinstance(a, torch.Tensor)), torch.device('cpu'))
    key = None
    if _is_plain(*args):  # plain numbers: one cached device tensor per value (no host copy per call, CUDA-graph safe)
        import numpy as np
        key = ("light", kind) + tuple(tuple(np.asarray(a, dtype=np.float64).reshape(-1).tolist()) for a in args) + \
            (str(device),)
        if key in _CAMERA_CACHE:
            return _CAMERA_CACHE[key]

    def as_t(v, cols):
        t = v.to(device=device, dtype=torch.float32) if isinstance(v, torch.Tensor) else \
            torch.tensor(v, dtype=torch.float32, device=device)
        return t.reshape(-1, cols) if t.dim() <= 1 else t

    D = as_t(intensity, 1) * as_t(color, 3)
    K = as_t(intensity_specular, 1) * as_t(color_specular, 3)
    f = as_t(falloff, 1)
    parts = [D, K, as_t(x, 3), f]
    n = max(p.shape[0] for p in parts)
    if any(p.shape[0] not in (1, n) for p in parts):
        raise ValueError("light parameters must hold one entry or one per batch item")
    tail = torch.tensor([[kind, 0.0]], dtype=torch.float32, device=device)
    out = torch.cat([p.expand(n, -1) for p in parts] + [tail.expand(n, -1)], dim=1)
    return out if key is None else _cache_put(key, out)


def directional_light(direction, intensity=0.5, color=(1, 1, 1), intensity_specular=0.2, color_specular=(1, 1, 1),
                      device=None):
    """One directional light record [1|B,12] for F.light_set / rasterize(..., lights=...): {diffuse intensity * colour
    (3), specular intensity * colour (3), direction towards the light (3, not normalised), 0, 0 (directional), 0}.
    Built with torch ops, so tensor-valued arguments (intensities scalar or [B], colours and direction [3] or [B,3])
    receive gradients.  `device`: where plain numbers go (default: the device of the first tensor argument, else the
    CPU)."""
    return _light_record(0.0, direction, intensity, color, intensity_specular, color_specular, 0.0, device)


def point_light(position, intensity=0.5, color=(1, 1, 1), intensity_specular=0.2, color_specular=(1, 1, 1), falloff=0.0,
                device=None):
    """One point light record [1|B,12]: as F.directional_light with the light's position (in the frame of the shading
    positions and the eye) in slots 6-8, the falloff f in slot 9 (attenuation 1 / (1 + f r^2) at distance r; 0 = none,
    as PyTorch3D's PointLights) and kind 1.  The position and the falloff may be tensors that receive gradients."""
    return _light_record(1.0, position, intensity, color, intensity_specular, color_specular, falloff, device)


def light_set(*records):
    """Stack light records ([12], [1|B,12] from F.directional_light / F.point_light) into the [1|B,NL,12] set of
    rasterize(..., lights=...), NL <= 8, in order; records of one item serve every item.  Differentiable."""
    if not records:
        raise ValueError("light_set needs at least one light record")
    if len(records) > 8:
        raise ValueError("a light set holds at most 8 lights, got %d" % len(records))
    recs = [r.reshape(1, 12) if r.dim() == 1 else r for r in records]
    if any(r.dim() != 2 or r.shape[1] != 12 for r in recs):
        raise ValueError("light records must have shape [12] or [batch size, 12]")
    n = max(r.shape[0] for r in recs)
    if any(r.shape[0] not in (1, n) for r in recs):
        raise ValueError("light records must hold one entry or one per batch item")
    return torch.stack([r.expand(n, -1) for r in recs], dim=1)


# second-order real SH constants of include/nr_b200.h (nr_b200_sh_args): C0 = 1/(2 sqrt(pi)), C1 = sqrt(3/(4 pi)),
# C2 = sqrt(15/(4 pi)), C3 = sqrt(5/(16 pi)), C4 = sqrt(15/(16 pi))
SH_C = (0.5 / math.sqrt(math.pi), math.sqrt(3.0 / (4.0 * math.pi)), math.sqrt(15.0 / (4.0 * math.pi)),
        math.sqrt(5.0 / (16.0 * math.pi)), math.sqrt(15.0 / (16.0 * math.pi)))


def _sh_basis_torch(d):
    """The 9 real SH basis functions of include/nr_b200.h at directions d [...,3] -> [...,9] (d used as given)."""
    x, y, z = d.unbind(-1)
    c0, c1, c2, c3, c4 = SH_C
    return torch.stack([torch.full_like(x, c0), c1 * y, c1 * z, c1 * x, c2 * x * y, c2 * y * z, c3 * (3 * z * z - 1),
                        c2 * x * z, c4 * (x * x - y * y)], dim=-1)


def sh_from_environment_map(envmap):
    """Irradiance-ready second-order SH coefficients [1|B,9,3] (rasterize(..., environment_sh=...),
    Renderer.environment_sh) from a lat-long HDR environment map [He,We,3] / [1|B,He,We,3] of radiance.

    Convention: row 0 is the top.  Texel (i, j) is the direction omega = (sin t sin p, cos t, sin t cos p) with
    t_i = pi (i + 1/2) / He measured from +y and p_j = 2 pi (j + 1/2) / We, in the frame of the shading normals, and
    covers the solid angle dOmega_i = sin t_i (pi / He) (2 pi / We) (the midpoint rule).  Then
        S[k][c] = a_l sum_{i,j} env[i,j,c] Y_k(omega_ij) dOmega_i,   a_0 = 1, a_1 = 2/3, a_2 = 1/4
    (a_l = A_l / pi, the clamped-cosine convolution of Ramamoorthi & Hanrahan 2001, divided by pi), so a uniform map of
    radiance r gives S = (r / C0, 0, ...) and renders a white albedo as r.  Pure torch in the map's dtype and device,
    differentiable with respect to the map; rotate the map (or the geometry) to rotate the environment."""
    if not isinstance(envmap, torch.Tensor) or not envmap.is_floating_point():
        raise TypeError("envmap must be a floating point torch.Tensor")
    env = envmap[None] if envmap.dim() == 3 else envmap
    if env.dim() != 4 or env.shape[-1] != 3 or env.shape[1] < 1 or env.shape[2] < 1:
        raise ValueError("envmap must have shape [He, We, 3] or [batch size, He, We, 3], got %s" % (tuple(envmap.shape),))
    He, We = int(env.shape[1]), int(env.shape[2])
    kw = dict(dtype=env.dtype, device=env.device)
    t = math.pi * (torch.arange(He, **kw) + 0.5) / He
    p = 2.0 * math.pi * (torch.arange(We, **kw) + 0.5) / We
    st = torch.sin(t)[:, None]
    omega = torch.stack([st * torch.sin(p)[None, :], torch.cos(t)[:, None].expand(He, We), st * torch.cos(p)[None, :]], -1)
    dw = torch.sin(t) * (math.pi / He) * (2.0 * math.pi / We)  # [He]
    Y = _sh_basis_torch(omega) * dw[:, None, None]  # [He,We,9]
    a = torch.tensor([1.0] + [2.0 / 3.0] * 3 + [0.25] * 5, **kw)
    return torch.einsum('bhwc,hwk->bkc', env, Y) * a[None, :, None]


def vertex_tangents(vertices, faces, face_uvs, vertex_normals):
    """Per-vertex tangents [B,Nv,4] = (T, w) for a tangent-space normal map (F.corner_tangents, then
    rasterize(..., normal_map=, corner_tangents=), Renderer.normal_map).  vertices / vertex_normals [B,Nv,3], faces [F,3] /
    [1|B,F,3] (the original faces, not the fill_back-doubled set), face_uvs [F,3,2] / [1|B,F,3,2] (OBJ convention, v up).

    Per face, with e1 = v1 - v0, e2 = v2 - v0 and (du_k, dv_k) = uv_k - uv_0: s = sign(du1 dv2 - du2 dv1) (a face with
    s = 0 is skipped), T_f = s (e1 dv2 - e2 dv1) and B_f = s (e2 du1 - e1 du2).  The sums over a vertex's corners are
    orthogonalised against n_v and normalised, T_v = t / (|t| + 1e-5) with t = T - (n_v . T) n_v, and w_v = -1 where
    (n_v x T_v) . sum B_f < 0, else 1 (the map's +y then runs along +v).  An unreferenced vertex gets (0, 0, 0, 1).
    Tangents are summed by vertex, so a UV seam shares one tangent across it.  Pure torch, differentiable with
    respect to the vertices, the UVs and the normals (not through w)."""
    bs, nv = vertices.shape[:2]
    faces = faces[None] if faces.dim() == 2 else faces
    uvs = face_uvs[None] if face_uvs.dim() == 3 else face_uvs
    v, ok = _gather_vertices(vertices, faces)  # [B,F,3,3]
    uvs = uvs.to(v.dtype).expand(bs, -1, -1, -1)
    e1, e2 = v[:, :, 1] - v[:, :, 0], v[:, :, 2] - v[:, :, 0]
    d1, d2 = uvs[:, :, 1] - uvs[:, :, 0], uvs[:, :, 2] - uvs[:, :, 0]
    du1, dv1, du2, dv2 = d1[..., :1], d1[..., 1:], d2[..., :1], d2[..., 1:]
    s = torch.sign(du1 * dv2 - du2 * dv1) * ok.all(dim=2)[..., None].to(v.dtype)
    tf = s * (e1 * dv2 - e2 * dv1)
    bf = s * (e2 * du1 - e1 * du2)
    idx = faces.long().expand(bs, -1, -1)
    corner_ok = ((idx >= 0) & (idx < nv))[..., None].to(v.dtype)
    target = (idx.clamp(0, nv - 1) + (torch.arange(bs, device=vertices.device) * nv)[:, None, None]).reshape(-1)
    zeros = torch.zeros((bs * nv, 3), dtype=v.dtype, device=v.device)
    t = zeros.index_add(0, target, (tf[:, :, None, :] * corner_ok).reshape(-1, 3)).reshape(bs, nv, 3)
    b = zeros.index_add(0, target, (bf[:, :, None, :] * corner_ok).reshape(-1, 3)).reshape(bs, nv, 3)
    n = vertex_normals.to(v.dtype).expand(bs, nv, 3)
    t = t - (n * t).sum(dim=2, keepdim=True) * n
    t = t / (torch.linalg.vector_norm(t, dim=2, keepdim=True) + 1e-5)
    w = torch.where((torch.linalg.cross(n, t, dim=2) * b).sum(dim=2, keepdim=True) < 0, -1.0, 1.0).to(v.dtype)
    return torch.cat((t, w), dim=2)


def corner_tangents(vertex_tangents, faces, fill_back=False):
    """Per-corner tangents [B,F,3,4] for rasterize(..., corner_tangents=...): corner k of face f holds (T, w) of vertex
    faces[f,k] from `vertex_tangents` [B,Nv,4] (F.vertex_tangents).  `faces` [F,3] / [1|B,F,3] is the index set the
    rasterizer receives, as for F.corner_shading; with fill_back=True faces [F/2, F) are the reversed copies and get
    (-T, -w), so that their mapped normal is exactly the negated one of the original face.  An index outside [0, Nv)
    gives zeros.  Pure torch, differentiable with respect to the tangents."""
    assert vertex_tangents.dim() == 3 and vertex_tangents.shape[2] == 4
    faces = faces[None] if faces.dim() == 2 else faces
    nf = faces.shape[1]
    if fill_back and nf % 2:
        raise ValueError("fill_back needs an even number of faces (front faces, then their reversed copies)")
    bs, nv = vertex_tangents.shape[:2]
    idx = faces.long().expand(bs, -1, -1)
    ok = ((idx >= 0) & (idx < nv))[..., None].to(vertex_tangents.dtype)
    flat = idx.clamp(0, nv - 1) + (torch.arange(bs, device=vertex_tangents.device) * nv)[:, None, None]
    out = vertex_tangents.reshape(bs * nv, 4)[flat] * ok
    if fill_back:
        sign = torch.ones(nf, dtype=out.dtype, device=out.device)
        sign[nf // 2:] = -1
        out = out * sign[None, :, None, None]
    return out


def decode_normal_map(image, green_down=False):
    """A normal-map image of [0,1] colours [...,3] -> the decoded tangent-space vectors 2 image - 1 that
    rasterize(..., normal_map=...) and Renderer.normal_map take.  green_down=True negates y, for maps authored with +y
    along -v (the DirectX convention).  Differentiable; not renormalised (the shading normalises the mapped normal)."""
    m = 2.0 * image - 1.0
    if green_down:
        m = m * torch.tensor([1.0, -1.0, 1.0], dtype=m.dtype, device=m.device)
    return m


def specular_map(color, shininess):
    """A specular colour [...,H,W,3] and a shininess [...,H,W] (or a scalar / any tensor that broadcasts to [...,H,W])
    -> the [...,H,W,4] map (ks_r, ks_g, ks_b, shininess) that rasterize(..., specular_map=...) and Renderer.specular_map
    take.  Differentiable in both; the shininess is not clamped, so a fit may want to pass exp(log_shininess)."""
    if not isinstance(color, torch.Tensor) or color.dim() < 3 or color.shape[-1] != 3:
        raise ValueError("color must have shape [..., height, width, 3], got %s"
                         % (tuple(color.shape) if isinstance(color, torch.Tensor) else type(color).__name__,))
    sig = torch.as_tensor(shininess, dtype=color.dtype, device=color.device)
    try:
        sig = sig.expand(color.shape[:-1])
    except RuntimeError:
        raise ValueError("shininess must broadcast to %s, got %s" % (tuple(color.shape[:-1]), tuple(sig.shape))) from None
    return torch.cat((color, sig[..., None]), dim=-1)


def interpolate_face_attributes(pix_to_face, bary_coords, face_attributes):
    """Per-corner attributes interpolated at soft fragments (rasterize_soft_fragments): out[b,y,x,k] =
    sum_m bary_coords[b,y,x,k,m] face_attributes[(b,) pix_to_face[b,y,x,k], m], [B,H,W,K,C], zeros in empty slots
    (pix_to_face < 0).  face_attributes [F,3,C] (one set for every item) or [B,F,3,C] / [1,F,3,C].  With the fragments'
    bary_coords this is A_j of rasterize_soft_attributes for every selected face; blend the slots in torch (e.g.
    w = sigmoid(dists / sigma) times a depth softmax), or hand them to rasterize.blend_soft_fragments, which blends
    them by SoftRas's depth softmax in CUDA.  Torch glue, differentiable in bary_coords and face_attributes: one gather
    per corner and a multiply-add, without a [..., 3, C] intermediate.  rasterize.interpolate_soft_fragments computes
    the same in CUDA (per corner or per vertex), and is the one to use on the GPU; this one serves any dtype and device,
    float64 included."""
    if not isinstance(pix_to_face, torch.Tensor) or not isinstance(bary_coords, torch.Tensor) \
            or not isinstance(face_attributes, torch.Tensor):
        raise TypeError("pix_to_face, bary_coords and face_attributes must be torch.Tensors")
    if pix_to_face.dtype.is_floating_point or pix_to_face.dim() != 4:
        raise ValueError("pix_to_face must be an integer tensor [B,H,W,K], got %s %s"
                         % (pix_to_face.dtype, tuple(pix_to_face.shape)))
    if tuple(bary_coords.shape) != tuple(pix_to_face.shape) + (3,):
        raise ValueError("bary_coords must have shape %s, got %s"
                         % (tuple(pix_to_face.shape) + (3,), tuple(bary_coords.shape)))
    B = pix_to_face.shape[0]
    fa = face_attributes
    if fa.dim() == 4 and fa.shape[0] == 1:
        fa = fa[0]
    if not (fa.dim() == 3 or (fa.dim() == 4 and fa.shape[0] == B)) or fa.shape[-2] != 3:
        raise ValueError("face_attributes must have shape [F,3,C] or [B,F,3,C], got %s" % (tuple(face_attributes.shape),))
    F_, C = fa.shape[-3], fa.shape[-1]
    valid = pix_to_face >= 0
    ids = torch.where(valid, pix_to_face, torch.zeros_like(pix_to_face)).long()
    if fa.dim() == 4:
        ids = ids + (torch.arange(B, device=ids.device) * F_).view(B, 1, 1, 1)
        fa = fa.reshape(B * F_, 3, C)
    ids = ids.reshape(-1)
    out = None
    for m in range(3):
        a = fa[:, m].index_select(0, ids).reshape(*pix_to_face.shape, C)
        w = bary_coords[..., m:m + 1].to(a.dtype)
        out = a * w if out is None else torch.addcmul(out, a, w)
    return torch.where(valid[..., None], out, torch.zeros((), dtype=out.dtype, device=out.device))
