"""Host-side mirror of the reference's rasterizer interface (neural_renderer/rasterize.py) on top of the C ABI.

Same names, argument order, defaults and error conditions as the reference:

  rasterize_rgbad        rasterize.py:900-977
  rasterize              rasterize.py:980-1008
  rasterize_silhouettes  rasterize.py:1011-1034
  rasterize_depth        rasterize.py:1037-1060
  Rasterize              rasterize.py:19-897   (function object; returns un-flipped NHWC maps like forward_gpu)
  use_unsafe_rasterizer  rasterize.py:1063-1065

Tensors are CUDA `torch.Tensor`s instead of chainer Variables / cupy arrays; PyTorch only provides device memory,
the current stream and autograd bookkeeping -- all arithmetic happens in libnr_b200.so (hand-written sm_90a CUDA).
There is no CPU path (the reference raises NotImplementedError for CPU arrays as well, rasterize.py:893-897).
"""
from __future__ import annotations

import collections
import ctypes
import math
import os

import torch

from . import _lib

DEFAULT_IMAGE_SIZE = 256
DEFAULT_ANTI_ALIASING = True
DEFAULT_NEAR = 0.1
DEFAULT_FAR = 100
DEFAULT_EPS = 1e-4
DEFAULT_BACKGROUND_COLOR = (0, 0, 0)
USE_UNSAFE_IMPLEMENTATION = False

# rasterize.py:389 fetches the vertex depths for texture sampling from batch item 0.  Reference-exact by default;
# NEURAL_RENDERER_B200_FIX_TEXTURE_DEPTH=1 (or set_reference_exact(False)) samples with each item's own depths.
_REFERENCE_EXACT = not int(os.environ.get("NEURAL_RENDERER_B200_FIX_TEXTURE_DEPTH", "0"))
# NR_FWD_STAGE_TEXTURES (texture cubes staged in shared memory with cp.async.bulk): same pixels, measured slower than the
# direct gather on H100 -- kept selectable for measurements and tests, off by default.
_STAGE_TEXTURES = False


def set_stage_textures(flag):
    global _STAGE_TEXTURES
    _STAGE_TEXTURES = bool(flag)


def set_reference_exact(flag):
    global _REFERENCE_EXACT
    _REFERENCE_EXACT = bool(flag)


def use_unsafe_rasterizer(flag):
    """Accepted for interface compatibility (rasterize.py:1063).  The reference's 'unsafe' scanline/spin-lock
    variant is an alternative implementation of the same maps with arrival-order tie breaks; this package has a
    single deterministic forward path, so the flag changes nothing."""
    global USE_UNSAFE_IMPLEMENTATION
    USE_UNSAFE_IMPLEMENTATION = bool(flag)


def _ptr(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def _check_inputs(faces, textures, return_rgb, face_light=None, textures_fill_back=False, vertices=None, face_uvs=None,
                  corner_light=None, corner_shading=None, shading_params=None, lights=None, environment_sh=None,
                  normal_map=None, corner_tangents=None, specular_map=None):
    # rasterize.py:66-90 (chainer type_check) -> TypeError / ValueError with the same conditions
    if not isinstance(faces, torch.Tensor):
        raise TypeError("faces must be a torch.Tensor")
    if vertices is not None:
        # indexed geometry (vertices_to_faces.py:10-14 asserts): vertices [B,Nv,3] float, faces [B,F,3] / [1,F,3] / [F,3] int
        if not isinstance(vertices, torch.Tensor) or not vertices.is_floating_point():
            raise TypeError("vertices must be a floating point torch.Tensor")
        if vertices.dim() != 3 or vertices.shape[2] != 3:
            raise ValueError("vertices must have shape [batch size, num vertices, 3], got %s" % (tuple(vertices.shape),))
        if faces.is_floating_point():
            raise TypeError("with `vertices`, faces must hold integer vertex indices")
        if not ((faces.dim() == 2 and faces.shape[1] == 3)
                or (faces.dim() == 3 and faces.shape[2] == 3 and faces.shape[0] in (1, vertices.shape[0]))):
            raise ValueError("with `vertices`, faces must have shape [batch size, num faces, 3] or [num faces, 3], got %s"
                             % (tuple(faces.shape),))
        if not vertices.is_cuda or not faces.is_cuda:
            raise NotImplementedError("neural_renderer_b200 has no CPU implementation (inputs must be CUDA tensors)")
        batch_size, num_faces = vertices.shape[0], faces.shape[-2]
    else:
        if not faces.is_floating_point():
            raise TypeError("faces must be floating point")
        if faces.dim() != 4 or faces.shape[2] != 3 or faces.shape[3] != 3:
            raise ValueError("faces must have shape [batch size, num faces, 3, 3], got %s" % (tuple(faces.shape),))
        batch_size, num_faces = faces.shape[0], faces.shape[1]
    if return_rgb:
        if not isinstance(textures, torch.Tensor):
            raise TypeError("textures are required to draw RGB")
        if not textures.is_floating_point():
            raise TypeError("textures must be floating point")
        num_cubes = num_faces // 2 if textures_fill_back else num_faces
        if textures_fill_back and num_faces % 2:
            raise ValueError("textures_fill_back needs an even number of faces (front faces, then their reversed copies)")
    if return_rgb and face_uvs is not None:
        _check_uv_inputs(textures, face_uvs, batch_size, num_cubes)
    elif return_rgb:
        # batch size 1 with a larger geometry batch = ONE set of cubes shared by every item (a mesh seen from B viewpoints)
        if (textures.dim() != 6 or textures.shape[2] < 2 or textures.shape[2] != textures.shape[3]
                or textures.shape[3] != textures.shape[4] or textures.shape[5] != 3
                or textures.shape[0] not in (1, batch_size) or textures.shape[1] != num_cubes):
            raise ValueError("textures must have shape [batch size, num faces, ts, ts, ts, 3] with ts >= 2 and match "
                             "faces, got %s" % (tuple(textures.shape),))
    if lights is not None:
        _check_lights(lights, corner_shading, batch_size)
    if environment_sh is not None:
        _check_environment_sh(environment_sh, corner_shading, return_rgb, batch_size)
    if normal_map is not None or corner_tangents is not None:
        _check_normal_map(normal_map, corner_tangents, corner_shading, face_uvs, return_rgb, batch_size, num_faces)
    if specular_map is not None:
        _check_specular_map(specular_map, corner_shading, face_uvs, return_rgb, batch_size)
    if corner_shading is not None or shading_params is not None:
        _check_phong_inputs(corner_shading, shading_params, face_light, corner_light, return_rgb, batch_size, num_faces)
    if return_rgb and face_light is not None:
        if not isinstance(face_light, torch.Tensor) or tuple(face_light.shape) != (batch_size, num_faces, 3):
            raise ValueError("face_light must have shape [batch size, num faces, 3]")
        if not face_light.is_cuda:
            raise NotImplementedError("neural_renderer_b200 has no CPU implementation (inputs must be CUDA tensors)")
    if corner_light is not None:
        if face_light is not None:
            raise ValueError("face_light and corner_light are exclusive: give one light factor")
        if not return_rgb:
            raise ValueError("corner_light lights the RGB image: it needs return_rgb")
        if not isinstance(corner_light, torch.Tensor) or not corner_light.is_floating_point():
            raise TypeError("corner_light must be a floating point torch.Tensor")
        if tuple(corner_light.shape) != (batch_size, num_faces, 3, 3):
            raise ValueError("corner_light must have shape [batch size, num faces, 3, 3], got %s" % (tuple(corner_light.shape),))
        if not corner_light.is_cuda:
            raise NotImplementedError("neural_renderer_b200 has no CPU implementation (inputs must be CUDA tensors)")
    if not faces.is_cuda or (return_rgb and not textures.is_cuda) or (return_rgb and face_uvs is not None and not face_uvs.is_cuda):
        raise NotImplementedError("neural_renderer_b200 has no CPU implementation (inputs must be CUDA tensors)")


def _check_phong_inputs(corner_shading, shading_params, face_light, corner_light, return_rgb, batch_size, num_faces):
    # Phong shading: corner_shading [F,3,6] / [1|B,F,3,6] and shading_params [16] / [1|B,16], always together
    if corner_shading is None or shading_params is None:
        raise ValueError("corner_shading and shading_params must be given together (Phong shading)")
    if face_light is not None or corner_light is not None:
        raise ValueError("Phong shading (corner_shading / shading_params) is exclusive with face_light and corner_light")
    if not return_rgb:
        raise ValueError("Phong shading lights the RGB image: it needs return_rgb")
    for name, t in (("corner_shading", corner_shading), ("shading_params", shading_params)):
        if not isinstance(t, torch.Tensor) or not t.is_floating_point():
            raise TypeError("%s must be a floating point torch.Tensor" % name)
    cs, sp = corner_shading, shading_params
    if not ((cs.dim() == 3 or (cs.dim() == 4 and cs.shape[0] in (1, batch_size))) and tuple(cs.shape[-3:]) == (num_faces, 3, 6)):
        raise ValueError("corner_shading must have shape [num faces, 3, 6] or [batch size, num faces, 3, 6] (num faces counts "
                         "fill_back copies), got %s" % (tuple(cs.shape),))
    if not ((sp.dim() == 1 or (sp.dim() == 2 and sp.shape[0] in (1, batch_size))) and sp.shape[-1] == 16):
        raise ValueError("shading_params must have shape [16] or [batch size, 16], got %s" % (tuple(sp.shape),))
    if not cs.is_cuda or not sp.is_cuda:
        raise NotImplementedError("neural_renderer_b200 has no CPU implementation (inputs must be CUDA tensors)")


def _check_lights(lights, corner_shading, batch_size):
    # light set [NL,12] / [1|B,NL,12], NL <= 8, on top of Phong shading's light
    if corner_shading is None:
        raise ValueError("lights needs Phong shading (corner_shading / shading_params)")
    if not isinstance(lights, torch.Tensor) or not lights.is_floating_point():
        raise TypeError("lights must be a floating point torch.Tensor")
    if not ((lights.dim() == 2 or (lights.dim() == 3 and lights.shape[0] in (1, batch_size))) and lights.shape[-1] == 12
            and lights.shape[-2] <= 8):
        raise ValueError("lights must have shape [num lights, 12] or [batch size, num lights, 12] with at most 8 lights, "
                         "got %s" % (tuple(lights.shape),))
    if not lights.is_cuda:
        raise NotImplementedError("neural_renderer_b200 has no CPU implementation (inputs must be CUDA tensors)")


def _check_environment_sh(sh, corner_shading, return_rgb, batch_size):
    # irradiance-ready SH coefficients [9,3] / [1|B,9,3] on top of Phong shading's lights
    if corner_shading is None:
        raise ValueError("environment_sh needs Phong shading (corner_shading / shading_params)")
    if not return_rgb:
        raise ValueError("environment_sh lights the RGB image: it needs return_rgb")
    if not isinstance(sh, torch.Tensor) or not sh.is_floating_point():
        raise TypeError("environment_sh must be a floating point torch.Tensor")
    if not ((sh.dim() == 2 or (sh.dim() == 3 and sh.shape[0] in (1, batch_size))) and tuple(sh.shape[-2:]) == (9, 3)):
        raise ValueError("environment_sh must have shape [9, 3] or [batch size, 9, 3], got %s" % (tuple(sh.shape),))
    if not sh.is_cuda:
        raise NotImplementedError("neural_renderer_b200 has no CPU implementation (inputs must be CUDA tensors)")


def _check_normal_map(normal_map, corner_tangents, corner_shading, face_uvs, return_rgb, batch_size, num_faces):
    # decoded tangent-space normal map [Hm,Wm,3] / [1|B,Hm,Wm,3] and corner tangents [F,3,4] / [1|B,F,3,4], always together,
    # on top of Phong shading of a texture image
    if normal_map is None or corner_tangents is None:
        raise ValueError("normal_map and corner_tangents go together: give both")
    if corner_shading is None:
        raise ValueError("normal_map needs Phong shading (corner_shading / shading_params)")
    if not return_rgb:
        raise ValueError("normal_map shades the RGB image: it needs return_rgb")
    if face_uvs is None:
        raise ValueError("normal_map is addressed by the UVs: it needs a texture image with face_uvs")
    for name, t in (("normal_map", normal_map), ("corner_tangents", corner_tangents)):
        if not isinstance(t, torch.Tensor) or not t.is_floating_point():
            raise TypeError("%s must be a floating point torch.Tensor" % name)
    if not ((normal_map.dim() == 3 or (normal_map.dim() == 4 and normal_map.shape[0] in (1, batch_size)))
            and normal_map.shape[-1] == 3 and normal_map.shape[-2] >= 1 and normal_map.shape[-3] >= 1):
        raise ValueError("normal_map must have shape [height, width, 3] or [batch size, height, width, 3], got %s"
                         % (tuple(normal_map.shape),))
    if not ((corner_tangents.dim() == 3 or (corner_tangents.dim() == 4 and corner_tangents.shape[0] in (1, batch_size)))
            and tuple(corner_tangents.shape[-3:]) == (num_faces, 3, 4)):
        raise ValueError("corner_tangents must have shape [num faces, 3, 4] or [batch size, num faces, 3, 4] with num faces "
                         "= %d (the drawn faces, fill_back copies included), got %s" % (num_faces, tuple(corner_tangents.shape)))
    if not normal_map.is_cuda or not corner_tangents.is_cuda:
        raise NotImplementedError("neural_renderer_b200 has no CPU implementation (inputs must be CUDA tensors)")


def _check_specular_map(specular_map, corner_shading, face_uvs, return_rgb, batch_size):
    # specular map [Hq,Wq,4] / [1|B,Hq,Wq,4] of (ks_r, ks_g, ks_b, shininess) on top of Phong shading of a texture image
    if corner_shading is None:
        raise ValueError("specular_map needs Phong shading (corner_shading / shading_params)")
    if not return_rgb:
        raise ValueError("specular_map shades the RGB image: it needs return_rgb")
    if face_uvs is None:
        raise ValueError("specular_map is addressed by the UVs: it needs a texture image with face_uvs")
    if not isinstance(specular_map, torch.Tensor) or not specular_map.is_floating_point():
        raise TypeError("specular_map must be a floating point torch.Tensor")
    sm = specular_map
    if not ((sm.dim() == 3 or (sm.dim() == 4 and sm.shape[0] in (1, batch_size)))
            and sm.shape[-1] == 4 and sm.shape[-2] >= 1 and sm.shape[-3] >= 1):
        raise ValueError("specular_map must have shape [height, width, 4] or [batch size, height, width, 4], got %s"
                         % (tuple(sm.shape),))
    if not sm.is_cuda:
        raise NotImplementedError("neural_renderer_b200 has no CPU implementation (inputs must be CUDA tensors)")


def _check_uv_inputs(image, face_uvs, batch_size, num_uv_faces):
    # texture image [Ht,Wt,3] / [1|B,Ht,Wt,3] and per-corner UVs [F,3,2] / [1|B,F,3,2] (F/2 faces with textures_fill_back)
    if not isinstance(face_uvs, torch.Tensor) or not face_uvs.is_floating_point():
        raise TypeError("face_uvs must be a floating point torch.Tensor")
    if not ((face_uvs.dim() == 3 or (face_uvs.dim() == 4 and face_uvs.shape[0] in (1, batch_size)))
            and tuple(face_uvs.shape[-3:]) == (num_uv_faces, 3, 2)):
        raise ValueError("face_uvs must have shape [num faces, 3, 2] or [batch size, num faces, 3, 2] with num faces = %d "
                         "(half the faces with textures_fill_back), got %s" % (num_uv_faces, tuple(face_uvs.shape)))
    if not isinstance(image, torch.Tensor):
        raise TypeError("with face_uvs, textures must be the texture image (a torch.Tensor)")
    if not image.is_floating_point():
        raise TypeError("the texture image must be floating point")
    if not ((image.dim() == 3 or (image.dim() == 4 and image.shape[0] in (1, batch_size)))
            and image.shape[-1] == 3 and image.shape[-2] >= 1 and image.shape[-3] >= 1):
        raise ValueError("with face_uvs, textures must be an image of shape [height, width, 3] or [batch size, height, "
                         "width, 3], got %s" % (tuple(image.shape),))


# Optional hook between the two halves of the backward pass (neural_renderer_b200.distributed.overlap_texture_allreduce):
# called as hook(grad_textures) right after the texture-gradient kernels are enqueued and BEFORE the edge scan is;
# returns an object whose .wait() is called once the whole pass is enqueued.
_TEXTURE_GRAD_HOOK = None


def set_texture_grad_hook(hook):
    global _TEXTURE_GRAD_HOOK
    prev = _TEXTURE_GRAD_HOOK
    _TEXTURE_GRAD_HOOK = hook
    return prev


class _Config:
    __slots__ = ("S", "aa", "near", "far", "eps", "bg", "bg_batch", "flags", "reference_exact", "mip_hw", "interior")


def _make_config(image_size, anti_aliasing, near, far, eps, background_color, return_rgb, return_alpha, return_depth,
                 device, batch_size, reference_exact=None):
    if not any((return_rgb, return_alpha, return_depth)):
        raise Exception("nothing to draw")  # rasterize.py:25-27 raises a bare Exception
    cfg = _Config()
    cfg.aa = bool(anti_aliasing)
    cfg.S = int(image_size) * 2 if cfg.aa else int(image_size)
    cfg.near, cfg.far, cfg.eps = float(near), float(far), float(eps)
    cfg.mip_hw = None  # (Ht, Wt) of level 0 when `textures` is a packed mip pyramid (NR_TEX_MIPMAP)
    cfg.interior = False  # NR_GRAD_INTERIOR on the backward call (interior_gradient=True)
    flags = 0
    if return_rgb:
        flags |= _lib.NR_RETURN_RGB
    if return_alpha:
        flags |= _lib.NR_RETURN_ALPHA
    if return_depth:
        flags |= _lib.NR_RETURN_DEPTH
    if cfg.aa:
        flags |= _lib.NR_ANTI_ALIASING
    cfg.reference_exact = _REFERENCE_EXACT if reference_exact is None else bool(reference_exact)
    if cfg.reference_exact:
        flags |= _lib.NR_TEX_Z_BATCH0
    cfg.bg = (0.0, 0.0, 0.0)
    cfg.bg_batch = None
    if return_rgb:
        bg = background_color
        if isinstance(bg, torch.Tensor):
            bg = bg.detach().to(dtype=torch.float32)
        else:
            bg = torch.as_tensor(bg, dtype=torch.float32)
        if bg.dim() == 1 and bg.numel() == 3:
            cfg.bg = tuple(float(v) for v in bg.tolist())
        elif bg.dim() == 2 and bg.shape[1] == 3 and bg.shape[0] == batch_size:  # rasterize.py:464-465
            cfg.bg_batch = bg.to(device).contiguous()
            flags |= _lib.NR_BG_PER_BATCH
        else:
            raise ValueError("background_color must have shape (3,) or (batch size, 3)")
    cfg.flags = flags
    return cfg


def _stream_ptr(device):
    return ctypes.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def _index_set(indices):
    """integer faces [F,3] / [1|B,F,3] as int32; an expanded [F,3] index set (Mesh.get_batch) stays one shared set and is
    not materialised"""
    if indices.dim() == 3 and indices.shape[0] > 1 and indices.stride(0) == 0:
        indices = indices[:1]
    return indices.to(torch.int32).contiguous()


def _geometry(faces, vertices):
    """(geom, indices) of a call: vertices as float32 with faces as its index set, or faces as float32 and None"""
    if vertices is None:
        return (faces if faces.dtype == torch.float32 else faces.float()), None
    return (vertices if vertices.dtype == torch.float32 else vertices.float()), _index_set(faces)


def _set_geometry(a, geom_c, indices):
    """the geometry fields of an args struct (faces, or vertices / face_indices / num_vertices, and num_faces); returns
    its geometry flags (a 2-D index set is shared, as is a batch of 1 with a larger geometry batch)"""
    if indices is None:
        a.faces, a.num_faces = _ptr(geom_c), geom_c.shape[1]
        return 0
    a.vertices, a.face_indices, a.num_vertices = _ptr(geom_c), _ptr(indices), geom_c.shape[1]
    a.num_faces = indices.shape[-2]
    if indices.dim() == 2 or (indices.shape[0] == 1 and geom_c.shape[0] > 1):
        return _lib.NR_FACES_INDEXED | _lib.NR_INDICES_SHARED
    return _lib.NR_FACES_INDEXED


def _set_geometry_grad(a, indices, grad_geom):
    """the geometry gradient field of an args struct: grad_vertices when indexed, else grad_faces"""
    if indices is not None:
        a.grad_vertices = _ptr(grad_geom)
    else:
        a.grad_faces = _ptr(grad_geom)


class _RasterizeFunction(torch.autograd.Function):
    """autograd node of the hot path: forward = nr_b200_forward, backward = nr_b200_backward.

    `geom` is faces [B,F,3,3], or -- indexed geometry, `indices` given -- vertices [B,Nv,3] (the vertices_to_faces
    gather and its scatter-add backward happen inside the kernels).  Outputs are the API images (planar, image
    orientation, pooled when anti-aliasing) plus the raster-resolution maps (returned non-differentiable so tests /
    the `Rasterize` object can look at them)."""

    @staticmethod
    def forward(ctx, geom, textures, face_light, cfg, indices, face_uvs, corner_light, *phong):
        lib = _lib.load()
        dev = geom.device
        geom_c = geom.detach().contiguous()
        tex_c = textures.detach().contiguous() if textures is not None else None
        light_c = face_light.detach().to(torch.float32).contiguous() if face_light is not None else None
        corner_c = corner_light.detach().to(torch.float32).contiguous() if corner_light is not None else None
        # Phong shading: the inputs of _PHONG_DIMS with their batch axes (1 for a set shared by every item), or None
        phong_c = [t.detach().to(torch.float32).contiguous() if t is not None else None for t in phong]
        if phong_c[6] is not None and phong_c[6].data_ptr() % 16:
            phong_c[6] = phong_c[6].clone()  # specular_map: the kernels read a texel as one aligned 16-byte vector
        flags = cfg.flags
        if indices is not None:
            B, Nv = geom_c.shape[:2]
            F = indices.shape[-2]
            flags |= _lib.NR_FACES_INDEXED
            if indices.dim() == 2 or (indices.shape[0] == 1 and B > 1):
                flags |= _lib.NR_INDICES_SHARED
        else:
            B, F = geom_c.shape[:2]
            Nv = 0
        if tex_c is not None and tex_c.shape[0] == 1 and B > 1:
            flags |= _lib.NR_TEX_SHARED
        S = cfg.S
        ts = int(tex_c.shape[2]) if tex_c is not None else 0
        uv_c = None
        if face_uvs is not None:  # texture image [Bt,Ht,Wt,3] sampled through face_uvs (NR_TEX_UV)
            uv_c = face_uvs.detach().contiguous()
            flags |= _lib.NR_TEX_UV
            if uv_c.shape[0] == 1 and B > 1:
                flags |= _lib.NR_UV_SHARED
            ts = 0
        tex_hw = (int(tex_c.shape[1]), int(tex_c.shape[2])) if uv_c is not None else (0, 0)
        if uv_c is not None and cfg.mip_hw is not None:
            tex_hw = cfg.mip_hw  # `textures` is the packed pyramid [Bt,P,3] of an Ht x Wt image
        want_rgb = bool(flags & _lib.NR_RETURN_RGB)
        want_alpha = bool(flags & _lib.NR_RETURN_ALPHA)
        want_depth = bool(flags & _lib.NR_RETURN_DEPTH)
        with torch.cuda.device(dev):
            fim = torch.empty((B, S, S), dtype=torch.int32, device=dev)
            wmap = torch.empty((B, 3, S, S), dtype=torch.float32, device=dev)
            dmap = torch.empty((B, S, S), dtype=torch.float32, device=dev)
            rgb_map = torch.empty((B, 3, S, S), dtype=torch.float32, device=dev) if want_rgb else None
            alpha_map = torch.empty((B, S, S), dtype=torch.float32, device=dev) if want_alpha else None
            out_rgb = out_alpha = out_depth = None
            if cfg.aa:
                H = S // 2
                if want_rgb:
                    out_rgb = torch.empty((B, 3, H, H), dtype=torch.float32, device=dev)
                if want_alpha:
                    out_alpha = torch.empty((B, H, H), dtype=torch.float32, device=dev)
                if want_depth:
                    out_depth = torch.empty((B, H, H), dtype=torch.float32, device=dev)
            ws_bytes = lib.nr_b200_forward_workspace_bytes(B, F, S, ts, flags)
            ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=dev)
            a = _lib.ForwardArgs()
            a.struct_size = ctypes.sizeof(_lib.ForwardArgs)
            a.flags = flags
            a.batch_size, a.num_faces, a.raster_size, a.texture_size = B, F, S, ts
            a.near_, a.far_, a.eps = cfg.near, cfg.far, cfg.eps
            a.background[0], a.background[1], a.background[2] = cfg.bg
            if indices is not None:
                a.vertices, a.face_indices, a.num_vertices = _ptr(geom_c), _ptr(indices), Nv
            else:
                a.faces = _ptr(geom_c)
            a.textures, a.background_batch = _ptr(tex_c), _ptr(cfg.bg_batch)
            a.face_index_map, a.weight_map, a.depth_map = _ptr(fim), _ptr(wmap), _ptr(dmap)
            a.rgb_map, a.alpha_map = _ptr(rgb_map), _ptr(alpha_map)
            a.out_rgb, a.out_alpha, a.out_depth = _ptr(out_rgb), _ptr(out_alpha), _ptr(out_depth)
            a.workspace, a.workspace_bytes = _ptr(ws), ws_bytes
            a.face_light = _ptr(light_c)
            a.face_uvs, (a.texture_height, a.texture_width) = _ptr(uv_c), tex_hw
            a.corner_light = _ptr(corner_c)
            if phong_c[0] is None:
                _lib.check(lib.nr_b200_forward(ctypes.byref(a), _stream_ptr(dev)))
            else:  # every Phong render, with NULL structs where an input is absent
                _lib.check(lib.nr_b200_forward_specular_map(ctypes.byref(a), *_phong_structs(phong_c), _stream_ptr(dev)))
        ctx.cfg = cfg
        ctx.flags = flags
        ctx.ts = ts
        ctx.F = F
        ctx.tex_shape = tuple(textures.shape) if textures is not None else None
        ctx.tex_hw = tex_hw
        # the unlit textures are only needed again for d loss / d face_light (corner_light) and d loss / d face_uvs
        need_light_grad = light_c is not None and ctx.needs_input_grad[2]
        ctx.need_corner_grad = corner_c is not None and ctx.needs_input_grad[6]
        ctx.need_uv_grad = uv_c is not None and want_rgb and ctx.needs_input_grad[5]
        ctx.need_phong_grad = [t is not None and need for t, need in zip(phong_c, ctx.needs_input_grad[7:])]
        # interior_gradient: the backward differentiates the sampler, so it reads the textures (and face_uvs / corner_light)
        ctx.interior = cfg.interior and want_rgb and ctx.needs_input_grad[0]
        need_tex = need_light_grad or ctx.need_uv_grad or ctx.need_corner_grad or ctx.interior or any(ctx.need_phong_grad)
        ctx.save_for_backward(geom_c, fim, wmap, dmap, rgb_map, light_c, tex_c if need_tex else None, indices, uv_c, corner_c,
                              *phong_c)
        if cfg.aa:
            rgb_o, alpha_o, depth_o = out_rgb, out_alpha, out_depth
        else:
            rgb_o, alpha_o, depth_o = rgb_map, alpha_map, (dmap if want_depth else None)
        ctx.mark_non_differentiable(fim, wmap)
        return rgb_o, alpha_o, depth_o, fim, wmap

    @staticmethod
    def backward(ctx, g_rgb, g_alpha, g_depth, _g_fim, _g_wmap):
        lib = _lib.load()
        cfg = ctx.cfg
        flags = ctx.flags | (_lib.NR_GRAD_INTERIOR if ctx.interior else 0)
        geom_c, fim, wmap, dmap, rgb_map, light_c, tex_c, indices, uv_c, corner_c, *phong_c = ctx.saved_tensors
        dev = geom_c.device
        B, F = geom_c.shape[0], ctx.F
        want_rgb = bool(flags & _lib.NR_RETURN_RGB)

        def prep(g, wanted):
            if g is None or not wanted:
                return None
            return g.detach().to(torch.float32).contiguous()

        g_rgb = prep(g_rgb, want_rgb)
        g_alpha = prep(g_alpha, bool(flags & _lib.NR_RETURN_ALPHA))
        g_depth = prep(g_depth, bool(flags & _lib.NR_RETURN_DEPTH))
        with torch.cuda.device(dev):
            grad_geom = torch.empty_like(geom_c)  # grad_faces [B,F,3,3], or grad_vertices [B,Nv,3] when indexed
            grad_textures = torch.empty(ctx.tex_shape, dtype=torch.float32, device=dev) if want_rgb else None
            grad_light = torch.empty_like(light_c) if (want_rgb and light_c is not None and ctx.needs_input_grad[2]) else None
            grad_uvs = torch.empty_like(uv_c) if ctx.need_uv_grad else None  # same layout as face_uvs: [1|B,F',3,2]
            grad_corner = torch.empty_like(corner_c) if ctx.need_corner_grad else None
            grad_phong = [torch.empty_like(t) if need else None for t, need in zip(phong_c, ctx.need_phong_grad)]
            phong_structs = _phong_structs(phong_c, grad_phong) if phong_c[0] is not None else None
            ws_bytes = lib.nr_b200_backward_workspace_bytes(B, F, cfg.S, ctx.ts, flags)
            ws = torch.empty((max(ws_bytes, 16),), dtype=torch.uint8, device=dev)
            a = _lib.BackwardArgs()
            a.struct_size = ctypes.sizeof(_lib.BackwardArgs)
            a.batch_size, a.raster_size, a.texture_size = B, cfg.S, ctx.ts
            a.eps = cfg.eps
            _set_geometry(a, geom_c, indices)  # and num_faces = F
            _set_geometry_grad(a, indices, grad_geom)
            a.textures = _ptr(tex_c)
            a.face_uvs, (a.texture_height, a.texture_width) = _ptr(uv_c), ctx.tex_hw
            a.face_light, a.grad_face_light = _ptr(light_c), _ptr(grad_light)
            a.face_index_map, a.weight_map, a.depth_map, a.rgb_map = _ptr(fim), _ptr(wmap), _ptr(dmap), _ptr(rgb_map)
            a.grad_rgb, a.grad_alpha, a.grad_depth = _ptr(g_rgb), _ptr(g_alpha), _ptr(g_depth)
            a.grad_textures = _ptr(grad_textures)
            a.grad_face_uvs = _ptr(grad_uvs)  # filled by the texture half
            a.workspace, a.workspace_bytes = _ptr(ws), ws.numel()
            hook = _TEXTURE_GRAD_HOOK if (want_rgb and g_rgb is not None) else None

            def call():
                if phong_structs is not None:  # Phong: every Phong input's gradient is filled by the texture half
                    return lib.nr_b200_backward_specular_map(ctypes.byref(a), *phong_structs, _stream_ptr(dev))
                if corner_c is None:
                    return lib.nr_b200_backward(ctypes.byref(a), _stream_ptr(dev))
                # smooth shading: grad_corner_light is filled by the texture half
                return lib.nr_b200_backward_corner_light(ctypes.byref(a), _ptr(corner_c), _ptr(grad_corner),
                                                         _stream_ptr(dev))
            if hook is None:
                a.flags = flags
                _lib.check(call())
            else:
                # two halves: the texture gradient is complete (and may start its all-reduce on another stream)
                # before the edge scan is even enqueued
                a.flags = flags | _lib.NR_BWD_PART_TEXTURES
                _lib.check(call())
                pending = hook(grad_textures)
                a.flags = flags | _lib.NR_BWD_PART_FACES
                _lib.check(call())
                if pending is not None:
                    pending.wait()
        return (grad_geom, grad_textures, grad_light, None, None, grad_uvs, grad_corner, *grad_phong)


# The Phong inputs in the order of the C ABI (nr_b200_forward_specular_map), with the dimensions each has without a batch
# axis: corner_shading, shading_params, lights, environment_sh, normal_map, corner_tangents, specular_map
_PHONG_DIMS = (3, 1, 2, 2, 3, 3, 3)


def _phong_structs(t, g=(None,) * 7):
    """The five struct arguments of nr_b200_*_specular_map for the Phong inputs t (and their gradient buffers g), NULL
    where an input is absent: each NULL trailing struct makes the call exactly the narrower entry point's."""
    cs, sp, lt, sh, nm, tg, sm = t
    g_cs, g_sp, g_lt, g_sh, g_nm, g_tg, g_sm = g
    return (ctypes.byref(_phong_args(cs, sp, g_cs, g_sp)),
            ctypes.byref(_lights_args(lt, g_lt)) if lt is not None else None,
            ctypes.byref(_sh_args(sh, g_sh)) if sh is not None else None,
            ctypes.byref(_normal_map_args(nm, tg, g_nm, g_tg)) if nm is not None else None,
            ctypes.byref(_specular_map_args(sm, g_sm)) if sm is not None else None)


def _batched(t, batch_size, dims=None):
    """t as float32 with the batch axis added when it has `dims` dimensions; an expanded (stride-0) batch of batch_size
    collapses to one shared item, which the kernels read in place."""
    t = t if t.dtype == torch.float32 else t.float()
    if t.dim() == dims:
        t = t[None]
    if t.shape[0] == batch_size > 1 and t.stride(0) == 0:
        t = t[:1]
    return t


def _phong_args(cs_c, sp_c, grad_cs=None, grad_sp=None):
    ph = _lib.PhongArgs()
    ph.struct_size = ctypes.sizeof(_lib.PhongArgs)
    ph.shading_batch, ph.params_batch = int(cs_c.shape[0]), int(sp_c.shape[0])
    ph.corner_shading, ph.params = _ptr(cs_c), _ptr(sp_c)
    ph.grad_corner_shading, ph.grad_params = _ptr(grad_cs), _ptr(grad_sp)
    return ph


def _lights_args(lt_c, grad_lt=None):
    la = _lib.LightsArgs()
    la.struct_size = ctypes.sizeof(_lib.LightsArgs)
    la.lights_batch, la.num_lights = int(lt_c.shape[0]), int(lt_c.shape[1])
    la.lights, la.grad_lights = _ptr(lt_c), _ptr(grad_lt)
    return la


def _sh_args(sh_c, grad_sh=None):
    sa = _lib.ShArgs()
    sa.struct_size = ctypes.sizeof(_lib.ShArgs)
    sa.sh_batch = int(sh_c.shape[0])
    sa.sh, sa.grad_sh = _ptr(sh_c), _ptr(grad_sh)
    return sa


def _normal_map_args(nm_c, tg_c, grad_nm=None, grad_tg=None):
    na = _lib.NormalMapArgs()
    na.struct_size = ctypes.sizeof(_lib.NormalMapArgs)
    na.map_batch, na.tangent_batch = int(nm_c.shape[0]), int(tg_c.shape[0])
    na.map_height, na.map_width = int(nm_c.shape[1]), int(nm_c.shape[2])
    na.normal_map, na.corner_tangents = _ptr(nm_c), _ptr(tg_c)
    na.grad_normal_map, na.grad_corner_tangents = _ptr(grad_nm), _ptr(grad_tg)
    return na


def _specular_map_args(sm_c, grad_sm=None):
    qa = _lib.SpecularMapArgs()
    qa.struct_size = ctypes.sizeof(_lib.SpecularMapArgs)
    qa.map_batch, qa.map_height, qa.map_width = int(sm_c.shape[0]), int(sm_c.shape[1]), int(sm_c.shape[2])
    qa.specular_map, qa.grad_specular_map = _ptr(sm_c), _ptr(grad_sm)
    return qa


class _MipPyramid(torch.autograd.Function):
    """image [Bt,Ht,Wt,3] -> packed mip pyramid [Bt,P,3] (nr_b200_mip_build); the backward collapses the pyramid gradient
    into the image gradient (nr_b200_mip_collapse, the exact transpose of the build)."""

    @staticmethod
    def forward(ctx, image):
        lib = _lib.load()
        img = image.detach().contiguous()
        Bt, H, W = (int(n) for n in img.shape[:3])
        P = int(lib.nr_b200_mip_texels(H, W))
        dev = img.device
        with torch.cuda.device(dev):
            pyr = torch.empty((Bt, P, 3), dtype=torch.float32, device=dev)
            _lib.check(lib.nr_b200_mip_build(_ptr(img), Bt, H, W, _ptr(pyr), _stream_ptr(dev)))
        ctx.shape = (Bt, H, W)
        return pyr

    @staticmethod
    def backward(ctx, grad_pyr):
        lib = _lib.load()
        Bt, H, W = ctx.shape
        g = grad_pyr.detach().to(torch.float32).contiguous()
        dev = g.device
        with torch.cuda.device(dev):
            grad_image = torch.empty((Bt, H, W, 3), dtype=torch.float32, device=dev)
            _lib.check(lib.nr_b200_mip_collapse(_ptr(g), Bt, H, W, _ptr(grad_image), 0, _stream_ptr(dev)))
        return grad_image


TEXTURE_FILTERS = ('bilinear', 'trilinear')


def _run(faces, textures, image_size, anti_aliasing, near, far, eps, background_color, return_rgb, return_alpha,
         return_depth, face_light=None, textures_fill_back=False, vertices=None, reference_exact=None, face_uvs=None,
         texture_filter='bilinear', corner_light=None, interior_gradient=False, corner_shading=None, shading_params=None,
         lights=None, environment_sh=None, normal_map=None, corner_tangents=None, specular_map=None):
    if (corner_shading is not None or shading_params is not None) and interior_gradient:
        raise ValueError("interior_gradient=True is not supported with Phong shading (corner_shading / shading_params): no "
                         "vertex gradient flows through the interpolation of the per-pixel normal and position")
    if texture_filter not in TEXTURE_FILTERS:
        raise ValueError("texture_filter must be one of %s, got %r" % (TEXTURE_FILTERS, texture_filter))
    if texture_filter == 'trilinear' and face_uvs is None:
        raise ValueError("texture_filter='trilinear' samples a texture image: it needs face_uvs")
    geom_in = vertices if vertices is not None else faces
    if (return_rgb and interior_gradient and face_uvs is None and isinstance(geom_in, torch.Tensor) and geom_in.dim() >= 1
            and geom_in.shape[0] > 1 and (_REFERENCE_EXACT if reference_exact is None else reference_exact)):
        raise ValueError("interior_gradient=True with per-face cubes needs every item's own depths when the batch has more "
                         "than one item: the reference-exact sampler reads the depths of item 0 for every item, so its "
                         "derivative would cross items.  Pass reference_exact=False (or set_reference_exact(False))")
    _check_inputs(faces, textures, return_rgb, face_light, textures_fill_back, vertices, face_uvs, corner_light,
                  corner_shading, shading_params, lights, environment_sh, normal_map, corner_tangents, specular_map)
    phong = [corner_shading, shading_params, lights, environment_sh, normal_map, corner_tangents, specular_map]
    geom, indices = _geometry(faces, vertices)
    batch_size = geom.shape[0]
    if not return_rgb:
        face_uvs = None
        phong = [None] * len(_PHONG_DIMS)
    if return_rgb:
        # a texture image [Ht,Wt,3] (with face_uvs) is one image for every item; shared sets are read in place
        # (NR_TEX_SHARED, NR_UV_SHARED, and a batch of 1 for each Phong input)
        textures = _batched(textures, batch_size, 3 if face_uvs is not None else None)
        if face_uvs is not None:
            face_uvs = _batched(face_uvs, batch_size, 3)
        phong = [_batched(t, batch_size, dims) if t is not None else None for t, dims in zip(phong, _PHONG_DIMS)]
        if phong[2] is not None and phong[2].shape[1] == 0:
            phong[2] = None  # lights: no extra light is Phong exactly
    cfg = _make_config(image_size, anti_aliasing, near, far, eps, background_color, return_rgb, return_alpha,
                       return_depth, geom.device, batch_size, reference_exact)
    if return_rgb and textures_fill_back:
        cfg.flags |= _lib.NR_TEX_FILL_BACK
    if return_rgb and _STAGE_TEXTURES:
        cfg.flags |= _lib.NR_FWD_STAGE_TEXTURES
    cfg.interior = bool(return_rgb and interior_gradient)
    if return_rgb and texture_filter == 'trilinear':
        # the pyramid is built from the image (shared or per item, as the image is) and autograd chains its gradient
        # back into the image
        cfg.mip_hw = (int(textures.shape[1]), int(textures.shape[2]))
        cfg.flags |= _lib.NR_TEX_MIPMAP
        textures = _MipPyramid.apply(textures)
    return _RasterizeFunction.apply(geom, textures if return_rgb else None, face_light if return_rgb else None, cfg,
                                    indices, face_uvs, corner_light, *phong)


def rasterize_rgbad(
        faces,
        textures=None,
        image_size=DEFAULT_IMAGE_SIZE,
        anti_aliasing=DEFAULT_ANTI_ALIASING,
        near=DEFAULT_NEAR,
        far=DEFAULT_FAR,
        eps=DEFAULT_EPS,
        background_color=DEFAULT_BACKGROUND_COLOR,
        return_rgb=True,
        return_alpha=True,
        return_depth=True,
        *,
        face_light=None,
        textures_fill_back=False,
        vertices=None,
        reference_exact=None,
        face_uvs=None,
        texture_filter='bilinear',
        corner_light=None,
        interior_gradient=False,
        corner_shading=None,
        shading_params=None,
        lights=None,
        environment_sh=None,
        normal_map=None,
        corner_tangents=None,
        specular_map=None,
):
    """Generate RGB, alpha channel, and depth images from faces and textures (for RGB).  rasterize.py:900-977.

    Returns {'rgb': [B,3,H,W], 'alpha': [B,H,W], 'depth': [B,H,W]} (None for the ones not requested).

    Keyword-only extensions (not in the reference; `Renderer.render` uses them so that neither the lit nor the
    fill_back-doubled texture tensor is ever materialised):
      face_light [B,F,3]      per-face RGB factor of `lighting` applied at sample time (== sampling textures * light)
      textures_fill_back      faces [F/2, F) are the reversed copies of [0, F/2) and `textures` holds only the F/2
                              original cubes (the copies read them with reversed axes, renderer.py:80)
      vertices [B,Nv,3]       indexed geometry: `faces` then holds integer vertex indices ([B,F,3], or [F,3] / [1,F,3]
                              shared by the batch) and vertices_to_faces (vertices_to_faces.py:16-21) plus its
                              scatter-add backward run inside the rasterizer: no [B,F,3,3] tensor exists and the
                              gradient arrives in `vertices.grad`
      reference_exact         True / False overrides the module default (`set_reference_exact`) for this call: the
                              reference's texture sampler reads the vertex depths of batch item 0 for EVERY item
                              (rasterize.py:389).  True reproduces that bit for bit; False samples every item with its own
                              depths -- what one wants for batches of different meshes or cameras (the images of items
                              b > 0 and grad_textures differ, item 0 and all silhouettes / depths do not)
      face_uvs [F,3,2] / [B,F,3,2]  texture-image mode: `textures` is then an image [Ht,Wt,3] or [1|B,Ht,Wt,3] (row 0 =
                              top, as read from a PNG) and face_uvs the UV of every face corner (OBJ convention, v = 0 at
                              the bottom; F/2 faces with textures_fill_back).  Sampled bilinearly (clamp to edge) at the
                              perspective-correct UV, with every item's own vertex depths (`reference_exact` has no
                              effect).  The image and face_uvs receive gradients: d / d face_uvs is the derivative of
                              the bilinear sample within the texel cell the forward picked (include/nr_b200.h), with
                              the level of detail, the perspective weights and the [0,1] clamp held fixed (0 where a
                              UV is clamped).  A shared face_uvs ([F,3,2], [1,F,3,2] or expanded) gets the sum over
                              the items; with textures_fill_back the copies' gradient is folded into the F/2 faces.
      texture_filter          'bilinear' (default) or 'trilinear' (texture-image mode only): sample a mip pyramid of the
                              image at each pixel's level of detail, so minified images neither alias nor leave most
                              texels without gradient.  The pyramid is rebuilt from the image on every call and its
                              gradient collapsed back into the image; no gradient flows through the level of detail
                              (face_uvs gets the level-weighted sum of both levels' derivatives).
      corner_light [B,F,3,3]  smooth shading: an RGB light factor at each corner of every face (corners in the order of
                              `faces`; F counts fill_back copies), interpolated with the pixel's perspective-correct
                              weights and multiplied onto the unlit sample (include/nr_b200.h).  Exclusive with
                              face_light; needs return_rgb.  F.vertex_normals / F.corner_light compute the Lambertian
                              factor, but any per-corner factor works.  It receives d loss / d corner_light; no vertex
                              gradient flows through the interpolation weights unless interior_gradient=True.
      interior_gradient       False (default): the vertices receive the reference's gradient (edges through the rgb / alpha
                              images, depth).  True: also the derivative of the colour INSIDE each face through the
                              perspective weights -- the texture sampled at a moving position and the smooth light
                              (include/nr_b200.h, NR_GRAD_INTERIOR), with the cell, level of detail and clamps held fixed.
                              What photometric alignment of a textured mesh needs.  Per-face cubes with a batch > 1 need
                              reference_exact=False.
      corner_shading [F,3,6] / [1|B,F,3,6], shading_params [16] / [1|B,16]   Phong shading, always together: per face
                              corner (the order of `faces`; F counts fill_back copies, give them the negated normal) a
                              shading normal and a position, interpolated per pixel with the perspective-correct weights;
                              shading_params = {ambient[3], directional[3], direction[3], specular[3], shininess, eye[3]}
                              (F.corner_shading / F.phong_params build both).  rgb = (ambient + directional relu(n . d))
                              * sample + specular * q^shininess, the highlight of the reflected light towards the eye
                              (include/nr_b200.h).  Exclusive with face_light / corner_light and with
                              interior_gradient; both receive gradients (a batch of 1 gets the sum over the items).
      lights [NL,12] / [1|B,NL,12]   Phong shading with up to 8 more lights after shading_params' own, directional or
                              point (F.directional_light / F.point_light / F.light_set build them): each adds its diffuse
                              term a relu(n . l) to the light of the sample and its highlight a q^shininess, with a point
                              light's direction and attenuation a = 1 / (1 + falloff r^2) evaluated at every pixel
                              (include/nr_b200.h, nr_b200_lights_args).  Only with corner_shading / shading_params;
                              receives gradients (a batch of 1 gets the sum over the items).
      environment_sh [9,3] / [1|B,9,3]   Phong shading lit by an environment as well: second-order spherical-harmonic
                              coefficients (k major, channel minor; F.sh_from_environment_map makes them from a lat-long
                              map), irradiance-ready (S = (1/C0, 0, ...) gives irradiance 1).  The irradiance
                              E_c = sum_k S[k][c] Y_k(n) at the pixel's normal is added to the light of the sample after
                              every diffuse term, unclamped (include/nr_b200.h, nr_b200_sh_args).  Only with
                              corner_shading / shading_params; composes with `lights`; receives gradients (a batch of 1
                              gets the sum over the items).
      normal_map [Hm,Wm,3] / [1|B,Hm,Wm,3], corner_tangents [F,3,4] / [1|B,F,3,4]   Phong shading through a tangent-space
                              normal map, always given together: the map holds decoded vectors (F.decode_normal_map; row 0
                              = top, +y along +v) sampled bilinearly at the pixel's uv, and corner_tangents the (T, w)
                              of every drawn face's corners (F.corner_tangents; F counts the fill_back copies, as
                              corner_shading).  The shading normal becomes m_x t + m_y b + m_z n with b = sign(w) n x t
                              (include/nr_b200.h, nr_b200_normal_map_args), for every light and the environment.  Needs
                              corner_shading and a texture image with face_uvs; both receive gradients (a batch of 1
                              gets the sum over the items), and face_uvs receives the map's term too.
      specular_map [Hq,Wq,4] / [1|B,Hq,Wq,4]   Phong shading through a specular map: per texel (ks_r, ks_g, ks_b,
                              shininess) (F.specular_map packs them; row 0 = top), sampled bilinearly at the pixel's uv.
                              Every highlight's colour is multiplied by ks and the map's shininess replaces
                              shading_params' for shading_params' light and every light of `lights`; the diffuse terms
                              do not change (include/nr_b200.h, nr_b200_specular_map_args).  A map (1, 1, 1, shininess)
                              renders as no map.  Needs corner_shading and a texture image with face_uvs; composes with
                              lights, environment_sh and normal_map.  It receives gradients (a batch of 1 gets the sum
                              over the items; shading_params' shininess then gets none), and face_uvs receives the
                              map's term too.
    `textures` with batch size 1 (or an expanded stride-0 batch) while the geometry batch is larger = one texture set
    shared by every item (a mesh seen from B viewpoints, mesh.py:29-34); its gradient is the sum over the items."""
    rgb, alpha, depth, _, _ = _run(faces, textures, image_size, anti_aliasing, near, far, eps, background_color,
                                   return_rgb, return_alpha, return_depth, face_light, textures_fill_back, vertices,
                                   reference_exact, face_uvs, texture_filter, corner_light, interior_gradient,
                                   corner_shading, shading_params, lights, environment_sh, normal_map, corner_tangents,
                                   specular_map)
    return {
        'rgb': rgb if return_rgb else None,
        'alpha': alpha if return_alpha else None,
        'depth': depth if return_depth else None,
    }


def rasterize(
        faces,
        textures,
        image_size=DEFAULT_IMAGE_SIZE,
        anti_aliasing=DEFAULT_ANTI_ALIASING,
        near=DEFAULT_NEAR,
        far=DEFAULT_FAR,
        eps=DEFAULT_EPS,
        background_color=DEFAULT_BACKGROUND_COLOR,
        *,
        face_light=None,
        textures_fill_back=False,
        vertices=None,
        reference_exact=None,
        face_uvs=None,
        texture_filter='bilinear',
        corner_light=None,
        interior_gradient=False,
        corner_shading=None,
        shading_params=None,
        lights=None,
        environment_sh=None,
        normal_map=None,
        corner_tangents=None,
        specular_map=None,
):
    """RGB images [B,3,H,W] from faces and textures.  rasterize.py:980-1008 (keyword-only extras: rasterize_rgbad; in
    texture-image mode both the image and face_uvs receive gradients)."""
    return rasterize_rgbad(
        faces, textures, image_size, anti_aliasing, near, far, eps, background_color, True, False, False,
        face_light=face_light, textures_fill_back=textures_fill_back, vertices=vertices,
        reference_exact=reference_exact, face_uvs=face_uvs, texture_filter=texture_filter, corner_light=corner_light,
        interior_gradient=interior_gradient, corner_shading=corner_shading, shading_params=shading_params,
        lights=lights, environment_sh=environment_sh, normal_map=normal_map, corner_tangents=corner_tangents,
        specular_map=specular_map)['rgb']


def rasterize_silhouettes(
        faces,
        image_size=DEFAULT_IMAGE_SIZE,
        anti_aliasing=DEFAULT_ANTI_ALIASING,
        near=DEFAULT_NEAR,
        far=DEFAULT_FAR,
        eps=DEFAULT_EPS,
        *,
        vertices=None,
):
    """Alpha channels [B,H,W] from faces.  rasterize.py:1011-1034 (keyword-only `vertices`: rasterize_rgbad)."""
    return rasterize_rgbad(faces, None, image_size, anti_aliasing, near, far, eps, None, False, True, False,
                           vertices=vertices)['alpha']


def rasterize_depth(
        faces,
        image_size=DEFAULT_IMAGE_SIZE,
        anti_aliasing=DEFAULT_ANTI_ALIASING,
        near=DEFAULT_NEAR,
        far=DEFAULT_FAR,
        eps=DEFAULT_EPS,
        *,
        vertices=None,
):
    """Depth images [B,H,W] from faces.  rasterize.py:1037-1060 (keyword-only `vertices`: rasterize_rgbad)."""
    return rasterize_rgbad(faces, None, image_size, anti_aliasing, near, far, eps, None, False, False, True,
                           vertices=vertices)['depth']


class _InterpolateFunction(torch.autograd.Function):
    """autograd node of attribute interpolation: forward = nr_b200_interpolate on the maps of a forward call, backward =
    nr_b200_interpolate_backward (d loss / d attributes, and the interior vertex gradient through the perspective weights).

    `geom` / `indices` are the geometry exactly as the forward call that produced `fim` / `wmap` got it; `flags` holds the
    anti-aliasing and attribute-layout bits, `S` the raster size."""

    @staticmethod
    def forward(ctx, geom, attributes, fim, wmap, indices, flags, S):
        lib = _lib.load()
        dev = geom.device
        geom_c = geom.detach().contiguous()
        attr_c = attributes.detach().contiguous()
        B, C = geom_c.shape[0], attr_c.shape[-1]
        H = S // 2 if flags & _lib.NR_ANTI_ALIASING else S
        with torch.cuda.device(dev):
            out = torch.empty((B, C, H, H), dtype=torch.float32, device=dev)
            a = _interpolate_args(geom_c, attr_c, fim, wmap, indices, flags, S)
            a.out = _ptr(out)
            _lib.check(lib.nr_b200_interpolate(ctypes.byref(a), _stream_ptr(dev)))
        ctx.flags, ctx.S = flags, S
        ctx.save_for_backward(geom_c, attr_c, fim, wmap, indices)
        return out

    @staticmethod
    def backward(ctx, g):
        want_geom, want_attr = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        if g is None or not (want_geom or want_attr):
            return None, None, None, None, None, None, None
        lib = _lib.load()
        geom_c, attr_c, fim, wmap, indices = ctx.saved_tensors
        dev = geom_c.device
        g = g.detach().to(torch.float32).contiguous()
        with torch.cuda.device(dev):
            grad_geom = torch.empty_like(geom_c) if want_geom else None
            grad_attr = torch.empty_like(attr_c) if want_attr else None
            a = _interpolate_args(geom_c, attr_c, fim, wmap, indices, ctx.flags, ctx.S)
            a.grad_out, a.grad_attributes = _ptr(g), _ptr(grad_attr)
            _set_geometry_grad(a, indices, grad_geom)
            _lib.check(lib.nr_b200_interpolate_backward(ctypes.byref(a), _stream_ptr(dev)))
        return grad_geom, grad_attr, None, None, None, None, None


def _interpolate_args(geom_c, attr_c, fim, wmap, indices, flags, S):
    a = _lib.InterpolateArgs()
    a.struct_size = ctypes.sizeof(_lib.InterpolateArgs)
    B = geom_c.shape[0]
    flags |= _set_geometry(a, geom_c, indices)
    if attr_c.shape[0] == 1 and B > 1:
        flags |= _lib.NR_ATTR_SHARED
    a.flags = flags
    a.batch_size, a.raster_size, a.channels = B, S, attr_c.shape[-1]
    a.face_index_map, a.weight_map, a.attributes = _ptr(fim), _ptr(wmap), _ptr(attr_c)
    return a


def _check_attribute_inputs(faces, vertices, vertex_attributes, face_attributes):
    """argument errors of rasterize_attributes, all raised before any device check"""
    if (vertex_attributes is None) == (face_attributes is None):
        raise TypeError("give exactly one of vertex_attributes= and face_attributes=")
    per_vertex = vertex_attributes is not None
    attrs = vertex_attributes if per_vertex else face_attributes
    name = "vertex_attributes" if per_vertex else "face_attributes"
    if not isinstance(attrs, torch.Tensor) or not attrs.is_floating_point():
        raise TypeError("%s must be a floating point torch.Tensor" % name)
    if per_vertex and vertices is None:
        raise ValueError("vertex_attributes need indexed geometry: vertices= and integer faces")
    # the attribute shapes against the geometry's, when the geometry's own shape is valid (else _check_inputs says why)
    B = F = Nv = None
    if isinstance(faces, torch.Tensor) and faces.dim() >= 2:
        if isinstance(vertices, torch.Tensor) and vertices.dim() == 3:
            B, F, Nv = vertices.shape[0], faces.shape[-2], vertices.shape[1]
        elif vertices is None and faces.dim() == 4:
            B, F = faces.shape[0], faces.shape[1]
    if B is not None:
        rows = (Nv,) if per_vertex else (F, 3)
        nd = len(rows) + 1
        ok = attrs.dim() in (nd, nd + 1) and tuple(attrs.shape[-nd:-1]) == rows and attrs.shape[-1] >= 1
        if ok and attrs.dim() == nd + 1:
            ok = attrs.shape[0] in (1, B)
        if not ok:
            want = "[num vertices, C] or [batch size, num vertices, C]" if per_vertex else \
                "[num faces, 3, C] or [batch size, num faces, 3, C]"
            raise ValueError("%s must have shape %s with C >= 1 matching the geometry (num faces counts fill_back "
                             "copies), got %s" % (name, want, tuple(attrs.shape)))
    _check_inputs(faces, None, False, vertices=vertices)  # the geometry, then the device check
    if not attrs.is_cuda:
        raise NotImplementedError("neural_renderer_b200 has no CPU implementation (inputs must be CUDA tensors)")
    return attrs, per_vertex


def rasterize_attributes(
        faces,
        image_size=DEFAULT_IMAGE_SIZE,
        anti_aliasing=DEFAULT_ANTI_ALIASING,
        near=DEFAULT_NEAR,
        far=DEFAULT_FAR,
        eps=DEFAULT_EPS,
        *,
        vertices=None,
        vertex_attributes=None,
        face_attributes=None,
        return_alpha=False,
):
    """Images [B,C,H,W] of arbitrary per-vertex or per-corner attributes: normal maps, position maps, UV G-buffers,
    part labels, feature images.  Not in the reference (PyTorch3D: interpolate_face_attributes, nvdiffrast: interpolate).

    Exactly one of (keywords, because [B,Nv,C] and [F,3,C] cannot be told apart by shape):
      vertex_attributes [Nv,C] / [1|B,Nv,C]     one row per vertex; needs indexed geometry (`vertices`, integer faces)
      face_attributes [F,3,C] / [1|B,F,3,C]     one row per face corner, corners in the order of `faces` (F counts any
                                                fill_back copies: give them their corners, e.g. cat((a, a.flip(-2)), -3))
    A batch of 1 (or an expanded stride-0 batch) with a larger geometry batch is one set shared by every item; its
    gradient is the sum over the items.  Every covered pixel gets sum_k l_k a_k with the perspective-correct weights l_k
    of the winning face (include/nr_b200.h), uncovered pixels 0; with anti-aliasing the 2x2 mean.  No lighting.

    Gradients flow into the attributes and, through the interpolation weights, into the vertices (the interior
    derivative, with the weights' clamp held fixed).  The image has no edge or occlusion gradient: for that, use the
    alpha image of `return_alpha=True`, which is the rasterizer's and carries its usual silhouette gradient.  Returns
    the image, or (image, alpha)."""
    attrs, per_vertex = _check_attribute_inputs(faces, vertices, vertex_attributes, face_attributes)
    geom, indices = _geometry(faces, vertices)
    batch_size = geom.shape[0]
    attrs = _batched(attrs, batch_size, 2 if per_vertex else 3)  # an expanded shared set: NR_ATTR_SHARED
    _, alpha, _, fim, wmap = _run(indices if indices is not None else geom, None, image_size, anti_aliasing, near, far,
                                  eps, None, False, True, False, vertices=geom if indices is not None else None)
    flags = (_lib.NR_ANTI_ALIASING if anti_aliasing else 0) | (_lib.NR_ATTR_PER_VERTEX if per_vertex else 0)
    S = int(image_size) * 2 if anti_aliasing else int(image_size)
    image = _InterpolateFunction.apply(geom, attrs, fim, wmap, indices, flags, S)
    return (image, alpha) if return_alpha else image


DEFAULT_SOFT_SIGMA = 1e-5


def _positive_number(name, v):
    try:
        v = float(v)
    except (TypeError, ValueError):
        raise TypeError("%s must be a number, got %r" % (name, v))
    if not math.isfinite(v) or v <= 0:
        raise ValueError("%s must be finite and > 0, got %r" % (name, v))
    return v


class _SoftSilhouettesFunction(torch.autograd.Function):
    """autograd node of the soft silhouettes: forward = nr_b200_soft_silhouettes, backward =
    nr_b200_soft_silhouettes_backward from the saved alpha.  `geom` / `indices` as _RasterizeFunction."""

    @staticmethod
    def forward(ctx, geom, indices, S, sigma, near, far):
        lib = _lib.load()
        dev = geom.device
        geom_c = geom.detach().contiguous()
        with torch.cuda.device(dev):
            alpha = torch.empty((geom_c.shape[0], S, S), dtype=torch.float32, device=dev)
            a, ws = _soft_args(lib, geom_c, indices, S, sigma, near, far)
            a.alpha = _ptr(alpha)
            _lib.check(lib.nr_b200_soft_silhouettes(ctypes.byref(a), _stream_ptr(dev)))
        ctx.cfg = (S, sigma, near, far)
        ctx.save_for_backward(geom_c, indices, alpha)
        return alpha

    @staticmethod
    def backward(ctx, g):
        if g is None or not ctx.needs_input_grad[0]:
            return None, None, None, None, None, None
        lib = _lib.load()
        geom_c, indices, alpha = ctx.saved_tensors
        dev = geom_c.device
        g = g.detach().to(torch.float32).contiguous()
        with torch.cuda.device(dev):
            grad_geom = torch.empty_like(geom_c)
            a, ws = _soft_args(lib, geom_c, indices, *ctx.cfg)
            a.alpha, a.grad_alpha = _ptr(alpha), _ptr(g)
            _set_geometry_grad(a, indices, grad_geom)
            _lib.check(lib.nr_b200_soft_silhouettes_backward(ctypes.byref(a), _stream_ptr(dev)))
        return grad_geom, None, None, None, None, None


def _soft_args(lib, geom_c, indices, S, sigma, near, far):
    """nr_b200_soft_args of a call and its workspace (returned so that it lives until the launch is queued)"""
    a = _lib.SoftArgs()
    a.struct_size = ctypes.sizeof(_lib.SoftArgs)
    B = geom_c.shape[0]
    a.flags = _set_geometry(a, geom_c, indices)
    a.batch_size, a.image_size = B, S
    a.sigma, a.near_, a.far_ = sigma, near, far
    n = lib.nr_b200_soft_workspace_bytes(B, a.num_faces, S, sigma, a.flags)
    if n == 0:
        raise ValueError("rasterize_soft_silhouettes: sizes out of range (batch %d, %d faces, image %d)" % (B, a.num_faces, S))
    ws = torch.empty(n, dtype=torch.uint8, device=geom_c.device)
    a.workspace, a.workspace_bytes = _ptr(ws), n
    return a, ws


def rasterize_soft_silhouettes(
        faces,
        image_size=DEFAULT_IMAGE_SIZE,
        sigma=DEFAULT_SOFT_SIGMA,
        near=DEFAULT_NEAR,
        far=DEFAULT_FAR,
        *,
        vertices=None,
):
    """Soft silhouettes [B,H,W] (SoftRas, Liu et al. 2019): every face gives every pixel within reach the probability
    sigmoid(+-d^2 / sigma) of the pixel's squared NDC distance d^2 to the face (+ inside, - outside), and
    alpha = 1 - prod_j (1 - D_j) over the faces.  Unlike rasterize_silhouettes, the gradient reaches every vertex of every
    face within reach of a pixel -- faces a few pixels off a target outline, and faces hidden behind others -- so it suits
    fitting shapes to masks.  Not in the reference.

    Geometry as rasterize_silhouettes: faces [B,F,3,3], or `vertices` [B,Nv,3] with integer faces [F,3] / [1|B,F,3] (an
    expanded index set stays shared).  Winding does not matter: pass each face once (a fill_back copy would count twice).
    A face takes part only when all three vertex depths lie in [near, far] (a per-face test, not the hard rasterizer's
    per-pixel depth test).  sigma > 0 sets the softness: the reach is sqrt(sigma ln((1-eps)/eps)) image_size / 2 pixels
    with eps = 1e-4, about 1.2 px at 256 x 256 for the default 1e-5.  No anti-aliasing; deterministic forward.  The exact
    definition and its gradient are in include/nr_b200.h (nr_b200_soft_args)."""
    sigma = _positive_number("sigma", sigma)
    if not (float(near) <= float(far)):
        raise ValueError("near must be <= far, got near=%r far=%r" % (near, far))
    if int(image_size) < 1:
        raise ValueError("image_size must be >= 1, got %r" % (image_size,))
    _check_inputs(faces, None, False, vertices=vertices)  # the geometry, then the device check
    geom, indices = _geometry(faces, vertices)
    return _SoftSilhouettesFunction.apply(geom, indices, int(image_size), sigma, float(near), float(far))


DEFAULT_SOFT_GAMMA = 1e-4


class _SoftRgbFunction(torch.autograd.Function):
    """autograd node of the soft RGB: forward = nr_b200_soft_rgb_uv, backward = nr_b200_soft_rgb_uv_backward from the
    saved rgb, alpha and state.  `geom` / `indices` as _RasterizeFunction.  Cubes: `textures` [B|1,F,ts,ts,ts,3]
    (1 = shared) and `face_uvs` None, the NULL nr_b200_soft_uv_args of the cube call.  Texture image: `textures` is the
    image [B|1,Ht,Wt,3], or its packed pyramid [B|1,P,3] when `hw` = (Ht, Wt) of level 0 is given (trilinear), and
    `face_uvs` [B|1,F,3,2] (1 = shared)."""

    @staticmethod
    def forward(ctx, geom, textures, face_light, face_uvs, indices, cfg, hw):
        lib = _lib.load()
        dev = geom.device
        geom_c = geom.detach().contiguous()
        tex_c = textures.detach().contiguous()
        uv_c = face_uvs.detach().contiguous() if face_uvs is not None else None
        light_c = face_light.detach().contiguous() if face_light is not None else None
        B, S = geom_c.shape[0], cfg[0]
        with torch.cuda.device(dev):
            rgb = torch.empty((B, 3, S, S), dtype=torch.float32, device=dev)
            alpha = torch.empty((B, S, S), dtype=torch.float32, device=dev)
            state = torch.empty((B, 2, S, S), dtype=torch.float32, device=dev)
            a, u, ws = _soft_tex_args(lib, geom_c, indices, tex_c, light_c, uv_c, cfg, hw)
            a.rgb, a.alpha, a.state = _ptr(rgb), _ptr(alpha), _ptr(state)
            _lib.check(lib.nr_b200_soft_rgb_uv(ctypes.byref(a), u, _stream_ptr(dev)))
        ctx.cfg, ctx.hw = cfg, hw
        ctx.save_for_backward(geom_c, tex_c, light_c, uv_c, indices, rgb, alpha, state)
        return rgb, alpha

    @staticmethod
    def backward(ctx, g_rgb, g_alpha):
        lib = _lib.load()
        geom_c, tex_c, light_c, uv_c, indices, rgb, alpha, state = ctx.saved_tensors
        dev = geom_c.device
        need_geom, need_tex, need_light, need_uv = ctx.needs_input_grad[:4]
        none = (None,) * 7
        if not (need_geom or need_tex or need_light or need_uv) or (g_rgb is None and g_alpha is None):
            return none
        g_rgb = g_rgb.detach().to(torch.float32).contiguous() if g_rgb is not None else None
        g_alpha = g_alpha.detach().to(torch.float32).contiguous() if g_alpha is not None else None
        with torch.cuda.device(dev):
            grad_geom = torch.empty_like(geom_c)
            grad_tex = torch.empty_like(tex_c) if need_tex else None
            grad_light = torch.empty_like(light_c) if need_light and light_c is not None else None
            grad_uv = torch.empty_like(uv_c) if need_uv else None
            a, u, ws = _soft_tex_args(lib, geom_c, indices, tex_c, light_c, uv_c, ctx.cfg, ctx.hw, grad_uv)
            a.rgb, a.alpha, a.state = _ptr(rgb), _ptr(alpha), _ptr(state)
            a.grad_rgb, a.grad_alpha = _ptr(g_rgb), _ptr(g_alpha)
            _set_geometry_grad(a, indices, grad_geom)
            a.grad_textures, a.grad_face_light = _ptr(grad_tex), _ptr(grad_light)
            _lib.check(lib.nr_b200_soft_rgb_uv_backward(ctypes.byref(a), u, _stream_ptr(dev)))
        return grad_geom if need_geom else None, grad_tex, grad_light, grad_uv, None, None, None


def _soft_rgb_args(lib, geom_c, indices, S, sigma, near, far, gamma=0.0, flags=0, name="rasterize_soft"):
    """nr_b200_soft_rgb_args with the fields every soft RGB-family call sets (the geometry with its flags and `flags`,
    the sizes, sigma, gamma, near and far) and its workspace (returned so that it lives until the launch is queued)"""
    a = _lib.SoftRgbArgs()
    a.struct_size = ctypes.sizeof(_lib.SoftRgbArgs)
    B = geom_c.shape[0]
    a.flags = flags | _set_geometry(a, geom_c, indices)
    a.batch_size, a.image_size = B, S
    a.sigma, a.gamma, a.near_, a.far_ = sigma, gamma, near, far
    n = lib.nr_b200_soft_rgb_workspace_bytes(B, a.num_faces, S, a.flags)
    if n == 0:
        raise ValueError("%s: sizes out of range (batch %d, %d faces, image %d)" % (name, B, a.num_faces, S))
    ws = torch.empty(n, dtype=torch.uint8, device=geom_c.device)
    a.workspace, a.workspace_bytes = _ptr(ws), n
    return a, ws


def _soft_tex_args(lib, geom_c, indices, tex_c, light_c, uv_c, cfg, hw, grad_uv=None):
    """nr_b200_soft_rgb_args of a soft RGB call, a reference to its nr_b200_soft_uv_args (None for cubes) and the
    workspace"""
    S, sigma, gamma, near, far, eps, bg = cfg
    tex_shared = _lib.NR_TEX_SHARED if tex_c.shape[0] == 1 and geom_c.shape[0] > 1 else 0
    a, ws = _soft_rgb_args(lib, geom_c, indices, S, sigma, near, far, gamma, tex_shared)
    a.texture_size, a.eps = tex_c.shape[2], eps
    a.background[:] = bg
    a.textures, a.face_light = _ptr(tex_c), _ptr(light_c)
    if uv_c is None:
        return a, None, ws
    a.flags |= _lib.NR_TEX_UV
    if uv_c.shape[0] == 1 and geom_c.shape[0] > 1:
        a.flags |= _lib.NR_UV_SHARED
    if hw is not None:
        a.flags |= _lib.NR_TEX_MIPMAP
    u = _lib.SoftUvArgs()
    u.struct_size = ctypes.sizeof(_lib.SoftUvArgs)
    u.texture_height, u.texture_width = hw if hw is not None else (tex_c.shape[1], tex_c.shape[2])
    u.face_uvs, u.grad_face_uvs = _ptr(uv_c), _ptr(grad_uv)
    return a, ctypes.byref(u), ws


def rasterize_soft(
        faces,
        textures,
        image_size=DEFAULT_IMAGE_SIZE,
        sigma=DEFAULT_SOFT_SIGMA,
        gamma=DEFAULT_SOFT_GAMMA,
        near=DEFAULT_NEAR,
        far=DEFAULT_FAR,
        eps=DEFAULT_EPS,
        background_color=DEFAULT_BACKGROUND_COLOR,
        *,
        vertices=None,
        face_light=None,
        face_uvs=None,
        texture_filter='bilinear',
):
    """Soft RGB images [B,3,H,W] and soft silhouettes [B,H,W] (SoftRas, Liu et al. 2019): every face within reach of a
    pixel (the soft silhouettes' probability D_j, rasterize_soft_silhouettes) adds its texture colour with the weight
    D_j exp((zn_j - zmax) / gamma) of its normalised depth zn_j = (far - zp) / (far - near), against a background term at
    zn = 1e-3.  Unlike rasterize, the gradient reaches the vertices from every face within reach -- hidden faces and
    faces a few pixels off their target included -- and reaches the vertex depths, so the depth order itself can be
    learned.  Not in the reference.

    Geometry as rasterize_soft_silhouettes (pass each face once; fill_back copies would count twice).  textures: per-face
    cubes [B,F,ts,ts,ts,3], or [1,F,...] shared by every item (its gradient is the sum over the items), sampled at the
    perspective-correct clipped barycentrics with the clamp from `eps` as rasterize samples them.  face_light [B,F,3]
    (e.g. functional.face_light_from_vertices) multiplies every texel first; None = unlit.  gamma > 0 sets how sharply
    the nearer face wins.  Returns (rgb, alpha); alpha is bit-identical to rasterize_soft_silhouettes.  Deterministic
    forward.  Gradients into the geometry, the textures and face_light.  The exact definition is in include/nr_b200.h
    (nr_b200_soft_rgb_args).

    With face_uvs [F,3,2] / [1|B,F,3,2] (UV of every face corner; an expanded set stays shared), `textures` is a texture
    image [Ht,Wt,3] / [1|B,Ht,Wt,3] (row 0 = top) sampled at each face's perspective-correct UV: bilinearly, or through
    a mip pyramid with texture_filter='trilinear' (as rasterize_rgbad samples images).  Gradients then also reach the
    image and, when it requires grad, face_uvs (nr_b200_soft_uv_args)."""
    sigma, gamma = _positive_number("sigma", sigma), _positive_number("gamma", gamma)
    if not (float(near) < float(far)):
        raise ValueError("near must be < far, got near=%r far=%r" % (near, far))
    if int(image_size) < 1:
        raise ValueError("image_size must be >= 1, got %r" % (image_size,))
    bg = [float(c) for c in background_color]
    if len(bg) != 3:
        raise ValueError("background_color must have 3 components, got %r" % (background_color,))
    if face_light is not None and not isinstance(face_light, torch.Tensor):
        raise TypeError("face_light must be a torch.Tensor")
    if texture_filter not in TEXTURE_FILTERS:
        raise ValueError("texture_filter must be one of %s, got %r" % (TEXTURE_FILTERS, texture_filter))
    if texture_filter == 'trilinear' and face_uvs is None:
        raise ValueError("texture_filter='trilinear' samples a texture image: it needs face_uvs")
    # the shapes, then the device check
    _check_inputs(faces, textures, True, face_light=face_light, vertices=vertices, face_uvs=face_uvs)
    geom, indices = _geometry(faces, vertices)
    if face_light is not None and face_light.dtype != torch.float32:
        face_light = face_light.float()
    cfg = (int(image_size), sigma, gamma, float(near), float(far), float(eps), tuple(bg))
    hw = None
    if face_uvs is not None:
        batch_size = geom.shape[0]
        textures = _batched(textures, batch_size, 3)
        face_uvs = _batched(face_uvs, batch_size, 3)
        if texture_filter == 'trilinear':
            hw = (int(textures.shape[1]), int(textures.shape[2]))
            textures = _MipPyramid.apply(textures)
    else:
        if textures.shape[0] > 1 and textures.stride(0) == 0:
            textures = textures[:1]  # an expanded shared set stays one set
        textures = textures if textures.dtype == torch.float32 else textures.float()
    return _SoftRgbFunction.apply(geom, textures, face_light, face_uvs, indices, cfg, hw)


class _SoftAttrFunction(torch.autograd.Function):
    """autograd node of the soft attribute images: forward = nr_b200_soft_attributes, backward =
    nr_b200_soft_attributes_backward from the saved image, alpha and state.  `geom` / `indices` as _RasterizeFunction;
    `attributes` [B|1,F,3,C] per corner or [B|1,Nv,C] per vertex (1 = shared); `bg` [C] float32 on the device or None."""

    @staticmethod
    def forward(ctx, geom, attributes, indices, bg, per_vertex, cfg):
        lib = _lib.load()
        dev = geom.device
        geom_c = geom.detach().contiguous()
        attr_c = attributes.detach().contiguous()
        B, S, C = geom_c.shape[0], cfg[0], attr_c.shape[-1]
        with torch.cuda.device(dev):
            out = torch.empty((B, C, S, S), dtype=torch.float32, device=dev)
            alpha = torch.empty((B, S, S), dtype=torch.float32, device=dev)
            state = torch.empty((B, 2, S, S), dtype=torch.float32, device=dev)
            a, t, ws = _soft_attr_args(lib, geom_c, indices, attr_c, bg, per_vertex, cfg)
            a.alpha, a.state, t.out = _ptr(alpha), _ptr(state), _ptr(out)
            _lib.check(lib.nr_b200_soft_attributes(ctypes.byref(a), ctypes.byref(t), _stream_ptr(dev)))
        ctx.cfg, ctx.per_vertex = cfg, per_vertex
        ctx.save_for_backward(geom_c, attr_c, indices, bg, out, alpha, state)
        return out, alpha

    @staticmethod
    def backward(ctx, g_out, g_alpha):
        lib = _lib.load()
        geom_c, attr_c, indices, bg, out, alpha, state = ctx.saved_tensors
        dev = geom_c.device
        need_geom, need_attr = ctx.needs_input_grad[:2]
        none = (None,) * 6
        if not (need_geom or need_attr) or (g_out is None and g_alpha is None):
            return none
        g_out = g_out.detach().to(torch.float32).contiguous() if g_out is not None else None
        g_alpha = g_alpha.detach().to(torch.float32).contiguous() if g_alpha is not None else None
        with torch.cuda.device(dev):
            grad_geom = torch.empty_like(geom_c)
            grad_attr = torch.empty_like(attr_c) if need_attr else None
            a, t, ws = _soft_attr_args(lib, geom_c, indices, attr_c, bg, ctx.per_vertex, ctx.cfg)
            a.alpha, a.state, a.grad_alpha = _ptr(alpha), _ptr(state), _ptr(g_alpha)
            t.out, t.grad_out, t.grad_attributes = _ptr(out), _ptr(g_out), _ptr(grad_attr)
            _set_geometry_grad(a, indices, grad_geom)
            _lib.check(lib.nr_b200_soft_attributes_backward(ctypes.byref(a), ctypes.byref(t), _stream_ptr(dev)))
        return grad_geom if need_geom else None, grad_attr, None, None, None, None


def _soft_attr_args(lib, geom_c, indices, attr_c, bg, per_vertex, cfg):
    """nr_b200_soft_rgb_args and nr_b200_soft_attr_args of an attribute call, and the workspace (the soft RGB's)"""
    S, sigma, gamma, near, far = cfg
    a, ws = _soft_rgb_args(lib, geom_c, indices, S, sigma, near, far, gamma, name="rasterize_soft_attributes")
    if per_vertex:
        a.flags |= _lib.NR_ATTR_PER_VERTEX
    if attr_c.shape[0] == 1 and geom_c.shape[0] > 1:
        a.flags |= _lib.NR_ATTR_SHARED
    t = _lib.SoftAttrArgs()
    t.struct_size = ctypes.sizeof(_lib.SoftAttrArgs)
    t.channels = attr_c.shape[-1]
    t.attributes, t.background = _ptr(attr_c), _ptr(bg)
    return a, t, ws


def _device_background(values, device):
    """the background [C] float32 of a sequence of numbers on `device`: copied once per (values, device), then served
    from the small-constant cache of the camera and light parameters, so later calls enqueue no host copy"""
    from . import functional
    import numpy as np
    row = np.asarray(values, dtype=np.float32)
    key = ("soft_background", row.tobytes(), str(device))
    hit = functional._CAMERA_CACHE.get(key)
    if hit is None:
        hit = functional._cache_put(key, torch.from_numpy(row).to(device))
    return hit


def rasterize_soft_attributes(
        faces,
        image_size=DEFAULT_IMAGE_SIZE,
        sigma=DEFAULT_SOFT_SIGMA,
        gamma=DEFAULT_SOFT_GAMMA,
        near=DEFAULT_NEAR,
        far=DEFAULT_FAR,
        *,
        vertices=None,
        vertex_attributes=None,
        face_attributes=None,
        background=None,
        return_alpha=False,
):
    """Soft images [B,C,H,W] of arbitrary per-vertex or per-corner attributes (per-vertex colours, soft depth, normals,
    positions, features), aggregated as rasterize_soft aggregates colour (SoftRas, Liu et al. 2019): every face within
    reach of a pixel adds its perspective-correct interpolant A_j = sum_k l'_k a_k with the weight
    D_j exp((zn_j - zmax) / gamma), against a background term at zn = 1e-3.  Unlike rasterize_attributes, the gradient
    reaches the vertices' x, y and z from every face within reach -- hidden faces and faces a few pixels off their
    target included -- as well as the attributes.  Not in the reference.

    Geometry as rasterize_soft (pass each face once; fill_back copies would count twice).  Exactly one of (keywords, as
    rasterize_attributes): vertex_attributes [Nv,C] / [1|B,Nv,C] (needs indexed geometry) or face_attributes [F,3,C] /
    [1|B,F,3,C].  A batch of 1 (or an expanded stride-0 batch) with a larger geometry batch is one set shared by every
    item; its gradient is the sum over the items.  background: C numbers (or a tensor [C]) for the background term, None
    = zeros; it gets no gradient.  Each channel is computed on its own: channel c equals a one-channel render of it, bit
    for bit.  Deterministic forward.  Returns the image, or (image, alpha) with alpha bit-identical to
    rasterize_soft_silhouettes.  The exact definition is in include/nr_b200.h (nr_b200_soft_attr_args).

    CUDA graphs: a background tensor on the geometry's device is read in place, so a call with one can be captured.  A
    sequence of numbers is copied to the device on its first use and then cached per value and device, as the camera
    and light constants are: the capture of a call with a sequence needs one eager call with the same values before it
    (the usual warm-up does that), and a sequence first seen during a capture, or a background tensor on the host,
    makes a synchronising host-to-device copy, which a capture refuses."""
    sigma, gamma = _positive_number("sigma", sigma), _positive_number("gamma", gamma)
    if not (float(near) < float(far)):
        raise ValueError("near must be < far, got near=%r far=%r" % (near, far))
    if int(image_size) < 1:
        raise ValueError("image_size must be >= 1, got %r" % (image_size,))
    attrs_in = vertex_attributes if vertex_attributes is not None else face_attributes
    bg = None
    if background is not None:
        if isinstance(background, torch.Tensor):
            bg = background.detach().reshape(-1)     # used where it lies: no host round trip
        else:
            try:
                bg = tuple(float(c) for c in background)
            except (TypeError, ValueError):
                raise TypeError("background must be a sequence of numbers or a tensor, got %r" % (background,))
        n = bg.numel() if isinstance(bg, torch.Tensor) else len(bg)
        if isinstance(attrs_in, torch.Tensor) and attrs_in.dim() >= 1 and n != attrs_in.shape[-1]:
            raise ValueError("background must have one value per channel (%d), got %d" % (attrs_in.shape[-1], n))
    attrs, per_vertex = _check_attribute_inputs(faces, vertices, vertex_attributes, face_attributes)  # then the device
    geom, indices = _geometry(faces, vertices)
    attrs = _batched(attrs, geom.shape[0], 2 if per_vertex else 3)  # an expanded shared set: NR_ATTR_SHARED
    if isinstance(bg, torch.Tensor):
        bg = bg.to(device=geom.device, dtype=torch.float32).contiguous()
    elif bg is not None:
        bg = _device_background(bg, geom.device)
    cfg = (int(image_size), sigma, gamma, float(near), float(far))
    image, alpha = _SoftAttrFunction.apply(geom, attrs, indices, bg, per_vertex, cfg)
    return (image, alpha) if return_alpha else image


Fragments = collections.namedtuple("Fragments", ["pix_to_face", "zbuf", "bary_coords", "dists"])
Fragments.__doc__ = """The K nearest faces within reach of every pixel (rasterize_soft_fragments): pix_to_face [B,H,W,K] int64
(-1 = empty slot), zbuf [B,H,W,K], bary_coords [B,H,W,K,3] and dists [B,H,W,K] (+d^2 inside, -d^2 outside)."""


class _SoftFragFunction(torch.autograd.Function):
    """autograd node of the soft fragments: forward = nr_b200_soft_fragments, backward = nr_b200_soft_fragments_backward
    from the saved pix_to_face.  `geom` / `indices` as _RasterizeFunction; cfg = (S, sigma, K, near, far)."""

    @staticmethod
    def forward(ctx, geom, indices, cfg):
        lib = _lib.load()
        dev = geom.device
        geom_c = geom.detach().contiguous()
        B, S, K = geom_c.shape[0], cfg[0], cfg[2]
        with torch.cuda.device(dev):
            p2f = torch.empty((B, S, S, K), dtype=torch.int64, device=dev)
            zbuf = torch.empty((B, S, S, K), dtype=torch.float32, device=dev)
            bary = torch.empty((B, S, S, K, 3), dtype=torch.float32, device=dev)
            dists = torch.empty((B, S, S, K), dtype=torch.float32, device=dev)
            a, t, ws = _soft_frag_args(lib, geom_c, indices, cfg)
            t.pix_to_face, t.zbuf, t.bary, t.dists = _ptr(p2f), _ptr(zbuf), _ptr(bary), _ptr(dists)
            _lib.check(lib.nr_b200_soft_fragments(ctypes.byref(a), ctypes.byref(t), _stream_ptr(dev)))
        ctx.cfg = cfg
        ctx.mark_non_differentiable(p2f)
        ctx.save_for_backward(geom_c, indices, p2f)
        return p2f, zbuf, bary, dists

    @staticmethod
    def backward(ctx, _g_p2f, g_zbuf, g_bary, g_dists):
        if not ctx.needs_input_grad[0] or (g_zbuf is None and g_bary is None and g_dists is None):
            return None, None, None
        lib = _lib.load()
        geom_c, indices, p2f = ctx.saved_tensors
        dev = geom_c.device
        prep = lambda g: g.detach().to(torch.float32).contiguous() if g is not None else None  # noqa: E731
        g_zbuf, g_bary, g_dists = prep(g_zbuf), prep(g_bary), prep(g_dists)
        with torch.cuda.device(dev):
            grad_geom = torch.empty_like(geom_c)
            a, t, ws = _soft_frag_args(lib, geom_c, indices, ctx.cfg)
            t.pix_to_face = _ptr(p2f)
            t.grad_zbuf, t.grad_bary, t.grad_dists = _ptr(g_zbuf), _ptr(g_bary), _ptr(g_dists)
            _set_geometry_grad(a, indices, grad_geom)
            _lib.check(lib.nr_b200_soft_fragments_backward(ctypes.byref(a), ctypes.byref(t), _stream_ptr(dev)))
        return grad_geom, None, None


def _soft_frag_args(lib, geom_c, indices, cfg):
    """nr_b200_soft_rgb_args and nr_b200_soft_frag_args of a fragment call, and the workspace (the soft RGB's)"""
    S, sigma, K, near, far = cfg
    a, ws = _soft_rgb_args(lib, geom_c, indices, S, sigma, near, far, name="rasterize_soft_fragments")
    t = _lib.SoftFragArgs()
    t.struct_size = ctypes.sizeof(_lib.SoftFragArgs)
    t.faces_per_pixel = K
    return a, t, ws


def rasterize_soft_fragments(
        faces,
        image_size=DEFAULT_IMAGE_SIZE,
        sigma=DEFAULT_SOFT_SIGMA,
        faces_per_pixel=8,
        near=DEFAULT_NEAR,
        far=DEFAULT_FAR,
        *,
        vertices=None,
):
    """Soft fragments (PyTorch3D's MeshRasterizer with faces_per_pixel = K and a blur radius): for every pixel the K
    nearest faces within reach of it -- inside, or within the soft silhouettes' cut-off reach sqrt(sigma ln((1-eps)/eps))
    -- ordered by their perspective-correct depth (then by face index), each with its depth, its barycentrics and its
    signed squared distance.  Shade them in torch with any shader: interpolate_soft_fragments interpolates per-corner
    or per-vertex attributes at them in CUDA (functional.interpolate_face_attributes in torch), and
    w = sigmoid(dists / sigma) is SoftRas's coverage probability; blend_soft_fragments blends the shaded slots by
    SoftRas's depth softmax in CUDA.  Not in the reference.

    Geometry as rasterize_soft_silhouettes (faces [B,F,3,3], or `vertices` [B,Nv,3] with integer faces [F,3] /
    [1|B,F,3]).  A face takes part when its three vertex depths lie in [near, far]; a zero-area face is no fragment.
    1 <= faces_per_pixel <= 32.  Returns Fragments(pix_to_face [B,H,W,K] int64, the face index within its item;
    zbuf [B,H,W,K]; bary_coords [B,H,W,K,3], perspective-correct, clipped and renormalised; dists [B,H,W,K], +d^2
    inside and -d^2 outside in squared NDC units -- the opposite sign of PyTorch3D's).  Empty slots hold -1 in every
    field.  Row 0 is at the top.  Deterministic.  Gradients flow from zbuf, bary_coords and dists into the vertices'
    x, y and z with the selection held fixed.  The exact definition is in include/nr_b200.h (nr_b200_soft_frag_args)."""
    sigma = _positive_number("sigma", sigma)
    if isinstance(faces_per_pixel, bool) or not hasattr(faces_per_pixel, "__index__"):
        raise TypeError("faces_per_pixel must be an integer, got %r" % (faces_per_pixel,))
    K = faces_per_pixel.__index__()
    if not 1 <= K <= _lib.SOFT_MAX_FACES_PER_PIXEL:
        raise ValueError("faces_per_pixel must be in [1, %d], got %r" % (_lib.SOFT_MAX_FACES_PER_PIXEL, faces_per_pixel))
    if not (float(near) < float(far)):
        raise ValueError("near must be < far, got near=%r far=%r" % (near, far))
    if int(image_size) < 1:
        raise ValueError("image_size must be >= 1, got %r" % (image_size,))
    _check_inputs(faces, None, False, vertices=vertices)  # the geometry, then the device check
    geom, indices = _geometry(faces, vertices)
    return Fragments(*_SoftFragFunction.apply(geom, indices, (int(image_size), sigma, K, float(near), float(far))))


class _BlendFunction(torch.autograd.Function):
    """autograd node of the soft blend: forward = nr_b200_blend_fragments, backward = nr_b200_blend_fragments_backward
    from the saved inputs and out.  cfg = (sigma, gamma, near, far)."""

    @staticmethod
    def forward(ctx, zbuf, dists, colors, p2f, bg, cfg):
        lib = _lib.load()
        dev = colors.device
        B, H, W, K, C = colors.shape
        with torch.cuda.device(dev):
            out = torch.empty((B, C, H, W), dtype=torch.float32, device=dev)
            alpha = torch.empty((B, H, W), dtype=torch.float32, device=dev)
            a = _blend_args(zbuf, dists, colors, p2f, bg, cfg)
            a.out, a.alpha = _ptr(out), _ptr(alpha)
            _lib.check(lib.nr_b200_blend_fragments(ctypes.byref(a), _stream_ptr(dev)))
        ctx.cfg = cfg
        ctx.save_for_backward(zbuf, dists, colors, p2f, bg, out)
        return out, alpha

    @staticmethod
    def backward(ctx, g_out, g_alpha):
        want = ctx.needs_input_grad[:3]
        if not any(want) or (g_out is None and g_alpha is None):
            return None, None, None, None, None, None
        lib = _lib.load()
        zbuf, dists, colors, p2f, bg, out = ctx.saved_tensors
        dev = colors.device
        prep = lambda g: g.detach().to(torch.float32).contiguous() if g is not None else None  # noqa: E731
        g_out, g_alpha = prep(g_out), prep(g_alpha)
        with torch.cuda.device(dev):
            gz = torch.empty_like(zbuf) if want[0] else None
            gd = torch.empty_like(dists) if want[1] else None
            gc = torch.empty_like(colors) if want[2] else None
            a = _blend_args(zbuf, dists, colors, p2f, bg, ctx.cfg)
            a.out, a.grad_out, a.grad_alpha = _ptr(out), _ptr(g_out), _ptr(g_alpha)
            a.grad_zbuf, a.grad_dists, a.grad_colors = _ptr(gz), _ptr(gd), _ptr(gc)
            _lib.check(lib.nr_b200_blend_fragments_backward(ctypes.byref(a), _stream_ptr(dev)))
        return gz, gd, gc, None, None, None


def _blend_args(zbuf, dists, colors, p2f, bg, cfg):
    B, H, W, K, C = colors.shape
    a = _lib.BlendArgs()
    a.struct_size = ctypes.sizeof(_lib.BlendArgs)
    a.batch_size, a.height, a.width, a.faces_per_pixel, a.channels = B, H, W, K, C
    a.sigma, a.gamma, a.near_, a.far_ = cfg
    a.pix_to_face, a.zbuf, a.dists, a.colors = _ptr(p2f), _ptr(zbuf), _ptr(dists), _ptr(colors)
    a.background = _ptr(bg) if bg.numel() else None
    return a


def blend_soft_fragments(fragments, colors, sigma, gamma, near=DEFAULT_NEAR, far=DEFAULT_FAR, background=None):
    """SoftRas's depth-softmax blend of per-slot colours over soft fragments, in CUDA: the step a fragment pipeline ends
    with ("shade in torch, blend on the GPU").  fragments: a Fragments of rasterize_soft_fragments (pix_to_face, zbuf
    and dists are read; bary_coords is not), colors [B,H,W,K,C] the colour of every slot (any torch shader's output,
    e.g. interpolate_soft_fragments or functional.interpolate_face_attributes of the fragments).  Per pixel, over the valid slots (pix_to_face >= 0,
    in any order), with D_k = sigmoid(dists_k / sigma), zb = far - 1e-3 (far - near) and zref = min(zb, min_k zbuf_k):
      w_k = D_k exp((zref - zbuf_k) / ((far - near) gamma)),  w_b = exp((zref - zb) / ((far - near) gamma)),
      image_c = (sum_k w_k colors_kc + w_b background_c) / (sum_k w_k + w_b),  alpha = 1 - prod_k (1 - D_k).
    sigma and gamma are required: sigma must be the one the fragments were rasterized with (dists / sigma is their
    coverage), and no default could know it.  Returns (image [B,C,H,W], alpha [B,H,W]).  With the fragments' sigma and
    every pixel's candidate count below K,
    blend_soft_fragments(frag, interpolate_face_attributes(frag.pix_to_face, frag.bary_coords, a)) is
    rasterize_soft_attributes(..., face_attributes=a) up to fp32 rounding.  background: C numbers or a [C] tensor
    (default zeros; no gradient).  Gradients flow into colors and, through zbuf and dists, on into the fragments'
    vertices.  Deterministic, forward and backward.  Not in the reference; PyTorch3D's softmax_rgb_blend differs in the
    sign of dists, the background level (1e-10 there) and the layout (RGBA channels-last there).  The exact definition is
    in include/nr_b200.h (nr_b200_blend_args)."""
    if not isinstance(fragments, tuple) or len(fragments) != 4:
        raise TypeError("fragments must be a Fragments (pix_to_face, zbuf, bary_coords, dists)")
    p2f, zbuf, _, dists = fragments
    for name, t in (("pix_to_face", p2f), ("zbuf", zbuf), ("dists", dists), ("colors", colors)):
        if not isinstance(t, torch.Tensor):
            raise TypeError("%s must be a torch.Tensor, got %s" % (name, type(t).__name__))
    if p2f.dtype != torch.int64 or p2f.dim() != 4:
        raise ValueError("pix_to_face must be an int64 tensor [B,H,W,K], got %s %s" % (p2f.dtype, tuple(p2f.shape)))
    for name, t in (("zbuf", zbuf), ("dists", dists)):
        if not t.dtype.is_floating_point or tuple(t.shape) != tuple(p2f.shape):
            raise ValueError("%s must be a floating tensor of shape %s, got %s %s"
                             % (name, tuple(p2f.shape), t.dtype, tuple(t.shape)))
    if not colors.dtype.is_floating_point or colors.dim() != 5 or tuple(colors.shape[:4]) != tuple(p2f.shape):
        raise ValueError("colors must be a floating tensor [B,H,W,K,C] with [B,H,W,K] = %s, got %s %s"
                         % (tuple(p2f.shape), colors.dtype, tuple(colors.shape)))
    B, H, W, K, C = colors.shape
    if min(B, H, W, K, C) < 1:
        raise ValueError("every size of colors must be >= 1, got %s" % (tuple(colors.shape),))
    if K > _lib.SOFT_MAX_FACES_PER_PIXEL:
        raise ValueError("at most %d slots per pixel, got %d" % (_lib.SOFT_MAX_FACES_PER_PIXEL, K))
    sigma = _positive_number("sigma", sigma)
    gamma = _positive_number("gamma", gamma)
    near, far = float(near), float(far)
    if not (math.isfinite(near) and math.isfinite(far) and near < far):
        raise ValueError("near and far must be finite with near < far, got near=%r far=%r" % (near, far))
    bg = background
    if bg is not None:
        if isinstance(bg, torch.Tensor):
            if bg.dim() != 1 or bg.shape[0] != C or not bg.dtype.is_floating_point:
                raise ValueError("background must be a floating tensor [%d], got %s %s" % (C, bg.dtype, tuple(bg.shape)))
        else:
            try:
                bg = [float(v) for v in bg]
            except (TypeError, ValueError):
                raise TypeError("background must be a sequence of %d numbers or a tensor, got %r" % (C, background))
            if len(bg) != C:
                raise ValueError("background must have %d values, got %d" % (C, len(bg)))
    dev = colors.device
    for name, t in (("pix_to_face", p2f), ("zbuf", zbuf), ("dists", dists)):
        if t.device != dev:
            raise ValueError("%s is on %s, colors on %s" % (name, t.device, dev))
    if isinstance(bg, torch.Tensor) and bg.device != dev:
        raise ValueError("background is on %s, colors on %s" % (bg.device, dev))
    if not colors.is_cuda:
        raise NotImplementedError("neural_renderer_b200 has no CPU implementation (inputs must be CUDA tensors)")
    if bg is None:
        bg = torch.zeros(0, dtype=torch.float32, device=dev)
    elif isinstance(bg, torch.Tensor):
        bg = bg.detach().to(torch.float32).contiguous()
    else:
        bg = _device_background(bg, dev)
    f32 = lambda t: t.to(torch.float32).contiguous()  # noqa: E731
    return _BlendFunction.apply(f32(zbuf), f32(dists), f32(colors), p2f.contiguous(), bg, (sigma, gamma, near, far))


class _FragInterpFunction(torch.autograd.Function):
    """autograd node of the soft interpolation of fragments: forward = nr_b200_interpolate_fragments, backward =
    nr_b200_interpolate_fragments_backward from the saved inputs.  `attributes` [B|1,F,3,C] per corner or [B|1,Nv,C]
    per vertex (1 = shared), `indices` int32 [F,3] / [B|1,F,3] or None; cfg = (flags, F)."""

    @staticmethod
    def forward(ctx, bary, attributes, p2f, indices, cfg):
        lib = _lib.load()
        dev = bary.device
        B, H, W, K = p2f.shape
        with torch.cuda.device(dev):
            out = torch.empty((B, H, W, K, attributes.shape[-1]), dtype=torch.float32, device=dev)
            a = _frag_interp_args(bary, attributes, p2f, indices, cfg)
            a.out = _ptr(out)
            _lib.check(lib.nr_b200_interpolate_fragments(ctypes.byref(a), _stream_ptr(dev)))
        ctx.cfg = cfg
        ctx.save_for_backward(bary, attributes, p2f, indices)
        return out

    @staticmethod
    def backward(ctx, g_out):
        want_bary, want_attr = ctx.needs_input_grad[:2]
        if not (want_bary or want_attr) or g_out is None:
            return None, None, None, None, None
        lib = _lib.load()
        bary, attributes, p2f, indices = ctx.saved_tensors
        dev = bary.device
        g_out = g_out.detach().to(torch.float32).contiguous()
        with torch.cuda.device(dev):
            gb = torch.empty_like(bary) if want_bary else None
            ga = torch.empty_like(attributes) if want_attr else None
            a = _frag_interp_args(bary, attributes, p2f, indices, ctx.cfg)
            a.grad_out, a.grad_bary, a.grad_attributes = _ptr(g_out), _ptr(gb), _ptr(ga)
            _lib.check(lib.nr_b200_interpolate_fragments_backward(ctypes.byref(a), _stream_ptr(dev)))
        return gb, ga, None, None, None


def _frag_interp_args(bary, attributes, p2f, indices, cfg):
    flags, F = cfg
    B, H, W, K = p2f.shape
    a = _lib.FragInterpArgs()
    a.struct_size = ctypes.sizeof(_lib.FragInterpArgs)
    a.flags = flags
    a.batch_size, a.height, a.width, a.faces_per_pixel, a.channels = B, H, W, K, attributes.shape[-1]
    a.num_faces = F
    a.pix_to_face, a.bary, a.attributes = _ptr(p2f), _ptr(bary), _ptr(attributes)
    if indices is not None:
        a.face_indices, a.num_vertices = _ptr(indices), attributes.shape[-2]
    return a


def interpolate_soft_fragments(fragments, face_attributes=None, *, vertex_attributes=None, faces=None):
    """Per-corner or per-vertex attributes interpolated at soft fragments, in CUDA: the step every shader over fragments
    starts with (colours, normals, positions, UVs, features).  fragments: a Fragments of rasterize_soft_fragments
    (pix_to_face and bary_coords are read).  Exactly one of face_attributes [F,3,C] / [1|B,F,3,C] (per corner) and
    vertex_attributes [Nv,C] / [1|B,Nv,C] (per vertex, with the integer faces [F,3] / [1|B,F,3] that index them; a
    corner whose index lies outside [0, Nv) reads zeros).  A batch of 1 (or an expanded stride-0 batch) is one set
    shared by every item; its gradient is the sum over the items.  Per slot with f = pix_to_face in [0, F) and
    l = bary_coords: out[b,y,x,k,c] = fma(l_2, a_2c, fma(l_1, a_1c, l_0 a_0c)); any other f (-1 included) is an empty
    slot and gets exactly 0.  Returns [B,H,W,K,C] float32, the layout blend_soft_fragments reads.

    The same values as functional.interpolate_face_attributes (on the gathered corners, for per-vertex attributes) up
    to fp32 rounding, without its [B,H,W,K,C] temporaries and index_select backward, and without materialising
    [B,F,3,C] corners for per-vertex attributes.  Gradients flow into the attributes and into fragments.bary_coords,
    and through bary_coords on into the vertices of rasterize_soft_fragments.  Each channel is computed on its own
    (channel c equals a one-channel call on it, bit for bit), a per-vertex call equals the per-corner call on the
    gathered corners and a shared set equals the same set expanded, bit for bit; the forward and the barycentric
    gradient are deterministic.  Not in the reference.  The exact definition is in include/nr_b200.h
    (nr_b200_frag_interp_args)."""
    if not isinstance(fragments, tuple) or len(fragments) != 4:
        raise TypeError("fragments must be a Fragments (pix_to_face, zbuf, bary_coords, dists)")
    p2f, _, bary, _ = fragments
    for name, t in (("pix_to_face", p2f), ("bary_coords", bary)):
        if not isinstance(t, torch.Tensor):
            raise TypeError("%s must be a torch.Tensor, got %s" % (name, type(t).__name__))
    if p2f.dtype != torch.int64 or p2f.dim() != 4:
        raise ValueError("pix_to_face must be an int64 tensor [B,H,W,K], got %s %s" % (p2f.dtype, tuple(p2f.shape)))
    if not bary.dtype.is_floating_point or tuple(bary.shape) != tuple(p2f.shape) + (3,):
        raise ValueError("bary_coords must be a floating tensor of shape %s, got %s %s"
                         % (tuple(p2f.shape) + (3,), bary.dtype, tuple(bary.shape)))
    B, H, W, K = p2f.shape
    if min(B, H, W, K) < 1:
        raise ValueError("every size of pix_to_face must be >= 1, got %s" % (tuple(p2f.shape),))
    if K > _lib.SOFT_MAX_FACES_PER_PIXEL:
        raise ValueError("at most %d slots per pixel, got %d" % (_lib.SOFT_MAX_FACES_PER_PIXEL, K))
    if (face_attributes is None) == (vertex_attributes is None):
        raise TypeError("give exactly one of face_attributes and vertex_attributes=")
    per_vertex = vertex_attributes is not None
    attrs = vertex_attributes if per_vertex else face_attributes
    name = "vertex_attributes" if per_vertex else "face_attributes"
    if not isinstance(attrs, torch.Tensor) or not attrs.is_floating_point():
        raise TypeError("%s must be a floating point torch.Tensor" % name)
    rows = 1 if per_vertex else 2                                    # [Nv] or [F,3] before the channels
    if attrs.dim() not in (rows + 1, rows + 2) or (attrs.dim() == rows + 2 and attrs.shape[0] not in (1, B)) \
            or (not per_vertex and attrs.shape[-2] != 3) or attrs.shape[-1] < 1 or attrs.shape[-rows - 1] < 1:
        want = "[Nv,C] or [1|B,Nv,C]" if per_vertex else "[F,3,C] or [1|B,F,3,C]"
        raise ValueError("%s must have shape %s with C >= 1 (B = %d), got %s" % (name, want, B, tuple(attrs.shape)))
    if per_vertex:
        if faces is None:
            raise ValueError("vertex_attributes need the integer faces [F,3] / [1|B,F,3] that index them")
        if not isinstance(faces, torch.Tensor) or faces.dtype.is_floating_point or faces.dtype == torch.bool:
            raise TypeError("faces must be an integer torch.Tensor")
        if faces.dim() not in (2, 3) or faces.shape[-1] != 3 or faces.shape[-2] < 1 \
                or (faces.dim() == 3 and faces.shape[0] not in (1, B)):
            raise ValueError("faces must have shape [F,3] or [1|B,F,3] (B = %d), got %s" % (B, tuple(faces.shape)))
        F = faces.shape[-2]
    else:
        if faces is not None:
            raise TypeError("faces is only read with vertex_attributes")
        F = attrs.shape[-3]
    dev = bary.device
    for n, t in (("pix_to_face", p2f), (name, attrs), ("faces", faces)):
        if t is not None and t.device != dev:
            raise ValueError("%s is on %s, bary_coords on %s" % (n, t.device, dev))
    if not bary.is_cuda:
        raise NotImplementedError("neural_renderer_b200 has no CPU implementation (inputs must be CUDA tensors)")
    attrs = _batched(attrs, B, rows + 1)                              # an expanded shared set: NR_ATTR_SHARED
    flags = _lib.NR_ATTR_SHARED if attrs.shape[0] == 1 and B > 1 else 0
    indices = None
    if per_vertex:
        flags |= _lib.NR_ATTR_PER_VERTEX
        indices = _index_set(faces)
        if indices.dim() == 2 or (indices.shape[0] == 1 and B > 1):
            flags |= _lib.NR_INDICES_SHARED
    return _FragInterpFunction.apply(bary.to(torch.float32).contiguous(), attrs.contiguous(), p2f.contiguous(), indices,
                                     (flags, F))


class Rasterize(object):
    """The reference's function object (rasterize.py:19-64): `Rasterize(image_size, near, far, eps,
    background_color, return_rgb, return_alpha, return_depth)(faces[, textures]) -> (rgb, alpha, depth)` with the
    reference's internal conventions (NHWC rgb, rows NOT flipped, None for outputs not requested).  After the call
    `face_index_map` / `weight_map` hold the raster maps in those same conventions (as the reference instance does)."""

    def __init__(self, image_size, near, far, eps, background_color, return_rgb=False, return_alpha=False,
                 return_depth=False):
        if not any((return_rgb, return_alpha, return_depth)):
            raise Exception("nothing to draw")
        self.image_size = image_size
        self.near = near
        self.far = far
        self.eps = eps
        self.background_color = background_color
        self.return_rgb = return_rgb
        self.return_alpha = return_alpha
        self.return_depth = return_depth
        self.face_index_map = None
        self.weight_map = None

    def __call__(self, faces, textures=None):
        rgb, alpha, depth, fim, wmap = _run(faces, textures, self.image_size, False, self.near, self.far, self.eps,
                                            self.background_color, self.return_rgb, self.return_alpha,
                                            self.return_depth)
        self.face_index_map = fim.flip(1)
        self.weight_map = wmap.permute(0, 2, 3, 1).flip(1)
        rgb = rgb.permute(0, 2, 3, 1).flip(1) if self.return_rgb else None
        alpha = alpha.flip(1) if self.return_alpha else None
        depth = depth.flip(1) if self.return_depth else None
        return rgb, alpha, depth
