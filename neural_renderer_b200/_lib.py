"""ctypes binding of libnr_b200.so -- the C ABI declared in include/nr_b200.h.

There is no CPU fallback and no other backend: if the CUDA library is missing the import of any hot-path entry
point fails loudly (the reference likewise raises NotImplementedError for CPU arrays, rasterize.py:893-897).
"""
from __future__ import annotations

import ctypes
import os

PKG_DIR = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("NR_B200_LIB", os.path.join(PKG_DIR, "libnr_b200.so"))  # override: kernel A/B experiments

NR_OK = 0
NR_RETURN_RGB = 1
NR_RETURN_ALPHA = 2
NR_RETURN_DEPTH = 4
NR_ANTI_ALIASING = 8
NR_BG_PER_BATCH = 16
NR_TEX_Z_BATCH0 = 32
NR_GRAD_ACCUMULATE = 64
NR_CAM_PERSPECTIVE = 0x100
NR_TEX_FILL_BACK = 0x400
NR_CAM_SHARED = 0x200
NR_FACES_INDEXED = 0x800
NR_INDICES_SHARED = 0x1000
NR_TEX_SHARED = 0x2000
NR_BWD_PART_TEXTURES = 0x4000
NR_BWD_PART_FACES = 0x8000
NR_FWD_STAGE_TEXTURES = 0x10000
NR_TEX_UV = 0x20000
NR_UV_SHARED = 0x40000
NR_TEX_MIPMAP = 0x80000
NR_ATTR_PER_VERTEX = 0x100000
NR_ATTR_SHARED = 0x200000
NR_GRAD_INTERIOR = 0x400000

ABI_VERSION = 4

# every symbol include/nr_b200.h declares
EXPORTED_SYMBOLS = (
    "nr_b200_abi_version",
    "nr_b200_error_string",
    "nr_b200_forward_workspace_bytes",
    "nr_b200_backward_workspace_bytes",
    "nr_b200_forward",
    "nr_b200_backward",
    "nr_b200_backward_corner_light",
    "nr_b200_forward_phong",
    "nr_b200_backward_phong",
    "nr_b200_forward_lights",
    "nr_b200_backward_lights",
    "nr_b200_forward_sh",
    "nr_b200_backward_sh",
    "nr_b200_forward_normal_map",
    "nr_b200_backward_normal_map",
    "nr_b200_forward_specular_map",
    "nr_b200_backward_specular_map",
    "nr_b200_interpolate",
    "nr_b200_interpolate_backward",
    "nr_b200_soft_workspace_bytes",
    "nr_b200_soft_silhouettes",
    "nr_b200_soft_silhouettes_backward",
    "nr_b200_soft_rgb_workspace_bytes",
    "nr_b200_soft_rgb",
    "nr_b200_soft_rgb_backward",
    "nr_b200_soft_rgb_uv",
    "nr_b200_soft_rgb_uv_backward",
    "nr_b200_soft_attributes",
    "nr_b200_soft_attributes_backward",
    "nr_b200_soft_fragments",
    "nr_b200_soft_fragments_backward",
    "nr_b200_vertices_to_faces",
    "nr_b200_vertices_to_faces_backward",
    "nr_b200_camera_transform",
    "nr_b200_camera_transform_backward",
    "nr_b200_face_lighting",
    "nr_b200_face_lighting_backward",
    "nr_b200_vertex_normals_workspace_bytes",
    "nr_b200_vertex_normals",
    "nr_b200_vertex_normals_backward",
    "nr_b200_corner_lighting",
    "nr_b200_corner_lighting_backward",
    "nr_b200_corner_shading",
    "nr_b200_corner_shading_backward",
    "nr_b200_bake_textures",
    "nr_b200_mip_texels",
    "nr_b200_mip_build",
    "nr_b200_mip_collapse",
    "nr_b200_last_launch_count",
    "nr_b200_set_profiling",
    "nr_b200_read_profile",
)


class ForwardArgs(ctypes.Structure):
    _fields_ = [
        ("struct_size", ctypes.c_uint32), ("flags", ctypes.c_uint32),
        ("batch_size", ctypes.c_int32), ("num_faces", ctypes.c_int32),
        ("raster_size", ctypes.c_int32), ("texture_size", ctypes.c_int32),
        ("near_", ctypes.c_double), ("far_", ctypes.c_double), ("eps", ctypes.c_double),
        ("background", ctypes.c_float * 3), ("_pad0", ctypes.c_float),
        ("faces", ctypes.c_void_p), ("textures", ctypes.c_void_p), ("background_batch", ctypes.c_void_p),
        ("face_index_map", ctypes.c_void_p), ("weight_map", ctypes.c_void_p), ("depth_map", ctypes.c_void_p),
        ("rgb_map", ctypes.c_void_p), ("alpha_map", ctypes.c_void_p),
        ("out_rgb", ctypes.c_void_p), ("out_alpha", ctypes.c_void_p), ("out_depth", ctypes.c_void_p),
        ("workspace", ctypes.c_void_p), ("workspace_bytes", ctypes.c_size_t),
        ("face_light", ctypes.c_void_p),
        ("vertices", ctypes.c_void_p), ("face_indices", ctypes.c_void_p),
        ("num_vertices", ctypes.c_int32), ("_pad1", ctypes.c_int32),
        ("face_uvs", ctypes.c_void_p), ("texture_height", ctypes.c_int32), ("texture_width", ctypes.c_int32),
        ("corner_light", ctypes.c_void_p),  # appended within ABI 4; struct_size = ForwardArgs.corner_light.offset omits it
    ]


class BackwardArgs(ctypes.Structure):
    _fields_ = [
        ("struct_size", ctypes.c_uint32), ("flags", ctypes.c_uint32),
        ("batch_size", ctypes.c_int32), ("num_faces", ctypes.c_int32),
        ("raster_size", ctypes.c_int32), ("texture_size", ctypes.c_int32),
        ("eps", ctypes.c_double),
        ("faces", ctypes.c_void_p), ("textures", ctypes.c_void_p),
        ("face_index_map", ctypes.c_void_p), ("weight_map", ctypes.c_void_p), ("depth_map", ctypes.c_void_p),
        ("rgb_map", ctypes.c_void_p),
        ("grad_rgb", ctypes.c_void_p), ("grad_alpha", ctypes.c_void_p), ("grad_depth", ctypes.c_void_p),
        ("grad_faces", ctypes.c_void_p), ("grad_textures", ctypes.c_void_p),
        ("workspace", ctypes.c_void_p), ("workspace_bytes", ctypes.c_size_t),
        ("face_light", ctypes.c_void_p), ("grad_face_light", ctypes.c_void_p),
        ("vertices", ctypes.c_void_p), ("face_indices", ctypes.c_void_p), ("grad_vertices", ctypes.c_void_p),
        ("num_vertices", ctypes.c_int32), ("_pad1", ctypes.c_int32),
        ("face_uvs", ctypes.c_void_p), ("texture_height", ctypes.c_int32), ("texture_width", ctypes.c_int32),
        ("grad_face_uvs", ctypes.c_void_p),  # appended within ABI 4; struct_size = BackwardArgs.grad_face_uvs.offset omits it
    ]


class PhongArgs(ctypes.Structure):
    _fields_ = [
        ("struct_size", ctypes.c_uint32), ("shading_batch", ctypes.c_int32),
        ("params_batch", ctypes.c_int32), ("_pad0", ctypes.c_int32),
        ("corner_shading", ctypes.c_void_p), ("params", ctypes.c_void_p),
        ("grad_corner_shading", ctypes.c_void_p), ("grad_params", ctypes.c_void_p),
    ]


class LightsArgs(ctypes.Structure):
    _fields_ = [
        ("struct_size", ctypes.c_uint32), ("lights_batch", ctypes.c_int32),
        ("num_lights", ctypes.c_int32), ("_pad0", ctypes.c_int32),
        ("lights", ctypes.c_void_p), ("grad_lights", ctypes.c_void_p),
    ]


class ShArgs(ctypes.Structure):
    _fields_ = [
        ("struct_size", ctypes.c_uint32), ("sh_batch", ctypes.c_int32),
        ("sh", ctypes.c_void_p), ("grad_sh", ctypes.c_void_p),
    ]


class NormalMapArgs(ctypes.Structure):
    _fields_ = [
        ("struct_size", ctypes.c_uint32), ("map_batch", ctypes.c_int32), ("tangent_batch", ctypes.c_int32),
        ("map_height", ctypes.c_int32), ("map_width", ctypes.c_int32), ("_pad0", ctypes.c_int32),
        ("normal_map", ctypes.c_void_p), ("corner_tangents", ctypes.c_void_p),
        ("grad_normal_map", ctypes.c_void_p), ("grad_corner_tangents", ctypes.c_void_p),
    ]


class SpecularMapArgs(ctypes.Structure):
    _fields_ = [
        ("struct_size", ctypes.c_uint32), ("map_batch", ctypes.c_int32),
        ("map_height", ctypes.c_int32), ("map_width", ctypes.c_int32),
        ("specular_map", ctypes.c_void_p), ("grad_specular_map", ctypes.c_void_p),
    ]


class InterpolateArgs(ctypes.Structure):
    _fields_ = [
        ("struct_size", ctypes.c_uint32), ("flags", ctypes.c_uint32),
        ("batch_size", ctypes.c_int32), ("num_faces", ctypes.c_int32),
        ("raster_size", ctypes.c_int32), ("channels", ctypes.c_int32),
        ("faces", ctypes.c_void_p), ("vertices", ctypes.c_void_p), ("face_indices", ctypes.c_void_p),
        ("num_vertices", ctypes.c_int32), ("_pad0", ctypes.c_int32),
        ("face_index_map", ctypes.c_void_p), ("weight_map", ctypes.c_void_p),
        ("attributes", ctypes.c_void_p), ("out", ctypes.c_void_p),
        ("grad_out", ctypes.c_void_p), ("grad_attributes", ctypes.c_void_p),
        ("grad_faces", ctypes.c_void_p), ("grad_vertices", ctypes.c_void_p),
    ]


class SoftArgs(ctypes.Structure):
    _fields_ = [
        ("struct_size", ctypes.c_uint32), ("flags", ctypes.c_uint32),
        ("batch_size", ctypes.c_int32), ("num_faces", ctypes.c_int32),
        ("image_size", ctypes.c_int32), ("num_vertices", ctypes.c_int32),
        ("sigma", ctypes.c_float), ("near_", ctypes.c_float), ("far_", ctypes.c_float), ("_pad0", ctypes.c_int32),
        ("faces", ctypes.c_void_p), ("vertices", ctypes.c_void_p), ("face_indices", ctypes.c_void_p),
        ("alpha", ctypes.c_void_p), ("grad_alpha", ctypes.c_void_p),
        ("grad_faces", ctypes.c_void_p), ("grad_vertices", ctypes.c_void_p),
        ("workspace", ctypes.c_void_p), ("workspace_bytes", ctypes.c_size_t),
    ]


SOFT_EPS = 1e-4  # NR_SOFT_EPS: an outside face contributes while its D >= SOFT_EPS


class SoftRgbArgs(ctypes.Structure):
    _fields_ = [
        ("struct_size", ctypes.c_uint32), ("flags", ctypes.c_uint32),
        ("batch_size", ctypes.c_int32), ("num_faces", ctypes.c_int32),
        ("image_size", ctypes.c_int32), ("num_vertices", ctypes.c_int32), ("texture_size", ctypes.c_int32),
        ("sigma", ctypes.c_float), ("gamma", ctypes.c_float), ("near_", ctypes.c_float), ("far_", ctypes.c_float),
        ("eps", ctypes.c_float), ("background", ctypes.c_float * 3), ("_pad0", ctypes.c_int32),
        ("faces", ctypes.c_void_p), ("vertices", ctypes.c_void_p), ("face_indices", ctypes.c_void_p),
        ("textures", ctypes.c_void_p), ("face_light", ctypes.c_void_p),
        ("rgb", ctypes.c_void_p), ("alpha", ctypes.c_void_p), ("state", ctypes.c_void_p),
        ("grad_rgb", ctypes.c_void_p), ("grad_alpha", ctypes.c_void_p),
        ("grad_faces", ctypes.c_void_p), ("grad_vertices", ctypes.c_void_p),
        ("grad_textures", ctypes.c_void_p), ("grad_face_light", ctypes.c_void_p),
        ("workspace", ctypes.c_void_p), ("workspace_bytes", ctypes.c_size_t),
    ]


class SoftUvArgs(ctypes.Structure):
    _fields_ = [
        ("struct_size", ctypes.c_uint32), ("texture_height", ctypes.c_int32), ("texture_width", ctypes.c_int32),
        ("_pad0", ctypes.c_int32), ("face_uvs", ctypes.c_void_p), ("grad_face_uvs", ctypes.c_void_p),
    ]


class SoftAttrArgs(ctypes.Structure):
    _fields_ = [
        ("struct_size", ctypes.c_uint32), ("channels", ctypes.c_int32),
        ("attributes", ctypes.c_void_p), ("background", ctypes.c_void_p), ("out", ctypes.c_void_p),
        ("grad_out", ctypes.c_void_p), ("grad_attributes", ctypes.c_void_p),
    ]


class SoftFragArgs(ctypes.Structure):
    _fields_ = [
        ("struct_size", ctypes.c_uint32), ("faces_per_pixel", ctypes.c_int32),
        ("pix_to_face", ctypes.c_void_p), ("zbuf", ctypes.c_void_p), ("bary", ctypes.c_void_p), ("dists", ctypes.c_void_p),
        ("grad_zbuf", ctypes.c_void_p), ("grad_bary", ctypes.c_void_p), ("grad_dists", ctypes.c_void_p),
    ]


SOFT_MAX_FACES_PER_PIXEL = 32  # the largest K of nr_b200_soft_fragments

SOFT_BG_DEPTH = 1e-3  # NR_SOFT_BG_DEPTH: the normalised depth of the soft RGB's background term


_LIB = None


class LibraryMissing(ImportError):
    pass


def load():
    """dlopen libnr_b200.so; raises LibraryMissing (never falls back) when it has not been built."""
    global _LIB
    if _LIB is not None:
        return _LIB
    if not os.path.exists(LIB_PATH):
        raise LibraryMissing(
            "%s not found: build it with `python -m neural_renderer_b200.build` (or __graft_entry__.build()); "
            "this package has no CPU or pure-PyTorch fallback" % LIB_PATH)
    lib = ctypes.CDLL(LIB_PATH)
    lib.nr_b200_abi_version.restype = ctypes.c_int
    lib.nr_b200_error_string.restype = ctypes.c_char_p
    lib.nr_b200_error_string.argtypes = [ctypes.c_int]
    for name in ("nr_b200_forward_workspace_bytes", "nr_b200_backward_workspace_bytes"):
        fn = getattr(lib, name)
        fn.restype = ctypes.c_size_t
        fn.argtypes = [ctypes.c_int32, ctypes.c_int32, ctypes.c_int32, ctypes.c_int32, ctypes.c_uint32]
    lib.nr_b200_forward.restype = ctypes.c_int
    lib.nr_b200_forward.argtypes = [ctypes.POINTER(ForwardArgs), ctypes.c_void_p]
    lib.nr_b200_backward.restype = ctypes.c_int
    lib.nr_b200_backward.argtypes = [ctypes.POINTER(BackwardArgs), ctypes.c_void_p]
    lib.nr_b200_backward_corner_light.restype = ctypes.c_int
    lib.nr_b200_backward_corner_light.argtypes = [ctypes.POINTER(BackwardArgs), ctypes.c_void_p, ctypes.c_void_p,
                                                  ctypes.c_void_p]
    lib.nr_b200_forward_phong.restype = ctypes.c_int
    lib.nr_b200_forward_phong.argtypes = [ctypes.POINTER(ForwardArgs), ctypes.POINTER(PhongArgs), ctypes.c_void_p]
    lib.nr_b200_backward_phong.restype = ctypes.c_int
    lib.nr_b200_backward_phong.argtypes = [ctypes.POINTER(BackwardArgs), ctypes.POINTER(PhongArgs), ctypes.c_void_p]
    lib.nr_b200_forward_lights.restype = ctypes.c_int
    lib.nr_b200_forward_lights.argtypes = [ctypes.POINTER(ForwardArgs), ctypes.POINTER(PhongArgs), ctypes.POINTER(LightsArgs),
                                           ctypes.c_void_p]
    lib.nr_b200_backward_lights.restype = ctypes.c_int
    lib.nr_b200_backward_lights.argtypes = [ctypes.POINTER(BackwardArgs), ctypes.POINTER(PhongArgs),
                                            ctypes.POINTER(LightsArgs), ctypes.c_void_p]
    lib.nr_b200_forward_sh.restype = ctypes.c_int
    lib.nr_b200_forward_sh.argtypes = [ctypes.POINTER(ForwardArgs), ctypes.POINTER(PhongArgs), ctypes.POINTER(LightsArgs),
                                       ctypes.POINTER(ShArgs), ctypes.c_void_p]
    lib.nr_b200_backward_sh.restype = ctypes.c_int
    lib.nr_b200_backward_sh.argtypes = [ctypes.POINTER(BackwardArgs), ctypes.POINTER(PhongArgs), ctypes.POINTER(LightsArgs),
                                        ctypes.POINTER(ShArgs), ctypes.c_void_p]
    lib.nr_b200_forward_normal_map.restype = ctypes.c_int
    lib.nr_b200_forward_normal_map.argtypes = [ctypes.POINTER(ForwardArgs), ctypes.POINTER(PhongArgs),
                                               ctypes.POINTER(LightsArgs), ctypes.POINTER(ShArgs),
                                               ctypes.POINTER(NormalMapArgs), ctypes.c_void_p]
    lib.nr_b200_backward_normal_map.restype = ctypes.c_int
    lib.nr_b200_backward_normal_map.argtypes = [ctypes.POINTER(BackwardArgs), ctypes.POINTER(PhongArgs),
                                                ctypes.POINTER(LightsArgs), ctypes.POINTER(ShArgs),
                                                ctypes.POINTER(NormalMapArgs), ctypes.c_void_p]
    lib.nr_b200_forward_specular_map.restype = ctypes.c_int
    lib.nr_b200_forward_specular_map.argtypes = [ctypes.POINTER(ForwardArgs), ctypes.POINTER(PhongArgs),
                                                 ctypes.POINTER(LightsArgs), ctypes.POINTER(ShArgs),
                                                 ctypes.POINTER(NormalMapArgs), ctypes.POINTER(SpecularMapArgs),
                                                 ctypes.c_void_p]
    lib.nr_b200_backward_specular_map.restype = ctypes.c_int
    lib.nr_b200_backward_specular_map.argtypes = [ctypes.POINTER(BackwardArgs), ctypes.POINTER(PhongArgs),
                                                  ctypes.POINTER(LightsArgs), ctypes.POINTER(ShArgs),
                                                  ctypes.POINTER(NormalMapArgs), ctypes.POINTER(SpecularMapArgs),
                                                  ctypes.c_void_p]
    for name in ("nr_b200_interpolate", "nr_b200_interpolate_backward"):
        fn = getattr(lib, name)
        fn.restype = ctypes.c_int
        fn.argtypes = [ctypes.POINTER(InterpolateArgs), ctypes.c_void_p]
    lib.nr_b200_soft_workspace_bytes.restype = ctypes.c_size_t
    lib.nr_b200_soft_workspace_bytes.argtypes = [ctypes.c_int32] * 3 + [ctypes.c_float, ctypes.c_uint32]
    for name in ("nr_b200_soft_silhouettes", "nr_b200_soft_silhouettes_backward"):
        fn = getattr(lib, name)
        fn.restype = ctypes.c_int
        fn.argtypes = [ctypes.POINTER(SoftArgs), ctypes.c_void_p]
    lib.nr_b200_soft_rgb_workspace_bytes.restype = ctypes.c_size_t
    lib.nr_b200_soft_rgb_workspace_bytes.argtypes = [ctypes.c_int32] * 3 + [ctypes.c_uint32]
    for name in ("nr_b200_soft_rgb", "nr_b200_soft_rgb_backward"):
        fn = getattr(lib, name)
        fn.restype = ctypes.c_int
        fn.argtypes = [ctypes.POINTER(SoftRgbArgs), ctypes.c_void_p]
    for name in ("nr_b200_soft_rgb_uv", "nr_b200_soft_rgb_uv_backward"):
        fn = getattr(lib, name)
        fn.restype = ctypes.c_int
        fn.argtypes = [ctypes.POINTER(SoftRgbArgs), ctypes.POINTER(SoftUvArgs), ctypes.c_void_p]
    for name in ("nr_b200_soft_attributes", "nr_b200_soft_attributes_backward"):
        fn = getattr(lib, name)
        fn.restype = ctypes.c_int
        fn.argtypes = [ctypes.POINTER(SoftRgbArgs), ctypes.POINTER(SoftAttrArgs), ctypes.c_void_p]
    for name in ("nr_b200_soft_fragments", "nr_b200_soft_fragments_backward"):
        fn = getattr(lib, name)
        fn.restype = ctypes.c_int
        fn.argtypes = [ctypes.POINTER(SoftRgbArgs), ctypes.POINTER(SoftFragArgs), ctypes.c_void_p]
    lib.nr_b200_vertices_to_faces.restype = ctypes.c_int
    lib.nr_b200_vertices_to_faces.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int32, ctypes.c_int32,
                                              ctypes.c_int32, ctypes.c_void_p, ctypes.c_void_p]
    lib.nr_b200_vertices_to_faces_backward.restype = ctypes.c_int
    lib.nr_b200_vertices_to_faces_backward.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int32, ctypes.c_int32,
                                                       ctypes.c_int32, ctypes.c_void_p, ctypes.c_uint32, ctypes.c_void_p]
    lib.nr_b200_camera_transform.restype = ctypes.c_int
    lib.nr_b200_camera_transform.argtypes = [ctypes.c_void_p] * 4 + [ctypes.c_int32, ctypes.c_int32, ctypes.c_uint32,
                                                                    ctypes.c_void_p, ctypes.c_void_p]
    lib.nr_b200_camera_transform_backward.restype = ctypes.c_int
    lib.nr_b200_camera_transform_backward.argtypes = [ctypes.c_void_p] * 5 + [ctypes.c_int32, ctypes.c_int32, ctypes.c_uint32] + \
        [ctypes.c_void_p] * 5
    lib.nr_b200_face_lighting.restype = ctypes.c_int
    lib.nr_b200_face_lighting.argtypes = [ctypes.c_void_p] * 3 + [ctypes.c_int32] * 3 + [ctypes.c_uint32, ctypes.c_void_p,
                                                                                       ctypes.c_void_p]
    lib.nr_b200_face_lighting_backward.restype = ctypes.c_int
    lib.nr_b200_face_lighting_backward.argtypes = [ctypes.c_void_p] * 4 + [ctypes.c_int32] * 3 + [ctypes.c_uint32, ctypes.c_void_p,
                                                                                                ctypes.c_void_p]
    lib.nr_b200_vertex_normals_workspace_bytes.restype = ctypes.c_size_t
    lib.nr_b200_vertex_normals_workspace_bytes.argtypes = [ctypes.c_int32] * 3 + [ctypes.c_uint32]
    lib.nr_b200_vertex_normals.restype = ctypes.c_int
    lib.nr_b200_vertex_normals.argtypes = [ctypes.c_void_p] * 2 + [ctypes.c_int32] * 3 + [ctypes.c_uint32] + \
        [ctypes.c_void_p] * 2 + [ctypes.c_size_t, ctypes.c_void_p]
    lib.nr_b200_vertex_normals_backward.restype = ctypes.c_int
    lib.nr_b200_vertex_normals_backward.argtypes = [ctypes.c_void_p] * 3 + [ctypes.c_int32] * 3 + [ctypes.c_uint32] + \
        [ctypes.c_void_p] * 2 + [ctypes.c_size_t, ctypes.c_void_p]
    lib.nr_b200_corner_lighting.restype = ctypes.c_int
    lib.nr_b200_corner_lighting.argtypes = [ctypes.c_void_p] * 3 + [ctypes.c_int32] * 3 + [ctypes.c_uint32, ctypes.c_void_p,
                                                                                         ctypes.c_void_p]
    lib.nr_b200_corner_lighting_backward.restype = ctypes.c_int
    lib.nr_b200_corner_lighting_backward.argtypes = [ctypes.c_void_p] * 4 + [ctypes.c_int32] * 3 + [ctypes.c_uint32,
                                                                                                  ctypes.c_void_p, ctypes.c_void_p]
    lib.nr_b200_corner_shading.restype = ctypes.c_int
    lib.nr_b200_corner_shading.argtypes = [ctypes.c_void_p] * 3 + [ctypes.c_int32] * 3 + [ctypes.c_uint32, ctypes.c_void_p,
                                                                                        ctypes.c_void_p]
    lib.nr_b200_corner_shading_backward.restype = ctypes.c_int
    lib.nr_b200_corner_shading_backward.argtypes = [ctypes.c_void_p] * 2 + [ctypes.c_int32] * 3 + [ctypes.c_uint32] + \
        [ctypes.c_void_p] * 3
    lib.nr_b200_bake_textures.restype = ctypes.c_int
    lib.nr_b200_bake_textures.argtypes = [ctypes.c_void_p] * 3 + [ctypes.c_int32] * 4 + [ctypes.c_void_p, ctypes.c_void_p]
    lib.nr_b200_mip_texels.restype = ctypes.c_size_t
    lib.nr_b200_mip_texels.argtypes = [ctypes.c_int32, ctypes.c_int32]
    lib.nr_b200_mip_build.restype = ctypes.c_int
    lib.nr_b200_mip_build.argtypes = [ctypes.c_void_p] + [ctypes.c_int32] * 3 + [ctypes.c_void_p, ctypes.c_void_p]
    lib.nr_b200_mip_collapse.restype = ctypes.c_int
    lib.nr_b200_mip_collapse.argtypes = [ctypes.c_void_p] + [ctypes.c_int32] * 3 + [ctypes.c_void_p, ctypes.c_uint32,
                                                                                   ctypes.c_void_p]
    lib.nr_b200_last_launch_count.restype = ctypes.c_int
    lib.nr_b200_set_profiling.restype = None
    lib.nr_b200_set_profiling.argtypes = [ctypes.c_int]
    lib.nr_b200_read_profile.restype = ctypes.c_int
    lib.nr_b200_read_profile.argtypes = [ctypes.c_char_p, ctypes.c_size_t, ctypes.POINTER(ctypes.c_float), ctypes.c_int]
    if lib.nr_b200_abi_version() != ABI_VERSION:
        raise ImportError("libnr_b200.so ABI %d != binding ABI %d: rebuild" % (lib.nr_b200_abi_version(), ABI_VERSION))
    _LIB = lib
    return lib


def check(code):
    if code != NR_OK:
        raise RuntimeError("nr_b200: %s (code %d)" % (load().nr_b200_error_string(code).decode(), code))


def read_profile(max_entries=4096):
    """[(kernel name, milliseconds)] recorded since profiling was enabled / last read (synchronises)."""
    lib = load()
    names = ctypes.create_string_buffer(64 * max_entries)
    ms = (ctypes.c_float * max_entries)()
    n = lib.nr_b200_read_profile(names, len(names), ms, max_entries)
    parts = names.raw.split(b"\0")
    return [(parts[i].decode(), float(ms[i])) for i in range(n)]
