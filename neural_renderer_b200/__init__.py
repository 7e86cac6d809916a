"""neural_renderer_b200 -- H100-native (sm_90a) differentiable mesh rasterizer with the call surface of
hiroharu-kato/neural_renderer (export list of neural_renderer/__init__.py:1-16).

Hot path (hand-written sm_90a CUDA behind the C ABI in include/nr_b200.h): Rasterize, rasterize_rgbad, rasterize,
rasterize_silhouettes, rasterize_depth, rasterize_soft_silhouettes, rasterize_soft, rasterize_soft_attributes, rasterize_soft_fragments, blend_soft_fragments, interpolate_soft_fragments.  Everything
else is thin torch glue so that the reference's examples run with torch tensors in place of chainer Variables.
"""
from .functional import cross, get_points_from_angles, lighting, look, look_at, perspective, vertices_to_faces
from .rasterize import (
    rasterize_rgbad, rasterize, rasterize_silhouettes, rasterize_depth, use_unsafe_rasterizer, Rasterize,
    set_reference_exact, rasterize_attributes, rasterize_soft_silhouettes, rasterize_soft, rasterize_soft_attributes,
    rasterize_soft_fragments, Fragments, blend_soft_fragments, interpolate_soft_fragments, DEFAULT_SOFT_GAMMA)
from .renderer import Renderer
from .io import load_obj, save_obj
from .mesh import Mesh
from .optimizers import Adam

__version__ = '1.1.3+b200.1'
