"""Drop-in import name: `import neural_renderer` resolves to the H100-native package (neural_renderer_b200)."""
from neural_renderer_b200 import *  # noqa: F401,F403
from neural_renderer_b200 import (  # noqa: F401
    cross, get_points_from_angles, lighting, load_obj, look, look_at, Mesh, Adam, perspective, rasterize_rgbad,
    rasterize, rasterize_silhouettes, rasterize_depth, use_unsafe_rasterizer, Rasterize, Renderer, save_obj,
    rasterize_attributes, rasterize_soft_silhouettes, rasterize_soft, rasterize_soft_attributes, DEFAULT_SOFT_GAMMA,
    rasterize_soft_fragments, Fragments, blend_soft_fragments, interpolate_soft_fragments,
    vertices_to_faces, __version__)
