"""GPU: the texture-image mode (face_uvs + texture image, NR_TEX_UV).

The forward and the image / light gradients are checked against an op-by-op float64 torch oracle of the documented
sampler (include/nr_b200.h; oracles.oracle_rgb), built on the product's own face_index_map / weight_map / depth_map;
coverage against the cube mode; the vertex gradient against the reference's own K5 (oracle/refhost.py) fed with the
UV-mode rgb map.  The oracle forms the pixel's uv and texel positions in fp32 in the sampler's pinned operation order
(the header specifies fp32 there) and everything after that in float64: less independent of the kernel than a float64
uv, but one fp32 ulp of u would otherwise dominate the comparison."""
import os

import numpy as np
import pytest
import torch

from helpers import np_, rel_err
from oracles import oracle_rgb

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = torch.device("cuda")


def _R():
    import importlib
    return importlib.import_module("neural_renderer_b200.rasterize")


def _case(B=2, F=200, seed=0):
    from neural_renderer_b200 import synthetic
    return torch.from_numpy(synthetic.sphere_faces(B, F, seed=seed)).to(DEV)


def _uvs(shape, lo=0.0, hi=1.0, seed=1):
    g = torch.Generator().manual_seed(seed)
    return (lo + (hi - lo) * torch.rand(shape, generator=g, dtype=torch.float32)).to(DEV)


def _render(faces, image, uvs, S, aa, light=None, fill_back=False, reference_exact=None, bg=(0.1, 0.2, 0.3)):
    return _R()._run(faces, image, S, aa, 0.1, 100, 1e-4, bg, True, True, True, face_light=light,
                     textures_fill_back=fill_back, reference_exact=reference_exact, face_uvs=uvs)


CASES = [
    # aa, lit, fill_back, shared image, shared uvs, (Ht, Wt), uv range, API image size H, F
    (False, False, False, True, True, (32, 32), (0, 1), 48, 200),
    (True, False, False, True, True, (32, 32), (0, 1), 48, 200),
    (False, True, False, False, True, (17, 40), (0, 1), 48, 200),
    (True, True, True, True, False, (40, 17), (0, 1), 48, 200),
    (False, False, True, False, False, (16, 16), (0, 1), 48, 200),
    (False, True, True, True, True, (1, 9), (0, 1), 48, 200),
    (True, False, False, False, True, (12, 1), (0, 1), 48, 200),
    (False, False, False, True, False, (1, 1), (0, 1), 48, 200),
    (False, True, False, True, True, (24, 20), (-0.6, 1.7), 48, 200),
    (True, True, True, False, False, (9, 30), (-0.6, 1.7), 48, 200),
    # raster 257: odd, the edge scan keeps only the face index in its strip; 700 (image 350, odd) and 102 (image 51):
    # anti-aliasing with an odd pooled size, one-line strips at 700
    (False, True, False, True, True, (24, 20), (0, 1), 257, 300),
    (True, False, True, False, True, (33, 47), (-0.6, 1.7), 350, 300),
    (True, True, False, True, False, (16, 9), (0, 1), 51, 200),
]


@pytest.mark.parametrize("case", CASES)
def test_forward_and_gradients_vs_oracle(case):
    aa, lit, fill_back, shared_img, shared_uv, (Ht, Wt), (lo, hi), H, F = case
    B = 2
    S = 2 * H if aa else H
    faces = _case(B, F, seed=3)
    if fill_back:
        faces = torch.cat((faces, faces.flip(2)), dim=1)
    nuv = F
    uvs = _uvs((1 if shared_uv else B, nuv, 3, 2), lo, hi, seed=4)
    if shared_uv:
        uvs = uvs[0]
    img0 = _uvs((1 if shared_img else B, Ht, Wt, 3), seed=5)
    img = img0.clone().requires_grad_(True)
    light = (0.5 + _uvs((B, faces.shape[1], 3), seed=6)).requires_grad_(True) if lit else None
    rgb, alpha, depth, fim, wmap = _render(faces, img, uvs, H, aa, light, fill_back)
    g = torch.randn(rgb.shape, generator=torch.Generator().manual_seed(7)).to(DEV)
    (rgb * g).sum().backward()
    # the raster depth map (the product's own) comes from a second, depth-only call: identical coverage
    dmap = _R()._run(faces, None, S, False, 0.1, 100, 1e-4, None, False, False, True)[2]
    img64 = img0.double().requires_grad_(True)
    light64 = light.detach().double().requires_grad_(True) if lit else None
    ref = oracle_rgb(faces, fim, wmap, dmap, uvs if uvs.dim() == 4 else uvs[None], img64, light64, (0.1, 0.2, 0.3),
                     fill_back, aa)
    assert (fim >= 0).sum() > 500
    assert rel_err(np_(rgb), np_(ref)) <= 1e-5
    (ref * g.double()).sum().backward()
    assert rel_err(np_(img.grad), np_(img64.grad)) <= 1e-5
    if lit:
        assert rel_err(np_(light.grad), np_(light64.grad)) <= 1e-5


def test_coverage_does_not_depend_on_the_texture_model():
    from neural_renderer_b200 import synthetic
    B, F = 2, 400
    faces = _case(B, F, seed=8)
    cubes = torch.from_numpy(synthetic.random_textures(B, F, 4, seed=9)).to(DEV)
    for aa in (False, True):
        a = _R()._run(faces, cubes, 64, aa, 0.1, 100, 1e-4, (0, 0, 0), True, True, True)
        b = _render(faces, _uvs((20, 30, 3)), _uvs((F, 3, 2)), 64, aa)
        for k in (1, 2, 3, 4):  # alpha, depth, face_index_map, weight_map
            assert torch.equal(a[k], b[k]), (aa, k)


def test_reference_exact_has_no_effect():
    B, F = 3, 300
    faces = _case(B, F, seed=10)
    uvs, img = _uvs((F, 3, 2)), _uvs((1, 16, 24, 3))
    g = torch.randn((B, 3, 64, 64), generator=torch.Generator().manual_seed(1)).to(DEV)
    out = []
    for exact in (True, False):
        t = img.clone().requires_grad_(True)
        rgb = _render(faces, t, uvs, 64, False, reference_exact=exact)[0]
        (rgb * g).sum().backward()
        out.append((rgb.detach(), t.grad))
    assert torch.equal(out[0][0], out[1][0])
    assert rel_err(np_(out[0][1]), np_(out[1][1])) <= 1e-6


def test_shared_image_gradient_is_the_sum_over_items():
    B, F = 4, 300
    faces = _case(B, F, seed=11)
    uvs, base = _uvs((F, 3, 2)), _uvs((20, 20, 3))
    g = torch.randn((B, 3, 64, 64), generator=torch.Generator().manual_seed(2)).to(DEV)
    res = {}
    for kind in ("copy", "shared", "expanded"):
        t0 = base.clone().requires_grad_(True)
        t = {"copy": lambda: t0[None].expand(B, -1, -1, -1).contiguous(), "shared": lambda: t0,
             "expanded": lambda: t0[None].expand(B, -1, -1, -1)}[kind]()
        rgb = _render(faces, t, uvs[None].expand(B, -1, -1, -1), 64, False)[0]
        (rgb * g).sum().backward()
        res[kind] = (rgb.detach(), t0.grad)
    for kind in ("shared", "expanded"):
        assert torch.equal(res[kind][0], res["copy"][0])
        assert rel_err(np_(res[kind][1]), np_(res["copy"][1])) <= 1e-5


def test_two_part_backward_with_texture_hook():
    R = _R()
    B, F = 2, 800
    faces0 = _case(B, F, seed=3)
    uvs, img0 = _uvs((F, 3, 2)), _uvs((64, 64, 3))
    g = torch.randn((B, 3, 64, 64), generator=torch.Generator().manual_seed(1)).to(DEV)

    def run():
        f = faces0.clone().requires_grad_(True)
        t = img0.clone().requires_grad_(True)
        rgb = R._run(f, t, 64, False, 0.1, 100, 1e-4, (0, 0, 0), True, False, False, face_uvs=uvs)[0]
        (rgb * g).sum().backward()
        return f.grad, t.grad

    gf0, gt0 = run()
    seen = {}

    class Pending:
        def wait(self):
            seen["waited"] = True

    def hook(grad_textures):
        seen["tex"] = grad_textures.clone()
        return Pending()

    prev = R.set_texture_grad_hook(hook)
    try:
        gf1, gt1 = run()
    finally:
        R.set_texture_grad_hook(prev)
    assert seen.get("waited") and torch.equal(seen["tex"][0], gt1)
    assert rel_err(np_(gt1), np_(gt0)) <= 1e-6
    assert rel_err(np_(gf1), np_(gf0)) <= 1e-5


def _vertex_gradient_vs_reference_k5(S, F, ts, flags):
    import refhost
    if not refhost.available(S, F, ts, 0.1, 100, 1e-4, *flags):
        pytest.skip("reference kernels not built (oracle/_ref)")
    B = 2
    faces = _case(B, F, seed=12)
    uvs, img = _uvs((F, 3, 2)), _uvs((1, 32, 32, 3))
    bg = (0.2, 0.4, 0.6)
    g = torch.randn((B, 3, S, S), generator=torch.Generator().manual_seed(3)).to(DEV)
    f = faces.clone().requires_grad_(True)
    rgb = _R()._run(f, img, S, False, 0.1, 100, 1e-4, bg, *flags, face_uvs=uvs)[0]
    (rgb * g).sum().backward()
    placeholder = torch.zeros((B, F, ts, ts, ts, 3), device=DEV)  # K5 reads only the rgb map
    ref = refhost.rasterize_rgbad(faces, placeholder, S, False, 0.1, 100, 1e-4, bg, *flags)
    ref.fn.rgb_map = rgb.detach().permute(0, 2, 3, 1).flip(1).contiguous()  # API image -> the reference's NHWC, unflipped
    gf_ref, _ = ref.backward(g, None, None)
    assert rel_err(np_(f.grad), np_(gf_ref)) <= 1e-4


def test_vertex_gradient_vs_reference_k5():
    _vertex_gradient_vs_reference_k5(64, 200, 4, (1, 0, 0))


@pytest.mark.parametrize("S", [257, 1024])
def test_vertex_gradient_vs_reference_k5_at_other_raster_sizes(S):
    """257 (odd, face index only in the strip) and 1024 (one-line strips): the (1, 1, 1) binaries of
    oracle/ref_configs.py SIZES, with the product run with the same return flags (same strip width)"""
    from ref_configs import SIZES_F, SIZES_TS
    _vertex_gradient_vs_reference_k5(S, SIZES_F, SIZES_TS, (1, 1, 1))


@pytest.mark.parametrize("fill_back", [True, False])
def test_renderer_fused_matches_op_by_op(teapot, fill_back):
    import neural_renderer as nr
    v, f = teapot
    B = 2
    rot = np.array([[0.9, 0.0, 0.43], [0.0, 1.0, 0.0], [-0.43, 0.0, 0.9]], np.float32)
    vertices = torch.from_numpy(np.stack([v, v @ rot.T])).to(DEV)
    faces_idx = torch.from_numpy(np.stack([f, f])).to(DEV)
    uvs = _uvs((f.shape[0], 3, 2), seed=2)
    image = _uvs((B, 40, 56, 3), seed=3)
    g = torch.randn((B, 3, 128, 128), generator=torch.Generator().manual_seed(2)).to(DEV)
    results = []
    for fused in (False, True):
        r = nr.Renderer()
        r.image_size = 128
        r.fill_back = fill_back
        r.fused = fused
        r.eye = nr.get_points_from_angles(2.732, 30, 40)
        r.light_direction = [0.3, 1.0, -0.2]
        va = vertices.clone().requires_grad_(True)
        ta = image.clone().requires_grad_(True)
        img = r.render(va, faces_idx, ta, face_uvs=uvs)
        (img * g).sum().backward()
        results.append((img.detach(), va.grad, ta.grad))
    (img0, gv0, gt0), (img1, gv1, gt1) = results
    assert (img0 != 0).any()
    assert rel_err(np_(img1), np_(img0)) <= 1e-6  # the light factors differ by fp32 rounding (fused normalisation)
    assert rel_err(np_(gt1), np_(gt0)) <= 1e-5
    assert rel_err(np_(gv1), np_(gv0)) <= 1e-4


def test_display_model_renders_through_the_uv_loader():
    import neural_renderer as nr
    from neural_renderer_b200 import io
    path = os.path.join(ROOT, "tests", "golden", "display", "model.obj")
    v, f, uv, image = io.load_obj(path, load_texture=True, texture_mode="uv")
    r = nr.Renderer()
    r.eye = nr.get_points_from_angles(2.732, 20, 30)
    img = r.render(torch.from_numpy(v).to(DEV)[None], torch.from_numpy(f).to(DEV)[None],
                   torch.from_numpy(np.ascontiguousarray(image)).to(DEV), face_uvs=torch.from_numpy(uv).to(DEV))
    assert torch.isfinite(img).all() and img.shape == (1, 3, 256, 256)
    assert (img.sum(1) > 0).float().mean() > 0.05


def test_example5_optimises():
    import importlib.util
    spec = importlib.util.spec_from_file_location("example5", os.path.join(ROOT, "examples", "example5_optimize_texture_image.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    losses = mod.run(30)
    assert np.isfinite(losses).all()
    assert np.mean(losses[-5:]) < 0.8 * np.mean(losses[:5]), (losses[:5], losses[-5:])
