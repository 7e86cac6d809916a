"""GPU: trilinear sampling of a texture image through its mip pyramid (texture_filter='trilinear', NR_TEX_MIPMAP).

The pyramid build is checked against a float64 numpy restatement and the collapse as its adjoint; the forward and the
image / light gradients against a float64 torch oracle of the documented sampler (include/nr_b200.h) that computes its
level of detail from the faces, built on the product's own face_index_map / weight_map / depth_map like oracle_rgb of
test_gpu_uv.py (both in oracles.py)."""
import ctypes
import os

import numpy as np
import pytest
import torch

from helpers import np_, rel_err
from oracles import oracle_trilinear, pyramid64
from test_gpu_uv import CASES as UV_CASES

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = torch.device("cuda")


def _R():
    import importlib
    return importlib.import_module("neural_renderer_b200.rasterize")


def _rand(shape, lo=0.0, hi=1.0, seed=1):
    g = torch.Generator().manual_seed(seed)
    return (lo + (hi - lo) * torch.rand(shape, generator=g, dtype=torch.float32)).to(DEV)


def _spread_uvs(shape, lo, hi, seed):
    """UV corners around a random centre in [lo, hi] with a per-face spread from 1e-3 to 100: faces from strongly
    magnified (LOD clamped at 0) to strongly minified (clamped at the last level)."""
    g = torch.Generator().manual_seed(seed)
    centre = lo + (hi - lo) * torch.rand(shape[:-2] + (1, 2), generator=g, dtype=torch.float64)
    spread = 10.0 ** (-3 + 5 * torch.rand(shape[:-2] + (1, 1), generator=g, dtype=torch.float64))
    return (centre + spread * (torch.rand(shape, generator=g, dtype=torch.float64) - 0.5)).float().to(DEV)


def _pack(levels):
    return np.concatenate([l.reshape(l.shape[0], -1, 3) for l in levels], axis=1)


def _lib():
    from neural_renderer_b200 import _lib as L
    return L, L.load()


def _build(img):
    L, lib = _lib()
    Bt, H, W = img.shape[:3]
    pyr = torch.empty((Bt, lib.nr_b200_mip_texels(H, W), 3), device=DEV)
    L.check(lib.nr_b200_mip_build(ctypes.c_void_p(img.data_ptr()), Bt, H, W, ctypes.c_void_p(pyr.data_ptr()), None))
    assert lib.nr_b200_last_launch_count() <= 2
    return pyr


def _collapse(g, H, W, out=None, flags=0):
    L, lib = _lib()
    Bt = g.shape[0]
    out = torch.empty((Bt, H, W, 3), device=DEV) if out is None else out
    L.check(lib.nr_b200_mip_collapse(ctypes.c_void_p(g.data_ptr()), Bt, H, W, ctypes.c_void_p(out.data_ptr()), flags, None))
    assert lib.nr_b200_last_launch_count() == 1
    return out


SIZES = [(1, 1), (1, 9), (12, 1), (17, 40), (1023, 1025), (1024, 1024)]


@pytest.mark.parametrize("Bt", [1, 3])
@pytest.mark.parametrize("hw", SIZES)
def test_build_and_collapse(hw, Bt):
    H, W = hw
    img = _rand((Bt, H, W, 3), seed=H * 7 + W)
    pyr = _build(img)
    torch.cuda.synchronize()
    want = _pack(pyramid64(np_(img).astype(np.float64)))
    assert pyr.shape == want.shape
    assert rel_err(np_(pyr), want) <= 1e-6
    assert torch.equal(pyr[:, :H * W].reshape(Bt, H, W, 3), img)  # level 0 is a copy
    # the collapse is the build's adjoint (positive data: no cancellation in the inner products)
    G = _rand(pyr.shape, seed=3)
    I = _rand(img.shape, seed=4)
    lhs = float((_collapse(G, H, W).double() * I.double()).sum())
    rhs = float((G.double() * _build(I).double()).sum())
    assert abs(lhs - rhs) <= 1e-6 * abs(rhs)
    # NR_GRAD_ACCUMULATE adds into the image gradient
    acc = torch.ones_like(img)
    _collapse(G, H, W, out=acc, flags=_lib()[0].NR_GRAD_ACCUMULATE)
    assert rel_err(np_(acc), np_(_collapse(G, H, W) + 1)) <= 1e-6


def _render(faces, image, uvs, H, aa, light=None, fill_back=False, bg=(0.1, 0.2, 0.3), texture_filter="trilinear"):
    return _R()._run(faces, image, H, aa, 0.1, 100, 1e-4, bg, True, True, True, face_light=light,
                     textures_fill_back=fill_back, face_uvs=uvs, texture_filter=texture_filter)


def _faces(B, F, seed):
    from neural_renderer_b200 import synthetic
    return torch.from_numpy(synthetic.sphere_faces(B, F, seed=seed)).to(DEV)


# the UV matrix of test_gpu_uv.py plus large images on small rasters
CASES = list(UV_CASES) + [
    (False, False, False, True, True, (512, 512), (0, 1), 48, 200),
    (True, True, False, True, False, (1024, 1024), (0, 1), 32, 100),
    (False, True, True, False, True, (1023, 1025), (-0.6, 1.7), 40, 100),
]


def _run_case(case, lib_check=True):
    aa, lit, fill_back, shared_img, shared_uv, (Ht, Wt), (lo, hi), H, F = case
    B = 2
    S = 2 * H if aa else H
    faces = _faces(B, F, seed=3)
    if fill_back:
        faces = torch.cat((faces, faces.flip(2)), dim=1)
    uvs = _spread_uvs((1 if shared_uv else B, F, 3, 2), lo, hi, seed=4)
    if shared_uv:
        uvs = uvs[0]
    img0 = _rand((1 if shared_img else B, Ht, Wt, 3), seed=5)
    img = img0.clone().requires_grad_(True)
    light = (0.5 + _rand((B, faces.shape[1], 3), seed=6)).requires_grad_(True) if lit else None
    rgb, alpha, depth, fim, wmap = _render(faces, img, uvs, H, aa, light, fill_back)
    g = torch.randn(rgb.shape, generator=torch.Generator().manual_seed(7)).to(DEV)
    (rgb * g).sum().backward()
    dmap = _R()._run(faces, None, S, False, 0.1, 100, 1e-4, None, False, False, True)[2]
    img64 = img0.double().requires_grad_(True)
    light64 = light.detach().double().requires_grad_(True) if lit else None
    ref, lod, L = oracle_trilinear(faces, fim, wmap, dmap, uvs if uvs.dim() == 4 else uvs[None], img64, light64,
                                   (0.1, 0.2, 0.3), fill_back, aa)
    (ref * g.double()).sum().backward()
    return rgb, ref, img, img64, light, light64, lod, L, fim


@pytest.mark.parametrize("case", CASES)
def test_forward_and_gradients_vs_oracle(case):
    rgb, ref, img, img64, light, light64, lod, L, fim = _run_case(case)
    assert (fim >= 0).sum() > 500
    if L > 1:  # the case reaches all three regimes of the level of detail
        lc = lod[fim >= 0]
        assert (lc == 0).any() and ((lc > 0) & (lc < L - 1)).any() and (lc == L - 1).any(), (L, lc.min(), lc.max())
    assert rel_err(np_(rgb), np_(ref)) <= 1e-5
    assert rel_err(np_(img.grad), np_(img64.grad)) <= 1e-5
    if light is not None:
        assert rel_err(np_(light.grad), np_(light64.grad)) <= 1e-5


@pytest.mark.parametrize("hw, aa", [((64, 48), False), ((1024, 1024), True), ((33, 47), False)])
def test_forward_and_backward_pick_the_same_taps(hw, aa):
    """unlit: rgb is linear in the image on covered pixels, so <g, rgb(T) - rgb(0)> = <d loss / d T, T> exactly when
    the backward scatters to the taps and with the weights the forward blended (zero-mean g: a level or weight picked
    differently shows at its own size, not against a large positive total)"""
    B, F, H = 2, 300, 64
    faces = _faces(B, F, seed=21)
    uvs = _spread_uvs((F, 3, 2), 0, 1, seed=22)
    T = _rand((1, *hw, 3), seed=23).requires_grad_(True)
    rgb = _render(faces, T, uvs, H, aa)[0]
    g = torch.randn(rgb.shape, generator=torch.Generator().manual_seed(24)).to(DEV)
    (rgb * g).sum().backward()
    rgb0 = _render(faces, torch.zeros_like(T), uvs, H, aa)[0]
    lhs = float((g.double() * (rgb.detach().double() - rgb0.double())).sum())
    rhs = float((T.grad.double() * T.detach().double()).sum())
    assert abs(lhs - rhs) <= 1e-5 * abs(lhs), (lhs, rhs)


def test_trilinear_is_bilinear_without_minification():
    """a small image on a camera-facing square much larger than its texels: LOD 0 everywhere"""
    faces, uvs = _square()
    base = _rand((1, 48, 64, 3), seed=33)
    g = torch.randn((1, 3, 256, 256), generator=torch.Generator().manual_seed(34)).to(DEV)
    out = {}
    for tf in ("bilinear", "trilinear"):
        t = base.clone().requires_grad_(True)
        rgb = _render(faces, t, uvs, 256, False, texture_filter=tf)[0]
        (rgb * g).sum().backward()
        out[tf] = (rgb.detach(), t.grad)
    assert torch.equal(out["trilinear"][0], out["bilinear"][0])
    assert rel_err(np_(out["trilinear"][1]), np_(out["bilinear"][1])) <= 1e-6


def _square(z=2.0, r=0.9):
    """a camera-facing square (both windings of its two triangles, so that culling keeps one) with UVs over [0,1]^2"""
    v = torch.tensor([[-r, -r, z], [r, -r, z], [r, r, z], [-r, r, z]], dtype=torch.float32)
    t = torch.tensor([[0, 0], [1, 0], [1, 1], [0, 1]], dtype=torch.float32)
    tri = [[0, 1, 2], [0, 2, 3], [2, 1, 0], [3, 2, 0]]
    tri = torch.tensor(tri)
    return v[tri][None].to(DEV), t[tri].to(DEV)


def test_minified_checkerboard():
    """the point of the feature: a one-texel 1024^2 checkerboard on a square of about 58 x 58 pixels"""
    faces, uvs = _square()
    n = 1024
    ii = torch.arange(n)
    board = ((ii[:, None] + ii[None, :]) % 2).float()[None, ..., None].expand(1, n, n, 3).contiguous().to(DEV)
    res = {}
    for tf in ("bilinear", "trilinear"):
        t = board.clone().requires_grad_(True)
        rgb, alpha = _render(faces, t, uvs, 64, False, bg=(0, 0, 0), texture_filter=tf)[:2]
        rgb.sum().backward()
        cov = alpha[0] > 0
        res[tf] = (rgb[0][:, cov], t.grad[0])
    assert cov.sum() > 3000
    assert (res["trilinear"][0] - 0.5).abs().max() <= 1e-5
    assert res["bilinear"][0].std() > 0.1
    assert (res["trilinear"][1] != 0).all()
    assert (res["bilinear"][1] != 0).float().mean() < 0.02


def test_shared_image_equals_per_item_copies():
    B, F = 4, 300
    faces = _faces(B, F, seed=11)
    uvs, base = _spread_uvs((F, 3, 2), 0, 1, seed=12), _rand((200, 120, 3), seed=13)
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
    faces0 = _faces(B, F, seed=3)
    uvs, img0 = _spread_uvs((F, 3, 2), 0, 1, seed=1), _rand((256, 256, 3), seed=2)
    g = torch.randn((B, 3, 64, 64), generator=torch.Generator().manual_seed(1)).to(DEV)

    def run():
        f = faces0.clone().requires_grad_(True)
        t = img0.clone().requires_grad_(True)
        rgb = R._run(f, t, 64, False, 0.1, 100, 1e-4, (0, 0, 0), True, False, False, face_uvs=uvs,
                     texture_filter="trilinear")[0]
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
    assert seen.get("waited") and seen["tex"].shape == (1, _lib()[1].nr_b200_mip_texels(256, 256), 3)
    assert torch.equal(_collapse(seen["tex"], 256, 256)[0], gt1)  # the hook sees the pyramid gradient
    assert rel_err(np_(gt1), np_(gt0)) <= 1e-6
    assert rel_err(np_(gf1), np_(gf0)) <= 1e-5


def test_vertex_gradient_vs_reference_k5():
    import refhost
    S, F, ts, flags = 64, 200, 4, (1, 0, 0)
    if not refhost.available(S, F, ts, 0.1, 100, 1e-4, *flags):
        pytest.skip("reference kernels not built (oracle/_ref)")
    B = 2
    faces = _faces(B, F, seed=12)
    uvs, img = _spread_uvs((F, 3, 2), 0, 1, seed=1), _rand((1, 128, 128, 3), seed=2)
    bg = (0.2, 0.4, 0.6)
    g = torch.randn((B, 3, S, S), generator=torch.Generator().manual_seed(3)).to(DEV)
    f = faces.clone().requires_grad_(True)
    rgb = _R()._run(f, img, S, False, 0.1, 100, 1e-4, bg, *flags, face_uvs=uvs, texture_filter="trilinear")[0]
    (rgb * g).sum().backward()
    placeholder = torch.zeros((B, F, ts, ts, ts, 3), device=DEV)  # K5 reads only the rgb map
    ref = refhost.rasterize_rgbad(faces, placeholder, S, False, 0.1, 100, 1e-4, bg, *flags)
    ref.fn.rgb_map = rgb.detach().permute(0, 2, 3, 1).flip(1).contiguous()
    gf_ref, _ = ref.backward(g, None, None)
    assert rel_err(np_(f.grad), np_(gf_ref)) <= 1e-4


@pytest.mark.parametrize("fill_back", [True, False])
def test_renderer_fused_matches_op_by_op(teapot, fill_back):
    import neural_renderer as nr
    v, f = teapot
    B = 2
    rot = np.array([[0.9, 0.0, 0.43], [0.0, 1.0, 0.0], [-0.43, 0.0, 0.9]], np.float32)
    vertices = torch.from_numpy(np.stack([v, v @ rot.T])).to(DEV)
    faces_idx = torch.from_numpy(np.stack([f, f])).to(DEV)
    uvs = _rand((f.shape[0], 3, 2), seed=2)
    image = _rand((B, 300, 200, 3), seed=3)
    g = torch.randn((B, 3, 128, 128), generator=torch.Generator().manual_seed(2)).to(DEV)
    results = []
    for fused in (False, True):
        r = nr.Renderer()
        r.image_size = 128
        r.fill_back = fill_back
        r.fused = fused
        r.texture_filter = "trilinear"
        r.eye = nr.get_points_from_angles(2.732, 30, 40)
        r.light_direction = [0.3, 1.0, -0.2]
        va = vertices.clone().requires_grad_(True)
        ta = image.clone().requires_grad_(True)
        img = r.render(va, faces_idx, ta, face_uvs=uvs)
        (img * g).sum().backward()
        results.append((img.detach(), va.grad, ta.grad))
    (img0, gv0, gt0), (img1, gv1, gt1) = results
    assert (img0 != 0).any()
    assert rel_err(np_(img1), np_(img0)) <= 1e-6
    assert rel_err(np_(gt1), np_(gt0)) <= 1e-5
    assert rel_err(np_(gv1), np_(gv0)) <= 1e-4


def test_example5_trilinear_1024_optimises():
    import importlib.util
    spec = importlib.util.spec_from_file_location("example5", os.path.join(ROOT, "examples", "example5_optimize_texture_image.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    losses = mod.run(30, size=1024, texture_filter="trilinear")
    assert np.isfinite(losses).all()
    assert np.mean(losses[-5:]) < 0.8 * np.mean(losses[:5]), (losses[:5], losses[-5:])
