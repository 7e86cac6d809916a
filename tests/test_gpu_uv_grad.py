"""GPU: the face_uvs gradient of the texture-image samplers (bilinear NR_TEX_UV and trilinear NR_TEX_MIPMAP).

face_uvs.grad is held to the float64 oracles of oracles_uv_grad.py (the documented derivative of
include/nr_b200.h: the fp32 cell and clamp mask of the product, a float64 straight-through term for d uv / d uv_k), to a
central difference of the product's own forward (independent of the formula the oracle and the kernel share), and to the
other paths that reach the same gradient (shared / per-item UVs, the fused Renderer, the two-half backward, the C ABI
directly).  The rest of the backward must not notice that face_uvs wants a gradient."""
import ctypes

import numpy as np
import pytest
import torch

from helpers import elem_err, np_, rel_err
from oracles_uv_grad import oracle_rgb_uv_grad, oracle_trilinear_uv_grad
from test_gpu_mip import CASES as MIP_CASES, _spread_uvs
from test_gpu_uv import CASES as UV_CASES

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda")


def _R():
    import importlib
    return importlib.import_module("neural_renderer_b200.rasterize")


def _rand(shape, lo=0.0, hi=1.0, seed=1):
    g = torch.Generator().manual_seed(seed)
    return (lo + (hi - lo) * torch.rand(shape, generator=g, dtype=torch.float32)).to(DEV)


def _faces(B, F, seed):
    from neural_renderer_b200 import synthetic
    return torch.from_numpy(synthetic.sphere_faces(B, F, seed=seed)).to(DEV)


def _render(faces, image, uvs, H, aa, light=None, fill_back=False, texture_filter="bilinear", bg=(0.1, 0.2, 0.3)):
    return _R()._run(faces, image, H, aa, 0.1, 100, 1e-4, bg, True, True, True, face_light=light,
                     textures_fill_back=fill_back, face_uvs=uvs, texture_filter=texture_filter)


def _run_case(case, trilinear):
    aa, lit, fill_back, shared_img, shared_uv, (Ht, Wt), (lo, hi), H, F = case
    B = 2
    S = 2 * H if aa else H
    faces = _faces(B, F, seed=3)
    if fill_back:
        faces = torch.cat((faces, faces.flip(2)), dim=1)
    shape = (1 if shared_uv else B, F, 3, 2)
    uvs0 = _spread_uvs(shape, lo, hi, seed=4) if trilinear else _rand(shape, lo, hi, seed=4)
    if shared_uv:
        uvs0 = uvs0[0]
    uvs = uvs0.clone().requires_grad_(True)
    img = _rand((1 if shared_img else B, Ht, Wt, 3), seed=5)
    light = (0.5 + _rand((B, faces.shape[1], 3), seed=6)) if lit else None
    tf = "trilinear" if trilinear else "bilinear"
    rgb, alpha, depth, fim, wmap = _render(faces, img, uvs, H, aa, light, fill_back, tf)
    g = torch.randn(rgb.shape, generator=torch.Generator().manual_seed(7)).to(DEV)
    (rgb * g).sum().backward()
    dmap = _R()._run(faces, None, S, False, 0.1, 100, 1e-4, None, False, False, True)[2]
    uvs64 = uvs0.double().requires_grad_(True)
    args = (faces, fim, wmap, dmap, uvs64 if uvs64.dim() == 4 else uvs64[None], img.double(),
            light.double() if lit else None, (0.1, 0.2, 0.3), fill_back, aa)
    ref = oracle_trilinear_uv_grad(*args) if trilinear else oracle_rgb_uv_grad(*args)
    (ref * g.double()).sum().backward()
    assert (fim >= 0).sum() > 500
    return uvs.grad, uvs64.grad


@pytest.mark.parametrize("case", UV_CASES)
def test_bilinear_uv_gradient_vs_oracle(case):
    got, want = _run_case(case, trilinear=False)
    assert want.abs().max() > 0 or case[5] == (1, 1)  # a 1-texel axis only has a derivative along the other one
    print("uv-grad bilinear", case, rel_err(np_(got), np_(want)), elem_err(np_(got), np_(want)))
    assert rel_err(np_(got), np_(want)) <= 1e-4
    assert elem_err(np_(got), np_(want)) <= 1e-4


# The trilinear oracle computes the level of detail in float64 and the product in fp32: where the two land on different
# sides of a level boundary, or with a slightly different blend factor, a pixel weighs its two levels differently.
# Gates from the measured maxima over this case list on an H100 80GB HBM3 (400 W): rel_err 1.8e-6, elem_err 3.9e-4
# (bilinear: 2.9e-7 and 5.9e-5), the larger of two runs, about 5x and 4x headroom.
@pytest.mark.parametrize("case", MIP_CASES)
def test_trilinear_uv_gradient_vs_oracle(case):
    got, want = _run_case(case, trilinear=True)
    print("uv-grad trilinear", case, rel_err(np_(got), np_(want)), elem_err(np_(got), np_(want)))
    assert rel_err(np_(got), np_(want)) <= 1e-5
    assert elem_err(np_(got), np_(want)) <= 1.5e-3


def _smooth_image(H, W):
    """low-frequency, non-symmetric in u and v: one period per image axis, a different pattern per channel"""
    y = (torch.arange(H, dtype=torch.float64) + 0.5) / H
    x = (torch.arange(W, dtype=torch.float64) + 0.5) / W
    yy, xx = torch.meshgrid(1 - y, x, indexing="ij")  # row 0 = top = v near 1
    img = torch.stack((0.5 + 0.3 * torch.sin(2 * np.pi * xx + 0.3), 0.5 + 0.3 * torch.sin(2 * np.pi * yy + 1.1),
                       0.5 + 0.2 * torch.cos(2 * np.pi * (xx + 0.5 * yy))), dim=-1)
    return img.float()[None].to(DEV)


@pytest.mark.parametrize("tf, hw", [("bilinear", (48, 64)), ("trilinear", (512, 384))])
def test_directional_derivative_vs_central_difference(tf, hw):
    """<d L / d uv, delta> against (L(uv + h delta) - L(uv - h delta)) / 2h of the product's own forward, L = <g, rgb>,
    for a translation of every UV in u, one in v and (bilinear) a random direction: a sign error or a row flip of the
    derivative (in v especially) is far outside the 2 % gate.  A uniform translation leaves the corners' differences and
    so the level of detail unchanged (up to rounding), so the trilinear forward is differentiable along it."""
    B, F, H = 2, 300, 64
    faces = _faces(B, F, seed=31)
    uvs0 = _rand((F, 3, 2), 0.15, 0.85, seed=32) if tf == "bilinear" else _spread_uvs((F, 3, 2), 0.3, 0.7, seed=32)
    uvs0 = uvs0.clamp(0.05, 0.95)
    img = _smooth_image(*hw)
    g = torch.randn((B, 3, H, H), generator=torch.Generator().manual_seed(33)).to(DEV)
    uvs = uvs0.clone().requires_grad_(True)
    rgb = _render(faces, img, uvs, H, False, texture_filter=tf)[0]
    (rgb * g).sum().backward()
    grad = uvs.grad.double()

    def loss(u):
        with torch.no_grad():
            return float((_render(faces, img, u, H, False, texture_filter=tf)[0].double() * g.double()).sum())
    dirs = {"u": torch.zeros_like(uvs0), "v": torch.zeros_like(uvs0)}
    dirs["u"][..., 0] = 1.0
    dirs["v"][..., 1] = 1.0
    if tf == "bilinear":
        dirs["random"] = _rand((F, 3, 2), -1, 1, seed=34)
    h = 2e-3
    for name, d in dirs.items():
        analytic = float((grad * d.double()).sum())
        fd = (loss(uvs0 + h * d) - loss(uvs0 - h * d)) / (2 * h)
        assert abs(analytic) > 1.0, (name, analytic)
        assert abs(analytic - fd) <= 2e-2 * abs(fd), (name, analytic, fd)


@pytest.mark.parametrize("tf", ["bilinear", "trilinear"])
def test_rest_of_the_backward_is_unchanged(tf):
    """image, light and vertex gradients with and without face_uvs.requires_grad: the same pixels reach the same
    atomics (their order is not fixed from run to run, hence a gate at fp32 noise rather than equality).  Six runs of
    each on one H100 (700 W), bilinear: the same call twice differs by up to 4.2e-7 per tensor in the image gradient
    (2.1e-7 light, 5.4e-8 vertices), with against without face_uvs by up to 5.8e-7, and a run of the suite once went
    past 1e-6: the gate is 3e-6, about 25 ulps of each tensor's largest element.  A lost or doubled contribution moves
    an element by a whole pixel's share, far more than that."""
    B, F, H = 2, 400, 64
    faces0 = _faces(B, F, seed=41)
    uvs0, img0 = _spread_uvs((F, 3, 2), 0, 1, seed=42), _rand((1, 96, 80, 3), seed=43)
    light0 = 0.5 + _rand((B, F, 3), seed=44)
    g = torch.randn((B, 3, H, H), generator=torch.Generator().manual_seed(45)).to(DEV)
    out = []
    for want_uv in (False, True):
        f, t, l = (x.clone().requires_grad_(True) for x in (faces0, img0, light0))
        u = uvs0.clone().requires_grad_(want_uv)
        rgb = _render(f, t, u, H, True, light=l, texture_filter=tf)[0]
        (rgb * g).sum().backward()
        out.append((rgb.detach(), f.grad, t.grad, l.grad, u.grad))
    (rgb0, gf0, gt0, gl0, gu0), (rgb1, gf1, gt1, gl1, gu1) = out
    assert gu0 is None and gu1 is not None and (gu1 != 0).any()
    assert torch.equal(rgb0, rgb1)
    assert rel_err(np_(gt1), np_(gt0)) <= 3e-6
    assert rel_err(np_(gl1), np_(gl0)) <= 3e-6
    assert rel_err(np_(gf1), np_(gf0)) <= 3e-6


@pytest.mark.parametrize("tf", ["bilinear", "trilinear"])
def test_shared_uvs_get_the_sum_over_items(tf):
    B, F = 3, 300
    faces = _faces(B, F, seed=51)
    base, img = _spread_uvs((F, 3, 2), 0, 1, seed=52), _rand((1, 64, 64, 3), seed=53)
    g = torch.randn((B, 3, 64, 64), generator=torch.Generator().manual_seed(54)).to(DEV)
    res = {}
    for kind in ("copy", "shared", "shared1", "expanded"):
        u0 = base.clone().requires_grad_(True)
        u = {"copy": lambda: u0[None].expand(B, -1, -1, -1).contiguous(), "shared": lambda: u0,
             "shared1": lambda: u0[None], "expanded": lambda: u0[None].expand(B, -1, -1, -1)}[kind]()
        rgb = _render(faces, img, u, 64, False, texture_filter=tf)[0]
        (rgb * g).sum().backward()
        res[kind] = u0.grad
    per_item = []
    for b in range(B):  # each item on its own
        u0 = base.clone().requires_grad_(True)
        rgb = _render(faces[b:b + 1], img, u0, 64, False, texture_filter=tf)[0]
        (rgb * g[b:b + 1]).sum().backward()
        per_item.append(u0.grad)
    want = torch.stack(per_item).sum(0)
    for kind, got in res.items():
        assert rel_err(np_(got), np_(want)) <= 1e-5, kind


@pytest.mark.parametrize("fill_back", [True, False])
def test_renderer_fused_matches_op_by_op(teapot, fill_back):
    import neural_renderer as nr
    v, f = teapot
    B = 2
    rot = np.array([[0.9, 0.0, 0.43], [0.0, 1.0, 0.0], [-0.43, 0.0, 0.9]], np.float32)
    vertices = torch.from_numpy(np.stack([v, v @ rot.T])).to(DEV)
    faces_idx = torch.from_numpy(np.stack([f, f])).to(DEV)
    uvs0 = _rand((f.shape[0], 3, 2), seed=2)
    image = _rand((B, 40, 56, 3), seed=3)
    g = torch.randn((B, 3, 128, 128), generator=torch.Generator().manual_seed(2)).to(DEV)
    grads = []
    for fused in (False, True):
        r = nr.Renderer()
        r.image_size = 128
        r.fill_back = fill_back
        r.fused = fused
        r.eye = nr.get_points_from_angles(2.732, 30, 40)
        r.light_direction = [0.3, 1.0, -0.2]
        uvs = uvs0.clone().requires_grad_(True)
        img = r.render(vertices, faces_idx, image, face_uvs=uvs)
        (img * g).sum().backward()
        grads.append(uvs.grad)
    assert (grads[0] != 0).any()
    assert rel_err(np_(grads[1]), np_(grads[0])) <= 1e-5


def test_two_part_backward_with_texture_hook():
    R = _R()
    B, F = 2, 800
    faces = _faces(B, F, seed=3)
    uvs0, img0 = _spread_uvs((F, 3, 2), 0, 1, seed=1), _rand((128, 128, 3), seed=2)
    g = torch.randn((B, 3, 64, 64), generator=torch.Generator().manual_seed(1)).to(DEV)

    def run(tf):
        u = uvs0.clone().requires_grad_(True)
        t = img0.clone().requires_grad_(True)
        rgb = R._run(faces, t, 64, False, 0.1, 100, 1e-4, (0, 0, 0), True, False, False, face_uvs=u, texture_filter=tf)[0]
        (rgb * g).sum().backward()
        return u.grad

    for tf in ("bilinear", "trilinear"):
        one = run(tf)
        seen = {}
        prev = R.set_texture_grad_hook(lambda grad_textures: seen.setdefault("called", True) and None)
        try:
            two = run(tf)
        finally:
            R.set_texture_grad_hook(prev)
        assert seen.get("called") and (one != 0).any()
        assert rel_err(np_(two), np_(one)) <= 1e-6, tf


def test_direct_abi_call_writes_every_face_and_accumulates():
    from neural_renderer_b200 import _lib as L
    lib = L.load()
    B, F, S = 2, 300, 64
    faces = _faces(B, F, seed=61)
    uvs, img = _spread_uvs((1, F, 3, 2), 0, 1, seed=62), _rand((1, 40, 30, 3), seed=63)
    u_ref = uvs.clone().requires_grad_(True)
    rgb, _, _, fim, wmap = _R()._run(faces, img, S, False, 0.1, 100, 1e-4, (0, 0, 0), True, False, False, face_uvs=u_ref)
    g = torch.randn(rgb.shape, generator=torch.Generator().manual_seed(64)).to(DEV)
    (rgb * g).sum().backward()
    dmap = _R()._run(faces, None, S, False, 0.1, 100, 1e-4, None, False, False, True)[2]
    flags = L.NR_RETURN_RGB | L.NR_TEX_UV | L.NR_TEX_SHARED | L.NR_UV_SHARED
    ws_bytes = lib.nr_b200_backward_workspace_bytes(B, F, S, 0, flags)
    ws = torch.empty((max(ws_bytes, 16),), dtype=torch.uint8, device=DEV)
    gfaces, gimg = torch.zeros_like(faces), torch.zeros_like(img)

    def call(grad_uvs, extra=0, grad_rgb=g):
        a = L.BackwardArgs()
        a.struct_size = ctypes.sizeof(L.BackwardArgs)
        a.flags = flags | extra
        a.batch_size, a.num_faces, a.raster_size, a.texture_size = B, F, S, 0
        a.eps = 1e-4
        p = lambda t: None if t is None else ctypes.c_void_p(t.data_ptr())
        a.faces, a.textures, a.face_uvs = p(faces), p(img), p(uvs)
        a.texture_height, a.texture_width = 40, 30
        a.face_index_map, a.weight_map, a.depth_map, a.rgb_map = p(fim), p(wmap), p(dmap), p(rgb.detach())
        a.grad_rgb = p(grad_rgb)
        a.grad_faces, a.grad_textures, a.grad_face_uvs = p(gfaces), p(gimg), p(grad_uvs)
        a.workspace, a.workspace_bytes = p(ws), ws.numel()
        L.check(lib.nr_b200_backward(ctypes.byref(a), None))
        torch.cuda.synchronize()

    out = torch.full_like(uvs, float("nan"))
    call(out)
    assert torch.isfinite(out).all()
    seen = torch.zeros(F, dtype=torch.bool, device=DEV)
    seen[fim[fim >= 0].long()] = True
    assert (~seen).any() and seen.any()
    assert (out[0][~seen] == 0).all()
    assert rel_err(np_(out), np_(u_ref.grad)) <= 1e-6
    # NR_GRAD_ACCUMULATE adds into what is there
    pre = _rand(uvs.shape, -1, 1, seed=65)
    acc = pre.clone()
    call(acc, L.NR_GRAD_ACCUMULATE)
    assert rel_err(np_(acc - pre), np_(out)) <= 1e-5
    # no upstream rgb gradient: zeros
    out = torch.full_like(uvs, float("nan"))
    call(out, grad_rgb=None)
    assert (out == 0).all()


def _square():
    """a camera-facing square of two triangles, front-facing only, texture coordinates over [0.2, 0.8]^2"""
    z, r = 2.0, 0.9
    v = torch.tensor([[-r, -r, z], [r, -r, z], [r, r, z], [-r, r, z]], dtype=torch.float32)
    t = torch.tensor([[0.2, 0.2], [0.8, 0.2], [0.8, 0.8], [0.2, 0.8]], dtype=torch.float32)
    tri = torch.tensor([[0, 1, 2], [0, 2, 3]])
    faces = v[tri][None].to(DEV)
    if _R()._run(faces, None, 64, False, 0.1, 100, 1e-4, None, False, True, False)[1].sum() == 0:
        tri = tri.flip(1)  # the other winding is the front one
        faces = v[tri][None].to(DEV)
    return faces, t[tri].to(DEV)


@pytest.mark.parametrize("tf, hw", [("bilinear", (64, 64)), ("trilinear", (256, 256))])
def test_adam_recovers_shifted_uvs(tf, hw):
    """target: the square rendered with its UVs shifted by (0.04, -0.03) (2.5 / 1.9 texels of a 64^2 image; the
    trilinear image is minified, LOD about 1.4); from the unshifted UVs, Adam on the L2 image loss must cut the UV error
    at least 10x"""
    faces, uv_true0 = _square()
    img = _smooth_image(*hw)
    uv_true = uv_true0 + torch.tensor([0.04, -0.03], device=DEV)
    with torch.no_grad():
        target = _render(faces, img, uv_true, 64, False, texture_filter=tf, bg=(0, 0, 0))[0]
    assert (target.sum(1) > 0).float().mean() > 0.5
    uvs = uv_true0.clone().requires_grad_(True)
    opt = torch.optim.Adam([uvs], lr=4e-3)
    sched = torch.optim.lr_scheduler.ExponentialLR(opt, 0.99)
    err0 = float((uvs - uv_true).abs().max())
    for _ in range(300):
        opt.zero_grad()
        rgb = _render(faces, img, uvs, 64, False, texture_filter=tf, bg=(0, 0, 0))[0]
        ((rgb - target) ** 2).sum().backward()
        opt.step()
        sched.step()
    err = float((uvs.detach() - uv_true).abs().max())
    assert err <= err0 / 10, (err0, err)
