"""GPU: soft RGB through a texture image (rasterize_soft(face_uvs=...), nr_b200_soft_rgb_uv[_backward]) against the
float64 oracle of tests/oracles_soft_uv.py, the identities it must keep (alpha = the soft silhouettes, repeatability,
geometry forms, trilinear = bilinear where nothing is minified, constant-colour faces = the cube path), every gradient
against float64 autograd and central differences, the direct C ABI, two fits and Renderer.render_soft.

Forward gate (DESIGN.md section 4q): the soft RGB's gate, 4 tol(sigma) + 5e-4 (section 4p), plus what the UV adds.  The
screen barycentrics carry about 1e-7 / |A| (|A| >= 0.01 here), so l' and uv carry about 1e-5 (UV spans <= 1).  A tap
position moves by (Wt - 1) times that and the sample by the image's texel difference times that: the smooth images here
change by at most 3 / (Wt - 1) per texel, so the sample moves by at most 3e-5, and rgb by twice that.  The trilinear
level of detail is continuous in its inputs (the blend at an integer LOD is the same from both sides), so its fp32
error moves the sample by far less.  1e-4 covers both."""
import ctypes
import math
import os

import numpy as np
import pytest
import torch

import oracles
import oracles_soft as osoft
import oracles_soft_uv as ouv
from helpers import elem_err, rel_err

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
SIGMAS = (1e-5, 1e-4, 1e-3)
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def tol(sigma):
    return 1e-6 / math.sqrt(sigma) + 1e-6


def tol_rgb(sigma):
    return 4 * tol(sigma) + 5e-4 + 1e-4


def _nr():
    import neural_renderer_b200 as nr
    return nr


def _soup(B, F, seed, **kw):
    from neural_renderer_b200 import synthetic
    return torch.from_numpy(synthetic.triangle_soup(B, F, seed=seed, **kw)).to(DEV)


def _special_faces(B, sigma, seed, F=24):
    """the silhouette tests' special faces on a soup (as tests/test_gpu_soft_rgb.py)"""
    soup = _soup(B, F, seed, size=(0.05, 0.3), duplicates=False)
    reach = math.sqrt(osoft.cut(sigma))
    o = 1.0 + 0.5 * reach
    extra = [[[-1.1, -1.0, 2.5], [1.2, -0.9, 2.6], [0.1, 1.3, 2.4]],
             [[-0.9, 0.95, 2.0], [0.9, 0.9, 2.0], [0.0, 0.97, 2.0]],
             [[o, -0.3, 1.2], [o + 0.2, 0.0, 1.2], [o, 0.3, 1.2]],
             [[-0.3, -o, 1.2], [0.3, -o, 1.2], [0.0, -o - 0.2, 1.2]],
             [[-0.5, 0.1, 0.05], [-0.2, 0.1, 1.0], [-0.4, 0.4, 1.0]],
             [[0.2, -0.5, 1.0], [0.5, -0.5, 150.0], [0.3, -0.2, 1.0]],
             [[-0.6, -0.6, 1.0], [-0.2, -0.2, 1.0], [-0.4, -0.4, 1.0]],
             [[0.6, 0.2, 1.0], [0.6, 0.2, 1.0], [0.6, 0.2, 1.0]]]
    ex = torch.tensor(extra, dtype=torch.float32, device=DEV)[None].expand(B, -1, -1, -1)
    return torch.cat((soup, ex), 1).contiguous()


def _image(Bt, H, W, seed):
    """a smooth image: a few low-frequency waves, values in [0.1, 0.9], at most 3 / (W - 1) change per texel"""
    g = torch.Generator().manual_seed(seed)
    y = torch.linspace(0, 1, H, dtype=torch.float64)[:, None]
    x = torch.linspace(0, 1, W, dtype=torch.float64)[None]
    out = []
    for _ in range(Bt):
        ph = torch.rand(3, 2, generator=g, dtype=torch.float64) * 6.28
        out.append(torch.stack([0.5 + 0.2 * torch.sin(2.0 * x + ph[c, 0]) * torch.cos(1.5 * y + ph[c, 1]) + 0.15 * x * y
                                for c in range(3)], -1))
    return torch.stack(out).float().to(DEV)


def _uvs(Bu, F, seed, lo=-0.05, hi=1.05):
    g = torch.Generator().manual_seed(seed)
    return (lo + (hi - lo) * torch.rand(Bu, F, 3, 2, generator=g)).to(DEV)


def _light(B, F, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return 0.5 + torch.rand(B, F, 3, device=DEV, generator=g)


def _pyramid(img):
    from neural_renderer_b200.rasterize import _MipPyramid
    return _MipPyramid.apply(img.contiguous())


def _oracle(faces, img, uvs, S, sigma, gamma, bg, fl, tri, cut_scale=1.0):
    tex, hw = (img.double(), None) if not tri else (_pyramid(img).double(), tuple(img.shape[1:3]))
    return ouv.soft_uv(faces.double(), tex, uvs.double(), S, sigma, gamma, 0.1, 100.0, bg,
                       None if fl is None else fl.double(), hw, cut_scale)


def _check_forward(rgb, alpha, faces, img, uvs, S, sigma, gamma, bg, fl, tri):
    lo_rgb, lo_a = _oracle(faces, img, uvs, S, sigma, gamma, bg, fl, tri, 1 - 1e-5)
    hi_rgb, hi_a = _oracle(faces, img, uvs, S, sigma, gamma, bg, fl, tri, 1 + 1e-5)

    def bracket(x, lo, hi):
        x = x.double()
        return torch.maximum(torch.minimum(lo, hi) - x, x - torch.maximum(lo, hi)).clamp_min(0).max().item()

    ea, er = bracket(alpha, lo_a, hi_a), bracket(rgb, lo_rgb, hi_rgb)
    assert ea <= tol(sigma), (ea, tol(sigma))
    assert er <= tol_rgb(sigma), (er, tol_rgb(sigma))


@pytest.mark.parametrize("S", [64, 127, 256, 257])
@pytest.mark.parametrize("sigma", SIGMAS)
def test_forward_vs_oracle(S, sigma):
    nr = _nr()
    i = S + int(-math.log10(sigma))
    B = 2
    gamma = (1e-4, 1e-2)[i % 2]
    tri = bool(i % 3 == 0) or S == 256
    shared_img, shared_uv, light = bool((i // 2) % 2), bool((i // 3) % 2), bool((i // 5) % 2) or S == 257
    faces = _special_faces(B, sigma, seed=i)
    F = faces.shape[1]
    Ht, Wt = (96, 128) if tri else (17, 23)
    img = _image(1 if shared_img else B, Ht, Wt, seed=i)
    uvs = _uvs(1 if shared_uv else B, F, seed=i)
    fl = _light(B, F, i) if light else None
    bg = (0.2, 0.4, 0.6)
    kw = dict(background_color=bg, face_light=fl, face_uvs=uvs if not shared_uv else uvs[0],
              texture_filter='trilinear' if tri else 'bilinear')
    rgb, alpha = nr.rasterize_soft(faces, img if not shared_img else img[0], S, sigma, gamma, **kw)
    assert rgb.shape == (B, 3, S, S) and alpha.shape == (B, S, S)
    _check_forward(rgb, alpha, faces, img, uvs, S, sigma, gamma, bg, fl, tri)
    assert torch.equal(alpha, nr.rasterize_soft_silhouettes(faces, S, sigma))
    rgb2, alpha2 = nr.rasterize_soft(faces, img if not shared_img else img[0], S, sigma, gamma, **kw)
    assert torch.equal(rgb, rgb2) and torch.equal(alpha, alpha2)


@pytest.mark.parametrize("tri", [False, True])
def test_shared_sets_equal_repeated_sets_and_indexed_equals_materialised(tri):
    nr = _nr()
    S, sigma, gamma, B = 96, 1e-4, 1e-3, 3
    v = torch.from_numpy(np.random.default_rng(3).uniform(-0.8, 0.8, (B, 30, 3)).astype(np.float32)).to(DEV)
    v[..., 2] = v[..., 2].abs() * 2 + 1.5
    idx = torch.from_numpy(np.random.default_rng(4).integers(0, 30, (40, 3)).astype(np.int32)).to(DEV)
    faces = osoft.gather_faces(v, idx).float().contiguous()
    img, uvs, fl = _image(1, 40, 50, 5), _uvs(1, 40, 6), _light(B, 40, 7)
    filt = 'trilinear' if tri else 'bilinear'
    ref = nr.rasterize_soft(faces, img[0], S, sigma, gamma, face_light=fl, face_uvs=uvs[0], texture_filter=filt)
    rep = nr.rasterize_soft(faces, img.expand(B, -1, -1, -1).contiguous(), S, sigma, gamma, face_light=fl,
                            face_uvs=uvs.expand(B, -1, -1, -1).contiguous(), texture_filter=filt)
    exp = nr.rasterize_soft(faces, img.expand(B, -1, -1, -1), S, sigma, gamma, face_light=fl,
                            face_uvs=uvs.expand(B, -1, -1, -1), texture_filter=filt)
    idx_ = nr.rasterize_soft(idx, img[0], S, sigma, gamma, vertices=v, face_light=fl, face_uvs=uvs[0], texture_filter=filt)
    for got in (rep, exp, idx_):
        assert torch.equal(got[0], ref[0]) and torch.equal(got[1], ref[1])
    assert ref[1].max() > 0.5


def test_trilinear_is_bilinear_bit_for_bit_without_minification():
    nr = _nr()
    S, sigma, gamma, B = 128, 1e-4, 1e-3, 2
    faces = _soup(B, 20, seed=8, size=(0.3, 0.6), duplicates=False)
    fl = _light(B, 20, 9)
    one = _image(B, 1, 1, 10)
    a = nr.rasterize_soft(faces, one, S, sigma, gamma, face_light=fl, face_uvs=_uvs(B, 20, 11))
    b = nr.rasterize_soft(faces, one, S, sigma, gamma, face_light=fl, face_uvs=_uvs(B, 20, 11), texture_filter='trilinear')
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    img = _image(B, 8, 8, 12)
    uvs = 0.4 + 0.02 * torch.rand(B, 20, 3, 2, device=DEV, generator=torch.Generator(device=DEV).manual_seed(13))
    a = nr.rasterize_soft(faces, img, S, sigma, gamma, face_light=fl, face_uvs=uvs)
    b = nr.rasterize_soft(faces, img, S, sigma, gamma, face_light=fl, face_uvs=uvs, texture_filter='trilinear')
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


def test_constant_colour_faces_match_the_cube_path():
    nr = _nr()
    S, sigma, gamma, B, F = 96, 1e-4, 1e-3, 2, 20
    faces = _soup(B, F, seed=14, size=(0.1, 0.4), duplicates=False)
    Ht, Wt = 6, 7
    img = torch.rand(1, Ht, Wt, 3, device=DEV, generator=torch.Generator(device=DEV).manual_seed(15))
    g = torch.Generator().manual_seed(16)
    cols, rows = torch.randint(0, Wt, (F,), generator=g), torch.randint(0, Ht, (F,), generator=g)
    uvs = torch.stack((cols.double() / (Wt - 1), 1.0 - rows.double() / (Ht - 1)), -1).float()[:, None].expand(F, 3, 2)
    uvs = uvs.contiguous().to(DEV)
    cubes = img[0, rows.to(DEV), cols.to(DEV)][None, :, None, None, None].expand(1, F, 2, 2, 2, 3).contiguous()
    fl = _light(B, F, 17)
    f1 = faces.clone().requires_grad_(True)
    f2 = faces.clone().requires_grad_(True)
    r1 = nr.rasterize_soft(f1, img[0], S, sigma, gamma, face_light=fl, face_uvs=uvs)
    r2 = nr.rasterize_soft(f2, cubes, S, sigma, gamma, face_light=fl)
    assert (r1[0] - r2[0]).abs().max().item() <= 1e-6
    assert torch.equal(r1[1], r2[1])
    w = torch.randn(B, 3, S, S, device=DEV, generator=torch.Generator(device=DEV).manual_seed(18))
    (r1[0] * w).sum().backward()
    (r2[0] * w).sum().backward()
    assert (f1.grad - f2.grad).abs().max().item() <= 1e-4 * max(1.0, f2.grad.abs().max().item())


# ------------------------------------------------------------------------------------------------ backward
def _grads(faces, img, uvs, fl, S, sigma, gamma, bg, g_rgb, g_a, tri):
    nr = _nr()
    f, t, u, l = (x.clone().requires_grad_(True) for x in (faces, img, uvs, fl))
    rgb, alpha = nr.rasterize_soft(f, t, S, sigma, gamma, background_color=bg, face_light=l, face_uvs=u,
                                   texture_filter='trilinear' if tri else 'bilinear')
    loss = (rgb * g_rgb).sum() + ((alpha * g_a).sum() if g_a is not None else 0)
    loss.backward()
    return f.grad, t.grad, u.grad, l.grad


def _oracle_grads(faces, img, uvs, fl, S, sigma, gamma, bg, g_rgb, g_a, tri):
    f, t, u, l = (x.double().requires_grad_(True) for x in (faces, img, uvs, fl))
    if tri:
        levels = oracles.pyramid64(t)
        tex, hw = torch.cat([x.reshape(x.shape[0], -1, 3) for x in levels], 1), tuple(img.shape[1:3])
    else:
        tex, hw = t, None
    rgb, alpha = ouv.soft_uv(f, tex, u, S, sigma, gamma, 0.1, 100.0, bg, l, hw)
    loss = (rgb * g_rgb.double()).sum() + ((alpha * g_a.double()).sum() if g_a is not None else 0)
    gs = torch.autograd.grad(loss, (f, t, u, l), allow_unused=True)
    return tuple(torch.zeros_like(x) if gx is None else gx for x, gx in zip((f, t, u, l), gs))


@pytest.mark.parametrize("tri", [False, True])
@pytest.mark.parametrize("shared", [False, True])
def test_backward_vs_float64_autograd(tri, shared):
    S, B, sigma, gamma = 64, 2, 1e-3, 1e-2
    faces = _special_faces(B, sigma, seed=41, F=12)
    F = faces.shape[1]
    img = _image(1 if shared else B, 48, 40, 42)
    uvs = _uvs(1 if shared else B, F, 43, lo=0.05, hi=0.95)
    fl = _light(B, F, 44)
    gen = torch.Generator(device=DEV).manual_seed(45)
    g_rgb = torch.randn(B, 3, S, S, device=DEV, generator=gen)
    g_a = torch.randn(B, S, S, device=DEV, generator=gen)
    bg = (0.3, 0.3, 0.3)
    got = _grads(faces, img, uvs, fl, S, sigma, gamma, bg, g_rgb, g_a, tri)
    ref = _oracle_grads(faces, img, uvs, fl, S, sigma, gamma, bg, g_rgb, g_a, tri)
    for name, a, r in zip(("faces", "image", "face_uvs", "face_light"), got, ref):
        a, r = a.double().cpu().numpy(), r.cpu().numpy()
        assert np.isfinite(a).all(), name
        assert rel_err(a, r) <= 5e-3, (name, rel_err(a, r))
        assert elem_err(a, r, floor=2e-2) <= 5e-2, (name, elem_err(a, r, floor=2e-2))
    assert got[0][..., 2].abs().max() > 0 and got[2].abs().max() > 0


def test_backward_vs_central_differences_of_the_forward():
    nr = _nr()
    S, sigma, gamma = 64, 1e-3, 1e-2
    faces = _soup(1, 6, seed=21, size=(0.15, 0.4), offscreen=False, duplicates=False)
    img, uvs, fl = _image(1, 24, 20, 22), _uvs(1, 6, 23, lo=0.1, hi=0.9), _light(1, 6, 24)
    w = torch.randn(1, 3, S, S, device=DEV, generator=torch.Generator(device=DEV).manual_seed(7))
    d2, _ = osoft.face_terms(faces.double(), osoft.pixel_centres(S, device=DEV))
    w = w * ((d2 - osoft.cut(sigma)).abs() > 2e-4).all(1).reshape(1, 1, S, S)   # blind near the cut-off (section 4p)
    gf, gt, gu, gl = _grads(faces, img, uvs, fl, S, sigma, gamma, (0.5, 0.5, 0.5), w, None, False)

    def loss(ff, tt, uu, ll):
        rgb, _ = nr.rasterize_soft(ff, tt, S, sigma, gamma, background_color=(0.5, 0.5, 0.5), face_light=ll, face_uvs=uu)
        return float((rgb.double() * w.double()).sum())

    def fd(x, idx, h, which):
        xp, xm = x.clone(), x.clone()
        xp[idx] += h
        xm[idx] -= h
        args = [faces, img, uvs, fl]
        args[which] = xp
        lp = loss(*args)
        args[which] = xm
        return (lp - loss(*args)) / (xp[idx] - xm[idx]).item()

    scale = gf.abs().max().item()
    for idx in [(0, 0, 0, 0), (0, 1, 1, 1), (0, 2, 2, 2), (0, 3, 0, 1), (0, 5, 2, 0)]:
        assert abs(fd(faces, idx, 2e-4, 0) - gf[idx].item()) <= 3e-2 * scale, idx
    # image and light enter linearly: differences are exact up to rounding
    for idx in [(0, 3, 4, 0), (0, 12, 9, 1), (0, 20, 15, 2)]:
        assert abs(fd(img, idx, 1e-2, 1) - gt[idx].item()) <= 1e-2 * max(gt.abs().max().item(), 1e-6), idx
    for idx in [(0, 0, 0), (0, 3, 2)]:
        assert abs(fd(fl, idx, 1e-2, 3) - gl[idx].item()) <= 1e-2 * max(gl.abs().max().item(), 1e-6), idx
    # UVs move taps within their cells for a step below a texel
    su = gu.abs().max().item()
    for idx in [(0, 0, 0, 0), (0, 2, 1, 1), (0, 4, 2, 0)]:
        assert abs(fd(uvs, idx, 1e-4, 2) - gu[idx].item()) <= 5e-2 * su, (idx, gu[idx].item())


# ------------------------------------------------------------------------------------------------ direct ABI
def _guarded(shape, fill=float("nan"), guard=16):
    n = int(np.prod(shape))
    buf = torch.full((n + 2 * guard,), fill, dtype=torch.float32, device=DEV)
    buf[:guard] = 7.0
    buf[-guard:] = 7.0
    return buf, buf[guard:guard + n].view(*shape)


@pytest.mark.parametrize("tri", [False, True])
def test_abi_poison_guards_nulls_and_accumulate(tri):
    from neural_renderer_b200 import _lib
    lib = _lib.load()
    nr = _nr()
    S, sigma, gamma, B, F = 48, 1e-4, 1e-3, 2, 16
    faces = _soup(B, F, seed=31, size=(0.1, 0.5), duplicates=False)
    img, uvs, fl = _image(B, 20, 24, 32), _uvs(1, F, 33), _light(B, F, 34)
    tex = _pyramid(img).detach().contiguous() if tri else img
    ref_rgb, ref_a = nr.rasterize_soft(faces, img, S, sigma, gamma, face_light=fl, face_uvs=uvs[0],
                                       texture_filter='trilinear' if tri else 'bilinear')
    a = _lib.SoftRgbArgs(struct_size=ctypes.sizeof(_lib.SoftRgbArgs))
    a.flags = _lib.NR_TEX_UV | _lib.NR_UV_SHARED | (_lib.NR_TEX_MIPMAP if tri else 0)
    a.batch_size, a.num_faces, a.image_size, a.texture_size = B, F, S, 0
    a.sigma, a.gamma, a.near_, a.far_, a.eps = sigma, gamma, 0.1, 100.0, float("nan")
    a.faces, a.textures, a.face_light = faces.data_ptr(), tex.data_ptr(), fl.data_ptr()
    bufs = {k: _guarded(s) for k, s in (("rgb", (B, 3, S, S)), ("alpha", (B, S, S)), ("state", (B, 2, S, S)))}
    a.rgb, a.alpha, a.state = (bufs[k][1].data_ptr() for k in ("rgb", "alpha", "state"))
    n = lib.nr_b200_soft_rgb_workspace_bytes(B, F, S, 0)
    ws = torch.empty(n, dtype=torch.uint8, device=DEV)
    a.workspace, a.workspace_bytes = ws.data_ptr(), n
    u = _lib.SoftUvArgs(struct_size=ctypes.sizeof(_lib.SoftUvArgs), texture_height=20, texture_width=24,
                        face_uvs=uvs.data_ptr())
    assert lib.nr_b200_soft_rgb_uv(ctypes.byref(a), ctypes.byref(u), None) == 0
    torch.cuda.synchronize()
    assert torch.equal(bufs["rgb"][1], ref_rgb) and torch.equal(bufs["alpha"][1], ref_a)
    for buf, _ in bufs.values():
        assert torch.all(buf[:16] == 7.0) and torch.all(buf[-16:] == 7.0)
    # backward: every allowed NULL, poisoned outputs, and accumulation doubling the result
    g_rgb = torch.randn(B, 3, S, S, device=DEV, generator=torch.Generator(device=DEV).manual_seed(35))
    a.grad_rgb = g_rgb.data_ptr()
    outs = {k: _guarded(s) for k, s in (("gf", (B, F, 3, 3)), ("gt", tuple(tex.shape)), ("gl", (B, F, 3)),
                                       ("gu", (F, 3, 2)))}
    a.grad_faces, a.grad_textures, a.grad_face_light = (outs[k][1].data_ptr() for k in ("gf", "gt", "gl"))
    u.grad_face_uvs = outs["gu"][1].data_ptr()
    assert lib.nr_b200_soft_rgb_uv_backward(ctypes.byref(a), ctypes.byref(u), None) == 0
    torch.cuda.synchronize()
    first = {k: v[1].clone() for k, v in outs.items()}
    for k, (buf, view) in outs.items():
        assert torch.isfinite(view).all(), k
        assert torch.all(buf[:16] == 7.0) and torch.all(buf[-16:] == 7.0), k
    assert first["gu"].abs().max() > 0 and first["gt"].abs().max() > 0
    a.flags |= _lib.NR_GRAD_ACCUMULATE
    assert lib.nr_b200_soft_rgb_uv_backward(ctypes.byref(a), ctypes.byref(u), None) == 0
    torch.cuda.synchronize()
    for k, (buf, view) in outs.items():
        torch.testing.assert_close(view, 2 * first[k], rtol=1e-4, atol=1e-5)
    a.flags &= ~_lib.NR_GRAD_ACCUMULATE
    a.grad_textures = a.grad_face_light = None
    u.grad_face_uvs = None
    assert lib.nr_b200_soft_rgb_uv_backward(ctypes.byref(a), ctypes.byref(u), None) == 0
    torch.cuda.synchronize()
    torch.testing.assert_close(outs["gf"][1], first["gf"], rtol=1e-4, atol=1e-5)


# ------------------------------------------------------------------------------------------------ fits and Renderer
def test_per_item_image_is_recovered():
    nr = _nr()
    S, sigma, gamma, B = 64, 1e-4, 1e-3, 2
    faces = _soup(B, 30, seed=51, size=(0.3, 0.6), duplicates=False)
    uvs = _uvs(B, 30, 52, lo=0.0, hi=1.0)
    target = _image(B, 8, 8, 53)
    with torch.no_grad():
        want, _ = nr.rasterize_soft(faces, target, S, sigma, gamma, face_uvs=uvs)
    img = torch.full_like(target, 0.5).requires_grad_(True)
    opt = torch.optim.Adam([img], lr=0.05)
    losses = []
    for _ in range(150):
        opt.zero_grad()
        rgb, _ = nr.rasterize_soft(faces, img, S, sigma, gamma, face_uvs=uvs)
        loss = ((rgb - want) ** 2).sum()
        loss.backward()
        opt.step()
        losses.append(loss.item())
    assert losses[-1] < 0.01 * losses[0], (losses[0], losses[-1])


def test_uv_offset_is_recovered():
    nr = _nr()
    S, sigma, gamma = 64, 1e-4, 1e-3
    faces = _soup(1, 20, seed=61, size=(0.3, 0.6), duplicates=False)
    base = _uvs(1, 20, 62, lo=0.3, hi=0.6)
    img = _image(1, 32, 32, 63)
    shift = torch.tensor([0.06, -0.04], device=DEV)
    with torch.no_grad():
        want, _ = nr.rasterize_soft(faces, img, S, sigma, gamma, face_uvs=base + shift)
    off = torch.zeros(2, device=DEV, requires_grad=True)
    opt = torch.optim.Adam([off], lr=0.005)
    for _ in range(200):
        opt.zero_grad()
        rgb, _ = nr.rasterize_soft(faces, img, S, sigma, gamma, face_uvs=base + off)
        ((rgb - want) ** 2).sum().backward()
        opt.step()
    assert (off.detach() - shift).abs().max().item() < 0.01, off


def test_example5_soft_lowers_its_loss():
    import importlib.util
    spec = importlib.util.spec_from_file_location("example5", os.path.join(ROOT, "examples", "example5_optimize_texture_image.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    losses = mod.run(30, soft_sigma=1e-4, soft_gamma=1e-3)
    assert np.isfinite(losses).all()
    assert np.mean(losses[-5:]) < 0.8 * np.mean(losses[:5]), (losses[:5], losses[-5:])


@pytest.mark.parametrize("tri", [False, True])
def test_renderer_fused_op_by_op_fill_back_and_gradients(tri):
    nr = _nr()
    d = np.load(os.path.join(os.path.dirname(__file__), "golden", "teapot.npz"))
    v = torch.from_numpy(d["vertices"].astype(np.float32)).to(DEV)[None].expand(2, -1, -1).contiguous()
    f = torch.from_numpy(d["faces"].astype(np.int32)).to(DEV)[None].expand(2, -1, -1)
    F = f.shape[1]
    img = _image(1, 64, 64, 71)[0]
    uvs = _uvs(1, F, 72, lo=0.0, hi=1.0)[0]
    out = {}
    for fused in (True, False):
        for fill_back in (False, True):
            r = nr.Renderer()
            r.image_size = 64
            r.eye = nr.get_points_from_angles(2.732, 30, -15)
            r.fused, r.fill_back = fused, fill_back
            r.texture_filter = 'trilinear' if tri else 'bilinear'
            vv = v.clone().requires_grad_(True)
            uu = uvs.clone().requires_grad_(True)
            rgb, alpha = r.render_soft(vv, f, img, 1e-4, 1e-3, face_uvs=uu)
            (rgb.sum() + alpha.sum()).backward()
            out[(fused, fill_back)] = (rgb.detach(), alpha.detach(), vv.grad, uu.grad)
    ref = out[(True, False)]
    assert ref[2].abs().max() > 0 and ref[3].abs().max() > 0
    for key, got in out.items():
        torch.testing.assert_close(got[0], ref[0], rtol=0, atol=1e-6)
        assert torch.equal(got[1], ref[1])
        torch.testing.assert_close(got[2], ref[2], rtol=1e-3, atol=1e-3 * ref[2].abs().max().item())
        torch.testing.assert_close(got[3], ref[3], rtol=1e-3, atol=1e-3 * ref[3].abs().max().item())
