"""GPU: soft RGB (rasterize_soft, nr_b200_soft_rgb[_backward]) against the float64 oracle of tests/oracles_soft_rgb.py,
alpha bit-identical to the soft silhouettes, determinism, the geometry forms, every gradient against float64 autograd
and central differences, the direct C ABI (poisoned outputs, guard words, NULLs, accumulation, refusals), three fits the
hard rasterizer's rgb cannot make, and Renderer.render_soft.

Forward gate (DESIGN.md section 4p): D_j errs as in the silhouettes (tol(sigma) = 1e-6 / sqrt(sigma) + 1e-6 per face,
five faces within reach).  A weight's exponent (zref - zp_j) / ((far - near) gamma) carries the fp32 error of zp_j, a few
ulps (about 5e-7 relative), times zp / ((far - near) gamma): 1e-4 at zp 2 and gamma 1e-4.  The screen barycentrics carry
about 1e-7 / |A| (|A| >= 0.01 for every face drawn here), which moves texture coordinates by ts times that and zp by the
depth spread times that.  Each relative weight error moves rgb by at most that error times |C_j - rgb| <= 2 (colours in
[0, 1], light <= 1.5).  So |rgb - oracle| <= 4 tol(sigma) + 5e-4 holds with margin; the cut-off is bracketed as for the
silhouettes."""
import ctypes
import math
import os

import numpy as np
import pytest
import torch

import oracles_soft as osoft
import oracles_soft_rgb as orgb
from helpers import elem_err, rel_err

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
SIGMAS = (1e-5, 1e-4, 1e-3)


def tol(sigma):
    return 1e-6 / math.sqrt(sigma) + 1e-6


def tol_rgb(sigma):
    return 4 * tol(sigma) + 5e-4


def _nr():
    import neural_renderer_b200 as nr
    return nr


def _soup(B, F, seed, **kw):
    from neural_renderer_b200 import synthetic
    return torch.from_numpy(synthetic.triangle_soup(B, F, seed=seed, **kw)).to(DEV)


def _special_faces(B, sigma, seed, F=24):
    """the silhouette tests' special faces on a soup: wider than the wide-list cap, a sliver, off the image within
    reach, straddling near / far, collinear and a point"""
    soup = _soup(B, F, seed, size=(0.05, 0.3), duplicates=False)
    reach = math.sqrt(osoft.cut(sigma))
    o = 1.0 + 0.5 * reach
    extra = [[[-1.1, -1.0, 2.5], [1.2, -0.9, 2.6], [0.1, 1.3, 2.4]],           # covers the image: > 16 tiles
             [[-0.9, 0.95, 2.0], [0.9, 0.9, 2.0], [0.0, 0.97, 2.0]],            # a wide sliver
             [[o, -0.3, 1.2], [o + 0.2, 0.0, 1.2], [o, 0.3, 1.2]],              # right of the image, within reach
             [[-0.3, -o, 1.2], [0.3, -o, 1.2], [0.0, -o - 0.2, 1.2]],           # below the image, within reach
             [[-0.5, 0.1, 0.05], [-0.2, 0.1, 1.0], [-0.4, 0.4, 1.0]],           # one vertex nearer than near
             [[0.2, -0.5, 1.0], [0.5, -0.5, 150.0], [0.3, -0.2, 1.0]],          # one vertex beyond far
             [[-0.6, -0.6, 1.0], [-0.2, -0.2, 1.0], [-0.4, -0.4, 1.0]],         # collinear: zero area
             [[0.6, 0.2, 1.0], [0.6, 0.2, 1.0], [0.6, 0.2, 1.0]]]               # a point
    ex = torch.tensor(extra, dtype=torch.float32, device=DEV)[None].expand(B, -1, -1, -1)
    return torch.cat((soup, ex), 1).contiguous()


def _inputs(B, F, ts, seed, shared_tex=False, light=True):
    g = torch.Generator(device=DEV).manual_seed(seed)
    tex = torch.rand((1 if shared_tex else B), F, ts, ts, ts, 3, device=DEV, generator=g)
    fl = (0.5 + torch.rand(B, F, 3, device=DEV, generator=g)) if light else None
    return tex, fl


def _oracle(faces, tex, S, sigma, gamma, bg, fl, cut_scale=1.0, eps=1e-4):
    return orgb.soft_rgb(faces.double(), tex.double(), S, sigma, gamma, 0.1, 100.0, eps, bg,
                         None if fl is None else fl.double(), cut_scale)


def _check_forward(rgb, alpha, faces, tex, S, sigma, gamma, bg, fl):
    lo_rgb, lo_a = _oracle(faces, tex, S, sigma, gamma, bg, fl, 1 - 1e-5)
    hi_rgb, hi_a = _oracle(faces, tex, S, sigma, gamma, bg, fl, 1 + 1e-5)

    def bracket(x, lo, hi):
        x = x.double()
        return torch.maximum(torch.minimum(lo, hi) - x, x - torch.maximum(lo, hi)).clamp_min(0).max().item()

    ea, er = bracket(alpha, lo_a, hi_a), bracket(rgb, lo_rgb, hi_rgb)
    assert ea <= tol(sigma), (ea, tol(sigma))
    assert er <= tol_rgb(sigma), (er, tol_rgb(sigma))
    return er


@pytest.mark.parametrize("S", [64, 127, 256, 257])
@pytest.mark.parametrize("sigma", SIGMAS)
def test_forward_vs_oracle(S, sigma):
    nr = _nr()
    i = S + int(-math.log10(sigma))
    B = 2
    gamma = (1e-4, 1e-2)[i % 2]
    ts = (2, 4, 5)[i % 3]
    shared, light = bool((i // 2) % 2), bool((i // 3) % 2) or S == 257
    faces = _special_faces(B, sigma, seed=i)
    tex, fl = _inputs(B, faces.shape[1], ts, seed=i, shared_tex=shared, light=light)
    bg = (0.2, 0.4, 0.6)
    rgb, alpha = nr.rasterize_soft(faces, tex, S, sigma, gamma, background_color=bg, face_light=fl)
    assert rgb.shape == (B, 3, S, S) and alpha.shape == (B, S, S)
    _check_forward(rgb, alpha, faces, tex, S, sigma, gamma, bg, fl)
    # alpha is the soft silhouettes' bit for bit; rgb repeats bit for bit
    assert torch.equal(alpha, nr.rasterize_soft_silhouettes(faces, S, sigma))
    rgb2, alpha2 = nr.rasterize_soft(faces, tex, S, sigma, gamma, background_color=bg, face_light=fl)
    assert torch.equal(rgb, rgb2) and torch.equal(alpha, alpha2)


@pytest.mark.parametrize("gamma", [1e-4, 1e-2])
@pytest.mark.parametrize("ts", [2, 4, 5])
def test_forward_gamma_ts_texture_sharing_and_light(gamma, ts):
    nr = _nr()
    S, sigma, B = 96, 1e-4, 2
    faces = _special_faces(B, sigma, seed=ts * 7 + int(gamma * 1e4))
    bg = (0.9, 0.1, 0.3)
    for shared in (False, True):
        for light in (False, True):
            tex, fl = _inputs(B, faces.shape[1], ts, seed=ts, shared_tex=shared, light=light)
            rgb, alpha = nr.rasterize_soft(faces, tex, S, sigma, gamma, background_color=bg, face_light=fl)
            _check_forward(rgb, alpha, faces, tex, S, sigma, gamma, bg, fl)
            if shared:  # one shared set == the same cubes repeated per item
                r2, _ = nr.rasterize_soft(faces, tex.expand(B, -1, -1, -1, -1, -1).contiguous(), S, sigma, gamma,
                                          background_color=bg, face_light=fl)
                assert torch.equal(rgb, r2)


def _teapot(B=2):
    nr = _nr()
    d = np.load(os.path.join(os.path.dirname(__file__), "golden", "teapot.npz"))
    v = torch.from_numpy(d["vertices"].astype(np.float32)).to(DEV)
    f = torch.from_numpy(d["faces"].astype(np.int32)).to(DEV)
    r = nr.Renderer()
    r.eye = nr.get_points_from_angles(2.732, 30, -15)
    return r._transform(v[None].expand(B, -1, -1).contiguous()).contiguous(), f


def test_geometry_forms_are_bit_identical():
    nr = _nr()
    S, sigma, gamma = 128, 1e-4, 1e-4
    verts, idx = _teapot(2)
    B, Nv = verts.shape[:2]
    F = idx.shape[0]
    tex, fl = _inputs(B, F, 3, seed=3)
    idx_b = idx[None].repeat(B, 1, 1).clone()
    idx_b[0, 5, 1] = Nv
    idx_b[1, 7, 2] = -3
    faces = osoft.gather_faces(verts, idx_b).float().contiguous()
    r_mat = nr.rasterize_soft(faces, tex, S, sigma, gamma, face_light=fl)
    r_idx = nr.rasterize_soft(idx_b, tex, S, sigma, gamma, vertices=verts, face_light=fl)
    assert torch.equal(r_mat[0], r_idx[0]) and torch.equal(r_mat[1], r_idx[1])
    faces_s = osoft.gather_faces(verts, idx).float()
    ref = nr.rasterize_soft(faces_s, tex, S, sigma, gamma, face_light=fl)
    for ix in (idx, idx[None], idx[None].expand(B, -1, -1)):
        got = nr.rasterize_soft(ix, tex, S, sigma, gamma, vertices=verts, face_light=fl)
        assert torch.equal(got[0], ref[0]) and torch.equal(got[1], ref[1])
    assert ref[1].max() > 0.99


# ------------------------------------------------------------------------------------------------ backward
def _grads(faces, tex, fl, S, sigma, gamma, bg, g_rgb, g_a):
    """the product's gradients (faces, textures, face_light)"""
    nr = _nr()
    f = faces.clone().requires_grad_(True)
    t = tex.clone().requires_grad_(True)
    l = fl.clone().requires_grad_(True)
    rgb, alpha = nr.rasterize_soft(f, t, S, sigma, gamma, background_color=bg, face_light=l)
    loss = 0
    if g_rgb is not None:
        loss = loss + (rgb * g_rgb).sum()
    if g_a is not None:
        loss = loss + (alpha * g_a).sum()
    loss.backward()
    return f.grad, t.grad, l.grad


def _oracle_grads(faces, tex, fl, S, sigma, gamma, bg, g_rgb, g_a):
    f = faces.double().requires_grad_(True)
    t = tex.double().requires_grad_(True)
    l = fl.double().requires_grad_(True)
    rgb, alpha = orgb.soft_rgb(f, t, S, sigma, gamma, 0.1, 100.0, 1e-4, bg, l)
    loss = 0
    if g_rgb is not None:
        loss = loss + (rgb * g_rgb.double()).sum()
    if g_a is not None:
        loss = loss + (alpha * g_a.double()).sum()
    gs = torch.autograd.grad(loss, (f, t, l), allow_unused=True)
    return tuple(torch.zeros_like(x) if gx is None else gx for x, gx in zip((f, t, l), gs))


@pytest.mark.parametrize("which", ["rgb", "alpha", "both"])
@pytest.mark.parametrize("sigma,gamma", [(1e-4, 1e-2), (1e-3, 1e-3)])
def test_backward_vs_float64_autograd(which, sigma, gamma):
    S, B, ts = 64, 2, 3
    faces = _special_faces(B, sigma, seed=41, F=12)
    # keep the zero-area and off-range faces, drop the image-wide one (its gradient is dominated by a few pixels)
    tex, fl = _inputs(B, faces.shape[1], ts, seed=42)
    gen = torch.Generator(device=DEV).manual_seed(43)
    g_rgb = torch.randn(B, 3, S, S, device=DEV, generator=gen) if which != "alpha" else None
    g_a = torch.randn(B, S, S, device=DEV, generator=gen) if which != "rgb" else None
    bg = (0.3, 0.3, 0.3)
    got = _grads(faces, tex, fl, S, sigma, gamma, bg, g_rgb, g_a)
    ref = _oracle_grads(faces, tex, fl, S, sigma, gamma, bg, g_rgb, g_a)
    names = ("faces", "textures", "face_light")
    for name, a, r in zip(names, got, ref):
        a, r = a.double().cpu().numpy(), r.cpu().numpy()
        assert np.isfinite(a).all(), name
        if which == "alpha" and name != "faces":
            assert np.all(a == 0), name
            continue
        assert rel_err(a, r) <= 5e-3, (name, rel_err(a, r))
        assert elem_err(a, r, floor=2e-2) <= 5e-2, (name, elem_err(a, r, floor=2e-2))
    if which != "alpha":
        assert got[0][..., 2].abs().max() > 0  # the vertex depths receive a gradient
    # faces that take no part get exactly nothing
    F0 = faces.shape[1] - 8
    assert torch.all(got[0][:, F0 + 4:F0 + 6] == 0)


def test_backward_vs_central_differences_of_the_forward():
    nr = _nr()
    S, sigma, gamma, ts = 64, 1e-3, 1e-2, 2
    faces = _soup(1, 6, seed=21, size=(0.15, 0.4), offscreen=False, duplicates=False)
    tex, fl = _inputs(1, 6, ts, seed=22)
    w = torch.randn(1, 3, S, S, device=DEV, generator=torch.Generator(device=DEV).manual_seed(7))
    # A face entering reach at the cut-off (D = 1e-4) outweighs the background term, whose weight is exp(-zn / gamma)
    # smaller: rgb jumps there by design (the cut-off is held fixed).  Differences are taken with the loss blind to
    # pixels whose d^2 to some face lies within 2e-4 of the cut-off, which the steps below cannot cross.
    d2, _ = osoft.face_terms(faces.double(), osoft.pixel_centres(S, device=DEV))
    smooth = ((d2 - osoft.cut(sigma)).abs() > 2e-4).all(1).reshape(1, 1, S, S)
    w = w * smooth
    gf, gt, gl = _grads(faces, tex, fl, S, sigma, gamma, (0.5, 0.5, 0.5), w, None)

    def loss(ff, tt, ll):
        rgb, _ = nr.rasterize_soft(ff, tt, S, sigma, gamma, background_color=(0.5, 0.5, 0.5), face_light=ll)
        return float((rgb.double() * w.double()).sum())

    h = 2e-4
    scale = gf.abs().max().item()
    for (fi, k, c) in [(0, 0, 0), (1, 1, 1), (2, 2, 2), (3, 0, 1), (5, 2, 0), (4, 1, 2)]:
        fp, fm = faces.clone(), faces.clone()
        fp[0, fi, k, c] += h
        fm[0, fi, k, c] -= h
        fd = (loss(fp, tex, fl) - loss(fm, tex, fl)) / (fp[0, fi, k, c] - fm[0, fi, k, c]).item()
        assert abs(fd - gf[0, fi, k, c].item()) <= 3e-2 * scale, (fi, k, c, fd, gf[0, fi, k, c].item())
    # the texture and the light are linear in the forward: differences are exact up to rounding
    for (fi, corner, ch) in [(0, 0, 0), (2, 7, 1), (5, 3, 2)]:
        tp, tm = tex.clone(), tex.clone()
        idx = (0, fi) + tuple((corner >> k) & 1 for k in range(3)) + (ch,)
        tp[idx] += 1e-2
        tm[idx] -= 1e-2
        fd = (loss(faces, tp, fl) - loss(faces, tm, fl)) / 2e-2
        assert abs(fd - gt[idx].item()) <= 1e-2 * max(gt.abs().max().item(), 1e-6), (idx, fd, gt[idx].item())
    for (fi, ch) in [(0, 0), (3, 2)]:
        lp, lm = fl.clone(), fl.clone()
        lp[0, fi, ch] += 1e-2
        lm[0, fi, ch] -= 1e-2
        fd = (loss(faces, tex, lp) - loss(faces, tex, lm)) / 2e-2
        assert abs(fd - gl[0, fi, ch].item()) <= 1e-2 * max(gl.abs().max().item(), 1e-6), (fi, ch, fd)


# ------------------------------------------------------------------------------------------------ direct ABI
def _abi_call(faces=None, verts=None, idx=None, tex=None, fl=None, S=48, sigma=1e-4, gamma=1e-3, rgb=None, alpha=None,
              state=None, g_rgb=None, g_a=None, gf=None, gv=None, gt=None, gl=None, flags=0, backward=False):
    from neural_renderer_b200 import _lib
    lib = _lib.load()
    a = _lib.SoftRgbArgs()
    a.struct_size = ctypes.sizeof(_lib.SoftRgbArgs)
    ptr = lambda t: None if t is None else ctypes.c_void_p(t.data_ptr())  # noqa: E731
    if verts is not None:
        flags |= _lib.NR_FACES_INDEXED | (_lib.NR_INDICES_SHARED if idx.dim() == 2 else 0)
        a.vertices, a.face_indices, a.num_vertices, a.num_faces, B = ptr(verts), ptr(idx), verts.shape[1], idx.shape[-2], verts.shape[0]
    else:
        a.faces, a.num_faces, B = ptr(faces), faces.shape[1], faces.shape[0]
    if tex.shape[0] == 1 and B > 1:
        flags |= _lib.NR_TEX_SHARED
    a.flags, a.batch_size, a.image_size, a.texture_size = flags, B, S, tex.shape[2]
    a.sigma, a.gamma, a.near_, a.far_, a.eps = sigma, gamma, 0.1, 100.0, 1e-4
    a.background[:] = (0.1, 0.2, 0.3)
    a.textures, a.face_light = ptr(tex), ptr(fl)
    a.rgb, a.alpha, a.state = ptr(rgb), ptr(alpha), ptr(state)
    a.grad_rgb, a.grad_alpha = ptr(g_rgb), ptr(g_a)
    a.grad_faces, a.grad_vertices, a.grad_textures, a.grad_face_light = ptr(gf), ptr(gv), ptr(gt), ptr(gl)
    n = lib.nr_b200_soft_rgb_workspace_bytes(B, a.num_faces, S, flags)
    ws = torch.full((max(n, 16),), 0xAB, dtype=torch.uint8, device=DEV)
    a.workspace, a.workspace_bytes = ptr(ws), n
    fn = lib.nr_b200_soft_rgb_backward if backward else lib.nr_b200_soft_rgb
    rc = fn(ctypes.byref(a), ctypes.c_void_p(torch.cuda.current_stream(DEV).cuda_stream))
    torch.cuda.synchronize()
    return rc, lib.nr_b200_last_launch_count()


def _guarded(shape, fill=float("nan"), guard=16):
    buf = torch.full((int(np.prod(shape)) + guard,), fill, dtype=torch.float32, device=DEV)
    buf[-guard:] = 12345.0
    return buf, buf[:-guard].view(shape)


@pytest.mark.parametrize("indexed", [False, True])
def test_abi_poison_guards_nulls_accumulate_and_refusals(indexed):
    nr = _nr()
    B, S, sigma, gamma, ts = 2, 48, 1e-4, 1e-3, 3
    faces = _special_faces(B, sigma, seed=31, F=10)
    F = faces.shape[1]
    Nv = F * 3
    verts = faces.reshape(B, Nv, 3).contiguous()
    idx = torch.arange(Nv, dtype=torch.int32, device=DEV).reshape(-1, 3)
    geo = dict(verts=verts, idx=idx) if indexed else dict(faces=faces)
    tex, fl = _inputs(B, F, ts, seed=32)
    ref_rgb, ref_a = nr.rasterize_soft(faces, tex, S, sigma, gamma, background_color=(0.1, 0.2, 0.3), face_light=fl)
    bufs = [_guarded(s) for s in ((B, 3, S, S), (B, S, S), (B, 2, S, S))]
    (rb, rgb), (ab, alpha), (sb, state) = bufs
    rc, n = _abi_call(**geo, tex=tex, fl=fl, S=S, sigma=sigma, gamma=gamma, rgb=rgb, alpha=alpha, state=state)
    assert rc == 0 and n >= 6
    assert torch.equal(rgb, ref_rgb) and torch.equal(alpha, ref_a) and torch.isfinite(state).all()
    assert all(torch.all(b[-16:] == 12345.0) for b, _ in bufs)
    # backward: every NaN-poisoned gradient overwritten, guards intact, equal to the autograd path
    gen = torch.Generator(device=DEV).manual_seed(33)
    g_rgb, g_a = torch.randn(B, 3, S, S, device=DEV, generator=gen), torch.randn(B, S, S, device=DEV, generator=gen)
    gshape = (B, Nv, 3) if indexed else tuple(faces.shape)

    def run(flags=0, fill=float("nan"), **kw):
        outs = dict(geo=_guarded(gshape, fill), gt=_guarded(tuple(tex.shape), fill), gl=_guarded((B, F, 3), fill))
        for k in list(kw):
            if kw[k] is False:
                outs.pop(k)
                kw.pop(k)
        args = dict(g_rgb=g_rgb, g_a=g_a)
        args.update(kw)
        gk = "gv" if indexed else "gf"
        rc, _ = _abi_call(**geo, tex=tex, fl=fl, S=S, sigma=sigma, gamma=gamma, rgb=rgb, alpha=alpha, state=state,
                          backward=True, flags=flags, **{gk: outs["geo"][1]}, gt=outs.get("gt", (None, None))[1],
                          gl=outs.get("gl", (None, None))[1], **args)
        assert rc == 0
        for b, _ in outs.values():
            assert torch.all(b[-16:] == 12345.0)
        return {k: v[1] for k, v in outs.items()}

    got = run()
    f = faces.clone().requires_grad_(True)
    t = tex.clone().requires_grad_(True)
    l = fl.clone().requires_grad_(True)
    r, a = nr.rasterize_soft(f, t, S, sigma, gamma, background_color=(0.1, 0.2, 0.3), face_light=l)
    ((r * g_rgb).sum() + (a * g_a).sum()).backward()
    want = dict(geo=f.grad.reshape(gshape), gt=t.grad, gl=l.grad)
    for k in want:
        assert torch.isfinite(got[k]).all(), k
        assert rel_err(got[k].cpu().numpy(), want[k].cpu().numpy()) <= 1e-5, k
    # NR_GRAD_ACCUMULATE adds into every buffer
    from neural_renderer_b200 import _lib
    acc = run(flags=_lib.NR_GRAD_ACCUMULATE, fill=0.5)
    for k in want:
        assert rel_err((acc[k] - 0.5).cpu().numpy(), want[k].cpu().numpy()) <= 1e-5, k
    # the NULLs the header allows: grad_textures / grad_face_light not wanted, grad_rgb / grad_alpha = zeros
    only_geo = run(gt=False, gl=False)
    assert rel_err(only_geo["geo"].cpu().numpy(), want["geo"].cpu().numpy()) <= 1e-5
    zero = run(g_rgb=None, g_a=None)
    assert all(torch.all(v == 0) for v in zero.values())
    no_rgb = run(g_rgb=None)
    assert torch.all(no_rgb["gt"] == 0) and torch.all(no_rgb["gl"] == 0) and no_rgb["geo"].abs().sum() > 0
    # without a light the sample is unlit
    r0, _ = nr.rasterize_soft(faces, tex, S, sigma, gamma, background_color=(0.1, 0.2, 0.3))
    _abi_call(**geo, tex=tex, fl=None, S=S, sigma=sigma, gamma=gamma, rgb=rgb, alpha=alpha, state=state)
    assert torch.equal(rgb, r0)
    # refusals: nothing launched, outputs untouched
    rb2, rgb2 = _guarded((B, 3, S, S), fill=7.0)
    for bad in (dict(sigma=0.0), dict(gamma=0.0), dict(gamma=float("nan")), dict(S=0)):
        rc, n = _abi_call(**geo, tex=tex, fl=fl, rgb=rgb2, alpha=alpha, state=state,
                          **{"S": S, "sigma": sigma, "gamma": gamma, **bad})
        assert rc == -1 and n == 0 and torch.all(rgb2 == 7.0) and torch.all(rb2[-16:] == 12345.0)
    rc, n = _abi_call(**geo, tex=tex, fl=fl, S=S, rgb=rgb2, alpha=alpha, state=state, flags=_lib.NR_TEX_FILL_BACK)
    assert rc == -1 and n == 0 and torch.all(rgb2 == 7.0)


# ------------------------------------------------------------------------------------------------ what the hard rgb cannot do
def _square(cx, cy, half, z):
    """two faces of an axis-aligned square, depth z (a tensor, so that it can require grad)"""
    zz = z.expand(4) if z.dim() == 0 else z
    c = torch.stack([torch.tensor([cx - half, cy - half], device=DEV), torch.tensor([cx + half, cy - half], device=DEV),
                     torch.tensor([cx + half, cy + half], device=DEV), torch.tensor([cx - half, cy + half], device=DEV)])
    v = torch.cat((c, zz[:, None]), 1)
    return torch.stack((v[[0, 1, 2]], v[[0, 2, 3]]))


def test_depth_order_is_learned():
    nr = _nr()
    S, sigma, gamma = 64, 1e-4, 1e-3
    red = torch.tensor([1.0, 0.0, 0.0], device=DEV)
    blue = torch.tensor([0.0, 0.0, 1.0], device=DEV)
    tex = torch.cat((red.expand(1, 2, 2, 2, 2, 3), blue.expand(1, 2, 2, 2, 2, 3)), 1).contiguous()
    z_blue = torch.tensor(2.0, device=DEV)
    with torch.no_grad():  # target: red in front (z 1.5 < 2)
        tgt = torch.cat((_square(-0.1, 0.0, 0.4, torch.tensor(1.5, device=DEV)), _square(0.1, 0.0, 0.4, z_blue)))[None]
        target, _ = nr.rasterize_soft(tgt, tex, S, sigma, gamma)
    z = torch.tensor(2.5, device=DEV, requires_grad=True)  # red starts behind blue
    # the hard rasterizer's rgb gives the depth of the red square no gradient
    zr = z.detach().clone().requires_grad_(True)
    hf = torch.cat((_square(-0.1, 0.0, 0.4, zr), _square(0.1, 0.0, 0.4, z_blue)))[None]
    hard = nr.rasterize(hf, tex, S, False)
    ((hard - target) ** 2).sum().backward()
    assert zr.grad is not None and zr.grad.item() == 0.0
    opt = torch.optim.Adam([z], lr=0.02)
    for _ in range(150):
        opt.zero_grad()
        f = torch.cat((_square(-0.1, 0.0, 0.4, z), _square(0.1, 0.0, 0.4, z_blue)))[None]
        img, _ = nr.rasterize_soft(f, tex, S, sigma, gamma)
        ((img - target) ** 2).sum().backward()
        opt.step()
    assert z.item() < 1.9, z.item()  # red is in front now
    with torch.no_grad():
        f = torch.cat((_square(-0.1, 0.0, 0.4, z), _square(0.1, 0.0, 0.4, z_blue)))[None]
        img, _ = nr.rasterize_soft(f, tex, S, sigma, gamma)
    assert (img - target).abs().max() < 0.1


def _tri_at(cx, cy, s=4.0 / 128):
    return torch.stack([torch.stack([cx - s / 2, cy - s / 3, torch.full_like(cx, 1.5)]),
                        torch.stack([cx + s / 2, cy - s / 3, torch.full_like(cx, 1.5)]),
                        torch.stack([cx, cy + 2 * s / 3, torch.full_like(cx, 1.5)])])[None, None]


def test_translation_fit_from_the_rgb_loss_alone():
    nr = _nr()
    S, sigma, gamma = 128, 1e-4, 1e-4
    px = 2.0 / S
    tex = torch.tensor([0.9, 0.6, 0.1], device=DEV).expand(1, 1, 2, 2, 2, 3).contiguous()
    bg = (0.1, 0.1, 0.4)
    tx, ty = torch.tensor(0.1013, device=DEV), torch.tensor(-0.0521, device=DEV)
    with torch.no_grad():
        target, _ = nr.rasterize_soft(_tri_at(tx, ty), tex, S, sigma, gamma, background_color=bg)
        ht = nr.rasterize_silhouettes(_tri_at(tx, ty), S, False)
        hs = nr.rasterize_silhouettes(_tri_at(tx + 3 * px, ty), S, False)
    assert (ht * hs).sum() == 0  # no overlap at the start
    shift = torch.tensor([3 * px, 0.0], device=DEV, requires_grad=True)
    opt = torch.optim.Adam([shift], lr=0.2 * px)
    steps = 400
    for it in range(steps):
        for gr in opt.param_groups:
            gr["lr"] = px * (0.005 + 0.195 * 0.5 * (1 + math.cos(math.pi * it / steps)))
        opt.zero_grad()
        img, _ = nr.rasterize_soft(_tri_at(tx + shift[0], ty + shift[1]), tex, S, sigma, gamma, background_color=bg)
        ((img - target) ** 2).sum().backward()
        opt.step()
    err_px = (shift.detach().abs().max() / px).item()
    assert err_px < 0.1, err_px


def test_cube_textures_are_recovered():
    nr = _nr()
    S, sigma, gamma, ts = 64, 1e-4, 1e-4, 2
    faces = _soup(2, 12, seed=51, size=(0.2, 0.5), offscreen=False, duplicates=False)
    gen = torch.Generator(device=DEV).manual_seed(52)
    truth = torch.rand(2, 12, ts, ts, ts, 3, device=DEV, generator=gen)
    with torch.no_grad():
        target, _ = nr.rasterize_soft(faces, truth, S, sigma, gamma)
    tex = torch.full_like(truth, 0.5).requires_grad_(True)
    opt = torch.optim.Adam([tex], lr=0.05)
    losses = []
    for _ in range(300):
        opt.zero_grad()
        img, _ = nr.rasterize_soft(faces, tex, S, sigma, gamma)
        loss = ((img - target) ** 2).mean()
        loss.backward()
        opt.step()
        losses.append(loss.item())
    assert losses[-1] < 1e-2 * losses[0], (losses[0], losses[-1])


# ------------------------------------------------------------------------------------------------ Renderer
def test_renderer_fused_op_by_op_fill_back_and_camera_gradient():
    nr = _nr()
    d = np.load(os.path.join(os.path.dirname(__file__), "golden", "teapot.npz"))
    v = torch.from_numpy(d["vertices"].astype(np.float32)).to(DEV)[None].repeat(2, 1, 1)
    f = torch.from_numpy(d["faces"].astype(np.int32)).to(DEV)[None].expand(2, -1, -1)
    tex = torch.rand(1, f.shape[1], 2, 2, 2, 3, device=DEV, generator=torch.Generator(device=DEV).manual_seed(9))
    r = nr.Renderer()
    r.image_size = 128
    r.background_color = [0.2, 0.3, 0.4]
    r.eye = nr.get_points_from_angles(2.732, 20, 30)
    outs = {}
    for fused in (True, False):
        for fb in (True, False):
            r.fused, r.fill_back = fused, fb
            vv = v.clone().requires_grad_(True)
            tt = tex.clone().requires_grad_(True)
            rgb, alpha = r.render_soft(vv, f, tt, sigma=1e-4, gamma=1e-4)
            (rgb.sum() + alpha.sum()).backward()
            outs[(fused, fb)] = (rgb.detach(), alpha.detach(), vv.grad, tt.grad)
    base = outs[(True, True)]
    assert base[0].shape == (2, 3, 128, 128) and base[1].max() > 0.99
    assert torch.isfinite(base[2]).all() and base[2].abs().sum() > 0 and base[3].abs().sum() > 0
    for key, o in outs.items():
        if key[0]:
            assert torch.equal(o[0], base[0]) and torch.equal(o[1], base[1])  # fill_back makes no difference
        else:
            assert (o[0] - base[0]).abs().max() < 1e-5 and torch.equal(o[1], base[1])
        assert rel_err(o[2].cpu().numpy(), base[2].cpu().numpy()) < 1e-4
    r.shading = "smooth"
    with pytest.raises(ValueError):
        r.render_soft(v, f, tex)
