"""GPU: soft attribute images (rasterize_soft_attributes, nr_b200_soft_attributes[_backward], Renderer.render_soft_attributes
and render_soft_depth) against the float64 oracle of tests/oracles_soft_attr.py; bit identities with the soft
silhouettes, the soft RGB's state, the geometry and attribute forms and one-channel renders; the cube soft RGB with
constant cubes; the hard depth map; every gradient against float64 autograd and central differences; the direct C ABI;
the binning's 64-bit keys and the benchmark geometry; three fits; and the Renderer.

Forward gate.  out_c = sum_j w_j A_jc / Z + w_b bg_c / Z is the soft RGB's blend with A_jc in place of C_jc, so the
argument of DESIGN.md 4p carries over channel by channel: a relative error e of a weight moves out_c by at most
e |A_jc - out_c|, and an error of l'_k moves A_jc by that error times |a_kc|.  4p bounds both for colours in [0, 1]
(|C_j - rgb| <= 2 with light <= 1.5) by 4 tol(sigma) + 5e-4.  For a channel whose attributes and background lie in
[-R_c, R_c], |A_jc - out_c| <= 2 R_c and |a_kc| <= R_c, so every term of that bound scales by R_c / 1 at most: the gate
of channel c is (4 tol(sigma) + 5e-4) max(R_c, 1).  The cut-off is bracketed +-1e-5 as for the silhouettes."""
import ctypes
import math

import numpy as np
import pytest
import torch

import oracles_soft as osoft
import oracles_soft_attr as oattr
import soft_binning as sb
from helpers import elem_err, rel_err

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
SIGMAS = (1e-5, 1e-4, 1e-3)
NEAR, FAR = 0.1, 100.0


def tol(sigma):
    return 1e-6 / math.sqrt(sigma) + 1e-6


def tol_attr(sigma, R):
    """[C] gates of channels with attribute / background magnitudes R [C]"""
    return (4 * tol(sigma) + 5e-4) * torch.clamp(R, min=1.0)


def _nr():
    import neural_renderer_b200 as nr
    return nr


def _soup(B, F, seed, **kw):
    from neural_renderer_b200 import synthetic
    return torch.from_numpy(synthetic.triangle_soup(B, F, seed=seed, **kw)).to(DEV)


def _special_faces(B, sigma, seed, F=24):
    """the soft RGB tests' special faces on a soup: wider than the wide-list cap, a sliver, off the image within reach,
    straddling near / far, collinear and a point"""
    soup = _soup(B, F, seed, size=(0.05, 0.3), duplicates=False)
    o = 1.0 + 0.5 * math.sqrt(osoft.cut(sigma))
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


def _rand(shape, seed, lo=-1.0, hi=1.0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return lo + (hi - lo) * torch.rand(shape, device=DEV, generator=g)


def _as_vertices(faces):
    """(vertices [B,3F,3], shared indices [F,3]) drawing exactly `faces`"""
    B, F = faces.shape[:2]
    return faces.reshape(B, 3 * F, 3).contiguous(), torch.arange(3 * F, device=DEV, dtype=torch.int32).reshape(F, 3)


def _oracle(faces, ca, S, sigma, gamma, bg, cut_scale=1.0, pix=None):
    return oattr.soft_attributes(faces.double(), ca.double(), S, sigma, gamma, NEAR, FAR, bg, cut_scale, pix)


def _check_forward(out, alpha, faces, ca, S, sigma, gamma, bg):
    lo, lo_a = _oracle(faces, ca, S, sigma, gamma, bg, 1 - 1e-5)
    hi, hi_a = _oracle(faces, ca, S, sigma, gamma, bg, 1 + 1e-5)

    def excess(x, lo, hi):
        x = x.double()
        return torch.maximum(torch.minimum(lo, hi) - x, x - torch.maximum(lo, hi)).clamp_min(0)

    assert excess(alpha, lo_a, hi_a).max().item() <= tol(sigma)
    R = ca.abs().amax((0, 1, 2)).double()
    if bg is not None:
        R = torch.maximum(R, torch.tensor(bg, dtype=torch.float64, device=DEV).abs())
    e = excess(out, lo, hi).amax((0, 2, 3))
    gate = tol_attr(sigma, R)
    assert torch.all(e <= gate), (e.tolist(), gate.tolist())


@pytest.mark.parametrize("S", [64, 127, 256, 257])
@pytest.mark.parametrize("sigma", SIGMAS)
def test_forward_vs_oracle(S, sigma):
    nr = _nr()
    i = S + int(-math.log10(sigma))
    B = 2
    gamma = (1e-4, 1e-2)[i % 2]
    C = (1, 3, 16, 21)[i % 4]                     # 21: two channel blocks of 16
    per_vertex, shared = bool((i // 2) % 2), bool((i // 3) % 2)
    faces = _special_faces(B, sigma, seed=i)
    F = faces.shape[1]
    bg = tuple(float(v) for v in _rand((C,), i + 1, -2.0, 2.0).tolist())
    Ba = 1 if shared else B
    if per_vertex:
        verts, idx = _as_vertices(faces)
        va = _rand((Ba, 3 * F, C), i + 2, -3.0, 3.0)
        out, alpha = nr.rasterize_soft_attributes(idx, S, sigma, gamma, vertices=verts, vertex_attributes=va, background=bg,
                                                  return_alpha=True)
        ca = oattr.corner_attributes(va, idx)
    else:
        ca = _rand((Ba, F, 3, C), i + 2, -3.0, 3.0)
        out, alpha = nr.rasterize_soft_attributes(faces, S, sigma, gamma, face_attributes=ca, background=bg,
                                                  return_alpha=True)
    assert out.shape == (B, C, S, S) and alpha.shape == (B, S, S)
    _check_forward(out, alpha, faces, ca, S, sigma, gamma, bg)
    assert torch.equal(alpha, nr.rasterize_soft_silhouettes(faces, S, sigma))


def _soft_rgb_state(faces, S, sigma, gamma):
    """state [B,2,S,S] of nr_b200_soft_rgb called directly (unlit random cubes: the state does not depend on them)"""
    from neural_renderer_b200 import _lib
    lib = _lib.load()
    B, F = faces.shape[:2]
    tex = _rand((B, F, 2, 2, 2, 3), 5, 0.0, 1.0)
    a = _lib.SoftRgbArgs()
    a.struct_size = ctypes.sizeof(_lib.SoftRgbArgs)
    a.faces, a.num_faces, a.batch_size, a.image_size, a.texture_size = faces.data_ptr(), F, B, S, 2
    a.sigma, a.gamma, a.near_, a.far_, a.eps = sigma, gamma, NEAR, FAR, 1e-4
    a.textures = tex.data_ptr()
    rgb, alpha, state = (torch.empty(B, 3, S, S, device=DEV), torch.empty(B, S, S, device=DEV),
                         torch.empty(B, 2, S, S, device=DEV))
    a.rgb, a.alpha, a.state = rgb.data_ptr(), alpha.data_ptr(), state.data_ptr()
    n = lib.nr_b200_soft_rgb_workspace_bytes(B, F, S, 0)
    ws = torch.empty(n, dtype=torch.uint8, device=DEV)
    a.workspace, a.workspace_bytes = ws.data_ptr(), n
    assert lib.nr_b200_soft_rgb(ctypes.byref(a), ctypes.c_void_p(torch.cuda.current_stream(DEV).cuda_stream)) == 0
    torch.cuda.synchronize()
    return state, alpha


def _abi(faces, attrs, S, sigma, gamma, flags=0, bg=None, out=None, alpha=None, state=None, verts=None, idx=None,
         g_out=None, g_alpha=None, grad_geom=None, grad_attr=None, backward=False):
    """a direct nr_b200_soft_attributes[_backward] call; returns the code"""
    from neural_renderer_b200 import _lib
    lib = _lib.load()
    geom = faces if verts is None else verts
    B = geom.shape[0]
    F = faces.shape[1] if verts is None else idx.shape[-2]
    a = _lib.SoftRgbArgs()
    a.struct_size = ctypes.sizeof(_lib.SoftRgbArgs)
    if verts is not None:
        flags |= _lib.NR_FACES_INDEXED | (_lib.NR_INDICES_SHARED if idx.dim() == 2 else 0)
        a.vertices, a.face_indices, a.num_vertices = verts.data_ptr(), idx.data_ptr(), verts.shape[1]
    else:
        a.faces = faces.data_ptr()
    a.flags, a.num_faces, a.batch_size, a.image_size = flags, F, B, S
    a.sigma, a.gamma, a.near_, a.far_ = sigma, gamma, NEAR, FAR
    ptr = lambda t: None if t is None else t.data_ptr()
    a.alpha, a.state, a.grad_alpha = ptr(alpha), ptr(state), ptr(g_alpha)
    if verts is not None:
        a.grad_vertices = ptr(grad_geom)
    else:
        a.grad_faces = ptr(grad_geom)
    n = lib.nr_b200_soft_rgb_workspace_bytes(B, F, S, flags & (_lib.NR_FACES_INDEXED | _lib.NR_INDICES_SHARED))
    ws = torch.empty(n, dtype=torch.uint8, device=DEV)
    a.workspace, a.workspace_bytes = ws.data_ptr(), n
    t = _lib.SoftAttrArgs(struct_size=ctypes.sizeof(_lib.SoftAttrArgs), channels=attrs.shape[-1])
    t.attributes, t.background, t.out = attrs.data_ptr(), ptr(bg), ptr(out)
    t.grad_out, t.grad_attributes = ptr(g_out), ptr(grad_attr)
    fn = lib.nr_b200_soft_attributes_backward if backward else lib.nr_b200_soft_attributes
    rc = fn(ctypes.byref(a), ctypes.byref(t), ctypes.c_void_p(torch.cuda.current_stream(DEV).cuda_stream))
    torch.cuda.synchronize()
    return rc


def test_bit_identities():
    nr = _nr()
    S, sigma, gamma, B = 96, 1e-4, 1e-4, 2
    faces = _special_faces(B, sigma, seed=5)
    F = faces.shape[1]
    C = 20
    ca = _rand((B, F, 3, C), 6, -2.0, 2.0)
    bg = [float(v) for v in _rand((C,), 7).tolist()]
    out, alpha = nr.rasterize_soft_attributes(faces, S, sigma, gamma, face_attributes=ca, background=bg, return_alpha=True)
    # repeatable; alpha is the silhouettes'; each channel is its one-channel render; channel subsets agree
    out2, alpha2 = nr.rasterize_soft_attributes(faces, S, sigma, gamma, face_attributes=ca, background=bg, return_alpha=True)
    assert torch.equal(out, out2) and torch.equal(alpha, alpha2)
    assert torch.equal(alpha, nr.rasterize_soft_silhouettes(faces, S, sigma))
    for c in (0, 3, 15, 16, 19):
        one = nr.rasterize_soft_attributes(faces, S, sigma, gamma, face_attributes=ca[..., c:c + 1].contiguous(),
                                           background=[bg[c]])
        assert torch.equal(one[:, 0], out[:, c]), c
    three = nr.rasterize_soft_attributes(faces, S, sigma, gamma, face_attributes=ca[..., 14:17].contiguous(),
                                         background=bg[14:17])
    assert torch.equal(three, out[:, 14:17])
    # state equals the soft RGB's through the ABI
    state_rgb, alpha_rgb = _soft_rgb_state(faces, S, sigma, gamma)
    st, al = torch.empty(B, 2, S, S, device=DEV), torch.empty(B, S, S, device=DEV)
    o = torch.empty(B, C, S, S, device=DEV)
    assert _abi(faces, ca, S, sigma, gamma, bg=torch.tensor(bg, device=DEV), out=o, alpha=al, state=st) == 0
    assert torch.equal(st, state_rgb) and torch.equal(al, alpha_rgb) and torch.equal(o, out)
    # indexed == materialised, per vertex == its gathered corners, shared == repeated == expanded
    verts, idx = _as_vertices(faces)
    va = _rand((1, 3 * F, C), 8)
    pv = nr.rasterize_soft_attributes(idx, S, sigma, gamma, vertices=verts, vertex_attributes=va, background=bg)
    pc = nr.rasterize_soft_attributes(faces, S, sigma, gamma, face_attributes=oattr.corner_attributes(va, idx).contiguous(),
                                      background=bg)
    assert torch.equal(pv, pc)
    for vv in (va[0], va.expand(B, -1, -1), va.repeat(B, 1, 1)):
        assert torch.equal(nr.rasterize_soft_attributes(idx, S, sigma, gamma, vertices=verts, vertex_attributes=vv,
                                                        background=bg), pv)
    for ix in (idx[None], idx[None].expand(B, -1, -1), idx[None].repeat(B, 1, 1)):
        assert torch.equal(nr.rasterize_soft_attributes(ix, S, sigma, gamma, vertices=verts, vertex_attributes=va,
                                                        background=bg), pv)
    assert torch.equal(nr.rasterize_soft_attributes(faces, S, sigma, gamma, face_attributes=ca, background=bg),
                       nr.rasterize_soft_attributes(idx, S, sigma, gamma, vertices=verts, face_attributes=ca, background=bg))
    c1 = ca[:1]
    assert torch.equal(nr.rasterize_soft_attributes(faces, S, sigma, gamma, face_attributes=c1),
                       nr.rasterize_soft_attributes(faces, S, sigma, gamma, face_attributes=c1.expand(B, -1, -1, -1)))
    assert torch.equal(nr.rasterize_soft_attributes(faces, S, sigma, gamma, face_attributes=c1[0]),
                       nr.rasterize_soft_attributes(faces, S, sigma, gamma, face_attributes=c1.repeat(B, 1, 1, 1)))


def test_constant_face_attributes_match_the_cube_soft_rgb():
    nr = _nr()
    S, sigma, gamma, B = 80, 1e-4, 1e-3, 2
    faces = _special_faces(B, sigma, seed=9)
    F = faces.shape[1]
    col = _rand((B, F, 3), 10, 0.0, 1.0)
    bg = (0.2, 0.5, 0.8)
    f1 = faces.clone().requires_grad_(True)
    out, alpha = nr.rasterize_soft_attributes(f1, S, sigma, gamma, face_attributes=col[:, :, None].expand(B, F, 3, 3),
                                              background=bg, return_alpha=True)
    f2 = faces.clone().requires_grad_(True)
    rgb, alpha2 = nr.rasterize_soft(f2, col[:, :, None, None, None].expand(B, F, 2, 2, 2, 3).contiguous(), S, sigma, gamma,
                                    background_color=bg)
    assert torch.equal(alpha, alpha2)
    assert (out - rgb).abs().max().item() <= 1e-6
    w = torch.randn(B, 3, S, S, device=DEV, generator=torch.Generator(device=DEV).manual_seed(1))
    wa = torch.randn(B, S, S, device=DEV, generator=torch.Generator(device=DEV).manual_seed(2))
    ((out * w).sum() + (alpha * wa).sum()).backward()
    ((rgb * w).sum() + (alpha2 * wa).sum()).backward()
    assert (f1.grad - f2.grad).abs().max().item() <= 1e-4 * max(1.0, f2.grad.abs().max().item())


def test_soft_depth_matches_the_hard_depth_inside_faces():
    """render_soft_depth at sigma = gamma = 1e-7 against render_depth where one face decides the pixel: the nearest face
    within reach covers it more than 1 px from that face's edges, and every other face within reach lies more than
    1e-3 behind it (no depth tie)"""
    import os
    nr = _nr()
    r = nr.Renderer()
    r.image_size = 256
    d = np.load(os.path.join(os.path.dirname(__file__), "golden", "teapot.npz"))
    v = torch.from_numpy(d["vertices"].astype(np.float32)).to(DEV)[None]
    f = torch.from_numpy(d["faces"].astype(np.int32)).to(DEV)[None]
    r.eye = nr.get_points_from_angles(2.732, 30, -15)
    sigma = gamma = 1e-7
    soft = r.render_soft_depth(v, f, sigma=sigma, gamma=gamma)
    r.anti_aliasing = False
    hard = r.render_depth(v, f)
    S = r.image_size
    fv = osoft.gather_faces(r._transform(v), f[0]).double()
    p = osoft.pixel_centres(S, device=DEV)
    # per pixel, over the faces within reach: the two smallest depths, and whether the nearest covers the pixel and how
    # far it lies from its edges (face chunks keep the float64 terms to a few hundred MB)
    P = p.shape[0]
    first, second = torch.full((P,), math.inf, dtype=torch.float64, device=DEV), torch.full((P,), math.inf,
                                                                                               dtype=torch.float64, device=DEV)
    win_inside = torch.zeros(P, dtype=torch.bool, device=DEV)
    win_d2 = torch.zeros(P, dtype=torch.float64, device=DEV)
    reached = torch.zeros(P, dtype=torch.bool, device=DEV)
    for f0 in range(0, fv.shape[1], 128):
        fc = fv[:, f0:f0 + 128]
        d2, inside = osoft.face_terms(fc, p)                               # [1,Fc,P]
        on = osoft.participates(fc, r.near, r.far)[..., None] & (inside | (d2 <= 4 * osoft.cut(sigma)))
        zp = oattr.orgb.bary_terms(fc, p, sigma, r.near, r.far, 1.0)[4]
        vals = torch.cat((first[None], second[None], torch.where(on, zp, torch.full_like(zp, math.inf))[0]))
        ins = torch.cat((win_inside[None], torch.zeros_like(win_inside)[None], inside[0]))
        dd = torch.cat((win_d2[None], torch.zeros_like(win_d2)[None], d2[0]))
        zs = vals.sort(0)
        first, second = zs.values[0], zs.values[1]
        win_inside = torch.gather(ins, 0, zs.indices[:1])[0]
        win_d2 = torch.gather(dd, 0, zs.indices[:1])[0]
        reached |= on[0].any(0)
    m = torch.isfinite(first) & win_inside & (win_d2 > (2.0 / S) ** 2) & (second - first > 1e-3)
    m = m.reshape(S, S)
    assert m.sum().item() > 200, m.sum().item()
    err = (soft[0] - hard[0]).abs()[m]
    assert err.max().item() <= 1e-5 * hard[0][m].max().item(), err.max().item()
    # no face within reach: the background, far exactly
    empty = (~reached).reshape(S, S)
    assert empty.sum().item() > 1000 and torch.all(soft[0][empty] == r.far)


# ------------------------------------------------------------------------------------------------ backward
def _grads(faces, ca, S, sigma, gamma, bg, g_out, g_a, verts=None, idx=None, va=None):
    nr = _nr()
    if verts is not None:
        gv = verts.clone().requires_grad_(True)
        a = va.clone().requires_grad_(True)
        out, alpha = nr.rasterize_soft_attributes(idx, S, sigma, gamma, vertices=gv, vertex_attributes=a, background=bg,
                                                  return_alpha=True)
        leaves = (gv, a)
    else:
        f = faces.clone().requires_grad_(True)
        a = ca.clone().requires_grad_(True)
        out, alpha = nr.rasterize_soft_attributes(f, S, sigma, gamma, face_attributes=a, background=bg, return_alpha=True)
        leaves = (f, a)
    loss = 0
    if g_out is not None:
        loss = loss + (out * g_out).sum()
    if g_a is not None:
        loss = loss + (alpha * g_a).sum()
    loss.backward()
    return tuple(x.grad for x in leaves)


def _oracle_grads(faces, ca, S, sigma, gamma, bg, g_out, g_a, verts=None, idx=None, va=None):
    if verts is not None:
        gv = verts.double().requires_grad_(True)
        a = va.double().requires_grad_(True)
        fc, cc = osoft.gather_faces(gv, idx), oattr.corner_attributes(a, idx)
        # a face with an out-of-range corner reads the zero vertex (z = 0 < near) and takes no part; an off-image
        # stand-in keeps the float64 divisions by its z = 0 out of autograd
        pad = torch.tensor([[10.0, 10.0, 1.0], [10.5, 10.0, 1.0], [10.0, 10.5, 1.0]], dtype=torch.float64, device=DEV)
        fc = torch.where(osoft.participates(fc.detach(), NEAR, FAR)[..., None, None], fc, pad)
        leaves = (gv, a)
    else:
        fc = faces.double().requires_grad_(True)
        cc = ca.double().requires_grad_(True)
        leaves = (fc, cc)
    out, alpha = oattr.soft_attributes(fc, cc, S, sigma, gamma, NEAR, FAR, bg)
    loss = 0
    if g_out is not None:
        loss = loss + (out * g_out.double()).sum()
    if g_a is not None:
        loss = loss + (alpha * g_a.double()).sum()
    gs = torch.autograd.grad(loss, leaves, allow_unused=True)
    return tuple(torch.zeros_like(x) if gx is None else gx for x, gx in zip(leaves, gs))


@pytest.mark.parametrize("which", ["out", "alpha", "both"])
@pytest.mark.parametrize("form", ["corner", "corner_shared", "vertex_shared"])
def test_backward_vs_float64_autograd(which, form):
    S, B, sigma, gamma, C = 64, 2, 1e-4, 1e-2, 3
    faces = _special_faces(B, sigma, seed=41, F=12)
    F = faces.shape[1]
    gen = torch.Generator(device=DEV).manual_seed(43)
    g_out = torch.randn(B, C, S, S, device=DEV, generator=gen) if which != "alpha" else None
    g_a = torch.randn(B, S, S, device=DEV, generator=gen) if which != "out" else None
    bg = (0.3, -0.2, 0.5)
    kw = {}
    if form == "vertex_shared":
        verts, idx = _as_vertices(faces)
        idx = idx.clone()
        idx[2, 1] = 3 * F          # out of range: reads zeros, gets nothing
        idx[4, 0] = -1
        kw = dict(verts=verts, idx=idx, va=_rand((1, 3 * F, C), 44))
        ca = None
    else:
        ca = _rand((1 if form == "corner_shared" else B, F, 3, C), 44)
    got = _grads(faces, ca, S, sigma, gamma, bg, g_out, g_a, **kw)
    ref = _oracle_grads(faces, ca, S, sigma, gamma, bg, g_out, g_a, **kw)
    for name, a, r in zip(("geometry", "attributes"), got, ref):
        a, r = a.double().cpu().numpy(), r.cpu().numpy()
        assert np.isfinite(a).all(), name
        if which == "alpha" and name == "attributes":
            assert np.all(a == 0)
            continue
        assert rel_err(a, r) <= 5e-3, (name, rel_err(a, r))
        assert elem_err(a, r, floor=2e-2) <= 5e-2, (name, elem_err(a, r, floor=2e-2))
    if which != "alpha":
        assert got[0][..., 2].abs().max() > 0  # the vertex depths receive a gradient
    if form == "vertex_shared" and which != "alpha":
        # vertices only the out-of-range slots referenced get no attribute gradient
        assert torch.all(got[1][0, 3 * 2 + 1] == 0) and torch.all(got[1][0, 3 * 4] == 0)


def test_backward_vs_central_differences_of_the_forward():
    nr = _nr()
    S, sigma, gamma, C = 64, 1e-3, 1e-2, 3
    faces = _soup(1, 6, seed=21, size=(0.15, 0.4), offscreen=False, duplicates=False)
    ca = _rand((1, 6, 3, C), 22)
    w = torch.randn(1, C, S, S, device=DEV, generator=torch.Generator(device=DEV).manual_seed(7))
    # as the soft RGB's test: the loss is blind to pixels whose d^2 lies within 2e-4 of the cut-off
    d2, _ = osoft.face_terms(faces.double(), osoft.pixel_centres(S, device=DEV))
    w = w * ((d2 - osoft.cut(sigma)).abs() > 2e-4).all(1).reshape(1, 1, S, S)
    bg = (0.5, 0.5, 0.5)
    gf, ga = _grads(faces, ca, S, sigma, gamma, bg, w, None)

    def loss(ff, aa):
        out = nr.rasterize_soft_attributes(ff, S, sigma, gamma, face_attributes=aa, background=bg)
        return float((out.double() * w.double()).sum())

    h = 2e-4
    scale = gf.abs().max().item()
    for (fi, k, c) in [(0, 0, 0), (1, 1, 1), (2, 2, 2), (3, 0, 1), (5, 2, 0), (4, 1, 2)]:
        fp, fm = faces.clone(), faces.clone()
        fp[0, fi, k, c] += h
        fm[0, fi, k, c] -= h
        fd = (loss(fp, ca) - loss(fm, ca)) / (fp[0, fi, k, c] - fm[0, fi, k, c]).item()
        assert abs(fd - gf[0, fi, k, c].item()) <= 3e-2 * scale, (fi, k, c, fd, gf[0, fi, k, c].item())
    for (fi, k, c) in [(0, 0, 0), (2, 1, 1), (5, 2, 2)]:   # the image is linear in the attributes
        ap, am = ca.clone(), ca.clone()
        ap[0, fi, k, c] += 1e-2
        am[0, fi, k, c] -= 1e-2
        fd = (loss(faces, ap) - loss(faces, am)) / 2e-2
        assert abs(fd - ga[0, fi, k, c].item()) <= 1e-2 * max(ga.abs().max().item(), 1e-6), (fi, k, c, fd)


# ------------------------------------------------------------------------------------------------ direct ABI
def _guarded(shape, fill=float("nan"), guard=16):
    n = int(np.prod(shape))
    buf = torch.full((n + 2 * guard,), fill, device=DEV)
    buf[:guard] = 7.0
    buf[-guard:] = 7.0
    return buf, buf[guard:guard + n].view(*shape)


@pytest.mark.parametrize("indexed", [False, True])
def test_abi_poison_guards_nulls_and_accumulate(indexed):
    nr = _nr()
    S, sigma, gamma, B, C = 40, 1e-4, 1e-3, 2, 5
    faces = _special_faces(B, sigma, seed=61, F=10)
    F = faces.shape[1]
    verts, idx = _as_vertices(faces) if indexed else (None, None)
    ca = _rand((B, F, 3, C), 62)
    bg = _rand((C,), 63)
    ob, out = _guarded((B, C, S, S))
    ab, alpha = _guarded((B, S, S))
    sb_, state = _guarded((B, 2, S, S))
    assert _abi(faces, ca, S, sigma, gamma, bg=bg, out=out, alpha=alpha, state=state, verts=verts, idx=idx) == 0
    for buf in (ob, ab, sb_):
        assert torch.isfinite(buf).all() and torch.all(buf[:16] == 7.0) and torch.all(buf[-16:] == 7.0)
    ref = nr.rasterize_soft_attributes(faces, S, sigma, gamma, face_attributes=ca, background=bg.tolist())
    assert torch.equal(out, ref)
    # background NULL = zeros
    o0 = torch.empty_like(out)
    assert _abi(faces, ca, S, sigma, gamma, out=o0, alpha=alpha, state=state, verts=verts, idx=idx) == 0
    assert torch.equal(o0, nr.rasterize_soft_attributes(faces, S, sigma, gamma, face_attributes=ca, background=[0.0] * C))
    # backward: poisoned gradients are overwritten; NULL grad_out / grad_alpha / grad_attributes; accumulation
    gen = torch.Generator(device=DEV).manual_seed(64)
    g_out, g_a = torch.randn(B, C, S, S, device=DEV, generator=gen), torch.randn(B, S, S, device=DEV, generator=gen)
    geom = verts if indexed else faces
    gb, gg = _guarded(tuple(geom.shape))
    tb, gt = _guarded(tuple(ca.shape))
    kw = dict(bg=bg, out=out, alpha=alpha, state=state, verts=verts, idx=idx, backward=True)
    assert _abi(faces, ca, S, sigma, gamma, g_out=g_out, g_alpha=g_a, grad_geom=gg, grad_attr=gt, **kw) == 0
    for buf in (gb, tb):
        assert torch.isfinite(buf).all() and torch.all(buf[:16] == 7.0) and torch.all(buf[-16:] == 7.0)
    full_g, full_t = gg.clone(), gt.clone()
    assert (full_g != 0).any() and (full_t != 0).any()
    for g1, g2, want_t_zero in ((None, g_a, True), (g_out, None, False), (None, None, True)):
        g_geom, g_attr = torch.full_like(gg, float("nan")), torch.full_like(gt, float("nan"))
        assert _abi(faces, ca, S, sigma, gamma, g_out=g1, g_alpha=g2, grad_geom=g_geom, grad_attr=g_attr, **kw) == 0
        assert torch.isfinite(g_geom).all() and torch.isfinite(g_attr).all()
        assert torch.all(g_attr == 0) == want_t_zero
    g_geom = torch.full_like(gg, float("nan"))
    assert _abi(faces, ca, S, sigma, gamma, g_out=g_out, g_alpha=g_a, grad_geom=g_geom, grad_attr=None, **kw) == 0
    assert torch.allclose(g_geom, full_g, rtol=1e-5, atol=1e-6)
    # NR_GRAD_ACCUMULATE: prefill + fresh, the prefill bit for bit where the fresh gradient is 0
    from neural_renderer_b200 import _lib
    pre_g, pre_t = _rand(tuple(geom.shape), 65), _rand(tuple(ca.shape), 66)
    acc_g, acc_t = pre_g.clone(), pre_t.clone()
    assert _abi(faces, ca, S, sigma, gamma, flags=_lib.NR_GRAD_ACCUMULATE, g_out=g_out, g_alpha=g_a, grad_geom=acc_g,
                grad_attr=acc_t, **kw) == 0
    for acc, pre, fresh in ((acc_g, pre_g, full_g), (acc_t, pre_t, full_t)):
        assert torch.allclose(acc, pre + fresh, rtol=1e-5, atol=1e-5)
        assert torch.equal(acc[fresh == 0], pre[fresh == 0])
    # a call with an rgb-only pointer is refused before any launch
    lib = _lib.load()
    a = _lib.SoftRgbArgs(struct_size=ctypes.sizeof(_lib.SoftRgbArgs))
    t = _lib.SoftAttrArgs(struct_size=ctypes.sizeof(_lib.SoftAttrArgs), channels=C, attributes=ca.data_ptr(),
                          out=out.data_ptr())
    a.faces, a.num_faces, a.batch_size, a.image_size = faces.data_ptr(), F, B, S
    a.sigma, a.gamma, a.near_, a.far_ = sigma, gamma, NEAR, FAR
    a.alpha, a.state, a.rgb = alpha.data_ptr(), state.data_ptr(), out.data_ptr()
    assert lib.nr_b200_soft_attributes(ctypes.byref(a), ctypes.byref(t), None) == -1
    assert lib.nr_b200_last_launch_count() == 0


# ------------------------------------------------------------------------------------------------ scale
def test_64_bit_keys_bit_identical_across_face_counts():
    import test_gpu_soft_scale as tss
    nr = _nr()
    S, sigma, gamma = tss.S_KEY, tss.SIGMA_KEY, tss.GAMMA_KEY
    real = tss._real_faces(2, seed=1)
    B, Fr = real.shape[:2]
    assert sb.key_width(B, 65535, S)[2] is False and sb.key_width(B, 65536, S)[2] is True
    va = _rand((1, 3 * Fr, 3), 71, 0.0, 1.0)
    pix = tss._pixels_near(real, S, 4000, seed=2)
    ref_out = ref_a = ref_g = None
    g_out = _rand((B, 3, S, S), 72)
    for F in (Fr, 65535, 65536):
        faces, pos = tss._padded(real, F, seed=3)
        verts, idx = tss._indexed(faces, pos)
        vv = torch.cat((va, torch.zeros(1, 12, 3, device=DEV)), 1)
        v = verts.clone().requires_grad_(True)
        out, alpha = nr.rasterize_soft_attributes(idx, S, sigma, gamma, vertices=v, vertex_attributes=vv, return_alpha=True,
                                                  background=(0.1, 0.2, 0.3))
        (out * g_out).sum().backward()
        if ref_out is None:
            ref_out, ref_a, ref_g = out, alpha, v.grad[:, :3 * Fr]
            ca = oattr.corner_attributes(va, torch.arange(3 * Fr, device=DEV).reshape(Fr, 3))
            want, want_a = oattr.soft_attributes(real.double(), ca.double(), S, sigma, gamma, NEAR, FAR, (0.1, 0.2, 0.3),
                                                 pix=pix)
            got = torch.gather(out.reshape(B, 3, -1), 2, pix[:, None].expand(-1, 3, -1))
            # about 200 faces per item: the 4p gate with the safety factor of the benchmark-geometry check below
            assert (got.double() - want).abs().max().item() <= 4 * (4 * tol(sigma) + 5e-4)
        else:
            assert torch.equal(out, ref_out) and torch.equal(alpha, ref_a)
            # fp32 atomics land in another order: the gradient agrees per tensor, as test_gpu_soft_scale's
            assert rel_err(v.grad[:, :3 * Fr].cpu().numpy(), ref_g.cpu().numpy()) <= 1e-5
            assert torch.all(v.grad[:, 3 * Fr:] == 0)


def test_benchmark_geometry_tiles_and_gradients():
    """sphere_faces(64, 5000) at 256 x 256: three tiles per item against the sparse oracle, and every face's gradient
    from those tiles"""
    from neural_renderer_b200 import synthetic
    nr = _nr()
    B, F, S, gamma = 64, 5000, 256, 1e-4
    faces = torch.from_numpy(synthetic.sphere_faces(B, F)).to(DEV)
    C = 3
    ca = _rand((B, F, 3, C), 81, 0.0, 1.0)
    for sigma in SIGMAS:
        tiles = torch.tensor([[5, 7], [8, 8], [10, 6]], device=DEV)
        pix = torch.cat([(ty * 16 + torch.arange(16, device=DEV))[:, None] * S + (tx * 16 + torch.arange(16, device=DEV))[None]
                         for tx, ty in tiles.tolist()]).reshape(-1)
        mask = torch.zeros(S * S, device=DEV)
        mask[pix] = 1.0
        g = _rand((B, C, S, S), 82) * mask.reshape(1, 1, S, S)
        f = faces.clone().requires_grad_(True)
        a = ca.clone().requires_grad_(True)
        out = nr.rasterize_soft_attributes(f, S, sigma, gamma, face_attributes=a, background=(0.3, 0.3, 0.3))
        (out * g).sum().backward()
        items = [0, 17, 63]
        fo = faces[items].double().requires_grad_(True)
        co = ca[items].double().requires_grad_(True)
        want, _ = oattr.soft_attributes(fo, co, S, sigma, gamma, NEAR, FAR, (0.3, 0.3, 0.3), pix=pix)
        got = out[items].reshape(len(items), C, -1)[:, :, pix]
        assert (got.double() - want).abs().max().item() <= 4 * (4 * tol(sigma) + 5e-4)
        (want * g[items].reshape(len(items), C, -1)[:, :, pix].double()).sum().backward()
        for name, x, r in (("faces", f.grad[items], fo.grad), ("attributes", a.grad[items], co.grad)):
            x, r = x.double().cpu().numpy(), r.cpu().numpy()
            assert rel_err(x, r) <= 5e-3, (name, sigma, rel_err(x, r))


# ------------------------------------------------------------------------------------------------ fits
def _square(cx, cy, half, z):
    v = [[cx - half, cy - half, z], [cx + half, cy - half, z], [cx + half, cy + half, z], [cx - half, cy + half, z]]
    return torch.tensor(v, dtype=torch.float32, device=DEV), torch.tensor([[0, 1, 2], [0, 2, 3]], dtype=torch.int32,
                                                                            device=DEV)


def test_per_vertex_colours_are_recovered():
    nr = _nr()
    S, sigma, gamma = 64, 1e-4, 1e-3
    faces = _soup(1, 12, seed=91, size=(0.2, 0.5), offscreen=False, duplicates=False)
    verts, idx = _as_vertices(faces)
    target = _rand((1, verts.shape[1], 3), 92, 0.0, 1.0)
    img = nr.rasterize_soft_attributes(idx, S, sigma, gamma, vertices=verts, vertex_attributes=target)
    va = torch.full_like(target, 0.5).requires_grad_(True)
    opt = torch.optim.Adam([va], lr=0.05)
    sched = torch.optim.lr_scheduler.ExponentialLR(opt, 0.98)
    for _ in range(300):
        opt.zero_grad()
        out = nr.rasterize_soft_attributes(idx, S, sigma, gamma, vertices=verts, vertex_attributes=va)
        ((out - img) ** 2).sum().backward()
        opt.step()
        sched.step()
    final = ((nr.rasterize_soft_attributes(idx, S, sigma, gamma, vertices=verts, vertex_attributes=va) - img) ** 2).mean()
    assert final.item() < 1e-5, final.item()
    assert (va.detach() - target).abs().median().item() < 0.02   # hidden corners excepted, the colours themselves


def test_hidden_square_is_brought_forward_by_a_soft_depth_loss():
    """d out / d z_h = (w_h / Z) (1 - (z_h - out) / ((far - near) gamma)): with (far - near) gamma = 3 above the
    1-unit gap, moving the hidden square nearer lowers the depth where it lies, so the loss pulls it in front"""
    nr = _nr()
    S, sigma, gamma = 64, 1e-4, 3e-2
    vf, ff = _square(0.0, 0.0, 0.5, 2.0)    # the front square
    vb, fb = _square(0.1, 0.1, 0.3, 3.0)    # hidden behind it
    verts = torch.cat((vf, vb))[None]
    idx = torch.cat((ff, fb + 4))
    # target: the small square in front at depth 1.5
    vt = verts.clone()
    vt[0, 4:, 2] = 1.5
    fv = lambda v: osoft.gather_faces(v, idx).float()
    target = nr.rasterize_soft_attributes(fv(vt), S, sigma, gamma, face_attributes=fv(vt)[..., 2:3], background=[FAR])
    # the hard depth gives the hidden square no gradient
    vh = verts.clone().requires_grad_(True)
    hard = nr.rasterize_depth(idx, S, False, vertices=vh)
    ((hard - target[:, 0]) ** 2).sum().backward()
    assert torch.all(vh.grad[0, 4:] == 0)
    z = torch.full((4,), 3.0, device=DEV, requires_grad=True)
    opt = torch.optim.Adam([z], lr=0.05)
    for _ in range(150):
        opt.zero_grad()
        v = torch.cat((verts[0, :4], torch.cat((verts[0, 4:, :2], z[:, None]), 1)))[None]
        f = fv(v)
        out = nr.rasterize_soft_attributes(f, S, sigma, gamma, face_attributes=f[..., 2:3], background=[FAR])
        ((out - target) ** 2).mean().backward()
        opt.step()
    assert z.max().item() < 2.0, z.tolist()      # in front of the big square


def _tri_at(cx, cy, s=2.0 / 128):
    return torch.tensor([[[[cx - s, cy - s, 2.0], [cx + s, cy - s, 2.0], [cx, cy + s, 2.0]]]], device=DEV)


def test_translation_fit_from_a_three_channel_attribute_loss():
    nr = _nr()
    S, sigma, gamma = 128, 1e-4, 1e-3
    px = 2.0 / S
    col = torch.tensor([[[[1.0, 0.2, 0.4], [0.3, 1.0, 0.2], [0.2, 0.4, 1.0]]]], device=DEV)
    target = nr.rasterize_soft_attributes(_tri_at(0.0, 0.0), S, sigma, gamma, face_attributes=col)
    off = torch.tensor([3 * px, 0.0], device=DEV, requires_grad=True)   # 3 px off: no overlap with the 2-px triangle
    opt = torch.optim.Adam([off], lr=0.2 * px)
    sched = torch.optim.lr_scheduler.ExponentialLR(opt, 0.99)
    for _ in range(400):
        opt.zero_grad()
        f = _tri_at(0.0, 0.0) + torch.cat((off, off.new_zeros(1)))
        out = nr.rasterize_soft_attributes(f, S, sigma, gamma, face_attributes=col)
        ((out - target) ** 2).sum().backward()
        opt.step()
        sched.step()
    assert off.detach().abs().max().item() < 0.1 * px, (off / px).tolist()


# ------------------------------------------------------------------------------------------------ Renderer
def test_renderer_fused_op_by_op_fill_back_camera_gradient_and_soft_depth():
    nr = _nr()
    import os
    d = np.load(os.path.join(os.path.dirname(__file__), "golden", "teapot.npz"))
    v = torch.from_numpy(d["vertices"].astype(np.float32)).to(DEV)[None].repeat(2, 1, 1)
    f = torch.from_numpy(d["faces"].astype(np.int32)).to(DEV)[None].repeat(2, 1, 1)
    r = nr.Renderer()
    r.image_size = 96
    r.eye = nr.get_points_from_angles(2.732, 30, -15)
    va = _rand((1, v.shape[1], 4), 101, 0.0, 1.0)
    fa = oattr.corner_attributes(va, f[0])
    fused = r.render_soft_attributes(v, f, vertex_attributes=va, background=[0.1] * 4)
    r.fill_back = False
    assert torch.equal(fused, r.render_soft_attributes(v, f, vertex_attributes=va, background=[0.1] * 4))
    assert torch.equal(fused, r.render_soft_attributes(v, f, face_attributes=fa, background=[0.1] * 4))
    r.fused = False
    assert torch.equal(fused, r.render_soft_attributes(v, f, vertex_attributes=va, background=[0.1] * 4))
    assert torch.equal(fused, r.render_soft_attributes(v, f, face_attributes=fa, background=[0.1] * 4))
    r.fused, r.fill_back = True, True
    # render_soft_depth is render_soft_attributes with the camera z, on both paths
    depth = r.render_soft_depth(v, f)
    z = r._transform(v)[..., 2:3]
    assert depth.shape == (2, 96, 96)
    assert torch.equal(depth, r.render_soft_attributes(v, f, vertex_attributes=z, background=[r.far])[:, 0])
    r.fused = False
    assert torch.equal(depth, r.render_soft_depth(v, f))
    r.fused = True
    # a gradient reaches the vertices through the camera
    vv = v.clone().requires_grad_(True)
    (r.render_soft_depth(vv, f) * _rand((2, 96, 96), 102)).sum().backward()
    assert torch.isfinite(vv.grad).all() and vv.grad.abs().max() > 0
