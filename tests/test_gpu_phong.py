"""GPU: Phong shading -- normal and position interpolated at every pixel, ambient + diffuse times the unlit sample plus a
specular highlight (include/nr_b200.h, nr_b200_phong_args), the corner-shading glue kernels, and Renderer.shading = 'phong'.

The forward is held to a float64 oracle (oracles_phong.py) on the product's own maps, times the unlit sample: the float64
samplers of oracles.py for texture images, the product's own unlit render for cubes (bit-exact to the reference elsewhere).
The backward is held to float64 autograd of the same oracle and to central differences of the product's forward.  The
scenes, cases and sampler plumbing are those of test_gpu_smooth.py."""
import ctypes
import math

import numpy as np
import pytest
import torch

from helpers import elem_err, np_, rel_err
from oracles_phong import phong_rgb64, phong_terms64
from test_gpu_smooth import BG, FWD_CASES, GRAD_CASES, Scene, _mesh, _R, _rand, _renderer, _teapot_inputs, _upsample

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda")


def _shading_inputs(sc, sigma=16.0, K=(0.6, 0.5, 0.4), seed=21, Bc=None, Bp=None, d=(0.3, 0.5, -1.0), e=(0.2, -0.1, -4.0)):
    """random corner normals facing the viewer (-z), positions from the corners' own NDC x, y and depth; params"""
    Bc = sc.B if Bc is None else Bc
    Bp = sc.B if Bp is None else Bp
    g = torch.Generator().manual_seed(seed)
    n = torch.randn((Bc, sc.F, 3, 3), generator=g)
    n[..., 2] = -(n[..., 2].abs() + 1.0)
    pos = sc.faces[:Bc].cpu() if Bc <= sc.B else None
    cs = torch.cat((n, pos), dim=-1).to(DEV).contiguous()
    rows = []
    for b in range(Bp):
        rows.append([0.3, 0.25, 0.2, 0.6 + 0.1 * b, 0.7, 0.8, d[0], d[1] + 0.1 * b, d[2], *K, sigma, e[0], e[1], e[2]])
    return cs, torch.tensor(rows, dtype=torch.float32, device=DEV)


def _render(sc, cs, prm, tex=None, uvs=None, aa=None, H=None, bg=BG):
    aa = sc.aa if aa is None else aa
    H = sc.H if H is None else H
    geom, verts = sc.faces, None
    if sc.indexed:
        verts = sc.faces.reshape(sc.B, -1, 3)
        geom = torch.arange(verts.shape[1], device=DEV, dtype=torch.int32).reshape(-1, 3)
    return _R()._run(geom, sc.tex if tex is None else tex, H, aa, 0.1, 100, 1e-4, bg, True, True, True,
                     textures_fill_back=sc.fill_back, vertices=verts, face_uvs=sc.uvs if uvs is None else uvs,
                     texture_filter=sc.tf, corner_shading=cs, shading_params=prm)


def _fwd_tol(kind, sigma=1.0):
    # trilinear: the oracle's float64 level of detail (test_gpu_smooth.py); sigma = 64: q^sigma multiplies the fp32 relative
    # error of q by sigma (measured on an H100: at most 1.3e-5 against 2.6e-7 at sigma = 1)
    return 6e-5 if kind == "trilinear" else (2e-5 if sigma > 1.0 else 1e-5)


@pytest.mark.parametrize("case", FWD_CASES)
def test_forward_vs_oracle(case):
    kind, aa, fill_back, indexed = case
    sc = Scene(kind, aa, fill_back, indexed)
    fim, wmap, dmap = sc.maps()
    unlit = sc.unlit64(fim, wmap, dmap)
    for sigma in (1.0, 64.0):
        cs, prm = _shading_inputs(sc, sigma=sigma)
        rgb = _render(sc, cs, prm)[0]
        want = phong_rgb64(sc.faces, fim, wmap, dmap, cs, prm, unlit, BG, aa)
        _, h, _ = phong_terms64(sc.faces, fim, wmap, dmap, cs, prm)
        print("phong fwd", case, sigma, rel_err(np_(rgb), np_(want)), float((h > 1e-3).float().mean()))
        assert float((h > 1e-3).float().sum()) > 20  # the highlight is exercised
        assert rel_err(np_(rgb), np_(want)) <= _fwd_tol(kind, sigma)


@pytest.mark.parametrize("kind,H", [("cube4", 257), ("bilinear", 257), ("cube2", 1100), ("trilinear", 1100)])
def test_forward_vs_oracle_large_and_odd_rasters(kind, H):
    sc = Scene(kind, False, False, False, H=H, F=2000, B=1)
    cs, prm = _shading_inputs(sc, sigma=64.0)
    rgb = _render(sc, cs, prm)[0]
    fim, wmap, dmap = sc.maps()
    want = phong_rgb64(sc.faces, fim, wmap, dmap, cs, prm, sc.unlit64(fim, wmap, dmap), BG, False)
    print("phong fwd large", kind, H, rel_err(np_(rgb), np_(want)))
    assert rel_err(np_(rgb), np_(want)) <= _fwd_tol(kind, 64.0)


@pytest.mark.parametrize("kind", ["cube2", "cube4", "bilinear", "trilinear"])
@pytest.mark.parametrize("aa", [False, True])
def test_no_specular_equals_flat_and_ignores_position_and_eye(kind, aa):
    """K = 0 and one unit normal N_f at the three corners of each face: the flat render with face_light = A + D max(N_f . d,
    0) within 2e-5 (the 1e-5 of the normalisation); and then the image does not depend on P or e, bit for bit"""
    sc = Scene(kind, aa, kind == "cube4", False)
    cs, prm = _shading_inputs(sc, K=(0.0, 0.0, 0.0))
    nf = torch.nn.functional.normalize(cs[:, :, 0, :3], dim=-1)
    cs = cs.clone()
    cs[..., :3] = nf[:, :, None, :]
    A, D, d = prm[:, None, 0:3], prm[:, None, 3:6], prm[:, None, 6:9]
    light = A + D * torch.relu((nf * d).sum(-1, keepdim=True))
    flat = sc.render(face_light=light.contiguous())[0]
    phong = _render(sc, cs, prm)[0]
    print("K=0 vs flat", kind, aa, rel_err(np_(phong), np_(flat)))
    assert rel_err(np_(phong), np_(flat)) <= 2e-5
    cs2, prm2 = cs.clone(), prm.clone()
    cs2[..., 3:] = _rand(cs2[..., 3:].shape, -3, 3, seed=30)
    prm2[:, 13:16] = torch.tensor([5.0, -2.0, 1.0], device=DEV)
    assert torch.equal(_render(sc, cs2, prm2)[0], phong)


def test_analytic_highlight():
    """a camera-facing quad (normal -z) at constant depth, P = the corners' NDC (x, y, 0): the mirror point of the light
    towards the eye is p = e - t r with r = the reflected light direction and p_z = 0.  The argmax of the specular image
    (Phong minus its K = 0 twin) lies within one pixel of it."""
    H = 128
    quad = torch.tensor([[[-0.95, -0.95, 2.0], [0.95, -0.95, 2.0], [0.95, 0.95, 2.0]],
                         [[-0.95, -0.95, 2.0], [0.95, 0.95, 2.0], [-0.95, 0.95, 2.0]]], device=DEV)
    faces = torch.cat((quad, quad.flip(1)))[None]  # both orientations
    tex = torch.ones((1, 4, 2, 2, 2, 3), device=DEV)
    cs = torch.zeros((1, 4, 3, 6), device=DEV)
    cs[..., 2] = -1.0
    cs[..., 3:5] = faces[..., :2]
    d = np.array([0.2, 0.1, -1.0])
    e = np.array([-0.3, 0.1, -3.0])
    prm = torch.tensor([[0.2, 0.2, 0.2, 0.5, 0.5, 0.5, *d, 1.0, 1.0, 1.0, 64.0, *e]], dtype=torch.float32, device=DEV)
    prm0 = prm.clone()
    prm0[0, 9:12] = 0
    run = lambda p: _R()._run(faces, tex, H, False, 0.1, 100, 1e-4, (0, 0, 0), True, False, False, corner_shading=cs,
                              shading_params=p)[0]
    spec = (run(prm) - run(prm0))[0, 0]
    dh = d / np.linalg.norm(d)
    r = np.array([-dh[0], -dh[1], dh[2]])  # 2 (n . dh) n - dh with n = (0, 0, -1)
    t = e[2] / r[2]
    px, py = e[0] - t * r[0], e[1] - t * r[1]
    col, yi = (px * H + H - 1) / 2, (py * H + H - 1) / 2  # x_ndc = (2 col + 1 - H) / H
    row = H - 1 - yi
    k = int(torch.argmax(spec))
    got_row, got_col = divmod(k, H)
    print("highlight", (got_row, got_col), (row, col), float(spec.max()))
    assert float(spec.max()) > 0.9
    assert abs(got_row - row) <= 1 and abs(got_col - col) <= 1


def _grad_oracle(sc, cs, prm, tex64=None, uv64=None):
    fim, wmap, dmap = sc.maps()
    c64 = cs.double().requires_grad_(True)
    p64 = prm.double().requires_grad_(True)
    if sc.kind.startswith("cube"):
        unlit = sc.unlit64(fim, wmap, dmap)
    else:
        unlit = sc.unlit64(fim, wmap, dmap, tex=tex64, uvs=uv64, uv_grad=True)
    return fim, wmap, dmap, c64, p64, unlit


@pytest.mark.parametrize("case", GRAD_CASES)
def test_gradients_vs_oracle(case):
    kind, aa, fill_back = case
    sc = Scene(kind, aa, fill_back, False)
    cs0, prm0 = _shading_inputs(sc, sigma=16.0)
    cs = cs0.clone().requires_grad_(True)
    prm = prm0.clone().requires_grad_(True)
    tex = sc.tex.clone().requires_grad_(True)
    uvs = sc.uvs.clone().requires_grad_(True) if sc.uvs is not None else None
    rgb = _render(sc, cs, prm, tex=tex, uvs=uvs)[0]
    g = torch.randn(rgb.shape, generator=torch.Generator().manual_seed(7)).to(DEV)
    (rgb * g).sum().backward()
    tex64 = sc.tex.double().requires_grad_(True) if sc.uvs is not None else None
    uv64 = sc.uvs.double().requires_grad_(True) if sc.uvs is not None else None
    fim, wmap, dmap, c64, p64, unlit = _grad_oracle(sc, cs0, prm0, tex64, uv64)
    want = phong_rgb64(sc.faces, fim, wmap, dmap, c64, p64, unlit, BG, aa)
    (want * g.double()).sum().backward()
    if kind.startswith("cube"):
        # d / d textures = the unlit backward with upstream g * L (L from the float64 oracle)
        L, _, _ = phong_terms64(sc.faces, fim, wmap, dmap, cs0, prm0)
        tex_u = sc.tex.clone().requires_grad_(True)
        unlit32 = sc.render(tex=tex_u, aa=False, H=sc.S)[0]
        (unlit32 * (_upsample(g, aa) * L.float().permute(0, 3, 1, 2))).sum().backward()
        tex_want, tex_tol = tex_u.grad, 1e-4
    else:
        tex_want = tex64.grad
        tex_tol = 5e-4 if kind == "trilinear" else 1e-4
        uv_tol = 1.5e-3 if kind == "trilinear" else 1e-4
        print("uv", case, rel_err(np_(uvs.grad), np_(uv64.grad)), elem_err(np_(uvs.grad), np_(uv64.grad)))
        assert rel_err(np_(uvs.grad), np_(uv64.grad)) <= 1e-4
        assert elem_err(np_(uvs.grad), np_(uv64.grad)) <= uv_tol
    errs = {n: (rel_err(np_(a), np_(b)), elem_err(np_(a), np_(b)))
            for n, a, b in (("cs", cs.grad, c64.grad), ("params", prm.grad, p64.grad), ("tex", tex.grad, tex_want))}
    print("phong grad", case, errs)
    assert c64.grad.abs().max() > 0 and p64.grad[:, 12].abs().max() > 0
    for n, (r, e) in errs.items():
        assert r <= 1e-4, n
    # per element: the normalisations' derivatives and q^sigma in fp32 put the smallest corner components of
    # grad_corner_shading up to 1.1e-3 off (H100, these cases; per tensor 3.3e-6), the params up to 1.8e-4
    assert errs["cs"][1] <= 2e-3
    assert errs["params"][1] <= 5e-4
    assert errs["tex"][1] <= tex_tol


@pytest.mark.parametrize("kind", ["cube4", "bilinear", "trilinear"])
def test_params_gradient_vs_central_difference(kind):
    """sigma, d, e and K of the product's own forward by central differences.  Every normal faces the light (c > 0 with
    a margin), so no pixel sits at the [c > 0] kink; h -> 0 continuously at q = 0."""
    sc = Scene(kind, True, False, False, H=48, F=120, B=1)
    cs, prm0 = _shading_inputs(sc, sigma=6.0, d=(0.1, 0.2, -1.0), e=(0.1, 0.2, -3.0))
    prm = prm0.clone().requires_grad_(True)
    rgb = _render(sc, cs, prm)[0]
    g = torch.randn(rgb.shape, generator=torch.Generator().manual_seed(9)).to(DEV)
    (rgb * g).sum().backward()
    for i, h in ((12, 0.05), (6, 0.01), (7, 0.01), (8, 0.01), (13, 0.01), (14, 0.01), (15, 0.02), (9, 0.05), (10, 0.05)):
        with torch.no_grad():
            pp, pm = prm0.clone(), prm0.clone()
            pp[0, i] += h
            pm[0, i] -= h
            fd = float(((_render(sc, cs, pp)[0].double() - _render(sc, cs, pm)[0].double()) * g.double()).sum() / (2 * h))
        got = float(prm.grad[0, i])
        print("fd", kind, i, fd, got)
        assert abs(fd - got) <= 2e-2 * abs(got) + 1e-3, (i, fd, got)


# ------------------------------------------------------------------------------------------------- direct ABI calls
class _Abi:
    """one Phong forward through the C ABI on a cube scene, and the pieces of a backward call"""

    def __init__(self, Bc=2, Bp=2, kind="cube4"):
        from neural_renderer_b200 import _lib
        self.lib, self.L = _lib.load(), _lib
        self.sc = Scene(kind, True, True, False, H=48, F=200)
        self.cs, self.prm = _shading_inputs(self.sc, Bc=Bc, Bp=Bp)
        sc = self.sc
        self.flags = _lib.NR_RETURN_RGB | _lib.NR_RETURN_ALPHA | _lib.NR_ANTI_ALIASING | _lib.NR_TEX_FILL_BACK | \
            _lib.NR_TEX_Z_BATCH0
        self.maps = self.forward()
        self.g = torch.randn((sc.B, 3, sc.H, sc.H), generator=torch.Generator().manual_seed(5)).to(DEV)
        self.ga = torch.randn((sc.B, sc.H, sc.H), generator=torch.Generator().manual_seed(6)).to(DEV)

    def phong(self, cs=None, prm=None, gcs=None, gprm=None):
        ph = self.L.PhongArgs()
        ph.struct_size = ctypes.sizeof(self.L.PhongArgs)
        cs = self.cs if cs is None else cs
        prm = self.prm if prm is None else prm
        ph.shading_batch, ph.params_batch = cs.shape[0], prm.shape[0]
        ph.corner_shading, ph.params = cs.data_ptr(), prm.data_ptr()
        ph.grad_corner_shading = None if gcs is None else gcs.data_ptr()
        ph.grad_params = None if gprm is None else gprm.data_ptr()
        return ph

    def forward(self):
        sc, L = self.sc, self.L
        B, F, S = sc.B, sc.F, sc.S
        m = {"fim": torch.empty((B, S, S), dtype=torch.int32, device=DEV),
             "wmap": torch.empty((B, 3, S, S), device=DEV), "dmap": torch.empty((B, S, S), device=DEV),
             "rgb": torch.empty((B, 3, S, S), device=DEV), "alpha": torch.empty((B, S, S), device=DEV),
             "out_rgb": torch.empty((B, 3, S // 2, S // 2), device=DEV)}
        nb = self.lib.nr_b200_forward_workspace_bytes(B, F, S, 4, self.flags)
        ws = torch.empty((nb,), dtype=torch.uint8, device=DEV)
        a = L.ForwardArgs()
        a.struct_size = ctypes.sizeof(L.ForwardArgs)
        a.flags = self.flags
        a.batch_size, a.num_faces, a.raster_size, a.texture_size = B, F, S, 4
        a.near_, a.far_, a.eps = 0.1, 100.0, 1e-4
        a.background[0], a.background[1], a.background[2] = BG
        a.faces, a.textures = sc.faces.data_ptr(), sc.tex.data_ptr()
        a.face_index_map, a.weight_map, a.depth_map = m["fim"].data_ptr(), m["wmap"].data_ptr(), m["dmap"].data_ptr()
        a.rgb_map, a.alpha_map, a.out_rgb = m["rgb"].data_ptr(), m["alpha"].data_ptr(), m["out_rgb"].data_ptr()
        a.workspace, a.workspace_bytes = ws.data_ptr(), nb
        ph = self.phong()
        assert self.lib.nr_b200_forward_phong(ctypes.byref(a), ctypes.byref(ph), None) == 0
        torch.cuda.synchronize()
        return m

    def backward(self, flags, gcs=None, gprm=None, gfaces=None, gtex=None, phong=True, textures=True):
        sc, L, m = self.sc, self.L, self.maps
        B, F, S = sc.B, sc.F, sc.S
        nb = self.lib.nr_b200_backward_workspace_bytes(B, F, S, 4, self.flags)
        ws = torch.empty((nb,), dtype=torch.uint8, device=DEV)
        a = L.BackwardArgs()
        a.struct_size = ctypes.sizeof(L.BackwardArgs)
        a.flags = self.flags | flags
        a.batch_size, a.num_faces, a.raster_size, a.texture_size = B, F, S, 4
        a.eps = 1e-4
        a.faces, a.textures = sc.faces.data_ptr(), (sc.tex.data_ptr() if textures else None)
        a.face_index_map, a.weight_map, a.depth_map, a.rgb_map = (m[k].data_ptr() for k in ("fim", "wmap", "dmap", "rgb"))
        a.grad_rgb, a.grad_alpha = self.g.data_ptr(), self.ga.data_ptr()
        a.grad_faces = gfaces.data_ptr() if gfaces is not None else None
        a.grad_textures = gtex.data_ptr() if gtex is not None else None
        a.workspace, a.workspace_bytes = ws.data_ptr(), nb
        if phong:
            ph = self.phong(gcs=gcs, gprm=gprm)
            rc = self.lib.nr_b200_backward_phong(ctypes.byref(a), ctypes.byref(ph), None)
        else:
            rc = self.lib.nr_b200_backward(ctypes.byref(a), None)
        torch.cuda.synchronize()
        return rc


def _guarded(shape, fill=float("nan")):
    """a buffer with 64 guard floats on either side"""
    n = int(np.prod(shape))
    buf = torch.full((n + 128,), fill, device=DEV)
    buf[:64] = 7.0
    buf[-64:] = 7.0
    return buf, buf[64:64 + n].view(shape)


def test_abi_poison_guards_nulls_accumulate_and_two_halves():
    t = _Abi()
    sc, L = t.sc, t.L
    shapes = {"cs": tuple(t.cs.shape), "prm": tuple(t.prm.shape), "faces": tuple(sc.faces.shape), "tex": tuple(sc.tex.shape)}
    bufs = {k: _guarded(s) for k, s in shapes.items()}
    out = {k: v[1] for k, v in bufs.items()}
    assert t.backward(0, out["cs"], out["prm"], out["faces"], out["tex"]) == 0
    for k, (buf, _) in bufs.items():
        assert bool((buf[:64] == 7).all() and (buf[-64:] == 7).all()), k
        assert bool(torch.isfinite(out[k]).all()), k
    ref = {k: v.clone() for k, v in out.items()}
    assert ref["cs"].abs().max() > 0 and ref["prm"].abs().max() > 0
    # every allowed NULL: the other outputs are unchanged bit for bit except for atomics' order (fp32 sums)
    for drop in ("cs", "prm"):
        o = {k: _guarded(s)[1] for k, s in shapes.items()}
        o[drop] = None
        assert t.backward(0, o["cs"], o["prm"], o["faces"], o["tex"]) == 0
        for k in o:
            if o[k] is not None:
                assert rel_err(np_(o[k]), np_(ref[k])) <= 1e-5, (drop, k)
    # NR_GRAD_ACCUMULATE adds into what is there
    pre = {k: _rand(s, -1, 1, seed=40) for k, s in shapes.items()}
    acc = {k: v.clone() for k, v in pre.items()}
    assert t.backward(L.NR_GRAD_ACCUMULATE, acc["cs"], acc["prm"], acc["faces"], acc["tex"]) == 0
    for k in acc:
        assert rel_err(np_(acc[k] - pre[k]), np_(ref[k])) <= 1e-5, k
    # two halves: the Phong gradients come entirely from the texture half; the faces half leaves them untouched
    o = {k: _guarded(s)[1] for k, s in shapes.items()}
    assert t.backward(L.NR_BWD_PART_FACES, o["cs"], o["prm"], o["faces"], o["tex"]) == 0
    assert bool(torch.isnan(o["cs"]).all() and torch.isnan(o["prm"]).all())
    faces_half = o["faces"].clone()
    assert t.backward(L.NR_BWD_PART_TEXTURES, o["cs"], o["prm"], o["faces"], o["tex"]) == 0
    for k in ("cs", "prm", "tex"):
        assert rel_err(np_(o[k]), np_(ref[k])) <= 1e-5, k
    assert torch.equal(o["faces"], faces_half)
    # the faces half equals nr_b200_backward's faces half on the same maps (the edge scan's fp32 atomics are unordered)
    plain = _guarded(shapes["faces"])[1]
    assert t.backward(L.NR_BWD_PART_FACES, gfaces=plain, phong=False) == 0
    print("faces half bit-identical:", torch.equal(plain, faces_half), rel_err(np_(plain), np_(faces_half)))
    assert rel_err(np_(plain), np_(faces_half)) <= 1e-6
    # interior gradient: refused before any launch
    assert t.backward(L.NR_GRAD_INTERIOR, out["cs"], out["prm"], out["faces"], out["tex"]) == -4
    assert t.lib.nr_b200_last_launch_count() == 0


def test_abi_shared_sets_are_sums_and_forward_is_deterministic():
    per = _Abi()
    B = per.sc.B
    shared = _Abi(Bc=1, Bp=1)
    shared.cs, shared.prm = per.cs[:1].contiguous(), per.prm[:1].contiguous()
    per.cs = per.cs[:1].expand(B, -1, -1, -1, -1).contiguous()
    per.prm = per.prm[:1].expand(B, -1).contiguous()
    m1, m2 = per.forward(), shared.forward()
    assert torch.equal(m1["rgb"], m2["rgb"]) and torch.equal(m1["out_rgb"], m2["out_rgb"])
    assert torch.equal(per.forward()["rgb"], m1["rgb"])  # deterministic
    per.maps, shared.maps = m1, m2
    gs = [torch.empty_like(per.cs), torch.empty_like(per.prm), torch.empty_like(per.sc.faces), torch.empty_like(per.sc.tex)]
    gh = [torch.empty_like(shared.cs), torch.empty_like(shared.prm), torch.empty_like(per.sc.faces),
          torch.empty_like(per.sc.tex)]
    shared.g, shared.ga = per.g, per.ga
    assert per.backward(0, *gs) == 0 and shared.backward(0, *gh) == 0
    assert rel_err(np_(gh[0][0]), np_(gs[0].sum(0))) <= 1e-5
    assert rel_err(np_(gh[1][0]), np_(gs[1].sum(0))) <= 1e-5
    assert rel_err(np_(gh[3]), np_(gs[3])) <= 1e-5


# ------------------------------------------------------------------------------------------------- glue kernels
@pytest.mark.parametrize("shared", [True, False])
def test_corner_shading_glue_vs_float64(shared):
    from neural_renderer_b200 import functional as F
    verts, faces = _mesh(shared=shared)
    faces = faces.clone()
    faces[..., 3, 1] = 10 ** 6  # out of range: zeros
    faces[..., 8, 0] = -2
    n0 = torch.nn.functional.normalize(_rand(verts.shape, -1, 1, seed=3), dim=-1)
    fb = torch.cat((faces, faces.flip(-1)), dim=-2)
    for fill_back, idx in ((False, faces), (True, fb)):
        n = n0.clone().requires_grad_(True)
        v = verts.clone().requires_grad_(True)
        cs = F.corner_shading(n, v, idx, fill_back=fill_back)
        n64 = n0.double().requires_grad_(True)
        v64 = verts.double().requires_grad_(True)
        cs64 = F._corner_shading_torch(n64, v64, idx, fill_back)
        assert torch.equal(cs.double(), cs64.detach())
        g = torch.randn(cs.shape, generator=torch.Generator().manual_seed(1)).to(DEV)
        (cs * g).sum().backward()
        (cs64 * g.double()).sum().backward()
        assert rel_err(np_(n.grad), np_(n64.grad)) <= 1e-6 and rel_err(np_(v.grad), np_(v64.grad)) <= 1e-6
        assert elem_err(np_(v.grad), np_(v64.grad)) <= 1e-4  # fp32 atomics over the corners of a vertex


def test_corner_shading_backward_accumulate_and_null():
    from neural_renderer_b200 import _lib
    lib = _lib.load()
    verts, faces = _mesh(B=2)
    B, Nv, Nf = verts.shape[0], verts.shape[1], faces.shape[0]
    g = torch.randn((B, Nf, 3, 6), generator=torch.Generator().manual_seed(2)).to(DEV)
    gn, gv = torch.full_like(verts, float("nan")), torch.full_like(verts, float("nan"))
    fl = _lib.NR_INDICES_SHARED
    assert lib.nr_b200_corner_shading_backward(faces.data_ptr(), g.data_ptr(), B, Nv, Nf, fl, gn.data_ptr(), gv.data_ptr(),
                                               None) == 0
    gv2 = torch.ones_like(verts)
    assert lib.nr_b200_corner_shading_backward(faces.data_ptr(), g.data_ptr(), B, Nv, Nf, fl | _lib.NR_GRAD_ACCUMULATE, None,
                                               gv2.data_ptr(), None) == 0
    torch.cuda.synchronize()
    assert rel_err(np_(gv2 - 1), np_(gv)) <= 1e-6 and bool(torch.isfinite(gn).all())


# ------------------------------------------------------------------------------------------------- Renderer
def _phong_renderer(fill_back, fused):
    r = _renderer(fill_back, fused, "phong")
    r.light_intensity_specular, r.light_shininess = 0.5, 16.0
    return r


@pytest.mark.parametrize("kind", ["cube", "image"])
@pytest.mark.parametrize("fill_back", [False, True])
def test_renderer_phong_fused_matches_op_by_op(kind, fill_back):
    verts0, faces, tex0, uvs = _teapot_inputs(kind)
    out = []
    for fused in (True, False):
        v = verts0.clone().requires_grad_(True)
        tex = tex0.clone().requires_grad_(True)
        img = _phong_renderer(fill_back, fused).render(v, faces, tex, face_uvs=uvs)
        g = torch.randn(img.shape, generator=torch.Generator().manual_seed(3)).to(DEV)
        (img * g).sum().backward()
        out.append((img.detach(), tex.grad, v.grad))
    print("fused vs op", kind, fill_back, [rel_err(np_(a), np_(b)) for a, b in zip(*out)])
    assert rel_err(np_(out[0][0]), np_(out[1][0])) <= 1e-5
    assert rel_err(np_(out[0][1]), np_(out[1][1])) <= 1e-4
    assert rel_err(np_(out[0][2]), np_(out[1][2])) <= 1e-4


def test_renderer_phong_shared_mesh_matches_per_item():
    verts0, faces, tex0, uvs = _teapot_inputs("image")
    r = _phong_renderer(True, True)
    one = verts0[:1].expand(2, -1, -1)
    img_shared = r.render(one, faces, tex0, face_uvs=uvs)
    img_items = r.render(one.contiguous(), faces.contiguous(), tex0, face_uvs=uvs)
    assert rel_err(np_(img_shared), np_(img_items)) <= 1e-6


def test_renderer_phong_step_in_cuda_graph():
    verts0, faces, tex0, uvs = _teapot_inputs("image")
    r = _phong_renderer(True, True)
    v = verts0.clone().requires_grad_(True)
    g = torch.randn((2, 3, 64, 64), generator=torch.Generator().manual_seed(3)).to(DEV)

    def step():
        v.grad = None
        (r.render(v, faces, tex0, face_uvs=uvs) * g).sum().backward()
        return v.grad

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            step()
    torch.cuda.current_stream().wait_stream(s)
    eager = step().clone()
    graph = torch.cuda.CUDAGraph()
    v.grad = None
    with torch.cuda.graph(graph):
        (r.render(v, faces, tex0, face_uvs=uvs) * g).sum().backward()
    graph.replay()
    torch.cuda.synchronize()
    assert rel_err(np_(v.grad), np_(eager)) <= 1e-5


def test_renderer_tensor_light_attributes_and_eye_receive_gradients():
    verts0, faces, tex0, uvs = _teapot_inputs("cube")
    r = _phong_renderer(False, True)
    attrs = {"light_direction": torch.tensor([0.3, 0.8, -0.5], device=DEV),
             "light_color_specular": torch.tensor([1.0, 0.9, 0.8], device=DEV),
             "light_shininess": torch.tensor(16.0, device=DEV),
             "light_intensity_ambient": torch.tensor(0.4, device=DEV),
             "eye": torch.tensor([0.3, 0.5, -2.4], device=DEV)}
    for k, t in attrs.items():
        t.requires_grad_(True)
        setattr(r, k, t)
    img = r.render(verts0, faces, tex0)
    g = torch.randn(img.shape, generator=torch.Generator().manual_seed(4)).to(DEV)
    (img * g).sum().backward()
    for k, t in attrs.items():
        assert t.grad is not None and bool(torch.isfinite(t.grad).all()) and float(t.grad.abs().max()) > 0, k


def test_adam_recovers_light_direction_and_shininess():
    """a target Phong image of the teapot; start from a perturbed light direction and shininess and fit both with Adam on
    the image loss alone.  Measured on an H100: loss 1.5e-3 -> 8.5e-16, angle error 26.4 -> 0.000 degrees, shininess 12 ->
    24.00 (true 24)."""
    verts, faces, tex, _ = _teapot_inputs("cube", B=1)
    tex = torch.full_like(tex, 0.7)
    r = _phong_renderer(False, True)
    r.light_intensity_specular = 0.8
    d_true, s_true = torch.tensor([0.3, 0.8, -0.5], device=DEV), 24.0
    r.light_direction, r.light_shininess = d_true, torch.tensor(s_true, device=DEV)
    with torch.no_grad():
        target = r.render(verts, faces, tex)
    d = torch.tensor([0.6, 0.5, -0.7], device=DEV, requires_grad=True)
    log_s = torch.tensor(math.log(12.0), device=DEV, requires_grad=True)
    opt = torch.optim.Adam([d, log_s], lr=0.02)
    angle = lambda: math.degrees(math.acos(float(torch.nn.functional.cosine_similarity(d.detach(), d_true, dim=0).clamp(-1, 1))))
    a0, loss0 = angle(), None
    for it in range(300):
        opt.zero_grad()
        r.light_direction, r.light_shininess = d, log_s.exp()
        loss = ((r.render(verts, faces, tex) - target) ** 2).mean()
        loss.backward()
        opt.step()
        loss0 = float(loss.detach()) if loss0 is None else loss0
    print("adam fit: loss %.3e -> %.3e, angle %.2f -> %.3f deg, shininess %.2f (true %.1f)"
          % (loss0, float(loss), a0, angle(), float(log_s.exp()), s_true))
    assert float(loss) < 1e-2 * loss0
    assert angle() < 2.0
    assert abs(float(log_s.exp()) - s_true) < 0.1 * s_true
