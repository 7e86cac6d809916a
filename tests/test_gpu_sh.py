"""GPU: Phong shading lit by an environment -- second-order spherical-harmonic irradiance (include/nr_b200.h,
nr_b200_sh_args), rasterize(..., environment_sh=...), Renderer.environment_sh and F.sh_from_environment_map.

The forward is held to a float64 oracle (oracles_sh.py) on the product's own maps, times the unlit sample, as in
test_gpu_lights.py; the backward to float64 autograd of the same oracle and to central differences of the product's
forward.  A NULL struct runs the light-set / Phong kernels themselves, and S = 0 gives their forward bit for bit."""
import ctypes
import math

import numpy as np
import pytest
import torch

import abi_harness as H
from helpers import elem_err, np_, rel_err
from oracles_sh import C0, sh_rgb64, sh_terms64
from test_gpu_lights import _AbiL, _grads, _light_set, _lit_renderer
from test_gpu_phong import _guarded, _phong_renderer, _shading_inputs
from test_gpu_smooth import BG, FWD_CASES, GRAD_CASES, Scene, _R, _teapot_inputs, _upsample

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda")


def _env(B, seed=31):
    """[B,9,3] irradiance-ready coefficients: a bright, coloured, direction-dependent environment (E goes negative for
    a few normals, which the product passes through); item b is shifted by 0.05 b"""
    g = torch.Generator().manual_seed(seed)
    base = torch.randn((9, 3), generator=g) * 0.25
    base[0] = torch.tensor([0.8, 0.7, 0.6]) / C0
    return torch.stack([base + 0.05 * b for b in range(B)]).to(DEV).contiguous()


def _render_s(sc, cs, prm, lt, sh, tex=None, uvs=None, aa=None, H=None):
    aa = sc.aa if aa is None else aa
    H = sc.H if H is None else H
    geom, verts = sc.faces, None
    if sc.indexed:
        verts = sc.faces.reshape(sc.B, -1, 3)
        geom = torch.arange(verts.shape[1], device=DEV, dtype=torch.int32).reshape(-1, 3)
    return _R()._run(geom, sc.tex if tex is None else tex, H, aa, 0.1, 100, 1e-4, BG, True, True, True,
                     textures_fill_back=sc.fill_back, vertices=verts, face_uvs=sc.uvs if uvs is None else uvs,
                     texture_filter=sc.tf, corner_shading=cs, shading_params=prm, lights=lt, environment_sh=sh)


def _fwd_tol(kind, sigma):
    # the gates of test_gpu_phong.py / test_gpu_lights.py
    return 6e-5 if kind == "trilinear" else (2e-5 if sigma > 1.0 else 1e-5)


def _mode_inputs(sc, mode, sigma, B):
    """(cs, params, lights) of a forward mode: SH alone (params A = D = K = 0), SH + params, SH + params + 3 lights"""
    cs, prm = _shading_inputs(sc, sigma=sigma)
    lt = None
    if mode == "alone":
        prm = prm.clone()
        prm[:, 0:6] = 0
        prm[:, 9:12] = 0
    elif mode == "lights3":
        lt = torch.cat((_light_set("point_dir", B), _light_set("point", B)), dim=1).contiguous()
    return cs, prm, lt


# ------------------------------------------------------------------------------------------------ forward vs float64
@pytest.mark.parametrize("case", FWD_CASES)
@pytest.mark.parametrize("mode", ["alone", "params", "lights3"])
@pytest.mark.parametrize("shared", [True, False])
def test_forward_vs_oracle(case, mode, shared):
    kind, aa, fill_back, indexed = case
    sc = Scene(kind, aa, fill_back, indexed)
    fim, wmap, dmap = sc.maps()
    unlit = sc.unlit64(fim, wmap, dmap)
    sh = _env(1 if shared else sc.B)
    for sigma in (1.0, 64.0):
        cs, prm, lt = _mode_inputs(sc, mode, sigma, 1 if shared else sc.B)
        rgb = _render_s(sc, cs, prm, lt, sh)[0]
        want = sh_rgb64(sc.faces, fim, wmap, dmap, cs, prm, lt, sh, unlit, BG, aa)
        err = rel_err(np_(rgb), np_(want))
        print("sh fwd", case, mode, shared, sigma, err)
        assert err <= _fwd_tol(kind, sigma)


@pytest.mark.parametrize("kind,H", [("cube4", 257), ("bilinear", 257), ("cube2", 1100), ("trilinear", 1100)])
def test_forward_vs_oracle_large_and_odd_rasters(kind, H):
    sc = Scene(kind, False, False, False, H=H, F=2000, B=1)
    cs, prm, lt = _mode_inputs(sc, "lights3", 64.0, 1)
    sh = _env(1)
    rgb = _render_s(sc, cs, prm, lt, sh)[0]
    fim, wmap, dmap = sc.maps()
    want = sh_rgb64(sc.faces, fim, wmap, dmap, cs, prm, lt, sh, sc.unlit64(fim, wmap, dmap), BG, False)
    print("sh fwd large", kind, H, rel_err(np_(rgb), np_(want)))
    assert rel_err(np_(rgb), np_(want)) <= _fwd_tol(kind, 64.0)


# ------------------------------------------------------------------------------------------------ identities
class _AbiS(_AbiL):
    """_Abi through nr_b200_forward_sh / nr_b200_backward_sh with the light set `lt` (None = a NULL light struct) and
    the environment `sh` (None = a NULL SH struct)"""

    def __init__(self, sh, lt=None, Bc=2, Bp=2, kind="cube4", prm=None):
        self.sh = sh
        super().__init__(lt, Bc=Bc, Bp=Bp, kind=kind, prm=prm)

    def sh_args(self, gsh=None):
        if self.sh is None:
            return None
        sa = self.L.ShArgs()
        sa.struct_size = ctypes.sizeof(self.L.ShArgs)
        sa.sh_batch = self.sh.shape[0]
        sa.sh = self.sh.data_ptr()
        sa.grad_sh = None if gsh is None else gsh.data_ptr()
        return sa

    def forward(self):
        sa = self.sh_args()
        lib = self.lib

        class _Shim:  # _AbiL.forward calls nr_b200_forward_lights; route it through the SH entry point
            def __getattr__(self, n):
                return getattr(lib, n)

            def nr_b200_forward_lights(self, a, ph, la, s):
                return lib.nr_b200_forward_sh(a, ph, la, None if sa is None else ctypes.byref(sa), s)
        self.lib = _Shim()
        try:
            m = super().forward()
        finally:
            self.lib = lib
        return m

    def backward(self, flags, gcs=None, gprm=None, gfaces=None, gtex=None, phong=True, textures=True, glt=None, gsh=None):
        sa = self.sh_args(gsh)
        lib = self.lib

        class _Shim:
            def __getattr__(self, n):
                return getattr(lib, n)

            def nr_b200_backward_lights(self, a, ph, la, s):
                return lib.nr_b200_backward_sh(a, ph, la, None if sa is None else ctypes.byref(sa), s)
        self.lib = _Shim()
        try:
            rc = super().backward(flags, gcs, gprm, gfaces, gtex, phong, textures, glt)
        finally:
            self.lib = lib
        self.launches = lib.nr_b200_last_launch_count()
        return rc


def _call(t, flags, o):
    kw = {"gsh": o.get("sh")} if isinstance(t, _AbiS) else {}
    return t.backward(flags, o["cs"], o["prm"], o["faces"], o["tex"], glt=o.get("lt"), **kw)


@pytest.mark.parametrize("with_lights", [False, True])
def test_null_struct_and_zero_environment_are_the_lights_call(with_lights):
    """a NULL struct: the same launches and maps bit for bit; S = 0: the forward bit for bit, the gradients within the
    order of the texture half's fp32 atomics (two identical light-set calls differ as much)"""
    lt = _light_set("mixed8", 2) if with_lights else None
    ref = _AbiL(lt)
    ref_launch = ref.launches
    glt_shape = tuple(lt.shape) if lt is not None else None
    gr = _grads(ref, glt_shape)
    assert _call(ref, 0, gr) == 0
    bwd_launch = ref.launches
    t = _AbiS(None, lt)
    assert t.launches == ref_launch
    for k in ref.maps:
        assert torch.equal(t.maps[k], ref.maps[k]), k
    g = _grads(t, glt_shape)
    assert _call(t, 0, g) == 0
    assert t.launches == bwd_launch
    for k in g:
        print("NULL sh vs lights", k, rel_err(np_(g[k]), np_(gr[k])))
        assert rel_err(np_(g[k]), np_(gr[k])) <= 1e-6, k
    for bs in (1, 2):
        z = _AbiS(torch.zeros((bs, 9, 3), device=DEV), lt)
        for k in ref.maps:
            assert torch.equal(z.maps[k], ref.maps[k]), (bs, k)
        gz = _grads(z, glt_shape)
        gz["sh"] = torch.empty((bs, 9, 3), device=DEV)
        assert _call(z, 0, gz) == 0
        for k in gr:
            print("S = 0 vs lights", bs, k, rel_err(np_(gz[k]), np_(gr[k])))
            assert rel_err(np_(gz[k]), np_(gr[k])) <= 1e-6, (bs, k)
        assert float(gz["sh"].abs().max()) > 0


# ------------------------------------------------------------------------------------------------ analytic
def _sphere_run(sh, H=96):
    """a unit-normal sphere (radius 0.8 at depth 2.5, orthographic NDC faces) with a white texture and params
    A = D = K = 0: the image is E(nh) alone; also the normal image of rasterize_attributes and the alpha"""
    from neural_renderer_b200 import synthetic
    v, f = synthetic.sphere_mesh(3000)
    v = torch.tensor(v, dtype=torch.float32, device=DEV)
    fi = torch.tensor(f, device=DEV).long()
    fi = torch.cat((fi, fi.flip(1)))  # both windings: whichever faces the viewer is drawn
    faces = (v * 0.8 + torch.tensor([0.0, 0.0, 2.5], device=DEV))[fi][None]
    n = v[fi][None]                                                                     # [1,F,3,3] unit normals
    cs = torch.cat((n, faces), dim=-1).contiguous()
    prm = torch.tensor([[0.0] * 12 + [16.0, 0.0, 0.0, -4.0]], device=DEV)
    tex = torch.ones((1, faces.shape[1], 2, 2, 2, 3), device=DEV)
    rgb, alpha = _R()._run(faces, tex, H, False, 0.1, 100, 1e-4, (0, 0, 0), True, True, False, corner_shading=cs,
                           shading_params=prm, environment_sh=sh)[:2]
    nimg = _R().rasterize_attributes(faces, H, False, 0.1, 100, 1e-4, face_attributes=n)
    return rgb, alpha, nimg


def test_white_furnace():
    """S = (1/C0, 0, ...) under a white albedo renders 1 at every covered pixel (|nh| < 1 only touches k >= 1)"""
    sh = torch.zeros((1, 9, 3), device=DEV)
    sh[0, 0] = 1.0 / C0
    rgb, alpha, _ = _sphere_run(sh)
    cov = (alpha > 0)[:, None].expand_as(rgb)
    err = float((rgb[cov] - 1).abs().max())
    print("white furnace", err, int(cov.sum()))
    assert int(cov.sum()) > 1000
    assert err <= 1e-6


def test_linear_environment_from_the_helper():
    """F.sh_from_environment_map(1 + omega_y) lights a sphere as 1 + (2/3) nh_y, nh from rasterize_attributes"""
    from neural_renderer_b200 import functional as F
    He, We = 256, 512
    t = math.pi * (torch.arange(He, dtype=torch.float64) + 0.5) / He
    env = (1 + torch.cos(t))[:, None, None].expand(He, We, 3)
    sh = F.sh_from_environment_map(env).float().to(DEV)
    rgb, alpha, nimg = _sphere_run(sh)
    nh = nimg / (torch.linalg.vector_norm(nimg, dim=1, keepdim=True) + 1e-5)
    want = (1 + 2.0 / 3.0 * nh[:, 1:2]).expand_as(rgb)
    cov = (alpha > 0)[:, None].expand_as(rgb)
    err = float((rgb[cov] - want[cov]).abs().max())
    print("linear environment", err)
    # the midpoint rule at He = 256 errs by about 1e-5 (tests/test_sh_cpu.py), fp32 adds a few ulp
    assert err <= 1e-4


# ------------------------------------------------------------------------------------------------ gradients
@pytest.mark.parametrize("case", GRAD_CASES)
@pytest.mark.parametrize("mode", ["params", "lights3"])
def test_gradients_vs_oracle(case, mode):
    """mode "params": the Phong gradient kernel's variant without a light set; "lights3": its light-set variant"""
    kind, aa, fill_back = case
    sc = Scene(kind, aa, fill_back, False)
    cs0, prm0, lt0 = _mode_inputs(sc, mode, 16.0, sc.B)
    sh0 = _env(sc.B)
    cs, prm, sh = (t.clone().requires_grad_(True) for t in (cs0, prm0, sh0))
    lt = lt0.clone().requires_grad_(True) if lt0 is not None else None
    tex = sc.tex.clone().requires_grad_(True)
    uvs = sc.uvs.clone().requires_grad_(True) if sc.uvs is not None else None
    rgb = _render_s(sc, cs, prm, lt, sh, tex=tex, uvs=uvs)[0]
    g = torch.randn(rgb.shape, generator=torch.Generator().manual_seed(7)).to(DEV)
    (rgb * g).sum().backward()
    fim, wmap, dmap = sc.maps()
    c64, p64, s64 = (t.double().requires_grad_(True) for t in (cs0, prm0, sh0))
    l64 = lt0.double().requires_grad_(True) if lt0 is not None else None
    tex64 = sc.tex.double().requires_grad_(True) if sc.uvs is not None else None
    uv64 = sc.uvs.double().requires_grad_(True) if sc.uvs is not None else None
    if kind.startswith("cube"):
        unlit = sc.unlit64(fim, wmap, dmap)
    else:
        unlit = sc.unlit64(fim, wmap, dmap, tex=tex64, uvs=uv64, uv_grad=True)
    want = sh_rgb64(sc.faces, fim, wmap, dmap, c64, p64, l64, s64, unlit, BG, aa)
    (want * g.double()).sum().backward()
    if kind.startswith("cube"):
        L, _ = sh_terms64(sc.faces, fim, wmap, dmap, cs0, prm0, lt0, sh0)
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
    pairs = [("sh", sh.grad, s64.grad), ("cs", cs.grad, c64.grad), ("params", prm.grad, p64.grad), ("tex", tex.grad, tex_want)]
    if lt is not None:
        pairs.append(("lights", lt.grad[..., :10], l64.grad[..., :10]))
    errs = {n: (rel_err(np_(a), np_(b)), elem_err(np_(a), np_(b))) for n, a, b in pairs}
    print("sh grad", case, mode, errs)
    for n, (r, e) in errs.items():
        assert r <= 1e-4, n
    assert errs["cs"][1] <= 2e-3
    assert errs["params"][1] <= 5e-4
    if lt is not None:
        assert errs["lights"][1] <= 2e-4
    assert errs["sh"][1] <= 1e-4
    assert errs["tex"][1] <= tex_tol


@pytest.mark.parametrize("kind", ["cube4", "bilinear", "trilinear"])
def test_sh_gradient_vs_central_difference(kind):
    sc = Scene(kind, True, False, False, H=48, F=120, B=1)
    cs, prm, lt = _mode_inputs(sc, "lights3", 6.0, 1)
    sh0 = _env(1)
    sh = sh0.clone().requires_grad_(True)
    rgb = _render_s(sc, cs, prm, lt, sh)[0]
    g = torch.randn(rgb.shape, generator=torch.Generator().manual_seed(9)).to(DEV)
    (rgb * g).sum().backward()
    for k, c in ((0, 0), (1, 1), (3, 2), (4, 0), (6, 1), (8, 2)):
        h = 0.05
        with torch.no_grad():
            sp, sm = sh0.clone(), sh0.clone()
            sp[0, k, c] += h
            sm[0, k, c] -= h
            fd = float(((_render_s(sc, cs, prm, lt, sp)[0].double() - _render_s(sc, cs, prm, lt, sm)[0].double())
                        * g.double()).sum() / (2 * h))
        got = float(sh.grad[0, k, c])
        print("fd", kind, k, c, fd, got)
        assert abs(fd - got) <= 2e-3 * abs(got) + 1e-3, (k, c, fd, got)


# ------------------------------------------------------------------------------------------------ direct ABI calls
def test_abi_poison_guards_offsets_nulls_accumulate_and_two_halves():
    lt = _light_set("point_dir", 2)
    sh = _env(2)
    t = _AbiS(sh, lt)
    L = t.L
    shapes = {"cs": tuple(t.cs.shape), "prm": tuple(t.prm.shape), "faces": tuple(t.sc.faces.shape),
              "tex": tuple(t.sc.tex.shape), "lt": tuple(lt.shape), "sh": tuple(sh.shape)}
    bufs = {k: _guarded(s) for k, s in shapes.items()}
    out = {k: v[1] for k, v in bufs.items()}
    assert _call(t, 0, out) == 0
    for k, (buf, _) in bufs.items():
        assert bool((buf[:64] == 7).all() and (buf[-64:] == 7).all()), k
        assert bool(torch.isfinite(out[k]).all()), k
    ref = {k: v.clone() for k, v in out.items()}
    assert float(ref["sh"].abs().min()) > 0
    for off in (4, 8):
        o = {k: H.alloc(s, np.float32, off, DEV) for k, s in shapes.items()}
        for v in o.values():
            H.poison(v)
        assert _call(t, 0, o) == 0
        for k in o:
            assert H.guards_intact(o[k]), (off, k)
            assert rel_err(np_(o[k]), np_(ref[k])) <= 1e-5, (off, k)
    for drop in ("cs", "prm", "lt", "sh"):
        o = {k: _guarded(s)[1] for k, s in shapes.items()}
        o[drop] = None
        assert _call(t, 0, o) == 0
        for k in o:
            if o[k] is not None:
                assert rel_err(np_(o[k]), np_(ref[k])) <= 1e-5, (drop, k)
    pre = {k: torch.rand(s, generator=torch.Generator().manual_seed(40)).to(DEV) for k, s in shapes.items()}
    acc = {k: v.clone() for k, v in pre.items()}
    assert _call(t, L.NR_GRAD_ACCUMULATE, acc) == 0
    for k in acc:
        assert rel_err(np_(acc[k] - pre[k]), np_(ref[k])) <= 1e-5, k
    # two halves: the SH gradient comes from the texture half; the faces half writes no shading output
    o = {k: _guarded(s)[1] for k, s in shapes.items()}
    assert _call(t, L.NR_BWD_PART_FACES, o) == 0
    for k in ("cs", "prm", "lt", "sh"):
        assert bool(torch.isnan(o[k]).all()), k
    assert _call(t, L.NR_BWD_PART_TEXTURES, o) == 0
    for k in o:
        assert rel_err(np_(o[k]), np_(ref[k])) <= 1e-5, k
    assert _call(t, L.NR_GRAD_INTERIOR, out) == -4
    assert t.lib.nr_b200_last_launch_count() == 0


def test_abi_shared_environment_is_the_sum_and_forward_is_deterministic():
    sh = _env(1)
    per = _AbiS(sh.expand(2, -1, -1).contiguous())
    shared = _AbiS(sh.contiguous())
    assert torch.equal(per.maps["rgb"], shared.maps["rgb"]) and torch.equal(per.maps["out_rgb"], shared.maps["out_rgb"])
    assert torch.equal(per.forward()["rgb"], per.maps["rgb"])  # deterministic
    shared.g, shared.ga = per.g, per.ga
    gp, gs = _grads(per), _grads(shared)
    gp["sh"], gs["sh"] = torch.empty((2, 9, 3), device=DEV), torch.empty((1, 9, 3), device=DEV)
    assert _call(per, 0, gp) == 0
    assert _call(shared, 0, gs) == 0
    assert rel_err(np_(gs["sh"][0]), np_(gp["sh"].sum(0))) <= 1e-5
    assert rel_err(np_(gs["cs"]), np_(gp["cs"])) <= 1e-5


# ------------------------------------------------------------------------------------------------ Renderer
def _env_renderer(fill_back, fused, sh, lights=()):
    r = _lit_renderer(fill_back, fused, list(lights))
    r.environment_sh = sh
    return r


def test_renderer_no_environment_is_phong():
    verts, faces, tex, uvs = _teapot_inputs("image")
    a = _phong_renderer(True, True).render(verts, faces, tex, face_uvs=uvs)
    assert torch.equal(_env_renderer(True, True, None).render(verts, faces, tex, face_uvs=uvs), a)
    lit = _env_renderer(True, True, _env(1)).render(verts, faces, tex, face_uvs=uvs)
    assert float((lit - a).abs().max()) > 1e-2


@pytest.mark.parametrize("kind", ["cube", "image"])
@pytest.mark.parametrize("fill_back", [False, True])
def test_renderer_environment_fused_matches_op_by_op(kind, fill_back):
    from neural_renderer_b200 import functional as F
    verts0, faces, tex0, uvs = _teapot_inputs(kind)
    out = []
    for fused in (True, False):
        v = verts0.clone().requires_grad_(True)
        tex = tex0.clone().requires_grad_(True)
        sh = _env(1).clone().requires_grad_(True)
        r = _env_renderer(fill_back, fused, sh, [F.point_light((0.5, 1.0, -2.0), falloff=0.3, device=DEV)])
        img = r.render(v, faces, tex, face_uvs=uvs)
        g = torch.randn(img.shape, generator=torch.Generator().manual_seed(3)).to(DEV)
        (img * g).sum().backward()
        out.append((img.detach(), tex.grad, v.grad, sh.grad))
    print("fused vs op", kind, fill_back, [rel_err(np_(a), np_(b)) for a, b in zip(*out)])
    assert rel_err(np_(out[0][0]), np_(out[1][0])) <= 1e-5
    for i in (1, 2, 3):
        assert rel_err(np_(out[0][i]), np_(out[1][i])) <= 1e-4, i


def test_renderer_environment_step_in_cuda_graph():
    verts0, faces, tex0, uvs = _teapot_inputs("image")
    sh = _env(1).clone().requires_grad_(True)
    r = _env_renderer(True, True, sh)
    v = verts0.clone().requires_grad_(True)
    g = torch.randn((2, 3, 64, 64), generator=torch.Generator().manual_seed(3)).to(DEV)

    def step():
        v.grad = sh.grad = None
        (r.render(v, faces, tex0, face_uvs=uvs) * g).sum().backward()
        return v.grad, sh.grad

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            step()
    torch.cuda.current_stream().wait_stream(s)
    eager = [x.clone() for x in step()]
    graph = torch.cuda.CUDAGraph()
    v.grad = sh.grad = None
    with torch.cuda.graph(graph):
        (r.render(v, faces, tex0, face_uvs=uvs) * g).sum().backward()
    graph.replay()
    torch.cuda.synchronize()
    assert rel_err(np_(v.grad), np_(eager[0])) <= 1e-5
    assert rel_err(np_(sh.grad), np_(eager[1])) <= 1e-5


def test_renderer_environment_map_receives_gradients():
    from neural_renderer_b200 import functional as F
    verts0, faces, tex0, _ = _teapot_inputs("cube")
    env = (torch.rand((16, 32, 3), generator=torch.Generator().manual_seed(8)) + 0.5).to(DEV).requires_grad_(True)
    r = _env_renderer(False, True, F.sh_from_environment_map(env))
    img = r.render(verts0, faces, tex0)
    g = torch.randn(img.shape, generator=torch.Generator().manual_seed(4)).to(DEV)
    (img * g).sum().backward()
    assert env.grad is not None and bool(torch.isfinite(env.grad).all()) and float(env.grad.abs().max()) > 0


def test_adam_recovers_all_27_coefficients():
    """a textured sphere seen from six viewpoints, lit by the environment alone (A = D = K = 0); start from a uniform
    grey environment and fit all 27 coefficients with Adam on the image loss alone"""
    import neural_renderer_b200 as nr
    from neural_renderer_b200 import synthetic
    v, f = synthetic.sphere_mesh(2000)
    verts = torch.tensor(v * 0.8, dtype=torch.float32, device=DEV)[None]
    faces = torch.tensor(f, device=DEV)[None]
    tex = torch.rand((1, f.shape[0], 2, 2, 2, 3), generator=torch.Generator().manual_seed(5)).to(DEV) * 0.6 + 0.3
    r = nr.Renderer()
    r.image_size, r.fill_back, r.shading = 64, True, 'phong'
    r.light_intensity_ambient = r.light_intensity_directional = r.light_intensity_specular = 0.0
    eyes = [(0.0, 0.0, -2.7), (0.0, 0.0, 2.7), (2.7, 0.0, 0.0), (-2.7, 0.0, 0.0), (0.0, 1.9, -1.9), (0.3, -1.9, 1.9)]
    sh_true = _env(1, seed=33)

    def loss_at(sh, targets=None):
        out = []
        for i, e in enumerate(eyes):
            r.eye = e
            r.environment_sh = sh
            img = r.render(verts, faces, tex)
            out.append(img if targets is None else ((img - targets[i]) ** 2).mean())
        return out if targets is None else sum(out)

    with torch.no_grad():
        targets = loss_at(sh_true)
    sh = torch.zeros((1, 9, 3), device=DEV)
    sh[0, 0] = 0.5 / C0
    sh.requires_grad_(True)
    err0 = float((sh.detach() - sh_true).abs().max())
    opt = torch.optim.Adam([sh], lr=0.05)
    sched = torch.optim.lr_scheduler.ExponentialLR(opt, 0.99)
    loss0 = None
    for it in range(800):
        opt.zero_grad()
        loss = loss_at(sh, targets)
        loss.backward()
        opt.step()
        sched.step()
        loss0 = float(loss.detach()) if loss0 is None else loss0
    err = float((sh.detach() - sh_true).abs().max())
    print("adam sh: loss %.3e -> %.3e, max coefficient error %.4f -> %.2e" % (loss0, float(loss.detach()), err0, err))
    assert err0 >= 0.3
    assert err <= 1e-3
