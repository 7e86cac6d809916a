"""GPU: Phong shading with a light set -- up to eight directional and point lights on top of the Phong light
(include/nr_b200.h, nr_b200_lights_args), and Renderer.lights.

The forward is held to a float64 oracle (oracles_lights.py) on the product's own maps, times the unlit sample, as in
test_gpu_phong.py; the backward to float64 autograd of the same oracle and to central differences of the product's
forward.  NL = 0 and a directional record with params D = K = 0 give the forward of the Phong entry points bit for bit."""
import ctypes

import numpy as np
import pytest
import torch

import abi_harness as H
from helpers import elem_err, np_, rel_err
from oracles_lights import lights_rgb64, lights_terms64
from test_gpu_phong import _Abi, _guarded, _phong_renderer, _shading_inputs
from test_gpu_smooth import BG, FWD_CASES, GRAD_CASES, Scene, _R, _teapot_inputs, _upsample

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda")


def _point(pos, D=(0.5, 0.4, 0.3), K=(0.6, 0.5, 0.4), f=0.0):
    return [*D, *K, *pos, f, 1.0, 0.0]


def _dirl(d, D=(0.3, 0.35, 0.4), K=(0.4, 0.3, 0.2)):
    return [*D, *K, *d, 0.0, 0.0, 0.0]


# light sets in the frame of the scenes' positions (NDC x, y and depth 1..3); the eye of _shading_inputs is (0.2, -0.1, -4)
SETS = {
    "point": [_point((0.3, 0.4, -1.0))],
    "point_dir": [_point((-0.4, 0.2, -0.8), f=0.3), _dirl((-0.2, 0.6, -1.0))],
    "mixed8": [_point((0.3, 0.4, -1.0), f=0.2), _dirl((-0.2, 0.6, -1.0)), _point((-0.5, -0.3, -1.5), f=0.5),
               _dirl((0.5, -0.1, -0.8)), _point((0.0, 0.9, -0.5), f=1.0), _point((0.8, -0.6, -2.0)),
               _dirl((0.1, 0.1, -1.0), K=(0.0, 0.0, 0.0)), _point((-0.9, 0.7, -1.2), f=0.1)],
}


def _light_set(name, B):
    """[B,NL,12]: item b's positions / directions shifted by 0.1 b (B = 1: one set for every item)"""
    rows = []
    for b in range(B):
        rows.append([r[:6] + [r[6] + 0.1 * b, r[7] - 0.05 * b, r[8]] + r[9:] for r in SETS[name]])
    return torch.tensor(rows, dtype=torch.float32, device=DEV)


def _render_l(sc, cs, prm, lt, tex=None, uvs=None, aa=None, H=None):
    aa = sc.aa if aa is None else aa
    H = sc.H if H is None else H
    geom, verts = sc.faces, None
    if sc.indexed:
        verts = sc.faces.reshape(sc.B, -1, 3)
        geom = torch.arange(verts.shape[1], device=DEV, dtype=torch.int32).reshape(-1, 3)
    return _R()._run(geom, sc.tex if tex is None else tex, H, aa, 0.1, 100, 1e-4, BG, True, True, True,
                     textures_fill_back=sc.fill_back, vertices=verts, face_uvs=sc.uvs if uvs is None else uvs,
                     texture_filter=sc.tf, corner_shading=cs, shading_params=prm, lights=lt)


def _fwd_tol(kind, sigma):
    # the gates of test_gpu_phong.py: trilinear = the oracle's float64 level of detail; sigma = 64: q^sigma multiplies the
    # fp32 relative error of q by sigma
    return 6e-5 if kind == "trilinear" else (2e-5 if sigma > 1.0 else 1e-5)


# ------------------------------------------------------------------------------------------------ forward vs float64
@pytest.mark.parametrize("case", FWD_CASES)
@pytest.mark.parametrize("lset", sorted(SETS))
@pytest.mark.parametrize("shared", [True, False])
def test_forward_vs_oracle(case, lset, shared):
    kind, aa, fill_back, indexed = case
    sc = Scene(kind, aa, fill_back, indexed)
    fim, wmap, dmap = sc.maps()
    unlit = sc.unlit64(fim, wmap, dmap)
    lt = _light_set(lset, 1 if shared else sc.B)
    for sigma in (1.0, 64.0):
        cs, prm = _shading_inputs(sc, sigma=sigma)
        rgb = _render_l(sc, cs, prm, lt)[0]
        want = lights_rgb64(sc.faces, fim, wmap, dmap, cs, prm, lt, unlit, BG, aa)
        err = rel_err(np_(rgb), np_(want))
        print("lights fwd", case, lset, shared, sigma, err)
        assert err <= _fwd_tol(kind, sigma)


@pytest.mark.parametrize("kind,H", [("cube4", 257), ("bilinear", 257), ("cube2", 1100), ("trilinear", 1100)])
def test_forward_vs_oracle_large_and_odd_rasters(kind, H):
    sc = Scene(kind, False, False, False, H=H, F=2000, B=1)
    cs, prm = _shading_inputs(sc, sigma=64.0)
    lt = _light_set("mixed8", 1)
    rgb = _render_l(sc, cs, prm, lt)[0]
    fim, wmap, dmap = sc.maps()
    want = lights_rgb64(sc.faces, fim, wmap, dmap, cs, prm, lt, sc.unlit64(fim, wmap, dmap), BG, False)
    print("lights fwd large", kind, H, rel_err(np_(rgb), np_(want)))
    assert rel_err(np_(rgb), np_(want)) <= _fwd_tol(kind, 64.0)


# ------------------------------------------------------------------------------------------------ identity with Phong
class _AbiL(_Abi):
    """_Abi through nr_b200_forward_lights / nr_b200_backward_lights with the light set `lt` (None = a NULL struct)"""

    def __init__(self, lt, Bc=2, Bp=2, kind="cube4", prm=None):
        self.lt, self.prm_override = lt, prm
        super().__init__(Bc=Bc, Bp=Bp, kind=kind)

    def lights(self, glt=None):
        if self.lt is None:
            return None
        la = self.L.LightsArgs()
        la.struct_size = ctypes.sizeof(self.L.LightsArgs)
        la.lights_batch, la.num_lights = self.lt.shape[0], self.lt.shape[1]
        la.lights = self.lt.data_ptr() if self.lt.numel() else None
        la.grad_lights = None if glt is None else glt.data_ptr()
        return la

    def forward(self):
        if self.prm_override is not None:
            self.prm = self.prm_override
        la = self.lights()
        lib = self.lib

        class _Shim:  # _Abi.forward calls nr_b200_forward_phong; route it through the lights entry point
            def __getattr__(self, n):
                return getattr(lib, n)

            def nr_b200_forward_phong(self, a, ph, s):
                return lib.nr_b200_forward_lights(a, ph, None if la is None else ctypes.byref(la), s)
        self.lib = _Shim()
        try:
            m = super().forward()
        finally:
            self.lib = lib
        self.launches = lib.nr_b200_last_launch_count()
        return m

    def backward(self, flags, gcs=None, gprm=None, gfaces=None, gtex=None, phong=True, textures=True, glt=None):
        lib = self.lib
        la = self.lights(glt)

        class _Shim:
            def __getattr__(self, n):
                return getattr(lib, n)

            def nr_b200_backward_phong(self, a, ph, s):
                return lib.nr_b200_backward_lights(a, ph, None if la is None else ctypes.byref(la), s)
        self.lib = _Shim()
        try:
            rc = super().backward(flags, gcs, gprm, gfaces, gtex, phong, textures)
        finally:
            self.lib = lib
        self.launches = lib.nr_b200_last_launch_count()
        return rc


def _grads(t, glt_shape=None):
    o = {"cs": torch.empty_like(t.cs), "prm": torch.empty_like(t.prm), "faces": torch.empty_like(t.sc.faces),
         "tex": torch.empty_like(t.sc.tex)}
    if glt_shape is not None:
        o["lt"] = torch.empty(glt_shape, device=DEV)
    return o


def test_no_lights_is_phong():
    """the same launches and forward maps bit for bit; the gradients up to the order of the texture half's fp32 atomics"""
    ref = _Abi()
    ref_launch = ref.lib.nr_b200_last_launch_count()
    gr = _grads(ref)
    assert ref.backward(0, gr["cs"], gr["prm"], gr["faces"], gr["tex"]) == 0
    bwd_launch = ref.lib.nr_b200_last_launch_count()
    for lt in (None, torch.zeros((2, 0, 12), device=DEV)):
        t = _AbiL(lt)
        assert t.launches == ref_launch
        for k in ref.maps:
            assert torch.equal(t.maps[k], ref.maps[k]), k
        g = _grads(t)
        assert t.backward(0, g["cs"], g["prm"], g["faces"], g["tex"]) == 0
        assert t.launches == bwd_launch
        for k in g:  # the same kernels: equal up to the order of fp32 atomics
            print("NL = 0 vs Phong", k, torch.equal(g[k], gr[k]), rel_err(np_(g[k]), np_(gr[k])))
            assert rel_err(np_(g[k]), np_(gr[k])) <= 1e-6, k


def test_directional_record_is_the_params_light():
    """params D = K = 0 plus one directional record holding params' light: the forward bit for bit, the gradients slot
    for slot (D_j = D, K_j = K, x_j = d) within 1e-6"""
    ref = _Abi()
    prm0 = ref.prm.clone()
    prm0[:, 3:6] = 0
    prm0[:, 9:12] = 0
    lt = torch.cat((ref.prm[:, 3:6], ref.prm[:, 9:12], ref.prm[:, 6:9], torch.zeros((2, 3), device=DEV)), 1)[:, None]
    t = _AbiL(lt.contiguous(), prm=prm0)
    for k in ("rgb", "out_rgb", "fim", "wmap", "alpha"):
        assert torch.equal(t.maps[k], ref.maps[k]), k
    gr, g = _grads(ref), _grads(t, glt_shape=tuple(lt.shape))
    assert ref.backward(0, gr["cs"], gr["prm"], gr["faces"], gr["tex"]) == 0
    assert t.backward(0, g["cs"], g["prm"], g["faces"], g["tex"], glt=g["lt"]) == 0
    pairs = [(g["lt"][:, 0, 0:3], gr["prm"][:, 3:6]), (g["lt"][:, 0, 3:6], gr["prm"][:, 9:12]),
             (g["lt"][:, 0, 6:9], gr["prm"][:, 6:9]), (g["prm"][:, [0, 1, 2, 12, 13, 14, 15]],
                                                     gr["prm"][:, [0, 1, 2, 12, 13, 14, 15]]),
             (g["cs"], gr["cs"]), (g["tex"], gr["tex"]), (g["faces"], gr["faces"])]
    for i, (a, b) in enumerate(pairs):
        print("directional record vs params", i, rel_err(np_(a), np_(b)))
        assert rel_err(np_(a), np_(b)) <= 1e-6, i
    assert bool((g["lt"][..., 9:] == 0).all())


# ------------------------------------------------------------------------------------------------ analytic
def _quad_run(prm, lt, H=128):
    quad = torch.tensor([[[-0.95, -0.95, 2.0], [0.95, -0.95, 2.0], [0.95, 0.95, 2.0]],
                         [[-0.95, -0.95, 2.0], [0.95, 0.95, 2.0], [-0.95, 0.95, 2.0]]], device=DEV)
    faces = torch.cat((quad, quad.flip(1)))[None]
    tex = torch.ones((1, 4, 2, 2, 2, 3), device=DEV)
    cs = torch.zeros((1, 4, 3, 6), device=DEV)
    cs[..., 2] = -1.0
    cs[..., 3:5] = faces[..., :2]  # P = (x_ndc, y_ndc, 0)
    return _R()._run(faces, tex, H, False, 0.1, 100, 1e-4, (0, 0, 0), True, False, False, corner_shading=cs,
                     shading_params=prm, lights=lt)[0][0, 0]


def _px(x, y, H=128):
    return H - 1 - (y * H + H - 1) / 2, (x * H + H - 1) / 2  # (row, col) of NDC (x, y)


def test_analytic_point_light():
    H = 128
    e = np.array([-0.3, 0.1, -3.0])
    x = np.array([0.25, -0.2, -0.6])
    prm = torch.tensor([[0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, -1.0, 0.0, 0.0, 0.0, 64.0, *e]], dtype=torch.float32,
                       device=DEV)
    for f in (0.0, 0.7):
        # diffuse only: the brightest pixel is the foot of the perpendicular from the light to the plane
        lt = torch.tensor([[_point(x, D=(1.0, 1.0, 1.0), K=(0.0, 0.0, 0.0), f=f)]], device=DEV)
        img = _quad_run(prm, lt)
        row, col = _px(x[0], x[1])
        k = int(torch.argmax(img))
        print("foot", f, divmod(k, H), (row, col))
        assert abs(k // H - row) <= 1 and abs(k % H - col) <= 1
        if f > 0:  # two pixels at known distances: the ratio is (cos a) / (cos a)
            vals = []
            for (r_, c_) in ((20, 30), (100, 90)):
                px, py = (2 * c_ + 1 - H) / H, (2 * (H - 1 - r_) + 1 - H) / H
                u = x - np.array([px, py, 0.0])
                rr = np.linalg.norm(u)
                vals.append((float(img[r_, c_]), (-u[2] / (rr + 1e-5)) / (1 + f * rr * rr)))
            got, want = vals[0][0] / vals[1][0], vals[0][1] / vals[1][1]
            print("ratio", got, want)
            assert abs(got / want - 1) <= 1e-4
    # specular only (the render minus its K = 0 twin): the mirror point between the eye and the light
    lt = torch.tensor([[_point(x, D=(0.5, 0.5, 0.5), K=(1.0, 1.0, 1.0))]], device=DEV)
    lt0 = lt.clone()
    lt0[..., 3:6] = 0
    spec = _quad_run(prm, lt) - _quad_run(prm, lt0)
    xm = np.array([x[0], x[1], -x[2]])  # the light mirrored in the plane z = 0
    t = -e[2] / (xm[2] - e[2])
    mx, my = e[0] + t * (xm[0] - e[0]), e[1] + t * (xm[1] - e[1])
    row, col = _px(mx, my)
    k = int(torch.argmax(spec))
    print("mirror point", divmod(k, H), (row, col), float(spec.max()))
    assert float(spec.max()) > 0.9
    assert abs(k // H - row) <= 1 and abs(k % H - col) <= 1


# ------------------------------------------------------------------------------------------------ gradients
@pytest.mark.parametrize("case", GRAD_CASES)
def test_gradients_vs_oracle(case):
    kind, aa, fill_back = case
    sc = Scene(kind, aa, fill_back, False)
    cs0, prm0 = _shading_inputs(sc, sigma=16.0)
    lt0 = _light_set("point_dir", sc.B)
    lt0 = torch.cat((lt0, _light_set("point", sc.B)), dim=1)
    cs = cs0.clone().requires_grad_(True)
    prm = prm0.clone().requires_grad_(True)
    lt = lt0.clone().requires_grad_(True)
    tex = sc.tex.clone().requires_grad_(True)
    uvs = sc.uvs.clone().requires_grad_(True) if sc.uvs is not None else None
    rgb = _render_l(sc, cs, prm, lt, tex=tex, uvs=uvs)[0]
    g = torch.randn(rgb.shape, generator=torch.Generator().manual_seed(7)).to(DEV)
    (rgb * g).sum().backward()
    fim, wmap, dmap = sc.maps()
    c64, p64, l64 = (t.double().requires_grad_(True) for t in (cs0, prm0, lt0))
    tex64 = sc.tex.double().requires_grad_(True) if sc.uvs is not None else None
    uv64 = sc.uvs.double().requires_grad_(True) if sc.uvs is not None else None
    if kind.startswith("cube"):
        unlit = sc.unlit64(fim, wmap, dmap)
    else:
        unlit = sc.unlit64(fim, wmap, dmap, tex=tex64, uvs=uv64, uv_grad=True)
    want = lights_rgb64(sc.faces, fim, wmap, dmap, c64, p64, l64, unlit, BG, aa)
    (want * g.double()).sum().backward()
    if kind.startswith("cube"):
        L, _ = lights_terms64(sc.faces, fim, wmap, dmap, cs0, prm0, lt0)
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
    assert bool((lt.grad[..., 10:] == 0).all())
    errs = {n: (rel_err(np_(a), np_(b)), elem_err(np_(a), np_(b)))
            for n, a, b in (("cs", cs.grad, c64.grad), ("params", prm.grad, p64.grad),
                            ("lights", lt.grad[..., :10], l64.grad[..., :10]), ("tex", tex.grad, tex_want))}
    print("lights grad", case, errs)
    assert l64.grad[..., 6:10].abs().max() > 0
    for n, (r, e) in errs.items():
        assert r <= 1e-4, n
    assert errs["cs"][1] <= 2e-3
    assert errs["params"][1] <= 5e-4
    # grad_lights per element: at most 6.2e-5 on an H100 over these cases (trilinear); per tensor 2.2e-6
    assert errs["lights"][1] <= 2e-4
    assert errs["tex"][1] <= tex_tol


@pytest.mark.parametrize("kind", ["cube4", "bilinear", "trilinear"])
def test_light_gradient_vs_central_difference(kind):
    """a point light's position, falloff, D_j and K_j by central differences of the product's forward"""
    sc = Scene(kind, True, False, False, H=48, F=120, B=1)
    cs, prm = _shading_inputs(sc, sigma=6.0, d=(0.1, 0.2, -1.0), e=(0.1, 0.2, -3.0))
    lt0 = torch.tensor([[_point((0.2, 0.3, -1.2), f=0.4), _dirl((-0.2, 0.6, -1.0))]], device=DEV)
    lt = lt0.clone().requires_grad_(True)
    rgb = _render_l(sc, cs, prm, lt)[0]
    g = torch.randn(rgb.shape, generator=torch.Generator().manual_seed(9)).to(DEV)
    (rgb * g).sum().backward()
    for i, h in ((6, 0.01), (7, 0.01), (8, 0.01), (9, 0.02), (0, 0.02), (4, 0.02)):
        with torch.no_grad():
            lp, lm = lt0.clone(), lt0.clone()
            lp[0, 0, i] += h
            lm[0, 0, i] -= h
            fd = float(((_render_l(sc, cs, prm, lp)[0].double() - _render_l(sc, cs, prm, lm)[0].double())
                        * g.double()).sum() / (2 * h))
        got = float(lt.grad[0, 0, i])
        print("fd", kind, i, fd, got)
        assert abs(fd - got) <= 2e-2 * abs(got) + 1e-3, (i, fd, got)


# ------------------------------------------------------------------------------------------------ direct ABI calls
def test_abi_poison_guards_offsets_nulls_accumulate_and_two_halves():
    lt = _light_set("mixed8", 2)
    t = _AbiL(lt)
    L = t.L
    shapes = {"cs": tuple(t.cs.shape), "prm": tuple(t.prm.shape), "faces": tuple(t.sc.faces.shape),
              "tex": tuple(t.sc.tex.shape), "lt": tuple(lt.shape)}
    call = lambda flags, o: t.backward(flags, o["cs"], o["prm"], o["faces"], o["tex"], glt=o["lt"])
    bufs = {k: _guarded(s) for k, s in shapes.items()}
    out = {k: v[1] for k, v in bufs.items()}
    assert call(0, out) == 0
    for k, (buf, _) in bufs.items():
        assert bool((buf[:64] == 7).all() and (buf[-64:] == 7).all()), k
        assert bool(torch.isfinite(out[k]).all()), k
    ref = {k: v.clone() for k, v in out.items()}
    assert ref["lt"][..., :10].abs().max() > 0 and bool((ref["lt"][..., 10:] == 0).all())
    # 4- and 8-byte-offset buffers between guard words, poisoned
    for off in (4, 8):
        o = {k: H.alloc(s, np.float32, off, DEV) for k, s in shapes.items()}
        for v in o.values():
            H.poison(v)
        assert call(0, o) == 0
        for k in o:
            assert H.guards_intact(o[k]), (off, k)
            assert rel_err(np_(o[k]), np_(ref[k])) <= 1e-5, (off, k)
    # every allowed NULL
    for drop in ("cs", "prm", "lt"):
        o = {k: _guarded(s)[1] for k, s in shapes.items()}
        o[drop] = None
        assert call(0, o) == 0
        for k in o:
            if o[k] is not None:
                assert rel_err(np_(o[k]), np_(ref[k])) <= 1e-5, (drop, k)
    # NR_GRAD_ACCUMULATE adds into what is there (slots 10-11 of grad_lights keep the prefill)
    pre = {k: torch.rand(s, generator=torch.Generator().manual_seed(40)).to(DEV) for k, s in shapes.items()}
    acc = {k: v.clone() for k, v in pre.items()}
    assert call(L.NR_GRAD_ACCUMULATE, acc) == 0
    for k in acc:
        assert rel_err(np_(acc[k] - pre[k]), np_(ref[k])) <= 1e-5, k
    assert torch.equal(acc["lt"][..., 10:], pre["lt"][..., 10:])
    # two halves: the light gradients come from the texture half; the faces half writes no light output
    o = {k: _guarded(s)[1] for k, s in shapes.items()}
    assert call(L.NR_BWD_PART_FACES, o) == 0
    assert bool(torch.isnan(o["cs"]).all() and torch.isnan(o["prm"]).all() and torch.isnan(o["lt"]).all())
    assert call(L.NR_BWD_PART_TEXTURES, o) == 0
    for k in o:
        assert rel_err(np_(o[k]), np_(ref[k])) <= 1e-5, k
    assert call(L.NR_GRAD_INTERIOR, out) == -4
    assert t.lib.nr_b200_last_launch_count() == 0


def test_abi_shared_set_is_the_sum_and_forward_is_deterministic():
    lt = _light_set("mixed8", 1)
    per = _AbiL(lt.expand(2, -1, -1).contiguous())
    shared = _AbiL(lt.contiguous())
    assert torch.equal(per.maps["rgb"], shared.maps["rgb"]) and torch.equal(per.maps["out_rgb"], shared.maps["out_rgb"])
    assert torch.equal(per.forward()["rgb"], per.maps["rgb"])  # deterministic
    shared.g, shared.ga = per.g, per.ga
    gp, gs = _grads(per, glt_shape=(2, 8, 12)), _grads(shared, glt_shape=(1, 8, 12))
    assert per.backward(0, gp["cs"], gp["prm"], gp["faces"], gp["tex"], glt=gp["lt"]) == 0
    assert shared.backward(0, gs["cs"], gs["prm"], gs["faces"], gs["tex"], glt=gs["lt"]) == 0
    assert rel_err(np_(gs["lt"][0]), np_(gp["lt"].sum(0))) <= 1e-5
    assert rel_err(np_(gs["cs"]), np_(gp["cs"])) <= 1e-5


# ------------------------------------------------------------------------------------------------ Renderer
def _lit_renderer(fill_back, fused, lights):
    r = _phong_renderer(fill_back, fused)
    r.lights = lights
    return r


def test_renderer_empty_lights_is_phong():
    from neural_renderer_b200 import functional as F
    verts, faces, tex, uvs = _teapot_inputs("image")
    a = _phong_renderer(True, True).render(verts, faces, tex, face_uvs=uvs)
    for lights in ([], torch.zeros((0, 12), device=DEV)):
        assert torch.equal(_lit_renderer(True, True, lights).render(verts, faces, tex, face_uvs=uvs), a)
    lit = _lit_renderer(True, True, [F.point_light((0.5, 1.0, -2.0), falloff=0.3)]).render(verts, faces, tex, face_uvs=uvs)
    assert float((lit - a).abs().max()) > 1e-3


def _teapot_lights():
    """device records: a render captured in a CUDA graph must not copy host data"""
    from neural_renderer_b200 import functional as F
    return [F.point_light((0.5, 1.0, -2.0), 0.6, (1.0, 0.8, 0.6), 0.5, falloff=0.3, device=DEV),
            F.directional_light((-0.4, 0.2, -1.0), 0.3, intensity_specular=0.4, device=DEV)]


@pytest.mark.parametrize("kind", ["cube", "image"])
@pytest.mark.parametrize("fill_back", [False, True])
def test_renderer_lights_fused_matches_op_by_op(kind, fill_back):
    verts0, faces, tex0, uvs = _teapot_inputs(kind)
    out = []
    for fused in (True, False):
        v = verts0.clone().requires_grad_(True)
        tex = tex0.clone().requires_grad_(True)
        img = _lit_renderer(fill_back, fused, _teapot_lights()).render(v, faces, tex, face_uvs=uvs)
        g = torch.randn(img.shape, generator=torch.Generator().manual_seed(3)).to(DEV)
        (img * g).sum().backward()
        out.append((img.detach(), tex.grad, v.grad))
    print("fused vs op", kind, fill_back, [rel_err(np_(a), np_(b)) for a, b in zip(*out)])
    assert rel_err(np_(out[0][0]), np_(out[1][0])) <= 1e-5
    assert rel_err(np_(out[0][1]), np_(out[1][1])) <= 1e-4
    assert rel_err(np_(out[0][2]), np_(out[1][2])) <= 1e-4


def test_renderer_lights_step_in_cuda_graph():
    verts0, faces, tex0, uvs = _teapot_inputs("image")
    r = _lit_renderer(True, True, _teapot_lights())
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


def test_renderer_tensor_light_arguments_receive_gradients():
    from neural_renderer_b200 import functional as F
    verts0, faces, tex0, _ = _teapot_inputs("cube")
    ts = {"pos": torch.tensor([0.5, 1.0, -2.0], device=DEV), "falloff": torch.tensor(0.3, device=DEV),
          "color": torch.tensor([1.0, 0.8, 0.6], device=DEV), "dir": torch.tensor([-0.4, 0.2, -1.0], device=DEV),
          "spec": torch.tensor(0.4, device=DEV)}
    for t in ts.values():
        t.requires_grad_(True)
    r = _lit_renderer(False, True, [F.point_light(ts["pos"], 0.6, ts["color"], 0.5, falloff=ts["falloff"]),
                                    F.directional_light(ts["dir"], 0.3, intensity_specular=ts["spec"])])
    img = r.render(verts0, faces, tex0)
    g = torch.randn(img.shape, generator=torch.Generator().manual_seed(4)).to(DEV)
    (img * g).sum().backward()
    for k, t in ts.items():
        assert t.grad is not None and bool(torch.isfinite(t.grad).all()) and float(t.grad.abs().max()) > 0, k


def test_adam_recovers_point_light_position():
    """a textured sphere seen from four viewpoints, lit by params' weak directional light and one point light; start the
    light 0.64 units away and fit its position with Adam on the image loss alone.  Measured on an H100: loss 4.2e-3 ->
    8.8e-12, position error 0.640 -> 6.8e-5.  Near the optimum Adam's step is about its learning rate, hence the decay."""
    import neural_renderer_b200 as nr
    from neural_renderer_b200 import functional as F, synthetic
    v, f = synthetic.sphere_mesh(2000)
    verts = torch.tensor(v * 0.8, dtype=torch.float32, device=DEV)[None]
    faces = torch.tensor(f, device=DEV)[None]
    tex = torch.rand((1, f.shape[0], 2, 2, 2, 3), generator=torch.Generator().manual_seed(5)).to(DEV) * 0.6 + 0.3
    r = nr.Renderer()
    r.image_size, r.fill_back, r.shading = 64, True, 'phong'
    r.light_intensity_ambient, r.light_intensity_directional, r.light_intensity_specular = 0.2, 0.2, 0.0
    r.light_shininess = 16.0
    eyes = [(0.0, 0.0, -2.7), (1.9, 0.5, -1.9), (-1.9, 0.3, -1.9), (0.0, 1.9, -1.9)]
    x_true = torch.tensor([0.9, 1.0, -1.4], device=DEV)

    def loss_at(x, targets=None):
        out = []
        for i, e in enumerate(eyes):
            r.eye = e
            r.lights = [F.point_light(x, 0.7, (1.0, 0.9, 0.8), 0.6, falloff=0.2)]
            img = r.render(verts, faces, tex)
            out.append(img if targets is None else ((img - targets[i]) ** 2).mean())
        return out if targets is None else sum(out)

    with torch.no_grad():
        targets = loss_at(x_true)
    x = torch.tensor([0.5, 1.3, -1.8], device=DEV, requires_grad=True)
    err0 = float((x.detach() - x_true).norm())
    opt = torch.optim.Adam([x], lr=0.02)
    sched = torch.optim.lr_scheduler.ExponentialLR(opt, 0.993)
    loss0 = None
    for it in range(700):
        opt.zero_grad()
        loss = loss_at(x, targets)
        loss.backward()
        opt.step()
        sched.step()
        loss0 = float(loss.detach()) if loss0 is None else loss0
    err = float((x.detach() - x_true).norm())
    print("adam point light: loss %.3e -> %.3e, position error %.4f -> %.2e" % (loss0, float(loss.detach()), err0, err))
    assert err0 >= 0.5
    assert err <= 1e-3
