"""GPU: Phong shading through a tangent-space normal map (include/nr_b200.h, nr_b200_normal_map_args),
rasterize(..., normal_map=, corner_tangents=), Renderer.normal_map and the tangent glue of functional.py.

The forward is held to the float64 oracle of oracles_normal_map.py on the product's own maps, the backward to float64
autograd of the same oracle and to central differences of the product's forward.  A flat map renders as
nr_b200_forward_sh bit for bit, and a NULL struct is that call."""
import math

import numpy as np

import pytest
import torch

from helpers import elem_err, np_, rel_err
from oracles_normal_map import nm_rgb64
from test_gpu_lights import _light_set
from test_gpu_phong import _shading_inputs
from test_gpu_sh import _env
from test_gpu_smooth import BG, Scene, _R

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda")

# image kinds of test_gpu_smooth.FWD_CASES: (kind, aa, fill_back, indexed)
NM_CASES = [(k, aa, fb, ix) for k in ("bilinear", "trilinear") for (aa, fb, ix) in
            ((False, False, False), (True, True, False), (True, False, True), (False, True, True))]


def _map(Bm, Hm, Wm, seed=41, amp=0.4):
    """[Bm,Hm,Wm,3] decoded vectors around +z, tilted by up to `amp`"""
    g = torch.Generator().manual_seed(seed)
    m = torch.randn((Bm, Hm, Wm, 3), generator=g) * amp
    m[..., 2] = 1.0 + 0.2 * torch.rand((Bm, Hm, Wm), generator=g)
    return m.to(DEV).contiguous()


def _tangents(Bt, F, seed=43):
    """[Bt,F,3,4]: random tangents, handedness +1 or -1 per face (every corner of a face the same)"""
    g = torch.Generator().manual_seed(seed)
    t = torch.randn((Bt, F, 3, 3), generator=g)
    w = torch.where(torch.rand((Bt, F, 1), generator=g) < 0.5, -1.0, 1.0).expand(Bt, F, 3)
    return torch.cat((t, w[..., None]), dim=-1).to(DEV).contiguous()


def _inputs(sc, mode, sigma, Bsh):
    cs, prm = _shading_inputs(sc, sigma=sigma, Bc=Bsh, Bp=Bsh)
    lt = _light_set("point_dir", Bsh) if mode in ("lights", "both") else None
    sh = _env(Bsh) if mode in ("sh", "both") else None
    return cs, prm, lt, sh


def _render(sc, cs, prm, lt, sh, nm, tg, tex=None, uvs=None, aa=None, H=None):
    aa = sc.aa if aa is None else aa
    H = sc.H if H is None else H
    geom, verts = sc.faces, None
    if sc.indexed:
        verts = sc.faces.reshape(sc.B, -1, 3)
        geom = torch.arange(verts.shape[1], device=DEV, dtype=torch.int32).reshape(-1, 3)
    return _R()._run(geom, sc.tex if tex is None else tex, H, aa, 0.1, 100, 1e-4, BG, True, True, True,
                     textures_fill_back=sc.fill_back, vertices=verts, face_uvs=sc.uvs if uvs is None else uvs,
                     texture_filter=sc.tf, corner_shading=cs, shading_params=prm, lights=lt, environment_sh=sh,
                     normal_map=nm, corner_tangents=tg)


def _fwd_tol(kind, sigma):
    # the gates of test_gpu_phong.py
    return 6e-5 if kind == "trilinear" else (2e-5 if sigma > 1.0 else 1e-5)


# ------------------------------------------------------------------------------------------------ forward vs float64
@pytest.mark.parametrize("case", NM_CASES)
@pytest.mark.parametrize("mode", ["phong", "lights", "sh", "both"])
@pytest.mark.parametrize("hw", [(1, 1), (1, 23), (37, 53)])
def test_forward_vs_oracle(case, mode, hw):
    kind, aa, fill_back, indexed = case
    sc = Scene(kind, aa, fill_back, indexed)
    fim, wmap, dmap = sc.maps()
    unlit = sc.unlit64(fim, wmap, dmap)
    for shared in (True, False):
        B1 = 1 if shared else sc.B
        nm, tg = _map(B1, *hw), _tangents(sc.B if shared else 1, sc.F)  # Bm and Bt differ: both strides in play
        for sigma in (1.0, 64.0):
            cs, prm, lt, sh = _inputs(sc, mode, sigma, sc.B)
            rgb = _render(sc, cs, prm, lt, sh, nm, tg)[0]
            want = nm_rgb64(sc.faces, fim, wmap, dmap, cs, prm, lt, sh, nm, tg, sc.uvs, unlit, BG, aa, fill_back)
            err = rel_err(np_(rgb), np_(want))
            print("nm fwd", case, mode, hw, shared, sigma, err)
            assert err <= _fwd_tol(kind, sigma)


@pytest.mark.parametrize("kind,H", [("bilinear", 257), ("trilinear", 1100)])
def test_forward_vs_oracle_large_and_odd_rasters(kind, H):
    sc = Scene(kind, False, False, False, H=H, F=2000, B=1)
    cs, prm, lt, sh = _inputs(sc, "both", 64.0, 1)
    nm, tg = _map(1, 37, 53), _tangents(1, sc.F)
    rgb = _render(sc, cs, prm, lt, sh, nm, tg)[0]
    fim, wmap, dmap = sc.maps()
    want = nm_rgb64(sc.faces, fim, wmap, dmap, cs, prm, lt, sh, nm, tg, sc.uvs, sc.unlit64(fim, wmap, dmap), BG, False,
                    False)
    print("nm fwd large", kind, H, rel_err(np_(rgb), np_(want)))
    assert rel_err(np_(rgb), np_(want)) <= _fwd_tol(kind, 64.0)


# ------------------------------------------------------------------------------------------------ identities
def _all_grads(sc, cs, prm, lt, sh, nm, tg, g, seed_inputs=True):
    leaves = {"cs": cs, "prm": prm, "lt": lt, "sh": sh, "nm": nm, "tg": tg, "tex": sc.tex, "uvs": sc.uvs}
    leaves = {k: (v.detach().clone().requires_grad_(True) if v is not None else None) for k, v in leaves.items()}
    out = _render(sc, leaves["cs"], leaves["prm"], leaves["lt"], leaves["sh"], leaves["nm"], leaves["tg"],
                  tex=leaves["tex"], uvs=leaves["uvs"])
    (out[0] * g).sum().backward()
    return out, {k: v.grad for k, v in leaves.items() if v is not None}


@pytest.mark.parametrize("case", NM_CASES[:3])
@pytest.mark.parametrize("mode", ["phong", "both"])
def test_flat_map_is_the_sh_call(case, mode):
    """(0,0,1) everywhere: rgb, alpha and depth bit for bit those of nr_b200_forward_sh, the shared gradients within the
    spread of two identical SH calls; the map receives a gradient, the tangents exactly none (gt = m_x g' + sigma
    (m_y g' x n) = 0)"""
    kind, aa, fill_back, indexed = case
    sc = Scene(kind, aa, fill_back, indexed)
    cs, prm, lt, sh = _inputs(sc, mode, 16.0, sc.B)
    flat = torch.zeros((1, 5, 7, 3), device=DEV)
    flat[..., 2] = 1.0
    tg = _tangents(sc.B, sc.F)
    g = torch.randn((sc.B, 3, sc.H, sc.H), generator=torch.Generator().manual_seed(5)).to(DEV)
    o_nm, g_nm = _all_grads(sc, cs, prm, lt, sh, flat, tg, g)
    o_sh, g_sh = _all_grads(sc, cs, prm, lt, sh, None, None, g)
    _, g_sh2 = _all_grads(sc, cs, prm, lt, sh, None, None, g)
    for a, b in zip(o_nm[:3], o_sh[:3]):
        assert torch.equal(a, b)
    for k, v in g_sh.items():
        spread = float((g_sh2[k] - v).abs().max())
        err = float((g_nm[k] - v).abs().max())
        print("flat", case, mode, k, err, spread)
        assert err <= max(2 * spread, 1e-6 * float(v.abs().max()))
    assert float(g_nm["nm"].abs().max()) > 0 and float(g_nm["tg"].abs().max()) == 0


# ------------------------------------------------------------------------------------------------ analytic bump
def _bump_quad(H, mirror=False):
    """a camera-facing quad (normal -z) at depth 2 with UVs over [0,1]^2 (u -> 1 - u when mirrored), both windings"""
    r, z = 0.95, 2.0
    v = torch.tensor([[-r, -r, z], [r, -r, z], [r, r, z], [-r, r, z]], dtype=torch.float32)
    uv = torch.tensor([[0, 0], [1, 0], [1, 1], [0, 1]], dtype=torch.float32)
    if mirror:
        uv[:, 0] = 1 - uv[:, 0]
    tri = torch.tensor([[0, 1, 2], [0, 2, 3]])
    faces = torch.cat((v[tri], v[tri].flip(1)))[None].to(DEV)
    uvs = torch.cat((uv[tri], uv[tri].flip(1)))[None].to(DEV)
    return faces, uvs, v, tri


def _bump_map(Wm=64, Hm=16, deg=30.0):
    """left half tilted by -deg, right half by +deg about the v axis (unit vectors in the x-z plane of tangent space)"""
    a = math.radians(deg)
    m = torch.zeros((1, Hm, Wm, 3))
    m[:, :, : Wm // 2] = torch.tensor([-math.sin(a), 0.0, math.cos(a)])
    m[:, :, Wm // 2:] = torch.tensor([math.sin(a), 0.0, math.cos(a)])
    return m.to(DEV)


def _bump_render(faces, uvs, tg, d, H=128):
    cs = torch.zeros((1, 4, 3, 6), device=DEV)
    cs[..., 2] = -1.0
    cs[..., 3:5] = faces[..., :2]
    prm = torch.tensor([[0, 0, 0, 1, 1, 1, d[0], d[1], d[2], 0, 0, 0, 1.0, 0, 0, -4.0]], device=DEV)
    tex = torch.ones((1, 4, 4, 3), device=DEV)
    return _R()._run(faces, tex, H, False, 0.1, 100, 1e-4, (0, 0, 0), True, True, False, face_uvs=uvs,
                     corner_shading=cs, shading_params=prm, normal_map=_bump_map(), corner_tangents=tg)


def test_analytic_bump_and_mirror():
    H = 128
    faces, uvs, _, _ = _bump_quad(H)
    tg = torch.zeros((1, 4, 3, 4), device=DEV)
    tg[..., 0] = 1.0
    tg[..., 3] = 1.0
    tg[:, 2:, :, :] = -tg[:, 2:, :, :]  # the reversed copies: (-T, -w), as their normal is -N
    d = torch.tensor([0.3, 0.0, -1.0])
    d = d / d.norm()
    rgb, alpha = _bump_render(faces, uvs, tg, d.tolist())[:2]
    img = rgb[0, 0]
    # tangent-space (x, z) -> world: x along T = +x, z along n = -z
    a = math.radians(30.0)
    left = torch.tensor([-math.sin(a), 0.0, -math.cos(a)])
    right = torch.tensor([math.sin(a), 0.0, -math.cos(a)])
    want_l, want_r = float(max(left @ d, 0)), float(max(right @ d, 0))
    # pixel centre x -> u: the quad spans [-0.95, 0.95] in NDC; keep more than one texel (1/63 in u) off the seam and
    # two pixels off the edges
    xs = (2 * torch.arange(H, dtype=torch.float64) + 1 - H) / H
    u = (xs + 0.95) / 1.9
    cols_l = ((u > 0.03) & (u < 0.5 - 2.0 / 63)).nonzero().flatten()
    cols_r = ((u > 0.5 + 2.0 / 63) & (u < 0.97)).nonzero().flatten()
    rows = slice(8, H - 8)
    el = float((img[rows][:, cols_l] - want_l).abs().max())
    er = float((img[rows][:, cols_r] - want_r).abs().max())
    print("bump", want_l, want_r, el, er)
    assert el <= 3e-5 and er <= 3e-5
    assert abs(want_l - want_r) > 0.2  # the two halves really differ
    # mirrored UVs, tangents from F.vertex_tangents: T = (-1, 0, 0); a light in the y-z plane gives the mirror image
    from neural_renderer_b200 import functional as F
    faces_m, uvs_m, v, tri = _bump_quad(H, mirror=True)
    n = torch.tensor([[0.0, 0.0, -1.0]]).expand(4, 3)[None].to(DEV)
    vt = F.vertex_tangents(v[None].to(DEV), tri.to(DEV), uvs_m[0, :2], n)
    assert torch.allclose(vt[0, :, :3], torch.tensor([-1.0, 0.0, 0.0], device=DEV).expand(4, 3), atol=1e-4)
    tri_all = torch.cat((tri, tri.flip(1))).to(DEV)
    tg_m = F.corner_tangents(vt, tri_all, fill_back=True)
    d2 = [0.0, 0.4, -1.0]
    img0 = _bump_render(faces, uvs, tg, d2)[0][0, 0]
    img1 = _bump_render(faces_m, uvs_m, tg_m, d2)[0][0, 0]
    cov = _bump_render(faces, uvs, tg, d2)[1][0] > 0
    err = float((img1 - img0.flip(-1))[cov & cov.flip(-1)].abs().max())
    print("mirror", err)
    assert err <= 3e-5


# ------------------------------------------------------------------------------------------------ gradients
@pytest.mark.parametrize("case", [("bilinear", False, False, True), ("bilinear", True, True, False),
                                  ("trilinear", False, True, True), ("trilinear", True, False, False)])
@pytest.mark.parametrize("mode", ["phong", "both"])
def test_gradients_vs_float64(case, mode):
    kind, aa, fill_back, indexed = case
    sc = Scene(kind, aa, fill_back, indexed)
    cs, prm, lt, sh = _inputs(sc, mode, 16.0, sc.B)
    nm, tg = _map(1, 9, 11), _tangents(sc.B, sc.F)
    g = torch.randn((sc.B, 3, sc.H, sc.H), generator=torch.Generator().manual_seed(7)).to(DEV)
    _, got = _all_grads(sc, cs, prm, lt, sh, nm, tg, g)
    fim, wmap, dmap = sc.maps()
    ref = {k: v.detach().double().clone().requires_grad_(True) for k, v in
           {"cs": cs, "prm": prm, "lt": lt, "sh": sh, "nm": nm, "tg": tg, "tex": sc.tex, "uvs": sc.uvs}.items()
           if v is not None}
    unlit = sc.unlit64(fim, wmap, dmap, tex=ref["tex"], uvs=ref["uvs"], uv_grad=True)
    want = nm_rgb64(sc.faces, fim, wmap, dmap, ref["cs"], ref["prm"], ref.get("lt"), ref.get("sh"), ref["nm"], ref["tg"],
                    ref["uvs"], unlit, BG, aa, fill_back)
    (want * g.double()).sum().backward()
    for k, r in ref.items():
        err = rel_err(np_(got[k]), np_(r.grad))
        print("nm grad", case, mode, k, err, elem_err(np_(got[k]), np_(r.grad)))
        assert err <= 1e-4, k
    # the per-element gates of test_gpu_phong.py for the shading inputs
    assert elem_err(np_(got["cs"]), np_(ref["cs"].grad)) <= 2e-3
    assert elem_err(np_(got["prm"]), np_(ref["prm"].grad)) <= 5e-4


def test_central_differences():
    """the product's own forward, stepped in map texels, a tangent and a UV corner, against its gradient"""
    sc = Scene("bilinear", False, False, False, B=1)
    cs, prm, lt, sh = _inputs(sc, "phong", 4.0, 1)
    nm, tg = _map(1, 5, 6, amp=0.3), _tangents(1, sc.F)
    g = torch.randn((1, 3, sc.H, sc.H), generator=torch.Generator().manual_seed(9)).to(DEV)
    _, got = _all_grads(sc, cs, prm, lt, sh, nm, tg, g)
    fim = sc.maps()[0]
    f0 = int(fim[fim >= 0].flatten().mode().values)  # a face that covers pixels

    def loss(nm_, tg_, uvs_):
        return float((_render(sc, cs, prm, lt, sh, nm_, tg_, uvs=uvs_)[0].double() * g.double()).sum())
    checks = []
    for (i, j, c) in ((2, 3, 0), (1, 2, 1), (3, 4, 2)):
        checks.append(("nm", (0, i, j, c)))
    checks += [("tg", (0, f0, 1, 0)), ("tg", (0, f0, 2, 1)), ("uvs", (0, f0, 1, 0)), ("uvs", (0, f0, 2, 1))]
    for name, idx in checks:
        # n' is linear in t: a larger step keeps the fp32 sum's noise down; a small UV step crosses few texel edges,
        # where the bilinear derivative jumps
        h = {"nm": 1e-3, "tg": 1e-2, "uvs": 1e-4}[name]
        base = {"nm": nm, "tg": tg, "uvs": sc.uvs}
        p, m = base[name].clone(), base[name].clone()
        p[idx] += h
        m[idx] -= h
        args = lambda t: [t if k == name else base[k] for k in ("nm", "tg", "uvs")]
        num = (loss(*args(p)) - loss(*args(m))) / (2 * h)
        ana = float(got[name][idx])
        print("cd", name, idx, num, ana)
        assert abs(num - ana) <= 0.02 * abs(ana) + 1e-3  # 1e-3: the fp32 forward's noise over the step


# ------------------------------------------------------------------------------------------------ ABI behaviour
def test_binding_behaviour():
    """through the binding: a deterministic forward, shared sets (Bm = Bt = 1) = the per-item sums, no gradient into w,
    the two halves (texture half, hook, faces half) = one call, and each NULL output leaves the others unchanged"""
    R = _R()
    sc = Scene("bilinear", False, True, True)
    cs, prm, lt, sh = _inputs(sc, "both", 16.0, sc.B)
    nm, tg = _map(1, 9, 11), _tangents(1, sc.F)
    g = torch.randn((sc.B, 3, sc.H, sc.H), generator=torch.Generator().manual_seed(3)).to(DEV)
    r0 = _render(sc, cs, prm, lt, sh, nm, tg)[0]
    r1 = _render(sc, cs, prm, lt, sh, nm, tg)[0]
    assert torch.equal(r0, r1)
    _, ga = _all_grads(sc, cs, prm, lt, sh, nm, tg, g)
    # shared sets (Bm = Bt = 1) against the per-item gradients of expanded per-item copies
    _, gb = _all_grads(sc, cs, prm, lt, sh, nm.expand(sc.B, -1, -1, -1).contiguous(),
                       tg.expand(sc.B, -1, -1, -1).contiguous(), g)
    assert rel_err(np_(ga["nm"][0]), np_(gb["nm"].sum(0))) <= 1e-5
    assert rel_err(np_(ga["tg"][0]), np_(gb["tg"].sum(0))) <= 1e-5
    assert float(ga["tg"][..., 3].abs().max()) == 0  # no gradient into w
    # the two halves (texture half, then faces half) through the binding's texture-grad hook = one call
    calls = []
    prev = R.set_texture_grad_hook(lambda gt: calls.append(1))
    try:
        _, gh = _all_grads(sc, cs, prm, lt, sh, nm, tg, g)  # two halves (texture half, hook, faces half)
    finally:
        R.set_texture_grad_hook(prev)
    assert calls
    for k in ga:
        assert rel_err(np_(gh[k]), np_(ga[k])) <= 1e-5, k
    # each NULL output: a map that does not require grad leaves the other gradients as they were
    leaves = {k: v.detach().clone() for k, v in {"cs": cs, "prm": prm, "nm": nm, "tg": tg, "tex": sc.tex,
                                                   "uvs": sc.uvs}.items()}
    for skip in ("nm", "tg", "cs", "uvs"):
        req = {k: v.clone().requires_grad_(k != skip) for k, v in leaves.items()}
        out = _render(sc, req["cs"], req["prm"], lt, sh, req["nm"], req["tg"], tex=req["tex"], uvs=req["uvs"])
        (out[0] * g).sum().backward()
        for k, v in req.items():
            if k != skip:
                assert rel_err(np_(v.grad), np_(ga[k])) <= 1e-5, (skip, k)


# ------------------------------------------------------------------------------------------------ direct ABI calls
class _AbiNM:
    """a normal-mapped Phong render through the C ABI on an image scene (anti-aliasing, fill_back), with a light set and
    an SH environment, and the backward with every gradient output"""

    def __init__(self, Bm=2, Bt=2):
        import ctypes
        from neural_renderer_b200 import _lib
        self.ct, self.lib, self.L = ctypes, _lib.load(), _lib
        self.sc = sc = Scene("bilinear", True, True, False, H=48, F=200)
        self.cs, self.prm, self.lt, self.sh = _inputs(sc, "both", 16.0, sc.B)
        self.nm, self.tg = _map(Bm, 9, 11), _tangents(Bt, sc.F)
        self.flags = _lib.NR_RETURN_RGB | _lib.NR_RETURN_ALPHA | _lib.NR_ANTI_ALIASING | _lib.NR_TEX_FILL_BACK | \
            _lib.NR_TEX_UV
        self.maps = self.forward()
        self.g = torch.randn((sc.B, 3, sc.H, sc.H), generator=torch.Generator().manual_seed(5)).to(DEV)
        self.ga = torch.randn((sc.B, sc.H, sc.H), generator=torch.Generator().manual_seed(6)).to(DEV)

    def shapes(self):
        sc = self.sc
        return {"cs": tuple(self.cs.shape), "prm": tuple(self.prm.shape), "lt": tuple(self.lt.shape),
                "sh": tuple(self.sh.shape), "nm": tuple(self.nm.shape), "tg": tuple(self.tg.shape),
                "faces": tuple(sc.faces.shape), "tex": tuple(sc.tex.shape), "uvs": tuple(sc.uvs.shape)}

    def structs(self, o=None):
        ct, L = self.ct, self.L
        o = o or {}
        p = lambda k: None if o.get(k) is None else o[k].data_ptr()
        ph = L.PhongArgs()
        ph.struct_size = ct.sizeof(L.PhongArgs)
        ph.shading_batch, ph.params_batch = self.cs.shape[0], self.prm.shape[0]
        ph.corner_shading, ph.params = self.cs.data_ptr(), self.prm.data_ptr()
        ph.grad_corner_shading, ph.grad_params = p("cs"), p("prm")
        la = L.LightsArgs()
        la.struct_size = ct.sizeof(L.LightsArgs)
        la.lights_batch, la.num_lights = self.lt.shape[0], self.lt.shape[1]
        la.lights, la.grad_lights = self.lt.data_ptr(), p("lt")
        sa = L.ShArgs()
        sa.struct_size = ct.sizeof(L.ShArgs)
        sa.sh_batch, sa.sh, sa.grad_sh = self.sh.shape[0], self.sh.data_ptr(), p("sh")
        na = L.NormalMapArgs()
        na.struct_size = ct.sizeof(L.NormalMapArgs)
        na.map_batch, na.tangent_batch = self.nm.shape[0], self.tg.shape[0]
        na.map_height, na.map_width = self.nm.shape[1], self.nm.shape[2]
        na.normal_map, na.corner_tangents = self.nm.data_ptr(), self.tg.data_ptr()
        na.grad_normal_map, na.grad_corner_tangents = p("nm"), p("tg")
        return ph, la, sa, na

    def forward(self, with_nm=True):
        ct, sc, L = self.ct, self.sc, self.L
        B, F, S = sc.B, sc.F, sc.S
        m = {"fim": torch.empty((B, S, S), dtype=torch.int32, device=DEV),
             "wmap": torch.empty((B, 3, S, S), device=DEV), "dmap": torch.empty((B, S, S), device=DEV),
             "rgb": torch.empty((B, 3, S, S), device=DEV), "alpha": torch.empty((B, S, S), device=DEV),
             "out_rgb": torch.empty((B, 3, S // 2, S // 2), device=DEV)}
        nb = self.lib.nr_b200_forward_workspace_bytes(B, F, S, 0, self.flags)
        ws = torch.empty((nb,), dtype=torch.uint8, device=DEV)
        a = L.ForwardArgs()
        a.struct_size = ct.sizeof(L.ForwardArgs)
        a.flags = self.flags
        a.batch_size, a.num_faces, a.raster_size, a.texture_size = B, F, S, 0
        a.near_, a.far_, a.eps = 0.1, 100.0, 1e-4
        a.background[0], a.background[1], a.background[2] = BG
        a.faces, a.textures = sc.faces.data_ptr(), sc.tex.data_ptr()
        a.face_uvs, a.texture_height, a.texture_width = sc.uvs.data_ptr(), sc.tex.shape[1], sc.tex.shape[2]
        a.face_index_map, a.weight_map, a.depth_map = m["fim"].data_ptr(), m["wmap"].data_ptr(), m["dmap"].data_ptr()
        a.rgb_map, a.alpha_map, a.out_rgb = m["rgb"].data_ptr(), m["alpha"].data_ptr(), m["out_rgb"].data_ptr()
        a.workspace, a.workspace_bytes = ws.data_ptr(), nb
        ph, la, sa, na = self.structs()
        r = ct.byref
        if with_nm is None:  # the SH entry point itself
            rc = self.lib.nr_b200_forward_sh(r(a), r(ph), r(la), r(sa), None)
        else:
            rc = self.lib.nr_b200_forward_normal_map(r(a), r(ph), r(la), r(sa), r(na) if with_nm else None, None)
        assert rc == 0
        torch.cuda.synchronize()
        self.fwd_launches = self.lib.nr_b200_last_launch_count()
        return m

    def backward(self, flags, o, with_nm=True):
        ct, sc, L, m = self.ct, self.sc, self.L, self.maps
        B, F, S = sc.B, sc.F, sc.S
        nb = self.lib.nr_b200_backward_workspace_bytes(B, F, S, 0, self.flags)
        ws = torch.empty((nb,), dtype=torch.uint8, device=DEV)
        a = L.BackwardArgs()
        a.struct_size = ct.sizeof(L.BackwardArgs)
        a.flags = self.flags | flags
        a.batch_size, a.num_faces, a.raster_size, a.texture_size = B, F, S, 0
        a.eps = 1e-4
        a.faces, a.textures = sc.faces.data_ptr(), sc.tex.data_ptr()
        a.face_uvs, a.texture_height, a.texture_width = sc.uvs.data_ptr(), sc.tex.shape[1], sc.tex.shape[2]
        a.face_index_map, a.weight_map, a.depth_map, a.rgb_map = (m[k].data_ptr() for k in ("fim", "wmap", "dmap", "rgb"))
        a.grad_rgb, a.grad_alpha = self.g.data_ptr(), self.ga.data_ptr()
        p = lambda k: None if o.get(k) is None else o[k].data_ptr()
        a.grad_faces, a.grad_textures, a.grad_face_uvs = p("faces"), p("tex"), p("uvs")
        a.workspace, a.workspace_bytes = ws.data_ptr(), nb
        ph, la, sa, na = self.structs(o)
        r = ct.byref
        if with_nm is None:
            rc = self.lib.nr_b200_backward_sh(r(a), r(ph), r(la), r(sa), None)
        else:
            rc = self.lib.nr_b200_backward_normal_map(r(a), r(ph), r(la), r(sa), r(na) if with_nm else None, None)
        torch.cuda.synchronize()
        self.launches = self.lib.nr_b200_last_launch_count()
        return rc


def _guarded(shape, fill=float("nan")):
    """a buffer with 64 guard floats on either side, NaN-poisoned inside"""
    n = 1
    for d in shape:
        n *= d
    buf = torch.full((n + 128,), fill, device=DEV)
    buf[:64] = 7.0
    buf[-64:] = 7.0
    return buf, buf[64:64 + n].view(shape)


NEW = ("nm", "tg")
SHADING = ("cs", "prm", "lt", "sh", "nm", "tg", "uvs")


@pytest.mark.parametrize("Bm,Bt", [(2, 2), (1, 1), (1, 2)])
def test_abi_poison_guards_offsets_nulls_accumulate_and_two_halves(Bm, Bt):
    import abi_harness as H
    t = _AbiNM(Bm, Bt)
    L = t.L
    shapes = t.shapes()
    bufs = {k: _guarded(s) for k, s in shapes.items()}
    out = {k: v[1] for k, v in bufs.items()}
    assert t.backward(0, out) == 0
    for k, (buf, _) in bufs.items():
        assert bool((buf[:64] == 7).all() and (buf[-64:] == 7).all()), k
        assert bool(torch.isfinite(out[k]).all()), k
    ref = {k: v.clone() for k, v in out.items()}
    for k in NEW:
        assert float(ref[k].abs().max()) > 0, k
    assert float(ref["tg"][..., 3].abs().max()) == 0  # no gradient into w
    # buffers 4 and 8 bytes past a 16-byte boundary, between guard words
    for off in (4, 8):
        o = {k: H.alloc(s, np.float32, off, DEV) for k, s in shapes.items()}
        for v in o.values():
            H.poison(v)
        assert t.backward(0, o) == 0
        for k in o:
            assert H.guards_intact(o[k]), (off, k)
            assert rel_err(np_(o[k]), np_(ref[k])) <= 1e-5, (off, k)
    # every allowed NULL: the other outputs as before (fp32 atomics in another order)
    for drop in SHADING:
        o = {k: _guarded(s)[1] for k, s in shapes.items()}
        o[drop] = None
        assert t.backward(0, o) == 0
        for k in o:
            if o[k] is not None:
                assert rel_err(np_(o[k]), np_(ref[k])) <= 1e-5, (drop, k)
    # NR_GRAD_ACCUMULATE adds into what is there
    pre = {k: torch.rand(s, generator=torch.Generator().manual_seed(40)).to(DEV) for k, s in shapes.items()}
    acc = {k: v.clone() for k, v in pre.items()}
    assert t.backward(L.NR_GRAD_ACCUMULATE, acc) == 0
    for k in acc:
        assert rel_err(np_(acc[k] - pre[k]), np_(ref[k])) <= 1e-5, k
    # two halves: every shading output (the map's UV term included) comes from the texture half; the faces half alone
    # leaves them untouched
    o = {k: _guarded(s)[1] for k, s in shapes.items()}
    assert t.backward(L.NR_BWD_PART_FACES, o) == 0
    for k in SHADING + ("tex",):
        assert bool(torch.isnan(o[k]).all()), k
    faces_half = o["faces"].clone()
    assert t.backward(L.NR_BWD_PART_TEXTURES, o) == 0
    for k in o:
        assert rel_err(np_(o[k]), np_(ref[k])) <= 1e-5, k
    assert torch.equal(o["faces"], faces_half)
    assert t.backward(L.NR_GRAD_INTERIOR, out) == -4
    assert t.launches == 0


def test_abi_null_struct_is_the_sh_call():
    """a NULL nm through nr_b200_forward_normal_map / nr_b200_backward_normal_map: the maps of nr_b200_forward_sh bit for
    bit with the same launches, and the gradients of nr_b200_backward_sh (within fp32 atomics' order)"""
    t = _AbiNM()
    a = t.forward(with_nm=False)
    n_a = t.fwd_launches
    b = t.forward(with_nm=None)
    assert t.fwd_launches == n_a
    for k in a:
        assert torch.equal(a[k], b[k]), k
    assert not torch.equal(a["rgb"], t.maps["rgb"])  # the map does change the render
    t.maps = a
    shapes = {k: s for k, s in t.shapes().items() if k not in NEW}
    o1 = {k: _guarded(s)[1] for k, s in shapes.items()}
    o2 = {k: _guarded(s)[1] for k, s in shapes.items()}
    assert t.backward(0, o1, with_nm=False) == 0
    n1 = t.launches
    assert t.backward(0, o2, with_nm=None) == 0
    assert t.launches == n1
    for k in o1:
        assert bool(torch.isfinite(o1[k]).all()), k
        assert rel_err(np_(o1[k]), np_(o2[k])) <= 1e-6, k


# ------------------------------------------------------------------------------------------------ Renderer
def _grid(n=12, z=0.0):
    """a bumpy height field over [-0.7, 0.7]^2 with UVs = its xy mapped to [0,1]^2: vertices [1,Nv,3], faces [F,3], uvs"""
    xs = torch.linspace(-0.7, 0.7, n)
    X, Y = torch.meshgrid(xs, xs, indexing="xy")
    Z = z + 0.05 * torch.sin(3 * X) * torch.cos(2 * Y)
    v = torch.stack((X, Y, Z), -1).reshape(-1, 3)
    uv = torch.stack(((X + 0.7) / 1.4, (Y + 0.7) / 1.4), -1).reshape(-1, 2)
    f = []
    for i in range(n - 1):
        for j in range(n - 1):
            a, b, c, d = i * n + j, i * n + j + 1, (i + 1) * n + j + 1, (i + 1) * n + j
            f += [[a, c, b], [a, d, c]]
    f = torch.tensor(f, dtype=torch.int32)
    v, f = v[None].to(DEV), f[None].to(DEV)
    r = _renderer(False)
    if float(r.render_silhouettes(v, f).sum()) == 0:
        f = f.flip(2).contiguous()  # the other winding faces the camera
    return v, f, uv[f[0].long().cpu()].to(DEV)


def _renderer(fill_back):
    import neural_renderer_b200 as nr
    r = nr.Renderer()
    r.camera_mode = "look_at"
    r.image_size, r.shading, r.fill_back, r.anti_aliasing = 64, "phong", fill_back, False
    r.eye = [0.3, 0.2, -2.5]
    r.lights = []
    return r


@pytest.mark.parametrize("fill_back", [False, True])
def test_renderer_fused_vs_op_by_op(fill_back):
    v, f, uvs = _grid()
    v, f = v.expand(2, -1, -1).contiguous(), f.expand(2, -1, -1)  # the op-by-op path takes one index set per item
    tex = torch.rand((1, 16, 16, 3), generator=torch.Generator().manual_seed(1)).to(DEV)
    nm = _map(1, 16, 16, amp=0.3)
    g = torch.randn((2, 3, 64, 64), generator=torch.Generator().manual_seed(2)).to(DEV)
    res = {}
    for fused in (True, False):
        r = _renderer(fill_back)
        r.fused = fused
        m = nm.clone().requires_grad_(True)
        r.normal_map = m
        vv = v.clone().requires_grad_(True)
        img = r.render(vv, f, tex, face_uvs=uvs)
        (img * g).sum().backward()
        res[fused] = (img.detach(), vv.grad, m.grad)
    print("renderer", [rel_err(np_(a), np_(b)) for a, b in zip(res[True], res[False])])
    assert rel_err(np_(res[True][0]), np_(res[False][0])) <= 1e-5
    assert rel_err(np_(res[True][1]), np_(res[False][1])) <= 1e-4
    assert rel_err(np_(res[True][2]), np_(res[False][2])) <= 1e-5
    assert float(res[True][2].abs().max()) > 0


@pytest.mark.parametrize("per_item_uvs", [False, True])
def test_renderer_shared_mesh(per_item_uvs):
    """one mesh seen from two viewpoints (a stride-0 vertex batch and one index set): the fused path's shared corner
    set, with per-item UVs (item 1 mirrored in u, so its tangents differ) or shared ones, against op by op"""
    v, f, uvs = _grid()
    if per_item_uvs:
        uv2 = uvs.clone()
        uv2[..., 0] = 1 - uv2[..., 0]
        uvs = torch.stack((uvs, uv2))
    tex = torch.rand((1, 16, 16, 3), generator=torch.Generator().manual_seed(1)).to(DEV)
    nm = _map(1, 16, 16, amp=0.3)
    g = torch.randn((2, 3, 64, 64), generator=torch.Generator().manual_seed(2)).to(DEV)
    res = {}
    for fused in (True, False):
        r = _renderer(False)
        r.fused = fused
        r.eye = [0.0, 0.0, -2.5]
        m = nm.clone().requires_grad_(True)
        r.normal_map = m
        v0 = v.clone().requires_grad_(True)
        vv = v0.expand(2, -1, -1)
        img = r.render(vv, f if fused else f.expand(2, -1, -1), tex, face_uvs=uvs)
        (img * g).sum().backward()
        res[fused] = (img.detach(), v0.grad, m.grad)
    print("shared mesh", per_item_uvs, [rel_err(np_(a), np_(b)) for a, b in zip(res[True], res[False])])
    assert rel_err(np_(res[True][0]), np_(res[False][0])) <= 1e-5
    assert rel_err(np_(res[True][1]), np_(res[False][1])) <= 1e-4
    assert rel_err(np_(res[True][2]), np_(res[False][2])) <= 1e-5
    if per_item_uvs:  # the mirrored item's frame really differs: its image is not item 0's
        assert float((res[True][0][1] - res[True][0][0]).abs().max()) > 1e-3


def test_renderer_cuda_graph():
    v, f, uvs = _grid()
    tex = torch.rand((1, 16, 16, 3), generator=torch.Generator().manual_seed(1)).to(DEV)
    r = _renderer(False)
    m = _map(1, 16, 16, amp=0.3).requires_grad_(True)
    r.normal_map = m
    g = torch.randn((1, 3, 64, 64), generator=torch.Generator().manual_seed(2)).to(DEV)
    vv = v.clone().requires_grad_(True)

    def step():
        m.grad = None
        vv.grad = None
        (r.render(vv, f, tex, face_uvs=uvs) * g).sum().backward()
        return m.grad, vv.grad
    ref = [t.clone() for t in step()]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            step()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    m.grad = None
    vv.grad = None
    with torch.cuda.graph(graph):
        (r.render(vv, f, tex, face_uvs=uvs) * g).sum().backward()
    graph.replay()
    torch.cuda.synchronize()
    assert rel_err(np_(m.grad), np_(ref[0])) <= 1e-5
    assert rel_err(np_(vv.grad), np_(ref[1])) <= 1e-5


# ------------------------------------------------------------------------------------------------ photometric stereo
def test_photometric_stereo_recovers_a_map():
    """B = 4 views of one camera-facing quad, each under its own directional light (not coplanar, in front of every
    target normal), K = 0, a known white albedo: Adam from a flat map recovers the target map's directions"""
    H, Hm, Wm = 96, 6, 6
    faces, uvs, _, _ = _bump_quad(H)
    B = 4
    faces, uvs = faces.expand(B, -1, -1, -1).contiguous(), uvs.expand(B, -1, -1, -1).contiguous()
    cs = torch.zeros((1, 4, 3, 6), device=DEV)
    cs[..., 2] = -1.0
    cs[..., 3:5] = faces[:1, ..., :2]
    tg = torch.zeros((1, 4, 3, 4), device=DEV)
    tg[..., 0] = 1.0
    tg[..., 3] = -1.0  # with n = -z, b = -(n x t) = +y: the map's +y runs along +v
    tg[:, 2:] = -tg[:, 2:]
    dirs = torch.tensor([[0.0, 0.0, -1.0], [0.5, 0.0, -1.0], [0.0, 0.5, -1.0], [-0.4, -0.4, -1.0]])
    dirs = dirs / dirs.norm(dim=1, keepdim=True)
    prm = torch.zeros((B, 16))
    prm[:, 3:6] = 1.0
    prm[:, 6:9] = dirs
    prm[:, 12] = 1.0
    prm[:, 15] = -4.0
    prm = prm.to(DEV)
    gen = torch.Generator().manual_seed(11)
    target = torch.randn((1, Hm, Wm, 3), generator=gen) * 0.25
    target[..., 2] = 1.0
    target = (target / target.norm(dim=-1, keepdim=True)).to(DEV)
    tex = torch.ones((1, 4, 4, 3), device=DEV)

    def render(m):
        return _R()._run(faces, tex, H, False, 0.1, 100, 1e-4, (0, 0, 0), True, False, False, face_uvs=uvs,
                         corner_shading=cs, shading_params=prm, normal_map=m, corner_tangents=tg)[0]
    goal = render(target).detach()
    m = torch.zeros((1, Hm, Wm, 3), device=DEV)
    m[..., 2] = 1.0
    m.requires_grad_(True)
    opt = torch.optim.Adam([m], lr=0.02)
    for it in range(600):
        opt.zero_grad()
        loss = ((render(m) - goal) ** 2).mean()
        loss.backward()
        opt.step()
    a = m.detach() / m.detach().norm(dim=-1, keepdim=True)
    ang = torch.rad2deg(torch.acos((a * target).sum(-1).clamp(-1, 1)))
    # every item samples every texel: the quad covers the whole map in each view
    err = float(ang.mean())
    print("photometric stereo: mean angular error %.4f deg, loss %.3e" % (err, float(loss)))
    assert err < 1.0
