"""GPU: Phong shading through a specular map (include/nr_b200.h, nr_b200_specular_map_args),
rasterize(..., specular_map=), Renderer.specular_map and F.specular_map.

The forward is held to the float64 oracle of oracles_specular_map.py on the product's own maps, the backward to float64
autograd of the same oracle and to central differences of the product's forward.  A constant (1, 1, 1, sigma) map renders
as the call without it bit for bit, and a NULL struct is nr_b200_*_normal_map."""
import numpy as np

import pytest
import torch

from helpers import elem_err, np_, rel_err
from oracles_specular_map import sm_rgb64
from test_gpu_normal_map import (NM_CASES, _AbiNM, _bump_quad, _fwd_tol, _grid, _guarded, _inputs, _map, _renderer,
                                 _tangents)
from test_gpu_smooth import BG, Scene, _R

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda")
MODES = ["phong", "lights", "sh", "nm"]  # "nm": a normal map on top of the light set and the environment


def _smap(Bq, Hq, Wq, seed=51, sig=(1.0, 64.0)):
    """[Bq,Hq,Wq,4]: ks in [0.2, 1.4] per channel, shininess uniform in `sig`"""
    g = torch.Generator().manual_seed(seed)
    ks = 0.2 + 1.2 * torch.rand((Bq, Hq, Wq, 3), generator=g)
    s = sig[0] + (sig[1] - sig[0]) * torch.rand((Bq, Hq, Wq, 1), generator=g)
    return torch.cat((ks, s), -1).to(DEV).contiguous()


def _const(Bq, Hq, Wq, sigma):
    m = torch.ones((Bq, Hq, Wq, 4), device=DEV)
    m[..., 3] = sigma
    return m


def _mode_inputs(sc, mode, sigma):
    cs, prm, lt, sh = _inputs(sc, "both" if mode == "nm" else mode, sigma, sc.B)
    nm, tg = (_map(1, 9, 11), _tangents(sc.B, sc.F)) if mode == "nm" else (None, None)
    return cs, prm, lt, sh, nm, tg


def _render(sc, cs, prm, lt, sh, nm, tg, sm, tex=None, uvs=None):
    geom, verts = sc.faces, None
    if sc.indexed:
        verts = sc.faces.reshape(sc.B, -1, 3)
        geom = torch.arange(verts.shape[1], device=DEV, dtype=torch.int32).reshape(-1, 3)
    return _R()._run(geom, sc.tex if tex is None else tex, sc.H, sc.aa, 0.1, 100, 1e-4, BG, True, True, True,
                     textures_fill_back=sc.fill_back, vertices=verts, face_uvs=sc.uvs if uvs is None else uvs,
                     texture_filter=sc.tf, corner_shading=cs, shading_params=prm, lights=lt, environment_sh=sh,
                     normal_map=nm, corner_tangents=tg, specular_map=sm)


def _all_grads(sc, cs, prm, lt, sh, nm, tg, sm, g):
    leaves = {"cs": cs, "prm": prm, "lt": lt, "sh": sh, "nm": nm, "tg": tg, "sm": sm, "tex": sc.tex, "uvs": sc.uvs}
    leaves = {k: (v.detach().clone().requires_grad_(True) if v is not None else None) for k, v in leaves.items()}
    out = _render(sc, *(leaves[k] for k in ("cs", "prm", "lt", "sh", "nm", "tg", "sm")), tex=leaves["tex"],
                  uvs=leaves["uvs"])
    (out[0] * g).sum().backward()
    return out, {k: v.grad for k, v in leaves.items() if v is not None}


# ------------------------------------------------------------------------------------------------ identity
@pytest.mark.parametrize("case", NM_CASES)
@pytest.mark.parametrize("mode", MODES)
def test_constant_map_is_the_call_without_it(case, mode):
    """(1, 1, 1, sigma of params): rgb / alpha / depth bit for bit, every shared gradient within the spread of two
    identical calls, grad_params[12] = 0, and the map's gradient sums to what K, K_j and sigma received without it"""
    kind, aa, fill_back, indexed = case
    sc = Scene(kind, aa, fill_back, indexed)
    sigma = 16.0
    cs, prm, lt, sh, nm, tg = _mode_inputs(sc, mode, sigma)
    sm = _const(1, 5, 7, sigma)
    g = torch.randn((sc.B, 3, sc.H, sc.H), generator=torch.Generator().manual_seed(5)).to(DEV)
    o_sm, g_sm = _all_grads(sc, cs, prm, lt, sh, nm, tg, sm, g)
    o_0, g_0 = _all_grads(sc, cs, prm, lt, sh, nm, tg, None, g)
    # the spread of fp32 atomics in another order: the largest difference among three identical calls
    g_rep = [g_0] + [_all_grads(sc, cs, prm, lt, sh, nm, tg, None, g)[1] for _ in range(2)]
    for a, b in zip(o_sm[:3], o_0[:3]):
        assert torch.equal(a, b)
    for k, v in g_0.items():
        cut = (lambda t: t[:, :12]) if k == "prm" else (lambda t: t)
        a, reps = cut(g_sm[k]), [cut(r[k]) for r in g_rep]
        spread = max(float((x - y).abs().max()) for i, x in enumerate(reps) for y in reps[i + 1:])
        err = float((a - reps[0]).abs().max())
        print("const", case, mode, k, err, spread)
        assert err <= max(2 * spread, 2e-6 * float(reps[0].abs().max())), k
    assert float(g_sm["prm"][:, 12].abs().max()) == 0
    gm = g_sm["sm"].double().sum(dim=(0, 1, 2))
    want = [(prm[:, 9 + c].double() * g_0["prm"][:, 9 + c].double()).sum() for c in range(3)]
    if lt is not None:
        want = [w + (lt[..., 3 + c].double() * g_0["lt"][..., 3 + c].double()).sum() for c, w in enumerate(want)]
    want.append(g_0["prm"][:, 12].double().sum())
    for c in range(4):
        print("sums", case, mode, c, float(gm[c]), float(want[c]))
        assert abs(float(gm[c] - want[c])) <= 1e-5 * abs(float(want[c])) + 1e-7, c
    assert abs(float(want[3])) > 0 and abs(float(want[0])) > 0


# ------------------------------------------------------------------------------------------------ forward vs float64
@pytest.mark.parametrize("case", NM_CASES)
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("hw", [(1, 1), (1, 23), (37, 53)])
def test_forward_vs_oracle(case, mode, hw):
    kind, aa, fill_back, indexed = case
    sc = Scene(kind, aa, fill_back, indexed)
    fim, wmap, dmap = sc.maps()
    unlit = sc.unlit64(fim, wmap, dmap)
    cs, prm, lt, sh, nm, tg = _mode_inputs(sc, mode, 16.0)
    for Bq in (1, sc.B):
        for sig in ((1.0, 1.0), (1.0, 64.0)):
            sm = _smap(Bq, *hw, sig=sig)
            rgb = _render(sc, cs, prm, lt, sh, nm, tg, sm)[0]
            want = sm_rgb64(sc.faces, fim, wmap, dmap, cs, prm, lt, sh, nm, tg, sm, sc.uvs, unlit, BG, aa, fill_back)
            err = rel_err(np_(rgb), np_(want))
            print("sm fwd", case, mode, hw, Bq, sig, err)
            assert err <= _fwd_tol(kind, sig[1])


@pytest.mark.parametrize("kind,H", [("bilinear", 257), ("trilinear", 1100)])
def test_forward_vs_oracle_large_and_odd_rasters(kind, H):
    sc = Scene(kind, False, False, False, H=H, F=2000, B=1)
    cs, prm, lt, sh, nm, tg = _mode_inputs(sc, "nm", 16.0)
    sm = _smap(1, 37, 53)
    rgb = _render(sc, cs, prm, lt, sh, nm, tg, sm)[0]
    fim, wmap, dmap = sc.maps()
    want = sm_rgb64(sc.faces, fim, wmap, dmap, cs, prm, lt, sh, nm, tg, sm, sc.uvs, sc.unlit64(fim, wmap, dmap), BG,
                    False, False)
    print("sm fwd large", kind, H, rel_err(np_(rgb), np_(want)))
    assert rel_err(np_(rgb), np_(want)) <= _fwd_tol(kind, 64.0)


# ------------------------------------------------------------------------------------------------ exact split
def test_exact_split():
    """a camera-facing quad whose map is (0, 0, 0, .) on the left half and (1, 1, 1, sigma0) on the right: away from the
    seam, the left equals the K = 0 render and the right the render without a map at shininess sigma0, bit for bit"""
    H, sigma0 = 128, 24.0
    faces, uvs, _, _ = _bump_quad(H)
    cs = torch.zeros((1, 4, 3, 6), device=DEV)
    cs[..., 2] = -1.0
    cs[..., 3:5] = faces[..., :2]
    prm = torch.tensor([[0.1, 0.1, 0.1, 0.5, 0.5, 0.5, 0.2, 0.1, -1.0, 0.8, 0.7, 0.6, 5.0, 0.1, 0.0, -4.0]], device=DEV)
    lt = torch.tensor([[[0.2, 0.2, 0.2, 0.5, 0.6, 0.7, -0.4, 0.3, -1.5, 0.2, 1.0, 0.0]]], device=DEV)
    tex = torch.rand((1, 8, 8, 3), generator=torch.Generator().manual_seed(3)).to(DEV)
    Wq = 64
    sm = torch.zeros((1, 4, Wq, 4), device=DEV)
    sm[:, :, Wq // 2:, :3] = 1.0
    sm[..., 3] = sigma0
    sm[:, :, : Wq // 2, 3] = 3.0  # read, but multiplied by ks = 0

    def render(prm_, lt_, sm_):
        return _R()._run(faces, tex, H, False, 0.1, 100, 1e-4, (0, 0, 0), True, False, False, face_uvs=uvs,
                         corner_shading=cs, shading_params=prm_, lights=lt_, specular_map=sm_)[0][0]
    img = render(prm, lt, sm)
    p0, l0 = prm.clone(), lt.clone()
    p0[:, 9:12] = 0.0
    l0[..., 3:6] = 0.0
    left_ref = render(p0, l0, None)
    p1 = prm.clone()
    p1[:, 12] = sigma0
    right_ref = render(p1, lt, None)
    xs = (2 * torch.arange(H, dtype=torch.float64) + 1 - H) / H
    u = (xs + 0.95) / 1.9
    cols_l = ((u > 0.03) & (u < 0.5 - 2.0 / (Wq - 1))).nonzero().flatten()
    cols_r = ((u > 0.5 + 2.0 / (Wq - 1)) & (u < 0.97)).nonzero().flatten()
    rows = slice(8, H - 8)
    assert torch.equal(img[:, rows][:, :, cols_l], left_ref[:, rows][:, :, cols_l])
    assert torch.equal(img[:, rows][:, :, cols_r], right_ref[:, rows][:, :, cols_r])
    # the right half really has a highlight the left lacks
    assert float((right_ref - left_ref)[:, rows][:, :, cols_r].max()) > 1e-2


# ------------------------------------------------------------------------------------------------ gradients
@pytest.mark.parametrize("case", [("bilinear", False, False, True), ("bilinear", True, True, False),
                                  ("trilinear", False, True, True), ("trilinear", True, False, False)])
@pytest.mark.parametrize("mode", ["phong", "lights", "nm"])
def test_gradients_vs_float64(case, mode):
    kind, aa, fill_back, indexed = case
    sc = Scene(kind, aa, fill_back, indexed)
    cs, prm, lt, sh, nm, tg = _mode_inputs(sc, mode, 16.0)
    sm = _smap(1, 9, 11, sig=(2.0, 16.0))  # up to the shininess the Phong gradient gates were set at
    g = torch.randn((sc.B, 3, sc.H, sc.H), generator=torch.Generator().manual_seed(7)).to(DEV)
    _, got = _all_grads(sc, cs, prm, lt, sh, nm, tg, sm, g)
    fim, wmap, dmap = sc.maps()
    ref = {k: v.detach().double().clone().requires_grad_(True) for k, v in
           {"cs": cs, "prm": prm, "lt": lt, "sh": sh, "nm": nm, "tg": tg, "sm": sm, "tex": sc.tex,
            "uvs": sc.uvs}.items() if v is not None}
    unlit = sc.unlit64(fim, wmap, dmap, tex=ref["tex"], uvs=ref["uvs"], uv_grad=True)
    want = sm_rgb64(sc.faces, fim, wmap, dmap, ref["cs"], ref["prm"], ref.get("lt"), ref.get("sh"), ref.get("nm"),
                    ref.get("tg"), ref["sm"], ref["uvs"], unlit, BG, aa, fill_back)
    (want * g.double()).sum().backward()
    for k, r in ref.items():
        err = rel_err(np_(got[k]), np_(r.grad))
        print("sm grad", case, mode, k, err, elem_err(np_(got[k]), np_(r.grad)))
        assert err <= 1e-4, k
    assert float(got["prm"][:, 12].abs().max()) == 0
    # the per-element gates of test_gpu_phong.py / test_gpu_normal_map.py
    assert elem_err(np_(got["cs"]), np_(ref["cs"].grad)) <= 2e-3
    assert elem_err(np_(got["prm"]), np_(ref["prm"].grad)) <= 5e-4
    if lt is not None:
        assert elem_err(np_(got["lt"]), np_(ref["lt"].grad)) <= 2e-4


def test_central_differences():
    """the product's own forward, stepped in ks texels, shininess texels and UV corners, against its gradient"""
    sc = Scene("bilinear", False, False, False, B=1)
    cs, prm, lt, sh, nm, tg = _mode_inputs(sc, "lights", 4.0)
    sm = _smap(1, 5, 6, sig=(2.0, 8.0))
    g = torch.randn((1, 3, sc.H, sc.H), generator=torch.Generator().manual_seed(9)).to(DEV)
    _, got = _all_grads(sc, cs, prm, lt, sh, nm, tg, sm, g)
    fim = sc.maps()[0]
    f0 = int(fim[fim >= 0].flatten().mode().values)  # a face that covers pixels

    def loss(sm_, uvs_):
        return float((_render(sc, cs, prm, lt, sh, nm, tg, sm_, uvs=uvs_)[0].double() * g.double()).sum())
    checks = [("sm", (0, 2, 3, 0)), ("sm", (0, 1, 2, 1)), ("sm", (0, 3, 4, 2)), ("sm", (0, 2, 2, 3)),
              ("sm", (0, 1, 4, 3)), ("uvs", (0, f0, 1, 0)), ("uvs", (0, f0, 2, 1))]
    for name, idx in checks:
        h = {"sm": 1e-2, "uvs": 1e-4}[name]
        base = {"sm": sm, "uvs": sc.uvs}
        p, m = base[name].clone(), base[name].clone()
        p[idx] += h
        m[idx] -= h
        args = lambda t: [t if k == name else base[k] for k in ("sm", "uvs")]
        num = (loss(*args(p)) - loss(*args(m))) / (2 * h)
        ana = float(got[name][idx])
        print("cd", name, idx, num, ana)
        assert abs(num - ana) <= 0.02 * abs(ana) + 1e-3
    assert float(got["sm"][..., :3].abs().max()) > 0 and float(got["sm"][..., 3].abs().max()) > 0


# ------------------------------------------------------------------------------------------------ direct ABI calls
class _SmLib:
    """the library with the normal-map entry points routed through the specular-map ones, so that _AbiNM's calls carry
    the owner's specular map (owner.with_sm False: a NULL sm)"""

    def __init__(self, lib, owner):
        self.lib, self.owner = lib, owner

    def __getattr__(self, name):
        return getattr(self.lib, name)

    def nr_b200_forward_normal_map(self, a, ph, la, sa, na, stream):
        return self.lib.nr_b200_forward_specular_map(a, ph, la, sa, na, self.owner.qa(), stream)

    def nr_b200_backward_normal_map(self, a, ph, la, sa, na, stream):
        return self.lib.nr_b200_backward_specular_map(a, ph, la, sa, na, self.owner.qa(), stream)


class _AbiSM(_AbiNM):
    """_AbiNM's normal-mapped render (light set, SH, anti-aliasing, fill_back) through a specular map as well"""

    def __init__(self, Bq=2, Bm=2, Bt=2):
        from neural_renderer_b200 import _lib
        self.sm = _smap(Bq, 7, 10, sig=(2.0, 24.0))
        self.with_sm, self.o = True, {}
        self.raw = _lib.load()
        self._lib = _SmLib(self.raw, self)
        super().__init__(Bm, Bt)

    @property
    def lib(self):
        return self._lib

    @lib.setter
    def lib(self, _):  # _AbiNM.__init__ assigns the plain library
        pass

    def shapes(self):
        s = super().shapes()
        s["sm"] = tuple(self.sm.shape)
        return s

    def structs(self, o=None):
        self.o = o or {}
        return super().structs(o)

    def qa(self):
        if not self.with_sm:
            return None
        L = self.L
        qa = L.SpecularMapArgs()
        qa.struct_size = self.ct.sizeof(L.SpecularMapArgs)
        qa.map_batch, qa.map_height, qa.map_width = self.sm.shape[:3]
        qa.specular_map = self.sm.data_ptr()
        qa.grad_specular_map = None if self.o.get("sm") is None else self.o["sm"].data_ptr()
        return self.ct.byref(qa)


SHADING = ("cs", "prm", "lt", "sh", "nm", "tg", "sm", "uvs")


@pytest.mark.parametrize("Bq", [2, 1])
def test_abi_poison_guards_offsets_nulls_accumulate_and_two_halves(Bq):
    import abi_harness as H
    t = _AbiSM(Bq)
    L = t.L
    shapes = t.shapes()
    bufs = {k: _guarded(s) for k, s in shapes.items()}
    out = {k: v[1] for k, v in bufs.items()}
    assert t.backward(0, out) == 0
    for k, (buf, _) in bufs.items():
        assert bool((buf[:64] == 7).all() and (buf[-64:] == 7).all()), k
        assert bool(torch.isfinite(out[k]).all()), k
    ref = {k: v.clone() for k, v in out.items()}
    assert float(ref["sm"][..., :3].abs().max()) > 0 and float(ref["sm"][..., 3].abs().max()) > 0
    assert float(ref["prm"][:, 12].abs().max()) == 0
    # buffers 0, 4 and 8 bytes past a 16-byte boundary, between guard words
    for off in (0, 4, 8):
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
    # NR_GRAD_ACCUMULATE adds exactly one call into what is there
    pre = {k: torch.rand(s, generator=torch.Generator().manual_seed(40)).to(DEV) for k, s in shapes.items()}
    acc = {k: v.clone() for k, v in pre.items()}
    assert t.backward(L.NR_GRAD_ACCUMULATE, acc) == 0
    for k in acc:
        assert rel_err(np_(acc[k] - pre[k]), np_(ref[k])) <= 1e-5, k
    # two halves: the faces half alone leaves the map gradient untouched, the texture half completes it
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


def test_abi_null_struct_is_the_normal_map_call():
    """a NULL sm through nr_b200_forward_specular_map / nr_b200_backward_specular_map: the maps of
    nr_b200_forward_normal_map bit for bit with the same launches, and the gradients of nr_b200_backward_normal_map"""
    t = _AbiSM()
    with_map = t.maps
    t.with_sm = False
    a = t.forward()
    n_a = t.fwd_launches
    t._lib = t.raw  # the normal-map entry points themselves
    b = t.forward()
    assert t.fwd_launches == n_a
    for k in a:
        assert torch.equal(a[k], b[k]), k
    assert not torch.equal(a["rgb"], with_map["rgb"])  # the map does change the render
    t.maps = a
    shapes = {k: s for k, s in t.shapes().items() if k != "sm"}
    o1 = {k: _guarded(s)[1] for k, s in shapes.items()}
    o2 = {k: _guarded(s)[1] for k, s in shapes.items()}
    t._lib = _SmLib(t.raw, t)
    assert t.backward(0, o1) == 0
    n1 = t.launches
    t._lib = t.raw
    assert t.backward(0, o2) == 0
    assert t.launches == n1
    for k in o1:
        assert bool(torch.isfinite(o1[k]).all()), k
        assert rel_err(np_(o1[k]), np_(o2[k])) <= 1e-6, k


# ------------------------------------------------------------------------------------------------ Renderer
@pytest.mark.parametrize("fill_back", [False, True])
def test_renderer_fused_vs_op_by_op(fill_back):
    v, f, uvs = _grid()
    v, f = v.expand(2, -1, -1).contiguous(), f.expand(2, -1, -1)  # the op-by-op path takes one index set per item
    tex = torch.rand((1, 16, 16, 3), generator=torch.Generator().manual_seed(1)).to(DEV)
    sm = _smap(1, 16, 16, sig=(4.0, 32.0))
    g = torch.randn((2, 3, 64, 64), generator=torch.Generator().manual_seed(2)).to(DEV)
    res = {}
    for fused in (True, False):
        r = _renderer(fill_back)
        r.fused = fused
        m = sm.clone().requires_grad_(True)
        r.specular_map = m
        vv = v.clone().requires_grad_(True)
        img = r.render(vv, f, tex, face_uvs=uvs)
        (img * g).sum().backward()
        res[fused] = (img.detach(), vv.grad, m.grad)
    print("renderer", [rel_err(np_(a), np_(b)) for a, b in zip(res[True], res[False])])
    assert rel_err(np_(res[True][0]), np_(res[False][0])) <= 1e-5
    assert rel_err(np_(res[True][1]), np_(res[False][1])) <= 1e-4
    assert rel_err(np_(res[True][2]), np_(res[False][2])) <= 1e-5
    assert float(res[True][2][..., :3].abs().max()) > 0 and float(res[True][2][..., 3].abs().max()) > 0


def test_renderer_shared_mesh():
    """one mesh seen from two viewpoints (a stride-0 vertex batch and one index set) with a shared specular map and a
    normal map, fused against op by op"""
    v, f, uvs = _grid()
    tex = torch.rand((1, 16, 16, 3), generator=torch.Generator().manual_seed(1)).to(DEV)
    sm = _smap(1, 16, 16, sig=(4.0, 32.0))
    nm = _map(1, 16, 16, amp=0.3)
    g = torch.randn((2, 3, 64, 64), generator=torch.Generator().manual_seed(2)).to(DEV)
    res = {}
    for fused in (True, False):
        r = _renderer(False)
        r.fused = fused
        r.eye = [0.0, 0.0, -2.5]
        m = sm.clone().requires_grad_(True)
        r.specular_map, r.normal_map = m, nm
        v0 = v.clone().requires_grad_(True)
        img = r.render(v0.expand(2, -1, -1), f if fused else f.expand(2, -1, -1), tex, face_uvs=uvs)
        (img * g).sum().backward()
        res[fused] = (img.detach(), v0.grad, m.grad)
    print("shared mesh", [rel_err(np_(a), np_(b)) for a, b in zip(res[True], res[False])])
    assert rel_err(np_(res[True][0]), np_(res[False][0])) <= 1e-5
    assert rel_err(np_(res[True][1]), np_(res[False][1])) <= 1e-4
    assert rel_err(np_(res[True][2]), np_(res[False][2])) <= 1e-5


def test_renderer_cuda_graph():
    v, f, uvs = _grid()
    tex = torch.rand((1, 16, 16, 3), generator=torch.Generator().manual_seed(1)).to(DEV)
    r = _renderer(False)
    m = _smap(1, 16, 16, sig=(4.0, 32.0)).requires_grad_(True)
    r.specular_map = m
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


# ------------------------------------------------------------------------------------------------ fit
def test_fit_recovers_two_materials():
    """a quad with a 4x4 map of two materials (ks 0.2 / 0.9, shininess 8 / 32 in a checkerboard), seen from 4 eyes under
    4 point lights so that every texel carries a highlight, known albedo: Adam from a constant map, the shininess through
    exp, recovers ks and the shininess"""
    from neural_renderer_b200 import functional as F
    H, B = 96, 4
    faces, uvs, _, _ = _bump_quad(H)
    faces, uvs = faces.expand(B, -1, -1, -1).contiguous(), uvs.expand(B, -1, -1, -1).contiguous()
    cs = torch.zeros((1, 4, 3, 6), device=DEV)
    cs[..., 2] = -1.0
    cs[..., 3:5] = faces[:1, ..., :2]
    prm = torch.zeros((B, 16))
    prm[:, 0:3] = 0.2
    prm[:, 3:6] = 0.3
    prm[:, 6:9] = torch.tensor([0.0, 0.0, -1.0])
    prm[:, 9:12] = 0.0  # params' own light: diffuse only
    prm[:, 12] = 1.0
    eyes = torch.tensor([[0.0, 0.0, -3.0], [0.9, 0.5, -3.0], [-0.6, 0.8, -3.0], [-0.5, -0.9, -3.0]])
    prm[:, 13:16] = eyes
    prm = prm.to(DEV)
    lt = []
    for (x, y) in ((-0.5, -0.5), (0.5, -0.5), (-0.5, 0.5), (0.5, 0.5)):
        lt.append([0.1, 0.1, 0.1, 1.0, 1.0, 1.0, x, y, -1.5, 0.0, 1.0, 0.0])
    lt = torch.tensor([lt], device=DEV)
    tex = torch.full((1, 4, 4, 3), 0.5, device=DEV)
    chk = (torch.arange(4)[:, None] + torch.arange(4)[None, :]) % 2 == 0
    ks_t = torch.where(chk, 0.2, 0.9)[None, ..., None].expand(1, 4, 4, 3).to(DEV)
    sig_t = torch.where(chk, 8.0, 32.0)[None].to(DEV)

    def render(ks, sig):
        return _R()._run(faces, tex, H, False, 0.1, 100, 1e-4, (0, 0, 0), True, False, False, face_uvs=uvs,
                         corner_shading=cs, shading_params=prm, lights=lt, specular_map=F.specular_map(ks, sig))[0]
    goal = render(ks_t, sig_t).detach()
    ks = torch.full((1, 4, 4, 3), 0.5, device=DEV, requires_grad=True)
    log_sig = torch.full((1, 4, 4), float(np.log(16.0)), device=DEV, requires_grad=True)
    opt = torch.optim.Adam([ks, log_sig], lr=0.03)
    loss0 = float(((render(ks, log_sig.exp()) - goal) ** 2).mean())
    for it in range(1500):
        opt.zero_grad()
        loss = ((render(ks, log_sig.exp()) - goal) ** 2).mean()
        loss.backward()
        opt.step()
    loss = float(((render(ks, log_sig.exp()) - goal) ** 2).mean())
    ks_err = float((ks.detach() - ks_t).abs().mean())
    sig_err = float(((log_sig.detach().exp() - sig_t).abs() / sig_t).mean())
    print("fit: loss %.3e -> %.3e (x%.0f), mean |ks| error %.4f, mean relative shininess error %.4f"
          % (loss0, loss, loss0 / max(loss, 1e-30), ks_err, sig_err))
    assert loss0 / loss >= 100
    assert ks_err < 0.02
    assert sig_err < 0.05
