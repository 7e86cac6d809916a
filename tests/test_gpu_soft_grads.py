"""GPU: every soft render's backward -- the silhouettes, the RGB through cubes and through a texture image, the attribute
images and soft depth -- against float64 autograd at the kernels' own selection, each gradient component held to its
own maximum.

Method.  Each test renders the fragments of its geometry at K 32 with the same S, sigma, near and far
(rasterize_soft_fragments makes every soft kernel's fp32 cut-off decision with the same device test on the same face
records), and evaluates the float64 oracles restricted to that selection (tests/soft_selection.py).  The cut-off is then
no source of disagreement.  The upstream gradient is zero at:
  - full pixels (32 fragments), where the fragments are not the whole aggregated set;
  - band pixels, where a selected pair lies within its fp32 error of a remaining discontinuity of the gradient: the
    clamp of the barycentrics at 0 or 1, a tie of the nearest edge between edges whose nearest points differ, and the
    texel cell or the clamp of the sampled coordinate (soft_selection.band_pixels derives each band).
Every test asserts that the scene has no zero-area face and no face outside [near, far] (so every zp is finite), that
every pixel carrying upstream gradient has fewer than 32 fragments, that the band pixels are at most 1 % of the checked
pixels, and that the z components' maximum is at least 1e-3 of the x/y maximum (the faces' depths lie a few
(far - near) gamma apart, so the softmax weights at overlaps are mixed).  The forward is checked at the same selection
under tests/test_gpu_soft_scale.py's gates, at the cut-off band pixels too.

Gates, per component (x/y and z of the geometry separately; textures, face_light, face_uvs, the image with the
pyramid's gradient collapsed into it, attributes): elem_err(floor 1e-3) <= 2e-3, the gate of the fragment and blend
tests, except at sigma 1e-5 and at gamma 1e-4, where the gate is elem_err(floor 1e-3) <= 1e-2 (GATE_LOOSE).  That
gate was set from measurement, not derived as a bound.  Per pixel and face the fp32 error is about 1e-3 of the term:
x = d^2 / sigma carries 2 d delta / sigma, delta = 4 eps |v| (eps = 2^-23), which is 2 sqrt(9.2 / sigma) delta, about
1.1e-3 at the cut-off at sigma 1e-5; the depth softmax's exponent carries dzp / ((far - near) gamma), dzp = 8 eps zp +
3 dl zp^2 / min z (dl = 8 eps |e| (|e| + d) / |A|), about 1e-3 at gamma 1e-4.  A component sums such terms over its
pixels with upstream gradients of either sign, so where it cancels to near the floor its error relative to itself is a
multiple of that, which no per-pixel bound fixes; the worst measured is 0.71 of 1e-2.

The cut-off itself is tested by a constructed scene (test_cutoff_pairs_decided_by_the_kernels): horizontal edges at
fp32 offsets from a row of pixel centres searched so that soft_eval's fp32 test keeps pairs the float64 test drops
(soft_selection.cutoff_edges); the test asserts at least 50 such pairs in the fragments and runs the forward and
gradient checks there, so a fragment selection that drifted from the soft kernels' cut-off test fails it.

Measured on an H100 80GB HBM3 at a 700 W power limit, one run: worst elem_err / gate over the components, per test
(the tests print it with -s, with the band and checked pixel counts).
  test_silhouettes        [64-1e-05] 0.07  [64-0.0001] 0.17  [64-0.001] 0.11
                          [127-1e-05] 0.20  [127-0.0001] 0.20  [127-0.001] 0.12
  test_cubes              [2-False-False] 0.16  [2-False-True] 0.33  [2-True-False] 0.03  [2-True-True] 0.22
                          [4-False-False] 0.14  [4-False-True] 0.27  [4-True-False] 0.04  [4-True-True] 0.71
  test_cubes_upstream     [rgb] 0.27  [alpha] 0.12  [both] 0.27
  test_uv                 [False-False] 0.44  [False-True] 0.50  [True-False] 0.26  [True-True] 0.24
  test_attributes         [False-1] 0.19  [False-3] 0.21  [False-5] 0.05  [True-1] 0.22  [True-3] 0.26  [True-5] 0.24
  test_soft_depth 0.29    test_teapot_shared_indices [sil] 0.02  [cube] 0.45  [attr] 0.15
  test_per_item_indices   [cube] 0.19  [attr] 0.25        test_deep_tiles [sil] 0.02  [cube] 0.02
  test_benchmark_spheres  [sil] 0.03  [cube] 0.16  [uv] 0.07
  test_cutoff_pairs_decided_by_the_kernels  [sil] 0.02  [cube] 0.01  [uv] 0.14  [attr] 0.02  (192 cut-off pairs)
Band pixels: at most 0.92 % of the checked pixels.  The file ran in about 25 s."""
import math
import os

import numpy as np
import pytest
import torch

import oracles_soft as osoft
import oracles_soft_attr as oattr
import oracles_soft_frag as ofrag
import oracles_soft_rgb as orgb
import soft_binning as sb
import soft_selection as ss
from helpers import elem_err
from test_gpu_soft_scale import (FAR, NEAR, Scene, _bench_tiles, _deep_faces, _image, _tile_pixels,
                                 check_forward)

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
PEAK_LIMIT = int(2.2 * 2 ** 30)
K = 32
GATE = 2e-3
GATE_LOOSE = 1e-2
FLOOR = 1e-3
BAND_MAX = 0.01


def _nr():
    import neural_renderer_b200 as nr
    return nr


@pytest.fixture(autouse=True)
def _peak_memory():
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats(DEV)
    yield
    torch.cuda.synchronize()
    assert torch.cuda.max_memory_allocated(DEV) <= PEAK_LIMIT, torch.cuda.max_memory_allocated(DEV)


def _rand(shape, seed, lo=0.0, hi=1.0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return lo + (hi - lo) * torch.rand(*shape, device=DEV, generator=g)


# ------------------------------------------------------------------------------------------------ scenes
class Sel(Scene):
    """a Scene (test_gpu_soft_scale.Scene: 'sil', 'cube', 'uv') or kind 'attr' (tex = attributes: per corner
    [1|B,F,3,C], or per vertex [1|B,Nv,C] with indexed geometry), with optional indexed geometry: verts [B,Nv,3] and
    idx [F,3] / [B,F,3]; self.faces is always the gathered faces [B,F,3,3]"""

    def __init__(self, kind, faces, verts=None, idx=None, **kw):
        super().__init__(kind, faces, **kw)
        self.verts, self.idx = verts, idx

    def geometry(self, g=None):
        """(faces argument, vertices argument) of the renders, with the geometry leaf g"""
        if self.verts is None:
            return (self.faces if g is None else g), None
        return self.idx, (self.verts if g is None else g)

    def leaves(self):
        if self.kind != "attr":
            out = super().leaves()
            return out if self.verts is None else [self.verts] + out[1:]
        return [self.faces if self.verts is None else self.verts, self.tex]

    def names(self):
        out = ["faces" if self.verts is None else "vertices"]
        if self.kind == "attr":
            return out + ["attributes"]
        if self.kind != "sil":
            out.append("image" if self.kind == "uv" else "textures")
            if self.kind == "uv":
                out.append("face_uvs")
            if self.light is not None:
                out.append("face_light")
        return out

    def render_leaves(self, S, sigma, gamma, leaves):
        nr = _nr()
        faces, vertices = self.geometry(leaves[0])
        if self.kind == "attr":
            kw = dict(vertex_attributes=leaves[1]) if self.tex.dim() == 3 else dict(face_attributes=leaves[1])
            out, alpha = nr.rasterize_soft_attributes(faces, S, sigma, gamma, NEAR, FAR, vertices=vertices,
                                                      background=list(self.bg), return_alpha=True, **kw)
            return out, alpha
        kw = {"faces": faces, "vertices": vertices}
        if self.kind != "sil":
            kw["tex"] = leaves[1]
            if self.kind == "uv":
                kw["uvs"] = leaves[2]
            if self.light is not None:
                kw["light"] = leaves[-1]
        return self.render(S, sigma, gamma, **kw)

    def fragments(self, S, sigma):
        faces, vertices = self.geometry()
        return _nr().rasterize_soft_fragments(faces, S, sigma, K, NEAR, FAR, vertices=vertices)

    def corner_attrs(self, attrs, b0=0, b1=None):
        """per-corner attributes of the attribute leaf (gathered through idx for per-vertex ones), items b0:b1"""
        if attrs.dim() == 4:
            return attrs
        idx = self.idx if self.idx.dim() == 2 or self.idx.shape[0] == 1 else self.idx[b0:b1]
        return oattr.corner_attributes(attrs, idx)

    def flat(self):
        """the same render as a Scene over materialised faces (and per-corner attributes): the oracle's view"""
        if self.kind != "attr":
            return Scene(self.kind, self.faces, tex=self.tex, uvs=self.uvs, light=self.light, tri=self.tri, bg=self.bg)
        return ss.AttrScene(self.faces, self.corner_attrs(self.tex), self.bg, NEAR, FAR)


def _z_range(gamma, gaps=4.0):
    """depths a few (far - near) gamma apart: mixed softmax weights where faces overlap"""
    return (2.0, 2.0 + gaps * (FAR - NEAR) * gamma)


def _soup(B, F, seed, gamma, size=(0.06, 0.3)):
    """[B,F,3,3] well-shaped triangles (corners about 120 degrees apart around random centres: the fp32 barycentrics'
    error |e|^2 / |A| stays small, and with it every band), corner depths spread over a few (far - near) gamma"""
    rng = np.random.default_rng(seed)
    c = rng.uniform(-0.85, 0.85, (B, F, 1, 2))
    r = rng.uniform(size[0], size[1], (B, F, 1, 1))
    ang = rng.uniform(0, 2 * np.pi, (B, F, 1, 1)) + np.array([0.0, 2.1, 4.2])[None, None, :, None] \
        + rng.uniform(-0.3, 0.3, (B, F, 3, 1))
    z0, z1 = _z_range(gamma)
    z = rng.uniform(z0, z1, (B, F, 3, 1))
    xy = c + r * np.concatenate((np.cos(ang), np.sin(ang)), -1)
    return torch.from_numpy(np.concatenate((xy, z), -1).astype(np.float32)).to(DEV)


def _teapot(B, gamma, seed):
    """[B,Nv,3] screen-space teapots (each item turned differently about the vertical axis) and faces [F,3]: the
    faces whose doubled area is at least 1e-4 in every item (edge-on slivers carry fp32 barycentrics no fixed gate
    bounds; tests/test_gpu_soft_scale.py's slivers test covers them)"""
    d = np.load(os.path.join(os.path.dirname(__file__), "golden", "teapot.npz"))
    v = torch.from_numpy(d["vertices"].astype(np.float64))
    f = torch.from_numpy(d["faces"].astype(np.int64))
    out = []
    for b in range(B):
        a = 0.6 + 0.9 * b + 0.1 * seed
        rot = torch.tensor([[math.cos(a), 0, math.sin(a)], [0, 1, 0], [-math.sin(a), 0, math.cos(a)]], dtype=torch.float64)
        tilt = torch.tensor([[1, 0, 0], [0, math.cos(0.4), -math.sin(0.4)], [0, math.sin(0.4), math.cos(0.4)]],
                            dtype=torch.float64)
        w = v @ rot.T @ tilt.T
        z0, z1 = _z_range(gamma)
        zn = (w[:, 2] - w[:, 2].min()) / (w[:, 2].max() - w[:, 2].min())
        out.append(torch.stack((0.8 * w[:, 0], 0.8 * w[:, 1], z0 + (z1 - z0) * zn), -1))
    verts = torch.stack(out).float().to(DEV)
    faces = osoft.gather_faces(verts, f.to(DEV))
    keep = (ofrag.area32(faces).abs() >= 1e-4).all(0)
    return verts.contiguous(), f[keep.cpu()].to(torch.int32).to(DEV).contiguous()


def _scene(kind, faces, seed, shared=False, light=True, ts=2, tri=False, verts=None, idx=None):
    B, F = faces.shape[:2]
    fl = _rand((B, F, 3), seed + 1, 0.5, 1.5) if light else None
    Bt = 1 if shared else B
    if kind == "sil":
        return Sel("sil", faces, verts, idx)
    if kind == "cube":
        return Sel("cube", faces, verts, idx, tex=_rand((Bt, F, ts, ts, ts, 3), seed + 2), light=fl)
    if kind == "uv":
        # smooth image, inset UVs (as test_gpu_soft_scale._bench_scene): no clamp and no O(1) second differences
        uvs = _rand((Bt, F, 3, 2), seed + 3, 0.05, 0.95)
        return Sel("uv", faces, verts, idx, tex=_image(Bt, 24, 20, seed + 4), uvs=uvs, light=fl, tri=tri)
    raise ValueError(kind)


def _attr_scene(faces, C, per_vertex, seed, shared=False, verts=None, idx=None, depth=False):
    """attributes in [-1, 1] per corner, or per vertex (over verts, or over the faces' corners as 3F vertices);
    depth: the one channel z of every vertex against the background far (soft depth)"""
    B, F = faces.shape[:2]
    Bt = 1 if shared else B
    if per_vertex or depth:
        if verts is None:
            verts = faces.reshape(B, 3 * F, 3).contiguous()
            idx = torch.arange(3 * F, device=DEV, dtype=torch.int32).reshape(F, 3)
        attrs = verts[..., 2:].clone() if depth else _rand((Bt, verts.shape[1], C), seed, -1.0, 1.0)
    else:
        attrs = _rand((Bt, F, 3, C), seed, -1.0, 1.0)
    bg = [FAR] if depth else [0.1 * (c + 1) for c in range(attrs.shape[-1])]
    return Sel("attr", faces, verts, idx, tex=attrs, bg=tuple(bg))


# ------------------------------------------------------------------------------------------------ gradients
def kernel_grads(sc, S, sigma, gamma, g_rgb, g_a):
    leaves = [x.detach().clone().requires_grad_(True) for x in sc.leaves()]
    rgb, alpha = sc.render_leaves(S, sigma, gamma, leaves)
    loss = (alpha * g_a).sum() + ((rgb * g_rgb).sum() if rgb is not None else 0)
    loss.backward()
    return [torch.zeros_like(x) if x.grad is None else x.grad for x in leaves]


def oracle_grads(sc, S, sigma, gamma, pix, p2f, g_rgb, g_a, chunk=1024):
    """float64 autograd of sum(out g_rgb) + sum(alpha g_a) at the pixels pix [B,P] (g_rgb [B,C,P], g_a [B,P]),
    restricted to the selection p2f, one item and `chunk` pixels at a time (the loss is a sum over the pixels)"""
    leaves = [x.detach().double().requires_grad_(True) for x in sc.leaves()]
    B = sc.faces.shape[0]
    flat = sc.flat()
    for b0, c0 in [(b, c) for b in range(B) for c in range(0, pix.shape[1], chunk)]:
        b1 = b0 + 1
        keep = (g_a[b0, c0:c0 + chunk] != 0) | (g_rgb[b0, :, c0:c0 + chunk] != 0).any(0)
        if not keep.any():
            continue
        pc = pix[b0:b1, c0:c0 + chunk][:, keep]
        ga, gr = g_a[b0:b1, c0:c0 + chunk][:, keep], g_rgb[b0:b1, :, c0:c0 + chunk][:, :, keep]
        sl = [x[b0:b1] if x.shape[0] > 1 else x for x in leaves]
        if sc.verts is not None:
            idx = sc.idx if sc.idx.dim() == 2 else sc.idx[b0:b1]
            sl[0] = osoft.gather_faces(sl[0], idx)
        if sc.kind == "attr":
            sl[1] = sc.corner_attrs(sl[1], b0, b1)
        terms = ss.restrict(flat.oracle_terms(sl, S, sigma, ss.WIDE), p2f[b0:b1], pc)
        if sc.kind == "sil":
            alpha = osoft.sparse_eval(sl[0], S, pc, sigma, NEAR, FAR, ss.WIDE, terms)[0]
            loss = (alpha * ga).sum()
        else:
            alpha, out = osoft.sparse_eval(sl[0], S, pc, sigma, NEAR, FAR, ss.WIDE, terms,
                                           orgb.softmax_blend(gamma, sc.bg))
            loss = (out * gr).sum() + (alpha * ga).sum()
        loss.backward()
    return [torch.zeros_like(x) if x.grad is None else x.grad for x in leaves]


def check_grads(got, ref, names, sigma, gamma, what, z=True):
    """per component: the geometry's x/y and z apart, every other leaf whole; returns the worst error / gate.  z: the
    render has a depth gradient (not the silhouettes, nor an upstream on alpha alone)"""
    gate = GATE_LOOSE if sigma < 3e-5 or gamma < 3e-4 else GATE
    worst = 0.0
    for name, a, r in zip(names, got, ref):
        a, r = a.double(), r.double()
        assert torch.isfinite(a).all(), (what, name)
        parts = [(name + ".xy", a[..., :2], r[..., :2]), (name + ".z", a[..., 2], r[..., 2])] \
            if name in ("faces", "vertices") else [(name, a, r)]
        if name in ("faces", "vertices") and z:
            zr, xyr = r[..., 2].abs().max().item(), r[..., :2].abs().max().item()
            assert zr >= 1e-3 * xyr, (what, "z too small to test", zr, xyr)
        for n, x, y in parts:
            if n.endswith(".z") and not z:
                assert x.abs().max() == 0 and y.abs().max() == 0, (what, n)
                continue
            if not z and name not in ("faces", "vertices") and y.abs().max() == 0:
                assert x.abs().max() == 0, (what, n)           # alpha alone: nothing into the colours
                continue
            x, y = x.cpu().numpy(), y.cpu().numpy()
            assert np.abs(y).max() > 0, (what, n, "no reference gradient")
            e = elem_err(x, y, floor=FLOOR)
            assert e <= gate, (what, n, e, gate)
            worst = max(worst, e / gate)
    return worst


def run(sc, S, sigma, gamma, pix, up="both", seed=0, forward=1.0, min_checked=0.5):
    """the whole check of the module docstring at the pixels pix [B,P]; returns the record (worst ratios, counts).
    forward: the scale of the rendered values for the forward check (1: colours; far: soft depth)"""
    B = sc.faces.shape[0]
    faces = sc.faces
    assert (ofrag.area32(faces) != 0).all(), "zero-area face"
    assert osoft.participates(faces.double(), NEAR, FAR).all(), "a face outside [near, far]"
    fr = sc.fragments(S, sigma)
    p2f = fr.pix_to_face
    under = ss.under_full(p2f).reshape(B, -1)
    ts = sc.tex.shape[2] if sc.kind == "cube" else None
    uv = (sc.uvs, sc.tex.shape[1], sc.tex.shape[2], sc.tri) if sc.kind == "uv" else None
    band = ss.band_pixels(faces, p2f, S, cube_ts=ts, uv=uv, lam=sc.kind != "sil")
    checked = torch.gather(under, 1, pix)
    banded = torch.gather(band, 1, pix) & checked
    assert checked.double().mean().item() >= min_checked, (sc.kind, "checked", checked.double().mean().item())
    assert banded.double().sum().item() <= BAND_MAX * checked.double().sum().item(), \
        (sc.kind, "band pixels", banded.sum().item(), checked.sum().item())
    keep = (checked & ~banded).double()
    g = torch.Generator(device=DEV).manual_seed(seed)
    C = 0 if sc.kind == "sil" else (sc.tex.shape[-1] if sc.kind == "attr" else 3)
    g_a_p = torch.randn(B, pix.shape[1], device=DEV, generator=g, dtype=torch.float64) * keep * (up != "rgb")
    g_rgb_p = torch.randn(B, max(C, 1), pix.shape[1], device=DEV, generator=g, dtype=torch.float64) * keep[:, None] \
        * (up != "alpha")
    g_a = torch.zeros(B, S * S, device=DEV).scatter_(1, pix, g_a_p.float())
    g_rgb = torch.zeros(B, max(C, 1), S * S, device=DEV).scatter_(2, pix[:, None].expand(-1, max(C, 1), -1),
                                                                     g_rgb_p.float())
    carries = (g_a != 0) | (g_rgb != 0).any(1)
    assert not (carries & ~under).any(), "upstream gradient at a full pixel"
    got = kernel_grads(sc, S, sigma, gamma, g_rgb.reshape(B, -1, S, S), g_a.reshape(B, S, S))
    ref = oracle_grads(sc, S, sigma, gamma, pix, p2f, g_rgb_p[:, :C], g_a_p)
    what = (sc.kind, S, sigma, gamma, up)
    rec = {"grads": check_grads(got, ref, sc.names(), sigma, gamma, what, z=sc.kind != "sil" and up != "alpha"), "band": banded.sum().item(),
           "checked": checked.sum().item()}
    if forward:
        # the forward at the checked pixels (every pixel of pix with fewer than 32 fragments, band pixels included)
        n = int(checked.sum(1).min())
        fp = torch.stack([pix[b][checked[b]][:n] for b in range(B)])
        flat = sc.flat()
        with torch.no_grad():
            out, alpha = sc.render_leaves(S, sigma, gamma, [x.detach() for x in sc.leaves()])
        if forward != 1.0:
            # values of magnitude `forward` (soft depth: far): the colour gates apply to the image over that scale,
            # against the oracle of the attributes and background over the same scale
            flat = ss.AttrScene(flat.faces, flat.tex / forward, [v / forward for v in flat.bg], NEAR, FAR)
            out = out / forward
        leaves = [x.detach() for x in flat.leaves()]
        terms = ss.restrict(flat.oracle_terms(leaves, S, sigma, ss.WIDE), p2f, fp)
        rec["forward"] = check_forward(flat, out, alpha, S, sigma, gamma, fp, what, terms=terms, cull=ss.WIDE)
    print(what, rec)
    return rec


def _all(B, S):
    return torch.arange(S * S, device=DEV)[None].expand(B, -1).contiguous()


# ------------------------------------------------------------------------------------------------ soups
# (sigma, gamma): gamma 1e-2 with the widest sigma only -- at gamma 1e-2 the softmax moves by one unit per 1.0 of depth,
# and the z gradient falls below 1e-3 of the x/y gradient (which grows as 1 / sqrt(sigma)) at narrower sigma
SG = [(1e-5, 1e-4), (1e-4, 1e-4), (1e-3, 1e-2), (1e-3, 1e-4)]
SOUPS = {64: (2, 200), 127: (3, 250)}   # S: (B, F), up to about 20 faces per pixel


@pytest.mark.parametrize("sigma", [1e-5, 1e-4, 1e-3])
@pytest.mark.parametrize("S", [64, 127])
def test_silhouettes(S, sigma):
    B, F = SOUPS[S]
    faces = _soup(B, F, seed=S, gamma=1e-2)
    run(_scene("sil", faces, 1), S, sigma, 1e-2, _all(B, S), up="alpha", seed=2)


@pytest.mark.parametrize("shared", [False, True])
@pytest.mark.parametrize("light", [False, True])
@pytest.mark.parametrize("ts", [2, 4])
def test_cubes(ts, light, shared):
    S, (B, F) = 64, SOUPS[64]
    i = 4 * (ts == 4) + 2 * light + shared
    sigma, gamma = SG[i % 4]
    faces = _soup(B, F, seed=10 + i, gamma=gamma)
    run(_scene("cube", faces, 20 + i, shared=shared, light=light, ts=ts), S, sigma, gamma, _all(B, S), seed=i)


@pytest.mark.parametrize("up", ["rgb", "alpha", "both"])
def test_cubes_upstream(up):
    S, (B, F) = 127, SOUPS[127]
    faces = _soup(B, F, seed=30, gamma=1e-4)
    run(_scene("cube", faces, 31, light=True, ts=4), S, 1e-4, 1e-4, _all(B, S), up=up, seed=32)


@pytest.mark.parametrize("shared", [False, True])
@pytest.mark.parametrize("tri", [False, True])
def test_uv(tri, shared):
    S, (B, F) = 64, SOUPS[64]
    i = 2 * tri + shared
    sigma, gamma = SG[(i + 1) % 4]
    faces = _soup(B, F, seed=40 + i, gamma=gamma)
    run(_scene("uv", faces, 50 + i, shared=shared, tri=tri), S, sigma, gamma, _all(B, S), seed=i)


@pytest.mark.parametrize("C", [1, 3, 5])
@pytest.mark.parametrize("per_vertex", [False, True])
def test_attributes(per_vertex, C):
    S, (B, F) = 64, SOUPS[64]
    i = 3 * per_vertex + [1, 3, 5].index(C)
    sigma, gamma = SG[i % 4]
    faces = _soup(B, F, seed=60 + i, gamma=gamma)
    run(_attr_scene(faces, C, per_vertex, 70 + i, shared=(i % 2 == 1)), S, sigma, gamma, _all(B, S), seed=i)


def test_soft_depth():
    S, (B, F) = 127, SOUPS[127]
    faces = _soup(B, F, seed=80, gamma=1e-2)
    # depth runs to far = 100: the forward is checked at the scale of far
    run(_attr_scene(faces, 1, True, 81, depth=True), S, 1e-3, 1e-2, _all(B, S), seed=82, forward=FAR)


# ------------------------------------------------------------------------------------------------ indexed geometry
@pytest.mark.parametrize("kind", ["sil", "cube", "attr"])
def test_teapot_shared_indices(kind):
    S, B, sigma, gamma = 96, 2, 1e-4, 1e-4
    verts, idx = _teapot(B, gamma, seed=0)
    faces = osoft.gather_faces(verts, idx)
    if kind == "attr":
        sc = _attr_scene(faces, 3, True, 91, verts=verts, idx=idx)
    else:
        sc = _scene(kind, faces, 92, verts=verts, idx=idx)
    run(sc, S, sigma, gamma, _all(B, S), up="alpha" if kind == "sil" else "both", seed=93, min_checked=0.3)


@pytest.mark.parametrize("kind", ["cube", "attr"])
def test_per_item_indices(kind):
    """vertices [B,Nv,3] shared by the faces of an item through per-item index sets [B,F,3]: each item's faces a
    different permutation of the soup's corners"""
    S, (B, F) = 64, SOUPS[64]
    sigma, gamma = 1e-4, 1e-4
    soup = _soup(B, F, seed=100, gamma=gamma)
    verts = soup.reshape(B, 3 * F, 3).contiguous()
    rng = np.random.default_rng(101)
    perms = [torch.from_numpy(rng.permutation(F)).to(DEV) for _ in range(B)]
    idx = torch.stack([(3 * p[:, None] + torch.arange(3, device=DEV)) for p in perms]).to(torch.int32).contiguous()
    faces = osoft.gather_faces(verts, idx)
    sc = _attr_scene(faces, 3, True, 102, verts=verts, idx=idx) if kind == "attr" else \
        _scene("cube", faces, 103, verts=verts, idx=idx)
    run(sc, S, sigma, gamma, _all(B, S), seed=104)


# ------------------------------------------------------------------------------------------------ deep tiles, benchmark spheres
@pytest.mark.parametrize("kind", ["sil", "cube"])
def test_deep_tiles(kind):
    """the deep-tile scene of tests/test_gpu_soft_scale.py (tile lists over several staging rounds), the upstream on
    the deepest tile and a tile of the front face"""
    S, sigma, gamma = 128, 1e-3, 1e-2
    faces = _deep_faces()
    lb = sb.tile_entries_lower_bound(faces, S, sigma)[0]
    deep = int(lb.argmax())
    assert sb.rounds(lb[deep]).item() >= 3
    nt = sb.tiles_per_axis(S)
    pix = _tile_pixels(S, [deep, (45 // 16) * nt + 82 // 16, 0]).reshape(1, -1)
    sc = _scene(kind, faces, 110, light=True, ts=2)
    run(sc, S, sigma, gamma, pix, up="alpha" if kind == "sil" else "both", seed=111, min_checked=0.2)


@pytest.mark.parametrize("kind,sigma,gamma", [("sil", 1e-4, 1e-4), ("cube", 1e-4, 1e-4), ("uv", 1e-3, 1e-2)])
def test_benchmark_spheres(kind, sigma, gamma):
    """sphere_faces(2, 5000) at 256^2, the upstream on three tiles per item as tests/test_gpu_soft_scale.py picks them"""
    from neural_renderer_b200 import synthetic
    S, B = 256, 2
    faces = torch.from_numpy(synthetic.sphere_faces(B, 5000)).to(DEV)
    tiles, _ = _bench_tiles(faces, S, sigma, seed=5)
    pix = torch.stack([_tile_pixels(S, tiles[b]).reshape(-1) for b in range(B)])
    if kind == "uv":
        uvs = (0.02 + 0.96 * torch.from_numpy(synthetic.sphere_uvs(5000)).to(DEV))[None].contiguous()
        sc = Sel("uv", faces, tex=_image(1, 64, 64, 121), uvs=uvs, light=_rand((B, 5000, 3), 122, 0.5, 1.5),
                 tri=True)
    else:
        sc = _scene(kind, faces, 123, ts=4)
    run(sc, S, sigma, gamma, pix, up="alpha" if kind == "sil" else "both", seed=124, min_checked=0.3)


# ------------------------------------------------------------------------------------------------ the cut-off itself
@pytest.mark.parametrize("kind", ["sil", "cube", "uv", "attr"])
def test_cutoff_pairs_decided_by_the_kernels(kind):
    """faces whose edges lie within fp32 rounding of the cut-off from a row of pixel centres, searched so that the
    kernels' fp32 test keeps pairs the float64 test drops (soft_selection.cutoff_edges): the fragments must hold
    exactly the set every soft kernel aggregated there, or the forward (a D = 1e-4 face against the background
    decides an rgb pixel) and the gradients at the selection fail"""
    S, sigma, gamma = 64, 1e-3, 1e-2
    faces = ss.cutoff_faces(S, sigma, _z_range(gamma)).to(DEV)
    if kind == "attr":
        sc = _attr_scene(faces, 3, False, 131)
    else:
        sc = _scene(kind, faces, 132)
    p2f = sc.fragments(S, sigma).pix_to_face
    n = ss.cutoff_disagreements(faces, p2f, S, sigma)
    assert n >= 50, n
    rec = run(sc, S, sigma, gamma, _all(1, S), up="alpha" if kind == "sil" else "both", seed=133)
    print("cut-off pairs", n, rec)
