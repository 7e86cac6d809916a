"""CPU: the soft oracles restricted to a selection (tests/soft_selection.py) against the unrestricted oracles, and its
band masks on one triangle whose barycentrics, edge distances and texel cells are known in closed form."""
from fractions import Fraction

import pytest
import torch

import oracles_soft as osoft
import oracles_soft_rgb as orgb
import soft_selection as ss
from test_gpu_soft_scale import Scene

NEAR, FAR = 0.1, 100.0
S, SIGMA, GAMMA = 16, 1e-3, 1e-2


def _soup(B=2, F=10, seed=0):
    from neural_renderer_b200 import synthetic
    return torch.from_numpy(synthetic.triangle_soup(B, F, seed=seed, size=(0.1, 0.5), z_range=(2.0, 4.0),
                                                    duplicates=False, offscreen=False))


def _scene(kind, faces):
    B, F = faces.shape[:2]
    g = torch.Generator().manual_seed(1)
    light = 0.5 + torch.rand(B, F, 3, generator=g)
    if kind == "sil":
        return Scene("sil", faces)
    if kind == "cube":
        return Scene("cube", faces, tex=torch.rand(B, F, 3, 3, 3, 3, generator=g), light=light)
    if kind == "uv":
        return Scene("uv", faces, tex=torch.rand(1, 6, 5, 3, generator=g), uvs=0.05 + 0.9 * torch.rand(B, F, 3, 2,
                                                                                                       generator=g),
                     light=light)
    return ss.AttrScene(faces, torch.rand(B, F, 3, 3, generator=g), (0.2, 0.4, 0.6), NEAR, FAR)


def _terms(sc, leaves, cut_scale):
    return sc.oracle_terms(leaves, S, SIGMA, cut_scale)


def _leaves(sc):
    out = sc.leaves()
    return [x.detach().double().requires_grad_(True) for x in out]


def _eval(sc, pix, select=None, cull=1.0, cut_scale=1.0):
    """(values, gradients) of a fixed random loss of the oracle at the pixels pix [B,P], restricted by select(terms)"""
    leaves = _leaves(sc)
    terms = _terms(sc, leaves, cut_scale)
    if select is not None:
        terms = select(terms)
    if sc.kind == "sil":
        alpha = osoft.sparse_eval(leaves[0], S, pix, SIGMA, NEAR, FAR, cull, terms)[0]
        out = alpha[:, None]
    else:
        bg = (0.2, 0.4, 0.6)
        alpha, out = osoft.sparse_eval(leaves[0], S, pix, SIGMA, NEAR, FAR, cull, terms, orgb.softmax_blend(GAMMA, bg))
    g = torch.Generator().manual_seed(2)
    loss = (alpha * torch.randn(alpha.shape, generator=g, dtype=torch.float64)).sum() + \
        (out * torch.randn(out.shape, generator=g, dtype=torch.float64)).sum()
    loss.backward()
    return [alpha.detach(), out.detach()], [torch.zeros_like(x) if x.grad is None else x.grad for x in leaves]


def _own_selection(faces, pad=0):
    """the float64 oracle's own set as pix_to_face [B,S*S,K] (-1 padded, `pad` more empty slots)"""
    f = faces.double()
    d2, inside = osoft.face_terms(f, osoft.pixel_centres(S))
    on = osoft.participates(f, NEAR, FAR)[..., None] & (inside | (d2 <= osoft.cut(SIGMA)))    # [B,F,P]
    B, F, P = on.shape
    Kn = int(on.sum(1).max()) + pad
    fidx = torch.arange(F)[None, :, None].expand(B, -1, P)
    key = torch.where(on, fidx, torch.full_like(fidx, F))
    srt = key.sort(1).values[:, :Kn]                                                 # [B,Kn,P]
    return torch.where(srt < F, srt, torch.full_like(srt, -1)).permute(0, 2, 1).contiguous(), on


def _same(a, b):
    return all(torch.equal(x, y) for x, y in zip(a, b))


KINDS = ["sil", "cube", "uv", "attr"]


@pytest.mark.parametrize("kind", KINDS)
def test_own_selection_is_bit_identical(kind):
    faces = _soup()
    sc = _scene(kind, faces)
    B = faces.shape[0]
    pix = torch.arange(S * S)[None].expand(B, -1)
    p2f, _ = _own_selection(faces)
    v0, g0 = _eval(sc, pix)
    v1, g1 = _eval(sc, pix, lambda t: ss.restrict(t, p2f, pix))
    assert _same(v0, v1) and _same(g0, g1)
    # a subset of the pixels, per item, with the selection of every pixel
    sub = torch.stack([torch.randperm(S * S, generator=torch.Generator().manual_seed(b))[:40] for b in range(B)])
    v0, g0 = _eval(sc, sub)
    v1, g1 = _eval(sc, sub, lambda t: ss.restrict(t, p2f, sub))
    assert _same(v0, v1) and _same(g0, g1)


@pytest.mark.parametrize("kind", KINDS)
def test_empty_and_padding_slots_add_nothing(kind):
    faces = _soup()
    # a face far off the image: culled by every pixel (sparse_eval's padding slots carry its index)
    faces[:, -1] = torch.tensor([[5.0, 5.0, 2.0], [5.5, 5.0, 2.0], [5.0, 5.5, 2.0]])
    sc = _scene(kind, faces)
    B, F = faces.shape[:2]
    pix = torch.arange(S * S)[None].expand(B, -1)
    p2f, _ = _own_selection(faces)
    more, _ = _own_selection(faces, pad=5)
    assert (more[..., -5:] == -1).all()
    listed = more.clone()
    listed[:, ::7, -1] = F - 1                      # the culled face listed at some pixels
    v0, g0 = _eval(sc, pix, lambda t: ss.restrict(t, p2f, pix), cull=ss.WIDE, cut_scale=ss.WIDE)
    for sel in (more, listed):
        v1, g1 = _eval(sc, pix, lambda t: ss.restrict(t, sel, pix), cull=ss.WIDE, cut_scale=ss.WIDE)
        assert _same(v0, v1) and _same(g0, g1)
    assert g0[0][:, -1].abs().max() == 0


@pytest.mark.parametrize("kind", KINDS)
def test_removing_a_pair_changes_only_the_faces_at_that_pixel(kind):
    faces = _soup()
    sc = _scene(kind, faces)
    B = faces.shape[0]
    pix = torch.arange(S * S)[None].expand(B, -1)
    p2f, on = _own_selection(faces)
    base = _eval(sc, pix, lambda t: ss.restrict(t, p2f, pix))
    n = on.sum(1)                                                           # [B,P]
    for want in (1, 3):
        b, p = [int(x) for x in (n == want).nonzero()[0]]
        f = int(p2f[b, p, 0])
        cut = p2f.clone()
        cut[b, p] = torch.where(cut[b, p] == f, torch.full_like(cut[b, p], -1), cut[b, p])
        vals, grads = _eval(sc, pix, lambda t: ss.restrict(t, cut, pix))
        # the values change at that pixel only
        for v, v0 in zip(vals, base[0]):
            d = (v != v0).reshape(B, -1, S * S).any(1)
            assert d[b, p] and d.sum() == 1
        # the gradients change for the faces on at that pixel only, and for f
        at = on[b, :, p]
        for name, g, g0 in zip(range(9), grads, base[1]):
            if g.dim() >= 3 and g.shape[1] == faces.shape[1] and (g.shape[0] == B):
                changed = (g != g0).reshape(B, faces.shape[1], -1).any(-1)
                assert changed[b, f], (want, name)
                assert not changed[1 - b].any() and not changed[b, ~at].any(), (want, name)


# ------------------------------------------------------------------------------------------------ bands in closed form
S8 = 8
TRI = [[-0.625, -0.625, 2.0], [0.875, -0.625, 2.0], [-0.625, 0.875, 2.0]]   # legs of 1.5 on the pixel lattice


def _exact():
    """per pixel of the 8 x 8 image (pixel centres k / 8, k odd): exact barycentrics, d^2 and nearest point per edge"""
    v = [(Fraction(x).limit_denominator(8), Fraction(y).limit_denominator(8)) for x, y, _ in TRI]
    out = []
    for r in range(S8):
        for c in range(S8):
            px, py = Fraction(2 * c + 1 - S8, S8), Fraction(S8 - 1 - 2 * r, S8)
            l1, l2 = (px - v[0][0]) / Fraction(3, 2), (py - v[0][1]) / Fraction(3, 2)
            lam = [1 - l1 - l2, l1, l2]
            d2, near = [], []
            for k in range(3):
                a, b = v[k], v[(k + 1) % 3]
                ex, ey = b[0] - a[0], b[1] - a[1]
                t = min(max(((px - a[0]) * ex + (py - a[1]) * ey) / (ex * ex + ey * ey), Fraction(0)), Fraction(1))
                nx, ny = a[0] + t * ex, a[1] + t * ey
                d2.append((px - nx) ** 2 + (py - ny) ** 2)
                near.append((nx, ny))
            out.append((lam, d2, near))
    return out


def _bands(cube_ts=None, lam=True, sigma=0.015):
    faces = torch.tensor(TRI, dtype=torch.float32)[None, None]
    d2, inside = osoft.face_terms(faces.double(), osoft.pixel_centres(S8))
    on = inside | (d2 <= osoft.cut(sigma))                                   # [1,1,P]
    p2f = torch.where(on[0, 0], 0, -1).reshape(1, S8, S8, 1)
    return ss.band_pixels(faces, p2f, S8, cube_ts=cube_ts, lam=lam)[0], on[0, 0]


def test_bands_of_one_triangle_in_closed_form():
    ex = _exact()
    for what in ("tie", "lam", "cube"):
        got, on = _bands(cube_ts=4 if what == "cube" else None, lam=what == "lam")
        want = torch.zeros(S8 * S8, dtype=torch.bool)
        for i, (lam, d2, near) in enumerate(ex):
            if not on[i]:
                continue
            o = sorted(range(3), key=lambda k: d2[k])
            tie = d2[o[0]] == d2[o[1]] and near[o[0]] != near[o[1]]
            if what == "tie":
                want[i] = tie
            elif what == "lam":
                want[i] = tie or any(x in (0, 1) for x in lam)
            else:
                lh = [min(max(x, Fraction(0)), Fraction(1)) for x in lam]
                t = [3 * x / sum(lh) for x in lh]
                want[i] = tie or any(x in (1, 2) for x in t)
        assert want.any() and (on & ~want).any(), what
        assert torch.equal(got, want), (what, (got != want).nonzero())
    # the vertex region: both edges' nearest point is v0, equal d^2, no tie; inside on the diagonal: a tie
    tie, _ = _bands(lam=False)
    assert not tie[S8 * (S8 - 1) + 0] and tie[S8 * (S8 - 3) + 2]


def test_under_full_counts_the_slots():
    p2f = torch.tensor([[[[0, 1, -1], [0, 1, 2]], [[-1, -1, -1], [2, 0, 1]]]])
    assert torch.equal(ss.under_full(p2f), torch.tensor([[[True, False], [True, False]]]))


def test_cutoff_edges_are_decided_differently_in_fp32_and_float64():
    """the cut-off scene: at the row of every searched edge, the float64 d^2 lies within fp32 rounding of the cut,
    on the opposite side of it from soft_eval's fp32 decision (emulated: fl32(fl32(py - ay)^2) against fl32(cut))"""
    import numpy as np
    S64, sigma = 64, 1e-3
    edges = ss.cutoff_edges(S64, sigma)
    assert len(edges) >= 20
    faces = ss.cutoff_faces(S64, sigma, (2.0, 6.0))
    cut = osoft.cut(sigma)
    for i, (row, ay, kernel_on) in enumerate(edges):
        py = (2 * row + 1 - S64) / S64
        p = torch.tensor([[faces[0, i, 0, 0].item() + 0.125, py]], dtype=torch.float64)
        d2, inside = osoft.face_terms(faces[:, i:i + 1].double(), p)
        assert not inside.any() and abs(d2.item() / cut - 1) < 1e-6
        assert (d2.item() <= cut) != kernel_on
        dy = np.float32(np.float64(np.float32(py)) - np.float64(np.float32(ay)))
        assert bool(np.float32(np.float64(dy) ** 2) <= np.float32(cut)) == kernel_on
