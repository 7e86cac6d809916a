"""GPU: soft fragments (rasterize_soft_fragments, nr_b200_soft_fragments[_backward]) against their definition and the
float64 oracle of tests/oracles_soft_frag.py.

The selection is checked by its definition, pixel by pixel, at every pixel (none is excluded): every selected face is a
candidate; no duplicates and the slots fill front to back; the -1 tail is exact; zbuf is non-decreasing with face-index
order at exact ties; n lies between the counts of certain and possible candidates (the fp32 cut-off test may decide a
face within the band of oracles_soft_frag either way), capped at K; and no certain candidate left out is nearer than
the K-th slot by more than the two faces' tie bands.  The float64 zp of the oracle and the kernel's fp32 zp differ by
the derived zbuf gate, which is that tie band.

Then zbuf, bary and dists at the selected pairs are compared with the oracle's evaluation at the same pairs under the
derived gates of oracles_soft_frag's docstring (the error analysis of DESIGN.md 4o/4p with a safety factor of 4):
  dists 4 (2 d delta + delta^2 + 4 eps d^2), zbuf 4 (8 eps zp + 3 dl zp^2 / min z), bary 4 (dl zp / min z +
  max |l'| (dzp / zp + 4 eps)), dl = 8 eps |e| (|e| + d) / |A|, delta = 4 eps max(1, |v|), eps = 2^-23;
each plus 4 eps of the output's own rounding.  Gradients are compared with float64 autograd of the oracle's evaluation
at the kernel's own selection, so no tie can make them disagree."""
import ctypes
import math
import os

import numpy as np
import pytest
import torch

import oracles_soft as osoft
import oracles_soft_frag as ofrag
from helpers import elem_err, rel_err

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
NEAR, FAR = 0.1, 100.0
SIGMAS = (1e-5, 1e-4, 1e-3)
PEAK_LIMIT = int(2.2 * 2 ** 30)
INVALID = -1  # NR_ERR_INVALID_ARG


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


def _soup(B, F, seed, **kw):
    from neural_renderer_b200 import synthetic
    return torch.from_numpy(synthetic.triangle_soup(B, F, seed=seed, **kw)).to(DEV)


def _special_faces(B, sigma, seed, F=24):
    """a soup plus test_gpu_soft.py's special faces: wider than the wide-list cap, outside the image within reach,
    straddling near / far, exactly at near and far, zero-area (collinear and a point)"""
    soup = _soup(B, F, seed, size=(0.02, 0.3))
    reach = math.sqrt(osoft.cut(sigma))
    o = 1.0 + 0.5 * reach
    extra = [[[-1.1, -1.0, 1.5], [1.2, -0.9, 1.5], [0.1, 1.3, 1.5]],
             [[-0.9, 0.95, 2.0], [0.9, 0.9, 2.0], [0.0, 0.97, 2.0]],
             [[o, -0.3, 1.2], [o + 0.2, 0.0, 1.2], [o, 0.3, 1.2]],
             [[-0.3, -o, 1.2], [0.3, -o, 1.2], [0.0, -o - 0.2, 1.2]],
             [[-0.5, 0.1, 0.05], [-0.2, 0.1, 1.0], [-0.4, 0.4, 1.0]],
             [[0.2, -0.5, 1.0], [0.5, -0.5, 150.0], [0.3, -0.2, 1.0]],
             [[0.1, 0.5, 0.1], [0.3, 0.5, 100.0], [0.2, 0.7, 1.0]],
             [[-0.6, -0.6, 1.0], [-0.2, -0.2, 1.0], [-0.4, -0.4, 1.0]],
             [[0.6, 0.2, 1.0], [0.6, 0.2, 1.0], [0.6, 0.2, 1.0]]]
    ex = torch.tensor(extra, dtype=torch.float32, device=DEV)[None].expand(B, -1, -1, -1)
    return torch.cat((soup, ex), 1).contiguous()


def _teapot():
    d = np.load(os.path.join(os.path.dirname(__file__), "golden", "teapot.npz"))
    v = torch.from_numpy(d["vertices"].astype(np.float32)).to(DEV)[None]
    f = torch.from_numpy(d["faces"].astype(np.int32)).to(DEV)[None]
    return v, f


def _rand(shape, seed, lo=-1.0, hi=1.0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return lo + (hi - lo) * torch.rand(*shape, device=DEV, generator=g)


# ------------------------------------------------------------------------------------------------ checks
def check_selection(frag, faces, S, sigma, K, pix=None):
    """the selection of frag at the pixels pix ([P] flat, the same for every item; None = all) by its definition"""
    p2f, zbuf, bary, dists = frag
    B, F = faces.shape[:2]
    pixv = torch.arange(S * S, device=DEV) if pix is None else pix.to(DEV).unique()   # a pixel set: no repeats
    pix = None if pix is None else pixv
    P = pixv.numel()
    sp = p2f.reshape(B, S * S, K)[:, pixv]                                    # [B,P,K]
    sz = zbuf.reshape(B, S * S, K)[:, pixv]
    sb_ = bary.reshape(B, S * S, K, 3)[:, pixv]
    sd = dists.reshape(B, S * S, K)[:, pixv]
    sel = sp >= 0
    n = sel.sum(-1)
    # front to back, exact -1 tail
    assert torch.all(sel[..., 1:] <= sel[..., :-1])
    assert torch.all(sz[~sel] == -1) and torch.all(sd[~sel] == -1) and torch.all(sb_[~sel] == -1)
    assert torch.all(sp[sel] < F)
    # no duplicates; zbuf non-decreasing, face order at exact ties
    a, b2 = sp[..., :-1], sp[..., 1:]
    both = sel[..., 1:]
    za, zb = sz[..., :-1], sz[..., 1:]
    assert torch.all(~both | (zb > za) | ((zb == za) & (b2 > a)))
    # the oracle's candidates at these pixels
    cb, cpix, cf, czp, cert, band = (t.to(DEV) for t in ofrag.candidates(faces, S, sigma, NEAR, FAR, pix=pix))
    slot = torch.full((B, S * S), -1, dtype=torch.long, device=DEV)
    slot[:, pixv] = torch.arange(P, device=DEV)
    cp = slot[cb, cpix]
    assert torch.all(cp >= 0)
    key = lambda bb, pp, ff: (bb * P + pp) * F + ff                           # noqa: E731
    ck = key(cb, cp, cf)
    order = torch.argsort(ck)
    ck, czp, cert, band, cbb, cpp = ck[order], czp[order], cert[order], band[order], cb[order], cp[order]
    bi = torch.arange(B, device=DEV)[:, None, None].expand_as(sp)
    pi = torch.arange(P, device=DEV)[None, :, None].expand_as(sp)
    skey = key(bi, pi, sp.clamp_min(0))[sel]
    if ck.numel() == 0:                                                       # nothing within reach of these pixels
        assert not sel.any() and n.max().item() == 0
        return n
    at = torch.searchsorted(ck, skey).clamp(max=ck.numel() - 1)
    assert torch.all(ck[at] == skey), "a selected face is not a candidate"
    # n between the certain and the possible counts, capped at K
    n_pos = torch.zeros(B * P, dtype=torch.long, device=DEV).index_add_(0, cbb * P + cpp, torch.ones_like(cpp))
    n_cer = torch.zeros(B * P, dtype=torch.long, device=DEV).index_add_(0, cbb * P + cpp, cert.long())
    nf = n.reshape(-1)
    assert torch.all(nf >= n_cer.clamp(max=K)) and torch.all(nf <= n_pos.clamp(max=K))
    # no certain candidate left out nearer than the last slot of a full pixel by more than the tie bands
    chosen = torch.zeros_like(cert)
    chosen[at] = True
    left = cert & ~chosen
    full = (nf == K)[cbb * P + cpp]
    assert not torch.any(left & ~full), "a certain candidate is missing from a pixel with a free slot"
    # the K-th slot's own tie band (its face is a candidate: found above)
    lkey = key(bi[..., 0], pi[..., 0], sp[..., K - 1].clamp_min(0)).reshape(-1)
    lband = band[torch.searchsorted(ck, lkey).clamp(max=ck.numel() - 1)]
    lastz = sz[..., K - 1].reshape(-1)[cbb * P + cpp].double()
    bad = left & full & (czp < lastz - band - lband[cbb * P + cpp])
    assert not torch.any(bad), (czp[bad][:4], lastz[bad][:4])
    return n


def check_values(frag, faces, S):
    """zbuf, bary and dists at the selected pairs against the oracle's evaluation, under the derived gates"""
    p2f, zbuf, bary, dists = frag
    f64 = faces.double()
    zb, by, ds = ofrag.evaluate(f64, p2f, S)
    gz, gb, gd = ofrag.gates(f64, p2f, S)
    worst = {}
    for name, got, ref, gate in (("zbuf", zbuf, zb, gz), ("dists", dists, ds, gd), ("bary", bary, by, gb[..., None])):
        err = (got.double() - ref).abs()
        sel = (p2f >= 0) if got.dim() == 4 else (p2f >= 0)[..., None].expand_as(got)
        ratio = torch.where(sel, err / gate.expand_as(err).clamp_min(1e-300), torch.zeros_like(err))
        assert torch.all(got[~sel] == -1), name
        assert ratio.max().item() <= 1.0, (name, ratio.max().item())
        worst[name] = ratio.max().item()
    return worst


# ------------------------------------------------------------------------------------------------ forward
@pytest.mark.parametrize("K", [1, 3, 8, 32])
@pytest.mark.parametrize("sigma", SIGMAS)
@pytest.mark.parametrize("S", [64, 127, 256, 257])
def test_forward_by_definition_soups_and_special_faces(S, sigma, K):
    nr = _nr()
    seed = S + 7 * K + int(-math.log10(sigma))
    faces = _special_faces(2, sigma, seed)
    frag = nr.rasterize_soft_fragments(faces, S, sigma, K)
    assert frag.pix_to_face.shape == (2, S, S, K) and frag.pix_to_face.dtype == torch.int64
    assert frag.bary_coords.shape == (2, S, S, K, 3) and frag.zbuf.dtype == torch.float32
    n = check_selection(frag, faces, S, sigma, K)
    check_values(frag, faces, S)
    assert n.max().item() >= min(K, 2)
    # the zero-area faces (the last two) are never fragments
    F = faces.shape[1]
    assert not torch.any((frag.pix_to_face == F - 1) | (frag.pix_to_face == F - 2))


def test_forward_by_definition_teapot():
    nr = _nr()
    v, f = _teapot()
    r = nr.Renderer()
    r.eye = nr.get_points_from_angles(2.732, 30, -15)
    faces = osoft.gather_faces(r._transform(v), f[0]).float().contiguous()
    S, sigma, K = 128, 1e-4, 8
    frag = nr.rasterize_soft_fragments(faces, S, sigma, K)
    n = check_selection(frag, faces, S, sigma, K)
    check_values(frag, faces, S)
    assert (n == K).sum().item() > 20 and (n >= 2).sum().item() > 1000


def test_sphere_benchmark_geometry_three_tiles_per_item():
    from neural_renderer_b200 import synthetic
    import test_gpu_soft_scale as tss
    nr = _nr()
    B, Fn, S, sigma, K = 64, 5000, 256, 1e-4, 8
    faces = torch.from_numpy(synthetic.sphere_faces(B, Fn)).to(DEV)
    frag = nr.rasterize_soft_fragments(faces, S, sigma, K)
    tiles, _ = tss._bench_tiles(faces, S, sigma, 5)
    for b0 in range(0, B, 16):
        sub = tuple(t[b0:b0 + 16] for t in frag)
        for j in range(3):
            pix = tss._tile_pixels(S, tiles[b0:b0 + 1, j])[0]
            check_selection(sub, faces[b0:b0 + 16], S, sigma, K, pix=pix)
    sub = tuple(t[:2] for t in frag)
    check_values(sub, faces[:2], S)


def test_deep_tiles_by_definition_and_permutation():
    import test_gpu_soft_scale as tss
    nr = _nr()
    faces = tss._deep_faces()
    S, sigma, K = tss.S_DEEP, tss.SIGMA_DEEP, 8
    frag = nr.rasterize_soft_fragments(faces, S, sigma, K)
    n = check_selection(frag, faces, S, sigma, K)
    check_values(frag, faces, S)
    assert (n == K).sum().item() > 100
    perm = torch.randperm(faces.shape[1], generator=torch.Generator().manual_seed(3)).to(DEV)
    fp = nr.rasterize_soft_fragments(faces[:, perm].contiguous(), S, sigma, K)
    _assert_permuted(frag, fp, perm)


def _assert_permuted(frag, fp, perm):
    """fp = the fragments of faces[:, perm]: its face j is face perm[j] of frag; where no exact zp tie reorders a pixel,
    every field is bit-identical"""
    p2f, zb = frag.pix_to_face, frag.zbuf
    mapped = torch.where(fp.pix_to_face >= 0, perm_back(fp.pix_to_face, perm), fp.pix_to_face)
    tie = ((zb[..., 1:] == zb[..., :-1]) & (p2f[..., 1:] >= 0)).any(-1, keepdim=True)
    same = ~tie
    assert torch.equal(mapped[same.expand_as(mapped)], p2f[same.expand_as(p2f)])
    for a, b in ((frag.zbuf, fp.zbuf), (frag.dists, fp.dists), (frag.bary_coords, fp.bary_coords)):
        m = same if a.dim() == 4 else same[..., None]
        assert torch.equal(a[m.expand_as(a)], b[m.expand_as(b)])


def perm_back(p2f, perm):
    return torch.gather(perm[None].expand(p2f.shape[0], -1), 1, p2f.clamp_min(0).reshape(p2f.shape[0], -1)).reshape(p2f.shape)


def test_64_bit_keys_selection_bit_identical_across_face_counts():
    import soft_binning as sb
    import test_gpu_soft_scale as tss
    nr = _nr()
    B, S, sigma, K = 2, tss.S_KEY, tss.SIGMA_KEY, 2
    real = tss._real_faces(B, 21)
    outs = []
    for F in (65535, 65536):
        assert sb.key_width(B, F, S)[2] is (F == 65536)
        faces, pos = tss._padded(real, F, 22 + F)
        frag = nr.rasterize_soft_fragments(faces, S, sigma, K)
        p = frag.pix_to_face
        # back to the real faces' own indices
        idx = torch.full((F,), -7, dtype=torch.long, device=DEV)
        idx[pos] = torch.arange(pos.numel(), device=DEV)
        mapped = torch.where(p >= 0, idx[p.clamp_min(0)], p)
        assert torch.all(mapped >= -1), "a padding face was selected"
        outs.append((mapped, frag.zbuf, frag.bary_coords, frag.dists))
        if F == 65536:
            pix = tss._pixels_near(real, S, 256, 23)[0]
            check_selection(frag, faces, S, sigma, K, pix=pix)
        del frag, faces
    for a, b in zip(*outs):
        assert torch.equal(a, b)


# ------------------------------------------------------------------------------------------------ bit identities
def test_bit_identities():
    nr = _nr()
    S, sigma = 96, 1e-3
    faces = _special_faces(2, sigma, 41)
    B, F = faces.shape[:2]
    a = nr.rasterize_soft_fragments(faces, S, sigma, 8)
    b = nr.rasterize_soft_fragments(faces, S, sigma, 8)
    for x, y in zip(a, b):
        assert torch.equal(x, y)
    # K-prefix: the first K1 slots of a K2 call are the K1 call, across every kCap
    calls = {K: nr.rasterize_soft_fragments(faces, S, sigma, K) for K in (1, 2, 3, 4, 5, 8, 9, 16, 17, 32)}
    for K1 in calls:
        for K2 in calls:
            if K1 < K2:
                for x, y in zip(calls[K1], calls[K2]):
                    assert torch.equal(x, y[:, :, :, :K1]), (K1, K2)
    # indexed = materialised, with shared and out-of-range indices
    verts = faces.reshape(B, F * 3, 3).contiguous()
    idx = torch.arange(F * 3, device=DEV, dtype=torch.int32).reshape(F, 3)
    idx[3, 1] = F * 3 + 5      # out of range: the zero vertex (z = 0 < near: the face takes no part)
    mat = osoft.gather_faces(verts, idx).float().contiguous()
    for shared in (True, False):
        ii = idx if shared else idx[None].expand(B, -1, -1).contiguous()
        x = nr.rasterize_soft_fragments(ii, S, sigma, 8, vertices=verts)
        y = nr.rasterize_soft_fragments(mat, S, sigma, 8)
        for u, w in zip(x, y):
            assert torch.equal(u, w)
    # a face permutation
    perm = torch.randperm(F, generator=torch.Generator().manual_seed(5)).to(DEV)
    fp = nr.rasterize_soft_fragments(faces[:, perm].contiguous(), S, sigma, 32)
    _assert_permuted(calls[32], fp, perm)


# ------------------------------------------------------------------------------------------------ the existing soft path
def _blend(frag, ca, sigma, gamma, bg):
    """SoftRas's blend of the fragments in torch: w = sigmoid(dists / sigma) exp((zn - zmax) / gamma) with the
    background term at zn = 1e-3, colours by interpolate_face_attributes; [B,C,S,S]"""
    from neural_renderer_b200 import functional as Fn
    p2f, zbuf, bary, dists = frag
    sel = p2f >= 0
    A = Fn.interpolate_face_attributes(p2f, bary, ca)                           # [B,S,S,K,C]
    zn = (FAR - zbuf) / (FAR - NEAR)
    zmax = torch.where(sel, zn, torch.full_like(zn, -math.inf)).amax(-1, keepdim=True).clamp_min(1e-3).detach()
    w = torch.where(sel, torch.sigmoid(dists / sigma) * torch.exp((zn - zmax) / gamma), torch.zeros_like(zn))
    wb = torch.exp((1e-3 - zmax) / gamma)
    bgt = torch.tensor(bg, dtype=w.dtype, device=DEV)
    out = ((w[..., None] * A).sum(-2) + wb * bgt) / (w.sum(-1, keepdim=True) + wb)
    return out.permute(0, 3, 1, 2)


@pytest.mark.parametrize("gamma", [1e-4, 1e-2])
def test_blended_fragments_equal_the_soft_attributes(gamma):
    nr = _nr()
    S, sigma, K = 64, 1e-3, 16
    faces = _special_faces(2, sigma, 51, F=20)
    B, F = faces.shape[:2]
    ca = _rand((B, F, 3, 3), 52, 0.0, 1.0)
    bg = (0.2, 0.5, 0.8)
    fv = faces.clone().requires_grad_(True)
    cv = ca.clone().requires_grad_(True)
    frag = nr.rasterize_soft_fragments(fv, S, sigma, K)
    n = (frag.pix_to_face >= 0).sum(-1)
    assert (n < K).all()                                      # every pixel's fragment set is the contributing set
    out = _blend(frag, cv, sigma, gamma, bg)
    fw = faces.clone().requires_grad_(True)
    cw = ca.clone().requires_grad_(True)
    ref = nr.rasterize_soft_attributes(fw, S, sigma, gamma, face_attributes=cw, background=bg)
    gate = 4 * (1e-6 / math.sqrt(sigma) + 1e-6) + 5e-4
    assert (out - ref).abs().max().item() <= gate, (out - ref).abs().max().item()
    up = _rand(ref.shape, 53)
    (out * up).sum().backward()
    (ref * up).sum().backward()
    assert rel_err(cv.grad.cpu(), cw.grad.cpu()) <= 1e-4, rel_err(cv.grad.cpu(), cw.grad.cpu())
    assert rel_err(fv.grad.cpu(), fw.grad.cpu()) <= 2e-3, rel_err(fv.grad.cpu(), fw.grad.cpu())
    # soft depth: the camera z as the attribute, the background at far
    z = faces[..., 2:3].contiguous()
    dref = nr.rasterize_soft_attributes(faces, S, sigma, gamma, face_attributes=z, background=[FAR])
    dout = _blend(frag, z, sigma, gamma, (FAR,))
    assert ((dout - dref).abs() / dref.abs().clamp_min(1.0)).max().item() <= gate


def test_tiny_sigma_slot_zero_is_the_hard_rasterizer():
    nr = _nr()
    v, f = _teapot()
    r = nr.Renderer()
    r.eye = nr.get_points_from_angles(2.732, 30, -15)
    S = 256
    faces = osoft.gather_faces(r._transform(v), f[0]).float().contiguous()
    frag = nr.rasterize_soft_fragments(faces, S, 1e-7, 2)
    # the hard rasterizer draws one winding: give it the reversed copies too (face f + F is face f)
    both = torch.cat((faces, faces.flip(2)), 1).contiguous()
    F = faces.shape[1]
    hard = nr.Rasterize(S, NEAR, FAR, 1e-3, [0, 0, 0], return_depth=True)
    hard(both)
    fim = hard.face_index_map.flip(1).long()
    fim = torch.where(fim >= F, fim - F, fim)
    depth = nr.rasterize_depth(both, S, False, NEAR, FAR)
    # pixels inside slot 0's face more than 1 px from its edges, without a depth tie between the first two slots
    zb = frag.zbuf[0].reshape(-1, 2)
    clear = (frag.dists[0].reshape(-1, 2)[:, 0] > (2.0 / S) ** 2) & (frag.pix_to_face[0].reshape(-1, 2)[:, 0] >= 0)
    clear &= (frag.pix_to_face[0].reshape(-1, 2)[:, 1] < 0) | (zb[:, 1] - zb[:, 0] > 1e-3)
    clear = clear.reshape(S, S)
    assert clear.sum().item() > 500
    assert torch.equal(frag.pix_to_face[0, :, :, 0][clear], fim[0][clear])
    err = (frag.zbuf[0, :, :, 0] - depth[0]).abs()[clear]
    assert err.max().item() <= 1e-5 * depth[0][clear].max().item(), err.max().item()


# ------------------------------------------------------------------------------------------------ backward
def _oracle_grads(faces, frag, S, ups):
    fv = faces.double().requires_grad_(True)
    zb, by, ds = ofrag.evaluate(fv, frag.pix_to_face, S)
    loss = sum((o * u.double()).sum() for o, u in zip((zb, by, ds), ups) if u is not None)
    (g,) = torch.autograd.grad(loss, fv)
    return g


@pytest.mark.parametrize("which", ["zbuf", "bary", "dists", "all"])
@pytest.mark.parametrize("sigma", [1e-4, 1e-3])
def test_backward_vs_float64_autograd_at_the_kernel_selection(which, sigma):
    nr = _nr()
    S, K = 64, 8
    faces = _special_faces(2, sigma, 61)
    fv = faces.clone().requires_grad_(True)
    frag = nr.rasterize_soft_fragments(fv, S, sigma, K)
    shapes = (frag.zbuf.shape, frag.bary_coords.shape, frag.dists.shape)
    ups = [_rand(s, 62 + i) for i, s in enumerate(shapes)]
    names = ("zbuf", "bary", "dists")
    ups = [u if which in ("all", n) else None for u, n in zip(ups, names)]
    loss = sum((o * u).sum() for o, u in zip((frag.zbuf, frag.bary_coords, frag.dists), ups) if u is not None)
    (g,) = torch.autograd.grad(loss, fv)
    ref = _oracle_grads(faces, frag, S, ups)
    assert elem_err(g.cpu(), ref.cpu(), floor=1e-3) <= 2e-3, elem_err(g.cpu(), ref.cpu(), floor=1e-3)
    # faces with no fragment get exactly 0
    used = torch.zeros(faces.shape[:2], dtype=torch.bool, device=DEV)
    for b in range(faces.shape[0]):
        ids = frag.pix_to_face[b][frag.pix_to_face[b] >= 0].unique()
        used[b, ids] = True
    assert torch.all(g[~used] == 0)


def test_backward_indexed_shared_out_of_range_and_accumulate():
    from neural_renderer_b200 import _lib
    nr = _nr()
    S, sigma, K = 64, 1e-3, 4
    faces = _special_faces(2, sigma, 71)
    B, F = faces.shape[:2]
    verts = faces.reshape(B, F * 3, 3).contiguous()
    verts = torch.cat((verts, _rand((B, 4, 3), 72, 0.0, 0.5) + torch.tensor([0, 0, 2.0], device=DEV)), 1).contiguous()
    idx = torch.arange(F * 3, device=DEV, dtype=torch.int32).reshape(F, 3)
    idx[5, 2] = F * 3 + 99                                     # out of range: reads the zero vertex
    vv = verts.clone().requires_grad_(True)
    frag = nr.rasterize_soft_fragments(idx, S, sigma, K, vertices=vv)
    ups = [_rand(t.shape, 73 + i) for i, t in enumerate((frag.zbuf, frag.bary_coords, frag.dists))]
    loss = sum((o * u).sum() for o, u in zip((frag.zbuf, frag.bary_coords, frag.dists), ups))
    (g,) = torch.autograd.grad(loss, vv)
    fo = verts.double().requires_grad_(True)
    zb, by, ds = ofrag.evaluate(osoft.gather_faces(fo, idx), frag.pix_to_face, S)
    (ref,) = torch.autograd.grad(sum((o * u.double()).sum() for o, u in zip((zb, by, ds), ups)), fo)
    assert elem_err(g.cpu(), ref.cpu(), floor=1e-3) <= 2e-3
    assert torch.all(g[:, F * 3:] == 0)                        # the padding vertices no face uses
    # NR_GRAD_ACCUMULATE over a seeded prefill, through the C ABI
    lib = _lib.load()
    pre = _rand(verts.shape, 74)
    gv = pre.clone()
    a, t, ws = _abi_args(verts=verts, idx=idx, S=S, sigma=sigma, K=K, backward=True)
    a.flags |= _lib.NR_GRAD_ACCUMULATE
    a.grad_vertices = gv.data_ptr()
    p2f = frag.pix_to_face.contiguous()
    t.pix_to_face = p2f.data_ptr()
    uz, ub, ud = (u.contiguous() for u in ups)
    t.grad_zbuf, t.grad_bary, t.grad_dists = uz.data_ptr(), ub.data_ptr(), ud.data_ptr()
    assert lib.nr_b200_soft_fragments_backward(ctypes.byref(a), ctypes.byref(t), _stream()) == 0
    torch.cuda.synchronize()
    assert rel_err((gv - pre).cpu(), g.cpu()) <= 1e-5


def test_backward_vs_central_differences_of_the_forward():
    nr = _nr()
    S, sigma, K = 48, 1e-3, 2
    faces = torch.tensor([[[[-0.7, -0.6, 2.0], [0.5, -0.5, 3.0], [0.0, 0.6, 4.0]],
                           [[-0.2, 0.1, 1.5], [0.6, 0.3, 1.7], [0.1, 0.8, 1.6]]]], device=DEV)
    frag = nr.rasterize_soft_fragments(faces, S, sigma, K)
    # pixels well inside every selected face: a small step moves no selection there
    d2, inside = osoft.face_terms(faces.double(), osoft.pixel_centres(S, device=DEV))          # [1,2,P]
    far_out = (math.sqrt(osoft.cut(sigma)) + 0.02) ** 2
    inner = (((inside & (d2 > 4e-3)) | (~inside & (d2 > far_out))).all(1) & inside.any(1)).reshape(1, S, S)
    assert inner.sum().item() > 200
    ups = [_rand(t.shape, 81 + i) * (inner[..., None] if t.dim() == 4 else inner[..., None, None])
           for i, t in enumerate((frag.zbuf, frag.bary_coords, frag.dists))]

    def loss(ff):
        fr = nr.rasterize_soft_fragments(ff, S, sigma, K)
        assert torch.equal(fr.pix_to_face[inner], frag.pix_to_face[inner])
        return sum((o.double() * u.double()).sum() for o, u in zip((fr.zbuf, fr.bary_coords, fr.dists), ups))

    fv = faces.clone().requires_grad_(True)
    fr = nr.rasterize_soft_fragments(fv, S, sigma, K)
    (g,) = torch.autograd.grad(sum((o * u).sum() for o, u in zip((fr.zbuf, fr.bary_coords, fr.dists), ups)), fv)
    h = 1e-3
    num = torch.zeros_like(g)
    for i in range(faces.numel()):
        e = torch.zeros(faces.numel(), device=DEV)
        e[i] = h
        e = e.reshape(faces.shape)
        num.view(-1)[i] = ((loss(faces + e) - loss(faces - e)) / (2 * h)).float()
    assert rel_err(g.cpu(), num.cpu()) <= 2e-2, rel_err(g.cpu(), num.cpu())


# ------------------------------------------------------------------------------------------------ direct ABI
def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream(DEV).cuda_stream)


def _abi_args(faces=None, verts=None, idx=None, S=32, sigma=1e-3, K=4, backward=False):
    from neural_renderer_b200 import _lib
    lib = _lib.load()
    a = _lib.SoftRgbArgs()
    a.struct_size = ctypes.sizeof(_lib.SoftRgbArgs)
    if verts is not None:
        B, F = verts.shape[0], idx.shape[-2]
        a.flags = _lib.NR_FACES_INDEXED | (_lib.NR_INDICES_SHARED if idx.dim() == 2 else 0)
        a.vertices, a.face_indices, a.num_vertices = verts.data_ptr(), idx.data_ptr(), verts.shape[1]
    else:
        B, F = faces.shape[:2]
        a.faces = faces.data_ptr()
    a.batch_size, a.num_faces, a.image_size = B, F, S
    a.sigma, a.near_, a.far_ = sigma, NEAR, FAR
    n = lib.nr_b200_soft_rgb_workspace_bytes(B, F, S, a.flags)
    ws = torch.empty(n, dtype=torch.uint8, device=DEV)
    a.workspace, a.workspace_bytes = ws.data_ptr(), n
    t = _lib.SoftFragArgs(struct_size=ctypes.sizeof(_lib.SoftFragArgs), faces_per_pixel=K)
    return a, t, ws


def _guarded(n, dtype, fill, guard=16):
    buf = torch.full((n + 2 * guard,), fill, dtype=dtype, device=DEV)
    return buf, buf[guard:guard + n]


@pytest.mark.parametrize("K", [3, 8])
def test_abi_poison_guards_nulls_and_refusals(K):
    from neural_renderer_b200 import _lib
    nr = _nr()
    lib = _lib.load()
    S, sigma = 40, 1e-3
    faces = _special_faces(2, sigma, 91, F=12)
    B, F = faces.shape[:2]
    ref = nr.rasterize_soft_fragments(faces, S, sigma, K)
    n = B * S * S * K
    bufs = [_guarded(n, torch.int64, -12345), _guarded(n, torch.float32, float("nan")),
            _guarded(3 * n, torch.float32, float("nan")), _guarded(n, torch.float32, float("nan"))]
    a, t, ws = _abi_args(faces=faces, S=S, sigma=sigma, K=K)
    t.pix_to_face, t.zbuf, t.bary, t.dists = (v.data_ptr() for _, v in bufs)
    assert lib.nr_b200_soft_fragments(ctypes.byref(a), ctypes.byref(t), _stream()) == 0
    torch.cuda.synchronize()
    for (full, view), r in zip(bufs, ref):
        assert torch.equal(view, r.reshape(-1))
        guards = torch.cat((full[:16], full[-16:]))
        assert torch.all(guards == -12345) if guards.dtype == torch.int64 else torch.isnan(guards).all()
    # the backward: every allowed NULL upstream gradient, and all NULL (a zero-fill)
    g = torch.full_like(faces, float("nan"))
    ups = [_rand(s, 92 + i) for i, s in enumerate(((B, S, S, K), (B, S, S, K, 3), (B, S, S, K)))]
    for mask in range(8):
        a, t, ws = _abi_args(faces=faces, S=S, sigma=sigma, K=K, backward=True)
        a.grad_faces = g.data_ptr()
        t.pix_to_face = ref.pix_to_face.data_ptr()
        t.grad_zbuf = ups[0].data_ptr() if mask & 1 else None
        t.grad_bary = ups[1].data_ptr() if mask & 2 else None
        t.grad_dists = ups[2].data_ptr() if mask & 4 else None
        assert lib.nr_b200_soft_fragments_backward(ctypes.byref(a), ctypes.byref(t), _stream()) == 0
        torch.cuda.synchronize()
        assert torch.isfinite(g).all()
        if mask == 0:
            assert torch.all(g == 0)
        else:
            want = _oracle_grads(faces, ref, S, [u if mask & (1 << i) else None for i, u in enumerate(ups)])
            assert elem_err(g.cpu(), want.cpu(), floor=1e-3) <= 2e-3
    # refusals launch nothing and write nothing
    before = [v.clone() for _, v in bufs]
    a, t, ws = _abi_args(faces=faces, S=S, sigma=sigma, K=33)
    t.pix_to_face, t.zbuf, t.bary, t.dists = (v.data_ptr() for _, v in bufs)
    assert lib.nr_b200_soft_fragments(ctypes.byref(a), ctypes.byref(t), _stream()) == INVALID
    assert lib.nr_b200_last_launch_count() == 0
    a.rgb = bufs[1][1].data_ptr()
    t.faces_per_pixel = K
    assert lib.nr_b200_soft_fragments(ctypes.byref(a), ctypes.byref(t), _stream()) == INVALID
    torch.cuda.synchronize()
    for (_, v), w in zip(bufs, before):
        assert torch.all((v == w) | ((v != v) & (w != w)))


# ------------------------------------------------------------------------------------------------ fits, Renderer, graphs
def _tri_at(cx, cy, s=2.0 / 128):
    return torch.tensor([[[[cx - s, cy - s, 2.0], [cx + s, cy - s, 2.0], [cx, cy + s, 2.0]]]], device=DEV)


def test_translation_fit_through_a_torch_blend_of_fragments():
    nr = _nr()
    S, sigma, K = 128, 1e-4, 4
    px = 2.0 / S

    def silhouette(f):
        fr = nr.rasterize_soft_fragments(f, S, sigma, K)
        D = torch.where(fr.pix_to_face >= 0, torch.sigmoid(fr.dists / sigma), torch.zeros_like(fr.dists))
        return 1 - torch.prod(1 - D, -1)

    target = silhouette(_tri_at(0.0, 0.0)).detach()
    off = torch.tensor([3 * px, 0.0], device=DEV, requires_grad=True)   # 3 px off: no overlap with the 2-px triangle
    opt = torch.optim.Adam([off], lr=0.2 * px)
    sched = torch.optim.lr_scheduler.ExponentialLR(opt, 0.99)
    for _ in range(400):
        opt.zero_grad()
        ((silhouette(_tri_at(0.0, 0.0) + torch.cat((off, off.new_zeros(1)))) - target) ** 2).sum().backward()
        opt.step()
        sched.step()
    assert off.detach().abs().max().item() < 0.1 * px, (off / px).tolist()


def test_renderer_fused_op_by_op_fill_back_and_camera_gradient():
    nr = _nr()
    v, f = _teapot()
    v, f = v.repeat(2, 1, 1), f.repeat(2, 1, 1)
    r = nr.Renderer()
    r.image_size = 96
    r.eye = nr.get_points_from_angles(2.732, 30, -15)
    fused = r.render_soft_fragments(v, f, sigma=1e-4, faces_per_pixel=6)
    r.fill_back = False
    for x, y in zip(fused, r.render_soft_fragments(v, f, sigma=1e-4, faces_per_pixel=6)):
        assert torch.equal(x, y)
    r.fused = False
    for x, y in zip(fused, r.render_soft_fragments(v, f, sigma=1e-4, faces_per_pixel=6)):
        assert torch.equal(x, y)
    r.fused = True
    assert (fused.pix_to_face >= 0).sum().item() > 5000
    vv = v.clone().requires_grad_(True)
    fr = r.render_soft_fragments(vv, f, sigma=1e-4, faces_per_pixel=6)
    ((fr.zbuf * _rand(fr.zbuf.shape, 101)).sum() + (fr.dists * 1e3).sum()).backward()
    assert torch.isfinite(vv.grad).all() and vv.grad.abs().max() > 0


def test_cuda_graph_capture_replays_bit_identically():
    nr = _nr()
    S, sigma, K = 64, 1e-3, 8
    faces = _special_faces(2, sigma, 111)
    fv = faces.clone().requires_grad_(True)
    up = _rand((2, S, S, K, 3), 112)

    def step():
        fr = nr.rasterize_soft_fragments(fv, S, sigma, K)
        (g,) = torch.autograd.grad((fr.bary_coords * up).sum() + fr.zbuf.sum() + fr.dists.sum(), fv)
        return fr, g

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            eager = step()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        cap = step()
    graph.replay()
    torch.cuda.synchronize()
    for x, y in zip(eager[0], cap[0]):
        assert torch.equal(x, y)
    assert rel_err(cap[1].cpu(), eager[1].cpu()) <= 1e-6
