"""CPU: the sparse mode of the soft oracles (pixel sets, the exact cull, chunks of items and faces) against their dense
mode, and the host-side restatements of the tile binning (tests/soft_binning.py) that tests/test_gpu_soft_scale.py relies
on to show which branches of the kernels its scenes reach."""
import math

import pytest
import torch

import oracles
import oracles_soft as osoft
import oracles_soft_rgb as orgb
import oracles_soft_uv as ouv
import soft_binning as sb

S = 24
SIGMA, GAMMA = 1e-3, 1e-2


def _faces(B, F, seed):
    from neural_renderer_b200 import synthetic
    return torch.from_numpy(synthetic.triangle_soup(B, F, seed=seed, size=(0.05, 0.4), duplicates=False)).double()


def _pix(B, seed, per_item):
    """a pixel set with every corner and pixels on each border, plus random pixels"""
    g = torch.Generator().manual_seed(seed)
    border = torch.tensor([0, S - 1, S * (S - 1), S * S - 1, 5, S * 7, S * 9 + S - 1, S * (S - 1) + 11])
    if not per_item:
        return torch.cat((border, torch.randint(0, S * S, (40,), generator=g)))
    return torch.stack([torch.cat((border, torch.randint(0, S * S, (40,), generator=g))) for _ in range(B)])


def _at(dense, pix, B):
    """dense [B,...,S,S] at the pixel set: [B,...,P]"""
    flat = dense.reshape(*dense.shape[:-2], S * S)
    idx = pix.expand(B, -1) if pix.dim() == 1 else pix
    idx = idx.reshape(B, *([1] * (flat.dim() - 2)), -1).expand(*flat.shape[:-1], -1)
    return torch.gather(flat, -1, idx)


def _compare(fn, leaves, pix, B):
    """values to 1e-13 and autograd gradients to 1e-12 of fn(leaves, pix) against fn(leaves, None) at the pixels"""
    g = torch.Generator().manual_seed(7)
    ws = None
    out = {}
    for mode in ("dense", "sparse"):
        xs = [x.clone().requires_grad_(True) for x in leaves]
        vals = fn(xs, None if mode == "dense" else pix)
        if mode == "dense":
            vals = tuple(_at(v, pix, B) for v in vals)
        if ws is None:
            ws = [torch.randn(v.shape, generator=g, dtype=torch.float64) for v in vals]
        loss = sum((v * w).sum() for v, w in zip(vals, ws))
        grads = torch.autograd.grad(loss, xs, allow_unused=True)
        out[mode] = (vals, [torch.zeros_like(x) if gx is None else gx for x, gx in zip(xs, grads)])
    for a, b in zip(out["sparse"][0], out["dense"][0]):
        assert a.shape == b.shape
        assert (a - b).abs().max().item() <= 1e-13
    for a, b in zip(out["sparse"][1], out["dense"][1]):
        assert (a - b).abs().max().item() <= 1e-12 * max(1.0, b.abs().max().item())
    return out["sparse"]


@pytest.mark.parametrize("per_item", [False, True])
def test_sparse_silhouettes_equal_the_dense_oracle(per_item):
    B = 2
    faces = _faces(B, 18, seed=1)
    pix = _pix(B, 2, per_item)
    _compare(lambda xs, p: (osoft.soft_silhouettes(xs[0], S, SIGMA, pix=p),) if p is not None else
             (osoft.soft_silhouettes(xs[0], S, SIGMA),), [faces], pix, B)


@pytest.mark.parametrize("shared_tex", [False, True])
@pytest.mark.parametrize("per_item", [False, True])
def test_sparse_cube_rgb_equals_the_dense_oracle(shared_tex, per_item):
    B, F, ts = 2, 16, 3
    faces = _faces(B, F, seed=3)
    g = torch.Generator().manual_seed(4)
    tex = torch.rand((1 if shared_tex else B), F, ts, ts, ts, 3, generator=g, dtype=torch.float64)
    fl = 0.5 + torch.rand(B, F, 3, generator=g, dtype=torch.float64)
    pix = _pix(B, 5, per_item)
    bg = (0.2, 0.4, 0.6)

    def fn(xs, p):
        rgb, alpha = orgb.soft_rgb(xs[0], xs[1], S, SIGMA, GAMMA, background=bg, face_light=xs[2], pix=p)
        return rgb, alpha
    _compare(fn, [faces, tex, fl], pix, B)


@pytest.mark.parametrize("tri", [False, True])
@pytest.mark.parametrize("shared", [False, True])
def test_sparse_uv_equals_the_dense_oracle(tri, shared):
    B, F = 2, 16
    faces = _faces(B, F, seed=6)
    g = torch.Generator().manual_seed(8)
    img = torch.rand((1 if shared else B), 13, 10, 3, generator=g, dtype=torch.float64)
    uvs = torch.rand((1 if shared else B), F, 3, 2, generator=g, dtype=torch.float64) * 1.1 - 0.05
    fl = 0.5 + torch.rand(B, F, 3, generator=g, dtype=torch.float64)
    pix = _pix(B, 9, not shared)

    def fn(xs, p):
        if tri:
            tex, hw = torch.cat([x.reshape(x.shape[0], -1, 3) for x in oracles.pyramid64(xs[1])], 1), (13, 10)
        else:
            tex, hw = xs[1], None
        return ouv.soft_uv(xs[0], tex, xs[2], S, SIGMA, GAMMA, face_light=xs[3], hw=hw, pix=p)
    _compare(fn, [faces, img, uvs, fl], pix, B)


def test_sparse_chunks_of_items_and_faces_change_nothing():
    """a budget that forces one item per chunk and a few faces per chunk gives what one chunk gives"""
    B, F, ts = 3, 20, 2
    faces = _faces(B, F, seed=10)
    tex = torch.rand(B, F, ts, ts, ts, 3, generator=torch.Generator().manual_seed(11), dtype=torch.float64)
    pix = _pix(B, 12, True)
    p = pix.shape[1]

    def run(budget):
        def terms(b0, b1, idx, fc, pp):
            return orgb.cube_terms(fc, osoft.take(tex, b0, b1, idx), pp, SIGMA, 0.1, 100.0, 1e-4, None, 1.0)
        return osoft.sparse_eval(faces, S, pix, SIGMA, 0.1, 100.0, 1.0, terms, orgb.softmax_blend(GAMMA, (0.1, 0.2, 0.3)),
                                 budget=budget)
    a1, r1 = run(1 << 24)
    a2, r2 = run(3 * p)
    assert (a1 - a2).abs().max() <= 1e-15 and (r1 - r2).abs().max() <= 1e-14


def test_culled_faces_get_exactly_zero_gradient():
    """faces out of reach of every chosen pixel, faces that take no part (NaN, inf, beyond far, before near) and faces
    in reach but not on at any chosen pixel: the culled ones are never evaluated, so autograd gives them exactly 0"""
    B, ts = 2, 2
    real = _faces(B, 10, seed=13)
    far_away = real[:, :3].clone()
    far_away[..., 0] += 5.0                               # off the image, far beyond the reach
    bad = real[:, :4].clone()
    bad[:, 0, 1, 0] = float("nan")
    bad[:, 1, 2, 1] = float("inf")
    bad[:, 2, 0, 2] = 150.0
    bad[:, 3, 1, 2] = 0.05
    faces = torch.cat((real, far_away, bad), 1)
    F = faces.shape[1]
    tex = torch.rand(B, F, ts, ts, ts, 3, generator=torch.Generator().manual_seed(14), dtype=torch.float64)
    pix = _pix(B, 15, False)
    f = faces.clone().requires_grad_(True)
    t = tex.clone().requires_grad_(True)
    rgb, alpha = orgb.soft_rgb(f, t, S, SIGMA, GAMMA, pix=pix)
    (rgb.sum() + alpha.sum()).backward()
    keep = osoft.in_reach(faces, osoft.pixel_set(S, pix, B), SIGMA, 0.1, 100.0)
    assert not keep[:, 10:].any() and keep[:, :10].any()
    assert torch.all(f.grad[~keep] == 0) and torch.all(t.grad[~keep] == 0)
    assert torch.isfinite(f.grad).all() and f.grad[keep].abs().max() > 0


def test_cull_keeps_every_face_that_is_on_at_a_chosen_pixel():
    """the cull against the dense terms: a face on at any chosen pixel is kept, over several cut-off scales"""
    B = 2
    faces = _faces(B, 40, seed=16)
    pix = _pix(B, 17, True)
    p = osoft.pixel_set(S, pix, B)
    for sigma in (1e-5, 1e-3, 1e-2):
        for cs in (1 - 1e-5, 1.0, 1 + 1e-5):
            d2, inside = osoft.face_terms(faces, p)
            on = osoft.participates(faces, 0.1, 100.0)[..., None] & (inside | (d2 <= osoft.cut(sigma) * cs))
            keep = osoft.in_reach(faces, p, sigma, 0.1, 100.0, cs)
            assert torch.all(keep | ~on.any(-1))


def test_key_width_follows_the_layout_rule():
    assert sb.key_width(2, 65535, 2049) == (16, 32, False)
    assert sb.key_width(2, 65536, 2049) == (17, 33, True)
    # one item of 65536 faces at 2049 fits 32 bits again; the benchmark's shape is 32-bit
    assert sb.key_width(1, 65536, 2049)[2] is False
    assert sb.key_width(64, 5000, 256)[2] is False
    for B, F, S_ in [(1, 1, 1), (3, 7, 33), (64, 5000, 256), (2, 65536, 2049), (7, 100000, 4000)]:
        fbits, end_bit, wide = sb.key_width(B, F, S_)
        nt1 = sb.tiles_per_axis(S_) ** 2 + 1
        assert F - 1 <= (1 << fbits) - 2                 # every face index is below the sentinel's low bits
        assert ((B * nt1) << fbits) - 1 < (1 << end_bit)  # every key fits the sort's bits
        assert wide == (end_bit > 32)


def _brute_lower_bound(faces, S, sigma):
    """the lower bound face by face and tile by tile, in plain Python floats"""
    B, F = faces.shape[:2]
    nt = sb.tiles_per_axis(S)
    reach = math.sqrt(osoft.cut(sigma)) * S / 2
    out = torch.zeros(B, nt * nt, dtype=torch.int64)
    part = osoft.participates(faces, 0.1, 100.0)
    for b in range(B):
        for f in range(F):
            if not part[b, f]:
                continue
            xs, ys = faces[b, f, :, 0].tolist(), faces[b, f, :, 1].tolist()
            c0 = max(math.floor((min(xs) * S + S - 1) / 2 - reach), 0)
            c1 = min(math.ceil((max(xs) * S + S - 1) / 2 + reach), S - 1)
            r0 = max(math.floor(S - 1 - (max(ys) * S + S - 1) / 2 - reach), 0)
            r1 = min(math.ceil(S - 1 - (min(ys) * S + S - 1) / 2 + reach), S - 1)
            if c0 > c1 or r0 > r1:
                continue
            tiles = [ty * nt + tx for ty in range(r0 // 16, r1 // 16 + 1) for tx in range(c0 // 16, c1 // 16 + 1)]
            if len(tiles) > sb.WIDE_TILES:
                out[b] += 1
            else:
                out[b, tiles] += 1
    return out


def test_tile_lower_bound_counts_boxes_and_the_wide_list():
    S_, sigma = 80, 1e-4
    faces = _faces(2, 60, seed=18)
    faces[0, 3, 0, 2] = 200.0                  # takes no part
    faces[1, 5] = torch.tensor([[-1.0, -1.0, 2.0], [1.0, -1.0, 2.0], [0.0, 1.0, 2.0]])   # wide
    faces[1, 6] = torch.tensor([[5.0, 5.0, 2.0], [5.1, 5.0, 2.0], [5.0, 5.1, 2.0]])       # off the image
    lb = sb.tile_entries_lower_bound(faces, S_, sigma)
    assert torch.equal(lb, _brute_lower_bound(faces, S_, sigma))
    assert lb[1].min() >= 1                    # the wide face is on every tile's list
    assert sb.rounds(torch.tensor([0, 1, 256, 257, 513])).tolist() == [0, 1, 1, 2, 3]
