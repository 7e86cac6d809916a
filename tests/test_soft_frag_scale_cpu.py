"""CPU: the host side of tests/test_gpu_soft_frag_scale.py.  Its colliding-bucket scene is built from k_soft_frag_bwd's
table size and hash multiplier, restated in Python; these tests read both from csrc/nr_soft_frag.cu, so that a change
to either fails here rather than silently turning that scene into an ordinary one.  They also check the scenes
themselves: the permutation puts every face that can reach the chosen tile into the window of home buckets around the
wrap, and the dense field's float64 selection (oracles_soft_frag) gives tiles below and above the table's size."""
import math
import os
import re

import numpy as np
import torch

import oracles_soft_frag as ofrag
import test_gpu_soft_frag_scale as tfs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "neural_renderer_b200", "csrc", "nr_soft_frag.cu")


def test_table_size_and_hash_match_the_kernel():
    src = open(SRC).read()
    m = re.search(r"constexpr int kTable = (\d+);", src)
    assert m and int(m.group(1)) == tfs.K_TABLE, m and m.group(0)
    m = re.search(r"unsigned h = \(\(unsigned\)f \* (\d+)u\) >> (\d+);", src)
    assert m, "the home-bucket hash of k_soft_frag_bwd changed"
    assert int(m.group(1)) == tfs.HASH_MUL
    assert int(m.group(2)) == 32 - int(math.log2(tfs.K_TABLE))
    # linear probing that wraps from the last slot to the first
    assert "h = (h + 1) & (kTable - 1)" in src
    # home_bucket restates the kernel's 32-bit product
    f = np.array([0, 1, 2, 1023, 65535, 65536, 1 << 30, (1 << 31) - 1], dtype=np.int64)
    want = [((int(x) * tfs.HASH_MUL) & 0xFFFFFFFF) >> (32 - int(math.log2(tfs.K_TABLE))) for x in f]
    assert tfs.home_bucket(f).tolist() == want


def _tile_pixels(tile):
    ty, tx = tile
    S = tfs.S_DENSE
    return torch.tensor([(ty * 16 + i) * S + tx * 16 + j for i in range(16) for j in range(16)])


def test_windowed_scene_puts_the_tile_into_the_wrapping_window():
    S, sigma = tfs.S_DENSE, tfs.SIGMA_DENSE
    base = tfs.dense_field(2, 2)
    faces, counts = tfs.windowed(base, S, sigma, 3)
    assert min(counts) > 500
    for b in range(2):
        # a permutation of the item's faces
        a = np.sort(base[b].reshape(-1, 9).view(np.dtype((np.void, 36))).ravel())
        c = np.sort(faces[b].reshape(-1, 9).view(np.dtype((np.void, 36))).ravel())
        assert np.array_equal(a, c)
        # every float64 candidate at the tile's pixels is a face the permutation placed in the window
        cb, _, cf, _, _, _ = ofrag.candidates(torch.from_numpy(faces[b:b + 1]), S, sigma, pix=_tile_pixels(tfs.WINDOW_TILE))
        ids = cf.unique().numpy()
        assert ids.size > 300
        assert np.all(tfs.tile_reach(faces[b:b + 1], S, sigma, tfs.WINDOW_TILE)[0][ids])
        home = tfs.home_bucket(ids).astype(np.int64)
        hist = np.bincount(home, minlength=tfs.K_TABLE)
        inside = (np.arange(tfs.K_TABLE) + tfs.WINDOW // 2) % tfs.K_TABLE < tfs.WINDOW
        assert hist[~inside].sum() == 0 and hist[inside].sum() == ids.size
        # more faces start above the wrap than there are slots above it: the probe chain runs on into slot 0
        assert hist[tfs.K_TABLE - tfs.WINDOW // 2:].sum() > tfs.WINDOW // 2
        assert hist[0] > 0 and hist[tfs.K_TABLE - 1] > 0


def test_dense_field_tiles_below_and_above_the_table():
    """the float64 selection (the first K candidates by (zp, f)) at two tiles of one item: the sparse column stays
    below the table's size at K 16 and the dense column passes it"""
    S, sigma = tfs.S_DENSE, tfs.SIGMA_DENSE
    faces = torch.from_numpy(tfs.dense_field(1, 1))
    got = {}
    for tile in ((1, 1), (1, 3)):
        b, pp, f, zp, _, _ = ofrag.candidates(faces, S, sigma, pix=_tile_pixels(tile))
        order = ofrag.sort_key(b, pp, f, zp)
        pp, f = pp[order], f[order]
        _, inv, cnt = torch.unique_consecutive(pp, return_inverse=True, return_counts=True)
        rank = torch.arange(pp.numel()) - (torch.cumsum(cnt, 0) - cnt)[inv]
        got[tile] = f[rank < 16].unique().numel()
    assert tfs.K_TABLE // 2 < got[(1, 1)] <= tfs.K_TABLE, got
    assert got[(1, 3)] > tfs.K_TABLE, got
