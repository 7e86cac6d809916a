"""What the soft rasterizer's tile binning does with a scene, restated on the host for the tests that must know which of
its branches a scene reaches: the composite key width of the soft RGB's sort (nr_soft_rgb.cu, soft_rgb_layout) and a
float64 lower bound of every tile's list length (nr_soft.cuh, k_soft_setup).  The kernels stage a tile's entries
kThreads = 256 at a time, so a tile whose list holds more than 256 entries takes more than one staging round."""
import math

import torch

import oracles_soft as osoft

TILE = 16          # kTile
WIDE_TILES = 16    # kWideTiles: faces over more tiles go to the item's wide list
ROUND = 256        # kThreads: entries staged per round


def tiles_per_axis(S):
    return (S + TILE - 1) // TILE


def key_width(B, F, S):
    """(fbits, end_bit, 64-bit keys) of soft_rgb_layout: f takes fbits bits, below the segment (item, tile or wide list),
    and the last item's sentinel key ((B (ntiles + 1)) << fbits) - 1 sets the sort's end_bit; past 32 bits the keys are
    64-bit"""
    nt1 = tiles_per_axis(S) ** 2 + 1
    fbits = 1
    while (1 << fbits) <= F:
        fbits += 1
    max_key = ((B * nt1) << fbits) - 1
    end_bit = 1
    while end_bit < 64 and (max_key >> end_bit) != 0:
        end_bit += 1
    return fbits, end_bit, end_bit > 32


def tile_boxes(faces, S, sigma, near=0.1, far=100.0):
    """(ok, wide, tx0, tx1, ty0, ty1) [B,F] of every face: the tile box of its xy extent grown by the cut-off reach in
    float64, without the kernel's one-pixel guard, so each box is inside the kernel's (ok = takes part and reaches the
    image); wide = spans more than WIDE_TILES tiles here, so more there too: the face is on the item's wide list"""
    faces = faces.detach().to(torch.float64)
    reach = math.sqrt(osoft.cut(sigma)) * S / 2
    x, y = faces[..., 0], faces[..., 1]
    lim = S - 1
    c0 = torch.floor((x.amin(2) * S + lim) / 2 - reach).clamp_min(0)
    c1 = torch.ceil((x.amax(2) * S + lim) / 2 + reach).clamp_max(lim)
    r0 = torch.floor(lim - (y.amax(2) * S + lim) / 2 - reach).clamp_min(0)
    r1 = torch.ceil(lim - (y.amin(2) * S + lim) / 2 + reach).clamp_max(lim)
    ok = osoft.participates(faces, near, far) & (c0 <= c1) & (r0 <= r1)
    tx0, tx1 = (c0.nan_to_num(0) // TILE).long(), (c1.nan_to_num(0) // TILE).long()
    ty0, ty1 = (r0.nan_to_num(0) // TILE).long(), (r1.nan_to_num(0) // TILE).long()
    wide = ok & ((tx1 - tx0 + 1) * (ty1 - ty0 + 1) > WIDE_TILES)
    return ok, wide, tx0, tx1, ty0, ty1


def tile_entries_lower_bound(faces, S, sigma, near=0.1, far=100.0):
    """[B, ntiles] int64: a lower bound of the entries every (item, tile) stages, its own list plus the item's wide list
    (tile_boxes: a face wide here is on the wide list, which every tile of the item stages)"""
    ok, wide, tx0, tx1, ty0, ty1 = tile_boxes(faces, S, sigma, near, far)
    B = ok.shape[0]
    nt = tiles_per_axis(S)
    t = torch.arange(nt, device=ok.device)
    inx = (t[None, None] >= tx0[..., None]) & (t[None, None] <= tx1[..., None])      # [B,F,nt]
    iny = (t[None, None] >= ty0[..., None]) & (t[None, None] <= ty1[..., None])
    own = (ok & ~wide)[..., None, None] & iny[..., :, None] & inx[..., None, :]       # [B,F,nt(y),nt(x)]
    return own.sum(1).reshape(B, nt * nt) + wide.sum(1, keepdim=True)


def rounds(entries):
    """staging rounds of a tile with `entries` entries"""
    return (entries + ROUND - 1) // ROUND
