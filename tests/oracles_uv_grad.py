"""float64 oracles of the face_uvs gradient of the texture-image samplers (include/nr_b200.h, grad_face_uvs).

The same samplers as oracles.oracle_rgb / oracle_trilinear, on the product's own face_index_map / weight_map / depth_map,
and additionally differentiable in the UV corners: the texel positions, the cell and the clamp mask are the product's
fp32 ones, and a float64 straight-through term (px32 + (px64 - px64.detach()), see _uv_straight_through) gives autograd
the documented derivative -- the level of detail, the perspective weights and the clamp held fixed.  `uvs` is a float64
tensor with requires_grad; its .grad after backward is the reference face_uvs gradient."""
import torch

from oracles import _bg, lod64, pyramid64


def _uv_straight_through(uv32, uvk, w, zp, z):
    """float64 zero-valued term whose derivative in the UV corners is that of the pixel's uv, uv = sum_k l_k uv_k with
    l_k = w_k zp / z_k (float64), masked by the clamp (0 outside [0,1] and for NaN)."""
    lam = w.double() * (zp.double() / z.double())
    uv64 = (lam[..., None] * uvk).sum(-2)                             # [B,S,S,2]
    inside = (uv32 >= 0) & (uv32 <= 1)
    return torch.where(inside, uv64 - uv64.detach(), torch.zeros_like(uv64))


def _pixel_uvs(faces, fim, wmap, dmap, uvs, fill_back, z64):
    """(bidx, fi, uvk [B,S,S,3,2] differentiable, the fp32 uv before the clamp, the straight-through term)"""
    dev = fim.device
    B = faces.shape[0]
    S = fim.shape[-1]
    uvs = uvs.double().expand(B, -1, -1, -1)
    if fill_back:
        uvs = torch.cat((uvs, uvs.flip(2)), dim=1)                     # a fill_back copy: corners reversed
    fi = fim.clamp(min=0).long()
    bidx = torch.arange(B, device=dev)[:, None, None].expand(B, S, S)
    z = (faces.double() if z64 else faces)[..., 2][bidx, fi]
    # an uncovered pixel reads face 0, which may have a zero depth (an out-of-range index): keep 0 * inf out of autograd
    z = torch.where((fim >= 0)[..., None], z, torch.ones_like(z))
    w = wmap.permute(0, 2, 3, 1)
    zp = dmap[..., None]
    uvk = uvs[bidx, fi]
    # the pixel's uv in fp32 with the sampler's pinned operation order, as the image oracles form it
    lam32 = w.float() * (zp.float() / z.float())
    u32 = uvk.detach().float()
    uv_raw = (lam32[..., 0, None] * u32[..., 0, :] + lam32[..., 1, None] * u32[..., 1, :]) + lam32[..., 2, None] * u32[..., 2, :]
    return bidx, fi, uvk, uv_raw, _uv_straight_through(uv_raw, uvk, w, zp, z)


def _bilinear(img, uv, st, bidx, lt):
    """bilinear sample of img [B,h,w,3] at the fp32 clamped uv, with the straight-through term added to the positions"""
    h, wd = img.shape[1:3]
    px, py = (uv[..., 0] * (wd - 1)).double(), (uv[..., 1] * (h - 1)).double()
    ix, iy = px.floor().long().clamp(max=wd - 1), py.floor().long().clamp(max=h - 1)
    px, py = px + st[..., 0] * (wd - 1), py + st[..., 1] * (h - 1)      # exactly 0 in value: the cell stays the product's
    wx1, wy1 = px - ix, py - iy
    wx0, wy0 = 1 - wx1, 1 - wy1
    x1, y1 = (ix + 1).clamp(max=wd - 1), (iy + 1).clamp(max=h - 1)
    r0, r1 = h - 1 - iy, h - 1 - y1

    def tap(r, c):
        t = img[bidx, r, c]
        return t * lt if lt is not None else t
    return ((wx0 * wy0)[..., None] * tap(r0, ix) + (wx0 * wy1)[..., None] * tap(r1, ix)
            + (wx1 * wy0)[..., None] * tap(r0, x1) + (wx1 * wy1)[..., None] * tap(r1, x1))


def oracle_rgb_uv_grad(faces, fim, wmap, dmap, uvs, image, light, bg, fill_back, aa):
    """bilinear sampler (oracles.oracle_rgb), differentiable in `uvs` [1|B,F',3,2]; returns the API rgb [B,3,H,W]"""
    bidx, fi, _, uv_raw, st = _pixel_uvs(faces, fim, wmap, dmap, uvs, fill_back, z64=False)
    img = image.double().expand(faces.shape[0], -1, -1, -1)
    lt = light.double()[bidx, fi] if light is not None else None
    rgb = _bilinear(img, torch.nan_to_num(uv_raw.clamp(0, 1)), st, bidx, lt)
    rgb = torch.where((fim >= 0)[..., None], rgb, _bg(bg, fim.device)).permute(0, 3, 1, 2)
    return torch.nn.functional.avg_pool2d(rgb, 2, 2) if aa else rgb


def oracle_trilinear_uv_grad(faces, fim, wmap, dmap, uvs, image, light, bg, fill_back, aa):
    """trilinear sampler (oracles.oracle_trilinear: float64 pyramid and level of detail), differentiable in `uvs`; the
    level of detail is a constant.  Returns the API rgb [B,3,H,W]."""
    Ht, Wt = image.shape[1:3]
    return oracle_trilinear_levels_uv_grad(faces, fim, wmap, dmap, uvs, pyramid64(image.double()), Ht, Wt, light, bg,
                                           fill_back, aa)


def oracle_trilinear_levels_uv_grad(faces, fim, wmap, dmap, uvs, levels, Ht, Wt, light, bg, fill_back, aa, lod_fn=None):
    """oracle_trilinear_uv_grad on given pyramid levels [1|B,H_l,W_l,3] (e.g. oracles.unpack_pyramid of the packed
    `textures`); the level of detail from `lod_fn` (default oracles.lod64)"""
    B = faces.shape[0]
    S = fim.shape[-1]
    levels = [l.double().expand(B, -1, -1, -1) for l in levels]
    L = len(levels)
    bidx, fi, uvk, uv_raw, st = _pixel_uvs(faces, fim, wmap, dmap, uvs, fill_back, z64=True)
    lod = (lod_fn or lod64)(faces, fim, wmap, dmap, uvk.detach(), S, Ht, Wt, L)
    lt = light.double()[bidx, fi] if light is not None else None
    uv = torch.nan_to_num(uv_raw.clamp(0, 1))
    samples = torch.stack([_bilinear(l, uv, st, bidx, lt) for l in levels], dim=0)  # [L,B,S,S,3]
    l0 = lod.floor()
    f = (lod - l0)[..., None]
    l0 = l0.long()
    l1 = (l0 + 1).clamp(max=L - 1)
    pick = lambda l: samples.gather(0, l[None, ..., None].expand(1, B, S, S, 3))[0]
    rgb = (1 - f) * pick(l0) + f * pick(l1)
    rgb = torch.where((fim >= 0)[..., None], rgb, _bg(bg, fim.device)).permute(0, 3, 1, 2)
    return torch.nn.functional.avg_pool2d(rgb, 2, 2) if aa else rgb
