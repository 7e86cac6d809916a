"""float64 oracles of the interior vertex gradient of the RGB image (include/nr_b200.h, NR_GRAD_INTERIOR).

Two formulations of the same derivative, on the product's face_index_map / weight_map:
  rgb_held64       the lit sample of every covered raster pixel, differentiable in `faces`: the weights are
                   w = a(x) + (w_saved - a(x)).detach() (the clamp and renormalisation held fixed, as oracles_attr.interp64),
                   the perspective weights l_k follow from them, and the texel cell, the level of detail and the clamp
                   gates come from `select` (detached).  Autograd of sum(g * rgb) is the reference derivative.
  interior_grad64  the header's closed form: G_k = sum_c g_c (L_c E_kc + [smooth] C_kc s_c) with E_kc written out per
                   sampler, chained to the vertices with D_k, P_m as the header states it.
`select` takes the sampler's cell, gates and level from fp32 values formed in the product's operation order, so on the
GPU the oracle differentiates the cell the product picked."""
import torch

from oracles import lod64
from oracles_attr import _setup


class Tex:
    """the texture of a call: kind 'cube' (cubes [1|B,F',ts,ts,ts,3], eps), 'bilinear' / 'trilinear' (levels = list of
    [1|B,H_l,W_l,3] images, level 0 first; uvs [1|B,F',3,2]); fill_back = faces [F/2, F) are reversed copies"""

    def __init__(self, kind, data, uvs=None, eps=1e-4, fill_back=False):
        self.kind, self.data, self.uvs, self.eps, self.fill_back = kind, data, uvs, eps, fill_back


def _pixels(faces, fim, wmap, S):
    cov, fi, bidx, f, a, inv, P = _setup(faces, fim, S)
    wm = wmap.double().permute(0, 2, 3, 1)
    pt = (wm[..., None] * P).sum(-2).detach()
    aw = (inv[..., :2] * pt[..., None, :]).sum(-1) + inv[..., 2]
    w = torch.where(cov[..., None], aw + (wm - aw).detach(), a)  # value w_saved, vertex derivative that of a
    return cov, fi, bidx, f, inv, w, wm


def _float_le(d):
    f = torch.tensor(d, dtype=torch.float32)
    return f if float(f) <= d else torch.nextafter(f, torch.tensor(-float("inf")))


def select(faces, fim, wmap, S, tex, dmap=None):
    """the sampler's detached choices per covered raster pixel, from fp32 values in the product's operation order:
    cubes: (cell i [B,S,S,3], gate, clamped t); images: per level (ix, iy, in_u, in_v, clamped uv) and the level weights"""
    B = faces.shape[0]
    fi = fim.clamp(min=0).long()
    bidx = torch.arange(B, device=fim.device)[:, None, None].expand_as(fi)
    z32 = faces.detach()[..., 2][bidx, fi].float()
    z32 = torch.where((fim >= 0)[..., None], z32, torch.ones_like(z32))
    w32 = wmap.float().permute(0, 2, 3, 1)
    if dmap is None:
        q = w32 / z32
        zp32 = 1.0 / ((q[..., 0] + q[..., 1]) + q[..., 2])
    else:
        zp32 = dmap.float()
    zp32 = zp32[..., None]
    out = {}
    if tex.kind == "cube":
        ts = tex.data.shape[2]
        tmax = (ts - 1) - tex.eps
        cmp_, val = _float_le(tmax).to(fim.device), torch.tensor(tmax, dtype=torch.float32, device=fim.device)
        t = (w32 * (ts - 1)) * (zp32 / z32)
        gate = (t >= 0) & (t <= cmp_)
        tc = torch.where(t > cmp_, val, torch.nan_to_num(t.clamp(min=0), nan=0.0))
        i = tc.long()  # cvt.rzi of a non-negative value
        top = i > ts - 2
        out.update(i=torch.where(top, ts - 2, i), gate=gate, tcl=torch.where(top, float(ts - 1), tc.double()))
        return out
    uvk = _uv_corners(tex, fi, bidx).float()
    lam32 = w32 * (zp32 / z32)
    uv = (lam32[..., 0, None] * uvk[..., 0, :] + lam32[..., 1, None] * uvk[..., 1, :]) + lam32[..., 2, None] * uvk[..., 2, :]
    inside = (uv >= 0) & (uv <= 1)
    ucl = torch.nan_to_num(uv.clamp(0, 1), nan=0.0)
    lv = []
    for img in tex.data:
        h, wd = img.shape[1:3]
        px, py = (ucl[..., 0] * (wd - 1)).double(), (ucl[..., 1] * (h - 1)).double()
        lv.append((px.floor().long().clamp(max=wd - 1), py.floor().long().clamp(max=h - 1)))
    out.update(inside=inside, ucl=ucl.double(), lv=lv)
    if tex.kind == "trilinear":
        Ht, Wt = tex.data[0].shape[1:3]
        L = len(tex.data)
        lod = lod64(faces.detach(), fim, wmap, zp32[..., 0], uvk.double(), S, Ht, Wt, L)
        l0 = lod.floor()
        out.update(l0=l0.long(), l1=(l0.long() + 1).clamp(max=L - 1), f=lod - l0)
    return out


def _uv_corners(tex, fi, bidx):
    B = bidx.shape[0]
    uvs = tex.uvs.double().expand(B, -1, -1, -1)
    if tex.fill_back:
        uvs = torch.cat((uvs, uvs.flip(2)), dim=1)
    return uvs[bidx, fi]  # [B,S,S,3,2]


def _cube_texels(tex, fi, bidx, i):
    """the 8 texels of the cell, T [B,S,S,8,3] (corner pn: bit k = +1 on axis k)"""
    cubes = tex.data.double()
    B = bidx.shape[0]
    cubes = cubes.expand(B, *cubes.shape[1:])
    cube, rev = fi, torch.zeros_like(fi, dtype=torch.bool)
    if tex.fill_back:
        half = cubes.shape[1]
        rev = fi >= half
        cube = torch.where(rev, fi - half, fi)
    T = []
    for pn in range(8):
        i0, i1, i2 = (i[..., k] + ((pn >> k) & 1) for k in range(3))
        a0, a2 = torch.where(rev, i2, i0), torch.where(rev, i0, i2)
        T.append(cubes[bidx, cube, a0, i1, a2])
    return torch.stack(T, dim=-2)


def _bilinear(img, u, v, ix, iy, bidx):
    """bilinear sample and (d / du, d / dv) of img [B,h,w,3] at (u, v) in the cell (ix, iy) (no clamp gates)"""
    h, wd = img.shape[1:3]
    px, py = u * (wd - 1), v * (h - 1)
    wx1, wy1 = (px - ix)[..., None], (py - iy)[..., None]
    wx0, wy0 = 1 - wx1, 1 - wy1
    x1, y1 = (ix + 1).clamp(max=wd - 1), (iy + 1).clamp(max=h - 1)
    r0, r1 = h - 1 - iy, h - 1 - y1
    T00, T10, T01, T11 = img[bidx, r0, ix], img[bidx, r0, x1], img[bidx, r1, ix], img[bidx, r1, x1]
    s = wx0 * wy0 * T00 + wx0 * wy1 * T01 + wx1 * wy0 * T10 + wx1 * wy1 * T11
    du = (wd - 1) * (wy0 * (T10 - T00) + wy1 * (T11 - T01))
    dv = (h - 1) * (wx0 * (T01 - T00) + wx1 * (T11 - T10))
    return s, du, dv


def _sample(lam, sel, tex, fi, bidx):
    """unlit sample s [B,S,S,3] at the weights lam (float64, differentiable) and E [B,S,S,3 (k),3 (c)] = d s / d l_k"""
    if tex.kind == "cube":
        ts = tex.data.shape[2]
        T = _cube_texels(tex, fi, bidx, sel["i"])
        t = torch.where(sel["gate"], lam * (ts - 1), sel["tcl"])
        hi = t - sel["i"]
        lo = 1 - hi
        wgt = lambda pn, k: hi[..., k] if (pn >> k) & 1 else lo[..., k]
        s = sum((wgt(pn, 0) * wgt(pn, 1) * wgt(pn, 2))[..., None] * T[..., pn, :] for pn in range(8))
        E = []
        for k in range(3):
            j, m = (k + 1) % 3, (k + 2) % 3
            d = sum((wgt(pn, j) * wgt(pn, m))[..., None] * (T[..., pn | (1 << k), :] - T[..., pn, :])
                    for pn in range(8) if not (pn >> k) & 1)
            E.append(sel["gate"][..., k, None] * (ts - 1) * d)
        return s, torch.stack(E, dim=-2)
    uvk = _uv_corners(tex, fi, bidx)
    uv = (lam[..., None] * uvk).sum(-2)
    inside = sel["inside"]
    uvu = torch.where(inside, uv, sel["ucl"])
    B = bidx.shape[0]
    levels = [l.double().expand(B, -1, -1, -1) for l in tex.data]

    def level(n):
        ix, iy = sel["lv"][n]
        s, du, dv = _bilinear(levels[n], uvu[..., 0], uvu[..., 1], ix, iy, bidx)
        du, dv = inside[..., 0, None] * du, inside[..., 1, None] * dv
        E = du[..., None, :] * uvk[..., 0, None] + dv[..., None, :] * uvk[..., 1, None]  # [B,S,S,3 (k),3 (c)]
        return s, E
    if tex.kind == "bilinear":
        return level(0)
    per = [level(n) for n in range(len(levels))]
    def pick(l, q):  # level l [B,S,S] of output q of every pixel
        t = torch.stack([p[q] for p in per], 0)
        idx = l.reshape(1, *l.shape, *([1] * (t.dim() - 1 - l.dim()))).expand(1, *t.shape[1:])
        return t.gather(0, idx)[0]
    f = sel["f"]
    fs, fE = f[..., None], f[..., None, None]
    return (1 - fs) * pick(sel["l0"], 0) + fs * pick(sel["l1"], 0), (1 - fE) * pick(sel["l0"], 1) + fE * pick(sel["l1"], 1)


def _light(lam, fi, bidx, light, corner):
    if corner is not None:
        C = corner.double()[bidx, fi]  # [B,S,S,3 (k),3 (c)]
        return (lam[..., None] * C).sum(-2), C
    if light is not None:
        return light.double()[bidx, fi], None
    return None, None


def rgb_held64(faces, fim, wmap, S, tex, sel, light=None, corner=None):
    """the lit sample of every covered raster pixel [B,S,S,3] (0 elsewhere), differentiable in `faces` [B,F,3,3]"""
    cov, fi, bidx, f, inv, w, _ = _pixels(faces, fim, wmap, S)
    q = w / f[..., 2]
    lam = q / q.sum(-1, keepdim=True)
    s, _ = _sample(lam, sel, tex, fi, bidx)
    L, _ = _light(lam, fi, bidx, light, corner)
    rgb = s * L if L is not None else s
    return torch.where(cov[..., None], rgb, torch.zeros_like(rgb))


def interior_grad64(faces, fim, wmap, S, tex, sel, g, light=None, corner=None):
    """the header's closed form: d sum(g * rgb) / d faces [B,F,3,3] through l_k; g [B,3,S,S] raster layout"""
    with torch.no_grad():
        cov, fi, bidx, f, inv, _, wm = _pixels(faces, fim, wmap, S)
        z = f[..., 2]
        zp = 1.0 / (wm / z).sum(-1)
        lam = wm * zp[..., None] / z
        s, E = _sample(lam, sel, tex, fi, bidx)
        L, C = _light(lam, fi, bidx, light, corner)
        gp = g.double().permute(0, 2, 3, 1)  # [B,S,S,3]
        h = gp * L if L is not None else gp
        G = (E * h[..., None, :]).sum(-1)  # [B,S,S,3 (k)]
        if C is not None:
            G = G + (C * (gp * s)[..., None, :]).sum(-1)
        D = G[..., 1:] - G[..., :1]
        Gd = []
        for d in (0, 1):
            qd = inv[..., d] / z
            ld = zp[..., None] * (qd - lam * qd.sum(-1, keepdim=True))
            Gd.append((D * ld[..., 1:]).sum(-1))
        P = (lam * G).sum(-1, keepdim=True) - G
        gf = torch.stack((-wm * Gd[0][..., None] * S / 2, -wm * Gd[1][..., None] * S / 2, lam / z * P), dim=-1)
        B, F = faces.shape[:2]
        flat = (bidx * F + fi)[cov]
        res = torch.zeros((B * F, 3, 3), dtype=torch.float64, device=faces.device)
        res.index_add_(0, flat, gf[cov])
        return res.reshape(B, F, 3, 3)


def faces_to_vertices(grad_faces, indices, Nv):
    """the vertices_to_faces backward of a [B,F,3,3] gradient: [B,Nv,3] (indices [F,3] / [1|B,F,3])"""
    B = grad_faces.shape[0]
    idx = indices.long().expand(B, -1, -1) if indices.dim() == 3 else indices.long()[None].expand(B, -1, -1)
    out = torch.zeros((B, Nv, 3), dtype=grad_faces.dtype, device=grad_faces.device)
    out.scatter_add_(1, idx.reshape(B, -1, 1).expand(-1, -1, 3), grad_faces.reshape(B, -1, 3))
    return out
