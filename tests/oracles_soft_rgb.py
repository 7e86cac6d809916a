"""Float64 oracle of the soft RGB (include/nr_b200.h, nr_b200_soft_rgb_args): dense over every pixel x every face,
differentiable with torch autograd.  Reuses the soft silhouettes' distance field and participation test
(oracles_soft.face_terms / participates); the cube sampler is trilinear with the cell held by floor.  No binning, no
tiles, no sort, no running max: zmax is taken over all faces at once."""
import math

import torch

import oracles_soft as osoft

BG_DEPTH = 1e-3  # NR_SOFT_BG_DEPTH


def edge_functions(faces, p):
    """c_k [B,F,3,P] = (v_k+1 - v_k) x (p - v_k), p [P,2] or [B,P,2]"""
    a = faces[..., :2]
    e = a.roll(-1, dims=2) - a
    dp = osoft.points(p) - a[:, :, :, None]
    ee = e[:, :, :, None]
    return ee[..., 0] * dp[..., 1] - ee[..., 1] * dp[..., 0]


def doubled_area(faces):
    v = faces[..., :2]
    return (v[:, :, 1, 0] - v[:, :, 0, 0]) * (v[:, :, 2, 1] - v[:, :, 0, 1]) - \
        (v[:, :, 1, 1] - v[:, :, 0, 1]) * (v[:, :, 2, 0] - v[:, :, 0, 0])


def sample_cubes(textures, t, ts):
    """trilinear sample [B,F,P,3] of cubes [Bt,F,ts,ts,ts,3] at texture coordinates t [B,F,P,3] (already clamped); the
    cell is floor(t), moved down to ts - 2 at the top edge, and held fixed (no gradient through it)"""
    B, F, P = t.shape[:3]
    Bt = textures.shape[0]
    i = torch.floor(t.detach()).clamp(max=ts - 2).long()
    fr = t - i.to(t.dtype)
    cubes = textures.expand(B, -1, -1, -1, -1, -1).reshape(B, F, ts * ts * ts, 3) if Bt == 1 else \
        textures.reshape(B, F, ts * ts * ts, 3)
    out = 0
    for pn in range(8):
        d = [(pn >> k) & 1 for k in range(3)]
        w = 1
        for k in range(3):
            w = w * (fr[..., k] if d[k] else 1 - fr[..., k])
        idx = ((i[..., 0] + d[0]) * ts + (i[..., 1] + d[1])) * ts + (i[..., 2] + d[2])     # [B,F,P]
        tap = torch.gather(cubes, 2, idx.reshape(B, F, P, 1).expand(-1, -1, -1, 3).reshape(B, F, P, 3))
        out = out + w[..., None] * tap
    return out


def bary_terms(faces, p, sigma, near, far, cut_scale):
    """what the soft RGB oracles share per (item, face, pixel) of faces [B,F,3,3] float64 at p [P,2] / [B,P,2]: x, on,
    valid (on and a nonzero area), the clipped barycentrics l [B,F,3,P] and the perspective-correct depth zp [B,F,P]"""
    part = osoft.participates(faces, near, far)
    d2, inside = osoft.face_terms(faces, p)                               # [B,F,P]
    x = torch.where(inside, d2 / sigma, -d2 / sigma)
    on = part[..., None] & (inside | (d2 <= osoft.cut(sigma) * cut_scale))
    A = doubled_area(faces)[..., None]                                     # [B,F,1]
    valid = on & (A != 0)
    safeA = torch.where(A != 0, A, torch.ones_like(A))
    c = edge_functions(faces, p)                                           # [B,F,3,P]
    lam = c.roll(-1, dims=2) / safeA[:, :, None]                           # lam_k = c_{k+1} / A
    lam = torch.where((A != 0)[:, :, None], lam, torch.full_like(lam, 1.0 / 3.0))  # zero area: unused, kept finite
    lh = lam.clamp(0.0, 1.0)
    s = lh.sum(2, keepdim=True)
    l = lh / torch.where(s > 0, s, torch.ones_like(s))
    z = faces[..., 2][..., None]                                           # [B,F,3,1]
    zp = 1.0 / (l / z).sum(2)                                              # [B,F,P]
    return x, on, valid, l, zp


def cube_terms(faces, textures, p, sigma, near, far, eps, face_light, cut_scale):
    """(x, on, valid, zn, C) of soft_rgb per (item, face, pixel); textures [1|B,F,ts,ts,ts,3]"""
    ts = textures.shape[2]
    x, on, valid, l, zp = bary_terms(faces, p, sigma, near, far, cut_scale)
    z = faces[..., 2][..., None]
    t = (l * (ts - 1) * zp[:, :, None] / z).permute(0, 1, 3, 2)            # [B,F,P,3]
    t = t.clamp(0.0, ts - 1 - eps)
    C = sample_cubes(textures, t, ts)                                      # [B,F,P,3]
    if face_light is not None:
        C = C * face_light.to(torch.float64)[:, :, None, :]
    return x, on, valid, (far - zp) / (far - near), C


def zmax_of(valid, zn):
    """the per-pixel max [B,P] of zn over the valid faces (-inf without one), before the background's clamp"""
    return torch.where(valid, zn, torch.full_like(zn, -math.inf)).amax(1)


def blend_sums(x, valid, zn, C, zmax, gamma):
    """(sum_j w_j [B,P], sum_j w_j C_j [B,P,3]) over the faces, zmax the clamped, detached reference depth"""
    D = torch.sigmoid(x)
    ex = torch.where(valid, (zn - zmax[:, None]) / gamma, torch.full_like(zn, -math.inf))
    w = torch.where(valid, D * torch.exp(ex), torch.zeros_like(D))        # [B,F,P]
    return w.sum(1), (w[..., None] * torch.where(valid[..., None], C, torch.zeros_like(C))).sum(1)


def blend_finish(sums, zmax, gamma, background):
    """rgb [B,P,3] of the face sums and the background term at depth BG_DEPTH"""
    wb = torch.exp((BG_DEPTH - zmax) / gamma)                              # [B,P]
    bg = torch.tensor(background, dtype=torch.float64, device=zmax.device)
    return (sums[1] + wb[..., None] * bg) / (sums[0] + wb)[..., None]


def softmax_blend(gamma, background):
    """the blend of osoft.sparse_eval for terms (x, on, valid, zn, C): rgb [Bc,3,P]"""
    return (lambda r: zmax_of(r[0], r[1]).clamp_min(BG_DEPTH),
            lambda x, r, zmax: blend_sums(x, r[0], r[1], r[2], zmax, gamma),
            lambda sums, zmax: blend_finish(sums, zmax, gamma, background).permute(0, 2, 1))


def soft_rgb(faces, textures, S, sigma, gamma, near=0.1, far=100.0, eps=1e-4, background=(0.0, 0.0, 0.0),
             face_light=None, cut_scale=1.0, pix=None):
    """(rgb [B,3,S,S], alpha [B,S,S]) in float64 of faces [B,F,3,3], cubes [1|B,F,ts,ts,ts,3] and face_light [B,F,3].
    With pix (flat pixel indices [P] or [B,P]): (rgb [B,3,P], alpha [B,P]) from the faces in reach only (sparse_eval)."""
    textures = textures.to(torch.float64)
    if pix is not None:
        def terms(b0, b1, idx, fc, p):
            fl = None if face_light is None else osoft.take(face_light, b0, b1, idx)
            return cube_terms(fc, osoft.take(textures, b0, b1, idx), p, sigma, near, far, eps, fl, cut_scale)
        alpha, rgb = osoft.sparse_eval(faces, S, pix, sigma, near, far, cut_scale, terms, softmax_blend(gamma, background))
        return rgb, alpha
    faces = faces.to(torch.float64)
    B = faces.shape[0]
    p = osoft.pixel_centres(S, device=faces.device)
    x, on, valid, zn, C = cube_terms(faces, textures, p, sigma, near, far, eps, face_light, cut_scale)
    alpha = osoft.alpha_from_x(x.transpose(1, 2), on.transpose(1, 2)).reshape(B, S, S)
    zmax = zmax_of(valid, zn).clamp_min(BG_DEPTH).detach()                 # [B,P]
    rgb = blend_finish(blend_sums(x, valid, zn, C, zmax, gamma), zmax, gamma, background)
    return rgb.reshape(B, S, S, 3).permute(0, 3, 1, 2), alpha


def hard_rgb_cpu(faces, textures, S, near=0.1, far=100.0, eps=1e-4, background=(0.0, 0.0, 0.0)):
    """the hard rasterizer's rgb [B,3,S,S] in float64 at pixel centres: the nearest face by interpolated depth, sampled
    like soft_rgb (a reference for the sigma, gamma -> 0 limit)"""
    faces = faces.to(torch.float64)
    textures = textures.to(torch.float64)
    B, F = faces.shape[:2]
    ts = textures.shape[2]
    p = osoft.pixel_centres(S, device=faces.device)
    A = doubled_area(faces)[..., None]
    c = edge_functions(faces, p)
    lam = c.roll(-1, dims=2) / torch.where(A != 0, A, torch.ones_like(A))[:, :, None]
    cover = (lam > 0).all(2) & (A != 0)
    z = faces[..., 2][..., None]
    l = lam.clamp(0.0, 1.0)
    l = l / l.sum(2, keepdim=True).clamp_min(1e-300)
    zp = 1.0 / (l / z).sum(2)
    cover = cover & (zp >= near) & (zp <= far)
    depth = torch.where(cover, zp, torch.full_like(zp, math.inf))
    win = depth.argmin(1)                                                   # [B,P]
    t = (l * (ts - 1) * zp[:, :, None] / z).permute(0, 1, 3, 2).clamp(0.0, ts - 1 - eps)
    C = sample_cubes(textures, t, ts)
    Cw = torch.gather(C, 1, win[:, None, :, None].expand(-1, 1, -1, 3))[:, 0]
    any_cover = cover.any(1)
    bg = torch.tensor(background, dtype=torch.float64, device=faces.device)
    out = torch.where(any_cover[..., None], Cw, bg)
    return out.reshape(B, S, S, 3).permute(0, 3, 1, 2)
