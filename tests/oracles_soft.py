"""Float64 oracle of the soft silhouettes (include/nr_b200.h, nr_b200_soft_args): dense over every pixel x every face,
differentiable with torch autograd.  Independent of the kernels: no binning, no tiles, no cut-off reach, the log-domain
product in float64."""
import math

import torch

EPS = 1e-4  # NR_SOFT_EPS


def cut(sigma):
    """d^2 bound of an outside face that still contributes (D >= EPS)"""
    return sigma * math.log((1.0 - EPS) / EPS)


def pixel_centres(S, dtype=torch.float64, device=None):
    """[S*S, 2] NDC centres of the API pixels, row-major, row 0 at the top"""
    i = torch.arange(S, dtype=dtype, device=device)
    c = (2 * i + 1 - S) / S
    y = c.flip(0)  # row r shows raster row S-1-r
    return torch.stack((c[None, :].expand(S, S), y[:, None].expand(S, S)), -1).reshape(-1, 2)


def gather_faces(vertices, indices):
    """faces [B,F,3,3] of vertices [B,Nv,3] and indices [F,3] / [1|B,F,3]; an index outside [0, Nv) gathers zeros"""
    B, Nv = vertices.shape[:2]
    idx = indices.long()
    if idx.dim() == 2:
        idx = idx[None]
    idx = idx.expand(B, -1, -1)
    ok = (idx >= 0) & (idx < Nv)
    g = torch.gather(vertices, 1, idx.clamp(0, Nv - 1).reshape(B, -1, 1).expand(-1, -1, 3)).reshape(B, -1, 3, 3)
    return torch.where(ok[..., None], g, torch.zeros_like(g))


def face_terms(faces, p):
    """d^2 [B,F,P] to the closed triangle and the strict inside mask, faces [B,F,3,3] float64, p [P,2]"""
    a = faces[..., :2]                       # [B,F,3,2]
    e = a.roll(-1, dims=2) - a               # edge k: v_k -> v_{k+1}
    dp = p[None, None, None] - a[:, :, :, None]          # [B,F,3,P,2]
    ee = e[:, :, :, None]
    l2 = (e * e).sum(-1)[..., None]                      # [B,F,3,1]
    nz = l2 > 0
    t = torch.where(nz, (dp * ee).sum(-1) / torch.where(nz, l2, torch.ones_like(l2)), torch.zeros_like(l2))
    t = t.clamp(0.0, 1.0)
    q = dp - t[..., None] * ee
    d2 = (q * q).sum(-1).min(dim=2).values               # [B,F,P]
    c = ee[..., 0] * dp[..., 1] - ee[..., 1] * dp[..., 0]  # edge functions [B,F,3,P]
    inside = (c > 0).all(dim=2) | (c < 0).all(dim=2)
    return d2, inside


def participates(faces, near, far):
    z = faces[..., 2]
    xy = faces[..., :2]
    return ((z >= near) & (z <= far)).all(-1) & torch.isfinite(xy).all(-1).all(-1)   # [B,F]


def soft_silhouettes(faces, S, sigma, near=0.1, far=100.0, cut_scale=1.0, chunk=1 << 22):
    """alpha [B,S,S] (float64) of faces [B,F,3,3]; `cut_scale` moves the cut-off (the tests bracket its fp32 rounding)"""
    faces = faces.to(torch.float64)
    B, F = faces.shape[:2]
    p = pixel_centres(S, device=faces.device)
    part = participates(faces, near, far)
    lam = torch.zeros(B, p.shape[0], dtype=torch.float64, device=faces.device)
    step = max(1, chunk // max(1, p.shape[0]))
    for f0 in range(0, F, step):
        fc = faces[:, f0:f0 + step]
        d2, inside = face_terms(fc, p)
        x = torch.where(inside, d2 / sigma, -d2 / sigma)
        on = part[:, f0:f0 + step, None] & (inside | (d2 <= cut(sigma) * cut_scale))
        sp = torch.nn.functional.softplus(x)
        lam = lam - torch.where(on, sp, torch.zeros_like(sp)).sum(1)
    return (-torch.expm1(lam)).reshape(B, S, S)


def alpha_from_x(x, on):
    """alpha of per-(pixel, face) logits x [..., F] with the contribution mask `on` (the aggregation alone)"""
    sp = torch.nn.functional.softplus(x)
    return -torch.expm1(-torch.where(on, sp, torch.zeros_like(sp)).sum(-1))

