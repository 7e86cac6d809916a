"""Float64 oracle of the soft fragments (include/nr_b200.h, nr_b200_soft_frag_args), on the soft RGB oracle's terms
(oracles_soft_rgb.bary_terms, oracles_soft.face_terms / participates / in_reach).  Two modes:

  candidates(...)  selection: every candidate (item, pixel, face) with its float64 zp, whether it is a candidate for
                   certain or only possibly (the fp32 cut-off test may decide either way within a band), and the derived
                   zbuf gate that serves as its tie band; dense (every face at every pixel) or sparse at chosen pixels
                   (only the faces in reach of them, as oracles_soft.sparse_eval culls).  sort_key orders them by (zp, f).
  evaluate(...)    evaluation at a given pix_to_face: zbuf, bary and dists of those (pixel, face) pairs in float64,
                   differentiable in the faces; empty slots give -1.  The gradient tests use this mode at the kernel's
                   own selection, so no depth tie or cut-off decision can make the two disagree.

Derived gates (gates(...)), per selected pair, with eps = 2^-23, delta = 4 eps max(1, |v|) (a few ulps of the face's
coordinate magnitude), d = sqrt(d^2), |e| the longest edge, A the doubled area (the error analysis of DESIGN.md 4o/4p,
as tests/test_gpu_soft_scale.py derives it):
  dists: 2 d delta + delta^2 + 4 eps d^2                     (the fp32 distance to the nearest segment)
  dl:    8 eps |e| (|e| + d) / |A|                           (the barycentrics' error, edge functions over the area)
  zbuf:  8 eps zp + 3 dl zp^2 / min z
  bary:  dl zp / min z + max_k |l'_k| (zbuf / zp + 4 eps)    (l'_k = l_k zp / z_k)
each times SAFETY = 4, plus 4 eps for the outputs' own rounding.  The cut-off band of a candidate is the larger of 1e-5
cut (relative, as in DESIGN.md 4o) and the dists gate."""
import math

import torch

import oracles_soft as osoft
import oracles_soft_rgb as orgb

EPS32 = 2.0 ** -23
SAFETY = 4.0
CUT_REL = 1e-5


def area32(faces):
    """the doubled signed area in fp32 with plain products, as k_soft_rgb_fill computes it (A == 0: no fragment)"""
    v = faces.detach().to(torch.float32)
    return (v[..., 1, 0] - v[..., 0, 0]) * (v[..., 2, 1] - v[..., 0, 1]) - (v[..., 1, 1] - v[..., 0, 1]) * (v[..., 2, 0] - v[..., 0, 0])


def _error_terms(faces, d2, zp):
    """(delta [B,F,1], dl, dzp) of the gates above, faces [B,F,3,3] float64, d2 / zp [B,F,P]"""
    f = faces.detach()
    delta = 4 * EPS32 * f[..., :2].abs().nan_to_num(0.0, 0.0, 0.0).amax((-1, -2)).clamp_min(1.0)[..., None]
    a = f[..., :2]
    elen = (a.roll(-1, dims=2) - a).norm(dim=-1).amax(-1)[..., None]
    A = orgb.doubled_area(f).abs()[..., None]
    d = d2.clamp_min(0).sqrt()
    dl = 8 * EPS32 * elen * (elen + d) / A.clamp_min(1e-300)
    zmin = f[..., 2].amin(-1)[..., None]
    dzp = 8 * EPS32 * zp.abs() + 3 * dl * zp * zp / zmin.abs().clamp_min(1e-300)
    return delta, dl, dzp


def dists_gate(delta, d2):
    d = d2.clamp_min(0).sqrt()
    return SAFETY * (2 * d * delta + delta * delta + 4 * EPS32 * d2) + 4 * EPS32 * d2


def candidates(faces, S, sigma, near=0.1, far=100.0, pix=None, budget=1 << 21):
    """Every candidate of faces [B,F,3,3] (float32 as given to the kernel) at the pixels pix ([P] flat indices, the same
    for every item; None = all S^2 pixels, dense over every face), as flat tensors: (b, pixel, f, zp, certain, band) --
    certain = a candidate for sure (inside, or d^2 <= cut - band), else only possibly (d^2 <= cut + band); band = the
    derived zbuf gate, the tie band of its zp."""
    faces32 = faces.detach()
    f64 = faces32.to(torch.float64)
    B, F = f64.shape[:2]
    dense = pix is None
    allp = torch.arange(S * S, device=f64.device) if dense else torch.as_tensor(pix, device=f64.device).long()
    cutv = osoft.cut(sigma)
    nz = area32(faces32) != 0
    out = [[] for _ in range(6)]
    pstep = max(1, budget // max(1, F if dense else 64))
    for b in range(B):
        for p0 in range(0, allp.numel(), pstep):
            pc = allp[p0:p0 + pstep]
            p = osoft.pixel_set(S, pc, 1, f64.device)                               # [1,P,2]
            if dense:
                fidx = torch.arange(F, device=f64.device)
            else:
                keep = osoft.in_reach(f64[b:b + 1], p, sigma, near, far, cut_scale=2.0, margin=1e-6)[0]  # wider than any band
                fidx = keep.nonzero()[:, 0]
            if fidx.numel() == 0:
                continue
            for f0 in range(0, fidx.numel(), max(1, budget // pc.numel())):
                fi = fidx[f0:f0 + max(1, budget // pc.numel())]
                fc = f64[b:b + 1, fi]
                part = osoft.participates(fc, near, far)[..., None]                  # [1,Fc,1]
                d2, inside = osoft.face_terms(fc, p[0])                              # [1,Fc,P]
                _, _, _, _, zp = orgb.bary_terms(fc, p[0], sigma, near, far, 1.0)
                delta, dl, dzp = _error_terms(fc, d2, zp)
                band_cut = torch.maximum(torch.full_like(d2, CUT_REL * cutv), dists_gate(delta, d2))
                ok = part & nz[b, fi][None, :, None] & torch.isfinite(zp)
                possible = ok & (inside | (d2 <= cutv + band_cut))
                certain = ok & (inside | (d2 <= cutv - band_cut))
                fj, pj = possible[0].nonzero(as_tuple=True)
                out[0].append(torch.full_like(fj, b))
                out[1].append(pc[pj])
                out[2].append(fi[fj])
                out[3].append(zp[0, fj, pj])
                out[4].append(certain[0, fj, pj])
                out[5].append(SAFETY * dzp[0, fj, pj] + 4 * EPS32 * zp[0, fj, pj].abs())
    if not out[0]:
        z = torch.zeros(0, dtype=torch.long)
        return z, z, z, torch.zeros(0, dtype=torch.float64), torch.zeros(0, dtype=torch.bool), torch.zeros(0, dtype=torch.float64)
    return tuple(torch.cat(o) for o in out)


def sort_key(b, pixel, f, zp):
    """the order of the selection: by item and pixel, then (zp, f)"""
    order = torch.argsort(f, stable=True)
    order = order[torch.argsort(zp[order], stable=True)]
    order = order[torch.argsort(pixel[order], stable=True)]
    return order[torch.argsort(b[order], stable=True)]


def evaluate(faces, pix_to_face, S):
    """(zbuf [B,S,S,K], bary [B,S,S,K,3], dists [B,S,S,K]) in float64 at the pairs of pix_to_face [B,S,S,K] (face
    indices within the item, -1 = empty: -1 in every field), differentiable in faces [B,F,3,3]"""
    B, F = faces.shape[:2]
    K = pix_to_face.shape[-1]
    p2f = pix_to_face.long().cpu() if pix_to_face.device != faces.device else pix_to_face.long()
    sel = (p2f >= 0).reshape(-1)
    flat = p2f.reshape(B, -1)                                                        # [B, S*S*K]
    bi = torch.arange(B, device=faces.device)[:, None].expand_as(flat).reshape(-1)[sel]
    fi = flat.reshape(-1)[sel]
    pi = (torch.arange(S * S * K, device=faces.device) // K)[None].expand(B, -1).reshape(-1)[sel]
    fc = faces.to(torch.float64)[bi, fi][None]                                      # [1,N,3,3]
    p = osoft.pixel_centres(S, device=faces.device)[pi][None]                       # [1,N,2]
    # one pixel per fragment: the [1,N,3,N] terms of bary_terms would be quadratic, so evaluate the diagonal directly
    a = fc[..., :2]
    e = a.roll(-1, dims=2) - a
    dp = p[:, :, None, :] - a                                                        # [1,N,3,2]
    l2 = (e * e).sum(-1)
    nzl = l2 > 0
    t = torch.where(nzl, (dp * e).sum(-1) / torch.where(nzl, l2, torch.ones_like(l2)), torch.zeros_like(l2)).clamp(0.0, 1.0)
    q = dp - t[..., None] * e
    d2 = (q * q).sum(-1).min(-1).values                                              # [1,N]
    c = e[..., 0] * dp[..., 1] - e[..., 1] * dp[..., 0]                              # [1,N,3]
    inside = (c > 0).all(-1) | (c < 0).all(-1)
    A = orgb.doubled_area(fc)[..., None]
    lam = c.roll(-1, dims=2) / torch.where(A != 0, A, torch.ones_like(A))
    lh = lam.clamp(0.0, 1.0)
    l = lh / lh.sum(-1, keepdim=True)
    z = fc[..., 2]
    zp = 1.0 / (l / z).sum(-1)
    lp = l * zp[..., None] / z
    dist = torch.where(inside, d2, -d2)
    n = B * S * S * K
    zb = torch.full((n,), -1.0, dtype=torch.float64, device=faces.device).index_put((sel.nonzero()[:, 0],), zp[0])
    ds = torch.full((n,), -1.0, dtype=torch.float64, device=faces.device).index_put((sel.nonzero()[:, 0],), dist[0])
    by = torch.full((n, 3), -1.0, dtype=torch.float64, device=faces.device).index_put((sel.nonzero()[:, 0],), lp[0])
    return zb.reshape(B, S, S, K), by.reshape(B, S, S, K, 3), ds.reshape(B, S, S, K)


def gates(faces, pix_to_face, S):
    """the derived gates (zbuf, bary, dists) [B,S,S,K] at the pairs of pix_to_face (0 at empty slots)"""
    with torch.no_grad():
        faces = faces.detach().to(torch.float64)
        B = faces.shape[0]
        K = pix_to_face.shape[-1]
        zb, by, ds = evaluate(faces, pix_to_face, S)
        p2f = pix_to_face.long().to(faces.device)
        sel = p2f >= 0
        fc = torch.gather(faces, 1, p2f.clamp_min(0).reshape(B, -1, 1, 1).expand(-1, -1, 3, 3))       # [B,SSK,3,3]
        d2 = ds.abs().reshape(B, -1)
        delta, dl, dzp = _error_terms(fc, d2[..., None], zb.reshape(B, -1)[..., None])
        delta, dl, dzp = delta[..., 0], dl[..., 0], dzp[..., 0]
        zmin = fc[..., 2].amin(-1).abs()
        zp = zb.reshape(B, -1).abs()
        lpm = by.reshape(B, -1, 3).abs().amax(-1)
        g_z = SAFETY * dzp + 4 * EPS32 * zp
        g_b = SAFETY * (dl * zp / zmin + lpm * (dzp / zp.clamp_min(1e-300) + 4 * EPS32)) + 4 * EPS32
        g_d = dists_gate(delta, d2)
        z0 = torch.zeros_like(g_z)
        return tuple(torch.where(sel.reshape(B, -1), g, z0).reshape(B, S, S, K) for g in (g_z, g_b, g_d))
