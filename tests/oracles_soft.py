"""Float64 oracle of the soft silhouettes (include/nr_b200.h, nr_b200_soft_args): dense over every pixel x every face,
differentiable with torch autograd.  Independent of the kernels: no binning, no tiles, no cut-off reach, the log-domain
product in float64.

Given a pixel set (`pix`), the three soft oracles evaluate only those pixels and only the faces whose box, grown by the
cut-off reach, holds one of them (in_reach): every other face has on = False at every chosen pixel, so the cull changes
neither a value nor a gradient.  sparse_eval runs that in chunks of items and faces, which keeps the oracle feasible at
the benchmarks' 64 x 5000 faces."""
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


def pixel_set(S, pix, B, device=None):
    """[B,P,2] NDC centres of the flat pixel indices pix [P] (one set for every item) or [B,P] (row-major, row 0 at the
    top, as pixel_centres)"""
    pix = torch.as_tensor(pix, device=device).long()
    c = pixel_centres(S, device=device)
    return c[pix].expand(B, -1, -1) if pix.dim() == 1 else c[pix]


def points(p):
    """p [P,2] (every item) or [B,P,2] (per item), shaped to broadcast against face corners [B,F,3,1,2]"""
    return p[None, None, None] if p.dim() == 2 else p[:, None, None]


def face_terms(faces, p):
    """d^2 [B,F,P] to the closed triangle and the strict inside mask, faces [B,F,3,3] float64, p [P,2] or [B,P,2]"""
    a = faces[..., :2]                       # [B,F,3,2]
    e = a.roll(-1, dims=2) - a               # edge k: v_k -> v_{k+1}
    dp = points(p) - a[:, :, :, None]                    # [B,F,3,P,2]
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


def soft_silhouettes(faces, S, sigma, near=0.1, far=100.0, cut_scale=1.0, chunk=1 << 22, pix=None):
    """alpha [B,S,S] (float64) of faces [B,F,3,3]; `cut_scale` moves the cut-off (the tests bracket its fp32 rounding).
    With pix (flat pixel indices [P] or [B,P]): alpha [B,P] at those pixels, from the faces in reach only (sparse_eval)."""
    if pix is not None:
        def terms(b0, b1, idx, fc, p):
            d2, inside = face_terms(fc, p)
            x = torch.where(inside, d2 / sigma, -d2 / sigma)
            return x, participates(fc, near, far)[..., None] & (inside | (d2 <= cut(sigma) * cut_scale))
        return sparse_eval(faces, S, pix, sigma, near, far, cut_scale, terms)[0]
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



def in_reach(faces, p, sigma, near, far, cut_scale=1.0, margin=1e-9, chunk=1 << 22):
    """[B,F]: the faces that take part and whose xy box, grown by sqrt(cut cut_scale) + margin, holds a pixel of p
    [B,P,2].  Exact: a face on at a pixel has it inside (so inside its box) or within d^2 <= cut cut_scale of its nearest
    point (so within sqrt(cut cut_scale) of its box); the margin covers the float64 rounding of both tests."""
    with torch.no_grad():
        faces = faces.to(torch.float64)
        r = math.sqrt(cut(sigma) * cut_scale) + margin
        xy = faces[..., :2]
        lo, hi = xy.amin(2) - r, xy.amax(2) + r                 # [B,F,2]; NaN compares false
        q = p[:, None]                                           # [B,1,P,2]
        step = max(1, chunk // max(1, p.shape[1]))
        hit = [((q >= lo[:, f0:f0 + step, None]) & (q <= hi[:, f0:f0 + step, None])).all(-1).any(-1)
               for f0 in range(0, faces.shape[1], step)]
        return participates(faces, near, far) & torch.cat(hit, 1)


def take(t, b0, b1, idx):
    """t [1|B,F,...] of the items b0:b1 at the faces idx [b1-b0,Fc] (differentiable: a gather)"""
    tb = t[b0:b1] if t.shape[0] > 1 else t.expand(b1 - b0, *t.shape[1:])
    return torch.gather(tb, 1, idx.reshape(idx.shape + (1,) * (t.dim() - 2)).expand(*idx.shape, *t.shape[2:]))


def sparse_eval(faces, S, pix, sigma, near, far, cut_scale, terms, blend=None, budget=1 << 20):
    """The sparse evaluation of the soft oracles at the pixels pix ([P] or [B,P] flat indices): (alpha [B,P], out).

    Only the faces in_reach of an item's pixels are evaluated, in chunks of items and of their kept faces of at most
    `budget` (item, face, pixel) triples (the float64 terms of one chunk take a few hundred MB).  terms(b0, b1, idx, fc,
    p) gives the per-(item, face, pixel) terms of the faces fc [Bc,Fc,3,3] (= take(faces, b0, b1, idx), padding slots
    an off-image face) at p [Bc,P,2]: (x, on, *rest), with x and on as in soft_silhouettes.  Padding slots are masked off on, and
    on every boolean mask of rest.  blend = (first, partial, finish) aggregates what alpha does not: first(rest) -> a
    per-pixel reference over the faces of one chunk, max-reduced over the chunks without gradient in a first pass (the
    soft RGB's detached zmax); partial(x, rest, ref) -> a tuple of per-pixel sums; finish(sums, ref) -> out [Bc,...]."""
    faces = faces.to(torch.float64)
    B = faces.shape[0]
    p = pixel_set(S, pix, B, faces.device)
    P = p.shape[1]
    keep = in_reach(faces, p, sigma, near, far, cut_scale)
    # padding slots: an off-image face with finite terms everywhere (masked off on, so it adds nothing)
    pad = torch.tensor([[10.0, 10.0, 1.0], [10.5, 10.0, 1.0], [10.0, 10.5, 1.0]], dtype=faces.dtype, device=faces.device)
    nk = keep.sum(1)
    per_item = P * max(1, int(nk.max()))
    bstep = max(1, budget // per_item)
    alphas, outs = [], []
    for b0 in range(0, B, bstep):
        b1 = min(B, b0 + bstep)
        kc = keep[b0:b1]
        n = max(1, int(nk[b0:b1].max()))
        order = torch.argsort((~kc).to(torch.int8), dim=1, stable=True)[:, :n]   # each item's kept faces first
        real = torch.gather(kc, 1, order)
        pc = p[b0:b1]
        fstep = max(1, budget // ((b1 - b0) * P))

        def chunk(f0):
            idx, r = order[:, f0:f0 + fstep], real[:, f0:f0 + fstep]
            fc = torch.where(r[..., None, None], take(faces, b0, b1, idx), pad)
            out = terms(b0, b1, idx, fc, pc)
            rp = r[..., None]
            return (out[0],) + tuple(o & rp if o.dtype == torch.bool else o for o in out[1:])

        ref = None
        if blend is not None:
            with torch.no_grad():
                ref = torch.stack([blend[0](chunk(f0)[2:]) for f0 in range(0, n, fstep)]).amax(0)
        lam, sums = 0, None
        for f0 in range(0, n, fstep):
            x, on, *rest = chunk(f0)
            sp = torch.nn.functional.softplus(x)
            lam = lam + torch.where(on, sp, torch.zeros_like(sp)).sum(1)
            if blend is not None:
                part = blend[1](x, rest, ref)
                sums = part if sums is None else tuple(a + b for a, b in zip(sums, part))
        alphas.append(-torch.expm1(-lam))
        if blend is not None:
            outs.append(blend[2](sums, ref))
    return torch.cat(alphas), (torch.cat(outs) if blend is not None else None)
