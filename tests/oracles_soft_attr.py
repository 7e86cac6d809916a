"""Float64 oracle of the soft attribute images (include/nr_b200.h, nr_b200_soft_attr_args): dense over every pixel x
every face, or sparse at chosen pixels (oracles_soft.sparse_eval), differentiable with torch autograd in the geometry and
the attributes.  Everything up to the barycentrics, the participation test, alpha and the softmax is the soft RGB's
(oracles_soft_rgb.bary_terms / blend_sums / blend_finish); only the colour is the C-vector A_j = sum_k l'_k a_k."""
import torch

import oracles_soft as osoft
import oracles_soft_rgb as orgb


def corner_attributes(attrs, idx=None):
    """per-corner attributes [1|B,F,3,C] of per-corner attributes (idx None, returned as they are) or of per-vertex ones
    [1|B,Nv,C] through face indices [F,3] / [1|B,F,3] (an index outside [0, Nv) reads zeros); differentiable"""
    if idx is None:
        return attrs
    idx = idx.long()
    if idx.dim() == 2:
        idx = idx[None]
    B = max(attrs.shape[0], idx.shape[0])
    Nv, C = attrs.shape[1], attrs.shape[2]
    ok = (idx >= 0) & (idx < Nv)
    ii = torch.where(ok, idx, torch.zeros_like(idx)).expand(B, -1, -1)
    a = attrs.expand(B, -1, -1)
    g = torch.gather(a, 1, ii.reshape(B, -1, 1).expand(-1, -1, C)).reshape(B, -1, 3, C)
    return torch.where(ok.expand(B, -1, -1)[..., None], g, torch.zeros_like(g))


def attr_terms(faces, ca, p, sigma, near, far, cut_scale):
    """(x, on, valid, zn, A) per (item, face, pixel) of faces [B,F,3,3] at p [P,2] / [B,P,2]; ca [B,F,3,C] float64"""
    x, on, valid, l, zp = orgb.bary_terms(faces, p, sigma, near, far, cut_scale)
    z = faces[..., 2][..., None]                                           # [B,F,3,1]
    lp = l * zp[:, :, None] / z                                            # l'_k [B,F,3,P]
    A = torch.einsum("bfkp,bfkc->bfpc", lp, ca)                           # [B,F,P,C]
    return x, on, valid, (far - zp) / (far - near), A


def soft_attributes(faces, ca, S, sigma, gamma, near=0.1, far=100.0, background=None, cut_scale=1.0, pix=None):
    """(out [B,C,S,S], alpha [B,S,S]) in float64 of faces [B,F,3,3] and per-corner attributes ca [1|B,F,3,C]
    (corner_attributes); background: C numbers or None (zeros).  With pix (flat pixel indices [P] or [B,P]):
    (out [B,C,P], alpha [B,P]) from the faces in reach only (osoft.sparse_eval)."""
    ca = ca.to(torch.float64)
    C = ca.shape[-1]
    bg = tuple(float(v) for v in background) if background is not None else (0.0,) * C
    if pix is not None:
        def terms(b0, b1, idx, fc, p):
            return attr_terms(fc, osoft.take(ca, b0, b1, idx), p, sigma, near, far, cut_scale)
        alpha, out = osoft.sparse_eval(faces, S, pix, sigma, near, far, cut_scale, terms, orgb.softmax_blend(gamma, bg))
        return out, alpha
    faces = faces.to(torch.float64)
    B = faces.shape[0]
    p = osoft.pixel_centres(S, device=faces.device)
    x, on, valid, zn, A = attr_terms(faces, ca.expand(B, -1, -1, -1), p, sigma, near, far, cut_scale)
    alpha = osoft.alpha_from_x(x.transpose(1, 2), on.transpose(1, 2)).reshape(B, S, S)
    zmax = orgb.zmax_of(valid, zn).clamp_min(orgb.BG_DEPTH).detach()      # [B,P]
    out = orgb.blend_finish(orgb.blend_sums(x, valid, zn, A, zmax, gamma), zmax, gamma, bg)
    return out.reshape(B, S, S, C).permute(0, 3, 1, 2), alpha


def attribute_grad_closed_form(faces, ca, S, sigma, gamma, g, near=0.1, far=100.0, background=None):
    """d loss / d ca [B,F,3,C] of loss = sum(out * g) in closed form (include/nr_b200.h): l'_k w_j g_c / Z summed over
    the pixels (no autograd through the attributes)"""
    faces = faces.to(torch.float64)
    B = faces.shape[0]
    ca = ca.to(torch.float64).expand(B, -1, -1, -1)
    p = osoft.pixel_centres(S, device=faces.device)
    x, on, valid, l, zp = orgb.bary_terms(faces, p, sigma, near, far, 1.0)
    zn = (far - zp) / (far - near)
    zmax = orgb.zmax_of(valid, zn).clamp_min(orgb.BG_DEPTH)
    D = torch.sigmoid(x)
    w = torch.where(valid, D * torch.exp((zn - zmax[:, None]) / gamma), torch.zeros_like(D))   # [B,F,P]
    Z = w.sum(1) + torch.exp((orgb.BG_DEPTH - zmax) / gamma)                                    # [B,P]
    lp = l * zp[:, :, None] / faces[..., 2][..., None]                                           # [B,F,3,P]
    gp = g.to(torch.float64).reshape(B, g.shape[1], -1)                                          # [B,C,P]
    return torch.einsum("bfkp,bfp,bcp->bfkc", lp, w / Z[:, None], gp)
