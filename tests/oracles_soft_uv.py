"""Float64 oracle of the soft RGB through a texture image (include/nr_b200.h, nr_b200_soft_uv_args): dense over every
pixel x every face, differentiable with torch autograd in the geometry, the image / packed pyramid, the UVs and the
light.  Everything up to the barycentrics, the participation test, alpha and the softmax is the soft RGB's
(oracles_soft, oracles_soft_rgb.edge_functions / doubled_area); only the colour differs.  The cell of every tap is held
by floor with the uv_taps edge rules, the level of detail is computed without gradient from the face's screen-barycentric
derivatives."""
import math

import torch

import oracles
import oracles_soft as osoft
import oracles_soft_rgb as orgb


def level_table(Ht, Wt, device=None):
    """(offset in texels, height, width) of every pyramid level as int64 tensors [L]"""
    sizes = oracles.mip_levels(Ht, Wt)
    off, acc = [], 0
    for h, w in sizes:
        off.append(acc)
        acc += h * w
    as_t = lambda a: torch.tensor(a, dtype=torch.int64, device=device)
    return as_t(off), as_t([h for h, _ in sizes]), as_t([w for _, w in sizes])


def sample(flat, off, H, W, u, v):
    """bilinear sample [B,F,P,3] of the texels flat [B,T,3] (levels packed row-major, row 0 = top) at (u, v) [B,F,P] on
    the level at texel offset `off` of size H x W (ints or int64 tensors like u): clamp to [0, 1] (NaN -> 0), the cell
    held by floor, taps clamped into the level"""
    B, F, P = u.shape
    uc = torch.nan_to_num(u.clamp(0.0, 1.0), nan=0.0)
    vc = torch.nan_to_num(v.clamp(0.0, 1.0), nan=0.0)
    px, py = uc * (W - 1), vc * (H - 1)
    ix = torch.minimum(px.detach().floor().long(), torch.as_tensor(W - 1))
    iy = torch.minimum(py.detach().floor().long(), torch.as_tensor(H - 1))
    wx1, wy1 = px - ix, py - iy
    wx0, wy0 = 1 - wx1, 1 - wy1
    x1 = torch.minimum(ix + 1, torch.as_tensor(W - 1))
    y1 = torch.minimum(iy + 1, torch.as_tensor(H - 1))
    r0, r1 = H - 1 - iy, H - 1 - y1

    def tap(r, c):
        idx = (off + r * W + c).reshape(B, F * P, 1).expand(-1, -1, 3)
        return torch.gather(flat, 1, idx).reshape(B, F, P, 3)
    return ((wx0 * wy0)[..., None] * tap(r0, ix) + (wx0 * wy1)[..., None] * tap(r1, ix)
            + (wx1 * wy0)[..., None] * tap(r0, x1) + (wx1 * wy1)[..., None] * tap(r1, x1))


def lod(faces, l, zp, uvk, S, Ht, Wt, levels):
    """level of detail [B,F,P] (no gradient): mip_lod with d lam_k / d column = -(2/S) e_{k+1,y} / A, d lam_k / d row =
    -(2/S) e_{k+1,x} / A in place of K1's inverse, l in place of w"""
    with torch.no_grad():
        a = faces[..., :2]
        e = a.roll(-1, dims=2) - a                                     # e_m = v_{m+1} - v_m, [B,F,3,2]
        A = orgb.doubled_area(faces)
        A = torch.where(A != 0, A, torch.ones_like(A))[..., None]
        en = e.roll(-1, dims=2)                                        # e_{k+1}
        ix = -(2.0 / S) * en[..., 1] / A                               # [B,F,3]
        iy = -(2.0 / S) * en[..., 0] / A
        z = faces[..., 2]                                              # [B,F,3]
        lam = l * zp[:, :, None] / z[..., None]                        # [B,F,3,P]
        qx, qy = (ix / z)[..., None], (iy / z)[..., None]
        lx = zp[:, :, None] * (qx - lam * qx.sum(2, keepdim=True))
        ly = zp[:, :, None] * (qy - lam * qy.sum(2, keepdim=True))
        u, v = uvk[..., 0][..., None], uvk[..., 1][..., None]          # [B,F,3,1]
        dudx, dvdx = (u * lx).sum(2), (v * lx).sum(2)
        dudy, dvdy = (u * ly).sum(2), (v * ly).sum(2)
        rx = ((Wt - 1) * dudx) ** 2 + ((Ht - 1) * dvdx) ** 2
        ry = ((Wt - 1) * dudy) ** 2 + ((Ht - 1) * dvdy) ** 2
        out = 0.5 * torch.log2(torch.maximum(rx, ry))
        return torch.nan_to_num(out, nan=0.0, neginf=0.0).clamp(0.0, levels - 1)


def uv_terms(faces, tex, uvk, p, S, sigma, near, far, face_light, hw, cut_scale):
    """(x, on, valid, zn, C) of soft_uv per (item, face, pixel) of faces [B,F,3,3] at p [P,2] / [B,P,2]; tex [B,...]
    and uvk [B,F,3,2] float64 already expanded to the items"""
    B = faces.shape[0]
    x, on, valid, l, zp = orgb.bary_terms(faces, p, sigma, near, far, cut_scale)
    z = faces[..., 2][..., None]                                           # [B,F,3,1]
    lp = l * zp[:, :, None] / z                                            # l'_k [B,F,3,P]
    u = (lp * uvk[..., 0][..., None]).sum(2)
    v = (lp * uvk[..., 1][..., None]).sum(2)
    if hw is None:
        Ht, Wt = tex.shape[1:3]
        C = sample(tex.reshape(B, Ht * Wt, 3), 0, Ht, Wt, u, v)
    else:
        Ht, Wt = hw
        off, hs, ws = level_table(Ht, Wt, faces.device)
        L = off.numel()
        ld = lod(faces, l, zp, uvk, S, Ht, Wt, L)
        l0 = ld.floor().long()
        l1 = (l0 + 1).clamp(max=L - 1)
        f = (ld - l0)[..., None]
        C = (1 - f) * sample(tex, off[l0], hs[l0], ws[l0], u, v) + f * sample(tex, off[l1], hs[l1], ws[l1], u, v)
    if face_light is not None:
        C = C * face_light.to(torch.float64)[:, :, None, :]
    return x, on, valid, (far - zp) / (far - near), C


def soft_uv(faces, tex, uvs, S, sigma, gamma, near=0.1, far=100.0, background=(0.0, 0.0, 0.0), face_light=None,
            hw=None, cut_scale=1.0, pix=None):
    """(rgb [B,3,S,S], alpha [B,S,S]) in float64 of faces [B,F,3,3], uvs [1|B,F,3,2] and either an image
    [1|B,Ht,Wt,3] (bilinear, hw None) or a packed pyramid [1|B,P,3] of an image of hw = (Ht, Wt) (trilinear).  With pix
    (flat pixel indices [P] or [B,P]): (rgb [B,3,P], alpha [B,P]) from the faces in reach only (osoft.sparse_eval)."""
    tex = tex.to(torch.float64)
    uvs = uvs.to(torch.float64)
    if pix is not None:
        def terms(b0, b1, idx, fc, p):
            tc = tex[b0:b1] if tex.shape[0] > 1 else tex.expand(b1 - b0, *tex.shape[1:])
            fl = None if face_light is None else osoft.take(face_light, b0, b1, idx)
            return uv_terms(fc, tc, osoft.take(uvs, b0, b1, idx), p, S, sigma, near, far, fl, hw, cut_scale)
        alpha, rgb = osoft.sparse_eval(faces, S, pix, sigma, near, far, cut_scale, terms,
                                       orgb.softmax_blend(gamma, background))
        return rgb, alpha
    faces = faces.to(torch.float64)
    B = faces.shape[0]
    p = osoft.pixel_centres(S, device=faces.device)
    x, on, valid, zn, C = uv_terms(faces, tex.expand(B, *tex.shape[1:]), uvs.expand(B, -1, -1, -1), p, S, sigma, near,
                                   far, face_light, hw, cut_scale)
    alpha = osoft.alpha_from_x(x.transpose(1, 2), on.transpose(1, 2)).reshape(B, S, S)
    zmax = orgb.zmax_of(valid, zn).clamp_min(orgb.BG_DEPTH).detach()      # [B,P]
    rgb = orgb.blend_finish(orgb.blend_sums(x, valid, zn, C, zmax, gamma), zmax, gamma, background)
    return rgb.reshape(B, S, S, 3).permute(0, 3, 1, 2), alpha
