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


def soft_uv(faces, tex, uvs, S, sigma, gamma, near=0.1, far=100.0, background=(0.0, 0.0, 0.0), face_light=None,
            hw=None, cut_scale=1.0):
    """(rgb [B,3,S,S], alpha [B,S,S]) in float64 of faces [B,F,3,3], uvs [1|B,F,3,2] and either an image
    [1|B,Ht,Wt,3] (bilinear, hw None) or a packed pyramid [1|B,P,3] of an image of hw = (Ht, Wt) (trilinear)"""
    faces = faces.to(torch.float64)
    B, F = faces.shape[:2]
    dev = faces.device
    p = osoft.pixel_centres(S, device=dev)
    P = p.shape[0]
    part = osoft.participates(faces, near, far)
    d2, inside = osoft.face_terms(faces, p)                               # [B,F,P]
    x = torch.where(inside, d2 / sigma, -d2 / sigma)
    on = part[..., None] & (inside | (d2 <= osoft.cut(sigma) * cut_scale))
    alpha = osoft.alpha_from_x(x.transpose(1, 2), on.transpose(1, 2)).reshape(B, S, S)
    D = torch.sigmoid(x)
    A = orgb.doubled_area(faces)[..., None]                                # [B,F,1]
    valid = on & (A != 0)
    safeA = torch.where(A != 0, A, torch.ones_like(A))
    c = orgb.edge_functions(faces, p)                                      # [B,F,3,P]
    lam = c.roll(-1, dims=2) / safeA[:, :, None]                           # lam_k = c_{k+1} / A
    lam = torch.where((A != 0)[:, :, None], lam, torch.full_like(lam, 1.0 / 3.0))
    lh = lam.clamp(0.0, 1.0)
    s = lh.sum(2, keepdim=True)
    l = lh / torch.where(s > 0, s, torch.ones_like(s))
    z = faces[..., 2][..., None]                                           # [B,F,3,1]
    zp = 1.0 / (l / z).sum(2)                                              # [B,F,P]
    lp = l * zp[:, :, None] / z                                            # l'_k [B,F,3,P]
    uvk = uvs.to(torch.float64).expand(B, -1, -1, -1)                      # [B,F,3,2]
    u = (lp * uvk[..., 0][..., None]).sum(2)
    v = (lp * uvk[..., 1][..., None]).sum(2)
    tex = tex.to(torch.float64).expand(B, *tex.shape[1:])
    if hw is None:
        Ht, Wt = tex.shape[1:3]
        C = sample(tex.reshape(B, Ht * Wt, 3), 0, Ht, Wt, u, v)
    else:
        Ht, Wt = hw
        off, hs, ws = level_table(Ht, Wt, dev)
        L = off.numel()
        ld = lod(faces, l, zp, uvk, S, Ht, Wt, L)
        l0 = ld.floor().long()
        l1 = (l0 + 1).clamp(max=L - 1)
        f = (ld - l0)[..., None]
        C = (1 - f) * sample(tex, off[l0], hs[l0], ws[l0], u, v) + f * sample(tex, off[l1], hs[l1], ws[l1], u, v)
    if face_light is not None:
        C = C * face_light.to(torch.float64)[:, :, None, :]
    zn = (far - zp) / (far - near)
    neg = torch.full_like(zn, -math.inf)
    zmax = torch.where(valid, zn, neg).amax(1).clamp_min(orgb.BG_DEPTH).detach()   # [B,P]
    ex = torch.where(valid, (zn - zmax[:, None]) / gamma, neg)
    w = torch.where(valid, D * torch.exp(ex), torch.zeros_like(D))        # [B,F,P]
    wb = torch.exp((orgb.BG_DEPTH - zmax) / gamma)                         # [B,P]
    bg = torch.tensor(background, dtype=torch.float64, device=dev)
    num = (w[..., None] * torch.where(valid[..., None], C, torch.zeros_like(C))).sum(1) + wb[..., None] * bg
    Z = w.sum(1) + wb
    rgb = (num / Z[..., None]).reshape(B, S, S, 3).permute(0, 3, 1, 2)
    return rgb, alpha
