"""float64 restatement of attribute interpolation (include/nr_b200.h, nr_b200_interpolate) with face_index_map held
fixed: the weights are recomputed from the faces through a float64 K1 inverse, so autograd of the image reaches the
vertices; `interior_grad64` is the header's closed-form vertex gradient in float64."""
import torch


def _setup(faces, fim, S):
    """per raster pixel: covered mask, winner's faces [B,S,S,3,3] (a fixed, well-conditioned triangle where uncovered, so
    no NaN reaches autograd) and the unclamped barycentrics a [B,S,S,3] and K1 inverse rows inv [B,S,S,3 corners,3]"""
    dev = fim.device
    B = faces.shape[0]
    cov = fim >= 0
    fi = fim.clamp(min=0).long()
    bidx = torch.arange(B, device=dev)[:, None, None].expand(B, S, S)
    dummy = torch.tensor([[-0.5, -0.5, 2.0], [0.5, -0.5, 2.0], [0.0, 0.5, 2.0]], dtype=torch.float64, device=dev)
    f = torch.where(cov[..., None, None], faces.double()[bidx, fi], dummy)
    px, py = 0.5 * (f[..., 0] * S + S - 1), 0.5 * (f[..., 1] * S + S - 1)  # to_pixel
    inv = torch.linalg.inv(torch.stack((px, py, torch.ones_like(px)), dim=-2))  # rows = corners
    row = torch.arange(S, device=dev, dtype=torch.float64)
    yi = (S - 1 - row)[None, :, None].expand(B, S, S)  # image row r is raster row S-1-r
    xi = row[None, None, :].expand(B, S, S)
    p = torch.stack((xi, yi, torch.ones_like(xi)), dim=-1)
    a = (inv * p[..., None, :]).sum(-1)
    return cov, fi, bidx, f, a, inv, torch.stack((px, py), dim=-1)


def interp64(faces, fim, corner_attrs, S, aa, wmap=None):
    """API image [B,C,H,W]: faces [B,F,3,3] (NDC x, y, camera z), corner_attrs [B,F,3,C] (may require grad).  With `wmap`
    (the product's saved weights) the value uses them, and the derivative is taken at them with the clamp held fixed, as
    the product's backward: the barycentrics of the fixed point sum_k w_k P_k, whose vertex derivative is -w_m inv[3k]."""
    cov, fi, bidx, f, a, inv, P = _setup(faces, fim, S)
    w = a
    if wmap is not None:  # uncovered pixels keep a (their saved weights are 0: l = 0/0 would reach autograd)
        wm = wmap.double().permute(0, 2, 3, 1)
        pt = (wm[..., None] * P).sum(-2).detach()
        aw = (inv[..., :2] * pt[..., None, :]).sum(-1) + inv[..., 2]
        w = torch.where(cov[..., None], aw + (wm - aw).detach(), a)
    q = w / f[..., 2]
    lam = q / q.sum(-1, keepdim=True)
    A = corner_attrs.double()[bidx, fi]  # [B,S,S,3,C]
    out = (lam[..., None] * A).sum(-2)
    out = torch.where(cov[..., None], out, torch.zeros_like(out)).permute(0, 3, 1, 2)
    return torch.nn.functional.avg_pool2d(out, 2, 2) if aa else out


def interior_grad64(faces, fim, corner_attrs, g, S):
    """closed-form d sum(g * raster image) / d faces [B,F,3,3] at w = a (include/nr_b200.h), g [B,C,S,S] raster layout"""
    cov, fi, bidx, f, a, inv, _ = _setup(faces, fim, S)
    z = f[..., 2]
    zp = 1.0 / (a / z).sum(-1)
    lam = a * zp[..., None] / z
    A = corner_attrs.double()[bidx, fi]
    gp = g.double().permute(0, 2, 3, 1)
    out = (lam[..., None] * A).sum(-2)
    D = ((A[..., 1:, :] - A[..., :1, :]) * gp[..., None, :]).sum(-1)  # [B,S,S,2]
    G = []
    for d in (0, 1):
        qd = inv[..., d] / z
        ld = zp[..., None] * (qd - lam * qd.sum(-1, keepdim=True))
        G.append((D * ld[..., 1:]).sum(-1))
    Gz = lam / z * ((out[..., None, :] - A) * gp[..., None, :]).sum(-1)
    gf = torch.stack((-a * G[0][..., None] * S / 2, -a * G[1][..., None] * S / 2, Gz), dim=-1)  # [B,S,S,3,3]
    B, F = faces.shape[:2]
    flat = (bidx * F + fi)[cov]
    res = torch.zeros((B * F, 3, 3), dtype=torch.float64, device=faces.device)
    res.index_add_(0, flat, gf[cov])
    return res.reshape(B, F, 3, 3)


def clamp_active(faces, fim, S):
    """covered raster pixels [B,S,S] whose float64 barycentrics leave [0,1]: there the saved weights are clamped, and the
    product's derivative (clamp held fixed) is not the derivative of its forward"""
    cov, _, _, _, a, _, _ = _setup(faces, fim, S)
    return cov & ((a < 0) | (a > 1)).any(-1)
