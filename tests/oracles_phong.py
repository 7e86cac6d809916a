"""float64 restatement of Phong shading (include/nr_b200.h, nr_b200_phong_args) on the product's own maps: normal and
position interpolated with float64 perspective weights, ambient + diffuse times an unlit raster sample plus the specular
term, as the header writes it.  Differentiable: corner_shading, params and the unlit sample may require grad."""
import torch

from oracles import _bg


def _norm(x):
    return x / (torch.linalg.vector_norm(x, dim=-1, keepdim=True) + 1e-5)


def phong_terms64(faces, fim, wmap, dmap, corner_shading, params):
    """per raster pixel [B,S,S,...]: the light L [.,3] and the specular factor h [.] (float64).  faces [B,F,3,3] (the
    winner's own camera depths), corner_shading [1|B,F,3,6], params [1|B,16]."""
    dev = fim.device
    B, S = faces.shape[0], fim.shape[-1]
    fi = fim.clamp(min=0).long()
    bidx = torch.arange(B, device=dev)[:, None, None].expand(B, S, S)
    z = faces.double()[..., 2][bidx, fi]
    z = torch.where((fim >= 0)[..., None], z, torch.ones_like(z))  # keep 0 * inf of uncovered pixels out of autograd
    lam = wmap.double().permute(0, 2, 3, 1) * (dmap.double()[..., None] / z)              # [B,S,S,3]
    cs = corner_shading.double()
    C = cs[bidx if cs.shape[0] > 1 else torch.zeros_like(bidx), fi]                          # [B,S,S,3,6]
    n = (lam[..., None] * C[..., :3]).sum(dim=3)
    p = (lam[..., None] * C[..., 3:]).sum(dim=3)
    prm = params.double().expand(B, 16)[:, None, None, :]
    A, D, d, K, sig, e = prm[..., 0:3], prm[..., 3:6], prm[..., 6:9], prm[..., 9:12], prm[..., 12], prm[..., 13:16]
    nh, dh, vh = _norm(n), _norm(d), _norm(e - p)
    c = (nh * d).sum(-1)
    L = A + D * torch.relu(c)[..., None]
    nd = (nh * dh).sum(-1, keepdim=True)
    r = 2 * nd * nh - dh
    q = torch.relu((r * vh).sum(-1))
    on = (c > 0) & (q > 0) & (fim >= 0)
    qs = torch.where(on, q, torch.ones_like(q))  # no ln 0 in the unselected branch
    h = torch.where(on, qs ** sig, torch.zeros_like(q))
    return L, h, K


def phong_rgb64(faces, fim, wmap, dmap, corner_shading, params, unlit, bg, aa):
    """API rgb [B,3,H,W]: L s + K h where covered, the background elsewhere, 2x2 mean with anti-aliasing; unlit [B,3,S,S]"""
    L, h, K = phong_terms64(faces, fim, wmap, dmap, corner_shading, params)
    lit = L * unlit.double().permute(0, 2, 3, 1) + K * h[..., None]
    rgb = torch.where((fim >= 0)[..., None], lit, _bg(bg, fim.device)).permute(0, 3, 1, 2)
    return torch.nn.functional.avg_pool2d(rgb, 2, 2) if aa else rgb
