"""float64 restatement of Phong shading with a light set (include/nr_b200.h, nr_b200_lights_args) on the product's own maps:
the Phong expression of oracles_phong.py with the set's diffuse terms added to the light and their highlights to the
specular term, as the header writes it.  Differentiable: corner_shading, params, lights and the unlit sample may require
grad."""
import torch

from oracles import _bg
from oracles_phong import _norm


def lights_terms64(faces, fim, wmap, dmap, corner_shading, params, lights=None):
    """per raster pixel [B,S,S,...]: the light L [.,3] (every light's diffuse term) and the specular colour [.,3]
    (K h + sum_j K_j a_j h_j), float64.  faces [B,F,3,3] (the winner's own camera depths), corner_shading [1|B,F,3,6],
    params [1|B,16], lights [1|B,NL,12] or None."""
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
    nh, vh = _norm(n), _norm(e - p)
    covered = fim >= 0

    def spec(c, lh):
        r = 2 * (nh * lh).sum(-1, keepdim=True) * nh - lh
        q = torch.relu((r * vh).sum(-1))
        on = (c > 0) & (q > 0) & covered
        qs = torch.where(on, q, torch.ones_like(q))  # no ln 0 in the unselected branch
        return torch.where(on, qs ** sig, torch.zeros_like(q))

    c0 = (nh * d).sum(-1)
    L = A + D * torch.relu(c0)[..., None]
    spc = K * spec(c0, _norm(d))[..., None]
    if lights is not None:
        lt = lights.double()
        lt = lt.expand(B, -1, -1) if lt.shape[0] == 1 else lt
        for j in range(lt.shape[1]):
            rec = lt[:, j][:, None, None, :]                                                    # [B,1,1,12]
            Dj, Kj, x, f = rec[..., 0:3], rec[..., 3:6], rec[..., 6:9], rec[..., 9]
            point = rec[..., 10] > 0.5
            u = torch.where(point[..., None], x - p, x.expand_as(p))
            r = torch.linalg.vector_norm(u, dim=-1)
            lh = u / (r[..., None] + 1e-5)
            c = torch.where(point, (nh * lh).sum(-1), (nh * x).sum(-1))
            a = torch.where(point, 1 / (1 + f * r * r), torch.ones_like(r))
            L = L + Dj * (a * torch.relu(c))[..., None]
            spc = spc + Kj * (a * spec(c, lh))[..., None]
    return L, spc


def lights_rgb64(faces, fim, wmap, dmap, corner_shading, params, lights, unlit, bg, aa):
    """API rgb [B,3,H,W]: L s + the specular colour where covered, the background elsewhere, 2x2 mean with anti-aliasing;
    unlit [B,3,S,S]"""
    L, spc = lights_terms64(faces, fim, wmap, dmap, corner_shading, params, lights)
    lit = L * unlit.double().permute(0, 2, 3, 1) + spc
    rgb = torch.where((fim >= 0)[..., None], lit, _bg(bg, fim.device)).permute(0, 3, 1, 2)
    return torch.nn.functional.avg_pool2d(rgb, 2, 2) if aa else rgb
