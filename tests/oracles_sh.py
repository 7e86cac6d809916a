"""float64 restatement of Phong shading with an SH environment (include/nr_b200.h, nr_b200_sh_args) on the product's own
maps: the light-set expression of oracles_lights.py with the irradiance E_c = sum_k S[k][c] Y_k(nh) added to the light
after every diffuse term, nh = n / (|n| + 1e-5) used as is (not renormalised), as the header writes it.  Differentiable:
corner_shading, params, lights, sh and the unlit sample may require grad."""
import math

import torch

from oracles import _bg
from oracles_lights import lights_terms64
from oracles_phong import _norm

C0, C1, C2, C3, C4 = (0.5 / math.sqrt(math.pi), math.sqrt(3 / (4 * math.pi)), math.sqrt(15 / (4 * math.pi)),
                      math.sqrt(5 / (16 * math.pi)), math.sqrt(15 / (16 * math.pi)))


def sh_basis64(d):
    """the header's 9 basis functions at d [...,3] (used as given) -> [...,9]"""
    x, y, z = d.unbind(-1)
    return torch.stack([torch.full_like(x, C0), C1 * y, C1 * z, C1 * x, C2 * x * y, C2 * y * z, C3 * (3 * z * z - 1),
                        C2 * x * z, C4 * (x * x - y * y)], dim=-1)


def shading_normal64(faces, fim, wmap, dmap, corner_shading):
    """nh [B,S,S,3] of the Phong expression, float64 (the interpolation of lights_terms64)"""
    dev = fim.device
    B, S = faces.shape[0], fim.shape[-1]
    fi = fim.clamp(min=0).long()
    bidx = torch.arange(B, device=dev)[:, None, None].expand(B, S, S)
    z = faces.double()[..., 2][bidx, fi]
    z = torch.where((fim >= 0)[..., None], z, torch.ones_like(z))
    lam = wmap.double().permute(0, 2, 3, 1) * (dmap.double()[..., None] / z)
    cs = corner_shading.double()
    C = cs[bidx if cs.shape[0] > 1 else torch.zeros_like(bidx), fi]
    return _norm((lam[..., None] * C[..., :3]).sum(dim=3))


def sh_terms64(faces, fim, wmap, dmap, corner_shading, params, lights=None, sh=None):
    """per raster pixel [B,S,S,...]: the light L [.,3] (every light's diffuse term, then E) and the specular colour [.,3],
    float64.  sh [1|B,9,3] or None; the rest as lights_terms64."""
    L, spc = lights_terms64(faces, fim, wmap, dmap, corner_shading, params, lights)
    if sh is not None:
        B = faces.shape[0]
        Y = sh_basis64(shading_normal64(faces, fim, wmap, dmap, corner_shading))       # [B,S,S,9]
        S = sh.double().expand(B, 9, 3)
        L = L + torch.einsum('bijk,bkc->bijc', Y, S)
    return L, spc


def sh_rgb64(faces, fim, wmap, dmap, corner_shading, params, lights, sh, unlit, bg, aa):
    """API rgb [B,3,H,W]: L s + the specular colour where covered, the background elsewhere, 2x2 mean with anti-aliasing;
    unlit [B,3,S,S]"""
    L, spc = sh_terms64(faces, fim, wmap, dmap, corner_shading, params, lights, sh)
    lit = L * unlit.double().permute(0, 2, 3, 1) + spc
    rgb = torch.where((fim >= 0)[..., None], lit, _bg(bg, fim.device)).permute(0, 3, 1, 2)
    return torch.nn.functional.avg_pool2d(rgb, 2, 2) if aa else rgb
