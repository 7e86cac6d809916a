"""float64 restatement of smooth shading (include/nr_b200.h, corner_light) on the product's own maps: the per-pixel light
interpolated from the corner factors, and the lit API image from an unlit raster sample (oracles.py's samplers, or the
product's bit-exact unlit render)."""
import torch

from oracles import _bg


def smooth_light64(faces, fim, wmap, dmap, corner_light):
    """float64 per-pixel light [B,S,S,3]: l_k = w_k zp / z_k with the winner's own vertex depths, L_c = sum_k l_k C_kc.
    corner_light [B,F,3,3] may require grad."""
    dev = fim.device
    B = faces.shape[0]
    S = fim.shape[-1]
    fi = fim.clamp(min=0).long()
    bidx = torch.arange(B, device=dev)[:, None, None].expand(B, S, S)
    z = faces.double()[..., 2][bidx, fi]
    # an uncovered pixel reads face 0, which may have a zero depth (an out-of-range index): keep 0 * inf out of autograd
    z = torch.where((fim >= 0)[..., None], z, torch.ones_like(z))
    lam = wmap.double().permute(0, 2, 3, 1) * (dmap.double()[..., None] / z)   # [B,S,S,3]
    C = corner_light.double()[bidx, fi]                                         # [B,S,S,3 corners,3]
    return (lam[..., None] * C).sum(dim=3)


def smooth_rgb(unlit, light, fim, bg, aa):
    """API rgb [B,3,H,W] from the unlit raster sample [B,3,S,S] and smooth_light64: lit where covered, background
    elsewhere, 2x2 mean with anti-aliasing"""
    rgb = torch.where((fim >= 0)[..., None], light * unlit.double().permute(0, 2, 3, 1), _bg(bg, fim.device))
    rgb = rgb.permute(0, 3, 1, 2)
    return torch.nn.functional.avg_pool2d(rgb, 2, 2) if aa else rgb
