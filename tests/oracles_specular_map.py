"""float64 restatement of Phong shading through a specular map (include/nr_b200.h, nr_b200_specular_map_args) on the
product's own maps: the map's bilinear sample (ks, sigma') at the pixel's uv (oracles_normal_map.map_sample64's sampler
with four channels), then the light-set / SH / normal-map expression of oracles_normal_map.py with every highlight
multiplied by ks and sigma' in place of params' shininess.  Differentiable as oracles_normal_map.py, and in the map."""
import torch

from oracles import _bg
from oracles_normal_map import _lam, _per_item, map_sample64, mapped_normal64, nm_terms64
from oracles_phong import _norm
from oracles_sh import sh_basis64


def sm_sample64(faces, fim, wmap, dmap, uvs, specular_map, fill_back):
    """(ks [B,S,S,3], sigma' [B,S,S]): the map's bilinear sample at the pixel's (fp32, clamped) uv"""
    q = map_sample64(faces, fim, wmap, dmap, uvs, specular_map, fill_back)
    return q[..., :3], q[..., 3]


def sm_terms64(faces, fim, wmap, dmap, corner_shading, params, lights, sh, n, ks, sig):
    """nm_terms64 with the specular colour of every light times ks [B,S,S,3] and the per-pixel shininess sig [B,S,S]"""
    bidx, fi, lam = _lam(faces, fim, wmap, dmap)
    B = faces.shape[0]
    C = _per_item(corner_shading.double(), bidx, fi)
    p = (lam[..., None] * C[..., 3:]).sum(dim=3)
    prm = params.double().expand(B, 16)[:, None, None, :]
    A, D, d, K, e = prm[..., 0:3], prm[..., 3:6], prm[..., 6:9], prm[..., 9:12], prm[..., 13:16]
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
            rec = lt[:, j][:, None, None, :]
            Dj, Kj, x, f = rec[..., 0:3], rec[..., 3:6], rec[..., 6:9], rec[..., 9]
            point = rec[..., 10] > 0.5
            u = torch.where(point[..., None], x - p, x.expand_as(p))
            r = torch.linalg.vector_norm(u, dim=-1)
            lh = u / (r[..., None] + 1e-5)
            c = torch.where(point, (nh * lh).sum(-1), (nh * x).sum(-1))
            a = torch.where(point, 1 / (1 + f * r * r), torch.ones_like(r))
            L = L + Dj * (a * torch.relu(c))[..., None]
            spc = spc + Kj * (a * spec(c, lh))[..., None]
    if sh is not None:
        L = L + torch.einsum('bijk,bkc->bijc', sh_basis64(nh), sh.double().expand(B, 9, 3))
    return L, ks * spc


def sm_rgb64(faces, fim, wmap, dmap, corner_shading, params, lights, sh, normal_map, corner_tangents, specular_map, uvs,
             unlit, bg, aa, fill_back):
    """API rgb [B,3,H,W] as oracles_normal_map.nm_rgb64, through the specular map (normal_map None: the interpolated
    normal; specular_map None: nm_terms64 itself)"""
    if normal_map is not None:
        m = map_sample64(faces, fim, wmap, dmap, uvs, normal_map, fill_back)
        n = mapped_normal64(faces, fim, wmap, dmap, corner_shading, corner_tangents, m)[0]
    else:
        bidx, fi, lam = _lam(faces, fim, wmap, dmap)
        n = (lam[..., None] * _per_item(corner_shading.double(), bidx, fi)[..., :3]).sum(dim=3)
    if specular_map is None:
        L, spc = nm_terms64(faces, fim, wmap, dmap, corner_shading, params, lights, sh, n)
    else:
        ks, sig = sm_sample64(faces, fim, wmap, dmap, uvs, specular_map, fill_back)
        L, spc = sm_terms64(faces, fim, wmap, dmap, corner_shading, params, lights, sh, n, ks, sig)
    lit = L * unlit.double().permute(0, 2, 3, 1) + spc
    rgb = torch.where((fim >= 0)[..., None], lit, _bg(bg, fim.device)).permute(0, 3, 1, 2)
    return torch.nn.functional.avg_pool2d(rgb, 2, 2) if aa else rgb
