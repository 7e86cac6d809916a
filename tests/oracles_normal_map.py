"""float64 restatement of Phong shading through a tangent-space normal map (include/nr_b200.h, nr_b200_normal_map_args) on
the product's own maps: the mapped normal n' = m_x t + m_y b + m_z n with t = sum_k l_k T_k, b = sigma (n x t) and m the
map's bilinear sample at the pixel's uv, then the light-set / SH expression of oracles_sh.py with n' in place of n.
Differentiable: corner_shading, params, lights, sh, the map, the tangents, the unlit sample and (through the
straight-through uv of oracles_uv_grad.py, the cell and clamp held fixed) the UVs may require grad."""
import torch

from oracles import _bg
from oracles_phong import _norm
from oracles_sh import sh_basis64
from oracles_uv_grad import _bilinear, _pixel_uvs


def _lam(faces, fim, wmap, dmap):
    dev = fim.device
    B, S = faces.shape[0], fim.shape[-1]
    fi = fim.clamp(min=0).long()
    bidx = torch.arange(B, device=dev)[:, None, None].expand(B, S, S)
    z = faces.double()[..., 2][bidx, fi]
    z = torch.where((fim >= 0)[..., None], z, torch.ones_like(z))  # keep 0 * inf of uncovered pixels out of autograd
    return bidx, fi, wmap.double().permute(0, 2, 3, 1) * (dmap.double()[..., None] / z)


def _per_item(t, bidx, fi):
    return t[bidx if t.shape[0] > 1 else torch.zeros_like(bidx), fi]


def map_sample64(faces, fim, wmap, dmap, uvs, normal_map, fill_back):
    """m [B,S,S,3]: the map's bilinear sample at the pixel's (fp32, clamped) uv, differentiable in the map and the UVs"""
    B = faces.shape[0]
    bidx, _, _, uv_raw, st = _pixel_uvs(faces, fim, wmap, dmap, uvs, fill_back, z64=False)
    nm = normal_map.double().expand(B, -1, -1, -1)
    return _bilinear(nm, torch.nan_to_num(uv_raw.clamp(0, 1)), st, bidx, None)


def mapped_normal64(faces, fim, wmap, dmap, corner_shading, corner_tangents, m):
    """(n', n, t, b) [B,S,S,3] of the header's frame: n and t interpolated and not renormalised, sigma the majority vote"""
    bidx, fi, lam = _lam(faces, fim, wmap, dmap)
    C = _per_item(corner_shading.double(), bidx, fi)                       # [B,S,S,3,6]
    T = _per_item(corner_tangents.double(), bidx, fi)                      # [B,S,S,3,4]
    n = (lam[..., None] * C[..., :3]).sum(dim=3)
    t = (lam[..., None] * T[..., :3]).sum(dim=3)
    sigma = torch.where(T[..., 3].sum(-1) < 0, -1.0, 1.0).to(n.dtype)[..., None]
    b = sigma * torch.linalg.cross(n, t, dim=-1)
    return m[..., 0:1] * t + m[..., 1:2] * b + m[..., 2:3] * n, n, t, b


def nm_terms64(faces, fim, wmap, dmap, corner_shading, params, lights, sh, n):
    """per raster pixel [B,S,S,...]: the light L [.,3] and the specular colour [.,3] of the light-set / SH expression at the
    normal n [B,S,S,3] (the mapped one), float64; the rest as oracles_lights.lights_terms64 / oracles_sh.sh_terms64"""
    bidx, fi, lam = _lam(faces, fim, wmap, dmap)
    B = faces.shape[0]
    C = _per_item(corner_shading.double(), bidx, fi)
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
    return L, spc


def nm_rgb64(faces, fim, wmap, dmap, corner_shading, params, lights, sh, normal_map, corner_tangents, uvs, unlit, bg, aa,
             fill_back):
    """API rgb [B,3,H,W]: L s + the specular colour where covered, the background elsewhere, 2x2 mean with anti-aliasing;
    unlit [B,3,S,S], uvs [1|B,F',3,2] (F' = F/2 with fill_back: the copies read the corners reversed)"""
    m = map_sample64(faces, fim, wmap, dmap, uvs, normal_map, fill_back)
    n = mapped_normal64(faces, fim, wmap, dmap, corner_shading, corner_tangents, m)[0]
    L, spc = nm_terms64(faces, fim, wmap, dmap, corner_shading, params, lights, sh, n)
    lit = L * unlit.double().permute(0, 2, 3, 1) + spc
    rgb = torch.where((fim >= 0)[..., None], lit, _bg(bg, fim.device)).permute(0, 3, 1, 2)
    return torch.nn.functional.avg_pool2d(rgb, 2, 2) if aa else rgb
