"""GPU: the soft rasterizer where its tile binning changes shape, held to the float64 oracles in their sparse mode
(tests/oracles_soft*.py, pix=): 64-bit sort keys, tiles whose lists take several staging rounds, texture cubes past
the backward's per-warp shared-memory budget, the benchmarks' B 64 x F 5000 spheres, and slivers.  Every section
asserts that its scene reaches its branch (tests/soft_binning.py).

Forward gates (DESIGN.md sections 4o-4q).  Where at most five faces are on at a pixel the gates of
tests/test_gpu_soft*.py hold: tol(sigma) for alpha, 4 tol(sigma) + 6e-4 for rgb.  Where more are on, their five-face
assumption fails, and the bound is derived per pixel from the oracle's own terms of every face j on there:
  alpha: (1 - alpha) sum_j D_j (1 - D_j) |dx_j| + n 2^-40 + 4 eps, with |dx_j| <= (2 d_j delta + delta^2 + 4 eps d_j^2)
         / sigma and delta = 4 eps max(1, |v|) (a few ulps of the face's coordinate magnitude), eps = 2^-23;
  rgb:   sum_j (w_j / Z) [(|C_j| + |rgb|) e_j + |dC_j|], with e_j = |dx_j| (1 - D_j) + |dzp_j| / ((far - near) gamma) +
         8 eps (the rounding of the weight itself), |dzp_j| <= 8 eps zp + 3 dl_j zp^2 / min z, dl_j = 8 eps |e| (|e| + d_j)
         / |A| the barycentrics' error, and |dC_j| = 4 eps |C_j| + k_C dl_j (k_C: the colour's change per unit of l).
Each derived bound is multiplied by SAFETY.  Pixels within 2e-5 of the cut-off of some face are left out, since the
fp32 cut-off test may decide them either way (the bracketed tests of sections 4o-4q cover that); the tests assert these
pixels are rare.  A pixel over its gate is reported with its count of faces on.

Measured on an H100 80GB HBM3 at a 700 W power limit, one run (largest error / gate over the checked pixels; the tests
print them with -s): deep tiles alpha 0.026, rgb 0.013 (cube, gamma 1e-4); benchmark geometry alpha 0.022, rgb 0.0075
(cube), 0.0043 (UV).  The file ran in 50 s with 4.7 GB peak device memory."""
import ctypes
import math

import numpy as np
import pytest
import torch

import oracles
import oracles_soft as osoft
import oracles_soft_rgb as orgb
import oracles_soft_uv as ouv
import soft_binning as sb
from helpers import elem_err, rel_err

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
NEAR, FAR = 0.1, 100.0
EPS32 = 2.0 ** -23
SAFETY = 4.0


def _nr():
    import neural_renderer_b200 as nr
    return nr


def tol(sigma):
    return 1e-6 / math.sqrt(sigma) + 1e-6


def tol_rgb(sigma):
    return 4 * tol(sigma) + 6e-4


# ------------------------------------------------------------------------------------------------ oracle and gates
class Scene:
    """one render's inputs: faces [B,F,3,3] float32; cubes [1|B,F,ts,ts,ts,3] or image [1|B,H,W,3] with uvs
    [1|B,F,3,2] (tri = trilinear); light [B,F,3] or None.  kind: 'sil', 'cube' or 'uv'."""

    def __init__(self, kind, faces, tex=None, uvs=None, light=None, tri=False, bg=(0.2, 0.4, 0.6)):
        self.kind, self.faces, self.tex, self.uvs, self.light, self.tri, self.bg = kind, faces, tex, uvs, light, tri, bg

    def render(self, S, sigma, gamma, faces=None, tex=None, uvs=None, light=None, vertices=None):
        nr = _nr()
        faces = self.faces if faces is None else faces
        tex = self.tex if tex is None else tex
        uvs = self.uvs if uvs is None else uvs
        light = self.light if light is None else light
        if self.kind == "sil":
            return None, nr.rasterize_soft_silhouettes(faces, S, sigma, vertices=vertices)
        kw = dict(background_color=self.bg, face_light=light, vertices=vertices)
        if self.kind == "uv":
            kw.update(face_uvs=uvs, texture_filter='trilinear' if self.tri else 'bilinear')
        return nr.rasterize_soft(faces, tex, S, sigma, gamma, **kw)

    def leaves(self):
        out = [self.faces]
        if self.kind != "sil":
            out.append(self.tex)
            if self.kind == "uv":
                out.append(self.uvs)
            if self.light is not None:
                out.append(self.light)
        return out

    def oracle_terms(self, leaves, S, sigma, cut_scale=1.0):
        """terms(b0, b1, idx, fc, p) of osoft.sparse_eval for this scene, with leaves in the order of leaves()"""
        if self.kind == "sil":
            def terms(b0, b1, idx, fc, p):
                d2, inside = osoft.face_terms(fc, p)
                x = torch.where(inside, d2 / sigma, -d2 / sigma)
                on = osoft.participates(fc, NEAR, FAR)[..., None] & (inside | (d2 <= osoft.cut(sigma) * cut_scale))
                zn = torch.zeros_like(x)
                return x, on, on, zn, torch.zeros(*x.shape, 3, dtype=x.dtype, device=x.device)
            return terms
        tex = leaves[1].double()
        light = leaves[-1] if self.light is not None else None
        if self.kind == "cube":
            def terms(b0, b1, idx, fc, p):
                fl = None if light is None else osoft.take(light, b0, b1, idx)
                return orgb.cube_terms(fc, osoft.take(tex, b0, b1, idx), p, sigma, NEAR, FAR, 1e-4, fl, cut_scale)
            return terms
        uvs = leaves[2].double()
        if self.tri:
            hw = tuple(tex.shape[1:3])
            tex = torch.cat([x.reshape(x.shape[0], -1, 3) for x in oracles.pyramid64(tex)], 1)
        else:
            hw = None

        def terms(b0, b1, idx, fc, p):
            tc = tex[b0:b1] if tex.shape[0] > 1 else tex.expand(b1 - b0, *tex.shape[1:])
            fl = None if light is None else osoft.take(light, b0, b1, idx)
            return ouv.uv_terms(fc, tc, osoft.take(uvs, b0, b1, idx), p, S, sigma, NEAR, FAR, fl, hw, cut_scale)
        return terms

    def colour_sensitivity(self):
        """k_C: a bound of |dC| per unit change of the barycentrics, per (item, face) [B|1,F]"""
        B, F = self.faces.shape[:2]
        lmax = 1.0 if self.light is None else self.light.abs().amax(-1).double()
        if self.kind == "sil":
            return torch.zeros(1, F, dtype=torch.float64, device=DEV)
        if self.kind == "cube":
            t = self.tex.double().reshape(self.tex.shape[0], F, -1, 3)
            span = (t.amax(2) - t.amin(2)).amax(-1)                     # [Bt,F]
            return 3 * (self.tex.shape[2] - 1) * span * lmax
        img = self.tex.double()
        step = max((img[:, 1:] - img[:, :-1]).abs().max().item() if img.shape[1] > 1 else 0.0,
                   (img[:, :, 1:] - img[:, :, :-1]).abs().max().item() if img.shape[2] > 1 else 0.0)
        uv = self.uvs.double()
        span = (uv.amax(2) - uv.amin(2)).amax(-1) * max(img.shape[1:3])   # [Bu,F] texels per unit of l
        return 3 * span * step * lmax


def _gate_terms(scene, terms, sigma, gamma, ksens):
    """terms of sparse_eval that add, per (item, face, pixel), what the derived gates need"""
    def gt(b0, b1, idx, fc, p):
        x, on, valid, zn, C = terms(b0, b1, idx, fc, p)
        d2 = x.abs() * sigma
        d = d2.sqrt()
        delta = 4 * EPS32 * fc[..., :2].abs().flatten(2).amax(2).clamp_min(1.0)[..., None]        # [B,F,1]
        dx = (2 * d * delta + delta ** 2 + 4 * EPS32 * d2) / sigma
        a = fc[..., :2]
        elen = (a.roll(-1, dims=2) - a).norm(dim=-1).amax(2)[..., None]                         # [B,F,1]
        A = orgb.doubled_area(fc).abs()[..., None]
        dl = 8 * EPS32 * elen * (elen + d) / torch.where(A > 0, A, torch.ones_like(A))
        zp = FAR - zn * (FAR - NEAR)
        zmin = fc[..., 2].amin(2)[..., None].clamp_min(NEAR)
        dzp = 8 * EPS32 * zp + 3 * dl * zp * zp / zmin
        k = osoft.take(ksens[..., None], b0, b1, idx)                                         # [B,F,1]
        dC = 4 * EPS32 * C.abs() + (k * dl)[..., None]
        part = osoft.participates(fc, NEAR, FAR)[..., None]
        edge = part & (x < 0) & ((d2 - osoft.cut(sigma)).abs() <= 2e-5 * osoft.cut(sigma))
        return x, on, valid, zn, C, dx, dzp, dC, edge
    return gt


def _gate_blend(gamma, bg):
    def first(r):
        return orgb.zmax_of(r[0], r[1]).clamp_min(orgb.BG_DEPTH)

    def partial(x, r, zmax):
        valid, zn, C, dx, dzp, dC, edge = r
        D = torch.sigmoid(x)
        s0, s1 = orgb.blend_sums(x, valid, zn, C, zmax, gamma)
        ex = torch.where(valid, (zn - zmax[:, None]) / gamma, torch.full_like(zn, -math.inf))
        w = torch.where(valid, D * torch.exp(ex), torch.zeros_like(D))
        e = dx * (1 - D) + dzp / ((FAR - NEAR) * gamma) + 8 * EPS32
        return (s0, s1, (w[..., None] * C.abs() * e[..., None]).sum(1), (w * e).sum(1),
                (w[..., None] * dC).sum(1), edge.sum(1).double())

    def finish(sums, zmax):
        s0, s1, r1, r2, r3, edge = sums
        rgb = orgb.blend_finish((s0, s1), zmax, gamma, bg)
        Z = s0 + torch.exp((orgb.BG_DEPTH - zmax) / gamma)
        bound = (r1 + rgb.abs() * r2[..., None] + r3) / Z[..., None]
        return torch.cat((rgb, bound, edge[..., None]), -1)                                       # [B,P,7]
    return first, partial, finish


def _alpha_terms(terms, sigma):
    """per pixel: the count of faces on and sum_j D_j (1 - D_j) |dx_j| (sparse_eval of the silhouette part)"""
    def at(b0, b1, idx, fc, p):
        x, on = terms(b0, b1, idx, fc, p)[:2]
        d2 = x.abs() * sigma
        delta = 4 * EPS32 * fc[..., :2].abs().flatten(2).amax(2).clamp_min(1.0)[..., None]
        dx = (2 * d2.sqrt() * delta + delta ** 2 + 4 * EPS32 * d2) / sigma
        D = torch.sigmoid(x)
        return x, on, on, torch.where(on, D * (1 - D) * dx, torch.zeros_like(x))
    return at


def _count_blend():
    return (lambda r: torch.zeros(r[0].shape[0], r[0].shape[2], dtype=torch.float64, device=r[0].device),
            lambda x, r, ref: (r[0].sum(1).double(), r[1].sum(1)),
            lambda sums, ref: torch.stack(sums, -1))


def check_forward(scene, rgb, alpha, S, sigma, gamma, pix, what, terms=None, cull=1.0):
    """rgb [B,3,S,S] (or an attribute image [B,C,S,S]) / alpha [B,S,S] at the pixels pix [B,P] against the sparse
    oracle under the gates of the docstring; returns the largest error / gate ratios seen, for the record.  terms: the
    oracle's terms at the kernel's own selection (tests/soft_selection.py), culled at the cut-off scale `cull`; the
    fp32 cut-off decision is then the oracle's too, so the pixels near the cut-off are checked like every other."""
    B = scene.faces.shape[0]
    leaves = [x.detach() for x in scene.leaves()]
    selected = terms is not None
    if not selected:
        terms = scene.oracle_terms(leaves, S, sigma)
    with torch.no_grad():
        a_or, ac = osoft.sparse_eval(leaves[0], S, pix, sigma, NEAR, FAR, cull, _alpha_terms(terms, sigma),
                                     _count_blend())
        n, sdx = ac[..., 0], ac[..., 1]
        _, g = osoft.sparse_eval(leaves[0], S, pix, sigma, NEAR, FAR, cull,
                                 _gate_terms(scene, terms, sigma, gamma, scene.colour_sensitivity()),
                                 _gate_blend(gamma, scene.bg))
    edge = g[..., -1] > 0
    if selected:
        edge = torch.zeros_like(edge)
    assert edge.double().mean().item() <= 0.01, (what, edge.double().mean().item())
    flat = lambda t: t.reshape(B, *t.shape[1:-2], S * S)   # noqa: E731
    got_a = torch.gather(flat(alpha).double(), 1, pix)
    lam = -torch.log1p(-a_or.clamp(max=1 - 1e-16))
    gate_a = torch.where(n <= 5, torch.full_like(a_or, tol(sigma)),
                         SAFETY * ((1 - a_or) * sdx + n * 2.0 ** -40 + 4 * EPS32 * (1 + (1 - a_or) * lam.clamp(max=64))))
    err_a = (got_a - a_or).abs()
    worst = {}
    bad = (err_a > gate_a) & ~edge
    assert not bad.any(), (what, "alpha", [(int(b), int(pix[b, i]), int(n[b, i]), err_a[b, i].item(), gate_a[b, i].item())
                                           for b, i in bad.nonzero()[:8]])
    worst["alpha"] = (err_a / gate_a).masked_fill(edge, 0).max().item()
    if rgb is not None:
        nc = rgb.shape[1]                                   # 3, or the channels of an attribute image
        got = torch.gather(flat(rgb).double(), 2, pix[:, None].expand(-1, nc, -1)).permute(0, 2, 1)
        err = (got - g[..., :nc]).abs()
        gate = torch.where((n <= 5)[..., None], torch.full_like(err, tol_rgb(sigma)), SAFETY * g[..., nc:2 * nc])
        bad = (err > gate) & ~edge[..., None]
        assert not bad.any(), (what, "rgb", [(int(b), int(pix[b, i]), int(n[b, i]), err[b, i, c].item(), gate[b, i, c].item())
                                             for b, i, c in bad.nonzero()[:8]])
        worst["rgb"] = (err / gate).masked_fill(edge[..., None], 0).max().item()
    return worst


def oracle_grads(scene, S, sigma, gamma, pix, g_rgb, g_a, items=4):
    """float64 autograd gradients of sum(rgb g_rgb) + sum(alpha g_a) at the pixels pix [B,P] (g_* [B,3,P] / [B,P]),
    the items taken `items` at a time so that the graph stays small"""
    leaves = [x.detach().double().requires_grad_(True) for x in scene.leaves()]
    B = scene.faces.shape[0]
    for b0 in range(0, B, items):
        b1 = min(B, b0 + items)
        sl = [x[b0:b1] if x.shape[0] > 1 else x for x in leaves]
        terms = scene.oracle_terms(sl, S, sigma)
        if scene.kind == "sil":
            alpha = osoft.sparse_eval(sl[0], S, pix[b0:b1], sigma, NEAR, FAR, 1.0, terms)[0]
            loss = (alpha * g_a[b0:b1].double()).sum()
        else:
            alpha, rgb = osoft.sparse_eval(sl[0], S, pix[b0:b1], sigma, NEAR, FAR, 1.0, terms,
                                           orgb.softmax_blend(gamma, scene.bg))
            loss = (rgb * g_rgb[b0:b1].double()).sum() + (alpha * g_a[b0:b1].double()).sum()
        loss.backward()
    return [torch.zeros_like(x) if x.grad is None else x.grad for x in leaves]


def kernel_grads(scene, S, sigma, gamma, g_rgb, g_a):
    leaves = [x.detach().clone().requires_grad_(True) for x in scene.leaves()]
    kw = dict(faces=leaves[0])
    if scene.kind != "sil":
        kw["tex"] = leaves[1]
        if scene.kind == "uv":
            kw["uvs"] = leaves[2]
        if scene.light is not None:
            kw["light"] = leaves[-1]
    rgb, alpha = scene.render(S, sigma, gamma, **kw)
    loss = (alpha * g_a).sum() + ((rgb * g_rgb).sum() if rgb is not None else 0)
    loss.backward()
    return [x.grad for x in leaves]


def check_grads(got, ref, names, what):
    for name, a, r in zip(names, got, ref):
        a, r = a.double().cpu().numpy(), r.cpu().numpy()
        assert np.isfinite(a).all(), (what, name)
        assert rel_err(a, r) <= 5e-3, (what, name, rel_err(a, r))
        assert elem_err(a, r, floor=2e-2) <= 5e-2, (what, name, elem_err(a, r, floor=2e-2))


def names_of(scene):
    out = ["faces"]
    if scene.kind != "sil":
        out.append("textures")
        if scene.kind == "uv":
            out.append("face_uvs")
        if scene.light is not None:
            out.append("face_light")
    return out


def _image(Bt, H, W, seed):
    """a smooth image, values in [0.1, 0.9] (as tests/test_gpu_soft_uv.py)"""
    g = torch.Generator().manual_seed(seed)
    y = torch.linspace(0, 1, H, dtype=torch.float64)[:, None]
    x = torch.linspace(0, 1, W, dtype=torch.float64)[None]
    out = []
    for _ in range(Bt):
        ph = torch.rand(3, 2, generator=g, dtype=torch.float64) * 6.28
        out.append(torch.stack([0.5 + 0.2 * torch.sin(2.0 * x + ph[c, 0]) * torch.cos(1.5 * y + ph[c, 1]) + 0.15 * x * y
                                for c in range(3)], -1))
    return torch.stack(out).float().to(DEV)


def _rand(shape, seed, lo=0.0, hi=1.0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return lo + (hi - lo) * torch.rand(*shape, device=DEV, generator=g)


# ------------------------------------------------------------------------------------------------ a. key width
S_KEY, SIGMA_KEY, GAMMA_KEY = 2049, 1e-4, 1e-3


def _real_faces(B, seed):
    """about 200 faces per item, different per item: a soup, the silhouette tests' special faces, and wide faces"""
    from neural_renderer_b200 import synthetic
    soup = torch.from_numpy(synthetic.triangle_soup(B, 176, seed=seed, size=(0.02, 0.3), duplicates=False))
    reach = math.sqrt(osoft.cut(SIGMA_KEY))
    o = 1.0 + 0.5 * reach
    extra = [[[-1.1, -1.0, 2.5], [1.2, -0.9, 2.6], [0.1, 1.3, 2.4]],
             [[-0.9, 0.95, 2.0], [0.9, 0.9, 2.0], [0.0, 0.97, 2.0]],
             [[o, -0.3, 1.2], [o + 0.2, 0.0, 1.2], [o, 0.3, 1.2]],
             [[-0.3, -o, 1.2], [0.3, -o, 1.2], [0.0, -o - 0.2, 1.2]],
             [[-0.5, 0.1, 0.05], [-0.2, 0.1, 1.0], [-0.4, 0.4, 1.0]],
             [[0.2, -0.5, 1.0], [0.5, -0.5, 150.0], [0.3, -0.2, 1.0]],
             [[-0.6, -0.6, 1.0], [-0.2, -0.2, 1.0], [-0.4, -0.4, 1.0]],
             [[0.6, 0.2, 1.0], [0.6, 0.2, 1.0], [0.6, 0.2, 1.0]],
             # the last tile row and column of the raster: faces on the right and bottom borders
             [[0.97, -0.2, 1.5], [1.02, -0.1, 1.5], [0.99, 0.05, 1.5]],
             [[-0.2, -0.98, 1.6], [0.1, -1.01, 1.6], [0.0, -0.96, 1.6]]]
    ex = torch.tensor(extra, dtype=torch.float32)[None].expand(B, -1, -1, -1)
    return torch.cat((soup, ex), 1).contiguous().to(DEV)


_PAD = [[[0.0, 0.0, 2.0], [0.1, 0.0, 150.0], [0.0, 0.1, 2.0]],                    # a vertex beyond far
        [[0.0, 0.0, 2.0], [0.1, 0.0, 0.05], [0.0, 0.1, 2.0]],                     # a vertex nearer than near
        [[float("nan"), 0.0, 2.0], [0.1, 0.0, 2.0], [0.0, 0.1, 2.0]],             # NaN x
        [[0.0, 0.0, 2.0], [0.1, float("inf"), 2.0], [0.0, -float("inf"), 2.0]]]   # +-inf y


def _padded(real, F, seed):
    """(faces [B,F,3,3], positions of the real faces [Fr]): the real faces in their order at scattered indices, F - 1
    among them, every other slot one of the four kinds of padding face"""
    B, Fr = real.shape[:2]
    if F == Fr:
        return real, torch.arange(Fr, device=DEV)
    rng = np.random.default_rng(seed)
    pos = np.sort(np.concatenate((rng.choice(F - 1, Fr - 1, replace=False), [F - 1])))
    pos = torch.from_numpy(pos).to(DEV)
    pad = torch.tensor(_PAD, dtype=torch.float32, device=DEV)
    faces = pad[torch.arange(F, device=DEV) % 4][None].repeat(B, 1, 1, 1)
    faces[:, pos] = real
    return faces, pos


def _indexed(faces, pos):
    """vertices [B,3 Fr + 12,3] and shared indices [F,3] of the same faces: the real faces' corners, then the four
    padding faces' corners, which every padding slot indexes"""
    B, F = faces.shape[:2]
    Fr = pos.numel()
    pad = torch.tensor(_PAD, dtype=torch.float32, device=DEV).reshape(1, 12, 3).expand(B, -1, -1)
    verts = torch.cat((faces[:, pos].reshape(B, 3 * Fr, 3), pad), 1).contiguous()
    idx = (3 * Fr + 3 * (torch.arange(F, device=DEV) % 4))[:, None] + torch.arange(3, device=DEV)[None]
    idx[pos] = torch.arange(3 * Fr, device=DEV).reshape(Fr, 3)
    return verts, idx.to(torch.int32).contiguous()


def _key_scene(kind, real):
    B, Fr = real.shape[:2]
    light = _rand((B, Fr, 3), 11, 0.5, 1.5)
    if kind == "sil":
        return Scene("sil", real)
    if kind in ("cube", "cube_shared"):
        return Scene("cube", real, tex=_rand((1 if kind == "cube_shared" else B, Fr, 3, 3, 3, 3), 12), light=light)
    uvs = _rand((B, Fr, 3, 2), 13, 0.05, 0.95)
    return Scene("uv", real, tex=_image(1, 40, 56, 14), uvs=uvs, light=light, tri=kind == "uv_tri")


def _spread(t, pos, F, fill=0.0):
    """per-face data [Bt,Fr,...] of the real faces at their slots of F; padding slots get `fill`"""
    out = torch.full((t.shape[0], F) + tuple(t.shape[2:]), fill, dtype=t.dtype, device=DEV)
    out[:, pos] = t
    return out.contiguous()


def _workspace(B, F, S, flags=0):
    from neural_renderer_b200 import _lib
    return _lib.load().nr_b200_soft_rgb_workspace_bytes(B, F, S, flags)


def _state(faces, tex, light, S, sigma, gamma, bg):
    """(rgb, alpha, state) of nr_b200_soft_rgb called directly"""
    from neural_renderer_b200 import _lib
    lib = _lib.load()
    B, F = faces.shape[:2]
    a = _lib.SoftRgbArgs()
    a.struct_size = ctypes.sizeof(_lib.SoftRgbArgs)
    a.flags = _lib.NR_TEX_SHARED if tex.shape[0] == 1 and B > 1 else 0
    a.faces, a.num_faces, a.batch_size, a.image_size, a.texture_size = faces.data_ptr(), F, B, S, tex.shape[2]
    a.sigma, a.gamma, a.near_, a.far_, a.eps = sigma, gamma, NEAR, FAR, 1e-4
    a.background[:] = bg
    a.textures, a.face_light = tex.data_ptr(), light.data_ptr()
    rgb = torch.empty(B, 3, S, S, device=DEV)
    alpha = torch.empty(B, S, S, device=DEV)
    state = torch.empty(B, 2, S, S, device=DEV)
    a.rgb, a.alpha, a.state = rgb.data_ptr(), alpha.data_ptr(), state.data_ptr()
    n = lib.nr_b200_soft_rgb_workspace_bytes(B, F, S, a.flags)
    ws = torch.empty(n, dtype=torch.uint8, device=DEV)
    a.workspace, a.workspace_bytes = ws.data_ptr(), n
    assert lib.nr_b200_soft_rgb(ctypes.byref(a), ctypes.c_void_p(torch.cuda.current_stream(DEV).cuda_stream)) == 0
    torch.cuda.synchronize()
    return rgb, alpha, state


def test_key_width_workspace_and_binning_shape():
    B, S = 2, S_KEY
    assert sb.key_width(B, 65535, S)[2] is False and sb.key_width(B, 65536, S)[2] is True
    n31, n32 = _workspace(B, 65534, S), _workspace(B, 65535, S)
    n64 = _workspace(B, 65536, S)
    assert n31 > 0 and n32 > 0 and n64 > 0
    keys32 = 8 * B * 65535 * 16                   # the two key arrays grow from 4 to 8 bytes per entry
    assert n32 - n31 < 4096 and n64 - n32 >= keys32, (n31, n32, n64)
    real = _real_faces(B, seed=1)
    ok, wide = sb.tile_boxes(real, S, SIGMA_KEY)[:2]
    assert wide.sum(1).min() >= 20 and not torch.equal(real[0], real[1])


def _pixels_near(real, S, n_rand, seed):
    """[B,P] pixels at the real faces' centroids and corners, in the last tile row and column, and at random"""
    B = real.shape[0]
    g = torch.Generator(device=DEV).manual_seed(seed)
    out = []
    for b in range(B):
        f = real[b][osoft.participates(real[b:b + 1].double(), NEAR, FAR)[0]]
        pts = torch.cat((f[:, :, :2].mean(1), f[:, 0, :2]), 0)
        col = ((pts[:, 0] * S + S - 1) / 2).round().long().clamp(0, S - 1)
        row = (S - 1 - (pts[:, 1] * S + S - 1) / 2).round().long().clamp(0, S - 1)
        last = torch.randint(0, S, (64,), device=DEV, generator=g)
        edge = torch.cat(((S - 1) * S + last[:32], last[32:] * S + S - 1, torch.tensor([S * S - 1], device=DEV)))
        rnd = torch.randint(0, S * S, (n_rand,), device=DEV, generator=g)
        out.append(torch.cat((row * S + col, edge, rnd)))
    n = min(x.numel() for x in out)
    return torch.stack([x[:n] for x in out])


@pytest.mark.parametrize("kind", ["sil", "cube", "cube_shared", "uv_bil", "uv_tri"])
def test_key_width_forward_and_backward_agree_across_face_counts(kind):
    B, S, sigma, gamma = 2, S_KEY, SIGMA_KEY, GAMMA_KEY
    real = _real_faces(B, seed=1)
    Fr = real.shape[1]
    base = _key_scene(kind, real)
    gen = torch.Generator(device=DEV).manual_seed(21)
    g_rgb = torch.randn(B, 3, S, S, device=DEV, generator=gen)
    g_a = torch.randn(B, S, S, device=DEV, generator=gen)
    ref_fwd, ref_bwd = None, None
    for F in (Fr, 65535, 65536):
        assert sb.key_width(B, F, S)[2] == (F == 65536)
        faces, pos = _padded(real, F, seed=F)
        pad = torch.ones(F, dtype=torch.bool, device=DEV)
        pad[pos] = False
        sc = Scene(base.kind, faces, tri=base.tri, bg=base.bg,
                   tex=None if base.tex is None else (_spread(base.tex, pos, F, 0.5) if base.kind == "cube" else base.tex),
                   uvs=None if base.uvs is None else _spread(base.uvs, pos, F, 0.5),
                   light=None if base.light is None else _spread(base.light, pos, F, 1.0))
        verts, idx = _indexed(faces, pos)
        fwd_m = sc.render(S, sigma, gamma)
        fwd_i = sc.render(S, sigma, gamma, faces=idx, vertices=verts)
        for a, b in zip(fwd_m, fwd_i):
            assert a is None or torch.equal(a, b), (kind, F)
        if ref_fwd is None:
            ref_fwd = fwd_m
            pix = _pixels_near(real, S, 400, seed=22)
            check_forward(base, fwd_m[0], fwd_m[1], S, sigma, gamma, pix, ("key", kind))
        else:
            for a, b in zip(fwd_m, ref_fwd):
                assert a is None or torch.equal(a, b), (kind, F)
        if kind == "cube":
            st = _state(faces, sc.tex, sc.light, S, sigma, gamma, sc.bg)
            assert torch.equal(st[0], fwd_m[0]) and torch.equal(st[1], fwd_m[1])
            if F == Fr:
                ref_state = st[2]
            else:
                assert torch.equal(st[2], ref_state), F
            if F == 65536:
                # no leak between the items: each item alone (32-bit keys at B = 1) renders what it rendered at B = 2
                for b in range(B):
                    one = _state(faces[b:b + 1].contiguous(), sc.tex[b:b + 1].contiguous(),
                                 sc.light[b:b + 1].contiguous(), S, sigma, gamma, sc.bg)
                    assert sb.key_width(1, F, S)[2] is False
                    assert torch.equal(one[0][0], fwd_m[0][b]) and torch.equal(one[1][0], fwd_m[1][b])
                    assert torch.equal(one[2][0], st[2][b])
        # backward: materialised and indexed
        got = kernel_grads(sc, S, sigma, gamma, g_rgb, g_a)
        vv = verts.clone().requires_grad_(True)
        leaves_i = [x.detach().clone().requires_grad_(True) for x in sc.leaves()[1:]]
        kw = {}
        if sc.kind != "sil":
            kw["tex"] = leaves_i[0]
            if sc.kind == "uv":
                kw["uvs"] = leaves_i[1]
            kw["light"] = leaves_i[-1]
        rgb_i, a_i = sc.render(S, sigma, gamma, faces=idx, vertices=vv, **kw)
        ((a_i * g_a).sum() + ((rgb_i * g_rgb).sum() if rgb_i is not None else 0)).backward()
        gv = vv.grad
        Fr3 = 3 * Fr
        assert torch.all(gv[:, Fr3:] == 0), (kind, F)                  # the padding vertices
        real_grads = [got[0][:, pos]]
        assert torch.all(got[0][:, pad] == 0), (kind, F)
        assert rel_err(gv[:, :Fr3].reshape(B, Fr, 3, 3).cpu().numpy(), got[0][:, pos].cpu().numpy()) <= 1e-5
        for name, gk, gi in zip(names_of(sc)[1:], got[1:], [x.grad for x in leaves_i]):
            if gk is None:
                continue
            if name == "textures" and sc.kind == "uv":
                real_grads.append(gk)                                    # the image does not depend on F
                assert rel_err(gi.cpu().numpy(), gk.cpu().numpy()) <= 5e-5
                continue
            assert torch.all(gk[:, pad] == 0), (kind, F, name)
            real_grads.append(gk[:, pos])
            assert rel_err(gi[:, pos].cpu().numpy(), gk[:, pos].cpu().numpy()) <= 1e-5, (kind, F, name)
        if ref_bwd is None:
            ref_bwd = real_grads
            assert real_grads[0].abs().max() > 0
        else:
            for name, a, r in zip(names_of(sc), real_grads, ref_bwd):
                # the image's gradient sums the fp32 atomics of every face and pixel, then the pyramid's backward
                lim = 5e-5 if (name == "textures" and sc.kind == "uv") else 1e-5
                assert rel_err(a.cpu().numpy(), r.cpu().numpy()) <= lim, (kind, F, name)


# ------------------------------------------------------------------------------------------------ b. deep tiles
S_DEEP, SIGMA_DEEP = 128, 1e-3


def _deep_faces(seed=31):
    """[1,F,3,3]: 3000 small faces crowded into a 48-pixel square, 400 wide faces whose boxes miss some tiles, and at
    the highest index a wide face nearer than every other, so that it arrives in the last round"""
    rng = np.random.default_rng(seed)
    n_small, n_wide = 3000, 400
    half = 48 / S_DEEP                                    # 24 pixels in NDC
    c = rng.uniform(-half, half, (n_small, 1, 2))
    r = rng.uniform(0.5, 1.5, (n_small, 1, 1)) * 2.0 / S_DEEP * 1.5
    ang = rng.uniform(0, 2 * np.pi, (n_small, 1, 1)) + np.array([0, 2.1, 4.2])[None, :, None]
    xy = c + r * np.concatenate((np.cos(ang), np.sin(ang)), -1)
    z = rng.uniform(2.0, 3.0, (n_small, 1, 1)) + rng.uniform(-1e-3, 1e-3, (n_small, 3, 1))
    small = np.concatenate((xy, z), -1)
    cw = rng.uniform(-0.6, 0.6, (n_wide, 1, 2))
    rw = rng.uniform(0.55, 0.75, (n_wide, 1, 1))
    ang = rng.uniform(0, 2 * np.pi, (n_wide, 1, 1)) + np.array([0, 2.1, 4.2])[None, :, None]
    zw = rng.uniform(2.5, 3.5, (n_wide, 1, 1)) + rng.uniform(-0.05, 0.05, (n_wide, 3, 1))
    wide = np.concatenate((cw + rw * np.concatenate((np.cos(ang), np.sin(ang)), -1), zw), -1)
    front = np.array([[[0.1, 0.1, 1.5], [0.9, 0.2, 1.5], [0.3, 0.9, 1.5]]])          # over a corner of the square
    faces = np.concatenate((small, wide, front), 0)[None].astype(np.float32)
    perm = np.concatenate((rng.permutation(n_small + n_wide), [n_small + n_wide]))   # mixed, the front face last
    return torch.from_numpy(faces[:, perm].copy()).to(DEV)


def _deep_scene(kind, faces):
    F = faces.shape[1]
    light = _rand((1, F, 3), 32, 0.5, 1.5)
    if kind == "sil":
        return Scene("sil", faces)
    if kind == "cube":
        col = _rand((1, F, 1, 1, 1, 3), 33)                 # one colour per face (see the docstring's dC)
        return Scene("cube", faces, tex=col.expand(1, F, 2, 2, 2, 3).contiguous(), light=light)
    base = _rand((1, F, 1, 2), 34, 0.1, 0.88)
    uvs = (base + _rand((1, F, 3, 2), 35, 0.0, 0.02)).contiguous()   # small UV spans
    return Scene("uv", faces, tex=_image(1, 64, 48, 36), uvs=uvs, light=light, tri=kind == "uv_tri")


def _tile_pixels(S, tiles):
    """[T,256] flat pixels of the 16 x 16 tiles `tiles` (tile ty * nt + tx)"""
    nt = sb.tiles_per_axis(S)
    i = torch.arange(256, device=DEV)
    out = []
    for t in tiles:
        ty, tx = divmod(int(t), nt)
        row, col = ty * 16 + i // 16, tx * 16 + i % 16
        out.append(torch.where((row < S) & (col < S), row.clamp(max=S - 1) * S + col.clamp(max=S - 1),
                               torch.zeros_like(row)))
    return torch.stack(out)


def test_deep_tiles_take_several_rounds():
    faces = _deep_faces()
    lb = sb.tile_entries_lower_bound(faces, S_DEEP, SIGMA_DEEP)
    ok, wide = sb.tile_boxes(faces, S_DEEP, SIGMA_DEEP)[:2]
    assert sb.rounds(lb).max().item() >= 3, lb.max().item()
    assert wide.sum().item() > sb.ROUND and wide[0, -1]          # the wide list alone takes more than one round
    tx0, tx1, ty0, ty1 = sb.tile_boxes(faces, S_DEEP, SIGMA_DEEP)[2:]
    nt = sb.tiles_per_axis(S_DEEP)
    assert ((wide & ((tx1 - tx0 + 1) * (ty1 - ty0 + 1) < nt * nt))).sum().item() > 100   # boxes that miss tiles


@pytest.mark.parametrize("gamma", [1e-4, 1e-2])
@pytest.mark.parametrize("kind", ["sil", "cube", "uv_bil", "uv_tri"])
def test_deep_tiles_forward_every_pixel_and_gradients(kind, gamma):
    S, sigma = S_DEEP, SIGMA_DEEP
    faces = _deep_faces()
    F = faces.shape[1]
    sc = _deep_scene(kind, faces)
    rgb, alpha = sc.render(S, sigma, gamma)
    # every pixel, as a batch of tiles over the one item, so that the cull works tile by tile
    nt = sb.tiles_per_axis(S)
    tiles = torch.arange(nt * nt)
    T = tiles.numel()
    tsc = Scene(sc.kind, faces.expand(T, -1, -1, -1), tex=sc.tex, uvs=sc.uvs,
                light=None if sc.light is None else sc.light, tri=sc.tri, bg=sc.bg)
    pix = _tile_pixels(S, tiles)
    worst = check_forward(tsc, None if rgb is None else rgb.expand(T, -1, -1, -1),
                          alpha.expand(T, -1, -1), S, sigma, gamma, pix, ("deep", kind, gamma))
    print("deep", kind, gamma, worst)
    # the nearest face, at the highest index, wins the pixels it covers
    if kind == "cube" and gamma == 1e-4:
        c = sc.tex[0, F - 1, 0, 0, 0] * sc.light[0, F - 1]
        assert (rgb[0, :, 45, 82] - c).abs().max() < 1e-3   # pixel (45, 82) is inside the front face
    # gradients: the upstream gradient only on the deepest tile and a tile of the front face
    lb = sb.tile_entries_lower_bound(faces, S, sigma)[0]
    deep = int(lb.argmax())
    assert sb.rounds(lb[deep]).item() >= 3
    sel = _tile_pixels(S, [deep, (45 // 16) * nt + 82 // 16])   # and the tile of pixel (45, 82), in the front face
    g = torch.Generator(device=DEV).manual_seed(37)
    g_a_p = torch.randn(1, sel.numel(), device=DEV, generator=g, dtype=torch.float64)
    g_rgb_p = torch.randn(1, 3, sel.numel(), device=DEV, generator=g, dtype=torch.float64)
    g_a = torch.zeros(1, S * S, device=DEV)
    g_a[0, sel.reshape(-1)] = g_a_p[0].float()
    g_rgb = torch.zeros(1, 3, S * S, device=DEV)
    g_rgb[0][:, sel.reshape(-1)] = g_rgb_p[0].float()
    got = kernel_grads(sc, S, sigma, gamma, g_rgb.reshape(1, 3, S, S), g_a.reshape(1, S, S))
    ref = oracle_grads(sc, S, sigma, gamma, sel.reshape(1, -1), g_rgb_p, g_a_p)
    check_grads(got, ref, names_of(sc), ("deep", kind, gamma))
    # alpha bit-identical and rgb within fp32 rounding under a permutation of the faces
    perm = torch.from_numpy(np.random.default_rng(38).permutation(F)).to(DEV)
    ps = Scene(sc.kind, faces[:, perm].contiguous(), tri=sc.tri, bg=sc.bg,
               tex=None if sc.tex is None else (sc.tex[:, perm].contiguous() if sc.kind == "cube" else sc.tex),
               uvs=None if sc.uvs is None else sc.uvs[:, perm].contiguous(),
               light=None if sc.light is None else sc.light[:, perm].contiguous())
    rgb_p, alpha_p = ps.render(S, sigma, gamma)
    assert torch.equal(alpha_p, alpha)
    if rgb is not None:
        assert (rgb_p - rgb).abs().max().item() <= 2e-5


# ------------------------------------------------------------------------------------------------ c. cubes past the warp budget
@pytest.mark.parametrize("ts", [5, 6, 8])
@pytest.mark.parametrize("shared", [False, True])
def test_cube_gradient_past_the_warp_budget(ts, shared):
    from neural_renderer_b200 import _lib, synthetic
    nr = _nr()
    assert (ts * ts * ts * 3 > 384) == (ts >= 6)         # 384 floats: the per-warp shared-memory cube
    S, sigma, gamma, B, F = 64, 1e-3, 1e-2, 2, 14
    faces = torch.from_numpy(synthetic.triangle_soup(B, F, seed=40 + ts, size=(0.2, 0.6), offscreen=False,
                                                     duplicates=False)).to(DEV)
    tex = _rand((1 if shared else B, F, ts, ts, ts, 3), 41)
    fl = _rand((B, F, 3), 42, 0.5, 1.5)
    sc = Scene("cube", faces, tex=tex, light=fl)
    gen = torch.Generator(device=DEV).manual_seed(43)
    g_rgb = torch.randn(B, 3, S, S, device=DEV, generator=gen)
    g_a = torch.randn(B, S, S, device=DEV, generator=gen)
    got = kernel_grads(sc, S, sigma, gamma, g_rgb, g_a)
    pix = torch.arange(S * S, device=DEV)[None].expand(B, -1)
    ref = oracle_grads(sc, S, sigma, gamma, pix, g_rgb.reshape(B, 3, -1), g_a.reshape(B, -1))
    check_grads(got, ref, names_of(sc), ("cube", ts, shared))
    gt = got[1]
    assert (gt == 0).any() and (gt != 0).any()
    # NR_GRAD_ACCUMULATE over a seeded prefill; texels no pixel samples come back as the prefill, bit for bit
    a = _lib.SoftRgbArgs()
    a.struct_size = ctypes.sizeof(_lib.SoftRgbArgs)
    a.flags = _lib.NR_GRAD_ACCUMULATE | (_lib.NR_TEX_SHARED if shared else 0)
    a.faces, a.num_faces, a.batch_size, a.image_size, a.texture_size = faces.data_ptr(), F, B, S, ts
    a.sigma, a.gamma, a.near_, a.far_, a.eps = sigma, gamma, NEAR, FAR, 1e-4
    a.background[:] = sc.bg
    a.textures, a.face_light = tex.data_ptr(), fl.data_ptr()
    rgb, alpha = nr.rasterize_soft(faces, tex, S, sigma, gamma, background_color=sc.bg, face_light=fl)
    state = _state(faces, tex, fl, S, sigma, gamma, sc.bg)[2]
    a.rgb, a.alpha, a.state = rgb.data_ptr(), alpha.data_ptr(), state.data_ptr()
    a.grad_rgb, a.grad_alpha = g_rgb.data_ptr(), g_a.data_ptr()
    pre = [_rand(t.shape, 44 + i, -1.0, 1.0) for i, t in enumerate((faces, tex, fl))]
    outs = [p.clone() for p in pre]
    a.grad_faces, a.grad_textures, a.grad_face_light = (o.data_ptr() for o in outs)
    lib = _lib.load()
    n = lib.nr_b200_soft_rgb_workspace_bytes(B, F, S, a.flags)
    ws = torch.empty(n, dtype=torch.uint8, device=DEV)
    a.workspace, a.workspace_bytes = ws.data_ptr(), n
    stream = ctypes.c_void_p(torch.cuda.current_stream(DEV).cuda_stream)
    assert lib.nr_b200_soft_rgb_backward(ctypes.byref(a), stream) == 0
    torch.cuda.synchronize()
    for o, p, gk in zip(outs, pre, got):
        assert torch.equal(o[gk == 0], p[gk == 0])
        assert rel_err((o - p).cpu().numpy(), gk.cpu().numpy()) <= 1e-5
    # grad_textures NULL with grad_face_light wanted
    a.flags &= ~_lib.NR_GRAD_ACCUMULATE
    a.grad_textures = None
    gl = torch.full_like(fl, float("nan"))
    a.grad_face_light = gl.data_ptr()
    assert lib.nr_b200_soft_rgb_backward(ctypes.byref(a), stream) == 0
    torch.cuda.synchronize()
    assert rel_err(gl.cpu().numpy(), got[2].cpu().numpy()) <= 1e-5


# ------------------------------------------------------------------------------------------------ d. the benchmark geometry
S_BENCH, B_BENCH, F_BENCH = 256, 64, 5000


def _bench_scene(kind):
    from neural_renderer_b200 import synthetic
    faces = torch.from_numpy(synthetic.sphere_faces(B_BENCH, F_BENCH)).to(DEV)
    light = _rand((B_BENCH, F_BENCH, 3), 51, 0.5, 1.5)
    if kind == "sil":
        return Scene("sil", faces)
    if kind == "cube":
        return Scene("cube", faces, tex=torch.from_numpy(synthetic.random_textures(B_BENCH, F_BENCH, 4)).to(DEV), light=light)
    # a smooth image: the gradients of a bilinear tap jump where fp32 moves it across a texel's cell, by the image's
    # second difference, which noise would make O(1)
    img = _image(1, 1024, 1024, 53)
    # sphere_uvs puts the seam and the poles at u = 1 and v = 0 / 1 exactly, where the sampler's slope drops to 0 and the
    # fp32 rounding of the interpolated UV decides the face_uvs gradient: inset the mapping by 2 %
    uvs = (0.02 + 0.96 * torch.from_numpy(synthetic.sphere_uvs(F_BENCH)).to(DEV))[None].contiguous()
    return Scene("uv", faces, tex=img, uvs=uvs, light=light, tri=kind == "uv_tri")


def _bench_tiles(faces, S, sigma, seed):
    """[B,3] tiles per item: the densest by the CPU lower bound, one on the image border, one chosen by seed"""
    lb = sb.tile_entries_lower_bound(faces, S, sigma)
    nt = sb.tiles_per_axis(S)
    g = torch.Generator(device=DEV).manual_seed(seed)
    B = faces.shape[0]
    border = torch.tensor([t for t in range(nt * nt) if t // nt in (0, nt - 1) or t % nt in (0, nt - 1)], device=DEV)
    # the border tile nearest to the sphere's outline: the border tile with the most entries
    bt = border[lb[:, border].argmax(1)]
    rt = torch.randint(0, nt * nt, (B,), device=DEV, generator=g)
    return torch.stack((lb.argmax(1), bt, rt), 1), lb


@pytest.mark.parametrize("sigma", [1e-5, 1e-4, 1e-3])
@pytest.mark.parametrize("kind", ["cube", "uv_bil", "uv_tri", "sil"])
def test_benchmark_geometry_against_the_sparse_oracle(kind, sigma):
    S, gamma, B = S_BENCH, 1e-4, B_BENCH
    sc = _bench_scene(kind)
    assert sc.faces.shape == (64, 5000, 3, 3)
    tiles, lb = _bench_tiles(sc.faces, S, sigma, seed=int(-math.log10(sigma)))
    pix = torch.stack([_tile_pixels(S, tiles[b]).reshape(-1) for b in range(B)])        # [B,768]
    rgb, alpha = sc.render(S, sigma, gamma)
    worst = check_forward(sc, rgb, alpha, S, sigma, gamma, pix, ("bench", kind, sigma))
    print("bench", kind, sigma, worst, "max entries", lb.max().item())
    # backward: the upstream gradient only on the chosen tiles
    g = torch.Generator(device=DEV).manual_seed(52)
    g_a_p = torch.randn(B, pix.shape[1], device=DEV, generator=g, dtype=torch.float64)
    g_rgb_p = torch.randn(B, 3, pix.shape[1], device=DEV, generator=g, dtype=torch.float64)
    g_a = torch.zeros(B, S * S, device=DEV).scatter_(1, pix, g_a_p.float())
    g_rgb = torch.zeros(B, 3, S * S, device=DEV).scatter_(2, pix[:, None].expand(-1, 3, -1), g_rgb_p.float())
    got = kernel_grads(sc, S, sigma, gamma, g_rgb.reshape(B, 3, S, S), g_a.reshape(B, S, S))
    ref = oracle_grads(sc, S, sigma, gamma, pix, g_rgb_p, g_a_p)
    check_grads(got, ref, names_of(sc), ("bench", kind, sigma))
    # faces out of reach of every chosen pixel (with room for the fp32 cut-off test) get exactly nothing
    keep = osoft.in_reach(sc.faces, osoft.pixel_set(S, pix, B, DEV), sigma, NEAR, FAR, 1.001)
    assert torch.all(got[0][~keep] == 0)
    if kind == "cube":
        assert torch.all(got[1][~keep] == 0) and torch.all(got[2][~keep] == 0)
    assert keep.sum().item() < keep.numel() // 2 and got[0].abs().max() > 0


# ------------------------------------------------------------------------------------------------ e. slivers
@pytest.mark.parametrize("kind", ["cube", "uv_bil", "uv_tri"])
def test_slivers_stay_finite_and_inside_the_colour_hull(kind):
    """Needles (synthetic.needle_faces) through the soft RGB and UV paths: no oracle comparison, since the fp32
    barycentrics of a face of doubled area |A| carry about 1e-7 / |A|, which a sliver makes arbitrarily large.  What
    must hold: rgb is finite and inside the per-channel hull of what it blends (the background and every face's
    colours times its light), and every gradient is finite."""
    from neural_renderer_b200 import synthetic
    S, sigma, gamma, B, F = 64, 1e-4, 1e-3, 2, 40
    faces = torch.from_numpy(synthetic.needle_faces(B, F, S, seed=61)).to(DEV)
    light = _rand((B, F, 3), 62, 0.5, 1.5)
    if kind == "cube":
        sc = Scene("cube", faces, tex=_rand((B, F, 3, 3, 3, 3), 63), light=light)
        cols = sc.tex.reshape(B, F, -1, 3)
        lo, hi = (cols.amin(2) * light).amin(1), (cols.amax(2) * light).amax(1)          # [B,3]
    else:
        sc = Scene("uv", faces, tex=_image(1, 32, 32, 64), uvs=_rand((B, F, 3, 2), 65), light=light, tri=kind == "uv_tri")
        img = sc.tex.reshape(1, -1, 3)
        lo = (img.amin(1)[:, None] * light).amin(1)
        hi = (img.amax(1)[:, None] * light).amax(1)
    bg = torch.tensor(sc.bg, device=DEV)
    lo, hi = torch.minimum(lo, bg), torch.maximum(hi, bg)
    rgb, alpha = sc.render(S, sigma, gamma)
    assert torch.isfinite(rgb).all() and torch.isfinite(alpha).all()
    slack = 1e-6
    assert torch.all(rgb >= lo[:, :, None, None] - slack) and torch.all(rgb <= hi[:, :, None, None] + slack)
    gen = torch.Generator(device=DEV).manual_seed(66)
    got = kernel_grads(sc, S, sigma, gamma, torch.randn(B, 3, S, S, device=DEV, generator=gen),
                       torch.randn(B, S, S, device=DEV, generator=gen))
    for name, gk in zip(names_of(sc), got):
        assert torch.isfinite(gk).all(), name
    assert got[0].abs().max() > 0


def test_peak_device_memory():
    """the file's peak device memory, the oracles included, stays under 8 GB (runs last in the file)"""
    print("peak device memory", torch.cuda.max_memory_allocated(DEV))
    assert torch.cuda.max_memory_allocated(DEV) < 8 * 1024 ** 3, torch.cuda.max_memory_allocated(DEV)
