"""The float64 soft oracles restricted to a given selection, and the float64 bands where an fp32 kernel and a float64
oracle may still disagree about a gradient once they agree on the selection.

The soft kernels drop an outside face at the cut-off (d^2 > cut), decided in fp32; the float64 oracles decide it in
float64, so at pixels within the fp32 error of the cut-off the two aggregate different sets and their gradients differ by
a whole term.  rasterize_soft_fragments makes that decision with the same device test on the same face records (soft_eval
on k_soft_setup's records, with the same cut), and writes the set: at K = 32, every pixel with fewer than 32 fragments
holds exactly the set every soft kernel aggregates there (in a scene without zero-area faces or faces of non-finite
depth, which the fragments alone leave out).  restrict(terms, pix_to_face, pix) turns any terms(b0, b1, idx, fc, p) of
oracles_soft.sparse_eval into the same terms at that set: `on` and every boolean mask after it are ANDed with membership
of (item, face, pixel) in pix_to_face (-1 = an empty slot).  Build the terms with cut_scale WIDE and cull with WIDE, so
that every pair the kernel selected is evaluated (its float64 d^2 may lie just past the cut) and membership alone decides.

bands(...) gives, per selected pair, the remaining fp32 / float64 disagreements of a gradient (DESIGN.md 8 excludes
gradients through them): the clamp of the barycentrics at lam = 0 or 1, a tie of the nearest edge between two edges whose
nearest points differ, and the texel cell or the clamp of the sampled coordinate (the cube's t_k against its cell
boundaries and tex_cmp, the image's u (W - 1) and v (H - 1) against theirs, at both levels of a trilinear tap).  Each band
is the fp32 error bound of the quantity from oracles_soft_frag's derivation, without its SAFETY factor (the bounds
already count several ulps per operation; a band too narrow would show as a failing gradient, one too wide masks
pixels for nothing):
  lam, l:  dl = 8 eps |e| (|e| + d) / |A|                       the edge functions over the area
  d^2_k:   dists_gate(delta, d^2_k) per edge                     a tie when d^2_(1) - d^2_(0) <= the sum of both
  l'_k:    g_l = dl zp / min z + max_k |l'_k| (dzp / zp + 4 eps) + 4 eps
  t_k:     (ts - 1) g_l          u, v:  g_l sum_k |uv_k| + 4 eps, times (W - 1) or (H - 1) of the level."""
import torch

import oracles_soft as osoft
import oracles_soft_attr as oattr
import oracles_soft_frag as ofrag
import oracles_soft_rgb as orgb
import oracles_soft_uv as ouv

WIDE = 1.5     # the cut-off scale of the cull and of the terms under a selection: wider than any fp32 cut-off band
CUBE_EPS = 1e-4


class AttrScene:
    """a soft attribute render in the shape of test_gpu_soft_scale.Scene (what its check_forward and the oracles read):
    faces [B,F,3,3], per-corner attributes ca [1|B,F,3,C], background bg (C numbers), near and far; the colour
    sensitivity of the forward gates is 3 max |a| per face"""
    kind = "attr"

    def __init__(self, faces, ca, bg, near, far):
        self.faces, self.tex, self.bg, self.near, self.far = faces, ca, tuple(bg), near, far

    def leaves(self):
        return [self.faces, self.tex]

    def oracle_terms(self, leaves, S, sigma, cut_scale=1.0):
        ca = leaves[1].double()

        def terms(b0, b1, idx, fc, p):
            return oattr.attr_terms(fc, osoft.take(ca, b0, b1, idx), p, sigma, self.near, self.far, cut_scale)
        return terms

    def colour_sensitivity(self):
        return 3 * self.tex.double().abs().amax((-1, -2))


def flat_selection(pix_to_face):
    """pix_to_face [B,H,W,K] (or [B,S*S,K]) as [B,S*S,K] int64"""
    B, K = pix_to_face.shape[0], pix_to_face.shape[-1]
    return pix_to_face.reshape(B, -1, K).long()


def under_full(pix_to_face):
    """[B,H,W] bool: the pixels with fewer than K fragments, where the fragments are every face the soft kernels
    aggregate (at a full pixel they are only its K nearest)"""
    return (pix_to_face >= 0).sum(-1) < pix_to_face.shape[-1]


def restrict(terms, pix_to_face, pix):
    """terms of sparse_eval at the pixels pix ([P] or [B,P] flat indices, as given to sparse_eval) restricted to the
    selection pix_to_face ([B,H,W,K] / [B,S*S,K], face indices within the item, -1 empty)"""
    p2f = flat_selection(pix_to_face)
    B, K = p2f.shape[0], p2f.shape[-1]
    pix = torch.as_tensor(pix, device=p2f.device).long()
    if pix.dim() == 1:
        pix = pix[None].expand(B, -1)
    sel = torch.gather(p2f, 1, pix[..., None].expand(-1, -1, K))                 # [B,P,K]

    def rt(b0, b1, idx, fc, p):
        out = terms(b0, b1, idx, fc, p)
        m = (idx[:, :, None, None] == sel[b0:b1, None]).any(-1)                 # [Bc,Fc,P]
        return (out[0],) + tuple(o & m if o.dtype == torch.bool else o for o in out[1:])
    return rt


def pairs(pix_to_face):
    """(b, pixel, f) [N] of the selected pairs"""
    p2f = flat_selection(pix_to_face)
    b, pi, k = (p2f >= 0).nonzero(as_tuple=True)
    return b, pi, p2f[b, pi, k]


def pair_geometry(faces, b, pix, f, S):
    """float64 terms of the pairs (item b, pixel pix, face f) [N] of faces [B,F,3,3]: a dict of lam [N,3] (lam_k =
    c_{k+1} / A), l, lp (l'_k), zp, d2k (d^2 to each edge [N,3]), near (the nearest point of each edge [N,3,2]), and
    the fp32 error terms delta, dl, dzp, g_l of the module docstring"""
    with torch.no_grad():
        fc = faces.detach().to(torch.float64)[b, f]                              # [N,3,3]
        p = osoft.pixel_centres(S, device=fc.device)[pix]                        # [N,2]
        a = fc[..., :2]
        e = a.roll(-1, dims=1) - a
        dp = p[:, None] - a
        l2 = (e * e).sum(-1)
        t = ((dp * e).sum(-1) / torch.where(l2 > 0, l2, torch.ones_like(l2))).clamp(0.0, 1.0)
        near = a + t[..., None] * e
        q = p[:, None] - near
        d2k = (q * q).sum(-1)
        c = e[..., 0] * dp[..., 1] - e[..., 1] * dp[..., 0]
        A = orgb.doubled_area(fc[None])[0]
        lam = c.roll(-1, dims=1) / A[:, None]
        lh = lam.clamp(0.0, 1.0)
        l = lh / lh.sum(-1, keepdim=True)
        z = fc[..., 2]
        zp = 1.0 / (l / z).sum(-1)
        lp = l * zp[:, None] / z
        d2 = d2k.amin(-1)
        delta, dl, dzp = ofrag._error_terms(fc[None], d2[None, :, None], zp[None, :, None])
        delta, dl, dzp = delta[0, :, 0], dl[0, :, 0], dzp[0, :, 0]
        zmin = z.amin(-1).abs()
        g_l = dl * zp / zmin + lp.abs().amax(-1) * (dzp / zp + 4 * ofrag.EPS32) + 4 * ofrag.EPS32
        return dict(fc=fc, lam=lam, l=l, lp=lp, zp=zp, d2k=d2k, near=near, delta=delta, dl=dl, dzp=dzp, g_l=g_l)


def lam_band(g):
    """[N]: a barycentric within its error of the clamp at 0 or 1"""
    dl = g["dl"][:, None]
    return (((g["lam"].abs() <= dl) | ((g["lam"] - 1).abs() <= dl)).any(-1))


def tie_band(g):
    """[N]: the two nearest edges within the fp32 error of d^2 of each other, with nearest points apart (when both
    nearest points are their shared vertex the distance is one function and no gradient jumps)"""
    d2k, near, delta = g["d2k"], g["near"], g["delta"]
    s, o = d2k.sort(-1)
    n0 = torch.gather(near, 1, o[:, :1, None].expand(-1, -1, 2))[:, 0]
    n1 = torch.gather(near, 1, o[:, 1:2, None].expand(-1, -1, 2))[:, 0]
    gap = ofrag.dists_gate(delta, s[:, 0]) + ofrag.dists_gate(delta, s[:, 1])
    # near a vertex region's border the two are tangent: d^2_(1) - d^2_(0) = |n0 - n1|^2 (Pythagoras), and the
    # gradients differ by O(|n0 - n1| / |e|); a tie that moves a gradient is transversal, with |n0 - n1|^2 > the gap
    apart = ((n0 - n1) ** 2).sum(-1) > gap
    return (s[:, 1] - s[:, 0] <= gap) & apart


def cell_band(x, n, err):
    """x within err of an inner cell boundary of a sampler over n texels (1 .. n - 2; the clamps are the caller's)"""
    r = x.round()
    return ((x - r).abs() <= err) & (r >= 1) & (r <= n - 2)


def cube_band(g, ts):
    """[N]: some t_k = l'_k (ts - 1) within its error of a cell boundary of the cube or of tex_cmp (ts - 1 - eps)"""
    t = g["lp"] * (ts - 1)
    err = ((ts - 1) * g["g_l"])[:, None]
    inner = cell_band(t, ts, err)
    # t_k reaches ts - 1 only where l'_k = 1: in a vertex region, where every barycentric is clamped and t_k is
    # constant, so the clamp changes no gradient; elsewhere near the vertex it does
    top = ((t - (ts - 1 - CUBE_EPS)).abs() <= err) & ((g["l"] > 0).sum(-1, keepdim=True) > 1)
    return (inner | top).any(-1)


def uv_band(g, uvk, Ht, Wt, trilinear, S):
    """[N]: the sampled u (W - 1) or v (H - 1) within its error of a cell boundary or of the clamps, at the level
    (bilinear) or both levels of the tap (trilinear, the level of detail as oracles_soft_uv.lod); uvk [N,3,2]"""
    lp = g["lp"]
    u = (lp * uvk[..., 0]).sum(-1)
    v = (lp * uvk[..., 1]).sum(-1)
    eu = g["g_l"] * uvk[..., 0].abs().sum(-1) + 4 * ofrag.EPS32
    ev = g["g_l"] * uvk[..., 1].abs().sum(-1) + 4 * ofrag.EPS32
    out = (u <= eu) | (u >= 1 - eu) | (v <= ev) | (v >= 1 - ev)   # the clamps (inset UVs keep clear of them)
    if not trilinear:
        return out | cell_band(u * (Wt - 1), Wt, eu * (Wt - 1)) | cell_band(v * (Ht - 1), Ht, ev * (Ht - 1))
    off, hs, ws = ouv.level_table(Ht, Wt, lp.device)
    L = off.numel()
    ld = ouv.lod(g["fc"][None], g["l"][None, :, :, None], g["zp"][None, :, None], uvk[None], S, Ht, Wt, L)[0, :, 0]
    l0 = ld.floor().long()
    for lv in (l0, (l0 + 1).clamp(max=L - 1)):
        w, h = ws[lv].double(), hs[lv].double()
        out = out | cell_band(u * (w - 1), w, eu * (w - 1)) | cell_band(v * (h - 1), h, ev * (h - 1))
    return out


def band_pixels(faces, pix_to_face, S, cube_ts=None, uv=None, lam=True):
    """[B,S*S] bool: the pixels where a selected pair lies in a band (module docstring).  faces [B,F,3,3]; cube_ts: the
    cube's texels per axis (cube path); uv = (face_uvs [1|B,F,3,2], Ht, Wt, trilinear) (UV path); lam: whether the
    barycentrics' clamp matters (not for the silhouettes, whose terms use d^2 alone)"""
    B = faces.shape[0]
    b, pix, f = pairs(pix_to_face)
    g = pair_geometry(faces, b, pix, f, S)
    m = tie_band(g)
    if lam:
        m = m | lam_band(g)
    if cube_ts is not None:
        m = m | cube_band(g, cube_ts)
    if uv is not None:
        uvs, Ht, Wt, tri = uv
        uvs = uvs.detach().to(torch.float64)
        uvk = uvs[b if uvs.shape[0] > 1 else torch.zeros_like(b), f]
        m = m | uv_band(g, uvk, Ht, Wt, tri, S)
    out = torch.zeros(B, S * S, dtype=torch.bool, device=faces.device)
    out[b[m], pix[m]] = True
    return out



# ------------------------------------------------------------------------------------------------ a cut-off scene
def cutoff_edges(S, sigma, steps=40):
    """[(row, ay, kernel_on)]: horizontal edges y = ay (fp32) whose distance to the pixel centres of raster row `row` is
    decided differently at the cut-off by the kernels' fp32 test and by the float64 oracle.  For a horizontal edge
    soft_eval's d^2 is fl32(dy^2) with dy = fl32(py - ay) (qy = dy exactly, e.w = 0; qx^2 <= 1e-14 is far below half an
    ulp of d^2 near the cut), against cut = fl32(sigma ln((1 - 1e-4) / 1e-4)); the oracle tests (py - ay)^2 <= cut in
    float64.  Searched over `steps` fp32 values of ay either side of py +- sqrt(cut), every row."""
    import math

    import numpy as np
    cut64 = sigma * math.log((1.0 - osoft.EPS) / osoft.EPS)
    cut32 = np.float32(cut64)
    r = math.sqrt(cut64)
    out = []
    for row in range(S):
        py = np.float32((2 * row + 1 - S) / S)
        for sgn in (1.0, -1.0):
            a = np.float32(py + sgn * r)
            for _ in range(steps):
                a = np.nextafter(a, np.float32(-np.inf))
            for _ in range(2 * steps):
                dy = np.float32(np.float64(py) - np.float64(a))
                k = bool(np.float32(np.float64(dy) * np.float64(dy)) <= cut32)
                f = bool((np.float64(py) - np.float64(a)) ** 2 <= cut64)
                if k != f:
                    out.append((row, float(a), k))
                a = np.nextafter(a, np.float32(np.inf))
    return out


def cutoff_faces(S, sigma, z_range, seed=0, width=0.25, height=0.15):
    """[1,F,3,3] float32: one face per edge of cutoff_edges, its bottom (or top) edge that edge over `width` of the
    image, the face on the far side of the edge from the row, corner depths in z_range"""
    import numpy as np
    rng = np.random.default_rng(seed)
    faces = []
    for i, (row, ay, _) in enumerate(cutoff_edges(S, sigma)):
        py = (2 * row + 1 - S) / S
        x0 = -0.9 + (i * 0.37) % (1.8 - width)
        apex = ay + (height if ay > py else -height)
        z = rng.uniform(*z_range, 3)
        faces.append([[x0, ay, z[0]], [x0 + width, ay, z[1]], [x0 + width / 2, apex, z[2]]])
    return torch.tensor(faces, dtype=torch.float32)[None]


def cutoff_disagreements(faces, pix_to_face, S, sigma):
    """the selected pairs outside their face and past the cut-off in float64: the pairs the fp32 test kept and the
    oracle alone would drop"""
    b, pix, f = pairs(pix_to_face)
    g = pair_geometry(faces, b, pix, f, S)
    inside = ((g["lam"] > 0) & (g["lam"] < 1)).all(-1)
    return int((~inside & (g["d2k"].amin(-1) > osoft.cut(sigma))).sum())
