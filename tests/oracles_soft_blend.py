"""Float64 oracle of the soft blend of fragments (include/nr_b200.h, nr_b200_blend_args), differentiable in zbuf, dists
and colors.

blend(...) evaluates the definition: over the valid slots (pix_to_face >= 0), x_k = dists_k / sigma, D_k = sigmoid(x_k),
zb = far - 1e-3 (far - near), zref = min(zb, min_k zbuf_k) (held fixed: it cancels), w_k = D_k exp(e_k) with
e_k = (zref - zbuf_k) / ((far - near) gamma), w_b = exp(e_b), e_b = (zref - zb) / ((far - near) gamma), Z = w_b + sum w_k,
out_c = (w_b bg_c + sum_k w_k c_kc) / Z and alpha = -expm1(-sum_k softplus(x_k)).  Invalid slots are replaced by
harmless values before any arithmetic, so whatever they hold (NaN included) reaches neither a value nor a gradient.

gates(...) derives the fp32 error of the kernel per output element, with eps = 2^-23 (the error analysis of DESIGN.md 4t):
  x_k:  fl(dists fl(1/sigma)) has relative error <= 2 eps, so |dx_k| <= 2 eps |x_k|; D_k then moves by at most
        D_k (1 - D_k) |dx_k|, a relative 2 eps |x_k| (1 - D_k).
  e_k:  the difference zref - zbuf_k, the product with the fp32 1 / ((far - near) gamma) and that constant's own rounding
        give 3 eps |e_k|; expf adds 2 eps and the product with D_k 1 eps.  So w_k carries a relative
        delta_k = 3 eps |e_k| + 2 eps |x_k| (1 - D_k) + 4 eps.  |e_k| is unbounded in the arithmetic but w_k = 0 once
        e_k < -104 (fp32 underflow), so the term only matters up to there: w_k |e_k| <= w_max / e.
  out:  d out_c / d w_k = (c_kc - out_c) / Z, so the weights move out_c by sum_k w_k delta_k |c_kc - out_c| / Z (w_b
        likewise, with delta_b = 3 eps |e_b| + 3 eps); the K + 1 term sums of Z and of the numerator add
        (K + 2) eps (w_b |bg_c| + sum_k w_k |c_kc|) / Z + (K + 2) eps |out_c|, the division eps |out_c|.
  alpha: softplus_k moves by D_k |dx_k| + 4 eps softplus_k, the sum by K eps sum softplus more, and alpha by
        (1 - alpha) times that.
Each gate is SAFETY = 4 times its bound, plus 4 eps |value| + 1e-30 for the outputs' own rounding, as
oracles_soft_frag.py scales its gates."""
import torch

EPS32 = 2.0 ** -23
SAFETY = 4.0
BG_DEPTH = 1e-3  # NR_SOFT_BG_DEPTH


def _terms(p2f, zbuf, dists, colors, sigma, gamma, near, far):
    valid = p2f >= 0
    z = zbuf.to(torch.float64)
    d = dists.to(torch.float64)
    c = colors.to(torch.float64)
    fn = float(far) - float(near)
    zb = float(far) - BG_DEPTH * fn
    inf = torch.full_like(z, float("inf"))
    zref = torch.where(valid, z.detach(), inf).amin(-1).clamp_max(zb)           # [B,H,W]
    zs = torch.where(valid, z, zref[..., None])
    ds = torch.where(valid, d, torch.zeros_like(d))
    cs = torch.where(valid[..., None], c, torch.zeros_like(c))
    x = ds / float(sigma)
    D = torch.where(valid, torch.sigmoid(x), torch.zeros_like(x))
    e = (zref[..., None] - zs) / (fn * float(gamma))
    w = torch.where(valid, D * torch.exp(e), torch.zeros_like(x))
    eb = (zref - zb) / (fn * float(gamma))
    wb = torch.exp(eb)
    sp = torch.where(valid, torch.logaddexp(torch.zeros_like(x), x), torch.zeros_like(x))
    return valid, cs, x, D, e, w, eb, wb, sp


def blend(p2f, zbuf, dists, colors, sigma, gamma, near=0.1, far=100.0, background=None):
    """(out [B,C,H,W], alpha [B,H,W]) in float64; p2f [B,H,W,K], zbuf / dists [B,H,W,K], colors [B,H,W,K,C]"""
    valid, cs, x, D, e, w, eb, wb, sp = _terms(p2f, zbuf, dists, colors, sigma, gamma, near, far)
    C = colors.shape[-1]
    bg = torch.zeros(C, dtype=torch.float64, device=colors.device) if background is None else \
        torch.as_tensor(background, dtype=torch.float64).to(colors.device)
    Z = w.sum(-1) + wb
    out = ((w[..., None] * cs).sum(-2) + wb[..., None] * bg) / Z[..., None]
    alpha = -torch.expm1(-sp.sum(-1))
    return out.permute(0, 3, 1, 2), alpha


def gates(p2f, zbuf, dists, colors, sigma, gamma, near=0.1, far=100.0, background=None):
    """the derived gates (out [B,C,H,W], alpha [B,H,W]) of the module docstring"""
    with torch.no_grad():
        valid, cs, x, D, e, w, eb, wb, sp = _terms(p2f, zbuf, dists, colors, sigma, gamma, near, far)
        K, C = colors.shape[-2], colors.shape[-1]
        bg = torch.zeros(C, dtype=torch.float64, device=colors.device) if background is None else \
            torch.as_tensor(background, dtype=torch.float64).to(colors.device)
        Z = w.sum(-1) + wb
        out = ((w[..., None] * cs).sum(-2) + wb[..., None] * bg) / Z[..., None]          # [B,H,W,C]
        delta = 3 * EPS32 * e.abs() + 2 * EPS32 * x.abs() * (1 - D) + 4 * EPS32
        delta = torch.where(valid, delta, torch.zeros_like(delta))
        dw = (w * delta)[..., None] * (cs - out[..., None, :]).abs()
        dw = torch.where(valid[..., None], dw, torch.zeros_like(dw)).sum(-2)
        db = (wb * (3 * EPS32 * eb.abs() + 3 * EPS32))[..., None] * (bg - out).abs()
        sums = (K + 2) * EPS32 * ((w[..., None] * cs.abs()).sum(-2) + wb[..., None] * bg.abs())
        g_out = (dw + db + sums) / Z[..., None] + (K + 3) * EPS32 * out.abs()
        g_out = SAFETY * g_out + 4 * EPS32 * out.abs() + 1e-30
        S = sp.sum(-1)
        alpha = -torch.expm1(-S)
        dS = (D * 2 * EPS32 * x.abs() + 4 * EPS32 * sp).sum(-1) + K * EPS32 * S
        g_alpha = SAFETY * (1 - alpha) * dS + 4 * EPS32 * alpha + 1e-30
        return g_out.permute(0, 3, 1, 2), g_alpha
