"""GPU: soft silhouettes (rasterize_soft_silhouettes, nr_b200_soft_silhouettes[_backward]) against the float64 oracle of
tests/oracles_soft.py, the direct C ABI (poisoned outputs, guard words, NULLs, accumulation, refusals), determinism, a
shape fit that the hard silhouette cannot do, and Renderer.render_soft_silhouettes.

Forward gate (DESIGN.md section 4o): the kernels evaluate d^2 in fp32 from fp32 coordinates of magnitude <= ~1.5, so
|p - q| carries an absolute error of a few fp32 ulps of 1 (delta ~ 5e-7 NDC); x = d^2 / sigma then errs by 2 d delta /
sigma, and D = sigmoid(x) by sigmoid'(x) 2 d delta / sigma <= 0.4 delta / sqrt(sigma).  A pixel within reach of n faces
errs by at most n times that; the gate allows n = 5:  tol(sigma) = 1e-6 / sqrt(sigma) + 1e-6  (3.2e-4 at sigma 1e-5,
3.3e-5 at 1e-3).  The cut-off is a hard threshold on the fp32 d^2, so the oracle is evaluated with the cut-off moved by
+-1e-5 relative and the kernel's alpha must lie between the two (widened by tol)."""
import ctypes
import math
import os

import numpy as np
import pytest
import torch

import oracles_soft as osoft
from helpers import elem_err, rel_err

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
SIGMAS = (1e-5, 1e-4, 1e-3)


def tol(sigma):
    return 1e-6 / math.sqrt(sigma) + 1e-6


def _nr():
    import neural_renderer_b200 as nr
    return nr


def _soup(B, F, seed, **kw):
    from neural_renderer_b200 import synthetic
    return torch.from_numpy(synthetic.triangle_soup(B, F, seed=seed, **kw)).to(DEV)


def _check_forward(alpha, faces64, S, sigma, near=0.1, far=100.0):
    lo = osoft.soft_silhouettes(faces64, S, sigma, near, far, cut_scale=1 - 1e-5)
    hi = osoft.soft_silhouettes(faces64, S, sigma, near, far, cut_scale=1 + 1e-5)
    a = alpha.double()
    err = torch.maximum(torch.minimum(lo, hi) - a, a - torch.maximum(lo, hi)).clamp_min(0).max().item()
    assert err <= tol(sigma), (err, tol(sigma))
    return err


def _special_faces(B, S, sigma, seed):
    """a soup plus the special cases: faces wider than the wide-list cap, faces wholly outside the image but within
    reach, faces straddling near / far, zero-area faces (collinear and a single point)"""
    soup = _soup(B, 24, seed, size=(0.02, 0.3))
    reach = math.sqrt(osoft.cut(sigma))  # NDC
    extra = []
    extra.append([[-1.1, -1.0, 1.5], [1.2, -0.9, 1.5], [0.1, 1.3, 1.5]])           # covers the image: > 16 tiles
    extra.append([[-0.9, 0.95, 2.0], [0.9, 0.9, 2.0], [0.0, 0.97, 2.0]])            # a wide sliver
    o = 1.0 + 0.5 * reach
    extra.append([[o, -0.3, 1.2], [o + 0.2, 0.0, 1.2], [o, 0.3, 1.2]])              # right of the image, within reach
    extra.append([[-0.3, -o, 1.2], [0.3, -o, 1.2], [0.0, -o - 0.2, 1.2]])           # below the image, within reach
    extra.append([[-0.5, 0.1, 0.05], [-0.2, 0.1, 1.0], [-0.4, 0.4, 1.0]])           # one vertex nearer than near
    extra.append([[0.2, -0.5, 1.0], [0.5, -0.5, 150.0], [0.3, -0.2, 1.0]])          # one vertex beyond far
    extra.append([[0.1, 0.5, 0.1], [0.3, 0.5, 100.0], [0.2, 0.7, 1.0]])             # depths exactly near and far
    extra.append([[-0.6, -0.6, 1.0], [-0.2, -0.2, 1.0], [-0.4, -0.4, 1.0]])         # collinear: zero area
    extra.append([[0.6, 0.2, 1.0], [0.6, 0.2, 1.0], [0.6, 0.2, 1.0]])               # a point
    ex = torch.tensor(extra, dtype=torch.float32, device=DEV)[None].expand(B, -1, -1, -1)
    return torch.cat((soup, ex), 1).contiguous()


@pytest.mark.parametrize("S", [64, 127, 256, 257])
@pytest.mark.parametrize("sigma", SIGMAS)
def test_forward_vs_oracle_soups_and_special_faces(S, sigma):
    nr = _nr()
    faces = _special_faces(2, S, sigma, seed=S + int(-math.log10(sigma)))
    alpha = nr.rasterize_soft_silhouettes(faces, S, sigma)
    assert alpha.shape == (2, S, S) and alpha.dtype == torch.float32
    _check_forward(alpha, faces.double(), S, sigma)
    # the largest sigma reaches farther than a 16-pixel tile at 256
    if sigma == 1e-3 and S >= 256:
        assert math.sqrt(osoft.cut(sigma)) * S / 2 > 16 * 0.7
    a2 = nr.rasterize_soft_silhouettes(faces, S, sigma)
    assert torch.equal(alpha, a2)  # bit-for-bit deterministic


def _teapot_faces(B=2):
    nr = _nr()
    d = np.load(os.path.join(os.path.dirname(__file__), "golden", "teapot.npz"))
    v = torch.from_numpy(d["vertices"].astype(np.float32)).to(DEV)
    f = torch.from_numpy(d["faces"].astype(np.int32)).to(DEV)
    r = nr.Renderer()
    r.eye = nr.get_points_from_angles(2.732, 30, -15)
    verts = r._transform(v[None].expand(B, -1, -1).contiguous())
    return verts.contiguous(), f


@pytest.mark.parametrize("sigma", SIGMAS)
def test_forward_vs_oracle_teapot_and_geometry_forms(sigma):
    nr = _nr()
    S = 256
    verts, idx = _teapot_faces(2)
    B, Nv = verts.shape[:2]
    # out-of-range indices gather the zero vertex
    idx_b = idx[None].repeat(B, 1, 1).clone()
    idx_b[0, 5, 1] = Nv
    idx_b[1, 7, 2] = -3
    faces = osoft.gather_faces(verts, idx_b).float().contiguous()
    a_mat = nr.rasterize_soft_silhouettes(faces, S, sigma)
    a_idx = nr.rasterize_soft_silhouettes(idx_b, S, sigma, vertices=verts)
    _check_forward(a_mat, faces.double(), S, sigma)
    assert torch.equal(a_mat, a_idx)
    # shared [F,3], [1,F,3] and an expanded [B,F,3] index set
    faces_s = osoft.gather_faces(verts, idx).float()
    ref = nr.rasterize_soft_silhouettes(faces_s, S, sigma)
    for ix in (idx, idx[None], idx[None].expand(B, -1, -1)):
        assert torch.equal(nr.rasterize_soft_silhouettes(ix, S, sigma, vertices=verts), ref)
    assert ref.max() > 0.99 and ref.min() == 0.0


# ------------------------------------------------------------------------------------------------ backward
def _oracle_grads(faces, S, sigma, g, near=0.1, far=100.0):
    f64 = faces.double().detach().requires_grad_(True)
    a = osoft.soft_silhouettes(f64, S, sigma, near, far)
    (gf,) = torch.autograd.grad((a * g.double()).sum(), f64)
    return gf


@pytest.mark.parametrize("sigma", SIGMAS[1:])
@pytest.mark.parametrize("S", [64, 127])
def test_backward_vs_float64_autograd(S, sigma):
    nr = _nr()
    faces = _special_faces(2, S, sigma, seed=11 + S)
    g = torch.randn(2, S, S, device=DEV, generator=torch.Generator(device=DEV).manual_seed(5))
    f = faces.clone().requires_grad_(True)
    (nr.rasterize_soft_silhouettes(f, S, sigma) * g).sum().backward()
    ref = _oracle_grads(faces, S, sigma, g)
    got = f.grad.double()
    assert torch.all(got[..., 2] == 0)
    assert rel_err(got.cpu().numpy(), ref.cpu().numpy()) <= 2e-3
    assert elem_err(got[..., :2].cpu().numpy(), ref[..., :2].cpu().numpy(), floor=1e-2) <= 2e-2
    # faces that take no part (a vertex outside [near, far]) get exactly nothing
    F0 = faces.shape[1] - 9
    assert torch.all(got[:, F0 + 4:F0 + 6] == 0)


def test_backward_indexed_shared_reduces_over_items_and_matches_materialised():
    nr = _nr()
    S, sigma = 64, 1e-4
    verts, idx = _teapot_faces(2)
    g = torch.randn(2, S, S, device=DEV, generator=torch.Generator(device=DEV).manual_seed(6))
    v = verts.clone().requires_grad_(True)
    (nr.rasterize_soft_silhouettes(idx, S, sigma, vertices=v) * g).sum().backward()
    v64 = verts.double().requires_grad_(True)
    a = osoft.soft_silhouettes(osoft.gather_faces(v64, idx), S, sigma)
    (ref,) = torch.autograd.grad((a * g.double()).sum(), v64)
    assert rel_err(v.grad.cpu().numpy(), ref.cpu().numpy()) <= 2e-3
    # one vertex set shared by both items (an expanded batch): its gradient is the sum over the items
    v1 = verts[:1].clone().requires_grad_(True)
    (nr.rasterize_soft_silhouettes(idx, S, sigma, vertices=v1.expand(2, -1, -1)) * g).sum().backward()
    v64s = verts[:1].double().requires_grad_(True)
    a = osoft.soft_silhouettes(osoft.gather_faces(v64s.expand(2, -1, -1), idx), S, sigma)
    (ref_s,) = torch.autograd.grad((a * g.double()).sum(), v64s)
    assert rel_err(v1.grad.cpu().numpy(), ref_s.cpu().numpy()) <= 2e-3


def test_backward_vs_central_differences_of_the_forward():
    nr = _nr()
    S, sigma = 64, 1e-3
    faces = _soup(1, 6, seed=21, size=(0.1, 0.4), offscreen=False)
    w = torch.randn(1, S, S, device=DEV, generator=torch.Generator(device=DEV).manual_seed(7))
    f = faces.clone().requires_grad_(True)
    (nr.rasterize_soft_silhouettes(f, S, sigma) * w).sum().backward()

    def loss(ff):
        return float((nr.rasterize_soft_silhouettes(ff, S, sigma).double() * w.double()).sum())

    h = 2e-4
    scale = f.grad.abs().max().item()
    for (fi, k, c) in [(0, 0, 0), (1, 1, 1), (2, 2, 0), (3, 0, 1), (5, 2, 1)]:
        fp, fm = faces.clone(), faces.clone()
        fp[0, fi, k, c] += h
        fm[0, fi, k, c] -= h
        fd = (loss(fp) - loss(fm)) / (fp[0, fi, k, c] - fm[0, fi, k, c]).item()
        assert abs(fd - f.grad[0, fi, k, c].item()) <= 2e-2 * scale, (fi, k, c, fd, f.grad[0, fi, k, c].item())


# ------------------------------------------------------------------------------------------------ direct ABI
def _abi_call(faces=None, verts=None, idx=None, S=48, sigma=1e-4, alpha=None, g=None, gf=None, gv=None, flags=0,
              backward=False, ws_pad=0):
    from neural_renderer_b200 import _lib
    lib = _lib.load()
    a = _lib.SoftArgs()
    a.struct_size = ctypes.sizeof(_lib.SoftArgs)
    ptr = lambda t: None if t is None else ctypes.c_void_p(t.data_ptr())  # noqa: E731
    if verts is not None:
        flags |= _lib.NR_FACES_INDEXED | (_lib.NR_INDICES_SHARED if idx.dim() == 2 else 0)
        a.vertices, a.face_indices, a.num_vertices, a.num_faces, B = ptr(verts), ptr(idx), verts.shape[1], idx.shape[-2], verts.shape[0]
    else:
        a.faces, a.num_faces, B = ptr(faces), faces.shape[1], faces.shape[0]
    a.flags, a.batch_size, a.image_size, a.sigma, a.near_, a.far_ = flags, B, S, sigma, 0.1, 100.0
    a.alpha, a.grad_alpha, a.grad_faces, a.grad_vertices = ptr(alpha), ptr(g), ptr(gf), ptr(gv)
    n = lib.nr_b200_soft_workspace_bytes(B, a.num_faces, S, sigma, flags)
    ws = torch.full((n + ws_pad,), 0xAB, dtype=torch.uint8, device=DEV)
    a.workspace, a.workspace_bytes = ptr(ws), n
    fn = lib.nr_b200_soft_silhouettes_backward if backward else lib.nr_b200_soft_silhouettes
    rc = fn(ctypes.byref(a), ctypes.c_void_p(torch.cuda.current_stream(DEV).cuda_stream))
    torch.cuda.synchronize()
    return rc, lib.nr_b200_last_launch_count()


def _guarded(shape, fill=float("nan"), guard=16):
    buf = torch.full((int(np.prod(shape)) + guard,), fill, dtype=torch.float32, device=DEV)
    buf[-guard:] = 12345.0
    return buf, buf[:-guard].view(shape)


@pytest.mark.parametrize("indexed", [False, True])
def test_abi_poison_guards_nulls_accumulate_and_refusals(indexed):
    nr = _nr()
    B, S, sigma = 2, 48, 1e-4
    faces = _special_faces(B, S, sigma, seed=31)
    Nv = faces.shape[1] * 3
    verts = faces.reshape(B, Nv, 3).contiguous()
    idx = torch.arange(Nv, dtype=torch.int32, device=DEV).reshape(-1, 3)
    geo = dict(verts=verts, idx=idx) if indexed else dict(faces=faces)
    ref = nr.rasterize_soft_silhouettes(faces, S, sigma)
    buf, alpha = _guarded((B, S, S))
    rc, n = _abi_call(**geo, S=S, sigma=sigma, alpha=alpha)
    assert rc == 0 and n >= 4
    assert torch.equal(alpha, ref) and torch.all(buf[-16:] == 12345.0)
    # backward: NaN-poisoned gradient fully overwritten (zero-fill + adds), guards intact
    g = torch.randn(B, S, S, device=DEV, generator=torch.Generator(device=DEV).manual_seed(8))
    gshape = (B, Nv, 3) if indexed else tuple(faces.shape)
    gbuf, grad = _guarded(gshape)
    kw = dict(gv=grad) if indexed else dict(gf=grad)
    assert _abi_call(**geo, S=S, sigma=sigma, alpha=alpha, g=g, backward=True, **kw)[0] == 0
    assert torch.isfinite(grad).all() and torch.all(gbuf[-16:] == 12345.0)
    f = faces.clone().requires_grad_(True)
    (nr.rasterize_soft_silhouettes(f, S, sigma) * g).sum().backward()
    want = f.grad.reshape(gshape)
    assert rel_err(grad.cpu().numpy(), want.cpu().numpy()) <= 1e-5
    # NR_GRAD_ACCUMULATE adds into the buffer
    from neural_renderer_b200 import _lib
    acc = torch.full(gshape, 0.5, device=DEV)
    kw = dict(gv=acc) if indexed else dict(gf=acc)
    assert _abi_call(**geo, S=S, sigma=sigma, alpha=alpha, g=g, backward=True, flags=_lib.NR_GRAD_ACCUMULATE, **kw)[0] == 0
    assert rel_err((acc - 0.5).cpu().numpy(), want.cpu().numpy()) <= 1e-5
    # grad_alpha NULL = zeros: the zero-fill only (or nothing at all with NR_GRAD_ACCUMULATE)
    gbuf, grad = _guarded(gshape)
    kw = dict(gv=grad) if indexed else dict(gf=grad)
    assert _abi_call(**geo, S=S, sigma=sigma, alpha=alpha, g=None, backward=True, **kw)[0] == 0
    assert torch.all(grad == 0) and torch.all(gbuf[-16:] == 12345.0)
    acc = torch.full(gshape, 0.5, device=DEV)
    kw = dict(gv=acc) if indexed else dict(gf=acc)
    rc, n = _abi_call(**geo, S=S, sigma=sigma, alpha=alpha, g=None, backward=True, flags=_lib.NR_GRAD_ACCUMULATE, **kw)
    assert rc == 0 and n == 0 and torch.all(acc == 0.5)
    # refusals: nothing launched, outputs untouched
    buf, alpha2 = _guarded((B, S, S), fill=7.0)
    for bad in (dict(sigma=0.0), dict(sigma=float("nan")), dict(sigma=-1.0), dict(S=0)):
        rc, n = _abi_call(**geo, alpha=alpha2, **{"S": S, "sigma": sigma, **bad})
        assert rc == -1 and n == 0 and torch.all(alpha2 == 7.0) and torch.all(buf[-16:] == 12345.0)


# ------------------------------------------------------------------------------------------------ behaviour
def _tri_at(cx, cy, s=4.0 / 256):
    """a triangle about 2 px across at 256 x 256 (s = 2 px in NDC), centred at (cx, cy), depth 1.5"""
    return torch.stack([torch.stack([cx - s / 2, cy - s / 3, torch.full_like(cx, 1.5)]),
                        torch.stack([cx + s / 2, cy - s / 3, torch.full_like(cx, 1.5)]),
                        torch.stack([cx, cy + 2 * s / 3, torch.full_like(cx, 1.5)])])[None, None]


def test_translation_fit_recovers_a_shift_the_hard_silhouette_cannot_see():
    nr = _nr()
    S, sigma = 256, 1e-4
    px = 2.0 / S
    tx, ty = torch.tensor(0.1013, device=DEV), torch.tensor(-0.0521, device=DEV)
    with torch.no_grad():
        target = nr.rasterize_soft_silhouettes(_tri_at(tx, ty), S, sigma)
        hard_t = nr.rasterize_silhouettes(_tri_at(tx, ty), S, False)
    shift = torch.tensor([3 * px, 0.0], device=DEV, requires_grad=True)
    start = _tri_at(tx + 3 * px, ty)
    hard_s = nr.rasterize_silhouettes(start, S, False)
    assert (hard_t * hard_s).sum() == 0  # no overlap: the hard silhouettes' loss has no gradient towards the target
    opt = torch.optim.Adam([shift], lr=0.2 * px)
    steps = 400
    for it in range(steps):
        for gr in opt.param_groups:  # cosine decay to 0.005 px per step
            gr["lr"] = px * (0.005 + 0.195 * 0.5 * (1 + math.cos(math.pi * it / steps)))
        opt.zero_grad()
        img = nr.rasterize_soft_silhouettes(_tri_at(tx + shift[0], ty + shift[1]), S, sigma)
        ((img - target) ** 2).sum().backward()
        opt.step()
    err_px = (shift.detach().abs().max() / px).item()
    assert err_px < 0.1, err_px


@pytest.mark.parametrize("fused", [True, False])
def test_renderer_fill_back_invariance_and_gradient_through_the_camera(fused):
    nr = _nr()
    d = np.load(os.path.join(os.path.dirname(__file__), "golden", "teapot.npz"))
    v = torch.from_numpy(d["vertices"].astype(np.float32)).to(DEV)[None].repeat(2, 1, 1)
    f = torch.from_numpy(d["faces"].astype(np.int32)).to(DEV)[None].expand(2, -1, -1)
    r = nr.Renderer()
    r.image_size = 128
    r.fused = fused
    r.eye = nr.get_points_from_angles(2.732, 20, 30)
    outs = []
    for fb in (True, False):
        r.fill_back = fb
        vv = v.clone().requires_grad_(True)
        img = r.render_soft_silhouettes(vv, f, sigma=1e-4)
        img.sum().backward()
        outs.append((img.detach(), vv.grad))
    assert torch.equal(outs[0][0], outs[1][0])
    assert outs[0][0].shape == (2, 128, 128) and outs[0][0].max() > 0.99
    gv = outs[0][1]
    assert torch.isfinite(gv).all() and gv.abs().sum() > 0
    # the same image as the free function on the camera-transformed geometry, without fill_back copies
    want = nr.rasterize_soft_silhouettes(f, 128, 1e-4, r.near, r.far, vertices=r._transform(v))
    assert torch.equal(outs[0][0], want)
