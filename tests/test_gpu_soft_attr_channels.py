"""GPU: the soft attribute images (csrc/nr_soft_attr.cu) held to float64 along the axes its kernels are split by, and
the soft renders of the Renderer captured in CUDA graphs.

soft_attr_launch runs channel blocks of kCB = 4 numerators per pixel for C <= 4 and kCB = 16 above that (_kcb).  The
forward runs ceil(C / kCB) grid.z blocks.  The backward reads the upstream gradient of the channels past kCB from
global memory (the tails of gdot and G) and spreads the attribute gradient over the lanes 32 channels at a time.  Each
test asserts the branch it claims: C for the channel block, soft_binning.key_width for the key width and
soft_binning.rounds for the staging rounds of a tile.

  a. C in {1, 4, 5, 16, 17, 32, 33, 64} on the special-face soup: forward, geometry and attribute gradients against
     float64 autograd, the four attribute forms taken in turn (each meets the kCB = 16 kernels);
  b. the backward is linear in the channels: a C-channel backward equals the sum of C one-channel backwards (no oracle);
  c. deep tiles (several 256-face staging rounds) against the sparse oracle, under the gates of test_gpu_soft_scale;
  d. 64-bit sort keys with kCB = 16: bit-identical across face counts, padding faces get nothing;
  e. needle slivers: finite, inside each channel's hull;
  f. one captured step of every soft entry of the Renderer, replayed against the eager step.

The forward gate of a and d is test_gpu_soft_attr's (tol_attr, the cut-off bracketed +-1e-5), the gradient gates are
rel_err <= 5e-3 and elem_err(floor 2e-2) <= 5e-2 (test_gpu_soft_scale.check_grads)."""
import math

import numpy as np
import pytest
import torch

import oracles_soft as osoft
import oracles_soft_attr as oattr
import soft_binning as sb
import test_gpu_soft_attr as tsa
import test_gpu_soft_scale as tss
from helpers import np_, rel_err

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
NEAR, FAR = 0.1, 100.0


def _nr():
    import neural_renderer_b200 as nr
    return nr


def _kcb(C):
    """the channel block soft_attr_launch picks for C channels"""
    return 4 if C <= 4 else 16


# ------------------------------------------------------------------------------------------------ a. the channel axis
CHANNELS = (1, 4, 5, 16, 17, 32, 33, 64)
FORMS = ("corner", "corner_shared", "vertex_shared", "vertex")


def _oracle_faces(verts, idx):
    """the faces the kernels draw from indexed geometry, a face with an out-of-range corner (which takes no part) as an
    off-image stand-in, as tsa._oracle_grads builds them"""
    fc = osoft.gather_faces(verts.double(), idx)
    pad = torch.tensor([[10.0, 10.0, 1.0], [10.5, 10.0, 1.0], [10.0, 10.5, 1.0]], dtype=torch.float64, device=DEV)
    return torch.where(osoft.participates(fc, NEAR, FAR)[..., None, None], fc, pad)


@pytest.mark.parametrize("C", CHANNELS)
def test_channel_blocks_against_float64(C):
    nr = _nr()
    form = FORMS[CHANNELS.index(C) % len(FORMS)]
    S, B, sigma, gamma = 64, 2, 1e-4, 1e-2
    faces = tsa._special_faces(B, sigma, seed=41, F=12)
    F = faces.shape[1]
    assert sb.key_width(B, F, S)[2] is False
    kcb = _kcb(C)
    assert kcb == (16 if C >= 5 else 4)
    bg = tuple(float(v) for v in tsa._rand((C,), 500 + C, -2.0, 2.0).tolist())
    gen = torch.Generator(device=DEV).manual_seed(600 + C)
    g_out = torch.randn(B, C, S, S, device=DEV, generator=gen)
    g_a = torch.randn(B, S, S, device=DEV, generator=gen)
    kw = {}
    if form.startswith("vertex"):
        verts, idx = tsa._as_vertices(faces)
        if form == "vertex_shared":
            idx = idx.clone()
            idx[2, 1] = 3 * F              # out of range: reads zeros, the face takes no part
        va = tsa._rand((1 if form == "vertex_shared" else B, 3 * F, C), 700 + C, -3.0, 3.0)
        kw = dict(verts=verts, idx=idx, va=va)
        out, alpha = nr.rasterize_soft_attributes(idx, S, sigma, gamma, vertices=verts, vertex_attributes=va,
                                                  background=bg, return_alpha=True)
        fo, co = _oracle_faces(verts, idx), oattr.corner_attributes(va, idx)
        ca = None
    else:
        ca = tsa._rand((1 if form == "corner_shared" else B, F, 3, C), 700 + C, -3.0, 3.0)
        out, alpha = nr.rasterize_soft_attributes(faces, S, sigma, gamma, face_attributes=ca, background=bg,
                                                  return_alpha=True)
        fo, co = faces, ca
    assert out.shape == (B, C, S, S)
    tsa._check_forward(out, alpha, fo, co, S, sigma, gamma, bg)
    got = tsa._grads(faces, ca, S, sigma, gamma, bg, g_out, g_a, **kw)
    ref = tsa._oracle_grads(faces, ca, S, sigma, gamma, bg, g_out, g_a, **kw)
    tss.check_grads(got, ref, ("geometry", "attributes"), (C, form))
    # every channel's attributes receive a gradient, the second lane block's and the global-memory tail's included
    assert torch.all((got[1].reshape(-1, C) != 0).any(0)), C
    if form == "vertex_shared":
        assert torch.all(got[1][0, 3 * 2 + 1] == 0)     # only the out-of-range slot referenced this vertex


# ------------------------------------------------------------------------------------------------ b. channel linearity
@pytest.mark.parametrize("C", [33, 64])
def test_backward_is_the_sum_of_one_channel_backwards(C):
    """loss = sum_c sum_p g_c out_c, and out_c is a function of the geometry and channel c alone: with no alpha gradient
    the geometry gradient is the sum of the C one-channel geometry gradients and the attribute gradient of channel c is
    its one-channel one.  Only the order of the fp32 atomics differs."""
    from neural_renderer_b200 import synthetic
    nr = _nr()
    S, B, sigma, gamma = 64, 2, 1e-3, 1e-2
    faces = torch.from_numpy(synthetic.triangle_soup(B, 48, seed=111, size=(0.3, 0.8), offscreen=False,
                                                     duplicates=False)).to(DEV)
    d2, inside = osoft.face_terms(faces.double(), osoft.pixel_centres(S, device=DEV))
    n_on = (osoft.participates(faces.double(), NEAR, FAR)[..., None] & (inside | (d2 <= osoft.cut(sigma)))).sum(1)
    assert (n_on >= 4).double().mean().item() > 0.25        # several faces per pixel
    assert _kcb(C) == 16 and C > 32                          # the tails and a second lane block
    ca = tsa._rand((B, faces.shape[1], 3, C), 120 + C, -3.0, 3.0)
    bg = [float(v) for v in tsa._rand((C,), 130 + C, -2.0, 2.0).tolist()]
    g = torch.randn(B, C, S, S, device=DEV, generator=torch.Generator(device=DEV).manual_seed(140 + C))
    f = faces.clone().requires_grad_(True)
    a = ca.clone().requires_grad_(True)
    out = nr.rasterize_soft_attributes(f, S, sigma, gamma, face_attributes=a, background=bg)
    out.backward(g)
    geom = torch.zeros_like(faces)
    for c in range(C):
        f1 = faces.clone().requires_grad_(True)
        a1 = ca[..., c:c + 1].clone().requires_grad_(True)
        o1 = nr.rasterize_soft_attributes(f1, S, sigma, gamma, face_attributes=a1, background=[bg[c]])
        assert torch.equal(o1[:, 0], out[:, c]), c
        o1.backward(g[:, c:c + 1].contiguous())
        geom += f1.grad
        assert rel_err(np_(a.grad[..., c]), np_(a1.grad[..., 0])) <= 1e-5, (c, rel_err(np_(a.grad[..., c]),
                                                                                       np_(a1.grad[..., 0])))
    assert rel_err(np_(f.grad), np_(geom)) <= 1e-4, rel_err(np_(f.grad), np_(geom))


# ------------------------------------------------------------------------------------------------ c. deep tiles
class AttrScene(tss.Scene):
    """test_gpu_soft_scale's Scene of a soft attribute image: `tex` holds per-corner attributes [1|B,F,3,C], whose
    colour sensitivity k_C is 3 times the span of a face's corner values (|dA| <= span sum_k |dl_k|)"""

    def __init__(self, faces, ca, bg):
        super().__init__("attr", faces, tex=ca, bg=tuple(bg))

    def render(self, S, sigma, gamma, faces=None, tex=None, **kw):
        return _nr().rasterize_soft_attributes(self.faces if faces is None else faces, S, sigma, gamma,
                                               face_attributes=self.tex if tex is None else tex, background=self.bg,
                                               return_alpha=True)

    def oracle_terms(self, leaves, S, sigma, cut_scale=1.0):
        ca = leaves[1].double()

        def terms(b0, b1, idx, fc, p):
            return oattr.attr_terms(fc, osoft.take(ca, b0, b1, idx), p, sigma, NEAR, FAR, cut_scale)
        return terms

    def colour_sensitivity(self):
        t = self.tex.double()
        return 3 * (t.amax(2) - t.amin(2)).amax(-1)


GROUP = 7   # channels per forward check: the float64 gate terms grow with the channel count


@pytest.mark.parametrize("C, gamma", [(3, 1e-4), (21, 1e-2)])
def test_deep_tiles_forward_every_pixel_gradients_and_permutation(C, gamma):
    S, sigma = tss.S_DEEP, tss.SIGMA_DEEP
    faces = tss._deep_faces()
    F = faces.shape[1]
    lb = sb.tile_entries_lower_bound(faces, S, sigma)[0]
    deep = int(lb.argmax())
    assert sb.rounds(lb[deep]).item() >= 3 and _kcb(C) == (4 if C == 3 else 16)
    ca = tsa._rand((1, F, 3, C), 150 + C, -1.0, 1.0)
    bg = [float(v) for v in tsa._rand((C,), 160 + C, -1.0, 1.0).tolist()]
    sc = AttrScene(faces, ca, bg)
    out, alpha = sc.render(S, sigma, gamma)
    # every pixel, as a batch of tiles over the one item (the cull works tile by tile), a group of channels at a time
    nt = sb.tiles_per_axis(S)
    T = nt * nt
    pix = tss._tile_pixels(S, torch.arange(T))
    for c0 in range(0, C, GROUP):
        c1 = min(C, c0 + GROUP)
        tsc = AttrScene(faces.expand(T, -1, -1, -1), ca[..., c0:c1], bg[c0:c1])
        worst = tss.check_forward(tsc, out[:, c0:c1].expand(T, -1, -1, -1), alpha.expand(T, -1, -1), S, sigma, gamma,
                                  pix, ("deep attr", C, c0))
        print("deep attr", C, gamma, c0, worst)
    # gradients: the upstream gradient on the deepest tile and on the tile of pixel (45, 82), inside the front face
    sel = tss._tile_pixels(S, [deep, (45 // 16) * nt + 82 // 16]).reshape(1, -1)
    g = torch.Generator(device=DEV).manual_seed(170 + C)
    g_a_p = torch.randn(1, sel.shape[1], device=DEV, generator=g, dtype=torch.float64)
    g_out_p = torch.randn(1, C, sel.shape[1], device=DEV, generator=g, dtype=torch.float64)
    g_a = torch.zeros(1, S * S, device=DEV)
    g_a[0, sel[0]] = g_a_p[0].float()
    g_out = torch.zeros(1, C, S * S, device=DEV)
    g_out[0][:, sel[0]] = g_out_p[0].float()
    got = tss.kernel_grads(sc, S, sigma, gamma, g_out.reshape(1, C, S, S), g_a.reshape(1, S, S))
    ref = tss.oracle_grads(sc, S, sigma, gamma, sel, g_out_p, g_a_p)
    tss.check_grads(got, ref, ("faces", "attributes"), ("deep attr", C, gamma))
    # the front face, at the highest index, arrives in the last round and still receives its gradient
    assert got[0][0, F - 1].abs().max() > 0 and got[1][0, F - 1].abs().max() > 0
    # alpha bit-identical and every channel within fp32 rounding under a permutation of the faces
    perm = torch.from_numpy(np.random.default_rng(38).permutation(F)).to(DEV)
    out_p, alpha_p = AttrScene(faces[:, perm].contiguous(), ca[:, perm].contiguous(), bg).render(S, sigma, gamma)
    assert torch.equal(alpha_p, alpha)
    err = (out_p - out).abs().amax((0, 2, 3))
    assert torch.all(err <= 2e-5), err.tolist()


# ------------------------------------------------------------------------------------------------ d. 64-bit keys, kCB 16
def test_64_bit_keys_with_sixteen_channel_blocks():
    nr = _nr()
    S, sigma, gamma = tss.S_KEY, tss.SIGMA_KEY, tss.GAMMA_KEY
    C = 17
    real = tss._real_faces(2, seed=1)
    B, Fr = real.shape[:2]
    assert _kcb(C) == 16
    va = tsa._rand((1, 3 * Fr, C), 181, 0.0, 1.0)
    bg = tuple(float(v) for v in torch.linspace(0.05, 0.85, C).tolist())
    pix = tss._pixels_near(real, S, 4000, seed=2)
    g_out = tsa._rand((B, C, S, S), 182)
    ref = None
    for F in (Fr, 65535, 65536):
        assert sb.key_width(B, F, S)[2] == (F == 65536)
        faces, pos = tss._padded(real, F, seed=3)
        verts, idx = tss._indexed(faces, pos)
        v = verts.clone().requires_grad_(True)
        a = torch.cat((va, torch.zeros(1, 12, C, device=DEV)), 1).requires_grad_(True)
        out, alpha = nr.rasterize_soft_attributes(idx, S, sigma, gamma, vertices=v, vertex_attributes=a,
                                                  background=bg, return_alpha=True)
        out.backward(g_out)
        gv, ga = v.grad[:, :3 * Fr], a.grad[:, :3 * Fr]
        assert torch.all(v.grad[:, 3 * Fr:] == 0) and torch.all(a.grad[:, 3 * Fr:] == 0)   # the padding
        if ref is None:
            # the sparse oracle at the first count; the images of the others are compared on the host (their
            # [2,17,2049,2049] copies would double this test's device memory)
            ca = oattr.corner_attributes(va, torch.arange(3 * Fr, device=DEV).reshape(Fr, 3))
            want, want_a = oattr.soft_attributes(real.double(), ca.double(), S, sigma, gamma, NEAR, FAR, bg, pix=pix)
            got = torch.gather(out.reshape(B, C, -1), 2, pix[:, None].expand(-1, C, -1))
            assert (got.double() - want).abs().max().item() <= 4 * (4 * tsa.tol(sigma) + 5e-4)
            ref = (out.cpu(), alpha.cpu(), gv.clone(), ga.clone())
            assert gv.abs().max() > 0 and torch.all((ga.reshape(-1, C) != 0).any(0))
        else:
            assert torch.equal(out.cpu(), ref[0]) and torch.equal(alpha.cpu(), ref[1]), F
            # fp32 atomics land in another order: the gradients agree per tensor
            assert rel_err(np_(gv), np_(ref[2])) <= 1e-5, F
            assert rel_err(np_(ga), np_(ref[3])) <= 1e-5, F
        del out, alpha, v, a


# ------------------------------------------------------------------------------------------------ e. slivers
@pytest.mark.parametrize("C", [3, 17])
def test_slivers_stay_finite_and_inside_each_channel_hull(C):
    """needles (synthetic.needle_faces): A_jc = sum_k l'_k a_kc with the l'_k a convex combination, and out_c blends
    those with the background, so every channel lies inside the hull of the background and that channel's attributes"""
    from neural_renderer_b200 import synthetic
    nr = _nr()
    S, sigma, gamma, B, F = 64, 1e-4, 1e-3, 2, 40
    faces = torch.from_numpy(synthetic.needle_faces(B, F, S, seed=61)).to(DEV)
    ca = tsa._rand((B, F, 3, C), 190 + C, -1.0, 1.0)
    bg = tsa._rand((C,), 200 + C, -1.0, 1.0)
    lo = torch.minimum(ca.amin((1, 2)), bg)                          # [B,C]
    hi = torch.maximum(ca.amax((1, 2)), bg)
    f = faces.clone().requires_grad_(True)
    a = ca.clone().requires_grad_(True)
    out, alpha = nr.rasterize_soft_attributes(f, S, sigma, gamma, face_attributes=a, background=bg, return_alpha=True)
    assert torch.isfinite(out).all() and torch.isfinite(alpha).all()
    slack = 1e-5
    assert torch.all(out >= lo[:, :, None, None] - slack) and torch.all(out <= hi[:, :, None, None] + slack)
    gen = torch.Generator(device=DEV).manual_seed(210 + C)
    ((out * torch.randn(B, C, S, S, device=DEV, generator=gen)).sum() +
     (alpha * torch.randn(B, S, S, device=DEV, generator=gen)).sum()).backward()
    assert torch.isfinite(f.grad).all() and torch.isfinite(a.grad).all()
    assert f.grad.abs().max() > 0 and a.grad.abs().max() > 0


# ------------------------------------------------------------------------------------------------ f. CUDA graphs
def _teapot_renderer():
    import os
    nr = _nr()
    d = np.load(os.path.join(os.path.dirname(__file__), "golden", "teapot.npz"))
    v = torch.from_numpy(d["vertices"].astype(np.float32)).to(DEV)[None].repeat(2, 1, 1).requires_grad_(True)
    f = torch.from_numpy(d["faces"].astype(np.int32)).to(DEV)[None].repeat(2, 1, 1)
    r = nr.Renderer()
    r.image_size = 64
    r.eye = nr.get_points_from_angles(2.732, 30, -15)
    return r, v, f


def _captured_step_matches_eager(run, leaves):
    """run() renders and returns (outputs, loss).  One eager step, a warm-up on a side stream, then one step captured
    in a CUDA graph and replayed: the replayed outputs equal the eager ones bit for bit, the gradients to 1e-5 per
    tensor (the fp32 atomics land in any order)."""
    def step():
        for x in leaves:
            x.grad = None
        outs, loss = run()
        loss.backward()
        return [o.detach().clone() for o in outs], [x.grad.clone() for x in leaves]

    eager = step()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            step()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        got = step()
    for t in got[0] + got[1]:
        t.fill_(float("nan"))
    graph.replay()
    torch.cuda.synchronize()
    for a, b in zip(got[0], eager[0]):
        assert torch.equal(a, b)
    for x, a, b in zip(leaves, got[1], eager[1]):
        assert b.abs().max() > 0 and rel_err(np_(a), np_(b)) <= 1e-5, rel_err(np_(a), np_(b))


def _weights(shape, seed):
    return torch.randn(shape, device=DEV, generator=torch.Generator(device=DEV).manual_seed(seed))


def test_render_soft_silhouettes_step_in_cuda_graph():
    r, v, f = _teapot_renderer()
    g = _weights((2, 64, 64), 221)

    def run():
        sil = r.render_soft_silhouettes(v, f, sigma=1e-4)
        return (sil,), (sil * g).sum()
    _captured_step_matches_eager(run, [v])


def test_render_soft_cubes_step_in_cuda_graph():
    r, v, f = _teapot_renderer()
    tex = tsa._rand((2, f.shape[1], 2, 2, 2, 3), 222, 0.0, 1.0).requires_grad_(True)
    g, ga = _weights((2, 3, 64, 64), 223), _weights((2, 64, 64), 224)

    def run():
        rgb, alpha = r.render_soft(v, f, tex, sigma=1e-4, gamma=1e-3)
        return (rgb, alpha), (rgb * g).sum() + (alpha * ga).sum()
    _captured_step_matches_eager(run, [v, tex])


def test_render_soft_uv_trilinear_step_in_cuda_graph():
    r, v, f = _teapot_renderer()
    r.texture_filter = 'trilinear'
    img = tss._image(1, 32, 48, 225).requires_grad_(True)
    uvs = tsa._rand((f.shape[1], 3, 2), 226, 0.05, 0.95).requires_grad_(True)
    g, ga = _weights((2, 3, 64, 64), 227), _weights((2, 64, 64), 228)

    def run():
        rgb, alpha = r.render_soft(v, f, img, sigma=1e-4, gamma=1e-3, face_uvs=uvs)
        return (rgb, alpha), (rgb * g).sum() + (alpha * ga).sum()
    _captured_step_matches_eager(run, [v, img, uvs])


@pytest.mark.parametrize("background", ["list", "tensor", "none"])
def test_render_soft_attributes_step_in_cuda_graph(background):
    r, v, f = _teapot_renderer()
    C = 5
    va = tsa._rand((1, v.shape[1], C), 229, -1.0, 1.0).requires_grad_(True)
    bg = {"list": [0.1, -0.2, 0.3, 0.4, -0.5], "tensor": tsa._rand((C,), 230, -1.0, 1.0), "none": None}[background]
    g = _weights((2, C, 64, 64), 231)

    def run():
        out = r.render_soft_attributes(v, f, vertex_attributes=va, sigma=1e-4, gamma=1e-3, background=bg)
        return (out,), (out * g).sum()
    _captured_step_matches_eager(run, [v, va])


def test_render_soft_depth_step_in_cuda_graph():
    r, v, f = _teapot_renderer()
    g = _weights((2, 64, 64), 232)

    def run():
        d = r.render_soft_depth(v, f, sigma=1e-4, gamma=1e-3)
        return (d,), (d * g).sum()
    _captured_step_matches_eager(run, [v])
