"""GPU: the soft blend of fragments (blend_soft_fragments, nr_b200_blend_fragments[_backward]) against the float64
oracle of tests/oracles_soft_blend.py, under the derived gates of its docstring, and against the soft attribute images.

The synthetic fragment tensors have empty slots interleaved with valid ones (holding NaN and inf, which must not reach
anything), unsorted slots, all-empty pixels and exact zbuf ties; dists lie within the fragments' reach.  Gradients are
compared with float64 autograd of the oracle per element (helpers.elem_err).  No test peaks above 2.2 GiB of device
memory, so the scale tests' process-peak check still holds after this file."""
import ctypes
import math

import pytest
import torch

import oracles_soft_blend as oblend
from helpers import elem_err, rel_err

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
NEAR, FAR = 0.1, 100.0
PEAK_LIMIT = int(2.2 * 2 ** 30)
INVALID = -1  # NR_ERR_INVALID_ARG

# (K, C) past the staging budget of both kernels (the forward stages up to K 32 C 7, the backward up to K 32 C 5,
# K 16 C 17, K 8 C 40): these run the per-thread kernels
PER_THREAD_SHAPES = [(32, 16), (16, 24)]


def _nr():
    import neural_renderer_b200 as nr
    return nr


@pytest.fixture(autouse=True)
def _peak_memory():
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats(DEV)
    yield
    torch.cuda.synchronize()
    assert torch.cuda.max_memory_allocated(DEV) <= PEAK_LIMIT, torch.cuda.max_memory_allocated(DEV)


def _synthetic(B, H, W, K, C, sigma, seed):
    """(Fragments, colors): random faces in 30 % of the slots left empty, every 7th pixel empty, unsorted depths with
    exact ties, dists within +-8 sigma; empty slots hold NaN / inf in zbuf, dists and colours"""
    nr = _nr()
    g = torch.Generator(device=DEV).manual_seed(seed)
    p2f = torch.randint(0, 1000, (B, H, W, K), device=DEV, generator=g)
    p2f[torch.rand(B, H, W, K, device=DEV, generator=g) < 0.3] = -1
    p2f.view(B, -1, K)[:, ::7] = -1
    zb = 1.0 + 4.0 * torch.rand(B, H, W, K, device=DEV, generator=g)
    tie = torch.rand(B, H, W, K, device=DEV, generator=g) < 0.2
    zb = torch.where(tie, torch.round(zb * 4) / 4, zb)                           # exact ties
    ds = (torch.rand(B, H, W, K, device=DEV, generator=g) * 2 - 1) * 8 * sigma
    col = torch.rand(B, H, W, K, C, device=DEV, generator=g)
    empty = p2f < 0
    zb = torch.where(empty, torch.full_like(zb, float("nan")), zb)
    ds = torch.where(empty, torch.full_like(ds, float("inf")), ds)
    col = torch.where(empty[..., None], torch.full_like(col, float("nan")), col)
    return nr.Fragments(p2f, zb, None, ds), col


def _rand(shape, seed, lo=-1.0, hi=1.0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return lo + (hi - lo) * torch.rand(*shape, device=DEV, generator=g)


def _check_forward(frag, col, sigma, gamma, bg, out, alpha, rows=32):
    """out and alpha against the oracle under the derived gates, rows at a time (float64 stays small)"""
    H = col.shape[2]
    for r0 in range(0, H, rows):
        sl = slice(r0, r0 + rows)
        args = (frag.pix_to_face[:, sl], frag.zbuf[:, sl], frag.dists[:, sl], col[:, sl], sigma, gamma, NEAR, FAR, bg)
        ref_o, ref_a = oblend.blend(*args)
        g_o, g_a = oblend.gates(*args)
        err_o = (out[:, :, sl].double() - ref_o).abs()
        err_a = (alpha[:, sl].double() - ref_a).abs()
        assert torch.all(err_o <= g_o), (err_o - g_o).max().item()
        assert torch.all(err_a <= g_a), (err_a - g_a).max().item()


# ------------------------------------------------------------------------------------------------ forward
@pytest.mark.parametrize("HW", [(64, 64), (127, 129), (257, 257)])
@pytest.mark.parametrize("C", [1, 3, 4, 16, 21])
@pytest.mark.parametrize("K", [1, 3, 8, 32])
def test_forward_against_the_oracle(K, C, HW):
    nr = _nr()
    H, W = HW
    B = 1 if H > 200 else 3
    for i, (gamma, sigma) in enumerate(((1e-4, 1e-5), (1e-4, 1e-3), (1e-2, 1e-5), (1e-2, 1e-3))):
        frag, col = _synthetic(B, H, W, K, C, sigma, 1000 * K + 10 * C + i)
        bg = [0.1 * (c % 7) for c in range(C)] if i % 2 else None
        out, alpha = nr.blend_soft_fragments(frag, col, sigma, gamma, NEAR, FAR, background=bg)
        assert out.shape == (B, C, H, W) and alpha.shape == (B, H, W)
        _check_forward(frag, col, sigma, gamma, bg, out, alpha)
        empty = (frag.pix_to_face < 0).all(-1)
        want = torch.tensor(bg if bg else [0.0] * C, device=DEV)
        assert torch.equal(out.permute(0, 2, 3, 1)[empty], want.expand(int(empty.sum()), C))
        assert torch.all(alpha[empty] == 0)


@pytest.mark.parametrize("KC", PER_THREAD_SHAPES)
def test_forward_past_the_staging_budget(KC):
    nr = _nr()
    K, C = KC
    B, H, W, sigma, gamma = 2, 37, 41, 1e-4, 1e-3
    frag, col = _synthetic(B, H, W, K, C, sigma, 400 + C)
    bg = [0.01 * c for c in range(C)]
    out, alpha = nr.blend_soft_fragments(frag, col, sigma, gamma, NEAR, FAR, background=bg)
    _check_forward(frag, col, sigma, gamma, bg, out, alpha, rows=8)


# ------------------------------------------------------------------------------------------------ backward
def _grads(frag, col, sigma, gamma, bg, g_out, g_alpha, f64):
    nr = _nr()
    dt = torch.float64 if f64 else torch.float32
    zv = frag.zbuf.to(dt).requires_grad_(True)
    dv = frag.dists.to(dt).requires_grad_(True)
    cv = col.to(dt).requires_grad_(True)
    if f64:
        out, alpha = oblend.blend(frag.pix_to_face, zv, dv, cv, sigma, gamma, NEAR, FAR, bg)
    else:
        out, alpha = nr.blend_soft_fragments(nr.Fragments(frag.pix_to_face, zv, None, dv), cv, sigma, gamma, NEAR, FAR,
                                             background=bg)
    loss = 0
    if g_out is not None:
        loss = loss + (out * g_out.to(dt)).sum()
    if g_alpha is not None:
        loss = loss + (alpha * g_alpha.to(dt)).sum()
    grads = torch.autograd.grad(loss, (zv, dv, cv), allow_unused=True)
    return tuple(torch.zeros_like(t) if g is None else g for g, t in zip(grads, (zv, dv, cv)))


@pytest.mark.parametrize("which", ["out", "alpha", "both"])
@pytest.mark.parametrize("gamma", [1e-4, 1e-2])
@pytest.mark.parametrize("KC", [(8, 3), (5, 17), (32, 4)] + PER_THREAD_SHAPES)
def test_backward_against_float64_autograd(KC, gamma, which):
    K, C = KC
    B, H, W, sigma = 2, 33, 35, 1e-3
    frag, col = _synthetic(B, H, W, K, C, sigma, 77 + K)
    bg = [0.25] * C
    g_out = _rand((B, C, H, W), 78) if which != "alpha" else None
    g_alpha = _rand((B, H, W), 79) if which != "out" else None
    got = _grads(frag, col, sigma, gamma, bg, g_out, g_alpha, False)
    want = _grads(frag, col, sigma, gamma, bg, g_out, g_alpha, True)
    empty = frag.pix_to_face < 0
    for name, g, w in zip(("zbuf", "dists", "colors"), got, want):
        assert torch.isfinite(g).all(), name
        e = elem_err(g.cpu(), w.cpu(), floor=1e-3)
        assert e <= 2e-3, (name, e)
        ge = g[empty] if g.dim() == 4 else g[empty[..., None].expand_as(g)]
        assert torch.all(ge == 0), name                       # empty slots: exactly 0
    if which == "alpha":
        assert torch.all(got[2] == 0) and torch.all(got[0] == 0)  # no colour or depth gradient without grad_out


# ------------------------------------------------------------------------------------------------ bit identities
def test_bit_identities():
    nr = _nr()
    B, H, W, K, C, sigma, gamma = 2, 40, 41, 6, 5, 1e-4, 1e-3
    frag, col = _synthetic(B, H, W, K, C, sigma, 5)
    bg = [0.3, 0.1, 0.7, 0.2, 0.9]
    g_out, g_alpha = _rand((B, C, H, W), 6), _rand((B, H, W), 7)

    def run(fr, cl, bgv, go):
        zv = fr.zbuf.clone().requires_grad_(True)
        dv = fr.dists.clone().requires_grad_(True)
        cv = cl.clone().requires_grad_(True)
        out, alpha = nr.blend_soft_fragments(nr.Fragments(fr.pix_to_face, zv, None, dv), cv, sigma, gamma, NEAR, FAR,
                                             background=bgv)
        torch.autograd.backward((out, alpha), (go, g_alpha))
        return out.detach(), alpha.detach(), zv.grad, dv.grad, cv.grad

    ref = run(frag, col, bg, g_out)
    for x, y in zip(ref, run(frag, col, bg, g_out)):              # repeat
        assert torch.equal(x, y)
    # appending empty slots (K 6 -> 13) changes no bit
    p = 7
    pad = lambda t, v: torch.cat((t, torch.full((*t.shape[:3], p, *t.shape[4:]), v, dtype=t.dtype, device=DEV)), 3)  # noqa: E731
    fp = nr.Fragments(pad(frag.pix_to_face, -1), pad(frag.zbuf, float("nan")), None, pad(frag.dists, 5.0))
    got = run(fp, pad(col, float("nan")), bg, g_out)
    for x, y in zip(ref[:2], got[:2]):
        assert torch.equal(x, y)
    for x, y in zip(ref[2:], got[2:]):
        assert torch.equal(x, y[:, :, :, :K]) and torch.all(y[:, :, :, K:] == 0)
    # channel c of the C-channel call against a C = 1 call on that channel alone (forward, and its colour gradient)
    for c in range(C):
        one = run(frag, col[..., c:c + 1].contiguous(), [bg[c]], g_out[:, c:c + 1].contiguous())
        assert torch.equal(one[0][:, 0], ref[0][:, c])
        assert torch.equal(one[1], ref[1])
        assert torch.equal(one[4][..., 0], ref[4][..., c])


# ------------------------------------------------------------------------------------------------ end to end
def _e2e(faces, S, sigma, gamma, K, ca, bg, mask_overfull=False):
    """(blended, reference, blended grads, reference grads, n < K mask) of the fragment pipeline against
    rasterize_soft_attributes; mask_overfull: the upstream gradient is zero at pixels with K fragments (there the
    fragments are not the contributing set, so the two pipelines differ by definition)"""
    from neural_renderer_b200 import functional as Fn
    nr = _nr()
    fv, cv = faces.clone().requires_grad_(True), ca.clone().requires_grad_(True)
    frag = nr.rasterize_soft_fragments(fv, S, sigma, K)
    out, _ = nr.blend_soft_fragments(frag, Fn.interpolate_face_attributes(frag.pix_to_face, frag.bary_coords, cv),
                                     sigma, gamma, NEAR, FAR, background=bg)
    fw, cw = faces.clone().requires_grad_(True), ca.clone().requires_grad_(True)
    ref = nr.rasterize_soft_attributes(fw, S, sigma, gamma, face_attributes=cw, background=bg)
    up = _rand(ref.shape, 53)
    n = (frag.pix_to_face >= 0).sum(-1)
    if mask_overfull:
        up = up * (n < K)[:, None]
    (out * up).sum().backward()
    (ref * up).sum().backward()
    return out.detach(), ref.detach(), (fv.grad, cv.grad), (fw.grad, cw.grad), frag, n < K


@pytest.mark.parametrize("gamma", [1e-4, 1e-2])
def test_blended_fragments_equal_the_soft_attributes(gamma):
    from test_gpu_soft_frag import _blend, _special_faces
    S, sigma, K = 64, 1e-3, 16
    faces = _special_faces(2, sigma, 51, F=20)
    B, F = faces.shape[:2]
    ca = _rand((B, F, 3, 3), 52, 0.0, 1.0)
    bg = (0.2, 0.5, 0.8)
    out, ref, g, gr, frag, under = _e2e(faces, S, sigma, gamma, K, ca, bg)
    assert under.all()                                        # every pixel's fragment set is the contributing set
    gate = 4 * (1e-6 / math.sqrt(sigma) + 1e-6) + 5e-4       # test_gpu_soft_frag's gates
    assert (out - ref).abs().max().item() <= gate, (out - ref).abs().max().item()
    assert rel_err(g[1].cpu(), gr[1].cpu()) <= 1e-4, rel_err(g[1].cpu(), gr[1].cpu())
    assert rel_err(g[0].cpu(), gr[0].cpu()) <= 2e-3, rel_err(g[0].cpu(), gr[0].cpu())
    # the torch blend the fragment tests trust, on the same fragments
    from neural_renderer_b200 import functional as Fn
    nr = _nr()
    tb = _blend(frag, ca, sigma, gamma, bg)
    kb, _ = nr.blend_soft_fragments(frag, Fn.interpolate_face_attributes(frag.pix_to_face, frag.bary_coords, ca),
                                    sigma, gamma, NEAR, FAR, background=bg)
    assert (kb - tb).abs().max().item() <= gate, (kb - tb).abs().max().item()
    # soft depth: the camera z as the attribute, the background at far
    z = faces[..., 2:3].contiguous()
    dref = nr.rasterize_soft_attributes(faces, S, sigma, gamma, face_attributes=z, background=[FAR])
    dout, _ = nr.blend_soft_fragments(frag, Fn.interpolate_face_attributes(frag.pix_to_face, frag.bary_coords, z),
                                      sigma, gamma, NEAR, FAR, background=[FAR])
    assert ((dout - dref).abs() / dref.abs().clamp_min(1.0)).max().item() <= gate


def test_sphere_benchmark_geometry_at_256():
    from neural_renderer_b200 import synthetic
    S, sigma, gamma, K, B = 256, 1e-4, 1e-4, 32, 2
    faces = torch.from_numpy(synthetic.sphere_faces(B, 5000)).to(DEV)
    ca = _rand((B, 5000, 3, 3), 54, 0.0, 1.0)
    out, ref, g, gr, frag, under = _e2e(faces, S, sigma, gamma, K, ca, (0.2, 0.5, 0.8), mask_overfull=True)
    assert under.float().mean().item() >= 0.9, under.float().mean().item()
    m = under[:, None].expand_as(out)
    gate = 4 * (1e-6 / math.sqrt(sigma) + 1e-6) + 5e-4
    assert (out - ref)[m].abs().max().item() <= gate, (out - ref)[m].abs().max().item()
    # the gradients of the pixels with fewer than K fragments (the others get no upstream gradient)
    assert rel_err(g[1].cpu(), gr[1].cpu()) <= 1e-4, rel_err(g[1].cpu(), gr[1].cpu())
    assert rel_err(g[0].cpu(), gr[0].cpu()) <= 2e-3, rel_err(g[0].cpu(), gr[0].cpu())


# ------------------------------------------------------------------------------------------------ direct ABI
def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream(DEV).cuda_stream)


def _guarded(n, dtype, fill, offset=0, guard=16):
    buf = torch.full((n + 2 * guard + offset,), fill, dtype=dtype, device=DEV)
    return buf, buf[guard + offset:guard + offset + n]


def _abi(frag, col, sigma, gamma, bg=None):
    from neural_renderer_b200 import _lib
    B, H, W, K, C = col.shape
    a = _lib.BlendArgs(struct_size=ctypes.sizeof(_lib.BlendArgs), batch_size=B, height=H, width=W, faces_per_pixel=K,
                       channels=C, sigma=sigma, gamma=gamma, near_=NEAR, far_=FAR)
    a.pix_to_face, a.zbuf, a.dists, a.colors = (t.data_ptr() for t in (frag.pix_to_face, frag.zbuf, frag.dists, col))
    a.background = bg.data_ptr() if bg is not None else None
    return a


@pytest.mark.parametrize("KC", [(8, 3), (3, 5), (32, 8)])  # (32, 8): past the staging budget, per thread
def test_abi_poison_guards_misalignment_and_refusals(KC):
    from neural_renderer_b200 import _lib
    nr = _nr()
    lib = _lib.load()
    K, C = KC
    B, H, W, sigma, gamma = 2, 30, 31, 1e-3, 1e-3
    frag, col = _synthetic(B, H, W, K, C, sigma, 200 + K)
    bg = torch.linspace(0.1, 0.9, C, device=DEV)
    g_out, g_alpha = _rand((B, C, H, W), 201), _rand((B, H, W), 202)
    ref_o, ref_a = nr.blend_soft_fragments(frag, col, sigma, gamma, NEAR, FAR, background=bg)
    ref_g = _grads(frag, col, sigma, gamma, bg.tolist(), g_out, g_alpha, False)
    N = B * H * W * K
    for off in (0, 1):                                       # colours, zbuf and every output 4 bytes off 16
        zb_buf, zb = _guarded(N, torch.float32, 0.0, off)
        zb.copy_(frag.zbuf.reshape(-1))
        cl_buf, cl = _guarded(N * C, torch.float32, 0.0, off)
        cl.copy_(col.reshape(-1))
        fr = nr.Fragments(frag.pix_to_face, zb, None, frag.dists)
        ob, o = _guarded(B * C * H * W, torch.float32, float("nan"), off)
        ab, al = _guarded(B * H * W, torch.float32, float("nan"), off)
        a = _abi(fr, col, sigma, gamma, bg)
        a.zbuf, a.colors, a.out, a.alpha = zb.data_ptr(), cl.data_ptr(), o.data_ptr(), al.data_ptr()
        assert lib.nr_b200_blend_fragments(ctypes.byref(a), _stream()) == 0
        torch.cuda.synchronize()
        assert torch.equal(o, ref_o.reshape(-1)) and torch.equal(al, ref_a.reshape(-1))
        for full in (ob, ab):
            assert torch.isnan(torch.cat((full[:16 + off], full[-16:]))).all()
        # the backward: every subset of wanted outputs, every NULL upstream gradient
        outs = [_guarded(N, torch.float32, float("nan"), off), _guarded(N, torch.float32, float("nan"), off),
                _guarded(N * C, torch.float32, float("nan"), off)]
        for want in range(1, 8):
            for ups in range(4):
                for full, _ in outs:
                    full.fill_(float("nan"))
                a.grad_out = g_out.data_ptr() if ups & 1 else None
                a.grad_alpha = g_alpha.data_ptr() if ups & 2 else None
                a.grad_zbuf, a.grad_dists, a.grad_colors = (v.data_ptr() if want & (1 << i) else None
                                                            for i, (_, v) in enumerate(outs))
                assert lib.nr_b200_blend_fragments_backward(ctypes.byref(a), _stream()) == 0
                torch.cuda.synchronize()
                if ups != 3:
                    wg = _grads(frag, col, sigma, gamma, bg.tolist(), g_out if ups & 1 else None,
                                g_alpha if ups & 2 else None, False) if ups else tuple(torch.zeros_like(r) for r in ref_g)
                else:
                    wg = ref_g
                for i, (full, v) in enumerate(outs):
                    if want & (1 << i):
                        assert torch.equal(v, wg[i].reshape(-1)), (off, want, ups, i)
                        assert torch.isnan(torch.cat((full[:16 + off], full[-16:]))).all()
                    else:
                        assert torch.isnan(full).all()        # not wanted: untouched
    # refusals launch nothing and write nothing
    ob, o = _guarded(B * C * H * W, torch.float32, float("nan"))
    ab, al = _guarded(B * H * W, torch.float32, float("nan"))
    for kw in (dict(faces_per_pixel=33), dict(sigma=0.0), dict(gamma=float("nan")), dict(near_=FAR),
               dict(zbuf=frag.zbuf.data_ptr() + 2), dict(pix_to_face=frag.pix_to_face.data_ptr() + 4)):
        a = _abi(frag, col, sigma, gamma)
        a.out, a.alpha = o.data_ptr(), al.data_ptr()
        for k, v in kw.items():
            setattr(a, k, v)
        assert lib.nr_b200_blend_fragments(ctypes.byref(a), _stream()) == INVALID, kw
        assert lib.nr_b200_last_launch_count() == 0
    a = _abi(frag, col, sigma, gamma)
    a.out, a.alpha = o.data_ptr(), al.data_ptr()
    assert lib.nr_b200_blend_fragments_backward(ctypes.byref(a), _stream()) == INVALID   # no gradient output
    torch.cuda.synchronize()
    assert torch.isnan(ob).all() and torch.isnan(ab).all()


# ------------------------------------------------------------------------------------------------ a fit, graphs
def test_light_direction_fit_through_a_torch_lambert_shader():
    from neural_renderer_b200 import synthetic
    nr = _nr()
    S, sigma, gamma, K = 96, 1e-4, 1e-4, 8
    faces = torch.from_numpy(synthetic.sphere_faces(1, 800)).to(DEV)
    v = faces[0].double()
    n = torch.linalg.cross(v[:, 1] - v[:, 0], v[:, 2] - v[:, 0])
    n = (n / n.norm(dim=-1, keepdim=True)).float()
    n = torch.where((n * (v.mean(1) - torch.tensor([0, 0, 2.75], device=DEV, dtype=torch.float64)).float()).sum(-1,
                    keepdim=True) < 0, -n, n)               # outward
    frag = nr.rasterize_soft_fragments(faces, S, sigma, K)
    albedo = torch.tensor([0.9, 0.6, 0.3], device=DEV)

    def render(light):
        d = light / light.norm()
        lit = 0.2 + 0.8 * torch.relu(-(n @ d))             # faces towards the light (the camera looks along +z)
        shade = (lit[:, None] * albedo).expand(1, -1, 3)
        col = shade[0][frag.pix_to_face.clamp_min(0)]       # [1,S,S,K,3]; empty slots are ignored by the blend
        return nr.blend_soft_fragments(frag, col, sigma, gamma, NEAR, FAR)[0]

    target = render(torch.tensor([0.4, -0.5, 0.75], device=DEV)).detach()
    light = torch.tensor([-0.5, 0.4, 0.8], device=DEV, requires_grad=True)
    opt = torch.optim.Adam([light], lr=0.02)
    sched = torch.optim.lr_scheduler.ExponentialLR(opt, 0.99)
    for _ in range(300):
        opt.zero_grad()
        ((render(light) - target) ** 2).sum().backward()
        opt.step()
        sched.step()
    got = light.detach() / light.detach().norm()
    want = torch.tensor([0.4, -0.5, 0.75], device=DEV)
    want = want / want.norm()
    assert torch.dot(got, want).item() > math.cos(math.radians(2.0)), got.tolist()


@pytest.mark.parametrize("K", [8, 32])  # K 32: tiles past 48 KB, so the capture sets the shared-memory attribute
def test_cuda_graph_capture_replays_bit_identically(K):
    nr = _nr()
    B, H, W, C, sigma, gamma = 2, 48, 50, 3, 1e-3, 1e-3
    frag, col = _synthetic(B, H, W, K, C, sigma, 300)
    zv = frag.zbuf.clone().requires_grad_(True)
    dv = frag.dists.clone().requires_grad_(True)
    cv = col.clone().requires_grad_(True)
    g_out, g_alpha = _rand((B, C, H, W), 301), _rand((B, H, W), 302)
    bg = torch.tensor([0.1, 0.2, 0.3], device=DEV)

    def step():
        out, alpha = nr.blend_soft_fragments(nr.Fragments(frag.pix_to_face, zv, None, dv), cv, sigma, gamma, NEAR, FAR,
                                             background=bg)
        grads = torch.autograd.grad((out, alpha), (zv, dv, cv), (g_out, g_alpha))
        return (out, alpha) + grads

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            eager = step()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        cap = step()
    graph.replay()
    torch.cuda.synchronize()
    for x, y in zip(eager, cap):
        assert torch.equal(x, y)
