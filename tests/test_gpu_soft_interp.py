"""GPU: the soft interpolation of fragments (interpolate_soft_fragments, nr_b200_interpolate_fragments[_backward])
against functional.interpolate_face_attributes in float64, and through the whole fragment pipeline.

The fragments are real (rasterize_soft_fragments of a triangle soup with empty slots, of the teapot and of the
benchmark spheres); the attributes and the vertex indices are random, since the interpolation reads only pix_to_face,
bary_coords, the attributes and the indices.  The float64 reference gathers per-vertex attributes through the indices
first (out-of-range indices as zero rows) and then calls interpolate_face_attributes.

Forward gate.  The inputs are fp32 and exact in float64.  The kernel rounds three times: p = l_0 a_0, q = fma(l_1, a_1,
p), out = fma(l_2, a_2, q); each rounding errs by at most u = 2^-24 of its result, and every partial result is bounded by
S = sum_m |l_m a_m| (1 + u)^2.  So |out - exact| <= 3 u (1 + u)^2 S.  The float64 reference itself errs by far less
than 1e-15 S.  The gate is 3.001 u S + 1e-15 S per element, and 0 where S = 0 (exact zeros).

Gradients are compared with float64 autograd element by element (helpers.elem_err).  No test peaks above 2.2 GiB of
device memory, as in the other soft test files."""
import ctypes

import pytest
import torch

import oracles_soft_blend as oblend
import oracles_soft_frag as ofrag
from helpers import elem_err, rel_err

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
NEAR, FAR = 0.1, 100.0
PEAK_LIMIT = int(2.2 * 2 ** 30)
INVALID = -1  # NR_ERR_INVALID_ARG
U = 2.0 ** -24


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


def _rand(shape, seed, lo=-1.0, hi=1.0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return lo + (hi - lo) * torch.rand(*shape, device=DEV, generator=g)


_SCENES = {}


def _scene(name, K):
    """(Fragments, F) of a real scene, cached per (scene, K)"""
    key = (name, K)
    if key not in _SCENES:
        from neural_renderer_b200 import synthetic
        nr = _nr()
        if name == "soup":               # 2 items, overlapping and off-screen faces, many empty slots
            faces = torch.from_numpy(synthetic.triangle_soup(2, 40, seed=3, size=(0.02, 0.4))).to(DEV)
            frag = nr.rasterize_soft_fragments(faces, 40, 1e-3, K)
        elif name == "teapot":           # the teapot, twice
            from test_gpu_soft_frag import _teapot
            v, f = _teapot()
            v = torch.cat((v, v + torch.tensor([0.05, -0.03, 0.0], device=DEV)), 0)
            faces = v[:, f[0].long()]
            frag = nr.rasterize_soft_fragments(faces.contiguous(), 48, 1e-4, K)
        else:                            # the benchmark spheres at 256 x 256
            faces = torch.from_numpy(synthetic.sphere_faces(2, 5000)).to(DEV)
            frag = nr.rasterize_soft_fragments(faces, 256, 1e-4, K)
        if len(_SCENES) > 8:
            _SCENES.clear()
        _SCENES[key] = (frag, faces.shape[1])
    return _SCENES[key]


def _attributes(form, B, F, C, seed, Nv=None):
    """(kwargs for interpolate_soft_fragments, the [B|1,F,3,C] corners they stand for).  form: (per_vertex,
    shared attributes, shared indices)"""
    pv, sa, si = form
    ab = 1 if sa else B
    if not pv:
        fa = _rand((ab, F, 3, C), seed)
        return dict(face_attributes=fa[0] if sa else fa), fa
    Nv = Nv or max(3, F // 2 + 1)
    va = _rand((ab, Nv, C), seed)
    ib = 1 if si else B
    g = torch.Generator(device=DEV).manual_seed(seed + 1)
    idx = torch.randint(0, Nv, (ib, F, 3), device=DEV, generator=g)
    corners = _gather(va, idx)
    return dict(vertex_attributes=va[0] if sa else va, faces=idx[0] if si else idx), corners


def _gather(va, idx):
    """the corners [B',F,3,C] of vertex attributes [1|B,Nv,C] through indices [1|B,F,3]; out-of-range indices give
    zero rows"""
    B = max(va.shape[0], idx.shape[0])
    va, idx = va.expand(B, -1, -1), idx.expand(B, -1, -1)
    Nv = va.shape[1]
    ok = (idx >= 0) & (idx < Nv)
    rows = torch.stack([va[b][idx[b].clamp(0, Nv - 1)] for b in range(B)])
    return torch.where(ok[..., None], rows, torch.zeros((), dtype=va.dtype, device=va.device))


def _reference(frag, corners):
    from neural_renderer_b200 import functional as Fn
    ca = corners.double()
    return Fn.interpolate_face_attributes(frag.pix_to_face, frag.bary_coords.double(), ca[0] if ca.shape[0] == 1 else ca)


def _check_forward(frag, corners, out):
    B, H, W, K = frag.pix_to_face.shape
    ref = _reference(frag, corners)
    ca = corners.double().abs().expand(B, -1, -1, -1)
    p2f = frag.pix_to_face
    valid = p2f >= 0
    ids = p2f.clamp_min(0)
    S = torch.zeros_like(ref)
    for m in range(3):
        am = torch.stack([ca[b, :, m][ids[b]] for b in range(B)])          # [B,H,W,K,C]
        S = S + frag.bary_coords[..., m:m + 1].double().abs() * am
    S = torch.where(valid[..., None], S, torch.zeros_like(S))
    gate = (3.001 * U + 1e-15) * S
    err = (out.double() - ref).abs()
    assert torch.all(err <= gate), (err - gate).max().item()
    assert torch.all(out[~valid] == 0)                                    # empty slots: exactly 0


def _same_sums(x, y):
    """two attribute gradients scattered from the same terms by fp32 atomics, whose order changes from run to run: each
    atomic rounds at u = 2^-24 of its running sum, so two orders differ by a few ulps of the largest running sums, which
    for an element that cancels can be many times its own size.  They are held per tensor at 1e-5 of the largest value
    (the attribute gradients' per-tensor gate of the ABI matrix), and must be finite"""
    assert x.shape == y.shape and torch.isfinite(x).all()
    assert rel_err(x.cpu(), y.cpu()) <= 1e-5, rel_err(x.cpu(), y.cpu())


FORMS = [(False, False, False), (False, True, False),                     # per corner, per item / shared
         (True, False, False), (True, False, True), (True, True, False), (True, True, True)]


# ------------------------------------------------------------------------------------------------ forward
@pytest.mark.parametrize("C", [1, 3, 4, 5, 16, 33])
@pytest.mark.parametrize("K", [1, 3, 8, 32])
def test_forward_against_float64(K, C):
    nr = _nr()
    for scene in ("soup", "teapot"):
        frag, F = _scene(scene, K)
        B = frag.pix_to_face.shape[0]
        if scene == "soup":
            assert (frag.pix_to_face < 0).any() and (frag.pix_to_face >= 0).any()
        for i, form in enumerate(FORMS):
            kw, corners = _attributes(form, B, F, C, 100 * K + 10 * C + i)
            out = nr.interpolate_soft_fragments(frag, **kw)
            assert out.shape == (*frag.pix_to_face.shape, C) and out.dtype == torch.float32
            _check_forward(frag, corners, out)


@pytest.mark.parametrize("KC", [(8, 3), (32, 4), (8, 16)])
def test_sphere_benchmark_geometry_at_256(KC):
    nr = _nr()
    K, C = KC
    frag, F = _scene("spheres", K)
    for i, form in enumerate((FORMS[0], FORMS[5])):
        kw, corners = _attributes(form, 2, F, C, 7 + i, Nv=2600)
        out = nr.interpolate_soft_fragments(frag, **kw)
        _check_forward(frag, corners, out)


# ------------------------------------------------------------------------------------------------ bit identities
def _run(frag, g_out, **kw):
    """(out, grad_bary, grad of the attribute tensor) of one call"""
    nr = _nr()
    by = frag.bary_coords.clone().requires_grad_(True)
    name = "face_attributes" if "face_attributes" in kw else "vertex_attributes"
    at = kw[name].clone().requires_grad_(True)
    out = nr.interpolate_soft_fragments(frag._replace(bary_coords=by), **{**kw, name: at})
    gb, ga = torch.autograd.grad(out, (by, at), g_out)
    return out.detach(), gb, ga


def test_bit_identities():
    frag, F = _scene("soup", 8)
    B = frag.pix_to_face.shape[0]
    C = 5
    g_out = _rand((*frag.pix_to_face.shape, C), 11)
    kw, corners = _attributes((True, False, False), B, F, C, 12)
    ref = _run(frag, g_out, **kw)
    rep = _run(frag, g_out, **kw)                                        # repeat: forward and grad_bary
    assert torch.equal(ref[0], rep[0]) and torch.equal(ref[1], rep[1])
    empty = frag.pix_to_face < 0
    assert torch.all(ref[0][empty] == 0) and torch.all(ref[1][empty] == 0)
    # per vertex against per corner on the materialised attributes, forward and grad_bary
    pc = _run(frag, g_out, face_attributes=corners)
    assert torch.equal(pc[0], ref[0]) and torch.equal(pc[1], ref[1])
    # channel c against a one-channel call on channel c
    for c in range(C):
        one = _run(frag, g_out[..., c:c + 1].contiguous(), vertex_attributes=kw["vertex_attributes"][..., c:c + 1],
                   faces=kw["faces"])
        assert torch.equal(one[0][..., 0], ref[0][..., c])
    # shared attributes and shared indices against the same sets expanded per item
    kws, cs = _attributes((True, True, True), B, F, C, 13)
    sh = _run(frag, g_out, **kws)
    ex = _run(frag, g_out, vertex_attributes=kws["vertex_attributes"].expand(B, -1, -1).contiguous(),
              faces=kws["faces"].expand(B, -1, -1).contiguous())
    assert torch.equal(sh[0], ex[0]) and torch.equal(sh[1], ex[1])
    _same_sums(sh[2], ex[2].sum(0))
    nr = _nr()
    base = kws["vertex_attributes"].clone().requires_grad_(True)         # an expanded stride-0 batch is shared
    st = nr.interpolate_soft_fragments(frag, vertex_attributes=base[None].expand(B, -1, -1), faces=kws["faces"])
    assert torch.equal(st, sh[0])
    (gst,) = torch.autograd.grad(st, base, g_out)
    _same_sums(gst, sh[2])
    fas = _run(frag, g_out, face_attributes=cs[0])
    fae = _run(frag, g_out, face_attributes=cs.expand(B, -1, -1, -1).contiguous())
    assert torch.equal(fas[0], fae[0]) and torch.equal(fas[1], fae[1])


def test_pix_to_face_past_F_is_an_empty_slot():
    frag, F = _scene("soup", 8)
    B = frag.pix_to_face.shape[0]
    C = 3
    g_out = _rand((*frag.pix_to_face.shape, C), 21)
    kw, _ = _attributes((False, False, False), B, F, C, 22)
    p2f = frag.pix_to_face.clone()
    valid = p2f >= 0
    pick = valid & (_rand(p2f.shape, 23, 0.0, 1.0) < 0.3)
    edited = torch.where(pick, p2f + F, p2f)                              # F, F + 1, ...: past the face range
    edited[0, 0, 0, 0] = F + (1 << 40)
    emptied = torch.where(pick, torch.full_like(p2f, -1), p2f)
    emptied[0, 0, 0, 0] = -1
    got = _run(frag._replace(pix_to_face=edited), g_out, **kw)
    want = _run(frag._replace(pix_to_face=emptied), g_out, **kw)
    assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])
    _same_sums(got[2], want[2])


def test_out_of_range_vertex_index_reads_zero_and_gets_no_gradient():
    frag, F = _scene("soup", 4)
    B = frag.pix_to_face.shape[0]
    C, Nv = 3, 30
    g_out = _rand((*frag.pix_to_face.shape, C), 31)
    va = _rand((B, Nv, C), 32)
    g = torch.Generator(device=DEV).manual_seed(33)
    idx = torch.randint(0, Nv, (B, F, 3), device=DEV, generator=g)
    idx[:, ::3, 1] = Nv + 4
    idx[:, 1::5, 2] = -2
    out, gb, ga = _run(frag, g_out, vertex_attributes=va, faces=idx)
    pc = _run(frag, g_out, face_attributes=_gather(va, idx))
    assert torch.equal(out, pc[0]) and torch.equal(gb, pc[1])
    # the gradient: the corners' gradient scattered back through the in-range indices only
    want = torch.zeros(B, Nv, C, device=DEV)
    ok = (idx >= 0) & (idx < Nv)
    for b in range(B):
        want[b].index_add_(0, idx[b][ok[b]], pc[2][b][ok[b]])
    _same_sums(ga, want)


# ------------------------------------------------------------------------------------------------ gradients
@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("KC", [(1, 3), (3, 5), (8, 5), (32, 33)])
def test_gradients_against_float64_autograd(KC, form):
    K, C = KC
    frag, F = _scene("soup", K)
    B = frag.pix_to_face.shape[0]
    kw, _ = _attributes(form, B, F, C, 40 + K)
    g_out = _rand((*frag.pix_to_face.shape, C), 41)
    out, gb, ga = _run(frag, g_out, **kw)
    # float64 autograd of the reference, through the gather for per-vertex attributes
    by = frag.bary_coords.double().requires_grad_(True)
    name = "face_attributes" if "face_attributes" in kw else "vertex_attributes"
    at = kw[name].double().requires_grad_(True)
    if form[0]:
        corners = _gather(at if at.dim() == 3 else at[None], kw["faces"] if kw["faces"].dim() == 3 else kw["faces"][None])
    else:
        corners = at if at.dim() == 4 else at[None]
    ref = _reference(frag._replace(bary_coords=by), corners)
    rb, ra = torch.autograd.grad(ref, (by, at), g_out.double())
    assert elem_err(gb.cpu(), rb.cpu(), floor=1e-3) <= 1e-4, elem_err(gb.cpu(), rb.cpu(), floor=1e-3)
    assert elem_err(ga.cpu(), ra.cpu(), floor=1e-3) <= 5e-4, elem_err(ga.cpu(), ra.cpu(), floor=1e-3)
    assert torch.all(gb[frag.pix_to_face < 0] == 0)


def _pipeline(faces, ca, S, sigma, gamma, K, interp, bg=(0.2, 0.5, 0.8)):
    nr = _nr()
    fv, cv = faces.clone().requires_grad_(True), ca.clone().requires_grad_(True)
    frag = nr.rasterize_soft_fragments(fv, S, sigma, K)
    img, alpha = nr.blend_soft_fragments(frag, interp(frag, cv), sigma, gamma, NEAR, FAR, background=bg)
    return fv, cv, frag, img, alpha


def test_whole_pipeline_against_the_torch_arm_and_float64():
    from neural_renderer_b200 import functional as Fn
    from test_gpu_soft_frag import _special_faces
    nr = _nr()
    S, sigma, gamma, K = 48, 1e-3, 1e-3, 8
    faces = _special_faces(2, sigma, 81)
    B, F = faces.shape[:2]
    ca = _rand((B, F, 3, 3), 82, 0.0, 1.0)
    up, ua = _rand((B, 3, S, S), 83), _rand((B, S, S), 84)
    arms = {"cuda": lambda fr, c: nr.interpolate_soft_fragments(fr, c),
            "torch": lambda fr, c: Fn.interpolate_face_attributes(fr.pix_to_face, fr.bary_coords, c)}
    res = {}
    for k, interp in arms.items():
        fv, cv, frag, img, alpha = _pipeline(faces, ca, S, sigma, gamma, K, interp)
        gf, gc = torch.autograd.grad((img, alpha), (fv, cv), (up, ua))
        res[k] = (img.detach(), gf, gc, frag)
    c, t = res["cuda"], res["torch"]
    assert torch.equal(c[3].pix_to_face, t[3].pix_to_face)
    assert (c[0] - t[0]).abs().max().item() <= 1e-5
    assert rel_err(c[1].cpu(), t[1].cpu()) <= 1e-4, rel_err(c[1].cpu(), t[1].cpu())
    assert rel_err(c[2].cpu(), t[2].cpu()) <= 1e-4, rel_err(c[2].cpu(), t[2].cpu())
    # float64: the fragments evaluated at the kernel's selection, interpolated and blended by the oracles
    frag = c[3]
    fv = faces.double().requires_grad_(True)
    cv = ca.double().requires_grad_(True)
    zb, by, ds = ofrag.evaluate(fv, frag.pix_to_face, S)
    col = _reference(frag._replace(bary_coords=by), cv)
    img, alpha = oblend.blend(frag.pix_to_face, zb, ds, col, sigma, gamma, NEAR, FAR, [0.2, 0.5, 0.8])
    rf, rc = torch.autograd.grad((img, alpha), (fv, cv), (up.double(), ua.double()))
    assert elem_err(c[1].cpu(), rf.cpu(), floor=1e-3) <= 2e-3, elem_err(c[1].cpu(), rf.cpu(), floor=1e-3)
    assert elem_err(c[2].cpu(), rc.cpu(), floor=1e-3) <= 2e-3, elem_err(c[2].cpu(), rc.cpu(), floor=1e-3)


# ------------------------------------------------------------------------------------------------ direct ABI
def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream(DEV).cuda_stream)


def _guarded(n, dtype, fill, offset=0, guard=16):
    buf = torch.full((n + 2 * guard + offset,), fill, dtype=dtype, device=DEV)
    return buf, buf[guard + offset:guard + offset + n]


@pytest.mark.parametrize("pv", [False, True])
@pytest.mark.parametrize("C", [3, 8])                   # C 8: 16-byte vectors where the addresses allow
def test_abi_poison_guards_misalignment_nulls_and_accumulate(C, pv):
    from neural_renderer_b200 import _lib
    lib = _lib.load()
    frag, F = _scene("soup", 8)
    B, H, W, K = frag.pix_to_face.shape
    Nv = 25
    form = (pv, False, True)
    kw, corners = _attributes(form, B, F, C, 90 + C)
    if pv:
        kw["faces"] = kw["faces"].clone()
        kw["faces"][::4, 0] = Nv + 100                                  # out of range: read 0, no gradient
        kw["faces"] = kw["faces"].int()
        va = _rand((B, Nv, C), 91)
        kw["vertex_attributes"] = va
        corners = _gather(va, kw["faces"].long()[None])
    attr = kw["vertex_attributes"] if pv else kw["face_attributes"]
    g_out = _rand((B, H, W, K, C), 92)
    ref_out, ref_gb, ref_ga = _run(frag, g_out, **kw)
    N = B * H * W * K
    flags = (_lib.NR_ATTR_PER_VERTEX | _lib.NR_INDICES_SHARED) if pv else 0
    for off in (0, 1):                                   # every float buffer 4 bytes off 16
        by_buf, by = _guarded(N * 3, torch.float32, 0.0, off)
        by.copy_(frag.bary_coords.reshape(-1))
        at_buf, at = _guarded(attr.numel(), torch.float32, 0.0, off)
        at.copy_(attr.reshape(-1))
        a = _lib.FragInterpArgs(struct_size=ctypes.sizeof(_lib.FragInterpArgs), flags=flags, batch_size=B, height=H,
                                width=W, faces_per_pixel=K, channels=C, num_faces=F, num_vertices=Nv if pv else 0)
        a.pix_to_face, a.bary, a.attributes = frag.pix_to_face.data_ptr(), by.data_ptr(), at.data_ptr()
        if pv:
            a.face_indices = kw["faces"].data_ptr()
        ob, o = _guarded(N * C, torch.float32, float("nan"), off)
        a.out = o.data_ptr()
        assert lib.nr_b200_interpolate_fragments(ctypes.byref(a), _stream()) == 0
        torch.cuda.synchronize()
        assert torch.equal(o, ref_out.reshape(-1))
        assert torch.isnan(torch.cat((ob[:16 + off], ob[-16:]))).all()
        # the backward: every subset of wanted outputs, with and without grad_out, with and without accumulation
        gbb, gb = _guarded(N * 3, torch.float32, float("nan"), off)
        gab, ga = _guarded(attr.numel(), torch.float32, float("nan"), off)
        gob, go = _guarded(N * C, torch.float32, 0.0, off)
        go.copy_(g_out.reshape(-1))
        for want in (1, 2, 3):
            for ups in (True, False):
                gbb.fill_(float("nan"))
                gab.fill_(float("nan"))
                a.out = None
                a.grad_out = go.data_ptr() if ups else None
                a.grad_bary = gb.data_ptr() if want & 1 else None
                a.grad_attributes = ga.data_ptr() if want & 2 else None
                assert lib.nr_b200_interpolate_fragments_backward(ctypes.byref(a), _stream()) == 0
                torch.cuda.synchronize()
                for bit, (full, v, r) in ((1, (gbb, gb, ref_gb)), (2, (gab, ga, ref_ga))):
                    if want & bit:
                        if ups:
                            if bit == 1:
                                assert torch.equal(v, r.reshape(-1)), (off, want)
                            else:
                                _same_sums(v, r.reshape(-1))
                        else:
                            assert torch.all(v == 0)                   # grad_out NULL = zeros
                        assert torch.isnan(torch.cat((full[:16 + off], full[-16:]))).all()
                    else:
                        assert torch.isnan(full).all()                  # not wanted: untouched
        # NR_GRAD_ACCUMULATE adds into a prefill
        gb.fill_(0.5)
        ga.fill_(-0.25)
        a.grad_out, a.grad_bary, a.grad_attributes = go.data_ptr(), gb.data_ptr(), ga.data_ptr()
        a.flags = flags | _lib.NR_GRAD_ACCUMULATE
        assert lib.nr_b200_interpolate_fragments_backward(ctypes.byref(a), _stream()) == 0
        torch.cuda.synchronize()
        assert torch.equal(gb, (0.5 + ref_gb).reshape(-1))
        _same_sums(ga, (ref_ga - 0.25).reshape(-1))
        a.flags = flags
    # refusals launch nothing and write nothing
    ob, o = _guarded(N * C, torch.float32, float("nan"))
    for kw2 in (dict(faces_per_pixel=33), dict(channels=0), dict(num_faces=0), dict(flags=1),
                dict(bary=frag.bary_coords.data_ptr() + 2), dict(pix_to_face=frag.pix_to_face.data_ptr() + 4)):
        a = _lib.FragInterpArgs(struct_size=ctypes.sizeof(_lib.FragInterpArgs), flags=flags, batch_size=B, height=H,
                                width=W, faces_per_pixel=K, channels=C, num_faces=F, num_vertices=Nv)
        a.pix_to_face, a.bary, a.attributes, a.out = (frag.pix_to_face.data_ptr(), frag.bary_coords.data_ptr(),
                                                      attr.data_ptr(), o.data_ptr())
        a.face_indices = kw["faces"].data_ptr() if pv else None
        for k, v in kw2.items():
            setattr(a, k, v)
        assert lib.nr_b200_interpolate_fragments(ctypes.byref(a), _stream()) == INVALID, kw2
        assert lib.nr_b200_last_launch_count() == 0
    torch.cuda.synchronize()
    assert torch.isnan(ob).all()


# ------------------------------------------------------------------------------------------------ a fit, graphs
def test_per_vertex_colour_fit_through_fragments_and_the_blend():
    from neural_renderer_b200 import synthetic
    import numpy as np
    nr = _nr()
    S, sigma, gamma, K = 64, 1e-4, 1e-4, 8
    v, f = synthetic.sphere_mesh(800)
    verts = torch.from_numpy((0.8 * v + np.array([0.0, 0.0, 2.75])).astype(np.float32)).to(DEV)[None]
    faces = torch.from_numpy(f.astype(np.int64)).to(DEV)
    frag = nr.rasterize_soft_fragments(faces.int(), S, sigma, K, vertices=verts)
    Nv = verts.shape[1]
    target_cols = _rand((1, Nv, 3), 95, 0.0, 1.0)

    def render(cols):
        return nr.blend_soft_fragments(frag, nr.interpolate_soft_fragments(frag, vertex_attributes=cols, faces=faces),
                                       sigma, gamma, NEAR, FAR)[0]

    target = render(target_cols).detach()
    cols = torch.full((1, Nv, 3), 0.5, device=DEV, requires_grad=True)
    opt = torch.optim.Adam([cols], lr=0.05)
    losses = []
    for _ in range(60):
        opt.zero_grad()
        loss = ((render(cols) - target) ** 2).sum()
        loss.backward()
        opt.step()
        losses.append(loss.item())
    assert losses[-1] < 0.1 * losses[0], (losses[0], losses[-1])


@pytest.mark.parametrize("pv", [False, True])
def test_cuda_graph_capture_replays_bit_identically(pv):
    nr = _nr()
    frag, F = _scene("soup", 8)
    B = frag.pix_to_face.shape[0]
    C = 4
    kw, _ = _attributes((pv, False, False), B, F, C, 97)
    name = "vertex_attributes" if pv else "face_attributes"
    at = kw[name].clone().requires_grad_(True)
    by = frag.bary_coords.clone().requires_grad_(True)
    g_out = _rand((*frag.pix_to_face.shape, C), 98)

    def step():
        out = nr.interpolate_soft_fragments(frag._replace(bary_coords=by), **{**kw, name: at})
        return (out,) + torch.autograd.grad(out, (by, at), g_out)

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
    assert torch.equal(eager[0], cap[0]) and torch.equal(eager[1], cap[1])
    _same_sums(cap[2], eager[2])
    first = [t.clone() for t in cap]
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(first[0], cap[0]) and torch.equal(first[1], cap[1])
