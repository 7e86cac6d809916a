"""GPU: attribute interpolation (rasterize_attributes, Renderer.render_attributes, nr_b200_interpolate[_backward]).

The forward is held to the float64 oracle of oracles_attr.py fed with the product's own maps, and bit for bit to smooth
shading's interpolated light; the backward to float64 autograd of the oracle, to the depth gradient K7 (interpolating the
camera depth is the depth image), and to central differences of the product's own forward."""
import ctypes

import numpy as np
import pytest
import torch

from helpers import elem_err, np_, rel_err
from oracles_attr import clamp_active, interp64

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda")


def _R():
    import importlib
    return importlib.import_module("neural_renderer_b200.rasterize")


def _randn(shape, seed, scale=1.0, shift=0.0):
    return (shift + scale * torch.randn(shape, generator=torch.Generator().manual_seed(seed))).to(DEV)


class Case:
    """B items of a seeded sphere: F faces, every corner its own vertex for the indexed form (so per-vertex attributes are
    a permutation away from per-corner ones); attributes per vertex / per corner, shared or per item"""

    def __init__(self, C, per_vertex, shared, indexed, aa, H=64, F=300, B=2, seed=3):
        from neural_renderer_b200 import synthetic
        self.C, self.per_vertex, self.shared, self.indexed, self.aa, self.H, self.B = C, per_vertex, shared, indexed, aa, H, B
        self.S = 2 * H if aa else H
        self.faces = torch.from_numpy(synthetic.sphere_faces(B, F, seed=seed)).to(DEV)
        self.F = F
        if indexed:
            # vertices in a permuted order, so that face_indices is not the identity
            perm = torch.randperm(3 * F, generator=torch.Generator().manual_seed(seed + 1)).to(DEV)
            self.perm = perm  # vertex j is corner perm[j] of the faces
            self.idx = torch.argsort(perm).to(torch.int32).reshape(F, 3)
            self.verts = self.faces.reshape(B, 3 * F, 3)[:, perm].contiguous()
        nb = 1 if shared else B
        if per_vertex:
            self.attrs = _randn((nb, 3 * F, C), seed + 2, 1.0, 2.0)
        else:
            self.attrs = _randn((nb, F, 3, C), seed + 2, 1.0, 2.0)

    def corner_attrs(self, attrs=None, B=None):
        attrs = self.attrs if attrs is None else attrs
        if not self.per_vertex:
            return attrs.expand(self.B, -1, -1, -1)
        return attrs.expand(self.B, -1, -1)[:, self.idx.long().reshape(-1)].reshape(self.B, self.F, 3, self.C)

    def render(self, attrs=None, geom=None, return_alpha=False):
        import neural_renderer_b200 as nr
        attrs = self.attrs if attrs is None else attrs
        kw = {"vertex_attributes": attrs} if self.per_vertex else {"face_attributes": attrs}
        if self.indexed:
            return nr.rasterize_attributes(self.idx, self.H, self.aa, vertices=self.verts if geom is None else geom,
                                           return_alpha=return_alpha, **kw)
        return nr.rasterize_attributes(self.faces if geom is None else geom, self.H, self.aa, return_alpha=return_alpha, **kw)

    def maps(self):
        _, _, _, fim, wmap = _R()._run(self.faces, None, self.S, False, 0.1, 100, 1e-4, None, False, True, False)
        return fim, wmap


# (C, per_vertex, shared, indexed, aa, H): every C, each layout / sharing / geometry form / anti-aliasing level several times
FWD_CASES = [
    (1, False, False, False, False, 64), (1, True, True, True, True, 64),
    (2, False, True, True, False, 64), (2, True, False, True, True, 64),
    (3, True, True, True, False, 64), (3, False, False, False, True, 64),
    (4, False, False, True, True, 64), (4, True, False, True, False, 64),
    (7, False, True, False, True, 64), (7, True, True, True, False, 257),
    (16, True, False, True, True, 64), (16, False, False, False, False, 257), (16, False, True, True, False, 1100),
    (64, False, False, True, False, 64), (64, True, True, True, True, 64),
]


@pytest.mark.parametrize("case", FWD_CASES)
def test_forward_vs_oracle(case):
    C, pv, shared, indexed, aa, H = case
    B = 1 if H > 257 else 2
    cs = Case(C, pv, shared, indexed, aa, H=H, B=B, F=2000 if H > 257 else 300)
    img = cs.render()
    fim, wmap = cs.maps()
    assert (fim >= 0).sum() > 500
    want = interp64(cs.faces, fim, cs.corner_attrs(), cs.S, aa, wmap=wmap)
    print("fwd", case, rel_err(np_(img), np_(want)))
    assert img.shape == (B, C, H, H)
    assert rel_err(np_(img), np_(want)) <= 1e-6
    uncovered = (fim < 0)
    if aa:
        uncovered = torch.nn.functional.avg_pool2d(uncovered[:, None].float(), 2, 2)[:, 0] == 1
    assert uncovered.any()
    assert (img.permute(1, 0, 2, 3)[:, uncovered] == 0).all()
    assert torch.equal(img, cs.render())  # deterministic


def test_forward_above_2048():
    cs = Case(3, True, True, True, False, H=2051, B=1, F=5000)
    img = cs.render()
    fim, wmap = cs.maps()
    want = interp64(cs.faces, fim, cs.corner_attrs(), cs.S, False, wmap=wmap)
    assert rel_err(np_(img), np_(want)) <= 1e-6


@pytest.mark.parametrize("aa", [False, True])
def test_corner_light_reproduces_smooth_shading_bit_for_bit(aa):
    """interpolating corner_light as a C = 3 corner attribute gives k_resolve's L_c: with a 1 x 1 image of ones the
    bilinear sample is exactly 1, so the smooth render's rgb is L_c itself (and its zp is the z-buffer's)"""
    import neural_renderer_b200 as nr
    cs = Case(3, False, False, False, aa)
    corner = _randn((cs.B, cs.F, 3, 3), 9, 0.3, 0.8)
    ones = torch.ones((1, 1, 3), device=DEV)
    uvs = torch.zeros((cs.F, 3, 2), device=DEV)
    rgb = nr.rasterize(cs.faces, ones, cs.H, aa, background_color=(0, 0, 0), face_uvs=uvs, corner_light=corner)
    img = nr.rasterize_attributes(cs.faces, cs.H, aa, face_attributes=corner)
    assert torch.equal(img, rgb)


@pytest.mark.parametrize("aa", [False, True])
def test_camera_depth_attribute_matches_depth_gradient_k7(aa):
    """the camera depth as a per-vertex attribute (a view of the vertices: the gradient flows through the weights and the
    attribute) is the depth image: same covered pixels, same grad_vertices as the depth gradient K7"""
    import neural_renderer_b200 as nr
    cs = Case(1, True, False, True, aa)
    g = _randn((cs.B, cs.H, cs.H), 4)
    v1 = cs.verts.clone().requires_grad_(True)
    depth = nr.rasterize_depth(cs.idx, cs.H, aa, vertices=v1)
    (depth * g).sum().backward()
    v2 = cs.verts.clone().requires_grad_(True)
    img = nr.rasterize_attributes(cs.idx, cs.H, aa, vertices=v2, vertex_attributes=v2[..., 2:3])
    (img[:, 0] * g).sum().backward()
    fim, wmap = cs.maps()
    v64 = cs.verts.double().requires_grad_(True)
    f64 = v64[:, cs.idx.long()]
    (interp64(f64, fim, f64[..., 2:3], cs.S, aa, wmap=wmap)[:, 0] * g.double()).sum().backward()
    cov = fim >= 0
    if aa:
        cov = torch.nn.functional.avg_pool2d(cov[:, None].float(), 2, 2)[:, 0] == 1
    e_cross, e_ours, e_k7 = (elem_err(np_(v2.grad), np_(v1.grad)), elem_err(np_(v2.grad), np_(v64.grad)),
                             elem_err(np_(v1.grad), np_(v64.grad)))
    print("k7", aa, rel_err(np_(img[:, 0][cov]), np_(depth[cov])), "cross", e_cross, "ours-f64", e_ours, "k7-f64", e_k7)
    assert rel_err(np_(img[:, 0][cov]), np_(depth[cov])) <= 1e-6
    assert v1.grad.abs().max() > 0
    # both are fp32: where K7 itself is further than 1e-4 from float64 (cancellation in its sum_k inv[3k] / z_k), the two
    # may differ by that much
    assert e_cross <= max(1e-4, e_k7)


GRAD_CASES = [c for c in FWD_CASES if c[5] == 64]


@pytest.mark.parametrize("case", GRAD_CASES)
def test_gradients_vs_oracle(case):
    C, pv, shared, indexed, aa, H = case
    cs = Case(C, pv, shared, indexed, aa)
    attrs = cs.attrs.clone().requires_grad_(True)
    geom = (cs.verts if indexed else cs.faces).clone().requires_grad_(True)
    img = cs.render(attrs=attrs, geom=geom)
    g = _randn(img.shape, 7)
    (img * g).sum().backward()
    fim, wmap = cs.maps()
    a64 = cs.attrs.double().requires_grad_(True)
    geom64 = (cs.verts if indexed else cs.faces).double().requires_grad_(True)
    faces64 = geom64[:, cs.idx.long()] if indexed else geom64
    want = interp64(faces64, fim, cs.corner_attrs(a64), cs.S, aa, wmap=wmap)
    (want * g.double()).sum().backward()
    ra = rel_err(np_(attrs.grad), np_(a64.grad))
    ea, eg = elem_err(np_(attrs.grad), np_(a64.grad)), elem_err(np_(geom.grad), np_(geom64.grad))
    print("grad", case, ra, ea, eg)
    assert a64.grad.abs().max() > 0 and geom64.grad.abs().max() > 0
    assert ra <= 1e-5
    # per element: sums of l_k g_c over a face's pixels with random-sign g; an element at elem_err's floor (1e-3 of the
    # largest) carries the fp32 rounding of partial sums of ordinary size, about 2e-5 of its own value
    assert ea <= 1e-4
    # the interior vertex gradient sits as far from float64 as the depth gradient K7 does on this geometry (the fp32
    # pixel-space vertices and K1 inverse both use; test_camera_depth_attribute_matches_depth_gradient_k7: 2.7e-4 and
    # 4.4e-4 on H100); per element this matrix measured 9e-5 to 1.9e-3
    assert rel_err(np_(geom.grad), np_(geom64.grad)) <= 1e-4
    assert eg <= 2.5e-3


def test_vertex_gradient_vs_central_difference():
    """a central difference of the product's own forward in single vertex coordinates, with the upstream gradient zeroed
    on every pixel whose winning face changes under the step"""
    import neural_renderer_b200 as nr
    cs = Case(4, True, False, True, False, H=96, F=200, B=1)
    g0 = _randn((1, 4, 96, 96), 5)
    v = cs.verts.clone().requires_grad_(True)
    (cs.render(geom=v) * g0).sum().backward()
    # vertices of faces at least 30 pixels large: on a sliver seen edge-on a step is comparable to the face's width
    f = cs.faces[0].double() * 48
    area = 0.5 * torch.cross(f[:, 1] - f[:, 0], f[:, 2] - f[:, 0], dim=-1)[:, 2].abs()
    ok = (area[cs.perm // 3] >= 30).repeat_interleave(3)
    picks = torch.argsort(v.grad.reshape(-1).abs() * ok, descending=True)[:6].tolist()
    h = 2e-4
    bad = []
    for i in picks:
        vs = {}
        for s in (1, -1):
            vv = cs.verts.clone().reshape(-1)
            vv[i] += s * h
            vs[s] = vv.reshape(cs.verts.shape)
        fims = [_R()._run(cs.idx, None, 96, False, 0.1, 100, 1e-4, None, False, True, False, vertices=x)[3]
                for x in (cs.verts, vs[1], vs[-1])]
        same = (fims[0] == fims[1]) & (fims[0] == fims[2])
        for x, fm in zip((cs.verts, vs[1], vs[-1]), fims):  # the derivative holds the weights' clamp fixed
            same &= ~clamp_active(x[:, cs.idx.long()], fm, 96)
        g = g0 * same[:, None]
        vg = cs.verts.clone().requires_grad_(True)
        (cs.render(geom=vg) * g).sum().backward()
        with torch.no_grad():
            fd = float(((cs.render(geom=vs[1]).double() - cs.render(geom=vs[-1]).double()) * g.double()).sum() / (2 * h))
        an = float(vg.grad.reshape(-1)[i])
        fim, wmap = cs.maps()
        v64 = cs.verts.double().requires_grad_(True)
        (interp64(v64[:, cs.idx.long()], fim, cs.corner_attrs().double(), cs.S, False, wmap=wmap) * g.double()).sum().backward()
        print("fd", i, fd, an, "f64", float(v64.grad.reshape(-1)[i]))
        bad.append((i, fd, an)) if abs(fd - an) > 1e-2 * abs(an) + 1e-6 else None
    assert not bad, bad



# ----------------------------------------------------------------------------------------------------- direct C ABI
@pytest.mark.parametrize("indexed,pv,offset", [(False, False, 0), (True, True, 4), (True, False, 8)])
@pytest.mark.parametrize("mode", ["fresh", "accumulate"])
def test_abi_poisoned_offset_buffers_nulls_and_accumulate(indexed, pv, offset, mode):
    from abi_harness import alloc, guards_intact, poison
    from neural_renderer_b200 import _lib
    lib = _lib.load()
    cs = Case(5, pv, False, indexed, True, H=32, F=120)
    fim, wmap = cs.maps()
    s = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    B, S, C, H = cs.B, cs.S, cs.C, cs.H
    geom = cs.verts if indexed else cs.faces
    buf = {}
    for name, t in (("geom", geom), ("attr", cs.attrs), ("fim", fim), ("wmap", wmap)):
        buf[name] = alloc(tuple(t.shape), np.int32 if t.dtype == torch.int32 else np.float32, offset, DEV)
        buf[name].copy_(t)
    if indexed:
        buf["idx"] = alloc(tuple(cs.idx.shape), np.int32, offset, DEV)
        buf["idx"].copy_(cs.idx)
    buf["out"] = alloc((B, C, H, H), np.float32, offset, DEV)
    poison(buf["out"])

    def args():
        a = _lib.InterpolateArgs()
        a.struct_size = ctypes.sizeof(_lib.InterpolateArgs)
        a.flags = _lib.NR_ANTI_ALIASING | (_lib.NR_FACES_INDEXED | _lib.NR_INDICES_SHARED if indexed else 0) | \
            (_lib.NR_ATTR_PER_VERTEX if pv else 0)
        a.batch_size, a.num_faces, a.raster_size, a.channels = B, cs.F, S, C
        if indexed:
            a.vertices, a.face_indices, a.num_vertices = buf["geom"].data_ptr(), buf["idx"].data_ptr(), geom.shape[1]
        else:
            a.faces = buf["geom"].data_ptr()
        a.face_index_map, a.weight_map, a.attributes = buf["fim"].data_ptr(), buf["wmap"].data_ptr(), buf["attr"].data_ptr()
        return a
    a = args()
    a.out = buf["out"].data_ptr()
    assert lib.nr_b200_interpolate(ctypes.byref(a), s) == 0
    torch.cuda.synchronize()
    assert torch.equal(buf["out"], cs.render())
    # the autograd path's gradients, then the same through the ABI
    attrs = cs.attrs.clone().requires_grad_(True)
    gv = geom.clone().requires_grad_(True)
    img = cs.render(attrs=attrs, geom=gv)
    g = _randn(img.shape, 8)
    (img * g).sum().backward()
    buf["g"] = alloc(tuple(g.shape), np.float32, offset, DEV)
    buf["g"].copy_(g)
    buf["ga"] = alloc(tuple(cs.attrs.shape), np.float32, offset, DEV)
    buf["gv"] = alloc(tuple(geom.shape), np.float32, offset, DEV)
    pre_a, pre_v = _randn(cs.attrs.shape, 10), _randn(geom.shape, 11)
    for k in ("ga", "gv"):
        poison(buf[k])
    if mode == "accumulate":
        buf["ga"].copy_(pre_a)
        buf["gv"].copy_(pre_v)
    b = args()
    b.flags |= _lib.NR_GRAD_ACCUMULATE if mode == "accumulate" else 0
    b.grad_out, b.grad_attributes = buf["g"].data_ptr(), buf["ga"].data_ptr()
    if indexed:
        b.grad_vertices = buf["gv"].data_ptr()
    else:
        b.grad_faces = buf["gv"].data_ptr()
    assert lib.nr_b200_interpolate_backward(ctypes.byref(b), s) == 0
    torch.cuda.synchronize()
    base_a, base_v = (pre_a, pre_v) if mode == "accumulate" else (0, 0)
    assert rel_err(np_(buf["ga"]), np_(attrs.grad + base_a)) <= 1e-5
    assert rel_err(np_(buf["gv"]), np_(gv.grad + base_v)) <= 1e-5
    # every NULL the header allows: either gradient output alone, and no upstream gradient (zeros)
    for k in ("ga", "gv"):
        poison(buf[k])
    b.flags &= ~_lib.NR_GRAD_ACCUMULATE
    b.grad_vertices = b.grad_faces = None
    assert lib.nr_b200_interpolate_backward(ctypes.byref(b), s) == 0
    torch.cuda.synchronize()
    assert rel_err(np_(buf["ga"]), np_(attrs.grad)) <= 1e-5 and torch.isnan(buf["gv"]).all()
    b.grad_attributes = None
    if indexed:
        b.grad_vertices = buf["gv"].data_ptr()
    else:
        b.grad_faces = buf["gv"].data_ptr()
    assert lib.nr_b200_interpolate_backward(ctypes.byref(b), s) == 0
    torch.cuda.synchronize()
    assert rel_err(np_(buf["gv"]), np_(gv.grad)) <= 1e-5
    b.grad_out = None
    b.grad_attributes = buf["ga"].data_ptr()
    assert lib.nr_b200_interpolate_backward(ctypes.byref(b), s) == 0
    b.grad_attributes = b.grad_vertices = b.grad_faces = None
    assert lib.nr_b200_interpolate_backward(ctypes.byref(b), s) == 0
    torch.cuda.synchronize()
    assert (buf["ga"] == 0).all() and (buf["gv"] == 0).all()
    assert all(guards_intact(t) for t in buf.values())


# ------------------------------------------------------------------------------------------------------- Renderer
def _renderer(fill_back, fused):
    import neural_renderer_b200 as nr
    r = nr.Renderer()
    r.image_size = 64
    r.fill_back = fill_back
    r.fused = fused
    r.eye = (0.3, 0.5, -2.4)
    return r


def _teapot(B=2):
    import os
    d = np.load(os.path.join(os.path.dirname(__file__), "golden", "teapot.npz"))
    v = torch.from_numpy(d["vertices"].astype(np.float32)).to(DEV)
    f = torch.from_numpy(d["faces"].astype(np.int32)).to(DEV)
    verts = (v[None] * 0.9 + 0.01 * _randn((B,) + tuple(v.shape), 0)).contiguous()
    return verts, f[None].expand(B, -1, -1)


@pytest.mark.parametrize("form", ["vertex", "vertex_shared", "face"])
@pytest.mark.parametrize("fill_back", [False, True])
def test_renderer_fused_matches_op_by_op(form, fill_back):
    verts0, faces = _teapot()
    B, Nv, F = verts0.shape[0], verts0.shape[1], faces.shape[1]
    if form == "vertex":
        a0 = _randn((B, Nv, 6), 1)
    elif form == "vertex_shared":
        a0 = _randn((Nv, 6), 1)
    else:
        a0 = _randn((F, 3, 6), 1)
    out = []
    for fused in (True, False):
        v = verts0.clone().requires_grad_(True)
        a = a0.clone().requires_grad_(True)
        kw = {"face_attributes": a} if form == "face" else {"vertex_attributes": a}
        img = _renderer(fill_back, fused).render_attributes(v, faces, **kw)
        g = _randn(img.shape, 3)
        (img * g).sum().backward()
        out.append((img.detach(), a.grad, v.grad))
    (i0, a0g, v0), (i1, a1g, v1) = out
    print("fused vs op", form, fill_back, rel_err(np_(i0), np_(i1)), rel_err(np_(a0g), np_(a1g)), rel_err(np_(v0), np_(v1)))
    assert (i0 != 0).any()
    assert rel_err(np_(i0), np_(i1)) <= 1e-6
    assert rel_err(np_(a0g), np_(a1g)) <= 1e-5
    assert rel_err(np_(v0), np_(v1)) <= 1e-5


def test_renderer_shared_vertex_attributes_receive_the_sum_over_items():
    verts, faces = _teapot(B=3)
    a = _randn((verts.shape[1], 3), 2).requires_grad_(True)
    r = _renderer(True, True)
    img = r.render_attributes(verts, faces, vertex_attributes=a)
    g = _randn(img.shape, 4)
    (img * g).sum().backward()
    per = torch.zeros_like(a)
    for b in range(3):
        ab = a.detach().clone().requires_grad_(True)
        (r.render_attributes(verts[b:b + 1], faces[b:b + 1], vertex_attributes=ab) * g[b:b + 1]).sum().backward()
        per += ab.grad
    assert rel_err(np_(a.grad), np_(per)) <= 1e-5


def test_renderer_step_in_cuda_graph():
    from neural_renderer_b200 import functional as F
    verts0, faces = _teapot()
    r = _renderer(True, True)
    v = verts0.clone().requires_grad_(True)
    g = _randn((2, 3, 64, 64), 3)

    def loss():
        return (r.render_attributes(v, faces, vertex_attributes=F.vertex_normals(v, faces)) * g).sum()

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            v.grad = None
            loss().backward()
    torch.cuda.current_stream().wait_stream(s)
    v.grad = None
    loss().backward()
    eager = v.grad.clone()
    graph = torch.cuda.CUDAGraph()
    v.grad = None
    with torch.cuda.graph(graph):
        loss().backward()
    graph.replay()
    torch.cuda.synchronize()
    assert rel_err(np_(v.grad), np_(eager)) <= 1e-5


def test_attribute_loss_alone_fits_vertices_without_silhouette():
    """a grid that covers the whole view (no silhouette edge anywhere) carries fixed per-vertex UVs; its target image is
    rendered from displaced vertices.  Only the interior gradient through the interpolation weights can move the
    vertices back, and Adam on the attribute loss alone cuts the vertex error at least tenfold"""
    import neural_renderer_b200 as nr
    n = 15
    t = torch.linspace(-1.4, 1.4, n, device=DEV)
    yy, xx = torch.meshgrid(t, t, indexing="ij")
    xy0 = torch.stack((xx, yy), dim=-1).reshape(-1, 2)
    quads = [(i * n + j, i * n + j + 1, (i + 1) * n + j + 1, (i + 1) * n + j) for i in range(n - 1) for j in range(n - 1)]
    faces = torch.tensor([[a, b, c] for a, b, c, d in quads] + [[a, c, d] for a, b, c, d in quads], dtype=torch.int32,
                         device=DEV)
    uv = (xy0 + 1.4) / 2.8
    disp = 0.04 * torch.stack((torch.sin(2.0 * xy0[:, 1] + 0.3), torch.cos(1.7 * xy0[:, 0])), dim=-1)
    inner = (xy0.abs() < 0.85).all(dim=-1)
    z = torch.full((xy0.shape[0], 1), 2.0, device=DEV)

    def image(xy):
        verts = torch.cat((xy, z), dim=-1)[None]
        return nr.rasterize_attributes(faces, 128, False, vertices=verts, vertex_attributes=uv)

    with torch.no_grad():
        target = image(xy0 + disp)
    assert (nr.rasterize_silhouettes(faces, 128, False, vertices=torch.cat((xy0, z), -1)[None]) == 1).all()
    xy = xy0.clone().requires_grad_(True)
    opt = torch.optim.Adam([xy], lr=2e-3)
    sched = torch.optim.lr_scheduler.StepLR(opt, 100, 0.3)
    err0 = float((xy0 - (xy0 + disp))[inner].norm(dim=-1).mean())
    for _ in range(300):
        opt.zero_grad()
        ((image(xy) - target) ** 2).sum().backward()
        opt.step()
        sched.step()
    err = float((xy.detach() - (xy0 + disp))[inner].norm(dim=-1).mean())
    print("fit", err0, err)
    assert err <= 0.1 * err0
