"""GPU: smooth (Gouraud) shading -- corner_light interpolated at every pixel (include/nr_b200.h), the vertex-normal and
corner-light glue kernels, and Renderer.shading = 'smooth'.

The forward is held to a float64 oracle: the light interpolated with float64 perspective weights
(oracles_smooth.smooth_light64) times the unlit sample, which is the float64 sampler of oracles.py for texture images and the product's own unlit render
for cubes (bit-exact to the reference elsewhere).  Because the image is L * s(textures, uv), the texture and UV gradients
of a smooth render with upstream g equal those of the unlit render with upstream g * L: that, the float64 samplers through
autograd, and a central difference of the product's own forward in corner_light hold the backward."""
import ctypes
import os

import numpy as np
import pytest
import torch

from helpers import elem_err, np_, rel_err
from oracles import oracle_rgb, oracle_trilinear
from oracles_smooth import smooth_light64, smooth_rgb
from oracles_uv_grad import oracle_rgb_uv_grad, oracle_trilinear_uv_grad

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda")
BG = (0.1, 0.2, 0.3)


def _R():
    import importlib
    return importlib.import_module("neural_renderer_b200.rasterize")


def _rand(shape, lo=0.0, hi=1.0, seed=1):
    g = torch.Generator().manual_seed(seed)
    return (lo + (hi - lo) * torch.rand(shape, generator=g, dtype=torch.float32)).to(DEV)


def _faces(B, F, seed):
    from neural_renderer_b200 import synthetic
    return torch.from_numpy(synthetic.sphere_faces(B, F, seed=seed)).to(DEV)


def _upsample(g, aa):
    """API-layout upstream gradient -> the raster gradient the backward sees (pooling: each raster pixel gets g / 4)"""
    return g.repeat_interleave(2, -1).repeat_interleave(2, -2) * 0.25 if aa else g


class Scene:
    """B items, F front faces (+ reversed copies with fill_back), textures of one kind, a random corner_light"""

    def __init__(self, kind, aa, fill_back, indexed, H=64, F=300, B=2, seed=3):
        self.kind, self.aa, self.fill_back, self.indexed = kind, aa, fill_back, indexed
        self.B, self.H = B, H
        self.S = 2 * H if aa else H
        faces = _faces(B, F, seed)
        if fill_back:
            faces = torch.cat((faces, faces.flip(2)), dim=1)
        self.faces = faces
        self.F = faces.shape[1]
        if kind.startswith("cube"):
            ts = int(kind[4:])
            self.tex = _rand((B, F, ts, ts, ts, 3), 0.2, 1.0, seed=5)
            self.uvs, self.tf = None, "bilinear"
        else:
            self.tex = _rand((B, 37, 29, 3), 0.2, 1.0, seed=5)
            self.uvs = _rand((B, F, 3, 2), seed=4)
            self.tf = "trilinear" if kind == "trilinear" else "bilinear"
        self.corner = _rand((B, self.F, 3, 3), 0.3, 1.2, seed=6)

    def render(self, corner=None, tex=None, uvs=None, face_light=None, aa=None, H=None, bg=BG, return_all=True):
        aa = self.aa if aa is None else aa
        H = self.H if H is None else H
        geom, verts = self.faces, None
        if self.indexed:  # every corner its own vertex: the indexed path with the same geometry
            verts = self.faces.reshape(self.B, -1, 3)
            geom = torch.arange(verts.shape[1], device=DEV, dtype=torch.int32).reshape(-1, 3)
        tex = self.tex if tex is None else tex
        uvs = self.uvs if uvs is None else uvs
        return _R()._run(geom, tex, H, aa, 0.1, 100, 1e-4, bg, True, return_all, return_all, face_light=face_light,
                         textures_fill_back=self.fill_back, vertices=verts,
                         face_uvs=uvs, texture_filter=self.tf, corner_light=corner)

    def maps(self):
        _, _, _, fim, wmap = self.render(aa=False, H=self.S)
        dmap = _R()._run(self.faces, None, self.S, False, 0.1, 100, 1e-4, None, False, False, True)[2]
        return fim, wmap, dmap

    def unlit64(self, fim, wmap, dmap, tex=None, uvs=None, uv_grad=False):
        """float64 (images) / product (cubes) unlit raster sample [B,3,S,S], background 0"""
        tex = self.tex if tex is None else tex
        if self.kind.startswith("cube"):
            return self.render(aa=False, H=self.S, bg=(0, 0, 0))[0].double()
        uvs = self.uvs if uvs is None else uvs
        args = (self.faces, fim, wmap, dmap, uvs, tex, None, (0, 0, 0), self.fill_back, False)
        if uv_grad:
            return (oracle_trilinear_uv_grad if self.tf == "trilinear" else oracle_rgb_uv_grad)(*args)
        return oracle_trilinear(*args)[0] if self.tf == "trilinear" else oracle_rgb(*args)


FWD_CASES = [(k, aa, fb, ix) for k in ("cube2", "cube4", "bilinear", "trilinear") for aa in (False, True)
             for fb in (False, True) for ix in (False, True) if (aa, fb, ix) in ((False, False, False), (True, True, False),
                                                                               (True, False, True), (False, True, True))]


def _fwd_tol(kind):
    # the trilinear oracle evaluates the level of detail in float64 (test_gpu_abi_matrix.py: its image gate is 6e-5)
    return 6e-5 if kind == "trilinear" else 2e-6


@pytest.mark.parametrize("case", FWD_CASES)
def test_forward_vs_oracle(case):
    kind, aa, fill_back, indexed = case
    sc = Scene(kind, aa, fill_back, indexed)
    rgb = sc.render(corner=sc.corner)[0]
    fim, wmap, dmap = sc.maps()
    assert (fim >= 0).sum() > 500
    want = smooth_rgb(sc.unlit64(fim, wmap, dmap), smooth_light64(sc.faces, fim, wmap, dmap, sc.corner), fim, BG, aa)
    print("smooth fwd", case, rel_err(np_(rgb), np_(want)))
    assert rel_err(np_(rgb), np_(want)) <= _fwd_tol(kind)


@pytest.mark.parametrize("kind,H", [("cube4", 257), ("bilinear", 257), ("cube2", 1100), ("bilinear", 1100)])
def test_forward_vs_oracle_large_and_odd_rasters(kind, H):
    sc = Scene(kind, False, False, False, H=H, F=2000, B=1)
    rgb = sc.render(corner=sc.corner)[0]
    fim, wmap, dmap = sc.maps()
    want = smooth_rgb(sc.unlit64(fim, wmap, dmap), smooth_light64(sc.faces, fim, wmap, dmap, sc.corner), fim, BG, False)
    assert rel_err(np_(rgb), np_(want)) <= 2e-6


@pytest.mark.parametrize("kind", ["cube2", "cube4", "bilinear", "trilinear"])
@pytest.mark.parametrize("aa", [False, True])
def test_equal_corners_match_face_light(kind, aa):
    """all three corners of a face at its face_light: the bit-exact flat path within 1e-6"""
    sc = Scene(kind, aa, kind == "cube4", False)
    light = _rand((sc.B, sc.F, 3), 0.3, 1.2, seed=8)
    flat = sc.render(face_light=light)[0]
    smooth = sc.render(corner=light[:, :, None, :].expand(-1, -1, 3, -1).contiguous())[0]
    assert rel_err(np_(smooth), np_(flat)) <= 1e-6


GRAD_CASES = [("cube2", False, False), ("cube4", True, True), ("bilinear", False, True), ("bilinear", True, False),
              ("trilinear", False, False), ("trilinear", True, True)]


@pytest.mark.parametrize("case", GRAD_CASES)
def test_gradients_vs_oracle(case):
    kind, aa, fill_back = case
    sc = Scene(kind, aa, fill_back, False)
    corner = sc.corner.clone().requires_grad_(True)
    tex = sc.tex.clone().requires_grad_(True)
    uvs = sc.uvs.clone().requires_grad_(True) if sc.uvs is not None else None
    rgb = sc.render(corner=corner, tex=tex, uvs=uvs)[0]
    g = torch.randn(rgb.shape, generator=torch.Generator().manual_seed(7)).to(DEV)
    (rgb * g).sum().backward()
    fim, wmap, dmap = sc.maps()
    c64 = sc.corner.double().requires_grad_(True)
    L64 = smooth_light64(sc.faces, fim, wmap, dmap, c64)
    if kind.startswith("cube"):
        # d / d corner_light in float64 from the product's unlit sample; d / d textures = the unlit backward with g * L
        want = smooth_rgb(sc.unlit64(fim, wmap, dmap), L64, fim, BG, aa)
        (want * g.double()).sum().backward()
        tex_u = sc.tex.clone().requires_grad_(True)
        unlit = sc.render(tex=tex_u, aa=False, H=sc.S)[0]
        G = _upsample(g, aa) * L64.detach().float().permute(0, 3, 1, 2)
        (unlit * G).sum().backward()
        tex_want, tex_tol = tex_u.grad, 1e-4
    else:
        tex64 = sc.tex.double().requires_grad_(True)
        uv64 = sc.uvs.double().requires_grad_(True)
        want = smooth_rgb(sc.unlit64(fim, wmap, dmap, tex=tex64, uvs=uv64, uv_grad=True), L64, fim, BG, aa)
        (want * g.double()).sum().backward()
        tex_want = tex64.grad
        tex_tol = 5e-4 if kind == "trilinear" else 1e-4  # test_gpu_abi_matrix.py's pyramid gate
        uv_tol = 1.5e-3 if kind == "trilinear" else 1e-4  # test_gpu_uv_grad.py's gates
        print("uv", case, rel_err(np_(uvs.grad), np_(uv64.grad)), elem_err(np_(uvs.grad), np_(uv64.grad)))
        assert rel_err(np_(uvs.grad), np_(uv64.grad)) <= 1e-4
        assert elem_err(np_(uvs.grad), np_(uv64.grad)) <= uv_tol
    print("corner", case, rel_err(np_(corner.grad), np_(c64.grad)), elem_err(np_(corner.grad), np_(c64.grad)))
    print("tex", case, rel_err(np_(tex.grad), np_(tex_want)), elem_err(np_(tex.grad), np_(tex_want)))
    assert c64.grad.abs().max() > 0
    assert rel_err(np_(corner.grad), np_(c64.grad)) <= 1e-4
    assert elem_err(np_(corner.grad), np_(c64.grad)) <= (5e-4 if kind == "trilinear" else 1e-4)
    assert rel_err(np_(tex.grad), np_(tex_want)) <= 1e-4
    assert elem_err(np_(tex.grad), np_(tex_want)) <= tex_tol


@pytest.mark.parametrize("kind", ["cube4", "bilinear", "trilinear"])
def test_corner_light_gradient_vs_central_difference(kind):
    """the image is linear in corner_light: a central difference of the product's own forward is exact up to fp32"""
    sc = Scene(kind, True, False, False, H=32, F=60, B=1)
    corner = sc.corner.clone().requires_grad_(True)
    rgb = sc.render(corner=corner)[0]
    g = torch.randn(rgb.shape, generator=torch.Generator().manual_seed(9)).to(DEV)
    (rgb * g).sum().backward()
    grad = corner.grad.reshape(-1)
    picks = torch.argsort(grad.abs(), descending=True)[:12].tolist()
    h = 0.05
    with torch.no_grad():
        for i in picks:
            cp, cm = sc.corner.clone().reshape(-1), sc.corner.clone().reshape(-1)
            cp[i] += h
            cm[i] -= h
            fp = (sc.render(corner=cp.reshape(sc.corner.shape))[0].double() * g.double()).sum()
            fm = (sc.render(corner=cm.reshape(sc.corner.shape))[0].double() * g.double()).sum()
            fd = float((fp - fm) / (2 * h))
            assert abs(fd - float(grad[i])) <= 1e-3 * abs(float(grad[i])) + 1e-5, (i, fd, float(grad[i]))


# ------------------------------------------------------------------------------------------------- glue kernels
def _mesh(B=2, shared=True, seed=0):
    d = np.load(os.path.join(os.path.dirname(__file__), "golden", "teapot.npz"))
    v = torch.from_numpy(d["vertices"].astype(np.float32)).to(DEV)
    f = torch.from_numpy(d["faces"].astype(np.int32)).to(DEV)
    g = torch.Generator().manual_seed(seed)
    verts = (v[None] + 0.01 * torch.randn((B,) + tuple(v.shape), generator=g).to(DEV)).contiguous()
    if shared:
        return verts, f
    perm = torch.stack([torch.randperm(f.shape[0], generator=g) for _ in range(B)]).to(DEV)
    return verts, f[perm].contiguous()


LIGHT = (0.4, 0.6, (1.0, 0.9, 0.8), (0.7, 0.8, 1.0), (0.3, 0.8, -0.5))


@pytest.mark.parametrize("shared", [True, False])
def test_glue_kernels_vs_float64(shared):
    from neural_renderer_b200 import functional as F
    verts, faces = _mesh(shared=shared)
    v = verts.clone().requires_grad_(True)
    n = F.vertex_normals(v, faces)
    n2 = F.vertex_normals(verts, faces)
    assert torch.equal(n, n2)  # deterministic
    v64 = verts.double().requires_grad_(True)
    n64 = F._vertex_normals_torch(v64, faces.cpu().to(DEV))
    assert rel_err(np_(n), np_(n64)) <= 2e-6
    fb = torch.cat((faces, faces.flip(-1)), dim=-2)
    for fill_back, idx in ((False, faces), (True, fb)):
        cl = F.corner_light(n, idx, *LIGHT, fill_back=fill_back)
        cl64 = F._corner_light_torch(n64, idx, *LIGHT, fill_back=fill_back)
        assert rel_err(np_(cl), np_(cl64)) <= 2e-6
    g = torch.randn(cl.shape, generator=torch.Generator().manual_seed(1)).to(DEV)
    (cl * g).sum().backward()
    (cl64 * g.double()).sum().backward()
    print("glue grad", shared, rel_err(np_(v.grad), np_(v64.grad)))
    assert rel_err(np_(v.grad), np_(v64.grad)) <= 1e-4


def test_vertex_normals_abi_accumulate_and_out_of_range():
    from neural_renderer_b200 import _lib
    lib = _lib.load()
    verts, faces = _mesh(B=2)
    faces = faces.clone()
    faces[5, 1] = 10 ** 6  # skipped: that face contributes nothing
    faces[7, 0] = -3
    B, Nv, Nf = verts.shape[0], verts.shape[1], faces.shape[0]
    flags = _lib.NR_INDICES_SHARED
    nbytes = lib.nr_b200_vertex_normals_workspace_bytes(B, Nv, Nf, flags)
    assert nbytes > 0
    ws = torch.empty((nbytes,), dtype=torch.uint8, device=DEV)
    out = torch.full_like(verts, float("nan"))
    s = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    assert lib.nr_b200_vertex_normals(verts.data_ptr(), faces.data_ptr(), B, Nv, Nf, flags, out.data_ptr(), ws.data_ptr(),
                                      nbytes, s) == 0
    from neural_renderer_b200 import functional as F
    assert rel_err(np_(out), np_(F._vertex_normals_torch(verts.double(), faces))) <= 2e-6
    assert lib.nr_b200_vertex_normals(verts.data_ptr(), faces.data_ptr(), B, Nv, Nf, flags, out.data_ptr(), ws.data_ptr(),
                                      nbytes - 1, s) == _lib.NR_OK - 2
    gn = torch.randn(verts.shape, generator=torch.Generator().manual_seed(2)).to(DEV)
    fresh = torch.full_like(verts, float("nan"))
    assert lib.nr_b200_vertex_normals_backward(verts.data_ptr(), faces.data_ptr(), gn.data_ptr(), B, Nv, Nf, flags,
                                               fresh.data_ptr(), ws.data_ptr(), nbytes, s) == 0
    pre = torch.randn(verts.shape, generator=torch.Generator().manual_seed(3)).to(DEV)
    acc = pre.clone()
    assert lib.nr_b200_vertex_normals_backward(verts.data_ptr(), faces.data_ptr(), gn.data_ptr(), B, Nv, Nf,
                                               flags | _lib.NR_GRAD_ACCUMULATE, acc.data_ptr(), ws.data_ptr(), nbytes, s) == 0
    torch.cuda.synchronize()
    assert torch.isfinite(fresh).all()
    assert rel_err(np_(acc), np_(pre + fresh)) <= 1e-6


# ------------------------------------------------------------------------------------------------- direct C ABI
def _abi_scene():
    return Scene("bilinear", True, False, False, H=32, F=120)


def _fwd_args(sc, bufs, ws, corner=True, face_light=None):
    from neural_renderer_b200 import _lib
    a = _lib.ForwardArgs()
    a.struct_size = ctypes.sizeof(_lib.ForwardArgs)
    a.flags = _lib.NR_RETURN_RGB | _lib.NR_ANTI_ALIASING | _lib.NR_TEX_UV
    a.batch_size, a.num_faces, a.raster_size, a.texture_size = sc.B, sc.F, sc.S, 0
    a.near_, a.far_, a.eps = 0.1, 100.0, 1e-4
    a.background[0], a.background[1], a.background[2] = BG
    a.faces, a.textures, a.face_uvs = sc.faces.data_ptr(), sc.tex.data_ptr(), sc.uvs.data_ptr()
    a.texture_height, a.texture_width = sc.tex.shape[1], sc.tex.shape[2]
    for k in ("face_index_map", "weight_map", "depth_map", "rgb_map", "out_rgb"):
        setattr(a, k, bufs[k].data_ptr())
    a.workspace, a.workspace_bytes = ws.data_ptr(), ws.numel()
    a.corner_light = sc.corner.data_ptr() if corner else None
    a.face_light = face_light.data_ptr() if face_light is not None else None
    return a


def _fwd_bufs(sc):
    from abi_harness import alloc
    B, S = sc.B, sc.S
    return {"face_index_map": alloc((B, S, S), np.int32, 4, DEV), "weight_map": alloc((B, 3, S, S), np.float32, 4, DEV),
            "depth_map": alloc((B, S, S), np.float32, 0, DEV), "rgb_map": alloc((B, 3, S, S), np.float32, 4, DEV),
            "out_rgb": alloc((B, 3, S // 2, S // 2), np.float32, 4, DEV)}


def test_abi_forward_struct_sizes_and_rejections():
    from abi_harness import guards_intact, poison
    from neural_renderer_b200 import _lib
    lib = _lib.load()
    sc = _abi_scene()
    s = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    ws = torch.empty((lib.nr_b200_forward_workspace_bytes(sc.B, sc.F, sc.S, 0, 0),), dtype=torch.uint8, device=DEV)
    bufs = _fwd_bufs(sc)
    for t in bufs.values():
        poison(t)
    assert lib.nr_b200_forward(ctypes.byref(_fwd_args(sc, bufs, ws)), s) == 0
    torch.cuda.synchronize()
    assert all(torch.isfinite(t.float()).all() for t in bufs.values()) and all(guards_intact(t) for t in bufs.values())
    ref = sc.render(corner=sc.corner)[0]
    assert torch.equal(bufs["out_rgb"], ref)
    # the ABI-4 struct from before corner_light: an unlit render, whatever lies past it
    short = _fwd_args(sc, bufs, ws)
    short.struct_size = _lib.ForwardArgs.corner_light.offset
    assert lib.nr_b200_forward(ctypes.byref(short), s) == 0
    torch.cuda.synchronize()
    assert torch.equal(bufs["out_rgb"], sc.render()[0])
    # face_light with corner_light, corner_light without RGB
    assert lib.nr_b200_forward(ctypes.byref(_fwd_args(sc, bufs, ws, face_light=sc.corner)), s) == _lib.NR_OK - 1
    a = _fwd_args(sc, bufs, ws)
    a.flags = _lib.NR_RETURN_ALPHA
    a.alpha_map = bufs["depth_map"].data_ptr()
    assert lib.nr_b200_forward(ctypes.byref(a), s) == _lib.NR_OK - 1


@pytest.mark.parametrize("mode", ["fresh", "accumulate", "two_halves"])
def test_abi_backward_grad_corner_light(mode):
    from abi_harness import alloc, guards_intact, poison
    from neural_renderer_b200 import _lib
    lib = _lib.load()
    sc = _abi_scene()
    s = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    ws = torch.empty((lib.nr_b200_forward_workspace_bytes(sc.B, sc.F, sc.S, 0, 0),), dtype=torch.uint8, device=DEV)
    bufs = _fwd_bufs(sc)
    assert lib.nr_b200_forward(ctypes.byref(_fwd_args(sc, bufs, ws)), s) == 0
    corner = sc.corner.clone().requires_grad_(True)
    tex = sc.tex.clone().requires_grad_(True)
    rgb = sc.render(corner=corner, tex=tex)[0]
    g = torch.randn(rgb.shape, generator=torch.Generator().manual_seed(4)).to(DEV)
    (rgb * g).sum().backward()
    gcl = alloc(tuple(sc.corner.shape), np.float32, 4, DEV)
    gtex = alloc(tuple(sc.tex.shape), np.float32, 8, DEV)
    gfaces = alloc(tuple(sc.faces.shape), np.float32, 0, DEV)
    pre = torch.randn(gcl.shape, generator=torch.Generator().manual_seed(5)).to(DEV)
    flags = _lib.NR_RETURN_RGB | _lib.NR_ANTI_ALIASING | _lib.NR_TEX_UV
    if mode == "accumulate":
        gcl.copy_(pre); gtex.zero_(); gfaces.zero_()
        flags |= _lib.NR_GRAD_ACCUMULATE
    else:
        for t in (gcl, gtex, gfaces):
            poison(t)
    bws = torch.empty((lib.nr_b200_backward_workspace_bytes(sc.B, sc.F, sc.S, 0, flags),), dtype=torch.uint8, device=DEV)
    b = _lib.BackwardArgs()
    b.struct_size = ctypes.sizeof(_lib.BackwardArgs)
    b.batch_size, b.num_faces, b.raster_size, b.texture_size = sc.B, sc.F, sc.S, 0
    b.eps = 1e-4
    b.faces, b.textures, b.face_uvs = sc.faces.data_ptr(), sc.tex.data_ptr(), sc.uvs.data_ptr()
    b.texture_height, b.texture_width = sc.tex.shape[1], sc.tex.shape[2]
    b.face_index_map, b.weight_map = bufs["face_index_map"].data_ptr(), bufs["weight_map"].data_ptr()
    b.depth_map, b.rgb_map = bufs["depth_map"].data_ptr(), bufs["rgb_map"].data_ptr()
    gc = g.contiguous()
    b.grad_rgb = gc.data_ptr()
    b.grad_faces, b.grad_textures = gfaces.data_ptr(), gtex.data_ptr()
    b.workspace, b.workspace_bytes = bws.data_ptr(), bws.numel()
    cl, gcl_p = ctypes.c_void_p(sc.corner.data_ptr()), ctypes.c_void_p(gcl.data_ptr())
    calls = [flags | _lib.NR_BWD_PART_TEXTURES, flags | _lib.NR_BWD_PART_FACES] if mode == "two_halves" else [flags]
    for i, fl in enumerate(calls):
        b.flags = fl
        assert lib.nr_b200_backward_corner_light(ctypes.byref(b), cl, gcl_p, s) == 0
        torch.cuda.synchronize()
        if i == 0 and mode == "two_halves":  # the texture half alone delivers grad_corner_light
            assert torch.isfinite(gcl).all()
            assert rel_err(np_(gcl), np_(corner.grad)) <= 1e-5
    assert all(guards_intact(t) for t in (gcl, gtex, gfaces))
    want = corner.grad + (pre if mode == "accumulate" else 0)
    assert torch.isfinite(gcl).all()
    assert rel_err(np_(gcl), np_(want)) <= 1e-5
    assert rel_err(np_(gtex), np_(tex.grad)) <= 1e-5
    # rejections: face_light together with corner_light; grad_corner_light without textures
    b.flags = flags
    b.face_light = sc.corner.data_ptr()
    assert lib.nr_b200_backward_corner_light(ctypes.byref(b), cl, gcl_p, s) == _lib.NR_OK - 1
    b.face_light = None
    b.textures = None
    assert lib.nr_b200_backward_corner_light(ctypes.byref(b), cl, gcl_p, s) == _lib.NR_OK - 1


# ------------------------------------------------------------------------------------------------------ Renderer
def _renderer(fill_back, fused, shading="smooth"):
    import neural_renderer_b200 as nr
    r = nr.Renderer()
    r.image_size = 64
    r.fill_back = fill_back
    r.fused = fused
    r.shading = shading
    r.eye = (0.3, 0.5, -2.4)
    r.light_direction = (0.3, 0.8, -0.5)
    return r


def _teapot_inputs(kind, B=2):
    verts, faces = _mesh(B=B)
    verts = verts * 0.9
    F = faces.shape[0]
    if kind == "cube":
        tex = _rand((B, F, 2, 2, 2, 3), 0.2, 1.0, seed=11)
        return verts, faces[None].expand(B, -1, -1), tex, None
    uvs = _rand((F, 3, 2), seed=12)
    return verts, faces[None].expand(B, -1, -1), _rand((64, 48, 3), 0.2, 1.0, seed=13), uvs


@pytest.mark.parametrize("kind", ["cube", "image"])
@pytest.mark.parametrize("fill_back", [False, True])
def test_renderer_smooth_fused_matches_op_by_op(kind, fill_back):
    verts0, faces, tex0, uvs = _teapot_inputs(kind)
    out = []
    for fused in (True, False):
        v = verts0.clone().requires_grad_(True)
        tex = tex0.clone().requires_grad_(True)
        img = _renderer(fill_back, fused).render(v, faces, tex, face_uvs=uvs)
        g = torch.randn(img.shape, generator=torch.Generator().manual_seed(3)).to(DEV)
        (img * g).sum().backward()
        out.append((img.detach(), tex.grad, v.grad))
    (i0, t0, v0), (i1, t1, v1) = out
    print("fused vs op", kind, fill_back, rel_err(np_(i0), np_(i1)), rel_err(np_(t0), np_(t1)), rel_err(np_(v0), np_(v1)))
    assert rel_err(np_(i0), np_(i1)) <= 1e-6
    assert rel_err(np_(t0), np_(t1)) <= 1e-5
    assert rel_err(np_(v0), np_(v1)) <= 1e-4


def test_renderer_smooth_is_deterministic_and_differs_from_flat():
    verts, faces, tex, uvs = _teapot_inputs("image")
    r = _renderer(True, True)
    a, b = r.render(verts, faces, tex, face_uvs=uvs), r.render(verts, faces, tex, face_uvs=uvs)
    assert torch.equal(a, b)
    flat = _renderer(True, True, "flat").render(verts, faces, tex, face_uvs=uvs)
    assert (a - flat).abs().max() > 1e-3


def test_renderer_smooth_step_in_cuda_graph():
    verts0, faces, tex0, uvs = _teapot_inputs("image")
    r = _renderer(True, True)
    v = verts0.clone().requires_grad_(True)
    g = torch.randn((2, 3, 64, 64), generator=torch.Generator().manual_seed(3)).to(DEV)

    def step():
        v.grad = None
        (r.render(v, faces, tex0, face_uvs=uvs) * g).sum().backward()
        return v.grad

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            step()
    torch.cuda.current_stream().wait_stream(s)
    eager = step().clone()
    graph = torch.cuda.CUDAGraph()
    v.grad = None
    with torch.cuda.graph(graph):
        (r.render(v, faces, tex0, face_uvs=uvs) * g).sum().backward()
    graph.replay()
    torch.cuda.synchronize()
    assert rel_err(np_(v.grad), np_(eager)) <= 1e-5


def test_smooth_shading_gives_vertex_gradient_where_flat_cannot():
    """a sphere seen with its silhouette masked out: moving a vertex changes the shading of faces it does not belong to
    only through the vertex normals of their shared vertices -- smooth shading has that gradient, flat shading has none"""
    from neural_renderer_b200 import synthetic
    import neural_renderer_b200 as nr
    v_np, f_np = synthetic.sphere_mesh(400)
    verts = torch.from_numpy(np.asarray(v_np, np.float32))[None].to(DEV)
    faces = torch.from_numpy(np.asarray(f_np, np.int32))[None].to(DEV)
    tex = torch.ones((1, faces.shape[1], 2, 2, 2, 3), device=DEV)
    grads = {}
    for shading in ("flat", "smooth"):
        r = _renderer(False, True, shading)
        r.eye = (0.0, 0.0, -3.0)
        r.light_direction = (0.2, 0.5, -1.0)
        v = verts.clone().requires_grad_(True)
        img = r.render(v, faces, tex)
        alpha = r.render_silhouettes(verts, faces).detach()
        inner = torch.nn.functional.max_pool2d(-alpha[:, None], 9, 1, 4)[:, 0] < -0.5  # well inside the silhouette
        # differentiate one pixel well inside the silhouette: the vertices it reaches beyond the winner's own are the
        # edge scan's (both shadings) and, with smooth shading only, the one-ring of the winner's corners
        c = img.shape[-1] // 2
        assert inner[0, c, c]
        img[0, :, c, c].sum().backward()
        grads[shading] = v.grad[0]
    moved_flat = (grads["flat"].abs().sum(dim=1) > 0)
    moved_smooth = (grads["smooth"].abs().sum(dim=1) > 0)
    # smooth reaches strictly more vertices (the one-ring of the winner's corners) than flat (the winner's own corners)
    assert moved_smooth.sum() > moved_flat.sum()
    assert (moved_smooth & ~moved_flat).any()
