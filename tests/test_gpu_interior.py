"""GPU: the interior vertex gradient of the RGB image (rasterize(..., interior_gradient=True), NR_GRAD_INTERIOR).

The term is isolated through the direct ABI (tests/abi_harness.py buffers) with the saved rgb map replaced by zeros: the
edge scan K5 then has no colour difference to differentiate and adds exact zeros (the flag-off call must return an
all-zero face gradient), so the result is the new kernel alone, free of the run-to-run spread of K5's unordered fp32
atomics that grad(on) - grad(off) carries.  It is held to
  - the float64 closed form of oracles_interior on the product's maps, with the vertex-gradient gates of
    test_gpu_attr.py (per tensor 1e-4, per element 2.5e-3), over cubes / bilinear / trilinear, unlit / face / corner light,
    anti-aliasing, fill_back, indexed or materialised geometry, shared or per-item textures and UVs, rasters 257 and 1100;
  - the vertex gradient of nr_b200_interpolate_backward, an independent kernel, at 1e-5 (smooth shading of an all-ones
    texture is the corner light rendered as an attribute; an affine image is the attribute affine(uv_k); affine cubes are
    the attribute (ts - 1) coef_k + delta where no cube coordinate is clamped);
  - central differences of the product's own forward (on - off through autograd);
and the Python path to the isolated term, the direct ABI (offsets, guards, poison, both entry points, accumulate, the
two-half call, the short struct layout, the refusal), the Renderer (fused against op by op, a CUDA-graph step, the
ValueError) and an Adam fit of a textured grid from the RGB loss alone."""
import ctypes

import numpy as np
import pytest
import torch

from helpers import elem_err, np_, rel_err
from oracles import pyramid64
from oracles_interior import Tex, faces_to_vertices, interior_grad64, select
from oracles_attr import clamp_active

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _R():
    import importlib
    return importlib.import_module("neural_renderer_b200.rasterize")


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _grid(n, B, seed, jitter=0.02, lo=-0.9, hi=0.9):
    """an n x n vertex grid over [lo, hi]^2 per item (two triangles per quad), jittered, depths in [2, 3]"""
    g = _gen(seed)
    t = torch.linspace(lo, hi, n, device=DEV)
    yy, xx = torch.meshgrid(t, t, indexing="ij")
    xy = torch.stack((xx, yy), dim=-1).reshape(1, -1, 2).repeat(B, 1, 1)
    xy = xy + jitter * (torch.rand(xy.shape, generator=g, device=DEV) - 0.5)
    z = 2.0 + torch.rand((B, n * n, 1), generator=g, device=DEV)
    quads = [(i * n + j, i * n + j + 1, (i + 1) * n + j + 1, (i + 1) * n + j) for i in range(n - 1) for j in range(n - 1)]
    faces = torch.tensor([[a, b, c] for a, b, c, d in quads] + [[a, c, d] for a, b, c, d in quads], dtype=torch.int32,
                         device=DEV)
    return torch.cat((xy, z), dim=-1).contiguous(), faces


def _materialise(verts, idx):
    B = verts.shape[0]
    return verts[torch.arange(B, device=DEV)[:, None, None], idx.long()[None].expand(B, -1, -1)]


def _upsample(g, aa):
    return g.repeat_interleave(2, -1).repeat_interleave(2, -2) * 0.25 if aa else g


# (kind, light, aa, fill_back, indexed, shared, S)
CASES = [
    ("cube2", "unlit", False, False, True, False, 257),
    ("cube4", "face", True, True, False, True, 257),
    ("cube4", "corner", False, True, True, False, 257),
    ("cube2", "corner", True, False, False, True, 257),
    ("bilinear", "unlit", True, True, True, True, 257),
    ("bilinear", "face", False, False, False, False, 257),
    ("bilinear", "corner", False, True, False, True, 257),
    ("bilinear", "corner", True, False, True, False, 1100),
    ("trilinear", "unlit", False, True, False, False, 257),
    ("trilinear", "face", True, False, True, True, 257),
    ("trilinear", "corner", True, True, False, False, 257),
    ("cube4", "unlit", False, False, True, True, 1100),
    ("trilinear", "face", False, False, True, False, 1100),
]


def _setup_case(case, seed=0):
    kind, light, aa, fill_back, indexed, shared, S = case
    B = 2
    verts, idx = _grid(9, B, seed)
    if fill_back:
        idx = torch.cat((idx, idx.flip(1)), dim=0)
    F = idx.shape[0]
    nf = F // 2 if fill_back else F
    g = _gen(seed + 10)
    Bt = 1 if shared else B
    if kind.startswith("cube"):
        ts = int(kind[-1])
        tex = torch.rand((Bt, nf, ts, ts, ts, 3), generator=g, device=DEV)
        uvs = None
    else:
        tex = torch.rand((Bt, 37, 29, 3), generator=g, device=DEV)
        uvs = torch.rand((Bt, nf, 3, 2), generator=g, device=DEV) * 1.2 - 0.1
    lt = torch.rand((B, F, 3), generator=g, device=DEV) + 0.5 if light == "face" else None
    corner = torch.rand((B, F, 3, 3), generator=g, device=DEV) + 0.5 if light == "corner" else None
    H = S // 2 if aa else S  # an odd raster needs anti-aliasing off: 257 becomes 256 with it
    up = torch.randn((B, 3, H, H), generator=g, device=DEV)
    S = 2 * H if aa else S
    return dict(verts=verts, idx=idx, tex=tex, uvs=uvs, lt=lt, corner=corner, up=up, aa=aa, S=S, kind=kind,
                fill_back=fill_back, indexed=indexed, H=H)


def _grad(c, on, textures=None):
    """(d sum(up * rgb) / d geometry, d / d textures, maps) with the flag on or off"""
    R = _R()
    tex = (c["tex"] if textures is None else textures).clone().requires_grad_(True)
    geom = c["verts"] if c["indexed"] else _materialise(c["verts"], c["idx"])
    geom = geom.clone().requires_grad_(True)
    rgb, _, _, fim, wmap = R._run(c["idx"] if c["indexed"] else geom, tex, c["H"], c["aa"], 0.1, 100, 1e-4, (0, 0, 0), True, False,
                                  False, face_light=c["lt"], textures_fill_back=c["fill_back"],
                                  vertices=geom if c["indexed"] else None, reference_exact=False, face_uvs=c["uvs"],
                                  texture_filter="trilinear" if c["kind"] == "trilinear" else "bilinear",
                                  corner_light=c["corner"], interior_gradient=on)
    (rgb * c["up"]).sum().backward()
    return geom.grad, tex.grad, fim, wmap


def _oracle(c, fim, wmap):
    S = c["S"]
    faces64 = _materialise(c["verts"], c["idx"]).double()
    if c["kind"].startswith("cube"):
        tex = Tex("cube", c["tex"].double(), eps=c.get("eps", 1e-4), fill_back=c["fill_back"])
    else:
        levels = [c["tex"].double()] if c["kind"] == "bilinear" else pyramid64(c["tex"].double())
        tex = Tex(c["kind"], levels, uvs=c["uvs"].double(), fill_back=c["fill_back"])
    sel = select(faces64, fim, wmap, S, tex)
    g = _upsample(c["up"].double(), c["aa"])
    gf = interior_grad64(faces64, fim, wmap, S, tex, sel, g, c["lt"], c["corner"])
    return faces_to_vertices(gf, c["idx"], c["verts"].shape[1]) if c["indexed"] else gf


def _maps(c):
    """the raster maps of the case's forward (rgb_map, depth_map, face_index_map, weight_map): a forward without
    anti-aliasing at the raster size writes the same maps as the anti-aliased one"""
    R = _R()
    geom = c["verts"] if c["indexed"] else _materialise(c["verts"], c["idx"])
    rgb, _, dmap, fim, wmap = R._run(c["idx"] if c["indexed"] else geom, c["tex"], c["S"], False, 0.1, 100, c.get("eps", 1e-4),
                                     (0, 0, 0),
                                     True, False, True, face_light=c["lt"], textures_fill_back=c["fill_back"],
                                     vertices=geom if c["indexed"] else None, reference_exact=False, face_uvs=c["uvs"],
                                     texture_filter="trilinear" if c["kind"] == "trilinear" else "bilinear",
                                     corner_light=c["corner"])
    return rgb.contiguous(), dmap.contiguous(), fim, wmap


def _abi(c, maps, on, zero_rgb=True, offset=0, extra=0, struct_size=None, buf=None, prefill=None):
    """one direct backward call (nr_b200_backward, or nr_b200_backward_corner_light with a corner light) on abi_harness
    buffers: every input and output `offset` bytes past a 16-byte boundary between guard words, outputs poisoned (or
    `prefill`ed) unless `buf` of an earlier call is given.  zero_rgb: the saved rgb map is replaced by zeros, so the edge
    scan has no colour difference to differentiate and adds exact zeros -- the flag's term alone, with no run-to-run spread
    of K5's atomics in it.  Returns (return code, buffers); the guards are checked."""
    from abi_harness import alloc, guards_intact, poison, workspace
    from neural_renderer_b200 import _lib
    lib = _lib.load()
    R = _R()
    rgb, dmap, fim, wmap = maps
    B, F, S = c["verts"].shape[0], c["idx"].shape[0], c["S"]
    geom = c["verts"] if c["indexed"] else _materialise(c["verts"], c["idx"])
    tex = R._MipPyramid.apply(c["tex"]).detach() if c["kind"] == "trilinear" else c["tex"]
    if buf is None:
        inputs = {"geom": geom, "tex": tex, "fim": fim, "wmap": wmap, "dmap": dmap,
                  "rgb": torch.zeros_like(rgb) if zero_rgb else rgb, "g": c["up"]}
        for k in ("idx", "uvs", "lt", "corner"):
            if c[k] is not None and (k != "idx" or c["indexed"]):
                inputs[k] = c[k]
        buf = {}
        for k, t in inputs.items():
            buf[k] = alloc(tuple(t.shape), np.int32 if t.dtype == torch.int32 else np.float32, offset, DEV)
            buf[k].copy_(t)
        for k, t in (("gg", geom), ("gt", tex)):
            buf[k] = alloc(tuple(t.shape), np.float32, offset, DEV)
            poison(buf[k])
        if prefill is not None:
            buf["gg"].copy_(prefill)
    uv = c["uvs"] is not None
    flags = _lib.NR_RETURN_RGB | (_lib.NR_ANTI_ALIASING if c["aa"] else 0) | extra
    flags |= (_lib.NR_FACES_INDEXED | _lib.NR_INDICES_SHARED) if c["indexed"] else 0
    flags |= _lib.NR_TEX_SHARED if tex.shape[0] == 1 and B > 1 else 0
    flags |= _lib.NR_TEX_FILL_BACK if c["fill_back"] else 0
    flags |= _lib.NR_GRAD_INTERIOR if on else 0
    if uv:
        flags |= _lib.NR_TEX_UV | (_lib.NR_UV_SHARED if c["uvs"].shape[0] == 1 and B > 1 else 0)
        flags |= _lib.NR_TEX_MIPMAP if c["kind"] == "trilinear" else 0
    ts = 0 if uv else int(tex.shape[2])
    a = _lib.BackwardArgs()
    a.struct_size = ctypes.sizeof(_lib.BackwardArgs) if struct_size is None else struct_size
    a.flags = flags
    a.batch_size, a.num_faces, a.raster_size, a.texture_size = B, F, S, ts
    a.eps = c.get("eps", 1e-4)
    if c["indexed"]:
        a.vertices, a.face_indices, a.num_vertices = buf["geom"].data_ptr(), buf["idx"].data_ptr(), geom.shape[1]
        a.grad_vertices = buf["gg"].data_ptr()
    else:
        a.faces, a.grad_faces = buf["geom"].data_ptr(), buf["gg"].data_ptr()
    a.textures, a.grad_textures = buf["tex"].data_ptr(), buf["gt"].data_ptr()
    a.face_index_map, a.weight_map, a.depth_map = buf["fim"].data_ptr(), buf["wmap"].data_ptr(), buf["dmap"].data_ptr()
    a.rgb_map, a.grad_rgb = buf["rgb"].data_ptr(), buf["g"].data_ptr()
    if uv:
        a.face_uvs = buf["uvs"].data_ptr()
        a.texture_height, a.texture_width = int(c["tex"].shape[1]), int(c["tex"].shape[2])
    if c["lt"] is not None:
        a.face_light = buf["lt"].data_ptr()
    ws = workspace(lib.nr_b200_backward_workspace_bytes(B, F, S, ts, flags), DEV)
    a.workspace, a.workspace_bytes = ws.data_ptr(), ws.numel()
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    if c["corner"] is not None:
        rc = lib.nr_b200_backward_corner_light(ctypes.byref(a), ctypes.c_void_p(buf["corner"].data_ptr()), None, st)
    else:
        rc = lib.nr_b200_backward(ctypes.byref(a), st)
    torch.cuda.synchronize()
    assert all(guards_intact(t) for t in buf.values())
    return rc, buf


@pytest.mark.parametrize("case", CASES, ids=["-".join(str(x) for x in c) for c in CASES])
def test_interior_term_against_float64_oracle(case):
    """the flag's term alone (a constant rgb map: the edge scan adds exact zeros) against the float64 closed form"""
    c = _setup_case(case)
    maps = _maps(c)
    rc, on = _abi(c, maps, True)
    assert rc == 0
    rc, off = _abi(c, maps, False)
    assert rc == 0
    assert (off["gg"] == 0).all()  # the premise: nothing but the new kernel writes a non-zero face gradient
    ref = _oracle(c, maps[2], maps[3])
    got = on["gg"].double()
    r, e = rel_err(np_(got), np_(ref)), elem_err(np_(got), np_(ref))
    print("interior", case, "rel", r, "elem", e, "max", float(ref.abs().max()))
    assert ref.abs().max() > 0
    assert r <= 1e-4
    assert e <= 2.5e-3
    # the texture half is untouched by the flag
    assert rel_err(np_(on["gt"]), np_(off["gt"])) <= 1e-5
    # the Python path carries the same term: on - off through autograd, which adds K5 (unordered atomics) on both sides
    # of the subtraction; a fixed bound, 5x the largest per-tensor K5 spread measured over this matrix (H100)
    g_on, _, _, _ = _grad(c, True)
    g_off, _, _, _ = _grad(c, False)
    rp = rel_err(np_(g_on - g_off), np_(on["gg"]))
    print("  python path", rp)
    assert rp <= 2.5e-4


def _attr_case(verts, idx, tex, uvs=None, corner=None, up=None, kind="bilinear"):
    return dict(verts=verts, idx=idx, tex=tex, uvs=uvs, lt=None, corner=corner, up=up, aa=False, S=up.shape[-1], H=up.shape[-1],
                kind=kind, fill_back=False, indexed=True)


def _attribute_vertex_grad(idx, verts, attr, up):
    """d sum(up * attribute image) / d vertices: nr_b200_interpolate_backward (no edge term: alpha is not returned)"""
    import neural_renderer_b200 as nr
    v = verts.clone().requires_grad_(True)
    (nr.rasterize_attributes(idx, up.shape[-1], False, vertices=v, face_attributes=attr) * up).sum().backward()
    return v.grad


def test_smooth_shading_of_white_texture_equals_corner_light_attribute():
    """all-ones image: the sample is 1, E = 0, and the interior term is the corner light's own chain -- the vertex gradient
    nr_b200_interpolate_backward gives for corner_light rendered as a C = 3 attribute"""
    verts, idx = _grid(9, 2, 3)
    g = _gen(4)
    corner = torch.rand((2, idx.shape[0], 3, 3), generator=g, device=DEV) + 0.5
    img = torch.ones((1, 8, 8, 3), device=DEV)
    uvs = torch.rand((1, idx.shape[0], 3, 2), generator=g, device=DEV)
    up = torch.randn((2, 3, 200, 200), generator=g, device=DEV)
    c = _attr_case(verts, idx, img, uvs=uvs, corner=corner, up=up)
    rc, on = _abi(c, _maps(c), True)
    assert rc == 0
    want = _attribute_vertex_grad(idx, verts, corner, up)
    err = rel_err(np_(on["gg"]), np_(want))
    print("smooth vs attribute", err, elem_err(np_(on["gg"]), np_(want)))
    assert err <= 1e-5


def test_affine_image_equals_affine_uv_attribute():
    """an image affine in the tap position, UVs inside [0, 1]: the bilinear sample is affine(uv), so the interior term is
    the attribute gradient of affine(uv_k)"""
    verts, idx = _grid(9, 2, 5)
    g = _gen(6)
    Ht, Wt = 23, 31
    A = torch.tensor([[0.7, -0.3, 0.2], [0.1, 0.5, -0.4]], device=DEV)  # d colour / d (u, v)
    b0 = torch.tensor([0.1, 0.2, 0.3], device=DEV)
    x = torch.arange(Wt, device=DEV, dtype=torch.float32) / (Wt - 1)
    y = torch.arange(Ht, device=DEV, dtype=torch.float32).flip(0) / (Ht - 1)  # row 0 = top = v 1
    img = (x[None, :, None] * A[0] + y[:, None, None] * A[1] + b0)[None].contiguous()
    uvs = 0.05 + 0.9 * torch.rand((1, idx.shape[0], 3, 2), generator=g, device=DEV)
    up = torch.randn((2, 3, 200, 200), generator=g, device=DEV)
    c = _attr_case(verts, idx, img, uvs=uvs, up=up)
    rc, on = _abi(c, _maps(c), True)
    assert rc == 0
    attr = uvs[..., 0, None] * A[0] + uvs[..., 1, None] * A[1] + b0  # [1,F,3,3]
    want = _attribute_vertex_grad(idx, verts, attr, up)
    err = rel_err(np_(on["gg"]), np_(want))
    print("affine image vs attribute", err, elem_err(np_(on["gg"]), np_(want)))
    assert err <= 1e-5


@pytest.mark.parametrize("ts", [2, 4])
def test_affine_cube_equals_affine_attribute(ts):
    """cubes whose texel (i0, i1, i2) is delta + sum_k coef_k i_k: the trilinear sample at t_k = (ts - 1) l_k (own depths) is
    delta + (ts - 1) sum_k coef_k l_k, so on pixels where no cube coordinate is clamped the interior term is the attribute
    gradient of corner k's (ts - 1) coef_k + delta; the clamp-active pixels (a corner's t_k above ts - 1 - eps) get a zero
    upstream gradient.  eps = 0.3 puts the clamp on every pixel with some l_k above 1 - 0.3 / (ts - 1); with the full
    upstream gradient the term, clamp gate included, is held to the float64 oracle as well"""
    verts, idx = _grid(9, 2, 16)
    F = idx.shape[0]
    g = _gen(17)
    coef = torch.tensor([[0.30, -0.20, 0.10], [-0.15, 0.25, 0.20], [0.05, 0.10, -0.30]], device=DEV)  # [axis k, channel]
    delta = torch.tensor([0.2, 0.4, 0.3], device=DEV)
    i = torch.arange(ts, device=DEV, dtype=torch.float32)
    cube = (delta + i[:, None, None, None] * coef[0] + i[None, :, None, None] * coef[1] + i[None, None, :, None] * coef[2])
    tex = cube[None, None].expand(1, F, ts, ts, ts, 3).contiguous()
    up = torch.randn((2, 3, 200, 200), generator=g, device=DEV)
    c = _attr_case(verts, idx, tex, up=up, kind="cube")
    c["eps"] = 0.3
    maps = _maps(c)
    rc, full = _abi(c, maps, True)
    assert rc == 0
    ref = _oracle(c, maps[2], maps[3])
    ro, eo = rel_err(np_(full["gg"]), np_(ref)), elem_err(np_(full["gg"]), np_(ref))
    faces64 = _materialise(verts, idx).double()
    sel = select(faces64, maps[2], maps[3], 200, Tex("cube", tex.double(), eps=0.3))
    clamped = (maps[2] >= 0) & ~sel["gate"].all(-1)
    c["up"] = up * ~clamped[:, None]
    rc, on = _abi(c, maps, True)
    assert rc == 0
    attr = ((ts - 1) * coef + delta)[None, None].expand(1, F, 3, 3).contiguous()  # corner k: (ts - 1) coef_k + delta
    want = _attribute_vertex_grad(idx, verts, attr, c["up"])
    err = rel_err(np_(on["gg"]), np_(want))
    print("affine cube vs attribute", ts, err, elem_err(np_(on["gg"]), np_(want)), "clamp-active pixels", int(clamped.sum()),
          "oracle with them", ro, eo)
    assert int(clamped.sum()) > 0
    assert err <= 1e-5
    assert ro <= 1e-4 and eo <= 2.5e-3


@pytest.mark.parametrize("kind", ["bilinear", "smooth", "cube"])
def test_interior_term_vs_central_difference(kind):
    """the directional derivative of sum(g * rgb) over the pixels whose winner does not change and whose weights, UV or
    cube coordinate are not clamped, against (on - off) . direction with the upstream gradient zeroed elsewhere"""
    R = _R()
    S = 96
    verts, idx = _grid(7, 1, 7, lo=-0.7, hi=0.7)
    F = idx.shape[0]
    g = _gen(8)
    corner = torch.rand((1, F, 3, 3), generator=g, device=DEV) + 0.5 if kind == "smooth" else None
    if kind == "cube":
        tex, uvs = torch.rand((1, F, 4, 4, 4, 3), generator=g, device=DEV), None
    else:
        tex, uvs = torch.rand((1, 16, 16, 3), generator=g, device=DEV), 0.1 + 0.8 * torch.rand((1, F, 3, 2), generator=g, device=DEV)
    up = torch.randn((1, 3, S, S), generator=g, device=DEV)
    d = torch.randn(verts.shape, generator=g, device=DEV) * torch.tensor([1.0, 1.0, 0.3], device=DEV)

    def fwd(v, on=False):
        return R._run(idx, tex, S, False, 0.1, 100, 1e-4, (0, 0, 0), True, False, False, vertices=v, reference_exact=False,
                      face_uvs=uvs, corner_light=corner, interior_gradient=on)
    h = 5e-4
    outs = [fwd(verts + s * h * d) for s in (0, 1, -1)]
    fims = [o[3] for o in outs]
    keep = (fims[0] == fims[1]) & (fims[0] == fims[2]) & (fims[0] >= 0)
    tx = Tex("cube", tex.double()) if kind == "cube" else Tex("bilinear", [tex.double()], uvs=uvs.double())
    cells = []
    for s, o in zip((0, 1, -1), outs):
        f64 = _materialise(verts + s * h * d, idx).double()
        keep &= ~clamp_active(f64, fims[0], S)
        sel = select(f64, fims[0], o[4], S, tx)
        # the derivative holds the texel cell and the clamps fixed: so must the step
        if kind == "cube":
            cells.append(torch.cat((sel["i"], sel["gate"].long()), -1))
        else:
            cells.append(torch.cat((sel["lv"][0][0][..., None], sel["lv"][0][1][..., None], sel["inside"].long()), -1))
    keep &= ((cells[0] == cells[1]) & (cells[0] == cells[2])).all(-1)
    gm = up * keep[:, None]
    num = float(((outs[1][0].double() - outs[2][0].double()) * gm).sum() / (2 * h))
    grads = []
    for on in (True, False):
        v = verts.clone().requires_grad_(True)
        (fwd(v, on)[0] * gm).sum().backward()
        grads.append(v.grad)
    ana = float(((grads[0] - grads[1]).double() * d).sum())
    print("central difference", kind, num, ana, int(keep.sum()))
    assert abs(ana) > 0
    assert abs(num - ana) <= 0.01 * abs(ana)


ABI_CASES = [("bilinear", "corner", True, False, True, False, 64), ("cube4", "face", False, True, False, True, 64)]


@pytest.mark.parametrize("offset", [0, 4, 8])
@pytest.mark.parametrize("case", ABI_CASES, ids=["image-corner-light", "cube-face-light"])
def test_direct_abi_offsets_accumulate_two_halves_short_layout_and_rejection(case, offset):
    """both entry points with the flag on guarded, poisoned buffers 0 / 4 / 8 bytes past a 16-byte boundary (the image
    case through nr_b200_backward_corner_light): accumulate, the two-half call, the short struct layout and the refusal of
    the cubes' NR_TEX_Z_BATCH0 at B > 1, each against the fresh full call"""
    from neural_renderer_b200 import _lib
    lib = _lib.load()
    c = _setup_case(case)
    maps = _maps(c)
    rc, one = _abi(c, maps, True, offset=offset)
    assert rc == 0 and torch.isfinite(one["gg"]).all() and torch.isfinite(one["gt"]).all()
    assert one["gg"].abs().max() > 0
    # with the real rgb map the edge scan adds its term on top (the flag only adds)
    rc, full = _abi(c, maps, True, zero_rgb=False, offset=offset)
    rc0, full_off = _abi(c, maps, False, zero_rgb=False, offset=offset)
    assert rc == 0 and rc0 == 0
    assert rel_err(np_(full["gg"] - full_off["gg"]), np_(one["gg"])) <= 2.5e-4
    # accumulate into a prefilled buffer
    pre = torch.randn(one["gg"].shape, generator=_gen(21), device=DEV)
    rc, acc = _abi(c, maps, True, offset=offset, extra=_lib.NR_GRAD_ACCUMULATE, prefill=pre)
    assert rc == 0
    ea = rel_err(np_(acc["gg"] - pre), np_(one["gg"]))
    # two halves into the same buffers: the texture half leaves the face gradient alone, the faces half writes it
    rc, two = _abi(c, maps, True, offset=offset, extra=_lib.NR_BWD_PART_TEXTURES)
    assert rc == 0 and torch.isnan(two["gg"]).all()
    rc, two = _abi(c, maps, True, extra=_lib.NR_BWD_PART_FACES, buf=two)
    assert rc == 0
    eh = rel_err(np_(two["gg"]), np_(one["gg"]))
    assert rel_err(np_(two["gt"]), np_(one["gt"])) <= 1e-6
    # the ABI-4 layout before grad_face_uvs
    from neural_renderer_b200._lib import BackwardArgs
    rc, short = _abi(c, maps, True, offset=offset, struct_size=BackwardArgs.grad_face_uvs.offset)
    assert rc == 0
    es = rel_err(np_(short["gg"]), np_(one["gg"]))
    print("abi", case, offset, "accumulate", ea, "two halves", eh, "short", es)
    assert max(ea, eh, es) <= 1e-5
    if c["uvs"] is None:  # the refusal, before any launch: the outputs stay poisoned
        rc, bad = _abi(c, maps, True, offset=offset, extra=_lib.NR_TEX_Z_BATCH0)
        assert rc == -1 and lib.nr_b200_last_launch_count() == 0  # NR_ERR_INVALID_ARG
        assert torch.isnan(bad["gg"]).all() and torch.isnan(bad["gt"]).all()


def _mesh(B=2, seed=13):
    verts, idx = _grid(8, 1, seed, lo=-0.6, hi=0.6)
    v = verts[0].clone()
    v[:, 2] = v[:, 2] - 2.5 + 0.2 * torch.sin(3 * v[:, 0])  # a wavy sheet around the origin in world space
    return v[None].repeat(B, 1, 1).contiguous(), idx[None].expand(B, -1, -1)


@pytest.mark.parametrize("mode", ["cube", "image", "smooth-cube", "smooth-image"])
@pytest.mark.parametrize("fill_back", [False, True])
def test_renderer_fused_matches_op_by_op(mode, fill_back):
    import neural_renderer_b200 as nr
    verts, faces = _mesh()
    g = _gen(14)
    F = faces.shape[1]
    if "cube" in mode:
        tex, uvs = torch.rand((2, F, 4, 4, 4, 3), generator=g, device=DEV), None
    else:
        tex, uvs = torch.rand((1, 32, 32, 3), generator=g, device=DEV), torch.rand((F, 3, 2), generator=g, device=DEV)
    up = torch.randn((2, 3, 128, 128), generator=g, device=DEV)
    out = {}
    for fused in (True, False):
        for on in (True, False):
            r = nr.Renderer()
            r.image_size, r.fill_back, r.fused, r.reference_exact = 128, fill_back, fused, False
            r.shading = "smooth" if "smooth" in mode else "flat"
            r.interior_gradient = on
            v = verts.clone().requires_grad_(True)
            (r.render(v, faces, tex, face_uvs=uvs) * up).sum().backward()
            out[fused, on] = v.grad
    d_f, d_o = out[True, True] - out[True, False], out[False, True] - out[False, False]
    e = rel_err(np_(d_f), np_(d_o))
    print("fused vs op by op", mode, fill_back, e, rel_err(np_(out[True, True]), np_(out[False, True])))
    assert d_f.abs().max() > 0
    assert e <= 1e-3
    assert rel_err(np_(out[True, True]), np_(out[False, True])) <= 1e-3


def test_renderer_rejects_reference_exact_cubes_and_captures_a_graph():
    import neural_renderer_b200 as nr
    verts, faces = _mesh()
    g = _gen(15)
    tex = torch.rand((2, faces.shape[1], 4, 4, 4, 3), generator=g, device=DEV)
    r = nr.Renderer()
    r.image_size, r.interior_gradient, r.reference_exact = 64, True, True
    with pytest.raises(ValueError, match="reference_exact=False"):
        r.render(verts, faces, tex)
    r.reference_exact = False
    v = verts.clone().requires_grad_(True)
    up = torch.randn((2, 3, 64, 64), generator=g, device=DEV)
    r.shading = "smooth"
    img = torch.rand((1, 16, 16, 3), generator=g, device=DEV)
    uvs = torch.rand((faces.shape[1], 3, 2), generator=g, device=DEV)

    def loss():
        return (r.render(v, faces, img, face_uvs=uvs) * up).sum()
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
    assert rel_err(np_(v.grad), np_(eager)) <= 1e-4


def test_two_half_backward_through_the_hook_equals_one_call():
    R = _R()
    c = _setup_case(("bilinear", "corner", True, True, True, False, 257))
    one, tex_one, _, _ = _grad(c, True)
    prev = R.set_texture_grad_hook(lambda gt: None)
    try:
        two, tex_two, _, _ = _grad(c, True)
    finally:
        R.set_texture_grad_hook(prev)
    assert rel_err(np_(two), np_(one)) <= 1e-5 and rel_err(np_(tex_two), np_(tex_one)) <= 1e-5


def test_rgb_loss_alone_fits_a_textured_grid_without_silhouette():
    """test_attribute_loss_alone_fits_vertices_without_silhouette with a texture image instead of the UV attribute: the
    screen-covering grid carries a smooth image, and Adam on the RGB loss with interior_gradient=True must cut the vertex
    error at least tenfold in 300 steps.  The same loop without the flag is printed for comparison."""
    import neural_renderer_b200 as nr
    n = 15
    t = torch.linspace(-1.4, 1.4, n, device=DEV)
    yy, xx = torch.meshgrid(t, t, indexing="ij")
    xy0 = torch.stack((xx, yy), dim=-1).reshape(-1, 2)
    quads = [(i * n + j, i * n + j + 1, (i + 1) * n + j + 1, (i + 1) * n + j) for i in range(n - 1) for j in range(n - 1)]
    faces = torch.tensor([[a, b, c] for a, b, c, d in quads] + [[a, c, d] for a, b, c, d in quads], dtype=torch.int32,
                         device=DEV)
    uv = (xy0 + 1.4) / 2.8
    face_uvs = uv[faces.long()]
    s = torch.linspace(0, 1, 64, device=DEV)
    vv, uu = torch.meshgrid(s.flip(0), s, indexing="ij")  # row 0 = top = v 1
    image = torch.stack((uu, vv, 0.5 + 0.5 * torch.sin(6 * uu) * torch.cos(5 * vv)), dim=-1)
    disp = 0.04 * torch.stack((torch.sin(2.0 * xy0[:, 1] + 0.3), torch.cos(1.7 * xy0[:, 0])), dim=-1)
    inner = (xy0.abs() < 0.85).all(dim=-1)
    z = torch.full((xy0.shape[0], 1), 2.0, device=DEV)

    def render(xy, on):
        verts = torch.cat((xy, z), dim=-1)[None]
        return nr.rasterize(faces, image, 128, False, vertices=verts, face_uvs=face_uvs, interior_gradient=on)

    with torch.no_grad():
        target = render(xy0 + disp, False)
    err0 = float((xy0 - (xy0 + disp))[inner].norm(dim=-1).mean())
    res = {}
    for on in (True, False):
        xy = xy0.clone().requires_grad_(True)
        opt = torch.optim.Adam([xy], lr=2e-3)
        sched = torch.optim.lr_scheduler.StepLR(opt, 100, 0.3)
        for _ in range(300):
            opt.zero_grad()
            ((render(xy, on) - target) ** 2).sum().backward()
            opt.step()
            sched.step()
        res[on] = float((xy.detach() - (xy0 + disp))[inner].norm(dim=-1).mean())
    print("textured fit", err0, "with interior", res[True], "without", res[False], "factor", err0 / res[True])
    assert res[True] <= 0.1 * err0
