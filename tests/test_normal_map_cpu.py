"""CPU: tangent-space normal maps for Phong shading -- nr_b200_normal_map_args against the header, the new symbols and
their argtypes, the host rejections of nr_b200_forward_normal_map / nr_b200_backward_normal_map (all decided before any
device work), the float64 oracle (oracles_normal_map.py) against oracles_sh.py, the tangent glue of functional.py and
the Python argument errors."""
import ctypes
import os
import subprocess

import pytest
import torch

from oracles_normal_map import map_sample64, mapped_normal64, nm_rgb64
from oracles_sh import sh_rgb64
from test_lights_cpu import _lights
from test_phong_cpu import INVALID, OK_UP_TO_WORKSPACE, UNSUPPORTED, _P, _bwd, _fwd, _phong
from test_sh_cpu import _sh

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    from neural_renderer_b200 import build, _lib
    build.build_library()
    return _lib.load()


def test_normal_map_struct_matches_the_header(tmp_path):
    from neural_renderer_b200 import _lib
    fields = [f[0] for f in _lib.NormalMapArgs._fields_]
    exprs = ["sizeof(nr_b200_normal_map_args)"] + ["offsetof(nr_b200_normal_map_args, %s)" % f for f in fields] + \
        ["sizeof(nr_b200_sh_args)", "sizeof(nr_b200_lights_args)", "sizeof(nr_b200_phong_args)"]
    src = tmp_path / "s.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "nr_b200.h"\nint main(void){'
                   + "".join('printf("%%zu\\n", (size_t)(%s));' % e for e in exprs) + "return 0;}\n")
    exe = tmp_path / "s"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    vals = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert vals[0] == ctypes.sizeof(_lib.NormalMapArgs) == 56
    assert vals[1:1 + len(fields)] == [getattr(_lib.NormalMapArgs, f).offset for f in fields] == \
        [0, 4, 8, 12, 16, 20, 24, 32, 40, 48]
    assert vals[-3:] == [24, 32, 48]  # the SH, light-set and Phong structs are unchanged


def test_new_symbols_are_exported(lib):
    from neural_renderer_b200 import _lib
    out = subprocess.run(["nm", "-D", "--defined-only", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    for n in ("nr_b200_forward_normal_map", "nr_b200_backward_normal_map"):
        assert n in _lib.EXPORTED_SYMBOLS
        fn = getattr(lib, n)
        assert (" T " + n) in out, n
        assert fn.restype is ctypes.c_int
        assert [getattr(t, "_type_", t) for t in fn.argtypes[1:5]] == [_lib.PhongArgs, _lib.LightsArgs, _lib.ShArgs,
                                                                         _lib.NormalMapArgs]
        assert fn.argtypes[-1] is ctypes.c_void_p and len(fn.argtypes) == 6


def _nm(struct_size=None, bm=2, bt=2, hm=4, wm=5, nmap=True, tg=True, grad=True):
    from neural_renderer_b200 import _lib
    na = _lib.NormalMapArgs()
    na.struct_size = ctypes.sizeof(_lib.NormalMapArgs) if struct_size is None else struct_size
    na.map_batch, na.tangent_batch, na.map_height, na.map_width = bm, bt, hm, wm
    na.normal_map = _P if nmap else None
    na.corner_tangents = _P if tg else None
    na.grad_normal_map = na.grad_corner_tangents = _P if grad else None
    return na


def _uv(a, flags):
    from neural_renderer_b200 import _lib
    if flags & _lib.NR_TEX_UV:
        a.face_uvs = _P
        a.texture_height, a.texture_width = 8, 8
        a.texture_size = 0
    return a


def _rejections(run, lib):
    from neural_renderer_b200 import _lib
    rgb = _lib.NR_RETURN_RGB | _lib.NR_TEX_UV
    for bm in (1, 2):
        for bt in (1, 2):
            for la in (None, _lights(nl=0, lights=False), _lights(nl=3, bl=1)):
                for sa in (None, _sh(bs=1)):
                    assert run(rgb, la=la, sa=sa, na=_nm(bm=bm, bt=bt)) == OK_UP_TO_WORKSPACE, (bm, bt)
    assert run(rgb, na=_nm(hm=1, wm=1)) == OK_UP_TO_WORKSPACE
    assert run(rgb | _lib.NR_TEX_MIPMAP) == OK_UP_TO_WORKSPACE
    assert run(rgb | _lib.NR_ANTI_ALIASING) == OK_UP_TO_WORKSPACE
    assert run(rgb, na=None) == OK_UP_TO_WORKSPACE  # a NULL struct is the SH call
    assert run(_lib.NR_RETURN_RGB, na=None) == OK_UP_TO_WORKSPACE  # ... which needs no UVs
    for size in (0, 48, 55, 57, 64):
        assert run(rgb, na=_nm(struct_size=size)) == INVALID, size
    for b in (0, 3, -1):
        assert run(rgb, na=_nm(bm=b)) == INVALID, b
        assert run(rgb, na=_nm(bt=b)) == INVALID, b
    assert run(rgb, na=_nm(nmap=False)) == INVALID
    assert run(rgb, na=_nm(tg=False)) == INVALID
    for hm, wm in ((0, 4), (4, 0), (-1, 4)):
        assert run(rgb, na=_nm(hm=hm, wm=wm)) == INVALID, (hm, wm)
    assert run(_lib.NR_RETURN_RGB) == INVALID  # the map needs NR_TEX_UV
    assert run(rgb, na=_nm(hm=32768, wm=32768, bm=1)) == UNSUPPORTED  # 3 * 2^30 floats: beyond 32-bit offsets
    # everything the Phong, light-set and SH calls refuse
    assert run(rgb, ph=None) == INVALID
    assert run(rgb, ph=_phong(struct_size=56)) == INVALID
    assert run(rgb, ph=_phong(cs=False)) == INVALID
    assert run(rgb, la=_lights(nl=9)) == INVALID
    assert run(rgb, sa=_sh(bs=3)) == INVALID
    assert run(rgb, sa=_sh(sh=False)) == INVALID
    assert run(_lib.NR_RETURN_ALPHA | _lib.NR_TEX_UV) == INVALID
    assert lib.nr_b200_last_launch_count() == 0


def test_forward_normal_map_rejections(lib):
    from neural_renderer_b200 import _lib

    def run(flags, ph=_phong(), la=None, sa=None, na=_nm(), face_light=False):
        return lib.nr_b200_forward_normal_map(ctypes.byref(_uv(_fwd(flags, face_light), flags)),
                                              None if ph is None else ctypes.byref(ph),
                                              None if la is None else ctypes.byref(la),
                                              None if sa is None else ctypes.byref(sa),
                                              None if na is None else ctypes.byref(na), None)
    _rejections(run, lib)
    assert run(_lib.NR_RETURN_RGB | _lib.NR_TEX_UV, face_light=True) == INVALID
    assert lib.nr_b200_last_launch_count() == 0


def test_backward_normal_map_rejections(lib):
    from neural_renderer_b200 import _lib
    rgb = _lib.NR_RETURN_RGB | _lib.NR_TEX_UV

    def run(flags, ph=_phong(), la=None, sa=None, na=_nm(), textures=True):
        return lib.nr_b200_backward_normal_map(ctypes.byref(_uv(_bwd(flags, textures=textures), flags)),
                                               None if ph is None else ctypes.byref(ph),
                                               None if la is None else ctypes.byref(la),
                                               None if sa is None else ctypes.byref(sa),
                                               None if na is None else ctypes.byref(na), None)
    _rejections(run, lib)
    for ok in (rgb | _lib.NR_GRAD_ACCUMULATE, rgb | _lib.NR_BWD_PART_TEXTURES, rgb | _lib.NR_BWD_PART_FACES):
        assert run(ok) == OK_UP_TO_WORKSPACE, hex(ok)
    # grad_normal_map and grad_corner_tangents need the unlit sample s, so `textures`
    no_grads = _phong(grad_cs=False, grad_prm=False)
    assert run(rgb, ph=no_grads, textures=False) == INVALID
    for which in ("grad_normal_map", "grad_corner_tangents"):
        na = _nm(grad=False)
        setattr(na, which, _P)
        assert run(rgb, ph=no_grads, na=na, textures=False) == INVALID, which
    assert run(rgb, ph=no_grads, na=_nm(grad=False), textures=False) == OK_UP_TO_WORKSPACE
    assert run(rgb | _lib.NR_GRAD_INTERIOR) == UNSUPPORTED
    assert lib.nr_b200_last_launch_count() == 0


# ---------------------------------------------------------------------------------------------------- the oracle
def _scene(B=2, S=6, F=3, seed=0):
    """hand-made maps: every pixel covered by a random face with random weights (an oracle-only scene)"""
    g = torch.Generator().manual_seed(seed)
    faces = torch.rand((B, F, 3, 3), generator=g, dtype=torch.float64)
    faces[..., 2] = 1.0 + faces[..., 2]
    fim = torch.randint(0, F, (B, S, S), generator=g, dtype=torch.int32)
    w = torch.rand((B, 3, S, S), generator=g, dtype=torch.float64) + 0.1
    wmap = w / w.sum(1, keepdim=True)
    z = faces[..., 2][torch.arange(B)[:, None, None], fim.long()]
    dmap = 1.0 / (wmap.permute(0, 2, 3, 1) / z).sum(-1)
    cs = torch.cat((torch.randn((B, F, 3, 3), generator=g, dtype=torch.float64) - torch.tensor([0, 0, 2.0]),
                    faces), dim=-1)
    prm = torch.tensor([[0.3, 0.2, 0.1, 0.6, 0.7, 0.8, 0.3, 0.5, -1.0, 0.5, 0.4, 0.3, 8.0, 0.2, -0.1, -4.0]] * B,
                       dtype=torch.float64)
    uvs = torch.rand((B, F, 3, 2), generator=g, dtype=torch.float64)
    unlit = torch.rand((B, 3, S, S), generator=g, dtype=torch.float64)
    tg = torch.cat((torch.randn((B, F, 3, 3), generator=g, dtype=torch.float64),
                    torch.where(torch.rand((B, F, 3, 1), generator=g) < 0.5, -1.0, 1.0).double()), dim=-1)
    return faces, fim, wmap, dmap, cs, prm, uvs, unlit, tg


def test_flat_map_oracle_is_the_sh_oracle():
    faces, fim, wmap, dmap, cs, prm, uvs, unlit, tg = _scene()
    flat = torch.zeros((1, 4, 5, 3), dtype=torch.float64)
    flat[..., 2] = 1.0
    sh = torch.randn((1, 9, 3), generator=torch.Generator().manual_seed(1), dtype=torch.float64) * 0.2
    lt = _lights_t()
    for lights, env in ((None, None), (lt, None), (None, sh), (lt, sh)):
        a = nm_rgb64(faces, fim, wmap, dmap, cs, prm, lights, env, flat, tg, uvs, unlit, (0.1, 0.2, 0.3), False, False)
        b = sh_rgb64(faces, fim, wmap, dmap, cs, prm, lights, env, unlit, (0.1, 0.2, 0.3), False)
        assert float((a - b).abs().max()) <= 1e-12


def _lights_t():
    return torch.tensor([[[0.4, 0.3, 0.2, 0.3, 0.3, 0.3, 0.5, 0.5, -1.0, 0.0, 0.0, 0.0],
                          [0.2, 0.3, 0.4, 0.1, 0.2, 0.3, 0.5, -0.5, -2.0, 0.3, 1.0, 0.0]]], dtype=torch.float64)


def test_fill_back_copy_negates_the_mapped_normal():
    """a copy with corners (-N, P) and tangents (-T, -w), read at the same uv: n' exactly -n' of the original"""
    faces, fim, wmap, dmap, cs, prm, uvs, unlit, tg = _scene(F=2)
    cs_copy, tg_copy = cs.clone(), tg.clone()
    cs_copy[..., :3] = -cs[..., :3]
    tg_copy = -tg
    nm = torch.randn((1, 4, 5, 3), generator=torch.Generator().manual_seed(2), dtype=torch.float64)
    m = map_sample64(faces, fim, wmap, dmap, uvs, nm, False)
    a = mapped_normal64(faces, fim, wmap, dmap, cs, tg, m)[0]
    b = mapped_normal64(faces, fim, wmap, dmap, cs_copy, tg_copy, m)[0]
    assert torch.equal(b, -a)
    # the frame by hand at one pixel: b = sigma (n x t), n' = m_x t + m_y b + m_z n
    n, t, bb = mapped_normal64(faces, fim, wmap, dmap, cs, tg, m)[1:]
    f = int(fim[0, 2, 3])
    sigma = -1.0 if float(tg[0, f, :, 3].sum()) < 0 else 1.0
    assert torch.allclose(bb[0, 2, 3], sigma * torch.linalg.cross(n[0, 2, 3], t[0, 2, 3]), atol=1e-14)
    mm = m[0, 2, 3]
    assert torch.allclose(a[0, 2, 3], mm[0] * t[0, 2, 3] + mm[1] * bb[0, 2, 3] + mm[2] * n[0, 2, 3], atol=1e-14)


# ---------------------------------------------------------------------------------------------------- tangent glue
def _plane(mirror=False):
    v = torch.tensor([[0.0, 0.0, 0.0], [1.0, 0.0, 0.0], [1.0, 1.0, 0.0], [0.0, 1.0, 0.0]], dtype=torch.float64)[None]
    f = torch.tensor([[0, 1, 2], [0, 2, 3]])
    uv = v[0, :, :2].clone()
    if mirror:
        uv[:, 0] = 1 - uv[:, 0]
    n = torch.tensor([0.0, 0.0, 1.0], dtype=torch.float64).expand(1, 4, 3)
    return v, f, uv[f], n


def test_vertex_tangents_plane():
    from neural_renderer_b200 import functional as F
    v, f, uvs, n = _plane()
    t = F.vertex_tangents(v, f, uvs, n)
    want = torch.tensor([1.0 / (1 + 1e-5), 0.0, 0.0, 1.0], dtype=torch.float64).expand(1, 4, 4)
    assert torch.allclose(t, want, atol=1e-12)
    v, f, uvs, n = _plane(mirror=True)
    t = F.vertex_tangents(v, f, uvs, n)
    want = torch.tensor([-1.0 / (1 + 1e-5), 0.0, 0.0, -1.0], dtype=torch.float64).expand(1, 4, 4)
    assert torch.allclose(t, want, atol=1e-12)


def test_vertex_tangents_orthogonal_unreferenced_and_gradcheck():
    from neural_renderer_b200 import functional as F
    g = torch.Generator().manual_seed(4)
    v = torch.randn((2, 7, 3), generator=g, dtype=torch.float64)
    f = torch.tensor([[0, 1, 2], [0, 2, 3], [1, 4, 2], [3, 2, 5]])  # vertex 6 is unreferenced
    uvs = torch.rand((4, 3, 2), generator=g, dtype=torch.float64)
    n = F._vertex_normals_torch(v, f)
    t = F.vertex_tangents(v, f, uvs, n)
    assert t.shape == (2, 7, 4)
    # T perpendicular to n, up to the 1e-5 of the normals' own normalisation (|n| = 1 - O(1e-5))
    assert float((t[..., :3] * n).sum(-1)[:, :6].abs().max()) <= 2e-5
    t1 = F.vertex_tangents(v, f, uvs, n / n.norm(dim=-1, keepdim=True).clamp_min(1e-30))
    assert float((t1[..., :3] * n).sum(-1)[:, :6].abs().max()) <= 1e-12
    assert torch.equal(t[:, 6], torch.tensor([0.0, 0.0, 0.0, 1.0], dtype=torch.float64).expand(2, 4))
    assert set(t[..., 3].flatten().tolist()) <= {-1.0, 1.0}
    # a degenerate UV face (s = 0) is skipped
    uvd = uvs.clone()
    uvd[3] = uvd[3, :1]
    t0 = F.vertex_tangents(v, f[:3], uvs[:3], n)
    td = F.vertex_tangents(v, f, uvd, n)
    assert torch.allclose(td[:, :5], t0[:, :5], atol=1e-12)
    vv, uu, nn = v.clone().requires_grad_(True), uvs.clone().requires_grad_(True), n.clone().requires_grad_(True)
    assert torch.autograd.gradcheck(lambda a, b, c: F.vertex_tangents(a, f, b, c)[..., :3], (vv, uu, nn))


def test_corner_tangents_signs():
    from neural_renderer_b200 import functional as F
    vt = torch.arange(1, 1 + 2 * 4 * 4, dtype=torch.float64).reshape(2, 4, 4)
    f = torch.tensor([[0, 1, 2], [0, 2, 3]])
    fb = torch.cat((f, f.flip(1)))
    c = F.corner_tangents(vt, fb, fill_back=True)
    assert c.shape == (2, 4, 3, 4)
    assert torch.equal(c[:, :2], vt[:, f])
    assert torch.equal(c[:, 2:], -vt[:, f.flip(1)])
    assert torch.equal(F.corner_tangents(vt, f), vt[:, f])
    with pytest.raises(ValueError, match="even"):
        F.corner_tangents(vt, f[:1].expand(3, 3), fill_back=True)


def test_decode_normal_map():
    from neural_renderer_b200 import functional as F
    img = torch.tensor([[[0.5, 0.5, 1.0], [1.0, 0.0, 0.5]]])
    assert torch.equal(F.decode_normal_map(img), torch.tensor([[[0.0, 0.0, 1.0], [1.0, -1.0, 0.0]]]))
    assert torch.equal(F.decode_normal_map(img, green_down=True), torch.tensor([[[0.0, 0.0, 1.0], [1.0, 1.0, 0.0]]]))


# ---------------------------------------------------------------------------------------------------- Python errors
def test_python_argument_errors():
    import neural_renderer_b200 as nr
    faces = torch.rand((1, 4, 3, 3))
    img = torch.rand((8, 8, 3))
    uvs = torch.rand((4, 3, 2))
    cs, prm = torch.rand((1, 4, 3, 6)), torch.rand((1, 16))
    nm, tg = torch.rand((5, 6, 3)), torch.rand((4, 3, 4))
    with pytest.raises(ValueError, match="together"):
        nr.rasterize(faces, img, 8, face_uvs=uvs, corner_shading=cs, shading_params=prm, normal_map=nm)
    with pytest.raises(ValueError, match="together"):
        nr.rasterize(faces, img, 8, face_uvs=uvs, corner_shading=cs, shading_params=prm, corner_tangents=tg)
    with pytest.raises(ValueError, match="Phong"):
        nr.rasterize(faces, img, 8, face_uvs=uvs, normal_map=nm, corner_tangents=tg)
    with pytest.raises(ValueError, match="face_uvs"):
        nr.rasterize(faces, torch.rand((1, 4, 2, 2, 2, 3)), 8, corner_shading=cs, shading_params=prm, normal_map=nm,
                     corner_tangents=tg)
    with pytest.raises(ValueError, match="return_rgb"):
        nr.rasterize_rgbad(faces, img, 8, return_rgb=False, face_uvs=uvs, corner_shading=cs, shading_params=prm,
                           normal_map=nm, corner_tangents=tg)
    for bad in (torch.rand((5, 6, 4)), torch.rand((3, 5, 6, 3)), torch.rand((6, 3)), torch.rand((1, 1, 5, 6, 3))):
        with pytest.raises(ValueError, match="normal_map must have shape"):
            nr.rasterize(faces, img, 8, face_uvs=uvs, corner_shading=cs, shading_params=prm, normal_map=bad,
                         corner_tangents=tg)
    for bad in (torch.rand((4, 3, 3)), torch.rand((5, 3, 4)), torch.rand((3, 4, 3, 4))):
        with pytest.raises(ValueError, match="corner_tangents must have shape"):
            nr.rasterize(faces, img, 8, face_uvs=uvs, corner_shading=cs, shading_params=prm, normal_map=nm,
                         corner_tangents=bad)
    with pytest.raises(TypeError):
        nr.rasterize(faces, img, 8, face_uvs=uvs, corner_shading=cs, shading_params=prm,
                     normal_map=torch.zeros((5, 6, 3), dtype=torch.int32), corner_tangents=tg)
    with pytest.raises(NotImplementedError):  # a valid call on CPU tensors: no CPU implementation
        nr.rasterize(faces, img, 8, face_uvs=uvs, corner_shading=cs, shading_params=prm, normal_map=nm, corner_tangents=tg)


@pytest.mark.parametrize("shading", ["flat", "smooth"])
def test_renderer_normal_map_needs_phong(shading):
    import neural_renderer_b200 as nr
    r = nr.Renderer()
    r.shading = shading
    r.normal_map = torch.rand((4, 4, 3))
    v = torch.rand((1, 4, 3))
    f = torch.tensor([[0, 1, 2], [0, 2, 3]], dtype=torch.int32)
    with pytest.raises(ValueError, match="phong"):
        r.render(v, f, torch.rand((8, 8, 3)), face_uvs=torch.rand((2, 3, 2)))


def test_renderer_normal_map_needs_uvs():
    import neural_renderer_b200 as nr
    r = nr.Renderer()
    r.shading = "phong"
    r.normal_map = torch.rand((4, 4, 3))
    v = torch.rand((1, 4, 3))
    f = torch.tensor([[0, 1, 2], [0, 2, 3]], dtype=torch.int32)
    with pytest.raises(ValueError, match="face_uvs"):
        r.render(v, f, torch.rand((1, 2, 2, 2, 2, 3)))
