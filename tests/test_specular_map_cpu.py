"""CPU: specular maps for Phong shading -- nr_b200_specular_map_args against the header, the new symbols and their
argtypes, the host rejections of nr_b200_forward_specular_map / nr_b200_backward_specular_map (all decided before any
device work), the float64 oracle (oracles_specular_map.py) against oracles_normal_map.py, F.specular_map and the Python
argument errors."""
import ctypes
import os
import subprocess

import pytest
import torch

from oracles_normal_map import nm_rgb64
from oracles_specular_map import sm_rgb64
from test_lights_cpu import _lights
from test_normal_map_cpu import _lights_t, _nm, _scene, _uv
from test_phong_cpu import INVALID, OK_UP_TO_WORKSPACE, UNSUPPORTED, _P, _bwd, _fwd, _phong
from test_sh_cpu import _sh

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    from neural_renderer_b200 import build, _lib
    build.build_library()
    return _lib.load()


def test_specular_map_struct_matches_the_header(tmp_path):
    from neural_renderer_b200 import _lib
    fields = [f[0] for f in _lib.SpecularMapArgs._fields_]
    exprs = ["sizeof(nr_b200_specular_map_args)"] + ["offsetof(nr_b200_specular_map_args, %s)" % f for f in fields] + \
        ["sizeof(nr_b200_normal_map_args)"]
    src = tmp_path / "s.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "nr_b200.h"\nint main(void){'
                   + "".join('printf("%%zu\\n", (size_t)(%s));' % e for e in exprs) + "return 0;}\n")
    exe = tmp_path / "s"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    vals = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert vals[0] == ctypes.sizeof(_lib.SpecularMapArgs) == 32
    assert vals[1:1 + len(fields)] == [getattr(_lib.SpecularMapArgs, f).offset for f in fields] == [0, 4, 8, 12, 16, 24]
    assert vals[-1] == 56  # the normal-map struct is unchanged


def test_new_symbols_are_exported(lib):
    from neural_renderer_b200 import _lib
    out = subprocess.run(["nm", "-D", "--defined-only", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    for n in ("nr_b200_forward_specular_map", "nr_b200_backward_specular_map"):
        assert n in _lib.EXPORTED_SYMBOLS
        fn = getattr(lib, n)
        assert (" T " + n) in out, n
        assert fn.restype is ctypes.c_int
        assert [getattr(t, "_type_", t) for t in fn.argtypes[1:6]] == [_lib.PhongArgs, _lib.LightsArgs, _lib.ShArgs,
                                                                         _lib.NormalMapArgs, _lib.SpecularMapArgs]
        assert fn.argtypes[-1] is ctypes.c_void_p and len(fn.argtypes) == 7


def _sm(struct_size=None, bq=2, hq=4, wq=5, smap=_P, grad=True):
    from neural_renderer_b200 import _lib
    qa = _lib.SpecularMapArgs()
    qa.struct_size = ctypes.sizeof(_lib.SpecularMapArgs) if struct_size is None else struct_size
    qa.map_batch, qa.map_height, qa.map_width = bq, hq, wq
    qa.specular_map = smap
    qa.grad_specular_map = _P + 4 if grad else None  # a gradient buffer needs only 4-byte alignment
    return qa


def _rejections(run, lib):
    from neural_renderer_b200 import _lib
    rgb = _lib.NR_RETURN_RGB | _lib.NR_TEX_UV
    for bq in (1, 2):
        for la in (None, _lights(nl=0, lights=False), _lights(nl=3, bl=1)):
            for sa in (None, _sh(bs=1)):
                for na in (None, _nm(bm=1, bt=2)):
                    assert run(rgb, la=la, sa=sa, na=na, qa=_sm(bq=bq)) == OK_UP_TO_WORKSPACE, bq
    assert run(rgb, qa=_sm(hq=1, wq=1)) == OK_UP_TO_WORKSPACE
    assert run(rgb | _lib.NR_TEX_MIPMAP) == OK_UP_TO_WORKSPACE
    assert run(rgb | _lib.NR_ANTI_ALIASING | _lib.NR_TEX_FILL_BACK) == OK_UP_TO_WORKSPACE
    assert run(rgb, qa=None) == OK_UP_TO_WORKSPACE  # a NULL struct is the normal-map call
    assert run(_lib.NR_RETURN_RGB, qa=None) == OK_UP_TO_WORKSPACE  # ... which needs no UVs without a normal map
    for size in (0, 24, 31, 33, 56):
        assert run(rgb, qa=_sm(struct_size=size)) == INVALID, size
    for b in (0, 3, -1):
        assert run(rgb, qa=_sm(bq=b)) == INVALID, b
    assert run(rgb, qa=_sm(smap=None)) == INVALID
    for off in (4, 8, 12):  # texels are read as aligned 16-byte vectors
        assert run(rgb, qa=_sm(smap=_P + off)) == INVALID, off
    for hq, wq in ((0, 4), (4, 0), (-1, 4)):
        assert run(rgb, qa=_sm(hq=hq, wq=wq)) == INVALID, (hq, wq)
    assert run(_lib.NR_RETURN_RGB) == INVALID  # the map needs NR_TEX_UV (cubes have no UVs)
    assert run(rgb, qa=_sm(hq=32768, wq=16384, bq=1)) == UNSUPPORTED  # 2^31 floats: beyond 32-bit offsets
    assert run(rgb, qa=_sm(hq=16384, wq=16384, bq=2)) == UNSUPPORTED  # 2^30 floats per item, two items
    # everything the normal-map, Phong, light-set and SH calls refuse
    assert run(rgb, na=_nm(struct_size=48)) == INVALID
    assert run(rgb, na=_nm(tg=False)) == INVALID
    assert run(rgb, na=_nm(bm=3)) == INVALID
    assert run(rgb, ph=None) == INVALID
    assert run(rgb, ph=_phong(struct_size=56)) == INVALID
    assert run(rgb, ph=_phong(cs=False)) == INVALID
    assert run(rgb, la=_lights(nl=9)) == INVALID
    assert run(rgb, sa=_sh(bs=3)) == INVALID
    assert run(rgb, sa=_sh(sh=False)) == INVALID
    assert run(_lib.NR_RETURN_ALPHA | _lib.NR_TEX_UV) == INVALID
    assert lib.nr_b200_last_launch_count() == 0


def test_forward_specular_map_rejections(lib):
    from neural_renderer_b200 import _lib

    def run(flags, ph=_phong(), la=None, sa=None, na=None, qa=_sm(), face_light=False):
        return lib.nr_b200_forward_specular_map(ctypes.byref(_uv(_fwd(flags, face_light), flags)),
                                                None if ph is None else ctypes.byref(ph),
                                                None if la is None else ctypes.byref(la),
                                                None if sa is None else ctypes.byref(sa),
                                                None if na is None else ctypes.byref(na),
                                                None if qa is None else ctypes.byref(qa), None)
    _rejections(run, lib)
    assert run(_lib.NR_RETURN_RGB | _lib.NR_TEX_UV, face_light=True) == INVALID
    assert lib.nr_b200_last_launch_count() == 0


def test_backward_specular_map_rejections(lib):
    from neural_renderer_b200 import _lib
    rgb = _lib.NR_RETURN_RGB | _lib.NR_TEX_UV

    def run(flags, ph=_phong(), la=None, sa=None, na=None, qa=_sm(), textures=True):
        return lib.nr_b200_backward_specular_map(ctypes.byref(_uv(_bwd(flags, textures=textures), flags)),
                                                 None if ph is None else ctypes.byref(ph),
                                                 None if la is None else ctypes.byref(la),
                                                 None if sa is None else ctypes.byref(sa),
                                                 None if na is None else ctypes.byref(na),
                                                 None if qa is None else ctypes.byref(qa), None)
    _rejections(run, lib)
    for ok in (rgb | _lib.NR_GRAD_ACCUMULATE, rgb | _lib.NR_BWD_PART_TEXTURES, rgb | _lib.NR_BWD_PART_FACES):
        assert run(ok) == OK_UP_TO_WORKSPACE, hex(ok)
    # grad_specular_map needs the unlit sample s, so `textures`
    no_grads = _phong(grad_cs=False, grad_prm=False)
    assert run(rgb, ph=no_grads, textures=False) == INVALID
    assert run(rgb, ph=no_grads, qa=_sm(grad=False), textures=False) == OK_UP_TO_WORKSPACE
    assert run(rgb, ph=no_grads, na=_nm(grad=False), qa=_sm(), textures=False) == INVALID
    assert run(rgb | _lib.NR_GRAD_INTERIOR) == UNSUPPORTED
    assert lib.nr_b200_last_launch_count() == 0


# ---------------------------------------------------------------------------------------------------- the oracle
@pytest.mark.parametrize("with_nm", [False, True])
def test_constant_map_oracle_is_the_normal_map_oracle(with_nm):
    faces, fim, wmap, dmap, cs, prm, uvs, unlit, tg = _scene()
    g = torch.Generator().manual_seed(3)
    nm = torch.randn((1, 4, 5, 3), generator=g, dtype=torch.float64) * 0.3 + torch.tensor([0, 0, 1.0], dtype=torch.float64)
    flat = torch.zeros((1, 2, 3, 3), dtype=torch.float64)
    flat[..., 2] = 1.0
    sm = torch.ones((1, 3, 7, 4), dtype=torch.float64)
    sm[..., 3] = prm[0, 12]
    sh = torch.randn((1, 9, 3), generator=g, dtype=torch.float64) * 0.2
    lt = _lights_t()
    for lights, env in ((None, None), (lt, None), (None, sh), (lt, sh)):
        a = sm_rgb64(faces, fim, wmap, dmap, cs, prm, lights, env, nm if with_nm else None, tg, sm, uvs, unlit,
                     (0.1, 0.2, 0.3), False, False)
        b = nm_rgb64(faces, fim, wmap, dmap, cs, prm, lights, env, nm if with_nm else flat, tg, uvs, unlit,
                     (0.1, 0.2, 0.3), False, False)
        assert float((a - b).abs().max()) <= 1e-12


def test_oracle_scales_every_highlight_and_keeps_the_diffuse_part():
    """(ks, sigma) constant: rgb = L s + ks * (the highlights of params with shininess sigma)"""
    faces, fim, wmap, dmap, cs, prm, uvs, unlit, tg = _scene(seed=5)
    lt = _lights_t()
    ks, sig = torch.tensor([0.3, 0.6, 1.7], dtype=torch.float64), 21.0
    sm = torch.cat((ks, torch.tensor([sig], dtype=torch.float64))).expand(1, 2, 2, 4)
    a = sm_rgb64(faces, fim, wmap, dmap, cs, prm, lt, None, None, tg, sm, uvs, unlit, (0, 0, 0), False, False)
    diffuse = sm_rgb64(faces, fim, wmap, dmap, cs, prm, lt, None, None, tg, sm * torch.tensor([0, 0, 0, 1.0]), uvs, unlit,
                       (0, 0, 0), False, False)
    prm2 = prm.clone()
    prm2[:, 12] = sig
    full = sm_rgb64(faces, fim, wmap, dmap, cs, prm2, lt, None, None, tg, None, uvs, unlit, (0, 0, 0), False, False)
    assert torch.allclose(a - diffuse, ks[None, :, None, None] * (full - diffuse), atol=1e-12)
    assert float((full - diffuse).abs().max()) > 1e-3  # the scene has highlights


# ---------------------------------------------------------------------------------------------------- F.specular_map
def test_specular_map_packs_and_gradchecks():
    from neural_renderer_b200 import functional as F
    g = torch.Generator().manual_seed(6)
    col = torch.rand((2, 3, 5, 3), generator=g, dtype=torch.float64, requires_grad=True)
    sig = torch.rand((2, 3, 5), generator=g, dtype=torch.float64, requires_grad=True)
    m = F.specular_map(col, sig)
    assert m.shape == (2, 3, 5, 4)
    assert torch.equal(m[..., :3], col) and torch.equal(m[..., 3], sig)
    assert torch.equal(F.specular_map(col, 16.0)[..., 3], torch.full((2, 3, 5), 16.0, dtype=torch.float64))
    assert torch.autograd.gradcheck(F.specular_map, (col, sig))
    logs = torch.zeros((3, 5), dtype=torch.float64, requires_grad=True)  # broadcast over the batch
    assert torch.autograd.gradcheck(lambda c, s: F.specular_map(c, s.exp()), (col, logs))
    with pytest.raises(ValueError, match="color"):
        F.specular_map(torch.rand((3, 5, 4)), 1.0)
    with pytest.raises(ValueError, match="shininess"):
        F.specular_map(torch.rand((3, 5, 3)), torch.rand((4, 5)))


# ---------------------------------------------------------------------------------------------------- Python errors
def test_python_argument_errors():
    import neural_renderer_b200 as nr
    faces = torch.rand((1, 4, 3, 3))
    img = torch.rand((8, 8, 3))
    uvs = torch.rand((4, 3, 2))
    cs, prm = torch.rand((1, 4, 3, 6)), torch.rand((1, 16))
    sm = torch.rand((5, 6, 4))
    with pytest.raises(ValueError, match="Phong"):
        nr.rasterize(faces, img, 8, face_uvs=uvs, specular_map=sm)
    with pytest.raises(ValueError, match="face_uvs"):
        nr.rasterize(faces, torch.rand((1, 4, 2, 2, 2, 3)), 8, corner_shading=cs, shading_params=prm, specular_map=sm)
    with pytest.raises(ValueError, match="return_rgb"):
        nr.rasterize_rgbad(faces, img, 8, return_rgb=False, face_uvs=uvs, corner_shading=cs, shading_params=prm,
                           specular_map=sm)
    for bad in (torch.rand((5, 6, 3)), torch.rand((3, 5, 6, 4)), torch.rand((6, 4)), torch.rand((1, 1, 5, 6, 4)),
                torch.rand((0, 6, 4))):
        with pytest.raises(ValueError, match="specular_map must have shape"):
            nr.rasterize(faces, img, 8, face_uvs=uvs, corner_shading=cs, shading_params=prm, specular_map=bad)
    with pytest.raises(TypeError):
        nr.rasterize(faces, img, 8, face_uvs=uvs, corner_shading=cs, shading_params=prm,
                     specular_map=torch.zeros((5, 6, 4), dtype=torch.int32))
    with pytest.raises(NotImplementedError):  # a valid call on CPU tensors: no CPU implementation
        nr.rasterize(faces, img, 8, face_uvs=uvs, corner_shading=cs, shading_params=prm, specular_map=sm)


@pytest.mark.parametrize("shading", ["flat", "smooth"])
def test_renderer_specular_map_needs_phong(shading):
    import neural_renderer_b200 as nr
    r = nr.Renderer()
    r.shading = shading
    r.specular_map = torch.rand((4, 4, 4))
    v = torch.rand((1, 4, 3))
    f = torch.tensor([[0, 1, 2], [0, 2, 3]], dtype=torch.int32)
    with pytest.raises(ValueError, match="phong"):
        r.render(v, f, torch.rand((8, 8, 3)), face_uvs=torch.rand((2, 3, 2)))


def test_renderer_specular_map_needs_uvs():
    import neural_renderer_b200 as nr
    r = nr.Renderer()
    r.shading = "phong"
    r.specular_map = torch.rand((4, 4, 4))
    v = torch.rand((1, 4, 3))
    f = torch.tensor([[0, 1, 2], [0, 2, 3]], dtype=torch.int32)
    with pytest.raises(ValueError, match="face_uvs"):
        r.render(v, f, torch.rand((1, 2, 2, 2, 2, 3)))
