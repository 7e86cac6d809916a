"""CPU: Phong shading -- nr_b200_phong_args against the header, the new symbols, the host rejections of nr_b200_forward_phong,
nr_b200_backward_phong and the corner-shading glue (all decided before any device work), the unchanged forward / backward
structs, the torch formulations of F.corner_shading / F.phong_params against float64 loops, and the Python argument errors."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# Fake, never dereferenced device addresses (as test_smooth_cpu.py): a complete argument set gets as far as the workspace
# check (NR_ERR_WORKSPACE, no workspace given); each broken one must stop earlier.
_P = 0x10000
OK_UP_TO_WORKSPACE, INVALID, UNSUPPORTED = -2, -1, -4


@pytest.fixture(scope="module")
def lib():
    from neural_renderer_b200 import build, _lib
    build.build_library()
    return _lib.load()


def test_phong_struct_matches_the_header_and_old_structs_are_unchanged(tmp_path):
    from neural_renderer_b200 import _lib
    fields = [f[0] for f in _lib.PhongArgs._fields_]
    exprs = ["sizeof(nr_b200_phong_args)"] + ["offsetof(nr_b200_phong_args, %s)" % f for f in fields] + \
        ["sizeof(nr_b200_forward_args)", "offsetof(nr_b200_forward_args, corner_light)", "sizeof(nr_b200_backward_args)",
         "offsetof(nr_b200_backward_args, grad_face_uvs)"]
    src = tmp_path / "s.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "nr_b200.h"\nint main(void){'
                   + "".join('printf("%%zu\\n", (size_t)(%s));' % e for e in exprs) + "return 0;}\n")
    exe = tmp_path / "s"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    vals = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert vals[0] == ctypes.sizeof(_lib.PhongArgs) == 48
    assert vals[1:1 + len(fields)] == [getattr(_lib.PhongArgs, f).offset for f in fields]
    fsize, fcl, bsize, buv = vals[1 + len(fields):]
    # the Phong pointers travel in their own struct: corner_light stays the forward struct's last field
    assert fsize == ctypes.sizeof(_lib.ForwardArgs) == fcl + 8 and fcl == _lib.ForwardArgs.corner_light.offset
    assert bsize == ctypes.sizeof(_lib.BackwardArgs) == buv + 8 and buv == _lib.BackwardArgs.grad_face_uvs.offset


def test_new_symbols_are_exported(lib):
    from neural_renderer_b200 import _lib
    names = ("nr_b200_forward_phong", "nr_b200_backward_phong", "nr_b200_corner_shading", "nr_b200_corner_shading_backward")
    for n in names:
        assert n in _lib.EXPORTED_SYMBOLS
        assert getattr(lib, n) is not None
    out = subprocess.run(["nm", "-D", "--defined-only", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    for n in names:
        assert (" T " + n) in out, n


def _phong(struct_size=None, cs=True, prm=True, bc=2, bp=2, grad_cs=True, grad_prm=True):
    from neural_renderer_b200 import _lib
    ph = _lib.PhongArgs()
    ph.struct_size = ctypes.sizeof(_lib.PhongArgs) if struct_size is None else struct_size
    ph.shading_batch, ph.params_batch = bc, bp
    ph.corner_shading = _P if cs else None
    ph.params = _P if prm else None
    ph.grad_corner_shading = _P if grad_cs else None
    ph.grad_params = _P if grad_prm else None
    return ph


def _fwd(flags, face_light=False, corner_light=False):
    from neural_renderer_b200 import _lib
    a = _lib.ForwardArgs()
    a.struct_size = ctypes.sizeof(_lib.ForwardArgs)
    a.flags = flags
    a.batch_size, a.num_faces, a.raster_size, a.texture_size = 2, 4, 16, 2
    a.near_, a.far_, a.eps = 0.1, 100.0, 1e-4
    a.faces = a.textures = a.face_index_map = a.weight_map = a.depth_map = a.rgb_map = a.alpha_map = _P
    a.face_light = _P if face_light else None
    a.corner_light = _P if corner_light else None
    return a


def _bwd(flags, face_light=False, textures=True):
    from neural_renderer_b200 import _lib
    a = _lib.BackwardArgs()
    a.struct_size = ctypes.sizeof(_lib.BackwardArgs)
    a.flags = flags
    a.batch_size, a.num_faces, a.raster_size, a.texture_size = 2, 4, 16, 2
    a.eps = 1e-4
    a.faces = a.face_index_map = a.weight_map = a.depth_map = a.rgb_map = a.grad_faces = a.grad_textures = _P
    a.textures = _P if textures else None
    a.face_light = _P if face_light else None
    return a


def _common_rejections(run, lib):
    from neural_renderer_b200 import _lib
    rgb, alpha = _lib.NR_RETURN_RGB, _lib.NR_RETURN_ALPHA
    for bc, bp in ((2, 2), (1, 1), (1, 2), (2, 1)):
        assert run(rgb, ph=_phong(bc=bc, bp=bp)) == OK_UP_TO_WORKSPACE, (bc, bp)
    assert run(rgb | _lib.NR_ANTI_ALIASING) == OK_UP_TO_WORKSPACE
    assert run(rgb, ph=None) == INVALID
    for size in (0, 40, 47, 49, 56):
        assert run(rgb, ph=_phong(struct_size=size)) == INVALID, size
    assert run(rgb, ph=_phong(cs=False)) == INVALID
    assert run(rgb, ph=_phong(prm=False)) == INVALID
    for bc, bp in ((0, 2), (3, 2), (2, 0), (2, 3), (-1, 1)):
        assert run(rgb, ph=_phong(bc=bc, bp=bp)) == INVALID, (bc, bp)
    assert run(rgb, face_light=True) == INVALID
    assert run(alpha) == INVALID
    assert lib.nr_b200_last_launch_count() == 0


def test_forward_phong_rejections(lib):
    def run(flags, ph=_phong(), face_light=False, corner_light=False):
        return lib.nr_b200_forward_phong(ctypes.byref(_fwd(flags, face_light, corner_light)),
                                         None if ph is None else ctypes.byref(ph), None)
    from neural_renderer_b200 import _lib
    _common_rejections(run, lib)
    assert run(_lib.NR_RETURN_RGB, corner_light=True) == INVALID
    # the plain forward is unchanged: the same call without Phong
    assert lib.nr_b200_forward(ctypes.byref(_fwd(_lib.NR_RETURN_RGB)), None) == OK_UP_TO_WORKSPACE


def test_backward_phong_rejections(lib):
    from neural_renderer_b200 import _lib
    rgb, acc = _lib.NR_RETURN_RGB, _lib.NR_GRAD_ACCUMULATE

    def run(flags, ph=_phong(), face_light=False, textures=True):
        return lib.nr_b200_backward_phong(ctypes.byref(_bwd(flags, face_light, textures)),
                                          None if ph is None else ctypes.byref(ph), None)
    _common_rejections(run, lib)
    for ok in (rgb | acc, rgb | _lib.NR_BWD_PART_TEXTURES, rgb | _lib.NR_BWD_PART_FACES):
        assert run(ok) == OK_UP_TO_WORKSPACE, hex(ok)
    # both Phong gradients need the unlit sample s, so `textures`
    assert run(rgb, textures=False) == INVALID
    assert run(rgb, ph=_phong(grad_cs=False), textures=False) == INVALID
    assert run(rgb, ph=_phong(grad_prm=False), textures=False) == INVALID
    assert run(rgb, ph=_phong(grad_cs=False, grad_prm=False), textures=False) == OK_UP_TO_WORKSPACE
    # no vertex gradient through l_k of the Phong normal and position
    assert run(rgb | _lib.NR_GRAD_INTERIOR) == UNSUPPORTED
    assert lib.nr_b200_last_launch_count() == 0
    assert lib.nr_b200_backward(ctypes.byref(_bwd(rgb | _lib.NR_GRAD_INTERIOR)), None) == OK_UP_TO_WORKSPACE


def test_corner_shading_glue_rejections(lib):
    from neural_renderer_b200 import _lib
    fb = _lib.NR_TEX_FILL_BACK
    fwd = lambda n=_P, v=_P, f=_P, B=2, Nv=5, Nf=4, flags=0, out=_P: lib.nr_b200_corner_shading(n, v, f, B, Nv, Nf, flags,
                                                                                                 out, None)
    bwd = lambda f=_P, g=_P, B=2, Nv=5, Nf=4, flags=0, gn=_P, gv=_P: lib.nr_b200_corner_shading_backward(f, g, B, Nv, Nf, flags,
                                                                                                         gn, gv, None)
    for kw in ({"n": None}, {"v": None}, {"f": None}, {"out": None}, {"B": 0}, {"Nv": 0}, {"Nf": 0}, {"B": 65536},
               {"Nf": 5, "flags": fb}):
        assert fwd(**kw) == INVALID, kw
    for kw in ({"f": None}, {"g": None}, {"gn": None, "gv": None}, {"B": 0}, {"Nv": 0}, {"Nf": 0}, {"Nf": 3, "flags": fb}):
        assert bwd(**kw) == INVALID, kw
    assert lib.nr_b200_last_launch_count() == 0


# ---------------------------------------------------------------------------------------------- torch formulations
def _hand_corner_shading(n, v, faces, fill_back):
    n, v, faces = np.asarray(n, np.float64), np.asarray(v, np.float64), np.asarray(faces)
    F = len(faces)
    out = np.zeros((F, 3, 6))
    for f, tri in enumerate(faces):
        sgn = -1.0 if (fill_back and f >= F // 2) else 1.0
        for k, i in enumerate(tri):
            if 0 <= i < len(n):
                out[f, k, :3] = sgn * n[i]
                out[f, k, 3:] = v[i]
    return out


@pytest.mark.parametrize("fill_back", [False, True])
def test_corner_shading_formula(fill_back):
    from neural_renderer_b200 import functional as F
    g = torch.Generator().manual_seed(2)
    n = torch.randn((2, 7, 3), generator=g, dtype=torch.float64)
    v = torch.randn((2, 7, 3), generator=g, dtype=torch.float64)
    front = torch.tensor([[0, 1, 2], [2, 3, 4], [4, 5, 6], [6, 7, -1]])  # indices 7 and -1 are out of range: zeros
    faces = torch.cat((front, front.flip(1))) if fill_back else front
    got = F.corner_shading(n, v, faces, fill_back=fill_back)
    assert tuple(got.shape) == (2, faces.shape[0], 3, 6)
    for b in range(2):
        np.testing.assert_allclose(got[b].numpy(), _hand_corner_shading(n[b], v[b], faces, fill_back), rtol=0, atol=0)
    # per-item index sets
    fb = torch.stack((faces, faces.flip(0)))
    np.testing.assert_allclose(F.corner_shading(n, v, fb, fill_back=fill_back)[1].numpy(),
                               _hand_corner_shading(n[1], v[1], faces.flip(0), fill_back), rtol=0, atol=0)
    with pytest.raises(ValueError):
        F.corner_shading(n, v, front[:3], fill_back=True)


def test_phong_params_layout_and_gradients():
    from neural_renderer_b200 import functional as F
    p = F.phong_params(0.3, 0.6, 0.2, (1.0, 0.5, 0.25), (0.5, 1.0, 0.75), (0.25, 0.5, 1.0), (0.1, 0.9, -0.4), 32.0,
                       (0.0, 0.5, -3.0))
    want = np.concatenate([0.3 * np.array([1.0, 0.5, 0.25]), 0.6 * np.array([0.5, 1.0, 0.75]), [0.1, 0.9, -0.4],
                           0.2 * np.array([0.25, 0.5, 1.0]), [32.0], [0.0, 0.5, -3.0]])
    assert tuple(p.shape) == (1, 16) and p.dtype == torch.float32
    np.testing.assert_allclose(p[0].numpy(), want, rtol=1e-6)
    # tensor-valued attributes: a per-item direction, a tensor shininess and eye receive gradients
    d = torch.tensor([[0.0, 1.0, 0.0], [0.3, 0.3, 0.3]], requires_grad=True)
    sig = torch.tensor(16.0, requires_grad=True)
    eye = torch.tensor([0.0, 0.0, -2.0], requires_grad=True)
    p = F.phong_params(direction=d, shininess=sig, eye=eye)
    assert tuple(p.shape) == (2, 16)
    w = torch.arange(32, dtype=torch.float32).reshape(2, 16)
    (p * w).sum().backward()
    np.testing.assert_allclose(d.grad.numpy(), w[:, 6:9].numpy())
    assert float(sig.grad) == float(w[:, 12].sum())
    np.testing.assert_allclose(eye.grad.numpy(), w[:, 13:16].sum(0).numpy())
    with pytest.raises(ValueError):
        F.phong_params(direction=torch.zeros(2, 3), eye=torch.zeros(3, 3))


# ----------------------------------------------------------------------------------------------------- Python errors
def _cpu_scene():
    faces = torch.rand((1, 4, 3, 3))
    tex = torch.rand((1, 4, 2, 2, 2, 3))
    cs = torch.rand((1, 4, 3, 6))
    prm = torch.rand((1, 16))
    return faces, tex, cs, prm


def test_python_argument_errors():
    import neural_renderer_b200 as nr
    faces, tex, cs, prm = _cpu_scene()
    with pytest.raises(ValueError, match="together"):
        nr.rasterize(faces, tex, 8, corner_shading=cs)
    with pytest.raises(ValueError, match="together"):
        nr.rasterize(faces, tex, 8, shading_params=prm)
    with pytest.raises(ValueError, match="exclusive"):
        nr.rasterize(faces, tex, 8, corner_shading=cs, shading_params=prm, face_light=torch.rand((1, 4, 3)))
    with pytest.raises(ValueError, match="exclusive"):
        nr.rasterize(faces, tex, 8, corner_shading=cs, shading_params=prm, corner_light=torch.rand((1, 4, 3, 3)))
    with pytest.raises(ValueError, match="interior_gradient"):
        nr.rasterize(faces, tex, 8, corner_shading=cs, shading_params=prm, interior_gradient=True)
    with pytest.raises(ValueError, match="corner_shading must have shape"):
        nr.rasterize(faces, tex, 8, corner_shading=cs[:, :3], shading_params=prm)
    with pytest.raises(ValueError, match="shading_params must have shape"):
        nr.rasterize(faces, tex, 8, corner_shading=cs, shading_params=prm[:, :15])
    with pytest.raises(NotImplementedError):  # a valid call on CPU tensors: no CPU implementation
        nr.rasterize(faces, tex, 8, corner_shading=cs, shading_params=prm)


def test_renderer_phong_with_interior_gradient_raises():
    import neural_renderer_b200 as nr
    r = nr.Renderer()
    r.shading, r.interior_gradient = 'phong', True
    v = torch.rand((1, 4, 3))
    f = torch.tensor([[[0, 1, 2], [1, 2, 3]]], dtype=torch.int32)
    with pytest.raises(ValueError, match="interior_gradient"):
        r.render(v, f, torch.rand((1, 2, 2, 2, 2, 3)))
    assert (r.light_intensity_specular, r.light_color_specular, r.light_shininess) == (0.2, [1, 1, 1], 64.0)
