"""CPU: light sets for Phong shading -- nr_b200_lights_args against the header, the new symbols, the host rejections of
nr_b200_forward_lights / nr_b200_backward_lights (all decided before any device work), the light-record builders of
functional.py, the Python argument errors, and the float64 oracle (oracles_lights.py) against oracles_phong.py."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch

from oracles_lights import lights_terms64, lights_rgb64
from oracles_phong import phong_rgb64, phong_terms64
from test_phong_cpu import INVALID, OK_UP_TO_WORKSPACE, UNSUPPORTED, _P, _bwd, _fwd, _phong

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    from neural_renderer_b200 import build, _lib
    build.build_library()
    return _lib.load()


def test_lights_struct_matches_the_header(tmp_path):
    from neural_renderer_b200 import _lib
    fields = [f[0] for f in _lib.LightsArgs._fields_]
    exprs = ["sizeof(nr_b200_lights_args)"] + ["offsetof(nr_b200_lights_args, %s)" % f for f in fields] + \
        ["sizeof(nr_b200_phong_args)"]
    src = tmp_path / "s.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "nr_b200.h"\nint main(void){'
                   + "".join('printf("%%zu\\n", (size_t)(%s));' % e for e in exprs) + "return 0;}\n")
    exe = tmp_path / "s"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    vals = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert vals[0] == ctypes.sizeof(_lib.LightsArgs) == 32
    assert vals[1:1 + len(fields)] == [getattr(_lib.LightsArgs, f).offset for f in fields]
    assert vals[-1] == ctypes.sizeof(_lib.PhongArgs) == 48  # the Phong struct is unchanged


def test_new_symbols_are_exported(lib):
    from neural_renderer_b200 import _lib
    names = ("nr_b200_forward_lights", "nr_b200_backward_lights")
    out = subprocess.run(["nm", "-D", "--defined-only", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    for n in names:
        assert n in _lib.EXPORTED_SYMBOLS
        assert getattr(lib, n) is not None
        assert (" T " + n) in out, n


def _lights(struct_size=None, nl=2, bl=2, lights=True, grad=True):
    from neural_renderer_b200 import _lib
    la = _lib.LightsArgs()
    la.struct_size = ctypes.sizeof(_lib.LightsArgs) if struct_size is None else struct_size
    la.lights_batch, la.num_lights = bl, nl
    la.lights = _P if lights else None
    la.grad_lights = _P if grad else None
    return la


def _rejections(run, lib):
    from neural_renderer_b200 import _lib
    rgb = _lib.NR_RETURN_RGB
    for nl, bl in ((1, 1), (2, 2), (8, 1), (8, 2), (0, 2)):
        assert run(rgb, la=_lights(nl=nl, bl=bl)) == OK_UP_TO_WORKSPACE, (nl, bl)
    assert run(rgb, la=None) == OK_UP_TO_WORKSPACE  # a NULL light set is the Phong call
    assert run(rgb, la=_lights(nl=0, lights=False)) == OK_UP_TO_WORKSPACE
    for size in (0, 24, 31, 33, 48):
        assert run(rgb, la=_lights(struct_size=size)) == INVALID, size
    for nl in (-1, 9, 64):
        assert run(rgb, la=_lights(nl=nl)) == INVALID, nl
    assert run(rgb, la=_lights(lights=False)) == INVALID
    for bl in (0, 3, -1):
        assert run(rgb, la=_lights(bl=bl)) == INVALID, bl
    assert run(rgb, ph=None) == INVALID
    assert run(rgb, ph=_phong(struct_size=56)) == INVALID
    assert run(rgb, ph=_phong(cs=False)) == INVALID
    assert run(_lib.NR_RETURN_ALPHA) == INVALID
    assert lib.nr_b200_last_launch_count() == 0


def test_forward_lights_rejections(lib):
    def run(flags, ph=_phong(), la=_lights()):
        return lib.nr_b200_forward_lights(ctypes.byref(_fwd(flags)), None if ph is None else ctypes.byref(ph),
                                          None if la is None else ctypes.byref(la), None)
    _rejections(run, lib)


def test_backward_lights_rejections(lib):
    from neural_renderer_b200 import _lib
    rgb = _lib.NR_RETURN_RGB

    def run(flags, ph=_phong(), la=_lights(), textures=True):
        return lib.nr_b200_backward_lights(ctypes.byref(_bwd(flags, textures=textures)),
                                           None if ph is None else ctypes.byref(ph),
                                           None if la is None else ctypes.byref(la), None)
    _rejections(run, lib)
    for ok in (rgb | _lib.NR_GRAD_ACCUMULATE, rgb | _lib.NR_BWD_PART_TEXTURES, rgb | _lib.NR_BWD_PART_FACES):
        assert run(ok) == OK_UP_TO_WORKSPACE, hex(ok)
    # grad_lights needs the unlit sample s, so `textures` (also with NL = 0)
    no_grads = _phong(grad_cs=False, grad_prm=False)
    assert run(rgb, ph=no_grads, textures=False) == INVALID
    assert run(rgb, ph=no_grads, la=_lights(nl=0), textures=False) == INVALID
    assert run(rgb, ph=no_grads, la=_lights(grad=False), textures=False) == OK_UP_TO_WORKSPACE
    assert run(rgb | _lib.NR_GRAD_INTERIOR) == UNSUPPORTED
    assert lib.nr_b200_last_launch_count() == 0


# ---------------------------------------------------------------------------------------------- light records
def test_light_records_layout_and_gradients():
    from neural_renderer_b200 import functional as F
    d = F.directional_light((0.1, 0.9, -0.4), 0.6, (0.5, 1.0, 0.75), 0.2, (0.25, 0.5, 1.0))
    want = np.concatenate([0.6 * np.array([0.5, 1.0, 0.75]), 0.2 * np.array([0.25, 0.5, 1.0]), [0.1, 0.9, -0.4],
                           [0.0, 0.0, 0.0]])
    assert tuple(d.shape) == (1, 12) and d.dtype == torch.float32
    np.testing.assert_allclose(d[0].numpy(), want, rtol=1e-6)
    assert F.directional_light((0.1, 0.9, -0.4), 0.6, (0.5, 1.0, 0.75), 0.2, (0.25, 0.5, 1.0)) is d  # cached
    pos = torch.tensor([[0.0, 1.0, -2.0], [0.3, 0.3, 0.3]], requires_grad=True)
    f = torch.tensor(0.5, requires_grad=True)
    pt = F.point_light(pos, intensity=0.8, falloff=f)
    assert tuple(pt.shape) == (2, 12)
    np.testing.assert_allclose(pt[:, 9:].detach().numpy(), [[0.5, 1.0, 0.0]] * 2)
    s = F.light_set(d, pt, F.point_light((1.0, 2.0, 3.0)))
    assert tuple(s.shape) == (2, 3, 12)
    w = torch.arange(72, dtype=torch.float32).reshape(2, 3, 12)
    (s * w).sum().backward()
    np.testing.assert_allclose(pos.grad.numpy(), w[:, 1, 6:9].numpy())
    assert float(f.grad) == float(w[:, 1, 9].sum())
    with pytest.raises(ValueError):
        F.light_set(*([d] * 9))
    with pytest.raises(ValueError):
        F.light_set()
    with pytest.raises(ValueError):
        F.point_light(torch.zeros(2, 3), color=torch.ones(3, 3))


# ---------------------------------------------------------------------------------------------------- Python errors
def test_python_argument_errors():
    import neural_renderer_b200 as nr
    faces = torch.rand((1, 4, 3, 3))
    tex = torch.rand((1, 4, 2, 2, 2, 3))
    cs, prm = torch.rand((1, 4, 3, 6)), torch.rand((1, 16))
    lt = torch.rand((1, 2, 12))
    with pytest.raises(ValueError, match="Phong"):
        nr.rasterize(faces, tex, 8, lights=lt)
    with pytest.raises(ValueError, match="lights must have shape"):
        nr.rasterize(faces, tex, 8, corner_shading=cs, shading_params=prm, lights=torch.rand((1, 9, 12)))
    with pytest.raises(ValueError, match="lights must have shape"):
        nr.rasterize(faces, tex, 8, corner_shading=cs, shading_params=prm, lights=torch.rand((1, 2, 11)))
    with pytest.raises(TypeError):
        nr.rasterize(faces, tex, 8, corner_shading=cs, shading_params=prm, lights=[[0.0] * 12])
    with pytest.raises(NotImplementedError):  # a valid call on CPU tensors: no CPU implementation
        nr.rasterize(faces, tex, 8, corner_shading=cs, shading_params=prm, lights=lt)


@pytest.mark.parametrize("shading", ["flat", "smooth"])
def test_renderer_lights_need_phong(shading):
    import neural_renderer_b200 as nr
    from neural_renderer_b200 import functional as F
    r = nr.Renderer()
    assert r.lights == []
    r.shading = shading
    r.lights = [F.point_light((0.0, 1.0, -2.0))]
    v = torch.rand((1, 4, 3))
    f = torch.tensor([[[0, 1, 2], [1, 2, 3]]], dtype=torch.int32)
    with pytest.raises(ValueError, match="phong"):
        r.render(v, f, torch.rand((1, 2, 2, 2, 2, 3)))


# ---------------------------------------------------------------------------------------------- float64 oracle
def _oracle_scene(B=2, S=12, F=5, seed=0):
    g = torch.Generator().manual_seed(seed)
    faces = torch.rand((B, F, 3, 3), generator=g, dtype=torch.float64)
    faces[..., 2] += 1.0
    fim = torch.randint(-1, F, (B, S, S), generator=g, dtype=torch.int32)
    wmap = torch.rand((B, 3, S, S), generator=g, dtype=torch.float64)
    wmap = wmap / wmap.sum(1, keepdim=True)
    dmap = torch.rand((B, S, S), generator=g, dtype=torch.float64) + 1.0
    n = torch.randn((B, F, 3, 3), generator=g, dtype=torch.float64)
    n[..., 2] = -(n[..., 2].abs() + 1.0)
    cs = torch.cat((n, faces), dim=-1)
    prm = torch.tensor([[0.3, 0.25, 0.2, 0.6, 0.7, 0.8, 0.3, 0.5, -1.0, 0.6, 0.5, 0.4, 16.0, 0.2, -0.1, -4.0]],
                       dtype=torch.float64).expand(B, 16)
    unlit = torch.rand((B, 3, S, S), generator=g, dtype=torch.float64)
    return faces, fim, wmap, dmap, cs, prm, unlit


def test_oracle_without_lights_and_with_one_directional_light_is_phong():
    faces, fim, wmap, dmap, cs, prm, unlit = _oracle_scene()
    bg = (0.1, 0.2, 0.3)
    want = phong_rgb64(faces, fim, wmap, dmap, cs, prm, unlit, bg, False)
    for lights in (None, torch.zeros((1, 0, 12), dtype=torch.float64)):
        got = lights_rgb64(faces, fim, wmap, dmap, cs, prm, lights, unlit, bg, False)
        assert float((got - want).abs().max()) <= 1e-12
    # params' light moved into a directional record, params D = K = 0
    prm0 = prm.clone()
    prm0[:, 3:6] = 0
    prm0[:, 9:12] = 0
    rec = torch.cat((prm[:1, 3:6], prm[:1, 9:12], prm[:1, 6:9], torch.zeros((1, 3), dtype=torch.float64)), dim=1)[:, None]
    got = lights_rgb64(faces, fim, wmap, dmap, cs, prm0, rec, unlit, bg, True)
    assert float((got - phong_rgb64(faces, fim, wmap, dmap, cs, prm, unlit, bg, True)).abs().max()) <= 1e-12
    L, spc = lights_terms64(faces, fim, wmap, dmap, cs, prm, None)
    L0, h0, K0 = phong_terms64(faces, fim, wmap, dmap, cs, prm)
    assert float((L - L0).abs().max()) <= 1e-12 and float((spc - K0 * h0[..., None]).abs().max()) <= 1e-12


def test_oracle_point_light_by_hand():
    """one covered pixel, one point light: the header's expression written out with numpy"""
    faces, fim, wmap, dmap, cs, prm, unlit = _oracle_scene(B=1, S=4, F=2, seed=3)
    fim[:] = 1
    rec = torch.tensor([[[0.5, 0.4, 0.3, 0.7, 0.6, 0.5, 0.4, -0.3, -2.0, 0.8, 1.0, 0.0]]], dtype=torch.float64)
    L, spc = lights_terms64(faces, fim, wmap, dmap, cs, prm, rec)
    z = faces[0, 1, :, 2].numpy()
    w = wmap[0, :, 2, 1].numpy()
    lam = w * (float(dmap[0, 2, 1]) / z)
    C = cs[0, 1].numpy()
    n, p = lam @ C[:, :3], lam @ C[:, 3:]
    P = prm[0].numpy()
    nrm = lambda x: x / (np.linalg.norm(x) + 1e-5)
    nh, vh = nrm(n), nrm(P[13:16] - p)

    def h(c, lh):
        q = max(float((2 * (nh @ lh) * nh - lh) @ vh), 0.0)
        return q ** P[12] if (c > 0 and q > 0) else 0.0
    c0 = nh @ P[6:9]
    u = rec[0, 0, 6:9].numpy() - p
    r = np.linalg.norm(u)
    lh = u / (r + 1e-5)
    c1 = nh @ lh
    a = 1 / (1 + 0.8 * r * r)
    wantL = P[0:3] + P[3:6] * max(c0, 0) + rec[0, 0, 0:3].numpy() * a * max(c1, 0)
    wantS = P[9:12] * h(c0, nrm(P[6:9])) + rec[0, 0, 3:6].numpy() * a * h(c1, lh)
    np.testing.assert_allclose(L[0, 2, 1].numpy(), wantL, rtol=1e-12)
    np.testing.assert_allclose(spc[0, 2, 1].numpy(), wantS, rtol=1e-12, atol=1e-15)
