"""CPU: SH environment lighting for Phong shading -- nr_b200_sh_args against the header, the new symbols, the host
rejections of nr_b200_forward_sh / nr_b200_backward_sh (all decided before any device work), the Python argument errors,
the float64 oracle (oracles_sh.py) against oracles_lights.py, and F.sh_from_environment_map against analytic cases."""
import ctypes
import math
import os
import subprocess

import numpy as np
import pytest
import torch

from oracles_lights import lights_rgb64
from oracles_sh import C0, sh_basis64, sh_rgb64, sh_terms64
from test_lights_cpu import _lights, _oracle_scene
from test_phong_cpu import INVALID, OK_UP_TO_WORKSPACE, UNSUPPORTED, _P, _bwd, _fwd, _phong

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    from neural_renderer_b200 import build, _lib
    build.build_library()
    return _lib.load()


def test_sh_struct_matches_the_header(tmp_path):
    from neural_renderer_b200 import _lib
    fields = [f[0] for f in _lib.ShArgs._fields_]
    exprs = ["sizeof(nr_b200_sh_args)"] + ["offsetof(nr_b200_sh_args, %s)" % f for f in fields] + \
        ["sizeof(nr_b200_lights_args)", "sizeof(nr_b200_phong_args)"]
    src = tmp_path / "s.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "nr_b200.h"\nint main(void){'
                   + "".join('printf("%%zu\\n", (size_t)(%s));' % e for e in exprs) + "return 0;}\n")
    exe = tmp_path / "s"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    vals = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert vals[0] == ctypes.sizeof(_lib.ShArgs) == 24
    assert vals[1:1 + len(fields)] == [getattr(_lib.ShArgs, f).offset for f in fields] == [0, 4, 8, 16]
    assert vals[-2:] == [32, 48]  # the light-set and Phong structs are unchanged


def test_new_symbols_are_exported(lib):
    from neural_renderer_b200 import _lib
    names = ("nr_b200_forward_sh", "nr_b200_backward_sh")
    out = subprocess.run(["nm", "-D", "--defined-only", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    for n in names:
        assert n in _lib.EXPORTED_SYMBOLS
        assert getattr(lib, n) is not None
        assert (" T " + n) in out, n


def _sh(struct_size=None, bs=2, sh=True, grad=True):
    from neural_renderer_b200 import _lib
    sa = _lib.ShArgs()
    sa.struct_size = ctypes.sizeof(_lib.ShArgs) if struct_size is None else struct_size
    sa.sh_batch = bs
    sa.sh = _P if sh else None
    sa.grad_sh = _P if grad else None
    return sa


def _rejections(run, lib):
    from neural_renderer_b200 import _lib
    rgb = _lib.NR_RETURN_RGB
    for bs in (1, 2):
        for la in (None, _lights(nl=0, lights=False), _lights(nl=3, bl=1)):
            assert run(rgb, la=la, sa=_sh(bs=bs)) == OK_UP_TO_WORKSPACE, bs
    assert run(rgb, sa=None) == OK_UP_TO_WORKSPACE  # a NULL struct is the light-set call
    assert run(rgb | _lib.NR_ANTI_ALIASING) == OK_UP_TO_WORKSPACE
    for size in (0, 16, 23, 25, 32):
        assert run(rgb, sa=_sh(struct_size=size)) == INVALID, size
    for bs in (0, 3, -1):
        assert run(rgb, sa=_sh(bs=bs)) == INVALID, bs
    assert run(rgb, sa=_sh(sh=False)) == INVALID
    # everything the Phong and light-set calls refuse
    assert run(rgb, ph=None) == INVALID
    assert run(rgb, ph=_phong(struct_size=56)) == INVALID
    assert run(rgb, ph=_phong(cs=False)) == INVALID
    assert run(rgb, ph=_phong(prm=False)) == INVALID
    assert run(rgb, ph=_phong(bc=3)) == INVALID
    assert run(rgb, la=_lights(nl=9)) == INVALID
    assert run(rgb, la=_lights(struct_size=24)) == INVALID
    assert run(rgb, la=_lights(lights=False)) == INVALID
    assert run(_lib.NR_RETURN_ALPHA) == INVALID
    assert lib.nr_b200_last_launch_count() == 0


def test_forward_sh_rejections(lib):
    from neural_renderer_b200 import _lib
    rgb = _lib.NR_RETURN_RGB

    def run(flags, ph=_phong(), la=None, sa=_sh(), face_light=False, corner_light=False):
        return lib.nr_b200_forward_sh(ctypes.byref(_fwd(flags, face_light, corner_light)),
                                      None if ph is None else ctypes.byref(ph), None if la is None else ctypes.byref(la),
                                      None if sa is None else ctypes.byref(sa), None)
    _rejections(run, lib)
    assert run(rgb, face_light=True) == INVALID
    assert run(rgb, corner_light=True) == INVALID
    assert run(rgb | _lib.NR_ANTI_ALIASING, sa=_sh(bs=3)) == INVALID
    assert lib.nr_b200_last_launch_count() == 0


def test_backward_sh_rejections(lib):
    from neural_renderer_b200 import _lib
    rgb = _lib.NR_RETURN_RGB

    def run(flags, ph=_phong(), la=None, sa=_sh(), textures=True):
        return lib.nr_b200_backward_sh(ctypes.byref(_bwd(flags, textures=textures)),
                                       None if ph is None else ctypes.byref(ph), None if la is None else ctypes.byref(la),
                                       None if sa is None else ctypes.byref(sa), None)
    _rejections(run, lib)
    for ok in (rgb | _lib.NR_GRAD_ACCUMULATE, rgb | _lib.NR_BWD_PART_TEXTURES, rgb | _lib.NR_BWD_PART_FACES):
        assert run(ok) == OK_UP_TO_WORKSPACE, hex(ok)
    # grad_sh needs the unlit sample s, so `textures`
    no_grads = _phong(grad_cs=False, grad_prm=False)
    assert run(rgb, ph=no_grads, textures=False) == INVALID
    assert run(rgb, ph=no_grads, la=_lights(nl=0, lights=False), textures=False) == INVALID
    assert run(rgb, ph=no_grads, sa=_sh(grad=False), textures=False) == OK_UP_TO_WORKSPACE
    assert run(rgb, ph=no_grads, la=_lights(grad=False), sa=_sh(grad=False), textures=False) == OK_UP_TO_WORKSPACE
    assert run(rgb | _lib.NR_GRAD_INTERIOR) == UNSUPPORTED
    assert lib.nr_b200_last_launch_count() == 0


# ---------------------------------------------------------------------------------------------------- Python errors
def test_python_argument_errors():
    import neural_renderer_b200 as nr
    faces = torch.rand((1, 4, 3, 3))
    tex = torch.rand((1, 4, 2, 2, 2, 3))
    cs, prm = torch.rand((1, 4, 3, 6)), torch.rand((1, 16))
    sh = torch.rand((9, 3))
    with pytest.raises(ValueError, match="Phong"):
        nr.rasterize(faces, tex, 8, environment_sh=sh)
    with pytest.raises(ValueError, match="return_rgb"):
        nr.rasterize_rgbad(faces, tex, 8, return_rgb=False, corner_shading=cs, shading_params=prm, environment_sh=sh)
    for bad in (torch.rand((1, 9, 4)), torch.rand((1, 8, 3)), torch.rand((27,)), torch.rand((3, 9, 3)),
                torch.rand((1, 1, 9, 3))):
        with pytest.raises(ValueError, match="environment_sh must have shape"):
            nr.rasterize(faces, tex, 8, corner_shading=cs, shading_params=prm, environment_sh=bad)
    for bad in ([[0.0] * 3] * 9, torch.zeros((9, 3), dtype=torch.int32), np.zeros((9, 3), np.float32)):
        with pytest.raises(TypeError):
            nr.rasterize(faces, tex, 8, corner_shading=cs, shading_params=prm, environment_sh=bad)
    with pytest.raises(NotImplementedError):  # a valid call on CPU tensors: no CPU implementation
        nr.rasterize(faces, tex, 8, corner_shading=cs, shading_params=prm, environment_sh=sh)


@pytest.mark.parametrize("shading", ["flat", "smooth"])
def test_renderer_environment_needs_phong(shading):
    import neural_renderer_b200 as nr
    r = nr.Renderer()
    assert r.environment_sh is None
    r.shading = shading
    r.environment_sh = torch.zeros((9, 3))
    v = torch.rand((1, 4, 3))
    f = torch.tensor([[[0, 1, 2], [1, 2, 3]]], dtype=torch.int32)
    with pytest.raises(ValueError, match="phong"):
        r.render(v, f, torch.rand((1, 2, 2, 2, 2, 3)))


# ---------------------------------------------------------------------------------------------- float64 oracle
def test_oracle_at_zero_environment_is_the_lights_oracle():
    faces, fim, wmap, dmap, cs, prm, unlit = _oracle_scene()
    bg = (0.1, 0.2, 0.3)
    lights = torch.tensor([[[0.5, 0.4, 0.3, 0.7, 0.6, 0.5, 0.4, -0.3, -2.0, 0.8, 1.0, 0.0],
                            [0.2, 0.3, 0.4, 0.1, 0.2, 0.3, -0.3, 0.6, -1.0, 0.0, 0.0, 0.0]]], dtype=torch.float64)
    for lt in (None, lights):
        for aa in (False, True):
            want = lights_rgb64(faces, fim, wmap, dmap, cs, prm, lt, unlit, bg, aa)
            for sh in (None, torch.zeros((1, 9, 3), dtype=torch.float64), torch.zeros((2, 9, 3), dtype=torch.float64)):
                got = sh_rgb64(faces, fim, wmap, dmap, cs, prm, lt, sh, unlit, bg, aa)
                assert float((got - want).abs().max()) <= 1e-12


def test_oracle_by_hand():
    """one covered pixel: the header's irradiance written out with numpy, unclamped"""
    faces, fim, wmap, dmap, cs, prm, unlit = _oracle_scene(B=1, S=4, F=2, seed=3)
    fim[:] = 1
    g = torch.Generator().manual_seed(5)
    sh = torch.randn((1, 9, 3), generator=g, dtype=torch.float64)
    L, _ = sh_terms64(faces, fim, wmap, dmap, cs, prm, None, sh)
    L0, _ = sh_terms64(faces, fim, wmap, dmap, cs, prm, None, None)
    lam = wmap[0, :, 2, 1].numpy() * (float(dmap[0, 2, 1]) / faces[0, 1, :, 2].numpy())
    n = lam @ cs[0, 1].numpy()[:, :3]
    x, y, z = n / (np.linalg.norm(n) + 1e-5)
    c0, c1, c2, c3, c4 = 0.28209479, 0.48860251, 1.09254843, 0.31539157, 0.54627422
    Y = np.array([c0, c1 * y, c1 * z, c1 * x, c2 * x * y, c2 * y * z, c3 * (3 * z * z - 1), c2 * x * z, c4 * (x * x - y * y)])
    E = Y @ sh[0].numpy()
    assert E.min() < 0  # negative irradiance is passed through
    np.testing.assert_allclose((L - L0)[0, 2, 1].numpy(), E, rtol=1e-7)  # the header's 8-digit constants


# ------------------------------------------------------------------------------------------ sh_from_environment_map
def _grid(He, We):
    t = math.pi * (torch.arange(He, dtype=torch.float64) + 0.5) / He
    p = 2 * math.pi * (torch.arange(We, dtype=torch.float64) + 0.5) / We
    st = torch.sin(t)[:, None]
    w = torch.stack([st * torch.sin(p)[None], torch.cos(t)[:, None].expand(He, We), st * torch.cos(p)[None]], -1)
    dw = (torch.sin(t) * (math.pi / He) * (2 * math.pi / We))[:, None].expand(He, We)
    return w, dw


def _midpoint_gate(He):
    # the midpoint rule in theta errs by about h^2 / 24 times the integrand's second derivative, h = pi / He; the
    # integrands here (degree <= 4 in omega times sin theta) have second derivatives of order 10 relative to their size
    return 10 * (math.pi / He) ** 2 / 24


def test_basis_is_orthonormal_under_the_quadrature():
    He, We = 256, 512
    w, dw = _grid(He, We)
    Y = sh_basis64(w)                                              # [He,We,9]
    G = torch.einsum('hwk,hwl,hw->kl', Y, Y, dw)
    err = float((G - torch.eye(9, dtype=torch.float64)).abs().max())
    assert err <= _midpoint_gate(He), err
    assert err > 0  # a quadrature, not an identity


@pytest.mark.parametrize("He", [32, 128])
def test_uniform_environment(He):
    from neural_renderer_b200 import functional as F
    r = torch.tensor([0.5, 1.0, 2.0], dtype=torch.float64)
    S = F.sh_from_environment_map(r.expand(He, 2 * He, 3))
    assert tuple(S.shape) == (1, 9, 3) and S.dtype == torch.float64
    want = torch.zeros((9, 3), dtype=torch.float64)
    want[0] = r / C0
    err = float(((S[0] - want) / r.max()).abs().max())
    assert err <= _midpoint_gate(He) / C0, err
    # irradiance-ready: a white albedo renders r (up to the quadrature) at any normal
    n = torch.nn.functional.normalize(torch.randn((50, 3), dtype=torch.float64), dim=-1)
    E = sh_basis64(n) @ S[0]
    assert float((E - r).abs().max() / r.max()) <= 2 * _midpoint_gate(He)


@pytest.mark.parametrize("He", [32, 128])
def test_linear_environment(He):
    """env = 1 + omega_y gives E(n) = 1 + (2/3) n_y (a_1 = 2/3 of the clamped cosine)"""
    from neural_renderer_b200 import functional as F
    w, _ = _grid(He, 2 * He)
    env = (1 + w[..., 1])[..., None].expand(He, 2 * He, 3)
    S = F.sh_from_environment_map(env)
    n = torch.nn.functional.normalize(torch.randn((200, 3), dtype=torch.float64), dim=-1)
    E = sh_basis64(n) @ S[0]
    want = (1 + 2 / 3 * n[:, 1])[:, None].expand(-1, 3)
    err = float((E - want).abs().max())
    assert err <= 2 * _midpoint_gate(He), err


def test_batched_and_float32_maps():
    from neural_renderer_b200 import functional as F
    g = torch.Generator().manual_seed(1)
    env = torch.rand((3, 16, 32, 3), generator=g, dtype=torch.float64)
    S = F.sh_from_environment_map(env)
    assert tuple(S.shape) == (3, 9, 3)
    for b in range(3):
        assert torch.allclose(S[b], F.sh_from_environment_map(env[b])[0], rtol=1e-14, atol=0)
    S32 = F.sh_from_environment_map(env.float())
    assert S32.dtype == torch.float32 and torch.allclose(S32.double(), S, rtol=1e-5, atol=1e-6)
    with pytest.raises(ValueError):
        F.sh_from_environment_map(torch.rand((16, 32, 4)))
    with pytest.raises(ValueError):
        F.sh_from_environment_map(torch.rand((32, 3)))
    with pytest.raises(TypeError):
        F.sh_from_environment_map(np.zeros((16, 32, 3)))


def test_helper_gradcheck():
    from neural_renderer_b200 import functional as F
    g = torch.Generator().manual_seed(2)
    env = torch.rand((2, 6, 8, 3), generator=g, dtype=torch.float64, requires_grad=True)
    assert torch.autograd.gradcheck(F.sh_from_environment_map, (env,))
