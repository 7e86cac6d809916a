"""CPU: soft silhouettes -- nr_b200_soft_args against the header, the new symbols, the host rejections of both entry points
(all decided before any device work), the workspace query, the Python argument errors (raised before the device check),
the float64 oracle against closed forms, and the registers / spills of the new kernels."""
import ctypes
import math
import os
import re
import subprocess

import numpy as np
import pytest
import torch

import oracles_soft as osoft

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# Fake, never dereferenced device addresses: a complete argument set gets as far as the workspace check
# (NR_ERR_WORKSPACE, no workspace given); each broken one must stop earlier with NR_ERR_INVALID_ARG.
_P = 0x10000
WORKSPACE, INVALID = -2, -1


@pytest.fixture(scope="module")
def lib():
    from neural_renderer_b200 import build, _lib
    build.build_library()
    return _lib.load()


def test_soft_struct_matches_the_header(tmp_path):
    from neural_renderer_b200 import _lib
    fields = [f[0] for f in _lib.SoftArgs._fields_]
    exprs = ["sizeof(nr_b200_soft_args)"] + ["offsetof(nr_b200_soft_args, %s)" % f for f in fields] + ["NR_SOFT_EPS"]
    src = tmp_path / "s.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "nr_b200.h"\nint main(void){'
                   + "".join('printf("%%zu\\n", (size_t)(%s));' % e for e in exprs[:-1])
                   + 'printf("%.17g\\n", (double)(NR_SOFT_EPS));return 0;}\n')
    exe = tmp_path / "s"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    out = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()
    vals = [int(x) for x in out[:-1]]
    assert vals[0] == ctypes.sizeof(_lib.SoftArgs) == 112
    assert vals[1:] == [getattr(_lib.SoftArgs, f).offset for f in fields]
    assert float(out[-1]) == _lib.SOFT_EPS == osoft.EPS


def test_new_symbols_are_exported(lib):
    from neural_renderer_b200 import _lib
    names = ("nr_b200_soft_workspace_bytes", "nr_b200_soft_silhouettes", "nr_b200_soft_silhouettes_backward")
    out = subprocess.run(["nm", "-D", "--defined-only", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    for n in names:
        assert n in _lib.EXPORTED_SYMBOLS
        assert (" T " + n) in out, n


def test_workspace_query_is_pure_host(lib):
    n = lib.nr_b200_soft_workspace_bytes(64, 5000, 256, 1e-5, 0)
    # face records, tile boxes and at most 16 list entries per face
    assert n >= 64 * 5000 * (64 + 8 + 16 * 4)
    assert lib.nr_b200_soft_workspace_bytes(64, 5000, 256, 1e-3, 0) == n  # the list bound does not depend on sigma
    for bad in [(0, 5, 16, 1e-5), (1, 0, 16, 1e-5), (1, 5, 0, 1e-5), (1, 5, 16, 0.0), (1, 5, 16, -1.0),
                (1, 5, 16, float("nan")), (1, 5, 16, float("inf")), (65536, 1, 16, 1e-5), (1, 1, 32768, 1e-5),
                (1024, 1 << 17, 16, 1e-5)]:
        assert lib.nr_b200_soft_workspace_bytes(*bad, 0) == 0, bad


def _args(indexed=False, backward=False, **kw):
    from neural_renderer_b200 import _lib
    a = _lib.SoftArgs()
    a.struct_size = ctypes.sizeof(_lib.SoftArgs)
    a.flags = _lib.NR_FACES_INDEXED if indexed else 0
    a.batch_size, a.num_faces, a.image_size, a.num_vertices = 2, 4, 16, 6 if indexed else 0
    a.sigma, a.near_, a.far_ = 1e-4, 0.1, 100.0
    if indexed:
        a.vertices = a.face_indices = _P
    else:
        a.faces = _P
    a.alpha = _P
    if backward:
        a.grad_alpha = _P
        if indexed:
            a.grad_vertices = _P
        else:
            a.grad_faces = _P
    for k, v in kw.items():
        setattr(a, k, v)
    return a


def _call(lib, a, backward):
    fn = lib.nr_b200_soft_silhouettes_backward if backward else lib.nr_b200_soft_silhouettes
    return fn(ctypes.byref(a), None)


@pytest.mark.parametrize("backward", [False, True])
@pytest.mark.parametrize("indexed", [False, True])
def test_host_rejections(lib, indexed, backward):
    from neural_renderer_b200 import _lib
    ok = _args(indexed, backward)
    assert _call(lib, ok, backward) == WORKSPACE
    assert lib.nr_b200_last_launch_count() == 0
    # every allowed NULL: grad_alpha (zeros) and the shared index set
    assert _call(lib, _args(indexed, backward, grad_alpha=None), backward) == WORKSPACE
    if indexed:
        assert _call(lib, _args(indexed, backward, flags=_lib.NR_FACES_INDEXED | _lib.NR_INDICES_SHARED), backward) == WORKSPACE
    bad = [dict(struct_size=4), dict(struct_size=ctypes.sizeof(_lib.SoftArgs) + 8), dict(batch_size=0),
           dict(num_faces=0), dict(image_size=0), dict(batch_size=-1), dict(sigma=0.0), dict(sigma=-1e-5),
           dict(sigma=float("nan")), dict(sigma=float("inf")), dict(near_=2.0, far_=1.0), dict(near_=float("nan")),
           dict(alpha=None), dict(batch_size=65536), dict(image_size=32768), dict(batch_size=1024, num_faces=1 << 17)]
    if indexed:
        bad += [dict(vertices=None), dict(face_indices=None), dict(num_vertices=0)]
    else:
        bad += [dict(faces=None)]
    if backward:
        bad += [dict(grad_faces=_P)] if indexed else [dict(grad_vertices=_P)]
        bad += [dict(grad_vertices=None)] if indexed else [dict(grad_faces=None)]
    for kw in bad:
        assert _call(lib, _args(indexed, backward, **kw), backward) == INVALID, kw
        assert lib.nr_b200_last_launch_count() == 0
    fn = lib.nr_b200_soft_silhouettes_backward if backward else lib.nr_b200_soft_silhouettes
    assert fn(None, None) == INVALID


def test_python_argument_errors_come_before_the_device_check():
    import neural_renderer_b200 as nr
    faces = torch.zeros(1, 2, 3, 3)  # CPU: valid arguments end in NotImplementedError (no CPU path)
    with pytest.raises(NotImplementedError):
        nr.rasterize_soft_silhouettes(faces, 16)
    with pytest.raises(NotImplementedError):
        nr.rasterize_soft_silhouettes(torch.zeros(4, 3, dtype=torch.int32), 16, vertices=torch.zeros(1, 3, 3))
    for kw in (dict(sigma=0.0), dict(sigma=-1e-5), dict(sigma=float("nan")), dict(sigma=float("inf")),
               dict(near=2.0, far=1.0), dict(image_size=0)):
        with pytest.raises(ValueError):
            nr.rasterize_soft_silhouettes(faces, **{"image_size": 16, **kw})
    with pytest.raises(TypeError):
        nr.rasterize_soft_silhouettes(faces, 16, sigma="x")
    with pytest.raises(ValueError):
        nr.rasterize_soft_silhouettes(torch.zeros(1, 2, 3, 2), 16)
    with pytest.raises(TypeError):
        nr.rasterize_soft_silhouettes(torch.zeros(1, 2, 3, 3, dtype=torch.int32), 16)
    with pytest.raises(ValueError):
        nr.rasterize_soft_silhouettes(torch.zeros(4, 2, dtype=torch.int32), 16, vertices=torch.zeros(1, 3, 3))
    import neural_renderer
    assert neural_renderer.rasterize_soft_silhouettes is nr.rasterize_soft_silhouettes
    assert hasattr(nr.Renderer(), "render_soft_silhouettes")


# ------------------------------------------------------------------------------------------------ oracle self-checks
def _tri(pts, z=1.0):
    f = torch.tensor([[[p[0], p[1], z] for p in pts]], dtype=torch.float64)
    return f[None]  # [1,1,3,3]


def test_oracle_distance_field_of_one_triangle_against_closed_forms():
    a = 0.51  # no pixel centre on the hypotenuse
    faces = _tri([(0.0, 0.0), (a, 0.0), (0.0, a)])
    S = 40
    p = osoft.pixel_centres(S)
    d2, inside = osoft.face_terms(faces, p)
    d2, inside = d2[0, 0].numpy(), inside[0, 0].numpy()
    x, y = p[:, 0].numpy(), p[:, 1].numpy()
    want = np.empty_like(x)
    want_in = (x > 0) & (y > 0) & (x + y < a)
    for i in range(len(x)):
        if want_in[i]:
            want[i] = min(x[i], y[i], (a - x[i] - y[i]) / math.sqrt(2)) ** 2
        elif x[i] <= 0 and y[i] <= 0:
            want[i] = x[i] ** 2 + y[i] ** 2                      # nearest: corner (0, 0)
        elif 0 < x[i] < a and y[i] <= 0:
            want[i] = y[i] ** 2                                  # the bottom edge's interior
        elif x[i] <= 0 and 0 < y[i] < a:
            want[i] = x[i] ** 2                                  # the left edge's interior
        else:  # the hypotenuse or one of its corners
            t = min(max(((x[i] - a) * -a + y[i] * a) / (2 * a * a), 0.0), 1.0)
            qx, qy = a - t * a, t * a
            want[i] = min((x[i] - qx) ** 2 + (y[i] - qy) ** 2, (x[i] - a) ** 2 + y[i] ** 2, x[i] ** 2 + (y[i] - a) ** 2)
    assert (inside == want_in).all()
    np.testing.assert_allclose(d2, want, rtol=1e-12, atol=1e-15)


def test_oracle_is_winding_independent():
    g = torch.Generator().manual_seed(1)
    faces = torch.rand(2, 6, 3, 3, generator=g, dtype=torch.float64) * 1.6 - 0.8
    faces[..., 2] = 1.0
    a = osoft.soft_silhouettes(faces, 24, 1e-3)
    b = osoft.soft_silhouettes(faces.flip(2), 24, 1e-3)
    assert torch.equal(a, b) or (a - b).abs().max() < 1e-14
    assert a.max() > 0.5


def test_oracle_tends_to_the_hard_coverage():
    g = torch.Generator().manual_seed(2)
    faces = torch.rand(1, 5, 3, 3, generator=g, dtype=torch.float64) * 1.6 - 0.8
    faces[..., 2] = 1.0
    S = 48
    alpha = osoft.soft_silhouettes(faces, S, 1e-9)[0].numpy()
    # hard coverage by barycentric coordinates (a linear solve per face), and each pixel's distance to every edge line
    p = osoft.pixel_centres(S).numpy()
    cov = np.zeros(S * S, bool)
    near_edge = np.zeros(S * S, bool)
    for f in faces[0].numpy():
        T = np.array([[f[0, 0] - f[2, 0], f[1, 0] - f[2, 0]], [f[0, 1] - f[2, 1], f[1, 1] - f[2, 1]]])
        l01 = np.linalg.solve(T, (p - f[2, :2]).T).T
        lam = np.concatenate([l01, 1 - l01.sum(1, keepdims=True)], 1)
        cov |= (lam > 0).all(1)
        for k in range(3):
            a, b = f[k, :2], f[(k + 1) % 3, :2]
            e = b - a
            t = np.clip(((p - a) @ e) / (e @ e), 0, 1)
            d = np.linalg.norm(p - (a + t[:, None] * e), axis=1)
            near_edge |= d <= 2.0 / S  # 1 px = 2 / S in NDC
    far = ~near_edge
    assert far.sum() > S * S // 2
    np.testing.assert_allclose(alpha.reshape(-1)[far], cov[far].astype(np.float64), atol=1e-12)


def test_oracle_aggregation_gradient_is_one_minus_alpha_times_d():
    g = torch.Generator().manual_seed(3)
    x = (torch.randn(7, 9, generator=g, dtype=torch.float64) * 6).requires_grad_(True)
    on = torch.rand(7, 9, generator=g) > 0.3
    alpha = osoft.alpha_from_x(x, on)
    (gx,) = torch.autograd.grad(alpha.sum(), x)
    want = torch.where(on, (1 - alpha.detach())[:, None] * torch.sigmoid(x.detach()), torch.zeros_like(x))
    torch.testing.assert_close(gx, want, rtol=1e-12, atol=1e-15)
    # and alpha is the product form
    prod = 1 - torch.where(on, 1 - torch.sigmoid(x.detach()), torch.ones_like(x)).prod(-1)
    torch.testing.assert_close(alpha.detach(), prod, rtol=1e-12, atol=1e-15)


def test_new_kernels_compile_for_sm90a_without_spills(tmp_path):
    from neural_renderer_b200 import build
    nvcc = os.environ.get("NVCC", "nvcc")
    cmd = [nvcc] + build.NVCC_FLAGS + ["-Xptxas", "-v", "-c", os.path.join(build.CSRC, "nr_soft.cu"),
                                       "-o", str(tmp_path / "nr_soft.o")]
    log = subprocess.run(cmd, capture_output=True, text=True, check=True).stderr
    kernels = re.findall(r"Compiling entry function '(\w+)'", log)
    assert len(kernels) == 4 and all("k_soft_" in k for k in kernels), kernels
    spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", log)
    assert len(spills) == 4 and all(s == ("0", "0") for s in spills), log
    assert "sm_90a" in log
