"""CPU: soft attribute images -- nr_b200_soft_attr_args against the header, the new symbols, the host rejections of both
entry points (all decided before any launch), the workspace query, the Python and Renderer argument errors (raised
before the device check), the float64 oracle against the soft RGB oracle, the hard interpolant and its own closed-form
gradient, and the spills of the new kernels."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest
import torch

import oracles_attr
import oracles_soft_attr as oattr
import oracles_soft_rgb as orgb

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# Fake, never dereferenced device addresses: a complete argument set gets as far as the workspace check
# (NR_ERR_WORKSPACE, no workspace given); each broken one must stop earlier.
_P = 0x10000
WORKSPACE, INVALID, UNSUPPORTED = -2, -1, -4


@pytest.fixture(scope="module")
def lib():
    from neural_renderer_b200 import build, _lib
    build.build_library()
    return _lib.load()


def test_soft_attr_struct_matches_the_header(tmp_path):
    from neural_renderer_b200 import _lib
    fields = [f[0] for f in _lib.SoftAttrArgs._fields_]
    exprs = ["sizeof(nr_b200_soft_attr_args)"] + ["offsetof(nr_b200_soft_attr_args, %s)" % f for f in fields]
    src = tmp_path / "s.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "nr_b200.h"\nint main(void){'
                   + "".join('printf("%%zu\\n", (size_t)(%s));' % e for e in exprs) + "return 0;}\n")
    exe = tmp_path / "s"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    vals = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert vals[0] == ctypes.sizeof(_lib.SoftAttrArgs) == 48
    assert vals[1:] == [getattr(_lib.SoftAttrArgs, f).offset for f in fields]


def test_new_symbols_are_exported(lib):
    from neural_renderer_b200 import _lib
    out = subprocess.run(["nm", "-D", "--defined-only", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    for n in ("nr_b200_soft_attributes", "nr_b200_soft_attributes_backward"):
        assert n in _lib.EXPORTED_SYMBOLS
        assert (" T " + n) in out, n


def _args(indexed=False, backward=False, **kw):
    from neural_renderer_b200 import _lib
    a = _lib.SoftRgbArgs()
    a.struct_size = ctypes.sizeof(_lib.SoftRgbArgs)
    a.flags = _lib.NR_FACES_INDEXED if indexed else 0
    a.batch_size, a.num_faces, a.image_size, a.num_vertices, a.texture_size = 2, 4, 16, 6 if indexed else 0, 0
    a.sigma, a.gamma, a.near_, a.far_, a.eps = 1e-4, 1e-4, 0.1, 100.0, float("nan")  # texture_size and eps: ignored
    if indexed:
        a.vertices = a.face_indices = _P
    else:
        a.faces = _P
    a.alpha = a.state = _P
    if backward:
        a.grad_alpha = _P
        if indexed:
            a.grad_vertices = _P
        else:
            a.grad_faces = _P
    for k, v in kw.items():
        setattr(a, k, v)
    return a


def _attr(backward=False, **kw):
    from neural_renderer_b200 import _lib
    t = _lib.SoftAttrArgs(struct_size=ctypes.sizeof(_lib.SoftAttrArgs), channels=5, attributes=_P, out=_P)
    if backward:
        t.grad_out = _P
    for k, v in kw.items():
        setattr(t, k, v)
    return t


def _call(lib, a, t, backward):
    fn = lib.nr_b200_soft_attributes_backward if backward else lib.nr_b200_soft_attributes
    return fn(ctypes.byref(a) if a is not None else None, ctypes.byref(t) if t is not None else None, None)


@pytest.mark.parametrize("backward", [False, True])
@pytest.mark.parametrize("indexed", [False, True])
def test_host_rejections(lib, indexed, backward):
    from neural_renderer_b200 import _lib
    ok = _args(indexed, backward)
    assert _call(lib, ok, _attr(backward), backward) == WORKSPACE
    assert lib.nr_b200_last_launch_count() == 0
    fl = ok.flags
    allowed = [(dict(flags=fl | _lib.NR_ATTR_SHARED), {}), (dict(flags=fl | _lib.NR_GRAD_ACCUMULATE), {}),
               (dict(texture_size=1000), {}), (dict(eps=0.5), {}), ({}, dict(channels=1)), ({}, dict(channels=300)),
               ({}, dict(background=_P))]
    if backward:
        allowed += [(dict(grad_alpha=None), {}), ({}, dict(grad_out=None)), (dict(grad_alpha=None), dict(grad_out=None)),
                    ({}, dict(grad_attributes=_P))]
    if indexed:
        allowed += [(dict(flags=fl | _lib.NR_INDICES_SHARED), {}), (dict(flags=fl | _lib.NR_ATTR_PER_VERTEX), {}),
                    (dict(flags=fl | _lib.NR_ATTR_PER_VERTEX | _lib.NR_ATTR_SHARED | _lib.NR_INDICES_SHARED), {})]
    for kw, tkw in allowed:
        assert _call(lib, _args(indexed, backward, **kw), _attr(backward, **tkw), backward) == WORKSPACE, (kw, tkw)
    bad = [(dict(struct_size=4), {}), (dict(struct_size=ctypes.sizeof(_lib.SoftRgbArgs) + 8), {}),
           ({}, dict(struct_size=0)), ({}, dict(struct_size=ctypes.sizeof(_lib.SoftAttrArgs) + 8)),
           ({}, dict(channels=0)), ({}, dict(channels=-2)), ({}, dict(attributes=None)), ({}, dict(out=None)),
           (dict(batch_size=0), {}), (dict(num_faces=0), {}), (dict(image_size=0), {}), (dict(sigma=0.0), {}),
           (dict(sigma=float("nan")), {}), (dict(gamma=0.0), {}), (dict(gamma=float("inf")), {}),
           (dict(near_=2.0, far_=1.0), {}), (dict(near_=1.0, far_=1.0), {}), (dict(alpha=None), {}), (dict(state=None), {}),
           (dict(batch_size=65536), {}), (dict(image_size=32768), {}),
           # the soft RGB's colour buffers are refused
           (dict(textures=_P), {}), (dict(face_light=_P), {}), (dict(rgb=_P), {}), (dict(grad_rgb=_P), {}),
           (dict(grad_textures=_P), {}), (dict(grad_face_light=_P), {})]
    for f in (_lib.NR_TEX_SHARED, _lib.NR_TEX_UV, _lib.NR_UV_SHARED, _lib.NR_TEX_MIPMAP, _lib.NR_TEX_FILL_BACK,
              _lib.NR_GRAD_INTERIOR, _lib.NR_RETURN_RGB, _lib.NR_ANTI_ALIASING, 1 << 31):
        bad.append((dict(flags=fl | f), {}))
    if indexed:
        bad += [(dict(vertices=None), {}), (dict(face_indices=None), {}), (dict(num_vertices=0), {})]
    else:
        bad += [(dict(faces=None), {}), (dict(flags=fl | _lib.NR_ATTR_PER_VERTEX), {})]  # per vertex needs indices
    if backward:
        bad += [(dict(grad_faces=_P), {})] if indexed else [(dict(grad_vertices=_P), {})]
        bad += [(dict(grad_vertices=None), {})] if indexed else [(dict(grad_faces=None), {})]
    for kw, tkw in bad:
        assert _call(lib, _args(indexed, backward, **kw), _attr(backward, **tkw), backward) == INVALID, (kw, tkw)
        assert lib.nr_b200_last_launch_count() == 0
    assert _call(lib, None, _attr(backward), backward) == INVALID
    assert _call(lib, ok, None, backward) == INVALID
    # attribute offsets beyond 32 bits, or more channel blocks of 16 than grid.z holds: after every invalid argument,
    # before the workspace.  100000 faces (or vertices) make 300000 corner rows
    pv = _lib.NR_ATTR_PER_VERTEX if indexed else 0
    big = dict(num_faces=100000, num_vertices=300000 if indexed else 0)
    for flags, C, rc in ((fl | pv, 4000, UNSUPPORTED),                                  # 2 x 1.2e9 floats
                         (fl | pv | _lib.NR_ATTR_SHARED, 4000, WORKSPACE),             # one shared set of 1.2e9
                         (fl | pv | _lib.NR_ATTR_SHARED, 8000, UNSUPPORTED),           # 2.4e9 in one set
                         (fl, 16 * 65535, WORKSPACE), (fl, 16 * 65535 + 1, UNSUPPORTED)):
        kw = big if C < 10000 else {}
        assert _call(lib, _args(indexed, backward, flags=flags, **kw), _attr(backward, channels=C), backward) == rc, (flags, C)
        assert lib.nr_b200_last_launch_count() == 0
    assert _call(lib, _args(indexed, backward, alpha=None, flags=fl | pv, **big), _attr(backward, channels=4000),
                 backward) == INVALID


def test_workspace_is_the_soft_rgb_query(lib):
    from neural_renderer_b200 import _lib
    # the query needs a device (CUB sizes the sort for it): without one it returns 0 for every call alike
    geometry = (0, _lib.NR_FACES_INDEXED, _lib.NR_FACES_INDEXED | _lib.NR_INDICES_SHARED, _lib.NR_GRAD_ACCUMULATE)
    for flags in geometry:
        n = lib.nr_b200_soft_rgb_workspace_bytes(2, 100, 64, flags)
        assert n == lib.nr_b200_soft_rgb_workspace_bytes(2, 100, 64, 0)
    # the attribute flags are not workspace flags
    assert lib.nr_b200_soft_rgb_workspace_bytes(2, 100, 64, _lib.NR_ATTR_PER_VERTEX) == 0


def test_python_argument_errors_come_before_the_device_check():
    import neural_renderer_b200 as nr
    faces = torch.zeros(1, 2, 3, 3)
    fa = torch.zeros(2, 3, 4)
    with pytest.raises(NotImplementedError):  # valid arguments on the CPU: no CPU path
        nr.rasterize_soft_attributes(faces, 16, face_attributes=fa)
    with pytest.raises(NotImplementedError):
        nr.rasterize_soft_attributes(faces, 16, face_attributes=fa[None], background=[0.0] * 4, return_alpha=True)
    verts, idx = torch.zeros(1, 5, 3), torch.zeros(2, 3, dtype=torch.int64)
    with pytest.raises(NotImplementedError):
        nr.rasterize_soft_attributes(idx, 16, vertices=verts, vertex_attributes=torch.zeros(5, 2))
    for kw in (dict(sigma=0.0), dict(sigma=float("nan")), dict(gamma=0.0), dict(gamma=float("inf")),
               dict(near=2.0, far=1.0), dict(near=1.0, far=1.0), dict(image_size=0), dict(background=[0.0] * 3),
               dict(background=torch.zeros(5)), dict(face_attributes=torch.zeros(3, 3, 4)),
               dict(face_attributes=torch.zeros(2, 2, 4)), dict(face_attributes=torch.zeros(2, 3, 0)),
               dict(face_attributes=torch.zeros(2, 2, 3, 4))):
        with pytest.raises(ValueError):
            nr.rasterize_soft_attributes(faces, **{"image_size": 16, "face_attributes": fa, **kw})
    with pytest.raises(ValueError):  # per-vertex attributes need indexed geometry
        nr.rasterize_soft_attributes(faces, 16, vertex_attributes=torch.zeros(5, 2))
    with pytest.raises(ValueError):  # Nv rows
        nr.rasterize_soft_attributes(idx, 16, vertices=verts, vertex_attributes=torch.zeros(4, 2))
    for kw in (dict(), dict(face_attributes=fa, vertex_attributes=torch.zeros(5, 4)), dict(face_attributes=fa.int()),
               dict(face_attributes=fa, sigma="x"), dict(face_attributes=fa, background=["a"] * 4)):
        with pytest.raises(TypeError):
            nr.rasterize_soft_attributes(faces, 16, **kw)
    r = nr.Renderer()
    v, f = torch.zeros(1, 3, 3), torch.zeros(1, 1, 3, dtype=torch.int32)
    with pytest.raises(TypeError):
        r.render_soft_attributes(v, f)
    with pytest.raises(TypeError):
        r.render_soft_attributes(v, f, vertex_attributes=torch.zeros(3, 2), face_attributes=torch.zeros(1, 3, 2))
    with pytest.raises(ValueError):
        r.render_soft_attributes(v, f, face_attributes=torch.zeros(2, 3, 2))   # F = 1
    with pytest.raises(ValueError):
        r.render_soft_attributes(v, f, face_attributes=torch.zeros(1, 3, 2), background=[0.0])
    with pytest.raises(ValueError):
        r.render_soft_depth(v, f, sigma=-1.0)
    with pytest.raises(NotImplementedError):
        r.render_soft_depth(v, f)
    with pytest.raises(NotImplementedError):
        r.render_soft_attributes(v, f, vertex_attributes=torch.zeros(3, 2))


# ------------------------------------------------------------------------------------------------ oracle self-checks
def _faces(seed, F=5, B=1):
    g = torch.Generator().manual_seed(seed)
    faces = torch.rand(B, F, 3, 3, generator=g, dtype=torch.float64) * 1.6 - 0.8
    faces[..., 2] = 1.0 + 3.0 * torch.rand(B, F, 3, generator=g, dtype=torch.float64)
    return faces


def test_constant_corner_attributes_equal_the_soft_rgb_oracle_with_constant_cubes():
    g = torch.Generator().manual_seed(2)
    B, F, S = 2, 6, 24
    faces = _faces(1, F, B)
    col = torch.rand(B, F, 3, generator=g, dtype=torch.float64)
    ca = col[:, :, None].expand(B, F, 3, 3)
    cubes = col[:, :, None, None, None].expand(B, F, 2, 2, 2, 3)
    for sigma, gamma in ((1e-3, 1e-2), (1e-4, 1e-4)):
        want = orgb.soft_rgb(faces, cubes, S, sigma, gamma, background=(0.1, 0.2, 0.3))
        got = oattr.soft_attributes(faces, ca, S, sigma, gamma, background=(0.1, 0.2, 0.3))
        torch.testing.assert_close(got[0], want[0], rtol=1e-12, atol=1e-13)
        assert torch.equal(got[1], want[1])


def test_sigma_gamma_to_zero_is_the_hard_interpolant_inside_faces():
    g = torch.Generator().manual_seed(3)
    S, C = 32, 4
    faces = torch.tensor([[[[-0.7, -0.6, 2.0], [0.8, -0.5, 3.0], [0.1, 0.75, 4.0]],
                           [[-0.9, 0.2, 1.5], [-0.2, 0.3, 1.5], [-0.6, 0.9, 1.5]]]], dtype=torch.float64)
    ca = torch.rand(1, 2, 3, C, generator=g, dtype=torch.float64)
    out, alpha = oattr.soft_attributes(faces, ca, S, 1e-9, 1e-7)
    # the nearest face at every pixel well inside a face (barycentrics >= 0.05), then oracles_attr's hard interpolant
    xs = (2 * np.arange(S) + 1 - S) / S
    fim = torch.full((1, S, S), -1, dtype=torch.int64)
    for r in range(S):
        for c in range(S):
            best = None
            for f in range(2):
                v = faces[0, f].numpy()
                M = np.array([[v[0, 0], v[1, 0], v[2, 0]], [v[0, 1], v[1, 1], v[2, 1]], [1.0, 1.0, 1.0]])
                w = np.linalg.solve(M, [xs[c], xs[S - 1 - r], 1.0])
                zp = 1.0 / (w / v[:, 2]).sum()
                if w.min() >= 0.05 and (best is None or zp < best[0]):
                    best = (zp, f)
            if best is not None:
                fim[0, r, c] = best[1]
    hard = oracles_attr.interp64(faces, fim, ca, S, False)
    m = (fim >= 0)[:, None].expand_as(out)
    assert m.sum() > 100 * C
    torch.testing.assert_close(out[m], hard[m], rtol=0, atol=1e-9)
    assert torch.all(alpha[fim >= 0] > 1 - 1e-12)


def test_the_z_attribute_gives_zp():
    B, F, S = 1, 6, 20
    faces = _faces(4, F, B)
    ca = faces[..., 2:3]
    x, on, valid, zn, A = oattr.attr_terms(faces, ca, oattr.osoft.pixel_centres(S), 1e-3, 0.1, 100.0, 1.0)
    zp = 100.0 - zn * (100.0 - 0.1)
    torch.testing.assert_close(A[..., 0][valid], zp[valid], rtol=1e-12, atol=1e-12)
    assert valid.sum() > 50


def test_closed_form_attribute_gradient_agrees_with_autograd():
    g = torch.Generator().manual_seed(5)
    B, F, S, C = 2, 5, 20, 3
    faces = _faces(6, F, B)
    for shared in (False, True):
        ca = torch.rand(1 if shared else B, F, 3, C, generator=g, dtype=torch.float64).requires_grad_(True)
        up = torch.randn(B, C, S, S, generator=g, dtype=torch.float64)
        out, _ = oattr.soft_attributes(faces, ca, S, 1e-3, 1e-2, background=(0.5,) * C)
        (ga,) = torch.autograd.grad((out * up).sum(), ca)
        cf = oattr.attribute_grad_closed_form(faces, ca.detach(), S, 1e-3, 1e-2, up, background=(0.5,) * C)
        if shared:
            cf = cf.sum(0, keepdim=True)
        torch.testing.assert_close(ga, cf, rtol=1e-10, atol=1e-12)
    # per vertex: the gather's gradient, out-of-range indices read zeros and get nothing
    va = torch.rand(1, 7, C, generator=g, dtype=torch.float64).requires_grad_(True)
    idx = torch.randint(0, 7, (F, 3), generator=g)
    idx[1, 2] = 7
    idx[3, 0] = -1
    ca = oattr.corner_attributes(va, idx)
    assert torch.all(ca[:, 1, 2] == 0) and torch.all(ca[:, 3, 0] == 0)
    out, _ = oattr.soft_attributes(faces, ca, S, 1e-3, 1e-2)
    (gv,) = torch.autograd.grad((out * up).sum(), va)
    cf = oattr.attribute_grad_closed_form(faces, ca.detach(), S, 1e-3, 1e-2, up)            # [B,F,3,C]
    want = torch.zeros(7, C, dtype=torch.float64)
    for f in range(F):
        for k in range(3):
            if 0 <= int(idx[f, k]) < 7:
                want[int(idx[f, k])] += cf[:, f, k].sum(0)
    torch.testing.assert_close(gv[0], want, rtol=1e-10, atol=1e-12)


def test_sparse_evaluation_matches_dense():
    g = torch.Generator().manual_seed(8)
    B, F, S, C = 2, 8, 24, 2
    faces = _faces(9, F, B)
    ca = torch.rand(B, F, 3, C, generator=g, dtype=torch.float64)
    dense = oattr.soft_attributes(faces, ca, S, 1e-3, 1e-2, background=(0.2, 0.7))
    pix = torch.randperm(S * S, generator=g)[:50]
    sparse = oattr.soft_attributes(faces, ca, S, 1e-3, 1e-2, background=(0.2, 0.7), pix=pix)
    torch.testing.assert_close(sparse[0], dense[0].reshape(B, C, -1)[:, :, pix], rtol=1e-13, atol=1e-13)
    torch.testing.assert_close(sparse[1], dense[1].reshape(B, -1)[:, pix], rtol=1e-13, atol=1e-13)


def test_new_kernels_compile_for_sm90a_without_spills(tmp_path):
    from neural_renderer_b200 import build
    nvcc = os.environ.get("NVCC", "nvcc")
    cmd = [nvcc] + build.NVCC_FLAGS + ["-Xptxas", "-v", "-c", os.path.join(build.CSRC, "nr_soft_attr.cu"),
                                       "-o", str(tmp_path / "nr_soft_attr.o")]
    log = subprocess.run(cmd, capture_output=True, text=True, check=True).stderr
    entries = re.split(r"Compiling entry function '", log)[1:]
    names = [e.split("'")[0] for e in entries]
    # forward and backward, channel blocks of 4 and 16, 32- and 64-bit keys; the binning kernels are nr_soft_rgb.cu's
    assert len(entries) == 8 and all("k_soft_attr_" in n for n in names), names
    for e in entries:
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", e)
        assert m and m.groups() == ("0", "0", "0"), e[:400]
        assert "cumulative stack" not in e.split("Compile time")[0], e[:400]
    assert "sm_90a" in log
