"""CPU: soft RGB through a texture image -- nr_b200_soft_uv_args against the header, the new symbols, the host rejections
of both entry points (all decided before any launch), uv NULL as the cube call, the Python argument errors (raised before
the device check), the float64 oracle against the cube oracle and its limits, and the spills of the new kernels."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest
import torch

import oracles
import oracles_soft_rgb as orgb
import oracles_soft_uv as ouv

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


def test_soft_uv_struct_matches_the_header(tmp_path):
    from neural_renderer_b200 import _lib
    fields = [f[0] for f in _lib.SoftUvArgs._fields_]
    exprs = ["sizeof(nr_b200_soft_uv_args)"] + ["offsetof(nr_b200_soft_uv_args, %s)" % f for f in fields]
    src = tmp_path / "s.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "nr_b200.h"\nint main(void){'
                   + "".join('printf("%%zu\\n", (size_t)(%s));' % e for e in exprs) + "return 0;}\n")
    exe = tmp_path / "s"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    vals = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert vals[0] == ctypes.sizeof(_lib.SoftUvArgs) == 32
    assert vals[1:] == [getattr(_lib.SoftUvArgs, f).offset for f in fields]


def test_new_symbols_are_exported(lib):
    from neural_renderer_b200 import _lib
    out = subprocess.run(["nm", "-D", "--defined-only", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    for n in ("nr_b200_soft_rgb_uv", "nr_b200_soft_rgb_uv_backward"):
        assert n in _lib.EXPORTED_SYMBOLS
        assert (" T " + n) in out, n


def _args(indexed=False, backward=False, **kw):
    from neural_renderer_b200 import _lib
    a = _lib.SoftRgbArgs()
    a.struct_size = ctypes.sizeof(_lib.SoftRgbArgs)
    a.flags = (_lib.NR_FACES_INDEXED if indexed else 0) | _lib.NR_TEX_UV
    a.batch_size, a.num_faces, a.image_size, a.num_vertices, a.texture_size = 2, 4, 16, 6 if indexed else 0, 0
    a.sigma, a.gamma, a.near_, a.far_, a.eps = 1e-4, 1e-4, 0.1, 100.0, float("nan")  # texture_size and eps: ignored
    if indexed:
        a.vertices = a.face_indices = _P
    else:
        a.faces = _P
    a.textures = a.rgb = a.alpha = a.state = _P
    if backward:
        a.grad_rgb = a.grad_alpha = _P
        if indexed:
            a.grad_vertices = _P
        else:
            a.grad_faces = _P
    for k, v in kw.items():
        setattr(a, k, v)
    return a


def _uv(**kw):
    from neural_renderer_b200 import _lib
    u = _lib.SoftUvArgs(struct_size=ctypes.sizeof(_lib.SoftUvArgs), texture_height=8, texture_width=5, face_uvs=_P)
    for k, v in kw.items():
        setattr(u, k, v)
    return u


def _call(lib, a, u, backward):
    fn = lib.nr_b200_soft_rgb_uv_backward if backward else lib.nr_b200_soft_rgb_uv
    return fn(ctypes.byref(a), ctypes.byref(u) if u is not None else None, None)


@pytest.mark.parametrize("backward", [False, True])
@pytest.mark.parametrize("indexed", [False, True])
def test_host_rejections(lib, indexed, backward):
    from neural_renderer_b200 import _lib
    ok = _args(indexed, backward)
    assert _call(lib, ok, _uv(), backward) == WORKSPACE
    assert lib.nr_b200_last_launch_count() == 0
    fl = ok.flags
    allowed = [(dict(face_light=_P), {}), (dict(flags=fl | _lib.NR_UV_SHARED), {}), (dict(flags=fl | _lib.NR_TEX_MIPMAP), {}),
               (dict(flags=fl | _lib.NR_TEX_SHARED), {}), (dict(flags=fl | _lib.NR_GRAD_ACCUMULATE), {}),
               (dict(texture_size=1000), {}), (dict(eps=0.5), {}), ({}, dict(texture_height=1, texture_width=1))]
    if backward:
        allowed += [(dict(grad_rgb=None), {}), (dict(grad_alpha=None), {}), (dict(grad_rgb=None, grad_alpha=None), {}),
                    (dict(grad_textures=_P, grad_face_light=_P), dict(grad_face_uvs=_P))]
    if indexed:
        allowed += [(dict(flags=fl | _lib.NR_INDICES_SHARED), {})]
    for kw, ukw in allowed:
        assert _call(lib, _args(indexed, backward, **kw), _uv(**ukw), backward) == WORKSPACE, (kw, ukw)
    bad = [(dict(struct_size=4), {}), (dict(struct_size=ctypes.sizeof(_lib.SoftRgbArgs) + 8), {}),
           ({}, dict(struct_size=0)), ({}, dict(struct_size=ctypes.sizeof(_lib.SoftUvArgs) + 8)),
           (dict(flags=fl & ~_lib.NR_TEX_UV), {}), ({}, dict(face_uvs=None)), ({}, dict(texture_height=0)),
           ({}, dict(texture_width=0)), ({}, dict(texture_height=-3)),
           (dict(batch_size=0), {}), (dict(num_faces=0), {}), (dict(image_size=0), {}), (dict(sigma=0.0), {}),
           (dict(sigma=float("nan")), {}), (dict(gamma=0.0), {}), (dict(gamma=float("inf")), {}),
           (dict(near_=2.0, far_=1.0), {}), (dict(textures=None), {}), (dict(rgb=None), {}), (dict(alpha=None), {}),
           (dict(state=None), {}), (dict(batch_size=65536), {}), (dict(image_size=32768), {})]
    for f in (_lib.NR_TEX_FILL_BACK, _lib.NR_GRAD_INTERIOR, _lib.NR_RETURN_RGB, _lib.NR_RETURN_ALPHA,
              _lib.NR_RETURN_DEPTH, _lib.NR_ANTI_ALIASING, 1 << 31):
        bad.append((dict(flags=fl | f), {}))
    if indexed:
        bad += [(dict(vertices=None), {}), (dict(face_indices=None), {}), (dict(num_vertices=0), {})]
    else:
        bad += [(dict(faces=None), {})]
    if backward:
        bad += [(dict(grad_faces=_P), {})] if indexed else [(dict(grad_vertices=_P), {})]
        bad += [(dict(grad_vertices=None), {})] if indexed else [(dict(grad_faces=None), {})]
    for kw, ukw in bad:
        assert _call(lib, _args(indexed, backward, **kw), _uv(**ukw), backward) == INVALID, (kw, ukw)
        assert lib.nr_b200_last_launch_count() == 0
    # image offsets beyond 32 bits (face_uvs cannot get there within the binning's B F limit): after every invalid
    # argument, before the workspace
    for flags in (fl, fl | _lib.NR_TEX_MIPMAP):
        assert _call(lib, _args(indexed, backward, flags=flags), _uv(texture_height=30000, texture_width=30000),
                     backward) == UNSUPPORTED
        assert lib.nr_b200_last_launch_count() == 0
    assert _call(lib, _args(indexed, backward, textures=None), _uv(texture_height=30000, texture_width=30000),
                 backward) == INVALID
    fn = lib.nr_b200_soft_rgb_uv_backward if backward else lib.nr_b200_soft_rgb_uv
    assert fn(None, ctypes.byref(_uv()), None) == INVALID


@pytest.mark.parametrize("backward", [False, True])
def test_uv_null_is_the_cube_call(lib, backward):
    from neural_renderer_b200 import _lib
    cube = _args(False, backward, flags=0, texture_size=4, eps=1e-4)
    assert _call(lib, cube, None, backward) == WORKSPACE                  # accepted as nr_b200_soft_rgb(_backward)
    assert _call(lib, _args(False, backward, flags=0, texture_size=1, eps=1e-4), None, backward) == INVALID  # its rules
    assert _call(lib, _args(False, backward), None, backward) == INVALID  # NR_TEX_UV is refused by the cube call
    assert lib.nr_b200_last_launch_count() == 0
    # and the cube calls still refuse the image flags
    fn = lib.nr_b200_soft_rgb_backward if backward else lib.nr_b200_soft_rgb
    assert fn(ctypes.byref(_args(False, backward)), None) == INVALID


def test_python_argument_errors_come_before_the_device_check():
    import neural_renderer_b200 as nr
    faces = torch.zeros(1, 2, 3, 3)
    img = torch.zeros(8, 8, 3)
    uvs = torch.zeros(2, 3, 2)
    with pytest.raises(NotImplementedError):  # valid arguments on the CPU: no CPU path
        nr.rasterize_soft(faces, img, 16, face_uvs=uvs)
    with pytest.raises(NotImplementedError):
        nr.rasterize_soft(faces, img[None], 16, face_uvs=uvs[None], texture_filter='trilinear')
    for kw in (dict(texture_filter='nearest'), dict(texture_filter='trilinear', face_uvs=None),
               dict(face_uvs=torch.zeros(3, 3, 2)), dict(face_uvs=torch.zeros(2, 2, 2)), dict(face_uvs=torch.zeros(2, 2, 3, 2))):
        tex = img if kw.get("face_uvs", uvs) is not None else torch.zeros(1, 2, 4, 4, 4, 3)
        with pytest.raises(ValueError):
            nr.rasterize_soft(faces, tex, 16, **{"face_uvs": uvs, **kw})
    for tex in (torch.zeros(8, 8, 4), torch.zeros(2, 8, 8, 3), torch.zeros(1, 2, 4, 4, 4, 3)):
        with pytest.raises(ValueError):
            nr.rasterize_soft(faces, tex, 16, face_uvs=uvs)
    with pytest.raises(TypeError):
        nr.rasterize_soft(faces, img, 16, face_uvs=uvs.int())
    r = nr.Renderer()
    v, f = torch.zeros(1, 3, 3), torch.zeros(1, 1, 3, dtype=torch.int32)
    with pytest.raises(ValueError):
        r.render_soft(v, f, torch.zeros(8, 8, 3), face_uvs=torch.zeros(2, 3, 2))  # F = 1
    r.texture_filter = 'nearest'
    with pytest.raises(ValueError):
        r.render_soft(v, f, torch.zeros(8, 8, 3), face_uvs=torch.zeros(1, 3, 2))
    r = nr.Renderer()
    r.shading = 'phong'
    with pytest.raises(ValueError):
        r.render_soft(v, f, torch.zeros(8, 8, 3), face_uvs=torch.zeros(1, 3, 2))


# ------------------------------------------------------------------------------------------------ oracle self-checks
def _faces(seed, F=5, B=1):
    g = torch.Generator().manual_seed(seed)
    faces = torch.rand(B, F, 3, 3, generator=g, dtype=torch.float64) * 1.6 - 0.8
    faces[..., 2] = 1.0 + 3.0 * torch.rand(B, F, 3, generator=g, dtype=torch.float64)
    return faces


def test_uvs_on_one_texel_equal_the_cube_oracle_with_constant_cubes():
    g = torch.Generator().manual_seed(2)
    B, F, S, Ht, Wt = 1, 5, 24, 6, 7
    faces = _faces(1, F, B)
    img = torch.rand(1, Ht, Wt, 3, generator=g, dtype=torch.float64)
    cols = torch.randint(0, Wt, (F,), generator=g)
    rows = torch.randint(0, Ht, (F,), generator=g)
    uvs = torch.stack((cols.double() / (Wt - 1), 1.0 - rows.double() / (Ht - 1)), -1)[None, :, None].expand(1, F, 3, 2)
    cubes = img[0, rows, cols][None, :, None, None, None].expand(1, F, 2, 2, 2, 3)
    light = torch.rand(B, F, 3, generator=g, dtype=torch.float64)
    for kw in (dict(), dict(face_light=light)):
        want = orgb.soft_rgb(faces, cubes, S, 1e-3, 1e-2, background=(0.1, 0.2, 0.3), **kw)
        got = ouv.soft_uv(faces, img, uvs, S, 1e-3, 1e-2, background=(0.1, 0.2, 0.3), **kw)
        torch.testing.assert_close(got[0], want[0], rtol=1e-12, atol=1e-13)
        assert torch.equal(got[1], want[1])


def test_sigma_gamma_to_zero_is_a_hard_uv_sample_inside_one_face():
    g = torch.Generator().manual_seed(3)
    S, Ht, Wt = 32, 9, 11
    faces = torch.tensor([[[[-0.7, -0.6, 2.0], [0.8, -0.5, 3.0], [0.1, 0.75, 4.0]]]], dtype=torch.float64)
    uvs = torch.tensor([[[[0.1, 0.2], [0.9, 0.3], [0.4, 0.95]]]], dtype=torch.float64)
    img = torch.rand(1, Ht, Wt, 3, generator=g, dtype=torch.float64)
    rgb, alpha = ouv.soft_uv(faces, img, uvs, S, 1e-9, 1e-7)
    # independent restatement: screen barycentrics by a linear solve, perspective correction, then a bilinear tap blend
    xs = (2 * np.arange(S) + 1 - S) / S
    v = faces[0, 0].numpy()
    M = np.array([[v[0, 0], v[1, 0], v[2, 0]], [v[0, 1], v[1, 1], v[2, 1]], [1.0, 1.0, 1.0]])
    n = 0
    for r in range(S):
        for c in range(S):
            w = np.linalg.solve(M, [xs[c], xs[S - 1 - r], 1.0])
            if w.min() < 0.05:
                continue                                  # away from the edges
            q = w / v[:, 2]
            lp = q / q.sum()
            u, t = lp @ uvs[0, 0].numpy()
            px, py = u * (Wt - 1), t * (Ht - 1)
            ix, iy = int(np.floor(px)), int(np.floor(py))
            fx, fy = px - ix, py - iy
            I = img[0].numpy()[::-1]                      # tap coordinates: y up from the bottom row
            want = ((1 - fx) * (1 - fy) * I[iy, ix] + (1 - fx) * fy * I[iy + 1, ix] + fx * (1 - fy) * I[iy, ix + 1]
                    + fx * fy * I[iy + 1, ix + 1])
            np.testing.assert_allclose(rgb[0, :, r, c].numpy(), want, rtol=0, atol=1e-9)
            n += 1
    assert n > 100


def test_magnified_image_gives_trilinear_equal_to_bilinear():
    g = torch.Generator().manual_seed(4)
    S, Ht, Wt = 40, 5, 6
    faces = _faces(5, 4)
    uvs = 0.4 + 0.05 * torch.rand(1, 4, 3, 2, generator=g, dtype=torch.float64)  # well under a texel per pixel
    img = torch.rand(1, Ht, Wt, 3, generator=g, dtype=torch.float64)
    pyr = torch.cat([t.reshape(1, -1, 3) for t in oracles.pyramid64(img)], 1)
    bil = ouv.soft_uv(faces, img, uvs, S, 1e-4, 1e-3)
    tri = ouv.soft_uv(faces, pyr, uvs, S, 1e-4, 1e-3, hw=(Ht, Wt))
    torch.testing.assert_close(tri[0], bil[0], rtol=0, atol=0)
    # minified: the pyramid's coarser levels do change the image
    tri_min = ouv.soft_uv(faces, torch.cat([t.reshape(1, -1, 3) for t in oracles.pyramid64(
        torch.rand(1, 256, 256, 3, generator=g, dtype=torch.float64))], 1), uvs, S, 1e-4, 1e-3, hw=(256, 256))
    bil_min = ouv.soft_uv(faces, tri_min[0].new_zeros(1, 1, 1, 3), uvs, S, 1e-4, 1e-3)
    assert not torch.equal(tri_min[0], bil_min[0])


def test_new_kernels_compile_for_sm90a_without_spills(tmp_path):
    from neural_renderer_b200 import build
    nvcc = os.environ.get("NVCC", "nvcc")
    cmd = [nvcc] + build.NVCC_FLAGS + ["-Xptxas", "-v", "-c", os.path.join(build.CSRC, "nr_soft_uv.cu"),
                                       "-o", str(tmp_path / "nr_soft_uv.o")]
    log = subprocess.run(cmd, capture_output=True, text=True, check=True).stderr
    entries = re.split(r"Compiling entry function '", log)[1:]
    names = [e.split("'")[0] for e in entries]
    # forward and backward, bilinear and trilinear, 32- and 64-bit keys; the binning kernels are nr_soft_rgb.cu's
    assert len(entries) == 8 and all("k_soft_uv_" in n for n in names), names
    for e in entries:
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", e)
        assert m and m.groups() == ("0", "0", "0"), e[:400]
    assert "sm_90a" in log
