"""CPU: soft RGB -- nr_b200_soft_rgb_args against the header, the new symbols, the host rejections of both entry points
(all decided before any device work), the workspace query, the Python argument errors (raised before the device check),
the float64 oracle against closed forms and limits, and the registers / spills of the new kernels."""
import ctypes
import math
import os
import re
import subprocess

import pytest
import torch

import oracles_soft as osoft
import oracles_soft_rgb as orgb

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


def test_soft_rgb_struct_matches_the_header(tmp_path):
    from neural_renderer_b200 import _lib
    fields = [f[0] for f in _lib.SoftRgbArgs._fields_]
    exprs = ["sizeof(nr_b200_soft_rgb_args)"] + ["offsetof(nr_b200_soft_rgb_args, %s)" % f for f in fields]
    src = tmp_path / "s.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "nr_b200.h"\nint main(void){'
                   + "".join('printf("%%zu\\n", (size_t)(%s));' % e for e in exprs)
                   + 'printf("%.17g\\n", (double)(NR_SOFT_BG_DEPTH));return 0;}\n')
    exe = tmp_path / "s"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    out = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()
    vals = [int(x) for x in out[:-1]]
    assert vals[0] == ctypes.sizeof(_lib.SoftRgbArgs) == 192
    assert vals[1:] == [getattr(_lib.SoftRgbArgs, f).offset for f in fields]
    assert float(out[-1]) == _lib.SOFT_BG_DEPTH == orgb.BG_DEPTH


def test_new_symbols_are_exported(lib):
    from neural_renderer_b200 import _lib
    names = ("nr_b200_soft_rgb_workspace_bytes", "nr_b200_soft_rgb", "nr_b200_soft_rgb_backward")
    out = subprocess.run(["nm", "-D", "--defined-only", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    for n in names:
        assert n in _lib.EXPORTED_SYMBOLS
        assert (" T " + n) in out, n


def test_workspace_query(lib):
    from neural_renderer_b200 import _lib
    n = lib.nr_b200_soft_rgb_workspace_bytes(64, 5000, 256, 0)
    # CUB sizes the sort's scratch for the current device: without one the query returns 0
    if torch.cuda.is_available():
        # face and depth records, tile boxes, two key lists of at most 16 entries per face
        assert n >= 64 * 5000 * (64 + 16 + 8 + 2 * 16 * 4)
        assert lib.nr_b200_soft_rgb_workspace_bytes(64, 5000, 256, _lib.NR_FACES_INDEXED | _lib.NR_TEX_SHARED) == n
    for bad in [(0, 5, 16, 0), (1, 0, 16, 0), (1, 5, 0, 0), (65536, 1, 16, 0), (1, 1, 32768, 0), (1024, 1 << 17, 16, 0),
                (1, 5, 16, _lib.NR_TEX_UV), (1, 5, 16, _lib.NR_TEX_FILL_BACK), (1, 5, 16, _lib.NR_RETURN_RGB)]:
        assert lib.nr_b200_soft_rgb_workspace_bytes(*bad) == 0, bad


def _args(indexed=False, backward=False, **kw):
    from neural_renderer_b200 import _lib
    a = _lib.SoftRgbArgs()
    a.struct_size = ctypes.sizeof(_lib.SoftRgbArgs)
    a.flags = _lib.NR_FACES_INDEXED if indexed else 0
    a.batch_size, a.num_faces, a.image_size, a.num_vertices, a.texture_size = 2, 4, 16, 6 if indexed else 0, 4
    a.sigma, a.gamma, a.near_, a.far_, a.eps = 1e-4, 1e-4, 0.1, 100.0, 1e-4
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


def _call(lib, a, backward):
    fn = lib.nr_b200_soft_rgb_backward if backward else lib.nr_b200_soft_rgb
    return fn(ctypes.byref(a), None)


@pytest.mark.parametrize("backward", [False, True])
@pytest.mark.parametrize("indexed", [False, True])
def test_host_rejections(lib, indexed, backward):
    from neural_renderer_b200 import _lib
    ok = _args(indexed, backward)
    assert _call(lib, ok, backward) == WORKSPACE
    assert lib.nr_b200_last_launch_count() == 0
    # every allowed NULL and flag: face_light, grad_rgb / grad_alpha, grad_textures / grad_face_light, shared sets
    allowed = [dict(face_light=None), dict(face_light=_P), dict(flags=ok.flags | _lib.NR_TEX_SHARED),
               dict(flags=ok.flags | _lib.NR_GRAD_ACCUMULATE)]
    if backward:
        allowed += [dict(grad_rgb=None), dict(grad_alpha=None), dict(grad_rgb=None, grad_alpha=None),
                    dict(grad_textures=_P, grad_face_light=_P)]
    if indexed:
        allowed += [dict(flags=_lib.NR_FACES_INDEXED | _lib.NR_INDICES_SHARED)]
    for kw in allowed:
        assert _call(lib, _args(indexed, backward, **kw), backward) == WORKSPACE, kw
    bad = [dict(struct_size=4), dict(struct_size=ctypes.sizeof(_lib.SoftRgbArgs) + 8),
           dict(struct_size=ctypes.sizeof(_lib.SoftArgs)), dict(batch_size=0), dict(num_faces=0), dict(image_size=0),
           dict(batch_size=-1), dict(sigma=0.0), dict(sigma=-1e-5), dict(sigma=float("nan")), dict(sigma=float("inf")),
           dict(gamma=0.0), dict(gamma=-1e-4), dict(gamma=float("nan")), dict(gamma=float("inf")),
           dict(near_=2.0, far_=1.0), dict(near_=1.0, far_=1.0), dict(near_=float("nan")), dict(eps=float("nan")),
           dict(texture_size=1), dict(texture_size=0), dict(texture_size=1000), dict(textures=None), dict(rgb=None),
           dict(alpha=None), dict(state=None), dict(batch_size=65536), dict(image_size=32768),
           dict(batch_size=1024, num_faces=1 << 17)]
    for fl in (_lib.NR_TEX_UV, _lib.NR_TEX_MIPMAP, _lib.NR_TEX_FILL_BACK, _lib.NR_RETURN_RGB, _lib.NR_ANTI_ALIASING,
               _lib.NR_UV_SHARED, _lib.NR_GRAD_INTERIOR, 1 << 31):
        bad.append(dict(flags=ok.flags | fl))
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
    fn = lib.nr_b200_soft_rgb_backward if backward else lib.nr_b200_soft_rgb
    assert fn(None, None) == INVALID
    # the silhouettes' struct_size check still refuses exactly what it did
    assert lib.nr_b200_soft_silhouettes(ctypes.byref(_lib.SoftArgs(struct_size=ctypes.sizeof(_lib.SoftRgbArgs))), None) == INVALID


def test_python_argument_errors_come_before_the_device_check():
    import neural_renderer_b200 as nr
    faces = torch.zeros(1, 2, 3, 3)
    tex = torch.zeros(1, 2, 4, 4, 4, 3)
    with pytest.raises(NotImplementedError):  # valid arguments on the CPU: no CPU path
        nr.rasterize_soft(faces, tex, 16)
    with pytest.raises(NotImplementedError):
        nr.rasterize_soft(torch.zeros(2, 3, dtype=torch.int32), tex, 16, vertices=torch.zeros(1, 3, 3))
    for kw in (dict(sigma=0.0), dict(sigma=-1e-5), dict(sigma=float("nan")), dict(gamma=0.0), dict(gamma=-1.0),
               dict(gamma=float("inf")), dict(near=2.0, far=1.0), dict(near=1.0, far=1.0), dict(image_size=0),
               dict(background_color=(0, 0))):
        with pytest.raises(ValueError):
            nr.rasterize_soft(faces, tex, **{"image_size": 16, **kw})
    with pytest.raises(TypeError):
        nr.rasterize_soft(faces, tex, 16, gamma="x")
    with pytest.raises(ValueError):
        nr.rasterize_soft(faces, torch.zeros(1, 3, 4, 4, 4, 3), 16)         # cube count != faces
    with pytest.raises(ValueError):
        nr.rasterize_soft(faces, torch.zeros(1, 2, 1, 1, 1, 3), 16)         # ts < 2
    with pytest.raises(ValueError):
        nr.rasterize_soft(faces, tex, 16, face_light=torch.zeros(1, 2, 4))
    with pytest.raises(TypeError):
        nr.rasterize_soft(faces, None, 16)
    import neural_renderer
    assert neural_renderer.rasterize_soft is nr.rasterize_soft
    assert nr.DEFAULT_SOFT_GAMMA == neural_renderer.DEFAULT_SOFT_GAMMA == 1e-4
    r = nr.Renderer()
    for attr, val in (("shading", "smooth"), ("shading", "phong"), ("lights", [object()]),
                      ("environment_sh", torch.zeros(9, 3)), ("normal_map", torch.zeros(2, 2, 3)),
                      ("specular_map", torch.zeros(2, 2, 4))):
        r = nr.Renderer()
        setattr(r, attr, val)
        with pytest.raises(ValueError):
            r.render_soft(torch.zeros(1, 3, 3), torch.zeros(1, 3, dtype=torch.int32), torch.zeros(1, 1, 2, 2, 2, 3))


# ------------------------------------------------------------------------------------------------ oracle self-checks
def _tri(pts, z=1.0):
    return torch.tensor([[[[p[0], p[1], z] for p in pts]]], dtype=torch.float64)  # [1,1,3,3]


def _const_cube(color, ts=2, F=1):
    return torch.tensor(color, dtype=torch.float64).expand(1, F, ts, ts, ts, 3).clone()


def test_single_face_closed_form():
    faces = _tri([(-0.5, -0.4), (0.6, -0.3), (0.0, 0.7)], z=2.0)
    col, bg = (0.2, 0.5, 0.9), (0.3, 0.1, 0.05)
    S, sigma, gamma, near, far = 24, 1e-3, 1e-2, 0.1, 100.0
    rgb, alpha = orgb.soft_rgb(faces, _const_cube(col), S, sigma, gamma, near, far, background=bg)
    p = osoft.pixel_centres(S)
    d2, inside = osoft.face_terms(faces, p)
    x = torch.where(inside, d2 / sigma, -d2 / sigma)[0, 0]
    on = (inside | (d2 <= osoft.cut(sigma)))[0, 0]
    D = torch.sigmoid(x)
    zn = (far - 2.0) / (far - near)
    zmax = max(zn, orgb.BG_DEPTH)
    w = torch.where(on, D * math.exp((zn - zmax) / gamma), torch.zeros_like(D))
    wb = math.exp((orgb.BG_DEPTH - zmax) / gamma)
    for c in range(3):
        want = (w * col[c] + wb * bg[c]) / (w + wb)
        torch.testing.assert_close(rgb[0, c].reshape(-1), want, rtol=1e-12, atol=1e-14)
    torch.testing.assert_close(alpha[0].reshape(-1), torch.where(on, D, torch.zeros_like(D)), rtol=1e-12, atol=1e-14)


def test_pixel_without_a_face_is_the_background_exactly():
    faces = _tri([(-0.2, -0.2), (0.0, -0.2), (-0.1, 0.0)])
    bg = (0.25, 0.5, 0.75)
    rgb, alpha = orgb.soft_rgb(faces, _const_cube((1.0, 0.0, 0.0)), 32, 1e-5, 1e-4, background=bg)
    far_px = alpha[0] == 0
    assert far_px.sum() > 500
    for c in range(3):
        assert torch.all(rgb[0, c][far_px] == bg[c])


def test_shift_invariance_in_zmax():
    """the aggregation with zmax moved by any constant is the same image: it only rescales numerator and Z"""
    g = torch.Generator().manual_seed(4)
    w = torch.rand(5, 7, generator=g, dtype=torch.float64)
    zn = torch.rand(5, 7, generator=g, dtype=torch.float64)
    C = torch.rand(5, 7, 3, generator=g, dtype=torch.float64)
    gamma = 0.05

    def agg(zmax):
        e = w * torch.exp((zn - zmax[:, None]) / gamma)
        eb = torch.exp((orgb.BG_DEPTH - zmax) / gamma)
        return ((e[..., None] * C).sum(1) + eb[:, None] * 0.3) / (e.sum(1) + eb)[:, None]

    ref = agg(zn.amax(1).clamp_min(orgb.BG_DEPTH))
    for shift in (-0.2, 0.1, 0.5):
        torch.testing.assert_close(agg(zn.amax(1) + shift), ref, rtol=1e-12, atol=1e-13)


def test_zero_area_faces_count_in_alpha_but_not_in_rgb():
    S, sigma, gamma = 32, 1e-3, 1e-2
    tri = _tri([(-0.5, -0.5), (0.5, -0.5), (0.0, 0.5)], z=2.0)[0, 0]
    line = torch.tensor([[-0.6, -0.6, 1.0], [-0.2, -0.2, 1.0], [-0.4, -0.4, 1.0]], dtype=torch.float64)  # collinear
    point = torch.tensor([[0.6, 0.2, 1.0]] * 3, dtype=torch.float64)
    faces = torch.stack((tri, line, point))[None]
    tex = torch.cat((_const_cube((0.0, 1.0, 0.0)), _const_cube((1.0, 0.0, 0.0), F=2)), 1)
    assert torch.all(orgb.doubled_area(faces)[0, 1:] == 0)
    rgb, alpha = orgb.soft_rgb(faces, tex, S, sigma, gamma)
    rgb1, alpha1 = orgb.soft_rgb(faces[:, :1], tex[:, :1], S, sigma, gamma)
    assert torch.equal(rgb, rgb1)               # no red anywhere: the zero-area faces add no colour
    assert (alpha > alpha1 + 1e-6).sum() > 10   # but they do add coverage
    torch.testing.assert_close(alpha, osoft.soft_silhouettes(faces, S, sigma), rtol=1e-12, atol=1e-14)


def test_small_gamma_picks_the_nearest_face():
    S, sigma = 32, 1e-3
    a = _tri([(-0.7, -0.6), (0.7, -0.6), (0.0, 0.7)], z=3.0)[0, 0]
    b = a.clone()
    b[:, 2] = 2.0                               # the same triangle, nearer
    faces = torch.stack((a, b))[None]
    tex = torch.cat((_const_cube((1.0, 0.0, 0.0)), _const_cube((0.0, 0.0, 1.0))), 1)
    rgb, alpha = orgb.soft_rgb(faces, tex, S, sigma, 1e-6)
    inner = alpha[0] > 0.999
    assert inner.sum() > 100
    torch.testing.assert_close(rgb[0, 2][inner], torch.ones_like(rgb[0, 2][inner]), rtol=0, atol=1e-12)
    torch.testing.assert_close(rgb[0, 0][inner], torch.zeros_like(rgb[0, 0][inner]), rtol=0, atol=1e-12)


def test_sigma_gamma_to_zero_is_the_hard_rgb_away_from_edges_and_ties():
    g = torch.Generator().manual_seed(5)
    B, F, ts, S = 1, 6, 3, 40
    faces = torch.rand(B, F, 3, 3, generator=g, dtype=torch.float64) * 1.6 - 0.8
    faces[..., 2] = 1.0 + 3.0 * torch.rand(B, F, 3, generator=g, dtype=torch.float64)
    tex = torch.rand(B, F, ts, ts, ts, 3, generator=g, dtype=torch.float64)
    bg = (0.1, 0.2, 0.3)
    rgb, _ = orgb.soft_rgb(faces, tex, S, 1e-9, 1e-7, background=bg)
    hard = orgb.hard_rgb_cpu(faces, tex, S, background=bg)
    # pixels more than 1 px from every edge, and whose two nearest covering depths differ clearly
    p = osoft.pixel_centres(S)
    d2, _ = osoft.face_terms(faces, p)
    away = (d2 > (2.0 / S) ** 2).all(1)[0]
    A = orgb.doubled_area(faces)[..., None]
    lam = orgb.edge_functions(faces, p).roll(-1, dims=2) / A[:, :, None]
    cover = (lam > 0).all(2)
    l = lam.clamp(0, 1)
    zp = 1.0 / (l / l.sum(2, keepdim=True) / faces[..., 2][..., None]).sum(2)
    zs = torch.where(cover, zp, torch.full_like(zp, math.inf)).sort(1).values[0]
    untied = (zs[1] - zs[0] > 1e-3) | torch.isinf(zs[1])
    ok = away & untied
    assert ok.sum() > S * S // 2
    got, want = rgb[0].reshape(3, -1)[:, ok], hard[0].reshape(3, -1)[:, ok]
    torch.testing.assert_close(got, want, rtol=0, atol=1e-9)


def test_new_kernels_compile_for_sm90a_without_spills(tmp_path):
    from neural_renderer_b200 import build
    nvcc = os.environ.get("NVCC", "nvcc")
    cmd = [nvcc] + build.NVCC_FLAGS + ["-Xptxas", "-v", "-c", os.path.join(build.CSRC, "nr_soft_rgb.cu"),
                                       "-o", str(tmp_path / "nr_soft_rgb.o")]
    log = subprocess.run(cmd, capture_output=True, text=True, check=True).stderr
    entries = re.split(r"Compiling entry function '", log)[1:]
    ours = [e for e in entries if "k_soft_" in e.split("'")[0]]
    names = [e.split("'")[0] for e in ours]
    # keys, fill, forward and backward for 32- and 64-bit keys, and the silhouettes' setup reused
    assert len(ours) == 9, names
    for e in ours:
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", e)
        assert m and m.groups() == ("0", "0", "0"), e[:400]
    assert "sm_90a" in log
