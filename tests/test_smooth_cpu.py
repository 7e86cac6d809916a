"""CPU: smooth shading -- the torch formulations of F.vertex_normals / F.corner_light against float64 hand formulas, the
appended forward field corner_light against the header, the accepted struct sizes and the host-side rejections of
nr_b200_forward and nr_b200_backward_corner_light, all decided before any device work."""
import ctypes
import os

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# Fake, never dereferenced device addresses (as test_uv_grad_cpu.py): a complete argument set gets as far as the
# workspace check (NR_ERR_WORKSPACE, no workspace given); each broken one must stop earlier.
_P = 0x10000
OK_UP_TO_WORKSPACE, INVALID = -2, -1


@pytest.fixture(scope="module")
def lib():
    from neural_renderer_b200 import build, _lib
    build.build_library()
    return _lib.load()


# ---------------------------------------------------------------------------------------------- torch formulations
def _hand_normals(v, faces):
    """float64 loops: s_v = sum over corners (f, k) at v of cross(v0 - v1, v2 - v1), faces with an index out of range
    skipped, n = s / (|s| + 1e-5)"""
    v = np.asarray(v, np.float64)
    s = np.zeros_like(v)
    for tri in np.asarray(faces):
        if not all(0 <= i < len(v) for i in tri):
            continue
        c = np.cross(v[tri[0]] - v[tri[1]], v[tri[2]] - v[tri[1]])
        for i in tri:
            s[i] += c
    return s / (np.linalg.norm(s, axis=1, keepdims=True) + 1e-5)


def test_vertex_normals_are_area_weighted():
    from neural_renderer_b200 import functional as F
    # two triangles at vertex 0: a large one in the z = 0 plane and a small one in the x = 0 plane
    v = torch.tensor([[0, 0, 0], [4, 0, 0], [0, 4, 0], [0, 0, 1], [0, 1, 0]], dtype=torch.float64)
    faces = torch.tensor([[0, 1, 2], [0, 4, 3]])
    n = F.vertex_normals(v[None], faces)[0]
    np.testing.assert_allclose(n.numpy(), _hand_normals(v, faces), rtol=1e-12, atol=1e-15)
    # the large face dominates vertex 0 by its area: (0, 0, -16) + (-1, 0, 0) before normalising
    s = np.array([-1.0, 0.0, -16.0])
    np.testing.assert_allclose(n[0].numpy(), s / (np.linalg.norm(s) + 1e-5), rtol=1e-12)


def test_vertex_normals_unreferenced_and_out_of_range():
    from neural_renderer_b200 import functional as F
    g = torch.Generator().manual_seed(0)
    v = torch.randn((2, 9, 3), generator=g, dtype=torch.float64)
    faces = torch.tensor([[0, 1, 2], [2, 1, 3], [3, 4, 0], [4, 9, 1], [-1, 2, 3], [5, 6, 7]])  # vertex 8 unreferenced
    n = F.vertex_normals(v, faces)
    for b in range(2):
        np.testing.assert_allclose(n[b].numpy(), _hand_normals(v[b], faces), rtol=1e-12, atol=1e-15)
    assert (n[:, 8] == 0).all()
    # per-item index sets
    faces_b = torch.stack((faces, faces.flip(0)))
    np.testing.assert_allclose(F.vertex_normals(v, faces_b)[1].numpy(), _hand_normals(v[1], faces.flip(0)), rtol=1e-12,
                               atol=1e-15)


def _hand_corner_light(n, faces, amb, dirc, d, fill_back):
    n = np.asarray(n, np.float64)
    faces = np.asarray(faces)
    F = len(faces)
    out = np.zeros((F, 3, 3))
    for f, tri in enumerate(faces):
        sgn = -1.0 if (fill_back and f >= F // 2) else 1.0
        for k, i in enumerate(tri):
            nv = n[i] if 0 <= i < len(n) else np.zeros(3)
            out[f, k] = amb + dirc * max(sgn * float(nv @ d), 0.0)
    return out


@pytest.mark.parametrize("fill_back", [False, True])
def test_corner_light_formula_and_fill_back_sign(fill_back):
    from neural_renderer_b200 import functional as F
    g = torch.Generator().manual_seed(1)
    n = torch.nn.functional.normalize(torch.randn((1, 7, 3), generator=g, dtype=torch.float64), dim=2)
    front = torch.tensor([[0, 1, 2], [2, 3, 4], [4, 5, 6], [6, 7, 0]])  # index 7 is out of range: n = 0
    faces = torch.cat((front, front.flip(1))) if fill_back else front
    ia, idr, ca, cd, d = 0.3, 0.6, (1.0, 0.5, 0.2), (0.2, 0.9, 1.0), (0.3, -0.8, 0.5)
    got = F.corner_light(n, faces, ia, idr, ca, cd, d, fill_back=fill_back)[0]
    want = _hand_corner_light(n[0], faces, ia * np.array(ca), idr * np.array(cd), np.array(d), fill_back)
    np.testing.assert_allclose(got.numpy(), want, rtol=1e-12, atol=1e-15)
    if fill_back:  # a copy lit from the other side: one of a corner pair is ambient only
        lit = got[:4, :, 0] > ia * ca[0] + 1e-12
        lit_copy = got[4:, :, 0].flip(1) > ia * ca[0] + 1e-12
        assert not (lit & lit_copy).any()
    with pytest.raises(ValueError):
        F.corner_light(n, front[:3], fill_back=True)


def test_smooth_light_of_a_flat_mesh_equals_face_light():
    """a planar mesh: every vertex normal is the face normal, so corner light = face_light at every corner (up to the
    1e-5 of the normalisation, which weighs a sum of two face normals slightly differently from one)"""
    from neural_renderer_b200 import functional as F
    v = torch.tensor([[[0, 0, 0], [1, 0, 0], [1, 1, 0], [0, 1, 0]]], dtype=torch.float64)
    faces = torch.tensor([[0, 1, 2], [0, 2, 3]])
    args = (0.4, 0.6, (1, 1, 1), (1, 1, 1), (0.2, 0.3, -0.9))
    cl = F.corner_light(F.vertex_normals(v, faces), faces, *args)
    fl = F.face_light(F.vertices_to_faces(v, faces[None]), *args)
    np.testing.assert_allclose(cl.numpy(), fl[:, :, None, :].expand(-1, -1, 3, -1).numpy(), rtol=1e-5)


# ----------------------------------------------------------------------------------------------------- C ABI
def test_corner_light_field_matches_the_header(tmp_path):
    import subprocess
    from neural_renderer_b200 import _lib
    exprs = ["sizeof(nr_b200_forward_args)", "offsetof(nr_b200_forward_args, corner_light)",
             "offsetof(nr_b200_forward_args, texture_width) + sizeof(int32_t)", "sizeof(nr_b200_backward_args)"]
    src = tmp_path / "s.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "nr_b200.h"\nint main(void){'
                   + "".join('printf("%%zu\\n", (size_t)(%s));' % e for e in exprs) + "return 0;}\n")
    exe = tmp_path / "s"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    fsize, fcl, fend4, bsize = (int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split())
    assert fsize == ctypes.sizeof(_lib.ForwardArgs) and fcl == _lib.ForwardArgs.corner_light.offset
    assert fcl == fend4 and fsize == fcl + 8  # appended right after the ABI-4 fields, nothing else moved
    assert bsize == ctypes.sizeof(_lib.BackwardArgs)  # the backward struct is unchanged: its pointers are call arguments
    assert [f[0] for f in _lib.ForwardArgs._fields_][-4:] == ["face_uvs", "texture_height", "texture_width", "corner_light"]
    assert "corner_light" not in [f[0] for f in _lib.BackwardArgs._fields_]


def _fwd(flags, corner=True, face_light=False, struct_size=None):
    from neural_renderer_b200 import _lib
    a = _lib.ForwardArgs()
    a.struct_size = ctypes.sizeof(_lib.ForwardArgs) if struct_size is None else struct_size
    a.flags = flags
    a.batch_size, a.num_faces, a.raster_size, a.texture_size = 2, 4, 16, 2
    a.near_, a.far_, a.eps = 0.1, 100.0, 1e-4
    a.faces = a.textures = a.face_index_map = a.weight_map = a.depth_map = a.rgb_map = a.alpha_map = _P
    a.corner_light = _P if corner else None
    a.face_light = _P if face_light else None
    return a


def _bwd(flags, face_light=False, textures=True, struct_size=None):
    from neural_renderer_b200 import _lib
    a = _lib.BackwardArgs()
    a.struct_size = ctypes.sizeof(_lib.BackwardArgs) if struct_size is None else struct_size
    a.flags = flags
    a.batch_size, a.num_faces, a.raster_size, a.texture_size = 2, 4, 16, 2
    a.eps = 1e-4
    a.faces = a.face_index_map = a.weight_map = a.depth_map = a.rgb_map = a.grad_faces = a.grad_textures = _P
    a.textures = _P if textures else None
    a.face_light = _P if face_light else None
    return a


def test_forward_struct_sizes_and_rejections(lib):
    from neural_renderer_b200 import _lib
    rgb, alpha = _lib.NR_RETURN_RGB, _lib.NR_RETURN_ALPHA
    full, abi4 = ctypes.sizeof(_lib.ForwardArgs), _lib.ForwardArgs.corner_light.offset

    def run(a):
        return lib.nr_b200_forward(ctypes.byref(a), None)
    assert run(_fwd(rgb)) == OK_UP_TO_WORKSPACE
    assert run(_fwd(rgb | _lib.NR_ANTI_ALIASING)) == OK_UP_TO_WORKSPACE
    assert run(_fwd(rgb, struct_size=abi4)) == OK_UP_TO_WORKSPACE
    # the short struct does not read corner_light: with face_light also set, the long one is refused, the short one not
    assert run(_fwd(rgb, face_light=True, struct_size=abi4)) == OK_UP_TO_WORKSPACE
    assert run(_fwd(rgb, face_light=True)) == INVALID
    assert run(_fwd(alpha)) == INVALID                        # corner_light lights the RGB image only
    assert run(_fwd(alpha, corner=False)) == OK_UP_TO_WORKSPACE
    for size in (abi4 - 8, abi4 - 1, abi4 + 1, abi4 + 4, full - 1, full + 1, full + 8):
        assert run(_fwd(rgb, struct_size=size)) == INVALID, size


def test_backward_corner_light_rejections(lib):
    from neural_renderer_b200 import _lib
    rgb, alpha, acc = _lib.NR_RETURN_RGB, _lib.NR_RETURN_ALPHA, _lib.NR_GRAD_ACCUMULATE
    part_t, part_f = _lib.NR_BWD_PART_TEXTURES, _lib.NR_BWD_PART_FACES
    full, short = ctypes.sizeof(_lib.BackwardArgs), _lib.BackwardArgs.grad_face_uvs.offset

    def run(flags, corner=True, grad_corner=True, **kw):
        return lib.nr_b200_backward_corner_light(ctypes.byref(_bwd(flags, **kw)), _P if corner else None,
                                                 _P if grad_corner else None, None)
    for ok in (rgb, rgb | acc, rgb | part_t, rgb | part_f, rgb | alpha):
        assert run(ok) == OK_UP_TO_WORKSPACE, hex(ok)
    assert run(rgb, grad_corner=False) == OK_UP_TO_WORKSPACE
    assert run(rgb, struct_size=short) == OK_UP_TO_WORKSPACE     # both backward struct layouts
    assert run(rgb, face_light=True) == INVALID                  # exclusive with face_light
    assert run(alpha) == INVALID                                 # needs RGB
    assert run(rgb, textures=False) == INVALID                   # d / d corner_light reads the unlit textures
    assert run(rgb, textures=False, grad_corner=False) == OK_UP_TO_WORKSPACE
    assert run(rgb, corner=False) == INVALID                     # the entry point of a smooth-shaded forward
    assert run(rgb, corner=False, grad_corner=False) == INVALID
    for size in (short - 4, short + 4, full - 4, full + 8):
        assert run(rgb, struct_size=size) == INVALID, size
    # the plain backward is unchanged by all this: the same complete call without the pointers
    assert lib.nr_b200_backward(ctypes.byref(_bwd(rgb)), None) == OK_UP_TO_WORKSPACE
