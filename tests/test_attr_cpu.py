"""CPU: attribute interpolation -- the nr_b200_interpolate_args layout against the header, the exported entry points, every
host-side rejection of nr_b200_interpolate / nr_b200_interpolate_backward (decided before any device work), the Python
argument errors of rasterize_attributes, and the header's closed-form interior vertex gradient against float64 autograd of
the oracle in oracles_attr.py."""
import ctypes
import os

import numpy as np
import pytest
import torch

from oracles_attr import interior_grad64, interp64

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_P = 0x10000  # a fake, never dereferenced device address
INVALID = -1


@pytest.fixture(scope="module")
def lib():
    from neural_renderer_b200 import build, _lib
    build.build_library()
    return _lib.load()


def test_struct_layout_matches_the_header(tmp_path):
    import subprocess
    from neural_renderer_b200 import _lib
    names = [f[0] for f in _lib.InterpolateArgs._fields_]
    exprs = ["sizeof(nr_b200_interpolate_args)"] + ["offsetof(nr_b200_interpolate_args, %s)" % n for n in names]
    exprs += ["NR_ATTR_PER_VERTEX", "NR_ATTR_SHARED"]
    src = tmp_path / "s.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "nr_b200.h"\nint main(void){'
                   + "".join('printf("%%zu\\n", (size_t)(%s));' % e for e in exprs) + "return 0;}\n")
    exe = tmp_path / "s"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    vals = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert vals[0] == ctypes.sizeof(_lib.InterpolateArgs)
    assert vals[1:1 + len(names)] == [getattr(_lib.InterpolateArgs, n).offset for n in names]
    assert vals[-2:] == [_lib.NR_ATTR_PER_VERTEX, _lib.NR_ATTR_SHARED]


def test_entry_points_are_exported(lib):
    from neural_renderer_b200 import _lib
    for name in ("nr_b200_interpolate", "nr_b200_interpolate_backward"):
        assert name in _lib.EXPORTED_SYMBOLS
        assert getattr(lib, name).restype == ctypes.c_int


def _args(flags=0, indexed=False, **kw):
    from neural_renderer_b200 import _lib
    a = _lib.InterpolateArgs()
    a.struct_size = ctypes.sizeof(_lib.InterpolateArgs)
    a.flags = flags | (_lib.NR_FACES_INDEXED if indexed else 0)
    a.batch_size, a.num_faces, a.raster_size, a.channels = 2, 4, 16, 3
    if indexed:
        a.vertices, a.face_indices, a.num_vertices = _P, _P, 6
    else:
        a.faces = _P
    a.face_index_map = a.weight_map = a.attributes = a.out = _P
    for k, v in kw.items():
        setattr(a, k, v)
    return a


def _cases():
    """(description, args, forward rejects, backward rejects) -- every argument set the header refuses"""
    from neural_renderer_b200 import _lib
    pv, aa = _lib.NR_ATTR_PER_VERTEX, _lib.NR_ANTI_ALIASING
    size = ctypes.sizeof(_lib.InterpolateArgs)
    return [
        ("C = 0", _args(channels=0)), ("C < 0", _args(channels=-2)),
        ("B = 0", _args(batch_size=0)), ("F = 0", _args(num_faces=0)), ("S = 0", _args(raster_size=0)),
        ("no face_index_map", _args(face_index_map=None)), ("no weight_map", _args(weight_map=None)),
        ("no attributes", _args(attributes=None)),
        ("per vertex, faces geometry", _args(pv)),
        ("no faces", _args(faces=None)), ("indexed without vertices", _args(indexed=True, vertices=None)),
        ("indexed without indices", _args(indexed=True, face_indices=None)),
        ("indexed with Nv 0", _args(indexed=True, num_vertices=0)),
        ("per vertex with Nv 0", _args(pv, indexed=True, num_vertices=0)),
        ("odd raster with anti-aliasing", _args(aa, raster_size=15)),
        ("short struct", _args(struct_size=size - 8)), ("long struct", _args(struct_size=size + 8)),
        ("raster beyond 32767", _args(raster_size=32768)), ("batch beyond 65535", _args(batch_size=65536)),
    ]


def test_host_rejections_of_both_entry_points(lib):
    s = None
    for name, a in _cases():
        assert lib.nr_b200_interpolate(ctypes.byref(a), s) == INVALID, name
        assert lib.nr_b200_interpolate_backward(ctypes.byref(a), s) == INVALID, name
    assert lib.nr_b200_interpolate(None, s) == INVALID
    assert lib.nr_b200_interpolate_backward(None, s) == INVALID
    # forward only: no output image
    assert lib.nr_b200_interpolate(ctypes.byref(_args(out=None)), s) == INVALID
    # backward only: the vertex gradient in the other geometry form
    assert lib.nr_b200_interpolate_backward(ctypes.byref(_args(grad_vertices=_P)), s) == INVALID
    assert lib.nr_b200_interpolate_backward(ctypes.byref(_args(indexed=True, grad_faces=_P)), s) == INVALID


def _t(*shape, dtype=torch.float32):
    return torch.zeros(shape, dtype=dtype)


def test_python_argument_errors():
    import neural_renderer_b200 as nr
    faces = _t(2, 5, 3, 3)
    idx = _t(5, 3, dtype=torch.int32)
    verts = _t(2, 7, 3)
    with pytest.raises(TypeError):
        nr.rasterize_attributes(faces)  # no attributes
    with pytest.raises(TypeError):
        nr.rasterize_attributes(idx, vertices=verts, vertex_attributes=_t(7, 2), face_attributes=_t(5, 3, 2))
    with pytest.raises(TypeError):
        nr.rasterize_attributes(faces, face_attributes=_t(5, 3, 2, dtype=torch.int32))
    with pytest.raises(TypeError):
        nr.rasterize_attributes(faces, face_attributes=np.zeros((5, 3, 2), np.float32))
    with pytest.raises(ValueError):
        nr.rasterize_attributes(faces, vertex_attributes=_t(7, 2))  # per vertex needs indexed geometry
    for bad in (_t(4, 3, 2), _t(5, 2, 2), _t(5, 3, 0), _t(3, 5, 3, 2), _t(5, 3), _t(1, 1, 5, 3, 2)):
        with pytest.raises(ValueError):
            nr.rasterize_attributes(faces, face_attributes=bad)
    for bad in (_t(6, 2), _t(3, 7, 2), _t(7, 0), _t(7)):
        with pytest.raises(ValueError):
            nr.rasterize_attributes(idx, vertices=verts, vertex_attributes=bad)
    with pytest.raises(ValueError):
        nr.rasterize_attributes(_t(2, 5, 3), face_attributes=_t(5, 3, 2))  # the geometry's own shape
    # the Renderer says the same before it touches the camera
    with pytest.raises(TypeError):
        nr.Renderer().render_attributes(verts, idx[None].expand(2, -1, -1))
    # well-formed CPU tensors: there is no CPU implementation
    with pytest.raises(NotImplementedError):
        nr.rasterize_attributes(faces, face_attributes=_t(5, 3, 2))
    with pytest.raises(NotImplementedError):
        nr.rasterize_attributes(idx, vertices=verts, vertex_attributes=_t(1, 7, 4))


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_closed_form_interior_gradient_matches_float64_autograd(seed):
    """the header's d image / d vertices (oracles_attr.interior_grad64) against autograd of the same float64 oracle, on
    random faces and random (face, pixel) pairs -- the identity holds for any pixel, inside its face or not"""
    g = torch.Generator().manual_seed(seed)
    B, F, S, C = 2, 6, 12, 5
    xy = torch.rand((B, F, 3, 2), generator=g, dtype=torch.float64) * 1.6 - 0.8
    z = torch.rand((B, F, 3, 1), generator=g, dtype=torch.float64) * 2 + 1
    faces = torch.cat((xy, z), dim=-1).requires_grad_(True)
    fim = torch.randint(-1, F, (B, S, S), generator=g).to(torch.int32)
    attrs = torch.randn((B, F, 3, C), generator=g, dtype=torch.float64) + 5.0  # close together far from 0
    up = torch.randn((B, C, S, S), generator=g, dtype=torch.float64)
    (interp64(faces, fim, attrs, S, False) * up).sum().backward()
    want = interior_grad64(faces.detach(), fim, attrs, up, S)
    assert want.abs().max() > 0
    err = float((faces.grad - want).abs().max() / want.abs().max())
    assert err <= 1e-10, err
