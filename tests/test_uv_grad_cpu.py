"""CPU: the face_uvs gradient of the texture-image samplers (nr_b200_backward_args.grad_face_uvs) -- the appended field
against the header, the two accepted struct sizes, and the host-side rejections, all decided before any device work."""
import ctypes
import os

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# Fake, never dereferenced device addresses (as test_uv_cpu.py): a complete argument set gets as far as the workspace
# check (NR_ERR_WORKSPACE, no workspace given); each broken one must stop earlier.
_P = 0x10000
OK_UP_TO_WORKSPACE, INVALID, UNSUPPORTED = -2, -1, -4


@pytest.fixture(scope="module")
def lib():
    from neural_renderer_b200 import build, _lib
    build.build_library()
    return _lib.load()


def test_grad_face_uvs_field_matches_the_header(tmp_path):
    import subprocess
    from neural_renderer_b200 import _lib
    exprs = ["sizeof(nr_b200_backward_args)", "offsetof(nr_b200_backward_args, grad_face_uvs)",
             "offsetof(nr_b200_backward_args, texture_width) + sizeof(int32_t)"]
    src = tmp_path / "s.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "nr_b200.h"\nint main(void){'
                   + "".join('printf("%%zu\\n", (size_t)(%s));' % e for e in exprs) + "return 0;}\n")
    exe = tmp_path / "s"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    size, off, end_of_abi4 = (int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split())
    assert size == ctypes.sizeof(_lib.BackwardArgs)
    assert off == _lib.BackwardArgs.grad_face_uvs.offset
    assert off == end_of_abi4 and size == off + 8  # appended right after the ABI-4 fields, nothing else moved


def _bwd(flags, F=4, grad_uvs=True, textures=True, struct_size=None):
    from neural_renderer_b200 import _lib
    a = _lib.BackwardArgs()
    a.struct_size = ctypes.sizeof(_lib.BackwardArgs) if struct_size is None else struct_size
    a.flags = flags
    a.batch_size, a.num_faces, a.raster_size, a.texture_size = 2, F, 16, 0
    a.eps = 1e-4
    a.faces = a.face_index_map = a.weight_map = a.depth_map = a.rgb_map = _P
    a.textures = _P if textures else None
    a.grad_faces = a.grad_textures = _P
    a.face_uvs = _P
    a.grad_face_uvs = _P if grad_uvs else None
    a.texture_height, a.texture_width = 8, 8
    return a


def test_both_struct_layouts_are_accepted_and_no_other(lib):
    from neural_renderer_b200 import _lib
    uv, rgb = _lib.NR_TEX_UV, _lib.NR_RETURN_RGB
    full, abi4 = ctypes.sizeof(_lib.BackwardArgs), _lib.BackwardArgs.grad_face_uvs.offset

    def run(size, **kw):
        return lib.nr_b200_backward(ctypes.byref(_bwd(uv | rgb, struct_size=size, **kw)), None)
    assert run(full) == OK_UP_TO_WORKSPACE
    assert run(abi4, grad_uvs=False) == OK_UP_TO_WORKSPACE
    for size in (0, 4, abi4 - 8, abi4 - 1, abi4 + 1, abi4 + 4, full - 1, full + 1, full + 8):
        assert run(size) == INVALID, size


def test_short_struct_does_not_read_grad_face_uvs(lib):
    """with the ABI-4 size the host must not look at bytes past the caller's struct: a grad_face_uvs that WOULD be
    rejected (no NR_TEX_UV; textures NULL) is ignored, and the call is decided as one without it"""
    from neural_renderer_b200 import _lib
    abi4 = _lib.BackwardArgs.grad_face_uvs.offset
    rgb = _lib.NR_RETURN_RGB
    cubes = _bwd(rgb, struct_size=abi4)
    cubes.texture_size = 4
    assert lib.nr_b200_backward(ctypes.byref(cubes), None) == OK_UP_TO_WORKSPACE
    cubes.struct_size = ctypes.sizeof(_lib.BackwardArgs)
    assert lib.nr_b200_backward(ctypes.byref(cubes), None) == INVALID


def test_host_rejects_bad_uv_gradient_requests(lib):
    from neural_renderer_b200 import _lib
    uv, rgb, alpha, depth = _lib.NR_TEX_UV, _lib.NR_RETURN_RGB, _lib.NR_RETURN_ALPHA, _lib.NR_RETURN_DEPTH
    mip, fb, shared = _lib.NR_TEX_MIPMAP, _lib.NR_TEX_FILL_BACK, _lib.NR_UV_SHARED
    acc, part_t, part_f = _lib.NR_GRAD_ACCUMULATE, _lib.NR_BWD_PART_TEXTURES, _lib.NR_BWD_PART_FACES

    def run(flags, **kw):
        a = _bwd(flags, **kw)
        if not flags & uv:
            a.texture_size = 4  # a complete cube-mode call apart from grad_face_uvs
        return lib.nr_b200_backward(ctypes.byref(a), None)
    for ok in (uv | rgb, uv | rgb | mip, uv | rgb | fb | shared, uv | rgb | alpha | depth | acc, uv | rgb | part_t,
               uv | rgb | part_f):
        assert run(ok) == OK_UP_TO_WORKSPACE, hex(ok)
    assert run(rgb) == INVALID                      # cube textures have no UVs
    assert run(rgb, grad_uvs=False) == OK_UP_TO_WORKSPACE
    assert run(uv | alpha) == INVALID               # no RGB (UV mode itself needs it too)
    assert run(uv | rgb, textures=False) == INVALID  # the derivative reads the image
    assert run(uv | rgb | mip, textures=False) == INVALID
    assert run(uv | rgb, textures=False, grad_uvs=False) == OK_UP_TO_WORKSPACE  # the image gradient alone does not read it
    # the UV gradient has the layout of face_uvs: beyond 32-bit offsets the call is refused before any launch (the
    # face list of the edge scan is the first limit reached at these sizes)
    assert run(uv | rgb, F=1 << 28) == UNSUPPORTED


def test_python_binding_mirrors_the_field():
    from neural_renderer_b200 import _lib
    names = [f[0] for f in _lib.BackwardArgs._fields_]
    assert names[-1] == "grad_face_uvs" and names[-4:-1] == ["face_uvs", "texture_height", "texture_width"]
