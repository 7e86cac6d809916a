"""CPU: the soft interpolation of fragments -- nr_b200_frag_interp_args against the header, the new symbols, the host
rejections of both entry points (all decided before any launch), the Python argument errors of
interpolate_soft_fragments (raised before the device check), and the spills of the new kernels."""
import ctypes
import os
import re
import subprocess

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# Fake, never dereferenced device addresses: a complete argument set is accepted by the checks, so the tests below only
# ever pass broken sets to the library (a complete one would launch).
_P = 0x10000
INVALID = -1


@pytest.fixture(scope="module")
def lib():
    from neural_renderer_b200 import build, _lib
    build.build_library()
    return _lib.load()


def test_frag_interp_struct_matches_the_header(tmp_path):
    from neural_renderer_b200 import _lib
    fields = [f[0] for f in _lib.FragInterpArgs._fields_]
    exprs = ["sizeof(nr_b200_frag_interp_args)"] + ["offsetof(nr_b200_frag_interp_args, %s)" % f for f in fields]
    src = tmp_path / "s.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "nr_b200.h"\nint main(void){'
                   + "".join('printf("%%zu\\n", (size_t)(%s));' % e for e in exprs) + "return 0;}\n")
    exe = tmp_path / "s"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    vals = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert vals[0] == ctypes.sizeof(_lib.FragInterpArgs) == 104
    assert vals[1:] == [getattr(_lib.FragInterpArgs, f).offset for f in fields]


def test_new_symbols_are_exported(lib):
    from neural_renderer_b200 import _lib
    out = subprocess.run(["nm", "-D", "--defined-only", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    for n in ("nr_b200_interpolate_fragments", "nr_b200_interpolate_fragments_backward"):
        assert n in _lib.EXPORTED_SYMBOLS
        assert (" T " + n) in out, n


def _args(backward=False, **kw):
    from neural_renderer_b200 import _lib
    a = _lib.FragInterpArgs(struct_size=ctypes.sizeof(_lib.FragInterpArgs), batch_size=2, height=8, width=9,
                            faces_per_pixel=8, channels=3, num_faces=50, num_vertices=40)
    a.pix_to_face = a.bary = a.attributes = a.out = _P
    if backward:
        a.grad_out = a.grad_attributes = a.grad_bary = _P
    for k, v in kw.items():
        setattr(a, k, v)
    return a


@pytest.mark.parametrize("backward", [False, True])
def test_host_rejections(lib, backward):
    from neural_renderer_b200 import _lib
    fn = lib.nr_b200_interpolate_fragments_backward if backward else lib.nr_b200_interpolate_fragments
    pv = _lib.NR_ATTR_PER_VERTEX
    bad = [dict(struct_size=0), dict(struct_size=ctypes.sizeof(_lib.FragInterpArgs) + 8), dict(struct_size=4),
           dict(batch_size=0), dict(height=0), dict(width=-1), dict(channels=0), dict(num_faces=0),
           dict(faces_per_pixel=0), dict(faces_per_pixel=-1), dict(faces_per_pixel=33),
           dict(flags=pv, face_indices=_P, num_vertices=0),                 # Nv < 1 with per-vertex attributes
           # unknown flags, and per-vertex attributes without indices
           dict(flags=1), dict(flags=_lib.NR_FACES_INDEXED), dict(flags=1 << 31), dict(flags=pv),
           # NULL pointers each call needs
           dict(pix_to_face=None), dict(bary=None), dict(attributes=None),
           # element alignment: 8 bytes for pix_to_face, 4 for the rest
           dict(pix_to_face=_P + 4), dict(bary=_P + 2), dict(attributes=_P + 1), dict(out=_P + 2),
           dict(flags=pv, face_indices=_P + 2), dict(grad_out=_P + 3), dict(grad_attributes=_P + 1),
           dict(grad_bary=_P + 2),
           # sizes past the index width
           dict(batch_size=1 << 30, height=1 << 30, width=1 << 30),          # B H W K C past 64-bit offsets
           dict(batch_size=1 << 20, height=1 << 20, width=1 << 10, channels=1),  # B H W K / 256 CTAs past 2^31 - 1
           dict(channels=(1 << 20) + 1)]                                     # C past 2^20
    if not backward:
        bad += [dict(out=None), dict(flags=_lib.NR_GRAD_ACCUMULATE)]         # accumulation is a backward flag
    if backward:
        bad += [dict(grad_attributes=None, grad_bary=None)]
    for kw in bad:
        assert fn(ctypes.byref(_args(backward, **kw)), None) == INVALID, kw
        assert lib.nr_b200_last_launch_count() == 0
    assert fn(None, None) == INVALID
    assert lib.nr_b200_last_launch_count() == 0


def _frag(B=2, H=4, W=5, K=3):
    import neural_renderer_b200 as nr
    p2f = torch.full((B, H, W, K), -1, dtype=torch.int64)
    return nr.Fragments(p2f, torch.zeros(B, H, W, K), torch.zeros(B, H, W, K, 3), torch.zeros(B, H, W, K))


def test_python_argument_errors_come_before_the_device_check():
    import neural_renderer_b200 as nr
    B, H, W, K, F, Nv, C = 2, 4, 5, 3, 7, 6, 2
    frag = _frag(B, H, W, K)
    fa = torch.zeros(F, 3, C)
    va = torch.zeros(Nv, C)
    faces = torch.zeros(F, 3, dtype=torch.int64)
    # valid arguments on the CPU: no CPU path
    for call in (lambda: nr.interpolate_soft_fragments(frag, fa),
                 lambda: nr.interpolate_soft_fragments(frag, fa[None].expand(B, -1, -1, -1)),
                 lambda: nr.interpolate_soft_fragments(frag, vertex_attributes=va, faces=faces),
                 lambda: nr.interpolate_soft_fragments(frag, vertex_attributes=va[None], faces=faces[None].expand(B, -1, -1))):
        with pytest.raises(NotImplementedError):
            call()
    type_errors = [((frag[:2],), {}),                                        # not a Fragments
                   ((frag._replace(pix_to_face=frag.pix_to_face.tolist()), fa), {}),
                   ((frag._replace(bary_coords=None), fa), {}),
                   ((frag,), {}),                                            # neither attribute form
                   ((frag, fa), dict(vertex_attributes=va, faces=faces)),    # both
                   ((frag, fa.long()), {}), ((frag, fa.tolist()), {}),
                   ((frag,), dict(vertex_attributes=va.int(), faces=faces)),
                   ((frag,), dict(vertex_attributes=va, faces=faces.float())),
                   ((frag,), dict(vertex_attributes=va, faces=faces.tolist())),
                   ((frag, fa), dict(faces=faces))]                          # faces with per-corner attributes
    for args, kw in type_errors:
        with pytest.raises(TypeError):
            nr.interpolate_soft_fragments(*args, **kw)
    value_errors = [((frag._replace(pix_to_face=frag.pix_to_face.int()), fa), {}),     # dtype of pix_to_face
                    ((frag._replace(pix_to_face=frag.pix_to_face[0]), fa), {}),       # rank
                    ((frag._replace(bary_coords=frag.bary_coords[..., :2]), fa), {}),
                    ((frag._replace(bary_coords=frag.bary_coords.long()), fa), {}),
                    ((_frag(K=33), fa), {}),                                           # K past the cap
                    ((_frag(H=0), fa), {}),
                    ((frag, fa[:, :2]), {}), ((frag, fa[0]), {}), ((frag, fa[None].expand(3, -1, -1, -1)), {}),
                    ((frag, torch.zeros(F, 3, 0)), {}), ((frag, torch.zeros(0, 3, C)), {}),
                    ((frag,), dict(vertex_attributes=va)),                              # no faces
                    ((frag,), dict(vertex_attributes=va[0], faces=faces)),
                    ((frag,), dict(vertex_attributes=va[None].expand(3, -1, -1), faces=faces)),
                    ((frag,), dict(vertex_attributes=torch.zeros(Nv, 0), faces=faces)),
                    ((frag,), dict(vertex_attributes=va, faces=faces[:, :2])),
                    ((frag,), dict(vertex_attributes=va, faces=faces[0])),
                    ((frag,), dict(vertex_attributes=va, faces=faces[None].expand(3, -1, -1))),
                    ((frag,), dict(vertex_attributes=va, faces=faces[:0]))]
    for args, kw in value_errors:
        with pytest.raises(ValueError):
            nr.interpolate_soft_fragments(*args, **kw)
    if torch.cuda.is_available():                                            # mixed devices
        with pytest.raises(ValueError):
            nr.interpolate_soft_fragments(frag, fa.cuda())


def test_exported_from_both_package_names():
    import neural_renderer
    import neural_renderer_b200
    assert neural_renderer.interpolate_soft_fragments is neural_renderer_b200.interpolate_soft_fragments


def test_new_kernels_compile_for_sm90a_without_spills(tmp_path):
    from neural_renderer_b200 import build
    nvcc = os.environ.get("NVCC", "nvcc")
    for defines in ([], ["-DNR_B200_TUNING", "-DNR_SOFT_INTERP_GLOBAL_ATOMICS"]):  # the kept and the measured variant
        cmd = [nvcc] + build.NVCC_FLAGS + defines + ["-Xptxas", "-v", "-c", os.path.join(build.CSRC, "nr_soft_interp.cu"),
                                                     "-o", str(tmp_path / "nr_soft_interp.o")]
        log = subprocess.run(cmd, capture_output=True, text=True, check=True).stderr
        entries = re.split(r"Compiling entry function '", log)[1:]
        names = [e.split("'")[0] for e in entries]
        # the forward per corner / per vertex, scalar / 16-byte; the backward per corner / per vertex
        assert len(entries) == 6, names
        assert sum("k_soft_interp_fwd" in n for n in names) == 4 and sum("k_soft_interp_bwd" in n for n in names) == 2
        for e in entries:
            m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", e)
            assert m and m.groups() == ("0", "0", "0"), e[:400]
            assert "cumulative stack" not in e.split("Compile time")[0], e[:400]
        assert "sm_90a" in log
