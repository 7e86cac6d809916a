"""CPU: the interior vertex gradient of the RGB image (NR_GRAD_INTERIOR) -- the flag against the header, the host-side
rejections of nr_b200_backward / nr_b200_backward_corner_light (decided before any launch), the Python argument error,
and the header's float64 closed form (oracles_interior.interior_grad64) against float64 autograd of the held-fixed
formulation (oracles_interior.rgb_held64) for every sampler and light."""
import ctypes
import os

import pytest
import torch

from oracles import pyramid64
from oracles_interior import Tex, interior_grad64, rgb_held64, select

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_P = 0x10000  # a fake, never dereferenced device address
OK_UP_TO_WORKSPACE, INVALID = -2, -1


@pytest.fixture(scope="module")
def lib():
    from neural_renderer_b200 import build, _lib
    build.build_library()
    return _lib.load()


def test_flag_matches_the_header_and_collides_with_no_other(tmp_path):
    import subprocess
    from neural_renderer_b200 import _lib
    src = tmp_path / "s.c"
    src.write_text('#include <stdio.h>\n#include "nr_b200.h"\nint main(void){printf("%u\\n", (unsigned)NR_GRAD_INTERIOR);'
                   'return 0;}\n')
    exe = tmp_path / "s"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    assert int(subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout) == _lib.NR_GRAD_INTERIOR
    assert _lib.NR_GRAD_INTERIOR == 0x400000
    others = [v for k, v in vars(_lib).items() if k.startswith("NR_") and k not in ("NR_OK", "NR_GRAD_INTERIOR")]
    assert all(v & _lib.NR_GRAD_INTERIOR == 0 for v in others)


def _bwd(flags, B=2, uv=False, textures=True):
    from neural_renderer_b200 import _lib
    a = _lib.BackwardArgs()
    a.struct_size = ctypes.sizeof(_lib.BackwardArgs)
    a.flags = flags | (_lib.NR_TEX_UV if uv else 0)
    a.batch_size, a.num_faces, a.raster_size, a.texture_size = B, 4, 16, 0 if uv else 4
    a.eps = 1e-4
    a.faces = a.face_index_map = a.weight_map = a.depth_map = a.rgb_map = a.grad_rgb = _P
    a.textures = _P if textures else None
    a.grad_faces = a.grad_textures = _P
    if uv:
        a.face_uvs = _P
        a.texture_height, a.texture_width = 8, 8
    return a


def test_host_rejections_before_any_launch(lib):
    from neural_renderer_b200 import _lib
    I, rgb, alpha, zb0 = _lib.NR_GRAD_INTERIOR, _lib.NR_RETURN_RGB, _lib.NR_RETURN_ALPHA, _lib.NR_TEX_Z_BATCH0
    part_t, part_f, acc = _lib.NR_BWD_PART_TEXTURES, _lib.NR_BWD_PART_FACES, _lib.NR_GRAD_ACCUMULATE

    def both(a):
        """nr_b200_backward, then the corner-light entry point; each return code with the launch count it left"""
        out = []
        for smooth in (False, True):
            rc = (lib.nr_b200_backward_corner_light(ctypes.byref(a), ctypes.c_void_p(_P), None, None) if smooth
                  else lib.nr_b200_backward(ctypes.byref(a), None))
            out.append((rc, lib.nr_b200_last_launch_count()))
        return out
    for uv in (False, True):
        for extra in (0, part_t, part_f, acc, alpha):
            assert both(_bwd(I | rgb | extra, uv=uv)) == [(OK_UP_TO_WORKSPACE, 0)] * 2, (uv, extra)
        assert both(_bwd(I | alpha, uv=uv))[0] == (INVALID, 0)  # no NR_RETURN_RGB
        assert both(_bwd(I | rgb, uv=uv, textures=False)) == [(INVALID, 0)] * 2  # the derivative reads the texture
        assert both(_bwd(rgb, uv=uv, textures=False)) == [(OK_UP_TO_WORKSPACE, 0)] * 2  # without the flag it does not
    # cubes sampled with the depths of item 0: refused at B = 2, the plain sampler at B = 1; images ignore the flag
    assert both(_bwd(I | rgb | zb0, B=2)) == [(INVALID, 0)] * 2
    assert both(_bwd(I | rgb | zb0, B=1)) == [(OK_UP_TO_WORKSPACE, 0)] * 2
    assert both(_bwd(I | rgb | zb0, B=2, uv=True)) == [(OK_UP_TO_WORKSPACE, 0)] * 2
    assert both(_bwd(rgb | zb0, B=2)) == [(OK_UP_TO_WORKSPACE, 0)] * 2


def test_python_argument_error():
    """per-face cubes, batch > 1, reference_exact: a ValueError that names the remedy, before any device work"""
    import neural_renderer_b200 as nr
    faces = torch.zeros(2, 4, 3, 3)
    tex = torch.zeros(2, 4, 2, 2, 2, 3)
    with pytest.raises(ValueError, match="reference_exact=False"):
        nr.rasterize(faces, tex, 16, False, reference_exact=True, interior_gradient=True)
    with pytest.raises(NotImplementedError):  # accepted, then the device check
        nr.rasterize(faces, tex, 16, False, reference_exact=False, interior_gradient=True)
    with pytest.raises(NotImplementedError):
        nr.rasterize(faces[:1], tex[:1], 16, False, reference_exact=True, interior_gradient=True)
    assert nr.Renderer().interior_gradient is False


def _problem(seed, kind, light, fill_back):
    g = torch.Generator().manual_seed(seed)
    B, F, S = 2, 6, 12
    xy = torch.rand((B, F, 3, 2), generator=g, dtype=torch.float64) * 1.6 - 0.8
    z = torch.rand((B, F, 3, 1), generator=g, dtype=torch.float64) * 2 + 1
    faces = torch.cat((xy, z), dim=-1)
    fim = torch.randint(-1, F, (B, S, S), generator=g).to(torch.int32)
    w = torch.rand((B, 3, S, S), generator=g, dtype=torch.float64) + 0.05
    wmap = w / w.sum(1, keepdim=True)  # float64: sum_k w_k = 1 to 1e-16, the point of the header's -w_m inv[3k]
    nf = F // 2 if fill_back else F
    if kind == "cube":
        ts = 4 if seed % 2 else 2
        tex = Tex("cube", torch.rand((1 if seed == 2 else B, nf, ts, ts, ts, 3), generator=g, dtype=torch.float64),
                  eps=1e-4, fill_back=fill_back)
    else:
        img = torch.rand((1, 13, 10, 3), generator=g, dtype=torch.float64)
        uvs = torch.rand((B, nf, 3, 2), generator=g, dtype=torch.float64) * 1.3 - 0.15  # some clamp-active pixels
        if seed == 2:
            uvs = uvs[:1] + 0.6  # shared, close together far from 0 in part
        levels = [img] if kind == "bilinear" else pyramid64(img)
        tex = Tex(kind, levels, uvs=uvs, fill_back=fill_back)
    lt = corner = None
    if light == "face":
        lt = torch.rand((B, F, 3), generator=g, dtype=torch.float64) + 0.5
    elif light == "corner":
        corner = torch.rand((B, F, 3, 3), generator=g, dtype=torch.float64) + 0.5
    up = torch.randn((B, 3, S, S), generator=g, dtype=torch.float64)
    return faces, fim, wmap, S, tex, lt, corner, up


@pytest.mark.parametrize("fill_back", [False, True])
@pytest.mark.parametrize("light", ["unlit", "face", "corner"])
@pytest.mark.parametrize("kind", ["cube", "bilinear", "trilinear"])
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_closed_form_matches_float64_autograd(seed, kind, light, fill_back):
    """the header's closed form against autograd of the held-fixed sample, on random faces, weights and (face, pixel)
    pairs -- the identity holds for any pixel, inside its face or not"""
    faces, fim, wmap, S, tex, lt, corner, up = _problem(seed, kind, light, fill_back)
    sel = select(faces, fim, wmap, S, tex)
    fr = faces.clone().requires_grad_(True)
    (rgb_held64(fr, fim, wmap, S, tex, sel, lt, corner) * up.permute(0, 2, 3, 1)).sum().backward()
    want = interior_grad64(faces, fim, wmap, S, tex, sel, up, lt, corner)
    assert want.abs().max() > 0
    err = float((fr.grad - want).abs().max() / want.abs().max())
    assert err <= 1e-10, err
