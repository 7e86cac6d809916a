"""CPU: trilinear sampling through a mip pyramid (NR_TEX_MIPMAP) -- the flag against the header, the pyramid size, host
rejection of bad arguments before any device work, and the Python argument checks of texture_filter."""
import ctypes
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# fake, never dereferenced device address: every case below is decided on the host
_P = 0x10000


@pytest.fixture(scope="module")
def lib():
    from neural_renderer_b200 import build, _lib
    build.build_library()
    return _lib.load()


def mip_levels(H, W):
    """[(H_l, W_l)] of the pyramid: H_{l+1} = max(1, (H_l + 1) >> 1), until both sizes are 1."""
    out = [(H, W)]
    while out[-1] != (1, 1):
        h, w = out[-1]
        out.append((max(1, (h + 1) >> 1), max(1, (w + 1) >> 1)))
    return out


def test_flag_matches_the_header(lib):
    from neural_renderer_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "nr_b200.h")).read()
    m = re.search(r"#define NR_TEX_MIPMAP (0x[0-9a-fA-F]+)u", hdr)
    assert m and int(m.group(1), 16) == _lib.NR_TEX_MIPMAP == 0x80000
    assert lib.nr_b200_abi_version() == 4


@pytest.mark.parametrize("hw", [(1, 1), (1, 9), (12, 1), (17, 40), (1023, 1025), (1024, 1024)])
def test_mip_texels(lib, hw):
    import math
    levels = mip_levels(*hw)
    assert len(levels) == 1 + math.ceil(math.log2(max(hw)))
    assert lib.nr_b200_mip_texels(*hw) == sum(h * w for h, w in levels)


def test_mip_texels_of_empty_images_is_zero(lib):
    assert lib.nr_b200_mip_texels(0, 5) == 0 and lib.nr_b200_mip_texels(5, -1) == 0


def _fwd(flags, Ht=8, Wt=8):
    from neural_renderer_b200 import _lib
    a = _lib.ForwardArgs()
    a.struct_size = ctypes.sizeof(_lib.ForwardArgs)
    a.flags = flags
    a.batch_size, a.num_faces, a.raster_size, a.texture_size = 2, 4, 16, 0
    a.near_, a.far_, a.eps = 0.1, 100.0, 1e-4
    a.faces = a.textures = a.face_index_map = a.weight_map = a.depth_map = a.rgb_map = _P
    a.face_uvs = _P
    a.texture_height, a.texture_width = Ht, Wt
    return a


def _bwd(flags, Ht=8, Wt=8):
    from neural_renderer_b200 import _lib
    a = _lib.BackwardArgs()
    a.struct_size = ctypes.sizeof(_lib.BackwardArgs)
    a.flags = flags
    a.batch_size, a.num_faces, a.raster_size, a.texture_size = 2, 4, 16, 0
    a.eps = 1e-4
    a.faces = a.textures = a.face_index_map = a.weight_map = a.depth_map = a.rgb_map = _P
    a.grad_faces = a.grad_textures = _P
    a.face_uvs = _P
    a.texture_height, a.texture_width = Ht, Wt
    return a


def test_host_rejects_bad_mip_arguments(lib):
    from neural_renderer_b200 import _lib
    uv, rgb, mip, shared = _lib.NR_TEX_UV, _lib.NR_RETURN_RGB, _lib.NR_TEX_MIPMAP, _lib.NR_TEX_SHARED
    for call, make in ((lib.nr_b200_forward, _fwd), (lib.nr_b200_backward, _bwd)):
        def run(*args, **kw):
            return call(ctypes.byref(make(*args, **kw)), None)
        assert run(uv | rgb | mip) == -2                       # complete: reaches the workspace check
        assert run(uv | rgb | mip, Ht=1, Wt=1) == -2
        assert run(uv | rgb | mip | shared, Ht=1023, Wt=1025) == -2
        assert run(rgb | mip) == -1                            # NR_TEX_MIPMAP without NR_TEX_UV
        # two 17000^2 images fit 32-bit offsets, their pyramids (4/3 of them) do not
        assert run(uv | rgb, Ht=17000, Wt=17000) == -2
        assert run(uv | rgb | mip, Ht=17000, Wt=17000) == -4
        assert run(uv | rgb | mip | shared, Ht=17000, Wt=17000) == -2


def test_mip_build_and_collapse_reject_bad_arguments(lib):
    from neural_renderer_b200 import _lib
    build, collapse = lib.nr_b200_mip_build, lib.nr_b200_mip_collapse
    assert build(None, 1, 8, 8, _P, None) == -1
    assert build(_P, 1, 8, 8, None, None) == -1
    assert build(_P, 0, 8, 8, _P, None) == -1
    assert build(_P, 1, 0, 8, _P, None) == -1
    assert build(_P, 1, 8, -2, _P, None) == -1
    assert build(_P, 2, 30000, 20000, _P, None) == -4           # pyramid beyond 32-bit offsets
    assert collapse(None, 1, 8, 8, _P, 0, None) == -1
    assert collapse(_P, 1, 8, 8, None, 0, None) == -1
    assert collapse(_P, -1, 8, 8, _P, 0, None) == -1
    assert collapse(_P, 1, 8, 0, _P, _lib.NR_GRAD_ACCUMULATE, None) == -1
    assert collapse(_P, 1, 1 << 16, 1 << 16, _P, 0, None) == -4


def test_texture_filter_argument_checks():
    import neural_renderer_b200 as nr
    faces = torch.zeros(2, 6, 3, 3)
    img = torch.zeros(8, 8, 3)
    uvs = torch.zeros(6, 3, 2)
    with pytest.raises(ValueError):
        nr.rasterize(faces, img, 16, face_uvs=uvs, texture_filter="nearest")
    with pytest.raises(ValueError):
        nr.rasterize(faces, img, 16, face_uvs=uvs, texture_filter=None)
    with pytest.raises(ValueError):  # trilinear samples an image: it needs face_uvs
        nr.rasterize(faces, torch.zeros(2, 6, 4, 4, 4, 3), 16, texture_filter="trilinear")
    with pytest.raises(ValueError):
        nr.rasterize_rgbad(faces, img, 16, texture_filter="trilinear")
    for f in ("bilinear", "trilinear"):  # well-formed, but there is no CPU path
        with pytest.raises(NotImplementedError):
            nr.rasterize(faces, img, 16, face_uvs=uvs, texture_filter=f)
    import neural_renderer
    assert neural_renderer.Renderer().texture_filter == "bilinear"


def test_fp32_level_of_detail_restatement():
    """oracles.lod32 (the header's fp32 LOD, used where the float64 LOD alone moves a trilinear comparison) returns fp32
    values, agrees with oracles.lod64 to fp32 accuracy on well-conditioned faces and clamps as the header states"""
    from oracles import lod32, lod64
    g = torch.Generator().manual_seed(5)
    B, F, S, Ht, Wt = 2, 6, 12, 37, 29
    L = len(mip_levels(Ht, Wt))
    xy = (torch.rand((B, F, 3, 2), generator=g) * 1.6 - 0.8).double()
    z = (torch.rand((B, F, 3, 1), generator=g) * 2 + 1).double()
    faces = torch.cat((xy, z), dim=-1).float().double()
    fim = torch.randint(0, F, (B, S, S), generator=g).to(torch.int32)
    w = torch.rand((B, 3, S, S), generator=g) + 0.05
    wmap = w / w.sum(1, keepdim=True)
    fi, bidx = fim.long(), torch.arange(B)[:, None, None]
    zc = faces[..., 2][bidx, fi].float()  # [B,S,S,3]
    q = wmap.permute(0, 2, 3, 1) / zc
    dmap = 1.0 / ((q[..., 0] + q[..., 1]) + q[..., 2])
    spread = 10.0 ** torch.linspace(-3, 2, B * F).reshape(B, F, 1, 1).double()
    uvs = (0.5 + spread * (torch.rand((B, F, 3, 2), generator=g).double() - 0.5)).float().double()
    uvk = uvs[bidx, fi]
    a = lod64(faces, fim, wmap, dmap, uvk, S, Ht, Wt, L)
    b = lod32(faces, fim, wmap, dmap, uvk, S, Ht, Wt, L)
    assert torch.equal(b, b.float().double())
    assert ((b == 0) | (b == L - 1)).any() and ((b > 0) & (b < L - 1)).any()
    inner = (a > 0.01) & (a < L - 1.01)
    assert float((a - b).abs()[inner].max()) <= 1e-4 * L
