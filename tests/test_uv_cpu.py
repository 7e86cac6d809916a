"""CPU: the texture-image mode (NR_TEX_UV, ABI 4) -- struct layout against the header, host-side rejection of bad
arguments before any device work, Python argument checks, and the UV loader's atlas packing."""
import ctypes
import os

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")


@pytest.fixture(scope="module")
def lib():
    from neural_renderer_b200 import build, _lib
    build.build_library()
    return _lib.load()


def test_abi_version_4_and_flags_match_the_header(lib):
    import re
    from neural_renderer_b200 import _lib
    assert _lib.ABI_VERSION == 4 and lib.nr_b200_abi_version() == 4
    hdr = open(os.path.join(ROOT, "include", "nr_b200.h")).read()
    for name in ("NR_TEX_UV", "NR_UV_SHARED"):
        m = re.search(r"#define %s (0x[0-9a-fA-F]+)u" % name, hdr)
        assert m and int(m.group(1), 16) == getattr(_lib, name), name


def test_new_fields_match_the_header(tmp_path):
    import subprocess
    from neural_renderer_b200 import _lib
    fields = ("face_uvs", "texture_height", "texture_width")
    exprs = ["sizeof(nr_b200_forward_args)", "sizeof(nr_b200_backward_args)"]
    exprs += ["offsetof(nr_b200_%s_args, %s)" % (s, f) for s in ("forward", "backward") for f in fields]
    src = tmp_path / "s.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "nr_b200.h"\nint main(void){'
                   + "".join('printf("%%zu\\n", (size_t)%s);' % e for e in exprs) + "return 0;}\n")
    exe = tmp_path / "s"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    want = [ctypes.sizeof(_lib.ForwardArgs), ctypes.sizeof(_lib.BackwardArgs)]
    want += [getattr(S, f).offset for S in (_lib.ForwardArgs, _lib.BackwardArgs) for f in fields]
    assert got == want


# Fake, never dereferenced device addresses: every case below is decided on the host.  A complete argument set gets as
# far as the workspace check (NR_ERR_WORKSPACE, no workspace given); each broken one must stop earlier with -1.
_P = 0x10000


def _fwd_args(flags, F=4, uvs=True, Ht=8, Wt=8):
    from neural_renderer_b200 import _lib
    a = _lib.ForwardArgs()
    a.struct_size = ctypes.sizeof(_lib.ForwardArgs)
    a.flags = flags
    a.batch_size, a.num_faces, a.raster_size, a.texture_size = 2, F, 16, 0
    a.near_, a.far_, a.eps = 0.1, 100.0, 1e-4
    a.faces = a.textures = a.face_index_map = a.weight_map = a.depth_map = a.rgb_map = _P
    a.face_uvs = _P if uvs else None
    a.texture_height, a.texture_width = Ht, Wt
    return a


def _bwd_args(flags, F=4, uvs=True, Ht=8, Wt=8):
    from neural_renderer_b200 import _lib
    a = _lib.BackwardArgs()
    a.struct_size = ctypes.sizeof(_lib.BackwardArgs)
    a.flags = flags
    a.batch_size, a.num_faces, a.raster_size, a.texture_size = 2, F, 16, 0
    a.eps = 1e-4
    a.faces = a.textures = a.face_index_map = a.weight_map = a.depth_map = a.rgb_map = _P
    a.grad_faces = a.grad_textures = _P
    a.face_uvs = _P if uvs else None
    a.texture_height, a.texture_width = Ht, Wt
    return a


def test_host_rejects_bad_uv_arguments(lib):
    from neural_renderer_b200 import _lib
    uv, rgb, alpha, fb = _lib.NR_TEX_UV, _lib.NR_RETURN_RGB, _lib.NR_RETURN_ALPHA, _lib.NR_TEX_FILL_BACK
    for call, make in ((lib.nr_b200_forward, _fwd_args), (lib.nr_b200_backward, _bwd_args)):
        def run(*args, **kw):
            return call(ctypes.byref(make(*args, **kw)), None)
        assert run(uv | rgb) == -2                     # complete: reaches the workspace check
        assert run(uv | rgb | fb) == -2
        assert run(uv | rgb, Ht=1, Wt=1) == -2
        assert run(uv | alpha) == -1                   # UV mode without RGB
        assert run(uv | rgb, uvs=False) == -1          # NULL face_uvs
        assert run(uv | rgb, Ht=0) == -1               # empty image
        assert run(uv | rgb, Wt=-3) == -1
        assert run(uv | rgb | fb, F=5) == -1           # fill_back needs an even face count
        assert run(uv | rgb, Ht=1 << 15, Wt=1 << 15) == -4  # image offsets beyond 32 bits


def test_python_argument_checks():
    import neural_renderer_b200 as nr
    faces = torch.zeros(2, 6, 3, 3)
    img = torch.zeros(8, 8, 3)
    uvs = torch.zeros(6, 3, 2)
    with pytest.raises(ValueError):
        nr.rasterize(faces, img, 16, face_uvs=torch.zeros(5, 3, 2))         # wrong face count
    with pytest.raises(ValueError):
        nr.rasterize(faces, img, 16, face_uvs=torch.zeros(3, 6, 3, 2))      # batch neither 1 nor B
    with pytest.raises(ValueError):
        nr.rasterize(faces, img, 16, face_uvs=torch.zeros(6, 3, 3))
    with pytest.raises(ValueError):
        nr.rasterize(faces, torch.zeros(8, 8, 4), 16, face_uvs=uvs)         # not RGB
    with pytest.raises(ValueError):
        nr.rasterize(faces, torch.zeros(2, 6, 4, 4, 4, 3), 16, face_uvs=uvs)  # cubes given with face_uvs
    with pytest.raises(ValueError):
        nr.rasterize(faces, torch.zeros(0, 8, 3), 16, face_uvs=uvs)
    with pytest.raises(ValueError):  # fill_back: face_uvs holds F/2 faces
        nr.rasterize(faces, img, 16, face_uvs=uvs, textures_fill_back=True)
    with pytest.raises(TypeError):
        nr.rasterize(faces, img, 16, face_uvs=torch.zeros(6, 3, 2, dtype=torch.int32))
    with pytest.raises(TypeError):
        nr.rasterize(faces, None, 16, face_uvs=uvs)
    with pytest.raises(NotImplementedError):  # well-formed, but there is no CPU path
        nr.rasterize(faces, img, 16, face_uvs=uvs)
    with pytest.raises(ValueError):
        nr.load_obj(os.path.join(GOLDEN, "textured", "quads.obj"), load_texture=True, texture_mode="image")


def sample(img, u, v):
    """Bilinear sample with the kernels' addressing, in float32 (row 0 of `img` = top, v = 0 = bottom)."""
    img = np.asarray(img, np.float32)
    H, W = img.shape[:2]
    u = np.nan_to_num(np.clip(np.asarray(u, np.float32), 0, 1)).astype(np.float32)
    v = np.nan_to_num(np.clip(np.asarray(v, np.float32), 0, 1)).astype(np.float32)
    px, py = u * np.float32(W - 1), v * np.float32(H - 1)
    ix, iy = np.minimum(px.astype(np.int64), W - 1), np.minimum(py.astype(np.int64), H - 1)
    wx1, wy1 = px - ix.astype(np.float32), py - iy.astype(np.float32)
    wx0, wy0 = np.float32(1) - wx1, np.float32(1) - wy1
    x1, y1 = np.minimum(ix + 1, W - 1), np.minimum(iy + 1, H - 1)
    r0, r1 = H - 1 - iy, H - 1 - y1
    return ((wx0 * wy0)[:, None] * img[r0, ix] + (wx0 * wy1)[:, None] * img[r1, ix]
            + (wx1 * wy0)[:, None] * img[r0, x1] + (wx1 * wy1)[:, None] * img[r1, x1])


@pytest.mark.parametrize("model", [("display", "model.obj"), ("textured", "quads.obj")])
def test_atlas_sample_equals_material_image_sample(model):
    from neural_renderer_b200 import io
    path = os.path.join(GOLDEN, *model)
    uv0, names = io.parse_texture_faces(path)
    colors, files = io.load_mtl(os.path.splitext(path)[0] + ".mtl")
    _, faces, face_uvs, image = io.load_obj(path, load_texture=True, texture_mode="uv")
    assert face_uvs.shape == uv0.shape == (faces.shape[0], 3, 2) and face_uvs.dtype == np.float32
    assert image.ndim == 3 and image.shape[2] == 3 and image.dtype == np.float32
    if model[0] == "display":
        assert len(set(names)) == 7 and len(set(files.values())) == 2
    rng = np.random.default_rng(0)
    names = np.array(names)
    checked = 0
    for m in dict.fromkeys(names):
        sel = np.nonzero(names == m)[0]
        inside = sel[((uv0[sel] >= 0) & (uv0[sel] <= 1)).all(axis=(1, 2))]  # the remap is affine on [0,1]^2
        bary = rng.dirichlet(np.ones(3), size=(inside.shape[0], 8))         # 8 random points per face
        p0 = np.einsum("fnk,fkc->fnc", bary, uv0[inside].astype(np.float64)).reshape(-1, 2)
        p1 = np.einsum("fnk,fkc->fnc", bary, face_uvs[inside].astype(np.float64)).reshape(-1, 2).astype(np.float32)
        got = sample(image, p1[:, 0], p1[:, 1])
        if m in files:
            want = sample(io._read_image(os.path.join(os.path.dirname(path), files[m])), p0[:, 0], p0[:, 1])
        else:
            want = np.broadcast_to(colors.get(m, np.full(3, 0.5, np.float32)), got.shape)
        assert np.abs(got - want).max() <= 2e-4, m
        checked += inside.shape[0]
    assert checked >= 0.9 * faces.shape[0]


def test_single_image_model_keeps_image_and_uvs(tmp_path):
    from PIL import Image
    from neural_renderer_b200 import io
    img = (np.arange(5 * 7 * 3) % 251).astype(np.uint8).reshape(5, 7, 3)
    Image.fromarray(img, "RGB").save(tmp_path / "tex.png")
    (tmp_path / "m.mtl").write_text("newmtl a\nKd 1 0 0\nmap_Kd tex.png\nnewmtl b\nmap_Kd tex.png\n")
    (tmp_path / "m.obj").write_text("mtllib m.mtl\nv 0 0 0\nv 1 0 0\nv 1 1 0\nv 0 1 0\nvt 0 0\nvt 1 0\nvt 1 1\nvt 0.25 0.5\n"
                                    "usemtl a\nf 1/1 2/2 3/3\nusemtl b\nf 1/1 3/3 4/4\n")
    _, _, face_uvs, image = io.load_obj(str(tmp_path / "m.obj"), load_texture=True, texture_mode="uv")
    np.testing.assert_array_equal(image, img.astype(np.float32) / np.float32(255))
    np.testing.assert_array_equal(face_uvs, io.parse_texture_faces(str(tmp_path / "m.obj"))[0])


def test_sphere_uvs_follow_sphere_faces():
    from neural_renderer_b200 import synthetic
    v, f = synthetic.sphere_mesh(5000)
    uv = synthetic.sphere_uvs(5000)
    assert uv.shape == (5000, 3, 2) and uv.dtype == np.float32
    assert uv.min() >= 0 and uv.max() <= 1
    # v grows with the y coordinate (colatitude measured from +y); u with the longitude, 1 past the seam
    p = v[f]
    np.testing.assert_allclose(uv[..., 1], 1 - np.arccos(np.clip(p[..., 1], -1, 1)) / np.pi, atol=1e-6)
    lon = np.mod(np.arctan2(p[..., 2], p[..., 0]), 2 * np.pi) / (2 * np.pi)
    d = np.abs(uv[..., 0] - lon)
    assert (np.minimum(d, 1 - d) < 1e-5).all()
