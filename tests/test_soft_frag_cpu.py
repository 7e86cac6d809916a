"""CPU: soft fragments -- nr_b200_soft_frag_args against the header, the new symbols, the host rejections of both entry
points (all decided before any launch), the Python, Renderer and interpolate_face_attributes argument errors (raised
before the device check), the float64 oracle's self-checks (tests/oracles_soft_frag.py), and the spills of the new
kernels."""
import ctypes
import math
import os
import re
import subprocess

import pytest
import torch

import oracles_soft as osoft
import oracles_soft_attr as oattr
import oracles_soft_frag as ofrag

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# Fake, never dereferenced device addresses: a complete argument set gets as far as the workspace check
# (NR_ERR_WORKSPACE, no workspace given); each broken one must stop earlier.
_P = 0x10000
WORKSPACE, INVALID = -2, -1


@pytest.fixture(scope="module")
def lib():
    from neural_renderer_b200 import build, _lib
    build.build_library()
    return _lib.load()


def test_soft_frag_struct_matches_the_header(tmp_path):
    from neural_renderer_b200 import _lib
    fields = [f[0] for f in _lib.SoftFragArgs._fields_]
    exprs = ["sizeof(nr_b200_soft_frag_args)"] + ["offsetof(nr_b200_soft_frag_args, %s)" % f for f in fields]
    src = tmp_path / "s.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "nr_b200.h"\nint main(void){'
                   + "".join('printf("%%zu\\n", (size_t)(%s));' % e for e in exprs) + "return 0;}\n")
    exe = tmp_path / "s"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    vals = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert vals[0] == ctypes.sizeof(_lib.SoftFragArgs) == 64
    assert vals[1:] == [getattr(_lib.SoftFragArgs, f).offset for f in fields]


def test_new_symbols_are_exported(lib):
    from neural_renderer_b200 import _lib
    out = subprocess.run(["nm", "-D", "--defined-only", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    for n in ("nr_b200_soft_fragments", "nr_b200_soft_fragments_backward"):
        assert n in _lib.EXPORTED_SYMBOLS
        assert (" T " + n) in out, n


def _args(indexed=False, backward=False, **kw):
    from neural_renderer_b200 import _lib
    a = _lib.SoftRgbArgs()
    a.struct_size = ctypes.sizeof(_lib.SoftRgbArgs)
    a.flags = _lib.NR_FACES_INDEXED if indexed else 0
    a.batch_size, a.num_faces, a.image_size, a.num_vertices, a.texture_size = 2, 4, 16, 6 if indexed else 0, 0
    # gamma, texture_size and eps: ignored
    a.sigma, a.gamma, a.near_, a.far_, a.eps = 1e-4, float("nan"), 0.1, 100.0, float("nan")
    if indexed:
        a.vertices = a.face_indices = _P
    else:
        a.faces = _P
    if backward:
        if indexed:
            a.grad_vertices = _P
        else:
            a.grad_faces = _P
    for k, v in kw.items():
        setattr(a, k, v)
    return a


def _frag(backward=False, **kw):
    from neural_renderer_b200 import _lib
    t = _lib.SoftFragArgs(struct_size=ctypes.sizeof(_lib.SoftFragArgs), faces_per_pixel=8, pix_to_face=_P)
    if backward:
        t.grad_zbuf = t.grad_bary = t.grad_dists = _P
    else:
        t.zbuf = t.bary = t.dists = _P
    for k, v in kw.items():
        setattr(t, k, v)
    return t


def _call(lib, a, t, backward):
    fn = lib.nr_b200_soft_fragments_backward if backward else lib.nr_b200_soft_fragments
    return fn(ctypes.byref(a) if a is not None else None, ctypes.byref(t) if t is not None else None, None)


@pytest.mark.parametrize("backward", [False, True])
@pytest.mark.parametrize("indexed", [False, True])
def test_host_rejections(lib, indexed, backward):
    from neural_renderer_b200 import _lib
    ok = _args(indexed, backward)
    assert _call(lib, ok, _frag(backward), backward) == WORKSPACE
    assert lib.nr_b200_last_launch_count() == 0
    fl = ok.flags
    allowed = [(dict(flags=fl | _lib.NR_GRAD_ACCUMULATE), {}), (dict(texture_size=1000), {}), (dict(eps=0.5), {}),
               (dict(gamma=0.0), {}), (dict(gamma=float("inf")), {}), ({}, dict(faces_per_pixel=1)),
               ({}, dict(faces_per_pixel=32)), ({}, dict(faces_per_pixel=3))]
    if backward:
        allowed += [({}, dict(grad_zbuf=None)), ({}, dict(grad_bary=None)), ({}, dict(grad_dists=None)),
                    ({}, dict(grad_zbuf=None, grad_bary=None, grad_dists=None))]
        allowed += [({}, dict(zbuf=None, bary=None, dists=None))]                 # not read by the backward
    else:
        allowed += [({}, dict(grad_zbuf=_P, grad_bary=_P, grad_dists=_P))]        # not read by the forward
    if indexed:
        allowed += [(dict(flags=fl | _lib.NR_INDICES_SHARED), {})]
    for kw, tkw in allowed:
        assert _call(lib, _args(indexed, backward, **kw), _frag(backward, **tkw), backward) == WORKSPACE, (kw, tkw)
        assert lib.nr_b200_last_launch_count() == 0
    bad = [(dict(struct_size=4), {}), (dict(struct_size=ctypes.sizeof(_lib.SoftRgbArgs) + 8), {}),
           ({}, dict(struct_size=0)), ({}, dict(struct_size=ctypes.sizeof(_lib.SoftFragArgs) + 8)),
           ({}, dict(faces_per_pixel=0)), ({}, dict(faces_per_pixel=-1)), ({}, dict(faces_per_pixel=33)),
           ({}, dict(pix_to_face=None)),
           (dict(batch_size=0), {}), (dict(num_faces=0), {}), (dict(image_size=0), {}), (dict(sigma=0.0), {}),
           (dict(sigma=float("nan")), {}), (dict(sigma=float("inf")), {}), (dict(near_=2.0, far_=1.0), {}),
           (dict(near_=1.0, far_=1.0), {}), (dict(batch_size=65536), {}), (dict(image_size=32768), {}),
           # the soft RGB's colour, alpha and softmax buffers are refused
           (dict(textures=_P), {}), (dict(face_light=_P), {}), (dict(rgb=_P), {}), (dict(alpha=_P), {}),
           (dict(state=_P), {}), (dict(grad_rgb=_P), {}), (dict(grad_alpha=_P), {}), (dict(grad_textures=_P), {}),
           (dict(grad_face_light=_P), {})]
    if not backward:
        bad += [({}, dict(zbuf=None)), ({}, dict(bary=None)), ({}, dict(dists=None))]
    for f in (_lib.NR_TEX_SHARED, _lib.NR_TEX_UV, _lib.NR_UV_SHARED, _lib.NR_TEX_MIPMAP, _lib.NR_TEX_FILL_BACK,
              _lib.NR_GRAD_INTERIOR, _lib.NR_RETURN_RGB, _lib.NR_ANTI_ALIASING, _lib.NR_ATTR_PER_VERTEX,
              _lib.NR_ATTR_SHARED, 1 << 31):
        bad.append((dict(flags=fl | f), {}))
    if indexed:
        bad += [(dict(vertices=None), {}), (dict(face_indices=None), {}), (dict(num_vertices=0), {})]
    else:
        bad += [(dict(faces=None), {})]
    if backward:
        bad += [(dict(grad_faces=_P), {})] if indexed else [(dict(grad_vertices=_P), {})]
        bad += [(dict(grad_vertices=None), {})] if indexed else [(dict(grad_faces=None), {})]
    for kw, tkw in bad:
        assert _call(lib, _args(indexed, backward, **kw), _frag(backward, **tkw), backward) == INVALID, (kw, tkw)
        assert lib.nr_b200_last_launch_count() == 0
    assert _call(lib, None, _frag(backward), backward) == INVALID
    assert _call(lib, ok, None, backward) == INVALID
    assert lib.nr_b200_last_launch_count() == 0


def test_python_argument_errors_come_before_the_device_check():
    import neural_renderer_b200 as nr
    from neural_renderer_b200 import functional as F
    faces = torch.zeros(1, 2, 3, 3)
    with pytest.raises(NotImplementedError):  # valid arguments on the CPU: no CPU path
        nr.rasterize_soft_fragments(faces, 16)
    verts, idx = torch.zeros(1, 5, 3), torch.zeros(2, 3, dtype=torch.int64)
    with pytest.raises(NotImplementedError):
        nr.rasterize_soft_fragments(idx, 16, faces_per_pixel=32, vertices=verts)
    for kw in (dict(sigma=0.0), dict(sigma=float("nan")), dict(sigma=-1.0), dict(near=2.0, far=1.0),
               dict(near=1.0, far=1.0), dict(image_size=0), dict(faces_per_pixel=0), dict(faces_per_pixel=33)):
        with pytest.raises(ValueError):
            nr.rasterize_soft_fragments(faces, **{"image_size": 16, **kw})
    with pytest.raises(ValueError):
        nr.rasterize_soft_fragments(torch.zeros(1, 2, 3, 2), 16)
    for kw in (dict(sigma="x"), dict(faces_per_pixel=2.0), dict(faces_per_pixel=True), dict(faces_per_pixel="8")):
        with pytest.raises(TypeError):
            nr.rasterize_soft_fragments(faces, 16, **kw)
    with pytest.raises(TypeError):
        nr.rasterize_soft_fragments(faces.int(), 16)
    r = nr.Renderer()
    v, f = torch.zeros(1, 3, 3), torch.zeros(1, 1, 3, dtype=torch.int32)
    with pytest.raises(ValueError):
        r.render_soft_fragments(v, f, sigma=-1.0)
    with pytest.raises(ValueError):
        r.render_soft_fragments(v, f, faces_per_pixel=40)
    with pytest.raises(NotImplementedError):
        r.render_soft_fragments(v, f)
    # interpolate_face_attributes: shapes
    p2f = torch.full((1, 2, 2, 3), -1, dtype=torch.int64)
    bary = torch.zeros(1, 2, 2, 3, 3)
    with pytest.raises(ValueError):
        F.interpolate_face_attributes(p2f, bary[..., :2], torch.zeros(4, 3, 2))
    with pytest.raises(ValueError):
        F.interpolate_face_attributes(p2f.float(), bary, torch.zeros(4, 3, 2))
    with pytest.raises(ValueError):
        F.interpolate_face_attributes(p2f, bary, torch.zeros(4, 2, 2))
    with pytest.raises(ValueError):
        F.interpolate_face_attributes(p2f, bary, torch.zeros(2, 4, 3, 2))
    with pytest.raises(TypeError):
        F.interpolate_face_attributes(p2f, bary, [[0.0]])


def test_interpolate_face_attributes_against_a_loop():
    from neural_renderer_b200 import functional as F
    g = torch.Generator().manual_seed(1)
    B, S, K, Fn, C = 2, 3, 4, 5, 2
    p2f = torch.randint(-1, Fn, (B, S, S, K), generator=g)
    bary = torch.rand(B, S, S, K, 3, generator=g, dtype=torch.float64)
    for shared in (True, False):
        fa = torch.rand(*((Fn, 3, C) if shared else (B, Fn, 3, C)), generator=g, dtype=torch.float64)
        out = F.interpolate_face_attributes(p2f, bary, fa)
        want = torch.zeros(B, S, S, K, C, dtype=torch.float64)
        for b in range(B):
            for i in range(S):
                for j in range(S):
                    for k in range(K):
                        f = int(p2f[b, i, j, k])
                        if f >= 0:
                            a = fa[f] if shared else fa[b, f]
                            want[b, i, j, k] = (bary[b, i, j, k, :, None] * a).sum(0)
        torch.testing.assert_close(out, want, rtol=1e-14, atol=1e-14)
    # NaN attributes of face 0 stay out of empty slots
    fa = torch.full((Fn, 3, C), float("nan"), dtype=torch.float64)
    out = F.interpolate_face_attributes(torch.full((1, 1, 1, 2), -1), torch.ones(1, 1, 1, 2, 3, dtype=torch.float64), fa)
    assert torch.equal(out, torch.zeros_like(out))


# ------------------------------------------------------------------------------------------------ oracle self-checks
def _faces(seed, F=6, B=1):
    g = torch.Generator().manual_seed(seed)
    faces = torch.rand(B, F, 3, 3, generator=g) * 1.6 - 0.8
    faces[..., 2] = 1.0 + 3.0 * torch.rand(B, F, 3, generator=g)
    return faces


def test_one_triangle_signed_distance_in_closed_form():
    # a right triangle (0,0) (0.5,0) (0,0.5): inside, the distance to the nearest side; below it, to the base or a corner
    S = 16
    faces = torch.tensor([[[[0.0, 0.0, 2.0], [0.5, 0.0, 2.0], [0.0, 0.5, 2.0]]]])
    xs = (2 * torch.arange(S, dtype=torch.float64) + 1 - S) / S
    p2f = torch.zeros(1, S, S, 1, dtype=torch.int64)
    zb, by, ds = ofrag.evaluate(faces, p2f, S)
    for r in range(S):
        for c in range(S):
            x, y = float(xs[c]), float(xs[S - 1 - r])
            inside = x > 0 and y > 0 and x + y < 0.5
            if inside:
                want = min(x, y, (0.5 - x - y) / math.sqrt(2)) ** 2
            else:
                # the nearest point of the closed triangle, by projection onto each side
                best = math.inf
                for (ax, ay), (bx, by_) in (((0, 0), (0.5, 0)), ((0.5, 0), (0, 0.5)), ((0, 0.5), (0, 0))):
                    ex, ey = bx - ax, by_ - ay
                    t = min(max(((x - ax) * ex + (y - ay) * ey) / (ex * ex + ey * ey), 0.0), 1.0)
                    best = min(best, (x - ax - t * ex) ** 2 + (y - ay - t * ey) ** 2)
                want = -best
            assert abs(float(ds[0, r, c, 0]) - want) < 1e-12, (r, c)
            assert abs(float(zb[0, r, c, 0]) - 2.0) < 1e-12


def test_bary_sums_to_one_and_interpolates_zbuf():
    B, F, S, K, sigma = 2, 8, 20, 6, 1e-3
    faces = _faces(2, F, B)
    b, pix, f, zp, certain, band = ofrag.candidates(faces, S, sigma)
    assert b.numel() > 200
    p2f = torch.full((B, S * S, K), -1, dtype=torch.int64)
    order = ofrag.sort_key(b, pix, f, zp)
    seen = {}
    for i in order.tolist():
        key = (int(b[i]), int(pix[i]))
        k = seen.get(key, 0)
        if k < K:
            p2f[key[0], key[1], k] = f[i]
            seen[key] = k + 1
    p2f = p2f.reshape(B, S, S, K)
    zb, by, ds = ofrag.evaluate(faces, p2f, S)
    sel = p2f >= 0
    torch.testing.assert_close(by.sum(-1)[sel], torch.ones_like(zb[sel]), rtol=0, atol=1e-12)
    z = torch.gather(faces.to(torch.float64)[..., 2], 1, p2f.clamp_min(0).reshape(B, -1, 1).expand(-1, -1, 3))
    torch.testing.assert_close((by.reshape(B, -1, 3) * z).sum(-1).reshape(B, S, S, K)[sel], zb[sel], rtol=1e-12, atol=0)
    assert torch.all(zb[~sel] == -1) and torch.all(ds[~sel] == -1) and torch.all(by[~sel] == -1)
    # the selection is ordered by zp per pixel, and A_j of the soft attributes is sum_k l'_k a_k
    assert torch.all((zb[..., 1:] >= zb[..., :-1]) | ~sel[..., 1:])
    ca = torch.rand(B, F, 3, 2, dtype=torch.float64, generator=torch.Generator().manual_seed(3))
    from neural_renderer_b200 import functional as Fn
    got = Fn.interpolate_face_attributes(p2f, by, ca)
    x, on, valid, zn, A = oattr.attr_terms(faces.to(torch.float64), ca, osoft.pixel_centres(S), sigma, 0.1, 100.0, 1.0)
    for bb in range(B):
        for pp in range(0, S * S, 7):
            for k in range(K):
                fi = int(p2f.reshape(B, -1, K)[bb, pp, k])
                if fi >= 0:
                    torch.testing.assert_close(got.reshape(B, -1, K, 2)[bb, pp, k], A[bb, fi, pp], rtol=1e-12, atol=1e-13)


def test_sigma_to_zero_puts_the_covering_face_in_slot_zero():
    S = 32
    faces = torch.tensor([[[[-0.7, -0.6, 2.0], [0.8, -0.5, 3.0], [0.1, 0.75, 4.0]],
                           [[-0.9, 0.2, 1.5], [-0.2, 0.3, 1.5], [-0.6, 0.9, 1.5]],
                           [[-0.5, -0.5, 9.0], [0.5, -0.5, 9.0], [0.0, 0.5, 9.0]]]])
    b, pix, f, zp, certain, band = ofrag.candidates(faces, S, 1e-9)
    order = ofrag.sort_key(b, pix, f, zp)
    first = {}
    for i in order.tolist():
        first.setdefault(int(pix[i]), int(f[i]))
    xs = (2 * torch.arange(S, dtype=torch.float64) + 1 - S) / S
    n = 0
    for r in range(S):
        for c in range(S):
            best = None
            for j in range(3):
                v = faces[0, j].double()
                M = torch.stack((v[:, 0], v[:, 1], torch.ones(3, dtype=torch.float64)))
                w = torch.linalg.solve(M, torch.tensor([float(xs[c]), float(xs[S - 1 - r]), 1.0], dtype=torch.float64))
                if float(w.min()) >= 0.05:
                    z = 1.0 / float((w / v[:, 2]).sum())
                    if best is None or z < best[0]:
                        best = (z, j)
            if best is not None:
                assert first[r * S + c] == best[1], (r, c)
                n += 1
    assert n > 200


def test_sparse_selection_matches_dense():
    B, F, S, sigma = 2, 10, 24, 1e-3
    faces = _faces(9, F, B)
    dense = ofrag.candidates(faces, S, sigma)
    pix = torch.randperm(S * S, generator=torch.Generator().manual_seed(4))[:90]
    sparse = ofrag.candidates(faces, S, sigma, pix=pix)
    keep = torch.isin(dense[1], pix)
    od, os_ = ofrag.sort_key(*(t[keep] for t in dense[:4])), ofrag.sort_key(*sparse[:4])
    for td, ts in zip(dense, sparse):
        assert torch.equal(td[keep][od], ts[os_])


def test_new_kernels_compile_for_sm90a_without_spills(tmp_path):
    from neural_renderer_b200 import build
    nvcc = os.environ.get("NVCC", "nvcc")
    cmd = [nvcc] + build.NVCC_FLAGS + ["-Xptxas", "-v", "-c", os.path.join(build.CSRC, "nr_soft_frag.cu"),
                                       "-o", str(tmp_path / "nr_soft_frag.o")]
    log = subprocess.run(cmd, capture_output=True, text=True, check=True).stderr
    entries = re.split(r"Compiling entry function '", log)[1:]
    names = [e.split("'")[0] for e in entries]
    # the forward for kCap 4, 8, 16, 32 and 32- and 64-bit keys, and the backward; the binning kernels are nr_soft_rgb.cu's
    assert len(entries) == 9 and sum("k_soft_frag_fwd" in n for n in names) == 8, names
    assert sum("k_soft_frag_bwd" in n for n in names) == 1, names
    for e in entries:
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", e)
        assert m and m.groups() == ("0", "0", "0"), e[:400]
        assert "cumulative stack" not in e.split("Compile time")[0], e[:400]
    assert "sm_90a" in log
