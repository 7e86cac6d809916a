"""CPU: the soft blend of fragments -- nr_b200_blend_args against the header, the new symbols, the host rejections of
both entry points (all decided before any launch), the Python argument errors (raised before the device check), the
float64 oracle's self-checks (tests/oracles_soft_blend.py), and the spills of the new kernels."""
import ctypes
import math
import os
import re
import subprocess

import pytest
import torch

import oracles_soft_blend as oblend

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


def test_blend_struct_matches_the_header(tmp_path):
    from neural_renderer_b200 import _lib
    fields = [f[0] for f in _lib.BlendArgs._fields_]
    exprs = ["sizeof(nr_b200_blend_args)"] + ["offsetof(nr_b200_blend_args, %s)" % f for f in fields]
    src = tmp_path / "s.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "nr_b200.h"\nint main(void){'
                   + "".join('printf("%%zu\\n", (size_t)(%s));' % e for e in exprs) + "return 0;}\n")
    exe = tmp_path / "s"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    vals = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert vals[0] == ctypes.sizeof(_lib.BlendArgs) == 136
    assert vals[1:] == [getattr(_lib.BlendArgs, f).offset for f in fields]


def test_new_symbols_are_exported(lib):
    from neural_renderer_b200 import _lib
    out = subprocess.run(["nm", "-D", "--defined-only", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    for n in ("nr_b200_blend_fragments", "nr_b200_blend_fragments_backward"):
        assert n in _lib.EXPORTED_SYMBOLS
        assert (" T " + n) in out, n


def _args(backward=False, **kw):
    from neural_renderer_b200 import _lib
    a = _lib.BlendArgs(struct_size=ctypes.sizeof(_lib.BlendArgs), batch_size=2, height=8, width=9, faces_per_pixel=8,
                       channels=3, sigma=1e-4, gamma=1e-4, near_=0.1, far_=100.0)
    a.pix_to_face = a.zbuf = a.dists = a.colors = a.out = a.alpha = _P
    if backward:
        a.grad_out = a.grad_alpha = a.grad_colors = a.grad_zbuf = a.grad_dists = _P
    for k, v in kw.items():
        setattr(a, k, v)
    return a


@pytest.mark.parametrize("backward", [False, True])
def test_host_rejections(lib, backward):
    from neural_renderer_b200 import _lib
    fn = lib.nr_b200_blend_fragments_backward if backward else lib.nr_b200_blend_fragments
    bad = [dict(struct_size=0), dict(struct_size=ctypes.sizeof(_lib.BlendArgs) + 8), dict(struct_size=4),
           dict(batch_size=0), dict(height=0), dict(width=-1), dict(channels=0), dict(faces_per_pixel=0),
           dict(faces_per_pixel=-1), dict(faces_per_pixel=33),
           dict(batch_size=1 << 30, height=1 << 30, width=1 << 30),             # B H W K C past 64-bit indices
           dict(sigma=0.0), dict(sigma=-1.0), dict(sigma=float("nan")), dict(sigma=float("inf")), dict(sigma=1e-45),
           dict(gamma=0.0), dict(gamma=-1e-4), dict(gamma=float("nan")), dict(gamma=float("inf")), dict(gamma=1e-45),
           dict(near_=2.0, far_=1.0), dict(near_=1.0, far_=1.0), dict(near_=float("nan")), dict(far_=float("inf")),
           dict(near_=-3e38, far_=3e38),                                         # far - near overflows
           dict(pix_to_face=None), dict(zbuf=None), dict(dists=None), dict(colors=None), dict(out=None),
           # element alignment: 8 bytes for pix_to_face, 4 for the rest
           dict(pix_to_face=_P + 4), dict(zbuf=_P + 2), dict(dists=_P + 1), dict(colors=_P + 3), dict(out=_P + 2),
           dict(alpha=_P + 1), dict(background=_P + 2)]
    if not backward:
        bad += [dict(alpha=None)]                                           # the backward does not read alpha
    if backward:
        bad += [dict(grad_colors=None, grad_zbuf=None, grad_dists=None), dict(grad_out=_P + 2),
                dict(grad_alpha=_P + 1), dict(grad_colors=_P + 2), dict(grad_zbuf=_P + 1), dict(grad_dists=_P + 3)]
    for kw in bad:
        assert fn(ctypes.byref(_args(backward, **kw)), None) == INVALID, kw
        assert lib.nr_b200_last_launch_count() == 0
    assert fn(None, None) == INVALID
    assert lib.nr_b200_last_launch_count() == 0


def test_python_argument_errors_come_before_the_device_check():
    import neural_renderer_b200 as nr
    B, H, W, K, C = 1, 4, 5, 3, 2
    p2f = torch.full((B, H, W, K), -1, dtype=torch.int64)
    zb, ds = torch.zeros(B, H, W, K), torch.zeros(B, H, W, K)
    frag = nr.Fragments(p2f, zb, torch.zeros(B, H, W, K, 3), ds)
    col = torch.zeros(B, H, W, K, C)
    with pytest.raises(NotImplementedError):                   # valid arguments on the CPU: no CPU path
        nr.blend_soft_fragments(frag, col, 1e-4, 1e-4)
    with pytest.raises(NotImplementedError):
        nr.blend_soft_fragments(frag, col, 1e-4, 1e-4, background=[0.5, 0.25])
    for kw in (dict(sigma=0.0), dict(sigma=float("nan")), dict(sigma=-1.0), dict(sigma=float("inf")),
               dict(gamma=0.0), dict(gamma=float("nan")), dict(gamma=float("inf")), dict(near=2.0, far=1.0),
               dict(near=1.0, far=1.0), dict(near=float("nan")), dict(background=[0.0]),
               dict(background=torch.zeros(3)), dict(background=torch.zeros(1, 2))):
        with pytest.raises(ValueError):
            nr.blend_soft_fragments(frag, col, **{"sigma": 1e-4, "gamma": 1e-4, **kw})
    for kw in (dict(sigma="x"), dict(gamma=None), dict(background="ab")):
        with pytest.raises(TypeError):
            nr.blend_soft_fragments(frag, col, **{"sigma": 1e-4, "gamma": 1e-4, **kw})
    bad_frags = [nr.Fragments(p2f.int(), zb, None, ds),                  # dtype of pix_to_face
                 nr.Fragments(p2f[..., :2], zb, None, ds),               # K mismatch
                 nr.Fragments(p2f, zb[..., :2], None, ds),
                 nr.Fragments(p2f, zb, None, ds.long()),                 # dtype of dists
                 nr.Fragments(p2f[0], zb[0], None, ds[0])]               # rank
    for f in bad_frags:
        with pytest.raises(ValueError):
            nr.blend_soft_fragments(f, col, 1e-4, 1e-4)
    for c in (col[..., :2, :], col[0], col.long(), torch.zeros(B, H, W, K, 0)):  # K mismatch, rank, dtype, C = 0
        with pytest.raises(ValueError):
            nr.blend_soft_fragments(frag, c, 1e-4, 1e-4)
    with pytest.raises(ValueError):                            # K past the fragments' cap
        k = 33
        nr.blend_soft_fragments(nr.Fragments(torch.full((1, 1, 1, k), -1), torch.zeros(1, 1, 1, k), None,
                                             torch.zeros(1, 1, 1, k)), torch.zeros(1, 1, 1, k, 1), 1e-4, 1e-4)
    with pytest.raises(TypeError):                             # sigma and gamma are required
        nr.blend_soft_fragments(frag, col)
    with pytest.raises(TypeError):
        nr.blend_soft_fragments(frag, col, 1e-4)
    with pytest.raises(TypeError):
        nr.blend_soft_fragments((p2f, zb), col, 1e-4, 1e-4)
    with pytest.raises(TypeError):
        nr.blend_soft_fragments(frag, col.tolist(), 1e-4, 1e-4)
    if torch.cuda.is_available():                              # mixed devices
        with pytest.raises(ValueError):
            nr.blend_soft_fragments(frag, col.cuda(), 1e-4, 1e-4)


# ------------------------------------------------------------------------------------------------ oracle self-checks
def _inputs(seed, B=2, H=3, W=4, K=5, C=3, sigma=1e-3, empty=0.3):
    g = torch.Generator().manual_seed(seed)
    p2f = torch.randint(0, 50, (B, H, W, K), generator=g)
    p2f[torch.rand(B, H, W, K, generator=g) < empty] = -1
    zb = 1.0 + 4.0 * torch.rand(B, H, W, K, generator=g, dtype=torch.float64)
    ds = (torch.rand(B, H, W, K, generator=g, dtype=torch.float64) * 2 - 1) * 5 * sigma
    col = torch.rand(B, H, W, K, C, generator=g, dtype=torch.float64)
    return p2f, zb, ds, col


def test_one_slot_in_closed_form():
    sigma, gamma, near, far = 1e-3, 1e-2, 0.1, 100.0
    p2f, zb, ds, col = _inputs(1, K=1, empty=0.0)
    bg = [0.2, 0.4, 0.6]
    out, alpha = oblend.blend(p2f, zb, ds, col, sigma, gamma, near, far, bg)
    D = 1 / (1 + torch.exp(-ds[..., 0] / sigma))
    zbg = far - 1e-3 * (far - near)
    wb = torch.exp((zb[..., 0] - zbg) / ((far - near) * gamma))               # zref = the slot's depth
    want = (D[..., None] * col[..., 0, :] + wb[..., None] * torch.tensor(bg, dtype=torch.float64)) / (D + wb)[..., None]
    torch.testing.assert_close(out, want.permute(0, 3, 1, 2), rtol=1e-13, atol=1e-15)
    torch.testing.assert_close(alpha, D, rtol=1e-13, atol=1e-15)


def test_an_empty_pixel_gives_the_background_and_zero_alpha():
    p2f, zb, ds, col = _inputs(2)
    p2f[0, 1, 2] = -1
    zb[0, 1, 2], ds[0, 1, 2], col[0, 1, 2] = float("nan"), float("inf"), float("nan")   # whatever they hold
    out, alpha = oblend.blend(p2f, zb, ds, col, 1e-3, 1e-4, background=[0.1, 0.2, 0.3])
    assert out[0, :, 1, 2].tolist() == pytest.approx([0.1, 0.2, 0.3], abs=1e-15)
    assert alpha[0, 1, 2].item() == 0.0
    assert torch.isfinite(out).all() and torch.isfinite(alpha).all()
    # and no gradient leaks out of the invalid slots
    zv, dv, cv = (t.clone().requires_grad_(True) for t in (zb, ds, col))
    o, a = oblend.blend(p2f, zv, dv, cv, 1e-3, 1e-4)
    (o.sum() + a.sum()).backward()
    for g in (zv.grad, dv.grad):
        assert torch.isfinite(g).all() and torch.all(g[p2f < 0] == 0)
    assert torch.isfinite(cv.grad).all() and torch.all(cv.grad[p2f < 0] == 0)


def test_an_inside_fragment_gives_its_colour_as_gamma_goes_to_zero():
    sigma = 1e-4
    p2f = torch.tensor([[[[3, 7, -1, 2]]]])
    zb = torch.tensor([[[[2.0, 1.5, 0.5, 3.0]]]], dtype=torch.float64)           # slot 1 is the nearest valid one
    ds = torch.tensor([[[[2e-3, 3e-3, 0.0, 1e-3]]]], dtype=torch.float64)         # all well inside: D ~ 1
    col = torch.rand(1, 1, 1, 4, 3, generator=torch.Generator().manual_seed(3), dtype=torch.float64)
    out, _ = oblend.blend(p2f, zb, ds, col, sigma, 1e-6, background=[9.0, 9.0, 9.0])
    torch.testing.assert_close(out[0, :, 0, 0], col[0, 0, 0, 1], rtol=1e-9, atol=1e-12)


def test_slot_permutation_invariance_in_float64():
    p2f, zb, ds, col = _inputs(4, K=7)
    zb[0, 0, 0, 1] = zb[0, 0, 0, 4]                                           # a zbuf tie
    ref = oblend.blend(p2f, zb, ds, col, 1e-3, 1e-3, background=[0.3, 0.1, 0.7])
    perm = torch.randperm(7, generator=torch.Generator().manual_seed(5))
    got = oblend.blend(p2f[..., perm], zb[..., perm], ds[..., perm], col[..., perm, :], 1e-3, 1e-3,
                       background=[0.3, 0.1, 0.7])
    for r, g in zip(ref, got):
        torch.testing.assert_close(g, r, rtol=1e-13, atol=1e-15)


def test_gates_cover_a_float32_evaluation_of_the_definition():
    # the fp32 arithmetic the kernel performs, evaluated here in the same order, stays inside the derived gates
    sigma, gamma, near, far = 1e-4, 1e-4, 0.1, 100.0
    p2f, zb, ds, col = _inputs(6, B=2, H=8, W=8, K=8, C=3, sigma=sigma)
    zb, ds, col = zb.float(), ds.float(), col.float()
    valid = p2f >= 0
    fn = far - near
    inv_s = torch.tensor(1.0 / sigma, dtype=torch.float32)
    inv_fg = torch.tensor(1.0 / (fn * gamma), dtype=torch.float32)
    zbg = torch.tensor(far - 1e-3 * fn, dtype=torch.float32)
    zref = torch.minimum(torch.where(valid, zb, torch.full_like(zb, math.inf)).amin(-1), zbg)
    x = ds * inv_s
    w = torch.where(valid, torch.sigmoid(x) * torch.exp((zref[..., None] - zb) * inv_fg), torch.zeros_like(x))
    wb = torch.exp((zref - zbg) * inv_fg)
    Z, N = wb.clone(), torch.zeros_like(col[..., 0, :])
    for k in range(8):
        Z = Z + w[..., k]
        N = N + w[..., k, None] * torch.where(valid[..., k, None], col[..., k, :], torch.zeros_like(N))
    out32 = (N / Z[..., None]).permute(0, 3, 1, 2)
    ref, _ = oblend.blend(p2f, zb, ds, col, sigma, gamma, near, far)
    g_out, _ = oblend.gates(p2f, zb, ds, col, sigma, gamma, near, far)
    assert torch.all((out32.double() - ref).abs() <= g_out)
    assert g_out.max() < 1e-4


def test_new_kernels_compile_for_sm90a_without_spills(tmp_path):
    from neural_renderer_b200 import build
    nvcc = os.environ.get("NVCC", "nvcc")
    cmd = [nvcc] + build.NVCC_FLAGS + ["-Xptxas", "-v", "-c", os.path.join(build.CSRC, "nr_soft_blend.cu"),
                                       "-o", str(tmp_path / "nr_soft_blend.o")]
    log = subprocess.run(cmd, capture_output=True, text=True, check=True).stderr
    entries = re.split(r"Compiling entry function '", log)[1:]
    names = [e.split("'")[0] for e in entries]
    # the forward and the backward, each staged through shared memory and per thread
    assert len(entries) == 4, names
    assert sum("k_soft_blend_fwd" in n for n in names) == 2 and sum("k_soft_blend_bwd" in n for n in names) == 2, names
    for e in entries:
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", e)
        assert m and m.groups() == ("0", "0", "0"), e[:400]
        assert "cumulative stack" not in e.split("Compile time")[0], e[:400]
    assert "sm_90a" in log
