"""GPU parity at raster sizes whose code paths the product chooses from the raster size alone, against the reference's
own kernels (oracle/refhost.py; one (1, 1, 1) binary per size, oracle/ref_configs.py SIZES).  Strip widths are those
of a call that returns rgb + alpha (the product has to run with the reference binary's flags):

  raster  edge-scan strips (W lines)        what else the size selects
  255     W = 2, last strip one line        odd (zero padding pixel), colours kept in the strip (S <= 256)
  257     W = 2, last strip one line        odd, face index only in the strip: colours come from the global rgb map
  700     W = 1                             big-face tiles clipped at a size that is not a multiple of 64; image 350 + AA
  1024    W = 1                             image 512 + AA
  2048    W = 1, 48 KB strip                global-atomics binning (k_face_bbox, k_strip_bin_global, k_strip_scan)
  2051    W = 1, 49 248-byte strip          global binning, no pixel-centre table in the forward, shared-memory opt-in

Every case is checked on the CPU to contain what reaches those paths (big faces that win pixels, faces partly off
screen or behind the camera, needles that win pixels beyond their tip, coverage of the last strip line and the last
pixel column), so that a change of the inputs cannot silently stop exercising them.
"""
import numpy as np
import pytest
import torch

from helpers import np_, rel_err
from ref_configs import SIZES, SIZES_F as F, SIZES_TS as TS
from test_gpu_configs import _compare, _need, _per_element
from test_gpu_parity import _grads, _outside_box_wins, _run_product

pytestmark = pytest.mark.gpu

TOL = 1e-4
B, NEAR, FAR, EPS = 2, 0.1, 100, 1e-4
FLAGS = (1, 1, 1)
BG = (0.2, 0.4, 0.6)
DEV = torch.device("cuda")
MODES = {"rgb": ("rgb",), "alpha": ("alpha",), "rgb_alpha": ("rgb", "alpha"), "depth": ("depth",)}

_CASES = {}


@pytest.fixture(scope="module", autouse=True)
def _gpu():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from neural_renderer_b200 import _lib
    _lib.load()
    yield
    _CASES.clear()


def _backside(v):
    """the reference's back-face rule (rasterize.py:306) on [...,3,3] faces"""
    return (v[..., 2, 1] - v[..., 0, 1]) * (v[..., 1, 0] - v[..., 0, 0]) < \
        (v[..., 1, 1] - v[..., 0, 1]) * (v[..., 2, 0] - v[..., 0, 0])


def _front(v):
    """the same faces, two vertices swapped where the face is back-facing"""
    return np.where(_backside(v)[..., None, None], v[..., [0, 2, 1], :], v)


def _box_area(v, S):
    """clipped pixel-box area of [...,3,3] faces (nr_bbox.cuh face_pixel_box), 0 for back-facing faces"""
    px, py = 0.5 * (v[..., 0] * S + S - 1), 0.5 * (v[..., 1] * S + S - 1)
    w = np.minimum(np.ceil(px.max(-1) + 1 / 256), S - 1) - np.maximum(np.floor(px.min(-1) - 1 / 256), 0) + 1
    h = np.minimum(np.ceil(py.max(-1) + 1 / 256), S - 1) - np.maximum(np.floor(py.min(-1) - 1 / 256), 0) + 1
    return np.where(_backside(v), 0, np.clip(w, 0, None) * np.clip(h, 0, None))


def _big_area(S):
    return 4096 if S > 256 else 1024  # nr_forward.cu: p.big_area


NBIG, NNEEDLE = 6, 8


def _mesh(S, seed):
    """[B,F,3,3]: a triangle soup reaching behind the camera (z from -1) and partly off screen; faces [0, NBIG) are
    front-facing faces above the big-face threshold, [NBIG, NBIG + NNEEDLE) needles in front of the soup, and face F-1
    a near front-facing triangle over the top-right corner: it covers the last column and the last row of the raster
    (the last strips of both axes) and its long edge crosses both."""
    from neural_renderer_b200 import synthetic
    faces = synthetic.triangle_soup(B, F, seed=seed, size=(0.02, 0.25), z_range=(-1.0, 3.0))
    e = 3.5 * np.sqrt(_big_area(S)) / S  # extents of a few times the side of the threshold box
    big = synthetic.triangle_soup(B, NBIG, seed=seed + 1, size=(e, 1.5 * e), z_range=(1.0, 2.0), duplicates=False,
                                  offscreen=False)
    faces[:, :NBIG] = _front(big)
    faces[:, NBIG:NBIG + NNEEDLE] = synthetic.needle_faces(B, NNEEDLE, S, seed=seed + 2, z_range=(0.2, 0.5))
    corner = np.array([[0.55, 1.3, 0.6], [1.3, 0.55, 0.6], [1.3, 1.3, 0.6]], np.float32)
    faces[:, F - 1] = _front(corner)
    return faces


def _case(S):
    """(faces, textures, reference result) of raster S, computed once per module"""
    if S not in _CASES:
        from neural_renderer_b200 import synthetic
        refhost = _need(S, F, TS, NEAR, FAR, EPS, FLAGS)
        faces = _mesh(S, seed=S)
        tex = synthetic.random_textures(B, F, TS, seed=S + 7)
        ref = refhost.rasterize_rgbad(torch.from_numpy(faces).to(DEV), torch.from_numpy(tex).to(DEV), S, False, NEAR,
                                      FAR, EPS, BG, *FLAGS)
        _CASES[S] = (faces, tex, ref)
    return _CASES[S]


def _check_case_reaches_its_paths(faces, ref_fim, S):
    """ref_fim: the reference's face_index_map [B,S,S] (raster orientation, row y = raster row y)"""
    area = _box_area(faces, S)
    for b in range(B):
        big = np.nonzero(area[b] > _big_area(S))[0]
        assert len(big) >= 3, "item %d: too few faces above the big-face threshold" % b
        assert np.isin(ref_fim[b], big).sum() > 100, "item %d: big faces win no pixels" % b
        # the last strip line of both axes: raster column S-1 and raster row S-1
        assert (ref_fim[b, :, S - 1] >= 0).sum() > 2 and (ref_fim[b, S - 1, :] >= 0).sum() > 2, "item %d" % b
        assert (ref_fim[b] == F - 1).any(), "item %d: the corner face wins no pixel" % b
    xy = faces[..., :2]
    partly_off = (np.abs(xy) > 1).any(-1).any(-1) & (np.abs(xy) < 1).all(-1).any(-1)
    assert partly_off.sum() >= 20, "too few faces partly off screen"
    behind = (faces[..., 2] < NEAR).any(-1) & ~_backside(faces)
    assert any(np.isin(ref_fim[b], np.nonzero(behind[b])[0]).any() for b in range(B)), \
        "no face reaching behind the camera wins a pixel"
    assert _outside_box_wins(ref_fim, faces, S) >= 4, "the needles win no pixels beyond their tips"


@pytest.mark.parametrize("S", SIZES)
def test_forward_vs_reference_kernels(S):
    """face_index_map, weight_map and rgb / alpha / depth bit-exact; the case reaches the size's paths."""
    faces, tex, ref = _case(S)
    _check_case_reaches_its_paths(faces, np_(ref.fn.face_index_map), S)
    got = _run_product(faces, tex, S, False, NEAR, FAR, EPS, BG, FLAGS)
    _compare(ref, got, FLAGS, False, check_bwd=False)


def _k5_fp64(S, grads):
    """grad_faces of K5 for raster S with float64 sums (CPU oracle, nr_oracle.c nro_pixel_bwd sum_fp64), and the
    oracle's face_index_map.  The reference kernels add each face's terms one after the other in fp32: at raster 2048
    that sum alone is off by ~4e-4 of the tensor maximum, while the product sums in another order."""
    import nr_oracle as o
    faces, tex, _ = _case(S)
    if ("oracle", S) not in _CASES:
        r = o.rasterize_rgbad(faces, tex, S, False, NEAR, FAR, EPS, BG, *FLAGS)
        r.fn.k5_sum_fp64 = True
        _CASES["oracle", S] = r
    r = _CASES["oracle", S]
    gf, _ = r.backward(*[np_(grads[k]) if k in grads else None for k in ("rgb", "alpha")], None)
    return gf, r.fn.face_index_map


@pytest.mark.parametrize("S,mode", [(S, m) for S in SIZES for m in MODES], ids=lambda v: str(v))
def test_backward_mode_vs_reference_kernels(S, mode):
    """One backward mode at a time (the product picks the edge-scan variant from the upstream gradients it gets):
    grad_faces per tensor and per element, grad_textures per tensor.  The edge-scan modes compare grad_faces with the
    reference's K5 summed in float64, and with the reference kernels themselves up to twice their own fp32 summation
    error (which stays below the 1e-4 tolerance up to raster 1024)."""
    faces, tex, ref = _case(S)
    grads = {k: v for k, v in _grads(ref, seed=S + 1).items() if k in MODES[mode]}
    got = _run_product(faces, tex, S, False, NEAR, FAR, EPS, BG, FLAGS, grads)
    gf, gt = ref.backward(grads.get("rgb"), grads.get("alpha"), grads.get("depth"))
    assert float(gf.abs().max()) > 0
    exact = np_(gf)
    tol_ref = TOL
    if mode != "depth":
        exact, fim = _k5_fp64(S, grads)
        assert np.array_equal(fim, np_(ref.fn.face_index_map))
        tol_ref = max(TOL, 2 * rel_err(np_(gf), exact))
        assert rel_err(np_(got["grad_faces"]), exact) <= TOL, "grad_faces vs float64 sums"
    assert rel_err(np_(got["grad_faces"]), np_(gf)) <= tol_ref, "grad_faces"
    err, n = _per_element(np_(got["grad_faces"]), exact, floor=1e-3)
    assert err <= 2e-3, (err, n)
    if "rgb" in grads:
        assert rel_err(np_(got["grad_tex"]), np_(gt)) <= TOL, "grad_textures"
    else:
        assert got["grad_tex"] is None or float(got["grad_tex"].abs().max()) == 0.0


@pytest.mark.parametrize("S", SIZES)
def test_sparse_gradient_on_the_last_row_and_column(S):
    """Upstream gradients at a handful of pixels, most of them on the last row / column of the raster where the colour
    changes along it: every K5 term is visible on its own, and components the reference leaves at exactly zero must
    stay zero -- a padding pixel or a stray strip line feeding a scan shows up here."""
    faces, tex, ref = _case(S)
    fim = np_(ref.fn.face_index_map.flip(1))  # image orientation: image row 0 = raster row S-1
    rng = np.random.default_rng(S)
    g_rgb, g_alpha = torch.zeros_like(ref["rgb"]), torch.zeros_like(ref["alpha"])
    for b in range(B):
        col = np.nonzero(np.diff(fim[b, :, S - 1]))[0]        # image rows where the last column changes face
        row = np.nonzero(np.diff(fim[b, 0, :]))[0]            # columns where the last raster row changes face
        assert len(col) and len(row), "the last row / column holds no face edge"
        pix = [(int(r) + int(rng.integers(2)), S - 1) for r in rng.choice(col, min(3, len(col)), replace=False)]
        pix += [(0, int(c) + int(rng.integers(2))) for c in rng.choice(row, min(3, len(row)), replace=False)]
        pix += [(0, S - 1), (S - 1, S - 1), (int(rng.integers(S)), int(rng.integers(S)))]
        for y, x in pix:
            g_rgb[b, :, y, x] = torch.from_numpy(rng.normal(size=3).astype(np.float32)).to(DEV)
            g_alpha[b, y, x] = float(rng.normal())
    gf_ref, gt_ref = ref.backward(g_rgb, g_alpha, None)
    got = _run_product(faces, tex, S, False, NEAR, FAR, EPS, BG, FLAGS, {"rgb": g_rgb, "alpha": g_alpha})
    assert float(gf_ref.abs().max()) > 0
    assert rel_err(np_(got["grad_faces"]), np_(gf_ref)) <= TOL
    err, _ = _per_element(np_(got["grad_faces"]), np_(gf_ref))
    assert err <= 1e-3, err
    zero = gf_ref == 0
    assert float(got["grad_faces"][zero].abs().max()) <= 1e-6 * float(gf_ref.abs().max())
    assert rel_err(np_(got["grad_tex"]), np_(gt_ref)) <= TOL


@pytest.mark.parametrize("image_size", [350, 512])
def test_anti_aliased_vs_reference_kernels(image_size):
    """Anti-aliasing on the one-line-strip rasters: image 350 (odd pooled size) -> raster 700, 512 -> 1024."""
    from neural_renderer_b200 import synthetic
    S = 2 * image_size
    refhost = _need(S, F, TS, NEAR, FAR, EPS, FLAGS)
    faces = _mesh(S, seed=S + 3)
    tex = synthetic.random_textures(B, F, TS, seed=S + 4)
    ref = refhost.rasterize_rgbad(torch.from_numpy(faces).to(DEV), torch.from_numpy(tex).to(DEV), image_size, True,
                                  NEAR, FAR, EPS, BG, *FLAGS)
    _check_case_reaches_its_paths(faces, np_(ref.fn.face_index_map), S)
    grads = _grads(ref, seed=5)
    got = _run_product(faces, tex, image_size, True, NEAR, FAR, EPS, BG, FLAGS, grads)
    assert got["rgb"].shape == (B, 3, image_size, image_size)
    gf, _ = _compare(ref, got, FLAGS, True, True, grads)
    err, n = _per_element(np_(got["grad_faces"]), np_(gf), floor=1e-3)
    assert err <= 2e-3, (err, n)


def test_binning_path_follows_the_raster_size():
    """The backward bins faces into strips with shared-memory counters up to 2048 counters per axis and with global
    atomics above (nr_backward.cu kBinSmemStrips): 1024 one-line strips use the former, 2048 and 2051 the latter.  If
    the threshold moves, this says so instead of the parity tests above quietly checking the other path."""
    from neural_renderer_b200 import _lib
    from neural_renderer_b200 import synthetic
    lib = _lib.load()
    faces = synthetic.triangle_soup(1, 64, seed=1)
    tex = synthetic.random_textures(1, 64, TS, seed=2)
    launched = {}
    _lib.read_profile()  # drop earlier records
    lib.nr_b200_set_profiling(1)
    try:
        for S in (1024, 2048, 2051):
            g = {"rgb": torch.ones((1, 3, S, S), device=DEV), "alpha": torch.ones((1, S, S), device=DEV)}
            _run_product(faces, tex, S, False, NEAR, FAR, EPS, BG, FLAGS, g)
            launched[S] = {name for name, _ in _lib.read_profile()}
    finally:
        lib.nr_b200_set_profiling(0)
    for S in (1024, 2048, 2051):
        assert "k_edge_scan" in launched[S], (S, launched[S])
        glob = {"k_face_bbox", "k_strip_scan"} <= launched[S]
        assert glob == (S >= 2048), (S, sorted(launched[S]))


def test_indexed_geometry_at_2051():
    """NR_FACES_INDEXED at the largest odd size (global binning, no pixel-centre table): the maps equal those of the
    materialised faces bit for bit, and d loss / d vertices is the scatter-add of d loss / d faces."""
    import neural_renderer as nr
    import importlib
    from test_gpu_glue import _indexed_case
    R = importlib.import_module("neural_renderer_b200.rasterize")
    S, Bi = 2051, 2
    v_np, f_np = _indexed_case(Bi, seed=6)
    idx = torch.from_numpy(f_np).to(DEV)
    idx_b = idx[None].expand(Bi, -1, -1).contiguous()
    tex = torch.rand((Bi, f_np.shape[0], TS, TS, TS, 3), generator=torch.Generator().manual_seed(2)).to(DEV)
    gen = torch.Generator().manual_seed(3)
    g = [torch.randn(s, generator=gen).to(DEV) for s in ((Bi, 3, S, S), (Bi, S, S), (Bi, S, S))]
    v = torch.from_numpy(v_np).to(DEV).requires_grad_(True)
    a = R._run(idx, tex, S, False, NEAR, FAR, EPS, BG, *FLAGS, vertices=v)
    sum((o * gi).sum() for o, gi in zip(a[:3], g)).backward()
    fm = nr.vertices_to_faces(v.detach(), idx_b).contiguous().requires_grad_(True)
    m = R._run(fm, tex, S, False, NEAR, FAR, EPS, BG, *FLAGS)
    sum((o * gi).sum() for o, gi in zip(m[:3], g)).backward()
    for x, y in zip(a, m):
        assert torch.equal(x, y)
    assert (a[3] >= 0).float().mean() > 0.2
    scattered = torch.zeros_like(v).index_add_(1, idx.reshape(-1).long(), fm.grad.reshape(Bi, -1, 3))
    assert rel_err(np_(v.grad), np_(scattered)) <= 1e-5
