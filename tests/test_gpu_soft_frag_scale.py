"""GPU: the soft fragment backwards (k_soft_frag_bwd, k_soft_interp_bwd) and the blend behind them, held to float64 where
their merges of gradients branch: a tile with more distinct faces than k_soft_frag_bwd's hash table holds, home buckets
that collide and wrap from the last slot to the first, the deep-tile, 64-bit-key and benchmark scenes, and
interpolation groups of 32 pixels that straddle two items or end short.

Every reference is float64 autograd of oracles_soft_frag.evaluate at the kernel's own pix_to_face, so no tie or cut-off
decision can differ between the kernel and the oracle.  Where the upstream gradient sits only on chosen pixels, the
oracle gets a pix_to_face masked to -1 everywhere else.  Gates, as the sibling files pass them:
  - elem_err(floor=1e-3) <= 2e-3 for the vertex gradients of scenes as small as tests/test_gpu_soft_frag.py's (64^2,
    the teapot at 128^2);
  - test_gpu_soft_scale.check_grads (rel_err <= 5e-3, elem_err(floor=2e-2) <= 5e-2) at the deep-tile, 64-bit-key and
    benchmark scenes;
  - test_gpu_soft_interp's gates for the interpolation (elem_err(floor=1e-3) <= 1e-4 for grad_bary, 5e-4 for the
    attributes).
Each scene asserts on the host that it reaches its branch.  Every test stays below 2.2 GiB of device memory.

Measured on an H100 80GB HBM3 at a 700 W power limit, five runs in a row: the file ran in 18-24 s, and its largest test
(the spheres' long interpolation runs) peaked at 1.54 GiB of device memory."""
import math

import numpy as np
import pytest
import torch

import oracles_soft as osoft
import oracles_soft_blend as oblend
import oracles_soft_frag as ofrag
import soft_binning as sb
import test_gpu_soft_interp as tsi
import test_gpu_soft_scale as tss
from helpers import elem_err, rel_err
from test_gpu_soft_frag import _oracle_grads, _teapot, check_selection, check_values

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
NEAR, FAR = 0.1, 100.0
PEAK_LIMIT = int(2.2 * 2 ** 30)

# k_soft_frag_bwd's hash table (csrc/nr_soft_frag.cu; tests/test_soft_frag_scale_cpu.py reads both from the source)
K_TABLE = 1024
HASH_MUL = 2654435761


def home_bucket(f):
    """the table slot where face f's probe starts: (f * HASH_MUL mod 2^32) >> (32 - log2 K_TABLE)"""
    f = np.asarray(f, dtype=np.uint64)
    return ((f * np.uint64(HASH_MUL)) % np.uint64(1 << 32)) >> np.uint64(32 - int(math.log2(K_TABLE)))


def _nr():
    import neural_renderer_b200 as nr
    return nr


@pytest.fixture(autouse=True)
def _peak_memory():
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats(DEV)
    yield
    torch.cuda.synchronize()
    assert torch.cuda.max_memory_allocated(DEV) <= PEAK_LIMIT, torch.cuda.max_memory_allocated(DEV)


def _rand(shape, seed, lo=-1.0, hi=1.0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return lo + (hi - lo) * torch.rand(*shape, device=DEV, generator=g)


# ------------------------------------------------------------------------------------------------ the dense field
S_DENSE, F_DENSE = 64, 16384
SIGMA_DENSE = (2.0 / S_DENSE) ** 2 / math.log((1.0 - osoft.EPS) / osoft.EPS)     # a reach of exactly 1 pixel
WINDOW = 44                                                                      # home buckets 1002 .. 1023, 0 .. 21
WINDOW_TILE = (1, 0)                                                             # (ty, tx): the sparse column


def dense_field(B, seed):
    """[B,F,3,3] float32 numpy: F_DENSE near-equilateral faces of 0.2-0.4 px radius, 4 per pixel on average, their
    centres spread in x with density 1 + 6 t (t = (x + 1) / 2): about 1.75 faces per pixel in the left tile column and
    6.25 in the right one, so one launch has tiles below and above the table's 1024 faces.  Every vertex depth is drawn
    from [2, 3] on its own: the faces are tilted, so zbuf's partials in x and y, which go through differences of 1 / z_k
    across the face, are not a cancellation of nearly equal terms."""
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(B):
        u = rng.uniform(0.0, 1.0, F_DENSE)
        t = (np.sqrt(1.0 + 48.0 * u) - 1.0) / 6.0                                # inverse of the CDF (t + 3 t^2) / 4
        c = np.stack((2.0 * t - 1.0, rng.uniform(-1.0, 1.0, F_DENSE)), -1)[:, None]
        r = rng.uniform(0.2, 0.4, (F_DENSE, 1, 1)) * 2.0 / S_DENSE
        ang = rng.uniform(0.0, 2 * np.pi, (F_DENSE, 1, 1)) + np.array([0.0, 2.1, 4.2])[None, :, None]
        xy = c + r * np.concatenate((np.cos(ang), np.sin(ang)), -1)
        z = rng.uniform(2.0, 3.0, (F_DENSE, 3, 1))
        out.append(np.concatenate((xy, z), -1))
    return np.stack(out).astype(np.float32)


def tile_reach(faces, S, sigma, tile):
    """[B,F] bool numpy: the faces whose xy box, grown by the reach and one pixel more, meets the pixel centres of tile
    (ty, tx); every face the kernel can select in that tile is among them"""
    ty, tx = tile
    ctr = lambda i: (2.0 * i + 1.0 - S) / S                                      # noqa: E731
    grow = math.sqrt(osoft.cut(sigma)) + 2.0 / S
    x0, x1 = ctr(tx * 16) - grow, ctr(min(S, tx * 16 + 16) - 1) + grow
    y0, y1 = ctr(S - min(S, ty * 16 + 16)) - grow, ctr(S - 1 - ty * 16) + grow
    x, y = faces[..., 0].astype(np.float64), faces[..., 1].astype(np.float64)
    return (x.max(-1) >= x0) & (x.min(-1) <= x1) & (y.max(-1) >= y0) & (y.min(-1) <= y1)


def windowed(faces, S, sigma, seed, tile=WINDOW_TILE, width=WINDOW):
    """faces [B,F,3,3] numpy with the face indices permuted per item, so that every face that can reach `tile` takes an
    index whose home bucket lies in the `width` buckets around the wrap from slot K_TABLE - 1 to slot 0; the others
    take the remaining indices.  Returns (faces, the reaching faces' count per item)."""
    B, F = faces.shape[:2]
    home = home_bucket(np.arange(F)).astype(np.int64)
    win = np.nonzero((home + width // 2) % K_TABLE < width)[0]
    rest = np.nonzero((home + width // 2) % K_TABLE >= width)[0]
    near = tile_reach(faces, S, sigma, tile)
    rng = np.random.default_rng(seed)
    out, counts = np.empty_like(faces), []
    for b in range(B):
        mine, others = np.nonzero(near[b])[0], np.nonzero(~near[b])[0]
        assert mine.size <= win.size, (mine.size, win.size)
        dst = rng.permutation(win)[:mine.size]
        free = np.setdiff1d(np.arange(F), dst)
        out[b, dst] = faces[b, rng.permutation(mine)]
        out[b, free] = faces[b, rng.permutation(others)]
        counts.append(mine.size)
    assert rest.size + win.size == F
    return out, counts


def tile_face_keys(p2f, F=None):
    """the distinct (item, 16 x 16 tile, face) of pix_to_face [B,S,S,K], as keys (b tiles + tile) F + f"""
    B, S, _, K = p2f.shape
    nt = sb.tiles_per_axis(S)
    r = torch.arange(S, device=p2f.device)
    tile = ((r[:, None] // 16) * nt + r[None, :] // 16)[None, :, :, None].expand(B, -1, -1, K)
    b = torch.arange(B, device=p2f.device)[:, None, None, None].expand_as(p2f)
    F = int(p2f.max().item()) + 1 if F is None else F
    return ((b * nt * nt + tile) * F + p2f)[p2f >= 0].unique()


def tile_face_counts(p2f):
    """[B, tiles] distinct faces per (item, 16 x 16 tile) of pix_to_face [B,S,S,K]: the keys k_soft_frag_bwd's table holds
    for that CTA (every fragment with a nonzero upstream gradient)"""
    B, S = p2f.shape[:2]
    nt = sb.tiles_per_axis(S)
    F = int(p2f.max().item()) + 1
    return torch.bincount(tile_face_keys(p2f, F) // F, minlength=B * nt * nt).reshape(B, nt * nt)


def _dense(seed=1, B=2):
    return torch.from_numpy(dense_field(B, seed)).to(DEV)


def _used(p2f, F):
    used = torch.zeros(p2f.shape[0], F, dtype=torch.bool, device=DEV)
    for b in range(p2f.shape[0]):
        used[b, p2f[b][p2f[b] >= 0].unique()] = True
    return used


def _upstream(frag, which, seed, mask=None):
    """random upstream gradients on zbuf, bary_coords and dists (None where `which` leaves one out), zero outside the
    pixels `mask` [B,S,S] if given"""
    names = ("zbuf", "bary", "dists")
    ups = []
    for i, (t, n) in enumerate(zip((frag.zbuf, frag.bary_coords, frag.dists), names)):
        if which not in ("all", n):
            ups.append(None)
            continue
        u = _rand(t.shape, seed + i)
        if mask is not None:
            u = u * (mask[..., None] if t.dim() == 4 else mask[..., None, None])
        ups.append(u)
    return ups


def _kernel_grad(leaf, frag, ups):
    outs = [(o, u) for o, u in zip((frag.zbuf, frag.bary_coords, frag.dists), ups) if u is not None]
    (g,) = torch.autograd.grad([o for o, _ in outs], leaf, [u for _, u in outs])
    return g


def _check_small(g, ref):
    e = elem_err(g.cpu(), ref.cpu(), floor=1e-3)
    assert e <= 2e-3, e
    return e


def _check_backward_dense(faces, S, sigma, K, which, form, seed):
    """the vertex gradient of one call against float64, faces form or `vertices=` with shared indices; faces without a
    fragment get exactly 0.  Returns the fragments."""
    nr = _nr()
    B, F = faces.shape[:2]
    if form == "faces":
        leaf = faces.clone().requires_grad_(True)
        frag = nr.rasterize_soft_fragments(leaf, S, sigma, K)
    else:
        verts = faces.reshape(B, F * 3, 3).contiguous()
        idx = torch.arange(F * 3, device=DEV, dtype=torch.int32).reshape(F, 3)
        leaf = verts.clone().requires_grad_(True)
        frag = nr.rasterize_soft_fragments(idx, S, sigma, K, vertices=leaf)
    ups = _upstream(frag, which, seed)
    g = _kernel_grad(leaf, frag, ups)
    ref = _oracle_grads(faces, frag, S, ups)
    if form != "faces":
        ref = ref.reshape(B, F * 3, 3)
    if which == "dists":
        # dists alone.  A fragment's partials are +-2 g (1 - t) q and +-2 g t q for its nearest edge (a, b), q = p - a -
        # t e, and the kernel's q = fma(-t, e, p - a) rounds p - a, e and t once each: an absolute error of a few eps
        # (|q| + 2 |e|).  So an element errs by a few eps times the sum of its terms' sizes, not of their sum.  Here the
        # edges (|e| <= 0.7 px) are as long as q (|q| <= 1 px, the reach), so that sum of sizes is of the order of the
        # largest element, and an element whose terms cancel down to elem_err's floor (1e-3 of the largest element) may
        # err by a few eps / 1e-3, about 1e-3 of the floor, times however much its terms outweigh the largest element:
        # the small gate's 2e-3 is no bound.  check_grads' floor of 2e-2 leaves twenty times more.  (With zbuf or bary in the upstream, the barycentric partials, about 1 / |e|
        # larger, set the floor, and these errors fall far below it.)
        tss.check_grads([g], [ref], ["faces"], ("dense", K, which, form))
    else:
        _check_small(g, ref)
    used = _used(frag.pix_to_face, F)
    gf = g.reshape(B, F, 3, 3)
    assert torch.all(gf[~used] == 0) and gf[used].abs().max() > 0
    return frag


# ------------------------------------------------------------------------------------------------ 1. past a full table
@pytest.mark.parametrize("K,which,form", [(8, "all", "faces"), (16, "all", "faces"), (32, "all", "faces"),
                                          (16, "zbuf", "faces"), (16, "bary", "faces"), (16, "dists", "faces"),
                                          (16, "all", "vertices"), (32, "all", "vertices")])
def test_dense_field_fills_and_overflows_the_hash_table(K, which, form):
    faces = _dense()
    frag = _check_backward_dense(faces, S_DENSE, SIGMA_DENSE, K, which, form, 10 * K)
    n = tile_face_counts(frag.pix_to_face)
    print("dense K", K, "distinct faces per tile", n.min().item(), n.max().item())
    # one launch has tiles that fill the table and overflow it, and tiles that hold between half and all of it
    if K >= 16:
        assert (n > K_TABLE).any(), n.max().item()
    assert ((n > K_TABLE // 2) & (n <= K_TABLE)).any(), n


# ------------------------------------------------------------------------------------------------ 2. colliding home buckets
def _windowed_faces(B=2, seed=2):
    return torch.from_numpy(windowed(dense_field(B, seed), S_DENSE, SIGMA_DENSE, seed + 1)[0]).to(DEV)


@pytest.mark.parametrize("K,form", [(8, "faces"), (32, "faces"), (32, "vertices")])
def test_colliding_home_buckets_wrap_around_the_table(K, form):
    faces = _windowed_faces()
    frag = _check_backward_dense(faces, S_DENSE, SIGMA_DENSE, K, "all", form, 20 + K)
    ty, tx = WINDOW_TILE
    p = frag.pix_to_face[:, ty * 16:ty * 16 + 16, tx * 16:tx * 16 + 16]
    for b in range(faces.shape[0]):
        ids = p[b][p[b] >= 0].unique().cpu().numpy()
        home = home_bucket(ids).astype(np.int64)
        # every face of the tile starts its probe in the window, and more of them start in its upper part than it has
        # slots before the wrap, so the probe chain runs from slot K_TABLE - 1 on to slot 0
        assert np.all((home + WINDOW // 2) % K_TABLE < WINDOW), np.unique(home)
        upper = (home >= K_TABLE - WINDOW // 2).sum()
        assert upper > WINDOW // 2 and (home < WINDOW // 2).any(), (upper, ids.size)
        assert ids.size > 300, ids.size


# ------------------------------------------------------------------------------------------------ 3. the other shapes
@pytest.mark.parametrize("K", [4, 5, 16, 17])
def test_dense_field_forward_by_definition(K):
    nr = _nr()
    faces = _dense(seed=3)
    frag = nr.rasterize_soft_fragments(faces, S_DENSE, SIGMA_DENSE, K)
    n = check_selection(frag, faces, S_DENSE, SIGMA_DENSE, K)
    check_values(frag, faces, S_DENSE)
    assert (n == K).float().mean().item() > 0.2, (n == K).float().mean().item()


@pytest.mark.parametrize("K", [8, 32])
def test_deep_tiles_backward(K):
    nr = _nr()
    faces = tss._deep_faces()
    S, sigma = tss.S_DEEP, tss.SIGMA_DEEP
    fv = faces.clone().requires_grad_(True)
    frag = nr.rasterize_soft_fragments(fv, S, sigma, K)
    assert (sb.rounds(sb.tile_entries_lower_bound(faces, S, sigma)) >= 3).any()
    ups = _upstream(frag, "all", 30 + K)
    g = _kernel_grad(fv, frag, ups)
    ref = _oracle_grads(faces, frag, S, ups)
    tss.check_grads([g], [ref], ["faces"], ("deep", K))
    assert torch.all(g[~_used(frag.pix_to_face, faces.shape[1])] == 0)


def _p2f_only(p2f):
    """a Fragments holding only pix_to_face, all that _oracle_grads reads"""
    from neural_renderer_b200.rasterize import Fragments
    return Fragments(p2f, None, None, None)


def test_64_bit_keys_backward():
    """F 65535 (32-bit keys) and 65536 (64-bit): the upstream gradient near the real faces, the float64 oracle on the
    host (its [B,S,S,K] float64 fields at 2049^2 would not fit the device budget); padding faces get exactly 0"""
    nr = _nr()
    B, S, sigma, K = 2, tss.S_KEY, tss.SIGMA_KEY, 2
    real = tss._real_faces(B, 21)
    pix = tss._pixels_near(real, S, 256, 23)                                    # [B,P]
    mask = torch.zeros(B, S * S, dtype=torch.bool, device=DEV).scatter_(1, pix, True).reshape(B, S, S)
    grads = []
    for F in (65535, 65536):
        assert sb.key_width(B, F, S)[2] is (F == 65536)
        faces, pos = tss._padded(real, F, 22 + F)
        pad = torch.ones(F, dtype=torch.bool, device=DEV)
        pad[pos] = False
        fv = faces.clone().requires_grad_(True)
        frag = nr.rasterize_soft_fragments(fv, S, sigma, K)
        ups = _upstream(frag, "all", 40, mask)
        g = _kernel_grad(fv, frag, ups)
        assert torch.all(g[:, pad] == 0)
        p2f = torch.where(mask[..., None], frag.pix_to_face, torch.full_like(frag.pix_to_face, -1)).cpu()
        del frag
        ref = _oracle_grads(faces.cpu(), _p2f_only(p2f), S, [u.cpu() for u in ups])
        del ups
        tss.check_grads([g[:, pos]], [ref[:, pos.cpu()]], ["faces"], ("key", F))
        assert ref[:, pos.cpu()].abs().max() > 0
        grads.append(g[:, pos])
        del g, fv, faces
    # the same real faces at the same pixels: both key widths give the same gradient up to the atomics' order
    assert rel_err(grads[0].cpu().numpy(), grads[1].cpu().numpy()) <= 1e-5


def _sphere_tiles(S, sigma, seed):
    """(faces [2,5000,3,3], the pixel mask [2,S,S] of three tiles per item, as _bench_tiles chooses them)"""
    from neural_renderer_b200 import synthetic
    faces = torch.from_numpy(synthetic.sphere_faces(2, 5000)).to(DEV)
    tiles, _ = tss._bench_tiles(faces, S, sigma, seed)
    pix = torch.stack([tss._tile_pixels(S, tiles[b]).reshape(-1) for b in range(2)])
    mask = torch.zeros(2, S * S, dtype=torch.bool, device=DEV).scatter_(1, pix, True).reshape(2, S, S)
    return faces, mask


def _masked(frag, mask):
    return frag._replace(pix_to_face=torch.where(mask[..., None], frag.pix_to_face,
                                                 torch.full_like(frag.pix_to_face, -1)))


@pytest.mark.parametrize("K", [8, 32])
def test_sphere_benchmark_geometry_backward(K):
    nr = _nr()
    S, sigma = 256, 1e-4
    faces, mask = _sphere_tiles(S, sigma, K)
    fv = faces.clone().requires_grad_(True)
    frag = nr.rasterize_soft_fragments(fv, S, sigma, K)
    ups = _upstream(frag, "all", 50 + K, mask)
    g = _kernel_grad(fv, frag, ups)
    ref = _oracle_grads(faces, _masked(frag, mask), S, ups)
    tss.check_grads([g], [ref], ["faces"], ("spheres", K))
    assert torch.all(g[~_used(_masked(frag, mask).pix_to_face, faces.shape[1])] == 0)


def test_teapot_through_indexed_vertices_backward():
    nr = _nr()
    v, f = _teapot()
    r = nr.Renderer()
    r.eye = nr.get_points_from_angles(2.732, 30, -15)
    verts = r._transform(v).float().contiguous()
    idx = f[0].contiguous()
    S, sigma, K = 128, 1e-4, 8
    vv = verts.clone().requires_grad_(True)
    frag = nr.rasterize_soft_fragments(idx, S, sigma, K, vertices=vv)
    assert (frag.pix_to_face >= 0).sum().item() > 20000
    # faces whose fragments lie in several tiles (and every vertex of the mesh is shared by several faces)
    per_face = torch.bincount(tile_face_keys(frag.pix_to_face) % idx.shape[0], minlength=idx.shape[0])
    assert (per_face >= 2).sum().item() > 100
    ups = _upstream(frag, "all", 60)
    g = _kernel_grad(vv, frag, ups)
    fo = verts.double().requires_grad_(True)
    zb, by, ds = ofrag.evaluate(osoft.gather_faces(fo, idx), frag.pix_to_face, S)
    (ref,) = torch.autograd.grad(sum((o * u.double()).sum() for o, u in zip((zb, by, ds), ups)), fo)
    _check_small(g, ref)


# ------------------------------------------------------------------------------------------------ 4. interpolation groups
_FRAGS = {}


def _interp_scene(name, K):
    """(Fragments, F) of the interpolation scenes, cached per (scene, K).  H W is odd, so the backward's groups of 32
    pixels straddle two items and the last one ends short.  'quad': three faces larger than the image at three depths in
    front of a soup (so slots 0-2 show the same face at every pixel of every item, the last pixels of item b and the
    first of item b + 1 included), at 37 x 37, B 3."""
    key = (name, K)
    if key not in _FRAGS:
        from neural_renderer_b200 import synthetic
        nr = _nr()
        if name in ("soup37", "soup45"):
            S, B = (37, 2) if name == "soup37" else (45, 3)
            faces = torch.from_numpy(synthetic.triangle_soup(B, 40, seed=S, size=(0.02, 0.4))).to(DEV)
        else:
            S, B = 37, 3
            soup = torch.from_numpy(synthetic.triangle_soup(B, 30, seed=5, size=(0.02, 0.4))).to(DEV)
            # nearer than every soup face (z in [1, 3]), each one nearer than the next at every vertex
            big = torch.tensor([[[-1.5, -1.5, z], [4.0, -1.5, z + 0.05], [-1.5, 4.0, z + 0.1]] for z in (0.4, 0.6, 0.8)],
                               device=DEV)
            faces = torch.cat((big[None].expand(B, -1, -1, -1), soup), 1).contiguous()
        frag = nr.rasterize_soft_fragments(faces, S, 1e-3, K)
        if len(_FRAGS) > 8:
            _FRAGS.clear()
        _FRAGS[key] = (frag, faces.shape[1])
    return _FRAGS[key]


def _straddles(p2f, k):
    """groups of 32 flattened pixels that hold the last pixels of one item and the first of the next, with the same face
    at slot k on both sides of the boundary"""
    B, H, W, K = p2f.shape
    n = 0
    for b in range(1, B):
        q = b * H * W
        if q % 32 and p2f[b - 1, -1, -1, k] >= 0 and p2f[b - 1, -1, -1, k] == p2f[b, 0, 0, k]:
            n += 1
    return n


def _interp_check(frag, F, form, K, C, seed, g_mask=None):
    B = frag.pix_to_face.shape[0]
    kw, _ = tsi._attributes(form, B, F, C, seed)
    g_out = _rand((*frag.pix_to_face.shape, C), seed + 1)
    if g_mask is not None:
        g_out = g_out * g_mask[..., None, None]
    out, gb, ga = tsi._run(frag, g_out, **kw)
    by = frag.bary_coords.double().requires_grad_(True)
    name = "face_attributes" if "face_attributes" in kw else "vertex_attributes"
    at = kw[name].double().requires_grad_(True)
    if form[0]:
        corners = tsi._gather(at if at.dim() == 3 else at[None], kw["faces"] if kw["faces"].dim() == 3 else kw["faces"][None])
    else:
        corners = at if at.dim() == 4 else at[None]
    ref = tsi._reference(frag._replace(bary_coords=by), corners)
    rb, ra = torch.autograd.grad(ref, (by, at), g_out.double())
    eb, ea = elem_err(gb.cpu(), rb.cpu(), floor=1e-3), elem_err(ga.cpu(), ra.cpu(), floor=1e-3)
    assert eb <= 1e-4, (form, eb)
    assert ea <= 5e-4, (form, ea)
    assert torch.all(gb[frag.pix_to_face < 0] == 0)
    return ea


@pytest.mark.parametrize("C", [3, 33])
@pytest.mark.parametrize("K", [1, 3, 8, 32])
@pytest.mark.parametrize("scene", ["soup37", "soup45", "quad"])
def test_interpolation_groups_straddle_items_and_end_short(scene, K, C):
    frag, F = _interp_scene(scene, K)
    B, H, W, _ = frag.pix_to_face.shape
    assert (H * W) % 32 != 0 and (B * H * W) % 32 != 0
    if scene == "quad":
        assert _straddles(frag.pix_to_face, 0) == B - 1
        if K >= 3:
            assert _straddles(frag.pix_to_face, 2) == B - 1
    for i, form in enumerate(tsi.FORMS):
        _interp_check(frag, F, form, K, C, 1000 * K + 10 * C + i)


@pytest.mark.parametrize("scene,K,C", [("teapot", 8, 33), ("spheres", 32, 4)])
def test_interpolation_long_runs(scene, K, C):
    frag, F = tsi._scene(scene, K)
    # runs: consecutive pixels in B H W order whose slot 0 shows the same face of the same item
    B = frag.pix_to_face.shape[0]
    p = frag.pix_to_face[..., 0].reshape(B, -1)
    key = torch.where(p >= 0, torch.arange(B, device=DEV)[:, None] * F + p, torch.full_like(p, -1)).reshape(-1)
    vals, lens = torch.unique_consecutive(key, return_counts=True)
    lens = lens[vals >= 0]
    print(scene, "slot-0 runs: longest", lens.max().item(), "mean", lens.float().mean().item())
    longest, n_runs = {"teapot": (3, 100), "spheres": (4, 1000)}[scene]   # runs of 2 and more, about 270 at the teapot
    assert lens.max().item() >= longest and (lens >= 2).sum().item() > n_runs
    for i, form in enumerate(tsi.FORMS):
        _interp_check(frag, F, form, K, C, 2000 + 10 * K + i)


# ------------------------------------------------------------------------------------------------ 5. the whole pipeline
@pytest.mark.parametrize("K", [8, 32])
def test_whole_pipeline_at_the_benchmark_shapes(K):
    nr = _nr()
    S, sigma, gamma, C = 256, 1e-4, 1e-4, 3
    bg = (0.2, 0.5, 0.8)
    faces, mask = _sphere_tiles(S, sigma, 70 + K)
    B, F = faces.shape[:2]
    ca = _rand((B, F, 3, C), 71, 0.0, 1.0)
    fv, cv = faces.clone().requires_grad_(True), ca.clone().requires_grad_(True)
    frag = nr.rasterize_soft_fragments(fv, S, sigma, K)
    img, alpha = nr.blend_soft_fragments(frag, nr.interpolate_soft_fragments(frag, cv), sigma, gamma, NEAR, FAR,
                                         background=bg)
    up = _rand((B, C, S, S), 72) * mask[:, None]
    ua = _rand((B, S, S), 73) * mask
    gf, gc = torch.autograd.grad((img, alpha), (fv, cv), (up, ua))
    p2f = _masked(frag, mask).pix_to_face
    f64, c64 = faces.double().requires_grad_(True), ca.double().requires_grad_(True)
    zb, by, ds = ofrag.evaluate(f64, p2f, S)
    col = tsi._reference(frag._replace(pix_to_face=p2f, bary_coords=by), c64)
    ri, ra = oblend.blend(p2f, zb, ds, col, sigma, gamma, NEAR, FAR, list(bg))
    rf, rc = torch.autograd.grad((ri, ra), (f64, c64), (up.double(), ua.double()))
    tss.check_grads([gf, gc], [rf, rc], ["faces", "colors"], ("pipeline", K))
    assert (frag.pix_to_face[mask] >= 0).sum(-1).eq(K).any()                 # full pixels among the chosen ones
