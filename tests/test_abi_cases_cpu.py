"""CPU: the covering array of the C-ABI matrix (tests/abi_cases.py) -- every compatible pair of levels appears, the full
product of texture kind x fill_back x anti-aliasing x backward mode is there, the conjunctions the pairs do not force are
reached (the side fill's tail, the light and corner-light gradients, the own-depth reload of the corner-light cube
gradient, every phase of the face_uvs reduction, texture staging and its overflow), and every case passes the library's
host argument checks (forward and backward called with a NULL workspace, so the call stops at the workspace check before
touching a device; the interpolation, which has no workspace, only with arguments it rejects before any launch)."""
import ctypes
import itertools

import numpy as np
import pytest

import abi_cases

NR_ERR_INVALID_ARG, NR_ERR_WORKSPACE = -1, -2  # include/nr_b200.h


@pytest.fixture(scope="module")
def lib():
    from neural_renderer_b200 import build, _lib
    build.build_library()
    return _lib.load()


def test_generator_is_deterministic():
    assert abi_cases.cases() == abi_cases.cases()


def test_every_pair_of_levels_appears():
    cases = abi_cases.cases()
    covered = set().union(*(abi_cases.pairs_of(c) for c in cases))
    missing = abi_cases.required_pairs() - covered
    assert not missing, sorted(missing, key=repr)[:10]
    # every level of every dimension is reachable, and the rules exclude nothing else
    for name, levels in abi_cases.DIMS:
        assert {c[name] for c in cases if c[name] is not None} == set(levels), name
    assert len(cases) <= 180


def test_full_product_of_the_fused_paths():
    got = {(c["kind"], c["fill_back"], c["raster"] == "aa", c["backward"]) for c in abi_cases.cases()}
    want = set(itertools.product(abi_cases.LEVELS["kind"], (False, True), (False, True), abi_cases.LEVELS["backward"]))
    assert want <= got


def test_side_fill_tail_is_reached():
    """a case where the edge scan zero-fills grad_textures on the side and the float count leaves a scalar tail"""
    import abi_harness
    for c in abi_cases.cases():
        p = abi_harness.Plan(c)
        if p.kind in ("cube", "cube_shared") and c["backward"] == "one" and p.g_rgb and c["pointers"] == "fresh":
            n = int(np.prod(p.bufs["grad_textures"][0]))
            if n % 4:
                return
    raise AssertionError("no case reaches the tail of the side fill")


def test_light_gradient_is_held_to_the_oracle():
    """grad_face_light (lit, optional pointers given, rgb upstream gradient) for every texture kind, in fresh and
    accumulating, one-call and two-half backward passes, with and without fill_back and anti-aliasing"""
    import abi_harness
    seen = {}
    for c in abi_cases.cases():
        p = abi_harness.Plan(c)
        if "grad_face_light" in p.bufs and p.g_rgb:
            s = seen.setdefault(p.kind, set())
            s |= {("acc", p.accumulate), ("halves", len(p.backward_calls()) == 2), ("fill_back", p.fill_back),
                  ("aa", p.aa)}
    want = {(k, v) for k in ("acc", "halves", "fill_back", "aa") for v in (False, True)}
    for kind in ("cube", "cube_shared", "uv", "mip"):
        assert seen.get(kind, set()) >= want, (kind, want - seen.get(kind, set()))


def test_corner_light_gradient_is_held_to_the_oracle():
    """grad_corner_light (smooth shading, optional pointers given, rgb upstream gradient) for every texture kind, in fresh
    and accumulating, one-call and two-half backward passes, with and without fill_back and anti-aliasing"""
    import abi_harness
    seen = {}
    for c in abi_cases.cases():
        p = abi_harness.Plan(c)
        if "grad_corner_light" in p.bufs and p.g_rgb:
            s = seen.setdefault(p.kind, set())
            s |= {("acc", p.accumulate), ("halves", len(p.backward_calls()) == 2), ("fill_back", p.fill_back),
                  ("aa", p.aa)}
    want = {(k, v) for k in ("acc", "halves", "fill_back", "aa") for v in (False, True)}
    for kind in ("cube", "cube_shared", "uv", "mip"):
        assert seen.get(kind, set()) >= want, (kind, want - seen.get(kind, set()))


def test_corner_light_own_depth_reload_is_reached():
    """the cube texture gradient with corner light, NR_TEX_Z_BATCH0 and indexed geometry reloads every item's own depths
    (items other than 0 need it): for per-item and shared cubes"""
    import abi_harness
    kinds = set()
    for c in abi_cases.cases():
        p = abi_harness.Plan(c)
        if p.corner and c["z_batch0"] and p.B > 1 and p.indexed and p.g_rgb and "grad_corner_light" in p.bufs:
            kinds.add(p.kind)
    assert {"cube", "cube_shared"} <= kinds, kinds


def test_every_phase_of_the_face_uvs_reduction_is_reached():
    """red_add_6 picks its vector pattern from the phase of a face's 6 floats (address / 4 mod 4): every phase of
    grad_face_uvs, for both samplers, with and without corner light"""
    import abi_harness
    seen = {}
    for c in abi_cases.cases():
        p = abi_harness.Plan(c)
        if "grad_face_uvs" in p.bufs and p.g_rgb:
            shape = p.bufs["grad_face_uvs"][0]
            n_faces = int(np.prod(shape[:-2]))  # every item's faces, one after the other
            phases = {(p.offsets["grad_face_uvs"] // 4 + 6 * f) % 4 for f in range(n_faces)}
            seen.setdefault((p.kind, p.corner), set()).update(phases)
    for key in itertools.product(("uv", "mip"), (False, True)):
        assert seen.get(key, set()) == {0, 1, 2, 3}, (key, seen.get(key))


def test_texture_staging_runs_and_overflows():
    """NR_FWD_STAGE_TEXTURES really stages (the predicate of nr_b200_forward) in cases with per-item and shared cubes and
    with face light, and one case has a pixel row (one row segment of the staged resolve) with more runs of distinct
    cubes than there are slots, counted on the CPU oracle's face_index_map as the kernel counts them"""
    import abi_harness
    import nr_oracle
    staged, overflow = set(), False
    for c in abi_cases.cases():
        p = abi_harness.Plan(c)
        on, nslots = abi_harness.stage_runs(p)
        if not on:
            continue
        staged |= {p.kind, "lit" if p.lit else "unlit", p.ts}
        if overflow or p.ts != 6:
            continue
        d = abi_harness.make_inputs(p, c["id"])
        fn = nr_oracle.rasterize_rgbad(d["faces_mat"], None, p.S, False, abi_harness.NEAR, abi_harness.FAR,
                                       abi_harness.EPS, return_rgb=False, return_alpha=True, return_depth=False).fn
        fim = fn.face_index_map  # raster rows, as the staged resolve reads its z-buffer
        cube = np.where(fim >= p.F_front, fim - p.F_front, fim) if p.fill_back else fim
        bx = 256 if p.S >= 256 else (p.S + 31) // 32 * 32
        for b in range(p.B):
            for yi in range(p.S):
                for x0 in range(0, p.S, bx):
                    seg = cube[b, yi, x0:x0 + bx]
                    heads = sum(1 for i, f in enumerate(seg) if f >= 0 and (i % 32 == 0 or seg[i - 1] != f))
                    overflow |= heads > nslots
    assert {"cube", "cube_shared", "lit", "unlit", 2, 4, 6} <= staged, staged
    assert overflow, "no staged case has more runs in a row segment than slots"


def test_cases_hold_the_rules():
    for c in abi_cases.cases():
        assert abi_cases.compatible(c), c
        for name, _ in abi_cases.DIMS:
            assert (c[name] is not None) == abi_cases.active(name, c["kind"]), (name, c)


def test_every_case_passes_the_host_argument_checks(lib):
    import abi_harness
    n_offset = n_short = n_corner = n_attr = 0
    for c in abi_cases.cases():
        plan = abi_harness.Plan(c)
        ptr = plan.fake_pointers()
        n_offset += any(v % 16 for v in ptr.values())
        n_short += plan.short
        a = plan.forward_args(ptr, None, 0)
        assert lib.nr_b200_forward(ctypes.byref(a), None) == NR_ERR_WORKSPACE, abi_cases.case_id(c)
        for flags in plan.backward_calls():
            b = plan.backward_args(ptr, flags, None, 0)
            assert plan.call_backward(lib, b, ptr, None) == NR_ERR_WORKSPACE, (abi_cases.case_id(c), hex(flags))
            n_corner += plan.corner
        # a required pointer left out is rejected before the workspace is looked at
        for k in ("face_index_map", "rgb_map" if plan.rgb else "weight_map"):
            bad = dict(ptr)
            bad.pop(k)
            a = plan.forward_args(bad, None, 0)
            assert lib.nr_b200_forward(ctypes.byref(a), None) == NR_ERR_INVALID_ARG, (k, abi_cases.case_id(c))
        # the interpolation has no workspace gate: a valid call would launch, so only calls it rejects before any launch
        if plan.attr:
            n_attr += 1
            for backward in (False, True):
                a = plan.interpolate_args(ptr, backward)
                a.channels = 0
                fn = lib.nr_b200_interpolate_backward if backward else lib.nr_b200_interpolate
                assert fn(ctypes.byref(a), None) == NR_ERR_INVALID_ARG, abi_cases.case_id(c)
            if plan.indexed:
                a = plan.interpolate_args(ptr, True)
                a.grad_faces = 0x7000000
                assert lib.nr_b200_interpolate_backward(ctypes.byref(a), None) == NR_ERR_INVALID_ARG, abi_cases.case_id(c)
    assert n_offset >= 60 and n_short >= 15 and n_corner >= 20 and n_attr >= 40, (n_offset, n_short, n_corner, n_attr)
