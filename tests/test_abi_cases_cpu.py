"""CPU: the covering array of the C-ABI matrix (tests/abi_cases.py) -- every compatible pair of levels appears, the full
product of texture kind x fill_back x anti-aliasing x backward mode is there, and every case passes the library's host
argument checks (called with a NULL workspace, so the call stops at the workspace check before touching a device)."""
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
    assert len(cases) <= 130


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


def test_cases_hold_the_rules():
    for c in abi_cases.cases():
        assert abi_cases.compatible(c), c
        for name, _ in abi_cases.DIMS:
            assert (c[name] is not None) == abi_cases.active(name, c["kind"]), (name, c)


def test_every_case_passes_the_host_argument_checks(lib):
    import abi_harness
    n_offset = 0
    for c in abi_cases.cases():
        plan = abi_harness.Plan(c)
        ptr = plan.fake_pointers()
        n_offset += any(v % 16 for v in ptr.values())
        a = plan.forward_args(ptr, None, 0)
        assert lib.nr_b200_forward(ctypes.byref(a), None) == NR_ERR_WORKSPACE, abi_cases.case_id(c)
        for flags in plan.backward_calls():
            b = plan.backward_args(ptr, flags, None, 0)
            assert lib.nr_b200_backward(ctypes.byref(b), None) == NR_ERR_WORKSPACE, (abi_cases.case_id(c), hex(flags))
        # a required pointer left out is rejected before the workspace is looked at
        for k in ("face_index_map", "rgb_map" if plan.rgb else "weight_map"):
            bad = dict(ptr)
            bad.pop(k)
            a = plan.forward_args(bad, None, 0)
            assert lib.nr_b200_forward(ctypes.byref(a), None) == NR_ERR_INVALID_ARG, (k, abi_cases.case_id(c))
    assert n_offset >= 60
