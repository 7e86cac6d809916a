"""CPU: the covering array of the C-ABI matrix (tests/abi_cases.py) -- every compatible pair of levels appears, the full
product of texture kind x fill_back x anti-aliasing x backward mode is there, the conjunctions the pairs do not force are
reached (the side fill's tail, the light and corner-light gradients, the own-depth reload of the corner-light cube
gradient, every phase of the face_uvs reduction, texture staging and its overflow, the interior vertex gradient, the
Phong rows, the normal-map and specular-map rows), the cases from before the interior gradient, before the Phong modes
and before the maps joined are unchanged, and every case passes the library's host argument checks
(forward and backward called with a NULL workspace, so the call stops at the workspace check before touching a device;
the interpolation, which has no workspace, only with arguments it rejects before any launch)."""
import ctypes
import hashlib
import itertools

import numpy as np
import pytest

import abi_cases

NR_ERR_INVALID_ARG, NR_ERR_WORKSPACE, NR_ERR_UNSUPPORTED = -1, -2, -4  # include/nr_b200.h


@pytest.fixture(scope="module")
def lib():
    from neural_renderer_b200 import build, _lib
    build.build_library()
    return _lib.load()


def test_generator_is_deterministic():
    assert abi_cases.cases() == abi_cases.cases()


def test_cases_before_the_interior_gradient_are_frozen():
    """the 177 cases the matrix held before the interior gradient joined it keep their ids, levels and seeded inputs:
    without the `interior` key (always "off" there) and the Phong and map dimensions (None there) they hash to the list
    as it was"""
    old = [{k: v for k, v in c.items() if k != "interior" and k not in abi_cases.PHONG_DIMS + abi_cases.MAP_DIMS}
           for c in abi_cases.cases()[:177]]
    assert all(c["interior"] in (None, "off") for c in abi_cases.cases()[:177])
    assert hashlib.sha256(repr(old).encode()).hexdigest() == \
        "cde6f0825f0973a0dfd6be5efe813401024db41c1de100869a3a5c23bd7ed758"


def test_cases_before_the_phong_modes_are_frozen():
    """the 194 cases the matrix held before the Phong modes joined it keep their ids, levels and seeded inputs: without
    the Phong and map dimensions (None there) they hash to the list as it was"""
    cases = abi_cases.cases()[:194]
    assert all(c["light"] not in abi_cases.PHONG for c in cases)
    assert all(c[k] is None for c in cases for k in abi_cases.PHONG_DIMS + abi_cases.MAP_DIMS)
    old = [{k: v for k, v in c.items() if k not in abi_cases.PHONG_DIMS + abi_cases.MAP_DIMS} for c in cases]
    assert hashlib.sha256(repr(old).encode()).hexdigest() == \
        "a9d5ed5efe4abf6c0a8db1a19b93cdcc1de0f2be5b19492bd510d0d0178775ea"


def test_cases_before_the_maps_are_frozen():
    """the 271 cases the matrix held before the normal map and the specular map joined it keep their ids, levels and
    seeded inputs: they carry no map and go through the entry point they went through (maps "off" or None, map_entry
    "direct" or None, the other map dimensions None), and without the map dimensions they hash to the list as it was"""
    cases = abi_cases.cases()[:271]
    assert all(c["maps"] in (None, "off") and c["map_entry"] in (None, "direct") for c in cases)
    assert all(c[k] is None for c in cases for k in abi_cases.MAP_DIMS[2:])
    old = [{k: v for k, v in c.items() if k not in abi_cases.MAP_DIMS} for c in cases]
    assert hashlib.sha256(repr(old).encode()).hexdigest() == \
        "9928714d97dfdbff11151ce6d1a56e7cb6366f50d9553d1beebad80c6ad40eef"
    assert all(c["maps"] not in (None, "off") or c["map_entry"] != "direct" for c in abi_cases.cases()[271:351])  # the seeded rows


def test_every_pair_of_levels_appears():
    cases = abi_cases.cases()
    covered = set().union(*(abi_cases.pairs_of(c) for c in cases))
    missing = abi_cases.required_pairs() - covered
    assert not missing, sorted(missing, key=repr)[:10]
    # every level of every dimension is reachable, and the rules exclude nothing else
    for name, levels in abi_cases.DIMS:
        assert {c[name] for c in cases if c[name] is not None} == set(levels), name
    # 194 cases before the Phong modes, 77 Phong rows, 80 map rows seeded for conjunctions the pairs do not force and 26
    # more for the pairs; the cap keeps the matrix's run time in check (test_gpu_abi_matrix.py gives the measured time)
    assert len(cases) <= 385


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


def test_interior_gradient_is_held_to_the_oracle():
    """NR_GRAD_INTERIOR with an rgb upstream gradient, for every texture kind: every light, fresh and accumulating,
    one-call and two-half backward passes, with and without fill_back and anti-aliasing; and over all interior cases
    every geometry (per-item and shared index sets, out-of-range indices), every batch level, the odd cube sizes and a
    one-texel-high image for both samplers"""
    import abi_harness
    seen, every = {}, set()
    for c in abi_cases.cases():
        p = abi_harness.Plan(c)
        if not p.interior:
            continue
        every |= {("geometry", c["geometry"]), ("batch", c["batch"]), ("ts", p.ts), ("one_texel", p.kind, p.Ht == 1)}
        if p.g_rgb:
            s = seen.setdefault(p.kind, set())
            s |= {("light", c["light"]), ("acc", p.accumulate), ("halves", len(p.backward_calls()) == 2),
                  ("fill_back", p.fill_back), ("aa", p.aa)}
    want = {(k, v) for k in ("acc", "halves", "fill_back", "aa") for v in (False, True)}
    want |= {("light", v) for v in abi_cases.OLD_LIGHTS}  # the Phong modes refuse the interior gradient
    for kind in ("cube", "cube_shared", "uv", "mip"):
        assert seen.get(kind, set()) >= want, (kind, want - seen.get(kind, set()))
    want_every = {("geometry", v) for v in abi_cases.LEVELS["geometry"]} | {("batch", v) for v in abi_cases.LEVELS["batch"]}
    want_every |= {("ts", 3), ("ts", 5), ("ts", 6), ("one_texel", "uv", True), ("one_texel", "mip", True)}
    assert every >= want_every, want_every - every


def test_interior_gradient_next_to_other_outputs_is_reached():
    """interior cases at three items with per-item index sets and with per-item face and corner light (the scatter and
    the light reads address item b), z_batch0 cubes at B = 1 and z_batch0 images at B = 3, the rgb + alpha edge scan
    and the depth gradient in the same call, and the flag without an rgb upstream gradient"""
    import abi_harness
    seen = set()
    for c in abi_cases.cases():
        p = abi_harness.Plan(c)
        if not p.interior:
            continue
        cube = p.kind in ("cube", "cube_shared")
        if p.g_rgb and p.B == 3:
            seen |= {k for k, on in (("idx_item_B3", c["geometry"] == "idx_item"), ("lit_B3", p.lit),
                                     ("corner_B3", p.corner)) if on}
        if c["z_batch0"] and p.g_rgb and p.B == (1 if cube else 3):
            seen.add("z0_cube_B1" if cube else "z0_image_B3")
        if p.g_rgb and p.g_alpha and p.g_depth:
            seen.add("rgb_alpha_depth")
        if not p.g_rgb:
            seen.add("no_rgb")
    assert seen >= {"idx_item_B3", "lit_B3", "corner_B3", "z0_cube_B1", "z0_image_B3", "rgb_alpha_depth", "no_rgb"}, seen


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
            assert (c[name] is not None) == abi_cases.active(name, c), (name, c)


def test_every_case_passes_the_host_argument_checks(lib):
    import abi_harness
    from neural_renderer_b200 import _lib as lib_flags
    n_offset = n_short = n_corner = n_attr = n_interior = n_phong = n_maps = 0
    for c in abi_cases.cases():
        plan = abi_harness.Plan(c)
        ptr = plan.fake_pointers()
        n_offset += any(v % 16 for v in ptr.values())
        n_short += plan.short
        a = plan.forward_args(ptr, None, 0)
        assert plan.call_forward(lib, a, ptr, None) == NR_ERR_WORKSPACE, abi_cases.case_id(c)
        for flags in plan.backward_calls():
            b = plan.backward_args(ptr, flags, None, 0)
            assert plan.call_backward(lib, b, ptr, None) == NR_ERR_WORKSPACE, (abi_cases.case_id(c), hex(flags))
            n_corner += plan.corner
            if plan.interior:
                # the interior gradient reads the textures: NULL textures are refused for the flag alone -- without the
                # other gradients that read them, the same call without the flag passes the host checks
                n_interior += 1
                I = lib_flags.NR_GRAD_INTERIOR
                bare = {k: v for k, v in ptr.items() if k not in ("grad_face_light", "grad_face_uvs", "grad_corner_light")}
                for fl, want in ((flags & ~I, NR_ERR_WORKSPACE), (flags, NR_ERR_INVALID_ARG)):
                    b = plan.backward_args(bare, fl, None, 0)
                    b.textures = None
                    assert plan.call_backward(lib, b, bare, None) == want, (abi_cases.case_id(c), hex(fl))
                # z_batch0 at three items: refused for cubes with the flag only; images ignore z_batch0
                cube = plan.kind in ("cube", "cube_shared")
                for fl, want in ((flags & ~I, NR_ERR_WORKSPACE), (flags, NR_ERR_INVALID_ARG if cube else NR_ERR_WORKSPACE)):
                    b = plan.backward_args(ptr, fl | lib_flags.NR_TEX_Z_BATCH0, None, 0)
                    b.batch_size = 3
                    assert plan.call_backward(lib, b, ptr, None) == want, (abi_cases.case_id(c), hex(fl))
        # a required pointer left out is rejected before the workspace is looked at
        for k in ("face_index_map", "rgb_map" if plan.rgb else "weight_map"):
            bad = dict(ptr)
            bad.pop(k)
            a = plan.forward_args(bad, None, 0)
            assert plan.call_forward(lib, a, bad, None) == NR_ERR_INVALID_ARG, (k, abi_cases.case_id(c))
        if plan.phong:  # the Phong inputs are required, and the interior gradient is refused with them
            n_phong += 1
            for k in ("corner_shading", "params") + (("lights",) if plan.NL else ()) + (("sh",) if plan.sh else ()):
                bad = dict(ptr)
                bad.pop(k)
                a = plan.forward_args(bad, None, 0)
                assert plan.call_forward(lib, a, bad, None) == NR_ERR_INVALID_ARG, (k, abi_cases.case_id(c))
            b = plan.backward_args(ptr, plan.backward_calls()[0] | lib_flags.NR_GRAD_INTERIOR, None, 0)
            assert plan.call_backward(lib, b, ptr, None) == NR_ERR_UNSUPPORTED, abi_cases.case_id(c)
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
        if plan.nm or plan.sm:
            n_maps += 1
            _map_rows_are_refused(lib, lib_flags, plan, ptr, abi_cases.case_id(c))
    assert n_offset >= 60 and n_short >= 15 and n_corner >= 20 and n_attr >= 40 and n_interior >= 17 and n_phong >= 70 \
        and n_maps >= 90, (n_offset, n_short, n_corner, n_attr, n_interior, n_phong, n_maps)


def _map_rows_are_refused(lib, lib_flags, plan, ptr, cid):
    """what the map entry points refuse before they look at the workspace (include/nr_b200.h): a missing map or tangent
    pointer, a specular map off its 16-byte alignment, a batch that is neither 1 nor B, an empty map, a map gradient
    without `textures`, and a map without NR_TEX_UV -- each next to the same call without the fault, which gets as far as
    the workspace check"""
    import abi_harness
    c = plan.case
    inputs = (("normal_map", "corner_tangents") if plan.nm else ()) + (("specular_map",) if plan.sm else ())
    for k in inputs:
        bad = dict(ptr)
        bad.pop(k)
        for call, args in ((plan.call_forward, plan.forward_args(bad, None, 0)),
                           (plan.call_backward, plan.backward_args(bad, plan.backward_calls()[0], None, 0))):
            assert call(lib, args, bad, None) == NR_ERR_INVALID_ARG, (k, cid)
    if plan.sm:
        bad = {**ptr, "specular_map": ptr["specular_map"] + 4}
        assert plan.call_forward(lib, plan.forward_args(bad, None, 0), bad, None) == NR_ERR_INVALID_ARG, cid
    # three items: 1 and 3 are batches, 2 is not; and a map has at least one row
    faults = ([("Bm", 2), ("Bt", 2), ("Hm", 0)] if plan.nm else []) + ([("Bq", 2), ("Hq", 0)] if plan.sm else [])
    for field, value in [(None, None)] + faults:
        p2 = abi_harness.Plan(c)
        if field:
            setattr(p2, field, value)
        a = p2.forward_args(ptr, None, 0)
        a.batch_size = 3
        assert p2.call_forward(lib, a, ptr, None) == (NR_ERR_INVALID_ARG if field else NR_ERR_WORKSPACE), (field, cid)
    # a map gradient reads the unlit sample: refused without `textures`, which may be NULL when no such gradient is wanted
    bare = {k: v for k, v in ptr.items() if not (k.startswith("grad_") and k[5:] in
            ("corner_shading", "params", "lights", "sh", "face_uvs", "face_light") + inputs)}
    for k in (None,) + tuple("grad_" + k for k in inputs if "grad_" + k in plan.bufs):
        some = {**bare, **({k: ptr[k]} if k else {})}
        b = plan.backward_args(some, plan.backward_calls()[0], None, 0)
        b.textures = None
        assert plan.call_backward(lib, b, some, None) == (NR_ERR_INVALID_ARG if k else NR_ERR_WORKSPACE), (k, cid)
    # the maps are addressed by the UVs of a texture image: refused next to texture cubes, which the same call without
    # the maps may use
    for with_maps in (False, True):
        p2 = abi_harness.Plan(c)
        if not with_maps:
            p2.nm = p2.sm = False
        a = p2.forward_args(ptr, None, 0)
        a.flags &= ~(lib_flags.NR_TEX_UV | lib_flags.NR_TEX_MIPMAP | lib_flags.NR_UV_SHARED)
        a.texture_size = 4
        assert p2.call_forward(lib, a, ptr, None) == (NR_ERR_INVALID_ARG if with_maps else NR_ERR_WORKSPACE), (with_maps, cid)


def _phong_grads_run(p):
    """whether the case's backward runs k_phong_grad: Phong, every shading gradient given, an rgb upstream gradient (the
    texture half runs in every backward mode)"""
    return p.phong and p.given and p.g_rgb


def _variant(p):
    """the k_phong_grad instantiation of a Phong case: (kTex, kIdx, light variant)"""
    tex = {"cube": 0, "cube_shared": 0, "uv": 1, "mip": 2}[p.kind]
    var = {"phong": "none", "phong_set": "set"}.get(p.case["light"]) or ("sh_set" if p.NL else "sh_alone")
    return tex, p.indexed, var


def test_phong_gradients_are_held_to_the_oracle():
    """every Phong mode x every texture kind with every shading gradient and an rgb upstream gradient: fresh and
    accumulating, one call and two halves in both orders, with and without fill_back and anti-aliasing; every
    k_phong_grad<kTex, kIdx, kLights, kSH> instantiation (SH without a set and with one apart); NL = 8 for every kind;
    every entry point of every mode"""
    import abi_harness
    seen, variants, full_set, entries = {}, set(), set(), set()
    for c in abi_cases.cases():
        p = abi_harness.Plan(c)
        if not p.phong:
            continue
        entries.add((c["light"], p.entry))
        if not _phong_grads_run(p):
            continue
        s = seen.setdefault((c["light"], p.kind), set())
        s |= {("acc", p.accumulate), ("halves", len(p.backward_calls()) == 2), ("fill_back", p.fill_back), ("aa", p.aa),
              ("order", c["backward"])}
        variants.add(_variant(p))
        if p.NL == 8:
            full_set.add(p.kind)
    want = {(k, v) for k in ("acc", "halves", "fill_back", "aa") for v in (False, True)}
    want |= {("order", "faces_tex"), ("order", "acc_halves")}  # two halves, faces first and textures first
    for key in itertools.product(abi_cases.PHONG, ("cube", "cube_shared", "uv", "mip")):
        assert seen.get(key, set()) >= want, (key, want - seen.get(key, set()))
    want_v = set(itertools.product((0, 1, 2), (False, True), ("none", "set", "sh_alone", "sh_set")))
    assert variants == want_v, want_v - variants
    assert full_set == {"cube", "cube_shared", "uv", "mip"}, full_set
    assert entries == {("phong", "own"), ("phong", "via_sh"), ("phong", "via_lights_nl0"), ("phong_set", "own"),
                       ("phong_set", "via_sh"), ("phong_sh", "sh")}, entries


def test_phong_rows_next_to_other_flags_are_reached():
    """cube Phong with NR_TEX_Z_BATCH0 at three items on per-item index sets (every mode); the short layouts under every
    mode; every shading gradient without an rgb upstream gradient, fresh and accumulating, under every mode (a light
    set's grad_lights included); Bc = Bp = Bl = Bs = 1 and all = B at three items; shared textures / UVs at three items"""
    import abi_harness
    seen = set()
    for c in abi_cases.cases():
        p = abi_harness.Plan(c)
        if not p.phong:
            continue
        mode = c["light"]
        cube = p.kind in ("cube", "cube_shared")
        if cube and c["z_batch0"] and p.B == 3 and c["geometry"] == "idx_item" and _phong_grads_run(p):
            seen.add(("z0", mode))
        if p.short and p.given and p.g_rgb:
            seen.add(("short", mode))
        if p.given and not p.g_rgb and (p.g_alpha or p.g_depth) and (mode == "phong" or "grad_lights" in p.bufs):
            seen.add(("no_rgb", mode, p.accumulate))
        if p.B == 3 and p.sh and p.NL and _phong_grads_run(p):
            batches = {p.Bc, p.Bp, p.Bl, p.Bs}
            if len(batches) == 1:
                seen.add(("batches", batches.pop()))
        if p.B == 3 and _phong_grads_run(p) and ((p.flags & abi_harness._lib().NR_TEX_SHARED) or p.uv_shared):
            seen.add(("shared_tex", mode))
    want = {("z0", m) for m in abi_cases.PHONG} | {("short", m) for m in abi_cases.PHONG}
    want |= {("no_rgb", m, acc) for m in abi_cases.PHONG for acc in (False, True)}
    want |= {("batches", 1), ("batches", 3)} | {("shared_tex", m) for m in abi_cases.PHONG}
    assert seen >= want, want - seen


def _map_variant(p):
    """the k_phong_grad instantiation of a map row: (kTex, kIdx, light variant, kNM, kSM)"""
    return _variant(p) + (p.nm, p.sm)


def test_map_gradients_are_held_to_the_oracle():
    """every k_phong_grad<kTex, kIdx, kLights, kSH, kNM, kSM> instantiation with a map (48: both image samplers, per-face
    and indexed geometry, Phong alone / a set / SH without a set / SH with one, a normal map, a specular map or both)
    reached with every gradient and an rgb upstream gradient; for each of nm, sm, nm_sm and each sampler a fresh and an
    accumulating backward, one call and two halves in both orders, with and without fill_back and anti-aliasing; every
    entry point a maps level can travel through"""
    import abi_harness
    seen, variants, entries = {}, set(), set()
    for c in abi_cases.cases():
        p = abi_harness.Plan(c)
        if c["maps"] is None:
            continue
        entries.add((c["maps"], p.map_entry))
        if not (p.nm or p.sm) or not (_phong_grads_run(p) and c["map_grads"] == "all" and p.uv_grad):
            continue
        s = seen.setdefault((c["maps"], p.kind), set())
        s |= {("acc", p.accumulate), ("halves", len(p.backward_calls()) == 2), ("fill_back", p.fill_back), ("aa", p.aa),
              ("order", c["backward"])}
        variants.add(_map_variant(p))
    want = {(k, v) for k in ("acc", "halves", "fill_back", "aa") for v in (False, True)}
    want |= {("order", "faces_tex"), ("order", "tex_faces"), ("order", "acc_halves")}
    for key in itertools.product(("nm", "sm", "nm_sm"), ("uv", "mip")):
        assert seen.get(key, set()) >= want, (key, want - seen.get(key, set()))
    want_v = {(t, i, v, nm, sm) for t, i, v in itertools.product((1, 2), (False, True), ("none", "set", "sh_alone", "sh_set"))
              for nm, sm in ((True, False), (False, True), (True, True))}
    assert len(want_v) == 48 and variants == want_v, want_v - variants
    assert entries == {("off", "direct"), ("off", "via_nm"), ("off", "via_sm"), ("nm", "direct"), ("nm", "via_sm"),
                       ("sm", "direct"), ("nm_sm", "direct")}, entries


def test_map_rows_next_to_other_flags_are_reached():
    """the conjunctions of the map rows that the pairs do not force: NL = 8 with both maps for both samplers; the maps'
    UV term alone (grad_face_uvs wanted, every shading and map gradient NULL) for each maps level and sampler, the
    texels alone, and grad_corner_tangents without grad_corner_shading; shared UVs at three items with fill_back, next to
    a shared and a per-item image; the map batches against the shading batches at three items; grad_normal_map 0, 4 and
    8 bytes and grad_specular_map 0, 4, 8 and 12 bytes past a 16-byte boundary, each with a one-texel-wide and a wider
    map, and specular_map itself always aligned; the short layouts; no rgb upstream gradient, fresh and accumulating;
    NR_TEX_Z_BATCH0 on per-item index sets; NULL map structs under every earlier mode; out-of-range indices"""
    import abi_harness
    L = abi_harness._lib()
    seen = set()
    for c in abi_cases.cases():
        p = abi_harness.Plan(c)
        if c["maps"] is None:
            continue
        maps, mode = c["maps"], c["light"]
        if not (p.nm or p.sm):
            if p.map_entry != "direct" and _phong_grads_run(p):
                seen.add(("null_structs", mode, p.map_entry))
            continue
        assert p.offsets.get("specular_map", 0) == 0
        every = _phong_grads_run(p) and c["map_grads"] == "all"
        if every and p.NL == 8 and maps == "nm_sm":
            seen.add(("nl8", p.kind))
        if p.g_rgb and not p.given and not any(k in p.bufs for k in abi_harness.MAP_GRADS):
            if p.uv_grad:
                seen.add(("uv_term_alone", maps, p.kind))
        if p.g_rgb and not p.given and not p.uv_grad and c["map_grads"] == "texels":
            seen.add(("texels_alone", maps))
        if p.g_rgb and not p.given and c["map_grads"] == "tangents":
            seen.add("tangents_without_shading")
        if every and p.uv_grad and p.B == 3 and p.fill_back and (p.flags & L.NR_UV_SHARED):
            seen.add(("shared_uvs", maps, bool(p.flags & L.NR_TEX_SHARED)))
        if every and p.B == 3 and maps == "nm_sm" and p.sh and p.NL:
            ours, theirs = {p.Bm, p.Bt, p.Bq}, {p.Bc, p.Bp, p.Bl, p.Bs}
            if len(ours) == 1 and len(theirs) == 1:
                seen.add(("batches", ours.pop(), theirs.pop()))
        if p.g_rgb:
            for k, wide in (("grad_normal_map", p.Wm > 1), ("grad_specular_map", p.Wq > 1)):
                if k in p.bufs:
                    seen.add((k, p.offsets[k], wide))
            if "grad_corner_tangents" in p.bufs:
                seen.add(("grad_corner_tangents", p.offsets["grad_corner_tangents"]))
        if p.short and every:
            seen.add(("short", maps))
        if p.given and c["map_grads"] == "all" and not p.g_rgb and maps == "nm_sm" and "grad_lights" in p.bufs:
            seen.add(("no_rgb", p.accumulate))
        if every and maps == "nm_sm" and c["z_batch0"] and p.B == 3 and c["geometry"] == "idx_item":
            seen.add("z0")
        if every and maps == "nm" and p.map_entry == "via_sm":
            seen.add("nm_via_sm")
        if every and maps == "nm_sm" and c["geometry"] == "idx_shared_oor":
            seen.add("oor")
    levels = ("nm", "sm", "nm_sm")
    want = {("nl8", k) for k in ("uv", "mip")} | {("uv_term_alone", m, k) for m in levels for k in ("uv", "mip")}
    want |= {("texels_alone", m) for m in levels} | {"tangents_without_shading"}
    want |= {("shared_uvs", "nm", True), ("shared_uvs", "sm", False)}
    want |= {("batches", 1, 3), ("batches", 3, 1), ("batches", 1, 1), ("batches", 3, 3)}
    want |= {("grad_normal_map", o, w) for o in (0, 4, 8) for w in (False, True)}
    want |= {("grad_specular_map", o, w) for o in (0, 4, 8, 12) for w in (False, True)}
    want |= {("grad_corner_tangents", o) for o in (0, 4, 8)}
    want |= {("short", m) for m in levels} | {("no_rgb", False), ("no_rgb", True), "z0", "nm_via_sm", "oor"}
    want |= {("null_structs", m, via) for m in abi_cases.PHONG for via in ("via_nm", "via_sm")}
    assert seen >= want, want - seen
