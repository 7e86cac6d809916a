"""Deterministic covering array over the flag dimensions of nr_b200_forward / nr_b200_backward (test infrastructure).

`cases()` returns the case list of tests/test_gpu_abi_matrix.py: the full product of texture kind x fill_back x
anti-aliasing x backward mode, with every other dimension filled in greedily so that every compatible pair of levels of
any two dimensions appears in at least one case; rows are added until no pair is missing.  No randomness: the same list
on every machine.

A level that has no meaning for a case (ts without texture cubes, image / UV sharing without a texture image) is None and
takes part in no pair.  Combinations the ABI rejects are never generated: texture kinds other than "none" always draw
RGB and "none" never does, light needs RGB; fill_back doubles the faces (F even) and anti-aliasing doubles the raster
(even) by construction of the geometry, so no case is skipped."""
import itertools

DIMS = [
    ("kind", ["none", "cube", "cube_shared", "uv", "mip"]),
    ("fill_back", [False, True]),
    ("raster", ["even", "odd", "aa"]),
    ("backward", ["one", "tex_faces", "faces_tex", "acc_one", "acc_halves"]),
    ("geometry", ["faces", "idx_item", "idx_shared", "idx_shared_oor"]),
    ("ts", [2, 3, 5]),
    ("image", ["item", "shared"]),
    ("uvs", ["item", "shared"]),
    ("light", [False, True]),
    ("bg", ["uniform", "per_batch"]),
    ("outputs", ["r", "a", "d", "ra", "rd", "ad", "rad"]),
    ("z_batch0", [False, True]),
    ("batch", ["B1", "B1_shared_flags", "B3"]),
    ("upstream", ["all", "no_rgb", "only_rgb"]),
    ("pointers", ["fresh", "off4", "off8"]),
    ("optional", ["given", "null"]),
]
NAMES = [n for n, _ in DIMS]
LEVELS = dict(DIMS)


def active(dim, kind):
    """whether `dim` means anything for texture kind `kind`"""
    if dim == "ts":
        return kind in ("cube", "cube_shared")
    if dim in ("image", "uvs"):
        return kind in ("uv", "mip")
    return True


def compatible(a):
    """partial assignment {dim: level} -> False if it violates a rule (rules involve at most two dimensions)"""
    kind = a.get("kind")
    out = a.get("outputs")
    if kind is not None and out is not None and (kind == "none") == ("r" in out):
        return False  # the texture models draw RGB, "none" draws no RGB
    if kind == "none" and a.get("light"):
        return False
    return True


def required_pairs():
    """every pair ((dim1, level1), (dim2, level2)) some valid case can hold"""
    out = set()
    for (i, (d1, l1s)), (j, (d2, l2s)) in itertools.combinations(enumerate(DIMS), 2):
        for l1 in l1s:
            for l2 in l2s:
                a = {d1: l1, d2: l2}
                if not compatible(a):
                    continue
                kinds = [a["kind"]] if "kind" in a else LEVELS["kind"]
                if any(active(d1, k) and active(d2, k) and compatible({**a, "kind": k}) for k in kinds):
                    out.add(((d1, l1), (d2, l2)))
    return out


def pairs_of(case):
    ks = [(n, case[n]) for n in NAMES if case[n] is not None]
    return set(itertools.combinations(ks, 2))


def _fill(case, covered, order):
    """assign the unassigned dimensions one after the other, each to the level that covers most new pairs (ties: the
    level that comes first in `order`, a rotation of the level list that changes from row to row)"""
    for name in NAMES:
        if name in case:
            continue
        if not active(name, case["kind"]):
            case[name] = None
            continue
        levels = LEVELS[name]
        r = order % len(levels)
        best, best_gain = None, -1
        for lv in levels[r:] + levels[:r]:
            if name == "raster" and case.get("_aa") is not None and (lv == "aa") != case["_aa"]:
                continue
            trial = {**case, name: lv}
            if not compatible(trial):
                continue
            gain = sum(1 for n2 in NAMES if n2 != name and trial.get(n2) is not None and not n2.startswith("_")
                       and _key(name, lv, n2, trial[n2]) not in covered)
            if gain > best_gain:
                best, best_gain = lv, gain
        case[name] = best
    case.pop("_aa", None)
    return case


def _key(d1, l1, d2, l2):
    return ((d1, l1), (d2, l2)) if NAMES.index(d1) < NAMES.index(d2) else ((d2, l2), (d1, l1))


# rows the pairs alone would not force: the edge scan zero-fills grad_textures on the side (one call, both halves, rgb
# upstream gradient, 16-byte aligned buffer) with a float count that is not a multiple of 4 (ts 3 and an odd cube count:
# the scalar tail of the fill)
MUST = [{"kind": "cube", "ts": 3, "fill_back": False, "_aa": False, "backward": "one", "upstream": "all", "pointers": "fresh"},
        {"kind": "cube_shared", "ts": 5, "fill_back": True, "_aa": True, "backward": "one", "upstream": "only_rgb",
         "pointers": "fresh"}]
# the fused light gradient: grad_face_light comes back only when the case is lit, passes the optional pointers and has an
# rgb upstream gradient -- a conjunction the pairs do not force.  Every texture kind gets it in a fresh and an
# accumulating backward, one call and two halves, with and without fill_back and anti-aliasing.
LIGHT_ROWS = [(False, False, "one"), (True, True, "acc_halves"), (True, False, "tex_faces"), (False, True, "acc_one")]
MUST += [{"kind": kind, "fill_back": fb, "_aa": aa, "backward": bwd, "light": True, "optional": "given",
          "upstream": ("all", "only_rgb")[i % 2]}
         for kind in ("cube", "cube_shared", "uv", "mip") for i, (fb, aa, bwd) in enumerate(LIGHT_ROWS)]


def cases():
    covered = set()
    out = []
    for n, seed in enumerate(MUST):
        c = _fill(dict(seed), covered, n)
        covered |= pairs_of(c)
        out.append(c)
    for n, (kind, fb, aa, bwd) in enumerate(itertools.product(LEVELS["kind"], LEVELS["fill_back"], (False, True),
                                                             LEVELS["backward"])):
        c = _fill({"kind": kind, "fill_back": fb, "_aa": aa, "backward": bwd}, covered, n)
        covered |= pairs_of(c)
        out.append(c)
    missing = sorted(required_pairs() - covered, key=repr)
    n = len(out)
    while missing:
        (d1, l1), (d2, l2) = missing[0]
        seed = {d1: l1, d2: l2}
        if "kind" not in seed:  # a kind under which both levels mean something
            seed["kind"] = next(k for k in LEVELS["kind"] if active(d1, k) and active(d2, k) and compatible({**seed, "kind": k}))
        c = _fill(seed, covered, n)
        covered |= pairs_of(c)
        out.append(c)
        missing = sorted(required_pairs() - covered, key=repr)
        n += 1
    for i, c in enumerate(out):
        c["id"] = i
    return out


def case_id(c):
    parts = [c["kind"] + ("%d" % c["ts"] if c["ts"] else ""), "fb" if c["fill_back"] else "", c["raster"], c["backward"],
             c["geometry"], ("img-" + c["image"] + ",uv-" + c["uvs"]) if c["image"] else "", "lit" if c["light"] else "",
             "bgB" if c["bg"] == "per_batch" else "", c["outputs"], "z0" if c["z_batch0"] else "", c["batch"],
             "up-" + c["upstream"], c["pointers"], "nulls" if c["optional"] == "null" else ""]
    return "%03d-" % c["id"] + "-".join(p for p in parts if p)
