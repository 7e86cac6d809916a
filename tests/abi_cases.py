"""Deterministic covering array over the flag dimensions of nr_b200_forward / nr_b200_backward /
nr_b200_backward_corner_light and of the attribute interpolation that reads their maps, nr_b200_interpolate /
nr_b200_interpolate_backward (test infrastructure).

`cases()` returns the case list of tests/test_gpu_abi_matrix.py: the full product of texture kind x fill_back x
anti-aliasing x backward mode, with every other dimension filled in greedily so that every compatible pair of levels of
any two dimensions appears in at least one case; rows are added until no pair is missing.  No randomness: the same list
on every machine.  The cases are generated in frozen stages, each one exactly as it was when the next joined, so
the ids, inputs and oracle of every earlier case stay the same: the matrix as it stood before smooth shading, the
face_uvs gradient, texture staging, the short layouts and interpolation joined it (BASE); then the rows and pairs of
those levels, with the interior vertex gradient off (FROZEN); then the interior rows and the pairs of every level.

A level that has no meaning for a case (ts without texture cubes, image / UV sharing and the face_uvs gradient without a
texture image, staging and the interior gradient without RGB) is None and takes part in no pair.  Combinations the ABI
rejects are never generated: texture kinds other than "none" always draw RGB and "none" never does, light (per face or
per corner) needs RGB, the short struct layouts (ending before corner_light / grad_face_uvs) carry neither field,
per-vertex attributes need indexed geometry, and the interior gradient refuses per-face cubes sampled with the depths of
item 0 (NR_TEX_Z_BATCH0) at B > 1; fill_back doubles the faces (F even) and anti-aliasing doubles the raster (even) by
construction of the geometry, so no case is skipped.  The attribute channel count C is not a dimension: it rotates over
ATTR_CHANNELS with the case id (abi_harness.Plan).

The Phong light modes (light "phong", "phong_set", "phong_sh": nr_b200_*_phong / _lights / _sh) joined as a fourth
stage.  Their dimensions -- the batch of each shading input (Bc, Bp, Bl, Bs: one set shared by every item, or one per
item), the light count NL, the entry point and the shininess -- mean something only under a Phong level and are None
elsewhere, so the cases of the earlier stages keep every level they had.  Attribute interpolation reads only the maps,
which shading leaves as they are, so it is None under a Phong level.  Phong needs RGB and refuses the interior
gradient; NL = 0 (SH without a light set) exists only with the SH environment, and a set of NL = 0 lights has no batch.

The normal map and the specular map (nr_b200_*_normal_map / nr_b200_*_specular_map) joined as a fifth stage, after the
271 cases of the first four, which are generated exactly as they were with `maps` held "off" and `map_entry` "direct".
`maps` (off, nm, sm, nm_sm) and `map_entry` mean something under a Phong level on a texture image (the maps are addressed
by the image's UVs): "direct" is the narrowest entry point that takes the structs given (without a map, the call the
`entry` dimension chooses), "via_nm" nr_b200_*_normal_map with a NULL map struct, "via_sm" nr_b200_*_specular_map with
NULL for each absent map.  The batches Bm, Bt (with a normal map) and Bq (with a specular map) and `map_grads` -- which
of grad_normal_map / grad_corner_tangents / grad_specular_map are wanted: all, the texels only, the tangents only, none
-- are None elsewhere.  `map_grads` is independent of `optional`, which keeps governing the Phong shading gradients, and
of `uv_grad`: with both of the others off, grad_face_uvs receives the maps' UV term from a kernel that runs for it alone."""
import itertools

DIMS = [
    ("kind", ["none", "cube", "cube_shared", "uv", "mip"]),
    ("fill_back", [False, True]),
    ("raster", ["even", "odd", "aa"]),
    ("backward", ["one", "tex_faces", "faces_tex", "acc_one", "acc_halves"]),
    ("geometry", ["faces", "idx_item", "idx_shared", "idx_shared_oor"]),
    ("ts", [2, 3, 4, 5, 6]),
    ("image", ["item", "shared"]),
    ("uvs", ["item", "shared"]),
    ("light", ["none", "face", "corner", "phong", "phong_set", "phong_sh"]),
    ("bg", ["uniform", "per_batch"]),
    ("outputs", ["r", "a", "d", "ra", "rd", "ad", "rad"]),
    ("z_batch0", [False, True]),
    ("batch", ["B1", "B1_shared_flags", "B3"]),
    ("upstream", ["all", "no_rgb", "only_rgb"]),
    ("pointers", ["fresh", "off4", "off8"]),
    ("optional", ["given", "null"]),
    ("uv_grad", ["given", "null"]),
    ("stage", [False, True]),
    ("layout", ["full", "short"]),
    ("attr", ["off", "corner", "corner_shared", "vertex", "vertex_shared"]),
    ("interior", ["off", "on"]),
    # the Phong modes (abi_harness.Plan): NL, the entry point, Bc, Bp, Bl, Bs ("shared" = 1, "item" = B) and sigma (16:
    # the shininess the feature tests hold the gradients at; at 64, q^sigma multiplies the fp32 error of q by sigma and
    # grad_params / grad_lights per element reach 8.8e-4 / 5.2e-4 against gates of 5e-4 / 2e-4)
    ("nl", [0, 1, 3, 8]),
    ("entry", ["own", "via_sh", "via_lights_nl0"]),
    ("shading_batch", ["shared", "item"]),
    ("params_batch", ["shared", "item"]),
    ("lights_batch", ["shared", "item"]),
    ("sh_batch", ["shared", "item"]),
    ("sigma", [1.0, 16.0]),
    # the normal map and the specular map (abi_harness.Plan): which maps the call carries, the entry point they travel
    # through, Bm, Bt, Bq ("shared" = 1, "item" = B) and which of the maps' gradient outputs are wanted
    ("maps", ["off", "nm", "sm", "nm_sm"]),
    ("map_entry", ["direct", "via_nm", "via_sm"]),
    ("nm_batch", ["shared", "item"]),
    ("tg_batch", ["shared", "item"]),
    ("sm_batch", ["shared", "item"]),
    ("map_grads", ["all", "texels", "tangents", "null"]),
]
NAMES = [n for n, _ in DIMS]
LEVELS = dict(DIMS)


PHONG = ("phong", "phong_set", "phong_sh")
PHONG_DIMS = ["nl", "entry", "shading_batch", "params_batch", "lights_batch", "sh_batch", "sigma"]
OLD_LIGHTS = ["none", "face", "corner"]
MAP_DIMS = ["maps", "map_entry", "nm_batch", "tg_batch", "sm_batch", "map_grads"]


def active(dim, c):
    """whether `dim` means anything for the case (or partial case) `c`: its texture kind, and for the Phong dimensions
    its light and light count"""
    kind, light = c["kind"], c.get("light")
    if dim in MAP_DIMS:  # the maps are addressed by the UVs of a texture image
        maps = c.get("maps")
        return light in PHONG and kind in ("uv", "mip") and (
            dim in ("maps", "map_entry") or maps in {"sm_batch": ("sm", "nm_sm"), "map_grads": ("nm", "sm", "nm_sm")}.get(dim, ("nm", "nm_sm")))
    if dim in ("shading_batch", "params_batch", "sigma"):
        return light in PHONG
    if dim == "entry":  # nr_b200_*_sh is the SH mode's own entry point
        return light in ("phong", "phong_set")
    if dim == "nl":
        return light in ("phong_set", "phong_sh")
    if dim == "lights_batch":
        return light in ("phong_set", "phong_sh") and c.get("nl") != 0
    if dim == "sh_batch":
        return light == "phong_sh"
    if dim == "attr":  # the interpolation reads only the maps, which shading does not change
        return light not in PHONG
    if dim == "ts":
        return kind in ("cube", "cube_shared")
    if dim in ("image", "uvs", "uv_grad"):
        return kind in ("uv", "mip")
    if dim in ("stage", "interior"):
        return kind != "none"
    return True


def compatible(a):
    """partial assignment {dim: level} -> False if it violates a rule (rules involve at most two dimensions, except the
    interior gradient's refusal of z_batch0 cubes at three items, which involves four)"""
    kind = a.get("kind")
    out = a.get("outputs")
    if kind is not None and out is not None and (kind == "none") == ("r" in out):
        return False  # the texture models draw RGB, "none" draws no RGB
    if kind == "none" and a.get("light") not in (None, "none"):
        return False
    if a.get("layout") == "short" and (a.get("light") == "corner" or a.get("uv_grad") == "given"):
        return False  # the short forward struct ends before corner_light, the short backward before grad_face_uvs
    if a.get("geometry") == "faces" and str(a.get("attr")).startswith("vertex"):
        return False  # per-vertex attributes need NR_FACES_INDEXED
    if (a.get("interior") == "on" and kind in ("cube", "cube_shared") and a.get("z_batch0") is True
            and a.get("batch") == "B3"):
        return False  # the cubes would be sampled with item 0's depths: the derivative would cross items (refused)
    light = a.get("light")
    if light in PHONG and a.get("interior") == "on":
        return False  # no vertex gradient through the Phong normal and position (NR_ERR_UNSUPPORTED)
    if a.get("nl") == 0 and (light == "phong_set" or a.get("lights_batch") is not None):
        return False  # NL = 0 is SH without a set: the set modes have lights, and no set has no batch
    if a.get("entry") == "via_lights_nl0" and light not in (None, "phong"):
        return False  # an empty light set is the plain Phong call
    maps, via = a.get("maps"), a.get("map_entry")
    if via == "via_nm" and maps not in (None, "off"):
        return False  # nr_b200_*_normal_map is the direct call of a normal map, and takes no specular map
    if via == "via_sm" and maps in ("sm", "nm_sm"):
        return False  # nr_b200_*_specular_map is the direct call of a specular map
    if a.get("map_grads") == "tangents" and maps == "sm":
        return False  # grad_corner_tangents belongs to the normal map's struct
    return True


def _context(a):
    """the first completion of partial assignment `a` by a texture kind (and, for a Phong dimension, a light and NL)
    under which each of its dimensions means something and the rules hold, or None"""
    kinds = [a["kind"]] if "kind" in a else LEVELS["kind"]
    lights, nls, mapses = [None], [None], [None]
    if any(d in PHONG_DIMS or d in MAP_DIMS for d in a):
        lights = [a["light"]] if "light" in a else list(PHONG)
    if any(d in PHONG_DIMS for d in a):
        nls = [a["nl"]] if "nl" in a else [None] + LEVELS["nl"]
    if any(d in MAP_DIMS[2:] for d in a):
        mapses = [a["maps"]] if "maps" in a else LEVELS["maps"]
    for k, lt, nl, mp in itertools.product(kinds, lights, nls, mapses):
        c = {**a, "kind": k, **({"light": lt} if lt is not None else {}), **({"nl": nl} if nl is not None else {}),
             **({"maps": mp} if mp is not None else {})}
        if all(active(d, c) for d in a if d != "kind") and compatible(c):
            return c
    return None


def required_pairs(levels=LEVELS):
    """every pair ((dim1, level1), (dim2, level2)) some valid case can hold, over the dimensions and levels of `levels`"""
    out = set()
    for d1, d2 in itertools.combinations([n for n in NAMES if n in levels], 2):
        for l1 in levels[d1]:
            for l2 in levels[d2]:
                a = {d1: l1, d2: l2}
                if compatible(a) and _context(a) is not None:
                    out.add(((d1, l1), (d2, l2)))
    return out


def pairs_of(case):
    ks = [(n, case[n]) for n in NAMES if case[n] is not None]
    return set(itertools.combinations(ks, 2))


def _fill(case, covered, order, choices=LEVELS):
    """assign the unassigned dimensions one after the other, each to the level of `choices` that covers most new pairs
    (ties: the level that comes first in `order`, a rotation of the level list that changes from row to row)"""
    for name in NAMES:
        if name in case:
            continue
        if not active(name, case):
            case[name] = None
            continue
        levels = choices[name]
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


# The matrix as it stood before smooth shading, the face_uvs gradient, texture staging, the short struct layouts and
# attribute interpolation joined it: its dimensions and levels, the others held at the level that leaves the call as it
# was.  Its cases are generated first, exactly as before, so their ids and inputs stay what they were.
BASE = {**{n: LEVELS[n] for n in NAMES[:NAMES.index("optional") + 1]}, "ts": [2, 3, 5], "light": ["none", "face"],
        "uv_grad": ["null"], "stage": [False], "layout": ["full"], "attr": ["off"], "interior": ["off"]}
BASE_PAIRS = {n: BASE[n] for n in NAMES[:NAMES.index("optional") + 1]}

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
MUST += [{"kind": kind, "fill_back": fb, "_aa": aa, "backward": bwd, "light": "face", "optional": "given",
          "upstream": ("all", "only_rgb")[i % 2]}
         for kind in ("cube", "cube_shared", "uv", "mip") for i, (fb, aa, bwd) in enumerate(LIGHT_ROWS)]
# the same for smooth shading: grad_corner_light (nr_b200_backward_corner_light) with the same spread of backward modes
CORNER_ROWS = [(False, False, "faces_tex"), (True, True, "acc_halves"), (True, False, "one"), (False, True, "acc_one")]
MUST_NEW = [{"kind": kind, "fill_back": fb, "_aa": aa, "backward": bwd, "light": "corner", "optional": "given",
          "upstream": ("all", "only_rgb")[i % 2]}
         for kind in ("cube", "cube_shared", "uv", "mip") for i, (fb, aa, bwd) in enumerate(CORNER_ROWS)]
# corner light with NR_TEX_Z_BATCH0 on indexed geometry, three items: the cube texture gradient reloads each item's own
# depths for the perspective weights (the cube coordinates keep item 0's)
MUST_NEW += [{"kind": kind, "light": "corner", "z_batch0": True, "batch": "B3", "geometry": geom, "optional": "given",
          "upstream": "all"}
         for kind, geom in (("cube", "idx_item"), ("cube_shared", "idx_shared"))]
# grad_face_uvs at every phase of the 6-float reduction (4 bytes in: phases 1 / 3; fresh and 8 bytes in: 0 / 2), for both
# samplers, and once each with corner light (the kUvGrad && kCorner variants)
MUST_NEW += [{"kind": kind, "uv_grad": "given", "upstream": up, "pointers": ptr, "light": light}
         for kind in ("uv", "mip")
         for up, ptr, light in (("all", "off4", "none"), ("only_rgb", "fresh", "face"), ("all", "off8", "none"),
                                ("all", "off4", "corner"))]
# NR_FWD_STAGE_TEXTURES where it really stages (cube kinds, no anti-aliasing, 16-byte aligned textures, 16-byte cubes:
# ts even), and once with ts = 6 (2592-byte cubes, 12 slots per row segment) where a pixel row shows more runs of
# distinct faces than there are slots, so the runs beyond the capacity read global memory
MUST_NEW += [{"kind": "cube", "stage": True, "_aa": False, "pointers": "fresh", "ts": 2, "light": "face", "upstream": "all",
              "batch": "B3"},
         {"kind": "cube_shared", "stage": True, "_aa": False, "pointers": "fresh", "ts": 4, "light": "none"},
         {"kind": "cube", "stage": True, "_aa": False, "pointers": "fresh", "ts": 6, "light": "none", "fill_back": False,
          "batch": "B3", "raster": "even"}]
# the matrix as it stood before the interior vertex gradient joined it: every level but that flag, held off (and
# without the Phong modes)
FROZEN = {**LEVELS, "light": OLD_LIGHTS, "interior": ["off"]}
FROZEN_PAIRS = {n: FROZEN[n] for n in NAMES if n != "interior" and n not in PHONG_DIMS + MAP_DIMS}
# the matrix as it stood before the Phong modes joined it
INTERIOR = {**LEVELS, "light": OLD_LIGHTS}
INTERIOR_PAIRS = {n: INTERIOR[n] for n in NAMES if n not in PHONG_DIMS + MAP_DIMS}

# the interior vertex gradient (NR_GRAD_INTERIOR) with an rgb upstream gradient, for every texture kind: every light, a
# fresh and an accumulating backward, one call and two halves, with and without fill_back and anti-aliasing, spread over
# the four geometries and the three batch levels.  Per-item index sets and per-item light at three items (the scatter and
# the light reads address item b), ts 3 / 5 / 6, z_batch0 cubes at B = 1 and z_batch0 images at B = 3 (no effect there),
# K5 with rgb + alpha and K7 adding into the same buffer (outputs "rad"), NULL optional pointers.  The image size follows
# the case id (abi_harness.Plan): the rows sit so that the last uv row (id 188) and the third mip row (id 191) get the
# one-texel-high (1, 9) image.
_I = [  # kind, light, fill_back, aa, backward, geometry, batch, extra levels
    ("cube", "none", False, False, "one", "idx_item", "B3", {"ts": 3, "outputs": "rad", "upstream": "all"}),
    ("cube", "face", True, True, "acc_halves", "faces", "B3", {"ts": 5, "optional": "given"}),
    ("cube", "corner", True, False, "faces_tex", "idx_shared_oor", "B3", {"ts": 6, "optional": "given"}),
    ("cube", "face", False, True, "acc_one", "idx_shared", "B1", {"ts": 4, "z_batch0": True}),
    ("cube_shared", "corner", False, False, "one", "idx_item", "B3", {"ts": 5, "optional": "null"}),
    ("cube_shared", "none", True, True, "acc_halves", "idx_shared", "B1_shared_flags", {"ts": 3, "z_batch0": True}),
    ("cube_shared", "face", True, False, "tex_faces", "idx_item", "B3", {"ts": 6, "outputs": "rad", "upstream": "all"}),
    ("cube_shared", "corner", False, True, "acc_one", "faces", "B3", {"ts": 2}),
    ("uv", "face", False, False, "one", "idx_item", "B3", {"uv_grad": "given", "outputs": "rad", "upstream": "all"}),
    ("uv", "corner", True, True, "acc_halves", "idx_shared_oor", "B3", {"z_batch0": True}),
    ("uv", "none", True, False, "faces_tex", "faces", "B1", {"optional": "null"}),
    ("uv", "corner", False, True, "acc_one", "idx_item", "B3", {"image": "item", "uvs": "shared"}),
    ("mip", "corner", False, False, "one", "idx_item", "B3", {"outputs": "rad", "upstream": "all"}),
    ("mip", "face", True, True, "acc_halves", "faces", "B3", {"uv_grad": "given", "z_batch0": True}),
    ("mip", "none", True, False, "tex_faces", "idx_shared", "B1", {"image": "shared", "uvs": "item"}),
    ("mip", "face", False, True, "acc_one", "idx_item", "B3", {"optional": "null"}),
]
MUST_INTERIOR = [{"kind": kind, "light": light, "fill_back": fb, "_aa": aa, "backward": bwd, "geometry": geom, "batch": batch,
                  "interior": "on", "upstream": ("all", "only_rgb")[i % 2], **extra}
                 for i, (kind, light, fb, aa, bwd, geom, batch, extra) in enumerate(_I)]

# The Phong modes, every shading gradient given (optional pointers) with an rgb upstream gradient, for every texture
# kind: a fresh and an accumulating backward, one call and two halves in both orders, with and without fill_back and
# anti-aliasing.  The geometry and NL of the rows reach every instantiation k_phong_grad<kTex, kIdx, kLights, kSH>
# (nr_phong.cu) -- per-face and indexed geometry under Phong alone, a light set, SH without a set (NL = 0) and SH with
# one -- and the full set of 8 lights (s_lt[8][80]) at least once per texture kind.
PHONG_ROWS = [(False, False, "one", "faces"), (True, True, "acc_halves", "idx_item"), (True, False, "faces_tex", "idx_shared"),
              (False, True, "acc_one", "faces")]
PHONG_NL = {"phong_set": [8, 3, 1, 3], "phong_sh": [0, 0, 8, 1]}
MUST_PHONG = [{"kind": kind, "light": mode, "fill_back": fb, "_aa": aa, "backward": bwd, "geometry": geom,
               "optional": "given", "upstream": ("all", "only_rgb")[i % 2],
               **({"nl": PHONG_NL[mode][i]} if mode in PHONG_NL else {})}
              for mode in PHONG for kind in ("cube", "cube_shared", "uv", "mip")
              for i, (fb, aa, bwd, geom) in enumerate(PHONG_ROWS)]
# cube Phong with NR_TEX_Z_BATCH0 at three items on per-item index sets: the sampler (forward and k_phong_grad) reads item
# 0's depths, the perspective weights l_k of the normal and position the item's own
MUST_PHONG += [{"kind": kind, "light": mode, "z_batch0": True, "batch": "B3", "geometry": "idx_item", "optional": "given",
                "upstream": "all", **nl}
               for kind, mode, nl in (("cube", "phong", {}), ("cube", "phong_set", {"nl": 3}),
                                      ("cube_shared", "phong_sh", {"nl": 0}), ("cube_shared", "phong_sh", {"nl": 3}))]
# the short forward / backward layouts under every mode: the NaN field past the forward's struct_size is corner_light,
# which the host would refuse next to a Phong struct if it read it
MUST_PHONG += [{"kind": kind, "light": mode, "layout": "short", "optional": "given", "upstream": "all"}
               for kind, mode in (("cube", "phong"), ("uv", "phong_set"), ("mip", "phong_sh"))]
# every shading gradient given without an rgb upstream gradient: fresh ones come back 0, accumulated ones keep their
# prefill bit for bit (slots 10-11 of grad_lights included)
MUST_PHONG += [{"kind": kind, "light": mode, "upstream": "no_rgb", "outputs": "rad", "optional": "given", "backward": bwd,
                **nl}
               for kind, mode, nl in (("cube", "phong", {}), ("uv", "phong_set", {"nl": 3}), ("mip", "phong_sh", {"nl": 8}))
               for bwd in ("one", "acc_one")]
# Bc = Bp = Bl = Bs = 1 at three items, and all of them = B
MUST_PHONG += [{"kind": kind, "light": "phong_sh", "nl": 3, "batch": "B3", "optional": "given", "upstream": "all",
                **{d: lv for d in ("shading_batch", "params_batch", "lights_batch", "sh_batch")}}
               for kind, lv in (("cube", "shared"), ("uv", "item"), ("mip", "shared"), ("cube_shared", "item"))]
# shared textures / UVs at three items under every mode
MUST_PHONG += [{"kind": "uv", "light": "phong", "batch": "B3", "image": "shared", "uvs": "item", "optional": "given",
                "upstream": "all"},
               {"kind": "mip", "light": "phong_set", "nl": 1, "batch": "B3", "image": "item", "uvs": "shared",
                "optional": "given", "upstream": "all"},
               {"kind": "cube_shared", "light": "phong_sh", "nl": 3, "batch": "B3", "optional": "given",
                "upstream": "only_rgb"}]
# the matrix as it stood before the normal map and the specular map joined it: no map, through the entry point the
# `entry` dimension chooses
NO_MAPS = {**LEVELS, "maps": ["off"], "map_entry": ["direct"]}
NO_MAPS_PAIRS = {n: LEVELS[n] for n in NAMES if n not in MAP_DIMS}

# The maps (light modes 6 and 7: nr_b200_*_normal_map / nr_b200_*_specular_map), every gradient given with an rgb upstream
# gradient.  Each of the 48 instantiations k_phong_grad<kTex, kIdx, kLights, kSH, kNM, kSM> (nr_phong.cu) with kNM || kSM
# once: nm, sm and both x bilinear and trilinear albedo x per-face and indexed geometry x Phong alone, a light set, SH
# without a set and SH with one -- for sm alone these are also the four targets of the texture gradient's re-mapping of
# mode 7 (nr_backward.cu, tg_light), for both samplers.  The eight rows of a (maps, sampler) take the eight entries of
# MAP_ROWS, from a start that moves on, so each has a fresh and an accumulating backward, one call and two halves in both
# orders, with and without fill_back and anti-aliasing.  The rows' pointer levels walk fresh / 4 / 8 bytes in, and the
# map sizes follow the case id (abi_harness.Plan), so that grad_normal_map sits 0, 4 and 8 bytes and grad_specular_map
# 0, 4, 8 and 12 bytes past a 16-byte boundary, each with a one-texel-wide and a wider map (tests/test_abi_cases_cpu.py).
MAP_ROWS = [(False, False, "one"), (True, True, "acc_halves"), (True, False, "faces_tex"), (False, True, "acc_one"),
            (False, True, "tex_faces"), (True, False, "acc_one"), (False, False, "acc_halves"), (True, True, "one")]
MAP_VARIANTS = [("phong", {}), ("phong_set", {"nl": 3}), ("phong_sh", {"nl": 0}), ("phong_sh", {"nl": 1})]
_ALL = {"optional": "given", "map_grads": "all", "upstream": "all"}
MUST_MAPS = []
for _s, (_maps, _kind) in enumerate(itertools.product(("nm", "sm", "nm_sm"), ("uv", "mip"))):
    for _i, (_geom, (_mode, _nl)) in enumerate(itertools.product((False, True), MAP_VARIANTS)):
        _fb, _aa, _bwd = MAP_ROWS[(_i + 3 * _s) % 8]
        _j = len(MUST_MAPS)
        MUST_MAPS.append({"kind": _kind, "light": _mode, **_nl, "maps": _maps, "map_entry": "direct", "fill_back": _fb,
                          "_aa": _aa, "backward": _bwd, "uv_grad": "given",
                          "geometry": ("idx_item", "idx_shared")[_j % 2] if _geom else "faces",
                          "pointers": ("fresh", "off4", "off8")[_j % 3], **_ALL,
                          "upstream": ("all", "only_rgb")[_i % 2]})
# the full set of 8 lights (s_lt[8][80], the highest register use) with both maps, once per sampler
MUST_MAPS += [{"kind": kind, "light": mode, "nl": 8, "maps": "nm_sm", "uv_grad": "given", **_ALL}
              for kind, mode in (("uv", "phong_set"), ("mip", "phong_sh"))]
# the maps' UV term alone: grad_face_uvs wanted and every shading and map gradient NULL (k_phong_grad then runs for that
# term only), for both samplers; then the reverse, the maps' texels wanted and neither grad_face_uvs nor a shading gradient;
# and grad_corner_tangents alone (a branch of its own in the run reduction)
MUST_MAPS += [{"kind": kind, "light": mode, **nl, "maps": maps, "optional": "null", "map_grads": "null", "uv_grad": "given",
               "upstream": "all"}
              for kind in ("uv", "mip") for maps, mode, nl in (("nm", "phong", {}), ("sm", "phong_set", {"nl": 3}),
                                                               ("nm_sm", "phong_sh", {"nl": 1}))]
MUST_MAPS += [{"kind": kind, "light": "phong_set", "nl": 1, "maps": maps, "optional": "null", "map_grads": "texels",
               "uv_grad": "null", "upstream": "all"}
              for kind, maps in (("uv", "nm"), ("mip", "sm"), ("uv", "nm_sm"))]
MUST_MAPS += [{"kind": "mip", "light": "phong", "maps": "nm", "optional": "null", "map_grads": "tangents", "uv_grad": "given",
               "upstream": "all"}]
# shared UVs at three items with fill_back (the maps' UV term summed over the items, the copies' corners reversed: `rev`
# in nm_grad_tail / sm_grad_tail), with a shared and with a per-item image
MUST_MAPS += [{"kind": kind, "light": "phong_set", "nl": 3, "maps": maps, "batch": "B3", "uvs": "shared", "image": image,
               "fill_back": True, "uv_grad": "given", **_ALL}
              for kind, maps, image in (("uv", "nm", "shared"), ("mip", "sm", "item"))]
# Bm = Bt = Bq = 1 next to Bc = Bp = Bl = Bs = B at three items, the reverse, all of them 1 and all of them B
MUST_MAPS += [{"kind": kind, "light": "phong_sh", "nl": 3, "maps": "nm_sm", "batch": "B3", "uv_grad": "given", **_ALL,
               **{d: m for d in ("nm_batch", "tg_batch", "sm_batch")},
               **{d: o for d in ("shading_batch", "params_batch", "lights_batch", "sh_batch")}}
              for kind, m, o in (("uv", "shared", "item"), ("mip", "item", "shared"), ("mip", "shared", "shared"),
                                 ("uv", "item", "item"))]
# the short layouts: the NaN buffer behind the field past the short backward struct is where the maps' UV term would land
MUST_MAPS += [{"kind": kind, "light": mode, **nl, "maps": maps, "layout": "short", **_ALL}
              for kind, maps, mode, nl in (("uv", "nm", "phong", {}), ("mip", "sm", "phong_set", {"nl": 3}),
                                           ("uv", "nm_sm", "phong_sh", {"nl": 1}))]
# every gradient given without an rgb upstream gradient: fresh ones come back 0, accumulated ones keep their prefill
MUST_MAPS += [{"kind": kind, "light": "phong_set", "nl": 3, "maps": "nm_sm", "upstream": "no_rgb", "outputs": "rad",
               "optional": "given", "map_grads": "all", "uv_grad": "given", "backward": bwd}
              for kind, bwd in (("uv", "one"), ("mip", "acc_one"))]
# NR_TEX_Z_BATCH0 at three items on per-item index sets: images ignore the flag, and the maps must too
MUST_MAPS += [{"kind": "uv", "light": "phong_set", "nl": 1, "maps": "nm_sm", "z_batch0": True, "batch": "B3",
               "geometry": "idx_item", "uv_grad": "given", **_ALL}]
# no map through the map entry points (a NULL nm; a NULL nm and a NULL sm) under every earlier mode, and a normal map
# through nr_b200_*_specular_map with a NULL sm
MUST_MAPS += [{"kind": kind, "light": mode, **nl, "maps": "off", "map_entry": via, "optional": "given", "upstream": "all",
               "uv_grad": "given"}
              for via, kind in (("via_nm", "uv"), ("via_sm", "mip"))
              for mode, nl in (("phong", {}), ("phong_set", {"nl": 3}), ("phong_sh", {"nl": 3}))]
MUST_MAPS += [{"kind": "uv", "light": "phong_sh", "nl": 0, "maps": "nm", "map_entry": "via_sm", "uv_grad": "given", **_ALL}]
# out-of-range indices (faces that never win a pixel) with both maps
MUST_MAPS += [{"kind": "mip", "light": "phong_set", "nl": 3, "maps": "nm_sm", "geometry": "idx_shared_oor", "uv_grad": "given",
               **_ALL}]


def _complete(out, covered, choices, pairs):
    """append rows until every pair of `pairs` (required_pairs of some levels) is covered"""
    missing = sorted(pairs - covered, key=repr)
    n = len(out)
    while missing:
        (d1, l1), (d2, l2) = missing[0]
        seed = _context({d1: l1, d2: l2})  # with a kind (and light) under which both levels mean something
        c = _fill(seed, covered, n, choices)
        covered |= pairs_of(c)
        out.append(c)
        missing = sorted(pairs - covered, key=repr)
        n += 1


def cases():
    covered = set()
    out = []
    # the earlier matrix, first
    for n, seed in enumerate(MUST):
        c = _fill(dict(seed), covered, n, BASE)
        covered |= pairs_of(c)
        out.append(c)
    for n, (kind, fb, aa, bwd) in enumerate(itertools.product(LEVELS["kind"], LEVELS["fill_back"], (False, True),
                                                             LEVELS["backward"])):
        c = _fill({"kind": kind, "fill_back": fb, "_aa": aa, "backward": bwd}, covered, n, BASE)
        covered |= pairs_of(c)
        out.append(c)
    _complete(out, covered, BASE, required_pairs(BASE_PAIRS))
    # then the rows and pairs of every level but the interior gradient
    for seed in MUST_NEW:
        c = _fill(dict(seed), covered, len(out), FROZEN)
        covered |= pairs_of(c)
        out.append(c)
    _complete(out, covered, FROZEN, required_pairs(FROZEN_PAIRS))
    # then the interior rows and the pairs of every level but the Phong modes
    for seed in MUST_INTERIOR:
        c = _fill(dict(seed), covered, len(out), INTERIOR)
        covered |= pairs_of(c)
        out.append(c)
    _complete(out, covered, INTERIOR, required_pairs(INTERIOR_PAIRS))
    # then the Phong rows and the pairs of every level but the maps
    for seed in MUST_PHONG:
        c = _fill(dict(seed), covered, len(out), NO_MAPS)
        covered |= pairs_of(c)
        out.append(c)
    _complete(out, covered, NO_MAPS, required_pairs(NO_MAPS_PAIRS))
    # then the map rows and the pairs of every level
    for seed in MUST_MAPS:
        c = _fill(dict(seed), covered, len(out))
        covered |= pairs_of(c)
        out.append(c)
    _complete(out, covered, LEVELS, required_pairs())
    for i, c in enumerate(out):
        c["id"] = i
    return out


def case_id(c):
    parts = [c["kind"] + ("%d" % c["ts"] if c["ts"] else ""), "fb" if c["fill_back"] else "", c["raster"], c["backward"],
             c["geometry"], ("img-" + c["image"] + ",uv-" + c["uvs"]) if c["image"] else "",
             "uvgrad" if c["uv_grad"] == "given" else "", _light_id(c),
             "stage" if c["stage"] else "", "bgB" if c["bg"] == "per_batch" else "", c["outputs"],
             "z0" if c["z_batch0"] else "", c["batch"], "up-" + c["upstream"], c["pointers"],
             "nulls" if c["optional"] == "null" else "", "short" if c["layout"] == "short" else "",
             "" if c["attr"] in (None, "off") else "attr-" + c["attr"], "interior" if c["interior"] == "on" else ""]
    return "%03d-" % c["id"] + "-".join(p for p in parts if p)


def _light_id(c):
    light = c["light"]
    if light not in PHONG:
        return {"none": "", "face": "lit", "corner": "smooth"}[light]
    parts = [{"phong": "phong", "phong_set": "set%d", "phong_sh": "sh%d"}[light].replace("%d", str(c["nl"]))]
    parts += [c["entry"].replace("own", "") if c["entry"] else "", "s%g" % c["sigma"]]
    parts += [n + c[d][0] for n, d in (("Bc", "shading_batch"), ("Bp", "params_batch"), ("Bl", "lights_batch"),
                                       ("Bs", "sh_batch")) if c[d]]
    if c["maps"] not in (None, "off") or c["map_entry"] not in (None, "direct"):  # earlier ids keep their names
        parts += [c["maps"], c["map_entry"].replace("direct", "")]  # "off" here is a NULL map struct
        parts += [n + c[d][0] for n, d in (("Bm", "nm_batch"), ("Bt", "tg_batch"), ("Bq", "sm_batch")) if c[d]]
        parts += ["mg-" + c["map_grads"]] if c["map_grads"] else []
    return "-".join(p for p in parts if p)
