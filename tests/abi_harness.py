"""Direct C-ABI harness for nr_b200_forward, nr_b200_backward / nr_b200_backward_corner_light, the Phong entry points
nr_b200_{forward,backward}_{phong,lights,sh,normal_map,specular_map} and nr_b200_interpolate /
nr_b200_interpolate_backward (test infrastructure).

It fills _lib.ForwardArgs / BackwardArgs / InterpolateArgs itself -- no Python wrapper in between -- from a case of
abi_cases.py, so that each case controls the exact flag word, the struct size (the full layouts, or the short ones that
end before corner_light / grad_face_uvs), which optional pointers are NULL, where every user buffer sits (fresh, or 4
bytes into a slightly larger allocation; grad_textures, grad_face_uvs and grad_corner_light also 8 bytes in: 2-float but
not 4-float aligned) and what every output buffer holds before the call: NaN in each float output and a sentinel in
face_index_map, so an element the kernels fail to write shows, or seeded values for NR_GRAD_ACCUMULATE.  The Phong
inputs (corner_shading, params, lights, sh), the maps (normal_map, corner_tangents, specular_map) and their gradients
are user buffers like every other; grad_normal_map and grad_corner_tangents also sit 8 bytes in, grad_specular_map 8 or
12 (its 4-float reduction splits by phase), and specular_map itself always on a 16-byte boundary, as the ABI demands.  Guard words
around every buffer show a store just outside it.  With a short layout the field just past struct_size points at a real,
NaN-filled, guarded buffer: the forward would light the image with NaN if it read it, and the backward must leave it
as it was, bit for bit.

The alignment cases stay inside the ABI's promise (float alignment).  Every vector access of a user buffer in csrc/ is
behind a host check on its address: the edge scan's side fill of grad_textures (16 bytes, else a memset), the staged
strips of the edge scan (8 bytes on face_index_map, rgb_map, grad_rgb, grad_alpha), the TMA staging of texture cubes
(16 bytes), and the v4 / v2 reductions of k_texture_grad / k_image_grad (grad_textures, grad_face_uvs), which pick their
width from the address."""
import ctypes

import numpy as np

NEAR, FAR, EPS = 0.1, 100.0, 1e-4
UNIFORM_BG = (0.1, 0.2, 0.3)
FIM_SENTINEL = -7  # never a face index, never the -1 of an empty pixel
RASTER = {"even": (64, 64), "odd": (57, 57), "aa": (66, 33)}  # raster S, API image H (anti-aliased: odd pooled size)
F_FRONT = {False: 201, True: 101}  # front faces; fill_back appends the reversed copies: F = 201 or 202 (odd / even)
UV_SIZES = [(17, 41), (32, 32), (9, 30), (1, 9), (24, 13)]
MIP_SIZES = [(37, 29), (64, 48), (17, 41), (1, 9)]
ATTR_CHANNELS = [1, 3, 4, 16]
# normal-map and specular-map sizes (H, W): one texel, one row, one column (the clamped x1 == x0 of every pixel), odd, even
MAP_SIZES = [(1, 1), (1, 23), (19, 1), (37, 53), (16, 16), (9, 11)]
MAP_GRADS = ("grad_normal_map", "grad_corner_tangents", "grad_specular_map")
K_STAGE_BYTES = 32 * 1024  # shared memory of a staged k_resolve CTA (csrc/nr_forward.cu kStageBytes)


def _lib():
    from neural_renderer_b200 import _lib as L
    return L


class Plan:
    """shapes, flags and pointer layout of one case (pure host data: no device needed)"""

    def __init__(self, c):
        L = _lib()
        self.case = c
        self.kind = c["kind"]
        self.B = 3 if c["batch"] == "B3" else 1
        shared_flags = c["batch"] != "B1"  # B1: shared data at batch 1 without the flag bits; else the bits are set
        self.fill_back = c["fill_back"]
        self.F_front = F_FRONT[self.fill_back]
        self.F = 2 * self.F_front if self.fill_back else self.F_front
        self.S, self.H = RASTER[c["raster"]]
        self.aa = c["raster"] == "aa"
        self.rgb, self.alpha, self.depth = ("r" in c["outputs"]), ("a" in c["outputs"]), ("d" in c["outputs"])
        self.indexed = c["geometry"] != "faces"
        self.idx_shared = c["geometry"] in ("idx_shared", "idx_shared_oor")
        from neural_renderer_b200 import synthetic
        self.Nv = synthetic.sphere_mesh(self.F_front)[0].shape[0]
        self.ts = c["ts"] or 0
        self.uv = self.kind in ("uv", "mip")
        self.mip = self.kind == "mip"
        self.tex_shared = self.kind == "cube_shared" or (self.uv and c["image"] == "shared")
        self.uv_shared = self.uv and c["uvs"] == "shared"
        self.Ht = self.Wt = 0
        if self.uv:
            sizes = MIP_SIZES if self.mip else UV_SIZES
            self.Ht, self.Wt = sizes[c["id"] % len(sizes)]
        self.P = int(L.load().nr_b200_mip_texels(self.Ht, self.Wt)) if self.mip else 0
        self.lit = c["light"] == "face"
        self.corner = c["light"] == "corner"
        self.uv_grad = c["uv_grad"] == "given"
        self.short = c["layout"] == "short"
        self.bg_batch = c["bg"] == "per_batch"
        self.given = c["optional"] == "given"
        self.attr = c["attr"] not in (None, "off")  # None under the Phong modes
        self.attr_pv = self.attr and c["attr"].startswith("vertex")
        self.attr_shared = self.attr and c["attr"].endswith("_shared")
        self.C = ATTR_CHANNELS[c["id"] % len(ATTR_CHANNELS)] if self.attr else 0
        self.interior = c["interior"] == "on"  # NR_GRAD_INTERIOR: a backward-only bit (backward_calls)
        # the Phong modes: the entry point, the batch of each shading input (1 or B) and the light count
        self.phong = c["light"] in ("phong", "phong_set", "phong_sh")
        self.sh = c["light"] == "phong_sh"
        self.entry = "sh" if self.sh else c["entry"]
        per = lambda d: self.B if c[d] == "item" else 1
        self.Bc, self.Bp = (per("shading_batch"), per("params_batch")) if self.phong else (0, 0)
        self.NL = c["nl"] if c["light"] in ("phong_set", "phong_sh") else 0
        self.Bl = per("lights_batch") if self.NL else 0
        self.Bs = per("sh_batch") if self.sh else 0
        self.sigma = c["sigma"]
        # the maps: which of them the call carries, the entry point, the batch of each (1 or B), and their sizes, which
        # rotate with the case id independently of each other (and of the albedo's)
        self.nm, self.sm = c["maps"] in ("nm", "nm_sm"), c["maps"] in ("sm", "nm_sm")
        self.map_entry = c["map_entry"] or "direct"
        self.Bm, self.Bt = (per("nm_batch"), per("tg_batch")) if self.nm else (0, 0)
        self.Bq = per("sm_batch") if self.sm else 0
        self.Hm, self.Wm = MAP_SIZES[c["id"] % 6] if self.nm else (0, 0)
        self.Hq, self.Wq = MAP_SIZES[c["id"] // 2 % 6] if self.sm else (0, 0)
        f = 0
        f |= L.NR_RETURN_RGB if self.rgb else 0
        f |= L.NR_RETURN_ALPHA if self.alpha else 0
        f |= L.NR_RETURN_DEPTH if self.depth else 0
        f |= L.NR_ANTI_ALIASING if self.aa else 0
        f |= L.NR_BG_PER_BATCH if self.bg_batch else 0
        f |= L.NR_TEX_Z_BATCH0 if c["z_batch0"] else 0
        f |= L.NR_TEX_FILL_BACK if self.fill_back else 0
        f |= L.NR_FACES_INDEXED if self.indexed else 0
        f |= L.NR_INDICES_SHARED if (self.idx_shared and shared_flags) else 0
        f |= L.NR_TEX_SHARED if (self.tex_shared and shared_flags) else 0
        f |= L.NR_TEX_UV if self.uv else 0
        f |= L.NR_UV_SHARED if (self.uv_shared and shared_flags) else 0
        f |= L.NR_TEX_MIPMAP if self.mip else 0
        self.flags = f
        self.fwd_flags = f | (L.NR_FWD_STAGE_TEXTURES if c["stage"] else 0)  # a forward-only bit
        af = f & (L.NR_ANTI_ALIASING | L.NR_FACES_INDEXED | L.NR_INDICES_SHARED)
        af |= L.NR_ATTR_PER_VERTEX if self.attr_pv else 0
        af |= L.NR_ATTR_SHARED if (self.attr_shared and shared_flags) else 0
        self.attr_flags = af
        up = c["upstream"]
        self.g_rgb = self.rgb and up in ("all", "only_rgb")
        self.g_alpha = self.alpha and up in ("all", "no_rgb")
        self.g_depth = self.depth and up in ("all", "no_rgb")
        self.n_cubes = self.F_front if self.fill_back else self.F
        Bt = 1 if self.tex_shared else self.B
        if self.kind in ("cube", "cube_shared"):
            tex_shape = (Bt, self.n_cubes, self.ts, self.ts, self.ts, 3)
        elif self.mip:
            tex_shape = (Bt, self.P, 3)
        elif self.uv:
            tex_shape = (Bt, self.Ht, self.Wt, 3)
        else:
            tex_shape = None
        B, F, S, H, Nv = self.B, self.F, self.S, self.H, self.Nv
        f32, i32 = np.float32, np.int32
        # name -> (shape, dtype) of every user buffer the case passes; a name that is missing is NULL
        bufs = {}
        if self.indexed:
            bufs["vertices"] = ((B, Nv, 3), f32)
            bufs["face_indices"] = (((F, 3) if self.idx_shared else (B, F, 3)), i32)
            if self.given:  # ignored with NR_FACES_INDEXED: NaN faces in, grad_faces left as it was
                bufs["faces"] = ((B, F, 3, 3), f32)
        else:
            bufs["faces"] = ((B, F, 3, 3), f32)
        nu = self.F_front if self.fill_back else F
        uv_shape = (nu, 3, 2) if self.uv_shared else (B, nu, 3, 2)
        if self.rgb:
            bufs["textures"] = (tex_shape, f32)
            if self.lit:
                bufs["face_light"] = ((B, F, 3), f32)
            if self.corner:
                bufs["corner_light"] = ((B, F, 3, 3), f32)
            if self.uv:
                bufs["face_uvs"] = (uv_shape, f32)
            if self.phong:
                bufs["corner_shading"] = ((self.Bc, F, 3, 6), f32)
                bufs["params"] = ((self.Bp, 16), f32)
                if self.NL:
                    bufs["lights"] = ((self.Bl, self.NL, 12), f32)
                if self.sh:
                    bufs["sh"] = ((self.Bs, 9, 3), f32)
            if self.nm:
                bufs["normal_map"] = ((self.Bm, self.Hm, self.Wm, 3), f32)
                bufs["corner_tangents"] = ((self.Bt, F, 3, 4), f32)
            if self.sm:
                bufs["specular_map"] = ((self.Bq, self.Hq, self.Wq, 4), f32)
        if self.short:  # what the fields past the short layouts point at: never to be read
            bufs["past_end_fwd"] = ((B, F, 3, 3), f32)
            bufs["past_end_bwd"] = ((uv_shape if self.uv else (B, F, 3, 2)), f32)
        if self.bg_batch and (self.rgb or self.given):
            bufs["background_batch"] = ((B, 3), f32)
        bufs["face_index_map"] = ((B, S, S), i32)
        bufs["weight_map"] = ((B, 3, S, S), f32)
        bufs["depth_map"] = ((B, S, S), f32)
        if self.rgb:
            bufs["rgb_map"] = ((B, 3, S, S), f32)
        if self.alpha and self.given:
            bufs["alpha_map"] = ((B, S, S), f32)
        if self.aa and self.given:
            for k, want, shape in (("out_rgb", self.rgb, (B, 3, H, H)), ("out_alpha", self.alpha, (B, H, H)),
                                   ("out_depth", self.depth, (B, H, H))):
                if want:
                    bufs[k] = (shape, f32)
        if self.g_rgb:
            bufs["grad_rgb"] = ((B, 3, H, H), f32)
        if self.g_alpha:
            bufs["grad_alpha"] = ((B, H, H), f32)
        if self.g_depth:
            bufs["grad_depth"] = ((B, H, H), f32)
        if self.indexed:
            bufs["grad_vertices"] = ((B, Nv, 3), f32)
            if self.given:
                bufs["grad_faces"] = ((B, F, 3, 3), f32)
        else:
            bufs["grad_faces"] = ((B, F, 3, 3), f32)
        if self.rgb:
            bufs["grad_textures"] = (tex_shape, f32)
            if self.lit and self.given:
                bufs["grad_face_light"] = ((B, F, 3), f32)
            if self.corner and self.given:
                bufs["grad_corner_light"] = ((B, F, 3, 3), f32)
            if self.uv_grad:
                bufs["grad_face_uvs"] = (uv_shape, f32)
            if self.phong and self.given:
                for k in ("corner_shading", "params", "lights", "sh"):
                    if k in bufs:
                        bufs["grad_" + k] = (bufs[k][0], f32)
            wanted = {"all": ("normal_map", "corner_tangents", "specular_map"), "texels": ("normal_map", "specular_map"),
                      "tangents": ("corner_tangents",)}.get(c["map_grads"], ())
            for k in wanted:
                if k in bufs:
                    bufs["grad_" + k] = (bufs[k][0], f32)
        if self.attr:  # attribute interpolation on the forward's maps, with gradient buffers of its own
            C, Ba = self.C, (1 if self.attr_shared else B)
            bufs["attributes"] = (((Ba, Nv, C) if self.attr_pv else (Ba, F, 3, C)), f32)
            bufs["attr_out"] = ((B, C, H, H), f32)
            bufs["attr_grad_out"] = ((B, C, H, H), f32)
            bufs["attr_grad_attributes"] = (bufs["attributes"][0], f32)
            if self.given:  # the interior vertex gradient is optional (NULL = not wanted)
                bufs["attr_grad_vertices" if self.indexed else "attr_grad_faces"] = (((B, Nv, 3) if self.indexed
                                                                                      else (B, F, 3, 3)), f32)
        self.bufs = bufs
        # textures may be NULL in the backward unless a gradient that reads them is wanted (the interior gradient reads
        # the sampler's derivative from them, the Phong gradients the unlit sample)
        self.bwd_textures = self.rgb and (self.given or self.uv_grad or "grad_face_light" in bufs or self.interior
                                          or any(k in bufs for k in MAP_GRADS))
        p = c["pointers"]
        self.offsets = {k: (0 if p == "fresh" else 4) for k in bufs}
        if p == "off8":
            for k in ("grad_textures", "grad_face_uvs", "grad_corner_light", "grad_normal_map", "grad_corner_tangents",
                      "grad_specular_map"):
                if k in bufs:
                    self.offsets[k] = 8
            if "grad_specular_map" in bufs and c["id"] % 2:  # red_add_4 splits by phase: 12 bytes in on odd ids
                self.offsets["grad_specular_map"] = 12
        if self.sm:
            self.offsets["specular_map"] = 0  # read as 16-byte vectors: the ABI demands the alignment
        self.fwd_outputs = [k for k in ("face_index_map", "weight_map", "depth_map", "rgb_map", "alpha_map", "out_rgb",
                                        "out_alpha", "out_depth") if k in bufs]
        self.grad_outputs = [k for k in ("grad_faces", "grad_vertices", "grad_textures", "grad_face_light",
                                         "grad_corner_light", "grad_face_uvs", "grad_corner_shading", "grad_params",
                                         "grad_lights", "grad_sh", "attr_grad_attributes", "attr_grad_faces",
                                         "attr_grad_vertices") + MAP_GRADS if k in bufs]

    # ---- the argument structs, from name -> address (int) of each buffer the case passes
    def forward_args(self, ptr, workspace, workspace_bytes):
        L = _lib()
        a = L.ForwardArgs()
        a.struct_size = L.ForwardArgs.corner_light.offset if self.short else ctypes.sizeof(L.ForwardArgs)
        a.flags = self.fwd_flags
        a.batch_size, a.num_faces, a.raster_size, a.texture_size = self.B, self.F, self.S, self.ts
        a.near_, a.far_, a.eps = NEAR, FAR, EPS
        a.background[0], a.background[1], a.background[2] = UNIFORM_BG
        for k in ("faces", "textures", "background_batch", "face_index_map", "weight_map", "depth_map", "rgb_map",
                  "alpha_map", "out_rgb", "out_alpha", "out_depth", "face_light", "vertices", "face_indices", "face_uvs",
                  "corner_light"):
            setattr(a, k, ptr.get(k))
        if self.short:
            a.corner_light = ptr.get("past_end_fwd")
        a.num_vertices = self.Nv if self.indexed else 0
        a.texture_height, a.texture_width = self.Ht, self.Wt
        a.workspace, a.workspace_bytes = workspace, workspace_bytes
        return a

    def backward_args(self, ptr, flags, workspace, workspace_bytes):
        L = _lib()
        a = L.BackwardArgs()
        a.struct_size = L.BackwardArgs.grad_face_uvs.offset if self.short else ctypes.sizeof(L.BackwardArgs)
        a.flags = flags
        a.batch_size, a.num_faces, a.raster_size, a.texture_size = self.B, self.F, self.S, self.ts
        a.eps = EPS
        for k in ("faces", "face_index_map", "weight_map", "depth_map", "rgb_map", "grad_rgb", "grad_alpha",
                  "grad_depth", "grad_faces", "grad_textures", "face_light", "grad_face_light", "vertices",
                  "face_indices", "grad_vertices", "face_uvs", "grad_face_uvs"):
            setattr(a, k, ptr.get(k))
        if self.short:
            a.grad_face_uvs = ptr.get("past_end_bwd")
        a.textures = ptr.get("textures") if self.bwd_textures else None
        a.num_vertices = self.Nv if self.indexed else 0
        a.texture_height, a.texture_width = self.Ht, self.Wt
        a.workspace, a.workspace_bytes = workspace, workspace_bytes
        return a

    def shading_args(self, ptr, backward):
        """(PhongArgs, LightsArgs or None, ShArgs or None) of a Phong case: None is a NULL struct.  Entry "via_sh" passes
        NULL where a mode has no struct, "via_lights_nl0" an empty light set (NL = 0, lights NULL); the gradient pointers
        only in the backward"""
        L = _lib()
        g = (lambda k: ptr.get("grad_" + k)) if backward else (lambda k: None)
        ph = L.PhongArgs()
        ph.struct_size = ctypes.sizeof(L.PhongArgs)
        ph.shading_batch, ph.params_batch = self.Bc, self.Bp
        ph.corner_shading, ph.params = ptr.get("corner_shading"), ptr.get("params")
        ph.grad_corner_shading, ph.grad_params = g("corner_shading"), g("params")
        la = sa = None
        if self.NL or self.entry == "via_lights_nl0":
            la = L.LightsArgs()
            la.struct_size = ctypes.sizeof(L.LightsArgs)
            la.lights_batch, la.num_lights = max(self.Bl, 1), self.NL
            la.lights, la.grad_lights = ptr.get("lights"), g("lights")
        if self.sh:
            sa = L.ShArgs()
            sa.struct_size = ctypes.sizeof(L.ShArgs)
            sa.sh_batch, sa.sh, sa.grad_sh = self.Bs, ptr.get("sh"), g("sh")
        return ph, la, sa

    def normal_map_args(self, ptr, backward):
        """NormalMapArgs of a case with a normal map, else None (a NULL struct); the gradient pointers only in the
        backward"""
        if not self.nm:
            return None
        L = _lib()
        na = L.NormalMapArgs()
        na.struct_size = ctypes.sizeof(L.NormalMapArgs)
        na.map_batch, na.tangent_batch, na.map_height, na.map_width = self.Bm, self.Bt, self.Hm, self.Wm
        na.normal_map, na.corner_tangents = ptr.get("normal_map"), ptr.get("corner_tangents")
        if backward:
            na.grad_normal_map, na.grad_corner_tangents = ptr.get("grad_normal_map"), ptr.get("grad_corner_tangents")
        return na

    def specular_map_args(self, ptr, backward):
        """SpecularMapArgs of a case with a specular map, else None (a NULL struct)"""
        if not self.sm:
            return None
        L = _lib()
        qa = L.SpecularMapArgs()
        qa.struct_size = ctypes.sizeof(L.SpecularMapArgs)
        qa.map_batch, qa.map_height, qa.map_width = self.Bq, self.Hq, self.Wq
        qa.specular_map = ptr.get("specular_map")
        if backward:
            qa.grad_specular_map = ptr.get("grad_specular_map")
        return qa

    def _call(self, lib, a, ptr, stream, backward):
        """the case's entry point: nr_b200_{forward,backward}_{phong,lights,sh} for the Phong modes (or _sh with NULL
        structs, or _lights with an empty set), or with a map (or map_entry "via_nm" / "via_sm" without one: NULL map
        structs) nr_b200_*_normal_map / nr_b200_*_specular_map, the narrowest that takes the structs given unless
        map_entry says otherwise; else nr_b200_forward / nr_b200_backward[_corner_light]"""
        part = "backward" if backward else "forward"
        if not self.phong:
            if backward and self.corner:
                return lib.nr_b200_backward_corner_light(ctypes.byref(a), ptr.get("corner_light"),
                                                         ptr.get("grad_corner_light"), stream)
            return getattr(lib, "nr_b200_" + part)(ctypes.byref(a), stream)
        ph, la, sa = self.shading_args(ptr, backward)
        ref = lambda s: None if s is None else ctypes.byref(s)
        if self.nm or self.sm or self.map_entry != "direct":
            na, qa = self.normal_map_args(ptr, backward), self.specular_map_args(ptr, backward)
            if self.sm or self.map_entry == "via_sm":
                return getattr(lib, "nr_b200_%s_specular_map" % part)(ctypes.byref(a), ctypes.byref(ph), ref(la), ref(sa),
                                                                      ref(na), ref(qa), stream)
            return getattr(lib, "nr_b200_%s_normal_map" % part)(ctypes.byref(a), ctypes.byref(ph), ref(la), ref(sa),
                                                                ref(na), stream)
        if self.entry == "via_sh" or self.sh:
            return getattr(lib, "nr_b200_%s_sh" % part)(ctypes.byref(a), ctypes.byref(ph), ref(la), ref(sa), stream)
        if la is not None:  # a light set, or the empty one of "via_lights_nl0"
            return getattr(lib, "nr_b200_%s_lights" % part)(ctypes.byref(a), ctypes.byref(ph), ctypes.byref(la), stream)
        return getattr(lib, "nr_b200_%s_phong" % part)(ctypes.byref(a), ctypes.byref(ph), stream)

    def call_forward(self, lib, a, ptr, stream):
        return self._call(lib, a, ptr, stream, False)

    def call_backward(self, lib, a, ptr, stream):
        return self._call(lib, a, ptr, stream, True)

    def interpolate_args(self, ptr, backward):
        """InterpolateArgs of the case's attribute interpolation (forward, or backward with its gradient buffers)"""
        L = _lib()
        a = L.InterpolateArgs()
        a.struct_size = ctypes.sizeof(L.InterpolateArgs)
        a.flags = self.attr_flags | (L.NR_GRAD_ACCUMULATE if (backward and self.accumulate) else 0)
        a.batch_size, a.num_faces, a.raster_size, a.channels = self.B, self.F, self.S, self.C
        a.faces, a.vertices, a.face_indices = ptr.get("faces"), ptr.get("vertices"), ptr.get("face_indices")
        a.num_vertices = self.Nv if self.indexed else 0
        a.face_index_map, a.weight_map, a.attributes = ptr.get("face_index_map"), ptr.get("weight_map"), ptr.get("attributes")
        if backward:
            a.grad_out, a.grad_attributes = ptr.get("attr_grad_out"), ptr.get("attr_grad_attributes")
            a.grad_faces, a.grad_vertices = ptr.get("attr_grad_faces"), ptr.get("attr_grad_vertices")
        else:
            a.out = ptr.get("attr_out")
        return a

    def backward_calls(self):
        """[(flag word, accumulate?)] of the case's backward mode, in call order"""
        L = _lib()
        base = self.flags | (L.NR_GRAD_INTERIOR if self.interior else 0)
        acc = L.NR_GRAD_ACCUMULATE
        tex, faces = L.NR_BWD_PART_TEXTURES, L.NR_BWD_PART_FACES
        return {"one": [base], "tex_faces": [base | tex, base | faces], "faces_tex": [base | faces, base | tex],
                "acc_one": [base | acc], "acc_halves": [base | acc | tex, base | acc | faces]}[self.case["backward"]]

    @property
    def accumulate(self):
        return self.case["backward"].startswith("acc")

    def fake_pointers(self):
        """distinct non-NULL addresses with the case's offsets (host argument checks only: never dereferenced)"""
        return {k: 0x10000000 * (i + 1) + self.offsets[k] for i, k in enumerate(sorted(self.bufs))}


def make_inputs(plan, seed):
    """seeded numpy inputs of a case: the arrays the ABI calls read, plus `faces_mat` (the materialised fp32 faces)"""
    from neural_renderer_b200 import synthetic
    rng = np.random.default_rng(1000 + seed)
    B, F, Nv = plan.B, plan.F, plan.Nv
    verts, idx = synthetic.sphere_mesh(plan.F_front)
    if plan.fill_back:
        idx = np.concatenate((idx, idx[:, ::-1]), axis=0)
    v = np.empty((B, Nv, 3), np.float32)
    for b in range(B):
        vb = (verts * 0.8) @ synthetic._rotation(rng).T + rng.normal(scale=0.01, size=verts.shape)
        vb[:, 2] += 2.75
        v[b] = vb.astype(np.float32)
    d = {}
    if plan.indexed:
        if plan.idx_shared:
            ind = idx.astype(np.int32)
            if plan.case["geometry"] == "idx_shared_oor":  # about 3 % of the indices out of range, both sides
                sel = rng.random(ind.shape) < 0.03
                ind = np.where(sel, rng.choice(np.array([-1, -5, Nv, Nv + 7, 1 << 30], np.int32), size=ind.shape), ind)
            d["face_indices"] = np.ascontiguousarray(ind, np.int32)
            d["vertices"] = v
            full = np.broadcast_to(ind, (B,) + ind.shape)
        else:  # every item lists its vertices in its own order
            vv = np.empty_like(v)
            ind = np.empty((B,) + idx.shape, np.int32)
            for b in range(B):
                perm = rng.permutation(Nv)
                vv[b, perm] = v[b]
                ind[b] = perm[idx]
            d["vertices"], d["face_indices"] = vv, ind
            full = ind
        valid = (full >= 0) & (full < Nv)
        vsrc = d["vertices"]
        d["faces_mat"] = np.where(valid[..., None], vsrc[np.arange(B)[:, None, None], np.clip(full, 0, Nv - 1)], 0).astype(np.float32)
        if "faces" in plan.bufs:
            d["faces"] = np.full((B, F, 3, 3), np.nan, np.float32)  # must be ignored
    else:
        d["faces"] = np.ascontiguousarray(v[:, idx])
        d["faces_mat"] = d["faces"]
    if "textures" in plan.bufs:
        d["textures"] = rng.random(plan.bufs["textures"][0], dtype=np.float32)
    if "face_light" in plan.bufs:
        d["face_light"] = (0.5 + rng.random((B, F, 3))).astype(np.float32)
    if "corner_light" in plan.bufs:
        d["corner_light"] = (0.3 + 0.9 * rng.random((B, F, 3, 3))).astype(np.float32)
    if "face_uvs" in plan.bufs:
        shape = plan.bufs["face_uvs"][0]
        if plan.mip:  # per-face spread from 1e-3 to 100: magnified, fractional and last-level LODs
            centre = rng.random(shape[:-2] + (1, 2))
            spread = 10.0 ** (-3 + 5 * rng.random(shape[:-2] + (1, 1)))
            d["face_uvs"] = (centre + spread * (rng.random(shape) - 0.5)).astype(np.float32)
        else:
            d["face_uvs"] = (-0.2 + 1.4 * rng.random(shape)).astype(np.float32)
    if "background_batch" in plan.bufs:
        d["background_batch"] = rng.random((B, 3), dtype=np.float32)
    for k in ("grad_rgb", "grad_alpha", "grad_depth", "attr_grad_out"):
        if k in plan.bufs:
            d[k] = rng.standard_normal(plan.bufs[k][0]).astype(np.float32)
    if "attributes" in plan.bufs:
        d["attributes"] = (2.0 + rng.standard_normal(plan.bufs["attributes"][0])).astype(np.float32)
    for k in ("past_end_fwd", "past_end_bwd"):
        if k in plan.bufs:
            d[k] = np.full(plan.bufs[k][0], np.nan, np.float32)
    if plan.phong:
        phong_inputs(plan, d, np.random.default_rng(3000 + seed))
    if plan.nm or plan.sm:
        map_inputs(plan, d, np.random.default_rng(7000 + seed))
    return d


# the light records of the Phong cases (nr_b200_lights_args: D, K, x, falloff, kind), the first NL of them: directional
# and point lights on the viewer's side, two of them far enough off the axis that part of the sphere lies in their shadow
# (c_j < 0), the point lights with and without falloff.  Item b's positions / directions are shifted by 0.05 b.
LIGHTS = [[0.5, 0.4, 0.3, 0.3, 0.35, 0.4, 0.2, -0.3, -1.0, 0.0, 0.0, 0.0],
          [0.3, 0.45, 0.35, 0.5, 0.3, 0.2, 0.6, 0.4, -1.5, 0.4, 1.0, 0.0],
          [0.25, 0.2, 0.4, 0.2, 0.25, 0.3, -0.9, 0.35, -0.6, 0.0, 0.0, 0.0],
          [0.4, 0.3, 0.2, 0.35, 0.3, 0.25, -0.5, -0.6, -1.0, 0.0, 1.0, 0.0],
          [0.2, 0.3, 0.25, 0.3, 0.2, 0.35, 0.1, 0.8, -1.0, 0.0, 0.0, 0.0],
          [0.35, 0.25, 0.3, 0.25, 0.4, 0.3, 1.2, -0.15, 0.5, 0.15, 1.0, 0.0],
          [0.15, 0.2, 0.3, 0.4, 0.35, 0.3, -0.3, 0.1, -1.0, 0.0, 0.0, 0.0],
          [0.3, 0.2, 0.15, 0.2, 0.3, 0.25, 0.2, 0.5, -0.8, 0.8, 1.0, 0.0]]


def phong_inputs(plan, d, rng):
    """the Phong inputs of a case: corner_shading [Bc,F,3,6] -- the sphere's normals at the materialised corners
    (perturbed, turned towards the viewer at -z; the fill_back copies get the negated normal, as the header asks of
    callers) and the corners themselves as positions --, params [Bp,16], the first NL of LIGHTS [Bl,NL,12] and an SH
    environment [Bs,9,3] (bright and coloured, direction-dependent)"""
    from oracles_sh import C0
    B, F, Ff = plan.B, plan.F, plan.F_front
    pos = d["faces_mat"][:plan.Bc].astype(np.float64)
    centre = np.array([0.0, 0.0, 2.75])
    n = pos - centre
    n = n / (np.linalg.norm(n, axis=-1, keepdims=True) + 1e-6) + 0.15 * rng.standard_normal(pos.shape)
    n[..., 2] = -(np.abs(n[..., 2]) + 0.5)
    if plan.fill_back:
        n[:, Ff:] = -n[:, Ff:]
    d["corner_shading"] = np.ascontiguousarray(np.concatenate((n, pos), axis=-1), np.float32)
    rows = [[0.3, 0.25, 0.2, 0.6, 0.7 - 0.05 * b, 0.8, 0.3, 0.4 + 0.1 * b, -1.0, 0.6, 0.5, 0.4, plan.sigma,
             0.2, -0.1 - 0.05 * b, -0.5] for b in range(plan.Bp)]
    d["params"] = np.array(rows, np.float32)
    if plan.NL:
        lt = np.array([LIGHTS[:plan.NL]] * plan.Bl, np.float64)
        lt[..., 6:9] += 0.05 * np.arange(plan.Bl)[:, None, None]
        d["lights"] = lt.astype(np.float32)
    if plan.sh:
        base = 0.25 * rng.standard_normal((9, 3))
        base[0] = np.array([0.8, 0.7, 0.6]) / C0
        d["sh"] = np.stack([base + 0.05 * b for b in range(plan.Bs)]).astype(np.float32)


def map_inputs(plan, d, rng):
    """the map inputs of a case (from a generator of their own, so the other inputs keep their bits): normal_map
    [Bm,Hm,Wm,3] -- decoded unit vectors tilted up to 30 degrees from +z, every item its own --, corner_tangents
    [Bt,F,3,4] -- across the corner normals, two faces in five with handedness -1 and one in seven with mixed signs over
    its corners (the majority vote decides), the fill_back copies (-T, -w) at their reversed corners --, and specular_map
    [Bq,Hq,Wq,4] -- ks in [0.2, 1], shininess in [4, 24]; with fill_back every other copy then takes its normal back to
    the viewer's side.  With a specular map params' shininess is NaN: the header pins
    that a pixel shaded through the map never reads it, and a read would show in the image and in every gradient."""
    Ff = plan.F_front
    if plan.nm:
        shape = (plan.Bm, plan.Hm, plan.Wm)
        tilt, turn = np.radians(30.0) * np.sqrt(rng.random(shape)), 2 * np.pi * rng.random(shape)
        m = np.stack((np.sin(tilt) * np.cos(turn), np.sin(tilt) * np.sin(turn), np.cos(tilt)), axis=-1)
        d["normal_map"] = np.ascontiguousarray(m, np.float32)
        n = d["corner_shading"][..., :3].astype(np.float64)
        n = n[[min(b, n.shape[0] - 1) for b in range(plan.Bt)], :Ff]
        t = np.cross(n, np.array([0.3, 1.0, 0.2]) + 0.2 * rng.standard_normal(n.shape))
        t = t / np.linalg.norm(t, axis=-1, keepdims=True) + 0.1 * rng.standard_normal(n.shape)
        w = np.where(rng.random((plan.Bt, Ff, 1)) < 0.4, -1.0, 1.0) * np.ones((1, 1, 3))
        mixed = rng.random((plan.Bt, Ff)) < 1 / 7
        corner = rng.integers(0, 3, (plan.Bt, Ff))
        w[mixed, corner[mixed]] *= -1.0
        tg = np.concatenate((t, w[..., None]), axis=-1)
        if plan.fill_back:
            tg = np.concatenate((tg, -tg[:, :, ::-1]), axis=1)
        d["corner_tangents"] = np.ascontiguousarray(tg, np.float32)
    if plan.sm:
        shape = (plan.Bq, plan.Hq, plan.Wq)
        q = np.concatenate((0.2 + 0.8 * rng.random(shape + (3,)), 4.0 + 20.0 * rng.random(shape + (1,))), axis=-1)
        d["specular_map"] = np.ascontiguousarray(q, np.float32)
        d["params"][:, 12] = np.nan
        if plan.fill_back:
            # a copy's negated normal faces away from the viewer and the lights, so no copy would carry a highlight and
            # the specular map's gradient and UV term would be 0 on every copy's pixel (`rev` in sm_grad_tail unseen):
            # every other copy keeps its front face's side, as a two-sided material would
            d["corner_shading"][:, Ff::2, :, :3] *= -1.0


def stage_runs(plan):
    """whether the forward stages texture cubes (the predicate of nr_b200_forward; Phong ignores the flag), and the
    slots per row segment"""
    if not (plan.rgb and plan.case["stage"] and not plan.uv and not plan.corner and not plan.phong and not plan.aa):
        return False, 0
    cube_bytes = plan.ts ** 3 * 12
    ok = cube_bytes % 16 == 0 and cube_bytes <= K_STAGE_BYTES // 8 and plan.offsets["textures"] % 16 == 0
    bx = 256 if plan.S >= 256 else (plan.S + 31) // 32 * 32
    return ok, min(K_STAGE_BYTES // cube_bytes, bx)


# ---- device side
GUARD_WORDS = 4          # 16 bytes of guard before (keeps the data's 16-byte phase) and at least 16 after every buffer
GUARD_BITS = 0x7FBADBAD  # a NaN payload no kernel stores (and no face index)


def alloc(shape, dtype, offset_bytes, dev):
    """a tensor of `shape` whose data starts `offset_bytes` past a 16-byte boundary inside a fresh allocation (the
    allocator's blocks are 512-byte aligned), between guard words that guards_intact() checks after the calls: a store
    just before or past a buffer -- a tail store of the side fill, an overrunning vector reduction -- fails the case.
    The view keeps the allocation alive (it is t._base)."""
    import torch
    tdt = {np.float32: torch.float32, np.int32: torch.int32}[dtype]
    n = int(np.prod(shape))
    assert offset_bytes % 4 == 0 and offset_bytes < 16
    lo = GUARD_WORDS + offset_bytes // 4
    base = torch.empty(lo + n + GUARD_WORDS, dtype=tdt, device=dev)
    base.view(torch.int32).fill_(GUARD_BITS)
    assert base.data_ptr() % 16 == 0
    t = base[lo:lo + n].view(shape)
    assert t.data_ptr() % 16 == offset_bytes % 16
    return t


def guards_intact(t):
    """whether the guard words around a buffer from alloc() still hold their pattern"""
    import torch
    base = t._base
    lo = (t.data_ptr() - base.data_ptr()) // t.element_size()
    bits = base.view(torch.int32)
    return bool((bits[:lo] == GUARD_BITS).all()) and bool((bits[lo + t.numel():] == GUARD_BITS).all())


def poison(t):
    import torch
    if t.dtype == torch.int32:
        t.fill_(FIM_SENTINEL)
    else:
        t.fill_(float("nan"))


def workspace(nbytes, dev):
    import torch
    ws = torch.empty((max(int(nbytes), 16),), dtype=torch.uint8, device=dev)
    assert ws.data_ptr() % 16 == 0
    return ws


def forward(plan, buf, dev):
    """poison the forward outputs, call the case's forward entry point on the current stream, return the return code"""
    import torch
    L = _lib()
    lib = L.load()
    for k in plan.fwd_outputs:
        poison(buf[k])
    nbytes = lib.nr_b200_forward_workspace_bytes(plan.B, plan.F, plan.S, plan.ts, plan.fwd_flags)
    ws = workspace(nbytes, dev)
    ptr = {k: t.data_ptr() for k, t in buf.items()}
    a = plan.forward_args(ptr, ws.data_ptr(), ws.numel())
    rc = plan.call_forward(lib, a, ptr, ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream))
    torch.cuda.synchronize(dev)
    return rc


def backward(plan, buf, dev):
    """the case's backward calls in order; [return codes].  The caller prepares the gradient buffers: poisoned, or
    prefilled when the mode accumulates."""
    import torch
    L = _lib()
    lib = L.load()
    out = []
    ptr = {k: t.data_ptr() for k, t in buf.items()}
    stream = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    for flags in plan.backward_calls():
        nbytes = lib.nr_b200_backward_workspace_bytes(plan.B, plan.F, plan.S, plan.ts, flags)
        ws = workspace(nbytes, dev)
        a = plan.backward_args(ptr, flags, ws.data_ptr(), ws.numel())
        out.append(plan.call_backward(lib, a, ptr, stream))
    torch.cuda.synchronize(dev)
    return out


def interpolate(plan, buf, dev):
    """poison the attribute image, call nr_b200_interpolate on the saved maps, return the return code"""
    import torch
    lib = _lib().load()
    poison(buf["attr_out"])
    a = plan.interpolate_args({k: t.data_ptr() for k, t in buf.items()}, False)
    rc = lib.nr_b200_interpolate(ctypes.byref(a), ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream))
    torch.cuda.synchronize(dev)
    return rc


def interpolate_backward(plan, buf, dev):
    """nr_b200_interpolate_backward (NR_GRAD_ACCUMULATE when the case's backward mode accumulates); the caller prepares
    the gradient buffers as for backward()"""
    import torch
    lib = _lib().load()
    a = plan.interpolate_args({k: t.data_ptr() for k, t in buf.items()}, True)
    rc = lib.nr_b200_interpolate_backward(ctypes.byref(a), ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream))
    torch.cuda.synchronize(dev)
    return rc
