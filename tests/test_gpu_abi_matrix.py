"""GPU: every pair of the C-ABI flag levels of the rasterizer (forward, backward, smooth-shading backward, the three
Phong modes, the normal map and the specular map through each of their entry points) and of the attribute interpolation on its maps, called directly (tests/abi_harness.py), held to an unfused oracle.

The cases come from the covering array of tests/abi_cases.py.  The oracle never runs the product's fused paths:
  cubes       the inputs are materialised as a float64 torch function of (vertices | faces, textures, light) -- faces by
              gather (out-of-range indices read zeros), shared textures expanded, fill_back as
              cat(t, t.permute(0,1,4,3,2,5)), the light multiplied in (in fp32 for the forward: the header pins the fused
              light as bit-identical to sampling the product) -- and rendered by the CPU oracle (oracle/nr_oracle.py,
              with per-item background and the batch-0 depth quirk as flagged; K5 summed in float64).  Its face /
              texture gradients are chained back to vertices, textures and light by float64 autograd.  NR_FWD_STAGE_TEXTURES
              changes nothing here: a staged render is held bit-exact like any other.
  images      the float64 samplers of tests/oracles.py on the materialised geometry (bilinear, or trilinear on the
              packed pyramid passed as `textures`); the face / vertex gradient from the CPU oracle's K5 fed with the
              product's own raster rgb map.  grad_face_uvs from the straight-through samplers of tests/oracles_uv_grad.py,
              the fill_back fold and the sum over items of shared UVs by autograd.
  smooth      corner_light: the light oracles_smooth.smooth_light64 (each item's own depths, on the maps) times the unlit
              sample -- for cubes the CPU oracle's unlit render (bit-exact, NR_TEX_Z_BATCH0 honoured), for images the
              samplers above; grad_corner_light by float64 autograd of that image, the cube texture gradient from the
              CPU oracle's K6 sampling maps fed the raster upstream gradient times the light (summed in float64: the
              fp32 sums of the oracle's own K6 are up to 3e-5 per element off there), K5 fed the product's lit rgb map.
  attributes  oracles_attr.interp64 on the float64 materialised faces (fill_back copies included) and corner
              attributes gathered in float64 (out-of-range indices read zeros), at the product's weights; the attribute
              and interior vertex gradients by autograd back through the gathers.  A face with an out-of-range corner
              (a zero vertex: z = 0 puts zp below near) must never win a pixel, and that is checked.
  phong       the three Phong modes (nr_b200_{forward,backward}_{phong,lights,sh}, or _sh with NULL structs, or _lights
              with an empty set): the light L and the specular colour of oracles_sh.sh_terms64 (every mode) in float64 on
              the materialised faces and the product's maps, times the unlit sample as for corner light -- the CPU
              oracle's unlit cube render, or the float64 samplers -- plus the specular colour.  grad_corner_shading,
              grad_params, grad_lights and grad_sh by float64 autograd of that image; the cube texture gradient from K6
              fed g L, the image / pyramid and UV gradients through the samplers with L (and the specular colour) held.
              No Phong kernel is called.  A covered pixel within 1e-5 of a highlight's switch c_j = 0 (K_j != 0) fails
              the case as a fault of its inputs (near_kinks), and the inputs are chosen so that there is none.  Shading
              gradients that are 0 in the oracle must come back exactly 0 from a fresh call.
  maps        a normal map, a specular map or both (nr_b200_{forward,backward}_{normal_map,specular_map}, also with NULL
              map structs under the three Phong modes): the image is oracles_specular_map.sm_rgb64 on the product's maps
              and the float64 unlit sample of the Phong rows -- the mapped normal n', the map's (ks, sigma') in every
              highlight.  Every gradient by float64 autograd of that image: the shading inputs, the maps, the tangents,
              the image / pyramid, and grad_face_uvs with the UVs feeding the straight-through albedo sampler and the map
              samplers at once (the two terms add).  No Phong kernel is called.  The highlights' switches are those of n'
              (near_kinks).  params' shininess is NaN next to a specular map: the header pins that it is not read, and
              no row shows a trace of it (grad_params[12] comes back exactly 0).  grad_corner_tangents' handedness slots
              and every texel no pixel samples must come back exactly 0 (the prefill bit for bit when accumulating).
              Without a map through nr_b200_*_normal_map / _specular_map the forward's maps must equal, bit for bit,
              those of the direct call.
  interior    NR_GRAD_INTERIOR: float64 autograd of oracles_interior.rgb_held64 (the lit sample with the cell, level of
              detail and clamp gates held fixed) in the materialised faces, on the product's maps and the case's own
              cubes / image / unpacked pyramid, UVs and light, times the raster upstream gradient; added to the CPU
              oracle's K5 / K7 face gradient before the chain to the vertices.  Its sample must match the reference
              rgb_map at the covered pixels at the image gate, so it differentiates the image that was rendered.
Gates: face_index_map, weight_map and depth_map bit-exact; images bit-exact in non-anti-aliased, unlit or flat-lit cube
mode, 1e-5 relative elsewhere (2e-5 for Phong at sigma 16); every gradient tensor 1e-4 per tensor (helpers.rel_err) and per element (helpers.elem_err),
with the exceptions of the feature tests (test_gpu_smooth.py, test_gpu_uv_grad.py, test_gpu_attr.py, test_gpu_interior.py,
with their causes there; and test_gpu_phong.py, test_gpu_lights.py, test_gpu_sh.py for the Phong rows: per element
grad_corner_shading 2e-3, grad_params 5e-4, grad_lights 2e-4, grad_sh 1e-4): the trilinear sampler's image and
per-element gradients, the attribute image (1e-6), the
attribute gradient per tensor (1e-5), and the interior vertex gradients per element (2.5e-3) -- the interpolation's, and
grad_faces / grad_vertices of a case with NR_GRAD_INTERIOR and an rgb upstream gradient.
Measured maxima over this matrix (194 cases, 17 with NR_GRAD_INTERIOR) on an H100 80GB HBM3 at 400 W, per gate:
  raster / anti-aliased image, trilinear   4.4e-5 / 5.1e-6 (cases 101, 116)    gate 6e-5
  raster / anti-aliased image, smooth      1.6e-7 / 1.4e-7                      gate 1e-5
  pyramid gradient per element             3.6e-4 (case 101)                    gate 5e-4
    case 192 at the float64 / fp32 LOD     5.8e-4 / 2e-5 (TOL_GRAD_ELEM_MIP)    gate 5e-4 at the fp32 LOD
  grad_corner_light per tensor / element   4.9e-7 / 3.9e-5; trilinear 5.4e-5   gates 1e-4 / 1e-4, 5e-4
  grad_face_uvs per tensor / element       8.6e-7 / 4.1e-5; trilinear 7.1e-4   gates 1e-4 / 1e-4, 1.5e-3
    trilinear: case 192, face 50 of item 1, the pyramid gradient's fp32-LOD pixel; 1.1e-5 at the fp32 LOD
  attribute image                          2.3e-7                               gate 1e-6
  attribute gradient per tensor / element  9.8e-7 / 6.0e-5                      gates 1e-5 / 1e-4
  interpolation's interior vertex gradient 6.1e-5 / 1.5e-3 (case 129)           gates 1e-4 / 2.5e-3
  NR_GRAD_INTERIOR grad_vertices t / elem  2.3e-6 / 4.7e-4 (cases 185, 186)     gates 1e-4 / 2.5e-3
  NR_GRAD_INTERIOR grad_faces t / elem     9.0e-7 / 5.2e-5 (case 187)           gates 1e-4 / 2.5e-3
  its sample vs the reference rgb_map      6.0e-6; trilinear 8.6e-6 (185, 189)  gates 1e-5, 6e-5
  every other gradient per element         9.5e-5 (case 136; with NR_GRAD_ACCUMULATE 7.5e-5)
Measured maxima of the 77 Phong rows (cases 194-270) on an H100 80GB HBM3 at 700 W, per gate:
  image / anti-aliased image, sigma 1      4.1e-7 / 2.0e-7 (cases 218, 213)      gate 1e-5
  image / anti-aliased image, sigma 16     3.9e-6 / 1.6e-6 (cases 199, 201)      gate 2e-5
  image, trilinear                         6.2e-6 (case 241)                     gate 6e-5
  grad_corner_shading per tensor / elem    3.7e-6 / 8.3e-4 (cases 255, 259)      gates 1e-4 / 2e-3
  grad_params per tensor / element         2.0e-6 / 4.8e-4 (cases 206, 259)      gates 1e-4 / 5e-4
    case 259 over three runs                 4.7e-4 to 5.0e-4 (TOL_PARAMS_ELEM_259)  gate 6e-4 for that row
  grad_lights per tensor / element         2.3e-6 / 1.7e-4 (cases 245, 255)      gates 1e-4 / 2e-4
  grad_sh per tensor / element             6.2e-7 / 8.1e-5 (cases 239, 238)      gates 1e-4 / 1e-4
  grad_textures per element                6.1e-5; trilinear 3.0e-4 (219, 241)   gates 1e-4, 5e-4
  grad_face_uvs per element                4.7e-5; trilinear 1.1e-4 (204, 240)   gates 1e-4, 1.5e-3
  grad_faces per element                   2.1e-4 (case 214, TOL_GRAD_ELEM_214); 8.5e-5 elsewhere (case 229)
Measured maxima of the 106 map rows (cases 271-376) on an H100 80GB HBM3 at 700 W, per gate:
  image / anti-aliased image, no specular  3.9e-7 / 2.1e-7 (cases 372, 344)      gate 1e-5
  image / anti-aliased image, sigma > 1    3.4e-6 / 1.4e-6 (case 275)            gate 2e-5
  image, trilinear                         2.1e-5 (case 328)                     gate 6e-5
  grad_normal_map per tensor / element     6.8e-6 / 1.0e-3 (cases 303, 333)      gates 1e-4 / 2e-3
  grad_corner_tangents per tensor / elem   6.0e-6 / 7.1e-4 (case 303)            gates 1e-4 / 2e-3
  grad_specular_map per tensor / element   9.1e-6 / 6.6e-4 (cases 312, 314)      gates 1e-4 / 1.5e-3
  grad_corner_shading per tensor / elem    5.6e-6 / 9.1e-4 (cases 277, 283)      gates 1e-4 / 2e-3
  grad_params per tensor / element         1.7e-6 / 9.1e-4 (cases 291, 331)      gates 1e-4 / 2e-3 (5e-4 without a map)
  grad_lights per tensor / element         2.6e-6 / 2.4e-4 (cases 345, 296)      gates 1e-4 / 6e-4 (2e-4 without a map)
  grad_sh per tensor / element             7.0e-7 / 1.2e-4 (case 313)            gates 1e-4 / 3e-4 (1e-4 without a map)
  grad_face_uvs per element                3.8e-4; trilinear 5.0e-4 (333, 296)   gates 1e-3 (1e-4 without a map), 1.5e-3
  grad_textures per element                5.7e-5; trilinear 3.9e-4 (337, 282)   gates 1e-4, 5e-4
  grad_faces / grad_vertices per element   9.0e-5 / 2.6e-5 (cases 312, 283)      gate 1e-4
  With the gates the rows without a map have, six map rows were over per element and under 2e-6 per tensor: grad_face_uvs
  in 293, 304, 333 (2.1e-4 to 3.8e-4), grad_sh in 313, grad_params in 331, grad_lights in 296; the cause is at
  MAP_ROW_ELEM below.  The 377 cases take 26.5 s in one process on that H100 (9.3 s of it the 106 map rows), 34.3 s under pytest.
Every output is poisoned before a call (NaN, face-index sentinel), so an element the kernels do not write fails, and
guard words around every buffer must survive the calls, so a store just outside one fails; with NR_GRAD_ACCUMULATE the
gradients are prefilled with seeded values and must come back as prefill + fresh gradient, the prefill untouched bit for
bit wherever the oracle's fresh gradient is exactly 0.  With a short struct layout the field past its end points at a
NaN-filled buffer that must come back bit for bit (and would light the forward image with NaN if read)."""
import numpy as np
import pytest
import torch

import abi_cases
import abi_harness as H
from helpers import elem_err, rel_err

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda")
TOL_GRAD = 1e-4
TOL_IMAGE = 1e-5
# NR_TEX_MIPMAP relaxes two gates.  The product evaluates the level of detail in fp32 (include/nr_b200.h), the oracle in
# float64 (oracles.lod64), and the pyramid here is random data, so neighbouring levels differ by O(1) and a pixel's colour
# moves by about its LOD difference; a texel whose gradient comes only through a small blend weight f (or 1 - f) sees
# the same absolute difference relative to its own size (measured maxima in the module docstring).  The fp32 LOD loses
# up to 7e-5 to cancellation in d l_k / dx with this matrix's UV spread (1e-3 to 100): in case 192 a level-2 texel of
# item 1 takes its gradient through 1 - f = 0.12 at pixel (30, 58) (face 50), whose LOD is 2.884151 in float64 and
# 2.884083 in fp32, and the pyramid gradient is 5.8e-4 off per element.  So where the pyramid gradient exceeds
# TOL_GRAD_ELEM_MIP against the float64-LOD oracle, it must pass the same gate against the oracle at the fp32 LOD of the
# header's expression (oracles.lod32), which removes that part (about 2e-5 there); the per-tensor gate stays on float64.
TOL_IMAGE_MIP = 6e-5
TOL_GRAD_ELEM_MIP = 5e-4
# the gates of the smooth-shading, face_uvs-gradient and attribute tests (test_gpu_smooth.py, test_gpu_uv_grad.py,
# test_gpu_attr.py, with their causes there); measured maxima over this matrix in the module docstring
TOL_CORNER_ELEM_MIP = 5e-4   # grad_corner_light per element with NR_TEX_MIPMAP
TOL_UV_ELEM_MIP = 1.5e-3     # grad_face_uvs per element with NR_TEX_MIPMAP
TOL_ATTR_IMAGE = 1e-6        # interpolated attribute image
TOL_ATTR = 1e-5              # attribute gradient per tensor (per element TOL_GRAD)
TOL_INTERIOR = 1e-4          # interior vertex gradient of the interpolation per tensor
TOL_INTERIOR_ELEM = 2.5e-3   # and per element
# the gates of the Phong, light-set and SH tests (test_gpu_phong.py, test_gpu_lights.py, test_gpu_sh.py, with their causes
# there): the image at sigma > 1 (q^sigma multiplies the fp32 relative error of q by sigma), and the shading gradients per
# element
TOL_IMAGE_SIGMA = 2e-5
TOL_CS_ELEM = 2e-3           # grad_corner_shading
TOL_PARAMS_ELEM = 5e-4       # grad_params
TOL_LIGHTS_ELEM = 2e-4       # grad_lights
TOL_SH_ELEM = 1e-4           # grad_sh
# The maps' gradients per element, and the gates of three older outputs in a row that carries a map; measured maxima in
# the module docstring, every gate within three times its maximum and none looser than TOL_CS_ELEM.  The cause is
# TOL_CS_ELEM's: the highlight's gradient carries q^(sigma - 1) sigma, so the fp32 error of q comes back times the
# shininess -- up to 24 from a specular map, whatever params' sigma says -- and a normal map puts the tangent frame (a
# cross product of rounded products and three more fmas) in front of the normalisation that q is built on.  The map's UV
# term l_k (gu, gv) is made of that same normal gradient g' (gm = (g'.t, g'.b, g'.n)), so with a map grad_face_uvs carries
# the shading chain's per-element error next to the sampler's; grad_params, grad_lights and grad_sh see the mapped
# normal and the map's shininess through q and through the SH basis.  Every one of these goes with a per-tensor error below 1e-5, and the rows without a map
# keep the gates they had.
TOL_NM_ELEM = 2e-3           # grad_normal_map
TOL_TG_ELEM = 2e-3           # grad_corner_tangents
TOL_SM_ELEM = 1.5e-3         # grad_specular_map
# with a map (trilinear UVs keep TOL_UV_ELEM_MIP)
MAP_ROW_ELEM = {"grad_face_uvs": 1e-3, "grad_params": 2e-3, "grad_lights": 6e-4, "grad_sh": 3e-4}
KINK = 1e-5                  # |c_j| below this at a covered pixel: the highlight's switch [c_j > 0] is within fp32 reach
# Case 214 (cube_shared ts 6, light set NL = 8, rgb + depth) has a face gradient whose largest element is 3437: element
# [0, 43, 2, 0] (face 43 of item 0, corner 2, x) comes back 3.005895 against 3.005173 in float64 -- 7.2e-4 absolute,
# 2.1e-7 of the tensor's maximum, elem_err 2.1e-4.  It is the edge scan K5's fp32 sums on the lit rgb map: the same call
# without the rgb upstream gradient gives 2.2e-6, three runs give the same bits (run-to-run spread 5e-6), and the
# per-tensor error is 2.8e-7.  That one face gradient is held at TOL_GRAD_ELEM_214; every other row keeps TOL_GRAD.
TOL_GRAD_ELEM_214 = 2.5e-4
# Case 259 (bilinear image, Phong through an empty light set, sigma 16, three items, accumulating halves) sets the
# grad_params maximum of the table above, and its fp32 atomics land in another order from run to run: three runs of the
# same bits of input on one H100 gave 4.68e-4, 4.81e-4 and just over 5.0e-4 per element (1.4e-6 to 1.5e-6 per tensor), the
# last one over TOL_PARAMS_ELEM.  That one gradient is held at TOL_PARAMS_ELEM_259; every other row keeps 5e-4.
TOL_PARAMS_ELEM_259 = 6e-4
# Case 229 (cube_shared ts 6, SH with one light, accumulating) sets the grad_faces maximum outside case 214, and it too
# moves with the order of K5's fp32 atomics: 8.5e-5 and 7.6e-5 per element in two runs on one H100, and over TOL_GRAD in a
# third whose value was not kept.  Held at TOL_GRAD_ELEM_229; the cause is case 214's, at a smaller size.
TOL_GRAD_ELEM_229 = 1.5e-4
# Case 273 (shared image and UVs, Phong with SH through a normal map, sigma 16, fill_back) has an image gradient whose
# largest element is 41.1, summed by fp32 atomics whose order changes from run to run.  Six runs of the same input on
# one H100 (700 W) gave 1.3e-4, 1.1e-4, 5.0e-5, 1.1e-4, 7.2e-6 and 5.0e-5 per element -- a few ulps of the largest
# addend, 5e-6 absolute, on an element below 1e-3 of the maximum -- and 2.3e-7 to 4.5e-7 per tensor.  That one gradient is held at TOL_TEX_ELEM_273; every other row keeps TOL_GRAD.
TOL_TEX_ELEM_273 = 2.5e-4
PHONG_INPUTS = ("corner_shading", "params", "lights", "sh")
MAP_INPUTS = ("normal_map", "corner_tangents", "specular_map")
CASES = abi_cases.cases()


def materialise(plan, d, geom, tex, light):
    """(faces [B,F,3,3], cube textures [B,F,ts,ts,ts,3] with light) as a torch function of the case's inputs, in their
    dtype: fp32 for the oracle's forward, float64 with autograd for the chain of its gradients"""
    B, F = plan.B, plan.F
    if plan.indexed:
        ind = torch.from_numpy(d["face_indices"].astype(np.int64)).expand(B, F, 3)
        valid = ((ind >= 0) & (ind < plan.Nv))[..., None]
        g = geom[torch.arange(B)[:, None, None], ind.clamp(0, plan.Nv - 1)]
        faces = torch.where(valid, g, torch.zeros((), dtype=geom.dtype))
    else:
        faces = geom
    cubes = None
    if tex is not None and plan.kind in ("cube", "cube_shared"):
        cubes = tex.expand(B, -1, -1, -1, -1, -1)
        if plan.fill_back:
            cubes = torch.cat((cubes, cubes.permute(0, 1, 4, 3, 2, 5)), dim=1)
        if light is not None:
            cubes = cubes * light[:, :, None, None, None, :]
    return faces, cubes


def _upsample(g, aa):
    """API-layout upstream gradient -> the raster gradient the backward sees (pooling: each raster pixel gets g / 4)"""
    return g.repeat_interleave(2, -1).repeat_interleave(2, -2) * 0.25 if aa else g


def _k6_64(fn, G):
    """the CPU oracle's texture backward (K6: each covered raster pixel sends weight x upstream gradient to the 8 texels
    its sample blended, through the oracle's sampling maps), summed in float64; G [B,S,S,3] raster layout, float64"""
    B, F, ts = fn.batch_size, fn.num_faces, fn.texture_size
    out = np.zeros((B, F, ts ** 3, 3))
    fim = fn.face_index_map.reshape(B, -1)
    w = fn.sampling_weight_map.reshape(B, -1, 8).astype(np.float64)
    idx = fn.sampling_index_map.reshape(B, -1, 8)
    g = np.asarray(G, np.float64).reshape(B, -1, 3)
    for b in range(B):
        cov = fim[b] >= 0
        np.add.at(out[b], (np.repeat(fim[b][cov], 8), idx[b][cov].reshape(-1)),
                  (w[b][cov][..., None] * g[b][cov][:, None, :]).reshape(-1, 3))
    return out.reshape(fn.textures.shape)


def oracle(plan, d, got):
    """(forward reference {name: tensor in the product's layout}, fresh gradients {buffer name: float64 numpy})"""
    import nr_oracle
    from oracles import lod32, oracle_rgb, oracle_trilinear_levels, unpack_pyramid
    from oracles import _bg
    from oracles_sh import sh_terms64
    from oracles_specular_map import sm_rgb64
    from oracles_smooth import smooth_light64, smooth_rgb
    from oracles_uv_grad import oracle_rgb_uv_grad, oracle_trilinear_levels_uv_grad
    B, S = plan.B, plan.S
    t = lambda k, dt=torch.float32: torch.from_numpy(np.ascontiguousarray(d[k])).to(dt) if k in d else None
    geom_key = "vertices" if plan.indexed else "faces"
    faces32, cubes32 = materialise(plan, d, t(geom_key), t("textures"), t("face_light"))
    cube = cubes32 is not None
    bg = d["background_batch"] if plan.bg_batch and plan.rgb else np.array(H.UNIFORM_BG, np.float32)
    tex_in = cubes32.numpy() if cube else (np.zeros((B, plan.F, 2, 2, 2, 3), np.float32) if plan.rgb else None)
    res = nr_oracle.rasterize_rgbad(faces32.numpy(), tex_in, plan.H, plan.aa, H.NEAR, H.FAR, H.EPS, bg, plan.rgb,
                                    plan.alpha, plan.depth, tex_z_batch0=bool(plan.case["z_batch0"]))
    fn = res.fn
    ref = {"face_index_map": torch.from_numpy(fn.face_index_map).flip(1),
           "weight_map": torch.from_numpy(fn.weight_map).permute(0, 3, 1, 2).flip(2),
           "depth_map": torch.from_numpy(fn.depth_map).flip(1)}
    if plan.alpha:
        ref["alpha_map"] = torch.from_numpy(fn.alpha_map).flip(1)
    if plan.aa:
        for k in ("alpha", "depth") + (("rgb",) if cube and not (plan.corner or plan.phong) else ()):
            if res[k] is not None:
                ref["out_" + k] = torch.from_numpy(res[k])
    grads = {}
    g = lambda k: d.get(k)
    # the product's maps (held bit-exact to the oracle's above) for the float64 samplers, light and interpolation
    fim, wmap, dmap = (got[k] for k in ("face_index_map", "weight_map", "depth_map"))
    fm = torch.from_numpy(d["faces_mat"]).to(DEV)
    bgd = torch.from_numpy(np.asarray(bg)).to(DEV)
    g_rgb = torch.from_numpy(d["grad_rgb"]).to(DEV).double() if "grad_rgb" in d else None
    c64 = L64 = spc64 = None
    if plan.corner:  # smooth shading: float64 light from each item's own depths, times the unlit sample
        c64 = torch.from_numpy(d["corner_light"]).to(DEV).double().requires_grad_(True)
        L64 = smooth_light64(fm, fim, wmap, dmap, c64)
    # Phong (every mode): float64 light L and specular colour on the product's maps; the image is L s + spc
    ph64 = {k: torch.from_numpy(d[k]).to(DEV).double().requires_grad_(True) for k in PHONG_INPUTS if k in d}
    mapped = plan.nm or plan.sm  # the image is then oracles_specular_map.sm_rgb64, with either map or both
    mp64 = {k: torch.from_numpy(d[k]).to(DEV).double().requires_grad_(True) for k in MAP_INPUTS if k in d}
    if plan.phong and not mapped:
        L64, spc64 = sh_terms64(fm, fim, wmap, dmap, ph64["corner_shading"], ph64["params"], ph64.get("lights"),
                                ph64.get("sh"))
    shading_ins = [c64] if plan.corner else [ph64[k] for k in PHONG_INPUTS if "grad_" + k in plan.bufs]
    shading_outs = ["grad_corner_light"] if plan.corner else ["grad_" + k for k in PHONG_INPUTS if "grad_" + k in plan.bufs]
    shading_ins += [mp64[k] for k in MAP_INPUTS if "grad_" + k in plan.bufs]
    shading_outs += ["grad_" + k for k in MAP_INPUTS if "grad_" + k in plan.bufs]

    def lit(unlit, aa, L, spc):
        """the unlit raster sample [B,3,S,S] lit by the per-pixel light (and the Phong specular colour), the background
        where uncovered, pooled with anti-aliasing"""
        if spc is None:
            return smooth_rgb(unlit, L, fim, bgd, aa)
        rgb = torch.where((fim >= 0)[..., None], L * unlit.double().permute(0, 2, 3, 1) + spc, _bg(bgd, DEV))
        rgb = rgb.permute(0, 3, 1, 2)
        return torch.nn.functional.avg_pool2d(rgb, 2, 2) if aa else rgb

    def grad_of(out, ins):
        if g_rgb is None or not ins:
            return [torch.zeros_like(x) for x in ins]
        return torch.autograd.grad((out * g_rgb).sum(), ins)
    gt_corner = None
    if cube and (plan.corner or plan.phong):
        # the CPU oracle's unlit raster sample (bit-exact, NR_TEX_Z_BATCH0 honoured) lit by the float64 light
        unlit = torch.from_numpy(fn.rgb_map).permute(0, 3, 1, 2).flip(2).to(DEV)
        ref["rgb_map"] = lit(unlit, False, L64, spc64).detach()
        out = lit(unlit, plan.aa, L64, spc64)
        if plan.aa:
            ref["out_rgb"] = out.detach()
        for k, gk in zip(shading_outs, grad_of(out, shading_ins)):
            grads[k] = gk.detach().cpu().numpy()
        # K6 of the oracle fed the raster upstream gradient times the light, in float64
        if g_rgb is not None:
            G = (_upsample(g_rgb, plan.aa) * L64.detach().permute(0, 3, 1, 2)).flip(2).permute(0, 2, 3, 1)
            gt_corner = _k6_64(fn, G.cpu().numpy())
        else:
            gt_corner = np.zeros_like(fn.textures)
        fn.rgb_map = np.ascontiguousarray(got["rgb_map"].permute(0, 2, 3, 1).flip(1).cpu().numpy())
    elif cube:
        ref["rgb_map"] = torch.from_numpy(fn.rgb_map).permute(0, 3, 1, 2).flip(2)
    elif plan.rgb:
        # the texture-image sampler on the product's maps, in float64
        uvs = torch.from_numpy(d["face_uvs"]).to(DEV)
        uvs = uvs[None] if uvs.dim() == 3 else uvs
        tex64 = torch.from_numpy(d["textures"]).to(DEV).double().requires_grad_(True)
        light64 = torch.from_numpy(d["face_light"]).to(DEV).double().requires_grad_(True) if plan.lit else None
        zero_bg = torch.zeros(3, dtype=torch.float64, device=DEV)

        def sample(aa, bg_, light, uv, uv_grad, lod_fn):
            if plan.mip:
                levels = unpack_pyramid(tex64, plan.Ht, plan.Wt)
                if uv_grad:
                    return oracle_trilinear_levels_uv_grad(fm, fim, wmap, dmap, uv, levels, plan.Ht, plan.Wt, light, bg_,
                                                           plan.fill_back, aa, lod_fn)
                return oracle_trilinear_levels(fm, fim, wmap, dmap, uv, levels, plan.Ht, plan.Wt, light, bg_,
                                               plan.fill_back, aa, lod_fn)[0]
            if uv_grad:
                return oracle_rgb_uv_grad(fm, fim, wmap, dmap, uv, tex64, light, bg_, plan.fill_back, aa)
            return oracle_rgb(fm, fim, wmap, dmap, uv, tex64, light, bg_, plan.fill_back, aa)

        def image(aa, uv=uvs, uv_grad=False, L=None, spc=None, lod_fn=None):
            if mapped:  # the maps are sampled at the same UVs: with uv_grad their UV term joins the albedo's
                return sm_rgb64(fm, fim, wmap, dmap, ph64["corner_shading"], ph64["params"], ph64.get("lights"),
                                ph64.get("sh"), mp64.get("normal_map"), mp64.get("corner_tangents"),
                                mp64.get("specular_map"), uv, sample(False, zero_bg, None, uv, uv_grad, lod_fn), bgd, aa,
                                plan.fill_back)
            if plan.corner or plan.phong:  # the unlit sample times the interpolated light (plus the highlights)
                return lit(sample(False, zero_bg, None, uv, uv_grad, lod_fn), aa, L, spc)
            return sample(aa, bgd, light64, uv, uv_grad, lod_fn)
        # the light as a constant: the UV gradients come through the sampler alone
        Ld, spcd = (L64.detach() if L64 is not None else None), (spc64.detach() if spc64 is not None else None)
        ref["rgb_map"] = image(False, L=L64, spc=spc64).detach()
        out = image(plan.aa, L=L64, spc=spc64)
        if plan.aa:
            ref["out_rgb"] = out.detach()
        light_ins = [light64] if plan.lit else []
        gi = grad_of(out, [tex64] + light_ins + shading_ins)
        grads["grad_textures"] = gi[0].detach().cpu().numpy()
        if "grad_face_light" in plan.bufs:
            grads["grad_face_light"] = gi[1].detach().cpu().numpy()
        for k, gk in zip(shading_outs, gi[1 + len(light_ins):]):
            grads[k] = gk.detach().cpu().numpy()
        if plan.uv_grad:  # through the straight-through UV oracles; autograd folds fill_back and sums shared UVs
            uv64 = torch.from_numpy(d["face_uvs"]).to(DEV).double().requires_grad_(True)
            img = image(plan.aa, uv64[None] if uv64.dim() == 3 else uv64, True, Ld, spcd)
            grads["grad_face_uvs"] = grad_of(img, [uv64])[0].detach().cpu().numpy()
        if plan.mip:  # the same gradients at the product's fp32 level of detail (oracles.lod32; see TOL_GRAD_ELEM_MIP)
            alt = grads["lod32"] = {}
            alt["grad_textures"] = grad_of(image(plan.aa, L=Ld, spc=spcd, lod_fn=lod32), [tex64])[0].detach().cpu().numpy()
            if plan.uv_grad:
                img = image(plan.aa, uv64[None] if uv64.dim() == 3 else uv64, True, Ld, spcd, lod32)
                alt["grad_face_uvs"] = grad_of(img, [uv64])[0].detach().cpu().numpy()
        # K5 reads the rgb map: feed the oracle's edge scan the product's own (held to the float64 sampler above)
        fn.rgb_map = np.ascontiguousarray(got["rgb_map"].permute(0, 2, 3, 1).flip(1).cpu().numpy())
    fn.k5_sum_fp64 = True
    gf, gt = res.backward(g("grad_rgb") if plan.rgb else None, g("grad_alpha") if plan.alpha else None,
                          g("grad_depth") if plan.depth else None)
    if gt_corner is not None:
        gt = gt_corner
    gf = torch.from_numpy(gf).double()
    if plan.interior:  # the interior term joins K5 / K7's face gradient before the chain to the vertices
        g_int, ref["held_rgb"] = interior_oracle(plan, d, got, g_rgb)
        gf = gf + g_int
    # float64 chain of the oracle's face / cube gradients back to the inputs of the case
    geom64 = t(geom_key, torch.float64).requires_grad_(True)
    tex64 = t("textures", torch.float64).requires_grad_(True) if cube else None
    light64 = t("face_light", torch.float64).requires_grad_(True) if (cube and plan.lit) else None
    f64, c64 = materialise(plan, d, geom64, tex64, light64)
    outs, gouts, ins = [f64], [gf], [geom64]
    if cube:
        outs.append(c64)
        gouts.append(torch.from_numpy(gt).double())
        ins += [tex64] + ([light64] if light64 is not None else [])
    chained = torch.autograd.grad(outs, ins, gouts, allow_unused=True)
    chained = [torch.zeros_like(x) if c is None else c for c, x in zip(chained, ins)]
    grads["grad_vertices" if plan.indexed else "grad_faces"] = chained[0].numpy()
    if cube:
        grads["grad_textures"] = chained[1].numpy()
        if "grad_face_light" in plan.bufs:
            grads["grad_face_light"] = chained[2].numpy()
    if plan.attr:
        interp_oracle(plan, d, got, ref, grads)
    return ref, grads


def interior_oracle(plan, d, got, g_rgb):
    """NR_GRAD_INTERIOR: (d sum(g * rgb) / d faces [B,F,3,3] through the perspective weights, on the CPU; the lit sample
    [B,3,S,S] it differentiates, 0 at uncovered pixels) by float64 autograd of oracles_interior.rgb_held64 on the
    product's maps, in the case's materialised faces (a leaf: the caller's chain takes the gradient through the gathers).
    The sample is built from the case's own buffers -- unlit cubes (the fill_back copies reversed by Tex), the image or
    the levels of the packed pyramid, shared or per-item UVs, face or corner light -- and the cell, the level of detail
    and the clamp gates come from oracles_interior.select on the product's depth map.  Without an rgb upstream gradient
    the term is 0."""
    from oracles import unpack_pyramid
    from oracles_interior import Tex, rgb_held64, select
    dv = lambda k: torch.from_numpy(np.ascontiguousarray(d[k])).to(DEV).double() if k in d else None
    fim, wmap, dmap = (got[k] for k in ("face_index_map", "weight_map", "depth_map"))
    tex = dv("textures")
    if plan.kind in ("cube", "cube_shared"):
        T = Tex("cube", tex, eps=H.EPS, fill_back=plan.fill_back)
    else:
        uvs = dv("face_uvs")
        levels = unpack_pyramid(tex, plan.Ht, plan.Wt) if plan.mip else [tex]
        T = Tex("trilinear" if plan.mip else "bilinear", levels, uvs=uvs[None] if uvs.dim() == 3 else uvs,
                fill_back=plan.fill_back)
    faces = dv("faces_mat").requires_grad_(True)
    sel = select(faces, fim, wmap, plan.S, T, dmap)
    rgb = rgb_held64(faces, fim, wmap, plan.S, T, sel, dv("face_light"), dv("corner_light"))
    if g_rgb is None:
        gf = torch.zeros_like(faces)
    else:
        gf, = torch.autograd.grad((rgb * _upsample(g_rgb, plan.aa).permute(0, 2, 3, 1)).sum(), [faces])
    return gf.detach().cpu(), rgb.detach().permute(0, 3, 1, 2)


def interp_oracle(plan, d, got, ref, grads):
    """attribute interpolation: oracles_attr.interp64 on the float64 materialised faces (fill_back copies included) and
    corner attributes gathered in float64 (an out-of-range index reads zeros), at the product's weights; both gradients
    by autograd back through the gathers"""
    from oracles_attr import interp64
    B, F, Nv = plan.B, plan.F, plan.Nv
    fim, wmap = got["face_index_map"].cpu(), got["weight_map"].cpu()
    geom64 = torch.from_numpy(d["vertices" if plan.indexed else "faces"]).double().requires_grad_(True)
    f64 = materialise(plan, d, geom64, None, None)[0]
    a64 = torch.from_numpy(d["attributes"]).double().requires_grad_(True)
    if plan.attr_pv:
        ind = torch.from_numpy(d["face_indices"].astype(np.int64)).expand(B, F, 3)
        valid = ((ind >= 0) & (ind < Nv))[..., None]
        ga = a64.expand(B, -1, -1)[torch.arange(B)[:, None, None], ind.clamp(0, Nv - 1)]
        corner = torch.where(valid, ga, torch.zeros((), dtype=torch.float64))
    else:
        corner = a64.expand(B, -1, -1, -1)
    img = interp64(f64, fim, corner, plan.S, plan.aa, wmap=wmap)
    ref["attr_out"] = img.detach()
    ga, gg = torch.autograd.grad((img * torch.from_numpy(d["attr_grad_out"]).double()).sum(), [a64, geom64])
    grads["attr_grad_attributes"] = ga.numpy()
    for k in ("attr_grad_faces", "attr_grad_vertices"):
        if k in plan.bufs:
            grads[k] = gg.numpy()


def _bits(t):
    return t.contiguous().view(torch.int32)


# gates of the gradients: (per tensor, per element, per element with NR_TEX_MIPMAP), measured maxima in the docstring
GRAD_GATES = {"grad_corner_light": (TOL_GRAD, TOL_GRAD, TOL_CORNER_ELEM_MIP),
              "grad_face_uvs": (TOL_GRAD, TOL_GRAD, TOL_UV_ELEM_MIP),
              "attr_grad_attributes": (TOL_ATTR, TOL_GRAD, TOL_GRAD),
              "attr_grad_faces": (TOL_INTERIOR, TOL_INTERIOR_ELEM, TOL_INTERIOR_ELEM),
              "attr_grad_vertices": (TOL_INTERIOR, TOL_INTERIOR_ELEM, TOL_INTERIOR_ELEM),
              "grad_textures": (TOL_GRAD, TOL_GRAD, TOL_GRAD_ELEM_MIP),
              "grad_corner_shading": (TOL_GRAD, TOL_CS_ELEM, TOL_CS_ELEM),
              "grad_params": (TOL_GRAD, TOL_PARAMS_ELEM, TOL_PARAMS_ELEM),
              "grad_lights": (TOL_GRAD, TOL_LIGHTS_ELEM, TOL_LIGHTS_ELEM),
              "grad_sh": (TOL_GRAD, TOL_SH_ELEM, TOL_SH_ELEM),
              "grad_normal_map": (TOL_GRAD, TOL_NM_ELEM, TOL_NM_ELEM),
              "grad_corner_tangents": (TOL_GRAD, TOL_TG_ELEM, TOL_TG_ELEM),
              "grad_specular_map": (TOL_GRAD, TOL_SM_ELEM, TOL_SM_ELEM)}


def near_kinks(plan, d, got):
    """covered pixels within fp32 reach of a highlight's switch: |c_j| < KINK in float64 on the product's maps, for light
    0 of params (c = nh . d) and every light of the set (c_j = nh . x_j, or nh . lh_j for a point light), where K_j is
    not 0.  [c_j > 0] makes the highlight jump there, so such a pixel could fail for no kernel reason.  With a normal
    map the switches are those of the mapped normal n' (oracles_normal_map.mapped_normal64)."""
    from oracles_normal_map import map_sample64, mapped_normal64
    from oracles_phong import _norm
    fim, wmap, dmap = (got[k] for k in ("face_index_map", "weight_map", "depth_map"))
    B, S = plan.B, plan.S
    dv = lambda k: torch.from_numpy(d[k]).to(DEV).double()
    fi = fim.clamp(min=0).long()
    bidx = torch.arange(B, device=DEV)[:, None, None].expand(B, S, S)
    cov = fim >= 0
    z = torch.where(cov[..., None], dv("faces_mat")[..., 2][bidx, fi], torch.ones((), dtype=torch.float64, device=DEV))
    lam = wmap.double().permute(0, 2, 3, 1) * (dmap.double()[..., None] / z)
    cs = dv("corner_shading")
    C = cs[bidx if cs.shape[0] > 1 else torch.zeros_like(bidx), fi]
    nh = _norm((lam[..., None] * C[..., :3]).sum(dim=3))
    if plan.nm:
        uvs = dv("face_uvs")
        m = map_sample64(dv("faces_mat"), fim, wmap, dmap, uvs[None] if uvs.dim() == 3 else uvs, dv("normal_map"),
                         plan.fill_back)
        nh = _norm(mapped_normal64(dv("faces_mat"), fim, wmap, dmap, cs, dv("corner_tangents"), m)[0])
    p = (lam[..., None] * C[..., 3:]).sum(dim=3)
    prm = dv("params").expand(B, 16)[:, None, None, :]
    terms = [((nh * prm[..., 6:9]).sum(-1), prm[..., 9:12])]
    if "lights" in d:
        lt = dv("lights").expand(B, -1, -1)
        for j in range(lt.shape[1]):
            rec = lt[:, j][:, None, None, :]
            point = rec[..., 10] > 0.5
            lh = _norm(rec[..., 6:9] - p)
            terms.append((torch.where(point, (nh * lh).sum(-1), (nh * rec[..., 6:9]).sum(-1)), rec[..., 3:6]))
    return sum(int(((c.abs() < KINK) & cov & (K != 0).any(-1)).sum()) for c, K in terms)


def run_case(c, metrics=None):
    """every failure of the case as a message (empty = pass); `metrics`, a list, receives (case id, tensor, error kind,
    value) of every gated comparison"""
    note = (lambda *m: metrics.append((c["id"],) + m)) if metrics is not None else (lambda *m: None)
    plan = H.Plan(c)
    d = H.make_inputs(plan, c["id"])
    buf = {k: H.alloc(shape, dt, plan.offsets[k], DEV) for k, (shape, dt) in plan.bufs.items()}
    for k, a in d.items():
        if k in buf:
            buf[k].copy_(torch.from_numpy(np.ascontiguousarray(a)))
    fails = []
    rc = H.forward(plan, buf, DEV)
    if rc != 0:
        return ["forward returned %d" % rc]
    if plan.attr:
        rc = H.interpolate(plan, buf, DEV)
        if rc != 0:
            return ["nr_b200_interpolate returned %d" % rc]
    fails += ["%s: a guard word next to the buffer changed in the forward" % k for k in buf if not H.guards_intact(buf[k])]
    got = {k: buf[k] for k in plan.fwd_outputs}
    if plan.map_entry != "direct" and not (plan.nm or plan.sm):
        # a NULL map struct runs exactly the call without it (include/nr_b200.h): the same maps, bit for bit
        first = {k: _bits(t).clone() for k, t in got.items()}
        rc = H.forward(H.Plan({**c, "map_entry": "direct"}), buf, DEV)
        if rc != 0:
            return ["the direct forward returned %d" % rc]
        fails += ["%s: %s with NULL map structs differs from the direct call" % (k, plan.map_entry) for k in got
                  if not torch.equal(_bits(got[k]), first[k])]
    if plan.indexed:  # a face with an out-of-range corner has a zero vertex (z = 0): it must never win a pixel
        ind = np.broadcast_to(d["face_indices"], (plan.B, plan.F, 3))
        bad = ((ind < 0) | (ind >= plan.Nv)).any(-1)
        fimn = got["face_index_map"].cpu().numpy()
        won = bad[np.arange(plan.B)[:, None, None], np.clip(fimn, 0, plan.F - 1)] & (fimn >= 0)
        if won.any():
            fails.append("%d pixels won by a face with an out-of-range index" % int(won.sum()))
    ref, grads = oracle(plan, d, got)
    at_lod32 = grads.pop("lod32", {})  # trilinear: the oracle's gradients at the product's fp32 level of detail
    cov = int((got["face_index_map"] >= 0).sum())
    if cov < 300:
        fails.append("only %d covered pixels" % cov)
    cube = plan.kind in ("cube", "cube_shared")
    if plan.attr:
        got["attr_out"] = buf["attr_out"]
    for k in got:
        x, r = got[k].cpu(), ref[k].cpu()
        if k in ("face_index_map", "weight_map", "depth_map", "alpha_map") or (k == "rgb_map" and cube and not plan.corner
                                                                                and not plan.phong):
            if not torch.equal(x, r.to(x.dtype)):
                fails.append("%s: %d elements differ" % (k, int((x != r.to(x.dtype)).sum())))
        else:
            e = rel_err(x.numpy(), r.numpy()) if torch.isfinite(x).all() else float("nan")
            kind = "attr" if k == "attr_out" else ("mip" if plan.mip else ("smooth" if plan.corner else
                                                                           "phong" if plan.phong else "image"))
            if kind == "phong" and (plan.sigma > 1 or plan.sm):  # a specular map's shininess is 4 to 24
                kind = "phong_sigma"
            note(k, kind, e)
            if not e <= {"attr": TOL_ATTR_IMAGE, "mip": TOL_IMAGE_MIP, "phong_sigma": TOL_IMAGE_SIGMA}.get(kind, TOL_IMAGE):
                fails.append("%s: rel_err %.3g" % (k, e))
    if plan.phong:  # the inputs must keep every covered pixel off the highlights' switches (not masked out)
        n = near_kinks(plan, d, got)
        if n:
            fails.append("the case's inputs put %d covered pixels within %g of a highlight's switch c_j = 0 (K_j != 0): "
                         "choose other inputs" % (n, KINK))
    if plan.interior:  # the interior oracle differentiates the image the reference rendered (at the covered pixels)
        covm = (got["face_index_map"] >= 0)[:, None].expand(-1, 3, -1, -1)
        e = rel_err(ref["held_rgb"][covm].cpu().numpy(), ref["rgb_map"].to(DEV).double()[covm].cpu().numpy())
        note("held_rgb", "mip" if plan.mip else "image", e)
        if not e <= (TOL_IMAGE_MIP if plan.mip else TOL_IMAGE):
            fails.append("interior oracle's sample vs the reference rgb_map: rel_err %.3g" % e)
    # ---- backward
    rng = np.random.default_rng(2000 + c["id"])
    # ignored with NR_FACES_INDEXED; the field past the short backward struct
    untouched = [k for k in ("grad_faces", "past_end_fwd", "past_end_bwd")
                 if k in buf and (k != "grad_faces" or plan.indexed)]
    prefill = {}
    if plan.accumulate:  # per element about the size of the fresh gradient; where that is 0, a value of its scale
        for k in plan.grad_outputs:
            shape = plan.bufs[k][0]
            r = grads.get(k, np.zeros(shape))
            scale = float(np.abs(r).max()) or 1.0
            p = np.where(r != 0, r * rng.uniform(0.5, 1.5, shape), scale * rng.uniform(-1, 1, shape)).astype(np.float32)
            prefill[k] = p
            buf[k].copy_(torch.from_numpy(p))
    else:
        for k in plan.grad_outputs:
            H.poison(buf[k])
    before = {k: _bits(buf[k]).clone() for k in untouched}
    rcs = H.backward(plan, buf, DEV)
    if any(rcs):
        return fails + ["backward returned %s" % rcs]
    if plan.attr:
        rc = H.interpolate_backward(plan, buf, DEV)
        if rc != 0:
            return fails + ["nr_b200_interpolate_backward returned %d" % rc]
    fails += ["%s: a guard word next to the buffer changed in the backward" % k for k in buf if not H.guards_intact(buf[k])]
    for k in untouched:
        if not torch.equal(_bits(buf[k]), before[k]):
            fails.append("%s written although %s" % (k, "the geometry is indexed" if k == "grad_faces"
                                                     else "it lies past struct_size"))
    for k in plan.grad_outputs:
        if k in untouched:
            continue
        x = buf[k].double().cpu().numpy()
        r = grads[k]
        if not np.isfinite(x).all():
            fails.append("%s: %d elements not written / not finite" % (k, int((~np.isfinite(x)).sum())))
            continue
        if k.startswith("grad_") and k[5:] in PHONG_INPUTS + MAP_INPUTS and not plan.accumulate and (x[r == 0] != 0).any():
            # zero-filled, and no atomic reaches what no pixel differentiates (faces without pixels, slots 10-11 of a
            # light, texels no pixel samples, the handedness slots of grad_corner_tangents, every element without an rgb
            # upstream gradient)
            fails.append("%s: %d elements whose gradient is 0 are not 0" % (k, int((x[r == 0] != 0).sum())))
        if plan.accumulate:
            p = prefill[k]
            zero = r == 0
            if not np.array_equal(x[zero].astype(np.float32).view(np.int32), p[zero].view(np.int32)):
                fails.append("%s: prefill changed at %d of %d elements whose fresh gradient is 0"
                             % (k, int((x[zero] != p[zero]).sum()), int(zero.sum())))
            x = x - p.astype(np.float64)
        e1, e2 = rel_err(x, r), elem_err(x, r)
        tol_t, tol_e, tol_e_mip = GRAD_GATES.get(k, (TOL_GRAD, TOL_GRAD, TOL_GRAD))
        # without an rgb upstream gradient the interior term is 0, and the flag must change nothing: the usual gates
        interior = plan.interior and plan.g_rgb and k in ("grad_faces", "grad_vertices")
        if interior:
            tol_t, tol_e, tol_e_mip = TOL_INTERIOR, TOL_INTERIOR_ELEM, TOL_INTERIOR_ELEM
        if plan.nm or plan.sm:
            tol_e, tol_e_mip = max(tol_e, MAP_ROW_ELEM.get(k, 0)), max(tol_e_mip, MAP_ROW_ELEM.get(k, 0))
        tol_elem = tol_e_mip if plan.mip else tol_e
        if (c["id"], k) == (214, "grad_faces"):
            tol_elem = TOL_GRAD_ELEM_214
        if (c["id"], k) == (229, "grad_faces"):
            tol_elem = TOL_GRAD_ELEM_229
        if (c["id"], k) == (273, "grad_textures"):
            tol_elem = TOL_TEX_ELEM_273
        if (c["id"], k) == (259, "grad_params"):
            tol_elem = TOL_PARAMS_ELEM_259
        note(k, "tensor_interior" if interior else "tensor", e1)
        note(k, ("elem_interior" if interior else "elem_mip" if plan.mip and tol_e_mip != tol_e
                 else ("elem_acc" if plan.accumulate else "elem")), e2)
        ok = e1 <= tol_t and e2 <= tol_elem
        if k in at_lod32:
            e3 = elem_err(x, at_lod32[k])
            note(k, "elem_mip_lod32", e3)
            if k == "grad_textures" and not ok:  # what the float64 LOD alone moves must vanish at the fp32 LOD
                ok = e1 <= tol_t and e3 <= tol_elem
        if not ok:
            fails.append("%s: rel_err %.3g elem_err %.3g%s (max |ref| %.3g)"
                         % (k, e1, e2, " (%.3g at the fp32 LOD)" % e3 if k in at_lod32 else "", float(np.abs(r).max())))
    return fails


@pytest.mark.parametrize("case", CASES, ids=abi_cases.case_id)
def test_abi_case_vs_unfused_oracle(case):
    fails = run_case(case)
    assert not fails, "\n".join(fails)
