"""GPU: every pair of the rasterizer's C-ABI flags, called directly (tests/abi_harness.py), held to an unfused oracle.

The cases come from the covering array of tests/abi_cases.py.  The oracle never runs the product's fused paths:
  cubes       the inputs are materialised as a float64 torch function of (vertices | faces, textures, light) -- faces by
              gather (out-of-range indices read zeros), shared textures expanded, fill_back as
              cat(t, t.permute(0,1,4,3,2,5)), the light multiplied in (in fp32 for the forward: the header pins the fused
              light as bit-identical to sampling the product) -- and rendered by the CPU oracle (oracle/nr_oracle.py,
              with per-item background and the batch-0 depth quirk as flagged; K5 summed in float64).  Its face /
              texture gradients are chained back to vertices, textures and light by float64 autograd.
  images      the float64 samplers of tests/oracles.py on the materialised geometry (bilinear, or trilinear on the
              packed pyramid passed as `textures`); the face / vertex gradient from the CPU oracle's K5 fed with the
              product's own raster rgb map.
Gates: face_index_map, weight_map and depth_map bit-exact; images bit-exact in non-anti-aliased cube mode, 1e-5 relative
elsewhere; every gradient tensor 1e-4 per tensor (helpers.rel_err) and per element (helpers.elem_err); the mip sampler's
image and pyramid gradient are the two exceptions, with their cause and measured maxima below.  Every output is poisoned
before a call (NaN, face-index sentinel), so an element the kernels do not write fails, and guard words around every
buffer must survive both calls, so a store just outside one fails; with
NR_GRAD_ACCUMULATE the gradients are prefilled with seeded values and must come back as prefill + fresh gradient, the
prefill untouched bit for bit wherever the oracle's fresh gradient is exactly 0."""
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
# the same absolute difference relative to its own size.  Measured maxima over the matrix on an H100: raster image
# 4.4e-5, anti-aliased image 5.1e-6, pyramid gradient per element 3.6e-4 (both in case 101), light gradient per element
# 7.5e-5 (inside TOL_GRAD).  Every other gate holds at its nominal value (largest per-element gradient error 5.9e-5,
# with NR_GRAD_ACCUMULATE 4.0e-5).
TOL_IMAGE_MIP = 6e-5
TOL_GRAD_ELEM_MIP = 5e-4
CASES = abi_cases.cases()


def _rotation(rng):
    from neural_renderer_b200 import synthetic
    return synthetic._rotation(rng)


def make_inputs(plan, seed):
    """seeded numpy inputs of a case: the arrays the ABI call reads, plus `faces_mat` (the materialised fp32 faces)"""
    from neural_renderer_b200 import synthetic
    rng = np.random.default_rng(1000 + seed)
    B, F, Nv = plan.B, plan.F, plan.Nv
    verts, idx = synthetic.sphere_mesh(plan.F_front)
    if plan.fill_back:
        idx = np.concatenate((idx, idx[:, ::-1]), axis=0)
    v = np.empty((B, Nv, 3), np.float32)
    for b in range(B):
        vb = (verts * 0.8) @ _rotation(rng).T + rng.normal(scale=0.01, size=verts.shape)
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
    for k in ("grad_rgb", "grad_alpha", "grad_depth"):
        if k in plan.bufs:
            d[k] = rng.standard_normal(plan.bufs[k][0]).astype(np.float32)
    return d


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


def oracle(plan, d, got):
    """(forward reference {name: tensor in the product's layout}, fresh gradients {buffer name: float64 numpy})"""
    import nr_oracle
    from oracles import oracle_rgb, oracle_trilinear_levels, unpack_pyramid
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
        for k in ("alpha", "depth") + (("rgb",) if cube else ()):
            if res[k] is not None:
                ref["out_" + k] = torch.from_numpy(res[k])
    grads = {}
    g = lambda k: d.get(k)
    if cube:
        ref["rgb_map"] = torch.from_numpy(fn.rgb_map).permute(0, 3, 1, 2).flip(2)
    elif plan.rgb:
        # the texture-image sampler on the product's maps (held bit-exact to the oracle's above), in float64
        fim, wmap, dmap = (got[k] for k in ("face_index_map", "weight_map", "depth_map"))
        fm = torch.from_numpy(d["faces_mat"]).to(DEV)
        uvs = torch.from_numpy(d["face_uvs"]).to(DEV)
        uvs = uvs[None] if uvs.dim() == 3 else uvs
        tex64 = torch.from_numpy(d["textures"]).to(DEV).double().requires_grad_(True)
        light64 = torch.from_numpy(d["face_light"]).to(DEV).double().requires_grad_(True) if plan.lit else None
        bgd = torch.from_numpy(np.asarray(bg)).to(DEV)

        def sample(aa):
            if plan.mip:
                return oracle_trilinear_levels(fm, fim, wmap, dmap, uvs, unpack_pyramid(tex64, plan.Ht, plan.Wt),
                                               plan.Ht, plan.Wt, light64, bgd, plan.fill_back, aa)[0]
            return oracle_rgb(fm, fim, wmap, dmap, uvs, tex64, light64, bgd, plan.fill_back, aa)
        ref["rgb_map"] = sample(False).detach()
        api = sample(True) if plan.aa else None
        if plan.aa:
            ref["out_rgb"] = api.detach()
        out = api if plan.aa else sample(False)
        ins = [tex64] + ([light64] if plan.lit else [])
        if "grad_rgb" in d:
            gi = torch.autograd.grad((out * torch.from_numpy(d["grad_rgb"]).to(DEV).double()).sum(), ins)
        else:
            gi = [torch.zeros_like(x) for x in ins]
        grads["grad_textures"] = gi[0].detach().cpu().numpy()
        if "grad_face_light" in plan.bufs:
            grads["grad_face_light"] = gi[1].detach().cpu().numpy()
        # K5 reads the rgb map: feed the oracle's edge scan the product's own (held to the float64 sampler above)
        fn.rgb_map = np.ascontiguousarray(got["rgb_map"].permute(0, 2, 3, 1).flip(1).cpu().numpy())
    fn.k5_sum_fp64 = True
    gf, gt = res.backward(g("grad_rgb") if plan.rgb else None, g("grad_alpha") if plan.alpha else None,
                          g("grad_depth") if plan.depth else None)
    # float64 chain of the oracle's face / cube gradients back to the inputs of the case
    geom64 = t(geom_key, torch.float64).requires_grad_(True)
    tex64 = t("textures", torch.float64).requires_grad_(True) if cube else None
    light64 = t("face_light", torch.float64).requires_grad_(True) if (cube and plan.lit) else None
    f64, c64 = materialise(plan, d, geom64, tex64, light64)
    outs, gouts, ins = [f64], [torch.from_numpy(gf).double()], [geom64]
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
    return ref, grads


def _bits(t):
    return t.contiguous().view(torch.int32)


def run_case(c, metrics=None):
    """every failure of the case as a message (empty = pass); `metrics`, a list, receives (case id, tensor, error kind,
    value) of every gated comparison"""
    note = (lambda *m: metrics.append((c["id"],) + m)) if metrics is not None else (lambda *m: None)
    plan = H.Plan(c)
    d = make_inputs(plan, c["id"])
    buf = {k: H.alloc(shape, dt, plan.offsets[k], DEV) for k, (shape, dt) in plan.bufs.items()}
    for k, a in d.items():
        if k in buf:
            buf[k].copy_(torch.from_numpy(np.ascontiguousarray(a)))
    fails = []
    rc = H.forward(plan, buf, DEV)
    if rc != 0:
        return ["forward returned %d" % rc]
    fails += ["%s: a guard word next to the buffer changed in the forward" % k for k in buf if not H.guards_intact(buf[k])]
    got = {k: buf[k] for k in plan.fwd_outputs}
    ref, grads = oracle(plan, d, got)
    cov = int((got["face_index_map"] >= 0).sum())
    if cov < 300:
        fails.append("only %d covered pixels" % cov)
    cube = plan.kind in ("cube", "cube_shared")
    for k in plan.fwd_outputs:
        x, r = got[k].cpu(), ref[k].cpu()
        if k in ("face_index_map", "weight_map", "depth_map", "alpha_map") or (k == "rgb_map" and cube):
            if not torch.equal(x, r.to(x.dtype)):
                fails.append("%s: %d elements differ" % (k, int((x != r.to(x.dtype)).sum())))
        else:
            e = rel_err(x.numpy(), r.numpy()) if torch.isfinite(x).all() else float("nan")
            note(k, "mip" if plan.mip else "image", e)
            if not e <= (TOL_IMAGE_MIP if plan.mip else TOL_IMAGE):
                fails.append("%s: rel_err %.3g" % (k, e))
    # ---- backward
    rng = np.random.default_rng(2000 + c["id"])
    untouched = [k for k in ("grad_faces",) if plan.indexed and k in buf]  # ignored with NR_FACES_INDEXED
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
    fails += ["%s: a guard word next to the buffer changed in the backward" % k for k in buf if not H.guards_intact(buf[k])]
    for k in untouched:
        if not torch.equal(_bits(buf[k]), before[k]):
            fails.append("%s written although the geometry is indexed" % k)
    for k in plan.grad_outputs:
        if k in untouched:
            continue
        x = buf[k].double().cpu().numpy()
        r = grads[k]
        if not np.isfinite(x).all():
            fails.append("%s: %d elements not written / not finite" % (k, int((~np.isfinite(x)).sum())))
            continue
        if plan.accumulate:
            p = prefill[k]
            zero = r == 0
            if not np.array_equal(x[zero].astype(np.float32).view(np.int32), p[zero].view(np.int32)):
                fails.append("%s: prefill changed at %d of %d elements whose fresh gradient is 0"
                             % (k, int((x[zero] != p[zero]).sum()), int(zero.sum())))
            x = x - p.astype(np.float64)
        e1, e2 = rel_err(x, r), elem_err(x, r)
        mip_tex = plan.mip and k == "grad_textures"
        tol_elem = TOL_GRAD_ELEM_MIP if mip_tex else TOL_GRAD
        note(k, "tensor", e1)
        note(k, "elem_mip" if mip_tex else ("elem_acc" if plan.accumulate else "elem"), e2)
        if not (e1 <= TOL_GRAD and e2 <= tol_elem):
            fails.append("%s: rel_err %.3g elem_err %.3g (max |ref| %.3g)" % (k, e1, e2, float(np.abs(r).max())))
    return fails


@pytest.mark.parametrize("case", CASES, ids=abi_cases.case_id)
def test_abi_case_vs_unfused_oracle(case):
    fails = run_case(case)
    assert not fails, "\n".join(fails)
