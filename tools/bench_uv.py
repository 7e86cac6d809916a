#!/usr/bin/env python
"""Texture image vs texture cubes at the headline geometry: one JSON object.

Geometry: B 64 seeded spheres (synthetic.sphere_faces), F 5000, 256 x 256, no anti-aliasing, `rasterize()` forward +
backward with a dense N(0,1) upstream gradient (bench.py's headline step).  Textures:
  uv_shared_1024   one 1024 x 1024 image shared by every item (NR_TEX_SHARED), spherical UVs shared (NR_UV_SHARED)
  uv_item_256      one 256 x 256 image per item, spherical UVs shared
  cubes_ts4        the per-item ts = 4 cubes of bench.py
  uv_shared_1024_trilinear, uv_item_256_trilinear   the two image variants with texture_filter='trilinear': the mip
                   pyramid is built (k_mip_build) and its gradient collapsed (k_mip_collapse) on every step
  uv_shared_1024_uvgrad, uv_shared_1024_trilinear_uvgrad   uv_shared_1024 (bilinear / trilinear) with
                   face_uvs.requires_grad_(True): k_image_grad also returns d loss / d face_uvs
  cubes_ts4_smooth, uv_shared_1024_smooth, uv_shared_1024_trilinear_smooth   the same with smooth shading: every step
                   computes vertex normals (every corner its own vertex: faces viewed as [B,3F,3] vertices) and the
                   per-corner light with the glue kernels and passes corner_light to rasterize()
  teapot_render_flat, teapot_render_smooth   Renderer.render fwd + bwd (fused), the teapot at 256 x 256 with
                   anti-aliasing, batch 8, ts 4 cubes, flat vs smooth shading (README's Renderer row)
Whole step: CUDA events around `steps` steps after `warmup` warm-up steps, median over `reps` repetitions.  Per kernel:
the library's own CUDA-event profiler over `steps` further steps (ms per step).  Bytes held = texture + its gradient.
The roofline fraction of the image-gradient kernel and of the zero-fill uses bench.py's HBM figure.  For every image
variant, `lod_above_0` is the share of covered pixels whose trilinear level of detail is above 0 (how much the geometry
minifies the image), computed once with torch from the saved maps and not timed.

    python tools/bench_uv.py [--steps 20] [--warmup 3] [--reps 5] [--only name,name,...]

--only runs the named variants in the given order (e.g. a variant before and after its counterpart, to see how much of
a difference is the order of the run).
"""
import argparse
import collections
import json
import os
import sys

import numpy as np
import torch
import torch.nn.functional

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import neural_renderer as nr  # noqa: E402
import neural_renderer_b200 as nb  # noqa: E402
from neural_renderer_b200 import _lib, functional as NF, synthetic  # noqa: E402


def hbm_gbs():
    path = os.path.join(ROOT, "MEASURED_PEAKS.json")  # as bench.py: measured figure if present, else the data sheet
    if os.path.exists(path):
        with open(path) as f:
            return float(json.load(f)["hbm_gbs"])
    return 3350.0


def lod_above_0(faces, uvs, Ht, Wt, S):
    """share of covered pixels with a level of detail above 0 (include/nr_b200.h, NR_TEX_MIPMAP), float64 from the faces
    and the product's own face_index_map / weight_map / depth map"""
    R = sys.modules["neural_renderer_b200.rasterize"]
    with torch.no_grad():
        _, _, dmap, fim, wmap = R._run(faces, None, S, False, 0.1, 100, 1e-4, None, False, False, True)
        B = faces.shape[0]
        f64 = faces.double()
        px, py = 0.5 * (f64[..., 0] * S + S - 1), 0.5 * (f64[..., 1] * S + S - 1)
        M = torch.linalg.inv_ex(torch.stack((px, py, torch.ones_like(px)), dim=-2)).inverse
        cov = fim >= 0
        fi = fim.clamp(min=0).long()
        bidx = torch.arange(B, device=faces.device)[:, None, None].expand_as(fi)
        Mp, z = M[bidx, fi], f64[..., 2][bidx, fi]
        uvk = uvs.double().expand(B, -1, -1, -1)[bidx, fi]
        zp = dmap.double()[..., None]
        lam = wmap.double().permute(0, 2, 3, 1) * (zp / z)
        rho2 = []
        for d in (0, 1):
            q = Mp[..., d] / z
            dl = zp * (q - lam * q.sum(-1, keepdim=True))
            du, dv = (uvk[..., 0] * dl).sum(-1) * (Wt - 1), (uvk[..., 1] * dl).sum(-1) * (Ht - 1)
            rho2.append(du * du + dv * dv)
        lod = torch.nan_to_num(0.5 * torch.log2(torch.maximum(*rho2)), nan=0.0, neginf=0.0)
        return float((lod[cov] > 0).double().mean())


def teapot_render(smooth, a, lib, dev):
    """Renderer.render fwd + bwd (fused), teapot 256 x 256 anti-aliased, batch 8, ts 4 cubes: step time and kernels"""
    B = 8
    d = np.load(os.path.join(ROOT, "tests", "golden", "teapot.npz"))
    v = torch.from_numpy(np.stack([d["vertices"]] * B)).to(dev).requires_grad_(True)
    f = torch.from_numpy(np.stack([d["faces"]] * B)).to(dev)
    tex = torch.rand((B, f.shape[1], 4, 4, 4, 3), generator=torch.Generator().manual_seed(1)).to(dev).requires_grad_(True)
    g = torch.randn((B, 3, 256, 256), generator=torch.Generator().manual_seed(2)).to(dev)
    r = nb.Renderer()
    r.eye = nb.get_points_from_angles(2.732, 30, 40)
    r.shading = "smooth" if smooth else "flat"

    def step():
        v.grad = None
        tex.grad = None
        r.render(v, f, tex).backward(g)

    for _ in range(a.warmup):
        step()
    torch.cuda.synchronize()
    reps = []
    for _ in range(a.reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(a.steps):
            step()
        e1.record()
        torch.cuda.synchronize()
        reps.append(e0.elapsed_time(e1) / a.steps)
    lib.nr_b200_set_profiling(1)
    _lib.read_profile()
    for _ in range(a.steps):
        step()
    torch.cuda.synchronize()
    kern = collections.OrderedDict()
    for k, ms in _lib.read_profile():
        kern[k] = kern.get(k, 0.0) + ms / a.steps
    lib.nr_b200_set_profiling(0)
    return {"shading": r.shading, "step_ms_median": float(np.median(reps)), "step_ms_min_max": [min(reps), max(reps)],
            "step_ms_reps": reps, "kernels_ms_per_step": kern}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--faces", type=int, default=5000)
    ap.add_argument("--size", type=int, default=256)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--only", default=None, help="comma-separated variant names, run in this order")
    a = ap.parse_args()
    dev = torch.device("cuda")
    B, F, S = a.batch, a.faces, a.size
    faces = torch.from_numpy(synthetic.sphere_faces(B, F)).to(dev).requires_grad_(True)
    uvs = torch.from_numpy(synthetic.sphere_uvs(F)).to(dev)
    g = torch.randn((B, 3, S, S), generator=torch.Generator().manual_seed(0)).to(dev)
    img1024 = torch.from_numpy(synthetic.random_image(1, 1024, 1024)[0]).to(dev)
    img256 = torch.from_numpy(synthetic.random_image(B, 256, 256)).to(dev)
    cubes = torch.from_numpy(synthetic.random_textures(B, F, 4)).to(dev)
    variants = collections.OrderedDict([
        ("uv_shared_1024", (img1024, uvs, "bilinear", False)),
        ("uv_item_256", (img256, uvs, "bilinear", False)),
        ("cubes_ts4", (cubes, None, "bilinear", False)),
        ("uv_shared_1024_trilinear", (img1024, uvs, "trilinear", False)),
        ("uv_item_256_trilinear", (img256, uvs, "trilinear", False)),
        ("uv_shared_1024_uvgrad", (img1024, uvs, "bilinear", True)),
        ("uv_shared_1024_trilinear_uvgrad", (img1024, uvs, "trilinear", True)),
        ("cubes_ts4_smooth", (cubes, None, "bilinear", False)),
        ("uv_shared_1024_smooth", (img1024, uvs, "bilinear", False)),
        ("uv_shared_1024_trilinear_smooth", (img1024, uvs, "trilinear", False)),
        ("teapot_render_flat", None),
        ("teapot_render_smooth", None),
    ])
    corner_idx = torch.arange(3 * F, device=dev, dtype=torch.int32).reshape(F, 3)
    if a.only:
        variants = collections.OrderedDict((k, variants[k]) for k in a.only.split(","))
    lib = _lib.load()
    props = torch.cuda.get_device_properties(dev)
    out = {"gpu": torch.cuda.get_device_name(dev), "sm_count": props.multi_processor_count, "shape": {"batch": B, "faces": F, "size": S, "anti_aliasing": False},
           "hbm_gbs": hbm_gbs(), "variants": {}}
    for name, spec in variants.items():
        if spec is None:
            out["variants"][name] = teapot_render(name.endswith("smooth"), a, lib, dev)
            continue
        tex0, fuv0, tf, uv_grad = spec
        smooth = name.endswith("_smooth")
        tex = tex0.clone().requires_grad_(True)
        fuv = fuv0.clone().requires_grad_(True) if uv_grad else fuv0

        def step():
            faces.grad = None
            tex.grad = None
            if uv_grad:
                fuv.grad = None
            corner = None
            if smooth:
                verts = faces.reshape(B, 3 * F, 3)
                corner = NF.corner_light(NF.vertex_normals(verts, corner_idx), corner_idx)
            img = nb.rasterize(faces, tex, S, False, face_uvs=fuv, texture_filter=tf, corner_light=corner)
            img.backward(g)

        for _ in range(a.warmup):
            step()
        torch.cuda.synchronize()
        reps = []
        for _ in range(a.reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.steps):
                step()
            e1.record()
            torch.cuda.synchronize()
            reps.append(e0.elapsed_time(e1) / a.steps)
        lib.nr_b200_set_profiling(1)
        _lib.read_profile()
        for _ in range(a.steps):
            step()
        torch.cuda.synchronize()
        prof = _lib.read_profile()
        lib.nr_b200_set_profiling(0)
        kern = collections.OrderedDict()
        for k, ms in prof:
            kern[k] = kern.get(k, 0.0) + ms / a.steps
        tex_bytes = tex.numel() * 4
        if tf == "trilinear":  # the rasterizer samples (and its gradient is) the pyramid
            tex_bytes = tex.numel() // (tex.shape[-3] * tex.shape[-2]) * lib.nr_b200_mip_texels(*tex.shape[-3:-1]) * 4
        rec = {"texture_filter": tf, "uv_grad": uv_grad, "smooth": smooth, "step_ms_median": float(np.median(reps)),
               "step_ms_min_max": [min(reps), max(reps)], "step_ms_reps": reps,
               "kernels_ms_per_step": kern, "texture_bytes": tex_bytes, "texture_plus_grad_bytes": 2 * tex_bytes}
        if fuv is not None:
            rec["lod_above_0"] = lod_above_0(faces.detach(), fuv.detach()[None], tex.shape[-3], tex.shape[-2], S)
        grad_kernel = "k_image_grad" if fuv is not None else "k_texture_grad"
        if grad_kernel in kern:
            rec["grad_kernel"] = grad_kernel
        # The zero-fill of the texture gradient rides in k_edge_scan's CTAs when one call runs both halves of the
        # backward.  Timed on its own here: with a (no-op) texture hook the backward runs as two calls and the texture
        # half zero-fills with a memset of its own, the first "memset_grads" of every step.
        R = sys.modules["neural_renderer_b200.rasterize"]
        prev = R.set_texture_grad_hook(lambda grad: None)
        try:
            lib.nr_b200_set_profiling(1)
            _lib.read_profile()
            for _ in range(a.steps):
                step()
            torch.cuda.synchronize()
            prof2 = _lib.read_profile()
            lib.nr_b200_set_profiling(0)
        finally:
            R.set_texture_grad_hook(prev)
        fills = [ms for k, ms in prof2 if k == "memset_grads"][0::2]
        rec["zero_fill_bytes"] = tex_bytes
        rec["zero_fill_ms_separate_memset"] = float(np.median(fills)) if fills else None
        rec["zero_fill_ms_at_hbm_peak"] = tex_bytes / (out["hbm_gbs"] * 1e6)
        rec["split_backward_kernels_ms_per_step"] = {k: sum(ms for kk, ms in prof2 if kk == k) / a.steps
                                                     for k in dict.fromkeys(k for k, _ in prof2)}
        out["variants"][name] = rec
    print(json.dumps(out))


if __name__ == "__main__":
    main()
