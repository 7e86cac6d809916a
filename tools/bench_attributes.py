#!/usr/bin/env python
"""Attribute images (rasterize_attributes) at the headline geometry: one JSON object.

Geometry: bench.py's B 64 seeded spheres (synthetic.sphere_faces), F 5000, 256 x 256, no anti-aliasing; every step is the
silhouette forward that writes the maps, k_interp, and the backward with a dense N(0,1) upstream gradient, vertices
requiring grad.  Per-vertex variants use indexed geometry with every corner its own vertex (faces viewed as [B,3F,3]).
  normals_c3         per-vertex normals (per item), C 3
  shared_feat_c16    one shared per-vertex feature set [3F,16] (NR_ATTR_SHARED) requiring grad, C 16
  uv_gbuffer_c2      the shared face_uvs [F,3,2] as a per-corner C 2 UV G-buffer (materialised faces)
  feat_c16_no_vgrad  shared_feat_c16 with vertices NOT requiring grad: the backward skips the vertex gradient
  teapot_normals     Renderer.render_attributes of F.vertex_normals, the teapot at 256 x 256 with anti-aliasing, batch 8
Whole step: CUDA events around `steps` steps after `warmup` warm-up steps, median [min, max] over `reps` repetitions.
Per kernel: the library's own CUDA-event profiler over `steps` further steps (microseconds per step).  The forward
kernel's algorithmic bytes are the maps it reads (face_index_map + weight_map, 16 B per raster pixel), the image it
writes (4 C B per API pixel) and the attributes once; over the data-sheet HBM figure they give k_interp's floor.

    python tools/bench_attributes.py [--steps 20] [--warmup 3] [--reps 5] [--only name,name,...]
"""
import argparse
import collections
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import neural_renderer_b200 as nb  # noqa: E402
from neural_renderer_b200 import _lib, functional as NF, synthetic  # noqa: E402

HBM_GBS = 3350.0  # H100 SXM data sheet


def gpu_info(dev):
    """device name and board power limit, read in the same run as the measurement"""
    info = {"name": torch.cuda.get_device_name(dev), "power_limit_w": None}
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(dev.index or 0), "--query-gpu=power.limit,clocks.max.sm",
                              "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30).stdout
        lim, clk = (x.strip() for x in out.strip().split(","))
        info["power_limit_w"], info["max_sm_clock_mhz"] = float(lim), float(clk)
    except Exception as e:  # the timing is still valid; say why the power limit is missing
        info["power_limit_error"] = repr(e)
    return info


def measure(step, a, lib):
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
        kern[k] = kern.get(k, 0.0) + 1000.0 * ms / a.steps
    lib.nr_b200_set_profiling(0)
    return {"step_ms_median": float(np.median(reps)), "step_ms_min_max": [min(reps), max(reps)], "step_ms_reps": reps,
            "kernels_us_per_step": kern}


def fwd_bytes(B, S_raster, H, C, attr_floats):
    return B * S_raster * S_raster * 16 + B * C * H * H * 4 + attr_floats * 4


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
    lib = _lib.load()
    faces0 = torch.from_numpy(synthetic.sphere_faces(B, F)).to(dev)
    verts0 = faces0.reshape(B, 3 * F, 3).contiguous()
    idx = torch.arange(3 * F, device=dev, dtype=torch.int32).reshape(F, 3)
    uvs = torch.from_numpy(synthetic.sphere_uvs(F)).to(dev)
    normals = NF.vertex_normals(verts0, idx)
    feat = torch.randn((3 * F, 16), generator=torch.Generator().manual_seed(1)).to(dev)
    names = ["normals_c3", "shared_feat_c16", "uv_gbuffer_c2", "feat_c16_no_vgrad", "teapot_normals"]
    if a.only:
        names = a.only.split(",")
    out = {"gpu": gpu_info(dev), "hbm_gbs_datasheet": HBM_GBS,
           "shape": {"batch": B, "faces": F, "size": S, "anti_aliasing": False}, "variants": {}}
    for name in names:
        if name == "teapot_normals":
            Bt = 8
            d = np.load(os.path.join(ROOT, "tests", "golden", "teapot.npz"))
            v = torch.from_numpy(np.stack([d["vertices"]] * Bt)).to(dev).requires_grad_(True)
            f = torch.from_numpy(np.stack([d["faces"]] * Bt)).to(dev)
            g = torch.randn((Bt, 3, 256, 256), generator=torch.Generator().manual_seed(2)).to(dev)
            r = nb.Renderer()
            r.eye = nb.get_points_from_angles(2.732, 30, 40)

            def step():
                v.grad = None
                r.render_attributes(v, f, vertex_attributes=NF.vertex_normals(v, f)).backward(g)

            rec = measure(step, a, lib)
            rec["shape"] = {"batch": Bt, "faces": int(f.shape[1]), "size": 256, "anti_aliasing": True, "fill_back": True}
            out["variants"][name] = rec
            continue
        C = {"normals_c3": 3, "uv_gbuffer_c2": 2}.get(name, 16)
        g = torch.randn((B, C, S, S), generator=torch.Generator().manual_seed(0)).to(dev)
        geom = (faces0 if name == "uv_gbuffer_c2" else verts0).clone().requires_grad_(name != "feat_c16_no_vgrad")
        attr = {"normals_c3": normals, "uv_gbuffer_c2": uvs}.get(name, feat).clone()
        attr.requires_grad_(name in ("shared_feat_c16", "feat_c16_no_vgrad"))

        def step():
            geom.grad = None
            attr.grad = None
            if name == "uv_gbuffer_c2":
                img = nb.rasterize_attributes(geom, S, False, face_attributes=attr)
            else:
                img = nb.rasterize_attributes(idx, S, False, vertices=geom, vertex_attributes=attr)
            img.backward(g)

        rec = measure(step, a, lib)
        nbytes = fwd_bytes(B, S, S, C, attr.numel())
        rec["k_interp_bytes"] = nbytes
        rec["k_interp_floor_us"] = nbytes / (HBM_GBS * 1e3)
        t = rec["kernels_us_per_step"].get("k_interp")
        if t:
            rec["k_interp_gbs"] = nbytes / (t * 1e3)
            rec["k_interp_fraction_of_hbm_datasheet"] = rec["k_interp_floor_us"] / t
        out["variants"][name] = rec
    print(json.dumps(out))


if __name__ == "__main__":
    main()
