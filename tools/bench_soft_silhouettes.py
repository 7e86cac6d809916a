#!/usr/bin/env python
"""Soft silhouettes (rasterize_soft_silhouettes) next to the hard silhouette at the headline geometry: one JSON object.

Geometry: bench.py's B 64 seeded spheres (synthetic.sphere_faces), F 5000, 256 x 256, faces requiring grad; every step is
a forward plus a backward with a dense N(0,1) upstream gradient.  For each sigma in {1e-5, 1e-4, 1e-3} the soft step
alternates with the hard rasterize_silhouettes step (anti-aliasing off) on the same faces, repetition by repetition, so
both see the same clocks.  Then the teapot through Renderer.render_soft_silhouettes at 256 x 256, batch 8.
Whole step: CUDA events around `steps` steps after `warmup` warm-up steps, median [min, max] over `reps` repetitions.
Per kernel: the library's own CUDA-event profiler over `steps` further steps (microseconds per step).  The forward's
floor in bytes: the face records it must read once (64 B per face and item), the tile lists (4 B per list entry, counted
from the same binning on the host) and the alpha image it writes (4 B per pixel), over the data-sheet HBM figure.

    python tools/bench_soft_silhouettes.py [--steps 20] [--warmup 3] [--reps 5]
"""
import argparse
import collections
import json
import math
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import neural_renderer_b200 as nb  # noqa: E402
from neural_renderer_b200 import _lib, synthetic  # noqa: E402

HBM_GBS = 3350.0  # H100 SXM data sheet
TILE, WIDE = 16, 16  # nr_soft.cu: kTile, kWideTiles


def gpu_info(dev):
    """device name, board power limit and maximum SM clock, read in the same run as the measurement"""
    info = {"name": torch.cuda.get_device_name(dev), "power_limit_w": None}
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(dev.index or 0), "--query-gpu=power.limit,clocks.max.sm",
                              "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30).stdout
        lim, clk = (x.strip() for x in out.strip().split(","))
        info["power_limit_w"], info["max_sm_clock_mhz"] = float(lim), float(clk)
    except Exception as e:  # the timing is still valid; say why the power limit is missing
        info["power_limit_error"] = repr(e)
    return info


def time_step(step, steps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        step()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def kernels(step, steps, lib):
    lib.nr_b200_set_profiling(1)
    _lib.read_profile()
    for _ in range(steps):
        step()
    torch.cuda.synchronize()
    kern = collections.OrderedDict()
    for k, ms in _lib.read_profile():
        kern[k] = kern.get(k, 0.0) + 1000.0 * ms / steps
    lib.nr_b200_set_profiling(0)
    return kern


def summary(reps):
    return {"step_ms_median": float(np.median(reps)), "step_ms_min_max": [min(reps), max(reps)], "step_ms_reps": reps}


def list_entries(faces, S, sigma):
    """tile-list entries of the binning (the kernel's rule, on the host): tiles per face, wide faces once per tile"""
    f = faces.detach().double().cpu().numpy()
    reach = math.sqrt(sigma * math.log((1 - 1e-4) / 1e-4)) * S / 2 + 1
    x, y = f[..., 0], f[..., 1]
    c0 = np.clip(np.floor((x.min(-1) * S + S - 1) / 2 - reach), 0, S - 1)
    c1 = np.clip(np.ceil((x.max(-1) * S + S - 1) / 2 + reach), 0, S - 1)
    r0 = np.clip(np.floor(S - 1 - (y.max(-1) * S + S - 1) / 2 - reach), 0, S - 1)
    r1 = np.clip(np.ceil(S - 1 - (y.min(-1) * S + S - 1) / 2 + reach), 0, S - 1)
    nt = (c1 // TILE - c0 // TILE + 1) * (r1 // TILE - r0 // TILE + 1)
    ntiles = ((S + TILE - 1) // TILE) ** 2
    return int(np.where(nt > WIDE, ntiles, nt).sum())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--faces", type=int, default=5000)
    ap.add_argument("--size", type=int, default=256)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    dev = torch.device("cuda")
    B, F, S = a.batch, a.faces, a.size
    lib = _lib.load()
    faces = torch.from_numpy(synthetic.sphere_faces(B, F)).to(dev).requires_grad_(True)
    g = torch.randn((B, S, S), generator=torch.Generator().manual_seed(0)).to(dev)
    out = {"gpu": gpu_info(dev), "hbm_gbs_datasheet": HBM_GBS,
           "shape": {"batch": B, "faces": F, "size": S}, "sigmas": {}}

    def hard():
        faces.grad = None
        nb.rasterize_silhouettes(faces, S, False).backward(g)

    for sigma in (1e-5, 1e-4, 1e-3):
        def soft():
            faces.grad = None
            nb.rasterize_soft_silhouettes(faces, S, sigma).backward(g)

        for _ in range(a.warmup):
            soft()
            hard()
        torch.cuda.synchronize()
        rs, rh = [], []
        for _ in range(a.reps):  # alternate: the two paths see the same clocks
            rs.append(time_step(soft, a.steps))
            rh.append(time_step(hard, a.steps))
        rec = {"soft": summary(rs), "hard": summary(rh)}
        rec["soft"]["kernels_us_per_step"] = kernels(soft, a.steps, lib)
        rec["hard"]["kernels_us_per_step"] = kernels(hard, a.steps, lib)
        entries = list_entries(faces, S, sigma)
        nbytes = B * F * 64 + entries * 4 + B * S * S * 4
        rec["soft"]["list_entries"] = entries
        rec["soft"]["k_soft_fwd_bytes"] = nbytes
        rec["soft"]["k_soft_fwd_floor_us"] = nbytes / (HBM_GBS * 1e3)
        t = rec["soft"]["kernels_us_per_step"].get("k_soft_fwd")
        if t:
            rec["soft"]["k_soft_fwd_fraction_of_hbm_datasheet"] = rec["soft"]["k_soft_fwd_floor_us"] / t
        rec["soft_over_hard_median"] = rec["soft"]["step_ms_median"] / rec["hard"]["step_ms_median"]
        out["sigmas"][repr(sigma)] = rec

    Bt = 8
    d = np.load(os.path.join(ROOT, "tests", "golden", "teapot.npz"))
    v = torch.from_numpy(np.stack([d["vertices"]] * Bt)).to(dev).requires_grad_(True)
    f = torch.from_numpy(np.stack([d["faces"]] * Bt)).to(dev)
    gt = torch.randn((Bt, 256, 256), generator=torch.Generator().manual_seed(2)).to(dev)
    r = nb.Renderer()
    r.eye = nb.get_points_from_angles(2.732, 30, 40)

    def teapot():
        v.grad = None
        r.render_soft_silhouettes(v, f, 1e-4).backward(gt)

    for _ in range(a.warmup):
        teapot()
    torch.cuda.synchronize()
    rec = summary([time_step(teapot, a.steps) for _ in range(a.reps)])
    rec["kernels_us_per_step"] = kernels(teapot, a.steps, lib)
    rec["shape"] = {"batch": Bt, "faces": int(f.shape[1]), "size": 256, "sigma": 1e-4}
    out["teapot_renderer"] = rec
    print(json.dumps(out))


if __name__ == "__main__":
    main()
