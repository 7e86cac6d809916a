#!/usr/bin/env python
"""Soft RGB (rasterize_soft) next to the soft silhouettes and the hard rgb at the headline geometry: one JSON object.

Geometry: bench.py's B 64 seeded spheres (synthetic.sphere_faces), F 5000, 256 x 256, per-item cubes ts 4 and a face
light [B,F,3], faces, textures and light requiring grad; every step is a forward plus a backward with dense N(0,1)
upstream gradients (rgb and alpha).  For each sigma in {1e-5, 1e-4, 1e-3} at gamma 1e-4 the soft RGB step alternates
with the soft silhouette step and the hard rasterize rgb step (anti-aliasing off) on the same inputs, repetition by
repetition, so all three see the same clocks.  Then the teapot through Renderer.render_soft at 256 x 256, batch 8.
Whole step: CUDA events around `steps` steps after `warmup` warm-up steps, median [min, max] over `reps` repetitions.
Per kernel: the library's own CUDA-event profiler over `steps` further steps (microseconds per step), the sort included.

    python tools/bench_soft_rgb.py [--steps 20] [--warmup 3] [--reps 5]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import neural_renderer_b200 as nb  # noqa: E402
from neural_renderer_b200 import _lib, synthetic  # noqa: E402
from bench_soft_silhouettes import gpu_info, kernels, summary, time_step  # noqa: E402

GAMMA = 1e-4


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--faces", type=int, default=5000)
    ap.add_argument("--size", type=int, default=256)
    ap.add_argument("--texture-size", type=int, default=4)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    dev = torch.device("cuda")
    B, F, S, ts = a.batch, a.faces, a.size, a.texture_size
    lib = _lib.load()
    gen = torch.Generator().manual_seed(0)
    faces = torch.from_numpy(synthetic.sphere_faces(B, F)).to(dev).requires_grad_(True)
    tex = torch.rand((B, F, ts, ts, ts, 3), generator=gen).to(dev).requires_grad_(True)
    light = (0.5 + torch.rand((B, F, 3), generator=gen)).to(dev).requires_grad_(True)
    g_rgb = torch.randn((B, 3, S, S), generator=gen).to(dev)
    g_a = torch.randn((B, S, S), generator=gen).to(dev)
    out = {"gpu": gpu_info(dev), "shape": {"batch": B, "faces": F, "size": S, "texture_size": ts, "gamma": GAMMA},
           "sigmas": {}}

    def clear():
        faces.grad = tex.grad = light.grad = None

    def hard():
        clear()
        nb.rasterize(faces, tex, S, False, face_light=light).backward(g_rgb)

    for sigma in (1e-5, 1e-4, 1e-3):
        def soft_rgb():
            clear()
            rgb, alpha = nb.rasterize_soft(faces, tex, S, sigma, GAMMA, face_light=light)
            torch.autograd.backward((rgb, alpha), (g_rgb, g_a))

        def soft_sil():
            clear()
            nb.rasterize_soft_silhouettes(faces, S, sigma).backward(g_a)

        steps = {"soft_rgb": soft_rgb, "soft_silhouettes": soft_sil, "hard_rgb": hard}
        for _ in range(a.warmup):
            for st in steps.values():
                st()
        torch.cuda.synchronize()
        reps = {k: [] for k in steps}
        for _ in range(a.reps):  # alternate: the three paths see the same clocks
            for k, st in steps.items():
                reps[k].append(time_step(st, a.steps))
        rec = {k: summary(v) for k, v in reps.items()}
        for k, st in steps.items():
            rec[k]["kernels_us_per_step"] = kernels(st, a.steps, lib)
        rec["soft_rgb_over_hard_rgb_median"] = rec["soft_rgb"]["step_ms_median"] / rec["hard_rgb"]["step_ms_median"]
        rec["soft_rgb_over_soft_silhouettes_median"] = (rec["soft_rgb"]["step_ms_median"]
                                                         / rec["soft_silhouettes"]["step_ms_median"])
        out["sigmas"][repr(sigma)] = rec

    Bt = 8
    d = np.load(os.path.join(ROOT, "tests", "golden", "teapot.npz"))
    v = torch.from_numpy(np.stack([d["vertices"]] * Bt)).to(dev).requires_grad_(True)
    f = torch.from_numpy(np.stack([d["faces"]] * Bt)).to(dev)
    ttex = torch.rand((1, f.shape[1], ts, ts, ts, 3), generator=gen).to(dev).requires_grad_(True)
    gt_rgb = torch.randn((Bt, 3, 256, 256), generator=gen).to(dev)
    gt_a = torch.randn((Bt, 256, 256), generator=gen).to(dev)
    r = nb.Renderer()
    r.eye = nb.get_points_from_angles(2.732, 30, 40)

    def teapot():
        v.grad = ttex.grad = None
        rgb, alpha = r.render_soft(v, f, ttex, 1e-4, GAMMA)
        torch.autograd.backward((rgb, alpha), (gt_rgb, gt_a))

    for _ in range(a.warmup):
        teapot()
    torch.cuda.synchronize()
    rec = summary([time_step(teapot, a.steps) for _ in range(a.reps)])
    rec["kernels_us_per_step"] = kernels(teapot, a.steps, lib)
    rec["shape"] = {"batch": Bt, "faces": int(f.shape[1]), "size": 256, "sigma": 1e-4, "gamma": GAMMA,
                    "texture_size": ts}
    out["teapot_renderer"] = rec
    print(json.dumps(out))


if __name__ == "__main__":
    main()
