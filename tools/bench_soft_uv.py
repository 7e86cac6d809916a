#!/usr/bin/env python
"""Soft RGB through a texture image (rasterize_soft(face_uvs=...)) next to the cube soft RGB at the headline geometry:
one JSON object.

Geometry: bench.py's B 64 seeded spheres (synthetic.sphere_faces) with their UVs (synthetic.sphere_uvs), F 5000,
256 x 256, gamma 1e-4, a face light [B,F,3]; faces, texels, UVs and light require grad; every step is a forward plus a
backward with dense N(0,1) upstream gradients (rgb and alpha).  Variants: one shared 1024 x 1024 image sampled bilinearly
and trilinearly, and a per-item 256 x 256 image (bilinear); each alternates, repetition by repetition, with the cube
soft RGB at ts 4 on the same geometry, so both see the same clocks.  Whole step: CUDA events around `steps` steps after
`warmup` warm-up steps, median [min, max] over `reps` repetitions.  Per kernel: torch.profiler (CUDA activity) over
`steps` further steps in a run of its own, microseconds per step.  The card's name and power limit are read in the same
call.

    python tools/bench_soft_uv.py [--steps 20] [--warmup 3] [--reps 5]
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import neural_renderer_b200 as nb  # noqa: E402
from neural_renderer_b200 import synthetic  # noqa: E402
from bench_soft_silhouettes import gpu_info, summary, time_step  # noqa: E402

GAMMA = 1e-4


def profile_kernels(step, n):
    """device microseconds per step of every kernel and memset of `n` steps (torch.profiler, CUDA activity)"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(n):
            step()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = e.cuda_time_total
        if t > 0:
            out[e.key[:80]] = round(t / n, 1)
    return dict(sorted(out.items(), key=lambda kv: -kv[1])[:10])


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
    B, F, S, ts = a.batch, a.faces, a.size, 4
    gen = torch.Generator().manual_seed(0)
    faces = torch.from_numpy(synthetic.sphere_faces(B, F)).to(dev).requires_grad_(True)
    uvs = torch.from_numpy(synthetic.sphere_uvs(F)).to(dev).requires_grad_(True)
    cubes = torch.rand((B, F, ts, ts, ts, 3), generator=gen).to(dev).requires_grad_(True)
    shared = torch.rand((1024, 1024, 3), generator=gen).to(dev).requires_grad_(True)
    per_item = torch.rand((B, 256, 256, 3), generator=gen).to(dev).requires_grad_(True)
    light = (0.5 + torch.rand((B, F, 3), generator=gen)).to(dev).requires_grad_(True)
    g_rgb = torch.randn((B, 3, S, S), generator=gen).to(dev)
    g_a = torch.randn((B, S, S), generator=gen).to(dev)
    out = {"gpu": gpu_info(dev), "shape": {"batch": B, "faces": F, "size": S, "gamma": GAMMA, "cube_texture_size": ts},
           "sigmas": {}}

    def clear():
        for t in (faces, uvs, cubes, shared, per_item, light):
            t.grad = None

    for sigma in (1e-5, 1e-4, 1e-3):
        def cube():
            clear()
            rgb, alpha = nb.rasterize_soft(faces, cubes, S, sigma, GAMMA, face_light=light)
            torch.autograd.backward((rgb, alpha), (g_rgb, g_a))

        def image(img, filt):
            def step():
                clear()
                rgb, alpha = nb.rasterize_soft(faces, img, S, sigma, GAMMA, face_light=light, face_uvs=uvs,
                                               texture_filter=filt)
                torch.autograd.backward((rgb, alpha), (g_rgb, g_a))
            return step

        variants = {"shared_1024_bilinear": image(shared, "bilinear"), "shared_1024_trilinear": image(shared, "trilinear"),
                    "per_item_256_bilinear": image(per_item, "bilinear")}
        rec = {}
        for name, st in variants.items():
            steps = {name: st, "cube_ts4": cube}
            for _ in range(a.warmup):
                for s in steps.values():
                    s()
            torch.cuda.synchronize()
            reps = {k: [] for k in steps}
            for _ in range(a.reps):  # alternate: both paths see the same clocks
                for k, s in steps.items():
                    reps[k].append(time_step(s, a.steps))
            r = {k: summary(v) for k, v in reps.items()}
            r["over_cube_median"] = r[name]["step_ms_median"] / r["cube_ts4"]["step_ms_median"]
            rec[name] = r
        for name, st in list(variants.items()) + [("cube_ts4", cube)]:
            rec.setdefault(name, {})["kernels_us_per_step"] = profile_kernels(st, a.steps)
        out["sigmas"][repr(sigma)] = rec
    print(json.dumps(out))


if __name__ == "__main__":
    main()
