#!/usr/bin/env python
"""Soft attribute images (rasterize_soft_attributes) next to the cube soft RGB at the headline geometry: one JSON object.

Geometry: bench.py's B 64 seeded spheres (synthetic.sphere_faces), F 5000, 256 x 256, gamma 1e-4, drawn as indexed
geometry whose vertices are the faces' corners (Nv = 3F, one per corner); vertices and attributes require grad; every
step is a forward plus a backward with dense N(0,1) upstream gradients (image and alpha).  Variants: soft depth (the
vertices' z as a one-channel attribute, background = far), per-item per-vertex colours (C 3) and one shared set of
per-vertex features (C 16); each alternates, repetition by repetition, with the cube soft RGB at ts 4 on the same
geometry, so both see the same clocks.  Whole step: CUDA events around `steps` steps after `warmup` warm-up steps,
median [min, max] over `reps` repetitions.  Per kernel: torch.profiler (CUDA activity) over `steps` further steps in a
run of its own, microseconds per step.  The card's name and power limit are read in the same call.

    python tools/bench_soft_attributes.py [--steps 20] [--warmup 3] [--reps 5]
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
from bench_soft_uv import profile_kernels  # noqa: E402

GAMMA = 1e-4
FAR = 100.0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--faces", type=int, default=5000)
    ap.add_argument("--size", type=int, default=256)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--sigmas", default="1e-5,1e-4,1e-3")
    a = ap.parse_args()
    dev = torch.device("cuda")
    B, F, S, ts = a.batch, a.faces, a.size, 4
    gen = torch.Generator().manual_seed(0)
    faces = torch.from_numpy(synthetic.sphere_faces(B, F)).to(dev)
    verts = faces.reshape(B, 3 * F, 3).contiguous().requires_grad_(True)
    idx = torch.arange(3 * F, dtype=torch.int32, device=dev).reshape(F, 3)
    faces = faces.requires_grad_(True)
    cubes = torch.rand((B, F, ts, ts, ts, 3), generator=gen).to(dev).requires_grad_(True)
    colours = torch.rand((B, 3 * F, 3), generator=gen).to(dev).requires_grad_(True)
    features = torch.rand((1, 3 * F, 16), generator=gen).to(dev).requires_grad_(True)
    g = {C: torch.randn((B, C, S, S), generator=gen).to(dev) for C in (1, 3, 16)}
    g_a = torch.randn((B, S, S), generator=gen).to(dev)
    out = {"gpu": gpu_info(dev), "library": os.environ.get("NR_B200_LIB", "default"),
           "shape": {"batch": B, "faces": F, "size": S, "gamma": GAMMA, "cube_texture_size": ts}, "sigmas": {}}

    def clear():
        for t in (faces, verts, cubes, colours, features):
            t.grad = None

    for sigma in (float(s) for s in a.sigmas.split(",")):
        def cube():
            clear()
            rgb, alpha = nb.rasterize_soft(faces, cubes, S, sigma, GAMMA)
            torch.autograd.backward((rgb, alpha), (g[3], g_a))

        def attributes(make, C, bg):
            def step():
                clear()
                img, alpha = nb.rasterize_soft_attributes(idx, S, sigma, GAMMA, vertices=verts, vertex_attributes=make(),
                                                          background=bg, return_alpha=True)
                torch.autograd.backward((img, alpha), (g[C], g_a))
            return step

        variants = {"soft_depth_c1": attributes(lambda: verts[..., 2:3], 1, [FAR]),
                    "per_item_colours_c3": attributes(lambda: colours, 3, None),
                    "shared_features_c16": attributes(lambda: features, 16, None)}
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
