#!/usr/bin/env python
"""Phong shading (corner_shading / shading_params) against its smooth-shaded counterpart (corner_light): one JSON object.

Geometry: bench.py's B 64 seeded spheres (synthetic.sphere_faces), F 5000, 256 x 256, no anti-aliasing, a dense N(0,1)
upstream gradient; every step is rasterize + its backward, with the vertices (indexed, every corner its own vertex, as
tools/bench_interior.py), the textures and the light inputs requiring grad:
  cubes_ts4        per-face cubes ts 4
  image            one shared 1024 x 1024 texture image, bilinear (synthetic.sphere_uvs)
  image_trilinear  the same image through its mip pyramid
  teapot           Renderer.render of the teapot, 256 x 256 with anti-aliasing, batch 8, cubes ts 2 (shading 'smooth' vs
                   'phong', the default light attributes)
Each pair (smooth, phong) is alternated within one command: after warming both up, every repetition times `steps` smooth
steps, then `steps` Phong steps (CUDA events); the result is the median [min, max] over `reps` repetitions.  Per kernel:
the library's own CUDA-event profiler over `steps` further steps of each (microseconds per step).

    python tools/bench_phong.py [--steps 20] [--warmup 3] [--reps 7] [--only name,name,...]
"""
import argparse
import collections
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
from bench_attributes import gpu_info  # noqa: E402

NAMES = ["cubes_ts4", "image", "image_trilinear", "teapot"]


def _time(step, steps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        step()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def _kernels(step, steps, lib):
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


def measure_pair(steps_by_name, a, lib):
    for step in steps_by_name.values():
        for _ in range(a.warmup):
            step()
    torch.cuda.synchronize()
    reps = {k: [] for k in steps_by_name}
    for _ in range(a.reps):
        for k, step in steps_by_name.items():
            reps[k].append(_time(step, a.steps))
    out = {}
    for k, step in steps_by_name.items():
        r = reps[k]
        out[k] = {"step_ms_median": float(np.median(r)), "step_ms_min_max": [min(r), max(r)], "step_ms_reps": r,
                  "kernels_us_per_step": _kernels(step, a.steps, lib)}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--faces", type=int, default=5000)
    ap.add_argument("--size", type=int, default=256)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--only", default=None, help="comma-separated variant names, run in this order")
    a = ap.parse_args()
    dev = torch.device("cuda")
    B, F, S = a.batch, a.faces, a.size
    lib = _lib.load()
    gen = torch.Generator().manual_seed(0)
    faces0 = torch.from_numpy(synthetic.sphere_faces(B, F)).to(dev)
    verts0 = faces0.reshape(B, 3 * F, 3).contiguous()
    idx = torch.arange(3 * F, device=dev, dtype=torch.int32).reshape(F, 3)
    cubes = torch.rand((B, F, 4, 4, 4, 3), generator=gen).to(dev)
    image = torch.rand((1, 1024, 1024, 3), generator=gen).to(dev)
    uvs = torch.from_numpy(synthetic.sphere_uvs(F)).to(dev)
    corner = (0.5 + torch.rand((B, F, 3, 3), generator=gen)).to(dev).requires_grad_(True)
    normals = torch.nn.functional.normalize(torch.randn((B, F, 3, 3), generator=gen), dim=-1)
    cs = torch.cat((normals, faces0.cpu()), dim=-1).to(dev).requires_grad_(True)
    params = nb.functional.phong_params(0.4, 0.6, 0.3, direction=(0.3, 0.5, -1.0), shininess=32.0, eye=(0.0, 0.0, -3.0),
                                        device=dev).clone().requires_grad_(True)
    g = torch.randn((B, 3, S, S), generator=gen).to(dev)
    out = {"gpu": gpu_info(dev),
           "shape": {"batch": B, "faces": F, "size": S, "anti_aliasing": False, "indexed": True, "grad": "vertices"},
           "variants": {}}
    for name in (a.only.split(",") if a.only else NAMES):
        if name == "teapot":
            Bt = 8
            d = np.load(os.path.join(ROOT, "tests", "golden", "teapot.npz"))
            v = torch.from_numpy(np.stack([d["vertices"]] * Bt)).to(dev).requires_grad_(True)
            f = torch.from_numpy(np.stack([d["faces"]] * Bt)).to(dev)
            tex = torch.rand((Bt, f.shape[1], 2, 2, 2, 3), generator=gen).to(dev).requires_grad_(True)
            gt = torch.randn((Bt, 3, 256, 256), generator=gen).to(dev)
            steps = {}
            for shading in ("smooth", "phong"):
                r = nb.Renderer()
                r.eye = nb.get_points_from_angles(2.732, 30, 40)
                r.shading = shading

                def step(r=r):
                    v.grad = tex.grad = None
                    r.render(v, f, tex).backward(gt)
                steps[shading] = step
            rec = measure_pair(steps, a, lib)
            out["variants"]["teapot"] = {"shape": {"batch": Bt, "faces": int(f.shape[1]), "size": 256, "anti_aliasing": True,
                                                   "fill_back": True}, **rec}
            continue
        geom = verts0.clone().requires_grad_(True)
        if name == "cubes_ts4":
            tex, kw = cubes.clone().requires_grad_(True), {}
        else:
            tex = image.clone().requires_grad_(True)
            kw = dict(face_uvs=uvs, texture_filter="trilinear" if name == "image_trilinear" else "bilinear")
        steps = {}
        for shading, extra in (("smooth", dict(corner_light=corner)),
                               ("phong", dict(corner_shading=cs, shading_params=params))):
            def step(extra=extra):
                geom.grad = tex.grad = corner.grad = cs.grad = params.grad = None
                nb.rasterize(idx, tex, S, False, vertices=geom, **kw, **extra).backward(g)
            steps[shading] = step
        out["variants"][name] = measure_pair(steps, a, lib)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
