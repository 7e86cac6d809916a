#!/usr/bin/env python
"""Phong shading with a light set (lights=) against Phong alone: one JSON object.

Geometry and inputs: those of tools/bench_phong.py (bench.py's B 64 seeded spheres, F 5000, 256 x 256, indexed vertices,
textures, corner_shading, shading_params and the lights requiring grad, a dense N(0,1) upstream gradient), for
  cubes_ts4        per-face cubes ts 4
  image            one shared 1024 x 1024 texture image, bilinear
  image_trilinear  the same image through its mip pyramid
Variants per geometry: NL 0 (Phong alone), and NL 1, 4, 8 lights of a mixed set (point lights with falloff and
directional lights alternating, one set for every item).  All variants of a geometry are alternated within one command:
after warming each up, every repetition times `steps` steps of each in turn (CUDA events); the result is the median
[min, max] over `reps` repetitions.  Per kernel: the library's own CUDA-event profiler over `steps` further steps.

    python tools/bench_lights.py [--steps 20] [--warmup 3] [--reps 5] [--only name,name,...]
"""
import argparse
import json
import math
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import neural_renderer_b200 as nb  # noqa: E402
from neural_renderer_b200 import _lib, synthetic  # noqa: E402
from bench_attributes import gpu_info  # noqa: E402
from bench_phong import measure_pair  # noqa: E402

NAMES = ["cubes_ts4", "image", "image_trilinear"]
COUNTS = [0, 1, 4, 8]


def mixed_lights(n, dev):
    """n records: point lights (falloff 0.2) and directional lights alternating, around the spheres (z 1.95 .. 3.55)"""
    F = nb.functional
    recs = []
    for j in range(n):
        t = 2.0 * math.pi * j / 8
        if j % 2 == 0:
            recs.append(F.point_light((1.5 * math.cos(t), 1.5 * math.sin(t), 0.5), 0.4, intensity_specular=0.3, falloff=0.2,
                                      device=dev))
        else:
            recs.append(F.directional_light((math.cos(t), 0.5, -1.0), 0.3, intensity_specular=0.2, device=dev))
    return F.light_set(*recs) if recs else torch.zeros((1, 0, 12), device=dev)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--faces", type=int, default=5000)
    ap.add_argument("--size", type=int, default=256)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--only", default=None, help="comma-separated geometry names, run in this order")
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
    normals = torch.nn.functional.normalize(torch.randn((B, F, 3, 3), generator=gen), dim=-1)
    cs = torch.cat((normals, faces0.cpu()), dim=-1).to(dev).requires_grad_(True)
    params = nb.functional.phong_params(0.4, 0.6, 0.3, direction=(0.3, 0.5, -1.0), shininess=32.0, eye=(0.0, 0.0, -3.0),
                                        device=dev).clone().requires_grad_(True)
    lights = {n: mixed_lights(n, dev).clone().requires_grad_(n > 0) for n in COUNTS}
    g = torch.randn((B, 3, S, S), generator=gen).to(dev)
    out = {"gpu": gpu_info(dev),
           "shape": {"batch": B, "faces": F, "size": S, "anti_aliasing": False, "indexed": True, "grad": "vertices"},
           "variants": {}}
    for name in (a.only.split(",") if a.only else NAMES):
        geom = verts0.clone().requires_grad_(True)
        if name == "cubes_ts4":
            tex, kw = cubes.clone().requires_grad_(True), {}
        else:
            tex = image.clone().requires_grad_(True)
            kw = dict(face_uvs=uvs, texture_filter="trilinear" if name == "image_trilinear" else "bilinear")
        steps = {}
        for n, lt in lights.items():
            def step(lt=lt):
                geom.grad = tex.grad = cs.grad = params.grad = lt.grad = None
                nb.rasterize(idx, tex, S, False, vertices=geom, corner_shading=cs, shading_params=params, lights=lt,
                             **kw).backward(g)
            steps["NL%d" % n] = step
        out["variants"][name] = measure_pair(steps, a, lib)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
