#!/usr/bin/env python
"""Phong shading with an SH environment (environment_sh=) against the same render without it: one JSON object.

Geometry and inputs: those of tools/bench_lights.py (bench.py's B 64 seeded spheres, F 5000, 256 x 256, indexed
vertices, textures, corner_shading, shading_params, the lights and the SH coefficients requiring grad, a dense N(0,1)
upstream gradient), for
  cubes_ts4        per-face cubes ts 4
  image            one shared 1024 x 1024 texture image, bilinear
  image_trilinear  the same image through its mip pyramid
Variants per geometry: Phong, Phong + SH, NL 4 (bench_lights.py's mixed set) and NL 4 + SH, one environment for every
item.  All variants of a geometry are alternated within one command (bench_phong.measure_pair): after warming each up,
every repetition times `steps` steps of each in turn (CUDA events); the result is the median [min, max] over `reps`
repetitions.  Per kernel: the library's own CUDA-event profiler over `steps` further steps.

    python tools/bench_sh.py [--steps 20] [--warmup 3] [--reps 5] [--only name,name,...]
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
from neural_renderer_b200 import _lib, synthetic  # noqa: E402
from bench_attributes import gpu_info  # noqa: E402
from bench_lights import mixed_lights  # noqa: E402
from bench_phong import measure_pair  # noqa: E402

NAMES = ["cubes_ts4", "image", "image_trilinear"]


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
    lights4 = mixed_lights(4, dev).clone().requires_grad_(True)
    # an environment brighter above than below, slightly coloured
    env = 0.5 + 0.4 * torch.linspace(1.0, -1.0, 64)[:, None, None].expand(64, 128, 3) * torch.tensor([1.0, 0.9, 0.8])
    sh = nb.functional.sh_from_environment_map(env).to(dev).requires_grad_(True)
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
        for label, lt, e in (("phong", None, None), ("phong_sh", None, sh), ("NL4", lights4, None),
                             ("NL4_sh", lights4, sh)):
            def step(lt=lt, e=e):
                geom.grad = tex.grad = cs.grad = params.grad = lights4.grad = sh.grad = None
                nb.rasterize(idx, tex, S, False, vertices=geom, corner_shading=cs, shading_params=params, lights=lt,
                             environment_sh=e, **kw).backward(g)
            steps[label] = step
        out["variants"][name] = measure_pair(steps, a, lib)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
