#!/usr/bin/env python
"""Phong shading through a tangent-space normal map (normal_map=, corner_tangents=) against the same render without it:
one JSON object.

Geometry and inputs: those of tools/bench_sh.py (bench.py's B 64 seeded spheres, F 5000, 256 x 256, indexed vertices, a
dense N(0,1) upstream gradient), with one shared 1024 x 1024 albedo image and one shared 1024 x 1024 normal map, and
every input requiring grad: vertices, the image, face_uvs, corner_shading, shading_params, the lights, the SH
coefficients, the map and the tangents.  Variants, each alternated with its Phong twin (the same render without the map)
within one command (bench_phong.measure_pair): NL 0 and NL 4 (bench_lights.py's mixed set), each without and with an SH
environment, for the bilinear image (and --trilinear: the image through its mip pyramid; the map stays bilinear).
Every repetition times `steps` steps of each variant in turn (CUDA events); the result is the median [min, max] over
`reps` repetitions.  Per kernel: the library's own CUDA-event profiler over `steps` further steps.

    python tools/bench_normal_map.py [--steps 20] [--warmup 3] [--reps 5] [--trilinear]
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--faces", type=int, default=5000)
    ap.add_argument("--size", type=int, default=256)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--trilinear", action="store_true", help="also the albedo through its mip pyramid")
    a = ap.parse_args()
    dev = torch.device("cuda")
    B, F, S = a.batch, a.faces, a.size
    lib = _lib.load()
    gen = torch.Generator().manual_seed(0)
    faces0 = torch.from_numpy(synthetic.sphere_faces(B, F)).to(dev)
    verts0 = faces0.reshape(B, 3 * F, 3).contiguous()
    idx = torch.arange(3 * F, device=dev, dtype=torch.int32).reshape(F, 3)
    image = torch.rand((1, 1024, 1024, 3), generator=gen).to(dev)
    nmap = torch.randn((1, 1024, 1024, 3), generator=gen) * 0.2
    nmap[..., 2] = 1.0
    nmap = nmap.to(dev)
    uvs = torch.from_numpy(synthetic.sphere_uvs(F)).to(dev)
    normals = torch.nn.functional.normalize(torch.randn((B, F, 3, 3), generator=gen), dim=-1)
    cs = torch.cat((normals, faces0.cpu()), dim=-1).to(dev).requires_grad_(True)
    tangents = torch.nn.functional.normalize(torch.randn((B, F, 3, 3), generator=gen), dim=-1)
    tg = torch.cat((tangents, torch.ones((B, F, 3, 1))), dim=-1).to(dev).requires_grad_(True)
    params = nb.functional.phong_params(0.4, 0.6, 0.3, direction=(0.3, 0.5, -1.0), shininess=32.0, eye=(0.0, 0.0, -3.0),
                                        device=dev).clone().requires_grad_(True)
    lights4 = mixed_lights(4, dev).clone().requires_grad_(True)
    env = 0.5 + 0.4 * torch.linspace(1.0, -1.0, 64)[:, None, None].expand(64, 128, 3) * torch.tensor([1.0, 0.9, 0.8])
    sh = nb.functional.sh_from_environment_map(env).to(dev).requires_grad_(True)
    g = torch.randn((B, 3, S, S), generator=gen).to(dev)
    out = {"gpu": gpu_info(dev),
           "shape": {"batch": B, "faces": F, "size": S, "anti_aliasing": False, "indexed": True,
                     "image": [1024, 1024], "normal_map": [1024, 1024], "grad": "every input"},
           "variants": {}}
    for tf in (("bilinear", "trilinear") if a.trilinear else ("bilinear",)):
        for label, lt, e in (("NL0", None, None), ("NL0_sh", None, sh), ("NL4", lights4, None), ("NL4_sh", lights4, sh)):
            geom = verts0.clone().requires_grad_(True)
            tex = image.clone().requires_grad_(True)
            uv = uvs.clone().requires_grad_(True)
            nm = nmap.clone().requires_grad_(True)
            steps = {}
            for arm, with_map in (("phong", False), ("normal_map", True)):
                def step(lt=lt, e=e, with_map=with_map):
                    for t in (geom, tex, uv, cs, params, lights4, sh, nm, tg):
                        t.grad = None
                    nb.rasterize(idx, tex, S, False, vertices=geom, face_uvs=uv, texture_filter=tf, corner_shading=cs,
                                 shading_params=params, lights=lt, environment_sh=e,
                                 normal_map=nm if with_map else None,
                                 corner_tangents=tg if with_map else None).backward(g)
                steps[arm] = step
            out["variants"]["%s_%s" % (tf, label)] = measure_pair(steps, a, lib)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
