#!/usr/bin/env python
"""Phong shading through a specular map (specular_map=) against the same render without it: one JSON object.

Geometry and inputs: those of tools/bench_normal_map.py (bench.py's B 64 seeded spheres, F 5000, 256 x 256, indexed
vertices, a dense N(0,1) upstream gradient), with one shared 1024 x 1024 albedo image and one shared 1024 x 1024 specular
map, and every input requiring grad.  Variants, each alternated with its twin without the specular map within one command
(bench_phong.measure_pair): NL 0, NL 4 (bench_lights.py's mixed set), NL 4 with an SH environment, and NL 0 with a
1024 x 1024 normal map (its twin keeps the normal map).  Every repetition times `steps` steps of each arm in turn (CUDA
events); the result is the median [min, max] over `reps` repetitions.  Per kernel: the library's own CUDA-event profiler
over `steps` further steps.

    python tools/bench_specular_map.py [--steps 20] [--warmup 3] [--reps 5]
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
    a = ap.parse_args()
    dev = torch.device("cuda")
    B, F, S = a.batch, a.faces, a.size
    lib = _lib.load()
    gen = torch.Generator().manual_seed(0)
    faces0 = torch.from_numpy(synthetic.sphere_faces(B, F)).to(dev)
    verts0 = faces0.reshape(B, 3 * F, 3).contiguous()
    idx = torch.arange(3 * F, device=dev, dtype=torch.int32).reshape(F, 3)
    image = torch.rand((1, 1024, 1024, 3), generator=gen).to(dev)
    smap = torch.cat((0.2 + torch.rand((1, 1024, 1024, 3), generator=gen),
                      4.0 + 60.0 * torch.rand((1, 1024, 1024, 1), generator=gen)), -1).to(dev)
    nmap = torch.randn((1, 1024, 1024, 3), generator=gen) * 0.2
    nmap[..., 2] = 1.0
    nmap = nmap.to(dev).requires_grad_(True)
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
                     "image": [1024, 1024], "specular_map": [1024, 1024], "grad": "every input"},
           "variants": {}}
    for label, lt, e, nm in (("NL0", None, None, None), ("NL4", lights4, None, None), ("NL4_sh", lights4, sh, None),
                             ("NL0_nm", None, None, nmap)):
        geom = verts0.clone().requires_grad_(True)
        tex = image.clone().requires_grad_(True)
        uv = uvs.clone().requires_grad_(True)
        sm = smap.clone().requires_grad_(True)
        steps = {}
        for arm, with_map in (("without", False), ("specular_map", True)):
            def step(lt=lt, e=e, nm=nm, with_map=with_map):
                for t in (geom, tex, uv, cs, params, lights4, sh, nmap, tg, sm):
                    t.grad = None
                nb.rasterize(idx, tex, S, False, vertices=geom, face_uvs=uv, corner_shading=cs, shading_params=params,
                             lights=lt, environment_sh=e, normal_map=nm, corner_tangents=tg if nm is not None else None,
                             specular_map=sm if with_map else None).backward(g)
            steps[arm] = step
        out["variants"][label] = measure_pair(steps, a, lib)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
