#!/usr/bin/env python
"""The interior vertex gradient of the RGB image (interior_gradient=True, k_interior_grad) at the headline geometry: one
JSON object.

Geometry: bench.py's B 64 seeded spheres (synthetic.sphere_faces), F 5000, 256 x 256, no anti-aliasing, a dense N(0,1)
upstream gradient; every step is rasterize + its backward.  The geometry is indexed, vertices requiring grad (the faces
viewed as [B,3F,3] vertices, every corner its own vertex, as tools/bench_attributes.py), so the kernels scatter into
grad_vertices.  Each variant runs with the flag off and
then on, right next to each other:
  cubes_ts4        per-face cubes ts 4, every item with its own depths (reference_exact=False)
  image            one shared 1024 x 1024 texture image, bilinear (synthetic.sphere_uvs)
  image_trilinear  the same image through its mip pyramid
  ..._smooth       the same with a per-corner light (smooth shading)
  teapot_smooth    Renderer.render of the teapot, 256 x 256 with anti-aliasing, batch 8, smooth shading, a 1024^2 image
Whole step: CUDA events around `steps` steps after `warmup` warm-up steps, median [min, max] over `reps` repetitions.
Per kernel: the library's own CUDA-event profiler over `steps` further steps (microseconds per step).  k_interior_grad's
algorithmic bytes are the maps and the upstream gradient it reads (face_index_map + weight_map + 3 gradient planes, 28 B
per raster pixel) before any texture or vertex tap; over the data-sheet HBM figure they give its floor.

    python tools/bench_interior.py [--steps 20] [--warmup 3] [--reps 5] [--only name,name,...]
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
from bench_attributes import HBM_GBS, gpu_info, measure  # noqa: E402

NAMES = ["cubes_ts4", "cubes_ts4_smooth", "image", "image_smooth", "image_trilinear", "image_trilinear_smooth",
         "teapot_smooth"]


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
    gen = torch.Generator().manual_seed(0)
    faces0 = torch.from_numpy(synthetic.sphere_faces(B, F)).to(dev)
    verts0 = faces0.reshape(B, 3 * F, 3).contiguous()
    idx = torch.arange(3 * F, device=dev, dtype=torch.int32).reshape(F, 3)
    cubes = torch.rand((B, F, 4, 4, 4, 3), generator=gen).to(dev)
    image = torch.rand((1, 1024, 1024, 3), generator=gen).to(dev)
    uvs = torch.from_numpy(synthetic.sphere_uvs(F)).to(dev)
    corner = (0.5 + torch.rand((B, F, 3, 3), generator=gen)).to(dev)
    g = torch.randn((B, 3, S, S), generator=gen).to(dev)
    nbytes = B * S * S * 28
    out = {"gpu": gpu_info(dev), "hbm_gbs_datasheet": HBM_GBS,
           "shape": {"batch": B, "faces": F, "size": S, "anti_aliasing": False, "indexed": True, "grad": "vertices"},
           "k_interior_grad_bytes": nbytes, "k_interior_grad_floor_us": nbytes / (HBM_GBS * 1e3), "variants": {}}
    for name in (a.only.split(",") if a.only else NAMES):
        for on in (False, True):
            key = "%s_%s" % (name, "on" if on else "off")
            if name == "teapot_smooth":
                Bt = 8
                d = np.load(os.path.join(ROOT, "tests", "golden", "teapot.npz"))
                v = torch.from_numpy(np.stack([d["vertices"]] * Bt)).to(dev).requires_grad_(True)
                f = torch.from_numpy(np.stack([d["faces"]] * Bt)).to(dev)
                tuv = torch.rand((f.shape[1], 3, 2), generator=gen).to(dev)
                gt = torch.randn((Bt, 3, 256, 256), generator=gen).to(dev)
                r = nb.Renderer()
                r.eye = nb.get_points_from_angles(2.732, 30, 40)
                r.shading, r.interior_gradient = "smooth", on

                def step():
                    v.grad = None
                    r.render(v, f, image, face_uvs=tuv).backward(gt)
                rec = measure(step, a, lib)
                rec["shape"] = {"batch": Bt, "faces": int(f.shape[1]), "size": 256, "anti_aliasing": True, "fill_back": True}
                out["variants"][key] = rec
                continue
            geom = verts0.clone().requires_grad_(True)
            smooth = name.endswith("_smooth")
            base = name[:-len("_smooth")] if smooth else name
            kw = dict(reference_exact=False, corner_light=corner if smooth else None, interior_gradient=on)
            if base == "cubes_ts4":
                tex = cubes
            else:
                tex = image
                kw.update(face_uvs=uvs, texture_filter="trilinear" if base == "image_trilinear" else "bilinear")

            def step():
                geom.grad = None
                nb.rasterize(idx, tex, S, False, vertices=geom, **kw).backward(g)
            rec = measure(step, a, lib)
            t = rec["kernels_us_per_step"].get("k_interior_grad")
            if t:
                rec["k_interior_grad_gbs"] = nbytes / (t * 1e3)
            out["variants"][key] = rec
    print(json.dumps(out))


if __name__ == "__main__":
    main()
