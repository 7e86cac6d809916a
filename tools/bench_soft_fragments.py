#!/usr/bin/env python
"""Soft fragments (rasterize_soft_fragments) next to the soft silhouettes at the headline geometry: one JSON object.

Geometry: bench.py's B 64 seeded spheres (synthetic.sphere_faces), F 5000, 256 x 256, faces requiring grad; every step
is a forward plus a backward with dense N(0,1) upstream gradients on zbuf, bary_coords and dists.  Variants: sigma in
{1e-5, 1e-4, 1e-3} x K in {1, 8, 32}; each alternates, repetition by repetition, with rasterize_soft_silhouettes at the
same sigma (a dense upstream gradient on alpha), so both see the same clocks.  Whole step: CUDA events around `steps`
steps after `warmup` warm-up steps, median [min, max] over `reps` repetitions.  Per kernel: torch.profiler (CUDA
activity) over `steps` further steps in a run of its own, microseconds per step.

The forward writes 28 K bytes per pixel (8 pix_to_face, 4 zbuf, 12 bary, 4 dists): write_floor_ms is those bytes over
the data sheet's 3.35 TB/s HBM3 bandwidth of the H100 SXM, and floor_share that floor over the measured k_soft_frag_fwd
time.  The card's name and power limit are read in the same call.

    python tools/bench_soft_fragments.py [--steps 20] [--warmup 3] [--reps 5]
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

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--faces", type=int, default=5000)
    ap.add_argument("--size", type=int, default=256)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--sigmas", default="1e-5,1e-4,1e-3")
    ap.add_argument("--ks", default="1,8,32")
    a = ap.parse_args()
    dev = torch.device("cuda")
    B, F, S = a.batch, a.faces, a.size
    gen = torch.Generator().manual_seed(0)
    faces = torch.from_numpy(synthetic.sphere_faces(B, F)).to(dev).requires_grad_(True)
    g_a = torch.randn((B, S, S), generator=gen).to(dev)
    out = {"gpu": gpu_info(dev), "library": os.environ.get("NR_B200_LIB", "default"),
           "shape": {"batch": B, "faces": F, "size": S}, "sigmas": {}}
    for sigma in (float(s) for s in a.sigmas.split(",")):
        def silhouettes():
            faces.grad = None
            nb.rasterize_soft_silhouettes(faces, S, sigma).backward(g_a)

        rec = {}
        for K in (int(k) for k in a.ks.split(",")):
            ups = tuple(torch.randn(shape, generator=gen).to(dev) for shape in ((B, S, S, K), (B, S, S, K, 3), (B, S, S, K)))

            def frag():
                faces.grad = None
                fr = nb.rasterize_soft_fragments(faces, S, sigma, K)
                torch.autograd.backward((fr.zbuf, fr.bary_coords, fr.dists), ups)

            steps = {"fragments": frag, "silhouettes": silhouettes}
            for _ in range(a.warmup):
                for s in steps.values():
                    s()
            torch.cuda.synchronize()
            reps = {k: [] for k in steps}
            for _ in range(a.reps):  # alternate: both paths see the same clocks
                for k, s in steps.items():
                    reps[k].append(time_step(s, a.steps))
            r = {k: summary(v) for k, v in reps.items()}
            r["over_silhouettes_median"] = r["fragments"]["step_ms_median"] / r["silhouettes"]["step_ms_median"]
            kern = profile_kernels(frag, a.steps)
            r["kernels_us_per_step"] = kern
            floor_ms = 28.0 * K * B * S * S / HBM_BYTES_PER_S * 1e3
            fwd_us = sum(v for k, v in kern.items() if "k_soft_frag_fwd" in k)
            r["write_floor_ms"] = floor_ms
            r["fwd_kernel_ms"] = fwd_us / 1e3
            r["floor_share"] = floor_ms / (fwd_us / 1e3) if fwd_us > 0 else None
            rec["K%d" % K] = r
            del ups
        rec["silhouettes_kernels_us_per_step"] = profile_kernels(silhouettes, a.steps)
        out["sigmas"][repr(sigma)] = rec
    print(json.dumps(out))


if __name__ == "__main__":
    main()
