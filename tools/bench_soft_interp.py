#!/usr/bin/env python
"""The soft interpolation of fragments (interpolate_soft_fragments) against functional.interpolate_face_attributes in
the same fragment pipeline, at the headline geometry: one JSON object.

Geometry: bench.py's B 64 seeded spheres (synthetic.sphere_faces), F 5000, 256 x 256, sigma 1e-4, gamma 1e-4; every
step is rasterize_soft_fragments + the interpolation + blend_soft_fragments, forward plus backward with a dense N(0,1)
upstream gradient on the image and on alpha, faces and attributes requiring grad.  Shapes: K in {1, 8, 32} at C 3 and
K 8 at C 16 with per-corner colours [B,F,3,C]; and "pv_K8_C3": per-vertex colours [B,Nv,3] on the same spheres as
indexed vertices (synthetic.sphere_mesh per item, rotated and jittered as sphere_faces), vertices and colours requiring
grad, whose torch arm gathers colours[:, faces] first.  Arms: "cuda" (interpolate_soft_fragments) and "torch"
(interpolate_face_attributes), checked to agree in one step (image, alpha and both gradients finite and within 1e-3 of
the largest value) before any timing, then alternated repetition by repetition so that both see the same clocks; the
torch arm is skipped where its estimated peak (8 tensors of [B,H,W,K,C] floats) would pass 40 GB.
Whole step: CUDA events around `steps` steps after `warmup` warm-up steps, median [min, max] over `reps` repetitions.
Peak: torch.cuda.max_memory_allocated of one step of each arm.
Per kernel: torch.profiler (CUDA activity) over `steps` further steps in a run of its own, microseconds per step: the
ten largest kernels, every interpolation kernel, and "torch_kernels_us_per_step", the sum of every kernel that is not
the project's (k_*) and not a memset: in the torch arm that is the torch interpolation (forward and backward) plus the
glue both arms share, which the cuda arm's own sum measures.

HBM floors: the forward reads 8 + 12 bytes per slot (pix_to_face, bary) and writes 4C (out); the backward reads
8 + 12 + 4C (pix_to_face, bary, grad_out) and writes 12 (grad_bary); the attribute reads and the attribute gradient's
scatter stay in L2 and are not counted.  Each floor is those bytes over the data sheet's 3.35 TB/s HBM3 bandwidth of
the H100 SXM; floor_share is the floor over the measured kernel time.  The card's name and power limit are read in the
same call.

    python tools/bench_soft_interp.py [--steps 20] [--warmup 3] [--reps 5] [--shapes 1x3,8x3,32x3,8x16,pv8x3]
                                      [--arms cuda,torch]
"""
import argparse
import json
import os
import re
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import neural_renderer_b200 as nb  # noqa: E402
from neural_renderer_b200 import functional as Fn  # noqa: E402
from neural_renderer_b200 import synthetic  # noqa: E402
from bench_soft_silhouettes import gpu_info, summary, time_step  # noqa: E402

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet
NEAR, FAR = 0.1, 100.0
TORCH_PEAK_CAP = 40e9
INTERP_KERNELS = ("k_soft_interp_fwd", "k_soft_interp_bwd")


def profile_kernels(step, n):
    """device microseconds per step of every kernel of `n` steps (torch.profiler, CUDA activity): the ten largest, every
    interpolation kernel, and the sum of the kernels that are not the project's and not memsets"""
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
            out[e.key] = t / n
    ranked = sorted(out.items(), key=lambda kv: -kv[1])
    keep = dict((k[:80], round(v, 1)) for k, v in ranked[:10] + [kv for kv in ranked[10:]
                                                                   if any(s in kv[0] for s in INTERP_KERNELS)])
    torch_us = sum(v for k, v in out.items() if not re.search(r"(^|::|\s)k_\w", k) and "memset" not in k.lower())
    return keep, round(torch_us, 1)


def sphere_vertices(B, F, radius=0.8, jitter=0.01, z_center=2.75, seed=1234):
    """[B,Nv,3] float32 indexed vertices and [F,3] int32 faces of synthetic.sphere_faces' spheres"""
    v0, faces = synthetic.sphere_mesh(F)
    out = np.empty((B,) + v0.shape, dtype=np.float32)
    for b in range(B):
        rng = np.random.default_rng(seed + b)
        v = (v0 * radius) @ synthetic._rotation(rng).T
        v = v + rng.normal(scale=jitter, size=v.shape)
        v[:, 2] += z_center
        out[b] = v
    return out, faces


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--faces", type=int, default=5000)
    ap.add_argument("--size", type=int, default=256)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--shapes", default="1x3,8x3,32x3,8x16,pv8x3", help="K x C pairs, pv: per-vertex colours")
    ap.add_argument("--arms", default="cuda,torch")
    a = ap.parse_args()
    dev = torch.device("cuda")
    B, F, S = a.batch, a.faces, a.size
    sigma = gamma = 1e-4
    gen = torch.Generator().manual_seed(0)
    faces = torch.from_numpy(synthetic.sphere_faces(B, F)).to(dev).requires_grad_(True)
    vnp, fnp = sphere_vertices(B, F)
    verts = torch.from_numpy(vnp).to(dev).requires_grad_(True)
    findex = torch.from_numpy(fnp).to(dev)
    fl = findex.long()
    out = {"gpu": gpu_info(dev), "library": os.environ.get("NR_B200_LIB", "default"),
           "shape": {"batch": B, "faces": F, "size": S, "sigma": sigma, "gamma": gamma, "vertices": vnp.shape[1]},
           "shapes": {}}
    for kc in a.shapes.split(","):
        pv = kc.startswith("pv")
        K, C = (int(v) for v in kc.lstrip("pv").split("x"))
        if pv:
            attrs = torch.rand((B, vnp.shape[1], C), generator=gen).to(dev).requires_grad_(True)
            geom = verts
            arms = {"cuda": lambda fr, at: nb.interpolate_soft_fragments(fr, vertex_attributes=at, faces=findex),
                    "torch": lambda fr, at: Fn.interpolate_face_attributes(fr.pix_to_face, fr.bary_coords, at[:, fl])}
            rasterize = lambda: nb.rasterize_soft_fragments(findex, S, sigma, K, vertices=verts)  # noqa: E731
        else:
            attrs = torch.rand((B, F, 3, C), generator=gen).to(dev).requires_grad_(True)
            geom = faces
            arms = {"cuda": lambda fr, at: nb.interpolate_soft_fragments(fr, at),
                    "torch": lambda fr, at: Fn.interpolate_face_attributes(fr.pix_to_face, fr.bary_coords, at)}
            rasterize = lambda: nb.rasterize_soft_fragments(faces, S, sigma, K)  # noqa: E731
        arms = {k: v for k, v in arms.items() if k in a.arms.split(",")}
        g_img = torch.randn((B, C, S, S), generator=gen).to(dev)
        g_a = torch.randn((B, S, S), generator=gen).to(dev)

        def step(interp):
            def run():
                geom.grad = None
                attrs.grad = None
                fr = rasterize()
                img, alpha = nb.blend_soft_fragments(fr, interp(fr, attrs), sigma, gamma, NEAR, FAR)
                torch.autograd.backward((img, alpha), (g_img, g_a))
            return run

        def one(interp):
            fr = rasterize()
            img, alpha = nb.blend_soft_fragments(fr, interp(fr, attrs), sigma, gamma, NEAR, FAR)
            gg, ga = torch.autograd.grad((img, alpha), (geom, attrs), (g_img, g_a))
            return [t.detach() for t in (img, alpha, gg, ga)]

        steps = {k: step(v) for k, v in arms.items()}
        rec = {}
        if "torch" in steps and 8 * 4.0 * B * S * S * K * C > TORCH_PEAK_CAP:
            del steps["torch"]
            rec["torch_skipped"] = "estimated peak past %.0f GB" % (TORCH_PEAK_CAP / 1e9)
        if len(steps) == 2:
            res = [one(arms["cuda"]), one(arms["torch"])]
            for name, x, y in zip(("image", "alpha", "grad_geometry", "grad_attributes"), *res):
                if not (torch.isfinite(x).all() and torch.isfinite(y).all()):
                    raise RuntimeError("%s: not finite" % name)
                err = ((x - y).abs().max() / y.abs().max().clamp_min(1e-30)).item()
                if err > 1e-3:
                    raise RuntimeError("%s: the arms differ by %.3g of the largest value" % (name, err))
                rec.setdefault("arms_max_rel_diff", {})[name] = err
            del res
        for k, s in steps.items():
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats(dev)
            s()
            torch.cuda.synchronize()
            rec.setdefault(k, {})["peak_bytes"] = torch.cuda.max_memory_allocated(dev)
        for _ in range(a.warmup):
            for s in steps.values():
                s()
        torch.cuda.synchronize()
        reps = {k: [] for k in steps}
        for _ in range(a.reps):  # alternate: both arms see the same clocks
            for k, s in steps.items():
                reps[k].append(time_step(s, a.steps))
        for k in steps:
            rec[k].update(summary(reps[k]))
            rec[k]["kernels_us_per_step"], rec[k]["torch_kernels_us_per_step"] = profile_kernels(steps[k], a.steps)
        if len(steps) == 2:
            rec["cuda_over_torch_median"] = rec["cuda"]["step_ms_median"] / rec["torch"]["step_ms_median"]
        if "cuda" in steps:
            nslot = B * S * S * K
            floors = {"k_soft_interp_fwd": (8.0 + 12.0 + 4.0 * C) * nslot / HBM_BYTES_PER_S * 1e3,
                      "k_soft_interp_bwd": (8.0 + 12.0 + 4.0 * C + 12.0) * nslot / HBM_BYTES_PER_S * 1e3}
            kern = rec["cuda"]["kernels_us_per_step"]
            for name, floor_ms in floors.items():
                t_us = sum(v for kk, v in kern.items() if name in kk)
                rec[name] = {"floor_ms": floor_ms, "kernel_ms": t_us / 1e3,
                             "floor_share": floor_ms / (t_us / 1e3) if t_us > 0 else None}
        out["shapes"][("pv_" if pv else "") + "K%d_C%d" % (K, C)] = rec
        del attrs, g_img, g_a, steps, arms
        torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
