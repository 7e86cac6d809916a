#!/usr/bin/env python
"""The soft blend of fragments (blend_soft_fragments) against the same pipeline blended in torch, at the headline
geometry: one JSON object.

Geometry: bench.py's B 64 seeded spheres (synthetic.sphere_faces), F 5000, 256 x 256, sigma 1e-4, gamma 1e-4, faces and
per-corner colours requiring grad; every step is rasterize_soft_fragments + functional.interpolate_face_attributes +
the blend, forward plus backward with a dense N(0,1) upstream gradient on the image and on alpha.  Arms: "fused" (the
CUDA blend) and "torch" (the same blend written in torch, as tests/test_gpu_soft_frag.py's _blend, plus alpha), checked
to agree in one step (image, alpha and both gradients finite and within 1 % of the largest value) before any timing, then
alternated repetition by repetition so that both see the same clocks; the torch arm is skipped where its estimated peak (14 tensors
of [B,H,W,K,C] floats on top of the fused arm's) would pass 40 GB.  Shapes: K in {1, 8, 32} at C 3, and K 8 at C 16.
Whole step: CUDA events around `steps` steps after `warmup` warm-up steps, median [min, max] over `reps` repetitions.
Per kernel: torch.profiler (CUDA activity) over `steps` further steps in a run of its own, microseconds per step.
Peak: torch.cuda.max_memory_allocated of one step of each arm.

HBM floors: the forward reads 8K + 4K + 4K + 4KC bytes per pixel (pix_to_face, zbuf, dists, colours) and writes 4C + 4
(out, alpha); the backward reads the same plus 8C + 4 (out, grad_out, grad_alpha) and writes 4KC + 8K (grad_colors,
grad_zbuf, grad_dists).  Each floor is those bytes over the data sheet's 3.35 TB/s HBM3 bandwidth of the H100 SXM;
floor_share is the floor over the measured kernel time.  The card's name and power limit are read in the same call.

    python tools/bench_soft_blend.py [--steps 20] [--warmup 3] [--reps 5]
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
from neural_renderer_b200 import functional as Fn  # noqa: E402
from neural_renderer_b200 import synthetic  # noqa: E402
from bench_soft_silhouettes import gpu_info, summary, time_step  # noqa: E402

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet
NEAR, FAR = 0.1, 100.0
TORCH_PEAK_CAP = 40e9


def profile_kernels(step, n):
    """device microseconds per step of every kernel of `n` steps (torch.profiler, CUDA activity): the ten largest, plus
    every blend kernel whatever its rank"""
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
    ranked = sorted(out.items(), key=lambda kv: -kv[1])
    return dict(ranked[:10] + [kv for kv in ranked[10:] if "k_soft_blend" in kv[0]])


def torch_blend(frag, colors, sigma, gamma):
    """SoftRas's blend in torch (the fragment tests' _blend, with alpha): [B,C,H,W], [B,H,W].  Empty slots hold -1 in
    zbuf and dists, so their depth and distance are replaced before the exponent: masking only the product would give
    0 * inf = NaN where exp((zn - zmax) / gamma) overflows, in the forward and in the backward."""
    p2f, zbuf, _, dists = frag
    sel = p2f >= 0
    zn = (FAR - zbuf) / (FAR - NEAR)
    zmax = torch.where(sel, zn, torch.full_like(zn, -torch.inf)).amax(-1, keepdim=True).clamp_min(1e-3).detach()
    zn = torch.where(sel, zn, zmax)
    D = torch.where(sel, torch.sigmoid(torch.where(sel, dists, torch.zeros_like(dists)) / sigma), torch.zeros_like(zn))
    w = D * torch.exp((zn - zmax) / gamma)
    wb = torch.exp((1e-3 - zmax) / gamma)
    out = ((w[..., None] * colors).sum(-2)) / (w.sum(-1, keepdim=True) + wb)
    alpha = 1 - torch.prod(1 - D, -1)
    return out.permute(0, 3, 1, 2), alpha


def check_arms_agree(faces, ca, S, sigma, gamma, K, g_img, g_a):
    """one step of each arm: the same image and alpha within fp32 rounding of the two exponent forms, finite gradients
    that agree; raises before any timing otherwise"""
    res = []
    for blend in (lambda fr, col: nb.blend_soft_fragments(fr, col, sigma, gamma, NEAR, FAR),
                  lambda fr, col: torch_blend(fr, col, sigma, gamma)):
        fr = nb.rasterize_soft_fragments(faces, S, sigma, K)
        col = Fn.interpolate_face_attributes(fr.pix_to_face, fr.bary_coords, ca)
        img, alpha = blend(fr, col)
        gf, gc = torch.autograd.grad((img, alpha), (faces, ca), (g_img, g_a))
        res.append([t.detach() for t in (img, alpha, gf, gc)])
    for name, x, y in zip(("image", "alpha", "grad_faces", "grad_colors"), *res):
        if not (torch.isfinite(x).all() and torch.isfinite(y).all()):
            raise RuntimeError("%s: not finite (fused %s, torch %s)" % (name, bool(torch.isfinite(x).all()),
                                                                         bool(torch.isfinite(y).all())))
        err = ((x - y).abs().max() / y.abs().max().clamp_min(1e-30)).item()
        if err > 1e-2:
            raise RuntimeError("%s: the arms differ by %.3g of the largest value" % (name, err))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--faces", type=int, default=5000)
    ap.add_argument("--size", type=int, default=256)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--shapes", default="1x3,8x3,32x3,8x16", help="K x C pairs")
    a = ap.parse_args()
    dev = torch.device("cuda")
    B, F, S = a.batch, a.faces, a.size
    sigma = gamma = 1e-4
    gen = torch.Generator().manual_seed(0)
    faces = torch.from_numpy(synthetic.sphere_faces(B, F)).to(dev).requires_grad_(True)
    out = {"gpu": gpu_info(dev), "library": os.environ.get("NR_B200_LIB", "default"),
           "shape": {"batch": B, "faces": F, "size": S, "sigma": sigma, "gamma": gamma}, "shapes": {}}
    for kc in a.shapes.split(","):
        K, C = (int(v) for v in kc.split("x"))
        ca = torch.rand((B, F, 3, C), generator=gen).to(dev).requires_grad_(True)
        g_img = torch.randn((B, C, S, S), generator=gen).to(dev)
        g_a = torch.randn((B, S, S), generator=gen).to(dev)

        def step(blend):
            def run():
                faces.grad = None
                ca.grad = None
                fr = nb.rasterize_soft_fragments(faces, S, sigma, K)
                col = Fn.interpolate_face_attributes(fr.pix_to_face, fr.bary_coords, ca)
                img, alpha = blend(fr, col)
                torch.autograd.backward((img, alpha), (g_img, g_a))
            return run

        steps = {"fused": step(lambda fr, col: nb.blend_soft_fragments(fr, col, sigma, gamma, NEAR, FAR)),
                 "torch": step(lambda fr, col: torch_blend(fr, col, sigma, gamma))}
        rec = {}
        if 14 * 4.0 * B * S * S * K * C > TORCH_PEAK_CAP:
            del steps["torch"]
            rec["torch_skipped"] = "estimated peak past %.0f GB" % (TORCH_PEAK_CAP / 1e9)
        else:
            check_arms_agree(faces, ca, S, sigma, gamma, K, g_img, g_a)
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
            rec[k]["kernels_us_per_step"] = profile_kernels(steps[k], a.steps)
        if "torch" in steps:
            rec["fused_over_torch_median"] = rec["fused"]["step_ms_median"] / rec["torch"]["step_ms_median"]
        npix = B * S * S
        floors = {"k_soft_blend_fwd": (16.0 * K + 4.0 * K * C + 4.0 * C + 4.0) * npix / HBM_BYTES_PER_S * 1e3,
                  "k_soft_blend_bwd": (16.0 * K + 4.0 * K * C + 8.0 * C + 4.0 + 4.0 * K * C + 8.0 * K) * npix
                  / HBM_BYTES_PER_S * 1e3}
        kern = rec["fused"]["kernels_us_per_step"]
        for name, floor_ms in floors.items():
            t_us = sum(v for kk, v in kern.items() if name in kk)
            rec[name] = {"floor_ms": floor_ms, "kernel_ms": t_us / 1e3,
                         "floor_share": floor_ms / (t_us / 1e3) if t_us > 0 else None}
        out["shapes"]["K%d_C%d" % (K, C)] = rec
        del ca, g_img, g_a
    print(json.dumps(out))


if __name__ == "__main__":
    main()
