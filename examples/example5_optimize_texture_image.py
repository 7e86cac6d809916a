"""Example 5 (not in the reference; follows example 3): optimise a 256 x 256 texture IMAGE of a UV-mapped model so that
renders from random viewpoints match renders of the model's own texture.  The model is tests/golden/display, loaded
with load_obj(texture_mode='uv'): its 7 materials (2 images) arrive as one atlas image plus per-corner UVs.

    python examples/example5_optimize_texture_image.py [--iters 50] [--size 256] [--texture-filter bilinear|trilinear]

A parameter image much larger than its footprint on screen (--size 1024 at the 256 x 256 renders) is minified: bilinear
sampling then aliases and gives most texels no gradient from a view; --texture-filter trilinear samples a mip pyramid of
it instead, so every texel receives gradient through the coarser levels.  --soft-sigma S [--soft-gamma G] fits through
the soft RGB image instead (Renderer.render_soft with face_uvs): every face within reach of a pixel, hidden ones
included, then sends gradient into the image.
"""
import argparse
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import neural_renderer  # noqa: E402
from neural_renderer_b200 import io  # noqa: E402


def run(iters=50, device="cuda", seed=0, size=256, texture_filter="bilinear", soft_sigma=None, soft_gamma=1e-4):
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden", "display", "model.obj")
    v, f, uv, image = io.load_obj(path, load_texture=True, texture_mode="uv")
    vertices = torch.from_numpy(v).to(device)[None]
    faces = torch.from_numpy(f).to(device)[None]
    face_uvs = torch.from_numpy(uv).to(device)
    target_image = torch.from_numpy(np.ascontiguousarray(image)).to(device)
    param = torch.zeros((size, size, 3), device=device, requires_grad=True)
    renderer = neural_renderer.Renderer()
    renderer.perspective = False
    renderer.texture_filter = texture_filter
    optimizer = neural_renderer.Adam([param], lr=0.1, betas=(0.5, 0.999))
    rng = np.random.default_rng(seed)
    losses = []
    for _ in range(iters):
        renderer.eye = neural_renderer.get_points_from_angles(2.732, float(rng.uniform(-30, 30)), float(rng.uniform(0, 360)))
        if soft_sigma is None:
            with torch.no_grad():
                target = renderer.render(vertices, faces, target_image, face_uvs=face_uvs)
            optimizer.zero_grad()
            image = renderer.render(vertices, faces, torch.sigmoid(param), face_uvs=face_uvs)
        else:
            with torch.no_grad():
                target = renderer.render_soft(vertices, faces, target_image, soft_sigma, soft_gamma, face_uvs=face_uvs)[0]
            optimizer.zero_grad()
            image = renderer.render_soft(vertices, faces, torch.sigmoid(param), soft_sigma, soft_gamma, face_uvs=face_uvs)[0]
        loss = ((image - target) ** 2).sum()
        loss.backward()
        optimizer.step()
        losses.append(float(loss.detach()))
    return losses


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--size", type=int, default=256)
    ap.add_argument("--texture-filter", default="bilinear", choices=("bilinear", "trilinear"))
    ap.add_argument("--soft-sigma", type=float, default=None, help="fit through the soft RGB image with this sigma")
    ap.add_argument("--soft-gamma", type=float, default=1e-4)
    args = ap.parse_args()
    ls = run(args.iters, size=args.size, texture_filter=args.texture_filter, soft_sigma=args.soft_sigma,
             soft_gamma=args.soft_gamma)
    print("loss: first %.1f -> last %.1f" % (ls[0], ls[-1]))
