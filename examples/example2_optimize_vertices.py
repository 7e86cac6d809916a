"""Example 2 of the reference (examples/example2.py:18-50, 61-98) with torch in place of Chainer: optimise the vertices
of a mesh so that its silhouette matches a target image.

The call sequence is the reference's: `neural_renderer.Renderer()`, `get_points_from_angles`, `render_silhouettes`,
sum of squared differences, Adam.  The target here is rendered from a squashed copy of the mesh instead of being read
from examples/data/example2_ref.png (no reference data is shipped in this repository).

    python examples/example2_optimize_vertices.py [--iters 100] [--out /tmp/example2.png] [--soft-sigma 1e-4]

--soft-sigma S fits the soft silhouette (Renderer.render_soft_silhouettes, softness S) to the target's soft silhouette
instead of the hard one: every face within reach of a pixel receives a gradient, not only the edges on the outline.
"""
import argparse
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import neural_renderer  # noqa: E402


class Model(torch.nn.Module):
    def __init__(self, vertices, faces, image_ref, soft_sigma=None):
        super().__init__()
        self.soft_sigma = soft_sigma
        self.vertices = torch.nn.Parameter(vertices[None, :, :])
        self.register_buffer("faces", faces[None, :, :])
        self.register_buffer("image_ref", image_ref)
        self.renderer = neural_renderer.Renderer()

    def forward(self):
        self.renderer.eye = neural_renderer.get_points_from_angles(2.732, 0, 90)
        if self.soft_sigma:
            image = self.renderer.render_soft_silhouettes(self.vertices, self.faces, self.soft_sigma)
        else:
            image = self.renderer.render_silhouettes(self.vertices, self.faces)
        return ((image - self.image_ref[None, :, :]) ** 2).sum()


def load_mesh():
    d = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden", "teapot.npz"))
    return torch.from_numpy(d["vertices"]), torch.from_numpy(d["faces"])


def run(iters=100, out=None, device="cuda", soft_sigma=None):
    vertices, faces = load_mesh()
    vertices, faces = vertices.to(device), faces.to(device)
    with torch.no_grad():  # target silhouette: the same mesh squashed along y
        r = neural_renderer.Renderer()
        r.eye = neural_renderer.get_points_from_angles(2.732, 0, 90)
        squashed = (vertices * torch.tensor([1.0, 0.6, 1.0], device=device))[None]
        if soft_sigma:
            target = r.render_soft_silhouettes(squashed, faces[None], soft_sigma)[0]
        else:
            target = r.render_silhouettes(squashed, faces[None])[0]
    model = Model(vertices, faces, target, soft_sigma).to(device)
    optimizer = neural_renderer.Adam(model.parameters(), lr=0.005)
    losses = []
    for _ in range(iters):
        optimizer.zero_grad()
        loss = model()
        loss.backward()
        optimizer.step()
        losses.append(float(loss.detach()))
    if out:
        from PIL import Image
        with torch.no_grad():
            img = model.renderer.render_silhouettes(model.vertices, model.faces)[0]
        Image.fromarray((img.clamp(0, 1) * 255).byte().cpu().numpy()).save(out)
    return losses


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--out", default=None)
    ap.add_argument("--soft-sigma", type=float, default=None,
                    help="fit soft silhouettes of this softness (e.g. 1e-4) instead of the hard ones")
    a = ap.parse_args()
    ls = run(a.iters, a.out, soft_sigma=a.soft_sigma)
    print("loss: first %.1f -> last %.1f" % (ls[0], ls[-1]))
