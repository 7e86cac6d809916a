"""Example 4 of the reference (examples/example4.py:18-57, 93-113) with torch in place of Chainer: find the camera
position from which a mesh's silhouette matches a target image.

The call sequence is the reference's: `Renderer()`, `renderer.eye = <parameter>`, `render_silhouettes`, sum of squared
differences, Adam(0.1).  The gradient reaches the camera through the fused look_at + perspective kernel
(`nr_b200_camera_transform_backward`: d loss / d eye through the translation and through the look_at rotation).  The
target is rendered from a known eye instead of being read from examples/data/example4_ref.png.

    python examples/example4_optimize_camera.py [--iters 200] [--soft-sigma 1e-4 --soft-gamma 1e-4]

--soft-sigma S fits the soft RGB image and soft silhouette (Renderer.render_soft, softness S, depth temperature
--soft-gamma G) of a textured teapot to the target's: the sum of squared differences of both.  Every face within reach
of a pixel sends the camera a gradient, and so does the colour, not only the silhouette's edges.
"""
import argparse
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import neural_renderer  # noqa: E402


class Model(torch.nn.Module):
    def __init__(self, vertices, faces, image_ref, start, textures=None, soft=None):
        super().__init__()
        self.register_buffer("vertices", vertices[None, :, :])
        self.register_buffer("faces", faces[None, :, :])
        self.register_buffer("image_ref", image_ref)
        self.textures = textures
        self.soft = soft  # (sigma, gamma) or None
        self.camera_position = torch.nn.Parameter(torch.tensor(start, dtype=torch.float32))
        self.renderer = neural_renderer.Renderer()
        self.renderer.eye = self.camera_position

    def forward(self):
        if self.soft:
            rgb, alpha = self.renderer.render_soft(self.vertices, self.faces, self.textures, *self.soft)
            return ((rgb - self.image_ref[None, :3]) ** 2).sum() + ((alpha - self.image_ref[None, 3]) ** 2).sum()
        image = self.renderer.render_silhouettes(self.vertices, self.faces)
        return ((image - self.image_ref[None, :, :]) ** 2).sum()


def teapot_textures(num_faces, device, ts=2):
    """per-face cubes coloured by face index (a fixed pattern the camera can be read from)"""
    g = torch.Generator().manual_seed(0)
    return torch.rand(1, num_faces, ts, ts, ts, 3, generator=g).to(device)


def run(iters=200, device="cuda", start=(6.0, 10.0, -14.0), soft_sigma=None, soft_gamma=1e-4):
    d = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden", "teapot.npz"))
    vertices, faces = torch.from_numpy(d["vertices"]).to(device), torch.from_numpy(d["faces"]).to(device)
    soft = (soft_sigma, soft_gamma) if soft_sigma else None
    textures = teapot_textures(faces.shape[0], device) if soft else None
    with torch.no_grad():
        r = neural_renderer.Renderer()
        r.eye = neural_renderer.get_points_from_angles(2.732, 30, -15)
        if soft:
            rgb, alpha = r.render_soft(vertices[None], faces[None], textures, *soft)
            target = torch.cat((rgb[0], alpha))  # [4,H,W]
        else:
            target = r.render_silhouettes(vertices[None], faces[None])[0]
    model = Model(vertices, faces, target, start, textures, soft).to(device)
    optimizer = neural_renderer.Adam(model.parameters(), lr=0.1)
    losses = []
    for _ in range(iters):
        optimizer.zero_grad()
        loss = model()
        loss.backward()
        optimizer.step()
        losses.append(float(loss.detach()))
        if losses[-1] < 70 and not soft:  # the reference's stopping rule (silhouettes)
            break
    return losses, model.camera_position.detach().cpu().numpy()


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--soft-sigma", type=float, default=None,
                    help="fit the soft RGB image and silhouette of this softness (e.g. 1e-4) instead of the hard silhouette")
    ap.add_argument("--soft-gamma", type=float, default=1e-4, help="depth temperature of the soft RGB image")
    a = ap.parse_args()
    losses, eye = run(a.iters, soft_sigma=a.soft_sigma, soft_gamma=a.soft_gamma)
    print("loss %.1f -> %.1f in %d iterations; camera at %s" % (losses[0], losses[-1], len(losses), np.round(eye, 3)))
