"""Seeded synthetic rasterizer inputs (numpy, deterministic across machines) for the benchmark and the parity tests.

`sphere_faces` is the workload SURVEY.md section 8(d) / BASELINE.md name for the headline metric: every batch item is
its own closed UV-sphere (n x n quads split into triangles; 50 x 50 -> 5000 faces), radius 0.8, per-item random
rotation (seed 1234 + item), vertices jittered by N(0, 0.01^2), already in the rasterizer's input space (x, y in NDC,
z = camera depth in [1.9, 3.6]); consistent winding, so about half of the faces are back-facing like a real mesh.
"""
from __future__ import annotations

import math

import numpy as np


def _rotation(rng):
    q = rng.normal(size=4)
    q /= np.linalg.norm(q)
    w, x, y, z = q
    return np.array([
        [1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
        [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
        [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def sphere_mesh(num_faces=5000):
    """UV-sphere with ~num_faces triangles: (vertices [Nv,3] f64 on the unit sphere, faces [num_faces,3] i32)."""
    n = max(2, int(math.ceil(math.sqrt(num_faces / 2.0))))
    n_lat = n_lon = n
    delta = 0.01  # keep the pole rings open so that no triangle is degenerate
    theta = np.pi * (np.arange(n_lat + 1) * (1 - 2 * delta) / n_lat + delta)
    phi = 2 * np.pi * np.arange(n_lon) / n_lon
    st, ct = np.sin(theta)[:, None], np.cos(theta)[:, None]
    v = np.stack([st * np.cos(phi)[None, :], ct * np.ones_like(phi)[None, :], st * np.sin(phi)[None, :]], axis=-1)
    vertices = v.reshape(-1, 3)
    i, j = np.meshgrid(np.arange(n_lat), np.arange(n_lon), indexing="ij")
    a = i * n_lon + j
    b = (i + 1) * n_lon + j
    c = (i + 1) * n_lon + (j + 1) % n_lon
    d = i * n_lon + (j + 1) % n_lon
    faces = np.stack([np.stack([a, b, c], axis=-1), np.stack([a, c, d], axis=-1)], axis=2).reshape(-1, 3)
    faces = np.ascontiguousarray(faces[:num_faces], dtype=np.int32)
    assert faces.shape[0] == num_faces
    return vertices, faces


def sphere_faces(batch_size, num_faces=5000, radius=0.8, jitter=0.01, z_center=2.75, seed=1234):
    """[B,F,3,3] float32 faces of per-item rotated / jittered spheres in rasterizer input space."""
    vertices, faces = sphere_mesh(num_faces)
    out = np.empty((batch_size, num_faces, 3, 3), dtype=np.float32)
    for b in range(batch_size):
        rng = np.random.default_rng(seed + b)
        v = (vertices * radius) @ _rotation(rng).T
        v = v + rng.normal(scale=jitter, size=v.shape)
        v[:, 2] += z_center
        out[b] = v[faces].astype(np.float32)
    return out


def sphere_uvs(num_faces=5000):
    """[num_faces,3,2] float32 spherical UVs of sphere_mesh's face corners (same faces as sphere_faces): u = longitude /
    2 pi, v = 1 - colatitude / pi (OBJ convention, v = 1 at the top pole); the corners past the seam get u = 1."""
    n = max(2, int(math.ceil(math.sqrt(num_faces / 2.0))))
    delta = 0.01
    i, j = np.meshgrid(np.arange(n), np.arange(n), indexing="ij")

    def corner(ii, jj):
        theta = (ii * (1 - 2 * delta) / n + delta)  # colatitude / pi, as in sphere_mesh
        return np.stack([jj / n, 1.0 - theta], axis=-1)

    a, b, c, d = corner(i, j), corner(i + 1, j), corner(i + 1, j + 1), corner(i, j + 1)
    uv = np.stack([np.stack([a, b, c], axis=-2), np.stack([a, c, d], axis=-2)], axis=2).reshape(-1, 3, 2)
    return np.ascontiguousarray(uv[:num_faces], dtype=np.float32)


def random_image(batch_size, height, width, seed=4322):
    """[batch_size,height,width,3] float32 texture images, uniform in [0, 1)."""
    rng = np.random.default_rng(seed)
    return rng.random((batch_size, height, width, 3), dtype=np.float32)


def random_textures(batch_size, num_faces, texture_size=4, seed=4321):
    rng = np.random.default_rng(seed)
    return rng.random((batch_size, num_faces, texture_size, texture_size, texture_size, 3), dtype=np.float32)


def triangle_soup(batch_size, num_faces, seed=0, size=(0.05, 0.5), z_range=(1.0, 3.0), duplicates=True,
                  offscreen=True):
    """Random, mutually intersecting triangles (stress for the z-test and the tie rule): random centres (some partly
    off screen), random extents, random winding; a few exact duplicates so that the lowest-index rule decides."""
    rng = np.random.default_rng(seed)
    lim = 1.2 if offscreen else 0.9
    c = rng.uniform(-lim, lim, size=(batch_size, num_faces, 1, 2))
    ext = rng.uniform(size[0], size[1], size=(batch_size, num_faces, 1, 1))
    xy = c + ext * rng.uniform(-1, 1, size=(batch_size, num_faces, 3, 2))
    z = rng.uniform(z_range[0], z_range[1], size=(batch_size, num_faces, 3, 1))
    f = np.concatenate([xy, z], axis=-1).astype(np.float32)
    if duplicates and num_faces >= 8:
        for b in range(batch_size):
            src = rng.integers(0, num_faces, size=max(1, num_faces // 16))
            dst = rng.integers(0, num_faces, size=src.shape[0])
            f[b, dst] = f[b, src]
    return f


def needle_faces(batch_size, num_faces, image_size, seed=0, thin=(1e-7, 1e-4), z_range=(1.0, 3.0)):
    """Front-facing needles that win a pixel BEYOND their tip: the tip sits a fraction of a pixel in front of a pixel
    centre on the needle's axis and the two long edges meet at `thin` (half width / length, log-uniform).  Candidates are
    drawn until the reference's own fp32 edge tests (rasterize.py:306-311, replayed here in numpy float32) accept that
    pixel centre -- a pixel outside the box of the three vertices (about one candidate in a thousand).  Stress for the
    conservative pixel box of the forward pass (nr_bbox.cuh: thin_face_margin)."""
    rng = np.random.default_rng(seed)
    S = image_size
    f32 = np.float32
    centres = ((2 * np.arange(S) + 1 - S) / S).astype(f32)
    out = np.empty((batch_size, num_faces, 3, 3), dtype=f32)
    for b in range(batch_size):
        kept = []
        while len(kept) < num_faces:
            n = 200000
            cx = centres[rng.integers(S // 8, S - S // 8, size=n)].astype(np.float64)
            cy = centres[rng.integers(S // 8, S - S // 8, size=n)].astype(np.float64)
            ang = rng.uniform(0, 2 * np.pi, size=n)
            dx, dy = np.cos(ang), np.sin(ang)
            back = rng.uniform(0.05, 1.5, size=n) * 2.0 / S
            ax, ay = cx - dx * back, cy - dy * back
            length = rng.uniform(0.2, 0.8, size=n)
            half = length * np.exp(rng.uniform(np.log(thin[0]), np.log(thin[1]), size=n))
            bx, by = ax - dx * length, ay - dy * length
            v = np.stack([np.stack([ax, ay], -1), np.stack([bx - dy * half, by + dx * half], -1),
                          np.stack([bx + dy * half, by - dx * half], -1)], 1).astype(f32)  # [n,3,2]
            # front-facing in the reference's sense (rasterize.py:306): swap two vertices if not
            back_side = (v[:, 2, 1] - v[:, 0, 1]) * (v[:, 1, 0] - v[:, 0, 0]) < (v[:, 1, 1] - v[:, 0, 1]) * (v[:, 2, 0] - v[:, 0, 0])
            v[back_side] = v[back_side][:, [0, 2, 1]]
            back_side = (v[:, 2, 1] - v[:, 0, 1]) * (v[:, 1, 0] - v[:, 0, 0]) < (v[:, 1, 1] - v[:, 0, 1]) * (v[:, 2, 0] - v[:, 0, 0])
            xp, yp = cx.astype(f32), cy.astype(f32)
            ok = ~back_side
            for k in range(3):
                k1 = (k + 1) % 3
                ok &= ~((yp - v[:, k, 1]) * (v[:, k1, 0] - v[:, k, 0]) < (xp - v[:, k, 0]) * (v[:, k1, 1] - v[:, k, 1]))
            # the aimed pixel must lie outside the vertices' pixel box
            px, py = 0.5 * (v[:, :, 0] * S + S - 1), 0.5 * (v[:, :, 1] * S + S - 1)
            ix, iy = 0.5 * (xp * S + S - 1), 0.5 * (yp * S + S - 1)
            outside = (ix > np.ceil(px.max(1) + 1 / 256)) | (ix < np.floor(px.min(1) - 1 / 256)) | \
                      (iy > np.ceil(py.max(1) + 1 / 256)) | (iy < np.floor(py.min(1) - 1 / 256))
            for i in np.nonzero(ok & outside)[0]:
                kept.append(v[i])
                if len(kept) == num_faces:
                    break
        z = rng.uniform(z_range[0], z_range[1], size=(num_faces, 3, 1)).astype(f32)
        out[b] = np.concatenate([np.stack(kept), z], axis=-1)
    return out
