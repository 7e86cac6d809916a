"""GPU: the glue entry points' backward calls through the C ABI against float64 torch autograd -- NR_GRAD_ACCUMULATE on
each of them, what they store and what they add, the shared camera / index flags, and the backward sequence of
INTEGRATION.md section 2 (camera backward writes the vertex gradient, lighting backward adds into it)."""
import ctypes

import numpy as np
import pytest
import torch

from helpers import elem_err, rel_err

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda")
TOL = 1e-4


def _L():
    from neural_renderer_b200 import _lib as L
    return L, L.load()


def _p(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def _mesh(B, seed):
    from neural_renderer_b200 import synthetic
    v, f = synthetic.sphere_mesh(300)
    rng = np.random.default_rng(seed)
    verts = np.stack([v * 0.8 + rng.normal(scale=0.05, size=v.shape) for _ in range(B)]).astype(np.float32)
    return torch.from_numpy(verts).to(DEV), torch.from_numpy(f).to(DEV)


def _rand(shape, seed, lo=-1.0, hi=1.0):
    g = torch.Generator().manual_seed(seed)
    return (lo + (hi - lo) * torch.rand(shape, generator=g, dtype=torch.float32)).to(DEV)


def _check(x, ref, what):
    x, ref = x.double().cpu().numpy(), ref.double().cpu().numpy()
    assert np.isfinite(x).all(), what
    e1, e2 = rel_err(x, ref), elem_err(x, ref)
    assert e1 <= TOL and e2 <= TOL, (what, e1, e2)


def test_vertices_to_faces_backward_accumulates():
    L, lib = _L()
    B, Nv, Nf = 3, 50, 400
    idx = torch.randint(-3, Nv + 3, (B, Nf, 3), generator=torch.Generator().manual_seed(1)).to(torch.int32).to(DEV)
    gf = _rand((B, Nf, 3, 3), 2)
    ok = (idx >= 0) & (idx < Nv)
    fresh = torch.zeros((B, Nv, 3), dtype=torch.float64, device=DEV)
    fresh.view(B * Nv, 3).index_add_(0, (idx.long().clamp(0, Nv - 1) + Nv * torch.arange(B, device=DEV)[:, None, None])[ok],
                                     gf.double()[ok])
    for flags, pre in ((0, float("nan")), (L.NR_GRAD_ACCUMULATE, None)):
        gv = _rand((B, Nv, 3), 3) if pre is None else torch.full((B, Nv, 3), pre, device=DEV)
        prefill = gv.clone()
        L.check(lib.nr_b200_vertices_to_faces_backward(_p(gf), _p(idx), B, Nv, Nf, _p(gv), flags, None))
        torch.cuda.synchronize()
        _check(gv.double() - (prefill.double() if pre is None else 0), fresh, "grad_vertices flags=%d" % flags)


def _light64(v, faces, params):
    """lighting.py:29-51 in float64: [B,F,3]"""
    B = v.shape[0]
    tri = v[torch.arange(B, device=DEV)[:, None, None], faces.long().expand(B, -1, -1)]  # [B,F,3,3]
    a, b = tri[:, :, 0] - tri[:, :, 1], tri[:, :, 2] - tri[:, :, 1]
    c = torch.cross(a, b, dim=-1)
    n = c / (c.norm(dim=-1, keepdim=True) + 1e-5)
    p = params.expand(B, -1)
    cos = torch.relu((n * p[:, None, 6:9]).sum(-1, keepdim=True))
    return p[:, None, 0:3] + p[:, None, 3:6] * cos


def _params(n, seed):
    d = torch.tensor([[0.3, 0.8, -0.5]]) / np.linalg.norm([0.3, 0.8, -0.5])
    p = torch.cat((torch.full((n, 3), 0.5), 0.3 + 0.4 * torch.rand((n, 3), generator=torch.Generator().manual_seed(seed)),
                   d.expand(n, 3)), dim=1)
    return p.float().to(DEV).contiguous()


@pytest.mark.parametrize("shared", [False, True])
def test_face_lighting_backward_accumulates(shared):
    """NR_INDICES_SHARED ([F,3] indices for every item) and NR_CAM_SHARED (one light for every item) against float64"""
    L, lib = _L()
    B = 3
    v, f = _mesh(B, seed=4)
    Nv, Nf = v.shape[1], f.shape[0]
    faces = f if shared else f[None].expand(B, -1, -1).contiguous()
    params = _params(1 if shared else B, 5)
    flags = (L.NR_INDICES_SHARED | L.NR_CAM_SHARED) if shared else 0
    gl = _rand((B, Nf, 3), 6)
    v64 = v.double().requires_grad_(True)
    (_light64(v64, f[None], params.double()) * gl.double()).sum().backward()
    light = torch.empty((B, Nf, 3), device=DEV)
    L.check(lib.nr_b200_face_lighting(_p(v), _p(faces), _p(params), B, Nv, Nf, flags, _p(light), None))
    torch.cuda.synchronize()
    _check(light, _light64(v.double(), f[None], params.double()), "face_light")
    for acc in (False, True):
        gv = _rand((B, Nv, 3), 7) if acc else torch.full((B, Nv, 3), float("nan"), device=DEV)
        prefill = gv.clone()
        L.check(lib.nr_b200_face_lighting_backward(_p(v), _p(faces), _p(params), _p(gl), B, Nv, Nf,
                                                   flags | (L.NR_GRAD_ACCUMULATE if acc else 0), _p(gv), None))
        torch.cuda.synchronize()
        _check(gv.double() - (prefill.double() if acc else 0), v64.grad, "grad_vertices acc=%s" % acc)


def _camera64(v, rot, eye, width, shared):
    B = v.shape[0]
    n = 1 if shared else B
    R = rot.view(n, 3, 3).expand(B, -1, -1)
    o = torch.einsum("bjk,bvk->bvj", R, v - eye.view(n, 1, 3))
    w = width.view(n, 1).expand(B, -1)
    return torch.stack((o[..., 0] / o[..., 2] / w, o[..., 1] / o[..., 2] / w, o[..., 2]), dim=-1)


def _camera(n, seed):
    """n look_at cameras (rows of rot = camera x, y, z axes) around the origin at distance 2.732, widths near tan(30 deg)"""
    g = torch.Generator().manual_seed(seed)
    rots, eyes = [], []
    for i in range(n):
        el, az = np.radians(10 + 20 * float(torch.rand((), generator=g))), np.radians(360 * float(torch.rand((), generator=g)))
        e = 2.732 * np.array([np.cos(el) * np.sin(az), np.sin(el), -np.cos(el) * np.cos(az)])
        z = -e / np.linalg.norm(e)
        x = np.cross([0, 1, 0], z)
        x /= np.linalg.norm(x)
        y = np.cross(z, x)
        rots.append(np.stack([x, y, z]).reshape(9))
        eyes.append(e)
    width = 0.5 + 0.2 * torch.rand((n,), generator=g, dtype=torch.float64)
    return (torch.tensor(np.stack(rots), dtype=torch.float32, device=DEV), torch.tensor(np.stack(eyes), dtype=torch.float32, device=DEV),
            width.float().to(DEV))


@pytest.mark.parametrize("shared", [False, True])
def test_camera_backward_stores_vertices_and_accumulates_camera(shared):
    """grad_vertices is written (a prefill does not survive, even with NR_GRAD_ACCUMULATE); grad_rot / grad_eye / grad_width
    are zero-filled, or added into with NR_GRAD_ACCUMULATE; NR_CAM_SHARED: one camera for per-item vertices"""
    L, lib = _L()
    B = 3
    v, _ = _mesh(B, seed=8)
    Nv = v.shape[1]
    n = 1 if shared else B
    rot, eye, width = _camera(n, 9)
    flags = L.NR_CAM_PERSPECTIVE | (L.NR_CAM_SHARED if shared else 0)
    go = _rand((B, Nv, 3), 10)
    leaves = [t.double().requires_grad_(True) for t in (v, rot, eye, width)]
    out64 = _camera64(*leaves, shared)
    (out64 * go.double()).sum().backward()
    out = torch.empty_like(v)
    L.check(lib.nr_b200_camera_transform(_p(v), _p(rot), _p(eye), _p(width), B, Nv, flags, _p(out), None))
    torch.cuda.synchronize()
    _check(out, out64.detach(), "camera out")
    for acc in (False, True):
        grads = [_rand(s, 11 + k) for k, s in enumerate(((B, Nv, 3), (n, 9), (n, 3), (n,)))]
        prefill = [g.clone() for g in grads]
        L.check(lib.nr_b200_camera_transform_backward(_p(v), _p(rot), _p(eye), _p(width), _p(go), B, Nv,
                                                      flags | (L.NR_GRAD_ACCUMULATE if acc else 0), *map(_p, grads), None))
        torch.cuda.synchronize()
        _check(grads[0], leaves[0].grad, "grad_vertices (stored) acc=%s" % acc)
        for k, name in ((1, "rot"), (2, "eye"), (3, "width")):
            _check(grads[k].double() - (prefill[k].double() if acc else 0), leaves[k].grad, "grad_%s acc=%s" % (name, acc))


def test_integration_backward_sequence():
    """INTEGRATION.md section 2: d loss / d vertices of  L = <G_f, vertices_to_faces(camera(V))> + <G_l, lighting(V)>
    through the C ABI -- vertices_to_faces backward, camera backward (writes grad_vertices), lighting backward with
    NR_GRAD_ACCUMULATE (adds into it) -- against float64 autograd of the op-by-op forward"""
    L, lib = _L()
    B = 2
    v, f = _mesh(B, seed=12)
    Nv, Nf = v.shape[1], f.shape[0]
    f2 = torch.cat((f, f.flip(1)), 0)  # fill_back
    faces = f2[None].expand(B, -1, -1).contiguous()
    rot, eye, width = _camera(1, 13)
    params = _params(1, 14)
    gf = _rand((B, 2 * Nf, 3, 3), 15)
    gl = _rand((B, 2 * Nf, 3), 16)
    v64 = v.double().requires_grad_(True)
    cam = _camera64(v64, rot.double(), eye.double(), width.double(), True)
    tri = cam[torch.arange(B, device=DEV)[:, None, None], faces.long()]
    loss = (tri * gf.double()).sum() + (_light64(v64, f2[None], params.double()) * gl.double()).sum()
    loss.backward()
    g_cam = torch.empty_like(v)
    gv = torch.full_like(v, float("nan"))
    shared = L.NR_CAM_SHARED
    L.check(lib.nr_b200_vertices_to_faces_backward(_p(gf), _p(faces), B, Nv, 2 * Nf, _p(g_cam), 0, None))
    L.check(lib.nr_b200_camera_transform_backward(_p(v), _p(rot), _p(eye), _p(width), _p(g_cam), B, Nv,
                                                  L.NR_CAM_PERSPECTIVE | shared, _p(gv), None, None, None, None))
    L.check(lib.nr_b200_face_lighting_backward(_p(v), _p(f2), _p(params), _p(gl), B, Nv, 2 * Nf,
                                               L.NR_INDICES_SHARED | shared | L.NR_GRAD_ACCUMULATE, _p(gv), None))
    torch.cuda.synchronize()
    _check(gv, v64.grad, "grad_vertices")
