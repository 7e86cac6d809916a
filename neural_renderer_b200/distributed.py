"""Multi-GPU helpers for the rasterizer (SURVEY.md section 8(e)).

The batch / viewpoint axis shards embarrassingly: every kernel treats the batch index as an independent outer
dimension, so one process per GPU renders its own contiguous slice and no data-path collective is needed
(`shard_range`).  The only exchange the path ever has is the gradient of a mesh SHARED by all viewpoints
(`Mesh.get_batch` broadcasts one mesh, mesh.py:29-34 of the reference): each rank reduces its own views locally
(autograd sums over the expanded batch axis) and the per-rank sums of `vertices.grad` / `textures.grad` are combined
with one sum-all-reduce each (`allreduce_shared_grads`; NCCL over NVLink on GPUs, gloo in the CPU tests).  A shared
learnable texture image and its `face_uvs` ([F,3,2]: the rasterizer sums its gradient over the rank's items) are
combined the same way: pass them to `allreduce_shared_grads` with the vertices.
"""
from __future__ import annotations

import torch


def shard_range(n_items, rank, world):
    """Contiguous shard [lo, hi) of `n_items` batch items / viewpoints owned by `rank`."""
    per = (n_items + world - 1) // world
    lo = min(n_items, rank * per)
    return lo, min(n_items, lo + per)


def allreduce_shared_grads(params, group=None, async_op=False):
    """Sum-all-reduce the `.grad` of parameters shared by all ranks (in place).  Large tensors are reduced as they
    are (no flattening copy); with async_op=True the work handles are returned so that the caller can overlap the
    texture-gradient reduction with other work and `wait()` later."""
    import torch.distributed as dist
    works = []
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
        return works
    for p in params:
        g = p.grad if isinstance(p, torch.Tensor) and p.grad is not None else None
        if g is None:
            continue
        w = dist.all_reduce(g, op=dist.ReduceOp.SUM, group=group, async_op=async_op)
        if async_op:
            works.append(w)
    return works


class _PendingAllReduce:
    """Handle returned to the rasterizer's backward: `.wait()` makes the CURRENT stream wait for the collective."""

    def __init__(self, work):
        self.work = work

    def wait(self):
        self.work.wait()


class overlap_texture_allreduce:
    """Context manager: while active, every rasterizer backward on this rank sum-all-reduces its texture gradient
    across `group` AS SOON AS the texture-gradient kernels are enqueued -- on a side stream, so that the (large)
    texture all-reduce runs underneath the edge scan / vertex-gradient kernels of the same backward pass instead of
    behind them (SURVEY.md 8(e): "overlap the texture all-reduce with the vertex-gradient scan").

    How: the C ABI issues the backward in two halves (NR_BWD_PART_TEXTURES, then NR_BWD_PART_FACES).  Between them the
    side stream picks up the compute stream's position (only the texture half is enqueued at that point) and launches
    the collective; after the second half is enqueued the compute stream waits for the collective, so what autograd
    accumulates into `textures.grad` is already the global sum.  The collective is linear, so this is correct for a
    shared texture set ([1,F,...], NR_TEX_SHARED: 96 MB at 1 M faces / ts 2) and for per-item textures alike.
    With texture_filter='trilinear' the hook receives the gradient of the mip pyramid (about 4/3 of the image); the
    collapse into the image runs afterwards on every rank and is linear too, so the image gradient is the same global sum.
    With one rank, or outside an initialised process group, the hook does nothing.
    """

    def __init__(self, group=None):
        self.group = group
        self._streams = {}
        self._prev = None
        self.launched = 0  # collectives started (for tests / launch accounting)

    def _hook(self, grad):
        import torch.distributed as dist
        if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(self.group) == 1:
            return None
        dev = grad.device
        side = self._streams.get(dev)
        if side is None:
            side = self._streams[dev] = torch.cuda.Stream(dev)
        side.wait_stream(torch.cuda.current_stream(dev))  # = the texture half; the edge scan is not enqueued yet
        with torch.cuda.stream(side):
            work = dist.all_reduce(grad, op=dist.ReduceOp.SUM, group=self.group, async_op=True)
        grad.record_stream(side)
        self.launched += 1
        return _PendingAllReduce(work)

    def __enter__(self):
        from .rasterize import set_texture_grad_hook
        self._prev = set_texture_grad_hook(self._hook)
        return self

    def __exit__(self, *exc):
        from .rasterize import set_texture_grad_hook
        set_texture_grad_hook(self._prev)
        return False
