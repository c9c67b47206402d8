"""Multi-GPU rendering: rays are independent, so they shard across ranks with replicated weights and the
per-ray results are exchanged with ONE all-gather per chunk (SURVEY.md §8e).  No collective sits on the data
path of a ray; the reference's own multi-GPU eval shards whole images per rank and exchanges results through
the filesystem (runner.py:390-403,495-510) — this is the same partitioning at chunk granularity.

Works with any torch.distributed backend (NCCL on GPUs; gloo in the CPU tests of the host logic).
"""
from __future__ import annotations

from typing import Callable, Dict, Optional, Tuple

import torch
import torch.distributed as dist


def shard_bounds(n: int, world: int, rank: int) -> Tuple[int, int]:
    """Contiguous, balanced split of n rays: the first n % world ranks get one extra ray."""
    base, extra = divmod(n, world)
    lo = rank * base + min(rank, extra)
    return lo, lo + base + (1 if rank < extra else 0)


def all_gather_rows(local: torch.Tensor, n_total: int, group=None) -> torch.Tensor:
    """Gather row-sharded [n_r, C] tensors (shard_bounds layout) into [n_total, C] on every rank with a single
    all_gather_into_tensor of equal-size (padded) blocks."""
    world = dist.get_world_size(group)
    if world == 1:
        return local
    cols = local.shape[1:]
    per = (n_total + world - 1) // world
    buf = local.new_zeros((per,) + tuple(cols))
    buf[:local.shape[0]] = local
    out = local.new_empty((world * per,) + tuple(cols))
    dist.all_gather_into_tensor(out, buf, group=group)
    pieces = []
    for r in range(world):
        lo, hi = shard_bounds(n_total, world, r)
        pieces.append(out[r * per:r * per + (hi - lo)])
    return torch.cat(pieces, 0)


def broadcast_state(modules, group=None) -> None:
    """DistributedDataParallel's start-up for `modules` (None entries skipped): every parameter and buffer - a MegaNeRF's
    `centroids` included - overwritten in place by the values of the group's rank 0."""
    src = dist.get_global_rank(group if group is not None else dist.group.WORLD, 0)
    with torch.no_grad():
        for m in modules:
            if m is None:
                continue
            for t in list(m.parameters()) + list(m.buffers()):
                dist.broadcast(t.detach(), src=src, group=group)


def grad_bucket(sizes, device: torch.device) -> Tuple[torch.Tensor, list]:
    """One zeroed fp32 allocation holding gradient blocks of the given float counts back to back, nothing between them, so that
    one collective covers them all -> (bucket, [block views])."""
    bucket = torch.zeros(sum(sizes), device=device, dtype=torch.float32)
    blocks, a = [], 0
    for n in sizes:
        blocks.append(bucket[a:a + n])
        a += n
    return bucket, blocks


def average_gradients(bucket: torch.Tensor, group=None) -> None:
    """The mean of `bucket` over the group's ranks, in place, as DistributedDataParallel's default reduction computes it: scale
    by the world size first, then all-reduce with SUM.  A pre-divided SUM rather than ReduceOp.AVG, which gloo does not offer:
    one arithmetic on every backend, exact for a power-of-two world size (there DDP's multiply by 1/world gives the same bits),
    and one elementwise pass over the bucket.  Capturable in a CUDA graph on NCCL."""
    bucket.div_(dist.get_world_size(group))
    dist.all_reduce(bucket, op=dist.ReduceOp.SUM, group=group)


def render_rays_sharded(render_fn: Callable[..., Tuple[Dict[str, torch.Tensor], bool]], rays: torch.Tensor,
                        image_indices: Optional[torch.Tensor], *args, group=None, **kwargs) -> Tuple[Dict[str, torch.Tensor], bool]:
    """Every rank holds the same `rays` [N,8]; rank r renders rays[lo_r:hi_r] with `render_fn`
    (mega_nerf_b200.render_rays or anything with its signature) and all ranks end up with the full result dict.
    All per-ray outputs are packed column-wise so that exactly one collective is issued."""
    if not dist.is_available() or not dist.is_initialized() or dist.get_world_size(group) == 1:
        return render_fn(rays, image_indices, *args, **kwargs)
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    n = rays.shape[0]
    lo, hi = shard_bounds(n, world, rank)
    idx = image_indices[lo:hi] if image_indices is not None else None
    res, present = render_fn(rays[lo:hi], idx, *args, **kwargs)
    keys = sorted(res)
    widths = [1 if res[k].dim() == 1 else res[k].shape[1] for k in keys]
    packed = torch.cat([res[k].reshape(hi - lo, w).float() for k, w in zip(keys, widths)] +
                       [torch.full((hi - lo, 1), float(present), device=rays.device)], 1)
    full = all_gather_rows(packed, n, group)
    out, c = {}, 0
    for k, w in zip(keys, widths):
        v = full[:, c:c + w]
        out[k] = v.squeeze(1) if res[k].dim() == 1 else v
        c += w
    return out, bool(full[:, c].max().item() > 0) if full.shape[0] else present


class PeerGather:
    """Fused form of the per-chunk all-gather (SURVEY.md §8e): a symmetric [n_total, 4] result buffer per rank, peer-mapped
    into every process (torch symmetric memory does the allocation / handle exchange / barriers - plumbing), and ONE kernel
    of ours (`mn_peer_gather_store`) that writes this rank's (rgb, depth) rows into all of them over NVLink.  Replaces
    `torch.cat` + `all_gather_into_tensor`; the result is valid on every rank when `gather` returns (stream-ordered)."""

    def __init__(self, n_total: int, device: torch.device, group=None):
        import torch.distributed._symmetric_memory as symm_mem
        self.group = group if group is not None else dist.group.WORLD
        self.buf = symm_mem.empty(n_total, 4, dtype=torch.float32, device=device)
        self.hdl = symm_mem.rendezvous(self.buf, self.group)
        self.world = self.hdl.world_size
        self.rank = self.hdl.rank
        import ctypes as C
        self._ptrs = (C.c_void_p * self.world)(*[int(p) for p in self.hdl.buffer_ptrs])
        self.n_total = n_total

    def gather(self, rgb: torch.Tensor, depth: Optional[torch.Tensor], row0: int) -> torch.Tensor:
        from . import _cabi as K
        dev = rgb.device
        h = K.ctx(dev)
        n = rgb.shape[0]
        if row0 < 0 or row0 + n > self.n_total:
            raise ValueError('rows outside the gather buffer')
        rgb = K.f32c(rgb)
        depth = K.f32c(depth) if depth is not None else None
        self.hdl.barrier(channel=0)            # every rank has finished reading the previous contents
        K.check(K.lib().mn_peer_gather_store(h, K.ptr(rgb), K.ptr(depth), n, row0, self._ptrs, self.world, K.stream_of(dev)), h)
        self.hdl.barrier(channel=1)            # every rank's stores have landed
        return self.buf
