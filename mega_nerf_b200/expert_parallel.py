"""Owner-computes ("one centroid per GPU") execution of a MegaNeRF over a process group - SURVEY.md §8f-5.

`models/mega_nerf.py:19-61` loops over the sub-modules on one device.  Here sub-module k lives on rank k % G only
(round-robin, BASELINE.json configs[2] / [3]): every rank routes ITS OWN sample rows (the centroids are tiny and
replicated), ships each (row, sub-module) pair to the owner with one all-to-all, the owners run their sub-modules on
what they received, a second all-to-all returns the (rgb, sigma) rows, and the home rank accumulates them in ascending
sub-module order with the blend weights - the same arithmetic as `results[mask] += sub_result * weights[mask, i]`
(`mega_nerf.py:46-49`).  Compositing stays on the home rank: it is non-linear along a ray, which is why a per-ray
all-gather alone cannot express this partitioning (SURVEY.md §8e).

Payload per routed pair: the child's input row (xyz, dir, image index: 28 B) + sub-module id (+ density noise) out,
16 B back.  The exchange is `torch.distributed.all_to_all_single` (NCCL over NVLink on GPUs, gloo in the CPU tests of
this host logic).  Every rank must issue the same sequence of queries (true for `render_rays` on the foreground network
with the same sampling configuration on every rank).

Training (CUDA tensors, device path): when autograd records, the owner call records a tape (mn_model_forward_assigned_train,
sized by the pairs that arrived: the query reads that count back once) and the result exchange is differentiable, so
`loss.backward()` runs mn_model_ep_combine_backward at home, the reverse all-to-all of the result gradients and
mn_model_backward_assigned at the owner.  Owned parameters receive the MEAN over ranks of what each rank's loss gives them
(divided by world in `_owner_backward`, nowhere else) - what DDP over a replicated MegaNeRF leaves in `.grad`; sub-modules
owned elsewhere get no `.grad` at all.  Conditions: every rank calls backward on the same sequence of queries (the coarse
and the fine query both feed the reference's loss), every rank queries the same row count, and the foreground network is
NOT wrapped in DistributedDataParallel (the owners already hold the reduced gradient).  The torch path is inference-only.

A query whose row count differs from rank to rank - `render_rays` queries a background network for the rays that reach the
background only - passes `rows_cap`, the largest count over the ranks (`max_over_ranks`), so that every rank sizes its
segments alike; a rank with no rows still takes part, sending empty segments.

CUDA tensors take the device path: `mn_model_route`, then `mn_model_ep_dispatch` writes the pairs straight into `world`
segments of a fixed capacity (B x max_multiplicity rows, the router's own slot bound), one all-to-all with equal splits
moves the segments and one the per-(rank, sub-module) counts, `mn_model_forward_assigned` runs every owned sub-module over
what arrived in one library call, a third all-to-all returns the results and `mn_model_ep_combine` blends them.  No step
synchronises the host, so a query can be captured in a CUDA graph (`GraphedRenderRays`); the price is that the segments
travel padded, and that every rank must query the same row count B.

The torch path - split sizes exchanged and read back (`counts.tolist()`, one host sync per query; the reference itself
syncs once per sub-module, `x[cluster_mask]`), one `NeRF.forward` per owned sub-module, a Python loop for the blend - serves
CPU tensors and injected device steps (`route_fn`, `sub_fn`), so that the dispatch / return / accumulation logic is
testable without a GPU; `plan_dispatch` is the order the device dispatch reproduces.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import Callable, List, Optional, Tuple

import torch
import torch.distributed as dist

from . import _cabi as K
from .modules import _Native, get_precision


def owner_of(k: int, world: int) -> int:
    """Round-robin sub-module -> rank (BASELINE.json configs[3])."""
    return k % world


def plan_dispatch(assign: Optional[torch.Tensor], weights: Optional[torch.Tensor], n_sub: int, world: int):
    """(row, sub-module) pairs of one query, ordered by (destination rank, sub-module, row).
    -> rows [P] int64, subs [P] int64, blend weights [P] or None, send counts [world] int64."""
    if weights is None:
        rows = torch.arange(assign.shape[0], device=assign.device)
        subs = assign
        w = None
    else:
        nz = (weights > 0).nonzero()
        rows, subs = nz[:, 0], nz[:, 1]
        w = weights[rows, subs]
    dest = subs % world
    order = torch.argsort(dest * n_sub + subs, stable=True)
    rows, subs, dest = rows[order], subs[order], dest[order]
    if w is not None:
        w = w[order]
    counts = torch.bincount(dest, minlength=world)
    return rows, subs, w, counts


class ExpertParallel:
    def __init__(self, mega, group=None, route_fn: Optional[Callable] = None, sub_fn: Optional[Callable] = None):
        self.mega = mega
        self.group = group
        self.n_sub = len(mega.sub_modules)
        self._native = None
        self._torch_path = route_fn is not None or sub_fn is not None
        self.route_fn = route_fn or self._route_native
        self.sub_fn = sub_fn or self._sub_native
        self._last = (0, 0)

    # routed pairs of the last query that originated on this rank, and pairs this rank computed for everybody; after a
    # device query these read the device counts back (a host sync) when accessed
    @property
    def last_pairs(self) -> int:
        return int(self._last[0])

    @property
    def last_owned(self) -> int:
        return int(self._last[1])

    # ---- device-side defaults
    def native(self, device: torch.device) -> _Native:
        """The native MegaNeRF of this rank: the centroids (routing) and the weights of the owned sub-modules only, packed
        on `device`; sub-modules owned elsewhere are never read."""
        m = self.mega
        if self._native is None:
            self._native = _Native(m, 2, list(m.sub_modules), m.centroids, m.boundary_margin, m.xyz_real, m.cluster_dim_start)
            self._native.packed_subs = set(self.owned())
            self._native.max_multiplicity = m._native().max_multiplicity
        self._native.centroids = m.centroids
        return self._native

    def sync(self, device: torch.device) -> None:
        """Re-pack the native weights if a parameter changed (in place: a captured graph keeps reading them)."""
        self.native(device).sync(device)

    def _route_device(self, x: torch.Tensor) -> Tuple[Optional[torch.Tensor], Optional[torch.Tensor]]:
        """-> (assign int32 [B] or None, weights [B,K] or None), like models/mega_nerf.py:21-30."""
        dev = x.device
        nat = self.native(dev)
        h = nat.sync(dev)
        rows = K.Rows()
        rows.mode, rows.x_d, rows.cols = 0, x.data_ptr(), x.shape[1]
        B = x.shape[0]
        if self.mega.boundary_margin > 1:
            w = torch.empty(B, self.n_sub, device=dev, dtype=torch.float32)
            K.check(K.lib().mn_model_route(h, nat.handle, C.byref(rows), B, None, K.ptr(w), K.stream_of(dev)), h)
            return None, w
        a = torch.empty(B, device=dev, dtype=torch.int32)
        K.check(K.lib().mn_model_route(h, nat.handle, C.byref(rows), B, K.ptr(a), None, K.stream_of(dev)), h)
        return a, None

    def _route_native(self, x):
        assign, w = self._route_device(K.f32c(x))
        return (assign.long() if assign is not None else None), w

    def _sub_native(self, k: int, rows: torch.Tensor, sigma_noise: Optional[torch.Tensor]) -> torch.Tensor:
        return self.mega.sub_modules[k](rows, sigma_noise=sigma_noise)

    def owned(self) -> List[int]:
        world, rank = dist.get_world_size(self.group), dist.get_rank(self.group)
        return [k for k in range(self.n_sub) if owner_of(k, world) == rank]

    # ---- nn.Module.__call__ of MegaNeRF on rows, distributed
    def forward(self, x: torch.Tensor, sigma_noise: Optional[torch.Tensor] = None, rows_cap: Optional[int] = None) -> torch.Tensor:
        """rows_cap: the capacity row count of the device path's segments, the same on every rank and >= x.shape[0] (default:
        x.shape[0], which every rank must then share).  The torch path exchanges its split sizes and ignores it."""
        if x.is_cuda and not self._torch_path:
            return self._forward_device(x, sigma_noise, rows_cap)
        if self._recording():
            raise RuntimeError('expert-parallel execution is inference-only (wrap the call in torch.no_grad())')
        return self._forward_torch(x, sigma_noise)

    def _recording(self) -> bool:
        return torch.is_grad_enabled() and any(p.requires_grad for p in self.mega.parameters())

    def max_over_ranks(self, n: int, device: torch.device) -> int:
        """The largest of every rank's `n` over the group (one all-reduce, read back): the capacity that lets ranks with
        different row counts run the same query."""
        t = torch.tensor([n], device=device, dtype=torch.int64)
        dist.all_reduce(t, op=dist.ReduceOp.MAX, group=self.group)
        return int(t.item())

    # ---- device path: the three steps, each callable on its own (a test can play several ranks on one device).  When
    # autograd records (a parameter requires grad), `compute` and `combine` return differentiable results: the backward of
    # `combine` is mn_model_ep_combine_backward, that of `compute` mn_model_backward_assigned over the owner's tape.
    def dispatch(self, x: torch.Tensor, sigma_noise: Optional[torch.Tensor], world: int, rows_cap: Optional[int] = None) -> 'Dispatch':
        """Route x [B, cols] and write its pairs into `world` segments (mn_model_ep_dispatch) sized for `rows_cap` rows
        (default B; the same on every rank).  With B == 0 every slot is empty (id -1)."""
        dev = x.device
        x = K.f32c(x)
        assign, weights = self._route_device(x)
        nat = self.native(dev)
        L, h = K.lib(), K.ctx(dev)
        B, cols = x.shape
        B_cap = B if rows_cap is None else int(rows_cap)
        if B_cap < B:
            raise ValueError(f'rows_cap {B_cap} is below the row count {B}')
        c_in = cols - (3 if self.mega.xyz_real else 0)
        noise = K.f32c(sigma_noise).view(-1) if sigma_noise is not None else None
        if noise is not None and B == 0:
            noise = torch.empty(1, device=dev)        # the pointer sets the payload width; with no rows nothing is read
        cap = int(L.mn_model_ep_segment_rows(nat.handle, B_cap))
        i32 = dict(device=dev, dtype=torch.int32)
        d = Dispatch(world=world, cap=cap, c_in=c_in, has_noise=noise is not None, assign=assign, weights=weights,
                     send=torch.empty(world * cap, c_in + 1 + (noise is not None), device=dev, dtype=torch.float32),
                     counts=torch.empty(world, self.n_sub, **i32), pair_row=torch.empty(world * cap, **i32),
                     pair_w=torch.empty(world * cap, device=dev, dtype=torch.float32) if weights is not None else None,
                     row_slots=torch.empty(B * (self.n_sub if weights is not None else 1), **i32))
        ws = torch.empty(max(int(L.mn_model_ep_dispatch_workspace_bytes(nat.handle, B, world)), 256), device=dev, dtype=torch.uint8)
        K.check(L.mn_model_ep_dispatch(h, nat.handle, K.ptr(x), B, B_cap, cols, K.ptr(assign), K.ptr(weights), K.ptr(noise), world,
                                       K.ptr(d.send), K.ptr(d.counts), K.ptr(d.pair_row), K.ptr(d.pair_w), K.ptr(d.row_slots),
                                       K.ptr(ws), ws.numel(), K.stream_of(dev)), h)
        return d

    def compute(self, recv: torch.Tensor, c_in: int, has_noise: bool, max_pairs: Optional[int] = None, rank: Optional[int] = None,
                world: Optional[int] = None) -> torch.Tensor:
        """The owner's share: every received row through its own sub-module (mn_model_forward_assigned) -> [n, rgb_dim + 1];
        rows with sub-module id -1 are left unwritten.

        Recording (autograd on, a parameter requires grad): mn_model_forward_assigned_train, whose tape holds `max_pairs` pairs
        (default: the rows with an id, read back once); rows with id -1 are NaN, and more pairs than max_pairs raise here
        (a status check, which synchronises the host).  Its backward gives the parameters of the sub-modules owned by `rank`
        out of `world` (default: this rank of the group) their gradient divided by `world`; the others get none."""
        if self._recording():
            if rank is None or world is None:
                rank, world = dist.get_rank(self.group), dist.get_world_size(self.group)
            if max_pairs is None:
                max_pairs = int((recv[:, c_in] >= 0).sum())
            plist = self.native(recv.device).param_list()
            return _OwnerFn.apply(self, recv, c_in, has_noise, int(max_pairs), rank, world, *[p for _, _, p in plist])
        dev = recv.device
        nat = self.native(dev)
        L, h = K.lib(), nat.sync(dev)
        n = recv.shape[0]
        prec = K.PRECISIONS[get_precision()]
        res = torch.empty(n, self.mega.sub_modules[0].rgb_dim + 1, device=dev, dtype=torch.float32)
        ws = torch.empty(max(int(L.mn_model_forward_assigned_workspace_bytes(nat.handle, n, prec)), 256), device=dev,
                         dtype=torch.uint8)
        K.check(L.mn_model_forward_assigned(h, nat.handle, K.ptr(recv), n, c_in, int(has_noise), prec, K.ptr(res), K.ptr(ws),
                                            ws.numel(), K.stream_of(dev)), h)
        return res

    def combine(self, d: 'Dispatch', back: torch.Tensor) -> torch.Tensor:
        """Blend the returned results of a dispatch's pairs at home (mn_model_ep_combine) -> [B, rgb_dim + 1]."""
        if back.requires_grad and torch.is_grad_enabled():
            return _CombineFn.apply(self, d, back)
        dev = back.device
        nat = self.native(dev)
        B = d.row_slots.shape[0] // (self.n_sub if d.pair_w is not None else 1)
        out = torch.empty(B, back.shape[1], device=dev, dtype=torch.float32)
        h = K.ctx(dev)
        K.check(K.lib().mn_model_ep_combine(h, nat.handle, B, K.ptr(d.row_slots), K.ptr(d.pair_w), K.ptr(back), K.ptr(out),
                                            K.stream_of(dev)), h)
        return out

    def combine_backward(self, d: 'Dispatch', dout: torch.Tensor) -> torch.Tensor:
        """Gradient of `combine`'s output [B, rgb_dim + 1] -> gradient of the returned results [world * cap, rgb_dim + 1]
        (mn_model_ep_combine_backward): w x dout[home row] per slot, 0 past the pairs."""
        dev = dout.device
        nat = self.native(dev)
        n_slots = d.pair_row.shape[0]
        if dout.shape[0] == 0:
            return torch.zeros(n_slots, dout.shape[1], device=dev, dtype=torch.float32)      # no pairs: every slot is past them
        dback = torch.empty(n_slots, dout.shape[1], device=dev, dtype=torch.float32)
        h = K.ctx(dev)
        K.check(K.lib().mn_model_ep_combine_backward(h, nat.handle, n_slots, K.ptr(d.pair_row), K.ptr(d.pair_w), K.ptr(K.f32c(dout)),
                                                     K.ptr(dback), K.stream_of(dev)), h)
        return dback

    def _forward_device(self, x: torch.Tensor, sigma_noise: Optional[torch.Tensor], rows_cap: Optional[int] = None) -> torch.Tensor:
        world = dist.get_world_size(self.group)
        d = self.dispatch(x, sigma_noise, world, rows_cap)
        recv, recv_counts = torch.empty_like(d.send), torch.empty_like(d.counts)
        dist.all_to_all_single(recv, d.send, group=self.group)
        dist.all_to_all_single(recv_counts, d.counts, group=self.group)
        self._last = (_LazySum(d.counts), _LazySum(recv_counts))
        if self._recording():
            # training: the owner's tape is sized by the pairs that arrived (one host read), and the result exchange is
            # differentiable - its backward carries the result gradients from home back to the owners
            res = self.compute(recv, d.c_in, d.has_noise, int(recv_counts.sum()))
            return self.combine(d, _AllToAll.apply(res, self.group))
        res = self.compute(recv, d.c_in, d.has_noise)
        back = torch.empty_like(res)
        dist.all_to_all_single(back, res, group=self.group)
        return self.combine(d, back)

    def _record(self, recv: torch.Tensor, c_in: int, has_noise: bool, max_pairs: int) -> Tuple[torch.Tensor, 'OwnerTape']:
        """The recording owner call (mn_model_forward_assigned_train) in the training arithmetic of `set_train_precision`."""
        dev = recv.device
        nat = self.native(dev)
        L, h, st = K.lib(), nat.sync(dev), K.stream_of(dev)
        n = recv.shape[0]
        prec = K.PREC_TC_F16 if nat.train_on_tensor_cores() else K.PREC_FP32
        res = torch.empty(n, self.mega.sub_modules[0].rgb_dim + 1, device=dev, dtype=torch.float32)
        tape = torch.empty(max(int(L.mn_model_assigned_tape_bytes(nat.handle, max_pairs, prec)), 256), device=dev, dtype=torch.uint8)
        ws = torch.empty(max(int(L.mn_model_forward_assigned_train_workspace_bytes(nat.handle, n)), 256), device=dev, dtype=torch.uint8)
        K.check(L.mn_model_forward_assigned_train(h, nat.handle, K.ptr(recv), n, c_in, int(has_noise), max_pairs, prec, K.ptr(res),
                                                  K.ptr(tape), tape.numel(), K.ptr(ws), ws.numel(), st), h)
        K.check(L.mn_check_status(h, st), h)           # more pairs than max_pairs: raise before anything reads the tape
        return res, OwnerTape(tape=tape, n=n, max_pairs=max_pairs, precision=prec)

    def _owner_backward(self, t: 'OwnerTape', grad_res: torch.Tensor, rank: int, world: int) -> List[Optional[torch.Tensor]]:
        """Parameter gradients of a recording owner call (mn_model_backward_assigned), in param_list() order: the sub-modules
        owned by `rank` get the gradient divided by `world` - the one place the mean over ranks is taken, so that an owned
        parameter holds what DDP over a replicated MegaNeRF would leave in it - the others None."""
        dev = grad_res.device
        nat = self.native(dev)
        L, h = K.lib(), K.ctx(dev)
        gbuf = torch.zeros(int(L.mn_model_grad_floats(nat.handle)), device=dev, dtype=torch.float32)
        ws = torch.empty(max(int(L.mn_model_backward_assigned_workspace_bytes(nat.handle, t.max_pairs, t.precision)), 256), device=dev,
                         dtype=torch.uint8)
        g = K.f32c(grad_res)
        K.check(L.mn_model_backward_assigned(h, nat.handle, t.n, t.max_pairs, t.precision, K.ptr(g), K.ptr(t.tape), t.tape.numel(),
                                             K.ptr(gbuf), K.ptr(ws), ws.numel(), K.stream_of(dev)), h)
        gbuf.div_(world)
        off = nat._offsets()
        stride = off['stride']
        grads = []
        for k, key, p in nat.param_list():
            if owner_of(k, world) != rank:
                grads.append(None)
                continue
            a = k * stride + off[key]
            grads.append(gbuf[a:a + p.numel()].view(p.shape))
        return grads

    # ---- checkpoints
    def full_state_dict(self) -> dict:
        """The whole MegaNeRF's state dict under the reference's key names (`sub_modules.<k>.<name>`, `centroids`), every
        sub-module's tensors broadcast from their owner (rank k mod world), so that rank 0 can save it as `model_state_dict`
        and the reference loads it unchanged.  A collective: every rank calls it and gets the same tensors, each on the
        device of its own copy of that entry."""
        world = dist.get_world_size(self.group)
        comm = torch.device('cuda', torch.cuda.current_device()) if dist.get_backend(self.group) == 'nccl' else torch.device('cpu')
        out = {}
        for key, t in self.mega.state_dict().items():
            parts = key.split('.')
            if parts[0] != 'sub_modules':
                out[key] = t
                continue
            owner = owner_of(int(parts[1]), world)
            src = owner if self.group is None else dist.get_global_rank(self.group, owner)
            buf = t.detach().to(comm, copy=True).contiguous()
            dist.broadcast(buf, src=src, group=self.group)
            out[key] = buf.to(t.device)
        return out

    # ---- torch path
    def _forward_torch(self, x: torch.Tensor, sigma_noise: Optional[torch.Tensor] = None) -> torch.Tensor:
        world, rank = dist.get_world_size(self.group), dist.get_rank(self.group)
        B = x.shape[0]
        assign, weights = self.route_fn(x)
        rows, subs, w, counts = plan_dispatch(assign, weights, self.n_sub, world)
        child = x[:, 3:] if self.mega.xyz_real else x                        # mega_nerf.py:36
        cols = [child[rows], subs.to(x.dtype).unsqueeze(1)]
        if sigma_noise is not None:
            cols.append(sigma_noise.reshape(B, 1)[rows])
        payload = torch.cat(cols, 1).contiguous()
        width = payload.shape[1]

        # split sizes (one host sync), then the rows
        recv_counts = torch.empty_like(counts)
        dist.all_to_all_single(recv_counts, counts, group=self.group)
        send_l, recv_l = counts.tolist(), recv_counts.tolist()
        recv = payload.new_empty(sum(recv_l), width)
        dist.all_to_all_single(recv, payload, recv_l, send_l, group=self.group)

        # owners compute
        c_in = child.shape[1]
        rk = recv[:, c_in].long()
        out_cols = self.mega.sub_modules[0].rgb_dim + 1
        res = recv.new_zeros(recv.shape[0], out_cols)
        for k in self.owned():
            m = rk == k
            n = int(m.sum())
            if n == 0:
                continue
            nz = recv[m, c_in + 1] if sigma_noise is not None else None
            res[m] = self.sub_fn(k, recv[m, :c_in].contiguous(), nz.unsqueeze(1) if nz is not None else None).to(res.dtype)
        self._last = (int(rows.shape[0]), int(recv.shape[0]))

        # results travel back along the same routes
        back = res.new_empty(rows.shape[0], out_cols)
        dist.all_to_all_single(back, res, send_l, recv_l, group=self.group)

        # accumulate at home, ascending sub-module order (mega_nerf.py:34,46-49)
        out = back.new_zeros(B, out_cols)
        if w is None:
            out[rows] = back
        else:
            for k in range(self.n_sub):
                m = subs == k
                if bool(m.any()):
                    out[rows[m]] += back[m] * w[m].unsqueeze(-1)
        return out


@dataclass
class OwnerTape:
    """What the backward of a recording owner call needs (mn_model_backward_assigned)."""
    tape: torch.Tensor
    n: int                  # received rows
    max_pairs: int          # pairs the tape holds
    precision: int          # K.PREC_FP32 or K.PREC_TC_F16


class _OwnerFn(torch.autograd.Function):
    """`ExpertParallel.compute` under autograd: the parameters are inputs so that their gradients land like _ModelFn's."""

    @staticmethod
    def forward(ctx, ep, recv, c_in, has_noise, max_pairs, rank, world, *params):
        res, tape = ep._record(recv, c_in, has_noise, max_pairs)
        ctx.ep, ctx.tape, ctx.rank, ctx.world = ep, tape, rank, world
        return res

    @staticmethod
    def backward(ctx, grad_res):
        grads = ctx.ep._owner_backward(ctx.tape, grad_res, ctx.rank, ctx.world)
        ctx.tape = None
        need = ctx.needs_input_grad[7:]
        return (None,) * 7 + tuple(g if n else None for g, n in zip(grads, need))


class _CombineFn(torch.autograd.Function):
    """`ExpertParallel.combine` under autograd; no gradient reaches the blend weights (the routing is not differentiated)."""

    @staticmethod
    def forward(ctx, ep, d, back):
        ctx.ep, ctx.d = ep, d
        return ep.combine(d, back)          # autograd is off inside forward: the plain combine

    @staticmethod
    def backward(ctx, dout):
        return None, None, ctx.ep.combine_backward(ctx.d, dout)


class _AllToAll(torch.autograd.Function):
    """Equal-split all_to_all_single; its backward is the same exchange of the gradients, in the other direction."""

    @staticmethod
    def forward(ctx, x, group):
        ctx.group = group
        out = torch.empty_like(x)
        dist.all_to_all_single(out, x.contiguous(), group=group)
        return out

    @staticmethod
    def backward(ctx, g):
        out = torch.empty_like(g)
        dist.all_to_all_single(out, g.contiguous(), group=ctx.group)
        return out, None


class _LazySum:
    """Sum of a device tensor, read back when converted to int."""

    def __init__(self, t: torch.Tensor):
        self.t = t

    def __int__(self) -> int:
        return int(self.t.sum())


@dataclass
class Dispatch:
    """One query's dispatch (mn_model_ep_dispatch): `world` segments of `cap` rows each."""
    world: int
    cap: int
    c_in: int                          # child input columns of a payload row (then the sub-module id, then the noise)
    has_noise: bool
    assign: Optional[torch.Tensor]     # the router's output: int32 [B] (hard routing) ...
    weights: Optional[torch.Tensor]    # ... or blend weights [B, K]
    send: torch.Tensor                 # [world * cap, c_in + 1 (+1)] payload rows
    counts: torch.Tensor               # int32 [world, K] pairs per (destination, sub-module)
    pair_row: torch.Tensor             # int32 [world * cap] home row of each slot, -1 past the pairs
    pair_w: Optional[torch.Tensor]     # [world * cap] blend weight of each slot (blending only)
    row_slots: torch.Tensor            # int32 [B] or [B, K]: the slots of each row, for the combine


def enable(mega, group=None, **kw) -> ExpertParallel:
    """Attach owner-computes execution to a MegaNeRF: `render_rays` then queries it through the process group.
    Sub-modules this rank does not own are never evaluated here (their parameters may stay on the CPU)."""
    ep = ExpertParallel(mega, group, **kw)
    object.__setattr__(mega, '_ep', ep)
    return ep


def disable(mega) -> None:
    object.__setattr__(mega, '_ep', None)
