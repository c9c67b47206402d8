"""Times one training query (recording forward + backward, precision tc_f16) of a MegaNeRF two ways:
  routed  without expert parallelism: the whole MegaNeRF on this rank, mn_model_forward_train_tc + mn_model_backward_tc
  ep      the expert-parallel device path (mega_nerf_b200/expert_parallel.py): dispatch, all-to-alls, the recording owner call
          (mn_model_forward_assigned_train, one host read of the received pair count), combine; then the combine's backward,
          the reverse all-to-all of the result gradients and mn_model_backward_assigned
on the BASELINE configs[3] network (25 x 512 MegaNeRF, 5 x 5 centroid grid, boundary margin 1.15, 2-D clustering) and a query
of --rows rows (default 4096 rays x 128 fine samples) with density noise, each rank its own rows, sub-module k owned by rank
k mod world.

    python scripts/ep_train_time.py [--rows N] [--iters K] [--warmup W] [--out FILE]      one GPU, a one-rank NCCL group
    torchrun --nproc-per-node G scripts/ep_train_time.py [...]                             G ranks, one GPU each

Each line: ms per training query (CUDA events over --iters queries after --warmup, the slowest rank), the peak device memory
one query allocates beyond what was allocated before it (torch's caching-allocator statistics, the largest rank), and for the
ep line the relative L2 distance of its parameter gradients from the routed query's (at world 1 both are the same sum).
The card's name and power limit are read in the same call."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, 'tests')):
    sys.path.insert(0, p)
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

import mega_nerf_b200 as M  # noqa: E402
from mega_nerf_b200 import expert_parallel as EP  # noqa: E402
from mega_nerf_b200.synthetic import build_net  # noqa: E402
from oracle import mn_oracle as O  # noqa: E402
import cases as C  # noqa: E402


def smi(fields: str, dev: int) -> str:
    return subprocess.run(['nvidia-smi', '-i', str(dev), f'--query-gpu={fields}', '--format=csv,noheader'], stdout=subprocess.PIPE,
                          text=True).stdout.strip()


def per_query_ms(fn, iters: int, warmup: int) -> float:
    for _ in range(warmup):
        fn()
    dist.barrier()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    t = torch.tensor([a.elapsed_time(b) / iters], device='cuda')
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t)


def peak_bytes(fn) -> int:
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    t = torch.tensor([torch.cuda.max_memory_allocated() - base], device='cuda', dtype=torch.int64)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return int(t)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rows', type=int, default=4096 * 128)
    ap.add_argument('--iters', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('ep_train_time.py measures on a CUDA device; none found')
    rank, world = int(os.environ.get('RANK', 0)), int(os.environ.get('WORLD_SIZE', 1))
    local = int(os.environ.get('LOCAL_RANK', 0))
    dev = torch.device('cuda', local)
    torch.cuda.set_device(dev)
    os.environ.setdefault('MASTER_ADDR', '127.0.0.1')
    os.environ.setdefault('MASTER_PORT', '29683')
    dist.init_process_group('nccl', rank=rank, world_size=world, device_id=dev)
    card = smi('name,power.limit', local)

    M.set_train_precision('tc_f16')
    net = O.make_net('mega', O.NerfSpec(layer_dim=512), seed=3, n_sub=25, centroids=O.grid_centroids(5, 5), boundary_margin=1.15,
                     cluster_2d=True)
    pn = build_net(net, dev, trainable=True)
    x = C.mega_rows(net, args.rows, 51 + rank).to(dev)
    g = torch.Generator().manual_seed(7 + rank)
    nz = torch.rand(args.rows, 1, generator=g).to(dev)
    cot = ((torch.rand(args.rows, 4, generator=g) - 0.5) * 1e-4).to(dev)
    ep = EP.ExpertParallel(pn)

    def routed():
        pn.zero_grad(set_to_none=True)
        (pn(x, sigma_noise=nz) * cot).sum().backward()

    def expert_parallel():
        pn.zero_grad(set_to_none=True)
        (ep.forward(x, nz) * cot).sum().backward()

    def grads():
        return torch.cat([p.grad.reshape(-1) for p in pn.parameters() if p.grad is not None]).double()

    routed()
    on_tc = pn._native().train_on_tensor_cores()
    g_routed = grads() if world == 1 else None
    expert_parallel()
    rel_l2 = float((grads() - g_routed).norm() / g_routed.norm()) if world == 1 else None
    lines = []
    for impl, fn in (('routed', routed), ('ep', expert_parallel)):
        ms = per_query_ms(fn, args.iters, args.warmup)
        peak = peak_bytes(fn)
        line = dict(impl=impl, world=world, rows=args.rows, precision='tc_f16', on_tensor_cores=on_tc, ms_per_train_query=round(ms, 3),
                    peak_bytes=peak, card=card)
        if impl == 'ep':
            line.update(pairs_rank0=ep.last_pairs, grads_rel_l2_vs_routed=rel_l2)
        lines.append(line)
        if rank == 0:
            print(json.dumps(line), flush=True)
    if rank == 0 and args.out:
        with open(args.out, 'w') as f:
            json.dump(dict(card=card, lines=lines), f, indent=1)
    dist.barrier()
    dist.destroy_process_group()


if __name__ == '__main__':
    main()
