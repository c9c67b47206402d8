"""Times one expert-parallel model query (mega_nerf_b200/expert_parallel.py) three ways:
  torch   the torch path: split sizes exchanged and read back, one NeRF call per owned sub-module, a Python blend loop
  device  the device path: mn_model_route + mn_model_ep_dispatch, equal-split all-to-alls, mn_model_forward_assigned,
          mn_model_ep_combine, no host sync
  graph   the device path captured once in a CUDA graph and replayed
on the BASELINE configs[3] network (25 x 512 MegaNeRF, 5 x 5 centroid grid, boundary margin 1.15, 2-D clustering; tc_f16) and
a query of --rows rows (default 4096 rays x 128 fine samples), each rank its own rows, sub-module k owned by rank k mod world.

    python scripts/ep_time.py [--rows N] [--iters K] [--warmup W] [--out FILE]          one GPU, a one-rank NCCL group
    torchrun --nproc-per-node G scripts/ep_time.py [...]                                 G ranks, one GPU each

Each line: ms per query (CUDA events over --iters queries after --warmup, the slowest rank), the bytes one rank sends per
exchange (outbound rows, counts or split sizes, and the returned results; in a one-rank group the all-to-alls are local
copies of that size), and whether the result equals the torch path's.  The card's name and power limit are read in the same
call."""
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
from mega_nerf_b200 import _cabi as K  # noqa: E402
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rows', type=int, default=4096 * 128)
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('ep_time.py measures on a CUDA device; none found')
    rank, world = int(os.environ.get('RANK', 0)), int(os.environ.get('WORLD_SIZE', 1))
    local = int(os.environ.get('LOCAL_RANK', 0))
    dev = torch.device('cuda', local)
    torch.cuda.set_device(dev)
    os.environ.setdefault('MASTER_ADDR', '127.0.0.1')
    os.environ.setdefault('MASTER_PORT', '29681')
    dist.init_process_group('nccl', rank=rank, world_size=world, device_id=dev)
    card = smi('name,power.limit', local)

    M.set_precision('tc_f16')
    net = O.make_net('mega', O.NerfSpec(layer_dim=512), seed=3, n_sub=25, centroids=O.grid_centroids(5, 5), boundary_margin=1.15,
                     cluster_2d=True)
    pn = build_net(net, dev)
    x = C.mega_rows(net, args.rows, 51 + rank).to(dev)
    torch_ep = EP.ExpertParallel(pn, sub_fn=lambda k, rows, nz: pn.sub_modules[k](rows, sigma_noise=nz))
    dev_ep = EP.ExpertParallel(pn)
    lines = []
    with torch.no_grad():
        want = torch_ep.forward(x)
        pairs = torch_ep.last_pairs
        got = dev_ep.forward(x)
        same_dev = torch.equal(got, want)

        # graph: warm up on a side stream, capture, replay (as GraphedRenderRays does)
        side = torch.cuda.Stream(dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):
            for _ in range(2):
                dev_ep.forward(x)
        torch.cuda.current_stream(dev).wait_stream(side)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, capture_error_mode='thread_local'):
            replayed = dev_ep.forward(x)
        g.replay()
        torch.cuda.synchronize()
        same_graph = torch.equal(replayed, want)

        width = x.shape[1] + 1                               # child input (7 columns) + sub-module id
        out_cols = pn.sub_modules[0].rgb_dim + 1
        cap = int(K.lib().mn_model_ep_segment_rows(dev_ep.native(dev).handle, args.rows))
        seg_bytes = dict(rows_out=world * cap * width * 4, counts=world * len(pn.sub_modules) * 4, results_back=world * cap * out_cols * 4)
        torch_bytes = dict(rows_out=pairs * width * 4, split_sizes=world * 8, results_back=pairs * out_cols * 4)
        for impl, fn, nbytes, same in (('torch', lambda: torch_ep.forward(x), torch_bytes, True),
                                       ('device', lambda: dev_ep.forward(x), seg_bytes, same_dev),
                                       ('graph', g.replay, seg_bytes, same_graph)):
            ms = per_query_ms(fn, args.iters, args.warmup)
            lines.append(dict(impl=impl, world=world, rows=args.rows, pairs_rank0=pairs, segment_rows=cap, ms_per_query=round(ms, 3),
                              bytes_per_rank=nbytes, equals_torch_path=same, card=card))
            if rank == 0:
                print(json.dumps(lines[-1]), flush=True)
        # device memory of one query at a few world sizes: segments out and in, results out and in, the owner call's workspace
        h = dev_ep.native(dev).handle
        for w in (1, 2, 8):
            buf = dict(world=w, segment_rows=cap, send_and_recv_bytes=2 * w * cap * width * 4,
                       results_bytes=2 * w * cap * out_cols * 4,
                       owner_workspace_bytes=int(K.lib().mn_model_forward_assigned_workspace_bytes(h, w * cap, K.PREC_TC_F16)))
            lines.append(dict(buffers=buf))
            if rank == 0:
                print(json.dumps(lines[-1]), flush=True)
    del g
    if rank == 0 and args.out:
        with open(args.out, 'w') as f:
            json.dump(dict(card=card, lines=lines), f, indent=1)
    dist.barrier()
    dist.destroy_process_group()


if __name__ == '__main__':
    main()
