"""CPU-only, world_size 2 over gloo: ExpertParallel.full_state_dict() assembles the whole MegaNeRF's state dict, under the
reference's key names, from ranks that each hold only their own sub-modules' true weights (sub-module k on rank k % 2)."""
import os
import sys

import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import cases  # noqa: F401
from test_dist_gloo import free_port

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def worker(rank, world, port, mname, q):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, 'tests'))
    import cases as C
    from mega_nerf_b200.expert_parallel import ExpertParallel, owner_of
    from mega_nerf_b200.synthetic import build_net
    os.environ['MASTER_ADDR'] = '127.0.0.1'
    os.environ['MASTER_PORT'] = str(port)
    dist.init_process_group('gloo', rank=rank, world_size=world)
    net = C.mega_net(mname)
    mega = build_net(net)
    want = {k: v.clone() for k, v in mega.state_dict().items()}
    # this rank's copies of the sub-modules owned elsewhere hold garbage: only the owner's tensors may reach the result
    with torch.no_grad():
        for k, sub in enumerate(mega.sub_modules):
            if owner_of(k, world) != rank:
                for p in sub.parameters():
                    p.fill_(float('nan') if k % 3 else 1e3 + rank)
    got = ExpertParallel(mega).full_state_dict()
    ok = list(got) == list(want) and all(torch.equal(got[k], want[k]) for k in want)
    q.put((rank, ok, len(want)))
    dist.barrier()
    dist.destroy_process_group()


def run(mname):
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    port = free_port()
    ps = [ctx.Process(target=worker, args=(r, 2, port, mname, q)) for r in range(2)]
    for p in ps:
        p.start()
    out = sorted([q.get(timeout=180) for _ in ps])
    for p in ps:
        p.join(timeout=60)
        assert p.exitcode == 0
    return out


def test_full_state_dict_gathers_every_sub_module_from_its_owner():
    for mname in ('blend2d', 'hard3d_bgreal'):
        out = run(mname)
        assert [r for r, _, _ in out] == [0, 1]
        for rank, ok, n_keys in out:
            assert ok, (mname, rank)
            assert n_keys > 8 * 10, (mname, n_keys)
