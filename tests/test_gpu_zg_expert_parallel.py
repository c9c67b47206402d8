"""GPU: owner-computes execution (mega_nerf_b200/expert_parallel.py, SURVEY.md §8f-5) through the device-side defaults
(mn_model_route + the owned sub-modules' own forward) in a process group of ONE rank: the all-to-alls are then identity
exchanges, so the result must equal the ordinary MegaNeRF call and render_rays must return what it returns without the
process group.  The multi-rank dispatch logic itself is covered on CPU by tests/test_dist_gloo.py (world_size 2, gloo);
a real multi-GPU run is `bench.py --gpus 2 --parallelism experts` under torchrun.  Sorted last."""
import os
from argparse import Namespace

import pytest
import torch
import torch.distributed as dist

import cases as C
from test_gpu_parity import DEV, M, product_net, relerr

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def one_rank_group():
    if dist.is_initialized():
        yield None
        return
    os.environ.setdefault('MASTER_ADDR', '127.0.0.1')
    os.environ.setdefault('MASTER_PORT', '29653')
    dist.init_process_group('nccl', rank=0, world_size=1, device_id=DEV)
    yield None
    dist.destroy_process_group()


@pytest.mark.parametrize('mname', ['hard2d', 'blend2d', 'hard3d_bgreal'])
def test_rows_through_expert_parallel(one_rank_group, mname):
    from mega_nerf_b200 import expert_parallel as EP
    M().set_precision('fp32')
    net = C.mega_net(mname)
    x = C.mega_rows(net, 700, 51).to(DEV)
    pn = product_net(net)
    with torch.no_grad():
        want = pn(x)
        ep = EP.ExpertParallel(pn)
        got = ep.forward(x)
    assert ep.last_pairs == ep.last_owned >= 700
    assert relerr(got, want) <= 1e-6


def test_render_rays_through_expert_parallel(one_rank_group):
    from mega_nerf_b200 import expert_parallel as EP
    m = M()
    m.set_precision('tc_f16')
    net, _, rays, idx, opts, _, _ = C.render_case('c2_mega8_blend')
    pn = product_net(net)
    hp = Namespace(**vars(opts))
    with torch.no_grad():
        want, _ = m.render_rays(pn, None, rays.to(DEV), idx.to(DEV), hp, None, None, True, True, False)
        EP.enable(pn)
        try:
            got, _ = m.render_rays(pn, None, rays.to(DEV), idx.to(DEV), hp, None, None, True, True, False)
        finally:
            EP.disable(pn)
    assert set(got) == set(want)
    for k in want:
        # same kernels per sub-module; rows are grouped per sub-module call instead of one bucketed launch
        assert relerr(got[k], want[k]) <= (5e-5 if 'variance' in k else 1e-5), k
