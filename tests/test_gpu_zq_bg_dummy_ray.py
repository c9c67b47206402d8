"""GPU: distributed training on a batch in which no ray reaches the background (rendering.py:143-171).  With RANK set, a
train()-mode `render_rays` renders one dummy ray through the background network and adds none of it to the results, so that
this rank still takes part in the background network's gradient all-reduce: the results are those of the same call without
RANK, and every background parameter gets an all-zero gradient instead of none."""
from argparse import Namespace

import pytest
import torch

import cases as C
from test_gpu_parity import DEV, M, product_net
from test_gpu_zp_fused_bg import no_bg

pytestmark = pytest.mark.gpu

# foreground gradients with and without the dummy ray: the same graph, up to the order of the backward's atomic sums
FG_GRAD_TOL = 1e-5


def _train_step(rname):
    m = M()
    m.set_precision('fp32')
    net, bg_net, rays, idx, opts, c, rd = C.render_case(rname)
    pn = product_net(net).requires_grad_(True).train()
    pb = product_net(bg_net).requires_grad_(True).train()
    c, rd = c.to(DEV), rd.to(DEV)
    r = no_bg(rays.to(DEV), c, rd)
    torch.manual_seed(7)
    res, present = m.render_rays(pn, pb, r, idx.to(DEV) if idx is not None else None, Namespace(**vars(opts)), c, rd,
                                 True, True, False)
    loss = sum((v * torch.linspace(0.5, 1.5, v.numel(), device=DEV).view_as(v)).sum()
               for v in res.values() if v.requires_grad)
    loss.backward()
    return res, present, pn, pb


@pytest.mark.parametrize('rname', ['bg_single', 'bg_cascade'])
def test_dummy_bg_ray(monkeypatch, rname):
    want, present, pn_want, pb_want = _train_step(rname)
    assert not present
    assert all(p.grad is None for p in pb_want.parameters())

    monkeypatch.setenv('RANK', '0')
    got, present, pn, pb = _train_step(rname)
    assert present
    assert set(got) == set(want), set(got) ^ set(want)
    for k in want:
        assert torch.equal(got[k], want[k]), (k, float((got[k] - want[k]).abs().max()))
    for name, p in pb.named_parameters():
        assert p.grad is not None, name
        assert not p.grad.any(), (name, float(p.grad.abs().max()))
    for (name, p), q in zip(pn.named_parameters(), pn_want.parameters()):
        assert (p.grad is None) == (q.grad is None), name
        if p.grad is not None:
            scale = float(q.grad.abs().max())
            assert float((p.grad - q.grad).abs().max()) <= FG_GRAD_TOL * scale, name
