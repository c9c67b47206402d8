"""GPU: mn_render_rays (the whole foreground inference path in one C call) returns exactly what render_rays returns -
it sequences the same stage entry points on the same stream.  Sorted last: written without hardware access."""
from argparse import Namespace

import pytest
import torch

import cases as C
from test_gpu_parity import DEV, M, product_net

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize('rname,prec', [('c2_mega8_blend', 'tc_f16'), ('c2_mega8_hard', 'fp32'), ('c5_sh2', 'tc_f16'),
                                        ('single_fine', 'tc_f16x3'), ('cascade_fine', 'tc_f16'), ('c1_cascade_noapp', 'fp32')])
def test_fused_call_equals_staged_calls(rname, prec):
    m = M()
    m.set_precision(prec)
    net, bg_net, rays, idx, opts, _, _ = C.render_case(rname)
    assert bg_net is None
    pn = product_net(net)
    hp = Namespace(**vars(opts))
    r = rays.to(DEV)
    i = idx.to(DEV) if idx is not None else None
    with torch.no_grad():
        want, _ = m.render_rays(pn, None, r, i, hp, None, None, True, True, False)
        got = m.render_rays_fused(pn, r, i, hp, True, True)
    assert set(got) == set(want), set(got) ^ set(want)
    for k in want:
        assert torch.equal(got[k], want[k]), (k, float((got[k] - want[k]).abs().max()))
    with torch.no_grad():
        only_rgb = m.render_rays_fused(pn, r, i, hp, False, False)
    typ = 'fine' if opts.fine_samples > 0 else 'coarse'
    assert set(only_rgb) == {f'rgb_{typ}'} | ({'rgb_coarse'} if (opts.use_cascade and opts.fine_samples > 0) else set())
    assert torch.equal(only_rgb[f'rgb_{typ}'], want[f'rgb_{typ}'])
