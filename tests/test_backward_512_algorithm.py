"""CPU-only: the tensor-core training arithmetic of the 512-wide networks (BASELINE configs[3], 25 x 512) on the fused engine
(csrc/mn_mlp_wg.cuh tc_mlp_wg_kernel<PP_TRAIN_FWD / PP_DGRAD, false, true>, csrc/mn_mlp_tc.cu::mn_train_tc_backward).

The fused kernel runs each N = 512 GEMM as two N = 256 chunks, but every output element is still one fp32 accumulation over
the whole K of fp16 operands, and the images it writes (activation tape, gradient tape) are those of the layer-GEMM path.  So
the restatement of tests/test_backward_wide_algorithm.py describes it: run without rounding it must equal autograd, run with
fp16 rounding its error figures must sit inside a third of the GPU bounds of tests/test_gpu_zo_train_512.py, with S x dZ far
below the fp16 maximum."""
import pytest
import torch

import cases as C
from oracle import mn_oracle as O
from tc_train_ref import errors, h16, wide_tc_chain
from test_backward_wide_algorithm import TC_L2, TC_TENSOR

L = 512

SPECS = {
    'fg': O.NerfSpec(layer_dim=L),                                   # appearance 48 + dir 4, skip layer 4: the C4 sub-module
    'nerf_q1': O.NerfSpec(layer_dim=L, appearance_dim=0),
    'bg_relu': O.NerfSpec(layer_dim=L, xyz_dim=4, shifted_softplus=False, skip_layers=(2, 5)),
    'sh27': O.NerfSpec(layer_dim=L, pos_dir_dim=0, rgb_dim=27),
}


def case(vname, n=640):
    spec = SPECS[vname]
    net = O.make_net('nerf', spec, seed=21)
    if not spec.shifted_softplus:
        net.weights[0]['sigma.bias'] = net.weights[0]['sigma.bias'] + 0.5
    x = C.nerf_rows(spec, n, 31)
    g = torch.Generator().manual_seed(5)
    cot = (torch.rand(n, spec.rgb_dim + 1, generator=g) - 0.3) * 1e-3
    noise = torch.rand(n, 1, generator=g)
    _, want = O.net_forward_grads(net, x, cot, sigma_noise=noise)
    return spec, net.weights[0], x, cot, noise, want[0]


@pytest.mark.parametrize('vname', list(SPECS))
def test_chain_equals_autograd_without_rounding(vname):
    spec, w, x, cot, noise, want = case(vname)
    with torch.no_grad():
        got = wide_tc_chain(spec, w, x, cot, noise, lambda t: t)
    assert set(got) == set(want)
    l2, worst = errors(got, want)
    assert l2 <= 2e-5 and worst[1] <= 5e-4, (l2, worst)


@pytest.mark.parametrize('vname', list(SPECS))
def test_fp16_chain_error_within_gpu_bounds(vname):
    spec, w, x, cot, noise, want = case(vname)
    stats = []
    with torch.no_grad():
        got = wide_tc_chain(spec, w, x, cot, noise, h16, stats)
    l2, worst = errors(got, want)
    print(f'{vname} (L = {spec.layer_dim}): fp16 restatement vs fp32 autograd: rel L2 {l2:.2e}, worst tensor {worst[0]} {worst[1]:.2e}; '
          + ', '.join(f'{k} {v:.3g}' for k, v in stats))
    assert l2 <= TC_L2 / 3 and worst[1] <= TC_TENSOR / 3, (l2, worst)
    assert max(v for k, v in stats if k != 'S') < 65504 / 16
