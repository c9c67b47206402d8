"""CPU-only: the tensor-core training arithmetic of the layer-GEMM path (layer_dim 768..2048; csrc/mn_layer_gemm.cuh,
csrc/mn_mlp_tc.cu::mn_train_tc_backward) restated with plain tensor algebra at L = 768 (and 2048 for one net) and checked against the oracle's autograd.

The restatement follows the kernels step by step: fp16 operands with fp32 accumulation in every GEMM, fp16 activations on
the tape, the head stage in fp32, gradient images S x dZ rounded to fp16 with S = 2^(10 - ceil(log2 max|grad_out|)), the
data-gradient chain dF = dZ_G W_dira[:, :L], dH_last = dF W_final + dsigma sigma_w, dZ_{l-1} = mask(dZ_l W_l[:, hidden]),
weight gradients dZ^T X / S, and the appearance-embedding gradient from per-image sums of dZ_G rows.  Run without rounding
it must equal autograd (the algebra); run with fp16 rounding its error figures predict the GPU bounds of
tests/test_gpu_zn_train_wide.py (TC_L2 = 3e-2 on the whole gradient vector, TC_TENSOR = 3.5e-1 per tensor)."""
import pytest
import torch

import cases as C
from oracle import mn_oracle as O
from tc_train_ref import errors, grad_scale, h16, wide_tc_chain

L = 768
TC_L2, TC_TENSOR = 3e-2, 3.5e-1          # tests/test_gpu_zk_train_tc.py


SPECS = {
    'fg': O.NerfSpec(layer_dim=L),                                   # appearance 48 + dir 4, skip layer 4
    'fg_2048': O.NerfSpec(layer_dim=2048),                           # the width of the shipped configs
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
    """The algebra: skip layers contribute only their hidden columns, dsigma x sigma_w joins before the last ReLU mask,
    the embedding gradient comes from per-image sums, and S cancels exactly (a power of two)."""
    spec, w, x, cot, noise, want = case(vname)
    with torch.no_grad():
        got = wide_tc_chain(spec, w, x, cot, noise, lambda t: t)
    assert set(got) == set(want)
    l2, worst = errors(got, want)
    # fp32 in another summation order; the layer-0 weights of the ReLU-sigma net sum gradients that mostly cancel
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
    # fp16 headroom: S x dZ stays far below the fp16 maximum (65504) through every layer
    assert max(v for k, v in stats if k != 'S') < 65504 / 16


def test_grad_scale_is_the_kernels_power_of_two():
    """tc_grad_scale_kernel: S = 2^(10 - ceil(log2 max|g|)), so S max|g| lies in (512, 1024]."""
    for m in (1e-6, 3e-4, 0.5, 1.0, 7.0):
        S = grad_scale(torch.tensor([m, -m / 3]))
        assert 512 < S * m <= 1024, (m, S)
        assert S == 2.0 ** round(torch.tensor(S).log2().item())
