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
import torch.nn.functional as F

import cases as C
from oracle import mn_oracle as O

L = 768
TC_L2, TC_TENSOR = 3e-2, 3.5e-1          # tests/test_gpu_zk_train_tc.py


def h16(t):
    return t.half().float()


def grad_scale(cot):
    m = float(cot.abs().max())
    return 2.0 ** (10 - torch.tensor(m).log2().ceil().item()) if 0 < m < 3e38 else 1.0


def wide_tc_chain(spec: O.NerfSpec, w, x, cot, noise, rnd, stats=None):
    """-> gradient dict in state-dict layout.  rnd: fp16 rounding of every tensor-core operand and tape image, or identity."""
    L, layers, in_xyz = spec.layer_dim, spec.layers, spec.in_xyz
    R = lambda t: rnd(t)                                                              # noqa: E731
    mm = lambda a, b: a @ b                                                           # fp32 accumulation
    # ---- recording forward (layer_launch with a tape)
    pe = R(O.embed(x[:, :spec.xyz_dim], spec.pos_xyz_dim))
    aux = []
    if spec.pos_dir_dim > 0:
        aux.append(O.embed(x[:, -4:-1], spec.pos_dir_dim))
    ids = x[:, -1].long() if spec.appearance_dim > 0 else None
    if spec.appearance_dim > 0:
        aux.append(w['embedding_a.weight'][ids])
    aux = R(torch.cat(aux, -1))
    h, xin = [], []
    cur = pe
    for i in range(layers):
        inp = torch.cat([pe, cur], -1) if i in spec.skip_layers else cur
        xin.append(inp)
        cur = R(torch.relu(mm(inp, R(w[f'xyz_encodings.{i}.0.weight']).t()) + w[f'xyz_encodings.{i}.0.bias']))
        h.append(cur)
    sig_pre = mm(h[-1], w['sigma.weight'].t())[:, 0] + w['sigma.bias'] + noise.view(-1)      # fp32, CUDA cores
    f = R(mm(h[-1], R(w['xyz_encoding_final.weight']).t()) + w['xyz_encoding_final.bias'])
    fx = torch.cat([f, aux], -1)
    g = R(torch.relu(mm(fx, R(w['dir_a_encoding.0.weight']).t()) + w['dir_a_encoding.0.bias']))
    lin = mm(g, w['rgb.weight'].t()) + w['rgb.bias']
    s = torch.sigmoid(lin) if spec.rgb_dim == 3 else lin

    # ---- head stage (tc_layer_head_dgrad_kernel), fp32
    S = grad_scale(cot)
    go_rgb, go_sig = cot[:, :spec.rgb_dim], cot[:, spec.rgb_dim]
    if spec.shifted_softplus:
        y = sig_pre - 1
        dsp = torch.where(y > 20, torch.ones_like(y), 1 / (1 + torch.exp(-y)))
    else:
        dsp = (sig_pre > 0).float()
    ds = go_sig * dsp
    d = go_rgb * (1 - s) * s if spec.rgb_dim == 3 else go_rgb
    dzg = mm(d, w['rgb.weight']) * (g > 0)                                           # fp32, unscaled
    dzg_img = R(dzg * S)

    G = {k: torch.zeros_like(v) for k, v in w.items()}

    def wop(name, dz_img, xx):                                                        # tc_wgrad_kernel: dZ^T X / S
        G[name + '.weight'] += mm(dz_img.t(), xx) / S
        G[name + '.bias'] += dz_img.sum(0) / S

    # ---- heads (tc_heads_wgrad_kernel) and the embedding (per-image sums x W_e, tc_emb_grad_kernel)
    G['sigma.weight'] += mm(ds.unsqueeze(0), h[-1])
    G['sigma.bias'] += ds.sum().view(1)
    G['rgb.weight'] += mm(d.t(), g)
    G['rgb.bias'] += d.sum(0)
    if spec.appearance_dim > 0:
        sums = torch.zeros(spec.appearance_count, L // 2).index_add_(0, ids, dzg)
        G['embedding_a.weight'] += mm(sums, w['dir_a_encoding.0.weight'][:, L + spec.in_dir:])
    # ---- data-gradient chain (tc_layer_gemm_kernel<false, true>) interleaved with the weight gradients
    Wd = w['dir_a_encoding.0.weight']
    wop('dir_a_encoding.0', dzg_img, fx)
    df = R(mm(dzg_img, R(Wd[:, :L])))                                                 # no mask: F has no activation
    wop('xyz_encoding_final', df, h[-1])
    dz = R((mm(df, R(w['xyz_encoding_final.weight'])) + (ds * S).unsqueeze(-1) * w['sigma.weight']) * (h[-1] > 0))
    if stats is not None:
        stats.append(('S', S))
    for i in range(layers - 1, -1, -1):
        if stats is not None:
            stats.append((f'max |S dZ_{i}|', float(dz.abs().max())))
        wop(f'xyz_encodings.{i}.0', dz, xin[i])
        if i == 0:
            break
        Wi = w[f'xyz_encodings.{i}.0.weight']
        Wh = Wi[:, in_xyz:] if i in spec.skip_layers else Wi                          # hidden columns only
        dz = R(mm(dz, R(Wh)) * (h[i - 1] > 0))
    return G


def errors(got, want):
    num = den = 0.0
    worst = ('', 0.0)
    for k, v in want.items():
        num += float((got[k].double() - v.double()).square().sum())
        den += float(v.double().square().sum())
        scale = float(v.abs().max())
        if scale > 0:
            e = float((got[k] - v).abs().max()) / scale
            if e > worst[1]:
                worst = (k, e)
    return (num / den) ** 0.5, worst


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
