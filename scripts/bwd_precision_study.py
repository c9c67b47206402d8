#!/usr/bin/env python
"""CPU study for the tensor-core backward (DESIGN.md §10 item 4): how large is the parameter-gradient error if the tapes
and operands are 16-bit, as the tensor-core backward keeps them?  The chain rule of tests/test_backward_algorithm.py is
re-run with the operands of every GEMM rounded to fp16 / bf16 (fp32 accumulation, like the MMA) and compared with fp32
autograd, for upstream gradients of realistic magnitude (render_rays' own dL/d(rgb, sigma) on a grad case) with and
without a power-of-two loss scale.  Prints the worst per-tensor deviation relative to the tensor's max.

    python scripts/bwd_precision_study.py
"""
import os
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
import cases as C  # noqa: E402
from oracle import mn_oracle as O  # noqa: E402


def rnd(t, dt):
    return t if dt is None else t.to(dt).float()


def quantised_grads(spec, w, x, cot, act_dt, grad_dt, w_dt, scale=1.0):
    """nerf.py:115-160 forward with activations rounded to act_dt, backward with dZ rounded to grad_dt; weights w_dt."""
    L, layers = spec.layer_dim, spec.layers
    W = {k: rnd(v, w_dt) if k.endswith('weight') and v.dim() == 2 and 'embedding' not in k else v for k, v in w.items()}
    pe = rnd(O.embed(x[:, :3], spec.pos_xyz_dim), act_dt)
    aux = rnd(torch.cat([O.embed(x[:, -4:-1], spec.pos_dir_dim), w['embedding_a.weight'][x[:, -1].long()]], -1), act_dt)
    h, xin, cur = [], [], pe
    for i in range(layers):
        inp = torch.cat([pe, cur], -1) if i in spec.skip_layers else cur
        xin.append(inp)
        cur = rnd(torch.relu(F.linear(inp, W[f'xyz_encodings.{i}.0.weight'], w[f'xyz_encodings.{i}.0.bias'])), act_dt)
        h.append(cur)
    sig_pre = F.linear(h[-1], w['sigma.weight'], w['sigma.bias'])[:, 0]
    f = rnd(F.linear(h[-1], W['xyz_encoding_final.weight'], w['xyz_encoding_final.bias']), act_dt)
    g = rnd(torch.relu(F.linear(torch.cat([f, aux], -1), W['dir_a_encoding.0.weight'], w['dir_a_encoding.0.bias'])), act_dt)
    s = torch.sigmoid(F.linear(g, w['rgb.weight'], w['rgb.bias']))
    G = {}
    q = lambda t: rnd(t, grad_dt)                                              # noqa: E731  what the gradient tape would hold
    cot = cot * scale                                                           # loss scaling: once, upstream

    def wop(name, dz, xx):
        G[name + '.weight'] = dz.t() @ xx / scale
        G[name + '.bias'] = dz.sum(0) / scale
    ds = cot[:, 3] * torch.sigmoid(sig_pre - 1)
    dr = q(cot[:, :3] * (1 - s) * s)
    wop('rgb', dr, g)
    dz = q((dr @ w['rgb.weight']) * (g > 0))
    wop('dir_a_encoding.0', dz, torch.cat([f, aux], -1))
    dzf = q(dz @ W['dir_a_encoding.0.weight'][:, :L])
    wop('xyz_encoding_final', dzf, h[-1])
    dz = q((dzf @ W['xyz_encoding_final.weight'] + ds.unsqueeze(-1) * w['sigma.weight']) * (h[-1] > 0))
    for i in range(layers - 1, -1, -1):
        wop(f'xyz_encodings.{i}.0', dz, xin[i])
        if i == 0:
            break
        Wi = W[f'xyz_encodings.{i}.0.weight']
        dz = q((dz @ (Wi[:, spec.in_xyz:] if i in spec.skip_layers else Wi)) * (h[i - 1] > 0))
    return G


def main():
    torch.manual_seed(0)
    spec = O.NerfSpec()                                   # 8 x 256
    net = O.make_net('nerf', spec, seed=21)
    x = C.nerf_rows(spec, 4096, 31)
    # upstream gradients with the magnitude render_rays produces: mean over 1024 rays x 192 samples of an MSE loss
    cot = torch.randn(4096, 4) * (2.0 / (3 * 1024)) * torch.rand(4096, 1) * 0.05
    _, want = O.net_forward_grads(net, x, cot)
    want = want[0]
    print(f'upstream gradient magnitude: max {float(cot.abs().max()):.2e}, median {float(cot.abs().median()):.2e}')
    for label, act_dt, grad_dt, w_dt, scale in (
            ('fp16 acts / fp16 grads, no scale', torch.float16, torch.float16, torch.float16, 1.0),
            ('fp16 acts / fp16 grads, x65536 (GradScaler)', torch.float16, torch.float16, torch.float16, 65536.0),
            ('fp16 acts / bf16 grads, no scale', torch.float16, torch.bfloat16, torch.float16, 1.0),
            ('bf16 acts / bf16 grads, no scale', torch.bfloat16, torch.bfloat16, torch.bfloat16, 1.0),
            ('fp16 acts + weights, fp32 grads', torch.float16, None, torch.float16, 1.0),
            ('fp32 acts + weights, bf16 grads', None, torch.bfloat16, None, 1.0),
            ('fp32 acts + weights, fp16 grads x65536', None, torch.float16, None, 65536.0),
            ('fp32 reference chain (sanity)', None, None, None, 1.0)):
        with torch.no_grad():
            got = quantised_grads(spec, net.weights[0], x, cot, act_dt, grad_dt, w_dt, scale)
        worst, l2n, l2d = 0.0, 0.0, 0.0
        for k, v in got.items():
            ref = want[k]
            worst = max(worst, float((v - ref).abs().max() / ref.abs().max()))
            l2n += float((v - ref).square().sum())
            l2d += float(ref.square().sum())
        print(f'{label:46s} worst per-tensor {worst:.2e}   whole-gradient relative L2 {(l2n / l2d) ** 0.5:.2e}')


if __name__ == '__main__':
    main()
