"""Generate tests/golden/wide_backward_v1.pt by running the UNMODIFIED reference (imported read-only from $MEGA_NERF_REFERENCE)
forward and backward on seeded rows of wide NeRFs: a 2048-wide net of the nerf / npp configs, the 2048-wide mega-nerf-dense
foreground net and a 768-wide net.  The loss is sum(out * cotangent) with seeded cotangents and density noise; the file holds,
per parameter, the norm of param.grad and 64 seeded entries of it, plus the weight checksum.  Weights are regenerated from
seeds (tests/cases.py).  The case table is imported by tests/test_oracle_wide_backward_golden.py; the reference is imported
only when the file is run.  Both run on one CPU thread, so the reductions of the matrix products happen in the same order.

    MEGA_NERF_REFERENCE=<path> python tests/golden/make_wide_backward.py
"""
from __future__ import annotations

import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import cases as C  # noqa: E402
from oracle import mn_oracle as O  # noqa: E402

WIDE_BACKWARD_PATH = os.path.join(ROOT, 'tests', 'golden', 'wide_backward_v1.pt')
WIDE_BACKWARD_CASES = {
    'nerf_2048': O.NerfSpec(layer_dim=2048, appearance_dim=0),       # configs/nerf, npp: no appearance, dir 4
    'dense_fg_2048': O.NerfSpec(layer_dim=2048),                     # configs/mega-nerf-dense foreground
    'fg_768': O.NerfSpec(layer_dim=768),
}
ROWS = 160
PICKS = 64


def inputs(spec: O.NerfSpec):
    """(weights, rows, cotangent, density noise) of a case, all from seeds."""
    net = O.make_net('nerf', spec, seed=23)
    x = C.nerf_rows(spec, ROWS, 33)
    g = torch.Generator().manual_seed(34)
    cot = torch.rand(ROWS, spec.rgb_dim + 1, generator=g) - 0.3
    noise = torch.rand(ROWS, 1, generator=g)
    return net, x, cot, noise


def picks(shape, seed: int) -> torch.Tensor:
    n = 1
    for s in shape:
        n *= s
    return torch.randint(0, n, (PICKS,), generator=torch.Generator().manual_seed(seed))


def summary(grads):
    """name -> (norm, flat indices, values) of each gradient tensor."""
    out = {}
    for i, k in enumerate(sorted(grads)):
        g = grads[k]
        idx = picks(g.shape, 1000 + i)
        out[k] = dict(norm=torch.linalg.vector_norm(g).clone(), idx=idx, val=g.flatten()[idx].clone())
    return out


def main():
    sys.path.insert(0, os.environ['MEGA_NERF_REFERENCE'])     # a checkout of the reference repository
    from make_wide import ref_nerf
    torch.set_num_threads(1)
    G = {}
    for name, spec in WIDE_BACKWARD_CASES.items():
        net, x, cot, noise = inputs(spec)
        ref = ref_nerf(spec, net.weights[0])
        for p in ref.parameters():
            p.requires_grad_(True)
        out = ref(x, sigma_noise=noise)
        (out * cot).sum().backward()
        grads = {k: p.grad.detach().clone() for k, p in ref.named_parameters()}
        _, mine = O.net_forward_grads(net, x, cot, sigma_noise=noise)
        worst = max(float((grads[k].double() - mine[0][k].double()).abs().max()) for k in grads)
        print(f'{name}: {len(grads)} tensors, oracle max abs diff {worst:.3e}')
        G[name] = dict(wsum=C.net_checksum(net), grads=summary(grads))
    torch.save(G, WIDE_BACKWARD_PATH)
    print(f'wrote {WIDE_BACKWARD_PATH} ({os.path.getsize(WIDE_BACKWARD_PATH)} bytes)')


if __name__ == '__main__':
    main()
