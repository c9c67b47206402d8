"""Generate tests/golden/backward_v1.pt: parameter gradients of the UNMODIFIED reference
(imported read-only from the reference checkout) on the seeded cases `GRAD_CASES` of tests/cases.py.

The reference's training step (runner.py:346-378, :265) is `render_rays(..., get_depth=False,
get_depth_variance=True, get_bg_fg_rgb=False)` followed by `loss.backward()`; here the loss is
sum_k sum(results[k] * cotangent[k]) over the differentiable outputs with seeded cotangents, the
modules are in eval() mode (no jitter / sigma noise: those only add random inputs, the gradient
arithmetic is identical) and gradients are read from `param.grad`.

Needs a checkout of the reference:    MEGA_NERF_REFERENCE=<path> python tests/golden/make_golden_backward.py
It also asserts that the oracle's autograd (oracle/mn_oracle.py::render_grads) agrees.
"""
from __future__ import annotations

import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as MG  # noqa: E402  (sets sys.path for cases / oracle / reference)

C, O, R_render = MG.C, MG.O, MG.R_render


def ref_grads(mod, net: O.Net):
    """param.grad of a reference module, re-keyed per sub-module like the oracle's weight dicts."""
    if net.kind == 'nerf':
        subs = [mod]
    elif net.kind == 'cascade':
        subs = [mod.coarse, mod.fine]
    else:
        subs = list(mod.sub_modules)
    out = []
    for s in subs:
        out.append({k: (p.grad.detach().clone() if p.grad is not None else torch.zeros_like(p))
                    for k, p in s.named_parameters()})
    return out


def main():
    G = {}
    worst = 0.0
    for name in C.GRAD_CASES:
        net, bg_net, rays, idx, opts, center, radius = C.render_case(name)
        cot = C.grad_cotangents(name, rays.shape[0])
        rn = MG.ref_net(net)
        rb = MG.ref_net(bg_net) if bg_net is not None else None
        for m in (rn, rb):
            if m is not None:
                for p in m.parameters():
                    p.requires_grad_(True)
        res, _ = R_render.render_rays(rn, rb, rays, idx, MG.hparams_of(opts), center, radius, False, True, False)
        loss = sum((res[k] * c).sum() for k, c in cot.items() if k in res and res[k].requires_grad)
        loss.backward()
        gn = ref_grads(rn, net)
        gb = ref_grads(rb, bg_net) if rb is not None else None
        ores, ogn, ogb = O.render_grads(net, bg_net, rays, idx, opts, center, radius, cot)
        for tag, a, b in (('net', gn, ogn), ('bg', gb, ogb)):
            if a is None:
                continue
            for i, (ga, gb_) in enumerate(zip(a, b)):
                assert set(ga) == set(gb_), (name, tag, set(ga) ^ set(gb_))
                for k in ga:
                    d = float((ga[k].double() - gb_[k].double()).abs().max())
                    worst = max(worst, d)
                    if d != 0.0:
                        print(f'  {name}/{tag}[{i}]/{k}: oracle != reference, max abs diff {d:.3e} '
                              f'(max |g| {float(ga[k].abs().max()):.3e})')
        G[name] = dict(net=gn, bg=gb, out={k: v.detach().clone() for k, v in res.items()},
                       wsum=C.net_checksum(net) + (C.net_checksum(bg_net) if bg_net else 0.0),
                       xsum=C.checksum(rays, idx, *cot.values()))
        nz = sum(int((g.abs() > 0).any()) for sub in gn for g in sub.values())
        print(f'{name}: keys={sorted(res)}  non-zero grad tensors {nz}/{sum(len(s) for s in gn)}')
    C.save_golden(G, C.GRAD_GOLDEN_PATH)
    print(f'wrote {C.GRAD_GOLDEN_PATH}.part*; '
          f'worst oracle-vs-reference gradient diff {worst:.3e}')


if __name__ == '__main__':
    main()
