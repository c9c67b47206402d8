"""Generate tests/golden/train_mode_v1.pt: the UNMODIFIED reference in train() mode (stratified jitter, density noise,
random inverse-CDF draws - rendering.py:83,294,321,511) under a fixed torch seed, forward results for several cases and
parameter gradients for one.  The oracle must consume the global RNG in exactly the reference's order to reproduce them.
Needs a checkout of the reference:    MEGA_NERF_REFERENCE=<path> python tests/golden/make_golden_train_mode.py"""
from __future__ import annotations

import dataclasses
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as MG  # noqa: E402
import make_golden_backward as MB  # noqa: E402

C, O, R_render = MG.C, MG.O, MG.R_render
CASES = ['g_single', 'g_cascade', 'g_mega_blend', 'g_bg_single', 'g_sh2', 'g_coarse_only']
SEED = 99


def main():
    G = {}
    for name in CASES:
        net, bg, rays, idx, opts, c, r = C.render_case(name)
        rn = MG.ref_net(net).train()
        rb = MG.ref_net(bg).train() if bg is not None else None
        torch.manual_seed(SEED)
        with torch.no_grad():
            ref, present = R_render.render_rays(rn, rb, rays, idx, MG.hparams_of(opts), c, r, True, True, False)
        torch.manual_seed(SEED)
        with torch.no_grad():
            got, _ = O.render_rays(dataclasses.replace(net, training=True), dataclasses.replace(bg, training=True) if bg else None,
                                   rays, idx, opts, c, r, True, True, False)
        for k in ref:
            assert torch.equal(ref[k], got[k]), (name, k)
        G[name] = dict(out={k: v.clone() for k, v in ref.items()}, present=present)
        print(name, sorted(ref))
    # gradients in train() mode for one case
    name = 'g_single'
    net, bg, rays, idx, opts, c, r = C.render_case(name)
    cot = C.grad_cotangents(name, rays.shape[0])
    rn = MG.ref_net(net).train()
    for p in rn.parameters():
        p.requires_grad_(True)
    torch.manual_seed(SEED)
    res, _ = R_render.render_rays(rn, None, rays, idx, MG.hparams_of(opts), c, r, False, True, False)
    (res['rgb_fine'] * cot['rgb_fine']).sum().backward()
    gref = MB.ref_grads(rn, net)
    torch.manual_seed(SEED)
    _, gor, _ = O.render_grads(dataclasses.replace(net, training=True), None, rays, idx, opts, c, r, cot)
    for k in gref[0]:
        assert torch.equal(gref[0][k], gor[0][k]), k
    G['grads_g_single'] = gref
    G['seed'] = SEED
    torch.save(G, C.TRAIN_GOLDEN_PATH)
    print(f'wrote {C.TRAIN_GOLDEN_PATH} ({os.path.getsize(C.TRAIN_GOLDEN_PATH) / 1e3:.0f} kB); oracle == reference (bit-exact)')


if __name__ == '__main__':
    main()
