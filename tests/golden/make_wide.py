"""Generate tests/golden/wide_v1.pt by running the UNMODIFIED reference (imported read-only from $MEGA_NERF_REFERENCE) on seeded
rows of 2048-wide NeRFs: the shapes the nerf / npp and mega-nerf-dense configs build.  Weights are regenerated from seeds
(tests/cases.py), so the file holds outputs and weight checksums only.  The case table is imported by
tests/test_oracle_wide_golden.py; the reference is imported only when the file is run.

    MEGA_NERF_REFERENCE=<path> python tests/golden/make_wide.py
"""
from __future__ import annotations

import os
import sys

import torch
from torch import nn

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

import cases as C  # noqa: E402
from oracle import mn_oracle as O  # noqa: E402

WIDE_PATH = os.path.join(ROOT, 'tests', 'golden', 'wide_v1.pt')
# name -> (spec, sigma_only)
WIDE_CASES = {
    'nerf_q1': (O.NerfSpec(layer_dim=2048, appearance_dim=0), False),     # configs/nerf, npp: no appearance, dir 4 (quirk Q1)
    'dense_fg': (O.NerfSpec(layer_dim=2048), False),                      # configs/mega-nerf-dense foreground
    'dense_bg': (O.NerfSpec(layer_dim=2048, xyz_dim=4), False),           # configs/mega-nerf-dense background
    'dense_fg_sigma_only': (O.NerfSpec(layer_dim=2048), True),
}
ROWS = 160


def ref_nerf(spec: O.NerfSpec, w) -> nn.Module:
    from mega_nerf.models.nerf import NeRF as R_NeRF, ShiftedSoftplus as R_SSP
    m = R_NeRF(spec.pos_xyz_dim, spec.pos_dir_dim, spec.layers, list(spec.skip_layers), spec.layer_dim,
               spec.appearance_dim, spec.affine_appearance, spec.appearance_count, spec.rgb_dim, spec.xyz_dim,
               R_SSP() if spec.shifted_softplus else nn.ReLU())
    m.load_state_dict(w)
    return m.eval()


def main():
    sys.path.insert(0, os.environ['MEGA_NERF_REFERENCE'])     # a checkout of the reference repository
    G = {}
    with torch.inference_mode():
        for name, (spec, sigma_only) in WIDE_CASES.items():
            net = O.make_net('nerf', spec, seed=21)
            x = C.nerf_rows(spec, ROWS, 31, sigma_only=sigma_only)
            out = ref_nerf(spec, net.weights[0])(x, sigma_only=sigma_only)
            mine = O.nerf_forward(spec, net.weights[0], x, sigma_only=sigma_only)
            d = float((out.double() - mine.double()).abs().max())
            print(f'{name}: out {tuple(out.shape)}, oracle max abs diff {d:.3e}')
            G[name] = dict(wsum=C.net_checksum(net), out=out.clone())
    torch.save(G, WIDE_PATH)
    print(f'wrote {WIDE_PATH} ({os.path.getsize(WIDE_PATH)} bytes)')


if __name__ == '__main__':
    main()
