"""CPU-only: the oracle's spherical-harmonics heads of degree 3 and 4 (rgb_dim 48 and 75, pos_dir_dim 0) against the reference's
own outputs in tests/golden/sh_deg34_v1.pt (tests/golden/make_sh_deg34.py), and live against the reference copy oracle/_ref/
where it exists: NeRF rows at widths 64 and 256 (with sigma_only and sigma_noise), render_rays of a small MegaNeRF with the head
at sh_deg 3 and 4, and the parameter gradients of one training-mode render (in the fixture: shape, float64 checksum and the
first 64 values of every tensor; live: whole tensors).  Bit for bit, as the other reference pins."""
import dataclasses
import os
import sys

import pytest
import torch

import cases as C
from oracle import mn_oracle as O

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden'))
import make_sh_deg34 as MS  # noqa: E402


@pytest.fixture(scope='module')
def golden():
    return torch.load(MS.PATH, map_location='cpu', weights_only=False)


def oracle_outputs() -> dict:
    G = {}
    with torch.inference_mode():
        for name in MS.NERF_CASES:
            net, x, xs, noise = MS.nerf_case(name)
            w = net.weights[0]
            G[f'nerf_{name}'] = dict(wsum=C.net_checksum(net), out=O.nerf_forward(net.spec, w, x),
                                     sigma_only=O.nerf_forward(net.spec, w, xs, sigma_only=True),
                                     noise_out=O.nerf_forward(net.spec, w, x, sigma_noise=noise))
    for deg in (3, 4):
        net, rays, idx, opts, cot = MS.render_case(deg)
        with torch.inference_mode():
            torch.manual_seed(0)
            out, _ = O.render_rays(net, None, rays, idx, opts, None, None, True, True, False)
        G[f'render_d{deg}'] = dict(wsum=C.net_checksum(net), out=out)
        torch.manual_seed(deg)
        res, gn, _ = O.render_grads(dataclasses.replace(net, training=True), None, rays, idx, opts, None, None, {'rgb_fine': cot})
        G[f'grads_d{deg}'] = dict(rgb_fine=res['rgb_fine'], grads=gn)
    return G


def assert_same(got: dict, want: dict):
    assert set(got) == set(want), set(got) ^ set(want)
    for name, w in want.items():
        g = got[name]
        for k, v in w.items():
            if k == 'wsum':
                assert g[k] == v, name
            elif k == 'grads':
                assert len(g[k]) == len(v), name
                for a, b in zip(g[k], v):
                    assert set(a) == set(b), (name, set(a) ^ set(b))
                    for p in b:
                        if isinstance(b[p], dict):          # the fixture's pin of the reference's gradient
                            t = a[p].detach()
                            assert tuple(t.shape) == b[p]['shape'], (name, p)
                            assert torch.equal(t.flatten()[:64], b[p]['head']), (name, p)
                            assert C.checksum(t) == b[p]['checksum'], (name, p)
                        else:
                            assert torch.equal(a[p].detach(), b[p]), (name, p, float((a[p].detach() - b[p]).abs().max()))
            elif k == 'out' and isinstance(v, dict):
                assert set(g[k]) == set(v), (name, set(g[k]) ^ set(v))
                for kk in v:
                    assert torch.equal(g[k][kk], v[kk]), (name, kk, float((g[k][kk] - v[kk]).abs().max()))
            else:
                assert torch.equal(g[k].detach(), v), (name, k, float((g[k].detach() - v).abs().max()))


def test_fixture_shapes(golden):
    for name, c in MS.NERF_CASES.items():
        assert golden[f'nerf_{name}']['out'].shape == (MS.N_ROWS, MS.SH_DIM[c['deg']] + 1)
        assert golden[f'nerf_{name}']['sigma_only'].shape == (MS.N_ROWS, 1)
    for deg in (3, 4):
        g = golden[f'grads_d{deg}']['grads']
        assert len(g) == 4 and all(d['rgb.weight']['shape'] == (MS.SH_DIM[deg], 32) for d in g)
        assert any(float(d['rgb.weight']['head'].abs().max()) > 0 for d in g)


def test_oracle_matches_reference_fixture(golden):
    assert_same(oracle_outputs(), golden)


def test_oracle_matches_reference_live():
    ref = MS.load_reference()
    if ref is None:
        pytest.skip('oracle/_ref/ (the reference copy build() makes) is not present')
    assert_same(oracle_outputs(), MS.run_reference(ref))
