"""GPU: networks ingested from the reference's on-disk formats (SURVEY.md §8f-4) render like the oracle built
from the same tensors: the merged TorchScript container of tests/golden/container_v1.pt (written by the
reference's MegaNeRFContainer, scripts/merge_submodules.py:70-77) and a `module.`-prefixed checkpoint."""
from argparse import Namespace

import pytest
import torch

import cases as C
from oracle import mn_oracle as O
from test_gpu_parity import DEV, M, relerr

pytestmark = pytest.mark.gpu


def test_container_model_matches_oracle():
    m = M()
    m.set_precision('fp32')
    fg, bg, _ = C.container_nets()
    hp = C.container_hparams(container_path=C.container_path())
    net = m.get_nerf(hp, 10).to(DEV).eval().requires_grad_(False)
    bnet = m.get_bg_nerf(hp, 10).to(DEV).eval().requires_grad_(False)
    x = C.mega_rows(fg, 500, 77)
    xb = C.mega_rows(bg, 500, 78)
    with torch.inference_mode():
        assert relerr(net(x.to(DEV)), O.mega_forward(fg, x)) <= 1e-5
        assert relerr(bnet(xb.to(DEV)), O.mega_forward(bg, xb)) <= 1e-5


def test_container_render_with_background():
    m = M()
    m.set_precision('fp32')
    fg, bg, _ = C.container_nets()
    hp = C.container_hparams(container_path=C.container_path())
    net = m.get_nerf(hp, 10).to(DEV).eval().requires_grad_(False)
    bnet = m.get_bg_nerf(hp, 10).to(DEV).eval().requires_grad_(False)
    rays = O.synthetic_rays(40, seed=4, far=1e5)
    rays[::2, 7] = 0.4
    idx = O.synthetic_indices(40, 10)
    center, radius = torch.tensor([0.05, -0.02, 0.03]), torch.tensor([0.8, 0.9, 1.0])
    opts = O.RenderOpts(coarse_samples=32, fine_samples=32, container_path=C.container_path())
    with torch.inference_mode():
        want, wp = O.render_rays(fg, bg, rays, idx, opts, center, radius, True, True, True)
        rp = Namespace(**vars(opts), **{k: v for k, v in vars(hp).items() if k not in vars(opts)})
        got, gp = m.render_rays(net, bnet, rays.to(DEV), idx.to(DEV), rp, center.to(DEV), radius.to(DEV), True, True, True)
    assert gp == wp and set(got) == set(want)
    for k, v in want.items():
        assert relerr(got[k], v) <= (5e-4 if 'variance' in k else 1e-4), k


def test_checkpoint_model_matches_oracle(tmp_path):
    m = M()
    m.set_precision('fp32')
    spec = O.NerfSpec(layer_dim=64, appearance_count=7)
    ref = O.make_net('nerf', spec, seed=41)
    ck = tmp_path / '100.pt'
    torch.save({'model_state_dict': {'module.' + k: v for k, v in ref.weights[0].items()}}, ck)
    net = m.get_nerf(C.container_hparams(ckpt_path=str(ck)), 7).to(DEV).eval().requires_grad_(False)
    x = C.nerf_rows(spec, 200, 5)
    with torch.inference_mode():
        assert relerr(net(x.to(DEV)), O.nerf_forward(spec, ref.weights[0], x)) <= 1e-5
