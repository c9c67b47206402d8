"""CPU-only host logic: the model factories and weight ingestion of mega_nerf_b200/modules.py
(mega_nerf/models/model_utils.py:12-69; SURVEY.md §8f-4): constructor parity with the reference's state-dict
layout, checkpoint loading with the `module.` prefix (runner.py:521-536, model_utils.py:45-51), merged
TorchScript containers (scripts/merge_submodules.py:70-77 -> tests/golden/container_v1.pt) and install()."""
import sys

import pytest
import torch

import cases as C
from oracle import mn_oracle as O


def M():
    import mega_nerf_b200 as m
    return m


def test_get_nerf_matches_reference_state_dict_layout():
    m = M()
    for over, spec in ((dict(), O.NerfSpec(layer_dim=64, appearance_count=7)),
                       (dict(pos_dir_dim=0, sh_deg=2), O.NerfSpec(layer_dim=64, appearance_count=7, pos_dir_dim=0, rgb_dim=27)),
                       (dict(affine_appearance=True), O.NerfSpec(layer_dim=64, appearance_count=7, affine_appearance=True)),
                       (dict(appearance_dim=0), O.NerfSpec(layer_dim=64, appearance_dim=0))):
        hp = C.container_hparams(**over)
        torch.manual_seed(3)
        net = m.get_nerf(hp, 7)
        torch.manual_seed(3)
        want = O.init_nerf_weights(spec)          # pinned to the reference constructor (tests/golden/make_golden.py)
        sd = net.state_dict()
        assert set(sd) == set(want)
        for k in want:
            assert torch.equal(sd[k], want[k]), k   # same RNG consumption order as the reference constructor
    bg = m.get_bg_nerf(C.container_hparams(), 7)
    assert bg.xyz_dim == 4 and bg.state_dict()['xyz_encodings.0.0.weight'].shape == (64, 100)
    casc = m.get_nerf(C.container_hparams(use_cascade=True), 7)
    assert isinstance(casc, m.Cascade) and {k.split('.')[0] for k in casc.state_dict()} == {'coarse', 'fine'}


def test_checkpoint_ingestion_strips_ddp_prefix(tmp_path):
    m = M()
    spec = O.NerfSpec(layer_dim=64, appearance_count=7)
    fg = O.make_net('nerf', spec, seed=41)
    bgspec = O.NerfSpec(layer_dim=64, appearance_count=7, xyz_dim=4)
    bg = O.make_net('nerf', bgspec, seed=42)
    ck = tmp_path / '100.pt'
    torch.save({'model_state_dict': {'module.' + k: v for k, v in fg.weights[0].items()},
                'bg_model_state_dict': {'module.' + k: v for k, v in bg.weights[0].items()},
                'iteration': 100}, ck)
    hp = C.container_hparams(ckpt_path=str(ck))
    net, bnet = m.get_nerf(hp, 7), m.get_bg_nerf(hp, 7)
    for got, want in ((net, fg), (bnet, bg)):
        sd = got.state_dict()
        for k, v in want.weights[0].items():
            assert torch.equal(sd[k], v), k


def test_train_mega_nerf_metadata(tmp_path):
    m = M()
    meta = tmp_path / 'params.pt'
    cents = O.grid_centroids(2, 2)
    torch.save({'centroids': cents, 'cluster_2d': True}, meta)
    net = m.get_nerf(C.container_hparams(train_mega_nerf=str(meta)), 7)
    assert isinstance(net, m.MegaNeRF) and len(net.sub_modules) == 4
    assert net.boundary_margin == 1 and net.joint_training and net.cluster_dim_start == 1 and not net.xyz_real
    assert torch.equal(net.centroids, cents)
    assert m.get_bg_nerf(C.container_hparams(train_mega_nerf=str(meta)), 7).xyz_real


def test_container_ingestion():
    """container_v1.pt was written by the reference's own MegaNeRFContainer + torch.jit.script."""
    m = M()
    fg, bg, cents = C.container_nets()
    hp = C.container_hparams(container_path=C.container_path())
    net, bnet = m.get_nerf(hp, 10), m.get_bg_nerf(hp, 10)
    for got, want, real in ((net, fg, False), (bnet, bg, True)):
        assert isinstance(got, m.MegaNeRF) and len(got.sub_modules) == 4
        assert got.xyz_real == real and got.cluster_dim_start == 1 and got.boundary_margin == 1.15
        assert torch.equal(got.centroids, cents)
        for sub, w in zip(got.sub_modules, want.weights):
            sd = sub.state_dict()
            assert set(sd) == set(w)
            for k, v in w.items():
                assert torch.equal(sd[k], v), k
    assert bnet.sub_modules[0].xyz_dim == 4


def test_install_aliases_reference_module_names():
    m = M()
    saved = {k: v for k, v in sys.modules.items() if k == 'mega_nerf' or k.startswith('mega_nerf.')}
    try:
        m.install()
        from mega_nerf.rendering import render_rays
        from mega_nerf.models.model_utils import get_nerf, get_bg_nerf
        from mega_nerf.ray_utils import get_rays, get_ray_directions, get_rays_batch
        from mega_nerf.models.nerf import NeRF
        assert render_rays is m.render_rays and get_nerf is m.get_nerf and get_bg_nerf is m.get_bg_nerf
        assert get_rays is m.get_rays and get_ray_directions is m.get_ray_directions and get_rays_batch is m.get_rays_batch
        assert NeRF is m.NeRF
    finally:
        for k in [k for k in sys.modules if k == 'mega_nerf' or k.startswith('mega_nerf.')]:
            del sys.modules[k]
        sys.modules.update(saved)


def test_param_list_order_is_stable():
    """The autograd binding passes parameters positionally (mega_nerf_b200/autograd.py)."""
    m = M()
    net = m.get_nerf(C.container_hparams(use_cascade=True), 7)
    pl = net._native().param_list()
    assert [i for i, _, _ in pl] == sorted(i for i, _, _ in pl)
    assert len(pl) == len(list(net.parameters()))
    names = [k for i, k, _ in pl if i == 0]
    assert names == sorted(names) and 'xyz_encodings.0.0.weight' in names
    assert not net._native().needs_grad() or torch.is_grad_enabled()
    with torch.no_grad():
        assert not net._native().needs_grad()
    net.requires_grad_(False)
    assert not net._native().needs_grad()
