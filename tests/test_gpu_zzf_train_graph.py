"""GPU: the recording foreground render as one library call (`render_rays_train`: mn_render_rays_train and its backward) and a
whole training step replayed as one CUDA graph (`GraphedTrainStep`).

render_rays_train draws its random numbers with render_rays' calls in render_rays' order, so for the same seed its results must
equal the stage path's exactly, and its gradients must equal them to the stage path's own repeatability (fp32: the gradient
atomics reorder sums from run to run) or to the tensor-core bounds of tests/test_gpu_zk_train_tc.py (tc_f16, whose gradient
scale is chosen from each model call's own result gradients).  The graph must train like the eager one-call step: same losses,
same parameters after five Adam steps, a falling loss over thirty steps, no host launch per replay, and weights loaded between
replays are the ones the next replay trains."""
import dataclasses
from argparse import Namespace

import pytest
import torch
import torch.nn.functional as Fn

import cases as C
from oracle import mn_oracle as O
from test_gpu_parity import DEV, M, product_net
from test_gpu_zk_train_tc import compare, grads_of

pytestmark = pytest.mark.gpu

# name -> (kind, spec, grid, margin, rays, coarse, fine, cascade, sh_deg); c2 and c5 as in tests/cases.py
EXTRA = {
    'cascade256_q1': ('cascade', O.NerfSpec(appearance_dim=0), None, 1.0, 48, 32, 64, True, None),
    'cascade2048': ('cascade', O.NerfSpec(layer_dim=2048, appearance_count=10), None, 1.0, 16, 16, 16, True, None),
}
CASES = [('c2_mega8_blend', 'fp32'), ('c2_mega8_blend', 'tc_f16'), ('cascade256_q1', 'fp32'), ('cascade256_q1', 'tc_f16'),
         ('c5_sh2', 'fp32'), ('c5_sh2', 'tc_f16'), ('c4_mega25_512', 'fp32'), ('c4_mega25_512', 'tc_f16'),
         ('cascade2048', 'tc_f16')]


def make_case(name: str):
    """-> (oracle net, rays [N, 8] and image indices on the device (or None), hparams)."""
    if name not in EXTRA:
        net, _, rays, idx, opts, _, _ = C.render_case(name)
        return net, rays.to(DEV), None if idx is None else idx.to(DEV), Namespace(**vars(opts))
    kind, spec, grid, margin, n, coarse, fine, cascade, sh = EXTRA[name]
    cents = O.grid_centroids(*grid) if grid else None
    net = O.make_net(kind, spec, seed=0, n_sub=0 if cents is None else cents.shape[0], centroids=cents, boundary_margin=margin,
                     cluster_2d=True)
    rays = O.synthetic_rays(n, seed=0, far=0.6)
    idx = O.synthetic_indices(n, spec.appearance_count) if spec.appearance_dim > 0 else None
    opts = O.RenderOpts(coarse_samples=coarse, fine_samples=fine, use_cascade=cascade, perturb=1.0, pos_dir_dim=spec.pos_dir_dim,
                        sh_deg=sh, model_chunk_size=32 * 1024)
    return net, rays.to(DEV), None if idx is None else idx.to(DEV), Namespace(**vars(opts))


@pytest.fixture
def train_precision():
    m = M()
    yield m.set_train_precision
    m.set_train_precision('fp32')


def photo_loss(res, target, hp):
    """The runner's loss (runner.py:366-379): MSE of rgb_fine, averaged with the coarse MSE for a Cascade."""
    loss = Fn.mse_loss(res['rgb_fine'], target)
    if hp.use_cascade:
        loss = (loss + Fn.mse_loss(res['rgb_coarse'], target)) / 2
    return loss


def stage_step(pn, rays, idx, hp, target, seed):
    pn.zero_grad(set_to_none=True)
    torch.manual_seed(seed)
    res, _ = M().render_rays(pn, None, rays, idx, hp, None, None, True, True, False)
    photo_loss(res, target, hp).backward()
    return res, grads_of(pn)


def one_call_step(pn, rays, idx, hp, target, seed):
    pn.zero_grad(set_to_none=True)
    torch.manual_seed(seed)
    res = M().render_rays_train(pn, rays, idx, hp, True, True)
    photo_loss(res, target, hp).backward()
    return res, grads_of(pn)


@pytest.mark.parametrize('name,prec', CASES)
def test_forward_and_gradients_equal_the_stage_path(name, prec, train_precision):
    train_precision(prec)
    net, rays, idx, hp = make_case(name)
    pn = product_net(net).requires_grad_(True).train()
    target = torch.rand(rays.shape[0], 3, generator=torch.Generator().manual_seed(2)).to(DEV)
    res_s, g_s = stage_step(pn, rays, idx, hp, target, 7)
    assert pn._native().train_on_tensor_cores() == (prec == 'tc_f16')
    res_o, g_o = one_call_step(pn, rays, idx, hp, target, 7)
    assert list(res_o) == list(res_s)
    for k in res_s:
        assert torch.equal(res_o[k], res_s[k]), (name, prec, k, float((res_o[k] - res_s[k]).abs().max()))
    assert set(g_o) == set(g_s)
    if prec == 'tc_f16':
        l2, worst = compare(g_o, g_s, f'{name} one call vs stages')
        print(f'{name} tc_f16: gradients rel L2 {l2:.2e}, worst {worst}')
        return
    # fp32: within what two stage-path runs of the same step differ by (fp32 atomics).  The one call accumulates the coarse and
    # the fine query's gradients into one block where the stage path adds two blocks, so the floor is that reordering: 1e-5 of
    # the tensor's scale
    _, g_s2 = stage_step(pn, rays, idx, hp, target, 7)
    for k, ref in g_s.items():
        rep = float((g_s2[k] - ref).abs().max())
        scale = float(ref.abs().max())
        diff = float((g_o[k] - ref).abs().max())
        assert diff <= max(2 * rep, 1e-5 * scale), (name, k, diff, rep, scale)


def batches(rays, n_batches, seed):
    """n_batches batches of the case's rays, each a different permutation with jittered origins, and their target colours."""
    g = torch.Generator().manual_seed(seed)
    out = []
    for _ in range(n_batches):
        perm = torch.randperm(rays.shape[0], generator=g).to(DEV)
        r = rays[perm].clone()
        r[:, :3] += 0.01 * (torch.rand(rays.shape[0], 3, generator=g).to(DEV) - 0.5)
        out.append((r, torch.rand(rays.shape[0], 3, generator=g).to(DEV), perm))
    return out


@pytest.mark.parametrize('prec', ['fp32', 'tc_f16'])
def test_graph_equals_eager_and_trains(prec, train_precision):
    train_precision(prec)
    m = M()
    net, rays, idx, hp = make_case('c2_mega8_blend')
    pg = product_net(net).requires_grad_(True).train()
    pe = product_net(net).requires_grad_(True).train()
    start = [p.detach().clone() for p in pg.parameters()]
    opt_g = torch.optim.Adam(pg.parameters(), lr=5e-4, capturable=True)
    opt_e = torch.optim.Adam(pe.parameters(), lr=5e-4, capturable=True)
    step = m.GraphedTrainStep(pg, hp, rays.shape[0], DEV, opt_g)
    data = batches(rays, 5, 3)
    loss_g, loss_e = [], []
    for k, (r, rgb, perm) in enumerate(data):
        torch.manual_seed(100 + k)
        loss, psnr, dv = step.step(r, rgb, idx[perm])
        loss_g.append(float(loss))
        if k == 0:
            g_graph = grads_of(pg)
        assert torch.isfinite(psnr) and torch.isfinite(dv)
    for k, (r, rgb, perm) in enumerate(data):
        torch.manual_seed(100 + k)
        opt_e.zero_grad(set_to_none=True)
        loss = photo_loss(m.render_rays_train(pe, r, idx[perm], hp, False, True), rgb, hp)
        loss.backward()
        opt_e.step()
        loss_e.append(float(loss))
        if k == 0:
            g_eager = grads_of(pe)
    tol = 1e-5 if prec == 'fp32' else 2e-3
    for a, b in zip(loss_g, loss_e):
        assert abs(a - b) <= tol * abs(b), (prec, loss_g, loss_e)
    # the parameters after 5 steps: the updates agree (Adam's normalisation can turn last-bit gradient differences of
    # near-zero entries into visible update differences, so the bound is on the whole update vector)
    num = den = 0.0
    for p0, a, b in zip(start, pg.parameters(), pe.parameters()):
        num += float((a.detach() - b.detach()).double().square().sum())
        den += float((b.detach() - p0).double().square().sum())
    rel = (num / den) ** 0.5
    print(f'{prec}: graph vs eager losses {loss_g} / {loss_e}; parameter updates rel L2 {rel:.2e}')
    assert rel <= (1e-3 if prec == 'fp32' else 2e-2), rel
    # the first step's gradients, at the same weights (later steps start from weights that the atomics' summation order has
    # already moved apart; test_load_state_dict_between_replays_is_repacked checks the repack at changed weights)
    l2, worst = compare(g_graph, g_eager, f'{prec} graph vs eager, step 1')
    print(f'{prec}: step-1 gradients graph vs eager rel L2 {l2:.2e}, worst {worst}')
    assert l2 <= (1e-4 if prec == 'fp32' else 1e-2), l2

    # 30 more replays on two alternating batches of a fixed target: the loss falls
    two = batches(rays, 2, 4)
    losses = []
    for k in range(30):
        r, rgb, perm = two[k % 2]
        losses.append(float(step.step(r, rgb, idx[perm])[0]))
    assert losses[-1] < 0.9 * losses[1], losses


def test_replay_issues_no_host_launch(train_precision):
    train_precision('tc_f16')
    m = M()
    from mega_nerf_b200 import _cabi as K
    net, rays, idx, hp = make_case('c2_mega8_blend')
    pn = product_net(net).requires_grad_(True).train()
    step = m.GraphedTrainStep(pn, hp, rays.shape[0], DEV, torch.optim.Adam(pn.parameters(), lr=5e-4, capturable=True))
    target = torch.rand(rays.shape[0], 3, device=DEV)
    step.step(rays, target, idx)                 # capture, then the first replay
    h = K.ctx(DEV)
    before = K.lib().mn_launch_count(h)
    step.step(rays, target, idx)
    torch.cuda.synchronize()
    assert K.lib().mn_launch_count(h) == before


@pytest.mark.parametrize('prec', ['fp32', 'tc_f16'])
def test_load_state_dict_between_replays_is_repacked(prec, train_precision):
    train_precision(prec)
    m = M()
    net, rays, idx, hp = make_case('c2_mega8_blend')
    pn = product_net(net).requires_grad_(True).train()
    step = m.GraphedTrainStep(pn, hp, rays.shape[0], DEV, torch.optim.Adam(pn.parameters(), lr=5e-4, capturable=True))
    target = torch.rand(rays.shape[0], 3, generator=torch.Generator().manual_seed(5)).to(DEV)
    for _ in range(2):
        step.step(rays, target, idx)
    other = product_net(dataclasses.replace(net, weights=O.make_net('mega', net.spec, seed=9, n_sub=len(net.weights),
                                                                     centroids=net.centroids, boundary_margin=net.boundary_margin,
                                                                     cluster_2d=True).weights)).requires_grad_(True).train()
    pn.load_state_dict(other.state_dict())       # in place: the parameters keep their storage
    torch.manual_seed(21)
    got = float(step.step(rays, target, idx)[0])
    torch.manual_seed(21)
    loss = photo_loss(m.render_rays_train(other, rays, idx, hp, False, True), target, hp)
    loss.backward()
    want = float(loss)
    assert abs(got - want) <= 1e-6 * abs(want), (got, want)
    # the gradients at the loaded weights: stale images - the forward ones or, on the tensor cores, the transposed ones of the
    # backward - would give the gradients of other weights
    l2, worst = compare(grads_of(pn), grads_of(other), f'{prec} after load_state_dict')
    print(f'{prec}: gradients after load_state_dict, graph vs eager rel L2 {l2:.2e}, worst {worst}')
    assert l2 <= (1e-5 if prec == 'fp32' else 1e-2), l2


@pytest.mark.parametrize('name,prec', [('c2_mega8_blend', 'fp32'), ('c2_mega8_blend', 'tc_f16'), ('cascade256_q1', 'fp32'),
                                       ('c5_sh2', 'tc_f16')])
def test_variance_without_depth_equals_the_stage_path(name, prec, train_precision):
    """get_depth=False, get_depth_variance=True - what the runner and GraphedTrainStep ask for - where the one call computes the
    depth in a scratch buffer."""
    train_precision(prec)
    net, rays, idx, hp = make_case(name)
    pn = product_net(net).requires_grad_(True).train()
    torch.manual_seed(13)
    res_s, _ = M().render_rays(pn, None, rays, idx, hp, None, None, False, True, False)
    torch.manual_seed(13)
    res_o = M().render_rays_train(pn, rays, idx, hp, False, True)
    assert list(res_o) == list(res_s) and 'depth_variance_fine' in res_o and 'depth_fine' not in res_o
    for k in res_s:
        assert torch.equal(res_o[k], res_s[k]), (name, prec, k)


def test_second_graph_and_learning_rate(train_precision):
    """A second graph of the same network (e.g. for a smaller last batch) leaves the first one working; a tensor lr follows its
    scheduler at every replay, a number lr changed after the capture raises."""
    train_precision('tc_f16')
    m = M()
    net, rays, idx, hp = make_case('c2_mega8_blend')
    pn = product_net(net).requires_grad_(True).train()
    opt = torch.optim.Adam(pn.parameters(), lr=torch.tensor(5e-4, device=DEV), capturable=True)
    target = torch.rand(rays.shape[0], 3, generator=torch.Generator().manual_seed(6)).to(DEV)
    a = m.GraphedTrainStep(pn, hp, rays.shape[0], DEV, opt)
    a.step(rays, target, idx)
    b = m.GraphedTrainStep(pn, hp, rays.shape[0] // 2, DEV, opt)
    b.step(rays[::2], target[::2], idx[::2])
    ref = product_net(net).requires_grad_(True).train()
    ref.load_state_dict(pn.state_dict())
    torch.manual_seed(31)
    got = float(a.step(rays, target, idx)[0])
    torch.manual_seed(31)
    want = float(photo_loss(m.render_rays_train(ref, rays, idx, hp, False, True), target, hp))
    assert abs(got - want) <= 2e-6 * abs(want), (got, want)
    # lr 5e-34 through a scheduler: the next replay moves no parameter by more than ~lr
    torch.optim.lr_scheduler.ExponentialLR(opt, gamma=1e-30).step()
    assert float(opt.param_groups[0]['lr']) < 1e-32
    before = [p.detach().clone() for p in pn.parameters()]
    a.step(rays, target, idx)
    assert max(float((p0 - p.detach()).abs().max()) for p0, p in zip(before, pn.parameters())) <= 1e-30
    # a number lr is a constant of the capture
    pf = product_net(net).requires_grad_(True).train()
    optf = torch.optim.Adam(pf.parameters(), lr=5e-4, capturable=True)
    c = m.GraphedTrainStep(pf, hp, rays.shape[0], DEV, optf)
    c.step(rays, target, idx)
    optf.param_groups[0]['lr'] = 2.5e-4
    with pytest.raises(ValueError):
        c.step(rays, target, idx)


def test_refusals(tmp_path):
    m = M()
    net, rays, idx, hp = make_case('c2_mega8_blend')
    pn = product_net(net).requires_grad_(True).train()
    adam = lambda: torch.optim.Adam(pn.parameters(), lr=5e-4, capturable=True)
    n = rays.shape[0]
    with pytest.raises(ValueError):      # a background network
        m.GraphedTrainStep(pn, hp, n, DEV, adam(), bg_nerf=product_net(net).train())
    with pytest.raises(ValueError):      # not capturable
        m.GraphedTrainStep(pn, hp, n, DEV, torch.optim.Adam(pn.parameters(), lr=5e-4))
    with pytest.raises(ValueError):      # a GradScaler
        m.GraphedTrainStep(pn, hp, n, DEV, adam(), scaler=torch.amp.GradScaler('cuda'))
    pn._ep = object()                    # what expert_parallel.shard() attaches
    try:
        with pytest.raises(ValueError):
            m.GraphedTrainStep(pn, hp, n, DEV, adam())
    finally:
        del pn._ep
    import torch.distributed as dist
    dist.init_process_group('gloo', init_method=f'file://{tmp_path / "pg"}', rank=0, world_size=1)
    try:
        ddp = torch.nn.parallel.DistributedDataParallel(pn)
        with pytest.raises(ValueError):
            m.GraphedTrainStep(ddp, hp, n, DEV, torch.optim.Adam(ddp.parameters(), lr=5e-4, capturable=True))
        with pytest.raises(ValueError):  # the one call would bypass DDP's forward and never synchronise the gradients
            m.render_rays_train(ddp, rays, idx, hp, False, True)
    finally:
        dist.destroy_process_group()
