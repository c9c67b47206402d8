"""GPU: training with a background (NeRF++) network in one library call (`render_rays_train(..., bg_nerf=...)`:
mn_render_rays_train_bg and its backward) and replayed as one CUDA graph (`GraphedTrainStep(..., bg_nerf=...)`).

The eager call draws render_rays' random stream - the background draws shaped by the number of background rays, read back once -
so for the same seed it returns the stage path's results exactly, and its gradients match the stage path's to its fp32
repeatability or to the tensor-core bounds.  The graph cannot read that count, so it draws fixed-shape blocks, row i for ray i;
through the C ABI such ray-indexed blocks give exactly what their rows at the background rays give as compacted blocks, so the
graph runs the reference's algorithm on other numbers, and it must equal the eager step of the same per-ray draws."""
import dataclasses
import re
from argparse import Namespace

import pytest
import torch

from mega_nerf_b200 import _cabi as K
from oracle import mn_oracle as O
from test_gpu_parity import DEV, M, product_net
from test_gpu_zk_train_tc import compare, grads_of
from test_gpu_zp_fused_bg import fg_far
from test_gpu_zzf_train_graph import photo_loss, train_precision  # noqa: F401  (fixture)
from test_gpu_zzg_train_graph_shapes import IMAGES, assert_same_images, grads_match, images, update_rel_l2

pytestmark = pytest.mark.gpu

CENTER, RADIUS = torch.tensor([0.05, -0.02, 0.03]), torch.tensor([0.8, 0.9, 1.0])
# name -> (kind, spec, grid, rays, coarse, fine, cascade, sh_deg, real-xyz MegaNeRF (train_mega_nerf), cluster_2d, precisions)
SHAPES = {
    'mega8': ('mega', O.NerfSpec(), (2, 4), 48, 32, 32, False, None, True, False, ('fp32', 'tc_f16')),
    'mega8_c2d': ('mega', O.NerfSpec(), (2, 4), 48, 32, 32, False, None, True, True, ('fp32', 'tc_f16')),
    'nerf_q0': ('nerf', O.NerfSpec(appearance_dim=0), None, 48, 32, 32, False, None, False, False, ('fp32', 'tc_f16')),
    'cascade': ('cascade', O.NerfSpec(), None, 40, 32, 32, True, None, False, False, ('fp32', 'tc_f16')),
    'sh2': ('nerf', O.NerfSpec(pos_dir_dim=0, rgb_dim=27), None, 40, 32, 32, False, 2, False, False, ('fp32', 'tc_f16')),
    'npp2048': ('cascade', O.NerfSpec(layer_dim=2048, appearance_count=10), None, 12, 16, 16, True, None, False, False, ('tc_f16',)),
}
CASES = [(n, p) for n, s in SHAPES.items() for p in s[-1]]


def make_case(name):
    """-> (fg oracle net, bg oracle net, rays [N, 8] (far 1e5), image indices or None, hparams)."""
    kind, spec, grid, n, coarse, fine, cascade, sh, real, c2d, _ = SHAPES[name]
    cents = O.grid_centroids(*grid) if grid else None
    n_sub = 0 if cents is None else cents.shape[0]
    net = O.make_net(kind, spec, seed=0, n_sub=n_sub, centroids=cents, cluster_2d=c2d)
    bg = O.make_net(kind, dataclasses.replace(spec, xyz_dim=4), seed=5, n_sub=n_sub, centroids=cents, xyz_real=real, cluster_2d=c2d)
    rays = O.synthetic_rays(n, seed=0, far=1e5).to(DEV)
    idx = O.synthetic_indices(n, spec.appearance_count).to(DEV) if spec.appearance_dim > 0 else None
    opts = O.RenderOpts(coarse_samples=coarse, fine_samples=fine, use_cascade=cascade, perturb=1.0, pos_dir_dim=spec.pos_dir_dim,
                        sh_deg=sh, model_chunk_size=32 * 1024, train_mega_nerf='x' if real else None)
    return net, bg, rays, idx, Namespace(**vars(opts))


def split(rays, how):
    """The rays with about half ('half'), none or all of them reaching the background."""
    r = rays.clone()
    c, rd = CENTER.to(DEV), RADIUS.to(DEV)
    if how == 'half':
        r[::2, 7] = 0.4
    elif how == 'none':
        r[:, 7] = torch.minimum(torch.full_like(r[:, 7], 0.4), fg_far(r, c, rd))
    n_bg = int((r[:, 7] > fg_far(r, c, rd)).sum())
    assert n_bg == {'none': 0, 'all': r.shape[0]}.get(how, n_bg) and (how != 'half' or 0 < n_bg < r.shape[0]), (how, n_bg)
    return r


def trainable(net):
    return product_net(net).requires_grad_(True).train()


def both_grads(pn, pb):
    return grads_of(pn), grads_of(pb)


def fine_loss(res, target, hp):
    """The MSE of rgb_fine alone: a Cascade's rgb_coarse gets no gradient (the one call's backward takes grad_rgb_coarse NULL)."""
    return torch.nn.functional.mse_loss(res['rgb_fine'], target)


def stage_step(pn, pb, rays, idx, hp, target, seed, loss=photo_loss):
    pn.zero_grad(set_to_none=True)
    pb.zero_grad(set_to_none=True)
    torch.manual_seed(seed)
    res, _ = M().render_rays(pn, pb, rays, idx, hp, CENTER.to(DEV), RADIUS.to(DEV), True, True, True)
    loss(res, target, hp).backward()
    return res, both_grads(pn, pb)


def one_call_step(pn, pb, rays, idx, hp, target, seed, loss=photo_loss):
    pn.zero_grad(set_to_none=True)
    pb.zero_grad(set_to_none=True)
    torch.manual_seed(seed)
    res = M().render_rays_train(pn, rays, idx, hp, True, True, bg_nerf=pb, sphere_center=CENTER.to(DEV),
                                sphere_radius=RADIUS.to(DEV), get_bg_fg_rgb=True)
    loss(res, target, hp).backward()
    return res, both_grads(pn, pb)


def assert_grads_like_stage(got, want, again, prec, tag):
    """Gradients of the one call against the stage path: tc_f16 to the tensor-core bounds; fp32 to twice what two stage-path runs
    differ by (fp32 atomics), or 1e-5 of the parameter's scale (the one call sums the coarse and fine queries into one block).  The
    scale is the largest gradient of that parameter in any sub-module, as in grads_match: a sub-module the batch barely reaches
    has gradients at the rounding level of the others."""
    assert set(got) == set(want), (tag, set(got) ^ set(want))
    if prec == 'tc_f16':
        if want:
            compare(got, want, tag)
        return
    strip = lambda k: re.sub(r'^(sub_modules\.\d+\.|coarse\.|fine\.)', '', k)
    scale = {}
    for k, v in want.items():
        scale[strip(k)] = max(scale.get(strip(k), 0.0), float(v.abs().max()))
    for k, ref in want.items():
        rep = float((again[k] - ref).abs().max())
        diff = float((got[k] - ref).abs().max())
        assert diff <= max(2 * rep, 1e-5 * scale[strip(k)]), (tag, k, diff, rep, scale[strip(k)])


@pytest.mark.parametrize('how', ['half', 'none', 'all'])
# 'cascade:fine_loss': the Cascade trained on rgb_fine alone, whose backward skips both networks' coarse passes
@pytest.mark.parametrize('name,prec', CASES + [('cascade:fine_loss', p) for p in SHAPES['cascade'][-1]])
def test_eager_equals_the_stage_path(name, prec, how, train_precision):
    train_precision(prec)
    shape, _, fine_only = name.partition(':')
    loss = fine_loss if fine_only else photo_loss
    net, bg, rays, idx, hp = make_case(shape)
    rays = split(rays, how)
    pn, pb = trainable(net), trainable(bg)
    target = torch.rand(rays.shape[0], 3, generator=torch.Generator().manual_seed(2)).to(DEV)
    res_s, (gs, gsb) = stage_step(pn, pb, rays, idx, hp, target, 7, loss)
    res_o, (go, gob) = one_call_step(pn, pb, rays, idx, hp, target, 7, loss)
    assert pn._native().train_on_tensor_cores() == (prec == 'tc_f16') == pb._native().train_on_tensor_cores()
    assert list(res_o) == list(res_s)
    for k in res_s:
        assert torch.equal(res_o[k], res_s[k]), (name, prec, how, k, float((res_o[k] - res_s[k]).abs().max()))
    if how == 'none':
        assert not gsb and not gob                  # no background ray: no gradient for the background, as on the stage path
    _, (gs2, gsb2) = stage_step(pn, pb, rays, idx, hp, target, 7, loss)
    if fine_only:
        # the stage path gives the coarse networks no gradient, the one call's gradient block an exactly zero one
        for got, want in ((go, gs), (gob, gsb)):
            for k in set(got) - set(want):
                assert not got.pop(k).any(), (name, prec, how, k)
    assert_grads_like_stage(go, gs, gs2, prec, f'{name} {prec} {how} foreground')
    assert_grads_like_stage(gob, gsb, gsb2, prec, f'{name} {prec} {how} background')


@pytest.mark.parametrize('name,prec', [('mega8', 'tc_f16'), ('cascade', 'fp32')])
def test_distributed_batch_without_background_ray(name, prec, train_precision, monkeypatch):
    """'RANK' set, no background ray: the draws of the reference's dummy ray are consumed (the random stream after the call is the
    stage path's), the values are untouched and the background parameters get the dummy ray's zero gradient."""
    train_precision(prec)
    monkeypatch.setenv('RANK', '0')
    net, bg, rays, idx, hp = make_case(name)
    rays = split(rays, 'none')
    pn, pb = trainable(net), trainable(bg)
    target = torch.rand(rays.shape[0], 3, generator=torch.Generator().manual_seed(2)).to(DEV)
    res_s, (gs, gsb) = stage_step(pn, pb, rays, idx, hp, target, 11)
    after_s = torch.rand(4, device=DEV)
    res_o, (go, gob) = one_call_step(pn, pb, rays, idx, hp, target, 11)
    after_o = torch.rand(4, device=DEV)
    assert torch.equal(after_o, after_s)
    assert list(res_o) == list(res_s) and all(torch.equal(res_o[k], res_s[k]) for k in res_s)
    assert set(gob) == set(gsb) and gob and all(float(g.abs().max()) == 0 for g in gob.values())
    _, (gs2, _) = stage_step(pn, pb, rays, idx, hp, target, 11)
    assert_grads_like_stage(go, gs, gs2, prec, f'{name} {prec} RANK')


def per_ray_call(pn, pb, rays, idx, hp, by_ray, draws):
    """One mn_render_rays_train_bg call and its backward with given background draw blocks -> (outputs, fg block, bg block)."""
    from mega_nerf_b200 import autograd as AG
    n, nb = pn._native(), pb._native()
    n.sync(DEV)
    nb.sync(DEV)
    N = rays.shape[0]
    Sc, Sf = hp.coarse_samples, hp.fine_samples
    Sq = Sc + Sf if hp.use_cascade else Sf
    g = torch.Generator().manual_seed(3)
    fg = [torch.rand(N, Sc, generator=g), torch.rand(N * Sc, 1, generator=g), torch.rand(N, Sf, generator=g),
          torch.rand(N * Sq, 1, generator=g)]
    fg = [t.to(DEV) for t in fg]
    sh = hp.sh_deg if (hp.pos_dir_dim == 0 and hp.sh_deg is not None) else -1
    real = hp.train_mega_nerf is not None
    call = AG.RenderTrainBgCall(n, nb, rays, idx, CENTER.to(DEV), RADIUS.to(DEV), real, real and getattr(pn, 'cluster_dim_start', 0) == 1,
                                torch.linspace(0, 1, Sc, device=DEV), torch.linspace(0, 1, Sc // 2, device=DEV), fg[0], draws[0], 1.0,
                                fg[1], draws[1], fg[2], draws[2], fg[3], draws[3], Sc, Sf, bool(hp.use_cascade), sh, by_ray, True,
                                True, True)
    out = call.forward()
    cot = torch.randn(N, 3, generator=torch.Generator().manual_seed(4)).to(DEV)
    cot_c = torch.randn(N, 3, generator=torch.Generator().manual_seed(5)).to(DEV) if hp.use_cascade else None
    gf, gb = call.backward(cot, cot_c, n.param_list(), nb.param_list())
    torch.cuda.synchronize()
    return out, torch.cat([t.reshape(-1) for t in gf]), torch.cat([t.reshape(-1) for t in gb])


@pytest.mark.parametrize('name,prec', [('mega8', 'fp32'), ('mega8_c2d', 'tc_f16'), ('cascade', 'tc_f16'), ('sh2', 'fp32'),
                                       ('nerf_q0', 'tc_f16')])
def test_ray_indexed_draws_are_the_compacted_algorithm(name, prec, train_precision):
    """A call with ray-indexed background draw blocks equals a call with compacted blocks made of those blocks' rows at the
    background rays in ascending order: forward outputs bit for bit; both gradient blocks to the reordering of their fp32 atomic
    sums (the routing's slot order and the gradient atomics depend on scheduling): twice the spread of two compacted calls, or
    1e-5 of the block's largest gradient."""
    train_precision(prec)
    net, bg, rays, idx, hp = make_case(name)
    rays = split(rays, 'half')
    pn, pb = trainable(net), trainable(bg)
    N, Sb, Fb = rays.shape[0], hp.coarse_samples // 2, hp.fine_samples // 2
    Sqb = Sb + Fb if hp.use_cascade else Fb
    g = torch.Generator().manual_seed(8)
    by_ray = [torch.rand(N, Sb, generator=g), torch.rand(N, Sb, generator=g), torch.rand(N, Fb, generator=g),
              torch.rand(N, Sqb, generator=g)]
    by_ray = [t.to(DEV) for t in by_ray]
    ids = torch.nonzero(rays[:, 7] > fg_far(rays, CENTER.to(DEV), RADIUS.to(DEV))).view(-1)
    compacted = [t[ids].contiguous() for t in by_ray]
    a, ga, gba = per_ray_call(pn, pb, rays, idx, hp, False, compacted)
    a2, ga2, gba2 = per_ray_call(pn, pb, rays, idx, hp, False, compacted)
    b, gb, gbb = per_ray_call(pn, pb, rays, idx, hp, True, by_ray)
    assert set(a) == set(b)
    for k in a:
        assert torch.equal(a[k], a2[k]) and torch.equal(b[k], a[k]), (name, prec, k)
    for got, ref, again, tag in ((gb, ga, ga2, 'foreground'), (gbb, gba, gba2, 'background')):
        assert float(ref.abs().max()) > 0, tag
        spread = float((again - ref).abs().max())
        diff = float((got - ref).abs().max())
        assert diff <= max(2 * spread, 1e-5 * float(ref.abs().max())), (name, prec, tag, diff, spread)


def graph_batches(rays, hows, seed):
    """Batches with the given splits: each a permutation of the rays, origins jittered, then split; and target colours."""
    g = torch.Generator().manual_seed(seed)
    out = []
    for how in hows:
        perm = torch.randperm(rays.shape[0], generator=g).to(DEV)
        r = rays[perm].clone()
        r[:, :3] += 0.01 * (torch.rand(rays.shape[0], 3, generator=g).to(DEV) - 0.5)
        out.append((split(r, how), torch.rand(rays.shape[0], 3, generator=g).to(DEV), perm))
    return out


def sel(idx, perm):
    return None if idx is None else idx[perm]


def eager_per_ray_steps(net, bg, data, idx, hp):
    """Adam over the eager per-ray step (the graph's draws, outside a graph) on each batch, seeded as the replays."""
    from mega_nerf_b200.render import _render_train_bg
    pn, pb = trainable(net), trainable(bg)
    opt = torch.optim.Adam(list(pn.parameters()) + list(pb.parameters()), lr=5e-4, capturable=True)
    losses = []
    for k, (r, rgb, perm) in enumerate(data):
        torch.manual_seed(100 + k)
        opt.zero_grad(set_to_none=True)
        n, nb = pn._native(), pb._native()
        n.sync(DEV)
        nb.sync(DEV)
        res = _render_train_bg(pn, n, pb, nb, r, sel(idx, perm), hp, CENTER.to(DEV), RADIUS.to(DEV), False, True, False, by_ray=True)
        loss = photo_loss(res, rgb, hp)
        loss.backward()
        opt.step()
        losses.append(float(loss.detach()))
        if k == 0:
            g1 = both_grads(pn, pb)
    return losses, g1, pn, pb


HOWS = ['half', 'none', 'all', 'half', 'all']


@pytest.mark.parametrize('name,prec', CASES)
def test_graph_equals_eager_per_ray(name, prec, train_precision):
    """Five replays over batches with half, none and all of the rays reaching the background (consecutive batches of different
    counts through one graph) against the eager per-ray step: losses, step-1 gradients of both networks and the parameters after
    five Adam steps, to the bounds of tests/test_gpu_zzg_train_graph_shapes.py (b)."""
    train_precision(prec)
    net, bg, rays, idx, hp = make_case(name)
    fp32 = prec == 'fp32'
    pn, pb = trainable(net), trainable(bg)
    start = [p.detach().clone() for p in list(pn.parameters()) + list(pb.parameters())]
    opt = torch.optim.Adam(list(pn.parameters()) + list(pb.parameters()), lr=5e-4, capturable=True)
    step = M().GraphedTrainStep(pn, hp, rays.shape[0], DEV, opt, bg_nerf=pb, sphere_center=CENTER.to(DEV),
                                sphere_radius=RADIUS.to(DEV))
    data = graph_batches(rays, HOWS, 3)
    loss_g = []
    for k, (r, rgb, perm) in enumerate(data):
        torch.manual_seed(100 + k)
        loss_g.append(float(step.step(r, rgb, sel(idx, perm))[0]))
        if k == 0:
            g_graph = both_grads(pn, pb)
    step.check()
    loss_e, g_eager, qn, qb = eager_per_ray_steps(net, bg, data, idx, hp)
    for a, b in zip(loss_g, loss_e):
        assert abs(a - b) <= (1e-5 if fp32 else 2e-3) * abs(b), (name, prec, loss_g, loss_e)
    for got, want, tag in ((g_graph[0], g_eager[0], 'foreground'), (g_graph[1], g_eager[1], 'background')):
        l2, worst = grads_match(got, want, f'{name} {prec} {tag}')
        print(f'{name} {prec} {tag}: step-1 gradients rel L2 {l2:.2e}, worst {worst}')
        assert l2 <= (1e-4 if fp32 else 1e-2) and worst[1] <= 1e-3, (name, prec, tag, l2, worst)
    # two eager runs bound the update spread (gradient sums reordered by atomics)
    _, _, rn, rb = eager_per_ray_steps(net, bg, data, idx, hp)

    class Both(torch.nn.Module):
        def __init__(self, a, b):
            super().__init__()
            self.a, self.b = a, b

    rel = update_rel_l2(start, Both(pn, pb), Both(qn, qb))
    spread = update_rel_l2(start, Both(rn, rb), Both(qn, qb))
    print(f'{name} {prec}: parameter updates rel L2 {rel:.2e} (eager spread {spread:.2e}); losses {loss_g}')
    assert rel <= max(1e-3 if fp32 else 2e-2, 3 * spread), (rel, spread)


def test_graph_lifecycle(train_precision):
    """No host launch per replay; an in-place load_state_dict on either network reaches the next replay; both networks' weight
    images equal a fresh pack byte for byte after replays; a batch with no background ray gives the background parameters an
    exactly zero gradient and the foreground the eager results."""
    train_precision('tc_f16')
    m = M()
    net, bg, rays, idx, hp = make_case('mega8')
    pn, pb = trainable(net), trainable(bg)
    opt = torch.optim.Adam(list(pn.parameters()) + list(pb.parameters()), lr=5e-4, capturable=True)
    step = m.GraphedTrainStep(pn, hp, rays.shape[0], DEV, opt, bg_nerf=pb, sphere_center=CENTER.to(DEV), sphere_radius=RADIUS.to(DEV))
    data = graph_batches(rays, ['half', 'all', 'none'], 6)
    for k, (r, rgb, perm) in enumerate(data[:2]):
        step.step(r, rgb, sel(idx, perm))
    h = K.ctx(DEV)
    before = K.lib().mn_launch_count(h)
    step.step(*data[0][:2], sel(idx, data[0][2]))
    torch.cuda.synchronize()
    assert K.lib().mn_launch_count(h) == before

    # weight images after replays: what mn_model_set_weights packs from the same values into twins whose transposed images exist
    # (a first recording call on the tensor cores allocates them)
    tf, tb = trainable(net), trainable(bg)
    torch.manual_seed(1)
    m.render_rays_train(tf, rays, idx, hp, False, True, bg_nerf=tb, sphere_center=CENTER.to(DEV),
                        sphere_radius=RADIUS.to(DEV))['rgb_fine'].sum().backward()
    for live, twin, oracle_net in ((pn, tf, net), (pb, tb, bg)):
        live._native().repack(DEV)
        twin.load_state_dict(live.state_dict())
        twin._native().sync(DEV)
        assert_same_images(images(live), images(twin), len(oracle_net.weights), 'after replays')

    # load_state_dict on both networks between replays
    other_f = trainable(dataclasses.replace(net, weights=O.make_net('mega', net.spec, seed=9, n_sub=8).weights))
    other_b = trainable(dataclasses.replace(bg, weights=O.make_net('mega', bg.spec, seed=10, n_sub=8).weights))
    pn.load_state_dict(other_f.state_dict())
    pb.load_state_dict(other_b.state_dict())
    r, rgb, perm = data[0]
    torch.manual_seed(21)
    got = float(step.step(r, rgb, sel(idx, perm))[0])
    from mega_nerf_b200.render import _render_train_bg
    torch.manual_seed(21)
    n, nb = other_f._native(), other_b._native()
    n.sync(DEV)
    nb.sync(DEV)
    res = _render_train_bg(other_f, n, other_b, nb, r, sel(idx, perm), hp, CENTER.to(DEV), RADIUS.to(DEV), False, True, False,
                           by_ray=True)
    want = float(photo_loss(res, rgb, hp).detach())
    assert abs(got - want) <= 1e-6 * abs(want), (got, want)

    # a batch with no background ray: the foreground as eager, the background's gradient exactly zero
    r, rgb, perm = data[2]
    ref_f = trainable(net)
    ref_b = trainable(bg)
    ref_f.load_state_dict(pn.state_dict())
    ref_b.load_state_dict(pb.state_dict())
    torch.manual_seed(33)
    got = float(step.step(r, rgb, sel(idx, perm))[0])
    assert all(float(p.grad.abs().max()) == 0 for p in pb.parameters())
    torch.manual_seed(33)
    n, nb = ref_f._native(), ref_b._native()
    n.sync(DEV)
    nb.sync(DEV)
    res = _render_train_bg(ref_f, n, ref_b, nb, r, sel(idx, perm), hp, CENTER.to(DEV), RADIUS.to(DEV), False, True, False,
                           by_ray=True)
    loss = photo_loss(res, rgb, hp)
    loss.backward()
    assert abs(got - float(loss)) <= 1e-6 * abs(float(loss))
    l2, worst = grads_match(grads_of(pn), grads_of(ref_f), 'no background ray')
    assert l2 <= 1e-2 and worst[1] <= 1e-3, (l2, worst)
    assert all(float(p.grad.abs().max()) == 0 for p in ref_b.parameters())


def test_camera_outside_the_ellipsoid(train_precision):
    """Eager raises the reference's Exception; after a replay, check() raises it, and the next batch's replay trains normally."""
    train_precision('tc_f16')
    m = M()
    net, bg, rays, idx, hp = make_case('nerf_q0')
    rays = split(rays, 'half')
    pn, pb = trainable(net), trainable(bg)
    bad = rays.clone()
    bad[0, :3] = torch.tensor([3.0, 0, 0])
    bad[0, 3:6] = torch.tensor([0.0, 1.0, 0])
    target = torch.rand(rays.shape[0], 3, device=DEV)
    with pytest.raises(Exception, match='bounded by the unit sphere'):
        m.render_rays_train(pn, bad, idx, hp, False, True, bg_nerf=pb, sphere_center=CENTER.to(DEV), sphere_radius=RADIUS.to(DEV))
    opt = torch.optim.Adam(list(pn.parameters()) + list(pb.parameters()), lr=5e-4, capturable=True)
    step = m.GraphedTrainStep(pn, hp, rays.shape[0], DEV, opt, bg_nerf=pb, sphere_center=CENTER.to(DEV), sphere_radius=RADIUS.to(DEV))
    step.step(rays, target, idx)
    step.check()
    step.step(bad, target, idx)
    with pytest.raises(Exception, match='bounded by the unit sphere'):
        step.check()
    ref_f, ref_b = trainable(net), trainable(bg)
    ref_f.load_state_dict(pn.state_dict())
    ref_b.load_state_dict(pb.state_dict())
    torch.manual_seed(5)
    got = float(step.step(rays, target, idx)[0])
    step.check()
    from mega_nerf_b200.render import _render_train_bg
    torch.manual_seed(5)
    n, nb = ref_f._native(), ref_b._native()
    n.sync(DEV)
    nb.sync(DEV)
    want = float(photo_loss(_render_train_bg(ref_f, n, ref_b, nb, rays, idx, hp, CENTER.to(DEV), RADIUS.to(DEV), False, True, False,
                                             by_ray=True), target, hp))
    assert abs(got - want) <= 2e-6 * abs(want), (got, want)


def test_refusals(tmp_path):
    m = M()
    net, bg, rays, idx, hp = make_case('mega8')
    pn, pb = trainable(net), trainable(bg)
    c, r = CENTER.to(DEV), RADIUS.to(DEV)
    n = rays.shape[0]
    adam = lambda: torch.optim.Adam(list(pn.parameters()) + list(pb.parameters()), lr=5e-4, capturable=True)
    with pytest.raises(ValueError):          # no sphere bound
        m.GraphedTrainStep(pn, hp, n, DEV, adam(), bg_nerf=pb, sphere_center=c)
    with pytest.raises(ValueError):
        m.render_rays_train(pn, rays, idx, hp, False, True, bg_nerf=pb, sphere_radius=r)
    _, cbg, _, _, _ = make_case('cascade')
    with pytest.raises(ValueError):          # use_cascade does not match the background network
        m.GraphedTrainStep(pn, hp, n, DEV, adam(), bg_nerf=trainable(cbg), sphere_center=c, sphere_radius=r)
    with pytest.raises(ValueError):
        m.render_rays_train(pn, rays, idx, hp, False, True, bg_nerf=trainable(cbg), sphere_center=c, sphere_radius=r)
    pb._ep = object()                        # what expert_parallel.shard() attaches
    try:
        with pytest.raises(ValueError):
            m.GraphedTrainStep(pn, hp, n, DEV, adam(), bg_nerf=pb, sphere_center=c, sphere_radius=r)
        with pytest.raises(ValueError):
            m.render_rays_train(pn, rays, idx, hp, False, True, bg_nerf=pb, sphere_center=c, sphere_radius=r)
    finally:
        del pb._ep
    import torch.distributed as dist
    dist.init_process_group('gloo', init_method=f'file://{tmp_path / "pg"}', rank=0, world_size=1)
    try:
        ddp = torch.nn.parallel.DistributedDataParallel(pb)
        with pytest.raises(ValueError):
            m.GraphedTrainStep(pn, hp, n, DEV, adam(), bg_nerf=ddp, sphere_center=c, sphere_radius=r)
        with pytest.raises(ValueError):
            m.render_rays_train(pn, rays, idx, hp, False, True, bg_nerf=ddp, sphere_center=c, sphere_radius=r)
    finally:
        dist.destroy_process_group()
