"""GPU: the graphed training step (`GraphedTrainStep`) at every foreground network shape it trains, in each train precision
that trains the shape.

At the start of every replay the graph rebuilds each weight image of the model - the fp32 forward and data-gradient layouts,
the fp16 tensor-core forward images and, on the tensor cores, the transposed images of the data-gradient chain - from the
bound parameters (`mn_model_repack`, one chunked launch over a table of re-layouts recorded by `mn_model_bind_weights`).  An
image or a chunk the table misses keeps the weights of the capture: the graph still replays and the loss still falls, but
the forward or the gradients are those of other weights.  So, per shape:
  (a) the repack is a fresh pack: after a repack from overwritten parameters, and again after three replays, the four images
      read back with `mn_debug_weight_images` equal byte for byte those `mn_model_set_weights` writes from the same values
      into a twin model (every image is zeroed at allocation, so padding compares too);
  (b) the graph trains like the eager one-call step: the losses of five steps, the first step's gradients and the parameter
      update after five Adam steps;
  (c) the first replay against the oracle's fp32 autograd of the same step (same seed and draw order, TF32 off: a float64
      oracle would draw other random numbers): the loss to 2e-3 relative, the gradients to E2E_L2 (fp32) / TC_L2 (tc_f16);
  (d) parameters loaded between replays are the ones the next replay trains: its loss and gradients are the eager ones at
      the loaded weights.
The fp32 kernels refuse layer_dim > 512, and the refusal is asserted; tc_f16 trains the shapes it does not cover on the fp32
kernels, which is asserted too.  Lifecycle: transposed images allocated after a bind make the repack refuse until the
weights are bound again, and a graph whose table a later bind retired keeps replaying what it captured."""
import dataclasses
import re
from argparse import Namespace

import pytest
import torch

import cases as C
from mega_nerf_b200 import _cabi as K
from oracle import mn_oracle as O
from test_gpu_parity import DEV, M, product_net
from test_gpu_zc_backward import E2E_L2, global_rel_l2, sub_modules
from test_gpu_zk_train_tc import TC_L2, grads_of
from test_gpu_zn_train_wide import no_tf32
from test_gpu_zzb_sample_counts import e2e_case
from test_gpu_zzf_train_graph import EXTRA, batches, photo_loss, train_precision  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu

IMAGES = ('packed', 'packed_bwd', 'tc_packed', 'tc_dgrad')     # `which` 0..3 of mn_debug_weight_images


def _nerf(spec, rays=32, coarse=32, fine=32, sh_deg=None):
    net, _, r, idx, opts, _, _ = e2e_case('single', n_rays=rays, spec=dataclasses.replace(spec, appearance_count=10),
                                          coarse=coarse, fine=fine, sh_deg=sh_deg)
    return net, r, idx, opts


def _render_case(name, coarse=32, fine=64):
    net, _, r, idx, opts, _, _ = C.render_case(name)
    return net, r, idx, dataclasses.replace(opts, coarse_samples=coarse, fine_samples=fine)


def _hard_with_empty_sub():
    """c2's 8 x 256 MegaNeRF under hard routing, its last centroid moved far from every sample: sub-module 7 gets no rows."""
    net, r, idx, opts = _render_case('c2_mega8_hard')
    cents = net.centroids.clone()
    cents[-1] = torch.tensor([0.0, 40.0, 40.0])
    return dataclasses.replace(net, centroids=cents), r, idx, opts


def _blend64():
    """64 sub-modules (MN_MAX_SUB) on an 8 x 8 grid, 64 wide, blended routing."""
    spec = O.NerfSpec(layer_dim=64, appearance_count=10)
    net = O.make_net('mega', spec, seed=0, n_sub=64, centroids=O.grid_centroids(8, 8), boundary_margin=1.15, cluster_2d=True)
    rays = O.synthetic_rays(48, seed=0, far=0.6)
    opts = O.RenderOpts(coarse_samples=32, fine_samples=64, perturb=1.0, pos_dir_dim=spec.pos_dir_dim, model_chunk_size=32 * 1024)
    return net, rays, O.synthetic_indices(48, spec.appearance_count), opts


def _cascade(name):
    kind, spec, _, margin, n, coarse, fine, cascade, sh = EXTRA[name]
    net = O.make_net(kind, spec, seed=0, boundary_margin=margin)
    rays = O.synthetic_rays(n, seed=0, far=0.6)
    idx = O.synthetic_indices(n, spec.appearance_count) if spec.appearance_dim > 0 else None
    opts = O.RenderOpts(coarse_samples=coarse, fine_samples=fine, use_cascade=cascade, perturb=1.0, pos_dir_dim=spec.pos_dir_dim,
                        sh_deg=sh, model_chunk_size=32 * 1024)
    return net, rays, idx, opts


SHAPES = {
    # name: (builder, the train precisions that train it)
    'w64': (lambda: _nerf(O.NerfSpec(layer_dim=64)), ('fp32',)),                     # 64 x 64 weights: one 4096-element chunk
    'c2_mega8_hard_empty': (_hard_with_empty_sub, ('fp32', 'tc_f16')),
    'c4_mega25_512': (lambda: _render_case('c4_mega25_512'), ('fp32', 'tc_f16')),       # the 512-wide engine, 25 sub-modules
    'blend64': (_blend64, ('fp32',)),
    'cascade256_q1': (lambda: _cascade('cascade256_q1'), ('fp32', 'tc_f16')),
    'cascade2048': (lambda: _cascade('cascade2048'), ('tc_f16',)),                      # layer engine
    'nerf320': (lambda: _nerf(O.NerfSpec(layer_dim=320)), ('fp32', 'tc_f16')),          # layer engine, padded K / N
    'nerf1000': (lambda: _nerf(O.NerfSpec(layer_dim=1000), rays=16, coarse=16, fine=16), ('tc_f16',)),
    'd12_512': (lambda: _nerf(O.NerfSpec(layer_dim=512, layers=12, skip_layers=(4, 8)), rays=16, coarse=16, fine=32),
                ('fp32', 'tc_f16')),
    'd16_256': (lambda: _nerf(O.NerfSpec(layers=16, skip_layers=(4, 8))), ('fp32', 'tc_f16')),    # layer engine on the tc
    'c5_sh2': (lambda: _render_case('c5_sh2'), ('fp32', 'tc_f16')),
    'sh3': (lambda: _nerf(O.NerfSpec(pos_dir_dim=0, rgb_dim=48), sh_deg=3), ('fp32', 'tc_f16')),
    'sh4': (lambda: _nerf(O.NerfSpec(pos_dir_dim=0, rgb_dim=75), sh_deg=4), ('fp32', 'tc_f16')),
    'affine': (lambda: _nerf(O.NerfSpec(affine_appearance=True)), ('fp32',)),
    'nodir_noapp': (lambda: _nerf(O.NerfSpec(pos_dir_dim=0, appearance_dim=0)), ('fp32',)),     # rgb head reads the trunk
    # the lifecycle tests' shape (its graph at every shape: tests/test_gpu_zzf_train_graph.py)
    'c2_mega8_blend': (lambda: _render_case('c2_mega8_blend'), ()),
}
CASES = [(name, prec) for name, (_, precs) in SHAPES.items() for prec in precs]
FP32_REFUSED = ['cascade2048', 'nerf1000']                      # layer_dim > 512
TC_UNCOVERED = ['w64', 'blend64', 'affine', 'nodir_noapp']      # 64 wide, affine appearance, no dir_a_encoding


def make_case(name):
    """-> (oracle net, rays [N, 8] and image indices on the device (or None), the oracle's RenderOpts, hparams)."""
    net, rays, idx, opts = SHAPES[name][0]()
    return net, rays.to(DEV), None if idx is None else idx.to(DEV), opts, Namespace(**vars(opts))


def sel(idx, perm):
    return None if idx is None else idx[perm]


def reseeded(net, seed):
    """The same network (centroids, routing) with another seed's weights."""
    return dataclasses.replace(net, weights=O.make_net(net.kind, net.spec, seed=seed, n_sub=len(net.weights)).weights)


def trainable(net):
    return product_net(net).requires_grad_(True).train()


def recording_call(pn, rays, idx, hp):
    """One recording render and its backward: on the tensor cores, the first one allocates the transposed images."""
    torch.manual_seed(1)
    M().render_rays_train(pn, rays, idx, hp, False, True)['rgb_fine'].sum().backward()
    pn.zero_grad(set_to_none=True)


def images(pn):
    """The four weight images of pn's native model as bytes (empty where the image is not allocated)."""
    L, h = K.lib(), pn._native().handle
    st = K.stream_of(DEV)
    out = {}
    for which, name in enumerate(IMAGES):
        n = L.mn_debug_weight_images(h, which, None, 0, st)
        buf = torch.empty(n, dtype=torch.uint8, device=DEV)
        if n:
            assert L.mn_debug_weight_images(h, which, K.ptr(buf), n, st) == n, L.mn_last_error(K.ctx(DEV)).decode()
        out[name] = buf
    torch.cuda.synchronize()
    return out


def assert_same_images(got, want, n_sub, tag):
    for name in IMAGES:
        a, b = got[name], want[name]
        assert a.numel() == b.numel(), (tag, name, a.numel(), b.numel())
        if not torch.equal(a, b):
            bad = (a != b).nonzero().view(-1)
            first = int(bad[0])
            raise AssertionError(f'{tag}: {name} differs in {bad.numel()} of {a.numel()} bytes, the first at byte {first} '
                                 f'(sub-module {first // (a.numel() // n_sub)})')


def test_weight_image_hook_sizes(train_precision):
    """The hook's sizes are those of the layouts: n_sub x the per-sub-module images; the transposed images exist only once a
    recording call ran on the tensor cores."""
    train_precision('tc_f16')
    net, rays, idx, _, hp = make_case('c2_mega8_blend')
    pn = trainable(net)
    pn._native().sync(DEV)
    L, h = K.lib(), pn._native().handle
    sizes = [L.mn_debug_weight_images(h, which, None, 0, None) for which in range(4)]
    assert all(s > 0 for s in sizes[:3]) and sizes[3] == 0, sizes
    assert sizes[0] == 8 * pn._native()._offsets()['stride'] * 4       # n_sub x PackedLayout::total floats
    assert L.mn_debug_weight_images(h, 4, None, 0, None) == 0 and L.mn_debug_weight_images(h, -1, None, 0, None) == 0
    recording_call(pn, rays, idx, hp)
    assert L.mn_debug_weight_images(h, 3, None, 0, None) > 0
    # a capped copy writes cap bytes and reports the whole size
    buf = torch.full((sizes[0] + 64,), 7, dtype=torch.uint8, device=DEV)
    assert L.mn_debug_weight_images(h, 0, K.ptr(buf), 64, K.stream_of(DEV)) == sizes[0]
    torch.cuda.synchronize()
    assert torch.equal(buf[:64], images(pn)['packed'][:64]) and bool((buf[64:] == 7).all())


@pytest.mark.parametrize('name,prec', CASES)
def test_repack_is_a_fresh_pack(name, prec, train_precision):
    train_precision(prec)
    net, rays, idx, _, hp = make_case(name)
    a, b = trainable(net), trainable(net)
    for pn in (a, b):
        recording_call(pn, rays, idx, hp)
    on_tc = a._native().train_on_tensor_cores()
    assert on_tc == (prec == 'tc_f16')
    n_sub = len(net.weights)
    a._native().bind(DEV)
    before = images(a)
    assert (before['tc_dgrad'].numel() > 0) == on_tc and before['packed'].numel() > 0
    other = trainable(reseeded(net, 9))
    a.load_state_dict(other.state_dict())        # in place: the bound tensors keep their storage
    a._native().repack(DEV)
    b.load_state_dict(other.state_dict())
    b._native().sync(DEV)
    got = images(a)
    for k in IMAGES:                              # every allocated image changed with the weights
        assert got[k].numel() == 0 or not torch.equal(got[k], before[k]), (name, prec, k)
    assert_same_images(got, images(b), n_sub, f'{name} [{prec}] repack after an in-place overwrite')

    # three replays train the bound parameters; a repack then packs what they hold
    step = M().GraphedTrainStep(a, hp, rays.shape[0], DEV, torch.optim.Adam(a.parameters(), lr=5e-4, capturable=True))
    for k, (r, rgb, perm) in enumerate(batches(rays, 3, 4)):
        torch.manual_seed(40 + k)
        step.step(r, rgb, sel(idx, perm))
    assert any(not torch.equal(p, q) for p, q in zip(a.parameters(), other.parameters()))
    a._native().repack(DEV)
    b.load_state_dict(a.state_dict())
    b._native().sync(DEV)
    assert_same_images(images(a), images(b), n_sub, f'{name} [{prec}] repack after three replays')


def grads_match(got, want, tag):
    """Gradients of the same step from two paths -> (whole-vector relative L2, (worst tensor, its largest error over the largest
    gradient of that parameter in any sub-module)).  The per-tensor scale is the parameter's, not the tensor's own: a
    sub-module that only a few low-weight samples reach has gradients at the rounding level of the others, where an own-scale
    relative error measures the order of the gradient sums rather than the weights the step read."""
    assert set(got) == set(want), (tag, set(got) ^ set(want))
    strip = lambda k: re.sub(r'^(sub_modules\.\d+\.|coarse\.|fine\.)', '', k)
    scale = {}
    for k, v in want.items():
        scale[strip(k)] = max(scale.get(strip(k), 0.0), float(v.abs().max()))
    num = den = 0.0
    worst = ('', 0.0)
    for k, ref in want.items():
        assert torch.isfinite(got[k]).all(), (tag, k)
        num += float((got[k].double() - ref.double()).square().sum())
        den += float(ref.double().square().sum())
        e = float((got[k] - ref).abs().max()) / max(scale[strip(k)], 1e-30)
        if e > worst[1]:
            worst = (k, e)
    l2 = (num / max(den, 1e-300)) ** 0.5
    return l2, worst


def eager_steps(net, data, idx, hp):
    """Adam over the eager one-call step on each batch, seeded as the graph's replays -> (losses, step-1 gradients, module)."""
    pe = trainable(net)
    opt = torch.optim.Adam(pe.parameters(), lr=5e-4, capturable=True)
    losses = []
    for k, (r, rgb, perm) in enumerate(data):
        torch.manual_seed(100 + k)
        opt.zero_grad(set_to_none=True)
        loss = photo_loss(M().render_rays_train(pe, r, sel(idx, perm), hp, False, True), rgb, hp)
        loss.backward()
        opt.step()
        losses.append(float(loss.detach()))
        if k == 0:
            g1 = grads_of(pe)
    return losses, g1, pe


def update_rel_l2(start, pa, pb):
    """|pa - pb| / |pb - start| over all parameters: how far two training runs from `start` ended apart."""
    num = den = 0.0
    for p0, a, b in zip(start, pa.parameters(), pb.parameters()):
        num += float((a.detach() - b.detach()).double().square().sum())
        den += float((b.detach() - p0).double().square().sum())
    return (num / den) ** 0.5


@pytest.mark.parametrize('name,prec', CASES)
def test_graph_step_equals_eager_and_oracle(name, prec, train_precision):
    train_precision(prec)
    m = M()
    net, rays, idx, opts, hp = make_case(name)
    fp32 = prec == 'fp32'
    pg = trainable(net)
    start = [p.detach().clone() for p in pg.parameters()]
    step = m.GraphedTrainStep(pg, hp, rays.shape[0], DEV, torch.optim.Adam(pg.parameters(), lr=5e-4, capturable=True))
    data = batches(rays, 5, 3)
    loss_g = []
    for k, (r, rgb, perm) in enumerate(data):
        torch.manual_seed(100 + k)
        loss_g.append(float(step.step(r, rgb, sel(idx, perm))[0]))
        if k > 0:
            continue
        assert pg._native().train_on_tensor_cores() == (not fp32)
        g_graph = grads_of(pg)
        if name == 'c2_mega8_hard_empty':         # the edge is there: no row reached sub-module 7
            assert all(p.grad is None or float(p.grad.abs().max()) == 0 for p in sub_modules(pg, net)[7].parameters())
        # (c) the first replay against the oracle's fp32 autograd of the same step
        torch.manual_seed(100)
        with no_tf32():
            n2 = O._leaf_copy(O.net_to(dataclasses.replace(net, training=True), DEV))
            ores, _ = O.render_rays(n2, None, r, sel(idx, perm), opts, None, None, False, True, False)
            oloss = photo_loss(ores, rgb, hp)
            oloss.backward()
        oloss = float(oloss.detach())
        c_loss = abs(loss_g[0] - oloss) / abs(oloss)
        c_l2 = global_rel_l2(pg, net, [{key: v.cpu() for key, v in g.items()} for g in O._collect_grads(n2)])

    # (b) the eager one-call step on the same batches and seeds, twice: Adam's normalisation turns last-bit gradient differences
    # of near-zero entries (the order of the gradient sums) into visible update differences, so the bound on the update after
    # five steps is the larger of a fixed one and three times what two eager runs differ by
    loss_e, g_eager, pe = eager_steps(net, data, idx, hp)
    _, _, pe2 = eager_steps(net, data, idx, hp)
    b_loss = max(abs(a - b) / abs(b) for a, b in zip(loss_g, loss_e))
    b_l2, b_worst = grads_match(g_graph, g_eager, f'{name} [{prec}] graph vs eager, step 1')
    b_upd, rep_upd = update_rel_l2(start, pg, pe), update_rel_l2(start, pe2, pe)

    # (d) weights loaded between replays are the ones the next replay trains
    other = trainable(reseeded(net, 9))
    pg.load_state_dict(other.state_dict())
    r, rgb, perm = data[0]
    torch.manual_seed(21)
    got = float(step.step(r, rgb, sel(idx, perm))[0])
    torch.manual_seed(21)
    loss = photo_loss(m.render_rays_train(other, r, sel(idx, perm), hp, False, True), rgb, hp)
    loss.backward()
    want = float(loss.detach())
    d_loss = abs(got - want) / abs(want)
    d_l2, d_worst = grads_match(grads_of(pg), grads_of(other), f'{name} [{prec}] after load_state_dict')

    print(f'{name} [{prec}]: (b) losses rel {b_loss:.2e}, step-1 gradients rel L2 {b_l2:.2e} (worst tensor {b_worst[1]:.1e}), 5-step update rel L2 {b_upd:.2e} '
          f'(eager vs eager {rep_upd:.2e}); '
          f'(c) loss rel {c_loss:.2e}, gradients rel L2 {c_l2:.2e}; (d) loss rel {d_loss:.2e}, gradients rel L2 {d_l2:.2e} (worst tensor {d_worst[1]:.1e})')
    assert b_loss <= (1e-5 if fp32 else 2e-3), (loss_g, loss_e)
    assert b_l2 <= (1e-4 if fp32 else 1e-2) and b_worst[1] <= 1e-3, (b_l2, b_worst)
    assert b_upd <= max(1e-3 if fp32 else 2e-2, 3 * rep_upd), (b_upd, rep_upd)
    assert c_loss <= 2e-3, (loss_g[0], oloss)
    assert c_l2 <= (E2E_L2 if fp32 else TC_L2), c_l2
    assert d_loss <= 1e-6, d_loss
    assert d_l2 <= (1e-5 if fp32 else 1e-2) and d_worst[1] <= 1e-3, (d_l2, d_worst)


@pytest.mark.parametrize('name', FP32_REFUSED)
def test_fp32_refuses_the_wide_networks(name, train_precision):
    """The fp32 training kernels take layer_dim 64..512: the graphed step of a wider network in fp32 raises their message."""
    train_precision('fp32')
    net, rays, idx, _, hp = make_case(name)
    pn = trainable(net)
    step = M().GraphedTrainStep(pn, hp, rays.shape[0], DEV, torch.optim.Adam(pn.parameters(), lr=5e-4, capturable=True))
    with pytest.raises(RuntimeError, match=r'layer_dim in \{64,...,512\}'):
        step.step(rays, torch.rand(rays.shape[0], 3, device=DEV), idx)


@pytest.mark.parametrize('name', TC_UNCOVERED)
def test_tc_f16_trains_uncovered_shapes_on_the_fp32_kernels(name, train_precision):
    """64-wide networks, affine appearance and heads without dir_a_encoding stay outside tensor-core training: under tc_f16
    their recording calls run the fp32 kernels and allocate no transposed images, so their graphs are the fp32 graphs above."""
    train_precision('tc_f16')
    net, rays, idx, _, hp = make_case(name)
    pn = trainable(net)
    recording_call(pn, rays, idx, hp)
    assert not pn._native().train_on_tensor_cores()
    assert images(pn)['tc_dgrad'].numel() == 0


@pytest.mark.parametrize('name', ['c2_mega8_blend', 'nerf320'])
def test_repack_refuses_images_allocated_after_the_bind(name, train_precision):
    """Bound in fp32, then a first tc_f16 recording call allocates the transposed images: the repack would leave them with
    the old weights, so it refuses until the weights are bound again, and then packs all four images afresh."""
    train_precision('fp32')
    net, rays, idx, _, hp = make_case(name)
    a, b = trainable(net), trainable(net)
    recording_call(a, rays, idx, hp)
    a._native().bind(DEV)
    a._native().repack(DEV)
    assert images(a)['tc_dgrad'].numel() == 0
    train_precision('tc_f16')
    for pn in (a, b):
        recording_call(pn, rays, idx, hp)
    assert a._native().train_on_tensor_cores()
    with pytest.raises(RuntimeError, match='bind again'):
        a._native().repack(DEV)
    a._native().bind(DEV)
    other = trainable(reseeded(net, 9))
    a.load_state_dict(other.state_dict())
    a._native().repack(DEV)
    b.load_state_dict(other.state_dict())
    b._native().sync(DEV)
    got = images(a)
    assert got['tc_dgrad'].numel() > 0
    assert_same_images(got, images(b), len(net.weights), f'{name} repack after binding again')


@pytest.mark.parametrize('name', ['c2_mega8_blend', 'nerf320'])
def test_graphs_with_different_repack_tables(name, train_precision):
    """An fp32 graph, then a tc_f16 graph of the same network: the second bind covers the transposed images, so it builds a
    new table and retires the first graph's.  Alternating replays each equal their eager step: the retired table still serves
    the fp32 graph."""
    m = M()
    net, rays, idx, _, hp = make_case(name)
    pn = trainable(net)
    adam = lambda: torch.optim.Adam(pn.parameters(), lr=5e-4, capturable=True)
    data = batches(rays, 2, 5)
    r, rgb, perm = data[0]
    train_precision('fp32')
    g32 = m.GraphedTrainStep(pn, hp, rays.shape[0], DEV, adam())
    g32.step(r, rgb, sel(idx, perm))
    assert images(pn)['tc_dgrad'].numel() == 0    # the fp32 graph's table has no transposed images to cover
    train_precision('tc_f16')
    g16 = m.GraphedTrainStep(pn, hp, rays.shape[0], DEV, adam())
    g16.step(r, rgb, sel(idx, perm))
    assert pn._native().train_on_tensor_cores()
    for k in range(4):
        prec, step = (('fp32', g32), ('tc_f16', g16))[k % 2]
        r, rgb, perm = data[k // 2]
        ref = trainable(net)
        ref.load_state_dict(pn.state_dict())
        train_precision(prec)
        torch.manual_seed(60 + k)
        got = float(step.step(r, rgb, sel(idx, perm))[0])
        torch.manual_seed(60 + k)
        loss = photo_loss(m.render_rays_train(ref, r, sel(idx, perm), hp, False, True), rgb, hp)
        loss.backward()
        want = float(loss.detach())
        assert abs(got - want) <= 2e-6 * abs(want), (name, k, prec, got, want)
        if prec == 'tc_f16':     # the fp32 graph's gradients live in its own tensors: pn.grad is the tc_f16 graph's
            l2, worst = grads_match(grads_of(pn), grads_of(ref), f'{name} replay {k} [{prec}]')
            assert l2 <= 1e-2 and worst[1] <= 1e-3, (name, k, l2, worst)
