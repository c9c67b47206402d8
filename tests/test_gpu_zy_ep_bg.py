"""GPU: the background (NeRF++) network under expert parallelism (mega_nerf_b200/expert_parallel.py, render.py): the dispatch
of a capacity above the row count and of no rows, render_rays in a process group of one rank (eval against the torch path and
the non-EP render, a chunk with no background ray, training against the non-EP step, Adam, full_state_dict), several ranks
played as threads on one device through a fake process group - one of them with no background ray - and the refusal of the
one-call paths."""
import dataclasses
import os
import threading
from argparse import Namespace

import pytest
import torch
import torch.distributed as dist

import cases as C
from test_gpu_parity import DEV, M, product_net, relerr
from test_gpu_zk_train_tc import TC_L2
from test_gpu_zp_fused_bg import no_bg
from test_gpu_zv_ep_device import EP, inputs, pair_slots
from test_gpu_zx_ep_train import FP32_L2, grads_of, rel_l2

pytestmark = pytest.mark.gpu

FLAGS = (True, True, True)          # get_depth, get_depth_variance, get_bg_fg_rgb: every key, fg_* / bg_* included


@pytest.fixture(scope='module')
def one_rank_group():
    if dist.is_initialized():
        yield None
        return
    os.environ.setdefault('MASTER_ADDR', '127.0.0.1')
    os.environ['MASTER_PORT'] = '29677'
    dist.init_process_group('nccl', rank=0, world_size=1, device_id=DEV)
    yield None
    dist.destroy_process_group()


@pytest.fixture()
def train_precision():
    yield M().set_train_precision
    M().set_train_precision('fp32')


def bg_case(hard=False):
    """bg_mega_real (foreground and real-xyz background MegaNeRFs, margin 1.15) or its hard-routed variant."""
    net, bg_net, rays, idx, opts, c, rd = C.render_case('bg_mega_real')
    if hard:
        net = dataclasses.replace(net, boundary_margin=1.0)
        bg_net = dataclasses.replace(bg_net, boundary_margin=1.0)
    return net, bg_net, rays.to(DEV), idx.to(DEV), Namespace(**vars(opts)), c.to(DEV), rd.to(DEV)


def render(m, pn, pb, r, i, hp, c, rd, flags=FLAGS):
    with torch.no_grad():
        return m.render_rays(pn, pb, r, i, hp, c, rd, *flags)[0]


def bg_rays(r, c, rd):
    from test_gpu_zp_fused_bg import bg_count
    return bg_count(r, c, rd)


# ---- 1. dispatch ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('noise', [False, True])
@pytest.mark.parametrize('world', [1, 3])
@pytest.mark.parametrize('mname', ['hard3d_bgreal', 'blend2d'])
def test_dispatch_of_no_rows_sends_empty_segments(one_rank_group, mname, world, noise):
    net, x, nz = inputs(mname, n=700, noise=noise)
    pn = product_net(net)
    ep = EP().ExpertParallel(pn)
    with torch.no_grad():
        full = ep.dispatch(x, nz, world)
        d = ep.dispatch(x[:0], nz[:0] if noise else None, world, rows_cap=700)
    assert d.cap == full.cap > 0
    assert d.send.shape == (world * d.cap, d.c_in + 1 + int(noise))
    assert bool((d.send[:, d.c_in] == -1).all())
    assert bool((d.pair_row == -1).all())
    assert int(d.counts.abs().sum()) == 0
    if d.pair_w is not None:
        assert bool((d.pair_w == 0).all())
    assert d.row_slots.numel() == 0


@pytest.mark.parametrize('noise', [False, True])
@pytest.mark.parametrize('world', [1, 2, 3])
@pytest.mark.parametrize('mname', ['hard3d_bgreal', 'blend2d', 'blend25'])
def test_dispatch_capacity_above_row_count(one_rank_group, mname, world, noise):
    n, n_cap = 3000, 4100
    net, x, nz = inputs(mname, n=n, noise=noise)
    pn = product_net(net)
    ep = EP().ExpertParallel(pn)
    with torch.no_grad():
        a = ep.dispatch(x, nz, world)
        b = ep.dispatch(x, nz, world, rows_cap=n_cap)
        with pytest.raises(ValueError, match='rows_cap'):
            ep.dispatch(x, nz, world, rows_cap=n - 1)
    assert b.cap == a.cap // n * n_cap
    assert torch.equal(a.counts, b.counts)
    per = a.counts.long().sum(1)
    sa, sb = pair_slots(a, per), pair_slots(b, per)
    assert torch.equal(a.send[sa], b.send[sb])
    assert torch.equal(a.pair_row[sa], b.pair_row[sb])
    if a.pair_w is not None:
        assert torch.equal(a.pair_w[sa], b.pair_w[sb])
    pad = torch.ones(world * b.cap, dtype=torch.bool, device=DEV)
    pad[sb] = False
    assert bool((b.send[pad, b.c_in] == -1).all()) and bool((b.pair_row[pad] == -1).all())
    # the combine's slots move to the larger stride
    rs = a.row_slots.long()
    want = torch.where(rs >= 0, rs // a.cap * b.cap + rs % a.cap, rs)
    assert torch.equal(b.row_slots.long(), want)


# ---- 2. eval in a one-rank group -----------------------------------------------------------------------------------------
def enable(nets, **kw):
    return [EP().enable(x, **kw) for x in nets]


def disable(nets):
    for x in nets:
        EP().disable(x)


@pytest.mark.parametrize('prec', ['fp32', 'tc_f16'])
@pytest.mark.parametrize('which', ['both', 'bg'])
@pytest.mark.parametrize('hard', [False, True])
def test_render_eval_one_rank(one_rank_group, hard, which, prec):
    m = M()
    m.set_precision(prec)
    net, bg_net, r, i, hp, c, rd = bg_case(hard)
    pn, pb = product_net(net), product_net(bg_net)
    assert 0 < bg_rays(r, c, rd) < r.shape[0]
    plain = render(m, pn, pb, r, i, hp, c, rd)
    nets = [pb] + ([pn] if which == 'both' else [])
    for x in nets:
        EP().enable(x, sub_fn=lambda k, rows, nz, x=x: x.sub_modules[k](rows, sigma_noise=nz))
    try:
        torch_path = render(m, pn, pb, r, i, hp, c, rd)
    finally:
        disable(nets)
    eps = enable(nets)
    try:
        got = render(m, pn, pb, r, i, hp, c, rd)
    finally:
        disable(nets)
    assert all(e.last_pairs == e.last_owned > 0 for e in eps)
    assert set(got) == set(plain) == set(torch_path)
    assert any(k.startswith('bg_') for k in got) and any(k.startswith('fg_') for k in got)
    for k in plain:
        assert torch.equal(got[k], torch_path[k]), k
        assert relerr(got[k], plain[k]) <= (5e-5 if 'variance' in k else 1e-5), k


def test_render_eval_chunk_without_background(one_rank_group):
    m = M()
    m.set_precision('tc_f16')
    net, bg_net, r, i, hp, c, rd = bg_case()
    pn, pb = product_net(net), product_net(bg_net)
    r = no_bg(r, c, rd)
    assert bg_rays(r, c, rd) == 0
    plain = render(m, pn, pb, r, i, hp, c, rd)
    fg_ep, bg_ep = enable([pn, pb])
    try:
        got = render(m, pn, pb, r, i, hp, c, rd)
    finally:
        disable([pn, pb])
    assert bg_ep.last_pairs == 0 and fg_ep.last_pairs > 0        # no rank has a background ray: the pass is skipped
    assert set(got) == set(plain)
    for k in plain:
        assert relerr(got[k], plain[k]) <= (5e-5 if 'variance' in k else 1e-5), k


# ---- 3. training in a one-rank group -------------------------------------------------------------------------------------
def train_nets(net, bg_net):
    return product_net(net).requires_grad_(True).train(), product_net(bg_net).requires_grad_(True).train()


def loss_of(m, pn, pb, r, i, hp, c, rd, target):
    res, _ = m.render_rays(pn, pb, r, i, hp, c, rd, False, False, False)
    return torch.nn.functional.mse_loss(res['rgb_fine'], target)


def both_grads(pn, pb):
    return {**{f'fg.{k}': v for k, v in grads_of(pn).items()}, **{f'bg.{k}': v for k, v in grads_of(pb).items()}}


def train_step(m, pn, pb, r, i, hp, c, rd, target, seed):
    pn.zero_grad(set_to_none=True)
    pb.zero_grad(set_to_none=True)
    torch.manual_seed(seed)
    loss = loss_of(m, pn, pb, r, i, hp, c, rd, target)
    loss.backward()
    return float(loss.detach()), both_grads(pn, pb)


@pytest.mark.parametrize('prec,which,hard', [('fp32', 'both', False), ('fp32', 'bg', False), ('fp32', 'both', True),
                                             ('tc_f16', 'both', False), ('tc_f16', 'bg', True)])
def test_render_training_step_one_rank(one_rank_group, train_precision, prec, which, hard):
    m = M()
    train_precision(prec)
    net, bg_net, r, i, hp, c, rd = bg_case(hard)
    target = torch.rand(r.shape[0], 3, generator=torch.Generator().manual_seed(2)).to(DEV)
    pn, pb = train_nets(net, bg_net)
    l_plain, g_plain = train_step(m, pn, pb, r, i, hp, c, rd, target, 11)
    assert any(k.startswith('bg.') for k in g_plain)
    nets = [pb] + ([pn] if which == 'both' else [])
    eps = enable(nets)
    try:
        l_ep, g_ep = train_step(m, pn, pb, r, i, hp, c, rd, target, 11)
    finally:
        disable(nets)
    assert all(e.last_pairs == e.last_owned > 0 for e in eps)
    assert abs(l_ep - l_plain) <= (1e-5 if prec == 'fp32' else 2e-3) * abs(l_plain), (l_ep, l_plain)
    l2 = rel_l2(g_ep, g_plain)
    print(f'render_rays step with the background under EP [{prec} {which} hard={hard}]: loss {l_ep:.6f} vs {l_plain:.6f}, '
          f'grads rel L2 {l2:.2e}')
    assert l2 <= (FP32_L2 if prec == 'fp32' else TC_L2), l2


def test_adam_steps_and_full_state_dict(one_rank_group, train_precision):
    m = M()
    train_precision('tc_f16')
    net, bg_net, r, i, hp, c, rd = bg_case()
    target = torch.rand(r.shape[0], 3, generator=torch.Generator().manual_seed(2)).to(DEV)
    pn, pb = train_nets(net, bg_net)
    fg_ep, bg_ep = enable([pn, pb])
    try:
        opt = torch.optim.Adam(list(pn.parameters()) + list(pb.parameters()), lr=5e-4)
        losses = []
        for it in range(30):
            opt.zero_grad(set_to_none=True)
            loss = loss_of(m, pn, pb, r, i, hp, c, rd, target)
            loss.backward()
            opt.step()
            losses.append(float(loss.detach()))
        assert losses[-1] < 0.9 * losses[0], losses
        full, want = bg_ep.full_state_dict(), pb.state_dict()
        assert set(full) == set(want)
        for k in want:
            assert torch.equal(full[k], want[k]), k
    finally:
        disable([pn, pb])


# ---- 4. several ranks on one device --------------------------------------------------------------------------------------
class Ranks:
    """`world` ranks as threads on one device, exactly one running at a time: the running rank hands over only at a
    collective or when it returns, and every rank's CPU and CUDA random state is saved and restored at each switch.  A
    collective completes when every rank has entered it; all must enter it with the same tag.  A rank that waits longer
    than TIMEOUT seconds, or a collective that some rank never enters, fails the run instead of hanging it."""
    TIMEOUT = 300

    def __init__(self, world):
        self.world = world
        self.cv = threading.Condition()
        self.turn = 0
        self.done = [False] * world
        self.local = threading.local()
        self.entered, self.results = {}, {}
        self.error = None
        self.log = [[] for _ in range(world)]

    @property
    def rank(self):
        return self.local.rank

    def _wait(self, r):
        if not self.cv.wait_for(lambda: self.turn == r or self.error is not None, timeout=self.TIMEOUT):
            self.error = TimeoutError(f'rank {r} waited {self.TIMEOUT} s for its turn')
            self.cv.notify_all()
        if self.error is not None:
            raise RuntimeError(f'rank {r} stops: {self.error}')

    def _hand_over(self, r):
        for j in range(1, self.world + 1):
            nxt = (r + j) % self.world
            if not self.done[nxt]:
                self.turn = nxt
                break
        self.cv.notify_all()

    def collective(self, tag, value, fn):
        """Enter collective number n of this rank with `value`; fn(values of every rank) -> one result per rank."""
        r = self.rank
        n = self.local.seq
        self.local.seq += 1
        self.log[r].append(tag)
        with self.cv:
            self.entered.setdefault(n, {})[r] = (tag, value)
            if len(self.entered[n]) == self.world:
                tags = {t for t, _ in self.entered[n].values()}
                if len(tags) != 1:
                    self.error = AssertionError(f'collective {n} entered with different tags {tags}')
                    self.cv.notify_all()
                    raise self.error
                self.results[n] = fn([self.entered[n][o][1] for o in range(self.world)])
            state = (torch.get_rng_state(), torch.cuda.get_rng_state(DEV))
            self._hand_over(r)
            self._wait(r)
            torch.set_rng_state(state[0])
            torch.cuda.set_rng_state(state[1], DEV)
            if n not in self.results:
                self.error = AssertionError(f'rank {r} is in collective {n}, which another rank never entered')
                self.cv.notify_all()
                raise self.error
            return self.results[n][r]

    def run(self, fns, seeds):
        """fns[r]() on rank r after torch.manual_seed(seeds[r]) -> the list of their results."""
        out, errs = [None] * self.world, []

        def body(r):
            self.local.rank, self.local.seq = r, 0
            try:
                with self.cv:
                    self._wait(r)
                torch.manual_seed(seeds[r])
                out[r] = fns[r]()
            except BaseException as e:          # noqa: B902 - re-raised in the main thread
                errs.append(e)
                with self.cv:
                    self.error = self.error or e
            finally:
                with self.cv:
                    self.done[r] = True
                    self._hand_over(r)

        threads = [threading.Thread(target=body, args=(r,)) for r in range(self.world)]
        for t in threads:
            t.start()
        for t in threads:
            t.join(self.TIMEOUT * 2)
        assert not any(t.is_alive() for t in threads), 'a rank did not finish'
        if errs:
            raise errs[0]
        return out


class FakeDist:
    """The part of torch.distributed that expert_parallel uses, over the threads of `Ranks`; the group argument is a name."""
    ReduceOp = dist.ReduceOp

    def __init__(self, ranks):
        self.ranks = ranks

    def get_world_size(self, group=None):
        return self.ranks.world

    def get_rank(self, group=None):
        return self.ranks.rank

    def all_to_all_single(self, output, input, output_split_sizes=None, input_split_sizes=None, group=None):
        assert output_split_sizes is None and input_split_sizes is None
        w = self.ranks.world

        def fn(xs):
            c = xs[0].shape[0] // w
            return [torch.cat([x[r * c:(r + 1) * c] for x in xs]) for r in range(w)]
        output.copy_(self.ranks.collective((group, 'all_to_all', tuple(input.shape)), input.clone(), fn))

    def all_reduce(self, t, op=None, group=None):
        assert op == dist.ReduceOp.MAX
        t.copy_(self.ranks.collective((group, 'all_reduce_max'), t.clone(),
                                      lambda xs: [torch.stack(xs).amax(0)] * len(xs)))


def fake_all_to_all(ranks):
    """_AllToAll over the threads: the exchange is slices and a concatenation, so autograd carries the reverse exchange."""

    class Fake:
        @staticmethod
        def apply(x, group):
            w = ranks.world

            def fn(xs):
                c = xs[0].shape[0] // w
                return [torch.cat([y[r * c:(r + 1) * c] for y in xs]) for r in range(w)]
            return ranks.collective((group, 'results', tuple(x.shape)), x, fn)
    return Fake


def tagging_all_to_all(ranks, bwd_log):
    """_AllToAll that exchanges nothing: it records (network, pass) and returns zeros, and so does its backward."""

    class Zero(torch.autograd.Function):
        @staticmethod
        def forward(ctx, x, tag, log):
            ctx.tag, ctx.log = tag, log
            return torch.zeros_like(x)

        @staticmethod
        def backward(ctx, g):
            ctx.log.append(ctx.tag)
            return torch.zeros_like(g), None, None

    class Fake:
        @staticmethod
        def apply(x, group):
            r = ranks.rank
            k = sum(1 for t in ranks.log[r] if t[:2] == (group, 'results'))
            ranks.log[r].append((group, 'results', k))
            return Zero.apply(x, (group, k), bwd_log[r])
    return Fake


def rank_rays(world):
    """Every rank renders 16 rays; the last rank's reach no background, and at world 3 all of rank 1's do."""
    _, _, r, i, _, c, rd = bg_case()
    rays, idx = [], []
    for k in range(world):
        rr, ii = r[16 * k:16 * (k + 1)].clone(), i[16 * k:16 * (k + 1)]
        if k == world - 1:
            rr = no_bg(rr, c, rd)
        elif k == 1:
            rr[:, 7] = 1e5
        rays.append(rr)
        idx.append(ii)
    counts = [bg_rays(x, c, rd) for x in rays]
    assert counts[-1] == 0 and all(n > 0 for n in counts[:-1]) and len(set(counts)) == world, counts
    return rays, idx


def rank_nets(net, bg_net, world, train):
    """Every rank's own copy of both networks, under expert parallelism over the fake group ('fg' / 'bg')."""
    out = []
    for _ in range(world):
        pn, pb = train_nets(net, bg_net) if train else (product_net(net), product_net(bg_net))
        EP().enable(pn, group='fg')
        EP().enable(pb, group='bg')
        out.append((pn, pb))
    return out


@pytest.fixture()
def fake_group(monkeypatch):
    def make(world, exchange=fake_all_to_all, **kw):
        ranks = Ranks(world)
        monkeypatch.setattr(EP(), 'dist', FakeDist(ranks))
        monkeypatch.setattr(EP(), '_AllToAll', exchange(ranks, **kw))
        return ranks
    return make


@pytest.mark.parametrize('hard', [False, True])
@pytest.mark.parametrize('world', [2, 3])
def test_eval_with_ranks_on_one_device(one_rank_group, fake_group, world, hard):
    m = M()
    m.set_precision('tc_f16')
    net, bg_net, _, _, hp, c, rd = bg_case(hard)
    rays, idx = rank_rays(world)
    # each rank's own render in the one-rank group
    pn, pb = product_net(net), product_net(bg_net)
    enable([pn, pb])
    try:
        want = [render(m, pn, pb, r, i, hp, c, rd) for r, i in zip(rays, idx)]
    finally:
        disable([pn, pb])
    nets = rank_nets(net, bg_net, world, False)
    ranks = fake_group(world)
    got = ranks.run([lambda k=k: render(m, *nets[k], rays[k], idx[k], hp, c, rd) for k in range(world)], [0] * world)
    for k in range(world):
        assert set(got[k]) == set(want[k])
        for key in want[k]:
            assert torch.equal(got[k][key], want[k][key]), (k, key)
    # the background's exchanges ran on every rank, the one with no background ray included
    assert all(sum(1 for t in ranks.log[k] if t[0] == 'bg') == sum(1 for t in ranks.log[0] if t[0] == 'bg') > 0
               for k in range(world))


def owned_grads(nets, world):
    """The gradient of every sub-module's parameters from the rank that owns it; no other rank holds one."""
    out = {}
    for k in range(world):
        for name, mod in (('fg', nets[k][0]), ('bg', nets[k][1])):
            for j, sub in enumerate(mod.sub_modules):
                for pname, p in sub.named_parameters():
                    key = f'{name}.sub_modules.{j}.{pname}'
                    if j % world == k:
                        assert p.grad is not None, (k, key)
                        out[key] = p.grad.detach().clone()
                    else:
                        assert p.grad is None, (k, key)
    return out


@pytest.mark.parametrize('prec', ['fp32', 'tc_f16'])
@pytest.mark.parametrize('world', [2, 3])
def test_training_with_ranks_on_one_device(one_rank_group, train_precision, fake_group, world, prec):
    m = M()
    train_precision(prec)
    net, bg_net, _, _, hp, c, rd = bg_case()
    rays, idx = rank_rays(world)
    targets = [torch.rand(16, 3, generator=torch.Generator().manual_seed(40 + k)).to(DEV) for k in range(world)]
    seeds = [100 + k for k in range(world)]
    # non-EP training on every rank's rays with that rank's random stream, gradients averaged over the ranks (DDP's .grad)
    pn, pb = train_nets(net, bg_net)
    g_mean = {}
    for k in range(world):
        _, g = train_step(m, pn, pb, rays[k], idx[k], hp, c, rd, targets[k], seeds[k])
        for key, v in g.items():
            g_mean[key] = g_mean.get(key, 0) + v / world
    nets = rank_nets(net, bg_net, world, True)
    ranks = fake_group(world)
    losses = ranks.run([lambda k=k: loss_of(m, *nets[k], rays[k], idx[k], hp, c, rd, targets[k]) for k in range(world)], seeds)
    sum(losses).backward()          # one backward: the autograd engine runs every rank's nodes on its one device thread
    g_ep = owned_grads(nets, world)
    l2 = rel_l2(g_ep, g_mean)
    print(f'background + foreground under EP, {world} ranks [{prec}]: owned grads vs mean of non-EP, rel L2 {l2:.2e}')
    assert l2 <= (FP32_L2 if prec == 'fp32' else TC_L2), l2


@pytest.mark.parametrize('world', [2, 3])
def test_exchange_order_is_the_same_on_every_rank(one_rank_group, train_precision, fake_group, world):
    m = M()
    train_precision('fp32')
    net, bg_net, _, _, hp, c, rd = bg_case()
    rays, idx = rank_rays(world)
    targets = [torch.rand(16, 3, generator=torch.Generator().manual_seed(40 + k)).to(DEV) for k in range(world)]
    nets = rank_nets(net, bg_net, world, True)
    bwd = [[] for _ in range(world)]
    ranks = fake_group(world, tagging_all_to_all, bwd_log=bwd)
    losses = ranks.run([lambda k=k: loss_of(m, *nets[k], rays[k], idx[k], hp, c, rd, targets[k]) for k in range(world)],
                       [100 + k for k in range(world)])
    for loss in losses:
        loss.backward()             # each rank's backward on its own: the tagging exchange never waits for another rank
    fwd = [[t for t in ranks.log[k] if t[1] == 'results'] for k in range(world)]
    assert fwd[0] == [('bg', 'results', 0), ('bg', 'results', 1), ('fg', 'results', 0), ('fg', 'results', 1)], fwd[0]
    assert all(ranks.log[k] == ranks.log[0] for k in range(world))
    assert sorted(bwd[0]) == sorted(t[::2] for t in fwd[0])
    assert all(b == bwd[0] for b in bwd), bwd


# ---- 5. the one-call paths refuse ----------------------------------------------------------------------------------------
def test_one_call_paths_refuse_background_under_expert_parallelism():
    m = M()
    net, bg_net, r, i, hp, c, rd = bg_case()
    pn, pb = product_net(net), product_net(bg_net)
    EP().enable(pb)
    try:
        with pytest.raises(ValueError, match='render_rays'):
            m.render_rays_fused(pn, r, i, hp, True, False, bg_nerf=pb, sphere_center=c, sphere_radius=rd)
        with pytest.raises(ValueError, match='render_rays'):
            m.GraphedRenderRays(pn, hp, r.shape[0], DEV, bg_nerf=pb, sphere_center=c, sphere_radius=rd)
    finally:
        EP().disable(pb)
