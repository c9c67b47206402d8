"""CPU-only: the arithmetic of the merge + composite kernels (composite_kernel, composite_bwd_kernel in csrc/mn_sample.cu)
restated step by step in torch, and a first-order model of its rounding error against a float64 reference of the same
operation.

The kernels compute, per merged sample j, in fp32: delta_j, alpha_j = 1 - expf(-delta_j sigma_j) and
x_j = (1 - alpha_j) + 1e-8; the exclusive transmittance T_j is an fp64 prefix product of the x_k rounded to fp32, the
weights w_j = alpha_j T_j are fp32, the products w_j c_j are fp32 and are summed in fp64.  The backward pass rebuilds T the
same way, forms d alpha_j = T_j G_j - (sum_{i>j} w_i G_i + lambda g_lambda) / x_j with G_j = g.c_j and the suffix sum in
fp64, and rounds d sigma_j = d alpha_j delta_j exp(-delta_j sigma_j) to fp32 once.

`error_bounds` turns that into a bound per output element, built from the float64 quantities of the exact computation:
the rounding of every fp32 step, the relative error of T_j as the product of the relative errors of the x_k before it,
and the propagation of both into the sums and the gradients.  This file checks that the emulation stays inside the bound
at every shape the GPU tests use (tests/test_gpu_zzb_sample_counts.py, which holds the kernels to the same bound) and that
the bound is tight enough to reject a tie taken in the wrong order or a dropped sample.  The tolerances of the GPU tests
come from here."""
from typing import Dict

import pytest
import torch

from oracle import mn_oracle as O

U = 2.0 ** -24          # unit roundoff of fp32
U64 = 2.0 ** -53
TINY = 2.0 ** -150      # half the least fp32 subnormal: the absolute error of a result that underflows
SAFETY = 2.0            # the bounds are first order; second-order terms are far below this factor at every shape here

# (S, S2): own samples and stored (merged) samples per ray.  The production counts (256 coarse + 512 fine, and the
# background's 128 + 256), run lengths around a warp, and the 4096-sample limit of the shared-memory merge.
SHAPES = [(256, 512), (128, 256), (1, 0), (31, 0), (33, 0), (256, 0), (4096, 0), (33, 31), (512, 512), (513, 512),
          (1024, 3072)]
N_RAYS = 203            # not a multiple of the 4 rays of a CTA
REGIMES = ('zero', 'saturating', 'sparse', 'degenerate', 'dense')


def merges(S2: int, flip: bool):
    """How the stored run arrives: 'sorted' (both runs in the pass's order: the rank merge), 'shuffled' (the bitonic sort),
    'mixed' (flip only: an ascending own run against a descending stored one, as in the background pass)."""
    if S2 == 0:
        return ['none']
    return ['sorted', 'shuffled'] + (['mixed'] if flip else [])


def all_cases():
    return [(S, S2, flip, merge) for S, S2 in SHAPES for flip in (False, True) for merge in merges(S2, flip)]


def case_id(c) -> str:
    S, S2, flip, merge = c
    return f'{S}+{S2}-flip{int(flip)}-{merge}'


def composite_case(S: int, S2: int, flip: bool, merge: str, n: int = N_RAYS, seed: int = 0) -> Dict[str, torch.Tensor]:
    """Seeded fp32 inputs of one merged composite.  Ray r has the density regime REGIMES[r % 5]: all zero; saturating
    (sigma delta >= 50, so T falls to 1e-8^k and underflows); sparse; degenerate (near == far: every depth equal); dense.
    Every third ray has a finite last delta (given in the kernel's convention: the kernel subtracts the max own depth), the
    others 1e10.  On even rays the stored run takes some of its depths from the own run (exact ties between the runs)."""
    g = torch.Generator().manual_seed(seed * 1000 + S * 7 + S2 * 3 + int(flip))
    regime = [REGIMES[r % len(REGIMES)] for r in range(n)]

    def depths(m):
        return torch.rand(n, m, generator=g) * 0.8 + 0.05

    z = depths(S)
    z2 = depths(S2) if S2 > 0 else None
    if S2 > 0:
        for r in range(0, n, 2):
            k = min(S, S2, max(1, S2 // 3))
            src = torch.randperm(S, generator=g)[:k]
            dst = torch.randperm(S2, generator=g)[:k]
            z2[r, dst] = z[r, src]
    for r in range(n):
        if regime[r] == 'degenerate':
            z[r] = 0.3
            if S2 > 0:
                z2[r] = 0.3

    def order(t, descending):
        return torch.sort(t, -1, descending=descending)[0]

    z = order(z, flip and merge != 'mixed')
    if S2 > 0:
        z2 = order(z2, flip)
        if merge == 'shuffled':
            z2 = torch.gather(z2, 1, torch.argsort(torch.rand(n, S2, generator=g), -1))

    def densities(m):
        sig = torch.rand(n, m, generator=g) * 30
        for r in range(n):
            if regime[r] == 'zero':
                sig[r] = 0
            elif regime[r] == 'saturating':
                sig[r] = 1e6 * (1 + sig[r])
            elif regime[r] == 'sparse':
                sig[r] *= 3 * (torch.rand(m, generator=g) < 0.05).float()
        return sig

    raw = torch.cat([torch.rand(n, S, 3, generator=g), densities(S).unsqueeze(-1)], -1)
    raw2 = torch.cat([torch.rand(n, S2, 3, generator=g), densities(S2).unsqueeze(-1)], -1) if S2 > 0 else None
    dreal = dreal2 = None
    if flip:        # the background pass composites the real depths of its samples
        dreal = torch.rand(n, S, generator=g) * 9 + 1
        dreal2 = torch.rand(n, S2, generator=g) * 9 + 1 if S2 > 0 else None
    zmax = z.max(-1)[0]
    ld = torch.full((n,), 1e10)
    ld[::3] = zmax[::3] + 1.0 + torch.rand((n + 2) // 3, generator=g)
    return dict(raw=raw, z=z, dreal=dreal, raw2=raw2, z2=z2, dreal2=dreal2, last_delta=ld, flip=flip,
                cot_rgb=torch.randn(n, 3, generator=g), cot_lam=torch.randn(n, generator=g))


def merged(c: Dict[str, torch.Tensor]):
    """The merged run as the kernels order it: (depth, index) with the own samples first on ties, i.e. a stable sort of
    cat([own, stored]).  -> (raw [n,m,4], z [n,m], depth values [n,m], order [n,m] into cat([own, stored]))."""
    raw, z, dd = c['raw'], c['z'], c['dreal'] if c['dreal'] is not None else c['z']
    if c['z2'] is None:
        return raw, z, dd, torch.arange(z.shape[1]).expand_as(z)
    zc = torch.cat([z, c['z2']], -1)
    zs, order = torch.sort(zc, dim=-1, descending=bool(c['flip']), stable=True)
    rawc = torch.cat([raw, c['raw2']], 1)
    ddc = torch.cat([dd, c['dreal2'] if c['dreal2'] is not None else c['z2']], -1)
    return torch.gather(rawc, 1, order.unsqueeze(-1).expand(-1, -1, 4)), zs, torch.gather(ddc, 1, order), order


def last_delta_eff(c, dtype):
    """The last delta of each ray: ld - max(own depths) where ld < 1e10 (rendering.py:191-193), in `dtype`."""
    ld, zmax = c['last_delta'].to(dtype), c['z'].to(dtype).max(-1)[0]
    return torch.where(ld < 1e10, ld - zmax, ld)


def unmerge(t: torch.Tensor, order: torch.Tensor, S: int):
    out = torch.empty_like(t)
    out.scatter_(1, order.unsqueeze(-1).expand_as(t) if t.dim() == 3 else order, t)
    return out[:, :S], out[:, S:]


def _deltas(z, ld, flip):
    d = (z[:, :-1] - z[:, 1:]) if flip else (z[:, 1:] - z[:, :-1])
    return torch.cat([d, ld.unsqueeze(-1)], -1)


def emulate(raw, z, dd, ld32, flip, cot_rgb, cot_lam) -> Dict[str, torch.Tensor]:
    """composite_kernel + composite_bwd_kernel on an already merged fp32 run, rounding where the kernels round."""
    rgbs, sig = raw[..., :3], raw[..., 3]
    delta = _deltas(z, ld32, flip)
    ex = torch.exp(-delta * sig)
    alpha = 1 - ex
    x = (1 - alpha) + 1e-8
    P = torch.cumprod(x.double(), -1)                                   # fp64 prefix product
    T = torch.cat([torch.ones_like(x[:, :1]), P[:, :-1].float()], -1)   # rounded to fp32: exclusive transmittance
    w = alpha * T
    rgb = (w.unsqueeze(-1) * rgbs).double().sum(1).float()
    depth = (w * dd).double().sum(1).float()
    t = z - depth.unsqueeze(-1)
    var = (w * (t * t)).double().sum(1).float()
    lam = P[:, -1].float()
    g = cot_rgb
    G = g[:, 0:1].double() * rgbs[..., 0].double() + g[:, 1:2].double() * rgbs[..., 1].double() \
        + g[:, 2:3].double() * rgbs[..., 2].double()
    wG = w.double() * G
    later = torch.flip(torch.cumsum(torch.flip(wG, [-1]), -1), [-1]) - wG
    lt = (lam.double() * cot_lam.double()).unsqueeze(-1) if cot_lam is not None else 0.0
    d_alpha = T.double() * G - (later + lt) / x.double()
    d_sigma = (d_alpha * delta.double() * ex.double()).float()
    d_rgb = w.unsqueeze(-1) * g.unsqueeze(1)
    return dict(weights=w, rgb=rgb, depth=depth, depth_variance=var, bg_lambda=lam,
                grad_raw=torch.cat([d_rgb, d_sigma.unsqueeze(-1)], -1))


def emulate_case(c, with_lambda: bool):
    raw, z, dd, order = merged(c)
    out = emulate(raw, z, dd, last_delta_eff(c, torch.float32), c['flip'], c['cot_rgb'], c['cot_lam'] if with_lambda else None)
    out['grad_raw'], out['grad_raw2'] = unmerge(out['grad_raw'], order, c['z'].shape[1])
    return out


def reference64(c, with_lambda: bool) -> Dict[str, torch.Tensor]:
    """The float64 oracle composite of the merged run, and its autograd w.r.t. the per-sample (rgb, sigma)."""
    raw, z, dd, order = merged(c)
    r = raw.double().requires_grad_(True)
    o = O.composite(r[..., :3], r[..., 3], z.double(), last_delta_eff(c, torch.float64).unsqueeze(-1), c['flip'],
                    dd.double())
    loss = (o['rgb'] * c['cot_rgb'].double()).sum()
    if with_lambda:
        loss = loss + (o['bg_lambda'] * c['cot_lam'].double()).sum()
    loss.backward()
    out = {k: v.detach() for k, v in o.items()}
    out['grad_raw'], out['grad_raw2'] = unmerge(r.grad, order, c['z'].shape[1])
    return out


def error_bounds(c, with_lambda: bool) -> Dict[str, torch.Tensor]:
    """First-order bound on |fp32 kernel - float64 reference| per output element, from the float64 quantities."""
    raw, z, dd, order = merged(c)
    raw, z, dd = raw.double(), z.double(), dd.double()
    flip = c['flip']
    rgbs, sig = raw[..., :3], raw[..., 3]
    n = z.shape[1]
    delta = _deltas(z, last_delta_eff(c, torch.float64), flip)
    a = delta * sig
    e = torch.exp(-a)
    alpha = 1 - e
    x = (1 - alpha) + 1e-8
    P = torch.cumprod(x, -1)
    T = torch.cat([torch.ones_like(x[:, :1]), P[:, :-1]], -1)
    w = alpha * T
    j = torch.arange(n, dtype=torch.float64)

    d_delta = U * delta.abs()                                # one fp32 subtraction (1e10 is exact)
    d_a = d_delta * sig + U * a.abs()
    d_e = e * (d_a + 4 * U)                                  # expf: <= 2 ulp
    d_alpha = d_e + torch.minimum(U * alpha.abs(), e)      # 1 - e rounds to the nearer of its neighbours; 1 is one of them
    d_x = d_alpha + U * (1 - alpha).abs() + 2 * U * x        # 1 - alpha, + 1e-8 (and 1e-8's own fp32 rounding)
    rx = torch.cumsum(d_x / x, -1)                           # relative error of the prefix products, summed
    # a run of nearly opaque samples makes the relative error of T large while T itself vanishes: the clamp keeps T * rT
    # finite (a T that small is below fp32's range, where TINY bounds the error)
    rT = torch.expm1(torch.cat([torch.zeros_like(rx[:, :1]), rx[:, :-1]], -1).clamp(max=80.0)) + U + j * 2 * U64
    d_T = T * rT + TINY
    d_w = d_alpha * T + alpha * d_T + U * w + TINY

    def sum_bound(v, dv, prod):
        """|error| of fl64-sum of fp32 products v_j w_j, rounded to fp32, given |error| dv of each w_j: propagated error,
        the product rounding, the fp64 sum and the final rounding (|exact result| <= sum |prod|)."""
        s = prod.abs().sum(-1)
        return (v.abs() * dv).sum(-1) + U * s + n * TINY + n * U64 * s + U * prod.sum(-1).abs()

    out = {'weights': d_w}
    out['rgb'] = torch.stack([sum_bound(rgbs[..., k], d_w, w * rgbs[..., k]) for k in range(3)], -1)
    depth = (w * dd).sum(-1)
    out['depth'] = sum_bound(dd, d_w, w * dd)
    t = z - depth.unsqueeze(-1)
    d_t = out['depth'].unsqueeze(-1) + U * t.abs()
    d_t2 = 2 * t.abs() * d_t + U * t * t
    out['depth_variance'] = (d_w * t * t + w * d_t2 + U * w * t * t).sum(-1) + n * TINY + (n * U64 + U) * (w * t * t).sum(-1)
    lam = P[:, -1]
    out['bg_lambda'] = lam * (torch.expm1(rx[:, -1].clamp(max=80.0)) + U + n * 2 * U64) + TINY

    g = c['cot_rgb'].double()
    gl = c['cot_lam'].double() if with_lambda else torch.zeros(z.shape[0], dtype=torch.float64)
    d_grad_rgb = g.abs().unsqueeze(1) * d_w.unsqueeze(-1) + U * (w.unsqueeze(-1) * g.unsqueeze(1)).abs() + TINY
    G = (rgbs * g.unsqueeze(1)).sum(-1)
    Gabs = (rgbs * g.unsqueeze(1)).abs().sum(-1)
    wG = w * G
    later = torch.flip(torch.cumsum(torch.flip(wG, [-1]), -1), [-1]) - wG
    d_later = torch.flip(torch.cumsum(torch.flip(Gabs * d_w, [-1]), -1), [-1]) - Gabs * d_w \
        + n * U64 * (w * Gabs).sum(-1, keepdim=True)
    lt = (lam * gl).unsqueeze(-1)
    d_lt = (gl.abs() * out['bg_lambda']).unsqueeze(-1)
    tail = later + lt
    da = T * G - tail / x
    d_da = d_T * Gabs + (d_later + d_lt) / x + tail.abs() * d_x / (x * x) + 4 * U64 * (T * Gabs + tail.abs() / x)
    ds = da * delta * e
    d_ds = d_da * (delta * e).abs() + da.abs() * (d_delta * e + delta.abs() * d_e) + U * ds.abs() + TINY
    out['grad_raw'], out['grad_raw2'] = unmerge(torch.cat([d_grad_rgb, d_ds.unsqueeze(-1)], -1), order, c['z'].shape[1])
    return {k: SAFETY * v for k, v in out.items()}


def worst_ratio(got: Dict[str, torch.Tensor], want: Dict[str, torch.Tensor], bound: Dict[str, torch.Tensor],
                keys=None) -> Dict[str, float]:
    """max over elements of |got - want| / bound, per output (> 1: outside the bound)."""
    out = {}
    for k in keys or bound:
        if k not in got or got[k] is None or (k == 'grad_raw2' and want[k].numel() == 0):
            continue
        err = (got[k].detach().double().cpu() - want[k].double()).abs()
        out[k] = float((err / bound[k]).max()) if err.numel() else 0.0
    return out


FWD = ('weights', 'rgb', 'depth', 'depth_variance', 'bg_lambda')
BWD = ('grad_raw', 'grad_raw2')


# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('case', all_cases(), ids=case_id)
def test_emulation_inside_bound(case):
    """(a) The kernels' arithmetic, emulated, sits inside the bound at every shape, merge path and density regime."""
    c = composite_case(*case)
    for with_lambda in (False, True):
        ref = reference64(c, with_lambda)
        bound = error_bounds(c, with_lambda)
        emu = emulate_case(c, with_lambda)
        r = worst_ratio(emu, ref, bound, FWD + BWD)
        assert max(r.values()) <= 1.0, (case_id(case), with_lambda, r)
        for k in FWD + BWD:
            if k in emu and emu[k].numel():
                assert torch.isfinite(emu[k]).all(), k


def _tie_ray(c):
    """A ray whose merged run has an own and a stored sample at the same depth, both with real weight."""
    raw, z, _, order = merged(c)
    S = c['z'].shape[1]
    em = emulate_case(c, False)
    w = em['weights']
    own = order < S
    for r in range(z.shape[0]):
        for p in range(z.shape[1] - 2):
            if z[r, p] == z[r, p + 1] and own[r, p] and not own[r, p + 1] and \
                    w[r, p + 1] > 1e-3 and (raw[r, p] - raw[r, p + 1]).abs().max() > 0.1:
                return r, p
    raise AssertionError('no usable tie')


@pytest.mark.parametrize('S,S2,flip', [(256, 512, False), (128, 256, True)])
def test_bound_rejects_swapped_tie(S, S2, flip):
    """(b) Stored sample first on a tie - the other order of the merge - moves the ray's outputs outside the bound."""
    c = composite_case(S, S2, flip, 'sorted')
    ref, bound = reference64(c, True), error_bounds(c, True)
    r, p = _tie_ray(c)
    raw, z, dd, _ = merged(c)
    perm = torch.arange(z.shape[1])
    perm[p], perm[p + 1] = p + 1, p
    rr = slice(r, r + 1)
    bad = emulate(raw[rr][:, perm], z[rr][:, perm], dd[rr][:, perm], last_delta_eff(c, torch.float32)[rr], flip,
                  c['cot_rgb'][rr], c['cot_lam'][rr])
    refr = {k: v[rr] for k, v in ref.items() if k in FWD}
    bnd = {k: v[rr] for k, v in bound.items() if k in FWD}
    ratios = worst_ratio(bad, refr, bnd, ('rgb', 'depth', 'weights'))
    assert max(ratios.values()) > 1.0, ratios


@pytest.mark.parametrize('S,S2,flip', [(256, 512, False), (128, 256, True), (4096, 0, False)])
def test_bound_rejects_dropped_sample(S, S2, flip):
    """(b) Leaving out one sample with a non-negligible weight moves the ray's colour and depth outside the bound."""
    c = composite_case(S, S2, flip, 'sorted' if S2 else 'none')
    ref, bound = reference64(c, False), error_bounds(c, False)
    raw, z, dd, _ = merged(c)
    r = 4                                               # a 'dense' ray
    assert REGIMES[r % len(REGIMES)] == 'dense'
    p = int(torch.argmax(ref['weights'][r, :-1]))
    assert float(ref['weights'][r, p]) > 1e-3
    keep = torch.cat([torch.arange(p), torch.arange(p + 1, z.shape[1])])
    rr = slice(r, r + 1)
    bad = emulate(raw[rr][:, keep], z[rr][:, keep], dd[rr][:, keep], last_delta_eff(c, torch.float32)[rr], flip,
                  c['cot_rgb'][rr], None)
    ratios = worst_ratio(bad, {k: v[rr] for k, v in ref.items()}, {k: v[rr] for k, v in bound.items()}, ('rgb', 'depth'))
    assert min(ratios.values()) > 1.0, ratios

