"""GPU: fp32 training (mn_model_forward_train + mn_model_backward, the CUDA-core kernels) stage by stage against the float64
restatement of tests/fp32_train_ref.py.

The two calls run through ctypes on a tape and a backward workspace this test owns; mn_debug_fp32_train_layout says where
each intermediate lies.  Every stage is checked from the kernels' own inputs to it (the previous tape layer, the next Linear's
dZ), every parameter gradient per element, the routed tape against O.route, `out` against the tape and the fp32 inference
call bit for bit.  Shapes: every TM of the fp32 kernels (64 up to 256 wide, 32 above), the partly filled second 256-column
pass (320, 384, 448), depths 1, 13 and 16, weight gradients over several chunks, up to 64 sub-modules."""
import ctypes as C

import pytest
import torch

import cases as C_
import fp32_train_ref as R
from oracle import mn_oracle as O
from test_gpu_parity import DEV, product_net

pytestmark = pytest.mark.gpu

CNT_TOTAL = 4 * R.MAX_SUB + 4


def run(net, x, cot, noise, use_coarse=True, probes=()):
    """Record and differentiate in fp32; -> capture (fp32_train_ref), counters or None, and one capture per probe (the same
    tape, differentiated again with grad_out nonzero in one row only: a row, or a function of the capture that picks one)."""
    from mega_nerf_b200 import _cabi as K
    from mega_nerf_b200.modules import _rows_matrix
    lib = K.lib()
    nat = product_net(net).requires_grad_(True)._native()
    h = nat.sync(DEV)
    mh = nat.handle
    B = x.shape[0]
    lay = (C.c_int64 * 64)()
    n = lib.mn_debug_fp32_train_layout(mh, B, lay, 64)
    assert n == K.F32L['COUNT'], n
    lay = {k: lay[i] for k, i in K.F32L.items() if i < n}
    assert lay['TAPE_BYTES'] == lib.mn_model_tape_bytes(mh, B)
    assert lay['BWD_BYTES'] == lib.mn_model_backward_workspace_bytes(mh, B)
    rows, xin = _rows_matrix(x.to(DEV))
    C1 = net.spec.rgb_dim + 1
    out = torch.empty(B, C1, device=DEV)
    out_inf = torch.empty(B, C1, device=DEV)
    ws = torch.empty(max(int(lib.mn_model_workspace_bytes(mh, B, K.PREC_FP32)), 256), device=DEV, dtype=torch.uint8)
    tape = torch.zeros(lay['TAPE_BYTES'], device=DEV, dtype=torch.uint8)
    nz = noise.to(DEV).contiguous().view(-1) if noise is not None else None
    st = K.stream_of(DEV)
    uc = 1 if use_coarse else 0
    K.check(lib.mn_model_forward_train(h, mh, C.byref(rows), B, uc, K.ptr(nz), K.ptr(out), K.ptr(tape), tape.numel(), K.ptr(ws),
                                       ws.numel(), st), h)
    K.check(lib.mn_model_forward(h, mh, C.byref(rows), B, uc, 0, K.ptr(nz), K.PREC_FP32, K.ptr(out_inf), K.ptr(ws), ws.numel(), st), h)
    off = nat._offsets()
    TM, nt = lay['TM'], lay['N_TILES']
    tl = {k.lower(): lay[k] for k in lay if k.startswith('A_') or k.startswith('G_')}
    tl['n_aux'] = tl['a_h'] - tl['a_aux']

    def backward(g):
        gbuf = torch.zeros(int(lib.mn_model_grad_floats(mh)), device=DEV)
        bws = torch.zeros(lay['BWD_BYTES'], device=DEV, dtype=torch.uint8)
        K.check(lib.mn_model_backward(h, mh, B, uc, K.ptr(K.f32c(g.to(DEV))), K.ptr(tape), tape.numel(), K.ptr(gbuf), K.ptr(bws),
                                      bws.numel(), st), h)
        torch.cuda.synchronize()
        grads = [{k: gbuf[s * off['stride'] + off[k]:][:v.numel()].view(v.shape).double() for k, v in w.items()}
                 for s, w in enumerate(net.weights)]
        gt = lay['G_TOTAL']
        grad = bws[lay['BWD_GRAD']:][:nt * gt * TM * 4].view(torch.float32).view(nt, gt, TM).permute(0, 2, 1).reshape(nt * TM, gt)
        return grad.double(), grads

    torch.cuda.synchronize()
    at = lay['A_TOTAL']
    act = tape[lay['TAPE_ACT']:][:nt * at * TM * 4].view(torch.float32).view(nt, at, TM).permute(0, 2, 1).reshape(nt * TM, at)
    routed = net.kind == 'mega'
    counters = None
    if routed:
        counters = tape[lay['TAPE_COUNTERS']:][:CNT_TOTAL * 4].view(torch.int32)
        n_slots = int(counters[3 * R.MAX_SUB + 1])
        slot_row = tape[lay['TAPE_SLOT_ROW']:][:nt * TM * 4].view(torch.int32).long()
        slot_w = tape[lay['TAPE_SLOT_W']:][:nt * TM * 4].view(torch.float32).double() if lay['TAPE_SLOT_W'] >= 0 else None
        K_ = len(net.weights)
        starts, subs = [int(v) for v in counters[R.MAX_SUB:R.MAX_SUB + K_ + 1]], list(range(K_))
    else:
        n_slots = B
        slot_row = torch.arange(nt * TM, device=DEV)
        slot_row[slot_row >= B] = -1
        slot_w = None
        S = -(-B // TM) * TM
        starts, subs = [0, S], [0 if net.kind == 'nerf' or use_coarse else 1]
    S = -(-n_slots // TM) * TM
    xc = x[:, 3:] if net.xyz_real else x
    base = dict(TM=TM, chunk=lay['CHUNK_TILES'], tl=tl, act=act[:S].double(), slot_row=slot_row[:S], n_slots=n_slots,
                slot_w=slot_w[:S] if slot_w is not None else None, starts=starts, subs=subs, x=xc.to(DEV),
                noise=nz, out=out, out_inf=out_inf)
    grad, grads = backward(cot)
    cap = dict(base, grad=grad[:S], grads=grads, go=cot.to(DEV))
    pcaps = {}
    for name, row in probes:
        row = row(cap) if callable(row) else row
        g = torch.zeros_like(cot)
        g[row] = cot[row]
        grad, grads = backward(g)
        pcaps[name] = (row, dict(base, grad=grad[:S], grads=grads, go=g.to(DEV)))
    return cap, counters, pcaps


def weights_on_device(net):
    return [{k: v.to(DEV) for k, v in w.items()} for w in net.weights]


def check(net, x, cot, noise, name, use_coarse=True, probes=()):
    cap, counters, pcaps = run(net, x, cot, noise, use_coarse, probes)
    rep = R.Report()
    R.check_call(net.spec, weights_on_device(net), cap, rep)
    rep.exact('out: fp32 inference = recording (bitwise)', cap['out_inf'], cap['out'])
    if counters is not None:
        R.check_routing(net, x, cap, counters, rep)
    for pname, (row, pc) in pcaps.items():
        R.check_probe(net.spec, pc, row, rep, f'{pname} ')
    print(f'\n{name} (TM {cap["TM"]}, {cap["act"].shape[0]} slots)\n{rep.text()}')
    assert not rep.failures(), rep.failures()
    return cap, rep


def rows_and_grads(spec, n, seed, scale=1e-2):
    x = C_.nerf_rows(spec, n, seed)
    g = torch.Generator().manual_seed(seed + 1)
    cot = (torch.rand(n, spec.rgb_dim + 1, generator=g) - 0.4) * scale
    noise = torch.randn(n, 1, generator=g)
    if spec.appearance_dim > 0:      # a third of the rows on 3 images, the rest spread
        x[: n // 3, -1] = (torch.arange(n // 3) % 3).float()
    return x, cot, noise


def make(spec, seed=21, kind='nerf'):
    net = O.make_net(kind, spec, seed=seed)
    if not spec.shifted_softplus:
        for w in net.weights:
            w['sigma.bias'] = w['sigma.bias'] + 0.5
    return net


BG = dict(xyz_dim=4, shifted_softplus=False, skip_layers=(2, 5))
SPECS = {
    # rgb + appearance head at every TM of the fp32 kernels
    'w64': O.NerfSpec(layer_dim=64),
    'w192': O.NerfSpec(layer_dim=192),
    'w256': O.NerfSpec(),
    'w320': O.NerfSpec(layer_dim=320),
    'w384': O.NerfSpec(layer_dim=384),
    'w448': O.NerfSpec(layer_dim=448),
    'w512': O.NerfSpec(layer_dim=512),
    # heads
    'sh4_448': O.NerfSpec(layer_dim=448, pos_dir_dim=0, rgb_dim=75),
    'affine192': O.NerfSpec(layer_dim=192, affine_appearance=True),
    'nodira320': O.NerfSpec(layer_dim=320, pos_dir_dim=0, appearance_dim=0),
    'bg256': O.NerfSpec(**BG),
    # depths
    'd1_256': O.NerfSpec(layers=1, skip_layers=()),
    'd13_256': O.NerfSpec(layers=13, skip_layers=(4, 8)),
    'd16_256': O.NerfSpec(layers=16, skip_layers=(4, 8)),
    'd13_512': O.NerfSpec(layer_dim=512, layers=13, skip_layers=(4, 8)),
    'd16_512': O.NerfSpec(layer_dim=512, layers=16, skip_layers=(4, 8)),
}


@pytest.mark.parametrize('vname', list(SPECS))
def test_stages(vname):
    spec = SPECS[vname]
    x, cot, noise = rows_and_grads(spec, 200, 5)
    check(make(spec), x, cot, noise, vname)


def chunks3(TM):
    return 2 * 64 * TM + 37


@pytest.mark.parametrize('vname,n', [('w192', 1), ('w192', 63), ('w192', 65), ('w192', 129), ('w384', 33),
                                     ('w192', chunks3(64)), ('w448', chunks3(32))])
def test_row_counts(vname, n):
    """Ragged tiles, and two full weight-gradient chunks plus a ragged third at each TM."""
    spec = SPECS[vname]
    x, cot, noise = rows_and_grads(spec, n, 11 + n)
    cap, _ = check(make(spec), x, cot, noise, f'{vname}[{n}]')
    TM = cap['TM']
    assert cap['TM'] == (64 if spec.layer_dim <= 256 else 32)
    if n > 64 * TM:
        assert cap['act'].shape[0] > 2 * cap['chunk'] * TM


@pytest.mark.parametrize('vname', ['w192', 'w448'])
def test_probes(vname):
    """One-hot grad_out rows: the first slot of the second weight-gradient chunk, the last slot before a bucket boundary,
    the last row of the batch."""
    spec = SPECS[vname]
    TM = 64 if spec.layer_dim <= 256 else 32
    n = chunks3(TM)
    x, cot, noise = rows_and_grads(spec, n, 3)
    probes = [('second chunk', 64 * TM), ('bucket end', R.MN_BUCKET - 1), ('last row', n - 1)]
    check(make(spec), x, cot, noise, f'{vname} probes', probes=probes)


def mega(grid, margin, layer_dim=64, cluster_2d=True, xyz_real=False, seed=3):
    spec = O.NerfSpec(layer_dim=layer_dim, xyz_dim=4 if xyz_real else 3)
    cents = O.grid_centroids(*grid)
    if not cluster_2d:
        g = torch.Generator().manual_seed(11)
        cents = cents.clone()
        cents[:, 0] = torch.rand(cents.shape[0], generator=g) * 0.4 - 0.2
    return O.make_net('mega', spec, seed=seed, n_sub=cents.shape[0], centroids=cents, boundary_margin=margin,
                      xyz_real=xyz_real, cluster_2d=cluster_2d)


MEGA = {
    'hard8': dict(grid=(2, 4), margin=1.0),
    'blend8': dict(grid=(2, 4), margin=1.15),
    'blend25': dict(grid=(5, 5), margin=1.15),
    'hard33': dict(grid=(3, 11), margin=1.0),
    'blend33': dict(grid=(3, 11), margin=1.15),
    'hard64': dict(grid=(8, 8), margin=1.0),
    'blend64': dict(grid=(8, 8), margin=1.15),
    'hard8_3d_real': dict(grid=(2, 4), margin=1.0, cluster_2d=False, xyz_real=True),
}


def mega_case(mname, n=3000, seed=13):
    net = mega(**MEGA[mname])
    x = C_.mega_rows(net, n, seed)
    if mname in ('hard8', 'blend8'):          # drop the rows routed to the last centroid: that sub-module owns no slot
        assign, wts = O.route(net, x)
        x = x[(assign != len(net.weights) - 1) if wts is None else ~(wts[:, -1] > 0)]
    g = torch.Generator().manual_seed(6)
    cot = (torch.rand(x.shape[0], 4, generator=g) - 0.5) * 1e-2
    noise = torch.rand(x.shape[0], 1, generator=g)
    return net, x, cot, noise


@pytest.mark.parametrize('mname', list(MEGA))
def test_routed(mname):
    net, x, cot, noise = mega_case(mname)
    cap, rep = check(net, x, cot, noise, mname)
    if mname in ('hard8', 'blend8'):
        assert any(r['stage'].startswith('[7] no slots') for r in rep.rows)


def test_routed_many_chunks():
    """Rows concentrated in one cell: sub-module 0 owns more than MN_WG_CHUNK_TILES x TM slots.  Probes: the first slot of
    its second chunk, a row blended into two or more sub-modules, the last row of the batch."""
    net = mega(grid=(2, 4), margin=1.15)
    n = 6000
    x = C_.mega_rows(net, n, 17)
    g = torch.Generator().manual_seed(8)
    c0 = net.centroids[0]
    x[:4800, 1:3] = c0[1:] + (torch.rand(4800, 2, generator=g) - 0.5) * 0.2
    cot = (torch.rand(n, 4, generator=g) - 0.5) * 1e-2
    noise = torch.rand(n, 1, generator=g)
    _, wts = O.route(net, x)
    multi = int(torch.nonzero((wts > 0).sum(1) >= 2)[0])

    def second_chunk(cap):       # the slot order inside a bucket follows the router's atomics: read the row off this call's tape
        TM, chunk = cap['TM'], cap['chunk']
        assert cap['starts'][1] - cap['starts'][0] > chunk * TM
        row = int(cap['slot_row'][cap['starts'][0] + chunk * TM])
        assert row >= 0
        return row

    check(net, x, cot, noise, 'many chunks', probes=[('blended row', multi), ('last row', n - 1), ('second chunk', second_chunk)])


@pytest.mark.parametrize('use_coarse', [True, False])
def test_cascade(use_coarse):
    spec = SPECS['w192']
    net = make(spec, kind='cascade')
    x, cot, noise = rows_and_grads(spec, 300, 4)
    check(net, x, cot, noise, f'cascade use_coarse={use_coarse}', use_coarse=use_coarse)


@pytest.mark.parametrize('edge', ['zero_grad', 'outlier', 'zero_preact', 'softplus_threshold'])
def test_edges(edge):
    spec = SPECS['w256']
    net = make(spec)
    x, cot, noise = rows_and_grads(spec, 300, 9)
    w = net.weights[0]
    if edge == 'zero_grad':
        cot = torch.zeros_like(cot)
    elif edge == 'outlier':                   # one row 2^20 above the rest
        cot[17] *= 2.0 ** 20
    elif edge == 'zero_preact':               # pre-activations exactly 0: both ReLU masks 0
        for i in (2, 6):
            w[f'xyz_encodings.{i}.0.weight'][:40] = 0.0
            w[f'xyz_encodings.{i}.0.bias'][:40] = 0.0
        w['dir_a_encoding.0.weight'][:10] = 0.0
        w['dir_a_encoding.0.bias'][:10] = 0.0
    else:                                     # sigma pre-activation 21.0 (y = 20: the sigmoid branch) and 21.5
        w['sigma.weight'].zero_()
        w['sigma.bias'].fill_(21.0)
        noise = torch.zeros_like(noise)
        noise[::2] = 0.5
    cap, rep = check(net, x, cot, noise, edge)
    if edge == 'zero_grad':
        assert all(bool((v == 0).all()) for g in cap['grads'] for v in g.values())
    if edge == 'zero_preact':
        L = spec.layer_dim
        h2 = R.ch(cap, 'a_h', 40, 2 * L)[cap['slot_row'] >= 0]
        assert bool((h2 == 0).all())
    if edge == 'softplus_threshold':
        pre = R.ch(cap, 'a_sig')[cap['slot_row'] >= 0]
        assert set(pre.view(-1).tolist()) == {21.0, 21.5}
