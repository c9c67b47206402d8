"""GPU: tensor-core training (precision 'tc_f16') stage by stage against the float64 restatement of tests/tc_train_ref.py.

mn_model_forward_train_tc and mn_model_backward_tc run through ctypes on a tape and a backward workspace this test owns;
mn_debug_tc_train_layout says where each intermediate lies.  Every stage is checked from the kernel's own inputs to it (the
previous tape image, the previous dZ image, the fp32 head blocks), so the bound of a stage is one rounding step wide and
does not grow with depth: encoder tiles, every activation image, the fp32 head block, S (bit-exact), the head-gradient
blocks, every dZ image still in the workspace (all of them on the fused engine; dZ_G and the last two ping-pong images on the
layer engine, called with one tile group), and every parameter gradient per element.  The layer engine's other weight
gradients are compared with the restatement's own fp16 dZ chain, seeded with the kernel's forward tape, at LAYER_TOL of each
tensor's max."""
import ctypes as C

import pytest
import torch

import cases as C_
import tc_train_ref as T
from oracle import mn_oracle as O
from test_gpu_parity import DEV, product_net

pytestmark = pytest.mark.gpu

# per-tensor tolerance (fraction of the tensor's max) of the layer engine's gradients below its resident dZ images against the
# restatement seeded with the same forward tape: measured at most 9.1e-4 on an H100 80GB HBM3 (700 W) over every case here
LAYER_TOL = 4e-3
MAX_SUB = 64          # MN_MAX_SUB: counters[MAX_SUB + s] is the first slot of sub-module s, counters[3 MAX_SUB + 1] the slot count


def images(buf, base, tile_bytes, n_tiles, off, cols):
    """[n_tiles * 128, cols] float64 of the fp16 tile images [cols/8][128][8] at base + t tile_bytes + off."""
    t = buf[base:base + n_tiles * tile_bytes].view(n_tiles, tile_bytes)[:, off:off + cols * 256].contiguous()
    return t.view(torch.float16).view(n_tiles, cols // 8, 128, 8).permute(0, 2, 1, 3).reshape(n_tiles * 128, cols).double()


def f32_blocks(buf, base, rows, n_tiles):
    """[n_tiles * 128, rows] of the fp32 blocks [tiles][rows][128] at base."""
    t = buf[base:base + n_tiles * rows * 512].contiguous().view(torch.float32).view(n_tiles, rows, 128)
    return t.permute(0, 2, 1).reshape(n_tiles * 128, rows).double()


def run(net, x, cot, noise):
    """Record and differentiate on the tensor cores; -> (layout, tape bytes, workspace bytes, gradient dict per sub-module)."""
    from mega_nerf_b200 import _cabi as K
    from mega_nerf_b200.modules import _rows_matrix
    lib = K.lib()
    pn = product_net(net).requires_grad_(True)
    nat = pn._native()
    h = nat.sync(DEV)
    mh = nat.handle
    assert lib.mn_model_train_tc_supported(mh)
    B = x.shape[0]
    lay = (C.c_int64 * 256)()
    n = lib.mn_debug_tc_train_layout(mh, B, lay, 256)
    assert n > 0, n
    lay = list(lay)[:n]
    rows, xin = _rows_matrix(x.to(DEV))
    out = torch.empty(B, net.spec.rgb_dim + 1, device=DEV)
    ws = torch.empty(max(int(lib.mn_model_workspace_bytes(mh, B, K.PREC_FP32)), 256), device=DEV, dtype=torch.uint8)
    tape = torch.zeros(lay[K.TCL['TAPE_BYTES']], device=DEV, dtype=torch.uint8)
    assert tape.numel() == lib.mn_model_tape_bytes_tc(mh, B)
    nz = noise.to(DEV).contiguous().view(-1)
    st = K.stream_of(DEV)
    K.check(lib.mn_model_forward_train_tc(h, mh, C.byref(rows), B, 1, K.ptr(nz), K.ptr(out), K.ptr(tape), tape.numel(),
                                          K.ptr(ws), ws.numel(), st), h)
    gbuf = torch.zeros(int(lib.mn_model_grad_floats(mh)), device=DEV)
    bws = torch.zeros(lay[K.TCL['BWD_BYTES']], device=DEV, dtype=torch.uint8)
    assert bws.data_ptr() % 256 == 0
    g = K.f32c(cot.to(DEV))
    K.check(lib.mn_model_backward_tc(h, mh, B, 1, K.ptr(g), K.ptr(tape), tape.numel(), K.ptr(gbuf), K.ptr(bws), bws.numel(), st), h)
    torch.cuda.synchronize()
    off = nat._offsets()
    grads = []
    for s, w in enumerate(net.weights):
        grads.append({k: gbuf[s * off['stride'] + off[k]:][:v.numel()].view(v.shape).double().cpu() for k, v in w.items()})
    return lay, tape.cpu(), bws.cpu(), grads


def captures(net, x, cot, noise, lay, tape, bws, grads):
    """One capture per sub-module that owns slots (tc_train_ref.check_stages) and the list of sub-modules that own none."""
    from mega_nerf_b200._cabi import TCL
    spec = net.spec
    L, layers, R = spec.layer_dim, spec.layers, spec.rgb_dim
    nt_all = lay[TCL['N_TILES']]
    routed = net.kind == 'mega'
    cnt = tape[lay[TCL['TAPE_COUNTERS']]:][:4096].contiguous().view(torch.int32)
    B = x.shape[0]
    if routed:
        n_slots = int(cnt[3 * MAX_SUB + 1])
        starts = [int(cnt[MAX_SUB + s]) for s in range(len(net.weights) + 1)]
        slot_row = tape[lay[TCL['TAPE_SLOT_ROW']]:][:nt_all * 512].contiguous().view(torch.int32).long()
        so = lay[TCL['TAPE_SLOT_W']]
        slot_w = tape[so:][:nt_all * 512].contiguous().view(torch.float32).double() if so >= 0 else None
    else:
        n_slots = B
        starts = [0, -(-B // 128) * 128]
        slot_row = torch.arange(nt_all * 128)
        slot_w = None
    n_tiles = -(-n_slots // 128)
    act_tile, x_tile = lay[TCL['ACT_TILE']], lay[TCL['X_TILE']]
    kpe, kaux = lay[TCL['KPE']], lay[TCL['KAUX']]
    nimg = lay[TCL['N_IMG']]
    imgs = [(lay[TCL['IMG'] + 2 * j], lay[TCL['IMG'] + 2 * j + 1]) for j in range(nimg)]
    xreg = images(tape, lay[TCL['TAPE_XREG']], x_tile, n_tiles, 0, kpe + kaux)
    act = [images(tape, lay[TCL['TAPE_ACT']], act_tile, n_tiles, o, c) for o, c in imgs]
    f32 = f32_blocks(tape, lay[TCL['TAPE_F32']], lay[TCL['F32_ROWS']], n_tiles)
    S = float(bws[lay[TCL['BWD_SCALE']]:][:4].contiguous().view(torch.float32))
    fused = lay[TCL['ENGINE']] == 1
    g32r = lay[TCL['G32_ROWS']]
    dz = {}
    if fused:
        gf32 = f32_blocks(bws, lay[TCL['BWD_GF32']], g32r, n_tiles)
        dz = {j: images(bws, lay[TCL['BWD_DZ']], act_tile, n_tiles, o, c) for j, (o, c) in enumerate(imgs)}
    else:
        assert n_tiles <= lay[TCL['BWD_HEAD_TILES']], 'the layer engine is checked with one tile group'
        gf32 = f32_blocks(bws, lay[TCL['BWD_GF32']], g32r, n_tiles)
        hc, gc = lay[TCL['HC']], lay[TCL['GC']]
        dz[layers + 1] = images(bws, lay[TCL['BWD_DZG']], gc * 256, n_tiles, 0, gc)
        for i in (0, 1):       # dZ of trunk layer i was written to ping-pong buffer (layers - i) % 2
            pp = lay[TCL['BWD_PP0'] if (layers - i) % 2 == 0 else TCL['BWD_PP1']]
            dz[i] = images(bws, pp, hc * 256, n_tiles, 0, hc)
    emb_k = lay[TCL['BWD_EMB_K']]
    n_sub = len(net.weights)
    emb = None
    if spec.appearance_dim > 0:
        emb = bws[lay[TCL['BWD_EMB']]:][:n_sub * spec.appearance_count * emb_k * 4].contiguous().view(torch.float32)
        emb = emb.view(n_sub, spec.appearance_count, emb_k).double()
    xd = x.double()
    caps, empty = [], []
    for s in range(n_sub):
        a, b = starts[s], min(starts[s + 1], n_tiles * 128)
        if b <= a:
            empty.append(s)
            continue
        b = -(-b // 128) * 128
        sl = slice(a, b)
        rr = slot_row[sl].clone()
        if not routed:
            rr[rr >= B] = -1
        slot = torch.arange(a, b)
        valid = (rr >= 0) & (slot < n_slots)
        ri = rr.clamp(min=0)
        cap = dict(valid=valid, x=torch.where(valid.view(-1, 1), xd[ri], torch.zeros_like(xd[ri])),
                   noise=torch.where(valid, noise.double().view(-1)[ri], torch.zeros(len(ri), dtype=torch.float64)),
                   go=torch.where(valid.view(-1, 1), cot.double()[ri], torch.zeros_like(cot.double()[ri])),
                   bw=slot_w[sl] if slot_w is not None else torch.ones(b - a, dtype=torch.float64),
                   xpe=xreg[sl, :kpe], xaux=xreg[sl, kpe:], img=[m[sl] for m in act],
                   sig=f32[sl, lay[TCL['F32_SIGMA']]], rgb=f32[sl, lay[TCL['F32_RGB']]:lay[TCL['F32_RGB']] + 3],
                   id=f32[sl, lay[TCL['F32_ID']]], S=S, gf32=gf32[sl], dz={j: z[sl] for j, z in dz.items()},
                   emb_sum=emb[s] if emb is not None else None, grads=grads[s])
        if not fused:
            want = T.seeded_chain(spec, {k: v.double() for k, v in net.weights[s].items()}, cap, S)
            cap['seed_grads'] = {k: (v, LAYER_TOL) for k, v in want.items()
                                 if not (k.startswith('xyz_encodings.0.') or k.startswith('xyz_encodings.1.'))}
        caps.append((s, cap))
    return caps, empty, S, fused


def check(net, x, cot, noise, name, expect_engine):
    lay, tape, bws, grads = run(net, x, cot, noise)
    from mega_nerf_b200._cabi import TCL
    assert lay[TCL['ENGINE']] == expect_engine, lay[TCL['ENGINE']]
    caps, empty, S, fused = captures(net, x, cot, noise, lay, tape, bws, grads)
    assert S == T.grad_scale(cot), (S, T.grad_scale(cot))        # bit-exact power of two
    rep = T.Report()
    for s, cap in caps:
        w = {k: v.double() for k, v in net.weights[s].items()}
        T.check_stages(net.spec, w, cap, fused, rep, tag=f'[{s}] ' if len(net.weights) > 1 else '')
    for s in empty:          # a sub-module that receives no rows gets gradients of exactly 0
        for k, v in grads[s].items():
            rep.exact(f'[{s}] no rows: {k}', v, torch.zeros_like(v))
    print(f'\n{name}: S = {S}\n{rep.text()}')
    assert not rep.failures(), rep.failures()
    return rep


def rows_and_grads(spec, n, seed, scale=1e-3):
    x = C_.nerf_rows(spec, n, seed)
    g = torch.Generator().manual_seed(seed + 1)
    cot = (torch.rand(n, spec.rgb_dim + 1, generator=g) - 0.3) * scale
    noise = torch.randn(n, 1, generator=g)
    if spec.appearance_dim > 0:      # uneven image ids: a third of the rows on 3 images, the rest spread
        ids = x[:, -1]
        ids[: n // 3] = (torch.arange(n // 3) % 3).float()
    return x, cot, noise


def make(spec, seed=21, relu_bias=True):
    net = O.make_net('nerf', spec, seed=seed)
    if not spec.shifted_softplus and relu_bias:
        net.weights[0]['sigma.bias'] = net.weights[0]['sigma.bias'] + 0.5
    return net


SPECS = {
    'fused256_app': (O.NerfSpec(), 1),
    'fused256_d12_sh2': (O.NerfSpec(layers=12, pos_dir_dim=0, rgb_dim=27), 1),
    'fused512': (O.NerfSpec(layer_dim=512, appearance_dim=0), 1),
    'layer768': (O.NerfSpec(layer_dim=768, appearance_dim=0), 2),
    'layer2048_sh4': (O.NerfSpec(layer_dim=2048, pos_dir_dim=0, rgb_dim=75), 2),
    'layer384': (O.NerfSpec(layer_dim=384, appearance_dim=0), 2),
    'bg256': (O.NerfSpec(xyz_dim=4, shifted_softplus=False, skip_layers=(2, 5)), 1),
}


@pytest.mark.parametrize('n', [1, 127, 129])
@pytest.mark.parametrize('vname', list(SPECS))
def test_stages(vname, n):
    spec, engine = SPECS[vname]
    x, cot, noise = rows_and_grads(spec, n, 31 + n)
    check(make(spec), x, cot, noise, f'{vname}[{n}]', engine)


@pytest.mark.parametrize('vname', ['fused256_app', 'layer384'])
def test_stages_many_tiles(vname):
    """More rows than 3 x SMs x 128 on the fused engine (every wgrad chunk of several tiles); a full tile group of the layer
    engine with a ragged last weight-gradient chunk."""
    spec, engine = SPECS[vname]
    n = 3 * torch.cuda.get_device_properties(DEV).multi_processor_count * 128 + 77 if engine == 1 else 384 * 128 - 5
    x, cot, noise = rows_and_grads(spec, n, 7)
    check(make(spec), x, cot, noise, f'{vname}[{n}]', engine)


@pytest.mark.parametrize('mname', ['hard2d', 'blend2d'])
def test_stages_routed(mname):
    """MegaNeRF: hard routing (margin 1) with a sub-module that receives no rows, and blending (1.15) with slot weights."""
    net = C_.mega_net(mname, layer_dim=256)
    x = C_.mega_rows(net, 3000, 13)
    if mname == 'hard2d':    # drop the rows of the last centroid's cell: that sub-module owns no slot
        assign, _ = O.route(net, x)
        x = x[assign != len(net.weights) - 1]
    g = torch.Generator().manual_seed(6)
    cot = (torch.rand(x.shape[0], 4, generator=g) - 0.5) * 1e-4
    noise = torch.rand(x.shape[0], 1, generator=g)
    check(net, x, cot, noise, mname, 1)


@pytest.mark.parametrize('edge', ['zero_grad', 'outlier', 'tiny_preact'])
def test_edges(edge):
    spec, _ = SPECS['fused256_app']
    net = make(spec)
    x, cot, noise = rows_and_grads(spec, 640, 3)
    if edge == 'zero_grad':
        cot = torch.zeros_like(cot)
    elif edge == 'outlier':   # one row 2^12 above the rest: small dZ go subnormal or to zero in fp16
        cot[17] *= 4096.0
    else:                     # pre-activations in (0, 2^-25): fp16 mask 0 while the fp32 ReLU' is 1
        w = net.weights[0]
        for i in (2, 6):
            w[f'xyz_encodings.{i}.0.weight'][:40] = 0.0
            w[f'xyz_encodings.{i}.0.bias'][:40] = 2.0 ** -27
    rep = check(net, x, cot, noise, edge, 1)
    if edge == 'zero_grad':
        assert all((v == 0).all() for v in run(net, x, cot, noise)[3][0].values())
    if edge == 'tiny_preact':
        assert any(r['stage'].startswith('dZ_2 zero') and r['n'] > 0 for r in rep.rows)


def test_trained_like_weights_stress():
    """The amplification of tests/test_gpu_parity.py::test_trained_like_weights_stress (weights scaled up): S |dZ| stays below
    the fp16 maximum at every stage, and every stage holds its bound."""
    spec = O.NerfSpec()
    net = make(spec)
    w = net.weights[0]
    for k in w:
        if k.endswith('weight') and k.startswith('xyz_encodings'):
            w[k] = w[k] * 1.6
    x, cot, noise = rows_and_grads(spec, 640, 9, scale=1.0)
    rep = check(net, x, cot, noise, 'stress', 1)
    assert all(r['fail'] == 0 for r in rep.rows if 'below fp16 max' in r['stage'])
