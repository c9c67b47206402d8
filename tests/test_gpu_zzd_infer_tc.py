"""GPU: tensor-core inference (precision 'tc_f16') element by element, through the recording forward.

For each case the same rows go through two calls: mn_model_forward at tc_f16 (the inference kernel: activations in registers
up to 256 wide) and mn_debug_tc_forward_record (the recording forward, same plan, packed weights, encoder, GEMM K order and
epilogue arithmetic) on a tape this test owns.  Then:
  - the two outputs are equal bit for bit over every row (the register-A and shared-memory-A forms of wgmma give the same fp32
    results for the same operands in the same K order), and a sigma_only call equals the sigma column of the full call;
  - the recording's encoder tiles, every activation image, the fp32 head block (tc_train_ref.check_forward) and `out`
    (check_output: sigma activation, colour / SH / affine head, blend weight and the ascending-sub-module combine) are checked
    against the float64 restatement, each stage seeded from the kernel's own previous image, so no bound grows with depth.
Large unrouted calls are checked on chosen tiles: the first, the ragged last, the last of the first round of the persistent
tile loop and the first of the second, and on the layer engine the tiles on each side of a tile-group boundary."""
import ctypes as C

import pytest
import torch

import cases as C_
import tc_train_ref as T
from oracle import mn_oracle as O
from test_gpu_parity import DEV, product_net

pytestmark = pytest.mark.gpu

MAX_SUB = 64          # MN_MAX_SUB: counters[MAX_SUB + s] is the first slot of sub-module s, counters[3 MAX_SUB + 1] the slot count
GROUP_TILES = 384     # kLgGroupTiles: tiles per launch group of the layer engine


def images_at(buf, base, tile_bytes, tiles, off, cols):
    """[len(tiles) * 128, cols] float64 of the fp16 tile images [cols/8][128][8] at base + t tile_bytes + off, t in tiles."""
    t = buf[base:base + (int(tiles.max()) + 1) * tile_bytes].view(-1, tile_bytes)[tiles.to(buf.device)][:, off:off + cols * 256]
    t = t.contiguous().cpu().view(torch.float16).view(len(tiles), cols // 8, 128, 8)
    return t.permute(0, 2, 1, 3).reshape(len(tiles) * 128, cols).double()


def f32_at(buf, base, rows, tiles):
    """[len(tiles) * 128, rows] of the fp32 blocks [tiles][rows][128] at base."""
    t = buf[base:base + (int(tiles.max()) + 1) * rows * 512].view(-1, rows * 512)[tiles.to(buf.device)].contiguous().cpu()
    return t.view(torch.float32).view(len(tiles), rows, 128).permute(0, 2, 1).reshape(len(tiles) * 128, rows)


def run(net, x, noise):
    """-> (layout, tape on the device, inference out, recording out, sigma_only out), all rows."""
    from mega_nerf_b200 import _cabi as K
    from mega_nerf_b200.modules import _rows_matrix
    lib = K.lib()
    nat = product_net(net)._native()
    h = nat.sync(DEV)
    mh = nat.handle
    B = x.shape[0]
    lay = (C.c_int64 * 256)()
    n = lib.mn_debug_tc_train_layout(mh, B, lay, 256)
    assert n > 0, n
    lay = list(lay)[:n]
    R = net.spec.rgb_dim
    st = K.stream_of(DEV)
    nz = noise.to(DEV).contiguous().view(-1) if noise is not None else None
    rows, xin = _rows_matrix(x.to(DEV))
    rows_s, xin_s = _rows_matrix(x[:, :net.spec.xyz_dim].contiguous().to(DEV))
    ws = torch.empty(max(int(lib.mn_model_workspace_bytes(mh, B, K.PREC_TC_F16)), 256), device=DEV, dtype=torch.uint8)
    out_inf = torch.full((B, R + 1), float('nan'), device=DEV)
    K.check(lib.mn_model_forward(h, mh, C.byref(rows), B, 1, 0, K.ptr(nz), K.PREC_TC_F16, K.ptr(out_inf), K.ptr(ws), ws.numel(), st), h)
    out_sig = torch.full((B, 1), float('nan'), device=DEV)
    K.check(lib.mn_model_forward(h, mh, C.byref(rows_s), B, 1, 1, K.ptr(nz), K.PREC_TC_F16, K.ptr(out_sig), K.ptr(ws), ws.numel(),
                                 st), h)
    ws_rec = torch.empty(max(int(lib.mn_model_workspace_bytes(mh, B, K.PREC_FP32)), 256), device=DEV, dtype=torch.uint8)
    tape = torch.zeros(lay[K.TCL['TAPE_BYTES']], device=DEV, dtype=torch.uint8)
    out_rec = torch.full((B, R + 1), float('nan'), device=DEV)
    K.check(lib.mn_debug_tc_forward_record(h, mh, C.byref(rows), B, 1, K.ptr(nz), K.ptr(out_rec), K.ptr(tape), tape.numel(),
                                           K.ptr(ws_rec), ws_rec.numel(), st), h)
    torch.cuda.synchronize()
    return lay, tape, out_inf.cpu(), out_rec.cpu(), out_sig.cpu()


def chosen_tiles(n_tiles, engine, n_sm):
    """The tiles a large unrouted call is checked on."""
    want = {0, 1, n_tiles - 1, n_sm - 1, n_sm}
    if engine == 2:
        for g in range(GROUP_TILES, n_tiles, GROUP_TILES):
            want |= {g - 1, g}
    return torch.tensor(sorted(t for t in want if 0 <= t < n_tiles))


def check(net, x, noise, name, expect_engine, all_tiles=True):
    from mega_nerf_b200._cabi import TCL
    lay, tape, out_inf, out_rec, out_sig = run(net, x, noise)
    spec = net.spec
    R, B = spec.rgb_dim, x.shape[0]
    assert lay[TCL['ENGINE']] == expect_engine, lay[TCL['ENGINE']]
    # ---- inference == recording, bit for bit, every row (NaN-free: NaN != NaN would hide nothing here)
    assert not torch.isnan(out_rec).any()
    diff = (out_inf != out_rec).any(1)
    assert torch.equal(out_inf, out_rec), f'{int(diff.sum())} rows differ, first {diff.nonzero()[:8].view(-1).tolist()}'
    assert torch.equal(out_sig[:, 0], out_inf[:, R]), 'sigma_only call != sigma column of the full call'

    routed = net.kind == 'mega'
    cnt = tape[lay[TCL['TAPE_COUNTERS']]:][:4096].cpu().view(torch.int32)
    nt_all = lay[TCL['N_TILES']]
    n_sub = len(net.weights)
    if routed:
        n_slots = int(cnt[3 * MAX_SUB + 1])
        starts = [int(cnt[MAX_SUB + s]) for s in range(n_sub + 1)]
        slot_row = tape[lay[TCL['TAPE_SLOT_ROW']]:][:nt_all * 512].cpu().view(torch.int32).long()
        so = lay[TCL['TAPE_SLOT_W']]
        slot_w = tape[so:][:nt_all * 512].cpu().view(torch.float32) if so >= 0 else None
    else:
        n_slots = B
        starts = [0, nt_all * 128]
        slot_row = torch.arange(nt_all * 128)
        slot_row[slot_row >= B] = -1
        slot_w = None
    n_tiles = -(-n_slots // 128)
    tiles = torch.arange(n_tiles) if all_tiles else \
        chosen_tiles(n_tiles, expect_engine, torch.cuda.get_device_properties(DEV).multi_processor_count)
    assert routed is False or all_tiles, 'routed calls are checked on every tile (output rows gather several sub-modules)'
    act_tile, x_tile = lay[TCL['ACT_TILE']], lay[TCL['X_TILE']]
    kpe, kaux = lay[TCL['KPE']], lay[TCL['KAUX']]
    nimg = lay[TCL['N_IMG']]
    assert nimg == (spec.layers + 2 if spec.has_dir_a else spec.layers)
    xreg = images_at(tape, lay[TCL['TAPE_XREG']], x_tile, tiles, 0, kpe + kaux)
    act = [images_at(tape, lay[TCL['TAPE_ACT']], act_tile, tiles, lay[TCL['IMG'] + 2 * j], lay[TCL['IMG'] + 2 * j + 1])
           for j in range(nimg)]
    f32 = f32_at(tape, lay[TCL['TAPE_F32']], lay[TCL['F32_ROWS']], tiles)
    slots = (tiles.view(-1, 1) * 128 + torch.arange(128)).view(-1)
    sub_of = torch.searchsorted(torch.tensor(starts[1:n_sub]), slots, right=True) if routed else torch.zeros_like(slots)
    xd = x.double()
    nzd = noise.double().view(-1) if noise is not None else torch.zeros(B, dtype=torch.float64)
    fused = expect_engine == 1
    rep = T.Report()
    pieces = []
    for s in range(n_sub):
        sel = (sub_of == s).nonzero().view(-1)
        if len(sel) == 0:
            continue
        rr = slot_row[slots[sel]]
        valid = (rr >= 0) & (slots[sel] < n_slots)
        ri = rr.clamp(min=0)
        cap = dict(valid=valid, x=torch.where(valid.view(-1, 1), xd[ri], torch.zeros_like(xd[ri])),
                   noise=torch.where(valid, nzd[ri], torch.zeros(len(ri), dtype=torch.float64)),
                   xpe=xreg[sel, :kpe], xaux=xreg[sel, kpe:], img=[m[sel] for m in act],
                   sig=f32[sel, lay[TCL['F32_SIGMA']]].double(), rgb=f32[sel, lay[TCL['F32_RGB']]:lay[TCL['F32_RGB']] + 3].double(),
                   id=f32[sel, lay[TCL['F32_ID']]].double())
        w = {k: v.double() for k, v in net.weights[s].items()}
        tag = f'[{s}] ' if n_sub > 1 else ''
        T.check_forward(spec, w, cap, fused, rep, tag)
        pieces.append((rr[valid], slot_w[slots[sel]][valid] if slot_w is not None else None, T.slot_outputs(spec, w, cap, fused)))
    # ---- output assembly over the rows whose slots were all checked (every row unless tiles were chosen)
    rows_chk = torch.unique(torch.cat([p[0] for p in pieces]))
    if all_tiles:
        assert len(rows_chk) == B
    index = torch.full((B,), -1, dtype=torch.long)
    index[rows_chk] = torch.arange(len(rows_chk))
    T.check_output(spec, out_rec[rows_chk], [(index[r], bw, so) for r, bw, so in pieces], rep)
    print(f'\n{name}: {B} rows, {len(tiles)} of {n_tiles} tiles checked\n{rep.text()}')
    assert not rep.failures(), rep.failures()
    return rep


def make(spec, seed=21):
    net = O.make_net('nerf', spec, seed=seed)
    if not spec.shifted_softplus:        # the random-init ReLU density head is dead: lift its bias
        net.weights[0]['sigma.bias'] = net.weights[0]['sigma.bias'] + 0.5
    return net


def rows_and_noise(spec, n, seed, noise=True):
    x = C_.nerf_rows(spec, n, seed)
    if spec.appearance_dim > 0:      # uneven image ids: a third of the rows on 3 images, the rest spread
        x[: n // 3, -1] = (torch.arange(n // 3) % 3).float()
    return x, torch.randn(n, 1, generator=torch.Generator().manual_seed(seed + 1)) if noise else None


_G = dict(layer_dim=64, appearance_count=10)
SPECS = {                # name: (spec, engine)
    'fused64': (O.NerfSpec(**_G), 1),
    'fg128_l4': (O.NerfSpec(layer_dim=128, layers=4, skip_layers=(2,)), 1),
    'fused192': (O.NerfSpec(layer_dim=192), 1),
    'fused256_app': (O.NerfSpec(), 1),
    'fused256_d12_sh2': (O.NerfSpec(layers=12, pos_dir_dim=0, rgb_dim=27), 1),
    'affine': (O.NerfSpec(affine_appearance=True), 1),
    'affine64': (O.NerfSpec(affine_appearance=True, **_G), 1),
    'nodir_noapp': (O.NerfSpec(pos_dir_dim=0, appearance_dim=0), 1),
    'noapp_q1': (O.NerfSpec(appearance_dim=0), 1),
    'relu_sigma': (O.NerfSpec(shifted_softplus=False), 1),
    'bg256': (O.NerfSpec(xyz_dim=4), 1),
    'sh2': (O.NerfSpec(pos_dir_dim=0, rgb_dim=27), 1),
    'fused512': (O.NerfSpec(layer_dim=512), 1),
    'layer96': (O.NerfSpec(layer_dim=96), 2),
    'layer160': (O.NerfSpec(layer_dim=160), 2),
    'layer160_nodir': (O.NerfSpec(layer_dim=160, pos_dir_dim=0, appearance_dim=0), 2),
    'layer384': (O.NerfSpec(layer_dim=384, appearance_dim=0), 2),
    'layer768': (O.NerfSpec(layer_dim=768, appearance_dim=0), 2),
    'layer2048_sh4': (O.NerfSpec(layer_dim=2048, pos_dir_dim=0, rgb_dim=75), 2),
}


@pytest.mark.parametrize('vname', list(SPECS))
def test_infer_equals_recording(vname):
    spec, engine = SPECS[vname]
    x, noise = rows_and_noise(spec, 200, 31)
    check(make(spec), x, noise, vname, engine)


@pytest.mark.parametrize('n', [1, 63, 64, 65, 127, 128, 129])
@pytest.mark.parametrize('vname', ['fused64', 'fused256_app'])
def test_row_counts(vname, n):
    """Rows 63 | 64 and 64 | 65 are the boundary between the two consumer warpgroups' rows of a tile."""
    spec, engine = SPECS[vname]
    x, noise = rows_and_noise(spec, n, 7 + n, noise=n % 2 == 1)
    check(make(spec), x, noise, f'{vname}[{n}]', engine)


@pytest.mark.parametrize('vname', ['fused64', 'fused192', 'fused256_app', 'fused512', 'layer96'])
def test_many_tiles(vname):
    """The persistent tile loop (3 x SMs x 128 + 77 rows) on the fused engine; past one tile group on the layer engine."""
    spec, engine = SPECS[vname]
    sm = torch.cuda.get_device_properties(DEV).multi_processor_count
    n = 3 * sm * 128 + 77 if engine == 1 else GROUP_TILES * 128 + 77
    x, noise = rows_and_noise(spec, n, 5)
    check(make(spec), x, noise, f'{vname}[{n}]', engine, all_tiles=False)


@pytest.mark.parametrize('edge', ['dead_rows', 'tiny_preact'])
@pytest.mark.parametrize('vname', ['fused64', 'fused256_app', 'layer160'])
def test_edges(vname, edge):
    """dead_rows: trunk layer 0's pre-activations are x (all negative where x < 0), so H0 is all zero on about half the rows.
    tiny_preact: 40 channels of layers 1 and 2 have the pre-activation 2^-27, below fp16's smallest subnormal (rounds to 0)."""
    spec, engine = SPECS[vname]
    net = make(spec)
    w = net.weights[0]
    if edge == 'dead_rows':
        w['xyz_encodings.0.0.weight'] = torch.zeros_like(w['xyz_encodings.0.0.weight'])
        w['xyz_encodings.0.0.weight'][:, 0] = 1.0
        w['xyz_encodings.0.0.bias'] = torch.zeros_like(w['xyz_encodings.0.0.bias'])
    else:
        for i in (1, 2):
            w[f'xyz_encodings.{i}.0.weight'][:40] = 0.0
            w[f'xyz_encodings.{i}.0.bias'][:40] = 2.0 ** -27
    x, noise = rows_and_noise(spec, 300, 11)
    check(net, x, noise, f'{vname} {edge}', engine)


@pytest.mark.parametrize('mname', ['hard2d', 'blend2d', 'blend25'])
def test_routed(mname):
    """MegaNeRF: hard routing (margin 1) with a sub-module that receives no rows; blending (1.15); and 25 blended sub-modules
    over more tiles than 3 x SMs, so every CTA runs tiles of several sub-modules and restages the fp32 block."""
    net = C_.mega_net(mname)
    n = 3000
    if mname == 'blend25':
        n = 3 * torch.cuda.get_device_properties(DEV).multi_processor_count * 128
    x = C_.mega_rows(net, n, 13)
    if mname == 'hard2d':    # drop the rows of the last centroid's cell: that sub-module owns no slot
        assign, _ = O.route(net, x)
        x = x[assign != len(net.weights) - 1]
    noise = torch.rand(x.shape[0], 1, generator=torch.Generator().manual_seed(6))
    check(net, x, noise, mname, 1)
