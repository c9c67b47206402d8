"""CPU: the training programs of the tensor-core MLP kernel (csrc/mn_mlp_wg.cuh) for the 11- and 12-layer networks at 256 and
512 wide, read through the host-only hook mn_debug_tp_program_mode.  tc_f16 training runs these depths on the fused kernel in two
launches per step: the recording forward (tc_mlp_wg_kernel<PP_TRAIN_FWD>, the forward plan in a layout with the activation image
in shared memory) and the data-gradient chain of the backward (tc_mlp_wg_kernel<PP_DGRAD>, one GEMM per Linear from
dir_a_encoding down to trunk layer 1 on the transposed weight images).  Each program must stream its weight plane exactly once
per tile and feed every accumulator its whole K range in order, and the barrier protocol (tests/tp_protocol_sim.py) must neither
deadlock nor read a stale ring stage, at the ring depth the launcher picks and at the smallest one it accepts (2 stages).

The shapes are the reference's `--layers 11` / `--layers 12` with `--skip_layers 4` or `4 8`, at the default width (256) and
BASELINE configs[3]'s (512), with the colour head (direction + appearance), the SH degree 2 head of mega-nerf-sh-3 and the
background network's (xyz_dim 4)."""
import ctypes as C

import pytest

import tp_protocol_sim as S
from mega_nerf_b200 import _cabi as K
from test_tp_program import WS_CHUNK_FIRST, WS_CHUNK_LAST, WS_FROM_X, WS_LO, WS_X_FIRST, desc

MN_TP_INFER, MN_TP_TRAIN_FWD, MN_TP_DGRAD = 0, 1, 2
MN_ERR_UNSUPPORTED = 6
SMEM_MAX = 227 * 1024

HEADS = {
    'rgb_app': dict(),
    'sh2': dict(pos_dir_dim=0, rgb_dim=27),
    'bg': dict(xyz_dim=4),
}
SKIPS = {'skip4': (4,), 'skip4_8': (4, 8)}
DEEP = [(w, n, s, h) for w in (256, 512) for n in (11, 12) for s in SKIPS for h in HEADS]


def deep_desc(width, layers, skips, head):
    d = desc(layer_dim=width, layers=layers, skips=SKIPS[skips], **{k: v for k, v in HEADS[head].items() if k != 'xyz_dim'})
    d.xyz_dim = HEADS[head].get('xyz_dim', 3)
    return d


def program_mode(d, mode):
    """-> (rc, entries, info) of one launch of the kernel (entries as in test_tp_program.program)."""
    cap = 8192
    tab = (C.c_uint * (8 * cap))()
    info = (C.c_int * 8)()
    rc = K.lib().mn_debug_tp_program_mode(C.byref(d), mode, tab, cap, info)
    if rc != 0:
        return rc, None, None
    keys = ('w_off', 'w_bytes', 'nw', 'kc', 'a_col', 'x_off', 'x_bytes', 'code')
    ent = []
    for i in range(info[0]):
        e = dict(zip(keys, (tab[8 * i + j] for j in range(8))))
        e['flags'], e['gemm'], e['chunk'] = e['code'] & 0xFF, (e['code'] >> 8) & 0xFF, e['code'] >> 16
        ent.append(e)
    return rc, ent, list(info)


def check_stream(prog, info):
    """Every weight slab fits a ring stage and the slabs tile the weight plane; every accumulator (GEMM, N-chunk) is opened and
    closed once and walks its K range in order."""
    n, n_t, plane_bytes, stages, smem, x_tile, stage_bytes, slab = info
    assert len(prog) == n and 2 <= stages and smem <= SMEM_MAX
    for e in prog:
        assert e['kc'] % 16 == 0 and 16 <= e['kc'] <= slab and e['w_bytes'] == e['kc'] * e['nw'] * 2 <= stage_bytes
        assert not e['flags'] & WS_LO
    spans = sorted((e['w_off'], e['w_off'] + e['w_bytes']) for e in prog)
    assert spans[0][0] == 0 and spans[-1][1] == plane_bytes
    assert all(a1 == b0 for (_, a1), (b0, _) in zip(spans, spans[1:])), 'gap or overlap in the weight image'
    open_acc = None
    for e in prog:
        key = (e['gemm'], e['chunk'])
        if e['flags'] & WS_CHUNK_FIRST:
            assert open_acc is None
            open_acc, h_seen = key, 0
        assert open_acc == key
        if not e['flags'] & WS_FROM_X:                              # the activation segment, walked from column 0 in order
            assert e['a_col'] == h_seen, (key, e['a_col'], h_seen)
            h_seen += e['kc']
        if e['flags'] & WS_CHUNK_LAST:
            open_acc = None
    assert open_acc is None


@pytest.mark.parametrize('width,layers,skips,head', DEEP)
def test_recording_forward_streams_the_inference_program(width, layers, skips, head):
    """The recording forward runs the inference plan: the same ring traffic, entry for entry, in the training variant's
    layout (the activation image in shared memory, so a shallower ring at 256 wide)."""
    d = deep_desc(width, layers, skips, head)
    rc, prog_i, info_i = program_mode(d, MN_TP_INFER)
    rc_t, prog, info = program_mode(d, MN_TP_TRAIN_FWD)
    assert rc == 0 and rc_t == 0
    assert prog == prog_i and info[:3] == info_i[:3] and info[5:] == info_i[5:]
    check_stream(prog, info)
    assert len({e['gemm'] for e in prog}) == layers + 3             # trunk, xyz_encoding_final, dir_a_encoding, rgb
    # PE at layer 0 and each skip layer (once per 256-column chunk of the GEMM), direction + appearance at dir_a_encoding
    # (L / 2 <= 256 outputs: one chunk)
    assert sum(1 for e in prog if e['flags'] & WS_X_FIRST) == (len(SKIPS[skips]) + 1) * (width // 256) + 1


@pytest.mark.parametrize('width,layers,skips,head', DEEP)
def test_data_gradient_program(width, layers, skips, head):
    """One GEMM per Linear from dir_a_encoding down to trunk layer 1, N = layer_dim (two 256-column chunks at 512), K = the
    Linear's output columns (L / 2 for dir_a_encoding, L otherwise), A always from the activation image."""
    rc, prog, info = program_mode(deep_desc(width, layers, skips, head), MN_TP_DGRAD)
    assert rc == 0
    check_stream(prog, info)
    assert info[1] == info[0] and info[5] == 0                      # no sigma_only form, no feature tile
    gemms = sorted({e['gemm'] for e in prog})
    assert gemms == list(range(layers + 1))
    for gi in gemms:
        es = [e for e in prog if e['gemm'] == gi]
        assert {e['chunk'] for e in es} == set(range(width // 256))
        k = width // 2 if gi == 0 else width
        for ch in range(width // 256):
            assert sum(e['kc'] for e in es if e['chunk'] == ch) == k
    assert not any(e['flags'] & (WS_FROM_X | WS_X_FIRST) for e in prog)
    assert info[2] == 2 * width * (width // 2 + layers * width)      # the transposed images, fp16


@pytest.mark.parametrize('mode', [MN_TP_TRAIN_FWD, MN_TP_DGRAD])
@pytest.mark.parametrize('width,layers,skips,head', [s for s in DEEP if s[3] != 'bg'])
@pytest.mark.parametrize('odd_tail', [False, True])
def test_training_protocol_no_deadlock_no_stale_read(width, layers, skips, head, mode, odd_tail):
    """The barrier protocol under randomised timing, at the launcher's ring depth and at the smallest ring it accepts.  (The
    background head changes only the feature tile's contents, not the program: it is covered by the two tests above.)"""
    rc, prog, info = program_mode(deep_desc(width, layers, skips, head), mode)
    assert rc == 0
    n_tiles = 3 if odd_tail else 4
    for seed in range(2):
        S.simulate(prog, info[3], n_tiles=n_tiles, seed=seed)
    S.simulate(prog, 2, n_tiles=n_tiles, seed=11)


@pytest.mark.parametrize('width', [256, 512])
def test_training_ring_depth(width):
    """The fp32 block the consumers stage (bias_stride floats per GEMM, then sigma_w) grows with depth and takes shared memory
    from the weight ring: at 256 wide the recording forward keeps 4 stages up to 10 layers and 3 at 11 and 12; at 512, 3 up to
    11 layers and 2 at 12.  The data-gradient chain stages no feature tile and a depth-independent block (sigma_w, rgb_w)."""
    want_fwd = {256: {8: 4, 10: 4, 11: 3, 12: 3}, 512: {8: 3, 10: 3, 11: 3, 12: 2}}[width]
    dgrad = set()
    for layers, stages in want_fwd.items():
        d = desc(layer_dim=width, layers=layers, skips=(4, 8) if layers > 8 else (4,))
        assert program_mode(d, MN_TP_TRAIN_FWD)[2][3] == stages, (width, layers)
        dgrad.add(program_mode(d, MN_TP_DGRAD)[2][3])
    assert len(dgrad) == 1 and min(dgrad) >= 4


@pytest.mark.parametrize('layers,fused', [(2, True), (10, True), (11, True), (12, True), (13, False), (16, False)])
@pytest.mark.parametrize('width', [256, 512])
def test_depth_boundary_of_the_fused_training_kernel(width, layers, fused):
    """Up to 12 layers the fused kernel trains (and renders) the network; from 13 on both go to the layer-GEMM engine, for
    which the hook returns MN_ERR_UNSUPPORTED."""
    d = desc(layer_dim=width, layers=layers, skips=(4, 8) if layers > 8 else (1,) if layers == 2 else (4,))
    for mode in (MN_TP_INFER, MN_TP_TRAIN_FWD, MN_TP_DGRAD):
        rc = program_mode(d, mode)[0]
        assert (rc == 0) == fused and rc in (0, MN_ERR_UNSUPPORTED), (mode, rc)


@pytest.mark.parametrize('layers', [11, 12])
@pytest.mark.parametrize('shape', ['affine', 'nodir', 'w128', 'single_layer'])
def test_uncovered_shapes_have_no_training_program(shape, layers):
    """Affine appearance, heads without dir_a_encoding, widths below 256 and one-layer networks stay off tensor-core training
    at every depth: the fused kernel renders them (inference program) but has no training program for them."""
    kw = dict(affine=dict(affine=1), nodir=dict(pos_dir_dim=0, appearance_dim=0), w128=dict(layer_dim=128),
              single_layer=dict(layers=1, skips=()))[shape]
    d = desc(**{'layers': layers, 'skips': (4, 8), **kw})
    assert program_mode(d, MN_TP_INFER)[0] == 0
    assert program_mode(d, MN_TP_TRAIN_FWD)[0] == MN_ERR_UNSUPPORTED
    assert program_mode(d, MN_TP_DGRAD)[0] == MN_ERR_UNSUPPORTED


def test_mode_out_of_range_is_invalid():
    assert program_mode(desc(), 3)[0] == 1 and program_mode(desc(), -1)[0] == 1
