"""CPU: invariants of the stage program of the tensor-core MLP kernel (csrc/mn_mlp_wg.cuh), read through the host-only test hook
mn_debug_tp_program.  The TMA producer and both consumer warpgroups walk this program (wg_walk_chunk), one entry per weight-ring
stage: it must stream every weight image exactly once per tile, feed every accumulator the whole K range of its GEMM in order,
load every feature segment before the stages that read it, and fit the ring in shared memory.  The kernel follows
models/nerf.py:115-160 (the Linear chain of one NeRF); the shapes below are the reference's configs (configs/mega-nerf/*.yaml:
8 x 256 with a skip at 4) plus the narrower / SH / no-direction / 512-wide variants the parity tests use."""
import ctypes as C

import pytest

from mega_nerf_b200 import _cabi as K

WS_FROM_X, WS_X_FIRST, WS_X_LAST, WS_LO, WS_CHUNK_FIRST, WS_CHUNK_LAST = 1, 2, 4, 8, 16, 32


def desc(layer_dim=256, layers=8, skips=(4,), pos_dir_dim=4, appearance_dim=48, rgb_dim=3, affine=0, pos_xyz_dim=12):
    d = K.ModelDesc()
    d.kind, d.n_sub = 0, 1
    d.pos_xyz_dim, d.pos_dir_dim = pos_xyz_dim, pos_dir_dim
    d.layers, d.layer_dim = layers, layer_dim
    d.appearance_dim, d.affine_appearance, d.appearance_count = appearance_dim, affine, 100
    d.rgb_dim, d.xyz_dim, d.shifted_softplus = rgb_dim, 3, 1
    d.n_skip = len(skips)
    for i, s in enumerate(skips):
        d.skip_layers[i] = s
    d.boundary_margin, d.xyz_real, d.cluster_dim_start = 1.0, 1, 1
    return d


def program(d):
    """-> (rc, entries, entries of a sigma_only call, info); an entry is a dict of the hook's eight fields."""
    cap = 4096
    tab = (C.c_uint * (8 * cap))()
    info = (C.c_int * 8)()
    rc = K.lib().mn_debug_tp_program(C.byref(d), tab, cap, info)
    if rc != 0:
        return rc, None, None, None
    keys = ('w_off', 'w_bytes', 'nw', 'kc', 'a_col', 'x_off', 'x_bytes', 'code')
    ent = []
    for i in range(info[0]):
        e = dict(zip(keys, (tab[8 * i + j] for j in range(8))))
        e['flags'], e['gemm'], e['chunk'] = e['code'] & 0xFF, (e['code'] >> 8) & 0xFF, e['code'] >> 16
        ent.append(e)
    return rc, ent, ent[:info[1]], list(info)


SHAPES = {
    'c2_8x256': dict(),
    'sh_head': dict(pos_dir_dim=0, appearance_dim=0, rgb_dim=27),
    'narrow_64': dict(layer_dim=64, layers=4, skips=(2,)),
    'narrow_128': dict(layer_dim=128, layers=4, skips=()),
    'w192': dict(layer_dim=192, layers=3, skips=(1,)),
    'no_appearance': dict(appearance_dim=0),
    'pe16': dict(pos_xyz_dim=16),                 # 99 encoding columns -> a 112-column feature segment
    'deep_12': dict(layers=12, skips=(4, 8)),
    'wide_512': dict(layer_dim=512),              # every GEMM in two N = 256 chunks
}


@pytest.mark.parametrize('name', sorted(SHAPES))
def test_tables_describe_the_same_ring_traffic(name):
    rc, prog, prog_t, info = program(desc(**SHAPES[name]))
    assert rc == 0
    n, n_t, plane_bytes, stages, smem, x_tile, stage_bytes, slab = info
    assert 0 < n_t < n and len(prog) == n
    assert stages >= 2 and smem <= 227 * 1024
    # a sigma_only call runs the trunk GEMMs only: a prefix of the program
    assert {e['gemm'] for e in prog_t} == set(range(max(e['gemm'] for e in prog_t) + 1))
    assert all(e['gemm'] > prog_t[-1]['gemm'] for e in prog[n_t:])
    # weight slabs: each fits a ring stage, inside the plane, non-overlapping, covering the plane completely
    for e in prog:
        assert e['kc'] % 16 == 0 and 16 <= e['kc'] <= slab and e['w_bytes'] == e['kc'] * e['nw'] * 2 <= stage_bytes
        assert e['nw'] % 8 == 0 and 8 <= e['nw'] <= 256 and not e['flags'] & WS_LO      # tc_f16: one pass, hi planes
    spans = sorted((e['w_off'], e['w_off'] + e['w_bytes']) for e in prog)
    assert spans[0][0] == 0 and spans[-1][1] == plane_bytes
    for (a0, a1), (b0, b1) in zip(spans, spans[1:]):
        assert a1 == b0, 'gap or overlap in the weight image'
    # every accumulator (GEMM, N-chunk) is opened by exactly one first stage and closed by one last stage, and its stages
    # walk the K range of each operand segment in order; feature segments are loaded by their first stage and released by
    # their last one, and lie inside the tile's feature record
    open_acc, x_open, x_cols, x_seen = None, False, 0, 0
    for e in prog:
        key = (e['gemm'], e['chunk'])
        if e['flags'] & WS_CHUNK_FIRST:
            assert open_acc is None
            open_acc, col = key, 0
        assert open_acc == key
        if e['flags'] & WS_FROM_X:
            if e['flags'] & WS_X_FIRST:
                assert not x_open and e['a_col'] == 0 and e['x_bytes'] > 0 and e['x_off'] + e['x_bytes'] <= x_tile
                x_open, x_cols, x_seen = True, e['x_bytes'] // (128 * 2), 0
            assert x_open and e['a_col'] == x_seen
            x_seen += e['kc']
            assert x_seen <= x_cols
            if e['flags'] & WS_X_LAST:
                assert x_seen == x_cols
                x_open = False
        else:
            assert not x_open and e['x_bytes'] == 0
        if e['flags'] & WS_CHUNK_LAST:
            assert not x_open
            open_acc = None
    assert open_acc is None and not x_open


def test_c2_counts():
    """8 x 256 with a skip at 4: 11 GEMMs in 44 ring stages of 64 K-columns per tile (32 for a sigma_only call), one weight
    plane = every Linear of the network in fp16."""
    rc, prog, prog_t, info = program(desc())
    assert rc == 0 and len(prog) == 44 and len(prog_t) == 32 and info[7] == 64
    assert len({e['gemm'] for e in prog}) == 11
    assert sum(1 for e in prog if e['flags'] & WS_X_FIRST) == 3                 # PE for layers 0 and 4, direction + appearance
    assert info[2] == 2 * (80 * 256 + 3 * 256 * 256 + (80 + 256) * 256 + 3 * 256 * 256 + 256 * 256 + (256 + 80) * 128 + 128 * 32)


def test_unsupported_shapes_are_refused():
    assert program(desc(layer_dim=96))[0] != 0           # not a multiple of 64: fp32 kernels only
    assert program(desc(layer_dim=1024))[0] != 0         # wider than the 512-wide form of the kernel
    assert program(desc(rgb_dim=48, pos_dir_dim=0, appearance_dim=0))[0] != 0    # rgb head wider than one N = 32 MMA
