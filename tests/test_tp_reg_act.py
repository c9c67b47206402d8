"""CPU: shared-memory layout of the tc_f16 inference launch of the tensor-core MLP kernel (csrc/mn_mlp_wg.cuh), as the host-only
hook mn_debug_tp_program reports it.  Up to 256 wide each consumer warpgroup keeps its activations in registers (the A operand
of the register form of wgmma), so the layout has no activation image and the weight ring takes its place; the 512-wide kernel
keeps the image."""
import pytest

from test_tp_program import SHAPES, desc, program

SMEM_MAX = 227 * 1024
TILE = 128


def expected_layout(prog, info, layer_dim):
    """-> (stages, total bytes) of wg_layout for the tc_f16 inference launch, from the program's own shapes."""
    n, n_t, plane_bytes, stages, smem, x_tile, stage_bytes, slab = info
    kx = max(e['x_bytes'] for e in prog) // (TILE * 2)                  # widest feature segment
    n_gemm = len({e['gemm'] for e in prog})
    f32_floats = n_gemm * (512 if layer_dim > 256 else 256) + layer_dim + 4
    h_bytes = layer_dim * TILE * 2 if layer_dim > 256 else 0
    fixed = h_bytes + kx * TILE * 2 + (f32_floats + 3) // 4 * 16 + TILE * 4 + 256
    st = min((SMEM_MAX - fixed) // stage_bytes, 8)
    return st, st * stage_bytes + fixed


@pytest.mark.parametrize('name', sorted(SHAPES))
def test_layout_of_the_inference_launch(name):
    shape = SHAPES[name]
    rc, prog, prog_t, info = program(desc(**shape))
    assert rc == 0
    stages, total = expected_layout(prog, info, shape.get('layer_dim', 256))
    assert info[3] == stages and info[4] == total <= SMEM_MAX


def test_c2_ring_has_six_stages():
    """8 x 256: without the 64 KiB activation image the ring grows from 4 to 6 stages of 64 K-columns x 256 N (32 KiB)."""
    rc, prog, prog_t, info = program(desc())
    assert rc == 0 and info[3] == 6 and info[6] == 64 * 256 * 2 and info[7] == 64
