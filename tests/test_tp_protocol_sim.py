"""CPU: the barrier protocol of the tensor-core MLP kernel (csrc/mn_mlp_wg.cuh) in a discrete-event model driven by the kernel's
real stage program (tests/tp_protocol_sim.py): no deadlock and no stale read - ring stages, feature buffer - under randomised
timing, for every network shape the parity tests use, full and sigma_only calls, odd and even tile counts per CTA (the barrier
phases wrap differently) and the smallest ring the launcher accepts.  A ring too small for the stages a warpgroup keeps in
flight must be reported as a deadlock (the model can fail)."""
import pytest

import tp_protocol_sim as S
from test_tp_program import SHAPES, desc, program


@pytest.mark.parametrize('name', sorted(SHAPES))
@pytest.mark.parametrize('odd_tail', [False, True])
def test_no_deadlock_no_stale_read(name, odd_tail):
    rc, prog, prog_t, info = program(desc(**SHAPES[name]))
    assert rc == 0
    stages = info[3]
    n_tiles = 3 if odd_tail else 4
    for seed in range(3):
        S.simulate(prog, stages, n_tiles=n_tiles, seed=seed)
    S.simulate(prog, 2, n_tiles=n_tiles, seed=11)                       # smallest ring the launcher accepts
    S.simulate(prog_t, stages, n_tiles=n_tiles, seed=5)                 # sigma_only: trunk prefix


def test_model_reports_a_ring_smaller_than_a_block():
    """A warpgroup releases a ring stage only after issuing the next stage's MMAs, so it holds two stages at a time: a
    one-stage ring must deadlock in the model (the launcher requires at least two)."""
    rc, prog, prog_t, info = program(desc())
    assert rc == 0 and info[3] >= 2
    with pytest.raises(S.Deadlock):
        S.simulate(prog, 1, n_tiles=2, seed=0)


def test_model_reports_a_missing_release():
    """Dropping the second warpgroup's release of the feature buffer starves the producer at the next feature segment: the model
    must notice."""
    rc, prog, prog_t, info = program(desc())
    orig = S.release
    try:
        S.release = lambda bar, who: None if who == ('xa', 1) else orig(bar, who)
        with pytest.raises(S.Deadlock):
            S.simulate(prog, info[3], n_tiles=2, seed=0)
    finally:
        S.release = orig
