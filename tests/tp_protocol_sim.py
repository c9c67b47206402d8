"""Discrete-event model of the barrier protocol of the tensor-core MLP kernel (csrc/mn_mlp_wg.cuh), driven by the kernel's REAL
stage program (mn_debug_tp_program).  Three actors - the producer thread and the two consumer warpgroups - exchange the kernel's
mbarriers (full / empty per ring stage, xa_full / xa_empty of the feature buffer); copies land and warpgroup MMAs complete after
random times, so many seeds explore many interleavings.  A consumer releases a ring stage the way the kernel does: after the
MMAs of the NEXT stage are issued and `wgmma.wait_group 1` says the stage's own MMAs have completed; at the end of a feature
segment and of an accumulator it waits for all of them.  Independent of the barriers, the model tracks WHAT each buffer holds
(which program entry of which tile a ring stage contains, which feature segment the feature buffer holds, how many unfinished
MMAs read them) and asserts that every MMA reads what the kernel's arithmetic needs and that no copy overwrites a buffer an MMA
still reads.  A deadlock (every actor blocked, nothing in flight) raises Deadlock.  Test infrastructure only."""
import heapq
import random

WS_FROM_X, WS_X_FIRST, WS_X_LAST, WS_LO, WS_CHUNK_FIRST, WS_CHUNK_LAST = 1, 2, 4, 8, 16, 32


class MBar:
    """mbarrier: `count` arrivals complete a phase; wait(parity) passes once the phase with that parity has completed."""

    def __init__(self, count, name=''):
        self.count, self.pending, self.phase, self.name = count, count, 0, name

    def arrive(self, n=1):
        for _ in range(n):
            self.pending -= 1
            if self.pending == 0:
                self.pending, self.phase = self.count, self.phase ^ 1

    def passed(self, parity):
        return self.phase != parity


class Deadlock(AssertionError):
    pass


def release(bar, who):
    """One consumer warpgroup's arrival on an `empty` barrier (`who` = ('stage' | 'xa', warpgroup)); tests replace it to model a
    missing release."""
    bar.arrive()


def simulate(prog, n_stages, n_tiles, seed=0, max_steps=5_000_000):
    """prog: the stage program of one tile (entries as returned by tests/test_tp_program.py::program)."""
    rnd = random.Random(seed)
    full = [MBar(1, 'full') for _ in range(n_stages)]
    empty = [MBar(2, 'empty') for _ in range(n_stages)]
    xa_full, xa_empty = MBar(1, 'xa_full'), MBar(2, 'xa_empty')
    stage_holds = [None] * n_stages              # (tile, entry) a ring stage contains
    stage_readers = [0] * n_stages               # issued, unfinished MMAs that read a ring stage
    xa = dict(holds=None, readers=0)             # (tile, entry of the segment's first stage), unfinished MMAs reading it
    seg_of = {}
    cur = None
    for i, e in enumerate(prog):
        if e['flags'] & WS_X_FIRST:
            cur = i
        if e['flags'] & WS_FROM_X:
            seg_of[i] = cur
    events, now, seq = [], [0.0], [0]

    def later(dt, fn):
        seq[0] += 1
        heapq.heappush(events, (now[0] + dt, seq[0], fn))

    # ---- actors are generators yielding a condition (callable) to wait for, or a float to sleep
    def producer():
        stage, phase, xphase = 0, 0, 0
        for tile in range(n_tiles):
            for i, e in enumerate(prog):
                if e['flags'] & WS_X_FIRST:
                    yield lambda p=xphase: xa_empty.passed(p ^ 1)
                    assert xa['readers'] == 0, f'feature copy issued under {xa["readers"]} unfinished MMA(s)'

                    def land_x(tile=tile, i=i):
                        assert xa['readers'] == 0, 'feature copy lands under an unfinished MMA'
                        xa['holds'] = (tile, i)
                        xa_full.arrive()
                    later(rnd.uniform(0.5, 3.0), land_x)
                    xphase ^= 1
                yield lambda s=stage, p=phase: empty[s].passed(p ^ 1)
                assert stage_readers[stage] == 0, f'copy into ring stage {stage} issued under an unfinished MMA'

                def land(s=stage, tile=tile, i=i):
                    assert stage_readers[s] == 0, f'copy lands in ring stage {s} under an unfinished MMA'
                    stage_holds[s] = (tile, i)
                    full[s].arrive()
                later(rnd.uniform(0.5, 3.0), land)
                stage += 1
                if stage == n_stages:
                    stage, phase = 0, phase ^ 1
                yield rnd.uniform(0.0, 0.3)

    def consumer(wg):
        stage, phase, xphase = 0, 0, 0
        groups = []                                  # per committed group: [unfinished flag]
        last_done = [0.0]                            # completion time of the most recently issued group

        def pending():
            return sum(1 for g in groups if g[0])
        for tile in range(n_tiles):
            prev = -1
            for i, e in enumerate(prog):
                if e['flags'] & WS_X_FIRST:
                    yield lambda p=xphase: xa_full.passed(p)
                    xphase ^= 1
                yield lambda s=stage, p=phase: full[s].passed(p)
                assert stage_holds[stage] == (tile, i), f'warpgroup {wg} reads ring stage {stage} = {stage_holds[stage]}, needs {(tile, i)}'
                fx = bool(e['flags'] & WS_FROM_X)
                if fx:
                    assert xa['holds'] == (tile, seg_of[i]), f'warpgroup {wg} reads feature segment {xa["holds"]}, needs {(tile, seg_of[i])}'
                stage_readers[stage] += 1
                xa['readers'] += fx
                g = [True]
                groups.append(g)

                def done(g=g, s=stage, fx=fx):
                    g[0] = False
                    stage_readers[s] -= 1
                    xa['readers'] -= fx
                # a warpgroup's MMA groups complete in issue order
                last_done[0] = max(last_done[0], now[0]) + rnd.uniform(1.0, 4.0) * e['kc'] / 32
                later(last_done[0] - now[0], done)
                if prev >= 0:
                    yield lambda: pending() <= 1                 # wgmma.wait_group 1
                    release(empty[prev], ('stage', wg))
                prev = stage
                stage += 1
                if stage == n_stages:
                    stage, phase = 0, phase ^ 1
                if e['flags'] & WS_X_LAST:
                    yield lambda: pending() == 0                 # wgmma.wait_group 0
                    release(empty[prev], ('stage', wg))
                    release(xa_empty, ('xa', wg))
                    prev = -1
                if e['flags'] & WS_CHUNK_LAST:
                    yield lambda: pending() == 0
                    if prev >= 0:
                        release(empty[prev], ('stage', wg))
                    prev = -1
                    yield rnd.uniform(0.5, 4.0)                  # epilogue
                groups[:] = [g for g in groups if g[0]]

    actors = [producer(), consumer(0), consumer(1)]
    waiting = [None] * len(actors)                   # current condition of each actor; 'sleep' while a wake-up is queued
    done_ = [False] * len(actors)

    def step(k):
        """Advance actor k as far as it can go now."""
        while not done_[k]:
            w = waiting[k]
            if w == 'sleep':
                return
            if w is not None and not w():
                return
            try:
                req = next(actors[k])
            except StopIteration:
                done_[k] = True
                return
            if callable(req):
                waiting[k] = req
            else:
                waiting[k] = 'sleep'

                def wake(k=k):
                    waiting[k] = None
                later(req, wake)
    steps = 0
    while not all(done_):
        for k in range(len(actors)):
            step(k)
        if all(done_):
            break
        if not events:
            blocked = [k for k in range(len(actors)) if not done_[k]]
            raise Deadlock(f'actors {blocked} blocked with nothing in flight at t={now[0]:.1f}')
        t, _, fn = heapq.heappop(events)
        now[0] = t
        fn()
        steps += 1
        if steps > max_steps:
            raise Deadlock('no progress within the step budget')
