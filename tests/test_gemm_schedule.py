"""CPU model of the consumer schedules of the GEMM engine (csrc/gemm.cu, gemm_wgmma_kernel), no GPU: ping-pong, and the
cooperative split of CTAs that have a single tile.

The integer stage / phase bookkeeping of the two TMA producer warps and the two consumer warpgroups of one CTA is restated
line for line and run under random interleavings against a model of the mbarriers and the named barriers.  A protocol
error shows up here as an assertion or a deadlock instead of as the kernel's watchdog trap on the GPU.
"""
import random

import pytest


class MBar:
    """mbarrier: `count` arrivals complete a phase; try_wait.parity(P) succeeds once the phase of parity P completed."""

    def __init__(self, count):
        self.count, self.pending, self.done, self.fills = count, 0, 0, []

    def arrive(self, fill):
        self.fills.append(fill)
        assert len(set(self.fills)) == 1, f'one phase collects arrivals of different fills: {self.fills}'
        self.pending += 1
        if self.pending == self.count:
            self.pending, self.fills = 0, []
            self.done += 1

    def ready(self, parity):
        return (self.done & 1) != parity


class NamedBar:
    """bar.sync / bar.arrive over two warpgroups: the barrier completes when both have reached it."""

    def __init__(self):
        self.members, self.gen = [], 0

    def join(self, kind):
        self.members.append(kind)
        if len(self.members) == 2:
            # a completion without a waiting warpgroup would let two arrivals of the same side pass each other
            assert sorted(self.members) == ['arrive', 'sync'], self.members
            self.members = []
            self.gen += 1


def n_local_of(num_tiles, grid, cta):
    return (num_tiles - cta + grid - 1) // grid                 # the consumers' n_local


def simulate(n_local, k_blocks, stages, rnd, coop=False):
    """coop: every CTA has one tile (num_tiles <= grid) and both consumers read every fill (half c each)."""
    assert not coop or n_local == 1
    full = [MBar(2) for _ in range(stages)]                      # one arrive.expect_tx per producer warp
    empty = [MBar(2 if coop else 1) for _ in range(stages)]      # one arrival per consumer that reads the stage
    order = [NamedBar(), NamedBar()]                             # kOrderBar + c
    slot = [None] * stages                                       # which fill a stage holds
    consumed, released = {}, {}                                  # fill -> set of consumers

    def producer():
        stage, phase = 0, 0
        for j in range(n_local):
            for kb in range(k_blocks):
                f = j * k_blocks + kb
                yield lambda s=stage, ph=phase: empty[s].ready(ph ^ 1)
                assert empty[stage].done == f // stages, 'producer passed its empty wait on the wrong phase'
                assert f < stages or len(released.get(f - stages, ())) == (2 if coop else 1), \
                    'stage refilled before every reader of its previous fill released it'
                slot[stage] = f
                full[stage].arrive(f)
                stage += 1
                if stage == stages:
                    stage, phase = 0, phase ^ 1

    def consumer(cw):
        st = {'stage': 0, 'phase': 0}

        def skip_tile():
            st['stage'] += k_blocks
            st['phase'] ^= (st['stage'] // stages) & 1
            st['stage'] %= stages

        def release(s):
            f = slot[s]
            assert cw in consumed[f] and cw not in released.setdefault(f, set())
            released[f].add(cw)
            empty[s].arrive(f)

        if cw == 1 and not coop:
            skip_tile()
        for j in range(0 if coop else cw, n_local, 2):
            if j > 0:
                g0 = order[cw].gen
                order[cw].join('sync')
                yield lambda b=order[cw], g0=g0: b.gen > g0
            prev = -1
            for kb in range(k_blocks):
                f = j * k_blocks + kb
                s, ph = st['stage'], st['phase']
                yield lambda s=s, ph=ph: full[s].ready(ph)
                assert full[s].done == f // stages + 1, 'consumer passed its full wait on the wrong phase'
                assert slot[s] == f and cw not in consumed.setdefault(f, set())
                consumed[f].add(cw)
                if prev >= 0:
                    release(prev)
                prev = s
                st['stage'] += 1
                if st['stage'] == stages:
                    st['stage'], st['phase'] = 0, st['phase'] ^ 1
            if j + 1 < n_local:
                order[cw ^ 1].join('arrive')
            release(prev)
            skip_tile()

    agents = [producer(), producer(), consumer(0), consumer(1)]
    conds = []
    for a in agents:
        conds.append(next(a, None))
    while True:
        live = [i for i, c in enumerate(conds) if c is not None]
        if not live:
            break
        ready = [i for i in live if conds[i]()]
        assert ready, f'deadlock: n_local={n_local} k_blocks={k_blocks} stages={stages} waiting agents {live}'
        i = rnd.choice(ready)
        conds[i] = next(agents[i], None)

    fills = n_local * k_blocks
    assert sorted(consumed) == list(range(fills)) and sorted(released) == list(range(fills))
    owners = lambda f: {0, 1} if coop else {(f // k_blocks) % 2}
    assert all(consumed[f] == owners(f) == released[f] for f in range(fills))
    assert all(b.pending == 0 for b in full + empty)
    assert all(not b.members for b in order), 'a named-barrier arrival is left over at the end of the kernel'


def test_cta_tiles_partition_the_problem():
    for num_tiles, grid in ((1, 1), (2, 2), (2, 1), (3, 1), (7, 3), (2 * 132 + 5, 132), (3 * 132 + 68, 132)):
        owner = {}
        for cta in range(grid):
            for j in range(n_local_of(num_tiles, grid, cta)):
                tile = cta + j * grid
                assert tile < num_tiles and tile not in owner
                owner[tile] = cta
        assert len(owner) == num_tiles


@pytest.mark.parametrize('k_blocks', [1, 2, 8, 32])
def test_pingpong_consumers_take_every_fill_once_with_the_right_parity(k_blocks):
    # local tile counts of the CTAs of (num_tiles, grid): 1, 2, odd, and more than two tiles per consumer
    n_locals = {n_local_of(t, g, cta) for t, g in ((1, 1), (2, 1), (3, 1), (2 * 132 + 5, 132), (9, 1), (10, 1))
                for cta in range(g)}
    assert n_locals == {1, 2, 3, 9, 10}
    for n_local in sorted(n_locals):
        for stages in range(3, 17):
            simulate(n_local, k_blocks, stages, random.Random(1000 * n_local + 10 * k_blocks + stages))


@pytest.mark.parametrize('k_blocks', [1, 2, 8, 32])
def test_cooperative_single_tile_ctas_release_each_stage_after_both_consumers(k_blocks):
    # num_tiles <= grid: every CTA has exactly one tile
    assert {n_local_of(t, t, cta) for t in (1, 57, 132) for cta in range(t)} == {1}
    for stages in range(3, 17):
        simulate(1, k_blocks, stages, random.Random(7 * k_blocks + stages), coop=True)
