"""Discrete-event simulation of the barrier protocol of k_multiply_tc5 (sdk_b200/csrc/tc5_kernels.cu): the roles
(bulk-copy producer warp, two consumer warpgroups) are transcribed loop for loop as coroutines over a model of mbarrier
phases / transaction counts, with randomised completion delays for the asynchronous agents (bulk copies, wgmma groups).
Checked: the run terminates (no deadlock), no shared-memory stage / B buffer is overwritten before its readers are done,
nothing is read before it has been written, and no barrier ever runs two phases ahead of a waiter (which would make a
parity wait miss its phase).  This is a model of the protocol, not of the
hardware: it guards the design against the one failure a GPU run cannot afford, a hang."""
import heapq
import random

import pytest

CONSUMERS = 2                        # warpgroups; each arrives once on a ring stage / B buffer it has finished reading


class Bar:
    def __init__(self, count):
        self.count, self.pending, self.tx, self.phase = count, count, 0, 0

    def _maybe_flip(self):
        if self.pending == 0 and self.tx == 0:
            self.phase += 1
            self.pending = self.count

    def arrive(self):
        assert self.pending > 0, "more arrivals than the barrier expects in one phase"
        self.pending -= 1
        self._maybe_flip()

    def expect_tx(self, n):          # mbarrier.arrive.expect_tx: one arrival + n pending bytes
        self.tx += n
        self.pending -= 1
        self._maybe_flip()

    def complete_tx(self, n):
        self.tx -= n
        assert self.tx >= 0
        self._maybe_flip()

    def passed(self, parity):        # try_wait.parity
        return (self.phase & 1) != parity


def simulate(n_items, tiles_per_item, ks, seed, STAGES=5, KS_PER_STAGE=4, BBUFS=2):
    """STAGES ring stages of KS_PER_STAGE k-steps, BBUFS buffers of the query operand: the template / run-time parameters of
    k_multiply_tc5."""
    rng = random.Random(seed)
    full = [Bar(1) for _ in range(STAGES)]
    empty = [Bar(CONSUMERS) for _ in range(STAGES)]
    bfull, bempty = [Bar(1) for _ in range(BBUFS)], [Bar(CONSUMERS) for _ in range(BBUFS)]
    stages_per_tile = (ks + KS_PER_STAGE - 1) // KS_PER_STAGE
    now = [0.0]
    events = []                      # (time, seq, fn)
    seq = [0]

    def later(dt, fn):
        seq[0] += 1
        heapq.heappush(events, (now[0] + dt, seq[0], fn))

    # ground truth for the hazard checks
    a_content = [None] * STAGES      # (item, tile, st) the stage currently holds, or ("loading", ...)
    a_readers = [0] * STAGES         # MMA groups issued on the stage and not yet complete
    b_content, b_readers = [None] * BBUFS, [0] * BBUFS
    log = {"tiles_done": 0}

    def wait(bar, parity):
        while not bar.passed(parity):
            yield

    def producer():
        stage, sphase, it = 0, 0, 0
        for item in range(n_items):
            bb = it % BBUFS
            yield from wait(bempty[bb], ((it // BBUFS) & 1) ^ 1)
            assert b_readers[bb] == 0, "B buffer overwritten while MMAs still read it"
            bfull[bb].expect_tx(ks)
            b_content[bb] = ("loading", item)
            def done_b(bb=bb, item=item):
                b_content[bb] = item
                bfull[bb].complete_tx(ks)
            later(rng.uniform(0.5, 3.0), done_b)
            for t in range(tiles_per_item):
                for st in range(stages_per_tile):
                    ks_here = min(KS_PER_STAGE, ks - st * KS_PER_STAGE)
                    yield from wait(empty[stage], sphase ^ 1)
                    assert a_readers[stage] == 0, "A stage overwritten while MMAs still read it"
                    full[stage].expect_tx(ks_here)
                    a_content[stage] = ("loading", item, t, st)
                    def done_a(stage=stage, item=item, t=t, st=st, n=ks_here):
                        a_content[stage] = (item, t, st)
                        full[stage].complete_tx(n)
                    later(rng.uniform(0.2, 2.0), done_a)
                    stage += 1
                    if stage == STAGES:
                        stage, sphase = 0, sphase ^ 1
                    yield
            it += 1

    def consumer(wg):
        stage, sphase, it = 0, 0, 0
        groups = []                  # completion flags of this warpgroup's committed wgmma groups, oldest first

        def wait_groups(pending):    # wgmma.wait_group(pending): every group but the newest `pending` has completed
            while not all(g[0] for g in groups[:len(groups) - pending]):
                yield

        for item in range(n_items):
            bb = it % BBUFS
            yield from wait(bfull[bb], (it // BBUFS) & 1)
            assert b_content[bb] == item, "MMA reads a B buffer that does not hold this item"
            b_readers[bb] += 1
            for t in range(tiles_per_item):
                prev = None
                for st in range(stages_per_tile):
                    yield from wait(full[stage], sphase)
                    assert a_content[stage] == (item, t, st), "MMA reads an A stage that does not hold its tile"
                    a_readers[stage] += 1
                    flag = [False]
                    groups.append(flag)
                    def complete(flag=flag, stage=stage):
                        flag[0] = True
                        a_readers[stage] -= 1
                    later(rng.uniform(0.1, 1.5), complete)
                    yield from wait_groups(1)
                    if prev is not None:
                        empty[prev].arrive()
                    prev = stage
                    stage += 1
                    if stage == STAGES:
                        stage, sphase = 0, sphase ^ 1
                    yield
                yield from wait_groups(0)
                if prev is not None:
                    empty[prev].arrive()
                for _ in range(rng.randint(1, 4)):   # the epilogue works on registers only
                    yield
                if wg == 0:
                    log["tiles_done"] += 1
            b_readers[bb] -= 1
            bempty[bb].arrive()
            it += 1

    roles = [producer()] + [consumer(wg) for wg in range(CONSUMERS)]
    alive = list(roles)
    idle_rounds = 0
    while alive:
        progressed = False
        order = list(alive)
        rng.shuffle(order)
        before = (tuple(b.phase for b in full + empty + bfull + bempty), len(events))
        for r in order:
            try:
                next(r)
            except StopIteration:
                alive.remove(r)
                progressed = True
        if events and (rng.random() < 0.7 or not progressed):
            tm, _, fn = heapq.heappop(events)
            now[0] = tm
            fn()
            progressed = True
        after = (tuple(b.phase for b in full + empty + bfull + bempty), len(events))
        idle_rounds = 0 if (progressed and before != after) or events else idle_rounds + 1
        assert idle_rounds < 10000, "deadlock: no role can make progress and no asynchronous event is pending"
    while events:                    # drain trailing completions
        tm, _, fn = heapq.heappop(events)
        fn()
    return log["tiles_done"]


@pytest.mark.parametrize("n_items,tiles,ks", [(1, 1, 1), (3, 1, 2), (5, 8, 16), (4, 3, 5), (7, 2, 16), (2, 32, 16)])
def test_tc5_barrier_protocol_terminates_without_hazards(n_items, tiles, ks):
    for seed in range(6):
        assert simulate(n_items, tiles, ks, seed) == n_items * tiles
        # the shipped configurations: 32 KiB stages beside a double- or single-buffered query operand, 16 KiB stages
        assert simulate(n_items, tiles, ks, seed, STAGES=5, KS_PER_STAGE=8, BBUFS=1) == n_items * tiles
        assert simulate(n_items, tiles, ks, seed, STAGES=3, KS_PER_STAGE=8, BBUFS=2) == n_items * tiles
        assert simulate(n_items, tiles, ks, seed, STAGES=10, KS_PER_STAGE=4, BBUFS=1) == n_items * tiles
        assert simulate(n_items, tiles, ks, seed, STAGES=2, KS_PER_STAGE=4, BBUFS=1) == n_items * tiles
