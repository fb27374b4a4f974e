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
        assert self.tx >= 0, "bulk copies completed more transaction bytes than expect_tx announced"
        self._maybe_flip()

    def passed(self, parity):        # try_wait.parity
        return (self.phase & 1) != parity


def simulate(n_items, tiles_per_item, ks, seed, STAGES=5, KS_PER_STAGE=4, BBUFS=2, masks=None, consumer_masks=None,
             copy_full_stage=False, consumer_ignores_km=False):
    """STAGES ring stages of KS_PER_STAGE k-steps, BBUFS buffers of the query operand: the template / run-time parameters of
    k_multiply_tc5.  masks[item][tile]: the tile_mask word of the tile (bit k = k-step k is present; None = every k-step
    present).  The remaining arguments break the protocol on purpose, to show that the checks catch it:
    consumer_masks = the masks the consumers read instead of `masks`; copy_full_stage = the producer copies the whole stage
    but expects only the present k-steps; consumer_ignores_km = the consumers multiply every k-step of a fetched stage."""
    rng = random.Random(seed)
    full_ks = (1 << ks) - 1
    if masks is None:
        masks = [[full_ks] * tiles_per_item for _ in range(n_items)]
    if consumer_masks is None:
        consumer_masks = masks
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

    def stage_mask(mask, st):        # km of the kernel: the k-steps of stage st that hold a present tile
        ks_here = min(KS_PER_STAGE, ks - st * KS_PER_STAGE)
        return ks_here, (mask >> (st * KS_PER_STAGE)) & ((1 << ks_here) - 1)

    # ground truth for the hazard checks
    a_content = [[None] * KS_PER_STAGE for _ in range(STAGES)]   # per k-step slot: (item, tile, st, kk) or ("loading", ...)
    a_readers = [0] * STAGES         # MMA groups issued on the stage and not yet complete
    b_content, b_readers = [None] * BBUFS, [0] * BBUFS
    log = {"tiles_done": 0, "fetched": 0, "mults": [set() for _ in range(CONSUMERS)]}

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
                    ks_here, km = stage_mask(masks[item][t], st)
                    if km == 0:              # nothing present in this stage: no ring slot
                        continue
                    yield from wait(empty[stage], sphase ^ 1)
                    assert a_readers[stage] == 0, "A stage overwritten while MMAs still read it"
                    full[stage].expect_tx(bin(km).count("1"))
                    log["fetched"] += 1
                    if km == (1 << ks_here) - 1 or copy_full_stage:
                        copies = [list(range(ks_here))]                       # one bulk copy of the whole stage
                    else:
                        copies = [[kk] for kk in range(ks_here) if (km >> kk) & 1]   # one bulk copy per present k-step
                    for kks in copies:
                        for kk in kks:
                            a_content[stage][kk] = ("loading", item, t, st, kk)
                        def done_a(stage=stage, item=item, t=t, st=st, kks=kks):
                            for kk in kks:
                                a_content[stage][kk] = (item, t, st, kk)
                            full[stage].complete_tx(len(kks))
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
                ring_ops = 0             # waits and arrivals on the A ring for this tile
                for st in range(stages_per_tile):
                    ks_here, km = stage_mask(consumer_masks[item][t], st)
                    if km == 0:
                        continue
                    yield from wait(full[stage], sphase)
                    ring_ops += 1
                    for kk in range(KS_PER_STAGE):
                        if (km >> kk) & 1 or (consumer_ignores_km and kk < ks_here):
                            assert a_content[stage][kk] == (item, t, st, kk), "MMA reads a k-step slot that does not hold its tile"
                            log["mults"][wg].add((item, t, st, kk))
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
                        ring_ops += 1
                    prev = stage
                    stage += 1
                    if stage == STAGES:
                        stage, sphase = 0, sphase ^ 1
                    yield
                yield from wait_groups(0)
                if prev is not None:
                    empty[prev].arrive()
                    ring_ops += 1
                if consumer_masks[item][t] & full_ks == 0:
                    assert ring_ops == 0, "a tile without a present k-step touched the A ring"
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
    # every fetched stage went through exactly one full and one empty phase, and no transaction is left over
    assert sum(b.phase for b in full) == sum(b.phase for b in empty) == log["fetched"]
    assert all(b.tx == 0 and b.pending == b.count for b in full + empty + bfull + bempty)
    # each warpgroup multiplied exactly the present k-steps
    present = {(item, t, st, kk) for item in range(n_items) for t in range(tiles_per_item) for st in range(stages_per_tile)
               for kk in range(KS_PER_STAGE) if (stage_mask(masks[item][t], st)[1] >> kk) & 1}
    for wg in range(CONSUMERS):
        assert log["mults"][wg] == present, "the multiplied k-steps are not the present ones"
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


# ---- tile skipping (tile_mask), in the ring configurations the launcher picks ----------------------------------------------
TC5_TILE = 4096
TC5_SMEM_BUDGET = 227 * 1024 - 1024
TC5_MAX_STAGES = 24


def tc5_ring_stages(ks, ksps, bbufs):
    """tc5_ring_stages (tc5_kernels.cu), with C's truncating division."""
    num = TC5_SMEM_BUDGET - bbufs * ks * TC5_TILE
    n = num // (ksps * TC5_TILE) if num >= 0 else -(-num // (ksps * TC5_TILE))
    return min(n, TC5_MAX_STAGES)


def launch_config(dim0):
    """(ks, KSPS, BBUFS, ring stages) as launch_multiply_tc5 picks them."""
    ks = (dim0 + 31) // 32
    ksps, bbufs = 8, 2
    if tc5_ring_stages(ks, ksps, bbufs) < 2:
        ksps = 4
    if tc5_ring_stages(ks, ksps, bbufs) < 2:
        bbufs = 1
    return ks, ksps, bbufs, tc5_ring_stages(ks, ksps, bbufs)


DIM0S = [2, 32, 64, 256, 512, 1024]


def test_launch_config_transcription():
    for dim0 in DIM0S[:-1]:
        ks, ksps, bbufs, stages = launch_config(dim0)
        assert (ksps, bbufs) == (8, 2) and stages >= 2, dim0
    assert launch_config(512) == (16, 8, 2, 3)
    assert launch_config(1024) == (32, 4, 1, 6)               # 8 stages per tile through a 6-stage ring


def mask_patterns(n_items, tiles, ks, ksps, rng):
    """name -> masks[item][tile] (bit k = k-step k holds a present item)."""
    full = (1 << ks) - 1
    spt = (ks + ksps - 1) // ksps

    def per_stage(pick):             # one bit pattern per stage, pick(ks_here, st) -> bits of the stage
        m = 0
        for st in range(spt):
            m |= pick(min(ksps, ks - st * ksps), st) << (st * ksps)
        return m

    grid = lambda f: [[f(i, t) for t in range(tiles)] for i in range(n_items)]
    single = rng.randrange(n_items), rng.randrange(tiles), rng.randrange(ks)
    return {
        "empty": grid(lambda i, t: 0),
        "full": grid(lambda i, t: full),
        "single bit": grid(lambda i, t: 1 << single[2] if (i, t) == single[:2] else 0),
        "one k-step per stage": grid(lambda i, t: per_stage(lambda n, st: 1 << ((st + i + t) % n))),
        "all k-steps of a stage but one": grid(lambda i, t: per_stage(lambda n, st: ((1 << n) - 1) & ~(1 << ((st + t) % n)))),
        "empty items between full items": grid(lambda i, t: full if i % 2 == 0 else 0),
        "random 0.05": grid(lambda i, t: sum(1 << k for k in range(ks) if rng.random() < 0.05)),
        "random 0.5": grid(lambda i, t: sum(1 << k for k in range(ks) if rng.random() < 0.5)),
    }


@pytest.mark.parametrize("dim0", DIM0S)
def test_tc5_tile_skipping_protocol(dim0):
    ks, ksps, bbufs, stages = launch_config(dim0)
    n_items, tiles = 4, 3
    for seed in range(3):
        rng = random.Random(1000 * dim0 + seed)
        for name, masks in mask_patterns(n_items, tiles, ks, ksps, rng).items():
            got = simulate(n_items, tiles, ks, seed, STAGES=stages, KS_PER_STAGE=ksps, BBUFS=bbufs, masks=masks)
            assert got == n_items * tiles, (dim0, seed, name)


@pytest.mark.parametrize("dim0", [64, 512, 1024])
def test_tc5_skip_model_catches_expect_tx_mismatch(dim0):
    """The producer copies a whole partly present stage but announces only the present k-steps: the copies complete more
    bytes than expected (on the GPU, the phase accounting is broken and the kernel hangs)."""
    ks, ksps, bbufs, stages = launch_config(dim0)
    masks = mask_patterns(3, 2, ks, ksps, random.Random(5))["all k-steps of a stage but one"]
    with pytest.raises(AssertionError, match="transaction bytes"):
        simulate(3, 2, ks, 0, STAGES=stages, KS_PER_STAGE=ksps, BBUFS=bbufs, masks=masks, copy_full_stage=True)


@pytest.mark.parametrize("dim0", [64, 512, 1024])
def test_tc5_skip_model_catches_role_mask_disagreement(dim0):
    """The consumers read a different mask from the producer's: they wait for stages that are never fetched."""
    ks, ksps, bbufs, stages = launch_config(dim0)
    pats = mask_patterns(3, 2, ks, ksps, random.Random(6))
    with pytest.raises(AssertionError, match="deadlock"):
        simulate(3, 2, ks, 0, STAGES=stages, KS_PER_STAGE=ksps, BBUFS=bbufs, masks=pats["empty"], consumer_masks=pats["full"])
    with pytest.raises(AssertionError, match="deadlock"):
        simulate(3, 2, ks, 0, STAGES=stages, KS_PER_STAGE=ksps, BBUFS=bbufs, masks=pats["single bit"],
                 consumer_masks=pats["full"])


@pytest.mark.parametrize("dim0", [64, 512, 1024])
def test_tc5_skip_model_catches_absent_k_steps_multiplied(dim0):
    """The consumers multiply every k-step of a fetched stage: the slots of absent k-steps hold another tile's data or none."""
    ks, ksps, bbufs, stages = launch_config(dim0)
    masks = mask_patterns(3, 2, ks, ksps, random.Random(7))["one k-step per stage"]
    with pytest.raises(AssertionError, match="does not hold its tile"):
        simulate(3, 2, ks, 0, STAGES=stages, KS_PER_STAGE=ksps, BBUFS=bbufs, masks=masks, consumer_ignores_km=True)
