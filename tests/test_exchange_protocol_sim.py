"""Model of bench.py's copy-engine exchange (N > 1): every rank expands its queries into its own slot of a gather-buffer
set, the copy engines push the slot into every peer's set, a 4-byte all-reduce ordered after the pushes says "landed",
the first dimension reads the whole set.  NBUF sets rotate over the steps and, when pipelined, the expansion + pushes of
step k + 1 are enqueued before the compute of step k.

The model replays the host program of bench.py (ce_expand_push / ce_compute / step_dev) for every rank into a graph of
operations on FIFO streams with event dependencies, gives every operation a random duration, and computes start / end
times.  Checked over many random timings:
  * safety: a push never overlaps a read of the buffer it overwrites, and a first dimension never starts before every
    slot of its set has landed;
  * three sets (what bench.py uses; the argument beside the code needs only the barriers) are safe when pipelined; two
    are safe as well, but only because the survivors' all-gather of step k - 2 orders every rank's first dimension before
    anybody's expansion of step k; ONE set is not (the checker must find that hazard, which also shows it has teeth);
    one set is enough without the pipeline;
  * at N = 8: with the "landed" all-reduces on the same communicator as the survivors' all-gather, a step waits for the
    NEXT step's transfer; on their own communicator it does not.
No GPU, no torch: this is host logic."""
import random

import pytest


class Op:
    __slots__ = ("name", "rank", "stream", "deps", "dur", "start", "end", "group", "step", "kind", "peer")

    def __init__(self, name, rank, stream, deps, dur, kind, step, peer=None):
        self.name, self.rank, self.stream, self.deps, self.dur = name, rank, stream, list(deps), dur
        self.start = self.end = None
        self.group = None                  # collectives: the list of the per-rank ops of one collective call
        self.step, self.kind, self.peer = step, kind, peer


class Model:
    """Streams are FIFO: an op starts when its predecessor on the same (rank, stream) and all its deps have ended.  A
    collective's per-rank op "arrives" like any op and ends, on every rank, when the last rank has arrived (+ its duration)."""

    def __init__(self, n, rng, dur):
        self.n, self.rng, self.dur = n, rng, dur
        self.tail = {}                      # (rank, stream) -> last op
        self.ops = []
        self.coll = {}                      # (comm, seq) -> [op per rank]
        self.coll_seq = {}                  # (rank, comm) -> next sequence number

    def op(self, rank, stream, kind, step, deps=(), peer=None):
        lo, hi = self.dur[kind]
        o = Op("%s[%d]@%d" % (kind, step, rank), rank, stream, deps, self.rng.uniform(lo, hi), kind, step, peer)
        prev = self.tail.get((rank, stream))
        if prev is not None:
            o.deps.append(prev)
        self.tail[(rank, stream)] = o
        self.ops.append(o)
        return o

    def collective(self, rank, comm, kind, step, deps):
        """NCCL: one stream per communicator and rank; the k-th call on a communicator matches the k-th call of every rank."""
        o = self.op(rank, "nccl:" + comm, kind, step, deps)
        seq = self.coll_seq.get((rank, comm), 0)
        self.coll_seq[(rank, comm)] = seq + 1
        g = self.coll.setdefault((comm, seq), [])
        g.append(o)
        o.group = g
        return o

    def solve(self):
        import sys
        sys.setrecursionlimit(100000)
        arrive = {}

        def t_arrive(o):
            if id(o) not in arrive:
                arrive[id(o)] = max([0.0] + [t_end(d) for d in o.deps])
            return arrive[id(o)]

        def t_end(o):
            if o.end is None:
                if o.group is not None:
                    assert len(o.group) == self.n, ("collective not entered by every rank", o.name)
                    assert len({(g.kind, g.step) for g in o.group}) == 1, ("mismatched collective", [g.name for g in o.group])
                    start = max(t_arrive(g) for g in o.group)
                    for g in o.group:
                        g.start, g.end = start, start + o.group[0].dur
                else:
                    o.start = t_arrive(o)
                    o.end = o.start + o.dur
            return o.end

        for o in self.ops:
            t_end(o)


def build(n, steps, nbuf, pipelined, own_barrier_comm, rng, dur):
    """The host program of bench.py's step_dev(), exchange == 'ce', W == 1, replayed for every rank."""
    m = Model(n, rng, dur)
    prev_barrier = [None] * n
    barriers = {}

    def expand_push(r, k):
        ex = m.op(r, "main", "expand", k)                                    # writes slot r of r's set k % nbuf
        deps = [ex] + ([prev_barrier[r]] if prev_barrier[r] is not None else [])
        go = m.op(r, "copy", "go", k, deps)
        done = [m.op(r, "peer%d" % s, "push", k, [go], peer=s) for s in range(n) if s != r]
        joined = m.op(r, "copy", "join", k, done)
        prev_barrier[r] = m.collective(r, "bar" if own_barrier_comm else "data", "barrier", k, [joined])
        barriers[(r, k)] = prev_barrier[r]

    def compute(r, k):
        fd = m.op(r, "main", "first_dim", k, [barriers.pop((r, k))])         # reads every slot of r's set k % nbuf
        ag = m.collective(r, "data", "gather", k, [fd])
        m.op(r, "main", "finish", k, [ag])                                   # reads slot r of r's set k % nbuf (v)

    # the ranks' host threads run the same program; interleave them rank by rank per host step (order between ranks is irrelevant
    # for the graph: only per-rank issue order matters)
    for k in range(steps):
        for r in range(n):
            if pipelined:
                if k == 0:
                    expand_push(r, 0)
                expand_push(r, k + 1)
                compute(r, k)
            else:
                expand_push(r, k)
                compute(r, k)
    if pipelined:                                # drain: the extra expansion's barrier must be entered by everyone (it is)
        pass
    m.solve()
    return m


def hazards(m, nbuf):
    """[(what, op names)] over the solved model."""
    by = {}
    for o in m.ops:
        by.setdefault((o.kind, o.rank, o.step), []).append(o)
    bad = []
    for o in m.ops:
        if o.kind == "push":
            dst, k = o.peer, o.step
            # readers of the slot being overwritten: the destination's first dimension of the previous users of this set
            for old in range(k - nbuf, -1, -nbuf):
                for rd in by.get(("first_dim", dst, old), []):
                    if o.start < rd.end:
                        bad.append(("push overwrites a set still being read", o.name, rd.name))
            # and the destination must not read step k before this push has landed
            for rd in by.get(("first_dim", dst, k), []):
                if rd.start < o.end:
                    bad.append(("first dimension before the slot landed", rd.name, o.name))
        if o.kind == "expand":
            r, k = o.rank, o.step
            for old in range(k - nbuf, -1, -nbuf):
                for kind in ("first_dim", "finish"):
                    for rd in by.get((kind, r, old), []):
                        if o.start < rd.end:
                            bad.append(("expansion overwrites its own slot too early", o.name, rd.name))
                for ps in m.ops:                                             # its own pushes of the old step read the slot too
                    if ps.kind == "push" and ps.rank == r and ps.step == old and o.start < ps.end:
                        bad.append(("expansion overwrites a slot still being pushed", o.name, ps.name))
    return bad


WILD = {"expand": (0.1, 5.0), "go": (0.0, 0.0), "push": (0.1, 12.0), "join": (0.0, 0.0), "barrier": (0.01, 0.3),
        "first_dim": (0.1, 8.0), "gather": (0.01, 1.0), "finish": (0.05, 2.0)}


@pytest.mark.parametrize("n", [2, 4, 8])
def test_three_sets_are_safe_when_pipelined(n):
    for seed in range(60):
        m = build(n, 9, 3, True, seed % 2 == 0, random.Random(seed * 31 + n), WILD)
        assert hazards(m, 3) == [], seed


def test_two_sets_are_safe_too_thanks_to_the_all_gather():
    for seed in range(60):
        m = build(4, 9, 2, True, True, random.Random(seed), WILD)
        assert hazards(m, 2) == [], seed


def test_one_set_is_not_enough_when_pipelined_and_the_checker_sees_it():
    found = 0
    for seed in range(60):
        m = build(4, 9, 1, True, True, random.Random(seed), WILD)
        found += bool(hazards(m, 1))
    assert found > 30


@pytest.mark.parametrize("n", [2, 8])
def test_one_set_is_enough_without_the_pipeline(n):
    for seed in range(40):
        m = build(n, 8, 1, False, True, random.Random(seed + 1000 * n), WILD)
        assert hazards(m, 1) == [], seed


def test_shared_communicator_queues_the_gather_behind_the_next_transfer():
    """Model durations of an 8-GPU step (expansion 2.6 ms, first dimension + local fold 5.75 ms, pushes 6-10 ms, finish
    0.3 ms; stage proportions of the S8 workload, not an H100 measurement).  Shared communicator: ~12.5 ms per step; own
    communicator for the barriers: ~9-10 ms."""
    dur = {"expand": (2.6, 2.65), "go": (0, 0), "push": (6.0, 10.0), "join": (0, 0), "barrier": (0.03, 0.05),
           "first_dim": (5.7, 5.8), "gather": (0.3, 0.5), "finish": (0.27, 0.3)}

    def ms_per_step(own):
        m = build(8, 24, 3, True, own, random.Random(7), dur)
        ends = sorted(o.end for o in m.ops if o.kind == "finish" and o.rank == 0)
        return (ends[-1] - ends[3]) / (len(ends) - 4)

    shared, own = ms_per_step(False), ms_per_step(True)
    assert 11.5 < shared < 14.0, shared
    assert own < 10.6 and shared - own > 1.5, (shared, own)
