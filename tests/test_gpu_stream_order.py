"""Stream order of the device-pointer entry points, and of the host entry points beside other work on the GPU.

bench.py hands the library torch's current stream (the legacy default stream) and measures b200pir_process_query_batch_dev, the
three-phase calls, the two NTT _dev calls and the DoublePIR matvec there; include/b200pir.h promises that these calls are
stream-ordered and synchronise nothing.  A test that synchronises the host between steps cannot tell stream order from luck, so
every case here holds the stream back deterministically: torch.cuda._sleep() is queued first, sized from a measurement of the
same work in the same test (3x its device time plus 50 ms), and the inputs are copied in, the library is called, the outputs
are copied out and the inputs overwritten, all behind the sleep, before the host waits once.  Every buffer starts out holding
other valid data (other queries, other responses, other partials), so work issued on the wrong stream reads the wrong bytes
rather than garbage.  Results are compared byte for byte with the host path on the context's own stream, or with the oracle.

A  the _dev entry points on a caller's non-blocking stream and on the legacy default stream (bench.py's set_stream(0))
B  a warmed _dev call returns while its stream, or a busy legacy stream beside it, is still running
C  the host entry points (context and database creation, every writer, DoublePIR) beside a busy legacy or unrelated stream
D  switching streams between calls, and the profiling levels"""
import gc
import time

import numpy as np
import pytest

import oracle_lib as O
import update_rows_oracle as U

pytestmark = pytest.mark.gpu

SEED = 0xB1755
Q0, Q1 = 268369921, 249561089
GIB = 1 << 30
POLY = 2048
SLEEP_BUDGET_MS = 30000.0


# ------------------------------------------------------------------------------------------------ holding a stream back
class _Delay:
    """torch.cuda._sleep() calibrated once with CUDA events; keeps the file's total sleep time in check."""

    def __init__(self):
        import torch
        self.torch = torch
        s = torch.cuda.Stream()
        best = 0.0
        for cycles in (5_000_000, 20_000_000, 20_000_000):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            with torch.cuda.stream(s):
                e0.record()
                torch.cuda._sleep(cycles)
                e1.record()
            s.synchronize()
            best = max(best, cycles / max(e0.elapsed_time(e1), 1e-3))
        self.cycles_per_ms = best             # the fastest clock seen: a sleep of n ms lasts at least n ms
        self.total_ms = 0.0

    def sleep(self, stream, ms):
        assert self.total_ms + ms < SLEEP_BUDGET_MS, "this file's sleeps would exceed %.0f s" % (SLEEP_BUDGET_MS / 1e3)
        self.total_ms += ms
        with self.torch.cuda.stream(stream):
            self.torch.cuda._sleep(int(ms * self.cycles_per_ms))

    def device_ms(self, stream, fn):
        """device time of fn()'s work on `stream` (events around one undelayed call)"""
        torch = self.torch
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        with torch.cuda.stream(stream):
            e0.record()
            fn()
            e1.record()
        stream.synchronize()
        return e0.elapsed_time(e1)

    def ordered(self, stream, work_ms, before, call, after):
        """sleep (3x the work + 50 ms), then before(), call(), after() on `stream`; one host wait at the end"""
        self.sleep(stream, 3 * work_ms + 50)
        with self.torch.cuda.stream(stream):
            before()
            call()
            after()
        stream.synchronize()


@pytest.fixture(scope="module")
def delay():
    d = _Delay()
    yield d
    print("\ntest_gpu_stream_order: %.2f s of sleeps" % (d.total_ms / 1e3))


@pytest.fixture(scope="module")
def streams():
    """(caller's non-blocking stream, a second one, the legacy default stream): they outlive every context of this module"""
    import torch
    return torch.cuda.Stream(), torch.cuda.Stream(), torch.cuda.default_stream()


def _lib():
    from sdk_b200._lib import LIB, check
    return LIB, check


def _dev_u64(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a).view(np.int64)).cuda()


# ------------------------------------------------------------------------------------------------ S8, the benchmark's geometry
def _s8_items(P, count):
    """item 0, the last item, one in the last 32-row tile, one in the last 32-j tile, then a spread"""
    n_items = P.dim0 * P.num_per
    special = [0, n_items - 1, 3 * P.num_per + (P.num_per - 26), (P.dim0 - 12) * P.num_per + 7]
    spread = [(7919 * k + 31) % n_items for k in range(count)]
    return (special + [i for i in spread if i not in special])[:count]


class _S8:
    def __init__(self):
        import torch
        import sdk_b200.spiral as S
        self.torch, self.S = torch, S
        self.P = P = O.Params.named("S8")
        self.cl = O.Client(P, 8)
        self.pp = self.cl.generate_keys()
        gc.collect()
        torch.cuda.empty_cache()
        self.free_at_start, self.total = torch.cuda.mem_get_info()
        self.G = G = S.Params(**P.kw)
        self.gdb = S.Database(G)
        self.gdb.fill_synthetic(SEED)
        self.gpp = S.PublicParameters(G, self.pp["pack"], self.pp.get("left"), self.pp.get("right"), self.pp.get("conv"))
        G.set_option("batch", 16)                                  # bench.py's setting at S8
        self.rb = G.response_bytes
        # the workspace of the largest call, reserved up front (Q = 128: eight database passes)
        self.qmax, self.skip128 = 128, None
        try:
            G.reserve(128, P.num_per)
        except S.B200PirError as e:
            if "out of memory" not in str(e).lower():
                raise
            self.qmax = 32
            G.reserve(32, P.num_per)
            self.skip128 = ("the workspace of 128 S8 queries does not fit: %.1f GiB were free of %.1f GiB before the database (%s)"
                            % (self.free_at_start / GIB, self.total / GIB, e))
        self.idxs = _s8_items(P, self.qmax)
        self.cts = np.concatenate([self.cl.generate_query(i)["ct"] for i in self.idxs])
        other = [(104729 * k + 17) % (P.dim0 * P.num_per) for k in range(self.qmax)]
        self.decoy_cts = np.concatenate([self.cl.generate_query(i)["ct"] for i in other])
        # the reference: the host path on the context's own stream, in passes of at most 16 queries
        qw = 2 * POLY
        self.refs = np.concatenate([S.process_query_batch(G, self.gpp, self.cts[k * qw:(k + 16) * qw], self.gdb)
                                    for k in range(0, self.qmax, 16)])
        for k, i in enumerate(self.idxs):
            assert np.array_equal(self.cl.decode_response(self.refs[k]), P.db_plain_item(SEED, i)), (k, i)
        self.d_real = _dev_u64(self.cts)
        self.d_decoy = _dev_u64(self.decoy_cts)
        self.d_q = self.d_decoy.clone()
        self.d_out = torch.zeros(self.qmax * self.rb, dtype=torch.uint8, device="cuda")
        self.out_copy = torch.zeros_like(self.d_out)
        torch.cuda.synchronize()                                   # the buffers above were filled on the legacy stream

    def call(self, Q, q=None, out=None):
        LIB, check = _lib()
        check(LIB.b200pir_process_query_batch_dev(self.G._h, self.gdb._h, self.gpp._h, (q if q is not None else self.d_q).data_ptr(),
                                                  Q, (out if out is not None else self.d_out).data_ptr()))

    def run_ordered(self, delay, stream, Q):
        """decoys through the same call undelayed (timed; leaves the workspace and d_out holding their results), then the real
        queries behind the sleep; returns the Q responses copied out on the stream"""
        torch = self.torch
        self.G.set_stream(stream.cuda_stream)
        with torch.cuda.stream(stream):
            self.d_q.copy_(self.d_decoy)
            self.out_copy.zero_()
        ms = delay.device_ms(stream, lambda: self.call(Q))
        n = Q * 2 * POLY

        def before():
            self.d_q[:n].copy_(self.d_real[:n])

        def after():
            self.out_copy[:Q * self.rb].copy_(self.d_out[:Q * self.rb])
            self.d_q.copy_(self.d_decoy)

        delay.ordered(stream, ms, before, lambda: self.call(Q), after)
        return self.out_copy[:Q * self.rb].cpu().numpy().reshape(Q, self.rb)

    def close(self):
        for h in (self.gpp, self.gdb, self.G):
            h.close()


@pytest.fixture(scope="module")
def s8(streams):
    f = _S8()
    yield f
    f.close()


def _stream(streams, which):
    return streams[0] if which == "caller" else streams[2]


@pytest.mark.parametrize("which", ["caller", "legacy"])
@pytest.mark.parametrize("Q", [1, 16, 17, 32, 128])
def test_a_process_query_batch_dev_on_callers_stream(s8, delay, streams, Q, which):
    if Q > s8.qmax:
        pytest.skip(s8.skip128)
    got = s8.run_ordered(delay, _stream(streams, which), Q)
    for k in range(Q):
        assert np.array_equal(got[k], s8.refs[k]), (Q, which, k, s8.idxs[k])


def test_a_s8_image_flow_world_2_equals_single_gpu(s8, delay, streams):
    """bench.py's N = 2 flow on one GPU at S8: each rank expands 16 queries into one tile image, both shards multiply from both
    images and fold, each rank finishes its own 16; no host synchronise between the phases."""
    torch = s8.torch
    LIB, check = _lib()
    P, G, S = s8.P, s8.G, s8.S
    world, per_rank = 2, 16
    total = world * per_rank
    shards = []
    try:
        for r in range(world):
            sh = S.Database(G, shard_index=r, shard_count=world, fmt=2)
            sh.fill_synthetic(SEED)
            shards.append(sh)
        stream = streams[0]
        G.set_stream(stream.cuda_stream)
        img = int(LIB.b200pir_query_image_bytes(G._h))
        fold_words = P.nu_2 * 2 * 2 * P.t_gsw * 2 * P.N
        part_words = total * P.slices * 4 * P.N
        images = torch.zeros(world * img, dtype=torch.uint8, device="cuda")
        vf = torch.zeros(total * fold_words, dtype=torch.int32, device="cuda")
        gathered = torch.zeros(world * part_words, dtype=torch.int32, device="cuda")
        out = torch.zeros(total * s8.rb, dtype=torch.uint8, device="cuda")
        out_copy = torch.zeros_like(out)
        d_q = s8.d_decoy[:total * 2 * POLY].clone()
        torch.cuda.synchronize()

        def flow():
            for r in range(world):
                check(LIB.b200pir_expand_queries_images_dev(G._h, s8.gpp._h, d_q.data_ptr() + r * per_rank * 2 * POLY * 8, per_rank,
                                                            images.data_ptr() + r * img, vf.data_ptr() + r * per_rank * fold_words * 4))
            for r in range(world):
                check(LIB.b200pir_first_dim_fold_images_dev(G._h, shards[r]._h, images.data_ptr(), world, per_rank, vf.data_ptr(),
                                                            gathered.data_ptr() + r * part_words * 4))
            for r in range(world):
                check(LIB.b200pir_finish_queries_dev(G._h, s8.gpp._h, gathered.data_ptr(), world, total, r * per_rank, per_rank,
                                                     vf.data_ptr() + r * per_rank * fold_words * 4,
                                                     out.data_ptr() + r * per_rank * s8.rb))

        ms = delay.device_ms(stream, flow)                     # the decoys: every buffer now holds their images and partials
        delay.ordered(stream, ms, lambda: d_q.copy_(s8.d_real[:total * 2 * POLY]), flow,
                      lambda: (out_copy.copy_(out), d_q.copy_(s8.d_decoy[:total * 2 * POLY])))
        got = out_copy.cpu().numpy().reshape(total, s8.rb)
        for k in range(total):
            assert np.array_equal(got[k], s8.refs[k]), (k, s8.idxs[k])
    finally:
        for sh in shards:
            sh.close()


# ------------------------------------------------------------------------------------------------ the small sets, sharded
_small = {}


class _Small:
    """one of the oracle's small sets, world = 2 row shards (format 2), the oracle's responses to `count` queries"""

    def __init__(self, name, count=4):
        import torch
        import sdk_b200.spiral as S
        self.torch, self.S = torch, S
        self.P = P = O.Params.named(name)
        self.cl = O.Client(P, 77)
        self.pp = self.cl.generate_keys()
        self.db = P.generate_db(SEED)
        self.G = G = S.Params(**P.kw)
        self.gpp = S.PublicParameters(G, self.pp["pack"], self.pp.get("left"), self.pp.get("right"), self.pp.get("conv"))
        self.world = 2
        slice_words = P.dim0 * P.num_per * P.N
        self.shards = []
        for r in range(self.world):
            sh = S.Database(G, shard_index=r, shard_count=self.world, fmt=2)
            for sl in range(P.slices):
                sh.upload_slice(sl, self.db[sl * slice_words:(sl + 1) * slice_words])
            self.shards.append(sh)
        n_items = P.dim0 * P.num_per
        self.count = count
        self.idxs = [0, n_items - 1] + [(37 * k + 11) % n_items for k in range(count - 2)]
        qs = [self.cl.generate_query(i)["ct"] for i in self.idxs]
        self.cts = np.concatenate(qs)
        self.refs = [P.process_query(self.pp, dict(ct=q), self.db) for q in qs]
        self.d_real = _dev_u64(self.cts)
        self.d_decoy = _dev_u64(np.concatenate([self.cl.generate_query((i + 5) % n_items)["ct"] for i in self.idxs]))
        self.rb = G.response_bytes

    def close(self):
        for h in self.shards + [self.gpp, self.G]:
            h.close()


def small(name):
    if name not in _small:
        _small[name] = _Small(name)
    return _small[name]


@pytest.fixture(scope="module", autouse=True)
def _close_small(streams):
    yield
    for f in _small.values():
        f.close()
    _small.clear()


class _ThreePhase:
    """expand -> first_dim_fold -> finish for world = 2 on one GPU (uint4 operands or tile images), caller-owned buffers"""

    def __init__(self, f, images):
        torch = f.torch
        LIB, check = _lib()
        self.f, self.images = f, images
        P = f.P
        self.per = f.count // f.world
        self.fold_words = P.nu_2 * 2 * 2 * P.t_gsw * 2 * P.N
        self.part_words = f.count * P.slices * 4 * P.N
        self.img = int(LIB.b200pir_query_image_bytes(f.G._h))
        self.qexp_words = P.dim0 * P.N * 4
        self.q = torch.zeros(f.world * self.img if images else f.count * self.qexp_words * 4, dtype=torch.uint8, device="cuda")
        self.vf = torch.zeros(f.count * self.fold_words, dtype=torch.int32, device="cuda")
        self.gathered = torch.zeros(f.world * self.part_words, dtype=torch.int32, device="cuda")
        self.out = torch.zeros(f.count * f.rb, dtype=torch.uint8, device="cuda")
        self.out_copy = torch.zeros_like(self.out)
        self.d_q = f.d_decoy.clone()
        torch.cuda.synchronize()

    def run(self):
        LIB, check = _lib()
        f, G = self.f, self.f.G
        for r in range(f.world):
            src = self.d_q.data_ptr() + r * self.per * 2 * POLY * 8
            vf = self.vf.data_ptr() + r * self.per * self.fold_words * 4
            if self.images:
                check(LIB.b200pir_expand_queries_images_dev(G._h, f.gpp._h, src, self.per, self.q.data_ptr() + r * self.img, vf))
            else:
                check(LIB.b200pir_expand_queries_dev(G._h, f.gpp._h, src, self.per,
                                                     self.q.data_ptr() + r * self.per * self.qexp_words * 4, vf))
        for r in range(f.world):
            part = self.gathered.data_ptr() + r * self.part_words * 4
            if self.images:
                check(LIB.b200pir_first_dim_fold_images_dev(G._h, f.shards[r]._h, self.q.data_ptr(), f.world, self.per,
                                                            self.vf.data_ptr(), part))
            else:
                check(LIB.b200pir_first_dim_fold_dev(G._h, f.shards[r]._h, self.q.data_ptr(), self.vf.data_ptr(), f.count, part))
        for r in range(f.world):
            check(LIB.b200pir_finish_queries_dev(G._h, f.gpp._h, self.gathered.data_ptr(), f.world, f.count, r * self.per, self.per,
                                                 self.vf.data_ptr() + r * self.per * self.fold_words * 4,
                                                 self.out.data_ptr() + r * self.per * f.rb))

    def before(self):
        self.d_q.copy_(self.f.d_real)

    def after(self):
        self.out_copy.copy_(self.out)
        self.d_q.copy_(self.f.d_decoy)

    def check(self, what):
        got = self.out_copy.cpu().numpy().reshape(self.f.count, self.f.rb)
        for k in range(self.f.count):
            assert np.array_equal(got[k], self.f.refs[k]), what + (k, self.f.idxs[k])


@pytest.mark.parametrize("which", ["caller", "legacy"])
@pytest.mark.parametrize("images", [False, True])
@pytest.mark.parametrize("name", ["T0", "T1"])
def test_a_three_phase_world_2_on_callers_stream(delay, streams, name, images, which):
    f = small(name)
    stream = _stream(streams, which)
    f.G.set_stream(stream.cuda_stream)
    tp = _ThreePhase(f, images)
    ms = delay.device_ms(stream, tp.run)                    # the decoys first: every buffer holds their results
    delay.ordered(stream, ms, tp.before, tp.run, tp.after)
    tp.check((name, images, which))


@pytest.mark.parametrize("which", ["caller", "legacy"])
def test_a_stage_a_stage_b_world_2_on_callers_stream(delay, streams, which):
    LIB, check = _lib()
    f = small("T")
    torch = f.torch
    P, G = f.P, f.G
    stream = _stream(streams, which)
    G.set_stream(stream.cuda_stream)
    part_words = f.count * P.slices * 4 * P.N
    gathered = torch.zeros(f.world * part_words, dtype=torch.int32, device="cuda")
    out = torch.zeros(f.count * f.rb, dtype=torch.uint8, device="cuda")
    out_copy = torch.zeros_like(out)
    d_q = f.d_decoy.clone()
    torch.cuda.synchronize()

    def run():
        for r in range(f.world):
            check(LIB.b200pir_query_stage_a_dev(G._h, f.shards[r]._h, f.gpp._h, d_q.data_ptr(), f.count,
                                                gathered.data_ptr() + r * part_words * 4))
        check(LIB.b200pir_query_stage_b_dev(G._h, f.gpp._h, gathered.data_ptr(), f.world, f.count, out.data_ptr()))

    ms = delay.device_ms(stream, run)
    delay.ordered(stream, ms, lambda: d_q.copy_(f.d_real), run, lambda: (out_copy.copy_(out), d_q.copy_(f.d_decoy)))
    got = out_copy.cpu().numpy().reshape(f.count, f.rb)
    for k in range(f.count):
        assert np.array_equal(got[k], f.refs[k]), (which, k, f.idxs[k])


# ------------------------------------------------------------------------------------------------ BASELINE config #5 transforms
def _ntt_batch(poly_len, count, seed):
    rng = np.random.default_rng(seed)
    h = np.empty((count, 2, poly_len), dtype=np.uint32)
    h[:, 0, :] = rng.integers(0, Q0, (count, poly_len), dtype=np.uint32)
    h[:, 1, :] = rng.integers(0, Q1, (count, poly_len), dtype=np.uint32)
    h[0] = 0
    h[1, 0, :], h[1, 1, :] = Q0 - 1, Q1 - 1
    return h


def _oracle_fwd(poly_len, poly, Po):
    ref = np.ascontiguousarray(poly.astype(np.uint64).reshape(-1))
    if poly_len == 2048:
        return Po.ntt_forward(ref)
    assert O.LIB.orc_ntt4096(O._p64(ref), 1, 0) == 0
    return ref


@pytest.mark.parametrize("which", ["caller", "legacy"])
@pytest.mark.parametrize("poly_len", [2048, 4096])
def test_a_ntt_dev_on_callers_stream_from_a_fresh_context(delay, streams, poly_len, which):
    """forward then inverse on 2^12 polynomials behind the sleep; the first transform is the context's first call"""
    import torch
    import sdk_b200.spiral as S
    LIB, check = _lib()
    Po = O.Params.named("T")
    count = 1 << 12
    host = _ntt_batch(poly_len, count, poly_len + 1)
    other = _ntt_batch(poly_len, count, poly_len + 2)
    fn = LIB.b200pir_ntt32_dev if poly_len == 2048 else LIB.b200pir_ntt4096_dev
    stream = _stream(streams, which)
    src = torch.from_numpy(host.view(np.int32)).cuda()
    garbage = torch.from_numpy(other.view(np.int32)).cuda()
    d = garbage.clone()
    fwd, inv = torch.zeros_like(d), torch.zeros_like(d)
    torch.cuda.synchronize()
    # the device time of the pair, on a context of its own, so that the one under test starts fresh
    Gt = S.Params(**Po.kw)
    Gt.set_stream(stream.cuda_stream)
    ms = delay.device_ms(stream, lambda: (check(fn(Gt._h, d.data_ptr(), count, 0)), check(fn(Gt._h, d.data_ptr(), count, 1))))
    Gt.close()
    G = S.Params(**Po.kw)
    try:
        G.set_stream(stream.cuda_stream)
        delay.ordered(stream, ms, lambda: d.copy_(src),
                      lambda: (check(fn(G._h, d.data_ptr(), count, 0)), fwd.copy_(d), check(fn(G._h, d.data_ptr(), count, 1))),
                      lambda: (inv.copy_(d), d.copy_(garbage)))
    finally:
        G.close()
    f = fwd.cpu().numpy().view(np.uint32)
    for i in (0, 1, 2, 777, count // 2, count - 1):
        assert np.array_equal(f[i].astype(np.uint64).reshape(-1), _oracle_fwd(poly_len, host[i], Po)), (poly_len, which, i)
    assert np.array_equal(inv.cpu().numpy().view(np.uint32), host), (poly_len, which)


# ------------------------------------------------------------------------------------------------ DoublePIR config #4 matvec
def test_a_dpir_matvec_packed_dev_on_callers_stream(delay, streams):
    import torch
    import sdk_b200.doublepir as D
    import test_gpu_dpir_end_to_end as TE
    import test_oracle_doublepir_e2e as E
    LIB, check = _lib()
    rows, cols = 16899, 1366
    a, b = TE.extreme_operands(rows, cols, 4)
    _, b2 = TE.extreme_operands(rows, cols, 5)
    ref = E.np_matvec_packed(a, b, rows, cols)
    stream = streams[0]
    m = D.PackedMatrix(a, rows, cols)
    try:
        check(LIB.b200pir_dpir_set_stream(m._h, stream.cuda_stream))
        real = torch.from_numpy(b.view(np.int32)).cuda()
        decoy = torch.from_numpy(b2.view(np.int32)).cuda()
        b_dev = decoy.clone()
        out = torch.zeros(rows, dtype=torch.int32, device="cuda")
        out_copy = torch.zeros_like(out)
        torch.cuda.synchronize()
        for variant in (0, 1, 2, 4):                           # 1, 2 and 4 are retired tilings: accepted, and they select nothing
            call = lambda: check(LIB.b200pir_dpir_matvec_packed_dev(m._h, b_dev.data_ptr(), out.data_ptr(), variant))
            ms = delay.device_ms(stream, call)                 # out now holds the decoy vector's product
            delay.ordered(stream, ms, lambda: b_dev.copy_(real), call, lambda: (out_copy.copy_(out), b_dev.copy_(decoy)))
            assert np.array_equal(out_copy.cpu().numpy().view(np.uint32), ref), variant
    finally:
        m.close()


# ------------------------------------------------------------------------------------------------ B: nothing is synchronised
def _returns_while_busy(delay, busy, call, work_ms):
    """queue a long sleep on `busy`, make the call, and report whether `busy` was still running when the call returned"""
    delay.sleep(busy, 3 * work_ms + 200)
    call()
    still_busy = not busy.query()
    busy.synchronize()
    return still_busy


@pytest.mark.parametrize("busy", ["caller", "legacy"])
def test_b_process_query_batch_dev_does_not_synchronise(s8, delay, streams, busy):
    """caller: the context runs on the stream the sleep is on; legacy: the sleep is on the legacy default stream and the
    context on a non-blocking stream of its own"""
    import torch
    stream = streams[0] if busy == "caller" else streams[1]
    busy_stream = stream if busy == "caller" else streams[2]
    s8.G.set_stream(stream.cuda_stream)
    with torch.cuda.stream(stream):
        s8.d_q.copy_(s8.d_real)
    ms = delay.device_ms(stream, lambda: s8.call(16))           # warm: same pp, same batch, workspace reserved
    with torch.cuda.stream(stream):
        s8.d_out.zero_()
    assert _returns_while_busy(delay, busy_stream, lambda: s8.call(16), ms), busy
    torch.cuda.synchronize()
    got = s8.d_out[:16 * s8.rb].cpu().numpy().reshape(16, s8.rb)
    assert np.array_equal(got, s8.refs[:16]), busy


@pytest.mark.parametrize("busy", ["caller", "legacy"])
def test_b_three_phase_does_not_synchronise(delay, streams, busy):
    import torch
    f = small("T0")
    stream = streams[0] if busy == "caller" else streams[1]
    busy_stream = stream if busy == "caller" else streams[2]
    f.G.set_stream(stream.cuda_stream)
    for images in (False, True):
        tp = _ThreePhase(f, images)
        with torch.cuda.stream(stream):
            tp.before()
        ms = delay.device_ms(stream, tp.run)
        with torch.cuda.stream(stream):
            tp.out.zero_()
        assert _returns_while_busy(delay, busy_stream, tp.run, ms), (busy, images)
        torch.cuda.synchronize()
        tp.out_copy.copy_(tp.out)
        tp.check((busy, images))


@pytest.mark.parametrize("busy", ["caller", "legacy"])
@pytest.mark.parametrize("poly_len", [2048, 4096])
def test_b_ntt_dev_first_call_does_not_synchronise(delay, streams, poly_len, busy):
    """the first transform on a fresh context: for poly_len 4096 it once built and uploaded its tables on first use"""
    import torch
    import sdk_b200.spiral as S
    LIB, check = _lib()
    Po = O.Params.named("T")
    count = 1 << 12
    host = _ntt_batch(poly_len, count, poly_len + 3)
    fn = LIB.b200pir_ntt32_dev if poly_len == 2048 else LIB.b200pir_ntt4096_dev
    stream = streams[0] if busy == "caller" else streams[1]
    busy_stream = stream if busy == "caller" else streams[2]
    d = torch.from_numpy(host.view(np.int32)).cuda()
    Gt = S.Params(**Po.kw)
    Gt.set_stream(stream.cuda_stream)
    ms = delay.device_ms(stream, lambda: check(fn(Gt._h, d.data_ptr(), count, 0)))
    Gt.close()
    d.copy_(torch.from_numpy(host.view(np.int32)))
    torch.cuda.synchronize()
    G = S.Params(**Po.kw)
    try:
        G.set_stream(stream.cuda_stream)
        assert _returns_while_busy(delay, busy_stream, lambda: check(fn(G._h, d.data_ptr(), count, 0)), ms), (poly_len, busy)
        torch.cuda.synchronize()
        f = d.cpu().numpy().view(np.uint32)
        for i in (0, 1, count - 1):
            assert np.array_equal(f[i].astype(np.uint64).reshape(-1), _oracle_fwd(poly_len, host[i], Po)), (poly_len, busy, i)
        # and a warmed call, inverse
        assert _returns_while_busy(delay, busy_stream, lambda: check(fn(G._h, d.data_ptr(), count, 1)), ms), (poly_len, busy)
        torch.cuda.synchronize()
        assert np.array_equal(d.cpu().numpy().view(np.uint32), host), (poly_len, busy)
    finally:
        G.close()


# ------------------------------------------------------------------------------------------------ C: host entry points beside work
_C_ITEMS = dict(plain=200, upsert=77, raw=130, many=(5, 255))


def _c_inputs(P):
    """the writes of the sequence and the plaintext every read must decode to"""
    rng = np.random.default_rng(61)
    n_items = P.dim0 * P.num_per
    other = P.generate_db(SEED + 1)
    slice_words = P.dim0 * P.num_per * P.N
    up_slice, iu = 1, _C_ITEMS["upsert"]
    poly = np.ascontiguousarray(other[up_slice * slice_words:(up_slice + 1) * slice_words]
                                .reshape(P.N, P.num_per, P.dim0)[:, iu % P.num_per, iu // P.num_per])
    raw = rng.integers(0, 256, P.slices * P.bytes_per_chunk, dtype=np.uint8)
    many = {i: rng.integers(0, 256, P.slices * P.bytes_per_chunk, dtype=np.uint8) for i in _C_ITEMS["many"]}
    body = b"".join(U.entry(i, d) for i, d in many.items())
    file_words = P.generate_db(SEED + 2)
    expect_a = {}
    for i in (_C_ITEMS["plain"], iu, _C_ITEMS["raw"]) + _C_ITEMS["many"]:
        expect_a[i] = P.db_plain_item(SEED, i).reshape(P.slices, P.N).copy()
    expect_a[iu][up_slice] = P.db_plain_item(SEED + 1, iu).reshape(P.slices, P.N)[up_slice]
    for i, d in [(_C_ITEMS["raw"], raw)] + list(many.items()):
        e = np.zeros((P.slices, P.N), dtype=np.uint64)
        e[:, :P.bytes_per_chunk] = d.reshape(P.slices, P.bytes_per_chunk)
        expect_a[i] = e
    expect_b = {i: P.db_plain_item(SEED + 2, i).reshape(P.slices, P.N) for i in (0, n_items - 1, 100)}
    return dict(up_slice=up_slice, poly=poly, raw=raw, body=body, file_words=file_words, expect_a=expect_a, expect_b=expect_b)


def _c_sequence(P, pp, fmt, w, path, busy):
    """context, database A (synthetic fill, upsert_item, update_item_raw, update_many_items), database B (load_file), one
    busy() before each creation; then torch.cuda.synchronize() and the reads.  Returns {(db, item): response}."""
    import torch
    import sdk_b200.spiral as S
    busy()
    G = S.Params(**P.kw)
    dbs = []
    try:
        busy()
        a = S.Database(G, fmt=fmt)
        dbs.append(a)
        a.fill_synthetic(SEED)
        a.upsert_item(w["up_slice"], _C_ITEMS["upsert"], w["poly"])
        a.update_item_raw(_C_ITEMS["raw"], w["raw"])
        a.update_many_items(w["body"])
        busy()
        b = S.Database.from_file(G, path, fmt=fmt)
        dbs.append(b)
        gpp = S.PublicParameters(G, pp["pack"], pp.get("left"), pp.get("right"), pp.get("conv"))
        dbs.append(gpp)
        torch.cuda.synchronize()
        out = {}
        for name, db, items in (("a", a, w["expect_a"]), ("b", b, w["expect_b"])):
            assert db.info()["format"] == fmt
            for i in items:
                out[(name, i)] = S.process_query(G, gpp, S.Query(ct=w["cts"][i]), db)
        return out
    finally:
        for h in reversed(dbs):
            h.close()
        G.close()


@pytest.fixture(scope="module")
def c_case(tmp_path_factory):
    P = O.Params.named("T")
    cl = O.Client(P, 62)
    pp = cl.generate_keys()
    w = _c_inputs(P)
    w["cts"] = {i: cl.generate_query(i)["ct"] for i in set(w["expect_a"]) | set(w["expect_b"])}
    path = tmp_path_factory.mktemp("stream_order") / "db.bin"
    w["file_words"].tofile(path)
    return P, cl, pp, w, path


@pytest.mark.parametrize("busy", ["legacy", "other"])
@pytest.mark.parametrize("fmt", [0, 1, 2])
def test_c_create_write_and_read_beside_a_busy_stream(c_case, delay, streams, fmt, busy):
    """format 2: the tile mask of a new database must be cleared on the context's stream, or a memset queued behind the busy
    legacy stream zeroes the mask words the first writes upload, and every tile is then skipped as absent"""
    P, cl, pp, w, path = c_case
    t0 = time.perf_counter()
    idle = _c_sequence(P, pp, fmt, w, path, lambda: None)
    idle_ms = (time.perf_counter() - t0) * 1e3
    stream = streams[2] if busy == "legacy" else streams[1]
    got = _c_sequence(P, pp, fmt, w, path, lambda: delay.sleep(stream, 3 * idle_ms + 50))
    for key, resp in got.items():
        exp = (w["expect_a"] if key[0] == "a" else w["expect_b"])[key[1]]
        assert np.array_equal(cl.decode_response(resp).reshape(P.slices, P.N), exp), (fmt, busy, key)
        assert np.array_equal(resp, idle[key]), (fmt, busy, key)


def test_c_dpir_create_and_answer_many_beside_a_busy_legacy_stream(delay, streams):
    import torch
    import sdk_b200.doublepir as D
    import test_gpu_dpir_end_to_end as TE
    import test_gpu_dpir_serve as TS
    import test_oracle_doublepir_e2e as E
    rows, cols = 4099, 1366
    a, b = TE.extreme_operands(rows, cols, 9)
    ref = E.np_matvec_packed(a, b, rows, cols)
    num_entries, bits, seed = 1 << 16, 32, 4
    prm, data, info, delta, a_1, a_2, st, got = TE.gpu_prepared(num_entries, bits, seed)
    rng = np.random.default_rng(71)
    pool = [E.query(int(i), a_1, a_2, prm, info, rng)[1] for i in rng.integers(0, num_entries, 5)]
    reqs = [pool[:1], pool[1:3], pool[3:]]
    wires = [D.serialize_request(q) for q in reqs]
    want = [TS.wire(E.run_answer(st, prm, info, delta, q), prm, info, delta) for q in reqs]
    # the one-shot ops: matmul, matrix_mul_transposed_packed and transpose_expand_concat_cols_squish
    mm_a = (rng.integers(0, 65536, (300, 70)).astype(np.int64) - 32768).astype(np.uint32)
    mm_b = rng.integers(0, 2**32, (70, 130), dtype=np.uint64).astype(np.uint32)
    mm_ref = ((mm_a.astype(np.uint64) @ mm_b.astype(np.uint64)) & np.uint64(0xFFFFFFFF)).astype(np.uint32)
    t_rows, t_cols, t_brows = 40, 150, 24
    t_a = rng.integers(0, 2**32, t_rows * t_cols, dtype=np.uint64).astype(np.uint32)
    t_b = rng.integers(0, 2**32, t_brows * 3 * t_cols, dtype=np.uint64).astype(np.uint32)
    t_ref = E.np_matrix_mul_transposed_packed(t_a, t_b, t_rows, t_cols, t_brows, 3 * t_cols)
    x_rows, x_cols, x_mod, x_delta, x_concat = 4 * 65, 3, 991, 4, 4
    x_a = rng.integers(0, 2**32, x_rows * x_cols, dtype=np.uint64).astype(np.uint32)
    x_ref = E.np_transpose_expand_concat_cols_squish(x_a, x_rows, x_cols, x_mod, x_delta, x_concat)

    def sequence():
        m = D.PackedMatrix(a, rows, cols)
        try:
            mv = D.matrix_mul_vec_packed(m, b)
        finally:
            m.close()
        dbm, srv = TS.setup_server(got, prm, info, num_entries, bits)
        try:
            many = srv.answer_many(wires)
        finally:
            srv.close()
            dbm.close()
        ops = (D.matmul(mm_a, mm_b), D.matrix_mul_transposed_packed(t_a, t_rows, t_cols, t_b, t_brows, 3 * t_cols),
               D.transpose_expand_concat_cols_squish(x_a, x_rows, x_cols, x_mod, x_delta, x_concat))
        return mv, many, ops

    def check_ops(ops):
        mm, mt, (x, xr, xc) = ops
        assert np.array_equal(mm, mm_ref)
        assert np.array_equal(mt, t_ref)
        assert (xr, xc) == x_ref[1:] and np.array_equal(x, x_ref[0])

    t0 = time.perf_counter()
    mv, many, ops = sequence()
    idle_ms = (time.perf_counter() - t0) * 1e3
    assert np.array_equal(mv, ref) and many == want
    check_ops(ops)
    delay.sleep(streams[2], 3 * idle_ms + 50)
    mv, many, ops = sequence()
    torch.cuda.synchronize()
    assert np.array_equal(mv, ref)
    assert many == want
    check_ops(ops)


# ------------------------------------------------------------------------------------------------ D: switching streams, profiling
def test_d_set_stream_between_dev_calls(delay, streams):
    """host path on the context's private stream first; then _dev calls on a caller's stream, the legacy stream, a second
    caller's stream and the first again, each behind a sleep on the stream it was handed"""
    import torch
    f = small("T")
    import sdk_b200.spiral as S
    P = f.P
    G = S.Params(**P.kw)
    try:
        gdb = S.Database.from_words(G, f.db)
        gpp = S.PublicParameters(G, f.pp["pack"], f.pp.get("left"), f.pp.get("right"), f.pp.get("conv"))
        host = S.process_query_batch(G, gpp, f.cts, gdb)                  # the private stream
        for k in range(f.count):
            assert np.array_equal(host[k], f.refs[k]), k
        LIB, check = _lib()
        d_q = f.d_decoy.clone()
        out = torch.zeros(f.count * f.rb, dtype=torch.uint8, device="cuda")
        out_copy = torch.zeros_like(out)
        torch.cuda.synchronize()
        call = lambda: check(LIB.b200pir_process_query_batch_dev(G._h, gdb._h, gpp._h, d_q.data_ptr(), f.count, out.data_ptr()))
        for n, stream in enumerate((streams[0], streams[2], streams[1], streams[0])):
            G.set_stream(stream.cuda_stream)
            with torch.cuda.stream(stream):
                d_q.copy_(f.d_decoy)
            ms = delay.device_ms(stream, call)
            delay.ordered(stream, ms, lambda: d_q.copy_(f.d_real), call, lambda: (out_copy.copy_(out), d_q.copy_(f.d_decoy)))
            assert np.array_equal(out_copy.cpu().numpy().reshape(f.count, f.rb), host), n
        gpp.close()
        gdb.close()
    finally:
        G.close()


def test_d_profile_levels_give_the_same_bytes_and_stage_times(s8, delay, streams):
    stream = streams[0]
    try:
        for level in (0, 1, 2):
            s8.G.set_option("profile", level)
            got = s8.run_ordered(delay, stream, 17)
            for k in range(17):
                assert np.array_equal(got[k], s8.refs[k]), (level, k)
        s8.G.set_option("profile", 2)                             # accumulate over the next calls
        for _ in range(3):
            s8.call(32)
        st = s8.G.last_stage_ms()
    finally:
        s8.G.set_option("profile", 0)
    assert st["multiply_launches"] == 3 * 2                       # two passes of 16 queries per call
    for k in ("expand", "multiply", "from_ntt", "fold", "pack", "encode"):
        assert st[k] > 0, (k, st)
    parts = sum(st[k] for k in ("expand", "multiply", "from_ntt", "fold", "pack", "encode", "query_image"))
    assert abs(st["total"] - parts) <= 1e-6 * max(parts, 1.0), st
