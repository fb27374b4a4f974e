"""DoublePIR entry updates on the GPU (b200pir_dpir_server_update): after every batch the squished store, the server's h_1 and
the returned hint equal what load() gives for the modified bytes (and, at small shapes, the oracle's load -> derive -> setup()),
answers equal a fresh server's on the modified bytes, and the numpy client decodes the new values with the new hint."""
import threading

import numpy as np
import pytest

import dpir_load_oracle as L
import oracle_lib as O
import test_oracle_doublepir_e2e as E

pytestmark = pytest.mark.gpu

E_BADARG, E_SHAPE, E_UNSUPPORTED = -1, -2, -4


def _D():
    import sdk_b200.doublepir as D
    return D


def _launches():
    from sdk_b200._lib import LIB
    return LIB.b200pir_kernel_launches()


class Db:
    """A loaded database, its server and the bytes it holds now."""

    def __init__(self, prm, num_entries, bits, data, bits_format, max_queries=65):
        D = _D()
        self.prm, self.num_entries, self.bits, self.bits_format = prm, num_entries, bits, bits_format
        self.fmt = D.ENTRY_BITS if bits_format else D.ENTRY_BYTES
        self.data = np.array(data, dtype=np.uint8)
        self.count = 8 * self.data.size if bits_format else self.data.size
        self.dbm, out, self.info = D.load(prm, num_entries, bits, self.data, self.fmt)
        self.h2, self.a2_t = out["h2"], out["a2_t"]
        self.srv = D.Server(self.dbm, out["h1_squished"], out["a2_t"], prm, num_entries, bits, max_queries=max_queries)

    def entry(self, i):
        return (int(self.data[i >> 3]) >> (i & 7)) & 1 if self.bits_format else int(self.data[i])

    def hi(self):
        return 2 if self.bits_format else (1 << self.bits if self.info["packing"] else 256)

    def update(self, upd):
        idx = np.array([i for i, _ in upd], dtype=np.uint64)
        val = np.array([v for _, v in upd], dtype=np.uint8)
        self.h2 = self.srv.update(idx, val, self.h2)
        for i, v in upd:
            if self.bits_format:
                self.data[i >> 3] = (int(self.data[i >> 3]) & ~(1 << (i & 7))) | (v << (i & 7))
            else:
                self.data[i] = v

    def reload(self):
        return _D().load(self.prm, self.num_entries, self.bits, self.data, self.fmt)

    def assert_equals_reload(self):
        dbm, out, _ = self.reload()
        assert np.array_equal(self.dbm.download(), dbm.download())
        assert np.array_equal(self.srv.state(), out["h1_squished"])
        assert np.array_equal(self.h2, out["h2"])
        dbm.close()
        return out

    def assert_equals_oracle(self):
        D = _D()
        prm, info = self.prm, self.info
        l, m, n, x = prm["l"], prm["m"], prm["n"], info["x"]
        db = L.dpir_load_data(self.data, self.bits_format, self.num_entries, self.bits, l, m, prm["p"])
        a_1 = L.dpir_derive_from_seed(m, n, D.SEED_A1)
        a_2 = L.dpir_derive_from_seed(l // x, n, D.SEED_A2)
        st = O.dpir_setup(db, l, m, a_1, n, a_2, prm["p"], info["delta"], x)
        assert np.array_equal(self.dbm.download(), st["db_sq"])
        assert np.array_equal(self.srv.state(), st["h1_sq"])
        assert np.array_equal(self.h2, st["h2"])

    def close(self):
        self.srv.close()
        self.dbm.close()


def batches(db, rng):
    """The batch kinds every shape runs, in sequence (index lists stay inside the entries the load read)."""
    count, packing, hi = db.count, db.info["packing"], db.hi()
    m = db.prm["m"]
    rnd = lambda: int(rng.integers(0, hi))
    per = max(packing, 1)
    out = [[(0, 1 - (db.entry(0) & 1))],                                   # index 0
           [(count - 1, rnd())],                                           # the last index
           [(i, rnd()) for i in range(per * 5, per * 6)],                  # every entry of one element
           [(i, rnd()) for i in range(per * 9, per * 12)],                 # all three fields of one store word
           [(7, 0), (7, 1), (7, hi - 1)],                                  # a repeated index: the last value wins
           [(3, db.entry(3))]]                                             # a no-op value
    if packing and count % packing:
        out.append([(count - 1 - t, rnd()) for t in range(count % packing)])   # the partial last element
    # three adjacent h_1 columns sharing one h1_squished word (layout rows 3C, 3C + 1, 3C + 2 at x = 1), and rows in both blocks
    # at x = 2: one entry at the start of each of six consecutive layout rows
    rows_per_entry_row = db.info["ne"]
    first = lambda r: (r // rows_per_entry_row) * m if not packing else r * m * packing
    cand = [first(r) for r in range(0, 6 * rows_per_entry_row, rows_per_entry_row)]
    out.append([(i, rnd()) for i in cand])
    out = [[(i, v) for i, v in b if i < count] for b in out]             # small shapes hold fewer entries than some kinds name
    return [b for b in out if b]


# ------------------------------------------------------------------ small shapes: every batch kind, against reload and oracle
# (num_entries, bits, p, l, m, nbytes): packing 9 with a partial last group; ne = x = 2 at p = 16; ne = x = 2 at p = 512;
# few entries in a mostly untouched matrix
SMALL = [(1000, 1, 512, 2, 64, 1000), (300, 8, 16, 10, 64, 300), (130, 10, 512, 10, 32, 130), (9, 1, 512, 3, 7, 9)]


@pytest.mark.parametrize("bits_format", [False, True])
@pytest.mark.parametrize("num_entries,bits,p,l,m,nbytes", SMALL)
def test_update_small_equals_reload_and_oracle(num_entries, bits, p, l, m, nbytes, bits_format):
    rng = np.random.default_rng(num_entries + bits + bits_format)
    prm = dict(n=64, l=l, m=m, logq=32, p=p)
    nb = (nbytes + 7) // 8 if bits_format else nbytes
    hi = 256 if bits_format else min(256, 1 << bits)
    db = Db(prm, num_entries, bits, rng.integers(0, hi, nb, dtype=np.uint8), bits_format)
    for upd in batches(db, rng):
        db.update(upd)
        db.assert_equals_reload()
        db.assert_equals_oracle()
    db.close()


def test_count_zero_changes_nothing():
    prm = dict(n=64, l=2, m=64, logq=32, p=512)
    db = Db(prm, 1000, 1, np.ones(1000, dtype=np.uint8), False)
    store, state, h2 = db.dbm.download(), db.srv.state(), db.h2.copy()
    db.update([])
    assert np.array_equal(db.dbm.download(), store) and np.array_equal(db.srv.state(), state) and np.array_equal(db.h2, h2)
    db.close()


# ------------------------------------------------------------------ the reference's shapes
_cache = {}


def reference_db(num_entries, bits, bits_format, seed=5):
    key = (num_entries, bits, bits_format)
    if key not in _cache:
        for k in list(_cache):
            _cache.pop(k).close()
        rng = np.random.default_rng(seed)
        prm = E.pick_params(num_entries, bits, E.SEC_PARAM, E.LOGQ)
        nbytes = num_entries // 8 if bits_format else num_entries
        _cache[key] = Db(prm, num_entries, bits, rng.integers(0, 256, nbytes, dtype=np.uint8), bits_format)
    return _cache[key]


REF = [(1 << 24, 1, True, 29), (1 << 20, 10, False, 32), (1 << 30, 1, True, 1821)]


@pytest.mark.parametrize("num_entries,bits,bits_format,l", REF)
def test_update_reference_shapes_equal_reload(num_entries, bits, bits_format, l):
    db = reference_db(num_entries, bits, bits_format)
    assert db.prm["l"] == l and db.prm["n"] == 1024
    rng = np.random.default_rng(l)
    seq = batches(db, rng)
    big = sorted(set(int(i) for i in rng.integers(0, db.count, 5000 * max(db.info["packing"], 1))))
    seq.append([(i, int(rng.integers(0, db.hi()))) for i in big])          # more than one group of 4096 changed elements
    if l != 1821:
        for upd in seq:
            db.update(upd)
            db.assert_equals_reload()
    else:                                                                 # three batches in sequence, then one reload
        for upd in seq[-3:]:
            db.update(upd)
        db.assert_equals_reload()


def _requests(db, rng, k, queries=1):
    D = _D()
    dcols, c1, e = db.dbm.cols, db.srv.state().shape[1], db.info["ne"] // db.info["x"]
    return [D.serialize_request([[rng.integers(0, 1 << 32, 3 * dcols, dtype=np.uint64).astype(np.uint32)] +
                                 [rng.integers(0, 1 << 32, 3 * c1, dtype=np.uint64).astype(np.uint32) for _ in range(e)]
                                 for _ in range(queries)]) for _ in range(k)]


def _fresh_server(db):
    D = _D()
    dbm, out, _ = db.reload()
    return dbm, D.Server(dbm, out["h1_squished"], out["a2_t"], db.prm, db.num_entries, db.bits, max_queries=65)


def test_answers_equal_fresh_server_and_decode():
    db = reference_db(1 << 24, 1, True)
    rng = np.random.default_rng(11)
    upd = [(int(i), int(rng.integers(0, 2))) for i in rng.integers(0, db.count, 300)] + [(0, 1 - db.entry(0))]
    db.update(upd)
    reqs = _requests(db, rng, 65)
    dbm, fresh = _fresh_server(db)
    assert db.srv.answer_many(reqs) == fresh.answer_many(reqs)           # a tensor-core pass of 64 and a remainder of 1
    assert db.srv.answer(reqs[0]) == fresh.answer(reqs[0])
    fresh.close()
    dbm.close()
    # the numpy client with the new hint decodes the new values and their untouched neighbours
    D = _D()
    prm, info = db.prm, dict(db.info, bits=1)
    a_1 = D.derive_from_seed(prm["m"], prm["n"], D.SEED_A1)
    a_2 = D.derive_from_seed(prm["l"], prm["n"], D.SEED_A2)
    h1 = db.srv.state()
    for i in [0, 1, upd[5][0], min(upd[5][0] + 1, db.count - 1)]:
        client, qmsg = E.query(i, a_1, a_2, prm, info, rng)
        ans = D.answer(db.dbm, [qmsg], (h1.reshape(-1), h1.shape[0], h1.shape[1]),
                       (db.a2_t.reshape(-1), prm["n"], db.a2_t.shape[1]), prm["p"], info["delta"], info["x"], info["ne"])
        assert E.recover(i, db.h2, qmsg, ans, a_2, client, prm, info) == db.entry(i), i


# ------------------------------------------------------------------ errors: a code, nothing written, the server still serves
def _raw_update(srv, idx, val, h2, null=None):
    from sdk_b200._lib import LIB
    idx = np.ascontiguousarray(idx, dtype=np.uint64)
    val = np.ascontiguousarray(val, dtype=np.uint8)
    args = [srv._h, idx.ctypes.data, val.ctypes.data, idx.size, h2.ctypes.data]
    if null is not None:
        args[null] = None
    return LIB.b200pir_dpir_server_update(*args)


def _assert_refused(db, rc_want, idx, val, srv=None, null=None, reqs=None, answers=None):
    srv = srv or db.srv
    store, state, h2 = db.dbm.download(), db.srv.state(), db.h2.copy()
    buf = db.h2.copy()
    assert _raw_update(srv, idx, val, buf, null=null) == rc_want
    assert np.array_equal(buf, h2)
    assert np.array_equal(db.dbm.download(), store) and np.array_equal(db.srv.state(), state)
    if reqs is not None:
        assert db.srv.answer_many(reqs) == answers


def test_update_errors_write_nothing():
    D = _D()
    rng = np.random.default_rng(3)
    prm = dict(n=64, l=4, m=64, logq=32, p=512)
    db = Db(prm, 1000, 1, rng.integers(0, 2, 1000, dtype=np.uint8), False)
    reqs = _requests(db, rng, 3)
    answers = db.srv.answer_many(reqs)
    kw = dict(reqs=reqs, answers=answers)
    for null in (0, 1, 2, 4):
        _assert_refused(db, E_BADARG, [1], [1], null=null, **kw)
    _assert_refused(db, E_SHAPE, [5, 1000], [1, 1], **kw)                                  # index past the entries read
    _assert_refused(db, E_BADARG, [5, 6], [1, 2], **kw)                                    # 2 does not fit one bit
    wrong = D.Server(db.dbm, db.srv.state(), db.a2_t, prm, 999, 1)                         # num_entries differs from the load
    _assert_refused(db, E_SHAPE, [1], [1], srv=wrong, **kw)
    wrong.close()
    wrong = D.Server(db.dbm, db.srv.state(), db.a2_t, prm, 1000, 2)                        # bits_per_entry differs
    _assert_refused(db, E_SHAPE, [1], [1], srv=wrong, **kw)
    wrong.close()
    dbp = D.PackedMatrix(db.dbm.download(), db.dbm.rows, db.dbm.cols)                      # a .dbp: not from a load
    other = D.Server(dbp, db.srv.state(), db.a2_t, prm, 1000, 1)
    _assert_refused(db, E_UNSUPPORTED, [1], [1], srv=other, **kw)
    other.close()
    dbp.close()
    big = dict(prm, l=8)                                                                   # a chunk: 4 of 8 rows
    _, outb, _ = D.load(big, 1000, 1, db.data)
    chunk = D.Server(db.dbm, outb["h1_squished"], outb["a2_t"], big, 1000, 1)
    _assert_refused(db, E_UNSUPPORTED, [1], [1], srv=chunk, **kw)
    chunk.close()
    db.update([(5, 1 - db.entry(5))])                                                      # and it still updates
    db.assert_equals_reload()
    db.close()
    # bits: a value above 1; packed bytes: a value wider than bits_per_entry; bytes wider than their 3-bit field at load
    db = Db(dict(prm, l=2), 1000, 1, rng.integers(0, 256, 125, dtype=np.uint8), True)
    _assert_refused(db, E_BADARG, [3], [2])
    _assert_refused(db, E_SHAPE, [1000], [1])
    db.close()
    db = Db(dict(n=64, l=6, m=64, logq=32, p=512), 999, 3, rng.integers(0, 256, 999, dtype=np.uint8), False)
    _assert_refused(db, E_UNSUPPORTED, [3], [2])
    db.close()
    db = Db(dict(n=64, l=6, m=64, logq=32, p=512), 999, 3, rng.integers(0, 8, 999, dtype=np.uint8), False)
    _assert_refused(db, E_BADARG, [3], [8])
    db.update([(3, 7)])
    db.assert_equals_reload()
    db.close()


# ------------------------------------------------------------------ isolation
def test_updates_beside_answer_many_threads():
    db = reference_db(1 << 24, 1, True)
    rng = np.random.default_rng(21)
    reqs = _requests(db, rng, 4)
    seq = [[(int(i), int(rng.integers(0, 2))) for i in rng.integers(0, db.count, 200)] for _ in range(3)]
    states = [db.data.copy()]
    got, err = [], []
    stop = threading.Event()

    def answers():
        try:
            while not stop.is_set():
                got.append(db.srv.answer_many(reqs))
        except Exception as e:          # noqa: BLE001 - reported below
            err.append(e)

    t = threading.Thread(target=answers)
    t.start()
    try:
        for upd in seq:
            db.update(upd)
            states.append(db.data.copy())
    finally:
        stop.set()
        t.join()
    assert not err and got
    final = db.assert_equals_reload()
    assert np.array_equal(db.h2, final["h2"])
    want = []
    for data in states:
        D = _D()
        dbm, out, _ = D.load(db.prm, db.num_entries, db.bits, data, db.fmt)
        srv = D.Server(dbm, out["h1_squished"], out["a2_t"], db.prm, db.num_entries, db.bits, max_queries=65)
        want.append(srv.answer_many(reqs))
        srv.close()
        dbm.close()
    for resp in got:
        assert resp in want


def test_update_beside_busy_legacy_stream():
    import torch
    db = reference_db(1 << 24, 1, True)
    rng = np.random.default_rng(31)
    torch.cuda.synchronize()
    torch.cuda._sleep(200_000_000)                        # about 0.1 s at H100 clocks, on the legacy default stream
    db.update([(int(i), int(rng.integers(0, 2))) for i in rng.integers(0, db.count, 100)])
    torch.cuda.synchronize()
    db.assert_equals_reload()


def test_launches_do_not_scale_with_the_database():
    counts = []
    for num_entries in (1 << 24, 1 << 30):
        db = reference_db(num_entries, 1, True)
        upd = [(i * 1009 + 3, 1 - db.entry(i * 1009 + 3)) for i in range(50)]
        before = _launches()
        db.update(upd)
        counts.append(_launches() - before)
    assert counts[0] == counts[1] and counts[0] > 0
