"""DoublePIR over row shards (b200pir_dpir_load*_sharded, b200pir_dpir_server_create_sharded): loads, answers, updates and
server state byte for byte the one-device code's for the same input, with every shard on device 0 (a repeated device is a
valid configuration) and, where two GPUs are visible, on devices 0 and 1; responses decode with the numpy client."""
import ctypes as C
import os
import shutil
import tempfile
import threading

import numpy as np
import pytest

import test_gpu_dpir_load as LT
import test_gpu_dpir_load_bands as LB
import test_gpu_dpir_serve as S
import test_gpu_dpir_update as UT
import test_oracle_doublepir_e2e as E

pytestmark = pytest.mark.gpu

E_BADARG, E_SHAPE, E_UNSUPPORTED = -1, -2, -4
GIB = 1 << 30


def _D():
    import sdk_b200.doublepir as D
    return D


def _ngpus():
    import torch
    return torch.cuda.device_count()


def _devices(kind, G):
    if kind == "two":
        if _ngpus() < 2:
            pytest.skip("needs two GPUs")
        return [g % 2 for g in range(G)]
    return [0] * G


def _close(mats):
    for m in mats:
        m.close()


def assert_same_load(one, sharded, G):
    dbm, out, info = one
    mats, sout, sinfo = sharded
    assert sinfo == info and len(mats) == G
    for k in ("h1_squished", "a2_t", "h2"):
        assert np.array_equal(sout[k], out[k]), k
    assert np.array_equal(np.concatenate([m.download() for m in mats]), dbm.download())
    end = 0
    for m in mats:
        si = m.shard_info()
        assert si["row_begin"] == m.row_begin == end and si["rows"] == m.rows and si["cols"] == dbm.cols
        end += m.rows
    assert end == dbm.rows


# ------------------------------------------------------------------ loads
# (num_entries, bits, p, l, m, nbytes, high): the layouts of test_gpu_dpir_load.SMALL with l grown to at least five units of
# 3x rows: packing 9 with a partial last group and rows of 63 entries (shard edges mid-byte in the bit format); ne = x = 2 at
# p = 16; oversized bytes in 3-bit fields; ne = x = 2 at p = 512; few entries in a mostly untouched matrix
SMALL = [(1000, 1, 512, 30, 7, 1000, 2), (300, 8, 16, 36, 64, 300, 256), (999, 3, 512, 15, 64, 999, 256),
         (130, 10, 512, 30, 32, 130, 256), (9, 1, 512, 15, 7, 9, 2)]


@pytest.mark.parametrize("scratch", [0, 1])
@pytest.mark.parametrize("G", [2, 3, 5])
@pytest.mark.parametrize("bits_format", [False, True])
@pytest.mark.parametrize("num_entries,bits,p,l,m,nbytes,high", SMALL)
def test_load_sharded_equals_load(num_entries, bits, p, l, m, nbytes, high, bits_format, G, scratch):
    D = _D()
    rng = np.random.default_rng(num_entries + 17 * bits + G)
    nbytes = (nbytes + 7) // 8 if bits_format else nbytes
    data = rng.integers(0, 256 if bits_format else high, nbytes, dtype=np.uint8)
    prm = dict(n=64, l=l, m=m, logq=32, p=p)
    fmt = D.ENTRY_BITS if bits_format else D.ENTRY_BYTES
    one = D.load(prm, num_entries, bits, data, fmt)
    sh = D.load_sharded(prm, num_entries, bits, data, [0] * G, fmt, scratch_bytes=scratch)   # 1 byte: one group a band
    try:
        assert_same_load(one, sh, G)
        assert [(mm.row_begin, mm.rows) for mm in sh[0]] == D.shard_rows(prm, num_entries, bits, G)
    finally:
        _close(sh[0])
        one[0].close()


@pytest.mark.parametrize("kind", ["same", "two"])
@pytest.mark.parametrize("num_entries,bits,bits_format", [(1 << 24, 1, True), (1 << 20, 10, False)])
def test_load_file_sharded_equals_load_sharded_and_load(num_entries, bits, bits_format, kind, tmp_path):
    D = _D()
    rng, prm, data, one = LT.reference_shape(num_entries, bits, bits_format, 1)
    fmt = D.ENTRY_BITS if bits_format else D.ENTRY_BYTES
    path = str(tmp_path / "db.bin")
    data.tofile(path)
    for G in (2, 3, 5):
        devs = _devices(kind, G)
        a = D.load_sharded(prm, num_entries, bits, data, devs, fmt, scratch_bytes=64 << 20)
        b = D.load_file_sharded(prm, num_entries, bits, path, devs, fmt)
        try:
            assert_same_load(one, a, G)
            assert_same_load(one, b, G)
            assert [mm.shard_info()["device"] for mm in a[0]] == devs
        finally:
            _close(a[0])
            _close(b[0])


def _sharded_rc(prm, num_entries, bits, data, fmt, devices, null=None):
    from sdk_b200._lib import LIB
    D = _D()
    data = np.ascontiguousarray(data, dtype=np.uint8)
    k = len(devices)
    devs = (C.c_int * max(k, 1))(*devices)
    hs = (C.c_void_p * max(k, 1))()
    bufs = [np.zeros(1 << 16, dtype=np.uint32) for _ in range(3)]
    args = [devs, k, C.byref(D._params(prm)), num_entries, bits, data.ctypes.data, data.size, fmt, 0, hs] + [b.ctypes.data for b in bufs]
    if null is not None:
        args[null] = None
    rc = LIB.b200pir_dpir_load_sharded(*args)
    assert not any(hs[:k])
    return rc


def test_load_sharded_errors_return_no_handle():
    D = _D()
    prm = dict(n=64, l=30, m=7, logq=32, p=512)                # 10 units of 3 rows, 63 entries a row, 1890 in all
    data = np.ones(1890, dtype=np.uint8)
    for g, (r0, rows) in enumerate(D.shard_rows(prm, 1890, 1, 3)):
        for r in (r0, r0 + rows - 1):                          # one packed word of shard g past the setup GEMM's range
            bad = data.copy()
            bad[r * 63 + 9: r * 63 + 18] = 255
            assert _sharded_rc(prm, 1890, 1, bad, D.ENTRY_BYTES, [0] * 3) == E_UNSUPPORTED, (g, r)
    assert _sharded_rc(prm, 1890, 1, data, D.ENTRY_BYTES, []) == E_SHAPE          # no shards
    assert _sharded_rc(prm, 1890, 1, data, D.ENTRY_BYTES, [0] * 11) == E_SHAPE    # more shards than units
    assert _sharded_rc(prm, 1890, 1, data, D.ENTRY_BYTES, [0, -1]) == E_BADARG
    assert _sharded_rc(prm, 1890, 1, data, 2, [0, 0]) == E_BADARG                 # unknown entry format
    for null in (0, 2, 5, 9, 10, 11, 12):
        assert _sharded_rc(prm, 1890, 1, data, D.ENTRY_BYTES, [0, 0], null=null) == E_BADARG, null
    mats, out, _ = D.load_sharded(prm, 1890, 1, data, [0, 0])          # and a valid call still works
    _close(mats)


# ------------------------------------------------------------------ answers
_servers = {}


def served(num_entries, bits, bits_format, G, kind="same", max_queries=72):
    """(prm, data, info, a_1, a_2, out, one-device server, sharded server) over the reference shape, cached per configuration"""
    key = (num_entries, bits, bits_format, G, kind)
    if key not in _servers:
        for k in [k for k in _servers if k != "one"]:           # one sharded server at a time; the one-device ones stay
            v = _servers.pop(k)
            v[-1].close()
            _close(v[-2])
        D = _D()
        rng, prm, data, one = LT.reference_shape(num_entries, bits, bits_format, 1)
        dbm, out, info, a_1, a_2 = LT._client_view(prm, one)
        info = dict(info, bits=bits)
        srv1 = _servers.get("one", {}).get((num_entries, bits))
        if srv1 is None:
            srv1 = D.Server(dbm, out["h1_squished"], out["a2_t"], prm, num_entries, bits, max_queries=max_queries)
            _servers.setdefault("one", {})[(num_entries, bits)] = srv1
        mats, sout, _ = D.load_sharded(prm, num_entries, bits, data, _devices(kind, G),
                                       D.ENTRY_BITS if bits_format else D.ENTRY_BYTES)
        srv = D.Server(mats, sout["h1_squished"], sout["a2_t"], prm, num_entries, bits, max_queries=max_queries)
        _servers[key] = (prm, data, info, a_1, a_2, out, srv1, mats, srv)
    return _servers[key]


@pytest.fixture(scope="module", autouse=True)
def _cleanup():
    yield
    for k, v in list(_servers.items()):
        if k == "one":
            for s in v.values():
                s.close()
        else:
            v[-1].close()
            _close(v[-2])
    _servers.clear()


def _want(data, i, bits_format):
    return LT._bit(data, i) if bits_format else int(data[i])


@pytest.mark.parametrize("kind", ["same", "two"])
@pytest.mark.parametrize("G", [2, 3, 5])
@pytest.mark.parametrize("num_entries,bits,bits_format", [(1 << 24, 1, True), (1 << 20, 10, False)])
def test_single_requests_equal_one_device_and_decode(num_entries, bits, bits_format, G, kind):
    D = _D()
    prm, data, info, a_1, a_2, out, srv1, mats, srv = served(num_entries, bits, bits_format, G, kind)
    rng = np.random.default_rng(G + 7)
    per_row = prm["m"] * max(info["packing"], 1) // info["ne"] if not info["packing"] else prm["m"] * info["packing"]
    edges = [m.row_begin * per_row for m in mats[1:]]        # first entries of every shard after the first
    for i in [0, num_entries - 1] + [e for e in edges if e < num_entries] + [int(v) for v in rng.integers(0, num_entries, 2)]:
        client, qmsg = E.query(i, a_1, a_2, prm, info, rng)
        req = D.serialize_request([qmsg])
        resp = srv.answer(req)
        assert len(resp) == srv.answer_size(req)
        assert resp == srv1.answer(req), i
        assert E.recover(i, out["h2"], qmsg, S.flat(resp), a_2, client, prm, info) == _want(data, i, bits_format), i


@pytest.mark.parametrize("kind", ["same", "two"])
@pytest.mark.parametrize("nq", [2, 3, 8, 30])
def test_batched_requests_equal_one_device_and_decode(nq, kind):
    # l = 29 over three shards: rows [0, 12), [12, 21), [21, 29); batch edges at 14 (nq 2) and 9, 18 (nq 3) fall inside shards,
    # those of nq 8 (every 3 rows) on both shard edges; at nq 30 every batch but the last is empty
    D = _D()
    num_entries = 1 << 24
    prm, data, info, a_1, a_2, out, srv1, mats, srv = served(num_entries, 1, True, 3, kind)
    assert [(m.row_begin, m.rows) for m in mats] == [(0, 12), (12, 9), (21, 8)]
    rows = S.T.batch_rows(prm["l"], nq)
    per_row = prm["m"] * info["packing"]
    rng = np.random.default_rng(300 + nq)
    idxs = [int(rng.integers(r0 * per_row, min(r1 * per_row, num_entries))) if r1 > r0 else int(rng.integers(0, num_entries))
            for r0, r1 in rows]
    qs = [E.query(i, a_1, a_2, prm, info, rng) for i in idxs]
    req = D.serialize_request([q for _, q in qs])
    resp = srv.answer(req)
    assert resp == srv1.answer(req)
    ans = S.flat(resp)
    for b, ((r0, r1), i, (client, qmsg)) in enumerate(zip(rows, idxs, qs)):
        if r1 > r0:
            assert E.recover(i, out["h2"], qmsg, ans, a_2, client, prm, info, batch_index=b) == LT._bit(data, i), (b, i)


@pytest.mark.parametrize("kind", ["same", "two"])
@pytest.mark.parametrize("count", [1, 8, 9, 64, 72])
def test_answer_many_equals_one_device(count, kind):
    # 72 = max_queries; 8 and fewer requests run the integer passes, more the tensor-core passes
    D = _D()
    num_entries = 1 << 24
    prm, data, info, a_1, a_2, out, srv1, mats, srv = served(num_entries, 1, True, 5, kind)
    rng = np.random.default_rng(500 + count)
    idxs = [int(i) for i in rng.integers(0, num_entries, count)]
    qs = [E.query(i, a_1, a_2, prm, info, rng) for i in idxs]
    wires = [D.serialize_request([q]) for _, q in qs]
    many = srv.answer_many(wires)
    assert many == srv1.answer_many(wires)
    for k in range(0, count, max(1, count // 6)):
        i, (client, qmsg) = idxs[k], qs[k]
        assert many[k] == srv.answer(wires[k]), k
        assert E.recover(i, out["h2"], qmsg, S.flat(many[k]), a_2, client, prm, info) == LT._bit(data, i), k
    mixed = S.make_requests([q for _, q in qs[:20]] or [qs[0][1]], [1, 2, 3, 8][:min(4, count)], 1)
    mw = [D.serialize_request(q) for q in mixed]
    assert srv.answer_many(mw) == srv1.answer_many(mw)


def test_concurrent_callers_get_their_own_bytes():
    D = _D()
    num_entries = 1 << 24
    prm, data, info, a_1, a_2, out, srv1, mats, srv = served(num_entries, 1, True, 5)
    rng = np.random.default_rng(800)
    reqs = [D.serialize_request([E.query(int(i), a_1, a_2, prm, info, rng)[1] for i in rng.integers(0, num_entries, 1 + k % 3)])
            for k in range(12)]
    want = [srv1.answer(r) for r in reqs]
    errors = []

    def worker(t):
        try:
            for rep in range(3):
                k = (t + rep) % len(reqs)
                if (t + rep) % 2:
                    assert srv.answer(reqs[k]) == want[k]
                else:
                    ks = [k, (k + 5) % len(reqs)]
                    assert srv.answer_many([reqs[j] for j in ks]) == [want[j] for j in ks]
        except Exception as e:          # noqa: BLE001 - reported below
            errors.append(e)

    th = [threading.Thread(target=worker, args=(t,)) for t in range(6)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert not errors, errors


# ------------------------------------------------------------------ servers from create_shard, and every refusal
def test_create_shard_servers_and_errors():
    from sdk_b200._lib import LIB
    D = _D()
    num_entries = 1 << 24
    prm, data, info, a_1, a_2, out, srv1, mats, srv = served(num_entries, 1, True, 3)
    store = np.concatenate([m.download() for m in mats])
    cut = [(m.row_begin, m.rows) for m in mats]                # (0, 12), (12, 9), (21, 8)
    rng = np.random.default_rng(900)
    good_q = [E.query(int(i), a_1, a_2, prm, info, rng)[1] for i in rng.integers(0, num_entries, 3)]
    good = D.serialize_request(good_q)
    want = srv1.answer(good)

    def shards(spans):
        return [D.PackedMatrix.shard(store[r0:r0 + rows], r0) for r0, rows in spans]

    made = shards(cut)
    s2 = D.Server(made, out["h1_squished"], out["a2_t"], prm, num_entries, 1, max_queries=8)
    try:
        assert s2.answer(good) == want
        assert s2.answer_many([good, good]) == [want, want]
        assert np.array_equal(s2.state(), out["h1_squished"])
        # chunked answers are refused, write nothing, and the server answers afterwards
        size = s2.answer_size(good)
        buf = C.create_string_buffer(b"\xa5" * size, size)
        n = C.c_size_t(size)
        assert LIB.b200pir_dpir_answer(s2._h, good, len(good), 0, buf, C.byref(n)) == E_UNSUPPORTED
        assert buf.raw == b"\xa5" * size and n.value == size
        assert s2.answer(good) == want
        # a loaded store made by create_shard is not from a load: updates are refused
        with pytest.raises(D.B200PirError) as e:
            s2.update([0], [1], out["h2"])
        assert e.value.code == E_UNSUPPORTED
        assert s2.answer(good) == want
    finally:
        s2.close()
        _close(made)
    h1, a2 = out["h1_squished"], out["a2_t"]
    bad = {"gapped": [(0, 12), (21, 8)], "overlapping": [(0, 12), (9, 12), (21, 8)], "out of order": [cut[1], cut[0], cut[2]],
           "misaligned": [(0, 13), (13, 8), (21, 8)], "short of l": cut[:2], "past l": [(0, 12), (12, 9), (21, 8), (29, 1)]}
    for name, spans in bad.items():
        spans = [(r0, min(rows, len(store) - r0)) for r0, rows in spans]
        ms = [D.PackedMatrix.shard(store[r0:r0 + rows] if rows else store[:1], r0) for r0, rows in spans]
        try:
            hs = (C.c_void_p * len(ms))(*[m._h for m in ms])
            h = C.c_void_p()
            rc = LIB.b200pir_dpir_server_create_sharded(C.byref(D._params(prm)), num_entries, 1, hs, len(ms), h1.ctypes.data,
                                                        a2.ctypes.data, 8, C.byref(h))
            assert rc == E_SHAPE and not h.value, name
        finally:
            _close(ms)
    hs = (C.c_void_p * 3)(*[m._h for m in mats])
    h = C.c_void_p()
    p = C.byref(D._params(prm))
    assert LIB.b200pir_dpir_server_create_sharded(p, num_entries, 1, hs, 0, h1.ctypes.data, a2.ctypes.data, 8, C.byref(h)) == E_SHAPE
    assert LIB.b200pir_dpir_server_create_sharded(p, num_entries, 1, hs, 3, h1.ctypes.data, a2.ctypes.data, 0, C.byref(h)) == E_BADARG
    assert LIB.b200pir_dpir_server_create_sharded(p, num_entries, 1, None, 3, h1.ctypes.data, a2.ctypes.data, 8, C.byref(h)) == E_BADARG
    assert not h.value
    assert srv.answer(good) == want


# ------------------------------------------------------------------ updates
class Pair:
    """One load served unsharded (test_gpu_dpir_update.Db) and the same bytes loaded and served in G row shards"""

    def __init__(self, prm, num_entries, bits, data, bits_format, G, devices):
        D = _D()
        self.one = UT.Db(prm, num_entries, bits, data, bits_format)
        self.mats, out, _ = D.load_sharded(prm, num_entries, bits, self.one.data, devices, self.one.fmt)
        self.h2 = out["h2"]
        self.srv = D.Server(self.mats, out["h1_squished"], out["a2_t"], prm, num_entries, bits, max_queries=65)

    def update(self, upd):
        self.h2 = self.srv.update(np.array([i for i, _ in upd], dtype=np.uint64), np.array([v for _, v in upd], dtype=np.uint8), self.h2)
        self.one.update(upd)

    def assert_same(self, reqs):
        assert np.array_equal(np.concatenate([m.download() for m in self.mats]), self.one.dbm.download())
        assert np.array_equal(self.srv.state(), self.one.srv.state())
        assert np.array_equal(self.h2, self.one.h2)
        assert self.srv.answer_many(reqs) == self.one.srv.answer_many(reqs)

    def edge_entries(self):
        """the first and last entry of every shard's rows"""
        info, m = self.one.info, self.one.prm["m"]
        first = lambda r: (r // info["ne"]) * m if not info["packing"] else r * m * info["packing"]
        out = []
        for mm in self.mats:
            out += [first(mm.row_begin), first(mm.row_begin + mm.rows) - 1]
        return [i for i in out if 0 <= i < self.one.count]

    def close(self):
        self.srv.close()
        _close(self.mats)
        self.one.close()


def _run_updates(pair, rng, reqs):
    hi = pair.one.hi()
    seq = UT.batches(pair.one, rng)
    edges = pair.edge_entries()
    seq.append([(i, int(rng.integers(0, hi))) for i in edges])                        # every shard, at its edges
    seq.append([(int(i), int(rng.integers(0, hi))) for i in rng.integers(0, pair.one.count, 50)])
    for upd in seq:
        pair.update(upd)
        pair.assert_same(reqs)
    pair.one.assert_equals_reload()


@pytest.mark.parametrize("kind", ["same", "two"])
@pytest.mark.parametrize("bits_format", [False, True])
@pytest.mark.parametrize("num_entries,bits,p,l,m,nbytes", [(1000, 1, 512, 30, 7, 1000), (300, 8, 16, 36, 64, 300),
                                                           (130, 10, 512, 30, 32, 130)])
def test_updates_equal_one_device(num_entries, bits, p, l, m, nbytes, bits_format, kind):
    rng = np.random.default_rng(num_entries + bits + bits_format)
    prm = dict(n=64, l=l, m=m, logq=32, p=p)
    nb = (nbytes + 7) // 8 if bits_format else nbytes
    hi = 256 if bits_format else min(256, 1 << bits)
    pair = Pair(prm, num_entries, bits, rng.integers(0, hi, nb, dtype=np.uint8), bits_format, 3, _devices(kind, 3))
    try:
        reqs = UT._requests(pair.one, rng, 3, queries=2)
        _run_updates(pair, rng, reqs)
    finally:
        pair.close()


@pytest.mark.parametrize("kind", ["same", "two"])
def test_updates_equal_one_device_at_a_reference_shape(kind):
    num_entries = 1 << 24
    rng = np.random.default_rng(24)
    prm = E.pick_params(num_entries, 1, E.SEC_PARAM, E.LOGQ)
    pair = Pair(prm, num_entries, 1, rng.integers(0, 256, num_entries // 8, dtype=np.uint8), True, 5, _devices(kind, 5))
    try:
        reqs = UT._requests(pair.one, rng, 4)
        _run_updates(pair, rng, reqs)
    finally:
        pair.close()


# ------------------------------------------------------------------ scale: 2^36 one-bit entries (l m > 2^32) as two shards
def test_two_shards_past_the_old_limit(monkeypatch):
    # Both loads on device 0.  The stores are compared through the answers (every q_1 reads every row of its batch) rather
    # than downloaded: two 11 GB downloads would need more host memory than the check is worth
    import torch
    D = _D()
    for k in list(_servers):                                   # free the cached servers' device memory first
        v = _servers.pop(k)
        if k == "one":
            for s in v.values():
                s.close()
        else:
            v[-1].close()
            _close(v[-2])
    LT._loaded.clear()
    num_entries = 1 << 36
    prm = E.pick_params(num_entries, 1, E.SEC_PARAM, E.LOGQ)
    l, m, n = prm["l"], prm["m"], prm["n"]
    assert l * m > 1 << 32
    cols = (m + 2) // 3
    store = l * cols * 4
    nbytes = num_entries // 8
    torch.cuda.empty_cache()
    free_dev = torch.cuda.mem_get_info()[0]
    need_dev = 2 * store + 2 * 4 * n * (3 * m + 4 * l) + 6 * GIB
    if free_dev < need_dev:
        pytest.skip("device memory: %.1f GiB free, %.1f GiB needed" % (free_dev / GIB, need_dev / GIB))
    tmp = tempfile.mkdtemp(prefix="dpir_shards_")
    try:
        free_disk = shutil.disk_usage(tmp).free
        if free_disk < nbytes + GIB:
            pytest.skip("disk: %.1f GiB free in %s, %.1f GiB needed" % (free_disk / GIB, tmp, (nbytes + GIB) / GIB))
        need_host = 6 * m * n * 8 + 2 * GIB
        if LB._mem_available() < need_host:
            pytest.skip("host memory: %.1f GiB available, %.1f GiB needed" % (LB._mem_available() / GIB, need_host / GIB))
        path = os.path.join(tmp, "db.bin")
        LB._write_seeded(path, nbytes, 36)
        dbm, out, info = D.load_file(prm, num_entries, 1, path, D.ENTRY_BITS)
        mats, sout, _ = D.load_file_sharded(prm, num_entries, 1, path, [0, 0], D.ENTRY_BITS)
        fd = os.open(path, os.O_RDONLY)
        bit = lambda i: (os.pread(fd, 1, i >> 3)[0] >> (i & 7)) & 1
        os.remove(path)
        srv = srv1 = None
        try:
            for k in ("h1_squished", "a2_t", "h2"):
                assert np.array_equal(sout[k], out[k]), k
            assert sum(mm.rows for mm in mats) == l
            info = dict(info, bits=1)
            a_1 = D.derive_from_seed(m, n, D.SEED_A1)
            a_2 = D.derive_from_seed(l // info["x"], n, D.SEED_A2)
            a_2_sums = (a_2.astype(np.uint64).sum(axis=0) & np.uint64(0xFFFFFFFF)).reshape(1, n)
            monkeypatch.setattr(E, "mat_vec", LB._mat_vec_exact)
            per_row = m * info["packing"]
            rng = np.random.default_rng(37)
            edge = mats[1].row_begin * per_row
            idxs = [0, num_entries - 1, edge - 1, edge] + [int(v) for v in rng.integers(0, num_entries, 12)]
            srv1 = D.Server(dbm, out["h1_squished"], out["a2_t"], prm, num_entries, 1, max_queries=len(idxs))
            srv = D.Server(mats, sout["h1_squished"], sout["a2_t"], prm, num_entries, 1, max_queries=len(idxs))
            qs = [E.query(i, a_1, a_2, prm, info, rng) for i in idxs]
            wires = [D.serialize_request([q]) for _, q in qs]
            many = srv.answer_many(wires)
            assert many == srv1.answer_many(wires)
            for k, (i, (client, qmsg)) in enumerate(zip(idxs, qs)):
                assert E.recover(i, sout["h2"], qmsg, S.flat(many[k]), a_2_sums, client, prm, info) == bit(i), (k, i)
            assert srv.answer(wires[0]) == many[0]
        finally:
            os.close(fd)
            for s in (srv, srv1):
                if s is not None:
                    s.close()
            _close(mats)
            dbm.close()
            LB._halves.clear()
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
        torch.cuda.empty_cache()


def test_sharded_load_counts_its_launches():
    # the shards load on worker threads; their kernel launches still count on the calling thread
    from sdk_b200._lib import LIB
    D = _D()
    prm = dict(n=64, l=30, m=7, logq=32, p=512)
    data = np.ones(1890, dtype=np.uint8)
    counts = []
    for G in (None, 1, 3):
        k0 = LIB.b200pir_kernel_launches()
        mats = [D.load(prm, 1890, 1, data)[0]] if G is None else D.load_sharded(prm, 1890, 1, data, [0] * G)[0]
        counts.append(LIB.b200pir_kernel_launches() - k0)
        _close(mats)
    assert counts[0] > 0 and counts[1] == counts[0] and counts[2] > counts[0], counts
