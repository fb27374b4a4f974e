"""DoublePIR's answer() served from HBM (sdk_b200.doublepir.Server, b200pir_dpir_server_*): wire-format requests in, response
bytes out, bit for bit against the oracle's answer() (serialised as serializer.rs does) and against the existing host-buffer
chain, decoded by the numpy client; answer_many against each request answered alone; chunked servers as e2e.rs combines them;
the multi-vector kernel against numpy; and every error code, after which the server keeps answering."""
import ctypes as C

import numpy as np
import pytest

import test_gpu_dpir_end_to_end as T
import test_oracle_doublepir_e2e as E

pytestmark = pytest.mark.gpu

U32 = np.uint32
E_BADARG, E_SHAPE = -1, -2
SHAPES = list(T.SHAPES)


def _D():
    import sdk_b200.doublepir as D
    return D


def wire(msg, prm, info, delta):
    """msg.serialize() of an answer() given as the oracle returns it (flat arrays): msg[0] is (delta x) x n, the rest columns"""
    D = _D()
    return D.serialize_state([np.asarray(msg[0]).reshape(delta * info["x"], prm["n"])] + [np.asarray(v).reshape(-1) for v in msg[1:]])


def flat(resp):
    return [m.reshape(-1) for m in _D().deserialize_state(resp)]


def setup_server(got, prm, info, num_entries, bits, max_queries=32, rows=None):
    """(PackedMatrix, Server) over the setup() output `got` (rows [r0, r1) only when rows is given)"""
    D = _D()
    sq = np.ascontiguousarray(got["db_squished"] if rows is None else got["db_squished"][rows[0]:rows[1]])
    dbm = D.PackedMatrix(sq.reshape(-1), sq.shape[0], sq.shape[1])
    try:
        srv = D.Server(dbm, got["h1_squished"], got["a2_t"], prm, num_entries, bits, max_queries=max_queries)
    except Exception:
        dbm.close()
        raise
    return dbm, srv


# ------------------------------------------------------------------ one request at the reference's shapes
@pytest.mark.parametrize("num_entries,bits,seed", SHAPES)
def test_serve_answer_equals_oracle_and_chain_and_decodes(num_entries, bits, seed):
    D = _D()
    prm, data, info, delta, a_1, a_2, st, got = T.gpu_prepared(num_entries, bits, seed)
    rng = np.random.default_rng(seed + 200)
    dbm, srv = setup_server(got, prm, info, num_entries, bits)
    try:
        for i in T.probe_indices(num_entries, prm, info, rng):
            client, qmsg = E.query(i, a_1, a_2, prm, info, rng)
            req = D.serialize_request([qmsg])
            resp = srv.answer(req)
            assert len(resp) == srv.answer_size(req)
            assert resp == wire(E.run_answer(st, prm, info, delta, [qmsg]), prm, info, delta), i
            assert resp == wire(T.gpu_answer(dbm, got, prm, info, delta, [qmsg]), prm, info, delta), i
            assert E.recover(i, got["h2"], qmsg, flat(resp), a_2, client, prm, info) == int(data[i]), i
    finally:
        srv.close()
        dbm.close()


@pytest.mark.parametrize("num_entries,bits,bits_format", [(1 << 24, 1, True), (1 << 20, 10, False)])
def test_serve_from_load_output_decodes(num_entries, bits, bits_format):
    # the server over b200pir_dpir_load's resident database and host matrices, shared matrices derived from the reference's seeds
    import test_gpu_dpir_load as LT
    D = _D()
    rng, prm, data, loaded = LT.reference_shape(num_entries, bits, bits_format, 1)
    dbm, out, info, a_1, a_2 = LT._client_view(prm, loaded)
    info = dict(info, bits=bits)
    delta = info["delta"]
    st = dict(db_sq=dbm.download(), h1_sq=out["h1_squished"], a2_t=out["a2_t"])
    srv = D.Server(dbm, out["h1_squished"], out["a2_t"], prm, num_entries, bits)
    try:
        for i in [0, num_entries - 1] + [int(v) for v in rng.integers(0, num_entries, 2)]:
            client, qmsg = E.query(i, a_1, a_2, prm, info, rng)
            resp = srv.answer(D.serialize_request([qmsg]))
            assert resp == wire(E.run_answer(st, prm, info, delta, [qmsg]), prm, info, delta), i
            assert resp == wire(LT._answer(dbm, out, prm, info, [qmsg]), prm, info, delta), i
            want = LT._bit(data, i) if bits_format else int(data[i])
            assert E.recover(i, out["h2"], qmsg, flat(resp), a_2, client, prm, info) == want, i
    finally:
        srv.close()


# ------------------------------------------------------------------ batched requests on l = 29
@pytest.mark.parametrize("nq", [2, 3, 8, 30])
def test_serve_batched_request(nq):
    D = _D()
    num_entries = 1 << 24
    prm, data, info, delta, a_1, a_2, st, got = T.gpu_prepared(num_entries, 1, 1)
    rows = T.batch_rows(prm["l"], nq)                            # 30 > l: every batch but the last is empty
    per_row = prm["m"] * info["packing"]
    rng = np.random.default_rng(300 + nq)
    idxs = [int(rng.integers(r0 * per_row, min(r1 * per_row, num_entries))) if r1 > r0 else int(rng.integers(0, num_entries))
            for r0, r1 in rows]
    qs = [E.query(i, a_1, a_2, prm, info, rng) for i in idxs]
    queries = [q for _, q in qs]
    dbm, srv = setup_server(got, prm, info, num_entries, 1)
    try:
        resp = srv.answer(D.serialize_request(queries))
    finally:
        srv.close()
        dbm.close()
    assert resp == wire(E.run_answer(st, prm, info, delta, queries), prm, info, delta)
    ans = flat(resp)
    assert len(ans) == 1 + 2 * nq
    for b, ((r0, r1), i, (client, qmsg)) in enumerate(zip(rows, idxs, qs)):
        if r1 > r0:
            assert E.recover(i, got["h2"], qmsg, ans, a_2, client, prm, info, batch_index=b) == int(data[i]), (b, i)


# ------------------------------------------------------------------ answer_many
@pytest.fixture(scope="module")
def l29():
    D = _D()
    num_entries = 1 << 24
    prm, data, info, delta, a_1, a_2, st, got = T.gpu_prepared(num_entries, 1, 1)
    rng = np.random.default_rng(500)
    pool = [E.query(int(i), a_1, a_2, prm, info, rng)[1] for i in rng.integers(0, num_entries, 20)]
    dbm, srv = setup_server(got, prm, info, num_entries, 1, max_queries=64)
    yield D, prm, info, delta, st, got, pool, dbm, srv
    srv.close()
    dbm.close()


def make_requests(pool, sizes, offset):
    """requests of the given query counts, each of its own mix of the pool's queries"""
    reqs, k = [], offset
    for s in sizes:
        reqs.append([pool[(k + j * 7) % len(pool)] for j in range(s)])
        k += 3
    return reqs


@pytest.mark.parametrize("count", [1, 2, 5, 16, 17, "max"])
def test_serve_answer_many_equals_each_alone_and_oracle(l29, count):
    D, prm, info, delta, st, got, pool, dbm, srv = l29
    if count == "max":
        sizes = [8] * 7 + [3, 2, 1, 1, 1]                         # 64 queries: exactly max_queries
    else:
        sizes = [[1, 2, 3, 8][k % 4] for k in range(count)]      # 17 requests: 57 queries, two passes of the database
    assert sum(sizes) <= 64
    reqs = make_requests(pool, sizes, count if isinstance(count, int) else 11)
    wires = [D.serialize_request(q) for q in reqs]
    many = srv.answer_many(wires)
    assert len(many) == len(reqs)
    for k, (q, w, r) in enumerate(zip(reqs, wires, many)):
        assert r == srv.answer(w), k
        assert r == wire(E.run_answer(st, prm, info, delta, q), prm, info, delta), k


def test_serve_answer_many_over_the_query_limit(l29):
    D, prm, info, delta, st, got, pool, dbm, srv = l29
    wires = [D.serialize_request(q) for q in make_requests(pool, [8] * 8 + [1], 0)]      # 65 queries
    with pytest.raises(D.B200PirError) as e:
        srv.answer_many(wires)
    assert e.value.code == E_SHAPE and "64" in str(e.value)
    with pytest.raises(D.B200PirError) as e:
        srv.answer(D.serialize_request(make_requests(pool, [65], 0)[0]))
    assert e.value.code == E_SHAPE
    one = D.serialize_request(make_requests(pool, [2], 5)[0])
    assert srv.answer_many([one])[0] == srv.answer(one)


# ------------------------------------------------------------------ chunked servers (e2e.rs:62-105)
@pytest.mark.parametrize("chunks", [2, 3])
def test_serve_chunked_answers_add_up_and_decode(chunks):
    D = _D()
    num_entries = 1 << 24
    prm, data, info, delta, a_1, a_2, st, got = T.gpu_prepared(num_entries, 1, 1)
    rows = T.batch_rows(prm["l"], chunks)
    per_row = prm["m"] * info["packing"]
    rng = np.random.default_rng(600 + chunks)
    idxs = [int(rng.integers(r0 * per_row, min(r1 * per_row, num_entries))) for r0, r1 in rows]
    qs = [E.query(i, a_1, a_2, prm, info, rng) for i in idxs]
    queries = [q for _, q in qs]
    req = D.serialize_request(queries)
    resp = []
    for c, r in enumerate(rows):
        dbm, srv = setup_server(got, prm, info, num_entries, 1, rows=r)      # each server holds only its rows
        try:
            resp.append(srv.answer(req, chunk_idx=c))
            with pytest.raises(D.B200PirError) as e:                          # an unchunked answer needs all l rows
                srv.answer(req)
            assert e.value.code == E_SHAPE
        finally:
            srv.close()
            dbm.close()
    for c in range(chunks):
        assert resp[c] == wire(E.run_answer(st, prm, info, delta, queries, chunk_idx=c), prm, info, delta), c
    parts = [flat(r) for r in resp]
    summed = []
    for k in range(len(parts[0])):
        if k % 2 == 1:
            assert all(np.array_equal(parts[0][k], p[k]) for p in parts), k
            summed.append(parts[0][k])
        else:
            summed.append(sum(p[k].astype(np.uint64) for p in parts).astype(U32))      # wrapping u32
    dbm, srv = setup_server(got, prm, info, num_entries, 1)
    try:
        whole = flat(srv.answer(req))
    finally:
        srv.close()
        dbm.close()
    for k in range(len(whole)):
        assert np.array_equal(summed[k], whole[k]), k
    for b, (i, (client, qmsg)) in enumerate(zip(idxs, qs)):
        assert E.recover(i, got["h2"], qmsg, summed, a_2, client, prm, info, batch_index=b) == int(data[i]), (b, i)


# ------------------------------------------------------------------ the multi-vector kernel against numpy
# Tasks are 32-row tiles; the k range is staged 256 packed columns at a time and split over CTAs when there are fewer than two
# tiles an SM (4096 rows: 128 tiles, split; 20000 rows: 625 tiles, not); vectors run in passes of up to 16.
MANY_SHAPES = ([(r, c) for r in (1, 7, 29) for c in (1, 2, 3, 4, 5)] + [(29, c) for c in (17062, 17063, 17064, 17065, 17066, 21846)]
               + [(1, 21846), (7, 21846), (4096, 5), (4096, 300), (20000, 3), (20000, 257)])
SENTINEL = 0x5A5A5A5A


@pytest.mark.parametrize("rows,cols", MANY_SHAPES)
def test_matvec_packed_many_against_numpy(rows, cols):
    from sdk_b200._lib import LIB, check
    D = _D()
    a, _ = T.extreme_operands(rows, cols, rows * 7919 + cols)
    m = D.PackedMatrix(a, rows, cols)
    try:
        fields = E.unpack_fields(a, rows, cols)
        for v in (1, 2, 15, 16, 17, 33):
            rng = np.random.default_rng(v * 31 + cols)
            b = rng.integers(0, 2**32, (v, 3 * cols), dtype=np.uint64).astype(U32)
            b[0, :] = 0xFFFFFFFF
            b[-1, :3] = 0xFFFFFFFF
            ref = ((fields @ b.astype(np.uint64).T) & np.uint64(0xFFFFFFFF)).astype(U32).T          # (v, rows)
            out = np.full(v * rows + 64, SENTINEL, dtype=U32)
            check(LIB.b200pir_dpir_matvec_packed_many(m._h, b.ctypes.data, v, out.ctypes.data))
            assert np.array_equal(out[:v * rows].reshape(v, rows), ref), v
            assert (out[v * rows:] == SENTINEL).all(), v
            if v in (1, 17):
                assert np.array_equal(D.matrix_mul_vec_packed_many(m, b), ref), v
                assert np.array_equal(D.matrix_mul_vec_packed(m, b[-1]), ref[-1]), v
    finally:
        m.close()


# ------------------------------------------------------------------ errors: a code, nothing written, the server still answers
def test_serve_errors_write_nothing_and_the_server_recovers(l29):
    from sdk_b200._lib import LIB
    D, prm, info, delta, st, got, pool, dbm, srv = l29
    good_q = make_requests(pool, [3], 2)[0]
    good = D.serialize_request(good_q)
    want = wire(E.run_answer(st, prm, info, delta, good_q), prm, info, delta)
    size = srv.answer_size(good)
    q1, q2 = pool[0][0], pool[0][1]
    bad = {
        "truncated": good[:-1],
        "header only": good[:4],
        "empty": b"",
        "zero queries": (0).to_bytes(4, "big"),
        "count 2^28": (1 << 28).to_bytes(4, "big") + good[4:],
        "missing q_2": D.serialize_request([[q1]]),
        "short q_1": D.serialize_request([[q1[:-1], q2]]),
        "q_1 as a row": (1).to_bytes(4, "big") + D.serialize_state([q1.reshape(1, -1), q2]),
        "long q_2": D.serialize_request([[q1, np.concatenate([q2, q2[:3]])]]),
    }

    def answer_rc(req, chunk=-1, cap=size, null=None):
        out = C.create_string_buffer(b"\xa5" * max(cap, 1), max(cap, 1))
        n = C.c_size_t(cap)
        args = [srv._h, req, len(req), chunk, out, C.byref(n)]
        if null is not None:
            args[null] = None
        rc = LIB.b200pir_dpir_answer(*args)
        assert out.raw == b"\xa5" * max(cap, 1) and n.value == cap          # nothing written
        return rc

    def many_rc(reqs, caps=None, null=None):
        k = len(reqs)
        caps = caps or [size] * k
        outs = [C.create_string_buffer(b"\xa5" * c, c) for c in caps]
        arrs = [(C.c_void_p * k)(*[C.cast(C.c_char_p(r), C.c_void_p) for r in reqs]), (C.c_size_t * k)(*[len(r) for r in reqs]),
                (C.c_void_p * k)(*[C.cast(o, C.c_void_p) for o in outs]), (C.c_size_t * k)(*caps)]
        args = [srv._h, arrs[0], arrs[1], k, arrs[2], arrs[3]]
        if null is not None:
            args[null] = None
        rc = LIB.b200pir_dpir_answer_many(*args)
        assert all(o.raw == b"\xa5" * c for o, c in zip(outs, caps)) and list(arrs[3]) == caps
        return rc

    for name, req in bad.items():
        assert answer_rc(req) == E_SHAPE, name
        assert many_rc([good, req]) == E_SHAPE, name
        assert srv.answer(good) == want, name
    assert answer_rc(good, chunk=3) == E_SHAPE                   # chunk index == query count
    assert answer_rc(good, chunk=1 << 40) == E_SHAPE
    assert answer_rc(good, cap=size - 1) == E_BADARG             # the output is too small
    assert many_rc([good, good], caps=[size, size - 4]) == E_BADARG
    for null in (0, 1, 4, 5):
        assert answer_rc(good, null=null) == E_BADARG, null
    for null in (1, 2, 4, 5):
        assert many_rc([good], null=null) == E_BADARG, null
    assert srv.answer(good) == want
    assert srv.answer_many([good, good]) == [want, want]
