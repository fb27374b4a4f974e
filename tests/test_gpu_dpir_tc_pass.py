"""DoublePIR's database pass on the tensor cores (dpir_tc.cu, k_dpir_matvec_tc): the kernel against numpy and against one vector
at a time, at vector counts on both sides of the selection threshold and of the pass size P = 64, over ragged shapes, odd rows
that are only 8-byte aligned and operand extremes; answer_many on the tensor-core path byte for byte against each request alone
(which runs the integer kernel) and against the oracle, decoded; a server built by `load` at 2^30 entries serving 65 requests;
and every error code, after which the server still answers."""
import numpy as np
import pytest

import test_gpu_dpir_end_to_end as T
import test_gpu_dpir_serve as S
import test_oracle_doublepir_e2e as E

pytestmark = pytest.mark.gpu

U32 = np.uint32
P = 64
SENTINEL = 0x5A5A5A5A


def _D():
    import sdk_b200.doublepir as D
    return D


def ref_matvec(a, rows, cols, b):
    """(v, rows) = matrix_mul_vec_packed of every row of b, in row blocks (wrapping u32)"""
    out = np.zeros((b.shape[0], rows), dtype=U32)
    bt = b.astype(np.uint64).T
    for r0 in range(0, rows, 64):
        r1 = min(rows, r0 + 64)
        f = E.unpack_fields(a[r0 * cols:r1 * cols], r1 - r0, cols)
        out[:, r0:r1] = ((f @ bt) & np.uint64(0xFFFFFFFF)).astype(U32).T
    return out


def vectors(v, cols, seed):
    rng = np.random.default_rng(seed)
    b = rng.integers(0, 2**32, (v, 3 * cols), dtype=np.uint64).astype(U32)
    b[0, :] = 0xFFFFFFFF                               # every query word all ones
    b[-1, :3] = 0xFFFFFFFF
    return b


def tc_many(m, b):
    from sdk_b200._lib import LIB, check
    D = _D()
    v = b.shape[0]
    out = np.full(v * m.rows + 64, SENTINEL, dtype=U32)
    check(LIB.b200pir_dpir_matvec_packed_many_on(m._h, np.ascontiguousarray(b).ctypes.data, v, out.ctypes.data, D.MV_TC))
    assert (out[v * m.rows:] == SENTINEL).all()
    return out[:v * m.rows].reshape(v, m.rows)


# ------------------------------------------------------------------ the kernel against numpy
SMALL_ROWS = (1, 31, 32, 33, 63, 64, 65, 127, 128, 129)
SHAPES = ([(r, c) for r in SMALL_ROWS for c in (1, 2, 3, 4, 5, 31, 32, 33)]
          + [(r, 21846) for r in (1, 29, 33, 65)] + [(1821, 33), (1821, 21846)])


@pytest.mark.parametrize("rows,cols", SHAPES)
def test_tc_pass_against_numpy_and_one_vector_at_a_time(rows, cols):
    D = _D()
    a, _ = T.extreme_operands(rows, cols, rows * 7919 + cols)        # words with bits 30 and 31 set, all-ones words
    m = D.PackedMatrix(a, rows, cols)
    try:
        # the selection picks the tensor cores above 8 vectors; P = 64 vectors a pass
        vs = (1, 2, 3, 8, 9, P - 1, P, P + 1, 2 * P + 1) if cols < 100 else ((1, 2, 9, P, P + 1) if rows < 1000 else (P,))
        for v in vs:
            b = vectors(v, cols, v * 31 + cols)
            want = ref_matvec(a, rows, cols, b)
            got = tc_many(m, b)
            assert np.array_equal(got, want), v
            assert np.array_equal(D.matrix_mul_vec_packed_many(m, b), want), v
            for k in {0, v - 1}:
                assert np.array_equal(got[k], D.matrix_mul_vec_packed(m, b[k])), (v, k)
        b = vectors(P + 1, cols, 7)
        assert np.array_equal(tc_many(m, b), D._matvec_packed_many_on(m, b, D.MV_MULTI))
    finally:
        m.close()


def test_tc_pass_refuses_an_unknown_kernel():
    D = _D()
    m = D.PackedMatrix(np.arange(6, dtype=U32), 2, 3)
    try:
        with pytest.raises(D.B200PirError) as e:
            D._matvec_packed_many_on(m, np.zeros((1, 9), dtype=U32), 3)
        assert e.value.code == S.E_BADARG
    finally:
        m.close()


# ------------------------------------------------------------------ answer_many on the tensor-core path
@pytest.mark.parametrize("num_entries,bits,seed", S.SHAPES)
def test_tc_answer_many_at_reference_shapes(num_entries, bits, seed):
    D = _D()
    prm, data, info, delta, a_1, a_2, st, got = T.gpu_prepared(num_entries, bits, seed)
    rng = np.random.default_rng(seed + 900)
    idxs = T.probe_indices(num_entries, prm, info, rng)
    qs = [E.query(i, a_1, a_2, prm, info, rng) for i in idxs]
    pool = [q for _, q in qs]
    dbm, srv = S.setup_server(got, prm, info, num_entries, bits, max_queries=3 * P)
    try:
        sizes = [1 + (k % 3) for k in range(P + 6)]                   # 71 requests, 141 queries: rows cut into segments
        reqs = S.make_requests(pool, sizes, 0)
        wires = [D.serialize_request(q) for q in reqs]
        many = srv.answer_many(wires)
        for k, (q, w, r) in enumerate(zip(reqs, wires, many)):
            assert r == srv.answer(w), k
            if k < 6:
                assert r == S.wire(E.run_answer(st, prm, info, delta, q), prm, info, delta), k
        singles = srv.answer_many([D.serialize_request([q]) for q in pool] * 12)     # single-query requests, > P of them
        for k, (i, (client, qmsg)) in enumerate(zip(idxs, qs)):
            assert singles[k] == srv.answer(D.serialize_request([qmsg])), k
            assert E.recover(i, got["h2"], qmsg, S.flat(singles[k]), a_2, client, prm, info) == int(data[i]), i
    finally:
        srv.close()
        dbm.close()


@pytest.fixture(scope="module")
def l29_big():
    D = _D()
    num_entries = 1 << 24
    prm, data, info, delta, a_1, a_2, st, got = T.gpu_prepared(num_entries, 1, 1)
    rng = np.random.default_rng(700)
    pool = [E.query(int(i), a_1, a_2, prm, info, rng)[1] for i in rng.integers(0, num_entries, 20)]
    dbm, srv = S.setup_server(got, prm, info, num_entries, 1, max_queries=2 * P + 1)
    yield D, prm, info, delta, st, got, pool, dbm, srv
    srv.close()
    dbm.close()


@pytest.mark.parametrize("count", [P - 1, P, P + 1, "max"])
def test_tc_answer_many_counts(l29_big, count):
    D, prm, info, delta, st, got, pool, dbm, srv = l29_big
    sizes = [1] * (2 * P + 1) if count == "max" else [[1, 2, 1, 1][k % 4] for k in range(count)]
    assert sum(sizes) <= 2 * P + 1
    reqs = S.make_requests(pool, sizes, 3)
    wires = [D.serialize_request(q) for q in reqs]
    many = srv.answer_many(wires)
    for k, (q, w, r) in enumerate(zip(reqs, wires, many)):
        assert r == srv.answer(w), k
        if k % 16 == 0:
            assert r == S.wire(E.run_answer(st, prm, info, delta, q), prm, info, delta), k


def test_tc_errors_write_nothing_and_the_server_recovers(l29_big):
    # the error walk of the integer-kernel server, on a server whose answer_many runs the tensor-core passes; then > P requests
    S.test_serve_errors_write_nothing_and_the_server_recovers(l29_big)
    D, prm, info, delta, st, got, pool, dbm, srv = l29_big
    wires = [D.serialize_request(q) for q in S.make_requests(pool, [1] * (P + 1), 5)]
    assert srv.answer_many(wires) == [srv.answer(w) for w in wires]


def test_tc_server_from_load_at_2_30_serves_65_requests():
    import test_gpu_dpir_load as LT
    D = _D()
    num_entries = 1 << 30
    prm = E.pick_params(num_entries, 1, E.SEC_PARAM, E.LOGQ)
    assert (prm["l"], prm["m"]) == (1821, 65536)
    data = np.random.default_rng(31).integers(0, 256, num_entries // 8, dtype=np.uint8)
    loaded = D.load(prm, num_entries, 1, data, D.ENTRY_BITS)
    dbm, out, info, a_1, a_2 = LT._client_view(prm, loaded)
    srv = D.Server(dbm, out["h1_squished"], out["a2_t"], prm, num_entries, 1, max_queries=P + 1)
    try:
        rng = np.random.default_rng(32)
        idxs = [0, num_entries - 1] + [int(v) for v in rng.integers(0, num_entries, 11)]
        qs = [E.query(i, a_1, a_2, prm, info, rng) for i in idxs]
        wires = [D.serialize_request([q]) for _, q in qs] * 5              # 65 requests of 13 clients' queries
        many = srv.answer_many(wires)
        assert len(many) == P + 1
        for k, w in enumerate(wires):
            assert many[k] == many[k % len(idxs)], k
        for k, (i, (client, qmsg)) in enumerate(zip(idxs, qs)):
            assert many[k] == srv.answer(wires[k]), k
            assert E.recover(i, out["h2"], qmsg, S.flat(many[k]), a_2, client, prm, info) == LT._bit(data, i), i
    finally:
        srv.close()
        dbm.close()
