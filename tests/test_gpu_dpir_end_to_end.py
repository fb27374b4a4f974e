"""DoublePIR on the GPU end to end, and its kernels swept against numpy.

The reference has no known-answer vectors for DoublePIR's setup() / answer(): its tests recover planted entries end to end
(doublepir.rs:469-716).  Here GPU setup() and GPU answer() run on the databases pick_params lays out for real entry counts
(n = 1024, so m = 65536 columns and 1 to 64 rows), their outputs are compared word for word with the oracle, and the numpy
client of test_oracle_doublepir_e2e.py decodes the GPU answer back to the planted entry.  The kernels behind answer() are
also swept against numpy definitions (uint64 sums masked to 32 bits) at the shapes where their dispatch changes."""
import numpy as np
import pytest

import test_oracle_doublepir_e2e as E

pytestmark = pytest.mark.gpu

U32 = np.uint32
E_SHAPE, E_UNSUPPORTED = -2, -4


def _D():
    import sdk_b200.doublepir as D
    return D


# ------------------------------------------------------------------ setup() and answer() at the reference's shapes
# (entries, bits, seed) -> (l, packing, x): the layouts pick_params gives these databases (p = 512, delta = 4 for all)
SHAPES = {(1 << 24, 1, 1): (29, 9, 1),         # the reference's simple / batched / chunked tests
          (1 << 20, 10, 2): (32, 0, 2),        # the reference's multi-element test: ne = x = 2, l / x = 16
          (1 << 22, 8, 3): (64, 1, 1),
          (1 << 16, 32, 4): (4, 0, 4),         # l / x = 1
          (1 << 12, 64, 5): (8, 0, 8)}         # l / x = 1, x = 8: h_2 GEMM of 32768 x 1 x 1024

_gpu_state = {}


def gpu_prepared(num_entries, bits, seed):
    """E.prepare (oracle setup, cached per process) plus GPU setup() on the same database and matrices (cached too)."""
    rng, prm, data, info, delta, a_1, a_2, st = E.prepare(num_entries, bits, seed, full_width=True)
    key = (num_entries, bits, seed)
    if key not in _gpu_state:
        _, db = E.db_with_data(num_entries, bits, prm, data)
        _gpu_state[key] = _D().setup(db, a_1, a_2, prm["p"], delta, info["x"])
    return prm, data, info, delta, a_1, a_2, st, _gpu_state[key]


def gpu_answer(dbm, got, prm, info, delta, queries):
    n, l, p, x = prm["n"], prm["l"], prm["p"], info["x"]
    h_1 = (got["h1_squished"].reshape(-1), n * delta * x, got["h1_squished"].shape[1])
    a2t = (got["a2_t"].reshape(-1), n, got["a2_t"].shape[1])
    return _D().answer(dbm, queries, h_1, a2t, p, delta, x, info["ne"])


def packed_db(got, prm):
    return _D().PackedMatrix(np.ascontiguousarray(got["db_squished"]).reshape(-1), prm["l"], got["db_squished"].shape[1])


@pytest.mark.parametrize("num_entries,bits,seed", list(SHAPES))
def test_dpir_setup_equals_oracle_at_reference_shapes(num_entries, bits, seed):
    prm, data, info, delta, a_1, a_2, st, got = gpu_prepared(num_entries, bits, seed)
    l, packing, x = SHAPES[(num_entries, bits, seed)]
    assert (prm["l"], prm["m"], prm["p"], info["packing"], info["x"], delta) == (l, 65536, 512, packing, x, 4)
    assert np.array_equal(got["db_squished"], st["db_sq"])
    assert np.array_equal(got["h1_squished"], st["h1_sq"])
    assert np.array_equal(got["a2_t"], st["a2_t"])
    assert np.array_equal(got["h2"], st["h2"])


def probe_indices(num_entries, prm, info, rng):
    """index 0, the last index, the first entry of the last row, the entry in the last column of row 0, two random ones"""
    m, per = prm["m"], max(info["packing"], 1)
    elems = -(-num_entries // per)
    idx = [0, num_entries - 1, (elems - 1) // m * m * per, (m - 1) * per] + [int(v) for v in rng.integers(0, num_entries, 2)]
    return sorted({i for i in idx if i < num_entries})


@pytest.mark.parametrize("num_entries,bits,seed", list(SHAPES))
def test_dpir_gpu_answer_decodes_at_reference_shapes(num_entries, bits, seed):
    prm, data, info, delta, a_1, a_2, st, got = gpu_prepared(num_entries, bits, seed)
    rng = np.random.default_rng(seed + 100)
    dbm = packed_db(got, prm)
    try:
        for i in probe_indices(num_entries, prm, info, rng):
            client, qmsg = E.query(i, a_1, a_2, prm, info, rng)
            ans = gpu_answer(dbm, got, prm, info, delta, [qmsg])
            ref = E.run_answer(st, prm, info, delta, [qmsg])
            assert len(ans) == len(ref) == 1 + 2 * (info["ne"] // info["x"])
            for k, (g, r) in enumerate(zip(ans, ref)):
                assert np.array_equal(g, r), (i, k)
            assert E.recover(i, got["h2"], qmsg, ans, a_2, client, prm, info) == int(data[i]), i
    finally:
        dbm.close()


def batch_rows(l, nq):
    """answer()'s row batches (doublepir.rs:292-303): l // nq rows each, the remainder in the last"""
    b = l // nq
    return [(k * b, l if k == nq - 1 else (k + 1) * b) for k in range(nq)]


@pytest.mark.parametrize("nq", [2, 3])
def test_dpir_gpu_batched_answer_decodes(nq):
    # doublepir.rs:526-606 with 2 and 3 queries on l = 29: batches of 14 + 15 and 9 + 9 + 11 rows, query k selects from batch k
    num_entries = 1 << 24
    prm, data, info, delta, a_1, a_2, st, got = gpu_prepared(num_entries, 1, 1)
    rows = batch_rows(prm["l"], nq)
    assert [r1 - r0 for r0, r1 in rows] == {2: [14, 15], 3: [9, 9, 11]}[nq]
    per_row = prm["m"] * info["packing"]
    rng = np.random.default_rng(40 + nq)
    dbm = packed_db(got, prm)
    try:
        first = [r0 * per_row for r0, _ in rows]                                     # the first entry of every batch
        drawn = [int(rng.integers(r0 * per_row, min(r1 * per_row, num_entries))) for r0, r1 in rows]
        last = [min(r1 * per_row, num_entries) - 1 for _, r1 in rows]                # the last entry of every batch
        for idxs in (first, drawn, last):
            qs = [E.query(i, a_1, a_2, prm, info, rng) for i in idxs]
            ans = gpu_answer(dbm, got, prm, info, delta, [q for _, q in qs])
            ref = E.run_answer(st, prm, info, delta, [q for _, q in qs])
            assert len(ans) == len(ref) == 1 + 2 * nq
            for k, (g, r) in enumerate(zip(ans, ref)):
                assert np.array_equal(g, r), (idxs, k)
            for b, (i, (client, qmsg)) in enumerate(zip(idxs, qs)):
                assert E.recover(i, got["h2"], qmsg, ans, a_2, client, prm, info, batch_index=b) == int(data[i]), (b, i)
    finally:
        dbm.close()


def chunk_answer(server_db, chunk, rows, queries, got, prm, info, delta):
    """answer() of a server that holds only the rows of batch `chunk` (doublepir.rs:262-303 with raw_data and chunk_idx): the
    other batches contribute zero rows.  Composed from the library's primitives; the library has no chunked answer()."""
    D = _D()
    n, l, p, x = prm["n"], prm["l"], prm["p"], info["x"]
    parts = [D.matrix_mul_vec_packed(server_db, q[0]) if b == chunk else np.zeros(r1 - r0, dtype=U32)
             for b, ((r0, r1), q) in enumerate(zip(rows, queries))]
    a_1, r1, c1 = D.transpose_expand_concat_cols_squish(np.concatenate(parts), l, 1, p, delta, x)
    msg = [D.matrix_mul_transposed_packed(a_1, r1, c1, got["a2_t"].reshape(-1), n, got["a2_t"].shape[1])]
    hm = D.PackedMatrix(got["h1_squished"].reshape(-1), n * delta * x, got["h1_squished"].shape[1])
    am = D.PackedMatrix(a_1, r1, c1)
    try:
        for q in queries:
            for j in range(info["ne"] // x):
                msg.append(D.matrix_mul_vec_packed(hm, q[1 + j]))
                msg.append(D.matrix_mul_vec_packed(am, q[1 + j]))
    finally:
        hm.close()
        am.close()
    return msg


def test_dpir_gpu_chunked_answers_add_up_and_decode():
    # doublepir.rs:607-716 (DESIGN section 6: the sharding model): each of two servers holds one batch of rows
    D = _D()
    num_entries = 1 << 24
    prm, data, info, delta, a_1, a_2, st, got = gpu_prepared(num_entries, 1, 1)
    rows = batch_rows(prm["l"], 2)
    per_row = prm["m"] * info["packing"]
    rng = np.random.default_rng(77)
    idxs = [int(rng.integers(r0 * per_row, min(r1 * per_row, num_entries))) for r0, r1 in rows]
    qs = [E.query(i, a_1, a_2, prm, info, rng) for i in idxs]
    queries = [q for _, q in qs]
    cols = got["db_squished"].shape[1]
    servers = [D.PackedMatrix(np.ascontiguousarray(got["db_squished"][r0:r1]).reshape(-1), r1 - r0, cols) for r0, r1 in rows]
    dbm = packed_db(got, prm)
    try:
        resp = [chunk_answer(servers[c], c, rows, queries, got, prm, info, delta) for c in range(2)]
        whole = gpu_answer(dbm, got, prm, info, delta, queries)
    finally:
        for h in servers + [dbm]:
            h.close()
    for c in range(2):
        ref = E.run_answer(st, prm, info, delta, queries, chunk_idx=c)
        for k, (g, r) in enumerate(zip(resp[c], ref)):
            assert np.array_equal(g, r), (c, k)
    summed = []
    for k in range(len(whole)):
        if k % 2 == 1:                                           # h_1 * q_2 does not depend on the rows a server holds
            assert np.array_equal(resp[0][k], resp[1][k]), k
            summed.append(resp[0][k])
        else:
            summed.append(resp[0][k] + resp[1][k])               # wrapping u32
        assert np.array_equal(summed[k], whole[k]), k
    for b, (i, (client, qmsg)) in enumerate(zip(idxs, qs)):
        assert E.recover(i, got["h2"], qmsg, summed, a_2, client, prm, info, batch_index=b) == int(data[i]), (b, i)


# ------------------------------------------------------------------ matvec dispatch (launch_dpir_matvec) against numpy
# `b` is staged in shared memory up to 17064 packed words a row (3 * 17064 * 4 bytes = 200 KiB), wider rows take the wide
# kernel (17065, 17066).  Below that, even cols run k_dpir_matvec_row and odd cols (1, 3, 5, ...) k_dpir_matvec.  A grid-stride
# pass covers 8448 rows in k_dpir_matvec_row and 33792 in k_dpir_matvec.  Variants 1, 2 and 4 are retired tilings: accepted,
# and they must give the same bytes.
MATVEC_SHAPES = ([(r, c) for r in (1, 7, 8, 9) for c in (1, 2, 3, 4, 5)]
                 + [(9, c) for c in (17062, 17063, 17064, 17065, 17066)]
                 + [(16899, 2), (67589, 3), (67589, 4)])
SENTINEL = 0x5A5A5A5A


def extreme_operands(rows, cols, seed):
    """full 32-bit words (bits 30 and 31 are set in most; the kernels must ignore them), row 0 all ones (every field 1023),
    a word with only the top bits; b with 0xffffffff in its first and last entries"""
    rng = np.random.default_rng(seed)
    a = rng.integers(0, 2**32, rows * cols, dtype=np.uint64).astype(U32)
    a[:cols] = 0xFFFFFFFF
    a[-1] = 0xC0000000
    b = rng.integers(0, 2**32, 3 * cols, dtype=np.uint64).astype(U32)
    b[:3] = 0xFFFFFFFF
    b[-3:] = 0xFFFFFFFF
    return a, b


@pytest.mark.parametrize("rows,cols", MATVEC_SHAPES)
def test_dpir_matvec_dispatch_against_numpy(rows, cols):
    import torch
    from sdk_b200._lib import LIB, check
    D = _D()
    a, b = extreme_operands(rows, cols, rows * 100003 + cols)
    ref = E.np_matvec_packed(a, b, rows, cols)
    stream = torch.cuda.Stream()
    m = D.PackedMatrix(a, rows, cols)
    try:
        check(LIB.b200pir_dpir_set_stream(m._h, stream.cuda_stream))
        b_dev = torch.from_numpy(b.view(np.int32)).cuda()
        out = torch.empty(rows + 64, dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        for variant in (0, 1, 2, 4):
            with torch.cuda.stream(stream):
                out.fill_(SENTINEL)
            check(LIB.b200pir_dpir_matvec_packed_dev(m._h, b_dev.data_ptr(), out.data_ptr(), variant))
            stream.synchronize()
            got = out.cpu().numpy().view(U32)
            assert np.array_equal(got[:rows], ref), variant
            assert (got[rows:] == SENTINEL).all(), variant          # no word written past the output
        assert np.array_equal(D.matrix_mul_vec_packed(m, b), ref)   # the host entry point, on the caller's stream too
    finally:
        m.close()


@pytest.mark.parametrize("rows,cols", [(67, 5), (67, 6), (9, 17065)])
def test_dpir_matvec_row_ranges_against_numpy(rows, cols):
    # matrix_mul_vec_packed(db.rows(start, n), q) (doublepir.rs:301): odd starts with odd and even cols (a row pointer that is
    # only 4-byte aligned), the last row alone, the whole range, empty ranges
    D = _D()
    a, b = extreme_operands(rows, cols, rows + cols)
    ref = E.np_matvec_packed(a, b, rows, cols)
    m = D.PackedMatrix(a, rows, cols)
    try:
        for begin, count in [(1, rows - 2), (3, 5), (5, 1), (rows - 1, 1), (0, rows), (4, 0), (rows, 0)]:
            assert np.array_equal(D.matrix_mul_vec_packed_rows(m, begin, count, b), ref[begin:begin + count]), (begin, count)
        for begin, count in [(rows, 1), (rows - 1, 2), (0, rows + 1), (2**64 - 1, 2)]:
            with pytest.raises(D.B200PirError) as e:
                D.matrix_mul_vec_packed_rows(m, begin, count, b)
            assert e.value.code == E_SHAPE, (begin, count)
    finally:
        m.close()


# ------------------------------------------------------------------ answer() tail against numpy
@pytest.mark.parametrize("concat", [1, 2, 3, 4, 8])
def test_dpir_transpose_expand_concat_cols_squish_against_numpy(concat):
    D = _D()
    rng = np.random.default_rng(concat)
    for delta in (1, 2, 4, 5):
        for modulus in (2, 3, 512, 991, 1024):
            for rem in (0, 1, 2):                                   # (rows / concat) mod 3: a full, a one- and a two-field last word
                rows, cols = concat * (6 + rem), 1 + rem
                a = rng.integers(0, 2**32, rows * cols, dtype=np.uint64).astype(U32)
                a[: rows * cols // 2] = 0xFFFFFFFF
                out, orows, ocols = D.transpose_expand_concat_cols_squish(a, rows, cols, modulus, delta, concat)
                ref, rr, rc = E.np_transpose_expand_concat_cols_squish(a, rows, cols, modulus, delta, concat)
                assert (orows, ocols) == (rr, rc) and np.array_equal(out, ref), (delta, modulus, rem)


@pytest.mark.parametrize("a_rows,a_cols,b_rows", [(24, 5, 8), (40, 11, 16), (1, 1, 8),        # a_rows > a_cols / a_rows = a_cols
                                                  (3, 40, 8), (8, 150, 24), (5, 21846, 16)])    # a_rows < a_cols
def test_dpir_matrix_mul_transposed_packed_against_numpy(a_rows, a_cols, b_rows):
    D = _D()
    rng = np.random.default_rng(a_rows * 7 + a_cols)
    a = rng.integers(0, 2**32, a_rows * a_cols, dtype=np.uint64).astype(U32)
    a[:a_cols] = 0xFFFFFFFF
    b = rng.integers(0, 2**32, b_rows * 3 * a_cols, dtype=np.uint64).astype(U32)
    b[: 3 * a_cols] = 0xFFFFFFFF
    got = D.matrix_mul_transposed_packed(a, a_rows, a_cols, b, b_rows, 3 * a_cols)
    assert np.array_equal(got, E.np_matrix_mul_transposed_packed(a, b, a_rows, a_cols, b_rows, 3 * a_cols))


# ------------------------------------------------------------------ GEMM and setup() limits
def test_dpir_matmul_rows_beyond_one_grid():
    """More row tiles than gridDim.y can hold (65535): 128 * 65535 + 1 rows, K = N = 1."""
    D = _D()
    rows = 128 * 65535 + 1
    rng = np.random.default_rng(9)
    a = (rng.integers(0, 65536, (rows, 1)).astype(np.int64) - 32768).astype(U32)
    a[-1, 0] = 32767
    b = np.array([[0xFFFFFFF1]], dtype=U32)
    want = ((a.astype(np.uint64) * np.uint64(0xFFFFFFF1)) & np.uint64(0xFFFFFFFF)).astype(U32)
    assert np.array_equal(D.matmul(a, b), want)


def test_dpir_matmul_left_operand_range():
    D = _D()
    b = np.array([[3, 0xFFFFFFFF]], dtype=U32)
    for v in (-32768, 32767):
        a = np.array([[v]], dtype=np.int64).astype(U32)
        assert np.array_equal(D.matmul(a, b), ((a.astype(np.uint64) @ b.astype(np.uint64)) & np.uint64(0xFFFFFFFF)).astype(U32))
    for v in (32768, -32769):
        with pytest.raises(D.B200PirError) as e:
            D.matmul(np.array([[v]], dtype=np.int64).astype(U32), b)
        assert e.value.code == E_UNSUPPORTED, v


def test_dpir_setup_refuses_bad_parameters():
    from sdk_b200._lib import LIB
    D = _D()
    l, m, n, x = 6, 5, 4, 2
    db = np.zeros((l, m), dtype=U32)
    a1 = np.zeros((m, n), dtype=U32)
    a2 = np.zeros((l // x, n), dtype=U32)
    for p in (1, 1025):
        with pytest.raises(D.B200PirError) as e:
            D.setup(db, a1, a2, p, 4, x)
        assert e.value.code == E_UNSUPPORTED, p
    # l % x != 0 through the C ABI (the Python wrapper refuses it before the call)
    outs = [np.zeros(1 << 12, dtype=U32) for _ in range(4)]
    rc = LIB.b200pir_dpir_setup(0, db.ctypes.data, l, m, a1.ctypes.data, n, a2.ctypes.data, 512, 4, 4,
                                *[o.ctypes.data for o in outs])
    assert rc == E_SHAPE
    with pytest.raises(ValueError):
        D.setup(db, a1, np.zeros((1, n), dtype=U32), 512, 4, 4)
