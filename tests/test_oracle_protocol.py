"""Semantic (decrypt-and-compare) tests of the CPU oracle, mirroring the reference's own stage
and full-protocol tests (lib/spiral-rs/src/server.rs:787-1047)."""
import numpy as np
import pytest

import oracle_lib as O


def _full_protocol(name, idx, seed=7, **over):
    P = O.Params.named(name, **over)
    cl = O.Client(P, seed)
    pp = cl.generate_keys()
    q = cl.generate_query(idx)
    db = P.generate_db(0xB1755)
    resp, d = P.process_query(pp, q, db, dump=True)
    assert resp.size == P.response_bytes()
    dec = cl.decode_response(resp)
    assert np.array_equal(dec, P.db_plain_item(0xB1755, idx))
    return P, cl, pp, q, db, resp, d


@pytest.mark.parametrize("name,idx", [("T", 77), ("T1", 200), ("T0", 131)])
def test_full_protocol_is_correct(name, idx):
    # server.rs:995-1048 full_protocol_is_correct (+ version-1 packing, lib/server pack.rs:45-98)
    _full_protocol(name, idx)


def test_full_protocol_direct_upload():
    # util.rs:139-153 no-expansion mode (direct_upload): query = v_buf + v_ct
    _full_protocol("T", 19, expand_queries=False)


def test_multiply_reg_by_database_is_correct():
    # server.rs:870-925: one-hot Regev selector over dim0, decrypt row target%num_per
    P = O.Params.named("T")
    cl = O.Client(P, 11)
    cl.generate_keys()
    db = P.generate_db(5)
    target = 0x2B % (P.dim0 * P.num_per) + 100
    t0, t1 = target // P.num_per, target % P.num_per
    scale_k = P.modulus // P.p
    cts = []
    for i in range(P.dim0):
        sigma = np.zeros(P.N, dtype=np.uint64)
        sigma[0] = scale_k if i == t0 else 0
        cts.append(cl.encrypt_reg(sigma).reshape(2, 2, P.N))
    cts = np.stack(cts)  # [j][r][n][z]
    v = (cts[:, :, 0, :] | (cts[:, :, 1, :] << np.uint64(32))).transpose(2, 0, 1).copy()  # [z][j][r]
    out = P.multiply_reg_by_database(db[: P.dim0 * P.num_per * P.N], v.reshape(-1))
    dec = cl.decrypt_reg(out.reshape(P.num_per, 4 * P.N)[t1])
    resc = np.array([O.LIB.orc_rescale(int(x), P.modulus, P.p) for x in dec], dtype=np.uint64)
    plain = P.db_plain_item(5, target).reshape(P.n * P.n, P.N)[0]
    assert np.array_equal(resc, plain)


def test_fold_matches_process_query_dump():
    # the fold stage inside process_query equals the stand-alone fold on the same inputs
    P, cl, pp, q, db, resp, d = _full_protocol("T", 5)
    inter = P.from_ntt(d["first_mult"])          # num_per x (2x1) raw
    folded = P.fold_ciphertexts(inter, d["v_folding"], d["v_folding_neg"])
    assert np.array_equal(folded[: 2 * P.N], d["folded"][: 2 * P.N])
    assert np.array_equal(P.get_v_folding_neg(d["v_folding"]), d["v_folding_neg"])
    # sparse-server zero shortcut (lib/server fold.rs:37-43) is inert on a dense DB
    folded_s = P.fold_ciphertexts(inter, d["v_folding"], d["v_folding_neg"], sparse=True)
    assert np.array_equal(folded_s, folded)


def test_dpir_matvec_matches_numpy():
    # kernels.rs:14-113 vs a plain numpy evaluation of SURVEY A.12; rows not a multiple of 8
    rng = np.random.default_rng(9)
    rows, cols = 43, 37
    a = rng.integers(0, 2**30, rows * cols, dtype=np.uint32)
    b = rng.integers(0, 2**32, 3 * cols, dtype=np.uint32)
    out = O.dpir_matvec_packed(a, b, rows, cols)
    A = a.reshape(rows, cols).astype(np.uint64)
    B = b.astype(np.uint64).reshape(cols, 3)
    exp = np.zeros(rows, dtype=np.uint64)
    for m in range(3):
        exp += (((A >> np.uint64(10 * m)) & np.uint64(1023)) * B[:, m][None, :]).sum(axis=1)
    assert np.array_equal(out, (exp & np.uint64(0xFFFFFFFF)).astype(np.uint32))


def test_avx2_multiply_equals_scalar_u128_path():
    # the SIMD form used for the CPU baseline must agree with server.rs:155-221 on worst-case operands too
    P = O.Params.named("T")
    rng = np.random.default_rng(12)
    Q0, Q1 = 268369921, 249561089
    for dim0, num_per, worst in ((64, 4, False), (1024, 2, True)):
        n = dim0 * num_per * P.N
        if worst:
            db = np.full(n, (Q0 - 1) | ((Q1 - 1) << 32), dtype=np.uint64)
            v = np.full(dim0 * 2 * P.N, (Q0 - 1) | ((Q1 - 1) << 32), dtype=np.uint64)
        else:
            db = rng.integers(0, Q0, n, dtype=np.uint64) | (rng.integers(0, Q1, n, dtype=np.uint64) << np.uint64(32))
            v = (rng.integers(0, Q0, dim0 * 2 * P.N, dtype=np.uint64)
                 | (rng.integers(0, Q1, dim0 * 2 * P.N, dtype=np.uint64) << np.uint64(32)))
        ref = P.multiply_reg_by_database(db, v, dim0, num_per)
        out = np.zeros_like(ref)
        O._ck(O.LIB.orc_multiply_reg_by_database_avx2(P.hp, O._p64(out), O._p64(db), O._p64(v), O.C.c_size_t(dim0), O.C.c_size_t(num_per)))
        assert np.array_equal(out, ref)


@pytest.mark.parametrize("name", ["T", "T1", "T0"])
def test_wire_formats_round_trip(name):
    # client.rs:848-955 public_parameters_serialization_is_correct / query_serialization_is_correct
    P = O.Params.named(name)
    cl = O.Client(P, 606)
    pp = cl.generate_keys()
    b = cl.pp_bytes()
    assert b.size == P.setup_bytes
    pp2 = P.pp_deserialize(b)
    for k in ("pack", "left", "right", "conv"):
        if pp[k] is None:
            assert pp2[k] is None or not pp2[k].any() or k == "right"
        else:
            assert np.array_equal(pp[k], pp2[k][: pp[k].size]), k
    q = cl.generate_query(9)
    qb = cl.query_bytes()
    assert qb.size == P.query_bytes
    assert np.array_equal(P.query_deserialize(qb), q["ct"])


def test_direct_upload_wire_format_round_trip():
    # client.rs:939-955 no_expansion_query_serialization_is_correct (serialize . deserialize . serialize), strengthened:
    # the deserialized query must equal the generated one word for word (the even-indexed words of v_buf and the first rows
    # of v_ct are regenerated from the 32-byte seed), and it must still decode to the planted item
    P = O.Params.named("T", expand_queries=False)
    cl = O.Client(P, 717)
    pp = cl.generate_keys()
    idx = 23
    q = cl.generate_query(idx)
    qb = cl.query_bytes()
    assert qb.size == P.query_bytes == 32 + (P.dim0 + P.nu_2 * 2 * P.t_gsw) * P.N * 8
    q2 = P.query_deserialize_direct(qb)
    assert np.array_equal(q2["v_buf"], q["v_buf"])
    assert np.array_equal(q2["v_ct"], q["v_ct"])
    db = P.generate_db(0xB1755)
    assert np.array_equal(cl.decode_response(P.process_query(pp, q2, db)), P.db_plain_item(0xB1755, idx))


def test_dpir_setup_restatement_against_its_definition():
    # doublepir.rs:76-108: the oracle's setup() against an independent numpy evaluation of the same definition
    # (h_1 = db a_1; transpose; base-p digits centred; concat_cols(x); h_2 = h_1 a_2; squish with 3 x 10 bits)
    rng = np.random.default_rng(1)
    l, m, n, p, delta, x = 24, 20, 8, 929, 4, 2
    db = (rng.integers(0, p, (l, m)).astype(np.int64) - p // 2).astype(np.uint32)
    a1 = rng.integers(0, 2**32, (m, n), dtype=np.uint64).astype(np.uint32)
    a2 = rng.integers(0, 2**32, (l // x, n), dtype=np.uint64).astype(np.uint32)
    o = O.dpir_setup(db, l, m, a1, n, a2, p, delta, x)
    h1 = ((db.astype(np.uint64) @ a1.astype(np.uint64)) & 0xFFFFFFFF).T.copy()
    ex = np.zeros((n * delta, l), dtype=np.uint64)
    v = h1.copy()
    for f in range(delta):
        ex[f::delta] = ((v % p) - p // 2) & 0xFFFFFFFF
        v //= p
    cc = np.zeros((n * delta * x, l // x), dtype=np.uint64)
    for j in range(l):
        cc[np.arange(n * delta) + n * delta * (j % x), j // x] = ex[:, j]
    assert np.array_equal(((cc @ a2.astype(np.uint64)) & 0xFFFFFFFF).astype(np.uint32), o["h2"])
    raw = (cc + p // 2) & 0xFFFFFFFF
    sq = np.zeros((n * delta * x, (l // x + 2) // 3), dtype=np.uint64)
    for k in range(l // x):
        sq[:, k // 3] += raw[:, k] << (10 * (k % 3))
    assert np.array_equal((sq & 0xFFFFFFFF).astype(np.uint32), o["h1_sq"])
    assert np.array_equal(o["a2_t"][:, : l // x], a2.T) and not o["a2_t"][:, l // x:].any()
    assert np.array_equal(O.dpir_mul(db, a1, l, m, n), ((db.astype(np.uint64) @ a1.astype(np.uint64)) & 0xFFFFFFFF).astype(np.uint32))


def test_dpir_answer_tail_restatement_against_its_definition():
    # answer()'s tail in the oracle (matrix_mul_transposed_packed, kernels.rs:180-278; transpose_expand_concat_cols_squish,
    # indexing.rs:117-143) against the numpy definitions the GPU sweeps also use; words with bits 30 and 31 set, 0xffffffff
    import test_oracle_doublepir_e2e as E
    rng = np.random.default_rng(2)
    for a_rows, a_cols, b_rows in [(24, 5, 8), (3, 40, 16), (1, 1, 8), (8, 150, 24)]:     # both of the reference's branches
        a = rng.integers(0, 2**32, a_rows * a_cols, dtype=np.uint64).astype(np.uint32)
        a[:a_cols] = 0xFFFFFFFF
        b = rng.integers(0, 2**32, b_rows * 3 * a_cols, dtype=np.uint64).astype(np.uint32)
        b[0] = 0xFFFFFFFF
        assert np.array_equal(O.dpir_matrix_mul_transposed_packed(a, b, a_rows, a_cols, b_rows, 3 * a_cols),
                              E.np_matrix_mul_transposed_packed(a, b, a_rows, a_cols, b_rows, 3 * a_cols)), (a_rows, a_cols)
    for concat in (1, 2, 3, 4, 8):
        for delta in (1, 2, 4, 5):
            for modulus in (2, 3, 512, 991, 1024):
                for rem in (0, 1, 2):
                    rows, cols = concat * (6 + rem), 1 + rem
                    a = rng.integers(0, 2**32, rows * cols, dtype=np.uint64).astype(np.uint32)
                    a[: rows * cols // 2] = 0xFFFFFFFF
                    o, orows, ocols = O.dpir_transpose_expand_concat_cols_squish(a, rows, cols, modulus, delta, concat)
                    r, rr, rc = E.np_transpose_expand_concat_cols_squish(a, rows, cols, modulus, delta, concat)
                    assert (orows, ocols) == (rr, rc) and np.array_equal(o, r), (concat, delta, modulus, rem)
    a = rng.integers(0, 2**32, 9 * 4, dtype=np.uint64).astype(np.uint32)
    b = rng.integers(0, 2**32, 12, dtype=np.uint64).astype(np.uint32)
    assert np.array_equal(O.dpir_matvec_packed(a, b, 9, 4), E.np_matvec_packed(a, b, 9, 4))


def test_oracle_reproduces_golden_fixtures():
    # tests/golden/spiral_golden.json was frozen from this oracle after the KAT pinning; any drift shows up here
    import json
    import os
    import golden_cases as GC
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "spiral_golden.json")) as f:
        gold = json.load(f)
    assert gold["seed_client"] == GC.GOLDEN_SEED_CLIENT and gold["seed_db"] == GC.GOLDEN_SEED_DB
    for case in GC.GOLDEN_CASES:
        assert GC.oracle_record(case) == gold["cases"][case], case


def test_sparse_server_fold_shortcut_semantics():
    # lib/server/src/compute/fold.rs:37-43: an all-zero first operand is replaced by the second, an all-zero second operand
    # leaves the first untouched; with no all-zero ciphertext the sparse fold is the dense fold
    P = O.Params.named("T")
    cl = O.Client(P, 77)
    pp = cl.generate_keys()
    q = cl.generate_query(5)
    _, vf = P.expand_query(pp, q["ct"])
    vfn = P.get_v_folding_neg(vf)
    rng = np.random.default_rng(8)
    num = 4
    cts = rng.integers(0, P.modulus, num * 2 * P.N, dtype=np.uint64).reshape(num, 2 * P.N)
    dims = 2
    mat = 4 * P.t_gsw * P.W
    vf2, vfn2 = vf[: dims * mat], vfn[: dims * mat]
    assert np.array_equal(P.fold_ciphertexts(cts, vf2, vfn2, sparse=True), P.fold_ciphertexts(cts, vf2, vfn2))
    z = cts.copy()
    z[0] = 0                                   # pair (0, 2): first operand zero -> slot 0 becomes ct 2
    z[3] = 0                                   # pair (1, 3): second operand zero -> slot 1 stays ct 1
    out = P.fold_ciphertexts(z, vf2, vfn2, sparse=True).reshape(num, 2 * P.N)
    one_round = np.stack([z[2], z[1]])         # what round 1 leaves in slots 0, 1
    ref = P.fold_ciphertexts(one_round, vf2[:mat], vfn2[:mat]).reshape(2, 2 * P.N)   # round 2 is a normal external product
    assert np.array_equal(out[0], ref[0])
    assert not np.array_equal(out[0], P.fold_ciphertexts(z, vf2, vfn2).reshape(num, 2 * P.N)[0])


def test_sparse_database_decodes_with_the_sparse_server_fold():
    # a database with whole second-dimension rows absent: populated items still decode under lib/server's fold
    P = O.Params.named("T")
    cl = O.Client(P, 78)
    pp = cl.generate_keys()
    db = P.generate_db(0xABCD).reshape(P.slices, P.N, P.num_per, P.dim0).copy()
    db[:, :, 1::2, :] = 0                       # every odd row ii empty
    db = db.reshape(-1)
    for idx in (0, 2 * 7, P.num_per * 3 + 4):   # items in even rows (item index = j * num_per + ii)
        q = cl.generate_query(idx)
        dense = P.process_query(pp, q, db)
        sparse = P.process_query(pp, q, db, sparse_fold=True)
        assert not np.array_equal(dense, sparse)
        assert np.array_equal(cl.decode_response(sparse), P.db_plain_item(0xABCD, idx))
        assert np.array_equal(cl.decode_response(dense), P.db_plain_item(0xABCD, idx))


def test_load_db_from_seek_restatement():
    # server.rs:277-357: raw file -> database words.  (i) With db_item_size a multiple of the chunk count every item equals
    # what update_item_raw (loading.rs:317-359) builds from the same bytes; (ii) otherwise the last chunk of an item runs
    # into the next item's bytes, as the reference's seek + read does; (iii) items past the end of the file are zero.
    P = O.Params.named("T")
    rng = np.random.default_rng(12)
    total = P.dim0 * P.num_per
    raw = rng.integers(0, 256, total * P.db_item_size - 5000, dtype=np.uint8)      # short file: the last item is truncated
    db = P.load_db_from_bytes(raw).reshape(P.slices, P.N, P.num_per, P.dim0)
    padded = np.concatenate([raw, np.zeros(5000, dtype=np.uint8)])
    for idx in (0, 1, 77, total - 1):
        polys = P.update_item_raw(padded[idx * P.db_item_size:(idx + 1) * P.db_item_size]).reshape(P.slices, P.N)
        ii, j = idx % P.num_per, idx // P.num_per
        assert np.array_equal(db[:, :, ii, j], polys), idx
    kw = dict(P.kw)
    kw["db_item_size"] = P.db_item_size - 2                                          # 4 chunks of ceil((size)/4) bytes overlap
    P2 = O.Params(**kw)
    assert P2.bytes_per_chunk * P2.slices > P2.db_item_size
    raw2 = rng.integers(0, 256, total * P2.db_item_size, dtype=np.uint8)
    db2 = P2.load_db_from_bytes(raw2).reshape(P2.slices, P2.N, P2.num_per, P2.dim0)
    idx = 5
    bpc = P2.bytes_per_chunk
    chunks = [raw2[idx * P2.db_item_size + c * bpc: idx * P2.db_item_size + (c + 1) * bpc] for c in range(P2.slices)]
    assert chunks[-1].size == bpc                                                     # reaches into item idx + 1
    polys = P2.update_item_raw(np.concatenate(chunks)).reshape(P2.slices, P2.N)
    assert np.array_equal(db2[:, :, idx % P2.num_per, idx // P2.num_per], polys)


# ------------------------------------------------------------------ the reference's remaining stage tests, restated on the oracle
def _dec_reg(P, cl, ct_ntt, scale_k):
    # server.rs:753-770 dec_reg: coefficient 0, centred, rounded by scale_k; 0 -> 0, anything else -> 1
    val = int(cl.decrypt_reg(ct_ntt)[0])
    if val >= P.modulus // 2:
        val -= P.modulus
    return 0 if round(val / scale_k) == 0 else 1


def test_coefficient_expansion_is_correct():
    # server.rs:787-830: Enc(scale_k * X^7) expands into 2^g ciphertexts of which exactly number 7 is non-zero
    P = O.Params.named("T")
    cl = O.Client(P, 21)
    pp = cl.generate_keys()
    g = (P.t_gsw * P.nu_2 + P.dim0 - 1).bit_length()
    assert (1 << g) == 1 << (P.nu_1 + 1)                      # the vector length the reference's test allocates
    scale_k = P.modulus // P.p
    target = 7
    sigma = np.zeros(P.N, dtype=np.uint64)
    sigma[target] = scale_k
    v = np.zeros(((1 << g), 2 * P.W), dtype=np.uint64)
    v[0] = cl.encrypt_reg(sigma)
    test_ct = cl.encrypt_reg(sigma)
    out = P.coefficient_expansion(v.reshape(-1), pp).reshape(1 << g, 2 * P.W)
    assert _dec_reg(P, cl, test_ct, scale_k) == 0             # coefficient 0 of the unexpanded ciphertext is empty
    for i in range(1 << g):
        assert _dec_reg(P, cl, out[i], scale_k) == (1 if i == target else 0), i


def test_regev_to_gsw_is_correct():
    # server.rs:832-868 (db_dim_2 = 1): Regev encryptions of 2^(bits_per * i) -> a GSW ciphertext of 1; of zeros -> of 0
    P = O.Params.named("T", nu_2=1)
    cl = O.Client(P, 22)
    pp = cl.generate_keys()
    bits_per = P.bits_per(P.t_gsw)

    def enc_constant(val):
        sigma = np.zeros(P.N, dtype=np.uint64)
        sigma[0] = val
        return cl.encrypt_reg(sigma)

    def dec_gsw(gsw):
        # server.rs:772-785: the last column (index 2 t_gsw - 1), coefficient 0: "this offset should encode a large value"
        m = gsw.reshape(2, 2 * P.t_gsw, P.W)
        val = int(cl.decrypt_reg(np.concatenate([m[0, 2 * P.t_gsw - 1], m[1, 2 * P.t_gsw - 1]]))[0])
        if val >= P.modulus // 2:
            val -= P.modulus
        return 0 if abs(val) < (1 << 10) else 1

    conv = pp["conv"].reshape(-1)[: 2 * 2 * P.t_conv * P.W]                                  # v_conversion[0]
    ones = np.concatenate([enc_constant(1 << (bits_per * i)) for i in range(P.t_gsw)])
    zeros = np.concatenate([enc_constant(0) for _ in range(P.t_gsw)])
    assert dec_gsw(P.regev_to_gsw(ones, conv)) == 1
    assert dec_gsw(P.regev_to_gsw(zeros, conv)) == 0


@pytest.mark.parametrize("target_row,hot_row,expect", [(2, 2, 1), (3, 3, 1), (0, 0, 1), (2, 1, 0)])
def test_fold_ciphertexts_is_correct(target_row, hot_row, expect):
    # server.rs:927-993: num_per Regev ciphertexts, a scale_k only in row `hot_row`; GSW encryptions of the bits of
    # `target_row` select it.  The reference builds the GSW ciphertexts inline from the secret key; here they come from the
    # oracle client's direct-upload query (client.rs:660-721 builds them the same way: column pairs (sk * sigma, sigma) with
    # sigma = bit * 2^(bits_per * j)).
    P = O.Params.named("T", expand_queries=False)
    cl = O.Client(P, 23)
    cl.generate_keys()
    scale_k = P.modulus // P.p
    q = cl.generate_query(5 * P.num_per + target_row)          # second-dimension part of the index = target_row
    v_folding = P.to_ntt(q["v_ct"])                             # nu_2 x (2 x 2 t_gsw)
    v_folding_neg = P.get_v_folding_neg(v_folding)
    rows = []
    for i in range(P.num_per):
        sigma = np.zeros(P.N, dtype=np.uint64)
        sigma[0] = scale_k if i == hot_row else 0
        rows.append(P.from_ntt(cl.encrypt_reg(sigma)))
    folded = P.fold_ciphertexts(np.concatenate(rows), v_folding, v_folding_neg)
    assert _dec_reg(P, cl, P.to_ntt(folded[: 2 * P.N]), scale_k) == expect
