"""Parity of the CUDA path (through the C ABI) against the CPU oracle, stage by stage and end to end.
Bit-exact: every comparison is array equality on integers/bytes."""
import numpy as np
import pytest

import oracle_lib as O

pytestmark = pytest.mark.gpu

SEED_DB = 0xB1755
Q0, Q1 = 268369921, 249561089


def _gpu():
    import sdk_b200.spiral as S
    return S


_cache = {}


def setup_case(name, expand=True):
    """oracle params + client + keys + DB, and the matching GPU context / handles (cached per module)."""
    key = (name, expand)
    if key in _cache:
        return _cache[key]
    S = _gpu()
    P = O.Params.named(name, expand_queries=expand)
    cl = O.Client(P, 1234)
    pp = cl.generate_keys()
    db = P.generate_db(SEED_DB)
    G = S.Params(expand_queries=expand, **P.kw)
    gdb = S.Database.from_words(G, db)
    gpp = S.PublicParameters(G, pp["pack"], pp.get("left"), pp.get("right"), pp.get("conv"))
    _cache[key] = (S, P, cl, pp, db, G, gdb, gpp)
    return _cache[key]


CASES = ["T", "T1", "T0"]


# ------------------------------------------------------------------ primitives
def test_sizes_match_reference_formulas():
    S, P, cl, pp, db, G, gdb, gpp = setup_case("T")
    for name in ("E0", "E1", "S8", "T1", "T0"):
        Po = O.Params.named(name)
        Gp = S.Params(**Po.kw)
        assert (Gp.setup_bytes, Gp.query_bytes, Gp.response_bytes) == (Po.setup_bytes, Po.query_bytes, Po.response_bytes())
        Gp.close()


def test_ntt_forward_inverse_match_oracle():
    S, P, cl, pp, db, G, gdb, gpp = setup_case("T")
    rng = np.random.default_rng(1)
    count = 37
    v = np.empty((count, 2, 2048), dtype=np.uint64)
    v[:, 0, :] = rng.integers(0, Q0, (count, 2048), dtype=np.uint64)
    v[:, 1, :] = rng.integers(0, Q1, (count, 2048), dtype=np.uint64)
    v[0] = 0
    v[1, 0, :] = Q0 - 1
    v[1, 1, :] = Q1 - 1
    v[2] = 0
    v[2, :, 0] = 100                       # ntt.rs:400-409 KAT input
    v = v.reshape(-1)
    ref = P.ntt_forward(v)
    got = v.copy()
    S.ntt_forward(G, got)
    assert np.array_equal(got, ref)
    assert np.all(got.reshape(count, 2, 2048)[2] == 100)
    back = got.copy()
    S.ntt_inverse(G, back)
    assert np.array_equal(back, P.ntt_inverse(ref))
    assert np.array_equal(back, v)


def test_ntt_forward_lazy_inputs():
    # to_ntt_no_reduce feeds un-reduced (< 4q) values (poly.rs:625-638)
    S, P, cl, pp, db, G, gdb, gpp = setup_case("T")
    rng = np.random.default_rng(2)
    v = rng.integers(0, 4 * Q1, 5 * 2 * 2048, dtype=np.uint64)
    got = v.copy()
    S.ntt_forward(G, got)
    assert np.array_equal(got, P.ntt_forward(v))


def test_to_ntt_from_ntt_match_oracle():
    S, P, cl, pp, db, G, gdb, gpp = setup_case("T")
    rng = np.random.default_rng(3)
    raw = rng.integers(0, P.modulus, 9 * 2048, dtype=np.uint64)
    raw[:2048] = 0
    raw[2048:4096] = P.modulus            # the non-canonical value q (SURVEY A.6)
    raw[4096:6144] = P.modulus - 1
    ntt = S.to_ntt(G, raw)
    assert np.array_equal(ntt, P.to_ntt(raw))
    assert np.array_equal(S.from_ntt(G, ntt), P.from_ntt(ntt))
    ntt_r = np.concatenate([rng.integers(0, Q0, 2048, dtype=np.uint64), rng.integers(0, Q1, 2048, dtype=np.uint64)])
    assert np.array_equal(S.from_ntt(G, ntt_r), P.from_ntt(ntt_r))


# ------------------------------------------------------------------ first dimension
@pytest.mark.parametrize("name", CASES)
def test_multiply_reg_by_database_matches_oracle(name):
    S, P, cl, pp, db, G, gdb, gpp = setup_case(name)
    rng = np.random.default_rng(4)
    v = (rng.integers(0, Q0, P.dim0 * 2 * P.N, dtype=np.uint64)
         | (rng.integers(0, Q1, P.dim0 * 2 * P.N, dtype=np.uint64) << np.uint64(32)))
    slice_words = P.dim0 * P.num_per * P.N
    for s in sorted({0, P.slices - 1}):
        ref = P.multiply_reg_by_database(db[s * slice_words:(s + 1) * slice_words], v)
        for variant in (0, 1, 2, 3):
            G.set_option("mul_variant", variant)
            got = S.multiply_reg_by_database(G, gdb, s, v)
            assert np.array_equal(got, ref), (name, s, variant)
    G.set_option("mul_variant", 0)


def test_multiply_worst_case_operands_do_not_overflow():
    # all residues q-1, dim0 = 64: checks the 64-bit accumulation / periodic reduction path
    S, P, cl, pp, db, G, gdb, gpp = setup_case("T")
    w = np.uint64((Q0 - 1) | ((Q1 - 1) << 32))
    dbw = np.full(P.dim0 * P.num_per * P.N, w, dtype=np.uint64)
    v = np.full(P.dim0 * 2 * P.N, w, dtype=np.uint64)
    d2 = S.Database(G)
    for s in range(P.slices):
        d2.upload_slice(s, dbw)
    got = S.multiply_reg_by_database(G, d2, 1, v)
    assert np.array_equal(got, P.multiply_reg_by_database(dbw, v))
    d2.close()


def test_multiply_long_first_dimension_reduction():
    # dim0 = 1024 (nu_1 = 10) with maximal operands exercises the mid-loop reduction (>256 products)
    S = _gpu()
    kw = dict(O.PARAM_SETS["T"])
    kw.update(nu_1=10, nu_2=1, n=1, db_item_size=2048)
    P = O.Params(**kw)
    G = S.Params(**kw)
    w = np.uint64((Q0 - 1) | ((Q1 - 1) << 32))
    rng = np.random.default_rng(5)
    dbw = np.full(P.dim0 * P.num_per * P.N, w, dtype=np.uint64)
    dbw[::7] = rng.integers(0, Q0, dbw[::7].size, dtype=np.uint64) | (rng.integers(0, Q1, dbw[::7].size, dtype=np.uint64) << np.uint64(32))
    v = np.full(P.dim0 * 2 * P.N, w, dtype=np.uint64)
    gdb = S.Database.from_words(G, dbw)
    assert np.array_equal(S.multiply_reg_by_database(G, gdb, 0, v), P.multiply_reg_by_database(dbw, v))
    gdb.close()
    G.close()


def test_synthetic_db_matches_oracle_generator():
    S, P, cl, pp, db, G, gdb, gpp = setup_case("T")
    d2 = S.Database(G)
    d2.fill_synthetic(SEED_DB)
    rng = np.random.default_rng(6)
    v = (rng.integers(0, Q0, P.dim0 * 2 * P.N, dtype=np.uint64)
         | (rng.integers(0, Q1, P.dim0 * 2 * P.N, dtype=np.uint64) << np.uint64(32)))
    for s in range(P.slices):
        assert np.array_equal(S.multiply_reg_by_database(G, d2, s, v), S.multiply_reg_by_database(G, gdb, s, v))
    d2.close()


def test_upsert_item_equals_bulk_upload():
    # lib/server db/loading.rs:317-359: one preprocessed item poly replaces db[idx]
    S, P, cl, pp, db, G, gdb, gpp = setup_case("T")
    d2 = S.Database(G)       # all-zero database
    slice_words = P.dim0 * P.num_per * P.N
    sl = db[:slice_words].reshape(P.N, P.num_per, P.dim0)
    rng = np.random.default_rng(7)
    items = [0, 5, P.dim0 * P.num_per - 1, 77]
    for it in items:
        ii, j = it % P.num_per, it // P.num_per
        d2.upsert_item(0, it, np.ascontiguousarray(sl[:, ii, j]))
    sparse = np.zeros_like(sl)
    for it in items:
        ii, j = it % P.num_per, it // P.num_per
        sparse[:, ii, j] = sl[:, ii, j]
    v = (rng.integers(0, Q0, P.dim0 * 2 * P.N, dtype=np.uint64)
         | (rng.integers(0, Q1, P.dim0 * 2 * P.N, dtype=np.uint64) << np.uint64(32)))
    assert np.array_equal(S.multiply_reg_by_database(G, d2, 0, v), P.multiply_reg_by_database(sparse.reshape(-1), v))
    d2.close()


# ------------------------------------------------------------------ second dimension
@pytest.mark.parametrize("name", CASES)
def test_fold_and_folding_neg_match_oracle(name):
    S, P, cl, pp, db, G, gdb, gpp = setup_case(name)
    q = cl.generate_query(3)
    resp, d = P.process_query(pp, q, db, dump=True)
    assert np.array_equal(S.get_v_folding_neg(G, d["v_folding"]), d["v_folding_neg"])
    inter = P.from_ntt(d["first_mult"])
    ref = P.fold_ciphertexts(inter, d["v_folding"], d["v_folding_neg"])
    got = inter.copy()
    S.fold_ciphertexts(G, got, d["v_folding"], d["v_folding_neg"])
    # the reference leaves partially folded values in slots >= 1; every slot must agree
    assert np.array_equal(got, ref)
    # fast path (v_folding_neg implied, as in process_query): same bytes in every slot
    fast = inter.copy()
    S.fold_ciphertexts(G, fast, d["v_folding"])
    assert np.array_equal(fast, ref)
    # a sub-fold (len 2) uses only v_folding[0]  (server.rs:398-420)
    two = inter[: 2 * 2 * P.N].copy()
    ref2 = P.fold_ciphertexts(two, d["v_folding"], d["v_folding_neg"])
    S.fold_ciphertexts(G, two, d["v_folding"], d["v_folding_neg"])
    assert np.array_equal(two, ref2)
    one = inter[: 2 * P.N].copy()
    S.fold_ciphertexts(G, one, d["v_folding"], d["v_folding_neg"])      # len 1: no-op (server.rs:394-396)
    assert np.array_equal(one, inter[: 2 * P.N])


# ------------------------------------------------------------------ expansion
# expand_pair_min_ctas: rounds with at least that many active ciphertexts use the paired kernel (one CTA = both outputs
# of an input, inverse transform shared through the negacyclic shift); 1 = every round, 1 << 30 = never, 8 = mixed
@pytest.mark.parametrize("pair_min", [1, 8, 1 << 30])
@pytest.mark.parametrize("name", CASES)
def test_expand_query_matches_oracle(name, pair_min):
    S, P, cl, pp, db, G, gdb, gpp = setup_case(name)
    q = cl.generate_query(P.dim0 * P.num_per - 2)
    vreg_ref, vf_ref = P.expand_query(pp, q["ct"])
    G.set_option("expand_pair_min_ctas", pair_min)
    try:
        vreg, vf = S.expand_query(G, gpp, S.Query(ct=q["ct"]))
    finally:
        G.set_option("expand_pair_min_ctas", 528)
    assert np.array_equal(vreg, vreg_ref)
    assert np.array_equal(vf, vf_ref)


@pytest.mark.parametrize("pair_min,variant", [(1, 0), (4, 0), (1, 2), (4, 2), (1 << 30, 0)])
@pytest.mark.parametrize("name", ["T0", "T"])
def test_coefficient_expansion_matches_oracle_all_slots(name, pair_min, variant):
    # expand_variant 0: paired rounds as inverse-transform kernel + single-modulus CTAs; 2: paired rounds in one kernel
    S, P, cl, pp, db, G, gdb, gpp = setup_case(name)
    q = cl.generate_query(9)
    v = np.zeros((1 << P.g) * 2 * P.W, dtype=np.uint64)
    v[: 2 * P.W] = P.to_ntt(q["ct"])
    ref = P.coefficient_expansion(v, pp)
    got = v.copy()
    G.set_option("expand_pair_min_ctas", pair_min)
    G.set_option("expand_variant", variant)
    try:
        S.coefficient_expansion(G, gpp, got)
    finally:
        G.set_option("expand_pair_min_ctas", 528)
        G.set_option("expand_variant", 0)
    assert np.array_equal(got, ref)


def test_process_query_with_paired_expansion_everywhere():
    S, P, cl, pp, db, G, gdb, gpp = setup_case("T")
    idxs = [1, 200, 33, 255, 128]
    qs = np.concatenate([cl.generate_query(i)["ct"] for i in idxs])
    G.set_option("expand_pair_min_ctas", 1)
    try:
        out = S.process_query_batch(G, gpp, qs, gdb)
    finally:
        G.set_option("expand_pair_min_ctas", 528)
    for k, i in enumerate(idxs):
        assert np.array_equal(out[k], P.process_query(pp, dict(ct=qs[k * 2 * P.N:(k + 1) * 2 * P.N]), db)), k
        assert np.array_equal(cl.decode_response(out[k]), P.db_plain_item(SEED_DB, i))


# ------------------------------------------------------------------ pack / encode
@pytest.mark.parametrize("name", CASES)
def test_pack_and_encode_match_oracle(name):
    S, P, cl, pp, db, G, gdb, gpp = setup_case(name)
    q = cl.generate_query(11)
    resp, d = P.process_query(pp, q, db, dump=True)
    nn = P.n * P.n
    for inst in range(P.instances):
        cts = d["folded"][inst * nn * 2 * P.N:(inst + 1) * nn * 2 * P.N]
        assert np.array_equal(S.pack(G, gpp, cts), P.pack(cts, pp["pack"]))
    assert np.array_equal(S.encode(G, d["packed"]), P.encode(d["packed"]))
    assert np.array_equal(S.encode(G, d["packed"]), resp)
    # extreme inputs to rescale (arith.rs:429-444): 0, q/2 boundaries, q-1
    ext = d["packed"].copy()
    ext[:6] = [0, 1, P.modulus // 2 - 1, P.modulus // 2, P.modulus // 2 + 1, P.modulus - 1]
    assert np.array_equal(S.encode(G, ext), P.encode(ext))


# ------------------------------------------------------------------ end to end
@pytest.mark.parametrize("name", CASES)
def test_process_query_bytes_and_decode(name):
    S, P, cl, pp, db, G, gdb, gpp = setup_case(name)
    for idx in (0, 77 % (P.dim0 * P.num_per), P.dim0 * P.num_per - 1):
        q = cl.generate_query(idx)
        ref = P.process_query(pp, q, db)
        got = S.process_query(G, gpp, S.Query(ct=q["ct"]), gdb)
        assert np.array_equal(got, ref), (name, idx)
        assert np.array_equal(cl.decode_response(got), P.db_plain_item(SEED_DB, idx))


def test_process_query_direct_upload():
    S, P, cl, pp, db, G, gdb, gpp = setup_case("T", expand=False)
    q = cl.generate_query(42)
    ref = P.process_query(pp, q, db)
    got = S.process_query(G, gpp, S.Query(v_buf=q["v_buf"], v_ct=q["v_ct"]), gdb)
    assert np.array_equal(got, ref)
    assert np.array_equal(cl.decode_response(got), P.db_plain_item(SEED_DB, 42))


@pytest.mark.parametrize("group", [1, 2, 4])
def test_process_query_batch_equals_single(group):
    S, P, cl, pp, db, G, gdb, gpp = setup_case("T")
    idxs = [1, 200, 33, 255, 128, 7, 64]
    qs = np.concatenate([cl.generate_query(i)["ct"] for i in idxs])
    G.set_option("batch", group)
    out = S.process_query_batch(G, gpp, qs, gdb)
    G.set_option("batch", 16)
    for k, i in enumerate(idxs):
        ref = P.process_query(pp, dict(ct=qs[k * 2 * P.N:(k + 1) * 2 * P.N]), db)
        assert np.array_equal(out[k], ref), (group, k)
        assert np.array_equal(cl.decode_response(out[k]), P.db_plain_item(SEED_DB, i))


def test_error_behaviour():
    S, P, cl, pp, db, G, gdb, gpp = setup_case("T")
    with pytest.raises(S.B200PirError):
        S.multiply_reg_by_database(G, gdb, 99, np.zeros(P.dim0 * 2 * P.N, dtype=np.uint64))      # slice out of range
    with pytest.raises((S.B200PirError, ValueError)):
        S.fold_ciphertexts(G, np.zeros(3 * 2 * P.N, dtype=np.uint64), np.zeros(1, dtype=np.uint64), np.zeros(1, dtype=np.uint64))
    with pytest.raises(S.B200PirError):
        S.Params(device=99, **P.kw)
    with pytest.raises(S.B200PirError):
        S.Database.from_words(G, np.zeros(17, dtype=np.uint64))
    # short buffers are refused by the host mirror (the C ABI, like the Rust slices it stands for, carries no lengths there)
    with pytest.raises(ValueError):
        S.PublicParameters(G, pp["pack"][:-1], pp["left"], pp["right"], pp["conv"])
    with pytest.raises(ValueError):
        S.process_query(G, gpp, S.Query(ct=np.zeros(2 * P.N - 1, dtype=np.uint64)), gdb)
    with pytest.raises(ValueError):
        S.pack(G, gpp, np.zeros(5, dtype=np.uint64))
    # gadget dimension 2 = 29-bit digits, above q_n: outside the transforms' input range, rejected (no reference parameter set uses it)
    with pytest.raises(S.B200PirError) as ei:
        S.Params(**dict(P.kw, t_gsw=2))
    assert ei.value.code == -4          # B200PIR_E_UNSUPPORTED


# ------------------------------------------------------------------ DoublePIR
@pytest.mark.parametrize("rows,cols", [(43, 37), (64, 1366), (29, 256), (1000, 5)])
def test_dpir_matvec_matches_oracle(rows, cols):
    import sdk_b200.doublepir as D
    rng = np.random.default_rng(rows * 131 + cols)
    a = rng.integers(0, 2**30, rows * cols, dtype=np.uint32)
    b = rng.integers(0, 2**32, 3 * cols, dtype=np.uint32)
    m = D.PackedMatrix(a, rows, cols)
    ref = O.dpir_matvec_packed(a, b, rows, cols)
    assert np.array_equal(D.matrix_mul_vec_packed(m, b), ref)
    import torch
    from sdk_b200._lib import LIB, check
    db_ = torch.from_numpy(b.view(np.int32)).cuda()
    for variant in (0, 1, 2, 4):
        do = torch.zeros(rows, dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        check(LIB.b200pir_dpir_matvec_packed_dev(m._h, db_.data_ptr(), do.data_ptr(), variant))
        D.matrix_mul_vec_packed(m, b)      # host call on the same (library-owned) stream: synchronises it
        assert np.array_equal(do.cpu().numpy().view(np.uint32), ref), variant
    m.close()


# ------------------------------------------------------------------ C++ host mirror (include/b200pir.hpp)
def test_cpp_host_mirror_matches_python_path(tmp_path):
    import os
    import subprocess
    S = _gpu()
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = str(tmp_path / "host_mirror_smoke")
    subprocess.check_call(["/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++", "-std=c++17", "-O2", "-o", exe,
                           os.path.join(root, "tests", "cpp", "host_mirror_smoke.cpp"), "-L" + os.path.join(root, "sdk_b200"),
                           "-lb200pir", "-Wl,-rpath," + os.path.join(root, "sdk_b200")])
    size, h_cpp = subprocess.check_output([exe], text=True).split()
    # same xorshift64 stream on the Python side
    state = [88172645463325252]
    M = (1 << 64) - 1

    def nxt():
        s = state[0]
        s ^= (s << 13) & M
        s ^= s >> 7
        s ^= (s << 17) & M
        state[0] = s
        return s

    def ntt_mat(polys):
        v = np.empty(polys * 4096, dtype=np.uint64)
        for i in range(polys):
            v[i * 4096:i * 4096 + 2048] = [nxt() % Q0 for _ in range(2048)]
            v[i * 4096 + 2048:(i + 1) * 4096] = [nxt() % Q1 for _ in range(2048)]
        return v

    kw = dict(O.PARAM_SETS["T"])
    G = S.Params(**kw)
    pack, left, right, conv = ntt_mat(2 * 3 * 4), ntt_mat(7 * 2 * 8), ntt_mat(5 * 2 * 8), ntt_mat(2 * 8)
    gpp = S.PublicParameters(G, pack, left, right, conv)
    gdb = S.Database(G)
    gdb.fill_synthetic(SEED_DB)
    ct = np.array([nxt() % (Q0 * Q1) for _ in range(4096)], dtype=np.uint64)
    resp = S.process_query(G, gpp, S.Query(ct=ct), gdb)
    h = 1469598103934665603
    for b in resp.tobytes():
        h = ((h ^ b) * 1099511628211) & M
    assert int(size) == resp.size and int(h_cpp) == h
    # and the oracle agrees on the same synthetic inputs
    P = O.Params(**kw)
    ref = P.process_query(dict(pack=pack, left=left, right=right, conv=conv), dict(ct=ct), P.generate_db(SEED_DB))
    assert np.array_equal(resp, ref)


# ------------------------------------------------------------------ multi-GPU composition, emulated on one GPU
@pytest.mark.parametrize("name,world", [("T0", 2), ("T0", 4), ("T", 4), ("T1", 2)])
def test_sharded_stages_equal_single_gpu(name, world):
    """stage A on every row shard (ii = s mod G) + concatenation (what the NCCL all-gather produces) + stage B
    == single-GPU process_query == oracle, byte for byte."""
    import ctypes as C
    import torch
    from sdk_b200._lib import LIB, check
    S, P, cl, pp, db, G, gdb, gpp = setup_case(name)
    idxs = [5, P.dim0 * P.num_per - 3]
    qs = np.concatenate([cl.generate_query(i)["ct"] for i in idxs])
    count = len(idxs)
    d_q = torch.from_numpy(qs.view(np.int64)).cuda()
    ct_words = 4 * P.N                                    # residue-form ciphertext, u32 words
    gathered = torch.zeros(world * count * P.slices * ct_words, dtype=torch.int32, device="cuda")
    slice_words = P.dim0 * P.num_per * P.N
    shards = []
    for s in range(world):
        sh = S.Database(G, shard_index=s, shard_count=world)
        for sl in range(P.slices):
            sh.upload_slice(sl, db[sl * slice_words:(sl + 1) * slice_words])
        shards.append(sh)
        part = gathered[s * count * P.slices * ct_words:(s + 1) * count * P.slices * ct_words]
        check(LIB.b200pir_query_stage_a_dev(G._h, sh._h, gpp._h, d_q.data_ptr(), count, part.data_ptr()))
    out = torch.zeros(count * G.response_bytes, dtype=torch.uint8, device="cuda")
    check(LIB.b200pir_query_stage_b_dev(G._h, gpp._h, gathered.data_ptr(), world, count, out.data_ptr()))
    G.synchronize()
    got = out.cpu().numpy().reshape(count, G.response_bytes)
    for k, i in enumerate(idxs):
        ref = P.process_query(pp, dict(ct=qs[k * 2 * P.N:(k + 1) * 2 * P.N]), db)
        assert np.array_equal(got[k], ref), (name, world, k)
        assert np.array_equal(cl.decode_response(got[k]), P.db_plain_item(SEED_DB, i))
    # the synthetic generator honours the shard mapping too
    sh2 = S.Database(G, shard_index=world - 1, shard_count=world)
    sh2.fill_synthetic(SEED_DB)
    rng = np.random.default_rng(8)
    v = (rng.integers(0, Q0, P.dim0 * 2 * P.N, dtype=np.uint64)
         | (rng.integers(0, Q1, P.dim0 * 2 * P.N, dtype=np.uint64) << np.uint64(32)))
    assert np.array_equal(S.multiply_reg_by_database(G, sh2, 0, v), S.multiply_reg_by_database(G, shards[-1], 0, v))
    for sh in shards + [sh2]:
        sh.close()


# ------------------------------------------------------------------ BASELINE configs[0]: the e2e parameter files, full size
@pytest.mark.parametrize("name", ["E1", "E0"])
def test_e2e_params_full_size_bytes_and_decode(name):
    """e2e-tests/params/v1.json / v0.json with every one of the 2^14 rows populated (4 GiB packed database):
    first-dimension words, folded ciphertexts and response bytes equal the oracle's; the decoded item equals the
    planted one (SURVEY 8d, config #1)."""
    S = _gpu()
    P = O.Params.named(name)
    cl = O.Client(P, 2024)
    pp = cl.generate_keys()
    db = P.generate_db(SEED_DB)
    G = S.Params(**P.kw)
    gdb = S.Database.from_words(G, db)
    gpp = S.PublicParameters(G, pp["pack"], pp.get("left"), pp.get("right"), pp.get("conv"))
    idx = 12345
    q = cl.generate_query(idx)
    ref, d = P.process_query(pp, q, db, dump=True)
    got = S.process_query(G, gpp, S.Query(ct=q["ct"]), gdb)
    assert np.array_equal(got, ref)
    assert np.array_equal(cl.decode_response(got), P.db_plain_item(SEED_DB, idx))
    slice_words = P.dim0 * P.num_per * P.N
    assert np.array_equal(S.multiply_reg_by_database(G, gdb, 0, d["v_firstdim"]), d["first_mult"])
    inter = P.from_ntt(d["first_mult"])
    S.fold_ciphertexts(G, inter, d["v_folding"])
    assert np.array_equal(inter[: 2 * P.N], d["folded"][: 2 * P.N])
    # the GPU-side generator builds the same 4 GiB database
    g2 = S.Database(G)
    g2.fill_synthetic(SEED_DB)
    assert np.array_equal(S.multiply_reg_by_database(G, g2, P.slices - 1, d["v_firstdim"]),
                          P.multiply_reg_by_database(db[(P.slices - 1) * slice_words:], d["v_firstdim"]))
    for h in (g2, gdb, gpp, G):
        h.close()


# ------------------------------------------------------------------ INT8 tensor-core first dimension (db format 1)
@pytest.mark.parametrize("name", CASES)
def test_imma_multiply_and_process_query_match_oracle(name):
    S, P, cl, pp, db, G, gdb, gpp = setup_case(name)
    fdb = S.Database.from_words(G, db, fmt=1)
    G.set_option("db_format", -1)
    rng = np.random.default_rng(14)
    v = (rng.integers(0, Q0, P.dim0 * 2 * P.N, dtype=np.uint64)
         | (rng.integers(0, Q1, P.dim0 * 2 * P.N, dtype=np.uint64) << np.uint64(32)))
    slice_words = P.dim0 * P.num_per * P.N
    for s in sorted({0, P.slices - 1}):
        ref = P.multiply_reg_by_database(db[s * slice_words:(s + 1) * slice_words], v)
        assert np.array_equal(S.multiply_reg_by_database(G, fdb, s, v), ref), (name, s)
    # worst-case operands: every limb 127-ish, checks the exactness bounds of the s32 accumulators
    w = np.uint64((Q0 - 1) | ((Q1 - 1) << 32))
    vmax = np.full(P.dim0 * 2 * P.N, w, dtype=np.uint64)
    assert np.array_equal(S.multiply_reg_by_database(G, fdb, 0, vmax), P.multiply_reg_by_database(db[:slice_words], vmax))
    # full pipeline, 11 queries: groups of 4+4+3 (batch 4) and 8+3 (batch 8: two column tiles)
    idxs = [0, 3, P.dim0 * P.num_per - 1, 17, 5, 9, 2, 11, 1, 30, 6]
    qs = np.concatenate([cl.generate_query(i)["ct"] for i in idxs])
    refs = [P.process_query(pp, dict(ct=qs[k * 2 * P.N:(k + 1) * 2 * P.N]), db) for k in range(len(idxs))]
    # imma_variant 0 = cp.async-pipelined 8-query kernel (default), 1 = load-then-use kernel
    # batch 16: one pass of 11 queries on the four-column-tile kernel (third tile partly, fourth tile entirely padding)
    for group, variant in ((4, 0), (8, 0), (8, 1), (16, 0)):
        G.set_option("batch", group)
        G.set_option("imma_variant", variant)
        out = S.process_query_batch(G, gpp, qs, fdb)
        for k in range(len(idxs)):
            assert np.array_equal(out[k], refs[k]), (name, group, variant, k)
    # 19 queries at batch 16: a full 16-query pass followed by a 3-query pass
    if name == "T":
        more = [7, 64, 100, 250, 12, 99, 180, 201]
        qs2 = np.concatenate([qs] + [cl.generate_query(i)["ct"] for i in more])
        out = S.process_query_batch(G, gpp, qs2, fdb)
        for k in range(len(idxs)):
            assert np.array_equal(out[k], refs[k]), (name, "19", k)
        for k, i in enumerate(more):
            kk = len(idxs) + k
            assert np.array_equal(out[kk], P.process_query(pp, dict(ct=qs2[kk * 2 * P.N:(kk + 1) * 2 * P.N]), db)), (name, "19", kk)
    G.set_option("batch", 16)
    G.set_option("imma_variant", 0)
    # synthetic generator and item upsert in fragment order
    f2 = S.Database(G, fmt=1)
    f2.fill_synthetic(SEED_DB)
    assert np.array_equal(S.multiply_reg_by_database(G, f2, P.slices - 1, v), S.multiply_reg_by_database(G, fdb, P.slices - 1, v))
    f3 = S.Database(G, fmt=1)
    G.set_option("db_format", -1)
    sl = db[:slice_words].reshape(P.N, P.num_per, P.dim0)
    items = [0, 5, P.dim0 * P.num_per - 1, 33 % (P.dim0 * P.num_per)]
    sparse = np.zeros_like(sl)
    for it in items:
        ii, j = it % P.num_per, it // P.num_per
        f3.upsert_item(0, it, np.ascontiguousarray(sl[:, ii, j]))
        sparse[:, ii, j] = sl[:, ii, j]
    assert np.array_equal(S.multiply_reg_by_database(G, f3, 0, v), P.multiply_reg_by_database(sparse.reshape(-1), v))
    for h in (fdb, f2, f3):
        h.close()


def test_imma_multiply_many_tiles_long_k():
    # dim0 = 1024 (32 k-steps, accumulators near their exactness bound), 64 rows (4 row tiles over the warps), max operands
    S = _gpu()
    kw = dict(O.PARAM_SETS["T"])
    kw.update(nu_1=10, nu_2=6, n=1, db_item_size=2048)
    P = O.Params(**kw)
    G = S.Params(**kw)
    w = np.uint64((Q0 - 1) | ((Q1 - 1) << 32))
    rng = np.random.default_rng(15)
    dbw = np.full(P.dim0 * P.num_per * P.N, w, dtype=np.uint64)
    dbw[::5] = rng.integers(0, Q0, dbw[::5].size, dtype=np.uint64) | (rng.integers(0, Q1, dbw[::5].size, dtype=np.uint64) << np.uint64(32))
    v = np.full(P.dim0 * 2 * P.N, w, dtype=np.uint64)
    v[::3] = rng.integers(0, Q0, v[::3].size, dtype=np.uint64) | (rng.integers(0, Q1, v[::3].size, dtype=np.uint64) << np.uint64(32))
    fdb = S.Database.from_words(G, dbw, fmt=1)
    assert np.array_equal(S.multiply_reg_by_database(G, fdb, 0, v), P.multiply_reg_by_database(dbw, v))
    fdb.close()
    G.close()


@pytest.mark.parametrize("name,world", [("T0", 2), ("T1", 4), ("T", 2)])
def test_three_phase_flow_with_tile_images_equals_oracle(name, world):
    """bench.py's N>1 flow on format-2 databases: every "rank" expands its queries straight into an operand tile image (one image per
    rank), the images are concatenated (the copy-engine pushes), every rank multiplies from the images of ALL ranks on its row
    shard and folds, survivors are concatenated, each rank finishes its own queries.  Responses == oracle bytes."""
    import torch
    from sdk_b200._lib import LIB, check
    S, P, cl, pp, db, G, gdb, gpp = setup_case(name)
    per_rank = 3
    total = per_rank * world
    idxs = [(11 * k + 5) % (P.dim0 * P.num_per) for k in range(total)]
    qs = np.concatenate([cl.generate_query(i)["ct"] for i in idxs])
    d_q = torch.from_numpy(qs.view(np.int64)).cuda()
    img_bytes = int(LIB.b200pir_query_image_bytes(G._h))
    fold_words = P.nu_2 * 2 * 2 * P.t_gsw * 2 * P.N
    ct_words = 4 * P.N
    images = torch.zeros(world * img_bytes, dtype=torch.uint8, device="cuda")
    vf = torch.zeros(total * fold_words, dtype=torch.int32, device="cuda")
    for r in range(world):
        check(LIB.b200pir_expand_queries_images_dev(G._h, gpp._h, d_q.data_ptr() + r * per_rank * 2 * P.N * 8, per_rank,
                                                    images.data_ptr() + r * img_bytes, vf.data_ptr() + r * per_rank * fold_words * 4))
    gathered = torch.zeros(world * total * P.slices * ct_words, dtype=torch.int32, device="cuda")
    slice_words = P.dim0 * P.num_per * P.N
    shards = []
    for r in range(world):
        sh = S.Database(G, shard_index=r, shard_count=world, fmt=2)
        for sl in range(P.slices):
            sh.upload_slice(sl, db[sl * slice_words:(sl + 1) * slice_words])
        shards.append(sh)
        check(LIB.b200pir_first_dim_fold_images_dev(G._h, sh._h, images.data_ptr(), world, per_rank, vf.data_ptr(),
                                                    gathered.data_ptr() + r * total * P.slices * ct_words * 4))
    out = torch.zeros(total * G.response_bytes, dtype=torch.uint8, device="cuda")
    for r in range(world):
        check(LIB.b200pir_finish_queries_dev(G._h, gpp._h, gathered.data_ptr(), world, total, r * per_rank, per_rank,
                                             vf.data_ptr() + r * per_rank * fold_words * 4,
                                             out.data_ptr() + r * per_rank * G.response_bytes))
    G.synchronize()
    got = out.cpu().numpy().reshape(total, G.response_bytes)
    for k, i in enumerate(idxs):
        ref = P.process_query(pp, dict(ct=qs[k * 2 * P.N:(k + 1) * 2 * P.N]), db)
        assert np.array_equal(got[k], ref), (name, world, k)
    for sh in shards:
        sh.close()


@pytest.mark.parametrize("name,world,fmt", [("T0", 2, 1), ("T0", 4, 0), ("T1", 2, 1), ("T0", 2, 2), ("T1", 2, 2)])
def test_three_phase_multi_gpu_flow_equals_oracle(name, world, fmt):
    """bench.py's N>1 flow on one GPU: every "rank" expands its own queries, expanded queries are concatenated
    (all-gather), every rank runs first dimension + local fold for ALL queries on its row shard, survivors are
    concatenated (all-gather), each rank finishes its own queries.  Responses == oracle bytes."""
    import torch
    from sdk_b200._lib import LIB, check
    S, P, cl, pp, db, G, gdb, gpp = setup_case(name)
    per_rank = 2
    total = per_rank * world
    idxs = [(7 * k + 3) % (P.dim0 * P.num_per) for k in range(total)]
    qs = np.concatenate([cl.generate_query(i)["ct"] for i in idxs])
    d_q = torch.from_numpy(qs.view(np.int64)).cuda()
    qexp_words = P.dim0 * P.N * 4
    fold_words = P.nu_2 * 2 * 2 * P.t_gsw * 2 * P.N
    ct_words = 4 * P.N
    qexp = torch.zeros(total * qexp_words, dtype=torch.int32, device="cuda")
    vf = torch.zeros(total * fold_words, dtype=torch.int32, device="cuda")
    for r in range(world):          # phase 1 on every rank, results land where the all-gather would put them
        check(LIB.b200pir_expand_queries_dev(G._h, gpp._h, d_q.data_ptr() + r * per_rank * 2 * P.N * 8, per_rank,
                                             qexp.data_ptr() + r * per_rank * qexp_words * 4,
                                             vf.data_ptr() + r * per_rank * fold_words * 4))
    gathered = torch.zeros(world * total * P.slices * ct_words, dtype=torch.int32, device="cuda")
    slice_words = P.dim0 * P.num_per * P.N
    shards = []
    for r in range(world):          # phase 2
        sh = S.Database(G, shard_index=r, shard_count=world, fmt=fmt)
        for sl in range(P.slices):
            sh.upload_slice(sl, db[sl * slice_words:(sl + 1) * slice_words])
        shards.append(sh)
        check(LIB.b200pir_first_dim_fold_dev(G._h, sh._h, qexp.data_ptr(), vf.data_ptr(), total,
                                             gathered.data_ptr() + r * total * P.slices * ct_words * 4))
    G.set_option("db_format", -1)
    out = torch.zeros(total * G.response_bytes, dtype=torch.uint8, device="cuda")
    for r in range(world):          # phase 3
        check(LIB.b200pir_finish_queries_dev(G._h, gpp._h, gathered.data_ptr(), world, total, r * per_rank, per_rank,
                                             vf.data_ptr() + r * per_rank * fold_words * 4,
                                             out.data_ptr() + r * per_rank * G.response_bytes))
    G.synchronize()
    got = out.cpu().numpy().reshape(total, G.response_bytes)
    for k, i in enumerate(idxs):
        ref = P.process_query(pp, dict(ct=qs[k * 2 * P.N:(k + 1) * 2 * P.N]), db)
        assert np.array_equal(got[k], ref), (name, world, k)
    for sh in shards:
        sh.close()


# ------------------------------------------------------------------ DoublePIR offline setup (doublepir.rs:76-108)
@pytest.mark.parametrize("rows,kdim,cols", [(128, 32, 128), (45, 70, 33), (300, 257, 1024), (129, 1, 5)])
def test_dpir_matmul_limb_gemm_matches_oracle(rows, kdim, cols):
    """`&Matrix * &Matrix` (matrix/ops.rs:169-191) on the wgmma limb GEMM: small signed left operand (centred mod p, and the
    extremes -2^15 / 2^15 - 1), full 32-bit right operand including 0xffffffff; ragged shapes (zero padded tiles)."""
    import sdk_b200.doublepir as D
    rng = np.random.default_rng(rows * 7 + kdim)
    a = (rng.integers(0, 929, (rows, kdim)).astype(np.int64) - 464).astype(np.uint32)
    a[0, 0] = np.uint32(2**32 - 32768)
    a[-1, -1] = 32767
    b = rng.integers(0, 2**32, (kdim, cols), dtype=np.uint64).astype(np.uint32)
    b[0, 0] = 0xFFFFFFFF
    assert np.array_equal(D.matmul(a, b), O.dpir_mul(a, b, rows, kdim, cols))
    with pytest.raises(D.B200PirError):
        bad = a.copy()
        bad[0, 0] = 40000
        D.matmul(bad, b)


@pytest.mark.parametrize("l,m,n,p,delta,x", [(24, 20, 8, 929, 4, 2), (256, 192, 64, 552, 4, 1), (96, 130, 1024, 1024, 4, 3)])
def test_dpir_setup_matches_oracle(l, m, n, p, delta, x):
    """setup(): hint h_2 and the three server-state matrices (squished database, squished expanded h_1, padded transposed a_2)
    == the oracle's restatement, word for word."""
    import sdk_b200.doublepir as D
    rng = np.random.default_rng(l + m + n)
    db = (rng.integers(0, p, (l, m)).astype(np.int64) - p // 2).astype(np.uint32)
    a1 = rng.integers(0, 2**32, (m, n), dtype=np.uint64).astype(np.uint32)
    a2 = rng.integers(0, 2**32, (l // x, n), dtype=np.uint64).astype(np.uint32)
    ref = O.dpir_setup(db, l, m, a1, n, a2, p, delta, x)
    got = D.setup(db, a1, a2, p, delta, x)
    assert np.array_equal(got["h2"], ref["h2"])
    assert np.array_equal(got["db_squished"], ref["db_sq"])
    assert np.array_equal(got["h1_squished"], ref["h1_sq"])
    assert np.array_equal(got["a2_t"], ref["a2_t"])


# ------------------------------------------------------------------ /write path: raw bucket bytes -> HBM (lib/server db/loading.rs)
@pytest.mark.parametrize("fmt", [0, 1, 2])
def test_update_item_raw_bytes_roundtrip(fmt):
    """update_item_raw (loading.rs:317-359) on the GPU == oracle's packed item polynomials, and a private read of the
    written items returns the written bytes (what e2e-tests/tests/simple.ts checks through the HTTP server)."""
    S, P, cl, pp, db, G, gdb, gpp = setup_case("T")
    rng = np.random.default_rng(21)
    wdb = S.Database(G, fmt=fmt)
    G.set_option("db_format", -1)
    sparse = np.zeros((P.slices, P.N, P.num_per, P.dim0), dtype=np.uint64)
    written = {}
    for idx, nbytes in ((7, P.db_item_size), (200, 100), (P.dim0 * P.num_per - 1, 1), (31, 0)):
        data = rng.integers(0, 256, nbytes, dtype=np.uint8)
        wdb.update_item_raw(idx, data)
        polys = P.update_item_raw(data).reshape(P.slices, P.N)
        sparse[:, :, idx % P.num_per, idx // P.num_per] = polys
        written[idx] = data
    v = (rng.integers(0, Q0, P.dim0 * 2 * P.N, dtype=np.uint64)
         | (rng.integers(0, Q1, P.dim0 * 2 * P.N, dtype=np.uint64) << np.uint64(32)))
    for s in range(P.slices):
        assert np.array_equal(S.multiply_reg_by_database(G, wdb, s, v),
                              P.multiply_reg_by_database(np.ascontiguousarray(sparse[s]).reshape(-1), v))
    pt_len = P.bytes_per_chunk
    for idx, data in written.items():
        q = cl.generate_query(idx)
        resp = S.process_query(G, gpp, S.Query(ct=q["ct"]), wdb)
        dec = cl.decode_response(resp).reshape(P.slices, P.N)        # (instance*n + trial/n, trial%n) row-major == slice order
        got = dec[:, :pt_len].astype(np.uint8).reshape(-1)
        exp = np.zeros(P.slices * pt_len, dtype=np.uint8)
        exp[: data.size] = data
        assert np.array_equal(got, exp), idx
    with pytest.raises(S.B200PirError):
        wdb.update_item_raw(0, np.zeros(P.slices * pt_len + 1, dtype=np.uint8))      # InvalidLength (loading.rs:308-310)
    with pytest.raises(S.B200PirError):
        wdb.update_item_raw(P.dim0 * P.num_per, np.zeros(4, dtype=np.uint8))         # bad db idx (loading.rs:333-340)
    wdb.close()


# ------------------------------------------------------------------ degenerate second dimension (server.rs:554-577, :394-396)
@pytest.mark.parametrize("nu_2", [0, 1])
@pytest.mark.parametrize("fmt", [0, 1, 2])
def test_small_second_dimension(nu_2, fmt):
    S = _gpu()
    kw = dict(O.PARAM_SETS["T"])
    kw.update(nu_2=nu_2)
    P = O.Params(**kw)
    cl = O.Client(P, 77)
    pp = cl.generate_keys()
    db = P.generate_db(SEED_DB)
    G = S.Params(**kw)
    gdb = S.Database.from_words(G, db, fmt=fmt)
    gpp = S.PublicParameters(G, pp["pack"], pp.get("left"), pp.get("right"), pp.get("conv"))
    for idx in (0, P.dim0 * P.num_per - 1, 17):
        q = cl.generate_query(idx)
        ref = P.process_query(pp, q, db)
        got = S.process_query(G, gpp, S.Query(ct=q["ct"]), gdb)
        assert np.array_equal(got, ref), (nu_2, fmt, idx)
        assert np.array_equal(cl.decode_response(got), P.db_plain_item(SEED_DB, idx))
    for h in (gdb, gpp, G):
        h.close()


# ------------------------------------------------------------------ DoublePIR answer() tail
def test_dpir_answer_matches_oracle():
    import sdk_b200.doublepir as D
    rng = np.random.default_rng(31)
    L, cols = 96, 50                   # database: 96 rows x 50 packed words (150 Z_p columns)
    p, delta, x, ne = 991, 4, 2, 4     # transpose_expand: a_1 -> (1*4*2) x ceil(48/3) = 8 x 16
    db = rng.integers(0, 2**30, L * cols, dtype=np.uint32)
    r1, c1 = delta * x, (L // x + 2) // 3
    h_rows = 20
    h_1 = rng.integers(0, 2**30, h_rows * c1, dtype=np.uint32)
    a2_rows, a2_cols = 10, 3 * c1
    a2t = rng.integers(0, 2**32, a2_rows * a2_cols, dtype=np.uint32)
    queries = []
    for _ in range(2):
        q = [rng.integers(0, 2**32, 3 * cols, dtype=np.uint32)]
        q += [rng.integers(0, 2**32, 3 * c1, dtype=np.uint32) for _ in range(ne // x)]
        queries.append(q)
    ref = O.dpir_answer(db, L, cols, queries, h_1, h_rows, c1, a2t, a2_rows, a2_cols, p, delta, x, ne)
    m = D.PackedMatrix(db, L, cols)
    got = D.answer(m, queries, (h_1, h_rows, c1), (a2t, a2_rows, a2_cols), p, delta, x, ne)
    assert len(got) == len(ref) == 1 + 2 * 2 * (ne // x)
    for g, r in zip(got, ref):
        assert np.array_equal(g, r)
    # stand-alone pieces on awkward shapes
    a = rng.integers(0, 2**32, 35 * 3, dtype=np.uint32)
    out, orows, ocols = D.transpose_expand_concat_cols_squish(a, 35, 3, 1000, 3, 5)
    ref2, rr, rc = O.dpir_transpose_expand_concat_cols_squish(a, 35, 3, 1000, 3, 5)
    assert (orows, ocols) == (rr, rc) and np.array_equal(out, ref2)
    m.close()


# ------------------------------------------------------------------ wire formats (client.rs:198-329)
@pytest.mark.parametrize("name", CASES)
def test_wire_formats_deserialize_and_process(name):
    """PublicParameters::deserialize / Query::deserialize on the GPU (ChaCha20 first rows regenerated from the seed)
    against the oracle's restatement, then process_query over the serialized bytes."""
    S, P, _, _, db, G, gdb, _ = setup_case(name)
    cl = O.Client(P, 4321)
    pp = cl.generate_keys()
    ppb = cl.pp_bytes()
    assert ppb.size == G.setup_bytes
    gpp = S.PublicParameters.deserialize(G, ppb)
    idxs = [3, P.dim0 * P.num_per - 1, 100 % (P.dim0 * P.num_per)]
    blobs = []
    for idx in idxs:
        q = cl.generate_query(idx)
        qb = cl.query_bytes()
        assert qb.size == G.query_bytes
        got_ct = S.Query.deserialize(G, qb).ct
        assert np.array_equal(got_ct, P.query_deserialize(qb))
        assert np.array_equal(got_ct, q["ct"])
        blobs.append((qb, q))
    out = S.process_query_bytes(G, gpp, np.concatenate([b for b, _ in blobs]), gdb)
    for k, (qb, q) in enumerate(blobs):
        ref = P.process_query(pp, q, db)
        assert np.array_equal(out[k], ref), (name, k)
        assert np.array_equal(cl.decode_response(out[k]), P.db_plain_item(SEED_DB, idxs[k]))
    # deserialized parameters == parameters uploaded as arrays
    gpp2 = S.PublicParameters(G, pp["pack"], pp.get("left"), pp.get("right"), pp.get("conv"))
    assert np.array_equal(S.process_query(G, gpp2, S.Query(ct=blobs[0][1]["ct"]), gdb), out[0])
    with pytest.raises(S.B200PirError):
        S.PublicParameters.deserialize(G, ppb[:-8])
    with pytest.raises(S.B200PirError):
        S.Query.deserialize(G, blobs[0][0][:-1])
    gpp.close()
    gpp2.close()


def test_queries_of_different_clients_share_one_pass():
    """lib/server serves each request with the public parameters of ITS client (bin/server.rs:113-117).  Two clients with
    different keys, their queries interleaved in one b200pir_process_queries call: every response == the oracle's for that
    client, and decodes under that client's secret key."""
    S, P, cl_a, pp_a, db, G, gdb, gpp_a = setup_case("T")
    cl_b = O.Client(P, 777)
    pp_b = cl_b.generate_keys()
    gpp_b = S.PublicParameters(G, pp_b["pack"], pp_b["left"], pp_b["right"], pp_b["conv"])
    plan = [(cl_a, pp_a, gpp_a, 5), (cl_b, pp_b, gpp_b, 9), (cl_b, pp_b, gpp_b, 200), (cl_a, pp_a, gpp_a, 77), (cl_b, pp_b, gpp_b, 0)]
    qs = [cl.generate_query(idx)["ct"] for cl, _, _, idx in plan]
    out = S.process_queries(G, [g for _, _, g, _ in plan], qs, gdb)
    for k, (cl, pp, _, idx) in enumerate(plan):
        assert np.array_equal(out[k], P.process_query(pp, dict(ct=qs[k]), db)), k
        assert np.array_equal(cl.decode_response(out[k]), P.db_plain_item(SEED_DB, idx))
    gpp_b.close()


def test_direct_upload_queries_over_the_wire():
    """Query::deserialize's direct-upload branch (client.rs:316-327) on the GPU: the seed-derived halves of v_buf and the
    first rows of v_ct are regenerated from the 32-byte seed; response bytes == the oracle's process_query on the generated
    (never serialized) query, for a batch of three queries in one call; public parameters arrive serialized too
    (the handler's body is setup || query, bin/server.rs:122-137)."""
    S, P, _, _, db, G, gdb, _ = setup_case("T", expand=False)
    cl = O.Client(P, 99)
    pp = cl.generate_keys()
    gpp = S.PublicParameters.deserialize(G, cl.pp_bytes())
    idxs = [0, 77, P.dim0 * P.num_per - 1]
    blobs, refs = [], []
    for idx in idxs:
        q = cl.generate_query(idx)
        qb = cl.query_bytes()
        assert qb.size == G.query_bytes
        blobs.append(qb)
        refs.append(P.process_query(pp, q, db))
    out = S.process_query_bytes(G, gpp, np.concatenate(blobs), gdb)
    for k, idx in enumerate(idxs):
        assert np.array_equal(out[k], refs[k]), k
        assert np.array_equal(cl.decode_response(out[k]), P.db_plain_item(SEED_DB, idx))
    with pytest.raises((S.B200PirError, ValueError)):
        S.process_query_bytes(G, gpp, blobs[0][:-8], gdb)
    gpp.close()


# ------------------------------------------------------------------ golden fixtures (tests/golden/spiral_golden.json)
@pytest.mark.parametrize("case", ["T_expand", "T1_expand", "T0_expand", "T_direct"])
def test_cuda_path_reproduces_golden_fixtures(case):
    """Response bytes of the CUDA path == the frozen fixtures (sha256), for both database layouts."""
    import json
    import os
    import golden_cases as GC
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "spiral_golden.json")) as f:
        gold = json.load(f)["cases"][case]
    S = _gpu()
    P, cl, pp, db, queries = GC.build_case(case)
    expand = GC.GOLDEN_CASES[case][1]
    assert GC.sha(db) == gold["db_sha256"]
    G = S.Params(expand_queries=expand, **P.kw)
    gpp = S.PublicParameters(G, pp["pack"], pp.get("left"), pp.get("right"), pp.get("conv"))
    for fmt in (2, 1, 0):
        gdb = S.Database.from_words(G, db, fmt=fmt)
        for (idx, q), g in zip(queries, gold["queries"]):
            assert idx == g["idx"]
            query = S.Query(ct=q["ct"]) if expand else S.Query(v_buf=q["v_buf"], v_ct=q["v_ct"])
            got = S.process_query(G, gpp, query, gdb)
            assert GC.sha(got) == g["response_sha256"], (case, fmt, idx)
            assert [int(x) for x in got[:16]] == g["response_head"]
        gdb.close()
    gpp.close()
    G.close()


# ------------------------------------------------------------------ preprocessed database file (server.rs:373-386)
@pytest.mark.parametrize("fmt", [0, 1, 2])
def test_database_loaded_from_file_equals_uploaded_database(fmt, tmp_path):
    S, P, cl, pp, db, G, gdb, gpp = setup_case("T")
    path = tmp_path / "db.bin"
    db.tofile(str(path))                                   # native-endian u64 stream, what load_file reads
    fdb = S.Database.from_file(G, path, fmt=fmt)
    G.set_option("db_format", -1)
    rng = np.random.default_rng(31)
    v = (rng.integers(0, Q0, P.dim0 * 2 * P.N, dtype=np.uint64)
         | (rng.integers(0, Q1, P.dim0 * 2 * P.N, dtype=np.uint64) << np.uint64(32)))
    slice_words = P.dim0 * P.num_per * P.N
    for s in sorted({0, P.slices - 1}):
        ref = P.multiply_reg_by_database(db[s * slice_words:(s + 1) * slice_words], v)
        assert np.array_equal(S.multiply_reg_by_database(G, fdb, s, v), ref), (fmt, s)
    q = cl.generate_query(200)
    assert np.array_equal(S.process_query(G, gpp, S.Query(ct=q["ct"]), fdb), P.process_query(pp, q, db))
    fdb.close()
    short = tmp_path / "short.bin"
    db[:-1].tofile(str(short))
    with pytest.raises(S.B200PirError):
        S.Database.from_file(G, short, fmt=fmt)
    with pytest.raises(S.B200PirError):
        S.Database.from_file(G, tmp_path / "missing.bin", fmt=fmt)
    G.set_option("db_format", -1)


# ------------------------------------------------------------------ raw database file (load_db_from_seek, server.rs:277-357)
@pytest.mark.parametrize("fmt,shrink", [(1, 0), (0, 2), (2, 1)])
def test_database_loaded_from_raw_file_matches_oracle(fmt, shrink, tmp_path):
    """shrink = 2: db_item_size not a multiple of the chunk count, so an item's last chunk reads into the next item."""
    S = _gpu()
    kw = dict(O.PARAM_SETS["T"])
    kw["db_item_size"] -= shrink
    P = O.Params(**kw)
    G = S.Params(**kw)
    rng = np.random.default_rng(33)
    total = P.dim0 * P.num_per
    raw = rng.integers(0, 256, total * P.db_item_size - 3000, dtype=np.uint8)        # truncated last item
    path = tmp_path / "raw.bin"
    raw.tofile(str(path))
    ref_db = P.load_db_from_bytes(raw)
    gdb = S.Database.from_raw_file(G, path, fmt=fmt)
    G.set_option("db_format", -1)
    v = (rng.integers(0, Q0, P.dim0 * 2 * P.N, dtype=np.uint64)
         | (rng.integers(0, Q1, P.dim0 * 2 * P.N, dtype=np.uint64) << np.uint64(32)))
    slice_words = P.dim0 * P.num_per * P.N
    for s in range(P.slices):
        ref = P.multiply_reg_by_database(ref_db[s * slice_words:(s + 1) * slice_words], v)
        assert np.array_equal(S.multiply_reg_by_database(G, gdb, s, v), ref), (fmt, shrink, s)
    gdb.close()
    G.close()
