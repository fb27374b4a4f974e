"""Parity of the wgmma first dimension (database format 2, sdk_b200/csrc/tc5_kernels.cu) against the oracle.  Format 2 is
the default database format wherever the geometry fits."""
import numpy as np
import pytest

import oracle_lib as O
from test_gpu_parity import setup_case, SEED_DB, Q0, Q1

pytestmark = [pytest.mark.gpu]


@pytest.mark.parametrize("name", ["T", "T1", "T0"])
def test_tc5_multiply_matches_oracle(name):
    S, P, cl, pp, db, G, gdb, gpp = setup_case(name)
    tdb = S.Database.from_words(G, db, fmt=2)
    G.set_option("db_format", -1)
    rng = np.random.default_rng(21)
    v = (rng.integers(0, Q0, P.dim0 * 2 * P.N, dtype=np.uint64)
         | (rng.integers(0, Q1, P.dim0 * 2 * P.N, dtype=np.uint64) << np.uint64(32)))
    slice_words = P.dim0 * P.num_per * P.N
    for s in sorted({0, P.slices - 1}):
        ref = P.multiply_reg_by_database(db[s * slice_words:(s + 1) * slice_words], v)
        assert np.array_equal(S.multiply_reg_by_database(G, tdb, s, v), ref), (name, s)
    w = np.uint64((Q0 - 1) | ((Q1 - 1) << 32))
    vmax = np.full(P.dim0 * 2 * P.N, w, dtype=np.uint64)
    assert np.array_equal(S.multiply_reg_by_database(G, tdb, 0, vmax), P.multiply_reg_by_database(db[:slice_words], vmax))
    tdb.close()


def test_tc5_process_query_batches():
    S, P, cl, pp, db, G, gdb, gpp = setup_case("T")
    tdb = S.Database.from_words(G, db, fmt=2)
    G.set_option("db_format", -1)
    idxs = [0, 3, P.dim0 * P.num_per - 1, 17, 5, 9, 2, 11, 1, 30, 6, 7, 64, 100, 250, 12, 99, 180, 201]     # 16 + 3
    qs = np.concatenate([cl.generate_query(i)["ct"] for i in idxs])
    out = S.process_query_batch(G, gpp, qs, tdb)
    for k, i in enumerate(idxs):
        ref = P.process_query(pp, dict(ct=qs[k * 2 * P.N:(k + 1) * 2 * P.N]), db)
        assert np.array_equal(out[k], ref), k
        assert np.array_equal(cl.decode_response(out[k]), P.db_plain_item(SEED_DB, i))
    tdb.close()


def test_tc5_synthetic_and_upsert_equal_bulk_upload():
    S, P, cl, pp, db, G, gdb, gpp = setup_case("T")
    rng = np.random.default_rng(22)
    v = (rng.integers(0, Q0, P.dim0 * 2 * P.N, dtype=np.uint64)
         | (rng.integers(0, Q1, P.dim0 * 2 * P.N, dtype=np.uint64) << np.uint64(32)))
    t2 = S.Database(G, fmt=2)
    t2.fill_synthetic(SEED_DB)
    G.set_option("db_format", -1)
    assert np.array_equal(S.multiply_reg_by_database(G, t2, P.slices - 1, v), S.multiply_reg_by_database(G, gdb, P.slices - 1, v))
    slice_words = P.dim0 * P.num_per * P.N
    sl = db[:slice_words].reshape(P.N, P.num_per, P.dim0)
    t3 = S.Database(G, fmt=2)
    G.set_option("db_format", -1)
    items = [0, 5, P.dim0 * P.num_per - 1, 33 % (P.dim0 * P.num_per)]
    sparse = np.zeros_like(sl)
    for it in items:
        ii, j = it % P.num_per, it // P.num_per
        t3.upsert_item(0, it, np.ascontiguousarray(sl[:, ii, j]))
        sparse[:, ii, j] = sl[:, ii, j]
    assert np.array_equal(S.multiply_reg_by_database(G, t3, 0, v), P.multiply_reg_by_database(sparse.reshape(-1), v))
    t2.close()
    t3.close()


def test_tc5_long_k_many_tiles_worst_case():
    S, _, _, _, _, _, _, _ = setup_case("T")
    kw = dict(O.PARAM_SETS["T"])
    kw.update(n=1, db_item_size=2048)
    # dim0 = 1024: 32 k-steps, the largest accumulators the limb arithmetic allows (1024 x 127 x 127 < 2^24), a 128 KiB query
    # operand (single-buffered beside the ring); dim0 = 512: 16 k-steps, 128 rows = 4 row tiles, double-buffered operand
    for nu_1, nu_2 in ((10, 6), (9, 7)):
        kw.update(nu_1=nu_1, nu_2=nu_2)
        P = O.Params(**kw)
        G = S.Params(**kw)
        w = np.uint64((Q0 - 1) | ((Q1 - 1) << 32))
        rng = np.random.default_rng(23 + nu_1)
        dbw = np.full(P.dim0 * P.num_per * P.N, w, dtype=np.uint64)
        dbw[::5] = rng.integers(0, Q0, dbw[::5].size, dtype=np.uint64) | (rng.integers(0, Q1, dbw[::5].size, dtype=np.uint64) << np.uint64(32))
        v = np.full(P.dim0 * 2 * P.N, w, dtype=np.uint64)
        v[::3] = rng.integers(0, Q0, v[::3].size, dtype=np.uint64) | (rng.integers(0, Q1, v[::3].size, dtype=np.uint64) << np.uint64(32))
        tdb = S.Database.from_words(G, dbw, fmt=2)
        assert tdb.info()["format"] == 2
        assert np.array_equal(S.multiply_reg_by_database(G, tdb, 0, v), P.multiply_reg_by_database(dbw, v)), nu_1
        tdb.close()
        G.close()

