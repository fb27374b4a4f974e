"""The sparse server's fold (lib/server/src/compute/fold.rs:15-65: all-zero ciphertext shortcut) on the GPU, option
"sparse_fold" — against the oracle's restatement.  The default (dense, spiral-rs) fold is unaffected."""
import numpy as np
import pytest

import oracle_lib as O
from test_gpu_parity import setup_case, SEED_DB

pytestmark = [pytest.mark.gpu]


def test_stage_level_sparse_fold_matches_oracle():
    S, P, cl, pp, db, G, gdb, gpp = setup_case("T")
    q = cl.generate_query(5)
    _, vf = P.expand_query(pp, q["ct"])
    vfn = P.get_v_folding_neg(vf)
    rng = np.random.default_rng(8)
    num, dims = 4, 2                            # T has nu_2 = 2
    mat = 4 * P.t_gsw * P.W
    base = rng.integers(0, P.modulus, num * 2 * P.N, dtype=np.uint64).reshape(num, 2 * P.N)
    cases = {"first zero / second zero": (0, 3), "both operands of a pair zero": (1, 3), "no zero": ()}
    for name, zeros in cases.items():
        cts = base.copy()
        for z in zeros:
            cts[z] = 0
        G.set_option("sparse_fold", 1)
        try:
            got = cts.copy().reshape(-1)
            S.fold_ciphertexts(G, got, vf[: dims * mat], None)
        finally:
            G.set_option("sparse_fold", 0)
        ref = P.fold_ciphertexts(cts, vf[: dims * mat], vfn[: dims * mat], sparse=True)
        assert np.array_equal(got[: 2 * P.N], ref.reshape(-1)[: 2 * P.N]), name


@pytest.mark.parametrize("fmt", [1, 0, 2])
def test_process_query_on_sparse_database_matches_sparse_server(fmt):
    S, P, cl, pp, db, G, gdb, gpp = setup_case("T")
    sdb = db.reshape(P.slices, P.N, P.num_per, P.dim0).copy()
    sdb[:, :, 1::2, :] = 0                      # every odd second-dimension row empty
    sdb = sdb.reshape(-1)
    gs = S.Database.from_words(G, sdb, fmt=fmt)
    G.set_option("db_format", -1)
    idxs = [0, 14, P.num_per * 3 + 4, 7]        # the last one targets an empty row
    qs = np.concatenate([cl.generate_query(i)["ct"] for i in idxs])
    G.set_option("sparse_fold", 1)
    try:
        out = S.process_query_batch(G, gpp, qs, gs)
    finally:
        G.set_option("sparse_fold", 0)
    for k, i in enumerate(idxs):
        ref = P.process_query(pp, dict(ct=qs[k * 2 * P.N:(k + 1) * 2 * P.N]), sdb, sparse_fold=True)
        assert np.array_equal(out[k], ref), (fmt, k)
    dense = S.process_query_batch(G, gpp, qs, gs)
    assert not np.array_equal(dense[0], out[0])
    gs.close()
