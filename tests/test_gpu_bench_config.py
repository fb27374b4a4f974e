"""The bench configuration itself (BASELINE.json configs[1]: S8 = 2^17 items x 8 KiB = 1 GiB of plaintext, 8 GiB in HBM,
nu_2 = 8: the 256-row fold tree, the 16-queries-per-pass first dimension) — size-independent property at full size: the
decoded response equals the planted plaintext, recomputed from the counter PRNG the GPU database generator uses
(the generator itself is checked against the oracle's at small size in test_gpu_parity.py).  S8's bytes, stage by stage and
end to end, are compared with the oracle's in test_gpu_deep_geometry_parity.py.  Also DoublePIR config #4 and the
NTT sweep of config #5 at full size against oracle samples (DoublePIR at 2^23 rows: the 2^24-row matrix, 91.7 GB, does not
fit an 80 GB H100)."""
import numpy as np
import pytest

import oracle_lib as O
from test_gpu_parity import _gpu, Q0, Q1

pytestmark = [pytest.mark.gpu]
SEED = 0xB1755


@pytest.fixture(scope="module")
def s8():
    S = _gpu()
    P = O.Params.named("S8")
    cl = O.Client(P, 5)
    pp = cl.generate_keys()
    G = S.Params(**P.kw)
    gdb = S.Database(G)
    gdb.fill_synthetic(SEED)
    gpp = S.PublicParameters(G, pp["pack"], pp.get("left"), pp.get("right"), pp.get("conv"))
    yield S, P, cl, G, gdb, gpp
    gpp.close()
    gdb.close()
    G.close()


def test_s8_default_layout_is_tcgen05(s8):
    S, P, cl, G, gdb, gpp = s8
    info = gdb.info()
    assert info["format"] == 2 and info["local_rows"] == P.num_per and info["hbm_bytes"] == 8 << 30


@pytest.mark.parametrize("idx", [0, 12345, (1 << 17) - 1])
def test_s8_single_query_decodes_to_planted_item(s8, idx):
    S, P, cl, G, gdb, gpp = s8
    resp = S.process_query(G, gpp, S.Query(ct=cl.generate_query(idx)["ct"]), gdb)
    assert np.array_equal(cl.decode_response(resp), P.db_plain_item(SEED, idx))


def test_s8_batch_of_16_decodes_and_equals_single_queries(s8):
    S, P, cl, G, gdb, gpp = s8
    n_items = P.dim0 * P.num_per
    idxs = [0, n_items - 1, 12345] + [(7919 * k + 31) % n_items for k in range(13)]
    qs = [cl.generate_query(i)["ct"] for i in idxs]
    out = S.process_query_batch(G, gpp, np.concatenate(qs), gdb)              # one pass of the 16-query kernel
    for k, i in enumerate(idxs):
        assert np.array_equal(cl.decode_response(out[k]), P.db_plain_item(SEED, i)), (k, i)
    for k in (0, 5, 15):                                                       # bytes: batched == alone
        assert np.array_equal(out[k], S.process_query(G, gpp, S.Query(ct=qs[k]), gdb)), k


def test_s8_every_layout_gives_the_same_bytes(s8):
    S, P, cl, G, gdb, gpp = s8
    q = S.Query(ct=cl.generate_query(4242)["ct"])
    ref = S.process_query(G, gpp, q, gdb)
    for fmt in (1, 0):
        other = S.Database(G, fmt=fmt)
        other.fill_synthetic(SEED)
        assert np.array_equal(S.process_query(G, gpp, q, other), ref), fmt
        other.close()


# ------------------------------------------------------------------ BASELINE config #4: DoublePIR 2^23 x 1366 packed words
def test_dpir_config4_full_size_against_oracle_row_sample():
    import sdk_b200.doublepir as D
    rows, cols = 1 << 23, 1366
    m = D.PackedMatrix(rows=rows, cols=cols, synthetic_seed=7)                # 45.8 GB, generated on the GPU
    rng = np.random.default_rng(11)
    b = rng.integers(0, 1 << 32, 3 * cols, dtype=np.uint64).astype(np.uint32)
    b[-2:] = 0                                                                 # append_zeros, doublepir.rs:131-134
    out = D.matrix_mul_vec_packed(m, b)
    assert out.size == rows
    sample = sorted(set(list(range(8)) + list(range(rows - 8, rows)) + list(range(0, rows, 1 << 12))))
    for i in sample:
        idx = np.arange(i * cols, (i + 1) * cols, dtype=np.uint64)
        z = np.uint64(7) + (idx + np.uint64(1)) * np.uint64(0x9E3779B97F4A7C15)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        z = z ^ (z >> np.uint64(31))
        a_row = (z & np.uint64(0x3FFFFFFF)).astype(np.uint32)                 # three 10-bit values per word
        ref = O.dpir_matvec_packed(np.ascontiguousarray(a_row), b, 1, cols)[0]
        assert out[i] == ref, i
    m.close()


# ------------------------------------------------------------------ BASELINE config #5: 2^16 polynomials per batch, both sizes
@pytest.mark.parametrize("poly_len", [2048, 4096])
def test_ntt_config5_batch_against_oracle_sample(s8, poly_len):
    import torch
    from sdk_b200._lib import LIB, check
    S, P, cl, G, gdb, gpp = s8
    count = 1 << 16
    rng = np.random.default_rng(poly_len)
    host = np.empty((count, 2, poly_len), dtype=np.uint32)
    host[:, 0, :] = rng.integers(0, Q0, (count, poly_len), dtype=np.uint32)
    host[:, 1, :] = rng.integers(0, Q1, (count, poly_len), dtype=np.uint32)
    d = torch.from_numpy(host.view(np.int32)).cuda()
    fn = LIB.b200pir_ntt32_dev if poly_len == 2048 else LIB.b200pir_ntt4096_dev
    check(fn(G._h, d.data_ptr(), count, 0))
    G.synchronize()
    fwd = d.cpu().numpy().view(np.uint32)
    sample = [0, 1, 777, count // 2, count - 1]
    for i in sample:
        ref = np.ascontiguousarray(host[i].astype(np.uint64).reshape(-1))
        if poly_len == 2048:
            ref = P.ntt_forward(ref)
        else:
            assert O.LIB.orc_ntt4096(O._p64(ref), 1, 0) == 0
        assert np.array_equal(fwd[i].astype(np.uint64).reshape(-1), ref), (poly_len, i)
    check(fn(G._h, d.data_ptr(), count, 1))
    G.synchronize()
    back = d.cpu().numpy().view(np.uint32)
    assert np.array_equal(back, host)                                          # round trip over the whole batch
