"""DoublePIR's offline phase on the GPU from raw bytes: b200pir_dpir_load (load_data / load_data_fast -> init() -> setup()) and
b200pir_dpir_derive_from_seed, compared word for word with the oracle (tests/cpp/dpir_load_oracle.cpp), and decoded end to end with the
shared matrices derived from the reference's seeds, as a real DoublePirClient derives them."""
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


def oracle_load(prm, num_entries, bits, data, bits_format):
    """load_data (or load_data_fast) -> init() -> setup() on the oracle: (db layout, a_1, a_2, setup outputs, info)."""
    D = _D()
    info = L.dpir_db_info(num_entries, bits, prm["p"])
    delta = D.db_info(prm, num_entries, bits)["delta"]
    l, m, n, x = prm["l"], prm["m"], prm["n"], info["x"]
    db = L.dpir_load_data(data, bits_format, num_entries, bits, l, m, prm["p"])
    a_1 = L.dpir_derive_from_seed(m, n, D.SEED_A1)
    a_2 = L.dpir_derive_from_seed(l // x, n, D.SEED_A2)
    st = O.dpir_setup(db, l, m, a_1, n, a_2, prm["p"], delta, x)
    return db, a_1, a_2, st


def assert_load_equals(got, st):
    dbm, out, _ = got
    assert np.array_equal(dbm.download(), st["db_sq"])
    assert np.array_equal(out["h1_squished"], st["h1_sq"])
    assert np.array_equal(out["a2_t"], st["a2_t"])
    assert np.array_equal(out["h2"], st["h2"])


# ------------------------------------------------------------------ derivation
@pytest.mark.parametrize("rows,cols", [(65536, 1024), (29, 1024), (7, 3), (16385, 5), (1, 1)])
@pytest.mark.parametrize("which", [0, 1])
def test_derive_from_seed_equals_oracle(rows, cols, which):
    # (65536, 1024) = A_1 (4096 chunks); 29 x 1024 = A_2 at l = 29 (a partial chunk); 7 x 3 and 16385 x 5: partial last blocks
    D = _D()
    key = (D.SEED_A1, D.SEED_A2)[which]
    assert np.array_equal(D.derive_from_seed(rows, cols, key), L.dpir_derive_from_seed(rows, cols, key))


# ------------------------------------------------------------------ layout through load() at a small n
# (num_entries, bits, p, l, m, nbytes, data high): packing 9 with a partial last group; ne = 2 (p = 16, 8-bit entries);
# oversized bytes in 3-bit fields; ne = 2 at p = 512, x = 2; few entries in a mostly untouched matrix
SMALL = [(1000, 1, 512, 2, 64, 1000, 2), (300, 8, 16, 10, 64, 300, 256), (999, 3, 512, 6, 64, 999, 256),
         (130, 10, 512, 10, 32, 130, 256), (9, 1, 512, 3, 7, 9, 2)]


@pytest.mark.parametrize("bits_format", [False, True])
@pytest.mark.parametrize("num_entries,bits,p,l,m,nbytes,high", SMALL)
def test_load_small_equals_oracle(num_entries, bits, p, l, m, nbytes, high, bits_format):
    D = _D()
    rng = np.random.default_rng(num_entries + 17 * bits)
    nbytes = (nbytes + 7) // 8 if bits_format else nbytes
    data = rng.integers(0, 256 if bits_format else high, nbytes, dtype=np.uint8)
    prm = dict(n=64, l=l, m=m, logq=32, p=p)
    _, _, _, st = oracle_load(prm, num_entries, bits, data, bits_format)
    fmt = D.ENTRY_BITS if bits_format else D.ENTRY_BYTES
    got = D.load(prm, num_entries, bits, data, fmt)
    assert_load_equals(got, st)
    assert got[0].rows == l and got[0].cols == (m + 2) // 3
    got[0].close()


# ------------------------------------------------------------------ load() vs the oracle at the reference's shapes
_loaded = {}


def reference_shape(num_entries, bits, bits_format, seed):
    key = (num_entries, bits, bits_format, seed)
    if key not in _loaded:
        D = _D()
        rng = np.random.default_rng(seed)
        prm = E.pick_params(num_entries, bits, E.SEC_PARAM, E.LOGQ)
        nbytes = num_entries // 8 if bits_format else num_entries
        data = rng.integers(0, 256, nbytes, dtype=np.uint8)
        got = D.load(prm, num_entries, bits, data, D.ENTRY_BITS if bits_format else D.ENTRY_BYTES)
        _loaded[key] = (rng, prm, data, got)
    return _loaded[key]


@pytest.mark.parametrize("num_entries,bits,bits_format,shape", [(1 << 24, 1, True, (29, 512, 9, 1)),
                                                                 (1 << 20, 10, False, (32, 512, 0, 2))])
def test_load_equals_oracle_at_reference_shapes(num_entries, bits, bits_format, shape):
    rng, prm, data, got = reference_shape(num_entries, bits, bits_format, 1)
    info = got[2]
    assert (prm["l"], prm["p"], info["packing"], info["x"]) == shape and prm["m"] == 65536
    _, _, _, st = oracle_load(prm, num_entries, bits, data, bits_format)
    assert_load_equals(got, st)


def test_load_equals_host_setup_at_2_30_entries():
    # 2^30 one-bit entries: l = 1821.  The GEMMs are pinned elsewhere, so GPU setup() fed with the oracle's layout and
    # derived matrices isolates the new code at scale
    D = _D()
    num_entries = 1 << 30
    prm = E.pick_params(num_entries, 1, E.SEC_PARAM, E.LOGQ)
    assert (prm["l"], prm["m"], prm["p"]) == (1821, 65536, 512)
    data = np.random.default_rng(30).integers(0, 256, num_entries // 8, dtype=np.uint8)
    dbm, out, info = D.load(prm, num_entries, 1, data, D.ENTRY_BITS)
    db = L.dpir_load_data(data, True, num_entries, 1, prm["l"], prm["m"], prm["p"])
    a_1 = L.dpir_derive_from_seed(prm["m"], prm["n"], D.SEED_A1)
    a_2 = L.dpir_derive_from_seed(prm["l"], prm["n"], D.SEED_A2)
    want = D.setup(db, a_1, a_2, prm["p"], info["delta"], info["x"])
    del db
    assert np.array_equal(dbm.download(), want["db_squished"])
    for k in ("h1_squished", "a2_t", "h2"):
        assert np.array_equal(out[k], want[k]), k
    dbm.close()


# ------------------------------------------------------------------ end to end with the derived shared matrices
def _client_view(prm, got):
    D = _D()
    dbm, out, info = got
    info = dict(info, bits=1)
    a_1 = D.derive_from_seed(prm["m"], prm["n"], D.SEED_A1)
    a_2 = D.derive_from_seed(prm["l"] // info["x"], prm["n"], D.SEED_A2)
    return dbm, out, info, a_1, a_2


def _answer(dbm, out, prm, info, queries):
    n, delta, x = prm["n"], info["delta"], info["x"]
    h_1 = (out["h1_squished"].reshape(-1), n * delta * x, out["h1_squished"].shape[1])
    a2t = (out["a2_t"].reshape(-1), n, out["a2_t"].shape[1])
    return _D().answer(dbm, queries, h_1, a2t, prm["p"], delta, x, info["ne"])


def _bit(data, i):
    return (int(data[i >> 3]) >> (i & 7)) & 1


def test_simple_end_to_end_from_raw_bytes():
    # doublepir.rs:469-525 simple_end_to_end_test, as the reference runs it: shared matrices from SEEDS_SHORT
    num_entries = 1 << 24
    rng, prm, data, got = reference_shape(num_entries, 1, True, 1)
    dbm, out, info, a_1, a_2 = _client_view(prm, got)
    for i in [0, num_entries - 1] + [int(v) for v in rng.integers(0, num_entries, 3)]:
        client, qmsg = E.query(i, a_1, a_2, prm, info, rng)
        ans = _answer(dbm, out, prm, info, [qmsg])
        assert E.recover(i, out["h2"], qmsg, ans, a_2, client, prm, info) == _bit(data, i), i


def test_batched_end_to_end_from_raw_bytes():
    # doublepir.rs:526-606 batched_end_to_end_test: two queries, each from its own batch of rows
    num_entries = 1 << 24
    rng, prm, data, got = reference_shape(num_entries, 1, True, 1)
    dbm, out, info, a_1, a_2 = _client_view(prm, got)
    batch_sz = 14 * 65536 * 9
    i1 = int(rng.integers(0, batch_sz))
    idxs = sorted([i1, (i1 + batch_sz) % num_entries])
    qs = [E.query(i, a_1, a_2, prm, info, rng) for i in idxs]
    ans = _answer(dbm, out, prm, info, [q for _, q in qs])
    for b, (i, (client, qmsg)) in enumerate(zip(idxs, qs)):
        assert E.recover(i, out["h2"], qmsg, ans, a_2, client, prm, info, batch_index=b) == _bit(data, i), (b, i)


# ------------------------------------------------------------------ errors: a code, and no handle
def _load_rc(prm, num_entries, bits, data, fmt, device=0, null=None):
    import ctypes as C
    D = _D()
    from sdk_b200._lib import LIB
    data = np.ascontiguousarray(data, dtype=np.uint8)
    h = C.c_void_p()
    bufs = [np.zeros(1 << 22, dtype=np.uint32) for _ in range(3)]
    args = [device, C.byref(D._params(prm)), num_entries, bits, data.ctypes.data, data.size, fmt, C.byref(h)] + [b.ctypes.data for b in bufs]
    if null is not None:
        args[null] = None
    rc = LIB.b200pir_dpir_load(*args)
    assert not h.value
    return rc


def test_load_errors():
    D = _D()
    prm = dict(n=64, l=2, m=64, logq=32, p=512)
    data = np.ones(100, dtype=np.uint8)
    for null in (1, 4, 7, 8, 9, 10):
        assert _load_rc(prm, 100, 1, data, D.ENTRY_BYTES, null=null) == E_BADARG, null
    assert _load_rc(prm, 100, 1, data, D.ENTRY_BYTES, device=-1) == E_BADARG
    assert _load_rc(prm, 100, 1, data, D.ENTRY_BYTES, device=1 << 20) == E_BADARG
    assert _load_rc(prm, 100, 1, data, 2) == E_BADARG                                      # unknown entry format
    assert _load_rc(prm, 0, 1, data, D.ENTRY_BYTES) == E_BADARG                            # no entries
    assert _load_rc(prm, 100, 64, data, D.ENTRY_BYTES) == E_BADARG                         # bits_per_entry >= 64
    assert _load_rc(dict(prm, logq=31), 100, 1, data, D.ENTRY_BYTES) == E_UNSUPPORTED
    assert _load_rc(dict(prm, p=2048), 100, 1, data, D.ENTRY_BYTES) == E_UNSUPPORTED
    assert _load_rc(prm, 2 * 64 * 9 + 1, 1, data, D.ENTRY_BYTES) == E_SHAPE                # db_elems > l * m
    assert _load_rc(prm, 100, 1, np.ones(2 * 64 * 9 + 1, dtype=np.uint8), D.ENTRY_BYTES) == E_SHAPE   # too many entries
    assert _load_rc(prm, 100, 1, np.ones(2 * 64 * 9 // 8 + 1, dtype=np.uint8), D.ENTRY_BITS) == E_SHAPE
    assert _load_rc(dict(prm, p=16, l=3), 10, 8, np.ones(10, dtype=np.uint8), D.ENTRY_BYTES) == E_SHAPE   # l % x (ne = 2)
    # bytes of 255 packed 9 to a word give words past the setup GEMM's operand range
    assert _load_rc(prm, 100, 1, np.full(100, 255, dtype=np.uint8), D.ENTRY_BYTES) == E_UNSUPPORTED
    # the limits of db_info
    with pytest.raises(D.B200PirError) as e:
        D.db_info(dict(prm, l=1, m=1), 100, 1)
    assert e.value.code == E_SHAPE


def test_load_valid_call_returns_handle():
    D = _D()
    prm = dict(n=64, l=2, m=64, logq=32, p=512)
    dbm, out, info = D.load(prm, 100, 1, np.ones(100, dtype=np.uint8))
    assert info == dict(packing=9, ne=1, x=1, delta=4)
    assert dbm.download().shape == (2, 22)
    dbm.close()
