"""Reading the HBM database back as plaintext: b200pir_db_read_items (Database.read_items) and b200pir_db_save_raw_file
(Database.save_raw_file) in every layout.  Items written through the raw writers come back byte for byte, the oracle's
load_db_from_seek database decodes to its raw bytes, raw files round-trip through load_raw_file, a raw snapshot serves the same
responses as its source, sharded databases read the same as unsharded ones, and every refusal leaves files and the database
as they were."""
import glob
import hashlib
import os

import numpy as np
import pytest

import oracle_lib as O
import param_space_sets as PS
import update_rows_oracle as U

pytestmark = pytest.mark.gpu

Q0, Q1 = 268369921, 249561089
E_BADARG, E_SHAPE, E_UNSUPPORTED = -1, -2, -4
PRESENT, NOT_PLAINTEXT, PAST_CHUNK = 1, 2, 4
FORMATS = [0, 1, 2]


def _gpu():
    import sdk_b200.spiral as S
    return S


def _kw(shrink=0, item_size=None):
    kw = dict(O.PARAM_SETS["T"])
    kw["db_item_size"] = (item_size or kw["db_item_size"]) - shrink
    return kw


def _span(G):
    return G.slices * ((G.db_item_size + G.slices - 1) // G.slices)


def _items(G):
    return G.dim0 * G.num_per


def _raw_items(raw, G):
    """What load_db_from_seek reads for every item of a raw file image: span bytes from i * db_item_size, zero past the end."""
    span, isz, n = _span(G), G.db_item_size, _items(G)
    padded = np.zeros(n * isz + span, dtype=np.uint8)
    padded[:raw.size] = raw
    return np.stack([padded[i * isz:i * isz + span] for i in range(n)])


_ctx = {}


def _params(kw):
    key = tuple(sorted(kw.items()))
    if key not in _ctx:
        _ctx[key] = _gpu().Params(**kw)
    return _ctx[key]


@pytest.mark.parametrize("fmt", FORMATS)
def test_written_items_read_back_exactly(fmt):
    S = _gpu()
    G = _params(_kw())
    span, n = _span(G), _items(G)
    rng = np.random.default_rng(100 + fmt)
    plan = [(5, span), (17, 0), (n - 1, 3000), (17, 1234), (40, span - 1), (0, 1), (77, 2049), (5, 10)]
    body = b"".join(U.entry(i, rng.integers(0, 256, ln, dtype=np.uint8)) for i, ln in plan)
    want, off = {}, 0                                            # the last bytes of each db_idx, zero padded
    for i, ln in plan:
        data = np.frombuffer(body[off + 8:off + 8 + ln], dtype=np.uint8)
        want[i] = np.concatenate([data, np.zeros(span - ln, dtype=np.uint8)])
        off += 8 + ln
    gdb = S.Database(G, fmt=fmt)
    gdb.update_many_items(body)
    seq = S.Database(G, fmt=fmt)
    for i, ln in plan:
        seq.update_item_raw(i, want[i][:ln] if ln else np.zeros(0, dtype=np.uint8))
    idx = np.arange(n, dtype=np.uint64)
    for db in (gdb, seq):
        got, flags = db.read_items(idx)
        assert got.shape == (n, span)
        for i in range(n):
            if i in want:
                assert np.array_equal(got[i], want[i]), (fmt, i)
                assert flags[i] == PRESENT, (fmt, i, flags[i])
            else:
                assert not got[i].any() and flags[i] == 0, (fmt, i)
        # any order, repeated indices, a count of zero
        pick = np.array([n - 1, 5, 5, 3, 17], dtype=np.uint64)
        sub, f2 = db.read_items(pick)
        assert np.array_equal(sub, got[pick.astype(np.int64)]) and np.array_equal(f2, flags[pick.astype(np.int64)])
        empty, f0 = db.read_items(np.zeros(0, dtype=np.uint64))
        assert empty.shape == (0, span) and f0.size == 0
    gdb.close()
    seq.close()


@pytest.mark.parametrize("fmt", FORMATS)
def test_oracle_database_reads_as_its_raw_bytes(fmt):
    S = _gpu()
    kw = _kw()
    P = O.Params(**kw)
    G = _params(kw)
    rng = np.random.default_rng(33 + fmt)
    raw = rng.integers(0, 256, _items(G) * G.db_item_size - 3000, dtype=np.uint8)
    gdb = S.Database.from_words(G, P.load_db_from_bytes(raw), fmt=fmt)
    want = _raw_items(raw, G)
    idx = rng.integers(0, _items(G), 100, dtype=np.uint64)
    got, flags = gdb.read_items(idx)
    assert np.array_equal(got, want[idx.astype(np.int64)]), fmt
    assert (flags == PRESENT).all()
    gdb.close()


@pytest.mark.parametrize("shrink", [0, 2])
@pytest.mark.parametrize("fmt", FORMATS)
def test_raw_file_round_trip(fmt, shrink, tmp_path):
    """shrink = 2: an item's span is two bytes longer than db_item_size, so its last bytes are the next item's first ones."""
    S = _gpu()
    G = _params(_kw(shrink))
    n, isz = _items(G), G.db_item_size
    raw = np.random.default_rng(7 + shrink).integers(0, 256, n * isz - 3000, dtype=np.uint8)
    src = tmp_path / "raw.bin"
    raw.tofile(str(src))
    gdb = S.Database.from_raw_file(G, src, fmt=fmt)
    out = tmp_path / "saved.bin"
    gdb.save_raw_file(out)
    want = np.zeros(n * isz, dtype=np.uint8)
    want[:raw.size] = raw
    assert np.array_equal(np.fromfile(str(out), dtype=np.uint8), want), (fmt, shrink)
    assert not glob.glob(str(tmp_path / "*.tmp.*"))
    gdb.close()


@pytest.mark.parametrize("fmt", FORMATS)
def test_raw_snapshot_serves_the_same_responses(fmt, tmp_path):
    S = _gpu()
    kw = _kw()
    P = O.Params(**kw)
    cl = O.Client(P, 4242)
    pp = cl.generate_keys()
    G = _params(kw)
    gpp = S.PublicParameters(G, pp["pack"], pp.get("left"), pp.get("right"), pp.get("conv"))
    n, span = _items(G), _span(G)
    rng = np.random.default_rng(9)
    body = b"".join(U.entry(i, rng.integers(0, 256, int(rng.integers(0, span + 1)), dtype=np.uint8))
                    for i in rng.choice(n, n // 3, replace=False))
    src = S.Database(G, fmt=fmt)                                 # sparse: two thirds of the items absent
    src.update_many_items(body)
    path = tmp_path / "snap.raw"
    src.save_raw_file(path)
    assert os.path.getsize(path) == n * G.db_item_size
    back = S.Database.from_raw_file(G, path, fmt=fmt)
    assert np.array_equal(back.to_words(), src.to_words()), fmt
    assert back.info()["present_items"] == back.info()["capacity"]        # the raw format has no presence map
    blobs = []
    for i in (0, n - 1, 37, 100):
        cl.generate_query(i)
        blobs.append(cl.query_bytes())
    blob = np.concatenate(blobs)
    try:
        for sparse in (0, 1):
            G.set_option("sparse_fold", sparse)
            assert np.array_equal(S.process_query_bytes(G, gpp, blob, back), S.process_query_bytes(G, gpp, blob, src)), (fmt, sparse)
    finally:
        G.set_option("sparse_fold", 0)
    src.close()
    back.close()
    gpp.close()


@pytest.mark.parametrize("fmt", FORMATS)
def test_flags_and_refusals(fmt, tmp_path):
    S = _gpu()
    G = _params(_kw())
    n = _items(G)
    # an arbitrary polynomial is not plaintext, and no raw file holds it
    gdb = S.Database(G, fmt=fmt)
    gdb.update_item_raw(3, np.arange(100, dtype=np.uint8))
    rng = np.random.default_rng(5)
    poly = rng.integers(0, Q0, 2048, dtype=np.uint64) | (rng.integers(0, Q1, 2048, dtype=np.uint64) << np.uint64(32))
    gdb.upsert_item(1, 9, poly)
    got, flags = gdb.read_items(np.array([9, 3, 4], dtype=np.uint64))
    assert flags.tolist() == [PRESENT | NOT_PLAINTEXT, PRESENT, 0], flags
    target = tmp_path / "keep.raw"
    target.write_bytes(b"earlier snapshot")
    with pytest.raises(S.B200PirError) as e:
        gdb.save_raw_file(target)
    assert e.value.code == E_UNSUPPORTED and "item 9" in str(e.value)
    assert target.read_bytes() == b"earlier snapshot" and not glob.glob(str(tmp_path / "*.tmp.*"))
    gdb.close()
    # the synthetic fill draws all 2048 coefficients: with 1024-byte chunks the upper half is past the chunk
    H = _params(_kw(item_size=4096))
    syn = S.Database(H, fmt=fmt)
    syn.fill_synthetic(11)
    _, flags = syn.read_items(np.arange(8, dtype=np.uint64))
    assert (flags == PRESENT | PAST_CHUNK).all(), flags
    with pytest.raises(S.B200PirError) as e:
        syn.save_raw_file(target)
    assert e.value.code == E_UNSUPPORTED and "item 0" in str(e.value)
    syn.close()
    # shrink 2: items that disagree on the bytes they share in the file, and a last item with bytes past the end
    K = _params(_kw(2))
    span, isz = _span(K), K.db_item_size
    raw = np.random.default_rng(8).integers(0, 256, n * isz, dtype=np.uint8)
    src = tmp_path / "raw.bin"
    raw.tofile(str(src))
    over = S.Database.from_raw_file(K, src, fmt=fmt)
    item = raw[10 * isz:10 * isz + span].copy()
    item[-1] ^= 1                                                # item 11's second byte, as item 10 sees it
    over.update_item_raw(10, item)
    with pytest.raises(S.B200PirError) as e:
        over.save_raw_file(target)
    assert e.value.code == E_UNSUPPORTED and "item 10" in str(e.value)
    over.update_item_raw(10, raw[10 * isz:10 * isz + span])     # consistent again
    last = np.concatenate([raw[(n - 1) * isz:], np.array([0, 7], dtype=np.uint8)])
    over.update_item_raw(n - 1, last)
    with pytest.raises(S.B200PirError) as e:
        over.save_raw_file(target)
    assert e.value.code == E_UNSUPPORTED and "item %d" % (n - 1) in str(e.value)
    assert target.read_bytes() == b"earlier snapshot" and not glob.glob(str(tmp_path / "*.tmp.*"))
    over.update_item_raw(n - 1, raw[(n - 1) * isz:])
    over.save_raw_file(target)
    assert np.array_equal(np.fromfile(str(target), dtype=np.uint8), raw)
    over.close()


@pytest.mark.parametrize("shards", [2, 4])
@pytest.mark.parametrize("fmt", FORMATS)
def test_sharded_databases_read_as_unsharded(fmt, shards, tmp_path):
    S = _gpu()
    kw = _kw()
    G = _params(kw)
    n, span = _items(G), _span(G)
    raw = np.random.default_rng(21).integers(0, 256, n * G.db_item_size - 5000, dtype=np.uint8)
    src = tmp_path / "raw.bin"
    raw.tofile(str(src))
    whole = S.Database.from_raw_file(G, src, fmt=fmt)
    rng = np.random.default_rng(22)
    body = b"".join(U.entry(i, rng.integers(0, 256, span, dtype=np.uint8)) for i in (1, 6, n - 2))
    whole.update_many_items(body)
    ctxs = [S.Params(device=0, **kw) for _ in range(shards)]
    sdb = S.Database.from_words(ctxs[0], whole.to_words(), fmt=fmt, contexts=ctxs)
    idx = np.concatenate([np.arange(n), rng.integers(0, n, 50)]).astype(np.uint64)
    a, fa = whole.read_items(idx)
    b, fb = sdb.read_items(idx)
    assert np.array_equal(a, b) and np.array_equal(fa, fb), (fmt, shards)
    whole.save_raw_file(tmp_path / "u.raw")
    sdb.save_raw_file(tmp_path / "s.raw")
    assert (tmp_path / "u.raw").read_bytes() == (tmp_path / "s.raw").read_bytes()
    sdb.close()
    # a rank shard holds rows ii = 1 (mod 2): index 4 (row 0) lives elsewhere
    rank = S.Database(G, shard_index=1, shard_count=2, fmt=fmt)
    rank.update_item_raw(5, np.arange(10, dtype=np.uint8))
    got, flags = rank.read_items(np.array([5], dtype=np.uint64))
    assert np.array_equal(got[0, :10], np.arange(10, dtype=np.uint8)) and flags[0] == PRESENT
    with pytest.raises(S.B200PirError) as e:
        rank.read_items(np.array([5, 4], dtype=np.uint64))
    assert e.value.code == E_SHAPE
    with pytest.raises(S.B200PirError) as e:
        rank.save_raw_file(tmp_path / "r.raw")
    assert e.value.code == E_UNSUPPORTED and not (tmp_path / "r.raw").exists()
    rank.close()
    whole.close()


@pytest.mark.parametrize("fmt", FORMATS)
def test_read_only_and_errors(fmt, tmp_path):
    S = _gpu()
    G = _params(_kw())
    n, span = _items(G), _span(G)
    gdb = S.Database(G, fmt=fmt)
    rng = np.random.default_rng(3)
    gdb.update_many_items(b"".join(U.entry(i, rng.integers(0, 256, 700, dtype=np.uint8)) for i in (2, 9, 60)))
    before, info = gdb.to_words(), gdb.info()
    gdb.read_items(np.arange(n, dtype=np.uint64))
    gdb.save_raw_file(tmp_path / "a.raw")
    assert np.array_equal(gdb.to_words(), before) and gdb.info() == info
    L = S.LIB
    idx = np.array([2, 9], dtype=np.uint64)
    out = np.full((2, span), 0xAB, dtype=np.uint8)
    flags = np.full(2, 0xCD, dtype=np.uint8)
    assert L.b200pir_db_read_items(None, gdb._h, idx.ctypes.data, 2, out.ctypes.data, None) == E_BADARG
    assert L.b200pir_db_read_items(G._h, gdb._h, None, 2, out.ctypes.data, None) == E_BADARG
    assert L.b200pir_db_read_items(G._h, gdb._h, idx.ctypes.data, 2, None, None) == E_BADARG
    assert L.b200pir_db_read_items(G._h, None, idx.ctypes.data, 2, out.ctypes.data, None) == E_BADARG
    assert L.b200pir_db_save_raw_file(G._h, gdb._h, None) == E_BADARG
    assert L.b200pir_db_save_raw_file(None, gdb._h, str(tmp_path / "b.raw").encode()) == E_BADARG
    bad = np.array([2, n], dtype=np.uint64)
    assert L.b200pir_db_read_items(G._h, gdb._h, bad.ctypes.data, 2, out.ctypes.data, flags.ctypes.data) == E_SHAPE
    assert (out == 0xAB).all() and (flags == 0xCD).all()             # nothing written
    assert L.b200pir_db_read_items(G._h, gdb._h, idx.ctypes.data, 2, out.ctypes.data, None) == 0   # flags may be NULL
    assert L.b200pir_db_save_raw_file(G._h, gdb._h, str(tmp_path / "no" / "dir.raw").encode()) == E_BADARG
    gdb.close()
    # p != 256 and chunks longer than poly_len: the raw writers' refusals
    for kw, code in ((PS.kw("p16_q14"), E_UNSUPPORTED), (_kw(item_size=4 * 2048 + 4), E_SHAPE)):
        H = S.Params(**kw)
        hdb = S.Database(H, fmt=fmt)
        one = np.zeros(1, dtype=np.uint64)
        buf = np.zeros(H.slices * ((H.db_item_size + H.slices - 1) // H.slices), dtype=np.uint8)
        assert L.b200pir_db_read_items(H._h, hdb._h, one.ctypes.data, 1, buf.ctypes.data, None) == code, kw
        assert L.b200pir_db_save_raw_file(H._h, hdb._h, str(tmp_path / "c.raw").encode()) == code, kw
        assert not (tmp_path / "c.raw").exists()
        hdb.close()
        H.close()


@pytest.fixture(scope="module")
def s8_raw(tmp_path_factory):
    kw = O.PARAM_SETS["S8"]
    n = (1 << kw["nu_1"]) * (1 << kw["nu_2"])
    path = tmp_path_factory.mktemp("s8") / "s8.raw"
    rng = np.random.default_rng(0x58)
    with open(path, "wb") as f:
        for k in range(0, n, 8192):
            f.write(rng.integers(0, 256, 8192 * kw["db_item_size"], dtype=np.uint8).tobytes())
    h = hashlib.sha256()
    with open(path, "rb") as f:
        for block in iter(lambda: f.read(1 << 24), b""):
            h.update(block)
    return path, h.hexdigest()


@pytest.mark.parametrize("fmt", FORMATS)
def test_s8_raw_file_round_trip(fmt, s8_raw):
    S = _gpu()
    path, digest = s8_raw
    G = _params(dict(O.PARAM_SETS["S8"]))
    gdb = S.Database.from_raw_file(G, path, fmt=fmt)
    out = str(path) + ".saved"
    try:
        gdb.save_raw_file(out)
        gdb.close()
        h = hashlib.sha256()
        with open(out, "rb") as f:
            for block in iter(lambda: f.read(1 << 24), b""):
                h.update(block)
        assert h.hexdigest() == digest, fmt
    finally:
        if os.path.exists(out):
            os.unlink(out)
