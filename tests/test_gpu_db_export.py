"""Reading the HBM database back: b200pir_db_download(_slice) and b200pir_db_save_file (Database.to_words / save_file) in every
layout, against what was uploaded, the oracle's databases (update_many_items restated, generate_db, the synthetic items) and
the file b200pir_db_load_file reads."""
import ctypes as C
import os
import subprocess
import threading

import numpy as np
import pytest

import oracle_lib as O
import param_space_sets as PS
import update_rows_oracle as U

pytestmark = pytest.mark.gpu

Q0, Q1 = 268369921, 249561089
E_BADARG, E_SHAPE, E_UNSUPPORTED = -1, -2, -4
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MASK28 = np.uint64(0x0FFFFFFF0FFFFFFF)


def _gpu():
    import sdk_b200.spiral as S
    return S


_cache = {}


def setup_case(name):
    if name not in _cache:
        S = _gpu()
        P = O.Params.named(name)
        cl = O.Client(P, 5151)
        pp = cl.generate_keys()
        G = S.Params(**P.kw)
        gpp = S.PublicParameters(G, pp["pack"], pp.get("left"), pp.get("right"), pp.get("conv"))
        _cache[name] = (S, P, cl, pp, G, gpp)
    return _cache[name]


def _words(G):
    return G.slices * G.dim0 * G.num_per * G.poly_len


def _canonical(n, seed):
    rng = np.random.default_rng(seed)
    return rng.integers(0, Q0, n, dtype=np.uint64) | (rng.integers(0, Q1, n, dtype=np.uint64) << np.uint64(32))


def _db(S, G, fmt, **kw):
    try:
        return S.Database(G, fmt=fmt, **kw)
    except S.B200PirError as e:
        if e.code == E_UNSUPPORTED:
            pytest.skip("format %d does not support this geometry" % fmt)
        raise


ROUNDTRIP_SETS = ["T", "T1", "T0", "n1", "n1_nu2_0", "nu1_1", "nu1_2", "cfg16_shrunk", "client_default"]


@pytest.mark.parametrize("name", ROUNDTRIP_SETS)
@pytest.mark.parametrize("fmt", [0, 1, 2])
def test_upload_download_identity(name, fmt):
    S = _gpu()
    kw = O.PARAM_SETS[name] if name in O.PARAM_SETS else PS.kw(name)
    G = S.Params(**kw)
    words = _canonical(_words(G), 1000 + fmt)
    words[:4] = np.uint64((Q0 - 1) | ((Q1 - 1) << 32))                 # the all-(q - 1) word
    words[-1] = 0
    gdb = _db(S, G, fmt)
    check_none = gdb.info()["present_items"]
    assert check_none == 0
    S.LIB.b200pir_db_upload(G._h, gdb._h, words.ctypes.data, words.size)
    present = gdb.info()["present_items"]
    assert np.array_equal(gdb.to_words(), words), (name, fmt)
    for s in range(G.slices):
        assert np.array_equal(gdb.download_slice(s), words.reshape(G.slices, -1)[s]), (name, fmt, s)
    assert gdb.info()["present_items"] == present                         # read-only
    if fmt == 0:                                                           # format 0 keeps any 64-bit word
        arbitrary = np.random.default_rng(7).integers(0, 2**63, words.size, dtype=np.uint64) * np.uint64(2) + np.uint64(1)
        gdb2 = S.Database.from_words(G, arbitrary, fmt=0)
        assert np.array_equal(gdb2.to_words(), arbitrary)
        gdb2.close()
    else:                                                                  # limbs: the low 28 bits of each half
        arbitrary = np.random.default_rng(8).integers(0, 2**63, words.size, dtype=np.uint64) * np.uint64(2)
        gdb2 = S.Database.from_words(G, arbitrary, fmt=fmt)
        assert np.array_equal(gdb2.to_words(), arbitrary & MASK28)
        gdb2.close()
    gdb.close()
    G.close()


def _mixed_body(P, seed):
    rng = np.random.default_rng(seed)
    full = P.slices * P.bytes_per_chunk
    last = P.dim0 * P.num_per - 1
    plan = [(17, full), (0, 100), (last, 0), (17, 5), (40 % (last + 1), full - 1), (last, full), (3, 2049), (17, 777), (1, 0)]
    return b"".join(U.entry(idx, rng.integers(0, 256, n, dtype=np.uint8)) for idx, n in plan)


@pytest.mark.parametrize("name", ["T", "T1", "T0"])
@pytest.mark.parametrize("fmt", [0, 1, 2])
def test_written_database_downloads_word_for_word(name, fmt):
    S, P, cl, pp, G, gpp = setup_case(name)
    body = _mixed_body(P, 21)
    ref_db, _, err, applied = U.update_many_items(P, body)
    assert err is None
    gdb = S.Database(G, fmt=fmt)
    gdb.update_many_items(body)
    assert np.array_equal(gdb.to_words(), ref_db.reshape(-1)), (name, fmt)
    seq = S.Database(G, fmt=fmt)
    for idx, data in applied:
        seq.update_item_raw(idx, data)
    assert np.array_equal(seq.to_words(), ref_db.reshape(-1)), (name, fmt)
    gdb.close()
    seq.close()


@pytest.mark.parametrize("fmt", [0, 1, 2])
def test_synthetic_database_downloads_as_generate_db(fmt):
    S, P, cl, pp, G, gpp = setup_case("T0")
    gdb = S.Database(G, fmt=fmt)
    gdb.fill_synthetic(0x5EED)
    assert np.array_equal(gdb.to_words(), P.generate_db(0x5EED))
    gdb.close()


@pytest.mark.parametrize("world", [2, 4])
@pytest.mark.parametrize("fmt", [0, 1, 2])
def test_shards_assemble_the_whole_database(world, fmt):
    S, P, cl, pp, G, gpp = setup_case("T")
    whole = S.Database(G, fmt=fmt)
    whole.fill_synthetic(77)
    full = whole.to_words()
    sentinel = np.uint64(0xDEADBEEFCAFEF00D)
    shards = []
    for r in range(world):
        sh = S.Database(G, shard_index=r, shard_count=world, fmt=fmt)
        sh.fill_synthetic(77)
        shards.append(sh)
    one = np.full(full.size, sentinel, dtype=np.uint64)
    assert shards[1].to_words(out=one) is one
    v = one.reshape(P.slices, P.N, P.num_per, P.dim0)
    mine = (np.arange(P.num_per) % world) == 1
    assert np.array_equal(v[:, :, mine, :], full.reshape(v.shape)[:, :, mine, :])
    assert np.all(v[:, :, ~mine, :] == sentinel)
    assembled = np.full(full.size, sentinel, dtype=np.uint64)
    for sh in shards:
        sh.to_words(out=assembled)
    assert np.array_equal(assembled, full)
    with pytest.raises(S.B200PirError) as e:
        shards[0].save_file(os.devnull)
    assert e.value.code == E_UNSUPPORTED
    for h in shards + [whole]:
        h.close()


def test_across_layouts_same_words_and_responses():
    S, P, cl, pp, G, gpp = setup_case("T")
    src = S.Database(G, fmt=2)
    src.fill_synthetic(31)
    words = src.to_words()
    q = cl.generate_query(77)
    ref = S.process_query(G, gpp, S.Query(ct=q["ct"]), src)
    for fmt in (0, 1):
        dst = S.Database.from_words(G, words, fmt=fmt)
        assert np.array_equal(dst.to_words(), words), fmt
        assert np.array_equal(S.process_query(G, gpp, S.Query(ct=q["ct"]), dst), ref), fmt
        dst.close()
    src.close()


@pytest.mark.parametrize("fmt", [0, 1, 2])
def test_save_file_and_reload(tmp_path, fmt):
    S, P, cl, pp, G, gpp = setup_case("T")
    gdb = S.Database(G, fmt=fmt)
    gdb.update_many_items(_mixed_body(P, 22))
    words = gdb.to_words()
    path = tmp_path / "snap.bin"
    gdb.save_file(path)
    assert path.read_bytes() == words.tobytes()
    assert sorted(os.listdir(tmp_path)) == ["snap.bin"]
    q = cl.generate_query(17)
    resp = S.process_query(G, gpp, S.Query(ct=q["ct"]), gdb)
    assert np.array_equal(P.process_query(pp, q, np.fromfile(str(path), dtype=np.uint64)), resp)
    back = S.Database.from_file(G, path, fmt=fmt)
    assert np.array_equal(back.to_words(), words)
    assert np.array_equal(S.process_query(G, gpp, S.Query(ct=q["ct"]), back), resp)
    for r in range(2):                                                     # a snapshot reloads into shards
        sh = S.Database.from_file(G, path, fmt=fmt, shard_index=r, shard_count=2)
        out = np.zeros_like(words)
        sh.to_words(out=out)
        rows = (np.arange(P.num_per) % 2) == r
        shape = (P.slices, P.N, P.num_per, P.dim0)
        assert np.array_equal(out.reshape(shape)[:, :, rows, :], words.reshape(shape)[:, :, rows, :])
        sh.close()
    back.close()
    gdb.close()


def test_failed_save_leaves_earlier_snapshot_and_no_temporary(tmp_path):
    S, P, cl, pp, G, gpp = setup_case("T")
    gdb = S.Database(G)
    gdb.fill_synthetic(5)
    good = tmp_path / "snap.bin"
    good.write_bytes(b"earlier snapshot")
    with pytest.raises(S.B200PirError) as e:
        gdb.save_file(tmp_path / "missing" / "snap.bin")
    assert e.value.code == E_BADARG and "missing" in str(e.value)
    assert good.read_bytes() == b"earlier snapshot"
    assert sorted(os.listdir(tmp_path)) == ["snap.bin"]
    gdb.save_file(good)                                                   # replaces the earlier file
    assert good.read_bytes() == gdb.to_words().tobytes()
    assert sorted(os.listdir(tmp_path)) == ["snap.bin"]
    gdb.close()


def test_export_argument_errors():
    S, P, cl, pp, G, gpp = setup_case("T")
    gdb = S.Database(G)
    n = _words(G)
    buf = np.zeros(n, dtype=np.uint64)
    L = S.LIB
    assert L.b200pir_db_download(None, gdb._h, buf.ctypes.data, n) == E_BADARG
    assert L.b200pir_db_download(G._h, None, buf.ctypes.data, n) == E_BADARG
    assert L.b200pir_db_download(G._h, gdb._h, None, n) == E_BADARG
    assert L.b200pir_db_download(G._h, gdb._h, buf.ctypes.data, n - 1) == E_SHAPE
    per = n // G.slices
    assert L.b200pir_db_download_slice(G._h, gdb._h, 0, buf.ctypes.data, per + 1) == E_SHAPE
    assert L.b200pir_db_download_slice(G._h, gdb._h, G.slices, buf.ctypes.data, per) == E_SHAPE
    assert L.b200pir_db_download_slice(G._h, gdb._h, 0, None, per) == E_BADARG
    assert L.b200pir_db_save_file(G._h, gdb._h, None) == E_BADARG
    assert L.b200pir_db_save_file(None, gdb._h, b"/tmp/x") == E_BADARG
    with pytest.raises(ValueError):
        gdb.to_words(out=np.zeros(n + 1, dtype=np.uint64))
    with pytest.raises(TypeError):
        gdb.to_words(out=np.zeros(n, dtype=np.int64))
    gdb.close()


@pytest.mark.parametrize("what", ["save", "download"])
def test_queries_during_an_export(tmp_path, what):
    """8 threads issue single queries on the context while another thread exports: every response equals the serial one and
    the export equals the serial export."""
    S, P, cl, pp, G, gpp = setup_case("T0")
    gdb = S.Database(G)
    gdb.fill_synthetic(9)
    serial_words = gdb.to_words()
    queries = [cl.generate_query(i * 7) for i in range(8)]
    serial = [S.process_query(G, gpp, S.Query(ct=q["ct"]), gdb) for q in queries]
    errors, exports = [], []

    def query_loop(k):
        try:
            for _ in range(6):
                got = S.process_query(G, gpp, S.Query(ct=queries[k]["ct"]), gdb)
                if not np.array_equal(got, serial[k]):
                    errors.append(k)
        except Exception as e:                                             # pragma: no cover
            errors.append(repr(e))

    def export_loop():
        for i in range(4):
            if what == "save":
                p = tmp_path / ("s%d.bin" % i)
                gdb.save_file(p)
                exports.append(np.fromfile(str(p), dtype=np.uint64))
            else:
                exports.append(gdb.to_words())

    threads = [threading.Thread(target=query_loop, args=(k,)) for k in range(8)] + [threading.Thread(target=export_loop)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors
    assert len(exports) == 4 and all(np.array_equal(e, serial_words) for e in exports)
    gdb.close()


def test_full_size_e0_synthetic_downloads_as_generate_db():
    S = _gpu()
    P = O.Params.named("E0")
    G = S.Params(**P.kw)
    gdb = S.Database(G)
    gdb.fill_synthetic(0xE0)
    got = gdb.to_words()
    gdb.close()
    ref = P.generate_db(0xE0)
    assert np.array_equal(got, ref)
    G.close()


def test_full_size_s8_items_and_round_trip():
    """S8 (8 GiB, format 2): synthetic items equal the oracle's NTT of the recentred plaintext; download, re-upload into a fresh
    database and download again gives the same words and the same response bytes for 16 queries."""
    S = _gpu()
    P = O.Params.named("S8")
    cl = O.Client(P, 88)
    pp = cl.generate_keys()
    G = S.Params(**P.kw)
    gpp = S.PublicParameters(G, pp["pack"], pp.get("left"), pp.get("right"), pp.get("conv"))
    seed = 0x58
    gdb = S.Database(G, fmt=2)
    gdb.fill_synthetic(seed)
    words = gdb.to_words()
    view = words.reshape(P.slices, P.N, P.num_per, P.dim0)
    items = P.dim0 * P.num_per
    rng = np.random.default_rng(3)
    q = np.uint64(P.modulus)
    for idx in [0, items - 1] + [int(x) for x in rng.integers(0, items, 64)]:
        pt = P.db_plain_item(seed, idx).reshape(P.slices, P.N)
        raw = np.where(pt > P.p // 2, q - (np.uint64(P.p) - pt), pt).astype(np.uint64)
        ntt = P.to_ntt(raw.reshape(-1)).reshape(P.slices, 2, P.N)
        exp = ntt[:, 0, :] | (ntt[:, 1, :] << np.uint64(32))
        ii, j = idx % P.num_per, idx // P.num_per
        assert np.array_equal(view[:, :, ii, j], exp), idx
    qs = [cl.generate_query(int(i)) for i in rng.integers(0, items, 16)]
    ref = [S.process_query(G, gpp, S.Query(ct=x["ct"]), gdb) for x in qs]
    gdb.close()
    del view
    again = S.Database.from_words(G, words, fmt=2)
    back = again.to_words()
    assert np.array_equal(back, words)
    del back, words
    for x, r in zip(qs, ref):
        assert np.array_equal(S.process_query(G, gpp, S.Query(ct=x["ct"]), again), r)
    again.close()
    gpp.close()
    G.close()


def test_cpp_host_mirror_download_save_reload(tmp_path):
    S, P, cl, pp, G, gpp = setup_case("T")
    exe = str(tmp_path / "db_export_mirror")
    subprocess.check_call(["/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++", "-std=c++17", "-O2", "-o", exe,
                           os.path.join(ROOT, "tests", "cpp", "db_export_mirror.cpp"), "-L" + os.path.join(ROOT, "sdk_b200"),
                           "-lb200pir", "-Wl,-rpath," + os.path.join(ROOT, "sdk_b200")])
    words = _canonical(_words(G), 99)
    words.tofile(str(tmp_path / "words.bin"))
    out = subprocess.check_output([exe, str(tmp_path / "words.bin"), str(tmp_path / "snap.bin"), str(tmp_path / "out.bin")],
                                  text=True)
    assert out.split() == ["same"]
    assert (tmp_path / "snap.bin").read_bytes() == words.tobytes()
    assert np.array_equal(np.fromfile(str(tmp_path / "out.bin"), dtype=np.uint64), words)
