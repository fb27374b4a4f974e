"""b200pir_db_update_many_items (the /update-row body, lib/server/src/db/loading.rs:361-377) on the GPU against the restatement
of update_many_items in tests/update_rows_oracle.py, which applies the entries one by one into a host database with the CPU
oracle's update_item_raw.  Bit-exact: the first-dimension products of every slice are compared as integers."""
import os
import subprocess

import numpy as np
import pytest

import oracle_lib as O
import update_rows_oracle as U

pytestmark = pytest.mark.gpu

Q0, Q1 = 268369921, 249561089
E_SHAPE = -2
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _gpu():
    import sdk_b200.spiral as S
    return S


_cache = {}


def setup_case(name):
    if name not in _cache:
        S = _gpu()
        P = O.Params.named(name)
        cl = O.Client(P, 4242)
        pp = cl.generate_keys()
        G = S.Params(**P.kw)
        gpp = S.PublicParameters(G, pp["pack"], pp.get("left"), pp.get("right"), pp.get("conv"))
        _cache[name] = (S, P, cl, pp, G, gpp)
    return _cache[name]


def _v(P, seed):
    rng = np.random.default_rng(seed)
    return (rng.integers(0, Q0, P.dim0 * 2 * P.N, dtype=np.uint64)
            | (rng.integers(0, Q1, P.dim0 * 2 * P.N, dtype=np.uint64) << np.uint64(32)))


def _assert_db_equals(S, P, G, gdb, ref_db, v, what):
    for s in range(P.slices):
        ref = P.multiply_reg_by_database(np.ascontiguousarray(ref_db[s]).reshape(-1), v)
        assert np.array_equal(S.multiply_reg_by_database(G, gdb, s, v), ref), (what, s)


def _mixed_body(P, seed):
    """Full-length, short and zero-length entries, db_idx 0 and num_items - 1, one db_idx written three times."""
    rng = np.random.default_rng(seed)
    full = P.slices * P.bytes_per_chunk
    last = P.dim0 * P.num_per - 1
    plan = [(17, full), (0, 100), (last, 0), (17, 5), (40 % (last + 1), full - 1), (last, full), (3, 2049), (17, 777), (1, 0)]
    body = b"".join(U.entry(idx, rng.integers(0, 256, n, dtype=np.uint8)) for idx, n in plan)
    return body, plan


@pytest.mark.parametrize("name", ["T", "T1", "T0"])
@pytest.mark.parametrize("fmt", [0, 1, 2])
def test_update_many_items_matches_oracle(name, fmt):
    S, P, cl, pp, G, gpp = setup_case(name)
    body, plan = _mixed_body(P, 11)
    ref_db, ref_largest, ref_err, applied = U.update_many_items(P, body)
    assert ref_err is None and len(applied) == len(plan)
    gdb = S.Database(G, fmt=fmt)
    largest = gdb.update_many_items(body)
    assert largest == ref_largest
    v = _v(P, 3)
    _assert_db_equals(S, P, G, gdb, ref_db, v, (name, fmt))
    # the same entries through per-entry update_item_raw calls, in body order
    seq = S.Database(G, fmt=fmt)
    for idx, data in applied:
        seq.update_item_raw(idx, data)
    for s in range(P.slices):
        assert np.array_equal(S.multiply_reg_by_database(G, gdb, s, v), S.multiply_reg_by_database(G, seq, s, v)), (name, fmt, s)
    distinct = {idx for idx, _ in applied}
    assert gdb.info()["present_items"] == len(distinct) * P.slices == seq.info()["present_items"]
    # a private read of written items: response bytes == the oracle's process_query over the restated database, and the
    # response decodes to what the fold reads back (update_rows_oracle.read_back).  Decoded with the fold each version is
    # served with: spiral-rs's dense fold (the default) on version 0, lib/server's ("sparse_fold") on version 1, where the
    # dense fold loses the margin next to empty rows (test_oracle_written_items_decode.py).
    last = {idx: data for idx, data in applied}
    pt_len = P.bytes_per_chunk
    for idx in sorted(distinct)[:4]:
        q = cl.generate_query(idx)
        resp = S.process_query(G, gpp, S.Query(ct=q["ct"]), gdb)
        assert np.array_equal(resp, P.process_query(pp, q, ref_db.reshape(-1))), (name, fmt, idx)
        assert np.array_equal(resp, S.process_query(G, gpp, S.Query(ct=q["ct"]), seq)), (name, fmt, idx)
        if P.version == 1:
            G.set_option("sparse_fold", 1)
            try:
                resp = S.process_query(G, gpp, S.Query(ct=q["ct"]), gdb)
            finally:
                G.set_option("sparse_fold", 0)
            assert np.array_equal(resp, P.process_query(pp, q, ref_db.reshape(-1), sparse_fold=True)), (name, fmt, idx)
        got = cl.decode_response(resp).reshape(P.slices, P.N)[:, :pt_len].astype(np.uint8).reshape(-1)
        exp = U.read_back(P, ref_db, last, idx, sparse_fold=P.version == 1)
        assert np.array_equal(got, exp), (name, fmt, idx, int(np.count_nonzero(got != exp)))
    gdb.close()
    seq.close()


def _bad_bodies(P):
    """(case, body with entries 0..k-1 good, entry k bad, good entries after it), k = 3."""
    rng = np.random.default_rng(12)
    full = P.slices * P.bytes_per_chunk
    good = b"".join(U.entry(i * 5, rng.integers(0, 256, n, dtype=np.uint8)) for i, n in enumerate((full, 10, 0)))
    after = U.entry(1, rng.integers(0, 256, 50, dtype=np.uint8)) + U.entry(0, b"\x07" * 9)
    yield "over-long", good + U.entry(2, rng.integers(0, 256, full + 1, dtype=np.uint8)) + after
    yield "bad db_idx", good + U.entry(P.dim0 * P.num_per, b"\x01\x02") + after
    yield "header truncated", good + U.entry(2, b"\x05" * 30)[:3]
    yield "chunk truncated", good + U.entry(2, b"\x05" * 30)[:-1]
    yield "chunk_len < 4", good + (2).to_bytes(4, "big") + b"\x00\x01" + after


@pytest.mark.parametrize("case", ["over-long", "bad db_idx", "header truncated", "chunk truncated", "chunk_len < 4"])
def test_update_many_items_bad_entry_applies_prefix_only(case):
    S, P, cl, pp, G, gpp = setup_case("T")
    body = dict(_bad_bodies(P))[case]
    ref_db, _, ref_err, applied = U.update_many_items(P, body)
    assert ref_err is not None and len(applied) == 3
    gdb = S.Database(G)
    with pytest.raises(S.B200PirError) as e:
        gdb.update_many_items(body)
    assert e.value.code == E_SHAPE, case
    _assert_db_equals(S, P, G, gdb, ref_db, _v(P, 4), case)
    assert gdb.info()["present_items"] == 3 * P.slices
    gdb.close()


def test_update_many_items_empty_body_is_a_noop():
    S, P, cl, pp, G, gpp = setup_case("T")
    gdb = S.Database(G)
    gdb.update_item_raw(9, np.arange(100, dtype=np.uint8))
    v = _v(P, 5)
    before = [S.multiply_reg_by_database(G, gdb, s, v) for s in range(P.slices)]
    assert gdb.update_many_items(b"") == 0
    assert all(np.array_equal(S.multiply_reg_by_database(G, gdb, s, v), before[s]) for s in range(P.slices))
    assert gdb.info()["present_items"] == P.slices
    gdb.close()


@pytest.mark.parametrize("world", [2, 4])
def test_update_many_items_sharded(world):
    """Every shard of T0 gets the same body; the rows of each equal the matching rows of the unsharded database, and with a bad
    entry every shard stops at the same place with the same status."""
    S, P, cl, pp, G, gpp = setup_case("T0")
    body, _ = _mixed_body(P, 13)
    whole = S.Database(G)
    largest = whole.update_many_items(body)
    v = _v(P, 6)
    full = [S.multiply_reg_by_database(G, whole, s, v).reshape(P.num_per, -1) for s in range(P.slices)]
    bad = body + U.entry(P.dim0 * P.num_per + 3, b"") + U.entry(2, b"\x09" * 40)
    whole_bad = S.Database(G)
    with pytest.raises(S.B200PirError):
        whole_bad.update_many_items(bad)
    full_bad = [S.multiply_reg_by_database(G, whole_bad, s, v).reshape(P.num_per, -1) for s in range(P.slices)]
    for r in range(world):
        sh = S.Database(G, shard_index=r, shard_count=world)
        assert sh.update_many_items(body) == largest
        for s in range(P.slices):
            assert np.array_equal(S.multiply_reg_by_database(G, sh, s, v).reshape(P.num_per // world, -1), full[s][r::world]), (world, r, s)
        sh_bad = S.Database(G, shard_index=r, shard_count=world)
        with pytest.raises(S.B200PirError) as e:
            sh_bad.update_many_items(bad)
        assert e.value.code == E_SHAPE
        for s in range(P.slices):
            assert np.array_equal(S.multiply_reg_by_database(G, sh_bad, s, v).reshape(P.num_per // world, -1),
                                  full_bad[s][r::world]), (world, r, s)
        sh.close()
        sh_bad.close()
    whole.close()
    whole_bad.close()


def test_update_many_items_body_spans_several_staging_groups():
    """S8 (8 GiB): 2^14 full 8192-byte items to distinct random db_idx in one body of 134 MB, more than twice the 64 MiB
    staging budget, so the body is applied in three groups.  Items of the first and the last group decode through
    process_query, and response bytes equal those of a database written by per-item update_item_raw calls."""
    S = _gpu()
    P = O.Params.named("S8")
    cl = O.Client(P, 99)
    pp = cl.generate_keys()
    G = S.Params(**P.kw)
    gpp = S.PublicParameters(G, pp["pack"], pp.get("left"), pp.get("right"), pp.get("conv"))
    rng = np.random.default_rng(14)
    count = 1 << 14
    idxs = rng.choice(P.dim0 * P.num_per, count, replace=False)
    items = rng.integers(0, 256, (count, P.db_item_size), dtype=np.uint8)
    body = b"".join(U.entry(int(i), items[k]) for k, i in enumerate(idxs))
    assert len(body) > 2 * (64 << 20)
    gdb = S.Database(G)
    assert gdb.update_many_items(body) == 4 + P.db_item_size
    assert gdb.info()["present_items"] == count * P.slices
    seq = S.Database(G)
    for k, i in enumerate(idxs):
        seq.update_item_raw(int(i), items[k])
    for k in (0, 1, count // 2, count - 2, count - 1):
        q = cl.generate_query(int(idxs[k]))
        resp = S.process_query(G, gpp, S.Query(ct=q["ct"]), gdb)
        assert np.array_equal(resp, S.process_query(G, gpp, S.Query(ct=q["ct"]), seq)), k
        got = cl.decode_response(resp).reshape(P.slices, P.N)[:, :P.bytes_per_chunk].astype(np.uint8).reshape(-1)
        assert np.array_equal(got[:P.db_item_size], items[k]), k
    for h in (gdb, seq, gpp, G):
        h.close()


def test_cpp_host_mirror_update_many_items(tmp_path):
    """include/b200pir.hpp's Database::update_many_items (tests/cpp/update_many_mirror.cpp) on parameter set T: largest_update
    and the first-dimension product of slice 0 equal the Python path's on the same body."""
    S, P, cl, pp, G, gpp = setup_case("T")
    exe = str(tmp_path / "update_many_mirror")
    subprocess.check_call(["/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++", "-std=c++17", "-O2", "-o", exe,
                           os.path.join(ROOT, "tests", "cpp", "update_many_mirror.cpp"), "-L" + os.path.join(ROOT, "sdk_b200"),
                           "-lb200pir", "-Wl,-rpath," + os.path.join(ROOT, "sdk_b200")])
    body, _ = _mixed_body(P, 15)
    v = _v(P, 7)
    (tmp_path / "body.bin").write_bytes(body)
    v.tofile(str(tmp_path / "v.bin"))
    out = subprocess.check_output([exe, str(tmp_path / "body.bin"), str(tmp_path / "v.bin"), str(tmp_path / "out.bin")], text=True)
    gdb = S.Database(G)
    assert int(out.split()[0]) == gdb.update_many_items(body)
    got = np.fromfile(str(tmp_path / "out.bin"), dtype=np.uint64)
    assert np.array_equal(got, S.multiply_reg_by_database(G, gdb, 0, v))
    gdb.close()
