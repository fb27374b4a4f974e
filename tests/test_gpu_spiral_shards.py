"""One Spiral database in row shards over several contexts, served and written from one process
(b200pir_db_create_sharded).  Every response must be byte for byte that of an unsharded database holding the same contents on
the home context, and, for two queries per case, the oracle's bytes decoding to the planted items; every writer must leave the
same database (download, presence) as on an unsharded one."""
import threading

import numpy as np
import pytest

import oracle_lib as O
from test_gpu_parity import setup_case, SEED_DB, _gpu

pytestmark = pytest.mark.gpu

E_BADARG, E_UNSUPPORTED = -1, -4


def _contexts(S, P, devices, expand=True):
    return [S.Params(device=d, expand_queries=expand, **P.kw) for d in devices]


def _device_count():
    return int(_gpu().LIB.b200pir_device_count())


_refs = {}


def _unsharded(name, expand, fmt):
    """An unsharded database of the case's contents in layout `fmt` on the cached context."""
    key = (name, expand, fmt)
    if key not in _refs:
        S, P, cl, pp, db, G, gdb, gpp = setup_case(name, expand)
        _refs[key] = S.Database.from_words(G, db, fmt=fmt)
    return _refs[key]


def _batch_dev(S, H, sdb, gpp, cts):
    import torch
    count = cts.size // (2 * 2048)
    d_q = torch.from_numpy(np.ascontiguousarray(cts).view(np.int64)).cuda()
    d_out = torch.zeros(count * H.response_bytes, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    S.check(S.LIB.b200pir_process_query_batch_dev(H._h, sdb._h, gpp._h, d_q.data_ptr(), count, d_out.data_ptr()))
    H.synchronize()
    return d_out.cpu().numpy().reshape(count, H.response_bytes)


CASES = [("T0", True), ("T", True), ("T1", True), ("T", False)]


@pytest.mark.parametrize("fmt", [0, 1, 2])
@pytest.mark.parametrize("shards", [1, 2, 4])
@pytest.mark.parametrize("name,expand", CASES)
def test_sharded_responses_equal_unsharded_and_oracle(name, expand, shards, fmt):
    S, P, cl, pp, db, G, gdb, gpp = setup_case(name, expand)
    udb = _unsharded(name, expand, fmt)
    ctxs = _contexts(S, P, [0] * shards, expand)
    H = ctxs[0]
    sdb = S.Database.from_words(H, db, fmt=fmt, contexts=ctxs)
    info = sdb.info()
    assert info["format"] == udb.info()["format"] and info["local_rows"] == P.num_per
    # hbm_bytes sums the shards, each laid out (and padded) as the rank shard of b200pir_db_create(ctx, g, G)
    rank = [S.Database(G, shard_index=g, shard_count=shards, fmt=fmt) for g in range(shards)]
    assert info["hbm_bytes"] == sum(r.info()["hbm_bytes"] for r in rank)
    for r in rank:
        r.close()
    sparse = name == "T1"                       # version-1 servers fold like lib/server
    if sparse:
        H.set_option("sparse_fold", 1)
        G.set_option("sparse_fold", 1)
    try:
        n_items = P.dim0 * P.num_per
        idxs = [0, n_items - 1, 77 % n_items, 5, 130 % n_items]
        qs, blobs = [], []
        for i in idxs:
            qs.append(cl.generate_query(i))
            blobs.append(cl.query_bytes())
        # process_query: two queries against the oracle and the planted items
        for k in range(2):
            q = qs[k]
            query = S.Query(ct=q["ct"]) if expand else S.Query(v_buf=q["v_buf"], v_ct=q["v_ct"])
            got = S.process_query(H, gpp, query, sdb)
            assert np.array_equal(got, S.process_query(G, gpp, query, udb)), k
            assert np.array_equal(got, P.process_query(pp, q, db, sparse_fold=sparse)), k
            assert np.array_equal(cl.decode_response(got), P.db_plain_item(SEED_DB, idxs[k])), k
        # process_query_bytes with one query (the coalescer, in expanding mode) and with five
        one = S.process_query_bytes(H, gpp, blobs[0], sdb)
        assert np.array_equal(one, S.process_query_bytes(G, gpp, blobs[0], udb))
        five = S.process_query_bytes(H, gpp, np.concatenate(blobs), sdb)
        assert np.array_equal(five, S.process_query_bytes(G, gpp, np.concatenate(blobs), udb))
        if not expand:
            return
        # a batch of 17: one full group of 16 and a partial second group
        cts = np.concatenate([cl.generate_query((31 * k + 3) % n_items)["ct"] for k in range(17)])
        got = S.process_query_batch(H, gpp, cts, sdb)
        assert np.array_equal(got, S.process_query_batch(G, gpp, cts, udb))
        assert np.array_equal(_batch_dev(S, H, sdb, gpp, cts), got)
        # two clients' parameters in one call
        cl_b = O.Client(P, 777)
        pp_b = cl_b.generate_keys()
        gpp_b = S.PublicParameters(G, pp_b["pack"], pp_b["left"], pp_b["right"], pp_b["conv"])
        plan = [(cl, gpp, 5), (cl_b, gpp_b, 9 % n_items), (cl_b, gpp_b, 0), (cl, gpp, n_items - 1)]
        mixed = [c.generate_query(i)["ct"] for c, _, i in plan]
        got = S.process_queries(H, [g for _, g, _ in plan], mixed, sdb)
        assert np.array_equal(got, S.process_queries(G, [g for _, g, _ in plan], mixed, udb))
        for k, (c, _, i) in enumerate(plan):
            assert np.array_equal(c.decode_response(got[k]), P.db_plain_item(SEED_DB, i)), k
        gpp_b.close()
    finally:
        if sparse:
            G.set_option("sparse_fold", 0)
        sdb.close()


# ------------------------------------------------------------------ S8 geometry
@pytest.fixture(scope="module")
def s8():
    S = _gpu()
    P = O.Params.named("S8")
    cl = O.Client(P, 5)
    pp = cl.generate_keys()
    G = S.Params(**P.kw)
    gdb = S.Database(G)
    gdb.fill_synthetic(SEED_DB)
    gpp = S.PublicParameters(G, pp["pack"], pp["left"], pp["right"], pp["conv"])
    n_items = P.dim0 * P.num_per
    idxs = [(7919 * k + 31) % n_items for k in range(32)]
    cts = np.concatenate([cl.generate_query(i)["ct"] for i in idxs])
    yield S, P, cl, G, gdb, gpp, idxs, cts
    gpp.close()
    gdb.close()
    G.close()


@pytest.mark.parametrize("shards", [2, 4])
def test_s8_sharded_batches_equal_unsharded(s8, shards):
    S, P, cl, G, gdb, gpp, idxs, cts = s8
    ctxs = _contexts(S, P, [0] * shards)
    sdb = S.Database.sharded(ctxs)
    sdb.fill_synthetic(SEED_DB)
    assert sdb.info()["format"] == gdb.info()["format"]
    try:
        for count in (16, 32):
            part = cts[:count * 2 * 2048]
            got = S.process_query_batch(ctxs[0], gpp, part, sdb)
            assert np.array_equal(got, S.process_query_batch(G, gpp, part, gdb)), count
        assert np.array_equal(cl.decode_response(got[0]), P.db_plain_item(SEED_DB, idxs[0]))
    finally:
        sdb.close()


# ------------------------------------------------------------------ shards on two devices
@pytest.mark.parametrize("devices", [[0, 1], [0, 1, 0, 1]])
def test_two_devices_equal_unsharded(devices):
    if _device_count() < 2:
        pytest.skip("needs two GPUs")
    S, P, cl, pp, db, G, gdb, gpp = setup_case("T0")
    ctxs = _contexts(S, P, devices)
    H = ctxs[0]
    sdb = S.Database.from_words(H, db, contexts=ctxs)
    try:
        n_items = P.dim0 * P.num_per
        cts = np.concatenate([cl.generate_query((13 * k + 1) % n_items)["ct"] for k in range(17)])
        got = S.process_query_batch(H, gpp, cts, sdb)
        assert np.array_equal(got, S.process_query_batch(G, gpp, cts, gdb))
        assert np.array_equal(_batch_dev(S, H, sdb, gpp, cts), got)
        q = cl.generate_query(3)
        one = S.process_query_bytes(H, gpp, cl.query_bytes(), sdb)
        assert np.array_equal(one[0], P.process_query(pp, q, db))
        assert np.array_equal(sdb.to_words(), db)
    finally:
        sdb.close()


# ------------------------------------------------------------------ writers and readers
def _body(entries):
    out = bytearray()
    for idx, data in entries:
        out += (len(data) + 4).to_bytes(4, "big") + int(idx).to_bytes(4, "big") + bytes(data)
    return bytes(out)


def _same(S, P, cl, gpp, U, udb, H, sdb, what):
    assert np.array_equal(sdb.to_words(), udb.to_words()), what
    su, ss = udb.info(), sdb.info()
    assert (ss["present_items"], ss["capacity"]) == (su["present_items"], su["capacity"]), what
    n_items = P.dim0 * P.num_per
    blobs = []
    for i in (1, n_items - 2):
        cl.generate_query(i)
        blobs.append(cl.query_bytes())
    blob = np.concatenate(blobs)
    assert np.array_equal(S.process_query_bytes(H, gpp, blob, sdb), S.process_query_bytes(U, gpp, blob, udb)), what


@pytest.mark.parametrize("shards", [2])
def test_writers_equal_unsharded(shards, tmp_path):
    S, P, cl, pp, db, G, gdb, gpp = setup_case("T")
    U = S.Params(**P.kw)
    udb = S.Database(U)
    ctxs = _contexts(S, P, [0] * shards)
    H = ctxs[0]
    sdb = S.Database.sharded(ctxs)
    rng = np.random.default_rng(shards)
    n_items = P.dim0 * P.num_per
    span = P.slices * P.bytes_per_chunk
    try:
        # single-item writers on empty databases: presence counts only what was written
        poly = db[:2048].copy()
        for slice_idx, item in ((0, 3), (P.slices - 1, n_items - 1), (1, 6)):
            udb.upsert_item(slice_idx, item, poly)
            sdb.upsert_item(slice_idx, item, poly)
        _same(S, P, cl, gpp, U, udb, H, sdb, "upsert_item")
        for item in (2, 9, n_items - 3):
            data = rng.integers(0, 256, span, dtype=np.uint8)
            udb.update_item_raw(item, data)
            sdb.update_item_raw(item, data)
        _same(S, P, cl, gpp, U, udb, H, sdb, "update_item_raw")
        good = [(int(i), rng.integers(0, 256, span, dtype=np.uint8).tobytes()) for i in (4, 11, 4, 200 % n_items)]
        body = _body(good[:2] + [(n_items + 5, b"\x01" * 8)] + good[2:])          # a bad db_idx mid-body
        codes = []
        for d in (udb, sdb):
            with pytest.raises(S.B200PirError) as ei:
                d.update_many_items(body)
            codes.append(ei.value.code)
        assert codes[0] == codes[1]
        _same(S, P, cl, gpp, U, udb, H, sdb, "update_many_items with a bad entry")
        assert udb.update_many_items(_body(good)) == sdb.update_many_items(_body(good))
        _same(S, P, cl, gpp, U, udb, H, sdb, "update_many_items")
        slice_words = P.dim0 * P.num_per * 2048
        udb.upload_slice(1, db[slice_words:2 * slice_words].copy())
        sdb.upload_slice(1, db[slice_words:2 * slice_words].copy())
        _same(S, P, cl, gpp, U, udb, H, sdb, "upload_slice")
        for d, c in ((udb, U), (sdb, H)):
            S.check(S.LIB.b200pir_db_upload(c._h, d._h, db.ctypes.data, db.size))
        _same(S, P, cl, gpp, U, udb, H, sdb, "upload")
        assert np.array_equal(sdb.download_slice(2), db[2 * slice_words:3 * slice_words])
        udb.fill_synthetic(91)
        sdb.fill_synthetic(91)
        _same(S, P, cl, gpp, U, udb, H, sdb, "fill_synthetic")
        # save_file: the sharded snapshot is the unsharded one, and loads back into an unsharded database
        fu, fs = tmp_path / "u.db", tmp_path / "s.db"
        udb.save_file(fu)
        sdb.save_file(fs)
        assert fu.read_bytes() == fs.read_bytes()
        back = S.Database.from_file(U, fs)
        _same(S, P, cl, gpp, U, back, H, sdb, "save_file round trip")
        back.close()
        # load_file and load_raw_file into fresh databases
        db2 = P.generate_db(4242)
        f2 = tmp_path / "w.db"
        db2.tofile(f2)
        lu, ls = S.Database.from_file(U, f2), S.Database.from_file(H, f2, contexts=ctxs)
        assert np.array_equal(ls.to_words(), db2)
        _same(S, P, cl, gpp, U, lu, H, ls, "load_file")
        lu.close(), ls.close()
        raw = tmp_path / "raw.bin"
        raw.write_bytes(rng.integers(0, 256, (n_items - 7) * P.db_item_size + 11, dtype=np.uint8).tobytes())
        ru, rs = S.Database.from_raw_file(U, raw), S.Database.from_raw_file(H, raw, contexts=ctxs)
        _same(S, P, cl, gpp, U, ru, H, rs, "load_raw_file")
        ru.close(), rs.close()
    finally:
        sdb.close()
        udb.close()


# ------------------------------------------------------------------ concurrent callers
def test_concurrent_single_query_callers_share_batches():
    S, P, cl, pp, db, G, gdb, gpp = setup_case("T")
    ctxs = _contexts(S, P, [0, 0])
    H = ctxs[0]
    sdb = S.Database.from_words(H, db, contexts=ctxs)
    cl_b = O.Client(P, 4321)
    cl_b.generate_keys()
    gpp_b = S.PublicParameters.deserialize(G, cl_b.pp_bytes())
    n_items = P.dim0 * P.num_per
    jobs = []
    for k in range(64):
        c, g = (cl, gpp) if k % 2 == 0 else (cl_b, gpp_b)
        idx = (37 * k + 5) % n_items
        c.generate_query(idx)
        jobs.append((g, c.query_bytes(), c, idx))
    H.set_option("coalesce", 0)
    serial = [S.process_query_bytes(H, g, b, sdb)[0] for g, b, _, _ in jobs]
    H.set_option("coalesce", 1)
    b0, q0 = S.coalesce_stats(H)
    got = [None] * len(jobs)
    errors = []
    start = threading.Barrier(16)

    def worker(t):
        try:
            start.wait()
            for k in range(t * 4, t * 4 + 4):
                g, b, _, _ = jobs[k]
                got[k] = S.process_query_bytes(H, g, b, sdb)[0]
        except Exception as e:            # noqa: BLE001
            errors.append(e)

    threads = [threading.Thread(target=worker, args=(t,)) for t in range(16)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors
    for k, (_, _, c, idx) in enumerate(jobs):
        assert np.array_equal(got[k], serial[k]), k
        assert np.array_equal(c.decode_response(got[k]), P.db_plain_item(SEED_DB, idx)), k
    b1, q1 = S.coalesce_stats(H)
    assert q1 - q0 == len(jobs) and b1 - b0 < len(jobs)
    gpp_b.close()
    sdb.close()


# ------------------------------------------------------------------ refusals
def test_refusals(tmp_path):
    import ctypes as C
    import torch
    S, P, cl, pp, db, G, gdb, gpp = setup_case("T")
    LIB = S.LIB
    ctxs = _contexts(S, P, [0, 0, 0, 0])
    other = S.Params(**dict(P.kw, q2_bits=P.kw["q2_bits"] + 1))
    wide = _contexts(S, P, [0] * 8)
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]

    def create(cs):
        h = C.c_void_p()
        arr = (C.c_void_p * max(1, len(cs)))(*[c._h if c is not None else None for c in cs])
        rc = LIB.b200pir_db_create_sharded(arr, len(cs), C.byref(h))
        assert not h.value
        return rc, LIB.b200pir_last_error().decode()

    assert create([ctxs[0], ctxs[1], ctxs[0], ctxs[2]])[0] == E_BADARG                  # a repeated context
    assert create([ctxs[0], other])[0] == E_BADARG                                       # different parameters
    assert create([ctxs[0], None])[0] == E_BADARG
    h = C.c_void_p()
    assert LIB.b200pir_db_create_sharded(None, 2, C.byref(h)) == E_BADARG
    rank = C.c_void_p()
    assert LIB.b200pir_db_create(ctxs[0]._h, 0, 3, C.byref(rank)) == E_BADARG
    want = LIB.b200pir_last_error().decode()
    assert create(ctxs[:3]) == (E_BADARG, want)                                         # not a power of two
    assert create(wide)[0] == E_BADARG                                                   # 8 shards of num_per = 4 rows
    torch.cuda.synchronize()
    assert abs(torch.cuda.mem_get_info()[0] - free0) < (4 << 20)

    sdb = S.Database.from_words(ctxs[0], db, contexts=ctxs[:2])
    H = ctxs[0]
    with pytest.raises(S.B200PirError) as ei:
        S.multiply_reg_by_database(H, sdb, 0, np.zeros(P.dim0 * 2 * 2048, dtype=np.uint64))
    assert ei.value.code == E_UNSUPPORTED
    buf = torch.zeros(1 << 22, dtype=torch.uint8, device="cuda")
    p = buf.data_ptr()
    assert LIB.b200pir_query_stage_a_dev(H._h, sdb._h, gpp._h, p, 1, p) == E_UNSUPPORTED
    assert LIB.b200pir_first_dim_fold_dev(H._h, sdb._h, p, p, 1, p) == E_UNSUPPORTED
    assert LIB.b200pir_first_dim_fold_images_dev(H._h, sdb._h, p, 1, 1, p, p) == E_UNSUPPORTED
    # rank shards keep their refusal of the one-call query path, and of save_file
    shard = S.Database(G, shard_index=0, shard_count=2)
    with pytest.raises(S.B200PirError) as ei:
        S.process_query(G, gpp, S.Query(ct=cl.generate_query(1)["ct"]), shard)
    assert ei.value.code == E_BADARG
    with pytest.raises(S.B200PirError) as ei:
        shard.save_file(tmp_path / "never.db")
    assert ei.value.code == E_UNSUPPORTED
    shard.close()
    # one shard is an ordinary database on the home context
    single = S.Database.sharded(ctxs[:1])
    assert single.info()["local_rows"] == P.num_per
    single.close()
    sdb.close()
    other.close()
