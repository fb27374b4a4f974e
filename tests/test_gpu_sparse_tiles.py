"""Tile skipping in the wgmma first dimension (database format 2, k_multiply_tc5) on sparse databases.

k_multiply_tc5 is the one kernel whose data movement depends on the data: tile_mask[slice][mt] (one bit per 32-row x 32-j
tile, kept by b200pir_db::mark / mark_items / mark_slice) decides which ring stages the producer fetches, which k-steps the
consumers multiply, and which row tiles are stored as zeros.  Every database written item by item takes this path.  The
products are compared with a numpy reference that sums only the present items, and at the small geometries also with the
oracle on the zero-filled dense slice; responses with the oracle's process_query (both folds) or, where the oracle is slow,
with the same writes on format 1, which does not skip.

Geometries (overrides of T): dim0 x rows, slices, and the ring configuration the launcher picks (tests/test_tc5_protocol_sim.py
models the barriers of each one)."""
import os
import tempfile

import numpy as np
import pytest

import oracle_lib as O
import update_rows_oracle as U
from test_gpu_parity import SEED_DB, Q0, Q1

pytestmark = [pytest.mark.gpu]

N = 2048
M32 = np.uint64(0xFFFFFFFF)
WMAX = np.uint64((Q0 - 1) | ((Q1 - 1) << 32))

GEOMS = {
    "nu1_1": dict(nu_1=1),                                        # 2 x 4, 4 slices: ks = 1, partial k-tile and row tile
    "nu1_4": dict(nu_1=4),                                        # 16 x 4, 4 slices
    "T": dict(),                                                  # 64 x 4, 4 slices: one partial stage
    "T0": dict(O.PARAM_SETS["T0"]),                               # 32 x 8, 9 slices
    "9_6": dict(nu_1=9, nu_2=6, n=1, db_item_size=2048),          # 512 x 64: 2 stages per tile, 2 row tiles
    "9_7": dict(nu_1=9, nu_2=7, n=1, db_item_size=2048),          # 512 x 128: 4 row tiles
    "10_6": dict(nu_1=10, nu_2=6, n=1, db_item_size=2048),        # 1024 x 64: the <4, 1> kernel, 8 stages per tile
}
KSPS = {1024: 4}                                                  # k-steps per ring stage (8 below dim0 = 1024)
PATTERNS = ["empty", "corners", "one k-step per stage", "all k-steps of a stage but one", "last row tile",
            "alternating row tiles", "random 0.001", "random 0.01", "random 0.1", "random 0.5", "full"]
# slices of more than 2^15 items leave out the two densest patterns: 2^15 upserts each, and the dense tests
# (test_gpu_tcgen05.py) already run the full mask at 512 x 128 and 1024 x 64
MAX_DENSE_ITEMS = 1 << 15

_ctx = {}


def kw_of(geom):
    kw = dict(O.PARAM_SETS["T"])
    kw.update(GEOMS[geom])
    return kw


def ctx(geom):
    if geom not in _ctx:
        import sdk_b200.spiral as S
        _ctx[geom] = (S, O.Params(**kw_of(geom)), S.Params(**kw_of(geom)))
    return _ctx[geom]


@pytest.fixture(scope="module", autouse=True)
def _close():
    yield
    for S, P, G in _ctx.values():
        G.close()
    _ctx.clear()


def rand_words(rng, shape):
    return rng.integers(0, Q0, shape, dtype=np.uint64) | (rng.integers(0, Q1, shape, dtype=np.uint64) << np.uint64(32))


def patterns_for(P):
    return [p for p in PATTERNS if P.dim0 * P.num_per <= MAX_DENSE_ITEMS or p not in ("random 0.5", "full")]


def pattern(name, dim0, rows, rng):
    """The (ii, j) items of one slice."""
    ks, mt, ksps = (dim0 + 31) // 32, (rows + 31) // 32, KSPS.get(dim0, 8)
    spt = (ks + ksps - 1) // ksps
    row = lambda m, k: min(rows - 1, 32 * m + k % 32)                    # row k of row tile m
    col = lambda s, k: min(dim0 - 1, 32 * s + k % 32)                    # value k of k-step s
    out = set()
    if name == "corners":
        for m, s in {(0, 0), (mt - 1, ks - 1), (mt // 2, ks // 2)}:
            out |= {(row(m, a), col(s, b)) for a in (0, 31) for b in (0, 31)}
    elif name in ("one k-step per stage", "all k-steps of a stage but one"):
        for m in range(mt):
            for st in range(spt):
                here = min(ksps, ks - st * ksps)
                pick = (st + m) % here
                kks = [pick] if name == "one k-step per stage" else [k for k in range(here) if k != pick]
                out |= {(row(m, 7 * st + k), col(st * ksps + k, 5 * m + 3 * k)) for k in kks}
    elif name == "last row tile":
        out |= {(row(mt - 1, int(rng.integers(32))), col(s, int(rng.integers(32)))) for s in range(ks) for _ in range(2)}
    elif name == "alternating row tiles":                            # even row tiles: every k-step present; odd: empty
        out |= {(row(m, int(rng.integers(32))), col(s, int(rng.integers(32)))) for m in range(0, mt, 2) for s in range(ks)
                for _ in range(3)}
        if mt == 1:
            out |= {(row(0, 31), col(s, 31)) for s in range(ks)}
    elif name.startswith("random"):
        ii, jj = np.nonzero(rng.random((rows, dim0)) < float(name.split()[1]))
        out |= set(zip(ii.tolist(), jj.tolist()))
    elif name == "full":
        out |= {(i, j) for i in range(rows) for j in range(dim0)}
    return out


def sparse_product(P, rows, items, v):
    """multiply_reg_by_database restated over the present items only: out[ii][r][n][z] = sum over present j of
    db[z][ii][j]_n * v[z][j][r]_n mod q_n, every product reduced before it is added (dim0 x 2^28 < 2^64)."""
    out = np.zeros((rows, 2, 2, N), dtype=np.uint64)
    keys = sorted(items)
    V = v.reshape(N, P.dim0, 2)
    for c0 in range(0, len(keys), 2048):
        ck = keys[c0:c0 + 2048]
        ii = np.array([k[0] for k in ck])
        jj = np.array([k[1] for k in ck])
        polys = np.stack([items[k] for k in ck])                          # [K][z]
        starts = np.flatnonzero(np.r_[True, ii[1:] != ii[:-1]])
        for n, q in enumerate((Q0, Q1)):
            sh = np.uint64(32 * n)
            A = (polys >> sh) & M32
            for r in range(2):
                Vn = ((V[:, :, r] >> sh) & M32).T                         # [j][z]
                prod = A * Vn[jj] % np.uint64(q)
                out[ii[starts], r, n, :] += np.add.reduceat(prod, starts, axis=0)
    for n, q in enumerate((Q0, Q1)):
        out[:, :, n, :] %= np.uint64(q)
    return out.reshape(-1)


def dense_slice(P, rows, items):
    """The zero-filled slice in the reference layout [z][ii][j]."""
    d = np.zeros((N, rows, P.dim0), dtype=np.uint64)
    for (ii, j), poly in items.items():
        d[:, ii, j] = poly
    return d.reshape(-1)


def row_counts(P, rows, keys):
    """Product of a database whose present items are all q - 1 with v all q - 1: (q - 1)^2 = 1 mod q, so every output word is
    the number of present items in its row."""
    cnt = np.zeros(rows, dtype=np.uint64)
    for ii, _ in keys:
        cnt[ii] += 1
    return np.broadcast_to(cnt[:, None, None, None], (rows, 2, 2, N)).reshape(-1)


def check_product(S, P, G, db, s, items, v, oracle=False):
    got = S.multiply_reg_by_database(G, db, s, v)
    rows = P.num_per // db.shard_count
    assert np.array_equal(got, sparse_product(P, rows, items, v)), s
    if oracle:
        assert np.array_equal(got, P.multiply_reg_by_database(dense_slice(P, rows, items), v)), s
    return got


# ------------------------------------------------------------------ a. stage-level product
@pytest.mark.parametrize("geom", list(GEOMS))
def test_sparse_patterns_product(geom):
    """Every pattern in some slice (slices of one database differ), random v and worst-case operands.  The worst case rewrites
    every present item with q - 1, which must not change the count of present items."""
    S, P, G = ctx(geom)
    pats = patterns_for(P)
    rng = np.random.default_rng(list(GEOMS).index(geom))
    small = P.dim0 * P.num_per <= 256
    v = rand_words(rng, P.dim0 * 2 * N)
    vmax = np.full(P.dim0 * 2 * N, WMAX, dtype=np.uint64)
    for k in range(0, len(pats), P.slices):
        db = S.Database(G, fmt=2)
        assert db.info()["format"] == 2 and db.info()["present_items"] == 0
        per_slice = []
        for s in range(P.slices):
            keys = pattern(pats[(k + s) % len(pats)], P.dim0, P.num_per, rng)
            items = {key: rand_words(rng, N) for key in keys}
            for (ii, j), poly in items.items():
                db.upsert_item(s, j * P.num_per + ii, poly)
            per_slice.append(items)
        assert db.info()["present_items"] == sum(len(it) for it in per_slice)
        for s, items in enumerate(per_slice):
            check_product(S, P, G, db, s, items, v, oracle=small)
        for s, items in enumerate(per_slice):
            for ii, j in items:
                db.upsert_item(s, j * P.num_per + ii, np.full(N, WMAX, dtype=np.uint64))
        assert db.info()["present_items"] == sum(len(it) for it in per_slice)
        for s, items in enumerate(per_slice):
            assert np.array_equal(S.multiply_reg_by_database(G, db, s, vmax), row_counts(P, P.num_per, items)), (geom, s)
        db.close()


def test_tc5_sparse_database_skips_absent_tiles():
    """lib/server's SparseDb semantics as cost (db/sparse_db.rs:5-47, compute/dot_product.rs:35): an item exists once written;
    tiles (32 rows x 32 values of j) without a present item are neither fetched nor multiplied.  512 x 64 geometry = 16 k-steps
    in two 8-step ring stages x 2 row tiles: patterns with a completely empty database, an empty row tile, an empty ring
    stage, single k-steps inside a stage; the product must equal the oracle's on the zero-filled database every time."""
    S, P, G = ctx("9_6")
    rng = np.random.default_rng(77)
    v = rand_words(rng, P.dim0 * 2 * P.N)
    tdb = S.Database(G, fmt=2)
    info = tdb.info()
    assert info["format"] == 2 and info["present_items"] == 0 and info["capacity"] == P.dim0 * P.num_per
    dense = np.zeros((P.N, P.num_per, P.dim0), dtype=np.uint64)             # reference layout [z][ii][j] of the one slice
    assert not S.multiply_reg_by_database(G, tdb, 0, v).any()              # nothing present: all-zero product, no tile touched
    placed = 0
    # (j, ii): one k-step of stage 0 in row tile 0; then stage 1 only in row tile 1; then neighbours inside present tiles
    for j, ii in [(37, 3), (300, 40), (301, 63), (37, 4), (0, 0), (511, 63), (255, 31), (256, 32)]:
        poly = rand_words(rng, P.N)
        tdb.upsert_item(0, j * P.num_per + ii, poly)
        dense[:, ii, j] = poly
        placed += 1
        assert tdb.info()["present_items"] == placed
        assert np.array_equal(S.multiply_reg_by_database(G, tdb, 0, v), P.multiply_reg_by_database(dense.reshape(-1), v)), (j, ii)
    tdb.upsert_item(0, 37 * P.num_per + 3, dense[:, 3, 37].copy())          # rewriting an item does not count twice
    assert tdb.info()["present_items"] == placed
    # bulk upload marks everything present
    full = S.Database.from_words(G, dense.reshape(-1), fmt=2)
    assert full.info()["present_items"] == P.dim0 * P.num_per
    assert np.array_equal(S.multiply_reg_by_database(G, full, 0, v), P.multiply_reg_by_database(dense.reshape(-1), v))
    full.close()
    tdb.close()


# ------------------------------------------------------------------ b. writers
def written(P, rng, patterns, rewrites=0.25):
    """(entries [(db_idx, bytes)] in write order, with a share of the items written twice, and {db_idx: [slices][N] polys} of
    the last write of each)."""
    full = P.slices * P.bytes_per_chunk
    idxs = sorted({j * P.num_per + ii for name in patterns for ii, j in pattern(name, P.dim0, P.num_per, rng)})
    entries = [(i, rng.integers(0, 256, full, dtype=np.uint8).tobytes()) for i in idxs]
    again = [e[0] for e in entries if rng.random() < rewrites]
    entries += [(i, rng.integers(0, 256, full, dtype=np.uint8).tobytes()) for i in again]
    last = {i: P.update_item_raw(np.frombuffer(d, dtype=np.uint8)).reshape(P.slices, N) for i, d in entries}
    return entries, last


def slice_items(P, last, s, shard=(0, 1)):
    r, g = shard
    return {(i % P.num_per // g, i // P.num_per): polys[s] for i, polys in last.items() if i % P.num_per % g == r}


@pytest.mark.parametrize("geom", ["T", "T0", "9_6"])
def test_writers_build_the_same_sparse_database(geom):
    """upsert_item (per slice), update_item_raw and update_many_items: identical products, and present_items counts the
    distinct (slice, row, j) written, so a rewrite does not count twice."""
    S, P, G = ctx(geom)
    rng = np.random.default_rng(5)
    v = rand_words(rng, P.dim0 * 2 * N)
    for pats in (["corners", "one k-step per stage", "random 0.01"], ["last row tile", "all k-steps of a stage but one"]):
        entries, last = written(P, rng, pats)
        dbs = [S.Database(G, fmt=2) for _ in range(3)]
        for i, d in entries:
            polys = P.update_item_raw(np.frombuffer(d, dtype=np.uint8)).reshape(P.slices, N)
            for s in range(P.slices):
                dbs[0].upsert_item(s, i, np.ascontiguousarray(polys[s]))
            dbs[1].update_item_raw(i, np.frombuffer(d, dtype=np.uint8))
        dbs[2].update_many_items(b"".join(U.entry(i, d) for i, d in entries))
        for db in dbs:
            assert db.info()["present_items"] == P.slices * len(last), (geom, pats)
        for s in range(P.slices):
            items = slice_items(P, last, s)
            ref = check_product(S, P, G, dbs[0], s, items, v, oracle=P.dim0 * P.num_per <= 256)
            for db in dbs[1:]:
                assert np.array_equal(S.multiply_reg_by_database(G, db, s, v), ref), (geom, pats, s)
        for db in dbs:
            db.close()


# ------------------------------------------------------------------ c. mixed presence
def test_bulk_writes_over_a_sparse_database():
    S, P, G = ctx("T")
    rng = np.random.default_rng(9)
    v = rand_words(rng, P.dim0 * 2 * N)
    db = S.Database(G, fmt=2)
    per_slice = []
    for s in range(P.slices):
        items = {k: rand_words(rng, N) for k in pattern(["corners", "random 0.1", "empty", "one k-step per stage"][s], P.dim0,
                                                          P.num_per, rng)}
        for (ii, j), poly in items.items():
            db.upsert_item(s, j * P.num_per + ii, poly)
        per_slice.append(items)
    sparse_count = sum(len(it) for it in per_slice)
    assert db.info()["present_items"] == sparse_count
    refs = [S.multiply_reg_by_database(G, db, s, v) for s in range(P.slices)]
    # a snapshot loaded back is a dense database: every item present, the same products
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "db.bin")
        db.save_file(path)
        loaded = S.Database.from_file(G, path, fmt=2)
    assert loaded.info()["present_items"] == loaded.info()["capacity"]
    for s in range(P.slices):
        assert np.array_equal(S.multiply_reg_by_database(G, loaded, s, v), refs[s]), s
    loaded.close()
    # upload_slice makes its slice full and leaves the others sparse
    words = rand_words(rng, P.dim0 * P.num_per * N)
    db.upload_slice(2, words)
    per_slice[2] = {(ii, j): words.reshape(N, P.num_per, P.dim0)[:, ii, j].copy() for ii in range(P.num_per) for j in range(P.dim0)}
    assert db.info()["present_items"] == sparse_count + P.dim0 * P.num_per          # slice 2 was empty
    for s in range(P.slices):
        check_product(S, P, G, db, s, per_slice[s], v, oracle=True)
    # a synthetic fill makes every item present and gives the products of the fully synthetic database
    db.fill_synthetic(SEED_DB)
    assert db.info()["present_items"] == db.info()["capacity"]
    syn = P.generate_db(SEED_DB).reshape(P.slices, -1)
    for s in range(P.slices):
        assert np.array_equal(S.multiply_reg_by_database(G, db, s, v), P.multiply_reg_by_database(syn[s], v)), s
    db.close()


# ------------------------------------------------------------------ d, e, g. responses
def sparse_db_set(S, P, G, rng, fmts):
    """The same per-slice patterns written with upsert_item on each format in `fmts` -> ({fmt: db}, dense reference words)."""
    dbs = {f: S.Database(G, fmt=f) for f in fmts}
    dense = np.zeros((P.slices, N, P.num_per, P.dim0), dtype=np.uint64)
    names = ["empty", "alternating row tiles", "one k-step per stage", "random 0.1", "corners", "last row tile",
             "all k-steps of a stage but one", "random 0.01", "random 0.5"]
    for s in range(P.slices):
        for ii, j in pattern(names[s % len(names)], P.dim0, P.num_per, rng):
            poly = rand_words(rng, N)
            dense[s, :, ii, j] = poly
            for db in dbs.values():
                db.upsert_item(s, j * P.num_per + ii, poly)
    return dbs, dense.reshape(-1)


def keys_for(name, P):
    cl = O.Client(P, 4242)
    pp = cl.generate_keys()
    import sdk_b200.spiral as S
    G = ctx(name)[2]
    return cl, pp, S.PublicParameters(G, pp["pack"], pp.get("left"), pp.get("right"), pp.get("conv"))


COUNTS = (1, 5, 16, 17)                                     # 17 = 16 + 1: two database passes


def run_counts(S, G, gpp, qs, db, sparse_fold):
    G.set_option("sparse_fold", sparse_fold)
    try:
        return {c: S.process_query_batch(G, gpp, qs[:c * 2 * N], db) for c in COUNTS}
    finally:
        G.set_option("sparse_fold", 0)


def test_responses_on_sparse_databases_T():
    """Query counts 1, 5, 16 and 17 with both folds, after a batch on a dense format-2 database has left its values in the
    workspace (absent row tiles must be stored as zeros); response bytes equal the oracle's, formats 0, 1 and 2 agree, and
    a database written with update_many_items decodes to the written bytes."""
    S, P, G = ctx("T")
    cl, pp, gpp = keys_for("T", P)
    rng = np.random.default_rng(13)
    dbs, dense = sparse_db_set(S, P, G, rng, (2, 1, 0))
    full_db = S.Database.from_words(G, rand_words(rng, dense.size), fmt=2)
    idxs = [int(i) for i in rng.choice(P.dim0 * P.num_per, COUNTS[-1], replace=False)]
    qs = np.concatenate([cl.generate_query(i)["ct"] for i in idxs])
    v = rand_words(rng, P.dim0 * 2 * N)
    for s in range(P.slices):                                  # g. products of the three formats
        ref = S.multiply_reg_by_database(G, dbs[2], s, v)
        assert np.array_equal(ref, P.multiply_reg_by_database(dense.reshape(P.slices, -1)[s], v)), s
        for f in (0, 1):
            assert np.array_equal(S.multiply_reg_by_database(G, dbs[f], s, v), ref), (f, s)
    for sparse_fold in (0, 1):
        S.process_query_batch(G, gpp, qs, full_db)             # e. a dirty workspace
        got = run_counts(S, G, gpp, qs, dbs[2], sparse_fold)
        refs = [P.process_query(pp, dict(ct=qs[k * 2 * N:(k + 1) * 2 * N]), dense, sparse_fold=bool(sparse_fold))
                for k in range(COUNTS[-1])]
        for c, out in got.items():
            for k in range(c):
                assert np.array_equal(out[k], refs[k]), (sparse_fold, c, k)
        for f in (1, 0):
            other = run_counts(S, G, gpp, qs, dbs[f], sparse_fold)
            for c in COUNTS:
                assert np.array_equal(other[c], got[c]), (f, sparse_fold, c)
    # written with the /update-row path: decodes (version 0 decodes with both folds, test_gpu_written_decode.py)
    entries, last = written(P, rng, ["alternating row tiles", "random 0.1"], rewrites=0.0)
    wdb = S.Database(G, fmt=2)
    wdb.update_many_items(b"".join(U.entry(i, d) for i, d in entries))
    wdense, _, err, applied = U.update_many_items(P, b"".join(U.entry(i, d) for i, d in entries))
    assert err is None
    items = dict(applied)
    targets = sorted(items)[:COUNTS[-1]]
    wqs = np.concatenate([cl.generate_query(i)["ct"] for i in targets])
    for sparse_fold in (0, 1):
        S.process_query_batch(G, gpp, qs, full_db)
        got = run_counts(S, G, gpp, wqs, wdb, sparse_fold)
        for k, idx in enumerate(targets):
            ref = P.process_query(pp, dict(ct=wqs[k * 2 * N:(k + 1) * 2 * N]), wdense.reshape(-1), sparse_fold=bool(sparse_fold))
            assert np.array_equal(got[COUNTS[-1]][k], ref), (sparse_fold, idx)
            dec = cl.decode_response(got[COUNTS[-1]][k]).reshape(P.slices, N)[:, :P.bytes_per_chunk].astype(np.uint8).reshape(-1)
            assert np.array_equal(dec, U.read_back(P, wdense, items, idx, bool(sparse_fold))), (sparse_fold, idx)
    for db in list(dbs.values()) + [full_db, wdb, gpp]:
        db.close()


def test_responses_on_sparse_database_512x128():
    """4 row tiles, alternating empty and present: after a dense batch on the same context, responses equal those of the same
    writes on format 1, which does not skip."""
    S, P, G = ctx("9_7")
    cl, pp, gpp = keys_for("9_7", P)
    rng = np.random.default_rng(17)
    keys = pattern("alternating row tiles", P.dim0, P.num_per, rng) | pattern("random 0.01", P.dim0, P.num_per, rng)
    keys = {k for k in keys if (k[0] // 32) % 2 == 0}           # row tiles 1 and 3 stay empty
    d2, d1 = S.Database(G, fmt=2), S.Database(G, fmt=1)
    for ii, j in keys:
        poly = rand_words(rng, N)
        d2.upsert_item(0, j * P.num_per + ii, poly)
        d1.upsert_item(0, j * P.num_per + ii, poly)
    full_db = S.Database(G, fmt=2)
    full_db.fill_synthetic(3)
    idxs = [int(i) for i in rng.choice(P.dim0 * P.num_per, COUNTS[-1], replace=False)]
    qs = np.concatenate([cl.generate_query(i)["ct"] for i in idxs])
    for sparse_fold in (0, 1):
        S.process_query_batch(G, gpp, qs, full_db)
        got = run_counts(S, G, gpp, qs, d2, sparse_fold)
        ref = run_counts(S, G, gpp, qs, d1, sparse_fold)
        for c in COUNTS:
            assert np.array_equal(got[c], ref[c]), (sparse_fold, c)
    for h in (d2, d1, full_db, gpp):
        h.close()


# ------------------------------------------------------------------ f. shards
@pytest.mark.parametrize("shards", [2, 4])
def test_sharded_sparse_database(shards):
    """A shard holds rows ii = il * G + r: one of its tiles holds rows that are G apart.  Every shard gets every write; shard
    r keeps its own rows, counts only those, and its product is rows r::G of the unsharded product."""
    S, P, G = ctx("9_7")
    rng = np.random.default_rng(19 + shards)
    v = rand_words(rng, P.dim0 * 2 * N)
    keys = set()
    for name in ("corners", "one k-step per stage", "last row tile", "random 0.01"):
        keys |= pattern(name, P.dim0, P.num_per, rng)
    items = {k: rand_words(rng, N) for k in keys}
    whole = S.Database(G, fmt=2)
    parts = [S.Database(G, shard_index=r, shard_count=shards, fmt=2) for r in range(shards)]
    for (ii, j), poly in items.items():
        for db in [whole] + parts:
            db.upsert_item(0, j * P.num_per + ii, poly)
    ref = check_product(S, P, G, whole, 0, items, v).reshape(P.num_per, -1)
    for r, db in enumerate(parts):
        assert db.info()["present_items"] == sum(1 for ii, _ in keys if ii % shards == r), r
        got = S.multiply_reg_by_database(G, db, 0, v).reshape(P.num_per // shards, -1)
        assert np.array_equal(got, ref[r::shards]), r
    for db in [whole] + parts:
        db.close()
