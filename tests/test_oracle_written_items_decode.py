"""Decode-level checks of databases built by the write path (update_item_raw / update_many_items, lib/server's /write and
/update-row), on the CPU oracle alone.

Every other parity test compares the CUDA path with the oracle, so a mistake both make is invisible to them.  Decoding is the
check that does not depend on the oracle: the client must get back the bytes that were written.  Each written item of a small
database is read through process_query and decode_response and compared byte for byte, and the decryption margin is measured
exactly at every stage:
- the numerators decode_response rounds (client.rs:780-800), recomputed with integers;
- the dim0 expanded first-dimension ciphertexts (one-hot selection of the target column);
- each second-dimension row's first-dimension output (that row's item at the target column), every slice;
- the folded ciphertext of every slice (the target item).

Margins are in units of half a rounding interval: a coefficient decodes right while its error stays below 1.

The layouts are the ones that matter for the fold: a second-dimension row that is all-zero in a slice next to one that is
not.  spiral-rs's dense fold leaves an uncancelled error term there (the unsigned gadget digits of the non-zero ciphertext
have a non-zero mean, and only the pair's other, non-zero, product cancels it).  With t_gsw = 8 (T, T0) that term uses up
to 0.13 of the margin at the fold; with t_gsw = 7 (version 1: T1, E1) it uses 0.98, and bytes flip.  lib/server, the only
server of version-1 parameters, short-cuts all-zero ciphertexts in its fold ("sparse_fold"), so version-1 databases are read
with that fold here; version-0 databases are read with both.
"""
import numpy as np
import pytest

import oracle_lib as O
import update_rows_oracle as U

# Largest margin use allowed, per stage, in half rounding intervals.  Measured on the full synthetic database (generate_db,
# every item populated, item 17; test_synthetic_database_margins), the largest values over T, T0, T1 and T1 with
# instances = 1 are: expanded slots 1.0e-6, first-dimension rows 0.007, folded 0.098, decoded response 0.33 (rounding the
# response to q1 = 4p alone can use 0.25 of it).  Each bound sits well above its measurement and below 1.
SLOT_BOUND = 1e-3
ROW_BOUND = 0.05
FOLD_BOUND = 0.25
DECODE_BOUND = 0.5

NAMES = ["T", "T0", "T1", "T1_i1"]


def params(name):
    if name == "T1_i1":                                 # version 1, one instance
        return O.Params.named("T1", instances=1, db_item_size=8192)
    return O.Params.named(name)


_cache = {}


def setup(name):
    if name not in _cache:
        P = params(name)
        cl = O.Client(P, 4242)
        _cache[name] = (P, cl, cl.generate_keys())
    return _cache[name]


def at(P, ii, j):
    """db_idx of the item in second-dimension row ii and first-dimension column j."""
    return j * P.num_per + ii


def plain_items(P, data):
    """The written bytes as the [slices][N] plaintext update_item_raw encodes, recentred to (-p/2, p/2]."""
    buf = np.zeros(P.slices * P.bytes_per_chunk, dtype=np.int64)
    buf[:len(data)] = np.frombuffer(bytes(data), dtype=np.uint8)
    m = np.zeros((P.slices, P.N), dtype=np.int64)
    m[:, :P.bytes_per_chunk] = buf.reshape(P.slices, P.bytes_per_chunk)
    return np.where(m >= P.p // 2, m - P.p, m)


def _layouts(P):
    """name -> list of (db_idx, bytes).  Items placed in distinct rows and columns unless the layout says otherwise."""
    rng = np.random.default_rng(21)
    full = P.slices * P.bytes_per_chunk
    rnd = lambda: rng.integers(0, 256, full, dtype=np.uint8).tobytes()
    last = P.dim0 * P.num_per - 1
    one = np.zeros(full, dtype=np.uint8)
    one[(P.slices - 1) * P.bytes_per_chunk + 5] = 0x9C            # one non-zero byte, in the last slice
    out = {
        "lone": [(at(P, 1, 4), rnd())],
        "same column": [(at(P, 1, 4), rnd()), (at(P, 0, 4), rnd())],
        "same row": [(at(P, 1, 4), rnd()), (at(P, 1, 9), rnd())],
        "neither": [(at(P, 1, 4), rnd()), (at(P, 0, 10), rnd())],
        "first and last": [(0, rnd()), (last, rnd())],
        "one byte": [(at(P, 2, 7), one.tobytes()), (at(P, 0, 10), rnd())],
        "short": [(at(P, 1, 4), rnd()[:100]), (at(P, 0, 10), rnd())],
    }
    for b in (0x00, 0x7F, 0x80, 0xFF):
        out["bytes %02x" % b] = [(at(P, 3, 5), bytes([b]) * full), (at(P, 0, 10), rnd())]
    return out


LAYOUTS = list(_layouts(O.Params.named("T")))


def _centred(x, mod):
    x = np.asarray(x, dtype=np.int64) % mod
    return np.where(x > mod // 2, x - mod, x)


def _noise(P, dec, msg):
    """max |dec - scale * msg| (mod q, centred) in half rounding intervals (scale / 2)."""
    scale = P.modulus // P.p
    err = _centred(np.asarray(dec, dtype=np.int64) - _centred(msg * scale, P.modulus), P.modulus)
    return float(np.abs(err).max()) / (scale / 2)


def _slot_ct(P, v_firstdim, j):
    """First-dimension ciphertext j of the reoriented [z][j][r] (lo | hi << 32) buffer, as an NTT 2x1 matrix."""
    w = v_firstdim.reshape(P.N, P.dim0, 2)[:, j, :]
    ct = np.zeros(2 * P.W, dtype=np.uint64)
    for r in range(2):
        ct[r * P.W:r * P.W + P.N] = w[:, r] & np.uint64(0xFFFFFFFF)
        ct[r * P.W + P.N:(r + 1) * P.W] = w[:, r] >> np.uint64(32)
    return ct


def decode_margin(P, cl, resp, msg):
    """Recompute decode_response's rounding from its numerators with integers; returns (decoded [slices][N] mod p, margin
    against the expected plaintext `msg` [slices][N])."""
    num = cl.decode_numerators(resp).astype(np.int64).reshape(P.slices, P.N)
    denom = P.q2 * 4                                                # q2 * (q1 / p), q1 = 4p
    # client.rs: (r + sign(r) * (denom / 2)) / denom, truncating, then mod p
    q = (np.abs(num) + denom // 2) // denom * np.sign(num)
    decoded = q % P.p
    err = _centred(num - msg * denom, P.p * denom)
    return decoded, float(np.abs(err).max()) / (denom / 2)


def stage_margins(P, cl, pp, db, items_at, target, sparse_fold=False):
    """(slot, row, fold, decode) margins and the decoded [slices][N] plaintext of reading `target` from `db`.  items_at:
    (row ii, column j) -> [slices][N] recentred plaintext of every populated item; absent items are zero."""
    ii, jt = target % P.num_per, target // P.num_per
    zero = np.zeros((P.slices, P.N), dtype=np.int64)
    msg = items_at.get((ii, jt), zero)
    q = cl.generate_query(target)
    resp, d = P.process_query(pp, q, db.reshape(-1), dump=True, sparse_fold=sparse_fold)
    slot = 0.0
    for j in range(P.dim0):
        sel = np.zeros(P.N, dtype=np.int64)
        sel[0] = 1 if j == jt else 0
        slot = max(slot, _noise(P, cl.decrypt_reg(_slot_ct(P, d["v_firstdim"], j)), sel))
    dbs = db.reshape(P.slices, P.N, P.num_per, P.dim0)
    row = 0.0
    for s in range(P.slices):
        out = P.multiply_reg_by_database(np.ascontiguousarray(dbs[s]).reshape(-1), d["v_firstdim"]).reshape(P.num_per, -1)
        for r in range(P.num_per):
            row = max(row, _noise(P, cl.decrypt_reg(np.ascontiguousarray(out[r])), items_at.get((r, jt), zero)[s]))
    folded = d["folded"].reshape(P.slices, 2 * P.N)
    fold = max(_noise(P, cl.decrypt_reg(P.to_ntt(folded[s])), msg[s]) for s in range(P.slices))
    decoded, dec = decode_margin(P, cl, resp, msg)
    assert np.array_equal(decoded.reshape(-1), cl.decode_response(resp).astype(np.int64)), "integer rounding != decode_response"
    return slot, row, fold, dec, decoded


def written_db(P, items):
    """update_rows_oracle's host database after one /update-row body of `items`, and the plaintext of every written item
    keyed by (row ii, column j)."""
    body = b"".join(U.entry(idx, data) for idx, data in items)
    db, _, err, applied = U.update_many_items(P, body)
    assert err is None and len(applied) == len(items)
    return db, {(idx % P.num_per, idx // P.num_per): plain_items(P, data) for idx, data in applied}


# (parameter set, lib/server's fold): both folds on version 0, lib/server's on version 1 (T1, T1_i1)
FOLDS = [("T", False), ("T", True), ("T0", False), ("T0", True), ("T1", True), ("T1_i1", True)]


@pytest.mark.parametrize("layout", LAYOUTS)
@pytest.mark.parametrize("name,sparse_fold", FOLDS)
def test_written_items_decode(name, sparse_fold, layout):
    P, cl, pp = setup(name)
    items = _layouts(P)[layout]
    db, items_at = written_db(P, items)
    for idx, data in items:
        msg = plain_items(P, data)
        slot, row, fold, dec, decoded = stage_margins(P, cl, pp, db, items_at, idx, sparse_fold)
        what = (name, sparse_fold, layout, idx, "slot %.3g row %.3g fold %.3g decode %.3g" % (slot, row, fold, dec))
        got = decoded[:, :P.bytes_per_chunk].astype(np.uint8).reshape(-1)[:len(data)]
        assert np.array_equal(got, np.frombuffer(data, dtype=np.uint8)), what
        assert np.array_equal(decoded, msg % P.p), what
        assert slot < SLOT_BOUND and row < ROW_BOUND and fold < FOLD_BOUND and dec < DECODE_BOUND, what


@pytest.mark.parametrize("name", NAMES)
def test_synthetic_database_margins(name):
    """The measurement the bounds come from: every item populated, so no fold pairs a zero ciphertext."""
    P, cl, pp = setup(name)
    seed, idx = 0xB1755, 17
    db = P.generate_db(seed)
    items_at = {}
    for r in range(P.num_per):                      # the rows the first dimension selects for column idx // num_per
        m = P.db_plain_item(seed, at(P, r, idx // P.num_per)).astype(np.int64).reshape(P.slices, P.N)
        items_at[(r, idx // P.num_per)] = np.where(m >= P.p // 2, m - P.p, m)
    slot, row, fold, dec, decoded = stage_margins(P, cl, pp, db, items_at, idx)
    assert np.array_equal(decoded, P.db_plain_item(seed, idx).astype(np.int64).reshape(P.slices, P.N))
    print(name, "synthetic database: slot %.3g row %.3g fold %.3g decode %.3g" % (slot, row, fold, dec))
    assert slot < SLOT_BOUND and row < ROW_BOUND and fold < FOLD_BOUND and dec < DECODE_BOUND, (slot, row, fold, dec)


@pytest.mark.parametrize("name,loses", [("T", False), ("T0", False), ("T1", True), ("T1_i1", True)])
def test_dense_fold_margin_next_to_an_empty_row(name, loses):
    """Why version 1 is read with lib/server's fold: under spiral-rs's dense fold, an item whose row's fold partner is all-zero keeps
    its margin with t_gsw = 8 but loses it with t_gsw = 7.  The first dimension is unaffected; the fold stage is where the
    margin goes."""
    P, cl, pp = setup(name)
    items = _layouts(P)["neither"]
    db, items_at = written_db(P, items)
    idx, data = items[0]
    slot, row, fold, dec, decoded = stage_margins(P, cl, pp, db, items_at, idx, sparse_fold=False)
    print(name, "dense fold: slot %.3g row %.3g fold %.3g decode %.3g" % (slot, row, fold, dec))
    assert slot < SLOT_BOUND and row < ROW_BOUND, (slot, row)
    assert (fold > 0.5) == loses, (name, fold, dec)


@pytest.mark.parametrize("name,sparse_fold", FOLDS)
def test_every_item_of_an_update_row_body_reads_back(name, sparse_fold):
    """One /update-row body with short, empty, rewritten and full entries: every db_idx it names decodes to what
    update_rows_oracle.read_back predicts for the fold.  That is the written bytes under the dense fold; lib/server's fold
    differs from them only in slices where the target's row is empty.  The dense fold is checked where it keeps its margin
    (version 0; on version 1 it does not, test_dense_fold_margin_next_to_an_empty_row)."""
    P, cl, pp = setup(name)
    rng = np.random.default_rng(11)
    full = P.slices * P.bytes_per_chunk
    last = P.dim0 * P.num_per - 1
    plan = [(17, full), (0, 100), (last, 0), (17, 5), (40, full - 1), (last, full), (3, 2049), (17, 777), (1, 0)]
    body = b"".join(U.entry(idx, rng.integers(0, 256, n, dtype=np.uint8)) for idx, n in plan)
    db, _, err, applied = U.update_many_items(P, body)
    items = dict(applied)
    for idx in sorted(items):
        resp = P.process_query(pp, cl.generate_query(idx), db.reshape(-1), sparse_fold=sparse_fold)
        got = cl.decode_response(resp).reshape(P.slices, P.N)[:, :P.bytes_per_chunk].astype(np.uint8).reshape(-1)
        exp = U.read_back(P, db, items, idx, sparse_fold)
        assert np.array_equal(got, exp), (name, sparse_fold, idx, int(np.count_nonzero(got != exp)))
        if not sparse_fold:
            assert np.array_equal(exp[:items[idx].size], items[idx]) and not exp[items[idx].size:].any()
