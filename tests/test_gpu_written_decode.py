"""Private reads of databases built on the GPU by the write path (b200pir_db_update_many_items, the /update-row body, and
b200pir_db_update_item_raw, /write), on every database format and with both folds: response bytes equal the CPU oracle's over
the restated database (tests/update_rows_oracle.py), and the response decodes to the bytes the fold reads back
(update_rows_oracle.read_back: the written bytes, except where lib/server's fold meets an empty row).  The decode check does
not depend on the oracle.  The dense fold is decoded where it keeps its margin, on version 0; on version 1 it is compared
with the oracle only (tests/test_oracle_written_items_decode.py pins why)."""
import numpy as np
import pytest

import oracle_lib as O
import update_rows_oracle as U
from test_oracle_written_items_decode import _layouts

pytestmark = pytest.mark.gpu

_cache = {}


def setup_case(name):
    if name not in _cache:
        import sdk_b200.spiral as S
        P = O.Params.named(name)
        cl = O.Client(P, 4242)
        pp = cl.generate_keys()
        G = S.Params(**P.kw)
        gpp = S.PublicParameters(G, pp["pack"], pp.get("left"), pp.get("right"), pp.get("conv"))
        _cache[name] = (S, P, cl, pp, G, gpp, {})
    return _cache[name]


@pytest.fixture(scope="module", autouse=True)
def _close():
    yield
    for S, P, cl, pp, G, gpp, _ in _cache.values():
        gpp.close()
        G.close()
    _cache.clear()


def _reads(P, cl, pp, refs, name, layout, items, sparse):
    """(query, oracle response, expected decoded bytes) for every item of a layout; computed once per fold."""
    key = (layout, sparse)
    if key not in refs:
        db, _, err, applied = U.update_many_items(P, b"".join(U.entry(i, d) for i, d in items))
        assert err is None
        written = dict(applied)
        out = []
        for idx in sorted(written):
            q = cl.generate_query(idx)
            out.append((idx, q, P.process_query(pp, q, db.reshape(-1), sparse_fold=sparse),
                        U.read_back(P, db, written, idx, sparse)))
        refs[key] = out
    return refs[key]


@pytest.mark.parametrize("path", ["update_many_items", "update_item_raw"])
@pytest.mark.parametrize("sparse_fold", [0, 1])
@pytest.mark.parametrize("fmt", [0, 1, 2])
@pytest.mark.parametrize("name", ["T", "T1", "T0"])
def test_written_layouts_read_back(name, fmt, sparse_fold, path):
    S, P, cl, pp, G, gpp, refs = setup_case(name)
    decode = sparse_fold == 1 or P.version == 0
    for layout, items in _layouts(P).items():
        gdb = S.Database(G, fmt=fmt)
        if path == "update_many_items":
            gdb.update_many_items(b"".join(U.entry(i, d) for i, d in items))
        else:
            for i, d in items:
                gdb.update_item_raw(i, np.frombuffer(d, dtype=np.uint8))
        G.set_option("sparse_fold", sparse_fold)
        try:
            for idx, q, ref, exp in _reads(P, cl, pp, refs, name, layout, items, bool(sparse_fold)):
                resp = S.process_query(G, gpp, S.Query(ct=q["ct"]), gdb)
                what = (name, fmt, sparse_fold, path, layout, idx)
                assert np.array_equal(resp, ref), what
                if decode:
                    got = cl.decode_response(resp).reshape(P.slices, P.N)[:, :P.bytes_per_chunk].astype(np.uint8).reshape(-1)
                    assert np.array_equal(got, exp), what + (int(np.count_nonzero(got != exp)),)
        finally:
            G.set_option("sparse_fold", 0)                            # the context's default
            gdb.close()


def test_e1_written_items_decode_through_serialized_queries():
    """E1 (the reference's version-1 parameters, 2^14 items of 32 KiB, 4 instances) at full size: 384 items written in one
    /update-row body, 32 of them read with serialized queries through process_query_bytes (two batches of 16) and decoded.
    Read with lib/server's fold ("sparse_fold"), the one version-1 parameters are served with.  Every item is full, so each
    target's row is populated in every slice and that fold returns the target."""
    import sdk_b200.spiral as S
    P = O.Params.named("E1")
    cl = O.Client(P, 7)
    cl.generate_keys()
    G = S.Params(**P.kw)
    gpp = S.PublicParameters.deserialize(G, cl.pp_bytes())            # the setup bytes lib/server receives
    rng = np.random.default_rng(31)
    num_items = P.dim0 * P.num_per
    idxs = rng.choice(np.arange(1, num_items - 1), 384, replace=False)
    idxs[:2] = (0, num_items - 1)                                     # the first and the last db_idx, each written once
    items = rng.integers(0, 256, (idxs.size, P.slices * P.bytes_per_chunk), dtype=np.uint8)
    gdb = S.Database(G)
    assert gdb.update_many_items(b"".join(U.entry(int(i), items[k]) for k, i in enumerate(idxs))) == 4 + items.shape[1]
    reads = list(range(0, idxs.size, idxs.size // 32))[:32]
    blobs = []
    for k in reads:
        cl.generate_query(int(idxs[k]))
        blobs.append(cl.query_bytes())
    G.set_option("sparse_fold", 1)
    out = S.process_query_bytes(G, gpp, np.concatenate(blobs), gdb)
    for n, k in enumerate(reads):
        got = cl.decode_response(out[n]).reshape(P.slices, P.N)[:, :P.bytes_per_chunk].astype(np.uint8).reshape(-1)
        assert np.array_equal(got, items[k]), (k, int(idxs[k]), int(np.count_nonzero(got != items[k])))
    for h in (gdb, gpp, G):
        h.close()
