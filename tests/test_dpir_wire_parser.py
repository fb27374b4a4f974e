"""CPU-only: the DoublePIR wire parser (sdk_b200/csrc/dpir_wire.hpp, run through tests/cpp/dpir_wire_check.cpp) against a
restatement of serializer.rs and of the checks answer() makes (doublepir.rs:246-350): which requests are refused, where each
q_1 / q_2 lies in the request, and the response's framing."""
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MAX_LEN = 1 << 28                                                   # serializer.rs:8
E_SHAPE = -2


class Panic(Exception):
    pass


# ---- serializer.rs restated --------------------------------------------------------------------------------------------
def ser_matrix(rows, cols, data=None):                                # Matrix::serialize, serializer.rs:56-66
    data = np.zeros(rows * cols, dtype=np.uint32) if data is None else np.asarray(data, dtype=np.uint32).reshape(-1)
    return rows.to_bytes(4, "big") + cols.to_bytes(4, "big") + data.astype(">u4").tobytes()


def ser_vec(items):                                                   # Vec<T>::serialize, :85-94
    return len(items).to_bytes(4, "big") + b"".join(items)


def walk(req, e, c1):
    """Vec::<State>::deserialize (:68-107, read_u32_iter's unwrap and MAX_LEN asserts), then answer()'s reads: 1 + e matrices a
    query, each q_2 of 3 c1 x 1.  Returns [[(pos, rows, cols), ...] per query] or raises Panic."""
    pos = 0

    def u32():
        nonlocal pos
        if len(req) - pos < 4:
            raise Panic("truncated")
        pos += 4
        return int.from_bytes(req[pos - 4:pos], "big")

    nq = u32()
    if nq >= MAX_LEN:
        raise Panic("len")
    states = []
    for _ in range(nq):
        nm = u32()
        if nm >= MAX_LEN:
            raise Panic("len")
        mats = []
        for _ in range(nm):
            p = pos
            rows, cols = u32(), u32()
            if rows >= MAX_LEN or cols >= MAX_LEN:
                raise Panic("len")
            if len(req) - pos < 4 * rows * cols:
                raise Panic("truncated data")
            pos += 4 * rows * cols
            mats.append((p, rows, cols))
        states.append(mats)
    if nq == 0:
        raise Panic("db.num_rows() / 0")
    for mats in states:
        if len(mats) < 1 + e:
            raise Panic("q[1 + j]")
        for j in range(e):
            if mats[1 + j][1:] != (3 * c1, 1):
                raise Panic("q_2 shape")
    return [m[:1 + e] for m in states]


def batch_check(states, l, server_rows, db_cols, chunk):
    nq = len(states)
    if chunk >= 0 and chunk >= nq:
        raise Panic("chunk")
    need = l if chunk < 0 else (l - (nq - 1) * (l // nq) if chunk == nq - 1 else l // nq)
    if need > server_rows:
        raise Panic("rows")
    for k, mats in enumerate(states):
        if (chunk < 0 or k == chunk) and mats[0][1:] != (3 * db_cols, 1):
            raise Panic("q_1 shape")


def response_framing(nq, e, dx, n):
    """msg.serialize() with zero data: [a_1' a_2^T (dx x n)] + per query and j [h_1 q_2 (n dx x 1), a_1' q_2 (dx x 1)]"""
    mats = [ser_matrix(dx, n)]
    for _ in range(nq * e):
        mats += [ser_matrix(n * dx, 1), ser_matrix(dx, 1)]
    return ser_vec(mats)


# ---- the checker ---------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def checker(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("dwc") / "dpir_wire_check")
    subprocess.check_call(["/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++", "-O1", "-std=c++17", "-Wall", "-Werror",
                           "-o", exe, os.path.join(ROOT, "tests", "cpp", "dpir_wire_check.cpp")])
    return exe


# geometry: e = ne / x, c1 = packed cols of h_1, l, rows the server holds, packed db cols, delta x, n
G = dict(e=1, c1=2, l=5, server_rows=5, db_cols=3, dx=2, n=3)
G2 = dict(e=2, c1=1, l=8, server_rows=8, db_cols=4, dx=4, n=2)


def run(checker, tmp_path, req, g, chunk=-1):
    path, resp = tmp_path / "req.bin", tmp_path / "resp.bin"
    path.write_bytes(bytes(req))
    if resp.exists():
        resp.unlink()
    out = subprocess.check_output([checker, str(path)] + [str(g[k]) for k in ("e", "c1", "l", "server_rows", "db_cols")]
                                  + [str(chunk), str(g["dx"]), str(g["n"]), str(resp)], text=True).split("\n")
    rc = int(out[0].split()[1])
    if rc == 0:
        rc = int(out[1].split()[1])
    mats = [tuple(int(v) for v in ln.split()[1:]) for ln in out if ln.startswith("mat ")]
    size = [int(ln.split()[1]) for ln in out if ln.startswith("size ")]
    return rc, mats, (size[0] if size else None), (resp.read_bytes() if resp.exists() else None)


def expect(req, g, chunk=-1):
    try:
        states = walk(req, g["e"], g["c1"])
        batch_check(states, g["l"], g["server_rows"], g["db_cols"], chunk)
    except Panic:
        return None
    return [(k, t, p, r, c) for k, mats in enumerate(states) for t, (p, r, c) in enumerate(mats)]


def query(g, rng, extra=(), q1_shape=None):
    q1r, q1c = q1_shape or (3 * g["db_cols"], 1)
    mats = [ser_matrix(q1r, q1c, rng.integers(0, 2**32, q1r * q1c, dtype=np.uint64))]
    mats += [ser_matrix(3 * g["c1"], 1, rng.integers(0, 2**32, 3 * g["c1"], dtype=np.uint64)) for _ in range(g["e"])]
    return ser_vec(mats + list(extra))


def check(checker, tmp_path, req, g, chunk=-1):
    rc, mats, size, resp = run(checker, tmp_path, req, g, chunk)
    want = expect(req, g, chunk)
    if want is None:
        assert rc == E_SHAPE
        assert resp is None                                        # nothing is produced for a refused request
    else:
        assert rc == 0 and mats == want
        nq = len({m[0] for m in mats})
        assert resp == response_framing(nq, g["e"], g["dx"], g["n"]) and size == len(resp)
    return rc


@pytest.mark.parametrize("g", [G, G2], ids=["e1", "e2"])
@pytest.mark.parametrize("nq", [1, 2, 3, 7])
def test_good_requests_and_response_framing(checker, tmp_path, g, nq):
    rng = np.random.default_rng(nq)
    req = ser_vec([query(g, rng) for _ in range(nq)])
    assert check(checker, tmp_path, req, g) == 0
    # trailing bytes and extra matrices in a state are ignored
    assert check(checker, tmp_path, req + b"\x00\x01\x02\x03\x04", g) == 0
    extra = [ser_matrix(2, 3, np.arange(6)), ser_matrix(0, 5), ser_matrix(MAX_LEN - 1, 0), ser_matrix(0, MAX_LEN - 1)]
    assert check(checker, tmp_path, ser_vec([query(g, rng, extra) for _ in range(nq)]), g) == 0


def test_reference_serialization_shapes(checker, tmp_path):
    # serializer.rs:199-214 serialization_is_inverse_of_itself: one state of 10 x 35, 7 x 1 and 1 x 7.  Framing only (e = 0:
    # the parser records q_1), so the positions are checked; its q_1 is no database's, so answer() would refuse it.
    rng = np.random.default_rng(0)
    st = ser_vec([ser_matrix(10, 35, rng.integers(0, 2**32, 350, dtype=np.uint64)), ser_matrix(7, 1, np.arange(7)),
                  ser_matrix(1, 7, np.arange(7))])
    g = dict(G, e=0)
    for req in (ser_vec([st]), ser_vec([st, st])):
        assert [m[0] for m in walk(req, 0, 1)] == [(8 + k * len(st), 10, 35) for k in range(len(req) // len(st))]
        assert check(checker, tmp_path, req, g) == E_SHAPE         # the framing parses; its q_1 (10 x 35) is no database's
        rc, mats, _, _ = run(checker, tmp_path, req, g)
        assert mats == [(k, 0, 8 + k * (len(st)), 10, 35) for k in range(len(req) // len(st))]


def test_truncation_at_every_byte(checker, tmp_path):
    rng = np.random.default_rng(3)
    req = ser_vec([query(G, rng), query(G, rng, [ser_matrix(1, 2, [5, 6])])])
    for cut in range(len(req)):
        assert check(checker, tmp_path, req[:cut], G) == E_SHAPE, cut


@pytest.mark.parametrize("field", ["queries", "matrices", "rows", "cols"])
def test_counts_and_dimensions_at_max_len(checker, tmp_path, field):
    rng = np.random.default_rng(4)
    for v in (MAX_LEN - 1, MAX_LEN, 0xFFFFFFFF):
        if field == "queries":
            req = v.to_bytes(4, "big") + query(G, rng)
        elif field == "matrices":
            req = (1).to_bytes(4, "big") + v.to_bytes(4, "big") + query(G, rng)[4:]
        else:                                                      # an extra matrix with no data words
            bad = v.to_bytes(4, "big") + (0).to_bytes(4, "big") if field == "rows" else (0).to_bytes(4, "big") + v.to_bytes(4, "big")
            req = ser_vec([query(G, rng, [bad])])
        rc = check(checker, tmp_path, req, G)
        if field in ("rows", "cols") and v == MAX_LEN - 1:
            assert rc == 0, (field, v)                             # an empty (2^28 - 1) x 0 extra matrix is read and ignored
        else:
            assert rc == E_SHAPE, (field, v)


def test_zero_queries_and_missing_matrices(checker, tmp_path):
    rng = np.random.default_rng(5)
    assert check(checker, tmp_path, ser_vec([]), G) == E_SHAPE
    assert check(checker, tmp_path, ser_vec([]) + b"\x00" * 64, G) == E_SHAPE
    q = query(G2, rng)
    one_short = (2).to_bytes(4, "big") + q[4:4 + 8 + 4 * 12] + q[4 + 8 + 4 * 12:4 + 2 * 8 + 4 * 12 + 4 * 3]
    assert check(checker, tmp_path, ser_vec([one_short]), G2) == E_SHAPE
    assert check(checker, tmp_path, ser_vec([q, ser_vec([])]), G2) == E_SHAPE


def test_vector_shapes(checker, tmp_path):
    rng = np.random.default_rng(6)
    good = query(G, rng)
    for shape in [(3 * G["db_cols"] - 1, 1), (3 * G["db_cols"] + 1, 1), (3 * G["db_cols"], 2), (1, 3 * G["db_cols"]), (0, 1)]:
        req = ser_vec([good, query(G, rng, q1_shape=shape)])
        assert check(checker, tmp_path, req, G) == E_SHAPE, shape
        assert check(checker, tmp_path, req, G, chunk=0) == 0, shape          # chunk 0 reads only query 0's q_1
        assert check(checker, tmp_path, req, G, chunk=1) == E_SHAPE, shape
    for rows, cols in [(3 * G["c1"] - 1, 1), (3 * G["c1"] + 1, 1), (3 * G["c1"], 2), (0, 0)]:
        q = ser_vec([ser_matrix(3 * G["db_cols"], 1), ser_matrix(rows, cols)])
        for chunk in (-1, 0):
            assert check(checker, tmp_path, ser_vec([good, q]), G, chunk) == E_SHAPE, (rows, cols)


def test_chunks_and_rows_held(checker, tmp_path):
    rng = np.random.default_rng(7)
    for nq in (1, 2, 3, 6, 7):                                     # l = 5: 6 and 7 queries leave every batch but the last empty
        req = ser_vec([query(G, rng) for _ in range(nq)])
        for chunk in range(-1, nq + 2):
            for held in (0, 1, 2, 4, 5):
                check(checker, tmp_path, req, dict(G, server_rows=held), chunk)
        rc, *_ = run(checker, tmp_path, req, G, nq)
        assert rc == E_SHAPE                                       # chunk index == query count
