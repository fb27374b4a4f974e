"""The CPU oracle at the corners of the accepted parameter space (param_space_sets.py), against plain Python integers.

The GPU parity tests at these corners (test_gpu_param_space.py) compare the CUDA path with the oracle, so the oracle itself is
pinned here where nothing else runs it: gadget decomposition at every gadget dimension 3..56 (including the widths whose high
digits start at or past bit 64), rescale + the LSB-first bit stream of encode at every (p, q2_bits) the sets use plus the
extremes, and a decrypt-and-compare of every set that decodes."""
import numpy as np
import pytest

import oracle_lib as O
import param_space_sets as PS

SEED_DB = 0xB1755


def _params(**over):
    kw = dict(PS.BASE)
    kw.update(over)
    return O.Params(**kw)


# ------------------------------------------------------------------ gadget.rs:3-9, 34-60
def test_bits_per_every_gadget_dimension():
    P = _params()
    assert P.modulus_log2 == 56 and P.modulus == 268369921 * 249561089
    for t in range(3, 57):
        assert P.bits_per(t) == (1 if t == 56 else 56 // t + 1), t


@pytest.mark.parametrize("t", range(3, 57))
def test_gadget_invert_every_gadget_dimension(t):
    P = _params()
    q = P.modulus
    rng = np.random.default_rng(1000 + t)
    v = rng.integers(0, q, P.N, dtype=np.uint64)
    v[:4] = [0, q - 1, q, 1]                # q itself: the non-canonical raw coefficient (kernels.h)
    got = P.gadget_invert(v, 1, 1, t, rdim=1).reshape(t, P.N)
    bits = 1 if t == 56 else 56 // t + 1
    mask = (1 << bits) - 1
    vals = [int(x) for x in v]
    for k in range(t):
        off = k * bits
        exp = [0 if off >= 64 else (x >> off) & mask for x in vals]
        assert [int(x) for x in got[k]] == exp, (t, k)
        if off >= 64:
            assert not got[k].any(), (t, k)
    # the digits recompose every input: no bit below 2^(t * bits) is lost
    recomposed = [sum(int(got[k, z]) << (k * bits) for k in range(t)) for z in range(8)]
    assert recomposed == vals[:8]


# ------------------------------------------------------------------ arith.rs:429-444 rescale, server.rs:470-503 encode
def _rescale(a, inp_mod, out_mod):
    """round(centred(a mod inp_mod) * out_mod / inp_mod), ties away from zero, then mod out_mod."""
    x = a % inp_mod
    if x >= inp_mod // 2:
        x -= inp_mod
    num = x * out_mod
    r = (num + inp_mod // 2) // inp_mod if num >= 0 else -((-num + inp_mod // 2) // inp_mod)
    return r % out_mod


def _encode(P, packed):
    """LSB-first bit stream of the rescaled rows: per instance, row 0 (n polys) at q2_bits, rows 1..n at q1_bits, q1 = 4p."""
    q1 = 4 * P.p
    q1_bits = (q1 - 1).bit_length()
    n, N = P.n, P.N
    acc, off = 0, 0
    per = (n + 1) * n * N
    vals = [int(x) for x in packed]
    for inst in range(P.instances):
        m = vals[inst * per:(inst + 1) * per]
        for a in m[: n * N]:
            acc |= _rescale(a, P.modulus, P.q2) << off
            off += P.q2_bits
        for a in m[n * N:]:
            acc |= _rescale(a, P.modulus, q1) << off
            off += q1_bits
    nbytes = (off + 63) // 64 * 8
    return np.frombuffer(acc.to_bytes(nbytes, "little"), dtype=np.uint8)


def _pairs():
    pairs = {(kw["p"], kw["q2_bits"]) for kw in (PS.kw(nm) for nm in PS.SETS)}
    pairs |= {(p, q2) for p in (2, 1 << 20) for q2 in (14, 36)}
    return sorted(pairs)


@pytest.mark.parametrize("p,q2_bits", _pairs())
@pytest.mark.parametrize("n,instances", [(2, 1), (1, 3)])
def test_rescale_and_encode_match_python_integers(p, q2_bits, n, instances):
    P = _params(p=p, q2_bits=q2_bits, n=n, instances=instances)
    q = P.modulus
    assert P.q2 % 2 == 1 and 1 << 13 < P.q2 < 1 << q2_bits        # every rescaled value fits its q2_bits-wide field
    words = instances * (n + 1) * n * P.N
    rng = np.random.default_rng(p * 64 + q2_bits + n)
    packed = rng.integers(0, q, words, dtype=np.uint64)
    special = [0, 1, q // 2 - 1, q // 2, q // 2 + 1, q - 1, q]
    # in row 0 (rescaled to q2) and in the last row of the last instance (rescaled to q1)
    packed[: len(special)] = special
    packed[-len(special):] = special
    packed[n * P.N: n * P.N + len(special)] = special
    for a in special + [int(x) for x in packed[100:120]]:
        assert O.LIB.orc_rescale(a, q, P.q2) == _rescale(a, q, P.q2)
        assert O.LIB.orc_rescale(a, q, 4 * p) == _rescale(a, q, 4 * p)
    exp = _encode(P, packed)
    q1_bits = (4 * p - 1).bit_length()
    assert exp.size == P.response_bytes() == ((instances * (q2_bits * n + q1_bits * n * n) * P.N + 63) // 64) * 8
    got = P.encode(packed)
    assert got.size == exp.size
    assert np.array_equal(got, exp)


# ------------------------------------------------------------------ every set that decodes: process_query + decode_response
@pytest.mark.parametrize("name", [nm for nm in PS.SETS if PS.decodes(nm)])
def test_oracle_decodes_param_set(name):
    P = O.Params(expand_queries=PS.expand(name), **PS.kw(name))
    cl = O.Client(P, 1234)
    pp = cl.generate_keys()
    db = P.generate_db(SEED_DB)
    total = P.dim0 * P.num_per
    for idx in sorted({0, total - 1, total // 2}):
        q = cl.generate_query(idx)
        resp = P.process_query(pp, q, db)
        assert resp.size == P.response_bytes()
        assert np.array_equal(cl.decode_response(resp), P.db_plain_item(SEED_DB, idx)), (name, idx)
