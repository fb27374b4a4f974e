"""The fold, expansion and pack digit loops and the first dimension at their accumulators' exactness bounds, bit for bit
against the oracle.

Digit polynomials come from tests/golden/lz_extremes.bin (tests/lz_extremes.py): their relaxed-range transforms reach about
15.5q at one target slot, and every key residue there is q_n - 1.  tests/test_lz_extremes_witness.py replays the kernels'
accumulator schedules with them: where 16 products build up, the q0 peaks are 0.94-0.98 * 2^64 (fold fast path), 0.97-0.98
(pack, t = 28 and 56), 0.91 and 0.98 (expansion round 0, t = 28 and 56) and 0.91-0.98 (general fold path), except 0.86, 0.89
and 0.92 for the general path at t = 8, 9 and 14, whose digits past the live ones are zero.  Each record is tuned to one
modulus, so every case runs once per modulus.  k_regev_to_gsw decomposes expansion outputs and has no entry point of its
own; it is covered only through the expansion and end-to-end tests.  The first dimension runs with the residues whose 7-bit
limbs are the largest below each modulus, one query at a time and in a 16-query database pass."""
import numpy as np
import pytest

import lz_extremes as LZ
import oracle_lib as O
from test_gpu_param_space import _residues, _worst_params

pytestmark = pytest.mark.gpu

F = LZ.load()
Q0, Q1, Q = LZ.Q0, LZ.Q1, LZ.Q


def _gpu():
    import sdk_b200.spiral as S
    return S


E_UNSUPPORTED = -4


def _max_keys(words):
    return _residues(words, "max")


def _u64(a):
    return np.array([int(x) for x in a], dtype=np.uint64)


@pytest.fixture(scope="module", params=[(t, v) for t in LZ.WIDTHS for v in (0, 1)], ids=lambda p: f"t{p[0]}-v{p[1]}")
def ctx(request):
    S = _gpu()
    t, version = request.param
    P, kw = _worst_params(t, version)
    G = S.Params(**kw)
    pp = {k: (_max_keys(G.words[k]) if k != "right" or G.has_right else None) for k in ("pack", "left", "right", "conv")}
    gpp = S.PublicParameters(G, pp["pack"], pp["left"], pp["right"], pp["conv"])
    yield t, version, P, G, pp, gpp
    gpp.close()
    G.close()


def _fold_both(S, P, G, cts, vf, vfn=None):
    ref = P.fold_ciphertexts(cts, vf, P.get_v_folding_neg(vf) if vfn is None else vfn)
    got = cts.copy()
    if vfn is None:
        S.fold_ciphertexts(G, got, vf)                 # fast path: k_fold_res_lz
    else:
        S.fold_ciphertexts(G, got, vf, vfn)            # general path: k_fold_round
    return got, ref


@pytest.mark.parametrize("m", [0, 1])
def test_fold_fast_path_at_the_bound(ctx, m):
    """Round 0 of the fast path (byte path at t = 8, generic otherwise): every digit difference is the searched delta."""
    S = _gpu()
    t, version, P, G, pp, gpp = ctx
    vi, vh = LZ.fold_pair(F, m, t)
    cts = np.concatenate([_u64(vi), _u64(vi), _u64(vh), _u64(vh)])
    vf = _max_keys(G.words["v_folding"])
    got, ref = _fold_both(S, P, G, cts, vf)
    assert np.array_equal(got, ref), (t, version, m)


@pytest.mark.parametrize("m", [0, 1])
def test_fold_general_path_at_the_bound(ctx, m):
    """k_fold_round on raw words whose digits are the searched raw digits, with an explicit v_folding_neg of q_n - 1."""
    S = _gpu()
    t, version, P, G, pp, gpp = ctx
    c = _u64(LZ.raw_coeffs(F, m, t))
    cts = np.concatenate([c, c, c, c])
    vf = _max_keys(G.words["v_folding"])
    got, ref = _fold_both(S, P, G, cts, vf, vf.copy())
    assert np.array_equal(got, ref), (t, version, m)


@pytest.mark.parametrize("m", [0, 1])
def test_expansion_round0_at_the_bound(ctx, m):
    """Slot 0 holds the NTT of tau^-1(c): round 0's first output decomposes exactly the searched digits of c."""
    S = _gpu()
    t, version, P, G, pp, gpp = ctx
    t0 = (56 if version == 0 else t) if G.has_right else t
    a = _u64(LZ.expansion_slot(LZ.raw_coeffs(F, m, t0)))
    first = P.to_ntt(np.concatenate([a, a]))
    v = np.zeros((1 << P.g) * 2 * P.W, dtype=np.uint64)
    v[: first.size] = first
    ref = P.coefficient_expansion(v, pp)
    got = v.copy()
    S.coefficient_expansion(G, gpp, got)
    assert np.array_equal(got, ref), (t, version, m)


@pytest.mark.parametrize("m", [0, 1])
def test_pack_raw_at_the_bound(ctx, m):
    S = _gpu()
    t, version, P, G, pp, gpp = ctx
    c = _u64(LZ.raw_coeffs(F, m, t))
    cts = np.tile(c, P.n * P.n * 2)
    assert np.array_equal(S.pack(G, gpp, cts), P.pack(cts, pp["pack"])), (t, version, m)


def test_digit_extremes(ctx):
    """Every live digit 2^bits - 1 (the top one as large as a value < q allows), and fold pairs whose differences are
    +(2^bits - 1) and -(2^bits - 1) in every digit plane (both ends, 1 and 511, of byte_pair_diff's range at t = 8)."""
    S = _gpu()
    t, version, P, G, pp, gpp = ctx
    bits, live = LZ.bits_per(t), LZ.live_digits(t)
    top = LZ.top_limit(t)
    full = ((top + 1) << (bits * (live - 1))) - 1
    assert full < Q
    hi = np.full(LZ.N, full, dtype=np.uint64)
    lo = np.zeros(LZ.N, dtype=np.uint64)
    vf = _max_keys(G.words["v_folding"])
    for cts in (np.concatenate([lo, lo, hi, hi]), np.concatenate([hi, hi, lo, lo])):
        got, ref = _fold_both(S, P, G, cts, vf)
        assert np.array_equal(got, ref), (t, version)
        got, ref = _fold_both(S, P, G, cts, vf, vf.copy())
        assert np.array_equal(got, ref), (t, version)
    cts = np.tile(hi, P.n * P.n * 2)
    assert np.array_equal(S.pack(G, gpp, cts), P.pack(cts, pp["pack"])), (t, version)


# ------------------------------------------------------------------ first dimension
LIMB_MAX = (0x0FDFFFFF, 0x0EDFFFFF)        # the residues < q_n with the largest 7-bit limbs (tests/test_lz_extremes_witness.py)


def _operand(size, mix, rng):
    w = np.uint64(LIMB_MAX[0] | (LIMB_MAX[1] << 32))
    v = np.full(size, w, dtype=np.uint64)
    if mix == "qm1":
        v[::3] = np.uint64((Q0 - 1) | ((Q1 - 1) << 32))
    elif mix == "random":
        sel = rng.random(size) < 0.5
        v[sel] = (rng.integers(0, Q0, sel.sum(), dtype=np.uint64) | (rng.integers(0, Q1, sel.sum(), dtype=np.uint64) << np.uint64(32)))
    return v


def _database(S, G, words, fmt):
    """The database in layout fmt, or None when the layout refuses the geometry (and says B200PIR_E_UNSUPPORTED)."""
    try:
        return S.Database.from_words(G, words, fmt=fmt)
    except S.B200PirError as e:
        assert e.code == E_UNSUPPORTED, (fmt, str(e))
        return None


@pytest.mark.parametrize("nu_1", [10, 9])
@pytest.mark.parametrize("fmt", [0, 1, 2])
def test_first_dimension_limb_extremes(nu_1, fmt):
    """One query: limb-extreme residues in the database and the query, alone, mixed with q - 1 and with random values."""
    S = _gpu()
    kw = dict(O.PARAM_SETS["T"])
    kw.update(nu_1=nu_1, nu_2=1, n=1, db_item_size=2048)
    P = O.Params(**kw)
    G = S.Params(**kw)
    rng = np.random.default_rng(nu_1 * 10 + fmt)
    try:
        for mix in ("alone", "qm1", "random"):
            dbw = _operand(P.dim0 * P.num_per * P.N, mix, rng)         # one slice, the same in every slice
            v = _operand(P.dim0 * 2 * P.N, mix, rng)
            ref = P.multiply_reg_by_database(dbw, v)
            gdb = _database(S, G, np.tile(dbw, P.slices), fmt)
            if gdb is None:
                pytest.skip(f"layout {fmt} refuses dim0 = {P.dim0}")
            try:
                for s in sorted({0, P.slices - 1}):
                    assert np.array_equal(S.multiply_reg_by_database(G, gdb, s, v), ref), (nu_1, fmt, mix, s)
            finally:
                gdb.close()
    finally:
        G.close()


BATCH = 16


@pytest.fixture(scope="module")
def batch_case():
    """dim0 = 512, 16 queries of one client against databases of limb-extreme residues (alone, mixed with q - 1, mixed with
    random values), and the oracle's responses.  The batch entry point expands its queries, so the query side of the first
    dimension holds expansion outputs, not chosen residues."""
    S = _gpu()
    kw = dict(O.PARAM_SETS["T"])
    kw.update(nu_1=9, nu_2=1, n=1, db_item_size=2048)
    P = O.Params(**kw)
    cl = O.Client(P, 77)
    pp = cl.generate_keys()
    total = P.dim0 * P.num_per
    idxs = [(131 * k + 7) % total for k in range(BATCH)]
    qs = [cl.generate_query(i)["ct"] for i in idxs]
    rng = np.random.default_rng(512)
    dbs = {mix: _operand(P.slices * P.dim0 * P.num_per * P.N, mix, rng) for mix in ("alone", "qm1", "random")}
    refs = {mix: [P.process_query(pp, {"ct": q}, db) for q in qs] for mix, db in dbs.items()}
    G = S.Params(**kw)
    gpp = S.PublicParameters(G, pp["pack"], pp.get("left"), pp.get("right"), pp.get("conv"))
    yield S, G, gpp, np.concatenate(qs), dbs, refs
    gpp.close()
    G.close()


@pytest.mark.parametrize("fmt", [0, 1, 2])
def test_first_dimension_limb_extremes_16_queries(batch_case, fmt):
    S, G, gpp, qcts, dbs, refs = batch_case
    for mix, db in dbs.items():
        gdb = _database(S, G, db, fmt)
        if gdb is None:
            pytest.skip(f"layout {fmt} refuses dim0 = 512")
        try:
            out = S.process_query_batch(G, gpp, qcts, gdb)
        finally:
            gdb.close()
        assert out.shape == (BATCH, G.response_bytes)
        for k in range(BATCH):
            assert np.array_equal(out[k], refs[mix][k]), (fmt, mix, k)
