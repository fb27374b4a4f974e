"""Parity of the CUDA path with the CPU oracle across the accepted parameter space (param_space_sets.py): gadget widths above 8
(the fold's mid-loop accumulator reduction), 1-bit to 19-bit digits (digits past bit 64), n = 1 and n = 4, version 1 with and
without right-hand expansion keys, p from 2 to 2^20 with q2_bits from 14 to 36, first dimensions shorter than one k-tile, and
direct upload.  Bit-exact: every comparison is array equality on integers / bytes.  The second half drives the expansion, fold
and packing kernels with worst-case operands (every residue q_n - 1, every raw coefficient q - 1 or q) at every gadget width
class, which honest queries never produce."""
import numpy as np
import pytest

import oracle_lib as O
import param_space_sets as PS

pytestmark = pytest.mark.gpu

SEED_DB = 0xB1755
Q0, Q1 = 268369921, 249561089
E_UNSUPPORTED = -4
NAMES = list(PS.SETS)
# 512 x 64 items (2 GiB of database words): one or two indices, wgmma layout only
LARGE = "client_default"
EXPAND_NAMES = [nm for nm in NAMES if PS.expand(nm)]
BATCH = 17            # one full 16-query database pass and one more


def _gpu():
    import sdk_b200.spiral as S
    return S


class _Case:
    """Oracle params + client + keys + database, the GPU context and public parameters, and the oracle's responses, once per
    set and module."""

    def __init__(self, name):
        S = _gpu()
        self.name = name
        self.expand, self.decodes = PS.expand(name), PS.decodes(name)
        self.P = P = O.Params(expand_queries=self.expand, **PS.kw(name))
        self.cl = O.Client(P, 1234)
        self.pp = self.cl.generate_keys()
        self.db = P.generate_db(SEED_DB)
        self.G = S.Params(expand_queries=self.expand, **P.kw)
        self.gpp = S.PublicParameters(self.G, self.pp["pack"], self.pp.get("left"), self.pp.get("right"), self.pp.get("conv"))
        self.total = P.dim0 * P.num_per
        self.idxs = [self.total // 2 + 3, self.total - 1] if name == LARGE else sorted({0, self.total // 2, self.total - 1})
        self.queries = {i: self.cl.generate_query(i) for i in self.idxs}
        self.stage_idx = self.idxs[0]
        self.resp, self.dump = {}, None
        self.dbs = {}

    def ref(self, idx):
        if idx not in self.resp:
            if idx == self.stage_idx:
                self.resp[idx], self.dump = self.P.process_query(self.pp, self.queries[idx], self.db, dump=True)
            else:
                self.resp[idx] = self.P.process_query(self.pp, self.queries[idx], self.db)
        return self.resp[idx]

    def stages(self):
        self.ref(self.stage_idx)
        return self.dump

    def gquery(self, q):
        S = _gpu()
        return S.Query(ct=q["ct"]) if self.expand else S.Query(v_buf=q["v_buf"], v_ct=q["v_ct"])

    def gdb(self, fmt):
        """The database uploaded in layout fmt (None = the context's automatic choice).  A layout that refuses the geometry
        must say B200PIR_E_UNSUPPORTED, and the automatic choice must then pick another layout."""
        S = _gpu()
        if fmt not in self.dbs:
            try:
                self.dbs[fmt] = S.Database.from_words(self.G, self.db, fmt=fmt)
            except S.B200PirError as e:
                assert fmt is not None and e.code == E_UNSUPPORTED, (self.name, fmt, str(e))
                auto = self.gdb(None)
                assert auto.info()["format"] != fmt
                self.dbs[fmt] = auto
            else:
                assert fmt is None or self.dbs[fmt].info()["format"] == fmt
        return self.dbs[fmt]

    def close(self):
        for d in self.dbs.values():
            d.close()
        self.gpp.close()
        self.G.close()


_cache = {}


def case(name):
    if name not in _cache:
        _cache[name] = _Case(name)
    return _cache[name]


@pytest.fixture(scope="module", autouse=True)
def _release_cases():
    yield
    for c in _cache.values():
        c.close()
    _cache.clear()


def _fmts(name):
    return [2] if name == LARGE else [0, 1, 2]


def _check_response(c, idx, got):
    assert np.array_equal(got, c.ref(idx)), (c.name, idx)
    if c.decodes:
        assert np.array_equal(c.cl.decode_response(got), c.P.db_plain_item(SEED_DB, idx)), (c.name, idx)


# ------------------------------------------------------------------ sizes
@pytest.mark.parametrize("name", NAMES)
def test_sizes_match_oracle(name):
    c = case(name)
    assert (c.G.setup_bytes, c.G.query_bytes, c.G.response_bytes) == (c.P.setup_bytes, c.P.query_bytes, c.P.response_bytes())


def test_n5_is_unsupported():
    S = _gpu()
    with pytest.raises(S.B200PirError) as ei:
        S.Params(**dict(PS.BASE, n=5))
    assert ei.value.code == E_UNSUPPORTED


@pytest.mark.parametrize("over", [dict(t_gsw=9, nu_1=2, nu_2=2), dict(t_gsw=56, nu_1=1, nu_2=2), dict(t_gsw=3, nu_1=1, nu_2=6)])
def test_unbalanced_expansion_geometry_is_unsupported(over):
    """expand_query reads the first-dimension inputs from slots 2i (i < dim0) and the GSW inputs from slots 2i + 1
    (i < t_gsw * nu_2), out of 2^g slots with g = ceil(log2(t_gsw * nu_2 + dim0)).  When one half outgrows 2^(g-1) (t_gsw = 9,
    nu_2 = 2, dim0 = 4: slot 35 of 32) the reference panics; the context refuses the parameters.  Direct upload has no
    expansion and stays accepted."""
    S = _gpu()
    with pytest.raises(S.B200PirError) as ei:
        S.Params(**dict(PS.BASE, **over))
    assert ei.value.code == E_UNSUPPORTED
    S.Params(expand_queries=False, **dict(PS.BASE, **over)).close()
    # the balanced neighbours stay accepted: one more first-dimension bit makes 2^g large enough
    kw = dict(PS.BASE, **over)
    while 2 * max(1 << kw["nu_1"], kw["t_gsw"] * kw["nu_2"]) > 1 << (kw["t_gsw"] * kw["nu_2"] + (1 << kw["nu_1"]) - 1).bit_length():
        kw["nu_1"] += 1
    S.Params(**kw).close()


# ------------------------------------------------------------------ end to end, every database layout
@pytest.mark.parametrize("name,fmt", [(nm, f) for nm in NAMES for f in _fmts(nm)])
def test_process_query_every_layout(name, fmt):
    S = _gpu()
    c = case(name)
    gdb = c.gdb(fmt)
    for idx in c.idxs:
        _check_response(c, idx, S.process_query(c.G, c.gpp, c.gquery(c.queries[idx]), gdb))


@pytest.mark.parametrize("name", [nm for nm in EXPAND_NAMES if nm != LARGE])
def test_process_query_batch_crosses_a_pass(name):
    """17 queries in one call: a 16-query database pass and a 1-query pass; the per-query strides depend on t_gsw, n and
    instances."""
    S = _gpu()
    c = case(name)
    idxs = [(37 * k + 5) % c.total for k in range(BATCH)]
    idxs[0], idxs[8], idxs[-1] = c.idxs[0], c.idxs[-1], c.idxs[len(c.idxs) // 2]
    qs = [c.queries[i] if i in c.queries else c.cl.generate_query(i) for i in idxs]
    out = S.process_query_batch(c.G, c.gpp, np.concatenate([q["ct"] for q in qs]), c.gdb(None))
    assert out.shape == (BATCH, c.G.response_bytes)
    for k, (i, q) in enumerate(zip(idxs, qs)):
        ref = c.ref(i) if q is c.queries.get(i) else c.P.process_query(c.pp, q, c.db)
        assert np.array_equal(out[k], ref), (name, k, i)
        if c.decodes:
            assert np.array_equal(c.cl.decode_response(out[k]), c.P.db_plain_item(SEED_DB, i)), (name, k, i)


# ------------------------------------------------------------------ stage by stage
@pytest.mark.parametrize("name", NAMES)
def test_stages_match_oracle(name):
    S = _gpu()
    c = case(name)
    P, G = c.P, c.G
    d = c.stages()
    q = c.queries[c.stage_idx]
    if c.expand:
        vreg, vf = S.expand_query(G, c.gpp, S.Query(ct=q["ct"]))
        vreg_ref, vf_ref = P.expand_query(c.pp, q["ct"])
        assert np.array_equal(vreg, vreg_ref)
        assert np.array_equal(vf[: vf_ref.size], vf_ref)
        assert np.array_equal(vreg_ref, d["v_firstdim"]) and np.array_equal(vf_ref, d["v_folding"])
    if P.nu_2:
        assert np.array_equal(S.get_v_folding_neg(G, d["v_folding"]), d["v_folding_neg"])
        inter = P.from_ntt(d["first_mult"])
        ref = P.fold_ciphertexts(inter, d["v_folding"], d["v_folding_neg"])
        got = inter.copy()
        S.fold_ciphertexts(G, got, d["v_folding"], d["v_folding_neg"])      # k_fold_round
        assert np.array_equal(got, ref)
        fast = inter.copy()
        S.fold_ciphertexts(G, fast, d["v_folding"])                          # implied neg: k_fold_res_lz
        assert np.array_equal(fast, ref)
    nn = P.n * P.n
    for inst in range(P.instances):
        cts = d["folded"][inst * nn * 2 * P.N:(inst + 1) * nn * 2 * P.N]
        assert np.array_equal(S.pack(G, c.gpp, cts), P.pack(cts, c.pp["pack"])), inst
    enc = S.encode(G, d["packed"])
    assert np.array_equal(enc, P.encode(d["packed"]))
    assert np.array_equal(enc, c.ref(c.stage_idx))


# ------------------------------------------------------------------ wire formats
@pytest.mark.parametrize("name", NAMES)
def test_wire_formats(name):
    """PublicParameters::deserialize + process_query_bytes on the client's serialised bytes (direct upload: the seed-derived
    halves of each query are regenerated on the GPU)."""
    S = _gpu()
    c = case(name)
    ppb = c.cl.pp_bytes()
    assert ppb.size == c.G.setup_bytes
    gpp = S.PublicParameters.deserialize(c.G, ppb)
    idxs = c.idxs[-1:] if name == LARGE else [c.idxs[0], c.idxs[-1], (c.total // 3) | 1]
    blobs, refs = [], []
    for idx in idxs:
        q = c.cl.generate_query(idx)
        qb = c.cl.query_bytes()
        assert qb.size == c.G.query_bytes
        blobs.append(qb)
        refs.append(c.P.process_query(c.pp, q, c.db))
        if c.expand:
            assert np.array_equal(S.Query.deserialize(c.G, qb).ct, q["ct"])
    out = S.process_query_bytes(c.G, gpp, np.concatenate(blobs), c.gdb(None))
    for k, idx in enumerate(idxs):
        assert np.array_equal(out[k], refs[k]), (name, idx)
        if c.decodes:
            assert np.array_equal(c.cl.decode_response(out[k]), c.P.db_plain_item(SEED_DB, idx)), (name, idx)
    gpp.close()


# ------------------------------------------------------------------ synthetic database at p != 256
@pytest.mark.parametrize("name,fmt", [(nm, f) for nm in NAMES if PS.kw(nm)["p"] != 256 for f in _fmts(nm)])
def test_synthetic_db_equals_generated_db(name, fmt):
    S = _gpu()
    c = case(name)
    P = c.P
    syn = S.Database(c.G, fmt=fmt)
    syn.fill_synthetic(SEED_DB)
    rng = np.random.default_rng(6)
    v = (rng.integers(0, Q0, P.dim0 * 2 * P.N, dtype=np.uint64)
         | (rng.integers(0, Q1, P.dim0 * 2 * P.N, dtype=np.uint64) << np.uint64(32)))
    for s in sorted({0, P.slices - 1}):
        assert np.array_equal(S.multiply_reg_by_database(c.G, syn, s, v), S.multiply_reg_by_database(c.G, c.gdb(fmt), s, v)), s
    syn.close()


# ------------------------------------------------------------------ worst-case operands per gadget width
WIDTHS = [3, 7, 8, 9, 10, 14, 28, 56]


def _worst_params(t, version):
    # dim0 = 32 keeps both halves of the expansion within 2^(g-1) slots up to t_gsw = 56 (see test_unbalanced_expansion_...)
    kw = dict(PS.BASE, nu_1=5, nu_2=2, t_gsw=t, t_conv=t, t_exp_left=t, t_exp_right=t if version else 56, version=version)
    return O.Params(**kw), kw


def _residues(words, pattern):
    """NTT-form words ([poly][crt][z]): every residue q_n - 1, or 0 and q_n - 1 alternating along z."""
    v = np.empty((words // 4096, 2, 2048), dtype=np.uint64)
    v[:, 0], v[:, 1] = Q0 - 1, Q1 - 1
    if pattern == "alt":
        v[:, :, ::2] = 0
    return v.reshape(-1)


def _raw(P, polys, value):
    return np.full(polys * P.N, value, dtype=np.uint64)


@pytest.mark.parametrize("version", [0, 1])
@pytest.mark.parametrize("t", WIDTHS)
def test_worst_case_operands(t, version):
    S = _gpu()
    P, kw = _worst_params(t, version)
    G = S.Params(**kw)
    q = P.modulus
    try:
        for pattern in ("max", "alt"):
            pp = {k: (_residues(G.words[k], pattern) if k != "right" or G.has_right else None)
                  for k in ("pack", "left", "right", "conv")}
            gpp = S.PublicParameters(G, pp["pack"], pp["left"], pp["right"], pp["conv"])
            # coefficient_expansion over all 2^g slots: the first slot holds every residue q_n - 1, or the NTT of raw q
            for first in (_residues(2 * P.W, "max"), P.to_ntt(_raw(P, 2, q))):
                v = np.zeros((1 << P.g) * 2 * P.W, dtype=np.uint64)
                v[: first.size] = first
                ref = P.coefficient_expansion(v, pp)
                got = v.copy()
                S.coefficient_expansion(G, gpp, got)
                assert np.array_equal(got, ref), (t, version, pattern)
            # expand_query on raw ciphertexts of every coefficient q - 1, and of the non-canonical q
            for value in (q - 1, q):
                ct = _raw(P, 2, value)
                vreg, vf = S.expand_query(G, gpp, S.Query(ct=ct))
                vreg_ref, vf_ref = P.expand_query(pp, ct)
                assert np.array_equal(vreg, vreg_ref), (t, version, pattern, value)
                assert np.array_equal(vf, vf_ref), (t, version, pattern, value)
            # pack
            for value in (q - 1, q):
                cts = _raw(P, P.n * P.n * 2, value)
                assert np.array_equal(S.pack(G, gpp, cts), P.pack(cts, pp["pack"])), (t, version, pattern, value)
            gpp.close()
        # fold: v_folding with every residue q_n - 1; ciphertexts of every coefficient q - 1, of q, and mixed so that the
        # digit differences of a pair are maximal (q - 1 against 0) and non-canonical (q against 0 / q - 1 alternating)
        vf = _residues(G.words["v_folding"], "max")
        vfn = P.get_v_folding_neg(vf)
        assert np.array_equal(S.get_v_folding_neg(G, vf), vfn)
        alt = _raw(P, 2, q - 1)
        alt[::2] = 0
        for cts in (_raw(P, 2 * P.num_per, q - 1), _raw(P, 2 * P.num_per, q),
                    np.concatenate([_raw(P, 2, q - 1), _raw(P, 2, q), _raw(P, 2, 0), alt])):
            ref = P.fold_ciphertexts(cts, vf, vfn)
            got = cts.copy()
            S.fold_ciphertexts(G, got, vf, vfn)
            assert np.array_equal(got, ref), (t, version)
            fast = cts.copy()
            S.fold_ciphertexts(G, fast, vf)
            assert np.array_equal(fast, ref), (t, version)
    finally:
        G.close()
