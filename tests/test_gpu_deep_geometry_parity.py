"""Byte-exact parity with the CPU oracle at the geometry the kernels are tuned and benchmarked on, and past it.

S8 (bench.py's configuration: nu_1 = 9, nu_2 = 8, t_gsw = 8, 4 slices, 256 rows, 8 GiB in HBM) stage by stage and end to end,
and the overrides of T below, which reach what S8 does not at sizes the oracle can afford: fold trees of 7 to 12 rounds, the
generic-digit fold over 8 rounds, GSW halves larger than dim0, expansion over all 2048 slots, wgmma first dimensions of 512 to
4096 rows and the 1024-long first dimension of S256's per-GPU share.  Every comparison is array equality on integers or bytes,
so a wrong digit in a late fold round, a value left in [q, 2q) or a mis-scheduled expansion key fails here even where the
response still decodes."""
import math

import numpy as np
import pytest

import oracle_lib as O

pytestmark = pytest.mark.gpu

SEED = 0xB1755
Q0, Q1 = 268369921, 249561089
BATCH = 17                          # one full 16-query pass of the wgmma first dimension and one more

# name: (overrides of T, expected (g, stop_round, byte-digit fold))
SETS = {
    # 7 fold rounds; the GSW half t_gsw * nu_2 = 56 exceeds dim0 = 16, so the odd slots outrun the even ones
    "F7": (dict(n=2, nu_1=4, nu_2=7, db_item_size=8192), (7, 6, True)),
    # S8's fold tree (256 rows) and stop_round, with dim0 = 32: one k-tile
    "F8": (dict(n=2, nu_1=5, nu_2=8, db_item_size=8192), (7, 6, True)),
    # the generic-digit fold (t_gsw = 10: 6-bit digits) over 8 rounds
    "G8": (dict(n=1, nu_1=6, nu_2=8, t_gsw=10, db_item_size=2048), (8, 7, False)),
    # 10 rounds, 1024 rows: 32 wgmma row tiles
    "F10": (dict(n=1, nu_1=6, nu_2=10, db_item_size=2048), (8, 7, True)),
    # S256's 12-round fold tree, 4096 rows: 128 row tiles
    "F12": (dict(n=1, nu_1=6, nu_2=12, db_item_size=2048), (8, 7, True)),
    # expansion over all 2^11 = 2048 slots
    "G11": (dict(n=1, nu_1=10, nu_2=1, db_item_size=2048), (11, 3, True)),
    # S256's per-GPU first dimension: dim0 = 1024 (the <4, 1> wgmma kernel), 512 rows, g = 11
    "W512": (dict(n=1, nu_1=10, nu_2=9, db_item_size=2048), (11, 7, True)),
}
ALL_SLOTS = ("F7", "G11")           # coefficient_expansion compared in every slot, those the query path skips included


def _gpu():
    import sdk_b200.spiral as S
    return S


def _accepted(kw):
    """ctx_create's geometry checks (sdk_b200/csrc/api.cu, b200pir_ctx_create): -> (accepted, g, stop_round)."""
    dim0, gsw = 1 << kw["nu_1"], kw["t_gsw"] * kw["nu_2"]
    g = math.ceil(math.log2(gsw + dim0))
    stop_round = math.ceil(math.log2(gsw)) if kw["nu_2"] else 0
    return g <= 11 and 2 * max(dim0, gsw) <= 1 << g, g, stop_round


def _random_v(P, seed):
    """A first-dimension operand with residues over the whole of [0, q_n)."""
    rng = np.random.default_rng(seed)
    n = P.dim0 * 2 * P.N
    return rng.integers(0, Q0, n, dtype=np.uint64) | (rng.integers(0, Q1, n, dtype=np.uint64) << np.uint64(32))


class _Case:
    """Oracle params, client, keys and database; the GPU context, public parameters and format-2 database; BATCH queries
    (with their serialized bytes) and the oracle's responses to them, computed on first use.  Query 0 is also dumped stage
    by stage."""

    def __init__(self, name, kw, expect, formats, sources, layout_queries):
        S = _gpu()
        self.name, self.expect = name, expect
        self.formats, self.sources, self.layout_queries = formats, sources, layout_queries
        self.P = P = O.Params(**kw)
        self.cl = O.Client(P, 1234)
        self.pp = self.cl.generate_keys()
        self.db = P.generate_db(SEED)
        self.G = S.Params(**P.kw)
        self.gpp = S.PublicParameters(self.G, self.pp["pack"], self.pp.get("left"), self.pp.get("right"), self.pp.get("conv"))
        self.gdb = S.Database.from_words(self.G, self.db, fmt=2)
        self.total = P.dim0 * P.num_per
        self.slice_words = P.dim0 * P.num_per * P.N
        rng = np.random.default_rng(P.nu_1 * 64 + P.nu_2)
        # index 0, the last index, a random one, the last row of the first column, the middle row of the last column, then
        # random ones (item idx sits in row idx % num_per, column idx // num_per)
        idxs = [0, self.total - 1, int(rng.integers(1, self.total - 1)), P.num_per - 1,
                (P.dim0 - 1) * P.num_per + P.num_per // 2]
        while len(set(idxs)) < BATCH:
            idxs.append(int(rng.integers(0, self.total)))
        self.idxs = list(dict.fromkeys(idxs))[:BATCH]
        self.cts, self.qbytes = [], []
        for i in self.idxs:
            self.cts.append(self.cl.generate_query(i)["ct"])
            self.qbytes.append(self.cl.query_bytes())
        self.v = _random_v(P, P.nu_2)
        self._resp, self._dump, self._prod = {}, None, {}

    def ref(self, k):
        """The oracle's response to query k."""
        if k not in self._resp:
            if k == 0:
                self._resp[0], self._dump = self.P.process_query(self.pp, dict(ct=self.cts[0]), self.db, dump=True)
            else:
                self._resp[k] = self.P.process_query(self.pp, dict(ct=self.cts[k]), self.db)
        return self._resp[k]

    def stages(self):
        self.ref(0)
        return self._dump

    def product(self, s):
        """The oracle's multiply_reg_by_database of self.v over slice s."""
        if s not in self._prod:
            w = self.slice_words
            self._prod[s] = self.P.multiply_reg_by_database(self.db[s * w:(s + 1) * w], self.v)
        return self._prod[s]

    def close(self):
        for h in (self.gdb, self.gpp, self.G):
            h.close()
        self.db = None


def _deep_case(name):
    kw = dict(O.PARAM_SETS["T"])
    kw.update(SETS[name][0])
    fmts = (2, 1, 0) if 8 * kw["n"] ** 2 * (2048 << (kw["nu_1"] + kw["nu_2"])) <= 1 << 30 else (2, 1)
    return _Case(name, kw, SETS[name][1], fmts, ("words",), (0,))


class _Stages:
    """Every stage of the pipeline against the oracle.  The subclasses provide the case as the fixture `c`."""

    def test_context_accepts_the_geometry(self, c):
        P = c.P
        ok, g, stop_round = _accepted(P.kw)
        assert ok and (c.G.g, c.G.stop_round) == (P.g, P.stop_round) == (g, stop_round)
        assert (g, stop_round, P.bits_per(P.t_gsw) == 8) == c.expect
        info = c.gdb.info()
        assert info["format"] == 2 and info["local_rows"] == P.num_per

    def test_expand_query(self, c):
        S, P = _gpu(), c.P
        vreg_ref, vf_ref = P.expand_query(c.pp, c.cts[0])
        vreg, vf = S.expand_query(c.G, c.gpp, S.Query(ct=c.cts[0]))
        assert np.array_equal(vreg, vreg_ref)
        assert np.array_equal(vf, vf_ref)
        if c.name in ALL_SLOTS:
            v = np.zeros((1 << P.g) * 2 * P.W, dtype=np.uint64)
            v[: 2 * P.W] = P.to_ntt(c.cts[1])
            ref = P.coefficient_expansion(v, c.pp)
            S.coefficient_expansion(c.G, c.gpp, v)
            assert np.array_equal(v, ref)

    def test_every_layout(self, c):
        """The first-dimension product on the first and the last slice, and process_query, in every layout and from every
        source of the database."""
        S, P = _gpu(), c.P
        for fmt in c.formats:
            for src in c.sources:
                if (fmt, src) == (2, "words"):
                    d, own = c.gdb, False
                else:
                    d, own = (S.Database.from_words(c.G, c.db, fmt=fmt) if src == "words" else S.Database(c.G, fmt=fmt)), True
                    if src == "synthetic":
                        d.fill_synthetic(SEED)
                try:
                    assert d.info()["format"] == fmt
                    for s in sorted({0, P.slices - 1}):
                        assert np.array_equal(S.multiply_reg_by_database(c.G, d, s, c.v), c.product(s)), (fmt, src, s)
                    for k in c.layout_queries:
                        got = S.process_query(c.G, c.gpp, S.Query(ct=c.cts[k]), d)
                        assert np.array_equal(got, c.ref(k)), (fmt, src, c.idxs[k])
                finally:
                    if own:
                        d.close()

    def test_fold_three_ways(self, c):
        """fold_ciphertexts over all 2^nu_2 first-dimension outputs, compared in every slot (the reference folds in place and
        leaves partial sums behind): with the caller's v_folding_neg, on the fast path, and with the raw value q in the input,
        which the fast path cannot represent.  Also get_v_folding_neg."""
        S, P, d = _gpu(), c.P, c.stages()
        assert np.array_equal(S.get_v_folding_neg(c.G, d["v_folding"]), d["v_folding_neg"])
        inter = P.from_ntt(d["first_mult"])
        ref = P.fold_ciphertexts(inter, d["v_folding"], d["v_folding_neg"])
        got = inter.copy()
        S.fold_ciphertexts(c.G, got, d["v_folding"], d["v_folding_neg"])
        assert np.array_equal(got, ref)
        fast = inter.copy()
        S.fold_ciphertexts(c.G, fast, d["v_folding"])
        assert np.array_equal(fast, ref)
        # q in slot 0, in slot 1 (read by the last round only) and in the last slot (read by the first round only)
        withq = inter.copy().reshape(P.num_per, 2, P.N)
        withq[0, 0, 0] = withq[0, 1, P.N - 1] = P.modulus
        withq[min(1, P.num_per - 1), 1, 5] = P.modulus
        withq[P.num_per - 1, 0, 1000] = P.modulus
        withq = withq.reshape(-1)
        refq = P.fold_ciphertexts(withq, d["v_folding"], d["v_folding_neg"])
        S.fold_ciphertexts(c.G, withq, d["v_folding"])
        assert np.array_equal(withq, refq)

    def test_sub_folds(self, c):
        """Every shorter fold, 2^k ciphertexts for k = 1 .. nu_2 - 1: rounds k - 1 .. 0 of the tree, every slot, on both paths."""
        S, P, d = _gpu(), c.P, c.stages()
        inter = P.from_ntt(d["first_mult"])
        for k in range(1, P.nu_2):
            sub = inter[: (1 << k) * 2 * P.N].copy()
            ref = P.fold_ciphertexts(sub, d["v_folding"], d["v_folding_neg"])
            fast = sub.copy()
            S.fold_ciphertexts(c.G, fast, d["v_folding"])
            assert np.array_equal(fast, ref), k
            S.fold_ciphertexts(c.G, sub, d["v_folding"], d["v_folding_neg"])
            assert np.array_equal(sub, ref), k

    def test_pack_and_encode(self, c):
        S, P, d = _gpu(), c.P, c.stages()
        nn = P.n * P.n
        for inst in range(P.instances):
            cts = d["folded"][inst * nn * 2 * P.N:(inst + 1) * nn * 2 * P.N]
            assert np.array_equal(S.pack(c.G, c.gpp, cts), P.pack(cts, c.pp["pack"]))
        assert np.array_equal(S.encode(c.G, d["packed"]), c.ref(0))

    def test_responses(self, c):
        """process_query alone; process_query_batch of 16 queries (one database pass) and of 17 (two passes)."""
        S, P = _gpu(), c.P
        got = S.process_query(c.G, c.gpp, S.Query(ct=c.cts[0]), c.gdb)
        assert np.array_equal(got, c.ref(0))
        assert np.array_equal(c.cl.decode_response(got), P.db_plain_item(SEED, c.idxs[0]))
        for count in (16, BATCH):
            out = S.process_query_batch(c.G, c.gpp, np.concatenate(c.cts[:count]), c.gdb)
            for k in range(count):
                assert np.array_equal(out[k], c.ref(k)), (count, c.idxs[k])

    def test_serialized_queries(self, c):
        """16 serialized queries through process_query_bytes, with the public parameters deserialized too."""
        S = _gpu()
        gpp = S.PublicParameters.deserialize(c.G, c.cl.pp_bytes())
        try:
            out = S.process_query_bytes(c.G, gpp, np.concatenate(c.qbytes[:16]), c.gdb)
        finally:
            gpp.close()
        for k in range(16):
            assert np.array_equal(out[k], c.ref(k)), c.idxs[k]


@pytest.fixture(scope="class")
def s8():
    case = _Case("S8", O.PARAM_SETS["S8"], (10, 6, True), (2, 1, 0), ("words", "synthetic"), (0, 1, 2))
    yield case
    case.close()


@pytest.fixture(scope="class", params=list(SETS))
def deeper(request):
    case = _deep_case(request.param)
    yield case
    case.close()


class TestS8(_Stages):
    """bench.py's configuration, 8 GiB in HBM: the host database and from_words, and fill_synthetic on the GPU, in every
    layout."""

    @pytest.fixture
    def c(self, s8):
        return s8

    def test_queries_of_two_clients_in_one_pass(self, c):
        S, P = _gpu(), c.P
        cl_b = O.Client(P, 777)
        pp_b = cl_b.generate_keys()
        gpp_b = S.PublicParameters(c.G, pp_b["pack"], pp_b["left"], pp_b["right"], pp_b["conv"])
        idx_b = [5, c.total - 2, 99999, 256 * 3 + 255]
        cts_b = [cl_b.generate_query(i)["ct"] for i in idx_b]
        plan = []                                                   # (public parameters, ct, oracle response), interleaved
        for k in range(4):
            plan.append((c.gpp, c.cts[k], c.ref(k)))
            plan.append((gpp_b, cts_b[k], P.process_query(pp_b, dict(ct=cts_b[k]), c.db)))
        try:
            out = S.process_queries(c.G, [g for g, _, _ in plan], [q for _, q, _ in plan], c.gdb)
        finally:
            gpp_b.close()
        for k, (_, _, ref) in enumerate(plan):
            assert np.array_equal(out[k], ref), k
        for k, i in enumerate(idx_b):
            assert np.array_equal(cl_b.decode_response(out[2 * k + 1]), P.db_plain_item(SEED, i))


class TestDeeper(_Stages):
    @pytest.fixture
    def c(self, deeper):
        return deeper


def test_f10_sparse_fold_over_empty_upper_half():
    """lib/server's fold (option "sparse_fold": a pair with an all-zero ciphertext is not multiplied) on F10 with rows
    512 .. 1023 empty, so the first round meets zero ciphertexts everywhere and skips whole subtrees: the stage-level fold
    in every slot and the responses of a batch equal the oracle's sparse fold.  A response decodes wherever the oracle's
    does (an item in the empty half comes back as the item its lower twin holds, by design of that shortcut)."""
    S = _gpu()
    kw = dict(O.PARAM_SETS["T"])
    kw.update(SETS["F10"][0])
    P = O.Params(**kw)
    cl = O.Client(P, 4321)
    pp = cl.generate_keys()
    sdb = P.generate_db(SEED).reshape(P.slices, P.N, P.num_per, P.dim0)
    sdb[:, :, P.num_per // 2:, :] = 0
    sdb = sdb.reshape(-1)
    G = S.Params(**kw)
    gpp = S.PublicParameters(G, pp["pack"], pp["left"], pp["right"], pp["conv"])
    gdb = S.Database.from_words(G, sdb, fmt=2)
    try:
        half = P.num_per // 2
        # three items in the populated half of the rows, three in the empty half
        idxs = [3, (P.dim0 - 1) * P.num_per + half - 1, 40 * P.num_per + 7, half, 17 * P.num_per + half + 100,
                P.dim0 * P.num_per - 1]
        qs = [cl.generate_query(i)["ct"] for i in idxs]
        refs, dump = [], None
        for k, q in enumerate(qs):
            if k == 0:
                r, dump = P.process_query(pp, dict(ct=q), sdb, dump=True, sparse_fold=True)
            else:
                r = P.process_query(pp, dict(ct=q), sdb, sparse_fold=True)
            refs.append(r)
        # stage level: the first-dimension outputs of the upper half are zero
        inter = P.from_ntt(dump["first_mult"])
        assert not inter.reshape(P.num_per, -1)[half:].any() and inter.reshape(P.num_per, -1)[:half].any()
        ref = P.fold_ciphertexts(inter, dump["v_folding"], dump["v_folding_neg"], sparse=True)
        assert np.array_equal(ref[: 2 * P.N], dump["folded"][: 2 * P.N])
        G.set_option("sparse_fold", 1)
        try:
            got = inter.copy()
            S.fold_ciphertexts(G, got, dump["v_folding"])
            out = S.process_query_batch(G, gpp, np.concatenate(qs), gdb)
        finally:
            G.set_option("sparse_fold", 0)
        assert np.array_equal(got, ref)
        decoded = 0
        for k, i in enumerate(idxs):
            want = P.db_plain_item(SEED, i) if i % P.num_per < half else np.zeros(P.N * P.slices, dtype=np.uint64)
            oracle_decodes = np.array_equal(cl.decode_response(refs[k]), want)
            assert np.array_equal(out[k], refs[k]), i
            if oracle_decodes:
                decoded += 1
                assert np.array_equal(cl.decode_response(out[k]), want), i
        assert decoded >= 1
        # the option took effect: the dense fold gives other bytes on this database
        assert not np.array_equal(S.process_query(G, gpp, S.Query(ct=qs[0]), gdb), refs[0])
    finally:
        for h in (gdb, gpp, G):
            h.close()
