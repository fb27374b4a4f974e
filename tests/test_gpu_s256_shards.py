"""S256 (bench.py --workload S256: 2^22 items x 8 KiB, 256 GiB in HBM, rows sharded ii mod 8 over 8 GPUs, 32 GiB a GPU) on
one GPU, shard after shard.  One H100 80GB holds one 32 GiB shard, so the whole 8-GPU step runs here in turn: the copy-engine
pushes and the all-gathers of bench.py's N = 8 flow become concatenations.

  1. the N = 8 step end to end (format 2): 8 ranks expand 16 queries each into their operand tile image, every shard runs the
     first dimension and the 9 local fold rounds of all 128 queries, every rank finishes its 16 (3 rounds, pack, encode); all
     128 responses decode to the synthetic database's items;
  2. byte for byte against the oracle for two queries (item 0 and item 2^22 - 1, shard 7's local row 511 at j = 1023):
     expansion, the first dimension on a row sample of the full 32 GiB shard, the 9 local fold rounds over all 512 rows, and
     the finish;
  3. the mma.sync-fragment and IMAD layouts of shard 7 at 32 GiB give format 2's partials, bit for bit;
  4. raw writes at the far end of the store (the last item of the last slice, and the last row tile of a middle column), the
     pass rerun on shard 7 and the responses decoded again.

The host never holds a shard: the oracle's rows are built item by item from the plaintext generator.  A 32 GiB store puts
byte offsets past 2^34 and the synthetic generator's counter past 2^35, eight 16-query images make 8 groups in one pass, and
world = 8 makes 3 finishing rounds: S8 and the T-size multi-GPU tests reach none of these."""
import ast
import gc
import os

import numpy as np
import pytest

import oracle_lib as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SEED = 0xB1755                     # bench.py's fill_synthetic seed
Q0, Q1 = 268369921, 249561089
GIB = 1 << 30

S256 = dict(n=2, nu_1=10, nu_2=12, p=256, q2_bits=22, t_gsw=8, t_conv=4, t_exp_left=8, t_exp_right=8, instances=1,
            db_item_size=8192, version=0)
WORLD, PER_RANK = 8, 16            # bench.py's N = 8 step: 16 queries per GPU, 128 per step
TOTAL = WORLD * PER_RANK
NUM_PER, DIM0 = 1 << S256["nu_2"], 1 << S256["nu_1"]
ROWS = NUM_PER // WORLD            # local rows of a shard
LOCAL_ROUNDS = 9                   # log2(ROWS): rounds folded on the shard; the other 3 in the finish
SAMPLE_ROWS = (0, 1, 31, 32, 255, 480, 511)      # shard 7's local rows checked against the oracle (tile edges at 32)


def _item(shard, il, j):
    """The item at shard `shard`'s local row il, column j (item idx sits in row idx % num_per, column idx // num_per)."""
    return j * NUM_PER + il * WORLD + shard


LAST = DIM0 * NUM_PER - 1          # shard 7, local row 511, j = 1023: the end of the store
MID = _item(7, 480, 512)           # shard 7, the last row tile (480 .. 511), a middle column
PAIR = (0, LAST)                   # the two queries compared with the oracle stage by stage


def _indices():
    """128 distinct items: 0 and 2^22 - 1; MID; local rows 511, 31 and 32 on other shards; j = 1023; two on every shard;
    then random ones."""
    idxs = [0, LAST, MID, _item(0, 511, 1023), _item(2, 31, 5), _item(3, 32, 700), _item(5, 0, 1023), _item(6, 255, 1)]
    rng = np.random.default_rng(256)
    for s in range(WORLD):
        for _ in range(2):
            idxs.append(_item(s, int(rng.integers(0, ROWS)), int(rng.integers(0, DIM0))))
    while len(set(idxs)) < TOTAL:
        idxs.append(int(rng.integers(0, DIM0 * NUM_PER)))
    return list(dict.fromkeys(idxs))[:TOTAL]


def _item_words(P, idx, data=None):
    """Item idx's packed polynomials [slices][2048]: the plaintext bytes (p = 256: one byte per coefficient) through
    update_item_raw, which packs them exactly as generate_db does (test_item_polynomials_from_plaintext_bytes)."""
    if data is None:
        data = P.db_plain_item(SEED, idx).astype(np.uint8)
    return P.update_item_raw(data).reshape(P.slices, P.N)


def _host_rows(P, shard, rows, slices, written=None):
    """The reference layout [z][row][j] of local rows `rows` of shard `shard`, for each slice in `slices` (-> dict), built item
    by item; written: {idx: raw bytes} overrides."""
    written = written or {}
    out = {sl: np.zeros((P.N, len(rows), DIM0), dtype=np.uint64) for sl in slices}
    for r, il in enumerate(rows):
        for j in range(DIM0):
            idx = _item(shard, il, j)
            w = _item_words(P, idx, written.get(idx))
            for sl in slices:
                out[sl][:, r, j] = w[sl]
    return {sl: a.reshape(-1) for sl, a in out.items()}


def _raw_from_res(res):
    """Residue-form ciphertexts (u32 [poly][n][2048], coefficient domain) -> raw u64 [poly][2048] by the CRT."""
    r = np.ascontiguousarray(res).view(np.uint32).astype(np.uint64).reshape(-1, 2, 2048)
    r0, r1 = r[:, 0], r[:, 1]
    t = (r1 + np.uint64(Q1) - r0 % np.uint64(Q1)) % np.uint64(Q1) * np.uint64(pow(Q0, -1, Q1)) % np.uint64(Q1)
    return (r0 + np.uint64(Q0) * t).reshape(-1)


def _bench_workload(name):
    """bench.py's WORKLOADS[name], read from its source (importing bench.py would set its environment)."""
    tree = ast.parse(open(os.path.join(ROOT, "bench.py")).read())
    for node in tree.body:
        if isinstance(node, ast.Assign) and any(getattr(t, "id", None) == "WORKLOADS" for t in node.targets):
            for k, v in zip(node.value.keys, node.value.values):
                if isinstance(k, ast.Constant) and k.value == name:
                    return eval(compile(ast.Expression(v), "bench.py", "eval"), {"__builtins__": {}, "dict": dict})
    raise KeyError(name)


# ------------------------------------------------------------------------------------------------ CPU
def test_workload_is_bench_s256():
    assert _bench_workload("S256") == S256
    P = O.Params(**S256)
    assert (P.g, P.stop_round, P.slices, P.N) == (11, 7, 4, 2048)
    assert P.t_gsw * P.nu_2 == 96 and DIM0 * NUM_PER == 1 << 22 and P.db_item_size == P.slices * P.N


def test_item_polynomials_from_plaintext_bytes():
    """update_item_raw of an item's plaintext bytes gives that item's packed words in generate_db, so the oracle's rows of a
    shard can be built one item at a time (p = 256, one chunk of 2048 bytes per slice, as in S256)."""
    kw = dict(O.PARAM_SETS["T"])
    kw.update(nu_1=5, nu_2=3)
    P = O.Params(**kw)
    assert P.p == 256 and P.db_item_size == P.slices * P.N
    db = P.generate_db(SEED).reshape(P.slices, P.N, P.num_per, P.dim0)
    total = P.dim0 * P.num_per
    rng = np.random.default_rng(5)
    for idx in [0, 1, P.num_per - 1, P.num_per, total - 1] + [int(x) for x in rng.integers(0, total, 24)]:
        plain = P.db_plain_item(SEED, idx)
        assert plain.max() < 256
        assert np.array_equal(_item_words(P, idx), db[:, :, idx % P.num_per, idx // P.num_per]), idx


# ------------------------------------------------------------------------------------------------ GPU
def _shard_bytes(P):
    """A shard's store: slices x dim0 x local rows x 2048 packed words (Database.info()["hbm_bytes"], asserted in step 1)."""
    return P.slices * DIM0 * ROWS * P.N * 8


def _out_of_memory(e):
    return "out of memory" in str(e).lower()


class _Flow:
    """The client, the GPU context (workspace reserved as a bench rank of the N = 8 step would need it), the 128 queries, and
    step 1's results: the images and folding matrices of the 8 ranks, every shard's partials (gathered), the responses."""

    def __init__(self):
        import torch
        import sdk_b200.spiral as S
        from sdk_b200._lib import LIB, check
        self.torch, self.S, self.LIB, self.check = torch, S, LIB, check
        self.P = P = O.Params(**S256)
        # what earlier tests of this process left in torch's cache is free for this one
        gc.collect()
        torch.cuda.empty_cache()
        self.free_at_start, total = torch.cuda.mem_get_info()
        self.cl = O.Client(P, 256)
        self.pp = self.cl.generate_keys()
        self.G = G = S.Params(**S256)
        self.gpp = S.PublicParameters(G, self.pp["pack"], self.pp["left"], self.pp["right"], self.pp["conv"])
        self._db7, self._images = None, None
        self.idxs = _indices()
        self.cts = [self.cl.generate_query(i)["ct"] for i in self.idxs]
        self.d_q = torch.from_numpy(np.concatenate(self.cts).view(np.int64)).cuda()
        self.img_bytes = int(LIB.b200pir_query_image_bytes(G._h))
        self.fold_words = P.nu_2 * 2 * 2 * P.t_gsw * 2 * P.N
        self.ct_words = 4 * P.N
        self.part_words = TOTAL * P.slices * self.ct_words
        # The workspace is measured, not restated: reserve it, then see what is left for the shard.
        try:
            G.reserve(TOTAL, ROWS)
            self.vf = torch.zeros(TOTAL * self.fold_words, dtype=torch.int32, device="cuda")
            torch.cuda.synchronize()
        except (S.B200PirError, torch.cuda.OutOfMemoryError) as e:
            if not _out_of_memory(e):
                raise
            self.close()
            pytest.skip("S256's workspace does not fit: %.1f GiB free of %.1f GiB (%s)" % (self.free_at_start / GIB, total / GIB, e))
        self.free_beside_workspace = torch.cuda.mem_get_info()[0]
        # Beside it: a shard, the 8 images and 1 GiB for the stages' temporaries.
        need = _shard_bytes(P) + WORLD * self.img_bytes + GIB
        if self.free_beside_workspace < need:
            self.close()
            pytest.skip("S256's shard needs %.1f GiB beside the workspace (%.1f GiB); %.1f GiB are left of %.1f GiB"
                        % (need / GIB, (self.free_at_start - self.free_beside_workspace) / GIB,
                           self.free_beside_workspace / GIB, total / GIB))
        self.gathered = torch.zeros(WORLD * self.part_words, dtype=torch.int32, device="cuda")
        for s in range(WORLD):
            db = self.shard(s)
            if s == 0:
                self.info0 = db.info()
            self.first_dim_fold(db, self.gathered[s * self.part_words:(s + 1) * self.part_words])
            G.synchronize()
            if s == WORLD - 1:
                self._db7, self._db7_dirty = db, False          # kept for the stage-by-stage checks
            else:
                db.close()
        self.free_beside_shard = torch.cuda.mem_get_info()[0]
        self.responses = self.finish(self.gathered)
        self._ref = {}

    def images(self):
        """The 8 ranks' operand tile images (one per rank, 16 queries each); rank r also writes the folding matrices of its
        queries into vf.  Rebuilt on demand after release_images."""
        if self._images is None:
            t = self.torch
            self._images = t.zeros(WORLD * self.img_bytes, dtype=t.uint8, device="cuda")
            for r in range(WORLD):
                self.check(self.LIB.b200pir_expand_queries_images_dev(
                    self.G._h, self.gpp._h, self.d_q.data_ptr() + r * PER_RANK * 2 * self.P.N * 8, PER_RANK,
                    self._images.data_ptr() + r * self.img_bytes, self.vf.data_ptr() + r * PER_RANK * self.fold_words * 4))
        return self._images

    def release_images(self):
        self._images = None
        self.torch.cuda.empty_cache()           # back to the device, where the library allocates

    def shard(self, s, fmt=2):
        """Shard s, filled."""
        db = self.S.Database(self.G, shard_index=s, shard_count=WORLD, fmt=fmt)
        db.fill_synthetic(SEED)
        return db

    def shard7(self):
        """Shard 7 in format 2 as fill_synthetic leaves it."""
        if self._db7 is None or self._db7_dirty:
            self.release_shard7()
            self._db7, self._db7_dirty = self.shard(WORLD - 1), False
        return self._db7

    def release_shard7(self):
        if self._db7 is not None:
            self._db7.close()
        self._db7 = None

    def first_dim_fold(self, db, part):
        """b200pir_first_dim_fold_images_dev: 8 groups of 16 queries against one shard -> its partials [128][slices][ct]."""
        self.check(self.LIB.b200pir_first_dim_fold_images_dev(self.G._h, db._h, self.images().data_ptr(), WORLD, PER_RANK,
                                                              self.vf.data_ptr(), part.data_ptr()))

    def finish(self, gathered):
        """b200pir_finish_queries_dev on every rank -> the 128 responses (host)."""
        rb = self.G.response_bytes
        out = self.torch.zeros(TOTAL * rb, dtype=self.torch.uint8, device="cuda")
        for r in range(WORLD):
            self.check(self.LIB.b200pir_finish_queries_dev(
                self.G._h, self.gpp._h, gathered.data_ptr(), WORLD, TOTAL, r * PER_RANK, PER_RANK,
                self.vf.data_ptr() + r * PER_RANK * self.fold_words * 4, out.data_ptr() + r * PER_RANK * rb))
        self.G.synchronize()
        return out.cpu().numpy().reshape(TOTAL, rb)

    def partial(self, gathered, s, k, sl):
        """Shard s's survivor of query k, slice sl, in residue form (host u32)."""
        base = s * self.part_words + (k * self.P.slices + sl) * self.ct_words
        return gathered[base:base + self.ct_words].cpu().numpy().view(np.uint32)

    def ref(self, idx):
        """The oracle's expand_query of the query for item idx: (v_firstdim, v_folding, v_folding_neg)."""
        if idx not in self._ref:
            v, vf = self.P.expand_query(self.pp, self.cts[self.idxs.index(idx)])
            self._ref[idx] = (v, vf, self.P.get_v_folding_neg(vf))
        return self._ref[idx]

    def close(self):
        self.release_shard7()
        self.d_q = self.vf = self.gathered = None
        self.release_images()                   # also hands torch's cached blocks back to the device for the later tests
        for h in (self.gpp, self.G):
            h.close()


@pytest.fixture(scope="module")
def flow():
    f = _Flow()
    yield f
    f.close()


@pytest.mark.gpu
def test_n8_step_decodes_every_query(flow):
    """Step 1: all 128 responses of the N = 8 step (8 images of 16 queries, 8 shards, 3 finishing rounds) decode to the
    synthetic database's items."""
    P, G = flow.P, flow.G
    assert (G.g, G.stop_round) == (11, 7)
    assert flow.info0["format"] == 2 and flow.info0["local_rows"] == ROWS
    assert flow.info0["hbm_bytes"] == 32 * GIB and flow.info0["present_items"] == flow.info0["capacity"] == P.slices * ROWS * DIM0
    assert sorted({i % NUM_PER % WORLD for i in flow.idxs}) == list(range(WORLD))
    print("\nS256 N = 8 step: %.1f GiB free at the start, %.1f GiB beside the workspace, %.1f GiB beside it, a shard and the images"
          % (flow.free_at_start / GIB, flow.free_beside_workspace / GIB, flow.free_beside_shard / GIB))
    bad = [i for k, i in enumerate(flow.idxs)
           if not np.array_equal(flow.cl.decode_response(flow.responses[k]), P.db_plain_item(SEED, i))]
    assert not bad, bad


@pytest.mark.gpu
def test_expansion_and_folding_matrices_equal_oracle(flow):
    """Step 2a: expand_query of the two queries, and the folding matrices the image expansion of step 1 wrote for them."""
    S, P = flow.S, flow.P
    for idx in PAIR:
        k = flow.idxs.index(idx)
        v_ref, vf_ref, _ = flow.ref(idx)
        v, vf = S.expand_query(flow.G, flow.gpp, S.Query(ct=flow.cts[k]))
        assert np.array_equal(v, v_ref), idx
        assert np.array_equal(vf, vf_ref), idx
        got = flow.vf[k * flow.fold_words:(k + 1) * flow.fold_words].cpu().numpy().view(np.uint32).astype(np.uint64)
        assert np.array_equal(got, vf_ref), idx


@pytest.mark.gpu
def test_first_dimension_row_sample_equals_oracle(flow):
    """Step 2b: multiply_reg_by_database on the full 32 GiB shard 7, slices 0 and 3 (the last one ends the store), on local
    rows at both ends and at row-tile edges, equals the oracle's product of those rows."""
    S, P = flow.S, flow.P
    db = flow.shard7()
    host = _host_rows(P, WORLD - 1, SAMPLE_ROWS, (0, P.slices - 1))
    for idx in PAIR:
        v = flow.ref(idx)[0]
        for sl, rows_db in host.items():
            got = S.multiply_reg_by_database(flow.G, db, sl, v).reshape(ROWS, 4 * P.N)[list(SAMPLE_ROWS)]
            ref = P.multiply_reg_by_database(rows_db, v, dim0=DIM0, num_per=len(SAMPLE_ROWS)).reshape(len(SAMPLE_ROWS), -1)
            assert np.array_equal(got, ref), (idx, sl)


@pytest.mark.gpu
def test_local_fold_equals_oracle(flow):
    """Step 2c: the 9 local fold rounds over all 512 rows of shard 7, every slice: the oracle folds the GPU's first-dimension
    products with v_folding[11] .. v_folding[3] (server.rs:388-427 folds 2^d ciphertexts with v_folding[d - 1] .. [0], so the
    shard's 512 take the matrices of the first 9 of S256's 12 rounds), and the result equals shard 7's partials of step 1."""
    S, P = flow.S, flow.P
    db = flow.shard7()
    mat = 2 * 2 * P.t_gsw * P.W
    first = P.nu_2 - LOCAL_ROUNDS
    for idx in PAIR:
        k = flow.idxs.index(idx)
        v, vf, vfn = flow.ref(idx)
        vf_l, vfn_l = np.ascontiguousarray(vf[first * mat:]), np.ascontiguousarray(vfn[first * mat:])
        for sl in range(P.slices):
            raw = P.from_ntt(S.multiply_reg_by_database(flow.G, db, sl, v))
            ref = P.fold_ciphertexts(raw, vf_l, vfn_l)[: 2 * P.N]
            got = _raw_from_res(flow.partial(flow.gathered, WORLD - 1, k, sl))
            assert np.array_equal(got, ref), (idx, sl)


@pytest.mark.gpu
def test_finish_equals_oracle(flow):
    """Step 2d: the 8 shards' survivors of each slice, in shard order, folded with v_folding[2] .. [0]; pack, from_ntt and
    encode: the response bytes of step 1."""
    P = flow.P
    nn = P.n * P.n
    for idx in PAIR:
        k = flow.idxs.index(idx)
        _, vf, vfn = flow.ref(idx)
        folded = []
        for sl in range(P.slices):
            survivors = np.concatenate([_raw_from_res(flow.partial(flow.gathered, s, k, sl)) for s in range(WORLD)])
            folded.append(P.fold_ciphertexts(survivors, vf, vfn)[: 2 * P.N])
        packed = [P.from_ntt(P.pack(np.concatenate(folded[i * nn:(i + 1) * nn]), flow.pp["pack"])) for i in range(P.instances)]
        assert np.array_equal(P.encode(np.concatenate(packed)), flow.responses[k]), idx


@pytest.mark.gpu
def test_writes_at_the_far_end_of_the_store(flow):
    """Step 4: /update-row writes of item 2^22 - 1 (its slice-3 bytes end the store) and of an item in the last row tile of a
    middle column, on shard 7; shard 7's pass rerun on the same images, the other shards' partials reused.  The written items
    decode to the new bytes, every other query to its old item; presence stays dense; the row sample equals the oracle's with
    the written items converted by update_item_raw."""
    S, P = flow.S, flow.P
    db = flow.shard7()
    before = db.info()
    rng = np.random.default_rng(44)
    written = {i: rng.integers(0, 256, P.db_item_size, dtype=np.uint8) for i in (LAST, MID)}
    body = b"".join((4 + d.size).to_bytes(4, "big") + i.to_bytes(4, "big") + d.tobytes() for i, d in written.items())
    flow._db7_dirty = True
    assert db.update_many_items(body) == 4 + P.db_item_size
    after = db.info()
    assert after["present_items"] == before["present_items"] == before["capacity"]
    gathered = flow.gathered.clone()
    flow.first_dim_fold(db, gathered[(WORLD - 1) * flow.part_words:])
    responses = flow.finish(gathered)
    for k, i in enumerate(flow.idxs):
        want = written[i].astype(np.uint64) if i in written else P.db_plain_item(SEED, i)
        assert np.array_equal(flow.cl.decode_response(responses[k]), want), i
    host = _host_rows(P, WORLD - 1, SAMPLE_ROWS, (0, P.slices - 1), written)
    v = flow.ref(0)[0]
    for sl, rows_db in host.items():
        got = S.multiply_reg_by_database(flow.G, db, sl, v).reshape(ROWS, 4 * P.N)[list(SAMPLE_ROWS)]
        ref = P.multiply_reg_by_database(rows_db, v, dim0=DIM0, num_per=len(SAMPLE_ROWS)).reshape(len(SAMPLE_ROWS), -1)
        assert np.array_equal(got, ref), sl


@pytest.mark.gpu
def test_fragment_and_imad_layouts_at_32_gib(flow):
    """Step 3: shard 7 in format 1 (mma.sync fragments) and format 0 (IMAD cells), one at a time; the non-image flow
    (b200pir_expand_queries_dev per rank, b200pir_first_dim_fold_dev over all 128 queries) gives format 2's partials."""
    torch, S, P = flow.torch, flow.S, flow.P
    flow.release_shard7()
    flow.release_images()
    want = flow.gathered[(WORLD - 1) * flow.part_words:]
    qexp_words = DIM0 * P.N * 4
    qexp = vf = None
    for fmt in (1, 0):
        db = flow.shard(WORLD - 1, fmt=fmt)
        try:
            if qexp is None:
                qexp = torch.zeros(TOTAL * qexp_words, dtype=torch.int32, device="cuda")
                vf = torch.zeros_like(flow.vf)
                for r in range(WORLD):
                    flow.check(flow.LIB.b200pir_expand_queries_dev(
                        flow.G._h, flow.gpp._h, flow.d_q.data_ptr() + r * PER_RANK * 2 * P.N * 8, PER_RANK,
                        qexp.data_ptr() + r * PER_RANK * qexp_words * 4, vf.data_ptr() + r * PER_RANK * flow.fold_words * 4))
                assert torch.equal(vf, flow.vf)
            info = db.info()
            assert info["format"] == fmt and info["local_rows"] == ROWS
            part = torch.zeros_like(want)
            flow.check(flow.LIB.b200pir_first_dim_fold_dev(flow.G._h, db._h, qexp.data_ptr(), vf.data_ptr(), TOTAL,
                                                           part.data_ptr()))
            flow.G.synchronize()
            assert torch.equal(part, want), fmt
        finally:
            db.close()
