"""Host-side mirror of DoublePIR's packed matvec (lib/doublepir/src/matrix/kernels.rs:118-178)."""
import ctypes as C
import os

import numpy as np

from ._lib import LIB, check, B200PirError, DpirParams, DpirInfo  # noqa: F401

# init()'s keys (util/consts.rs:23-33): the first 16 bytes of SHA-256("blyss1") and of SHA-256("blyss2")
SEED_A1 = bytes.fromhex("9c22778545ac229741908e652d333a0f")
SEED_A2 = bytes.fromhex("5fffc482c72a854a10359e9fa2f5e07f")
ENTRY_BYTES, ENTRY_BITS = 0, 1          # load_data's one entry a byte / load_data_fast's eight a byte, LSB first


class PackedMatrix:
    """A squished database matrix (`Matrix` of u32, 3 x 10-bit per word; squish.rs:53-70) resident in HBM."""

    def __init__(self, a=None, rows=None, cols=None, device=0, synthetic_seed=None):
        h = C.c_void_p()
        if a is not None:
            if a.dtype != np.uint32 or not a.flags["C_CONTIGUOUS"] or a.size != rows * cols:
                raise TypeError("a must be a C-contiguous uint32 array of rows*cols words")
            check(LIB.b200pir_dpir_create(device, a.ctypes.data, rows, cols, C.byref(h)))
        else:
            check(LIB.b200pir_dpir_create_synthetic(device, rows, cols, int(synthetic_seed), C.byref(h)))
        self._h, self.rows, self.cols, self.row_begin = h, rows, cols, 0

    @classmethod
    def _adopt(cls, h, rows, cols, row_begin=0):
        m = cls.__new__(cls)
        m._h, m.rows, m.cols, m.row_begin = h, rows, cols, row_begin
        return m

    @classmethod
    def shard(cls, a, row_begin, device=0):
        """A row shard from host words (b200pir_dpir_create_shard): a (rows, cols) uint32 array holding the layout rows
        [row_begin, row_begin + rows) of a database, e.g. rows of the store a load returned or save_to_files wrote."""
        a = np.ascontiguousarray(a, dtype=np.uint32)
        if a.ndim != 2:
            raise TypeError("a must be a (rows, cols) array")
        h = C.c_void_p()
        check(LIB.b200pir_dpir_create_shard(device, a.ctypes.data, int(row_begin), a.shape[0], a.shape[1], C.byref(h)))
        return cls._adopt(h, a.shape[0], a.shape[1], int(row_begin))

    def shard_info(self):
        """dict(row_begin, rows, cols, device) as the handle reports it (b200pir_dpir_shard_info)."""
        r0, rows, cols, dev = C.c_uint64(), C.c_uint64(), C.c_uint64(), C.c_int()
        check(LIB.b200pir_dpir_shard_info(self._h, C.byref(r0), C.byref(rows), C.byref(cols), C.byref(dev)))
        return dict(row_begin=r0.value, rows=rows.value, cols=cols.value, device=dev.value)

    def download(self):
        """The packed words back from HBM (rows x cols u32): what server.rs:147-153 saves as `.dbp`."""
        out = np.zeros((self.rows, self.cols), dtype=np.uint32)
        check(LIB.b200pir_dpir_download(self._h, out.ctypes.data))
        return out

    def close(self):
        if getattr(self, "_h", None):
            LIB.b200pir_dpir_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def matrix_mul_vec_packed(a, b, basis=10, compression=3):
    """kernels.rs:118-178: asserts a.cols * compression == b.rows, basis == 10, compression == 3."""
    assert basis == 10 and compression == 3
    if b.dtype != np.uint32 or b.size != a.cols * compression:
        raise ValueError("a.cols %d compression %d b.rows %d" % (a.cols, compression, b.size))
    out = np.zeros(a.rows, dtype=np.uint32)
    check(LIB.b200pir_dpir_matvec_packed(a._h, b.ctypes.data, out.ctypes.data))
    return out


def matrix_mul_vec_packed_many(a, bs):
    """matrix_mul_vec_packed(a, b) for every b of bs, one pass over a per 64 vectors on the tensor cores (per 16 when too few
    vectors make the integer kernel the faster one): (len(bs), a.rows) uint32."""
    return _matvec_packed_many_on(a, bs, MV_AUTO)


MV_AUTO, MV_MULTI, MV_TC = 0, 1, 2        # B200PIR_DPIR_MV_*


def _matvec_packed_many_on(a, bs, kernel):
    """matrix_mul_vec_packed_many on a named kernel (MV_MULTI: the integer kernel, MV_TC: the tensor cores): for tests and
    measurements; the results do not depend on the kernel."""
    bs = np.ascontiguousarray(np.asarray(bs, dtype=np.uint32).reshape(-1, 3 * a.cols))
    out = np.zeros((bs.shape[0], a.rows), dtype=np.uint32)
    check(LIB.b200pir_dpir_matvec_packed_many_on(a._h, bs.ctypes.data, bs.shape[0], out.ctypes.data, kernel))
    return out


def matrix_mul_vec_packed_rows(a, row_begin, row_count, b):
    """matrix_mul_vec_packed(db.rows(start, n), q) (doublepir.rs:301)."""
    out = np.zeros(row_count, dtype=np.uint32)
    check(LIB.b200pir_dpir_matvec_packed_rows(a._h, row_begin, row_count, b.ctypes.data, out.ctypes.data))
    return out


def matrix_mul_transposed_packed(a, a_rows, a_cols, b, b_rows, b_cols, basis=10, compression=3, device=0):
    """kernels.rs:256-278."""
    assert basis == 10 and compression == 3
    out = np.zeros(a_rows * b_rows, dtype=np.uint32)
    check(LIB.b200pir_dpir_matrix_mul_transposed_packed(device, a.ctypes.data, a_rows, a_cols, b.ctypes.data, b_rows, b_cols,
                                                        out.ctypes.data))
    return out


def transpose_expand_concat_cols_squish(a, rows, cols, modulus, delta, concat, basis=10, d=3, device=0):
    """matrix/indexing.rs:117-143 -> (out, out_rows, out_cols)."""
    assert basis == 10 and d == 3
    orows, ocols = cols * delta * concat, (rows // concat + 2) // 3
    out = np.zeros(orows * ocols, dtype=np.uint32)
    r, c = C.c_uint64(), C.c_uint64()
    check(LIB.b200pir_dpir_transpose_expand_concat_cols_squish(device, a.ctypes.data, rows, cols, modulus, delta, concat,
                                                               out.ctypes.data, C.byref(r), C.byref(c)))
    return out, r.value, c.value


def answer(db, queries, h_1, a_2_transpose, p, delta, x, ne):
    """DoublePIR server answer (doublepir.rs:246-350, raw_data = None, chunk_idx = None).
    db: PackedMatrix; queries: list of [q_1, q_2, ...]; h_1 / a_2_transpose: (array, rows, cols)."""
    nq = len(queries)
    batch = db.rows // nq
    parts, last = [], 0
    for b, q in enumerate(queries):
        bs = db.rows - last if b == nq - 1 else batch
        parts.append(matrix_mul_vec_packed_rows(db, last, bs, q[0]))
        last += bs
    a_1 = np.concatenate(parts)
    a_1, r1, c1 = transpose_expand_concat_cols_squish(a_1, db.rows, 1, p, delta, x)
    a2, a2_rows, a2_cols = a_2_transpose
    msg = [matrix_mul_transposed_packed(a_1, r1, c1, a2, a2_rows, a2_cols)]
    h, h_rows, h_cols = h_1
    hm = PackedMatrix(h, h_rows, h_cols)
    am = PackedMatrix(a_1, r1, c1)
    for q in queries:
        for j in range(ne // x):
            msg.append(matrix_mul_vec_packed(hm, q[1 + j]))
            msg.append(matrix_mul_vec_packed(am, q[1 + j]))
    hm.close()
    am.close()
    return msg


def serialize_state(mats):
    """State::serialize (serializer.rs:56-94): u32 BE count, then per matrix u32 BE rows, cols and data.  A 1-D array is a
    column (len x 1), as answer()'s vectors are."""
    out = [len(mats).to_bytes(4, "big")]
    for a in mats:
        a = np.asarray(a, dtype=np.uint32)
        rows, cols = (a.shape[0], 1) if a.ndim == 1 else a.shape
        out += [int(rows).to_bytes(4, "big"), int(cols).to_bytes(4, "big"), a.astype(">u4").tobytes()]
    return b"".join(out)


def serialize_request(queries):
    """Vec<State>::serialize: what DoublePirServer::answer reads (queries: list of [q_1, q_2, ...])."""
    return len(queries).to_bytes(4, "big") + b"".join(serialize_state(q) for q in queries)


def deserialize_state(buf):
    """Vec<Matrix>::deserialize: a list of (rows, cols) uint32 arrays; trailing bytes are ignored."""
    buf = bytes(buf)
    count, pos, out = int.from_bytes(buf[:4], "big"), 4, []
    for _ in range(count):
        rows, cols = int.from_bytes(buf[pos:pos + 4], "big"), int.from_bytes(buf[pos + 4:pos + 8], "big")
        pos += 8
        out.append(np.frombuffer(buf, dtype=">u4", count=rows * cols, offset=pos).astype(np.uint32).reshape(rows, cols))
        pos += 4 * rows * cols
    return out


class Server:
    """DoublePirServer::answer / answer_inline (doublepir/server.rs:167-180, 235-247) served from HBM.  db: the PackedMatrix
    `load` returns (or one chunk's rows, for answer(.., chunk_idx)), or the list of row shards `load_sharded` returns, which
    may live on several devices (answers are byte for byte the one-GPU server's; no chunked answers); borrowed, it must stay
    open while the server is.  h1_squished / a2_t: the host matrices `load` / `setup` return, uploaded once.  max_queries
    bounds the queries of one call.  device: that of a single db (a sharded server uses its shards' devices)."""

    def __init__(self, db, h1_squished, a2_t, params, num_entries, bits_per_entry, max_queries=32, device=0):
        self.db = db
        self.max_queries = max_queries
        h1 = np.ascontiguousarray(h1_squished, dtype=np.uint32)
        a2 = np.ascontiguousarray(a2_t, dtype=np.uint32)
        h = C.c_void_p()
        if isinstance(db, (list, tuple)):
            dbs = (C.c_void_p * max(len(db), 1))(*[d._h for d in db])
            check(LIB.b200pir_dpir_server_create_sharded(C.byref(_params(params)), num_entries, bits_per_entry, dbs, len(db),
                                                         h1.ctypes.data, a2.ctypes.data, max_queries, C.byref(h)))
        else:
            check(LIB.b200pir_dpir_server_create(device, C.byref(_params(params)), num_entries, bits_per_entry, db._h,
                                                 h1.ctypes.data, a2.ctypes.data, max_queries, C.byref(h)))
        self._h = h
        self._h1_shape = h1.shape
        self._h2_words = h1.shape[0] * int(params["n"]) if h1.ndim == 2 else None     # h2: (n delta x) x n

    def answer_size(self, request):
        n = C.c_size_t()
        check(LIB.b200pir_dpir_answer_size(self._h, bytes(request), len(request), C.byref(n)))
        return n.value

    def _size_or_zero(self, request):
        # a malformed request gets no buffer; the answer call itself then reports why it is refused
        try:
            return self.answer_size(request)
        except B200PirError:
            return 0

    def answer(self, request, chunk_idx=None):
        """msg.serialize() of answer(); chunk_idx = k: answer_inline(.., Some(k)) with this server's matrix as the data."""
        request = bytes(request)
        n = C.c_size_t(self._size_or_zero(request))
        out = C.create_string_buffer(max(n.value, 1))
        check(LIB.b200pir_dpir_answer(self._h, request, len(request), -1 if chunk_idx is None else int(chunk_idx), out, C.byref(n)))
        return out.raw[:n.value]

    def answer_many(self, requests):
        """answer() of every request (different clients, unchunked) in one call: the database is read once per 64 requests on
        the tensor cores (once per 16 when the call has 8 or fewer)."""
        requests = [bytes(r) for r in requests]
        k = len(requests)
        sizes = [self._size_or_zero(r) for r in requests]
        outs = [C.create_string_buffer(max(s, 1)) for s in sizes]
        reqs = (C.c_void_p * k)(*[C.cast(C.c_char_p(r), C.c_void_p) for r in requests])
        lens = (C.c_size_t * k)(*[len(r) for r in requests])
        optr = (C.c_void_p * k)(*[C.cast(o, C.c_void_p) for o in outs])
        olen = (C.c_size_t * k)(*sizes)
        check(LIB.b200pir_dpir_answer_many(self._h, reqs, lens, k, optr, olen))
        return [o.raw[:olen[i]] for i, o in enumerate(outs)]

    def update(self, indices, values, h2):
        """Db::_set of entries `indices` to `values` (bytes, or bits 0/1 for ENTRY_BITS, as the load read them) on the database
        this server borrows, with the store, this server's h_1 and the hint patched to match (b200pir_dpir_server_update): returns
        the new hint, what load() returns as h2 for the modified bytes.  h2: the hint as load() or the previous update left it.
        A repeated index ends with its last value.  Clients must fetch the new hint before they query the updated entries."""
        idx = np.ascontiguousarray(indices, dtype=np.uint64).reshape(-1)
        vals = np.asarray(values).reshape(-1)
        if vals.size != idx.size:
            raise ValueError("%d indices but %d values" % (idx.size, vals.size))
        if vals.size and (vals.min() < 0 or vals.max() > 255):
            raise ValueError("values must be bytes")
        vals = np.ascontiguousarray(vals, dtype=np.uint8)
        out = np.array(h2, dtype=np.uint32, order="C", copy=True)
        if self._h2_words is not None and out.size != self._h2_words:
            raise ValueError("h2 has %d words; this server's hint has %d" % (out.size, self._h2_words))
        check(LIB.b200pir_dpir_server_update(self._h, idx.ctypes.data, vals.ctypes.data, idx.size, out.ctypes.data))
        return out

    def state(self):
        """server_state[0] as the server now holds it: h1_squished, shaped as it was given to the constructor."""
        out = np.zeros(self._h1_shape, dtype=np.uint32)
        check(LIB.b200pir_dpir_server_state(self._h, out.ctypes.data))
        return out

    def close(self):
        if getattr(self, "_h", None):
            LIB.b200pir_dpir_server_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def matmul(a, b, device=0):
    """`&Matrix * &Matrix` (matrix/ops.rs:169-191), wrapping u32, for a left operand with small signed entries (|a| < 2^15):
    exact 8-bit limb products on the tensor cores."""
    a = np.ascontiguousarray(a, dtype=np.uint32)
    b = np.ascontiguousarray(b, dtype=np.uint32)
    if a.ndim != 2 or b.ndim != 2 or a.shape[1] != b.shape[0]:
        raise ValueError("a.cols %r b.rows %r" % (a.shape, b.shape))
    out = np.zeros((a.shape[0], b.shape[1]), dtype=np.uint32)
    check(LIB.b200pir_dpir_matmul(device, a.ctypes.data, a.shape[0], a.shape[1], b.ctypes.data, b.shape[1], out.ctypes.data))
    return out


def setup(db, a1, a2, p, delta, x, device=0):
    """doublepir.rs:76-108 setup(): returns dict(db_squished, h1_squished, a2_t, h2) = (server_state pieces, hint).
    db: l x m with entries centred in [-p/2, p/2) (wrapping u32); a1: m x n; a2: (l/x) x n."""
    db = np.ascontiguousarray(db, dtype=np.uint32)
    a1 = np.ascontiguousarray(a1, dtype=np.uint32)
    a2 = np.ascontiguousarray(a2, dtype=np.uint32)
    l, m = db.shape
    n = a1.shape[1]
    if a1.shape[0] != m or a2.shape != (l // x, n) or l % x:
        raise ValueError("shapes: db (l, m), a1 (m, n), a2 (l/x, n)")
    lx = l // x
    rows1 = n * delta * x
    out = dict(db_squished=np.zeros((l, (m + 2) // 3), dtype=np.uint32), h1_squished=np.zeros((rows1, (lx + 2) // 3), dtype=np.uint32),
               a2_t=np.zeros((n, lx + (3 - lx % 3) % 3), dtype=np.uint32), h2=np.zeros((rows1, n), dtype=np.uint32))
    check(LIB.b200pir_dpir_setup(device, db.ctypes.data, l, m, a1.ctypes.data, n, a2.ctypes.data, p, delta, x,
                                 out["db_squished"].ctypes.data, out["h1_squished"].ctypes.data, out["a2_t"].ctypes.data,
                                 out["h2"].ctypes.data))
    return out


def _params(params):
    return DpirParams(*(int(params[k]) for k in ("n", "l", "m", "logq", "p")))


def db_info(params, num_entries, bits_per_entry):
    """DbInfo::new (database.rs:58-90) + Params::delta(): dict(packing, ne, x, delta).  params: dict with n, l, m, logq, p
    (pick_params' values)."""
    out = DpirInfo()
    check(LIB.b200pir_dpir_db_info(C.byref(_params(params)), num_entries, bits_per_entry, C.byref(out)))
    return dict(packing=out.packing, ne=out.ne, x=out.x, delta=out.delta)


def derive_from_seed(rows, cols, key, device=0):
    """Matrix::derive_from_seed (matrix.rs:125-135) computed on the GPU: rows x cols u32."""
    key = bytes(key)
    if len(key) != 16:
        raise ValueError("key must be 16 bytes")
    out = np.zeros((rows, cols), dtype=np.uint32)
    check(LIB.b200pir_dpir_derive_from_seed(device, key, rows, cols, out.ctypes.data))
    return out


def _load_outputs(params, info):
    n, l = int(params["n"]), int(params["l"])
    x, delta = info["x"], info["delta"]
    lx = l // x
    rows1 = n * delta * x
    return dict(h1_squished=np.zeros((rows1, (lx + 2) // 3), dtype=np.uint32), a2_t=np.zeros((n, lx + (3 - lx % 3) % 3), dtype=np.uint32),
                h2=np.zeros((rows1, n), dtype=np.uint32))


def load(params, num_entries, bits_per_entry, data, entry_format=ENTRY_BYTES, device=0, scratch_bytes=0):
    """DoublePirServer::new + load_data (ENTRY_BYTES) / load_data_fast (ENTRY_BITS) + setup() on the GPU (server.rs:160-165,
    201-229): A_1 and A_2 are derived from SEED_A1 / SEED_A2 on the device.  data: the raw bytes.  The layout is built and
    multiplied band by band of rows, each band in at most scratch_bytes of device scratch (0: 1 GiB); the outputs do not
    depend on it.  Returns (PackedMatrix of the squished database, resident in HBM; dict(h1_squished, a2_t, h2); db_info dict)."""
    info = db_info(params, num_entries, bits_per_entry)
    data = np.ascontiguousarray(np.frombuffer(data, dtype=np.uint8) if isinstance(data, (bytes, bytearray)) else data, dtype=np.uint8)
    out = _load_outputs(params, info)
    h = C.c_void_p()
    check(LIB.b200pir_dpir_load_banded(device, C.byref(_params(params)), num_entries, bits_per_entry, data.ctypes.data, data.size,
                                       entry_format, int(scratch_bytes), C.byref(h), out["h1_squished"].ctypes.data,
                                       out["a2_t"].ctypes.data, out["h2"].ctypes.data))
    return PackedMatrix._adopt(h, int(params["l"]), (int(params["m"]) + 2) // 3), out, info


def load_file(params, num_entries, bits_per_entry, path, entry_format=ENTRY_BITS, device=0, scratch_bytes=0):
    """load() with the raw bytes read from the file at `path` band by band, never held whole in host memory: what
    Db::load_data_fast does with a file (ENTRY_BITS, the default) or load_data with one entry a byte (ENTRY_BYTES)."""
    info = db_info(params, num_entries, bits_per_entry)
    out = _load_outputs(params, info)
    h = C.c_void_p()
    check(LIB.b200pir_dpir_load_file(device, C.byref(_params(params)), num_entries, bits_per_entry, os.fsencode(path), entry_format,
                                     int(scratch_bytes), C.byref(h), out["h1_squished"].ctypes.data, out["a2_t"].ctypes.data,
                                     out["h2"].ctypes.data))
    return PackedMatrix._adopt(h, int(params["l"]), (int(params["m"]) + 2) // 3), out, info


def band_bytes(params, num_entries, bits_per_entry, rows, entry_format=ENTRY_BITS):
    """The device scratch a load's band of `rows` layout rows takes (b200pir_dpir_band_bytes): a scratch_bytes of at least this
    gives bands of at least `rows` rows."""
    out = C.c_uint64()
    check(LIB.b200pir_dpir_band_bytes(C.byref(_params(params)), num_entries, bits_per_entry, entry_format, rows, C.byref(out)))
    return out.value


def shard_rows(params, num_entries, bits_per_entry, shards):
    """The row split of a sharded load (b200pir_dpir_shard_rows): [(row_begin, rows)] of each of `shards` shards, whole units
    of 3x rows, the first U mod G shards one unit longer."""
    out = []
    for g in range(shards):
        r0, rows = C.c_uint64(), C.c_uint64()
        check(LIB.b200pir_dpir_shard_rows(C.byref(_params(params)), num_entries, bits_per_entry, shards, g, C.byref(r0), C.byref(rows)))
        out.append((r0.value, rows.value))
    return out


def _sharded(fn, params, num_entries, bits_per_entry, src, src_len, devices, entry_format, scratch_bytes):
    info = db_info(params, num_entries, bits_per_entry)
    out = _load_outputs(params, info)
    k = len(devices)
    devs = (C.c_int * max(k, 1))(*[int(d) for d in devices])
    hs = (C.c_void_p * max(k, 1))()
    args = [devs, k, C.byref(_params(params)), num_entries, bits_per_entry, src] + ([src_len] if src_len is not None else [])
    check(fn(*args, entry_format, int(scratch_bytes), hs, out["h1_squished"].ctypes.data, out["a2_t"].ctypes.data,
             out["h2"].ctypes.data))
    cols = (int(params["m"]) + 2) // 3
    mats = []
    for h in hs[:k]:
        m = PackedMatrix._adopt(C.c_void_p(h), 0, cols)
        si = m.shard_info()
        m.rows, m.row_begin = si["rows"], si["row_begin"]
        mats.append(m)
    return mats, out, info


def load_sharded(params, num_entries, bits_per_entry, data, devices, entry_format=ENTRY_BYTES, scratch_bytes=0):
    """load() split by rows over len(devices) shards, shard g on devices[g] (a device may repeat): returns (list of
    PackedMatrix row shards, dict(h1_squished, a2_t, h2), db_info dict), the dict byte for byte load()'s and the shards'
    downloads, concatenated, its store.  Distinct devices load at once."""
    data = np.ascontiguousarray(np.frombuffer(data, dtype=np.uint8) if isinstance(data, (bytes, bytearray)) else data, dtype=np.uint8)
    return _sharded(LIB.b200pir_dpir_load_sharded, params, num_entries, bits_per_entry, data.ctypes.data, data.size, devices,
                    entry_format, scratch_bytes)


def load_file_sharded(params, num_entries, bits_per_entry, path, devices, entry_format=ENTRY_BITS, scratch_bytes=0):
    """load_sharded() with the raw bytes read from the file at `path`, each shard its own byte range."""
    return _sharded(LIB.b200pir_dpir_load_file_sharded, params, num_entries, bits_per_entry, os.fsencode(path), None, devices,
                    entry_format, scratch_bytes)
