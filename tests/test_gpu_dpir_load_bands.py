"""DoublePIR's banded load: b200pir_dpir_load_banded and b200pir_dpir_load_file lay out and multiply the database band by
band of rows, so that only the squished store, setup()'s n-wide buffers and one band of scratch are on the device.

* Band boundaries: the shapes of test_gpu_dpir_load.py (both entry formats, partial last groups, ne = 2 at p = 16 and p = 512,
  oversized bytes) at scratch budgets giving one group, a prime number of rows (of groups when a group is ne rows), l - 1 rows
  (l - ne) and every row a band, against the oracle's load_data -> derive -> setup(); bands that start mid-byte; an oversized
  word in any band refused with no handle.
* A file equals the same bytes in memory, at 2^24 and 2^30 entries in both formats and at small and default budgets; an
  empty file; the error codes.
* Past the old limit: seeded files of 2^36 and 2^37 one-bit entries (l * m > 2^32; a store of more than 2^32 words), loaded
  from the file and served, every response decoded by the numpy client.
* Stream order: load_file beside a busy legacy stream gives the same outputs."""
import ctypes as C
import os
import shutil
import tempfile

import numpy as np
import pytest

import test_gpu_dpir_load as T
import test_oracle_doublepir_e2e as E

pytestmark = pytest.mark.gpu

E_BADARG, E_SHAPE, E_UNSUPPORTED = -1, -2, -4
GIB = 1 << 30


def _D():
    import sdk_b200.doublepir as D
    return D


def _launches():
    from sdk_b200._lib import LIB
    LIB.b200pir_kernel_launches.restype = C.c_ulonglong
    return LIB.b200pir_kernel_launches()


def _group(info):
    return 1 if info["packing"] else info["ne"]


def _primes_upto(k):
    return [q for q in range(2, k + 1) if all(q % d for d in range(2, int(q ** 0.5) + 1))]


def _band_choices(l, g):
    """one group, a prime number of groups, l - g rows, every row"""
    groups = l // g
    primes = [q for q in _primes_upto(groups - 1) if q > 1]
    rows = {g, l - g if l > g else g, l}
    if primes:
        rows.add(primes[-1] * g)
    return sorted(r for r in rows if 0 < r <= l)


def _loaded(got):
    dbm, out, info = got
    return dbm.download(), {k: out[k].copy() for k in ("h1_squished", "a2_t", "h2")}


def _same(a, b):
    return np.array_equal(a[0], b[0]) and all(np.array_equal(a[1][k], b[1][k]) for k in a[1])


# ------------------------------------------------------------------ band boundaries against the oracle
@pytest.mark.parametrize("bits_format", [False, True])
@pytest.mark.parametrize("num_entries,bits,p,l,m,nbytes,high", T.SMALL)
def test_bands_equal_oracle(num_entries, bits, p, l, m, nbytes, high, bits_format):
    D = _D()
    rng = np.random.default_rng(num_entries + 17 * bits)
    nbytes = (nbytes + 7) // 8 if bits_format else nbytes
    data = rng.integers(0, 256 if bits_format else high, nbytes, dtype=np.uint8)
    prm = dict(n=64, l=l, m=m, logq=32, p=p)
    fmt = D.ENTRY_BITS if bits_format else D.ENTRY_BYTES
    _, _, _, st = T.oracle_load(prm, num_entries, bits, data, bits_format)
    info = D.db_info(prm, num_entries, bits)
    g = _group(info)
    launches = {}
    for rows in _band_choices(l, g):
        budget = D.band_bytes(prm, num_entries, bits, rows, fmt)
        for b in (budget, budget + 1):                      # exactly one band's bytes, and one byte more: the same bands
            before = _launches()
            got = D.load(prm, num_entries, bits, data, fmt, scratch_bytes=b)
            launches.setdefault(rows, set()).add(_launches() - before)
            T.assert_load_equals(got, st)
            got[0].close()
    # each band issues the same four launches (layout, GEMM image, GEMM, squish); the rest does not depend on the bands
    counts = {rows: c.pop() for rows, c in launches.items() if len(c) == 1}
    assert len(counts) == len(launches)
    for rows, c in counts.items():
        assert c - counts[l] == 4 * (-(-l // rows) - 1), (rows, counts)


@pytest.mark.parametrize("bits,m,l", [(1, 7, 12), (1, 13, 9), (10, 7, 12)])
def test_bands_start_mid_byte(bits, m, l):
    # bit format with odd m: a band of packed rows starts at entry r0 m 9, a band of base-p groups at (r0 / 2) m, mid-byte
    D = _D()
    prm = dict(n=64, l=l, m=m, logq=32, p=512)
    info = D.db_info(prm, 1, bits)
    per_row = m * info["packing"] if info["packing"] else m / info["ne"]
    num_entries = int(l * per_row) - 5                        # a partial last group as well
    data = np.random.default_rng(m * l + bits).integers(0, 256, (num_entries + 7) // 8, dtype=np.uint8)
    _, _, _, st = T.oracle_load(prm, num_entries, bits, data, True)
    g = _group(info)
    starts_mid_byte = False
    for rows in sorted({g, 2 * g, 5 * g}):
        starts_mid_byte |= any(int(r0 * per_row) % 8 for r0 in range(rows, l, rows))
        got = D.load(prm, num_entries, bits, data, D.ENTRY_BITS, scratch_bytes=D.band_bytes(prm, num_entries, bits, rows, D.ENTRY_BITS))
        T.assert_load_equals(got, st)
        got[0].close()
    assert starts_mid_byte


def _load_rc(fn, prm, num_entries, bits, src, fmt, scratch):
    D = _D()
    from sdk_b200._lib import LIB
    h = C.c_void_p()
    bufs = [np.zeros(1 << 22, dtype=np.uint32) for _ in range(3)]
    if fn == "file":
        rc = LIB.b200pir_dpir_load_file(0, C.byref(D._params(prm)), num_entries, bits, os.fsencode(src), fmt, scratch, C.byref(h),
                                        *[b.ctypes.data for b in bufs])
    else:
        src = np.ascontiguousarray(src, dtype=np.uint8)
        rc = LIB.b200pir_dpir_load_banded(0, C.byref(D._params(prm)), num_entries, bits, src.ctypes.data, src.size, fmt, scratch,
                                          C.byref(h), *[b.ctypes.data for b in bufs])
    assert not h.value
    return rc


@pytest.mark.parametrize("band", [0, 4, 9])
def test_oversized_word_in_any_band(band, tmp_path):
    # ten rows of 64 words, one row a band; nine bytes of 255 packed into one word of row `band`
    D = _D()
    prm = dict(n=64, l=10, m=64, logq=32, p=512)
    num_entries = 10 * 64 * 9
    data = np.ones(num_entries, dtype=np.uint8)
    w = band * 64 + 37
    data[9 * w:9 * w + 9] = 255
    one_row = D.band_bytes(prm, num_entries, 1, 1, D.ENTRY_BYTES)
    path = tmp_path / "db.bin"
    path.write_bytes(data.tobytes())
    for scratch in (one_row, 0):
        assert _load_rc("buf", prm, num_entries, 1, data, D.ENTRY_BYTES, scratch) == E_UNSUPPORTED
        assert _load_rc("file", prm, num_entries, 1, str(path), D.ENTRY_BYTES, scratch) == E_UNSUPPORTED


# ------------------------------------------------------------------ a file equals the same bytes in memory
@pytest.mark.parametrize("lg", [24, 30])
@pytest.mark.parametrize("bits_format", [True, False])
def test_file_equals_buffer(lg, bits_format, tmp_path):
    D = _D()
    num_entries = 1 << lg
    prm = E.pick_params(num_entries, 1, E.SEC_PARAM, E.LOGQ)
    fmt = D.ENTRY_BITS if bits_format else D.ENTRY_BYTES
    rng = np.random.default_rng(lg + 100 * bits_format)
    data = rng.integers(0, 256, num_entries // 8, dtype=np.uint8) if bits_format else rng.integers(0, 2, num_entries, dtype=np.uint8)
    path = tmp_path / "db.bin"
    data.tofile(path)
    want = _loaded(D.load(prm, num_entries, 1, data, fmt))
    if lg == 24:                                              # and the oracle, where the host can hold the layout
        _, _, _, st = T.oracle_load(prm, num_entries, 1, data, bits_format)
        assert np.array_equal(want[0], st["db_sq"]) and np.array_equal(want[1]["h2"], st["h2"])
    small = D.band_bytes(prm, num_entries, 1, 7, fmt)         # bands of 7 rows
    for scratch in (small, 0):
        got = D.load_file(prm, num_entries, 1, str(path), fmt, scratch_bytes=scratch)
        assert _same(_loaded(got), want), scratch
        got[0].close()
        if scratch:
            got = D.load(prm, num_entries, 1, data, fmt, scratch_bytes=scratch)
            assert _same(_loaded(got), want)
            got[0].close()


def test_empty_file_equals_empty_buffer(tmp_path):
    D = _D()
    prm = dict(n=64, l=4, m=64, logq=32, p=512)
    path = tmp_path / "empty.bin"
    path.write_bytes(b"")
    for fmt in (D.ENTRY_BITS, D.ENTRY_BYTES):
        want = _loaded(D.load(prm, 100, 1, np.zeros(1, dtype=np.uint8)[:0], fmt))
        _, _, _, st = T.oracle_load(prm, 100, 1, np.zeros(0, dtype=np.uint8), fmt == D.ENTRY_BITS)
        assert np.array_equal(want[0], st["db_sq"])
        got = D.load_file(prm, 100, 1, str(path), fmt, scratch_bytes=D.band_bytes(prm, 100, 1, 1, fmt))
        assert _same(_loaded(got), want)
        got[0].close()


def test_load_file_errors(tmp_path):
    D = _D()
    prm = dict(n=64, l=2, m=64, logq=32, p=512)
    assert _load_rc("file", prm, 100, 1, str(tmp_path / "missing.bin"), D.ENTRY_BYTES, 0) == E_BADARG
    assert _load_rc("file", prm, 100, 1, str(tmp_path), D.ENTRY_BYTES, 0) == E_SHAPE                 # a directory: the read fails
    big = tmp_path / "big.bin"
    big.write_bytes(b"\x01" * (2 * 64 * 9 + 1))                                                      # one entry more than l x m holds
    assert _load_rc("file", prm, 100, 1, str(big), D.ENTRY_BYTES, 0) == E_SHAPE
    assert _load_rc("buf", prm, 100, 1, np.ones(2 * 64 * 9 + 1, dtype=np.uint8), D.ENTRY_BYTES, 0) == E_SHAPE
    ok = tmp_path / "ok.bin"
    ok.write_bytes(b"\x01" * 100)
    assert _load_rc("file", prm, 100, 1, str(ok), 2, 0) == E_BADARG                                   # unknown entry format
    assert _load_rc("file", dict(prm, p=2048), 100, 1, str(ok), D.ENTRY_BYTES, 0) == E_UNSUPPORTED
    with pytest.raises(D.B200PirError) as e:
        D.band_bytes(prm, 100, 1, 3)                                                                  # more rows than l
    assert e.value.code == E_SHAPE


# ------------------------------------------------------------------ past the old limit: 2^36 and 2^37 one-bit entries
def _mem_available():
    with open("/proc/meminfo") as f:
        for line in f:
            if line.startswith("MemAvailable:"):
                return int(line.split()[1]) * 1024
    return 0


def _write_seeded(path, nbytes, seed):
    chunk = 256 << 20
    with open(path, "wb") as f:
        for k, off in enumerate(range(0, nbytes, chunk)):
            f.write(np.random.default_rng([seed, k]).bytes(min(chunk, nbytes - off)))


def _mat_vec_exact(a, v):
    """E.mat_vec (wrapping u32 a v) through float64 BLAS on 16-bit halves: with n = 1024 columns every dot product of halves
    stays below 2^42, so it is exact, and the ahi vhi 2^32 term vanishes modulo 2^32.  The halves of the two shared matrices
    are cached (the cache holds the matrix too, so its id cannot be reused)."""
    if a.size < 1 << 20:
        return _MAT_VEC(a, v)
    key = id(a)
    if key not in _halves:
        a64 = a.astype(np.uint64)
        _halves[key] = (a, (a64 >> np.uint64(16)).astype(np.float64), (a64 & np.uint64(0xFFFF)).astype(np.float64))
        del a64
    _, ahi, alo = _halves[key]
    v64 = np.asarray(v, dtype=np.uint32).astype(np.uint64)
    vhi, vlo = (v64 >> np.uint64(16)).astype(np.float64), (v64 & np.uint64(0xFFFF)).astype(np.float64)
    mod = lambda x: np.mod(x, 2.0 ** 32).astype(np.uint64)
    lo = mod(alo @ vlo)
    mid = (mod(ahi @ vlo) + mod(alo @ vhi)) & np.uint64(0xFFFF)
    return ((lo + (mid << np.uint64(16))) & np.uint64(0xFFFFFFFF)).astype(np.uint32)


_halves = {}
_MAT_VEC = E.mat_vec


@pytest.mark.parametrize("lg", [36, 37])
def test_past_the_old_limit(lg, monkeypatch):
    import torch
    D = _D()
    num_entries = 1 << lg
    prm = E.pick_params(num_entries, 1, E.SEC_PARAM, E.LOGQ)
    info = D.db_info(prm, num_entries, 1)
    l, m, n, p = prm["l"], prm["m"], prm["n"], prm["p"]
    assert l * m > 1 << 32 and p == 464 and info["packing"] == 8
    cols = (m + 2) // 3
    store = l * cols * 4
    if lg == 37:
        assert l * cols > 1 << 32
    nbytes = num_entries // 8
    torch.cuda.empty_cache()
    free_dev = torch.cuda.mem_get_info()[0]
    need_dev = store + 4 * n * (3 * m + 4 * l) + 6 * GIB      # the store, setup()'s n-wide buffers and the tail, band scratch
    if free_dev < need_dev:
        pytest.skip("device memory: %.1f GiB free, %.1f GiB needed" % (free_dev / GIB, need_dev / GIB))
    tmp = tempfile.mkdtemp(prefix="dpir_bands_")
    try:
        free_disk = shutil.disk_usage(tmp).free
        if free_disk < nbytes + GIB:
            pytest.skip("disk: %.1f GiB free in %s, %.1f GiB needed" % (free_disk / GIB, tmp, (nbytes + GIB) / GIB))
        need_host = 6 * m * n * 8 + 2 * GIB                    # the client's A_1 and A_2 with their float halves
        if _mem_available() < need_host:
            pytest.skip("host memory: %.1f GiB available, %.1f GiB needed" % (_mem_available() / GIB, need_host / GIB))
        path = os.path.join(tmp, "db.bin")
        _write_seeded(path, nbytes, lg)
        dbm, out, info = D.load_file(prm, num_entries, 1, path, D.ENTRY_BITS)
        fd = os.open(path, os.O_RDONLY)
        bit = lambda i: (os.pread(fd, 1, i >> 3)[0] >> (i & 7)) & 1
        os.remove(path)                                          # the load is done; the bytes it needs stay readable through fd
        srv = None
        try:
            assert dbm.rows == l and dbm.cols == cols
            info = dict(info, bits=1)
            a_1 = D.derive_from_seed(m, n, D.SEED_A1)
            a_2 = D.derive_from_seed(l // info["x"], n, D.SEED_A2)
            # recover() reads a_2 only through its column sums modulo 2^32; a one-row stand-in keeps it from summing 0.5 GB a call
            a_2_sums = (a_2.astype(np.uint64).sum(axis=0) & np.uint64(0xFFFFFFFF)).reshape(1, n)
            monkeypatch.setattr(E, "mat_vec", _mat_vec_exact)
            # the default budget's band, from the same bound the load applies
            band = 1
            while band < l and D.band_bytes(prm, num_entries, 1, band + 1, D.ENTRY_BITS) <= GIB:
                band += 1
            per_row = m * info["packing"]
            w = 1 << 32                                          # word 2^32 of the store: row w // cols, packed column w % cols
            r32, c32 = w // cols, w % cols
            idxs = [0, num_entries - 1, band * per_row, 2 * band * per_row - 1, (l - 1) * per_row]
            if r32 < l:
                idxs += [(r32 * m + min(3 * c32, m - 1)) * info["packing"] + 3, (r32 * m + m - 1) * info["packing"] + 7,
                         ((r32 + 1) * m) * info["packing"] if r32 + 1 < l else 0, (r32 * m) * info["packing"]]
            rng = np.random.default_rng(lg + 1)
            idxs += [int(v) for v in rng.integers(0, num_entries, 65 - len(idxs))]
            srv = D.Server(dbm, out["h1_squished"], out["a2_t"], prm, num_entries, 1, max_queries=len(idxs))
            qs = [E.query(i, a_1, a_2, prm, info, rng) for i in idxs]
            wires = [D.serialize_request([q]) for _, q in qs]
            assert len(wires) > 64
            many = srv.answer_many(wires)
            import test_gpu_dpir_serve as S
            for k, (i, (client, qmsg)) in enumerate(zip(idxs, qs)):
                want = bit(i)
                assert E.recover(i, out["h2"], qmsg, S.flat(many[k]), a_2_sums, client, prm, info) == want, ("many", k, i)
                if k < 12:
                    alone = srv.answer(wires[k])
                    assert E.recover(i, out["h2"], qmsg, S.flat(alone), a_2_sums, client, prm, info) == want, ("alone", k, i)
        finally:
            os.close(fd)
            if srv is not None:
                srv.close()
            dbm.close()
            _halves.clear()
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
        torch.cuda.empty_cache()


# ------------------------------------------------------------------ stream order
def test_load_file_beside_a_busy_legacy_stream(tmp_path):
    import torch
    D = _D()
    num_entries = 1 << 24
    prm = E.pick_params(num_entries, 1, E.SEC_PARAM, E.LOGQ)
    data = np.random.default_rng(77).integers(0, 256, num_entries // 8, dtype=np.uint8)
    path = tmp_path / "db.bin"
    data.tofile(path)
    small = D.band_bytes(prm, num_entries, 1, 3, D.ENTRY_BITS)
    want = _loaded(D.load(prm, num_entries, 1, data, D.ENTRY_BITS))
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    torch.cuda._sleep(1 << 20)
    e1.record()
    torch.cuda.synchronize()
    cycles = int((1 << 20) * 300.0 / max(e0.elapsed_time(e1), 1e-3))       # about 300 ms of the legacy stream
    for scratch in (small, 0):
        torch.cuda._sleep(cycles)                                          # the legacy default stream is busy
        got = D.load_file(prm, num_entries, 1, str(path), D.ENTRY_BITS, scratch_bytes=scratch)
        res = _loaded(got)
        got[0].close()
        torch.cuda.synchronize()
        assert _same(res, want), scratch
