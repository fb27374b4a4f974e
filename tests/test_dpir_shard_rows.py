"""The row split of a sharded DoublePIR database (b200pir_dpir_shard_rows), on the host: shards tile [0, l) in units of 3x rows,
the first U mod G shards one unit longer, for shapes where l / x is not a multiple of 3 and where x = 2."""
import pytest

E_BADARG, E_SHAPE = -1, -2


def _D():
    import sdk_b200.doublepir as D
    return D


# (params, num_entries, bits_per_entry, x): pick_params' 2^24 one-bit shape (l = 29), 2^20 10-bit entries (x = 2, l = 32),
# 2^30 and 2^37 one-bit entries; ne = x = 2 at p = 16 and at p = 512 with l / x = 20 and 25
SHAPES = [(dict(n=1024, l=29, m=65536, logq=32, p=512), 1 << 24, 1, 1),
          (dict(n=1024, l=32, m=65536, logq=32, p=512), 1 << 20, 10, 2),
          (dict(n=1024, l=1821, m=65536, logq=32, p=512), 1 << 30, 1, 1),
          (dict(n=1024, l=131072, m=131072, logq=32, p=464), 1 << 37, 1, 1),
          (dict(n=64, l=40, m=64, logq=32, p=16), 300, 8, 2),
          (dict(n=64, l=50, m=32, logq=32, p=512), 130, 10, 2)]


def expected(l, x, shards):
    unit = 3 * x
    units = (l + unit - 1) // unit
    out, u = [], 0
    for g in range(shards):
        k = units // shards + (1 if g < units % shards else 0)
        r0, r1 = u * unit, min(l, (u + k) * unit)
        out.append((r0, r1 - r0))
        u += k
    return out


@pytest.mark.parametrize("prm,num_entries,bits,x", SHAPES)
def test_shard_rows_tile_l(prm, num_entries, bits, x):
    D = _D()
    l = prm["l"]
    assert D.db_info(prm, num_entries, bits)["x"] == x
    units = -(-l // (3 * x))
    for G in sorted(set(list(range(1, 9)) + [units])):
        if G > units:
            continue
        got = D.shard_rows(prm, num_entries, bits, G)
        assert got == expected(l, x, G), G
        end = 0
        for r0, rows in got:
            assert r0 == end and r0 % (3 * x) == 0 and rows > 0
            end += rows
        assert end == l
        sizes = [rows for _, rows in got[:-1]]
        assert max(sizes or [0]) - min(sizes or [0]) <= 3 * x


@pytest.mark.parametrize("prm,num_entries,bits,x", SHAPES)
def test_shard_rows_refuses_zero_and_too_many(prm, num_entries, bits, x):
    D = _D()
    from sdk_b200._lib import LIB
    import ctypes as C
    units = -(-prm["l"] // (3 * x))
    r0, rows = C.c_uint64(7), C.c_uint64(7)
    for shards, index, want in [(0, 0, E_SHAPE), (units + 1, 0, E_SHAPE), (units, units, E_BADARG)]:
        rc = LIB.b200pir_dpir_shard_rows(C.byref(D._params(prm)), num_entries, bits, shards, index, C.byref(r0), C.byref(rows))
        assert rc == want, (shards, index)
        assert r0.value == 7 and rows.value == 7
    with pytest.raises(D.B200PirError) as e:
        D.shard_rows(dict(prm, l=prm["l"] + 1) if x == 2 else dict(prm, l=prm["l"]), num_entries, bits, units + 1)
    assert e.value.code == E_SHAPE
