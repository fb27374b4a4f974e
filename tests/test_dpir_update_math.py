"""The four patch identities behind DoublePIR entry updates (b200pir_dpir_server_update, DESIGN §4.5 "Entry updates"), as a
numpy model on the CPU: patching the squished store, h_1 = db A_1, h_1's squished base-p digits and the hint h_2 = H1e A_2 for
a set of changed entries gives exactly what setup() computes from the modified data.  The reference side is the oracle's
load_data and derive (tests/cpp/dpir_load_oracle.cpp) and its setup()."""
import math

import numpy as np
import pytest

import dpir_load_oracle as L
import oracle_lib as O

SEED_A1 = bytes.fromhex("9c22778545ac229741908e652d333a0f")
SEED_A2 = bytes.fromhex("5fffc482c72a854a10359e9fa2f5e07f")
M32 = (1 << 32) - 1


def element_patches(latest, info, bits, m, p):
    """{entry index: new value} -> {(r, c): (mask, val)}: new element = (old & ~mask) | val."""
    out = {}
    for i, v in sorted(latest.items()):
        if info["packing"]:
            e, sh = i // info["packing"], bits * (i % info["packing"])
            fm = ((1 << bits) - 1) << sh
            mask, val = out.get((e // m, e % m), (0, 0))
            out[(e // m, e % m)] = (mask | fm, (val & ~fm) | (v << sh))
        else:
            for j in range(info["ne"]):
                out[((i // m) * info["ne"] + j, i % m)] = (M32, (v // p ** j) % p)
    return out


def patch_digits(h1_sq, C, rows, dh, p, delta):
    """h_1 values stored as delta digits (field C % 3 of column C // 3, at rows[f]) moved by dh (one value per row set):
    returns the digit differences D, one row per digit f."""
    sh, col = 10 * (C % 3), C // 3
    fields = [(h1_sq[rows[f], col].astype(np.int64) >> sh) & 1023 for f in range(delta)]
    old = sum(fields[f] * p ** f for f in range(delta))
    new = (old + dh) & M32
    D = []
    for f in range(delta):
        dd = (new // p ** f) % p - (old // p ** f) % p
        assert np.array_equal((old // p ** f) % p, fields[f])        # the stored digits are the base-p split of the value
        h1_sq[rows[f], col] = ((h1_sq[rows[f], col].astype(np.int64) + (dd << sh)) & M32).astype(np.uint32)
        D.append(dd)
    return D


def model_update(st, a_1, prm, info, delta, bits, updates):
    """The update applied to setup()'s outputs st (db_sq, h1_sq, a2_t, h2), in the order the kernels apply it."""
    p, m, n, x = prm["p"], prm["m"], prm["n"], info["x"]
    st = {k: v.copy() for k, v in st.items()}
    latest = {}
    for i, v in updates:
        latest[int(i)] = int(v)                                      # a repeated index ends with its last value
    dh1 = {}
    for (r, c), (mask, val) in element_patches(latest, info, bits, m, p).items():   # 1. store patch
        sh = 10 * (c % 3)
        w = int(st["db_sq"][r, c // 3])
        old = (w >> sh) & 1023
        d = ((old & ~mask) | val) - old
        st["db_sq"][r, c // 3] = (w + (d << sh)) & M32
        dh1[r] = (dh1.get(r, 0) + d * a_1[c].astype(np.int64)) & M32   # 2. dh_1[r, :] = sum_c delta_rc A_1[c, :]
    for r, dv in dh1.items():                                        # 3. h_1 digits, 4. hint
        b, C = r % x, r // x
        rows = [np.arange(n) * delta + f + n * delta * b for f in range(delta)]
        D = patch_digits(st["h1_sq"], C, rows, dv, p, delta)
        a2 = st["a2_t"][:, C].astype(np.int64)                         # A_2[C, :] = column C of a_2^T
        for f in range(delta):
            st["h2"][rows[f]] = ((st["h2"][rows[f]].astype(np.int64) + D[f][:, None] * a2[None, :]) & M32).astype(np.uint32)
    return st


def setup_from_data(prm, num_entries, bits, data, bits_format):
    info = L.dpir_db_info(num_entries, bits, prm["p"])
    delta = math.ceil(32 / math.log2(prm["p"]))
    l, m, n, x = prm["l"], prm["m"], prm["n"], info["x"]
    db = L.dpir_load_data(data, bits_format, num_entries, bits, l, m, prm["p"])
    a_1 = L.dpir_derive_from_seed(m, n, SEED_A1)
    a_2 = L.dpir_derive_from_seed(l // x, n, SEED_A2)
    return info, delta, a_1, O.dpir_setup(db, l, m, a_1, n, a_2, prm["p"], delta, x)


def modified(data, updates, bits_format):
    data = data.copy()
    for i, v in updates:
        if bits_format:
            data[i >> 3] = (int(data[i >> 3]) & ~(1 << (i & 7))) | (v << (i & 7))
        else:
            data[i] = v
    return data


# (num_entries, bits, p, l, m): packing 9 with a partial last element; ne = x = 2 at p = 512
SHAPES = [(1000, 1, 512, 2, 64), (130, 10, 512, 10, 32)]


@pytest.mark.parametrize("bits_format", [False, True])
@pytest.mark.parametrize("num_entries,bits,p,l,m", SHAPES)
def test_model_reproduces_setup_of_modified_data(num_entries, bits, p, l, m, bits_format):
    prm = dict(n=10, l=l, m=m, logq=32, p=p)                          # n % 4 != 0: A_1 rows start inside AES blocks
    rng = np.random.default_rng(num_entries + 7 * bits + bits_format)
    nbytes = (num_entries + 7) // 8 if bits_format else num_entries
    count = 8 * nbytes if bits_format else nbytes
    hi = 2 if bits_format else min(256, 1 << bits)
    data = rng.integers(0, 256 if bits_format else hi, nbytes, dtype=np.uint8)
    info, delta, a_1, st = setup_from_data(prm, num_entries, bits, data, bits_format)
    packing = info["packing"]
    batches = [
        [(0, 1 - (_entry(data, 0, bits_format) & 1))],                 # index 0
        [(count - 1, hi - 1), (count - 1, 0)],                         # the last index, repeated: the last value wins
        [(i, int(rng.integers(0, hi))) for i in range(max(packing, 1) * 3)],   # whole elements, all three fields of a word
        [(int(i), int(rng.integers(0, hi))) for i in rng.integers(0, count, 40)],
        [(5, _entry(data, 5, bits_format))],                           # a no-op value
    ]
    if packing:
        batches.append([(count - 1 - t, 1) for t in range(count % packing or packing)])   # the partial last element
    for upd in batches:
        want_data = modified(data, upd, bits_format)
        _, _, _, want = setup_from_data(prm, num_entries, bits, want_data, bits_format)
        got = model_update(st, a_1, prm, info, delta, bits, upd)
        for k in ("db_sq", "h1_sq", "a2_t", "h2"):
            assert np.array_equal(got[k], want[k]), (upd[:3], k)
        data, st = want_data, got


def _entry(data, i, bits_format):
    return (int(data[i >> 3]) >> (i & 7)) & 1 if bits_format else int(data[i])


@pytest.mark.parametrize("p", [512, 16, 2])
def test_digit_patch_every_position_zero_and_top(p):
    # h_1 values whose digit f goes 0 -> p - 1 and back, at every position f, in all three fields of one squished word;
    # and the wrap 2^32 - 1 + 1 = 0, which changes every digit at once
    delta = math.ceil(32 / math.log2(p))
    for f in range(delta):
        step = (p - 1) * p ** f if f < delta - 1 else (((1 << 32) - 1) // p ** f) * p ** f   # top digit: as far as 2^32 allows
        top = step // p ** f
        for C in range(3):
            h1_sq = np.zeros((delta, 1), dtype=np.uint32)
            for g in range(3):                                          # the neighbours hold digits of another value
                if g != C:
                    h1_sq[:, 0] |= np.array([(g + 1 + j) % p for j in range(delta)], dtype=np.uint32) << np.uint32(10 * g)
            before = h1_sq.copy()
            rows = [np.array([j]) for j in range(delta)]
            D = patch_digits(h1_sq, C, rows, np.array([step]), p, delta)
            assert [int(d[0]) for d in D] == [top if j == f else 0 for j in range(delta)]
            D = patch_digits(h1_sq, C, rows, np.array([-step & M32]), p, delta)
            assert [int(d[0]) for d in D] == [-top if j == f else 0 for j in range(delta)]
            assert np.array_equal(h1_sq, before)
    h1_sq = np.zeros((delta, 1), dtype=np.uint32)
    rows = [np.array([j]) for j in range(delta)]
    patch_digits(h1_sq, 1, rows, np.array([M32]), p, delta)
    D = patch_digits(h1_sq, 1, rows, np.array([1]), p, delta)
    assert not h1_sq.any() and all(int(d[0]) <= 0 for d in D) and any(int(d[0]) == -(p - 1) for d in D)
