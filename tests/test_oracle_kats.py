"""Pin the CPU oracle against every known-answer test the reference holds for this path
(SURVEY.md §8c).  Each test cites the reference test it restates."""
import ctypes as C

import numpy as np
import pytest

import oracle_lib as O
from oracle_lib import LIB

Q0, Q1 = 268369921, 249561089
Q = Q0 * Q1


@pytest.fixture(scope="module")
def P():
    # util.rs:63-82 get_test_params (n2 nu 9/6 ... t_exp 8/56)
    return O.Params(n=2, nu_1=9, nu_2=6, p=256, q2_bits=20, t_gsw=8, t_conv=4, t_exp_left=8, t_exp_right=56,
                    instances=1, db_item_size=2048, version=0)


def test_build_ntt_tables_correct(P):
    # ntt.rs:379-398
    assert P.ntt_table(0, 2)[0] == 134184961
    assert P.ntt_table(0, 2)[1] == 96647580
    x = 0
    for m in range(2):
        for w in range(4):
            t = P.ntt_table(m, w)
            assert t.size == 2048
            x ^= int(np.bitwise_xor.reduce(t))
    assert x == 519370102


def test_minimal_primitive_roots():
    # SURVEY A.1 (number_theory.rs:41-55)
    assert LIB.orc_min_primitive_root(4096, Q0) == 66687
    assert LIB.orc_min_primitive_root(4096, Q1) == 158221


def test_ntt_forward_correct(P):
    # ntt.rs:400-409
    v = np.zeros(2 * 2048, dtype=np.uint64)
    v[0] = 100
    v[2048] = 100
    out = P.ntt_forward(v)
    assert out[50] == 100 and out[2048 + 50] == 100
    assert np.all(out == 100)


def test_ntt_inverse_correct(P):
    # ntt.rs:411-423
    v = np.full(2 * 2048, 100, dtype=np.uint64)
    out = P.ntt_inverse(v)
    assert out[0] == 100 and out[2048] == 100
    assert out[50] == 0 and out[2048 + 50] == 0


def test_ntt_roundtrip(P):
    # ntt.rs:425-443
    rng = np.random.default_rng(1)
    v = np.concatenate([rng.integers(0, Q0, 2048, dtype=np.uint64), rng.integers(0, Q1, 2048, dtype=np.uint64)])
    assert np.array_equal(P.ntt_inverse(P.ntt_forward(v)), v)


def test_ntt_matches_definition(P):
    # SURVEY A.3: out[k] = sum_i a_i psi^{(2 bitrev(k)+1) i}, checked directly for a few k
    rng = np.random.default_rng(2)
    a = rng.integers(0, Q0, 2048, dtype=np.uint64)
    v = np.concatenate([a, a % np.uint64(Q1)])
    out = P.ntt_forward(v)
    for q, psi, off in ((Q0, 66687, 0), (Q1, 158221, 2048)):
        for k in (0, 1, 5, 1000, 2047):
            br = int(format(k, "011b")[::-1], 2)
            e = 2 * br + 1
            w = pow(psi, e, q)
            acc, pw = 0, 1
            for i in range(2048):
                acc = (acc + int(v[off + i]) * pw) % q
                pw = pw * w % q
            assert out[off + k] == acc


def test_calc_index_correct():
    # ntt.rs:445-449
    def ci(i, l):
        a = np.array(i, dtype=np.uint64)
        b = np.array(l, dtype=np.uint64)
        return LIB.orc_calc_index(O._p64(a), O._p64(b), len(i))
    assert ci([2, 3, 4], [10, 10, 100]) == 2304
    assert ci([2, 3, 4], [3, 5, 7]) == 95


def test_get_barrett_crs_correct(P):
    # arith.rs:476-490
    out = np.zeros(2, dtype=np.uint64)
    for m, exp in ((Q0, (16144578669088582089, 68736257792)), (Q1, (10966983149909726427, 73916747789)),
                   (Q, (7906011006380390721, 275))):
        LIB.orc_barrett_crs(O.C.c_uint64(m), O._p64(out))
        assert (int(out[0]), int(out[1])) == exp
    assert (P.cr0_0, P.cr1_0) == (16144578669088582089, 68736257792)
    assert (P.cr0_mod, P.cr1_mod) == (7906011006380390721, 275)
    assert P.modulus == 66974689739603969  # arith.rs:494


def test_barrett_reduction_u128_raw_correct():
    # arith.rs:492-508 fixed vectors + REAL randomised checks (the reference's `combine` is vacuous, SURVEY A.4)
    f = lambda v: LIB.orc_barrett_reduction_u128_raw(Q, 7906011006380390721, 275, v & (2**64 - 1), v >> 64)
    assert f(Q) == 0
    assert f(Q + 1) == 1
    assert f(Q * 7 + 5) == 5
    rng = np.random.default_rng(3)
    for _ in range(20000):
        # the range crt_compose_2 produces: x*A + y*B with x,y < 2^28, A,B < q  (< 2^85)
        v = int(rng.integers(0, 2**62)) * int(rng.integers(0, 2**23)) + int(rng.integers(0, 2**62))
        assert f(v) == v % Q


def test_barrett_raw_u64_correct():
    # arith.rs:510-520, plus per-modulus constants
    rng = np.random.default_rng(4)
    for _ in range(20000):
        v = int(rng.integers(0, 2**64, dtype=np.uint64))
        assert LIB.orc_barrett_raw_u64(v, 275, Q) == v % Q
        assert LIB.orc_barrett_raw_u64(v, 68736257792, Q0) == v % Q0
        assert LIB.orc_barrett_raw_u64(v, 73916747789, Q1) == v % Q1


def test_div2_uint_mod_correct():
    # arith.rs:456-459
    assert LIB.orc_div2_uint_mod(3, 7) == 5


def test_multiply_negacyclic(P):
    # poly.rs:731-743: (100 X) * (7 X) = 700 X^2
    a = np.zeros(2048, dtype=np.uint64)
    b = np.zeros(2048, dtype=np.uint64)
    a[1] = 100
    b[1] = 7
    prod = P.from_ntt(P.multiply(P.to_ntt(a), P.to_ntt(b), 1, 1, 1))
    exp = np.zeros(2048, dtype=np.uint64)
    exp[2] = 700
    assert np.array_equal(prod, exp)
    # wrap-around sign: X^2047 * X = -1
    a[:] = 0
    b[:] = 0
    a[2047] = 1
    b[1] = 1
    prod = P.from_ntt(P.multiply(P.to_ntt(a), P.to_ntt(b), 1, 1, 1))
    assert prod[0] == Q - 1 and np.all(prod[1:] == 0)


def test_gadget_invert_is_correct(P):
    # gadget.rs:78-95
    mat = np.zeros(2 * 2048, dtype=np.uint64)
    mat[37] = 3
    mat[2048 + 37] = 6
    log_q = P.modulus_log2
    assert log_q == 56
    r = P.gadget_invert(mat, 2, 1, 2 * log_q).reshape(2 * log_q, 2048)
    assert (r[0, 37], r[2, 37], r[4, 37]) == (1, 1, 0)
    assert (r[1, 37], r[3, 37], r[5, 37], r[7, 37]) == (0, 1, 1, 0)


def test_bits_per(P):
    # SURVEY A.7 (gadget.rs:3-9)
    for t, b in ((8, 8), (7, 9), (4, 15), (3, 19), (5, 12), (10, 6), (56, 1)):
        assert P.bits_per(t) == b


def test_bit_io_roundtrip():
    # util.rs:410-428
    data = np.zeros(64, dtype=np.uint8)
    LIB.orc_write_bits(O._p8(data), O.C.c_uint64(33), 0, 20)
    LIB.orc_write_bits(O._p8(data), O.C.c_uint64(0xABCDE), 20, 20)
    LIB.orc_write_bits(O._p8(data), O.C.c_uint64(0x1FFFFF), 50, 21)   # straddles a 64-bit word
    assert LIB.orc_read_bits(O._p8(data), 0, 20) == 33
    assert LIB.orc_read_bits(O._p8(data), 20, 20) == 0xABCDE
    assert LIB.orc_read_bits(O._p8(data), 50, 21) == 0x1FFFFF


def test_params_derived_quantities():
    # util.rs:361-398 (params_from_json == Params::init) — derived fields for the e2e parameter files
    e0 = O.Params.named("E0")
    assert (e0.g, e0.stop_round) == (10, 6)          # t_gsw*nu_2 + dim0 = 40+512 -> 10 ; ceil(log2 40) = 6
    assert e0.query_bytes == 32 + 2048 * 8
    e1 = O.Params.named("E1")
    assert (e1.g, e1.stop_round) == (10, 6)          # 35+512 ; ceil(log2 35)
    # setup_bytes (params.rs:146-167): v1 with t_exp_left == t_exp_right drops the right matrices
    assert e1.setup_bytes == 32 + (2 * 2 * 3 + 10 * 5 + 0 + 2 * 3) * 2048 * 8
    assert e0.setup_bytes == 32 + (4 * 4 * 4 + 10 * 8 + 7 * 56 + 2 * 4) * 2048 * 8


def test_rescale_matches_rounding():
    # arith.rs:429-444: round-half-away-from-zero of centered(a)*out/in, lifted to [0,out)
    from fractions import Fraction
    rng = np.random.default_rng(5)
    for out_mod in (1024, 786433, 3604481):
        for _ in range(2000):
            a = int(rng.integers(0, Q))
            c = a - Q if a >= Q // 2 else a
            # the reference adds sign*(in/2) with in/2 floored, then truncates toward zero
            sign = 1 if c >= 0 else -1
            num = c * out_mod + sign * (Q // 2)
            r = abs(num) // Q * (1 if num >= 0 else -1)
            assert LIB.orc_rescale(a, Q, out_mod) == r % out_mod


def test_chacha20_block_rfc8439_vector():
    # RFC 8439 section 2.3.2 (key 00..1f, counter 1, nonce 00:00:00:09:00:00:00:4a:00:00:00:00): pins the block function
    # the wire formats' seed expansion is built on (rand_chacha 0.3.1; call sites client.rs:218, :309)
    init = np.array([0x61707865, 0x3320646e, 0x79622d32, 0x6b206574,
                     0x03020100, 0x07060504, 0x0b0a0908, 0x0f0e0d0c, 0x13121110, 0x17161514, 0x1b1a1918, 0x1f1e1d1c,
                     0x00000001, 0x09000000, 0x4a000000, 0x00000000], dtype=np.uint32)
    out = np.zeros(16, dtype=np.uint32)
    LIB.orc_chacha20_block(O._p32(init), O._p32(out))
    exp = [0xe4e7f110, 0x15593bd1, 0x1fdd0f50, 0xc47120a3, 0xc7f4d1c7, 0x0368c033, 0x9aaa2204, 0x4e6cd4c3,
           0x466482d2, 0x09aa9f07, 0x05d7c214, 0xa2028bd9, 0xd19c12b5, 0xb94e16de, 0xe883d0cb, 0x4e3c50a2]
    assert [int(x) for x in out] == exp


def test_chacha20rng_stream_matches_rand_chacha_published_vectors():
    # rand_chacha's own known-answer test for ChaCha20Rng (chacha.rs, test_chacha_true_values_a; the crate is a third-party
    # dependency absent from the reference tree, pinned at 0.3.1 in lib/spiral-rs/Cargo.lock): from_seed([0; 32]) yields the
    # keystream of the all-zero key, blocks 0 and 1 (= RFC 7539 appendix A.1 test vectors #1 and #2).  Pins what the block
    # vector above cannot: key placement, block counter in word 12 starting at 0 and incrementing per block, stream id 0,
    # output word order, and next_u64 = low word first (rand_core's BlockRng::next_u64).
    exp = [0xade0b876, 0x903df1a0, 0xe56a5d40, 0x28bd8653, 0xb819d2bd, 0x1aed8da0, 0xccef36a8, 0xc70d778b,
           0x7c5941da, 0x8d485751, 0x3fe02477, 0x374ad8b8, 0xf4b8436a, 0x1ca11815, 0x69b687c3, 0x8665eeb2,
           0xbee7079f, 0x7a385155, 0x7c97ba98, 0x0d082d73, 0xa0290fcb, 0x6965e348, 0x3e53c612, 0xed7aee32,
           0x7621b729, 0x434ee69c, 0xb03371d5, 0xd539d874, 0x281fed31, 0x45fb0a51, 0x1f0ae1ac, 0x6f4d794b]
    seed = np.zeros(32, dtype=np.uint8)
    w = np.zeros(32, dtype=np.uint32)
    LIB.orc_chacha20rng_u32(seed.ctypes.data_as(C.c_void_p), C.c_size_t(32), O._p32(w))
    assert [int(x) for x in w] == exp
    d = np.zeros(16, dtype=np.uint64)
    LIB.orc_chacha20rng_u64(seed.ctypes.data_as(C.c_void_p), C.c_size_t(16), O._p64(d))
    assert [int(x) for x in d] == [exp[2 * i] | (exp[2 * i + 1] << 32) for i in range(16)]
    # a non-trivial seed against an independent evaluation of the same definition
    seed = np.arange(32, dtype=np.uint8) * 7 + 3

    def rotl(v, c):
        return ((v << c) & 0xFFFFFFFF) | (v >> (32 - c))

    def block(init):
        x = list(init)

        def qr(a, b, c, dd):
            x[a] = (x[a] + x[b]) & 0xFFFFFFFF; x[dd] = rotl(x[dd] ^ x[a], 16)
            x[c] = (x[c] + x[dd]) & 0xFFFFFFFF; x[b] = rotl(x[b] ^ x[c], 12)
            x[a] = (x[a] + x[b]) & 0xFFFFFFFF; x[dd] = rotl(x[dd] ^ x[a], 8)
            x[c] = (x[c] + x[dd]) & 0xFFFFFFFF; x[b] = rotl(x[b] ^ x[c], 7)
        for _ in range(10):
            qr(0, 4, 8, 12); qr(1, 5, 9, 13); qr(2, 6, 10, 14); qr(3, 7, 11, 15)
            qr(0, 5, 10, 15); qr(1, 6, 11, 12); qr(2, 7, 8, 13); qr(3, 4, 9, 14)
        return [(x[i] + init[i]) & 0xFFFFFFFF for i in range(16)]
    key = [int.from_bytes(bytes(seed[4 * i:4 * i + 4]), "little") for i in range(8)]
    ref = []
    for ctr in range(3):
        ref += block([0x61707865, 0x3320646E, 0x79622D32, 0x6B206574] + key + [ctr, 0, 0, 0])
    w = np.zeros(48, dtype=np.uint32)
    LIB.orc_chacha20rng_u32(seed.ctypes.data_as(C.c_void_p), C.c_size_t(48), O._p32(w))
    assert [int(x) for x in w] == ref


def test_avx2_transforms_equal_scalar_transforms():
    # the CPU baseline's AVX2 NTTs (restating ntt.rs:120-210, :260-345 with the scalar code's >= comparisons) must be
    # bit-identical to the scalar transforms the parity tests use, including lazy-range and boundary inputs
    P = O.Params.named("T")
    if not LIB.orc_use_avx2_ntt(0):
        pytest.skip("oracle built without AVX2")
    rng = np.random.default_rng(99)
    q = [268369921, 249561089]
    count = 24
    v = np.empty((count, 2, 2048), dtype=np.uint64)
    for n in range(2):
        v[:, n, :] = rng.integers(0, q[n], (count, 2048), dtype=np.uint64)
        v[0, n, :] = 0
        v[1, n, :] = q[n] - 1
        v[2, n, :] = rng.integers(0, 4 * q[n], 2048, dtype=np.uint64)       # lazy-range inputs (< 4q)
        v[3, n, ::2] = q[n] - 1
        v[3, n, 1::2] = 0
    for inverse in (0, 1):
        a, b = v.copy(), v.copy()
        if inverse:      # inverse transforms take values in [0, 2q)
            for n in range(2):
                a[:, n, :] %= np.uint64(2 * q[n])
            b = a.copy()
        assert LIB.orc_ntt_scalar(P.hp, O._p64(a.reshape(-1)), count, inverse) == 0
        assert LIB.orc_ntt_avx2(P.hp, O._p64(b.reshape(-1)), count, inverse) == 0
        assert np.array_equal(a, b), inverse
