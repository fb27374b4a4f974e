"""Digit polynomials at the relaxed-range transform's output bound (tests/golden/lz_extremes.bin, made by
tests/golden/make_lz_extremes.py), the operands built from them, and a model of each digit loop's accumulator schedule.

The fold, expansion, conversion and pack kernels (sdk_b200/csrc/poly_kernels.cu) transform gadget-digit polynomials with
outputs < 16q and add their products with key residues (< q) into uint64_t accumulators, reducing whenever acc_room would
let more than 16 products build up.  256 q0^2 = 0.99951 * 2^64.  The fixtures push one transform output per record to
about 15.5q; the constructions here put them into every digit the kernels decompose, and schedule() replays the kernels'
acc_room / cnt sequence to give the accumulator's largest value at the target index."""
import os
import shutil
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
FIXTURE = os.path.join(HERE, "golden", "lz_extremes.bin")
SRC = os.path.join(HERE, "cpp", "ntt_lz_extremes.cpp")

Q0, Q1 = 268369921, 249561089
QN = (Q0, Q1)
Q = Q0 * Q1
N = 2048
WIDTHS = [3, 7, 8, 9, 10, 14, 28, 56]
FOLD, FOLD_TOP, RAW, RAW_TOP = 0, 1, 2, 3


def bits_per(t):
    return 1 if t == 56 else 56 // t + 1


def live_digits(t):
    b = bits_per(t)
    return min(t, -(-56 // b))


def top_limit(t):
    """The largest top live digit of a value < q whose lower digits are arbitrary: (q >> bits (live - 1)) - 1."""
    return (Q >> (bits_per(t) * (live_digits(t) - 1))) - 1


def load():
    """{(modulus, bits, window): (target index, int64[2048])}"""
    data = open(FIXTURE, "rb").read()
    out, pos = {}, 0
    while pos < len(data):
        m, bits, win, nb = data[pos:pos + 4]
        j = data[pos + 4] | (data[pos + 5] << 8)
        pos += 8
        vals = np.frombuffer(data, dtype="<i2" if nb == 2 else "<i4", count=N, offset=pos).astype(np.int64)
        pos += N * nb
        out[(m, bits, win)] = (j, vals)
    return out


def compose(digits, bits):
    """Raw coefficients from digit planes (list of int64[N], digit 0 first)."""
    v = np.zeros(N, dtype=object)
    for k, d in enumerate(digits):
        v = v + (d.astype(object) << (bits * k))
    return v


def fold_pair(F, m, t):
    """(vi, vh): raw coefficients < q whose digit differences vh - vi are the searched delta in every live digit but the
    top one, and the searched top-digit delta in the top one."""
    bits, live = bits_per(t), live_digits(t)
    _, d = F[(m, bits, FOLD)]
    _, dt = F[(m, bits, FOLD_TOP)]
    planes = [d] * (live - 1) + [dt]
    vh = compose([np.maximum(p, 0) for p in planes], bits)
    vi = compose([np.maximum(-p, 0) for p in planes], bits)
    return vi, vh


def raw_digits(F, m, t):
    """Digit planes of the raw-window construction: the searched digits in every live digit below the top two, the same
    raised to at least 1 in digit live - 2 (no coefficient is zero: after an automorphism's sign flip the expansion would
    see q in its place), and the searched top digit (<= top_limit(t), so every value is < q)."""
    bits, live = bits_per(t), live_digits(t)
    _, d = F[(m, bits, RAW)]
    _, dt = F[(m, bits, RAW_TOP)]
    return [d] * (live - 2) + [np.maximum(d, 1), dt]


def raw_coeffs(F, m, t):
    return compose(raw_digits(F, m, t), bits_per(t))


def expansion_slot(c):
    """Raw coefficients a with tau(a) = c for round 0's automorphism X -> X^(N + 1): coefficient k keeps its place and
    changes sign when k is odd (c must have no zero there)."""
    a = np.array(c, dtype=object)
    a[1::2] = Q - a[1::2]
    return a


def expansion_half1(a):
    """The coefficients round 0 decomposes for its second output: a shifted negacyclically by one place, then tau (the
    kernel's CRT lift of a negated residue pair is Q - v, zero stays zero; tau maps an odd-place zero to q)."""
    a = [int(x) for x in a]
    s = a[1:] + [(Q - a[0]) % Q]
    return np.array([(Q - v) if k & 1 else v for k, v in enumerate(s)], dtype=object)


def digits_of(v, bits, count):
    v = [int(x) for x in v]
    mask = (1 << bits) - 1
    return [np.array([(x >> (bits * k)) & mask for x in v], dtype=np.int64) for k in range(count)]


class Emul:
    """tests/cpp/ntt_lz_extremes.cpp eval: LAZY16 outputs of the library's own forward-transform passes."""

    def __init__(self, exe):
        self.exe = exe
        self.cache = {}

    def outputs(self, queries):
        """queries: [(modulus, index, inputs < 2q)] -> [output at index]"""
        todo = [qq for qq in queries if self._key(qq) not in self.cache]
        if todo:
            lines = "".join(f"{m} {j} " + " ".join(str(int(x)) for x in v) + "\n" for m, j, v in todo)
            out = subprocess.run([self.exe, "eval"], input=lines, capture_output=True, text=True, check=True).stdout.split()
            for qq, o in zip(todo, out):
                self.cache[self._key(qq)] = int(o)
        return [self.cache[self._key(qq)] for qq in queries]

    @staticmethod
    def _key(qq):
        m, j, v = qq
        return m, j, tuple(int(x) for x in v)


def build_emul(tmpdir):
    exe = os.path.join(str(tmpdir), "ntt_lz_extremes")
    subprocess.check_call([shutil.which("g++") or "g++", "-O2", "-std=c++17", "-o", exe, SRC])
    return Emul(exe)


def schedule(kernel, m, t, x, limit=16, carry_cnt=1):
    """Largest accumulator value of one kernel at modulus m at the target index, and the most products held at once.

    x(k, r) = the transform output at the target index of digit k of the polynomial r the kernel decomposes there
    (fold: row r; fold_round: r = 2 src + row; expand: half r; pack: 0).  Keys are q_n - 1.  The sequence is that of
    poly_kernels.cu: acc_room(n) reduces when cnt + n > limit (after which the residue counts as one), digits go in
    pairs where the kernel pairs them.  carry_cnt: what the expansion counts its carried digit as."""
    live = live_digits(t)
    return _Acc(QN[m], limit, carry_cnt).run(kernel, t, live, x)


class _Acc:
    def __init__(self, q_n, limit, carry_cnt):
        self.q_n, self.limit, self.carry_cnt = q_n, limit, carry_cnt

    def run(self, kernel, t, live, x):
        self.peaks = []
        self.key = None
        if kernel == "fold":                       # k_fold_res_lz
            self.start()
            for r in range(2):
                for k in range(0, live - 1, 2):
                    self.room(2)
                    self.add(x(k, r), x(k + 1, r))
            if live & 1:
                self.room(2)
                self.add(x(live - 1, 0), x(live - 1, 1))
        elif kernel == "fold_round":               # k_fold_round: t digits of each (source, row), one at a time
            self.start()
            for r in range(4):
                for k in range(t):
                    self.room(1)
                    self.add(x(k, r))
        elif kernel == "expand":                   # k_expand_round_res, half 1 then half 0
            for half in (1, 0):
                self.start()
                if half == 0 and live & 1:
                    self.add(x(live - 1, 0))
                    self.cnt = self.carry_cnt
                self.pairs(live & ~1, lambda k: x(k, half))
                if half == 1 and live & 1:
                    self.room(1)
                    self.add(x(live - 1, 1))
        elif kernel == "pack":                     # k_pack, raw ciphertexts: all t digits
            self.start()
            self.pairs(t, lambda k: x(k, 0))
        self.close()
        return max(p[0] for p in self.peaks), max(p[1] for p in self.peaks)

    def start(self):
        if self.key is not None:
            self.close()
        self.acc, self.cnt, self.held = 0, 0, 0
        self.key = True

    def pairs(self, ndig, xk):
        k = 0
        while k + 1 < ndig:
            self.room(2)
            self.add(xk(k), xk(k + 1))
            k += 2
        if k < ndig:
            self.room(1)
            self.add(xk(k))

    def room(self, n):
        if self.cnt + n > self.limit:
            self.close()
            self.acc %= self.q_n
            self.held = 0
            self.cnt = 1
        self.cnt += n

    def add(self, *vals):
        for v in vals:
            self.acc += v * (self.q_n - 1)
            self.held += 1

    def close(self):
        self.peaks.append((self.acc, self.held))
