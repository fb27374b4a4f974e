"""CPU-only: the live-digit count of sdk_b200/csrc/gadget.hpp (run through tests/cpp/live_digits_check.cpp).

The fold, expansion, conversion and pack kernels decompose values that are at most q into only live_digits(t) gadget digits.
That is exact only if every digit from live_digits(t) on is zero for such values, and it saves work only if no smaller count
would do.  Both are checked here for every gadget dimension 3..56: against plain Python integers and against the oracle's
gadget_invert of q, q - 1 and 2^55 (the largest values the kernels decompose, and the highest bit below q's)."""
import math
import os
import subprocess

import numpy as np
import pytest

import oracle_lib as O
import param_space_sets as PS

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def widths(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("ldc") / "live_digits_check")
    subprocess.check_call(["/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++", "-O1", "-std=c++17", "-Wall", "-Werror",
                           "-o", exe, os.path.join(ROOT, "tests", "cpp", "live_digits_check.cpp")])
    rows = [tuple(int(x) for x in ln.split()) for ln in subprocess.check_output([exe], text=True).splitlines()]
    return {t: (bits, live) for t, bits, live in rows}


def test_every_gadget_dimension_is_listed(widths):
    assert sorted(widths) == list(range(3, 57))


def test_live_digits_formula(widths):
    for t, (bits, live) in widths.items():
        assert bits == (1 if t == 56 else 56 // t + 1), t
        assert live == min(t, math.ceil(56 / bits)), t
    assert widths[8] == (8, 7)


@pytest.mark.parametrize("t", range(3, 57))
def test_digits_past_live_are_zero_and_the_last_live_digit_is_not(widths, t):
    kw = dict(PS.BASE)
    P = O.Params(**kw)
    q = P.modulus
    assert q.bit_length() == 56
    bits, live = widths[t]
    v = np.zeros(P.N, dtype=np.uint64)
    v[:3] = [q, q - 1, 1 << 55]
    got = P.gadget_invert(v, 1, 1, t, rdim=1).reshape(t, P.N)
    assert not got[live:].any(), (t, live)
    assert int(got[live - 1, 0]) == (q >> (bits * (live - 1))) & ((1 << bits) - 1) != 0, (t, live)
    for x in (q, q - 1, 1 << 55):                      # the same with plain integers
        assert x >> (bits * live) == 0, (t, x)
