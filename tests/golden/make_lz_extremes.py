"""Freeze the digit polynomials that drive the relaxed-range forward transform to its output bound.

    python tests/golden/make_lz_extremes.py        # rewrites tests/golden/lz_extremes.bin (about 20 s)

tests/cpp/ntt_lz_extremes.cpp searches, with a fixed seed, for inputs whose transform output at a chosen index comes as close
to 16q as it can, for both moduli, every gadget width of tests/test_gpu_param_space.py's WIDTHS and three input windows (fold
digit differences, the fold's top live digit, raw digits).  The record layout is described there and read by
tests/lz_extremes.py.  The search is deterministic: running this again reproduces the file byte for byte."""
import os
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))


def main():
    with tempfile.TemporaryDirectory() as tmp:
        exe = os.path.join(tmp, "ntt_lz_extremes")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-o", exe, os.path.join(ROOT, "tests", "cpp", "ntt_lz_extremes.cpp")])
        path = os.path.join(HERE, "lz_extremes.bin")
        subprocess.check_call([exe, "search", path], stderr=sys.stdout)
    print("wrote", path)


if __name__ == "__main__":
    main()
