// Gadget widths (gadget.rs:3-9), host side and free of CUDA so that tests/cpp/live_digits_check.cpp can compile it alone.
#pragma once

namespace b200pir {

constexpr int kModulusLog2 = 56;      // q = 268369921 * 249561089 < 2^56

// bits per digit of a gadget of dimension t (gadget.rs:3-9 with modulus_log2 = 56)
inline int bits_per(int t) {
  if (t == 56) return 1;
  return kModulusLog2 / t + 1;
}

// Digits of a gadget of dimension t that can be non-zero for a value <= q: digit k covers bits [bits k, bits (k + 1)), and
// q < 2^56, so every digit from ceil(56 / bits) on is zero.  At t = 8 that is the top byte.  A digit loop over values the
// library produced itself (canonical residues CRT-lifted to [0, q), automorphed coefficients in [0, q]) runs only over these:
// a zero digit polynomial transforms to zero, and its products with the key columns add 0 mod q_n to the accumulators.
// Key matrices keep all t columns.
inline int live_digits(int t) {
  const int bits = bits_per(t);
  const int need = (kModulusLog2 + bits - 1) / bits;
  return need < t ? need : t;
}

}  // namespace b200pir
