// Inputs that drive one output of the relaxed-range forward transform (ntt_core.cuh "lz", NTT_OUT_LAZY16: outputs < 16q)
// as close to 16q as a hill climb gets.  The fold, expansion, conversion and pack digit loops add up to 16 products of such
// outputs with key residues (< q) in a uint64_t accumulator between reductions, and 256 q0^2 is 0.9995 * 2^64: random or
// constant digits reach about half of the bound, so the accumulator's headroom is only exercised by inputs searched for it.
// The transform is run with the library's own pass functions (fwd_pass_{a,b,c,d}_lz, which ntt_forward_group_lz and
// ntt_forward_group2_lz are made of), thread by thread as tests/cpp/ntt_core_emul.cpp does.
//
//   ntt_lz_extremes search <out>    deterministic search; writes the records tests/golden/make_lz_extremes.py freezes
//   ntt_lz_extremes eval            stdin lines "<modulus 0|1> <index> <2048 inputs>": prints the LAZY16 output at <index>,
//                                   after checking that every output is < 16q, congruent to the oracle's transform, and
//                                   that no 32-bit sum inside the transform wrapped
#define NTT_RANGE_CHECK 1
#include "../../sdk_b200/csrc/ntt_core.cuh"
#include "../../sdk_b200/csrc/ntt_tables.hpp"
#include "../../oracle/spiral_oracle.hpp"
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <iostream>
#include <random>
#include <sstream>
#include <string>
#include <vector>

using namespace b200pir;
namespace b200pir { int ntt_range_violations = 0; }

namespace {

const uint32_t kQ[2] = {268369921u, 249561089u};

struct Lz {
  uint32_t q, two_q;
  std::vector<Twiddle> fwd, inv;
  std::vector<uint32_t> in, smA, smW;     // inputs (natural order), shared memory after pass A, scratch for passes B-D

  explicit Lz(uint32_t q_) : q(q_), two_q(2 * q_), in(NTT_N, 0), smA(NTT_SMEM_WORDS, 0), smW(NTT_SMEM_WORDS, 0) {
    tables::build_tables(q, fwd, inv);
  }
  // pass A of one thread (strided layout: the thread owns inputs a * 256 + tid)
  void pass_a(int tid) {
    uint32_t x[8];
    for (int a = 0; a < 8; a++) x[a] = in[a * 256 + tid];
    fwd_pass_a_lz<false>(tid, x, smA.data(), TwArray{fwd.data()}, q, two_q);
  }
  void load(const std::vector<uint32_t>& v) {
    in = v;
    for (int t = 0; t < 256; t++) pass_a(t);
  }
  void set(int i, uint32_t v) {
    in[i] = v;
    pass_a(i & 255);
  }
  // output j (contiguous layout: thread j / 8, register j % 8), running passes B-D only for the threads it depends on:
  // pass D thread j/8 reads words [8(j/8), 8(j/8) + 8), written by the 4 pass-C threads of H = j/32, which read the 32 words
  // [32H, 32H + 32), written by the 32 pass-B threads of hi = j/256
  uint32_t out_at(int j) {
    smW = smA;
    uint32_t x[8];
    for (int lo = 0; lo < 32; lo++) fwd_pass_b_lz((j >> 8) * 32 + lo, x, smW.data(), TwArray{fwd.data()}, q, two_q);
    for (int l2 = 0; l2 < 4; l2++) fwd_pass_c_lz((j >> 5) * 4 + l2, x, smW.data(), TwArray{fwd.data()}, q, two_q);
    fwd_pass_d_lz<NTT_OUT_LAZY16>(j >> 3, x, smW.data(), TwArray{fwd.data()}, q, two_q);
    return x[j & 7];
  }
  // every output, every thread
  std::vector<uint32_t> full() {
    std::vector<uint32_t> sm(NTT_SMEM_WORDS, 0), out(NTT_N);
    static uint32_t regs[256][8];
    for (int t = 0; t < 256; t++) for (int a = 0; a < 8; a++) regs[t][a] = in[a * 256 + t];
    for (int t = 0; t < 256; t++) fwd_pass_a_lz<false>(t, regs[t], sm.data(), TwArray{fwd.data()}, q, two_q);
    for (int t = 0; t < 256; t++) fwd_pass_b_lz(t, regs[t], sm.data(), TwArray{fwd.data()}, q, two_q);
    for (int t = 0; t < 256; t++) fwd_pass_c_lz(t, regs[t], sm.data(), TwArray{fwd.data()}, q, two_q);
    for (int t = 0; t < 256; t++) fwd_pass_d_lz<NTT_OUT_LAZY16>(t, regs[t], sm.data(), TwArray{fwd.data()}, q, two_q);
    for (int t = 0; t < 256; t++) for (int k = 0; k < 8; k++) out[t * 8 + k] = regs[t][k];
    return out;
  }
};

// Annealed climb on output j over inputs in [lo, hi]: single-coefficient moves to an end of the window or to a uniform value.
// A move that lowers the output by d is kept with probability exp(-d / T), T falling linearly from q / 2 to 0 (a plain
// climb stalls near 13q: the output is a sum of butterfly terms with a range correction part way, so single moves that
// would cross the correction's threshold only ever lose).  Returns the best inputs seen.
std::vector<uint32_t> climb(Lz& L, int j, uint32_t lo, uint32_t hi, int moves, std::mt19937_64& rng) {
  std::vector<uint32_t> v(NTT_N);
  for (auto& x : v) x = lo + (uint32_t)(rng() % ((uint64_t)hi - lo + 1));
  L.load(v);
  uint32_t cur = L.out_at(j), best = cur;
  std::vector<uint32_t> best_in = L.in;
  std::uniform_real_distribution<double> u01(0.0, 1.0);
  for (int m = 0; m < moves && hi > lo; m++) {
    const int i = (int)(rng() % NTT_N);
    const uint32_t old = L.in[i];
    const int kind = (int)(rng() % 4);
    const uint32_t nv = kind == 0 ? lo : kind == 1 ? hi : lo + (uint32_t)(rng() % ((uint64_t)hi - lo + 1));
    if (nv == old) continue;
    L.set(i, nv);
    const uint32_t s = L.out_at(j);
    const double temp = 0.5 * L.q * (1.0 - (double)m / moves);
    if (s >= cur || (temp > 0 && u01(rng) < std::exp(-((double)cur - s) / temp))) {
      cur = s;
      if (cur > best) { best = cur; best_in = L.in; }
    } else {
      L.set(i, old);
    }
  }
  L.load(best_in);
  return best_in;
}

int bits_of(int t) { return t == 56 ? 1 : 56 / t + 1; }     // gadget.hpp bits_per
int live_of(int t) { const int b = bits_of(t), need = (56 + b - 1) / b; return need < t ? need : t; }

// One record per (modulus, gadget width, window):
//   u8 modulus, u8 bits, u8 window (0 = fold q + delta, 1 = fold top digit q + delta, 2 = raw digit, 3 = raw top digit),
//   u8 bytes per value (2 or 4), u16 target index, u16 reserved (0), then 2048 little-endian signed values: delta
//   (windows 0, 1) or the digit (windows 2, 3)
// Windows 0 and 2 are those of every digit but the top live one: |delta| <= 2^bits - 1, digits in [0, 2^bits).  Windows 1
// and 3 are the top live digit's, limited by the value < q: |delta| <= (q >> bits (live - 1)) - 1, digits up to that limit.
int search(const char* path) {
  const int widths[] = {3, 7, 8, 9, 10, 14, 28, 56};
  // Target outputs, two per modulus in turn over the widths.  How close an output can get to 16q depends on the twiddles
  // on its path (a Shoup product exceeds q only through its quotient's rounding): index 0 and the last pass-D group
  // (2040..2047) stall near 13.3q for both moduli, so the targets are outputs from which the climb reaches 15q.
  const int targets[2][2] = {{1373, 1023}, {1373, 511}};
  const uint64_t Q = (uint64_t)kQ[0] * kQ[1];
  const int moves = 300000;
  std::FILE* f = std::fopen(path, "wb");
  if (!f) { std::perror(path); return 1; }
  for (int m = 0; m < 2; m++) {
    Lz L(kQ[m]);
    const uint32_t q = kQ[m];
    for (int w = 0; w < 8; w++) {
      const int t = widths[w], bits = bits_of(t), live = live_of(t);
      const int j = targets[m][w % 2];
      const int64_t dmax = (1 << bits) - 1, tmax = (int64_t)(Q >> (bits * (live - 1))) - 1;
      for (int win = 0; win < 4; win++) {
        std::mt19937_64 rng(0x5EED0000ull + (uint64_t)m * 1000 + (uint64_t)t * 10 + (uint64_t)win);
        const int64_t lo = win == 0 ? -dmax : win == 1 ? -tmax : 0;
        const int64_t hi = win == 0 || win == 2 ? dmax : tmax;
        const int64_t off = win >= 2 ? 0 : q;
        std::vector<uint32_t> v = climb(L, j, (uint32_t)(off + lo), (uint32_t)(off + hi), moves, rng);
        const uint32_t reached = L.full()[j];
        if (reached != L.out_at(j)) { std::fprintf(stderr, "incremental and full transform disagree\n"); return 1; }
        const int bytes = (hi <= 32767 && lo >= -32768) ? 2 : 4;
        uint8_t head[8] = {(uint8_t)m, (uint8_t)bits, (uint8_t)win, (uint8_t)bytes, (uint8_t)(j & 255), (uint8_t)(j >> 8), 0, 0};
        std::fwrite(head, 1, 8, f);
        for (uint32_t x : v) {
          const int64_t s = (int64_t)x - off;
          uint8_t b[4] = {(uint8_t)s, (uint8_t)(s >> 8), (uint8_t)(s >> 16), (uint8_t)(s >> 24)};
          std::fwrite(b, 1, bytes, f);
        }
        std::fprintf(stderr, "q%d t=%2d bits=%2d window %d index %4d: %.3f q\n", m, t, bits, win, j, (double)reached / q);
      }
    }
  }
  std::fclose(f);
  return 0;
}

int eval() {
  orc::Params p = orc::params_from_scalars(2, 6, 2, 256, 20, 8, 4, 8, 8, 1, 8192, 0, true);
  Lz L0(kQ[0]), L1(kQ[1]);
  std::string line;
  while (std::getline(std::cin, line)) {
    if (line.empty()) continue;
    std::istringstream is(line);
    int m, j;
    is >> m >> j;
    Lz& L = m ? L1 : L0;
    std::vector<uint32_t> v(NTT_N);
    std::vector<uint64_t> ref(2 * NTT_N, 0);
    for (int i = 0; i < NTT_N; i++) {
      uint64_t x;
      if (!(is >> x) || x >= 2ull * L.q) { std::fprintf(stderr, "bad input line (inputs must be < 2q)\n"); return 1; }
      v[i] = (uint32_t)x;
      ref[m * NTT_N + i] = x % L.q;
    }
    orc::ntt_forward(p, ref.data());
    L.in = v;
    const std::vector<uint32_t> out = L.full();
    for (int i = 0; i < NTT_N; i++)
      if (out[i] >= 16ull * L.q || out[i] % L.q != ref[m * NTT_N + i]) {
        std::fprintf(stderr, "output %d out of range or not congruent\n", i);
        return 1;
      }
    if (ntt_range_violations) { std::fprintf(stderr, "range violations: %d\n", ntt_range_violations); return 1; }
    std::printf("%u\n", out[j]);
  }
  return 0;
}

}  // namespace

int main(int argc, char** argv) {
  if (argc == 3 && !std::strcmp(argv[1], "search")) return search(argv[2]);
  if (argc == 2 && !std::strcmp(argv[1], "eval")) return eval();
  std::fprintf(stderr, "usage: %s search <out> | eval\n", argv[0]);
  return 2;
}
