// 2048-point negacyclic NTT over one 28-bit CRT modulus, computed cooperatively by a group of
// 256 threads holding 8 coefficients each (sm_90a; also compiles as plain C++ so the index /
// twiddle logic can be emulated thread-by-thread on the CPU, tests/test_ntt_core_emulation.py).
//
// Semantics follow the reference's scalar transforms exactly (lib/spiral-rs/src/ntt.rs:67-113
// forward, :212-258 inverse): Cooley-Tukey / Gentleman-Sande stages with the bit-reversed
// twiddle table `table[m + i]`, Harvey lazy butterflies with W' = floor(W 2^32 / q), final
// correction to the canonical range [0, q).  Outputs are therefore the canonical residues in the
// reference's (bit-reversed) order; only the work decomposition is different:
//
//   stage bits   10 9 8 | 7 6 5 | 4 3 2 | 1 0       (stage mm pairs indices differing in bit 10-mm)
//   pass            A       B       C      D
//   thread owns  e = a*256 + tid            (A: a = bits 10..8)      "strided layout"
//                e = hi*256 + a*32 + lo     (B: tid = hi*32 + lo)
//                e = H*32 + a*4 + l2        (C: tid = H*4 + l2)
//                e = tid*8 + k              (D: k = bits 2..0)       "contiguous layout"
//
// Between passes the 8 values go through shared memory with the padding phys(e) = e + 4*(e>>5)
// (2304 words per transform), which makes every access pattern above bank-conflict free,
// including the 128-bit accesses of pass D.
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define NTT_HD __host__ __device__ __forceinline__
#else
#define NTT_HD inline
#endif

namespace b200pir {

static const int NTT_N = 2048;
static const int NTT_LOG_N = 11;
static const int NTT_THREADS = 256;          // threads cooperating on one transform
static const int NTT_SMEM_WORDS = 2048 + 4 * 64;

struct Twiddle { uint32_t w, wp; };          // W and W' = floor(W * 2^32 / q)

NTT_HD uint32_t ntt_mulhi(uint32_t a, uint32_t b) {
#if defined(__CUDA_ARCH__)
  return __umulhi(a, b);
#else
  return (uint32_t)(((uint64_t)a * b) >> 32);
#endif
}
NTT_HD uint32_t ntt_min(uint32_t a, uint32_t b) { return a < b ? a : b; }
NTT_HD int ntt_phys(int e) { return e + 4 * (e >> 5); }

// Forward (CT) butterfly, ntt.rs:92-103.  x,y in [0,4q) -> x',y' in [0,4q).
NTT_HD void bfly_fwd(uint32_t& x, uint32_t& y, Twiddle tw, uint32_t q, uint32_t two_q) {
  uint32_t cx = ntt_min(x, x - two_q);                 // x - 2q if x >= 2q (unsigned wrap + min)
  uint32_t qt = ntt_mulhi(y, tw.wp);
  uint32_t t = tw.w * y - qt * q;                      // in [0, 2q)
  x = cx + t;
  y = cx + two_q - t;
}
// Inverse (GS) butterfly with the halving folded in, ntt.rs:236-248.  x,y in [0,2q) -> [0,2q).
NTT_HD void bfly_inv(uint32_t& x, uint32_t& y, Twiddle tw, uint32_t q, uint32_t two_q) {
  uint32_t tt = two_q - y + x;                         // in (0, 4q)
  uint32_t s = x + y;
  uint32_t cx = ntt_min(s, s - two_q);                 // x + y - 2q if x + y >= 2q
  uint32_t ht = ntt_mulhi(tt, tw.wp);
  x = (cx + ((tt & 1u) ? q : 0u)) >> 1;
  y = tw.w * tt - ht * q;
}
// final correction, ntt.rs:107-111 / :253-256
NTT_HD uint32_t ntt_canon(uint32_t v, uint32_t q, uint32_t two_q) {
  v = ntt_min(v, v - two_q);
  return ntt_min(v, v - q);
}

// Three butterfly stages over the 3 index bits held in registers (a = 0..7, bit2 = first stage).
// tw_base[s] is the table offset 2^mm of stage s; grp[s] the group index of the thread's a=0
// element at that stage (group of element a is grp[s] + (a >> (3 - s))).
// `tab` is any callable idx -> Twiddle (plain array, __constant__ bank, shared-memory copy ...).
// Accessors also provide load2 / load4 for runs of consecutive entries (index multiple of 2 / 4), so that
// shared-memory tables can be read with 16-byte accesses (conflict-free) instead of strided 8-byte ones.
struct TwArray {
  const Twiddle* p;
  NTT_HD Twiddle operator()(int i) const { return p[i]; }
  NTT_HD void load2(int i, Twiddle (&t)[2]) const { t[0] = p[i]; t[1] = p[i + 1]; }
  NTT_HD void load4(int i, Twiddle (&t)[4]) const { t[0] = p[i]; t[1] = p[i + 1]; t[2] = p[i + 2]; t[3] = p[i + 3]; }
};
template <typename Tab>
NTT_HD void radix8_fwd(uint32_t (&x)[8], Tab tab, int m0, int g0, uint32_t q, uint32_t two_q) {
  // stage s=0: pairs (a, a+4); group = g0                    table idx m0 + g0
  // stage s=1: pairs (a, a+2); group = 2*g0 + (a>>2)         table idx 2*m0 + ...
  // stage s=2: pairs (a, a+1); group = 4*g0 + (a>>1)
  Twiddle t0 = tab(m0 + g0);
  Twiddle t1[2], t2[4];
  tab.load2(2 * m0 + 2 * g0, t1);
  tab.load4(4 * m0 + 4 * g0, t2);
#pragma unroll
  for (int a = 0; a < 4; a++) bfly_fwd(x[a], x[a + 4], t0, q, two_q);
#pragma unroll
  for (int h = 0; h < 2; h++) {
#pragma unroll
    for (int a = 0; a < 2; a++) bfly_fwd(x[4 * h + a], x[4 * h + a + 2], t1[h], q, two_q);
  }
#pragma unroll
  for (int h = 0; h < 4; h++) bfly_fwd(x[2 * h], x[2 * h + 1], t2[h], q, two_q);
}
template <typename Tab>
NTT_HD void radix8_inv(uint32_t (&x)[8], Tab tab, int m0, int g0, uint32_t q, uint32_t two_q) {
  // exact reverse order of radix8_fwd
  Twiddle t1[2], t2[4];
  tab.load4(4 * m0 + 4 * g0, t2);
  tab.load2(2 * m0 + 2 * g0, t1);
#pragma unroll
  for (int h = 0; h < 4; h++) bfly_inv(x[2 * h], x[2 * h + 1], t2[h], q, two_q);
#pragma unroll
  for (int h = 0; h < 2; h++) {
#pragma unroll
    for (int a = 0; a < 2; a++) bfly_inv(x[4 * h + a], x[4 * h + a + 2], t1[h], q, two_q);
  }
  Twiddle t0 = tab(m0 + g0);
#pragma unroll
  for (int a = 0; a < 4; a++) bfly_inv(x[a], x[a + 4], t0, q, two_q);
}

// ---- per-pass thread-local steps.  `tid` in [0,256).  smem = this transform's 2304-word buffer.
// Pass A (stages 0..2) on the strided layout; then store.
template <typename Tab>
NTT_HD void fwd_pass_a(int tid, uint32_t (&x)[8], uint32_t* smem, Tab tab, uint32_t q, uint32_t two_q) {
  radix8_fwd(x, tab, 1, 0, q, two_q);                                  // m = 1,2,4 ; group base 0
#pragma unroll
  for (int a = 0; a < 8; a++) smem[ntt_phys(a * 256 + tid)] = x[a];
}
// Pass B (stages 3..5): e = hi*256 + a*32 + lo
template <typename Tab>
NTT_HD void fwd_pass_b(int tid, uint32_t (&x)[8], uint32_t* smem, Tab tab, uint32_t q, uint32_t two_q) {
  int hi = tid >> 5, lo = tid & 31;
#pragma unroll
  for (int a = 0; a < 8; a++) x[a] = smem[ntt_phys(hi * 256 + a * 32 + lo)];
  radix8_fwd(x, tab, 8, hi, q, two_q);                                 // m = 8,16,32
#pragma unroll
  for (int a = 0; a < 8; a++) smem[ntt_phys(hi * 256 + a * 32 + lo)] = x[a];
}
// Pass C (stages 6..8): e = H*32 + a*4 + l2
template <typename Tab>
NTT_HD void fwd_pass_c(int tid, uint32_t (&x)[8], uint32_t* smem, Tab tab, uint32_t q, uint32_t two_q) {
  int H = tid >> 2, l2 = tid & 3;
#pragma unroll
  for (int a = 0; a < 8; a++) x[a] = smem[ntt_phys(H * 32 + a * 4 + l2)];
  radix8_fwd(x, tab, 64, H, q, two_q);                                 // m = 64,128,256
#pragma unroll
  for (int a = 0; a < 8; a++) smem[ntt_phys(H * 32 + a * 4 + l2)] = x[a];
}
// Pass D (stages 9,10) on the contiguous layout e = tid*8 + k, then canonicalise.
// CANON = false leaves the outputs in the lazy range [0, 4q) (saves the final correction; legal when the values
// only feed a multiply-accumulate that is reduced mod q afterwards).
template <bool CANON = true, typename Tab>
NTT_HD void fwd_pass_d(int tid, uint32_t (&x)[8], const uint32_t* smem, Tab tab, uint32_t q, uint32_t two_q) {
  int base = ntt_phys(tid * 8);                                         // 8 contiguous words (two 16-byte chunks)
#pragma unroll
  for (int k = 0; k < 8; k++) x[k] = smem[base + k];
  Twiddle t9[2], t10[4];
  tab.load2(512 + 2 * tid, t9);
  tab.load4(1024 + 4 * tid, t10);
#pragma unroll
  for (int h = 0; h < 2; h++) {                                         // stage 9: m=512, group = 2*tid + h, pairs (k, k+2)
    bfly_fwd(x[4 * h + 0], x[4 * h + 2], t9[h], q, two_q);
    bfly_fwd(x[4 * h + 1], x[4 * h + 3], t9[h], q, two_q);
  }
#pragma unroll
  for (int h = 0; h < 4; h++) bfly_fwd(x[2 * h], x[2 * h + 1], t10[h], q, two_q);   // stage 10: m=1024, group = 4*tid + h
  if (CANON) {
#pragma unroll
    for (int k = 0; k < 8; k++) x[k] = ntt_canon(x[k], q, two_q);
  }
}

// Inverse: contiguous layout in (values in [0,2q)), strided layout out (canonical).
template <typename Tab>
NTT_HD void inv_pass_d(int tid, uint32_t (&x)[8], uint32_t* smem, Tab tab, uint32_t q, uint32_t two_q) {
  Twiddle t9[2], t10[4];
  tab.load4(1024 + 4 * tid, t10);
  tab.load2(512 + 2 * tid, t9);
#pragma unroll
  for (int h = 0; h < 4; h++) bfly_inv(x[2 * h], x[2 * h + 1], t10[h], q, two_q);   // stage mm=10
#pragma unroll
  for (int h = 0; h < 2; h++) {                                         // stage mm=9
    bfly_inv(x[4 * h + 0], x[4 * h + 2], t9[h], q, two_q);
    bfly_inv(x[4 * h + 1], x[4 * h + 3], t9[h], q, two_q);
  }
  int base = ntt_phys(tid * 8);
#pragma unroll
  for (int k = 0; k < 8; k++) smem[base + k] = x[k];
}
template <typename Tab>
NTT_HD void inv_pass_c(int tid, uint32_t (&x)[8], uint32_t* smem, Tab tab, uint32_t q, uint32_t two_q) {
  int H = tid >> 2, l2 = tid & 3;
#pragma unroll
  for (int a = 0; a < 8; a++) x[a] = smem[ntt_phys(H * 32 + a * 4 + l2)];
  radix8_inv(x, tab, 64, H, q, two_q);
#pragma unroll
  for (int a = 0; a < 8; a++) smem[ntt_phys(H * 32 + a * 4 + l2)] = x[a];
}
template <typename Tab>
NTT_HD void inv_pass_b(int tid, uint32_t (&x)[8], uint32_t* smem, Tab tab, uint32_t q, uint32_t two_q) {
  int hi = tid >> 5, lo = tid & 31;
#pragma unroll
  for (int a = 0; a < 8; a++) x[a] = smem[ntt_phys(hi * 256 + a * 32 + lo)];
  radix8_inv(x, tab, 8, hi, q, two_q);
#pragma unroll
  for (int a = 0; a < 8; a++) smem[ntt_phys(hi * 256 + a * 32 + lo)] = x[a];
}
template <typename Tab>
NTT_HD void inv_pass_a(int tid, uint32_t (&x)[8], const uint32_t* smem, Tab tab, uint32_t q, uint32_t two_q) {
#pragma unroll
  for (int a = 0; a < 8; a++) x[a] = smem[ntt_phys(a * 256 + tid)];
  radix8_inv(x, tab, 1, 0, q, two_q);
#pragma unroll
  for (int a = 0; a < 8; a++) x[a] = ntt_canon(x[a], q, two_q);
}

// =====================================================================================================================
// Relaxed-range transforms ("lz").  Same butterflies, same tables order, same outputs mod q — but the range corrections
// are scheduled per TRANSFORM instead of per butterfly, using the 4 bits of head-room a 28-bit modulus leaves in a u32
// (16 q < 2^32 for both moduli):
//
//  forward  x' = x + t, y' = x - t + 2q with t = W y - floor(y W'/2^32) q in [0, 2q) for ANY 32-bit y: the bound grows by
//           2q per stage.  Inputs < 2q -> < 16q after 7 stages; one min(v, v - 8q) on every value (inside pass C, after its
//           first stage) -> < 8q; the last 4 stages end < 16q.  9 range operations fewer per 11 butterflies.
//  inverse  Gentleman-Sande WITHOUT the per-stage halving: x' = x + y (corrected to < 8q where needed), y' = W (x - y + B)
//           with B the stage's input bound; the factor 1/N is folded into the LAST stage (its single twiddle is stored
//           pre-multiplied by 1/N, the sum branch is multiplied by 1/N): inverse table entry [0] = (1/N, (1/N)'),
//           entry [1] = psi^{-N/2}/N, entries >= 2 = psi^{-i} un-halved (ntt_tables.hpp: build_tables_lz).
// All arithmetic is exact modulo q, so the canonical outputs are bit-identical to the reference's transforms
// (ntt.rs:67-113, :212-258); tests/cpp/ntt_core_emul.cpp checks that, and with NTT_RANGE_CHECK that no u32 sum wraps.
#ifdef NTT_RANGE_CHECK
extern int ntt_range_violations;
#define NTT_RC_SUM(a, b) do { if ((uint64_t)(a) + (uint64_t)(b) > 0xffffffffull) ntt_range_violations++; } while (0)
#define NTT_RC_LT(a, b) do { if (!((uint64_t)(a) < (uint64_t)(b))) ntt_range_violations++; } while (0)
#else
#define NTT_RC_SUM(a, b)
#define NTT_RC_LT(a, b)
#endif

enum NttOut { NTT_OUT_LAZY16 = 0, NTT_OUT_LAZY4 = 1, NTT_OUT_CANON = 2 };

NTT_HD void bfly_fwd_lz(uint32_t& x, uint32_t& y, Twiddle tw, uint32_t q, uint32_t two_q) {
  const uint32_t qt = ntt_mulhi(y, tw.wp);
  const uint32_t t = tw.w * y - qt * q;                // [0, 2q) for any y
  NTT_RC_SUM(x, two_q);
  y = x + two_q - t;
  x = x + t;
}
NTT_HD uint32_t ntt_c8(uint32_t v, uint32_t eight_q) { return ntt_min(v, v - eight_q); }     // [0,16q) -> [0,8q)
// MID: apply the transform's single mid-way correction after the first of the three stages
template <bool MID, typename Tab>
NTT_HD void radix8_fwd_lz(uint32_t (&x)[8], Tab tab, int m0, int g0, uint32_t q, uint32_t two_q) {
  Twiddle t0 = tab(m0 + g0);
  Twiddle t1[2], t2[4];
  tab.load2(2 * m0 + 2 * g0, t1);
  tab.load4(4 * m0 + 4 * g0, t2);
#pragma unroll
  for (int a = 0; a < 4; a++) bfly_fwd_lz(x[a], x[a + 4], t0, q, two_q);
  if (MID) {
#pragma unroll
    for (int a = 0; a < 8; a++) x[a] = ntt_c8(x[a], 4 * two_q);
  }
#pragma unroll
  for (int h = 0; h < 2; h++) {
#pragma unroll
    for (int a = 0; a < 2; a++) bfly_fwd_lz(x[4 * h + a], x[4 * h + a + 2], t1[h], q, two_q);
  }
#pragma unroll
  for (int h = 0; h < 4; h++) bfly_fwd_lz(x[2 * h], x[2 * h + 1], t2[h], q, two_q);
}
// IN4Q: inputs are only known to be < 4q (to_ntt_no_reduce contract); otherwise they must be < 2q
template <bool IN4Q, typename Tab>
NTT_HD void fwd_pass_a_lz(int tid, uint32_t (&x)[8], uint32_t* smem, Tab tab, uint32_t q, uint32_t two_q) {
  if (IN4Q) {
#pragma unroll
    for (int a = 0; a < 8; a++) x[a] = ntt_min(x[a], x[a] - two_q);
  }
  radix8_fwd_lz<false>(x, tab, 1, 0, q, two_q);
#pragma unroll
  for (int a = 0; a < 8; a++) smem[ntt_phys(a * 256 + tid)] = x[a];
}
template <typename Tab>
NTT_HD void fwd_pass_b_lz(int tid, uint32_t (&x)[8], uint32_t* smem, Tab tab, uint32_t q, uint32_t two_q) {
  int hi = tid >> 5, lo = tid & 31;
#pragma unroll
  for (int a = 0; a < 8; a++) x[a] = smem[ntt_phys(hi * 256 + a * 32 + lo)];
  radix8_fwd_lz<false>(x, tab, 8, hi, q, two_q);
#pragma unroll
  for (int a = 0; a < 8; a++) smem[ntt_phys(hi * 256 + a * 32 + lo)] = x[a];
}
template <typename Tab>
NTT_HD void fwd_pass_c_lz(int tid, uint32_t (&x)[8], uint32_t* smem, Tab tab, uint32_t q, uint32_t two_q) {
  int H = tid >> 2, l2 = tid & 3;
#pragma unroll
  for (int a = 0; a < 8; a++) x[a] = smem[ntt_phys(H * 32 + a * 4 + l2)];
  radix8_fwd_lz<true>(x, tab, 64, H, q, two_q);                          // 7 stages done after its first stage: < 16q -> < 8q
#pragma unroll
  for (int a = 0; a < 8; a++) smem[ntt_phys(H * 32 + a * 4 + l2)] = x[a];
}
template <int OUT, typename Tab>
NTT_HD void fwd_pass_d_lz(int tid, uint32_t (&x)[8], const uint32_t* smem, Tab tab, uint32_t q, uint32_t two_q) {
  int base = ntt_phys(tid * 8);
#pragma unroll
  for (int k = 0; k < 8; k++) x[k] = smem[base + k];
  Twiddle t9[2], t10[4];
  tab.load2(512 + 2 * tid, t9);
  tab.load4(1024 + 4 * tid, t10);
#pragma unroll
  for (int h = 0; h < 2; h++) {
    bfly_fwd_lz(x[4 * h + 0], x[4 * h + 2], t9[h], q, two_q);
    bfly_fwd_lz(x[4 * h + 1], x[4 * h + 3], t9[h], q, two_q);
  }
#pragma unroll
  for (int h = 0; h < 4; h++) bfly_fwd_lz(x[2 * h], x[2 * h + 1], t10[h], q, two_q);
  if (OUT >= NTT_OUT_LAZY4) {
#pragma unroll
    for (int k = 0; k < 8; k++) { x[k] = ntt_min(x[k], x[k] - 4 * two_q); x[k] = ntt_min(x[k], x[k] - 2 * two_q); }   // < 4q
  }
  if (OUT == NTT_OUT_CANON) {
#pragma unroll
    for (int k = 0; k < 8; k++) x[k] = ntt_canon(x[k], q, two_q);
  }
}

// inverse butterfly without halving.  off = a multiple of q >= the bound of y (so x - y + off > 0); CORR: sums < 16q -> < 8q
template <bool CORR>
NTT_HD void bfly_inv_nh(uint32_t& x, uint32_t& y, Twiddle tw, uint32_t q, uint32_t off, uint32_t eight_q) {
  NTT_RC_SUM(x, y);
  NTT_RC_SUM(x, off);
  NTT_RC_LT(y, (uint64_t)off + 1);
  const uint32_t tt = x - y + off;
  uint32_t s = x + y;
  if (CORR) s = ntt_c8(s, eight_q);
  const uint32_t ht = ntt_mulhi(tt, tw.wp);
  x = s;
  y = tw.w * tt - ht * q;                              // [0, 2q)
}
NTT_HD uint32_t ntt_shoup(uint32_t v, Twiddle tw, uint32_t q) { return tw.w * v - ntt_mulhi(v, tw.wp) * q; }   // [0, 2q)
// three stages in reverse order, every value < 8q on entry and on exit
template <typename Tab>
NTT_HD void radix8_inv_nh(uint32_t (&x)[8], Tab tab, int m0, int g0, uint32_t q, uint32_t eight_q) {
  Twiddle t1[2], t2[4];
  tab.load4(4 * m0 + 4 * g0, t2);
  tab.load2(2 * m0 + 2 * g0, t1);
#pragma unroll
  for (int h = 0; h < 4; h++) bfly_inv_nh<true>(x[2 * h], x[2 * h + 1], t2[h], q, eight_q, eight_q);
#pragma unroll
  for (int h = 0; h < 2; h++) {
#pragma unroll
    for (int a = 0; a < 2; a++) bfly_inv_nh<true>(x[4 * h + a], x[4 * h + a + 2], t1[h], q, eight_q, eight_q);
  }
  Twiddle t0 = tab(m0 + g0);
#pragma unroll
  for (int a = 0; a < 4; a++) bfly_inv_nh<true>(x[a], x[a + 4], t0, q, eight_q, eight_q);
}
// pass D: stages 10 and 9 on inputs < 2q: bounds 2q -> 4q -> 8q, no correction needed
template <typename Tab>
NTT_HD void inv_pass_d_nh(int tid, uint32_t (&x)[8], uint32_t* smem, Tab tab, uint32_t q, uint32_t two_q) {
  Twiddle t9[2], t10[4];
  tab.load4(1024 + 4 * tid, t10);
  tab.load2(512 + 2 * tid, t9);
#pragma unroll
  for (int h = 0; h < 4; h++) bfly_inv_nh<false>(x[2 * h], x[2 * h + 1], t10[h], q, two_q, 0);
#pragma unroll
  for (int h = 0; h < 2; h++) {
    bfly_inv_nh<false>(x[4 * h + 0], x[4 * h + 2], t9[h], q, 2 * two_q, 0);
    bfly_inv_nh<false>(x[4 * h + 1], x[4 * h + 3], t9[h], q, 2 * two_q, 0);
  }
  int base = ntt_phys(tid * 8);
#pragma unroll
  for (int k = 0; k < 8; k++) smem[base + k] = x[k];
}
template <typename Tab>
NTT_HD void inv_pass_c_nh(int tid, uint32_t (&x)[8], uint32_t* smem, Tab tab, uint32_t q, uint32_t two_q) {
  int H = tid >> 2, l2 = tid & 3;
#pragma unroll
  for (int a = 0; a < 8; a++) x[a] = smem[ntt_phys(H * 32 + a * 4 + l2)];
  radix8_inv_nh(x, tab, 64, H, q, 4 * two_q);
#pragma unroll
  for (int a = 0; a < 8; a++) smem[ntt_phys(H * 32 + a * 4 + l2)] = x[a];
}
template <typename Tab>
NTT_HD void inv_pass_b_nh(int tid, uint32_t (&x)[8], uint32_t* smem, Tab tab, uint32_t q, uint32_t two_q) {
  int hi = tid >> 5, lo = tid & 31;
#pragma unroll
  for (int a = 0; a < 8; a++) x[a] = smem[ntt_phys(hi * 256 + a * 32 + lo)];
  radix8_inv_nh(x, tab, 8, hi, q, 4 * two_q);
#pragma unroll
  for (int a = 0; a < 8; a++) smem[ntt_phys(hi * 256 + a * 32 + lo)] = x[a];
}
// pass A: stages 2, 1 as above; stage 0 carries the factor 1/N (table entries 0 and 1) and is followed by the only
// canonicalisation of the transform (one min per value: both branches are Shoup products < 2q)
template <typename Tab>
NTT_HD void inv_pass_a_nh(int tid, uint32_t (&x)[8], const uint32_t* smem, Tab tab, uint32_t q, uint32_t two_q) {
#pragma unroll
  for (int a = 0; a < 8; a++) x[a] = smem[ntt_phys(a * 256 + tid)];
  const uint32_t eight_q = 4 * two_q;
  Twiddle t1[2], t2[4];
  tab.load4(4, t2);
  tab.load2(2, t1);
#pragma unroll
  for (int h = 0; h < 4; h++) bfly_inv_nh<true>(x[2 * h], x[2 * h + 1], t2[h], q, eight_q, eight_q);
#pragma unroll
  for (int h = 0; h < 2; h++) {
#pragma unroll
    for (int a = 0; a < 2; a++) bfly_inv_nh<true>(x[4 * h + a], x[4 * h + a + 2], t1[h], q, eight_q, eight_q);
  }
  const Twiddle ninv = tab(0), w1s = tab(1);
#pragma unroll
  for (int a = 0; a < 4; a++) {
    NTT_RC_SUM(x[a], x[a + 4]);
    const uint32_t s = x[a] + x[a + 4], tt = x[a] - x[a + 4] + eight_q;       // both < 16q
    const uint32_t u = ntt_shoup(s, ninv, q), v = ntt_shoup(tt, w1s, q);
    x[a] = ntt_min(u, u - q);
    x[a + 4] = ntt_min(v, v - q);
  }
}

#if defined(__CUDACC__)
// Group-cooperative transforms.  `gsync()` must synchronise the 256 threads of the group (and
// order their shared-memory accesses).  On entry to either function the group's smem buffer must
// not be in use; on return it may still be read by slower threads, so callers issue gsync()
// before the next transform reuses it (both functions start with that barrier themselves).
// `lo` serves table indices 1..63 (passes A, B: thread-uniform / warp-uniform -> constant bank),
// `hi` serves indices 64..2047 (passes C, D: per-thread -> shared memory or L1).
template <bool CANON = true, typename Sync, typename TabLo, typename TabHi>
__device__ __forceinline__ void ntt_forward_group(int tid, uint32_t (&x)[8], uint32_t* smem, TabLo lo, TabHi hi,
                                                  uint32_t q, Sync gsync) {
  const uint32_t two_q = 2 * q;
  gsync();
  fwd_pass_a(tid, x, smem, lo, q, two_q);
  gsync();
  fwd_pass_b(tid, x, smem, lo, q, two_q);
  gsync();
  fwd_pass_c(tid, x, smem, hi, q, two_q);
  gsync();
  fwd_pass_d<CANON>(tid, x, smem, hi, q, two_q);
}
// two independent transforms between the same barriers (instruction-level parallelism x2, half the
// barriers per transform)
template <bool CANON = true, typename Sync, typename TabLo, typename TabHi>
__device__ __forceinline__ void ntt_forward_group2(int tid, uint32_t (&x0)[8], uint32_t (&x1)[8], uint32_t* smem0,
                                                   uint32_t* smem1, TabLo lo, TabHi hi, uint32_t q, Sync gsync) {
  const uint32_t two_q = 2 * q;
  gsync();
  fwd_pass_a(tid, x0, smem0, lo, q, two_q);
  fwd_pass_a(tid, x1, smem1, lo, q, two_q);
  gsync();
  fwd_pass_b(tid, x0, smem0, lo, q, two_q);
  fwd_pass_b(tid, x1, smem1, lo, q, two_q);
  gsync();
  fwd_pass_c(tid, x0, smem0, hi, q, two_q);
  fwd_pass_c(tid, x1, smem1, hi, q, two_q);
  gsync();
  fwd_pass_d<CANON>(tid, x0, smem0, hi, q, two_q);
  fwd_pass_d<CANON>(tid, x1, smem1, hi, q, two_q);
}
template <typename Sync, typename TabLo, typename TabHi>
__device__ __forceinline__ void ntt_inverse_group(int tid, uint32_t (&x)[8], uint32_t* smem, TabLo lo, TabHi hi,
                                                  uint32_t q, Sync gsync) {
  const uint32_t two_q = 2 * q;
  gsync();
  inv_pass_d(tid, x, smem, hi, q, two_q);
  gsync();
  inv_pass_c(tid, x, smem, hi, q, two_q);
  gsync();
  inv_pass_b(tid, x, smem, lo, q, two_q);
  gsync();
  inv_pass_a(tid, x, smem, lo, q, two_q);
}
template <typename Sync, typename TabLo, typename TabHi>
__device__ __forceinline__ void ntt_inverse_group2(int tid, uint32_t (&x0)[8], uint32_t (&x1)[8], uint32_t* smem0,
                                                   uint32_t* smem1, TabLo lo, TabHi hi, uint32_t q, Sync gsync) {
  const uint32_t two_q = 2 * q;
  gsync();
  inv_pass_d(tid, x0, smem0, hi, q, two_q);
  inv_pass_d(tid, x1, smem1, hi, q, two_q);
  gsync();
  inv_pass_c(tid, x0, smem0, hi, q, two_q);
  inv_pass_c(tid, x1, smem1, hi, q, two_q);
  gsync();
  inv_pass_b(tid, x0, smem0, lo, q, two_q);
  inv_pass_b(tid, x1, smem1, lo, q, two_q);
  gsync();
  inv_pass_a(tid, x0, smem0, lo, q, two_q);
  inv_pass_a(tid, x1, smem1, lo, q, two_q);
}
// relaxed-range versions (see above).  Forward: inputs < 2q (IN4Q: < 4q), outputs per OUT; inverse: inputs < 2q,
// canonical outputs, `lo`/`hi` must serve the un-halved inverse tables of build_tables_lz.
template <int OUT, bool IN4Q = false, typename Sync, typename TabLo, typename TabHi>
__device__ __forceinline__ void ntt_forward_group_lz(int tid, uint32_t (&x)[8], uint32_t* smem, TabLo lo, TabHi hi,
                                                     uint32_t q, Sync gsync) {
  const uint32_t two_q = 2 * q;
  gsync();
  fwd_pass_a_lz<IN4Q>(tid, x, smem, lo, q, two_q);
  gsync();
  fwd_pass_b_lz(tid, x, smem, lo, q, two_q);
  gsync();
  fwd_pass_c_lz(tid, x, smem, hi, q, two_q);
  gsync();
  fwd_pass_d_lz<OUT>(tid, x, smem, hi, q, two_q);
}
template <int OUT, bool IN4Q = false, typename Sync, typename TabLo, typename TabHi>
__device__ __forceinline__ void ntt_forward_group2_lz(int tid, uint32_t (&x0)[8], uint32_t (&x1)[8], uint32_t* smem0,
                                                      uint32_t* smem1, TabLo lo, TabHi hi, uint32_t q, Sync gsync) {
  const uint32_t two_q = 2 * q;
  gsync();
  fwd_pass_a_lz<IN4Q>(tid, x0, smem0, lo, q, two_q);
  fwd_pass_a_lz<IN4Q>(tid, x1, smem1, lo, q, two_q);
  gsync();
  fwd_pass_b_lz(tid, x0, smem0, lo, q, two_q);
  fwd_pass_b_lz(tid, x1, smem1, lo, q, two_q);
  gsync();
  fwd_pass_c_lz(tid, x0, smem0, hi, q, two_q);
  fwd_pass_c_lz(tid, x1, smem1, hi, q, two_q);
  gsync();
  fwd_pass_d_lz<OUT>(tid, x0, smem0, hi, q, two_q);
  fwd_pass_d_lz<OUT>(tid, x1, smem1, hi, q, two_q);
}
template <typename Sync, typename TabLo, typename TabHi>
__device__ __forceinline__ void ntt_inverse_group_nh(int tid, uint32_t (&x)[8], uint32_t* smem, TabLo lo, TabHi hi,
                                                     uint32_t q, Sync gsync) {
  const uint32_t two_q = 2 * q;
  gsync();
  inv_pass_d_nh(tid, x, smem, hi, q, two_q);
  gsync();
  inv_pass_c_nh(tid, x, smem, hi, q, two_q);
  gsync();
  inv_pass_b_nh(tid, x, smem, lo, q, two_q);
  gsync();
  inv_pass_a_nh(tid, x, smem, lo, q, two_q);
}
template <typename Sync, typename TabLo, typename TabHi>
__device__ __forceinline__ void ntt_inverse_group2_nh(int tid, uint32_t (&x0)[8], uint32_t (&x1)[8], uint32_t* smem0,
                                                      uint32_t* smem1, TabLo lo, TabHi hi, uint32_t q, Sync gsync) {
  const uint32_t two_q = 2 * q;
  gsync();
  inv_pass_d_nh(tid, x0, smem0, hi, q, two_q);
  inv_pass_d_nh(tid, x1, smem1, hi, q, two_q);
  gsync();
  inv_pass_c_nh(tid, x0, smem0, hi, q, two_q);
  inv_pass_c_nh(tid, x1, smem1, hi, q, two_q);
  gsync();
  inv_pass_b_nh(tid, x0, smem0, lo, q, two_q);
  inv_pass_b_nh(tid, x1, smem1, lo, q, two_q);
  gsync();
  inv_pass_a_nh(tid, x0, smem0, lo, q, two_q);
  inv_pass_a_nh(tid, x1, smem1, lo, q, two_q);
}
#endif

}  // namespace b200pir
