// Index / limb arithmetic of the wgmma first dimension (tc5_kernels.cu), as __host__ __device__ functions so that the
// operand images and the epilogue can be emulated thread by thread on the CPU (tests/cpp/tc5_emul.cpp) against the
// canonical K-major, no-swizzle shared-memory layout of wgmma operands (PTX ISA, "Shared Memory Matrix Layout").
#pragma once
#include <stdint.h>
#include <stddef.h>

#if defined(__CUDACC__)
#define TC5_HD __host__ __device__ __forceinline__
#else
#define TC5_HD inline
#endif

namespace b200pir {

struct Tc5Geom { int dim0, rows, mt /* ceil(rows/32) */, ks /* ceil(dim0/32) */; };
inline Tc5Geom make_tc5_geom(int dim0, int rows) { return Tc5Geom{dim0, rows, (rows + 31) / 32, (dim0 + 31) / 32}; }

constexpr int TC5_M = 128, TC5_N = 128, TC5_K = 32;
constexpr int TC5_TILE = TC5_M * TC5_K;                 // 4096 bytes, A and B tiles alike
constexpr int TC5_LBO = 128;                            // bytes between the two 16-byte K halves of a core-matrix row group
constexpr int TC5_SBO = 256;                            // bytes between consecutive 8-row groups

// byte (midx, k) of a 128 x 32 tile: 8-row x 16-byte core matrices
TC5_HD int tc5_tile_off(int midx, int k) { return (midx >> 3) * TC5_SBO + (k >> 4) * TC5_LBO + (midx & 7) * 16 + (k & 15); }
// GEMM indices: M = 4 * row_local + l (database row within the 32-row tile, limb), N = 4 * col + m (col = 2 query + ct row)
TC5_HD int tc5_m_index(int row_local, int l) { return 4 * row_local + l; }
TC5_HD int tc5_n_index(int col, int m) { return 4 * col + m; }
TC5_HD size_t tc5_db_tile(const Tc5Geom& T, int slice, int n, int z, int mt, int ks) {
  return ((((size_t)slice * 2 + n) * 2048 + z) * T.mt + mt) * T.ks + ks;
}
TC5_HD size_t tc5_q_tile(const Tc5Geom& T, int n, int z, int ks) { return ((size_t)n * 2048 + z) * T.ks + ks; }
// limb l (7 bits) of four residues as four bytes, lowest address first
TC5_HD uint32_t tc5_limb4(const uint32_t (&r)[4], int l) {
  const int sh = 7 * l;
  return ((r[0] >> sh) & 127u) | (((r[1] >> sh) & 127u) << 8) | (((r[2] >> sh) & 127u) << 16) | (((r[3] >> sh) & 127u) << 24);
}

// ---- shared-memory matrix descriptor of wgmma (PTX ISA, "Matrix Descriptor Format"; checked field by field by
// tests/cpp/tc5_desc_check.cpp): start address, LBO, SBO in 16-byte units, base offset 0, layout type 0 (no swizzle)
TC5_HD uint64_t tc5_smem_desc(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr >> 4) & 0x3FFF);           // [0,14)   start address
  d |= (uint64_t)((TC5_LBO >> 4) & 0x3FFF) << 16;       // [16,30)  leading-dimension byte offset (K halves)
  d |= (uint64_t)((TC5_SBO >> 4) & 0x3FFF) << 32;       // [32,46)  stride byte offset (8-row groups)
  return d;                                             // [49,52) base offset 0, [62,64) no swizzle
}

// ---- database image: thread tid of the CTA of row tile mt / k-step ks handles one row and four consecutive j
struct Tc5DbThread { int row_local, kq, ii, jp0; };
TC5_HD Tc5DbThread tc5_db_thread(int tid, int mt, int ks) {
  Tc5DbThread t;
  t.row_local = tid >> 3;
  t.kq = tid & 7;
  t.ii = mt * 32 + t.row_local;
  t.jp0 = (ks * 32 + 4 * t.kq) >> 1;                    // the thread reads cells jp0 and jp0 + 1 (two j each)
  return t;
}
// res[i] = residue (one modulus) of j = ks*32 + 4 kq + i; writes the thread's four 4-byte words of one tile
TC5_HD void tc5_db_store(uint8_t* tile, const Tc5DbThread& t, const uint32_t (&res)[4]) {
  for (int l = 0; l < 4; l++) {
    const uint32_t v = tc5_limb4(res, l);
    uint8_t* p = tile + tc5_tile_off(tc5_m_index(t.row_local, l), 4 * t.kq);
    p[0] = (uint8_t)v; p[1] = (uint8_t)(v >> 8); p[2] = (uint8_t)(v >> 16); p[3] = (uint8_t)(v >> 24);
  }
}

// ---- query image: cell = (query, k, z parity) of the CTA of k-step ks
struct Tc5QueryCell { int zp, k, q; };
TC5_HD Tc5QueryCell tc5_query_cell(int cell) { return Tc5QueryCell{cell & 1, (cell >> 1) & 31, cell >> 6}; }
// value = residue (one modulus) of query q, ciphertext row r at (j = ks*32 + k): its four limb bytes
TC5_HD void tc5_query_store(uint8_t* tile, int q, int r, int k, uint32_t value) {
  for (int m = 0; m < 4; m++) tile[tc5_tile_off(tc5_n_index(2 * q + r, m), k)] = (uint8_t)((value >> (7 * m)) & 127u);
}

// ---- epilogue.  Two consumer warpgroups; warpgroup wg computes M rows [64 wg, 64 wg + 64) of the 128 x 128 tile with
// wgmma.m64n128k32, whose s32 accumulator fragment gives thread (warp w of the warpgroup, lane) the 64 values
//     acc[4 i + 2 h + c] = D[64 wg + 16 w + lane/4 + 8 h][8 i + 2 (lane%4) + c]          (i < 16, h < 2, c < 2)
// i.e. database row (M/4) 16 wg + 4 w + lane/16 + 2 h, limb l = (lane/4) % 4, GEMM column (N/4) 2 i + (lane/2) % 2 = query i,
// ciphertext row (lane/2) % 2, and the two query limbs m = 2 (lane%2) + c.  The residue is  sum_{l,m} D_{l,m} 2^{7(l+m)} mod q:
//   1. per (i, h): s = D_{l,m0} + D_{l,m0+1} 2^7 (< 2^32), split at bit 23 and weighted with w = 2^{7(l+m0)} mod q,
//      w' = 2^{7(l+m0)+23} mod q:  P = (s mod 2^23) w + (s >> 23) w'  < 2^52            (two wide multiply-adds)
//   2. reduce-scatter of the 32 partials over the eight lanes of a (row, column) that hold its four l and two m0
//      (lane bits 0, 2, 3), halving the top bit of the partial index each round: each lane keeps four sums (< 2^55)
//   3. one Barrett reduction per stored word, with 32-bit operations (tc5_barrett57).
TC5_HD int tc5_frag_row(int wg, int w, int lane, int h) { return 16 * wg + 4 * w + (lane >> 4) + 2 * h; }   // row_local
TC5_HD int tc5_frag_limb(int lane) { return (lane >> 2) & 3; }
TC5_HD int tc5_frag_ctrow(int lane) { return (lane >> 1) & 1; }
// the query of the f-th kept sum (f < 4) after the reduce-scatter; its row half is h = f & 1
TC5_HD int tc5_frag_query(int lane, int f) { return ((lane & 1) << 3) | (((lane >> 2) & 1) << 2) | (((lane >> 3) & 1) << 1) | (f >> 1); }
// the lane bit each reduce-scatter round exchanges over (partner = lane ^ (1 << bit))
TC5_HD int tc5_rs_lane_bit(int round) { return round == 0 ? 0 : (round == 1 ? 2 : 3); }
struct Tc5Weights { uint32_t w, wp, mu; };
TC5_HD Tc5Weights tc5_lane_weights(int lane, uint32_t q) {
  const int e = 7 * (tc5_frag_limb(lane) + 2 * (lane & 1));
  Tc5Weights W;
  W.w = (uint32_t)((1ull << e) % q);
  W.wp = (uint32_t)((1ull << (e + 23)) % q);
  W.mu = (uint32_t)((1ull << 58) / q);                                             // q > 2^27, so mu < 2^31
  return W;
}
// x mod q for x < 2^57 and 2^27 < q < 2^28: quotient estimate floor((x >> 26) mu / 2^32) is the true quotient or one less
// (x/2^58 + 2^26/q < 1), so the remainder estimate lies in [0, 2q) and its low 32 bits suffice.
TC5_HD uint32_t tc5_barrett57(uint64_t x, uint32_t mu, uint32_t q) {
  const uint32_t a = (uint32_t)(x >> 26);
#if defined(__CUDA_ARCH__)
  const uint32_t qh = __umulhi(a, mu);
#else
  const uint32_t qh = (uint32_t)(((uint64_t)a * mu) >> 32);
#endif
  const uint32_t r = (uint32_t)x - qh * q;
  const uint32_t r2 = r - q;
  return r < r2 ? r : r2;
}
// step 1 for one (i, h): v0, v1 = the accumulators of query limbs m0, m0 + 1
TC5_HD uint64_t tc5_lane_partial(uint32_t v0, uint32_t v1, uint32_t w, uint32_t wp) {
  const uint32_t s = v0 + (v1 << 7);                                               // < 2^32 (D < 2^24)
  return (uint64_t)(s & 0x7FFFFFu) * w + (uint64_t)(s >> 23) * wp;
}
// step 2, one round over NIN partials: a lane whose exchange bit is `up` keeps the upper half of the index range and sends the
// lower half, the others the opposite; the partner adds what it receives to what it keeps, entry by entry
template <int NIN>
TC5_HD void tc5_rs_split(bool up, const uint64_t (&in)[NIN], uint64_t (&send)[NIN / 2], uint64_t (&keep)[NIN / 2]) {
  for (int r = 0; r < NIN / 2; r++) { send[r] = up ? in[r] : in[r + NIN / 2]; keep[r] = up ? in[r + NIN / 2] : in[r]; }
}

}  // namespace b200pir
