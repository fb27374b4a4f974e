// Index maps of DoublePIR's database pass on the tensor cores (dpir_tc.cu), as __host__ __device__ functions free of CUDA
// types so that the operand images and the epilogue can be emulated thread by thread on the CPU (tests/cpp/dpir_tc_emul.cpp).
//
// The pass computes  out_v[r] = sum_k sum_{t<3} ((a[r][k] >> 10 t) & 1023) * b_v[3 k + t]  (mod 2^32, kernels.rs:14-113) as one
// u8 x u8 GEMM with the limb indices inside M and N (DESIGN §4.1, §4.5):
//   digit d = d0 + 2^8 d1 (d0 < 256, d1 < 4),  query word b = sum_j b_j 2^{8 j} (four bytes),  d b = sum_{i+j<=3} d_i b_j 2^{8(i+j)}
//   M = 2 row + i,  N = 4 vector + j,  K = (chunk c, digit plane t, word q): digit t of packed word 32 c + q.
// A k-step is 32 words of one digit plane; a chunk of 32 packed words is three k-steps (t = 0, 1, 2).
#pragma once
#include "tc5_layout.cuh"      // TC5_HD, tc5_tile_off (canonical K-major no-swizzle layout), tc5_smem_desc

namespace b200pir {

constexpr int DTC_ROWS = 64;             // database rows a CTA: two 32-row halves (M = 2 row + i: 64 M rows each)
constexpr int DTC_VECS = 64;             // vectors a pass (P): two 32-vector halves (N = 4 vector + j: 128 N rows each)
constexpr int DTC_KW = 32;               // packed words a chunk
constexpr int DTC_A_TILE = 64 * 32;      // one plane of one row half: 64 M rows x 32 bytes
constexpr int DTC_B_TILE = 128 * 32;     // one plane of one vector half: 128 N rows x 32 bytes
constexpr int DTC_IMG_CHUNK = 3 * 4 * 32;   // bytes of one vector's image per chunk: 3 planes x 4 bytes x 32 words

TC5_HD size_t dtc_chunks(size_t cols) { return (cols + DTC_KW - 1) / DTC_KW; }
// bytes of one vector's query image (every chunk, zero past `cols`)
TC5_HD size_t dtc_img_bytes(size_t cols) { return dtc_chunks(cols) * DTC_IMG_CHUNK; }

// the four B tiles and two A tiles of one k-step: plane t, vector half vh / row half rh (offsets in the stage's B region and in
// the A buffer)
TC5_HD int dtc_b_tile(int t, int vh) { return (t * 2 + vh) * DTC_B_TILE; }
TC5_HD int dtc_a_tile(int t, int rh) { return (t * 2 + rh) * DTC_A_TILE; }

// ---- query operand.  A vector's image holds, for each (chunk c, plane t, K half kh, byte j), the 16 bytes
// byte j of b[3 (32 c + 16 kh + e) + t], e < 16: exactly the four 16-byte core-matrix rows n = 4 v + j of the vector in a B tile.
TC5_HD size_t dtc_img_off(size_t c, int t, int kh, int j) { return ((c * 3 + t) * 2 + kh) * 64 + (size_t)j * 16; }
// the builder's thread (c, t, kh) reads 16 words of b (big-endian when `be`: bytes taken from the other end) and returns the four
// rows j as 4 x 4 words; words past `cols` are zero, so the last partial chunk multiplies into nothing
TC5_HD void dtc_img_rows(const uint32_t* b, size_t cols, bool be, size_t c, int t, int kh, uint32_t (&rows)[4][4]) {
  for (int j = 0; j < 4; j++)
    for (int q = 0; q < 4; q++) rows[j][q] = 0;
  for (int e = 0; e < 16; e++) {
    const size_t k = c * DTC_KW + 16 * kh + e;
    if (k >= cols) break;
    const uint32_t v = b[3 * k + t];
    for (int j = 0; j < 4; j++) {
      const uint32_t byte = (v >> (8 * (be ? 3 - j : j))) & 255u;
      rows[j][e >> 2] |= byte << (8 * (e & 3));
    }
  }
}
// where vector vl (< DTC_VECS) of a pass puts its 64 bytes of (plane t, K half kh) in the B region of a stage: tiles [t][vh],
// row n = 4 (vl % 32) + j of tile (t, vl / 32); the four rows j are consecutive 16-byte rows of one core-matrix group
TC5_HD int dtc_b_smem_off(int vl, int t, int kh) { return dtc_b_tile(t, vl >> 5) + tc5_tile_off(4 * (vl & 31), 16 * kh); }

// ---- database operand.  Raw staging: the chunk's 32 words of each of the CTA's 64 rows, [row][word]: copy idx (< 2048) is
// row idx / 32, word idx % 32.  Words past `cols` and rows past the task's are zero-filled, never read.
TC5_HD bool dtc_raw_ok(int r, uint32_t word, uint32_t rows, uint32_t cols) { return r < (int)rows && word < cols; }
// Unpacking thread tid: row tid / 8, words 4 (tid % 8) .. + 3.
struct DtcUnpack { int row, kq; };
TC5_HD DtcUnpack dtc_unpack_thread(int tid) { return DtcUnpack{tid >> 3, tid & 7}; }
// limb i of digit plane t of four consecutive words, as four bytes (lowest address = lowest word)
TC5_HD uint32_t dtc_limb4(const uint32_t (&w)[4], int t, int i) {
  uint32_t x = 0;
  for (int e = 0; e < 4; e++) {
    const uint32_t d = (w[e] >> (10 * t)) & 1023u;
    x |= (i ? d >> 8 : d & 255u) << (8 * e);
  }
  return x;
}
// byte offset in the A region of (row r < 64, plane t, limb i, word 4 kq): tiles [t][rh], M row 2 (r % 32) + i
TC5_HD int dtc_a_smem_off(int r, int t, int i, int kq) { return dtc_a_tile(t, r >> 5) + tc5_tile_off(2 * (r & 31) + i, 4 * kq); }

// ---- epilogue.  Four consumer warpgroups; warpgroup g takes row half rh = g / 2 and vector half vh = g % 2 with one
// wgmma.m64n128k32 per k-step, whose s32 accumulator fragment gives thread (warp w of the warpgroup, lane)
//     acc[4 ii + 2 h + c] = D[16 w + lane/4 + 8 h][8 ii + 2 (lane%4) + c]          (ii < 16, h < 2, c < 2)
// i.e. row (M/2) 8 w + lane/8 + 4 h of the half, limb i = (lane/4) % 2, vector (N/4) 2 ii + (lane/2) % 2, bytes j = 2 (lane%2) + c.
// out = sum_{i,j} D_{i,j} 2^{8(i+j)} mod 2^32 (the i = 1, j = 3 term vanishes): each lane weights its two accumulators, the
// lanes lane ^ 1 (the other byte pair) and lane ^ 4 (the other limb) add theirs, and one of the four stores.  An accumulator
// may wrap; D_{i,j} only matters modulo 2^{32 - 8(i+j)}, which the wrap leaves intact.
TC5_HD int dtc_frag_row(int w, int lane, int h) { return 8 * w + (lane >> 3) + 4 * h; }
TC5_HD int dtc_frag_vec(int lane, int ii) { return 2 * ii + ((lane >> 1) & 1); }
TC5_HD int dtc_frag_limb(int lane) { return (lane >> 2) & 1; }
TC5_HD int dtc_frag_byte(int lane, int c) { return 2 * (lane & 1) + c; }
TC5_HD uint32_t dtc_lane_partial(uint32_t a0, uint32_t a1, int lane) {
  const int s = 8 * (dtc_frag_limb(lane) + dtc_frag_byte(lane, 0));
  return (a0 << s) + (s + 8 < 32 ? a1 << (s + 8) : 0u);
}
// which of the four lanes holding the sum of (ii, h) stores it
TC5_HD bool dtc_frag_stores(int lane, int ii, int h) { return ((2 * ii + h) & 3) == ((lane & 1) | (((lane >> 2) & 1) << 1)); }

}  // namespace b200pir
