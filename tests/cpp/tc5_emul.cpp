// CPU emulation of the wgmma first dimension's data path (sdk_b200/csrc/tc5_layout.cuh + the structure of
// tc5_kernels.cu): the operand images are built by running the per-thread functions for every thread, the MMA is replaced
// by the DEFINITION of the canonical K-major no-swizzle shared-memory layout (byte (row, k) of an operand tile at
// (row/8)*SBO + (k/16)*LBO + (row%8)*16 + k%16; D[M][N] += A[M][k] * B[N][k]) and of the m64nNk32 s32 accumulator fragment
// (thread (warp w, lane) of warpgroup wg holds D[64 wg + 16 w + lane/4 + 8 h][8 i + 2 (lane%4) + c] in register 4 i + 2 h + c),
// and the epilogue runs lane by lane with the three shuffle rounds of its reduce-scatter emulated.  Result compared with sum_j a*b mod q in 128-bit
// arithmetic.  This checks every index / limb / lane computation that is ours; what it cannot check is that the hardware
// reads the descriptors the way the layout definition says.
#include "../../sdk_b200/csrc/tc5_layout.cuh"
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <random>
#include <vector>

using namespace b200pir;
typedef unsigned __int128 u128;

int main() {
  const uint32_t Q[2] = {268369921u, 249561089u};
  std::mt19937_64 rng(2026);
  int bad = 0;
  for (int trial = 0; trial < 3; trial++) {
    // trial 0: dim0 64, 40 rows (ragged last row tile), 5 queries, random; 1: dim0 512, 64 rows, 16 queries, all q-1;
    // 2: dim0 96 (3 k-steps), 32 rows, 11 queries
    const int dim0 = trial == 0 ? 64 : (trial == 1 ? 512 : 96), rows = trial == 0 ? 40 : (trial == 1 ? 64 : 32);
    const int nq = trial == 0 ? 5 : (trial == 1 ? 16 : 11);
    const Tc5Geom T = make_tc5_geom(dim0, rows);
    const int half = dim0 / 2;
    for (int n = 0; n < 2; n++) {
      const uint32_t q = Q[n];
      const uint64_t cr1 = (uint64_t)(((u128)1 << 64) / q);
      // operands for one (slice, z): a[ii][j], b[query][r][j]
      std::vector<uint32_t> a((size_t)rows * dim0), b((size_t)nq * 2 * dim0);
      for (auto& x : a) x = trial == 1 ? q - 1 : (uint32_t)(rng() % q);
      for (auto& x : b) x = trial == 1 ? q - 1 : (uint32_t)(rng() % q);
      // ---- database image: CTA (mt, ks), 256 threads each (k_db_import_tc5); the other modulus' tile is not needed here
      std::vector<uint8_t> dbt((size_t)T.mt * T.ks * TC5_TILE, 0xEE);
      for (int mt = 0; mt < T.mt; mt++)
        for (int ks = 0; ks < T.ks; ks++)
          for (int tid = 0; tid < 256; tid++) {
            const Tc5DbThread t = tc5_db_thread(tid, mt, ks);
            uint32_t res[4];
            for (int p = 0; p < 2; p++) {
              const int jp = t.jp0 + p;
              const bool in = t.ii < rows && jp < half;
              res[2 * p] = in ? a[(size_t)t.ii * dim0 + 2 * jp] : 0;
              res[2 * p + 1] = in ? a[(size_t)t.ii * dim0 + 2 * jp + 1] : 0;
            }
            tc5_db_store(dbt.data() + ((size_t)mt * T.ks + ks) * TC5_TILE, t, res);
          }
      for (uint8_t x : dbt) if (x == 0xEE) { bad++; break; }        // every byte of every tile must have been written
      // ---- query image: CTA (ks): 1024 cells (k_query_to_tc5), tiles start zeroed
      std::vector<uint8_t> qt((size_t)T.ks * TC5_TILE, 0);
      for (int ks = 0; ks < T.ks; ks++)
        for (int cell = 0; cell < 16 * 32 * 2; cell++) {
          const Tc5QueryCell qc = tc5_query_cell(cell);
          if (qc.zp != 0) continue;                                  // the emulation follows one z
          const int j = ks * 32 + qc.k;
          if (qc.q < nq && j < dim0)
            for (int r = 0; r < 2; r++) tc5_query_store(qt.data() + (size_t)ks * TC5_TILE, qc.q, r, qc.k, b[((size_t)qc.q * 2 + r) * dim0 + j]);
        }
      // ---- per row tile: MMA by the layout definition, then the epilogue
      std::vector<int> covered((size_t)rows * 32, 0);
      for (int mt = 0; mt < T.mt; mt++) {
        std::vector<int32_t> D((size_t)TC5_M * TC5_N, 0);
        for (int ks = 0; ks < T.ks; ks++) {
          const uint8_t* A = dbt.data() + ((size_t)mt * T.ks + ks) * TC5_TILE;
          const uint8_t* B = qt.data() + (size_t)ks * TC5_TILE;
          for (int M = 0; M < TC5_M; M++)
            for (int N = 0; N < TC5_N; N++) {
              int32_t s = 0;
              for (int k = 0; k < TC5_K; k++) {
                const int ao = (M / 8) * TC5_SBO + (k / 16) * TC5_LBO + (M % 8) * 16 + k % 16;
                const int bo = (N / 8) * TC5_SBO + (k / 16) * TC5_LBO + (N % 8) * 16 + k % 16;
                s += (int32_t)A[ao] * (int32_t)B[bo];
              }
              D[(size_t)M * TC5_N + N] += s;
            }
        }
        for (int wg = 0; wg < 2; wg++)
          for (int w = 0; w < 4; w++) {
            // step 1: per lane, the 32 weighted partials of its accumulator fragment; then the three rounds of the
            // reduce-scatter (every lane computes send/keep, then reads its partner's send)
            uint64_t p32[32][32], s16[32][16], k16[32][16], s8[32][8], k8[32][8], s4[32][4], k4[32][4];
            Tc5Weights W[32];
            for (int lane = 0; lane < 32; lane++) {
              uint32_t acc[64];
              for (int i = 0; i < 16; i++)
                for (int h = 0; h < 2; h++)
                  for (int c = 0; c < 2; c++)
                    acc[4 * i + 2 * h + c] = (uint32_t)D[(size_t)(64 * wg + 16 * w + lane / 4 + 8 * h) * TC5_N + 8 * i + 2 * (lane % 4) + c];
              W[lane] = tc5_lane_weights(lane, q);
              for (int i = 0; i < 16; i++)
                for (int h = 0; h < 2; h++) {
                  uint64_t& p = p32[lane][2 * i + h];
                  p = tc5_lane_partial(acc[4 * i + 2 * h], acc[4 * i + 2 * h + 1], W[lane].w, W[lane].wp);
                  if (p >> 52) { if (bad < 5) printf("partial sum bound exceeded\n"); bad++; }
                }
              tc5_rs_split<32>((lane >> tc5_rs_lane_bit(0)) & 1, p32[lane], s16[lane], k16[lane]);
            }
            for (int lane = 0; lane < 32; lane++) {
              for (int r = 0; r < 16; r++) k16[lane][r] += s16[lane ^ (1 << tc5_rs_lane_bit(0))][r];
              tc5_rs_split<16>((lane >> tc5_rs_lane_bit(1)) & 1, k16[lane], s8[lane], k8[lane]);
            }
            for (int lane = 0; lane < 32; lane++) {
              uint64_t k[8];
              for (int r = 0; r < 8; r++) k[r] = k8[lane][r] + s8[lane ^ (1 << tc5_rs_lane_bit(1))][r];
              tc5_rs_split<8>((lane >> tc5_rs_lane_bit(2)) & 1, k, s4[lane], k4[lane]);
            }
            for (int lane = 0; lane < 32; lane++)
              for (int f = 0; f < 4; f++) {
                const int qi = tc5_frag_query(lane, f), ii = mt * 32 + tc5_frag_row(wg, w, lane, f & 1), r = tc5_frag_ctrow(lane);
                if (qi >= nq || ii >= rows) continue;
                const uint64_t tot = k4[lane][f] + s4[lane ^ (1 << tc5_rs_lane_bit(2))][f];
                if (tot >> 55) { if (bad < 5) printf("column sum bound exceeded\n"); bad++; }
                const uint32_t got = tc5_barrett57(tot, W[lane].mu, q);
                u128 ref = 0;
                for (int j = 0; j < dim0; j++) ref += (u128)a[(size_t)ii * dim0 + j] * b[((size_t)qi * 2 + r) * dim0 + j];
                if (got != (uint32_t)(ref % q)) { if (bad < 5) printf("mismatch trial %d n %d row %d query %d r %d\n", trial, n, ii, qi, r); bad++; }
                covered[(size_t)ii * 32 + qi * 2 + r]++;
              }
          }
      }
      for (int ii = 0; ii < rows; ii++)                            // every (row, query, ct row) output stored exactly once
        for (int col = 0; col < 2 * nq; col++)
          if (covered[(size_t)ii * 32 + col] != 1) { if (bad < 5) printf("output row %d column %d stored %d times\n", ii, col, covered[(size_t)ii * 32 + col]); bad++; }
    }
  }
  // tc5_barrett57 against % on random and extreme inputs below 2^57
  for (int n = 0; n < 2; n++) {
    const uint32_t q = Q[n], mu = tc5_lane_weights(0, q).mu;
    for (int i = 0; i < 2000000; i++) {
      uint64_t x = rng() >> 7;
      if (i < 64) x = ((uint64_t)1 << 57) - 1 - i;
      else if (i < 128) x = (uint64_t)q * (i - 64) + (i & 1 ? q - 1 : 0);
      else if (i < 4096) x = (uint64_t)q * (rng() >> 36) - (i & 3);
      x &= ((uint64_t)1 << 57) - 1;
      if (tc5_barrett57(x, mu, q) != (uint32_t)(x % q)) { if (bad < 5) printf("barrett57 mismatch at %llu mod %u\n", (unsigned long long)x, q); bad++; }
    }
  }
  printf(bad ? "tc5 emulation: %d mismatches\n" : "tc5 emulation ok%.0d\n", bad);
  return bad ? 1 : 0;
}
