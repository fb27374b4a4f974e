// CPU emulation of DoublePIR's tensor-core pass (sdk_b200/csrc/dpir_tc.cu) through the index maps of dpir_tc_layout.cuh:
// the query images are built thread by thread by the builder's function into buffers pre-filled with garbage, each CTA's chunks
// are staged (raw words by the copy rule, images by the placement map) and unpacked by its 512 threads, the wgmma is replaced
// by the definitions of the canonical no-swizzle K-major layout (decoded from the descriptor the kernel builds) and of the
// m64nNk32 s32 accumulator fragment, and the epilogue runs lane by lane with its two shuffles.  Results are compared with the
// 64-bit definition of matrix_mul_vec_packed (kernels.rs:14-113).  Prints "dpir tc emulation ok".
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>
#include "../../sdk_b200/csrc/dpir_tc_layout.cuh"

using namespace b200pir;

static uint64_t rng_state = 0x9E3779B97F4A7C15ull;
static uint32_t rnd() {
  rng_state ^= rng_state << 13; rng_state ^= rng_state >> 7; rng_state ^= rng_state << 17;
  return (uint32_t)(rng_state >> 16);
}
static uint32_t bswap(uint32_t v) { return (v >> 24) | ((v >> 8) & 0xFF00u) | ((v << 8) & 0xFF0000u) | (v << 24); }

// byte (row, k) of a K-major no-swizzle operand at `base`, from the descriptor's LBO / SBO fields (PTX ISA, "Shared Memory
// Matrix Layout": 8-row x 16-byte core matrices; LBO = between K-adjacent ones, SBO = between 8-row groups)
static uint8_t layout_byte(const uint8_t* smem, uint32_t base, int row, int k) {
  const uint64_t d = tc5_smem_desc(base);
  const uint32_t start = (uint32_t)(d & 0x3FFF) << 4, lbo = (uint32_t)((d >> 16) & 0x3FFF) << 4, sbo = (uint32_t)((d >> 32) & 0x3FFF) << 4;
  return smem[start + (row / 8) * sbo + (k / 16) * lbo + (row % 8) * 16 + (k % 16)];
}

struct Case { const char* name; uint32_t rows, cols, nv; bool be; int ksplit; int fill; };   // fill 0 random, 1 all ones

static int fails = 0;

static void run(const Case& C) {
  std::vector<uint32_t> a((size_t)C.rows * C.cols), b((size_t)C.nv * 3 * C.cols);
  for (auto& x : a) x = C.fill ? 0xFFFFFFFFu : rnd();
  for (auto& x : b) x = C.fill ? 0xFFFFFFFFu : rnd();
  if (!C.fill) { a[0] = 0xFFFFFFFFu; b[0] = 0xFFFFFFFFu; }      // bits 30-31 set; an all-ones query word
  // 64-bit definition
  std::vector<uint32_t> ref((size_t)C.nv * C.rows);
  for (uint32_t v = 0; v < C.nv; v++)
    for (uint32_t r = 0; r < C.rows; r++) {
      uint64_t s = 0;
      for (uint32_t k = 0; k < C.cols; k++)
        for (int t = 0; t < 3; t++) s += (uint64_t)((a[(size_t)r * C.cols + k] >> (10 * t)) & 1023u) * b[(size_t)v * 3 * C.cols + 3 * k + t];
      ref[(size_t)v * C.rows + r] = (uint32_t)s;
    }
  // the vectors as the builder reads them (big-endian words when C.be)
  std::vector<uint32_t> bin(b);
  if (C.be) for (auto& x : bin) x = bswap(x);
  const size_t nch = dtc_chunks(C.cols), ib = dtc_img_bytes(C.cols);
  std::vector<uint8_t> img((size_t)C.nv * ib, 0xA5);
  for (uint32_t v = 0; v < C.nv; v++)
    for (size_t c = 0; c < nch; c++)
      for (int t = 0; t < 3; t++)
        for (int kh = 0; kh < 2; kh++) {
          uint32_t rows[4][4];
          dtc_img_rows(bin.data() + (size_t)v * 3 * C.cols, C.cols, C.be, c, t, kh, rows);
          for (int j = 0; j < 4; j++) memcpy(&img[(size_t)v * ib + dtc_img_off(c, t, kh, j)], rows[j], 16);
        }
  // the image's words past `cols` (the last partial chunk) are zero: the pass relies on them multiplying into nothing
  for (uint32_t v = 0; v < C.nv; v++)
    for (size_t k = C.cols; k < nch * DTC_KW; k++)
      for (int t = 0; t < 3; t++)
        for (int j = 0; j < 4; j++)
          if (img[(size_t)v * ib + dtc_img_off(k / DTC_KW, t, (k % DTC_KW) / 16, j) + k % 16]) {
            printf("%s: image byte past cols not zero\n", C.name);
            fails++;
            return;
          }
  std::vector<uint32_t> out((size_t)C.nv * C.rows, 0);
  std::vector<int> stores((size_t)C.nv * C.rows, 0);
  const uint32_t cps = (uint32_t)((nch + C.ksplit - 1) / C.ksplit);
  std::vector<uint8_t> raw(DTC_ROWS * DTC_KW * 4), bst(6 * DTC_B_TILE), ab(6 * DTC_A_TILE);
  static uint32_t D[4][64][128];
  for (uint32_t v0 = 0; v0 < C.nv; v0 += DTC_VECS)
    for (uint32_t r0 = 0; r0 < C.rows; r0 += DTC_ROWS)
      for (int y = 0; y < C.ksplit; y++) {
        const uint32_t trows = std::min<uint32_t>(DTC_ROWS, C.rows - r0), tnv = std::min<uint32_t>(DTC_VECS, C.nv - v0);
        const uint32_t c0 = y * cps, c1 = std::min<uint32_t>((uint32_t)nch, c0 + cps);
        memset(D, 0, sizeof(D));
        for (uint32_t c = c0; c < c1; c++) {
          memset(raw.data(), 0x5A, raw.size());                   // stale stage contents
          memset(bst.data(), 0x5A, bst.size());
          for (int idx = 0; idx < DTC_ROWS * DTC_KW; idx++) {     // 4-byte copies, zero-filled where the rule says so
            const int r = idx >> 5;
            const uint32_t word = c * DTC_KW + (idx & 31);
            const uint32_t x = dtc_raw_ok(r, word, trows, C.cols) ? a[(size_t)(r0 + r) * C.cols + word] : 0u;
            memcpy(&raw[4 * idx], &x, 4);
          }
          for (int vl = 0; vl < DTC_VECS; vl++)                   // 16-byte copies, zero-filled past the task's vectors
            for (int t = 0; t < 3; t++)
              for (int kh = 0; kh < 2; kh++)
                for (int j = 0; j < 4; j++) {
                  uint8_t* dst = &bst[dtc_b_smem_off(vl, t, kh) + 16 * j];
                  if (vl < (int)tnv) memcpy(dst, &img[(size_t)(v0 + vl) * ib + c * DTC_IMG_CHUNK + dtc_img_off(0, t, kh, j)], 16);
                  else memset(dst, 0, 16);
                }
          memset(ab.data(), 0x3C, ab.size());
          for (int tid = 0; tid < 512; tid++) {                    // unpacking
            const DtcUnpack U = dtc_unpack_thread(tid);
            uint32_t w[4];
            memcpy(w, &raw[(U.row * DTC_KW + 4 * U.kq) * 4], 16);
            for (int t = 0; t < 3; t++)
              for (int i = 0; i < 2; i++) {
                const uint32_t x = dtc_limb4(w, t, i);
                memcpy(&ab[dtc_a_smem_off(U.row, t, i, U.kq)], &x, 4);
              }
          }
          for (int g = 0; g < 4; g++) {                            // the MMAs: D += A (64 x 32) * B (128 x 32)^T per plane
            const int rh = g >> 1, vh = g & 1;
            const int mmax = std::min<int>(64, 2 * std::max<int>(0, (int)trows - 32 * rh));
            const int nmax = std::min<int>(128, 4 * std::max<int>(0, (int)tnv - 32 * vh));
            for (int t = 0; t < 3; t++)
              for (int m = 0; m < mmax; m++)
                for (int n = 0; n < nmax; n++) {
                  uint32_t s = 0;
                  for (int k = 0; k < 32; k++)
                    s += (uint32_t)layout_byte(ab.data(), dtc_a_tile(t, rh), m, k) * layout_byte(bst.data(), dtc_b_tile(t, vh), n, k);
                  D[g][m][n] += s;                                  // s32 accumulation, wrapping
                }
          }
        }
        for (int g = 0; g < 4; g++) {                              // epilogue, lane by lane
          const int rh = g >> 1, vh = g & 1;
          if (!(32 * rh < (int)trows && 32 * vh < (int)tnv)) continue;
          for (int w = 0; w < 4; w++)
            for (int ii = 0; ii < 16; ii++)
              for (int h = 0; h < 2; h++) {
                uint32_t p[32], s1[32], s2[32];
                for (int lane = 0; lane < 32; lane++) {
                  uint32_t acc[2];
                  for (int c = 0; c < 2; c++) acc[c] = D[g][16 * w + lane / 4 + 8 * h][8 * ii + 2 * (lane % 4) + c];
                  p[lane] = dtc_lane_partial(acc[0], acc[1], lane);
                }
                for (int lane = 0; lane < 32; lane++) s1[lane] = p[lane] + p[lane ^ 1];
                for (int lane = 0; lane < 32; lane++) s2[lane] = s1[lane] + s1[lane ^ 4];
                for (int lane = 0; lane < 32; lane++) {
                  const int r = 32 * rh + dtc_frag_row(w, lane, h), v = 32 * vh + dtc_frag_vec(lane, ii);
                  if (dtc_frag_stores(lane, ii, h) && r < (int)trows && v < (int)tnv) {
                    const size_t o = (size_t)(v0 + v) * C.rows + r0 + r;
                    out[o] += s2[lane];                             // a split k range adds (atomicAdd); else one store
                    stores[o]++;
                  }
                }
              }
        }
      }
  int bad = 0;
  for (size_t i = 0; i < out.size(); i++)
    if (out[i] != ref[i] || stores[i] != C.ksplit) bad++;
  if (bad) {
    printf("%s: %d of %zu outputs wrong\n", C.name, bad, out.size());
    fails++;
  }
}

int main() {
  const Case cases[] = {
      {"ragged rows, cols 45, V 3, big-endian", 67, 45, 3, true, 1, 0},
      {"rows 1, cols 1, V 1", 1, 1, 1, false, 1, 0},
      {"rows 33, cols 31, V 37 (both vector halves)", 33, 31, 37, false, 1, 0},
      {"rows 64, cols 33, V 65 (two passes), big-endian", 64, 33, 65, true, 1, 0},
      {"rows 129, cols 70, V 5, split k in 3", 129, 70, 5, false, 3, 0},
      {"rows 31, cols 100, V 64, all ones", 31, 100, 64, true, 2, 1},
      {"K past the s32 range: cols 22100, all ones", 2, 22100, 2, false, 1, 1},
      {"K past the s32 range: cols 22018, random, big-endian", 3, 22018, 3, true, 1, 0},
  };
  for (const Case& C : cases) run(C);
  if (fails) return 1;
  printf("dpir tc emulation ok\n");
  return 0;
}
