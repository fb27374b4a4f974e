// DoublePIR offline setup (lib/doublepir/src/doublepir/doublepir.rs:76-108) on the Hopper tensor cores (wgmma).
//
// The two products of setup(),  h_1 = db.data * a_1  and  h_2 = h_1' * a_2  (matrix/ops.rs:169-191, wrapping u32), have a SMALL
// signed left operand (database entries / base-p digits centred in [-p/2, p/2), p <= 2^10) and a full 32-bit right operand.
// Exact decomposition into 8-bit limbs, everything modulo 2^32:
//     a = a0 + 2^8 a1        a0 = a & 255 (unsigned),  a1 = a >> 8 (arithmetic, signed, |a| < 2^15)
//     b = b0 + 2^8 b1 + 2^16 b2 + 2^24 b3   (unsigned bytes)
//     a b = sum_{i + j <= 3} a_i b_j 2^{8 (i + j)}            (terms with i + j >= 4 vanish mod 2^32)
// Seven limb products per k-step, grouped by shift s = i + j into four s32 register accumulators (wgmma .u8.u8 or .s8.u8 per
// instruction; no saturation, so the accumulators wrap modulo 2^32 — and only their low 32 - 8 s bits matter):  D0 = a0 b0,  D1 = a0 b1 + a1 b0,  D2 = a0 b2 + a1 b1,  D3 = a0 b3 + a1 b2;  c = D0 + D1 << 8 + D2 << 16 + D3 << 24.
//
// Operand images: each limb plane of A ([M][K] bytes) and of B' ([N][K] bytes, i.e. B transposed) is stored as 128 x 32 byte
// tiles in the canonical K-major no-swizzle layout of tc5_layout.cuh, so a tile (or a 32-row quarter of it) is one bulk copy.
// One CTA per 128 x 32 output tile (128 rows of A, one 32-row quarter of a B' tile): warpgroups 0 and 1 compute rows 0..63
// and 64..127 (four 64 x 32 accumulators = 64 registers a thread: wider tiles push ptxas into spilling accumulators of
// in-flight MMAs), warp 8 = producer (ring of k-steps: 2 A tiles + 4 B quarter tiles = 12 KiB per stage).  This is an offline step; the kernel is written for exactness and clarity, not tuned beyond
// keeping the tensor pipe fed.
#include "kernels.h"
#include "tc5_ptx.cuh"

namespace b200pir {

namespace {
using namespace tc5;

constexpr int G_STAGES = 8;
constexpr int G_HALF = TC5_TILE / 2;                    // rows 64..127 of a tile image: 8 row groups = 2048 bytes
constexpr int G_QUARTER = TC5_TILE / 4;                 // 32 rows of a tile image: 4 row groups = 1024 bytes
constexpr int G_STAGE_BYTES = 2 * TC5_TILE + 4 * G_QUARTER; // a0, a1, b0, b1, b2, b3 (32 rows of B')
constexpr int G_THREADS = 2 * 128 + 32;

// limb planes of A (row-major rows x cols u32, small signed entries) as tile images [plane(2)][mt][ks][4096]
__global__ void k_gemm_a_image(uint8_t* __restrict__ img, const uint32_t* __restrict__ a, size_t rows, size_t cols, int mt, int ks) {
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;          // over mt * ks * 128 * 8 (row, group of 4 k)
  if (idx >= (size_t)mt * ks * 128 * 8) return;
  const int kq = (int)(idx & 7), r = (int)((idx >> 3) & 127);
  const size_t tile = idx >> 10;
  const int k_t = (int)(tile % ks), m_t = (int)(tile / ks);
  const size_t row = (size_t)m_t * 128 + r;
  uint32_t w0 = 0, w1 = 0;
#pragma unroll
  for (int i = 0; i < 4; i++) {
    const size_t col = (size_t)k_t * 32 + 4 * kq + i;
    const int32_t v = (row < rows && col < cols) ? (int32_t)a[row * cols + col] : 0;
    w0 |= (uint32_t)(v & 255) << (8 * i);
    w1 |= (uint32_t)((v >> 8) & 255) << (8 * i);
  }
  const size_t plane = (size_t)mt * ks * TC5_TILE;
  const size_t off = tile * TC5_TILE + tc5_tile_off(r, 4 * kq);
  *reinterpret_cast<uint32_t*>(img + off) = w0;
  *reinterpret_cast<uint32_t*>(img + plane + off) = w1;
}
// limb planes of B (row-major k_rows x n_cols u32) TRANSPOSED: tile images [plane(4)][nt][ks][4096], tile row = column of B
__global__ void k_gemm_b_image(uint8_t* __restrict__ img, const uint32_t* __restrict__ b, size_t k_rows, size_t n_cols, int nt, int ks) {
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;          // over nt * ks * 8 * 128, column fastest (coalesced reads)
  if (idx >= (size_t)nt * ks * 128 * 8) return;
  const int c = (int)(idx & 127), kq = (int)((idx >> 7) & 7);
  const size_t tile = idx >> 10;
  const int k_t = (int)(tile % ks), n_t = (int)(tile / ks);
  const size_t col = (size_t)n_t * 128 + c;
  uint32_t w[4] = {0, 0, 0, 0};
#pragma unroll
  for (int i = 0; i < 4; i++) {
    const size_t k = (size_t)k_t * 32 + 4 * kq + i;
    const uint32_t v = (col < n_cols && k < k_rows) ? b[k * n_cols + col] : 0u;
#pragma unroll
    for (int j = 0; j < 4; j++) w[j] |= ((v >> (8 * j)) & 255u) << (8 * i);
  }
  const size_t plane = (size_t)nt * ks * TC5_TILE;
  const size_t off = tile * TC5_TILE + tc5_tile_off(c, 4 * kq);
#pragma unroll
  for (int j = 0; j < 4; j++) *reinterpret_cast<uint32_t*>(img + j * plane + off) = w[j];
}

struct GemmSmem {
  uint64_t full[G_STAGES], empty[G_STAGES];
};

// c[m][n] = sum_k a[m][k] b[k][n] mod 2^32 for one 128 x 32 tile per CTA (grid = (4 nt, mt))
__global__ void __launch_bounds__(G_THREADS, 1)
k_dpir_gemm(const uint8_t* __restrict__ a_img, const uint8_t* __restrict__ b_img, uint32_t* __restrict__ c, size_t rows, size_t n_cols,
            int mt, int nt, int ks) {
  extern __shared__ __align__(1024) uint8_t gsm[];
  GemmSmem* S = reinterpret_cast<GemmSmem*>(gsm + (size_t)G_STAGES * G_STAGE_BYTES);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n_t = blockIdx.x >> 2, n_q = blockIdx.x & 3, m_t = blockIdx.y;
  const size_t a_plane = (size_t)mt * ks * TC5_TILE, b_plane = (size_t)nt * ks * TC5_TILE;
  if (threadIdx.x == 0) {
    for (int s = 0; s < G_STAGES; s++) { mbar_init(&S->full[s], 1); mbar_init(&S->empty[s], 2); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp == 8) {
    int stage = 0; uint32_t phase = 0;
    for (int k = 0; k < ks; k++) {
      mbar_wait(&S->empty[stage], phase ^ 1);
      if (elect_one()) {
        uint8_t* dst = gsm + (size_t)stage * G_STAGE_BYTES;
        mbar_expect_tx(&S->full[stage], G_STAGE_BYTES);
        const size_t a_off = ((size_t)m_t * ks + k) * TC5_TILE, b_off = ((size_t)n_t * ks + k) * TC5_TILE + n_q * G_QUARTER;
        bulk_g2s(dst + 0 * TC5_TILE, a_img + a_off, TC5_TILE, &S->full[stage]);
        bulk_g2s(dst + 1 * TC5_TILE, a_img + a_plane + a_off, TC5_TILE, &S->full[stage]);
#pragma unroll
        for (int j = 0; j < 4; j++) bulk_g2s(dst + 2 * TC5_TILE + j * G_QUARTER, b_img + j * b_plane + b_off, G_QUARTER, &S->full[stage]);
      }
      __syncwarp();
      if (++stage == G_STAGES) { stage = 0; phase ^= 1; }
    }
  } else if (warp < 8) {
    const int wg = warp >> 2, w = warp & 3;
    const bool leader = (threadIdx.x & 127) == 0;
    uint32_t d0[16], d1[16], d2[16], d3[16];                          // shift s accumulates into ds
#pragma unroll
    for (int i = 0; i < 16; i++) { d0[i] = 0; d1[i] = 0; d2[i] = 0; d3[i] = 0; }
    int stage = 0, prev = -1; uint32_t phase = 0;
    for (int k = 0; k < ks; k++) {
      mbar_wait(&S->full[stage], phase);
      const uint32_t base = smem_u32(gsm + (size_t)stage * G_STAGE_BYTES);
      const uint64_t a0 = tc5_smem_desc(base + wg * G_HALF), a1 = tc5_smem_desc(base + TC5_TILE + wg * G_HALF);
      uint64_t bd[4];
#pragma unroll
      for (int j = 0; j < 4; j++) bd[j] = tc5_smem_desc(base + 2 * TC5_TILE + j * G_QUARTER);
      wgmma_fence();
      wgmma_m64n32k32<false>(d0, a0, bd[0]);
      wgmma_m64n32k32<false>(d1, a0, bd[1]);
      wgmma_m64n32k32<true>(d1, a1, bd[0]);
      wgmma_m64n32k32<false>(d2, a0, bd[2]);
      wgmma_m64n32k32<true>(d2, a1, bd[1]);
      wgmma_m64n32k32<false>(d3, a0, bd[3]);
      wgmma_m64n32k32<true>(d3, a1, bd[2]);
      wgmma_commit();
      wgmma_wait<1>();                                                // the previous stage's MMAs have completed: release it
      if (prev >= 0 && leader) mbar_arrive(&S->empty[prev]);
      prev = stage;
      if (++stage == G_STAGES) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
    wgmma_fence_operands(d0);
    wgmma_fence_operands(d1);
    wgmma_fence_operands(d2);
    wgmma_fence_operands(d3);
    // accumulator fragment: d[4 i + 2 h + e] = D[16 w + lane/4 + 8 h][8 i + 2 (lane%4) + e]
#pragma unroll
    for (int h = 0; h < 2; h++) {
      const size_t row = (size_t)m_t * 128 + wg * 64 + w * 16 + (lane >> 2) + 8 * h;
      if (row >= rows) continue;
#pragma unroll
      for (int i = 0; i < 4; i++)
#pragma unroll
        for (int e = 0; e < 2; e++) {
          const int r = 4 * i + 2 * h + e;
          const size_t col = (size_t)n_t * 128 + n_q * 32 + 8 * i + 2 * (lane & 3) + e;
          if (col < n_cols) c[row * n_cols + col] = d0[r] + (d1[r] << 8) + (d2[r] << 16) + (d3[r] << 24);
        }
    }
  }
}

// doublepir.rs:83-85: transpose, expand (matrix/contract.rs:62-78: delta digits base p, centred), concat_cols (indexing.rs:82-101)
//   h (l x n)  ->  out ((n delta x) x (l / x)),  out[(i delta + f) + n delta (j % x)][j / x] = digit_f(h[j][i]) - p / 2
__global__ void k_dpir_transpose_expand_concat(uint32_t* __restrict__ out, const uint32_t* __restrict__ h, size_t l, size_t n, uint32_t p,
                                               int delta, size_t x) {
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;          // over l * n, i (column of h) fastest
  if (idx >= l * n) return;
  const size_t i = idx % n, j = idx / n;
  uint32_t val = h[j * n + i];
  const size_t out_cols = l / x;
  for (int f = 0; f < delta; f++) {
    out[((i * delta + f) + n * delta * (j % x)) * out_cols + j / x] = (val % p) - p / 2;
    val /= p;
  }
}
// squish(m + add) (matrix/squish.rs:52-70 with the default parameters: three 10-bit values per word)
__global__ void k_dpir_add_squish(uint32_t* __restrict__ out, const uint32_t* __restrict__ m, size_t rows, size_t cols, uint32_t add) {
  const size_t out_cols = (cols + 2) / 3;
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= rows * out_cols) return;
  const size_t i = idx / out_cols, j = idx % out_cols;
  uint32_t w = 0;
  for (int k = 0; k < 3; k++)
    if (3 * j + k < cols) w += (m[i * cols + 3 * j + k] + add) << (10 * k);
  out[idx] = w;
}
// a_2_copy: rows padded with zero rows to a multiple of 3, transposed (doublepir.rs:96-100)
__global__ void k_dpir_pad_transpose(uint32_t* __restrict__ out, const uint32_t* __restrict__ a, size_t rows, size_t cols, size_t rows3) {
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;          // over cols * rows3
  if (idx >= cols * rows3) return;
  const size_t r = idx % rows3, c = idx / rows3;
  out[idx] = r < rows ? a[r * cols + c] : 0u;
}

inline unsigned blocks(size_t total, int block) { return (unsigned)((total + block - 1) / block); }

}  // namespace

// c (rows x n_cols, device) = a (rows x k_dim, device, entries in [-2^15, 2^15) as wrapping u32) * b (k_dim x n_cols, device) mod 2^32
void launch_dpir_gemm(uint32_t* c, const uint32_t* a, const uint32_t* b, size_t rows, size_t k_dim, size_t n_cols, cudaStream_t s) {
  const int mt = (int)((rows + 127) / 128), nt = (int)((n_cols + 127) / 128), ks = (int)((k_dim + 31) / 32);
  uint8_t *a_img = nullptr, *b_img = nullptr;
  B200_CUDA(cudaMalloc(&a_img, (size_t)2 * mt * ks * TC5_TILE));
  B200_CUDA(cudaMalloc(&b_img, (size_t)4 * nt * ks * TC5_TILE));
  g_kernel_launches += 3;
  k_gemm_a_image<<<blocks((size_t)mt * ks * 1024, 256), 256, 0, s>>>(a_img, a, rows, k_dim, mt, ks);
  k_gemm_b_image<<<blocks((size_t)nt * ks * 1024, 256), 256, 0, s>>>(b_img, b, k_dim, n_cols, nt, ks);
  const size_t smem = (size_t)G_STAGES * G_STAGE_BYTES + sizeof(GemmSmem) + 16;
  opt_in_smem(k_dpir_gemm, (int)smem);
  k_dpir_gemm<<<dim3(4 * nt, mt), G_THREADS, smem, s>>>(a_img, b_img, c, rows, n_cols, mt, nt, ks);
  cudaError_t e = cudaStreamSynchronize(s);
  cudaFree(a_img);
  cudaFree(b_img);
  if (e != cudaSuccess) throw Error(-3, std::string("dpir gemm: ") + cudaGetErrorString(e));
}
void launch_dpir_transpose_expand_concat(uint32_t* out, const uint32_t* h, size_t l, size_t n, uint32_t p, int delta, size_t x,
                                         cudaStream_t s) {
  ++g_kernel_launches;
  k_dpir_transpose_expand_concat<<<blocks(l * n, 256), 256, 0, s>>>(out, h, l, n, p, delta, x);
}
void launch_dpir_add_squish(uint32_t* out, const uint32_t* m, size_t rows, size_t cols, uint32_t add, cudaStream_t s) {
  ++g_kernel_launches;
  k_dpir_add_squish<<<blocks(rows * ((cols + 2) / 3), 256), 256, 0, s>>>(out, m, rows, cols, add);
}
void launch_dpir_pad_transpose(uint32_t* out, const uint32_t* a, size_t rows, size_t cols, size_t rows3, cudaStream_t s) {
  ++g_kernel_launches;
  k_dpir_pad_transpose<<<blocks(cols * rows3, 256), 256, 0, s>>>(out, a, rows, cols, rows3);
}

}  // namespace b200pir
