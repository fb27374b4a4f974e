// First-dimension kernels on the IMAD layout (format 0): multiply_reg_by_database (lib/spiral-rs/src/server.rs:155-221) over
// an HBM-resident database and the query operand it reads; the single-item upsert into any layout; and DoublePIR's
// single-vector packed matvec (lib/doublepir/src/matrix/kernels.rs:14-178) with the small kernels of answer()'s tail.  The
// item writer (k_write_items) runs the NTT and so lives with the other transforms in poly_kernels.cu.  The products are pure
// streams of the database: 8 bytes read -> 4 (u32 x u32 -> u64) multiply-adds, so the design goal is coalesced 16-byte loads,
// many of them in flight per SM, and no shared-memory or shuffle traffic at all.
//
// Device layout of one slice (format 0, built from the reference layout at upload, export_kernels.cu; the C ABI accepts
// the reference layout [z][ii][j], server.rs:263-266):
//     db_dev[ii][jp][z] = uint4{ w(j=2jp).lo, w(2jp).hi, w(2jp+1).lo, w(2jp+1).hi }      (lo = mod q0, hi = mod q1)
// so thread z of a warp reads 16 contiguous bytes and the warp 512 contiguous bytes.  The NTT
// coordinate z is the one fully independent axis of the product, so it is the thread axis: each
// thread owns one z, R database rows and all j, and keeps its 4R (x NQ queries) 64-bit partial sums
// in registers.  Products are < 2^56, so the sums are reduced mod q_n every 256 terms (the reference
// accumulates in u128 and reduces once; both give the canonical residue).
#include "kernels.h"
#include "item_place.cuh"
#include <algorithm>

namespace b200pir {

namespace {

template <int R, int NQ, int UNROLL>
__global__ void __launch_bounds__(512)
k_multiply(DevParams P, MulGeom G, const uint4* __restrict__ db, const uint4* __restrict__ qv, uint32_t* __restrict__ out,
           int slice_begin, size_t q_stride, size_t out_stride) {
  const int z = blockIdx.x * blockDim.x + threadIdx.x;
  const int rowgroup = blockIdx.y * blockDim.y + threadIdx.y;
  const int ii0 = rowgroup * R;
  const int slice = slice_begin + blockIdx.z;
  if (ii0 >= G.num_per) return;
  const int half = G.dim0 >> 1;
  const size_t row_stride = (size_t)half * POLY;
  const uint4* dbp = db + ((size_t)slice * G.num_per + ii0) * row_stride + z;
  const uint4* qp = qv + z;

  uint64_t acc[NQ][R][4];
#pragma unroll
  for (int a = 0; a < NQ; a++)
#pragma unroll
    for (int r = 0; r < R; r++)
#pragma unroll
      for (int c = 0; c < 4; c++) acc[a][r][c] = 0;

  for (int jp0 = 0; jp0 < half; jp0 += 128) {
    const int jend = min(jp0 + 128, half);
#pragma unroll UNROLL
    for (int jp = jp0; jp < jend; jp++) {
      uint4 d[R];
#pragma unroll
      for (int r = 0; r < R; r++) d[r] = ld_stream_v4(dbp + (size_t)r * row_stride + (size_t)jp * POLY);
#pragma unroll
      for (int a = 0; a < NQ; a++) {
        const uint4 qa = __ldg(qp + (size_t)a * q_stride + (size_t)(2 * jp) * POLY);
        const uint4 qb = __ldg(qp + (size_t)a * q_stride + (size_t)(2 * jp + 1) * POLY);
#pragma unroll
        for (int r = 0; r < R; r++) {
          acc[a][r][0] += (uint64_t)d[r].x * qa.x;     // n0, row 0 of the ciphertext
          acc[a][r][1] += (uint64_t)d[r].x * qa.z;     // n0, row 1
          acc[a][r][2] += (uint64_t)d[r].y * qa.y;     // n1, row 0
          acc[a][r][3] += (uint64_t)d[r].y * qa.w;     // n1, row 1
          acc[a][r][0] += (uint64_t)d[r].z * qb.x;
          acc[a][r][1] += (uint64_t)d[r].z * qb.z;
          acc[a][r][2] += (uint64_t)d[r].w * qb.y;
          acc[a][r][3] += (uint64_t)d[r].w * qb.w;
        }
      }
    }
    if (jend < half) {       // 256 products per accumulator so far: fold back below 2^28
#pragma unroll
      for (int a = 0; a < NQ; a++)
#pragma unroll
        for (int r = 0; r < R; r++) {
          acc[a][r][0] = barrett64(acc[a][r][0], P.cr1[0], P.q[0]);
          acc[a][r][1] = barrett64(acc[a][r][1], P.cr1[0], P.q[0]);
          acc[a][r][2] = barrett64(acc[a][r][2], P.cr1[1], P.q[1]);
          acc[a][r][3] = barrett64(acc[a][r][3], P.cr1[1], P.q[1]);
        }
    }
  }
  // out[ii].data[r*2N + n*N + z]   (server.rs:204-217)
#pragma unroll
  for (int a = 0; a < NQ; a++)
#pragma unroll
    for (int r = 0; r < R; r++) {
      uint32_t* o = out + (size_t)a * out_stride + ((size_t)slice * G.num_per + ii0 + r) * 4 * POLY + z;
      o[0 * POLY] = barrett64(acc[a][r][0], P.cr1[0], P.q[0]);      // row 0, n0
      o[1 * POLY] = barrett64(acc[a][r][2], P.cr1[1], P.q[1]);      // row 0, n1
      o[2 * POLY] = barrett64(acc[a][r][1], P.cr1[0], P.q[0]);      // row 1, n0
      o[3 * POLY] = barrett64(acc[a][r][3], P.cr1[1], P.q[1]);      // row 1, n1
    }
}

template <int R, int NQ, int UNROLL>
void launch_mul_t(const DevParams& P, const MulGeom& G, const uint4* db, const uint4* q, uint32_t* out, int slice_begin,
                  int slice_count, size_t q_stride, size_t out_stride, int groups, cudaStream_t s) {
  int rowgroups = G.num_per / R;
  if (rowgroups * R != G.num_per) throw Error(-2, "multiply: num_per must be a multiple of the row tile");
  if (groups > rowgroups) groups = rowgroups;
  while (rowgroups % groups) groups--;
  dim3 block(128, groups);
  dim3 grid(POLY / 128, rowgroups / groups, slice_count);
  ++g_kernel_launches;
  k_multiply<R, NQ, UNROLL><<<grid, block, 0, s>>>(P, G, db, q, out, slice_begin, q_stride, out_stride);
}

__global__ void k_query_to_dev(MulGeom G, uint4* q_dev, const uint64_t* v) {
  size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;     // over dim0 * 2048, z fastest
  if (idx >= (size_t)G.dim0 * POLY) return;
  int z = (int)(idx % POLY), j = (int)(idx / POLY);
  const uint64_t* src = v + ((size_t)z * G.dim0 + j) * 2;
  uint64_t a0 = src[0], a1 = src[1];
  q_dev[((size_t)(j >> 1) * 2 + (j & 1)) * POLY + z] =
      make_uint4((uint32_t)a0, (uint32_t)(a0 >> 32), (uint32_t)a1, (uint32_t)(a1 >> 32));
}

// one item polynomial (2048 packed words lo|hi<<32) into the database, in any layout
__global__ void k_db_upsert(DbLayout L, int slice, int il, int j, const uint64_t* poly) {
  const int z = blockIdx.x * blockDim.x + threadIdx.x;
  if (z >= POLY) return;
  const uint64_t w = poly[z];
  place_item(L, slice, il, j, z, (uint32_t)w, (uint32_t)(w >> 32));
}

// ------------------------------------------------------------------ DoublePIR
// out[i] = sum_k sum_{m<3} ((a[i][k] >> 10m) & 1023) * b[3k+m]   (wrapping u32; kernels.rs:52-93)
// Odd column counts, whose rows are not 8-byte aligned: one warp per ROWS rows, lanes stride over k.  b is staged in shared
// memory as three planes bm[m][k].
__global__ void __launch_bounds__(256)
k_dpir_matvec(uint32_t* __restrict__ out, const uint32_t* __restrict__ a, const uint32_t* __restrict__ b, size_t rows,
              size_t cols, size_t cols_pad) {
  constexpr int ROWS = 4;
  extern __shared__ __align__(16) uint32_t bsm[];          // [3][cols_pad]
  for (size_t k = threadIdx.x; k < cols; k += blockDim.x) {
    bsm[k] = b[3 * k];
    bsm[cols_pad + k] = b[3 * k + 1];
    bsm[2 * cols_pad + k] = b[3 * k + 2];
  }
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  // launch_dpir_matvec sends even column counts to k_dpir_matvec_row, so vec2 is never true.  The branch stays because without
  // it the odd-column loop compiles to 40 registers instead of 32 and ran 0.2 % slower at 2^23 x 1365 on H100.
  const bool vec2 = (cols & 1) == 0;
  for (size_t row0 = ((size_t)blockIdx.x * nwarps + warp) * ROWS; row0 < rows; row0 += (size_t)gridDim.x * nwarps * ROWS) {
    uint32_t acc[ROWS];
#pragma unroll
    for (int r = 0; r < ROWS; r++) acc[r] = 0;
    if (vec2) {
      for (size_t k = 2 * (size_t)lane; k < cols; k += 64) {
        uint2 b0 = *reinterpret_cast<const uint2*>(bsm + k);
        uint2 b1 = *reinterpret_cast<const uint2*>(bsm + cols_pad + k);
        uint2 b2 = *reinterpret_cast<const uint2*>(bsm + 2 * cols_pad + k);
#pragma unroll
        for (int r = 0; r < ROWS; r++) {
          if (row0 + r < rows) {
            uint2 d;
            asm volatile("ld.global.nc.L1::no_allocate.v2.u32 {%0,%1}, [%2];"
                         : "=r"(d.x), "=r"(d.y) : "l"(a + (row0 + r) * cols + k));
            acc[r] += (d.x & 1023u) * b0.x + ((d.x >> 10) & 1023u) * b1.x + ((d.x >> 20) & 1023u) * b2.x;
            acc[r] += (d.y & 1023u) * b0.y + ((d.y >> 10) & 1023u) * b1.y + ((d.y >> 20) & 1023u) * b2.y;
          }
        }
      }
    } else {
      for (size_t k = lane; k < cols; k += 32) {
        uint32_t b0 = bsm[k], b1 = bsm[cols_pad + k], b2 = bsm[2 * cols_pad + k];
#pragma unroll
        for (int r = 0; r < ROWS; r++) {
          if (row0 + r < rows) {
            uint32_t d = __ldg(a + (row0 + r) * cols + k);
            acc[r] += (d & 1023u) * b0 + ((d >> 10) & 1023u) * b1 + ((d >> 20) & 1023u) * b2;
          }
        }
      }
    }
#pragma unroll
    for (int r = 0; r < ROWS; r++) {
      uint32_t v = acc[r];
#pragma unroll
      for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
      if (lane == 0 && row0 + r < rows) out[row0 + r] = v;
    }
  }
}

// Even column counts: one row per warp; every lane keeps U independent 8-byte streaming loads in flight before it consumes
// them.  b is staged in shared memory as three planes bm[m][k], so a lane's two consecutive k read one conflict-free 8-byte
// word per plane.
__global__ void __launch_bounds__(256)
k_dpir_matvec_row(uint32_t* __restrict__ out, const uint32_t* __restrict__ a, const uint32_t* __restrict__ b, size_t rows,
                  size_t cols, size_t cols_pad) {
  constexpr int U = 8;
  extern __shared__ __align__(16) uint32_t bsm[];          // [3][cols_pad]
  for (size_t k = threadIdx.x; k < cols_pad; k += blockDim.x) {
    bool in = k < cols;
    bsm[k] = in ? b[3 * k] : 0u;
    bsm[cols_pad + k] = in ? b[3 * k + 1] : 0u;
    bsm[2 * cols_pad + k] = in ? b[3 * k + 2] : 0u;
  }
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  const size_t pairs = cols >> 1;                           // cols is even on this path
  for (size_t row = (size_t)blockIdx.x * nwarps + warp; row < rows; row += (size_t)gridDim.x * nwarps) {
    const uint2* ar = reinterpret_cast<const uint2*>(a + row * cols);
    uint32_t acc = 0;
    for (size_t p0 = 0; p0 < pairs; p0 += 32 * U) {
      uint2 d[U];
#pragma unroll
      for (int u = 0; u < U; u++) {
        size_t p = p0 + (size_t)u * 32 + lane;
        d[u] = make_uint2(0u, 0u);
        if (p < pairs)
          asm volatile("ld.global.nc.L1::no_allocate.v2.u32 {%0,%1}, [%2];" : "=r"(d[u].x), "=r"(d[u].y) : "l"(ar + p));
      }
#pragma unroll
      for (int u = 0; u < U; u++) {
        size_t p = p0 + (size_t)u * 32 + lane;
        if (p < pairs) {
          uint2 b0 = *reinterpret_cast<const uint2*>(bsm + 2 * p);
          uint2 b1 = *reinterpret_cast<const uint2*>(bsm + cols_pad + 2 * p);
          uint2 b2 = *reinterpret_cast<const uint2*>(bsm + 2 * cols_pad + 2 * p);
          acc += (d[u].x & 1023u) * b0.x + ((d[u].x >> 10) & 1023u) * b1.x + ((d[u].x >> 20) & 1023u) * b2.x;
          acc += (d[u].y & 1023u) * b0.y + ((d[u].y >> 10) & 1023u) * b1.y + ((d[u].y >> 20) & 1023u) * b2.y;
        }
      }
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, off);
    if (lane == 0) out[row] = acc;
  }
}

// Rows too wide for `b` to fit in shared memory (3 * cols words > 200 KiB; the reference's short-and-wide databases, e.g.
// l = 29, m = 65536 for 2^24 one-bit entries, doublepir.rs:471-483): one CTA per row, `b` read through L2.
__global__ void __launch_bounds__(256)
k_dpir_matvec_wide(uint32_t* __restrict__ out, const uint32_t* __restrict__ a, const uint32_t* __restrict__ b, size_t rows,
                   size_t cols) {
  __shared__ uint32_t part[8];
  const size_t row = blockIdx.x;
  if (row >= rows) return;
  const uint32_t* ar = a + row * cols;
  uint32_t acc = 0;
  for (size_t k = threadIdx.x; k < cols; k += blockDim.x) {
    const uint32_t d = __ldg(ar + k);
    const uint32_t* bp = b + 3 * k;
    acc += (d & 1023u) * __ldg(bp) + ((d >> 10) & 1023u) * __ldg(bp + 1) + ((d >> 20) & 1023u) * __ldg(bp + 2);
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, off);
  if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    uint32_t t = 0;
    for (int w = 0; w < 8; w++) t += part[w];
    out[row] = t;
  }
}

// kernels.rs:180-278: out[i][j] = sum_k sum_m ((a[i][k] >> 10m) & 1023) * b[j][3k+m]   (one warp per output)
__global__ void k_dpir_mul_transposed(uint32_t* __restrict__ out, const uint32_t* __restrict__ a, const uint32_t* __restrict__ b,
                                      size_t a_rows, size_t a_cols, size_t b_rows, size_t b_cols) {
  const size_t warp = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= a_rows * b_rows) return;
  const size_t i = warp / b_rows, j = warp % b_rows;
  uint32_t acc = 0;
  for (size_t k = lane; k < a_cols; k += 32) {
    uint32_t d = __ldg(a + i * a_cols + k);
    const uint32_t* bp = b + j * b_cols + 3 * k;
    acc += (d & 1023u) * __ldg(bp) + ((d >> 10) & 1023u) * __ldg(bp + 1) + ((d >> 20) & 1023u) * __ldg(bp + 2);
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, off);
  if (lane == 0) out[i * b_rows + j] = acc;
}
// matrix/indexing.rs:117-143 (basis 10, d 3): one thread per output word
__global__ void k_dpir_transpose_expand(uint32_t* __restrict__ out, const uint32_t* __restrict__ a, size_t rows, size_t cols,
                                        uint64_t modulus, size_t delta, size_t concat, size_t out_rows, size_t out_cols) {
  size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= out_rows * out_cols) return;
  const size_t r = idx / out_cols, cd = idx % out_cols;
  const size_t jmod = r / (cols * delta), rem = r % (cols * delta), i = rem / delta, f = rem % delta;
  uint32_t acc = 0;
  for (size_t cc = 0; cc < 3; cc++) {
    const size_t c = cd * 3 + cc, j = c * concat + jmod;
    if (j < rows) {
      uint64_t val = a[i + j * cols];
      for (size_t t = 0; t < f; t++) val /= modulus;
      acc += (uint32_t)((val % modulus) << (10 * cc));
    }
  }
  out[idx] = acc;
}

}  // namespace

void launch_dpir_mul_transposed(uint32_t* out, const uint32_t* a, const uint32_t* b, size_t a_rows, size_t a_cols,
                                size_t b_rows, size_t b_cols, cudaStream_t s) {
  ++g_kernel_launches;
  k_dpir_mul_transposed<<<grid1d(a_rows * b_rows * 32, 256), 256, 0, s>>>(out, a, b, a_rows, a_cols, b_rows, b_cols);
}
void launch_dpir_transpose_expand(uint32_t* out, const uint32_t* a, size_t rows, size_t cols, uint64_t modulus, size_t delta,
                                  size_t concat, size_t out_rows, size_t out_cols, cudaStream_t s) {
  ++g_kernel_launches;
  k_dpir_transpose_expand<<<grid1d(out_rows * out_cols, 256), 256, 0, s>>>(out, a, rows, cols, modulus, delta, concat,
                                                                           out_rows, out_cols);
}
void launch_multiply(const DevParams& P, const MulGeom& G, const uint4* db_dev, const uint4* q_dev, uint32_t* out,
                     int slice_begin, int slice_count, int nq, size_t q_stride, size_t out_stride, cudaStream_t s) {
  if (G.dim0 < 2 || (G.dim0 & 1)) throw Error(-2, "multiply: dim0 must be even");
  // row tile: the largest of {8,4,2,1} dividing num_per (num_per is a power of two)
  const int R = G.num_per >= 8 ? 8 : G.num_per;
#define MUL_CASE(RR, QQ, UU, GG)                                                                                     \
  launch_mul_t<RR, QQ, UU>(P, G, db_dev, q_dev, out, slice_begin, slice_count, q_stride, out_stride, GG, s)
  if (nq == 1) {
    if (R == 8) MUL_CASE(8, 1, 1, 2);
    else if (R == 4) MUL_CASE(4, 1, 2, 4);
    else if (R == 2) MUL_CASE(2, 1, 2, 2);
    else MUL_CASE(1, 1, 2, 1);
  } else if (nq == 2) {
    if (R >= 4) { if (G.num_per % 4) throw Error(-2, "multiply: bad num_per"); MUL_CASE(4, 2, 1, 2); }
    else if (R == 2) MUL_CASE(2, 2, 1, 2);
    else MUL_CASE(1, 2, 1, 1);
  } else if (nq == 4) {
    if (R >= 2) MUL_CASE(2, 4, 1, 2);
    else MUL_CASE(1, 4, 1, 1);
  } else {
    throw Error(-2, "multiply: nq must be 1, 2 or 4");
  }
#undef MUL_CASE
}
void launch_query_to_dev(const MulGeom& G, uint4* q_dev, const uint64_t* v_firstdim, cudaStream_t s) {
  size_t total = (size_t)G.dim0 * POLY;
  ++g_kernel_launches;
  k_query_to_dev<<<grid1d(total, 256), 256, 0, s>>>(G, q_dev, v_firstdim);
}
void launch_db_upsert(const DbLayout& L, int slice, int il, int j, const uint64_t* poly, cudaStream_t s) {
  ++g_kernel_launches;
  k_db_upsert<<<POLY / 256, 256, 0, s>>>(L, slice, il, j, poly);
}
void launch_dpir_matvec(uint32_t* out, const uint32_t* a, const uint32_t* b, size_t rows, size_t cols, cudaStream_t s) {
  size_t cols_pad = (cols + 3) & ~(size_t)3;
  size_t smem = 3 * cols_pad * 4;
  if (rows == 0) return;
  if (smem > 200 * 1024) {
    if (rows > 0x7FFFFFFFull) throw Error(-2, "dpir: too many rows for the wide-row kernel");
    ++g_kernel_launches;
    k_dpir_matvec_wide<<<(unsigned)rows, 256, 0, s>>>(out, a, b, rows, cols);
    return;
  }
  if ((cols & 1) == 0) {
    unsigned g = (unsigned)std::min<size_t>((rows + 7) / 8, (size_t)132 * 8);
    cudaFuncSetAttribute(k_dpir_matvec_row, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    ++g_kernel_launches;
    k_dpir_matvec_row<<<g, 256, smem, s>>>(out, a, b, rows, cols, cols_pad);
    return;
  }
  size_t warps_needed = (rows + 3) / 4;
  unsigned grid = (unsigned)std::min<size_t>((warps_needed + 7) / 8, (size_t)132 * 8);
  cudaFuncSetAttribute(k_dpir_matvec, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  ++g_kernel_launches;
  k_dpir_matvec<<<grid, 256, smem, s>>>(out, a, b, rows, cols, cols_pad);
}

}  // namespace b200pir
