// DoublePIR's packed matrix x vector kernels off the tensor cores (sm_90a).  The single-vector matvec
// (lib/doublepir/src/matrix/kernels.rs:14-178) with the small kernels of answer()'s tail; and the matrix x many vectors of
// the database pass, the h_1 pass and the a_1' * q_2 products of answer() (doublepir.rs:246-350) for every request of a call,
// one matrix read per pass of up to kDpirMvMaxVecs vectors.
#include "dpir_kernels.h"

namespace b200pir {
namespace {

constexpr int kMvThreads = 256;
constexpr int kMvRowsPerWarp = kDpirMvRows / (kMvThreads / 32);
constexpr int kMvChunk = 256;                 // k (packed columns) staged per round: V x 256 x 16 bytes of shared memory

__device__ __forceinline__ uint32_t bswap32(uint32_t v) { return __byte_perm(v, 0, 0x0123); }

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

// out_v[r] = sum_k sum_{t<3} ((a[r][k] >> 10t) & 1023) * b_v[3k+t]   (wrapping u32; kernels.rs:52-93), for the nv <= V vectors
// of one task.  CTA = one task's rows (8 warps x RB rows) over the packed columns [y * k_per_split, ...).  The task's vectors
// are staged through shared memory as uint4 {b[3k], b[3k+1], b[3k+2], 0}, [v][k], so the lanes of a warp read consecutive
// 16-byte cells.  Each lane reads one matrix word per row, splits it into its three digits once, and applies them to all V
// vectors; a staged cell serves the warp's RB rows.  Partial sums of a split k range are combined with atomicAdd (exact: the
// arithmetic is modulo 2^32 and order-free).
template <int V, int U>
__global__ void __launch_bounds__(kMvThreads, 2)
k_dpir_matvec_multi(const DpirMvTask* __restrict__ tasks, const DpirMvVec* __restrict__ vecs, uint32_t cols, uint32_t k_per_split,
                    int flags) {
  constexpr int RB = kMvRowsPerWarp;
  extern __shared__ uint4 bs[];                                  // [V][kMvChunk]
  const DpirMvTask t = tasks[blockIdx.x];
  const uint32_t kbeg = blockIdx.y * k_per_split;
  const uint32_t kend = min(cols, kbeg + k_per_split);
  const int lane = threadIdx.x & 31, r0 = (threadIdx.x >> 5) * RB;
  const bool b_be = flags & DPIR_MV_B_BE;
  uint32_t acc[V][RB];
#pragma unroll
  for (int v = 0; v < V; v++)
#pragma unroll
    for (int r = 0; r < RB; r++) acc[v][r] = 0;
  for (uint32_t kc0 = kbeg; kc0 < kend; kc0 += kMvChunk) {
    const uint32_t kn = min((uint32_t)kMvChunk, kend - kc0);
    __syncthreads();                                             // the previous chunk has been consumed
    for (uint32_t i = threadIdx.x; i < t.nv * kn; i += kMvThreads) {
      const uint32_t v = i / kn, kk = i - v * kn;
      const uint32_t* bp = vecs[t.vec0 + v].b + 3 * (size_t)(kc0 + kk);
      uint32_t x0 = __ldg(bp), x1 = __ldg(bp + 1), x2 = __ldg(bp + 2);
      if (b_be) { x0 = bswap32(x0); x1 = bswap32(x1); x2 = bswap32(x2); }
      bs[v * kMvChunk + kk] = make_uint4(x0, x1, x2, 0u);
    }
    __syncthreads();
    if (r0 >= (int)t.rows) continue;                             // warp-uniform: this warp has no rows in the task
    for (uint32_t k0 = lane; k0 < kn; k0 += 32 * U) {
      uint32_t d[U][RB];
#pragma unroll
      for (int u = 0; u < U; u++)
#pragma unroll
        for (int r = 0; r < RB; r++) {
          const uint32_t k = k0 + 32 * u;
          d[u][r] = 0u;
          if (k < kn && r0 + r < (int)t.rows) {
            const uint32_t* p = t.a + (size_t)(r0 + r) * cols + kc0 + k;
            asm volatile("ld.global.nc.L1::no_allocate.u32 %0, [%1];" : "=r"(d[u][r]) : "l"(p));
          }
        }
#pragma unroll
      for (int u = 0; u < U; u++) {
        const uint32_t k = k0 + 32 * u;
        if (k >= kn) break;
        uint32_t d0[RB], d1[RB], d2[RB];
#pragma unroll
        for (int r = 0; r < RB; r++) { d0[r] = d[u][r] & 1023u; d1[r] = (d[u][r] >> 10) & 1023u; d2[r] = (d[u][r] >> 20) & 1023u; }
#pragma unroll
        for (int v = 0; v < V; v++) {
          const uint4 b = bs[v * kMvChunk + k];
#pragma unroll
          for (int r = 0; r < RB; r++) acc[v][r] += d0[r] * b.x + d1[r] * b.y + d2[r] * b.z;
        }
      }
    }
  }
  if (r0 >= (int)t.rows) return;
  const bool atomic = gridDim.y > 1, out_be = flags & DPIR_MV_OUT_BE;
#pragma unroll
  for (int v = 0; v < V; v++)
#pragma unroll
    for (int r = 0; r < RB; r++) {
      uint32_t s = acc[v][r];
#pragma unroll
      for (int off = 16; off > 0; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
      if (lane == 0 && v < (int)t.nv && r0 + r < (int)t.rows) {
        uint32_t* o = vecs[t.vec0 + v].out + t.out_off + r0 + r;
        if (atomic) atomicAdd(o, s);
        else *o = out_be ? bswap32(s) : s;
      }
    }
}

__global__ void k_dpir_bswap(uint32_t* __restrict__ dst, const uint32_t* __restrict__ src, size_t words) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < words) dst[i] = bswap32(src[i]);
}

// dst[i] = byte-swapped (sum over g < nparts of parts[g * stride + i]), wrapping: the partial responses of a sharded server's
// shards into the wire-order response
__global__ void k_dpir_sum_be(uint32_t* __restrict__ dst, const uint32_t* __restrict__ parts, size_t stride, int nparts, size_t words) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < words; i += (size_t)gridDim.x * blockDim.x) {
    uint32_t v = 0;
    for (int g = 0; g < nparts; g++) v += parts[(size_t)g * stride + i];
    dst[i] = bswap32(v);
  }
}

template <int V>
void launch_mv(const DpirMvTask* tasks, size_t ntasks, const DpirMvVec* vecs, size_t cols, int ksplit, int flags, cudaStream_t s) {
  constexpr int U = V >= 8 ? 2 : 4;
  const int smem = V * kMvChunk * (int)sizeof(uint4);
  if (smem > 48 * 1024) opt_in_smem(k_dpir_matvec_multi<V, U>, smem);
  const uint32_t kps = (uint32_t)((cols + ksplit - 1) / ksplit);
  ++g_kernel_launches;
  k_dpir_matvec_multi<V, U><<<dim3((unsigned)ntasks, (unsigned)ksplit), kMvThreads, smem, s>>>(tasks, vecs, (uint32_t)cols, kps, flags);
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

int dpir_mv_ksplit(size_t ntasks, size_t cols, int sm_count) {
  const size_t target = 2 * (size_t)sm_count;                     // two CTAs an SM fit (launch bounds, <= 64 KiB shared)
  if (ntasks == 0 || ntasks >= target) return 1;
  const size_t ks = std::min((target + ntasks - 1) / ntasks, (cols + kMvChunk - 1) / kMvChunk);   // at least one chunk a CTA
  return (int)std::max<size_t>(1, std::min<size_t>(ks, 65535));
}

void launch_dpir_matvec_multi(const DpirMvTask* tasks, size_t ntasks, const DpirMvVec* vecs, size_t cols, int vmax, int ksplit,
                              int flags, cudaStream_t s) {
  if (ntasks == 0 || cols == 0) return;
  if (ntasks > 0x7FFFFFFFull || cols > 0xFFFFFFFFull || ksplit < 1 || ksplit > 65535) throw Error(-2, "dpir: multi matvec grid too large");
  if (ksplit > 1 && (flags & DPIR_MV_OUT_BE)) throw Error(-2, "dpir: a split k range accumulates natively");
  if (vmax <= 1) launch_mv<1>(tasks, ntasks, vecs, cols, ksplit, flags, s);
  else if (vmax <= 2) launch_mv<2>(tasks, ntasks, vecs, cols, ksplit, flags, s);
  else if (vmax <= 4) launch_mv<4>(tasks, ntasks, vecs, cols, ksplit, flags, s);
  else if (vmax <= 8) launch_mv<8>(tasks, ntasks, vecs, cols, ksplit, flags, s);
  else if (vmax <= kDpirMvMaxVecs) launch_mv<16>(tasks, ntasks, vecs, cols, ksplit, flags, s);
  else throw Error(-2, "dpir: more vectors in a task than a pass holds");
}

void launch_dpir_bswap(uint32_t* dst, const uint32_t* src, size_t words, cudaStream_t s) {
  if (words == 0) return;
  ++g_kernel_launches;
  k_dpir_bswap<<<(unsigned)((words + 255) / 256), 256, 0, s>>>(dst, src, words);
}

void launch_dpir_sum_be(uint32_t* dst, const uint32_t* parts, size_t stride, size_t nparts, size_t words, cudaStream_t s) {
  if (words == 0) return;
  if (nparts > 0x7FFFFFFF) throw Error(-2, "dpir: too many partial responses");
  ++g_kernel_launches;
  k_dpir_sum_be<<<(unsigned)std::min<size_t>((words + 255) / 256, 132 * 16), 256, 0, s>>>(dst, parts, stride, (int)nparts, words);
}

}  // namespace b200pir
