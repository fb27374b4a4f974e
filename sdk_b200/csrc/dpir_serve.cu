// DoublePIR's packed matrix x many vectors (sm_90a): the database pass, the h_1 pass and the a_1' * q_2 products of
// answer() (doublepir.rs:246-350) for every request of a call, one matrix read per pass of up to kDpirMvMaxVecs vectors.
#include "kernels.h"

namespace b200pir {
namespace {

constexpr int kMvThreads = 256;
constexpr int kMvRowsPerWarp = kDpirMvRows / (kMvThreads / 32);
constexpr int kMvChunk = 256;                 // k (packed columns) staged per round: V x 256 x 16 bytes of shared memory

__device__ __forceinline__ uint32_t bswap32(uint32_t v) { return __byte_perm(v, 0, 0x0123); }

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

}  // namespace b200pir
