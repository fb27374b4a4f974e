// DoublePIR's packed matrix x many vectors on the Hopper tensor cores (sm_90a): the database pass and the h_1 pass of answer()
// (doublepir.rs:246-350) for up to DTC_VECS = 64 vectors a matrix read.  The index maps are in dpir_tc_layout.cuh.
//
// CTA = 64 rows of one task x its (up to 64) vectors, 512 threads = four consumer warpgroups (row half x vector half), each with
// one m64n128k32 s32 accumulator (64 registers).  Per chunk of 32 packed words the CTA:
//   * copies the chunk's raw words of its 64 rows into shared memory with 4-byte cp.async (zero-filled past `cols` and past the
//     task's rows).  A row is `cols` words, so a row start is only 4-byte aligned in general (at m = 65 536 a row is 87 384
//     bytes: odd rows are 8- but not 16-byte aligned), which rules out 16-byte and bulk copies of row segments; a warp's 32
//     4-byte copies cover 128 consecutive bytes of one row, so the memory transactions are as wide as 16-byte copies would make;
//   * copies the chunk's query images (built once per pass by k_dpir_tc_image, 16-byte aligned) with 16-byte cp.async;
//   * unpacks the raw words into the three digit planes' two 8-bit limbs, as canonical no-swizzle A tiles (12 KiB, double
//     buffered), and runs three wgmma per warpgroup (one per digit plane).
// Copies run DTC_DIST chunks ahead through a ring of DTC_STAGES stages; two barriers a chunk order the copies, the unpacking and
// the MMAs (a stage is refilled only after every warpgroup's wgmma_wait has retired the MMAs that read it).  Partial sums of a
// split k range are added with atomicAdd into zeroed outputs (exact modulo 2^32; not with big-endian outputs).
#include "dpir_kernels.h"
#include "tc5_ptx.cuh"
#include "dpir_tc_layout.cuh"

namespace b200pir {
namespace {
using namespace tc5;

constexpr int DTC_THREADS = 512;
constexpr int DTC_STAGES = 5, DTC_DIST = DTC_STAGES - 2;
constexpr int DTC_RAW_BYTES = DTC_ROWS * DTC_KW * 4;                 // 8 KiB
constexpr int DTC_STAGE_BYTES = DTC_RAW_BYTES + 6 * DTC_B_TILE;     // + 24 KiB of query tiles [t][vh]
constexpr int DTC_A_BYTES = 6 * DTC_A_TILE;                         // 12 KiB of database tiles [t][rh]
constexpr int DTC_SMEM = DTC_STAGES * DTC_STAGE_BYTES + 2 * DTC_A_BYTES;
constexpr int DTC_IMG_THREADS = 256;

__device__ __forceinline__ uint32_t bswap32(uint32_t v) { return __byte_perm(v, 0, 0x0123); }
__device__ __forceinline__ void cp_async4(void* dst, const void* src, uint32_t src_bytes) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(smem_u32(dst)), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async16(void* dst, const void* src, uint32_t src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_u32(dst)), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
// generic-proxy shared-memory writes (cp.async, st.shared) made visible to the async proxy that wgmma reads through
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// one job's query image: thread (c, t, kh) writes its four 16-byte rows
__global__ void k_dpir_tc_image(const DpirTcImage* __restrict__ jobs, int flags) {
  const DpirTcImage J = jobs[blockIdx.y];
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;      // over chunks x 3 planes x 2 halves
  if (idx >= dtc_chunks(J.cols) * 6) return;
  const int kh = (int)(idx & 1), t = (int)((idx >> 1) % 3);
  const size_t c = idx / 6;
  uint32_t rows[4][4];
  dtc_img_rows(J.b, J.cols, flags & DPIR_MV_B_BE, c, t, kh, rows);
#pragma unroll
  for (int j = 0; j < 4; j++)
    *reinterpret_cast<uint4*>(J.img + dtc_img_off(c, t, kh, j)) = make_uint4(rows[j][0], rows[j][1], rows[j][2], rows[j][3]);
}

__global__ void __launch_bounds__(DTC_THREADS, 1)
k_dpir_matvec_tc(const DpirMvTask* __restrict__ tasks, const DpirMvVec* __restrict__ vecs, uint32_t cols, uint32_t chunks_per_split,
                 int flags) {
  extern __shared__ __align__(128) uint8_t sm[];
  const DpirMvTask T = tasks[blockIdx.x];
  const uint32_t nch = (cols + DTC_KW - 1) / DTC_KW;
  const uint32_t c0 = blockIdx.y * chunks_per_split, c1 = min(nch, c0 + chunks_per_split);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int rh = warp >> 3, vh = (warp >> 2) & 1, w = warp & 3;
  const bool live = 32 * rh < (int)T.rows && 32 * vh < (int)T.nv;      // warpgroup-uniform: this quarter has rows and vectors
  uint8_t* const a_buf = sm + DTC_STAGES * DTC_STAGE_BYTES;

  // this thread's copies: raw words idx = tid + 512 q (row idx / 32, word idx % 32); image pieces idx = tid + 512 q over
  // (vector idx / 24, piece idx % 24 = (t, kh, j))
  const uint8_t* img[3];
  int b_off[3];
  uint32_t img_ok[3];
#pragma unroll
  for (int q = 0; q < 3; q++) {
    const int idx = tid + DTC_THREADS * q, vl = idx / 24, p = idx % 24, j = p & 3, kh = (p >> 2) & 1, t = p >> 3;
    img_ok[q] = vl < (int)T.nv ? 16u : 0u;
    img[q] = reinterpret_cast<const uint8_t*>(vecs[T.vec0 + (vl < (int)T.nv ? vl : 0)].b) + dtc_img_off(0, t, kh, j);
    b_off[q] = DTC_RAW_BYTES + dtc_b_smem_off(vl, t, kh) + 16 * j;
  }
  auto issue = [&](uint32_t c) {
    uint8_t* st = sm + (c % DTC_STAGES) * DTC_STAGE_BYTES;
#pragma unroll
    for (int q = 0; q < 4; q++) {
      const int idx = tid + DTC_THREADS * q, r = idx >> 5;
      const uint32_t word = c * DTC_KW + (idx & 31);
      const bool ok = dtc_raw_ok(r, word, T.rows, cols);
      cp_async4(st + 4 * idx, ok ? T.a + (size_t)r * cols + word : T.a, ok ? 4u : 0u);
    }
#pragma unroll
    for (int q = 0; q < 3; q++) cp_async16(st + b_off[q], img[q] + (size_t)c * DTC_IMG_CHUNK, img_ok[q]);
  };

  uint32_t acc[64];
#pragma unroll
  for (int i = 0; i < 64; i++) acc[i] = 0;
#pragma unroll
  for (int d = 0; d < DTC_DIST; d++) {
    if (c0 + d < c1) issue(c0 + d);
    cp_async_commit();
  }
  const DtcUnpack U = dtc_unpack_thread(tid);
  for (uint32_t c = c0; c < c1; c++) {
    cp_async_wait<DTC_DIST - 1>();        // this thread's copies of chunk c have landed
    __syncthreads();                      // everyone's have; the MMAs of chunk c - 2 have retired (wgmma_wait<1> below)
    if (c + DTC_DIST < c1) issue(c + DTC_DIST);                    // into the stage chunk c - 2 used
    cp_async_commit();
    const uint8_t* st = sm + (c % DTC_STAGES) * DTC_STAGE_BYTES;
    uint8_t* ab = a_buf + ((c - c0) & 1) * DTC_A_BYTES;
    {
      const uint4 raw = *reinterpret_cast<const uint4*>(st + (U.row * DTC_KW + 4 * U.kq) * 4);
      const uint32_t wv[4] = {raw.x, raw.y, raw.z, raw.w};
#pragma unroll
      for (int t = 0; t < 3; t++)
#pragma unroll
        for (int i = 0; i < 2; i++) *reinterpret_cast<uint32_t*>(ab + dtc_a_smem_off(U.row, t, i, U.kq)) = dtc_limb4(wv, t, i);
    }
    fence_proxy_async();
    __syncthreads();                      // the chunk's A tiles are complete
    // every warpgroup multiplies (an empty quarter multiplies zeros): a branch around wgmma makes ptxas serialise them all
    const uint32_t a_base = smem_u32(ab), b_base = smem_u32(st + DTC_RAW_BYTES);
    wgmma_fence();
#pragma unroll
    for (int t = 0; t < 3; t++)
      wgmma_m64n128k32_u8(acc, tc5_smem_desc(a_base + dtc_a_tile(t, rh)), tc5_smem_desc(b_base + dtc_b_tile(t, vh)));
    wgmma_commit();
    wgmma_wait<1>();
  }
  cp_async_wait<0>();
  wgmma_wait<0>();
  wgmma_fence_operands(acc);
  if (!live) return;
  const bool atomic = gridDim.y > 1, out_be = flags & DPIR_MV_OUT_BE;
#pragma unroll
  for (int ii = 0; ii < 16; ii++)
#pragma unroll
    for (int h = 0; h < 2; h++) {
      uint32_t s = dtc_lane_partial(acc[4 * ii + 2 * h], acc[4 * ii + 2 * h + 1], lane);
      s += __shfl_xor_sync(0xffffffffu, s, 1);            // the other byte pair
      s += __shfl_xor_sync(0xffffffffu, s, 4);            // the other limb
      const int r = 32 * rh + dtc_frag_row(w, lane, h), v = 32 * vh + dtc_frag_vec(lane, ii);
      if (dtc_frag_stores(lane, ii, h) && r < (int)T.rows && v < (int)T.nv) {
        uint32_t* o = vecs[T.vec0 + v].out + T.out_off + r;
        if (atomic) atomicAdd(o, s);
        else *o = out_be ? bswap32(s) : s;
      }
    }
}

}  // namespace

// Measured on an H100 (DESIGN §4.5) at l = 1 821 and 14 564: the tensor-core pass takes about the same time for 1 to 64 vectors
// (0.25 / 1.82 ms), k_dpir_matvec_multi grows with V and is faster up to V = 8 (0.18 / 1.33 ms) and slower from its V = 16
// instantiation on (0.41 / 2.37 ms), which also serves 9 to 15 vectors.  Both matrices were measured at the same widths, so the
// rule does not depend on the rows.
bool dpir_use_tc(size_t nv, size_t rows) {
  (void)rows;
  return nv > 8;
}

int dpir_tc_ksplit(size_t ntasks, size_t cols, int sm_count) {
  const size_t target = 4 * (size_t)sm_count;                       // one CTA an SM: about four waves
  if (ntasks == 0 || ntasks >= target) return 1;
  const size_t ks = std::min((target + ntasks - 1) / ntasks, (size_t)dtc_chunks(cols));
  return (int)std::max<size_t>(1, std::min<size_t>(ks, 65535));
}

void launch_dpir_tc_image(const DpirTcImage* jobs, size_t njobs, size_t max_cols, int flags, cudaStream_t s) {
  if (njobs == 0 || max_cols == 0) return;
  const size_t threads = dtc_chunks(max_cols) * 6;
  for (size_t j0 = 0; j0 < njobs; j0 += 65535) {          // gridDim.y is capped at 65535
    ++g_kernel_launches;
    k_dpir_tc_image<<<dim3((unsigned)((threads + DTC_IMG_THREADS - 1) / DTC_IMG_THREADS), (unsigned)std::min<size_t>(njobs - j0, 65535)),
                      DTC_IMG_THREADS, 0, s>>>(jobs + j0, flags);
  }
}

void launch_dpir_matvec_tc(const DpirMvTask* tasks, size_t ntasks, const DpirMvVec* vecs, size_t cols, int ksplit, int flags,
                           cudaStream_t s) {
  if (ntasks == 0 || cols == 0) return;
  if (ntasks > 0x7FFFFFFFull || cols > 0xFFFFFFFFull || ksplit < 1 || ksplit > 65535) throw Error(-2, "dpir: tensor-core pass grid too large");
  if (ksplit > 1 && (flags & DPIR_MV_OUT_BE)) throw Error(-2, "dpir: a split k range accumulates natively");
  opt_in_smem(k_dpir_matvec_tc, DTC_SMEM);
  const uint32_t nch = (uint32_t)dtc_chunks(cols), cps = (nch + ksplit - 1) / ksplit;
  ++g_kernel_launches;
  k_dpir_matvec_tc<<<dim3((unsigned)ntasks, (unsigned)ksplit), DTC_THREADS, DTC_SMEM, s>>>(tasks, vecs, (uint32_t)cols, cps, flags);
}

}  // namespace b200pir
