// DoublePIR entry updates: Db::_set (lib/doublepir/src/database/database.rs:264-266, a todo!() in the reference) on a database
// loaded into HBM, and setup()'s outputs (doublepir.rs:76-108) patched to match instead of recomputed.  setup() is linear in the
// database and every piece of state it derives is local to a layout row, so a patch costs in proportion to the changed
// elements (DESIGN §4.5, "Entry updates"):
//   store  : element (r, c) is field c % 3 of squished word (r, c / 3) and holds the element itself; delta_rc = new - old
//   h_1    : dh_1[r, :] = sum_c delta_rc A_1[c, :] (mod 2^32), the A_1 rows derived here from SEED_A1
//   digits : h_1[r, i] is stored as delta base-p digits at rows i delta + f + n delta (r % x), column r / x of h1_squished;
//            old + dh_1 is split again, and the digit differences are the columns of D
//   hint   : dh_2[block b] = D_b A_2[changed rows of b, :], on the setup GEMM (dpir_gemm.cu), then added into h_2
// Every patch of a squished field is a wrapping add of (new - old) << 10 k.  Fields stay in [0, p) (p <= 2^10), so the adds
// never carry into a neighbour and commute: the elements of one word, or the h_1 columns of one word, need no ordering.
#include "dpir_aes.cuh"

namespace b200pir {

namespace {

constexpr int kBlock = 256;

__global__ void __launch_bounds__(kBlock) k_dpir_upd_store(uint32_t* __restrict__ store, uint64_t dcols, const DpirUpdElem* __restrict__ el,
                                                           uint32_t n_el, int32_t* __restrict__ delta) {
  const uint32_t i = blockIdx.x * kBlock + threadIdx.x;
  if (i >= n_el) return;
  const DpirUpdElem e = el[i];
  uint32_t* w = store + e.r * dcols + e.c / 3;
  const uint32_t sh = 10 * (uint32_t)(e.c % 3);
  // only this thread changes this field; the adds of the word's other fields never reach it
  const uint32_t old = (*w >> sh) & 1023u, nw = (old & ~e.mask) | e.val;
  const int32_t d = (int32_t)nw - (int32_t)old;
  if (d) atomicAdd(w, (uint32_t)d << sh);
  delta[i] = d;
}

// One CTA per changed row: the (element, 16-byte block) pairs of its A_1 rows spread over the threads, products summed in
// shared memory.  A_1[c, :] is words [c n, c n + n) of derive(m x n), which starts inside a block when n % 4 != 0.
__global__ void __launch_bounds__(kBlock) k_dpir_upd_dh1(uint32_t* __restrict__ dh1, const DpirUpdRow* __restrict__ rows,
                                                         const DpirUpdElem* __restrict__ el, const int32_t* __restrict__ delta,
                                                         uint64_t n, const __grid_constant__ DpirAesKey key) {
  __shared__ uint32_t te[4][256];
  __shared__ uint32_t sb[256];
  extern __shared__ uint32_t acc[];
  dpir_aes_tables(te, sb, key);
  for (uint64_t j = threadIdx.x; j < n; j += kBlock) acc[j] = 0;
  __syncthreads();
  const DpirUpdRow R = rows[blockIdx.x];
  const uint64_t nblk = (n + 3) / 4 + 1;               // the most blocks n consecutive words touch
  for (uint64_t t = threadIdx.x; t < (uint64_t)R.ne * nblk; t += kBlock) {
    const uint64_t k = t / nblk;
    const int32_t d = delta[R.e0 + k];
    if (!d) continue;
    const uint64_t w0 = el[R.e0 + k].c * n, b = w0 / 4 + (t - k * nblk);
    if (4 * b >= w0 + n) continue;
    const uint4 o = dpir_aes_block(te, sb, key, b);
    const uint32_t w[4] = {o.x, o.y, o.z, o.w};
#pragma unroll
    for (int u = 0; u < 4; u++)
      if (4 * b + u >= w0 && 4 * b + u < w0 + n) atomicAdd(&acc[4 * b + u - w0], (uint32_t)d * w[u]);
  }
  __syncthreads();
  for (uint64_t j = threadIdx.x; j < n; j += kBlock) dh1[(uint64_t)blockIdx.x * n + j] = acc[j];
}

// One thread per (changed row k, column i of h_1).  The stored digits are exactly the base-p split of the old value (p^delta >=
// 2^32), so the old digits are recomputed from it rather than read twice.
__global__ void __launch_bounds__(kBlock) k_dpir_upd_digits(uint32_t* __restrict__ h1sq, uint64_t c1, int32_t* __restrict__ D,
                                                            const DpirUpdRow* __restrict__ rows, uint32_t nrows,
                                                            const uint32_t* __restrict__ dh1, uint64_t n, uint32_t p, uint32_t delta,
                                                            uint64_t x) {
  const uint64_t idx = (uint64_t)blockIdx.x * kBlock + threadIdx.x;
  if (idx >= (uint64_t)nrows * n) return;
  const uint64_t k = idx / n, i = idx - k * n;
  const DpirUpdRow R = rows[k];
  const uint64_t C = R.r / x, r0 = i * delta + n * delta * (R.r % x);     // h1_squished row of digit 0
  uint32_t* col = h1sq + C / 3;
  const uint32_t sh = 10 * (uint32_t)(C % 3);
  uint64_t old = 0, pw = 1;
  for (uint32_t f = 0; f < delta; f++) {
    old += (uint64_t)((col[(r0 + f) * c1] >> sh) & 1023u) * pw;
    pw *= p;
  }
  uint32_t ov = (uint32_t)old, nv = ov + dh1[idx];
  for (uint32_t f = 0; f < delta; f++) {
    const int32_t dd = (int32_t)(nv % p) - (int32_t)(ov % p);
    if (dd) atomicAdd(&col[(r0 + f) * c1], (uint32_t)dd << sh);
    D[R.doff + (i * delta + f) * R.kb + R.dcol] = dd;
    ov /= p;
    nv /= p;
  }
}

__global__ void k_dpir_upd_gather_a2(uint32_t* __restrict__ a2g, const uint32_t* __restrict__ a2t, uint64_t lx3,
                                     const DpirUpdRow* __restrict__ rows, uint32_t nrows, uint64_t n, uint64_t x) {
  const uint64_t idx = (uint64_t)blockIdx.x * kBlock + threadIdx.x;
  if (idx >= (uint64_t)nrows * n) return;
  const uint64_t k = idx / n, j = idx - k * n;
  a2g[idx] = a2t[j * lx3 + rows[k].r / x];
}

__global__ void k_dpir_upd_add(uint32_t* __restrict__ dst, const uint32_t* __restrict__ src, size_t words) {
  const size_t i = (size_t)blockIdx.x * kBlock + threadIdx.x;
  if (i < words) dst[i] += src[i];
}

unsigned blocks_for(uint64_t items) { return (unsigned)((items + kBlock - 1) / kBlock); }

}  // namespace

void launch_dpir_upd_store(uint32_t* store, uint64_t dcols, const DpirUpdElem* el, uint32_t n_el, int32_t* delta, cudaStream_t s) {
  ++g_kernel_launches;
  k_dpir_upd_store<<<blocks_for(n_el), kBlock, 0, s>>>(store, dcols, el, n_el, delta);
}
void launch_dpir_upd_dh1(uint32_t* dh1, const DpirUpdRow* rows, uint32_t nrows, const DpirUpdElem* el, const int32_t* delta, uint64_t n,
                         const DpirAesKey& key, cudaStream_t s) {
  const int smem = (int)(n * 4);
  if (smem > 48 * 1024) opt_in_smem(k_dpir_upd_dh1, smem);
  ++g_kernel_launches;
  k_dpir_upd_dh1<<<nrows, kBlock, smem, s>>>(dh1, rows, el, delta, n, key);
}
void launch_dpir_upd_digits(uint32_t* h1sq, uint64_t c1, int32_t* D, const DpirUpdRow* rows, uint32_t nrows, const uint32_t* dh1,
                            uint64_t n, uint32_t p, uint32_t delta, uint64_t x, cudaStream_t s) {
  ++g_kernel_launches;
  k_dpir_upd_digits<<<blocks_for((uint64_t)nrows * n), kBlock, 0, s>>>(h1sq, c1, D, rows, nrows, dh1, n, p, delta, x);
}
void launch_dpir_upd_gather_a2(uint32_t* a2g, const uint32_t* a2t, uint64_t lx3, const DpirUpdRow* rows, uint32_t nrows, uint64_t n,
                               uint64_t x, cudaStream_t s) {
  ++g_kernel_launches;
  k_dpir_upd_gather_a2<<<blocks_for((uint64_t)nrows * n), kBlock, 0, s>>>(a2g, a2t, lx3, rows, nrows, n, x);
}
void launch_dpir_upd_add(uint32_t* dst, const uint32_t* src, size_t words, cudaStream_t s) {
  ++g_kernel_launches;
  k_dpir_upd_add<<<blocks_for(words), kBlock, 0, s>>>(dst, src, words);
}

}  // namespace b200pir
