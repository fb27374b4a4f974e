// First dimension on the Hopper tensor cores (wgmma, s32 accumulators in registers) — database format 2.
//
// The arithmetic is the one of the mma.sync path (imma_kernels.cu): 28-bit residues as four 7-bit limbs, exact s32
// accumulation, recombination with powers of 2^7 and one Barrett reduction per output word.
//
// multiply_reg_by_database (lib/spiral-rs/src/server.rs:155-221) for one NTT coordinate z and modulus n is the integer
// GEMM  C[ii][(query,row)] = sum_j A[ii][j] * B[j][(query,row)] mod q_n.  Here both operands carry their limb index as
// part of the GEMM's M / N index, so one 128 x 128 tile produces all 16 limb-pair products separately:
//
//     M index = 4 * row_local + l      (32 database rows x 4 limbs  = 128: two wgmma M = 64 halves)
//     N index = 4 * col       + m      (32 columns = 16 queries x 2 ciphertext rows, x 4 limbs = 128 = wgmma N)
//     K       = 32 values of j per instruction (u8 x u8), dim0 / 32 instructions per tile and warpgroup
//     D[M][N] = sum_j a_l(ii, j) * b_m(j, col)  < dim0 * 2^14 <= 2^24        (exact in s32)
//
// The epilogue (tc5_layout.cuh) works on the accumulator fragment in registers: it folds pairs of m-limbs with a shift,
// weights the sum with 2^{7(l+m)} mod q in two wide multiply-adds, reduce-scatters over the eight lanes that hold the limbs
// of one output (three shuffle rounds) and finishes with one 32-bit Barrett per stored word.
//
// Operand images.  Both operands are stored in global memory as exact images of the shared-memory tiles wgmma reads
// (canonical K-major, no swizzle: 8-row x 16-byte core matrices, LBO = 128 B between the two K halves, SBO = 256 B
// between 8-row groups; byte (midx, k) of a tile lives at (midx>>3)*256 + (k>>4)*128 + (midx&7)*16 + (k&15)), so a tile
// moves with ONE 1-D bulk copy (cp.async.bulk ... mbarrier::complete_tx::bytes) and needs no tensor map:
//     dbT[slice][n][z][mt][ks][4096 B]      (mt: 32 rows, ks: 32 values of j)     == 8 bytes per database word, as before
//     qT [n][z][ks][4096 B]                 (16 queries)
// One persistent CTA per SM walks the (n, z) pairs; warpgroups 0 and 1 = consumers (M rows 0..63 and 64..127 of every tile),
// warp 8 = bulk-copy producer.  Pipelines: A ring (full/empty mbarriers), double-buffered B operand (bfull/bempty).  The ring
// keeps the copies in flight while the consumers run the epilogue of a tile.
#include "kernels.h"
#include "tc5_ptx.cuh"

namespace b200pir {

namespace {

constexpr int TC5_SMEM_BUDGET = 227 * 1024 - 1024;      // dynamic shared memory of the CTA minus barriers / alignment slack
constexpr int TC5_THREADS = 2 * 128 + 32;              // two consumer warpgroups, producer warp

using namespace tc5;

// ---- operand images ---------------------------------------------------------------------------------------------------
// format 0 slice (uint4 [row][jp][z]) -> tile images.  CTA = (z, mt, ks); thread = (row_local, group of 4 values of j).
__global__ void __launch_bounds__(256)
k_db_to_tc5(Tc5Geom T, const uint4* __restrict__ db0_slice, uint8_t* __restrict__ dbt, int slice) {
  const int z = blockIdx.x, mt = blockIdx.y, ks = blockIdx.z;
  const Tc5DbThread t = tc5_db_thread(threadIdx.x, mt, ks);
  const int half = T.dim0 >> 1;
  uint32_t res[2][4];
#pragma unroll
  for (int p = 0; p < 2; p++) {
    const int jp = t.jp0 + p;
    uint4 w = make_uint4(0, 0, 0, 0);
    if (t.ii < T.rows && jp < half) w = db0_slice[((size_t)t.ii * half + jp) * POLY + z];
    res[0][2 * p] = w.x; res[1][2 * p] = w.y; res[0][2 * p + 1] = w.z; res[1][2 * p + 1] = w.w;
  }
#pragma unroll
  for (int n = 0; n < 2; n++) tc5_db_store(dbt + tc5_db_tile(T, slice, n, z, mt, ks) * TC5_TILE, t, res[n]);
}

// one item polynomial (2048 packed words lo|hi<<32) into the tile images (byte writes)
__global__ void k_db_upsert_tc5(Tc5Geom T, uint8_t* dbt, int slice, int il, int j, const uint64_t* poly) {
  const int z = blockIdx.x * blockDim.x + threadIdx.x;
  if (z >= POLY) return;
  const int mt = il >> 5, row_local = il & 31, ks = j >> 5, k = j & 31;
  const uint64_t w = poly[z];
#pragma unroll
  for (int n = 0; n < 2; n++) {
    const uint32_t r = n ? (uint32_t)(w >> 32) : (uint32_t)w;
    uint8_t* tile = dbt + tc5_db_tile(T, slice, n, z, mt, ks) * TC5_TILE;
#pragma unroll
    for (int l = 0; l < 4; l++) tile[tc5_tile_off(tc5_m_index(row_local, l), k)] = (uint8_t)((r >> (7 * l)) & 127u);
  }
}

// expanded queries (uint4 [j][z] per query, q_stride apart) -> qT.  CTA = (pair of z, ks): every 32-byte sector it reads is
// fully used; the four 4 KiB tiles (2 z x 2 n) are assembled in shared memory and written out contiguously.
__global__ void __launch_bounds__(256)
k_query_to_tc5(Tc5Geom T, const uint4* __restrict__ q_dev, size_t q_stride, int nq, uint8_t* __restrict__ qt) {
  __shared__ __align__(16) uint8_t img[2][2][TC5_TILE];          // [z parity][n]
  const int z0 = blockIdx.x * 2, ks = blockIdx.y;
  for (int i = threadIdx.x; i < 2 * 2 * TC5_TILE / 16; i += blockDim.x) reinterpret_cast<uint4*>(&img[0][0][0])[i] = make_uint4(0, 0, 0, 0);
  __syncthreads();
  // 16 queries x 32 values of j x 2 z = 1024 cells, 4 per thread; consecutive threads take consecutive z, then j, then query
  for (int cell = threadIdx.x; cell < 16 * 32 * 2; cell += blockDim.x) {
    const Tc5QueryCell qc = tc5_query_cell(cell);
    const int j = ks * 32 + qc.k;
    if (qc.q < nq && j < T.dim0) {
      const uint4 w = q_dev[(size_t)qc.q * q_stride + (size_t)j * POLY + z0 + qc.zp];
#pragma unroll
      for (int r = 0; r < 2; r++)
#pragma unroll
        for (int n = 0; n < 2; n++) tc5_query_store(img[qc.zp][n], qc.q, r, qc.k, r ? (n ? w.w : w.z) : (n ? w.y : w.x));
    }
  }
  __syncthreads();
#pragma unroll
  for (int zp = 0; zp < 2; zp++)
#pragma unroll
    for (int n = 0; n < 2; n++) {
      uint4* dst = reinterpret_cast<uint4*>(qt + tc5_q_tile(T, n, z0 + zp, ks) * TC5_TILE);
      dst[threadIdx.x] = reinterpret_cast<const uint4*>(&img[zp][n][0])[threadIdx.x];
    }
}

// The same images straight from the expansion workspace (reorient_reg_ciphertexts, util.rs:323-355, fused with the re-tiling):
// v = ntt32 [query][slot][ct row][n][z] (v_stride words per query), first-dimension ciphertext j = slot idx_factor * j.
// CTA = (8 consecutive z, ks): 2048 polynomial segments of 8 words (one 32-byte sector each), 8 per thread; the sixteen 4 KiB
// tiles (8 z x 2 n) are assembled in shared memory and written out contiguously.
__global__ void __launch_bounds__(256)
k_reorient_to_tc5(Tc5Geom T, const uint32_t* __restrict__ v, size_t v_stride, int idx_factor, int nq, uint8_t* __restrict__ qt) {
  extern __shared__ __align__(16) uint8_t rimg[];                    // [8 z][2 n][TC5_TILE]
  const int z0 = blockIdx.x * 8, ks = blockIdx.y;
  for (int i = threadIdx.x; i < 16 * TC5_TILE / 16; i += 256) reinterpret_cast<uint4*>(rimg)[i] = make_uint4(0, 0, 0, 0);
  __syncthreads();
  for (int seg = threadIdx.x; seg < 16 * 32 * 4; seg += 256) {
    const int n = seg & 1, r = (seg >> 1) & 1, k = (seg >> 2) & 31, q = seg >> 7;
    const int j = ks * 32 + k;
    if (q >= nq || j >= T.dim0) continue;
    const uint32_t* src = v + (size_t)q * v_stride + ((size_t)idx_factor * j * 4 + r * 2 + n) * 2048 + z0;
    const uint4 a = __ldg(reinterpret_cast<const uint4*>(src)), b = __ldg(reinterpret_cast<const uint4*>(src) + 1);
    const uint32_t w[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
#pragma unroll
    for (int zz = 0; zz < 8; zz++) tc5_query_store(rimg + ((size_t)zz * 2 + n) * TC5_TILE, q, r, k, w[zz]);
  }
  __syncthreads();
#pragma unroll
  for (int zz = 0; zz < 8; zz++)
#pragma unroll
    for (int n = 0; n < 2; n++) {
      uint4* dst = reinterpret_cast<uint4*>(qt + tc5_q_tile(T, n, z0 + zz, ks) * TC5_TILE);
      dst[threadIdx.x] = reinterpret_cast<const uint4*>(rimg + ((size_t)zz * 2 + n) * TC5_TILE)[threadIdx.x];
    }
}

// ---- the multiply -----------------------------------------------------------------------------------------------------
constexpr int TC5_MAX_STAGES = 24;
struct Tc5Smem {
  uint64_t full[TC5_MAX_STAGES], empty[TC5_MAX_STAGES];
  uint64_t bfull[2], bempty[2];
};
// ring stages that fit beside the query operand: the bytes in flight per SM bound the HBM bandwidth the kernel can pull
// (latency x bandwidth = about 50 KiB per SM at 3.35 TB/s and 2 us), and a stage is out of flight while its MMAs run
__host__ __device__ inline int tc5_ring_stages(int ks, int ksps, int bbufs) {
  const int n = (TC5_SMEM_BUDGET - bbufs * ks * TC5_TILE) / (ksps * TC5_TILE);
  return n > TC5_MAX_STAGES ? TC5_MAX_STAGES : n;
}

// out_zm[query][slice][n][z][row][ct_row] (u32), the format of k_multiply_imma
// KSPS = k-steps (4 KiB tiles) per ring stage.  BBUFS: buffers of the query operand (2 = the next (n, z) pair's operand loads
// under the current pair's MMAs; 1 = its 64 KiB go to the database ring instead, at the price of a reload bubble per pair).
template <int KSPS, int BBUFS>
__global__ void __launch_bounds__(TC5_THREADS, 1)
k_multiply_tc5(DevParams P, Tc5Geom T, const uint8_t* __restrict__ dbt, const uint8_t* __restrict__ qt,
               uint32_t* __restrict__ out_zm, size_t out_stride, int nq, int slice_begin, int slice_count,
               const uint32_t* __restrict__ tile_mask /* [slice][mt]: bit ks = the 32-row x 32-j tile holds a present item */) {
  constexpr int TC5_STAGE_BYTES = KSPS * TC5_TILE;
  const int TC5_STAGES = tc5_ring_stages(T.ks, KSPS, BBUFS);
  extern __shared__ __align__(1024) uint8_t tc5_smem[];
  uint8_t* smem_b = tc5_smem;                                         // [BBUFS][ks][4096]
  uint8_t* smem_a = smem_b + (size_t)BBUFS * T.ks * TC5_TILE;         // [STAGES][KSPS x 4 KiB]
  Tc5Smem* S = reinterpret_cast<Tc5Smem*>(smem_a + (size_t)TC5_STAGES * TC5_STAGE_BYTES);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int stages_per_tile = (T.ks + KSPS - 1) / KSPS;
  const int tiles_per_item = slice_count * T.mt;
  const int n_items = 2 * POLY;
  const uint32_t b_bytes = (uint32_t)T.ks * TC5_TILE;

  if (threadIdx.x == 0) {
    for (int s = 0; s < TC5_STAGES; s++) { mbar_init(&S->full[s], 1); mbar_init(&S->empty[s], 2); }
    for (int b = 0; b < 2; b++) { mbar_init(&S->bfull[b], 1); mbar_init(&S->bempty[b], 2); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  // The producer loop runs CONVERGED (all 32 lanes, warp-uniform values); only the copies themselves are issued by one
  // elected lane, so that ptxas does not serialise every operand of the bulk copies per thread.
  if (warp == 8) {
    // ===== producer =====
    int stage = 0; uint32_t sphase = 0;
    int it = 0;
    for (int item = blockIdx.x; item < n_items; item += gridDim.x, it++) {
      const int n = item & 1, z = item >> 1, bb = it % BBUFS;
      mbar_wait(&S->bempty[bb], ((it / BBUFS) & 1) ^ 1);
      if (elect_one()) {
        mbar_expect_tx(&S->bfull[bb], b_bytes);
        bulk_g2s(smem_b + (size_t)bb * b_bytes, qt + tc5_q_tile(T, n, z, 0) * TC5_TILE, b_bytes, &S->bfull[bb]);
      }
      __syncwarp();
      for (int sl = 0; sl < slice_count; sl++)
        for (int mt = 0; mt < T.mt; mt++) {
          const uint8_t* src = dbt + tc5_db_tile(T, slice_begin + sl, n, z, mt, 0) * TC5_TILE;
          // lib/server's sparse database (db/sparse_db.rs, compute/dot_product.rs:35): tiles without a present item are neither
          // fetched nor multiplied (they are zero: the sums are unchanged); a stage without any such tile takes no ring slot
          const uint32_t mask = __ldg(tile_mask + (size_t)(slice_begin + sl) * T.mt + mt);
          for (int st = 0; st < stages_per_tile; st++) {
            const int ks_here = min(KSPS, T.ks - st * KSPS);
            const uint32_t full_m = ks_here == 32 ? 0xffffffffu : ((1u << ks_here) - 1u);
            const uint32_t km = (mask >> (st * KSPS)) & full_m;
            if (km == 0) continue;
            mbar_wait(&S->empty[stage], sphase ^ 1);
            if (elect_one()) {
              uint8_t* dst = smem_a + (size_t)stage * TC5_STAGE_BYTES;
              const uint8_t* from = src + (size_t)st * TC5_STAGE_BYTES;
              mbar_expect_tx(&S->full[stage], (uint32_t)__popc(km) * TC5_TILE);
              if (km == full_m) bulk_g2s(dst, from, (uint32_t)ks_here * TC5_TILE, &S->full[stage]);
              else
                for (int kk = 0; kk < ks_here; kk++)
                  if ((km >> kk) & 1u) bulk_g2s(dst + (size_t)kk * TC5_TILE, from + (size_t)kk * TC5_TILE, TC5_TILE, &S->full[stage]);
            }
            __syncwarp();
            if (++stage == TC5_STAGES) { stage = 0; sphase ^= 1; }
          }
        }
    }
  } else if (warp < 8) {
    // ===== consumers: warpgroup wg owns M rows [64 wg, 64 wg + 64) of every tile =====
    const int wg = warp >> 2, w = warp & 3;
    const bool leader = (threadIdx.x & 127) == 0;                     // arrives on the ring barriers for its warpgroup
    int stage = 0; uint32_t sphase = 0;
    int it = 0;
    for (int item = blockIdx.x; item < n_items; item += gridDim.x, it++) {
      const int n = item & 1, z = item >> 1, bb = it % BBUFS;
      const uint32_t q = n ? P.q[1] : P.q[0];
      const Tc5Weights W = tc5_lane_weights(lane, q);
      mbar_wait(&S->bfull[bb], (it / BBUFS) & 1);
      const uint32_t b_addr = smem_u32(smem_b + (size_t)bb * b_bytes);
      for (int t = 0, slice = slice_begin, mt = 0; t < tiles_per_item; t++, mt++) {
        if (mt == T.mt) { mt = 0; slice++; }
        const uint32_t mask = __ldg(tile_mask + (size_t)slice * T.mt + mt);
        uint32_t acc[64];
#pragma unroll
        for (int c = 0; c < 64; c++) acc[c] = 0;
        int prev = -1;                                                // ring stage whose MMAs may still be in flight
        for (int st = 0; st < stages_per_tile; st++) {
          const int ks_here = min(KSPS, T.ks - st * KSPS);
          const uint32_t km = (mask >> (st * KSPS)) & (ks_here == 32 ? 0xffffffffu : ((1u << ks_here) - 1u));
          if (km == 0) continue;                                      // nothing fetched for this stage (see the producer)
          mbar_wait(&S->full[stage], sphase);
          const uint32_t a_addr = smem_u32(smem_a + (size_t)stage * TC5_STAGE_BYTES) + wg * (TC5_TILE / 2);
          wgmma_fence();
#pragma unroll
          for (int kk = 0; kk < KSPS; kk++)
            if ((km >> kk) & 1u)
              wgmma_m64n128k32_u8(acc, tc5_smem_desc(a_addr + kk * TC5_TILE), tc5_smem_desc(b_addr + (st * KSPS + kk) * TC5_TILE));
          wgmma_commit();
          wgmma_wait<1>();                                            // the previous stage's MMAs have completed: release it
          if (prev >= 0 && leader) mbar_arrive(&S->empty[prev]);
          prev = stage;
          if (++stage == TC5_STAGES) { stage = 0; sphase ^= 1; }
        }
        wgmma_wait<0>();
        wgmma_fence_operands(acc);
        if (prev >= 0 && leader) mbar_arrive(&S->empty[prev]);
        // epilogue: 32 weighted partials (index 2 i + h), three reduce-scatter rounds, four stored words per thread
        uint64_t p32[32], s16[16], k16[16], s8[8], k8[8], s4[4], k4[4];
#pragma unroll
        for (int i = 0; i < 16; i++)
#pragma unroll
          for (int h = 0; h < 2; h++) p32[2 * i + h] = tc5_lane_partial(acc[4 * i + 2 * h], acc[4 * i + 2 * h + 1], W.w, W.wp);
        tc5_rs_split<32>((lane >> tc5_rs_lane_bit(0)) & 1, p32, s16, k16);
#pragma unroll
        for (int r = 0; r < 16; r++) k16[r] += shfl_xor_u64(s16[r], 1 << tc5_rs_lane_bit(0));
        tc5_rs_split<16>((lane >> tc5_rs_lane_bit(1)) & 1, k16, s8, k8);
#pragma unroll
        for (int r = 0; r < 8; r++) k8[r] += shfl_xor_u64(s8[r], 1 << tc5_rs_lane_bit(1));
        tc5_rs_split<8>((lane >> tc5_rs_lane_bit(2)) & 1, k8, s4, k4);
#pragma unroll
        for (int r = 0; r < 4; r++) k4[r] += shfl_xor_u64(s4[r], 1 << tc5_rs_lane_bit(2));
#pragma unroll
        for (int f = 0; f < 4; f++) {
          const int qi = tc5_frag_query(lane, f), ii = mt * 32 + tc5_frag_row(wg, w, lane, f & 1);
          if (qi < nq && ii < T.rows)
            out_zm[(size_t)qi * out_stride + ((((size_t)slice * 2 + n) * POLY + z) * T.rows + ii) * 2 + tc5_frag_ctrow(lane)] =
                tc5_barrett57(k4[f], W.mu, q);
        }
      }
      if (leader) mbar_arrive(&S->bempty[bb]);                        // every MMA of this warpgroup reading the B buffer has completed
    }
  }
}

}  // namespace

size_t tc5_db_bytes(const Tc5Geom& T, int slices) { return (size_t)slices * 2 * POLY * T.mt * T.ks * TC5_TILE; }
size_t tc5_query_bytes(const Tc5Geom& T) { return (size_t)2 * POLY * T.ks * TC5_TILE; }
static size_t tc5_smem_bytes(const Tc5Geom& T, int ksps, int bbufs) {
  return (size_t)bbufs * T.ks * TC5_TILE + (size_t)tc5_ring_stages(T.ks, ksps, bbufs) * ksps * TC5_TILE + sizeof(Tc5Smem) + 16;
}
// at least two ring stages beside a single-buffered query operand
bool tc5_supported(const Tc5Geom& T) { return T.dim0 % 2 == 0 && tc5_ring_stages(T.ks, 4, 1) >= 2; }

void launch_db_to_tc5(const Tc5Geom& T, const uint4* db0_slice, uint8_t* dbt, int slice, cudaStream_t s) {
  ++g_kernel_launches;
  k_db_to_tc5<<<dim3(POLY, T.mt, T.ks), 256, 0, s>>>(T, db0_slice, dbt, slice);
}
void launch_db_upsert_tc5(const Tc5Geom& T, uint8_t* dbt, int slice, int il, int j, const uint64_t* poly, cudaStream_t s) {
  ++g_kernel_launches;
  k_db_upsert_tc5<<<POLY / 256, 256, 0, s>>>(T, dbt, slice, il, j, poly);
}
void launch_query_to_tc5(const Tc5Geom& T, const uint4* q_dev, size_t q_stride, int nq, uint8_t* qt, cudaStream_t s) {
  if (nq < 1 || nq > 16) throw Error(-2, "wgmma multiply: 1..16 queries per pass");
  ++g_kernel_launches;
  k_query_to_tc5<<<dim3(POLY / 2, T.ks), 256, 0, s>>>(T, q_dev, q_stride, nq, qt);
}
void launch_reorient_to_tc5(const Tc5Geom& T, const uint32_t* v, size_t v_stride, int idx_factor, int nq, uint8_t* qt, cudaStream_t s) {
  if (nq < 1 || nq > 16) throw Error(-2, "wgmma multiply: 1..16 queries per pass");
  ++g_kernel_launches;
  opt_in_smem(k_reorient_to_tc5, 16 * TC5_TILE);
  k_reorient_to_tc5<<<dim3(POLY / 8, T.ks), 256, 16 * TC5_TILE, s>>>(T, v, v_stride, idx_factor, nq, qt);
}
void launch_multiply_tc5(const DevParams& P, const Tc5Geom& T, const uint8_t* dbt, const uint32_t* tile_mask, const uint8_t* qt,
                         uint32_t* out_zm, size_t out_stride, int nq, int slice_begin, int slice_count, int sm_count, cudaStream_t s) {
  if (nq < 1 || nq > 16) throw Error(-2, "wgmma multiply: 1..16 queries per pass");
  if (!tc5_supported(T)) throw Error(-2, "wgmma multiply: dim0 too large for one CTA's shared memory");
  ++g_kernel_launches;
  const int grid = sm_count > 0 ? (sm_count < 2 * POLY ? sm_count : 2 * POLY) : 132;
  int ksps = 8, bbufs = 2;
  if (tc5_ring_stages(T.ks, ksps, bbufs) < 2) ksps = 4;                  // large dim0: smaller stages,
  if (tc5_ring_stages(T.ks, ksps, bbufs) < 2) bbufs = 1;                 // single-buffered operand
  const size_t smem = tc5_smem_bytes(T, ksps, bbufs);
#define TC5_LAUNCH(K, B)                                                                                                       \
  do {                                                                                                                         \
    opt_in_smem(k_multiply_tc5<K, B>, 227 * 1024);                                                                             \
    k_multiply_tc5<K, B><<<grid, TC5_THREADS, smem, s>>>(P, T, dbt, qt, out_zm, out_stride, nq, slice_begin, slice_count, tile_mask); \
  } while (0)
  if (ksps == 4) { if (bbufs == 2) TC5_LAUNCH(4, 2); else TC5_LAUNCH(4, 1); }
  else { if (bbufs == 2) TC5_LAUNCH(8, 2); else TC5_LAUNCH(8, 1); }
#undef TC5_LAUNCH
}

}  // namespace b200pir
