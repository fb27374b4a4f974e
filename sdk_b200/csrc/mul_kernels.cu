// First-dimension kernels on the IMAD layout (format 0): multiply_reg_by_database (lib/spiral-rs/src/server.rs:155-221) over
// an HBM-resident database and the query operand it reads; and the single-item upsert into any layout.  The item writer
// (k_write_items) runs the NTT and so lives with the other transforms in poly_kernels.cu.  The products are pure
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

}  // namespace

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

}  // namespace b200pir
