// Database export: the inverse of the loaders (b200pir_db_download / b200pir_db_save_file).  One launch un-tiles a chunk of
// one slice (a range of z, the local rows) from the device layout into the reference layout restricted to this GPU's rows,
//     out u64 [zc][rows][dim0] = lo | hi << 32,
// which the host copies out and scatters to ii = il * shard_count + shard_index.  Addresses come from item_place.cuh, the
// module the writers place items with.  The un-tiling reads every byte of the chunk once and writes every output word once.
#include "kernels.h"

namespace b200pir {

namespace {

// format 0: the cell uint4 (il, jp, z) is exactly the output pair (w(2jp), w(2jp+1)), so the chunk is a transpose of
// [il][jp][z] into [z][il][jp] in 16-byte elements.  CTA = (il, 32 values of jp, 32 values of z), staged through a padded
// shared-memory tile: reads are runs of z (512 bytes), writes runs of jp (512 bytes when dim0 >= 64).
__global__ void __launch_bounds__(256)
k_db_export_imad(MulGeom G, const uint4* __restrict__ db, int slice, int z0, int zc, uint64_t* __restrict__ out) {
  __shared__ uint4 tile[32][33];
  const int half = G.dim0 >> 1;
  const int il = blockIdx.x, jb = blockIdx.y * 32, zb = blockIdx.z * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
#pragma unroll
  for (int r = ty; r < 32; r += 8) {
    const int jp = jb + r, zl = zb + tx;
    if (jp < half && zl < zc) tile[r][tx] = db[imad_cell(G, slice, il, 2 * jp, z0 + zl)];
  }
  __syncthreads();
  uint4* o = reinterpret_cast<uint4*>(out);
#pragma unroll
  for (int r = ty; r < 32; r += 8) {
    const int zl = zb + r, jp = jb + tx;
    if (jp < half && zl < zc) o[((size_t)zl * G.num_per + il) * half + jp] = tile[tx][r];
  }
}

// formats 1 and 2: CTA = (z, row group mt, k-step ks).  The group's two limb images (n = 0, 1; ROWS rows x 32 values of j,
// GROUP bytes each) are staged in shared memory with 16-byte loads; thread (row, kq) reads, per modulus, the four 4-byte
// words that hold limbs 0..3 of j = ks*32 + 4 kq .. + 3, rebuilds the four residues and writes four output words (32
// contiguous bytes; the eight threads of a row write its 256 bytes).  Rows past `rows` and j past dim0 are the padding of
// partial groups and are skipped.
template <int ROWS>
__global__ void __launch_bounds__(ROWS * 8)
k_db_export_limbs(const uint8_t* __restrict__ db, int mt_count, int ks_count, int rows, int dim0, int slice, int z0,
                  uint64_t* __restrict__ out) {
  constexpr int GROUP = ROWS * 32 * 4;                 // FRAG_GROUP (16 rows) or TC5_TILE (32 rows)
  constexpr int THREADS = ROWS * 8;
  static_assert(GROUP == (ROWS == 16 ? FRAG_GROUP : TC5_TILE), "group size");
  __shared__ __align__(16) uint8_t img[2][GROUP];
  const int zl = blockIdx.x, mt = blockIdx.y, ks = blockIdx.z;
  const size_t group = ((size_t)mt * ks_count + ks) * GROUP;
#pragma unroll
  for (int n = 0; n < 2; n++) {
    const uint4* src = reinterpret_cast<const uint4*>(db + limb_plane(mt_count, ks_count, GROUP, slice, n, z0 + zl) + group);
#pragma unroll
    for (int i = threadIdx.x; i < GROUP / 16; i += THREADS) reinterpret_cast<uint4*>(img[n])[i] = src[i];
  }
  __syncthreads();
  const int row = threadIdx.x >> 3, kq = threadIdx.x & 7;
  const int il = mt * ROWS + row, j0 = ks * 32 + 4 * kq;
  if (il >= rows || j0 >= dim0) return;
  uint32_t r[2][4];
#pragma unroll
  for (int n = 0; n < 2; n++) {
    uint32_t w[4];
#pragma unroll
    for (int l = 0; l < 4; l++)
      w[l] = *reinterpret_cast<const uint32_t*>(img[n] + (ROWS == 16 ? frag_word(row, kq, l) : tc5_word(row, kq, l)));
    join_limb_words(w, r[n]);
  }
  uint64_t* dst = out + ((size_t)zl * rows + il) * dim0 + j0;
  if (j0 + 4 <= dim0) {
    reinterpret_cast<uint4*>(dst)[0] = make_uint4(r[0][0], r[1][0], r[0][1], r[1][1]);
    reinterpret_cast<uint4*>(dst)[1] = make_uint4(r[0][2], r[1][2], r[0][3], r[1][3]);
  } else {
    for (int i = 0; i < dim0 - j0; i++) dst[i] = (uint64_t)r[0][i] | (uint64_t)r[1][i] << 32;
  }
}

}  // namespace

void launch_db_export(const DbLayout& L, int slice, int z0, int zc, uint64_t* out, cudaStream_t s) {
  if (zc <= 0) return;
  ++g_kernel_launches;
  if (L.format == 0) {
    const dim3 grid((unsigned)L.G.num_per, (unsigned)((L.G.dim0 / 2 + 31) / 32), (unsigned)((zc + 31) / 32));
    k_db_export_imad<<<grid, 256, 0, s>>>(L.G, reinterpret_cast<const uint4*>(L.base), slice, z0, zc, out);
  } else if (L.format == 2) {
    k_db_export_limbs<32><<<dim3((unsigned)zc, (unsigned)L.T.mt, (unsigned)L.T.ks), 256, 0, s>>>(
        L.base, L.T.mt, L.T.ks, L.T.rows, L.T.dim0, slice, z0, out);
  } else {
    k_db_export_limbs<16><<<dim3((unsigned)zc, (unsigned)L.F.mt, (unsigned)L.F.ks), 128, 0, s>>>(
        L.base, L.F.mt, L.F.ks, L.F.rows, L.F.dim0, slice, z0, out);
  }
}

}  // namespace b200pir
