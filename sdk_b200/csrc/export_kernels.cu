// Database import and export: the bulk loaders (b200pir_db_upload(_slice), b200pir_db_load_file) and their inverse
// (b200pir_db_download(_slice), b200pir_db_save_file).  One launch moves a chunk of one slice (a range of z) between the device
// layout and the reference layout:
//     import: ref u64 [zc][num_per_global][dim0], all rows as the caller stages them; this GPU's rows ii = il * shard_count +
//             shard_index are selected on the device
//     export: out u64 [zc][rows][dim0], this GPU's rows only; the host scatters them to ii = il * shard_count + shard_index
// with words lo | hi << 32.  Addresses come from item_place.cuh, the module the item writers place items with.  Each kernel
// reads every byte it needs once and writes every byte of its output once; the import writes the zero padding of partial
// groups too.
#include "kernels.h"

namespace b200pir {

namespace {

// format 0 import: ref [zc][num_per_global][dim0] -> db_slice [il][jp][z] (the slice's first cell), one thread per cell.
__global__ void k_db_import_imad(MulGeom G, Shard sh, uint4* db_slice, const uint64_t* ref, int z0, int zc) {
  size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;     // over num_per * half * zc, z fastest
  const int half = G.dim0 >> 1;
  size_t total = (size_t)G.num_per * half * zc;
  if (idx >= total) return;
  int zl = (int)(idx % zc);
  size_t rest = idx / zc;
  int jp = (int)(rest % half), ii = (int)(rest / half);
  const size_t ii_global = (size_t)ii * sh.count + sh.index;
  const uint64_t* src = ref + ((size_t)zl * G.num_per * sh.count + ii_global) * G.dim0 + 2 * jp;
  uint64_t w0 = src[0], w1 = src[1];
  db_slice[((size_t)ii * half + jp) * POLY + z0 + zl] =
      make_uint4((uint32_t)w0, (uint32_t)(w0 >> 32), (uint32_t)w1, (uint32_t)(w1 >> 32));
}

// format 1 import: one warp per (z, mt, ks).  Lane (g = lane / 4, t = lane % 4) holds the A fragment of rows 16 mt + g and
// + 8, j = 32 ks + 4 t .. + 3 and + 16 (frag_byte): it reads those four runs of 4 consecutive u64 and writes its four
// 16-byte limb words of each modulus' group.
__global__ void __launch_bounds__(256)
k_db_import_frag(ImmaGeom F, Shard sh, const uint64_t* __restrict__ ref, int slice, int z0, int zc, uint4* __restrict__ dbf) {
  const int lane = threadIdx.x & 31;
  const size_t warp = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const size_t total = (size_t)zc * F.mt * F.ks;
  if (warp >= total) return;
  const int ks = (int)(warp % F.ks);
  const int mt = (int)((warp / F.ks) % F.mt);
  const int zl = (int)(warp / ((size_t)F.ks * F.mt));
  const int g = lane >> 2, t = lane & 3;
  uint32_t res[2][2][2][4];        // [n][row half (g, g+8)][k half (0, +16)][i]
#pragma unroll
  for (int rh = 0; rh < 2; rh++) {
    const int ii = mt * 16 + g + 8 * rh;
    const uint64_t* src = ref + ((size_t)zl * F.rows * sh.count + (size_t)ii * sh.count + sh.index) * F.dim0;
#pragma unroll
    for (int kh = 0; kh < 2; kh++) {
      const int j0 = ks * 32 + 16 * kh + 4 * t;
#pragma unroll
      for (int i = 0; i < 4; i++) {
        const uint64_t w = ii < F.rows && j0 + i < F.dim0 ? src[j0 + i] : 0;
        res[0][rh][kh][i] = (uint32_t)w;
        res[1][rh][kh][i] = (uint32_t)(w >> 32);
      }
    }
  }
#pragma unroll
  for (int n = 0; n < 2; n++) {
    uint4* dst = dbf + frag_db_group(F, slice, n, z0 + zl, mt, ks) * (FRAG_GROUP / 16) + lane;
#pragma unroll
    for (int l = 0; l < 4; l++)      // a0..a3: (row g, k lo), (row g+8, k lo), (row g, k hi), (row g+8, k hi)
      dst[(size_t)l * 32] = make_uint4(tc5_limb4(res[n][0][0], l), tc5_limb4(res[n][1][0], l), tc5_limb4(res[n][0][1], l),
                                       tc5_limb4(res[n][1][1], l));
  }
}

// format 2 import: CTA = (z, mt, ks), thread = (row, kq) of tc5_db_thread.  A row's eight threads read its 256 contiguous
// bytes of j = 32 ks .. + 31 and each writes the four 4-byte limb words of its four values of j in both moduli's tiles.
__global__ void __launch_bounds__(256)
k_db_import_tc5(Tc5Geom T, Shard sh, const uint64_t* __restrict__ ref, int slice, int z0, uint8_t* __restrict__ dbt) {
  const int zl = blockIdx.x, mt = blockIdx.y, ks = blockIdx.z;
  const Tc5DbThread t = tc5_db_thread(threadIdx.x, mt, ks);
  const int j0 = 2 * t.jp0;                                       // the thread's four values of j: j0 .. j0 + 3
  const uint64_t* src = ref + ((size_t)zl * T.rows * sh.count + (size_t)t.ii * sh.count + sh.index) * T.dim0 + j0;
  uint32_t res[2][4];
#pragma unroll
  for (int i = 0; i < 4; i++) {
    const uint64_t w = t.ii < T.rows && j0 + i < T.dim0 ? src[i] : 0;
    res[0][i] = (uint32_t)w;
    res[1][i] = (uint32_t)(w >> 32);
  }
#pragma unroll
  for (int n = 0; n < 2; n++) tc5_db_store(dbt + tc5_db_tile(T, slice, n, z0 + zl, mt, ks) * TC5_TILE, t, res[n]);
}

// format 0 export: the cell uint4 (il, jp, z) is exactly the output pair (w(2jp), w(2jp+1)), so the chunk is a transpose of
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

// formats 1 and 2 export: CTA = (z, row group mt, k-step ks).  The group's two limb images (n = 0, 1; ROWS rows x 32 values of j,
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

void launch_db_import(const DbLayout& L, Shard sh, int slice, const uint64_t* ref_chunk, int z0, int zc, cudaStream_t s) {
  if (zc <= 0) return;
  ++g_kernel_launches;
  if (L.format == 0) {
    const size_t cells = (size_t)L.G.num_per * (L.G.dim0 >> 1) * zc;
    k_db_import_imad<<<(unsigned)((cells + 255) / 256), 256, 0, s>>>(
        L.G, sh, reinterpret_cast<uint4*>(L.base) + imad_cell(L.G, slice, 0, 0, 0), ref_chunk, z0, zc);
  } else if (L.format == 2) {
    k_db_import_tc5<<<dim3((unsigned)zc, (unsigned)L.T.mt, (unsigned)L.T.ks), 256, 0, s>>>(L.T, sh, ref_chunk, slice, z0, L.base);
  } else {
    const size_t warps = (size_t)zc * L.F.mt * L.F.ks;
    k_db_import_frag<<<(unsigned)((warps + 7) / 8), 256, 0, s>>>(L.F, sh, ref_chunk, slice, z0, zc, reinterpret_cast<uint4*>(L.base));
  }
}

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
