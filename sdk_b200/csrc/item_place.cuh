// Where one NTT coordinate z of one database item lives in each device layout, and how it is read back.  Item (slice, local
// row il, column j) holds, at every z, the residue mod q0 (`lo`) and mod q1 (`hi`) of the packed word lo | hi << 32
// (loading.rs:34-41 pack_ntt_poly).  The single-item upsert (mul_kernels.cu), the batched item writer (k_write_items in
// poly_kernels.cu: raw bytes or the synthetic database), its inverse (k_read_items) and the import and export kernels
// (export_kernels.cu) all address the database through these maps, so
// every writer and reader agrees on the layouts; the host sizes the store with db_bytes.  The maps are __host__ __device__
// and use no CUDA types: tests/cpp/db_layout_inverse.cpp checks on the CPU that place and fetch are mutually inverse, that no
// two items share a byte and that every byte a writer touches lies inside db_bytes.
#pragma once
#include <stdint.h>
#include <stddef.h>
#include "tc5_layout.cuh"

#if defined(__CUDA_ARCH__)
#define ITEM_UNROLL _Pragma("unroll")
#else
#define ITEM_UNROLL
#endif

namespace b200pir {

static const int POLY = 2048;

// first-dimension geometries of one database (num_per / rows = the rows this GPU holds)
struct MulGeom { int dim0, num_per, slices; };
struct ImmaGeom { int dim0, rows, mt /* ceil(rows/16) */, ks /* ceil(dim0/32) */; };
inline ImmaGeom make_imma_geom(int dim0, int rows) { return ImmaGeom{dim0, rows, (rows + 15) / 16, (dim0 + 31) / 32}; }

// ---- format 0 (mul_kernels.cu): uint4 [slice][il][jp = j/2][z] = {w(2jp).lo, w(2jp).hi, w(2jp+1).lo, w(2jp+1).hi}
// 16-byte cell of w(j), and the u32 word of w(j).lo in it; w(j).hi is the next word
TC5_HD size_t imad_cell(const MulGeom& G, int slice, int il, int j, int z) {
  const int half = G.dim0 >> 1;
  return (((size_t)slice * G.num_per + il) * half + (j >> 1)) * POLY + z;
}
TC5_HD size_t imad_word(const MulGeom& G, int slice, int il, int j, int z) { return imad_cell(G, slice, il, j, z) * 4 + 2 * (j & 1); }
TC5_HD void place_imad(const MulGeom& G, uint32_t* db, int slice, int il, int j, int z, uint32_t lo, uint32_t hi) {
#if defined(__CUDA_ARCH__)
  *(reinterpret_cast<uint2*>(reinterpret_cast<uint4*>(db) + imad_cell(G, slice, il, j, z)) + (j & 1)) = make_uint2(lo, hi);
#else
  uint32_t* w = db + imad_word(G, slice, il, j, z);
  w[0] = lo; w[1] = hi;
#endif
}
TC5_HD uint64_t fetch_imad(const MulGeom& G, const uint32_t* db, int slice, int il, int j, int z) {
  const uint32_t* w = db + imad_word(G, slice, il, j, z);
  return (uint64_t)w[0] | (uint64_t)w[1] << 32;
}

// ---- formats 1 and 2 store each residue r as four 7-bit limbs (r >> 7l) & 127, one byte each.  Both are planes per
// (slice, n, z) of mt x ks groups; a group holds ROWS rows x 32 values of j of one modulus: 2048 bytes (format 1, 16 rows)
// or one 4096-byte wgmma tile image (format 2, 32 rows).
TC5_HD size_t limb_plane(int mt, int ks, int group_bytes, int slice, int n, int z) {
  return (((size_t)slice * 2 + n) * POLY + z) * mt * ks * group_bytes;
}

// format 1 (imma_kernels.cu): dbF[slice][n][z][mt][ks][limb l][lane] = uint4{a0, a1, a2, a3} (mma.sync A fragments)
constexpr int FRAG_GROUP = 4 * 32 * 16;
// byte of (row < 16, k < 32, limb l) in a group: a0..a3 = (row g, k lo), (row g+8, k lo), (row g, k hi), (row g+8, k hi)
TC5_HD int frag_byte(int row, int k, int l) {
  const int g = row & 7, rh = row >> 3, kh = k >> 4, t = (k & 15) >> 2, i = k & 3;
  return (l * 32 + g * 4 + t) * 16 + (rh + 2 * kh) * 4 + i;
}
TC5_HD size_t frag_in_plane(const ImmaGeom& F, int il, int j, int l) {
  return ((size_t)(il >> 4) * F.ks + (j >> 5)) * FRAG_GROUP + frag_byte(il & 15, j & 31, l);
}
TC5_HD size_t frag_plane(const ImmaGeom& F, int slice, int n, int z) { return limb_plane(F.mt, F.ks, FRAG_GROUP, slice, n, z); }
// index of the group (mt, ks) of plane (slice, n, z), in FRAG_GROUP-byte units (the import kernel writes whole groups)
TC5_HD size_t frag_db_group(const ImmaGeom& F, int slice, int n, int z, int mt, int ks) {
  return ((((size_t)slice * 2 + n) * POLY + z) * F.mt + mt) * F.ks + ks;
}

// format 2 (tc5_kernels.cu): tile images dbT[slice][n][z][mt][ks][4096 B], byte tc5_tile_off(4 row + l, k)
TC5_HD size_t tc5_in_plane(const Tc5Geom& T, int il, int j, int l) {
  return ((size_t)(il >> 5) * T.ks + (j >> 5)) * TC5_TILE + tc5_tile_off(tc5_m_index(il & 31, l), j & 31);
}
TC5_HD size_t tc5_plane(const Tc5Geom& T, int slice, int n, int z) { return limb_plane(T.mt, T.ks, TC5_TILE, slice, n, z); }

// the limb-l bytes of k = 4 kq .. 4 kq + 3 of one row are consecutive in both layouts: the export kernels read them as one
// 4-byte word (byte offset within the group)
TC5_HD int frag_word(int row, int kq, int l) { return frag_byte(row, 4 * kq, l); }
TC5_HD int tc5_word(int row, int kq, int l) { return tc5_tile_off(tc5_m_index(row, l), 4 * kq); }
// four residues from the four limb words of k = 4 kq .. 4 kq + 3 (limb l of k = 4 kq + i is byte i of word l)
TC5_HD void join_limb_words(const uint32_t (&w)[4], uint32_t (&r)[4]) {
  ITEM_UNROLL
  for (int i = 0; i < 4; i++)
    r[i] = ((w[0] >> (8 * i)) & 127u) | (((w[1] >> (8 * i)) & 127u) << 7) | (((w[2] >> (8 * i)) & 127u) << 14) |
           (((w[3] >> (8 * i)) & 127u) << 21);
}

TC5_HD void place_frag(const ImmaGeom& F, uint8_t* dbf, int slice, int il, int j, int z, uint32_t lo, uint32_t hi) {
  ITEM_UNROLL
  for (int n = 0; n < 2; n++) {
    const uint32_t r = n ? hi : lo;
    uint8_t* plane = dbf + frag_plane(F, slice, n, z);
    ITEM_UNROLL
    for (int l = 0; l < 4; l++) plane[frag_in_plane(F, il, j, l)] = (uint8_t)((r >> (7 * l)) & 127u);
  }
}
TC5_HD uint64_t fetch_frag(const ImmaGeom& F, const uint8_t* dbf, int slice, int il, int j, int z) {
  uint64_t w = 0;
  for (int n = 0; n < 2; n++) {
    const uint8_t* plane = dbf + frag_plane(F, slice, n, z);
    for (int l = 0; l < 4; l++) w |= (uint64_t)plane[frag_in_plane(F, il, j, l)] << (32 * n + 7 * l);
  }
  return w;
}

TC5_HD void place_tc5(const Tc5Geom& T, uint8_t* dbt, int slice, int il, int j, int z, uint32_t lo, uint32_t hi) {
  ITEM_UNROLL
  for (int n = 0; n < 2; n++) {
    const uint32_t r = n ? hi : lo;
    uint8_t* plane = dbt + tc5_plane(T, slice, n, z);
    ITEM_UNROLL
    for (int l = 0; l < 4; l++) plane[tc5_in_plane(T, il, j, l)] = (uint8_t)((r >> (7 * l)) & 127u);
  }
}
TC5_HD uint64_t fetch_tc5(const Tc5Geom& T, const uint8_t* dbt, int slice, int il, int j, int z) {
  uint64_t w = 0;
  for (int n = 0; n < 2; n++) {
    const uint8_t* plane = dbt + tc5_plane(T, slice, n, z);
    for (int l = 0; l < 4; l++) w |= (uint64_t)plane[tc5_in_plane(T, il, j, l)] << (32 * n + 7 * l);
  }
  return w;
}

// ---- one database as every writer and reader sees it: its layout, the geometries of the three layouts (local rows) and its
// store, db_bytes(layout, slices) bytes at `base` (cudaMalloc's 256-byte alignment covers the uint4 view of format 0)
struct DbLayout {
  int format;               // 0: IMAD cells, 1: mma.sync fragments, 2: wgmma tile images
  MulGeom G; ImmaGeom F; Tc5Geom T;
  uint8_t* base;
};
// bytes of the first `slices` slices of the store; every size and slice offset of a store is counted here, in bytes
TC5_HD size_t db_bytes(const DbLayout& L, int slices) {
  if (L.format == 0) return imad_cell(L.G, slices, 0, 0, 0) * 16;
  if (L.format == 2) return limb_plane(L.T.mt, L.T.ks, TC5_TILE, slices, 0, 0);
  return limb_plane(L.F.mt, L.F.ks, FRAG_GROUP, slices, 0, 0);
}
TC5_HD size_t slice_bytes(const DbLayout& L) { return db_bytes(L, 1); }

TC5_HD void place_item(const DbLayout& L, int slice, int il, int j, int z, uint32_t lo, uint32_t hi) {
  if (L.format == 0) place_imad(L.G, reinterpret_cast<uint32_t*>(L.base), slice, il, j, z, lo, hi);
  else if (L.format == 2) place_tc5(L.T, L.base, slice, il, j, z, lo, hi);
  else place_frag(L.F, L.base, slice, il, j, z, lo, hi);
}
TC5_HD uint64_t fetch_item(const DbLayout& L, int slice, int il, int j, int z) {
  if (L.format == 0) return fetch_imad(L.G, reinterpret_cast<const uint32_t*>(L.base), slice, il, j, z);
  if (L.format == 2) return fetch_tc5(L.T, L.base, slice, il, j, z);
  return fetch_frag(L.F, L.base, slice, il, j, z);
}

// ---- plaintext bytes of an item (p = 256).  convert_pt_to_poly (loading.rs:278-299) stores coefficient byte x as
// recenter_mod(x, 256, q) (arith.rs:415) mod both q_n: x for x <= 128, q - (256 - x) above.  The item reader (k_read_items)
// inverts it coefficient by coefficient; tests/cpp/pt_byte_decode.cpp checks the rule on the CPU.
TC5_HD uint32_t pt_byte_residue(uint32_t x, uint32_t q) { return x <= 128 ? x : q - (256 - x); }
// The byte x whose residues mod q0 and q1 are r0 and r1, or -1 when the pair is not the image of one byte ("not plaintext").
// Any 32-bit words are accepted: each is reduced mod its modulus first (format 0 keeps uploaded halves verbatim).
TC5_HD int pt_byte_decode(uint32_t r0, uint32_t r1, uint32_t q0, uint32_t q1) {
  r0 %= q0;
  r1 %= q1;
  uint32_t x;
  if (r0 <= 128) x = r0;
  else if (r0 >= q0 - 127) x = r0 - (q0 - 256);
  else return -1;
  return r1 == pt_byte_residue(x, q1) ? (int)x : -1;
}

}  // namespace b200pir
