// Where one NTT coordinate z of one database item lives in each device layout.  Item (slice, local row il, column j) holds,
// at every z, the residue mod q0 (`lo`) and mod q1 (`hi`) of the packed word lo | hi << 32 (loading.rs:34-41 pack_ntt_poly).
// Used by the single-item upserts and by the batched raw-byte writer (k_write_items), so every writer agrees on the layouts.
#pragma once
#include "kernels.h"

namespace b200pir {

// format 0 (mul_kernels.cu): uint4 [slice][il][jp = j/2][z] = {w(2jp).lo, w(2jp).hi, w(2jp+1).lo, w(2jp+1).hi}
__device__ __forceinline__ void place_imad(const MulGeom& G, uint4* db, int slice, int il, int j, int z, uint32_t lo, uint32_t hi) {
  const int half = G.dim0 >> 1;
  uint2* cell = reinterpret_cast<uint2*>(db + (((size_t)slice * G.num_per + il) * half + (j >> 1)) * POLY + z) + (j & 1);
  *cell = make_uint2(lo, hi);
}

// format 1 (imma_kernels.cu): dbF[slice][n][z][mt][ks][limb l][lane] = uint4{a0, a1, a2, a3}; one byte per limb
__device__ __forceinline__ void place_frag(const ImmaGeom& F, uint4* dbf, int slice, int il, int j, int z, uint32_t lo, uint32_t hi) {
  const int mt = il >> 4, row = il & 15, ks = j >> 5, k = j & 31;
  const int g = row & 7, rh = row >> 3, kh = k >> 4, t = (k & 15) >> 2, i = k & 3;
  const int lane = g * 4 + t, reg = rh + 2 * kh;       // a0..a3 = (row g,k lo), (row g+8,k lo), (row g,k hi), (row g+8,k hi)
#pragma unroll
  for (int n = 0; n < 2; n++) {
    const uint32_t r = n ? hi : lo;
    uint8_t* base = reinterpret_cast<uint8_t*>(dbf + (((((size_t)slice * 2 + n) * POLY + z) * F.mt + mt) * F.ks + ks) * 4 * 32);
#pragma unroll
    for (int l = 0; l < 4; l++) base[((size_t)l * 32 + lane) * 16 + reg * 4 + i] = (uint8_t)((r >> (7 * l)) & 127u);
  }
}

// format 2 (tc5_kernels.cu): tile images dbT[slice][n][z][mt][ks][4096 B]; one byte per limb
__device__ __forceinline__ void place_tc5(const Tc5Geom& T, uint8_t* dbt, int slice, int il, int j, int z, uint32_t lo, uint32_t hi) {
  const int mt = il >> 5, row_local = il & 31, ks = j >> 5, k = j & 31;
#pragma unroll
  for (int n = 0; n < 2; n++) {
    const uint32_t r = n ? hi : lo;
    uint8_t* tile = dbt + tc5_db_tile(T, slice, n, z, mt, ks) * TC5_TILE;
#pragma unroll
    for (int l = 0; l < 4; l++) tile[tc5_tile_off(tc5_m_index(row_local, l), k)] = (uint8_t)((r >> (7 * l)) & 127u);
  }
}

}  // namespace b200pir
