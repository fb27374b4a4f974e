// One 16-byte block of the keystream Matrix::derive_from_seed reads (matrix/derivation.rs:11-22), for every kernel that derives
// A_1 or A_2 words: k_dpir_derive (whole matrices, dpir_load.cu) and the entry update (single rows of A_1, dpir_update.cu).
// T-tables (FIPS-197 section 5.2.1's round as four 32-bit table lookups per column) in shared memory.  The lookups are
// data-dependent, so this is NOT constant-time: that is fine here, because the key and the output are public (the reference
// derives public matrices only, matrix.rs:120-124) and nothing secret ever passes through it.
#pragma once
#include "dpir_kernels.h"

namespace b200pir {

__device__ __forceinline__ uint32_t dpir_ror8(uint32_t v, int n) { return __funnelshift_r(v, v, n); }

// the four T-tables and the S-box of `key` into shared memory, by every thread of the CTA; the caller synchronises
__device__ __forceinline__ void dpir_aes_tables(uint32_t (*te)[256], uint32_t* sb, const DpirAesKey& key) {
  for (int i = threadIdx.x; i < 256; i += blockDim.x) {
    const uint32_t t = key.te0[i];
    te[0][i] = t; te[1][i] = dpir_ror8(t, 8); te[2][i] = dpir_ror8(t, 16); te[3][i] = dpir_ror8(t, 24);
    sb[i] = key.sbox[i];
  }
}

// Matrix words 4b .. 4b + 3 of derive_with_aes: block b encrypts BE64(b / 4096) || BE64(b % 4096) (Ctr64BE restarted every
// 64 KiB chunk), and the matrix reads the keystream's bytes as little-endian u32 words.
__device__ __forceinline__ uint4 dpir_aes_block(const uint32_t (*te)[256], const uint32_t* sb, const DpirAesKey& key, uint64_t b) {
  // derive_with_aes_at(key, i as u32, chunk): the chunk index is cast to u32 before it is widened into the IV
  const uint64_t chunk = (uint32_t)(b >> 12), ctr = b & 4095;
  // state columns as big-endian words (FIPS-197 section 3.4), round key 0 added
  uint32_t s0 = (uint32_t)(chunk >> 32) ^ key.rk[0], s1 = (uint32_t)chunk ^ key.rk[1];
  uint32_t s2 = (uint32_t)(ctr >> 32) ^ key.rk[2], s3 = (uint32_t)ctr ^ key.rk[3];
#pragma unroll
  for (int r = 1; r < 10; r++) {
    const uint32_t t0 = te[0][s0 >> 24] ^ te[1][(s1 >> 16) & 255] ^ te[2][(s2 >> 8) & 255] ^ te[3][s3 & 255] ^ key.rk[4 * r];
    const uint32_t t1 = te[0][s1 >> 24] ^ te[1][(s2 >> 16) & 255] ^ te[2][(s3 >> 8) & 255] ^ te[3][s0 & 255] ^ key.rk[4 * r + 1];
    const uint32_t t2 = te[0][s2 >> 24] ^ te[1][(s3 >> 16) & 255] ^ te[2][(s0 >> 8) & 255] ^ te[3][s1 & 255] ^ key.rk[4 * r + 2];
    const uint32_t t3 = te[0][s3 >> 24] ^ te[1][(s0 >> 16) & 255] ^ te[2][(s1 >> 8) & 255] ^ te[3][s2 & 255] ^ key.rk[4 * r + 3];
    s0 = t0; s1 = t1; s2 = t2; s3 = t3;
  }
  // last round: SubBytes, ShiftRows, AddRoundKey (no MixColumns)
  const uint32_t o0 = (sb[s0 >> 24] << 24 | sb[(s1 >> 16) & 255] << 16 | sb[(s2 >> 8) & 255] << 8 | sb[s3 & 255]) ^ key.rk[40];
  const uint32_t o1 = (sb[s1 >> 24] << 24 | sb[(s2 >> 16) & 255] << 16 | sb[(s3 >> 8) & 255] << 8 | sb[s0 & 255]) ^ key.rk[41];
  const uint32_t o2 = (sb[s2 >> 24] << 24 | sb[(s3 >> 16) & 255] << 16 | sb[(s0 >> 8) & 255] << 8 | sb[s1 & 255]) ^ key.rk[42];
  const uint32_t o3 = (sb[s3 >> 24] << 24 | sb[(s0 >> 16) & 255] << 16 | sb[(s1 >> 8) & 255] << 8 | sb[s2 & 255]) ^ key.rk[43];
  // keystream bytes 4w..4w+3 are big-endian column w
  return make_uint4(__byte_perm(o0, 0, 0x0123), __byte_perm(o1, 0, 0x0123), __byte_perm(o2, 0, 0x0123), __byte_perm(o3, 0, 0x0123));
}

}  // namespace b200pir
