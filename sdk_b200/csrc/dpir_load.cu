// DoublePIR offline load on the GPU: the shared matrices derived from their seeds, and raw entries laid out as the database
// matrix, both straight into HBM (DoublePirServer::new + load_data / load_data_fast, lib/doublepir/src/doublepir/server.rs:160-165,
// 201-229).  setup() then runs on these device buffers (dpir_gemm.cu), so nothing the load produces crosses PCIe but the hint.
//
// k_dpir_derive: Matrix::derive_from_seed (matrix/matrix.rs:125-135) = derive_with_aes (matrix/derivation.rs:11-22): the
// matrix's bytes are the AES-128 keystream in Ctr64BE mode, restarted every 64 KiB chunk with IV = BE64(chunk) || 0^8, i.e.
// block b of the matrix encrypts BE64(b / 4096) || BE64(b % 4096).  u32 words are read little-endian from the keystream.
// One thread per 16-byte block, through the block function of dpir_aes.cuh.
//
// k_dpir_layout: Db::load_data / load_data_fast (database/database.rs:168-247) as a gather, one thread per word of one band of
// rows of the l x m matrix, then "Map DB elems to [-p/2; p/2]" (the wrapping subtraction of p/2 from every word, touched or
// not).  A band's entries are one contiguous range of the input, so only that range needs to be on the device (dpir_api.cu
// stages the input band by band).
//
// k_dpir_synth: the words of b200pir_dpir_create_synthetic's matrix, a counter PRNG (splitmix64) of the word index.
#include "dpir_aes.cuh"

namespace b200pir {

namespace {

// ---- AES-128 (FIPS-197) on the host: the S-box from its definition (section 5.1.1: multiplicative inverse in GF(2^8), then
// the affine map), the key expansion (section 5.2) and the encryption T-table Te0 (Te1..Te3 are its byte rotations)
uint8_t gf_mul(uint8_t a, uint8_t b) {
  uint8_t r = 0;
  while (b) {
    if (b & 1) r ^= a;
    a = (uint8_t)((a << 1) ^ ((a & 0x80) ? 0x1b : 0));
    b >>= 1;
  }
  return r;
}
void aes_sbox(uint8_t s[256]) {
  for (int x = 0; x < 256; x++) {
    uint8_t inv = 0;
    for (int y = 1; y < 256 && x; y++)
      if (gf_mul((uint8_t)x, (uint8_t)y) == 1) { inv = (uint8_t)y; break; }
    uint8_t v = inv, r = inv;
    for (int i = 0; i < 4; i++) { r = (uint8_t)((r << 1) | (r >> 7)); v ^= r; }
    s[x] = (uint8_t)(v ^ 0x63);
  }
}

// grid-stride over the 16-byte blocks of an out_words-word matrix
__global__ void __launch_bounds__(256) k_dpir_derive(uint32_t* __restrict__ out, size_t out_words, const __grid_constant__ DpirAesKey key) {
  __shared__ uint32_t te[4][256];
  __shared__ uint32_t sb[256];
  dpir_aes_tables(te, sb, key);
  __syncthreads();
  const size_t blocks = (out_words + 3) / 4;
  for (size_t b = (size_t)blockIdx.x * blockDim.x + threadIdx.x; b < blocks; b += (size_t)gridDim.x * blockDim.x) {
    const uint4 o = dpir_aes_block(te, sb, key, b);
    // the last block may be partial (rows * cols * 4 is a multiple of 4 only): its words past the end are not written
    if (4 * b + 4 <= out_words) {
      *reinterpret_cast<uint4*>(out + 4 * b) = o;
    } else {
      const uint32_t w[4] = {o.x, o.y, o.z, o.w};
      for (int i = 0; i < 4 && 4 * b + i < out_words; i++) out[4 * b + i] = w[i];
    }
  }
}

// entry i of the input: a byte (load_data's Iterator<Item = u8>) or bit i % 8 of byte i / 8 (load_data_fast's bits_from_byte,
// least significant bit first)
template <bool BITS>
__device__ __forceinline__ uint32_t entry(const uint8_t* __restrict__ data, size_t i) {
  if (BITS) return (data[i >> 3] >> (i & 7)) & 1u;
  return data[i];
}

// word k of the l x m matrix (row-major, k = row * m + col), then minus p/2, for the words of rows [r0, r0 + rows): band word
// kb is word r0 m + kb.  `count` = number of entries the iterator yields; entry i is read at i - base of the staged data.
//   packing > 0: element k = sum_t e_{k packing + t} * coeff_t, coeff_0 = 1, coeff_{t+1} = coeff_t * 2^bits (wrapping u32, no
//                masking: an entry wider than `bits` spills into the next field); the last group may be partial
//                (the `iter.peek().is_none()` flush).
//   packing = 0: data[(i / m) ne + j][i % m] = base_p(p, e_i, j), so word (row, col) holds digit row % ne of entry
//                (row / ne) m + col.
// Sets bit 0 of *out_of_range when a centred word lies outside [-2^15, 2^15), the operand range of the setup GEMM
// (dpir_gemm.cu), and bit 1 when a packed entry is wider than `bits` (its element then no longer decodes field by field).
template <bool BITS>
__global__ void k_dpir_layout(uint32_t* __restrict__ band, const uint8_t* __restrict__ data, uint64_t base, uint64_t count,
                              uint64_t r0, uint64_t rows, uint64_t m, uint32_t packing, uint32_t bits, uint32_t ne, uint32_t p,
                              int* __restrict__ out_of_range) {
  const uint64_t words = rows * m, k0 = r0 * m;
  bool bad = false;
  uint32_t wide = 0;
  for (uint64_t kb = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; kb < words; kb += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t k = k0 + kb;
    uint32_t v = 0;
    if (packing) {
      const uint64_t first = k * packing;
      if (first < count) {
        uint32_t coeff = 1;
        const uint64_t last = first + packing < count ? first + packing : count;
        for (uint64_t i = first; i < last; i++) {
          const uint32_t e = entry<BITS>(data, i - base);
          if (!BITS) wide |= e >> bits;                                // a bit always fits its field
          v += e * coeff;
          coeff *= 1u << bits;
        }
      }
    } else {
      const uint64_t row = k / m, col = k - row * m;
      const uint64_t i = (row / ne) * m + col;
      if (i < count) {
        uint32_t e = entry<BITS>(data, i - base);
        for (uint32_t j = (uint32_t)(row % ne); j; j--) e /= p;       // base_p (arith.rs:16-22)
        v = e % p;
      }
    }
    v -= p / 2;
    band[kb] = v;
    bad |= (int32_t)v < -32768 || (int32_t)v > 32767;
  }
  if (bad || wide) atomicOr(out_of_range, (bad ? 1 : 0) | (wide ? 2 : 0));
}

__global__ void k_dpir_synth(uint32_t* a, size_t words, uint64_t seed, size_t index0) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= words) return;
  a[i] = (uint32_t)splitmix64_at(seed, index0 + i) & 0x3FFFFFFFu;
}

unsigned grid_for(size_t items, int block) {
  const size_t need = (items + block - 1) / block;
  return (unsigned)std::min<size_t>(need ? need : 1, 132 * 32);
}

}  // namespace

DpirAesKey dpir_aes_key(const uint8_t key[16]) {
  DpirAesKey k;
  aes_sbox(k.sbox);
  for (int i = 0; i < 4; i++) k.rk[i] = (uint32_t)key[4 * i] << 24 | (uint32_t)key[4 * i + 1] << 16 | (uint32_t)key[4 * i + 2] << 8 | key[4 * i + 3];
  uint8_t rcon = 1;
  for (int i = 4; i < 44; i++) {                          // FIPS-197 section 5.2 KeyExpansion, Nk = 4
    uint32_t t = k.rk[i - 1];
    if (i % 4 == 0) {
      t = (t << 8) | (t >> 24);                           // RotWord
      t = (uint32_t)k.sbox[t >> 24] << 24 | (uint32_t)k.sbox[(t >> 16) & 255] << 16 | (uint32_t)k.sbox[(t >> 8) & 255] << 8 |
          k.sbox[t & 255];                                // SubWord
      t ^= (uint32_t)rcon << 24;
      rcon = gf_mul(rcon, 2);
    }
    k.rk[i] = k.rk[i - 4] ^ t;
  }
  for (int x = 0; x < 256; x++) {                         // column (2s, s, s, 3s) of MixColumns applied to S-box output s
    const uint8_t s = k.sbox[x];
    k.te0[x] = (uint32_t)gf_mul(s, 2) << 24 | (uint32_t)s << 16 | (uint32_t)s << 8 | gf_mul(s, 3);
  }
  return k;
}

void launch_dpir_derive(uint32_t* out, size_t words, const DpirAesKey& key, cudaStream_t s) {
  ++g_kernel_launches;
  k_dpir_derive<<<grid_for((words + 3) / 4, 256), 256, 0, s>>>(out, words, key);
}

void launch_dpir_synth(uint32_t* a, size_t words, uint64_t seed, cudaStream_t s) {
  for (size_t off = 0, cur; off < words; off += cur) {      // 2^30 words a launch
    cur = std::min<size_t>((size_t)1 << 30, words - off);
    k_dpir_synth<<<(unsigned)((cur + 255) / 256), 256, 0, s>>>(a + off, cur, seed, off);
  }
}

void launch_dpir_layout(uint32_t* band, const uint8_t* data, uint64_t base, uint64_t count, bool bits_format, uint64_t r0,
                        uint64_t rows, uint64_t m, uint32_t packing, uint32_t bits, uint32_t ne, uint32_t p, int* out_of_range,
                        cudaStream_t s) {
  ++g_kernel_launches;
  const unsigned g = grid_for(rows * m, 256);
  if (bits_format) k_dpir_layout<true><<<g, 256, 0, s>>>(band, data, base, count, r0, rows, m, packing, bits, ne, p, out_of_range);
  else k_dpir_layout<false><<<g, 256, 0, s>>>(band, data, base, count, r0, rows, m, packing, bits, ne, p, out_of_range);
}

}  // namespace b200pir
