// ORACLE — TEST INFRASTRUCTURE ONLY.  CPU restatement of DoublePIR's init() and load_data (lib/doublepir/src): AES-128 restated
// from FIPS-197, derive_with_aes, DbInfo::new and load_data / load_data_fast.  The GPU load (sdk_b200/csrc/dpir_load.cu) is
// compared with it; tests/dpir_load_oracle.py compiles it into a temporary directory and binds it with ctypes.
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstddef>
#include <cstring>
#include <exception>
#include <string>
#include <vector>

namespace dpir {

// ---- init() and load_data: the shared matrices from their seeds, raw entries into the l x m matrix ------------------------
// AES-128 as FIPS-197 states it, byte by byte (section 5.1: SubBytes, ShiftRows, MixColumns, AddRoundKey; section 5.2 key
// expansion), with the S-box written out as the standard's Figure 7.  The reference uses the `aes` crate; this restatement
// is pinned to FIPS-197 Appendix C.1 and SP 800-38A F.5.1 by the tests.
static const uint8_t AES_SBOX[256] = {
    0x63, 0x7c, 0x77, 0x7b, 0xf2, 0x6b, 0x6f, 0xc5, 0x30, 0x01, 0x67, 0x2b, 0xfe, 0xd7, 0xab, 0x76, 0xca, 0x82, 0xc9, 0x7d, 0xfa, 0x59,
    0x47, 0xf0, 0xad, 0xd4, 0xa2, 0xaf, 0x9c, 0xa4, 0x72, 0xc0, 0xb7, 0xfd, 0x93, 0x26, 0x36, 0x3f, 0xf7, 0xcc, 0x34, 0xa5, 0xe5, 0xf1,
    0x71, 0xd8, 0x31, 0x15, 0x04, 0xc7, 0x23, 0xc3, 0x18, 0x96, 0x05, 0x9a, 0x07, 0x12, 0x80, 0xe2, 0xeb, 0x27, 0xb2, 0x75, 0x09, 0x83,
    0x2c, 0x1a, 0x1b, 0x6e, 0x5a, 0xa0, 0x52, 0x3b, 0xd6, 0xb3, 0x29, 0xe3, 0x2f, 0x84, 0x53, 0xd1, 0x00, 0xed, 0x20, 0xfc, 0xb1, 0x5b,
    0x6a, 0xcb, 0xbe, 0x39, 0x4a, 0x4c, 0x58, 0xcf, 0xd0, 0xef, 0xaa, 0xfb, 0x43, 0x4d, 0x33, 0x85, 0x45, 0xf9, 0x02, 0x7f, 0x50, 0x3c,
    0x9f, 0xa8, 0x51, 0xa3, 0x40, 0x8f, 0x92, 0x9d, 0x38, 0xf5, 0xbc, 0xb6, 0xda, 0x21, 0x10, 0xff, 0xf3, 0xd2, 0xcd, 0x0c, 0x13, 0xec,
    0x5f, 0x97, 0x44, 0x17, 0xc4, 0xa7, 0x7e, 0x3d, 0x64, 0x5d, 0x19, 0x73, 0x60, 0x81, 0x4f, 0xdc, 0x22, 0x2a, 0x90, 0x88, 0x46, 0xee,
    0xb8, 0x14, 0xde, 0x5e, 0x0b, 0xdb, 0xe0, 0x32, 0x3a, 0x0a, 0x49, 0x06, 0x24, 0x5c, 0xc2, 0xd3, 0xac, 0x62, 0x91, 0x95, 0xe4, 0x79,
    0xe7, 0xc8, 0x37, 0x6d, 0x8d, 0xd5, 0x4e, 0xa9, 0x6c, 0x56, 0xf4, 0xea, 0x65, 0x7a, 0xae, 0x08, 0xba, 0x78, 0x25, 0x2e, 0x1c, 0xa6,
    0xb4, 0xc6, 0xe8, 0xdd, 0x74, 0x1f, 0x4b, 0xbd, 0x8b, 0x8a, 0x70, 0x3e, 0xb5, 0x66, 0x48, 0x03, 0xf6, 0x0e, 0x61, 0x35, 0x57, 0xb9,
    0x86, 0xc1, 0x1d, 0x9e, 0xe1, 0xf8, 0x98, 0x11, 0x69, 0xd9, 0x8e, 0x94, 0x9b, 0x1e, 0x87, 0xe9, 0xce, 0x55, 0x28, 0xdf, 0x8c, 0xa1,
    0x89, 0x0d, 0xbf, 0xe6, 0x42, 0x68, 0x41, 0x99, 0x2d, 0x0f, 0xb0, 0x54, 0xbb, 0x16};
inline uint8_t xtime(uint8_t b) { return (uint8_t)((b << 1) ^ ((b & 0x80) ? 0x1b : 0)); }   // FIPS-197 section 4.2.1
struct Aes128 {
  uint8_t w[176];                               // the key schedule, 11 round keys of 16 bytes
  explicit Aes128(const uint8_t key[16]) {
    std::memcpy(w, key, 16);
    uint8_t rcon = 1;
    for (int i = 4; i < 44; i++) {
      uint8_t t[4] = {w[4 * i - 4], w[4 * i - 3], w[4 * i - 2], w[4 * i - 1]};
      if (i % 4 == 0) {                         // RotWord, SubWord, Rcon
        const uint8_t t0 = t[0];
        t[0] = (uint8_t)(AES_SBOX[t[1]] ^ rcon); t[1] = AES_SBOX[t[2]]; t[2] = AES_SBOX[t[3]]; t[3] = AES_SBOX[t0];
        rcon = xtime(rcon);
      }
      for (int j = 0; j < 4; j++) w[4 * i + j] = (uint8_t)(w[4 * i - 16 + j] ^ t[j]);
    }
  }
  void encrypt(const uint8_t in[16], uint8_t out[16]) const {   // state byte r + 4c = row r, column c (section 3.4)
    uint8_t s[16];
    for (int i = 0; i < 16; i++) s[i] = (uint8_t)(in[i] ^ w[i]);
    for (int round = 1; round <= 10; round++) {
      uint8_t t[16];
      for (int c = 0; c < 4; c++)
        for (int r = 0; r < 4; r++) t[r + 4 * c] = AES_SBOX[s[r + 4 * ((c + r) % 4)]];   // SubBytes + ShiftRows
      if (round < 10)
        for (int c = 0; c < 4; c++) {                                                   // MixColumns
          const uint8_t a0 = t[4 * c], a1 = t[4 * c + 1], a2 = t[4 * c + 2], a3 = t[4 * c + 3], all = (uint8_t)(a0 ^ a1 ^ a2 ^ a3);
          t[4 * c] = (uint8_t)(a0 ^ all ^ xtime((uint8_t)(a0 ^ a1)));
          t[4 * c + 1] = (uint8_t)(a1 ^ all ^ xtime((uint8_t)(a1 ^ a2)));
          t[4 * c + 2] = (uint8_t)(a2 ^ all ^ xtime((uint8_t)(a2 ^ a3)));
          t[4 * c + 3] = (uint8_t)(a3 ^ all ^ xtime((uint8_t)(a3 ^ a0)));
        }
      for (int i = 0; i < 16; i++) s[i] = (uint8_t)(t[i] ^ w[16 * round + i]);
    }
    std::memcpy(out, s, 16);
  }
};
// matrix/derivation.rs:11-22 derive_with_aes: 64 KiB chunks, chunk i = AES-128-Ctr64BE keystream from IV = BE64(i as u32) || 0^8
// (the counter is the low 8 bytes, big-endian).  Matrix::derive_from_seed (matrix.rs:125-135) reads the bytes as LE u32 words.
inline void derive_with_aes(const uint8_t key[16], uint8_t* out, size_t len) {
  const Aes128 aes(key);
  const size_t chunk = 65536;
#pragma omp parallel for schedule(static)
  for (size_t c = 0; c < (len + chunk - 1) / chunk; c++) {
    const uint64_t iv_hi = (uint32_t)c;
    for (size_t off = c * chunk; off < std::min(len, (c + 1) * chunk); off += 16) {
      const uint64_t ctr = (off - c * chunk) / 16;
      uint8_t in[16], ks[16];
      for (int b = 0; b < 8; b++) { in[b] = (uint8_t)(iv_hi >> (56 - 8 * b)); in[8 + b] = (uint8_t)(ctr >> (56 - 8 * b)); }
      aes.encrypt(in, ks);
      for (size_t b = 0; b < 16 && off + b < len; b++) out[off + b] = ks[b];
    }
  }
}
// database.rs:58-90 DbInfo::new, :345-372 num_db_entries / compute_num_entries_base_p (f64 log2 and ceil as written)
struct DbInfo { size_t db_elems, packing, ne, x; };
inline DbInfo db_info(uint64_t num_entries, uint64_t bits, uint64_t p) {
  DbInfo o;
  if ((double)bits <= std::log2((double)p)) {
    const uint64_t logp = (uint64_t)std::log2((double)p);
    o.packing = logp / bits;
    o.db_elems = (size_t)std::ceil((double)num_entries / (double)o.packing);
    o.ne = 1;
  } else {
    o.ne = (size_t)std::ceil((double)bits / std::log2((double)p));
    o.db_elems = num_entries * o.ne;
    o.packing = 0;
  }
  o.x = o.ne;
  while (o.ne % o.x != 0) o.x++;
  return o;
}
// database.rs:168-247 load_data / load_data_fast: `entries` (one value each, the iterator's items) -> the l x m matrix, minus p/2.
// Returns false where the reference indexes past the matrix (its Index impl slices data[row * m .. row * m + m] and panics).
inline bool load_data(std::vector<uint32_t>& db, const uint8_t* entries, size_t count, size_t l, size_t m, uint64_t bits, uint64_t p, const DbInfo& info) {
  db.assign(l * m, 0);
  if (info.packing > 0) {
    size_t at = 0;
    uint32_t cur = 0, coeff = 1;
    for (size_t i = 0; i < count; i++) {
      cur += (uint32_t)entries[i] * coeff;
      coeff *= 1u << bits;
      if ((i + 1) % info.packing == 0 || i + 1 == count) {
        if (at / m >= l) return false;
        db[at] = cur;
        at++; cur = 0; coeff = 1;
      }
    }
  } else {
    for (size_t i = 0; i < count; i++)
      for (size_t j = 0; j < info.ne; j++) {
        const size_t row = (i / m) * info.ne + j, col = i % m;
        if (row >= l) return false;
        uint64_t v = entries[i];
        for (size_t k = 0; k < j; k++) v /= p;                 // arith.rs:16-22 base_p
        db[row * m + col] = (uint32_t)(v % p);
      }
  }
  for (auto& v : db) v -= (uint32_t)(p / 2);             // "Map DB elems to [-p/2; p/2]" (wrapping)
  return true;
}
// database.rs:1-19 bits_from_byte, flattened (load_data_fast): 8 entries a byte, least significant bit first
inline std::vector<uint8_t> bits_from_bytes(const uint8_t* data, size_t len) {
  std::vector<uint8_t> e(8 * len);
  for (size_t i = 0; i < len; i++)
    for (int b = 0; b < 8; b++) e[8 * i + b] = (uint8_t)((data[i] >> b) & 1);
  return e;
}

}  // namespace dpir

static thread_local std::string g_err;
#define ORC_TRY try {
#define ORC_CATCH } catch (const std::exception& e) { g_err = e.what(); return -1; } return 0;

extern "C" {
const char* orc_load_last_error() { return g_err.c_str(); }
// AES-128 (FIPS-197) of one block
int orc_aes128_encrypt(const uint8_t* key, const uint8_t* in, uint8_t* out) {
  ORC_TRY
  dpir::Aes128(key).encrypt(in, out);
  ORC_CATCH
}
// derive_with_aes over len bytes
int orc_dpir_derive_with_aes(const uint8_t* key, uint8_t* out, size_t len) {
  ORC_TRY
  dpir::derive_with_aes(key, out, len);
  ORC_CATCH
}
// DbInfo::new: out = {db_elems, packing, ne, x}
int orc_dpir_db_info(uint64_t num_entries, uint64_t bits, uint64_t p, uint64_t* out) {
  ORC_TRY
  const dpir::DbInfo i = dpir::db_info(num_entries, bits, p);
  out[0] = i.db_elems; out[1] = i.packing; out[2] = i.ne; out[3] = i.x;
  ORC_CATCH
}
// load_data (bits_format 0: one entry a byte) / load_data_fast (1: eight a byte) into out (l x m).  Returns 1 where the
// reference would panic (index past the matrix), out untouched.
int orc_dpir_load_data(const uint8_t* data, size_t len, int bits_format, uint64_t num_entries, uint64_t bits, size_t l, size_t m,
                       uint64_t p, uint32_t* out) {
  ORC_TRY
  const dpir::DbInfo info = dpir::db_info(num_entries, bits, p);
  std::vector<uint8_t> e = bits_format ? dpir::bits_from_bytes(data, len) : std::vector<uint8_t>(data, data + len);
  std::vector<uint32_t> db;
  if (!dpir::load_data(db, e.data(), e.size(), l, m, bits, p, info)) return 1;
  std::memcpy(out, db.data(), l * m * 4);
  ORC_CATCH
}
}  // extern "C"
