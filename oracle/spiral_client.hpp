// ORACLE — TEST INFRASTRUCTURE ONLY (see spiral_oracle.hpp).
//
// Harness-only restatement of the Spiral CLIENT (keygen / query generation / response
// decoding) so that the tests can build valid queries and decrypt server output the same way
// the reference's own tests do (lib/spiral-rs/src/server.rs:787-1047).  The client is OUT OF
// SCOPE as product; nothing here is ever shipped or benchmarked.
//
// Randomness: the reference draws from ChaCha20Rng::from_entropy() (client.rs:547,626), so no
// reference stream exists to match; we use a seeded xoshiro256** so tests are reproducible.
#pragma once
#include "spiral_oracle.hpp"

namespace orc {

struct Rng {                       // xoshiro256**, seeded through splitmix64
  u64 s[4];
  explicit Rng(u64 seed) {
    for (int i = 0; i < 4; i++) {
      seed += 0x9E3779B97F4A7C15ULL;
      u64 z = seed;
      z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL;
      z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL;
      s[i] = z ^ (z >> 31);
    }
  }
  static u64 rotl(u64 x, int k) { return (x << k) | (x >> (64 - k)); }
  u64 next() {
    u64 result = rotl(s[1] * 5, 7) * 9, t = s[1] << 17;
    s[2] ^= s[0]; s[3] ^= s[1]; s[1] ^= s[2]; s[0] ^= s[3];
    s[2] ^= t; s[3] = rotl(s[3], 45);
    return result;
  }
};

// ChaCha20 keystream as rand_chacha 0.3.1's ChaCha20Rng consumes it (lib/spiral-rs/Cargo.lock; call sites
// client.rs:218, :309): RFC 8439 block function (20 rounds), 32-byte seed = key, 64-bit block counter in words 12-13
// starting at 0, stream id (words 14-15) = 0, output words in keystream order, next_u64 = word[i] | word[i+1] << 32.
// The crate is absent from the reference tree and the reference stores no serialized vectors, so this cannot be checked against
// reference output here; it is pinned instead (tests/test_oracle_kats.py) by the RFC 8439 section 2.3.2 block vector and by
// rand_chacha's own published known-answer test for ChaCha20Rng::from_seed([0; 32]) (first 32 output words = RFC 7539 A.1
// vectors #1, #2), which fixes key placement, counter position / start / increment and word order.  How the call sites
// consume the stream (q - next_u64() % q, matrix by matrix) is restated from client.rs, which IS in the reference.
inline void chacha20_block(const u32 init[16], u32 out[16]) {
  u32 x[16];
  for (int i = 0; i < 16; i++) x[i] = init[i];
  auto rotl = [](u32 v, int c) { return (v << c) | (v >> (32 - c)); };
  auto qr = [&](int a, int b, int c, int d) {
    x[a] += x[b]; x[d] ^= x[a]; x[d] = rotl(x[d], 16);
    x[c] += x[d]; x[b] ^= x[c]; x[b] = rotl(x[b], 12);
    x[a] += x[b]; x[d] ^= x[a]; x[d] = rotl(x[d], 8);
    x[c] += x[d]; x[b] ^= x[c]; x[b] = rotl(x[b], 7);
  };
  for (int r = 0; r < 10; r++) {
    qr(0, 4, 8, 12); qr(1, 5, 9, 13); qr(2, 6, 10, 14); qr(3, 7, 11, 15);
    qr(0, 5, 10, 15); qr(1, 6, 11, 12); qr(2, 7, 8, 13); qr(3, 4, 9, 14);
  }
  for (int i = 0; i < 16; i++) out[i] = x[i] + init[i];
}
struct ChaCha20Rng {
  u32 st[16];
  u32 buf[16];
  int idx = 16;
  ChaCha20Rng() { std::memset(st, 0, sizeof(st)); }
  explicit ChaCha20Rng(const uint8_t seed[32]) {
    st[0] = 0x61707865; st[1] = 0x3320646e; st[2] = 0x79622d32; st[3] = 0x6b206574;
    for (int i = 0; i < 8; i++) st[4 + i] = (u32)seed[4 * i] | ((u32)seed[4 * i + 1] << 8) | ((u32)seed[4 * i + 2] << 16) | ((u32)seed[4 * i + 3] << 24);
    st[12] = st[13] = st[14] = st[15] = 0;
  }
  u32 next_u32() {
    if (idx == 16) {
      chacha20_block(st, buf);
      if (++st[12] == 0) ++st[13];
      idx = 0;
    }
    return buf[idx++];
  }
  u64 next() { u64 lo = next_u32(); u64 hi = next_u32(); return lo | (hi << 32); }
};

// discrete_gaussian.rs:64-139
struct DiscreteGaussian {
  std::vector<u64> cdf_table;
  i64 max_val;
  explicit DiscreteGaussian(double noise_width) {
    max_val = (i64)std::ceil(noise_width * 4.0);
    std::vector<double> table;
    double total = 0.0;
    for (i64 i = -max_val; i <= max_val; i++) {
      double pv = std::exp(-M_PI * (double)(i * i) / (noise_width * noise_width));
      table.push_back(pv);
      total += pv;
    }
    double cum = 0.0;
    for (double pv : table) {
      cum += pv / total;
      double scaled = std::round(cum * 18446744073709551615.0);
      cdf_table.push_back(scaled >= 18446744073709551615.0 ? ~(u64)0 : (u64)scaled);
    }
  }
  u64 sample(u64 modulus, Rng& rng) const {
    u64 sampled = rng.next();
    size_t len = (size_t)(2 * max_val + 1);
    u64 to_output = 0;
    for (size_t i = len; i-- > 0;) {
      i64 out_val = (i64)i - max_val;
      if (out_val < 0) out_val += (i64)modulus;
      if (!(sampled > cdf_table[i])) to_output = (u64)out_val;
    }
    return to_output;
  }
};

template <typename R>
inline PolyMatrix random_raw(const Params& p, size_t rows, size_t cols, R& rng) {   // poly.rs:105-117
  PolyMatrix m = raw_zero(p, rows, cols);
  for (auto& x : m.data) x = rng.next() % p.modulus;
  return m;
}
inline PolyMatrix noise_raw(const Params& p, size_t rows, size_t cols, const DiscreteGaussian& dg, Rng& rng) {
  PolyMatrix m = raw_zero(p, rows, cols);
  for (auto& x : m.data) x = dg.sample(p.modulus, rng);
  return m;
}
inline PolyMatrix neg_raw(const Params& p, const PolyMatrix& a) {
  PolyMatrix r = raw_zero(p, a.rows, a.cols);
  invert(p, r, a);
  return r;
}
inline PolyMatrix single_poly(const Params& p, u64 val) {
  PolyMatrix r = raw_zero(p, 1, 1);
  r.data[0] = val;
  return r;
}
// client.rs:332-338
inline PolyMatrix matrix_with_identity(const Params& p, const PolyMatrix& m) {
  PolyMatrix r = raw_zero(p, m.rows, m.rows + 1);
  r.copy_into(m, 0, 0);
  for (size_t i = 0; i < m.rows; i++) r.poly(i, 1 + i)[0] = 1;
  return r;
}

struct Client {
  const Params& p;
  PolyMatrix sk_gsw, sk_reg, sk_gsw_full, sk_reg_full;
  DiscreteGaussian dg;
  Rng rng;                     // secret randomness (the reference: ChaCha20Rng::from_entropy, client.rs:547,626)
  ChaCha20Rng rng_pub;         // public randomness, regenerated by the server from the 32-byte seed (client.rs:551,631)
  Rng seeder;
  uint8_t pp_seed[32], query_seed[32];
  PublicParameters last_pp;
  PolyMatrix last_query_ct;
  Query last_query;             // the last generated query in full (direct-upload serialization needs v_buf / v_ct)
  Client(const Params& params, u64 seed)
      : p(params), sk_gsw(raw_zero(params, params.n, 1)), sk_reg(raw_zero(params, 1, 1)),
        dg(params.noise_width), rng(seed), seeder(seed ^ 0xA5A5A5A55A5A5A5AULL) {
    sk_gsw_full = matrix_with_identity(p, sk_gsw);
    sk_reg_full = matrix_with_identity(p, sk_reg);
    fresh_seed(pp_seed);
    rng_pub = ChaCha20Rng(pp_seed);
  }
  void fresh_seed(uint8_t out[32]) {
    for (int i = 0; i < 4; i++) { u64 v = seeder.next(); std::memcpy(out + 8 * i, &v, 8); }
  }
  // client.rs:130-144 (HAMMING_WEIGHT = 256, :13)
  void gen_ternary_mat(PolyMatrix& mat) {
    const size_t hamming = 256;
    for (size_t r = 0; r < mat.rows; r++)
      for (size_t c = 0; c < mat.cols; c++) {
        u64* pol = mat.poly(r, c);
        for (size_t i = 0; i < p.poly_len; i++) pol[i] = 0;
        for (size_t i = 0; i < hamming; i++) pol[i] = 1;
        for (size_t i = hamming; i < 2 * hamming; i++) pol[i] = p.modulus - 1;
        for (size_t i = p.poly_len; i-- > 1;) std::swap(pol[i], pol[rng.next() % (i + 1)]);
      }
  }
  // client.rs:419-449
  PolyMatrix get_regev_sample() {
    PolyMatrix a = random_raw(p, 1, 1, rng_pub);
    PolyMatrix e = noise_raw(p, 1, 1, dg, rng);
    PolyMatrix b_p = mul(p, to_ntt_alloc(p, sk_reg), to_ntt_alloc(p, a));
    PolyMatrix b = add_alloc(p, to_ntt_alloc(p, e), b_p);
    PolyMatrix out = ntt_zero(p, 2, 1);
    out.copy_into(to_ntt_alloc(p, neg_raw(p, a)), 0, 0);
    out.copy_into(b, 1, 0);
    return out;
  }
  PolyMatrix get_fresh_reg_public_key(size_t m) {
    PolyMatrix out = ntt_zero(p, 2, m);
    for (size_t i = 0; i < m; i++) out.copy_into(get_regev_sample(), 0, i);
    return out;
  }
  // client.rs:401-417
  PolyMatrix get_fresh_gsw_public_key(size_t m) {
    PolyMatrix a = random_raw(p, 1, m, rng_pub);
    PolyMatrix e = noise_raw(p, p.n, m, dg, rng);
    PolyMatrix a_inv = neg_raw(p, a);
    PolyMatrix b_p = mul(p, to_ntt_alloc(p, sk_gsw), to_ntt_alloc(p, a));
    PolyMatrix b = add_alloc(p, to_ntt_alloc(p, e), b_p);
    return stack(p, a_inv, from_ntt_alloc(p, b));
  }
  // client.rs:451-472
  PolyMatrix encrypt_matrix_gsw(const PolyMatrix& ag) {
    PolyMatrix pk = get_fresh_gsw_public_key(ag.cols);
    return add_alloc(p, to_ntt_alloc(p, pk), ag.pad_top(p, 1));
  }
  PolyMatrix encrypt_matrix_reg(const PolyMatrix& a) {
    PolyMatrix pk = get_fresh_reg_public_key(a.cols);
    return add_alloc(p, pk, a.pad_top(p, 1));
  }
  PolyMatrix decrypt_matrix_reg(const PolyMatrix& a) { return mul(p, to_ntt_alloc(p, sk_reg_full), a); }   // :474-476
  // client.rs:482-502
  std::vector<PolyMatrix> generate_expansion_params(size_t num_exp, size_t m_exp) {
    PolyMatrix g_exp_ntt = to_ntt_alloc(p, build_gadget(p, 1, m_exp));
    std::vector<PolyMatrix> res;
    for (size_t i = 0; i < num_exp; i++) {
      size_t t = (p.poly_len / ((size_t)1 << i)) + 1;
      PolyMatrix tau = raw_zero(p, 1, 1);
      automorph(p, tau, sk_reg, t);
      PolyMatrix prod = mul(p, to_ntt_alloc(p, tau), g_exp_ntt);
      res.push_back(encrypt_matrix_reg(prod));
    }
    return res;
  }
  // client.rs:533-616
  PublicParameters generate_keys() {
    fresh_seed(pp_seed);
    rng_pub = ChaCha20Rng(pp_seed);
    gen_ternary_mat(sk_gsw);
    gen_ternary_mat(sk_reg);
    sk_gsw_full = matrix_with_identity(p, sk_gsw);
    sk_reg_full = matrix_with_identity(p, sk_reg);
    PolyMatrix sk_reg_ntt = to_ntt_alloc(p, sk_reg), sk_gsw_ntt = to_ntt_alloc(p, sk_gsw);
    PublicParameters pp;
    PolyMatrix gadget_conv_ntt = to_ntt_alloc(p, build_gadget(p, 1, p.t_conv));
    size_t num_packing = p.version == 0 ? p.n : 1;
    for (size_t i = 0; i < num_packing; i++) {
      PolyMatrix scaled = ntt_zero(p, 1, p.t_conv);
      scalar_multiply(p, scaled, sk_reg_ntt, gadget_conv_ntt);
      PolyMatrix ag = ntt_zero(p, p.n, p.t_conv);
      ag.copy_into(scaled, i, 0);
      pp.v_packing.push_back(encrypt_matrix_gsw(ag));
    }
    if (p.version > 0) {
      PolyMatrix scaled = mul(p, sk_gsw_ntt, gadget_conv_ntt);
      pp.v_packing.push_back(encrypt_matrix_gsw(shift_rows_by_one(p, scaled)));
    }
    if (p.expand_queries) {
      pp.v_expansion_left = generate_expansion_params(p.g(), p.t_exp_left);
      if (p.version == 0 || p.t_exp_right != p.t_exp_left) {
        pp.v_expansion_right = generate_expansion_params(p.stop_round() + 1, p.t_exp_right);
        pp.has_right = true;
      }
      PolyMatrix g_conv = build_gadget(p, 2, 2 * p.t_conv);
      PolyMatrix sk_sq = mul(p, sk_reg_ntt, sk_reg_ntt);
      PolyMatrix conv = ntt_zero(p, 2, 2 * p.t_conv);
      for (size_t i = 0; i < 2 * p.t_conv; i++) {
        PolyMatrix sigma;
        if (i % 2 == 0) sigma = mul(p, sk_sq, to_ntt_alloc(p, single_poly(p, g_conv.poly(0, i)[0])));
        else sigma = mul(p, sk_reg_ntt, to_ntt_alloc(p, single_poly(p, g_conv.poly(1, i)[0])));
        conv.copy_into(encrypt_matrix_reg(sigma), 0, i);
      }
      pp.v_conversion.push_back(conv);
    }
    last_pp = pp;
    return pp;
  }
  // client.rs:618-721
  Query generate_query(size_t idx_target) {
    size_t further_dims = p.db_dim_2;
    size_t idx_dim0 = idx_target / ((size_t)1 << further_dims);
    size_t idx_further = idx_target % ((size_t)1 << further_dims);
    u64 scale_k = p.modulus / p.pt_modulus;
    size_t bits_per = get_bits_per(p, p.t_gsw);
    fresh_seed(query_seed);
    rng_pub = ChaCha20Rng(query_seed);
    Query q;
    if (p.expand_queries) {
      PolyMatrix sigma = raw_zero(p, 1, 1);
      u64 inv_first = 0, inv_rest = 0;
      invert_uint_mod((u64)1 << p.g(), p.modulus, inv_first);
      invert_uint_mod((u64)1 << (p.stop_round() + 1), p.modulus, inv_rest);
      if (p.db_dim_2 == 0) {
        for (size_t i = 0; i < ((size_t)1 << p.db_dim_1); i++) if (i == idx_dim0) sigma.data[i] = scale_k;
        for (size_t i = 0; i < p.poly_len; i++) sigma.data[i] = multiply_uint_mod(sigma.data[i], inv_first, p.modulus);
      } else {
        for (size_t i = 0; i < ((size_t)1 << p.db_dim_1); i++) if (i == idx_dim0) sigma.data[2 * i] = scale_k;
        for (size_t i = 0; i < further_dims; i++) {
          u64 mask = (u64)1 << i;
          bool bit = ((u64)idx_further & mask) == mask;
          for (size_t j = 0; j < p.t_gsw; j++) {
            size_t idx = i * p.t_gsw + j;
            sigma.data[2 * idx + 1] = bit ? ((u64)1 << (bits_per * j)) : 0;
          }
        }
        for (size_t i = 0; i < p.poly_len / 2; i++) {
          sigma.data[2 * i] = multiply_uint_mod(sigma.data[2 * i], inv_first, p.modulus);
          sigma.data[2 * i + 1] = multiply_uint_mod(sigma.data[2 * i + 1], inv_rest, p.modulus);
        }
      }
      q.ct = from_ntt_alloc(p, encrypt_matrix_reg(to_ntt_alloc(p, sigma)));
      last_query_ct = q.ct;
    } else {
      size_t num_expanded = (size_t)1 << p.db_dim_1;
      std::vector<PolyMatrix> reg_cts;
      for (size_t i = 0; i < num_expanded; i++) {
        u64 value = (i == idx_dim0) ? scale_k : 0;
        reg_cts.push_back(encrypt_matrix_reg(to_ntt_alloc(p, single_poly(p, value))));
      }
      q.v_buf.assign(num_expanded * 2 * p.poly_len, 0);
      reorient_reg_ciphertexts(p, q.v_buf.data(), reg_cts);
      for (size_t i = 0; i < further_dims; i++) {
        u64 bit = ((u64)idx_further >> i) & 1;
        PolyMatrix ct_gsw = ntt_zero(p, 2, 2 * p.t_gsw);
        for (size_t j = 0; j < p.t_gsw; j++) {
          u64 value = ((u64)1 << (bits_per * j)) * bit;
          PolyMatrix sigma_ntt = to_ntt_alloc(p, single_poly(p, value));
          PolyMatrix prod = mul(p, to_ntt_alloc(p, sk_reg), sigma_ntt);
          ct_gsw.copy_into(encrypt_matrix_reg(prod), 0, 2 * j);
          ct_gsw.copy_into(encrypt_matrix_reg(sigma_ntt), 0, 2 * j + 1);
        }
        q.v_ct.push_back(from_ntt_alloc(p, ct_gsw));
      }
    }
    last_query = q;
    return q;
  }
  // client.rs:732-810.  Returns the decoded (instances*n) x n plaintext matrix (mod p), i.e.
  // `result` before `to_vec` (:809).  `numer` (optional, same shape): the numerator each coefficient is rounded from,
  // val_first * q1 + val_rest * q2 (:780-800); the coefficient is that divided by q2 * (q1 / p), rounded half away from zero.
  PolyMatrix decode_response_poly(const uint8_t* data, int64_t* numer = nullptr) {
    u64 pm = p.pt_modulus;
    u64 q1 = 4 * p.pt_modulus;
    size_t q1_bits = log2_ceil(q1);
    u64 q2 = Q2_VALUES[p.q2_bits];
    size_t q2_bits = p.q2_bits;
    Params q2p = params_init(p.poly_len, {q2}, p.noise_width, p.n, p.pt_modulus, p.q2_bits, p.t_conv, p.t_exp_left,
                             p.t_exp_right, p.t_gsw, p.expand_queries, p.db_dim_1, p.db_dim_2, p.instances,
                             p.db_item_size, p.version);
    PolyMatrix sk_q2 = raw_zero(q2p, p.n, 1);
    for (size_t i = 0; i < p.poly_len * p.n; i++) sk_q2.data[i] = recenter(sk_gsw.data[i], p.modulus, q2);
    PolyMatrix sk_q2_ntt = to_ntt_alloc(q2p, sk_q2);
    PolyMatrix result = raw_zero(p, p.instances * p.n, p.n);
    size_t bit_offs = 0;
    size_t N = p.poly_len;
    for (size_t inst = 0; inst < p.instances; inst++) {
      PolyMatrix first_row = raw_zero(q2p, 1, p.n);
      PolyMatrix rest_rows = raw_zero(p, p.n, p.n);
      for (size_t i = 0; i < p.n * N; i++) { first_row.data[i] = read_arbitrary_bits(data, bit_offs, q2_bits); bit_offs += q2_bits; }
      for (size_t i = 0; i < p.n * p.n * N; i++) { rest_rows.data[i] = read_arbitrary_bits(data, bit_offs, q1_bits); bit_offs += q1_bits; }
      PolyMatrix first_ntt = to_ntt_alloc(q2p, first_row);
      PolyMatrix sk_prod = from_ntt_alloc(q2p, mul(q2p, sk_q2_ntt, first_ntt));
      i64 q1_i = (i64)q1, q2_i = (i64)q2;
      i128 p_i = (i128)pm;
      for (size_t i = 0; i < p.n * p.n * N; i++) {
        i64 val_first = (i64)sk_prod.data[i];
        if (val_first >= q2_i / 2) val_first -= q2_i;
        i64 val_rest = (i64)rest_rows.data[i];
        if (val_rest >= q1_i / 2) val_rest -= q1_i;
        i64 denom = (i64)(q2 * (q1 / pm));
        i64 r = val_first * q1_i + val_rest * q2_i;
        if (numer) numer[inst * p.n * p.n * N + i] = r;
        i64 sign = r >= 0 ? 1 : -1;
        i128 res = ((i128)(r + sign * (denom / 2))) / (i128)denom;
        res = (res + ((i128)denom / p_i) * p_i + 2 * p_i) % p_i;
        result.data[inst * p.n * p.n * N + i] = (u64)res;
      }
    }
    return result;
  }
};

// poly.rs:213-235 (PolyMatrixRaw::to_vec)
inline std::vector<uint8_t> raw_to_vec(const Params& p, const PolyMatrix& m, size_t modulus_bits, size_t num_coeffs) {
  size_t sz_bits = m.rows * m.cols * num_coeffs * modulus_bits;
  size_t sz_bytes = (sz_bits + 7) / 8 + 32;
  size_t rounded = ((sz_bytes + 15) / 16) * 16;
  std::vector<uint8_t> data(rounded, 0);
  size_t bit_offs = 0;
  for (size_t r = 0; r < m.rows; r++)
    for (size_t c = 0; c < m.cols; c++) {
      for (size_t z = 0; z < num_coeffs; z++) {
        write_arbitrary_bits(data.data(), m.poly(r, c)[z], bit_offs, modulus_bits);
        bit_offs += modulus_bits;
      }
      bit_offs = (bit_offs / 8) * 8;
    }
  return data;
}

// server.rs:223-275 with a seeded counter PRNG instead of the reference's unseeded SmallRng.
// Plaintext coefficient (instance,trial,item i, z) = splitmix64(seed, index) % p — the same
// generator the GPU-side DB loader uses, so full-size DBs never have to be built on the CPU.
inline u64 splitmix64_at(u64 seed, u64 index) {
  u64 z = seed + (index + 1) * 0x9E3779B97F4A7C15ULL;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL;
  return z ^ (z >> 31);
}
inline u64 db_plain_coeff(const Params& p, u64 seed, size_t slice, size_t item, size_t z) {
  u64 index = ((u64)slice * p.num_items() + item) * p.poly_len + z;
  return splitmix64_at(seed, index) % p.pt_modulus;
}
inline void generate_db(const Params& p, u64 seed, u64* db /* [slices][z][ii][j] */) {
  size_t trials = p.n * p.n, dim0 = (size_t)1 << p.db_dim_1, num_per = (size_t)1 << p.db_dim_2;
  size_t num_items = dim0 * num_per, N = p.poly_len;
  for (size_t slice = 0; slice < p.instances * trials; slice++) {
#pragma omp parallel for schedule(static)
    for (size_t i = 0; i < num_items; i++) {
      size_t ii = i % num_per, j = i / num_per;
      PolyMatrix item = raw_zero(p, 1, 1);
      for (size_t z = 0; z < N; z++)
        item.data[z] = recenter_mod(db_plain_coeff(p, seed, slice, i, z), p.pt_modulus, p.modulus);
      PolyMatrix nt = to_ntt_alloc(p, item);
      for (size_t z = 0; z < N; z++)
        db[((slice * N + z) * num_per + ii) * dim0 + j] = nt.data[z] | (nt.data[N + z] << 32);
    }
  }
}

// ---- wire formats (client.rs:47-93, 198-259, 279-329)
inline void ser_matrix_excl_first_row(std::vector<uint8_t>& out, const Params& p, const PolyMatrix& raw) {   // :55-60
  size_t offs = raw.cols * p.poly_len, cnt = (raw.rows - 1) * raw.cols * p.poly_len;
  size_t pos = out.size();
  out.resize(pos + cnt * 8);
  std::memcpy(out.data() + pos, raw.data.data() + offs, cnt * 8);
}
inline std::vector<uint8_t> serialize_pp(const Params& p, const PublicParameters& pp, const uint8_t seed[32]) {  // :198-210
  std::vector<uint8_t> out(seed, seed + 32);
  for (auto& m : pp.v_packing) ser_matrix_excl_first_row(out, p, from_ntt_alloc(p, m));
  for (auto& m : pp.v_expansion_left) ser_matrix_excl_first_row(out, p, from_ntt_alloc(p, m));
  if (pp.has_right) for (auto& m : pp.v_expansion_right) ser_matrix_excl_first_row(out, p, from_ntt_alloc(p, m));
  for (auto& m : pp.v_conversion) ser_matrix_excl_first_row(out, p, from_ntt_alloc(p, m));
  return out;
}
inline size_t deser_matrix_rng(const Params& p, PolyMatrix& a, const uint8_t* data, ChaCha20Rng& rng) {   // :68-80
  size_t first = a.cols * p.poly_len;
  for (size_t i = 0; i < first; i++) a.data[i] = p.modulus - (rng.next() % p.modulus);            // get_inv_from_rng :47-49
  size_t rest = (a.rows - 1) * a.cols * p.poly_len;
  std::memcpy(a.data.data() + first, data, rest * 8);
  return rest * 8;
}
inline PublicParameters deserialize_pp(const Params& p, const uint8_t* data, size_t len) {   // :212-259
  if (len != p.setup_bytes()) throw std::runtime_error("setup data has the wrong length");
  ChaCha20Rng rng(data);
  size_t idx = 32;
  PublicParameters pp;
  auto take = [&](std::vector<PolyMatrix>& dst, size_t count, size_t rows, size_t cols) {
    for (size_t i = 0; i < count; i++) {
      PolyMatrix raw = raw_zero(p, rows, cols);
      idx += deser_matrix_rng(p, raw, data + idx, rng);
      dst.push_back(to_ntt_alloc(p, raw));
    }
  };
  take(pp.v_packing, p.n, p.n + 1, p.t_conv);                 // :221 (always params.n matrices)
  if (p.expand_queries) {
    take(pp.v_expansion_left, p.g(), 2, p.t_exp_left);
    if (p.version == 0 || p.t_exp_right != p.t_exp_left) { take(pp.v_expansion_right, p.stop_round() + 1, 2, p.t_exp_right); pp.has_right = true; }
    take(pp.v_conversion, 1, 2, 2 * p.t_conv);
  }
  return pp;
}
inline std::vector<uint8_t> serialize_query(const Params& p, const PolyMatrix& ct, const uint8_t seed[32]) {   // :279-301
  std::vector<uint8_t> out(seed, seed + 32);
  ser_matrix_excl_first_row(out, p, ct);
  return out;
}
// direct upload (expand_queries == false), client.rs:279-301: seed || the odd-indexed words of v_buf (extract_excl_rng_data
// :97-105: the even-indexed ones are regenerated from the seed) || rows 1.. of every v_ct matrix
inline std::vector<uint8_t> serialize_query_direct(const Params& p, const Query& q, const uint8_t seed[32]) {
  std::vector<uint8_t> out(seed, seed + 32);
  for (size_t i = 1; i < q.v_buf.size(); i += 2) {
    const uint8_t* w = reinterpret_cast<const uint8_t*>(&q.v_buf[i]);
    out.insert(out.end(), w, w + 8);
  }
  for (auto& m : q.v_ct) ser_matrix_excl_first_row(out, p, m);
  return out;
}
// client.rs:316-327 with interleave_rng_data (:107-131): for every first-dimension ciphertext the row 0 polynomial is
// q - (rng % q) per coefficient (row 1 stays zero), transformed and reoriented; its packed words are the even-indexed words
// of v_buf, the uploaded words the odd-indexed ones.  Then the v_ct matrices, first rows from the same stream.
inline Query deserialize_query_direct(const Params& p, const uint8_t* data, size_t len) {
  if (len != p.query_bytes()) throw std::runtime_error("query has the wrong length");
  if (p.expand_queries) throw std::runtime_error("expansion-mode queries are handled by deserialize_query");
  ChaCha20Rng rng(data);
  const size_t num_expanded = (size_t)1 << p.db_dim_1, N = p.poly_len;
  const size_t v_buf_words = num_expanded * N;                                              // query_v_buf_bytes / 8, params.rs:184-186
  std::vector<PolyMatrix> reg_cts;
  for (size_t j = 0; j < num_expanded; j++) {
    PolyMatrix sigma = raw_zero(p, 2, 1);
    for (size_t z = 0; z < N; z++) sigma.data[z] = p.modulus - (rng.next() % p.modulus);
    reg_cts.push_back(to_ntt_alloc(p, sigma));
  }
  std::vector<u64> reg_buf(num_expanded * 2 * N, 0);
  reorient_reg_ciphertexts(p, reg_buf.data(), reg_cts);
  Query q;
  q.v_buf.resize(2 * v_buf_words);
  for (size_t i = 0; i < v_buf_words; i++) {
    q.v_buf[2 * i] = reg_buf[2 * i];
    std::memcpy(&q.v_buf[2 * i + 1], data + 32 + 8 * i, 8);
  }
  size_t idx = 32 + 8 * v_buf_words;
  for (size_t i = 0; i < p.db_dim_2; i++) {
    PolyMatrix m = raw_zero(p, 2, 2 * p.t_gsw);
    idx += deser_matrix_rng(p, m, data + idx, rng);
    q.v_ct.push_back(m);
  }
  return q;
}
inline PolyMatrix deserialize_query(const Params& p, const uint8_t* data, size_t len) {   // :303-315 (expand_queries)
  if (len != p.query_bytes()) throw std::runtime_error("query has the wrong length");
  if (!p.expand_queries) throw std::runtime_error("direct-upload queries are not handled here");
  ChaCha20Rng rng(data);
  PolyMatrix ct = raw_zero(p, 2, 1);
  deser_matrix_rng(p, ct, data + 32, rng);
  return ct;
}

// lib/server/src/db/loading.rs:278-299 convert_pt_to_poly (+ :34-41 pack_ntt_poly) and :317-359 update_item_raw:
// the bucket bytes are zero-padded to instances*n^2 chunks of bytes_per_chunk; chunk c becomes the item polynomial of
// slice c (coefficient i = byte i, recentred mod q, NTT'd, packed lo | hi << 32).  out: [slices][poly_len].
inline void update_item_raw(const Params& p, const uint8_t* data, size_t len, u64* out) {
  if (log2_ceil(p.pt_modulus) != 8) throw std::runtime_error("convert_pt_to_poly asserts logp == 8");
  size_t chunks = p.instances * p.n * p.n, pt_len = p.bytes_per_chunk(), N = p.poly_len;
  if (len > chunks * pt_len) throw std::runtime_error("update too long");
  if (pt_len > N) throw std::runtime_error("chunk longer than poly_len");
  std::vector<uint8_t> bucket(chunks * pt_len, 0);
  std::memcpy(bucket.data(), data, len);
  for (size_t c = 0; c < chunks; c++) {
    PolyMatrix item = raw_zero(p, 1, 1);
    for (size_t i = 0; i < pt_len; i++) item.data[i] = recenter_mod(bucket[c * pt_len + i], p.pt_modulus, p.modulus);
    PolyMatrix nt = to_ntt_alloc(p, item);
    for (size_t z = 0; z < N; z++) out[c * N + z] = nt.data[z] | (nt.data[N + z] << 32);
  }
}

// lib/spiral-rs/src/server.rs:277-357 load_item_from_seek + load_db_from_seek (twin: lib/server/src/db/loading.rs:192-247) over
// an in-memory image of the file: item i, chunk c = instance * n^2 + trial starts at byte i * db_item_size + c * bytes_per_chunk
// and is bytes_per_chunk long, clipped at the end of the file (NOT at the end of the item: when db_item_size is not a
// multiple of the chunk count the last chunk of an item runs into the next item, as in the reference).  logp == 8 here, so
// read_arbitrary_bits(data, i * 8, 8) is byte i.  db: [instance][trial][z][ii][j], packed lo | hi << 32.
inline void load_db_from_bytes(const Params& p, const uint8_t* file, size_t len, u64* db) {
  if (log2_ceil(p.pt_modulus) != 8) throw std::runtime_error("load_item_from_seek: only logp == 8 is restated");
  const size_t chunks = p.instances * p.n * p.n, bpc = p.bytes_per_chunk(), N = p.poly_len;
  if (bpc > N) throw std::runtime_error("chunk longer than poly_len");                 // server.rs:292
  const size_t dim0 = (size_t)1 << p.db_dim_1, num_per = (size_t)1 << p.db_dim_2, num_items = dim0 * num_per;
#pragma omp parallel for schedule(dynamic)
  for (size_t idx = 0; idx < chunks * num_items; idx++) {
    const size_t c = idx / num_items, i = idx % num_items, ii = i % num_per, j = i / num_per;
    const size_t pos = i * p.db_item_size + c * bpc;
    const size_t got = pos < len ? std::min(bpc, len - pos) : 0;
    PolyMatrix item = raw_zero(p, 1, 1);
    for (size_t k = 0; k < got; k++) item.data[k] = file[pos + k];
    for (size_t z = 0; z < N; z++) item.data[z] = recenter_mod(item.data[z], p.pt_modulus, p.modulus);
    PolyMatrix nt = to_ntt_alloc(p, item);
    for (size_t z = 0; z < N; z++) db[((c * N + z) * num_per + ii) * dim0 + j] = nt.data[z] | (nt.data[N + z] << 32);
  }
}

}  // namespace orc
