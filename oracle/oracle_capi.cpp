// ORACLE — TEST INFRASTRUCTURE ONLY (see spiral_oracle.hpp).  extern "C" surface so that
// tests/ and bench.py's cpu_baseline leg can drive the CPU restatement through ctypes.
#include "spiral_oracle.hpp"
#include "spiral_client.hpp"
#include "dpir_oracle.hpp"
#include <string>
#include <chrono>
#ifdef _OPENMP
#include <omp.h>
#endif

using namespace orc;

static thread_local std::string g_err;
#define ORC_TRY try {
#define ORC_CATCH } catch (const std::exception& e) { g_err = e.what(); return -1; } return 0;

static PolyMatrix load_mat(const Params& p, const u64* src, size_t rows, size_t cols, bool ntt) {
  PolyMatrix m(p, rows, cols, ntt);
  std::memcpy(m.data.data(), src, m.data.size() * 8);
  return m;
}
static std::vector<PolyMatrix> load_vec(const Params& p, const u64* src, size_t count, size_t rows, size_t cols, bool ntt) {
  std::vector<PolyMatrix> v;
  if (!src) return v;
  size_t words = rows * cols * (ntt ? p.crt_count * p.poly_len : p.poly_len);
  for (size_t i = 0; i < count; i++) v.push_back(load_mat(p, src + i * words, rows, cols, ntt));
  return v;
}
static void store_vec(u64* dst, const std::vector<PolyMatrix>& v) {
  size_t off = 0;
  for (auto& m : v) { std::memcpy(dst + off, m.data.data(), m.data.size() * 8); off += m.data.size(); }
}
static size_t num_packing(const Params& p) { return p.version == 0 ? p.n : 2; }
static PublicParameters load_pp(const Params& p, const u64* pack, const u64* left, const u64* right, const u64* conv) {
  PublicParameters pp;
  pp.v_packing = load_vec(p, pack, num_packing(p), p.n + 1, p.t_conv, true);
  if (p.expand_queries) {
    pp.v_expansion_left = load_vec(p, left, p.g(), 2, p.t_exp_left, true);
    if (right) { pp.v_expansion_right = load_vec(p, right, p.stop_round() + 1, 2, p.t_exp_right, true); pp.has_right = true; }
    pp.v_conversion = load_vec(p, conv, 1, 2, 2 * p.t_conv, true);
  }
  return pp;
}

extern "C" {

const char* orc_last_error() { return g_err.c_str(); }
int orc_num_threads() {
#ifdef _OPENMP
  return omp_get_max_threads();
#else
  return 1;
#endif
}
void orc_set_num_threads(int n) {
#ifdef _OPENMP
  omp_set_num_threads(n);
#else
  (void)n;
#endif
}

void* orc_params_new(uint64_t n, uint64_t nu_1, uint64_t nu_2, uint64_t p, uint64_t q2_bits, uint64_t t_gsw,
                     uint64_t t_conv, uint64_t t_exp_left, uint64_t t_exp_right, uint64_t instances,
                     uint64_t db_item_size, uint64_t version, int expand_queries) {
  try {
    return new Params(params_from_scalars(n, nu_1, nu_2, p, q2_bits, t_gsw, t_conv, t_exp_left, t_exp_right, instances,
                                          db_item_size, version, expand_queries != 0));
  } catch (const std::exception& e) { g_err = e.what(); return nullptr; }
}
// generic single/multi-modulus params (used for the q2 NTT KAT and poly_len sweeps)
void* orc_params_new_raw(uint64_t poly_len, const uint64_t* moduli, uint64_t nmod) {
  try {
    std::vector<u64> m(moduli, moduli + nmod);
    return new Params(params_init(poly_len, m, 6.4, 2, 256, 20, 4, 8, 8, 8, true, 6, 2, 1, 8192, 0));
  } catch (const std::exception& e) { g_err = e.what(); return nullptr; }
}
void orc_params_free(void* h) { delete (Params*)h; }

// out[0..] = poly_len, crt_count, q0, q1, modulus, modulus_log2, cr0[0], cr1[0], cr0[1], cr1[1], cr0_mod, cr1_mod,
//            mod0_inv_mod1, mod1_inv_mod0, g, stop_round, setup_bytes, query_bytes, bytes_per_chunk, modp_words_per_chunk
int orc_params_info(void* h, uint64_t* out) {
  ORC_TRY
  const Params& p = *(Params*)h;
  u64 v[] = {p.poly_len, p.crt_count, p.moduli[0], p.moduli[1], p.modulus, p.modulus_log2, p.barrett_cr_0[0],
             p.barrett_cr_1[0], p.barrett_cr_0[1], p.barrett_cr_1[1], p.barrett_cr_0_modulus, p.barrett_cr_1_modulus,
             p.mod0_inv_mod1, p.mod1_inv_mod0, p.g(), p.stop_round(), p.setup_bytes(), p.query_bytes(),
             p.bytes_per_chunk(), p.modp_words_per_chunk()};
  std::memcpy(out, v, sizeof(v));
  ORC_CATCH
}
int orc_ntt_table(void* h, int mod, int which, uint64_t* out) {
  ORC_TRY
  const Params& p = *(Params*)h;
  std::memcpy(out, p.ntt_tables.at(mod).at(which).data(), p.poly_len * 8);
  ORC_CATCH
}
int orc_ntt_forward(void* h, uint64_t* data, size_t count) {
  ORC_TRY
  const Params& p = *(Params*)h;
  size_t W = p.crt_count * p.poly_len;
#pragma omp parallel for schedule(static)
  for (size_t i = 0; i < count; i++) ntt_forward(p, data + i * W);
  ORC_CATCH
}
int orc_ntt_inverse(void* h, uint64_t* data, size_t count) {
  ORC_TRY
  const Params& p = *(Params*)h;
  size_t W = p.crt_count * p.poly_len;
#pragma omp parallel for schedule(static)
  for (size_t i = 0; i < count; i++) ntt_inverse(p, data + i * W);
  ORC_CATCH
}
int orc_to_ntt(void* h, uint64_t* out, const uint64_t* in, size_t npolys, int no_reduce) {
  ORC_TRY
  const Params& p = *(Params*)h;
  PolyMatrix b = load_mat(p, in, npolys, 1, false), a = ntt_zero(p, npolys, 1);
  if (no_reduce) to_ntt_no_reduce(p, a, b); else to_ntt(p, a, b);
  std::memcpy(out, a.data.data(), a.data.size() * 8);
  ORC_CATCH
}
int orc_from_ntt(void* h, uint64_t* out, const uint64_t* in, size_t npolys) {
  ORC_TRY
  const Params& p = *(Params*)h;
  PolyMatrix b = load_mat(p, in, npolys, 1, true), a = raw_zero(p, npolys, 1);
  from_ntt(p, a, b);
  std::memcpy(out, a.data.data(), a.data.size() * 8);
  ORC_CATCH
}
int orc_multiply(void* h, uint64_t* out, const uint64_t* a, const uint64_t* b, size_t ar, size_t ac, size_t bc) {
  ORC_TRY
  const Params& p = *(Params*)h;
  PolyMatrix r = mul(p, load_mat(p, a, ar, ac, true), load_mat(p, b, ac, bc, true));
  std::memcpy(out, r.data.data(), r.data.size() * 8);
  ORC_CATCH
}
int orc_gadget_invert(void* h, uint64_t* out, const uint64_t* in, size_t in_rows, size_t in_cols, size_t out_rows, size_t rdim) {
  ORC_TRY
  const Params& p = *(Params*)h;
  PolyMatrix o = raw_zero(p, out_rows, in_cols);
  gadget_invert_rdim(p, o, load_mat(p, in, in_rows, in_cols, false), rdim);
  std::memcpy(out, o.data.data(), o.data.size() * 8);
  ORC_CATCH
}
int orc_build_gadget(void* h, uint64_t* out, size_t rows, size_t cols) {
  ORC_TRY
  const Params& p = *(Params*)h;
  PolyMatrix g = build_gadget(p, rows, cols);
  std::memcpy(out, g.data.data(), g.data.size() * 8);
  ORC_CATCH
}
uint64_t orc_get_bits_per(void* h, size_t dim) { return get_bits_per(*(Params*)h, dim); }
int orc_automorph(void* h, uint64_t* out, const uint64_t* in, size_t rows, size_t t) {
  ORC_TRY
  const Params& p = *(Params*)h;
  PolyMatrix o = raw_zero(p, rows, 1);
  automorph(p, o, load_mat(p, in, rows, 1, false), t);
  std::memcpy(out, o.data.data(), o.data.size() * 8);
  ORC_CATCH
}

// ---- scalar KAT helpers
void orc_barrett_crs(uint64_t m, uint64_t* out2) { get_barrett_crs(m, out2[0], out2[1]); }
uint64_t orc_barrett_reduction_u128_raw(uint64_t m, uint64_t cr0, uint64_t cr1, uint64_t lo, uint64_t hi) {
  return barrett_reduction_u128_raw(m, cr0, cr1, ((u128)hi << 64) | lo);
}
uint64_t orc_barrett_raw_u64(uint64_t v, uint64_t cr1, uint64_t m) { return barrett_raw_u64(v, cr1, m); }
uint64_t orc_div2_uint_mod(uint64_t a, uint64_t m) { return div2_uint_mod(a, m); }
uint64_t orc_calc_index(const uint64_t* idx, const uint64_t* len, uint64_t n) {
  std::vector<size_t> a(idx, idx + n), b(len, len + n);
  return calc_index(a.data(), b.data(), n);
}
uint64_t orc_rescale(uint64_t a, uint64_t in_mod, uint64_t out_mod) { return rescale(a, in_mod, out_mod); }
uint64_t orc_recenter_mod(uint64_t a, uint64_t s, uint64_t l) { return recenter_mod(a, s, l); }
uint64_t orc_min_primitive_root(uint64_t degree, uint64_t m) { u64 r = 0; get_minimal_primitive_root(degree, m, r); return r; }
uint64_t orc_invert_uint_mod(uint64_t v, uint64_t m) { u64 r = 0; invert_uint_mod(v, m, r); return r; }
void orc_write_bits(uint8_t* data, uint64_t val, size_t bit_offs, size_t num_bits) { write_arbitrary_bits(data, val, bit_offs, num_bits); }
uint64_t orc_read_bits(const uint8_t* data, size_t bit_offs, size_t num_bits) { return read_arbitrary_bits(data, bit_offs, num_bits); }

// ---- pipeline stages
int orc_multiply_reg_by_database(void* h, uint64_t* out, const uint64_t* db_slice, const uint64_t* v_firstdim) {
  ORC_TRY
  const Params& p = *(Params*)h;
  multiply_reg_by_database(p, out, db_slice, v_firstdim, (size_t)1 << p.db_dim_1, (size_t)1 << p.db_dim_2);
  ORC_CATCH
}
// generic-shape variant (dim0 / num_per given explicitly; bench samples a sub-range of rows)
int orc_multiply_reg_by_database_shape(void* h, uint64_t* out, const uint64_t* db_slice, const uint64_t* v_firstdim,
                                       size_t dim0, size_t num_per) {
  ORC_TRY
  multiply_reg_by_database(*(Params*)h, out, db_slice, v_firstdim, dim0, num_per);
  ORC_CATCH
}
int orc_fold_ciphertexts(void* h, uint64_t* v_cts, size_t num, const uint64_t* v_folding, const uint64_t* v_folding_neg,
                         int sparse) {
  ORC_TRY
  const Params& p = *(Params*)h;
  size_t dims = num > 1 ? log2_floor(num) : 0;
  std::vector<PolyMatrix> cts = load_vec(p, v_cts, num, 2, 1, false);
  std::vector<PolyMatrix> vf = load_vec(p, v_folding, dims, 2, 2 * p.t_gsw, true);
  std::vector<PolyMatrix> vfn = load_vec(p, v_folding_neg, dims, 2, 2 * p.t_gsw, true);
  fold_ciphertexts(p, cts, vf, vfn, sparse != 0);
  store_vec(v_cts, cts);
  ORC_CATCH
}
int orc_get_v_folding_neg(void* h, uint64_t* out, const uint64_t* v_folding) {
  ORC_TRY
  const Params& p = *(Params*)h;
  store_vec(out, get_v_folding_neg(p, load_vec(p, v_folding, p.db_dim_2, 2, 2 * p.t_gsw, true)));
  ORC_CATCH
}
int orc_expand_query(void* h, const uint64_t* left, const uint64_t* right, const uint64_t* conv, const uint64_t* query_ct,
                     uint64_t* out_v_firstdim, uint64_t* out_v_folding) {
  ORC_TRY
  const Params& p = *(Params*)h;
  PublicParameters pp = load_pp(p, nullptr, left, right, conv);
  std::vector<u64> vreg;
  std::vector<PolyMatrix> vf;
  expand_query(p, pp, load_mat(p, query_ct, 2, 1, false), vreg, vf);
  std::memcpy(out_v_firstdim, vreg.data(), vreg.size() * 8);
  store_vec(out_v_folding, vf);
  ORC_CATCH
}
// v: in/out 2^g NTT 2x1 ciphertexts
int orc_coefficient_expansion(void* h, uint64_t* v, const uint64_t* left, const uint64_t* right) {
  ORC_TRY
  const Params& p = *(Params*)h;
  size_t g = p.g();
  std::vector<PolyMatrix> vv = load_vec(p, v, (size_t)1 << g, 2, 1, true);
  std::vector<PolyMatrix> l = load_vec(p, left, g, 2, p.t_exp_left, true);
  std::vector<PolyMatrix> r = right ? load_vec(p, right, p.stop_round() + 1, 2, p.t_exp_right, true) : l;
  coefficient_expansion(p, vv, g, p.stop_round(), l, r, get_v_neg1(p), p.t_gsw * p.db_dim_2);
  store_vec(v, vv);
  ORC_CATCH
}
int orc_regev_to_gsw(void* h, uint64_t* out, const uint64_t* v_inp, size_t n_inp, const uint64_t* conv) {
  ORC_TRY
  const Params& p = *(Params*)h;
  std::vector<PolyMatrix> inp = load_vec(p, v_inp, n_inp, 2, 1, true);
  std::vector<PolyMatrix> gsw(n_inp / p.t_gsw, ntt_zero(p, 2, 2 * p.t_gsw));
  regev_to_gsw(p, gsw, inp, load_mat(p, conv, 2, 2 * p.t_conv, true), 1, 0);
  store_vec(out, gsw);
  ORC_CATCH
}
int orc_pack(void* h, uint64_t* out, const uint64_t* v_ct, const uint64_t* v_packing) {
  ORC_TRY
  const Params& p = *(Params*)h;
  std::vector<PolyMatrix> cts = load_vec(p, v_ct, p.n * p.n, 2, 1, false);
  std::vector<PolyMatrix> w = load_vec(p, v_packing, num_packing(p), p.n + 1, p.t_conv, true);
  PolyMatrix r = pack(p, cts.data(), w);
  std::memcpy(out, r.data.data(), r.data.size() * 8);
  ORC_CATCH
}
int orc_encode(void* h, uint8_t* out, size_t* out_len, const uint64_t* packed_raw) {
  ORC_TRY
  const Params& p = *(Params*)h;
  std::vector<PolyMatrix> v = load_vec(p, packed_raw, p.instances, p.n + 1, p.n, false);
  std::vector<uint8_t> b = encode(p, v);
  std::memcpy(out, b.data(), b.size());
  *out_len = b.size();
  ORC_CATCH
}
size_t orc_response_bytes(void* h) {
  const Params& p = *(Params*)h;
  size_t q1_bits = log2_ceil(4 * p.pt_modulus);
  size_t num_bits = p.instances * ((p.q2_bits * p.n * p.poly_len) + (q1_bits * p.n * p.n * p.poly_len));
  return ((num_bits + 63) / 64) * 8;
}
// Full dense process_query.  query_ct: raw 2x1 (expand) ; or v_buf + v_ct (direct upload).
// Optional dumps (may be NULL): v_firstdim, v_folding, v_folding_neg, first_mult (slice 0), folded (per slice), packed.
int orc_process_query(void* h, const uint64_t* pack, const uint64_t* left, const uint64_t* right, const uint64_t* conv,
                      const uint64_t* query_ct, const uint64_t* v_buf, const uint64_t* v_ct, const uint64_t* db,
                      uint8_t* out, size_t* out_len, uint64_t* d_v_firstdim, uint64_t* d_v_folding,
                      uint64_t* d_v_folding_neg, uint64_t* d_first_mult, uint64_t* d_folded, uint64_t* d_packed) {
  ORC_TRY
  const Params& p = *(Params*)h;
  PublicParameters pp = load_pp(p, pack, left, right, conv);
  Query q;
  if (p.expand_queries) q.ct = load_mat(p, query_ct, 2, 1, false);
  else {
    q.v_buf.assign(v_buf, v_buf + p.num_expanded() * 2 * p.poly_len);
    q.v_ct = load_vec(p, v_ct, p.db_dim_2, 2, 2 * p.t_gsw, false);
  }
  StageDump dump;
  std::vector<uint8_t> b = process_query(p, pp, q, db, &dump);
  std::memcpy(out, b.data(), b.size());
  *out_len = b.size();
  if (d_v_firstdim) std::memcpy(d_v_firstdim, dump.v_firstdim.data(), dump.v_firstdim.size() * 8);
  if (d_v_folding) store_vec(d_v_folding, dump.v_folding);
  if (d_v_folding_neg) store_vec(d_v_folding_neg, dump.v_folding_neg);
  if (d_first_mult) std::memcpy(d_first_mult, dump.first_mult.data(), dump.first_mult.size() * 8);
  if (d_folded) store_vec(d_folded, dump.folded);
  if (d_packed) store_vec(d_packed, dump.packed);
  ORC_CATCH
}

// ---- client (harness only)
void* orc_client_new(void* h, uint64_t seed) { return new Client(*(Params*)h, seed); }
void orc_client_free(void* c) { delete (Client*)c; }
// sizes (in u64 words) of the four pp arrays: pack, left, right (0 if absent), conv
int orc_pp_sizes(void* h, uint64_t* out4) {
  ORC_TRY
  const Params& p = *(Params*)h;
  size_t W = p.crt_count * p.poly_len;
  out4[0] = num_packing(p) * (p.n + 1) * p.t_conv * W;
  out4[1] = p.expand_queries ? p.g() * 2 * p.t_exp_left * W : 0;
  out4[2] = (p.expand_queries && (p.version == 0 || p.t_exp_right != p.t_exp_left)) ? (p.stop_round() + 1) * 2 * p.t_exp_right * W : 0;
  out4[3] = p.expand_queries ? 2 * 2 * p.t_conv * W : 0;
  ORC_CATCH
}
int orc_client_generate_keys(void* c, uint64_t* pack, uint64_t* left, uint64_t* right, uint64_t* conv) {
  ORC_TRY
  Client& cl = *(Client*)c;
  PublicParameters pp = cl.generate_keys();
  store_vec(pack, pp.v_packing);
  if (left) store_vec(left, pp.v_expansion_left);
  if (right && pp.has_right) store_vec(right, pp.v_expansion_right);
  if (conv) store_vec(conv, pp.v_conversion);
  ORC_CATCH
}
int orc_client_generate_query(void* c, uint64_t idx, uint64_t* query_ct, uint64_t* v_buf, uint64_t* v_ct) {
  ORC_TRY
  Client& cl = *(Client*)c;
  Query q = cl.generate_query(idx);
  if (cl.p.expand_queries) std::memcpy(query_ct, q.ct.data.data(), q.ct.data.size() * 8);
  else { std::memcpy(v_buf, q.v_buf.data(), q.v_buf.size() * 8); store_vec(v_ct, q.v_ct); }
  ORC_CATCH
}
// out: (instances*n) x n raw polys of plaintext coefficients mod p
int orc_client_decode_response(void* c, const uint8_t* data, size_t len, uint64_t* out) {
  ORC_TRY
  Client& cl = *(Client*)c;
  std::vector<uint8_t> buf(data, data + len);
  buf.resize(len + 16, 0);
  PolyMatrix r = cl.decode_response_poly(buf.data());
  std::memcpy(out, r.data.data(), r.data.size() * 8);
  ORC_CATCH
}
uint64_t orc_q2_value(size_t q2_bits) { return Q2_VALUES[q2_bits]; }
// out: the pre-rounding numerators of decode_response (client.rs:780-800), one int64 per coefficient of the
// (instances*n) x n result
int orc_client_decode_numerators(void* c, const uint8_t* data, size_t len, int64_t* out) {
  ORC_TRY
  Client& cl = *(Client*)c;
  std::vector<uint8_t> buf(data, data + len);
  buf.resize(len + 16, 0);
  cl.decode_response_poly(buf.data(), out);
  ORC_CATCH
}
// encrypt a raw 1x1 plaintext poly (already scaled) as a Regev ciphertext; returns NTT 2x1 (stage tests)
int orc_client_encrypt_reg(void* c, const uint64_t* sigma_raw, uint64_t* out_ntt) {
  ORC_TRY
  Client& cl = *(Client*)c;
  PolyMatrix ct = cl.encrypt_matrix_reg(to_ntt_alloc(cl.p, load_mat(cl.p, sigma_raw, 1, 1, false)));
  std::memcpy(out_ntt, ct.data.data(), ct.data.size() * 8);
  ORC_CATCH
}
// decrypt an NTT 2x1 Regev ciphertext -> raw 1x1 (mod q)
int orc_client_decrypt_reg(void* c, const uint64_t* ct_ntt, uint64_t* out_raw) {
  ORC_TRY
  Client& cl = *(Client*)c;
  PolyMatrix d = from_ntt_alloc(cl.p, cl.decrypt_matrix_reg(load_mat(cl.p, ct_ntt, 2, 1, true)));
  std::memcpy(out_raw, d.data.data(), d.data.size() * 8);
  ORC_CATCH
}
// ---- wire formats
void orc_chacha20_block(const uint32_t* init16, uint32_t* out16) { chacha20_block(init16, out16); }
// the generator the wire formats draw from: n consecutive next_u32() / next_u64() values of ChaCha20Rng::from_seed(seed)
void orc_chacha20rng_u32(const uint8_t* seed32, size_t n, uint32_t* out) { ChaCha20Rng r(seed32); for (size_t i = 0; i < n; i++) out[i] = r.next_u32(); }
void orc_chacha20rng_u64(const uint8_t* seed32, size_t n, uint64_t* out) { ChaCha20Rng r(seed32); for (size_t i = 0; i < n; i++) out[i] = r.next(); }
int orc_client_pp_bytes(void* c, uint8_t* out, size_t* out_len) {
  ORC_TRY
  Client& cl = *(Client*)c;
  std::vector<uint8_t> b = serialize_pp(cl.p, cl.last_pp, cl.pp_seed);
  std::memcpy(out, b.data(), b.size());
  *out_len = b.size();
  ORC_CATCH
}
int orc_client_query_bytes(void* c, uint8_t* out, size_t* out_len) {       // Query::serialize of the last generated query
  ORC_TRY
  Client& cl = *(Client*)c;
  std::vector<uint8_t> b = cl.p.expand_queries ? serialize_query(cl.p, cl.last_query_ct, cl.query_seed)
                                               : serialize_query_direct(cl.p, cl.last_query, cl.query_seed);
  std::memcpy(out, b.data(), b.size());
  *out_len = b.size();
  ORC_CATCH
}
int orc_query_deserialize_direct(void* h, const uint8_t* data, size_t len, uint64_t* v_buf, uint64_t* v_ct) {
  ORC_TRY
  const Params& p = *(Params*)h;
  Query q = deserialize_query_direct(p, data, len);
  std::memcpy(v_buf, q.v_buf.data(), q.v_buf.size() * 8);
  store_vec(v_ct, q.v_ct);
  ORC_CATCH
}
int orc_pp_deserialize(void* h, const uint8_t* data, size_t len, uint64_t* pack, uint64_t* left, uint64_t* right, uint64_t* conv) {
  ORC_TRY
  const Params& p = *(Params*)h;
  PublicParameters pp = deserialize_pp(p, data, len);
  store_vec(pack, pp.v_packing);
  if (left) store_vec(left, pp.v_expansion_left);
  if (right && pp.has_right) store_vec(right, pp.v_expansion_right);
  if (conv) store_vec(conv, pp.v_conversion);
  ORC_CATCH
}
int orc_query_deserialize(void* h, const uint8_t* data, size_t len, uint64_t* ct) {
  ORC_TRY
  const Params& p = *(Params*)h;
  PolyMatrix m = deserialize_query(p, data, len);
  std::memcpy(ct, m.data.data(), m.data.size() * 8);
  ORC_CATCH
}

int orc_generate_db(void* h, uint64_t seed, uint64_t* db) {
  ORC_TRY
  generate_db(*(Params*)h, seed, db);
  ORC_CATCH
}
// plaintext (mod p) of item `idx` as the (instances*n) x n matrix decode_response returns
int orc_db_plain_item(void* h, uint64_t seed, uint64_t idx, uint64_t* out) {
  ORC_TRY
  const Params& p = *(Params*)h;
  size_t trials = p.n * p.n, N = p.poly_len;
  for (size_t inst = 0; inst < p.instances; inst++)
    for (size_t trial = 0; trial < trials; trial++) {
      size_t row = inst * p.n + trial / p.n, col = trial % p.n;
      for (size_t z = 0; z < N; z++)
        out[(row * p.n + col) * N + z] = db_plain_coeff(p, seed, inst * trials + trial, idx, z);
    }
  ORC_CATCH
}
uint64_t orc_splitmix64_at(uint64_t seed, uint64_t index) { return splitmix64_at(seed, index); }
// lib/server/src/db/loading.rs:317-359: bucket bytes -> one packed item polynomial per slice
int orc_update_item_raw(void* h, const uint8_t* data, size_t len, uint64_t* out) {
  ORC_TRY
  update_item_raw(*(Params*)h, data, len, out);
  ORC_CATCH
}

int orc_load_db_from_bytes(void* h, const uint8_t* file, size_t len, uint64_t* db) {
  ORC_TRY
  load_db_from_bytes(*(Params*)h, file, len, db);
  ORC_CATCH
}

// ---- DoublePIR
int orc_dpir_matvec_packed(uint32_t* out, const uint32_t* a, const uint32_t* b, size_t rows, size_t cols) {
  ORC_TRY
  dpir::matrix_mul_vec_packed(out, a, b, rows, cols);
  ORC_CATCH
}

int orc_dpir_matrix_mul_transposed_packed(uint32_t* out, const uint32_t* a, const uint32_t* b, size_t a_rows, size_t a_cols,
                                          size_t b_rows, size_t b_cols) {
  ORC_TRY
  dpir::matrix_mul_transposed_packed(out, a, b, a_rows, a_cols, b_rows, b_cols);
  ORC_CATCH
}
// out must hold cols*delta*concat * ceil((rows/concat)/3) words
int orc_dpir_transpose_expand_concat_cols_squish(uint32_t* out, const uint32_t* a, size_t rows, size_t cols, uint64_t modulus,
                                                 size_t delta, size_t concat) {
  ORC_TRY
  std::vector<uint32_t> o;
  size_t r, c;
  dpir::transpose_expand_concat_cols_squish(o, r, c, a, rows, cols, modulus, delta, concat, 10, 3);
  std::memcpy(out, o.data(), o.size() * 4);
  ORC_CATCH
}

// BASELINE config #5 at poly_len = 4096: the same scalar transforms / table construction instantiated at the larger size
// (the reference's parameterisation stops at 2048, util.rs:246; both moduli are 1 mod 8192)
// DoublePIR offline setup (doublepir.rs:76-108).  Outputs (caller-allocated): db_sq l x ceil(m/3); h1_sq (n delta x) x ceil((l/x)/3);
// a2_t n x (l/x rounded up to a multiple of 3); h2 (n delta x) x n.
int orc_dpir_setup(const uint32_t* db, size_t l, size_t m, const uint32_t* a1, size_t n, const uint32_t* a2, uint32_t p,
                   size_t delta, size_t x, uint32_t* db_sq, uint32_t* h1_sq, uint32_t* a2_t, uint32_t* h2) {
  ORC_TRY
  dpir::Mat D(l, m), A1(m, n), A2(l / x, n);
  std::memcpy(D.data.data(), db, l * m * 4);
  std::memcpy(A1.data.data(), a1, m * n * 4);
  std::memcpy(A2.data.data(), a2, (l / x) * n * 4);
  dpir::SetupOut o = dpir::setup(D, A1, A2, p, delta, x);
  std::memcpy(db_sq, o.db_squished.data.data(), o.db_squished.data.size() * 4);
  std::memcpy(h1_sq, o.h1_squished.data.data(), o.h1_squished.data.size() * 4);
  std::memcpy(a2_t, o.a2_t.data.data(), o.a2_t.data.size() * 4);
  std::memcpy(h2, o.h2.data.data(), o.h2.data.size() * 4);
  ORC_CATCH
}
int orc_dpir_mul(uint32_t* out, const uint32_t* a, const uint32_t* b, size_t ar, size_t ac, size_t bc) {
  ORC_TRY
  dpir::Mat A(ar, ac), B(ac, bc);
  std::memcpy(A.data.data(), a, ar * ac * 4);
  std::memcpy(B.data.data(), b, ac * bc * 4);
  dpir::Mat C = dpir::mul(A, B);
  std::memcpy(out, C.data.data(), ar * bc * 4);
  ORC_CATCH
}

int orc_ntt4096(uint64_t* polys, size_t count, int inverse) {
  ORC_TRY
  static const Params p4k = params_init(4096, {268369921ULL, 249561089ULL}, 6.4, 2, 256, 20, 4, 8, 8, 8, true, 6, 2, 1, 8192, 0);
  for (size_t i = 0; i < count; i++) {
    if (inverse) ntt_inverse_scalar(p4k, polys + i * 2 * 4096);
    else ntt_forward_scalar(p4k, polys + i * 2 * 4096);
  }
  ORC_CATCH
}

// CPU-baseline switch: 1 = AVX2 transforms everywhere ntt_forward / ntt_inverse are called (bit-identical to the scalar ones)
int orc_use_avx2_ntt(int on) {
#if defined(__AVX2__)
  g_use_avx2_ntt = on != 0;
  return 1;
#else
  (void)on;
  return 0;
#endif
}
// direct entry points for the equality test
int orc_ntt_scalar(void* h, uint64_t* polys, size_t count, int inverse) {
  ORC_TRY
  const Params& p = *(Params*)h;
  for (size_t i = 0; i < count; i++) {
    if (inverse) ntt_inverse_scalar(p, polys + i * p.crt_count * p.poly_len);
    else ntt_forward_scalar(p, polys + i * p.crt_count * p.poly_len);
  }
  ORC_CATCH
}
int orc_ntt_avx2(void* h, uint64_t* polys, size_t count, int inverse) {
  ORC_TRY
#if defined(__AVX2__)
  const Params& p = *(Params*)h;
  for (size_t i = 0; i < count; i++) {
    if (inverse) ntt_inverse_avx2(p, polys + i * p.crt_count * p.poly_len);
    else ntt_forward_avx2(p, polys + i * p.crt_count * p.poly_len);
  }
#else
  (void)h; (void)polys; (void)count; (void)inverse;
  throw std::runtime_error("built without AVX2");
#endif
  ORC_CATCH
}

// 1: process_query uses lib/server's fold (all-zero ciphertext shortcut, lib/server/src/compute/fold.rs:37-43)
int orc_set_sparse_fold(int on) { g_sparse_fold = on != 0; return 0; }

// CPU-baseline switch: 1 = AVX2 first-dimension kernel inside process_query (returns 0 when not compiled with AVX2)
int orc_use_avx2_multiply(int on) {
#if defined(__AVX2__)
  g_use_avx2_multiply = on != 0;
  return 1;
#else
  (void)on;
  return 0;
#endif
}
int orc_multiply_reg_by_database_avx2(void* h, uint64_t* out, const uint64_t* db_slice, const uint64_t* v_firstdim,
                                      size_t dim0, size_t num_per) {
  ORC_TRY
#if defined(__AVX2__)
  multiply_reg_by_database_avx2(*(Params*)h, out, db_slice, v_firstdim, dim0, num_per);
#else
  throw std::runtime_error("built without AVX2");
#endif
  ORC_CATCH
}

// ---- timing helper for the CPU baseline: runs fn-equivalent loops natively, returns seconds
double orc_time_multiply(void* h, const uint64_t* db_slice, const uint64_t* v_firstdim, size_t dim0, size_t num_per,
                         uint64_t* out, int reps) {
  const Params& p = *(Params*)h;
  auto t0 = std::chrono::steady_clock::now();
  for (int r = 0; r < reps; r++) multiply_reg_by_database(p, out, db_slice, v_firstdim, dim0, num_per);
  return std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count() / reps;
}

}  // extern "C"
