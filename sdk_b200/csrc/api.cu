// C-ABI implementation (include/b200pir.h): contexts, public parameters and the host-side orchestration of
// spiral_rs::server::process_query (lib/spiral-rs/src/server.rs:650-741) as a stream of sm_90a kernel launches; the database
// handle is in db_api.cu.  No CPU fallback exists anywhere on this path: every entry point either runs on the GPU or returns
// an error.
#include "spiral_api.hpp"
#include "ntt_tables.hpp"
#include "gadget.hpp"
#include <atomic>
#include <cmath>
#include <memory>
#include <set>
#include <utility>

namespace b200pir {
thread_local unsigned long long g_kernel_launches = 0;
thread_local std::string g_last_error;

int fail(const std::exception& e) {
  cudaGetLastError();        // a failed runtime call leaves its code as the "last error": clear it, or the next entry point's check reports it
  g_last_error = e.what();
  const Error* pe = dynamic_cast<const Error*>(&e);
  return pe ? pe->code : B200PIR_E_CUDA;
}

void opt_in_smem_impl(const void* kernel, int bytes) {
  static std::mutex mu;
  static std::set<std::pair<const void*, int>> done;      // (kernel, device) pairs already opted in
  int dev = 0;
  B200_CUDA(cudaGetDevice(&dev));
  std::lock_guard<std::mutex> lk(mu);
  if (done.count({kernel, dev})) return;
  B200_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
  done.insert({kernel, dev});
}
}  // namespace b200pir

namespace {

using b200pir::tables::build_tables;
using b200pir::tables::invmod;
uint64_t log2_ceil_u64(uint64_t a) { return (uint64_t)std::ceil(std::log2((double)a)); }
using b200pir::bits_per;
using b200pir::live_digits;
const uint64_t kQ2Values[37] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 12289ULL, 12289ULL, 61441ULL, 65537ULL,
                                65537ULL, 520193ULL, 786433ULL, 786433ULL, 3604481ULL, 7340033ULL, 16515073ULL,
                                33292289ULL, 67043329ULL, 132120577ULL, 268369921ULL, 469762049ULL, 1073479681ULL,
                                2013265921ULL, 4293918721ULL, 8588886017ULL, 17175674881ULL, 34359214081ULL,
                                68718428161ULL};   // params.rs:8-46

}  // namespace

struct b200pir_pp {
  b200pir_ctx* ctx;
  DevBuf<uint32_t> pack, left, right, conv;    // ntt32
};

namespace {

// The public parameters of a call's queries: `each[i]` for query i (a multi-client batch) or, where `each` is null, `one` for
// every query
struct Keys {
  b200pir_pp* one = nullptr;
  b200pir_pp* const* each = nullptr;
  b200pir_pp* operator[](size_t i) const { return each ? each[i] : one; }
};

// The context's per-query parameter table for queries [0, count) of `keys`; uploaded only when its contents change
PpTable pp_table(b200pir_ctx* c, Keys keys, size_t count) {
  size_t& cap = c->pptab_cap;
  if (count > cap) {
    cap = std::max<size_t>(count, 16);
    c->d_pptab.alloc(4 * cap);
    c->h_pptab.clear();
  }
  std::vector<const uint32_t*> h(4 * cap, nullptr);
  for (size_t i = 0; i < count; i++) {
    const b200pir_pp* p = keys[i];
    h[0 * cap + i] = p->pack.p;
    h[1 * cap + i] = p->left.p;
    h[2 * cap + i] = p->right.p ? p->right.p : p->left.p;     // unwrap_or(v_w_left), server.rs:549
    h[3 * cap + i] = p->conv.p;
  }
  if (h != c->h_pptab) {
    B200_CUDA(cudaMemcpyAsync(c->d_pptab.p, h.data(), h.size() * sizeof(const uint32_t*), cudaMemcpyHostToDevice, c->stream));
    c->h_pptab = h;
  }
  const uint32_t* const* d = c->d_pptab.p;
  return PpTable{d, d + cap, d + 2 * cap, d + 3 * cap};
}

// Where a fold left its survivors: the residue-form ciphertext of (query qi, slice t) at p + (qi * slices + t) * stride
struct Survivors {
  const uint32_t* p;
  size_t stride;
};

// The first-dimension operand as tile images (format-2 databases): image g holds queries [g * per_group, (g + 1) * per_group),
// per_group <= 16.  p == nullptr: no images, the operand is q_dev.
struct Images {
  const uint8_t* p;
  size_t per_group;
};

// `words` u64 host words of NTT form (each < 2^32) into the ntt32 device words `dst`, on the context's stream, staged through
// `wide`, which must live until the caller has synchronised
void upload_narrow(b200pir_ctx* c, uint32_t* dst, DevBuf<uint64_t>& wide, const uint64_t* host, size_t words) {
  wide.ensure(words);
  B200_CUDA(cudaMemcpyAsync(wide.p, host, words * 8, cudaMemcpyHostToDevice, c->stream));
  launch_narrow(dst, wide.p, words, c->stream);
}
// `words` ntt32 device words widened into the u64 host buffer `host`: the call's final synchronise
void download_widen(b200pir_ctx* c, uint64_t* host, const uint32_t* src, size_t words) {
  DevBuf<uint64_t> wide(words);
  launch_widen(wide.p, src, words, c->stream);
  B200_CUDA(cudaMemcpyAsync(host, wide.p, words * 8, cudaMemcpyDeviceToHost, c->stream));
  B200_CUDA(cudaStreamSynchronize(c->stream));
}
// upload u64 NTT-form matrices (words < 2^32) as ntt32
void upload_ntt32(b200pir_ctx* c, DevBuf<uint32_t>& dst, const uint64_t* host, size_t words) {
  dst.alloc(words);
  DevBuf<uint64_t> wide;
  upload_narrow(c, dst.p, wide, host, words);
  B200_CUDA(cudaStreamSynchronize(c->stream));
}

// ---- pipeline pieces (all stream-ordered, device pointers)

// server.rs:19-121 over `nq` queries at once (v: [nq][2^g][4][2048], v_stride words apart)
void run_coefficient_expansion(b200pir_ctx* c, Keys keys, uint32_t* v, size_t v_stride, int nq, bool all_slots) {
  const auto& hp = c->hp;
  cudaStream_t s = c->stream;
  const int g = c->g;
  const int stop_round = hp.nu_2 > 0 ? c->stop_round : 0;
  const int max_right = hp.nu_2 > 0 ? (int)(hp.t_gsw * hp.nu_2) : 0;
  const PpTable T = pp_table(c, keys, (size_t)nq);
  for (int r = 0; r < g; r++) {
    const int num_in = 1 << r;
    ExpandRound R;
    R.r = r; R.num_in = num_in; R.stop_round = stop_round; R.max_bits_to_gen_right = max_right;
    R.fill_skipped = all_slots ? 1 : 0;
    R.t_auto = (POLY >> r) + 1;
    R.t_left = (int)hp.t_exp_left; R.bits_left = c->bits_left; R.live_left = c->live_left;
    R.tab_left = T.left; R.off_left = (size_t)r * 2 * hp.t_exp_left * 2 * POLY;
    if (hp.nu_2 > 0 && c->has_right) {
      // v_w_right has stop_round+1 matrices; rounds beyond that never take the right branch for a
      // processed (even) index except r == 0 (server.rs:60-73), so clamp the pointer for safety.
      int rr = r <= c->stop_round ? r : c->stop_round;
      R.t_right = (int)hp.t_exp_right; R.bits_right = c->bits_right; R.live_right = c->live_right;
      R.tab_right = T.right; R.off_right = (size_t)rr * 2 * hp.t_exp_right * 2 * POLY;
    } else {
      R.t_right = R.t_left; R.bits_right = R.bits_left; R.live_right = R.live_left; R.tab_right = T.left; R.off_right = R.off_left;   // unwrap_or(v_w_left), server.rs:549
    }
    const size_t xr_stride = (size_t)num_in * 2 * POLY;
    c->w_xr.ensure((size_t)nq * xr_stride);
    launch_expand_round_res(c->dp, v, v_stride, c->w_xr.p, xr_stride, nq, R, c->d_neg1.p + (size_t)r * 2 * POLY, s);
  }
}

// server.rs:525-591 for `nq` queries.  v: [nq][2^g][4][2048]; writes v_fold of every query and the first-dimension operand:
// q_dev (uint4 [query][dim0][2048], reorient_reg_ciphertexts util.rs:323-355) or, when `images` is given (format-2 databases),
// the operand tile images of groups of 16 queries directly (image g = queries 16g .., tc5_query_bytes apart): no intermediate.
void run_expand_query(b200pir_ctx* c, Keys keys, const uint64_t* query_raw, uint32_t* v, uint4* q_dev, uint32_t* v_fold,
                      int nq, uint8_t* images) {
  const auto& hp = c->hp;
  cudaStream_t s = c->stream;
  // no clear of v: every slot the query path reads (even slots < 2 dim0, odd slots < 2 t_gsw nu_2) is written by the rounds
  launch_to_ntt_strided(c->dp, v, c->v_words(), query_raw, (size_t)2 * POLY, 2, nq, s);   // v[0] = query.ct.ntt()
  run_coefficient_expansion(c, keys, v, c->v_words(), nq, false);
  const int factor = hp.nu_2 > 0 ? 2 : 1;
  if (images) {
    const Tc5Geom T = make_tc5_geom(c->dim0, 32);
    for (int q0 = 0; q0 < nq; q0 += 16)
      launch_reorient_to_tc5(T, v + (size_t)q0 * c->v_words(), c->v_words(), factor, std::min(16, nq - q0),
                             images + (size_t)(q0 / 16) * tc5_query_bytes(T), s);
  } else {
    launch_reorient(c->geom(c->num_per), q_dev, (size_t)c->dim0 * POLY, v, c->v_words(), nq, factor, s);
  }
  if (hp.nu_2 > 0)
    launch_regev_to_gsw(c->dp, v_fold, c->fold_words(), v, c->v_words(), nq, (int)hp.nu_2, 2, 1, pp_table(c, keys, (size_t)nq).conv,
                        (int)hp.t_gsw, (int)hp.t_conv, c->bits_conv, c->live_conv, s);
}

// fold `num` ciphertexts per batch entry with matrices k = k0, k0-1, ...
void run_fold(b200pir_ctx* c, uint64_t* cts, size_t batch, size_t batch_stride, size_t num, int k0,
              const uint32_t* vfold, const uint32_t* vfold_neg, int slices_per_query) {
  const size_t mat = (size_t)2 * 2 * c->hp.t_gsw * 2 * POLY;
  int k = k0;
  for (size_t half = num / 2; half >= 1; half /= 2, k--) {
    launch_fold_round(c->dp, cts, batch, batch_stride, (int)half, vfold + (size_t)k * mat, vfold_neg + (size_t)k * mat,
                      c->fold_words(), slices_per_query, (int)c->hp.t_gsw, c->bits_gsw, c->stream);
  }
}

// Fast path on residue-form ciphertexts: ping-pong between `a` (input of the first round) and `b`.
// Returns the buffer holding the survivors (entry 0 of each batch element).  `sparse`: lib/server's fold shortcut (the
// "sparse_fold" option of the context whose call this is).
const uint32_t* run_fold_res(b200pir_ctx* c, uint32_t* a, uint32_t* b, size_t batch, size_t batch_stride, size_t num,
                             int k0, const uint32_t* vfold, int slices_per_query, bool sparse) {
  const size_t mat = (size_t)2 * 2 * c->hp.t_gsw * 2 * POLY;
  int k = k0;
  uint32_t* src = a;
  uint32_t* dst = b;
  uint32_t* zero_flags = nullptr;                      // lib/server's fold shortcut (fold.rs:37-43) when "sparse_fold" is set
  if (sparse) {
    c->w_zflags.ensure(batch * num);
    zero_flags = c->w_zflags.p;
  }
  for (size_t half = num / 2; half >= 1; half /= 2, k--) {
    launch_fold_res(c->dp, src, dst, batch, batch_stride, (int)half, vfold + (size_t)k * mat, c->fold_words(),
                    slices_per_query, (int)c->hp.t_gsw, c->bits_gsw, c->live_gsw, zero_flags, c->stream);
    std::swap(src, dst);
  }
  return src;
}

// expansion (or direct upload) for `count` queries already in w_query / w_qdev,w_vfold
// (`images`: the expansion writes the first-dimension operand to w_qt as tile images, for a format-2 database)
void run_prepare(b200pir_ctx* c, Keys keys, size_t count, bool images) {
  b200pir_ctx::Scope sc(c, ST_EXPAND);
  if (images) c->w_qt.ensure((count + 15) / 16 * tc5_query_bytes(make_tc5_geom(c->dim0, 32)));
  if (c->hp.expand_queries)
    run_expand_query(c, keys, c->w_query.p, c->w_v.p, c->w_qdev.p, c->w_vfold.p, (int)count, images ? c->w_qt.p : nullptr);
  // v_folding_neg (server.rs:680) is not materialised: the fold fast path uses G - C_k implicitly.
}

// The first-dimension product of `count` queries (operands qdev + qi * dim0 * POLY, or `images`) over slices [slice_begin,
// slice_begin + slice_count), into `out` (queries slices * rows * 4 * POLY words apart) in the form db.zmajor_product() names.
void run_first_dim(b200pir_ctx* c, const DbStore& db, size_t count, const uint4* qdev, Images images, uint32_t* out,
                   int slice_begin, int slice_count) {
  const DbLayout& L = db.layout;
  const size_t q_stride = (size_t)c->dim0 * POLY;
  const size_t out_stride = (size_t)c->slices * db.rows * 4 * POLY;
  if (L.format == 0) {
    // IMAD path: 4, 2 or 1 queries per database pass
    b200pir_ctx::Scope sc(c, ST_MUL);
    size_t qi = 0;
    while (qi < count) {
      int nq = 1;
      if (count - qi >= 4 && c->max_group >= 4) nq = 4;
      else if (count - qi >= 2 && c->max_group >= 2) nq = 2;
      launch_multiply(c->dp, L.G, reinterpret_cast<const uint4*>(L.base), qdev + qi * q_stride, out + qi * out_stride,
                      slice_begin, slice_count, nq, q_stride, out_stride, c->stream);
      c->mul_launches++;
      qi += nq;
    }
  } else if (L.format == 2) {
    // wgmma path: same z-major product as the mma.sync path, 16 queries per database pass
    if (!images.p) c->w_qt.ensure(tc5_query_bytes(L.T));
    const size_t step = images.p ? images.per_group : 16;
    for (size_t qi = 0, g = 0; qi < count; qi += step, g++) {
      const int nq = (int)std::min<size_t>(step, count - qi);
      const uint8_t* qt = images.p ? images.p + g * tc5_query_bytes(L.T) : c->w_qt.p;
      if (!images.p) {
        b200pir_ctx::Scope sq(c, ST_QIMG);
        launch_query_to_tc5(L.T, qdev + qi * q_stride, q_stride, nq, c->w_qt.p, c->stream);
      }
      b200pir_ctx::Scope sc(c, ST_MUL);
      launch_multiply_tc5(c->dp, L.T, L.base, db.tile_mask.p, qt, out + qi * out_stride, out_stride, nq, slice_begin,
                          slice_count, c->sm_count, c->stream);
      c->mul_launches++;
    }
  } else {
    // INT8 tensor-core path
    c->w_qf.ensure(imma_query_cells(L.F));
    const size_t per_pass = (c->max_group >= 16 && imma_supports_16(L.F)) ? 16 : (c->max_group >= 8 ? 8 : 4);
    for (size_t qi = 0; qi < count; qi += per_pass) {
      const int nq = (int)std::min<size_t>(per_pass, count - qi);
      {
        b200pir_ctx::Scope sq(c, ST_QIMG);
        launch_query_to_frag(L.F, qdev + qi * q_stride, q_stride, nq, c->w_qf.p, c->stream);
      }
      {
        b200pir_ctx::Scope sc(c, ST_MUL);
        launch_multiply_imma(c->dp, L.F, reinterpret_cast<const uint4*>(L.base), c->w_qf.p, out + qi * out_stride, out_stride,
                             nq, slice_begin, slice_count, c->stream);
        c->mul_launches++;
      }
    }
  }
}

// first dimension (operand qdev or `images`) + from_ntt + local fold with the folding matrices vfold (fold shortcut when
// `sparse`); returns the survivors (in w_mult or w_cts), one per (query, slice)
Survivors run_first_dim_and_fold(b200pir_ctx* c, const DbStore& db, size_t count, const uint4* qdev, Images images,
                                 const uint32_t* vfold, bool sparse) {
  const int rows = db.rows;
  const size_t out_stride = (size_t)c->slices * rows * 4 * POLY;
  // server.rs:707-709 from_ntt, minus the CRT lift, into w_mult in residue form: a z-major product goes to w_cts (free until
  // the fold starts) and is inverse-transformed from there; an ntt32 product is inverse-transformed in place
  const bool zmajor = db.zmajor_product();
  run_first_dim(c, db, count, qdev, images, zmajor ? c->w_cts.p : c->w_mult.p, 0, c->slices);
  {
    b200pir_ctx::Scope sc(c, ST_FROMNTT);
    if (zmajor) launch_intt_from_zmajor(c->dp, db.layout.F, c->w_cts.p, out_stride, c->w_mult.p, (int)count, c->slices, c->stream);
    else launch_ntt32(c->dp, c->w_mult.p, count * c->slices * rows * 2, true, c->stream);
  }
  b200pir_ctx::Scope sc(c, ST_FOLD);
  Survivors s{c->w_mult.p, (size_t)rows * 4 * POLY};
  if (rows > 1) s.p = run_fold_res(c, c->w_mult.p, c->w_cts.p, count * c->slices, s.stride, rows, (int)c->hp.nu_2 - 1, vfold, c->slices, sparse);
  return s;
}

// pack + encode for `count` queries
void run_pack_encode(b200pir_ctx* c, Keys keys, Survivors s, size_t count, uint8_t* out_dev) {
  const auto& hp = c->hp;
  const size_t packed_words = (size_t)hp.instances * (hp.n + 1) * hp.n * POLY;
  {
    b200pir_ctx::Scope sc(c, ST_PACK);
    launch_pack(c->dp, c->w_packed.p, packed_words, s.p, s.stride, (size_t)c->slices * s.stride, (int)count, pp_table(c, keys, count).pack,
                (int)hp.n, (int)hp.instances, (int)hp.t_conv, c->bits_conv, c->live_conv, (int)hp.version, c->stream);
  }
  {
    b200pir_ctx::Scope sc(c, ST_ENCODE);
    launch_encode(c->dp, out_dev, c->response_bytes, c->w_packed.p, packed_words, (int)count, (int)hp.n, (int)hp.instances,
                  c->q2, (int)hp.q2_bits, c->q1, c->q1_bits, c->stream);
  }
}

void check_pp(b200pir_ctx* c, b200pir_pp* pp) {
  if (!pp || !same_params(pp->ctx, c)) throw Error(B200PIR_E_BADARG, "pp handle was created for different parameters / device");
}

}  // namespace

extern "C" {

const char* b200pir_last_error(void) { return g_last_error.c_str(); }
int b200pir_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) return 0;
  return n;
}

int b200pir_ctx_create(const b200pir_params* params, int device, b200pir_ctx** out) {
  API_BEGIN
  if (!params || !out) throw Error(B200PIR_E_BADARG, "null argument");
  use_device(device);
  std::unique_ptr<b200pir_ctx> c(new b200pir_ctx());
  static std::atomic<uint64_t> next_seq{0};
  c->seq = next_seq++;
  c->device = device;
  B200_CUDA(cudaDeviceGetAttribute(&c->sm_count, cudaDevAttrMultiProcessorCount, device));
  c->hp = *params;
  auto& hp = c->hp;
  if (hp.q2_bits < 14) hp.q2_bits = 14;                       // util.rs:230, params.rs:7
  if (hp.q2_bits > 36) throw Error(B200PIR_E_BADARG, "q2_bits out of range");
  if (hp.instances == 0) hp.instances = 1;
  if (hp.n < 1 || hp.n > 4) throw Error(B200PIR_E_UNSUPPORTED, "n must be 1..4");
  if (hp.nu_1 < 1 || hp.nu_1 > 16 || hp.nu_2 > 16) throw Error(B200PIR_E_BADARG, "nu_1/nu_2 out of range");
  if (hp.version > 1) throw Error(B200PIR_E_BADARG, "unknown version");
  if (hp.p < 2 || (hp.p & (hp.p - 1)) || hp.p > (1u << 20)) throw Error(B200PIR_E_BADARG, "p must be a power of two <= 2^20");
  for (uint64_t t : {hp.t_gsw, hp.t_conv, hp.t_exp_left, hp.t_exp_right})
    if (t < 3 || t > 56)   // t = 2 would mean 29-bit digits: above q, outside the transforms' input range (and no parameter
      throw Error(B200PIR_E_UNSUPPORTED, "gadget dimensions must be in 3..56");   // set of the reference uses it)
  if (hp.db_item_size == 0) hp.db_item_size = hp.instances * hp.n * hp.n * 2048 * log2_ceil_u64(hp.p) / 8;
  c->dim0 = 1 << hp.nu_1;
  c->num_per = 1 << hp.nu_2;
  c->trials = (int)(hp.n * hp.n);
  c->slices = (int)(hp.instances * c->trials);
  c->slice_words = (size_t)c->dim0 * c->num_per * POLY;
  c->bytes_per_chunk = (hp.db_item_size + c->slices - 1) / c->slices;
  c->g = (int)log2_ceil_u64(hp.t_gsw * hp.nu_2 + c->dim0);
  c->stop_round = hp.nu_2 ? (int)log2_ceil_u64(hp.t_gsw * hp.nu_2) : 0;
  if (c->g > 11) throw Error(B200PIR_E_UNSUPPORTED, "expansion needs more than 2048 slots");
  // expand_query takes the first-dimension ciphertexts from the even slots and the GSW inputs from the odd slots
  // (server.rs:565-571), so each half must fit in 2^(g-1) slots; 2^g only bounds their sum.  With t_gsw * nu_2 = 18 and
  // dim0 = 4, for instance, g = 5 and the odd slots run to 35: the reference panics on the index, and the expansion and
  // conversion kernels would read past the query's workspace.
  if (hp.expand_queries && hp.nu_2 > 0 && 2 * std::max<uint64_t>(c->dim0, hp.t_gsw * hp.nu_2) > (1ull << c->g))
    throw Error(B200PIR_E_UNSUPPORTED, "expansion: dim0 and t_gsw * nu_2 must each fit in half of the 2^g slots");
  c->num_packing = hp.version == 0 ? (int)hp.n : 2;
  c->has_right = hp.expand_queries && (hp.version == 0 || hp.t_exp_right != hp.t_exp_left);
  c->bits_gsw = bits_per((int)hp.t_gsw);
  c->bits_conv = bits_per((int)hp.t_conv);
  c->bits_left = bits_per((int)hp.t_exp_left);
  c->bits_right = bits_per((int)hp.t_exp_right);
  c->live_gsw = live_digits((int)hp.t_gsw);
  c->live_conv = live_digits((int)hp.t_conv);
  c->live_left = live_digits((int)hp.t_exp_left);
  c->live_right = live_digits((int)hp.t_exp_right);
  c->q2 = kQ2Values[hp.q2_bits];
  c->q1 = 4 * hp.p;
  c->q1_bits = (int)log2_ceil_u64(c->q1);
  {
    uint64_t bits = hp.instances * (hp.q2_bits * hp.n * 2048 + (uint64_t)c->q1_bits * hp.n * hp.n * 2048);
    c->response_bytes = ((bits + 63) / 64) * 8;
    uint64_t sz = (uint64_t)c->num_packing * hp.n * hp.t_conv;
    if (hp.expand_queries) {
      uint64_t right = (uint64_t)(c->stop_round + 1) * hp.t_exp_right;
      if (hp.version > 0 && hp.t_exp_left == hp.t_exp_right) right = 0;
      sz += (uint64_t)c->g * hp.t_exp_left + right + 2 * hp.t_conv;
    }
    c->setup_bytes = 32 + sz * 2048 * 8;
    uint64_t qp = hp.expand_queries ? 1 : (uint64_t)c->dim0 + hp.nu_2 * 2 * hp.t_gsw;
    c->query_bytes = 32 + qp * 2048 * 8;
  }
  B200_CUDA(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking));
  // tables
  const uint64_t q0 = 268369921ULL, q1m = 249561089ULL;            // util.rs:246-247
  std::vector<Twiddle> f0, i0, f1, i1;
  build_tables(q0, f0, i0);
  build_tables(q1m, f1, i1);
  std::vector<Twiddle> l0, l1;                                     // relaxed-range inverse tables (ntt_core.cuh "lz")
  b200pir::tables::build_inverse_table_lz(q0, l0);
  b200pir::tables::build_inverse_table_lz(q1m, l1);
  // Every table goes up on the context's own stream, which the synchronise at the end of this function waits for: copies on
  // the legacy default stream would wait for whatever the caller has queued there, and a pageable cudaMemcpy may return
  // before its data has landed, while the first transform below already runs on the non-blocking context stream.  The host
  // vectors outlive that synchronise.
  c->d_tw.alloc(6 * POLY);
  const size_t tw_bytes = POLY * sizeof(Twiddle);
  B200_CUDA(cudaMemcpyAsync(c->d_tw.p + 4 * POLY, l0.data(), tw_bytes, cudaMemcpyHostToDevice, c->stream));
  B200_CUDA(cudaMemcpyAsync(c->d_tw.p + 5 * POLY, l1.data(), tw_bytes, cudaMemcpyHostToDevice, c->stream));
  B200_CUDA(cudaMemcpyAsync(c->d_tw.p, f0.data(), tw_bytes, cudaMemcpyHostToDevice, c->stream));
  B200_CUDA(cudaMemcpyAsync(c->d_tw.p + POLY, i0.data(), tw_bytes, cudaMemcpyHostToDevice, c->stream));
  B200_CUDA(cudaMemcpyAsync(c->d_tw.p + 2 * POLY, f1.data(), tw_bytes, cudaMemcpyHostToDevice, c->stream));
  B200_CUDA(cudaMemcpyAsync(c->d_tw.p + 3 * POLY, i1.data(), tw_bytes, cudaMemcpyHostToDevice, c->stream));
  std::vector<Twiddle> lo(2 * 3 * 64);                             // [n][forward, inverse, relaxed-range inverse][64]
  for (int i = 0; i < 64; i++) { lo[(0 * 3 + 0) * 64 + i] = f0[i]; lo[(0 * 3 + 1) * 64 + i] = i0[i]; lo[(0 * 3 + 2) * 64 + i] = l0[i];
                                 lo[(1 * 3 + 0) * 64 + i] = f1[i]; lo[(1 * 3 + 1) * 64 + i] = i1[i]; lo[(1 * 3 + 2) * 64 + i] = l1[i]; }
  upload_poly_constants(lo.data(), c->stream);
  // poly_len = 4096 (config #5): built here rather than on the first b200pir_ntt4096_dev call, so that call neither allocates
  // nor copies from the host
  std::vector<Twiddle> tw4k;
  for (const uint64_t q : {q0, q1m}) {
    std::vector<Twiddle> f, i;
    build_tables(q, f, i, 4096, 12);
    tw4k.insert(tw4k.end(), f.begin(), f.end());
    tw4k.insert(tw4k.end(), i.begin(), i.end());
  }
  c->d_tw4k.alloc(tw4k.size());
  B200_CUDA(cudaMemcpyAsync(c->d_tw4k.p, tw4k.data(), tw4k.size() * sizeof(Twiddle), cudaMemcpyHostToDevice, c->stream));
  DevParams& dp = c->dp;
  dp.q[0] = (uint32_t)q0; dp.q[1] = (uint32_t)q1m;
  dp.cr1[0] = (uint64_t)(((u128)1 << 64) / q0);
  dp.cr1[1] = (uint64_t)(((u128)1 << 64) / q1m);
  dp.modulus = q0 * q1m;
  dp.cr1_mod = (uint64_t)(((u128)1 << 64) / dp.modulus);
  dp.q1_inv_mod_q0 = (uint32_t)invmod(q1m % q0, q0);
  dp.fwd[0] = c->d_tw.p; dp.inv[0] = c->d_tw.p + POLY; dp.fwd[1] = c->d_tw.p + 2 * POLY; dp.inv[1] = c->d_tw.p + 3 * POLY;
  dp.inv_lz[0] = c->d_tw.p + 4 * POLY; dp.inv_lz[1] = c->d_tw.p + 5 * POLY;
  dp.mu58[0] = (uint32_t)(((uint64_t)1 << 58) / q0); dp.mu58[1] = (uint32_t)(((uint64_t)1 << 58) / q1m);
  // v_neg1 (params.rs:98-107): NTT of -(X^{N - 2^i})
  {
    std::vector<uint32_t> h((size_t)NTT_LOG_N * 2 * POLY, 0);
    for (int i = 0; i < NTT_LOG_N; i++) {
      int idx = POLY - (1 << i);
      h[((size_t)i * 2 + 0) * POLY + idx] = (uint32_t)(q0 - 1);
      h[((size_t)i * 2 + 1) * POLY + idx] = (uint32_t)(q1m - 1);
    }
    c->d_neg1.alloc(h.size());
    B200_CUDA(cudaMemcpyAsync(c->d_neg1.p, h.data(), h.size() * 4, cudaMemcpyHostToDevice, c->stream));
    launch_ntt32(dp, c->d_neg1.p, NTT_LOG_N, false, c->stream);
    B200_CUDA(cudaStreamSynchronize(c->stream));
  }
  B200_CUDA(cudaGetLastError());
  *out = c.release();
  API_END
}

void b200pir_ctx_destroy(b200pir_ctx* c) {
  if (!c) return;
  cudaSetDevice(c->device);
  cudaDeviceSynchronize();
  for (auto e : c->event_pool) cudaEventDestroy(e);
  c->release_export_pinned();
  for (auto e : c->export_done) if (e) cudaEventDestroy(e);
  if (c->own_stream && c->stream) cudaStreamDestroy(c->stream);
  delete c;
}
int b200pir_ctx_set_stream(b200pir_ctx* c, void* cuda_stream) {
  API_BEGIN
  if (!c) throw Error(B200PIR_E_BADARG, "null ctx");
  Guard gd(c);
  B200_CUDA(cudaStreamSynchronize(c->stream));
  if (c->own_stream && c->stream) cudaStreamDestroy(c->stream);
  c->stream = (cudaStream_t)cuda_stream;
  c->own_stream = false;
  API_END
}
int b200pir_ctx_synchronize(b200pir_ctx* c) {
  API_BEGIN
  if (!c) throw Error(B200PIR_E_BADARG, "null ctx");
  Guard gd(c);
  B200_CUDA(cudaStreamSynchronize(c->stream));
  B200_CUDA(cudaGetLastError());
  API_END
}
int b200pir_ctx_reserve(b200pir_ctx* c, size_t queries, size_t rows_local) {
  API_BEGIN
  if (!c) throw Error(B200PIR_E_BADARG, "null ctx");
  if (queries == 0 || queries > 4096 || rows_local == 0 || rows_local > ((size_t)1 << c->hp.nu_2))
    throw Error(B200PIR_E_BADARG, "reserve: 1..4096 queries, 1..num_per rows");
  Guard gd(c);
  B200_CUDA(cudaStreamSynchronize(c->stream));          // buffers may be replaced: nothing in flight may still use them
  c->ensure_workspace(queries, rows_local);
  B200_CUDA(cudaGetLastError());
  API_END
}
int b200pir_ctx_set_option(b200pir_ctx* c, const char* key, int64_t value) {
  API_BEGIN
  if (!c || !key) throw Error(B200PIR_E_BADARG, "null argument");
  Guard gd(c);
  std::string k(key);
  if (k == "batch") { if (value != 1 && value != 2 && value != 4 && value != 8 && value != 16) throw Error(B200PIR_E_BADARG, "batch must be 1, 2, 4, 8 or 16"); c->max_group = (int)value; }
  // one kernel each now; the keys stay accepted so existing callers keep working
  else if (k == "mul_variant" || k == "fold_variant" || k == "intt_variant" || k == "imma_variant" || k == "expand_variant" ||
           k == "expand_pair_min_ctas") {}
  else if (k == "sparse_fold") c->sparse_fold = value != 0;
  else if (k == "coalesce") c->coalesce = value != 0;
  else if (k == "coalesce_window_us") { if (value < 0 || value > 100000) throw Error(B200PIR_E_BADARG, "coalesce_window_us must be 0..100000"); c->coalesce_window_us = (int)value; }
  else if (k == "db_format") { if (value < -1 || value > 2) throw Error(B200PIR_E_BADARG, "db_format must be -1 (automatic), 0, 1 or 2"); c->db_format = (int)value; }
  else if (k == "profile") {
    if (value < 0 || value > 2) throw Error(B200PIR_E_BADARG, "profile must be 0, 1 or 2");
    c->profile = (int)value;
    c->spans.clear(); c->event_next = 0; c->mul_launches = 0;
  }
  else throw Error(B200PIR_E_BADARG, "unknown option " + k);
  API_END
}
int b200pir_ctx_sizes(b200pir_ctx* c, uint64_t* setup_bytes, uint64_t* query_bytes, uint64_t* response_bytes) {
  API_BEGIN
  if (!c) throw Error(B200PIR_E_BADARG, "null ctx");
  if (setup_bytes) *setup_bytes = c->setup_bytes;
  if (query_bytes) *query_bytes = c->query_bytes;
  if (response_bytes) *response_bytes = c->response_bytes;
  API_END
}


// ---------------------------------------------------------------- public parameters
int b200pir_pp_create(b200pir_ctx* c, const uint64_t* v_packing, const uint64_t* left, const uint64_t* right,
                      const uint64_t* conv, b200pir_pp** out) {
  API_BEGIN
  if (!c || !out || !v_packing) throw Error(B200PIR_E_BADARG, "null argument");
  Guard gd(c);
  const auto& hp = c->hp;
  std::unique_ptr<b200pir_pp> pp(new b200pir_pp());
  pp->ctx = c;
  const size_t W = 2 * POLY;
  upload_ntt32(c, pp->pack, v_packing, (size_t)c->num_packing * (hp.n + 1) * hp.t_conv * W);
  if (hp.expand_queries) {
    if (!left || !conv) throw Error(B200PIR_E_BADARG, "expansion parameters missing");
    upload_ntt32(c, pp->left, left, (size_t)c->g * 2 * hp.t_exp_left * W);
    if (c->has_right) {
      if (!right) throw Error(B200PIR_E_BADARG, "v_expansion_right missing");
      upload_ntt32(c, pp->right, right, (size_t)(c->stop_round + 1) * 2 * hp.t_exp_right * W);
    }
    upload_ntt32(c, pp->conv, conv, (size_t)2 * 2 * hp.t_conv * W);
  }
  *out = pp.release();
  API_END
}

namespace {
// One group of serialized matrices (client.rs:55-80): `count` raw matrices rows x cols; row 0 regenerated from the seed's
// keystream (u64 position `word`), rows 1.. copied from the byte stream.  Result: NTT form, ntt32 layout, in `dst`.
void deserialize_group(b200pir_ctx* c, DevBuf<uint32_t>& dst, const uint8_t* seed, const uint8_t*& data, uint64_t& word,
                       size_t count, size_t rows, size_t cols) {
  const size_t row_words = cols * POLY, mat_words = rows * row_words, rest = (rows - 1) * row_words;
  DevBuf<uint64_t> raw(count * mat_words);
  launch_chacha_first_rows(raw.p, seed, word, (uint32_t)count, (uint32_t)row_words, mat_words, c->dp.modulus, c->stream);
  word += count * row_words;
  for (size_t i = 0; i < count; i++) {
    B200_CUDA(cudaMemcpyAsync(raw.p + i * mat_words + row_words, data, rest * 8, cudaMemcpyHostToDevice, c->stream));
    data += rest * 8;
  }
  dst.alloc(count * mat_words * 2);
  launch_to_ntt(c->dp, dst.p, raw.p, count * rows * cols, c->stream);
  B200_CUDA(cudaStreamSynchronize(c->stream));
}
}  // namespace

// PublicParameters::deserialize (client.rs:212-259)
int b200pir_pp_create_from_bytes(b200pir_ctx* c, const uint8_t* data, size_t len, b200pir_pp** out) {
  API_BEGIN
  if (!c || !out || !data) throw Error(B200PIR_E_BADARG, "null argument");
  if (len != c->setup_bytes) throw Error(B200PIR_E_SHAPE, "setup data: expected " + std::to_string(c->setup_bytes) + " bytes");
  Guard gd(c);
  const auto& hp = c->hp;
  std::unique_ptr<b200pir_pp> pp(new b200pir_pp());
  pp->ctx = c;
  const uint8_t* seed = data;
  const uint8_t* cur = data + 32;
  uint64_t word = 0;
  deserialize_group(c, pp->pack, seed, cur, word, (size_t)c->num_packing, hp.n + 1, hp.t_conv);
  if (hp.expand_queries) {
    deserialize_group(c, pp->left, seed, cur, word, (size_t)c->g, 2, hp.t_exp_left);
    if (c->has_right) deserialize_group(c, pp->right, seed, cur, word, (size_t)c->stop_round + 1, 2, hp.t_exp_right);
    deserialize_group(c, pp->conv, seed, cur, word, 1, 2, 2 * hp.t_conv);
  }
  if ((size_t)(cur - data) != len) throw Error(B200PIR_E_SHAPE, "setup data: trailing bytes");
  *out = pp.release();
  API_END
}

namespace {
// Query::deserialize, expand_queries branch (client.rs:303-315): `count` serialized queries -> [count] PolyMatrixRaw(2,1) on device
void deserialize_queries(b200pir_ctx* c, const uint8_t* data, size_t count, uint64_t* dst_dev) {
  for (size_t i = 0; i < count; i++) {
    const uint8_t* q = data + i * c->query_bytes;
    launch_chacha_first_rows(dst_dev + i * 2 * POLY, q, 0, 1, POLY, 2 * POLY, c->dp.modulus, c->stream);
    B200_CUDA(cudaMemcpyAsync(dst_dev + i * 2 * POLY + POLY, q + 32, POLY * 8, cudaMemcpyHostToDevice, c->stream));
  }
}
// Query::deserialize, direct-upload branch (client.rs:316-327): one serialized query -> the device-format first-dimension
// operand (q_dev) and the NTT-form folding matrices (v_fold) of workspace slot `slot`.
// Keystream order (interleave_rng_data :107-131, deserialize_vec_polymatrix_rng :81-93): 2048 words per first-dimension
// ciphertext (its row 0), then the first rows (2 t_gsw polynomials) of the nu_2 GSW matrices.
void deserialize_query_direct(b200pir_ctx* c, const uint8_t* q, size_t slot) {
  const size_t dim0 = (size_t)c->dim0, t2 = 2 * c->hp.t_gsw, nu2 = c->hp.nu_2;
  cudaStream_t s = c->stream;
  // row 0 of every first-dimension ciphertext: a raw 1 x 1 "matrix" per ciphertext (row 1 of sigma stays zero and is never used)
  DevBuf<uint64_t> sig_raw(dim0 * POLY);
  DevBuf<uint32_t> sig_ntt(dim0 * 2 * POLY);
  launch_chacha_first_rows(sig_raw.p, q, 0, (uint32_t)dim0, POLY, POLY, c->dp.modulus, s);
  launch_to_ntt(c->dp, sig_ntt.p, sig_raw.p, dim0, s);
  DevBuf<uint64_t> wire(dim0 * POLY);
  B200_CUDA(cudaMemcpyAsync(wire.p, q + 32, dim0 * POLY * 8, cudaMemcpyHostToDevice, s));
  launch_direct_query_to_dev(c->w_qdev.p + slot * dim0 * POLY, sig_ntt.p, wire.p, (int)dim0, s);
  if (nu2) {
    DevBuf<uint64_t> raw(nu2 * 2 * t2 * POLY);
    launch_chacha_first_rows(raw.p, q, dim0 * POLY, (uint32_t)nu2, (uint32_t)(t2 * POLY), 2 * t2 * POLY, c->dp.modulus, s);
    const uint8_t* rest = q + 32 + dim0 * POLY * 8;
    for (size_t i = 0; i < nu2; i++)
      B200_CUDA(cudaMemcpyAsync(raw.p + (i * 2 + 1) * t2 * POLY, rest + i * t2 * POLY * 8, t2 * POLY * 8, cudaMemcpyHostToDevice, s));
    launch_to_ntt(c->dp, c->w_vfold.p + slot * c->fold_words(), raw.p, nu2 * 2 * t2, s);
  }
  B200_CUDA(cudaStreamSynchronize(s));        // the staging buffers above are freed on return
}
}  // namespace

int b200pir_query_from_bytes(b200pir_ctx* c, const uint8_t* data, size_t len, uint64_t* query_ct) {
  API_BEGIN
  if (!c || !data || !query_ct) throw Error(B200PIR_E_BADARG, "null argument");
  if (!c->hp.expand_queries) throw Error(B200PIR_E_UNSUPPORTED, "serialized direct-upload queries are not supported");
  if (len != c->query_bytes) throw Error(B200PIR_E_SHAPE, "query: expected " + std::to_string(c->query_bytes) + " bytes");
  Guard gd(c);
  DevBuf<uint64_t> ct(2 * POLY);
  deserialize_queries(c, data, 1, ct.p);
  B200_CUDA(cudaMemcpyAsync(query_ct, ct.p, 2 * POLY * 8, cudaMemcpyDeviceToHost, c->stream));
  B200_CUDA(cudaStreamSynchronize(c->stream));
  API_END
}

void b200pir_pp_destroy(b200pir_pp* pp) {
  if (!pp) return;
  cudaSetDevice(pp->ctx->device);
  delete pp;
}

// ---------------------------------------------------------------- stage-level entry points
static int ntt_host(b200pir_ctx* c, uint64_t* polys, size_t count, bool inverse) {
  API_BEGIN
  if (!c || (!polys && count)) throw Error(B200PIR_E_BADARG, "null argument");
  Guard gd(c);
  if (count == 0) return 0;
  DevBuf<uint64_t> d(count * 2 * POLY);
  B200_CUDA(cudaMemcpyAsync(d.p, polys, d.n * 8, cudaMemcpyHostToDevice, c->stream));
  launch_ntt_u64(c->dp, d.p, count, inverse, c->stream);
  B200_CUDA(cudaMemcpyAsync(polys, d.p, d.n * 8, cudaMemcpyDeviceToHost, c->stream));
  B200_CUDA(cudaStreamSynchronize(c->stream));
  B200_CUDA(cudaGetLastError());
  API_END
}
int b200pir_ntt_forward(b200pir_ctx* c, uint64_t* polys, size_t count) { return ntt_host(c, polys, count, false); }
int b200pir_ntt_inverse(b200pir_ctx* c, uint64_t* polys, size_t count) { return ntt_host(c, polys, count, true); }

int b200pir_ntt32_dev(b200pir_ctx* c, uint32_t* polys_dev, size_t count, int inverse) {
  API_BEGIN
  if (!c || !polys_dev) throw Error(B200PIR_E_BADARG, "null argument");
  Guard gd(c);
  launch_ntt32(c->dp, polys_dev, count, inverse != 0, c->stream);
  B200_CUDA(cudaGetLastError());
  API_END
}

// ---- poly_len = 4096 transforms (BASELINE config #5; not part of the reference's parameterisation, util.rs:246); the tables
// are built in b200pir_ctx_create
int b200pir_ntt4096_dev(b200pir_ctx* c, uint32_t* polys_dev, size_t count, int inverse) {
  API_BEGIN
  if (!c || !polys_dev) throw Error(B200PIR_E_BADARG, "null argument");
  Guard gd(c);
  launch_ntt32_4k(c->dp.q[0], c->dp.q[1], c->d_tw4k.p, polys_dev, count, inverse != 0, c->stream);
  B200_CUDA(cudaGetLastError());
  API_END
}
int b200pir_ntt4096(b200pir_ctx* c, uint64_t* polys, size_t count, int inverse) {
  API_BEGIN
  if (!c || (!polys && count)) throw Error(B200PIR_E_BADARG, "null argument");
  Guard gd(c);
  if (count == 0) return 0;
  const size_t words = count * 2 * 4096;
  DevBuf<uint64_t> wide;
  DevBuf<uint32_t> nar(words);
  upload_narrow(c, nar.p, wide, polys, words);
  launch_ntt32_4k(c->dp.q[0], c->dp.q[1], c->d_tw4k.p, nar.p, count, inverse != 0, c->stream);
  download_widen(c, polys, nar.p, words);
  B200_CUDA(cudaGetLastError());
  API_END
}

int b200pir_to_ntt(b200pir_ctx* c, uint64_t* out_ntt, const uint64_t* raw, size_t count) {
  API_BEGIN
  if (!c || !out_ntt || !raw) throw Error(B200PIR_E_BADARG, "null argument");
  Guard gd(c);
  DevBuf<uint64_t> in(count * POLY);
  DevBuf<uint32_t> o(count * 2 * POLY);
  B200_CUDA(cudaMemcpyAsync(in.p, raw, in.n * 8, cudaMemcpyHostToDevice, c->stream));
  launch_to_ntt(c->dp, o.p, in.p, count, c->stream);
  download_widen(c, out_ntt, o.p, o.n);
  B200_CUDA(cudaGetLastError());
  API_END
}
int b200pir_from_ntt(b200pir_ctx* c, uint64_t* out_raw, const uint64_t* ntt, size_t count) {
  API_BEGIN
  if (!c || !out_raw || !ntt) throw Error(B200PIR_E_BADARG, "null argument");
  Guard gd(c);
  DevBuf<uint64_t> wide, o(count * POLY);
  DevBuf<uint32_t> in(count * 2 * POLY);
  upload_narrow(c, in.p, wide, ntt, in.n);
  launch_from_ntt(c->dp, o.p, in.p, count, c->stream);
  B200_CUDA(cudaMemcpyAsync(out_raw, o.p, o.n * 8, cudaMemcpyDeviceToHost, c->stream));
  B200_CUDA(cudaStreamSynchronize(c->stream));
  B200_CUDA(cudaGetLastError());
  API_END
}

int b200pir_multiply_reg_by_database(b200pir_ctx* c, b200pir_db* db, uint64_t slice, const uint64_t* v_firstdim,
                                     uint64_t* out) {
  API_BEGIN
  if (!c || !v_firstdim || !out) throw Error(B200PIR_E_BADARG, "null argument");
  Guard gd(c);
  check_db(c, db);
  const DbStore& s = db->single("multiply_reg_by_database: not on a sharded database");
  if (slice >= (uint64_t)c->slices) throw Error(B200PIR_E_SHAPE, "slice out of range");
  const int rows = s.rows;
  const bool zmajor = s.zmajor_product();
  DevBuf<uint64_t> vq((size_t)c->dim0 * 2 * POLY);
  DevBuf<uint4> qd((size_t)c->dim0 * POLY);
  DevBuf<uint32_t> o((size_t)c->slices * rows * 4 * POLY), zm(zmajor ? o.n : 0);
  B200_CUDA(cudaMemcpyAsync(vq.p, v_firstdim, vq.n * 8, cudaMemcpyHostToDevice, c->stream));
  launch_query_to_dev(s.layout.G, qd.p, vq.p, c->stream);
  run_first_dim(c, s, 1, qd.p, Images{}, zmajor ? zm.p : o.p, (int)slice, 1);
  uint32_t* o_slice = o.p + (size_t)slice * rows * 4 * POLY;          // ntt32 [row][ct_row][n][z] of this slice
  if (zmajor) launch_zmajor_to_ntt32(s.layout.F, zm.p, o_slice, (int)slice, c->stream);
  download_widen(c, out, o_slice, (size_t)rows * 4 * POLY);
  B200_CUDA(cudaGetLastError());
  API_END
}

int b200pir_fold_ciphertexts(b200pir_ctx* c, uint64_t* v_cts, size_t num, const uint64_t* v_folding,
                             const uint64_t* v_folding_neg) {
  API_BEGIN
  if (!c || !v_cts) throw Error(B200PIR_E_BADARG, "null argument");
  Guard gd(c);
  if (num == 0 || (num & (num - 1))) throw Error(B200PIR_E_SHAPE, "number of ciphertexts must be a power of two");
  if (num == 1) return 0;                                          // server.rs:394-396
  if (!v_folding) throw Error(B200PIR_E_BADARG, "null argument");
  int dims = 0;
  while (((size_t)1 << dims) < num) dims++;
  if (dims > (int)c->hp.nu_2) throw Error(B200PIR_E_SHAPE, "more ciphertexts than 2^nu_2");
  const size_t mat = (size_t)2 * 2 * c->hp.t_gsw * 2 * POLY;
  DevBuf<uint64_t> cts(num * 2 * POLY), wide;
  DevBuf<uint32_t> vf(c->fold_words());
  B200_CUDA(cudaMemcpyAsync(cts.p, v_cts, cts.n * 8, cudaMemcpyHostToDevice, c->stream));
  upload_narrow(c, vf.p, wide, v_folding, dims * mat);
  // The fast path works on residues, where a raw coefficient q (kernels.h) is stored as 0: its gadget digits would be 0's, and
  // a slot the loop never folds would come back as 0.  process_query never hands q to the fold (its inputs come out of from_ntt),
  // but a caller of this stage may: such inputs take the raw-coefficient path with v_folding_neg computed from v_folding.
  const bool has_q = std::find(v_cts, v_cts + cts.n, c->dp.modulus) != v_cts + cts.n;
  if ((v_folding_neg || has_q) && !c->sparse_fold) {
    // general path: honours an arbitrary v_folding_neg exactly as server.rs:405-425 does
    DevBuf<uint32_t> vfn(c->fold_words());
    if (v_folding_neg) upload_narrow(c, vfn.p, wide, v_folding_neg, dims * mat);
    else launch_folding_neg(c->dp, vfn.p, vf.p, dims, (int)c->hp.t_gsw, c->bits_gsw, c->stream);
    run_fold(c, cts.p, 1, num * 2 * POLY, num, dims - 1, vf.p, vfn.p, 1);
  } else {
    // fast path (what process_query uses): v_folding_neg = get_v_folding_neg(v_folding) implied.
    // Round results are copied back so every slot ends up as the reference's in-place loop leaves it.
    // With "sparse_fold" set this is lib/server's fold (compute/fold.rs:15-65): v_folding_neg is then taken to be
    // get_v_folding_neg(v_folding), which is what that server passes (lib/server/src/server.rs).
    DevBuf<uint32_t> a(num * 4 * POLY), b(num * 4 * POLY);
    DevBuf<uint32_t> zflags;
    if (c->sparse_fold) zflags.alloc(num);
    launch_raw_to_res(c->dp, a.p, cts.p, num * 2, c->stream);
    int k = dims - 1;
    for (size_t half = num / 2; half >= 1; half /= 2, k--) {
      launch_fold_res(c->dp, a.p, b.p, 1, num * 4 * POLY, (int)half, vf.p + (size_t)k * mat, c->fold_words(), 1,
                      (int)c->hp.t_gsw, c->bits_gsw, c->live_gsw, zflags.p, c->stream);
      B200_CUDA(cudaMemcpyAsync(a.p, b.p, half * 4 * POLY * 4, cudaMemcpyDeviceToDevice, c->stream));
    }
    launch_res_to_raw(c->dp, cts.p, a.p, num * 2, c->stream);
  }
  B200_CUDA(cudaMemcpyAsync(v_cts, cts.p, cts.n * 8, cudaMemcpyDeviceToHost, c->stream));
  B200_CUDA(cudaStreamSynchronize(c->stream));
  B200_CUDA(cudaGetLastError());
  API_END
}

int b200pir_get_v_folding_neg(b200pir_ctx* c, uint64_t* out, const uint64_t* v_folding) {
  API_BEGIN
  if (!c || !out || !v_folding) throw Error(B200PIR_E_BADARG, "null argument");
  Guard gd(c);
  const size_t words = c->fold_words();
  if (!words) return 0;
  DevBuf<uint64_t> wide;
  DevBuf<uint32_t> in(words), o(words);
  upload_narrow(c, in.p, wide, v_folding, words);
  launch_folding_neg(c->dp, o.p, in.p, (int)c->hp.nu_2, (int)c->hp.t_gsw, c->bits_gsw, c->stream);
  download_widen(c, out, o.p, words);
  B200_CUDA(cudaGetLastError());
  API_END
}

int b200pir_coefficient_expansion(b200pir_ctx* c, b200pir_pp* pp, uint64_t* v) {
  API_BEGIN
  if (!c || !v) throw Error(B200PIR_E_BADARG, "null argument");
  Guard gd(c);
  check_pp(c, pp);
  if (!c->hp.expand_queries) throw Error(B200PIR_E_BADARG, "context was created with expand_queries = 0");
  const size_t words = c->v_words();
  DevBuf<uint64_t> wide;
  DevBuf<uint32_t> dv(words);
  upload_narrow(c, dv.p, wide, v, words);
  run_coefficient_expansion(c, Keys{pp}, dv.p, words, 1, true);
  download_widen(c, v, dv.p, words);
  B200_CUDA(cudaGetLastError());
  API_END
}

int b200pir_expand_query(b200pir_ctx* c, b200pir_pp* pp, const uint64_t* query_ct, uint64_t* out_v_firstdim,
                         uint64_t* out_v_folding) {
  API_BEGIN
  if (!c || !query_ct || !out_v_firstdim) throw Error(B200PIR_E_BADARG, "null argument");
  Guard gd(c);
  check_pp(c, pp);
  if (!c->hp.expand_queries) throw Error(B200PIR_E_BADARG, "context was created with expand_queries = 0");
  c->ensure_workspace(1, 1);
  B200_CUDA(cudaMemcpyAsync(c->w_query.p, query_ct, 2 * POLY * 8, cudaMemcpyHostToDevice, c->stream));
  run_expand_query(c, Keys{pp}, c->w_query.p, c->w_v.p, c->w_qdev.p, c->w_vfold.p, 1, nullptr);
  // q_dev -> reference layout [z][j][r]
  const size_t qwords = (size_t)c->dim0 * 2 * POLY;
  std::vector<uint32_t> hq(qwords * 2);
  B200_CUDA(cudaMemcpyAsync(hq.data(), c->w_qdev.p, hq.size() * 4, cudaMemcpyDeviceToHost, c->stream));
  B200_CUDA(cudaStreamSynchronize(c->stream));
  for (int j = 0; j < c->dim0; j++)
    for (int z = 0; z < POLY; z++) {
      const uint32_t* cell = hq.data() + (((size_t)(j >> 1) * 2 + (j & 1)) * POLY + z) * 4;
      out_v_firstdim[((size_t)z * c->dim0 + j) * 2 + 0] = (uint64_t)cell[0] | ((uint64_t)cell[1] << 32);
      out_v_firstdim[((size_t)z * c->dim0 + j) * 2 + 1] = (uint64_t)cell[2] | ((uint64_t)cell[3] << 32);
    }
  if (out_v_folding && c->fold_words()) download_widen(c, out_v_folding, c->w_vfold.p, c->fold_words());
  B200_CUDA(cudaGetLastError());
  API_END
}

int b200pir_pack(b200pir_ctx* c, b200pir_pp* pp, const uint64_t* v_ct, uint64_t* out_ntt) {
  API_BEGIN
  if (!c || !v_ct || !out_ntt) throw Error(B200PIR_E_BADARG, "null argument");
  Guard gd(c);
  check_pp(c, pp);
  const auto& hp = c->hp;
  const size_t nn = hp.n * hp.n, outp = (hp.n + 1) * hp.n;
  DevBuf<uint64_t> cts(nn * 2 * POLY), raw(outp * POLY);
  DevBuf<uint32_t> o(outp * 2 * POLY), res(nn * 4 * POLY);
  B200_CUDA(cudaMemcpyAsync(cts.p, v_ct, cts.n * 8, cudaMemcpyHostToDevice, c->stream));
  launch_raw_to_res(c->dp, res.p, cts.p, nn * 2, c->stream);
  launch_pack(c->dp, raw.p, 0, res.p, 4 * POLY, 0, 1, pp_table(c, Keys{pp}, 1).pack, (int)hp.n, 1, (int)hp.t_conv, c->bits_conv, c->live_conv, (int)hp.version, c->stream,
              cts.p);
  // the reference's pack returns the NTT-form matrix (server.rs:467); the kernel already applied .raw()
  launch_to_ntt(c->dp, o.p, raw.p, outp, c->stream);
  download_widen(c, out_ntt, o.p, o.n);
  B200_CUDA(cudaGetLastError());
  API_END
}

int b200pir_encode(b200pir_ctx* c, const uint64_t* v_packed_raw, uint8_t* out, size_t* out_len) {
  API_BEGIN
  if (!c || !v_packed_raw || !out) throw Error(B200PIR_E_BADARG, "null argument");
  Guard gd(c);
  const auto& hp = c->hp;
  const size_t words = (size_t)hp.instances * (hp.n + 1) * hp.n * POLY;
  DevBuf<uint64_t> in(words);
  DevBuf<uint8_t> o(c->response_bytes);
  B200_CUDA(cudaMemcpyAsync(in.p, v_packed_raw, words * 8, cudaMemcpyHostToDevice, c->stream));
  launch_encode(c->dp, o.p, c->response_bytes, in.p, 0, 1, (int)hp.n, (int)hp.instances, c->q2, (int)hp.q2_bits, c->q1, c->q1_bits, c->stream);
  B200_CUDA(cudaMemcpyAsync(out, o.p, c->response_bytes, cudaMemcpyDeviceToHost, c->stream));
  B200_CUDA(cudaStreamSynchronize(c->stream));
  if (out_len) *out_len = c->response_bytes;
  B200_CUDA(cudaGetLastError());
  API_END
}

// ---------------------------------------------------------------- process_query
extern "C++" {
namespace {
// Where the responses of a query call go: device memory `dev` (count * response_bytes, stream-ordered: the call returns without
// waiting for them), or host memory, `host` (count * response_bytes) or `each` (response_bytes per query); then the call waits,
// and *len, where given, becomes response_bytes
struct Responses {
  uint8_t* dev = nullptr;
  uint8_t* host = nullptr;
  uint8_t* const* each = nullptr;
  size_t* len = nullptr;
};

// the survivors `s`, [count][slices], into partial_dev as a dense buffer of residue-form ciphertexts; partial_dev may be on
// another device (a part of a sharded database gathering to the home device)
void gather_survivors(b200pir_ctx* c, Survivors s, size_t count, uint32_t* partial_dev) {
  B200_CUDA(cudaMemcpy2DAsync(partial_dev, 4 * POLY * 4, s.p, s.stride * 4, 4 * POLY * 4, count * c->slices,
                              cudaMemcpyDefault, c->stream));
}

// The last phase for queries [first, first + count) of the `total_count` whose partial survivors `world` ranks gathered: their
// fold across the ranks with the folding matrices v_folding, then pack and encode into out_dev
void run_finish(b200pir_ctx* c, Keys keys, const uint32_t* gathered_dev, size_t world, size_t total_count, size_t first,
                size_t count, const uint32_t* v_folding, uint8_t* out_dev) {
  // gathered: [world][total_count][slices][ct]  ->  w_mult as [count][slices][world][ct]   (ct = 4*2048 u32)
  const size_t ct = 4 * POLY;
  for (size_t w = 0; w < world; w++)
    B200_CUDA(cudaMemcpy2DAsync(c->w_mult.p + w * ct, world * ct * 4, gathered_dev + (w * total_count + first) * c->slices * ct,
                                ct * 4, ct * 4, count * c->slices, cudaMemcpyDeviceToDevice, c->stream));
  int dims = 0;
  while (((size_t)1 << dims) < world) dims++;
  Survivors s{c->w_mult.p, world * ct};
  {
    b200pir_ctx::Scope sc(c, ST_FOLD);
    if (world > 1) s.p = run_fold_res(c, c->w_mult.p, c->w_cts.p, count * c->slices, s.stride, world, dims - 1, v_folding, c->slices, c->sparse_fold);
  }
  run_pack_encode(c, keys, s, count, out_dev);
}

// The query schedule of a sharded database (b200pir_db_create_sharded) once the calling context c, the home, has put the
// call's first-dimension operand (`images`, or c->w_qdev) and folding matrices (c->w_vfold) in place: every part runs the
// first dimension and the fold rounds nu_2 - 1 .. log2 G on its store, on the stream of its own context (db->worker), and
// gathers its survivors into slot g of db->gathered; c then folds across the parts (rounds log2 G - 1 .. 0), packs and
// encodes into out_dev.  A part on c's device reads c's buffers directly; a part on another device receives them in its own
// buffers by copy engine.
// Options that change the response bytes ("sparse_fold") are c's for every part.
//
// Stream order, with no host synchronisation:
//  - Every part's stream waits on db->expanded, recorded on c's stream after the expansion, before it copies or reads the
//    operands; c's stream waits on every part's `done`, recorded after the part's gather, before the finish.  So the next
//    call's expansion, queued on c's stream after this finish, cannot overwrite an operand a part is still copying or reading.
//    A call from another context on the home device first waits on db->finished, which carries the same order over.
//  - A part's receive buffers are written only by copies on the part's own stream, queued after that stream's previous first
//    dimension, which read them: the copies of the next call cannot overtake it.
//  - db->gathered is written by the parts after db->expanded and read by the finish before db->finished, so the next call's
//    gathers come after this call's finish has read it.
void run_shards(b200pir_ctx* c, b200pir_db* db, Keys keys, size_t count, Images images, uint8_t* out_dev) {
  const size_t G = db->parts.size();
  db->ensure_exchange(count);
  const size_t op_bytes = db->operand_bytes(count), fold_bytes = count * c->fold_words() * 4;
  const uint8_t* op = images.p ? images.p : reinterpret_cast<const uint8_t*>(c->w_qdev.p);
  B200_CUDA(cudaEventRecord(db->expanded, c->stream));
  for (size_t g = 0; g < G; g++) {
    b200pir_db::Part& part = db->parts[g];
    b200pir_ctx* x = db->worker(c, g);
    B200_CUDA(cudaSetDevice(x->device));
    if (x->stream != c->stream) B200_CUDA(cudaStreamWaitEvent(x->stream, db->expanded, 0));
    const uint8_t* xop = op;
    const uint32_t* xfold = c->w_vfold.p;
    if (x->device != c->device) {
      B200_CUDA(cudaMemcpyPeerAsync(part.operand.p, x->device, op, c->device, op_bytes, x->stream));
      if (fold_bytes) B200_CUDA(cudaMemcpyPeerAsync(part.vfold.p, x->device, c->w_vfold.p, c->device, fold_bytes, x->stream));
      xop = part.operand.p;
      xfold = part.vfold.p;
    }
    x->ensure_workspace_lite(count, part.store->rows);
    const Images xim{images.p ? xop : nullptr, images.per_group};
    const Survivors s = run_first_dim_and_fold(x, *part.store, count, images.p ? nullptr : reinterpret_cast<const uint4*>(xop),
                                               xim, xfold, c->sparse_fold);
    gather_survivors(x, s, count, db->gathered.p + g * count * c->slices * 4 * POLY);
    B200_CUDA(cudaEventRecord(part.done, x->stream));
  }
  B200_CUDA(cudaSetDevice(c->device));
  for (size_t g = 0; g < G; g++)
    if (db->worker(c, g)->stream != c->stream) B200_CUDA(cudaStreamWaitEvent(c->stream, db->parts[g].done, 0));
  run_finish(c, keys, db->gathered.p, G, count, 0, count, c->w_vfold.p, out_dev);
  B200_CUDA(cudaEventRecord(db->finished, c->stream));
}

// One single-GPU query call on `count` queries: the checks, stage(), which puts the queries into the workspace (w_query, or
// w_qdev and w_vfold for direct upload), one database pass and the responses.  `keys.each`: a multi-client batch, whose
// workspace is sized once for a full coalesced batch (batch sizes vary from call to call, the buffers do not).
// `needs_expand`: the queries are ciphertexts, which only an expanding context takes.
// A sharded database runs the same checks and staging and then run_shards in place of the one-context database pass.
template <typename Stage>
void run_queries(b200pir_ctx* c, b200pir_db* db, Keys keys, size_t count, bool needs_expand, Stage stage,
                 const Responses& out) {
  Guard gd(c, db);
  check_db(c, db);
  if (keys.each)
    for (size_t i = 0; i < count; i++) check_pp(c, keys.each[i]);
  else
    check_pp(c, keys.one);
  if (!db->whole()) throw Error(B200PIR_E_BADARG, "sharded database: use the stage_a / stage_b entry points");
  if (needs_expand && !c->hp.expand_queries)
    throw Error(B200PIR_E_BADARG, keys.each ? "multi-client batches need expand_queries" : "batch entry point needs expand_queries");
  if (count == 0) return;
  // a sharded database's home workspace holds the finish's G survivors per (query, slice), not local rows
  const size_t rows = db->sharded() ? db->parts.size() : (size_t)db->parts[0].store->rows;
  c->ensure_workspace(keys.each && c->coalesce ? std::max(count, b200pir_ctx::kCoalesceMax) : count, rows);
  c->prof_reset();
  if (db->sharded()) B200_CUDA(cudaStreamWaitEvent(c->stream, db->finished, 0));
  stage();
  // format-2 databases get their operand as tile images straight from the expansion
  const bool images = db->parts[0].store->layout.format == 2 && c->hp.expand_queries;
  run_prepare(c, keys, count, images);
  const Images im{images ? c->w_qt.p : nullptr, 16};
  uint8_t* resp = out.dev ? out.dev : c->w_resp.p;
  if (db->sharded()) run_shards(c, db, keys, count, im, resp);
  else run_pack_encode(c, keys, run_first_dim_and_fold(c, *db->parts[0].store, count, c->w_qdev.p, im, c->w_vfold.p, c->sparse_fold), count, resp);
  if (!out.dev) {
    const size_t rb = c->response_bytes;
    if (out.each)
      for (size_t i = 0; i < count; i++)
        B200_CUDA(cudaMemcpyAsync(out.each[i], c->w_resp.p + i * rb, rb, cudaMemcpyDeviceToHost, c->stream));
    else
      B200_CUDA(cudaMemcpyAsync(out.host, c->w_resp.p, count * rb, cudaMemcpyDeviceToHost, c->stream));
    B200_CUDA(cudaStreamSynchronize(c->stream));
    if (c->profile == 1) c->prof_collect();
    if (out.len) *out.len = rb;
  }
  B200_CUDA(cudaGetLastError());
}

// the queries of a multi-client batch into w_query: per query a host ciphertext cts[i] or, where bytes[i] is given, the
// serialized query bytes[i]
void stage_each(b200pir_ctx* c, const uint64_t* const* cts, const uint8_t* const* bytes, size_t count) {
  for (size_t i = 0; i < count; i++) {
    if (bytes && bytes[i]) deserialize_queries(c, bytes[i], 1, c->w_query.p + i * 2 * POLY);
    else B200_CUDA(cudaMemcpyAsync(c->w_query.p + i * 2 * POLY, cts[i], 2 * POLY * 8, cudaMemcpyHostToDevice, c->stream));
  }
}
}  // namespace
}  // extern "C++"

int b200pir_process_query_batch_dev(b200pir_ctx* c, b200pir_db* db, b200pir_pp* pp, const uint64_t* query_cts_dev,
                                    size_t count, uint8_t* out_dev) {
  API_BEGIN
  if (!c || !out_dev || !query_cts_dev) throw Error(B200PIR_E_BADARG, "null argument");
  run_queries(c, db, Keys{pp}, count, true, [&] {
    B200_CUDA(cudaMemcpyAsync(c->w_query.p, query_cts_dev, count * 2 * POLY * 8, cudaMemcpyDeviceToDevice, c->stream));
  }, Responses{out_dev});
  API_END
}

int b200pir_process_query_batch(b200pir_ctx* c, b200pir_db* db, b200pir_pp* pp, const uint64_t* query_cts, size_t count,
                                uint8_t* out, size_t* out_len_each) {
  API_BEGIN
  if (!c || !out || !query_cts) throw Error(B200PIR_E_BADARG, "null argument");
  run_queries(c, db, Keys{pp}, count, true, [&] {
    B200_CUDA(cudaMemcpyAsync(c->w_query.p, query_cts, count * 2 * POLY * 8, cudaMemcpyHostToDevice, c->stream));
  }, Responses{nullptr, out, nullptr, out_len_each});
  API_END
}

namespace {
// one query through the combiner (see b200pir_ctx::Pending)
int coalesced_query(b200pir_ctx* c, b200pir_db* db, b200pir_pp* pp, const uint64_t* query_ct, const uint8_t* query_bytes,
                    uint8_t* out) {
  b200pir_ctx::Pending me;
  me.db = db; me.pp = pp; me.query_ct = query_ct; me.query_bytes = query_bytes; me.out = out;
  std::unique_lock<std::mutex> lk(c->qmu);
  c->pending.push_back(&me);
  c->qcv.notify_all();                       // a leader may be holding its batch open for us
  while (!me.done) {
    if (c->leader_active) { c->qcv.wait(lk); continue; }
    // become the leader: take the queued requests for the database at the head of the queue
    c->leader_active = true;
    if (c->coalesce_window_us > 0 && c->last_batch > 1 && c->pending.size() < std::min(c->last_batch, b200pir_ctx::kPassQueries)) {
      const auto now = std::chrono::steady_clock::now();
      if (now - c->last_batch_end < std::chrono::milliseconds(1)) {
        const size_t want = std::min(c->last_batch, b200pir_ctx::kPassQueries);
        c->qcv.wait_until(lk, now + std::chrono::microseconds(c->coalesce_window_us), [&] { return c->pending.size() >= want; });
      }
    }
    std::vector<b200pir_ctx::Pending*> batch;
    b200pir_db* bdb = c->pending.front()->db;
    size_t avail = 0;
    for (auto* p : c->pending) avail += p->db == bdb;
    size_t take = std::min(avail, b200pir_ctx::kCoalesceMax);
    if (take > b200pir_ctx::kPassQueries) take -= take % b200pir_ctx::kPassQueries;
    for (auto it = c->pending.begin(); it != c->pending.end() && batch.size() < take;) {
      if ((*it)->db == bdb) { batch.push_back(*it); it = c->pending.erase(it); } else ++it;
    }
    lk.unlock();
    int rc = 0;
    std::string err;
    try {
      std::vector<b200pir_pp*> pps; std::vector<const uint64_t*> cts; std::vector<const uint8_t*> bys; std::vector<uint8_t*> outs;
      for (auto* p : batch) { pps.push_back(p->pp); cts.push_back(p->query_ct); bys.push_back(p->query_bytes); outs.push_back(p->out); }
      run_queries(c, bdb, Keys{nullptr, pps.data()}, batch.size(), true, [&] { stage_each(c, cts.data(), bys.data(), batch.size()); },
                  Responses{nullptr, nullptr, outs.data()});
    } catch (const std::exception& e) { rc = fail(e); err = e.what(); }
    lk.lock();
    c->coalesced_batches++; c->coalesced_queries += batch.size();
    c->last_batch = batch.size();
    c->last_batch_end = std::chrono::steady_clock::now();
    for (auto* p : batch) { p->rc = rc; p->err = err; p->done = true; }
    c->leader_active = false;
    c->qcv.notify_all();
  }
  if (me.rc) g_last_error = me.err;
  return me.rc;
}
}  // namespace

int b200pir_process_queries(b200pir_ctx* c, b200pir_db* db, b200pir_pp* const* pps, const uint64_t* const* query_cts, size_t count,
                            uint8_t* const* outs) {
  API_BEGIN
  if (!c || !pps || !query_cts || !outs) throw Error(B200PIR_E_BADARG, "null argument");
  for (size_t i = 0; i < count; i++)
    if (!pps[i] || !query_cts[i] || !outs[i]) throw Error(B200PIR_E_BADARG, "null entry");
  if (count == 0) return 0;
  run_queries(c, db, Keys{nullptr, pps}, count, true, [&] { stage_each(c, query_cts, nullptr, count); }, Responses{nullptr, nullptr, outs});
  API_END
}
int b200pir_coalesce_stats(b200pir_ctx* c, uint64_t* batches, uint64_t* queries) {
  API_BEGIN
  if (!c) throw Error(B200PIR_E_BADARG, "null ctx");
  std::lock_guard<std::mutex> lk(c->qmu);
  if (batches) *batches = c->coalesced_batches;
  if (queries) *queries = c->coalesced_queries;
  API_END
}

// process_query over the wire format: `count` serialized queries (Query::serialize, client.rs:279-301) back to back
int b200pir_process_query_bytes(b200pir_ctx* c, b200pir_db* db, b200pir_pp* pp, const uint8_t* queries, size_t len,
                                size_t count, uint8_t* out, size_t* out_len_each) {
  API_BEGIN
  if (!c || !out || !queries) throw Error(B200PIR_E_BADARG, "null argument");
  if (len != count * c->query_bytes) throw Error(B200PIR_E_SHAPE, "queries: expected " + std::to_string(count * c->query_bytes) + " bytes");
  if (count == 1 && c->coalesce && c->hp.expand_queries && db && pp) {          // the /private-read handler's call: one query per request
    const int rc = coalesced_query(c, db, pp, nullptr, queries, out);
    if (rc == 0 && out_len_each) *out_len_each = c->response_bytes;
    return rc;
  }
  run_queries(c, db, Keys{pp}, count, false, [&] {
    if (c->hp.expand_queries) {
      deserialize_queries(c, queries, count, c->w_query.p);
    } else {
      // direct upload (client.rs:316-327; the body lib/server's handler parses at bin/server.rs:122-137 is setup || query):
      // every query arrives expanded; nothing to prepare beyond the deserialization
      for (size_t i = 0; i < count; i++) deserialize_query_direct(c, queries + i * c->query_bytes, i);
    }
  }, Responses{nullptr, out, nullptr, out_len_each});
  API_END
}

int b200pir_process_query(b200pir_ctx* c, b200pir_db* db, b200pir_pp* pp, const uint64_t* query_ct, const uint64_t* v_buf,
                          const uint64_t* v_ct, uint8_t* out, size_t* out_len) {
  if (!c) { g_last_error = "null ctx"; return B200PIR_E_BADARG; }
  if (c->hp.expand_queries) {
    if (!query_ct || !out || !db || !pp) { g_last_error = "null argument"; return B200PIR_E_BADARG; }
    if (!c->coalesce) return b200pir_process_query_batch(c, db, pp, query_ct, 1, out, out_len);
    const int rc = coalesced_query(c, db, pp, query_ct, nullptr, out);
    if (rc == 0 && out_len) *out_len = c->response_bytes;
    return rc;
  }
  API_BEGIN
  if (!v_buf || (!v_ct && c->hp.nu_2) || !out) throw Error(B200PIR_E_BADARG, "null argument");
  DevBuf<uint64_t> vq, raw;        // staging, in use until the call's final synchronise
  run_queries(c, db, Keys{pp}, 1, false, [&] {
    // server.rs:666-678: v_reg_reoriented = query.v_buf ; v_folding = v_ct.map(ntt)
    vq.alloc((size_t)c->dim0 * 2 * POLY);
    B200_CUDA(cudaMemcpyAsync(vq.p, v_buf, vq.n * 8, cudaMemcpyHostToDevice, c->stream));
    launch_query_to_dev(db->parts[0].store->layout.G, c->w_qdev.p, vq.p, c->stream);
    const size_t npolys = (size_t)c->hp.nu_2 * 2 * 2 * c->hp.t_gsw;
    raw.alloc(std::max<size_t>(npolys, 1) * POLY);
    if (npolys) {
      B200_CUDA(cudaMemcpyAsync(raw.p, v_ct, npolys * POLY * 8, cudaMemcpyHostToDevice, c->stream));
      launch_to_ntt(c->dp, c->w_vfold.p, raw.p, npolys, c->stream);
    }
  }, Responses{nullptr, out, nullptr, out_len});
  API_END
}

// ---- multi-GPU building blocks: the three phases with caller-owned device buffers in between, so the host can put a
// collective between them (bench.py: queries are expanded by the rank that received them, everything is all-gathered)
namespace {
// The expansion phase of `count` queries into the caller's buffers: the first-dimension operand as q_dev or, with `images`, as
// the tile images of one group of 1..16 queries; the folding matrices into v_folding_dev
int expand_dev(b200pir_ctx* c, b200pir_pp* pp, const uint64_t* query_cts_dev, size_t count, void* operand_dev,
               uint32_t* v_folding_dev, bool images) {
  API_BEGIN
  if (!c || !query_cts_dev || !operand_dev || (!v_folding_dev && c->hp.nu_2)) throw Error(B200PIR_E_BADARG, "null argument");
  Guard gd(c);
  check_pp(c, pp);
  if (!c->hp.expand_queries) throw Error(B200PIR_E_BADARG, "needs expand_queries");
  if (images) {
    if (count == 0 || count > 16) throw Error(B200PIR_E_SHAPE, "one image holds 1..16 queries");
    if (!tc5_supported(make_tc5_geom(c->dim0, 32))) throw Error(B200PIR_E_UNSUPPORTED, "dim0 too large for the wgmma kernel");
  }
  if (count == 0) return 0;
  c->w_v.ensure(count * c->v_words());
  c->prof_reset();
  {
    b200pir_ctx::Scope sc(c, ST_EXPAND);
    run_expand_query(c, Keys{pp}, query_cts_dev, c->w_v.p, images ? nullptr : (uint4*)operand_dev, v_folding_dev, (int)count,
                     images ? (uint8_t*)operand_dev : nullptr);
  }
  B200_CUDA(cudaGetLastError());
  API_END
}

// The first dimension and local fold of `count` queries, their survivors into partial_dev: the operand as q_dev or, with
// `images`, as tile images of per_group queries each (format-2 databases)
int first_dim_fold_dev(b200pir_ctx* c, b200pir_db* db, const void* operand_dev, size_t count, bool images, size_t per_group,
                       const uint32_t* v_folding_dev, uint32_t* partial_dev) {
  API_BEGIN
  if (!c || !operand_dev || !partial_dev || (!v_folding_dev && c->hp.nu_2)) throw Error(B200PIR_E_BADARG, "null argument");
  Guard gd(c);
  check_db(c, db);
  const DbStore& s = db->single("a sharded database runs its own schedule: use the query entry points");
  if (images) {
    if (s.layout.format != 2) throw Error(B200PIR_E_BADARG, "tile images need a wgmma-layout database (db_format 2)");
    if (per_group == 0 || per_group > 16) throw Error(B200PIR_E_SHAPE, "one image holds 1..16 queries");
  }
  if (count == 0) return 0;
  c->ensure_workspace_lite(count, s.rows);
  const uint4* qdev = images ? nullptr : (const uint4*)operand_dev;
  const Images im{images ? (const uint8_t*)operand_dev : nullptr, per_group};
  gather_survivors(c, run_first_dim_and_fold(c, s, count, qdev, im, v_folding_dev, c->sparse_fold), count, partial_dev);
  B200_CUDA(cudaGetLastError());
  API_END
}
}  // namespace

int b200pir_expand_queries_dev(b200pir_ctx* c, b200pir_pp* pp, const uint64_t* query_cts_dev, size_t count,
                               void* q_expanded_dev, uint32_t* v_folding_dev) {
  return expand_dev(c, pp, query_cts_dev, count, q_expanded_dev, v_folding_dev, false);
}
int b200pir_first_dim_fold_dev(b200pir_ctx* c, b200pir_db* db, const void* q_expanded_dev, const uint32_t* v_folding_dev,
                               size_t count, uint32_t* partial_dev) {
  return first_dim_fold_dev(c, db, q_expanded_dev, count, false, 0, v_folding_dev, partial_dev);
}
// The same two phases with the first-dimension operand exchanged as operand tile images (format-2 databases): the rank that expands a
// group of <= 16 queries also re-tiles it, once; the receivers multiply straight from the image.
size_t b200pir_query_image_bytes(b200pir_ctx* c) { return c ? tc5_query_bytes(make_tc5_geom(c->dim0, 32)) : 0; }
int b200pir_expand_queries_images_dev(b200pir_ctx* c, b200pir_pp* pp, const uint64_t* query_cts_dev, size_t count, void* image_dev,
                                      uint32_t* v_folding_dev) {
  return expand_dev(c, pp, query_cts_dev, count, image_dev, v_folding_dev, true);
}
int b200pir_first_dim_fold_images_dev(b200pir_ctx* c, b200pir_db* db, const void* images_dev, size_t groups, size_t per_group,
                                      const uint32_t* v_folding_dev, uint32_t* partial_dev) {
  return first_dim_fold_dev(c, db, images_dev, groups * per_group, true, per_group, v_folding_dev, partial_dev);
}
int b200pir_finish_queries_dev(b200pir_ctx* c, b200pir_pp* pp, const uint32_t* gathered_dev, size_t world, size_t total_count,
                               size_t first, size_t count, const uint32_t* v_folding_dev, uint8_t* out_dev) {
  API_BEGIN
  if (!c || !gathered_dev || !out_dev || (!v_folding_dev && world > 1)) throw Error(B200PIR_E_BADARG, "null argument");
  Guard gd(c);
  check_pp(c, pp);
  if (world == 0 || (world & (world - 1)) || world > (size_t)c->num_per) throw Error(B200PIR_E_SHAPE, "bad world size");
  if (first + count > total_count) throw Error(B200PIR_E_SHAPE, "query range out of bounds");
  if (count == 0) return 0;
  c->ensure_workspace_lite(count, world);
  run_finish(c, Keys{pp}, gathered_dev, world, total_count, first, count, v_folding_dev, out_dev);
  B200_CUDA(cudaGetLastError());
  API_END
}

int b200pir_query_stage_a_dev(b200pir_ctx* c, b200pir_db* db, b200pir_pp* pp, const uint64_t* query_cts_dev, size_t count,
                              uint32_t* partial_dev) {
  API_BEGIN
  if (!c || !query_cts_dev || !partial_dev) throw Error(B200PIR_E_BADARG, "null argument");
  Guard gd(c);
  check_db(c, db);
  check_pp(c, pp);
  const DbStore& s = db->single("a sharded database runs its own schedule: use the query entry points");
  if (!c->hp.expand_queries) throw Error(B200PIR_E_BADARG, "needs expand_queries");
  c->ensure_workspace(count, s.rows);
  c->prof_reset();
  B200_CUDA(cudaMemcpyAsync(c->w_query.p, query_cts_dev, count * 2 * POLY * 8, cudaMemcpyDeviceToDevice, c->stream));
  run_prepare(c, Keys{pp}, count, false);
  gather_survivors(c, run_first_dim_and_fold(c, s, count, c->w_qdev.p, Images{}, c->w_vfold.p, c->sparse_fold), count, partial_dev);
  B200_CUDA(cudaGetLastError());
  API_END
}

int b200pir_query_stage_b_dev(b200pir_ctx* c, b200pir_pp* pp, const uint32_t* gathered_dev, size_t world, size_t count,
                              uint8_t* out_dev) {
  API_BEGIN
  if (!c || !gathered_dev || !out_dev) throw Error(B200PIR_E_BADARG, "null argument");
  Guard gd(c);
  check_pp(c, pp);
  if (world == 0 || (world & (world - 1)) || world > (size_t)c->num_per) throw Error(B200PIR_E_SHAPE, "bad world size");
  c->ensure_workspace(count, world);
  run_finish(c, Keys{pp}, gathered_dev, world, count, 0, count, c->w_vfold.p, out_dev);
  B200_CUDA(cudaGetLastError());
  API_END
}

unsigned long long b200pir_kernel_launches(void) { return g_kernel_launches; }

// ---- peer memory (CUDA IPC) for the copy-engine exchange of the multi-GPU flow
int b200pir_peer_alloc(int device, size_t bytes, void** out_ptr, uint8_t out_handle[64]) {
  API_BEGIN
  if (!out_ptr || !out_handle || !bytes) throw Error(B200PIR_E_BADARG, "null or empty argument");
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
  B200_CUDA(cudaSetDevice(device));
  void* p = nullptr;
  B200_CUDA(cudaMalloc(&p, bytes));
  cudaIpcMemHandle_t h;
  cudaError_t e = cudaIpcGetMemHandle(&h, p);
  if (e != cudaSuccess) { cudaFree(p); throw Error(B200PIR_E_CUDA, std::string("cudaIpcGetMemHandle: ") + cudaGetErrorString(e)); }
  std::memcpy(out_handle, &h, 64);
  *out_ptr = p;
  API_END
}
int b200pir_peer_open(int device, const uint8_t handle[64], void** out_ptr) {
  API_BEGIN
  if (!handle || !out_ptr) throw Error(B200PIR_E_BADARG, "null argument");
  B200_CUDA(cudaSetDevice(device));
  cudaIpcMemHandle_t h;
  std::memcpy(&h, handle, 64);
  B200_CUDA(cudaIpcOpenMemHandle(out_ptr, h, cudaIpcMemLazyEnablePeerAccess));
  API_END
}
int b200pir_peer_close(int device, void* mapped_ptr) {
  API_BEGIN
  B200_CUDA(cudaSetDevice(device));
  if (mapped_ptr) B200_CUDA(cudaIpcCloseMemHandle(mapped_ptr));
  API_END
}
int b200pir_peer_free(int device, void* ptr) {
  API_BEGIN
  B200_CUDA(cudaSetDevice(device));
  if (ptr) B200_CUDA(cudaFree(ptr));
  API_END
}
int b200pir_peer_copy_async(void* dst, const void* src, size_t bytes, void* cuda_stream) {
  API_BEGIN
  if (!dst || !src) throw Error(B200PIR_E_BADARG, "null argument");
  if (bytes) B200_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDefault, (cudaStream_t)cuda_stream));
  API_END
}

int b200pir_last_stage_ms(b200pir_ctx* c, double* out9) {
  API_BEGIN
  if (!c || !out9) throw Error(B200PIR_E_BADARG, "null argument");
  Guard gd(c);
  c->prof_collect();
  for (int i = 0; i < 9; i++) out9[i] = c->last_ms[i];
  API_END
}

}  // extern "C"
