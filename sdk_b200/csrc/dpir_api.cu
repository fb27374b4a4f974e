// C-ABI implementation of DoublePIR (include/b200pir.h): the resident matrix handle, its matvecs, the one-shot ops, setup()
// and the banded offline load, as host-side orchestration of the dpir_*.cu kernels.  The answer() server is in
// dpir_server_api.cu.
#include "dpir_api.hpp"
#include <cerrno>
#include <fcntl.h>
#include <sys/stat.h>
#include <unistd.h>
#include <cmath>
#include <functional>
#include <memory>
#include <string>
#include <thread>

b200pir_dpir_info b200pir::dpir_info(const b200pir_dpir_params* prm, uint64_t num_entries, uint64_t bits, uint64_t max_bits) {
  if (!prm) throw Error(B200PIR_E_BADARG, "null argument");
  if (num_entries == 0 || bits < 1 || bits > max_bits)
    throw Error(B200PIR_E_BADARG, "DbInfo: need entries > 0 and 1 <= bits_per_entry <= " + std::to_string(max_bits));
  if (!prm->n || !prm->l || !prm->m) throw Error(B200PIR_E_BADARG, "params: n, l and m must be positive");
  if (prm->logq != 32) throw Error(B200PIR_E_UNSUPPORTED, "params: logq must be 32 (doublepir.rs:9)");
  if (prm->p < 2 || prm->p > 1024) throw Error(B200PIR_E_UNSUPPORTED, "params: p must lie in [2, 2^10] (squish basis, database.rs:274)");
  b200pir_dpir_info o;
  const double log_p = std::log2((double)prm->p);
  uint64_t elems;
  if ((double)bits <= log_p) {                                   // pack several entries into one Z_p element
    o.packing = (uint64_t)log_p / bits;
    elems = (uint64_t)std::ceil((double)num_entries / (double)o.packing);
    o.ne = 1;
  } else {                                                       // several Z_p elements per entry
    o.packing = 0;
    o.ne = (uint64_t)std::ceil((double)bits / log_p);
    if (num_entries > UINT64_MAX / o.ne) throw Error(B200PIR_E_SHAPE, "DbInfo: more Z_p elements than the database holds");
    elems = num_entries * o.ne;
  }
  o.x = o.ne;                                                    // `while info.ne % info.x != 0 { info.x += 1 }` from x = ne
  o.delta = (uint64_t)std::ceil((double)prm->logq / log_p);
  if (prm->l > UINT64_MAX / prm->m || elems > prm->l * prm->m) throw Error(B200PIR_E_SHAPE, "DbInfo: more Z_p elements than l * m");
  return o;
}

b200pir::DpirShardRows b200pir::dpir_shard_rows(uint64_t l, uint64_t x, size_t shards, size_t index) {
  const uint64_t unit = 3 * x, units = (l + unit - 1) / unit;
  if (shards == 0 || shards > units)
    throw Error(B200PIR_E_SHAPE, "cannot split " + std::to_string(units) + " units of 3x rows over " + std::to_string(shards) + " shards");
  const uint64_t per = units / shards, extra = units % shards;
  const uint64_t u0 = index * per + std::min<uint64_t>(index, extra), u1 = u0 + per + (index < extra ? 1 : 0);
  const uint64_t r0 = u0 * unit, r1 = std::min(l, u1 * unit);
  return DpirShardRows{r0, r1 - r0};
}

extern "C" {

namespace {
b200pir_dpir* dpir_new(int device, uint64_t rows, uint64_t cols) {
  use_device(device);
  if (rows == 0 || cols == 0) throw Error(B200PIR_E_SHAPE, "empty matrix");
  std::unique_ptr<b200pir_dpir> m(new b200pir_dpir());
  m->device = device; m->rows = rows; m->cols = cols;
  B200_CUDA(cudaStreamCreateWithFlags(&m->stream, cudaStreamNonBlocking));
  m->a.alloc(rows * cols);
  m->b.alloc(3 * cols);
  m->out.alloc(rows);
  return m.release();
}
}  // namespace

int b200pir_dpir_create(int device, const uint32_t* a, uint64_t rows, uint64_t cols, b200pir_dpir** out) {
  API_BEGIN
  if (!a || !out) throw Error(B200PIR_E_BADARG, "null argument");
  b200pir_dpir* m = dpir_new(device, rows, cols);
  // on the handle's stream, and waited for: a pageable cudaMemcpy queues behind the legacy default stream's work and may return
  // before its data has landed, while the matvecs run on the non-blocking m->stream
  cudaError_t e = cudaMemcpyAsync(m->a.p, a, rows * cols * 4, cudaMemcpyHostToDevice, m->stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(m->stream);
  if (e != cudaSuccess) { b200pir_dpir_destroy(m); throw Error(B200PIR_E_CUDA, cudaGetErrorString(e)); }
  *out = m;
  API_END
}
int b200pir_dpir_create_synthetic(int device, uint64_t rows, uint64_t cols, uint64_t seed, b200pir_dpir** out) {
  API_BEGIN
  if (!out) throw Error(B200PIR_E_BADARG, "null argument");
  b200pir_dpir* m = dpir_new(device, rows, cols);
  launch_dpir_synth(m->a.p, rows * cols, seed, m->stream);
  cudaError_t e = cudaStreamSynchronize(m->stream);
  if (e != cudaSuccess) { b200pir_dpir_destroy(m); throw Error(B200PIR_E_CUDA, cudaGetErrorString(e)); }
  *out = m;
  API_END
}
namespace {
// doublepir.rs:76-108 setup() in two parts, so that the l x m layout never has to be on the device at once.
// The per-row part, for the centred layout rows [r0, r0 + rows) in d_band (rows x m, device): those rows of h_1 = db.data * a_1
// (against a_1's GEMM image a1_img, through the caller's a image a_img of dpir_gemm_a_bytes(rows, m) bytes) into d_h (l x n),
// and db.data += p/2; db.squish() of the same rows into d_dbsq (l x ceil(m/3)).  No allocation, no synchronisation.
void dpir_setup_rows(const uint32_t* d_band, uint64_t r0, uint64_t rows, uint64_t m, uint64_t n, uint32_t p, const uint8_t* a1_img,
                     uint8_t* a_img, uint32_t* d_h, uint32_t* d_dbsq, cudaStream_t s) {
  launch_dpir_gemm_rows(d_h + r0 * n, a_img, d_band, rows, m, a1_img, n, s);                // h_1 = db.data * a_1
  launch_dpir_add_squish(d_dbsq + r0 * ((m + 2) / 3), d_band, rows, m, p / 2, s);         // db.data += p/2; db.squish()
}
// The tail, on the h_1 rows [r0, r0 + rows) of an l-row database (rows x n, device; r0 a multiple of 3x, rows of x) and the
// whole a2 (l/x x n, device): transpose / expand / concat, h_2 = h_1 * a_2 over the range's columns, h_1 += p/2 and squish,
// a_2_copy.  Host buffers: the range's squished columns [r0 / 3x, ..) of h1_squished ((n delta x) x ceil(l/3x)); h2, the
// range's partial of h_2 (all of it for the range [0, l)); a2_t, skipped when null.  Synchronises s.
void dpir_setup_tail(const uint32_t* d_h, const uint32_t* d_a2, uint64_t l, uint64_t r0, uint64_t rows, uint64_t n, uint32_t p,
                     uint64_t delta, uint64_t x, uint32_t* h1_squished, uint32_t* a2_t, uint32_t* h2, cudaStream_t s) {
  const size_t lx = l / x, rows1 = n * delta * x, lx3 = lx + (3 - lx % 3) % 3, lxg = rows / x, c1 = (lx + 2) / 3, c1g = (lxg + 2) / 3;
  DevBuf<uint32_t> d_hc(rows1 * lxg), d_h2(rows1 * n);
  DevBuf<uint32_t> d_h1sq(rows1 * c1g), d_a2t(a2_t ? n * lx3 : 0);
  launch_dpir_transpose_expand_concat(d_hc.p, d_h, rows, n, p, (int)delta, x, s);       // transpose, expand, concat_cols
  launch_dpir_gemm(d_h2.p, d_hc.p, d_a2 + r0 / x * n, rows1, lxg, n, s);                // h_2 = h_1 * a_2
  launch_dpir_add_squish(d_h1sq.p, d_hc.p, rows1, lxg, p / 2, s);                        // h_1 += p/2; squish
  if (a2_t) launch_dpir_pad_transpose(d_a2t.p, d_a2, lx, n, lx3, s);                     // a_2_copy
  B200_CUDA(cudaMemcpy2DAsync(h1_squished + r0 / (3 * x), c1 * 4, d_h1sq.p, c1g * 4, c1g * 4, rows1, cudaMemcpyDeviceToHost, s));
  if (a2_t) B200_CUDA(cudaMemcpyAsync(a2_t, d_a2t.p, d_a2t.n * 4, cudaMemcpyDeviceToHost, s));
  B200_CUDA(cudaMemcpyAsync(h2, d_h2.p, d_h2.n * 4, cudaMemcpyDeviceToHost, s));
  B200_CUDA(cudaStreamSynchronize(s));
  B200_CUDA(cudaGetLastError());
}
}  // namespace

// doublepir.rs:76-108 setup(): both matrix products on the tensor cores (dpir_gemm.cu), the rest as small kernels.  Host pointers.
int b200pir_dpir_setup(int device, const uint32_t* db, uint64_t l, uint64_t m, const uint32_t* a1, uint64_t n, const uint32_t* a2,
                       uint32_t p, uint64_t delta, uint64_t x, uint32_t* db_squished, uint32_t* h1_squished, uint32_t* a2_t,
                       uint32_t* h2) {
  API_BEGIN
  if (!db || !a1 || !a2 || !db_squished || !h1_squished || !a2_t || !h2) throw Error(B200PIR_E_BADARG, "null argument");
  if (!l || !m || !n || !x || !delta || l % x) throw Error(B200PIR_E_SHAPE, "setup: l must be a positive multiple of x");
  if (p < 2 || p > 1024) throw Error(B200PIR_E_UNSUPPORTED, "setup: p must be at most 2^10 (squish basis, database.rs:274)");
  use_device(device);
  OwnedStream st;
  const cudaStream_t s = st.s;
  const size_t lx = l / x;
  DevBuf<uint32_t> d_db(l * m), d_a1(m * n), d_a2(lx * n), d_dbsq(l * ((m + 2) / 3)), d_h(l * n);
  DevBuf<uint8_t> a1_img(dpir_gemm_b_bytes(m, n)), a_img(dpir_gemm_a_bytes(l, m));
  B200_CUDA(cudaMemcpyAsync(d_db.p, db, l * m * 4, cudaMemcpyHostToDevice, s));
  B200_CUDA(cudaMemcpyAsync(d_a1.p, a1, m * n * 4, cudaMemcpyHostToDevice, s));
  B200_CUDA(cudaMemcpyAsync(d_a2.p, a2, lx * n * 4, cudaMemcpyHostToDevice, s));
  launch_dpir_gemm_b_image(a1_img.p, d_a1.p, m, n, s);
  dpir_setup_rows(d_db.p, 0, l, m, n, p, a1_img.p, a_img.p, d_h.p, d_dbsq.p, s);        // every row as one band
  dpir_setup_tail(d_h.p, d_a2.p, l, 0, l, n, p, delta, x, h1_squished, a2_t, h2, s);
  B200_CUDA(cudaMemcpyAsync(db_squished, d_dbsq.p, d_dbsq.n * 4, cudaMemcpyDeviceToHost, s));
  B200_CUDA(cudaStreamSynchronize(s));
  B200_CUDA(cudaGetLastError());
  API_END
}
// &Matrix * &Matrix (matrix/ops.rs:169-191) for a left operand with small signed entries (|a| < 2^15): out = a * b mod 2^32
int b200pir_dpir_matmul(int device, const uint32_t* a, uint64_t a_rows, uint64_t a_cols, const uint32_t* b, uint64_t b_cols,
                        uint32_t* out) {
  API_BEGIN
  if (!a || !b || !out || !a_rows || !a_cols || !b_cols) throw Error(B200PIR_E_BADARG, "null or empty argument");
  use_device(device);
  for (size_t i = 0; i < (size_t)a_rows * a_cols; i++)
    if ((int32_t)a[i] < -32768 || (int32_t)a[i] > 32767) throw Error(B200PIR_E_UNSUPPORTED, "matmul: left operand entries must lie in [-2^15, 2^15)");
  OwnedStream st;
  DevBuf<uint32_t> da(a_rows * a_cols), dbm(a_cols * b_cols), dc(a_rows * b_cols);
  B200_CUDA(cudaMemcpyAsync(da.p, a, da.n * 4, cudaMemcpyHostToDevice, st.s));
  B200_CUDA(cudaMemcpyAsync(dbm.p, b, dbm.n * 4, cudaMemcpyHostToDevice, st.s));
  launch_dpir_gemm(dc.p, da.p, dbm.p, a_rows, a_cols, b_cols, st.s);
  B200_CUDA(cudaMemcpyAsync(out, dc.p, dc.n * 4, cudaMemcpyDeviceToHost, st.s));
  B200_CUDA(cudaStreamSynchronize(st.s));
  API_END
}
void b200pir_dpir_destroy(b200pir_dpir* m) {
  if (!m) return;
  cudaSetDevice(m->device);
  cudaDeviceSynchronize();
  if (m->own_stream && m->stream) cudaStreamDestroy(m->stream);
  delete m;
}
int b200pir_dpir_set_stream(b200pir_dpir* m, void* cuda_stream) {
  API_BEGIN
  if (!m) throw Error(B200PIR_E_BADARG, "null handle");
  std::lock_guard<std::mutex> lk(m->mu);
  cudaSetDevice(m->device);
  B200_CUDA(cudaStreamSynchronize(m->stream));                     // pending work on the old stream first
  if (m->own_stream && m->stream) cudaStreamDestroy(m->stream);
  m->stream = (cudaStream_t)cuda_stream;
  m->own_stream = false;
  API_END
}
int b200pir_dpir_matvec_packed_dev(b200pir_dpir* m, const uint32_t* b_dev, uint32_t* out_dev, int /* variant: selects nothing */) {
  API_BEGIN
  if (!m || !b_dev || !out_dev) throw Error(B200PIR_E_BADARG, "null argument");
  std::lock_guard<std::mutex> lk(m->mu);
  cudaSetDevice(m->device);
  launch_dpir_matvec(out_dev, m->a.p, b_dev, m->rows, m->cols, m->stream);
  B200_CUDA(cudaGetLastError());
  API_END
}
// matrix_mul_vec_packed over the row range [row_begin, row_begin + row_count)  (answer(): db.rows(start, batch), doublepir.rs:301)
int b200pir_dpir_matvec_packed_rows(b200pir_dpir* m, uint64_t row_begin, uint64_t row_count, const uint32_t* b, uint32_t* out) {
  API_BEGIN
  if (!m || !b || !out) throw Error(B200PIR_E_BADARG, "null argument");
  if (row_begin > m->rows || row_count > m->rows - row_begin) throw Error(B200PIR_E_SHAPE, "row range out of bounds");
  if (row_count == 0) return 0;
  std::lock_guard<std::mutex> lk(m->mu);
  cudaSetDevice(m->device);
  B200_CUDA(cudaMemcpyAsync(m->b.p, b, 3 * m->cols * 4, cudaMemcpyHostToDevice, m->stream));
  launch_dpir_matvec(m->out.p, m->a.p + row_begin * m->cols, m->b.p, row_count, m->cols, m->stream);
  B200_CUDA(cudaMemcpyAsync(out, m->out.p, row_count * 4, cudaMemcpyDeviceToHost, m->stream));
  B200_CUDA(cudaStreamSynchronize(m->stream));
  B200_CUDA(cudaGetLastError());
  API_END
}
int b200pir_dpir_matrix_mul_transposed_packed(int device, const uint32_t* a, uint64_t a_rows, uint64_t a_cols, const uint32_t* b,
                                              uint64_t b_rows, uint64_t b_cols, uint32_t* out) {
  API_BEGIN
  if (!a || !b || !out) throw Error(B200PIR_E_BADARG, "null argument");
  if (b_cols != 3 * a_cols) throw Error(B200PIR_E_SHAPE, "b.cols must equal 3 * a.cols");
  B200_CUDA(cudaSetDevice(device));
  OwnedStream st;
  DevBuf<uint32_t> da(a_rows * a_cols), db_(b_rows * b_cols), dout(a_rows * b_rows);
  B200_CUDA(cudaMemcpyAsync(da.p, a, da.n * 4, cudaMemcpyHostToDevice, st.s));
  B200_CUDA(cudaMemcpyAsync(db_.p, b, db_.n * 4, cudaMemcpyHostToDevice, st.s));
  launch_dpir_mul_transposed(dout.p, da.p, db_.p, a_rows, a_cols, b_rows, b_cols, st.s);
  B200_CUDA(cudaMemcpyAsync(out, dout.p, dout.n * 4, cudaMemcpyDeviceToHost, st.s));
  B200_CUDA(cudaStreamSynchronize(st.s));
  B200_CUDA(cudaGetLastError());
  API_END
}
int b200pir_dpir_transpose_expand_concat_cols_squish(int device, const uint32_t* a, uint64_t rows, uint64_t cols, uint64_t modulus,
                                                     uint64_t delta, uint64_t concat, uint32_t* out, uint64_t* out_rows,
                                                     uint64_t* out_cols) {
  API_BEGIN
  if (!a || !out) throw Error(B200PIR_E_BADARG, "null argument");
  if (modulus < 2 || modulus > 1024 || delta == 0 || concat == 0) throw Error(B200PIR_E_BADARG, "bad modulus / delta / concat");
  if (rows % concat) throw Error(B200PIR_E_SHAPE, "rows must be a multiple of concat");
  B200_CUDA(cudaSetDevice(device));
  const uint64_t orows = cols * delta * concat, ocols = (rows / concat + 2) / 3;
  OwnedStream st;
  DevBuf<uint32_t> da(rows * cols), dout(orows * ocols);
  B200_CUDA(cudaMemcpyAsync(da.p, a, da.n * 4, cudaMemcpyHostToDevice, st.s));
  launch_dpir_transpose_expand(dout.p, da.p, rows, cols, modulus, delta, concat, orows, ocols, st.s);
  B200_CUDA(cudaMemcpyAsync(out, dout.p, dout.n * 4, cudaMemcpyDeviceToHost, st.s));
  B200_CUDA(cudaStreamSynchronize(st.s));
  if (out_rows) *out_rows = orows;
  if (out_cols) *out_cols = ocols;
  B200_CUDA(cudaGetLastError());
  API_END
}

int b200pir_dpir_matvec_packed(b200pir_dpir* m, const uint32_t* b, uint32_t* out) {
  return b200pir_dpir_matvec_packed_rows(m, 0, m ? m->rows : 0, b, out);
}

// ---------------------------------------------------------------- DoublePIR offline load (dpir_load.cu)
namespace {
const uint8_t kDpirSeedA2[16] = B200PIR_DPIR_SEED_A2;
struct DpirDeleter { void operator()(b200pir_dpir* m) const { b200pir_dpir_destroy(m); } };
}  // namespace

int b200pir_dpir_db_info(const b200pir_dpir_params* params, uint64_t num_entries, uint64_t bits_per_entry, b200pir_dpir_info* out) {
  API_BEGIN
  if (!out) throw Error(B200PIR_E_BADARG, "null argument");
  *out = dpir_info(params, num_entries, bits_per_entry);
  API_END
}

int b200pir_dpir_derive_from_seed(int device, const uint8_t key[16], uint64_t rows, uint64_t cols, uint32_t* out) {
  API_BEGIN
  if (!key || !out) throw Error(B200PIR_E_BADARG, "null argument");
  if (rows && cols > SIZE_MAX / 4 / rows) throw Error(B200PIR_E_SHAPE, "derive: matrix too large");
  if (rows * cols == 0) return 0;
  use_device(device);
  OwnedStream s;
  DevBuf<uint32_t> d(rows * cols);
  launch_dpir_derive(d.p, d.n, dpir_aes_key(key), s.s);
  B200_CUDA(cudaGetLastError());
  B200_CUDA(cudaMemcpyAsync(out, d.p, d.n * 4, cudaMemcpyDeviceToHost, s.s));
  B200_CUDA(cudaStreamSynchronize(s.s));
  API_END
}

namespace {
constexpr uint64_t kDpirDefaultScratch = 1ull << 30;   // device bytes of band scratch when the caller passes 0
constexpr size_t kDpirStagePiece = 16ull << 20;        // bytes of one pinned staging buffer (two of them)

// The input of a load: copies bytes [off, off + n) of the raw entries to dst, or throws
using DpirFill = std::function<void(uint8_t* dst, uint64_t off, size_t n)>;

// One band of layout rows, and the input it reads
struct DpirBandGeom {
  bool bits_format;
  uint64_t l, m, packing, ne, count;   // count: the entries the iterator yields
  // rows in a band come in groups: a base-p entry spans ne rows, so bands are whole groups of ne rows
  uint64_t group() const { return packing ? 1 : ne; }
  // the first entry of layout row r (r a multiple of group()): packed elements r m .., or entries (r / ne) m ..
  uint64_t first_entry(uint64_t r) const { return packing ? r * m * packing : (r / ne) * m; }
  // bytes of the input a band of `rows` rows can span: one more in the bit format, where a band may start mid-byte
  uint64_t raw_bytes(uint64_t rows) const {
    const uint64_t e = packing ? rows * m * packing : (rows / ne) * m;
    return bits_format ? (e + 7) / 8 + 1 : e;
  }
  // device scratch a band of `rows` rows takes: its centred words, its GEMM image and its input bytes
  uint64_t band_bytes(uint64_t rows) const { return 4 * rows * m + dpir_gemm_a_bytes(rows, m) + raw_bytes(rows); }
  // the most rows, a whole number of groups and at least one, whose band fits `budget` bytes of scratch
  uint64_t band_rows(uint64_t budget) const {
    uint64_t lo = 1, hi = l / group();                 // in groups
    if (band_bytes(group()) > budget) return group();
    while (lo < hi) {
      const uint64_t mid = lo + (hi - lo + 1) / 2;
      if (band_bytes(mid * group()) <= budget) lo = mid;
      else hi = mid - 1;
    }
    return lo * group();
  }
};

DpirBandGeom dpir_band_geom(const b200pir_dpir_params* params, const b200pir_dpir_info& info, int entry_format, uint64_t len) {
  if (entry_format != B200PIR_DPIR_ENTRY_BYTES && entry_format != B200PIR_DPIR_ENTRY_BITS)
    throw Error(B200PIR_E_BADARG, "unknown entry format");
  const bool bits_format = entry_format == B200PIR_DPIR_ENTRY_BITS;
  if (bits_format && len > UINT64_MAX / 8) throw Error(B200PIR_E_SHAPE, "too many entries");
  return DpirBandGeom{bits_format, params->l, params->m, info.packing, info.ne, bits_format ? 8 * len : len};
}

// fill(dst, off, n) split over up to 4 threads: a large copy out of host memory or the page cache runs at several times one
// thread's rate
void dpir_fill_parallel(const DpirFill& fill, uint8_t* dst, uint64_t off, size_t n) {
  constexpr size_t kPart = 4ull << 20;
  const size_t parts = std::min<size_t>(4, (n + kPart - 1) / kPart);
  if (parts <= 1) {
    if (n) fill(dst, off, n);
    return;
  }
  const size_t per = (n + parts - 1) / parts;
  std::vector<std::exception_ptr> err(parts);
  std::vector<std::thread> th;
  for (size_t t = 0; t < parts; t++)
    th.emplace_back([&, t] {
      const size_t a = t * per, b = std::min(n, a + per);
      try {
        if (a < b) fill(dst + a, off + a, b - a);
      } catch (...) { err[t] = std::current_exception(); }
    });
  for (auto& t : th) t.join();
  for (auto& e : err)
    if (e) std::rethrow_exception(e);
}

// Two pinned host buffers that take turns: a buffer is refilled once the upload that last read it has run
struct DpirStaging {
  cudaStream_t s;
  uint8_t* buf[2] = {nullptr, nullptr};
  cudaEvent_t done[2] = {nullptr, nullptr};
  size_t cap = 0;
  int next = 0;
  DpirStaging(cudaStream_t st, size_t bytes) : s(st), cap(bytes) {
    for (int i = 0; i < 2; i++) {
      B200_CUDA(cudaMallocHost(&buf[i], std::max<size_t>(cap, 1)));
      B200_CUDA(cudaEventCreateWithFlags(&done[i], cudaEventDisableTiming));
    }
  }
  ~DpirStaging() {
    cudaStreamSynchronize(s);                          // no upload may still read a buffer that is freed
    for (int i = 0; i < 2; i++) {
      if (done[i]) cudaEventDestroy(done[i]);
      if (buf[i]) cudaFreeHost(buf[i]);
    }
  }
  // input bytes [off, off + n) to dst (device) on s
  void upload(const DpirFill& fill, uint8_t* dst, uint64_t off, uint64_t n) {
    for (uint64_t done_bytes = 0; done_bytes < n;) {
      const size_t piece = (size_t)std::min<uint64_t>(cap, n - done_bytes);
      const int i = next;
      next ^= 1;
      B200_CUDA(cudaEventSynchronize(done[i]));
      dpir_fill_parallel(fill, buf[i], off + done_bytes, piece);
      B200_CUDA(cudaMemcpyAsync(dst + done_bytes, buf[i], piece, cudaMemcpyHostToDevice, s));
      B200_CUDA(cudaEventRecord(done[i], s));
      done_bytes += piece;
    }
  }
};

// What every load checks before it touches a device: the DbInfo shape, the entry format, and that the entries fit l x m
struct DpirLoadShape {
  b200pir_dpir_info info;
  DpirBandGeom G;
};
DpirLoadShape dpir_load_shape(const b200pir_dpir_params* params, uint64_t num_entries, uint64_t bits_per_entry, uint64_t len,
                              int entry_format) {
  const b200pir_dpir_info info = dpir_info(params, num_entries, bits_per_entry);
  const DpirBandGeom G = dpir_band_geom(params, info, entry_format, len);
  const uint64_t l = params->l, m = params->m, count = G.count;
  // where load_data would index past the matrix (and panic): the last packed element, or the last digit row of the last entry
  if (info.packing ? (count + info.packing - 1) / info.packing > l * m : (count && ((count - 1) / m + 1) > l / info.ne))
    throw Error(B200PIR_E_SHAPE, "the entries do not fit the l x m database");
  if (l % info.x) throw Error(B200PIR_E_SHAPE, "l must be a multiple of x (concat_cols)");
  return DpirLoadShape{info, G};
}

// DoublePirServer::new + load_data / load_data_fast + setup() (server.rs:160-165, 201-229) for the layout rows [r0, r1) on one
// device, band by band: for each band of rows the band's input bytes are staged and uploaded, laid out, multiplied into the
// range's rows of h_1 and squished into the resident store; setup()'s tail then runs on the range's h_1 (dpir_setup_tail: its
// columns of h1_squished, its partial of h2, and a2_t unless null).  The band scratch is allocated once, sized by scratch_bytes.
// The whole database is the range [0, l); a shard's range has r0 a multiple of 3x (dpir_shard_rows).
b200pir_dpir* dpir_load_range(int device, const b200pir_dpir_params* params, const DpirLoadShape& S, uint64_t num_entries,
                              uint64_t bits_per_entry, int entry_format, uint64_t scratch_bytes, const DpirFill& fill, uint64_t r0,
                              uint64_t r1, uint32_t* h1_squished, uint32_t* a2_t, uint32_t* h2) {
  const b200pir_dpir_info& info = S.info;
  const DpirBandGeom& G = S.G;
  const uint64_t l = params->l, m = params->m, n = params->n, x = info.x, count = G.count, rows_g = r1 - r0;
  const uint32_t p = (uint32_t)params->p;
  std::unique_ptr<b200pir_dpir, DpirDeleter> h(dpir_new(device, rows_g, (m + 2) / 3));
  h->row_begin = r0;
  cudaStream_t s = h->stream;
  const uint64_t band = std::min(G.band_rows(scratch_bytes ? scratch_bytes : kDpirDefaultScratch), rows_g);
  DevBuf<uint32_t> d_h(rows_g * n), d_a2((l / x) * n);
  {
    DevBuf<uint8_t> a1_img(dpir_gemm_b_bytes(m, n));
    {
      DevBuf<uint32_t> d_a1(m * n);
      launch_dpir_derive(d_a1.p, d_a1.n, dpir_aes_key(kDpirSeedA1), s);           // init(): A_1 = derive(m x n, SEEDS_SHORT[0])
      launch_dpir_gemm_b_image(a1_img.p, d_a1.p, m, n, s);                        // a_1 is only read through its GEMM image
      B200_CUDA(cudaStreamSynchronize(s));
    }
    launch_dpir_derive(d_a2.p, d_a2.n, dpir_aes_key(kDpirSeedA2), s);              //         A_2 = derive(l/x x n, SEEDS_SHORT[1])
    DevBuf<uint32_t> d_band(band * m);
    DevBuf<uint8_t> a_img(dpir_gemm_a_bytes(band, m)), d_raw(G.raw_bytes(band));
    DevBuf<int> d_flag(1);
    B200_CUDA(cudaMemsetAsync(d_flag.p, 0, sizeof(int), s));
    DpirStaging stage(s, (size_t)std::min<uint64_t>(kDpirStagePiece, G.raw_bytes(band)));
    for (uint64_t b = r0; b < r1; b += band) {
      const uint64_t rows = std::min(band, r1 - b);
      // the band's entries [e0, e1) are bytes [b0, b1) of the input (bits: the band may start and end mid-byte)
      const uint64_t e0 = std::min(G.first_entry(b), count), e1 = std::min(G.first_entry(b + rows), count);
      const uint64_t b0 = G.bits_format ? e0 / 8 : e0, b1 = G.bits_format ? (e1 + 7) / 8 : e1;
      stage.upload(fill, d_raw.p, b0, b1 - b0);
      launch_dpir_layout(d_band.p, d_raw.p, G.bits_format ? 8 * b0 : b0, count, G.bits_format, b, rows, m, (uint32_t)info.packing,
                         (uint32_t)bits_per_entry, (uint32_t)info.ne, p, d_flag.p, s);
      dpir_setup_rows(d_band.p, b - r0, rows, m, n, p, a1_img.p, a_img.p, d_h.p, h->a.p, s);
    }
    B200_CUDA(cudaGetLastError());
    int flag = 0;
    B200_CUDA(cudaMemcpyAsync(&flag, d_flag.p, sizeof(int), cudaMemcpyDeviceToHost, s));
    B200_CUDA(cudaStreamSynchronize(s));
    if (flag & 1) throw Error(B200PIR_E_UNSUPPORTED, "load: a packed database word lies outside [-2^15, 2^15) (entries far wider than bits_per_entry)");
    h->fields_exact = !(flag & 2);
  }
  dpir_setup_tail(d_h.p, d_a2.p, l, r0, rows_g, n, p, info.delta, x, h1_squished, a2_t, h2, s);
  h->from_load = true;
  h->entry_format = entry_format;
  h->load_count = count;
  h->num_entries = num_entries;
  h->bits_per_entry = bits_per_entry;
  h->params = *params;
  return h.release();
}

b200pir_dpir* dpir_load_bands(int device, const b200pir_dpir_params* params, uint64_t num_entries, uint64_t bits_per_entry,
                              uint64_t len, int entry_format, uint64_t scratch_bytes, const DpirFill& fill, uint32_t* h1_squished,
                              uint32_t* a2_t, uint32_t* h2) {
  const DpirLoadShape S = dpir_load_shape(params, num_entries, bits_per_entry, len, entry_format);
  return dpir_load_range(device, params, S, num_entries, bits_per_entry, entry_format, scratch_bytes, fill, 0, params->l,
                         h1_squished, a2_t, h2);
}

// The load over `shards` row shards (dpir_shard_rows), shard g on devices[g]: one host thread a distinct device, each loading
// its shards one after another, so distinct devices read their byte ranges and load at once.  Every range writes its own columns
// of h1_squished; shard 0 writes a2_t; h2 is the sum of the ranges' partials mod 2^32.  On any error every handle is destroyed.
void dpir_load_sharded(const int* devices, size_t shards, const b200pir_dpir_params* params, uint64_t num_entries,
                       uint64_t bits_per_entry, uint64_t len, int entry_format, uint64_t scratch_bytes, const DpirFill& fill,
                       b200pir_dpir** dbs_out, uint32_t* h1_squished, uint32_t* a2_t, uint32_t* h2) {
  const DpirLoadShape S = dpir_load_shape(params, num_entries, bits_per_entry, len, entry_format);
  if (shards == 0) throw Error(B200PIR_E_SHAPE, "no shards");
  std::vector<DpirShardRows> R(shards);
  for (size_t g = 0; g < shards; g++) R[g] = dpir_shard_rows(params->l, S.info.x, shards, g);
  for (size_t g = 0; g < shards; g++) use_device(devices[g]);
  const size_t h2_words = (size_t)params->n * S.info.delta * S.info.x * params->n;
  std::vector<std::vector<uint32_t>> part(shards, std::vector<uint32_t>(h2_words));
  std::vector<std::unique_ptr<b200pir_dpir, DpirDeleter>> out(shards);
  std::vector<std::exception_ptr> err(shards);
  std::vector<int> distinct;
  for (size_t g = 0; g < shards; g++)
    if (std::find(distinct.begin(), distinct.end(), devices[g]) == distinct.end()) distinct.push_back(devices[g]);
  // g_kernel_launches is per thread: each worker reports what it launched, and the caller's count takes it in after the join
  std::vector<unsigned long long> launched(distinct.size(), 0);
  std::vector<std::thread> th;
  for (size_t t = 0; t < distinct.size(); t++)
    th.emplace_back([&, t] {
      const int dev = distinct[t];
      const unsigned long long k0 = g_kernel_launches;
      for (size_t g = 0; g < shards; g++) {
        if (devices[g] != dev) continue;
        try {
          out[g].reset(dpir_load_range(dev, params, S, num_entries, bits_per_entry, entry_format, scratch_bytes, fill, R[g].begin,
                                       R[g].begin + R[g].rows, h1_squished, g == 0 ? a2_t : nullptr, part[g].data()));
        } catch (...) {
          err[g] = std::current_exception();
          break;                                         // this device's later shards are not loaded: the call fails anyway
        }
      }
      launched[t] = g_kernel_launches - k0;
    });
  for (auto& t : th) t.join();
  for (unsigned long long k : launched) g_kernel_launches += k;
  for (auto& e : err)
    if (e) std::rethrow_exception(e);                    // `out` destroys every handle that was made
  for (size_t i = 0; i < h2_words; i++) {
    uint32_t v = 0;
    for (size_t g = 0; g < shards; g++) v += part[g][i];
    h2[i] = v;
  }
  for (size_t g = 0; g < shards; g++) dbs_out[g] = out[g].release();
}

// pread of bytes [off, off + n) of an open file, as the file loads read it
DpirFill dpir_file_fill(int fd) {
  return [fd](uint8_t* dst, uint64_t off, size_t n) {
    while (n) {
      const ssize_t r = pread(fd, dst, n, (off_t)off);
      if (r < 0 && errno == EINTR) continue;
      if (r <= 0) throw Error(B200PIR_E_SHAPE, "short read from the database file");
      dst += r; off += (uint64_t)r; n -= (size_t)r;
    }
  };
}

// The database file at `path`, open, with its size
struct DpirFile {
  int fd = -1;
  uint64_t size = 0;
  explicit DpirFile(const char* path) {
    fd = open(path, O_RDONLY | O_CLOEXEC);
    if (fd < 0) throw Error(B200PIR_E_BADARG, std::string("cannot open ") + path);
    struct stat st;
    if (fstat(fd, &st)) throw Error(B200PIR_E_BADARG, std::string("cannot stat ") + path);
    // the entry count comes from the file size, as load_data_fast's takes it from the bytes it is given; a directory or a
    // device has no such size, and reading it fails
    if (!S_ISREG(st.st_mode)) throw Error(B200PIR_E_SHAPE, "short read from the database file (not a regular file)");
    size = (uint64_t)st.st_size;
  }
  ~DpirFile() { if (fd >= 0) close(fd); }
  DpirFile(const DpirFile&) = delete;
  DpirFile& operator=(const DpirFile&) = delete;
};

DpirFill dpir_memory_fill(const uint8_t* data) {
  return [data](uint8_t* dst, uint64_t off, size_t n) { std::memcpy(dst, data + off, n); };
}
}  // namespace

int b200pir_dpir_load(int device, const b200pir_dpir_params* params, uint64_t num_entries, uint64_t bits_per_entry,
                      const uint8_t* data, uint64_t len, int entry_format, b200pir_dpir** db_out, uint32_t* h1_squished,
                      uint32_t* a2_t, uint32_t* h2) {
  return b200pir_dpir_load_banded(device, params, num_entries, bits_per_entry, data, len, entry_format, 0, db_out, h1_squished,
                                  a2_t, h2);
}

int b200pir_dpir_load_banded(int device, const b200pir_dpir_params* params, uint64_t num_entries, uint64_t bits_per_entry,
                             const uint8_t* data, uint64_t len, int entry_format, uint64_t scratch_bytes, b200pir_dpir** db_out,
                             uint32_t* h1_squished, uint32_t* a2_t, uint32_t* h2) {
  API_BEGIN
  if (!params || !data || !db_out || !h1_squished || !a2_t || !h2) throw Error(B200PIR_E_BADARG, "null argument");
  *db_out = dpir_load_bands(device, params, num_entries, bits_per_entry, len, entry_format, scratch_bytes, dpir_memory_fill(data),
                            h1_squished, a2_t, h2);
  API_END
}

int b200pir_dpir_load_file(int device, const b200pir_dpir_params* params, uint64_t num_entries, uint64_t bits_per_entry,
                           const char* path, int entry_format, uint64_t scratch_bytes, b200pir_dpir** db_out, uint32_t* h1_squished,
                           uint32_t* a2_t, uint32_t* h2) {
  API_BEGIN
  if (!params || !path || !db_out || !h1_squished || !a2_t || !h2) throw Error(B200PIR_E_BADARG, "null argument");
  DpirFile file(path);
  *db_out = dpir_load_bands(device, params, num_entries, bits_per_entry, file.size, entry_format, scratch_bytes,
                            dpir_file_fill(file.fd), h1_squished, a2_t, h2);
  API_END
}

int b200pir_dpir_shard_rows(const b200pir_dpir_params* params, uint64_t num_entries, uint64_t bits_per_entry, size_t shards,
                            size_t index, uint64_t* row_begin, uint64_t* rows) {
  API_BEGIN
  if (!row_begin || !rows) throw Error(B200PIR_E_BADARG, "null argument");
  const b200pir_dpir_info info = dpir_info(params, num_entries, bits_per_entry, 64);
  if (params->l % info.x) throw Error(B200PIR_E_SHAPE, "l must be a multiple of x (concat_cols)");
  if (shards && index >= shards) throw Error(B200PIR_E_BADARG, "shard index >= the shard count");
  const DpirShardRows r = dpir_shard_rows(params->l, info.x, shards, index);
  *row_begin = r.begin;
  *rows = r.rows;
  API_END
}

int b200pir_dpir_load_sharded(const int* devices, size_t shards, const b200pir_dpir_params* params, uint64_t num_entries,
                              uint64_t bits_per_entry, const uint8_t* data, uint64_t len, int entry_format, uint64_t scratch_bytes,
                              b200pir_dpir** dbs_out, uint32_t* h1_squished, uint32_t* a2_t, uint32_t* h2) {
  API_BEGIN
  if (!devices || !params || !data || !dbs_out || !h1_squished || !a2_t || !h2) throw Error(B200PIR_E_BADARG, "null argument");
  dpir_load_sharded(devices, shards, params, num_entries, bits_per_entry, len, entry_format, scratch_bytes, dpir_memory_fill(data),
                    dbs_out, h1_squished, a2_t, h2);
  API_END
}

int b200pir_dpir_load_file_sharded(const int* devices, size_t shards, const b200pir_dpir_params* params, uint64_t num_entries,
                                   uint64_t bits_per_entry, const char* path, int entry_format, uint64_t scratch_bytes,
                                   b200pir_dpir** dbs_out, uint32_t* h1_squished, uint32_t* a2_t, uint32_t* h2) {
  API_BEGIN
  if (!devices || !params || !path || !dbs_out || !h1_squished || !a2_t || !h2) throw Error(B200PIR_E_BADARG, "null argument");
  DpirFile file(path);
  dpir_load_sharded(devices, shards, params, num_entries, bits_per_entry, file.size, entry_format, scratch_bytes,
                    dpir_file_fill(file.fd), dbs_out, h1_squished, a2_t, h2);
  API_END
}

int b200pir_dpir_create_shard(int device, const uint32_t* a, uint64_t row_begin, uint64_t rows, uint64_t cols, b200pir_dpir** out) {
  API_BEGIN
  if (!out) throw Error(B200PIR_E_BADARG, "null argument");
  b200pir_dpir* m = nullptr;
  if (int rc = b200pir_dpir_create(device, a, rows, cols, &m)) return rc;
  m->row_begin = row_begin;
  *out = m;
  API_END
}

int b200pir_dpir_shard_info(b200pir_dpir* m, uint64_t* row_begin, uint64_t* rows, uint64_t* cols, int* device) {
  API_BEGIN
  if (!m || !row_begin || !rows || !cols || !device) throw Error(B200PIR_E_BADARG, "null argument");
  *row_begin = m->row_begin;
  *rows = m->rows;
  *cols = m->cols;
  *device = m->device;
  API_END
}

int b200pir_dpir_band_bytes(const b200pir_dpir_params* params, uint64_t num_entries, uint64_t bits_per_entry, int entry_format,
                            uint64_t rows, uint64_t* out) {
  API_BEGIN
  if (!out) throw Error(B200PIR_E_BADARG, "null argument");
  const b200pir_dpir_info info = dpir_info(params, num_entries, bits_per_entry);
  const DpirBandGeom G = dpir_band_geom(params, info, entry_format, 0);
  if (rows == 0 || rows > G.l || rows % G.group()) throw Error(B200PIR_E_SHAPE, "rows must be a whole number of groups of at most l");
  *out = G.band_bytes(rows);
  API_END
}

int b200pir_dpir_download(b200pir_dpir* m, uint32_t* out) {
  API_BEGIN
  if (!m || !out) throw Error(B200PIR_E_BADARG, "null argument");
  std::lock_guard<std::mutex> lk(m->mu);
  cudaSetDevice(m->device);
  B200_CUDA(cudaMemcpyAsync(out, m->a.p, m->rows * m->cols * 4, cudaMemcpyDeviceToHost, m->stream));
  B200_CUDA(cudaStreamSynchronize(m->stream));
  B200_CUDA(cudaGetLastError());
  API_END
}

// matrix_mul_vec_packed for `count` vectors, one pass over the matrix per 64 (tensor cores) or 16 (k_dpir_matvec_multi) of them
// (host buffers; the multi-vector kernels' test face).  kernel: B200PIR_DPIR_MV_AUTO picks as the answer path does.
int b200pir_dpir_matvec_packed_many_on(b200pir_dpir* m, const uint32_t* b, size_t count, uint32_t* out, int kernel) {
  API_BEGIN
  if (!m || !b || !out) throw Error(B200PIR_E_BADARG, "null argument");
  if (kernel != B200PIR_DPIR_MV_AUTO && kernel != B200PIR_DPIR_MV_MULTI && kernel != B200PIR_DPIR_MV_TC)
    throw Error(B200PIR_E_BADARG, "unknown matvec kernel");
  if (count == 0) return 0;
  if (m->rows > 0xFFFFFFFFull || count > 0xFFFFFFFFull) throw Error(B200PIR_E_SHAPE, "too many rows or vectors");
  std::lock_guard<std::mutex> lk(m->mu);
  cudaSetDevice(m->device);
  int sms = 0;
  B200_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, m->device));
  const bool tc = kernel == B200PIR_DPIR_MV_TC || (kernel == B200PIR_DPIR_MV_AUTO && dpir_use_tc(count, m->rows));
  const size_t img = dtc_img_bytes(m->cols);
  DevBuf<uint32_t> d_b(count * 3 * m->cols), d_out(count * m->rows);
  DevBuf<uint8_t> d_img(tc ? count * img : 0);
  DpirMvPlan plan;
  for (size_t v = 0; v < count; v++) {
    const uint32_t* bv = d_b.p + v * 3 * m->cols;
    plan.vecs.push_back(DpirMvVec{tc ? plan.image(bv, d_img.p + v * img, m->cols) : bv, d_out.p + v * m->rows});
  }
  DpirMvPass pass = plan.pass(tc, m->cols);
  plan.add(pass, m->a.p, m->rows, count);
  std::vector<uint8_t> h_tab(plan.bytes());
  DevBuf<uint8_t> d_tab(h_tab.size());
  plan.place(h_tab.data(), d_tab.p);
  B200_CUDA(cudaMemcpyAsync(d_tab.p, h_tab.data(), h_tab.size(), cudaMemcpyHostToDevice, m->stream));
  B200_CUDA(cudaMemcpyAsync(d_b.p, b, d_b.n * 4, cudaMemcpyHostToDevice, m->stream));
  B200_CUDA(cudaMemsetAsync(d_out.p, 0, d_out.n * 4, m->stream));
  launch_dpir_tc_image(plan.d_jobs, plan.jobs.size(), m->cols, 0, m->stream);
  plan.launch(pass, true, sms, 0, m->stream);
  B200_CUDA(cudaGetLastError());
  B200_CUDA(cudaMemcpyAsync(out, d_out.p, d_out.n * 4, cudaMemcpyDeviceToHost, m->stream));
  B200_CUDA(cudaStreamSynchronize(m->stream));
  B200_CUDA(cudaGetLastError());
  API_END
}

int b200pir_dpir_matvec_packed_many(b200pir_dpir* m, const uint32_t* b, size_t count, uint32_t* out) {
  return b200pir_dpir_matvec_packed_many_on(m, b, count, out, B200PIR_DPIR_MV_AUTO);
}

}  // extern "C"
