// C-ABI implementation of DoublePIR (include/b200pir.h): the resident matrix handle, setup(), the banded offline load and the
// answer() server, as host-side orchestration of the dpir_*.cu kernels.
#include "api_internal.hpp"
#include "dpir_wire.hpp"
#include <cerrno>
#include <fcntl.h>
#include <sys/stat.h>
#include <unistd.h>
#include <algorithm>
#include <array>
#include <cmath>
#include <cstring>
#include <functional>
#include <memory>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

using namespace b200pir;

struct b200pir_dpir {
  int device;
  std::mutex mu;            // calls on one handle stage through its b / out buffers: serialised
  cudaStream_t stream = nullptr;
  bool own_stream = true;
  uint64_t rows, cols;
  DevBuf<uint32_t> a;
  DevBuf<uint32_t> b, out;
  // what b200pir_dpir_load* laid out in `a`, for b200pir_dpir_server_update; from_load stays false for b200pir_dpir_create*
  bool from_load = false;
  int entry_format = 0;
  uint64_t load_count = 0;               // entries the load iterated: len bytes, or 8 len bits
  uint64_t num_entries = 0, bits_per_entry = 0;
  b200pir_dpir_params params{};
  bool fields_exact = false;             // no packed entry was wider than bits_per_entry: every element decodes field by field
};

extern "C" {

namespace {
// A non-blocking stream owned by one scope: destroyed when the scope is left, unless release()d to a longer-lived owner
struct OwnedStream {
  cudaStream_t s = nullptr;
  OwnedStream() { B200_CUDA(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking)); }
  ~OwnedStream() { if (s) cudaStreamDestroy(s); }
  cudaStream_t release() { cudaStream_t r = s; s = nullptr; return r; }
  OwnedStream(const OwnedStream&) = delete;
  OwnedStream& operator=(const OwnedStream&) = delete;
};

__global__ void k_dpir_synth(uint32_t* a, size_t words, uint64_t seed, size_t index0) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= words) return;
  a[i] = (uint32_t)splitmix64_at(seed, index0 + i) & 0x3FFFFFFFu;
}
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
  size_t words = rows * cols;
  const size_t chunk = (size_t)1 << 30;
  for (size_t off = 0; off < words; off += chunk) {
    size_t cur = std::min(chunk, words - off);
    k_dpir_synth<<<(unsigned)((cur + 255) / 256), 256, 0, m->stream>>>(m->a.p + off, cur, seed, off);
  }
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
// The tail, on the whole h_1 (l x n, device) and a2 (l/x x n, device): transpose / expand / concat, h_2 = h_1 * a_2, h_1 += p/2
// and squish, a_2_copy.  h1_squished, a2_t and h2 are host buffers.  Synchronises s.
void dpir_setup_tail(const uint32_t* d_h, const uint32_t* d_a2, uint64_t l, uint64_t n, uint32_t p, uint64_t delta, uint64_t x,
                     uint32_t* h1_squished, uint32_t* a2_t, uint32_t* h2, cudaStream_t s) {
  const size_t lx = l / x, rows1 = n * delta * x, lx3 = lx + (3 - lx % 3) % 3;
  DevBuf<uint32_t> d_hc(rows1 * lx), d_h2(rows1 * n);
  DevBuf<uint32_t> d_h1sq(rows1 * ((lx + 2) / 3)), d_a2t(n * lx3);
  launch_dpir_transpose_expand_concat(d_hc.p, d_h, l, n, p, (int)delta, x, s);          // transpose, expand, concat_cols
  launch_dpir_gemm(d_h2.p, d_hc.p, d_a2, rows1, lx, n, s);                               // h_2 = h_1 * a_2
  launch_dpir_add_squish(d_h1sq.p, d_hc.p, rows1, lx, p / 2, s);                         // h_1 += p/2; squish
  launch_dpir_pad_transpose(d_a2t.p, d_a2, lx, n, lx3, s);                               // a_2_copy
  B200_CUDA(cudaMemcpyAsync(h1_squished, d_h1sq.p, d_h1sq.n * 4, cudaMemcpyDeviceToHost, s));
  B200_CUDA(cudaMemcpyAsync(a2_t, d_a2t.p, d_a2t.n * 4, cudaMemcpyDeviceToHost, s));
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
  dpir_setup_tail(d_h.p, d_a2.p, l, n, p, delta, x, h1_squished, a2_t, h2, s);
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
  DevBuf<uint32_t> da(a_rows * a_cols), dbm(a_cols * b_cols), dc(a_rows * b_cols);
  B200_CUDA(cudaMemcpy(da.p, a, da.n * 4, cudaMemcpyHostToDevice));
  B200_CUDA(cudaMemcpy(dbm.p, b, dbm.n * 4, cudaMemcpyHostToDevice));
  launch_dpir_gemm(dc.p, da.p, dbm.p, a_rows, a_cols, b_cols, nullptr);
  B200_CUDA(cudaMemcpy(out, dc.p, dc.n * 4, cudaMemcpyDeviceToHost));
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
  DevBuf<uint32_t> da(a_rows * a_cols), db_(b_rows * b_cols), dout(a_rows * b_rows);
  B200_CUDA(cudaMemcpy(da.p, a, da.n * 4, cudaMemcpyHostToDevice));
  B200_CUDA(cudaMemcpy(db_.p, b, db_.n * 4, cudaMemcpyHostToDevice));
  launch_dpir_mul_transposed(dout.p, da.p, db_.p, a_rows, a_cols, b_rows, b_cols, 0);
  B200_CUDA(cudaMemcpy(out, dout.p, dout.n * 4, cudaMemcpyDeviceToHost));
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
  DevBuf<uint32_t> da(rows * cols), dout(orows * ocols);
  B200_CUDA(cudaMemcpy(da.p, a, da.n * 4, cudaMemcpyHostToDevice));
  launch_dpir_transpose_expand(dout.p, da.p, rows, cols, modulus, delta, concat, orows, ocols, 0);
  B200_CUDA(cudaMemcpy(out, dout.p, dout.n * 4, cudaMemcpyDeviceToHost));
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
const uint8_t kDpirSeedA1[16] = B200PIR_DPIR_SEED_A1;
const uint8_t kDpirSeedA2[16] = B200PIR_DPIR_SEED_A2;

// DbInfo::new (database.rs:58-90) with num_db_entries (:352-372) and compute_num_entries_base_p (:345-350); Params::delta().
// db_elems is num_db_entries' first value.  max_bits: 63 where entries are laid out; the server, which only needs the shape,
// takes full 64-bit entries too.
b200pir_dpir_info dpir_info(const b200pir_dpir_params* prm, uint64_t num_entries, uint64_t bits, uint64_t* db_elems,
                            uint64_t max_bits = 63) {
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
  if (db_elems) *db_elems = elems;
  return o;
}
struct DpirDeleter { void operator()(b200pir_dpir* m) const { b200pir_dpir_destroy(m); } };
}  // namespace

int b200pir_dpir_db_info(const b200pir_dpir_params* params, uint64_t num_entries, uint64_t bits_per_entry, b200pir_dpir_info* out) {
  API_BEGIN
  if (!out) throw Error(B200PIR_E_BADARG, "null argument");
  *out = dpir_info(params, num_entries, bits_per_entry, nullptr);
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

// DoublePirServer::new + load_data / load_data_fast + setup() (server.rs:160-165, 201-229), band by band: for each band of
// layout rows the band's input bytes are staged and uploaded, laid out, multiplied into h_1's rows and squished into the
// resident store; setup()'s tail then runs on the whole h_1.  The band scratch is allocated once, sized by scratch_bytes.
b200pir_dpir* dpir_load_bands(int device, const b200pir_dpir_params* params, uint64_t num_entries, uint64_t bits_per_entry,
                              uint64_t len, int entry_format, uint64_t scratch_bytes, const DpirFill& fill, uint32_t* h1_squished,
                              uint32_t* a2_t, uint32_t* h2) {
  const b200pir_dpir_info info = dpir_info(params, num_entries, bits_per_entry, nullptr);
  const DpirBandGeom G = dpir_band_geom(params, info, entry_format, len);
  const uint64_t l = params->l, m = params->m, n = params->n, x = info.x, count = G.count;
  const uint32_t p = (uint32_t)params->p;
  // where load_data would index past the matrix (and panic): the last packed element, or the last digit row of the last entry
  if (info.packing ? (count + info.packing - 1) / info.packing > l * m : (count && ((count - 1) / m + 1) > l / info.ne))
    throw Error(B200PIR_E_SHAPE, "the entries do not fit the l x m database");
  if (l % x) throw Error(B200PIR_E_SHAPE, "l must be a multiple of x (concat_cols)");
  std::unique_ptr<b200pir_dpir, DpirDeleter> h(dpir_new(device, l, (m + 2) / 3));
  cudaStream_t s = h->stream;
  const uint64_t band = G.band_rows(scratch_bytes ? scratch_bytes : kDpirDefaultScratch);
  DevBuf<uint32_t> d_h(l * n), d_a2((l / x) * n);
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
    for (uint64_t r0 = 0; r0 < l; r0 += band) {
      const uint64_t rows = std::min(band, l - r0);
      // the band's entries [e0, e1) are bytes [b0, b1) of the input (bits: the band may start and end mid-byte)
      const uint64_t e0 = std::min(G.first_entry(r0), count), e1 = std::min(G.first_entry(r0 + rows), count);
      const uint64_t b0 = G.bits_format ? e0 / 8 : e0, b1 = G.bits_format ? (e1 + 7) / 8 : e1;
      stage.upload(fill, d_raw.p, b0, b1 - b0);
      launch_dpir_layout(d_band.p, d_raw.p, G.bits_format ? 8 * b0 : b0, count, G.bits_format, r0, rows, m, (uint32_t)info.packing,
                         (uint32_t)bits_per_entry, (uint32_t)info.ne, p, d_flag.p, s);
      dpir_setup_rows(d_band.p, r0, rows, m, n, p, a1_img.p, a_img.p, d_h.p, h->a.p, s);
    }
    B200_CUDA(cudaGetLastError());
    int flag = 0;
    B200_CUDA(cudaMemcpyAsync(&flag, d_flag.p, sizeof(int), cudaMemcpyDeviceToHost, s));
    B200_CUDA(cudaStreamSynchronize(s));
    if (flag & 1) throw Error(B200PIR_E_UNSUPPORTED, "load: a packed database word lies outside [-2^15, 2^15) (entries far wider than bits_per_entry)");
    h->fields_exact = !(flag & 2);
  }
  dpir_setup_tail(d_h.p, d_a2.p, l, n, p, info.delta, x, h1_squished, a2_t, h2, s);
  h->from_load = true;
  h->entry_format = entry_format;
  h->load_count = count;
  h->num_entries = num_entries;
  h->bits_per_entry = bits_per_entry;
  h->params = *params;
  return h.release();
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
  *db_out = dpir_load_bands(device, params, num_entries, bits_per_entry, len, entry_format, scratch_bytes,
                            [data](uint8_t* dst, uint64_t off, size_t n) { std::memcpy(dst, data + off, n); }, h1_squished, a2_t, h2);
  API_END
}

int b200pir_dpir_load_file(int device, const b200pir_dpir_params* params, uint64_t num_entries, uint64_t bits_per_entry,
                           const char* path, int entry_format, uint64_t scratch_bytes, b200pir_dpir** db_out, uint32_t* h1_squished,
                           uint32_t* a2_t, uint32_t* h2) {
  API_BEGIN
  if (!params || !path || !db_out || !h1_squished || !a2_t || !h2) throw Error(B200PIR_E_BADARG, "null argument");
  struct Closer { int fd; ~Closer() { if (fd >= 0) close(fd); } } file{open(path, O_RDONLY | O_CLOEXEC)};
  if (file.fd < 0) throw Error(B200PIR_E_BADARG, std::string("cannot open ") + path);
  struct stat st;
  if (fstat(file.fd, &st)) throw Error(B200PIR_E_BADARG, std::string("cannot stat ") + path);
  // the entry count comes from the file size, as load_data_fast's takes it from the bytes it is given; a directory or a
  // device has no such size, and reading it fails
  if (!S_ISREG(st.st_mode)) throw Error(B200PIR_E_SHAPE, "short read from the database file (not a regular file)");
  const int fd = file.fd;
  *db_out = dpir_load_bands(device, params, num_entries, bits_per_entry, (uint64_t)st.st_size, entry_format, scratch_bytes,
                            [fd](uint8_t* dst, uint64_t off, size_t n) {
                              while (n) {
                                const ssize_t r = pread(fd, dst, n, (off_t)off);
                                if (r < 0 && errno == EINTR) continue;
                                if (r <= 0) throw Error(B200PIR_E_SHAPE, "short read from the database file");
                                dst += r; off += (uint64_t)r; n -= (size_t)r;
                              }
                            },
                            h1_squished, a2_t, h2);
  API_END
}

int b200pir_dpir_band_bytes(const b200pir_dpir_params* params, uint64_t num_entries, uint64_t bits_per_entry, int entry_format,
                            uint64_t rows, uint64_t* out) {
  API_BEGIN
  if (!out) throw Error(B200PIR_E_BADARG, "null argument");
  const b200pir_dpir_info info = dpir_info(params, num_entries, bits_per_entry, nullptr);
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

// ---------------------------------------------------------------- DoublePIR online: answer() from HBM (dpir_serve.cu)
struct b200pir_dpir_server {
  int device = 0, sm_count = 0;
  std::mutex mu;                 // calls stage through one workspace: serialised
  cudaStream_t stream = nullptr;
  b200pir_dpir* db = nullptr;    // borrowed
  uint64_t n = 0, l = 0, p = 0, delta = 0, x = 0, e = 0;       // e = ne / x: q_2 vectors a query
  uint64_t dx = 0, rows1 = 0, c1 = 0, lx3 = 0, dcols = 0;      // delta x; n delta x; packed cols of h_1 and a_1'; 3 c1; db cols
  size_t max_queries = 0;
  DevBuf<uint32_t> h1, a2t;      // server_state, resident
  // workspace for max_queries queries (and as many requests): staged vectors + task tables (one upload), a_1 / a_1' / msg[0]
  // per request, the responses in wire layout (one download)
  size_t stage_cap = 0, resp_cap = 0, task_cap = 0, vec_cap = 0;
  uint8_t* h_stage = nullptr;
  uint8_t* h_resp = nullptr;
  DevBuf<uint8_t> d_stage, d_resp;
  DevBuf<uint32_t> d_a1, d_a1sq, d_msg0;
  DevBuf<uint8_t> d_img;         // query images of the passes that run on the tensor cores (every q_1, then every q_2)
  size_t img_q1 = 0, img_q2 = 0; // bytes of one q_1 / q_2 image
  b200pir_dpir_params params{};  // as created, with num_entries and bits_per_entry: an update checks them against the load
  uint64_t num_entries = 0, bits_per_entry = 0;
  // update scratch, allocated by the first update and grown only for a larger one: per group of at most upd_cap elements
  // (and as many rows), plus the tables of the whole batch and the hint
  size_t upd_cap = 0, upd_tab = 0;
  DevBuf<DpirUpdElem> u_el;
  DevBuf<DpirUpdRow> u_rows;
  DevBuf<int32_t> u_delta, u_D;
  DevBuf<uint32_t> u_dh1, u_a2g, u_dh2, u_h2;
  DevBuf<uint8_t> u_aimg, u_bimg;
  DpirAesKey a1_key;             // SEED_A1's tables, expanded by the first update
  bool have_a1_key = false;
  ~b200pir_dpir_server() {
    if (h_stage) cudaFreeHost(h_stage);
    if (h_resp) cudaFreeHost(h_resp);
  }
};

namespace {
size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }
uint64_t ceil_div(uint64_t a, uint64_t b) { return (a + b - 1) / b; }

struct DpirCall {               // one request of a call
  const uint8_t* req;
  DpirWireRequest w;
  DpirResponseLayout L;
  size_t resp_off = 0;          // byte offset of its response in d_resp
  std::vector<const uint32_t*> q1, q2;   // device addresses of its staged vectors ([k], [k * e + j]); q1[k] null when not read
  std::vector<const uint32_t*> q1i, q2i; // the same vectors' query images, for passes on the tensor cores
};

// The tasks of one pass of vectors [vec0, vec0 + nv) over the `rows` x `cols` packed matrix `a`: one a tile of rows each,
// DTC_ROWS on the tensor cores (tc), kDpirMvRows on k_dpir_matvec_multi
void add_tiles(std::vector<DpirMvTask>& tasks, const uint32_t* a, uint64_t rows, uint64_t cols, uint32_t vec0, uint32_t nv, bool tc) {
  const uint64_t tr = tc ? DTC_ROWS : kDpirMvRows;
  for (uint64_t t0 = 0; t0 < rows; t0 += tr)
    tasks.push_back(DpirMvTask{a + t0 * cols, (uint32_t)std::min<uint64_t>(tr, rows - t0), vec0, nv, (uint32_t)t0});
}

// The `ntasks` device tasks on the tensor cores (tc; the vectors are query images) or on k_dpir_matvec_multi (vmax: the most
// vectors a task holds), k split over the SMs when `split` is set (only a pass that adds into zeroed outputs may split k)
void launch_matvec_pass(bool tc, const DpirMvTask* tasks, size_t ntasks, const DpirMvVec* vecs, uint64_t cols, int vmax, bool split,
                        int sm_count, int flags, cudaStream_t s) {
  if (tc) launch_dpir_matvec_tc(tasks, ntasks, vecs, cols, split ? dpir_tc_ksplit(ntasks, cols, sm_count) : 1, flags, s);
  else launch_dpir_matvec_multi(tasks, ntasks, vecs, cols, vmax, split ? dpir_mv_ksplit(ntasks, cols, sm_count) : 1, flags, s);
}

// Parse + the checks of doublepir.rs:246-350 for one request; chunk < 0: unchunked.
int dpir_prepare_call(b200pir_dpir_server* S, const uint8_t* req, size_t len, int64_t chunk, DpirCall& c, std::string& err) {
  c.req = req;
  int rc = parse_dpir_request(req, len, S->e, S->c1, c.w, err);
  if (!rc) rc = check_dpir_batches(c.w, S->l, S->db->rows, S->dcols, chunk, err);
  c.L = DpirResponseLayout{c.w.queries, S->e, S->dx, S->n, S->rows1};
  return rc;
}

// The passes of answer() for every request of `calls` on the server's stream; responses to outs[i].  Everything has been
// checked; no allocation, no device-wide synchronisation, one upload and one download.
void dpir_serve(b200pir_dpir_server* S, std::vector<DpirCall>& calls, int64_t chunk, uint8_t* const* outs, size_t* out_lens) {
  const size_t R = calls.size();
  cudaStream_t s = S->stream;
  // ---- stage the vectors the passes read (the request's bytes as they are: big-endian words, swapped by the kernels)
  size_t off = 0;
  auto stage = [&](const DpirCall& c, const DpirWireMat& m) {
    const size_t bytes = (size_t)m.rows * 4;
    if (off + bytes > S->stage_cap) throw Error(B200PIR_E_SHAPE, "dpir: staging overflow");
    std::memcpy(S->h_stage + off, c.req + m.data_pos(), bytes);
    const uint32_t* dev = reinterpret_cast<const uint32_t*>(S->d_stage.p + off);
    off = align_up(off + bytes, 16);
    return dev;
  };
  size_t resp_total = 0;
  for (auto& c : calls) {
    c.q1.assign(c.w.queries, nullptr);
    c.q2.assign(c.w.queries * S->e, nullptr);
    for (size_t k = 0; k < c.w.queries; k++) {
      if (chunk < 0 || (uint64_t)chunk == k) c.q1[k] = stage(c, c.w.q1(k));
      for (size_t j = 0; j < S->e; j++) c.q2[k * S->e + j] = stage(c, c.w.q2(k, j));
    }
    c.resp_off = resp_total;
    resp_total += c.L.bytes();
  }
  if (resp_total > S->resp_cap) throw Error(B200PIR_E_SHAPE, "dpir: response workspace overflow");
  // ---- which kernel each pass runs, from the vectors it holds and the matrix rows; the tensor-core passes read query images
  uint64_t total_q = 0;
  for (const auto& c : calls) total_q += c.w.queries;
  const bool tc_db = dpir_use_tc(chunk >= 0 ? 1 : R, chunk >= 0 ? dpir_batch_rows(S->l, calls[0].w.queries, chunk) : S->l);
  const bool tc_h1 = dpir_use_tc(total_q * S->e, S->rows1);
  const size_t cap_db = tc_db ? DTC_VECS : kDpirMvMaxVecs, cap_h1 = tc_h1 ? DTC_VECS : kDpirMvMaxVecs;
  std::vector<DpirTcImage> jobs;
  {
    size_t n1 = 0, n2 = 0;
    for (auto& c : calls) {
      c.q1i.assign(c.q1.size(), nullptr);
      c.q2i.assign(c.q2.size(), nullptr);
      for (size_t k = 0; tc_db && k < c.q1.size(); k++)
        if (c.q1[k]) {
          uint8_t* img = S->d_img.p + n1++ * S->img_q1;
          jobs.push_back(DpirTcImage{c.q1[k], img, (uint32_t)S->dcols});
          c.q1i[k] = reinterpret_cast<const uint32_t*>(img);
        }
      for (size_t k = 0; tc_h1 && k < c.q2.size(); k++) {
        uint8_t* img = S->d_img.p + S->max_queries * S->img_q1 + n2++ * S->img_q2;
        jobs.push_back(DpirTcImage{c.q2[k], img, (uint32_t)S->c1});
        c.q2i[k] = reinterpret_cast<const uint32_t*>(img);
      }
    }
    if (n1 > S->max_queries || n2 > S->max_queries * S->e) throw Error(B200PIR_E_SHAPE, "dpir: query image workspace overflow");
  }
  // ---- task tables: database pass, h_1 pass, a_1' * q_2
  std::vector<DpirMvTask> tasks;
  std::vector<DpirMvVec> vecs;
  uint8_t* resp = S->d_resp.p;
  int vmax_db = 1, vmax_h1 = 1, vmax_a1 = 1;
  if (chunk >= 0) {             // one request: batch `chunk` from rows [0, its size) of the server's matrix
    const DpirCall& c = calls[0];
    const uint64_t nq = c.w.queries, rows = dpir_batch_rows(S->l, nq, chunk);
    vecs.push_back(DpirMvVec{tc_db ? c.q1i[chunk] : c.q1[chunk], S->d_a1.p + dpir_batch_begin(S->l, nq, chunk)});
    add_tiles(tasks, S->db->a.p, rows, S->dcols, 0, 1, tc_db);
  } else {                      // the rows cut at every request's batch boundaries: one q_1 per request in each segment
    std::vector<uint64_t> cuts{0, S->l};
    for (const auto& c : calls)
      for (uint64_t k = 1; k < c.w.queries; k++) cuts.push_back(dpir_batch_begin(S->l, c.w.queries, k));
    std::sort(cuts.begin(), cuts.end());
    cuts.erase(std::unique(cuts.begin(), cuts.end()), cuts.end());
    for (size_t g = 0; g + 1 < cuts.size(); g++) {
      const uint64_t s0 = cuts[g], s1 = cuts[g + 1];
      for (size_t i0 = 0; i0 < R; i0 += cap_db) {
        const uint32_t vec0 = (uint32_t)vecs.size(), nv = (uint32_t)std::min<size_t>(cap_db, R - i0);
        for (size_t i = i0; i < i0 + nv; i++) {
          const uint64_t nq = calls[i].w.queries, bs = S->l / nq;
          const uint64_t k = bs ? std::min(s0 / bs, nq - 1) : nq - 1;
          vecs.push_back(DpirMvVec{tc_db ? calls[i].q1i[k] : calls[i].q1[k], S->d_a1.p + i * S->l + s0});
        }
        vmax_db = std::max<int>(vmax_db, nv);
        add_tiles(tasks, S->db->a.p + s0 * S->dcols, s1 - s0, S->dcols, vec0, nv, tc_db);
      }
    }
  }
  const size_t t_h1 = tasks.size();
  {
    std::vector<DpirMvVec> all;
    for (const auto& c : calls)
      for (size_t k = 0; k < c.w.queries; k++)
        for (size_t j = 0; j < S->e; j++)
          all.push_back(DpirMvVec{tc_h1 ? c.q2i[k * S->e + j] : c.q2[k * S->e + j],
                                  reinterpret_cast<uint32_t*>(resp + c.resp_off + c.L.a2_data(k, j))});
    for (size_t v0 = 0; v0 < all.size(); v0 += cap_h1) {
      const uint32_t vec0 = (uint32_t)vecs.size(), nv = (uint32_t)std::min<size_t>(cap_h1, all.size() - v0);
      vecs.insert(vecs.end(), all.begin() + v0, all.begin() + v0 + nv);
      vmax_h1 = std::max<int>(vmax_h1, nv);
      add_tiles(tasks, S->h1.p, S->rows1, S->c1, vec0, nv, tc_h1);
    }
  }
  const size_t t_a1 = tasks.size();
  for (size_t i = 0; i < R; i++) {
    const DpirCall& c = calls[i];
    std::vector<DpirMvVec> mine;
    for (size_t k = 0; k < c.w.queries; k++)
      for (size_t j = 0; j < S->e; j++)
        mine.push_back(DpirMvVec{c.q2[k * S->e + j], reinterpret_cast<uint32_t*>(resp + c.resp_off + c.L.h2_data(k, j))});
    for (size_t v0 = 0; v0 < mine.size(); v0 += kDpirMvMaxVecs) {
      const uint32_t vec0 = (uint32_t)vecs.size(), nv = (uint32_t)std::min<size_t>(kDpirMvMaxVecs, mine.size() - v0);
      vecs.insert(vecs.end(), mine.begin() + v0, mine.begin() + v0 + nv);
      vmax_a1 = std::max<int>(vmax_a1, nv);
      add_tiles(tasks, S->d_a1sq.p + i * S->dx * S->c1, S->dx, S->c1, vec0, nv, false);
    }
  }
  if (tasks.size() > S->task_cap || vecs.size() > S->vec_cap) throw Error(B200PIR_E_SHAPE, "dpir: task table overflow");
  const size_t off_tasks = off, off_vecs = align_up(off_tasks + tasks.size() * sizeof(DpirMvTask), 16);
  const size_t off_jobs = align_up(off_vecs + vecs.size() * sizeof(DpirMvVec), 16);
  const size_t used = off_jobs + jobs.size() * sizeof(DpirTcImage);
  if (used > S->stage_cap) throw Error(B200PIR_E_SHAPE, "dpir: staging overflow");
  std::memcpy(S->h_stage + off_tasks, tasks.data(), tasks.size() * sizeof(DpirMvTask));
  std::memcpy(S->h_stage + off_vecs, vecs.data(), vecs.size() * sizeof(DpirMvVec));
  std::memcpy(S->h_stage + off_jobs, jobs.data(), jobs.size() * sizeof(DpirTcImage));
  const DpirMvTask* d_tasks = reinterpret_cast<const DpirMvTask*>(S->d_stage.p + off_tasks);
  const DpirMvVec* d_vecs = reinterpret_cast<const DpirMvVec*>(S->d_stage.p + off_vecs);
  // ---- the passes: the h_1 and a_1' passes store big-endian results, so they never split k; the database pass adds into
  // zeroed a_1
  B200_CUDA(cudaMemcpyAsync(S->d_stage.p, S->h_stage, used, cudaMemcpyHostToDevice, s));
  B200_CUDA(cudaMemsetAsync(S->d_a1.p, 0, R * S->l * 4, s));   // split-k partial sums add into it; unread batches stay zero
  launch_dpir_tc_image(reinterpret_cast<const DpirTcImage*>(S->d_stage.p + off_jobs), jobs.size(), std::max(S->dcols, S->c1),
                       DPIR_MV_B_BE, s);
  launch_matvec_pass(tc_db, d_tasks, t_h1, d_vecs, S->dcols, vmax_db, true, S->sm_count, DPIR_MV_B_BE, s);
  for (size_t i = 0; i < R; i++)        // a_1.transpose_expand_concat_cols_squish(p, delta, x, 10, 3)
    launch_dpir_transpose_expand(S->d_a1sq.p + i * S->dx * S->c1, S->d_a1.p + i * S->l, S->l, 1, S->p, S->delta, S->x, S->dx,
                                 S->c1, s);
  // msg[0] = matrix_mul_transposed_packed(a_1', a_2^T) of every request at once (their a_1' are stacked)
  launch_dpir_mul_transposed(S->d_msg0.p, S->d_a1sq.p, S->a2t.p, R * S->dx, S->c1, S->n, S->lx3, s);
  for (size_t i = 0; i < R; i++)
    launch_dpir_bswap(reinterpret_cast<uint32_t*>(resp + calls[i].resp_off + calls[i].L.msg0_data()), S->d_msg0.p + i * S->dx * S->n,
                      S->dx * S->n, s);
  launch_matvec_pass(tc_h1, d_tasks + t_h1, t_a1 - t_h1, d_vecs, S->c1, vmax_h1, false, S->sm_count,
                     DPIR_MV_B_BE | DPIR_MV_OUT_BE, s);
  launch_matvec_pass(false, d_tasks + t_a1, tasks.size() - t_a1, d_vecs, S->c1, vmax_a1, false, S->sm_count,
                     DPIR_MV_B_BE | DPIR_MV_OUT_BE, s);
  B200_CUDA(cudaGetLastError());
  B200_CUDA(cudaMemcpyAsync(S->h_resp, S->d_resp.p, resp_total, cudaMemcpyDeviceToHost, s));
  B200_CUDA(cudaStreamSynchronize(s));
  B200_CUDA(cudaGetLastError());
  for (size_t i = 0; i < R; i++) {
    const DpirCall& c = calls[i];
    std::memcpy(outs[i], S->h_resp + c.resp_off, c.L.bytes());
    write_dpir_response_headers(c.L, outs[i]);
    out_lens[i] = c.L.bytes();
  }
}
}  // namespace

int b200pir_dpir_server_create(int device, const b200pir_dpir_params* params, uint64_t num_entries, uint64_t bits_per_entry,
                               b200pir_dpir* db, const uint32_t* h1_squished, const uint32_t* a2_t, size_t max_queries,
                               b200pir_dpir_server** out) {
  API_BEGIN
  if (!params || !db || !h1_squished || !a2_t || !out) throw Error(B200PIR_E_BADARG, "null argument");
  if (max_queries == 0 || max_queries >= kDpirWireMaxLen) throw Error(B200PIR_E_BADARG, "max_queries must lie in [1, 2^28)");
  const b200pir_dpir_info info = dpir_info(params, num_entries, bits_per_entry, nullptr, 64);
  if (device != db->device) throw Error(B200PIR_E_BADARG, "the database lives on another device");
  const uint64_t l = params->l, x = info.x;
  if (l % x) throw Error(B200PIR_E_SHAPE, "l must be a multiple of x (concat_cols)");
  if (db->cols != (params->m + 2) / 3) throw Error(B200PIR_E_SHAPE, "the database's packed columns are not ceil(m / 3)");
  if (db->rows > l) throw Error(B200PIR_E_SHAPE, "the database has more than l rows");
  use_device(device);
  std::unique_ptr<b200pir_dpir_server> S(new b200pir_dpir_server());
  S->device = device;
  S->db = db;
  S->params = *params;
  S->num_entries = num_entries;
  S->bits_per_entry = bits_per_entry;
  S->n = params->n; S->l = l; S->p = params->p; S->delta = info.delta; S->x = x; S->e = info.ne / x;
  S->dx = info.delta * x; S->rows1 = S->n * S->dx; S->c1 = (l / x + 2) / 3; S->lx3 = 3 * S->c1; S->dcols = db->cols;
  S->max_queries = max_queries;
  B200_CUDA(cudaDeviceGetAttribute(&S->sm_count, cudaDevAttrMultiProcessorCount, device));
  OwnedStream st;
  S->stream = st.s;
  const uint64_t Q = max_queries, e = S->e;
  // bounds of one call: at most Q requests and Q queries; the database pass has at most Q row segments (each request of k
  // queries adds k - 1 cuts), each tiled and repeated once per pass of vectors.  A pass on k_dpir_matvec_multi (32 rows a task,
  // 16 vectors a pass) makes at least as many tasks as one on the tensor cores (64 rows, 64 vectors), so its count bounds both.
  S->task_cap = (ceil_div(l, kDpirMvRows) + Q) * ceil_div(Q, kDpirMvMaxVecs)
              + ceil_div(S->rows1, kDpirMvRows) * ceil_div(Q * e, kDpirMvMaxVecs)
              + ceil_div(S->dx, kDpirMvRows) * Q * e;
  S->vec_cap = Q * Q + 2 * Q * e;
  S->stage_cap = Q * (align_up(3 * S->dcols * 4, 16) + e * align_up(3 * S->c1 * 4, 16)) + align_up(S->task_cap * sizeof(DpirMvTask), 16)
               + align_up(S->vec_cap * sizeof(DpirMvVec), 16) + Q * (1 + e) * sizeof(DpirTcImage);
  S->img_q1 = dtc_img_bytes(S->dcols);
  S->img_q2 = dtc_img_bytes(S->c1);
  S->resp_cap = Q * (12 + S->dx * S->n * 4) + Q * e * DpirResponseLayout{1, e, S->dx, S->n, S->rows1}.pair_bytes();
  B200_CUDA(cudaMallocHost(&S->h_stage, S->stage_cap));
  B200_CUDA(cudaMallocHost(&S->h_resp, S->resp_cap));
  S->d_stage.alloc(S->stage_cap);
  S->d_resp.alloc(S->resp_cap);
  S->d_a1.alloc(Q * l);
  S->d_a1sq.alloc(Q * S->dx * S->c1);
  S->d_msg0.alloc(Q * S->dx * S->n);
  S->d_img.alloc(Q * S->img_q1 + Q * e * S->img_q2);
  S->h1.alloc(S->rows1 * S->c1);
  S->a2t.alloc(S->n * S->lx3);
  B200_CUDA(cudaMemcpyAsync(S->h1.p, h1_squished, S->h1.n * 4, cudaMemcpyHostToDevice, S->stream));
  B200_CUDA(cudaMemcpyAsync(S->a2t.p, a2_t, S->a2t.n * 4, cudaMemcpyHostToDevice, S->stream));
  B200_CUDA(cudaStreamSynchronize(S->stream));
  st.release();
  *out = S.release();
  API_END
}

void b200pir_dpir_server_destroy(b200pir_dpir_server* S) {
  if (!S) return;
  cudaSetDevice(S->device);
  if (S->stream) {
    cudaStreamSynchronize(S->stream);
    cudaStreamDestroy(S->stream);
  }
  delete S;
}

int b200pir_dpir_answer_size(b200pir_dpir_server* S, const uint8_t* request, size_t len, size_t* out_len) {
  API_BEGIN
  if (!S || !request || !out_len) throw Error(B200PIR_E_BADARG, "null argument");
  DpirWireRequest w;
  std::string err;
  if (int rc = parse_dpir_request(request, len, S->e, S->c1, w, err)) throw Error(rc, err);
  *out_len = DpirResponseLayout{w.queries, S->e, S->dx, S->n, S->rows1}.bytes();
  API_END
}

int b200pir_dpir_answer(b200pir_dpir_server* S, const uint8_t* request, size_t len, int64_t chunk_idx, uint8_t* out,
                        size_t* out_len) {
  API_BEGIN
  if (!S || !request || !out || !out_len) throw Error(B200PIR_E_BADARG, "null argument");
  std::vector<DpirCall> calls(1);
  std::string err;
  if (int rc = dpir_prepare_call(S, request, len, chunk_idx < 0 ? -1 : chunk_idx, calls[0], err)) throw Error(rc, err);
  if (calls[0].w.queries > S->max_queries)
    throw Error(B200PIR_E_SHAPE, "the request has " + std::to_string(calls[0].w.queries) + " queries; this server answers at most " +
                                     std::to_string(S->max_queries) + " a call (max_queries)");
  if (*out_len < calls[0].L.bytes()) throw Error(B200PIR_E_BADARG, "the output holds fewer bytes than the response");
  std::lock_guard<std::mutex> lk(S->mu);
  cudaSetDevice(S->device);
  dpir_serve(S, calls, chunk_idx < 0 ? -1 : chunk_idx, &out, out_len);
  API_END
}

int b200pir_dpir_answer_many(b200pir_dpir_server* S, const uint8_t* const* requests, const size_t* lens, size_t count,
                             uint8_t* const* outs, size_t* out_lens) {
  API_BEGIN
  if (!S || (count && (!requests || !lens || !outs || !out_lens))) throw Error(B200PIR_E_BADARG, "null argument");
  for (size_t i = 0; i < count; i++)
    if (!requests[i] || !outs[i]) throw Error(B200PIR_E_BADARG, "null request or output " + std::to_string(i));
  if (count == 0) return 0;
  std::vector<DpirCall> calls(count);
  uint64_t total = 0;
  for (size_t i = 0; i < count; i++) {
    std::string err;
    if (int rc = dpir_prepare_call(S, requests[i], lens[i], -1, calls[i], err)) throw Error(rc, "request " + std::to_string(i) + ": " + err);
    total += calls[i].w.queries;
  }
  if (total > S->max_queries)
    throw Error(B200PIR_E_SHAPE, "the call has " + std::to_string(total) + " queries; this server answers at most " +
                                     std::to_string(S->max_queries) + " a call (max_queries)");
  for (size_t i = 0; i < count; i++)
    if (out_lens[i] < calls[i].L.bytes()) throw Error(B200PIR_E_BADARG, "output " + std::to_string(i) + " holds fewer bytes than its response");
  std::lock_guard<std::mutex> lk(S->mu);
  cudaSetDevice(S->device);
  dpir_serve(S, calls, -1, outs, out_lens);
  API_END
}

// ---------------------------------------------------------------- DoublePIR entry updates (dpir_update.cu)
namespace {
constexpr size_t kDpirUpdGroup = 4096;    // changed elements (and so at most as many changed rows) patched per group

// The batch as element patches sorted by (row, column): a repeated index ends with its last value, and the entries of one
// packed element are combined into one patch.  Everything has been checked.
std::vector<DpirUpdElem> dpir_update_elems(const b200pir_dpir* db, const b200pir_dpir_info& info, const uint64_t* idx, const uint8_t* val,
                                           size_t count) {
  std::vector<size_t> ord(count);
  for (size_t k = 0; k < count; k++) ord[k] = k;
  std::stable_sort(ord.begin(), ord.end(), [idx](size_t a, size_t b) { return idx[a] < idx[b]; });
  const uint64_t m = db->params.m, bits = db->bits_per_entry;
  const uint32_t p = (uint32_t)db->params.p;
  std::vector<DpirUpdElem> el;
  for (size_t k = 0; k < count; k++) {
    if (k + 1 < count && idx[ord[k + 1]] == idx[ord[k]]) continue;        // a later value of the same index wins
    const uint64_t i = idx[ord[k]];
    const uint32_t v = val[ord[k]];
    if (info.packing) {                   // bit field i % packing of element i / packing (sorted indices: elements in order)
      const uint64_t e = i / info.packing;
      const uint32_t sh = (uint32_t)(bits * (i % info.packing)), fm = ((1u << bits) - 1) << sh;
      if (el.empty() || el.back().r * m + el.back().c != e) el.push_back(DpirUpdElem{e / m, e % m, 0, 0});
      el.back().mask |= fm;
      el.back().val = (el.back().val & ~fm) | (v << sh);
    } else {                              // digit j = base_p(p, v, j) at row (i / m) ne + j, column i % m
      uint32_t d = v;
      for (uint64_t j = 0; j < info.ne; j++, d /= p) el.push_back(DpirUpdElem{(i / m) * info.ne + j, i % m, 0xFFFFFFFFu, d % p});
    }
  }
  if (!info.packing)
    std::sort(el.begin(), el.end(), [](const DpirUpdElem& a, const DpirUpdElem& b) { return a.r != b.r ? a.r < b.r : a.c < b.c; });
  return el;
}

// One group of the batch: elements [e_off, e_off + n_el) and their rows [r_off, r_off + n_rows); blocks: (b, k0_b, k_b) of the
// blocks b = r % x that have changed rows
struct DpirUpdGroup {
  size_t e_off, n_el, r_off, n_rows;
  std::vector<std::array<uint64_t, 3>> blocks;
};

// Store, h_1 and hint patches of every group on the server's stream; h2 (host, (n delta x) x n) in and out.  Synchronises.
void dpir_update(b200pir_dpir_server* S, const std::vector<DpirUpdElem>& el, uint32_t* h2) {
  const cudaStream_t s = S->stream;
  const uint64_t n = S->n, x = S->x, nd = n * S->delta;
  std::vector<DpirUpdRow> rows;
  std::vector<DpirUpdGroup> groups;
  for (size_t g0 = 0; g0 < el.size(); g0 += kDpirUpdGroup) {
    DpirUpdGroup G{g0, std::min(kDpirUpdGroup, el.size() - g0), rows.size(), 0, {}};
    std::vector<DpirUpdRow> gr;
    for (size_t k = 0; k < G.n_el; k++) {
      if (gr.empty() || gr.back().r != el[g0 + k].r) gr.push_back(DpirUpdRow{el[g0 + k].r, 0, (uint32_t)k, 0, 0, 0});
      gr.back().ne++;
    }
    std::stable_sort(gr.begin(), gr.end(), [x](const DpirUpdRow& a, const DpirUpdRow& b) { return a.r % x < b.r % x; });
    for (size_t k0 = 0; k0 < gr.size();) {
      size_t k1 = k0;
      while (k1 < gr.size() && gr[k1].r % x == gr[k0].r % x) k1++;
      for (size_t k = k0; k < k1; k++) {
        gr[k].doff = nd * k0;
        gr[k].dcol = (uint32_t)(k - k0);
        gr[k].kb = (uint32_t)(k1 - k0);
      }
      G.blocks.push_back({gr[k0].r % x, k0, k1 - k0});
      k0 = k1;
    }
    G.n_rows = gr.size();
    rows.insert(rows.end(), gr.begin(), gr.end());
    groups.push_back(std::move(G));
  }
  // scratch: sized for the largest group this batch can have, grown only for a larger batch
  const size_t cap = std::min(kDpirUpdGroup, el.size());
  if (cap > S->upd_cap) {
    S->u_dh1.alloc(cap * n);
    S->u_a2g.alloc(cap * n);
    S->u_D.alloc(nd * cap);
    S->u_aimg.alloc(dpir_gemm_a_bytes(nd, cap));
    S->u_bimg.alloc(dpir_gemm_b_bytes(cap, n));
    S->upd_cap = cap;
  }
  if (el.size() > S->upd_tab) {
    S->u_el.alloc(el.size());
    S->u_rows.alloc(el.size());
    S->u_delta.alloc(el.size());
    S->upd_tab = el.size();
  }
  S->u_dh2.ensure(nd * n);
  S->u_h2.ensure(nd * x * n);
  if (!S->have_a1_key) {
    S->a1_key = dpir_aes_key(kDpirSeedA1);
    S->have_a1_key = true;
  }
  b200pir_dpir* db = S->db;
  B200_CUDA(cudaStreamSynchronize(db->stream));          // work still queued on the database handle's own stream first
  B200_CUDA(cudaMemcpyAsync(S->u_el.p, el.data(), el.size() * sizeof(DpirUpdElem), cudaMemcpyHostToDevice, s));
  B200_CUDA(cudaMemcpyAsync(S->u_rows.p, rows.data(), rows.size() * sizeof(DpirUpdRow), cudaMemcpyHostToDevice, s));
  B200_CUDA(cudaMemcpyAsync(S->u_h2.p, h2, nd * x * n * 4, cudaMemcpyHostToDevice, s));
  for (const DpirUpdGroup& G : groups) {
    const DpirUpdElem* gel = S->u_el.p + G.e_off;
    const DpirUpdRow* grows = S->u_rows.p + G.r_off;
    int32_t* gdelta = S->u_delta.p + G.e_off;
    launch_dpir_upd_store(db->a.p, db->cols, gel, (uint32_t)G.n_el, gdelta, s);
    launch_dpir_upd_dh1(S->u_dh1.p, grows, (uint32_t)G.n_rows, gel, gdelta, n, S->a1_key, s);
    launch_dpir_upd_digits(S->h1.p, S->c1, S->u_D.p, grows, (uint32_t)G.n_rows, S->u_dh1.p, n, (uint32_t)S->p, (uint32_t)S->delta, x, s);
    launch_dpir_upd_gather_a2(S->u_a2g.p, S->a2t.p, S->lx3, grows, (uint32_t)G.n_rows, n, x, s);
    for (const auto& B : G.blocks) {                     // dh_2[block b] = D_b (nd x k_b) * A_2 rows (k_b x n)
      const uint64_t b = B[0], k0 = B[1], kb = B[2];
      launch_dpir_gemm_b_image(S->u_bimg.p, S->u_a2g.p + k0 * n, kb, n, s);
      launch_dpir_gemm_rows(S->u_dh2.p, S->u_aimg.p, reinterpret_cast<const uint32_t*>(S->u_D.p) + nd * k0, nd, kb, S->u_bimg.p, n, s);
      launch_dpir_upd_add(S->u_h2.p + b * nd * n, S->u_dh2.p, nd * n, s);
    }
  }
  B200_CUDA(cudaGetLastError());
  B200_CUDA(cudaMemcpyAsync(h2, S->u_h2.p, nd * x * n * 4, cudaMemcpyDeviceToHost, s));
  B200_CUDA(cudaStreamSynchronize(s));
  B200_CUDA(cudaGetLastError());
}
}  // namespace

int b200pir_dpir_server_update(b200pir_dpir_server* S, const uint64_t* indices, const uint8_t* values, size_t count, uint32_t* h2) {
  API_BEGIN
  if (!S || !h2 || (count && (!indices || !values))) throw Error(B200PIR_E_BADARG, "null argument");
  b200pir_dpir* db = S->db;
  if (!db->from_load) throw Error(B200PIR_E_UNSUPPORTED, "update: the server's database was not laid out by b200pir_dpir_load*");
  if (db->rows < S->l) throw Error(B200PIR_E_UNSUPPORTED, "update: the server holds a chunk of the database (fewer than l rows)");
  if (!db->fields_exact)
    throw Error(B200PIR_E_UNSUPPORTED, "update: the load packed entries wider than bits_per_entry; its elements do not decode field by field");
  const b200pir_dpir_params& P = db->params;
  if (S->num_entries != db->num_entries || S->bits_per_entry != db->bits_per_entry || S->params.n != P.n || S->params.l != P.l ||
      S->params.m != P.m || S->params.logq != P.logq || S->params.p != P.p)
    throw Error(B200PIR_E_SHAPE, "update: the server's parameters, num_entries or bits_per_entry differ from its database's load");
  if (S->n * 4 > 200 * 1024) throw Error(B200PIR_E_UNSUPPORTED, "update: n above 51200");
  const b200pir_dpir_info info = dpir_info(&P, db->num_entries, db->bits_per_entry, nullptr);
  const bool bits_format = db->entry_format == B200PIR_DPIR_ENTRY_BITS;
  for (size_t k = 0; k < count; k++) {
    if (indices[k] >= db->load_count)
      throw Error(B200PIR_E_SHAPE, "update: index " + std::to_string(indices[k]) + " is past the " + std::to_string(db->load_count) +
                                       " entries the load read");
    if ((bits_format && values[k] > 1) || (info.packing && (values[k] >> db->bits_per_entry)))
      throw Error(B200PIR_E_BADARG, "update: value " + std::to_string(values[k]) + " of entry " + std::to_string(indices[k]) +
                                        " does not fit the entry format");
  }
  if (count == 0) return 0;
  const std::vector<DpirUpdElem> el = dpir_update_elems(db, info, indices, values, count);
  std::lock_guard<std::mutex> lk(S->mu);
  std::lock_guard<std::mutex> lk_db(db->mu);
  cudaSetDevice(S->device);
  dpir_update(S, el, h2);
  API_END
}

int b200pir_dpir_server_state(b200pir_dpir_server* S, uint32_t* h1_squished) {
  API_BEGIN
  if (!S || !h1_squished) throw Error(B200PIR_E_BADARG, "null argument");
  std::lock_guard<std::mutex> lk(S->mu);
  cudaSetDevice(S->device);
  B200_CUDA(cudaMemcpyAsync(h1_squished, S->h1.p, S->h1.n * 4, cudaMemcpyDeviceToHost, S->stream));
  B200_CUDA(cudaStreamSynchronize(S->stream));
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
  const size_t cap = tc ? DTC_VECS : kDpirMvMaxVecs, img = dtc_img_bytes(m->cols);
  DevBuf<uint32_t> d_b(count * 3 * m->cols), d_out(count * m->rows);
  DevBuf<uint8_t> d_img(tc ? count * img : 0);
  std::vector<DpirMvTask> tasks;
  std::vector<DpirMvVec> vecs;
  std::vector<DpirTcImage> jobs;
  int vmax = 1;
  for (size_t v0 = 0; v0 < count; v0 += cap) {
    const uint32_t vec0 = (uint32_t)vecs.size(), nv = (uint32_t)std::min<size_t>(cap, count - v0);
    for (size_t v = v0; v < v0 + nv; v++) {
      const uint32_t* bv = d_b.p + v * 3 * m->cols;
      if (tc) jobs.push_back(DpirTcImage{bv, d_img.p + v * img, (uint32_t)m->cols});
      vecs.push_back(DpirMvVec{tc ? reinterpret_cast<const uint32_t*>(d_img.p + v * img) : bv, d_out.p + v * m->rows});
    }
    vmax = std::max<int>(vmax, nv);
    add_tiles(tasks, m->a.p, m->rows, m->cols, vec0, nv, tc);
  }
  DevBuf<DpirMvTask> d_tasks(tasks.size());
  DevBuf<DpirMvVec> d_vecs(vecs.size());
  DevBuf<DpirTcImage> d_jobs(jobs.size());
  B200_CUDA(cudaMemcpyAsync(d_tasks.p, tasks.data(), tasks.size() * sizeof(DpirMvTask), cudaMemcpyHostToDevice, m->stream));
  B200_CUDA(cudaMemcpyAsync(d_vecs.p, vecs.data(), vecs.size() * sizeof(DpirMvVec), cudaMemcpyHostToDevice, m->stream));
  if (tc) B200_CUDA(cudaMemcpyAsync(d_jobs.p, jobs.data(), jobs.size() * sizeof(DpirTcImage), cudaMemcpyHostToDevice, m->stream));
  B200_CUDA(cudaMemcpyAsync(d_b.p, b, d_b.n * 4, cudaMemcpyHostToDevice, m->stream));
  B200_CUDA(cudaMemsetAsync(d_out.p, 0, d_out.n * 4, m->stream));
  if (tc) launch_dpir_tc_image(d_jobs.p, jobs.size(), m->cols, 0, m->stream);
  launch_matvec_pass(tc, d_tasks.p, tasks.size(), d_vecs.p, m->cols, vmax, true, sms, 0, m->stream);
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
