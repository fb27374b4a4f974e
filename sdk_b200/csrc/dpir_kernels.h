// Launch wrappers (host side) for DoublePIR's sm_90a kernels, in the conventions of kernels.h: DEVICE pointers unless noted,
// every launch on the given stream, returning immediately.
#pragma once
#include "kernels.h"
#include "dpir_tc_layout.cuh"   // DTC_ROWS, DTC_VECS, dtc_img_bytes

namespace b200pir {

// ---- DoublePIR packed matvec (K6, dpir_serve.cu): lib/doublepir/src/matrix/kernels.rs:14-178
// even cols: k_dpir_matvec_row, odd cols: k_dpir_matvec, rows too wide for `b` in shared memory: k_dpir_matvec_wide
void launch_dpir_matvec(uint32_t* out, const uint32_t* a, const uint32_t* b, size_t rows, size_t cols, cudaStream_t s);

// lib/doublepir/src/matrix/kernels.rs:180-278 and matrix/indexing.rs:117-143 (the small tail of answer())
void launch_dpir_mul_transposed(uint32_t* out, const uint32_t* a, const uint32_t* b, size_t a_rows, size_t a_cols,
                                size_t b_rows, size_t b_cols, cudaStream_t s);
void launch_dpir_transpose_expand(uint32_t* out, const uint32_t* a, size_t rows, size_t cols, uint64_t modulus, size_t delta,
                                  size_t concat, size_t out_rows, size_t out_cols, cudaStream_t s);

// ---- DoublePIR packed matrix x many vectors (dpir_serve.cu): the passes of answer() over every request of a call
// A task is one CTA: rows [0, rows) (rows <= kDpirMvRows) of the matrix at `a` (rows `cols` words apart) against the vectors
// vecs[vec0, vec0 + nv) (nv <= kDpirMvMaxVecs); vector v's result for row r goes to vecs[vec0 + v].out[out_off + r].
constexpr int kDpirMvRows = 32;
constexpr int kDpirMvMaxVecs = 16;
struct DpirMvTask { const uint32_t* a; uint32_t rows, vec0, nv, out_off; };
struct DpirMvVec { const uint32_t* b; uint32_t* out; };          // b: 3 * cols words
enum { DPIR_MV_B_BE = 1,        // vector words are big-endian (wire order): swapped as they are staged
       DPIR_MV_OUT_BE = 2 };    // results are stored big-endian (wire order); needs ksplit == 1
// ksplit > 1 splits every task's k range over that many CTAs whose partial sums are added with atomicAdd into outputs the
// caller has zeroed.  vmax = the largest nv of any task.
void launch_dpir_matvec_multi(const DpirMvTask* tasks, size_t ntasks, const DpirMvVec* vecs, size_t cols, int vmax, int ksplit,
                              int flags, cudaStream_t s);
// the k split that gives `ntasks` tasks about two CTAs an SM, each at least one 256-column chunk
int dpir_mv_ksplit(size_t ntasks, size_t cols, int sm_count);
// dst[i] = byte-swapped src[i]
void launch_dpir_bswap(uint32_t* dst, const uint32_t* src, size_t words, cudaStream_t s);
// dst[i] = byte-swapped (sum over g < nparts of parts[g * stride + i]) mod 2^32, for i < words: a sharded server's partial
// responses, one buffer of stride words per shard, into the wire-order response
void launch_dpir_sum_be(uint32_t* dst, const uint32_t* parts, size_t stride, size_t nparts, size_t words, cudaStream_t s);

// ---- the same passes on the tensor cores (dpir_tc.cu, index maps in dpir_tc_layout.cuh): tasks of up to DTC_ROWS rows and
// DTC_VECS vectors, whose DpirMvVec::b points at the vector's query image (dtc_img_bytes(cols) bytes, 16-byte aligned) instead of
// its words.  Flags and ksplit as launch_dpir_matvec_multi (DPIR_MV_B_BE is applied when the images are built).
struct DpirTcImage { const uint32_t* b; uint8_t* img; uint32_t cols; };   // b: 3 * cols words -> img
void launch_dpir_tc_image(const DpirTcImage* jobs, size_t njobs, size_t max_cols, int flags, cudaStream_t s);
void launch_dpir_matvec_tc(const DpirMvTask* tasks, size_t ntasks, const DpirMvVec* vecs, size_t cols, int ksplit, int flags,
                           cudaStream_t s);
// the k split that gives `ntasks` tasks about four waves of one CTA an SM, each at least one 32-word chunk
int dpir_tc_ksplit(size_t ntasks, size_t cols, int sm_count);
// which kernel a pass of `nv` vectors (the most any task of the pass holds) over `rows` matrix rows runs on
bool dpir_use_tc(size_t nv, size_t rows);

// ---- DoublePIR offline setup (dpir_gemm.cu): doublepir.rs:76-108
// c (rows x n_cols) = a (rows x k_dim, entries in [-2^15, 2^15) as wrapping u32) * b (k_dim x n_cols) mod 2^32; device pointers;
// 8-bit limb products on the tensor cores (wgmma) (exact); synchronises the stream
void launch_dpir_gemm(uint32_t* c, const uint32_t* a, const uint32_t* b, size_t rows, size_t k_dim, size_t n_cols, cudaStream_t s);
// The same in two steps on caller-owned operand images, with no allocation and no synchronisation: the image of b once
// (dpir_gemm_b_bytes), then any number of row ranges of a, each through an a image of dpir_gemm_a_bytes(rows, k_dim) bytes
size_t dpir_gemm_a_bytes(size_t rows, size_t k_dim);
size_t dpir_gemm_b_bytes(size_t k_dim, size_t n_cols);
void launch_dpir_gemm_b_image(uint8_t* b_img, const uint32_t* b, size_t k_dim, size_t n_cols, cudaStream_t s);
void launch_dpir_gemm_rows(uint32_t* c, uint8_t* a_img, const uint32_t* a, size_t rows, size_t k_dim, const uint8_t* b_img,
                           size_t n_cols, cudaStream_t s);
// transpose + expand (contract.rs:62-78) + concat_cols (indexing.rs:82-101): h (l x n) -> out ((n delta x) x (l / x)), centred digits
void launch_dpir_transpose_expand_concat(uint32_t* out, const uint32_t* h, size_t l, size_t n, uint32_t p, int delta, size_t x,
                                         cudaStream_t s);
// squish(m + add), three 10-bit values per word (squish.rs:52-70)
void launch_dpir_add_squish(uint32_t* out, const uint32_t* m, size_t rows, size_t cols, uint32_t add, cudaStream_t s);
// rows padded with zeros to rows3, then transposed (doublepir.rs:96-100)
void launch_dpir_pad_transpose(uint32_t* out, const uint32_t* a, size_t rows, size_t cols, size_t rows3, cudaStream_t s);

// ---- DoublePIR offline load (dpir_load.cu)
// AES-128 expanded on the host (FIPS-197): round keys as big-endian column words, the S-box and the T-table Te0
struct DpirAesKey { uint32_t rk[44]; uint32_t te0[256]; uint8_t sbox[256]; };
DpirAesKey dpir_aes_key(const uint8_t key[16]);
// Matrix::derive_from_seed (matrix.rs:125-135, derivation.rs:11-22): out[0 .. words) = the AES-128-Ctr64BE keystream, 64 KiB chunks
void launch_dpir_derive(uint32_t* out, size_t words, const DpirAesKey& key, cudaStream_t s);
// a synthetic matrix (b200pir_dpir_create_synthetic): a[i] = splitmix64(seed, i) & (2^30 - 1), three full 10-bit fields a word.
// Not counted in g_kernel_launches.
void launch_dpir_synth(uint32_t* a, size_t words, uint64_t seed, cudaStream_t s);
// Db::load_data (bits_format false) / load_data_fast (true), database.rs:168-247, for the band of layout rows [r0, r0 + rows):
// the band's words of the l x m matrix minus p/2 (every word written) into band (rows x m).  Of the `count` entries the
// iterator yields, `data` holds those from entry `base` on (entry i is at data[i - base], or at bit (i - base) % 8 of byte
// (i - base) / 8).  *out_of_range |= 1 when a word lies outside the setup GEMM's [-2^15, 2^15), |= 2 when a packed entry
// is wider than `bits` (b200pir_dpir_server_update can then not rebuild its element from the store)
void launch_dpir_layout(uint32_t* band, const uint8_t* data, uint64_t base, uint64_t count, bool bits_format, uint64_t r0,
                        uint64_t rows, uint64_t m, uint32_t packing, uint32_t bits, uint32_t ne, uint32_t p, int* out_of_range,
                        cudaStream_t s);

// ---- DoublePIR entry updates (dpir_update.cu): Db::_set on a loaded database, and setup()'s outputs patched to match
// One changed Z_p element of the l x m layout: new = (old & ~mask) | val, old read from its squished store field
struct DpirUpdElem { uint64_t r, c; uint32_t mask, val; };
// One changed layout row of a group: its elements are [e0, e0 + ne) of the group's element table.  Rows are ordered by block
// r % x, so row k of the table is column k of the group's digit-difference matrix D, and the rows of block b are columns
// [k0_b, k0_b + k_b); D_b (n delta x k_b, row-major) starts at word doff = n delta k0_b of D, and this row is its column dcol.
struct DpirUpdRow { uint64_t r, doff; uint32_t e0, ne, dcol, kb; };
// store patch: each element's field rewritten in the squished store (dcols words a row) and its change new - old to delta[]
void launch_dpir_upd_store(uint32_t* store, uint64_t dcols, const DpirUpdElem* el, uint32_t n_el, int32_t* delta, cudaStream_t s);
// dh1 (nrows x n) = sum over each row's elements of delta * A_1[c, :], the A_1 rows derived from `key` in the kernel
void launch_dpir_upd_dh1(uint32_t* dh1, const DpirUpdRow* rows, uint32_t nrows, const DpirUpdElem* el, const int32_t* delta, uint64_t n,
                         const DpirAesKey& key, cudaStream_t s);
// h_1's base-p digits in h1_squished (c1 words a row) moved by dh1, the digit differences written into D
void launch_dpir_upd_digits(uint32_t* h1sq, uint64_t c1, int32_t* D, const DpirUpdRow* rows, uint32_t nrows, const uint32_t* dh1,
                            uint64_t n, uint32_t p, uint32_t delta, uint64_t x, cudaStream_t s);
// a2g (nrows x n) = the rows A_2[r / x, :] of the changed rows, read from a_2^T (a2t: n x lx3)
void launch_dpir_upd_gather_a2(uint32_t* a2g, const uint32_t* a2t, uint64_t lx3, const DpirUpdRow* rows, uint32_t nrows, uint64_t n,
                               uint64_t x, cudaStream_t s);
// dst[i] += src[i], wrapping
void launch_dpir_upd_add(uint32_t* dst, const uint32_t* src, size_t words, cudaStream_t s);

}  // namespace b200pir
