/* b200pir — C ABI of the GPU-native (H100, sm_90a) server-side PIR query path.
 *
 * This is the drop-in boundary: every entry point replaces one Rust function of blyssprivacy/sdk
 * (reference @ fdb7206); the Rust host code keeps its own signature and forwards here through a thin
 * `extern "C"` shim (see INTEGRATION.md).  The reference has no FFI of its own, so the ABI flattens
 * the reference's argument types to plain pointers + sizes:
 *
 *   PolyMatrixRaw   rows x cols polys, each 2048 u64 coefficients            (lib/spiral-rs/src/poly.rs:59-64)
 *   PolyMatrixNTT   rows x cols polys, each [crt(2)][2048] u64 residues     (poly.rs:66-71, :263-265)
 *   db: &[u64]      [instance][trial][z][ii][j] words = q0-residue | q1-residue << 32   (server.rs:263-269)
 *   v_firstdim      [z][j][r] words, same packing                            (util.rs:343-350)
 *
 * All buffers are HOST memory owned by the caller unless the name says `_dev`.  Outputs are caller
 * allocated.  Nothing unwinds across the boundary: every function returns 0 on success or a negative
 * code (B200PIR_E_*), and b200pir_last_error() returns the message for the calling thread.
 * Concurrent calls on one context are serialised internally (one CUDA stream per context); use one
 * context per host thread / GPU for concurrency.
 */
#ifndef B200PIR_H
#define B200PIR_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200PIR_E_BADARG (-1)
#define B200PIR_E_SHAPE (-2)
#define B200PIR_E_CUDA (-3)
#define B200PIR_E_UNSUPPORTED (-4)

typedef struct b200pir_ctx b200pir_ctx;  /* params + tables + workspace on one GPU */
typedef struct b200pir_db b200pir_db;    /* HBM-resident database                   */
typedef struct b200pir_pp b200pir_pp;    /* HBM-resident PublicParameters of a client */
typedef struct b200pir_dpir b200pir_dpir; /* HBM-resident DoublePIR packed matrix    */

/* The scalar fields of spiral_rs::params::Params that params_from_json_obj reads
 * (lib/spiral-rs/src/util.rs:224-263); poly_len = 2048 and the two CRT moduli are fixed there (:246-247). */
typedef struct {
  uint64_t n, nu_1, nu_2, p, q2_bits, t_gsw, t_conv, t_exp_left, t_exp_right, instances, db_item_size, version;
  int32_t expand_queries; /* 0 = direct_upload */
} b200pir_params;

const char* b200pir_last_error(void);
int b200pir_device_count(void);

/* Params::init (params.rs:224-296): builds NTT tables, Barrett constants, v_neg1 on `device`. */
int b200pir_ctx_create(const b200pir_params* params, int device, b200pir_ctx** out);
void b200pir_ctx_destroy(b200pir_ctx* ctx);
/* Use an externally owned cudaStream_t for all work of this context from now on: a non-blocking stream of the caller's, or NULL
 * for the legacy default stream (torch's current stream unless one is set).  Waits for the work already queued on the old
 * stream, then destroys it if the context created it; the caller's stream must outlive the context or the next set_stream.
 * Every kernel launch and copy of the context, host entry points included, then goes to that stream; the _dev entry points
 * are ordered after whatever the caller queued there before the call. */
int b200pir_ctx_set_stream(b200pir_ctx* ctx, void* cuda_stream);
int b200pir_ctx_synchronize(b200pir_ctx* ctx);
/* knobs: "batch" (max queries per database pass: 1, 2, 4, 8 or 16;
 * the IMAD layout uses at most 4), "db_format" (layout of databases created afterwards: -1 = automatic (default): 2 wherever the
 * wgmma kernel supports the geometry, else 1; 0 = IMAD, 1 = mma.sync INT8 fragments, 2 = wgmma tile images, tc5_kernels.cu), "profile" (0 off, 1 per call,
 * 2 accumulate over calls until set again); "mul_variant", "fold_variant", "intt_variant", "imma_variant", "expand_variant",
 * "expand_pair_min_ctas" (accepted, no effect: one kernel, tiling or schedule each remains); "coalesce" (1 = default: concurrent single-query callers
 * share database passes, see b200pir_coalesce_stats), "coalesce_window_us" (default 200: how long a batch that directly
 * follows a multi-query batch is held open for the callers of that batch to return; 0 = never), "sparse_fold" (1 = fold like lib/server's sparse server,
 * compute/fold.rs:15-65: an all-zero ciphertext short-cuts the external product; 0 = spiral-rs's dense fold, default; version-1
 * servers set 1: with t_gsw = 7 the dense fold does not decode items whose row is folded against an empty one);
 * unknown keys -> B200PIR_E_BADARG */
int b200pir_ctx_set_option(b200pir_ctx* ctx, const char* key, int64_t value);
/* Size the context's workspace once, up front, for `queries` concurrent queries against a database with `rows_local`
 * second-dimension rows (num_per for an unsharded database): afterwards the query, expansion, first-dimension, fold, pack and
 * response buffers are not reallocated for batches up to that size (the workspace otherwise grows on first use; coalesced
 * single-query calls size it for 32 queries).  Three small buffers still grow on the first call with a larger batch than
 * before: the expansion rounds' scratch, the first dimension's query tile images and the per-query parameter table.
 * B200PIR_E_CUDA when the device cannot hold it. */
int b200pir_ctx_reserve(b200pir_ctx* ctx, size_t queries, size_t rows_local);
/* params.setup_bytes / query_bytes / response length (params.rs:146-182, server.rs:476-481) */
int b200pir_ctx_sizes(b200pir_ctx* ctx, uint64_t* setup_bytes, uint64_t* query_bytes, uint64_t* response_bytes);

/* ---- database: replaces the `db: &[u64]` argument of process_query (server.rs:650-655) ---------- */
/* Allocates slices*dim0*num_per*2048 words in HBM (zero = every item empty).
 * Multi-GPU row sharding (DESIGN.md): with shard_count = G (a power of two dividing num_per) this GPU holds
 * the second-dimension rows ii = shard_index (mod G); pass 0,1 for the whole database. */
int b200pir_db_create(b200pir_ctx* ctx, uint64_t shard_index, uint64_t shard_count, b200pir_db** out);
/* One database over several contexts, served and written from one process: shard g holds the rows ii = g (mod G) on ctxs[g],
 * laid out as b200pir_db_create(ctxs[g], g, G) lays them out, G = `shards` (a power of two dividing num_per).  The contexts must
 * be distinct and have identical parameters; their devices may differ or repeat (several shards on one device is valid).  The
 * layout is resolved once from ctxs[0]'s "db_format" and used for every shard.  G = 1 gives an ordinary database on ctxs[0].
 * The handle belongs to ctxs[0], the home context, and the member contexts must outlive it; b200pir_db_destroy frees each shard
 * on its own device.  Peer access is enabled between the home device and each other device where the hardware allows it.
 *
 * Queries (process_query, process_query_bytes, process_query_batch, process_queries, process_query_batch_dev), called with the
 * home context or any context b200pir_db_* accepts for it: the home context expands, each shard runs the first dimension and
 * the fold rounds nu_2-1 .. log2 G over its rows on its own context's stream (a shard on another device receives the operand by
 * copy engine), and the home context folds across the shards, packs and encodes.  Responses are byte for byte those of an
 * unsharded database with the same contents; "sparse_fold" is read from the calling context for every shard.  The _dev call
 * stays stream-ordered on the calling context's stream.  A call takes the calling context's lock and every member context's,
 * in creation order.  Workspace: the survivor and receive buffers belong to the database and are sized for 32 queries, growing
 * for a larger batch; b200pir_ctx_reserve(ctxs[g], Q, num_per / G) sizes each member's, and b200pir_ctx_reserve(ctxs[0], Q,
 * max(num_per / G, G)) the home's.
 * Writers (upload, upload_slice, load_file, load_raw_file, fill_synthetic, upsert_item, update_item_raw, update_many_items)
 * read their input once and give each shard its rows; a single-item write touches only the owning shard.  download,
 * download_slice and save_file assemble every shard's rows; present_items sums over the shards (capacity = the whole database);
 * db_info reports local_rows = num_per and hbm_bytes summed over the shards.
 * Refused with B200PIR_E_UNSUPPORTED: multiply_reg_by_database, query_stage_a_dev, first_dim_fold_dev and
 * first_dim_fold_images_dev (the multi-process building blocks take rank shards from b200pir_db_create).
 * Errors: null pointers, a repeated context or contexts with different parameters -> B200PIR_E_BADARG; a shard count that is not
 * a power of two dividing num_per -> B200PIR_E_BADARG as b200pir_db_create; no handle is returned and no device memory stays
 * allocated on any error. */
int b200pir_db_create_sharded(b200pir_ctx* const* ctxs, size_t shards, b200pir_db** out);
void b200pir_db_destroy(b200pir_db* db);
/* Upload one (instance,trial) slice in the reference layout [z][ii][j] (server.rs:263-266). */
int b200pir_db_upload_slice(b200pir_ctx* ctx, b200pir_db* db, uint64_t slice, const uint64_t* words, size_t n_words);
/* Whole db: &[u64] of instances*n^2 slices. */
int b200pir_db_upload(b200pir_ctx* ctx, b200pir_db* db, const uint64_t* words, size_t n_words);
/* load_preprocessed_db_from_file (server.rs:373-386; lib/server/src/db/loading.rs:263-276): `path` holds the native-endian
 * u64 stream of the whole database (slices*dim0*num_per*2048 words, the layout b200pir_db_upload takes); it is streamed
 * to the GPU through a staging buffer. */
int b200pir_db_load_file(b200pir_ctx* ctx, b200pir_db* db, const char* path);
/* load_db_from_seek (server.rs:277-357; lib/server/src/db/loading.rs:192-247): `path` is the RAW database, item i at byte
 * i*db_item_size; chunk c of an item = bytes_per_chunk bytes from i*db_item_size + c*bytes_per_chunk, clipped at the end of
 * the file; conversion (recenter, NTT, pack) on the GPU.  logp == 8 only. */
int b200pir_db_load_raw_file(b200pir_ctx* ctx, b200pir_db* db, const char* path);
/* One preprocessed item polynomial: 2048 packed words (lib/server/src/db/loading.rs:34-41 pack_ntt_poly,
 * :317-359 update_item_raw -> db.upsert(inst_trial*num_items + db_idx)); item_idx = j*num_per + ii. */
int b200pir_db_upsert_item(b200pir_ctx* ctx, b200pir_db* db, uint64_t slice, uint64_t item_idx, const uint64_t* poly);
/* lib/server/src/db/loading.rs:317-359 update_item_raw (the /write and /update-row path): `data` = the raw bucket bytes
 * of item db_idx (at most instances*n^2*bytes_per_chunk, zero padded); chunk c becomes the item polynomial of slice c
 * (convert_pt_to_poly :278-299: coefficient i = byte i, recenter_mod, NTT; pack_ntt_poly :34-41), all on the GPU. */
int b200pir_db_update_item_raw(b200pir_ctx* ctx, b200pir_db* db, uint64_t db_idx, const uint8_t* data, size_t len);
/* lib/server/src/db/loading.rs:361-377 update_many_items (the /update-row body): entries [u32 BE chunk_len][chunk_len bytes],
 * each chunk = [u32 BE db_idx][raw bucket bytes] as update_item (:301-315).  *largest_update = max chunk_len (written on
 * success; may be NULL).  The final database equals the reference's entry-by-entry loop: the entries before the first bad one
 * are applied, nothing from it on, and its code is returned (B200PIR_E_SHAPE for a header or chunk past the end of the body,
 * chunk_len < 4, chunk_len > 4 + instances*n^2*bytes_per_chunk or db_idx >= num_items; B200PIR_E_UNSUPPORTED for p != 256).
 * A db_idx written more than once ends with its last bytes.  On a shard every entry is checked and only its own rows are
 * written.  Conversion and placement run on the GPU; synchronises the context's stream before it returns. */
int b200pir_db_update_many_items(b200pir_ctx* ctx, b200pir_db* db, const uint8_t* body, size_t len, uint64_t* largest_update);
/* ---- reading the database back (the inverse of the loaders above) ----
 * Write slice `slice` in the reference layout [z][ii][j] (n_words = dim0*num_per*2048), the inverse of b200pir_db_upload_slice.
 * Only the words of the rows this database holds are written (ii = shard_index mod shard_count); the words of other shards'
 * rows are left untouched, so the G shards of a database downloading into one buffer assemble the whole slice.  Absent items
 * are zero words.  Round trip: a word whose halves are canonical residues (lo < q0, hi < q1), the only words any writer of this
 * library produces, comes back exactly as it was uploaded.  Format 0 stores both 32-bit halves verbatim and returns any
 * uploaded word unchanged; formats 1 and 2 store four 7-bit limbs per residue and return the low 28 bits of each half.
 * Read-only: the database, its presence map and b200pir_db_present_items are unchanged.  The context lock is held only while
 * one staging chunk (<= 64 MiB) is un-tiled and copied to pinned host memory, not while it is scattered into `words`, so
 * queries on the same context keep being served during an export; exports on one context run one at a time.  Consistency
 * with writers is the caller's: hold the read side of the lock that writers take exclusively (INTEGRATION.md §4).
 * Null pointers -> B200PIR_E_BADARG; wrong n_words or slice >= slices -> B200PIR_E_SHAPE. */
int b200pir_db_download_slice(b200pir_ctx* ctx, b200pir_db* db, uint64_t slice, uint64_t* words, size_t n_words);
/* Every slice: the `db: &[u64]` that b200pir_db_upload takes (n_words = slices*dim0*num_per*2048). */
int b200pir_db_download(b200pir_ctx* ctx, b200pir_db* db, uint64_t* words, size_t n_words);
/* Write the whole database to `path` as the native-endian u64 stream that b200pir_db_load_file and the reference's
 * load_preprocessed_db_from_file read.  Atomic: the words go to a temporary file in the same directory (mode 0600), which is
 * fsync'ed and renamed over `path`; if the save fails, an earlier file at `path` is intact and no temporary file is left.
 * Locking as b200pir_db_download.  Whole databases only, unsharded or from b200pir_db_create_sharded (whose chunks are
 * assembled on the host from every shard's export, one staging chunk at a time); a rank shard -> B200PIR_E_UNSUPPORTED; a file that cannot be created
 * or written -> B200PIR_E_BADARG, with the path in b200pir_last_error(). */
int b200pir_db_save_file(b200pir_ctx* ctx, b200pir_db* db, const char* path);
/* Bits of the per-item flags of b200pir_db_read_items */
#define B200PIR_ITEM_PRESENT 1u        /* the item is present (b200pir_db_present_items counts it) */
#define B200PIR_ITEM_NOT_PLAINTEXT 2u  /* some coefficient of some slice is not the image of a byte (e.g. after upsert_item of an
                                          arbitrary polynomial); it reads as 0 */
#define B200PIR_ITEM_PAST_CHUNK 4u     /* some coefficient at index >= bytes_per_chunk is a nonzero byte, which is not returned
                                          (fill_synthetic fills all 2048) */
/* The inverse of the raw writers (update_item_raw, update_many_items, load_raw_file): item db_idx[k] read back as bytes, on
 * the GPU.  Each slice's polynomial is inverse-transformed mod both CRT moduli and every coefficient decoded to the byte x whose
 * recenter_mod(x, 256, q) it is (convert_pt_to_poly, loading.rs:278-299).  out receives count x instances*n^2*bytes_per_chunk
 * bytes: chunk c of item k at k*span + c*bytes_per_chunk, which is the zero-padded bucket update_item_raw stores
 * (loading.rs:327-329).  flags[k] (flags may be NULL) gets the B200PIR_ITEM_* bits; an absent item reads as zero bytes with
 * flags 0.  count has no limit (the items are decoded in staging groups); on a sharded database each item is read from the
 * shard that holds it.  Read-only, locking as b200pir_db_download.
 * Errors, with nothing written: null pointers -> B200PIR_E_BADARG; db_idx >= num_items, or on a rank shard (b200pir_db_create
 * with shard_count > 1) an item whose row it does not hold -> B200PIR_E_SHAPE; p != 256 -> B200PIR_E_UNSUPPORTED;
 * bytes_per_chunk > 2048 -> B200PIR_E_SHAPE. */
int b200pir_db_read_items(b200pir_ctx* ctx, b200pir_db* db, const uint64_t* db_idx, size_t count, uint8_t* out, uint8_t* flags);
/* Write the raw database file that b200pir_db_load_raw_file and the reference's load_db_from_seek read: num_items x
 * db_item_size bytes, file byte o being byte o - i*db_item_size of item i = o / db_item_size (read as b200pir_db_read_items
 * does).  8 times smaller than b200pir_db_save_file's snapshot.  The raw format has no presence map: b200pir_db_load_raw_file
 * builds a dense database (every item present), so present_items and the tiles the wgmma pass skips differ from the source's,
 * while every response byte is the same.  Streamed in groups of whole items: the host writes one group while the GPU decodes
 * the next.  Atomic as b200pir_db_save_file; locking as b200pir_db_download.
 * Refused with B200PIR_E_UNSUPPORTED, `path` untouched and no temporary file left, when no raw file loads back to this
 * database: an item flagged NOT_PLAINTEXT or PAST_CHUNK, or, where instances*n^2*bytes_per_chunk > db_item_size, two
 * consecutive items that disagree on a byte they share in the file (the last item's bytes past the end must be zero);
 * b200pir_last_error() names the first such item.  A rank shard -> B200PIR_E_UNSUPPORTED; other errors as
 * b200pir_db_read_items and b200pir_db_save_file. */
int b200pir_db_save_raw_file(b200pir_ctx* ctx, b200pir_db* db, const char* path);
/* Synthetic database generated on the GPU: plaintext coefficient = splitmix64(seed, ((slice*items+item)*2048+z)) % p,
 * then recenter_mod / NTT / pack as generate_random_db_and_get_item does (server.rs:223-275). */
int b200pir_db_fill_synthetic(b200pir_ctx* ctx, b200pir_db* db, uint64_t seed);
/* What `db` is: its layout (the "db_format" it was created with, resolved when that was -1), the second-dimension rows
 * this GPU holds, and its size in HBM.  Any out pointer may be NULL. */
int b200pir_db_info(b200pir_db* db, int* format, uint64_t* local_rows, uint64_t* hbm_bytes);
/* lib/server's SparseDb (db/sparse_db.rs:5-47): an item exists once it has been written (upsert / update_item_raw; bulk uploads,
 * file loads and the synthetic fill write every item).  `items` = present items on this GPU, `capacity` = slices x local rows x
 * dim0.  Absent items are zero polynomials in HBM, so results equal the sparse server's sums; on the wgmma layout every
 * 32-row x 32-j tile without a present item is neither fetched nor multiplied (multiply_reg_by_sparse_database skips absent
 * items, compute/dot_product.rs:35). */
int b200pir_db_present_items(b200pir_db* db, uint64_t* items, uint64_t* capacity);

/* ---- public parameters: replaces &PublicParameters (client.rs:146-152), all matrices in NTT form ---- */
/* v_packing: num_packing x (n+1) x t_conv ; v_expansion_left: g x 2 x t_exp_left ;
 * v_expansion_right: (stop_round+1) x 2 x t_exp_right or NULL (-> left, server.rs:549) ; v_conversion: 2 x 2 t_conv.
 * Expansion / conversion may be NULL when expand_queries == 0. */
int b200pir_pp_create(b200pir_ctx* ctx, const uint64_t* v_packing, const uint64_t* v_expansion_left,
                      const uint64_t* v_expansion_right, const uint64_t* v_conversion, b200pir_pp** out);
/* PublicParameters::deserialize (client.rs:212-259): data = 32-byte seed || rows 1.. of every matrix (raw u64, native
 * endian) in the order v_packing, v_expansion_left, v_expansion_right (if present), v_conversion; len == setup_bytes.
 * The first rows are regenerated on the GPU from ChaCha20Rng::from_seed(seed) (rand_chacha 0.3.1 keystream order). */
int b200pir_pp_create_from_bytes(b200pir_ctx* ctx, const uint8_t* data, size_t len, b200pir_pp** out);
void b200pir_pp_destroy(b200pir_pp* pp);

/* ---- stage-level entry points (each == one reference function, host buffers) ----------------------- */
/* ntt.rs:67-113 ntt_forward / :212-258 ntt_inverse over `count` polys of [2][2048] u64, in place. */
int b200pir_ntt_forward(b200pir_ctx* ctx, uint64_t* polys, size_t count);
int b200pir_ntt_inverse(b200pir_ctx* ctx, uint64_t* polys, size_t count);
/* Device-resident batch (BASELINE config #5): `count` polys of u32 [2][2048] residues, in place, stream-ordered: enqueued on the
 * context's stream, nothing synchronised, nothing allocated (the tables of both sizes are built by b200pir_ctx_create). */
int b200pir_ntt32_dev(b200pir_ctx* ctx, uint32_t* polys_dev, size_t count, int inverse);
/* BASELINE config #5, poly_len = 4096 (not a size the reference's parameterisation uses, util.rs:246): the same transform
 * definition (ntt.rs:67-113, :212-258) and table construction (ntt.rs:39-65) over the same two moduli.
 * _dev: polys_dev = count x [2][4096] u32 on the device, in place; host variant: count x [2][4096] u64. */
int b200pir_ntt4096_dev(b200pir_ctx* ctx, uint32_t* polys_dev, size_t count, int inverse);
int b200pir_ntt4096(b200pir_ctx* ctx, uint64_t* polys, size_t count, int inverse);
/* poly.rs:613-623 to_ntt / :646-663 from_ntt over `count` polys. */
int b200pir_to_ntt(b200pir_ctx* ctx, uint64_t* out_ntt, const uint64_t* raw, size_t count);
int b200pir_from_ntt(b200pir_ctx* ctx, uint64_t* out_raw, const uint64_t* ntt, size_t count);
/* server.rs:155-221 multiply_reg_by_database on slice `slice`: out = num_per x PolyMatrixNTT(2,1). */
int b200pir_multiply_reg_by_database(b200pir_ctx* ctx, b200pir_db* db, uint64_t slice, const uint64_t* v_firstdim,
                                     uint64_t* out);
/* server.rs:388-427 fold_ciphertexts: v_cts = num x PolyMatrixRaw(2,1) in place (result in v_cts[0]);
 * v_folding / v_folding_neg = log2(num) x PolyMatrixNTT(2, 2 t_gsw).  v_folding_neg may be NULL, meaning
 * get_v_folding_neg(v_folding) as process_query always passes (server.rs:680): the library then uses its
 * fast path, which never materialises the negated matrices (same bytes). */
int b200pir_fold_ciphertexts(b200pir_ctx* ctx, uint64_t* v_cts, size_t num, const uint64_t* v_folding,
                             const uint64_t* v_folding_neg);
/* server.rs:505-523 get_v_folding_neg */
int b200pir_get_v_folding_neg(b200pir_ctx* ctx, uint64_t* out, const uint64_t* v_folding);
/* server.rs:19-121 coefficient_expansion over v = 2^g x PolyMatrixNTT(2,1), in place */
int b200pir_coefficient_expansion(b200pir_ctx* ctx, b200pir_pp* pp, uint64_t* v);
/* server.rs:525-591 expand_query: query ct (PolyMatrixRaw 2x1) -> v_firstdim [z][j][r], v_folding nu_2 x (2 x 2 t_gsw) */
int b200pir_expand_query(b200pir_ctx* ctx, b200pir_pp* pp, const uint64_t* query_ct, uint64_t* out_v_firstdim,
                         uint64_t* out_v_folding);
/* server.rs:429-468 pack (version 0) / lib/server/src/compute/pack.rs:45-98 (version 1):
 * v_ct = n*n x PolyMatrixRaw(2,1) of one instance -> PolyMatrixNTT(n+1, n) */
int b200pir_pack(b200pir_ctx* ctx, b200pir_pp* pp, const uint64_t* v_ct, uint64_t* out_ntt);
/* server.rs:470-503 encode: instances x PolyMatrixRaw(n+1, n) -> response bytes */
int b200pir_encode(b200pir_ctx* ctx, const uint64_t* v_packed_raw, uint8_t* out, size_t* out_len);

/* ---- the drop-in: spiral_rs::server::process_query (server.rs:650-741) ------------------------------- */
/* expand_queries != 0: query_ct = Query.ct (PolyMatrixRaw 2x1), v_buf = v_ct = NULL.
 * expand_queries == 0: query_ct = NULL, v_buf = Query.v_buf ([z][j][r]), v_ct = nu_2 x PolyMatrixRaw(2, 2 t_gsw).
 * out: response_bytes bytes. */
int b200pir_process_query(b200pir_ctx* ctx, b200pir_db* db, b200pir_pp* pp, const uint64_t* query_ct,
                          const uint64_t* v_buf, const uint64_t* v_ct, uint8_t* out, size_t* out_len);
/* Query::deserialize (client.rs:303-315, expand_queries only): data = seed || row 1 of ct; query_ct: PolyMatrixRaw(2,1). */
int b200pir_query_from_bytes(b200pir_ctx* ctx, const uint8_t* data, size_t len, uint64_t* query_ct);
/* process_query on `count` serialized queries (count x query_bytes, back to back); out: count x response_bytes.
 * Replaces Query::deserialize + process_query as lib/server's /private-read handler chains them (bin/server.rs:99-141).
 * Both branches of Query::deserialize (client.rs:303-329): expand_queries != 0 -> seed || row 1 of ct;
 * expand_queries == 0 (direct upload) -> seed || the odd-indexed words of v_buf || rows 1 of the nu_2 v_ct matrices, the
 * seed-derived halves being regenerated on the GPU.  (In direct-upload mode the handler's body is setup || query: pass the
 * first setup_bytes to b200pir_pp_create_from_bytes and the rest here.) */
int b200pir_process_query_bytes(b200pir_ctx* ctx, b200pir_db* db, b200pir_pp* pp, const uint8_t* queries, size_t len,
                                size_t count, uint8_t* out, size_t* out_len_each);
/* `count` queries of DIFFERENT clients in one database pass: pps[i] = the public parameters of the client that sent query_cts[i]
 * (host PolyMatrixRaw(2,1) each; expand_queries only); outs[i] receives response_bytes bytes.  lib/server looks the parameters up
 * per request (bin/server.rs:113-117); the kernels take them per query. */
int b200pir_process_queries(b200pir_ctx* ctx, b200pir_db* db, b200pir_pp* const* pps, const uint64_t* const* query_cts,
                            size_t count, uint8_t* const* outs);
/* Concurrent callers: b200pir_process_query and single-query b200pir_process_query_bytes calls on one context are coalesced —
 * requests that arrive while a batch is running are served together (up to 32) in one database pass by the next caller to
 * find the GPU free; a lone caller is served at once.  Option "coalesce" = 0 restores strictly serial calls.  Counters: */
int b200pir_coalesce_stats(b200pir_ctx* ctx, uint64_t* batches, uint64_t* queries);
/* `count` queries of one client in one call; the database is streamed once per group of up to 4 (IMAD layout)
 * or 16 (INT8 tensor-core layout) queries.
 * queries: count x PolyMatrixRaw(2,1); out: count x response_bytes. */
int b200pir_process_query_batch(b200pir_ctx* ctx, b200pir_db* db, b200pir_pp* pp, const uint64_t* query_cts,
                                size_t count, uint8_t* out, size_t* out_len_each);
/* Device-resident variants for measurement and multi-GPU composition: inputs/outputs are DEVICE pointers
 * and nothing is synchronised (stream-ordered): the call reads its inputs and writes its outputs in the order of the context's
 * stream (b200pir_ctx_set_stream) and returns without waiting for that stream or the legacy default stream, so the caller
 * may queue the input copies before the call and the output copies after it, on the same stream.  The same holds for the
 * three-phase and stage _dev entry points below.  What may still block the host on first use: growing a workspace buffer
 * (cudaFree of the smaller one waits for the whole device) on the first call with a larger batch than the context has served
 * or reserved (b200pir_ctx_reserve, which lists the buffers it does not size), and a per-query parameter table whose contents
 * changed (a different pp or count than the previous call: a small pageable copy, which the driver may stage synchronously).
 * A warmed call, same pp and count as the previous one, does neither.
 * query_dev: count x PolyMatrixRaw(2,1) (u64); out_dev: count x response_bytes. */
int b200pir_process_query_batch_dev(b200pir_ctx* ctx, b200pir_db* db, b200pir_pp* pp, const uint64_t* query_cts_dev,
                                    size_t count, uint8_t* out_dev);
/* Multi-GPU row sharding (DESIGN.md "multi-GPU"): stage A = expansion + first dimension + local fold rounds
 * on this GPU's rows; writes this rank's surviving ciphertexts to `partial_dev` as count x slices ciphertexts
 * in residue form (u32 [row(2)][crt(2)][2048] = coefficients mod q0 / q1, 32 KiB each).  Stage B = remaining
 * log2(world) fold rounds + pack + encode over the all-gathered `gathered_dev` ([world][count][slices][2][2][2048]). */
int b200pir_query_stage_a_dev(b200pir_ctx* ctx, b200pir_db* db, b200pir_pp* pp, const uint64_t* query_cts_dev,
                              size_t count, uint32_t* partial_dev);
int b200pir_query_stage_b_dev(b200pir_ctx* ctx, b200pir_pp* pp, const uint32_t* gathered_dev, size_t world,
                              size_t count, uint8_t* out_dev);

/* The same three phases with caller-owned device buffers in between (so a collective can sit between them):
 *   expand:  count queries -> q_expanded_dev (count x dim0 x 2048 x 16 B, the first-dimension operand) and
 *            v_folding_dev (count x nu_2 x 2 x 2 t_gsw x 2 x 2048 u32, NTT form)
 *   first_dim_fold: any `count` expanded queries against this GPU's rows -> partial_dev (count x slices residue-form cts)
 *   finish:  queries [first, first+count) of gathered_dev ([world][total_count][slices][ct]) -> responses; v_folding_dev holds
 *            the folding matrices of exactly those `count` queries. */
int b200pir_expand_queries_dev(b200pir_ctx* ctx, b200pir_pp* pp, const uint64_t* query_cts_dev, size_t count,
                               void* q_expanded_dev, uint32_t* v_folding_dev);
int b200pir_first_dim_fold_dev(b200pir_ctx* ctx, b200pir_db* db, const void* q_expanded_dev, const uint32_t* v_folding_dev,
                               size_t count, uint32_t* partial_dev);
/* The first two phases with the first-dimension operand exchanged as wgmma operand tile images (format-2 databases): the rank that
 * expands a group of <= 16 queries also re-tiles it, once (fused with reorient_reg_ciphertexts, util.rs:323-355); the receivers
 * multiply straight from the images.  image_dev: b200pir_query_image_bytes(ctx) bytes per group; partial_dev as above with
 * query index = group * per_group + i. */
size_t b200pir_query_image_bytes(b200pir_ctx* ctx);
int b200pir_expand_queries_images_dev(b200pir_ctx* ctx, b200pir_pp* pp, const uint64_t* query_cts_dev, size_t count, void* image_dev,
                                      uint32_t* v_folding_dev);
int b200pir_first_dim_fold_images_dev(b200pir_ctx* ctx, b200pir_db* db, const void* images_dev, size_t groups, size_t per_group,
                                      const uint32_t* v_folding_dev, uint32_t* partial_dev);
int b200pir_finish_queries_dev(b200pir_ctx* ctx, b200pir_pp* pp, const uint32_t* gathered_dev, size_t world,
                               size_t total_count, size_t first, size_t count, const uint32_t* v_folding_dev,
                               uint8_t* out_dev);

/* Per-stage device time of the last profiled call, in milliseconds, measured with CUDA events on the
 * context's stream.  Enable with b200pir_ctx_set_option(ctx, "profile", 1).
 * out[0..8] = expand, first-dim multiply kernel, from_ntt, fold, pack, encode, total, multiply launches, re-tiling of the query
 * operand for the tensor-core first dimension (k_query_to_tc5 / k_query_to_frag) */
int b200pir_last_stage_ms(b200pir_ctx* ctx, double* out9);
/* ---- peer memory for the multi-GPU exchange (one process per GPU, NVLink) ------------------------------------------------
 * The expanded queries every rank needs (24 MiB per query) are PUSHED into the peers' gather buffers by the copy engines
 * (cudaMemcpyAsync over CUDA-IPC mappings), not all-gathered by SM-resident collective kernels that compete with the
 * compute kernels for SMs.  b200pir_peer_alloc: device buffer + the 64-byte IPC handle to hand to the other ranks (any
 * transport); b200pir_peer_open: map a peer's buffer (handle from ANOTHER process) for access from `device`;
 * b200pir_peer_copy_async: stream-ordered copy between any two device pointers (local or mapped). */
int b200pir_peer_alloc(int device, size_t bytes, void** out_ptr, uint8_t out_handle[64]);
int b200pir_peer_open(int device, const uint8_t handle[64], void** out_ptr);
int b200pir_peer_close(int device, void* mapped_ptr);
int b200pir_peer_free(int device, void* ptr);
int b200pir_peer_copy_async(void* dst, const void* src, size_t bytes, void* cuda_stream);
/* Number of CUDA kernels this library has launched from the calling host thread since load. */
unsigned long long b200pir_kernel_launches(void);

/* ---- DoublePIR: matrix_mul_vec_packed(a, b, basis=10, compression=3) (lib/doublepir/src/matrix/kernels.rs:118-178) */
int b200pir_dpir_create(int device, const uint32_t* a, uint64_t rows, uint64_t cols, b200pir_dpir** out);
/* synthetic a: word(i,k) = low 30 bits of splitmix64(seed, i*cols+k) */
int b200pir_dpir_create_synthetic(int device, uint64_t rows, uint64_t cols, uint64_t seed, b200pir_dpir** out);
/* Offline setup (lib/doublepir/src/doublepir/doublepir.rs:76-108): h_1 = db.data * a_1 and h_2 = h_1' * a_2 as exact 8-bit limb
 * products on the tensor cores (wgmma) (small signed left operand x 32-bit right operand, modulo 2^32), transpose / expand /
 * concat_cols / squish as small kernels.  Host pointers.  db: l x m, entries centred in [-p/2, p/2) as wrapping u32, p <= 2^10;
 * a1: m x n; a2: (l/x) x n; delta = params.delta(), x = db.info.x.  Outputs: db_squished l x ceil(m/3); h1_squished
 * (n delta x) x ceil((l/x)/3); a2_t n x ((l/x) rounded up to a multiple of 3); h2 (n delta x) x n. */
int b200pir_dpir_setup(int device, const uint32_t* db, uint64_t l, uint64_t m, const uint32_t* a1, uint64_t n, const uint32_t* a2,
                       uint32_t p, uint64_t delta, uint64_t x, uint32_t* db_squished, uint32_t* h1_squished, uint32_t* a2_t,
                       uint32_t* h2);
/* `&Matrix * &Matrix` (matrix/ops.rs:169-191) on the same kernel: out (a_rows x b_cols) = a * b mod 2^32, entries of a in [-2^15, 2^15). */
int b200pir_dpir_matmul(int device, const uint32_t* a, uint64_t a_rows, uint64_t a_cols, const uint32_t* b, uint64_t b_cols,
                        uint32_t* out);
void b200pir_dpir_destroy(b200pir_dpir* m);
int b200pir_dpir_set_stream(b200pir_dpir* m, void* cuda_stream);
/* b: 3*cols u32 ; out: rows u32 */
int b200pir_dpir_matvec_packed(b200pir_dpir* m, const uint32_t* b, uint32_t* out);
/* _dev: device pointers, on the handle's stream.  `variant` is accepted and has no effect: one kernel per shape remains. */
int b200pir_dpir_matvec_packed_dev(b200pir_dpir* m, const uint32_t* b_dev, uint32_t* out_dev, int variant);
/* same over the row range [row_begin, row_begin+row_count): answer()'s `db.rows(start, batch)` (doublepir.rs:301) */
int b200pir_dpir_matvec_packed_rows(b200pir_dpir* m, uint64_t row_begin, uint64_t row_count, const uint32_t* b, uint32_t* out);
/* The small tail of answer() (doublepir.rs:317-349), host buffers:
 * matrix_mul_transposed_packed (kernels.rs:180-278): out (a_rows x b_rows); b_cols must be 3*a_cols.
 * transpose_expand_concat_cols_squish (matrix/indexing.rs:117-143, basis 10, d 3): out (cols*delta*concat) x ceil((rows/concat)/3). */
int b200pir_dpir_matrix_mul_transposed_packed(int device, const uint32_t* a, uint64_t a_rows, uint64_t a_cols, const uint32_t* b,
                                              uint64_t b_rows, uint64_t b_cols, uint32_t* out);
int b200pir_dpir_transpose_expand_concat_cols_squish(int device, const uint32_t* a, uint64_t rows, uint64_t cols, uint64_t modulus,
                                                     uint64_t delta, uint64_t concat, uint32_t* out, uint64_t* out_rows,
                                                     uint64_t* out_cols);

/* ---- DoublePIR offline load: raw entries -> database layout -> init() -> setup(), all in HBM ----------------------------- */
/* Params {n, l, m, logq, p} as pick_params returned them (lib/doublepir/src/params/params.rs:5-15; sigma is not used here). */
typedef struct {
  uint64_t n, l, m, logq, p;
} b200pir_dpir_params;
/* DbInfo fields the layout depends on, plus Params::delta() (params.rs:21-23): packing = entries per Z_p element (0 when an
 * entry takes several), ne = Z_p elements per entry, x (= ne: DbInfo::new's search starts at ne), delta = base-p digits of a
 * 32-bit value. */
typedef struct {
  uint64_t packing, ne, x, delta;
} b200pir_dpir_info;
/* Keys of the two shared matrices (lib/doublepir/src/util/consts.rs:23-33): the first 16 bytes of SHA-256("blyss1") and of
 * SHA-256("blyss2").  A_1 = derive(m x n, key 1), A_2 = derive((l/x) x n, key 2) (init(), doublepir.rs:46-51). */
#define B200PIR_DPIR_SEED_A1 {0x9c, 0x22, 0x77, 0x85, 0x45, 0xac, 0x22, 0x97, 0x41, 0x90, 0x8e, 0x65, 0x2d, 0x33, 0x3a, 0x0f}
#define B200PIR_DPIR_SEED_A2 {0x5f, 0xff, 0xc4, 0x82, 0xc7, 0x2a, 0x85, 0x4a, 0x10, 0x35, 0x9e, 0x9f, 0xa2, 0xf5, 0xe0, 0x7f}
/* Entry formats of b200pir_dpir_load: one entry per byte (Db::load_data's Iterator<Item = u8>, database.rs:168-205), or eight
 * entries per byte, least significant bit first (Db::load_data_fast's bits_from_byte, database.rs:1-19, :207-247). */
#define B200PIR_DPIR_ENTRY_BYTES 0
#define B200PIR_DPIR_ENTRY_BITS 1
/* DbInfo::new (lib/doublepir/src/database/database.rs:58-90, num_db_entries :352-372, with f64 log2 / ceil as written) plus
 * Params::delta().  Host only.  Zero entries or bits_per_entry outside [1, 63], null pointers or a zero n / l / m ->
 * B200PIR_E_BADARG; logq != 32 or p outside [2, 1024] (the squish basis is 10 bits, database.rs:274) -> B200PIR_E_UNSUPPORTED;
 * more Z_p elements than l * m (the reference's `assert!(db_elems <= params.l * params.m)`) -> B200PIR_E_SHAPE. */
int b200pir_dpir_db_info(const b200pir_dpir_params* params, uint64_t num_entries, uint64_t bits_per_entry, b200pir_dpir_info* out);
/* Matrix::derive_from_seed(rows, cols, key) (matrix/matrix.rs:125-135, derive_with_aes matrix/derivation.rs:11-22) on the GPU,
 * into the host buffer out (rows * cols u32): the AES-128 keystream in Ctr64BE mode, restarted every 64 KiB with
 * IV = BE64(chunk index) || 0^8, read as little-endian u32 words. */
int b200pir_dpir_derive_from_seed(int device, const uint8_t key[16], uint64_t rows, uint64_t cols, uint32_t* out);
/* DoublePirServer::new + load_data / load_data_fast (doublepir/server.rs:160-165, 201-229): db_info as above, A_1 and A_2 derived
 * on the device from the two keys above, the `len` bytes of `data` laid out as the l x m matrix (database.rs:168-247; BITS gives
 * 8 len entries, including the trailing bits of the last byte), then setup() (doublepir.rs:76-108) as b200pir_dpir_setup.  The
 * squished database stays in HBM: *db_out is a new handle of l x ceil(m/3) packed words for the matvec entry points.
 * h1_squished, a2_t and h2 are host buffers shaped as b200pir_dpir_setup's.  Synchronous, on a non-blocking stream of its own.
 * The l x m layout is never held whole: the rows are laid out and multiplied band by band (b200pir_dpir_load_banded with the
 * default scratch budget), so the device holds the squished store, setup()'s n-wide buffers and one band of scratch.
 * Errors (no handle is returned and no device memory stays allocated): those of b200pir_dpir_db_info; null pointers, a bad
 * device or an unknown entry_format -> B200PIR_E_BADARG; entries that would index past the l x m matrix (where the reference
 * panics), or l not a multiple of x -> B200PIR_E_SHAPE; a laid-out word outside [-2^15, 2^15) (bytes far wider than
 * bits_per_entry packed together; the setup GEMM's operand range) -> B200PIR_E_UNSUPPORTED. */
int b200pir_dpir_load(int device, const b200pir_dpir_params* params, uint64_t num_entries, uint64_t bits_per_entry,
                      const uint8_t* data, uint64_t len, int entry_format, b200pir_dpir** db_out, uint32_t* h1_squished,
                      uint32_t* a2_t, uint32_t* h2);
/* b200pir_dpir_load with a budget of scratch_bytes bytes of device scratch for a band of layout rows (0: 1 GiB).  The band is
 * the largest whole number of row groups (ne rows when entries take several Z_p elements, else 1 row) whose
 * b200pir_dpir_band_bytes fit the budget, and at least one group.  The input is staged through two pinned host buffers of at
 * most 16 MiB, so that copying the next band's bytes overlaps the current band's kernels.  Outputs and errors as
 * b200pir_dpir_load; they do not depend on the budget. */
int b200pir_dpir_load_banded(int device, const b200pir_dpir_params* params, uint64_t num_entries, uint64_t bits_per_entry,
                             const uint8_t* data, uint64_t len, int entry_format, uint64_t scratch_bytes, b200pir_dpir** db_out,
                             uint32_t* h1_squished, uint32_t* a2_t, uint32_t* h2);
/* b200pir_dpir_load_banded with the raw bytes read from the file at `path` band by band (pread into the pinned staging), as
 * Db::load_data_fast reads a file without holding it: `len` is the file's size.  Errors as b200pir_dpir_load, and: a file that
 * cannot be opened -> B200PIR_E_BADARG; a read that fails or comes up short (a directory, a file truncated while it loads)
 * -> B200PIR_E_SHAPE. */
int b200pir_dpir_load_file(int device, const b200pir_dpir_params* params, uint64_t num_entries, uint64_t bits_per_entry,
                           const char* path, int entry_format, uint64_t scratch_bytes, b200pir_dpir** db_out, uint32_t* h1_squished,
                           uint32_t* a2_t, uint32_t* h2);
/* The device scratch a band of `rows` layout rows takes: 4 rows m (its centred words) + the GEMM operand image of the band
 * (2 bytes a word, rows rounded up to 128 and m to 32) + the input bytes it can span (rows m packing entries, or rows / ne
 * m entries when packing = 0; one byte each, or one bit each plus one byte).  Host only.  rows not a positive multiple of the
 * group, or more than l -> B200PIR_E_SHAPE. */
int b200pir_dpir_band_bytes(const b200pir_dpir_params* params, uint64_t num_entries, uint64_t bits_per_entry, int entry_format,
                            uint64_t rows, uint64_t* out);
/* Reads a packed matrix back (rows * cols u32): the squished database server.rs:147-153 writes as `.dbp`. */
int b200pir_dpir_download(b200pir_dpir* m, uint32_t* out);

/* ---- DoublePIR online: answer() served from HBM ---------------------------------------------------------------------------- */
typedef struct b200pir_dpir_server b200pir_dpir_server;
/* matrix_mul_vec_packed (kernels.rs:118-178) for `count` vectors: b = count x 3*cols u32, out = count x rows u32, host buffers,
 * on the handle's stream.  The matrix is read once per pass of up to 64 vectors on the tensor cores, or of up to 16 on the
 * integer kernel; the kernel is chosen as the answer path chooses it.  Null pointers -> B200PIR_E_BADARG. */
int b200pir_dpir_matvec_packed_many(b200pir_dpir* m, const uint32_t* b, size_t count, uint32_t* out);
/* The same on a named kernel, for tests and measurements: B200PIR_DPIR_MV_AUTO (as above), B200PIR_DPIR_MV_MULTI (the integer
 * kernel, 16 vectors a pass) or B200PIR_DPIR_MV_TC (the tensor cores, 64 vectors a pass).  Results do not depend on the kernel.
 * Another value -> B200PIR_E_BADARG. */
#define B200PIR_DPIR_MV_AUTO 0
#define B200PIR_DPIR_MV_MULTI 1
#define B200PIR_DPIR_MV_TC 2
int b200pir_dpir_matvec_packed_many_on(b200pir_dpir* m, const uint32_t* b, size_t count, uint32_t* out, int kernel);
/* The state DoublePirServer::answer reads (doublepir/server.rs:201-247): `db` (borrowed: the handle of b200pir_dpir_load, or
 * b200pir_dpir_create of a `.dbp`, or of one chunk's rows for a chunked server; it must outlive the server) plus server_state =
 * [h_1, a_2^T] (doublepir.rs:104-106) as b200pir_dpir_load / b200pir_dpir_setup return them, uploaded once: h1_squished
 * (n delta x) x ceil((l/x)/3), a2_t n x 3 ceil((l/x)/3).  p, delta, x and ne come from b200pir_dpir_db_info(params, num_entries,
 * bits_per_entry).  The server owns a non-blocking stream, a mutex that serialises its calls, and a workspace for max_queries
 * queries per call (the total over all requests of an answer_many).  Errors: those of b200pir_dpir_db_info (which here also takes
 * bits_per_entry = 64: the server lays out no entries); null pointers, a bad
 * device or max_queries == 0 -> B200PIR_E_BADARG; db with cols != ceil(m/3) or more than l rows, or l not a multiple of x ->
 * B200PIR_E_SHAPE. */
int b200pir_dpir_server_create(int device, const b200pir_dpir_params* params, uint64_t num_entries, uint64_t bits_per_entry,
                               b200pir_dpir* db, const uint32_t* h1_squished, const uint32_t* a2_t, size_t max_queries,
                               b200pir_dpir_server** out);
void b200pir_dpir_server_destroy(b200pir_dpir_server* s);
/* The response length of `request` (Vec<State>::serialize(), serializer.rs): 4 + 8 + 4 delta x n + queries * ne/x * (16 +
 * 4 (n delta x) + 4 delta x).  Checks the framing and the q_2 shapes (the checks that do not depend on the chunk). */
int b200pir_dpir_answer_size(b200pir_dpir_server* s, const uint8_t* request, size_t len, size_t* out_len);
/* DoublePirServer::answer (server.rs:235-247) when chunk_idx < 0; answer_inline(request, data, Some(chunk_idx))
 * (server.rs:167-180) when chunk_idx >= 0, the server's matrix being `data`: batch chunk_idx's rows are rows [0, batch size) of
 * it (doublepir.rs:270-279) and the other batches contribute zero rows.  out receives msg.serialize(); *out_len is its capacity
 * on entry and the response length on return.  Row batches, message order and byte order are answer()'s and serializer.rs's.
 * Where the reference panics, B200PIR_E_SHAPE and nothing is written: a header or data word past the end, a count, rows or
 * cols >= 2^28, zero queries, a query with fewer than 1 + ne/x matrices, a q_1 / q_2 whose rows are not 3 x the packed columns
 * or whose cols != 1, a chunk index >= the query count, a batch needing more rows than the server holds (an unchunked answer
 * needs all l).  More than max_queries queries -> B200PIR_E_SHAPE (the limit in b200pir_last_error()); null pointers or
 * *out_len below the response length -> B200PIR_E_BADARG.  Matrices past the first 1 + ne/x of a query and trailing bytes are
 * ignored, as deserialize_iter ignores them.  The server stays usable after any error. */
int b200pir_dpir_answer(b200pir_dpir_server* s, const uint8_t* request, size_t len, int64_t chunk_idx, uint8_t* out,
                        size_t* out_len);
/* `count` independent requests of different clients, unchunked, in one call: response i is byte for byte answer(requests[i]);
 * the database is read once per pass of up to 64 requests and h_1 once per 64 q_2 vectors of the call, on the tensor cores;
 * a pass of 8 or fewer vectors runs on the integer kernel, 16 a pass (DESIGN §4.5).  out_lens[i]: capacity
 * of outs[i] on entry, response length on return.  Errors as b200pir_dpir_answer (the query limit counts every request); on an
 * error nothing is written to any output. */
int b200pir_dpir_answer_many(b200pir_dpir_server* s, const uint8_t* const* requests, const size_t* lens, size_t count,
                             uint8_t* const* outs, size_t* out_lens);
/* Db::_set for `count` entries (database.rs:264-266, a todo!() in the reference), on the database this server borrows, and
 * setup()'s outputs patched to match: afterwards the squished store (b200pir_dpir_download), the server's h_1
 * (b200pir_dpir_server_state) and h2 are byte for byte what b200pir_dpir_load* returns for the same bytes with those entries
 * replaced.  values[k] = entry indices[k] as the load read it: a byte (ENTRY_BYTES) or a bit 0/1 (ENTRY_BITS).  A repeated
 * index ends with its last value.  h2: (n delta x) x n host matrix in/out, the hint as the load or the previous update left it.
 * The cost grows with the number of changed entries, not with the database (DESIGN §4.5): the changed store fields are
 * rewritten, only the rows of A_1 at changed columns are derived, and the hint moves by a rank-k product on the setup GEMM.
 * count = 0 succeeds and changes nothing.  Everything is checked before any device work, and a refused call writes nothing
 * (store, h_1 and h2 stay as they were, and the server keeps serving): null pointers -> B200PIR_E_BADARG; an index at or past
 * the entries the load read (len, or 8 len bits) -> B200PIR_E_SHAPE; a value the format cannot hold (above 1 for bits, or
 * 2^bits_per_entry or more where entries are packed several to an element) -> B200PIR_E_BADARG; a server whose parameters,
 * num_entries or bits_per_entry differ from its database's load -> B200PIR_E_SHAPE; a database not made by b200pir_dpir_load*
 * (b200pir_dpir_create of a `.dbp`, say), a server holding fewer than l rows (a chunk), or a load that packed entries wider
 * than bits_per_entry (its elements then do not decode field by field), or n above 51200 -> B200PIR_E_UNSUPPORTED.
 * Holds the server's and the database handle's mutexes, so an answer sees all of an update or none of it; runs on the
 * server's stream and synchronises.  Scratch belongs to the server: allocated by the first update, grown only by a larger
 * batch.  Large batches are applied in groups of 4096 changed elements; the results do not depend on the grouping.  Other
 * servers that borrow the same database handle keep their own h_1, which goes stale. */
int b200pir_dpir_server_update(b200pir_dpir_server* s, const uint64_t* indices, const uint8_t* values, size_t count, uint32_t* h2);
/* server_state[0] as the server now holds it: h1_squished, (n delta x) x ceil((l/x)/3) u32 (what save_to_files writes as
 * .state).  Null pointers -> B200PIR_E_BADARG. */
int b200pir_dpir_server_state(b200pir_dpir_server* s, uint32_t* h1_squished);

/* ---- DoublePIR over several GPUs: a database split by rows, driven by one process (DESIGN §4.5) ----------------------------
 * The split rule: the l layout rows fall into U = ceil(l / 3x) units of 3x rows (x from the DbInfo shape), the last one
 * clipped at l, and shard g of G takes the next floor(U / G) units, one more when g < U mod G.  Every contraction of setup()
 * and answer() that crosses rows is a wrapping u32 sum over l/x, and edges on multiples of 3x keep each packed column of h_1,
 * a_1' and a_2^T inside one shard, so the sum of the shards' partials mod 2^32 is bit for bit the one-GPU result.
 * Shard `index` of `shards`: its first row and row count.  Host only.  Errors: those of the db info (bits_per_entry up to 64);
 * l not a multiple of x, shards == 0, or more shards than units -> B200PIR_E_SHAPE; null pointers or index >= shards ->
 * B200PIR_E_BADARG. */
int b200pir_dpir_shard_rows(const b200pir_dpir_params* params, uint64_t num_entries, uint64_t bits_per_entry, size_t shards,
                            size_t index, uint64_t* row_begin, uint64_t* rows);
/* The load of b200pir_dpir_load_banded, split into `shards` row shards by the rule above: dbs_out[g] is a handle on devices[g]
 * holding the squished store rows of shard g (a device may appear more than once).  h1_squished, a2_t and h2 are the whole host
 * matrices, byte for byte b200pir_dpir_load_banded's.  Distinct devices load at once, one host thread each; shards that share a
 * device load one after another.  scratch_bytes bounds each shard's band scratch.  Errors as b200pir_dpir_load_banded, and a
 * shard count the rule refuses -> B200PIR_E_SHAPE; on any error no handle is returned and no device memory stays allocated. */
int b200pir_dpir_load_sharded(const int* devices, size_t shards, const b200pir_dpir_params* params, uint64_t num_entries,
                              uint64_t bits_per_entry, const uint8_t* data, uint64_t len, int entry_format, uint64_t scratch_bytes,
                              b200pir_dpir** dbs_out, uint32_t* h1_squished, uint32_t* a2_t, uint32_t* h2);
/* The same with the raw bytes read from the file at `path` (pread, each shard its own byte range); errors as
 * b200pir_dpir_load_file. */
int b200pir_dpir_load_file_sharded(const int* devices, size_t shards, const b200pir_dpir_params* params, uint64_t num_entries,
                                   uint64_t bits_per_entry, const char* path, int entry_format, uint64_t scratch_bytes,
                                   b200pir_dpir** dbs_out, uint32_t* h1_squished, uint32_t* a2_t, uint32_t* h2);
/* A shard from host words: rows x cols packed words that are the layout rows [row_begin, row_begin + rows) of a database (rows
 * of a saved `.dbp`, say).  Errors as b200pir_dpir_create. */
int b200pir_dpir_create_shard(int device, const uint32_t* a, uint64_t row_begin, uint64_t rows, uint64_t cols, b200pir_dpir** out);
/* What a handle holds: its first layout row (0 for the handles of the unsharded creators and loads), rows, packed columns and
 * device.  Null pointers -> B200PIR_E_BADARG. */
int b200pir_dpir_shard_info(b200pir_dpir* m, uint64_t* row_begin, uint64_t* rows, uint64_t* cols, int* device);
/* A server over the row shards dbs[0 .. shards) of one database (borrowed; they must outlive the server), each shard on its
 * handle's device, the first one's device being where responses are summed.  Each shard uploads its column band of
 * h1_squished and of a2_t (the last band with the padding column).  The shards must tile [0, l) in order with every inner edge
 * a multiple of 3x, and have ceil(m/3) packed columns; otherwise B200PIR_E_SHAPE.  Other errors as b200pir_dpir_server_create.
 * The server is an ordinary b200pir_dpir_server: answer_size, answer (unchunked), answer_many, server_update, server_state and
 * server_destroy keep their meaning, byte for byte the one-GPU results.  Each shard runs the passes of answer() over its rows on
 * its device; the shards' partial responses go to the first shard's device (cudaMemcpyPeerAsync) and one kernel adds them.
 * An update splits its changes by owning shard, and h2 passes through each shard's hint patch in turn; server_state gathers the
 * whole h1_squished.  answer with chunk_idx >= 0 -> B200PIR_E_UNSUPPORTED (a sharded server holds every row). */
int b200pir_dpir_server_create_sharded(const b200pir_dpir_params* params, uint64_t num_entries, uint64_t bits_per_entry,
                                       b200pir_dpir* const* dbs, size_t shards, const uint32_t* h1_squished, const uint32_t* a2_t,
                                       size_t max_queries, b200pir_dpir_server** out);

#ifdef __cplusplus
}
#endif
#endif
