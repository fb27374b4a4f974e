// What the Spiral translation units (api.cu: context, public parameters and the query path; db_api.cu: the database handle)
// share: the context, the database handle, the context lock and the handle check.
#pragma once
#include "api_internal.hpp"
#include <algorithm>
#include <chrono>
#include <condition_variable>
#include <cstring>
#include <deque>
#include <memory>
#include <mutex>
#include <vector>

using namespace b200pir;     // the handle structs below live outside the namespace, as the C ABI names them

enum Stage { ST_EXPAND = 0, ST_MUL, ST_FROMNTT, ST_FOLD, ST_PACK, ST_ENCODE, ST_QIMG /* query operand re-tiling */, ST_COUNT };

struct b200pir_ctx {
  uint64_t seq = 0;          // creation order: the order in which a call that spans several contexts takes their locks
  int device = 0;
  cudaStream_t stream = nullptr;
  bool own_stream = true;
  std::recursive_mutex mu;
  b200pir_params hp;
  // derived (params.rs:116-200)
  int dim0, num_per, slices, trials, g, stop_round, num_packing;
  int bits_gsw, bits_conv, bits_left, bits_right;
  int live_gsw, live_conv, live_left, live_right;     // live_digits() of each gadget
  bool has_right;
  uint64_t q2, q1, setup_bytes, query_bytes, response_bytes;
  int q1_bits;
  size_t slice_words;        // u64 words of one slice in the reference layout: dim0 * num_per * 2048
  size_t bytes_per_chunk;    // params.bytes_per_chunk(): plaintext bytes of an item in each slice
  DevParams dp;
  DevBuf<Twiddle> d_tw;      // fwd0, inv0, fwd1, inv1, inv_lz0, inv_lz1
  DevBuf<Twiddle> d_tw4k;    // fwd0, inv0, fwd1, inv1 for poly_len 4096 (config #5 sweep)
  DevBuf<uint32_t> d_neg1;   // [11][2][2048] ntt32 (params.rs:98-107)
  // options
  int max_group = 16, profile = 0;  // max_group: queries per database pass (IMAD path: <= 4)
  int sparse_fold = 0;           // 1: lib/server's fold (all-zero ciphertext shortcut, compute/fold.rs:37-43); 0: spiral-rs dense fold
  int db_format = -1;            // format given to databases created from now on: -1 = automatic (2 where the wgmma kernel
                                 // supports the geometry, else 1), 0 = IMAD layout, 1 = mma.sync fragments, 2 = wgmma tile images
  DevBuf<uint2> w_qf;            // B operand of the IMMA path (one group of <= 16 queries)
  DevBuf<uint8_t> w_qt;          // B operand of the wgmma path (tile images, 16 queries)
  int sm_count = 0;
  // workspace, sized for `ws_queries` queries
  size_t ws_queries = 0, ws_rows = 0;
  DevBuf<uint64_t> w_query;      // [Q][2][2048] raw
  DevBuf<uint32_t> w_v;          // [Q][2^g][2][2][2048]
  DevBuf<uint32_t> w_zflags;     // all-zero flags of the current fold round's ciphertexts ("sparse_fold")
  DevBuf<uint32_t> w_xr;         // [Q][num_in][2][2048] residues of row 0 (expansion rounds)
  DevBuf<uint4> w_qdev;          // [Q][dim0][2048]
  DevBuf<uint32_t> w_vfold;      // [Q][nu_2][2][2t][2][2048]
  DevBuf<uint32_t> w_mult;       // [Q][slices][rows][2][2][2048]  NTT form, then residue form in place
  DevBuf<uint32_t> w_cts;        // ping-pong partner of w_mult for the fold rounds (same size)
  DevBuf<uint64_t> w_packed;     // [Q][inst][n+1][n][2048]
  DevBuf<uint8_t> w_resp;        // [Q][response_bytes]
  // database writers (upsert, update_item_raw, update_many_items, load_raw_file, uploads): raw item bytes and their item
  // descriptors, one group of whole items at a time; sized on the first write, so later writes neither allocate nor free
  // device memory
  static constexpr size_t kWriteStageBytes = (size_t)64 << 20;
  static constexpr size_t kWriteStageItems = 65536;
  DevBuf<uint8_t> w_wbytes;
  DevBuf<ItemWrite> w_witems;
  // database exports (download, save_file): chunks are un-tiled into w_wbytes and copied to one of two pinned buffers, one
  // event each; allocated on the first export, freed in b200pir_ctx_destroy.  Exports share them, so export_mu serialises
  // exports with each other; queries only contend for `mu`, which an export holds per chunk.
  std::mutex export_mu;
  uint8_t* h_export[2] = {nullptr, nullptr};
  size_t h_export_bytes = 0;
  cudaEvent_t export_done[2] = {nullptr, nullptr};
  void ensure_export_staging(size_t bytes) {
    w_wbytes.ensure(std::max(kWriteStageBytes, bytes));
    if (!export_done[0])
      for (auto& e : export_done) B200_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming | cudaEventBlockingSync));
    if (bytes <= h_export_bytes) return;
    release_export_pinned();
    const size_t n = std::max(kWriteStageBytes, bytes);
    for (auto& h : h_export) B200_CUDA(cudaHostAlloc(reinterpret_cast<void**>(&h), n, cudaHostAllocDefault));
    h_export_bytes = n;
  }
  void release_export_pinned() {
    for (auto& h : h_export) { if (h) cudaFreeHost(h); h = nullptr; }
    h_export_bytes = 0;
  }
  // Coalescing of concurrent callers ("coalesce", default on): lib/server takes a READ lock around process_query
  // (bin/server.rs:102), so actix workers call it concurrently.  Requests arriving while a batch runs queue up here; the
  // thread that finds no batch in flight becomes the leader and serves everything queued (up to kCoalesceMax) in ONE
  // database pass.  A lone caller is served immediately.  Two refinements for sustained load: a batch larger than one
  // database pass (16 queries) is trimmed to whole passes, the remainder joining the next batch (it would have finished no
  // earlier inside this one); and a leader that follows a multi-query batch by less than 1 ms gives the callers of that batch
  // up to "coalesce_window_us" (default 200) to come back before it starts, so closed-loop clients do not alternate between
  // full and near-empty passes.
  struct Pending {
    b200pir_db* db; b200pir_pp* pp; const uint64_t* query_ct; const uint8_t* query_bytes; uint8_t* out;
    int rc = 0; std::string err; bool done = false;
  };
  static constexpr size_t kCoalesceMax = 32;
  static constexpr size_t kPassQueries = 16;
  int coalesce = 1;
  int coalesce_window_us = 200;
  size_t last_batch = 0;
  std::chrono::steady_clock::time_point last_batch_end{};
  std::mutex qmu;
  std::condition_variable qcv;
  std::deque<Pending*> pending;
  bool leader_active = false;
  unsigned long long coalesced_batches = 0, coalesced_queries = 0;
  // per-query public parameters (PpTable, kernels.h): device arrays [4][pptab_cap] of base pointers, filled by pp_table (api.cu)
  DevBuf<const uint32_t*> d_pptab;
  size_t pptab_cap = 0;
  std::vector<const uint32_t*> h_pptab;          // what d_pptab holds (skip the upload when unchanged)
  // profiling
  struct Span { int stage; cudaEvent_t a, b; };
  std::vector<Span> spans;
  std::vector<cudaEvent_t> event_pool;
  size_t event_next = 0;
  int mul_launches = 0;
  double last_ms[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};   // expand, multiply, from_ntt, fold, pack, encode, total, multiply launches, query image

  size_t v_words() const { return ((size_t)1 << g) * 4 * POLY; }
  size_t fold_words() const { return (size_t)hp.nu_2 * 2 * 2 * hp.t_gsw * 2 * POLY; }
  MulGeom geom(int rows) const { return MulGeom{dim0, rows, slices}; }

  cudaEvent_t get_event() {
    if (event_next == event_pool.size()) {
      cudaEvent_t e;
      B200_CUDA(cudaEventCreate(&e));
      event_pool.push_back(e);
    }
    return event_pool[event_next++];
  }
  struct Scope {
    b200pir_ctx* c; int stage; cudaEvent_t a = nullptr;
    Scope(b200pir_ctx* ctx, int st) : c(ctx), stage(st) {
      if (c->profile) { a = c->get_event(); cudaEventRecord(a, c->stream); }
    }
    ~Scope() {
      if (c->profile) { cudaEvent_t b = c->get_event(); cudaEventRecord(b, c->stream); c->spans.push_back({stage, a, b}); }
    }
  };
  // profile == 1: per call; profile == 2: accumulate over calls until the option is set again
  void prof_reset() { if (profile == 2) return; spans.clear(); event_next = 0; mul_launches = 0; }
  void prof_collect() {
    if (!profile) return;
    B200_CUDA(cudaStreamSynchronize(stream));
    for (int i = 0; i < 9; i++) last_ms[i] = 0;
    for (auto& s : spans) {
      float ms = 0;
      cudaEventElapsedTime(&ms, s.a, s.b);
      last_ms[s.stage == ST_QIMG ? 8 : s.stage] += ms;
      last_ms[6] += ms;
    }
    last_ms[7] = mul_launches;
  }
  // buffers of the first dimension / fold / pack only (queries expanded elsewhere)
  void ensure_workspace_lite(size_t queries, size_t rows) {
    w_mult.ensure(queries * slices * rows * 4 * POLY);
    w_cts.ensure(queries * slices * rows * 4 * POLY);
    w_packed.ensure(queries * hp.instances * (hp.n + 1) * hp.n * POLY);
  }
  void ensure_workspace(size_t queries, size_t rows) {
    if (queries <= ws_queries && rows <= ws_rows) return;
    queries = std::max(queries, ws_queries);
    rows = std::max(rows, ws_rows);
    w_query.ensure(queries * 2 * POLY);
    if (hp.expand_queries) w_v.ensure(queries * v_words());
    w_qdev.ensure(queries * (size_t)dim0 * POLY);
    w_vfold.ensure(queries * std::max<size_t>(fold_words(), 1));
    w_mult.ensure(queries * slices * rows * 4 * POLY);
    w_cts.ensure(queries * slices * rows * 4 * POLY);
    w_packed.ensure(queries * hp.instances * (hp.n + 1) * hp.n * POLY);
    w_resp.ensure(queries * response_bytes);
    ws_queries = queries;
    ws_rows = rows;
  }
};

// One row shard's storage on the context that created it: rows ii = shard.index (mod shard.count) of every slice.
struct DbStore {
  b200pir_ctx* ctx;
  Shard shard;
  int rows;                 // local second-dimension rows
  DbLayout layout;          // format (0: IMAD cells, 1: mma.sync fragments, 2: wgmma tile images), geometries, store.p
  DevBuf<uint8_t> store;    // db_bytes(layout, slices) bytes
  // The first dimension's product is z-major (formats 1 and 2: u32 [query][slice][n][z][row][ct_row]) or ntt32 (format 0)
  bool zmajor_product() const { return layout.format != 0; }
  // Presence (lib/server's SparseDb, db/sparse_db.rs:5-47: an item exists once it has been written).  Storage stays dense in HBM
  // (absent = zero polynomial, so every sum is unchanged); what the map buys is COST: on the wgmma path whole 32-row x 32-j
  // tiles without a present item are neither fetched nor multiplied (tile_mask, one bit per tile, kept on the device).
  // Maintained in db_api.cu.
  std::vector<uint64_t> present;          // bit ((slice * rows + il) * dim0 + j)
  uint64_t present_count = 0;
  std::vector<uint32_t> h_tile_mask;      // [slice][mt], bit ks
  DevBuf<uint32_t> tile_mask;
  uint64_t capacity() const { return (uint64_t)ctx->slices * rows * ctx->dim0; }
  void mark_items(const ItemWrite* items, size_t count, int slice_begin, int slice_end, cudaStream_t s);
  void mark_slices(int slice_begin, int slice_end, cudaStream_t s);
};

// A database handle, owned by the home context `ctx`: a list of row-shard stores.  b200pir_db_create gives one part, the
// whole database or one rank shard of it; b200pir_db_create_sharded gives G parts, part g holding shard g of G on its own
// context.  With several parts a query call expands on the home context, hands the operand to every part, and finishes on the
// home context from the survivors the parts gather in `gathered`: that exchange state exists only then (db_api.cu creates it,
// api.cu's run_shards uses it).
struct b200pir_db {
  b200pir_ctx* ctx;
  struct Part {
    std::unique_ptr<DbStore> store;
    DevBuf<uint8_t> operand;      // the call's first-dimension operand, on a part whose device is not the home device
    DevBuf<uint32_t> vfold;       // the call's folding matrices, likewise
    cudaEvent_t done = nullptr;   // recorded on the part's stream after its survivors are gathered
  };
  std::vector<Part> parts;        // at least one
  size_t exchange_queries = 0;    // queries the buffers below and the parts' receive buffers hold
  DevBuf<uint32_t> gathered;      // on the home device: [G][count][slices][4 * 2048] survivors
  cudaEvent_t expanded = nullptr; // recorded on the calling context's stream once the operands are in place
  cudaEvent_t finished = nullptr; // recorded after the finish: the next call's calling stream waits on it
  bool sharded() const { return parts.size() > 1; }
  // every row of the database, not one rank shard of it
  bool whole() const { return parts.size() == (size_t)parts[0].store->shard.count; }
  // The context that does part g's work in a call on context c: c itself with one part, so that contexts sharing a database
  // each run on their own stream; the part's own context with several
  b200pir_ctx* worker(b200pir_ctx* c, size_t g) const { return sharded() ? parts[g].store->ctx : c; }
  // The one store of a database that is not sharded; a sharded one runs its own schedule and is refused with `refusal`
  const DbStore& single(const char* refusal) const {
    if (sharded()) throw Error(B200PIR_E_UNSUPPORTED, refusal);
    return *parts[0].store;
  }
  size_t operand_bytes(size_t queries) const;
  void ensure_exchange(size_t queries);
  ~b200pir_db();
};

namespace b200pir {

// The calling context's lock and the lock of every context that does a part's work (b200pir_db::worker: only c's for a
// database of one part, which keeps contexts that share it concurrent), taken in creation order so that calls on databases
// that share contexts, and direct calls on a member context, cannot deadlock; the current device becomes c's.
struct Guard {
  std::vector<b200pir_ctx*> held;
  explicit Guard(b200pir_ctx* c, const b200pir_db* db = nullptr) {
    held.push_back(c);
    if (db)
      for (size_t g = 0; g < db->parts.size(); g++) held.push_back(db->worker(c, g));
    std::sort(held.begin(), held.end(), [](const b200pir_ctx* a, const b200pir_ctx* b) { return a->seq < b->seq; });
    held.erase(std::unique(held.begin(), held.end()), held.end());
    for (auto* h : held) h->mu.lock();
    cudaSetDevice(c->device);
  }
  ~Guard() {
    for (auto it = held.rbegin(); it != held.rend(); ++it) (*it)->mu.unlock();
  }
  Guard(const Guard&) = delete;
  Guard& operator=(const Guard&) = delete;
};

// handles may be used from any context with identical parameters on the same device (one context per host
// thread / CUDA stream sharing one HBM-resident database)
inline bool same_params(const b200pir_ctx* a, const b200pir_ctx* b) {
  return a == b || (a->device == b->device && std::memcmp(&a->hp, &b->hp, sizeof(b200pir_params)) == 0);
}
inline void check_db(b200pir_ctx* c, b200pir_db* db) {
  if (!db || !same_params(db->ctx, c)) throw Error(B200PIR_E_BADARG, "db handle was created for different parameters / device");
}

}  // namespace b200pir
