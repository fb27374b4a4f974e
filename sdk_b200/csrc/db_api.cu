// C-ABI implementation of the HBM-resident database handle (include/b200pir.h): creation, bulk uploads and file loads,
// exports, the plaintext read-back (read_items, save_raw_file), the item writers and the presence map.  Every writer works over
// the parts of the handle (several for b200pir_db_create_sharded), on the contexts members() names, from inputs read once,
// and makes the same three decisions in one place each: which member holds an item (owner), how raw items are staged in
// groups and written (RawWriter, in the context's write staging w_wbytes / w_witems), and how the call ends (settle: presence,
// then a synchronise of each member written).
#include "spiral_api.hpp"
#include "update_body.hpp"
#include <cstdio>
#include <cerrno>
#include <fcntl.h>
#include <unistd.h>
#include <memory>
#include <optional>
#include <utility>

static_assert(B200PIR_ITEM_NOT_PLAINTEXT == kReadNotPlaintext && B200PIR_ITEM_PAST_CHUNK == kReadPastChunk &&
              (B200PIR_ITEM_PRESENT & (kReadNotPlaintext | kReadPastChunk)) == 0, "k_read_items' flag bits are the ABI's");

// ---------------------------------------------------------------- presence
// every item of `items` written in slices [slice_begin, slice_end): one upload of the whole mask when any word changed
void DbStore::mark_items(const ItemWrite* items, size_t count, int slice_begin, int slice_end, cudaStream_t s) {
  bool changed = false;
  for (size_t k = 0; k < count; k++)
    for (int sl = slice_begin; sl < slice_end; sl++) {
      const uint64_t bit = ((uint64_t)sl * rows + items[k].il) * ctx->dim0 + items[k].j;
      if (!((present[bit >> 6] >> (bit & 63)) & 1)) { present[bit >> 6] |= 1ull << (bit & 63); present_count++; }
      uint32_t& w = h_tile_mask[(size_t)sl * layout.T.mt + (items[k].il >> 5)];
      const uint32_t nv = w | (1u << (items[k].j >> 5));
      changed |= nv != w;
      w = nv;
    }
  if (changed)
    B200_CUDA(cudaMemcpyAsync(tile_mask.p, h_tile_mask.data(), h_tile_mask.size() * 4, cudaMemcpyHostToDevice, s));
}
// whole slices [slice_begin, slice_end) written at once (bulk upload, file load, synthetic fill): every item of them exists
// from now on
void DbStore::mark_slices(int slice_begin, int slice_end, cudaStream_t s) {
  const uint64_t lo = (uint64_t)slice_begin * rows * ctx->dim0, hi = (uint64_t)slice_end * rows * ctx->dim0;
  for (uint64_t b = lo; b < hi; b++)
    if (!((present[b >> 6] >> (b & 63)) & 1)) { present[b >> 6] |= 1ull << (b & 63); present_count++; }
  const Tc5Geom& T = layout.T;
  const uint32_t full = T.ks >= 32 ? 0xffffffffu : ((1u << T.ks) - 1u);
  const size_t w0 = (size_t)slice_begin * T.mt, w1 = (size_t)slice_end * T.mt;
  for (size_t w = w0; w < w1; w++) h_tile_mask[w] = full;
  B200_CUDA(cudaMemcpyAsync(tile_mask.p + w0, &h_tile_mask[w0], (w1 - w0) * 4, cudaMemcpyHostToDevice, s));
}

b200pir_db::~b200pir_db() {
  for (auto& p : parts) {
    if (!p.store) continue;                   // a creation that failed before this part
    cudaSetDevice(p.store->ctx->device);
    if (p.done) cudaEventDestroy(p.done);
    p.operand.release();
    p.vfold.release();
    p.store.reset();
  }
  cudaSetDevice(ctx->device);
  if (expanded) cudaEventDestroy(expanded);
  if (finished) cudaEventDestroy(finished);
}

// Bytes of the first-dimension operand of `queries` queries as the query path hands it to a part: tile images of 16 queries
// for a format-2 database whose queries are expanded, q_dev otherwise
size_t b200pir_db::operand_bytes(size_t queries) const {
  if (parts[0].store->layout.format == 2 && ctx->hp.expand_queries) return (queries + 15) / 16 * tc5_query_bytes(make_tc5_geom(ctx->dim0, 32));
  return queries * ctx->dim0 * POLY * sizeof(uint4);
}

// The survivor buffer and the receive buffers of the other-device parts, for `queries` queries.  Replacing them waits for every
// part's stream and the last finish, so no call still in flight uses them.  Leaves the home device current.
void b200pir_db::ensure_exchange(size_t queries) {
  if (queries <= exchange_queries) return;
  for (auto& p : parts) {
    B200_CUDA(cudaSetDevice(p.store->ctx->device));
    B200_CUDA(cudaStreamSynchronize(p.store->ctx->stream));
  }
  B200_CUDA(cudaSetDevice(ctx->device));
  B200_CUDA(cudaEventSynchronize(finished));
  gathered.alloc(parts.size() * queries * ctx->slices * 4 * POLY);
  for (auto& p : parts) {
    if (p.store->ctx->device == ctx->device) continue;
    B200_CUDA(cudaSetDevice(p.store->ctx->device));
    p.operand.alloc(operand_bytes(queries));
    p.vfold.alloc(queries * ctx->fold_words());
  }
  B200_CUDA(cudaSetDevice(ctx->device));
  exchange_queries = queries;
}

namespace {

// Where a writer or an export of `db` called on context c does its work: every part's store, on the context
// b200pir_db::worker names
struct Member { b200pir_ctx* ctx; DbStore* store; };
std::vector<Member> members(b200pir_ctx* c, b200pir_db* db) {
  std::vector<Member> ms;
  for (size_t g = 0; g < db->parts.size(); g++) ms.push_back(Member{db->worker(c, g), db->parts[g].store.get()});
  return ms;
}

// The member of `ms` that holds global item idx, with the item's local row il and column j; none when the database is a rank
// shard that does not hold the item's row
struct Owner { size_t g; int il, j; };
std::optional<Owner> owner(const std::vector<Member>& ms, uint64_t idx) {
  for (size_t g = 0; g < ms.size(); g++) {
    int il, j;
    if (ms[g].store->shard.local_item(idx, ms[g].ctx->num_per, il, j)) return Owner{g, il, j};
  }
  return std::nullopt;
}

// How every writer ends.  On each member the call wrote, presence is marked on the member's stream and the stream is
// synchronised: items[g], member g's written items, in slices [slice_begin, slice_end), or without `items` those whole slices
// on every member.  A member that received nothing is not touched.  Writers hold the host write lock (bin/server.rs:35,49), so
// a write is complete when the call returns.  Leaves the home device current.
void settle(b200pir_ctx* c, const std::vector<Member>& ms, int slice_begin, int slice_end,
            const std::vector<std::vector<ItemWrite>>* items = nullptr) {
  for (size_t g = 0; g < ms.size(); g++) {
    if (items && (*items)[g].empty()) continue;
    B200_CUDA(cudaSetDevice(ms[g].ctx->device));
    if (items) ms[g].store->mark_items((*items)[g].data(), (*items)[g].size(), slice_begin, slice_end, ms[g].ctx->stream);
    else ms[g].store->mark_slices(slice_begin, slice_end, ms[g].ctx->stream);
    B200_CUDA(cudaStreamSynchronize(ms[g].ctx->stream));
  }
  B200_CUDA(cudaSetDevice(c->device));
  B200_CUDA(cudaGetLastError());
}

// One slice in the reference's z-major layout, delivered chunk by chunk: fetch(word_offset, n_words) returns a host pointer
// to that range of the slice (valid until the next call).
template <typename Fetch>
void upload_slice_impl(b200pir_ctx* c, b200pir_db* db, uint64_t slice, Fetch fetch) {
  // reference layout is z-major: stage a range of z at a time in the writers' staging (w_wbytes, at least 64 MiB).  An export
  // may still be copying its last chunk out of it; that copy is queued on the context's stream, ahead of this upload's copies.
  // Each range is fetched once and staged to every member (a pageable copy has taken its source when it returns).
  const std::vector<Member> ms = members(c, db);
  const size_t per_z = (size_t)c->dim0 * c->num_per;
  int zc = (int)std::max<size_t>(1, std::min<size_t>(POLY, b200pir_ctx::kWriteStageBytes / (per_z * 8)));
  for (const Member& m : ms) {
    B200_CUDA(cudaSetDevice(m.ctx->device));
    m.ctx->w_wbytes.ensure(std::max(b200pir_ctx::kWriteStageBytes, per_z * zc * 8));
  }
  for (int z0 = 0; z0 < POLY; z0 += zc) {
    int cur = std::min(zc, POLY - z0);
    const uint64_t* src = fetch((size_t)z0 * per_z, per_z * cur);
    for (const Member& m : ms) {
      B200_CUDA(cudaSetDevice(m.ctx->device));
      uint64_t* stage = reinterpret_cast<uint64_t*>(m.ctx->w_wbytes.p);
      B200_CUDA(cudaMemcpyAsync(stage, src, per_z * cur * 8, cudaMemcpyHostToDevice, m.ctx->stream));
      launch_db_import(m.store->layout, m.store->shard, (int)slice, stage, z0, cur, m.ctx->stream);
    }
    for (const Member& m : ms) B200_CUDA(cudaStreamSynchronize(m.ctx->stream));
  }
  settle(c, ms, (int)slice, (int)slice + 1);
}

// The raw-item writer (update_item_raw, update_many_items, load_raw_file).  The caller adds the items of one group, whose bytes
// lie in one host span, then writes the group from that span; finish() settles the call.  Presence: every written item in
// every slice, or, `dense`, every slice of every member (a whole database was loaded).
struct RawWriter {
  b200pir_ctx* c;
  std::vector<Member> ms;
  bool dense;
  std::vector<std::vector<ItemWrite>> group, written;   // per member: the group's items, and those of the groups written
  bool full = false;                                    // some member's share of the group fills its item staging
  RawWriter(b200pir_ctx* c, b200pir_db* db, bool dense) : c(c), ms(members(c, db)), dense(dense), group(ms.size()), written(ms.size()) {}
  // item db_idx at bytes [off, off + len) of the group's span, for the member that holds it
  void add(uint64_t db_idx, size_t off, uint32_t len) {
    const std::optional<Owner> o = owner(ms, db_idx);
    if (!o) return;
    group[o->g].push_back(ItemWrite{(uint32_t)off, len, (uint32_t)o->il, (uint32_t)o->j});
    full |= group[o->g].size() >= b200pir_ctx::kWriteStageItems;
  }
  // Stages `span` bytes from `host` to each member that received items of the group and writes them there: one
  // conversion-and-placement launch over (item, slice).  Stream-ordered: the staging buffers are only overwritten by the next
  // group's copies, which run after this launch.
  void write(const uint8_t* host, size_t span) {
    for (size_t g = 0; g < ms.size(); g++) {
      std::vector<ItemWrite>& items = group[g];
      if (items.empty()) continue;
      b200pir_ctx* x = ms[g].ctx;
      B200_CUDA(cudaSetDevice(x->device));
      x->w_wbytes.ensure(std::max(b200pir_ctx::kWriteStageBytes, span));
      x->w_witems.ensure(std::max(b200pir_ctx::kWriteStageItems, items.size()));
      // pageable sources: staged before the copies return, so `host` and `items` may be refilled
      if (span) B200_CUDA(cudaMemcpyAsync(x->w_wbytes.p, host, span, cudaMemcpyHostToDevice, x->stream));
      B200_CUDA(cudaMemcpyAsync(x->w_witems.p, items.data(), items.size() * sizeof(ItemWrite), cudaMemcpyHostToDevice, x->stream));
      launch_write_items(x->dp, ms[g].store->layout, x->w_wbytes.p, x->w_witems.p, (int)items.size(), x->slices,
                         (int)x->bytes_per_chunk, x->hp.p, x->stream);
      if (!dense) written[g].insert(written[g].end(), items.begin(), items.end());
      items.clear();
    }
    full = false;
  }
  void finish() { settle(c, ms, 0, c->slices, dense ? nullptr : &written); }
};

// Device-to-host streaming, shared by the exports (b200pir_db_download(_slice), b200pir_db_save_file) and the item readers
// (b200pir_db_read_items, b200pir_db_save_raw_file).  Under each member's context lock, fill(k, g, stage) queues the device
// work that leaves chunk k of member g in its writers' staging (w_wbytes, at least `stage_bytes`, the 64 MiB minimum) and
// returns its size; the chunk is queued for a copy to one of the two pinned buffers, the locks are released, and
// sink(k - 1, src) consumes the previous chunk once its copies have landed (src[g] = member g's bytes) while the GPU produces
// and copies this one.  Everything is ordered on each context's stream, so a chunk never overwrites staging that the previous
// chunk's copy still reads.  A sharded database produces each chunk on every part, on the part's context.
template <typename Fill, typename Sink>
void stream_out(b200pir_ctx* c, b200pir_db* db, size_t chunks, size_t stage_bytes, Fill fill, Sink sink) {
  const std::vector<Member> ms = members(c, db);
  std::vector<b200pir_ctx*> order;
  for (const Member& m : ms) order.push_back(m.ctx);
  std::sort(order.begin(), order.end(), [](const b200pir_ctx* a, const b200pir_ctx* b) { return a->seq < b->seq; });
  std::vector<std::unique_lock<std::mutex>> ex;
  for (b200pir_ctx* x : order) ex.emplace_back(x->export_mu);
  for (const Member& m : ms) {
    Guard gd(m.ctx);
    m.ctx->ensure_export_staging(stage_bytes);
  }
  std::vector<const uint8_t*> src(ms.size());
  auto consume = [&](size_t k) {
    const int b = (int)(k & 1);
    for (size_t g = 0; g < ms.size(); g++) {
      B200_CUDA(cudaEventSynchronize(ms[g].ctx->export_done[b]));
      src[g] = ms[g].ctx->h_export[b];
    }
    sink(k, src);
  };
  try {
    for (size_t k = 0; k < chunks; k++) {
      for (size_t g = 0; g < ms.size(); g++) {
        Guard gd(ms[g].ctx);
        b200pir_ctx* x = ms[g].ctx;
        const size_t bytes = fill(k, g, x->w_wbytes.p);
        if (bytes) B200_CUDA(cudaMemcpyAsync(x->h_export[k & 1], x->w_wbytes.p, bytes, cudaMemcpyDeviceToHost, x->stream));
        B200_CUDA(cudaEventRecord(x->export_done[k & 1], x->stream));
      }
      if (k > 0) consume(k - 1);
    }
    if (chunks) consume(chunks - 1);
  } catch (...) {
    for (const Member& m : ms)
      for (auto e : m.ctx->export_done) cudaEventSynchronize(e);     // no copy may still land in the pinned buffers
    cudaSetDevice(c->device);
    throw;
  }
  B200_CUDA(cudaSetDevice(c->device));
  B200_CUDA(cudaGetLastError());
}

// Database export.  A chunk is one slice and a range of z of the local rows, at most the writers' 64 MiB staging: one launch
// un-tiles it into [zc][rows][dim0] u64 there, and `sink(slice, z0, zc, words)` consumes it, `words[g]` being member g's.
template <typename Sink>
void export_impl(b200pir_ctx* c, b200pir_db* db, int slice_begin, int slice_end, Sink sink) {
  const std::vector<Member> ms = members(c, db);
  const size_t per_z = (size_t)ms[0].store->rows * c->dim0;
  const int zc = (int)std::max<size_t>(1, std::min<size_t>(POLY, b200pir_ctx::kWriteStageBytes / (per_z * 8)));
  struct Chunk { int slice, z0, zc; };
  std::vector<Chunk> chunks;
  for (int s = slice_begin; s < slice_end; s++)
    for (int z0 = 0; z0 < POLY; z0 += zc) chunks.push_back(Chunk{s, z0, std::min(zc, POLY - z0)});
  std::vector<const uint64_t*> words(ms.size());
  stream_out(c, db, chunks.size(), per_z * zc * 8,
             [&](size_t k, size_t g, uint8_t* stage) {
               launch_db_export(ms[g].store->layout, chunks[k].slice, chunks[k].z0, chunks[k].zc, reinterpret_cast<uint64_t*>(stage),
                                ms[g].ctx->stream);
               return per_z * chunks[k].zc * 8;
             },
             [&](size_t k, const std::vector<const uint8_t*>& src) {
               for (size_t g = 0; g < ms.size(); g++) words[g] = reinterpret_cast<const uint64_t*>(src[g]);
               sink(chunks[k].slice, chunks[k].z0, chunks[k].zc, words);
             });
}

// Items read back as the bytes the raw writers take (b200pir_db_read_items, b200pir_db_save_raw_file): the `count` global
// indices idx(0 .. count-1), which the caller has checked, in groups of whole items that fit the staging.  For each group every
// member decodes the items it holds with one k_read_items launch: its m-th item of the group goes to slot m of its staging
// (span = slices * bytes_per_chunk bytes), followed by one flag byte per (slot, slice).  Then sink(k0, n, bytes, flags)
// consumes items k0 .. k0+n-1: bytes(k) points at item k's span, flags(k) is its B200PIR_ITEM_* bits.
template <typename Index, typename Sink>
void read_items_impl(b200pir_ctx* c, b200pir_db* db, size_t count, Index idx, Sink sink) {
  const std::vector<Member> ms = members(c, db);
  const size_t slices = (size_t)c->slices, span = slices * c->bytes_per_chunk;
  const size_t group = std::max<size_t>(1, std::min(b200pir_ctx::kWriteStageItems, b200pir_ctx::kWriteStageBytes / (span + slices)));
  // where each item of the groups in flight (two: one being filled, one being consumed) lives
  struct Where { uint32_t g, slot; uint8_t present; };
  std::vector<Where> where[2];
  std::vector<size_t> held[2];                     // items of the group per member
  std::vector<ItemWrite> items;
  for (auto& h : held) h.assign(ms.size(), 0);
  stream_out(c, db, (count + group - 1) / group, group * (span + slices),
             [&](size_t k, size_t g, uint8_t* stage) -> size_t {
               const size_t k0 = k * group, n = std::min(group, count - k0);
               std::vector<Where>& w = where[k & 1];
               w.resize(n);
               const DbStore* m = ms[g].store;
               items.clear();
               for (size_t i = 0; i < n; i++) {
                 const std::optional<Owner> o = owner(ms, idx(k0 + i));
                 if (!o || o->g != g) continue;                                // row lives on another member
                 uint8_t present = 0;
                 for (size_t sl = 0; sl < slices; sl++) {
                   const uint64_t bit = ((uint64_t)sl * m->rows + o->il) * c->dim0 + o->j;
                   present |= (m->present[bit >> 6] >> (bit & 63)) & 1;
                 }
                 w[i] = Where{(uint32_t)g, (uint32_t)items.size(), present ? (uint8_t)B200PIR_ITEM_PRESENT : (uint8_t)0};
                 items.push_back(ItemWrite{(uint32_t)items.size(), 0, (uint32_t)o->il, (uint32_t)o->j});
               }
               held[k & 1][g] = items.size();
               if (items.empty()) return 0;
               b200pir_ctx* x = ms[g].ctx;
               x->w_witems.ensure(std::max(b200pir_ctx::kWriteStageItems, items.size()));
               // pageable: staged before the call returns, so `items` may be refilled for the next member
               B200_CUDA(cudaMemcpyAsync(x->w_witems.p, items.data(), items.size() * sizeof(ItemWrite), cudaMemcpyHostToDevice, x->stream));
               launch_read_items(x->dp, m->layout, x->w_witems.p, (int)items.size(), (int)slices, (int)c->bytes_per_chunk, stage,
                                 stage + items.size() * span, x->stream);
               return items.size() * (span + slices);
             },
             [&](size_t k, const std::vector<const uint8_t*>& src) {
               const std::vector<Where>& w = where[k & 1];
               const std::vector<size_t>& h = held[k & 1];
               sink(k * group, w.size(),
                    [&](size_t i) { return src[w[i - k * group].g] + (size_t)w[i - k * group].slot * span; },
                    [&](size_t i) {
                      const Where& e = w[i - k * group];
                      const uint8_t* f = src[e.g] + h[e.g] * span + (size_t)e.slot * slices;
                      uint8_t bits = e.present;
                      for (size_t sl = 0; sl < slices; sl++) bits |= f[sl];
                      return bits;
                    });
             });
}

// Write `path` atomically: write(f) fills a temporary file in the same directory (mode 0600), which is flushed, fsync'ed and
// renamed over `path`, and the directory is fsync'ed.  On any failure the temporary file is removed and `path` keeps its
// earlier content; an Error from write(f) keeps its code, a failed file operation is B200PIR_E_BADARG naming the path.
template <typename Write>
void write_atomically(const char* path, Write write) {
  const std::string target(path);
  std::string tmp = target + ".tmp.XXXXXX";
  const int fd = mkstemp(&tmp[0]);
  if (fd < 0) throw Error(B200PIR_E_BADARG, "cannot create a temporary file next to " + target + ": " + std::strerror(errno));
  FILE* f = fdopen(fd, "wb");
  if (!f) close(fd);
  // drop the temporary file and report `why`: `path` is left as it was
  auto discard = [&](const std::string& why, int code) {
    if (f) fclose(f);
    f = nullptr;
    unlink(tmp.c_str());
    throw Error(code, code == B200PIR_E_BADARG ? "cannot write " + target + ": " + why : why);
  };
  if (!f) discard(std::strerror(errno), B200PIR_E_BADARG);
  try {
    write(f);
  } catch (const Error& e) {
    discard(e.what(), e.code);
  } catch (const std::exception& e) {
    discard(e.what(), B200PIR_E_CUDA);
  }
  if (fflush(f) != 0 || fsync(fileno(f)) != 0) discard(std::strerror(errno), B200PIR_E_BADARG);
  const int closed = fclose(f);
  f = nullptr;
  if (closed != 0) discard(std::strerror(errno), B200PIR_E_BADARG);
  if (rename(tmp.c_str(), target.c_str()) != 0) discard(std::strerror(errno), B200PIR_E_BADARG);
  // make the rename itself durable
  const size_t slash = target.find_last_of('/');
  const std::string dir = slash == std::string::npos ? "." : (slash == 0 ? "/" : target.substr(0, slash));
  const int dfd = open(dir.c_str(), O_RDONLY);
  if (dfd >= 0) { fsync(dfd); close(dfd); }
}

// the checks the raw writers make (update_item_raw, load_raw_file): bytes <-> coefficients is defined for p = 256 and chunks of
// at most poly_len bytes
void check_raw_params(const b200pir_ctx* c) {
  if (c->hp.p != 256) throw Error(B200PIR_E_UNSUPPORTED, "convert_pt_to_poly asserts logp == 8 (loading.rs:291)");
  if (c->bytes_per_chunk > (size_t)POLY) throw Error(B200PIR_E_SHAPE, "bytes_per_chunk exceeds poly_len");
}

// Chunk (zc values of z) of every member, `src[g]` being member g's [zc][rows][dim0], scattered into `dst`, the same range of z
// of a slice in the reference layout [z][num_per][dim0]
void scatter_rows(b200pir_ctx* c, const std::vector<Member>& ms, int zc, const std::vector<const uint64_t*>& src, uint64_t* dst) {
  const size_t d0 = (size_t)c->dim0, npg = (size_t)c->num_per;
  for (size_t g = 0; g < ms.size(); g++) {
    const DbStore* m = ms[g].store;
    const size_t rows = (size_t)m->rows;
    if (m->shard.count == 1) { std::memcpy(dst, src[g], (size_t)zc * rows * d0 * 8); continue; }
    for (size_t zl = 0; zl < (size_t)zc; zl++)
      for (size_t il = 0; il < rows; il++)
        std::memcpy(dst + (zl * npg + m->shard.global_row(il)) * d0, src[g] + (zl * rows + il) * d0, d0 * 8);
  }
}

// the local rows of slices [slice_begin, slice_end) into `words` (the reference layout of those slices)
void download_impl(b200pir_ctx* c, b200pir_db* db, int slice_begin, int slice_end, uint64_t* words) {
  const std::vector<Member> ms = members(c, db);
  export_impl(c, db, slice_begin, slice_end, [&](int s, int z0, int zc, const std::vector<const uint64_t*>& src) {
    scatter_rows(c, ms, zc, src, words + (size_t)(s - slice_begin) * c->slice_words + (size_t)z0 * c->num_per * c->dim0);
  });
}

// `path` opened for reading, and its size (ftello: negative when it cannot be told)
std::pair<std::unique_ptr<FILE, int (*)(FILE*)>, off_t> open_sized(const char* path) {
  std::unique_ptr<FILE, int (*)(FILE*)> f(fopen(path, "rb"), fclose);
  if (!f) throw Error(B200PIR_E_BADARG, std::string("cannot open ") + path);
  if (fseeko(f.get(), 0, SEEK_END)) throw Error(B200PIR_E_BADARG, "cannot seek in the database file");
  const off_t bytes = ftello(f.get());
  return {std::move(f), bytes};
}

// Rows ii = shard.index (mod shard.count) on context c in layout `format` (-1: automatic); c's lock is held
std::unique_ptr<DbStore> create_store(b200pir_ctx* c, Shard shard, int format) {
  std::unique_ptr<DbStore> s(new DbStore());
  s->ctx = c;
  s->shard = shard;
  s->rows = c->num_per / shard.count;
  DbLayout& L = s->layout;
  L.G = c->geom(s->rows);
  L.F = make_imma_geom(c->dim0, s->rows);
  L.T = make_tc5_geom(c->dim0, s->rows);
  L.format = format >= 0 ? format : (tc5_supported(L.T) ? 2 : 1);
  s->present.assign((s->capacity() + 63) / 64, 0);
  s->h_tile_mask.assign((size_t)c->slices * L.T.mt, 0u);
  s->tile_mask.alloc(s->h_tile_mask.size());
  // on the context's stream: a cudaMemset would queue on the legacy default stream, behind whatever the caller has there,
  // and could land after the first writer's mask upload on the context's stream
  B200_CUDA(cudaMemsetAsync(s->tile_mask.p, 0, s->h_tile_mask.size() * 4, c->stream));
  if (L.format == 2 && !tc5_supported(L.T)) throw Error(B200PIR_E_UNSUPPORTED, "db_format 2: dim0 too large for the wgmma kernel");
  s->store.alloc(db_bytes(L, c->slices));
  L.base = s->store.p;
  B200_CUDA(cudaMemsetAsync(s->store.p, 0, s->store.n, c->stream));
  B200_CUDA(cudaStreamSynchronize(c->stream));
  return s;
}

// lets the current device reach `peer`'s memory directly where the hardware allows it
void enable_peer(int device, int peer) {
  int can = 0;
  B200_CUDA(cudaDeviceCanAccessPeer(&can, device, peer));
  if (!can) return;
  B200_CUDA(cudaSetDevice(device));
  const cudaError_t e = cudaDeviceEnablePeerAccess(peer, 0);
  if (e == cudaErrorPeerAccessAlreadyEnabled) cudaGetLastError();
  else B200_CUDA(e);
}

// The handle whose part g is row shard shard_index + g of shard_count on ctxs[g], for `parts` = 1 (b200pir_db_create) or
// shard_count parts from shard 0 (b200pir_db_create_sharded), in the home context's db_format; the exchange state only with
// several parts
std::unique_ptr<b200pir_db> create_db(b200pir_ctx* const* ctxs, size_t parts, uint64_t shard_index, uint64_t shard_count) {
  b200pir_ctx* home = ctxs[0];
  int format;
  {
    Guard gd(home);
    if (shard_index >= shard_count || (shard_count & (shard_count - 1)) || (uint64_t)home->num_per % shard_count)
      throw Error(B200PIR_E_BADARG, "shard_count must be a power of two dividing num_per");
    format = home->db_format;
  }
  std::unique_ptr<b200pir_db> db(new b200pir_db());
  db->ctx = home;
  db->parts = std::vector<b200pir_db::Part>(parts);     // Part holds device buffers: built in place, never moved
  for (size_t g = 0; g < parts; g++) {
    b200pir_ctx* c = ctxs[g];
    Guard gd(c);
    b200pir_db::Part& p = db->parts[g];
    p.store = create_store(c, Shard{(int)(shard_index + g), (int)shard_count}, format);
    if (parts == 1) return db;
    B200_CUDA(cudaEventCreateWithFlags(&p.done, cudaEventDisableTiming));
    if (c->device != home->device) {
      enable_peer(c->device, home->device);
      enable_peer(home->device, c->device);
    }
  }
  Guard gd(home, db.get());
  B200_CUDA(cudaEventCreateWithFlags(&db->expanded, cudaEventDisableTiming));
  B200_CUDA(cudaEventCreateWithFlags(&db->finished, cudaEventDisableTiming));
  B200_CUDA(cudaEventRecord(db->finished, home->stream));
  db->ensure_exchange(b200pir_ctx::kCoalesceMax);
  return db;
}
}  // namespace

extern "C" {

int b200pir_db_create(b200pir_ctx* c, uint64_t shard_index, uint64_t shard_count, b200pir_db** out) {
  API_BEGIN
  if (!c || !out) throw Error(B200PIR_E_BADARG, "null argument");
  if (shard_count == 0) { shard_count = 1; shard_index = 0; }
  *out = create_db(&c, 1, shard_index, shard_count).release();
  API_END
}
int b200pir_db_create_sharded(b200pir_ctx* const* ctxs, size_t shards, b200pir_db** out) {
  API_BEGIN
  if (!ctxs || !out) throw Error(B200PIR_E_BADARG, "null argument");
  if (shards == 0) throw Error(B200PIR_E_BADARG, "shard_count must be a power of two dividing num_per");
  for (size_t g = 0; g < shards; g++) {
    if (!ctxs[g]) throw Error(B200PIR_E_BADARG, "null context");
    for (size_t h = 0; h < g; h++)
      if (ctxs[h] == ctxs[g]) throw Error(B200PIR_E_BADARG, "a context appears more than once");
    if (std::memcmp(&ctxs[g]->hp, &ctxs[0]->hp, sizeof(b200pir_params)) != 0)
      throw Error(B200PIR_E_BADARG, "the contexts of a sharded database must have identical parameters");
  }
  *out = create_db(ctxs, shards, 0, shards).release();
  API_END
}
void b200pir_db_destroy(b200pir_db* db) {
  delete db;                                  // frees each part on its own device
}

int b200pir_db_upload_slice(b200pir_ctx* c, b200pir_db* db, uint64_t slice, const uint64_t* words, size_t n_words) {
  API_BEGIN
  if (!c || !words) throw Error(B200PIR_E_BADARG, "null argument");
  Guard gd(c, db);
  check_db(c, db);
  if (slice >= (uint64_t)c->slices) throw Error(B200PIR_E_SHAPE, "slice out of range");
  if (n_words != c->slice_words) throw Error(B200PIR_E_SHAPE, "slice must hold dim0*num_per*2048 words");
  upload_slice_impl(c, db, slice, [&](size_t off, size_t) { return words + off; });
  API_END
}
// load_preprocessed_db_from_file (lib/spiral-rs/src/server.rs:373-386, lib/server/src/db/loading.rs:263-276): the file is the
// native-endian u64 stream of the whole `db: &[u64]`; it is streamed through a 64 MiB staging buffer, never held in RAM.
int b200pir_db_load_file(b200pir_ctx* c, b200pir_db* db, const char* path) {
  API_BEGIN
  if (!c || !path) throw Error(B200PIR_E_BADARG, "null argument");
  Guard gd(c, db);
  check_db(c, db);
  const auto [file, bytes] = open_sized(path);
  if (bytes < 0 || (uint64_t)bytes != (uint64_t)c->slice_words * c->slices * 8)
    throw Error(B200PIR_E_SHAPE, "database file must hold slices*dim0*num_per*2048 u64 words");
  std::vector<uint64_t> buf;
  for (int s = 0; s < c->slices; s++) {
    upload_slice_impl(c, db, (uint64_t)s, [&, f = file.get()](size_t off, size_t n) -> const uint64_t* {
      buf.resize(n);
      if (fseeko(f, (off_t)(((size_t)s * c->slice_words + off) * 8), SEEK_SET) || fread(buf.data(), 8, n, f) != n)
        throw Error(B200PIR_E_SHAPE, "short read from the database file");
      return buf.data();
    });
  }
  API_END
}
int b200pir_db_upload(b200pir_ctx* c, b200pir_db* db, const uint64_t* words, size_t n_words) {
  if (!c) { g_last_error = "null ctx"; return B200PIR_E_BADARG; }
  if (n_words != c->slice_words * c->slices) { g_last_error = "db must hold slices*dim0*num_per*2048 words"; return B200PIR_E_SHAPE; }
  for (int s = 0; s < c->slices; s++) {
    int rc = b200pir_db_upload_slice(c, db, s, words + (size_t)s * c->slice_words, c->slice_words);
    if (rc) return rc;
  }
  return 0;
}
int b200pir_db_download_slice(b200pir_ctx* c, b200pir_db* db, uint64_t slice, uint64_t* words, size_t n_words) {
  API_BEGIN
  if (!c || !words) throw Error(B200PIR_E_BADARG, "null argument");
  check_db(c, db);
  if (slice >= (uint64_t)c->slices) throw Error(B200PIR_E_SHAPE, "slice out of range");
  if (n_words != c->slice_words) throw Error(B200PIR_E_SHAPE, "slice must hold dim0*num_per*2048 words");
  download_impl(c, db, (int)slice, (int)slice + 1, words);
  API_END
}
int b200pir_db_download(b200pir_ctx* c, b200pir_db* db, uint64_t* words, size_t n_words) {
  API_BEGIN
  if (!c || !words) throw Error(B200PIR_E_BADARG, "null argument");
  check_db(c, db);
  if (n_words != c->slice_words * c->slices) throw Error(B200PIR_E_SHAPE, "db must hold slices*dim0*num_per*2048 words");
  download_impl(c, db, 0, c->slices, words);
  API_END
}
// The file b200pir_db_load_file reads, written atomically: a temporary file in the target's directory is written chunk by
// chunk (an unsharded chunk is a contiguous run of the file), flushed to disk and renamed over `path`; on any failure it is
// removed, so `path` holds either its earlier content or the complete new snapshot.
int b200pir_db_save_file(b200pir_ctx* c, b200pir_db* db, const char* path) {
  API_BEGIN
  if (!c || !path) throw Error(B200PIR_E_BADARG, "null argument");
  check_db(c, db);
  if (!db->whole()) throw Error(B200PIR_E_UNSUPPORTED, "save_file: a shard holds only part of the database (use download)");
  const std::vector<Member> ms = members(c, db);
  write_atomically(path, [&](FILE* f) {
    // a chunk of row shards is assembled from their exports first: host memory stays bounded by the staging
    std::vector<uint64_t> whole;
    export_impl(c, db, 0, c->slices, [&](int, int, int zc, const std::vector<const uint64_t*>& src) {
      const size_t n = (size_t)zc * c->num_per * c->dim0;
      const uint64_t* words = src[0];
      if (ms[0].store->shard.count != 1) {
        whole.resize(n);
        scatter_rows(c, ms, zc, src, whole.data());
        words = whole.data();
      }
      if (fwrite(words, 8, n, f) != n) throw Error(B200PIR_E_BADARG, std::strerror(errno));
    });
  });
  API_END
}
int b200pir_db_read_items(b200pir_ctx* c, b200pir_db* db, const uint64_t* db_idx, size_t count, uint8_t* out, uint8_t* flags) {
  API_BEGIN
  if (!c || (count && (!db_idx || !out))) throw Error(B200PIR_E_BADARG, "null argument");
  check_db(c, db);
  check_raw_params(c);
  const uint64_t num_items = (uint64_t)c->dim0 * c->num_per;
  const std::vector<Member> ms = members(c, db);
  for (size_t k = 0; k < count; k++) {
    if (db_idx[k] >= num_items) throw Error(B200PIR_E_SHAPE, "bad db idx " + std::to_string(db_idx[k]));
    if (!owner(ms, db_idx[k]))
      throw Error(B200PIR_E_SHAPE, "db idx " + std::to_string(db_idx[k]) + " lies in a row this shard does not hold");
  }
  const size_t span = (size_t)c->slices * c->bytes_per_chunk;
  read_items_impl(c, db, count, [&](size_t k) { return db_idx[k]; },
                  [&](size_t k0, size_t n, auto bytes, auto bits) {
                    for (size_t k = k0; k < k0 + n; k++) {
                      std::memcpy(out + k * span, bytes(k), span);
                      if (flags) flags[k] = bits(k);
                    }
                  });
  API_END
}
// The raw file b200pir_db_load_raw_file reads: item i's first db_item_size bytes at i * db_item_size.  When an item's span
// (slices * bytes_per_chunk) is longer than db_item_size, its last bytes are the next item's first ones in the file, so they
// must agree, and the last item's must be zero (load_raw_file reads zeros past the end of the file).
int b200pir_db_save_raw_file(b200pir_ctx* c, b200pir_db* db, const char* path) {
  API_BEGIN
  if (!c || !path) throw Error(B200PIR_E_BADARG, "null argument");
  check_db(c, db);
  check_raw_params(c);
  if (!db->whole()) throw Error(B200PIR_E_UNSUPPORTED, "save_raw_file: a shard holds only part of the database");
  const size_t num_items = (size_t)c->dim0 * c->num_per, isz = c->hp.db_item_size;
  const size_t span = (size_t)c->slices * c->bytes_per_chunk, tail = span - isz;   // span >= isz: bytes_per_chunk rounds up
  write_atomically(path, [&](FILE* f) {
    std::vector<uint8_t> carry(tail, 0), file;                // carry: the last `tail` bytes of the previous item
    read_items_impl(c, db, num_items, [](size_t k) { return (uint64_t)k; },
                    [&](size_t k0, size_t n, auto bytes, auto bits) {
                      file.resize(n * isz);
                      for (size_t i = k0; i < k0 + n; i++) {
                        const uint8_t fl = bits(i);
                        if (fl & B200PIR_ITEM_NOT_PLAINTEXT)
                          throw Error(B200PIR_E_UNSUPPORTED, "save_raw_file: item " + std::to_string(i) + " holds a coefficient that is not a byte");
                        if (fl & B200PIR_ITEM_PAST_CHUNK)
                          throw Error(B200PIR_E_UNSUPPORTED, "save_raw_file: item " + std::to_string(i) + " has bytes past bytes_per_chunk");
                        const uint8_t* b = bytes(i);
                        if (tail && i > 0 && std::memcmp(carry.data(), b, tail) != 0)
                          throw Error(B200PIR_E_UNSUPPORTED, "save_raw_file: the last bytes of item " + std::to_string(i - 1) +
                                                                 " differ from the first bytes of item " + std::to_string(i) + ", which the raw file shares");
                        std::memcpy(carry.data(), b + isz, tail);
                        std::memcpy(file.data() + (i - k0) * isz, b, isz);
                      }
                      if (k0 + n == num_items && std::any_of(carry.begin(), carry.end(), [](uint8_t v) { return v != 0; }))
                        throw Error(B200PIR_E_UNSUPPORTED, "save_raw_file: the last bytes of item " + std::to_string(num_items - 1) +
                                                               " lie past the end of the raw file and are not zero");
                      if (fwrite(file.data(), 1, file.size(), f) != file.size()) throw Error(B200PIR_E_BADARG, std::strerror(errno));
                    });
  });
  API_END
}
int b200pir_db_upsert_item(b200pir_ctx* c, b200pir_db* db, uint64_t slice, uint64_t item_idx, const uint64_t* poly) {
  API_BEGIN
  if (!c || !poly) throw Error(B200PIR_E_BADARG, "null argument");
  Guard gd(c, db);
  check_db(c, db);
  if (slice >= (uint64_t)c->slices || item_idx >= (uint64_t)c->dim0 * c->num_per) throw Error(B200PIR_E_SHAPE, "index out of range");
  const std::vector<Member> ms = members(c, db);
  std::vector<std::vector<ItemWrite>> written(ms.size());
  if (const std::optional<Owner> o = owner(ms, item_idx)) {
    b200pir_ctx* x = ms[o->g].ctx;
    B200_CUDA(cudaSetDevice(x->device));
    x->w_wbytes.ensure(b200pir_ctx::kWriteStageBytes);                     // the writers' staging, like RawWriter
    B200_CUDA(cudaMemcpyAsync(x->w_wbytes.p, poly, POLY * 8, cudaMemcpyHostToDevice, x->stream));
    launch_db_upsert(ms[o->g].store->layout, (int)slice, o->il, o->j, reinterpret_cast<const uint64_t*>(x->w_wbytes.p), x->stream);
    written[o->g].push_back(ItemWrite{0, 0, (uint32_t)o->il, (uint32_t)o->j});
  }
  settle(c, ms, (int)slice, (int)slice + 1, &written);
  API_END
}
int b200pir_db_update_item_raw(b200pir_ctx* c, b200pir_db* db, uint64_t db_idx, const uint8_t* data, size_t len) {
  API_BEGIN
  if (!c || (!data && len)) throw Error(B200PIR_E_BADARG, "null argument");
  Guard gd(c, db);
  check_db(c, db);
  check_raw_params(c);
  if (len > (size_t)c->slices * c->bytes_per_chunk) throw Error(B200PIR_E_SHAPE, "update longer than instances*n^2*bytes_per_chunk");   // loading.rs:308-310
  if (db_idx >= (uint64_t)c->dim0 * c->num_per) throw Error(B200PIR_E_SHAPE, "bad db idx");                      // loading.rs:333-340
  RawWriter w(c, db, false);                                                  // a group of one item
  w.add(db_idx, 0, (uint32_t)len);
  w.write(data, len);
  w.finish();
  API_END
}

// lib/server/src/db/loading.rs:361-377 update_many_items (the /update-row body).  The whole body is parsed on the host first
// (update_body.hpp); the valid prefix is applied and the error of the first bad entry, if any, returned afterwards, which is
// the database state the reference's entry-by-entry loop leaves.  Only the last occurrence of each db_idx is written, so how
// the entries are split into staging groups cannot change the result.  Every shard checks every entry and writes its own rows.
int b200pir_db_update_many_items(b200pir_ctx* c, b200pir_db* db, const uint8_t* body, size_t len, uint64_t* largest_update) {
  API_BEGIN
  if (!c || (!body && len)) throw Error(B200PIR_E_BADARG, "null argument");
  Guard gd(c, db);
  check_db(c, db);
  const BodyParse parsed = parse_update_body(body, len, 4 + (size_t)c->slices * c->bytes_per_chunk, (uint64_t)c->dim0 * c->num_per);
  // the reference reaches convert_pt_to_poly, which asserts logp == 8 (loading.rs:291), at the first well-formed entry
  if (c->hp.p != 256 && !parsed.entries.empty()) throw Error(B200PIR_E_UNSUPPORTED, "convert_pt_to_poly asserts logp == 8 (loading.rs:291)");
  if (c->bytes_per_chunk > (size_t)POLY && !parsed.entries.empty()) throw Error(B200PIR_E_SHAPE, "bytes_per_chunk exceeds poly_len");
  const std::vector<BodyEntry> kept = keep_last_occurrence(parsed.entries);
  RawWriter w(c, db, false);
  for (size_t k = 0; k < kept.size();) {
    // one staging group: whole entries in body order, their bytes (dropped duplicates in between included) within the budget
    const size_t k0 = k, base = kept[k].data_pos();
    size_t end = base;
    for (; k < kept.size() && !w.full; k++) {
      const size_t e = kept[k].data_pos() + kept[k].data_len();
      if (k > k0 && e - base > b200pir_ctx::kWriteStageBytes) break;
      end = e;
      w.add(kept[k].db_idx, kept[k].data_pos() - base, kept[k].data_len());
    }
    w.write(body + base, end - base);
  }
  w.finish();
  if (parsed.error) throw Error(parsed.error, parsed.message);
  if (largest_update) *largest_update = parsed.largest_update;
  API_END
}

// load_db_from_seek (lib/spiral-rs/src/server.rs:277-357; lib/server/src/db/loading.rs:192-247): `path` is the raw database,
// item i at byte i * db_item_size.  Chunk c of item i is the bytes_per_chunk bytes at i * db_item_size + c * bytes_per_chunk,
// clipped at the end of the FILE (as the reference's read does), each byte one plaintext coefficient; items past the end
// of the file are zero polynomials.  The file is read in groups of whole items (one read and one conversion-and-placement
// launch per group, within the writers' staging budget); an item's bytes may overlap the next item's, as its chunks do.
int b200pir_db_load_raw_file(b200pir_ctx* c, b200pir_db* db, const char* path) {
  API_BEGIN
  if (!c || !path) throw Error(B200PIR_E_BADARG, "null argument");
  Guard gd(c, db);
  check_db(c, db);
  if (c->hp.p != 256) throw Error(B200PIR_E_UNSUPPORTED, "load_item_from_seek is restated for logp == 8 only");
  if (c->bytes_per_chunk > (size_t)POLY) throw Error(B200PIR_E_SHAPE, "bytes_per_chunk exceeds poly_len");     // server.rs:292
  const auto [file, fbytes] = open_sized(path);
  if (fbytes < 0) throw Error(B200PIR_E_BADARG, "cannot size the database file");
  const size_t flen = (size_t)fbytes;
  const size_t num_items = (size_t)c->dim0 * c->num_per;
  const size_t item_span = (size_t)c->slices * c->bytes_per_chunk, isz = c->hp.db_item_size;
  const size_t group = std::max<size_t>(1, std::min(b200pir_ctx::kWriteStageItems,
                                                    b200pir_ctx::kWriteStageBytes / std::max<size_t>(1, std::max(isz, item_span))));
  RawWriter w(c, db, true);                                                   // load_db_from_seek builds a dense database
  std::vector<uint8_t> host;
  for (size_t i0 = 0; i0 < num_items; i0 += group) {
    const size_t cnt = std::min(group, num_items - i0);
    const size_t lo = i0 * isz, hi = std::min(flen, (i0 + cnt - 1) * isz + item_span);
    const size_t span = hi > lo ? hi - lo : 0;
    host.resize(span);
    if (span && (fseeko(file.get(), (off_t)lo, SEEK_SET) || fread(host.data(), 1, span, file.get()) != span))
      throw Error(B200PIR_E_SHAPE, "short read from the database file");
    for (size_t idx = i0; idx < i0 + cnt; idx++) {
      const size_t pos = idx * isz, len = pos < flen ? std::min(item_span, flen - pos) : 0;   // clipped at the end of the file
      w.add(idx, len ? pos - lo : 0, (uint32_t)len);
    }
    w.write(host.data(), span);                                               // one read, staged to every member
  }
  w.finish();
  API_END
}

int b200pir_db_present_items(b200pir_db* db, uint64_t* items, uint64_t* capacity) {
  API_BEGIN
  if (!db) throw Error(B200PIR_E_BADARG, "null db");
  uint64_t n = 0, cap = 0;
  for (const auto& p : db->parts) { n += p.store->present_count; cap += p.store->capacity(); }
  if (items) *items = n;
  if (capacity) *capacity = cap;
  API_END
}
int b200pir_db_info(b200pir_db* db, int* format, uint64_t* local_rows, uint64_t* hbm_bytes) {
  API_BEGIN
  if (!db) throw Error(B200PIR_E_BADARG, "null db");
  uint64_t rows = 0, bytes = 0;
  for (const auto& p : db->parts) { rows += p.store->rows; bytes += p.store->store.n; }
  if (format) *format = db->parts[0].store->layout.format;
  if (local_rows) *local_rows = rows;
  if (hbm_bytes) *hbm_bytes = bytes;
  API_END
}
int b200pir_db_fill_synthetic(b200pir_ctx* c, b200pir_db* db, uint64_t seed) {
  API_BEGIN
  if (!c) throw Error(B200PIR_E_BADARG, "null ctx");
  Guard gd(c, db);
  check_db(c, db);
  const std::vector<Member> ms = members(c, db);
  for (const Member& m : ms) {                                  // every member launches before any is waited on: distinct
    B200_CUDA(cudaSetDevice(m.ctx->device));                    // devices fill at the same time
    launch_write_synthetic(m.ctx->dp, m.store->layout, m.store->shard, seed, c->hp.p, m.ctx->stream);
  }
  settle(c, ms, 0, c->slices);
  API_END
}

}  // extern "C"
