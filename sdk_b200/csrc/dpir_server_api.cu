// C-ABI implementation of DoublePIR's answer() server (include/b200pir.h): the server state resident in HBM beside a matrix
// handle (or beside the row shards of one database, on one or several devices), answer() / answer_many on wire-format requests,
// and entry updates that patch the database, h_1 and the hint in place.
#include "dpir_api.hpp"
#include "dpir_wire.hpp"
#include <array>
#include <memory>
#include <string>

namespace {
// What a server keeps on the device of one database handle: the rows [r0, r0 + rows) of the database, the packed columns
// [r0 / 3x, r0 / 3x + c1) of h_1 and of a_1' (so the columns [r0 / x, r0 / x + 3 c1) of a_2^T and of every q_2), and the
// workspace of the passes over them.  An unsharded server has one, with r0 = 0 and rows = l (a chunk server's handle holds fewer
// rows; its batch is rows [0, its size) of the handle).
struct DpirShard {
  int device = 0, sm_count = 0;
  cudaStream_t stream = nullptr;
  cudaEvent_t done = nullptr;    // sharded: this shard's partial responses are complete
  b200pir_dpir* db = nullptr;    // borrowed
  uint64_t r0 = 0, rows = 0, c1 = 0, lx3 = 0, q2_off = 0;      // lx3 = 3 c1; q2_off = r0 / x: the first word of its q_2 slice
  DevBuf<uint32_t> h1, a2t;      // its columns of server_state, resident
  // workspace for max_queries queries: staged vectors + task tables (one upload), a_1 / a_1' / msg[0] per request
  size_t stage_cap = 0, task_cap = 0, vec_cap = 0, img_q2 = 0;
  uint8_t* h_stage = nullptr;
  DevBuf<uint8_t> d_stage;
  DevBuf<uint32_t> d_a1, d_a1sq, d_msg0;
  DevBuf<uint8_t> d_img;         // query images of the passes that run on the tensor cores (every q_1, then every q_2 slice)
  DevBuf<uint8_t> d_part;        // sharded, shards after the first: partial responses, little-endian, laid out as the responses
  // update scratch, allocated by the first update and grown only for a larger one: per group of at most upd_cap elements
  // (and as many rows), plus the tables of the whole batch and the hint
  size_t upd_cap = 0, upd_tab = 0;
  DevBuf<DpirUpdElem> u_el;
  DevBuf<DpirUpdRow> u_rows;
  DevBuf<int32_t> u_delta, u_D;
  DevBuf<uint32_t> u_dh1, u_a2g, u_dh2, u_h2;
  DevBuf<uint8_t> u_aimg, u_bimg;
  ~DpirShard() {
    cudaSetDevice(device);
    if (stream) {
      cudaStreamSynchronize(stream);
      cudaStreamDestroy(stream);
    }
    if (done) cudaEventDestroy(done);
    if (h_stage) cudaFreeHost(h_stage);
  }
};
}  // namespace

extern "C" {
// ---------------------------------------------------------------- DoublePIR online: answer() from HBM (dpir_serve.cu)
struct b200pir_dpir_server {
  int device = 0;                // shard 0's: where responses are summed and downloaded
  std::mutex mu;                 // calls stage through one workspace: serialised
  bool sharded = false;          // made by b200pir_dpir_server_create_sharded: no chunked answers
  uint64_t n = 0, l = 0, p = 0, delta = 0, x = 0, e = 0;       // e = ne / x: q_2 vectors a query
  uint64_t dx = 0, rows1 = 0, c1 = 0, dcols = 0, held = 0;     // delta x; n delta x; packed cols of h_1 and a_1'; db cols; rows held
  size_t max_queries = 0, img_q1 = 0;                          // img_q1: bytes of one q_1 image
  // the responses in wire layout (one download), and, with several shards, every shard's partials on shard 0's device
  size_t resp_cap = 0;
  uint8_t* h_resp = nullptr;
  DevBuf<uint8_t> d_resp, d_gather;
  b200pir_dpir_params params{};  // as created, with num_entries and bits_per_entry: an update checks them against the load
  uint64_t num_entries = 0, bits_per_entry = 0;
  DpirAesKey a1_key;             // SEED_A1's tables, expanded by the first update
  bool have_a1_key = false;
  std::vector<std::unique_ptr<DpirShard>> shards;
  ~b200pir_dpir_server() {
    shards.clear();
    cudaSetDevice(device);
    if (h_resp) cudaFreeHost(h_resp);
  }
};

namespace {
uint64_t ceil_div(uint64_t a, uint64_t b) { return (a + b - 1) / b; }

struct DpirCall {               // one request of a call
  const uint8_t* req;
  DpirWireRequest w;
  DpirResponseLayout L;
  size_t resp_off = 0;          // byte offset of its response in d_resp
  // device addresses of its staged vectors ([k], [k * e + j]) on the shard being planned; q1[k] null when not read, and its
  // query image when the database pass runs on the tensor cores
  std::vector<const uint32_t*> q1, q2;
};

// Parse + the checks of doublepir.rs:246-350 for one request; chunk < 0: unchunked.
int dpir_prepare_call(b200pir_dpir_server* S, const uint8_t* req, size_t len, int64_t chunk, DpirCall& c, std::string& err) {
  c.req = req;
  int rc = parse_dpir_request(req, len, S->e, S->c1, c.w, err);
  if (!rc) rc = check_dpir_batches(c.w, S->l, S->held, S->dcols, chunk, err);
  c.L = DpirResponseLayout{c.w.queries, S->e, S->dx, S->n, S->rows1};
  return rc;
}

// The passes of answer() over shard D's rows for every request of `calls`, on D's stream, into the responses at `resp` (device,
// laid out as the call's responses).  partial: data words as little-endian partial sums, the headers left as zeros; otherwise
// the responses' data words in wire order.  Everything has been checked; no allocation, no synchronisation, one upload.
void dpir_serve_shard(b200pir_dpir_server* S, DpirShard& D, std::vector<DpirCall>& calls, int64_t chunk, uint8_t* resp,
                      size_t resp_total, bool partial) {
  const size_t R = calls.size();
  B200_CUDA(cudaSetDevice(D.device));
  cudaStream_t s = D.stream;
  const uint64_t r0 = D.r0, r1 = D.r0 + D.rows;
  // ---- which kernel the database pass runs, from the vectors it holds and the matrix rows
  const bool tc_db = dpir_use_tc(chunk >= 0 ? 1 : R, chunk >= 0 ? dpir_batch_rows(S->l, calls[0].w.queries, chunk) : D.rows);
  // ---- stage the vectors the passes read (the request's bytes as they are: big-endian words, swapped by the kernels): every
  // q_1 whole, and this shard's slice of every q_2; a database pass on the tensor cores reads query images of its q_1 instead
  DpirMvPlan plan;
  size_t off = 0, n1 = 0, n2 = 0;
  auto stage = [&](const DpirCall& c, size_t pos, uint64_t words) {
    const size_t bytes = (size_t)words * 4;
    if (off + bytes > D.stage_cap) throw Error(B200PIR_E_SHAPE, "dpir: staging overflow");
    std::memcpy(D.h_stage + off, c.req + pos, bytes);
    const uint32_t* dev = reinterpret_cast<const uint32_t*>(D.d_stage.p + off);
    off = align_up(off + bytes, 16);
    return dev;
  };
  uint64_t total_q = 0;
  for (auto& c : calls) {
    total_q += c.w.queries;
    c.q1.assign(c.w.queries, nullptr);
    c.q2.assign(c.w.queries * S->e, nullptr);
    for (size_t k = 0; k < c.w.queries; k++) {
      if (chunk < 0 || (uint64_t)chunk == k) c.q1[k] = stage(c, c.w.q1(k).data_pos(), c.w.q1(k).rows);
      if (tc_db && c.q1[k]) c.q1[k] = plan.image(c.q1[k], D.d_img.p + n1++ * S->img_q1, S->dcols);
      for (size_t j = 0; j < S->e; j++) c.q2[k * S->e + j] = stage(c, c.w.q2(k, j).data_pos() + 4 * D.q2_off, 3 * D.c1);
    }
  }
  // ---- task tables: database pass, h_1 pass (on the tensor cores, from query images, by the same rule), a_1' * q_2
  DpirMvPass db_pass = plan.pass(tc_db, S->dcols);
  if (chunk >= 0) {             // one request: batch `chunk` from rows [0, its size) of the server's matrix
    const uint64_t nq = calls[0].w.queries;
    plan.vecs.push_back(DpirMvVec{calls[0].q1[chunk], D.d_a1.p + dpir_batch_begin(S->l, nq, chunk)});
    plan.add(db_pass, D.db->a.p, dpir_batch_rows(S->l, nq, chunk), 1);
  } else {                      // the shard's rows cut at every request's batch boundaries: one q_1 per request in each segment
    std::vector<uint64_t> cuts{r0, r1};
    for (const auto& c : calls)
      for (uint64_t k = 1; k < c.w.queries; k++) {
        const uint64_t b = dpir_batch_begin(S->l, c.w.queries, k);
        if (b > r0 && b < r1) cuts.push_back(b);
      }
    std::sort(cuts.begin(), cuts.end());
    cuts.erase(std::unique(cuts.begin(), cuts.end()), cuts.end());
    for (size_t g = 0; g + 1 < cuts.size(); g++) {
      const uint64_t s0 = cuts[g], s1 = cuts[g + 1];
      for (size_t i = 0; i < R; i++) {
        const uint64_t nq = calls[i].w.queries, bs = S->l / nq;
        const uint64_t k = bs ? std::min(s0 / bs, nq - 1) : nq - 1;
        plan.vecs.push_back(DpirMvVec{calls[i].q1[k], D.d_a1.p + i * D.rows + (s0 - r0)});
      }
      plan.add(db_pass, D.db->a.p + (s0 - r0) * S->dcols, s1 - s0, R);
    }
  }
  const bool tc_h1 = dpir_use_tc(total_q * S->e, S->rows1);
  DpirMvPass h1_pass = plan.pass(tc_h1, D.c1);
  for (const auto& c : calls)
    for (size_t k = 0; k < c.w.queries; k++)
      for (size_t j = 0; j < S->e; j++) {
        const uint32_t* b = c.q2[k * S->e + j];
        if (tc_h1) b = plan.image(b, D.d_img.p + S->max_queries * S->img_q1 + n2++ * D.img_q2, D.c1);
        plan.vecs.push_back(DpirMvVec{b, reinterpret_cast<uint32_t*>(resp + c.resp_off + c.L.a2_data(k, j))});
      }
  plan.add(h1_pass, D.h1.p, S->rows1, total_q * S->e);
  if (n1 > S->max_queries || n2 > S->max_queries * S->e) throw Error(B200PIR_E_SHAPE, "dpir: query image workspace overflow");
  DpirMvPass a1_pass = plan.pass(false, D.c1);
  for (size_t i = 0; i < R; i++) {
    const DpirCall& c = calls[i];
    for (size_t k = 0; k < c.w.queries; k++)
      for (size_t j = 0; j < S->e; j++)
        plan.vecs.push_back(DpirMvVec{c.q2[k * S->e + j], reinterpret_cast<uint32_t*>(resp + c.resp_off + c.L.h2_data(k, j))});
    plan.add(a1_pass, D.d_a1sq.p + i * S->dx * D.c1, S->dx, c.w.queries * S->e);
  }
  if (plan.tasks.size() > D.task_cap || plan.vecs.size() > D.vec_cap) throw Error(B200PIR_E_SHAPE, "dpir: task table overflow");
  const size_t used = off + plan.bytes();
  if (used > D.stage_cap) throw Error(B200PIR_E_SHAPE, "dpir: staging overflow");
  plan.place(D.h_stage + off, D.d_stage.p + off);
  // ---- the passes: the h_1 and a_1' passes store their results whole (big-endian, or partials), so they never split k; the
  // database pass adds into zeroed a_1
  const int out_be = partial ? 0 : DPIR_MV_OUT_BE;
  B200_CUDA(cudaMemcpyAsync(D.d_stage.p, D.h_stage, used, cudaMemcpyHostToDevice, s));
  if (partial) B200_CUDA(cudaMemsetAsync(resp, 0, resp_total, s));   // header words stay zero: the sum leaves them to the host
  B200_CUDA(cudaMemsetAsync(D.d_a1.p, 0, R * D.rows * 4, s));   // split-k partial sums add into it; unread batches stay zero
  launch_dpir_tc_image(plan.d_jobs, plan.jobs.size(), std::max(S->dcols, D.c1), DPIR_MV_B_BE, s);
  plan.launch(db_pass, true, D.sm_count, DPIR_MV_B_BE, s);
  for (size_t i = 0; i < R; i++)        // a_1.transpose_expand_concat_cols_squish(p, delta, x, 10, 3)
    launch_dpir_transpose_expand(D.d_a1sq.p + i * S->dx * D.c1, D.d_a1.p + i * D.rows, D.rows, 1, S->p, S->delta, S->x, S->dx,
                                 D.c1, s);
  // msg[0] = matrix_mul_transposed_packed(a_1', a_2^T) of every request at once (their a_1' are stacked)
  launch_dpir_mul_transposed(D.d_msg0.p, D.d_a1sq.p, D.a2t.p, R * S->dx, D.c1, S->n, D.lx3, s);
  for (size_t i = 0; i < R; i++) {
    uint8_t* m0 = resp + calls[i].resp_off + calls[i].L.msg0_data();
    if (partial) B200_CUDA(cudaMemcpyAsync(m0, D.d_msg0.p + i * S->dx * S->n, S->dx * S->n * 4, cudaMemcpyDeviceToDevice, s));
    else launch_dpir_bswap(reinterpret_cast<uint32_t*>(m0), D.d_msg0.p + i * S->dx * S->n, S->dx * S->n, s);
  }
  plan.launch(h1_pass, false, D.sm_count, DPIR_MV_B_BE | out_be, s);
  plan.launch(a1_pass, false, D.sm_count, DPIR_MV_B_BE | out_be, s);
  if (partial) B200_CUDA(cudaEventRecord(D.done, s));
  B200_CUDA(cudaGetLastError());
}

// answer() for every request of `calls`; responses to outs[i].  One shard: its passes store the responses.  Several: each
// shard's partials (shard 0's straight into the gather buffer) go to shard 0's device with cudaMemcpyPeerAsync (the copy
// engines; no peer access needed), after its passes, and one kernel sums them mod 2^32 into the big-endian responses.  One
// download; synchronises shard 0's stream, which has waited for every shard.
void dpir_serve(b200pir_dpir_server* S, std::vector<DpirCall>& calls, int64_t chunk, uint8_t* const* outs, size_t* out_lens) {
  const size_t R = calls.size(), G = S->shards.size();
  size_t resp_total = 0;
  for (auto& c : calls) {
    c.resp_off = resp_total;
    resp_total += c.L.bytes();
  }
  if (resp_total > S->resp_cap) throw Error(B200PIR_E_SHAPE, "dpir: response workspace overflow");
  for (size_t g = 0; g < G; g++) {
    DpirShard& D = *S->shards[g];
    uint8_t* resp = G == 1 ? S->d_resp.p : g == 0 ? S->d_gather.p : D.d_part.p;
    dpir_serve_shard(S, D, calls, chunk, resp, resp_total, G > 1);
  }
  DpirShard& H = *S->shards[0];
  B200_CUDA(cudaSetDevice(H.device));
  if (G > 1) {
    for (size_t g = 1; g < G; g++) {
      const DpirShard& D = *S->shards[g];
      B200_CUDA(cudaStreamWaitEvent(H.stream, D.done, 0));
      B200_CUDA(cudaMemcpyPeerAsync(S->d_gather.p + g * S->resp_cap, H.device, D.d_part.p, D.device, resp_total, H.stream));
    }
    launch_dpir_sum_be(reinterpret_cast<uint32_t*>(S->d_resp.p), reinterpret_cast<const uint32_t*>(S->d_gather.p), S->resp_cap / 4,
                       G, resp_total / 4, H.stream);
  }
  B200_CUDA(cudaGetLastError());
  B200_CUDA(cudaMemcpyAsync(S->h_resp, S->d_resp.p, resp_total, cudaMemcpyDeviceToHost, H.stream));
  B200_CUDA(cudaStreamSynchronize(H.stream));
  B200_CUDA(cudaGetLastError());
  for (size_t i = 0; i < R; i++) {
    const DpirCall& c = calls[i];
    std::memcpy(outs[i], S->h_resp + c.resp_off, c.L.bytes());
    write_dpir_response_headers(c.L, outs[i]);
    out_lens[i] = c.L.bytes();
  }
}

// A server over the database handles dbs, handle g holding the rows [r0[g], r0[g] + rows[g]) (one handle: r0 = 0, rows = l).
// Everything about the handles has been checked; h1_squished / a2_t are the whole host matrices, of which each shard uploads its
// column band.
b200pir_dpir_server* dpir_server_new(const b200pir_dpir_params* params, uint64_t num_entries, uint64_t bits_per_entry,
                                     const b200pir_dpir_info& info, const std::vector<b200pir_dpir*>& dbs,
                                     const std::vector<DpirShardRows>& spans, const uint32_t* h1_squished, const uint32_t* a2_t,
                                     size_t max_queries, bool sharded) {
  const size_t G = dbs.size();
  std::unique_ptr<b200pir_dpir_server> S(new b200pir_dpir_server());
  S->device = dbs[0]->device;
  S->sharded = sharded;
  S->params = *params;
  S->num_entries = num_entries;
  S->bits_per_entry = bits_per_entry;
  S->n = params->n; S->l = params->l; S->p = params->p; S->delta = info.delta; S->x = info.x; S->e = info.ne / info.x;
  S->dx = info.delta * info.x; S->rows1 = S->n * S->dx; S->c1 = (S->l / S->x + 2) / 3; S->dcols = dbs[0]->cols;
  S->held = sharded ? S->l : dbs[0]->rows;
  S->max_queries = max_queries;
  S->img_q1 = dtc_img_bytes(S->dcols);
  const uint64_t Q = max_queries, e = S->e, lx3 = 3 * S->c1;
  S->resp_cap = Q * (12 + S->dx * S->n * 4) + Q * e * DpirResponseLayout{1, e, S->dx, S->n, S->rows1}.pair_bytes();
  for (size_t g = 0; g < G; g++) {
    S->shards.emplace_back(new DpirShard());
    DpirShard& D = *S->shards.back();
    D.device = dbs[g]->device;
    use_device(D.device);
    D.db = dbs[g];
    D.r0 = spans[g].begin;
    D.rows = spans[g].rows;
    D.c1 = (D.rows / S->x + 2) / 3;
    D.lx3 = 3 * D.c1;
    D.q2_off = D.r0 / S->x;
    const uint64_t c1_off = D.r0 / (3 * S->x);
    B200_CUDA(cudaDeviceGetAttribute(&D.sm_count, cudaDevAttrMultiProcessorCount, D.device));
    B200_CUDA(cudaStreamCreateWithFlags(&D.stream, cudaStreamNonBlocking));
    if (G > 1) B200_CUDA(cudaEventCreateWithFlags(&D.done, cudaEventDisableTiming));
    // bounds of one call: at most Q requests and Q queries; the database pass has at most Q row segments (each request of k
    // queries adds k - 1 cuts), each tiled and repeated once per pass of vectors.  A pass on k_dpir_matvec_multi (32 rows a
    // task, 16 vectors a pass) makes at least as many tasks as one on the tensor cores (64 rows, 64 vectors), so its count
    // bounds both.
    D.task_cap = (ceil_div(D.rows, kDpirMvRows) + Q) * ceil_div(Q, kDpirMvMaxVecs)
               + ceil_div(S->rows1, kDpirMvRows) * ceil_div(Q * e, kDpirMvMaxVecs)
               + ceil_div(S->dx, kDpirMvRows) * Q * e;
    D.vec_cap = Q * Q + 2 * Q * e;
    D.stage_cap = Q * (align_up(3 * S->dcols * 4, 16) + e * align_up(3 * D.c1 * 4, 16)) + align_up(D.task_cap * sizeof(DpirMvTask), 16)
                + align_up(D.vec_cap * sizeof(DpirMvVec), 16) + Q * (1 + e) * sizeof(DpirTcImage);
    D.img_q2 = dtc_img_bytes(D.c1);
    B200_CUDA(cudaMallocHost(&D.h_stage, D.stage_cap));
    D.d_stage.alloc(D.stage_cap);
    D.d_a1.alloc(Q * D.rows);
    D.d_a1sq.alloc(Q * S->dx * D.c1);
    D.d_msg0.alloc(Q * S->dx * S->n);
    D.d_img.alloc(Q * S->img_q1 + Q * e * D.img_q2);
    if (G > 1 && g > 0) D.d_part.alloc(S->resp_cap);
    D.h1.alloc(S->rows1 * D.c1);
    D.a2t.alloc(S->n * D.lx3);
    B200_CUDA(cudaMemcpy2DAsync(D.h1.p, D.c1 * 4, h1_squished + c1_off, S->c1 * 4, D.c1 * 4, S->rows1, cudaMemcpyHostToDevice, D.stream));
    B200_CUDA(cudaMemcpy2DAsync(D.a2t.p, D.lx3 * 4, a2_t + 3 * c1_off, lx3 * 4, D.lx3 * 4, S->n, cudaMemcpyHostToDevice, D.stream));
    B200_CUDA(cudaStreamSynchronize(D.stream));
  }
  use_device(S->device);
  B200_CUDA(cudaMallocHost(&S->h_resp, S->resp_cap));
  S->d_resp.alloc(S->resp_cap);
  if (G > 1) S->d_gather.alloc(G * S->resp_cap);
  return S.release();
}
}  // namespace

int b200pir_dpir_server_create(int device, const b200pir_dpir_params* params, uint64_t num_entries, uint64_t bits_per_entry,
                               b200pir_dpir* db, const uint32_t* h1_squished, const uint32_t* a2_t, size_t max_queries,
                               b200pir_dpir_server** out) {
  API_BEGIN
  if (!params || !db || !h1_squished || !a2_t || !out) throw Error(B200PIR_E_BADARG, "null argument");
  if (max_queries == 0 || max_queries >= kDpirWireMaxLen) throw Error(B200PIR_E_BADARG, "max_queries must lie in [1, 2^28)");
  const b200pir_dpir_info info = dpir_info(params, num_entries, bits_per_entry, 64);
  if (device != db->device) throw Error(B200PIR_E_BADARG, "the database lives on another device");
  const uint64_t l = params->l, x = info.x;
  if (l % x) throw Error(B200PIR_E_SHAPE, "l must be a multiple of x (concat_cols)");
  if (db->cols != (params->m + 2) / 3) throw Error(B200PIR_E_SHAPE, "the database's packed columns are not ceil(m / 3)");
  if (db->rows > l) throw Error(B200PIR_E_SHAPE, "the database has more than l rows");
  use_device(device);
  *out = dpir_server_new(params, num_entries, bits_per_entry, info, {db}, {DpirShardRows{0, l}}, h1_squished, a2_t, max_queries, false);
  API_END
}

int b200pir_dpir_server_create_sharded(const b200pir_dpir_params* params, uint64_t num_entries, uint64_t bits_per_entry,
                                       b200pir_dpir* const* dbs, size_t shards, const uint32_t* h1_squished, const uint32_t* a2_t,
                                       size_t max_queries, b200pir_dpir_server** out) {
  API_BEGIN
  if (!params || !dbs || !h1_squished || !a2_t || !out) throw Error(B200PIR_E_BADARG, "null argument");
  for (size_t g = 0; g < shards; g++)
    if (!dbs[g]) throw Error(B200PIR_E_BADARG, "null shard " + std::to_string(g));
  if (max_queries == 0 || max_queries >= kDpirWireMaxLen) throw Error(B200PIR_E_BADARG, "max_queries must lie in [1, 2^28)");
  const b200pir_dpir_info info = dpir_info(params, num_entries, bits_per_entry, 64);
  const uint64_t l = params->l, x = info.x;
  if (l % x) throw Error(B200PIR_E_SHAPE, "l must be a multiple of x (concat_cols)");
  if (shards == 0) throw Error(B200PIR_E_SHAPE, "no shards");
  std::vector<b200pir_dpir*> v(dbs, dbs + shards);
  std::vector<DpirShardRows> spans;
  uint64_t end = 0;
  for (size_t g = 0; g < shards; g++) {
    const b200pir_dpir* d = dbs[g];
    if (d->cols != (params->m + 2) / 3) throw Error(B200PIR_E_SHAPE, "shard " + std::to_string(g) + ": packed columns are not ceil(m / 3)");
    if (d->row_begin != end)
      throw Error(B200PIR_E_SHAPE, "shard " + std::to_string(g) + " begins at row " + std::to_string(d->row_begin) + ", not at " +
                                       std::to_string(end) + ": the shards must tile [0, l) in order");
    if (d->row_begin % (3 * x)) throw Error(B200PIR_E_SHAPE, "shard " + std::to_string(g) + " begins off a multiple of 3x rows");
    if (d->rows > l - end) throw Error(B200PIR_E_SHAPE, "shard " + std::to_string(g) + " runs past row l");
    spans.push_back(DpirShardRows{d->row_begin, d->rows});
    end += d->rows;
  }
  if (end != l) throw Error(B200PIR_E_SHAPE, "the shards end at row " + std::to_string(end) + ", not at l");
  for (size_t g = 0; g < shards; g++) use_device(dbs[g]->device);
  *out = dpir_server_new(params, num_entries, bits_per_entry, info, v, spans, h1_squished, a2_t, max_queries, true);
  API_END
}

void b200pir_dpir_server_destroy(b200pir_dpir_server* S) {
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
  if (S->sharded && chunk_idx >= 0)
    throw Error(B200PIR_E_UNSUPPORTED, "a sharded server holds every row: chunked answers are for a server holding one batch");
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

// Store, h_1 and hint patches of every group on shard D's stream, its elements' rows local to the shard; h2 (host, (n delta x) x
// n) in and out.  Synchronises.
void dpir_update(b200pir_dpir_server* S, DpirShard& D, const std::vector<DpirUpdElem>& el, uint32_t* h2) {
  B200_CUDA(cudaSetDevice(D.device));
  const cudaStream_t s = D.stream;
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
  if (cap > D.upd_cap) {
    D.u_dh1.alloc(cap * n);
    D.u_a2g.alloc(cap * n);
    D.u_D.alloc(nd * cap);
    D.u_aimg.alloc(dpir_gemm_a_bytes(nd, cap));
    D.u_bimg.alloc(dpir_gemm_b_bytes(cap, n));
    D.upd_cap = cap;
  }
  if (el.size() > D.upd_tab) {
    D.u_el.alloc(el.size());
    D.u_rows.alloc(el.size());
    D.u_delta.alloc(el.size());
    D.upd_tab = el.size();
  }
  D.u_dh2.ensure(nd * n);
  D.u_h2.ensure(nd * x * n);
  if (!S->have_a1_key) {
    S->a1_key = dpir_aes_key(kDpirSeedA1);
    S->have_a1_key = true;
  }
  b200pir_dpir* db = D.db;
  B200_CUDA(cudaStreamSynchronize(db->stream));          // work still queued on the database handle's own stream first
  B200_CUDA(cudaMemcpyAsync(D.u_el.p, el.data(), el.size() * sizeof(DpirUpdElem), cudaMemcpyHostToDevice, s));
  B200_CUDA(cudaMemcpyAsync(D.u_rows.p, rows.data(), rows.size() * sizeof(DpirUpdRow), cudaMemcpyHostToDevice, s));
  B200_CUDA(cudaMemcpyAsync(D.u_h2.p, h2, nd * x * n * 4, cudaMemcpyHostToDevice, s));
  for (const DpirUpdGroup& G : groups) {
    const DpirUpdElem* gel = D.u_el.p + G.e_off;
    const DpirUpdRow* grows = D.u_rows.p + G.r_off;
    int32_t* gdelta = D.u_delta.p + G.e_off;
    launch_dpir_upd_store(db->a.p, db->cols, gel, (uint32_t)G.n_el, gdelta, s);
    launch_dpir_upd_dh1(D.u_dh1.p, grows, (uint32_t)G.n_rows, gel, gdelta, n, S->a1_key, s);
    launch_dpir_upd_digits(D.h1.p, D.c1, D.u_D.p, grows, (uint32_t)G.n_rows, D.u_dh1.p, n, (uint32_t)S->p, (uint32_t)S->delta, x, s);
    launch_dpir_upd_gather_a2(D.u_a2g.p, D.a2t.p, D.lx3, grows, (uint32_t)G.n_rows, n, x, s);
    for (const auto& B : G.blocks) {                     // dh_2[block b] = D_b (nd x k_b) * A_2 rows (k_b x n)
      const uint64_t b = B[0], k0 = B[1], kb = B[2];
      launch_dpir_gemm_b_image(D.u_bimg.p, D.u_a2g.p + k0 * n, kb, n, s);
      launch_dpir_gemm_rows(D.u_dh2.p, D.u_aimg.p, reinterpret_cast<const uint32_t*>(D.u_D.p) + nd * k0, nd, kb, D.u_bimg.p, n, s);
      launch_dpir_upd_add(D.u_h2.p + b * nd * n, D.u_dh2.p, nd * n, s);
    }
  }
  B200_CUDA(cudaGetLastError());
  B200_CUDA(cudaMemcpyAsync(h2, D.u_h2.p, nd * x * n * 4, cudaMemcpyDeviceToHost, s));
  B200_CUDA(cudaStreamSynchronize(s));
  B200_CUDA(cudaGetLastError());
}
}  // namespace

int b200pir_dpir_server_update(b200pir_dpir_server* S, const uint64_t* indices, const uint8_t* values, size_t count, uint32_t* h2) {
  API_BEGIN
  if (!S || !h2 || (count && (!indices || !values))) throw Error(B200PIR_E_BADARG, "null argument");
  b200pir_dpir* db = S->shards[0]->db;
  for (const auto& D : S->shards) {
    const b200pir_dpir* d = D->db;
    if (!d->from_load) throw Error(B200PIR_E_UNSUPPORTED, "update: the server's database was not laid out by b200pir_dpir_load*");
    if (!S->sharded && d->rows < S->l) throw Error(B200PIR_E_UNSUPPORTED, "update: the server holds a chunk of the database (fewer than l rows)");
    if (!d->fields_exact)
      throw Error(B200PIR_E_UNSUPPORTED, "update: the load packed entries wider than bits_per_entry; its elements do not decode field by field");
    const b200pir_dpir_params& P = d->params;
    if (S->num_entries != d->num_entries || S->bits_per_entry != d->bits_per_entry || S->params.n != P.n || S->params.l != P.l ||
        S->params.m != P.m || S->params.logq != P.logq || S->params.p != P.p || d->entry_format != db->entry_format ||
        d->load_count != db->load_count)
      throw Error(B200PIR_E_SHAPE, "update: the server's parameters, num_entries or bits_per_entry differ from its database's load");
  }
  if (S->n * 4 > 200 * 1024) throw Error(B200PIR_E_UNSUPPORTED, "update: n above 51200");
  const b200pir_dpir_info info = dpir_info(&db->params, db->num_entries, db->bits_per_entry);
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
  std::vector<std::unique_lock<std::mutex>> lk_db;
  for (const auto& D : S->shards) lk_db.emplace_back(D->db->mu);
  if (S->shards.size() == 1) {
    dpir_update(S, *S->shards[0], el, h2);
  } else {                      // each shard patches its own elements, rows rebased to its first; h2 passes through each in turn
    size_t k = 0;
    for (const auto& D : S->shards) {
      std::vector<DpirUpdElem> mine;
      for (; k < el.size() && el[k].r < D->r0 + D->rows; k++) mine.push_back(DpirUpdElem{el[k].r - D->r0, el[k].c, el[k].mask, el[k].val});
      if (!mine.empty()) dpir_update(S, *D, mine, h2);
    }
  }
  cudaSetDevice(S->device);
  API_END
}

int b200pir_dpir_server_state(b200pir_dpir_server* S, uint32_t* h1_squished) {
  API_BEGIN
  if (!S || !h1_squished) throw Error(B200PIR_E_BADARG, "null argument");
  std::lock_guard<std::mutex> lk(S->mu);
  for (const auto& D : S->shards) {
    B200_CUDA(cudaSetDevice(D->device));
    B200_CUDA(cudaMemcpy2DAsync(h1_squished + D->r0 / (3 * S->x), S->c1 * 4, D->h1.p, D->c1 * 4, D->c1 * 4, S->rows1,
                                cudaMemcpyDeviceToHost, D->stream));
    B200_CUDA(cudaStreamSynchronize(D->stream));
  }
  cudaSetDevice(S->device);
  B200_CUDA(cudaGetLastError());
  API_END
}

}  // extern "C"
