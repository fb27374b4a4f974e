// What the DoublePIR translation units (dpir_api.cu: the matrix handle, the one-shot ops and the offline load;
// dpir_server_api.cu: the answer() server and entry updates) share: the matrix handle, an owned stream, the DbInfo shape, the
// A_1 seed and the planner of the packed matrix x vectors passes.
#pragma once
#include "api_internal.hpp"
#include "dpir_kernels.h"
#include <algorithm>
#include <cstring>
#include <mutex>
#include <vector>

using namespace b200pir;     // the handle struct below lives outside the namespace, as the C ABI names it

struct b200pir_dpir {
  int device;
  std::mutex mu;            // calls on one handle stage through its b / out buffers: serialised
  cudaStream_t stream = nullptr;
  bool own_stream = true;
  uint64_t rows, cols;
  uint64_t row_begin = 0;   // the layout row of row 0: nonzero for a row shard (b200pir_dpir_load*_sharded, b200pir_dpir_create_shard)
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

namespace b200pir {

// A non-blocking stream owned by one scope: destroyed when the scope is left, unless release()d to a longer-lived owner
struct OwnedStream {
  cudaStream_t s = nullptr;
  OwnedStream() { B200_CUDA(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking)); }
  ~OwnedStream() { if (s) cudaStreamDestroy(s); }
  cudaStream_t release() { cudaStream_t r = s; s = nullptr; return r; }
  OwnedStream(const OwnedStream&) = delete;
  OwnedStream& operator=(const OwnedStream&) = delete;
};

const uint8_t kDpirSeedA1[16] = B200PIR_DPIR_SEED_A1;

// DbInfo::new (database.rs:58-90) with num_db_entries (:352-372) and compute_num_entries_base_p (:345-350); Params::delta().
// max_bits: 63 where entries are laid out; the server, which only needs the shape, takes full 64-bit entries too.
b200pir_dpir_info dpir_info(const b200pir_dpir_params* prm, uint64_t num_entries, uint64_t bits, uint64_t max_bits = 63);

inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

// The row split of a sharded database (b200pir_dpir_shard_rows): the l rows fall into units of 3x rows, the last one clipped at
// l, and shard g of G takes the next floor(U / G) units, one more when g < U mod G.  Edges on multiples of 3x keep every packed
// column of h_1', a_1' and a_2^T (three l/x positions a word) inside one shard.  {row_begin, rows}; throws B200PIR_E_SHAPE for
// G = 0 or more shards than units.
struct DpirShardRows { uint64_t begin, rows; };
DpirShardRows dpir_shard_rows(uint64_t l, uint64_t x, size_t shards, size_t index);

// One pass of packed matrix x vectors: on the tensor cores (tc: tasks of DTC_ROWS rows and up to DTC_VECS vectors, whose b are
// query images) or on k_dpir_matvec_multi (kDpirMvRows rows, up to kDpirMvMaxVecs vectors); its tasks are [t0, t1) of its plan
// and vmax the most vectors any of them holds
struct DpirMvPass {
  bool tc;
  uint64_t cols;            // packed words a matrix row
  size_t t0, t1;
  int vmax;
};

// The task and vector tables of one call's passes, and the jobs that make the query images its tensor-core passes read (in
// slots the caller picks), laid out in one host block so that one upload moves them
struct DpirMvPlan {
  std::vector<DpirMvTask> tasks;
  std::vector<DpirMvVec> vecs;
  std::vector<DpirTcImage> jobs;
  const DpirMvTask* d_tasks = nullptr;    // where the tables land on the device (place())
  const DpirMvVec* d_vecs = nullptr;
  const DpirTcImage* d_jobs = nullptr;

  // a pass that starts after the plan's last task; add() its vectors before the next pass begins
  DpirMvPass pass(bool tc, uint64_t cols) const { return DpirMvPass{tc, cols, tasks.size(), tasks.size(), 1}; }
  // the last n vectors appended to vecs against the rows [0, rows) of the packed matrix a: per group of at most DTC_VECS /
  // kDpirMvMaxVecs of them, one task for each tile of rows
  void add(DpirMvPass& P, const uint32_t* a, uint64_t rows, size_t n) {
    const size_t cap = P.tc ? DTC_VECS : kDpirMvMaxVecs;
    const uint64_t tr = P.tc ? DTC_ROWS : kDpirMvRows;
    for (size_t v0 = vecs.size() - n; v0 < vecs.size(); v0 += cap) {
      const uint32_t nv = (uint32_t)std::min(cap, vecs.size() - v0);
      P.vmax = std::max<int>(P.vmax, nv);
      for (uint64_t r0 = 0; r0 < rows; r0 += tr)
        tasks.push_back(DpirMvTask{a + r0 * P.cols, (uint32_t)std::min<uint64_t>(tr, rows - r0), (uint32_t)v0, nv, (uint32_t)r0});
    }
    P.t1 = tasks.size();
  }
  // a job that makes the query image img (for a pass on the tensor cores) of the vector b, cols packed words wide; the image
  // is what the pass reads
  const uint32_t* image(const uint32_t* b, uint8_t* img, uint64_t cols) {
    jobs.push_back(DpirTcImage{b, img, (uint32_t)cols});
    return reinterpret_cast<const uint32_t*>(img);
  }
  // the tables as place() lays them out: tasks, then vectors and jobs, each from a 16-byte boundary
  size_t vecs_at() const { return align_up(tasks.size() * sizeof(DpirMvTask), 16); }
  size_t jobs_at() const { return align_up(vecs_at() + vecs.size() * sizeof(DpirMvVec), 16); }
  size_t bytes() const { return jobs_at() + jobs.size() * sizeof(DpirTcImage); }
  // the tables into host block h (bytes() long), and where they are once the block has been uploaded to d (16-byte aligned)
  void place(uint8_t* h, uint8_t* d) {
    std::memcpy(h, tasks.data(), tasks.size() * sizeof(DpirMvTask));
    std::memcpy(h + vecs_at(), vecs.data(), vecs.size() * sizeof(DpirMvVec));
    std::memcpy(h + jobs_at(), jobs.data(), jobs.size() * sizeof(DpirTcImage));
    d_tasks = reinterpret_cast<const DpirMvTask*>(d);
    d_vecs = reinterpret_cast<const DpirMvVec*>(d + vecs_at());
    d_jobs = reinterpret_cast<const DpirTcImage*>(d + jobs_at());
  }
  // pass P, its k range split over the SMs when `split` is set (only a pass that adds into zeroed outputs may split k)
  void launch(const DpirMvPass& P, bool split, int sm_count, int flags, cudaStream_t s) const {
    const size_t n = P.t1 - P.t0;
    if (P.tc) launch_dpir_matvec_tc(d_tasks + P.t0, n, d_vecs, P.cols, split ? dpir_tc_ksplit(n, P.cols, sm_count) : 1, flags, s);
    else launch_dpir_matvec_multi(d_tasks + P.t0, n, d_vecs, P.cols, P.vmax, split ? dpir_mv_ksplit(n, P.cols, sm_count) : 1, flags, s);
  }
};

}  // namespace b200pir
