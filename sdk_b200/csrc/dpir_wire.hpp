// DoublePIR's wire format (lib/doublepir/src/serializer/serializer.rs), parsed on the host before anything reaches the GPU.
//
// A request is `Vec<State>::serialize()`: u32 BE query count, then per query (a State = Vec<Matrix>) a u32 BE matrix count, then
// per matrix u32 BE rows, u32 BE cols and rows * cols u32 BE words.  DoublePirServer::answer (doublepir/server.rs:235-247) runs
// `Vec::<State>::deserialize` and then answer() (doublepir.rs:246-350), which reads q[0] (q_1) of every query whose row batch it
// computes and q[1 + j], j < ne / x (the q_2 vectors), of every query.  The parser records where those matrices are and checks
// what the reference asserts; it converts no data word (the kernels byte-swap as they stage the vectors).  Where the reference
// panics, the request is refused with B200PIR_E_SHAPE:
//   a header or data word past the end of the request (read_u32_iter's unwrap)
//   a query count, matrix count, rows or cols >= 2^28 (MAX_LEN)
//   zero queries (answer() divides the rows by the count)
//   a query with fewer than 1 + ne / x matrices (q[1 + j])
//   a q_1 or q_2 whose rows differ from 3 * the matrix's packed columns, or whose cols != 1 (matrix_mul_vec_packed's asserts)
//   a chunk index >= the query count, or a batch needing more rows than the server holds (MatrixRef::rows' slice)
// Matrices past the first 1 + ne / x of a query, and bytes after the last query, are read past and ignored, as the reference
// ignores them.  rows * cols is taken in 64 bits: data that would run past the request is truncation.
// The response is `msg.serialize()` in the same format: msg[0] = a_1' * a_2^T ((delta x) x n), then per query and j the pair
// h_1 * q_2 ((n delta x) x 1) and a_1' * q_2 ((delta x) x 1).
// Plain C++, no CUDA: tests/cpp/dpir_wire_check.cpp runs it on the CPU.
#pragma once
#include "../../include/b200pir.h"
#include <stddef.h>
#include <stdint.h>
#include <string>
#include <vector>

namespace b200pir {

constexpr uint32_t kDpirWireMaxLen = 1u << 28;   // serializer.rs:8 MAX_LEN

struct DpirWireMat {
  size_t pos;            // the matrix's rows header is request[pos, pos + 4); its data words start at pos + 8
  uint32_t rows, cols;
  size_t data_pos() const { return pos + 8; }
};

struct DpirWireRequest {
  std::vector<DpirWireMat> mats;   // the first `per_query` matrices of every query: query k's are mats[k * per_query ...]
  size_t queries = 0, per_query = 0;
  const DpirWireMat& q1(size_t k) const { return mats[k * per_query]; }
  const DpirWireMat& q2(size_t k, size_t j) const { return mats[k * per_query + 1 + j]; }
};

inline uint32_t dpir_load_be32(const uint8_t* p) {
  return ((uint32_t)p[0] << 24) | ((uint32_t)p[1] << 16) | ((uint32_t)p[2] << 8) | (uint32_t)p[3];
}
inline void dpir_store_be32(uint8_t* p, uint32_t v) {
  p[0] = (uint8_t)(v >> 24); p[1] = (uint8_t)(v >> 16); p[2] = (uint8_t)(v >> 8); p[3] = (uint8_t)v;
}

// Vec::<State>::deserialize plus answer()'s need for 1 + e matrices a query (e = ne / x) and the q_2 shape (3 * c1 x 1, c1 =
// packed columns of h_1).  Returns 0 or B200PIR_E_SHAPE with `err` set; r is filled only on success.
inline int parse_dpir_request(const uint8_t* req, size_t len, size_t e, uint64_t c1, DpirWireRequest& r, std::string& err) {
  size_t offs = 0;
  auto u32 = [&](uint32_t& v, const char* what) {
    if (len - offs < 4) { err = std::string("request truncated in ") + what; return false; }
    v = dpir_load_be32(req + offs);
    offs += 4;
    return true;
  };
  uint32_t nq = 0;
  if (!u32(nq, "the query count")) return B200PIR_E_SHAPE;
  if (nq >= kDpirWireMaxLen) { err = "query count >= 2^28"; return B200PIR_E_SHAPE; }
  if (nq == 0) { err = "zero queries"; return B200PIR_E_SHAPE; }
  DpirWireRequest out;
  out.queries = nq;
  out.per_query = 1 + e;
  out.mats.reserve((size_t)nq * (1 + e));
  for (uint32_t k = 0; k < nq; k++) {
    uint32_t nm = 0;
    if (!u32(nm, "a matrix count")) return B200PIR_E_SHAPE;
    if (nm >= kDpirWireMaxLen) { err = "query " + std::to_string(k) + ": matrix count >= 2^28"; return B200PIR_E_SHAPE; }
    for (uint32_t t = 0; t < nm; t++) {
      const size_t pos = offs;
      uint32_t rows = 0, cols = 0;
      if (!u32(rows, "a matrix header") || !u32(cols, "a matrix header")) return B200PIR_E_SHAPE;
      if (rows >= kDpirWireMaxLen || cols >= kDpirWireMaxLen) {
        err = "query " + std::to_string(k) + ": matrix rows or cols >= 2^28";
        return B200PIR_E_SHAPE;
      }
      const uint64_t words = (uint64_t)rows * cols;
      if ((len - offs) / 4 < words) { err = "request truncated in matrix data"; return B200PIR_E_SHAPE; }
      offs += (size_t)words * 4;
      if (t < 1 + e) out.mats.push_back(DpirWireMat{pos, rows, cols});
    }
    if (nm < 1 + e) {
      err = "query " + std::to_string(k) + " has " + std::to_string(nm) + " matrices; answer() reads " + std::to_string(1 + e);
      return B200PIR_E_SHAPE;
    }
  }
  for (size_t k = 0; k < nq; k++)
    for (size_t j = 0; j < e; j++) {
      const DpirWireMat& q = out.q2(k, j);
      if (q.cols != 1 || q.rows != 3 * c1) {
        err = "query " + std::to_string(k) + ": q_2 is " + std::to_string(q.rows) + " x " + std::to_string(q.cols) + ", h_1 needs " +
              std::to_string(3 * c1) + " x 1";
        return B200PIR_E_SHAPE;
      }
    }
  r = std::move(out);
  return 0;
}

// answer()'s row batches (doublepir.rs:261-268): l / nq rows each, the remainder in the last; batch k starts at k * (l / nq)
inline uint64_t dpir_batch_begin(uint64_t l, uint64_t nq, uint64_t k) { return k * (l / nq); }
inline uint64_t dpir_batch_rows(uint64_t l, uint64_t nq, uint64_t k) { return k == nq - 1 ? l - (nq - 1) * (l / nq) : l / nq; }

// The checks that depend on the rows a server holds and on the chunk.  Unchunked (chunk < 0): every batch reads its own rows of
// the whole l-row database, so the server must hold all l, and every q_1 must be 3 * db_cols x 1.  Chunked: only batch `chunk`
// is computed, from rows [0, its size) of the server's matrix (doublepir.rs:270-279), and only its q_1 is read.
inline int check_dpir_batches(const DpirWireRequest& r, uint64_t l, uint64_t server_rows, uint64_t db_cols, int64_t chunk,
                              std::string& err) {
  const uint64_t nq = r.queries;
  if (chunk >= 0 && (uint64_t)chunk >= nq) {
    err = "chunk index " + std::to_string(chunk) + " >= the " + std::to_string(nq) + " queries";
    return B200PIR_E_SHAPE;
  }
  const uint64_t need = chunk < 0 ? l : dpir_batch_rows(l, nq, (uint64_t)chunk);
  if (need > server_rows) {
    err = "the batch needs " + std::to_string(need) + " rows; the server holds " + std::to_string(server_rows);
    return B200PIR_E_SHAPE;
  }
  for (uint64_t k = 0; k < nq; k++) {
    if (chunk >= 0 && k != (uint64_t)chunk) continue;
    const DpirWireMat& q = r.q1(k);
    if (q.cols != 1 || q.rows != 3 * db_cols) {
      err = "query " + std::to_string(k) + ": q_1 is " + std::to_string(q.rows) + " x " + std::to_string(q.cols) + ", the database needs " +
            std::to_string(3 * db_cols) + " x 1";
      return B200PIR_E_SHAPE;
    }
  }
  return 0;
}

// The response of one request: its length and where its data words go.  dx = delta * x (rows of a_1'), rows1 = n delta x.
struct DpirResponseLayout {
  uint64_t nq, e, dx, n, rows1;
  uint64_t msgs() const { return 1 + 2 * nq * e; }
  uint64_t pair_bytes() const { return 8 + rows1 * 4 + 8 + dx * 4; }
  uint64_t bytes() const { return 4 + 8 + dx * n * 4 + nq * e * pair_bytes(); }
  uint64_t msg0_data() const { return 12; }
  // byte offsets of the data of h_1 * q_2 (a_2) and a_1' * q_2 (h_2) for query k, vector j
  uint64_t a2_data(uint64_t k, uint64_t j) const { return 12 + dx * n * 4 + (k * e + j) * pair_bytes() + 8; }
  uint64_t h2_data(uint64_t k, uint64_t j) const { return a2_data(k, j) + rows1 * 4 + 8; }
};

// Every header word of the response (data words are left as they are): the message count and each matrix's rows and cols.
inline void write_dpir_response_headers(const DpirResponseLayout& L, uint8_t* out) {
  dpir_store_be32(out, (uint32_t)L.msgs());
  dpir_store_be32(out + 4, (uint32_t)L.dx);
  dpir_store_be32(out + 8, (uint32_t)L.n);
  for (uint64_t k = 0; k < L.nq; k++)
    for (uint64_t j = 0; j < L.e; j++) {
      uint8_t* a2 = out + L.a2_data(k, j) - 8;
      dpir_store_be32(a2, (uint32_t)L.rows1);
      dpir_store_be32(a2 + 4, 1);
      uint8_t* h2 = out + L.h2_data(k, j) - 8;
      dpir_store_be32(h2, (uint32_t)L.dx);
      dpir_store_be32(h2 + 4, 1);
    }
}

}  // namespace b200pir
