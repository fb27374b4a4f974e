// Runs the DoublePIR wire parser (sdk_b200/csrc/dpir_wire.hpp) on one request file and prints what it found, for
// tests/test_dpir_wire_parser.py.  Usage:
//   dpir_wire_check <request> <e> <c1> <l> <server_rows> <db_cols> <chunk> <dx> <n> <response_out>
// Prints "parse <rc>", "batches <rc>" (when the parse succeeded), "mat <query> <index> <pos> <rows> <cols>" for every recorded
// matrix and "size <bytes>"; on success writes a response of zero data words with its headers to <response_out>.
#include "../../sdk_b200/csrc/dpir_wire.hpp"
#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <iterator>
#include <vector>

int main(int argc, char** argv) {
  if (argc != 11) { std::fprintf(stderr, "usage: see the header\n"); return 2; }
  std::ifstream f(argv[1], std::ios::binary);
  std::vector<uint8_t> req((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>());
  auto arg = [&](int i) { return std::strtoull(argv[i], nullptr, 10); };
  const size_t e = arg(2);
  const uint64_t c1 = arg(3), l = arg(4), server_rows = arg(5), db_cols = arg(6), dx = arg(8), n = arg(9);
  const int64_t chunk = std::strtoll(argv[7], nullptr, 10);
  b200pir::DpirWireRequest r;
  std::string err;
  int rc = b200pir::parse_dpir_request(req.data(), req.size(), e, c1, r, err);
  std::printf("parse %d\n", rc);
  if (rc) { std::printf("error %s\n", err.c_str()); return 0; }
  rc = b200pir::check_dpir_batches(r, l, server_rows, db_cols, chunk, err);
  std::printf("batches %d\n", rc);
  if (rc) std::printf("error %s\n", err.c_str());
  for (size_t k = 0; k < r.queries; k++)
    for (size_t t = 0; t < r.per_query; t++) {
      const b200pir::DpirWireMat& m = r.mats[k * r.per_query + t];
      std::printf("mat %zu %zu %zu %u %u\n", k, t, m.pos, m.rows, m.cols);
    }
  const b200pir::DpirResponseLayout L{r.queries, e, dx, n, n * dx};
  std::printf("size %llu\n", (unsigned long long)L.bytes());
  if (rc) return 0;
  std::vector<uint8_t> out(L.bytes(), 0);
  b200pir::write_dpir_response_headers(L, out.data());
  std::ofstream o(argv[10], std::ios::binary);
  o.write(reinterpret_cast<const char*>(out.data()), (std::streamsize)out.size());
  return 0;
}
