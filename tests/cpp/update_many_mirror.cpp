// The /update-row call through the C++ host mirror (include/b200pir.hpp) on cuda:0, parameter set T:
//   update_many_mirror <body file> <v_firstdim file (u64)> <out file>
// applies the body with Database::update_many_items, prints largest_update and writes the first-dimension product of slice 0
// (num_per x 2 x 2 x 2048 u64) to <out file>.  tests/test_gpu_update_many.py compares both with the Python path.
#include "../../include/b200pir.hpp"
#include <cstdio>
#include <cstring>
#include <vector>

static std::vector<uint8_t> read_file(const char* path) {
  std::vector<uint8_t> v;
  FILE* f = fopen(path, "rb");
  if (!f) throw std::runtime_error(std::string("cannot open ") + path);
  int ch;
  while ((ch = fgetc(f)) != EOF) v.push_back((uint8_t)ch);
  fclose(f);
  return v;
}

int main(int argc, char** argv) {
  if (argc != 4) { fprintf(stderr, "usage: %s body v_firstdim out\n", argv[0]); return 2; }
  b200pir_params p{2, 6, 2, 256, 20, 8, 4, 8, 8, 1, 8192, 0, 1};
  try {
    spiral_rs::Params params(p, 0);
    spiral_rs::Database db(params);
    const std::vector<uint8_t> body = read_file(argv[1]), vb = read_file(argv[2]);
    const uint64_t largest = db.update_many_items(body.data(), body.size());
    std::vector<uint64_t> v(vb.size() / 8);
    std::memcpy(v.data(), vb.data(), v.size() * 8);
    std::vector<spiral_rs::PolyMatrixNTT> out;
    spiral_rs::server::multiply_reg_by_database(out, db, 0, v.data(), params);
    FILE* f = fopen(argv[3], "wb");
    if (!f) throw std::runtime_error("cannot write the output");
    for (const auto& m : out) fwrite(m.data.data(), 8, m.data.size(), f);
    fclose(f);
    printf("%llu\n", (unsigned long long)largest);
  } catch (const std::exception& e) { fprintf(stderr, "%s\n", e.what()); return 1; }
  return 0;
}
