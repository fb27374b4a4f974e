// Reading the database back through the C++ host mirror (include/b200pir.hpp) on cuda:0, parameter set T:
//   db_export_mirror <words file (u64)> <snapshot path> <out file>
// uploads the words, downloads them with Database::words(), saves a snapshot with Database::save_file, loads it into a second
// database with b200pir_db_load_file and writes that database's words() to <out file>.  Prints "same" when the first download
// equals the uploaded words.  tests/test_gpu_db_export.py checks the snapshot and <out file> against the Python path.
#include "../../include/b200pir.hpp"
#include <cstdio>
#include <vector>

int main(int argc, char** argv) {
  if (argc != 4) { fprintf(stderr, "usage: %s words snapshot out\n", argv[0]); return 2; }
  b200pir_params p{2, 6, 2, 256, 20, 8, 4, 8, 8, 1, 8192, 0, 1};
  try {
    spiral_rs::Params params(p, 0);
    std::vector<uint64_t> words(params.slices() * params.dim0() * params.num_per() * 2048);
    FILE* f = fopen(argv[1], "rb");
    if (!f || fread(words.data(), 8, words.size(), f) != words.size()) throw std::runtime_error("cannot read the words");
    fclose(f);
    spiral_rs::Database db(params, words.data(), words.size());
    const std::vector<uint64_t> back = db.words();
    db.save_file(argv[2]);
    spiral_rs::Database loaded(params);
    spiral_rs::check(b200pir_db_load_file(params.ctx, loaded.h, argv[2]));
    const std::vector<uint64_t> again = loaded.words();
    f = fopen(argv[3], "wb");
    if (!f || fwrite(again.data(), 8, again.size(), f) != again.size()) throw std::runtime_error("cannot write the output");
    fclose(f);
    printf("%s\n", back == words ? "same" : "different");
  } catch (const std::exception& e) { fprintf(stderr, "%s\n", e.what()); return 1; }
  return 0;
}
