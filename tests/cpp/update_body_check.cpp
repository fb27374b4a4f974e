// CPU run of the /update-row body parser (sdk_b200/csrc/update_body.hpp), no GPU and no library:
//   update_body_check <body file> <max_chunk_len> <num_items>
// prints "error <code>", "largest <largest_update>", one "entry <pos> <chunk_len> <db_idx>" line per entry of the valid prefix
// and one "kept <pos>" line per entry keep_last_occurrence keeps.  tests/test_update_body_parser.py compares the lines with
// the restatement of update_many_items in tests/update_rows_oracle.py.
#include "../../sdk_b200/csrc/update_body.hpp"
#include <cstdio>
#include <cstdlib>
#include <vector>

int main(int argc, char** argv) {
  if (argc != 4) { fprintf(stderr, "usage: %s body max_chunk_len num_items\n", argv[0]); return 2; }
  FILE* f = fopen(argv[1], "rb");
  if (!f) { perror(argv[1]); return 2; }
  std::vector<uint8_t> body;
  int ch;
  while ((ch = fgetc(f)) != EOF) body.push_back((uint8_t)ch);
  fclose(f);
  const b200pir::BodyParse r = b200pir::parse_update_body(body.data(), body.size(), strtoull(argv[2], nullptr, 10),
                                                          strtoull(argv[3], nullptr, 10));
  printf("error %d\nlargest %llu\n", r.error, (unsigned long long)r.largest_update);
  for (const auto& e : r.entries) printf("entry %zu %u %u\n", e.pos, e.chunk_len, e.db_idx);
  for (const auto& e : b200pir::keep_last_occurrence(r.entries)) printf("kept %zu\n", e.pos);
  return 0;
}
