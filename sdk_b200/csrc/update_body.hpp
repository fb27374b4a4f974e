// The body of POST /update-row (lib/server/src/bin/server.rs:31-43), parsed on the host before anything is written.
//
// update_many_items (lib/server/src/db/loading.rs:361-377) walks the body as entries [u32 BE chunk_len][chunk_len bytes] and
// hands each chunk to update_item (:301-315): chunk = [u32 BE db_idx][raw bucket bytes].  It applies entries one by one and
// stops at the first bad one, so everything before that entry is written and nothing from it on.  parse_update_body finds that
// valid prefix and the error of the first bad entry without applying anything.  The checks, per entry and in the reference's
// order:
//   header past the end of the body, chunk past the end (the reference panics on the slice)        -> B200PIR_E_SHAPE
//   chunk_len > 4 + instances * n^2 * bytes_per_chunk (update_item: InvalidLength)                  -> B200PIR_E_SHAPE
//   chunk_len < 4 (update_item panics reading db_idx)                                                -> B200PIR_E_SHAPE
//   db_idx >= num_items (update_item_raw: "bad db idx")                                              -> B200PIR_E_SHAPE
// Plain C++, no CUDA: tests/cpp/update_body_check.cpp runs it on the CPU.
#pragma once
#include "../../include/b200pir.h"
#include <stddef.h>
#include <stdint.h>
#include <string>
#include <unordered_set>
#include <vector>

namespace b200pir {

struct BodyEntry {
  size_t pos;            // the entry's chunk_len header is body[pos, pos + 4); its raw bucket bytes start at pos + 8
  uint32_t chunk_len;    // 4 + number of raw bucket bytes
  uint32_t db_idx;
  size_t data_pos() const { return pos + 8; }
  uint32_t data_len() const { return chunk_len - 4; }
};

struct BodyParse {
  std::vector<BodyEntry> entries;   // the valid prefix, in body order
  int error = 0;                    // 0 or the code of the first bad entry, which is entries.size()
  std::string message;
  uint64_t largest_update = 0;      // max chunk_len over the valid prefix (what update_many_items returns on success)
};

inline uint32_t load_be32(const uint8_t* p) {
  return ((uint32_t)p[0] << 24) | ((uint32_t)p[1] << 16) | ((uint32_t)p[2] << 8) | (uint32_t)p[3];
}

// max_chunk_len = 4 + instances * n^2 * bytes_per_chunk; num_items = dim0 * num_per
inline BodyParse parse_update_body(const uint8_t* body, size_t len, size_t max_chunk_len, uint64_t num_items) {
  BodyParse r;
  size_t offs = 0;
  auto fail = [&](const std::string& m) { r.error = B200PIR_E_SHAPE; r.message = "update entry " + std::to_string(r.entries.size()) + ": " + m; };
  while (offs < len) {
    if (len - offs < 4) { fail("header runs past the end of the body"); break; }
    const uint32_t chunk_len = load_be32(body + offs);
    if (len - offs - 4 < chunk_len) { fail("chunk runs past the end of the body"); break; }
    if (chunk_len > max_chunk_len) { fail("update longer than 4 + instances*n^2*bytes_per_chunk"); break; }
    if (chunk_len < 4) { fail("chunk shorter than its 4-byte db_idx"); break; }
    const uint32_t db_idx = load_be32(body + offs + 4);
    if (db_idx >= num_items) { fail("bad db idx " + std::to_string(db_idx)); break; }
    r.entries.push_back(BodyEntry{offs, chunk_len, db_idx});
    if (chunk_len > r.largest_update) r.largest_update = chunk_len;
    offs += 4 + (size_t)chunk_len;
  }
  return r;
}

// Applied in order, a later entry for the same db_idx overwrites an earlier one entirely (update_item_raw writes every slice),
// so only the last occurrence of each db_idx matters.  Returns those, in body order.
inline std::vector<BodyEntry> keep_last_occurrence(const std::vector<BodyEntry>& entries) {
  std::unordered_set<uint32_t> seen;
  seen.reserve(entries.size() * 2);
  std::vector<BodyEntry> kept;
  for (size_t k = entries.size(); k-- > 0;)
    if (seen.insert(entries[k].db_idx).second) kept.push_back(entries[k]);
  return std::vector<BodyEntry>(kept.rbegin(), kept.rend());
}

}  // namespace b200pir
