// The item maps of sdk_b200/csrc/item_place.cuh, on the CPU: for every geometry, every (il, j) and several z,
//   - db_bytes is each layout's store size in bytes, as restated here, and slice_bytes is its share of one slice;
//   - every byte an item is placed at, and every byte the slice import kernels address, lies inside db_bytes;
//   - the bytes different items (and moduli, limbs, z) occupy never overlap, in all three layouts;
//   - fetch_item(place_item(w)) == w for canonical residues, including the all-(q - 1) words, and an unwritten cell fetches as 0;
//   - the four limb-l bytes of j = 4 kq .. 4 kq + 3 are one 4-byte word at frag_word / tc5_word (what the export kernels read),
//     and join_limb_words recovers the residues from those words.
// place_item/fetch_item run on whole stores where the database is small enough; for the larger geometries the same checks run on
// the per-plane maps they are built from (frag_in_plane / tc5_in_plane inside one (slice, n, z) plane, imad_word for format 0).
#include "../../sdk_b200/csrc/item_place.cuh"
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <vector>

using namespace b200pir;

static const uint32_t Q0 = 268369921u, Q1 = 249561089u;
static int failures = 0;
#define CHECK(cond, ...) do { if (!(cond)) { if (failures++ < 20) { std::printf(__VA_ARGS__); std::printf("\n"); } } } while (0)

static uint64_t rng_state = 0x9E3779B97F4A7C15ull;
static uint64_t next64() { rng_state ^= rng_state << 13; rng_state ^= rng_state >> 7; rng_state ^= rng_state << 17; return rng_state; }
// a canonical word for (il, j, z): mostly random, every 5th the all-(q - 1) word, every 7th zero halves mixed in
static uint64_t word_for(int il, int j, int z) {
  const uint64_t k = ((uint64_t)il * 1315423911u) ^ ((uint64_t)j * 2654435761u) ^ ((uint64_t)z * 97u);
  if (k % 5 == 0) return (uint64_t)(Q0 - 1) | (uint64_t)(Q1 - 1) << 32;
  const uint64_t r = next64();
  const uint32_t lo = (uint32_t)(r % Q0), hi = (uint32_t)((r >> 32) % Q1);
  return k % 7 == 0 ? (uint64_t)lo : ((uint64_t)lo | (uint64_t)hi << 32);
}

static void no_overlap(std::vector<size_t>& offs, const char* what, int dim0, int rows) {
  std::sort(offs.begin(), offs.end());
  CHECK(std::adjacent_find(offs.begin(), offs.end()) == offs.end(), "%s: two bytes coincide (dim0 %d rows %d)", what, dim0, rows);
}

static void check_geometry(int dim0, int rows) {
  const int zs[] = {0, 1, 777, 2047};
  const int slices = 2, slice = 1;
  const MulGeom G{dim0, rows, slices};
  const ImmaGeom F = make_imma_geom(dim0, rows);
  const Tc5Geom T = make_tc5_geom(dim0, rows);
  DbLayout L[3] = {{0, G, F, T, nullptr}, {1, G, F, T, nullptr}, {2, G, F, T, nullptr}};
  // ---- store sizes in bytes: format 0 is slices x rows x dim0/2 x 2048 16-byte cells, format 1 slices x 2 x 2048 x mt x ks
  // groups of 4 x 32 16-byte fragments, format 2 slices x 2 x 2048 x mt x ks 4096-byte tile images
  {
    const size_t want[3] = {(size_t)slices * rows * (dim0 / 2) * POLY * 16, (size_t)slices * 2 * POLY * F.mt * F.ks * 4 * 32 * 16,
                            (size_t)slices * 2 * POLY * T.mt * T.ks * 4096};
    for (int f = 0; f < 3; f++) {
      CHECK(db_bytes(L[f], slices) == want[f], "format %d: db_bytes %zu, want %zu (dim0 %d rows %d)", f, db_bytes(L[f], slices),
            want[f], dim0, rows);
      CHECK(slice_bytes(L[f]) * slices == want[f], "format %d: slice_bytes (dim0 %d rows %d)", f, dim0, rows);
    }
  }
  // ---- the bulk writers stay inside the store: the import kernels write slice s of format 0 at imad_cell (k_db_import_imad),
  // of format 1 in whole groups at frag_db_group (k_db_import_frag) and of format 2 in whole tiles at tc5_db_tile
  // (k_db_import_tc5), within [s, s + 1) * slice_bytes
  for (int s = 0; s < slices; s++) {
    const size_t lo[3] = {imad_cell(G, s, 0, 0, 0) * 16, frag_db_group(F, s, 0, 0, 0, 0) * FRAG_GROUP,
                          tc5_db_tile(T, s, 0, 0, 0, 0) * TC5_TILE};
    const size_t end[3] = {(imad_cell(G, s, rows - 1, dim0 - 1, POLY - 1) + 1) * 16,
                           (frag_db_group(F, s, 1, POLY - 1, F.mt - 1, F.ks - 1) + 1) * FRAG_GROUP,
                           (tc5_db_tile(T, s, 1, POLY - 1, T.mt - 1, T.ks - 1) + 1) * TC5_TILE};
    for (int f = 0; f < 3; f++)
      CHECK(lo[f] == s * slice_bytes(L[f]) && end[f] <= (s + 1) * slice_bytes(L[f]) &&
            (s + 1) * slice_bytes(L[f]) <= db_bytes(L[f], slices), "format %d import of slice %d past its slice (dim0 %d rows %d)",
            f, s, dim0, rows);
  }
  if (failures) return;      // the stores below are db_bytes long: a wrong size would be written out of bounds
  // ---- disjointness of every byte of every item at the chosen z (both slices' planes of z, both moduli, all limbs)
  {
    std::vector<size_t> o0, o1, o2;
    for (int s = 0; s < slices; s++)
      for (int z : zs)
        for (int il = 0; il < rows; il++)
          for (int j = 0; j < dim0; j++) {
            const size_t w = imad_word(G, s, il, j, z);
            o0.push_back(w); o0.push_back(w + 1);
            for (int n = 0; n < 2; n++)
              for (int l = 0; l < 4; l++) {
                o1.push_back(frag_plane(F, s, n, z) + frag_in_plane(F, il, j, l));
                o2.push_back(tc5_plane(T, s, n, z) + tc5_in_plane(T, il, j, l));
              }
          }
    // the bytes place_item writes: o0 holds u32 words
    CHECK((*std::max_element(o0.begin(), o0.end()) + 1) * 4 <= db_bytes(L[0], slices), "format 0 word out of the store");
    CHECK(*std::max_element(o1.begin(), o1.end()) < db_bytes(L[1], slices), "format 1 byte out of the store");
    CHECK(*std::max_element(o2.begin(), o2.end()) < db_bytes(L[2], slices), "format 2 byte out of the store");
    no_overlap(o0, "format 0", dim0, rows);
    no_overlap(o1, "format 1", dim0, rows);
    no_overlap(o2, "format 2", dim0, rows);
  }
  // ---- the 4-byte words of the export kernels, and join_limb_words
  for (int row = 0; row < 32; row++)
    for (int kq = 0; kq < 8; kq++)
      for (int l = 0; l < 4; l++)
        for (int i = 0; i < 4; i++) {
          if (row < 16) CHECK(frag_byte(row, 4 * kq + i, l) == frag_word(row, kq, l) + i, "frag_word row %d kq %d l %d", row, kq, l);
          CHECK(tc5_tile_off(tc5_m_index(row, l), 4 * kq + i) == tc5_word(row, kq, l) + i, "tc5_word row %d kq %d l %d", row, kq, l);
        }
  for (int t = 0; t < 1000; t++) {
    uint32_t r[4], w[4] = {0, 0, 0, 0}, back[4];
    for (int i = 0; i < 4; i++) r[i] = t == 0 ? Q0 - 1 : (uint32_t)(next64() % Q0);
    for (int l = 0; l < 4; l++)
      for (int i = 0; i < 4; i++) w[l] |= ((r[i] >> (7 * l)) & 127u) << (8 * i);
    join_limb_words(w, back);
    for (int i = 0; i < 4; i++) CHECK(back[i] == r[i], "join_limb_words");
  }
  // ---- fetch_item(place_item(w)) == w, on stores of exactly db_bytes followed by a guard no write may reach
  const size_t items = (size_t)rows * dim0;
  if (items * POLY * 8 * slices <= ((size_t)64 << 20)) {
    const size_t guard = 4096;
    std::vector<uint32_t> store[3];
    for (int f = 0; f < 3; f++) {
      store[f].assign((db_bytes(L[f], slices) + guard) / 4, 0);
      // a placed residue (< 2^28) or limb byte (< 2^7) never leaves a guard word all ones
      std::fill(store[f].end() - guard / 4, store[f].end(), 0xFFFFFFFFu);
      L[f].base = reinterpret_cast<uint8_t*>(store[f].data());
    }
    // every second item stays unwritten
    rng_state = 0x9E3779B97F4A7C15ull;
    for (int z : zs)
      for (int il = 0; il < rows; il++)
        for (int j = 0; j < dim0; j++) {
          if ((il + j) & 1) continue;
          const uint64_t w = word_for(il, j, z);
          for (int f = 0; f < 3; f++) place_item(L[f], slice, il, j, z, (uint32_t)w, (uint32_t)(w >> 32));
        }
    for (int f = 0; f < 3; f++)
      CHECK(std::all_of(store[f].end() - guard / 4, store[f].end(), [](uint32_t v) { return v == 0xFFFFFFFFu; }),
            "format %d: place_item wrote past db_bytes (dim0 %d rows %d)", f, dim0, rows);
    rng_state = 0x9E3779B97F4A7C15ull;
    for (int z : zs)
      for (int il = 0; il < rows; il++)
        for (int j = 0; j < dim0; j++) {
          const bool written = !((il + j) & 1);
          const uint64_t w = written ? word_for(il, j, z) : 0;
          for (int f = 0; f < 3; f++) {
            CHECK(fetch_item(L[f], slice, il, j, z) == w, "format %d (%d,%d) il %d j %d z %d", f, dim0, rows, il, j, z);
            CHECK(fetch_item(L[f], 0, il, j, z) == 0, "format %d: slice 0 is unwritten", f);
          }
        }
  } else {
    // one (slice, n, z) plane of each limb layout at a time: the in-plane maps the whole-buffer functions add the plane base to
    std::vector<uint8_t> p1((size_t)F.mt * F.ks * FRAG_GROUP), p2((size_t)T.mt * T.ks * TC5_TILE);
    for (int n = 0; n < 2; n++) {
      std::fill(p1.begin(), p1.end(), 0);
      std::fill(p2.begin(), p2.end(), 0);
      std::vector<uint32_t> vals(items);
      for (int il = 0; il < rows; il++)
        for (int j = 0; j < dim0; j++) {
          const uint64_t w = ((il + j) & 1) ? 0 : word_for(il, j, n);
          const uint32_t r = n ? (uint32_t)(w >> 32) : (uint32_t)w;
          vals[(size_t)il * dim0 + j] = r;
          if ((il + j) & 1) continue;
          for (int l = 0; l < 4; l++) {
            p1[frag_in_plane(F, il, j, l)] = (uint8_t)((r >> (7 * l)) & 127u);
            p2[tc5_in_plane(T, il, j, l)] = (uint8_t)((r >> (7 * l)) & 127u);
          }
        }
      for (int il = 0; il < rows; il++)
        for (int j = 0; j < dim0; j++) {
          uint32_t a = 0, b = 0;
          for (int l = 0; l < 4; l++) { a |= (uint32_t)p1[frag_in_plane(F, il, j, l)] << (7 * l); b |= (uint32_t)p2[tc5_in_plane(T, il, j, l)] << (7 * l); }
          CHECK(a == vals[(size_t)il * dim0 + j] && b == vals[(size_t)il * dim0 + j], "plane (%d,%d) il %d j %d n %d", dim0, rows, il, j, n);
        }
    }
  }
}

int main() {
  const int dims[] = {2, 4, 32, 64, 512, 1024};
  const int rowss[] = {1, 2, 16, 31, 32, 48, 256};
  for (int d : dims)
    for (int r : rowss) check_geometry(d, r);
  if (failures) { std::printf("%d failures\n", failures); return 1; }
  std::printf("layout maps ok\n");
  return 0;
}
