// The plaintext decode rule of sdk_b200/csrc/item_place.cuh, on the CPU:
//   - every byte round-trips: pt_byte_decode(pt_byte_residue(x, q0), pt_byte_residue(x, q1)) == x, and pt_byte_residue is
//     recenter_mod(x, 256, q) as restated here;
//   - the accepted pairs are exactly the 256 images: every pair drawn from the two acceptance windows and their edges is
//     checked (mixed pairs, where each residue alone names a byte but the two name different bytes, included), every residue
//     of each modulus is swept against the other modulus's images, and random pairs are rejected;
//   - words that are not canonical residues (r + k q below 2^32) decode as their residue.
#include "../../sdk_b200/csrc/item_place.cuh"
#include <cstdio>
#include <vector>

using namespace b200pir;

static const uint32_t Q0 = 268369921u, Q1 = 249561089u;
static int failures = 0;
#define CHECK(cond, ...) do { if (!(cond)) { if (failures++ < 20) { std::printf(__VA_ARGS__); std::printf("\n"); } } } while (0)

static uint64_t rng_state = 0x2545F4914F6CDD1Dull;
static uint64_t next64() { rng_state ^= rng_state << 13; rng_state ^= rng_state >> 7; rng_state ^= rng_state << 17; return rng_state; }

// recenter_mod(x, 256, q) (arith.rs:415): x as a signed value in (-128, 128], then mod q
static uint32_t recenter(uint32_t x, uint32_t q) {
  const int64_t v = x > 128 ? (int64_t)x - 256 : (int64_t)x;
  return (uint32_t)((v % (int64_t)q + (int64_t)q) % (int64_t)q);
}

int main() {
  for (uint32_t x = 0; x < 256; x++) {
    CHECK(pt_byte_residue(x, Q0) == recenter(x, Q0) && pt_byte_residue(x, Q1) == recenter(x, Q1), "residue of byte %u", x);
    CHECK(pt_byte_decode(pt_byte_residue(x, Q0), pt_byte_residue(x, Q1), Q0, Q1) == (int)x, "byte %u does not round-trip", x);
  }
  auto img_byte = [](uint32_t r, uint32_t q) -> int {      // the restated inverse of one modulus
    for (uint32_t x = 0; x < 256; x++)
      if (recenter(x, q) == r) return (int)x;
    return -1;
  };
  // ---- the windows and their edges: [0, 130] and [q - 130, q) in both moduli, every pair
  std::vector<uint32_t> w0, w1;
  for (uint32_t r = 0; r <= 130; r++) { w0.push_back(r); w1.push_back(r); }
  for (uint32_t r = Q0 - 130; r < Q0; r++) w0.push_back(r);
  for (uint32_t r = Q1 - 130; r < Q1; r++) w1.push_back(r);
  std::vector<int> b0(w0.size()), b1(w1.size());
  for (size_t a = 0; a < w0.size(); a++) b0[a] = img_byte(w0[a], Q0);
  for (size_t a = 0; a < w1.size(); a++) b1[a] = img_byte(w1[a], Q1);
  size_t accepted = 0, mixed = 0;
  for (size_t a = 0; a < w0.size(); a++)
    for (size_t b = 0; b < w1.size(); b++) {
      const int want = (b0[a] >= 0 && b0[a] == b1[b]) ? b0[a] : -1;
      const int got = pt_byte_decode(w0[a], w1[b], Q0, Q1);
      CHECK(got == want, "pair (%u, %u): decoded %d, want %d", w0[a], w1[b], got, want);
      accepted += got >= 0;
      mixed += b0[a] >= 0 && b1[b] >= 0 && b0[a] != b1[b];
    }
  CHECK(accepted == 256, "%zu window pairs accepted, want 256", accepted);
  CHECK(mixed == 256 * 255, "%zu mixed pairs checked", mixed);
  // ---- every residue of one modulus against the image of the byte it would be if it were one: a residue that is no byte's
  // image is rejected whatever the other residue is
  for (uint32_t r = 0; r < Q0; r++) {
    const uint32_t x = r <= 128 ? r : (r >= Q0 - 127 ? r - (Q0 - 256) : (r & 255));
    const bool image = r <= 128 || r >= Q0 - 127;
    const int got = pt_byte_decode(r, pt_byte_residue(x, Q1), Q0, Q1);
    if (got != (image ? (int)x : -1)) CHECK(false, "q0 residue %u: decoded %d", r, got);
  }
  for (uint32_t r = 0; r < Q1; r++) {
    const uint32_t x = r <= 128 ? r : (r >= Q1 - 127 ? r - (Q1 - 256) : (r & 255));
    const bool image = r <= 128 || r >= Q1 - 127;
    const int got = pt_byte_decode(pt_byte_residue(x, Q0), r, Q0, Q1);
    if (got != (image ? (int)x : -1)) CHECK(false, "q1 residue %u: decoded %d", r, got);
  }
  // ---- random pairs: an accepted one is an image pair
  for (int t = 0; t < 1000000; t++) {
    const uint64_t v = next64();
    const uint32_t r0 = (uint32_t)(v % Q0), r1 = (uint32_t)((v >> 32) % Q1);
    const int got = pt_byte_decode(r0, r1, Q0, Q1);
    CHECK(got == -1 || (pt_byte_residue((uint32_t)got, Q0) == r0 && pt_byte_residue((uint32_t)got, Q1) == r1),
          "random pair (%u, %u) decoded %d", r0, r1, got);
  }
  // ---- non-canonical words: every r + k q below 2^32 decodes as r, for images and non-images alike
  for (uint32_t x = 0; x < 256; x++) {
    const uint32_t r0 = pt_byte_residue(x, Q0), r1 = pt_byte_residue(x, Q1);
    for (uint64_t k0 = 0; r0 + k0 * Q0 <= 0xFFFFFFFFull; k0++)
      for (uint64_t k1 = 0; r1 + k1 * Q1 <= 0xFFFFFFFFull; k1++)
        CHECK(pt_byte_decode((uint32_t)(r0 + k0 * Q0), (uint32_t)(r1 + k1 * Q1), Q0, Q1) == (int)x, "byte %u + (%llu q0, %llu q1)",
              x, (unsigned long long)k0, (unsigned long long)k1);
  }
  CHECK(pt_byte_decode(0xFFFFFFFFu, 0xFFFFFFFFu, Q0, Q1) == img_byte(0xFFFFFFFFu % Q0, Q0) &&
        img_byte(0xFFFFFFFFu % Q0, Q0) == -1, "all-ones words");
  CHECK(pt_byte_decode(Q0, Q1, Q0, Q1) == 0, "q itself is zero");
  CHECK(pt_byte_decode(Q0 + 200, Q1, Q0, Q1) == -1, "q0 + 200 is not an image");
  if (failures) { std::printf("%d failures\n", failures); return 1; }
  std::printf("decode rule ok\n");
  return 0;
}
