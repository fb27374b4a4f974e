// The wgmma shared-memory matrix descriptor built by sdk_b200/csrc/tc5_layout.cuh, compared field by field with a bit-field
// struct written from the PTX ISA's "Matrix Descriptor Format" table (wgmma, sm_90a).  Host-only.
#include <cstdio>
#include <cstdint>
#include <initializer_list>
#include "../../sdk_b200/csrc/tc5_layout.cuh"

union GmmaDesc {
  uint64_t desc;
  struct {
    uint64_t start_address : 14, : 2;          // bits 0-13: (address & 0x3FFFF) >> 4
    uint64_t leading_byte_offset : 14, : 2;    // bits 16-29: LBO >> 4
    uint64_t stride_byte_offset : 14, : 3;     // bits 32-45: SBO >> 4
    uint64_t base_offset : 3, : 10;            // bits 49-51
    uint64_t layout_type : 2;                  // bits 62-63: 0 = no swizzle (interleave), 1 = 128 B, 2 = 64 B, 3 = 32 B
  } f;
};

int main() {
  int bad = 0;
  for (uint32_t addr : {0x0u, 0x400u, 0x12340u, 0x3FFF0u}) {
    GmmaDesc s;
    s.desc = 0;
    s.f.start_address = (addr & 0x3FFFF) >> 4;
    s.f.leading_byte_offset = b200pir::TC5_LBO >> 4;
    s.f.stride_byte_offset = b200pir::TC5_SBO >> 4;
    s.f.base_offset = 0;
    s.f.layout_type = 0;
    if (s.desc != b200pir::tc5_smem_desc(addr)) {
      printf("smem desc %016llx vs %016llx\n", (unsigned long long)s.desc, (unsigned long long)b200pir::tc5_smem_desc(addr));
      bad++;
    }
  }
  printf(bad ? "descriptor mismatch\n" : "descriptors ok\n");
  return bad;
}
