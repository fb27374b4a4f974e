// CPU run of the gadget-width helpers (sdk_b200/csrc/gadget.hpp), no GPU and no library: prints "<t> <bits_per> <live_digits>"
// for every gadget dimension 3..56.  tests/test_live_digits.py checks the lines against plain integers and the oracle's
// gadget decomposition.
#include "../../sdk_b200/csrc/gadget.hpp"
#include <cstdio>

int main() {
  for (int t = 3; t <= 56; t++) printf("%d %d %d\n", t, b200pir::bits_per(t), b200pir::live_digits(t));
  return 0;
}
