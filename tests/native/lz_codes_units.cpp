// The branch-free length / distance codes of zb_common.h (what k_lz's batch pass converts every match with)
// against the closed forms with early returns, for tests/test_lz_codes_units.py.
#include <stdint.h>

#include "../../zippy_b200/csrc/zb_common.h"

// every length 3..258 and distance 1..32768: code and extra value against zb_len_code / zb_len_base and
// zb_dist_code / zb_dist_base, and the extra value fits the code's extra bits
extern "C" int t_codes_compare(void) {
  int bad = 0;
  for (uint32_t l = 3; l <= 258; l++) {
    uint32_t ex;
    const uint32_t c = zb_len_code_bf(l, ex);
    bad += c != (uint32_t)zb_len_code(l) || ex != l - zb_len_base((int)c) || (ex >> zb_len_extra_bits((int)c)) != 0u;
  }
  for (uint32_t d = 1; d <= 32768; d++) {
    uint32_t ex;
    const uint32_t c = zb_dist_code_bf(d, ex);
    bad += c != (uint32_t)zb_dist_code(d) || ex != d - zb_dist_base((int)c) || (ex >> zb_dist_extra_bits((int)c)) != 0u;
  }
  return bad;
}
