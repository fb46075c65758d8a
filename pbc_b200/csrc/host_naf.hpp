// host_naf.hpp -- non-adjacent form of the group order, one-time host-side setup for the
// signed-digit Miller loops (type A1; types F, D and G).  The reference scans the plain bits of n
// ("TODO: sliding NAF", ecc/a_param.c:1978); a signed scan evaluates the same Miller function up to
// vertical lines and constants in F_p^*, which the final exponentiation removes, with one chord per
// three bits instead of one per two.  Shared with tests/host/a_steps_host.cpp.
#pragma once
#include <stdint.h>
#include <vector>

#include "host_bigint.hpp"

namespace pbcb200 {

// digits[i] in {-1, 0, +1}, least significant first, no two adjacent non-zero, top digit +1
inline std::vector<int8_t> naf_digits(const BigUInt& n) {
  std::vector<uint32_t> w = n.w;
  w.push_back(0);                                   // room for the carry of n + 1
  std::vector<int8_t> d;
  auto is_zero = [&]() { for (uint32_t x : w) if (x) return false; return true; };
  while (!is_zero()) {
    int8_t digit = 0;
    if (w[0] & 1u) {
      digit = (w[0] & 2u) ? -1 : 1;                 // n mod 4 == 3 -> -1, == 1 -> +1
      if (digit == 1) {
        w[0] &= ~1u;                                // n - 1 (n is odd: no borrow)
      } else {
        for (size_t i = 0; i < w.size(); i++) { if (++w[i] != 0) break; }   // n + 1
      }
    }
    d.push_back(digit);
    for (size_t i = 0; i + 1 < w.size(); i++) w[i] = (w[i] >> 1) | (w[i + 1] << 31);
    w.back() >>= 1;
  }
  return d;
}

}  // namespace pbcb200
