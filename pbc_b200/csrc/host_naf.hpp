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

// The digits the Miller loops walk for a group order r (odd).  The reference scans the bits of r from
// the second highest down to bit 1 and ends on a tangent, so it evaluates f_{r-1,P}.  A signed scan of
// r itself ends on the tangent at (r + 1)/2 P where r = 3 mod 4, i.e. evaluates f_{r+1,P}; the two
// differ by the lines through P and (r - 1) P, r P, which are vertical (killed by the final
// exponentiation) only when r P = O.  So where the curve has points outside E[r] (cofactor > 1) the
// walk takes the digits of r - 1: digit 0 is 0 and never read, the others are the non-adjacent form of
// (r - 1)/2, and the walk gives f_{r-1,P} for every P on the curve.  Where r = 1 mod 4 these are the
// digits of r with digit 0 cleared, the same walk.  With cofactor 1 every point has r P = O and the
// digits of r are kept (for g149 they have one chord fewer).
inline std::vector<int8_t> miller_naf_digits(const BigUInt& r, bool cofactor_one) {
  return cofactor_one ? naf_digits(r) : naf_digits(r - BigUInt(1));
}

}  // namespace pbcb200
