// a_steps_host.cpp -- CPU instantiation of the slot programs of pbc_b200/csrc/a_steps.cuh.
//
// TEST INFRASTRUCTURE.  The device kernels run these templates against Ops<N, FULL, BLOCK> (shared-
// memory slots, Montgomery limbs); here the same templates run against a big-integer policy class,
// following k_a1_miller / k_a1_finalexp step for step, so the formulas (Jacobian doubling with the
// tangent, chord + mixed addition, Lucas final exponentiation) are pinned to reference fixtures
// without a GPU.  The Miller loop runs the five-temporary programs; argument "5t": on the bits of n, "5t-naf": on its
// signed digits (as k_a1_miller), "pp": on the bits of n, then the fixed-argument table programs must give the same
// pairing.  stdin: p n l count, then count lines "Px Py Qx Qy" (decimal); stdout: "Re Im" (hex).
#include <stdio.h>
#include <iostream>
#include <string>

#include "../../pbc_b200/csrc/host_bigint.hpp"
#include "../../pbc_b200/csrc/host_naf.hpp"
#include "../../pbc_b200/csrc/a_steps.cuh"

using pbcb200::BigUInt;

struct HostOps {
  static BigUInt s[32];
  static BigUInt p;
  static void mul(int d, int a, int b) { s[d] = BigUInt::mulmod(s[a], s[b], p); }
  static void sqr(int d, int a) { s[d] = BigUInt::mulmod(s[a], s[a], p); }
  static void add(int d, int a, int b) { s[d] = BigUInt::addmod(s[a], s[b], p); }
  static void sub(int d, int a, int b) { s[d] = BigUInt::submod(s[a], s[b], p); }
  static void dbl(int d, int a, int k = 1) {
    BigUInt x = s[a];
    for (int i = 0; i < k; i++) x = BigUInt::addmod(x, x, p);
    s[d] = x;
  }
  static void halve(int d, int a, int k = 1) {
    BigUInt x = s[a];
    for (int i = 0; i < k; i++) {
      if (x.bit(0)) x = x + p;
      BigUInt q;
      BigUInt::divmod(x, BigUInt(2), &q, nullptr);
      x = q;
    }
    s[d] = x;
  }
  static void copy(int d, int a) { s[d] = s[a]; }
};
BigUInt HostOps::s[32];
BigUInt HostOps::p;

struct HostTable {
  std::vector<BigUInt> rows;
  template <class O> void store(size_t row, int slot) {
    if (rows.size() <= row) rows.resize(row + 1);
    rows[row] = O::s[slot];
  }
  template <class O> void load(int slot, size_t row) const { O::s[slot] = rows[row]; }
};

static std::string hex(const BigUInt& x) {
  if (x.is_zero()) return "0";
  std::string r;
  char buf[16];
  for (size_t i = x.w.size(); i-- > 0;) {
    snprintf(buf, sizeof buf, i + 1 == x.w.size() ? "%x" : "%08x", x.w[i]);
    r += buf;
  }
  return r;
}

int main(int argc, char** argv) {
  using namespace pbcb200;
  const bool pp_mode = argc > 1 && std::string(argv[1]) == "pp";
  const std::string mode = argc > 1 ? argv[1] : "";
  const bool naf = mode == "5t-naf";                            // signed-digit scan of n (host_naf.hpp)
  using O = HostOps;
  std::string sp, sn, sl;
  int count;
  std::cin >> sp >> sn >> sl >> count;
  BigUInt n, l;
  BigUInt::from_dec(sp, &O::p);
  BigUInt::from_dec(sn, &n);
  BigUInt::from_dec(sl, &l);
  const BigUInt& p = O::p;
  enum { sPX = 20, sPY = 21, sD = 22, sN = 23, sP = 24, sV0 = 25, sV1 = 26, sT = 27, sTWO = 28 };
  for (int c = 0; c < count; c++) {
    std::string a, b, x, y;
    std::cin >> a >> b >> x >> y;
    BigUInt Px, Py;
    BigUInt::from_dec(a, &Px);
    BigUInt::from_dec(b, &Py);
    BigUInt::from_dec(x, &O::s[aQX]);
    BigUInt::from_dec(y, &O::s[aQY]);
    // k_a1_miller
    O::s[aX] = Px; O::s[aY] = Py;
    O::s[aZ] = BigUInt(1); O::s[aZ2] = BigUInt(1);
    O::s[aF0] = BigUInt(1); O::s[aF1] = BigUInt();
    O::s[aT5] = BigUInt(0xdead);                        // must never be read or written
    std::vector<int8_t> dg = naf_digits(n);
    if (naf) {
      // self-check of the digit table: sum d_i 2^i == n, no two adjacent non-zero digits
      BigUInt pos, negs;
      for (size_t i = 0; i < dg.size(); i++) {
        if (dg[i] > 0) pos = pos + BigUInt(1).shl(i);
        if (dg[i] < 0) negs = negs + BigUInt(1).shl(i);
        if (i && dg[i] && dg[i - 1]) { fprintf(stderr, "adjacent digits\n"); return 3; }
      }
      if (!(pos - negs == n) || dg.back() != 1) { fprintf(stderr, "bad digit table\n"); return 3; }
    }
    const int top = naf ? (int)dg.size() - 2 : (int)n.bits() - 2;
    const BigUInt mPy = O::p - Py;
    for (int m = top; m >= 0; m--) {
      const bool chord = m > 0 && (naf ? dg[m] != 0 : n.bit((size_t)m));
      const bool minus = naf && dg[m] < 0;
      a_double_step_5t<O>();
      if (chord)
        a1_chord_add_5t<O>([&](int slot, int coord) { O::s[slot] = coord ? (minus ? mPy : Py) : Px; });
    }
    if (!(O::s[aT5] == BigUInt(0xdead))) { fprintf(stderr, "aT5 was touched\n"); return 2; }
    if (pp_mode) {
      // k_a1_pp_init for P, then k_a1_pp_apply for Q: must give the same pairing
      HostTable T;
      size_t row = 0;
      BigUInt Qx = O::s[aQX], Qy = O::s[aQY];
      O::s[aX] = Px; O::s[aY] = Py; O::s[aQX] = Px; O::s[aQY] = Py;
      O::s[aZ] = BigUInt(1); O::s[aZ2] = BigUInt(1);
      for (int m = (int)n.bits() - 2; m >= 0; m--) {
        a1_pp_tangent<O>(T, row);
        if (m > 0 && n.bit((size_t)m)) a1_pp_chord<O>(T, row);
      }
      enum { qF0 = 0, qF1, qQX, qQY, qT0, qT1, qT2, qT3, qT4 };
      O::s[qF0] = BigUInt(1); O::s[qF1] = BigUInt(); O::s[qQX] = Qx; O::s[qQY] = Qy;
      row = 0;
      for (int m = (int)n.bits() - 2; m >= 0; m--) {
        a_fsqr<O>(qF0, qF1, qT0, qT1);
        a1_pp_eval<O>(T, row, false, qF0, qF1, qQX, qQY, qT0, qT1, qT2, qT3, qT4);
        row += 3;
        if (m > 0 && n.bit((size_t)m)) {
          a1_pp_eval<O>(T, row, true, qF0, qF1, qQX, qQY, qT0, qT1, qT2, qT3, qT4);
          row += 3;
        }
      }
      BigUInt g0 = O::s[qF0], g1 = O::s[qF1];
      O::s[aF0] = g0; O::s[aF1] = g1;
    }
    // a1_publish + k_batch_invert
    BigUInt f0 = O::s[aF0], f1 = O::s[aF1];
    BigUInt N = BigUInt::addmod(BigUInt::mulmod(f0, f0, p), BigUInt::mulmod(f1, f1, p), p);
    BigUInt D = BigUInt::mulmod(N, BigUInt::mulmod(f0, f1, p), p);
    O::s[sD] = BigUInt::invmod(D, p);
    // k_a1_finalexp
    O::s[sTWO] = BigUInt(2);
    uint32_t lw[2] = {l.word(0), l.word(1)};
    a_lucas_final<O>(aF0, aF1, sD, sN, sP, sV0, sV1, sT, sTWO, lw, (int)l.bits());
    printf("%s %s\n", hex(O::s[sV0]).c_str(), hex(O::s[sV1]).c_str());
  }
  return 0;
}
