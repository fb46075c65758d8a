// a_steps.cuh -- slot programs shared by the Type A and Type A1 kernels.
//
// Each routine is a straight-line sequence of field operations on numbered slots, written against
// a policy class O (Ops<N, FULL, BLOCK> of slots.cuh on the device).  Nothing here depends on the
// limb count, the modulus or CUDA: tests/host/a_steps_host.cpp instantiates the same templates
// with a big-integer O on the CPU and checks them against reference fixtures, so the formulas are
// pinned without a GPU.
#pragma once

#ifdef __CUDACC__
#define PBC_STEP __device__ __forceinline__
#else
#define PBC_STEP inline
#endif

namespace pbcb200 {

// slot map of the Miller kernel
enum ASlot { aX, aY, aZ, aZ2, aF0, aF1, aQX, aQY, aT0, aT1, aT2, aT3, aT4, aT5, kASlots };

// f *= (L0 + i L1), Karatsuba (arith/fieldquadratic.c:425-457 fi_mul), temporaries t0..t2
template <class O>
PBC_STEP void a_fmul(int f0, int f1, int l0, int l1, int t0, int t1, int t2) {
  O::add(t0, f0, f1);
  O::add(t1, l0, l1);
  O::mul(t0, t0, t1);
  O::mul(t1, f0, l0);
  O::mul(t2, f1, l1);
  O::sub(f0, t1, t2);
  O::sub(t0, t0, t1);
  O::sub(f1, t0, t2);
}

// One Miller doubling step:  f <- f^2 * l_{V,V}(phi(Q)),  V <- 2V   (Jacobian, a = 1).
// 13 multiplications + 6 squarings (reference: 23 multiplications, ecc/a_param.c:1082-1139).
// Five temporaries (aT0..aT4), aT5 is never touched: 13 slots instead of 14, which at 136 bytes per slot
// is the difference between 96 and 128 threads per block for the 34-limb field (one warp per scheduler
// instead of three warps on four).
template <class O>
PBC_STEP void a_double_step_5t() {
  // f = f^2
  O::add(aT0, aF0, aF1);
  O::sub(aT1, aF0, aF1);
  O::mul(aF1, aF0, aF1);
  O::dbl(aF1, aF1);
  O::mul(aF0, aT0, aT1);
  O::sqr(aT0, aX);
  O::sqr(aT1, aZ2);
  O::dbl(aT2, aT0);
  O::add(aT0, aT0, aT2);
  O::add(aT0, aT0, aT1);           // M = 3 X^2 + Z^4
  O::sqr(aT1, aY);                 // Y^2
  O::mul(aT4, aT0, aZ2);
  O::mul(aT4, aT4, aQX);           // M Z^2 Qx
  O::mul(aT3, aX, aT0);
  O::sub(aT3, aT3, aT1);
  O::sub(aT3, aT3, aT1);
  O::add(aT4, aT4, aT3);           // Re l = X M - 2 Y^2 + M Z^2 Qx
  O::mul(aT2, aX, aT1);
  O::dbl(aT2, aT2, 2);             // S = 4 X Y^2   (last use of the old X)
  O::mul(aZ, aY, aZ);
  O::dbl(aZ, aZ);                  // Z' = 2 Y Z    (last use of the old Y)
  O::mul(aT3, aZ, aZ2);
  O::mul(aT3, aT3, aQY);           // Im l = Z' Z^2 Qy
  O::sqr(aZ2, aZ);
  O::sqr(aX, aT0);
  O::sub(aX, aX, aT2);
  O::sub(aX, aX, aT2);             // X' = M^2 - 2 S
  O::sqr(aT1, aT1);
  O::dbl(aT1, aT1, 3);             // 8 Y^4
  O::sub(aT2, aT2, aX);
  O::mul(aY, aT0, aT2);
  O::sub(aY, aY, aT1);             // Y' = M (S - X') - 8 Y^4
  a_fmul<O>(aF0, aF1, aT4, aT3, aT0, aT1, aT2);
}
// Chord through V = (X, Y, Z) (Jacobian, Z2 = Z^2) and the affine point P = (xP, yP), evaluated at
// phi(Q); then V <- V + P.
// Device replacement for compute_abc_line_proj + a_miller_evalfn + proj_add of a1_pairing_proj
// (ecc/a_param.c:1820-1837, :306-315, :1869-1896); same line, same point, fewer products:
//   H = xP Z^2 - X,  R = yP Z^3 - Y
//   a = -R,  b = H Z (= Z of the sum),  c = yP Z X - xP Y;   l(phi(Q)) = (c - a Qx) + i (b Qy)
//   X3 = R^2 - H^3 - 2 X H^2,  Y3 = R (X H^2 - X3) - Y H^3,  Z3 = b
// 16 multiplications + 3 squarings including the f update.  Temporaries aT0..aT4 and aZ2.
// P is fetched through `ldP(slot, coordinate)` (0 = x, 1 = y) when it is needed: x into aT4, y into
// the Z^2 slot once Z^2 has had its last use; the point addition is finished before the f update
// so that the update finds three free temporaries.
template <class O, class LoadP>
PBC_STEP void a1_chord_add_5t(LoadP ldP) {
  ldP(aT4, 0);                     // xP
  O::mul(aT0, aZ2, aZ);            // Z^3
  O::mul(aT1, aT4, aZ2);
  O::sub(aT1, aT1, aX);            // H            (last use of Z^2)
  ldP(aZ2, 1);                     // yP
  O::mul(aT0, aZ2, aT0);           // yP Z^3
  O::sub(aT2, aY, aT0);            // a = Y - yP Z^3
  O::sub(aT0, aT0, aY);            // R
  O::mul(aT3, aZ2, aZ);
  O::mul(aT3, aT3, aX);            // yP Z X
  O::mul(aT4, aT4, aY);            // xP Y
  O::sub(aT3, aT3, aT4);           // c
  O::mul(aZ, aT1, aZ);             // b = H Z = Z of the sum
  O::mul(aT2, aT2, aQX);
  O::sub(aT2, aT3, aT2);           // Re l = c - a Qx
  O::mul(aT4, aZ, aQY);            // Im l = b Qy
  O::sqr(aT3, aT1);                // H^2
  O::mul(aZ2, aT3, aT1);           // H^3
  O::mul(aT3, aT3, aX);            // X H^2
  O::sqr(aX, aT0);
  O::sub(aX, aX, aZ2);
  O::sub(aX, aX, aT3);
  O::sub(aX, aX, aT3);             // X3
  O::sub(aT3, aT3, aX);
  O::mul(aT3, aT3, aT0);           // R (X H^2 - X3)
  O::mul(aZ2, aZ2, aY);            // Y H^3
  O::sub(aY, aT3, aZ2);            // Y3
  a_fmul<O>(aF0, aF1, aT2, aT4, aT0, aT1, aT3);
  O::sqr(aZ2, aZ);
}

// ---- fixed first argument (pairing_pp_init / pairing_pp_apply, ecc/a_param.c:1632-1818) ----
// Tab: line-coefficient table;  tab.template store<O>(row, slot) / tab.template load<O>(slot, row).
// Rows come in groups of three (a, b, c), in loop order.
//
// Tangent at V = (aX, aY, aZ, aZ2) (compute_abc_tangent_proj, :86-112, sign-flipped as a whole):
//   a = M Z^2, b = 2 Y Z^3, c = X M - 2 Y^2, M = 3 X^2 + Z^4;   l(phi(Q)) = (c + a Qx) + i (b Qy)
// then V <- 2V.  Temporaries aT0..aT3, aT5.
template <class O, class Tab>
PBC_STEP void a1_pp_tangent(Tab& tab, size_t& row) {
  O::sqr(aT0, aX);
  O::sqr(aT1, aZ2);
  O::dbl(aT2, aT0);
  O::add(aT0, aT0, aT2);
  O::add(aT0, aT0, aT1);          // M
  O::sqr(aT1, aY);                // Y^2
  O::mul(aT3, aT0, aZ2);
  tab.template store<O>(row++, aT3);   // a
  O::mul(aT2, aX, aT1);
  O::dbl(aT2, aT2, 2);            // S = 4 X Y^2
  O::mul(aT5, aX, aT0);
  O::sub(aT5, aT5, aT1);
  O::sub(aT5, aT5, aT1);          // c
  O::mul(aZ, aY, aZ);
  O::dbl(aZ, aZ);                 // Z' = 2 Y Z
  O::mul(aT3, aZ, aZ2);
  tab.template store<O>(row++, aT3);   // b
  tab.template store<O>(row++, aT5);   // c
  O::sqr(aZ2, aZ);
  O::sqr(aT5, aT0);
  O::sub(aX, aT5, aT2);
  O::sub(aX, aX, aT2);            // X' = M^2 - 2 S
  O::sqr(aT1, aT1);
  O::dbl(aT1, aT1, 3);            // 8 Y^4
  O::sub(aT2, aT2, aX);
  O::mul(aY, aT0, aT2);
  O::sub(aY, aY, aT1);            // Y' = M (S - X') - 8 Y^4
}
// Chord through V and the affine P = (aQX, aQY) (compute_abc_line_proj, :1820-1837):
//   a = Y - yP Z^3, b = (xP Z^2 - X) Z, c = yP Z X - xP Y;   l(phi(Q)) = (c - a Qx) + i (b Qy)
// then V <- V + P (proj_add, :1869-1896).  Temporaries aT0..aT4.
template <class O, class Tab>
PBC_STEP void a1_pp_chord(Tab& tab, size_t& row) {
  O::mul(aT0, aZ2, aZ);            // Z^3
  O::mul(aT1, aQX, aZ2);
  O::sub(aT1, aT1, aX);            // H
  O::mul(aT0, aQY, aT0);           // yP Z^3
  O::sub(aT2, aY, aT0);            // a
  tab.template store<O>(row++, aT2);
  O::sub(aT0, aT0, aY);            // R
  O::mul(aT3, aQY, aZ);
  O::mul(aT3, aT3, aX);            // yP Z X
  O::mul(aT4, aQX, aY);            // xP Y
  O::sub(aT3, aT3, aT4);           // c
  O::mul(aZ, aT1, aZ);             // b = H Z
  tab.template store<O>(row++, aZ);
  tab.template store<O>(row++, aT3);
  O::sqr(aT2, aT1);                // H^2
  O::mul(aT3, aT2, aT1);           // H^3
  O::mul(aT2, aT2, aX);            // X H^2
  O::sqr(aX, aT0);
  O::sub(aX, aX, aT3);
  O::sub(aX, aX, aT2);
  O::sub(aX, aX, aT2);             // X3
  O::sub(aT2, aT2, aX);
  O::mul(aT2, aT2, aT0);
  O::mul(aT3, aT3, aY);
  O::sub(aY, aT2, aT3);            // Y3
  O::sqr(aZ2, aZ);
}
// f *= line(row .. row+2) evaluated at phi(Q) = (-Qx, i Qy)
template <class O, class Tab>
PBC_STEP void a1_pp_eval(const Tab& tab, size_t row, bool chord, int sF0, int sF1, int sQX, int sQY,
                         int t0, int t1, int t2, int t3, int t4) {
  tab.template load<O>(t0, row);             // a
  O::mul(t0, t0, sQX);
  tab.template load<O>(t1, row + 2);         // c
  if (chord) O::sub(t0, t1, t0); else O::add(t0, t1, t0);
  tab.template load<O>(t1, row + 1);         // b
  O::mul(t1, t1, sQY);
  a_fmul<O>(sF0, sF1, t0, t1, t2, t3, t4);
}
// f = f^2  (arith/fieldquadratic.c:459-477)
template <class O>
PBC_STEP void a_fsqr(int sF0, int sF1, int t0, int t1) {
  O::add(t0, sF0, sF1);
  O::sub(t1, sF0, sF1);
  O::mul(sF1, sF0, sF1);
  O::dbl(sF1, sF1);
  O::mul(sF0, t0, t1);
}

// Final exponentiation f -> f^((q-1) h) for q = 3 mod 4, h even, on slots (a_tateexp / lucas_odd,
// ecc/a_param.c:226-303; for Type A1 the reference calls element_pow_mpz by l instead,
// :2003-2007 -- same group element, hence the same canonical bytes).
//   in:  sF0, sF1 = f;  sD = 1 / ((f0^2 + f1^2) f0 f1);  sTWO = 2
//   out: sV0 = Re, sV1 = Im.   h: little-endian words, hbits significant bits.
template <class O>
PBC_STEP void a_lucas_final(int sF0, int sF1, int sD, int sN, int sP, int sV0, int sV1, int sT0,
                            int sTWO, const unsigned* h, int hbits) {
  // N = f0^2 + f1^2, W = f0 f1;  1/N = D W;  P = 2 (f0^2 - f1^2) / N  = trace of conj(f)/f
  O::sqr(sV0, sF0);
  O::sqr(sV1, sF1);
  O::add(sN, sV0, sV1);
  O::sub(sP, sV0, sV1);
  O::dbl(sP, sP);
  O::mul(sT0, sF0, sF1);
  O::mul(sT0, sT0, sD);
  O::mul(sP, sP, sT0);
  // Lucas ladder: V_0 = 2, V_1 = P
  O::copy(sV0, sTWO);
  O::copy(sV1, sP);
  for (int j = hbits - 1; j >= 0; j--) {
    bool bit = j > 0 && ((h[j >> 5] >> (j & 31)) & 1u);   // last step takes the clear branch
    int d = bit ? sV0 : sV1, s = bit ? sV1 : sV0;
    O::mul(d, sV0, sV1);
    O::sub(d, d, sP);
    O::sqr(s, s);
    O::sub(s, s, sTWO);
  }
  // Re = V_h / 2;  Im = (2 V_{h+1} - P V_h) N^2 D / 8
  O::dbl(sV1, sV1);
  O::mul(sT0, sP, sV0);
  O::sub(sV1, sV1, sT0);
  O::sqr(sN, sN);
  O::mul(sN, sN, sD);
  O::mul(sV1, sV1, sN);
  O::halve(sV1, sV1, 3);
  O::halve(sV0, sV0);
}

}  // namespace pbcb200
