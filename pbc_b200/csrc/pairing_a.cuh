// pairing_a.cuh -- Type A pairing kernels (y^2 = x^3 + x over F_q, k = 2, 512-bit q).
//
// Device replacement for ecc/a_param.c: a_pairing_proj (:1053-1198), a_miller_evalfn
// (:306-315), compute_abc_tangent_proj (:86-112), compute_abc_line (:114-130), a_tateexp /
// lucas_odd (:226-303), a_pairings_affine (:1283-1383).  Same values, different formulas:
//   * the whole Miller loop is inversion-free.  The reference converts V to affine twice
//     (point_to_affine, :1073-1080) and inverts f when sign1 < 0; here the chord through
//     V = 2^exp2 P and V1 = +-2^exp1 P is evaluated on Jacobian coordinates scaled by
//     Z^3 Z1^3 in F_q, and 1/f is replaced by conj(f) (they differ by the norm, in F_q).  Factors
//     in F_q^* vanish under the (q-1) part of the final exponent, so the reduced pairing -- a
//     canonical residue -- is bit-identical.
//   * the final exponentiation needs 1/N(f) and 1/(f0 f1) only (lucas_odd's P^2-4 equals
//     -4 in1^2 on the norm-1 torus); both come from ONE inversion of N f0 f1, and that inversion
//     is batched across pairings with Montgomery's trick (batch_invert kernel).
// Pipeline per batch:  k_a_miller9 -> k_batch_invert -> k_a_finalexp.
#pragma once
#include "slots.cuh"
#include "a_steps.cuh"
#include "prod_v.cuh"

namespace pbcb200 {

struct AConsts {
  uint32_t h[12];       // cofactor (q+1)/r, little-endian words (Lucas exponent)
  uint32_t hbits;
  int32_t exp2, exp1, sign1;
  uint32_t two[16];     // Montgomery 2
};
__constant__ AConsts c_a;

constexpr int kNA = 16;        // 32-bit limbs of the 512-bit prime
constexpr int kWA = 64;        // wire bytes per coordinate

// Loads P and Q (wire format), converts to Montgomery form, validates y^2 = x^3 + x
// (ecc/curve.c:57-76, :611-623: off-curve input becomes O).  Returns false for O.
// The 2-torsion point (0, 0) -- on the curve, outside G1, the one affine point without a tangent
// line -- is decoded as O as well (documented in include/pbc_b200.h; the reference inverts Z = 0
// there and returns a by-product of that).
template <class O>
__device__ __forceinline__ bool a_load_point(int sx, int sy, int st0, int st1, const uint8_t* p) {
  uint32_t x[kNA];
  limbs_from_be<kNA, kWA>(x, p);
  mont_mul<kNA, true>(x, x, c_fp.r2);
  O::st(sx, x);
  limbs_from_be<kNA, kWA>(x, p + kWA);
  mont_mul<kNA, true>(x, x, c_fp.r2);
  O::st(sy, x);
  O::sqrp(st0, sx);
  O::set_const(st1, c_fp.one);
  O::add(st0, st0, st1);      // x^2 + 1
  O::mul(st0, st0, sx);       // x^3 + x
  O::sqrp(st1, sy);
  return O::eq(st0, st1) && !O::is_zero(sy);
}

// ---------------------------------------------------------------------------------------------
// The Miller loop on NINE slots (round 2).  Round 1's kernel kept 14 slots = 112 KB per
// 128-thread block: two blocks = 8 warps per SM, shared-memory bound (the top stall is the
// fixed-latency wait of the carry chains).  Here
//   * Q (used twice per step, as one operand of a multiplication) lives in a limb-major global array
//     in Montgomery form and is read through Ops::mulg -- L2-resident, the latency is covered by the
//     other warps;
//   * the step is re-scheduled around slot lifetimes (below): V = (X, Y, Z), f and four temporaries;
//   * the two Karatsuba sums of the f update never get a slot (Ops::mul2).
// 9 x 64 B x 128 threads = 72 KB per block: THREE blocks = 12 warps per SM, three per scheduler.
// Cost: 2 Y Z is a product instead of (Y + Z)^2 - B - C (+120 of 8 136 IMAD.WIDE per step); the
// additive calls drop from 22 to 16 (+ one copy).
//
//   g = f^2:            g0 = (f0 + f1)(f0 - f1),  g1 = 2 f0 f1
//   A = X^2, B = Y^2, C = Z^2;  T = A - C,  A' = A + C,  U = 2 A' + T = 3A + C
//   Re l = U Z Qx + X T,   Im l = 2 Y Z Qy
//   X' = T^2,  E = 2 A'^2 - X',  F = (T + Y)^2 - B - X',  Y' = E F,  Z' = 4 B
//   f' = g (Re l + i Im l)
// ---------------------------------------------------------------------------------------------
enum A9Slot { nX, nY, nZ, nF0, nF1, nT0, nT1, nT2, nT3, kA9Slots };

// qx, qy: this thread's Q coordinates in the global array (Montgomery form), vectors n apart.
// a_step_9_line: on entry g = (nT0, nF1) and the f0 slot is free; on exit f' = g l in (nF0, nF1), V doubled.
// LAZY: Re l and f' take one Montgomery reduction per sum of products (Ops::lazy), 544 of the step's 8 256
// multiplier units fewer.  Ops::lazy needs about 130 registers; k_a_miller9 fits it in 168 (three blocks
// per SM), k_a_miller9_shared keeps more live across its calls and does not, so it runs LAZY = false.
template <class O, bool LAZY>
__device__ __forceinline__ void a_step_9_line(const uint4* qx, const uint4* qy, size_t n) {
  O::sqrp(nT1, nX);                                   // A
  O::sqrp(nT2, nY);                                   // B
  O::sqrp(nT3, nZ);                                   // C
  O::sub(nF0, nT1, nT3);                             // T = A - C
  O::add(nT3, nT1, nT3);                             // A' = A + C
  O::dbl(nT1, nT3);
  O::add(nT1, nT1, nF0);                             // U = 3A + C
  O::mulp(nT1, nT1, nZ);                             // U Z
  if constexpr (LAZY) {
    O::lazy(nT1, O::LZ_TWO | O::LZ_GLOBAL_B, nT1, 0, nX, nF0, 0, 0, qx, n);   // Re l = U Z Qx + X T, one reduction
  } else {
    O::mulg(nT1, nT1, qx, n);                        // U Z Qx
    O::mulp(nX, nX, nF0);                            // X T
    O::add(nT1, nT1, nX);                            // Re l                   (X slot is free)
  }
  O::sqrp(nX, nF0);                                  // X' = T^2
  O::sqrx(nT3, nT3, O::SX_SUB_1, 0, 1, nX, 0);       // E = 2 A'^2 - X'
  O::sqrx(nF0, nF0, O::SX_ADD_A | O::SX_SUB_1 | O::SX_SUB_2, nY, 0, nT2, nX);   // F = (T + Y)^2 - B - X'
  O::mulp(nT3, nT3, nF0);                            // Y' (kept in T3 until Y has had its last use)
  O::mulp(nF0, nY, nZ);
  O::dbl(nF0, nF0);
  O::mulg(nF0, nF0, qy, n);                          // Im l = 2 Y Z Qy
  O::dbl(nZ, nT2, 2);                                // Z' = 4 B                (B and Y are dead)
  if constexpr (LAZY) {
    // f' = g l with unreduced products P1 = g0 Re l, P2 = g1 Im l:  f0' = (P1 - P2 + q R) / R,
    // S' = P1 + P2 (- q R) into (nT2, nY), g0 + g1 into nT0, Re l + Im l into nT1
    O::lazy(nF0, O::LZ_TWO | O::LZ_SUB | O::LZ_ADD_QR | O::LZ_KARATSUBA, nT0, nT1, nF1, nF0, nT2, nY, nullptr, 0);
    O::lazy(nF1, O::LZ_SUB_S | O::LZ_ADD_QR, nT0, nT1, 0, 0, nT2, nY, nullptr, 0);   // f1' = ((g0 + g1)(Re l + Im l) - S' + q R) / R
  } else {
    O::template mul2<false>(nT2, nT0, nF1, nT1, nF0);  // (g0 + g1)(Re l + Im l)
    O::mulp(nT0, nT0, nT1);                            // g0 Re l
    O::mulp(nF1, nF1, nF0);                            // g1 Im l
    O::sub(nF0, nT0, nF1);                             // f0'
    O::sub(nT2, nT2, nT0);
    O::sub(nF1, nT2, nF1);                             // f1'
  }
  O::copy(nY, nT3);
}
// g = f^2 into (nT0, nF1): g0 = (f0 + f1)(f0 - f1), g1 = 2 f0 f1   (the f0 slot is free afterwards)
template <class O>
__device__ __forceinline__ void a_step_9_square() {
  O::template mul2<true>(nT0, nF0, nF1, nF0, nF1);
  O::mulp(nF1, nF0, nF1);
  O::dbl(nF1, nF1);
}
template <class O>
__device__ __forceinline__ void a_double_step_9(const uint4* qx, const uint4* qy, size_t n) {
  a_step_9_square<O>();
  a_step_9_line<O, true>(qx, qy, n);
}

// f *= (l0 + i l1) with two temporaries (t0, t1); l0, l1 are preserved
template <class O>
__device__ __forceinline__ void a_fmul_2t(int f0, int f1, int l0, int l1, int t0, int t1) {
  O::template mul2<false>(t0, f0, f1, l0, l1);
  O::mulp(f0, f0, l0);
  O::mulp(f1, f1, l1);
  O::sub(t1, f0, f1);
  O::sub(t0, t0, f0);
  O::sub(f1, t0, f1);
  O::copy(f0, t1);
}

// The chord through V = (x, y, z) and the saved V1 = (X1, Y1, Z1) of pair `idx`, evaluated at phi(Q):
// Re l into t3, Im l into t2; V is consumed.  Weight-(1,2) coordinates, scaled by Z^2 Z1^2
// (compute_abc_line :114-130).
template <class O>
__device__ __forceinline__ void a_chord_line(int x, int y, int z, int t0, int t1, int t2, int t3, const uint4* save,
                                             const uint4* qx, const uint4* qy, size_t n, size_t idx) {
  //   a = Y Z1^2 - Y1 Z^2,  b = Z Z1 (X1 Z - X Z1),  c = X Z Y1 - Y X1 Z1
  O::ld_global(t0, save, 2, n, idx);           // Z1
  O::ld_global(t1, save, 0, n, idx);           // X1
  O::mulp(t2, t1, z);                           // X1 Z
  O::mulp(t3, x, t0);                           // X Z1
  O::sub(t2, t2, t3);
  O::mulp(t2, t2, z);
  O::mulp(t2, t2, t0);                          // b
  O::mulp(t3, x, z);                            // X Z               (last use of X)
  O::ld_global(x, save, 1, n, idx);            // Y1
  O::mulp(t3, t3, x);                           // X Z Y1
  O::mulp(t1, t1, t0);                          // X1 Z1
  O::mulp(t1, t1, y);                           // Y X1 Z1
  O::sub(t3, t3, t1);                           // c
  O::sqrp(t0, t0);                               // Z1^2
  O::mulp(t0, t0, y);                           // Y Z1^2
  O::sqrp(t1, z);                                // Z^2
  O::mulp(t1, t1, x);                           // Y1 Z^2
  O::sub(t0, t0, t1);                           // a
  O::mulg(t0, t0, qx, n);
  O::sub(t3, t3, t0);                           // Re l = c - a Qx
  O::mulg(t2, t2, qy, n);                       // Im l = b Qy
}
// f *= the chord through V = (nX, nY, nZ) and the saved V1 of pair `idx`
template <class O>
__device__ __forceinline__ void a_chord_9(const uint4* save, const uint4* qx, const uint4* qy, size_t n, size_t idx) {
  a_chord_line<O>(nX, nY, nZ, nT0, nT1, nT2, nT3, save, qx, qy, n, idx);
  a_fmul_2t<O>(nF0, nF1, nT3, nT2, nT0, nT1);
}

// f: [2][4][n] uint4 (Montgomery F_q^2), dprod: [4][n] uint4 = N(f) f0 f1 (0 marks "output
// identity"), save: [5][4][n] uint4 scratch for V1 and f1, qm: [2][4][n] uint4 scratch (Montgomery-form Q)
template <int BLOCK>
__global__ void __launch_bounds__(BLOCK)
k_a_miller9(const uint8_t* __restrict__ P, const uint8_t* __restrict__ Q, uint4* __restrict__ f,
            uint4* __restrict__ dprod, uint4* __restrict__ save, uint4* __restrict__ qm, size_t n) {
  using O = Ops<kNA, true, BLOCK>;
  size_t idx = (size_t)blockIdx.x * BLOCK + threadIdx.x;
  const bool live = idx < n;                 // every thread runs the loop: block-wide barrier inside
  if (!live) idx = 0;
  bool okP = a_load_point<O>(nX, nY, nT0, nT1, P + idx * (2 * kWA));
  bool okQ = a_load_point<O>(nT2, nT3, nT0, nT1, Q + idx * (2 * kWA));
  bool valid = okP && okQ;
  if (live) {
    O::st_global(qm, 0, n, idx, nT2);
    O::st_global(qm, 1, n, idx, nT3);
  }
  const uint4* qx = qm + idx;
  const uint4* qy = qm + 4 * n + idx;

  O::set_const(nZ, c_fp.one);
  O::set_const(nF0, c_fp.one);
  uint32_t zero[kNA] = {0};
  O::st(nF1, zero);

  const int exp1 = c_a.exp1, exp2 = c_a.exp2;
  for (int i = 0; i < exp2; i++) {
    __syncthreads();                         // the loop is uniform: keep the block's warps in the same routine (instruction cache)
    if (i == exp1 && live) {
      // V1 = +-V, f1 = f or conj(f) ~ 1/f   (ecc/a_param.c:1162-1169)
      if (c_a.sign1 < 0) { O::neg(nT0, nY); O::neg(nT1, nF1); }
      else               { O::copy(nT0, nY); O::copy(nT1, nF1); }
      O::st_global(save, 0, n, idx, nX);
      O::st_global(save, 1, n, idx, nT0);
      O::st_global(save, 2, n, idx, nZ);
      O::st_global(save, 3, n, idx, nF0);
      O::st_global(save, 4, n, idx, nT1);
    }
    a_double_step_9<O>(qx, qy, n);
  }
  if (!live) return;

  // f *= f1
  O::ld_global(nT2, save, 3, n, idx);
  O::ld_global(nT3, save, 4, n, idx);
  a_fmul_2t<O>(nF0, nF1, nT2, nT3, nT0, nT1);
  a_chord_9<O>(save, qx, qy, n, idx);

  // D = (f0^2 + f1^2) f0 f1;  invalid inputs publish D = 0 (-> identity)
  O::sqrp(nT0, nF0);
  O::sqrp(nT1, nF1);
  O::add(nT0, nT0, nT1);
  O::mulp(nT1, nF0, nF1);
  O::mulp(nT0, nT0, nT1);
  if (!valid) O::st(nT0, zero);
  O::st_global(f, 0, n, idx, nF0);
  O::st_global(f, 1, n, idx, nF1);
  O::st_global(dprod, 0, n, idx, nT0);
}

// ---------------------------------------------------------------------------------------------
// Shared Miller accumulator (a_pairings_affine, ecc/a_param.c:1283-1383: ONE f for the n pairs of a
// product, f <- f^2 once per step, then f <- f l_j for every pair).  One thread owns M consecutive pairs
// of one product: per step it squares f once and runs the line / doubling part of the nine-slot step
// for each pair in turn, the pair's V = (X, Y, Z) parked in a limb-major global array between its turns.
// 2 + 15 M multiplications per step instead of 17 M.  The thread count drops by M, so M stays small
// (the host picks it; M = 1 is k_a_miller9): with 2^16 outputs of 16 pairs a wave (three 128-thread
// blocks per SM: 50 688 threads on the 132 SMs of an H100) is already 5 % of the batch at M = 1.
//   f, dprod: [..][n_thr] (one partial Miller value per thread);  save, qm, vj: per pair, n_pairs = n_thr M
// ---------------------------------------------------------------------------------------------
template <int BLOCK>
__global__ void __launch_bounds__(BLOCK)
k_a_miller9_shared(const uint8_t* __restrict__ P, const uint8_t* __restrict__ Q, uint4* __restrict__ f,
                   uint4* __restrict__ dprod, uint4* __restrict__ save, uint4* __restrict__ qm,
                   uint4* __restrict__ vj, size_t n_thr, size_t M) {
  using O = Ops<kNA, true, BLOCK>;
  size_t idx = (size_t)blockIdx.x * BLOCK + threadIdx.x;
  const bool live = idx < n_thr;
  if (!live) idx = 0;
  const size_t np = n_thr * M, p0 = idx * M;
  bool valid = true;
  for (size_t j = 0; j < M; j++) {
    const size_t pr = p0 + j;
    bool okP = a_load_point<O>(nX, nY, nT0, nT1, P + pr * (2 * kWA));
    bool okQ = a_load_point<O>(nT2, nT3, nT0, nT1, Q + pr * (2 * kWA));
    valid = valid && okP && okQ;
    O::set_const(nZ, c_fp.one);
    if (live) {
      O::st_global(qm, 0, np, pr, nT2);
      O::st_global(qm, 1, np, pr, nT3);
      O::st_global(vj, 0, np, pr, nX);
      O::st_global(vj, 1, np, pr, nY);
      O::st_global(vj, 2, np, pr, nZ);
    }
  }
  O::set_const(nF0, c_fp.one);
  uint32_t zero[kNA] = {0};
  O::st(nF1, zero);

  const int exp1 = c_a.exp1, exp2 = c_a.exp2;
  for (int i = 0; i < exp2; i++) {
    __syncthreads();
    if (i == exp1 && live) {
      // f1 = f or conj(f) ~ 1/f, once per thread (kept with the thread's first pair)
      if (c_a.sign1 < 0) O::neg(nT1, nF1); else O::copy(nT1, nF1);
      O::st_global(save, 3, np, p0, nF0);
      O::st_global(save, 4, np, p0, nT1);
    }
    a_step_9_square<O>();
    for (size_t j = 0; j < M; j++) {
      const size_t pr = p0 + j;
      if (j) O::copy(nT0, nF0);               // the running product where the step expects g0
      O::ld_global(nX, vj, 0, np, pr);
      O::ld_global(nY, vj, 1, np, pr);
      O::ld_global(nZ, vj, 2, np, pr);
      if (i == exp1 && live) {
        // V1 = +-V of this pair   (ecc/a_param.c:1162-1169)
        if (c_a.sign1 < 0) O::neg(nF0, nY); else O::copy(nF0, nY);
        O::st_global(save, 0, np, pr, nX);
        O::st_global(save, 1, np, pr, nF0);
        O::st_global(save, 2, np, pr, nZ);
      }
      a_step_9_line<O, false>(qm + pr, qm + 4 * np + pr, np);
      if (live) {
        O::st_global(vj, 0, np, pr, nX);
        O::st_global(vj, 1, np, pr, nY);
        O::st_global(vj, 2, np, pr, nZ);
      }
    }
  }
  if (!live) return;

  O::ld_global(nT2, save, 3, np, p0);
  O::ld_global(nT3, save, 4, np, p0);
  a_fmul_2t<O>(nF0, nF1, nT2, nT3, nT0, nT1);          // f *= f1
  for (size_t j = 0; j < M; j++) {
    const size_t pr = p0 + j;
    O::ld_global(nX, vj, 0, np, pr);
    O::ld_global(nY, vj, 1, np, pr);
    O::ld_global(nZ, vj, 2, np, pr);
    a_chord_9<O>(save, qm + pr, qm + 4 * np + pr, np, pr);
  }
  O::sqrp(nT0, nF0);
  O::sqrp(nT1, nF1);
  O::add(nT0, nT0, nT1);
  O::mulp(nT1, nF0, nF1);
  O::mulp(nT0, nT0, nT1);
  if (!valid) O::st(nT0, zero);
  O::st_global(f, 0, n_thr, idx, nF0);
  O::st_global(f, 1, n_thr, idx, nF1);
  O::st_global(dprod, 0, n_thr, idx, nT0);
}

// ---------------------------------------------------------------------------------------------
// element_prod_pairing (include/pbc_pairing.h:153-171 -> a_pairings_affine, ecc/a_param.c:1283-1383).
// The reference shares one accumulator f between the k Miller loops; here every (P_j, Q_j) pair
// runs its own k_a_miller9 thread (k times more parallelism for a 2^16-output batch) and the k
// Miller values of one output are multiplied afterwards.  prod_j f_j differs from the reference's
// shared accumulator only by factors in F_q^*, which the final exponentiation kills.
//   f_in [2][4][n_in], d_in [4][n_in]  (n_in = n_out * k; d = 0 marks an O / off-curve input),
//   f_out[2][4][n_out], d_out[4][n_out] = N(F) F0 F1, or 0: ANY bad input -> the whole product is 1.
// ---------------------------------------------------------------------------------------------
enum APSlot { pF0, pF1, pL0, pL1, pT0, pT1, pT2, kAPSlots };

template <int BLOCK>
__global__ void __launch_bounds__(BLOCK)
k_a_prod(const uint4* __restrict__ f_in, const uint4* __restrict__ d_in, uint4* __restrict__ f_out,
         uint4* __restrict__ d_out, size_t k, size_t n_out, size_t n_in) {
  using O = Ops<kNA, true, BLOCK>;
  size_t idx = (size_t)blockIdx.x * BLOCK + threadIdx.x;
  if (idx >= n_out) return;
  bool valid = true;
  uint32_t zero[kNA] = {0};
  O::set_const(pF0, c_fp.one);
  O::st(pF1, zero);
  for (size_t j = 0; j < k; j++) {
    size_t src = idx * k + j;
    O::ld_global(pL0, f_in, 0, n_in, src);
    O::ld_global(pL1, f_in, 1, n_in, src);
    O::ld_global(pT0, d_in, 0, n_in, src);
    valid = valid && !O::is_zero(pT0);
    a_fmul<O>(pF0, pF1, pL0, pL1, pT0, pT1, pT2);
  }
  O::sqrp(pT0, pF0);
  O::sqrp(pT1, pF1);
  O::add(pT0, pT0, pT1);
  O::mul(pT1, pF0, pF1);
  O::mul(pT0, pT0, pT1);
  if (!valid) O::st(pT0, zero);
  O::st_global(f_out, 0, n_out, idx, pF0);
  O::st_global(f_out, 1, n_out, idx, pF1);
  O::st_global(d_out, 0, n_out, idx, pT0);
}

// ---------------------------------------------------------------------------------------------
// pairing_pp_init / pairing_pp_apply (ecc/a_param.c:149-220, 317-360): one fixed first argument.
// k_a_pp_init walks V = P, 2P, 4P, ... once (one thread; Jacobian, inversion-free) and stores the
// line coefficients (a, b, c) of every tangent plus the final chord, each scaled by some element of
// F_q^* (the reference stores the affine ones; the scale dies in the final exponentiation):
//   tab[(3 i + {0,1,2}) * 16 ..]  i < exp2: tangent at 2^i P;  i = exp2: chord through V, V1
//   tab[3 (exp2 + 1) * 16]        1 if P decoded to a finite point on the curve, else 0.
// k_a_pp_apply then costs 7 multiplications per bit instead of 19:
//   f <- f^2 (c - a Qx + i b Qy).
// ---------------------------------------------------------------------------------------------
template <int BLOCK>
__global__ void __launch_bounds__(BLOCK)
k_a_pp_init(const uint8_t* __restrict__ P, uint32_t* __restrict__ tab) {
  using O = Ops<kNA, true, BLOCK>;
  if (blockIdx.x != 0 || threadIdx.x != 0) return;
  // slots: aX aY aZ aZ2 = V; aQX aQY aF0 = V1 (X1, Y1, Z1); aT0..aT5 scratch
  bool okP = a_load_point<O>(aX, aY, aT0, aT1, P);
  O::set_const(aZ, c_fp.one);
  O::set_const(aZ2, c_fp.one);
  const int exp1 = c_a.exp1, exp2 = c_a.exp2;
  uint32_t x[kNA];
  auto emit = [&](int row, int slot) {
    O::ld(x, slot);
#pragma unroll
    for (int k = 0; k < kNA; k++) tab[(size_t)row * kNA + k] = x[k];
  };
  for (int i = 0; i < exp2; i++) {
    if (i == exp1) {
      O::copy(aQX, aX);
      if (c_a.sign1 < 0) O::neg(aQY, aY); else O::copy(aQY, aY);
      O::copy(aF0, aZ);
    }
    // tangent (compute_abc_tangent_proj, ecc/a_param.c:86-112), sign-flipped as a whole:
    //   a = M Z^2, b = 2 Y Z^3, c = X M - 2 Y^2     with M = 3 X^2 + Z^4;  line = c + a Qx... see apply
    O::sqrp(aT0, aX);
    O::sqrp(aT1, aZ2);
    O::dbl(aT2, aT0);
    O::add(aT0, aT0, aT2);
    O::add(aT0, aT0, aT1);          // M
    O::sqrp(aT1, aY);                // Y^2
    O::mul(aT3, aT0, aZ2);          // a = M Z^2
    emit(3 * i + 0, aT3);
    O::mul(aT5, aX, aT0);
    O::sub(aT5, aT5, aT1);
    O::sub(aT5, aT5, aT1);          // c = X M - 2 Y^2
    emit(3 * i + 2, aT5);
    O::mul(aT2, aX, aT1);
    O::dbl(aT2, aT2, 2);            // S = 4 X Y^2
    O::mul(aZ, aY, aZ);
    O::dbl(aZ, aZ);                 // Z' = 2 Y Z
    O::mul(aT3, aZ, aZ2);           // b = Z' Z^2
    emit(3 * i + 1, aT3);
    O::sqrp(aZ2, aZ);
    O::sqrp(aT5, aT0);
    O::sub(aX, aT5, aT2);
    O::sub(aX, aX, aT2);            // X' = M^2 - 2 S
    O::sqrp(aT1, aT1);
    O::dbl(aT1, aT1, 3);            // 8 Y^4
    O::sub(aT2, aT2, aX);
    O::mulsub(aY, aT0, aT2, aT1);   // Y' = M (S - X') - 8 Y^4
  }
  // chord through V = (X, Y, Z) and V1 = (X1, Y1, Z1), scaled by Z^3 Z1^3 (compute_abc_line :114-130)
  //   a = Y Z1^3 - Y1 Z^3,  b = X1 Z1 Z^3 - X Z Z1^3,  c = X Z Y1 - Y X1 Z1
  O::mul(aT1, aZ2, aZ);             // Z^3
  O::sqrp(aT2, aF0);
  O::mul(aT2, aT2, aF0);            // Z1^3
  O::mul(aT3, aX, aZ);              // X Z
  O::mul(aT4, aQX, aF0);            // X1 Z1
  O::mul(aT0, aT3, aQY);            // X Z Y1
  O::mul(aT5, aY, aT4);             // Y X1 Z1
  O::sub(aT0, aT0, aT5);            // c
  emit(3 * exp2 + 2, aT0);
  O::mul(aT4, aT4, aT1);
  O::mul(aT3, aT3, aT2);
  O::sub(aT4, aT4, aT3);            // b
  emit(3 * exp2 + 1, aT4);
  O::mul(aT2, aY, aT2);
  O::mul(aT1, aQY, aT1);
  O::sub(aT2, aT2, aT1);            // a
  emit(3 * exp2 + 0, aT2);
  tab[(size_t)3 * (exp2 + 1) * kNA] = okP ? 1u : 0u;
}

enum APPSlot { qF0, qF1, qQX, qQY, qS0, qS1, qT0, qT1, qT2, qT3, qT4, kAPPSlots };

// tangent rows hold (a, b, c) with line value  (c + a Qx) + i (b Qy);  the chord row holds the
// reference's (a, b, c) with line value (c - a Qx) + i (b Qy)   (a_miller_evalfn :306-315).
template <int BLOCK>
__global__ void __launch_bounds__(BLOCK)
k_a_pp_apply(const uint32_t* __restrict__ tab, const uint8_t* __restrict__ Q, uint4* __restrict__ f,
             uint4* __restrict__ dprod, size_t n) {
  using O = Ops<kNA, true, BLOCK>;
  size_t idx = (size_t)blockIdx.x * BLOCK + threadIdx.x;
  bool live = idx < n;
  size_t src = live ? idx : 0;
  bool okQ = a_load_point<O>(qQX, qQY, qT0, qT1, Q + src * (2 * kWA));
  const int exp1 = c_a.exp1, exp2 = c_a.exp2;
  bool valid = okQ && tab[(size_t)3 * (exp2 + 1) * kNA] != 0;
  uint32_t zero[kNA] = {0};
  O::set_const(qF0, c_fp.one);
  O::st(qF1, zero);
  for (int i = 0; i <= exp2; i++) {
    const uint32_t* row = tab + (size_t)3 * i * kNA;
    if (i == exp1) {
      O::copy(qS0, qF0);
      if (c_a.sign1 < 0) O::neg(qS1, qF1); else O::copy(qS1, qF1);
    }
    if (i < exp2) {
      // f = f^2
      O::add(qT0, qF0, qF1);
      O::sub(qT1, qF0, qF1);
      O::mul(qF1, qF0, qF1);
      O::dbl(qF1, qF1);
      O::mul(qF0, qT0, qT1);
    } else {
      a_fmul<O>(qF0, qF1, qS0, qS1, qT0, qT1, qT2);   // f *= f1
    }
    O::set_const(qT0, row);                  // a
    O::mul(qT0, qT0, qQX);
    O::set_const(qT1, row + 2 * kNA);        // c
    if (i < exp2) O::add(qT0, qT1, qT0); else O::sub(qT0, qT1, qT0);
    O::set_const(qT1, row + kNA);            // b
    O::mul(qT1, qT1, qQY);
    a_fmul<O>(qF0, qF1, qT0, qT1, qT2, qT3, qT4);
  }
  if (!live) return;
  O::sqrp(qT0, qF0);
  O::sqrp(qT1, qF1);
  O::add(qT0, qT0, qT1);
  O::mul(qT1, qF0, qF1);
  O::mul(qT0, qT0, qT1);
  if (!valid) O::st(qT0, zero);
  O::st_global(f, 0, n, idx, qF0);
  O::st_global(f, 1, n, idx, qF1);
  O::st_global(dprod, 0, n, idx, qT0);
}

// slot map of the final-exponentiation kernel: the Lucas ladder keeps V_0, V_1 and P, plus W = N^2 Dinv
// for the end; the constant 2 is read from c_a.  4 x 64 B x 128 threads = 32 KB per block: six blocks
// (24 warps) per SM.
enum AFSlot { fV0, fV1, fP, fW, kAFSlots };

// out: n * 128 bytes, wire format of F_q^2 (arith/fieldquadratic.c:323-329: x || y).
template <int BLOCK>
__global__ void __launch_bounds__(BLOCK, 6)
k_a_finalexp(const uint4* __restrict__ f, const uint4* __restrict__ dinv, uint8_t* __restrict__ out,
             size_t n) {
  using O = Ops<kNA, true, BLOCK>;
  size_t idx = (size_t)blockIdx.x * BLOCK + threadIdx.x;
  if (idx >= n) return;
  O::ld_global(fV0, f, 0, n, idx);
  O::ld_global(fV1, f, 1, n, idx);
  O::ld_global(fW, dinv, 0, n, idx);
  bool identity = O::is_zero(fW);
  // N = f0^2 + f1^2;  1/N = Dinv f0 f1;  P = 2 (f0^2 - f1^2) / N;  W = N^2 Dinv
  O::mul(fP, fV0, fV1);
  O::mul(fP, fP, fW);                       // 1/N
  O::sqr(fW, fV1);
  O::sqr(fV1, fV0);
  O::sub(fV0, fV1, fW);
  O::add(fV1, fV1, fW);                     // N
  O::dbl(fV0, fV0);
  O::mul(fP, fP, fV0);                      // P
  O::sqr(fW, fV1);
  O::mulg(fW, fW, dinv + idx, n);           // W (Dinv read again inside the call: no registers held)
  // Lucas ladder, lucas_odd (ecc/a_param.c:226-262): V_0 = 2, V_1 = P
  O::set_const(fV0, c_a.two);
  O::copy(fV1, fP);
  for (int j = (int)c_a.hbits - 1; j >= 0; j--) {
    bool bit = j > 0 && ((c_a.h[j >> 5] >> (j & 31)) & 1u);   // last step takes the clear branch
    int d = bit ? fV0 : fV1, s = bit ? fV1 : fV0;
    O::mulsub(d, fV0, fV1, fP);
    O::sqrsub(s, s, c_a.two);
  }
  // out0 = V_h / 2;  out1 = (2 V_{h+1} - P V_h) W / 8
  O::dbl(fV1, fV1);
  O::mul(fP, fP, fV0);
  O::sub(fV1, fV1, fP);
  O::mul(fV1, fV1, fW);
  O::halve(fV1, fV1, 3);
  O::halve(fV0, fV0);

  uint32_t x[kNA], one[kNA] = {1};
  uint8_t* o = out + idx * (2 * kWA);
  O::ld(x, fV0);
  mont_mul<kNA, true>(x, x, one);           // leave Montgomery form (arith/montfp.c:64-80)
  if (identity) {
#pragma unroll
    for (int k = 0; k < kNA; k++) x[k] = one[k];
  }
  limbs_to_be<kNA, kWA>(o, x);
  O::ld(x, fV1);
  mont_mul<kNA, true>(x, x, one);
  if (identity) {
#pragma unroll
    for (int k = 0; k < kNA; k++) x[k] = 0;
  }
  limbs_to_be<kNA, kWA>(o + kWA, x);
}

}  // namespace pbcb200
