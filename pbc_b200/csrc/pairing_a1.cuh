// pairing_a1.cuh -- Type A1 pairing kernels: the Type A curve y^2 = x^3 + x over an arbitrary
// prime p = l n - 1 = 3 mod 4 (k = 2), group order n of any shape (composite-order groups).
//
// Device replacement for ecc/a_param.c:1564-2273: a1_pairing_proj (:1840-2015), a1_pairings_affine
// (:2100-2193), a1_pairing_pp_init / _apply (:1632-1818).  Same values, different formulas:
//   * one pairing per thread, field elements in the shared-memory slot machine of slots.cuh with
//     N = 34 limbs (any p below 2^1087; param/a1.param has 1033 bits);
//   * the loop over the bits of n is the reference's (tangent, double, chord + add where the bit is
//     set, square), V in Jacobian coordinates against the affine P, no inversion anywhere;
//   * final exponent (p - 1) l: f^(p-1) = conj(f)/f needs 1/N(f), batched across pairings with
//     Montgomery's trick (k_batch_invert); the power by l runs as a Lucas ladder on the trace
//     (a_lucas_final) where the reference calls element_pow_mpz (:2003-2007).  The result is the
//     same element of F_p^2, so its canonical bytes are identical.
//   * products of pairings: every (P_j, Q_j) runs its own Miller thread and the Miller values of
//     one output are multiplied afterwards (the reference shares one accumulator, :2147-2160);
//     factors in F_p^* die in the final exponentiation.
//   * fixed first argument: the line coefficients of every tangent and chord are tabulated once
//     per P; the reference merges tangent and chord into one conic (:1689-1713), here they stay
//     separate rows -- same product.
// Pipeline per batch:  k_a1_miller (-> k_a1_prod) -> k_batch_invert<34> -> k_a1_finalexp.
#pragma once
#include "common_kernels.cuh"
#include "a_steps.cuh"
#include "prod_v.cuh"

namespace pbcb200 {

constexpr int kNA1 = 34;       // 32-bit limbs: p < 2^1087

// The Miller kernel runs the five-temporary slot programs of a_steps.cuh: 13 slots, 128 threads per
// block = one warp per scheduler (a block of four warps takes about the time of a block of three, so more
// pairings finish per SM).  It scans the non-adjacent form of n (host_naf.hpp) instead of its bits: a
// third fewer chord steps (-11 % multiplier work for a1.param).  Both are pinned on the CPU
// (tests/test_a_steps_host.py).
constexpr int kA1MillerSlots = 13;
constexpr int kA1MillerBlock = 128;

struct alignas(16) A1Consts {
  uint32_t n[kMaxLimbs];       // group order (plain integer, little-endian words)
  uint32_t two[kMaxLimbs];     // Montgomery 2
  uint32_t l[2];               // cofactor (p + 1) / n, even (Lucas exponent)
  uint32_t lbits;
  uint32_t nbits;
  uint32_t wb;                 // wire bytes per F_p coordinate = ceil(bits(p) / 8)
  uint32_t pad[3];
};
__constant__ A1Consts c_a1;
struct alignas(16) A1Naf {
  uint32_t nz[kMaxLimbs];      // bit i: digit i is non-zero
  uint32_t neg[kMaxLimbs];     // bit i: digit i is -1
  uint32_t len;                // number of digits (top digit is +1)
  uint32_t pad[3];
};
__constant__ A1Naf c_a1naf;

// wire bytes (big-endian, wb per coordinate, any alignment) -> limbs
__device__ __forceinline__ void a1_limbs_from_be(uint32_t* x, const uint8_t* p, int wb) {
#pragma unroll
  for (int k = 0; k < kNA1; k++) {
    uint32_t w = 0;
#pragma unroll
    for (int j = 0; j < 4; j++) {
      int pos = wb - 1 - (4 * k + j);
      if (pos >= 0) w |= (uint32_t)p[pos] << (8 * j);
    }
    x[k] = w;
  }
}
__device__ __forceinline__ void a1_limbs_to_be(uint8_t* p, const uint32_t* x, int wb) {
#pragma unroll
  for (int k = 0; k < kNA1; k++) {
#pragma unroll
    for (int j = 0; j < 4; j++) {
      int pos = wb - 1 - (4 * k + j);
      if (pos >= 0) p[pos] = (uint8_t)(x[k] >> (8 * j));
    }
  }
}

// Loads one point (wire format x || y), converts to Montgomery form, validates y^2 = x^3 + x
// (ecc/curve.c:57-76, :611-623: off-curve input becomes O).  Returns false for O.
template <class O>
__device__ __noinline__ bool a1_load_point(int sx, int sy, int st0, int st1, const uint8_t* p) {
  const int wb = (int)c_a1.wb;
  uint32_t x[kNA1];
  O::set_const(st0, c_fp.r2);
  a1_limbs_from_be(x, p, wb);
  O::st(sx, x);
  O::mul(sx, st0, sx);        // R^2 is the full operand, the wire value the scanned one: any
  a1_limbs_from_be(x, p + wb, wb);   // value below 2^(8 wb) comes out fully reduced (mpz_mod of
  O::st(sy, x);                      // fp_set_mpz, arith/montfp.c:100-110)
  O::mul(sy, st0, sy);
  O::sqr(st0, sx);
  O::set_const(st1, c_fp.one);
  O::add(st0, st0, st1);      // x^2 + 1
  O::mul(st0, st0, sx);       // x^3 + x
  O::sqr(st1, sy);
  return O::eq(st0, st1) && !O::is_zero(sy);    // (0, 0), the 2-torsion point, decodes as O (see pairing_a.cuh)
}

// D = N(f) f0 f1 (the one quantity the final exponentiation needs inverted); 0 marks "output 1"
template <class O>
__device__ __forceinline__ void a1_publish(int sF0, int sF1, int t0, int t1, bool valid, void* f,
                                           void* dprod, size_t n, size_t idx) {
  O::sqr(t0, sF0);
  O::sqr(t1, sF1);
  O::add(t0, t0, t1);
  O::mul(t1, sF0, sF1);
  O::mul(t0, t0, t1);
  if (!valid) {
    uint32_t zero[kNA1] = {0};
    O::st(t0, zero);
  }
  O::st_global(f, 0, n, idx, sF0);
  O::st_global(f, 1, n, idx, sF1);
  O::st_global(dprod, 0, n, idx, t0);
}

// f: [2][17][n] uint2 (Montgomery F_p^2), dprod: [17][n] uint2, pm: [2][17][n] uint2 scratch that
// keeps the Montgomery-form P for the chord steps.  strideP = 0: one P for the whole batch.
template <int BLOCK>
__global__ void __launch_bounds__(BLOCK)
k_a1_miller(const uint8_t* __restrict__ P, const uint8_t* __restrict__ Q, void* __restrict__ f,
            void* __restrict__ dprod, void* __restrict__ pm, size_t n, size_t strideP) {
  using O = Ops<kNA1, false, BLOCK>;
  size_t idx = (size_t)blockIdx.x * BLOCK + threadIdx.x;
  if (idx >= n) return;
  const size_t wire = 2 * (size_t)c_a1.wb;
  bool okP = a1_load_point<O>(aX, aY, aT0, aT1, P + idx * strideP);
  bool okQ = a1_load_point<O>(aQX, aQY, aT0, aT1, Q + idx * wire);
  O::st_global(pm, 0, n, idx, aX);
  O::st_global(pm, 1, n, idx, aY);
  O::set_const(aZ, c_fp.one);
  O::set_const(aZ2, c_fp.one);
  O::set_const(aF0, c_fp.one);
  uint32_t zero[kNA1] = {0};
  O::st(aF1, zero);
  // ecc/a_param.c:1979-1993: tangent; V = 2V; chord and V += P where the digit is non-zero; f = f^2.
  // a_double_step_5t squares first, which is the same product because f starts at 1.
  const int top = (int)c_a1naf.len - 2;
  for (int m = top; m >= 0; m--) {
    const bool chord = m > 0 && ((c_a1naf.nz[m >> 5] >> (m & 31)) & 1u);
    const bool minus = (c_a1naf.neg[m >> 5] >> (m & 31)) & 1u;      // V <- V - P: the chord through V and -P
    a_double_step_5t<O>();
    if (chord)
      a1_chord_add_5t<O>([&](int slot, int coord) {
        O::ld_global(slot, pm, coord, n, idx);
        if (coord == 1 && minus) O::neg(slot, slot);
      });
  }
  a1_publish<O>(aF0, aF1, aT0, aT1, okP && okQ, f, dprod, n, idx);
}

// element_prod_pairing (include/pbc_pairing.h:153-171 -> a1_pairings_affine): multiply the k
// Miller values of one output; ANY O / off-curve input makes the whole product 1.
template <int BLOCK>
__global__ void __launch_bounds__(BLOCK)
k_a1_prod(const void* __restrict__ f_in, const void* __restrict__ d_in, void* __restrict__ f_out,
          void* __restrict__ d_out, size_t k, size_t n_out, size_t n_in) {
  using O = Ops<kNA1, false, BLOCK>;
  enum { pF0, pF1, pL0, pL1, pT0, pT1, pT2, kSlots };
  size_t idx = (size_t)blockIdx.x * BLOCK + threadIdx.x;
  if (idx >= n_out) return;
  bool valid = true;
  uint32_t zero[kNA1] = {0};
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
  a1_publish<O>(pF0, pF1, pT0, pT1, valid, f_out, d_out, n_out, idx);
}
constexpr int kA1ProdSlots = 7;

// pairing_pp_init: one thread walks V over the bits of n once and tabulates, per step, the
// tangent (a, b, c) and -- where the bit is set -- the chord (a, b, c), each up to a factor in F_p^*:
//   tab[row * 34 ..], rows in loop order;  tab[rows * 34] = 1 if P is a finite point on the curve.
// Line values:  tangent  (c + a Qx) + i (b Qy),   chord  (c - a Qx) + i (b Qy).
struct A1Table {
  uint32_t* t;
  template <class O> __device__ __forceinline__ void store(size_t row, int slot) {
    uint32_t x[kNA1];
    O::ld(x, slot);
#pragma unroll
    for (int k = 0; k < kNA1; k++) t[row * kNA1 + k] = x[k];
  }
  template <class O> __device__ __forceinline__ void load(int slot, size_t row) const {
    O::set_const(slot, t + row * kNA1);
  }
};

template <int BLOCK>
__global__ void __launch_bounds__(BLOCK)
k_a1_pp_init(const uint8_t* __restrict__ P, uint32_t* __restrict__ tab, size_t rows) {
  using O = Ops<kNA1, false, BLOCK>;
  if (blockIdx.x != 0 || threadIdx.x != 0) return;
  // slots: aX aY aZ aZ2 = V; aQX aQY = P (affine); aT0..aT5 scratch
  bool okP = a1_load_point<O>(aX, aY, aT0, aT1, P);
  O::copy(aQX, aX);
  O::copy(aQY, aY);
  O::set_const(aZ, c_fp.one);
  O::set_const(aZ2, c_fp.one);
  A1Table T{tab};
  size_t row = 0;
  for (int m = (int)c_a1.nbits - 2; m >= 0; m--) {
    a1_pp_tangent<O>(T, row);
    if (m > 0 && ((c_a1.n[m >> 5] >> (m & 31)) & 1u)) a1_pp_chord<O>(T, row);
  }
  tab[rows * kNA1] = okP ? 1u : 0u;
}

// pairing_pp_apply: f <- f^2 l_tangent(Q) [l_chord(Q)] per bit of n, 7 (12) multiplications
template <int BLOCK>
__global__ void __launch_bounds__(BLOCK)
k_a1_pp_apply(const uint32_t* __restrict__ tab, const uint8_t* __restrict__ Q, void* __restrict__ f,
              void* __restrict__ dprod, size_t n, size_t rows) {
  using O = Ops<kNA1, false, BLOCK>;
  enum { qF0, qF1, qQX, qQY, qT0, qT1, qT2, qT3, qT4, kSlots };
  size_t idx = (size_t)blockIdx.x * BLOCK + threadIdx.x;
  if (idx >= n) return;
  bool okQ = a1_load_point<O>(qQX, qQY, qT0, qT1, Q + idx * 2 * (size_t)c_a1.wb);
  bool valid = okQ && tab[rows * kNA1] != 0;
  uint32_t zero[kNA1] = {0};
  O::set_const(qF0, c_fp.one);
  O::st(qF1, zero);
  const A1Table T{const_cast<uint32_t*>(tab)};
  size_t row = 0;
  for (int m = (int)c_a1.nbits - 2; m >= 0; m--) {
    a_fsqr<O>(qF0, qF1, qT0, qT1);
    a1_pp_eval<O>(T, row, false, qF0, qF1, qQX, qQY, qT0, qT1, qT2, qT3, qT4);
    row += 3;
    if (m > 0 && ((c_a1.n[m >> 5] >> (m & 31)) & 1u)) {
      a1_pp_eval<O>(T, row, true, qF0, qF1, qQX, qQY, qT0, qT1, qT2, qT3, qT4);
      row += 3;
    }
  }
  a1_publish<O>(qF0, qF1, qT0, qT1, valid, f, dprod, n, idx);
}
constexpr int kA1PPSlots = 9;

// out: n * 2 wb bytes, wire format of F_p^2 (arith/fieldquadratic.c:323-329: x || y)
template <int BLOCK>
__global__ void __launch_bounds__(BLOCK)
k_a1_finalexp(const void* __restrict__ f, const void* __restrict__ dinv, uint8_t* __restrict__ out,
              size_t n) {
  using O = Ops<kNA1, false, BLOCK>;
  enum { fF0, fF1, fD, fN, fP, fV0, fV1, fT0, fTWO, kSlots };
  size_t idx = (size_t)blockIdx.x * BLOCK + threadIdx.x;
  if (idx >= n) return;
  O::ld_global(fF0, f, 0, n, idx);
  O::ld_global(fF1, f, 1, n, idx);
  O::ld_global(fD, dinv, 0, n, idx);
  bool identity = O::is_zero(fD);
  O::set_const(fTWO, c_a1.two);
  a_lucas_final<O>(fF0, fF1, fD, fN, fP, fV0, fV1, fT0, fTWO, c_a1.l, (int)c_a1.lbits);

  const int wb = (int)c_a1.wb;
  uint32_t x[kNA1], one[kNA1] = {1};
  uint8_t* o = out + idx * 2 * (size_t)wb;
  O::st(fT0, one);
  O::mul(fV0, fV0, fT0);                    // leave Montgomery form (arith/montfp.c:64-80)
  O::mul(fV1, fV1, fT0);
  O::ld(x, fV0);
  if (identity) {
#pragma unroll
    for (int k = 0; k < kNA1; k++) x[k] = one[k];
  }
  a1_limbs_to_be(o, x, wb);
  O::ld(x, fV1);
  if (identity) {
#pragma unroll
    for (int k = 0; k < kNA1; k++) x[k] = 0;
  }
  a1_limbs_to_be(o + wb, x, wb);
}
constexpr int kA1FinalSlots = 9;

// F_p differential-test hook for the 34-limb field (analogue of guru/fp_test.c): operands and
// result in the wire format of one coordinate (wb bytes, big-endian, canonical).
template <int BLOCK>
__global__ void __launch_bounds__(BLOCK)
k_a1_fp_op(int op, uint8_t* __restrict__ out, const uint8_t* __restrict__ a,
           const uint8_t* __restrict__ b, size_t n) {
  using O = Ops<kNA1, false, BLOCK>;
  size_t idx = (size_t)blockIdx.x * BLOCK + threadIdx.x;
  if (idx >= n) return;
  const int wb = (int)c_a1.wb;
  uint32_t x[kNA1], one[kNA1] = {1};
  O::set_const(2, c_fp.r2);
  a1_limbs_from_be(x, a + idx * wb, wb);
  O::st(0, x);
  O::mul(0, 2, 0);
  a1_limbs_from_be(x, b + idx * wb, wb);
  O::st(1, x);
  O::mul(1, 2, 1);
  switch (op) {
    case 0: O::mul(0, 0, 1); break;
    case 1: O::add(0, 0, 1); break;
    case 2: O::sub(0, 0, 1); break;
    case 3: O::set_const(2, c_fp.one); slot_fermat_inverse<O, kNA1>(3, 0, 2); O::copy(0, 3); break;
    case 4: O::halve(0, 0); break;
    case 5: O::neg(0, 0); break;
    case 6: O::sqr(0, 0); break;
    case 7: O::mul(0, 0, 1); O::sub(0, 0, 1); break;
  }
  O::st(1, one);
  O::mul(0, 0, 1);
  O::ld(x, 0);
  a1_limbs_to_be(out + idx * wb, x, wb);
}

}  // namespace pbcb200
