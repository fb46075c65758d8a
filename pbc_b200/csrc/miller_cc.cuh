// miller_cc.cuh -- the Miller loop shared by the Type F and Type D pairings.
//
// Device replacement for cc_miller_no_denom (ecc/f_param.c:97-248) and
// cc_miller_no_denom_affine (ecc/d_param.c:321-422): same loop shape over the bits of r (tangent,
// double, optional chord + add, square), but the multiples of P are kept in Jacobian coordinates so
// no step needs a field inversion (the reference inverts once per tangent and once per chord).
// Each line a X + b Y + c is therefore scaled by some element of F_q^*; the final exponent is a
// multiple of q - 1, so the reduced pairing is unchanged (tools/proto_fd.py checks exactly this
// against the oracle).
//
//   tangent at V = (X, Y, Z):  M = 3 X^2 + A Z^4
//        a = -M Z^2,  b = 2 Y Z^3,  c = M X - 2 Y^2                       (affine line times Z^6)
//   chord through V and P = (xP, yP):
//        a = Y - yP Z^3,  b = (xP Z^2 - X) Z,  c = yP Z X - xP Y          (affine line times Z^3)
//   V <- 2V: dbl-2007-bl style with general A;  V <- V + P: mixed Jacobian + affine addition.
#pragma once
#include "fq_small.cuh"

namespace pbcb200 {

// resident blocks per SM the F/D kernels are compiled for (caps registers at 65536 / (BLOCK * this))
constexpr int kCCMinBlocks = 4;
// threads per block of the F/D/G Miller kernels.  A block-wide barrier at the top of every Miller iteration
// keeps the warps of a block in the same code region (the loop over the digits of r is uniform across
// pairings), so they share instruction-cache lines; every thread of the block has to run the loop.
constexpr int kCCMillerBlock = 256;

template <int NS>
struct CCConstsT {
  uint32_t A[NS], B[NS];       // curve y^2 = x^3 + A x + B over F_q (Montgomery form)
  uint32_t r[NS];              // group order (plain integer, little-endian words)
  uint32_t rbits;
  uint32_t a_is_zero;
};
typedef CCConstsT<kNS> CCConsts;
__constant__ CCConsts c_cc;

// The loop scans signed digits (miller_naf_digits, host_naf.hpp: the non-adjacent form of r - 1, or of
// r where the cofactor is 1) instead of the bits of r: one chord + addition per three positions instead
// of one per two; where the digit is -1 the chord goes through V and -P.  Vertical lines and constants
// lie in the subfield the final exponentiation kills, so the reduced pairing is the same element for
// every P on the curve (the reference keeps the plain scan).  Faster for F, D and G (fewer chord steps).
struct CCNaf {
  uint32_t nz[8], neg[8];      // bit i: digit i non-zero / digit i is -1   (r below 2^255)
  uint32_t len;                // number of digits; the top one is +1
  uint32_t pad[3];
};
__constant__ CCNaf c_ccnaf;

// y^2 == x^3 + A x + B  (ecc/curve.c:57-76)
__device__ __forceinline__ bool cc_on_curve(const Fq& x, const Fq& y) {
  Fq t, u, A, B;
  fq_set(A, c_cc.A);
  fq_set(B, c_cc.B);
  fq_sqr(t, x);
  fq_add(t, t, A);
  fq_mul(t, t, x);
  fq_add(t, t, B);
  fq_sqr(u, y);
  return fq_eq(t, u) && !fq_is_zero(y);    // a 2-torsion point (y = 0) has no tangent line: decoded as O
}

// T supplies:  struct Acc;  struct Ctx;
//   static void mul_line(Acc* v, const Fq* a, const Fq* b, const Fq* c, const Ctx* ctx);   v *= line
//   static void sqr(Acc* v);                                                               v  = v^2

// The walk over the digits of r, generic in what happens to each line: `sink.line(a, b, c)` receives
// the coefficients of every tangent and chord in loop order, `sink.sqr()` marks the squaring between
// iterations.  Two sinks: the Miller accumulator (below) and the fixed-argument table (pairing_pp_init).
template <class Sink>
__device__ __forceinline__ void miller_cc_walk(Sink& sink, const Fq& xP, const Fq& yP) {
  Fq X = xP, Y = yP, Z, a, b, c, M, Y2, Z2, t, u;
  fq_one(Z);
  int m = (int)c_ccnaf.len - 2;
  Fq yN;
  fq_neg(yN, yP);
  for (;;) {
    if (Sink::kBarriers) __syncthreads();
    // ---- tangent at V ----
    fq_sqr(Z2, Z);
    fq_sqr(t, X);
    fq_add(M, t, t);
    fq_add(M, M, t);                       // 3 X^2
    if (!c_cc.a_is_zero) {
      fq_sqr(u, Z2);
      fq_set(t, c_cc.A);
      fq_mul(u, u, t);
      fq_add(M, M, u);                     // + A Z^4
    }
    fq_sqr(Y2, Y);
    fq_mul(a, M, Z2);
    fq_neg(a, a);                          // a = -M Z^2
    fq_mul(u, Y, Z);
    fq_add(u, u, u);                          // Z' = 2 Y Z
    fq_mul(b, u, Z2);                      // b = Z' Z^2
    fq_mul(c, M, X);
    fq_sub(c, c, Y2);
    fq_sub(c, c, Y2);                      // c = M X - 2 Y^2
    sink.line(a, b, c);
    if (m == 0) break;
    // ---- V = 2 V ----
    fq_mul(t, X, Y2);
    fq_add(t, t, t);
    fq_add(t, t, t);                          // S = 4 X Y^2
    Z = u;
    fq_sqr(X, M);
    fq_sub(X, X, t);
    fq_sub(X, X, t);                       // X' = M^2 - 2 S
    fq_sqr(Y2, Y2);
    fq_add(Y2, Y2, Y2);
    fq_add(Y2, Y2, Y2);
    fq_add(Y2, Y2, Y2);                        // 8 Y^4
    fq_sub(t, t, X);
    fq_mul(Y, M, t);
    fq_sub(Y, Y, Y2);                      // Y' = M (S - X') - 8 Y^4
    if ((c_ccnaf.nz[m >> 5] >> (m & 31)) & 1u) {
      // ---- chord through V and +-P, then V = V +- P ----
      const Fq& yS = ((c_ccnaf.neg[m >> 5] >> (m & 31)) & 1u) ? yN : yP;
      Fq H, R;
      fq_sqr(Z2, Z);
      fq_mul(t, Z2, Z);                    // Z^3
      fq_mul(H, xP, Z2);
      fq_sub(H, H, X);                     // H = xP Z^2 - X
      fq_mul(R, yS, t);
      fq_sub(a, Y, R);                     // a = Y - yS Z^3
      fq_sub(R, R, Y);                     // R = yP Z^3 - Y
      fq_mul(b, H, Z);                     // b = H Z = Z of the sum
      fq_mul(t, yS, Z);
      fq_mul(t, t, X);
      fq_mul(u, xP, Y);
      fq_sub(c, t, u);                     // c = yP Z X - xP Y
      sink.line(a, b, c);
      fq_sqr(t, H);                        // H^2
      fq_mul(u, t, H);                     // H^3
      fq_mul(t, t, X);                     // X H^2
      fq_sqr(X, R);
      fq_sub(X, X, u);
      fq_sub(X, X, t);
      fq_sub(X, X, t);                     // X3 = R^2 - H^3 - 2 X H^2
      fq_sub(t, t, X);
      fq_mul(t, t, R);
      fq_mul(u, u, Y);
      fq_sub(Y, t, u);                     // Y3 = R (X H^2 - X3) - Y H^3
      Z = b;
    }
    m--;
    sink.sqr();
  }
}

template <class T>
struct MillerSink {
  static constexpr bool kBarriers = true;
  typename T::Acc* v;
  const typename T::Ctx* ctx;
  __device__ __forceinline__ void line(Fq& a, Fq& b, Fq& c) { T::mul_line(v, &a, &b, &c, ctx); }
  __device__ __forceinline__ void sqr() { T::sqr(v); }
};
template <class T>
__device__ __forceinline__ void miller_cc(typename T::Acc* v, const Fq& xP, const Fq& yP,
                                          const typename T::Ctx* ctx) {
  MillerSink<T> sink{v, ctx};
  miller_cc_walk(sink, xP, yP);
}

// ---------------------------------------------------------------------------------------------
// Fixed first argument (pairing_pp_init / pairing_pp_apply; d_pairing_pp_init ecc/d_param.c:794-966
// stores the coefficients of every tangent and chord of the walk over P; the reference's generic
// fall-back, ecc/pairing.c:48-72, stores only P).  Here for every type on this loop (f, d, g):
//   tab[(3 row + {0, 1, 2}) * kNS ..] = a, b, c of line `row` in loop order (Montgomery form, each
//   line scaled by some element of F_q^*, as in the plain loop);  tab[3 rows kNS] = 1 if P decoded
//   to a finite point of the curve.
// The apply loop does no point arithmetic at all.
// ---------------------------------------------------------------------------------------------
struct TableSink {
  static constexpr bool kBarriers = false;
  uint32_t* tab;
  size_t row;
  __device__ __forceinline__ void line(Fq& a, Fq& b, Fq& c) {
#pragma unroll
    for (int k = 0; k < kNS; k++) {
      tab[(3 * row + 0) * kNS + k] = a.v[k];
      tab[(3 * row + 1) * kNS + k] = b.v[k];
      tab[(3 * row + 2) * kNS + k] = c.v[k];
    }
    row++;
  }
  __device__ __forceinline__ void sqr() {}
};

template <int WB>
__global__ void k_cc_pp_init(const uint8_t* __restrict__ P, uint32_t* __restrict__ tab, size_t rows) {
  if (blockIdx.x != 0 || threadIdx.x != 0) return;
  Fq xP, yP;
  fq_from_wire_w<WB>(xP, P);
  fq_from_wire_w<WB>(yP, P + wire_w<WB>());
  bool ok = cc_on_curve(xP, yP);
  TableSink sink{tab, 0};
  miller_cc_walk(sink, xP, yP);
  tab[3 * rows * kNS] = (ok && sink.row == rows) ? 1u : 0u;
}

// v <- Miller value from the table (the same sequence of line products and squarings as miller_cc)
template <class T>
__device__ __forceinline__ void miller_cc_tab(typename T::Acc* v, const uint32_t* __restrict__ tab,
                                              const typename T::Ctx* ctx) {
  Fq a, b, c;
  size_t row = 0;
  int m = (int)c_ccnaf.len - 2;
  for (;;) {
    __syncthreads();
    fq_set(a, tab + (3 * row + 0) * kNS); fq_set(b, tab + (3 * row + 1) * kNS); fq_set(c, tab + (3 * row + 2) * kNS);
    row++;
    T::mul_line(v, &a, &b, &c, ctx);
    if (m == 0) break;
    if ((c_ccnaf.nz[m >> 5] >> (m & 31)) & 1u) {
      fq_set(a, tab + (3 * row + 0) * kNS); fq_set(b, tab + (3 * row + 1) * kNS); fq_set(c, tab + (3 * row + 2) * kNS);
      row++;
      T::mul_line(v, &a, &b, &c, ctx);
    }
    m--;
    T::sqr(v);
  }
}

}  // namespace pbcb200
