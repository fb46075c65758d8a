// pairing_e.cuh -- Type E pairing kernels: y^2 = x^3 + a x + b over F_q, k = 1 (G1 = G2 = E(F_q),
// GT = the order-r subgroup of F_q^*), r = 2^exp2 + sign1 2^exp1 + sign0, q = h r^2 + 1 below 2^1087
// (at most 1087 bits, the bound of the 34-limb field; param/e.param: 1020).
//
// Device replacement for ecc/e_param.c:64-300 (e_miller_proj) and :472-482 (e_pairing):
//   e(P, Q) = (f_P(Q + R) / f_P(R))^((q - 1)/r)
// with R a fixed point outside E[r].  The reference draws R at random per pairing_init; for P in G1
// the value does not depend on R (changing R multiplies f_P(Q+R)/f_P(R) by an r-th power), so R is
// chosen once on the host (engine.cu, init_type_e) and read back with pbc_b200_derived_constant("R").
//
// Same loop as the reference (exp1 tangent/double/vertical steps, a save, exp2 - exp1 more, one
// chord), numerator v and denominator vd carried apart.  What differs, and why the bytes do not:
//   * k = 1: the final exponent has no factor q - 1, so a stray constant c in F_q^* would survive as
//     c^((q-1)/r).  Only two kinds of change are allowed: scaling a line's coefficients when the same
//     coefficients are evaluated at both Q + R and R (the scale cancels in v / vd), and factors that
//     are r-th powers.
//   * V stays in Jacobian coordinates (the reference makes it affine twice, with an inversion each):
//     lines are scaled by powers of Z, the same scale at both points.
//   * Q + R stays Jacobian (X, Y, Z) and the lines are evaluated homogenised, l(X, Y, Z) = Z^3 l(x, y),
//     verticals Z^2 (x - c).  Over the whole loop that multiplies f_P(Q+R) by Z^r (the pole order of
//     f_P at O is r) -- an r-th power, because P has order r.  For P outside G1 the value is
//     unspecified, as it is in the reference (whose bytes then depend on its random R).
//   * Every line of the loop vanishes only at multiples of P.  R is outside E[r], so for Q in G1 no line
//     vanishes at Q + R or at R.  Q = R (the mixed addition below has H = 0) and Q with Q + R in <P>
//     are the on-curve second arguments whose value is unspecified (include/pbc_b200.h).
//   * The save point and the end use V + Z1 = -sign0 P for P of order r: the last vertical is at
//     x(P); with sign0 = +1 it cancels the reference's extra vertical at x(P), so both are skipped.
//   * the values at R are evaluated at the affine R; with a fixed first argument (k_e_pp_init) all of
//     them are folded into one numerator / denominator pair per P.
// Pipeline per batch:  k_e_miller (-> k_e_prod) | k_e_pp_apply  ->  k_batch_invert<34>  ->  k_e_finalexp.
// The 34-limb slot machine, wire conversion, scalar decoding and table rows are type A1's.
#pragma once
#include "pairing_a1.cuh"
#include "prod_v.cuh"

namespace pbcb200 {

struct alignas(16) EConsts {
  uint8_t dig[32 * kMaxLimbs];  // final exponent (q - 1)/r as a left-to-right window: digit at the
                                // lowest bit of each window, odd, 1..15; 0 elsewhere
  uint32_t dstart;              // position of the top window's digit
  uint32_t exp1, exp2;
  int32_t sign1, sign0;
  uint32_t a_zero;              // curve coefficient a = 0: the doubling skips a Z^4
  uint32_t pad[2];
};
__constant__ EConsts c_e;
// curve coefficients and R, Montgomery form, element e at g_e_pts + 17 e (read with stride 1 as the
// global operand of Ops::mulx, or into a slot with ld_global(.., 1, 0))
enum { kEA = 0, kEB = 1, kERX = 2, kERY = 3 };
__device__ uint2 g_e_pts[4 * (kNA1 / 2)];

// an element of a limb-major global array (vectors `stride` apart): per-thread arrays [e][17][n] use
// stride n, table rows and g_e_pts stride 1
__device__ __forceinline__ const uint2* e_el(const void* base, int e, size_t n, size_t idx) {
  return reinterpret_cast<const uint2*>(base) + (size_t)e * (kNA1 / 2) * n + idx;
}
__device__ __forceinline__ const uint2* e_row(const uint32_t* tab, size_t row) {
  return reinterpret_cast<const uint2*>(tab + row * kNA1);
}
__device__ __forceinline__ const uint2* e_pt(int e) { return g_e_pts + e * (kNA1 / 2); }

enum ESlot { eX, eY, eZ, eZ2, eV, eVD, eT0, eT1, eT2, eT3, eT4, eT5, eT6, kESlots };

// Loads one point (x || y), converts to Montgomery form, validates y^2 = x^3 + a x + b (off-curve
// input becomes O, ecc/curve.c:611-623).  Returns false when not on the curve.
template <class O>
__device__ __noinline__ bool e_load_point(int sx, int sy, int st0, int st1, const uint8_t* p) {
  const int wb = (int)c_a1.wb;
  uint32_t x[kNA1];
  O::set_const(st0, c_fp.r2);
  a1_limbs_from_be(x, p, wb);
  O::st(sx, x);
  O::mul(sx, st0, sx);
  a1_limbs_from_be(x, p + wb, wb);
  O::st(sy, x);
  O::mul(sy, st0, sy);
  O::sqr(st0, sx);
  O::ld_global(st1, g_e_pts, kEA, 1, 0);
  O::add(st0, st0, st1);
  O::mul(st0, st0, sx);        // x^3 + a x
  O::ld_global(st1, g_e_pts, kEB, 1, 0);
  O::add(st0, st0, st1);
  O::sqr(st1, sy);
  return O::eq(st0, st1);
}

// Q + R, Q affine in (sx, sy), R affine: Jacobian (X, Y, Z) -> homogenised operands
//   sx = X, sy = Y, t3 = X Z, t1 = Z^2, t2 = Z^3.   t0 is scratch.
template <class O>
__device__ __noinline__ void e_q_plus_r(int sx, int sy, int t0, int t1, int t2, int t3) {
  O::ld_global(t0, g_e_pts, kERX, 1, 0);
  O::sub(t0, t0, sx);          // H = xR - xQ
  O::ld_global(t1, g_e_pts, kERY, 1, 0);
  O::sub(t1, t1, sy);          // rr = yR - yQ
  O::sqr(t2, t0);              // H^2
  O::mul(t3, t2, t0);          // H^3
  O::mul(t2, sx, t2);          // U = xQ H^2
  O::sqr(sx, t1);
  O::sub(sx, sx, t3);
  O::sub(sx, sx, t2);
  O::sub(sx, sx, t2);          // X = rr^2 - H^3 - 2U
  O::sub(t2, t2, sx);
  O::mul(t2, t1, t2);
  O::mul(t3, sy, t3);
  O::sub(sy, t2, t3);          // Y = rr (U - X) - yQ H^3
  O::sqr(t1, t0);              // Z^2 (Z = H)
  O::mul(t2, t1, t0);          // Z^3
  O::mul(t3, sx, t0);          // X Z
}

// d = s1 g1 + s2 g2 + s3 g3: a line a x + b y + c at the homogenised Q + R, one side in slots, the
// other in global memory (stride apart)
template <class O>
__device__ __forceinline__ void e_line_hom(int d, int t, int s1, const uint2* g1, int s2, const uint2* g2, int s3,
                                           const uint2* g3, size_t stride) {
  O::mulg(d, s1, g1, stride);
  O::mulg(t, s2, g2, stride);
  O::add(d, d, t);
  O::mulg(t, s3, g3, stride);
  O::add(d, d, t);
}
// d = s1 g1 - s2 g2: a vertical at the homogenised Q + R
template <class O>
__device__ __forceinline__ void e_vert_hom(int d, int t, int s1, const uint2* g1, int s2, const uint2* g2,
                                           size_t stride) {
  O::mulg(d, s1, g1, stride);
  O::mulg(t, s2, g2, stride);
  O::sub(d, d, t);
}
// d = a xR + b yR + c (slots a, b, c)
template <class O>
__device__ __forceinline__ void e_line_r(int d, int t, int sa, int sb, int sc) {
  O::mulg(d, sa, e_pt(kERX), 1);
  O::mulg(t, sb, e_pt(kERY), 1);
  O::add(d, d, t);
  O::add(d, d, sc);
}
// d = xR Z^2 - X: the vertical at V = (X, Y, Z) evaluated at R, scaled by Z^2
template <class O>
__device__ __forceinline__ void e_vert_r(int d) {
  O::mulg(d, eZ2, e_pt(kERX), 1);
  O::sub(d, d, eX);
}

// One step of e_miller_proj (ecc/e_param.c:222-228) after the squarings: the tangent at V, V = 2V,
// the vertical at the new V.  Tangent (scaled by Z^2 Z'): a = -M Z^2, b = 2 Y Z^3, c = X M - 2 Y^2 with
// M = 3 X^2 + a Z^4; the same line as the reference's do_tangent.  S receives the coefficients
// (slots eT3, eT4, eT2) and then the new V; it may use eT5 and eT6.
template <class O, class S>
__device__ __forceinline__ void e_dbl_step(S& s) {
  O::sqr(eT0, eX);
  O::dbl(eT2, eT0);
  O::add(eT0, eT0, eT2);
  if (!c_e.a_zero) {
    O::sqr(eT1, eZ2);
    O::mulg(eT1, eT1, e_pt(kEA), 1);
    O::add(eT0, eT0, eT1);         // M = 3 X^2 + a Z^4
  }
  O::sqr(eT1, eY);                 // Y^2
  O::mul(eT2, eX, eT0);
  O::sub(eT2, eT2, eT1);
  O::sub(eT2, eT2, eT1);           // c = X M - 2 Y^2
  O::mul(eT3, eT0, eZ2);
  O::neg(eT3, eT3);                // a = -M Z^2
  O::mul(eZ, eY, eZ);
  O::dbl(eZ, eZ);                  // Z' = 2 Y Z
  O::mul(eT4, eZ, eZ2);            // b = Z' Z^2 = 2 Y Z^3
  s.tangent(eT3, eT4, eT2);
  O::sqr(eZ2, eZ);
  O::mul(eT2, eX, eT1);
  O::dbl(eT2, eT2, 2);             // S = 4 X Y^2
  O::sqr(eX, eT0);
  O::sub(eX, eX, eT2);
  O::sub(eX, eX, eT2);             // X' = M^2 - 2 S
  O::sqr(eT1, eT1);
  O::dbl(eT1, eT1, 3);             // 8 Y^4
  O::sub(eT2, eT2, eX);
  O::mulsub(eY, eT0, eT2, eT1);    // Y' = M (S - X') - 8 Y^4
  s.vertical();
}

// the chord through V (slots) and Z1 = (X1, Y1, Z1) (global, stride apart), scaled by Zv^3 Z1^3:
//   a = Yv Z1^3 - Y1 Zv^3,  b = (X1 Zv^2 - Xv Z1^2) Z1 Zv,  c = Xv Y1 Zv - Yv X1 Z1
// -> slots eT2 (a), eT4 (b), eT5 (c); the reference's do_line through the affine Z and Z1 up to that scale.
template <class O>
__device__ __forceinline__ void e_chord(const uint2* x1, const uint2* y1, const uint2* z1, size_t stride) {
  O::ld_global(eT6, z1, 0, stride, 0);
  O::sqr(eT0, eT6);                // Z1^2
  O::mul(eT1, eT0, eT6);           // Z1^3
  O::mul(eT2, eY, eT1);
  O::mul(eT3, eZ2, eZ);            // Zv^3
  O::mulg(eT4, eT3, y1, stride);
  O::sub(eT2, eT2, eT4);           // a
  O::mulg(eT4, eZ2, x1, stride);
  O::mul(eT5, eX, eT0);
  O::sub(eT4, eT4, eT5);
  O::mul(eT4, eT4, eT6);
  O::mul(eT4, eT4, eZ);            // b
  O::mul(eT5, eX, eZ);
  O::mulg(eT5, eT5, y1, stride);
  O::mul(eT3, eY, eT6);
  O::mulg(eT3, eT3, x1, stride);
  O::sub(eT5, eT5, eT3);           // c
}

// f = v, d = vd (0 marks "output 1")
template <class O>
__device__ __forceinline__ void e_publish(int sV, int sD, bool valid, void* f, void* dprod, size_t n, size_t idx) {
  if (!valid) {
    uint32_t zero[kNA1] = {0};
    O::st(sD, zero);
  }
  O::st_global(f, 0, n, idx, sV);
  O::st_global(dprod, 0, n, idx, sD);
}

// per-thread workspace of k_e_miller, [e][17][n] each:
//   px [1]: x(P);  qd [5]: homogenised Q + R (X, Y, X Z, Z^2, Z^3);  sv [5]: X1, Y1, Z1, v1, vd1 at the save
enum { kQX, kQY, kQXZ, kQZ2, kQZ3, kQWords };
enum { kSX, kSY, kSZ, kSV, kSVD, kSWords };

template <class O>
struct EMillerSink {
  const void* qd;
  size_t n, idx;
  __device__ __forceinline__ void tangent(int sa, int sb, int sc) {
    e_line_r<O>(eT5, eT6, sa, sb, sc);
    O::mul(eVD, eVD, eT5);
    e_line_hom<O>(eT5, eT6, sa, e_el(qd, kQXZ, n, idx), sb, e_el(qd, kQY, n, idx), sc, e_el(qd, kQZ3, n, idx), n);
    O::mul(eV, eV, eT5);
  }
  __device__ __forceinline__ void vertical() {
    e_vert_hom<O>(eT5, eT6, eZ2, e_el(qd, kQX, n, idx), eX, e_el(qd, kQZ2, n, idx), n);
    O::mul(eVD, eVD, eT5);
    e_vert_r<O>(eT5);
    O::mul(eV, eV, eT5);
  }
};

// f, dprod: [17][n] uint2; px [17][n], qd [5][17][n], sv [5][17][n] scratch.  strideP = 0: one P for
// the whole batch.
template <int BLOCK>
__global__ void __launch_bounds__(BLOCK)
k_e_miller(const uint8_t* __restrict__ P, const uint8_t* __restrict__ Q, void* __restrict__ f,
           void* __restrict__ dprod, void* __restrict__ px, void* __restrict__ qd, void* __restrict__ sv,
           size_t n, size_t strideP) {
  using O = Ops<kNA1, false, BLOCK>;
  size_t idx = (size_t)blockIdx.x * BLOCK + threadIdx.x;
  if (idx >= n) return;
  const size_t wire = 2 * (size_t)c_a1.wb;
  bool okQ = e_load_point<O>(eT0, eT1, eT2, eT3, Q + idx * wire);
  e_q_plus_r<O>(eT0, eT1, eT2, eT3, eT4, eT5);
  O::st_global(qd, kQX, n, idx, eT0);
  O::st_global(qd, kQY, n, idx, eT1);
  O::st_global(qd, kQXZ, n, idx, eT5);
  O::st_global(qd, kQZ2, n, idx, eT3);
  O::st_global(qd, kQZ3, n, idx, eT4);
  bool okP = e_load_point<O>(eX, eY, eT0, eT1, P + idx * strideP);
  O::st_global(px, 0, n, idx, eX);
  O::set_const(eZ, c_fp.one);
  O::set_const(eZ2, c_fp.one);
  O::set_const(eV, c_fp.one);
  O::set_const(eVD, c_fp.one);
  EMillerSink<O> s{qd, n, idx};
  const int exp1 = (int)c_e.exp1, exp2 = (int)c_e.exp2;
  for (int i = 0; i < exp2; i++) {
    if (i == exp1) {
      // ecc/e_param.c:229-240: (v1, vd1, Z1) = (v, vd, V), or for sign1 < 0 (vd, v, -V) with the
      // vertical at V (numerator side into vd1, denominator side into v1)
      if (c_e.sign1 < 0) {
        e_vert_hom<O>(eT5, eT6, eZ2, e_el(qd, kQX, n, idx), eX, e_el(qd, kQZ2, n, idx), n);
        O::mul(eT5, eV, eT5);
        O::st_global(sv, kSVD, n, idx, eT5);
        e_vert_r<O>(eT5);
        O::mul(eT5, eVD, eT5);
        O::st_global(sv, kSV, n, idx, eT5);
        O::neg(eT5, eY);
        O::st_global(sv, kSY, n, idx, eT5);
      } else {
        O::st_global(sv, kSV, n, idx, eV);
        O::st_global(sv, kSVD, n, idx, eVD);
        O::st_global(sv, kSY, n, idx, eY);
      }
      O::st_global(sv, kSX, n, idx, eX);
      O::st_global(sv, kSZ, n, idx, eZ);
    }
    O::sqr(eV, eV);
    O::sqr(eVD, eVD);
    e_dbl_step<O>(s);
  }
  // :246-252: v *= v1, vd *= vd1, the chord through V and Z1
  O::mulg(eV, eV, e_el(sv, kSV, n, idx), n);
  O::mulg(eVD, eVD, e_el(sv, kSVD, n, idx), n);
  e_chord<O>(e_el(sv, kSX, n, idx), e_el(sv, kSY, n, idx), e_el(sv, kSZ, n, idx), n);
  e_line_r<O>(eT0, eT1, eT2, eT4, eT5);
  O::mul(eVD, eVD, eT0);
  e_line_hom<O>(eT0, eT1, eT2, e_el(qd, kQXZ, n, idx), eT4, e_el(qd, kQY, n, idx), eT5, e_el(qd, kQZ3, n, idx), n);
  O::mul(eV, eV, eT0);
  if (c_e.sign0 < 0) {
    // :253: the vertical at V + Z1 = P (sign0 = +1: it cancels against :275-277, both skipped)
    O::ld_global(eT2, px, 0, n, idx);
    O::mulg(eT0, eT2, e_el(qd, kQZ2, n, idx), n);
    O::ld_global(eT1, qd, kQX, n, idx);
    O::sub(eT0, eT1, eT0);         // X - x(P) Z^2
    O::mul(eVD, eVD, eT0);
    O::ld_global(eT0, g_e_pts, kERX, 1, 0);
    O::sub(eT0, eT0, eT2);         // xR - x(P)
    O::mul(eV, eV, eT0);
  }
  e_publish<O>(eV, eVD, okP && okQ, f, dprod, n, idx);
}

// element_prod_pairing (include/pbc_pairing.h:153-171): the k numerators and the k denominators of
// one output multiplied; ANY O / off-curve input makes the whole product 1.
template <int BLOCK>
__global__ void __launch_bounds__(BLOCK)
k_e_prod(const void* __restrict__ f_in, const void* __restrict__ d_in, void* __restrict__ f_out,
         void* __restrict__ d_out, size_t k, size_t n_out, size_t n_in) {
  using O = Ops<kNA1, false, BLOCK>;
  enum { pF, pD, pT, kSlots };
  size_t idx = (size_t)blockIdx.x * BLOCK + threadIdx.x;
  if (idx >= n_out) return;
  bool valid = true;
  O::set_const(pF, c_fp.one);
  O::set_const(pD, c_fp.one);
  for (size_t j = 0; j < k; j++) {
    size_t src = idx * k + j;
    O::ld_global(pT, d_in, 0, n_in, src);
    valid = valid && !O::is_zero(pT);
    O::mul(pD, pD, pT);
    O::mulg(pF, pF, e_el(f_in, 0, n_in, src), n_in);
  }
  e_publish<O>(pF, pD, valid, f_out, d_out, n_out, idx);
}
constexpr int kEProdSlots = 3;

// the same product over a run table (prod_v.cuh, pbc_b200_prod_pairings_apply_v): numerator and
// denominator multiplied separately; every pass stores through e_publish (vd = 0 marks an invalid pair)
template <class O>
struct ProdVE {
  enum { pF, pD, pT, kSlots };
  static constexpr int kMinBlocks = 1;
  bool ok;
  __device__ __forceinline__ void first(const ProdVBuf& in, size_t j) {
    O::ld_global(pF, in.v, 0, in.n, j);
    O::ld_global(pD, in.d, 0, in.n, j);
    ok = !O::is_zero(pD);
  }
  __device__ __forceinline__ void next(const ProdVBuf& in, size_t j) {
    O::ld_global(pT, in.d, 0, in.n, j);
    ok = ok && !O::is_zero(pT);
    O::mul(pD, pD, pT);
    O::mulg(pF, pF, e_el(in.v, 0, in.n, j), in.n);
  }
  __device__ __forceinline__ void store(const ProdVBuf& out, size_t r, bool) {
    e_publish<O>(pF, pD, ok, out.v, out.d, out.n, r);
  }
};

// ---- fixed first argument ----
// Table rows (34 words each, Montgomery form), for step i < exp2: 5 i + {a, b, c} of the tangent,
// 5 i + {3, 4} = (Z^2, X) of the new V (its vertical); then from kERowBase = 5 exp2:
enum {
  kPPChordA, kPPChordB, kPPChordC,   // the chord
  kPPPx,                             // x(P)
  kPPVR, kPPVDR,                     // every value at R, folded: numerator, denominator
  kPPSaveZ2, kPPSaveX,               // the vertical at the save point (sign1 < 0)
  kPPX1, kPPY1, kPPZ1, kPPV1, kPPVD1,   // scratch of k_e_pp_init
  kPPExtraRows
};
__host__ __device__ constexpr size_t e_pp_rows(uint32_t exp2) { return 5 * (size_t)exp2 + kPPExtraRows; }

template <class O>
struct EPPInitSink {
  uint32_t* tab;
  size_t row;
  __device__ __forceinline__ void tangent(int sa, int sb, int sc) {
    A1Table T{tab};
    T.store<O>(row, sa);
    T.store<O>(row + 1, sb);
    T.store<O>(row + 2, sc);
    e_line_r<O>(eT5, eT6, sa, sb, sc);
    O::mul(eVD, eVD, eT5);
  }
  __device__ __forceinline__ void vertical() {
    A1Table T{tab};
    T.store<O>(row + 3, eZ2);
    T.store<O>(row + 4, eX);
    e_vert_r<O>(eT5);
    O::mul(eV, eV, eT5);
    row += 5;
  }
};

// pairing_pp_init: one thread walks V once, tabulates every line's coefficients and folds every value
// at R into (kPPVR, kPPVDR).  tab[rows * 34] = 1 if P is on the curve.
template <int BLOCK>
__global__ void __launch_bounds__(BLOCK)
k_e_pp_init(const uint8_t* __restrict__ P, uint32_t* __restrict__ tab) {
  using O = Ops<kNA1, false, BLOCK>;
  constexpr int eP = kESlots;      // one slot more than the Miller kernel: x(P)
  if (blockIdx.x != 0 || threadIdx.x != 0) return;
  const size_t rows = e_pp_rows(c_e.exp2), base = 5 * (size_t)c_e.exp2;
  bool okP = e_load_point<O>(eX, eY, eT0, eT1, P);
  O::copy(eP, eX);
  O::set_const(eZ, c_fp.one);
  O::set_const(eZ2, c_fp.one);
  O::set_const(eV, c_fp.one);      // the R side of v and vd
  O::set_const(eVD, c_fp.one);
  A1Table T{tab};
  EPPInitSink<O> s{tab, 0};
  const int exp1 = (int)c_e.exp1, exp2 = (int)c_e.exp2;
  for (int i = 0; i < exp2; i++) {
    if (i == exp1) {
      T.store<O>(base + kPPSaveZ2, eZ2);
      T.store<O>(base + kPPSaveX, eX);
      if (c_e.sign1 < 0) {
        e_vert_r<O>(eT5);
        O::mul(eT5, eVD, eT5);
        T.store<O>(base + kPPV1, eT5);
        T.store<O>(base + kPPVD1, eV);
        O::neg(eT5, eY);
        T.store<O>(base + kPPY1, eT5);
      } else {
        T.store<O>(base + kPPV1, eV);
        T.store<O>(base + kPPVD1, eVD);
        T.store<O>(base + kPPY1, eY);
      }
      T.store<O>(base + kPPX1, eX);
      T.store<O>(base + kPPZ1, eZ);
    }
    O::sqr(eV, eV);
    O::sqr(eVD, eVD);
    e_dbl_step<O>(s);
  }
  O::mulg(eV, eV, e_row(tab, base + kPPV1), 1);
  O::mulg(eVD, eVD, e_row(tab, base + kPPVD1), 1);
  e_chord<O>(e_row(tab, base + kPPX1), e_row(tab, base + kPPY1), e_row(tab, base + kPPZ1), 1);
  T.store<O>(base + kPPChordA, eT2);
  T.store<O>(base + kPPChordB, eT4);
  T.store<O>(base + kPPChordC, eT5);
  e_line_r<O>(eT0, eT1, eT2, eT4, eT5);
  O::mul(eVD, eVD, eT0);
  if (c_e.sign0 < 0) {
    O::ld_global(eT0, g_e_pts, kERX, 1, 0);
    O::sub(eT0, eT0, eP);
    O::mul(eV, eV, eT0);
  }
  T.store<O>(base + kPPPx, eP);
  T.store<O>(base + kPPVR, eV);
  T.store<O>(base + kPPVDR, eVD);
  tab[rows * kNA1] = okP ? 1u : 0u;
}
constexpr int kEPPInitSlots = kESlots + 1;

// pairing_pp_apply: only the values at Q + R, about 9 products per step.  pv: [2][17][n] scratch
// (the numerator and denominator at the save point).
template <int BLOCK>
__global__ void __launch_bounds__(BLOCK)
k_e_pp_apply(const uint32_t* __restrict__ tab, const uint8_t* __restrict__ Q, void* __restrict__ f,
             void* __restrict__ dprod, void* __restrict__ pv, size_t n) {
  using O = Ops<kNA1, false, BLOCK>;
  enum { qX, qY, qXZ, qZ2, qZ3, qV, qVD, qT0, qT1, kSlots };
  size_t idx = (size_t)blockIdx.x * BLOCK + threadIdx.x;
  if (idx >= n) return;
  const size_t rows = e_pp_rows(c_e.exp2), base = 5 * (size_t)c_e.exp2;
  bool okQ = e_load_point<O>(qX, qY, qT0, qT1, Q + idx * 2 * (size_t)c_a1.wb);
  e_q_plus_r<O>(qX, qY, qV, qZ2, qZ3, qXZ);
  bool valid = okQ && tab[rows * kNA1] != 0;
  O::set_const(qV, c_fp.one);
  O::set_const(qVD, c_fp.one);
  const int exp1 = (int)c_e.exp1, exp2 = (int)c_e.exp2;
  size_t row = 0;
  for (int i = 0; i < exp2; i++) {
    if (i == exp1) {
      if (c_e.sign1 < 0) {
        e_vert_hom<O>(qT0, qT1, qX, e_row(tab, base + kPPSaveZ2), qZ2, e_row(tab, base + kPPSaveX), 1);
        O::mul(qT0, qV, qT0);
        O::st_global(pv, 1, n, idx, qT0);
        O::st_global(pv, 0, n, idx, qVD);
      } else {
        O::st_global(pv, 0, n, idx, qV);
        O::st_global(pv, 1, n, idx, qVD);
      }
    }
    O::sqr(qV, qV);
    O::sqr(qVD, qVD);
    e_line_hom<O>(qT0, qT1, qXZ, e_row(tab, row), qY, e_row(tab, row + 1), qZ3, e_row(tab, row + 2), 1);
    O::mul(qV, qV, qT0);
    e_vert_hom<O>(qT0, qT1, qX, e_row(tab, row + 3), qZ2, e_row(tab, row + 4), 1);
    O::mul(qVD, qVD, qT0);
    row += 5;
  }
  O::mulg(qV, qV, e_el(pv, 0, n, idx), n);
  O::mulg(qVD, qVD, e_el(pv, 1, n, idx), n);
  e_line_hom<O>(qT0, qT1, qXZ, e_row(tab, base + kPPChordA), qY, e_row(tab, base + kPPChordB), qZ3,
                e_row(tab, base + kPPChordC), 1);
  O::mul(qV, qV, qT0);
  if (c_e.sign0 < 0) {
    O::mulg(qT0, qZ2, e_row(tab, base + kPPPx), 1);
    O::sub(qT0, qX, qT0);
    O::mul(qVD, qVD, qT0);
  }
  O::mulg(qV, qV, e_row(tab, base + kPPVR), 1);
  O::mulg(qVD, qVD, e_row(tab, base + kPPVDR), 1);
  e_publish<O>(qV, qVD, valid, f, dprod, n, idx);
}
constexpr int kEPPSlots = 9;

// (v / vd)^((q-1)/r): one left-to-right window of width 4 over the constant exponent (odd powers
// x, x^3, .., x^15 in slots 0..7).  out: n * wb bytes, canonical; an inverted denominator of 0 -> 1.
template <int BLOCK>
__global__ void __launch_bounds__(BLOCK)
k_e_finalexp(const void* __restrict__ f, const void* __restrict__ dinv, uint8_t* __restrict__ out, size_t n) {
  using O = Ops<kNA1, false, BLOCK>;
  enum { fAcc = 8, kSlots };
  size_t idx = (size_t)blockIdx.x * BLOCK + threadIdx.x;
  if (idx >= n) return;
  O::ld_global(0, f, 0, n, idx);
  O::ld_global(fAcc, dinv, 0, n, idx);
  const bool identity = O::is_zero(fAcc);
  O::mul(0, 0, fAcc);
  O::sqr(fAcc, 0);
  for (int j = 1; j < 8; j++) O::mul(j, j - 1, fAcc);
  int i = (int)c_e.dstart;
  O::copy(fAcc, c_e.dig[i] >> 1);
  for (i--; i >= 0; i--) {
    O::sqr(fAcc, fAcc);
    const int d = c_e.dig[i];
    if (d) O::mul(fAcc, fAcc, d >> 1);
  }
  const int wb = (int)c_a1.wb;
  uint32_t x[kNA1], one[kNA1] = {1};
  O::st(0, one);
  O::mul(fAcc, fAcc, 0);           // leave Montgomery form
  O::ld(x, fAcc);
  if (identity) {
#pragma unroll
    for (int k = 0; k < kNA1; k++) x[k] = one[k];
  }
  a1_limbs_to_be(out + idx * (size_t)wb, x, wb);
}
constexpr int kEFinalSlots = 9;

}  // namespace pbcb200
