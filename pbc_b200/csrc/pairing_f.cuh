// pairing_f.cuh -- Type F pairing kernels (BN curve y^2 = x^3 + b, k = 12, 158-bit q).
//
// Device replacement for ecc/f_param.c: f_pairing (:289-311), cc_miller_no_denom (:97-248),
// f_tateexp (:250-283) and the tower it runs on -- F_q^2 = F_q[s]/(s^2 - beta)
// (arith/fieldquadratic.c:197-309) and F_q^12 = F_q^2[x]/(x^6 + alpha) (arith/poly.c:932-1143).
// Same field representation as the reference (so the 240 output bytes are the coefficients as
// they stand), different multiplication schedules:
//   * F_q^12 is multiplied as the quadratic extension F_q^6[x]/(x^2 - y) of
//     F_q^6 = F_q^2[y]/(y^3 - xi), xi = -alpha, y = x^2: even coefficients form the "real" F_q^6
//     half, odd coefficients the "imaginary" half.  mul = 3 Karatsuba F_q^6 products, square =
//     2 (complex squaring).  The reference uses one degree-6 Karatsuba + table reduction (mul) and
//     a schoolbook square.
//   * the Miller line c + (b Qy) x^3 + (a Qx) x^4 is multiplied in sparsely: 12 F_q^2 products.
//   * the Miller loop is inversion-free (miller_cc.cuh); the one F_q^12 inversion of the final
//     exponentiation goes down the tower to a single F_q inversion.
// Kernels: k_f_miller (one pairing per thread, Miller value to the workspace), k_f_prod (products
// of k Miller values), k_f_finalexp.
#pragma once
#include "miller_cc.cuh"
#include "prod_v.cuh"

namespace pbcb200 {

struct F2 { Fq a, b; };            // a + b s,  s^2 = beta
struct F12 { F2 c[6]; };           // sum c[i] x^i,  x^6 = xi = -alpha

struct FConsts {
  uint32_t beta[kNS];              // quadratic non-residue of F_q (Montgomery form)
  uint32_t xi[2][kNS];             // -alpha in F_q^2
  uint32_t xi_inv[2][kNS];         // 1 / (-alpha): untwisting factor (ecc/f_param.c:296-303)
  uint32_t twist_b[2][kNS];        // -alpha * b: G2 curve Y^2 = X^3 + twist_b (:367-378)
  uint32_t xpowq2[2][kNS];         // x^(q^2) = xpowq2 * x   (:422-444)
  uint32_t xpowq6[2][kNS];
  uint32_t xpowq8[2][kNS];
  uint32_t tateexp[16];            // (q^4 - q^2 + 1) / r   (:408-420), plain integer
  uint32_t tatebits;
  // BN structure (q = 36u^4 + 36u^3 + 24u^2 + 6u + 1, what f_param gen produces, ecc/f_param.c:449-):
  uint32_t bn;                     // 1 if u was recovered at init; 0 -> generic 472-bit power
  uint32_t u_neg;                  // sign of u
  uint32_t u_bits;
  uint32_t u_abs[2];               // |u|
  uint32_t pad[2];
  uint32_t frob[3][5][2][kNS];     // frob[k-1][i-1] = xi^(i (q^k - 1)/6): x^i -> frob * x^i under q^k
  // Internal basis (q = 3 mod 4 and a small xi' found at init; tools/proto_f_nice_basis.py):
  //   K = F_q[i]/(i^2 + 1),  F_q^12 = K[z]/(z^6 - xi'),  xi' = xi_a + xi_b i with small integers.
  //   phi2(a + b s) = a + (sigma b) i;  x -> tau z.  When nice == 0 the reference basis is used as is
  //   (sigma = 1, tau = 1, kx = ky = 1/xi).  xi, twist_b and frob hold the values of the basis in use.
  uint32_t nice;
  uint32_t xi_a, xi_b;
  uint32_t pad2;
  uint32_t sigma[kNS], sigma_inv[kNS];
  uint32_t kx[2][kNS], ky[2][kNS];     // second argument: Qx'' = phi2(Qx) kx, Qy'' = phi2(Qy) ky
  uint32_t tau[5][2][kNS];             // tau^j,  j = 1..5  (wire -> internal, test hook)
  uint32_t tau_inv[5][2][kNS];         // tau^-j, j = 1..5  (internal -> wire)
  uint32_t qsq[2 * kNS];               // q^2 as a plain double-width integer (lazy reduction offset)
  uint32_t qsqm[3][2 * kNS];           // q^2, 2 q^2, 3 q^2: starting values of the double-width accumulators
  uint32_t slots_ok;                   // internal basis in use and 3 q < 2^160: the slot-machine kernels apply
  uint32_t pad3[3];
};
__constant__ FConsts c_f;

// ---------------------------------------------------------------------------------------------
// F_q^2  (arith/fieldquadratic.c:197-309 fq_*)
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void f2_set(F2& r, const uint32_t c[2][kNS]) { fq_set(r.a, c[0]); fq_set(r.b, c[1]); }
// one out-of-line copy of the F_q^2 addition and subtraction (the tower routines contain dozens of them;
// inlined they make up most of f6_mul / f12_sqr and the kernels are instruction-fetch bound at full occupancy)
__device__ __noinline__ void f2_add_call(F2* r, const F2* x, const F2* y) { fq_add(r->a, x->a, y->a); fq_add(r->b, x->b, y->b); }
__device__ __noinline__ void f2_sub_call(F2* r, const F2* x, const F2* y) { fq_sub(r->a, x->a, y->a); fq_sub(r->b, x->b, y->b); }
__device__ __forceinline__ void f2_add(F2& r, const F2& x, const F2& y) { f2_add_call(&r, &x, &y); }
__device__ __forceinline__ void f2_sub(F2& r, const F2& x, const F2& y) { f2_sub_call(&r, &x, &y); }
__device__ __forceinline__ void f2_dbl(F2& r, const F2& x) { fq_dbl(r.a, x.a); fq_dbl(r.b, x.b); }
__device__ __forceinline__ void f2_neg(F2& r, const F2& x) { fq_neg(r.a, x.a); fq_neg(r.b, x.b); }
__device__ __forceinline__ void f2_zero(F2& r) { fq_zero(r.a); fq_zero(r.b); }
__device__ __forceinline__ bool f2_eq(const F2& x, const F2& y) { return fq_eq(x.a, y.a) && fq_eq(x.b, y.b); }

// (x0 + x1 s)(y0 + y1 s) = x0 y0 + beta x1 y1 + ((x0 + x1)(y0 + y1) - x0 y0 - x1 y1) s;
// internal basis: beta = -1, three multiplications.
// Internal basis, lazily reduced: three unreduced products, the Karatsuba combination on
// double-width values, two reductions:  re = x0 y0 - x1 y1 + q^2 (< 2 q^2),  im = (x0 + x1)(y0 + y1)
// - x0 y0 - x1 y1 (< 2 q^2); the operand sums stay below 2q < 2^160 and need no reduction.
__device__ __noinline__ void f2_mul(F2* r, const F2* x, const F2* y) {
  if (c_f.nice) {
    Fq x0 = x->a, x1 = x->b, y0 = y->a, y1 = y->b, sx, sy;
    FqW t0, t1, t2, qq;
    fq_add_nr(sx, x0, x1);
    fq_add_nr(sy, y0, y1);
    t0 = fq_mulw_call(x0, y0);
    t1 = fq_mulw_call(x1, y1);
    t2 = fq_mulw_call(sx, sy);
    fqw_sub(t2, t2, t0);
    fqw_sub(t2, t2, t1);
#pragma unroll
    for (int k = 0; k < 2 * kNS; k++) qq.v[k] = c_f.qsq[k];
    fqw_add(t0, t0, qq);
    fqw_sub(t0, t0, t1);
    r->a = fq_redc_call(t0);
    r->b = fq_redc_call(t2);
    return;
  }
  Fq t0, t1, t2, u;
  fq_add(t2, x->a, x->b);
  fq_add(u, y->a, y->b);
  fq_mul(t2, t2, u);
  fq_mul(t0, x->a, y->a);
  fq_mul(t1, x->b, y->b);
  fq_sub(t2, t2, t0);
  fq_sub(t2, t2, t1);
  if (c_f.nice) {
    fq_sub(r->a, t0, t1);
  } else {
    fq_set(u, c_f.beta);
    fq_mul(t1, t1, u);
    fq_add(r->a, t0, t1);
  }
  r->b = t2;
}
// x0^2 + beta x1^2 + 2 x0 x1 s;  internal basis: (x0 + x1)(x0 - x1) + 2 x0 x1 i
__device__ __noinline__ void f2_sqr(F2* r, const F2* x) {
  Fq t0, t1, t2, u;
  fq_mul(t2, x->a, x->b);
  if (c_f.nice) {
    fq_add(t0, x->a, x->b);
    fq_sub(t1, x->a, x->b);
    fq_mul(r->a, t0, t1);
  } else {
    fq_sqr(t0, x->a);
    fq_sqr(t1, x->b);
    fq_set(u, c_f.beta);
    fq_mul(t1, t1, u);
    fq_add(r->a, t0, t1);
  }
  fq_dbl(r->b, t2);
}
// multiplication by an element of F_q
__device__ __forceinline__ void f2_scale(F2& r, const F2& x, const Fq& k) { fq_mul(r.a, x.a, k); fq_mul(r.b, x.b, k); }
// Stack discipline for everything below (nvcc 12.9 was seen to give two LIVE address-taken
// temporaries the same stack slot when inlined helpers had left several disjoint-lifetime
// temporaries behind -- tests/test_gpu_towers.py op 4 caught it): a routine whose locals have their
// address taken is __noinline__ and declares them at function scope; inlined helpers take no
// addresses of their own locals.  Constants are passed as pointers into __constant__ memory.
__device__ __forceinline__ const F2* f2_const(const uint32_t c[2][kNS]) { return reinterpret_cast<const F2*>(c); }
// r (+)= k x for k in 0..7 given x, 2x, 4x: at most two additions, branches are warp-uniform
__device__ __forceinline__ void fq_small_combo(Fq& r, uint32_t k, const Fq& x1, const Fq& x2, const Fq& x4) {
  bool have = false;
  if (k & 4u) { r = x4; have = true; }
  if (k & 2u) { if (have) fq_add(r, r, x2); else r = x2; have = true; }
  if (k & 1u) { if (have) fq_add(r, r, x1); else r = x1; have = true; }
  if (!have) fq_zero(r);
}
// r = xi x.  Internal basis: xi' = a + b i with small integers a, b <= 7:
//   (a x0 - b x1) + (b x0 + a x1) i, the multiples built from x, 2x, 4x (6 additions for 4 + 2i;
// the first version ran four generic double-and-add loops here and spent 14% of k_f_miller's
// instructions in this routine).  Reference basis: a full F_q^2 product by xi.
__device__ __noinline__ void f2_mul_xi(F2& r, const F2& x) {
  if (c_f.nice) {
    const uint32_t a = c_f.xi_a, b = c_f.xi_b, m = a | b;
    Fq a1 = x.a, b1 = x.b, a2, a4, b2, b4, p, q2, s2, t;
    if (m & 6u) { fq_dbl(a2, a1); fq_dbl(b2, b1); }
    if (m & 4u) { fq_dbl(a4, a2); fq_dbl(b4, b2); }
    fq_small_combo(p, a, a1, a2, a4);      // a x0
    fq_small_combo(q2, b, b1, b2, b4);     // b x1
    fq_small_combo(s2, b, a1, a2, a4);     // b x0
    fq_small_combo(t, a, b1, b2, b4);      // a x1
    fq_sub(r.a, p, q2);
    fq_add(r.b, s2, t);
  } else {
    f2_mul(&r, &x, f2_const(c_f.xi));
  }
}
// 1/(x0 + x1 s) = (x0 - x1 s)/(x0^2 - beta x1^2)   (arith/fieldquadratic.c:290-309)
__device__ __noinline__ void f2_inv(F2* r, const F2* x) {
  Fq t0, t1, u;
  fq_sqr(t0, x->a);
  fq_sqr(t1, x->b);
  if (c_f.nice) {
    fq_add(t0, t0, t1);                // norm x0^2 + x1^2
  } else {
    fq_set(u, c_f.beta);
    fq_mul(t1, t1, u);
    fq_sub(t0, t0, t1);
  }
  fq_inv(&t0, &t0);
  fq_mul(r->a, x->a, t0);
  fq_mul(t1, x->b, t0);
  fq_neg(r->b, t1);
}

// ---------------------------------------------------------------------------------------------
// F_q^6 = F_q^2[y]/(y^3 - xi) on three strided coefficients of an F12 (stride 2: y = x^2)
// ---------------------------------------------------------------------------------------------
struct F6 { F2 c[3]; };

// Karatsuba: 6 F_q^2 products + 2 multiplications by xi
__device__ __noinline__ void f6_mul(F6* r, const F6* a, const F6* b) {
  F2 v0, v1, v2, s, t, u, c0, c1;
  f2_mul(&v0, &a->c[0], &b->c[0]);
  f2_mul(&v1, &a->c[1], &b->c[1]);
  f2_mul(&v2, &a->c[2], &b->c[2]);
  // c0 = v0 + xi ((a1 + a2)(b1 + b2) - v1 - v2)
  f2_add(s, a->c[1], a->c[2]);
  f2_add(t, b->c[1], b->c[2]);
  f2_mul(&u, &s, &t);
  f2_sub(u, u, v1);
  f2_sub(u, u, v2);
  f2_mul_xi(u, u);
  f2_add(c0, v0, u);
  // c1 = (a0 + a1)(b0 + b1) - v0 - v1 + xi v2
  f2_add(s, a->c[0], a->c[1]);
  f2_add(t, b->c[0], b->c[1]);
  f2_mul(&u, &s, &t);
  f2_sub(u, u, v0);
  f2_sub(u, u, v1);
  f2_mul_xi(c1, v2);
  f2_add(c1, c1, u);
  // c2 = (a0 + a2)(b0 + b2) - v0 - v2 + v1
  f2_add(s, a->c[0], a->c[2]);
  f2_add(t, b->c[0], b->c[2]);
  f2_mul(&u, &s, &t);
  f2_sub(u, u, v0);
  f2_sub(u, u, v2);
  f2_add(r->c[2], u, v1);
  r->c[0] = c0;
  r->c[1] = c1;
}
__device__ __forceinline__ void f6_add(F6& r, const F6& a, const F6& b) {
#pragma unroll
  for (int i = 0; i < 3; i++) f2_add(r.c[i], a.c[i], b.c[i]);
}
__device__ __forceinline__ void f6_sub(F6& r, const F6& a, const F6& b) {
#pragma unroll
  for (int i = 0; i < 3; i++) f2_sub(r.c[i], a.c[i], b.c[i]);
}
// r = y a:  (a0, a1, a2) -> (xi a2, a0, a1)
__device__ __noinline__ void f6_mul_y(F6& r, const F6& a) {
  F2 t;
  f2_mul_xi(t, a.c[2]);
  r.c[2] = a.c[1];
  r.c[1] = a.c[0];
  r.c[0] = t;
}
// 1/a via the norm to F_q^2:  with A = a0^2 - xi a1 a2, B = xi a2^2 - a0 a1, C = a1^2 - a0 a2,
//   a (A + B y + C y^2) = a0 A + xi (a2 B + a1 C)  in F_q^2
__device__ __noinline__ void f6_inv(F6* r, const F6* a) {
  F2 A, B, C, t, u;
  f2_sqr(&A, &a->c[0]);
  f2_mul(&t, &a->c[1], &a->c[2]);
  f2_mul_xi(t, t);
  f2_sub(A, A, t);
  f2_sqr(&B, &a->c[2]);
  f2_mul_xi(B, B);
  f2_mul(&t, &a->c[0], &a->c[1]);
  f2_sub(B, B, t);
  f2_sqr(&C, &a->c[1]);
  f2_mul(&t, &a->c[0], &a->c[2]);
  f2_sub(C, C, t);
  f2_mul(&t, &a->c[2], &B);
  f2_mul(&u, &a->c[1], &C);
  f2_add(t, t, u);
  f2_mul_xi(t, t);
  f2_mul(&u, &a->c[0], &A);
  f2_add(t, t, u);
  f2_inv(&t, &t);
  f2_mul(&r->c[0], &A, &t);
  f2_mul(&r->c[1], &B, &t);
  f2_mul(&r->c[2], &C, &t);
}

// ---------------------------------------------------------------------------------------------
// F_q^12 = F_q^6[x]/(x^2 - y): even coefficients = real half, odd = imaginary half
// ---------------------------------------------------------------------------------------------
// Storage order: the three even coefficients (the "real" F_q^6 half) first, then the three odd ones, so
// both halves are F6 objects in place and no routine copies them around:
//   coefficient j of x^j lives at c[f12_pos(j)],  f12_pos = 0 3 1 4 2 5.
__device__ __forceinline__ constexpr int f12_pos(int j) { return (j >> 1) + 3 * (j & 1); }
#define F12C(v, j) ((v).c[f12_pos(j)])
__device__ __forceinline__ F6* f12_lo(F12* v) { return reinterpret_cast<F6*>(&v->c[0]); }
__device__ __forceinline__ F6* f12_hi(F12* v) { return reinterpret_cast<F6*>(&v->c[3]); }
__device__ __forceinline__ const F6* f12_lo(const F12* v) { return reinterpret_cast<const F6*>(&v->c[0]); }
__device__ __forceinline__ const F6* f12_hi(const F12* v) { return reinterpret_cast<const F6*>(&v->c[3]); }
__device__ __forceinline__ void f12_one(F12& v) {
#pragma unroll
  for (int i = 0; i < 6; i++) f2_zero(v.c[i]);
  fq_one(v.c[0].a);
}

// (A + B x)(C + D x) = AC + y BD + ((A + B)(C + D) - AC - BD) x;  r may alias p or q
__device__ __noinline__ void f12_mul(F12* r, const F12* p, const F12* q) {
  F6 t0, t1, t2, s1, s2;
  f6_mul(&t0, f12_lo(p), f12_lo(q));
  f6_mul(&t1, f12_hi(p), f12_hi(q));
  f6_add(s1, *f12_lo(p), *f12_hi(p));
  f6_add(s2, *f12_lo(q), *f12_hi(q));
  f6_mul(&t2, &s1, &s2);
  f6_sub(t2, t2, t0);
  f6_sub(t2, t2, t1);
  f6_mul_y(t1, t1);
  f6_add(*f12_lo(r), t0, t1);
  *f12_hi(r) = t2;
}
// (A + B x)^2 = (A + B)(A + y B) - AB - y AB + 2 AB x, in place
__device__ __noinline__ void f12_sqr(F12* v) {
  F6 t0, t1, t2;
  f6_mul(&t0, f12_lo(v), f12_hi(v));
  f6_mul_y(t1, *f12_hi(v));
  f6_add(t1, t1, *f12_lo(v));
  f6_add(t2, *f12_lo(v), *f12_hi(v));
  f6_mul(&t2, &t2, &t1);
  f6_sub(t2, t2, t0);
  f6_mul_y(t1, t0);
  f6_sub(*f12_lo(v), t2, t1);
  f6_add(*f12_hi(v), t0, t0);
}
// 1/(A + B x) = (A - B x)/(A^2 - y B^2);  r may alias p
__device__ __noinline__ void f12_inv(F12* r, const F12* p) {
  F6 t0, t1;
  f6_mul(&t0, f12_lo(p), f12_lo(p));
  f6_mul(&t1, f12_hi(p), f12_hi(p));
  f6_mul_y(t1, t1);
  f6_sub(t0, t0, t1);
  f6_inv(&t0, &t0);
  f6_mul(&t1, f12_hi(p), &t0);
  f6_mul(f12_lo(r), f12_lo(p), &t0);
#pragma unroll
  for (int i = 0; i < 3; i++) f2_neg(f12_hi(r)->c[i], t1.c[i]);
}

// double-width x y for F_q^2 operands in the internal basis (i^2 = -1), added into (re, im):
//   re += x0 y0 - x1 y1 + q^2,  im += (x0 + x1)(y0 + y1) - x0 y0 - x1 y1       (each term < 2 q^2)
__device__ __forceinline__ void f2_mulw_acc(FqW& re, FqW& im, const F2& x, const F2& y, const FqW& qq, bool first) {
  Fq sx, sy;
  FqW t0, t1, t2;
  fq_add_nr(sx, x.a, x.b);
  fq_add_nr(sy, y.a, y.b);
  t0 = fq_mulw_call(x.a, y.a);
  t1 = fq_mulw_call(x.b, y.b);
  t2 = fq_mulw_call(sx, sy);
  fqw_sub(t2, t2, t0);
  fqw_sub(t2, t2, t1);
  fqw_add(t0, t0, qq);
  fqw_sub(t0, t0, t1);
  if (first) { re = t0; im = t2; } else { fqw_add(re, re, t0); fqw_add(im, im, t2); }
}
__device__ __noinline__ void f12_mul_line(F12* v, const Fq* c, const F2* L3, const F2* L4) {
  // m3[0] = xi L3 (used when the product wraps past x^5), m3[1] = L3; same for L4.  (Indexing an
  // array instead of selecting between two pointers: nvcc 12.9 merged the stack slots of two live
  // temporaries when the operand pointer came from a select -- see tests/test_gpu_towers.py op 4.)
  F2 m3[2], m4[2], t, u, w;
  F12 o;
  FqW re, im, qq, sc;
  m3[1] = *L3;
  m4[1] = *L4;
  f2_mul_xi(m3[0], m3[1]);
  f2_mul_xi(m4[0], m4[1]);
  if (c_f.nice) {
    // every output coefficient is the sum of three products: accumulate them unreduced and reduce
    // once (5 q^2 < 2 q R: fq_redc2) -- 12 reductions per line instead of 36
#pragma unroll
    for (int k = 0; k < 2 * kNS; k++) qq.v[k] = c_f.qsq[k];
#pragma unroll 1
    for (int k = 0; k < 6; k++) {
      int i3 = k >= 3 ? k - 3 : k + 3, i4 = k >= 4 ? k - 4 : k + 2;
      f2_mulw_acc(re, im, m3[k >= 3 ? 1 : 0], F12C(*v, i3), qq, true);
      f2_mulw_acc(re, im, m4[k >= 4 ? 1 : 0], F12C(*v, i4), qq, false);
      sc = fq_mulw_call(*c, F12C(*v, k).a);
      fqw_add(re, re, sc);
      sc = fq_mulw_call(*c, F12C(*v, k).b);
      fqw_add(im, im, sc);
      F12C(o, k).a = fq_redc2_call(re);
      F12C(o, k).b = fq_redc2_call(im);
    }
    *v = o;
    return;
  }
#pragma unroll 1
  for (int k = 0; k < 6; k++) {
    int i3 = k >= 3 ? k - 3 : k + 3, i4 = k >= 4 ? k - 4 : k + 2;
    f2_mul(&t, &m3[k >= 3 ? 1 : 0], &F12C(*v, i3));
    f2_mul(&u, &m4[k >= 4 ? 1 : 0], &F12C(*v, i4));
    f2_scale(w, F12C(*v, k), *c);
    f2_add(t, t, u);
    f2_add(F12C(o, k), t, w);
  }
  *v = o;
}

// ---------------------------------------------------------------------------------------------
// Miller loop plumbing
// ---------------------------------------------------------------------------------------------
struct FTower {
  typedef F12 Acc;
  struct Ctx { F2 Qx, Qy; };     // untwisted second argument
  static __device__ __noinline__ void mul_line(F12* v, const Fq* a, const Fq* b, const Fq* c,
                                              const Ctx* q) {
    F2 L3, L4;
    f2_scale(L3, q->Qy, *b);
    f2_scale(L4, q->Qx, *a);
    f12_mul_line(v, c, &L3, &L4);
  }
  static __device__ __forceinline__ void sqr(F12* v) { f12_sqr(v); }
};

constexpr int kF12Words = 12 * kNS;    // 60 words per Miller value in the workspace

__device__ __forceinline__ void f12_st_global(uint32_t* g, size_t n, size_t idx, const F12& v) {
#pragma unroll
  for (int i = 0; i < 6; i++) {
    fq_st_global(g, 2 * i, n, idx, v.c[i].a);
    fq_st_global(g, 2 * i + 1, n, idx, v.c[i].b);
  }
}
__device__ __forceinline__ void f12_ld_global(F12& v, const uint32_t* g, size_t n, size_t idx) {
#pragma unroll
  for (int i = 0; i < 6; i++) {
    fq_ld_global(v.c[i].a, g, 2 * i, n, idx);
    fq_ld_global(v.c[i].b, g, 2 * i + 1, n, idx);
  }
}

// internal basis -> reference basis (identity when nice == 0): c_j = phi2^-1(d_j tau^-j)
__device__ __noinline__ void f12_to_reference(F12& v) {
  Fq k;
  if (!c_f.nice) return;
#pragma unroll 1
  for (int j = 1; j < 6; j++) f2_mul(&F12C(v, j), &F12C(v, j), f2_const(c_f.tau_inv[j - 1]));
  fq_set(k, c_f.sigma_inv);
#pragma unroll 1
  for (int j = 0; j < 6; j++) fq_mul(v.c[j].b, v.c[j].b, k);
}
// reference basis -> internal basis (test hook)
__device__ __noinline__ void f12_to_internal(F12& v) {
  Fq k;
  if (!c_f.nice) return;
  fq_set(k, c_f.sigma);
#pragma unroll 1
  for (int j = 0; j < 6; j++) fq_mul(v.c[j].b, v.c[j].b, k);
#pragma unroll 1
  for (int j = 1; j < 6; j++) f2_mul(&F12C(v, j), &F12C(v, j), f2_const(c_f.tau[j - 1]));
}

// P: n1 x 40 bytes (stride1 = 0 shares one P: pairing_pp_*), Q: n x 80 bytes.
// mv: [60][n] words, flag[n]: 1 = both inputs finite points on their curves.
template <int BLOCK>
__global__ void __launch_bounds__(BLOCK, (kCCMinBlocks * 128) / BLOCK)
k_f_miller(const uint8_t* __restrict__ P, const uint8_t* __restrict__ Q, uint32_t* __restrict__ mv,
           uint32_t* __restrict__ flag, size_t n, size_t stride1, const uint32_t* __restrict__ tab, size_t rows) {
  size_t idx = (size_t)blockIdx.x * BLOCK + threadIdx.x;
  const bool live = idx < n;      // every thread runs the loop (block-wide barrier inside)
  if (!live) idx = 0;
  Fq xP, yP, yP2;
  bool ok;
  if (tab) {
    ok = tab[3 * rows * kNS] != 0;             // fixed first argument: lines from the table (k_cc_pp_init)
  } else {
    const uint8_t* p = P + idx * stride1;
    fq_from_wire(xP, p);
    fq_from_wire(yP, p + kWS);
    ok = cc_on_curve(xP, yP);
  }
  FTower::Ctx ctx;
  F2 t, u;
  F12 v;
  const uint8_t* q = Q + idx * (4 * kWS);
  fq_from_wire(ctx.Qx.a, q);
  fq_from_wire(ctx.Qx.b, q + kWS);
  fq_from_wire(ctx.Qy.a, q + 2 * kWS);
  fq_from_wire(ctx.Qy.b, q + 3 * kWS);
  // into the basis in use: phi2(a + b s) = a + (sigma b) i  (sigma = 1 in the reference basis)
  fq_set(yP2, c_f.sigma);
  fq_mul(ctx.Qx.b, ctx.Qx.b, yP2);
  fq_mul(ctx.Qy.b, ctx.Qy.b, yP2);
  // Y^2 == X^3 + twist_b on the twist (ecc/curve.c:57-76 over F_q^2; phi2 is a field isomorphism)
  f2_sqr(&t, &ctx.Qx);
  f2_mul(&t, &t, &ctx.Qx);
  f2_add(t, t, *f2_const(c_f.twist_b));
  f2_sqr(&u, &ctx.Qy);
  ok = ok && f2_eq(t, u);
  // untwist (ecc/f_param.c:296-303) and scale for the line's x^4 / x^3 positions: kx = tau^4 / xi,
  // ky = tau^3 / xi  (both 1 / xi in the reference basis)
  f2_mul(&ctx.Qx, &ctx.Qx, f2_const(c_f.kx));
  f2_mul(&ctx.Qy, &ctx.Qy, f2_const(c_f.ky));
  f12_one(v);
  if (tab) miller_cc_tab<FTower>(&v, tab, &ctx);
  else miller_cc<FTower>(&v, xP, yP, &ctx);   // off-curve inputs run too (total arithmetic) and are flagged
  if (!live) return;
  if (!ok) f12_one(v);
  f12_st_global(mv, n, idx, v);
  flag[idx] = ok ? 1u : 0u;
}

// generic_prod_pairings (ecc/pairing.c:35-46) multiplies k complete pairings; the final
// exponentiation is a homomorphism, so the k Miller values are multiplied here and exponentiated
// once.  Any O input -> identity (include/pbc_pairing.h:161-168).
template <int BLOCK>
__global__ void __launch_bounds__(BLOCK, kCCMinBlocks)
k_f_prod(const uint32_t* __restrict__ mv_in, const uint32_t* __restrict__ flag_in,
         uint32_t* __restrict__ mv_out, uint32_t* __restrict__ flag_out, size_t k, size_t n_out,
         size_t n_in) {
  size_t idx = (size_t)blockIdx.x * BLOCK + threadIdx.x;
  if (idx >= n_out) return;
  F12 acc, t;
  bool ok = true;
  f12_ld_global(acc, mv_in, n_in, idx * k);
  ok = flag_in[idx * k] != 0;
  for (size_t j = 1; j < k; j++) {
    f12_ld_global(t, mv_in, n_in, idx * k + j);
    ok = ok && flag_in[idx * k + j] != 0;
    f12_mul(&acc, &acc, &t);
  }
  f12_st_global(mv_out, n_out, idx, acc);
  flag_out[idx] = ok ? 1u : 0u;
}

// the same product over a run table (prod_v.cuh, pbc_b200_prod_pairings_apply_v)
struct F12ProdV {
  using E = F12;
  static constexpr int kMinBlocks = kCCMinBlocks;
  static __device__ __forceinline__ void ld(E& v, const uint32_t* g, size_t n, size_t i) { f12_ld_global(v, g, n, i); }
  static __device__ __forceinline__ void st(uint32_t* g, size_t n, size_t i, const E& v) { f12_st_global(g, n, i, v); }
  static __device__ __forceinline__ void mul(E* r, const E* x, const E* y) { f12_mul(r, x, y); }
};

// f^(q^6): x -> -x
__device__ __forceinline__ void f12_conj(F12& r, const F12& f) {
#pragma unroll
  for (int i = 0; i < 3; i++) {            // storage: even coefficients 0..2, odd ones 3..5
    r.c[i] = f.c[i];
    f2_neg(r.c[3 + i], f.c[3 + i]);
  }
}
// f^(q^k), k = 1, 2, 3: coefficient i is conjugated in F_q^2 for odd k and scaled by frob[k-1][i-1]
__device__ __noinline__ void f12_frob(F12& r, const F12& f, int k) {
  F2 t;
  r.c[0] = f.c[0];
  if (k & 1) fq_neg(r.c[0].b, f.c[0].b);
#pragma unroll 1
  for (int i = 1; i < 6; i++) {
    t = F12C(f, i);
    if (k & 1) fq_neg(t.b, t.b);
    f2_mul(&F12C(r, i), &t, f2_const(c_f.frob[k - 1][i - 1]));
  }
}
// (a + b s)^2 in F_q^4 = F_q^2[s]/(s^2 - xi), s = x^3:  (a^2 + xi b^2, (a + b)^2 - a^2 - b^2)
__device__ __noinline__ void f4_sqr(F2* r0, F2* r1, const F2* a, const F2* b) {
  F2 sa, sb, t;
  f2_sqr(&sa, a);
  f2_sqr(&sb, b);
  f2_add(t, *a, *b);
  f2_sqr(&t, &t);
  f2_sub(t, t, sa);
  f2_sub(*r1, t, sb);
  f2_mul_xi(sb, sb);
  f2_add(*r0, sa, sb);
}
// Squaring in the cyclotomic subgroup (Granger-Scott; tools/proto_f_cyclo_sqr.py): with F_q^12 seen as
// F_q^4[x]/(x^3 - s), f = u0 + u1 x + u2 x^2, u0 = (c0, c3), u1 = (c1, c4), u2 = (c2, c5):
//   f^2 = (3 u0^2 - 2 conj u0) + (3 s u2^2 + 2 conj u1) x + (3 u1^2 - 2 conj u2) x^2
// 9 F_q^2 squarings instead of the 12 products of the generic square.  Valid after the easy part of
// the final exponentiation only.
__device__ __noinline__ void f12_cyc_sqr(F12* v) {
  F2 A0, A1, B0, B1, C0, C1, t;
  f4_sqr(&A0, &A1, &F12C(*v, 0), &F12C(*v, 3));
  f4_sqr(&B0, &B1, &F12C(*v, 1), &F12C(*v, 4));
  f4_sqr(&C0, &C1, &F12C(*v, 2), &F12C(*v, 5));
  // 3X -+ 2u: X + 2 (X -+ u)
  f2_sub(t, A0, F12C(*v, 0)); f2_dbl(t, t); f2_add(F12C(*v, 0), t, A0);
  f2_add(t, A1, F12C(*v, 3)); f2_dbl(t, t); f2_add(F12C(*v, 3), t, A1);
  f2_sub(t, B0, F12C(*v, 2)); f2_dbl(t, t); f2_add(F12C(*v, 2), t, B0);
  f2_add(t, B1, F12C(*v, 5)); f2_dbl(t, t); f2_add(F12C(*v, 5), t, B1);
  f2_mul_xi(C1, C1);                       // s (C0 + C1 s) = xi C1 + C0 s
  f2_add(t, C1, F12C(*v, 1)); f2_dbl(t, t); f2_add(F12C(*v, 1), t, C1);
  f2_sub(t, C0, F12C(*v, 4)); f2_dbl(t, t); f2_add(F12C(*v, 4), t, C0);
}

// f^u for the BN parameter u (on the cyclotomic subgroup the inverse is the conjugate)
__device__ __noinline__ void f12_pow_u(F12& r, const F12& f) {
  F12 acc;
  acc = f;
  for (int j = (int)c_f.u_bits - 2; j >= 0; j--) {
    __syncthreads();        // uniform loop: keep the block's warps in step
    f12_cyc_sqr(&acc);
    if ((c_f.u_abs[j >> 5] >> (j & 31)) & 1u) f12_mul(&acc, &acc, &f);
  }
  if (c_f.u_neg) f12_conj(r, acc); else r = acc;
}

// f_tateexp (ecc/f_param.c:250-283): f^((q^6 - 1)(q^2 + 1)) then the power (q^4 - q^2 + 1)/r.
// Same value, different route (tools/proto_f_finalexp.py checks it against the oracle):
//   easy part  g = conj(f)/f,  f <- g^(q^2) g             (the reference multiplies four q-powers)
//   hard part  (q^4 - q^2 + 1)/r = l0 + l1 q + l2 q^2 + q^3 with l_i polynomials in the BN
//              parameter u: three powers by u (39 bits for f.param) and the fixed multiplication
//              chain of Scott et al. -- about 120 squarings instead of the 472 of the windowed power
//              the reference runs (arith/field.c:14-126).  Parameter sets that are not of BN form
//              take the generic square-and-multiply over c_f.tateexp.
__device__ __noinline__ void f12_final_exp(F12& acc, F12& f) {
  F12 fu, fu2, fu3, t0, t1, x, y;
  f12_inv(&x, &f);
  f12_conj(y, f);
  f12_mul(&x, &x, &y);                 // f^(q^6 - 1)
  f12_frob(y, x, 2);
  f12_mul(&f, &y, &x);                 // ^(q^2 + 1)
  if (!c_f.bn) {
    acc = f;
    for (int j = (int)c_f.tatebits - 2; j >= 0; j--) {
      f12_sqr(&acc);
      if ((c_f.tateexp[j >> 5] >> (j & 31)) & 1u) f12_mul(&acc, &acc, &f);
    }
    return;
  }
  f12_pow_u(fu, f);
  f12_pow_u(fu2, fu);
  f12_pow_u(fu3, fu2);
  f12_frob(x, fu3, 1);
  f12_mul(&x, &x, &fu3);
  f12_conj(t0, x);                     // y6 = 1/(f^(u^3) f^(u^3 q))
  f12_cyc_sqr(&t0);
  f12_frob(x, fu2, 1);
  f12_mul(&x, &x, &fu);
  f12_conj(y, x);                      // y4 = 1/(f^u f^(u^2 q))
  f12_mul(&t0, &t0, &y);
  f12_conj(y, fu2);                    // y5 = 1/f^(u^2)
  f12_mul(&t0, &t0, &y);
  f12_frob(x, fu, 1);
  f12_conj(t1, x);                     // y3 = 1/f^(u q)
  f12_mul(&t1, &t1, &y);
  f12_mul(&t1, &t1, &t0);
  f12_frob(x, fu2, 2);                 // y2 = f^(u^2 q^2)
  f12_mul(&t0, &t0, &x);
  f12_cyc_sqr(&t1);
  f12_mul(&t1, &t1, &t0);
  f12_cyc_sqr(&t1);
  f12_conj(y, f);                      // y1 = 1/f
  f12_mul(&t0, &t1, &y);
  f12_frob(x, f, 1);
  f12_frob(y, f, 2);
  f12_mul(&x, &x, &y);
  f12_frob(y, f, 3);
  f12_mul(&x, &x, &y);                 // y0 = f^q f^(q^2) f^(q^3)
  f12_mul(&t1, &t1, &x);
  f12_cyc_sqr(&t0);
  f12_mul(&acc, &t0, &t1);
}

// f_tateexp (ecc/f_param.c:250-283): f^((q^6 - 1)(q^2 + 1)) by Frobenius constants and one
// inversion, then the 472-bit power (q^4 - q^2 + 1)/r.  out: n x 240 bytes, coefficient order
// x^0..x^5, each (re, im) (arith/poly.c:718-727, arith/fieldquadratic.c:323-329).
template <int BLOCK>
__global__ void __launch_bounds__(BLOCK, (kCCMinBlocks * 128) / BLOCK)
k_f_finalexp(const uint32_t* __restrict__ mv, const uint32_t* __restrict__ flag,
             uint8_t* __restrict__ out, size_t n) {
  size_t idx = (size_t)blockIdx.x * BLOCK + threadIdx.x;
  const bool live = idx < n;             // padding threads of the last block run too: f12_pow_u has block-wide barriers
  if (!live) idx = 0;
  F12 f, acc;
  const bool ok = flag[idx] != 0;
  // every thread runs the exponentiation (block-wide barriers inside f12_pow_u); flagged-off
  // entries exponentiate 1 and are overwritten with the identity afterwards
  f12_ld_global(f, mv, n, idx);
  if (!ok) f12_one(f);
  f12_final_exp(acc, f);
  if (!live) return;                     // after the last barrier
  f12_to_reference(acc);
  if (!ok) f12_one(acc);
  uint8_t* o = out + idx * (12 * kWS);
#pragma unroll 1
  for (int i = 0; i < 6; i++) {
    fq_to_wire(o + (2 * i) * kWS, F12C(acc, i).a);
    fq_to_wire(o + (2 * i + 1) * kWS, F12C(acc, i).b);
  }
}

__device__ __forceinline__ void f12_from_wire(F12& v, const uint8_t* p) {
#pragma unroll 1
  for (int i = 0; i < 6; i++) {
    fq_from_wire(F12C(v, i).a, p + (2 * i) * kWS);
    fq_from_wire(F12C(v, i).b, p + (2 * i + 1) * kWS);
  }
}
__device__ __forceinline__ void f12_to_wire(uint8_t* p, const F12& v) {
#pragma unroll 1
  for (int i = 0; i < 6; i++) {
    fq_to_wire(p + (2 * i) * kWS, F12C(v, i).a);
    fq_to_wire(p + (2 * i + 1) * kWS, F12C(v, i).b);
  }
}

// Differential-test hook on GT-sized operands (240 wire bytes): op 0 = a*b, 1 = a^2, 2 = 1/a,
// 3 = f_tateexp(a), 5 = cyclotomic square of a (a must be in the cyclotomic subgroup), 4 = a * line, the line c + L3 x^3 + L4 x^4 taken from b's coefficients 0 (real
// part only), 3 and 4.
__global__ void k_f_tower_op(int op, uint8_t* __restrict__ out, const uint8_t* __restrict__ a,
                             const uint8_t* __restrict__ b, size_t n) {
  size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const bool live = idx < n;             // op 3 reaches the barriers of f12_pow_u: no early exit
  if (!live) idx = 0;
  F12 x, y, r;
  f12_from_wire(x, a + idx * (12 * kWS));
  f12_from_wire(y, b + idx * (12 * kWS));
  f12_to_internal(x);
  f12_to_internal(y);
  switch (op) {
    case 0: f12_mul(&r, &x, &y); break;
    case 1: r = x; f12_sqr(&r); break;
    case 2: f12_inv(&r, &x); break;
    case 3: f12_final_exp(r, x); break;
    case 5: r = x; f12_cyc_sqr(&r); break;
    default: r = x; f12_mul_line(&r, &F12C(y, 0).a, &F12C(y, 3), &F12C(y, 4)); break;
  }
  if (!live) return;
  f12_to_reference(r);
  f12_to_wire(out + idx * (12 * kWS), r);
}
// test hook of tower op 6: GT wire elements into the limb-major Miller-value layout k_f_finalexp and
// k_f_finalexp_s read (internal basis, Montgomery form), every flag set
__global__ void k_f_mv_from_wire(uint32_t* __restrict__ mv, uint32_t* __restrict__ flag, const uint8_t* __restrict__ a,
                                 size_t n) {
  size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n) return;
  F12 x;
  f12_from_wire(x, a + idx * (12 * kWS));
  f12_to_internal(x);
  f12_st_global(mv, n, idx, x);
  flag[idx] = 1u;
}

}  // namespace pbcb200
