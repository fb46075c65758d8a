// pairing_d.cuh -- Type D pairing kernels (MNT curve y^2 = x^3 + a x + b, k = 6, 159-bit q).
//
// Device replacement for ecc/d_param.c: cc_pairing (:570-587), cc_miller_no_denom_affine
// (:321-422), d_miller_evalfn (:99-111), cc_tatepower (:505-564), lucas_even (:441-502),
// cc_pairings_affine (:710-736), on the tower F_q^3 = F_q[x]/(x^3 + c2 x^2 + c1 x + c0)
// (arith/poly.c:870-930, 1049-1089, 1302-1333) and F_q^6 = F_q^3[w]/(w^2 - v), v in F_q
// (arith/fieldquadratic.c:197-309).  Same representation as the reference (the 120 output bytes are
// the coefficients as they stand); the Miller loop is inversion-free (miller_cc.cuh) and the
// extension-field inversions go down to a single F_q inversion each by way of the Frobenius
// constants x^q, x^(2q) the reference already computes (ecc/d_param.c:1043-1049).
#pragma once
#include "miller_cc.cuh"
#include "prod_v.cuh"

namespace pbcb200 {

struct F3 { Fq c[3]; };            // c0 + c1 x + c2 x^2
struct F6D { F3 a, b; };           // a + b w,  w^2 = v

template <int NS>
struct DConstsT {
  uint32_t xpwr3[3][NS];          // x^3 mod the field polynomial (arith/poly.c:1302-1333)
  uint32_t xpwr4[3][NS];          // x^4
  uint32_t xpowq[3][NS];          // x^q      (ecc/d_param.c:1043-1049)
  uint32_t xpowq2[3][NS];         // x^(2q)
  uint32_t nqr[NS];               // v
  uint32_t nqrinv[NS];            // 1/v    : untwisting factors (ecc/d_param.c:576-582)
  uint32_t nqrinv2[NS];           // 1/v^2
  uint32_t twist_a[NS];           // a v^2, b v^3: G2 curve over F_q^3 (ecc/curve.c:885-892)
  uint32_t twist_b[NS];
  uint32_t two[NS];               // Montgomery 2
  uint32_t phikonr[8];             // (q^2 - q + 1)/r, plain integer (ecc/d_param.c:1035-1041)
  uint32_t phibits;
  // Internal cubic basis (q = 2 mod 3; tools/proto_d_basis.py):  F_q^3 = F_q[w]/(w^3 + p w + 1) with
  // x = lam w - s, s = c2/3, lam^3 = c0 - c1 c2/3 + 2 c2^3/27, p = (c1 - c2^2/3)/lam^2.  A product
  // then folds its two high coefficients with 2 multiplications (by p) instead of 6.  nice == 0: the
  // reference polynomial (xpwr3/xpwr4 rows).  xpowq / xpowq2 hold the values of the basis in use.
  uint32_t nice;
  uint32_t pad[2];
  uint32_t pcoef[NS];             // p
  uint32_t bs[NS], bs2[NS], b2s[NS];          // s, s^2, 2 s
  uint32_t blam[NS], blam2[NS], blami[NS], blami2[NS];   // lam, lam^2, 1/lam, 1/lam^2
  uint32_t qsqm[2][2 * NS];       // q^2, 2 q^2 as plain double-width integers (offsets of the lazy F_q^3 product)
};
typedef DConstsT<kNS> DConsts;
__constant__ DConsts c_d;

// ---------------------------------------------------------------------------------------------
// F_q^3
// ---------------------------------------------------------------------------------------------
// The additions stay inline: out-of-line copies (as f2_add_call in pairing_f.cuh) were slower on type D,
// whose F_q^3 routines are smaller than F_q^12's.
__device__ __forceinline__ void f3_add(F3& r, const F3& x, const F3& y) {
#pragma unroll
  for (int i = 0; i < 3; i++) fq_add(r.c[i], x.c[i], y.c[i]);
}
__device__ __forceinline__ void f3_sub(F3& r, const F3& x, const F3& y) {
#pragma unroll
  for (int i = 0; i < 3; i++) fq_sub(r.c[i], x.c[i], y.c[i]);
}
__device__ __forceinline__ void f3_neg(F3& r, const F3& x) {
#pragma unroll
  for (int i = 0; i < 3; i++) fq_neg(r.c[i], x.c[i]);
}
__device__ __forceinline__ void f3_zero(F3& r) {
#pragma unroll
  for (int i = 0; i < 3; i++) fq_zero(r.c[i]);
}
__device__ __forceinline__ void f3_set(F3& r, const uint32_t c[3][kNS]) {
#pragma unroll
  for (int i = 0; i < 3; i++) fq_set(r.c[i], c[i]);
}
__device__ __forceinline__ bool f3_eq(const F3& x, const F3& y) {
  return fq_eq(x.c[0], y.c[0]) && fq_eq(x.c[1], y.c[1]) && fq_eq(x.c[2], y.c[2]);
}
__device__ __forceinline__ void f3_scale(F3& r, const F3& x, const Fq& k) {
#pragma unroll
  for (int i = 0; i < 3; i++) fq_mul(r.c[i], x.c[i], k);
}

// degree-4 product d0..d4 folded with the x^3, x^4 rows (polymod_mul_degree3, arith/poly.c:870-930);
// internal basis: w^3 = -p w - 1, w^4 = -p w^2 - w:  r0 = d0 - d3, r1 = d1 - p d3 - d4, r2 = d2 - p d4
__device__ __forceinline__ void f3_reduce(F3* r, const Fq& d0, const Fq& d1, const Fq& d2, const Fq& d3,
                                          const Fq& d4) {
  Fq t, k;
  if (c_d.nice) {
    fq_set(k, c_d.pcoef);
    fq_sub(r->c[0], d0, d3);
    fq_mul(t, d3, k);
    fq_sub(r->c[1], d1, t);
    fq_sub(r->c[1], r->c[1], d4);
    fq_mul(t, d4, k);
    fq_sub(r->c[2], d2, t);
    return;
  }
#pragma unroll
  for (int i = 0; i < 3; i++) {
    const Fq& lo = i == 0 ? d0 : (i == 1 ? d1 : d2);
    fq_set(k, c_d.xpwr3[i]);
    fq_mul(t, d3, k);
    fq_add(r->c[i], lo, t);
    fq_set(k, c_d.xpwr4[i]);
    fq_mul(t, d4, k);
    fq_add(r->c[i], r->c[i], t);
  }
}
// reference basis -> basis in use:  b0 = a0 - a1 s + a2 s^2,  b1 = lam (a1 - 2 s a2),  b2 = lam^2 a2
__device__ __noinline__ void f3_to_internal(F3& v) {
  Fq k, t, u;
  if (!c_d.nice) return;
  fq_set(k, c_d.bs);
  fq_mul(t, v.c[1], k);
  fq_sub(v.c[0], v.c[0], t);
  fq_set(k, c_d.bs2);
  fq_mul(t, v.c[2], k);
  fq_add(v.c[0], v.c[0], t);
  fq_set(k, c_d.b2s);
  fq_mul(t, v.c[2], k);
  fq_sub(u, v.c[1], t);
  fq_set(k, c_d.blam);
  fq_mul(v.c[1], u, k);
  fq_set(k, c_d.blam2);
  fq_mul(v.c[2], v.c[2], k);
}
// basis in use -> reference basis:  a2 = b2 / lam^2,  a1 = b1 / lam + 2 s a2,  a0 = b0 + a1 s - a2 s^2
__device__ __noinline__ void f3_to_reference(F3& v) {
  Fq k, t;
  if (!c_d.nice) return;
  fq_set(k, c_d.blami2);
  fq_mul(v.c[2], v.c[2], k);
  fq_set(k, c_d.blami);
  fq_mul(v.c[1], v.c[1], k);
  fq_set(k, c_d.b2s);
  fq_mul(t, v.c[2], k);
  fq_add(v.c[1], v.c[1], t);
  fq_set(k, c_d.bs);
  fq_mul(t, v.c[1], k);
  fq_add(v.c[0], v.c[0], t);
  fq_set(k, c_d.bs2);
  fq_mul(t, v.c[2], k);
  fq_sub(v.c[0], v.c[0], t);
}
// Internal basis only: the F_q^3 product and square keep their five partial
// coefficients double width -- Karatsuba on unreduced 320-bit values, six fqw_mul -- reduce d3 and d4,
// fold them with two more products by p and reduce three times: 8 x 25 + 5 x 30 = 350 multiplier
// operations and 14 double-width additions instead of 8 Montgomery products (440) and 13 modular additions.
//   w^3 = -p w - 1, w^4 = -p w^2 - w:   r0 = d0 - d3,  r1 = d1 - p d3 - d4,  r2 = d2 - p d4
// with d1, d3 < 2 q^2, d2 < 3 q^2, d0, d4 < q^2; the offsets 2 q^2 / q^2 keep every value in (0, 4 q^2),
// below the 2 q R that fqw_redc_os<true> takes (2 q <= R for every q this build accepts).
__device__ __forceinline__ void f3_fold_lazy(F3* r, const FqW& d0, const FqW& d1, const FqW& d2, const FqW& d3,
                                             const FqW& d4) {
  Fq d3r, d4r, p;
  FqW w, t, q1, q2;
  fqw_redc_os<true>(d3r, d3);
  fqw_redc_os<true>(d4r, d4);
  fq_set(p, c_d.pcoef);
#pragma unroll
  for (int k = 0; k < 2 * kNS; k++) { q1.v[k] = c_d.qsqm[0][k]; q2.v[k] = c_d.qsqm[1][k]; }
  fqw_add(w, d0, q2);
  fqw_sub(w, w, d3);
  fqw_redc_os<true>(r->c[0], w);
  fqw_mul(t, p, d3r);
  fqw_add(w, d1, q2);
  fqw_sub(w, w, t);
  fqw_sub(w, w, d4);
  fqw_redc_os<true>(r->c[1], w);
  fqw_mul(t, p, d4r);
  fqw_add(w, d2, q1);
  fqw_sub(w, w, t);
  fqw_redc_os<true>(r->c[2], w);
}
__device__ __noinline__ void f3_mul(F3* r, const F3* x, const F3* y) {
  if (c_d.nice) {
    const Fq x0 = x->c[0], x1 = x->c[1], x2 = x->c[2], y0 = y->c[0], y1 = y->c[1], y2 = y->c[2];
    Fq s, t;
    FqW d0, d1, d2, d3, d4, m1;
    fqw_mul(d0, x0, y0);
    fqw_mul(m1, x1, y1);
    fqw_mul(d4, x2, y2);
    fq_add_nr(s, x0, x1); fq_add_nr(t, y0, y1);
    fqw_mul(d1, s, t); fqw_sub(d1, d1, d0); fqw_sub(d1, d1, m1);
    fq_add_nr(s, x1, x2); fq_add_nr(t, y1, y2);
    fqw_mul(d3, s, t); fqw_sub(d3, d3, m1); fqw_sub(d3, d3, d4);
    fq_add_nr(s, x0, x2); fq_add_nr(t, y0, y2);
    fqw_mul(d2, s, t); fqw_sub(d2, d2, d0); fqw_sub(d2, d2, d4); fqw_add(d2, d2, m1);
    f3_fold_lazy(r, d0, d1, d2, d3, d4);
    return;
  }
  Fq d0, d1, d2, d3, d4, m1, s, t;
  fq_mul(d0, x->c[0], y->c[0]);
  fq_mul(m1, x->c[1], y->c[1]);
  fq_mul(d4, x->c[2], y->c[2]);
  fq_add(s, x->c[0], x->c[1]);
  fq_add(t, y->c[0], y->c[1]);
  fq_mul(d1, s, t);
  fq_sub(d1, d1, d0);
  fq_sub(d1, d1, m1);
  fq_add(s, x->c[1], x->c[2]);
  fq_add(t, y->c[1], y->c[2]);
  fq_mul(d3, s, t);
  fq_sub(d3, d3, m1);
  fq_sub(d3, d3, d4);
  fq_add(s, x->c[0], x->c[2]);
  fq_add(t, y->c[0], y->c[2]);
  fq_mul(d2, s, t);
  fq_sub(d2, d2, d0);
  fq_sub(d2, d2, d4);
  fq_add(d2, d2, m1);
  f3_reduce(r, d0, d1, d2, d3, d4);
}
__device__ __noinline__ void f3_sqr(F3* r, const F3* x) {
  if (c_d.nice) {
    const Fq x0 = x->c[0], x1 = x->c[1], x2 = x->c[2];
    FqW d0, d1, d2, d3, d4, w;
    fqw_mul(d0, x0, x0);
    fqw_mul(d4, x2, x2);
    fqw_mul(d1, x0, x1); fqw_add(d1, d1, d1);
    fqw_mul(d3, x1, x2); fqw_add(d3, d3, d3);
    fqw_mul(d2, x0, x2); fqw_add(d2, d2, d2);
    fqw_mul(w, x1, x1); fqw_add(d2, d2, w);
    f3_fold_lazy(r, d0, d1, d2, d3, d4);
    return;
  }
  Fq d0, d1, d2, d3, d4, t;
  fq_sqr(d0, x->c[0]);
  fq_sqr(d4, x->c[2]);
  fq_mul(d1, x->c[0], x->c[1]);
  fq_dbl(d1, d1);
  fq_mul(d3, x->c[1], x->c[2]);
  fq_dbl(d3, d3);
  fq_mul(d2, x->c[0], x->c[2]);
  fq_dbl(d2, d2);
  fq_sqr(t, x->c[1]);
  fq_add(d2, d2, t);
  f3_reduce(r, d0, d1, d2, d3, d4);
}
// (c0 + c1 x + c2 x^2)^q = c0 + c1 x^q + c2 x^(2q)   (ecc/d_param.c:507-513)
__device__ __forceinline__ void f3_frob(F3& r, const F3& x) {
  F3 t, u;
  f3_set(t, c_d.xpowq);
  f3_scale(t, t, x.c[1]);
  f3_set(u, c_d.xpowq2);
  f3_scale(u, u, x.c[2]);
  f3_add(t, t, u);
  fq_add(r.c[0], t.c[0], x.c[0]);
  r.c[1] = t.c[1];
  r.c[2] = t.c[2];
}
// 1/x = x^q x^(q^2) / N(x)   (the reference runs a polynomial ext-Euclid, arith/poly.c:454-536)
__device__ __noinline__ void f3_inv(F3* r, const F3* x) {
  F3 t, u;
  Fq n;
  f3_frob(t, *x);
  f3_frob(u, t);
  f3_mul(&t, &t, &u);
  f3_mul(&u, &t, x);              // the norm: only coefficient 0 is non-zero
  fq_inv(&n, &u.c[0]);
  f3_scale(*r, t, n);
}

// ---------------------------------------------------------------------------------------------
// F_q^6 = F_q^3[w]/(w^2 - v)
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void f3_mul_v(F3& r, const F3& x) {
  Fq v;
  fq_set(v, c_d.nqr);
  f3_scale(r, x, v);
}
__device__ __noinline__ void f6d_mul(F6D* r, const F6D* x, const F6D* y) {
  F3 t0, t1, t2, s;
  f3_add(t2, x->a, x->b);
  f3_add(s, y->a, y->b);
  f3_mul(&t2, &t2, &s);
  f3_mul(&t0, &x->a, &y->a);
  f3_mul(&t1, &x->b, &y->b);
  f3_sub(t2, t2, t0);
  f3_sub(t2, t2, t1);
  f3_mul_v(t1, t1);
  f3_add(r->a, t0, t1);
  r->b = t2;
}
// (a + b w)^2 = (a + b)(a + v b) - ab - v ab + 2ab w
__device__ __noinline__ void f6d_sqr(F6D* r) {
  F3 t0, t1, t2;
  f3_mul(&t0, &r->a, &r->b);
  f3_mul_v(t1, r->b);
  f3_add(t1, t1, r->a);
  f3_add(t2, r->a, r->b);
  f3_mul(&t2, &t2, &t1);
  f3_sub(t2, t2, t0);
  f3_mul_v(t1, t0);
  f3_sub(r->a, t2, t1);
  f3_add(r->b, t0, t0);
}
__device__ __noinline__ void f6d_inv(F6D* r, const F6D* x) {
  F3 t0, t1;
  f3_sqr(&t0, &x->a);
  f3_sqr(&t1, &x->b);
  f3_mul_v(t1, t1);
  f3_sub(t0, t0, t1);
  f3_inv(&t0, &t0);
  f3_mul(&r->a, &x->a, &t0);
  f3_mul(&t1, &x->b, &t0);
  f3_neg(r->b, t1);
}
__device__ __forceinline__ void f6d_one(F6D& r) {
  f3_zero(r.a);
  f3_zero(r.b);
  fq_one(r.a.c[0]);
}

struct DTower {
  typedef F6D Acc;
  struct Ctx { F3 Qx, Qy; };
  // v *= (a Qx + c) + (b Qy) w   (d_miller_evalfn, ecc/d_param.c:99-111)
  // (own frame for the address-taken temporary: see the stack-discipline note in pairing_f.cuh)
  static __device__ __noinline__ void mul_line(F6D* v, const Fq* a, const Fq* b, const Fq* c,
                                              const Ctx* q) {
    F6D l;
    f3_scale(l.a, q->Qx, *a);
    fq_add(l.a.c[0], l.a.c[0], *c);
    f3_scale(l.b, q->Qy, *b);
    f6d_mul(v, v, &l);
  }
  static __device__ __forceinline__ void sqr(F6D* v) { f6d_sqr(v); }
};

constexpr int kF6DWords = 6 * kNS;

__device__ __forceinline__ void f6d_st_global(uint32_t* g, size_t n, size_t idx, const F6D& v) {
#pragma unroll
  for (int i = 0; i < 3; i++) {
    fq_st_global(g, i, n, idx, v.a.c[i]);
    fq_st_global(g, 3 + i, n, idx, v.b.c[i]);
  }
}
__device__ __forceinline__ void f6d_ld_global(F6D& v, const uint32_t* g, size_t n, size_t idx) {
#pragma unroll
  for (int i = 0; i < 3; i++) {
    fq_ld_global(v.a.c[i], g, i, n, idx);
    fq_ld_global(v.b.c[i], g, 3 + i, n, idx);
  }
}

// P: 40 bytes each (stride1 = 0 shares one P), Q: n x 120 bytes (x: 3 coefficients, y: 3).
// tab != nullptr: the line coefficients of the (one) first argument come from the table (k_cc_pp_init).
template <int BLOCK>
__global__ void __launch_bounds__(BLOCK, (kCCMinBlocks * 128) / BLOCK)
k_d_miller(const uint8_t* __restrict__ P, const uint8_t* __restrict__ Q, uint32_t* __restrict__ mv,
           uint32_t* __restrict__ flag, size_t n, size_t stride1, const uint32_t* __restrict__ tab, size_t rows) {
  size_t idx = (size_t)blockIdx.x * BLOCK + threadIdx.x;
  const bool live = idx < n;      // every thread runs the loop (block-wide barrier inside)
  if (!live) idx = 0;
  Fq xP, yP;
  bool ok;
  if (tab) {
    ok = tab[3 * rows * kNS] != 0;
  } else {
    const uint8_t* p = P + idx * stride1;
    fq_from_wire(xP, p);
    fq_from_wire(yP, p + fq_wb());
    ok = cc_on_curve(xP, yP);
  }
  DTower::Ctx ctx;
  F3 t, u;
  F6D v;
  Fq k;
  const uint8_t* q = Q + idx * (6 * fq_wb());
#pragma unroll
  for (int i = 0; i < 3; i++) {
    fq_from_wire(ctx.Qx.c[i], q + i * fq_wb());
    fq_from_wire(ctx.Qy.c[i], q + (3 + i) * fq_wb());
  }
  f3_to_internal(ctx.Qx);
  f3_to_internal(ctx.Qy);
  // Y^2 == X^3 + (a v^2) X + b v^3 over F_q^3 (ecc/curve.c:57-76; the coefficients lie in F_q, so
  // the identity holds in either basis)
  f3_sqr(&t, &ctx.Qx);
  fq_set(k, c_d.twist_a);
  fq_add(t.c[0], t.c[0], k);
  f3_mul(&t, &t, &ctx.Qx);
  fq_set(k, c_d.twist_b);
  fq_add(t.c[0], t.c[0], k);
  f3_sqr(&u, &ctx.Qy);
  ok = ok && f3_eq(t, u);
  // untwist: Qx / v, Qy / v^2 (ecc/d_param.c:576-582)
  fq_set(k, c_d.nqrinv);
  f3_scale(ctx.Qx, ctx.Qx, k);
  fq_set(k, c_d.nqrinv2);
  f3_scale(ctx.Qy, ctx.Qy, k);
  f6d_one(v);
  if (tab) miller_cc_tab<DTower>(&v, tab, &ctx);
  else miller_cc<DTower>(&v, xP, yP, &ctx);   // off-curve inputs run too (total arithmetic) and are flagged
  if (!live) return;
  if (!ok) f6d_one(v);
  f6d_st_global(mv, n, idx, v);
  flag[idx] = ok ? 1u : 0u;
}

// cc_pairings_affine (ecc/d_param.c:710-736): product of the k Miller values, one final power.
template <int BLOCK>
__global__ void __launch_bounds__(BLOCK, kCCMinBlocks)
k_d_prod(const uint32_t* __restrict__ mv_in, const uint32_t* __restrict__ flag_in,
         uint32_t* __restrict__ mv_out, uint32_t* __restrict__ flag_out, size_t k, size_t n_out,
         size_t n_in) {
  size_t idx = (size_t)blockIdx.x * BLOCK + threadIdx.x;
  if (idx >= n_out) return;
  F6D acc, t;
  f6d_ld_global(acc, mv_in, n_in, idx * k);
  bool ok = flag_in[idx * k] != 0;
  for (size_t j = 1; j < k; j++) {
    f6d_ld_global(t, mv_in, n_in, idx * k + j);
    ok = ok && flag_in[idx * k + j] != 0;
    f6d_mul(&acc, &acc, &t);
  }
  f6d_st_global(mv_out, n_out, idx, acc);
  flag_out[idx] = ok ? 1u : 0u;
}

// the same product over a run table (prod_v.cuh, pbc_b200_prod_pairings_apply_v)
struct F6DProdV {
  using E = F6D;
  // eight limbs (engine_d_wide.cu): at kCCMinBlocks the 128-register cap spills the accumulator
  static constexpr int kMinBlocks = kNS > 5 ? 3 : kCCMinBlocks;
  static __device__ __forceinline__ void ld(E& v, const uint32_t* g, size_t n, size_t i) { f6d_ld_global(v, g, n, i); }
  static __device__ __forceinline__ void st(uint32_t* g, size_t n, size_t i, const E& v) { f6d_st_global(g, n, i, v); }
  static __device__ __forceinline__ void mul(E* r, const E* x, const E* y) { f6d_mul(r, x, y); }
};

// cc_tatepower, k = 6 branch (ecc/d_param.c:505-564) followed by lucas_even (:441-502)
__device__ __noinline__ void f6d_final_exp(F3& out0, F3& out1, F6D& f) {
  F6D e0, e3;
  F3 t1, v0, v1, tmp, two, d;
  f3_frob(e3.a, f.a);
  f3_frob(e3.b, f.b);                  // qpower(1)
  e0.a = f.a;
  f3_neg(e0.b, f.b);                   // conjugate = f^(q^3)
  f6d_mul(&e3, &e3, &e0);
  f3_frob(e0.a, f.a);
  f3_frob(e0.b, f.b);
  f3_neg(e0.b, e0.b);                  // qpower(-1)
  f6d_mul(&e0, &e0, &f);
  f6d_inv(&e0, &e0);
  f6d_mul(&f, &e3, &e0);
  // lucas_even on in = f: t0 = 2, t1 = 2 in0
  f3_zero(two);
  fq_set(two.c[0], c_d.two);
  f3_add(t1, f.a, f.a);
  v0 = two;
  v1 = t1;
  for (int j = (int)c_d.phibits - 1; j >= 0; j--) {
    bool bit = j > 0 && ((c_d.phikonr[j >> 5] >> (j & 31)) & 1u);   // last step: clear branch
    f3_mul(&tmp, &v0, &v1);
    f3_sub(tmp, tmp, t1);
    if (bit) {
      v0 = tmp;
      f3_sqr(&v1, &v1);
      f3_sub(v1, v1, two);
    } else {
      v1 = tmp;
      f3_sqr(&v0, &v0);
      f3_sub(v0, v0, two);
    }
  }
  f3_add(v0, v0, v0);
  f3_mul(&tmp, &t1, &v1);
  f3_sub(tmp, tmp, v0);
  f3_sqr(&d, &t1);
  f3_sub(d, d, two);
  f3_sub(d, d, two);
  f3_inv(&d, &d);
#pragma unroll
  for (int i = 0; i < 3; i++) fq_halve(out0.c[i], v1.c[i]);
  f3_mul(&tmp, &tmp, &d);
  f3_mul(&out1, &tmp, &f.b);
}

// cc_tatepower, k = 6 branch (ecc/d_param.c:505-564) + lucas_even (:441-502).
// out: n x 120 bytes: real half (3 coefficients) then imaginary half.
template <int BLOCK>
__global__ void __launch_bounds__(BLOCK, kCCMinBlocks)
k_d_finalexp(const uint32_t* __restrict__ mv, const uint32_t* __restrict__ flag,
             uint8_t* __restrict__ out, size_t n) {
  size_t idx = (size_t)blockIdx.x * BLOCK + threadIdx.x;
  if (idx >= n) return;
  F6D f;
  F3 out0, out1;
  if (flag[idx]) {
    f6d_ld_global(f, mv, n, idx);
    f6d_final_exp(out0, out1, f);
    f3_to_reference(out0);
    f3_to_reference(out1);
  } else {
    f3_zero(out0);
    f3_zero(out1);
    fq_one(out0.c[0]);
  }
  uint8_t* o = out + idx * (6 * fq_wb());
#pragma unroll 1
  for (int i = 0; i < 3; i++) {
    fq_to_wire(o + i * fq_wb(), out0.c[i]);
    fq_to_wire(o + (3 + i) * fq_wb(), out1.c[i]);
  }
}

__device__ __forceinline__ void f6d_from_wire(F6D& v, const uint8_t* p) {
#pragma unroll 1
  for (int i = 0; i < 3; i++) {
    fq_from_wire(v.a.c[i], p + i * fq_wb());
    fq_from_wire(v.b.c[i], p + (3 + i) * fq_wb());
  }
}
__device__ __forceinline__ void f6d_to_wire(uint8_t* p, const F6D& v) {
#pragma unroll 1
  for (int i = 0; i < 3; i++) {
    fq_to_wire(p + i * fq_wb(), v.a.c[i]);
    fq_to_wire(p + (3 + i) * fq_wb(), v.b.c[i]);
  }
}

// Differential-test hook on GT-sized operands (120 wire bytes): op 0 = a*b, 1 = a^2, 2 = 1/a,
// 3 = cc_tatepower(a), 5 = F_q^3 product of the real halves, 6 = F_q^3 inverse of a's real half.
__global__ void k_d_tower_op(int op, uint8_t* __restrict__ out, const uint8_t* __restrict__ a,
                             const uint8_t* __restrict__ b, size_t n) {
  size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n) return;
  F6D x, y, r;
  f6d_from_wire(x, a + idx * (6 * fq_wb()));
  f6d_from_wire(y, b + idx * (6 * fq_wb()));
  f3_to_internal(x.a); f3_to_internal(x.b); f3_to_internal(y.a); f3_to_internal(y.b);
  switch (op) {
    case 0: f6d_mul(&r, &x, &y); break;
    case 1: r = x; f6d_sqr(&r); break;
    case 2: f6d_inv(&r, &x); break;
    case 3: f6d_final_exp(r.a, r.b, x); break;
    case 5: f3_mul(&r.a, &x.a, &y.a); f3_zero(r.b); break;
    default: f3_inv(&r.a, &x.a); f3_zero(r.b); break;
  }
  f3_to_reference(r.a); f3_to_reference(r.b);
  f6d_to_wire(out + idx * (6 * fq_wb()), r);
}

}  // namespace pbcb200
