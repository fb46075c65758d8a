// pairing_g.cuh -- Type G pairing kernels (Freeman curve, k = 10, 149-bit q: param/g149.param).
//
// Device replacement for ecc/g_param.c: cc_pairing (:541-558), cc_miller_no_denom_affine (:308-411),
// the line evaluation (:86-102), tatepower10 (:471-536), lucas_even (:413-469), on the tower
// F_q^5 = F_q[x]/(x^5 + c4 x^4 + ... + c0) (arith/poly.c polymod_*) and F_q^10 = F_q^5[w]/(w^2 - v).
// The construction is type D's one level up, so the structure of pairing_d.cuh carries over: shared
// inversion-free Miller loop (miller_cc.cuh), Frobenius by the constants x^q .. x^(4q) the reference
// computes itself (:1308-1317), inversions through the norm, Lucas ladder over F_q^5 for the
// 447-bit exponent (q^4 - q^3 + q^2 - q + 1)/r.
// The F_q^5 product is lazily reduced: q has 149 bits against R = 2^160, so all 25 + 20 partial
// products of a multiplication are accumulated as double-width integers and reduced once per
// coefficient (9 reductions instead of 45).
// Wire format: 19 bytes per F_q coordinate (not a multiple of four: byte-wise conversion).
#pragma once
#include "miller_cc.cuh"
#include "prod_v.cuh"

namespace pbcb200 {

constexpr int kWG = 19;            // wire bytes per coordinate for g149

struct F5 { Fq c[5]; };            // c0 + c1 x + ... + c4 x^4
struct F10 { F5 a, b; };           // a + b w,  w^2 = v

struct GConsts {
  uint32_t xpwr[4][5][kNS];        // x^5 .. x^8 modulo the field polynomial (arith/poly.c:1302-1333)
  uint32_t xpowq[4][5][kNS];       // x^q, x^(2q), x^(3q), x^(4q)   (ecc/g_param.c:1308-1317)
  uint32_t nqr[kNS], nqrinv[kNS], nqrinv2[kNS];   // v, 1/v, 1/v^2  (:1322-1325)
  uint32_t twist_a[kNS], twist_b[kNS];            // a v^2, b v^3   (ecc/curve.c:885-892)
  uint32_t two[kNS];
  uint32_t phikonr[16];            // (q^4 - q^3 + q^2 - q + 1)/r, plain integer (:1290-1306)
  uint32_t phibits;
  uint32_t pad[3];
};
__constant__ GConsts c_g;

// ---------------------------------------------------------------------------------------------
// F_q^5
// ---------------------------------------------------------------------------------------------
__device__ __noinline__ void f5_add_call(F5* r, const F5* x, const F5* y) {
#pragma unroll
  for (int i = 0; i < 5; i++) fq_add(r->c[i], x->c[i], y->c[i]);
}
__device__ __noinline__ void f5_sub_call(F5* r, const F5* x, const F5* y) {
#pragma unroll
  for (int i = 0; i < 5; i++) fq_sub(r->c[i], x->c[i], y->c[i]);
}
__device__ __forceinline__ void f5_add(F5& r, const F5& x, const F5& y) { f5_add_call(&r, &x, &y); }
__device__ __forceinline__ void f5_sub(F5& r, const F5& x, const F5& y) { f5_sub_call(&r, &x, &y); }
__device__ __forceinline__ void f5_neg(F5& r, const F5& x) {
#pragma unroll
  for (int i = 0; i < 5; i++) fq_neg(r.c[i], x.c[i]);
}
__device__ __forceinline__ void f5_zero(F5& r) {
#pragma unroll
  for (int i = 0; i < 5; i++) fq_zero(r.c[i]);
}
__device__ __forceinline__ bool f5_eq(const F5& x, const F5& y) {
  bool e = true;
#pragma unroll
  for (int i = 0; i < 5; i++) e = e && fq_eq(x.c[i], y.c[i]);
  return e;
}
// multiplication by an element of F_q
// (the scalar travels by value: an inlined helper must not take the address of one of its own
// locals -- stack discipline note in pairing_f.cuh)
__device__ __noinline__ void f5_scale_call(F5* r, const F5* x, Fq k) {
#pragma unroll 1
  for (int i = 0; i < 5; i++) fq_mul(r->c[i], x->c[i], k);
}
__device__ __forceinline__ void f5_scale(F5& r, const F5& x, const Fq& k) { f5_scale_call(&r, &x, k); }

// x y: schoolbook, the nine coefficients of the product accumulated double-width, the four high
// ones reduced and folded in with the rows x^5 .. x^8, one reduction per output coefficient.
// Bounds: at most 25 + 20 products below q^2 each < 2^298; 45 q^2 < 2^304 < q R (2^309).
__device__ __noinline__ void f5_mul(F5* r, const F5* x, const F5* y) {
  FqW d[9], t;
  Fq hi[4], k;
  F5 o;
#pragma unroll 1
  for (int s = 0; s < 9; s++) {
    bool first = true;
#pragma unroll 1
    for (int i = (s < 5 ? 0 : s - 4); i <= (s < 5 ? s : 4); i++) {
      t = fq_mulw_call(x->c[i], y->c[s - i]);
      if (first) { d[s] = t; first = false; } else fqw_add(d[s], d[s], t);
    }
  }
#pragma unroll 1
  for (int s = 0; s < 4; s++) hi[s] = fq_redc_call(d[5 + s]);
#pragma unroll 1
  for (int i = 0; i < 5; i++) {
#pragma unroll 1
    for (int s = 0; s < 4; s++) {
      fq_set(k, c_g.xpwr[s][i]);
      t = fq_mulw_call(hi[s], k);
      fqw_add(d[i], d[i], t);
    }
    o.c[i] = fq_redc_call(d[i]);
  }
  *r = o;
}
// x^2 = x x: a dedicated squaring with the ten cross products doubled (15 + 20 products but more code) did not
// pay here (DESIGN.md §3.8)
__device__ __forceinline__ void f5_sqr(F5* r, const F5* x) { f5_mul(r, x, x); }

// (sum c_i x^i)^q = c0 + sum_{i >= 1} c_i x^(iq)   (ecc/g_param.c:483-493)
__device__ __noinline__ void f5_frob(F5* r, const F5* x) {
  FqW acc[5], t;
  Fq k, xc[5];
#pragma unroll
  for (int i = 0; i < 5; i++) xc[i] = x->c[i];
#pragma unroll 1
  for (int j = 0; j < 5; j++) {
#pragma unroll 1
    for (int i = 1; i < 5; i++) {
      fq_set(k, c_g.xpowq[i - 1][j]);
      t = fq_mulw_call(xc[i], k);
      if (i == 1) acc[j] = t; else fqw_add(acc[j], acc[j], t);
    }
    r->c[j] = fq_redc_call(acc[j]);
  }
  fq_add(r->c[0], r->c[0], xc[0]);
}
// 1/x = x^q x^(q^2) x^(q^3) x^(q^4) / N(x)   (the reference runs a polynomial ext-Euclid)
__device__ __noinline__ void f5_inv(F5* r, const F5* x) {
  F5 f1, f2, t;
  Fq n;
  f5_frob(&f1, x);
  f5_frob(&f2, &f1);
  f5_mul(&t, &f1, &f2);
  f5_frob(&f1, &f2);
  f5_mul(&t, &t, &f1);
  f5_frob(&f2, &f1);
  f5_mul(&t, &t, &f2);
  f5_mul(&f1, &t, x);             // the norm: only coefficient 0 is non-zero
  fq_inv(&n, &f1.c[0]);
  f5_scale(*r, t, n);
}

// ---------------------------------------------------------------------------------------------
// F_q^10 = F_q^5[w]/(w^2 - v)
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void f5_mul_v(F5& r, const F5& x) {
  Fq v;
  fq_set(v, c_g.nqr);
  f5_scale(r, x, v);
}
__device__ __noinline__ void f10_mul(F10* r, const F10* x, const F10* y) {
  F5 t0, t1, t2, s;
  f5_add(t2, x->a, x->b);
  f5_add(s, y->a, y->b);
  f5_mul(&t2, &t2, &s);
  f5_mul(&t0, &x->a, &y->a);
  f5_mul(&t1, &x->b, &y->b);
  f5_sub(t2, t2, t0);
  f5_sub(t2, t2, t1);
  f5_mul_v(t1, t1);
  f5_add(r->a, t0, t1);
  r->b = t2;
}
__device__ __noinline__ void f10_sqr(F10* r) {
  F5 t0, t1, t2;
  f5_mul(&t0, &r->a, &r->b);
  f5_mul_v(t1, r->b);
  f5_add(t1, t1, r->a);
  f5_add(t2, r->a, r->b);
  f5_mul(&t2, &t2, &t1);
  f5_sub(t2, t2, t0);
  f5_mul_v(t1, t0);
  f5_sub(r->a, t2, t1);
  f5_add(r->b, t0, t0);
}
__device__ __noinline__ void f10_inv(F10* r, const F10* x) {
  F5 t0, t1;
  f5_sqr(&t0, &x->a);
  f5_sqr(&t1, &x->b);
  f5_mul_v(t1, t1);
  f5_sub(t0, t0, t1);
  f5_inv(&t0, &t0);
  f5_mul(&r->a, &x->a, &t0);
  f5_mul(&t1, &x->b, &t0);
  f5_neg(r->b, t1);
}
__device__ __forceinline__ void f10_one(F10& r) {
  f5_zero(r.a);
  f5_zero(r.b);
  fq_one(r.a.c[0]);
}

struct GTower {
  typedef F10 Acc;
  struct Ctx { F5 Qx, Qy; };
  // v *= (a Qx + c) + (b Qy) w   (ecc/g_param.c:86-102)
  static __device__ __noinline__ void mul_line(F10* v, const Fq* a, const Fq* b, const Fq* c,
                                              const Ctx* q) {
    F10 l;
    f5_scale(l.a, q->Qx, *a);
    fq_add(l.a.c[0], l.a.c[0], *c);
    f5_scale(l.b, q->Qy, *b);
    f10_mul(v, v, &l);
  }
  static __device__ __forceinline__ void sqr(F10* v) { f10_sqr(v); }
};

constexpr int kF10Words = 10 * kNS;

__device__ __forceinline__ void f10_st_global(uint32_t* g, size_t n, size_t idx, const F10& v) {
#pragma unroll
  for (int i = 0; i < 5; i++) {
    fq_st_global(g, i, n, idx, v.a.c[i]);
    fq_st_global(g, 5 + i, n, idx, v.b.c[i]);
  }
}
__device__ __forceinline__ void f10_ld_global(F10& v, const uint32_t* g, size_t n, size_t idx) {
#pragma unroll
  for (int i = 0; i < 5; i++) {
    fq_ld_global(v.a.c[i], g, i, n, idx);
    fq_ld_global(v.b.c[i], g, 5 + i, n, idx);
  }
}
__device__ __forceinline__ void f10_from_wire(F10& v, const uint8_t* p) {
#pragma unroll 1
  for (int i = 0; i < 5; i++) {
    fq_from_wire_b<kWG>(v.a.c[i], p + i * kWG);
    fq_from_wire_b<kWG>(v.b.c[i], p + (5 + i) * kWG);
  }
}
__device__ __forceinline__ void f10_to_wire(uint8_t* p, const F10& v) {
#pragma unroll 1
  for (int i = 0; i < 5; i++) {
    fq_to_wire_b<kWG>(p + i * kWG, v.a.c[i]);
    fq_to_wire_b<kWG>(p + (5 + i) * kWG, v.b.c[i]);
  }
}

// P: 38 bytes each (stride1 = 0 shares one P), Q: n x 190 bytes (x: 5 coefficients, y: 5).
template <int BLOCK>
__global__ void __launch_bounds__(BLOCK, (kCCMinBlocks * 128) / BLOCK)
k_g_miller(const uint8_t* __restrict__ P, const uint8_t* __restrict__ Q, uint32_t* __restrict__ mv,
           uint32_t* __restrict__ flag, size_t n, size_t stride1, const uint32_t* __restrict__ tab, size_t rows) {
  size_t idx = (size_t)blockIdx.x * BLOCK + threadIdx.x;
  const bool live = idx < n;      // every thread runs the loop (block-wide barrier inside)
  if (!live) idx = 0;
  Fq xP, yP, k;
  bool ok;
  if (tab) {
    ok = tab[3 * rows * kNS] != 0;             // fixed first argument: lines from the table (k_cc_pp_init)
  } else {
    const uint8_t* p = P + idx * stride1;
    fq_from_wire_b<kWG>(xP, p);
    fq_from_wire_b<kWG>(yP, p + kWG);
    ok = cc_on_curve(xP, yP);
  }
  GTower::Ctx ctx;
  F5 t, u;
  F10 v;
  const uint8_t* q = Q + idx * (10 * kWG);
#pragma unroll 1
  for (int i = 0; i < 5; i++) {
    fq_from_wire_b<kWG>(ctx.Qx.c[i], q + i * kWG);
    fq_from_wire_b<kWG>(ctx.Qy.c[i], q + (5 + i) * kWG);
  }
  // Y^2 == X^3 + (a v^2) X + b v^3 over F_q^5 (ecc/curve.c:57-76)
  f5_sqr(&t, &ctx.Qx);
  fq_set(k, c_g.twist_a);
  fq_add(t.c[0], t.c[0], k);
  f5_mul(&t, &t, &ctx.Qx);
  fq_set(k, c_g.twist_b);
  fq_add(t.c[0], t.c[0], k);
  f5_sqr(&u, &ctx.Qy);
  ok = ok && f5_eq(t, u);
  // untwist: Qx / v, Qy / v^2 (ecc/g_param.c:549-553)
  fq_set(k, c_g.nqrinv);
  f5_scale(ctx.Qx, ctx.Qx, k);
  fq_set(k, c_g.nqrinv2);
  f5_scale(ctx.Qy, ctx.Qy, k);
  f10_one(v);
  if (tab) miller_cc_tab<GTower>(&v, tab, &ctx);
  else miller_cc<GTower>(&v, xP, yP, &ctx);   // off-curve inputs run too (total arithmetic) and are flagged
  if (!live) return;
  if (!ok) f10_one(v);
  f10_st_global(mv, n, idx, v);
  flag[idx] = ok ? 1u : 0u;
}

// generic_prod_pairings (ecc/pairing.c:35-46): product of the k Miller values, one final power
template <int BLOCK>
__global__ void __launch_bounds__(BLOCK, kCCMinBlocks)
k_g_prod(const uint32_t* __restrict__ mv_in, const uint32_t* __restrict__ flag_in,
         uint32_t* __restrict__ mv_out, uint32_t* __restrict__ flag_out, size_t k, size_t n_out,
         size_t n_in) {
  size_t idx = (size_t)blockIdx.x * BLOCK + threadIdx.x;
  if (idx >= n_out) return;
  F10 acc, t;
  f10_ld_global(acc, mv_in, n_in, idx * k);
  bool ok = flag_in[idx * k] != 0;
  for (size_t j = 1; j < k; j++) {
    f10_ld_global(t, mv_in, n_in, idx * k + j);
    ok = ok && flag_in[idx * k + j] != 0;
    f10_mul(&acc, &acc, &t);
  }
  f10_st_global(mv_out, n_out, idx, acc);
  flag_out[idx] = ok ? 1u : 0u;
}

// the same product over a run table (prod_v.cuh, pbc_b200_prod_pairings_apply_v)
struct F10ProdV {
  using E = F10;
  static constexpr int kMinBlocks = kCCMinBlocks;
  static __device__ __forceinline__ void ld(E& v, const uint32_t* g, size_t n, size_t i) { f10_ld_global(v, g, n, i); }
  static __device__ __forceinline__ void st(uint32_t* g, size_t n, size_t i, const E& v) { f10_st_global(g, n, i, v); }
  static __device__ __forceinline__ void mul(E* r, const E* x, const E* y) { f10_mul(r, x, y); }
};

// tatepower10 (ecc/g_param.c:471-536) followed by lucas_even (:413-469)
__device__ __noinline__ void f10_final_exp(F5& out0, F5& out1, F10& f) {
  F10 e0, e3;
  F5 t1, v0, v1, tmp, two, d;
  f5_frob(&e3.a, &f.a);
  f5_frob(&e3.b, &f.b);                // qpower(1)
  e0.a = f.a;
  f5_neg(e0.b, f.b);                   // conjugate = f^(q^5)
  f10_mul(&e3, &e3, &e0);
  f5_frob(&e0.a, &f.a);
  f5_frob(&e0.b, &f.b);
  f5_neg(e0.b, e0.b);                  // qpower(-1)
  f10_mul(&e0, &e0, &f);
  f10_inv(&e0, &e0);
  f10_mul(&f, &e3, &e0);
  // lucas_even on in = f: t0 = 2, t1 = 2 in0
  f5_zero(two);
  fq_set(two.c[0], c_g.two);
  f5_add(t1, f.a, f.a);
  v0 = two;
  v1 = t1;
  for (int j = (int)c_g.phibits - 1; j >= 0; j--) {
    bool bit = j > 0 && ((c_g.phikonr[j >> 5] >> (j & 31)) & 1u);   // last step: clear branch
    f5_mul(&tmp, &v0, &v1);
    f5_sub(tmp, tmp, t1);
    if (bit) {
      v0 = tmp;
      f5_sqr(&v1, &v1);
      f5_sub(v1, v1, two);
    } else {
      v1 = tmp;
      f5_sqr(&v0, &v0);
      f5_sub(v0, v0, two);
    }
  }
  f5_add(v0, v0, v0);
  f5_mul(&tmp, &t1, &v1);
  f5_sub(tmp, tmp, v0);
  f5_sqr(&d, &t1);
  f5_sub(d, d, two);
  f5_sub(d, d, two);
  f5_inv(&d, &d);
#pragma unroll
  for (int i = 0; i < 5; i++) fq_halve(out0.c[i], v1.c[i]);
  f5_mul(&tmp, &tmp, &d);
  f5_mul(&out1, &tmp, &f.b);
}

// out: n x 190 bytes: real half (5 coefficients) then imaginary half
template <int BLOCK>
__global__ void __launch_bounds__(BLOCK, (kCCMinBlocks * 128) / BLOCK)
k_g_finalexp(const uint32_t* __restrict__ mv, const uint32_t* __restrict__ flag,
             uint8_t* __restrict__ out, size_t n) {
  size_t idx = (size_t)blockIdx.x * BLOCK + threadIdx.x;
  const bool live = idx < n;             // padding threads run on entry 0 and store nothing
  if (!live) idx = 0;
  F10 f;
  F5 out0, out1;
  const bool ok = flag[idx] != 0;
  // flagged-off entries power 1
  f10_ld_global(f, mv, n, idx);
  if (!ok) f10_one(f);
  f10_final_exp(out0, out1, f);
  if (!live) return;
  if (!ok) {
    f5_zero(out0);
    f5_zero(out1);
    fq_one(out0.c[0]);
  }
  uint8_t* o = out + idx * (10 * kWG);
#pragma unroll 1
  for (int i = 0; i < 5; i++) {
    fq_to_wire_b<kWG>(o + i * kWG, out0.c[i]);
    fq_to_wire_b<kWG>(o + (5 + i) * kWG, out1.c[i]);
  }
}

// Differential-test hook on GT-sized operands (190 wire bytes): op 0 = a*b, 1 = a^2, 2 = 1/a,
// 3 = tatepower10(a), 5 = F_q^5 product of the real halves, 6 = F_q^5 inverse of a's real half.
__global__ void k_g_tower_op(int op, uint8_t* __restrict__ out, const uint8_t* __restrict__ a,
                             const uint8_t* __restrict__ b, size_t n) {
  size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const bool live = idx < n;
  if (!live) idx = 0;
  F10 x, y, r;
  f10_from_wire(x, a + idx * (10 * kWG));
  f10_from_wire(y, b + idx * (10 * kWG));
  switch (op) {
    case 0: f10_mul(&r, &x, &y); break;
    case 1: r = x; f10_sqr(&r); break;
    case 2: f10_inv(&r, &x); break;
    case 3: f10_final_exp(r.a, r.b, x); break;
    case 5: f5_mul(&r.a, &x.a, &y.a); f5_zero(r.b); break;
    default: f5_inv(&r.a, &x.a); f5_zero(r.b); break;
  }
  if (!live) return;
  f10_to_wire(out + idx * (10 * kWG), r);
}

}  // namespace pbcb200
