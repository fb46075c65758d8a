// group_cc.cuh -- the operations either side of the Type F / Type D pairings (SURVEY 8f ranks 2, 3):
//   element_pow_zn on G1 = E(F_q)  (ecc/curve.c:455-482 -> arith/field.c:113-126 windowed power over
//       curve_double / curve_mul, one inversion per affine operation)
//   element_pow_zn on GT (ecc/pairing.c:199-231 -> windowed power in F_q^12 / F_q^6)
// Same values, different route: left-to-right double-and-add on Jacobian coordinates (the formulas
// of miller_cc.cuh without the lines) with one Fermat inversion at the end, and square-and-multiply
// on the tower routines of pairing_f.cuh / pairing_d.cuh.  G2 (the twists over F_q^2 for type f, F_q^3
// for type d; ecc/f_param.c:367-378, ecc/d_param.c:1060-1070) runs the same double-and-add on the
// tower's field routines through a small policy struct.
#pragma once
#include "group_a.cuh"
#include "pairing_d.cuh"
#if !PBC_FQ_WIDE
#include "pairing_f.cuh"
#include "pairing_g.cuh"
#endif

namespace pbcb200 {

// out[i] = k[i] * in[i] on y^2 = x^3 + A x + B over the five-limb field.  O -> zero bytes.
template <int BLOCK, int W>
__global__ void __launch_bounds__(BLOCK, kCCMinBlocks)
k_cc_g1_mul(const uint8_t* __restrict__ P, const uint8_t* __restrict__ K, uint8_t* __restrict__ out,
            size_t n) {
  size_t idx = (size_t)blockIdx.x * BLOCK + threadIdx.x;
  if (idx >= n) return;
  Fq xP, yP, X, Y, Z, Z2, M, Y2, t, u, H, R;
  fq_from_wire_w<W>(xP, P + idx * (2 * wire_w<W>()));
  fq_from_wire_w<W>(yP, P + idx * (2 * wire_w<W>()) + wire_w<W>());
  bool ok = cc_on_curve(xP, yP);
  uint32_t k[kZW];
  zr_from_wire(k, K + idx * c_zr.zlen);
  int top = zr_top_bit(k);
  X = xP;
  Y = yP;
  fq_one(Z);
  auto dbl = [&]() {                   // V = 2V
    fq_sqr(Z2, Z);
    fq_sqr(t, X);
    fq_dbl(M, t);
    fq_add(M, M, t);
    if (!c_cc.a_is_zero) {
      fq_sqr(u, Z2);
      fq_set(t, c_cc.A);
      fq_mul(u, u, t);
      fq_add(M, M, u);
    }
    fq_sqr(Y2, Y);
    fq_mul(u, Y, Z);
    fq_dbl(Z, u);
    fq_mul(t, X, Y2);
    fq_dbl(t, t);
    fq_dbl(t, t);
    fq_sqr(X, M);
    fq_sub(X, X, t);
    fq_sub(X, X, t);
    fq_sqr(Y2, Y2);
    fq_dbl(Y2, Y2);
    fq_dbl(Y2, Y2);
    fq_dbl(Y2, Y2);
    fq_sub(t, t, X);
    fq_mul(Y, M, t);
    fq_sub(Y, Y, Y2);
  };
  for (int j = top - 1; j >= 0; j--) {
    dbl();
    if ((k[j >> 5] >> (j & 31)) & 1u) {
      // V = V + P (mixed; V = O, V = P and V = -P as in g_add_affine, group_a.cuh)
      fq_sqr(Z2, Z);
      fq_mul(t, Z2, Z);
      fq_mul(H, xP, Z2);
      fq_sub(H, H, X);
      fq_mul(R, yP, t);
      fq_sub(R, R, Y);
      if (fq_is_zero(H) || fq_is_zero(Z)) {
        if (fq_is_zero(Z)) { X = xP; Y = yP; fq_one(Z); }
        else if (fq_is_zero(R)) dbl();
        else fq_zero(Z);
        continue;
      }
      fq_mul(Z, H, Z);
      fq_sqr(t, H);
      fq_mul(u, t, H);
      fq_mul(t, t, X);
      fq_sqr(X, R);
      fq_sub(X, X, u);
      fq_sub(X, X, t);
      fq_sub(X, X, t);
      fq_sub(t, t, X);
      fq_mul(t, t, R);
      fq_mul(u, u, Y);
      fq_sub(Y, t, u);
    }
  }
  bool inf = !ok || top < 0 || fq_is_zero(Z);
  fq_inv(&t, &Z);
  fq_sqr(u, t);
  fq_mul(X, X, u);
  fq_mul(u, u, t);
  fq_mul(Y, Y, u);
  if (inf) { fq_zero(X); fq_zero(Y); }
  fq_to_wire_w<W>(out + idx * (2 * wire_w<W>()), X);
  fq_to_wire_w<W>(out + idx * (2 * wire_w<W>()) + wire_w<W>(), Y);
}

#if PBC_FQ_WIDE
// Tonelli-Shanks (q = 1 mod 8, the wide instance; HashConsts::sqrt_mode 3):  q - 1 = 2^s Q, Q odd,
// x = t^((Q-1)/2), y = t x, b = y x = t^Q, c = z^Q (z a non-residue).  While b != 1: the least i with
// b^(2^i) = 1 (none below m: t is not a square, y is left as it is and fails the caller's y^2 == t),
// w = c^(2^(m-i-1)), y = y w, c = w^2, b = b c, m = i.  y is then a root of t; which of the two does not
// matter, the callers normalise its sign as the reference does (ecc/curve.c).
__device__ __noinline__ void fq_sqrt_ts(Fq* out, const Fq* tp) {
  Fq t = *tp, x, y, b, c, w, one;
  fq_one(one);
  x = t;
  for (int j = (int)c_hash.expbits - 2; j >= 0; j--) {
    fq_sqr(x, x);
    if ((c_hash.exp[j >> 5] >> (j & 31)) & 1u) fq_mul(x, x, t);
  }
  if (c_hash.expbits == 0) x = one;
  fq_mul(y, t, x);
  fq_mul(b, y, x);
  fq_set(c, c_fqx.ts_c);
  int m = (int)c_fqx.ts_s;
  for (int it = 0; it < 64 && !fq_eq(b, one); it++) {
    int i = 1;
    fq_sqr(w, b);
    while (i < m && !fq_eq(w, one)) { fq_sqr(w, w); i++; }
    if (i >= m) break;
    w = c;
    for (int j = 0; j < m - i - 1; j++) fq_sqr(w, w);
    fq_mul(y, y, w);
    fq_sqr(c, w);
    fq_mul(b, b, c);
    m = i;
  }
  *out = y;
}
#endif

// element_from_hash on G1 for the five-limb fields (ecc/curve.c:455-482): try-and-increment, the odd
// square root (q = 3 mod 4: t^((q+1)/4); q = 5 mod 8: Atkin's b = (2t)^((q-5)/8), i = 2 t b^2,
// root = t b (i - 1)), then the cofactor multiple (d159: h = 3; type f: none).
template <int BLOCK, int W>
__global__ void __launch_bounds__(BLOCK, kCCMinBlocks)
k_cc_g1_from_hash(const uint8_t* __restrict__ data, int len, uint8_t* __restrict__ out, size_t n) {
  size_t idx = (size_t)blockIdx.x * BLOCK + threadIdx.x;
  if (idx >= n) return;
  Fq x, y, t, b, u, w, A, B, one, X, Y, Z, Z2, M, Y2, H, R;
  uint32_t xw[kNS];
  hash_to_words<kNS>(xw, data + idx * (size_t)len, len);
  fq_set(x, xw);
  fq_set(t, c_fp.r2);
  fq_mul(x, x, t);
  fq_set(A, c_cc.A);
  fq_set(B, c_cc.B);
  fq_one(one);
  for (int tries = 0; tries < 64; tries++) {
    fq_sqr(t, x);
    fq_add(t, t, A);
    fq_mul(t, t, x);
    fq_add(t, t, B);                       // t = x^3 + A x + B
#if PBC_FQ_WIDE
    if (c_hash.sqrt_mode == 3) {
      fq_sqrt_ts(&y, &t);
      fq_sqr(w, y);
      if (fq_eq(w, t)) break;
      fq_sqr(x, x);
      fq_add(x, x, one);
      continue;
    }
#endif
    if (c_hash.sqrt_mode == 1) u = t; else fq_dbl(u, t);
    b = u;
    for (int j = (int)c_hash.expbits - 2; j >= 0; j--) {
      fq_sqr(b, b);
      if ((c_hash.exp[j >> 5] >> (j & 31)) & 1u) fq_mul(b, b, u);
    }
    if (c_hash.expbits == 0) b = one;
    if (c_hash.sqrt_mode == 1) {
      y = b;
    } else {
      fq_sqr(w, b);
      fq_mul(w, w, u);                     // i = 2 t b^2
      fq_sub(w, w, one);
      fq_mul(y, t, b);
      fq_mul(y, y, w);                     // t b (i - 1)
    }
    fq_sqr(w, y);
    if (fq_eq(w, t)) break;
    fq_sqr(x, x);
    fq_add(x, x, one);
  }
  {
    uint32_t c[kNS], o1[kNS] = {1};
    mont_mul_ps<kNS, false>(c, y.v, o1);
    if (!(c[0] & 1u) && !fp_is_zero<kNS>(c)) fq_neg(y, y);
  }
  if (c_hash.cofbits <= 1) {               // cofactor 1: the point itself
    fq_to_wire_w<W>(out + idx * (2 * wire_w<W>()), x);
    fq_to_wire_w<W>(out + idx * (2 * wire_w<W>()) + wire_w<W>(), y);
    return;
  }
  X = x;
  Y = y;
  fq_one(Z);
  for (int j = (int)c_hash.cofbits - 2; j >= 0; j--) {
    fq_sqr(Z2, Z);
    fq_sqr(t, X);
    fq_dbl(M, t);
    fq_add(M, M, t);
    if (!c_cc.a_is_zero) {
      fq_sqr(u, Z2);
      fq_mul(u, u, A);
      fq_add(M, M, u);
    }
    fq_sqr(Y2, Y);
    fq_mul(u, Y, Z);
    fq_dbl(Z, u);
    fq_mul(t, X, Y2);
    fq_dbl(t, t);
    fq_dbl(t, t);
    fq_sqr(X, M);
    fq_sub(X, X, t);
    fq_sub(X, X, t);
    fq_sqr(Y2, Y2);
    fq_dbl(Y2, Y2);
    fq_dbl(Y2, Y2);
    fq_dbl(Y2, Y2);
    fq_sub(t, t, X);
    fq_mul(Y, M, t);
    fq_sub(Y, Y, Y2);
    if ((c_hash.cofac[j >> 5] >> (j & 31)) & 1u) {
      fq_sqr(Z2, Z);
      fq_mul(t, Z2, Z);
      fq_mul(H, x, Z2);
      fq_sub(H, H, X);
      fq_mul(R, y, t);
      fq_sub(R, R, Y);
      fq_mul(Z, H, Z);
      fq_sqr(t, H);
      fq_mul(u, t, H);
      fq_mul(t, t, X);
      fq_sqr(X, R);
      fq_sub(X, X, u);
      fq_sub(X, X, t);
      fq_sub(X, X, t);
      fq_sub(t, t, X);
      fq_mul(t, t, R);
      fq_mul(u, u, Y);
      fq_sub(Y, t, u);
    }
  }
  bool inf = fq_is_zero(Z);
  fq_inv(&t, &Z);
  fq_sqr(u, t);
  fq_mul(X, X, u);
  fq_mul(u, u, t);
  fq_mul(Y, Y, u);
  if (inf) { fq_zero(X); fq_zero(Y); }
  fq_to_wire_w<W>(out + idx * (2 * wire_w<W>()), X);
  fq_to_wire_w<W>(out + idx * (2 * wire_w<W>()) + wire_w<W>(), Y);
}

// element_from_bytes_compressed on G1 for the five-limb fields (ecc/curve.c:799-813): x (20 bytes) ||
// sign byte -> x || y.  No square root -> zero bytes.
template <int BLOCK, int W>
__global__ void __launch_bounds__(BLOCK, kCCMinBlocks)
k_cc_g1_decompress(const uint8_t* __restrict__ in, uint8_t* __restrict__ out, size_t n) {
  size_t idx = (size_t)blockIdx.x * BLOCK + threadIdx.x;
  if (idx >= n) return;
  const uint8_t* p = in + idx * (wire_w<W>() + 1);
  Fq x, y, t, b, u, w, one, k;
  fq_from_wire_b<W>(x, p);             // items are W + 1 bytes apart: byte loads
  fq_one(one);
  fq_sqr(t, x);
  fq_set(k, c_cc.A);
  fq_add(t, t, k);
  fq_mul(t, t, x);
  fq_set(k, c_cc.B);
  fq_add(t, t, k);
#if PBC_FQ_WIDE
  if (c_hash.sqrt_mode == 3) fq_sqrt_ts(&y, &t); else {
#endif
  if (c_hash.sqrt_mode == 1) u = t; else fq_dbl(u, t);
  b = u;
  for (int j = (int)c_hash.expbits - 2; j >= 0; j--) {
    fq_sqr(b, b);
    if ((c_hash.exp[j >> 5] >> (j & 31)) & 1u) fq_mul(b, b, u);
  }
  if (c_hash.expbits == 0) b = one;
  if (c_hash.sqrt_mode == 1) {
    y = b;
  } else {
    fq_sqr(w, b);
    fq_mul(w, w, u);
    fq_sub(w, w, one);
    fq_mul(y, t, b);
    fq_mul(y, y, w);
  }
#if PBC_FQ_WIDE
  }
#endif
  fq_sqr(w, y);
  bool ok = fq_eq(w, t);
  uint32_t c[kNS], o1[kNS] = {1};
  mont_mul_ps<kNS, false>(c, y.v, o1);
  bool odd = (c[0] & 1u) != 0, want_odd = p[wire_w<W>()] != 0;
  if (odd != want_odd && !fp_is_zero<kNS>(c)) fq_neg(y, y);
  if (!ok) { fq_zero(x); fq_zero(y); }
  fq_to_wire_w<W>(out + idx * (2 * wire_w<W>()), x);
  fq_to_wire_w<W>(out + idx * (2 * wire_w<W>()) + wire_w<W>(), y);
}

// ---------------------------------------------------------------------------------------------
// G2: y^2 = x^3 + a' x + b' over K = F_q^2 (type f, a' = 0) or F_q^3 (type d).  KF supplies the
// field: struct El; mul/sqr/inv on pointers (the tower's out-of-line routines), add/sub/dbl inline,
// wire <-> basis-in-use conversion, and the curve constants.
// ---------------------------------------------------------------------------------------------

// element_from_hash and compressed points on G2 (curve_from_hash / element_from_bytes_compressed on the
// twist): the square-root data of K, derived at init (engine.cu, fill_g2_hash)
template <int NS>
struct G2HashConstsT {
  uint32_t exp[24];      // type f: (q + 1)/4, roots in F_q.  Types d, g (Q = q^k, k odd): mode 1 (Q + 1)/4,
                         // mode 2 (Q - 5)/8 (Atkin), mode 3 (Qo - 1)/2 with Q - 1 = 2^s Qo (Tonelli-Shanks)
  uint32_t leg[8];       // (q - 1)/2: the Legendre symbol of a norm
  uint32_t expbits, legbits, mode, ts_s;
  uint32_t ts_c[NS];     // mode 3: z^Qo for a non-residue z of F_q (it lies in F_q), Montgomery form
  uint32_t isq[NS];      // type f: i^2 of the basis in use (-1 internal, beta reference), Montgomery form
  uint32_t isq_inv[NS];
};
typedef G2HashConstsT<kNS> G2HashConsts;
__constant__ G2HashConsts c_g2h;

// a^e, e a plain little-endian exponent of `bits` bits (a^0 = 1)
__device__ __noinline__ void fq_pow_words(Fq* r, const Fq* a, const uint32_t* e, int bits) {
  Fq x = *a, acc = *a;
  for (int j = bits - 2; j >= 0; j--) {
    fq_sqr(acc, acc);
    if ((e[j >> 5] >> (j & 31)) & 1u) fq_mul(acc, acc, x);
  }
  if (bits == 0) fq_one(acc);
  *r = acc;
}
// n^((q - 1)/2) == 1: n is a non-zero square of F_q.  The helpers below whose locals have their
// address taken are out of line with those locals at function scope: inlined into the G2 kernels, such
// a local of KF5::is_sqr was seen to share its stack slot with the kernel's live t (stack discipline
// note in pairing_f.cuh)
__device__ __noinline__ bool fq_is_nonzero_sqr(Fq n) {
  Fq l, one;
  fq_pow_words(&l, &n, c_g2h.leg, (int)c_g2h.legbits);
  fq_one(one);
  return fq_eq(l, one);
}
// fp_sgn_odd (arith/montfp.c:460-472): 0 for zero, 1 for an odd canonical residue, -1 for an even one
__device__ __forceinline__ int fq_sgn(const Fq& a) {
  uint32_t c[kNS], o1[kNS] = {1};
  mont_mul_ps<kNS, false>(c, a.v, o1);
  if (fp_is_zero<kNS>(c)) return 0;
  return (c[0] & 1u) ? 1 : -1;
}
// K^* of odd degree k has a square root method by q mod 8 (Q = q^k = q mod 8); t a non-zero square
// (out of line, locals at function scope: the stack discipline note in pairing_f.cuh)
template <class KF>
__device__ __noinline__ void kf_pow(typename KF::El* r, const typename KF::El* a, const uint32_t* e, int bits) {
  typename KF::El x = *a, acc = *a;
  for (int j = bits - 2; j >= 0; j--) {
    KF::sqr(&acc, &acc);
    if ((e[j >> 5] >> (j & 31)) & 1u) KF::mul(&acc, &acc, &x);
  }
  if (bits == 0) KF::one(acc);
  *r = acc;
}
template <class KF>
__device__ __noinline__ void kf_sqrt_odd(typename KF::El* yp, const typename KF::El* tp) {
  typedef typename KF::El El;
  El y, t = *tp, b, w, u, one;
  const int mode = (int)c_g2h.mode, bits = (int)c_g2h.expbits;
  if (mode == 1) {                       // t^((Q + 1)/4)
    kf_pow<KF>(yp, &t, c_g2h.exp, bits);
    return;
  }
  if (mode == 2) {                       // Atkin: b = (2t)^((Q - 5)/8), i = 2 t b^2, root = t b (i - 1)
    KF::add(u, t, t);
    kf_pow<KF>(&b, &u, c_g2h.exp, bits);
    KF::sqr(&w, &b);
    KF::mul(&w, &w, &u);
    KF::one(one);
    KF::sub(w, w, one);
    KF::mul(&y, &t, &b);
    KF::mul(yp, &y, &w);
    return;
  }
  // Tonelli-Shanks: x = t^((Qo - 1)/2), y = t x, b = y x = t^Qo.  q^(k-1) + .. + q + 1 is odd, so the
  // 2-Sylow subgroup of K^* is that of F_q^*: b, c and every w below lie in F_q (coefficient 0)
  kf_pow<KF>(&w, &t, c_g2h.exp, bits);
  KF::mul(&y, &t, &w);
  KF::mul(&b, &y, &w);
  Fq bq = b.c[0], c, wq, fone;
  fq_set(c, c_g2h.ts_c);
  fq_one(fone);
  int m = (int)c_g2h.ts_s;
  for (int it = 0; it < 64 && !fq_eq(bq, fone); it++) {
    int i = 1;
    fq_sqr(wq, bq);
    while (i < m && !fq_eq(wq, fone)) { fq_sqr(wq, wq); i++; }
    if (i >= m) break;
    wq = c;
    for (int j = 0; j < m - i - 1; j++) fq_sqr(wq, wq);
    KF::scale(y, y, wq);
    fq_sqr(c, wq);
    fq_mul(bq, bq, c);
    m = i;
  }
  *yp = y;
}

#if !PBC_FQ_WIDE
// F_q^2 = F_q[i]/(i^2 - isq): x0 + x1 i is a square iff its norm x0^2 - isq x1^2 is one in F_q, zero
// included (fq_is_sqr, arith/fieldquadratic.c:339-355)
__device__ __noinline__ bool f2_is_sqr(const F2* t) {
  Fq n, u, k;
  fq_sqr(n, t->a);
  fq_sqr(u, t->b);
  fq_set(k, c_g2h.isq);
  fq_mul(u, u, k);
  fq_sub(n, n, u);
  return fq_is_zero(n) || fq_is_nonzero_sqr(n);
}
// a root of the square t, the norm method of fq_sqrt (arith/fieldquadratic.c:357-391):  m = sqrt(N(t)),
// z = (x0 +- m)/2 whichever is a square, y0 = sqrt(z), y1 = x1 / (2 y0).  x1 = 0 separately: then the root
// is sqrt(x0) or sqrt(x0 / isq) i.  F_q roots are z^((q + 1)/4) (q = 3 mod 4).
__device__ __noinline__ void f2_sqrt(F2* r, const F2* tp) {
  const F2 t = *tp;
  const int eb = (int)c_g2h.expbits;
  Fq n, m, z, y0, u, k;
  if (fq_is_zero(t.b)) {
    fq_pow_words(&y0, &t.a, c_g2h.exp, eb);
    fq_sqr(u, y0);
    if (fq_eq(u, t.a)) { r->a = y0; fq_zero(r->b); return; }
    fq_set(k, c_g2h.isq_inv);
    fq_mul(u, t.a, k);
    fq_pow_words(&r->b, &u, c_g2h.exp, eb);
    fq_zero(r->a);
    return;
  }
  fq_sqr(n, t.a);
  fq_sqr(u, t.b);
  fq_set(k, c_g2h.isq);
  fq_mul(u, u, k);
  fq_sub(n, n, u);
  fq_pow_words(&m, &n, c_g2h.exp, eb);
  fq_add(z, t.a, m);
  fq_halve(z, z);
  fq_pow_words(&y0, &z, c_g2h.exp, eb);
  fq_sqr(u, y0);
  if (!fq_eq(u, z)) {
    fq_sub(z, z, m);
    fq_pow_words(&y0, &z, c_g2h.exp, eb);
  }
  fq_dbl(u, y0);
  fq_inv(&u, &u);
  fq_mul(r->b, t.b, u);
  r->a = y0;
}
// N(x) = x x^q x^(q^2) x^(q^3) x^(q^4) in F_q^5 (as f5_inv)
__device__ __noinline__ void f5_norm(Fq* n, const F5* x) {
  F5 f1, f2, t;
  f5_frob(&f1, x);
  f5_frob(&f2, &f1);
  f5_mul(&t, &f1, &f2);
  f5_frob(&f1, &f2);
  f5_mul(&t, &t, &f1);
  f5_frob(&f2, &f1);
  f5_mul(&t, &t, &f2);
  f5_mul(&f1, &t, x);
  *n = f1.c[0];
}
__device__ __noinline__ bool f5_is_sqr(const F5* t) {
  Fq n;
  f5_norm(&n, t);
  return fq_is_nonzero_sqr(n);
}
#endif
// N(x) = x x^q x^(q^2) (coefficient 0 of the product; the others are zero)
__device__ __noinline__ void f3_norm(Fq* n, const F3* x) {
  F3 t, u;
  f3_frob(t, *x);
  f3_frob(u, t);
  f3_mul(&t, &t, &u);
  f3_mul(&u, &t, x);
  *n = u.c[0];
}
__device__ __noinline__ bool f3_is_sqr(const F3* t) {
  Fq n;
  f3_norm(&n, t);
  return fq_is_nonzero_sqr(n);
}
// polymod_sgn (arith/poly.c:1189-1199) on the reference basis: the first non-zero coefficient
__device__ __noinline__ int f3_sgn_ref(const F3* y) {
  F3 o = *y;
  f3_to_reference(o);
  int s = fq_sgn(o.c[0]);
  if (!s) s = fq_sgn(o.c[1]);
  if (!s) s = fq_sgn(o.c[2]);
  return s;
}

#if !PBC_FQ_WIDE
struct KF2 {                       // type f
  typedef F2 El;
  static __device__ __forceinline__ int wire() { return 2 * kWS; }
  static __device__ __forceinline__ void mul(El* r, const El* a, const El* b) { f2_mul(r, a, b); }
  static __device__ __forceinline__ void sqr(El* r, const El* a) { f2_sqr(r, a); }
  static __device__ __forceinline__ void inv(El* r, const El* a) { f2_inv(r, a); }
  static __device__ __forceinline__ void add(El& r, const El& a, const El& b) { f2_add(r, a, b); }
  static __device__ __forceinline__ void sub(El& r, const El& a, const El& b) { f2_sub(r, a, b); }
  static __device__ __forceinline__ void one(El& r) { f2_zero(r); fq_one(r.a); }
  static __device__ __forceinline__ bool is_zero(const El& a) { return fq_is_zero(a.a) && fq_is_zero(a.b); }
  static __device__ __forceinline__ bool eq(const El& a, const El& b) { return f2_eq(a, b); }
  static __device__ __forceinline__ bool a_is_zero() { return true; }
  static __device__ __forceinline__ void add_curve_a(El&) {}
  static __device__ __forceinline__ void mul_curve_a(El&) {}
  static __device__ __forceinline__ void add_curve_b(El& r) { f2_add(r, r, *f2_const(c_f.twist_b)); }
  static __device__ __forceinline__ void from_wire(El& r, const uint8_t* p) {
    Fq s;
    fq_from_wire(r.a, p);
    fq_from_wire(r.b, p + kWS);
    fq_set(s, c_f.sigma);
    fq_mul(r.b, r.b, s);
  }
  static __device__ __forceinline__ void to_wire(uint8_t* p, const El& a, bool zero) {
    Fq s, b;
    fq_set(s, c_f.sigma_inv);
    fq_mul(b, a.b, s);
    El o;
    o.a = a.a;
    o.b = b;
    if (zero) f2_zero(o);
    fq_to_wire(p, o.a);
    fq_to_wire(p + kWS, o.b);
  }
  // element_from_hash, compressed points
  static __device__ __forceinline__ void from_wire_b(El& r, const uint8_t* p) {    // no alignment needed
    Fq s;
    fq_from_wire_b<kWS>(r.a, p);
    fq_from_wire_b<kWS>(r.b, p + kWS);
    fq_set(s, c_f.sigma);
    fq_mul(r.b, r.b, s);
  }
  // fq_from_hash (arith/fieldquadratic.c:311-316): x0 from the first len/2 bytes, x1 from the rest
  static __device__ __forceinline__ void from_hash(El& r, const uint8_t* data, int len) {
    uint32_t w[kNS];
    Fq s;
    const int k = len / 2;
    hash_to_words<kNS>(w, data, k);
    fq_set(r.a, w);
    hash_to_words<kNS>(w, data + k, len - k);
    fq_set(r.b, w);
    fq_set(s, c_fp.r2);
    fq_mul(r.a, r.a, s);
    fq_mul(r.b, r.b, s);
    fq_set(s, c_f.sigma);
    fq_mul(r.b, r.b, s);
  }
  static __device__ __forceinline__ bool is_sqr(const El& t) { return f2_is_sqr(&t); }
  static __device__ __forceinline__ void sqrt(El& r, const El& t) { f2_sqrt(&r, &t); }
  static __device__ __forceinline__ void neg(El& r, const El& a) { f2_neg(r, a); }
  // fq_sign (arith/fieldquadratic.c:159-165) on the reference basis: x1 = sigma^-1 times the one in use
  static __device__ __forceinline__ int sign(const El& y) {
    int s = fq_sgn(y.a);
    if (s) return s;
    Fq k, b;
    fq_set(k, c_f.sigma_inv);
    fq_mul(b, y.b, k);
    return fq_sgn(b);
  }
};
#endif
#if PBC_FQ_WIDE
constexpr int kWB3 = 0;            // the run-time width
#else
constexpr int kWB3 = kWS;
#endif
struct KF3 {                       // type d
  typedef F3 El;
  static __device__ __forceinline__ int wire() { return 3 * fq_wb(); }
  static __device__ __forceinline__ void mul(El* r, const El* a, const El* b) { f3_mul(r, a, b); }
  static __device__ __forceinline__ void sqr(El* r, const El* a) { f3_sqr(r, a); }
  static __device__ __forceinline__ void inv(El* r, const El* a) { f3_inv(r, a); }
  static __device__ __forceinline__ void add(El& r, const El& a, const El& b) { f3_add(r, a, b); }
  static __device__ __forceinline__ void sub(El& r, const El& a, const El& b) { f3_sub(r, a, b); }
  static __device__ __forceinline__ void one(El& r) { f3_zero(r); fq_one(r.c[0]); }
  static __device__ __forceinline__ bool is_zero(const El& a) { return fq_is_zero(a.c[0]) && fq_is_zero(a.c[1]) && fq_is_zero(a.c[2]); }
  static __device__ __forceinline__ bool eq(const El& a, const El& b) { return f3_eq(a, b); }
  static __device__ __forceinline__ bool a_is_zero() { return false; }
  static __device__ __forceinline__ void add_curve_a(El& r) { Fq k; fq_set(k, c_d.twist_a); fq_add(r.c[0], r.c[0], k); }
  static __device__ __forceinline__ void mul_curve_a(El& r) { Fq k; fq_set(k, c_d.twist_a); f3_scale(r, r, k); }
  static __device__ __forceinline__ void add_curve_b(El& r) { Fq k; fq_set(k, c_d.twist_b); fq_add(r.c[0], r.c[0], k); }
  static __device__ __forceinline__ void from_wire(El& r, const uint8_t* p) {
#pragma unroll
    for (int i = 0; i < 3; i++) fq_from_wire(r.c[i], p + i * fq_wb());
    f3_to_internal(r);
  }
  static __device__ __forceinline__ void to_wire(uint8_t* p, const El& a, bool zero) {
    El o = a;
    f3_to_reference(o);
    if (zero) f3_zero(o);
#pragma unroll
    for (int i = 0; i < 3; i++) fq_to_wire(p + i * fq_wb(), o.c[i]);
  }
  // element_from_hash, compressed points
  static __device__ __forceinline__ void from_wire_b(El& r, const uint8_t* p) {    // no alignment needed
#pragma unroll
    for (int i = 0; i < 3; i++) fq_from_wire_b<kWB3>(r.c[i], p + i * fq_wb());
    f3_to_internal(r);
  }
  // polymod_from_hash (arith/poly.c:341-348): every coefficient is the hash of the whole data
  static __device__ __forceinline__ void from_hash(El& r, const uint8_t* data, int len) {
    uint32_t w[kNS];
    Fq s;
    hash_to_words<kNS>(w, data, len);
    fq_set(r.c[0], w);
    fq_set(s, c_fp.r2);
    fq_mul(r.c[0], r.c[0], s);
    r.c[1] = r.c[0];
    r.c[2] = r.c[0];
    f3_to_internal(r);
  }
  // polymod_is_sqr (arith/poly.c:617-632): t^((Q - 1)/2) == 1 = N(t)^((q - 1)/2) == 1; zero is not a square
  static __device__ __forceinline__ bool is_sqr(const El& t) { return f3_is_sqr(&t); }
  static __device__ __forceinline__ void sqrt(El& r, const El& t) { kf_sqrt_odd<KF3>(&r, &t); }
  static __device__ __forceinline__ void scale(El& r, const El& a, const Fq& k) { f3_scale(r, a, k); }
  static __device__ __forceinline__ void neg(El& r, const El& a) { f3_neg(r, a); }
  static __device__ __forceinline__ int sign(const El& y) { return f3_sgn_ref(&y); }
};

#if !PBC_FQ_WIDE
struct KF5 {                       // type g (19-byte coordinates)
  typedef F5 El;
  static __device__ __forceinline__ int wire() { return 5 * kWG; }
  static __device__ __forceinline__ void mul(El* r, const El* a, const El* b) { f5_mul(r, a, b); }
  static __device__ __forceinline__ void sqr(El* r, const El* a) { f5_sqr(r, a); }
  static __device__ __forceinline__ void inv(El* r, const El* a) { f5_inv(r, a); }
  static __device__ __forceinline__ void add(El& r, const El& a, const El& b) { f5_add(r, a, b); }
  static __device__ __forceinline__ void sub(El& r, const El& a, const El& b) { f5_sub(r, a, b); }
  static __device__ __forceinline__ void one(El& r) { f5_zero(r); fq_one(r.c[0]); }
  static __device__ __forceinline__ bool is_zero(const El& a) {
    bool z = true;
#pragma unroll
    for (int i = 0; i < 5; i++) z = z && fq_is_zero(a.c[i]);
    return z;
  }
  static __device__ __forceinline__ bool eq(const El& a, const El& b) { return f5_eq(a, b); }
  static __device__ __forceinline__ bool a_is_zero() { return false; }
  static __device__ __forceinline__ void add_curve_a(El& r) { Fq k; fq_set(k, c_g.twist_a); fq_add(r.c[0], r.c[0], k); }
  static __device__ __forceinline__ void mul_curve_a(El& r) { Fq k; fq_set(k, c_g.twist_a); f5_scale(r, r, k); }
  static __device__ __forceinline__ void add_curve_b(El& r) { Fq k; fq_set(k, c_g.twist_b); fq_add(r.c[0], r.c[0], k); }
  static __device__ __forceinline__ void from_wire(El& r, const uint8_t* p) {
#pragma unroll 1
    for (int i = 0; i < 5; i++) fq_from_wire_b<kWG>(r.c[i], p + i * kWG);
  }
  static __device__ __forceinline__ void to_wire(uint8_t* p, const El& a, bool zero) {
    El o = a;
    if (zero) f5_zero(o);
#pragma unroll 1
    for (int i = 0; i < 5; i++) fq_to_wire_b<kWG>(p + i * kWG, o.c[i]);
  }
  // element_from_hash, compressed points (the reference basis is the one in use)
  static __device__ __forceinline__ void from_wire_b(El& r, const uint8_t* p) { from_wire(r, p); }
  static __device__ __forceinline__ void from_hash(El& r, const uint8_t* data, int len) {
    uint32_t w[kNS];
    Fq s;
    hash_to_words<kNS>(w, data, len);
    fq_set(r.c[0], w);
    fq_set(s, c_fp.r2);
    fq_mul(r.c[0], r.c[0], s);
#pragma unroll
    for (int i = 1; i < 5; i++) r.c[i] = r.c[0];
  }
  static __device__ __forceinline__ bool is_sqr(const El& t) { return f5_is_sqr(&t); }
  static __device__ __forceinline__ void sqrt(El& r, const El& t) { kf_sqrt_odd<KF5>(&r, &t); }
  static __device__ __forceinline__ void scale(El& r, const El& a, const Fq& k) { f5_scale(r, a, k); }
  static __device__ __forceinline__ void neg(El& r, const El& a) { f5_neg(r, a); }
  static __device__ __forceinline__ int sign(const El& y) {
    int s = 0;
#pragma unroll 1
    for (int i = 0; i < 5 && !s; i++) s = fq_sgn(y.c[i]);
    return s;
  }
};

#endif

// out[i] = k[i] * in[i] on the twist.  One thread per point; all temporaries that are passed by
// address live at function scope (stack discipline note in pairing_f.cuh).
template <class KF, int BLOCK>
__global__ void __launch_bounds__(BLOCK, kCCMinBlocks)
k_cc_g2_mul(const uint8_t* __restrict__ P, const uint8_t* __restrict__ K, uint8_t* __restrict__ out, size_t n) {
  typedef typename KF::El El;
  size_t idx = (size_t)blockIdx.x * BLOCK + threadIdx.x;
  if (idx >= n) return;
  El xP, yP, X, Y, Z, Z2, M, Y2, t, u, H, R;
  KF::from_wire(xP, P + idx * (2 * KF::wire()));
  KF::from_wire(yP, P + idx * (2 * KF::wire()) + KF::wire());
  // on the curve?  y^2 == (x^2 + a') x + b'
  KF::sqr(&t, &xP);
  KF::add_curve_a(t);
  KF::mul(&t, &t, &xP);
  KF::add_curve_b(t);
  KF::sqr(&u, &yP);
  bool ok = KF::eq(t, u);
  uint32_t k[kZW];
  zr_from_wire(k, K + idx * c_zr.zlen);
  int top = zr_top_bit(k);
  X = xP;
  Y = yP;
  KF::one(Z);
  auto dbl = [&]() {                   // V = 2V:  M = 3 X^2 + a' Z^4
    KF::sqr(&Z2, &Z);
    KF::sqr(&t, &X);
    KF::add(M, t, t);
    KF::add(M, M, t);
    if (!KF::a_is_zero()) {
      KF::sqr(&u, &Z2);
      KF::mul_curve_a(u);
      KF::add(M, M, u);
    }
    KF::sqr(&Y2, &Y);
    KF::mul(&u, &Y, &Z);
    KF::add(Z, u, u);
    KF::mul(&t, &X, &Y2);
    KF::add(t, t, t);
    KF::add(t, t, t);                    // S = 4 X Y^2
    KF::sqr(&X, &M);
    KF::sub(X, X, t);
    KF::sub(X, X, t);
    KF::sqr(&Y2, &Y2);
    KF::add(Y2, Y2, Y2);
    KF::add(Y2, Y2, Y2);
    KF::add(Y2, Y2, Y2);                 // 8 Y^4
    KF::sub(t, t, X);
    KF::mul(&Y, &M, &t);
    KF::sub(Y, Y, Y2);
  };
  for (int j = top - 1; j >= 0; j--) {
    dbl();
    if ((k[j >> 5] >> (j & 31)) & 1u) {
      // V = V + P (mixed; V = O, V = P and V = -P as in g_add_affine, group_a.cuh)
      KF::sqr(&Z2, &Z);
      KF::mul(&t, &Z2, &Z);
      KF::mul(&H, &xP, &Z2);
      KF::sub(H, H, X);
      KF::mul(&R, &yP, &t);
      KF::sub(R, R, Y);
      if (KF::is_zero(H) || KF::is_zero(Z)) {
        if (KF::is_zero(Z)) { X = xP; Y = yP; KF::one(Z); }
        else if (KF::is_zero(R)) dbl();
        else Z = El();
        continue;
      }
      KF::mul(&Z, &H, &Z);
      KF::sqr(&t, &H);
      KF::mul(&u, &t, &H);
      KF::mul(&t, &t, &X);
      KF::sqr(&X, &R);
      KF::sub(X, X, u);
      KF::sub(X, X, t);
      KF::sub(X, X, t);
      KF::sub(t, t, X);
      KF::mul(&t, &t, &R);
      KF::mul(&u, &u, &Y);
      KF::sub(Y, t, u);
    }
  }
  bool inf = !ok || top < 0 || KF::is_zero(Z);
  KF::inv(&t, &Z);
  KF::sqr(&u, &t);
  KF::mul(&X, &X, &u);
  KF::mul(&u, &u, &t);
  KF::mul(&Y, &Y, &u);
  KF::to_wire(out + idx * (2 * KF::wire()), X, inf);
  KF::to_wire(out + idx * (2 * KF::wire()) + KF::wire(), Y, inf);
}

// element_from_hash on G2 (curve_from_hash, ecc/curve.c:455-482, on the twist): x from the hash, then
// x <- x^2 + 1 until x^3 + a' x + b' is a square (at most 64 tries, as on G1), y its root with
// sign(y) >= 0.  The twist has no cofactor (ecc/f_param.c:383, d_param.c:1057, g_param.c:1319): the point
// found is the output, usually outside the order-r subgroup.
template <class KF, int BLOCK>
__global__ void __launch_bounds__(BLOCK, kCCMinBlocks)
k_cc_g2_from_hash(const uint8_t* __restrict__ data, int len, uint8_t* __restrict__ out, size_t n) {
  typedef typename KF::El El;
  size_t idx = (size_t)blockIdx.x * BLOCK + threadIdx.x;
  if (idx >= n) return;
  El x, y, t, one;
  KF::from_hash(x, data + idx * (size_t)len, len);
  KF::one(one);
  for (int tries = 0; tries < 64; tries++) {
    KF::sqr(&t, &x);
    KF::add_curve_a(t);
    KF::mul(&t, &t, &x);
    KF::add_curve_b(t);
    if (KF::is_sqr(t)) break;
    KF::sqr(&x, &x);
    KF::add(x, x, one);
  }
  KF::sqrt(y, t);
  if (KF::sign(y) < 0) KF::neg(y, y);
  KF::to_wire(out + idx * (2 * KF::wire()), x, false);
  KF::to_wire(out + idx * (2 * KF::wire()) + KF::wire(), y, false);
}

// element_from_bytes_compressed on G2 (ecc/curve.c:799-813): x || sign byte -> x || y, y the root with
// sign > 0 for a non-zero byte and the other one for zero.  x^3 + a' x + b' = 0 gives (x, 0); no root
// gives zero bytes.
template <class KF, int BLOCK>
__global__ void __launch_bounds__(BLOCK, kCCMinBlocks)
k_cc_g2_decompress(const uint8_t* __restrict__ in, uint8_t* __restrict__ out, size_t n) {
  typedef typename KF::El El;
  size_t idx = (size_t)blockIdx.x * BLOCK + threadIdx.x;
  if (idx >= n) return;
  const uint8_t* p = in + idx * (size_t)(KF::wire() + 1);
  El x, y, t;
  KF::from_wire_b(x, p);               // items are wire + 1 bytes apart: byte loads
  KF::sqr(&t, &x);
  KF::add_curve_a(t);
  KF::mul(&t, &t, &x);
  KF::add_curve_b(t);
  bool ok = true;
  y = El();
  if (!KF::is_zero(t)) {
    ok = KF::is_sqr(t);
    if (ok) {
      KF::sqrt(y, t);
      const int s = KF::sign(y);
      if (p[KF::wire()] ? s < 0 : s > 0) KF::neg(y, y);
    }
  }
  KF::to_wire(out + idx * (2 * KF::wire()), x, !ok);
  KF::to_wire(out + idx * (2 * KF::wire()) + KF::wire(), y, !ok);
}

#if !PBC_FQ_WIDE
// out[i] = in[i]^k[i] in GT (type f: 240-byte F_q^12 elements)
template <int BLOCK>
__global__ void __launch_bounds__(BLOCK, kCCMinBlocks)
k_f_gt_pow(const uint8_t* __restrict__ G, const uint8_t* __restrict__ K, uint8_t* __restrict__ out,
           size_t n) {
  size_t idx = (size_t)blockIdx.x * BLOCK + threadIdx.x;
  if (idx >= n) return;
  F12 base, acc;
  uint32_t k[kZW];
  f12_from_wire(base, G + idx * (12 * kWS));
  f12_to_internal(base);
  zr_from_wire(k, K + idx * c_zr.zlen);
  int top = zr_top_bit(k);
  acc = base;
  for (int j = top - 1; j >= 0; j--) {
    f12_sqr(&acc);
    if ((k[j >> 5] >> (j & 31)) & 1u) f12_mul(&acc, &acc, &base);
  }
  if (top < 0) f12_one(acc);
  f12_to_reference(acc);
  f12_to_wire(out + idx * (12 * kWS), acc);
}

#endif

// type d: 120-byte F_q^6 elements
template <int BLOCK>
__global__ void __launch_bounds__(BLOCK, kCCMinBlocks)
k_d_gt_pow(const uint8_t* __restrict__ G, const uint8_t* __restrict__ K, uint8_t* __restrict__ out,
           size_t n) {
  size_t idx = (size_t)blockIdx.x * BLOCK + threadIdx.x;
  if (idx >= n) return;
  F6D base, acc;
  uint32_t k[kZW];
  f6d_from_wire(base, G + idx * (6 * fq_wb()));
  f3_to_internal(base.a);
  f3_to_internal(base.b);
  zr_from_wire(k, K + idx * c_zr.zlen);
  int top = zr_top_bit(k);
  acc = base;
  for (int j = top - 1; j >= 0; j--) {
    f6d_sqr(&acc);
    if ((k[j >> 5] >> (j & 31)) & 1u) f6d_mul(&acc, &acc, &base);
  }
  if (top < 0) f6d_one(acc);
  f3_to_reference(acc.a);
  f3_to_reference(acc.b);
  f6d_to_wire(out + idx * (6 * fq_wb()), acc);
}

#if !PBC_FQ_WIDE
// type g: 190-byte F_q^10 elements
template <int BLOCK>
__global__ void __launch_bounds__(BLOCK, kCCMinBlocks)
k_g_gt_pow(const uint8_t* __restrict__ G, const uint8_t* __restrict__ K, uint8_t* __restrict__ out,
           size_t n) {
  size_t idx = (size_t)blockIdx.x * BLOCK + threadIdx.x;
  if (idx >= n) return;
  F10 base, acc;
  uint32_t k[kZW];
  f10_from_wire(base, G + idx * (10 * kWG));
  zr_from_wire(k, K + idx * c_zr.zlen);
  int top = zr_top_bit(k);
  acc = base;
  for (int j = top - 1; j >= 0; j--) {
    f10_sqr(&acc);
    if ((k[j >> 5] >> (j & 31)) & 1u) f10_mul(&acc, &acc, &base);
  }
  if (top < 0) f10_one(acc);
  f10_to_wire(out + idx * (10 * kWG), acc);
}
#endif

}  // namespace pbcb200
