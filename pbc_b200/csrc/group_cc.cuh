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
};
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
