// group_a.cuh -- the operations either side of the Type A pairing (SURVEY 8f ranks 2 and 3):
//   element_pow_zn on G1 = G2 = E(F_q): y^2 = x^3 + x  (ecc/curve.c:455-482 curve_mul ->
//       arith/field.c:113-126 generic windowed power over curve_double / curve_mul)
//   element_pow_zn on GT (ecc/pairing.c:199-231 -> the same windowed power over fi_mul / fi_square,
//       arith/fieldquadratic.c:425-477)
// Same values (a multiple of a point / a power of a field element is canonical), different route:
// left-to-right double-and-add on Jacobian coordinates with ONE inversion per point, batched across
// the launch by k_batch_invert (the reference inverts once per affine addition), and plain
// square-and-multiply in F_q^2.  Scalars are Zr wire bytes (20, big-endian), reduced mod r like
// element_from_bytes does (arith/montfp.c:498-517).
//   k_a_g1_mul -> k_batch_invert -> k_a_g1_finish          k_a_gt_pow
#pragma once
#include "pairing_a.cuh"

namespace pbcb200 {

// words of a scalar: 5 (every type of engine.cu has r < 2^160), 8 in the wide type D instance
// (engine_d_wide.cu: r < 2^256)
#ifndef PBC_ZR_WORDS
#define PBC_ZR_WORDS 5
#endif
constexpr int kZW = PBC_ZR_WORDS;
template <int NW>
struct ZrConstsT {
  uint32_t r[NW];        // group order, little-endian words
  uint32_t zlen;         // Zr wire bytes: ceil(bits(r)/8) (20 for a, f, d159; 19 for g149)
  uint32_t pad[2];
};
typedef ZrConstsT<kZW> ZrConsts;
__constant__ ZrConsts c_zr;

// element_from_hash on G1 (ecc/curve.c:455-482): square-root exponent and cofactor, plain integers
struct HashConsts {
  uint32_t q[16];        // the field order (limit of pbc_mpz_from_hash, arith/field.c:643-668)
  uint32_t exp[16];      // sqrt_mode 1: (q + 1) / 4 (q = 3 mod 4);  2: (q - 5) / 8 (q = 5 mod 8, Atkin)
  uint32_t cofac[12];    // cofactor of G1 (h for types a and d, 1 for type f)
  uint32_t expbits, cofbits, sqrt_mode, count;   // count = bytes of q
};
__constant__ HashConsts c_hash;

// pbc_mpz_from_hash: fill `count` bytes with the data repeated, a counter byte after each copy
// (arith/field.c:649-661), read big-endian into NW little-endian words, halve while > q (:665-667).
template <int NW>
__device__ __forceinline__ void hash_to_words(uint32_t* x, const uint8_t* data, int len) {
  uint8_t buf[4 * NW];
  const int count = (int)c_hash.count;
  int i = 0;
  uint8_t counter = 0;
  for (;;) {
    int n;
    bool done;
    if (len >= count - i) { n = count - i; done = true; } else { n = len; done = false; }
    for (int k = 0; k < n; k++) buf[i + k] = data[k];
    i += n;
    if (done) break;
    buf[i] = counter++;
    i++;
    if (i == count) break;
  }
#pragma unroll
  for (int w = 0; w < NW; w++) {
    uint32_t v = 0;
#pragma unroll
    for (int b = 0; b < 4; b++) {
      int pos = count - 1 - (4 * w + b);       // byte of weight 256^(4w+b); count need not be a multiple of 4
      if (pos >= 0) v |= (uint32_t)buf[pos] << (8 * b);
    }
    x[w] = v;
  }
  for (int it = 0; it < 8; it++) {
    bool gt = false, decided = false;
#pragma unroll
    for (int w = NW - 1; w >= 0; w--) {
      if (!decided && x[w] != c_hash.q[w]) { gt = x[w] > c_hash.q[w]; decided = true; }
    }
    if (!gt) break;
#pragma unroll
    for (int w = 0; w < NW - 1; w++) x[w] = __funnelshift_r(x[w], x[w + 1], 1);
    x[NW - 1] >>= 1;
  }
}

constexpr int kWZ = 20;  // Zr wire bytes of a.param, f.param, d159.param (c_zr.zlen is authoritative)

// c_zr.zlen big-endian bytes -> five little-endian words, reduced mod r (r > 2^(8 zlen - 11): a few
// subtractions at most)
__device__ __forceinline__ void zr_from_wire(uint32_t* k, const uint8_t* p) {
  const int zlen = (int)c_zr.zlen;
#pragma unroll
  for (int i = 0; i < kZW; i++) {
    uint32_t w = 0;
#pragma unroll
    for (int b = 0; b < 4; b++) {
      int pos = zlen - 1 - (4 * i + b);
      if (pos >= 0) w |= (uint32_t)p[pos] << (8 * b);
    }
    k[i] = w;
  }
  for (int it = 0; it < 4096; it++) {
    uint32_t d[kZW], borrow;
    PBC_ASM("sub.cc.u32 %0, %1, %2;" : "=r"(d[0]) : "r"(k[0]), "r"(c_zr.r[0]));
#pragma unroll
    for (int i = 1; i < kZW; i++) PBC_ASM("subc.cc.u32 %0, %1, %2;" : "=r"(d[i]) : "r"(k[i]), "r"(c_zr.r[i]));
    PBC_ASM("subc.u32 %0, 0, 0;" : "=r"(borrow));
    if (borrow) break;
#pragma unroll
    for (int i = 0; i < kZW; i++) k[i] = d[i];
  }
}
__device__ __forceinline__ int zr_top_bit(const uint32_t* k) {
  for (int j = 32 * kZW - 1; j >= 0; j--)
    if ((k[j >> 5] >> (j & 31)) & 1u) return j;
  return -1;
}

enum GSlot { gX, gY, gZ, gZ2, gPX, gPY, gT0, gT1, gT2, gT3, gT4, kGSlots };

// V = 2V, Jacobian, a = 1 (Z2 = Z^2 is kept alongside): 3 M + 6 S
template <class O>
__device__ __forceinline__ void g_double() {
  O::sqr(gT0, gX);
  O::sqr(gT1, gZ2);
  O::dbl(gT2, gT0);
  O::add(gT0, gT0, gT2);
  O::add(gT0, gT0, gT1);           // M = 3 X^2 + Z^4
  O::sqr(gT1, gY);                 // Y^2
  O::mul(gT2, gX, gT1);
  O::dbl(gT2, gT2, 2);             // S = 4 X Y^2
  O::mul(gZ, gY, gZ);
  O::dbl(gZ, gZ);                  // Z' = 2 Y Z
  O::sqr(gZ2, gZ);
  O::sqr(gX, gT0);
  O::sub(gX, gX, gT2);
  O::sub(gX, gX, gT2);             // X' = M^2 - 2 S
  O::sqr(gT1, gT1);
  O::dbl(gT1, gT1, 3);             // 8 Y^4
  O::sub(gT2, gT2, gX);
  O::mulsub(gY, gT0, gT2, gT1);    // Y' = M (S - X') - 8 Y^4
}
// V = V + P, P affine in (gPX, gPY), for any V: 8 M + 3 S.  V = O (Z = 0), V = P and V = -P (H = 0)
// happen when the order of P is not r (a point of small order, or of order p1 in type a1's composite
// group); they take a branch of their own: V = O gives P, V = P the doubling `dbl` (the curve's
// g_double), V = -P gives O.
template <class O, class Dbl>
__device__ __forceinline__ void g_add_affine(Dbl dbl) {
  O::mul(gT0, gZ2, gZ);            // Z^3
  O::mul(gT1, gPX, gZ2);
  O::sub(gT1, gT1, gX);            // H = xP Z^2 - X
  O::mul(gT0, gPY, gT0);
  O::sub(gT0, gT0, gY);            // R = yP Z^3 - Y
  if (O::is_zero(gT1) || O::is_zero(gZ)) {
    if (O::is_zero(gZ)) {
      O::copy(gX, gPX);
      O::copy(gY, gPY);
      O::set_const(gZ, c_fp.one);
      O::set_const(gZ2, c_fp.one);
    } else if (O::is_zero(gT0)) {
      dbl();
    } else {
      uint32_t zero[O::kVecs * O::kVecWords] = {0};
      O::st(gZ, zero);
      O::st(gZ2, zero);
    }
    return;
  }
  O::mul(gZ, gZ, gT1);             // Z' = Z H
  O::sqr(gZ2, gZ);
  O::sqr(gT2, gT1);                // H^2
  O::mul(gT1, gT2, gT1);           // H^3
  O::mul(gT2, gT2, gX);            // X H^2
  O::sqr(gX, gT0);
  O::sub(gX, gX, gT1);
  O::sub(gX, gX, gT2);
  O::sub(gX, gX, gT2);             // X' = R^2 - H^3 - 2 X H^2
  O::sub(gT2, gT2, gX);
  O::mul(gT2, gT2, gT0);
  O::mul(gT1, gT1, gY);
  O::sub(gY, gT2, gT1);            // Y' = R (X H^2 - X') - Y H^3
}

// out: xyz [3][4][n] uint4 (Jacobian, Montgomery), zinv [4][n] = Z (0 marks "result is O")
template <int BLOCK>
__global__ void __launch_bounds__(BLOCK)
k_a_g1_mul(const uint8_t* __restrict__ P, const uint8_t* __restrict__ K, uint4* __restrict__ xyz,
           uint4* __restrict__ zarr, size_t n) {
  using O = Ops<kNA, true, BLOCK>;
  size_t idx = (size_t)blockIdx.x * BLOCK + threadIdx.x;
  bool live = idx < n;
  size_t src = live ? idx : 0;
  bool okP = a_load_point<O>(gPX, gPY, gT0, gT1, P + src * (2 * kWA));
  uint32_t k[5];
  zr_from_wire(k, K + src * c_zr.zlen);
  int top = zr_top_bit(k);
  O::copy(gX, gPX);
  O::copy(gY, gPY);
  O::set_const(gZ, c_fp.one);
  O::set_const(gZ2, c_fp.one);
  for (int j = top - 1; j >= 0; j--) {
    g_double<O>();
    if ((k[j >> 5] >> (j & 31)) & 1u) g_add_affine<O>([] { g_double<O>(); });
  }
  if (!live) return;
  uint32_t zero[kNA] = {0};
  if (!okP || top < 0) O::st(gZ, zero);
  O::st_global(xyz, 0, n, idx, gX);
  O::st_global(xyz, 1, n, idx, gY);
  O::st_global(zarr, 0, n, idx, gZ);
}

// zinv = 1/Z (batch inverted in place) -> x = X zinv^2, y = Y zinv^3 -> wire bytes; O -> zero bytes
// (the reference leaves stale coordinates behind an infinity flag, ecc/curve.c:603-609).
template <int BLOCK>
__global__ void __launch_bounds__(BLOCK)
k_a_g1_finish(const uint4* __restrict__ xyz, const uint4* __restrict__ zinv, uint8_t* __restrict__ out,
              size_t n) {
  using O = Ops<kNA, true, BLOCK>;
  size_t idx = (size_t)blockIdx.x * BLOCK + threadIdx.x;
  if (idx >= n) return;
  O::ld_global(0, xyz, 0, n, idx);
  O::ld_global(1, xyz, 1, n, idx);
  O::ld_global(2, zinv, 0, n, idx);
  bool inf = O::is_zero(2);
  O::sqr(3, 2);
  O::mul(0, 0, 3);
  O::mul(3, 3, 2);
  O::mul(1, 1, 3);
  uint32_t x[kNA], one[kNA] = {1};
  uint8_t* o = out + idx * (2 * kWA);
#pragma unroll 1
  for (int c = 0; c < 2; c++) {
    O::ld(x, c);
    mont_mul<kNA, true>(x, x, one);
    if (inf) {
#pragma unroll
      for (int k = 0; k < kNA; k++) x[k] = 0;
    }
    limbs_to_be<kNA, kWA>(o + c * kWA, x);
  }
}

// element_from_hash on G1, type a (q = 3 mod 4): try-and-increment on x, y = the odd root of
// x^3 + x via t^((q+1)/4), then the cofactor multiple (h = (q + 1)/r, 353 bits for a.param).
// Output as k_a_g1_mul leaves it (Jacobian X, Y and Z for the batched inversion).
template <int BLOCK>
__global__ void __launch_bounds__(BLOCK)
k_a_g1_from_hash(const uint8_t* __restrict__ data, int len, uint4* __restrict__ xyz,
                 uint4* __restrict__ zarr, size_t n) {
  using O = Ops<kNA, true, BLOCK>;
  size_t idx = (size_t)blockIdx.x * BLOCK + threadIdx.x;
  bool live = idx < n;
  size_t src = live ? idx : 0;
  uint32_t x[kNA], one[kNA] = {1};
  hash_to_words<kNA>(x, data + src * (size_t)len, len);
  mont_mul<kNA, true>(x, x, c_fp.r2);            // also reduces z == q to 0
  O::st(gPX, x);
  O::set_const(gT4, c_fp.one);
  for (int tries = 0; tries < 64; tries++) {
    O::sqr(gT0, gPX);
    O::add(gT0, gT0, gT4);
    O::mul(gT0, gT0, gPX);                       // t = x^3 + x
    O::copy(gPY, gT0);
    for (int j = (int)c_hash.expbits - 2; j >= 0; j--) {
      O::sqr(gPY, gPY);
      if ((c_hash.exp[j >> 5] >> (j & 31)) & 1u) O::mul(gPY, gPY, gT0);
    }
    O::sqr(gT1, gPY);
    if (O::eq(gT1, gT0)) break;                  // t is a square (0 included), gPY = a root
    O::sqr(gPX, gPX);
    O::add(gPX, gPX, gT4);                       // x <- x^2 + 1
  }
  // keep the odd root (fp_sgn_odd, arith/montfp.c:460-472)
  O::ld(x, gPY);
  mont_mul<kNA, true>(x, x, one);
  if (!(x[0] & 1u) && !fp_is_zero<kNA>(x)) O::neg(gPY, gPY);
  // cofactor multiple
  O::copy(gX, gPX);
  O::copy(gY, gPY);
  O::set_const(gZ, c_fp.one);
  O::set_const(gZ2, c_fp.one);
  for (int j = (int)c_hash.cofbits - 2; j >= 0; j--) {
    g_double<O>();
    if ((c_hash.cofac[j >> 5] >> (j & 31)) & 1u) g_add_affine<O>([] { g_double<O>(); });
  }
  if (!live) return;
  O::st_global(xyz, 0, n, idx, gX);
  O::st_global(xyz, 1, n, idx, gY);
  O::st_global(zarr, 0, n, idx, gZ);
}

// element_from_bytes_compressed on G1, type a (ecc/curve.c:799-813): x (64 bytes) || sign byte ->
// x || y with y = the root of x^3 + x whose parity the flag asks for (1 = odd, fp_sgn_odd).  An x
// whose right-hand side is not a square has no point: written as zero bytes (the reference's
// Tonelli loop returns garbage there).
template <int BLOCK>
__global__ void __launch_bounds__(BLOCK)
k_a_g1_decompress(const uint8_t* __restrict__ in, uint8_t* __restrict__ out, size_t n) {
  using O = Ops<kNA, true, BLOCK>;
  enum { sX, sY, sT, sU, sONE };
  size_t idx = (size_t)blockIdx.x * BLOCK + threadIdx.x;
  bool live = idx < n;
  size_t src = live ? idx : 0;
  const uint8_t* p = in + src * (kWA + 1);
  uint32_t x[kNA], one[kNA] = {1};
  limbs_from_be_bytes<kNA, kWA>(x, p);     // items are 65 bytes apart: byte loads
  mont_mul<kNA, true>(x, x, c_fp.r2);
  O::st(sX, x);
  O::set_const(sONE, c_fp.one);
  O::sqr(sT, sX);
  O::add(sT, sT, sONE);
  O::mul(sT, sT, sX);
  O::copy(sY, sT);
  for (int j = (int)c_hash.expbits - 2; j >= 0; j--) {
    O::sqr(sY, sY);
    if ((c_hash.exp[j >> 5] >> (j & 31)) & 1u) O::mul(sY, sY, sT);
  }
  O::sqr(sU, sY);
  bool ok = O::eq(sU, sT);
  if (!live) return;
  uint32_t y[kNA];
  O::ld(y, sY);
  mont_mul<kNA, true>(y, y, one);
  bool odd = (y[0] & 1u) != 0, want_odd = p[kWA] != 0;
  if (odd != want_odd && !fp_is_zero<kNA>(y)) {
    O::neg(sY, sY);
    O::ld(y, sY);
    mont_mul<kNA, true>(y, y, one);
  }
  O::ld(x, sX);
  mont_mul<kNA, true>(x, x, one);
  if (!ok) {
#pragma unroll
    for (int k = 0; k < kNA; k++) { x[k] = 0; y[k] = 0; }
  }
  limbs_to_be<kNA, kWA>(out + idx * (2 * kWA), x);
  limbs_to_be<kNA, kWA>(out + idx * (2 * kWA) + kWA, y);
}

// out[i] = in[i]^k[i] in F_q^2 (GT wire format: re || im)
template <int BLOCK>
__global__ void __launch_bounds__(BLOCK)
k_a_gt_pow(const uint8_t* __restrict__ G, const uint8_t* __restrict__ K, uint8_t* __restrict__ out,
           size_t n) {
  using O = Ops<kNA, true, BLOCK>;
  enum { sB0, sB1, sA0, sA1, sT0, sT1, sT2 };
  size_t idx = (size_t)blockIdx.x * BLOCK + threadIdx.x;
  bool live = idx < n;
  size_t src = live ? idx : 0;
  uint32_t x[kNA], one[kNA] = {1};
  limbs_from_be<kNA, kWA>(x, G + src * (2 * kWA));
  mont_mul<kNA, true>(x, x, c_fp.r2);
  O::st(sB0, x);
  limbs_from_be<kNA, kWA>(x, G + src * (2 * kWA) + kWA);
  mont_mul<kNA, true>(x, x, c_fp.r2);
  O::st(sB1, x);
  uint32_t k[5];
  zr_from_wire(k, K + src * c_zr.zlen);
  int top = zr_top_bit(k);
  O::copy(sA0, sB0);
  O::copy(sA1, sB1);
  for (int j = top - 1; j >= 0; j--) {
    O::add(sT0, sA0, sA1);
    O::sub(sT1, sA0, sA1);
    O::mul(sA1, sA0, sA1);
    O::dbl(sA1, sA1);
    O::mul(sA0, sT0, sT1);
    if ((k[j >> 5] >> (j & 31)) & 1u) a_fmul<O>(sA0, sA1, sB0, sB1, sT0, sT1, sT2);
  }
  if (!live) return;
  uint8_t* o = out + idx * (2 * kWA);
#pragma unroll 1
  for (int c = 0; c < 2; c++) {
    O::ld(x, c == 0 ? sA0 : sA1);
    mont_mul<kNA, true>(x, x, one);
    if (top < 0) {                       // k = 0: the identity
#pragma unroll
      for (int i = 0; i < kNA; i++) x[i] = (c == 0 && i == 0) ? 1u : 0u;
    }
    limbs_to_be<kNA, kWA>(o + c * kWA, x);
  }
}

// out[i] = a[i] * b[i] in F_q^2: element_mul on GT (ecc/pairing.c:199-201 -> fi_mul, arith/fieldquadratic.c:425-457)
template <int BLOCK>
__global__ void __launch_bounds__(BLOCK)
k_a_gt_mul(const uint8_t* __restrict__ A, const uint8_t* __restrict__ B, uint8_t* __restrict__ out, size_t n) {
  using O = Ops<kNA, true, BLOCK>;
  enum { sA0, sA1, sB0, sB1, sT0, sT1, sT2 };
  size_t idx = (size_t)blockIdx.x * BLOCK + threadIdx.x;
  if (idx >= n) return;
  uint32_t x[kNA], one[kNA] = {1};
#pragma unroll 1
  for (int c = 0; c < 4; c++) {
    const uint8_t* src = (c < 2 ? A : B) + idx * (2 * kWA) + (c & 1) * kWA;
    limbs_from_be<kNA, kWA>(x, src);
    mont_mul<kNA, true>(x, x, c_fp.r2);
    O::st(sA0 + c, x);
  }
  a_fmul<O>(sA0, sA1, sB0, sB1, sT0, sT1, sT2);
  uint8_t* o = out + idx * (2 * kWA);
#pragma unroll 1
  for (int c = 0; c < 2; c++) {
    O::ld(x, sA0 + c);
    mont_mul<kNA, true>(x, x, one);
    limbs_to_be<kNA, kWA>(o + c * kWA, x);
  }
}

}  // namespace pbcb200
