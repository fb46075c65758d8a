// group_a1.cuh -- the operations either side of the Type A1 pairing: element_pow_zn on
// G1 = G2 = E(F_p) and on GT = F_p^2, element_from_hash and element_from_bytes_compressed on G1.
// Type A's kernels (group_a.cuh) on the 34-limb slot machine of pairing_a1.cuh: same curve
// y^2 = x^3 + x, same Jacobian double-and-add programs (g_double, g_add_affine), one inversion per
// point batched across the launch; what changes is the width -- scalars are Zr elements of up to
// 1087 bits (zlen = ceil(bits(n)/8) wire bytes, reduced mod n like element_from_bytes does,
// arith/montfp.c:498-517), the square-root exponent (p + 1)/4 and the hash limit are 34 words.
//   k_a1_g1_mul -> k_batch_invert<34> -> k_a1_g1_finish       k_a1_gt_pow
//   k_a1_g1_from_hash -> k_batch_invert<34> -> k_a1_g1_finish  k_a1_g1_decompress
#pragma once
#include "group_a.cuh"
#include "pairing_a1.cuh"

namespace pbcb200 {

struct alignas(16) A1GroupConsts {
  uint32_t n[kMaxLimbs];       // group order (scalars are reduced modulo it)
  uint32_t sqrt_exp[kMaxLimbs];   // (p + 1) / 4
  uint32_t q[kMaxLimbs];       // p (limit of pbc_mpz_from_hash)
  uint32_t expbits;
  uint32_t zlen;               // Zr wire bytes
  uint32_t count;              // bytes of p
  uint32_t pad;
};
__constant__ A1GroupConsts c_a1g;

// zlen big-endian bytes -> 34 little-endian words, reduced mod n.  n >= 2^(8 zlen - 8), so fewer
// than 256 subtractions.
__device__ __noinline__ void a1_zr_from_wire(uint32_t* k, const uint8_t* p) {
  a1_limbs_from_be(k, p, (int)c_a1g.zlen);
  for (int it = 0; it < 256; it++) {
    uint32_t d[kNA1], borrow;
    PBC_ASM("sub.cc.u32 %0, %1, %2;" : "=r"(d[0]) : "r"(k[0]), "r"(c_a1g.n[0]));
#pragma unroll
    for (int i = 1; i < kNA1; i++) PBC_ASM("subc.cc.u32 %0, %1, %2;" : "=r"(d[i]) : "r"(k[i]), "r"(c_a1g.n[i]));
    PBC_ASM("subc.u32 %0, 0, 0;" : "=r"(borrow));
    if (borrow) break;
#pragma unroll
    for (int i = 0; i < kNA1; i++) k[i] = d[i];
  }
}
__device__ __forceinline__ int a1_top_bit(const uint32_t* k) {
  for (int j = 32 * kNA1 - 1; j >= 0; j--)
    if ((k[j >> 5] >> (j & 31)) & 1u) return j;
  return -1;
}

// out: xyz [2][17][n] uint2 (Jacobian X, Y; Montgomery), zarr [17][n] = Z (0 marks "result is O")
template <int BLOCK>
__global__ void __launch_bounds__(BLOCK)
k_a1_g1_mul(const uint8_t* __restrict__ P, const uint8_t* __restrict__ K, void* __restrict__ xyz,
            void* __restrict__ zarr, size_t n) {
  using O = Ops<kNA1, false, BLOCK>;
  size_t idx = (size_t)blockIdx.x * BLOCK + threadIdx.x;
  if (idx >= n) return;
  bool okP = a1_load_point<O>(gPX, gPY, gT0, gT1, P + idx * 2 * (size_t)c_a1.wb);
  uint32_t k[kNA1];
  a1_zr_from_wire(k, K + idx * (size_t)c_a1g.zlen);
  int top = a1_top_bit(k);
  O::copy(gX, gPX);
  O::copy(gY, gPY);
  O::set_const(gZ, c_fp.one);
  O::set_const(gZ2, c_fp.one);
  for (int j = top - 1; j >= 0; j--) {
    g_double<O>();
    if ((k[j >> 5] >> (j & 31)) & 1u) g_add_affine<O>([] { g_double<O>(); });
  }
  uint32_t zero[kNA1] = {0};
  if (!okP || top < 0) O::st(gZ, zero);
  O::st_global(xyz, 0, n, idx, gX);
  O::st_global(xyz, 1, n, idx, gY);
  O::st_global(zarr, 0, n, idx, gZ);
}

// zinv = 1/Z (batch inverted in place) -> x = X zinv^2, y = Y zinv^3 -> wire bytes; O -> zero bytes
template <int BLOCK>
__global__ void __launch_bounds__(BLOCK)
k_a1_g1_finish(const void* __restrict__ xyz, const void* __restrict__ zinv, uint8_t* __restrict__ out,
               size_t n) {
  using O = Ops<kNA1, false, BLOCK>;
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
  const int wb = (int)c_a1.wb;
  uint32_t x[kNA1], one[kNA1] = {1};
  O::st(3, one);
  O::mul(0, 0, 3);                          // leave Montgomery form
  O::mul(1, 1, 3);
  uint8_t* o = out + idx * 2 * (size_t)wb;
#pragma unroll 1
  for (int c = 0; c < 2; c++) {
    O::ld(x, c);
    if (inf) {
#pragma unroll
      for (int i = 0; i < kNA1; i++) x[i] = 0;
    }
    a1_limbs_to_be(o + c * wb, x, wb);
  }
}

// out[i] = in[i]^k[i] in F_p^2 (GT wire format: re || im)
template <int BLOCK>
__global__ void __launch_bounds__(BLOCK)
k_a1_gt_pow(const uint8_t* __restrict__ G, const uint8_t* __restrict__ K, uint8_t* __restrict__ out,
            size_t n) {
  using O = Ops<kNA1, false, BLOCK>;
  enum { sB0, sB1, sA0, sA1, sT0, sT1, sT2 };
  size_t idx = (size_t)blockIdx.x * BLOCK + threadIdx.x;
  if (idx >= n) return;
  const int wb = (int)c_a1.wb;
  uint32_t x[kNA1], one[kNA1] = {1};
  O::set_const(sT0, c_fp.r2);
  a1_limbs_from_be(x, G + idx * 2 * (size_t)wb, wb);
  O::st(sB0, x);
  O::mul(sB0, sT0, sB0);
  a1_limbs_from_be(x, G + idx * 2 * (size_t)wb + wb, wb);
  O::st(sB1, x);
  O::mul(sB1, sT0, sB1);
  uint32_t k[kNA1];
  a1_zr_from_wire(k, K + idx * (size_t)c_a1g.zlen);
  int top = a1_top_bit(k);
  O::copy(sA0, sB0);
  O::copy(sA1, sB1);
  for (int j = top - 1; j >= 0; j--) {
    a_fsqr<O>(sA0, sA1, sT0, sT1);
    if ((k[j >> 5] >> (j & 31)) & 1u) a_fmul<O>(sA0, sA1, sB0, sB1, sT0, sT1, sT2);
  }
  O::st(sT0, one);
  O::mul(sA0, sA0, sT0);                    // leave Montgomery form
  O::mul(sA1, sA1, sT0);
  uint8_t* o = out + idx * 2 * (size_t)wb;
#pragma unroll 1
  for (int c = 0; c < 2; c++) {
    O::ld(x, c == 0 ? sA0 : sA1);
    if (top < 0) {                          // k = 0: the identity
#pragma unroll
      for (int i = 0; i < kNA1; i++) x[i] = (c == 0 && i == 0) ? 1u : 0u;
    }
    a1_limbs_to_be(o + c * wb, x, wb);
  }
}

// pbc_mpz_from_hash (arith/field.c:643-668) for the 34-word field: fill `count` bytes with the data
// repeated, a counter byte after each copy, read big-endian, halve while the value exceeds p.
__device__ __noinline__ void a1_hash_to_words(uint32_t* x, const uint8_t* data, int len) {
  uint8_t buf[4 * kNA1];
  const int count = (int)c_a1g.count;
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
  a1_limbs_from_be(x, buf, count);
  for (int it = 0; it < 8; it++) {
    bool gt = false, decided = false;
#pragma unroll
    for (int w = kNA1 - 1; w >= 0; w--) {
      if (!decided && x[w] != c_a1g.q[w]) { gt = x[w] > c_a1g.q[w]; decided = true; }
    }
    if (!gt) break;
#pragma unroll
    for (int w = 0; w < kNA1 - 1; w++) x[w] = __funnelshift_r(x[w], x[w + 1], 1);
    x[kNA1 - 1] >>= 1;
  }
}

// t^((p+1)/4) on slots: sY = root candidate of sT (sT is left untouched)
template <class O>
__device__ __forceinline__ void a1_sqrt_candidate(int sY, int sT) {
  O::copy(sY, sT);
  for (int j = (int)c_a1g.expbits - 2; j >= 0; j--) {
    O::sqr(sY, sY);
    if ((c_a1g.sqrt_exp[j >> 5] >> (j & 31)) & 1u) O::mul(sY, sY, sT);
  }
}

// element_from_hash on G1 (ecc/curve.c:455-482 curve_from_hash): try-and-increment on x, the odd
// root of x^3 + x, then the cofactor multiple by l.  Output as k_a1_g1_mul leaves it.
template <int BLOCK>
__global__ void __launch_bounds__(BLOCK)
k_a1_g1_from_hash(const uint8_t* __restrict__ data, int len, void* __restrict__ xyz,
                  void* __restrict__ zarr, size_t n) {
  using O = Ops<kNA1, false, BLOCK>;
  size_t idx = (size_t)blockIdx.x * BLOCK + threadIdx.x;
  if (idx >= n) return;
  uint32_t x[kNA1], one[kNA1] = {1};
  a1_hash_to_words(x, data + idx * (size_t)len, len);
  O::st(gPX, x);
  O::set_const(gT4, c_fp.r2);
  O::mul(gPX, gT4, gPX);                         // to Montgomery form; also reduces z == p to 0
  O::set_const(gT4, c_fp.one);
  for (int tries = 0; tries < 64; tries++) {
    O::sqr(gT0, gPX);
    O::add(gT0, gT0, gT4);
    O::mul(gT0, gT0, gPX);                       // t = x^3 + x
    a1_sqrt_candidate<O>(gPY, gT0);
    O::sqr(gT1, gPY);
    if (O::eq(gT1, gT0)) break;                  // t is a square (0 included), gPY = a root
    O::sqr(gPX, gPX);
    O::add(gPX, gPX, gT4);                       // x <- x^2 + 1
  }
  // keep the odd root (fp_sgn_odd, arith/montfp.c:460-472)
  O::st(gT1, one);
  O::mul(gT1, gPY, gT1);
  O::ld(x, gT1);
  if (!(x[0] & 1u) && !fp_is_zero<kNA1>(x)) O::neg(gPY, gPY);
  // cofactor multiple by l
  O::copy(gX, gPX);
  O::copy(gY, gPY);
  O::set_const(gZ, c_fp.one);
  O::set_const(gZ2, c_fp.one);
  for (int j = (int)c_a1.lbits - 2; j >= 0; j--) {
    g_double<O>();
    if ((c_a1.l[j >> 5] >> (j & 31)) & 1u) g_add_affine<O>([] { g_double<O>(); });
  }
  O::st_global(xyz, 0, n, idx, gX);
  O::st_global(xyz, 1, n, idx, gY);
  O::st_global(zarr, 0, n, idx, gZ);
}

// element_from_bytes_compressed on G1 (ecc/curve.c:799-813): x (wb bytes) || sign byte -> x || y
// with y = the root of x^3 + x whose parity the flag asks for (1 = odd).  An x without a point is
// written as zero bytes.
template <int BLOCK>
__global__ void __launch_bounds__(BLOCK)
k_a1_g1_decompress(const uint8_t* __restrict__ in, uint8_t* __restrict__ out, size_t n) {
  using O = Ops<kNA1, false, BLOCK>;
  enum { sX, sY, sT, sU, sONE };
  size_t idx = (size_t)blockIdx.x * BLOCK + threadIdx.x;
  if (idx >= n) return;
  const int wb = (int)c_a1.wb;
  const uint8_t* p = in + idx * (size_t)(wb + 1);
  uint32_t x[kNA1], y[kNA1], one[kNA1] = {1};
  a1_limbs_from_be(x, p, wb);
  O::st(sX, x);
  O::set_const(sT, c_fp.r2);
  O::mul(sX, sT, sX);
  O::set_const(sONE, c_fp.one);
  O::sqr(sT, sX);
  O::add(sT, sT, sONE);
  O::mul(sT, sT, sX);
  a1_sqrt_candidate<O>(sY, sT);
  O::sqr(sU, sY);
  bool ok = O::eq(sU, sT);
  O::st(sONE, one);                         // plain 1 from here on: leaves Montgomery form
  O::mul(sU, sY, sONE);
  O::ld(y, sU);
  bool odd = (y[0] & 1u) != 0, want_odd = p[wb] != 0;
  if (odd != want_odd && !fp_is_zero<kNA1>(y)) {
    O::neg(sY, sY);
    O::mul(sU, sY, sONE);
    O::ld(y, sU);
  }
  O::mul(sU, sX, sONE);
  O::ld(x, sU);
  if (!ok) {
#pragma unroll
    for (int k = 0; k < kNA1; k++) { x[k] = 0; y[k] = 0; }
  }
  a1_limbs_to_be(out + idx * 2 * (size_t)wb, x, wb);
  a1_limbs_to_be(out + idx * 2 * (size_t)wb + wb, y, wb);
}

// out[i] = a[i] * b[i] in F_p^2: element_mul on GT of type a1
template <int BLOCK>
__global__ void __launch_bounds__(BLOCK)
k_a1_gt_mul(const uint8_t* __restrict__ A, const uint8_t* __restrict__ B, uint8_t* __restrict__ out, size_t n) {
  using O = Ops<kNA1, false, BLOCK>;
  enum { sA0, sA1, sB0, sB1, sT0, sT1, sT2 };
  size_t idx = (size_t)blockIdx.x * BLOCK + threadIdx.x;
  if (idx >= n) return;
  const int wb = (int)c_a1.wb;
  uint32_t x[kNA1], one[kNA1] = {1};
  O::set_const(sT0, c_fp.r2);
#pragma unroll 1
  for (int c = 0; c < 4; c++) {
    a1_limbs_from_be(x, (c < 2 ? A : B) + idx * 2 * (size_t)wb + (size_t)(c & 1) * wb, wb);
    O::st(sA0 + c, x);
    O::mul(sA0 + c, sT0, sA0 + c);          // into Montgomery form (R^2 as the full operand, see a1_load_point)
  }
  a_fmul<O>(sA0, sA1, sB0, sB1, sT0, sT1, sT2);
  O::st(sT0, one);
  O::mul(sA0, sA0, sT0);
  O::mul(sA1, sA1, sT0);
  uint8_t* o = out + idx * 2 * (size_t)wb;
#pragma unroll 1
  for (int c = 0; c < 2; c++) {
    O::ld(x, sA0 + c);
    a1_limbs_to_be(o + c * wb, x, wb);
  }
}

}  // namespace pbcb200
