// group_e.cuh -- the operations either side of the Type E pairing: element_pow_zn on
// G1 = G2 = E(F_q) (y^2 = x^3 + a x + b) and on GT (F_q^*), element_mul on GT.
// G1 powers run type A's Jacobian double-and-add with the general coefficient a in the doubling;
// scalars are decoded and reduced mod r by type A1's a1_zr_from_wire (c_a1g.n holds r for a type E
// handle), and the result goes through k_batch_invert<34> and k_a1_g1_finish like type A1's.
//   k_e_g1_mul -> k_batch_invert<34> -> k_a1_g1_finish       k_e_gt_pow       k_e_gt_mul
#pragma once
#include "group_a1.cuh"
#include "pairing_e.cuh"

namespace pbcb200 {

// g_double (group_a.cuh) with M = 3 X^2 + a Z^4
template <class O>
__device__ __forceinline__ void e_g_double() {
  O::sqr(gT0, gX);
  O::dbl(gT2, gT0);
  O::add(gT0, gT0, gT2);
  if (!c_e.a_zero) {
    O::sqr(gT1, gZ2);
    O::mulg(gT1, gT1, e_pt(kEA), 1);
    O::add(gT0, gT0, gT1);         // M = 3 X^2 + a Z^4
  }
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

// out: xyz [2][17][n] uint2 (Jacobian X, Y; Montgomery), zarr [17][n] = Z (0 marks "result is O")
template <int BLOCK>
__global__ void __launch_bounds__(BLOCK)
k_e_g1_mul(const uint8_t* __restrict__ P, const uint8_t* __restrict__ K, void* __restrict__ xyz,
           void* __restrict__ zarr, size_t n) {
  using O = Ops<kNA1, false, BLOCK>;
  size_t idx = (size_t)blockIdx.x * BLOCK + threadIdx.x;
  if (idx >= n) return;
  bool okP = e_load_point<O>(gPX, gPY, gT0, gT1, P + idx * 2 * (size_t)c_a1.wb);
  uint32_t k[kNA1];
  a1_zr_from_wire(k, K + idx * (size_t)c_a1g.zlen);
  int top = a1_top_bit(k);
  O::copy(gX, gPX);
  O::copy(gY, gPY);
  O::set_const(gZ, c_fp.one);
  O::set_const(gZ2, c_fp.one);
  for (int j = top - 1; j >= 0; j--) {
    e_g_double<O>();
    if ((k[j >> 5] >> (j & 31)) & 1u) g_add_affine<O>([] { e_g_double<O>(); });
  }
  uint32_t zero[kNA1] = {0};
  if (!okP || top < 0) O::st(gZ, zero);
  O::st_global(xyz, 0, n, idx, gX);
  O::st_global(xyz, 1, n, idx, gY);
  O::st_global(zarr, 0, n, idx, gZ);
}

// out[i] = in[i]^k[i] in F_q (GT wire format: wb bytes)
template <int BLOCK>
__global__ void __launch_bounds__(BLOCK)
k_e_gt_pow(const uint8_t* __restrict__ G, const uint8_t* __restrict__ K, uint8_t* __restrict__ out, size_t n) {
  using O = Ops<kNA1, false, BLOCK>;
  enum { sB, sA, sT };
  size_t idx = (size_t)blockIdx.x * BLOCK + threadIdx.x;
  if (idx >= n) return;
  const int wb = (int)c_a1.wb;
  uint32_t x[kNA1], one[kNA1] = {1};
  O::set_const(sT, c_fp.r2);
  a1_limbs_from_be(x, G + idx * (size_t)wb, wb);
  uint32_t nz = 0;
#pragma unroll
  for (int i = 0; i < kNA1; i++) nz |= x[i];
  O::st(sB, x);
  O::mul(sB, sT, sB);
  uint32_t k[kNA1];
  a1_zr_from_wire(k, K + idx * (size_t)c_a1g.zlen);
  int top = a1_top_bit(k);
  O::copy(sA, sB);
  for (int j = top - 1; j >= 0; j--) {
    O::sqr(sA, sA);
    if ((k[j >> 5] >> (j & 31)) & 1u) O::mul(sA, sA, sB);
  }
  O::st(sT, one);
  O::mul(sA, sA, sT);              // leave Montgomery form
  O::ld(x, sA);
  if (top < 0 && nz) {             // k = 0: the identity, except for a zero base: fp_pow_mpz
                                   // (arith/montfp.c:379-396) leaves 0 at 0 whatever the exponent
#pragma unroll
    for (int i = 0; i < kNA1; i++) x[i] = one[i];
  }
  a1_limbs_to_be(out + idx * (size_t)wb, x, wb);
}

// out[i] = a[i] * b[i] in F_q: element_mul on GT of type e
template <int BLOCK>
__global__ void __launch_bounds__(BLOCK)
k_e_gt_mul(const uint8_t* __restrict__ A, const uint8_t* __restrict__ B, uint8_t* __restrict__ out, size_t n) {
  using O = Ops<kNA1, false, BLOCK>;
  enum { sA, sB, sT };
  size_t idx = (size_t)blockIdx.x * BLOCK + threadIdx.x;
  if (idx >= n) return;
  const int wb = (int)c_a1.wb;
  uint32_t x[kNA1], one[kNA1] = {1};
  O::set_const(sT, c_fp.r2);
  a1_limbs_from_be(x, A + idx * (size_t)wb, wb);
  O::st(sA, x);
  O::mul(sA, sT, sA);
  a1_limbs_from_be(x, B + idx * (size_t)wb, wb);
  O::st(sB, x);
  O::mul(sB, sT, sB);
  O::mul(sA, sA, sB);
  O::st(sT, one);
  O::mul(sA, sA, sT);              // leave Montgomery form
  O::ld(x, sA);
  a1_limbs_to_be(out + idx * (size_t)wb, x, wb);
}
constexpr int kEGroupSlots = 3;

}  // namespace pbcb200
