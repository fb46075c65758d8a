// common_kernels.cuh -- batch inversion (replaces the per-pairing mpz_invert calls of
// arith/montfp.c:401-422) and the F_p / IMAD micro-kernels used by bench.py's roofline.
#pragma once
#include "slots.cuh"

namespace pbcb200 {

// r = a^(p-2) on slots (Fermat; the modulus is prime: arith/fp.c:36-49 requires it too).
template <class O, int N>
__device__ __forceinline__ void slot_fermat_inverse(int r, int a, int one_slot) {
  O::copy(r, one_slot);
  int top = N * 32 - 1;
  while (top > 0 && !((c_fp.pm2[top >> 5] >> (top & 31)) & 1u)) top--;
  for (int j = top; j >= 0; j--) {
    O::sqr(r, r);
    if ((c_fp.pm2[j >> 5] >> (j & 31)) & 1u) O::mul(r, r, a);
  }
}

// In-place inversion of n Montgomery-form elements d[VPE][n] (limb-major vectors).
// Montgomery's simultaneous-inversion trick (the reference uses it only inside
// element_multi_double, ecc/curve.c:210-281): thread t owns the chain {t, t+T, t+2T, ...},
// T = number of chains, so every access is coalesced; one Fermat inversion per chain.
// Zero elements stay zero and do not poison their chain.  prefix: scratch of the same shape.
template <int N, bool FULL, int BLOCK>
__global__ void __launch_bounds__(BLOCK)
k_batch_invert(void* __restrict__ d, void* __restrict__ prefix, size_t n, size_t T) {
  using O = Ops<N, FULL, BLOCK>;
  enum { sACC, sE, sINV, sONE, sT, kSlots };
  size_t t = (size_t)blockIdx.x * BLOCK + threadIdx.x;
  if (t >= T) return;
  O::set_const(sONE, c_fp.one);
  O::copy(sACC, sONE);
  size_t K = (n + T - 1) / T;
  for (size_t j = 0; j < K; j++) {
    size_t idx = j * T + t;
    if (idx >= n) break;
    O::ld_global(sE, d, 0, n, idx);
    if (!O::is_zero(sE)) O::mul(sACC, sACC, sE);
    O::st_global(prefix, 0, n, idx, sACC);
  }
  slot_fermat_inverse<O, N>(sINV, sACC, sONE);
  for (size_t j = K; j-- > 0;) {
    size_t idx = j * T + t;
    if (idx >= n) continue;
    O::ld_global(sE, d, 0, n, idx);
    if (O::is_zero(sE)) continue;                 // stays zero; chain product skipped it
    if (j > 0) O::ld_global(sT, prefix, 0, n, idx - T); else O::copy(sT, sONE);
    O::mul(sT, sT, sINV);                         // 1/e_j = inv * prefix_{j-1}
    O::mul(sINV, sINV, sE);
    O::st_global(d, 0, n, idx, sT);
  }
}

// ---- micro-kernels for the integer-pipe roofline --------------------------------------------
// Dependent chain of `iters` Montgomery multiplications per thread, operands in registers.
template <int N, bool FULL, int IMPL>
__global__ void k_fpmul_chain(uint32_t* __restrict__ out, const uint32_t* __restrict__ in,
                              int iters) {
  size_t T = (size_t)gridDim.x * blockDim.x, t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  uint32_t a[N], b[N];
#pragma unroll
  for (int k = 0; k < N; k++) { a[k] = in[(2 * k) * T + t]; b[k] = in[(2 * k + 1) * T + t]; }
  for (int i = 0; i < iters; i++) {
    if (IMPL == 0) mont_mul<N, FULL>(a, a, b);
    else if (IMPL == 1) mont_mul_ps<N, FULL>(a, a, b);
    else fp_sqr<N, FULL>(a, a);
  }
#pragma unroll
  for (int k = 0; k < N; k++) out[k * T + t] = a[k];
}

// Same chain through the shared-memory slot machine (what the pairing kernels execute).
// MIX 0: multiplications only; 3: squarings only (O::sqr); 4: the lazy two-product routine of the
// type A Miller step (O::lazy: 2 x 256 products + one 272-unit reduction).
template <int N, bool FULL, int BLOCK, int MIX>
__global__ void __launch_bounds__(BLOCK, MIX == 4 ? 3 : 1)
k_fpmul_slots(uint32_t* __restrict__ out, const uint32_t* __restrict__ in, int iters) {
  using O = Ops<N, FULL, BLOCK>;
  size_t T = (size_t)gridDim.x * BLOCK, t = (size_t)blockIdx.x * BLOCK + threadIdx.x;
  uint32_t a[N], b[N];
#pragma unroll
  for (int k = 0; k < N; k++) { a[k] = in[(2 * k) * T + t]; b[k] = in[(2 * k + 1) * T + t]; }
  O::st(0, a); O::st(1, b);
  for (int i = 0; i < iters; i++) {
    if (MIX == 0) O::mul(0, 0, 1);
    else if (MIX == 4) O::lazy(0, O::LZ_TWO, 0, 1, 1, 0, 0, 0, nullptr, 0);   // (a b + b a) / R: two products, one reduction
    else O::sqr(0, 0);
  }
  O::ld(a, 0);
#pragma unroll
  for (int k = 0; k < N; k++) out[k * T + t] = a[k];
}

// IMAD.WIDE.U32 issue-rate probe: four independent carry chains of eight IMAD.WIDE.U32(.X) per
// thread and step -- the instruction the multipliers above are made of (32 per step).  The
// multiplicand of every link is data dependent, so nothing can be hoisted or strength-reduced
// (a first version with loop-invariant operands was folded into 64-bit adds by ptxas and
// over-reported the ceiling by 2x).  SURVEY 8d: "measure peak IMAD/s with a dependency-free
// microkernel" -- this is that denominator.
__global__ void k_imad_peak(uint64_t* __restrict__ out, uint32_t seed, int iters) {
  uint32_t y = seed * 3u + blockIdx.x + threadIdx.x;
  uint32_t a[4][16];
#pragma unroll
  for (int c = 0; c < 4; c++)
#pragma unroll
    for (int k = 0; k < 16; k++) a[c][k] = seed + 16 * c + k;
  for (int i = 0; i < iters; i++) {
#pragma unroll
    for (int c = 0; c < 4; c++) {
      asm volatile("mad.lo.cc.u32 %0, %2, %3, %0; madc.hi.cc.u32 %1, %2, %3, %1;"
                   : "+r"(a[c][0]), "+r"(a[c][1]) : "r"(a[c][15]), "r"(y));
#pragma unroll
      for (int k = 2; k < 16; k += 2)
        asm volatile("madc.lo.cc.u32 %0, %2, %3, %0; madc.hi.cc.u32 %1, %2, %3, %1;"
                     : "+r"(a[c][k]), "+r"(a[c][k + 1]) : "r"(a[c][k - 1]), "r"(y));
    }
  }
  uint32_t s = 0;
#pragma unroll
  for (int c = 0; c < 4; c++)
#pragma unroll
    for (int k = 0; k < 16; k++) s ^= a[c][k];
  out[(size_t)blockIdx.x * blockDim.x + threadIdx.x] = s;
}

// The same probe without carries: eight independent chains of IMAD.WIDE.U32 with a 64-bit addend,
// acc = lo(acc) * y + acc, four links each per step (again 32 per thread and step).  The carry-in
// form of k_imad_peak does not issue at the multiplier pipe's full rate on every GPU (on the H100 the
// kernels' own multipliers outran it), so the peak is the faster of the two probes.
__global__ void k_imad_peak_wide(uint64_t* __restrict__ out, uint32_t seed, int iters) {
  const uint32_t y = seed * 3u + blockIdx.x + threadIdx.x;
  uint64_t acc[8];
#pragma unroll
  for (int c = 0; c < 8; c++) acc[c] = ((uint64_t)(seed + c) << 32) | (seed ^ (uint32_t)c);
  for (int i = 0; i < iters; i++) {
#pragma unroll
    for (int k = 0; k < 4; k++)
#pragma unroll
      for (int c = 0; c < 8; c++) acc[c] += (uint64_t)(uint32_t)acc[c] * y;
  }
  uint64_t s = 0;
#pragma unroll
  for (int c = 0; c < 8; c++) s ^= acc[c];
  out[(size_t)blockIdx.x * blockDim.x + threadIdx.x] = s;
}

}  // namespace pbcb200
