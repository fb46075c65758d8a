// prod_v.cuh -- products of pairings with a pair count per output (pbc_b200_prod_pairings_apply_v):
// the segmented product of the Miller values, for every representation.
//
// The per-pair Miller kernels leave one value per pair; output i multiplies the values of pairs
// [offsets[i], offsets[i+1]).  One launch of k_prod_v is one pass: thread r multiplies run r, at most
// kProdVRun consecutive values of one output, and writes its partial product to position r.  The runs of
// one output are consecutive, so a pass leaves the partial products of each output contiguous and the
// next pass is the same kernel on the shorter batch.  The host (engine.cu, ProdPlan) builds the run
// table of every pass from the offsets: ceil(log_L(longest)) passes, the last with one run per output.
// A 2^18-pair product takes five passes of at most sixteen multiplications per thread, not 2^18
// multiplications on one thread.
//
// A policy P holds one thread's accumulator and knows its representation: first(in, j) loads value j,
// next(in, j) multiplies value j in, store(out, r, last) writes the partial product.  Validity travels
// with every partial exactly as the uniform product kernels compute it (d = 0 for types a and a1, vd = 0
// for type e, the flag word for types f, d and g); only the last pass publishes what the final stage
// reads (type a's and a1's N(F) F0 F1, e_publish), intermediate passes store the accumulator itself.
#pragma once
#include "slots.cuh"
#include "a_steps.cuh"

namespace pbcb200 {

constexpr int kProdVRun = 16;   // values per run (at most)

// one batch of values: limb-major arrays with `n` elements per vector row (the Miller kernels' layout)
struct ProdVBuf {
  void* v;      // the value
  void* d;      // its validity: d (types a, a1), vd (type e), the flag words (types f, d, g)
  size_t n;     // element stride
};

// runs: n_runs + 1 input indices; run r covers values [runs[r], runs[r + 1]), 1 to kProdVRun of them
template <class P, int BLOCK>
__global__ void __launch_bounds__(BLOCK, P::kMinBlocks)
k_prod_v(ProdVBuf in, ProdVBuf out, const uint64_t* __restrict__ runs, size_t n_runs, int last) {
  size_t r = (size_t)blockIdx.x * BLOCK + threadIdx.x;
  if (r >= n_runs) return;
  const size_t j0 = runs[r], j1 = runs[r + 1];
  P acc;
  acc.first(in, j0);
  for (size_t j = j0 + 1; j < j1; j++) acc.next(in, j);
  acc.store(out, r, last != 0);
}

// F_q^2 values on the slot machine (types a and a1): f [2][..][n], d [..][n].  d = N(f) f0 f1 of a
// Miller value, 0 for an invalid pair or a degenerate value; a partial stores d = 1 or 0 (valid or not),
// the last pass N(F) F0 F1 or 0, as k_a_prod and a1_publish do.
template <class O, int N>
struct ProdVF2 {
  enum { pF0, pF1, pL0, pL1, pT0, pT1, pT2, kSlots };
  static constexpr int kMinBlocks = 1;
  bool ok;
  __device__ __forceinline__ void first(const ProdVBuf& in, size_t j) {
    O::ld_global(pF0, in.v, 0, in.n, j);
    O::ld_global(pF1, in.v, 1, in.n, j);
    O::ld_global(pT0, in.d, 0, in.n, j);
    ok = !O::is_zero(pT0);
  }
  __device__ __forceinline__ void next(const ProdVBuf& in, size_t j) {
    O::ld_global(pL0, in.v, 0, in.n, j);
    O::ld_global(pL1, in.v, 1, in.n, j);
    O::ld_global(pT0, in.d, 0, in.n, j);
    ok = ok && !O::is_zero(pT0);
    a_fmul<O>(pF0, pF1, pL0, pL1, pT0, pT1, pT2);
  }
  __device__ __forceinline__ void store(const ProdVBuf& out, size_t r, bool last) {
    if (last) {
      O::sqr(pT0, pF0);
      O::sqr(pT1, pF1);
      O::add(pT0, pT0, pT1);
      O::mul(pT1, pF0, pF1);
      O::mul(pT0, pT0, pT1);
    } else {
      O::set_const(pT0, c_fp.one);
    }
    if (!ok) {
      uint32_t zero[N] = {0};
      O::st(pT0, zero);
    }
    O::st_global(out.v, 0, out.n, r, pF0);
    O::st_global(out.v, 1, out.n, r, pF1);
    O::st_global(out.d, 0, out.n, r, pT0);
  }
};

// register-resident tower elements (types f, d, g): T is a traits struct with the element type E and
// its ld / st (limb-major, stride n) and mul.  The flag word is 1 for a valid pair; the Miller kernels
// already store 1 as the value of an invalid pair, so the product needs no publish step.
template <class T>
struct ProdVCC {
  static constexpr int kMinBlocks = T::kMinBlocks;
  typename T::E acc;
  bool ok;
  __device__ __forceinline__ void first(const ProdVBuf& in, size_t j) {
    T::ld(acc, (const uint32_t*)in.v, in.n, j);
    ok = ((const uint32_t*)in.d)[j] != 0;
  }
  __device__ __forceinline__ void next(const ProdVBuf& in, size_t j) {
    typename T::E t;
    T::ld(t, (const uint32_t*)in.v, in.n, j);
    ok = ok && ((const uint32_t*)in.d)[j] != 0;
    T::mul(&acc, &acc, &t);
  }
  __device__ __forceinline__ void store(const ProdVBuf& out, size_t r, bool) {
    T::st((uint32_t*)out.v, out.n, r, acc);
    ((uint32_t*)out.d)[r] = ok ? 1u : 0u;
  }
};

}  // namespace pbcb200
