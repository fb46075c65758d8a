// fp.cuh -- F_p arithmetic for sm_90a: fixed-limb Montgomery multiplication, all limbs in registers.
//
// Replaces, for the device path, the reference's arith/montfp.c (mont_mul :334-364,
// fp_add/sub/double/halve/neg :220-330).  Same value semantics (x is held as x*R mod p,
// R = 2^(32 N)), different mechanics:
//   * limbs are 32-bit words (N = 16 for the 512-bit Type-A prime, 6 for the 158/159-bit F/D
//     primes); two words = one of the reference's 64-bit limbs, same little-endian order.
//   * the product a*b and the reduction m*p are both accumulated with
//     mad.lo.cc.u32 / madc.hi.cc.u32 carry chains laid out so that every 32x32 product is ONE
//     IMAD.WIDE.U32 with predicate carry-in/out in SASS: products whose low word lands on an even
//     column go to accumulator `ev`, odd columns to `od`; the two are merged once at the end.
//   * coarsely-integrated operand scanning: after each b-limb the running sum is divisible by
//     2^32, the implied one-word shift swaps the roles of ev and od (no data movement).
//   * no zero flag: zero is all-zero limbs (reference: arith/montfp.c:36-39 keeps a flag).
//
// The modulus and its constants live in __constant__ memory so they appear as c[bank][off]
// operands of IMAD and never cost registers.
#pragma once
#include <stdint.h>

namespace pbcb200 {

constexpr int kMaxLimbs = 36;     // type a1 uses 34; 36 keeps every field 16-byte aligned

struct FpConsts {
  uint32_t p[kMaxLimbs];     // modulus
  uint32_t r2[kMaxLimbs];    // R^2 mod p   (to Montgomery form: mont_mul(x, r2))
  uint32_t one[kMaxLimbs];   // R mod p     (Montgomery 1)
  uint32_t pm2[kMaxLimbs];   // p - 2       (Fermat inversion exponent)
  uint32_t np0;              // -p^-1 mod 2^32
  uint32_t nlimbs;
  uint32_t pad[10];          // 8 words more than alignment needs: they keep c_fp at its size, so the constant-bank
                             // offsets of every later __constant__ symbol (and with them most kernels' code) stay put
};

__constant__ FpConsts c_fp;   // single translation unit (engine.cu)

// ---------------------------------------------------------------------------------------------
// carry-chain building blocks.  `volatile` keeps the PTX in source order; ptxas tracks CC.CF and
// is free to interleave independent chains when it schedules SASS.
// ---------------------------------------------------------------------------------------------
#define PBC_ASM asm volatile

// acc[0..N) (+)= x[0], x[2], ... , x[N-2] times y, pairs (acc[j],acc[j+1]) receive x[j]*y.
// `x` is indexed with stride 2 starting at x[0]; returns nothing, leaves carry-out in CC.CF.
template <int N>
__device__ __forceinline__ void chain_mad(uint32_t* acc, const uint32_t* x, uint32_t y) {
  PBC_ASM("mad.lo.cc.u32 %0, %2, %3, %0; madc.hi.cc.u32 %1, %2, %3, %1;"
          : "+r"(acc[0]), "+r"(acc[1]) : "r"(x[0]), "r"(y));
#pragma unroll
  for (int j = 2; j < N; j += 2)
    PBC_ASM("madc.lo.cc.u32 %0, %2, %3, %0; madc.hi.cc.u32 %1, %2, %3, %1;"
            : "+r"(acc[j]), "+r"(acc[j + 1]) : "r"(x[j]), "r"(y));
}

// acc[j],acc[j+1] = x[j]*y  (no carries involved)
template <int N>
__device__ __forceinline__ void chain_mul(uint32_t* acc, const uint32_t* x, uint32_t y) {
#pragma unroll
  for (int j = 0; j < N; j += 2)
    PBC_ASM("mul.lo.u32 %0, %2, %3; mul.hi.u32 %1, %2, %3;"
            : "=r"(acc[j]), "=r"(acc[j + 1]) : "r"(x[j]), "r"(y));
}

// The shifting chain: acc[j],acc[j+1] = x[j]*y + acc[j+2],acc[j+3] (+ incoming CC.CF), the top
// pair adds `top` (the overflow word of the previous round) instead.  Leaves carry-out in CC.CF.
template <int N>
__device__ __forceinline__ void chain_mad_shift(uint32_t* acc, const uint32_t* x, uint32_t y,
                                                uint32_t top) {
#pragma unroll
  for (int j = 0; j < N - 2; j += 2)
    PBC_ASM("madc.lo.cc.u32 %0, %2, %3, %4; madc.hi.cc.u32 %1, %2, %3, %5;"
            : "=r"(acc[j]), "=r"(acc[j + 1])
            : "r"(x[j]), "r"(y), "r"(acc[j + 2]), "r"(acc[j + 3]));
  PBC_ASM("madc.lo.cc.u32 %0, %2, %3, 0; madc.hi.cc.u32 %1, %2, %3, %4;"
          : "=r"(acc[N - 2]), "=r"(acc[N - 1]) : "r"(x[N - 2]), "r"(y), "r"(top));
}

__device__ __forceinline__ uint32_t carry_out() {
  uint32_t c;
  PBC_ASM("addc.u32 %0, 0, 0;" : "=r"(c));
  return c;
}

// ---------------------------------------------------------------------------------------------
// One round of the interleaved multiply/reduce.  On entry (first == false) `z` is the
// accumulator whose low word is zero (even-aligned before the implied shift), `w` the
// odd-aligned one, `top` the overflow word above w.  On exit w's low word is zero: the caller swaps.
// FULL = modulus uses all 32N bits (Type A): the running sum needs one more bit than N+1 words.
// ---------------------------------------------------------------------------------------------
template <int N, bool FULL>
__device__ __forceinline__ void mont_round(uint32_t* z, uint32_t* w, uint32_t& top,
                                           const uint32_t* a, uint32_t bi, bool first) {
  if (first) {
    chain_mul<N>(z, a + 1, bi);   // columns 1.. (odd-aligned)
    chain_mul<N>(w, a, bi);       // columns 0.. (even-aligned)
    top = 0;
  } else {
    // shift by one word: w becomes even-aligned as is; z loses its zero word, z[1] is a lone
    // column-0 word, z[2..] become odd-aligned.
    PBC_ASM("add.cc.u32 %0, %0, %1;" : "+r"(w[0]) : "r"(z[1]));
    chain_mad_shift<N>(z, a + 1, bi, top);    // carry of the add enters at column 1
    if (FULL) top = carry_out();
    chain_mad<N>(w, a, bi);
    if (FULL) {
      PBC_ASM("addc.cc.u32 %0, %0, 0;" : "+r"(z[N - 1]));
      PBC_ASM("addc.u32 %0, %0, 0;" : "+r"(top));
    } else {
      PBC_ASM("addc.u32 %0, %0, 0;" : "+r"(z[N - 1]));
    }
  }
  uint32_t m = w[0] * c_fp.np0;
  chain_mad<N>(z, c_fp.p + 1, m);
  if (FULL) {
    uint32_t c = carry_out();
    top += c;
  }
  chain_mad<N>(w, c_fp.p, m);
  if (FULL) {
    PBC_ASM("addc.cc.u32 %0, %0, 0;" : "+r"(z[N - 1]));
    PBC_ASM("addc.u32 %0, %0, 0;" : "+r"(top));
  } else {
    PBC_ASM("addc.u32 %0, %0, 0;" : "+r"(z[N - 1]));
  }
}

// r = (z >> 32) + w (+ top << 32N), then one conditional subtraction of p.  z has zero low word.
template <int N, bool FULL>
__device__ __forceinline__ void mont_finish(uint32_t* r, const uint32_t* z, const uint32_t* w,
                                            uint32_t top) {
  uint32_t t[N];
  PBC_ASM("add.cc.u32 %0, %1, %2;" : "=r"(t[0]) : "r"(z[1]), "r"(w[0]));
#pragma unroll
  for (int k = 1; k < N - 1; k++)
    PBC_ASM("addc.cc.u32 %0, %1, %2;" : "=r"(t[k]) : "r"(z[k + 1]), "r"(w[k]));
  PBC_ASM("addc.cc.u32 %0, %1, 0;" : "=r"(t[N - 1]) : "r"(w[N - 1]));
  if (FULL) PBC_ASM("addc.u32 %0, %0, 0;" : "+r"(top));
  // d = t - p
  uint32_t d[N], borrow;
  PBC_ASM("sub.cc.u32 %0, %1, %2;" : "=r"(d[0]) : "r"(t[0]), "r"(c_fp.p[0]));
#pragma unroll
  for (int k = 1; k < N; k++)
    PBC_ASM("subc.cc.u32 %0, %1, %2;" : "=r"(d[k]) : "r"(t[k]), "r"(c_fp.p[k]));
  PBC_ASM("subc.u32 %0, 0, 0;" : "=r"(borrow));   // 0 if t >= p, 0xffffffff otherwise
  bool use_d = FULL ? (top != 0 || borrow == 0) : (borrow == 0);
#pragma unroll
  for (int k = 0; k < N; k++) r[k] = use_d ? d[k] : t[k];
}

// r = a*b/R mod p, inputs and output fully reduced.  r may alias a or b.
template <int N, bool FULL>
__device__ __forceinline__ void mont_mul(uint32_t* r, const uint32_t* a, const uint32_t* b) {
  uint32_t x[N], y[N], top;
  mont_round<N, FULL>(x, y, top, a, b[0], true);
#pragma unroll
  for (int i = 1; i < N; i += 2) {
    mont_round<N, FULL>(y, x, top, a, b[i], false);
    if (i + 1 < N) mont_round<N, FULL>(x, y, top, a, b[i + 1], false);
  }
  // N even: the last round ran as (y, x): x has the zero low word
  mont_finish<N, FULL>(r, x, y, top);
}

// ---------------------------------------------------------------------------------------------
// Double width: lazy reduction.  A sum of products is accumulated unreduced in 2N + 1 words and
// reduced once, so each product after the first costs N^2 IMAD.WIDE instead of N^2 + N^2 + N.
// The caller keeps the value handed to redc_wide in [0, 2 q R) (q < R = 2^(32N) for any q):
//   a b + c d < 2 q^2,  a b - c d + q R < q^2 + q R,  and a stored S' < q R in  a b - S' + q R.
// Intermediate values may be negative: the 2N + 1 words are exact modulo 2^(32(2N+1)).
// ---------------------------------------------------------------------------------------------
// One row of the plain product: mont_round without the m p half.  w[0] on exit is a finished
// column.  The running sum a (b mod 2^(32(i+1))) / 2^(32i) stays below 2^(32(N+1)): no top word.
template <int N>
__device__ __forceinline__ void wide_round(uint32_t* z, uint32_t* w, const uint32_t* a, uint32_t bi, bool first) {
  if (first) {
    chain_mul<N>(z, a + 1, bi);
    chain_mul<N>(w, a, bi);
  } else {
    PBC_ASM("add.cc.u32 %0, %0, %1;" : "+r"(w[0]) : "r"(z[1]));
    chain_mad_shift<N>(z, a + 1, bi, 0);
    chain_mad<N>(w, a, bi);
    PBC_ASM("addc.u32 %0, %0, 0;" : "+r"(z[N - 1]));
  }
}

// p[0..2N) = a*b, operand scanning on the even / odd accumulators: one IMAD.WIDE per product.
template <int N>
__device__ __forceinline__ void mul_wide(uint32_t* p, const uint32_t* a, const uint32_t* b) {
  static_assert(N % 2 == 0, "even limb count");
  uint32_t x[N], y[N];
  wide_round<N>(x, y, a, b[0], true);
  p[0] = y[0];
#pragma unroll
  for (int i = 1; i < N; i += 2) {
    wide_round<N>(y, x, a, b[i], false);
    p[i] = x[0];
    if (i + 1 < N) {
      wide_round<N>(x, y, a, b[i + 1], false);
      p[i + 1] = y[0];
    }
  }
  // the last row ran as (y, x): the high half is (x >> 32) + y
  PBC_ASM("add.cc.u32 %0, %1, %2;" : "=r"(p[N]) : "r"(x[1]), "r"(y[0]));
#pragma unroll
  for (int k = 1; k < N - 1; k++)
    PBC_ASM("addc.cc.u32 %0, %1, %2;" : "=r"(p[N + k]) : "r"(x[k + 1]), "r"(y[k]));
  PBC_ASM("addc.u32 %0, %1, 0;" : "=r"(p[2 * N - 1]) : "r"(y[N - 1]));
}

// acc[0..2N] += p[0..2N)
template <int N>
__device__ __forceinline__ void wide_add(uint32_t* acc, const uint32_t* p) {
  PBC_ASM("add.cc.u32 %0, %0, %1;" : "+r"(acc[0]) : "r"(p[0]));
#pragma unroll
  for (int k = 1; k < 2 * N; k++) PBC_ASM("addc.cc.u32 %0, %0, %1;" : "+r"(acc[k]) : "r"(p[k]));
  PBC_ASM("addc.u32 %0, %0, 0;" : "+r"(acc[2 * N]));
}

// acc[0..2N] -= p[0..2N)
template <int N>
__device__ __forceinline__ void wide_sub(uint32_t* acc, const uint32_t* p) {
  PBC_ASM("sub.cc.u32 %0, %0, %1;" : "+r"(acc[0]) : "r"(p[0]));
#pragma unroll
  for (int k = 1; k < 2 * N; k++) PBC_ASM("subc.cc.u32 %0, %0, %1;" : "+r"(acc[k]) : "r"(p[k]));
  PBC_ASM("subc.u32 %0, %0, 0;" : "+r"(acc[2 * N]));
}

// acc[0..2N] += p R
template <int N>
__device__ __forceinline__ void wide_add_pR(uint32_t* acc) {
  PBC_ASM("add.cc.u32 %0, %0, %1;" : "+r"(acc[N]) : "r"(c_fp.p[0]));
#pragma unroll
  for (int k = 1; k < N; k++) PBC_ASM("addc.cc.u32 %0, %0, %1;" : "+r"(acc[N + k]) : "r"(c_fp.p[k]));
  PBC_ASM("addc.u32 %0, %0, 0;" : "+r"(acc[2 * N]));
}

// acc[0..2N] -= p R if acc >= p R.  For 0 <= acc < 2 p R the result is below p R (acc[2N] = 0).
template <int N>
__device__ __forceinline__ void wide_sub_pR_if_ge(uint32_t* acc) {
  uint32_t d[N + 1], borrow;
  PBC_ASM("sub.cc.u32 %0, %1, %2;" : "=r"(d[0]) : "r"(acc[N]), "r"(c_fp.p[0]));
#pragma unroll
  for (int k = 1; k < N; k++) PBC_ASM("subc.cc.u32 %0, %1, %2;" : "=r"(d[k]) : "r"(acc[N + k]), "r"(c_fp.p[k]));
  PBC_ASM("subc.cc.u32 %0, %1, 0;" : "=r"(d[N]) : "r"(acc[2 * N]));
  PBC_ASM("subc.u32 %0, 0, 0;" : "=r"(borrow));   // 0 if acc >= p R
#pragma unroll
  for (int k = 0; k <= N; k++) acc[N + k] = borrow ? acc[N + k] : d[k];
}

// One row of the Montgomery reduction of a stored value: mont_round without the a b_i half.  The
// running sum starts as the low N words of t; the shift by one word rides on the odd-aligned chain.
template <int N>
__device__ __forceinline__ void redc_round(uint32_t* z, uint32_t* w, uint32_t& top, bool first) {
  uint32_t m;
  if (first) {
    m = w[0] * c_fp.np0;
    chain_mul<N>(z, c_fp.p + 1, m);
    top = 0;
  } else {
    // w[0] + z[1] is column 0; its carry enters the shifting chain at column 1
    PBC_ASM("add.cc.u32 %0, %0, %2; mul.lo.u32 %1, %0, %3;" : "+r"(w[0]), "=r"(m) : "r"(z[1]), "r"(c_fp.np0));
    chain_mad_shift<N>(z, c_fp.p + 1, m, top);
    top = carry_out();
  }
  chain_mad<N>(w, c_fp.p, m);
  PBC_ASM("addc.cc.u32 %0, %0, 0;" : "+r"(z[N - 1]));
  PBC_ASM("addc.u32 %0, %0, 0;" : "+r"(top));
}

// r = t / R mod p, fully reduced, for 0 <= t < 2 p R (t[0..2N], t[2N] the top word).
// (t_lo + M p) / R <= p is formed on the even / odd accumulators (N^2 IMAD.WIDE + N IMAD), t_hi < 2p is
// added, and the sum (< 3p) takes up to two conditional subtractions of p.  PASSES = 1 is for t < p R (a
// single product or square of reduced operands): t_hi < p, the sum is below 2p and one subtraction is enough.
template <int N, int PASSES = 2>
__device__ __forceinline__ void redc_wide(uint32_t* r, const uint32_t* t) {
  static_assert(N % 2 == 0, "even limb count");
  uint32_t x[N], y[N], top;
#pragma unroll
  for (int k = 0; k < N; k++) y[k] = t[k];
  redc_round<N>(x, y, top, true);
#pragma unroll
  for (int i = 1; i < N; i += 2) {
    redc_round<N>(y, x, top, false);
    if (i + 1 < N) redc_round<N>(x, y, top, false);
  }
  // s = (x >> 32) + y + top 2^(32N) + t_hi
  uint32_t s[N];
  PBC_ASM("add.cc.u32 %0, %1, %2;" : "=r"(s[0]) : "r"(x[1]), "r"(y[0]));
#pragma unroll
  for (int k = 1; k < N - 1; k++) PBC_ASM("addc.cc.u32 %0, %1, %2;" : "=r"(s[k]) : "r"(x[k + 1]), "r"(y[k]));
  PBC_ASM("addc.cc.u32 %0, %1, 0;" : "=r"(s[N - 1]) : "r"(y[N - 1]));
  PBC_ASM("addc.u32 %0, %0, 0;" : "+r"(top));
  PBC_ASM("add.cc.u32 %0, %0, %1;" : "+r"(s[0]) : "r"(t[N]));
#pragma unroll
  for (int k = 1; k < N; k++) PBC_ASM("addc.cc.u32 %0, %0, %1;" : "+r"(s[k]) : "r"(t[N + k]));
  PBC_ASM("addc.u32 %0, %0, %1;" : "+r"(top) : "r"(t[2 * N]));
#pragma unroll
  for (int pass = 0; pass < PASSES; pass++) {
    uint32_t d[N], dtop;
    PBC_ASM("sub.cc.u32 %0, %1, %2;" : "=r"(d[0]) : "r"(s[0]), "r"(c_fp.p[0]));
#pragma unroll
    for (int k = 1; k < N; k++) PBC_ASM("subc.cc.u32 %0, %1, %2;" : "=r"(d[k]) : "r"(s[k]), "r"(c_fp.p[k]));
    PBC_ASM("subc.cc.u32 %0, %1, 0;" : "=r"(dtop) : "r"(top));
    uint32_t borrow;
    PBC_ASM("subc.u32 %0, 0, 0;" : "=r"(borrow));   // 0 if s >= p
#pragma unroll
    for (int k = 0; k < N; k++) s[k] = borrow ? s[k] : d[k];
    top = borrow ? top : dtop;
  }
#pragma unroll
  for (int k = 0; k < N; k++) r[k] = s[k];
}

// ---------------------------------------------------------------------------------------------
// Row-wise squaring on the even / odd accumulators.  The cross products a_i a_j (i < j) are summed once,
// every one of them a single IMAD.WIDE.U32 with the carry in the flag, the sum is doubled by one carry chain
// and the diagonal a_i^2 is added as one run of N adjacent pairs: N(N-1)/2 + N products and about 3 N
// additions per limb pair, against N(N+1)/2 products each followed by an IADD3.X plus the per-column
// bookkeeping of the product-scanning squarer.
//
// Accumulators are indexed by absolute column: the pair (e[c], e[c+1]), c even, and (o[c], o[c+1]), c odd,
// receive the products whose low word lands on column c.  Row i holds a_i a_j for j = i+1 .. N-1: its odd
// chain starts at column 2i+1, its even chain at 2i+2, and its top product a_i a_{N-1} opens a new pair at
// column T = i+N-1.  The sum of rows 0..i is below 2^(32(i+N+1)), so nothing is carried beyond column T+1:
// the chain that does not own the new pair hands its carry to that pair's high word.  Columns 2i-1 and 2i
// are complete when row i starts; e and o are merged there and the merge carry enters the odd chain, so the
// live window shrinks as the finished words of p grow.
// ---------------------------------------------------------------------------------------------
template <int N, int I>
__device__ __forceinline__ void sqr_cross_row(uint32_t* p, uint32_t* e, uint32_t* o, const uint32_t* a) {
  constexpr int T = I + N - 1;
  constexpr bool kTopOdd = (T & 1) != 0;
  if constexpr (I == 0) {
    // nothing to add to yet: plain products
#pragma unroll
    for (int c = 1; c <= T; c += 2)
      PBC_ASM("mul.lo.u32 %0, %2, %3; mul.hi.u32 %1, %2, %3;" : "=r"(o[c]), "=r"(o[c + 1]) : "r"(a[0]), "r"(a[c]));
#pragma unroll
    for (int c = 2; c <= T; c += 2)
      PBC_ASM("mul.lo.u32 %0, %2, %3; mul.hi.u32 %1, %2, %3;" : "=r"(e[c]), "=r"(e[c + 1]) : "r"(a[0]), "r"(a[c]));
  } else {
    if constexpr (I == 1) {
      p[0] = 0;                 // no cross product lands on columns 0 and 1 of e
      p[1] = o[1];
      PBC_ASM("add.cc.u32 %0, %1, %2;" : "=r"(p[2]) : "r"(e[2]), "r"(o[2]));
    } else {
      PBC_ASM("add.cc.u32 %0, %1, %2;" : "=r"(p[2 * I - 1]) : "r"(e[2 * I - 1]), "r"(o[2 * I - 1]));
      PBC_ASM("addc.cc.u32 %0, %1, %2;" : "=r"(p[2 * I]) : "r"(e[2 * I]), "r"(o[2 * I]));
    }
    // odd columns: the merge carry enters at column 2I+1
#pragma unroll
    for (int c = 2 * I + 1; c <= T; c += 2) {
      if (c == T)
        PBC_ASM("madc.lo.cc.u32 %0, %2, %3, 0; madc.hi.cc.u32 %1, %2, %3, 0;"
                : "=r"(o[c]), "=r"(o[c + 1]) : "r"(a[I]), "r"(a[c - I]));
      else
        PBC_ASM("madc.lo.cc.u32 %0, %2, %3, %0; madc.hi.cc.u32 %1, %2, %3, %1;"
                : "+r"(o[c]), "+r"(o[c + 1]) : "r"(a[I]), "r"(a[c - I]));
    }
    uint32_t t = 0;
    if constexpr (!kTopOdd) t = carry_out();     // out of column T: the high word of the even chain's new pair
    // even columns
#pragma unroll
    for (int c = 2 * I + 2; c <= T; c += 2) {
      if (c == T && c == 2 * I + 2)
        PBC_ASM("mul.lo.u32 %0, %2, %3; mad.hi.u32 %1, %2, %3, %4;"
                : "=r"(e[c]), "=r"(e[c + 1]) : "r"(a[I]), "r"(a[c - I]), "r"(t));
      else if (c == T)
        PBC_ASM("madc.lo.cc.u32 %0, %2, %3, 0; madc.hi.u32 %1, %2, %3, %4;"
                : "=r"(e[c]), "=r"(e[c + 1]) : "r"(a[I]), "r"(a[c - I]), "r"(t));
      else if (c == 2 * I + 2)
        PBC_ASM("mad.lo.cc.u32 %0, %2, %3, %0; madc.hi.cc.u32 %1, %2, %3, %1;"
                : "+r"(e[c]), "+r"(e[c + 1]) : "r"(a[I]), "r"(a[c - I]));
      else
        PBC_ASM("madc.lo.cc.u32 %0, %2, %3, %0; madc.hi.cc.u32 %1, %2, %3, %1;"
                : "+r"(e[c]), "+r"(e[c + 1]) : "r"(a[I]), "r"(a[c - I]));
    }
    if constexpr (kTopOdd && 2 * I + 2 < T) PBC_ASM("addc.u32 %0, %0, 0;" : "+r"(o[T + 1]));
  }
  if constexpr (I + 2 < N) sqr_cross_row<N, I + 1>(p, e, o, a);
}

// p[0..2N) = a^2, exact.
template <int N>
__device__ __forceinline__ void sqr_wide(uint32_t* p, const uint32_t* a) {
  static_assert(N % 2 == 0 && N >= 4, "even limb count");
  uint32_t e[2 * N], o[2 * N];
  sqr_cross_row<N, 0>(p, e, o, a);
  // the last row (I = N-2) left columns 2N-3 and 2N-2; no pair of e reaches column 2N-2
  PBC_ASM("add.cc.u32 %0, %1, %2;" : "=r"(p[2 * N - 3]) : "r"(e[2 * N - 3]), "r"(o[2 * N - 3]));
  PBC_ASM("addc.cc.u32 %0, %1, 0;" : "=r"(p[2 * N - 2]) : "r"(o[2 * N - 2]));
  PBC_ASM("addc.u32 %0, 0, 0;" : "=r"(p[2 * N - 1]));
  // p = 2 p + sum a_i^2 2^(64 i)
  PBC_ASM("add.cc.u32 %0, %0, %0;" : "+r"(p[1]));
#pragma unroll
  for (int k = 2; k < 2 * N - 1; k++) PBC_ASM("addc.cc.u32 %0, %0, %0;" : "+r"(p[k]));
  PBC_ASM("addc.u32 %0, %0, %0;" : "+r"(p[2 * N - 1]));
  PBC_ASM("mad.lo.cc.u32 %0, %2, %2, %0; madc.hi.cc.u32 %1, %2, %2, %1;" : "+r"(p[0]), "+r"(p[1]) : "r"(a[0]));
#pragma unroll
  for (int i = 1; i < N; i++)
    PBC_ASM("madc.lo.cc.u32 %0, %2, %2, %0; madc.hi.cc.u32 %1, %2, %2, %1;"
            : "+r"(p[2 * i]), "+r"(p[2 * i + 1]) : "r"(a[i]));
}

// r = a^2/R mod p, input and output fully reduced.  r may alias a.  a^2 < p R: one conditional subtraction.
template <int N>
__device__ __forceinline__ void mont_sqr_os(uint32_t* r, const uint32_t* a) {
  uint32_t t[2 * N + 1];
  sqr_wide<N>(t, a);
  t[2 * N] = 0;
  redc_wide<N, 1>(r, t);
}

// ---------------------------------------------------------------------------------------------
// Product-scanning (column-wise) variant.  Every 32x32 product is one IMAD.WIDE.U32 with
// carry-OUT only (no carry-in: the .X form may issue at a lower rate), the carry
// is absorbed by an IADD3.X on the ALU pipe, so the FMA and ALU pipes alternate.  Two
// independent 96-bit accumulators (a*b and m*p) per column keep two dependency chains in flight.
// ---------------------------------------------------------------------------------------------
#define PBC_MAC3(t0, t1, t2, x, y)                                                           \
  PBC_ASM("mad.lo.cc.u32 %0, %3, %4, %0; madc.hi.cc.u32 %1, %3, %4, %1; addc.u32 %2, %2, 0;" \
          : "+r"(t0), "+r"(t1), "+r"(t2) : "r"(x), "r"(y))

template <int N, bool FULL>
__device__ __forceinline__ void mont_mul_ps(uint32_t* r, const uint32_t* a, const uint32_t* b) {
  uint32_t m[N], t[N];
  uint32_t u0 = 0, u1 = 0, u2 = 0, v0 = 0, v1 = 0, v2 = 0;
#pragma unroll
  for (int i = 0; i < N; i++) {
#pragma unroll
    for (int j = 0; j < i; j++) {
      PBC_MAC3(u0, u1, u2, a[j], b[i - j]);
      PBC_MAC3(v0, v1, v2, m[j], c_fp.p[i - j]);
    }
    PBC_MAC3(u0, u1, u2, a[i], b[0]);
    // v += u
    PBC_ASM("add.cc.u32 %0, %0, %3; addc.cc.u32 %1, %1, %4; addc.u32 %2, %2, %5;"
            : "+r"(v0), "+r"(v1), "+r"(v2) : "r"(u0), "r"(u1), "r"(u2));
    m[i] = v0 * c_fp.np0;
    PBC_MAC3(v0, v1, v2, m[i], c_fp.p[0]);   // v0 == 0 now
    v0 = v1; v1 = v2; v2 = 0;
    u0 = 0; u1 = 0; u2 = 0;
  }
#pragma unroll
  for (int i = N; i < 2 * N - 1; i++) {
#pragma unroll
    for (int j = i - N + 1; j < N; j++) {
      PBC_MAC3(u0, u1, u2, a[j], b[i - j]);
      PBC_MAC3(v0, v1, v2, m[j], c_fp.p[i - j]);
    }
    PBC_ASM("add.cc.u32 %0, %0, %3; addc.cc.u32 %1, %1, %4; addc.u32 %2, %2, %5;"
            : "+r"(v0), "+r"(v1), "+r"(v2) : "r"(u0), "r"(u1), "r"(u2));
    t[i - N] = v0;
    v0 = v1; v1 = v2; v2 = 0;
    u0 = 0; u1 = 0; u2 = 0;
  }
  t[N - 1] = v0;
  uint32_t top = v1;
  uint32_t d[N], borrow;
  PBC_ASM("sub.cc.u32 %0, %1, %2;" : "=r"(d[0]) : "r"(t[0]), "r"(c_fp.p[0]));
#pragma unroll
  for (int k = 1; k < N; k++)
    PBC_ASM("subc.cc.u32 %0, %1, %2;" : "=r"(d[k]) : "r"(t[k]), "r"(c_fp.p[k]));
  PBC_ASM("subc.u32 %0, 0, 0;" : "=r"(borrow));
  bool use_d = FULL ? (top != 0 || borrow == 0) : (borrow == 0);
#pragma unroll
  for (int k = 0; k < N; k++) r[k] = use_d ? d[k] : t[k];
}

// Squaring, product scanning: cross products a_j a_{i-j} (j < i-j) are accumulated once and
// doubled, the diagonal a_{i/2}^2 is added after.  N(N+1)/2 + N^2 products instead of 2 N^2.
// The columns below N (which make m[]) and from N on (which make t[]) are two loops, as in
// mont_mul_ps: as one loop of 2N - 1 columns nvcc does not unroll it for N = 16 and keeps m[] and t[]
// in a local-memory frame.
template <int N, bool FULL>
__device__ __forceinline__ void mont_sqr_ps(uint32_t* r, const uint32_t* a) {
  uint32_t m[N], t[N];
  uint32_t u0 = 0, u1 = 0, u2 = 0, v0 = 0, v1 = 0, v2 = 0;
#pragma unroll
  for (int i = 0; i < N; i++) {
#pragma unroll
    for (int j = 0; 2 * j < i; j++) PBC_MAC3(u0, u1, u2, a[j], a[i - j]);
#pragma unroll
    for (int j = 0; j < i; j++) PBC_MAC3(v0, v1, v2, m[j], c_fp.p[i - j]);
    // u = 2u (+ a_{i/2}^2), v += u
    PBC_ASM("add.cc.u32 %0, %0, %0; addc.cc.u32 %1, %1, %1; addc.u32 %2, %2, %2;"
            : "+r"(u0), "+r"(u1), "+r"(u2));
    if ((i & 1) == 0) PBC_MAC3(u0, u1, u2, a[i / 2], a[i / 2]);
    PBC_ASM("add.cc.u32 %0, %0, %3; addc.cc.u32 %1, %1, %4; addc.u32 %2, %2, %5;"
            : "+r"(v0), "+r"(v1), "+r"(v2) : "r"(u0), "r"(u1), "r"(u2));
    m[i] = v0 * c_fp.np0;
    PBC_MAC3(v0, v1, v2, m[i], c_fp.p[0]);
    v0 = v1; v1 = v2; v2 = 0;
    u0 = 0; u1 = 0; u2 = 0;
  }
#pragma unroll
  for (int i = N; i < 2 * N - 1; i++) {
#pragma unroll
    for (int j = i - N + 1; 2 * j < i; j++) PBC_MAC3(u0, u1, u2, a[j], a[i - j]);
#pragma unroll
    for (int j = i - N + 1; j < N; j++) PBC_MAC3(v0, v1, v2, m[j], c_fp.p[i - j]);
    PBC_ASM("add.cc.u32 %0, %0, %0; addc.cc.u32 %1, %1, %1; addc.u32 %2, %2, %2;"
            : "+r"(u0), "+r"(u1), "+r"(u2));
    if ((i & 1) == 0) PBC_MAC3(u0, u1, u2, a[i / 2], a[i / 2]);
    PBC_ASM("add.cc.u32 %0, %0, %3; addc.cc.u32 %1, %1, %4; addc.u32 %2, %2, %5;"
            : "+r"(v0), "+r"(v1), "+r"(v2) : "r"(u0), "r"(u1), "r"(u2));
    t[i - N] = v0;
    v0 = v1; v1 = v2; v2 = 0;
    u0 = 0; u1 = 0; u2 = 0;
  }
  t[N - 1] = v0;
  uint32_t top = v1;
  uint32_t d[N], borrow;
  PBC_ASM("sub.cc.u32 %0, %1, %2;" : "=r"(d[0]) : "r"(t[0]), "r"(c_fp.p[0]));
#pragma unroll
  for (int k = 1; k < N; k++)
    PBC_ASM("subc.cc.u32 %0, %1, %2;" : "=r"(d[k]) : "r"(t[k]), "r"(c_fp.p[k]));
  PBC_ASM("subc.u32 %0, 0, 0;" : "=r"(borrow));
  bool use_d = FULL ? (top != 0 || borrow == 0) : (borrow == 0);
#pragma unroll
  for (int k = 0; k < N; k++) r[k] = use_d ? d[k] : t[k];
}

// The multiplier the kernels use.  Operand scanning for products.  For squares the 16-limb full-width field
// (type A) takes the row-wise squarer, whose additions ride on the carry flag of the products; the other
// widths keep product scanning.  Both squarers issue N(N+1)/2 + N^2 IMAD.WIDE (408 for N = 16, against 528).
template <int N, bool FULL>
__device__ __forceinline__ void fp_mul(uint32_t* r, const uint32_t* a, const uint32_t* b) {
  mont_mul<N, FULL>(r, a, b);
}
template <int N, bool FULL>
__device__ __forceinline__ void fp_sqr(uint32_t* r, const uint32_t* a) {
  if constexpr (N == 16 && FULL) mont_sqr_os<N>(r, a);
  else mont_sqr_ps<N, FULL>(r, a);
}

// ---------------------------------------------------------------------------------------------
// additive operations (arith/montfp.c:220-330), branch-free conditional correction
// ---------------------------------------------------------------------------------------------
template <int N, bool FULL>
__device__ __forceinline__ void fp_add(uint32_t* r, const uint32_t* a, const uint32_t* b) {
  uint32_t t[N], d[N], c = 0, borrow;
  PBC_ASM("add.cc.u32 %0, %1, %2;" : "=r"(t[0]) : "r"(a[0]), "r"(b[0]));
#pragma unroll
  for (int k = 1; k < N; k++)
    PBC_ASM("addc.cc.u32 %0, %1, %2;" : "=r"(t[k]) : "r"(a[k]), "r"(b[k]));
  if (FULL) c = carry_out();
  PBC_ASM("sub.cc.u32 %0, %1, %2;" : "=r"(d[0]) : "r"(t[0]), "r"(c_fp.p[0]));
#pragma unroll
  for (int k = 1; k < N; k++)
    PBC_ASM("subc.cc.u32 %0, %1, %2;" : "=r"(d[k]) : "r"(t[k]), "r"(c_fp.p[k]));
  PBC_ASM("subc.u32 %0, 0, 0;" : "=r"(borrow));
  bool use_d = FULL ? (c != 0 || borrow == 0) : (borrow == 0);
#pragma unroll
  for (int k = 0; k < N; k++) r[k] = use_d ? d[k] : t[k];
}

template <int N>
__device__ __forceinline__ void fp_sub(uint32_t* r, const uint32_t* a, const uint32_t* b) {
  uint32_t t[N], borrow;
  PBC_ASM("sub.cc.u32 %0, %1, %2;" : "=r"(t[0]) : "r"(a[0]), "r"(b[0]));
#pragma unroll
  for (int k = 1; k < N; k++)
    PBC_ASM("subc.cc.u32 %0, %1, %2;" : "=r"(t[k]) : "r"(a[k]), "r"(b[k]));
  PBC_ASM("subc.u32 %0, 0, 0;" : "=r"(borrow));   // all-ones when a < b
  // add back p & mask
  PBC_ASM("add.cc.u32 %0, %1, %2;" : "=r"(r[0]) : "r"(t[0]), "r"(c_fp.p[0] & borrow));
#pragma unroll
  for (int k = 1; k < N; k++)
    PBC_ASM("addc.cc.u32 %0, %1, %2;" : "=r"(r[k]) : "r"(t[k]), "r"(c_fp.p[k] & borrow));
}

template <int N>
__device__ __forceinline__ bool fp_is_zero(const uint32_t* a) {
  uint32_t o = 0;
#pragma unroll
  for (int k = 0; k < N; k++) o |= a[k];
  return o == 0;
}

template <int N>
__device__ __forceinline__ void fp_neg(uint32_t* r, const uint32_t* a) {
  // p - a, and 0 stays 0
  uint32_t mask = fp_is_zero<N>(a) ? 0u : 0xffffffffu;
  uint32_t t[N];
  PBC_ASM("sub.cc.u32 %0, %1, %2;" : "=r"(t[0]) : "r"(c_fp.p[0]), "r"(a[0]));
#pragma unroll
  for (int k = 1; k < N; k++)
    PBC_ASM("subc.cc.u32 %0, %1, %2;" : "=r"(t[k]) : "r"(c_fp.p[k]), "r"(a[k]));
#pragma unroll
  for (int k = 0; k < N; k++) r[k] = t[k] & mask;
}

// r = a/2 mod p  (arith/montfp.c:282-301)
template <int N, bool FULL>
__device__ __forceinline__ void fp_halve(uint32_t* r, const uint32_t* a) {
  uint32_t mask = (a[0] & 1u) ? 0xffffffffu : 0u;
  uint32_t t[N], c;
  PBC_ASM("add.cc.u32 %0, %1, %2;" : "=r"(t[0]) : "r"(a[0]), "r"(c_fp.p[0] & mask));
#pragma unroll
  for (int k = 1; k < N; k++)
    PBC_ASM("addc.cc.u32 %0, %1, %2;" : "=r"(t[k]) : "r"(a[k]), "r"(c_fp.p[k] & mask));
  c = carry_out();
#pragma unroll
  for (int k = 0; k < N - 1; k++) r[k] = __funnelshift_r(t[k], t[k + 1], 1);
  r[N - 1] = __funnelshift_r(t[N - 1], c, 1);
}

template <int N>
__device__ __forceinline__ bool fp_eq(const uint32_t* a, const uint32_t* b) {
  uint32_t o = 0;
#pragma unroll
  for (int k = 0; k < N; k++) o |= a[k] ^ b[k];
  return o == 0;
}

}  // namespace pbcb200
