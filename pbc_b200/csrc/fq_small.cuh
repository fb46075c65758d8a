// fq_small.cuh -- the 158/159-bit base field of the Type F and Type D curves on five 32-bit limbs.
//
// Device replacement for arith/montfp.c on 3 x 64-bit limbs (the reference's F_q for f.param and
// d159.param): values are held as x * 2^160 mod q on FIVE 32-bit words (the reference rounds up to
// 192 bits; 25 instead of 36 word products per multiplication).  q < 2^159, so one conditional
// subtraction keeps everything canonical (FULL = false in fp.cuh).  Multiplication is the
// product-scanning Montgomery form of fp.cuh (works for odd limb counts).
//
// Tower elements (F_q^2, F_q^3, F_q^6, F_q^12) are plain structs of Fq; the compiler keeps the
// ones that are passed by pointer to the out-of-line tower routines in the per-thread local
// frame (LDL/STL, warp-interleaved 128-byte lines, L1-resident) -- the same role the explicit
// shared-memory slots play for the 512-bit field of Type A.
#pragma once
#include "slots.cuh"

namespace pbcb200 {

// PBC_NS: 32-bit limbs of the small field: 5 here, 8 in the wide instance below.
// PBC_FQ_WIDE = 1: the eight-limb instance of type D for 160- to 255-bit q (engine_d_wide.cu, its own
// translation unit and namespace): the wire width is a run-time constant there, and q = 1 mod 8 takes
// Tonelli-Shanks square roots.
#ifndef PBC_FQ_WIDE
#define PBC_FQ_WIDE 0
#endif
#ifndef PBC_NS
#define PBC_NS 5
#endif
constexpr int kNS = PBC_NS;    // 32-bit limbs
#if !PBC_FQ_WIDE
constexpr int kWS = 20;        // wire bytes per coordinate (arith/montfp.c:577)
__device__ __forceinline__ int fq_wb() { return kWS; }
#endif

// constants of the wide instance only: the wire width ceil(bits(q)/8) and, for q = 1 mod 8, the
// Tonelli-Shanks data (q - 1 = 2^s Q with Q odd, c = z^Q for a quadratic non-residue z, Montgomery form;
// the exponent (Q - 1)/2 sits in HashConsts::exp)
template <int NS>
struct FqWideConstsT {
  uint32_t wb;
  uint32_t ts_s;
  uint32_t pad[2];
  uint32_t ts_c[NS];
};
#if PBC_FQ_WIDE
__constant__ FqWideConstsT<kNS> c_fqx;
__device__ __forceinline__ int fq_wb() { return (int)c_fqx.wb; }
#endif
// coordinate width of the width-generic kernels: W, or for W = 0 the run-time width of the wide instance
template <int W>
__device__ __forceinline__ int wire_w() { return W ? W : fq_wb(); }

struct Fq { uint32_t v[kNS]; };

// One out-of-line copy of the multiplier and of the squarer, operands and result by value (five
// registers each way).  The tower routines contain dozens of products; fully inlined they outgrow the
// instruction cache (instruction fetch becomes the top stall of k_d_miller).  The five-limb multiplier is
// the row-wise product + row-wise reduction (fq_mul_os below: 55 products, about 100 instructions; a b < q R
// is all it needs, operands below 2q and q), the squarer the column-wise one of fp.cuh (40 products).
__device__ __forceinline__ void fq_mul_os(Fq& r, const Fq& a, const Fq& b);
__device__ __noinline__ Fq fq_mul_call(Fq a, Fq b) {
  Fq r;
  if constexpr (kNS % 2 == 0) mont_mul<kNS + (kNS & 1), false>(r.v, a.v, b.v);
  else fq_mul_os(r, a, b);
  return r;
}
__device__ __noinline__ Fq fq_sqr_call(Fq a) {
  Fq r;
  if constexpr (kNS % 2 == 0) mont_mul<kNS + (kNS & 1), false>(r.v, a.v, a.v);
  else mont_sqr_ps<kNS, false>(r.v, a.v);
  return r;
}
__device__ __forceinline__ void fq_mul(Fq& r, const Fq& a, const Fq& b) { r = fq_mul_call(a, b); }
__device__ __forceinline__ void fq_sqr(Fq& r, const Fq& a) { r = fq_sqr_call(a); }
__device__ __forceinline__ void fq_add(Fq& r, const Fq& a, const Fq& b) { fp_add<kNS, false>(r.v, a.v, b.v); }
__device__ __forceinline__ void fq_sub(Fq& r, const Fq& a, const Fq& b) { fp_sub<kNS>(r.v, a.v, b.v); }
__device__ __forceinline__ void fq_dbl(Fq& r, const Fq& a) { fp_add<kNS, false>(r.v, a.v, a.v); }
__device__ __forceinline__ void fq_neg(Fq& r, const Fq& a) { fp_neg<kNS>(r.v, a.v); }
__device__ __forceinline__ void fq_halve(Fq& r, const Fq& a) { fp_halve<kNS, false>(r.v, a.v); }
__device__ __forceinline__ bool fq_is_zero(const Fq& a) { return fp_is_zero<kNS>(a.v); }
__device__ __forceinline__ bool fq_eq(const Fq& a, const Fq& b) { return fp_eq<kNS>(a.v, b.v); }
__device__ __forceinline__ void fq_zero(Fq& r) {
#pragma unroll
  for (int k = 0; k < kNS; k++) r.v[k] = 0;
}
__device__ __forceinline__ void fq_set(Fq& r, const uint32_t* c) {
#pragma unroll
  for (int k = 0; k < kNS; k++) r.v[k] = c[k];
}
__device__ __forceinline__ void fq_one(Fq& r) { fq_set(r, c_fp.one); }

// ---------------------------------------------------------------------------------------------
// Lazy reduction: double-width (2 kNS words) unreduced products, combined with plain carry chains and
// reduced once.  fq_redc needs its input below q R (R = 2^(32 kNS)); the result is canonical.
// ---------------------------------------------------------------------------------------------
struct FqW { uint32_t v[2 * kNS]; };

// t = a b, schoolbook by columns (kNS^2 products)
__device__ __noinline__ FqW fq_mulw_call(Fq a, Fq b) {
  FqW t;
  uint32_t u0 = 0, u1 = 0, u2 = 0;
#pragma unroll
  for (int i = 0; i < 2 * kNS - 1; i++) {
#pragma unroll
    for (int j = (i < kNS ? 0 : i - kNS + 1); j <= (i < kNS ? i : kNS - 1); j++) PBC_MAC3(u0, u1, u2, a.v[j], b.v[i - j]);
    t.v[i] = u0;
    u0 = u1; u1 = u2; u2 = 0;
  }
  t.v[2 * kNS - 1] = u0;
  return t;
}
// (t + m q) / R with m chosen so the division is exact (Montgomery reduction), then one conditional
// subtraction: canonical for t < q R.
__device__ __noinline__ Fq fq_redc_call(FqW t) {
  uint32_t m[kNS], o[kNS];
  uint32_t v0 = 0, v1 = 0, v2 = 0;
#pragma unroll
  for (int i = 0; i < kNS; i++) {
#pragma unroll
    for (int j = 0; j < i; j++) PBC_MAC3(v0, v1, v2, m[j], c_fp.p[i - j]);
    PBC_ASM("add.cc.u32 %0, %0, %3; addc.cc.u32 %1, %1, 0; addc.u32 %2, %2, 0;" : "+r"(v0), "+r"(v1), "+r"(v2) : "r"(t.v[i]));
    m[i] = v0 * c_fp.np0;
    PBC_MAC3(v0, v1, v2, m[i], c_fp.p[0]);
    v0 = v1; v1 = v2; v2 = 0;
  }
#pragma unroll
  for (int i = kNS; i < 2 * kNS; i++) {
#pragma unroll
    for (int j = i - kNS + 1; j < kNS; j++) PBC_MAC3(v0, v1, v2, m[j], c_fp.p[i - j]);
    PBC_ASM("add.cc.u32 %0, %0, %3; addc.cc.u32 %1, %1, 0; addc.u32 %2, %2, 0;" : "+r"(v0), "+r"(v1), "+r"(v2) : "r"(t.v[i]));
    o[i - kNS] = v0;
    v0 = v1; v1 = v2; v2 = 0;
  }
  Fq r;
  uint32_t d[kNS], borrow;
  PBC_ASM("sub.cc.u32 %0, %1, %2;" : "=r"(d[0]) : "r"(o[0]), "r"(c_fp.p[0]));
#pragma unroll
  for (int k = 1; k < kNS; k++) PBC_ASM("subc.cc.u32 %0, %1, %2;" : "=r"(d[k]) : "r"(o[k]), "r"(c_fp.p[k]));
  PBC_ASM("subc.u32 %0, 0, 0;" : "=r"(borrow));
  bool use_d = v0 != 0 || borrow == 0;
#pragma unroll
  for (int k = 0; k < kNS; k++) r.v[k] = use_d ? d[k] : o[k];
  return r;
}
// the same for t < 2 q R (sums of several double-width terms): the quotient is below 3q, two
// conditional subtractions
__device__ __noinline__ Fq fq_redc2_call(FqW t) {
  Fq r = fq_redc_call(t);
  // fq_redc_call subtracted q once if the value was >= q (or overflowed a limb); one more may be due.
  // It cannot tell 2q <= x < 3q from q <= x < 2q by itself, so repeat the comparison here.
  uint32_t d[kNS], borrow;
  PBC_ASM("sub.cc.u32 %0, %1, %2;" : "=r"(d[0]) : "r"(r.v[0]), "r"(c_fp.p[0]));
#pragma unroll
  for (int k = 1; k < kNS; k++) PBC_ASM("subc.cc.u32 %0, %1, %2;" : "=r"(d[k]) : "r"(r.v[k]), "r"(c_fp.p[k]));
  PBC_ASM("subc.u32 %0, 0, 0;" : "=r"(borrow));
#pragma unroll
  for (int k = 0; k < kNS; k++) r.v[k] = borrow == 0 ? d[k] : r.v[k];
  return r;
}
__device__ __forceinline__ void fqw_add(FqW& r, const FqW& a, const FqW& b) {
  PBC_ASM("add.cc.u32 %0, %1, %2;" : "=r"(r.v[0]) : "r"(a.v[0]), "r"(b.v[0]));
#pragma unroll
  for (int k = 1; k < 2 * kNS; k++) PBC_ASM("addc.cc.u32 %0, %1, %2;" : "=r"(r.v[k]) : "r"(a.v[k]), "r"(b.v[k]));
}
__device__ __forceinline__ void fqw_sub(FqW& r, const FqW& a, const FqW& b) {
  PBC_ASM("sub.cc.u32 %0, %1, %2;" : "=r"(r.v[0]) : "r"(a.v[0]), "r"(b.v[0]));
#pragma unroll
  for (int k = 1; k < 2 * kNS; k++) PBC_ASM("subc.cc.u32 %0, %1, %2;" : "=r"(r.v[k]) : "r"(a.v[k]), "r"(b.v[k]));
}
// ---- inline double-width product and reduction (the slot-machine kernels, pairing_f_slots.cuh) ----
// t = a b (25 products), operand scanning on two accumulators.  The product a_j b_i is a 64-bit value
// at word column c = i + j; products on EVEN columns are accumulated in E (pairs (E[c], E[c+1])),
// products on ODD columns in O, so that within one row (one b_i) each accumulator sees a run of
// ADJACENT pairs: one IMAD.WIDE.U32 per product with the carry handed from pair to pair in the
// carry flag, no per-product carry word.  The pair two columns above a row's run has not been touched
// by earlier rows (row i' reaches column i' + 4 at most), so either the run's top pair is fresh and
// cannot overflow, or one addc into the fresh word above it absorbs the carry.  t = E + O at the end.
// The column-wise form this replaces (fq_mulw_call in fq_small.cuh) compiles to ~95 instructions per
// product of two elements -- IMAD.WIDE + IADD3.X per product plus SEL / IMAD.MOV / IMAD.X to move
// carries and re-align register pairs at every column, and those moves take multiplier-pipe slots; this one to ~40.
#define PBC_MADW_FIRST(lo, hi, x, y) PBC_ASM("mad.lo.cc.u32 %0, %2, %3, %0; madc.hi.cc.u32 %1, %2, %3, %1;" : "+r"(lo), "+r"(hi) : "r"(x), "r"(y))
#define PBC_MADW_NEXT(lo, hi, x, y) PBC_ASM("madc.lo.cc.u32 %0, %2, %3, %0; madc.hi.cc.u32 %1, %2, %3, %1;" : "+r"(lo), "+r"(hi) : "r"(x), "r"(y))
// (lo, hi) = x y.  Written as a multiply-add of zero: ptxas turns mad.lo.cc + madc.hi into ONE IMAD.WIDE.U32, while
// mul.lo + mul.hi stayed an IMAD + IMAD.HI pair in places.  Clobbers the carry flag (no run is in flight where a
// row starts).  Tiling the accumulators with nine plain products first, to avoid the "(carry word, 0)" top pairs and
// their zeroing moves, did not pay: ptxas moved other additions onto the multiplier pipe instead (IMAD.X / IMAD).
#define PBC_MULW_PAIR(lo, hi, x, y) PBC_ASM("mad.lo.cc.u32 %0, %2, %3, 0; madc.hi.u32 %1, %2, %3, 0;" : "=r"(lo), "=r"(hi) : "r"(x), "r"(y))
#define PBC_CARRY_TO(w) PBC_ASM("addc.u32 %0, 0, 0;" : "=r"(w))
#if PBC_NS == 5
__device__ __forceinline__ void fqw_mul(FqW& t, const Fq& a, const Fq& b) {
  static_assert(kNS == 5, "the row schedule below is written out for five limbs");
  uint32_t E[10], O[10];
  const uint32_t* x = a.v;
  const uint32_t* y = b.v;
  // row 0: every pair is fresh
  PBC_MULW_PAIR(E[0], E[1], x[0], y[0]);
  PBC_MULW_PAIR(E[2], E[3], x[2], y[0]);
  PBC_MULW_PAIR(E[4], E[5], x[4], y[0]);
  PBC_MULW_PAIR(O[1], O[2], x[1], y[0]);
  PBC_MULW_PAIR(O[3], O[4], x[3], y[0]);
  // row 1: E columns 2, 4 (+ carry into the fresh E[6]); O columns 1, 3, 5 (top pair fresh)
  O[5] = 0; O[6] = 0;
  PBC_MADW_FIRST(E[2], E[3], x[1], y[1]);
  PBC_MADW_NEXT(E[4], E[5], x[3], y[1]);
  PBC_CARRY_TO(E[6]);
  PBC_MADW_FIRST(O[1], O[2], x[0], y[1]);
  PBC_MADW_NEXT(O[3], O[4], x[2], y[1]);
  PBC_MADW_NEXT(O[5], O[6], x[4], y[1]);
  // row 2: E columns 2, 4, 6 (E[6] holds one carry bit, E[7] fresh: no overflow); O columns 3, 5 (+ carry into O[7])
  E[7] = 0;
  PBC_MADW_FIRST(E[2], E[3], x[0], y[2]);
  PBC_MADW_NEXT(E[4], E[5], x[2], y[2]);
  PBC_MADW_NEXT(E[6], E[7], x[4], y[2]);
  PBC_MADW_FIRST(O[3], O[4], x[1], y[2]);
  PBC_MADW_NEXT(O[5], O[6], x[3], y[2]);
  PBC_CARRY_TO(O[7]);
  // row 3: E columns 4, 6 (+ carry into E[8]); O columns 3, 5, 7 (O[8] fresh)
  O[8] = 0;
  PBC_MADW_FIRST(E[4], E[5], x[1], y[3]);
  PBC_MADW_NEXT(E[6], E[7], x[3], y[3]);
  PBC_CARRY_TO(E[8]);
  PBC_MADW_FIRST(O[3], O[4], x[0], y[3]);
  PBC_MADW_NEXT(O[5], O[6], x[2], y[3]);
  PBC_MADW_NEXT(O[7], O[8], x[4], y[3]);
  // row 4: E columns 4, 6, 8 (E[9] fresh); O columns 5, 7 (+ carry into O[9])
  E[9] = 0;
  PBC_MADW_FIRST(E[4], E[5], x[0], y[4]);
  PBC_MADW_NEXT(E[6], E[7], x[2], y[4]);
  PBC_MADW_NEXT(E[8], E[9], x[4], y[4]);
  PBC_MADW_FIRST(O[5], O[6], x[1], y[4]);
  PBC_MADW_NEXT(O[7], O[8], x[3], y[4]);
  PBC_CARRY_TO(O[9]);
  // t = E + O   (O[0] does not exist; the sum is below 2^320: no carry out of word 9)
  t.v[0] = E[0];
  PBC_ASM("add.cc.u32 %0, %1, %2;" : "=r"(t.v[1]) : "r"(E[1]), "r"(O[1]));
#pragma unroll
  for (int k = 2; k < 9; k++) PBC_ASM("addc.cc.u32 %0, %1, %2;" : "=r"(t.v[k]) : "r"(E[k]), "r"(O[k]));
  PBC_ASM("addc.u32 %0, %1, %2;" : "=r"(t.v[9]) : "r"(E[9]), "r"(O[9]));
}
#else
// any even limb count (the wide instance): the operand-scanning double-width product of fp.cuh
__device__ __forceinline__ void fqw_mul(FqW& t, const Fq& a, const Fq& b) { mul_wide<kNS>(t.v, a.v, b.v); }
#endif
// Montgomery reduction of t < 2 q R to the canonical residue (two conditional subtractions)
__device__ __forceinline__ void fqw_redc2(Fq& r, const FqW& t) {
  uint32_t m[kNS], o[kNS];
  uint32_t v0 = 0, v1 = 0, v2 = 0;
#pragma unroll
  for (int i = 0; i < kNS; i++) {
#pragma unroll
    for (int j = 0; j < i; j++) PBC_MAC3(v0, v1, v2, m[j], c_fp.p[i - j]);
    PBC_ASM("add.cc.u32 %0, %0, %3; addc.cc.u32 %1, %1, 0; addc.u32 %2, %2, 0;" : "+r"(v0), "+r"(v1), "+r"(v2) : "r"(t.v[i]));
    m[i] = v0 * c_fp.np0;
    PBC_MAC3(v0, v1, v2, m[i], c_fp.p[0]);
    v0 = v1; v1 = v2; v2 = 0;
  }
#pragma unroll
  for (int i = kNS; i < 2 * kNS; i++) {
#pragma unroll
    for (int j = i - kNS + 1; j < kNS; j++) PBC_MAC3(v0, v1, v2, m[j], c_fp.p[i - j]);
    PBC_ASM("add.cc.u32 %0, %0, %3; addc.cc.u32 %1, %1, 0; addc.u32 %2, %2, 0;" : "+r"(v0), "+r"(v1), "+r"(v2) : "r"(t.v[i]));
    o[i - kNS] = v0;
    v0 = v1; v1 = v2; v2 = 0;
  }
  // value = o + v0 2^160 < 3 q: subtract q while it is >= q
  uint32_t d[kNS], borrow;
  PBC_ASM("sub.cc.u32 %0, %1, %2;" : "=r"(d[0]) : "r"(o[0]), "r"(c_fp.p[0]));
#pragma unroll
  for (int k = 1; k < kNS; k++) PBC_ASM("subc.cc.u32 %0, %1, %2;" : "=r"(d[k]) : "r"(o[k]), "r"(c_fp.p[k]));
  PBC_ASM("subc.u32 %0, 0, 0;" : "=r"(borrow));
  bool use_d = v0 != 0 || borrow == 0;
#pragma unroll
  for (int k = 0; k < kNS; k++) o[k] = use_d ? d[k] : o[k];
  PBC_ASM("sub.cc.u32 %0, %1, %2;" : "=r"(d[0]) : "r"(o[0]), "r"(c_fp.p[0]));
#pragma unroll
  for (int k = 1; k < kNS; k++) PBC_ASM("subc.cc.u32 %0, %1, %2;" : "=r"(d[k]) : "r"(o[k]), "r"(c_fp.p[k]));
  PBC_ASM("subc.u32 %0, 0, 0;" : "=r"(borrow));
#pragma unroll
  for (int k = 0; k < kNS; k++) r.v[k] = borrow == 0 ? d[k] : o[k];
}

// a + b without reduction (the caller knows the sum fits the limbs)
__device__ __forceinline__ void fq_add_nr(Fq& r, const Fq& a, const Fq& b) {
  PBC_ASM("add.cc.u32 %0, %1, %2;" : "=r"(r.v[0]) : "r"(a.v[0]), "r"(b.v[0]));
#pragma unroll
  for (int k = 1; k < kNS; k++) PBC_ASM("addc.cc.u32 %0, %1, %2;" : "=r"(r.v[k]) : "r"(a.v[k]), "r"(b.v[k]));
}

// ---------------------------------------------------------------------------------------------
// Accumulating products: sums of several 5 x 5 products kept UNMERGED on the even / odd
// accumulators and merged once.  In the first slot kernels IADD3 outnumbered IMAD.WIDE in the instruction
// stream -- every product paid a ten-word merge of its two accumulators plus one or two
// ten-word additions into the running sums of an F_q^2 product, and the warps (two per scheduler) spent
// 1.7 cycles per issue waiting on those serial carry chains.  Here each of the three sums of an F_q^2
// Karatsuba product (a0 b0, a1 b1, (a0 + a1)(b0 + b1)) lives on one FqAcc across all the terms of a
// coefficient: a product adds 25 IMAD.WIDE and nine carry captures, the merge is paid once per sum.
//   value = E + O + sum_p K[p] 2^(32 (5 + p));  O[0] stays zero.
// Row i of a product (all a_j b_i) puts a_0, a_2, a_4 on the accumulator of i's parity (words i .. i+5) and
// a_1, a_3 on the other (words i+1 .. i+4); the carry out of either run is counted in K at the word
// above the run.  The total stays below 2^320 (callers' bounds), so nothing is carried out of word 9.
// ---------------------------------------------------------------------------------------------
struct FqAcc { uint32_t E[10], O[10], K[5]; };

#define PBC_CARRY_ADD(w) PBC_ASM("addc.u32 %0, %0, 0;" : "+r"(w))

// c = a b (the schedule of fqw_mul: every word of E and O is written, fresh words take the carries); K is
// NOT written: the first fqa_mac after it sets K (SETK), a lone product is merged with fqa_merge<false>.
#if PBC_NS == 5
__device__ __forceinline__ void fqa_mul(FqAcc& c, const Fq& a, const Fq& b) {
  static_assert(kNS == 5, "the row schedule below is written out for five limbs");
  uint32_t* E = c.E;
  uint32_t* O = c.O;
  const uint32_t* x = a.v;
  const uint32_t* y = b.v;
  PBC_MULW_PAIR(E[0], E[1], x[0], y[0]);
  PBC_MULW_PAIR(E[2], E[3], x[2], y[0]);
  PBC_MULW_PAIR(E[4], E[5], x[4], y[0]);
  PBC_MULW_PAIR(O[1], O[2], x[1], y[0]);
  PBC_MULW_PAIR(O[3], O[4], x[3], y[0]);
  O[0] = 0; O[5] = 0; O[6] = 0;
  PBC_MADW_FIRST(E[2], E[3], x[1], y[1]);
  PBC_MADW_NEXT(E[4], E[5], x[3], y[1]);
  PBC_CARRY_TO(E[6]);
  PBC_MADW_FIRST(O[1], O[2], x[0], y[1]);
  PBC_MADW_NEXT(O[3], O[4], x[2], y[1]);
  PBC_MADW_NEXT(O[5], O[6], x[4], y[1]);
  E[7] = 0;
  PBC_MADW_FIRST(E[2], E[3], x[0], y[2]);
  PBC_MADW_NEXT(E[4], E[5], x[2], y[2]);
  PBC_MADW_NEXT(E[6], E[7], x[4], y[2]);
  PBC_MADW_FIRST(O[3], O[4], x[1], y[2]);
  PBC_MADW_NEXT(O[5], O[6], x[3], y[2]);
  PBC_CARRY_TO(O[7]);
  O[8] = 0;
  PBC_MADW_FIRST(E[4], E[5], x[1], y[3]);
  PBC_MADW_NEXT(E[6], E[7], x[3], y[3]);
  PBC_CARRY_TO(E[8]);
  PBC_MADW_FIRST(O[3], O[4], x[0], y[3]);
  PBC_MADW_NEXT(O[5], O[6], x[2], y[3]);
  PBC_MADW_NEXT(O[7], O[8], x[4], y[3]);
  E[9] = 0;
  PBC_MADW_FIRST(E[4], E[5], x[0], y[4]);
  PBC_MADW_NEXT(E[6], E[7], x[2], y[4]);
  PBC_MADW_NEXT(E[8], E[9], x[4], y[4]);
  PBC_MADW_FIRST(O[5], O[6], x[1], y[4]);
  PBC_MADW_NEXT(O[7], O[8], x[3], y[4]);
  PBC_CARRY_TO(O[9]);
}
#endif
// c += a b.  SETK: the first accumulation after fqa_mul -- the first capture at each word writes K.
// (K[i+1] is first touched by row i's long run, K[0] by row 0's short run.)
template <bool SETK>
__device__ __forceinline__ void fqa_mac(FqAcc& c, const Fq& a, const Fq& b) {
  const uint32_t* x = a.v;
  const uint32_t* y = b.v;
#pragma unroll
  for (int i = 0; i < kNS; i++) {
    uint32_t* S = (i & 1) ? c.O : c.E;
    uint32_t* T = (i & 1) ? c.E : c.O;
    PBC_MADW_FIRST(S[i], S[i + 1], x[0], y[i]);
    PBC_MADW_NEXT(S[i + 2], S[i + 3], x[2], y[i]);
    PBC_MADW_NEXT(S[i + 4], S[i + 5], x[4], y[i]);
    if (i < 4) {                                            // carry into word i + 6
      if (SETK) PBC_CARRY_TO(c.K[i + 1]); else PBC_CARRY_ADD(c.K[i + 1]);
    }
    PBC_MADW_FIRST(T[i + 1], T[i + 2], x[1], y[i]);
    PBC_MADW_NEXT(T[i + 3], T[i + 4], x[3], y[i]);
    if (SETK && i == 0) PBC_CARRY_TO(c.K[0]); else PBC_CARRY_ADD(c.K[i]);   // carry into word i + 5
  }
}
// t = the value of c.  HASK = false: straight after fqa_mul (K not written).
template <bool HASK>
__device__ __forceinline__ void fqa_merge(FqW& t, const FqAcc& c) {
  t.v[0] = c.E[0];
  PBC_ASM("add.cc.u32 %0, %1, %2;" : "=r"(t.v[1]) : "r"(c.E[1]), "r"(c.O[1]));
#pragma unroll
  for (int k = 2; k < 9; k++) PBC_ASM("addc.cc.u32 %0, %1, %2;" : "=r"(t.v[k]) : "r"(c.E[k]), "r"(c.O[k]));
  PBC_ASM("addc.u32 %0, %1, %2;" : "=r"(t.v[9]) : "r"(c.E[9]), "r"(c.O[9]));
  if (HASK) {
    PBC_ASM("add.cc.u32 %0, %0, %1;" : "+r"(t.v[5]) : "r"(c.K[0]));
#pragma unroll
    for (int k = 1; k < 4; k++) PBC_ASM("addc.cc.u32 %0, %0, %1;" : "+r"(t.v[5 + k]) : "r"(c.K[k]));
    PBC_ASM("addc.u32 %0, %0, %1;" : "+r"(t.v[9]) : "r"(c.K[4]));
  }
}

// Montgomery reduction by rows (operand scanning): r = t / R mod q, canonical.  TWO = false: t < q R (one
// conditional subtraction); TWO = true: t < 2 q R.
// The quotient digits depend on the LOW half of t only: X = (t_lo + M q) / R with M = sum m_i 2^(32 i) is
// computed on a sliding pair of even / odd accumulators -- row i adds m_i (q_0, q_2, q_4) to the
// accumulator whose low word is column i (that word becomes zero and drops out) and m_i (q_1, q_3) to the
// other one -- and X <= q, so no run ever carries out of its fresh top pair except the short run into
// the word above it, which the next row's top pair takes as its addend.  r = X + t_hi - {0, q, 2q}.
// 25 IMAD.WIDE + 5 IMAD and about 30 additions; the column-wise fqw_redc2 needs about 60 and a serial
// chain of three-word column sums.
#if PBC_NS == 5
template <bool TWO>
__device__ __forceinline__ void fqw_redc_os(Fq& r, const FqW& t) {
  static_assert(kNS == 5, "written out for five limbs");
  const uint32_t* q = c_fp.p;
  // a: the accumulator with its low word at the current column (six words), b: the other (four words above
  // that column), top: the carry out of b's run, one word above it.  Words are named by absolute column.
  uint32_t E[10], O[10], top, m;
  // row 0: E = t_lo + m (q0, q2, q4) on words 0..5, O = m (q1, q3) on words 1..4
  m = t.v[0] * c_fp.np0;
  PBC_ASM("mad.lo.cc.u32 %0, %2, %3, %4; madc.hi.cc.u32 %1, %2, %3, %5;" : "=r"(E[0]), "=r"(E[1]) : "r"(m), "r"(q[0]), "r"(t.v[0]), "r"(t.v[1]));
  PBC_ASM("madc.lo.cc.u32 %0, %2, %3, %4; madc.hi.cc.u32 %1, %2, %3, %5;" : "=r"(E[2]), "=r"(E[3]) : "r"(m), "r"(q[2]), "r"(t.v[2]), "r"(t.v[3]));
  PBC_ASM("madc.lo.cc.u32 %0, %2, %3, %4; madc.hi.u32 %1, %2, %3, 0;" : "=r"(E[4]), "=r"(E[5]) : "r"(m), "r"(q[4]), "r"(t.v[4]));
  PBC_MULW_PAIR(O[1], O[2], m, q[1]);
  PBC_MULW_PAIR(O[3], O[4], m, q[3]);
  top = 0;
#pragma unroll
  for (int i = 1; i < kNS; i++) {
    uint32_t* S = (i & 1) ? O : E;
    uint32_t* T = (i & 1) ? E : O;
    // the lone word of T at column i joins S; the carry enters T's run at column i + 1
    PBC_ASM("add.cc.u32 %0, %0, %1;" : "+r"(S[i]) : "r"(T[i]));
    m = S[i] * c_fp.np0;
    PBC_ASM("madc.lo.cc.u32 %0, %2, %3, %0; madc.hi.cc.u32 %1, %2, %3, %1;" : "+r"(T[i + 1]), "+r"(T[i + 2]) : "r"(m), "r"(q[1]));
    PBC_ASM("madc.lo.cc.u32 %0, %2, %3, %0; madc.hi.cc.u32 %1, %2, %3, %1;" : "+r"(T[i + 3]), "+r"(T[i + 4]) : "r"(m), "r"(q[3]));
    uint32_t ntop;
    PBC_CARRY_TO(ntop);                                     // into word i + 5 of T: the next row's fresh low word
    PBC_MADW_FIRST(S[i], S[i + 1], m, q[0]);                // S[i] becomes zero
    PBC_MADW_NEXT(S[i + 2], S[i + 3], m, q[2]);
    PBC_ASM("madc.lo.cc.u32 %0, %2, %3, %4; madc.hi.u32 %1, %2, %3, 0;" : "=r"(S[i + 4]), "=r"(S[i + 5]) : "r"(m), "r"(q[4]), "r"(top));
    top = ntop;
  }
  // after row 4 (S = E): E holds words 5..9, O words 5..8, top is word 9 of O.  X = E + O + top 2^(32 * 9)
  uint32_t o[kNS], v0;
  PBC_ASM("add.cc.u32 %0, %1, %2;" : "=r"(o[0]) : "r"(E[5]), "r"(O[5]));
  PBC_ASM("addc.cc.u32 %0, %1, %2;" : "=r"(o[1]) : "r"(E[6]), "r"(O[6]));
  PBC_ASM("addc.cc.u32 %0, %1, %2;" : "=r"(o[2]) : "r"(E[7]), "r"(O[7]));
  PBC_ASM("addc.cc.u32 %0, %1, %2;" : "=r"(o[3]) : "r"(E[8]), "r"(O[8]));
  PBC_ASM("addc.u32 %0, %1, %2;" : "=r"(o[4]) : "r"(E[9]), "r"(top));
  // + t_hi: below (1 or 2) q + q + 1 <= 3 q < 2^161
  PBC_ASM("add.cc.u32 %0, %0, %1;" : "+r"(o[0]) : "r"(t.v[5]));
#pragma unroll
  for (int k = 1; k < kNS; k++) PBC_ASM("addc.cc.u32 %0, %0, %1;" : "+r"(o[k]) : "r"(t.v[5 + k]));
  PBC_CARRY_TO(v0);
  uint32_t d[kNS], borrow;
  PBC_ASM("sub.cc.u32 %0, %1, %2;" : "=r"(d[0]) : "r"(o[0]), "r"(q[0]));
#pragma unroll
  for (int k = 1; k < kNS; k++) PBC_ASM("subc.cc.u32 %0, %1, %2;" : "=r"(d[k]) : "r"(o[k]), "r"(q[k]));
  PBC_ASM("subc.u32 %0, 0, 0;" : "=r"(borrow));
  bool use_d = v0 != 0 || borrow == 0;
  if constexpr (!TWO) {
#pragma unroll
    for (int k = 0; k < kNS; k++) r.v[k] = use_d ? d[k] : o[k];
  } else {
#pragma unroll
    for (int k = 0; k < kNS; k++) o[k] = use_d ? d[k] : o[k];
    PBC_ASM("sub.cc.u32 %0, %1, %2;" : "=r"(d[0]) : "r"(o[0]), "r"(q[0]));
#pragma unroll
    for (int k = 1; k < kNS; k++) PBC_ASM("subc.cc.u32 %0, %1, %2;" : "=r"(d[k]) : "r"(o[k]), "r"(q[k]));
    PBC_ASM("subc.u32 %0, 0, 0;" : "=r"(borrow));
#pragma unroll
    for (int k = 0; k < kNS; k++) r.v[k] = borrow == 0 ? d[k] : o[k];
  }
}
// r = a b, one product with the row-wise reduction
__device__ __forceinline__ void fq_mul_os(Fq& r, const Fq& a, const Fq& b) {
  FqAcc c;
  FqW t;
  fqa_mul(c, a, b);
  fqa_merge<false>(t, c);
  fqw_redc_os<false>(r, t);
}
#else
// any even limb count (the wide instance): redc_wide of fp.cuh, which takes t < 2 q R and returns the
// canonical residue (two conditional subtractions), so TWO makes no difference
template <bool TWO>
__device__ __forceinline__ void fqw_redc_os(Fq& r, const FqW& t) {
  uint32_t w[2 * kNS + 1];
#pragma unroll
  for (int k = 0; k < 2 * kNS; k++) w[k] = t.v[k];
  w[2 * kNS] = 0;
  redc_wide<kNS>(r.v, w);
}
__device__ __forceinline__ void fq_mul_os(Fq& r, const Fq& a, const Fq& b) {
  FqW t;
  fqw_mul(t, a, b);
  fqw_redc_os<false>(r, t);
}
#endif

#if !PBC_FQ_WIDE
// wire bytes (big-endian, 20 per coordinate) -> Montgomery form (arith/montfp.c:498-517 reduces mod q)
__device__ __forceinline__ void fq_from_wire(Fq& r, const uint8_t* p) {
  limbs_from_be<kNS, kWS>(r.v, p);
  mont_mul_ps<kNS, false>(r.v, r.v, c_fp.r2);
}
// Montgomery form -> canonical residue -> wire bytes (arith/montfp.c:64-80, :487-496)
__device__ __forceinline__ void fq_to_wire(uint8_t* p, const Fq& a) {
  uint32_t one[kNS] = {1}, x[kNS];
  mont_mul_ps<kNS, false>(x, a.v, one);
  limbs_to_be<kNS, kWS>(p, x);
}
#else
// the wide instance: ceil(bits(q)/8) bytes per coordinate, a run-time constant, read and written byte
// by byte (no alignment).  Any wb-byte value is below 2^256 = R, and mont_mul_ps reduces a R q-bounded
// product to the canonical residue (a < R, b < q, q < R/2), as arith/montfp.c:498-517 reduces mod q.
__device__ __forceinline__ void fq_from_wire(Fq& r, const uint8_t* p) {
  const int wb = fq_wb();
#pragma unroll
  for (int k = 0; k < kNS; k++) {
    uint32_t w = 0;
#pragma unroll
    for (int b = 0; b < 4; b++) {
      int pos = wb - 1 - (4 * k + b);
      if (pos >= 0) w |= (uint32_t)p[pos] << (8 * b);
    }
    r.v[k] = w;
  }
  mont_mul_ps<kNS, false>(r.v, r.v, c_fp.r2);
}
__device__ __forceinline__ void fq_to_wire(uint8_t* p, const Fq& a) {
  const int wb = fq_wb();
  uint32_t one[kNS] = {1}, x[kNS];
  mont_mul_ps<kNS, false>(x, a.v, one);
#pragma unroll
  for (int k = 0; k < kNS; k++) {
#pragma unroll
    for (int b = 0; b < 4; b++) {
      int pos = wb - 1 - (4 * k + b);
      if (pos >= 0) p[pos] = (uint8_t)(x[k] >> (8 * b));
    }
  }
}
#endif

// the same for a coordinate width that is not a multiple of four bytes (g149: 19), byte by byte
template <int WB>
__device__ __forceinline__ void fq_from_wire_b(Fq& r, const uint8_t* p) {
  if constexpr (WB == 0) fq_from_wire(r, p);         // the run-time width of the wide instance
  else {
#pragma unroll
  for (int k = 0; k < kNS; k++) {
    uint32_t w = 0;
#pragma unroll
    for (int b = 0; b < 4; b++) {
      int pos = WB - 1 - (4 * k + b);        // byte of weight 256^(4k+b), counted from the end
      if (pos >= 0) w |= (uint32_t)p[pos] << (8 * b);
    }
    r.v[k] = w;
  }
  mont_mul_ps<kNS, false>(r.v, r.v, c_fp.r2);
  }
}
template <int WB>
__device__ __forceinline__ void fq_to_wire_b(uint8_t* p, const Fq& a) {
  uint32_t one[kNS] = {1}, x[kNS];
  mont_mul_ps<kNS, false>(x, a.v, one);
#pragma unroll
  for (int i = 0; i < WB; i++) {
    int byte = WB - 1 - i;                   // weight of output byte i
    p[i] = (uint8_t)(x[byte >> 2] >> (8 * (byte & 3)));
  }
}

// width-generic front ends: the word-wise path when the width allows it, else byte by byte; WB = 0: the
// run-time width of the wide instance
template <int WB>
__device__ __forceinline__ void fq_from_wire_w(Fq& r, const uint8_t* p) {
  if constexpr (WB == 0) fq_from_wire(r, p);
  else if constexpr (WB % 4 == 0) { limbs_from_be<kNS, WB>(r.v, p); mont_mul_ps<kNS, false>(r.v, r.v, c_fp.r2); }
  else fq_from_wire_b<WB>(r, p);
}
template <int WB>
__device__ __forceinline__ void fq_to_wire_w(uint8_t* p, const Fq& a) {
  if constexpr (WB == 0) fq_to_wire(p, a);
  else if constexpr (WB % 4 == 0) { uint32_t one[kNS] = {1}, x[kNS]; mont_mul_ps<kNS, false>(x, a.v, one); limbs_to_be<kNS, WB>(p, x); }
  else fq_to_wire_b<WB>(p, a);
}

// a^(q-2) (the reference calls mpz_invert, arith/montfp.c:401-422; the value is the same)
__device__ __noinline__ void fq_inv(Fq* r, const Fq* a) {
  Fq x = *a, acc;
  fq_one(acc);
  int top = kNS * 32 - 1;
  while (top > 0 && !((c_fp.pm2[top >> 5] >> (top & 31)) & 1u)) top--;
  for (int j = top; j >= 0; j--) {
    fq_sqr(acc, acc);
    if ((c_fp.pm2[j >> 5] >> (j & 31)) & 1u) fq_mul(acc, acc, x);
  }
  *r = acc;
}

// limb-major batch arrays in global memory: word w of element e of item idx at g[(e*kNS + w)*n + idx]
__device__ __forceinline__ void fq_st_global(uint32_t* g, int e, size_t n, size_t idx, const Fq& a) {
#pragma unroll
  for (int k = 0; k < kNS; k++) g[((size_t)e * kNS + k) * n + idx] = a.v[k];
}
__device__ __forceinline__ void fq_ld_global(Fq& a, const uint32_t* g, int e, size_t n, size_t idx) {
#pragma unroll
  for (int k = 0; k < kNS; k++) a.v[k] = g[((size_t)e * kNS + k) * n + idx];
}

}  // namespace pbcb200
