// pairing_f_slots.cuh -- Type F Miller loop on a shared-memory slot machine (round 2).
//
// Same function as k_f_miller of pairing_f.cuh (device replacement for cc_miller_no_denom,
// ecc/f_param.c:97-248, and the F_q^12 arithmetic it runs on, arith/poly.c:932-1143 +
// arith/fieldquadratic.c:197-309), same internal basis and lazy reduction, different machine:
//
//   * k_f_miller keeps its tower elements in the per-thread local frame (1 248 B per thread): with
//     every SM full that frame outgrows L2 and the loop waits on DRAM.  Here every long-lived value is an F_q
//     *slot* of shared memory -- word w of slot s of thread t at smem[(s * 5 + w) * BLOCK + t],
//     conflict-free 32-bit accesses -- 36 slots = 720 B per thread: the Miller value (12), one
//     12-slot scratch area whose role alternates with it, the line (9) and V = (X, Y, Z).  Q and P
//     (used by a few multiplications per iteration) stay in a limb-major global array.
//   * field operations are out-of-line routines on slot numbers that load their operands, work in
//     registers and store the result: the F_q^6 product is ONE routine (a loop over the nine
//     F_q^2 products of the schoolbook form, three double-width accumulations and six reductions:
//     855 multiplier operations against 810 for Karatsuba, but no additions and a third of the
//     shared-memory traffic); the sparse line product is one routine of the same shape.
//   * no local memory in the loop at all, 2 x 128 threads per SM (shared-memory bound, as type A).
//
// Needs the internal basis (c_f.nice) and 3 q < 2^160 for the accumulation bounds; the host falls
// back to k_f_miller otherwise.
#pragma once
#include "pairing_f.cuh"

namespace pbcb200 {

// Slots per thread: 36 = 720 B, two 128-thread blocks (8 warps) per SM, about 210 registers per thread.
// A 29-slot version (V = (X, Y, Z) and xi L3, xi L4 parked in the global scratch: three blocks = 12 warps
// per SM, registers capped at 168) was slower: the cap spills inside the product routines.  These kernels want registers more than they want warps.
// A block-wide barrier at the top of every Miller iteration and of every step of the powers by u keeps the
// warps of a block fetching the same routines (without it k_f_finalexp_s waits on instruction fetch).  Every
// thread of a block then has to run the loops.
constexpr int kFSlots = 36;
enum FSlotMap {
  fsV = 0,                             // 12: Miller value (coefficient j at 2 * f12_pos(j))
  fsT = 12,                            // 12: scratch / the other copy (roles alternate)
  fsX = 24, fsY = 25, fsZ = 26,        // V, Jacobian
  fsC = 27,                            // line: c + L3 x^3 + L4 x^4
  fsL3 = 28, fsL4 = 30, fsXL3 = 32, fsXL4 = 34,
};
// global scratch per pairing, F_q elements: Qx (0, 1), Qy (2, 3), xP (4), yP (5)
enum FGlobalMap { fgQx = 0, fgQy = 2, fgPx = 4, fgPy = 5 };
constexpr int kFGWords = 6 * kNS;

// ---- register-level pieces (fq_small.cuh) ----
// Products and squares alike are fq_mul_os: the full 25-product row schedule takes fewer instructions than
// the 15 + 25 product column-wise squarer.

// ---- F_q^2 products on three unmerged sums (FqAcc, fq_small.cuh) ----
//   A = sum x0 y0,  B = sum x1 y1,  C = sum (x0 + x1)(y0 + y1);   re = A - B,  im = C - A - B.
// Bounds: operands canonical, so a term adds less than q^2 to A and B and less than 4 q^2 to C; three terms
// keep C below 12 q^2 < 2^320 (c_f.slots_ok).
struct F2Acc { FqAcc A, B, C; };
// TERM 0: the first term (starts the sums), 1: the second (first carry counts), 2: any later one
template <int TERM>
__device__ __forceinline__ void f2a_term(F2Acc& g, const Fq& x0, const Fq& x1, const Fq& y0, const Fq& y1) {
  Fq sx, sy;
  fq_add_nr(sx, x0, x1);
  fq_add_nr(sy, y0, y1);
  if (TERM == 0) { fqa_mul(g.A, x0, y0); fqa_mul(g.B, x1, y1); fqa_mul(g.C, sx, sy); }
  else { fqa_mac<TERM == 1>(g.A, x0, y0); fqa_mac<TERM == 1>(g.B, x1, y1); fqa_mac<TERM == 1>(g.C, sx, sy); }
}
// (r0, r1) = (re, im) reduced.  offs: a multiple of q^2 (double width) not below B, HASK: more than one term.
template <bool HASK>
__device__ __forceinline__ void f2a_finish(Fq& r0, Fq& r1, const F2Acc& g, const uint32_t* offs) {
  FqW a, b, c;
  fqa_merge<HASK>(a, g.A);
  fqa_merge<HASK>(b, g.B);
  fqa_merge<HASK>(c, g.C);
  fqw_sub(c, c, a);
  fqw_sub(c, c, b);                        // im = C - A - B >= 0
  PBC_ASM("add.cc.u32 %0, %0, %1;" : "+r"(a.v[0]) : "r"(offs[0]));
#pragma unroll
  for (int k = 1; k < 2 * kNS; k++) PBC_ASM("addc.cc.u32 %0, %0, %1;" : "+r"(a.v[k]) : "r"(offs[k]));
  fqw_sub(a, a, b);                        // re = A + offs - B
  fqw_redc_os<true>(r0, a);
  fqw_redc_os<true>(r1, c);
}

// (x0 + x1 i) <- xi' (x0 + x1 i), xi' = a + b i with small a, b (see f2_mul_xi)
__device__ __forceinline__ void f2r_mul_xi(Fq& x0, Fq& x1) {
  const uint32_t a = c_f.xi_a, b = c_f.xi_b, m = a | b;
  Fq a1 = x0, b1 = x1, a2, a4, b2, b4, p, q2, s2, t;
  if (m & 6u) { fq_dbl(a2, a1); fq_dbl(b2, b1); }
  if (m & 4u) { fq_dbl(a4, a2); fq_dbl(b4, b2); }
  fq_small_combo(p, a, a1, a2, a4);      // a x0
  fq_small_combo(q2, b, b1, b2, b4);     // b x1
  fq_small_combo(s2, b, a1, a2, a4);     // b x0
  fq_small_combo(t, a, b1, b2, b4);      // a x1
  fq_sub(x0, p, q2);
  fq_add(x1, s2, t);
}

// (o0 + o1 i) = (x0 + x1 i)^2 = (x0 + x1)(x0 - x1) + 2 x0 x1 i, in registers
__device__ __forceinline__ void f2r_sqr(Fq& o0, Fq& o1, const Fq& x0, const Fq& x1) {
  Fq s, t;
  fq_add_nr(s, x0, x1);                    // below 2q < 2^160: fine as a multiplier operand
  fq_sub(t, x0, x1);
  fq_mul_os(s, s, t);
  fq_mul_os(t, x0, x1);
  fq_dbl(o1, t);
  o0 = s;
}
// (r0, r1) = (a + b s)^2 in F_q^4 = F_q^2[s]/(s^2 - xi): r0 = a^2 + xi b^2, r1 = (a + b)^2 - a^2 - b^2
__device__ __forceinline__ void f4r_sqr(Fq& r00, Fq& r01, Fq& r10, Fq& r11, const Fq& a0, const Fq& a1,
                                        const Fq& b0, const Fq& b1) {
  Fq sb0, sb1, t0, t1;
  f2r_sqr(r00, r01, a0, a1);               // a^2
  f2r_sqr(sb0, sb1, b0, b1);               // b^2
  fq_add(t0, a0, b0); fq_add(t1, a1, b1);
  f2r_sqr(r10, r11, t0, t1);               // (a + b)^2
  fq_sub(r10, r10, r00); fq_sub(r11, r11, r01);
  fq_sub(r10, r10, sb0); fq_sub(r11, r11, sb1);
  f2r_mul_xi(sb0, sb1);
  fq_add(r00, r00, sb0); fq_add(r01, r01, sb1);
}
// c <- 3 r + 2 c (PLUS) or 3 r - 2 c, one F_q coordinate
template <bool PLUS>
__device__ __forceinline__ void gs_combine(Fq& c, const Fq& r) {
  Fq t;
  if (PLUS) fq_add(t, r, c); else fq_sub(t, r, c);
  fq_dbl(t, t);
  fq_add(c, r, t);
}

// ---- the slot machine ----
template <int BLOCK>
struct FS {
  static __device__ __forceinline__ uint32_t* base() { return reinterpret_cast<uint32_t*>(pbc_smem) + threadIdx.x; }
  static __device__ __forceinline__ void ld(Fq& r, int s) {
    const uint32_t* b = base() + s * (kNS * BLOCK);
#pragma unroll
    for (int k = 0; k < kNS; k++) r.v[k] = b[k * BLOCK];
  }
  static __device__ __forceinline__ void st(int s, const Fq& r) {
    uint32_t* b = base() + s * (kNS * BLOCK);
#pragma unroll
    for (int k = 0; k < kNS; k++) b[k * BLOCK] = r.v[k];
  }
  // ---- F_q ----
  static __device__ __noinline__ void qmul(int d, int a, int b) {
    Fq x, y;
    ld(x, a); ld(y, b);
    fq_mul_os(x, x, y);
    st(d, x);
  }
  static __device__ __noinline__ void qsqr(int d, int a) {
    Fq x;
    ld(x, a);
    fq_mul_os(x, x, x);
    st(d, x);
  }
  // two / three independent products in ONE call, every operand read before any result is stored (so the
  // results may overwrite operands of the other products).  A lone F_q product is one serial carry chain;
  // the point arithmetic of a Miller step has them in independent pairs and triples, and two warps per
  // scheduler do not hide a chain's latency.
  static __device__ __noinline__ void qmul2(int d0, int a0, int b0, int d1, int a1, int b1) {
    Fq x0, y0, x1, y1;
    ld(x0, a0); ld(y0, b0); ld(x1, a1); ld(y1, b1);
    fq_mul_os(x0, x0, y0);
    fq_mul_os(x1, x1, y1);
    st(d0, x0); st(d1, x1);
  }
  static __device__ __noinline__ void qmul3(int d0, int a0, int b0, int d1, int a1, int b1, int d2, int a2, int b2) {
    Fq x0, y0, x1, y1, x2, y2;
    ld(x0, a0); ld(y0, b0); ld(x1, a1); ld(y1, b1); ld(x2, a2); ld(y2, b2);
    fq_mul_os(x0, x0, y0);
    fq_mul_os(x1, x1, y1);
    fq_mul_os(x2, x2, y2);
    st(d0, x0); st(d1, x1); st(d2, x2);
  }
  static __device__ __noinline__ void qsqr3(int d0, int a0, int d1, int a1, int d2, int a2) {
    Fq x0, x1, x2;
    ld(x0, a0); ld(x1, a1); ld(x2, a2);
    fq_mul_os(x0, x0, x0);
    fq_mul_os(x1, x1, x1);
    fq_mul_os(x2, x2, x2);
    st(d0, x0); st(d1, x1); st(d2, x2);
  }
  // d0 = a0 b0, d1 = a1^2, d2 = a2^2
  static __device__ __noinline__ void qmul1sqr2(int d0, int a0, int b0, int d1, int a1, int d2, int a2) {
    Fq x0, y0, x1, x2;
    ld(x0, a0); ld(y0, b0); ld(x1, a1); ld(x2, a2);
    fq_mul_os(x0, x0, y0);
    fq_mul_os(x1, x1, x1);
    fq_mul_os(x2, x2, x2);
    st(d0, x0); st(d1, x1); st(d2, x2);
  }
  static __device__ __noinline__ void qadd(int d, int a, int b) { Fq x, y; ld(x, a); ld(y, b); fq_add(x, x, y); st(d, x); }
  static __device__ __noinline__ void qsub(int d, int a, int b) { Fq x, y; ld(x, a); ld(y, b); fq_sub(x, x, y); st(d, x); }
  static __device__ __noinline__ void qdbl(int d, int a, int k = 1) {
    Fq x;
    ld(x, a);
    for (int i = 0; i < k; i++) fq_dbl(x, x);
    st(d, x);
  }
  static __device__ __forceinline__ void qneg(int d, int a) { Fq x; ld(x, a); fq_neg(x, x); st(d, x); }
  static __device__ __forceinline__ void qcopy(int d, int a) { Fq x; ld(x, a); st(d, x); }
  // slot <- element e of this thread's global scratch (word-major, words n apart), negated on request
  static __device__ __forceinline__ void qldg(int d, const uint32_t* g, int e, size_t n, bool neg) {
    Fq x;
#pragma unroll
    for (int k = 0; k < kNS; k++) x.v[k] = g[((size_t)e * kNS + k) * n];
    if (neg) fq_neg(x, x);
    st(d, x);
  }
  // slot <- kNS consecutive words (the same address for every thread: a table row)
  static __device__ __forceinline__ void qldc(int d, const uint32_t* c) {
    Fq x;
#pragma unroll
    for (int k = 0; k < kNS; k++) x.v[k] = c[k];
    st(d, x);
  }
  // (d, d+1) <- (global F_q^2 element at e, e+1) * slot a
  static __device__ __noinline__ void f2scale_g(int d, const uint32_t* g, int e, size_t n, int a) {
    Fq x, y0, y1;
#pragma unroll
    for (int k = 0; k < kNS; k++) { y0.v[k] = g[((size_t)e * kNS + k) * n]; y1.v[k] = g[((size_t)(e + 1) * kNS + k) * n]; }
    ld(x, a);
    fq_mul_os(y0, y0, x);
    fq_mul_os(y1, y1, x);
    st(d, y0); st(d + 1, y1);
  }
  // ---- F_q^2 (two consecutive slots) ----
  // d = a + b (MODE 0), a - b (1), 2 a (2), a + xi b (3), a - xi b (4), xi a (5)
  template <int MODE>
  static __device__ __noinline__ void f2op(int d, int a, int b) {
    Fq x0, x1, y0, y1;
    ld(x0, a); ld(x1, a + 1);
    if (MODE == 2) { fq_dbl(x0, x0); fq_dbl(x1, x1); }
    else if (MODE == 5) { f2r_mul_xi(x0, x1); }
    else {
      ld(y0, b); ld(y1, b + 1);
      if (MODE >= 3) f2r_mul_xi(y0, y1);
      if (MODE == 0 || MODE == 3) { fq_add(x0, x0, y0); fq_add(x1, x1, y1); }
      else { fq_sub(x0, x0, y0); fq_sub(x1, x1, y1); }
    }
    st(d, x0); st(d + 1, x1);
  }
  static __device__ __forceinline__ void f2add(int d, int a, int b) { f2op<0>(d, a, b); }
  static __device__ __forceinline__ void f2sub(int d, int a, int b) { f2op<1>(d, a, b); }
  static __device__ __forceinline__ void f2dbl(int d, int a) { f2op<2>(d, a, a); }
  static __device__ __forceinline__ void f2addxi(int d, int a, int b) { f2op<3>(d, a, b); }
  static __device__ __forceinline__ void f2subxi(int d, int a, int b) { f2op<4>(d, a, b); }
  static __device__ __forceinline__ void f2mulxi(int d, int a) { f2op<5>(d, a, a); }

  // d = a^2 = (a0 + a1)(a0 - a1) + 2 a0 a1 i
  static __device__ __noinline__ void f2sqr(int d, int a) {
    Fq x0, x1, s, t;
    ld(x0, a); ld(x1, a + 1);
    fq_add_nr(s, x0, x1);                  // below 2q < 2^160: fine as a multiplier operand
    fq_sub(t, x0, x1);
    fq_mul_os(s, s, t);
    fq_mul_os(t, x0, x1);
    fq_dbl(t, t);
    st(d, s); st(d + 1, t);
  }
  static __device__ __forceinline__ void f2neg(int d, int a) { qneg(d, a); qneg(d + 1, a + 1); }
  static __device__ __forceinline__ void f2copy(int d, int a) { qcopy(d, a); qcopy(d + 1, a + 1); }
  // d = 3 x + 2 c (PLUS) or 3 x - 2 c: the recombination of the cyclotomic squaring
  template <bool PLUS>
  static __device__ __noinline__ void f2gs(int d, int x, int c) {
    Fq x0, x1, c0, c1, t;
    ld(x0, x); ld(x1, x + 1); ld(c0, c); ld(c1, c + 1);
    if (PLUS) { fq_add(t, x0, c0); } else { fq_sub(t, x0, c0); }
    fq_dbl(t, t); fq_add(x0, x0, t);
    if (PLUS) { fq_add(t, x1, c1); } else { fq_sub(t, x1, c1); }
    fq_dbl(t, t); fq_add(x1, x1, t);
    st(d, x0); st(d + 1, x1);
  }
  // d = (conj) a * constant (an F_q^2 element in __constant__ memory, Montgomery form)
  static __device__ __noinline__ void f2mulc(int d, int a, const uint32_t (*c)[kNS], bool conj) {
    Fq x0, x1, y0, y1;
    ld(x0, a); ld(x1, a + 1);
    if (conj) fq_neg(x1, x1);
    fq_set(y0, c[0]); fq_set(y1, c[1]);
    F2Acc g;
    f2a_term<0>(g, x0, x1, y0, y1);
    f2a_finish<false>(x0, x1, g, c_f.qsqm[0]);
    st(d, x0); st(d + 1, x1);
  }

  // ---- F_q^6 = F_q^2[y]/(y^3 - xi): d = a b, operands are 3 consecutive F_q^2 = 6 slots; d must not
  // overlap a or b.  c_k = sum_i a_i b'_(k-i), b' = xi b where the index wrapped: three products per
  // coefficient accumulated double width (each term below 2 q^2, the sum below 6 q^2 < 2 q R), one
  // reduction per F_q.
  // xs: four scratch slots (they receive xi b_1 and xi b_2), apart from d, a, b.
  static __device__ __noinline__ void f6mul(int d, int a, int b, int xs) {
    // The three terms of a coefficient are written out: sums carried around a loop cost a register move per
    // accumulator pair and iteration.  The
    // wrapped operands xi b_1, xi b_2 are made once, so a term only selects its slot.
    f2mulxi(xs, b + 2);
    f2mulxi(xs + 2, b + 4);
#pragma unroll 1
    for (int k = 0; k < 3; k++) {
      F2Acc g;
      Fq x0, x1, y0, y1;
      ld(x0, a); ld(x1, a + 1); ld(y0, b + 2 * k); ld(y1, b + 2 * k + 1);      // a_0 b_k
      f2a_term<0>(g, x0, x1, y0, y1);
      const int s1 = k >= 1 ? b + 2 * (k - 1) : xs + 2;                        // a_1 b_(k-1)  or  a_1 (xi b_2)
      ld(x0, a + 2); ld(x1, a + 3); ld(y0, s1); ld(y1, s1 + 1);
      f2a_term<1>(g, x0, x1, y0, y1);
      const int s2 = k == 2 ? b : (k == 1 ? xs + 2 : xs);                      // a_2 b_0,  a_2 (xi b_2),  a_2 (xi b_1)
      ld(x0, a + 4); ld(x1, a + 5); ld(y0, s2); ld(y1, s2 + 1);
      f2a_term<2>(g, x0, x1, y0, y1);
      f2a_finish<true>(x0, x1, g, c_f.qsqm[2]);
      st(d + 2 * k, x0); st(d + 2 * k + 1, x1);
    }
  }
  // o = v * (c + L3 x^3 + L4 x^4)   (f12_mul_line): o and v are 12-slot F_q^12 areas, distinct.
  //   o_k = c v_k + m3 v_(k-3) + m4 v_(k-4), indices below zero wrap with xi (slots fsXL3 / fsXL4)
  static __device__ __noinline__ void line_mul(int o, int v) {
#pragma unroll 1
    for (int k = 0; k < 6; k++) {
      const int i3 = k >= 3 ? k - 3 : k + 3, i4 = k >= 4 ? k - 4 : k + 2;
      // re = A - B + c y0,  im = C - A - B + c y1:  c y0 joins A and c (y0 + y1) joins C
      F2Acc g;
      Fq x0, x1, y0, y1;
      const int m3 = k >= 3 ? fsL3 : fsXL3, m4 = k >= 4 ? fsL4 : fsXL4;
      ld(x0, m3); ld(x1, m3 + 1);
      ld(y0, v + 2 * f12_pos(i3)); ld(y1, v + 2 * f12_pos(i3) + 1);
      f2a_term<0>(g, x0, x1, y0, y1);
      ld(x0, m4); ld(x1, m4 + 1);
      ld(y0, v + 2 * f12_pos(i4)); ld(y1, v + 2 * f12_pos(i4) + 1);
      f2a_term<1>(g, x0, x1, y0, y1);
      ld(x0, fsC);
      ld(y0, v + 2 * f12_pos(k)); ld(y1, v + 2 * f12_pos(k) + 1);
      fq_add_nr(x1, y0, y1);
      fqa_mac<false>(g.A, x0, y0);
      fqa_mac<false>(g.C, x0, x1);
      f2a_finish<true>(x0, x1, g, c_f.qsqm[1]);
      st(o + 2 * f12_pos(k), x0); st(o + 2 * f12_pos(k) + 1, x1);
    }
  }
  // v <- v^2 in place with the 12-slot scratch t (f12_sqr: complex squaring over F_q^6).
  //   A = v[0..5], B = v[6..11];  t0 = A B;  t1 = (A + B)(A + y B);  A' = t1 - t0 - y t0,  B' = 2 t0
  static __device__ __forceinline__ void f12sqr(int v, int t, int xs) {
    f6mul(t, v, v + 6, xs);                                    // t0
    f2add(t + 6, v, v + 6); f2add(t + 8, v + 2, v + 8); f2add(t + 10, v + 4, v + 10);        // A + B
    f2addxi(v, v, v + 10); f2add(v + 2, v + 2, v + 6); f2add(v + 4, v + 4, v + 8);           // A + y B, in place
    f6mul(v + 6, t + 6, v, xs);                                // t1 over B (B is dead)
    f2sub(v, v + 6, t); f2subxi(v, v, t + 4);                  // A'0 = t1_0 - t0_0 - xi t0_2
    f2sub(v + 2, v + 8, t + 2); f2sub(v + 2, v + 2, t);        // A'1 = t1_1 - t0_1 - t0_0
    f2sub(v + 4, v + 10, t + 4); f2sub(v + 4, v + 4, t + 2);   // A'2 = t1_2 - t0_2 - t0_1
    f2dbl(v + 6, t); f2dbl(v + 8, t + 2); f2dbl(v + 10, t + 4);
  }
  // p <- p q with the 12-slot scratch t (f12_mul: Karatsuba over F_q^6); q is left as it was.
  //   p = A + B x, q = C + D x:  t0 = A C, t1 = B D, t2 = (A + B)(C + D);  lo = t0 + y t1, hi = t2 - t0 - t1
  static __device__ __forceinline__ void f12mul(int p, int q, int t, int xs) {
    f6mul(t, p, q, xs);                                        // t0
    f6mul(t + 6, p + 6, q + 6, xs);                            // t1
    f2add(p, p, p + 6); f2add(p + 2, p + 2, p + 8); f2add(p + 4, p + 4, p + 10);     // A + B over A
    f2add(q, q, q + 6); f2add(q + 2, q + 2, q + 8); f2add(q + 4, q + 4, q + 10);     // C + D over C
    f6mul(p + 6, p, q, xs);                                    // t2 over B
    f2sub(q, q, q + 6); f2sub(q + 2, q + 2, q + 8); f2sub(q + 4, q + 4, q + 10);     // C back
    f2sub(p + 6, p + 6, t); f2sub(p + 6, p + 6, t + 6);
    f2sub(p + 8, p + 8, t + 2); f2sub(p + 8, p + 8, t + 8);
    f2sub(p + 10, p + 10, t + 4); f2sub(p + 10, p + 10, t + 10);
    f2addxi(p, t, t + 10);                                     // lo0 = t0_0 + xi t1_2
    f2add(p + 2, t + 2, t + 6);                                // lo1 = t0_1 + t1_0
    f2add(p + 4, t + 4, t + 8);                                // lo2 = t0_2 + t1_1
  }
  // (r0, r1) = (a + b s)^2 in F_q^4 = F_q^2[s]/(s^2 - xi): (a^2 + xi b^2, (a + b)^2 - a^2 - b^2); e: one F_q^2 of scratch
  static __device__ __forceinline__ void f4sqr(int r0, int r1, int a, int b, int e) {
    f2sqr(r0, a);
    f2sqr(e, b);
    f2add(r1, a, b);
    f2sqr(r1, r1);
    f2sub(r1, r1, r0);
    f2sub(r1, r1, e);
    f2addxi(r0, r0, e);
  }
  // v <- v^2 for v in the cyclotomic subgroup (Granger-Scott, see f12_cyc_sqr), in place.  Coefficient j lives at
  // v + 2 f12_pos(j): c0 -> 0, c1 -> 6, c2 -> 2, c3 -> 8, c4 -> 4, c5 -> 10.
  //   A = (c0 + c3 s)^2:  c0' = 3 A0 - 2 c0,  c3' = 3 A1 + 2 c3
  //   B = (c1 + c4 s)^2:  c2' = 3 B0 - 2 c2,  c5' = 3 B1 + 2 c5
  //   C = (c2 + c5 s)^2:  c4' = 3 C0 - 2 c4,  c1' = 3 xi C1 + 2 c1
  // History: 28 calls of F_q^2 routines per squaring ran at 0.3 of the multiplier peak (5.5 instructions per
  // product); two fused routines working in registers (cyc_pair_a, cyc_pair_bc: the three F_q^4 squarings written out,
  // 2 200 instructions executed once per squaring) left the warps waiting for instructions
  // in k_f_finalexp_s.  Now ONE out-of-line F_q^4 squaring
  // with the recombination, called three times (B's square waits in the four scratch slots e while C -- which reads
  // what B's results overwrite -- is done).
  // (r0, r1) = (a + b s)^2 for the F_q^2 at slots a, b.  raw: tm <- r0, tp <- r1;  else tm <- 3 r0 - 2 tm and
  // tp <- 3 r1' + 2 tp with r1' = xi r1 when xi is set.
  static __device__ __noinline__ void f4sqr_gs(int a, int b, int tm, int tp, bool raw, bool xi) {
    Fq a0, a1, b0, b1, r00, r01, r10, r11;
    ld(a0, a); ld(a1, a + 1); ld(b0, b); ld(b1, b + 1);
    f4r_sqr(r00, r01, r10, r11, a0, a1, b0, b1);
    if (!raw) {
      if (xi) f2r_mul_xi(r10, r11);
      ld(a0, tm); ld(a1, tm + 1); ld(b0, tp); ld(b1, tp + 1);
      gs_combine<false>(a0, r00); gs_combine<false>(a1, r01);
      gs_combine<true>(b0, r10); gs_combine<true>(b1, r11);
      r00 = a0; r01 = a1; r10 = b0; r11 = b1;
    }
    st(tm, r00); st(tm + 1, r01); st(tp, r10); st(tp + 1, r11);
  }
  // e: four scratch slots
  static __device__ __forceinline__ void f12cycsqr(int v, int, int e) {
    f4sqr_gs(v + 6, v + 4, e, e + 2, true, false);            // B -> scratch
    f4sqr_gs(v, v + 8, v, v + 8, false, false);               // A
    f4sqr_gs(v + 2, v + 10, v + 4, v + 6, false, true);       // C (reads c2, c5; writes c4, c1)
    f2gs<false>(v + 2, e, v + 2);                             // c2' = 3 B0 - 2 c2
    f2gs<true>(v + 10, e + 2, v + 10);                        // c5' = 3 B1 + 2 c5
  }
  // v <- v^(q^k), k = 1, 2, 3 (f12_frob)
  static __device__ __noinline__ void f12frob(int v, int k) {
    if (k & 1) qneg(v + 1, v + 1);
#pragma unroll 1
    for (int j = 1; j < 6; j++) f2mulc(v + 2 * f12_pos(j), v + 2 * f12_pos(j), c_f.frob[k - 1][j - 1], (k & 1) != 0);
  }
  // v <- v^(q^6): x -> -x
  static __device__ __forceinline__ void f12conj(int v) { f2neg(v + 6, v + 6); f2neg(v + 8, v + 8); f2neg(v + 10, v + 10); }
  static __device__ __noinline__ void f12copy(int d, int a) {
#pragma unroll 1
    for (int s = 0; s < 12; s++) qcopy(d + s, a + s);
  }
  // 12 slots <-> a [12 * kNS][n] word-major global array (g already offset to this thread)
  static __device__ __noinline__ void f12ldg(int d, const uint32_t* g, size_t n) {
#pragma unroll 1
    for (int s = 0; s < 12; s++) qldg(d + s, g, s, n, false);
  }
  static __device__ __noinline__ void f12stg(uint32_t* g, size_t n, int a, bool live = true) {
    if (!live) return;                       // padding threads share index 0 with a real thread: they never write
#pragma unroll 1
    for (int s = 0; s < 12; s++) {
      Fq x;
      ld(x, a + s);
#pragma unroll
      for (int k = 0; k < kNS; k++) g[((size_t)s * kNS + k) * n] = x.v[k];
    }
  }
  // r0 <- r1^|u| (conjugated when u < 0) on the cyclotomic subgroup (f12_pow_u); r1 is preserved
  static __device__ __noinline__ void f12powu(int r0, int r1, int t, int e) {
    f12copy(r0, r1);
    for (int j = (int)c_f.u_bits - 2; j >= 0; j--) {
      __syncthreads();
      f12cycsqr(r0, t, e);
      if ((c_f.u_abs[j >> 5] >> (j & 31)) & 1u) f12mul(r0, r1, t, e);
    }
    if (c_f.u_neg) f12conj(r0);
  }
};

// Same interface as k_f_miller plus gq: [6 * kNS][n] words of scratch (Qx, Qy untwisted and scaled, P;
// Montgomery form, internal basis).
template <int BLOCK>
__global__ void __launch_bounds__(BLOCK)
k_f_miller_s(const uint8_t* __restrict__ P, const uint8_t* __restrict__ Q, uint32_t* __restrict__ mv,
             uint32_t* __restrict__ flag, uint32_t* __restrict__ gq, size_t n, size_t stride1,
             const uint32_t* __restrict__ tab, size_t rows) {
  using S = FS<BLOCK>;
  size_t idx = (size_t)blockIdx.x * BLOCK + threadIdx.x;
  const bool live = idx < n;               // padding threads of the last block run too (block-wide barriers below)
  if (!live) idx = 0;
  bool ok;
  {
    // decode, validate, move to the basis in use (as k_f_miller)
    Fq xP, yP, sg;
    if (tab) {
      ok = tab[3 * rows * kNS] != 0;           // fixed first argument: lines from the table (k_cc_pp_init)
      fq_zero(xP); fq_zero(yP);
    } else {
      const uint8_t* p = P + idx * stride1;
      fq_from_wire(xP, p);
      fq_from_wire(yP, p + kWS);
      ok = cc_on_curve(xP, yP);
    }
    F2 Qx, Qy, t, u;
    const uint8_t* q = Q + idx * (4 * kWS);
    fq_from_wire(Qx.a, q);
    fq_from_wire(Qx.b, q + kWS);
    fq_from_wire(Qy.a, q + 2 * kWS);
    fq_from_wire(Qy.b, q + 3 * kWS);
    fq_set(sg, c_f.sigma);
    fq_mul(Qx.b, Qx.b, sg);
    fq_mul(Qy.b, Qy.b, sg);
    f2_sqr(&t, &Qx);
    f2_mul(&t, &t, &Qx);
    f2_add(t, t, *f2_const(c_f.twist_b));
    f2_sqr(&u, &Qy);
    ok = ok && f2_eq(t, u);
    f2_mul(&Qx, &Qx, f2_const(c_f.kx));
    f2_mul(&Qy, &Qy, f2_const(c_f.ky));
    fq_st_global(gq, 0, n, idx, Qx.a); fq_st_global(gq, 1, n, idx, Qx.b);
    fq_st_global(gq, 2, n, idx, Qy.a); fq_st_global(gq, 3, n, idx, Qy.b);
    fq_st_global(gq, fgPx, n, idx, xP); fq_st_global(gq, fgPy, n, idx, yP);
    Fq one, zero;
    fq_one(one); fq_zero(zero);
    S::st(fsX, xP); S::st(fsY, yP); S::st(fsZ, one);
    S::st(fsV, one);
#pragma unroll 1
    for (int s = 1; s < 12; s++) S::st(fsV + s, zero);
  }
  const uint32_t* g = gq + idx;
  int V = fsV, T = fsT;
  size_t row = 0;
  int m = (int)c_ccnaf.len - 2;
  for (;;) {
    __syncthreads();
    if (tab) {
      // ---- fixed first argument: (a, b, c) of the next line from the table ----
      S::qldc(T + 4, tab + (3 * row + 0) * kNS); S::f2scale_g(fsL4, g, 0, n, T + 4);
      S::qldc(T + 4, tab + (3 * row + 1) * kNS); S::f2scale_g(fsL3, g, 2, n, T + 4);
      S::qldc(fsC, tab + (3 * row + 2) * kNS);
      S::f2mulxi(fsXL3, fsL3); S::f2mulxi(fsXL4, fsL4);
      row++;
    } else {
    // ---- tangent at V (a = -M Z^2, b = 2 Y Z^3, c = M X - 2 Y^2; the curve has A = 0), V <- 2V ----
    // (independent products grouped: 13 of them in five calls)
    S::qsqr3(T, fsZ, T + 5, fsX, T + 2, fsY);                            // Z^2, X^2, Y^2
    S::qdbl(T + 1, T + 5); S::qadd(T + 1, T + 1, T + 5);                // M = 3 X^2
    S::qmul2(T + 4, T + 1, T, T + 3, fsY, fsZ);                          // M Z^2, Y Z
    S::qneg(T + 4, T + 4);                                              // a
    S::f2scale_g(fsL4, g, 0, n, T + 4);                                 // L4 = Qx a
    S::qdbl(T + 3, T + 3);                                              // Z' = 2 Y Z
    S::qmul2(T + 4, T + 3, T, fsC, T + 1, fsX);                         // b = Z' Z^2, M X
    S::f2scale_g(fsL3, g, 2, n, T + 4);                                 // L3 = Qy b
    S::qsub(fsC, fsC, T + 2); S::qsub(fsC, fsC, T + 2);                 // c = M X - 2 Y^2
    S::f2mulxi(fsXL3, fsL3); S::f2mulxi(fsXL4, fsL4);
    if (m != 0) {
      S::qcopy(fsZ, T + 3);
      S::qmul1sqr2(T + 5, fsX, T + 2, fsX, T + 1, T + 2, T + 2);         // X Y^2, M^2, Y^4
      S::qdbl(T + 5, T + 5, 2);                                         // S = 4 X Y^2
      S::qsub(fsX, fsX, T + 5); S::qsub(fsX, fsX, T + 5);               // X' = M^2 - 2 S
      S::qdbl(T + 2, T + 2, 3);                                         // 8 Y^4
      S::qsub(T + 5, T + 5, fsX); S::qmul(fsY, T + 1, T + 5); S::qsub(fsY, fsY, T + 2);   // Y'
    }
    }
    S::line_mul(T, V);
    { int s = V; V = T; T = s; }
    if (m == 0) break;
    if ((c_ccnaf.nz[m >> 5] >> (m & 31)) & 1u) {
      const bool minus = (c_ccnaf.neg[m >> 5] >> (m & 31)) & 1u;
      if (tab) {
        S::qldc(T + 4, tab + (3 * row + 0) * kNS); S::f2scale_g(fsL4, g, 0, n, T + 4);
        S::qldc(T + 4, tab + (3 * row + 1) * kNS); S::f2scale_g(fsL3, g, 2, n, T + 4);
        S::qldc(fsC, tab + (3 * row + 2) * kNS);
        S::f2mulxi(fsXL3, fsL3); S::f2mulxi(fsXL4, fsL4);
        row++;
      } else {
      // ---- chord through V and +-P (a = Y - yS Z^3, b = (xP Z^2 - X) Z, c = yS Z X - xP Y), V <- V +- P ----
      // (14 products in six calls of independent pairs / triples)
      S::qldg(T + 6, g, 4, n, false);                    // xP
      S::qldg(T + 7, g, 5, n, minus);                    // yS
      S::qmul3(T, fsZ, fsZ, T + 8, T + 7, fsZ, T + 9, T + 6, fsY);       // Z^2, yS Z, xP Y
      S::qmul2(T + 1, T, fsZ, T + 2, T + 6, T);                          // Z^3, xP Z^2
      S::qsub(T + 2, T + 2, fsX);                                        // H = xP Z^2 - X
      S::qmul3(T + 3, T + 7, T + 1, T + 4, T + 2, fsZ, T + 8, T + 8, fsX);   // yS Z^3, b = H Z, yS Z X
      S::qsub(T + 5, fsY, T + 3);                                        // a = Y - yS Z^3
      S::f2scale_g(fsL4, g, 0, n, T + 5);
      S::qsub(T + 3, T + 3, fsY);                                        // R = yS Z^3 - Y
      S::f2scale_g(fsL3, g, 2, n, T + 4);
      S::qsub(fsC, T + 8, T + 9);                                        // c
      S::f2mulxi(fsXL3, fsL3); S::f2mulxi(fsXL4, fsL4);
      S::qcopy(fsZ, T + 4);                                              // Z of the sum
      S::qmul2(T, T + 2, T + 2, T + 10, T + 3, T + 3);                   // H^2, R^2
      S::qmul2(T + 1, T, T + 2, T, T, fsX);                              // H^3, X H^2
      S::qsub(fsX, T + 10, T + 1); S::qsub(fsX, fsX, T); S::qsub(fsX, fsX, T);   // X3 = R^2 - H^3 - 2 X H^2
      S::qsub(T, T, fsX);
      S::qmul2(T, T, T + 3, T + 1, T + 1, fsY);                          // R (X H^2 - X3), H^3 Y
      S::qsub(fsY, T, T + 1);                                            // Y3
      }
      S::line_mul(T, V);
      { int s = V; V = T; T = s; }
    }
    m--;
    S::f12sqr(V, T, fsL3);                   // the line's slots are dead here: scratch
  }
  if (!live) return;
  // publish (flagged-off inputs: the identity)
  Fq x;
#pragma unroll 1
  for (int s = 0; s < 12; s++) {
    S::ld(x, V + s);
    if (!ok) { if (s == 0) fq_one(x); else fq_zero(x); }
    fq_st_global(mv, s, n, idx, x);
  }
  flag[idx] = ok ? 1u : 0u;
}

// ---------------------------------------------------------------------------------------------
// Final exponentiation on the slot machine (f_tateexp, ecc/f_param.c:250-283; same route as
// f12_final_exp of pairing_f.cuh).  The easy part (one F_q^12 inversion, a tenth of the work) and the
// change of basis on the way out run on the structs of pairing_f.cuh; the hard part -- three powers
// by the BN parameter and the multiplication chain -- runs on slots: two resident F_q^12 values, the
// 12-slot scratch and two spare F_q^2 (40 slots = 800 B per thread; the spares hold xi b_1, xi b_2 inside f6mul), everything else parked in a
// limb-major global stash of four F_q^12 per pairing (about a dozen 240-byte moves each way).
// mv is overwritten (it holds f after the easy part).  Needs c_f.bn and c_f.slots_ok.
// ---------------------------------------------------------------------------------------------
constexpr int kFFinalSlots = 40;
constexpr int kFStashWords = 4 * kF12Words;

template <int BLOCK>
__global__ void __launch_bounds__(BLOCK)
k_f_finalexp_s(uint32_t* __restrict__ mv, const uint32_t* __restrict__ flag, uint8_t* __restrict__ out,
               uint32_t* __restrict__ stash, size_t n) {
  using S = FS<BLOCK>;
  enum { R0 = 0, R1 = 12, T = 24, E = 36 };
  size_t idx = (size_t)blockIdx.x * BLOCK + threadIdx.x;
  const bool live = idx < n;               // padding threads run the powers by u too (block-wide barriers inside)
  if (!live) idx = 0;
  const bool ok = flag[idx] != 0;
  uint32_t* g0 = mv + idx;                                     // f
  uint32_t* g1 = stash + idx;                                  // f^u
  uint32_t* g2 = g1 + (size_t)kF12Words * n;                   // f^(u^2)
  uint32_t* g3 = g2 + (size_t)kF12Words * n;
  uint32_t* g4 = g3 + (size_t)kF12Words * n;
  {
    F12 f, x, y;
    f12_ld_global(f, mv, n, idx);
    if (!ok) f12_one(f);
    f12_inv(&x, &f);
    f12_conj(y, f);
    f12_mul(&x, &x, &y);                 // f^(q^6 - 1)
    f12_frob(y, x, 2);
    f12_mul(&f, &y, &x);                 // ^(q^2 + 1)
    if (live) f12_st_global(mv, n, idx, f);
#pragma unroll 1
    for (int i = 0; i < 6; i++) { S::st(R1 + 2 * i, f.c[i].a); S::st(R1 + 2 * i + 1, f.c[i].b); }
  }
  S::f12powu(R0, R1, T, E);              // f^u
  S::f12stg(g1, n, R0, live);
  S::f12copy(R1, R0);
  S::f12powu(R0, R1, T, E);              // f^(u^2)
  S::f12stg(g2, n, R0, live);
  S::f12copy(R1, R0);
  S::f12powu(R0, R1, T, E);              // f^(u^3)
  // t0 = y6^2, y6 = 1 / (f^(u^3) f^(u^3 q))
  S::f12copy(R1, R0);
  S::f12frob(R1, 1);
  S::f12mul(R1, R0, T, E);
  S::f12conj(R1);
  S::f12cycsqr(R1, T, E);
  S::f12stg(g3, n, R1, live);                  // park t0
  // y4 = 1 / (f^u f^(u^2 q))
  S::f12ldg(R0, g2, n);
  S::f12frob(R0, 1);
  S::f12ldg(R1, g1, n);
  S::f12mul(R0, R1, T, E);
  S::f12conj(R0);
  S::f12ldg(R1, g3, n);
  S::f12mul(R1, R0, T, E);                  // t0 *= y4
  // y5 = 1 / f^(u^2)
  S::f12ldg(R0, g2, n);
  S::f12conj(R0);
  S::f12mul(R1, R0, T, E);                  // t0 *= y5
  S::f12stg(g3, n, R1, live);                  // park t0
  // t1 = y3 y5 t0, y3 = 1 / f^(u q)
  S::f12ldg(R1, g1, n);
  S::f12frob(R1, 1);
  S::f12conj(R1);
  S::f12mul(R1, R0, T, E);
  S::f12ldg(R0, g3, n);
  S::f12mul(R1, R0, T, E);                  // R0 = t0, R1 = t1
  // t0 *= y2, y2 = f^(u^2 q^2)
  S::f12stg(g4, n, R1, live);                  // park t1
  S::f12ldg(R1, g2, n);
  S::f12frob(R1, 2);
  S::f12mul(R0, R1, T, E);
  S::f12ldg(R1, g4, n);
  S::f12cycsqr(R1, T, E);
  S::f12mul(R1, R0, T, E);
  S::f12cycsqr(R1, T, E);                // t1 = (t1^2 t0)^2
  // t0 = t1 y1, y1 = 1 / f
  S::f12ldg(R0, g0, n);
  S::f12conj(R0);
  S::f12mul(R0, R1, T, E);
  S::f12stg(g3, n, R0, live);                  // park t0
  S::f12stg(g4, n, R1, live);                  // park t1
  // y0 = f^q f^(q^2) f^(q^3)
  S::f12ldg(R0, g0, n);
  S::f12frob(R0, 1);
  S::f12ldg(R1, g0, n);
  S::f12frob(R1, 2);
  S::f12mul(R0, R1, T, E);
  S::f12ldg(R1, g0, n);
  S::f12frob(R1, 3);
  S::f12mul(R0, R1, T, E);
  S::f12ldg(R1, g4, n);
  S::f12mul(R1, R0, T, E);                  // t1 *= y0
  S::f12ldg(R0, g3, n);
  S::f12cycsqr(R0, T, E);
  S::f12mul(R0, R1, T, E);                  // result
  if (!live) return;
  {
    F12 acc;
#pragma unroll 1
    for (int i = 0; i < 6; i++) { S::ld(acc.c[i].a, R0 + 2 * i); S::ld(acc.c[i].b, R0 + 2 * i + 1); }
    f12_to_reference(acc);
    if (!ok) f12_one(acc);
    uint8_t* o = out + idx * (12 * kWS);
#pragma unroll 1
    for (int i = 0; i < 6; i++) {
      fq_to_wire(o + (2 * i) * kWS, F12C(acc, i).a);
      fq_to_wire(o + (2 * i + 1) * kWS, F12C(acc, i).b);
    }
  }
}

}  // namespace pbcb200
