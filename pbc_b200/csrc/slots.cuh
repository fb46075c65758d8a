// slots.cuh -- per-thread "field register file" in shared memory + out-of-line field operations.
//
// One pairing runs per thread.  A 512-bit F_q element is 16 registers; the Miller loop of
// ecc/a_param.c:1053-1198 keeps ~14 of them live, which does not fit the register file at any
// useful occupancy and, fully inlined, would unroll to hundreds of KB of SASS.  Instead every
// long-lived element lives in a *slot* of shared memory and each field operation is a single
// out-of-line routine (one copy of the ~560-IMAD multiplier in the instruction cache):
//
//     slot s, 16-byte vector v, thread t  ->  smem[(s * VPE + v) * BLOCK + t]   (uint4 / uint2)
//
// so a warp's access to one vector is 32 consecutive 16-byte words: conflict-free LDS.128 /
// STS.128.  An operation loads its operands (8 LDS.128), runs entirely in registers, and stores
// the result (4 STS.128): ~12 shared-memory instructions against ~540 IMAD.WIDE.
#pragma once
#include "fp.cuh"

namespace pbcb200 {

extern __shared__ uint4 pbc_smem[];

template <int N, bool FULL, int BLOCK>
struct Ops {
  static constexpr int kVecWords = (N % 4 == 0) ? 4 : 2;
  static constexpr int kVecs = N / kVecWords;
  static constexpr int kSlotBytes = N * 4 * BLOCK;

  static __device__ __forceinline__ void ld(uint32_t* r, int s) {
    if constexpr (kVecWords == 4) {
      const uint4* b = pbc_smem + s * (kVecs * BLOCK) + threadIdx.x;
#pragma unroll
      for (int v = 0; v < kVecs; v++) {
        uint4 q = b[v * BLOCK];
        r[4 * v] = q.x; r[4 * v + 1] = q.y; r[4 * v + 2] = q.z; r[4 * v + 3] = q.w;
      }
    } else {
      const uint2* b = reinterpret_cast<const uint2*>(pbc_smem) + s * (kVecs * BLOCK) + threadIdx.x;
#pragma unroll
      for (int v = 0; v < kVecs; v++) {
        uint2 q = b[v * BLOCK];
        r[2 * v] = q.x; r[2 * v + 1] = q.y;
      }
    }
  }
  static __device__ __forceinline__ void st(int s, const uint32_t* r) {
    if constexpr (kVecWords == 4) {
      uint4* b = pbc_smem + s * (kVecs * BLOCK) + threadIdx.x;
#pragma unroll
      for (int v = 0; v < kVecs; v++)
        b[v * BLOCK] = make_uint4(r[4 * v], r[4 * v + 1], r[4 * v + 2], r[4 * v + 3]);
    } else {
      uint2* b = reinterpret_cast<uint2*>(pbc_smem) + s * (kVecs * BLOCK) + threadIdx.x;
#pragma unroll
      for (int v = 0; v < kVecs; v++) b[v * BLOCK] = make_uint2(r[2 * v], r[2 * v + 1]);
    }
  }

  // ---- out-of-line operations on slots (d may alias a or b) ----
  static __device__ __noinline__ void mul(int d, int a, int b) {
    uint32_t x[N], y[N];
    ld(x, a); ld(y, b);
    fp_mul<N, FULL>(x, x, y);
    st(d, x);
  }
  static __device__ __noinline__ void sqr(int d, int a) {
    uint32_t x[N];
    ld(x, a);
    fp_sqr<N, FULL>(x, x);
    st(d, x);
  }
  // ---- ONE multiplier routine for the kernels that need operand variants (k_a_miller9, k_a_miller9_shared) ----
  // d = x * y with  x = a [+ a2],  y = b [+ b2 | - b2]  or  y = the element at g (limb-major global
  // array, vectors n apart: a value used once or twice per loop iteration lives in L2 instead of a
  // slot).  All branches are warp-uniform.  One copy of the 528-product body instead of one per
  // variant: with 12 warps per SM the four separate copies (mul, mul2<+>, mul2<->, mulg: 3 200
  // instructions, 51 KB) made instruction fetch a leading stall.
  static constexpr uint32_t MX_ADD_A = 1u, MX_ADD_B = 2u, MX_SUB_B = 4u, MX_GLOBAL_B = 8u;
  // r = the element at g (limb-major global array, vectors n apart)
  static __device__ __forceinline__ void ld_g(uint32_t* r, const void* g, size_t n) {
    if constexpr (kVecWords == 4) {
      const uint4* p = reinterpret_cast<const uint4*>(g);
#pragma unroll
      for (int v = 0; v < kVecs; v++) {
        uint4 q = p[v * n];
        r[4 * v] = q.x; r[4 * v + 1] = q.y; r[4 * v + 2] = q.z; r[4 * v + 3] = q.w;
      }
    } else {
      const uint2* p = reinterpret_cast<const uint2*>(g);
#pragma unroll
      for (int v = 0; v < kVecs; v++) {
        uint2 q = p[v * n];
        r[2 * v] = q.x; r[2 * v + 1] = q.y;
      }
    }
  }
  static __device__ __noinline__ void mulx(int d, int a, int b, uint32_t mode, int a2, int b2, const void* g, size_t n) {
    uint32_t x[N], y[N];
    if (mode & MX_GLOBAL_B) ld_g(y, g, n);
    else ld(y, b);
    if (mode & (MX_ADD_B | MX_SUB_B)) {
      ld(x, b2);
      if (mode & MX_ADD_B) fp_add<N, FULL>(y, y, x); else fp_sub<N>(y, y, x);
    }
    ld(x, a);
    if (mode & MX_ADD_A) {
      uint32_t z[N];
      ld(z, a2);
      fp_add<N, FULL>(x, x, z);
    }
    fp_mul<N, FULL>(x, x, y);
    st(d, x);
  }
  template <bool SUBB>
  static __device__ __forceinline__ void mul2(int d, int a, int a2, int b, int b2) {
    mulx(d, a, b, MX_ADD_A | (SUBB ? MX_SUB_B : MX_ADD_B), a2, b2, nullptr, 0);
  }
  static __device__ __forceinline__ void mulg(int d, int a, const void* g, size_t n) {
    mulx(d, a, 0, MX_GLOBAL_B, 0, 0, g, n);
  }
  static __device__ __forceinline__ void mulp(int d, int a, int b) { mulx(d, a, b, 0, 0, 0, nullptr, 0); }

  // ---- ONE squaring routine with its additions folded in, as mulx is for products ----
  //   d = 2^k (a [+ a2])^2 [- s1] [- s2]
  // Each folded addition is a separate out-of-line call less: a shared-memory round trip of its operands during
  // which the warp feeds the multiplier nothing.  Every intermediate is fully reduced, so d is the value the
  // separate calls give.  All branches are warp-uniform; d may alias any operand.
  static constexpr uint32_t SX_ADD_A = 1u, SX_SUB_1 = 2u, SX_SUB_2 = 4u;
  static __device__ __noinline__ void sqrx(int d, int a, uint32_t mode, int a2, int k, int s1, int s2) {
    uint32_t x[N], y[N];
    ld(x, a);
    if (mode & SX_ADD_A) {
      ld(y, a2);
      fp_add<N, FULL>(x, x, y);
    }
    fp_sqr<N, FULL>(x, x);
    for (int i = 0; i < k; i++) fp_add<N, FULL>(x, x, x);
    const int subs = (mode & SX_SUB_1) ? ((mode & SX_SUB_2) ? 2 : 1) : 0;
#pragma unroll 1
    for (int i = 0; i < subs; i++) {
      ld(y, i ? s2 : s1);
      fp_sub<N>(x, x, y);
    }
    st(d, x);
  }
  static __device__ __forceinline__ void sqrp(int d, int a) { sqrx(d, a, 0, 0, 0, 0, 0); }

  // ---- lazy reduction (fp.cuh mul_wide / redc_wide; FULL, even N) ----
  //   d = (a0 b0 [+- a1 b1] [+ q R] [- S]) / R mod q,   S = the unreduced value in slots (s0, s1)
  // One Montgomery reduction for the whole sum: a second product costs N^2 IMAD.WIDE, not N^2 + N^2 + N.
  // LZ_GLOBAL_B: b0 is the element at g (as in mulx).  LZ_KARATSUBA (with LZ_TWO): also stores
  // S' = a0 b0 + a1 b1, less q R if that is >= q R, into (s0, s1), a0 + a1 into a0 and b0 + b1 into b0.
  // The caller keeps the sum in [0, 2 q R).  One 256-product body and one reduction body: the terms
  // are a loop, not unrolled.  d may alias any operand slot (everything is read before d is written).
  static constexpr uint32_t LZ_TWO = 1u, LZ_SUB = 2u, LZ_ADD_QR = 4u, LZ_SUB_S = 8u, LZ_GLOBAL_B = 16u,
                            LZ_KARATSUBA = 32u;
  static __device__ __noinline__ void lazy(int d, uint32_t mode, int a0, int b0, int a1, int b1, int s0, int s1,
                                           const void* g, size_t n) {
    static_assert(FULL && N % 2 == 0, "lazy reduction: 512-bit field");
    uint32_t acc[2 * N + 1];
    if (mode & LZ_SUB_S) {
      uint32_t z[2 * N];
      ld(z, s0); ld(z + N, s1);
#pragma unroll
      for (int k = 0; k <= 2 * N; k++) acc[k] = 0;
      wide_sub<N>(acc, z);
    } else {
#pragma unroll
      for (int k = 0; k <= 2 * N; k++) acc[k] = 0;
    }
    const int terms = (mode & LZ_TWO) ? 2 : 1;
#pragma unroll 1
    for (int t = 0; t < terms; t++) {
      uint32_t x[N], y[N], p[2 * N];
      if (t == 0 && (mode & LZ_GLOBAL_B)) ld_g(y, g, n);
      else ld(y, t ? b1 : b0);
      ld(x, t ? a1 : a0);
      mul_wide<N>(p, x, y);
      if (t == 1 && (mode & LZ_KARATSUBA)) {
        uint32_t s[2 * N + 1];
#pragma unroll
        for (int k = 0; k <= 2 * N; k++) s[k] = acc[k];
        wide_add<N>(s, p);
        wide_sub_pR_if_ge<N>(s);
        st(s0, s); st(s1, s + N);
      }
      if (t == 1 && (mode & LZ_SUB)) wide_sub<N>(acc, p);
      else wide_add<N>(acc, p);
    }
    if (mode & LZ_ADD_QR) wide_add_pR<N>(acc);
    if (mode & LZ_KARATSUBA) {
      uint32_t x[N], y[N];
      ld(x, a0); ld(y, a1);
      fp_add<N, FULL>(x, x, y);
      st(a0, x);
      ld(x, b0); ld(y, b1);
      fp_add<N, FULL>(x, x, y);
      st(b0, x);
    }
    uint32_t r[N];
    redc_wide<N>(r, acc);
    st(d, r);
  }
  // d = a*b - c
  static __device__ __noinline__ void mulsub(int d, int a, int b, int c) {
    uint32_t x[N], y[N];
    ld(x, a); ld(y, b);
    fp_mul<N, FULL>(x, x, y);
    ld(y, c);
    fp_sub<N>(x, x, y);
    st(d, x);
  }
  // d = a^2 - c, c a constant (not a slot: one slot fewer for the Lucas ladder of k_a_finalexp)
  static __device__ __noinline__ void sqrsub(int d, int a, const uint32_t* c) {
    uint32_t x[N], y[N];
    ld(x, a);
    fp_sqr<N, FULL>(x, x);
#pragma unroll
    for (int k = 0; k < N; k++) y[k] = c[k];
    fp_sub<N>(x, x, y);
    st(d, x);
  }
  static __device__ __noinline__ void add(int d, int a, int b) {
    uint32_t x[N], y[N];
    ld(x, a); ld(y, b);
    fp_add<N, FULL>(x, x, y);
    st(d, x);
  }
  static __device__ __noinline__ void sub(int d, int a, int b) {
    uint32_t x[N], y[N];
    ld(x, a); ld(y, b);
    fp_sub<N>(x, x, y);
    st(d, x);
  }
  // d = 2^k * a
  static __device__ __noinline__ void dbl(int d, int a, int k = 1) {
    uint32_t x[N];
    ld(x, a);
    for (int i = 0; i < k; i++) fp_add<N, FULL>(x, x, x);
    st(d, x);
  }
  static __device__ __noinline__ void neg(int d, int a) {
    uint32_t x[N];
    ld(x, a);
    fp_neg<N>(x, x);
    st(d, x);
  }
  static __device__ __noinline__ void halve(int d, int a, int k = 1) {
    uint32_t x[N];
    ld(x, a);
    for (int i = 0; i < k; i++) fp_halve<N, FULL>(x, x);
    st(d, x);
  }
  static __device__ __forceinline__ void copy(int d, int a) {
    uint32_t x[N];
    ld(x, a);
    st(d, x);
  }
  static __device__ __forceinline__ void set_const(int d, const uint32_t* c) {
    uint32_t x[N];
#pragma unroll
    for (int k = 0; k < N; k++) x[k] = c[k];
    st(d, x);
  }
  static __device__ __forceinline__ bool is_zero(int a) {
    uint32_t x[N];
    ld(x, a);
    return fp_is_zero<N>(x);
  }
  static __device__ __forceinline__ bool eq(int a, int b) {
    uint32_t x[N], y[N];
    ld(x, a); ld(y, b);
    return fp_eq<N>(x, y);
  }

  // ---- global <-> slot, limb-major batch arrays:  g[(e * kVecs + v) * n + idx]  ----
  static __device__ __forceinline__ void ld_global(int s, const void* g, int e, size_t n, size_t idx) {
    uint32_t x[N];
    if constexpr (kVecWords == 4) {
      const uint4* b = reinterpret_cast<const uint4*>(g) + (size_t)e * kVecs * n + idx;
#pragma unroll
      for (int v = 0; v < kVecs; v++) {
        uint4 q = b[v * n];
        x[4 * v] = q.x; x[4 * v + 1] = q.y; x[4 * v + 2] = q.z; x[4 * v + 3] = q.w;
      }
    } else {
      const uint2* b = reinterpret_cast<const uint2*>(g) + (size_t)e * kVecs * n + idx;
#pragma unroll
      for (int v = 0; v < kVecs; v++) {
        uint2 q = b[v * n];
        x[2 * v] = q.x; x[2 * v + 1] = q.y;
      }
    }
    st(s, x);
  }
  static __device__ __forceinline__ void st_global(void* g, int e, size_t n, size_t idx, int s) {
    uint32_t x[N];
    ld(x, s);
    if constexpr (kVecWords == 4) {
      uint4* b = reinterpret_cast<uint4*>(g) + (size_t)e * kVecs * n + idx;
#pragma unroll
      for (int v = 0; v < kVecs; v++)
        b[v * n] = make_uint4(x[4 * v], x[4 * v + 1], x[4 * v + 2], x[4 * v + 3]);
    } else {
      uint2* b = reinterpret_cast<uint2*>(g) + (size_t)e * kVecs * n + idx;
#pragma unroll
      for (int v = 0; v < kVecs; v++) b[v * n] = make_uint2(x[2 * v], x[2 * v + 1]);
    }
  }
};

// ---------------------------------------------------------------------------------------------
// wire format (arith/montfp.c:487-517): big-endian, fixed width WB bytes per F_q coordinate.
// ---------------------------------------------------------------------------------------------
// bytes -> little-endian 32-bit limbs (not yet reduced, not yet Montgomery)
template <int N, int WB>
__device__ __forceinline__ void limbs_from_be(uint32_t* x, const uint8_t* p) {
  static_assert(WB % 4 == 0 && WB <= 4 * N, "coordinate width");
#pragma unroll
  for (int k = 0; k < N; k++) {
    if (k < WB / 4) {
      uint32_t w = *reinterpret_cast<const uint32_t*>(p + WB - 4 - 4 * k);
      x[k] = __byte_perm(w, 0, 0x0123);
    } else {
      x[k] = 0;
    }
  }
}
// the same from a byte pointer of any alignment
template <int N, int WB>
__device__ __forceinline__ void limbs_from_be_bytes(uint32_t* x, const uint8_t* p) {
#pragma unroll
  for (int k = 0; k < N; k++) {
    if (k < WB / 4) {
      const uint8_t* b = p + WB - 4 - 4 * k;
      x[k] = ((uint32_t)b[0] << 24) | ((uint32_t)b[1] << 16) | ((uint32_t)b[2] << 8) | b[3];
    } else {
      x[k] = 0;
    }
  }
}
template <int N, int WB>
__device__ __forceinline__ void limbs_to_be(uint8_t* p, const uint32_t* x) {
#pragma unroll
  for (int k = 0; k < WB / 4; k++)
    *reinterpret_cast<uint32_t*>(p + WB - 4 - 4 * k) = __byte_perm(x[k], 0, 0x0123);
}

}  // namespace pbcb200
