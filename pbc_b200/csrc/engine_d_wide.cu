// engine_d_wide.cu -- the type D kernels on eight 32-bit limbs (R = 2^256), for MNT parameter sets with
// 160- to 255-bit q (the bundled d277699-175-167, d278027-190-181, d105171-196-185, d201 and d224).
//
// The same sources as the five-limb type D path of engine.cu (fq_small.cuh, miller_cc.cuh,
// pairing_d.cuh, group_cc.cuh), compiled a second time with PBC_NS = 8 into a namespace of their own,
// so that the kernels and the __constant__ symbols of the two instances never meet: the five-limb
// kernels compile exactly as before.  Differences of this instance, all selected at compile time:
//   * the wire width ceil(bits(q)/8) (22 .. 32 bytes) is a run-time constant (c_fqx.wb);
//   * single products are mont_mul<8, false>, the lazy F_q^3 product uses the double-width
//     product and reduction of fp.cuh (mul_wide<8>, redc_wide<8>);
//   * scalars have eight words (r < 2^255);
//   * q = 1 mod 8 takes Tonelli-Shanks square roots (element_from_hash, compressed points).
// engine.cu derives the constants and calls the launchers at the end of this file; nothing else of
// this translation unit is visible outside it.
#define PBC_NS 8
#define PBC_FQ_WIDE 1
#define PBC_ZR_WORDS 8
// every header opens `namespace pbcb200`; here that namespace is pbcb200_dw
#define pbcb200 pbcb200_dw

#include <cuda_runtime.h>
#include <string.h>

#include "engine_d_wide.h"
#include "group_cc.cuh"

namespace pbcb200 {

static constexpr int kBlockWMiller = kCCMillerBlock;   // as engine.cu's type D kernels
static constexpr int kBlockW = 128;

static unsigned grid(size_t n, int block) { return (unsigned)((n + block - 1) / block); }

int dw_upload(const DWideConsts& c) {
  if (c.fp_bytes != sizeof(FpConsts) || c.cc_bytes != sizeof(CCConsts) || c.naf_bytes != sizeof(CCNaf) ||
      c.d_bytes != sizeof(DConsts) || c.zr_bytes != sizeof(ZrConsts) || c.hash_bytes != sizeof(HashConsts) ||
      c.x_bytes != sizeof(FqWideConstsT<kNS>) || c.g2h_bytes != sizeof(G2HashConsts))
    return -1;
  cudaError_t e;
  if ((e = cudaMemcpyToSymbol(c_fp, c.fp, c.fp_bytes)) != cudaSuccess) return e;
  if ((e = cudaMemcpyToSymbol(c_cc, c.cc, c.cc_bytes)) != cudaSuccess) return e;
  if ((e = cudaMemcpyToSymbol(c_ccnaf, c.naf, c.naf_bytes)) != cudaSuccess) return e;
  if ((e = cudaMemcpyToSymbol(c_d, c.d, c.d_bytes)) != cudaSuccess) return e;
  if ((e = cudaMemcpyToSymbol(c_zr, c.zr, c.zr_bytes)) != cudaSuccess) return e;
  if ((e = cudaMemcpyToSymbol(c_hash, c.hash, c.hash_bytes)) != cudaSuccess) return e;
  if ((e = cudaMemcpyToSymbol(c_g2h, c.g2h, c.g2h_bytes)) != cudaSuccess) return e;
  return (int)cudaMemcpyToSymbol(c_fqx, c.x, c.x_bytes);
}

void dw_miller(const uint8_t* P, const uint8_t* Q, uint32_t* mv, uint32_t* flag, size_t m, size_t stride1,
               const uint32_t* tab, size_t rows, cudaStream_t st) {
  k_d_miller<kBlockWMiller><<<grid(m, kBlockWMiller), kBlockWMiller, 0, st>>>(P, Q, mv, flag, m, stride1, tab, rows);
}
void dw_prod(const uint32_t* mv, const uint32_t* flag, uint32_t* mvo, uint32_t* flago, size_t k, size_t n,
             size_t m, cudaStream_t st) {
  k_d_prod<kBlockW><<<grid(n, kBlockW), kBlockW, 0, st>>>(mv, flag, mvo, flago, k, n, m);
}
void dw_prod_v(const uint32_t* mv, const uint32_t* flag, size_t n, uint32_t* mvo, uint32_t* flago, size_t n_o,
               const uint64_t* runs, size_t n_runs, cudaStream_t st) {
  k_prod_v<ProdVCC<F6DProdV>, kBlockW><<<grid(n_runs, kBlockW), kBlockW, 0, st>>>(
      ProdVBuf{(void*)mv, (void*)flag, n}, ProdVBuf{mvo, flago, n_o}, runs, n_runs, 1);
}
void dw_finalexp(const uint32_t* mv, const uint32_t* flag, uint8_t* out, size_t n, cudaStream_t st) {
  k_d_finalexp<kBlockW><<<grid(n, kBlockW), kBlockW, 0, st>>>(mv, flag, out, n);
}
void dw_pp_init(const uint8_t* P, uint32_t* tab, size_t rows, cudaStream_t st) {
  k_cc_pp_init<0><<<1, 32, 0, st>>>(P, tab, rows);
}
void dw_group(int which, uint8_t* out, const uint8_t* in, const uint8_t* k, size_t n, cudaStream_t st) {
  if (which == 0) k_cc_g1_mul<kBlockW, 0><<<grid(n, kBlockW), kBlockW, 0, st>>>(in, k, out, n);
  else if (which == 2) k_cc_g2_mul<KF3, kBlockW><<<grid(n, kBlockW), kBlockW, 0, st>>>(in, k, out, n);
  else k_d_gt_pow<kBlockW><<<grid(n, kBlockW), kBlockW, 0, st>>>(in, k, out, n);
}
void dw_from_hash(const uint8_t* data, int len, uint8_t* out, size_t n, cudaStream_t st) {
  k_cc_g1_from_hash<kBlockW, 0><<<grid(n, kBlockW), kBlockW, 0, st>>>(data, len, out, n);
}
void dw_decompress(const uint8_t* in, uint8_t* out, size_t n, cudaStream_t st) {
  k_cc_g1_decompress<kBlockW, 0><<<grid(n, kBlockW), kBlockW, 0, st>>>(in, out, n);
}
void dw_g2_from_hash(const uint8_t* data, int len, uint8_t* out, size_t n, cudaStream_t st) {
  k_cc_g2_from_hash<KF3, kBlockW><<<grid(n, kBlockW), kBlockW, 0, st>>>(data, len, out, n);
}
void dw_g2_decompress(const uint8_t* in, uint8_t* out, size_t n, cudaStream_t st) {
  k_cc_g2_decompress<KF3, kBlockW><<<grid(n, kBlockW), kBlockW, 0, st>>>(in, out, n);
}
void dw_tower_op(int op, uint8_t* out, const uint8_t* a, const uint8_t* b, size_t n, cudaStream_t st) {
  k_d_tower_op<<<grid(n, 64), 64, 0, st>>>(op, out, a, b, n);
}

// F_q differential-test hook of the eight-limb field (op as k_fq_op in engine.cu, plus 8 = a square root
// of a by the path element_from_hash takes, zero bytes where a is not a square)
__global__ void k_fqw_op(int op, uint8_t* __restrict__ out, const uint8_t* __restrict__ a,
                         const uint8_t* __restrict__ b, size_t n) {
  size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n) return;
  const int wb = fq_wb();
  Fq x, y;
  fq_from_wire(x, a + idx * wb);
  fq_from_wire(y, b + idx * wb);
  switch (op) {
    case 0: fq_mul(x, x, y); break;
    case 1: fq_add(x, x, y); break;
    case 2: fq_sub(x, x, y); break;
    case 3: fq_inv(&x, &x); break;
    case 4: fq_halve(x, x); break;
    case 5: fq_neg(x, x); break;
    case 6: fq_sqr(x, x); break;
    case 7: fq_mul(x, x, y); fq_sub(x, x, y); break;
    case 8: {
      Fq t = x, w;
      fq_sqrt_ts(&x, &t);
      fq_sqr(w, x);
      if (!fq_eq(w, t)) fq_zero(x);
      break;
    }
    case 9: {                                  // the lazy double-width product and reduction
      FqW t;
      fqw_mul(t, x, y);
      fqw_redc_os<true>(x, t);
      break;
    }
  }
  fq_to_wire(out + idx * wb, x);
}
void dw_fq_op(int op, uint8_t* out, const uint8_t* a, const uint8_t* b, size_t n, cudaStream_t st) {
  k_fqw_op<<<grid(n, 128), 128, 0, st>>>(op, out, a, b, n);
}

}  // namespace pbcb200
