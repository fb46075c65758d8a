// engine_d_wide.h -- what engine.cu calls in engine_d_wide.cu (the eight-limb type D instance).
// The constants are handed over as byte images of the eight-limb structs (CCConstsT<8>, DConstsT<8>,
// ZrConstsT<8>, FqWideConstsT<8>, G2HashConstsT<8>; FpConsts, CCNaf and HashConsts do not depend on the limb count);
// dw_upload checks every size against its own structs.  Launchers enqueue on `st` and do not synchronise.
#ifndef PBC_ENGINE_D_WIDE_H
#define PBC_ENGINE_D_WIDE_H
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

namespace pbcb200_dw {

constexpr int kLimbs = 8;

struct DWideConsts {
  const void *fp, *cc, *naf, *d, *zr, *hash, *x, *g2h;
  size_t fp_bytes, cc_bytes, naf_bytes, d_bytes, zr_bytes, hash_bytes, x_bytes, g2h_bytes;
};

// -1: a size differs from this instance's structs; -2: no eight-limb instance in this build (a CPU
// simulator made from engine.cu alone); otherwise the cudaError_t of the copies
int dw_upload(const DWideConsts& c);
void dw_miller(const uint8_t* P, const uint8_t* Q, uint32_t* mv, uint32_t* flag, size_t m, size_t stride1,
               const uint32_t* tab, size_t rows, cudaStream_t st);
void dw_prod(const uint32_t* mv, const uint32_t* flag, uint32_t* mvo, uint32_t* flago, size_t k, size_t n,
             size_t m, cudaStream_t st);
// one pass of the segmented product (prod_v.cuh): runs[r] .. runs[r + 1] of (mv, flag), stride n, into
// element r of (mvo, flago), stride n_o
void dw_prod_v(const uint32_t* mv, const uint32_t* flag, size_t n, uint32_t* mvo, uint32_t* flago, size_t n_o,
               const uint64_t* runs, size_t n_runs, cudaStream_t st);
void dw_finalexp(const uint32_t* mv, const uint32_t* flag, uint8_t* out, size_t n, cudaStream_t st);
void dw_pp_init(const uint8_t* P, uint32_t* tab, size_t rows, cudaStream_t st);
// which: 0 = G1, 1 = GT, 2 = G2 (as engine.cu's enqueue_group)
void dw_group(int which, uint8_t* out, const uint8_t* in, const uint8_t* k, size_t n, cudaStream_t st);
void dw_from_hash(const uint8_t* data, int len, uint8_t* out, size_t n, cudaStream_t st);
void dw_decompress(const uint8_t* in, uint8_t* out, size_t n, cudaStream_t st);
// element_from_hash and element_from_bytes_compressed on G2 (the twist over F_q^3)
void dw_g2_from_hash(const uint8_t* data, int len, uint8_t* out, size_t n, cudaStream_t st);
void dw_g2_decompress(const uint8_t* in, uint8_t* out, size_t n, cudaStream_t st);
void dw_tower_op(int op, uint8_t* out, const uint8_t* a, const uint8_t* b, size_t n, cudaStream_t st);
void dw_fq_op(int op, uint8_t* out, const uint8_t* a, const uint8_t* b, size_t n, cudaStream_t st);

}  // namespace pbcb200_dw
#endif
