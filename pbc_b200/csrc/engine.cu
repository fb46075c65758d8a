// engine.cu -- host side of libpbc_b200.so: parameter parsing, constant derivation, device
// contexts, chunked multi-stream / multi-GPU batch pipeline, and the C ABI of include/pbc_b200.h.
//
// Mirrors the *roles* of ecc/param.c (text -> symbol table), ecc/pairing.c:74-102
// (pairing_init_set_buf -> init_pairing) and the per-type init_pairing functions, but shares no
// code with them: constants are derived with host_bigint.hpp and the pairing itself only ever
// runs on the GPU.
#include <cuda_runtime.h>
#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <atomic>
#include <map>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "../../include/pbc_b200.h"
#include "common_kernels.cuh"
#include "host_bigint.hpp"
#include "host_fields.hpp"
#include "host_naf.hpp"
#include "pairing_a.cuh"
#include "pairing_a1.cuh"
#include "pairing_d.cuh"
#include "pairing_f.cuh"
#include "pairing_f_slots.cuh"
#include "pairing_g.cuh"
#include "pairing_e.cuh"
#include "group_a.cuh"
#include "group_a1.cuh"
#include "group_cc.cuh"
#include "group_e.cuh"
#include "engine_d_wide.h"

#if defined(PBC_HOST_SIM) && !defined(PBC_HOST_SIM_D_WIDE)
// A CPU simulator made from this translation unit alone has no eight-limb type D instance (that is
// engine_d_wide.cu, a second one): type D with 160..255-bit q initialises, but its first device call
// fails with an error instead of reaching a kernel.  tests/host/make_host_sim_d_wide.py appends the
// instance and defines PBC_HOST_SIM_D_WIDE.
namespace pbcb200_dw {
int dw_upload(const DWideConsts&) { return -2; }
void dw_miller(const uint8_t*, const uint8_t*, uint32_t*, uint32_t*, size_t, size_t, const uint32_t*, size_t, cudaStream_t) {}
void dw_prod(const uint32_t*, const uint32_t*, uint32_t*, uint32_t*, size_t, size_t, size_t, cudaStream_t) {}
void dw_prod_v(const uint32_t*, const uint32_t*, size_t, uint32_t*, uint32_t*, size_t, const uint64_t*, size_t, cudaStream_t) {}
void dw_finalexp(const uint32_t*, const uint32_t*, uint8_t*, size_t, cudaStream_t) {}
void dw_pp_init(const uint8_t*, uint32_t*, size_t, cudaStream_t) {}
void dw_group(int, uint8_t*, const uint8_t*, const uint8_t*, size_t, cudaStream_t) {}
void dw_from_hash(const uint8_t*, int, uint8_t*, size_t, cudaStream_t) {}
void dw_decompress(const uint8_t*, uint8_t*, size_t, cudaStream_t) {}
void dw_g2_from_hash(const uint8_t*, int, uint8_t*, size_t, cudaStream_t) {}
void dw_g2_decompress(const uint8_t*, uint8_t*, size_t, cudaStream_t) {}
void dw_tower_op(int, uint8_t*, const uint8_t*, const uint8_t*, size_t, cudaStream_t) {}
void dw_fq_op(int, uint8_t*, const uint8_t*, const uint8_t*, size_t, cudaStream_t) {}
}  // namespace pbcb200_dw
#endif

namespace pbcb200 {
__global__ void k_fqmul_chain(uint32_t* __restrict__ out, const uint32_t* __restrict__ in, int iters, int mode);
}
using namespace pbcb200;

// type a, element_prod_pairing: pairs of one product handled by one thread with a shared Miller
// accumulator (k_a_miller9_shared); 1 = one thread per pair (k_a_miller9).  Overridable per handle with the
// parameter key "b200_prod_share".
#ifndef PBC_A_PROD_SHARE
#define PBC_A_PROD_SHARE 2
#endif

// ------------------------------------------------------------------------------------------
// errors (misc/utils.c:79-101 pbc_error -> here a thread-local message)
// ------------------------------------------------------------------------------------------
static thread_local char g_err[512] = "";
static int fail(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof g_err, fmt, ap);
  va_end(ap);
  return 1;
}
#define CUDA_OK(call)                                                                   \
  do {                                                                                  \
    cudaError_t e_ = (call);                                                            \
    if (e_ != cudaSuccess)                                                              \
      return fail("CUDA error %s at %s:%d (%s)", cudaGetErrorString(e_), __FILE__, __LINE__, #call); \
  } while (0)

// device allocation released at scope exit (the test hooks allocate per call; an early error
// return must not leak)
struct DevBuf {
  void* p = nullptr;
  ~DevBuf() { if (p) cudaFree(p); }
  cudaError_t alloc(size_t bytes) { return cudaMalloc(&p, bytes ? bytes : 1); }
  template <class T> T* as() const { return static_cast<T*>(p); }
};

static std::atomic<uint64_t> g_launches{0};
#define LAUNCHED() g_launches.fetch_add(1, std::memory_order_relaxed)

// ------------------------------------------------------------------------------------------
// parameter text (ecc/param.c:42-111): whitespace-separated "key value" tokens, '#' comments
// ------------------------------------------------------------------------------------------
static std::map<std::string, std::string> parse_param_text(const char* s, size_t len) {
  std::map<std::string, std::string> tab;
  std::vector<std::string> tok;
  size_t i = 0;
  while (i < len && s[i]) {
    char c = s[i];
    if (c == '#') { while (i < len && s[i] && s[i] != '\n') i++; continue; }
    if (c == ' ' || c == '\t' || c == '\n' || c == '\r') { i++; continue; }
    size_t j = i;
    while (j < len && s[j] && s[j] != ' ' && s[j] != '\t' && s[j] != '\n' && s[j] != '\r' && s[j] != '#') j++;
    tok.emplace_back(s + i, j - i);
    i = j;
  }
  for (size_t k = 0; k + 1 < tok.size(); k += 2) tab[tok[k]] = tok[k + 1];
  return tab;
}

// ------------------------------------------------------------------------------------------
// handle
// ------------------------------------------------------------------------------------------
struct DevCtx {
  int dev = -1;
  bool ready = false;
  int sms = 132;               // multiprocessors of this device (queried in ctx_prepare; 132 on an H100 SXM)
  cudaStream_t stream[2] = {nullptr, nullptr};
  // host-API staging, per stream
  uint8_t* d_in1[2] = {nullptr, nullptr};
  uint8_t* d_in2[2] = {nullptr, nullptr};
  uint8_t* d_out[2] = {nullptr, nullptr};
  void* ws[2] = {nullptr, nullptr};
  size_t cap_in1[2] = {0, 0}, cap_in2[2] = {0, 0}, cap_out[2] = {0, 0}, cap_ws[2] = {0, 0};   // bytes
  // device-API workspace: one per handle and device, shared by every _device entry point and by the
  // host paths of the group operations.  ws_ev orders its users: each enqueue records it on its
  // stream and the next user's stream waits for it, so calls on different streams serialise on the
  // workspace instead of racing on it.
  void* ws_dev = nullptr;
  size_t cap_dev = 0;          // bytes
  cudaEvent_t ws_ev = nullptr;
  bool ws_used = false;
  // optional per-stage timing of the device-API path (bench.py roofline)
  cudaEvent_t ev[4] = {nullptr, nullptr, nullptr, nullptr};
  // pinned staging of the run tables of pbc_b200_prod_pairings_apply_v (upload_plan): a call copies its
  // table here and enqueues the upload, so it returns without waiting for the stream and never reads
  // the caller's offsets afterwards.  Slots are reused round robin once their last upload has run.
  static constexpr int kPlanSlots = 4;
  uint64_t* plan_h[kPlanSlots] = {};
  size_t plan_cap[kPlanSlots] = {};    // bytes
  cudaEvent_t plan_ev[kPlanSlots] = {};
  int plan_next = 0;
};

struct pbc_b200_pairing_s {
  int type = 0;                // 'a', 'e', 'f', 'd', 'g'; '1' = a1
  int g1_len = 0, g2_len = 0, gt_len = 0;
  int nlimbs = 0;
  bool full = false;
  FpConsts fp;
  AConsts a;
  A1Consts a1;
  A1GroupConsts a1g;
  A1Naf a1naf;
  size_t a1_rows = 0;          // rows of the fixed-argument line table (3 per tangent / chord)
  EConsts e;                   // type e (also uses fp, a1.wb and a1g.n / zlen: the 34-limb pieces of type a1)
  uint32_t e_pts[4 * kNA1];    // a, b, x(R), y(R), Montgomery form (g_e_pts)
  size_t cc_rows = 0;          // types f, d, g: lines of the Miller walk (computed once at init)
  CCConsts cc;
  CCNaf ccnaf;
  FConsts f;
  DConsts d;
  // type d with 160..255-bit q: the eight-limb instance (engine_d_wide.cu) and its constants; fp and
  // hash above serve both instances (their layout does not depend on the limb count)
  bool dwide = false;
  CCConstsT<pbcb200_dw::kLimbs> dw_cc;
  DConstsT<pbcb200_dw::kLimbs> dw_d;
  ZrConstsT<pbcb200_dw::kLimbs> dw_zr;
  FqWideConstsT<pbcb200_dw::kLimbs> dw_x;
  CCNaf dw_naf;
  GConsts g;
  ZrConsts zr;
  HashConsts hash;
  bool hash_ok = false;        // element_from_hash available (q = 3 mod 4 or 5 mod 8)
  // element_from_hash and compressed points on G2 (types f, d, g): square roots in the twist's field K
  G2HashConsts g2h;
  G2HashConstsT<pbcb200_dw::kLimbs> dw_g2h;
  bool g2_hash_ok = false;
  int zr_len = 20;
  int ndev = 1;
  bool profile = false;        // record CUDA events between the kernels of the device-API path
  bool force_reference_basis = false;   // test switches, from "b200_*" keys of the parameter text
  bool force_generic_final_exp = false;
  int prod_share = PBC_A_PROD_SHARE;   // type a products: pairs per thread sharing one Miller accumulator ("b200_prod_share")
  bool prod_share_forced = false;      // set through the parameter key: use it whatever the batch size (tests, A/B runs)
  std::vector<DevCtx> ctx;     // indexed by device ordinal
  std::map<std::string, std::vector<BigUInt>> derived;   // canonical values of the derived constants (tests)
  std::mutex mu;
  uint64_t id;
};

static std::atomic<uint64_t> g_next_id{1};

static std::mutex g_const_mu;
static std::map<int, uint64_t> g_const_owner;   // device -> handle id whose constants are resident
// The curve constants live in __constant__ memory, one set per device at a time.  Blocking (host
// buffer) calls hold the device's lock from the constant check to their final synchronise, so calls
// on different handles from different threads serialise per device instead of racing on the
// constants.  The asynchronous _device entry points cannot hold it across the caller's stream: use
// one handle per device at a time there (documented in include/pbc_b200.h).
static std::mutex g_dev_mu[64];

static constexpr size_t kChunk = 1u << 18;      // pairings per pipeline chunk (host API)
static constexpr int kBlockMiller = 128;
static constexpr int kBlockFinal = 128;
static constexpr int kBlockInv = 128;
static constexpr int kBlockCC = 128;           // types f, d: threads per block
static constexpr int kBlockCCMiller = kCCMillerBlock;   // ... of the Miller kernels (lock-step barrier)

// pbc_b200_prod_pairings_apply_v: the passes of the segmented product (prod_v.cuh) for one batch,
// built on the host from the offsets.  Pass s has count[s] runs of at most kProdVRun consecutive values
// of one output; the last pass has one run per output.
struct ProdPlan {
  size_t pairs = 0;            // Miller values of the batch
  size_t part = 0;             // elements of each of the two partial-product buffers (0: one pass)
  std::vector<size_t> count;   // runs per pass
  std::vector<uint64_t> runs;  // per pass, count + 1 input indices: run r is [runs[r], runs[r + 1])
};
// off: n_out + 1 increasing entries, rebased here to off[0] = 0
static ProdPlan prod_plan(const size_t* off, size_t n_out) {
  ProdPlan pl;
  pl.pairs = off[n_out] - off[0];
  std::vector<uint64_t> cur(n_out + 1), next(n_out + 1);
  for (size_t i = 0; i <= n_out; i++) cur[i] = off[i] - off[0];
  for (;;) {
    bool last = true;
    size_t runs = 0;
    next[0] = 0;
    for (size_t i = 0; i < n_out; i++) {
      for (uint64_t j = cur[i]; j < cur[i + 1]; j += kProdVRun, runs++) pl.runs.push_back(j);
      if (cur[i + 1] - cur[i] > (uint64_t)kProdVRun) last = false;
      next[i + 1] = runs;
    }
    pl.runs.push_back(cur[n_out]);
    pl.count.push_back(runs);
    if (last) break;
    if (pl.count.size() == 1) pl.part = runs;    // the largest partial batch: later passes only shrink
    cur.swap(next);
  }
  return pl;
}

// The three reference operations that reach the GPU (include/pbc_pairing.h:141-171, :54-89), and
// element_prod_pairing with a pair count per output (kProdV).
enum Mode { kSingle = 0, kProd = 1, kPP = 2, kProdV = 3 };
struct Job {
  Mode mode = kSingle;
  size_t k = 1;                // kProd: pairings per output
  const ProdPlan* plan = nullptr;   // kProdV: pairs and passes
  // kPP through a pairing_pp_t (pbc_b200_pp_init): what the handle keeps on the device -- the
  // line-coefficient table (types a, a1) and the wire bytes of the fixed first argument (all types).
  // nullptr: the table is built inside the call (pbc_b200_pp_pairings_apply).
  const void* pp_tab = nullptr;
  const uint8_t* pp_in1 = nullptr;
};

static size_t cc_table_bytes(const pbc_b200_pairing_s* p);
// type e: the fixed-argument table (pairing_e.cuh, e_pp_rows) and its flag word
static size_t e_table_bytes(const pbc_b200_pairing_s* p) { return (e_pp_rows(p->e.exp2) * kNA1 + 4) * 4; }

// kProdV: bytes of the value of one partial product of the segmented product, and of its validity
static size_t prodv_value_bytes(const pbc_b200_pairing_s* p) {
  if (p->type == 'a') return 2 * 64;                        // f [2]
  if (p->type == '1') return 2 * (size_t)kNA1 * 4;          // f [2]
  if (p->type == 'e') return (size_t)kNA1 * 4;              // v
  const size_t W = p->type == 'f' ? kF12Words : (p->type == 'g' ? kF10Words : 6 * (size_t)p->nlimbs);
  return W * 4;
}
static size_t prodv_valid_bytes(const pbc_b200_pairing_s* p) {
  if (p->type == 'a') return 64;                            // d
  if (p->type == '1' || p->type == 'e') return (size_t)kNA1 * 4;   // d, vd
  return 4;                                                 // flag word
}
static size_t prodv_elem_bytes(const pbc_b200_pairing_s* p) { return prodv_value_bytes(p) + prodv_valid_bytes(p); }
static size_t round16(size_t b) { return (b + 15) & ~(size_t)15; }
static size_t ws_core(const pbc_b200_pairing_s* p, const Job& job, size_t n_out);
// kProdV: the run tables and the two partial-product buffers follow everything the uniform product
// lays out for the same Miller values (ws_core), the type F slot kernels' scratch included
static size_t prodv_tail_off(const pbc_b200_pairing_s* p, const Job& job, size_t n_out) {
  return round16(ws_core(p, job, n_out));
}
// workspace bytes for n_out outputs of `job`
static size_t ws_bytes(const pbc_b200_pairing_s* p, const Job& job, size_t n_out) {
  if (job.mode != kProdV) return ws_core(p, job, n_out);
  return prodv_tail_off(p, job, n_out) + round16(job.plan->runs.size() * 8) + 2 * job.plan->part * prodv_elem_bytes(p);
}
static size_t ws_core(const pbc_b200_pairing_s* p, const Job& job, size_t n_out) {
  // Miller values of a product batch (kProd, kProdV)
  const size_t n_in = job.mode == kProdV ? job.plan->pairs : n_out * job.k;
  const bool prod = job.mode == kProd || job.mode == kProdV;
  if (p->type == '1') {
    // f [2], dprod, prefix per output; Miller inputs add f [2], d and the Montgomery P [2]
    const size_t fq = (size_t)kNA1 * 4;
    if (job.mode == kSingle) return n_out * (2 + 1 + 1 + 2) * fq;
    if (prod) return n_in * (2 + 1 + 2) * fq + n_out * (2 + 1 + 1) * fq;
    return n_out * (2 + 1 + 1) * fq + (p->a1_rows * kNA1 + 4) * 4;
  }
  if (p->type == 'e') {
    // f, dprod, prefix per output; Miller inputs add f, d, x(P), Q + R [5] and the save [5]; pp adds
    // the save [2] and (one-shot) the line table
    const size_t fq = (size_t)kNA1 * 4;
    if (job.mode == kSingle) return n_out * (3 + kQWords + kSWords) * fq;
    if (prod) return n_in * (3 + kQWords + kSWords) * fq + n_out * 3 * fq;
    return n_out * (3 + 2) * fq + e_table_bytes(p);
  }
  if (p->type == 'a') {
    const size_t fq = 64;
    // f [2], dprod, prefix, save [5] (V1, f1), qm [2] (Montgomery-form Q of the Miller kernels)
    if (job.mode == kSingle) return n_out * (2 + 1 + 1 + 5 + 2) * fq;
    // products: + vj [3] per pair (V of the pairs that share an accumulator, k_a_miller9_shared)
    if (job.mode == kProd)
      return n_out * job.k * (2 + 1 + 5 + 2 + 3) * fq + n_out * (2 + 1 + 1) * fq;
    if (job.mode == kProdV) return n_in * (2 + 1 + 5 + 2) * fq + n_out * (2 + 1 + 1) * fq;   // no shared accumulator
    return n_out * (2 + 1 + 1) * fq + (size_t)(3 * (p->a.exp2 + 1) * kNA + 4) * 4;
  }
  // types f, d: Miller values [W][n] words + one flag word each; products add the reduced arrays
  size_t W = p->type == 'f' ? kF12Words : (p->type == 'g' ? kF10Words : 6 * (size_t)p->nlimbs);
  const size_t n_mv = prod ? n_in : n_out;
  size_t bytes = n_mv * (W + 1) * 4;
  if (p->type == 'f') bytes += n_mv * (size_t)kFGWords * 4;   // Q, P of the slot-machine Miller kernel
  if (p->type == 'f') bytes += n_out * (size_t)kFStashWords * 4;   // parked F_q^12 values of the slot-machine final exponentiation
  if (job.mode == kPP) bytes += cc_table_bytes(p);             // line table of the fixed first argument
  if (prod) bytes += n_out * (W + 1) * 4;
  return bytes;
}
// G1's cofactor (fill_hash) is 1: every point of E(F_q) has order r
static bool g1_cofactor_one(const pbc_b200_pairing_s* p) {
  for (int i = 1; i < 12; i++)
    if (p->hash.cofac[i]) return false;
  return p->hash.cofac[0] == 1;
}
// lines of the Miller walk of types f, d, g: one tangent per loop position, one chord per non-zero digit
// strictly between the top digit and digit 0 (miller_cc_walk)
static size_t cc_table_rows_compute(const pbc_b200_pairing_s* p) {
  BigUInt r;
  if (p->dwide) for (int i = pbcb200_dw::kLimbs; i-- > 0;) r = r.shl(32) + BigUInt((uint64_t)p->dw_cc.r[i]);
  else for (int i = kNS; i-- > 0;) r = r.shl(32) + BigUInt((uint64_t)p->cc.r[i]);
  std::vector<int8_t> dg = miller_naf_digits(r, g1_cofactor_one(p));
  size_t rows = dg.size() - 1;
  for (size_t m = 1; m + 1 < dg.size(); m++) rows += dg[m] ? 1 : 0;
  return rows;
}
static size_t cc_table_rows(const pbc_b200_pairing_s* p) { return p->cc_rows; }
static size_t cc_table_bytes(const pbc_b200_pairing_s* p) { return (cc_table_rows(p) * 3 * (size_t)p->nlimbs + 4) * 4; }

static size_t in1_elems(const Job& job, size_t n_out) {
  return job.mode == kProd ? n_out * job.k : (job.mode == kPP ? 1 : n_out);
}
static size_t in2_elems(const Job& job, size_t n_out) {
  return job.mode == kProd ? n_out * job.k : n_out;
}

// ------------------------------------------------------------------------------------------
// constant derivation
// ------------------------------------------------------------------------------------------
static void fill_fp_consts(FpConsts* c, const BigUInt& q, int nlimbs) {
  memset(c, 0, sizeof *c);
  BigUInt R = BigUInt(1).shl(32 * (size_t)nlimbs);
  q.to_words(c->p, nlimbs);
  (R % q).to_words(c->one, nlimbs);
  ((R * R) % q).to_words(c->r2, nlimbs);
  (q - BigUInt(2)).to_words(c->pm2, nlimbs);
  c->np0 = neg_inv32(q.word(0));
  c->nlimbs = (uint32_t)nlimbs;
}

static bool get_big(const std::map<std::string, std::string>& tab, const char* key, BigUInt* out) {
  auto it = tab.find(key);
  if (it == tab.end()) { fail("missing param: `%s'", key); return false; }   // ecc/param.c:134-140
  if (!BigUInt::from_dec(it->second, out)) { fail("bad number for param `%s'", key); return false; }
  return true;
}
static bool get_int(const std::map<std::string, std::string>& tab, const char* key, int* out) {
  auto it = tab.find(key);
  if (it == tab.end()) { fail("missing param: `%s'", key); return false; }
  *out = atoi(it->second.c_str());
  return true;
}

static void fill_hash(pbc_b200_pairing_s* p, const BigUInt& q, const BigUInt& cofac);
static void to_mont(uint32_t* out, const BigUInt& x, const BigUInt& q, int n);

static int init_type_a(pbc_b200_pairing_s* p, const std::map<std::string, std::string>& tab) {
  BigUInt q, r, h;
  int exp2, exp1, sign1, sign0;
  if (!get_big(tab, "q", &q) || !get_big(tab, "r", &r) || !get_big(tab, "h", &h)) return 1;
  if (!get_int(tab, "exp2", &exp2) || !get_int(tab, "exp1", &exp1) ||
      !get_int(tab, "sign1", &sign1) || !get_int(tab, "sign0", &sign0)) return 1;
  // 64-byte coordinates on the wire (arith/montfp.c fixed_length_in_bytes = ceil(bits(q) / 8)): 505..512 bits
  if (q.bits() > 512 || q.bits() <= 504) return fail("type a: this build supports 505..512-bit q (64-byte coordinates; got %zu bits)", q.bits());
  if (r.bits() > 160 || r.bits() < 3) return fail("type a: this build supports group orders of up to 160 bits (got %zu)", r.bits());
  if (q.word(0) % 4 != 3) return fail("type a: q must be 3 mod 4");
  if (!((r * h) == (q + BigUInt(1)))) return fail("type a: r*h != q+1");
  if (h.bits() > 384) return fail("type a: cofactor too large");
  if (exp1 <= 0 || exp2 <= exp1 || exp2 > 512) return fail("type a: bad exp1/exp2");
  p->type = 'a';
  memset(&p->zr, 0, sizeof p->zr);
  r.to_words(p->zr.r, 5);
  p->zr.zlen = (uint32_t)((r.bits() + 7) / 8);
  p->zr_len = (int)p->zr.zlen;               // host copies, the Python mirror and the kernels' stride agree
  p->nlimbs = kNA;
  p->full = true;
  p->g1_len = p->g2_len = p->gt_len = 128;
  fill_fp_consts(&p->fp, q, kNA);
  memset(&p->a, 0, sizeof p->a);
  h.to_words(p->a.h, 12);
  p->a.hbits = (uint32_t)h.bits();
  p->a.exp2 = exp2; p->a.exp1 = exp1; p->a.sign1 = sign1;
  fill_hash(p, q, h);                      // G1 cofactor = h (ecc/a_param.c:1451)
  BigUInt R = BigUInt(1).shl(512);
  ((R * BigUInt(2)) % q).to_words(p->a.two, kNA);
  return 0;
}

// Type A1 (a1_init_pairing, ecc/a_param.c:2230-2273; parameters p, n, l with p = l n - 1)
static int init_type_a1(pbc_b200_pairing_s* p, const std::map<std::string, std::string>& tab) {
  BigUInt q, n;
  int l;
  if (!get_big(tab, "p", &q) || !get_big(tab, "n", &n) || !get_int(tab, "l", &l)) return 1;
  if (q.bits() > 32 * (size_t)kNA1 - 1) return fail("type a1: this build supports p below 2^%d (got %zu bits)", 32 * kNA1 - 1, q.bits());
  if (q.bits() < 64) return fail("type a1: p too small");
  if (q.word(0) % 4 != 3) return fail("type a1: p must be 3 mod 4");
  if (l <= 0 || (l & 1)) return fail("type a1: l must be positive and even");
  if (!((n * BigUInt((uint64_t)l)) == (q + BigUInt(1)))) return fail("type a1: l*n != p+1");
  if (n.bits() < 3) return fail("type a1: n too small");
  p->type = '1';
  memset(&p->zr, 0, sizeof p->zr);
  p->zr.zlen = (uint32_t)((n.bits() + 7) / 8);
  p->zr_len = (int)p->zr.zlen;
  p->nlimbs = kNA1;
  p->full = false;
  int wb = (int)((q.bits() + 7) / 8);
  p->g1_len = p->g2_len = p->gt_len = 2 * wb;
  fill_fp_consts(&p->fp, q, kNA1);
  A1Consts& c = p->a1;
  memset(&c, 0, sizeof c);
  n.to_words(c.n, kNA1);
  c.nbits = (uint32_t)n.bits();
  BigUInt L((uint64_t)l);
  L.to_words(c.l, 2);
  c.lbits = (uint32_t)L.bits();
  c.wb = (uint32_t)wb;
  to_mont(c.two, BigUInt(2), q, kNA1);
  // one tangent per loop step, one chord per set bit strictly between the top bit and bit 0
  size_t lines = n.bits() - 1;
  for (size_t m = 1; m + 1 < n.bits(); m++) lines += n.bit(m) ? 1 : 0;
  p->a1_rows = 3 * lines;
  A1GroupConsts& gc = p->a1g;
  memset(&gc, 0, sizeof gc);
  n.to_words(gc.n, kNA1);
  q.to_words(gc.q, kNA1);
  BigUInt se = (q + BigUInt(1)) / BigUInt(4);      // p = 3 mod 4: t^((p+1)/4) is a root of a square t
  se.to_words(gc.sqrt_exp, kNA1);
  gc.expbits = (uint32_t)se.bits();
  gc.zlen = p->zr.zlen;
  gc.count = (uint32_t)wb;
  {
    std::vector<int8_t> dg = miller_naf_digits(n, false);       // E(F_p) has order l n, l > 1
    if (dg.size() > 32 * (size_t)kMaxLimbs) return fail("type a1: n too large for the signed-digit table");
    memset(&p->a1naf, 0, sizeof p->a1naf);
    for (size_t i = 0; i < dg.size(); i++) {
      if (dg[i]) p->a1naf.nz[i >> 5] |= 1u << (i & 31);
      if (dg[i] < 0) p->a1naf.neg[i >> 5] |= 1u << (i & 31);
    }
    p->a1naf.len = (uint32_t)dg.size();
  }
  p->hash_ok = false;
  return 0;
}

// element_from_hash constants (ecc/curve.c:455-482, arith/field.c:643-668)
static void fill_hash(pbc_b200_pairing_s* p, const BigUInt& q, const BigUInt& cofac) {
  HashConsts& h = p->hash;
  memset(&h, 0, sizeof h);
  q.to_words(h.q, 16);
  h.count = (uint32_t)((q.bits() + 7) / 8);
  BigUInt one(1), e;
  if (q.word(0) % 4 == 3) { h.sqrt_mode = 1; e = (q + one) / BigUInt(4); }
  else if (q.word(0) % 8 == 5) { h.sqrt_mode = 2; e = (q - BigUInt(5)) / BigUInt(8); }
  else { h.sqrt_mode = 0; }
  e.to_words(h.exp, 16);
  h.expbits = (uint32_t)e.bits();
  BigUInt c = cofac.is_zero() ? one : cofac;
  c.to_words(h.cofac, 12);
  h.cofbits = (uint32_t)c.bits();
  p->hash_ok = h.sqrt_mode != 0 && c.bits() <= 384;
}

// x -> x * 2^(32 n) mod q, as n little-endian words
static void to_mont(uint32_t* out, const BigUInt& x, const BigUInt& q, int n) {
  ((x % q).shl(32 * (size_t)n) % q).to_words(out, n);
}

// element_from_hash / compressed points on G2 (group_cc.cuh, G2HashConstsT): square roots in K = F_q^k.
// k = 2 (type f): the norm method over F_q roots z^((q + 1)/4), so q = 3 mod 4; isq is i^2 of the basis
// in use.  k = 3, 5: Q = q^k = q mod 8 picks t^((Q + 1)/4), Atkin or Tonelli-Shanks; for the last,
// q^(k-1) + .. + 1 is odd, so Q - 1 = 2^s Qo has the s of q - 1 and c = z^Qo lies in F_q.
template <int NS>
static void fill_g2_hash(pbc_b200_pairing_s* p, G2HashConstsT<NS>& c, const BigUInt& q, int k, const BigUInt& isq) {
  memset(&c, 0, sizeof c);
  p->g2_hash_ok = false;
  const BigUInt one(1), two(2), qm1 = q - one;
  BigUInt leg = qm1 / two, e;
  leg.to_words(c.leg, 8);
  c.legbits = (uint32_t)leg.bits();
  if (k == 2) {
    if (q.word(0) % 4 != 3) return;
    e = (q + one) / BigUInt(4);
    to_mont(c.isq, isq, q, NS);
    to_mont(c.isq_inv, BigUInt::invmod(isq % q, q), q, NS);
    c.mode = 1;
  } else {
    BigUInt Q = q;
    for (int i = 1; i < k; i++) Q = Q * q;
    if (q.word(0) % 4 == 3) { c.mode = 1; e = (Q + one) / BigUInt(4); }
    else if (q.word(0) % 8 == 5) { c.mode = 2; e = (Q - BigUInt(5)) / BigUInt(8); }
    else {
      BigUInt Qo = Q - one, z(2);
      uint32_t s = 0;
      while (!Qo.bit(0)) { Qo = Qo / two; s++; }
      for (int tries = 0; !(BigUInt::powmod(z, leg, q) == qm1); tries++) {
        if (tries == 200) return;
        z = z + one;
      }
      c.mode = 3;
      c.ts_s = s;
      e = (Qo - one) / two;
      to_mont(c.ts_c, BigUInt::powmod(z, Qo % qm1, q), q, NS);
      p->derived["g2_sqrt_nonresidue"] = {z};
    }
  }
  if (e.bits() > 32 * 24) return;
  e.to_words(c.exp, 24);
  c.expbits = (uint32_t)e.bits();
  p->g2_hash_ok = true;
}
template <int NS>
static void fill_cc(CCConstsT<NS>* c, const BigUInt& A, const BigUInt& B, const BigUInt& r, const BigUInt& q) {
  memset(c, 0, sizeof *c);
  to_mont(c->A, A, q, NS);
  to_mont(c->B, B, q, NS);
  r.to_words(c->r, NS);
  c->rbits = (uint32_t)r.bits();
  c->a_is_zero = (A % q).is_zero() ? 1u : 0u;
}

// Internal basis for type F (tools/proto_f_nice_basis.py is the executable specification):
//   K = F_q[i]/(i^2+1) (q = 3 mod 4), sigma^2 = -beta, phi2(a + b s) = a + sigma b i,
//   xi' = a' + b' i small with phi2(xi)/xi' a sixth power, tau^6 xi' = phi2(xi).
// The sixth root: N = q^2 - 1 = S m with S = 2^e2 3^e3, 6 t = 1 + k m; w = c^t has w^6 = c (c^m)^k and the
// correction lives in the cyclic subgroup of order S generated by phi2(xi)^m (xi is neither a square
// nor a cube), searched exhaustively (S = 144 for f.param).
struct FBasis {
  bool ok = false;
  BigUInt sigma;
  uint32_t a = 0, b = 0;
  HostF2 tau, xi1;
};
static FBasis find_f_basis(const BigUInt& q, const BigUInt& beta, const HostF2& xi) {
  FBasis B;
  if (q.word(0) % 4 != 3) return B;
  BigUInt one(1), negbeta = beta.is_zero() ? beta : q - beta;
  B.sigma = BigUInt::powmod(negbeta, (q + one) / BigUInt(4), q);
  if (!(BigUInt::mulmod(B.sigma, B.sigma, q) == negbeta)) return B;
  HostF2Field K{q, q - one};                       // i^2 = -1
  B.xi1 = HostF2{xi.a, BigUInt::mulmod(B.sigma, xi.b, q)};
  BigUInt N = q * q - one, m = N, two(2), three(3), six(6);
  uint64_t S = 1;
  while ((m % two).is_zero()) { m = m / two; S *= 2; if (S > 4096) return B; }
  while ((m % three).is_zero()) { m = m / three; S *= 3; if (S > 4096) return B; }
  uint32_t k = 0;
  BigUInt t;
  for (k = 1; k <= 6; k++) {
    BigUInt num = one + m * BigUInt(k);
    if ((num % six).is_zero()) { t = num / six; break; }
  }
  if (k > 6) return B;
  HostF2 g = K.pow(B.xi1, m), g6 = K.pow(g, six);
  HostF2 unit;
  unit.a = one;
  BigUInt N6 = N / six;
  const uint32_t kMaxSmall = 6;
  for (uint32_t total = 1; total <= 2 * kMaxSmall; total++) {
    for (uint32_t b = 1; b <= total; b++) {
      uint32_t a = total - b;
      if (a > kMaxSmall || b > kMaxSmall) continue;
      HostF2 xs{BigUInt(a), BigUInt(b)};
      HostF2 c = K.mul(B.xi1, K.inv(xs));
      HostF2 chk = K.pow(c, N6);
      if (!(chk.a == one && chk.b.is_zero())) continue;
      HostF2 w = K.pow(c, t);
      HostF2 D = K.inv(K.pow(K.pow(c, m), BigUInt(k)));
      HostF2 h = unit, h6 = unit;
      for (uint64_t j = 0; j < S; j++) {
        if (h6.a == D.a && h6.b == D.b) {
          B.tau = K.mul(w, h);
          HostF2 back = K.mul(K.pow(B.tau, six), xs);
          if (back.a == B.xi1.a && back.b == B.xi1.b) {
            B.ok = true;
            B.a = a;
            B.b = b;
            return B;
          }
        }
        h = K.mul(h, g);
        h6 = K.mul(h6, g6);
      }
    }
  }
  return B;
}

// f_init_pairing (ecc/f_param.c:335-447)
static int init_type_f(pbc_b200_pairing_s* p, const std::map<std::string, std::string>& tab) {
  BigUInt q, r, b, beta, a0, a1;
  if (!get_big(tab, "q", &q) || !get_big(tab, "r", &r) || !get_big(tab, "b", &b) ||
      !get_big(tab, "beta", &beta) || !get_big(tab, "alpha0", &a0) || !get_big(tab, "alpha1", &a1)) return 1;
  // 20-byte coordinates on the wire (ceil(bits(q) / 8), arith/montfp.c:577): 153..159 bits
  if (q.bits() > 159 || q.bits() < 153) return fail("type f: this build supports 153..159-bit q (20-byte coordinates; got %zu bits)", q.bits());
  if (r.bits() > 160 || r.bits() < 3) return fail("type f: bad group order");
  BigUInt six(6);
  if (!((q % six) == BigUInt(1))) return fail("type f: q must be 1 mod 6");
  p->type = 'f';
  memset(&p->zr, 0, sizeof p->zr);
  r.to_words(p->zr.r, 5);
  p->zr.zlen = (uint32_t)((r.bits() + 7) / 8);
  p->zr_len = (int)p->zr.zlen;
  p->nlimbs = kNS;
  p->full = false;
  p->g1_len = 2 * kWS; p->g2_len = 4 * kWS; p->gt_len = 12 * kWS;
  fill_fp_consts(&p->fp, q, kNS);
  fill_cc(&p->cc, BigUInt(), b, r, q);
  fill_hash(p, q, BigUInt(1));             // no cofactor on G1 (ecc/f_param.c:372)
  HostF2Field Kref{q, beta % q};
  HostF2 alpha{a0 % q, a1 % q};
  HostF2 xi = Kref.neg(alpha);
  if (xi.a.is_zero() && xi.b.is_zero()) return fail("type f: alpha is zero");
  HostF2 xi_inv = Kref.inv(xi);
  HostF2 tb = Kref.scale(xi, b % q);
  BigUInt q2 = q * q, q6 = q2 * q2 * q2, q8 = q6 * q2, one(1);
  FConsts& c = p->f;
  memset(&c, 0, sizeof c);
  auto put2 = [&](uint32_t dst[2][kNS], const HostF2& v) { to_mont(dst[0], v.a, q, kNS); to_mont(dst[1], v.b, q, kNS); };
  auto rec2 = [&](const char* name, const HostF2& v) { p->derived[name] = {v.a, v.b}; };
  // reference-basis constants (ecc/f_param.c:422-444), recorded for the tests
  HostF2 x2 = Kref.pow(xi, (q2 - one) / six), x6 = Kref.pow(xi, (q6 - one) / six), x8 = Kref.pow(xi, (q8 - one) / six);
  to_mont(c.beta, Kref.beta, q, kNS);
  put2(c.xi_inv, xi_inv);
  put2(c.xpowq2, x2); put2(c.xpowq6, x6); put2(c.xpowq8, x8);
  rec2("xi", xi); rec2("xi_inv", xi_inv); rec2("twist_b", tb);
  rec2("xpowq2", x2); rec2("xpowq6", x6); rec2("xpowq8", x8);

  // the basis the kernels compute in
  FBasis B;
  if (!p->force_reference_basis) B = find_f_basis(q, Kref.beta, xi);
  HostF2Field K = B.ok ? HostF2Field{q, q - one} : Kref;
  HostF2 xi_use = xi, tb_use = tb, kx = xi_inv, ky = xi_inv, unit;
  unit.a = one;
  BigUInt sigma = one, sigma_inv = one;
  std::vector<HostF2> taup(6, unit), tauinv(6, unit);
  if (B.ok) {
    sigma = B.sigma;
    sigma_inv = BigUInt::invmod(sigma, q);
    auto phi2 = [&](const HostF2& v) { return HostF2{v.a, BigUInt::mulmod(sigma, v.b, q)}; };
    xi_use = HostF2{BigUInt(B.a), BigUInt(B.b)};
    tb_use = phi2(tb);
    for (int j = 1; j < 6; j++) taup[j] = K.mul(taup[j - 1], B.tau);
    for (int j = 1; j < 6; j++) tauinv[j] = K.inv(taup[j]);
    HostF2 xi1inv = K.inv(B.xi1);
    kx = K.mul(xi1inv, taup[4]);
    ky = K.mul(xi1inv, taup[3]);
    c.nice = 1;
    c.xi_a = B.a;
    c.xi_b = B.b;
    p->derived["basis_sigma"] = {sigma};
    p->derived["basis_xi_small"] = {BigUInt(B.a), BigUInt(B.b)};
    rec2("basis_tau", B.tau);
  }
  put2(c.xi, xi_use);
  put2(c.twist_b, tb_use);
  put2(c.kx, kx);
  put2(c.ky, ky);
  (q * q).to_words(c.qsq, 2 * kNS);
  for (int k = 0; k < 3; k++) (q * q * BigUInt((uint64_t)(k + 1))).to_words(c.qsqm[k], 2 * kNS);
  // the slot-machine kernels accumulate up to three F_q^2 products (each below 2 q^2) before one
  // reduction of a value below 2 q R: needs 6 q^2 < 2 q 2^160
  // and keep three Karatsuba cross sums (each below 4 q^2) on ten words: 12 q^2 < 2^320
  c.slots_ok = (c.nice && (q * BigUInt(3)).bits() <= 160 && (q * q * BigUInt(12)).bits() <= 320) ? 1u : 0u;
  to_mont(c.sigma, sigma, q, kNS);
  to_mont(c.sigma_inv, sigma_inv, q, kNS);
  fill_g2_hash(p, p->g2h, q, 2, B.ok ? q - one : Kref.beta);     // i^2 = -1 internal, beta reference
  for (int j = 1; j < 6; j++) { put2(c.tau[j - 1], taup[j]); put2(c.tau_inv[j - 1], tauinv[j]); }

  BigUInt num = (q2 * q2 + one) - q2, te, rem;
  BigUInt::divmod(num, r, &te, &rem);
  if (!rem.is_zero()) return fail("type f: r does not divide q^4 - q^2 + 1");
  if (te.bits() > 512) return fail("type f: final exponent too large");
  te.to_words(c.tateexp, 16);
  c.tatebits = (uint32_t)te.bits();
  p->derived["tateexp"] = {te};
  // Frobenius tables frob[k-1][i-1] = xi^(i (q^k - 1)/6), k = 1, 2, 3, in the basis in use
  BigUInt q3 = q2 * q;
  const BigUInt* qk[3] = {&q, &q2, &q3};
  for (int k = 0; k < 3; k++) {
    HostF2 g = K.pow(xi_use, (*qk[k] - one) / six), acc = g;
    std::vector<BigUInt> rec;
    for (int i = 0; i < 5; i++) {
      put2(c.frob[k][i], acc);
      rec.push_back(acc.a); rec.push_back(acc.b);
      acc = K.mul(acc, g);
    }
    p->derived[std::string("frob") + char('1' + k)] = rec;
  }
  // BN parameter: q = 36u^4 + 36u^3 + 24u^2 + 6u + 1 and r = 36u^4 + 36u^3 + 18u^2 + 6u + 1 for
  // some integer u of either sign (f_param gen).  |u| < 2^40 here; search |u| by bisection.
  {
    auto poly = [](const BigUInt& a, bool neg, uint32_t c2) {
      // 36a^4 +- 36a^3 + c2 a^2 +- 6a + 1 (all terms kept non-negative by ordering)
      BigUInt a2 = a * a, a3 = a2 * a, a4 = a2 * a2;
      BigUInt pos = a4 * BigUInt(36) + a2 * BigUInt(c2) + BigUInt(1);
      BigUInt odd = a3 * BigUInt(36) + a * BigUInt(6);
      return neg ? pos - odd : pos + odd;
    };
    for (int neg = 0; neg < 2 && !c.bn; neg++) {
      BigUInt lo(1), hi = BigUInt(1).shl(q.bits() / 4 + 2);
      while (lo < hi) {
        BigUInt mid = (lo + hi) / BigUInt(2);
        if (poly(mid, neg, 24) < q) lo = mid + BigUInt(1); else hi = mid;
      }
      if (poly(lo, neg, 24) == q && poly(lo, neg, 18) == r && lo.bits() <= 64) {
        c.bn = 1;
        c.u_neg = (uint32_t)neg;
        c.u_bits = (uint32_t)lo.bits();
        lo.to_words(c.u_abs, 2);
        p->derived["bn_u"] = {lo};
      }
    }
  }
  if (p->force_generic_final_exp) c.bn = 0;
  return 0;
}

// d_init_pairing (ecc/d_param.c:993-1095), k = 6.
// Two instances of the type D kernels.  153..159-bit q (20-byte coordinates): five limbs, engine.cu's own
// kernels.  160..255-bit q (22..32-byte coordinates): eight limbs, R = 2^256 (engine_d_wide.cu).  The
// upper end is where the eight-limb code stops being exact, the least of:
//   * mont_mul<8, false>, fp_add<8, false>, fp_halve (FULL = false, no carry word): a + q <= 2^256 for the
//     operands they see, all canonical (< q): q < 2^255;
//   * the lazy F_q^3 product (pairing_d.cuh, internal basis): fq_add_nr sums below 2q < 2^256
//     fit the limbs, every value handed to the reduction lies in (0, 4 q^2), and redc_wide takes t < 2 q R:
//     4 q^2 < 2 q 2^256, again q < 2^255;
//   * fq_from_wire: any 32-byte input is below R and mont_mul_ps(x, R^2 mod q) of it is below 2q: q < 2^255;
//   * the signed-digit table of r (CCNaf, 256 digits) and the eight-word scalars: r < 2^255.
// So q < 2^255 (at most 255 bits) and r of at most 255 bits; the largest bundled set, d224, has 224.
template <int NS>
static int fill_type_d(pbc_b200_pairing_s* p, DConstsT<NS>& c, const BigUInt& q, const BigUInt& r, const BigUInt& a,
                       const BigUInt& b, const BigUInt& nqr, const BigUInt& c0, const BigUInt& c1, const BigUInt& c2) {
  memset(&c, 0, sizeof c);
  BigUInt v = nqr % q, vinv = BigUInt::invmod(v, q), one(1);
  BigUInt v2 = BigUInt::mulmod(v, v, q);
  to_mont(c.nqr, v, q, NS);
  to_mont(c.nqrinv, vinv, q, NS);
  to_mont(c.nqrinv2, BigUInt::mulmod(vinv, vinv, q), q, NS);
  to_mont(c.twist_a, BigUInt::mulmod(a % q, v2, q), q, NS);
  to_mont(c.twist_b, BigUInt::mulmod(b % q, BigUInt::mulmod(v2, v, q), q), q, NS);
  to_mont(c.two, BigUInt(2), q, NS);
  (q * q).to_words(c.qsqm[0], 2 * NS);
  (q * q * BigUInt(2)).to_words(c.qsqm[1], 2 * NS);
  HostF3Field Kref{q, {c0 % q, c1 % q, c2 % q}};
  HostF3 x;
  x.c[1] = one;
  HostF3 x3 = Kref.mul(Kref.mul(x, x), x), x4 = Kref.mul(x3, x);
  HostF3 xq_ref = Kref.pow(x, q), xq2_ref = Kref.mul(xq_ref, xq_ref);
  // internal cubic w^3 + p w + 1 (tools/proto_d_basis.py): x = lam w - s
  HostF3Field K = Kref;
  if (!p->force_reference_basis && (q % BigUInt(3)) == BigUInt(2)) {
    BigUInt i3 = BigUInt::invmod(BigUInt(3), q), i27 = BigUInt::invmod(BigUInt(27), q);
    BigUInt C0 = c0 % q, C1 = c1 % q, C2 = c2 % q;
    BigUInt s0 = BigUInt::mulmod(C2, i3, q);
    BigUInt C2sq = BigUInt::mulmod(C2, C2, q);
    BigUInt P = BigUInt::submod(C1, BigUInt::mulmod(C2sq, i3, q), q);
    BigUInt R0 = BigUInt::addmod(BigUInt::submod(C0, BigUInt::mulmod(BigUInt::mulmod(C1, C2, q), i3, q), q),
                                 BigUInt::mulmod(BigUInt::mulmod(BigUInt(2), BigUInt::mulmod(C2sq, C2, q), q), i27, q), q);
    BigUInt lam = BigUInt::powmod(R0, (q * BigUInt(2) - one) / BigUInt(3), q);
    BigUInt lam2 = BigUInt::mulmod(lam, lam, q);
    if (!R0.is_zero() && BigUInt::mulmod(lam2, lam, q) == R0) {
      BigUInt lami = BigUInt::invmod(lam, q);
      BigUInt pc = BigUInt::mulmod(P, BigUInt::mulmod(lami, lami, q), q);
      c.nice = 1;
      to_mont(c.pcoef, pc, q, NS);
      to_mont(c.bs, s0, q, NS);
      to_mont(c.bs2, BigUInt::mulmod(s0, s0, q), q, NS);
      to_mont(c.b2s, BigUInt::addmod(s0, s0, q), q, NS);
      to_mont(c.blam, lam, q, NS);
      to_mont(c.blam2, lam2, q, NS);
      to_mont(c.blami, lami, q, NS);
      to_mont(c.blami2, BigUInt::mulmod(lami, lami, q), q, NS);
      K = HostF3Field{q, {one, pc, BigUInt()}};
      p->derived["basis_cubic"] = {s0, lam, pc};
    }
  }
  HostF3 xq = K.pow(x, q), xq2 = K.mul(xq, xq);
  for (int i = 0; i < 3; i++) {
    to_mont(c.xpwr3[i], x3.c[i], q, NS);
    to_mont(c.xpwr4[i], x4.c[i], q, NS);
    to_mont(c.xpowq[i], xq.c[i], q, NS);
    to_mont(c.xpowq2[i], xq2.c[i], q, NS);
  }
  BigUInt num = (q * q + one) - q, ph, rem;
  BigUInt::divmod(num, r, &ph, &rem);
  if (!rem.is_zero()) return fail("type d: r does not divide q^2 - q + 1");
  if (ph.bits() > 256) return fail("type d: final exponent too large");
  ph.to_words(c.phikonr, 8);
  p->derived["phikonr"] = {ph};
  p->derived["xpwr3"] = {x3.c[0], x3.c[1], x3.c[2]};
  p->derived["xpwr4"] = {x4.c[0], x4.c[1], x4.c[2]};
  p->derived["xpowq"] = {xq_ref.c[0], xq_ref.c[1], xq_ref.c[2]};      // reference-basis values (tests)
  p->derived["xpowq2"] = {xq2_ref.c[0], xq2_ref.c[1], xq2_ref.c[2]};
  p->derived["xpowq_in_use"] = {xq.c[0], xq.c[1], xq.c[2]};
  p->derived["nqrinv"] = {vinv};
  p->derived["nqrinv2"] = {BigUInt::mulmod(vinv, vinv, q)};
  c.phibits = (uint32_t)ph.bits();
  return 0;
}

static int init_type_d(pbc_b200_pairing_s* p, const std::map<std::string, std::string>& tab) {
  BigUInt q, r, a, b, nqr, c0, c1, c2;
  int k = 0;
  if (!get_big(tab, "q", &q) || !get_big(tab, "r", &r) || !get_big(tab, "a", &a) || !get_big(tab, "b", &b) ||
      !get_int(tab, "k", &k) || !get_big(tab, "nqr", &nqr) || !get_big(tab, "coeff0", &c0) ||
      !get_big(tab, "coeff1", &c1) || !get_big(tab, "coeff2", &c2)) return 1;
  if (k != 6) return fail("type d: only embedding degree 6 is on the GPU hot path (got k = %d)", k);
  const bool wide = q.bits() >= 160 && q.bits() <= 255;
  if (!wide && (q.bits() > 159 || q.bits() < 153))
    return fail("type d: this build supports 153..159-bit q (20-byte coordinates) and 160..255-bit q (got %zu bits)", q.bits());
  if (r.bits() > (wide ? 255u : 160u) || r.bits() < 3) return fail("type d: bad group order");
  BigUInt hco(1);
  auto ith = tab.find("h");
  if (ith != tab.end()) BigUInt::from_dec(ith->second, &hco);
  p->type = 'd';
  p->full = false;
  p->zr_len = (int)((r.bits() + 7) / 8);
  if (!wide) {
    memset(&p->zr, 0, sizeof p->zr);
    r.to_words(p->zr.r, 5);
    p->zr.zlen = (uint32_t)p->zr_len;
    p->nlimbs = kNS;
    p->g1_len = 2 * kWS; p->g2_len = 6 * kWS; p->gt_len = 6 * kWS;
    fill_fp_consts(&p->fp, q, kNS);
    fill_cc(&p->cc, a, b, r, q);
    fill_hash(p, q, hco);                  // G1 cofactor = h (ecc/d_param.c:1016)
    fill_g2_hash(p, p->g2h, q, 3, BigUInt());
    return fill_type_d<kNS>(p, p->d, q, r, a, b, nqr, c0, c1, c2);
  }
  const int NW = pbcb200_dw::kLimbs;
  const int wb = (int)((q.bits() + 7) / 8);
  p->dwide = true;
  memset(&p->dw_zr, 0, sizeof p->dw_zr);
  r.to_words(p->dw_zr.r, NW);
  p->dw_zr.zlen = (uint32_t)p->zr_len;
  p->nlimbs = NW;
  p->g1_len = 2 * wb; p->g2_len = 6 * wb; p->gt_len = 6 * wb;
  fill_fp_consts(&p->fp, q, NW);
  fill_cc(&p->dw_cc, a, b, r, q);
  fill_hash(p, q, hco);
  memset(&p->dw_x, 0, sizeof p->dw_x);
  p->dw_x.wb = (uint32_t)wb;
  if (q.word(0) % 8 == 1) {
    // Tonelli-Shanks (group_cc.cuh, fq_sqrt_ts): q - 1 = 2^s Q, exponent (Q - 1)/2, c = z^Q for the
    // least non-residue z.  Any root serves: the kernels normalise its sign as the reference does.
    BigUInt one(1), two(2), Q = q - one, z(2);
    uint32_t s = 0;
    while (!Q.bit(0)) { Q = Q / two; s++; }
    const BigUInt qm1 = q - one, half = qm1 / two;
    while (!(BigUInt::powmod(z, half, q) == qm1)) z = z + one;
    HashConsts& h = p->hash;
    BigUInt e = (Q - one) / two;
    memset(h.exp, 0, sizeof h.exp);
    e.to_words(h.exp, 16);
    h.expbits = (uint32_t)e.bits();
    h.sqrt_mode = 3;
    p->hash_ok = h.cofbits <= 384;
    p->dw_x.ts_s = s;
    to_mont(p->dw_x.ts_c, BigUInt::powmod(z, Q, q), q, NW);
    p->derived["sqrt_nonresidue"] = {z};
  }
  {
    std::vector<int8_t> dg = miller_naf_digits(r, g1_cofactor_one(p));
    memset(&p->dw_naf, 0, sizeof p->dw_naf);
    for (size_t i = 0; i < dg.size(); i++) {
      if (dg[i]) p->dw_naf.nz[i >> 5] |= 1u << (i & 31);
      if (dg[i] < 0) p->dw_naf.neg[i >> 5] |= 1u << (i & 31);
    }
    p->dw_naf.len = (uint32_t)dg.size();
  }
  fill_g2_hash(p, p->dw_g2h, q, 3, BigUInt());
  return fill_type_d<NW>(p, p->dw_d, q, r, a, b, nqr, c0, c1, c2);
}

// g_init_pairing (ecc/g_param.c:1248-1353), k = 10
static int init_type_g(pbc_b200_pairing_s* p, const std::map<std::string, std::string>& tab) {
  BigUInt q, r, a, b, nqr, co[5];
  int k = 0;
  if (!get_big(tab, "q", &q) || !get_big(tab, "r", &r) || !get_big(tab, "a", &a) || !get_big(tab, "b", &b) ||
      !get_int(tab, "k", &k) || !get_big(tab, "nqr", &nqr)) return 1;
  for (int i = 0; i < 5; i++)
    if (!get_big(tab, ("coeff" + std::to_string(i)).c_str(), &co[i])) return 1;
  if (k != 10) return fail("type g: embedding degree must be 10 (got k = %d)", k);
  if ((q.bits() + 7) / 8 != (size_t)kWG)
    return fail("type g: this build supports 145..152-bit q (19-byte coordinates; got %zu bits)", q.bits());
  if (r.bits() > 160 || r.bits() < 3) return fail("type g: bad group order");
  p->type = 'g';
  memset(&p->zr, 0, sizeof p->zr);
  r.to_words(p->zr.r, 5);
  p->zr.zlen = (uint32_t)((r.bits() + 7) / 8);
  p->zr_len = (int)p->zr.zlen;
  p->nlimbs = kNS;
  p->full = false;
  p->g1_len = 2 * kWG; p->g2_len = 10 * kWG; p->gt_len = 10 * kWG;
  fill_fp_consts(&p->fp, q, kNS);
  fill_cc(&p->cc, a, b, r, q);
  {
    BigUInt hco(1);
    auto ith = tab.find("h");
    if (ith != tab.end()) BigUInt::from_dec(ith->second, &hco);
    fill_hash(p, q, hco);                  // G1 cofactor = h (ecc/g_param.c:1267)
  }
  fill_g2_hash(p, p->g2h, q, 5, BigUInt());
  GConsts& c = p->g;
  memset(&c, 0, sizeof c);
  BigUInt v = nqr % q, vinv = BigUInt::invmod(v, q), one(1);
  BigUInt v2 = BigUInt::mulmod(v, v, q);
  to_mont(c.nqr, v, q, kNS);
  to_mont(c.nqrinv, vinv, q, kNS);
  to_mont(c.nqrinv2, BigUInt::mulmod(vinv, vinv, q), q, kNS);
  to_mont(c.twist_a, BigUInt::mulmod(a % q, v2, q), q, kNS);
  to_mont(c.twist_b, BigUInt::mulmod(b % q, BigUInt::mulmod(v2, v, q), q), q, kNS);
  to_mont(c.two, BigUInt(2), q, kNS);
  HostPolyField K{q, {co[0] % q, co[1] % q, co[2] % q, co[3] % q, co[4] % q}};
  HostPolyField::El x(5), xp;
  x[1] = one;
  xp = K.mul(K.mul(x, x), K.mul(K.mul(x, x), x));            // x^5
  std::vector<BigUInt> rec;
  for (int s = 0; s < 4; s++) {
    for (int i = 0; i < 5; i++) { to_mont(c.xpwr[s][i], xp[i], q, kNS); rec.push_back(xp[i]); }
    xp = K.mul(xp, x);
  }
  p->derived["xpwr"] = rec;
  HostPolyField::El xq = K.pow(x, q), acc = xq;
  rec.clear();
  for (int s = 0; s < 4; s++) {
    for (int i = 0; i < 5; i++) { to_mont(c.xpowq[s][i], acc[i], q, kNS); rec.push_back(acc[i]); }
    acc = K.mul(acc, xq);
  }
  p->derived["xpowq"] = rec;
  BigUInt q2 = q * q, q3 = q2 * q, q4 = q2 * q2;
  BigUInt num = ((q4 + q2 + one) - q3) - q, ph, rem;
  BigUInt::divmod(num, r, &ph, &rem);
  if (!rem.is_zero()) return fail("type g: r does not divide q^4 - q^3 + q^2 - q + 1");
  if (ph.bits() > 512) return fail("type g: final exponent too large");
  ph.to_words(c.phikonr, 16);
  c.phibits = (uint32_t)ph.bits();
  p->derived["phikonr"] = {ph};
  return 0;
}

// a square root of t mod q (Tonelli-Shanks; t a square), host side.  Returns 0 where no root is found
// (every loop is bounded: q comes from the caller's parameter text and need not be prime).
static BigUInt host_sqrt(const BigUInt& t, const BigUInt& q) {
  const BigUInt one(1), two(2), qm1 = q - one;
  BigUInt Q = qm1, z(2);
  uint32_t s = 0;
  while (!Q.bit(0)) { Q = Q / two; s++; }
  for (int tries = 0; !(BigUInt::powmod(z, qm1 / two, q) == qm1); tries++) {
    if (tries == 200) return BigUInt();
    z = z + one;
  }
  BigUInt c = BigUInt::powmod(z, Q, q), x = BigUInt::powmod(t, (Q + one) / two, q), b = BigUInt::powmod(t, Q, q);
  uint32_t m = s;
  while (!(b == one) && !b.is_zero()) {
    uint32_t i = 0;
    BigUInt b2 = b;
    while (!(b2 == one) && i < m) { b2 = BigUInt::mulmod(b2, b2, q); i++; }
    if (i == m) return BigUInt();
    BigUInt g = c;
    for (uint32_t j = 0; j + 1 < m - i; j++) g = BigUInt::mulmod(g, g, q);
    x = BigUInt::mulmod(x, g, q);
    c = BigUInt::mulmod(g, g, q);
    b = BigUInt::mulmod(b, c, q);
    m = i;
  }
  return b.is_zero() ? BigUInt() : x;
}

// k P == O on y^2 = x^3 + a x + b over F_q, P affine (host side, Jacobian: no inversions)
static bool host_mul_is_inf(const BigUInt& k, const BigUInt& px, const BigUInt& py, const BigUInt& a, const BigUInt& q) {
  BigUInt X, Y, Z;                                 // Z = 0: O
  auto mm = [&](const BigUInt& u, const BigUInt& v) { return BigUInt::mulmod(u, v, q); };
  auto ad = [&](const BigUInt& u, const BigUInt& v) { return BigUInt::addmod(u, v, q); };
  auto sb = [&](const BigUInt& u, const BigUInt& v) { return BigUInt::submod(u, v, q); };
  auto dbl = [&]() {
    if (Z.is_zero() || Y.is_zero()) { Z = BigUInt(); return; }
    BigUInt Z2 = mm(Z, Z), X2 = mm(X, X), Y2 = mm(Y, Y);
    BigUInt M = ad(ad(ad(X2, X2), X2), mm(a, mm(Z2, Z2)));
    BigUInt S = mm(X, Y2);
    S = ad(S, S); S = ad(S, S);
    BigUInt Y4 = mm(Y2, Y2), E8 = ad(Y4, Y4);
    E8 = ad(E8, E8); E8 = ad(E8, E8);
    BigUInt Xn = sb(sb(mm(M, M), S), S);
    Z = mm(Y, Z); Z = ad(Z, Z);
    Y = sb(mm(M, sb(S, Xn)), E8);
    X = Xn;
  };
  for (size_t i = k.bits(); i-- > 0;) {
    dbl();
    if (!k.bit(i)) continue;
    if (Z.is_zero()) { X = px; Y = py; Z = BigUInt(1); continue; }
    BigUInt Z2 = mm(Z, Z), H = sb(mm(px, Z2), X), R = sb(mm(py, mm(Z2, Z)), Y);
    if (H.is_zero()) {
      if (R.is_zero()) dbl(); else Z = BigUInt();
      continue;
    }
    BigUInt H2 = mm(H, H), H3 = mm(H2, H), U = mm(X, H2);
    BigUInt Xn = sb(sb(sb(mm(R, R), H3), U), U);
    Y = sb(mm(R, sb(U, Xn)), mm(Y, H3));
    Z = mm(Z, H);
    X = Xn;
  }
  return Z.is_zero();
}

// e_init_pairing (ecc/e_param.c:840-880), k = 1.  34-limb field (type a1's slot machine): q below 2^1087.
static int init_type_e(pbc_b200_pairing_s* p, const std::map<std::string, std::string>& tab) {
  BigUInt q, r, h, a, b;
  int exp2, exp1, sign1, sign0;
  if (!get_big(tab, "q", &q) || !get_big(tab, "r", &r) || !get_big(tab, "h", &h) || !get_big(tab, "a", &a) ||
      !get_big(tab, "b", &b)) return 1;
  if (!get_int(tab, "exp2", &exp2) || !get_int(tab, "exp1", &exp1) ||
      !get_int(tab, "sign1", &sign1) || !get_int(tab, "sign0", &sign0)) return 1;
  if (q.bits() > 32 * (size_t)kNA1 - 1) return fail("type e: this build supports q below 2^%d (got %zu bits)", 32 * kNA1 - 1, q.bits());
  if (q.bits() < 64) return fail("type e: q too small");
  if ((sign1 != 1 && sign1 != -1) || (sign0 != 1 && sign0 != -1)) return fail("type e: sign1 and sign0 must be 1 or -1");
  if (exp1 <= 0 || exp2 <= exp1 || exp2 >= 32 * kNA1 - 1) return fail("type e: bad exp1/exp2");
  const BigUInt one(1), p2 = one.shl((size_t)exp2), p1 = one.shl((size_t)exp1);
  BigUInt rr = sign1 > 0 ? p2 + p1 : p2 - p1;
  rr = sign0 > 0 ? rr + one : rr - one;
  if (!(rr == r)) return fail("type e: r != 2^exp2 + sign1 2^exp1 + sign0");
  BigUInt ph, rem;
  BigUInt::divmod(q - one, r, &ph, &rem);
  if (!rem.is_zero()) return fail("type e: r does not divide q - 1");
  a = a % q;
  b = b % q;
  p->type = 'e';
  memset(&p->zr, 0, sizeof p->zr);
  p->zr.zlen = (uint32_t)((r.bits() + 7) / 8);
  p->zr_len = (int)p->zr.zlen;
  p->nlimbs = kNA1;
  p->full = false;
  const int wb = (int)((q.bits() + 7) / 8);
  p->g1_len = p->g2_len = 2 * wb;
  p->gt_len = wb;
  fill_fp_consts(&p->fp, q, kNA1);
  memset(&p->a1, 0, sizeof p->a1);
  p->a1.wb = (uint32_t)wb;
  memset(&p->a1g, 0, sizeof p->a1g);
  r.to_words(p->a1g.n, kNA1);                      // scalars are reduced mod r (a1_zr_from_wire)
  p->a1g.zlen = p->zr.zlen;
  p->a1g.count = (uint32_t)wb;
  p->hash_ok = false;                              // element_from_hash / compressed points: not for type e
  // R: the first x = 1, 2, .. with x^3 + a x + b a non-zero square, y the smaller root, r R != O
  BigUInt Rx, Ry;
  bool found = false;
  for (uint64_t x = 1; !found && x < 1000; x++) {
    BigUInt X(x), t = BigUInt::addmod(BigUInt::mulmod(BigUInt::addmod(BigUInt::mulmod(X, X, q), a, q), X, q), b, q);
    if (t.is_zero() || !(BigUInt::powmod(t, (q - one) / BigUInt(2), q) == one)) continue;
    BigUInt y = host_sqrt(t, q);
    if (!(BigUInt::mulmod(y, y, q) == t)) continue;
    if (q - y < y) y = q - y;
    if (host_mul_is_inf(r, X, y, a, q)) continue;
    Rx = X;
    Ry = y;
    found = true;
  }
  if (!found) return fail("type e: found no point R outside E[r]");
  p->derived["R"] = {Rx, Ry};
  p->derived["phikonr"] = {ph};
  memset(p->e_pts, 0, sizeof p->e_pts);
  to_mont(p->e_pts + kEA * kNA1, a, q, kNA1);
  to_mont(p->e_pts + kEB * kNA1, b, q, kNA1);
  to_mont(p->e_pts + kERX * kNA1, Rx, q, kNA1);
  to_mont(p->e_pts + kERY * kNA1, Ry, q, kNA1);
  EConsts& c = p->e;
  memset(&c, 0, sizeof c);
  c.exp1 = (uint32_t)exp1;
  c.exp2 = (uint32_t)exp2;
  c.sign1 = sign1;
  c.sign0 = sign0;
  c.a_zero = a.is_zero() ? 1u : 0u;
  // final exponent (q - 1)/r as a left-to-right window of width 4: scanning down from the top bit,
  // each window starts at a set bit and ends at the lowest set bit of the 4 below it
  if (ph.bits() > sizeof c.dig) return fail("type e: final exponent too large");
  int i = (int)ph.bits() - 1;
  bool first = true;
  while (i >= 0) {
    if (!ph.bit((size_t)i)) { i--; continue; }
    int j = i - 3 < 0 ? 0 : i - 3;
    while (!ph.bit((size_t)j)) j++;
    uint32_t d = 0;
    for (int k = i; k >= j; k--) d = 2 * d + (ph.bit((size_t)k) ? 1u : 0u);
    c.dig[j] = (uint8_t)d;
    if (first) { c.dstart = (uint32_t)j; first = false; }
    i = j - 1;
  }
  return 0;
}

// ------------------------------------------------------------------------------------------
// device contexts
// ------------------------------------------------------------------------------------------
// opt in to `bytes` of dynamic shared memory per block AND ask for the largest shared-memory carve-out:
// the slot kernels are sized so that 2 or 3 blocks fill the 228 KB of an H100 SM (227 KB at most per
// block); with the default preference the driver may configure a smaller carve-out that holds fewer
// blocks than the kernel was designed for (the nine-slot type A kernel would run two blocks per SM
// instead of three)
template <class K>
static cudaError_t allow_smem(K kernel, size_t bytes) {
  cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
  if (e != cudaSuccess) return e;
  return cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout, (int)cudaSharedmemCarveoutMaxShared);
}

static constexpr size_t kSmemAMiller9 = (size_t)kA9Slots * 64 * kBlockMiller;
// type F on the shared-memory slot machine (pairing_f_slots.cuh) where the parameters allow it, else the
// round-1 kernels (local-memory frames)
static constexpr int kBlockFS = 128;
// threads per block of the slot-machine Miller kernel: 128 -> two blocks (8 warps) per SM
static constexpr int kBlockFSM = 128;
static constexpr size_t kSmemFMillerS = (size_t)kFSlots * kNS * 4 * kBlockFSM;
static constexpr size_t kSmemFFinalS = (size_t)kFFinalSlots * kNS * 4 * kBlockFS;
static constexpr size_t kSmemAFinal = (size_t)kAFSlots * 64 * kBlockFinal;
static constexpr size_t kSmemInv16 = (size_t)5 * 64 * kBlockInv;
static constexpr int kBlockProd = 128;
static constexpr size_t kSmemAProd = (size_t)kAPSlots * 64 * kBlockProd;
static constexpr size_t kSmemAPPInit = (size_t)kASlots * 64 * 32;
static constexpr size_t kSmemAPPApply = (size_t)kAPPSlots * 64 * kBlockMiller;

// type a1: 34-limb slots (136 bytes per thread and slot)
static constexpr int kBlockA1 = kA1MillerBlock;  // 13 slots * 136 B * 128 threads = 221 KB of shared memory
static constexpr int kBlockA1Small = 128;      // kernels with at most 9 slots
static constexpr size_t kSlotA1 = (size_t)kNA1 * 4;
static constexpr size_t kSmemA1Miller = (size_t)kA1MillerSlots * kSlotA1 * kBlockA1;
static constexpr size_t kSmemA1Final = (size_t)kA1FinalSlots * kSlotA1 * kBlockA1Small;
static constexpr size_t kSmemA1Prod = (size_t)kA1ProdSlots * kSlotA1 * kBlockA1Small;
static constexpr size_t kSmemA1PP = (size_t)kA1PPSlots * kSlotA1 * kBlockA1Small;
static constexpr size_t kSmemA1PPInit = (size_t)kASlots * kSlotA1 * 32;
static constexpr size_t kSmemInv34 = (size_t)5 * kSlotA1 * kBlockA1Small;
// group operations of type a1 run 64 threads per block: their own instantiation of the slot machine,
// so the code generated for the measured pairing kernels does not move when these change
static constexpr int kBlockA1G = 64;
static constexpr size_t kSmemA1G = (size_t)kGSlots * kSlotA1 * kBlockA1G;   // 11 slots: 93.5 KB, two blocks per SM
// type e: the same 34-limb slots; Miller kernel 13 slots * 136 B * 128 threads = 221 KB, one block per SM
static constexpr int kBlockE = 128;
static constexpr size_t kSmemEMiller = (size_t)kESlots * kSlotA1 * kBlockE;
static constexpr size_t kSmemEFinal = (size_t)kEFinalSlots * kSlotA1 * kBlockA1Small;
static constexpr size_t kSmemEProd = (size_t)kEProdSlots * kSlotA1 * kBlockA1Small;
static constexpr size_t kSmemEPP = (size_t)kEPPSlots * kSlotA1 * kBlockA1Small;
static constexpr size_t kSmemEPPInit = (size_t)kEPPInitSlots * kSlotA1 * 32;
static constexpr size_t kSmemEGroup = (size_t)kEGroupSlots * kSlotA1 * kBlockA1G;
// the segmented product of pbc_b200_prod_pairings_apply_v (prod_v.cuh): its policies per representation,
// at the block sizes and slot counts of the uniform product kernels
using ProdVA = ProdVF2<Ops<kNA, true, kBlockProd>, kNA>;
using ProdVA1 = ProdVF2<Ops<kNA1, false, kBlockA1Small>, kNA1>;
using ProdVEl = ProdVE<Ops<kNA1, false, kBlockA1Small>>;
using ProdVF = ProdVCC<F12ProdV>;
using ProdVD = ProdVCC<F6DProdV>;
using ProdVG = ProdVCC<F10ProdV>;
static_assert((int)ProdVA::kSlots == (int)kAPSlots && (int)ProdVA1::kSlots == kA1ProdSlots && (int)ProdVEl::kSlots == kEProdSlots,
              "the segmented product runs in the shared memory of the uniform one");

static int ctx_prepare(pbc_b200_pairing_s* p, int dev) {
  if ((int)p->ctx.size() <= dev) p->ctx.resize(dev + 1);
  DevCtx& c = p->ctx[dev];
  CUDA_OK(cudaSetDevice(dev));
  if (!c.ready) {
    c.dev = dev;
    CUDA_OK(cudaDeviceGetAttribute(&c.sms, cudaDevAttrMultiProcessorCount, dev));
    for (int s = 0; s < 2; s++) CUDA_OK(cudaStreamCreateWithFlags(&c.stream[s], cudaStreamNonBlocking));
    if (p->type == 'a') {
      CUDA_OK(allow_smem(k_a_miller9<kBlockMiller>, kSmemAMiller9));
      CUDA_OK(allow_smem(k_a_miller9_shared<kBlockMiller>, kSmemAMiller9));
      CUDA_OK(allow_smem(k_a_finalexp<kBlockFinal>, kSmemAFinal));
      CUDA_OK(allow_smem(k_batch_invert<kNA, true, kBlockInv>, kSmemInv16));
      CUDA_OK(allow_smem(k_fpmul_slots<kNA, true, 128, 0>, 2 * 64 * 128));
      CUDA_OK(allow_smem(k_a_prod<kBlockProd>, kSmemAProd));
      CUDA_OK(allow_smem(k_prod_v<ProdVA, kBlockProd>, kSmemAProd));
      CUDA_OK(allow_smem(k_a_pp_init<32>, kSmemAPPInit));
      CUDA_OK(allow_smem(k_a_pp_apply<kBlockMiller>, kSmemAPPApply));
      CUDA_OK(allow_smem(k_a_g1_mul<kBlockMiller>, (size_t)kGSlots * 64 * kBlockMiller));
      CUDA_OK(allow_smem(k_a_g1_finish<kBlockFinal>, (size_t)4 * 64 * kBlockFinal));
      CUDA_OK(allow_smem(k_a_gt_pow<kBlockMiller>, (size_t)7 * 64 * kBlockMiller));
      CUDA_OK(allow_smem(k_a_gt_mul<kBlockMiller>, (size_t)7 * 64 * kBlockMiller));
      CUDA_OK(allow_smem(k_a_g1_from_hash<kBlockMiller>, (size_t)kGSlots * 64 * kBlockMiller));
      CUDA_OK(allow_smem(k_a_g1_decompress<kBlockMiller>, (size_t)5 * 64 * kBlockMiller));
    }
    if (p->type == 'f') CUDA_OK(allow_smem(k_f_miller_s<kBlockFSM>, kSmemFMillerS));
    if (p->type == 'f') CUDA_OK(allow_smem(k_f_finalexp_s<kBlockFS>, kSmemFFinalS));
    if (p->type == '1') {
      CUDA_OK(allow_smem(k_a1_miller<kBlockA1>, kSmemA1Miller));
      CUDA_OK(allow_smem(k_a1_finalexp<kBlockA1Small>, kSmemA1Final));
      CUDA_OK(allow_smem(k_a1_prod<kBlockA1Small>, kSmemA1Prod));
      CUDA_OK(allow_smem(k_prod_v<ProdVA1, kBlockA1Small>, kSmemA1Prod));
      CUDA_OK(allow_smem(k_a1_pp_init<32>, kSmemA1PPInit));
      CUDA_OK(allow_smem(k_a1_pp_apply<kBlockA1Small>, kSmemA1PP));
      CUDA_OK(allow_smem(k_batch_invert<kNA1, false, kBlockA1Small>, kSmemInv34));
      CUDA_OK(allow_smem(k_a1_fp_op<kBlockA1Small>, (size_t)4 * kSlotA1 * kBlockA1Small));
      CUDA_OK(allow_smem(k_a1_g1_mul<kBlockA1G>, kSmemA1G));
      CUDA_OK(allow_smem(k_a1_g1_from_hash<kBlockA1G>, kSmemA1G));
      CUDA_OK(allow_smem(k_a1_g1_finish<kBlockA1G>, (size_t)4 * kSlotA1 * kBlockA1G));
      CUDA_OK(allow_smem(k_a1_gt_pow<kBlockA1G>, (size_t)7 * kSlotA1 * kBlockA1G));
      CUDA_OK(allow_smem(k_a1_gt_mul<kBlockA1G>, (size_t)7 * kSlotA1 * kBlockA1G));
      CUDA_OK(allow_smem(k_a1_g1_decompress<kBlockA1G>, (size_t)5 * kSlotA1 * kBlockA1G));
    }
    if (p->type == 'e') {
      CUDA_OK(allow_smem(k_e_miller<kBlockE>, kSmemEMiller));
      CUDA_OK(allow_smem(k_e_prod<kBlockA1Small>, kSmemEProd));
      CUDA_OK(allow_smem(k_prod_v<ProdVEl, kBlockA1Small>, kSmemEProd));
      CUDA_OK(allow_smem(k_e_pp_init<32>, kSmemEPPInit));
      CUDA_OK(allow_smem(k_e_pp_apply<kBlockA1Small>, kSmemEPP));
      CUDA_OK(allow_smem(k_e_finalexp<kBlockA1Small>, kSmemEFinal));
      CUDA_OK(allow_smem(k_batch_invert<kNA1, false, kBlockA1Small>, kSmemInv34));
      CUDA_OK(allow_smem(k_a1_fp_op<kBlockA1Small>, (size_t)4 * kSlotA1 * kBlockA1Small));
      CUDA_OK(allow_smem(k_e_g1_mul<kBlockA1G>, kSmemA1G));
      CUDA_OK(allow_smem(k_a1_g1_finish<kBlockA1G>, (size_t)4 * kSlotA1 * kBlockA1G));
      CUDA_OK(allow_smem(k_e_gt_pow<kBlockA1G>, kSmemEGroup));
      CUDA_OK(allow_smem(k_e_gt_mul<kBlockA1G>, kSmemEGroup));
    }
    c.ready = true;
  }
  // make this handle's constants resident on the device
  std::lock_guard<std::mutex> lk(g_const_mu);
  if (g_const_owner[dev] != p->id && p->dwide) {
    CUDA_OK(cudaDeviceSynchronize());
    pbcb200_dw::DWideConsts w = {&p->fp, &p->dw_cc, &p->dw_naf, &p->dw_d, &p->dw_zr, &p->hash, &p->dw_x, &p->dw_g2h,
                                 sizeof p->fp, sizeof p->dw_cc, sizeof p->dw_naf, sizeof p->dw_d, sizeof p->dw_zr,
                                 sizeof p->hash, sizeof p->dw_x, sizeof p->dw_g2h};
    const int e = pbcb200_dw::dw_upload(w);
    if (e == -2) return fail("type d: this build has no eight-limb instance (160..255-bit q)");
    if (e < 0) return fail("type d: the constants of the eight-limb instance do not match its layout");
    CUDA_OK((cudaError_t)e);
    CUDA_OK(cudaDeviceSynchronize());
    g_const_owner[dev] = p->id;
  }
  if (g_const_owner[dev] != p->id) {
    CUDA_OK(cudaDeviceSynchronize());
    CUDA_OK(cudaMemcpyToSymbol(c_fp, &p->fp, sizeof(FpConsts)));
    if (p->type == 'a') CUDA_OK(cudaMemcpyToSymbol(c_a, &p->a, sizeof(AConsts)));
    if (p->type == '1') CUDA_OK(cudaMemcpyToSymbol(c_a1, &p->a1, sizeof(A1Consts)));
    if (p->type == '1') CUDA_OK(cudaMemcpyToSymbol(c_a1g, &p->a1g, sizeof(A1GroupConsts)));
    if (p->type == 'e') {                  // type a1's wire width and scalar order, and the type e block
      CUDA_OK(cudaMemcpyToSymbol(c_a1, &p->a1, sizeof(A1Consts)));
      CUDA_OK(cudaMemcpyToSymbol(c_a1g, &p->a1g, sizeof(A1GroupConsts)));
      CUDA_OK(cudaMemcpyToSymbol(c_e, &p->e, sizeof(EConsts)));
      CUDA_OK(cudaMemcpyToSymbol(g_e_pts, p->e_pts, sizeof p->e_pts));
    }
    if (p->type == '1') CUDA_OK(cudaMemcpyToSymbol(c_a1naf, &p->a1naf, sizeof(A1Naf)));
    CUDA_OK(cudaMemcpyToSymbol(c_zr, &p->zr, sizeof(ZrConsts)));
    CUDA_OK(cudaMemcpyToSymbol(c_hash, &p->hash, sizeof(HashConsts)));
    if (p->type == 'f' || p->type == 'd' || p->type == 'g') CUDA_OK(cudaMemcpyToSymbol(c_cc, &p->cc, sizeof(CCConsts)));
    if (p->type == 'f' || p->type == 'd' || p->type == 'g') {
      // signed digits of the Miller walk (miller_naf_digits, host_naf.hpp); r is what fill_cc stored
      BigUInt r;
      for (int i = kNS; i-- > 0;) r = r.shl(32) + BigUInt((uint64_t)p->cc.r[i]);
      std::vector<int8_t> dg = miller_naf_digits(r, g1_cofactor_one(p));
      memset(&p->ccnaf, 0, sizeof p->ccnaf);
      for (size_t i = 0; i < dg.size() && i < 256; i++) {
        if (dg[i]) p->ccnaf.nz[i >> 5] |= 1u << (i & 31);
        if (dg[i] < 0) p->ccnaf.neg[i >> 5] |= 1u << (i & 31);
      }
      p->ccnaf.len = (uint32_t)dg.size();
      CUDA_OK(cudaMemcpyToSymbol(c_ccnaf, &p->ccnaf, sizeof(CCNaf)));
    }
    if (p->type == 'f') CUDA_OK(cudaMemcpyToSymbol(c_f, &p->f, sizeof(FConsts)));
    if (p->type == 'd') CUDA_OK(cudaMemcpyToSymbol(c_d, &p->d, sizeof(DConsts)));
    if (p->type == 'g') CUDA_OK(cudaMemcpyToSymbol(c_g, &p->g, sizeof(GConsts)));
    if (p->type == 'f' || p->type == 'd' || p->type == 'g') CUDA_OK(cudaMemcpyToSymbol(c_g2h, &p->g2h, sizeof(G2HashConsts)));
    CUDA_OK(cudaDeviceSynchronize());
    g_const_owner[dev] = p->id;
  }
  return 0;
}

static void ctx_release(DevCtx& c) {
  if (!c.ready) return;
  cudaSetDevice(c.dev);
  for (int s = 0; s < 2; s++) {
    if (c.stream[s]) cudaStreamSynchronize(c.stream[s]);
    cudaFree(c.d_in1[s]); cudaFree(c.d_in2[s]); cudaFree(c.d_out[s]); cudaFree(c.ws[s]);
    if (c.stream[s]) cudaStreamDestroy(c.stream[s]);
  }
  cudaFree(c.ws_dev);
  if (c.ws_ev) cudaEventDestroy(c.ws_ev);
  for (int s = 0; s < DevCtx::kPlanSlots; s++) {
    if (c.plan_ev[s]) { cudaEventSynchronize(c.plan_ev[s]); cudaEventDestroy(c.plan_ev[s]); }
    cudaFreeHost(c.plan_h[s]);
  }
  for (int i = 0; i < 4; i++) if (c.ev[i]) cudaEventDestroy(c.ev[i]);
  c = DevCtx();
}

// the shared device workspace is about to be used by work enqueued on `st` / has just been used
static int ws_acquire(DevCtx& c, cudaStream_t st) {
  if (!c.ws_ev) CUDA_OK(cudaEventCreateWithFlags(&c.ws_ev, cudaEventDisableTiming));
  if (c.ws_used) CUDA_OK(cudaStreamWaitEvent(st, c.ws_ev, 0));
  return 0;
}
static int ws_release(DevCtx& c, cudaStream_t st) {
  CUDA_OK(cudaEventRecord(c.ws_ev, st));
  c.ws_used = true;
  return 0;
}

// kProdV: copy the run tables of `job` to `dst` (device memory) on `st` through the next pinned slot
static int upload_plan(DevCtx& c, const Job& job, void* dst, cudaStream_t st) {
  const int s = c.plan_next;
  c.plan_next = (s + 1) % DevCtx::kPlanSlots;
  if (!c.plan_ev[s]) CUDA_OK(cudaEventCreateWithFlags(&c.plan_ev[s], cudaEventDisableTiming));
  else CUDA_OK(cudaEventSynchronize(c.plan_ev[s]));     // the slot's last upload has run
  const size_t bytes = job.plan->runs.size() * 8;
  if (c.plan_cap[s] < bytes) {
    cudaFreeHost(c.plan_h[s]);
    c.plan_h[s] = nullptr;
    c.plan_cap[s] = 0;
    CUDA_OK(cudaHostAlloc(&c.plan_h[s], bytes, cudaHostAllocPortable));
    c.plan_cap[s] = bytes;
  }
  memcpy(c.plan_h[s], job.plan->runs.data(), bytes);
  CUDA_OK(cudaMemcpyAsync(dst, c.plan_h[s], bytes, cudaMemcpyHostToDevice, st));
  CUDA_OK(cudaEventRecord(c.plan_ev[s], st));
  return 0;
}
static uint64_t* prodv_runs(const pbc_b200_pairing_s* p, const Job& job, void* ws, size_t n_out) {
  return (uint64_t*)((uint8_t*)ws + prodv_tail_off(p, job, n_out));
}

// multiprocessors of the current device, as ctx_prepare read them
static size_t cur_sms(const pbc_b200_pairing_s* p) {
  int dev = 0;
  cudaGetDevice(&dev);
  return (size_t)((int)p->ctx.size() > dev ? p->ctx[dev].sms : DevCtx().sms);
}
// threads of a batch inversion: per_sm independent chains per multiprocessor, never more than n
static size_t inv_threads(const pbc_b200_pairing_s* p, size_t n, size_t per_sm) {
  const size_t t = cur_sms(p) * per_sm;
  return n < t ? n : t;
}

// ------------------------------------------------------------------------------------------
// the final stage of types a, a1 and e on n Miller values in the limb-major Montgomery layout the
// Miller kernels write: batch inversion of dprod in place (prefix: scratch of its shape), then the
// final exponentiation into d_out (GT wire format).  The one launch path of these stages: the pairings
// (enqueue_pairings) and the test hook (pbc_b200_tower_op op 3) both come here.
// ------------------------------------------------------------------------------------------
static int enqueue_final(pbc_b200_pairing_s* p, void* f, void* dprod, void* prefix, uint8_t* d_out, size_t n,
                         cudaStream_t st, cudaEvent_t* ev) {
  if (p->type == 'a') {
    size_t T = inv_threads(p, n, 256);
    unsigned gi = (unsigned)((T + kBlockInv - 1) / kBlockInv);
    k_batch_invert<kNA, true, kBlockInv><<<gi, kBlockInv, kSmemInv16, st>>>(dprod, prefix, n, T);
    LAUNCHED();
    if (ev) cudaEventRecord(ev[2], st);
    unsigned gf = (unsigned)((n + kBlockFinal - 1) / kBlockFinal);
    k_a_finalexp<kBlockFinal><<<gf, kBlockFinal, kSmemAFinal, st>>>((const uint4*)f, (const uint4*)dprod, d_out, n);
    LAUNCHED();
    return 0;
  }
  if (p->type != '1' && p->type != 'e') return fail("pairing type '%c' has no batched final stage", p->type);
  size_t T = inv_threads(p, n, 128);
  unsigned gi = (unsigned)((T + kBlockA1Small - 1) / kBlockA1Small);
  k_batch_invert<kNA1, false, kBlockA1Small><<<gi, kBlockA1Small, kSmemInv34, st>>>(dprod, prefix, n, T);
  LAUNCHED();
  if (ev) cudaEventRecord(ev[2], st);
  unsigned gf = (unsigned)((n + kBlockA1Small - 1) / kBlockA1Small);
  if (p->type == '1') k_a1_finalexp<kBlockA1Small><<<gf, kBlockA1Small, kSmemA1Final, st>>>(f, dprod, d_out, n);
  else k_e_finalexp<kBlockA1Small><<<gf, kBlockA1Small, kSmemEFinal, st>>>(f, dprod, d_out, n);
  LAUNCHED();
  return 0;
}

// ------------------------------------------------------------------------------------------
// kProdV: the passes of the segmented product (prod_v.cuh) from the Miller values `mil` to the layout
// the final stage reads (`fin`, one element per output).  The run tables are in the workspace
// (upload_plan), the two partial-product buffers after them.
// ------------------------------------------------------------------------------------------
static int enqueue_prod_v(pbc_b200_pairing_s* p, const Job& job, ProdVBuf mil, ProdVBuf fin, void* ws, size_t n,
                          cudaStream_t st) {
  const ProdPlan& pl = *job.plan;
  const uint64_t* runs = prodv_runs(p, job, ws, n);
  const size_t eb = prodv_elem_bytes(p), cap = pl.part;
  // value rows first, validity after them (the Miller kernels' order)
  const size_t vb = prodv_value_bytes(p);
  uint8_t* base = (uint8_t*)runs + round16(pl.runs.size() * 8);
  ProdVBuf part[2];
  for (int b = 0; b < 2; b++) {
    uint8_t* v = base + b * cap * eb;
    part[b] = ProdVBuf{v, v + vb * cap, cap};
  }
  ProdVBuf in = mil;
  size_t off = 0;
  for (size_t s = 0; s < pl.count.size(); off += pl.count[s] + 1, s++) {
    const int last = s + 1 == pl.count.size();
    const ProdVBuf out = last ? fin : part[s & 1];
    const size_t R = pl.count[s];
    const uint64_t* r = runs + off;
    if (p->type == 'a')
      k_prod_v<ProdVA, kBlockProd><<<(unsigned)((R + kBlockProd - 1) / kBlockProd), kBlockProd, kSmemAProd, st>>>(in, out, r, R, last);
    else if (p->type == '1')
      k_prod_v<ProdVA1, kBlockA1Small><<<(unsigned)((R + kBlockA1Small - 1) / kBlockA1Small), kBlockA1Small, kSmemA1Prod, st>>>(in, out, r, R, last);
    else if (p->type == 'e')
      k_prod_v<ProdVEl, kBlockA1Small><<<(unsigned)((R + kBlockA1Small - 1) / kBlockA1Small), kBlockA1Small, kSmemEProd, st>>>(in, out, r, R, last);
    else if (p->dwide)
      pbcb200_dw::dw_prod_v((const uint32_t*)in.v, (const uint32_t*)in.d, in.n, (uint32_t*)out.v, (uint32_t*)out.d, out.n, r, R, st);
    else if (p->type == 'f')
      k_prod_v<ProdVF, kBlockCC><<<(unsigned)((R + kBlockCC - 1) / kBlockCC), kBlockCC, 0, st>>>(in, out, r, R, last);
    else if (p->type == 'g')
      k_prod_v<ProdVG, kBlockCC><<<(unsigned)((R + kBlockCC - 1) / kBlockCC), kBlockCC, 0, st>>>(in, out, r, R, last);
    else
      k_prod_v<ProdVD, kBlockCC><<<(unsigned)((R + kBlockCC - 1) / kBlockCC), kBlockCC, 0, st>>>(in, out, r, R, last);
    LAUNCHED();
    in = out;
  }
  return 0;
}

// ------------------------------------------------------------------------------------------
// enqueue one batch of n_out outputs of `job`, device buffers, on `st`.  ws: ws_bytes() bytes.
// ------------------------------------------------------------------------------------------
static int enqueue_pairings(pbc_b200_pairing_s* p, const Job& job, uint8_t* d_out, const uint8_t* d_in1,
                            const uint8_t* d_in2, size_t n, void* ws, cudaStream_t st,
                            cudaEvent_t* ev = nullptr) {
  if (n == 0) return 0;
#define STAGE(i) do { if (ev) cudaEventRecord(ev[i], st); } while (0)
  if (p->type == '1') {
    // limb-major arrays of 34-limb elements: E = 17 uint2 vectors per element
    const size_t E = kNA1 / 2;
    uint2 *f, *dprod, *prefix;
    const size_t wire = (size_t)p->g1_len;
    STAGE(0);
    if (job.mode == kSingle) {
      f = (uint2*)ws;                            // [2][E][n]
      dprod = f + 2 * E * n;                     // [E][n]
      prefix = dprod + E * n;                    // [E][n]
      uint2* pm = prefix + E * n;                // [2][E][n]
      unsigned gm = (unsigned)((n + kBlockA1 - 1) / kBlockA1);
      k_a1_miller<kBlockA1><<<gm, kBlockA1, kSmemA1Miller, st>>>(d_in1, d_in2, f, dprod, pm, n, wire);
      LAUNCHED();
    } else if (job.mode == kProd || job.mode == kProdV) {
      size_t m = job.mode == kProd ? n * job.k : job.plan->pairs;
      uint2* fi = (uint2*)ws;                    // [2][E][m]
      uint2* di = fi + 2 * E * m;                // [E][m]
      uint2* pm = di + E * m;                    // [2][E][m]
      f = pm + 2 * E * m;                        // [2][E][n]
      dprod = f + 2 * E * n;
      prefix = dprod + E * n;
      unsigned gm = (unsigned)((m + kBlockA1 - 1) / kBlockA1);
      k_a1_miller<kBlockA1><<<gm, kBlockA1, kSmemA1Miller, st>>>(d_in1, d_in2, fi, di, pm, m, wire);
      LAUNCHED();
      if (job.mode == kProdV) {
        if (enqueue_prod_v(p, job, ProdVBuf{fi, di, m}, ProdVBuf{f, dprod, n}, ws, n, st)) return 1;
      } else {
        unsigned gp = (unsigned)((n + kBlockA1Small - 1) / kBlockA1Small);
        k_a1_prod<kBlockA1Small><<<gp, kBlockA1Small, kSmemA1Prod, st>>>(fi, di, f, dprod, job.k, n, m);
        LAUNCHED();
      }
    } else {
      f = (uint2*)ws;
      dprod = f + 2 * E * n;
      prefix = dprod + E * n;
      uint32_t* tab = (uint32_t*)(prefix + E * n);
      if (job.pp_tab) tab = (uint32_t*)job.pp_tab;
      else { k_a1_pp_init<32><<<1, 32, kSmemA1PPInit, st>>>(d_in1, tab, p->a1_rows); LAUNCHED(); }
      unsigned gm = (unsigned)((n + kBlockA1Small - 1) / kBlockA1Small);
      k_a1_pp_apply<kBlockA1Small><<<gm, kBlockA1Small, kSmemA1PP, st>>>(tab, d_in2, f, dprod, n, p->a1_rows);
      LAUNCHED();
    }
    STAGE(1);
    if (enqueue_final(p, f, dprod, prefix, d_out, n, st, ev)) return 1;
    STAGE(3);
    CUDA_OK(cudaGetLastError());
    return 0;
  }
  if (p->type == 'e') {
    // limb-major arrays of 34-limb elements: E = 17 uint2 vectors per element
    const size_t E = kNA1 / 2;
    uint2 *f, *dprod, *prefix;
    const size_t wire = (size_t)p->g1_len;
    STAGE(0);
    if (job.mode != kPP) {
      const size_t m = job.mode == kProd ? n * job.k : (job.mode == kProdV ? job.plan->pairs : n);
      uint2* fi = (uint2*)ws;                    // [E][m]
      uint2* di = fi + E * m;                    // [E][m]
      uint2* px = di + E * m;                    // [E][m]
      uint2* qd = px + E * m;                    // [kQWords][E][m]
      uint2* sv = qd + kQWords * E * m;          // [kSWords][E][m]
      unsigned gm = (unsigned)((m + kBlockE - 1) / kBlockE);
      k_e_miller<kBlockE><<<gm, kBlockE, kSmemEMiller, st>>>(d_in1, d_in2, fi, di, px, qd, sv, m, wire);
      LAUNCHED();
      if (job.mode == kSingle) {
        f = fi;
        dprod = di;
        prefix = px;                             // x(P) is dead once the Miller kernel has finished
      } else {
        f = sv + kSWords * E * m;                // [E][n]
        dprod = f + E * n;
        prefix = dprod + E * n;
        if (job.mode == kProdV) {
          if (enqueue_prod_v(p, job, ProdVBuf{fi, di, m}, ProdVBuf{f, dprod, n}, ws, n, st)) return 1;
        } else {
          unsigned gp = (unsigned)((n + kBlockA1Small - 1) / kBlockA1Small);
          k_e_prod<kBlockA1Small><<<gp, kBlockA1Small, kSmemEProd, st>>>(fi, di, f, dprod, job.k, n, m);
          LAUNCHED();
        }
      }
    } else {
      f = (uint2*)ws;
      dprod = f + E * n;
      prefix = dprod + E * n;
      uint2* pv = prefix + E * n;                // [2][E][n]
      uint32_t* tab = (uint32_t*)(pv + 2 * E * n);
      if (job.pp_tab) tab = (uint32_t*)job.pp_tab;
      else { k_e_pp_init<32><<<1, 32, kSmemEPPInit, st>>>(d_in1, tab); LAUNCHED(); }
      unsigned gm = (unsigned)((n + kBlockA1Small - 1) / kBlockA1Small);
      k_e_pp_apply<kBlockA1Small><<<gm, kBlockA1Small, kSmemEPP, st>>>(tab, d_in2, f, dprod, pv, n);
      LAUNCHED();
    }
    STAGE(1);
    if (enqueue_final(p, f, dprod, prefix, d_out, n, st, ev)) return 1;
    STAGE(3);
    CUDA_OK(cudaGetLastError());
    return 0;
  }
  if (p->type == 'a') {
    uint4 *f, *dprod, *prefix;
    STAGE(0);
    if (job.mode == kSingle) {
      f = (uint4*)ws;                            // [2][4][n]
      dprod = f + 8 * n;                         // [4][n]
      prefix = dprod + 4 * n;                    // [4][n]
      uint4* save = prefix + 4 * n;              // [5][4][n]
      uint4* qm = save + 20 * n;                 // [2][4][n]
      unsigned gm = (unsigned)((n + kBlockMiller - 1) / kBlockMiller);
      k_a_miller9<kBlockMiller><<<gm, kBlockMiller, kSmemAMiller9, st>>>(d_in1, d_in2, f, dprod, save, qm, n);
      LAUNCHED();
    } else if (job.mode == kProd) {
      size_t m = n * job.k;
      uint4* fi = (uint4*)ws;                    // [2][4][m]
      uint4* di = fi + 8 * m;                    // [4][m]
      uint4* save = di + 4 * m;                  // [5][4][m]
      uint4* qm = save + 20 * m;                 // [2][4][m]
      uint4* vj = qm + 8 * m;                    // [3][4][m]
      f = vj + 12 * m;                           // [2][4][n]
      dprod = f + 8 * n;
      prefix = dprod + 4 * n;
      // pairs per thread sharing one accumulator: the largest divisor of k not above the handle's setting
      // that still leaves four waves of threads (sharing divides the thread count, and with too few
      // threads the GPU idles)
      size_t share = 1;
      const size_t wave = cur_sms(p) * 3 * kBlockMiller;
      for (size_t c = (size_t)p->prod_share; c > 1; c--)
        if (job.k % c == 0 && (m / c >= 4 * wave || p->prod_share_forced)) { share = c; break; }
      size_t kk = job.k, mm = m;                 // pairs per output / Miller values that reach k_a_prod
      if (share > 1) {
        mm = m / share;
        kk = job.k / share;
        unsigned gs = (unsigned)((mm + kBlockMiller - 1) / kBlockMiller);
        k_a_miller9_shared<kBlockMiller><<<gs, kBlockMiller, kSmemAMiller9, st>>>(d_in1, d_in2, fi, di, save, qm, vj, mm, share);
      } else {
        unsigned gm = (unsigned)((m + kBlockMiller - 1) / kBlockMiller);
        k_a_miller9<kBlockMiller><<<gm, kBlockMiller, kSmemAMiller9, st>>>(d_in1, d_in2, fi, di, save, qm, m);
      }
      LAUNCHED();
      unsigned gp = (unsigned)((n + kBlockProd - 1) / kBlockProd);
      k_a_prod<kBlockProd><<<gp, kBlockProd, kSmemAProd, st>>>(fi, di, f, dprod, kk, n, mm);
      LAUNCHED();
    } else if (job.mode == kProdV) {
      // one k_a_miller9 thread per pair (no shared accumulator), then the segmented product
      const size_t m = job.plan->pairs;
      uint4* fi = (uint4*)ws;                    // [2][4][m]
      uint4* di = fi + 8 * m;                    // [4][m]
      uint4* save = di + 4 * m;                  // [5][4][m]
      uint4* qm = save + 20 * m;                 // [2][4][m]
      f = qm + 8 * m;                            // [2][4][n]
      dprod = f + 8 * n;
      prefix = dprod + 4 * n;
      unsigned gm = (unsigned)((m + kBlockMiller - 1) / kBlockMiller);
      k_a_miller9<kBlockMiller><<<gm, kBlockMiller, kSmemAMiller9, st>>>(d_in1, d_in2, fi, di, save, qm, m);
      LAUNCHED();
      if (enqueue_prod_v(p, job, ProdVBuf{fi, di, m}, ProdVBuf{f, dprod, n}, ws, n, st)) return 1;
    } else {
      f = (uint4*)ws;
      dprod = f + 8 * n;
      prefix = dprod + 4 * n;
      uint32_t* tab = (uint32_t*)(prefix + 4 * n);
      if (job.pp_tab) tab = (uint32_t*)job.pp_tab;
      else { k_a_pp_init<32><<<1, 32, kSmemAPPInit, st>>>(d_in1, tab); LAUNCHED(); }
      unsigned gm = (unsigned)((n + kBlockMiller - 1) / kBlockMiller);
      k_a_pp_apply<kBlockMiller><<<gm, kBlockMiller, kSmemAPPApply, st>>>(tab, d_in2, f, dprod, n);
      LAUNCHED();
    }
    STAGE(1);
    if (enqueue_final(p, f, dprod, prefix, d_out, n, st, ev)) return 1;
    STAGE(3);
    CUDA_OK(cudaGetLastError());
    return 0;
  }
  if (p->type == 'f' || p->type == 'd' || p->type == 'g') {
    const bool isf = p->type == 'f', isg = p->type == 'g', wide = p->dwide;
    const size_t W = isf ? kF12Words : (isg ? kF10Words : 6 * (size_t)p->nlimbs);
    const bool prod = job.mode == kProd || job.mode == kProdV;
    size_t m = job.mode == kProd ? n * job.k : (job.mode == kProdV ? job.plan->pairs : n);
    uint32_t* mv = (uint32_t*)ws;                // [W][m]
    uint32_t* flag = mv + W * m;                 // [m]
    size_t stride1 = job.mode == kPP ? 0 : (size_t)p->g1_len;
    if (job.mode == kPP && job.pp_in1) d_in1 = job.pp_in1;
    unsigned gm = (unsigned)((m + kBlockCCMiller - 1) / kBlockCCMiller);
    STAGE(0);
    // fixed first argument: the line table, from the pp handle or built here at the end of the workspace
    const uint32_t* tab = nullptr;
    size_t rows = 0;
    if (job.mode == kPP) {
      rows = cc_table_rows(p);
      if (job.pp_tab) tab = (const uint32_t*)job.pp_tab;
      else {
        uint32_t* t = (uint32_t*)((uint8_t*)ws + ws_bytes(p, job, n) - cc_table_bytes(p));
        if (wide) pbcb200_dw::dw_pp_init(d_in1, t, rows, st);
        else if (isg) k_cc_pp_init<kWG><<<1, 32, 0, st>>>(d_in1, t, rows);
        else k_cc_pp_init<kWS><<<1, 32, 0, st>>>(d_in1, t, rows);
        LAUNCHED();
        tab = t;
      }
    }
    if (wide) pbcb200_dw::dw_miller(d_in1, d_in2, mv, flag, m, stride1, tab, rows, st);
    else if (isf && p->f.slots_ok) {
      uint32_t* gq = mv + (W + 1) * m + (prod ? (W + 1) * n : 0);   // after the Miller values and flags
      k_f_miller_s<kBlockFSM><<<(unsigned)((m + kBlockFSM - 1) / kBlockFSM), kBlockFSM, kSmemFMillerS, st>>>(d_in1, d_in2, mv, flag, gq, m, stride1, tab, rows);
    } else if (isf) k_f_miller<kBlockCCMiller><<<gm, kBlockCCMiller, 0, st>>>(d_in1, d_in2, mv, flag, m, stride1, tab, rows);
    else if (isg) k_g_miller<kBlockCCMiller><<<gm, kBlockCCMiller, 0, st>>>(d_in1, d_in2, mv, flag, m, stride1, tab, rows);
    else k_d_miller<kBlockCCMiller><<<gm, kBlockCCMiller, 0, st>>>(d_in1, d_in2, mv, flag, m, stride1, tab, rows);
    LAUNCHED();
    STAGE(1);
    if (job.mode == kProd) {
      uint32_t* mvo = flag + m;                  // [W][n]
      uint32_t* flago = mvo + W * n;
      unsigned gp = (unsigned)((n + kBlockCC - 1) / kBlockCC);
      if (wide) pbcb200_dw::dw_prod(mv, flag, mvo, flago, job.k, n, m, st);
      else if (isf) k_f_prod<kBlockCC><<<gp, kBlockCC, 0, st>>>(mv, flag, mvo, flago, job.k, n, m);
      else if (isg) k_g_prod<kBlockCC><<<gp, kBlockCC, 0, st>>>(mv, flag, mvo, flago, job.k, n, m);
      else k_d_prod<kBlockCC><<<gp, kBlockCC, 0, st>>>(mv, flag, mvo, flago, job.k, n, m);
      LAUNCHED();
      mv = mvo; flag = flago;
    } else if (job.mode == kProdV) {
      uint32_t* mvo = flag + m;                  // [W][n]
      uint32_t* flago = mvo + W * n;
      if (enqueue_prod_v(p, job, ProdVBuf{mv, flag, m}, ProdVBuf{mvo, flago, n}, ws, n, st)) return 1;
      mv = mvo; flag = flago;
    }
    STAGE(2);
    unsigned gf = (unsigned)((n + kBlockCC - 1) / kBlockCC);
    unsigned gfm = (unsigned)((n + kBlockCCMiller - 1) / kBlockCCMiller);
    if (wide) pbcb200_dw::dw_finalexp(mv, flag, d_out, n, st);
    else if (isf && p->f.slots_ok && p->f.bn) {
      uint32_t* stash = (uint32_t*)ws + (W + 1) * m + (prod ? (W + 1) * n : 0) + (size_t)kFGWords * m;
      k_f_finalexp_s<kBlockFS><<<(unsigned)((n + kBlockFS - 1) / kBlockFS), kBlockFS, kSmemFFinalS, st>>>(mv, flag, d_out, stash, n);
    } else if (isf) k_f_finalexp<kBlockCCMiller><<<gfm, kBlockCCMiller, 0, st>>>(mv, flag, d_out, n);
    else if (isg) k_g_finalexp<kBlockCCMiller><<<gfm, kBlockCCMiller, 0, st>>>(mv, flag, d_out, n);
    else k_d_finalexp<kBlockCC><<<gf, kBlockCC, 0, st>>>(mv, flag, d_out, n);
    LAUNCHED();
    STAGE(3);
    CUDA_OK(cudaGetLastError());
    return 0;
  }
  return fail("pairing type '%c' has no device path in this build", p->type);
}

// ------------------------------------------------------------------------------------------
// host-buffer pipeline for one device: outputs [0, n) of this device's slice, chunked over two
// streams (H2D of chunk k+1 overlaps the kernels of chunk k)
// ------------------------------------------------------------------------------------------
static int run_slice(pbc_b200_pairing_s* p, int dev, const Job& job, unsigned char* out,
                     const unsigned char* in1, const unsigned char* in2, size_t n) {
  std::lock_guard<std::mutex> dev_lock(g_dev_mu[dev & 63]);
  if (ctx_prepare(p, dev)) return 1;
  DevCtx& c = p->ctx[dev];
  size_t per_out = job.mode == kProd ? job.k : 1;
  size_t max_chunk = kChunk / per_out ? kChunk / per_out : 1;
  size_t chunk = n < max_chunk ? n : max_chunk;
  size_t b1 = in1_elems(job, chunk) * p->g1_len, b2 = in2_elems(job, chunk) * p->g2_len;
  size_t bo = chunk * p->gt_len, bw = ws_bytes(p, job, chunk);
  for (int s = 0; s < 2; s++) {
    if (c.cap_in1[s] < b1) { cudaFree(c.d_in1[s]); c.d_in1[s] = nullptr; c.cap_in1[s] = 0;
      CUDA_OK(cudaMalloc(&c.d_in1[s], b1)); c.cap_in1[s] = b1; }
    if (c.cap_in2[s] < b2) { cudaFree(c.d_in2[s]); c.d_in2[s] = nullptr; c.cap_in2[s] = 0;
      CUDA_OK(cudaMalloc(&c.d_in2[s], b2)); c.cap_in2[s] = b2; }
    if (c.cap_out[s] < bo) { cudaFree(c.d_out[s]); c.d_out[s] = nullptr; c.cap_out[s] = 0;
      CUDA_OK(cudaMalloc(&c.d_out[s], bo)); c.cap_out[s] = bo; }
    if (c.cap_ws[s] < bw) { cudaFree(c.ws[s]); c.ws[s] = nullptr; c.cap_ws[s] = 0;
      CUDA_OK(cudaMalloc(&c.ws[s], bw)); c.cap_ws[s] = bw; }
    if (n <= chunk) break;   // a single chunk only ever uses stream 0
  }
  int k = 0;
  for (size_t off = 0; off < n; off += chunk, k++) {
    size_t m = n - off < chunk ? n - off : chunk;
    int s = k & 1;
    cudaStream_t st = c.stream[s];
    size_t o1 = job.mode == kPP ? 0 : in1_elems(job, off) * p->g1_len;
    if (!job.pp_in1)
      CUDA_OK(cudaMemcpyAsync(c.d_in1[s], in1 + o1, in1_elems(job, m) * p->g1_len, cudaMemcpyHostToDevice, st));
    CUDA_OK(cudaMemcpyAsync(c.d_in2[s], in2 + in2_elems(job, off) * p->g2_len, in2_elems(job, m) * p->g2_len,
                            cudaMemcpyHostToDevice, st));
    if (enqueue_pairings(p, job, c.d_out[s], c.d_in1[s], c.d_in2[s], m, c.ws[s], st)) return 1;
    CUDA_OK(cudaMemcpyAsync(out + off * p->gt_len, c.d_out[s], m * p->gt_len, cudaMemcpyDeviceToHost, st));
  }
  CUDA_OK(cudaStreamSynchronize(c.stream[0]));
  CUDA_OK(cudaStreamSynchronize(c.stream[1]));
  return 0;
}

// contiguous slices of the outputs, one host thread per device, results written at the slice offset
static int run_host(pbc_b200_pairing_s* p, const Job& job, unsigned char* out, const unsigned char* in1,
                    const unsigned char* in2, size_t n) {
  if (!p || (!out && n) || (!in1 && n && !job.pp_in1) || (!in2 && n)) return fail("null argument");
  if (n == 0) return 0;
  std::lock_guard<std::mutex> lk(p->mu);
  int cur = 0;
  CUDA_OK(cudaGetDevice(&cur));
  if (p->ndev <= 1 || job.pp_in1) return run_slice(p, cur, job, out, in1, in2, n);   // a pp handle lives on one device
  int nd = p->ndev;
  if ((int)p->ctx.size() < nd) p->ctx.resize(nd);   // sized here: the per-device threads must not resize it
  std::vector<int> rc(nd, 0);
  std::vector<std::string> msg(nd);
  std::vector<std::thread> th;
  size_t per = (n + nd - 1) / nd;
  for (int d = 0; d < nd; d++) {
    size_t lo = (size_t)d * per, hi = lo + per < n ? lo + per : n;
    if (lo >= hi) continue;
    th.emplace_back([=, &rc, &msg]() {
      size_t o1 = job.mode == kPP ? 0 : in1_elems(job, lo) * p->g1_len;
      rc[d] = run_slice(p, d, job, out + lo * p->gt_len, in1 + o1, in2 + in2_elems(job, lo) * p->g2_len, hi - lo);
      if (rc[d]) msg[d] = g_err;
    });
  }
  for (auto& t : th) t.join();
  cudaSetDevice(cur);
  for (int d = 0; d < nd; d++) if (rc[d]) return fail("device %d: %s", d, msg[d].c_str());
  return 0;
}

// (re)allocate a device buffer to at least `need` bytes
static int grow(void** buf, size_t* cap, size_t need) {
  if (*cap >= need) return 0;
  cudaFree(*buf);
  *buf = nullptr;
  *cap = 0;
  CUDA_OK(cudaMalloc(buf, need));
  *cap = need;
  return 0;
}

// host-buffer pipeline of pbc_b200_prod_pairings_apply_v on one device: outputs [0, n) with pairs
// [off[0], off[n]) (in1, in2 point at pair off[0]).  Chunks hold whole outputs, packed while their pair
// count stays at or below kChunk; an output with more pairs is a chunk of its own.  Two streams, as
// run_slice.
static int run_slice_v(pbc_b200_pairing_s* p, int dev, unsigned char* out, const unsigned char* in1,
                       const unsigned char* in2, const size_t* off, size_t n) {
  std::lock_guard<std::mutex> dev_lock(g_dev_mu[dev & 63]);
  if (ctx_prepare(p, dev)) return 1;
  DevCtx& c = p->ctx[dev];
  std::vector<size_t> lo{0};                     // first output of every chunk, then n
  for (size_t i = 0; i < n;) {
    size_t j = i + 1;
    while (j < n && off[j + 1] - off[i] <= kChunk) j++;
    lo.push_back(j);
    i = j;
  }
  const size_t chunks = lo.size() - 1;
  std::vector<ProdPlan> plan(chunks);
  size_t b1 = 0, b2 = 0, bo = 0, bw = 0;
  for (size_t k = 0; k < chunks; k++) {
    plan[k] = prod_plan(off + lo[k], lo[k + 1] - lo[k]);
    Job job{kProdV, 1, &plan[k]};
    b1 = std::max(b1, plan[k].pairs * p->g1_len);
    b2 = std::max(b2, plan[k].pairs * p->g2_len);
    bo = std::max(bo, (lo[k + 1] - lo[k]) * p->gt_len);
    bw = std::max(bw, ws_bytes(p, job, lo[k + 1] - lo[k]));
  }
  for (int s = 0; s < 2 && s < (int)chunks; s++) {
    if (grow((void**)&c.d_in1[s], &c.cap_in1[s], b1) || grow((void**)&c.d_in2[s], &c.cap_in2[s], b2) ||
        grow((void**)&c.d_out[s], &c.cap_out[s], bo) || grow(&c.ws[s], &c.cap_ws[s], bw)) return 1;
  }
  for (size_t k = 0; k < chunks; k++) {
    const int s = k & 1;
    cudaStream_t st = c.stream[s];
    const size_t m = lo[k + 1] - lo[k], j0 = off[lo[k]] - off[0];
    const Job job{kProdV, 1, &plan[k]};
    CUDA_OK(cudaMemcpyAsync(c.d_in1[s], in1 + j0 * p->g1_len, plan[k].pairs * p->g1_len, cudaMemcpyHostToDevice, st));
    CUDA_OK(cudaMemcpyAsync(c.d_in2[s], in2 + j0 * p->g2_len, plan[k].pairs * p->g2_len, cudaMemcpyHostToDevice, st));
    if (upload_plan(c, job, prodv_runs(p, job, c.ws[s], m), st)) return 1;
    if (enqueue_pairings(p, job, c.d_out[s], c.d_in1[s], c.d_in2[s], m, c.ws[s], st)) return 1;
    CUDA_OK(cudaMemcpyAsync(out + lo[k] * p->gt_len, c.d_out[s], m * p->gt_len, cudaMemcpyDeviceToHost, st));
  }
  CUDA_OK(cudaStreamSynchronize(c.stream[0]));
  CUDA_OK(cudaStreamSynchronize(c.stream[1]));
  return 0;
}

// first output of device g's slice: the first i with off[i] world >= g off[n] (pairs, not outputs, are
// balanced); g = world gives n
static size_t slice_start_v(const size_t* off, size_t n, int g, int world) {
  const unsigned __int128 goal = (unsigned __int128)g * off[n];
  size_t a = 0, b = n;                           // off is increasing: binary search
  while (a < b) {
    const size_t mid = a + (b - a) / 2;
    if ((unsigned __int128)off[mid] * (unsigned)world >= goal) b = mid; else a = mid + 1;
  }
  return a;
}

// contiguous slices of the outputs, balanced by pairs, one host thread per device (as run_host)
static int run_host_v(pbc_b200_pairing_s* p, unsigned char* out, const unsigned char* in1, const unsigned char* in2,
                      const size_t* off, size_t n) {
  if (!out || !in1 || !in2) return fail("null argument");
  std::lock_guard<std::mutex> lk(p->mu);
  int cur = 0;
  CUDA_OK(cudaGetDevice(&cur));
  if (p->ndev <= 1) return run_slice_v(p, cur, out, in1, in2, off, n);
  const int nd = p->ndev;
  if ((int)p->ctx.size() < nd) p->ctx.resize(nd);
  std::vector<int> rc(nd, 0);
  std::vector<std::string> msg(nd);
  std::vector<std::thread> th;
  for (int d = 0; d < nd; d++) {
    const size_t lo = slice_start_v(off, n, d, nd), hi = slice_start_v(off, n, d + 1, nd);
    if (lo >= hi) continue;
    th.emplace_back([=, &rc, &msg]() {
      rc[d] = run_slice_v(p, d, out + lo * p->gt_len, in1 + off[lo] * p->g1_len, in2 + off[lo] * p->g2_len, off + lo, hi - lo);
      if (rc[d]) msg[d] = g_err;
    });
  }
  for (auto& t : th) t.join();
  cudaSetDevice(cur);
  for (int d = 0; d < nd; d++) if (rc[d]) return fail("device %d: %s", d, msg[d].c_str());
  return 0;
}

static int run_device(pbc_b200_pairing_s* p, const Job& job, void* d_out, const void* d_in1,
                      const void* d_in2, size_t n, void* stream) {
  if (!p) return fail("null argument");
  if (n == 0) return 0;
  std::lock_guard<std::mutex> lk(p->mu);
  int dev = 0;
  CUDA_OK(cudaGetDevice(&dev));
  if (ctx_prepare(p, dev)) return 1;
  DevCtx& c = p->ctx[dev];
  size_t need = ws_bytes(p, job, n);
  if (c.cap_dev < need) {
    CUDA_OK(cudaDeviceSynchronize());
    cudaFree(c.ws_dev);
    c.ws_dev = nullptr; c.cap_dev = 0;
    CUDA_OK(cudaMalloc(&c.ws_dev, need));
    c.cap_dev = need;
  }
  if (p->profile && !c.ev[0])
    for (int i = 0; i < 4; i++) CUDA_OK(cudaEventCreate(&c.ev[i]));
  if (ws_acquire(c, (cudaStream_t)stream)) return 1;
  if (job.mode == kProdV && upload_plan(c, job, prodv_runs(p, job, c.ws_dev, n), (cudaStream_t)stream)) return 1;
  if (enqueue_pairings(p, job, (uint8_t*)d_out, (const uint8_t*)d_in1, (const uint8_t*)d_in2, n,
                       c.ws_dev, (cudaStream_t)stream, p->profile ? c.ev : nullptr)) return 1;
  return ws_release(c, (cudaStream_t)stream);
}

// ------------------------------------------------------------------------------------------
// C ABI
// ------------------------------------------------------------------------------------------
extern "C" {

const char* pbc_b200_last_error(void) { return g_err; }
uint64_t pbc_b200_kernel_launches(void) { return g_launches.load(); }

int pbc_b200_pairing_init_set_buf(pbc_b200_pairing_t** out, const char* param, size_t len) {
  if (!out || !param) return fail("null argument");
  *out = nullptr;
  auto tab = parse_param_text(param, len);
  auto it = tab.find("type");
  if (it == tab.end()) return fail("unknown pairing type");           // ecc/param.c:171-174
  pbc_b200_pairing_s* p = new pbc_b200_pairing_s();
  p->id = g_next_id.fetch_add(1);
  int rc;
  // test switches (ignored by the reference parser, which only looks up the keys it needs)
  p->force_reference_basis = tab.count("b200_reference_basis") && tab["b200_reference_basis"] != "0";
  p->force_generic_final_exp = tab.count("b200_generic_final_exp") && tab["b200_generic_final_exp"] != "0";
  if (tab.count("b200_prod_share")) {
    int m = atoi(tab["b200_prod_share"].c_str());
    if (m >= 1 && m <= 64) { p->prod_share = m; p->prod_share_forced = true; }
  }
  if (it->second == "a") rc = init_type_a(p, tab);
  else if (it->second == "a1") rc = init_type_a1(p, tab);
  else if (it->second == "f") rc = init_type_f(p, tab);
  else if (it->second == "d") rc = init_type_d(p, tab);
  else if (it->second == "g") rc = init_type_g(p, tab);
  else if (it->second == "e") rc = init_type_e(p, tab);
  else rc = fail("pairing type `%s' is not on the GPU hot path (supported: a, a1, d with k = 6, e, f, g)", it->second.c_str());
  if (rc) { delete p; return 1; }
  if (p->type == 'f' || p->type == 'd' || p->type == 'g') p->cc_rows = cc_table_rows_compute(p);
  *out = p;
  return 0;
}

int pbc_b200_pairing_init_set_str(pbc_b200_pairing_t** out, const char* param) {
  if (!param) return fail("null argument");
  return pbc_b200_pairing_init_set_buf(out, param, strlen(param));
}

void pbc_b200_pairing_clear(pbc_b200_pairing_t* p) {
  if (!p) return;
  for (auto& c : p->ctx) ctx_release(c);
  {
    std::lock_guard<std::mutex> lk(g_const_mu);
    for (auto& kv : g_const_owner) if (kv.second == p->id) kv.second = 0;
  }
  delete p;
}

int pbc_b200_pairing_length_in_bytes_G1(const pbc_b200_pairing_t* p) { return p->g1_len; }
int pbc_b200_pairing_length_in_bytes_G2(const pbc_b200_pairing_t* p) { return p->g2_len; }
int pbc_b200_pairing_length_in_bytes_GT(const pbc_b200_pairing_t* p) { return p->gt_len; }
int pbc_b200_pairing_type(const pbc_b200_pairing_t* p) { return p->type; }

int pbc_b200_derived_constant(const pbc_b200_pairing_t* p, const char* name, unsigned char* out,
                              size_t width, size_t cap) {
  if (!p || !name || !out || !width) { fail("null argument"); return -1; }
  auto it = p->derived.find(name);
  if (it == p->derived.end()) { fail("no derived constant `%s'", name); return -1; }
  size_t need = it->second.size() * width;
  if (need > cap) { fail("buffer too small"); return -1; }
  size_t o = 0;
  for (const BigUInt& v : it->second) {
    if (v.bits() > 8 * width) { fail("constant wider than %zu bytes", width); return -1; }
    for (size_t i = 0; i < width; i++) {
      size_t byte = width - 1 - i;                       // big-endian
      out[o + i] = (unsigned char)(v.word(byte / 4) >> (8 * (byte % 4)));
    }
    o += width;
  }
  return (int)need;
}

int pbc_b200_set_devices(pbc_b200_pairing_t* p, int count) {
  int have = 0;
  CUDA_OK(cudaGetDeviceCount(&have));
  if (have <= 0) return fail("no CUDA device");
  if (count <= 0 || count > have) count = have;
  p->ndev = count;
  return 0;
}

int pbc_b200_pairings_apply(pbc_b200_pairing_t* p, unsigned char* out, const unsigned char* in1,
                            const unsigned char* in2, size_t n) {
  return run_host(p, Job{kSingle, 1}, out, in1, in2, n);
}

int pbc_b200_pairings_apply_device(pbc_b200_pairing_t* p, void* d_out, const void* d_in1,
                                   const void* d_in2, size_t n, void* stream) {
  return run_device(p, Job{kSingle, 1}, d_out, d_in1, d_in2, n, stream);
}

int pbc_b200_prod_pairings_apply(pbc_b200_pairing_t* p, unsigned char* out, const unsigned char* in1,
                                 const unsigned char* in2, size_t k, size_t n_out) {
  if (k == 0) return fail("prod_pairings: k must be positive");
  return run_host(p, Job{kProd, k}, out, in1, in2, n_out);
}

int pbc_b200_prod_pairings_apply_device(pbc_b200_pairing_t* p, void* d_out, const void* d_in1,
                                        const void* d_in2, size_t k, size_t n_out, void* stream) {
  if (k == 0) return fail("prod_pairings: k must be positive");
  return run_device(p, Job{kProd, k}, d_out, d_in1, d_in2, n_out, stream);
}

// offsets of pbc_b200_prod_pairings_apply_v: checked before any CUDA call
static int check_offsets(const pbc_b200_pairing_s* p, const size_t* off, size_t n_out) {
  if (!off) return fail("prod_pairings_v: offsets is NULL");
  if (off[0] != 0) return fail("prod_pairings_v: offsets[0] must be 0 (got %zu)", off[0]);
  for (size_t i = 1; i <= n_out; i++)
    if (off[i] <= off[i - 1])
      return fail("prod_pairings_v: offsets[%zu] = %zu is not above offsets[%zu] = %zu (every output needs at least one pair)",
                  i, off[i], i - 1, off[i - 1]);
  const size_t wide = (size_t)(p->g1_len > p->g2_len ? p->g1_len : p->g2_len);
  if (off[n_out] > SIZE_MAX / wide || n_out > SIZE_MAX / (size_t)p->gt_len)
    return fail("prod_pairings_v: %zu pairs / %zu outputs overflow the byte count", off[n_out], n_out);
  return 0;
}

int pbc_b200_prod_pairings_apply_v(pbc_b200_pairing_t* p, unsigned char* out, const unsigned char* in1,
                                   const unsigned char* in2, const size_t* offsets, size_t n_out) {
  if (!p) return fail("null argument");
  if (n_out == 0) return 0;
  if (check_offsets(p, offsets, n_out)) return 1;
  return run_host_v(p, out, in1, in2, offsets, n_out);
}

int pbc_b200_prod_pairings_apply_v_device(pbc_b200_pairing_t* p, void* d_out, const void* d_in1, const void* d_in2,
                                          const size_t* offsets, size_t n_out, void* stream) {
  if (!p) return fail("null argument");
  if (n_out == 0) return 0;
  if (check_offsets(p, offsets, n_out)) return 1;
  const ProdPlan plan = prod_plan(offsets, n_out);
  return run_device(p, Job{kProdV, 1, &plan}, d_out, d_in1, d_in2, n_out, stream);
}

int pbc_b200_pp_pairings_apply(pbc_b200_pairing_t* p, unsigned char* out, const unsigned char* in1,
                               const unsigned char* in2, size_t n) {
  return run_host(p, Job{kPP, 1}, out, in1, in2, n);
}

int pbc_b200_pp_pairings_apply_device(pbc_b200_pairing_t* p, void* d_out, const void* d_in1,
                                      const void* d_in2, size_t n, void* stream) {
  return run_device(p, Job{kPP, 1}, d_out, d_in1, d_in2, n, stream);
}

// ---- pairing_pp_t (include/pbc_pairing.h:54-89): preprocessing kept on the device ----
struct pbc_b200_pp_s {
  pbc_b200_pairing_s* p = nullptr;
  int dev = 0;
  uint8_t* d_in1 = nullptr;     // wire bytes of the fixed first argument
  void* d_tab = nullptr;        // line-coefficient table
};

int pbc_b200_pp_init(pbc_b200_pairing_t* p, pbc_b200_pp_t** out, const unsigned char* in1) {
  if (!p || !out || !in1) return fail("null argument");
  *out = nullptr;
  std::lock_guard<std::mutex> lk(p->mu);
  int dev = 0;
  CUDA_OK(cudaGetDevice(&dev));
  std::lock_guard<std::mutex> dev_lock(g_dev_mu[dev & 63]);
  if (ctx_prepare(p, dev)) return 1;
  DevCtx& c = p->ctx[dev];
  pbc_b200_pp_s* pp = new pbc_b200_pp_s();
  pp->p = p;
  pp->dev = dev;
  cudaStream_t st = c.stream[0];
  size_t tab_bytes = 0;
  if (p->type == 'a') tab_bytes = (size_t)(3 * (p->a.exp2 + 1) * kNA + 4) * 4;
  if (p->type == '1') tab_bytes = (p->a1_rows * kNA1 + 4) * 4;
  if (p->type == 'e') tab_bytes = e_table_bytes(p);
  const bool cc = p->type == 'f' || p->type == 'd' || p->type == 'g';
  if (cc) tab_bytes = cc_table_bytes(p);
  cudaError_t e = cudaMalloc(&pp->d_in1, (size_t)p->g1_len);
  if (e == cudaSuccess && tab_bytes) e = cudaMalloc(&pp->d_tab, tab_bytes);
  if (e == cudaSuccess) e = cudaMemcpyAsync(pp->d_in1, in1, (size_t)p->g1_len, cudaMemcpyHostToDevice, st);
  if (e == cudaSuccess && p->type == 'a') { k_a_pp_init<32><<<1, 32, kSmemAPPInit, st>>>(pp->d_in1, (uint32_t*)pp->d_tab); LAUNCHED(); }
  if (e == cudaSuccess && p->type == '1') { k_a1_pp_init<32><<<1, 32, kSmemA1PPInit, st>>>(pp->d_in1, (uint32_t*)pp->d_tab, p->a1_rows); LAUNCHED(); }
  if (e == cudaSuccess && p->type == 'e') { k_e_pp_init<32><<<1, 32, kSmemEPPInit, st>>>(pp->d_in1, (uint32_t*)pp->d_tab); LAUNCHED(); }
  if (e == cudaSuccess && cc) {
    if (p->dwide) pbcb200_dw::dw_pp_init(pp->d_in1, (uint32_t*)pp->d_tab, cc_table_rows(p), st);
    else if (p->type == 'g') k_cc_pp_init<kWG><<<1, 32, 0, st>>>(pp->d_in1, (uint32_t*)pp->d_tab, cc_table_rows(p));
    else k_cc_pp_init<kWS><<<1, 32, 0, st>>>(pp->d_in1, (uint32_t*)pp->d_tab, cc_table_rows(p));
    LAUNCHED();
  }
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  if (e == cudaSuccess) e = cudaGetLastError();
  if (e != cudaSuccess) {
    cudaFree(pp->d_in1); cudaFree(pp->d_tab);
    delete pp;
    return fail("pp_init: %s", cudaGetErrorString(e));
  }
  *out = pp;
  return 0;
}

static Job pp_job(const pbc_b200_pp_s* pp) {
  Job j;
  j.mode = kPP;
  j.pp_tab = pp->d_tab;
  j.pp_in1 = pp->d_in1;
  return j;
}

int pbc_b200_pp_apply(pbc_b200_pp_t* pp, unsigned char* out, const unsigned char* in2, size_t n) {
  if (!pp) return fail("null argument");
  int cur = 0;
  CUDA_OK(cudaGetDevice(&cur));
  if (cur != pp->dev) CUDA_OK(cudaSetDevice(pp->dev));
  int rc = run_host(pp->p, pp_job(pp), out, nullptr, in2, n);
  if (cur != pp->dev) cudaSetDevice(cur);
  return rc;
}

int pbc_b200_pp_apply_device(pbc_b200_pp_t* pp, void* d_out, const void* d_in2, size_t n, void* stream) {
  if (!pp) return fail("null argument");
  int cur = 0;
  CUDA_OK(cudaGetDevice(&cur));
  if (cur != pp->dev) return fail("pp_apply_device: the handle was initialised on device %d", pp->dev);
  return run_device(pp->p, pp_job(pp), d_out, pp->d_in1, d_in2, n, stream);
}

void pbc_b200_pp_clear(pbc_b200_pp_t* pp) {
  if (!pp) return;
  int cur = 0;
  cudaGetDevice(&cur);
  cudaSetDevice(pp->dev);
  cudaDeviceSynchronize();
  cudaFree(pp->d_in1);
  cudaFree(pp->d_tab);
  cudaSetDevice(cur);
  delete pp;
}

int pbc_b200_set_stage_profiling(pbc_b200_pairing_t* p, int on) {
  if (!p) return fail("null argument");
  p->profile = on != 0;
  return 0;
}

/* milliseconds of the three stages (main kernel, batch inversion, final exponentiation) of the
 * LAST pbc_b200_pairings_apply_device call on the current device; caller must have synchronised. */
int pbc_b200_stage_times(pbc_b200_pairing_t* p, float* ms3) {
  if (!p || !ms3) return fail("null argument");
  int dev = 0;
  CUDA_OK(cudaGetDevice(&dev));
  if ((int)p->ctx.size() <= dev || !p->ctx[dev].ev[0]) return fail("stage profiling was not enabled");
  for (int i = 0; i < 3; i++) CUDA_OK(cudaEventElapsedTime(&ms3[i], p->ctx[dev].ev[i], p->ctx[dev].ev[i + 1]));
  return 0;
}

void* pbc_b200_host_alloc(size_t bytes) {
  void* ptr = nullptr;
  if (cudaHostAlloc(&ptr, bytes, cudaHostAllocPortable) != cudaSuccess) {
    fail("cudaHostAlloc(%zu) failed", bytes);
    return nullptr;
  }
  return ptr;
}
void pbc_b200_host_free(void* ptr) { if (ptr) cudaFreeHost(ptr); }

// ---- roofline probes ----
// smem > 0 (type a, the slot multiplier of mode 1 only): launch with that much dynamic shared memory per block
static double bench_fpmul(pbc_b200_pairing_t* p, int mode, int blocks, int iters, int reps, size_t smem) {
  if (!p) { fail("null argument"); return -1; }
  if (p->type == '1' || p->type == 'e') { fail("bench_fpmul: not built for the 34-limb field (types a1, e)"); return -1; }
  if (p->dwide) { fail("bench_fpmul: not built for the eight-limb type d field"); return -1; }
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || ctx_prepare(p, dev)) return -1;
  const int threads = 128;
  if (smem < 2 * 64 * 128) smem = 2 * 64 * 128;
  size_t T = (size_t)blocks * threads;
  int N = p->nlimbs;
  uint32_t *in = nullptr, *out = nullptr;
  if (cudaMalloc(&in, T * 2 * N * 4) != cudaSuccess || cudaMalloc(&out, T * N * 4) != cudaSuccess) {
    fail("cudaMalloc failed"); return -1;
  }
  // any residues below p will do: fill with a small pattern (top limb zero)
  std::vector<uint32_t> h(T * 2 * N);
  uint32_t s = 12345;
  for (size_t i = 0; i < h.size(); i++) { s = s * 1664525u + 1013904223u; h[i] = s; }
  for (size_t t = 0; t < T; t++) { h[(2 * (N - 1)) * T + t] = 0; h[(2 * (N - 1) + 1) * T + t] = 0; }
  cudaMemcpy(in, h.data(), h.size() * 4, cudaMemcpyHostToDevice);
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0); cudaEventCreate(&e1);
  cudaStream_t st = p->ctx[dev].stream[0];
  auto launch = [&]() {
    if (p->type == 'a') {
      if (mode == 0) k_fpmul_chain<kNA, true, 0><<<blocks, threads, 0, st>>>(out, in, iters);
      else if (mode == 2) k_fpmul_chain<kNA, true, 1><<<blocks, threads, 0, st>>>(out, in, iters);
      else if (mode == 3) k_fpmul_chain<kNA, true, 2><<<blocks, threads, 0, st>>>(out, in, iters);
      else if (mode == 6) k_fpmul_slots<kNA, true, 128, 3><<<blocks, threads, 2 * 64 * 128, st>>>(out, in, iters);
      else if (mode == 7) k_fpmul_slots<kNA, true, 128, 4><<<blocks, threads, 2 * 64 * 128, st>>>(out, in, iters);
      else k_fpmul_slots<kNA, true, 128, 0><<<blocks, threads, smem, st>>>(out, in, iters);
    } else {
      k_fqmul_chain<<<blocks, threads, 0, st>>>(out, in, iters, mode == 3 ? 1 : 0);
    }
    LAUNCHED();
  };
  launch();
  cudaStreamSynchronize(st);
  cudaEventRecord(e0, st);
  for (int r = 0; r < reps; r++) launch();
  cudaEventRecord(e1, st);
  cudaEventSynchronize(e1);
  float ms = 0;
  cudaEventElapsedTime(&ms, e0, e1);
  cudaError_t err = cudaGetLastError();
  cudaEventDestroy(e0); cudaEventDestroy(e1);
  cudaFree(in); cudaFree(out);
  if (err != cudaSuccess) { fail("bench_fpmul: %s", cudaGetErrorString(err)); return -1; }
  return ms / reps;
}
double pbc_b200_bench_fpmul(pbc_b200_pairing_t* p, int mode, int blocks, int iters, int reps) {
  return bench_fpmul(p, mode, blocks, iters, reps, 0);
}
double pbc_b200_bench_fpmul_smem(pbc_b200_pairing_t* p, int smem_bytes, int iters, int reps, int* blocks_per_sm) {
  if (!p || !blocks_per_sm || smem_bytes < 0) { fail("null or negative argument"); return -1; }
  if (p->type != 'a') { fail("bench_fpmul_smem: type a only"); return -1; }
#ifdef PBC_HOST_SIM
  (void)iters; (void)reps;
  fail("bench_fpmul_smem: needs a GPU");
  return -1;
#else
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || ctx_prepare(p, dev)) return -1;
  const size_t smem = smem_bytes < 2 * 64 * 128 ? 2 * 64 * 128 : (size_t)smem_bytes;
  auto kern = k_fpmul_slots<kNA, true, 128, 0>;
  int occ = 0;
  cudaError_t e = allow_smem(kern, smem);
  if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, 128, smem);
  if (e != cudaSuccess) { fail("bench_fpmul_smem: %s", cudaGetErrorString(e)); return -1; }
  *blocks_per_sm = occ;
  if (occ < 1) { fail("bench_fpmul_smem: %d bytes per block do not fit an SM", smem_bytes); return -1; }
  // one full wave: every block resident for the whole run
  return bench_fpmul(p, 1, occ * (int)p->ctx[dev].sms, iters, reps, smem);
#endif
}

// the faster of the two IMAD.WIDE.U32 probes (common_kernels.cuh), each warmed up, then timed over reps launches
double pbc_b200_bench_imad(int blocks, int threads, int iters, int reps) {
  uint64_t* out = nullptr;
  if (cudaMalloc(&out, (size_t)blocks * threads * 8) != cudaSuccess) { fail("cudaMalloc failed"); return -1; }
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0); cudaEventCreate(&e1);
  float best = 0;
  for (int v = 0; v < 2; v++) {
    for (int r = -1; r < reps; r++) {            // r = -1: the warm-up launch
      if (r == 0) { cudaDeviceSynchronize(); cudaEventRecord(e0); }
      const uint32_t seed = (uint32_t)(8 + r);
      if (v == 0) k_imad_peak<<<blocks, threads>>>(out, seed, iters);
      else k_imad_peak_wide<<<blocks, threads>>>(out, seed, iters);
      LAUNCHED();
    }
    cudaEventRecord(e1);
    cudaEventSynchronize(e1);
    float ms = 0;
    cudaEventElapsedTime(&ms, e0, e1);
    if (v == 0 || ms < best) best = ms;
  }
  cudaError_t err = cudaGetLastError();
  cudaEventDestroy(e0); cudaEventDestroy(e1);
  cudaFree(out);
  if (err != cudaSuccess) { fail("bench_imad: %s", cudaGetErrorString(err)); return -1; }
  return best / reps;
}

}  // extern "C"


// ------------------------------------------------------------------------------------------
// group operations either side of the pairing (SURVEY 8f): batched element_pow_zn on G1 and GT
// ------------------------------------------------------------------------------------------
static int enqueue_group(pbc_b200_pairing_s* p, int which /*0 = G1, 1 = GT, 2 = G2*/, uint8_t* d_out, const uint8_t* d_in,
                         const uint8_t* d_k, size_t n, void* ws, cudaStream_t st) {
  if (n == 0) return 0;
  if (p->type == '1') {
    unsigned g = (unsigned)((n + kBlockA1G - 1) / kBlockA1G);
    if (which == 0 || which == 2) {                // type a1: G2 = G1 (ecc/a_param.c:2261)
      const size_t E = kNA1 / 2;
      uint2* xyz = (uint2*)ws;                  // [2][E][n]  (X, Y)
      uint2* zarr = xyz + 2 * E * n;            // [E][n]
      uint2* prefix = zarr + E * n;             // [E][n]
      k_a1_g1_mul<kBlockA1G><<<g, kBlockA1G, kSmemA1G, st>>>(d_in, d_k, xyz, zarr, n);
      LAUNCHED();
      size_t T = inv_threads(p, n, 128);
      unsigned gi = (unsigned)((T + kBlockA1Small - 1) / kBlockA1Small);
      k_batch_invert<kNA1, false, kBlockA1Small><<<gi, kBlockA1Small, kSmemInv34, st>>>(zarr, prefix, n, T);
      LAUNCHED();
      k_a1_g1_finish<kBlockA1G><<<g, kBlockA1G, (size_t)4 * kSlotA1 * kBlockA1G, st>>>(xyz, zarr, d_out, n);
      LAUNCHED();
    } else {
      k_a1_gt_pow<kBlockA1G><<<g, kBlockA1G, (size_t)7 * kSlotA1 * kBlockA1G, st>>>(d_in, d_k, d_out, n);
      LAUNCHED();
    }
    CUDA_OK(cudaGetLastError());
    return 0;
  }
  if (p->type == 'e') {
    unsigned g = (unsigned)((n + kBlockA1G - 1) / kBlockA1G);
    if (which == 0 || which == 2) {                // type e: G2 = G1 (ecc/e_param.c:874)
      const size_t E = kNA1 / 2;
      uint2* xyz = (uint2*)ws;                  // [2][E][n]  (X, Y)
      uint2* zarr = xyz + 2 * E * n;            // [E][n]
      uint2* prefix = zarr + E * n;             // [E][n]
      k_e_g1_mul<kBlockA1G><<<g, kBlockA1G, kSmemA1G, st>>>(d_in, d_k, xyz, zarr, n);
      LAUNCHED();
      size_t T = inv_threads(p, n, 128);
      unsigned gi = (unsigned)((T + kBlockA1Small - 1) / kBlockA1Small);
      k_batch_invert<kNA1, false, kBlockA1Small><<<gi, kBlockA1Small, kSmemInv34, st>>>(zarr, prefix, n, T);
      LAUNCHED();
      k_a1_g1_finish<kBlockA1G><<<g, kBlockA1G, (size_t)4 * kSlotA1 * kBlockA1G, st>>>(xyz, zarr, d_out, n);
      LAUNCHED();
    } else {
      k_e_gt_pow<kBlockA1G><<<g, kBlockA1G, kSmemEGroup, st>>>(d_in, d_k, d_out, n);
      LAUNCHED();
    }
    CUDA_OK(cudaGetLastError());
    return 0;
  }
  if (p->type == 'a') {
    if (which == 0 || which == 2) {                // type a: G2 = G1 (ecc/a_param.c:1461-1462)
      uint4* xyz = (uint4*)ws;                 // [2][4][n]  (X, Y)
      uint4* zarr = xyz + 8 * n;               // [4][n]
      uint4* prefix = zarr + 4 * n;            // [4][n]
      unsigned g = (unsigned)((n + kBlockMiller - 1) / kBlockMiller);
      k_a_g1_mul<kBlockMiller><<<g, kBlockMiller, (size_t)kGSlots * 64 * kBlockMiller, st>>>(d_in, d_k, xyz, zarr, n);
      LAUNCHED();
      size_t T = inv_threads(p, n, 256);
      unsigned gi = (unsigned)((T + kBlockInv - 1) / kBlockInv);
      k_batch_invert<kNA, true, kBlockInv><<<gi, kBlockInv, kSmemInv16, st>>>(zarr, prefix, n, T);
      LAUNCHED();
      unsigned gf = (unsigned)((n + kBlockFinal - 1) / kBlockFinal);
      k_a_g1_finish<kBlockFinal><<<gf, kBlockFinal, (size_t)4 * 64 * kBlockFinal, st>>>(xyz, zarr, d_out, n);
      LAUNCHED();
    } else {
      unsigned g = (unsigned)((n + kBlockMiller - 1) / kBlockMiller);
      k_a_gt_pow<kBlockMiller><<<g, kBlockMiller, (size_t)7 * 64 * kBlockMiller, st>>>(d_in, d_k, d_out, n);
      LAUNCHED();
    }
  } else {
    unsigned g = (unsigned)((n + kBlockCC - 1) / kBlockCC);
    const bool isg = p->type == 'g';
    if (p->dwide) pbcb200_dw::dw_group(which, d_out, d_in, d_k, n, st);
    else if (which == 0 && isg) k_cc_g1_mul<kBlockCC, kWG><<<g, kBlockCC, 0, st>>>(d_in, d_k, d_out, n);
    else if (which == 0) k_cc_g1_mul<kBlockCC, kWS><<<g, kBlockCC, 0, st>>>(d_in, d_k, d_out, n);
    else if (which == 2 && isg) k_cc_g2_mul<KF5, kBlockCC><<<g, kBlockCC, 0, st>>>(d_in, d_k, d_out, n);
    else if (which == 1 && isg) k_g_gt_pow<kBlockCC><<<g, kBlockCC, 0, st>>>(d_in, d_k, d_out, n);
    else if (which == 2 && p->type == 'f') k_cc_g2_mul<KF2, kBlockCC><<<g, kBlockCC, 0, st>>>(d_in, d_k, d_out, n);
    else if (which == 2) k_cc_g2_mul<KF3, kBlockCC><<<g, kBlockCC, 0, st>>>(d_in, d_k, d_out, n);
    else if (p->type == 'f') k_f_gt_pow<kBlockCC><<<g, kBlockCC, 0, st>>>(d_in, d_k, d_out, n);
    else k_d_gt_pow<kBlockCC><<<g, kBlockCC, 0, st>>>(d_in, d_k, d_out, n);
    LAUNCHED();
  }
  CUDA_OK(cudaGetLastError());
  return 0;
}

static int run_group(pbc_b200_pairing_s* p, int which, unsigned char* out, const unsigned char* in,
                     const unsigned char* k, size_t n, bool device, void* stream) {
  if (!p || (n && (!out || !in || !k))) return fail("null argument");
  if (n == 0) return 0;
  std::lock_guard<std::mutex> lk(p->mu);
  int dev = 0;
  CUDA_OK(cudaGetDevice(&dev));
  std::unique_lock<std::mutex> dev_lock(g_dev_mu[dev & 63], std::defer_lock);
  if (!device) dev_lock.lock();
  if (ctx_prepare(p, dev)) return 1;
  DevCtx& c = p->ctx[dev];
  size_t elen = which == 0 ? (size_t)p->g1_len : (which == 2 ? (size_t)p->g2_len : (size_t)p->gt_len);
  size_t wsb = p->type == 'a' && which != 1 ? n * 64 * (2 + 1 + 1) : 16;
  if ((p->type == '1' || p->type == 'e') && which != 1) wsb = n * kSlotA1 * (2 + 1 + 1);
  size_t stage = device ? 0 : n * (2 * elen + (size_t)p->zr_len);
  if (c.cap_dev < wsb + stage) {
    CUDA_OK(cudaDeviceSynchronize());
    cudaFree(c.ws_dev);
    c.ws_dev = nullptr; c.cap_dev = 0;
    CUDA_OK(cudaMalloc(&c.ws_dev, wsb + stage));
    c.cap_dev = wsb + stage;
  }
  if (device) {
    if (ws_acquire(c, (cudaStream_t)stream)) return 1;
    if (enqueue_group(p, which, (uint8_t*)out, (const uint8_t*)in, (const uint8_t*)k, n, c.ws_dev, (cudaStream_t)stream)) return 1;
    return ws_release(c, (cudaStream_t)stream);
  }
  uint8_t* d_in = (uint8_t*)c.ws_dev + wsb;
  uint8_t* d_out = d_in + n * elen;
  uint8_t* d_k = d_out + n * elen;
  cudaStream_t st = c.stream[0];
  if (ws_acquire(c, st)) return 1;           // a _device call of this handle may still be using the workspace
  CUDA_OK(cudaMemcpyAsync(d_in, in, n * elen, cudaMemcpyHostToDevice, st));
  CUDA_OK(cudaMemcpyAsync(d_k, k, n * (size_t)p->zr_len, cudaMemcpyHostToDevice, st));
  if (enqueue_group(p, which, d_out, d_in, d_k, n, c.ws_dev, st)) return 1;
  CUDA_OK(cudaMemcpyAsync(out, d_out, n * elen, cudaMemcpyDeviceToHost, st));
  CUDA_OK(cudaStreamSynchronize(st));
  return 0;
}

extern "C" {
int pbc_b200_pairing_length_in_bytes_Zr(const pbc_b200_pairing_t* p) { return p->zr_len; }
int pbc_b200_g1_pow_zn(pbc_b200_pairing_t* p, unsigned char* out, const unsigned char* in, const unsigned char* k,
                       size_t n) {
  return run_group(p, 0, out, in, k, n, false, nullptr);
}
int pbc_b200_gt_pow_zn(pbc_b200_pairing_t* p, unsigned char* out, const unsigned char* in, const unsigned char* k,
                       size_t n) {
  return run_group(p, 1, out, in, k, n, false, nullptr);
}
int pbc_b200_g2_pow_zn(pbc_b200_pairing_t* p, unsigned char* out, const unsigned char* in, const unsigned char* k,
                       size_t n) {
  return run_group(p, 2, out, in, k, n, false, nullptr);
}
int pbc_b200_g2_pow_zn_device(pbc_b200_pairing_t* p, void* d_out, const void* d_in, const void* d_k, size_t n,
                              void* stream) {
  return run_group(p, 2, (unsigned char*)d_out, (const unsigned char*)d_in, (const unsigned char*)d_k, n, true, stream);
}
int pbc_b200_g1_pow_zn_device(pbc_b200_pairing_t* p, void* d_out, const void* d_in, const void* d_k, size_t n,
                              void* stream) {
  return run_group(p, 0, (unsigned char*)d_out, (const unsigned char*)d_in, (const unsigned char*)d_k, n, true, stream);
}
int pbc_b200_gt_pow_zn_device(pbc_b200_pairing_t* p, void* d_out, const void* d_in, const void* d_k, size_t n,
                              void* stream) {
  return run_group(p, 1, (unsigned char*)d_out, (const unsigned char*)d_in, (const unsigned char*)d_k, n, true, stream);
}
}


// types f, d, g: G2 is the twist, with kernels of its own; types a and a1: G2 = G1
static bool g2_is_twist(const pbc_b200_pairing_s* p) { return p->type == 'f' || p->type == 'd' || p->type == 'g'; }

// element_from_hash on G1 or G2 (include/pbc_field.h:202-212 -> ecc/curve.c:455-482), batched
static int run_from_hash(pbc_b200_pairing_s* p, unsigned char* out, const unsigned char* data, size_t len, size_t n,
                         bool device, void* stream, bool g2 = false) {
  if (!p || (n && (!out || !data))) return fail("null argument");
  if (p->type == 'e') return fail("element_from_hash: not available for type e (q = 1 mod 16 needs a 34-limb Tonelli-Shanks)");
  const bool twist = g2 && g2_is_twist(p);
  if (twist && !p->g2_hash_ok) return fail("element_from_hash on G2: needs square roots in the twist's field (type f: q = 3 mod 4)");
  if (!twist && p->type != '1' && !p->hash_ok) return fail("element_from_hash: needs q = 3 mod 4 or q = 5 mod 8 (or type d with 160..255-bit q) and a cofactor below 2^384");
  if (len == 0 || len > (1u << 20)) return fail("element_from_hash: hash length must be 1..2^20 bytes");
  if (n == 0) return 0;
  std::lock_guard<std::mutex> lk(p->mu);
  int dev = 0;
  CUDA_OK(cudaGetDevice(&dev));
  std::unique_lock<std::mutex> dev_lock(g_dev_mu[dev & 63], std::defer_lock);
  if (!device) dev_lock.lock();
  if (ctx_prepare(p, dev)) return 1;
  DevCtx& c = p->ctx[dev];
  size_t elen = twist ? (size_t)p->g2_len : (size_t)p->g1_len;
  size_t wsb = p->type == 'a' ? n * 64 * (2 + 1 + 1) : 16;
  if (p->type == '1') wsb = n * kSlotA1 * (2 + 1 + 1);
  size_t stage = device ? 0 : n * (elen + len);
  if (c.cap_dev < wsb + stage) {
    CUDA_OK(cudaDeviceSynchronize());
    cudaFree(c.ws_dev);
    c.ws_dev = nullptr; c.cap_dev = 0;
    CUDA_OK(cudaMalloc(&c.ws_dev, wsb + stage));
    c.cap_dev = wsb + stage;
  }
  cudaStream_t st = device ? (cudaStream_t)stream : c.stream[0];
  if (ws_acquire(c, st)) return 1;
  uint8_t* d_out = device ? (uint8_t*)out : (uint8_t*)c.ws_dev + wsb;
  const uint8_t* d_data = device ? (const uint8_t*)data : d_out + n * elen;
  if (!device) CUDA_OK(cudaMemcpyAsync((void*)d_data, data, n * len, cudaMemcpyHostToDevice, st));
  if (p->type == '1') {
    const size_t E = kNA1 / 2;
    uint2* xyz = (uint2*)c.ws_dev;
    uint2* zarr = xyz + 2 * E * n;
    uint2* prefix = zarr + E * n;
    unsigned g = (unsigned)((n + kBlockA1G - 1) / kBlockA1G);
    k_a1_g1_from_hash<kBlockA1G><<<g, kBlockA1G, kSmemA1G, st>>>(d_data, (int)len, xyz, zarr, n);
    LAUNCHED();
    size_t T = inv_threads(p, n, 128);
    unsigned gi = (unsigned)((T + kBlockA1Small - 1) / kBlockA1Small);
    k_batch_invert<kNA1, false, kBlockA1Small><<<gi, kBlockA1Small, kSmemInv34, st>>>(zarr, prefix, n, T);
    LAUNCHED();
    k_a1_g1_finish<kBlockA1G><<<g, kBlockA1G, (size_t)4 * kSlotA1 * kBlockA1G, st>>>(xyz, zarr, d_out, n);
    LAUNCHED();
  } else if (p->type == 'a') {
    uint4* xyz = (uint4*)c.ws_dev;
    uint4* zarr = xyz + 8 * n;
    uint4* prefix = zarr + 4 * n;
    unsigned g = (unsigned)((n + kBlockMiller - 1) / kBlockMiller);
    k_a_g1_from_hash<kBlockMiller><<<g, kBlockMiller, (size_t)kGSlots * 64 * kBlockMiller, st>>>(d_data, (int)len, xyz, zarr, n);
    LAUNCHED();
    size_t T = inv_threads(p, n, 256);
    unsigned gi = (unsigned)((T + kBlockInv - 1) / kBlockInv);
    k_batch_invert<kNA, true, kBlockInv><<<gi, kBlockInv, kSmemInv16, st>>>(zarr, prefix, n, T);
    LAUNCHED();
    unsigned gf = (unsigned)((n + kBlockFinal - 1) / kBlockFinal);
    k_a_g1_finish<kBlockFinal><<<gf, kBlockFinal, (size_t)4 * 64 * kBlockFinal, st>>>(xyz, zarr, d_out, n);
    LAUNCHED();
  } else if (twist) {
    unsigned g = (unsigned)((n + kBlockCC - 1) / kBlockCC);
    if (p->dwide) pbcb200_dw::dw_g2_from_hash(d_data, (int)len, d_out, n, st);
    else if (p->type == 'f') k_cc_g2_from_hash<KF2, kBlockCC><<<g, kBlockCC, 0, st>>>(d_data, (int)len, d_out, n);
    else if (p->type == 'g') k_cc_g2_from_hash<KF5, kBlockCC><<<g, kBlockCC, 0, st>>>(d_data, (int)len, d_out, n);
    else k_cc_g2_from_hash<KF3, kBlockCC><<<g, kBlockCC, 0, st>>>(d_data, (int)len, d_out, n);
    LAUNCHED();
  } else {
    unsigned g = (unsigned)((n + kBlockCC - 1) / kBlockCC);
    if (p->dwide) pbcb200_dw::dw_from_hash(d_data, (int)len, d_out, n, st);
    else if (p->type == 'g') k_cc_g1_from_hash<kBlockCC, kWG><<<g, kBlockCC, 0, st>>>(d_data, (int)len, d_out, n);
    else k_cc_g1_from_hash<kBlockCC, kWS><<<g, kBlockCC, 0, st>>>(d_data, (int)len, d_out, n);
    LAUNCHED();
  }
  CUDA_OK(cudaGetLastError());
  if (!device) {
    CUDA_OK(cudaMemcpyAsync(out, d_out, n * elen, cudaMemcpyDeviceToHost, st));
    CUDA_OK(cudaStreamSynchronize(st));
    return 0;
  }
  return ws_release(c, st);
}

extern "C" {
int pbc_b200_g1_from_hash(pbc_b200_pairing_t* p, unsigned char* out, const unsigned char* data, size_t len, size_t n) {
  return run_from_hash(p, out, data, len, n, false, nullptr);
}
int pbc_b200_g1_from_hash_device(pbc_b200_pairing_t* p, void* d_out, const void* d_data, size_t len, size_t n,
                                 void* stream) {
  return run_from_hash(p, (unsigned char*)d_out, (const unsigned char*)d_data, len, n, true, stream);
}
int pbc_b200_g2_from_hash(pbc_b200_pairing_t* p, unsigned char* out, const unsigned char* data, size_t len, size_t n) {
  return run_from_hash(p, out, data, len, n, false, nullptr, true);
}
int pbc_b200_g2_from_hash_device(pbc_b200_pairing_t* p, void* d_out, const void* d_data, size_t len, size_t n,
                                 void* stream) {
  return run_from_hash(p, (unsigned char*)d_out, (const unsigned char*)d_data, len, n, true, stream, true);
}
}


// element_from_bytes_compressed on G1 or G2 (ecc/curve.c:799-813), batched; host buffers
static int run_decompress(pbc_b200_pairing_t* p, unsigned char* out, const unsigned char* in, size_t n, bool g2) {
  if (!p || (n && (!out || !in))) return fail("null argument");
  if (p->type == 'e') return fail("element_from_bytes_compressed: not available for type e");
  const bool twist = g2 && g2_is_twist(p);
  if (twist && !p->g2_hash_ok) return fail("element_from_bytes_compressed on G2: needs square roots in the twist's field (type f: q = 3 mod 4)");
  if (!twist && p->type != '1' && !p->hash_ok) return fail("element_from_bytes_compressed: needs q = 3 mod 4 or q = 5 mod 8 (or type d with 160..255-bit q)");
  if (n == 0) return 0;
  std::lock_guard<std::mutex> lk(p->mu);
  int dev = 0;
  CUDA_OK(cudaGetDevice(&dev));
  std::lock_guard<std::mutex> dev_lock(g_dev_mu[dev & 63]);
  if (ctx_prepare(p, dev)) return 1;
  DevCtx& c = p->ctx[dev];
  size_t elen = twist ? (size_t)p->g2_len : (size_t)p->g1_len, clen = elen / 2 + 1, need = n * (clen + elen) + 16;
  if (c.cap_dev < need) {
    CUDA_OK(cudaDeviceSynchronize());
    cudaFree(c.ws_dev);
    c.ws_dev = nullptr; c.cap_dev = 0;
    CUDA_OK(cudaMalloc(&c.ws_dev, need));
    c.cap_dev = need;
  }
  cudaStream_t st = c.stream[0];
  if (ws_acquire(c, st)) return 1;
  uint8_t* d_out = (uint8_t*)c.ws_dev;               // element output first: keeps it 4-byte aligned
  uint8_t* d_in = d_out + n * elen;
  CUDA_OK(cudaMemcpyAsync(d_in, in, n * clen, cudaMemcpyHostToDevice, st));
  if (p->type == '1') {
    unsigned g = (unsigned)((n + kBlockA1G - 1) / kBlockA1G);
    k_a1_g1_decompress<kBlockA1G><<<g, kBlockA1G, (size_t)5 * kSlotA1 * kBlockA1G, st>>>(d_in, d_out, n);
  } else if (p->type == 'a') {
    unsigned g = (unsigned)((n + kBlockMiller - 1) / kBlockMiller);
    k_a_g1_decompress<kBlockMiller><<<g, kBlockMiller, (size_t)5 * 64 * kBlockMiller, st>>>(d_in, d_out, n);
  } else if (twist) {
    unsigned g = (unsigned)((n + kBlockCC - 1) / kBlockCC);
    if (p->dwide) pbcb200_dw::dw_g2_decompress(d_in, d_out, n, st);
    else if (p->type == 'f') k_cc_g2_decompress<KF2, kBlockCC><<<g, kBlockCC, 0, st>>>(d_in, d_out, n);
    else if (p->type == 'g') k_cc_g2_decompress<KF5, kBlockCC><<<g, kBlockCC, 0, st>>>(d_in, d_out, n);
    else k_cc_g2_decompress<KF3, kBlockCC><<<g, kBlockCC, 0, st>>>(d_in, d_out, n);
  } else {
    unsigned g = (unsigned)((n + kBlockCC - 1) / kBlockCC);
    if (p->dwide) pbcb200_dw::dw_decompress(d_in, d_out, n, st);
    else if (p->type == 'g') k_cc_g1_decompress<kBlockCC, kWG><<<g, kBlockCC, 0, st>>>(d_in, d_out, n);
    else k_cc_g1_decompress<kBlockCC, kWS><<<g, kBlockCC, 0, st>>>(d_in, d_out, n);
  }
  LAUNCHED();
  CUDA_OK(cudaGetLastError());
  CUDA_OK(cudaMemcpyAsync(out, d_out, n * elen, cudaMemcpyDeviceToHost, st));
  CUDA_OK(cudaStreamSynchronize(st));
  return 0;
}
extern "C" int pbc_b200_pairing_length_in_bytes_compressed_G1(const pbc_b200_pairing_t* p) { return p->g1_len / 2 + 1; }
extern "C" int pbc_b200_g1_from_bytes_compressed(pbc_b200_pairing_t* p, unsigned char* out, const unsigned char* in,
                                                 size_t n) {
  return run_decompress(p, out, in, n, false);
}
// the x of the twist point (types f, d, g) or of the G1 point (a, a1) and one sign byte
extern "C" int pbc_b200_pairing_length_in_bytes_compressed_G2(const pbc_b200_pairing_t* p) { return p->g2_len / 2 + 1; }
extern "C" int pbc_b200_g2_from_bytes_compressed(pbc_b200_pairing_t* p, unsigned char* out, const unsigned char* in,
                                                 size_t n) {
  return run_decompress(p, out, in, n, true);
}

// ------------------------------------------------------------------------------------------
// GT operations next to the pairing (SURVEY 8f rank 3): batched element_mul, element_cmp and
// is_almost_coddh.  Host buffers; device staging is allocated per call.
// ------------------------------------------------------------------------------------------
namespace pbcb200 {
__global__ void k_bytes_cmp(uint8_t* flags, const uint8_t* a, const uint8_t* b, size_t len, size_t n);
__global__ void k_coddh_flags(uint8_t* flags, const uint8_t* t0, const uint8_t* t1, const uint8_t* t2, size_t len, size_t wb, size_t n);
}
static int enqueue_gt_mul(pbc_b200_pairing_s* p, uint8_t* d_out, const uint8_t* d_a, const uint8_t* d_b, size_t n,
                          cudaStream_t st) {
  if (p->type == 'a') {
    unsigned g = (unsigned)((n + kBlockMiller - 1) / kBlockMiller);
    k_a_gt_mul<kBlockMiller><<<g, kBlockMiller, (size_t)7 * 64 * kBlockMiller, st>>>(d_a, d_b, d_out, n);
  } else if (p->type == 'e') {
    unsigned g = (unsigned)((n + kBlockA1G - 1) / kBlockA1G);
    k_e_gt_mul<kBlockA1G><<<g, kBlockA1G, kSmemEGroup, st>>>(d_a, d_b, d_out, n);
  } else if (p->type == '1') {
    unsigned g = (unsigned)((n + kBlockA1G - 1) / kBlockA1G);
    k_a1_gt_mul<kBlockA1G><<<g, kBlockA1G, (size_t)7 * kSlotA1 * kBlockA1G, st>>>(d_a, d_b, d_out, n);
  } else {
    unsigned g = (unsigned)((n + 63) / 64);
    if (p->dwide) pbcb200_dw::dw_tower_op(0, d_out, d_a, d_b, n, st);
    else if (p->type == 'f') k_f_tower_op<<<g, 64, 0, st>>>(0, d_out, d_a, d_b, n);
    else if (p->type == 'g') k_g_tower_op<<<g, 64, 0, st>>>(0, d_out, d_a, d_b, n);
    else k_d_tower_op<<<g, 64, 0, st>>>(0, d_out, d_a, d_b, n);
  }
  LAUNCHED();
  CUDA_OK(cudaGetLastError());
  return 0;
}

extern "C" int pbc_b200_gt_mul(pbc_b200_pairing_t* p, unsigned char* out, const unsigned char* a,
                               const unsigned char* b, size_t n) {
  if (!p || (n && (!out || !a || !b))) return fail("null argument");
  if (n == 0) return 0;
  std::lock_guard<std::mutex> lk(p->mu);
  int dev = 0;
  CUDA_OK(cudaGetDevice(&dev));
  std::lock_guard<std::mutex> dev_lock(g_dev_mu[dev & 63]);
  if (ctx_prepare(p, dev)) return 1;
  cudaStream_t st = p->ctx[dev].stream[0];
  size_t len = (size_t)p->gt_len;
  DevBuf da, db, dout;
  CUDA_OK(da.alloc(n * len)); CUDA_OK(db.alloc(n * len)); CUDA_OK(dout.alloc(n * len));
  CUDA_OK(cudaMemcpyAsync(da.p, a, n * len, cudaMemcpyHostToDevice, st));
  CUDA_OK(cudaMemcpyAsync(db.p, b, n * len, cudaMemcpyHostToDevice, st));
  if (enqueue_gt_mul(p, dout.as<uint8_t>(), da.as<uint8_t>(), db.as<uint8_t>(), n, st)) return 1;
  CUDA_OK(cudaMemcpyAsync(out, dout.p, n * len, cudaMemcpyDeviceToHost, st));
  CUDA_OK(cudaStreamSynchronize(st));
  return 0;
}

extern "C" int pbc_b200_gt_cmp(pbc_b200_pairing_t* p, unsigned char* flags, const unsigned char* a,
                               const unsigned char* b, size_t n) {
  if (!p || (n && (!flags || !a || !b))) return fail("null argument");
  if (n == 0) return 0;
  std::lock_guard<std::mutex> lk(p->mu);
  int dev = 0;
  CUDA_OK(cudaGetDevice(&dev));
  std::lock_guard<std::mutex> dev_lock(g_dev_mu[dev & 63]);
  if (ctx_prepare(p, dev)) return 1;
  cudaStream_t st = p->ctx[dev].stream[0];
  size_t len = (size_t)p->gt_len;
  DevBuf da, db, df;
  CUDA_OK(da.alloc(n * len)); CUDA_OK(db.alloc(n * len)); CUDA_OK(df.alloc(n));
  CUDA_OK(cudaMemcpyAsync(da.p, a, n * len, cudaMemcpyHostToDevice, st));
  CUDA_OK(cudaMemcpyAsync(db.p, b, n * len, cudaMemcpyHostToDevice, st));
  k_bytes_cmp<<<(unsigned)((n + 127) / 128), 128, 0, st>>>(df.as<uint8_t>(), da.as<uint8_t>(), db.as<uint8_t>(), len, n);
  LAUNCHED();
  CUDA_OK(cudaGetLastError());
  CUDA_OK(cudaMemcpyAsync(flags, df.p, n, cudaMemcpyDeviceToHost, st));
  CUDA_OK(cudaStreamSynchronize(st));
  return 0;
}

extern "C" int pbc_b200_is_almost_coddh(pbc_b200_pairing_t* p, unsigned char* flags, const unsigned char* a,
                                        const unsigned char* b, const unsigned char* c, const unsigned char* d,
                                        size_t n) {
  if (!p || (n && (!flags || !a || !b || !c || !d))) return fail("null argument");
  if (n == 0) return 0;
  std::lock_guard<std::mutex> lk(p->mu);
  int dev = 0;
  CUDA_OK(cudaGetDevice(&dev));
  std::lock_guard<std::mutex> dev_lock(g_dev_mu[dev & 63]);
  if (ctx_prepare(p, dev)) return 1;
  cudaStream_t st = p->ctx[dev].stream[0];
  const size_t l1 = (size_t)p->g1_len, l2 = (size_t)p->g2_len, lt = (size_t)p->gt_len;
  Job job;
  DevBuf da, db, dc, dd, t0, t1, t2, df, ws;
  CUDA_OK(da.alloc(n * l1)); CUDA_OK(db.alloc(n * l1)); CUDA_OK(dc.alloc(n * l2)); CUDA_OK(dd.alloc(n * l2));
  CUDA_OK(t0.alloc(n * lt)); CUDA_OK(t1.alloc(n * lt)); CUDA_OK(t2.alloc(n * lt)); CUDA_OK(df.alloc(n));
  CUDA_OK(ws.alloc(ws_bytes(p, job, n)));
  CUDA_OK(cudaMemcpyAsync(da.p, a, n * l1, cudaMemcpyHostToDevice, st));
  CUDA_OK(cudaMemcpyAsync(db.p, b, n * l1, cudaMemcpyHostToDevice, st));
  CUDA_OK(cudaMemcpyAsync(dc.p, c, n * l2, cudaMemcpyHostToDevice, st));
  CUDA_OK(cudaMemcpyAsync(dd.p, d, n * l2, cudaMemcpyHostToDevice, st));
  // t0 = e(a, d), t1 = e(b, c)
  if (enqueue_pairings(p, job, t0.as<uint8_t>(), da.as<uint8_t>(), dd.as<uint8_t>(), n, ws.p, st)) return 1;
  if (enqueue_pairings(p, job, t1.as<uint8_t>(), db.as<uint8_t>(), dc.as<uint8_t>(), n, ws.p, st)) return 1;
  if (enqueue_gt_mul(p, t2.as<uint8_t>(), t0.as<uint8_t>(), t1.as<uint8_t>(), n, st)) return 1;
  size_t wb = p->type == '1' ? (size_t)p->gt_len / 2 : (p->type == 'a' ? (size_t)kWA : (p->type == 'g' ? (size_t)kWG : (size_t)p->g1_len / 2));
  k_coddh_flags<<<(unsigned)((n + 127) / 128), 128, 0, st>>>(df.as<uint8_t>(), t0.as<uint8_t>(), t1.as<uint8_t>(),
                                                            t2.as<uint8_t>(), lt, wb, n);
  LAUNCHED();
  CUDA_OK(cudaGetLastError());
  CUDA_OK(cudaMemcpyAsync(flags, df.p, n, cudaMemcpyDeviceToHost, st));
  CUDA_OK(cudaStreamSynchronize(st));
  return 0;
}

// ------------------------------------------------------------------------------------------
// F_p differential-test hook
// ------------------------------------------------------------------------------------------
namespace pbcb200 {
template <int N, bool FULL, int WB, int BLOCK>
__global__ void __launch_bounds__(BLOCK)
k_fp_op(int op, uint8_t* __restrict__ out, const uint8_t* __restrict__ a, const uint8_t* __restrict__ b,
        size_t n) {
  using O = Ops<N, FULL, BLOCK>;
  size_t idx = (size_t)blockIdx.x * BLOCK + threadIdx.x;
  if (idx >= n) return;
  uint32_t x[N], y[N], one[N] = {1};
  limbs_from_be<N, WB>(x, a + idx * WB);
  limbs_from_be<N, WB>(y, b + idx * WB);
  mont_mul<N, FULL>(x, x, c_fp.r2);
  mont_mul<N, FULL>(y, y, c_fp.r2);
  O::st(0, x); O::st(1, y);
  switch (op) {
    case 0: O::mul(0, 0, 1); break;
    case 1: O::add(0, 0, 1); break;
    case 2: O::sub(0, 0, 1); break;
    case 3: O::set_const(2, c_fp.one); slot_fermat_inverse<O, N>(3, 0, 2); O::copy(0, 3); break;
    case 4: O::halve(0, 0); break;
    case 5: O::neg(0, 0); break;
    case 6: O::sqr(0, 0); break;
    case 7: O::mulsub(0, 0, 1, 1); break;
  }
  O::ld(x, 0);
  mont_mul<N, FULL>(x, x, one);
  limbs_to_be<N, WB>(out + idx * WB, x);
}
// Ops 8-14 of the type A hook: the slot routines of the Miller step (a_step_9_line, pairing_a.cuh) in its call
// sequences and with its mode flags; coordinates per item (in a, in b, in out) from fp_op_widths, a = (a0, a1),
// b = (b0, b1):
//    8  lazy(LZ_TWO | LZ_GLOBAL_B), b0 read from a limb-major global array as qx is:  a0 b0 + a1 b1
//    9  lazy(LZ_TWO | LZ_SUB | LZ_ADD_QR | LZ_KARATSUBA) then lazy(LZ_SUB_S | LZ_ADD_QR) on the stored S':
//       out = (a0 b0 - a1 b1, a0 b1 + a1 b0, S' low half, S' high half, a0 + a1, b0 + b1); the two halves of
//       S' are the raw 512-bit slot words (S' = A0 B0 + A1 B1, less q R if that is >= q R, A = a R mod q)
//   10  sqrx(SX_SUB_1, k = 1):                          2 a0^2 - b0
//   11  sqrx(SX_ADD_A | SX_SUB_1 | SX_SUB_2):           (a0 + a1)^2 - b0 - b1
//   12  mulx(MX_ADD_A | MX_ADD_B):                      (a0 + a1)(b0 + b1)
//   13  mulx(MX_ADD_A | MX_SUB_B):                      (a0 + a1)(b0 - b1)
//   14  mulx(MX_GLOBAL_B):                              a0 b0, b0 from the global array
// It runs in 64-thread blocks: an instantiation of the slot routines of its own, so that calling them from here
// leaves the code ptxas makes for the shipped 128-thread kernels as it is (the routines are shared, and their
// callers' constant mode arguments shape that code).  g: scratch for b0, N / 4 vectors per item, n apart.
__host__ __device__ inline void fp_op_widths(int op, int* wa, int* wb, int* wo) {
  *wa = (op == 8 || op == 9 || op == 11 || op == 12 || op == 13) ? 2 : 1;
  *wb = (op == 10 || op == 14 || op < 8) ? 1 : 2;
  *wo = op == 9 ? 6 : 1;
}
template <int N, int WB, int BLOCK>
__global__ void __launch_bounds__(BLOCK)
k_fp_slot_op(int op, uint8_t* __restrict__ out, const uint8_t* __restrict__ a, const uint8_t* __restrict__ b,
             uint4* __restrict__ g, size_t n) {
  using O = Ops<N, true, BLOCK>;
  size_t idx = (size_t)blockIdx.x * BLOCK + threadIdx.x;
  if (idx >= n) return;
  int wa, wb, wo;
  fp_op_widths(op, &wa, &wb, &wo);
  uint32_t x[N], one[N] = {1};
  // coordinate c of a into slot 2c, of b into slot 2c + 1, Montgomery form
  for (int c = 0; c < wa + wb; c++) {
    const bool isa = c < wa;
    limbs_from_be<N, WB>(x, isa ? a + (idx * wa + c) * WB : b + (idx * wb + c - wa) * WB);
    mont_mul<N, true>(x, x, c_fp.r2);
    O::st(isa ? 2 * c : 2 * (c - wa) + 1, x);
  }
  if (op == 8 || op == 14) {
    O::ld(x, 1);
#pragma unroll
    for (int v = 0; v < N / 4; v++) g[v * n + idx] = make_uint4(x[4 * v], x[4 * v + 1], x[4 * v + 2], x[4 * v + 3]);
  }
  int res[6] = {0, 0, 0, 0, 0, 0};
  bool raw[6] = {false, false, false, false, false, false};
  switch (op) {    // slot aliasing as in a_step_9_line: the result overwrites an operand
    case 8: O::lazy(0, O::LZ_TWO | O::LZ_GLOBAL_B, 0, 0, 2, 3, 0, 0, g + idx, n); break;
    case 9:
      O::lazy(3, O::LZ_TWO | O::LZ_SUB | O::LZ_ADD_QR | O::LZ_KARATSUBA, 0, 1, 2, 3, 4, 5, nullptr, 0);
      O::lazy(2, O::LZ_SUB_S | O::LZ_ADD_QR, 0, 1, 0, 0, 4, 5, nullptr, 0);
      res[0] = 3; res[1] = 2; res[2] = 4; res[3] = 5; res[4] = 0; res[5] = 1;
      raw[2] = raw[3] = true;
      break;
    case 10: O::sqrx(0, 0, O::SX_SUB_1, 0, 1, 1, 0); break;
    case 11: O::sqrx(0, 0, O::SX_ADD_A | O::SX_SUB_1 | O::SX_SUB_2, 2, 0, 1, 3); break;
    case 12: O::mulx(0, 0, 1, O::MX_ADD_A | O::MX_ADD_B, 2, 3, nullptr, 0); break;
    case 13: O::mulx(0, 0, 1, O::MX_ADD_A | O::MX_SUB_B, 2, 3, nullptr, 0); break;
    default: O::mulx(0, 0, 0, O::MX_GLOBAL_B, 0, 0, g + idx, n); break;
  }
  for (int c = 0; c < wo; c++) {
    O::ld(x, res[c]);
    if (!raw[c]) mont_mul<N, true>(x, x, one);
    limbs_to_be<N, WB>(out + (idx * wo + c) * WB, x);
  }
}
// same hook for the five-limb field of types f and d
template <int W>
__global__ void k_fq_op(int op, uint8_t* __restrict__ out, const uint8_t* __restrict__ a,
                        const uint8_t* __restrict__ b, size_t n) {
  size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n) return;
  Fq x, y;
  fq_from_wire_w<W>(x, a + idx * W);
  fq_from_wire_w<W>(y, b + idx * W);
  switch (op) {
    case 0: fq_mul(x, x, y); break;
    case 1: fq_add(x, x, y); break;
    case 2: fq_sub(x, x, y); break;
    case 3: fq_inv(&x, &x); break;
    case 4: fq_halve(x, x); break;
    case 5: fq_neg(x, x); break;
    case 6: fq_sqr(x, x); break;
    case 7: fq_mul(x, x, y); fq_sub(x, x, y); break;
  }
  fq_to_wire_w<W>(out + idx * W, x);
}

// ---- tower_op 3 for types a, a1 and e: GT wire elements -> the Miller-value layout of the final stage ----
// Element e of a limb-major batch array, as Ops::st_global writes it: vector v (VW words) at (e * N / VW + v) * n + idx.
template <int N, int VW>
__device__ __forceinline__ void mv_store(void* g, int e, size_t n, size_t idx, const uint32_t* x) {
  uint32_t* w = reinterpret_cast<uint32_t*>(g);
#pragma unroll
  for (int v = 0; v < N / VW; v++)
#pragma unroll
    for (int k = 0; k < VW; k++) w[(((size_t)e * (N / VW) + v) * n + idx) * VW + k] = x[v * VW + k];
}
// wire coordinate (wb bytes, big-endian, any value below 2^(8 wb)) -> Montgomery form, reduced mod q as
// element_from_bytes reduces it.  R^2 is the full operand and the wire value the scanned one (a1_load_point).
template <int N, bool FULL>
__device__ __forceinline__ void mv_coord(uint32_t* x, const uint8_t* p, int wb) {
  uint32_t w[N];
  if constexpr (N == kNA) limbs_from_be<kNA, kWA>(w, p);
  else a1_limbs_from_be(w, p, wb);
  mont_mul<N, FULL>(x, c_fp.r2, w);
}
// types a and a1: f = (x, y) from an F_q^2 element x || y, and D = N(f) f0 f1 = (f0^2 + f1^2) f0 f1 as the
// Miller kernels publish it (a_publish, a1_publish): 0 exactly when f0 f1 = 0, the final stage's shortcut to 1.
template <int N, bool FULL, int VW>
__global__ void k_a_mv_from_wire(void* __restrict__ f, void* __restrict__ dprod, const uint8_t* __restrict__ in,
                                 size_t n, int wb) {
  size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n) return;
  uint32_t f0[N], f1[N], s[N], t[N];
  mv_coord<N, FULL>(f0, in + idx * 2 * (size_t)wb, wb);
  mv_coord<N, FULL>(f1, in + idx * 2 * (size_t)wb + wb, wb);
  mv_store<N, VW>(f, 0, n, idx, f0);
  mv_store<N, VW>(f, 1, n, idx, f1);
  mont_mul<N, FULL>(s, f0, f0);
  mont_mul<N, FULL>(t, f1, f1);
  fp_add<N, FULL>(s, s, t);
  mont_mul<N, FULL>(t, f0, f1);
  mont_mul<N, FULL>(s, s, t);
  mv_store<N, VW>(dprod, 0, n, idx, s);
}
// type e: f = v from a, dprod = vd from b (e_publish), b == nullptr: vd = 1
__global__ void k_e_mv_from_wire(void* __restrict__ f, void* __restrict__ dprod, const uint8_t* __restrict__ a,
                                 const uint8_t* __restrict__ b, size_t n) {
  size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n) return;
  const int wb = (int)c_a1.wb;
  uint32_t x[kNA1];
  mv_coord<kNA1, false>(x, a + idx * (size_t)wb, wb);
  mv_store<kNA1, 2>(f, 0, n, idx, x);
  if (b) {
    mv_coord<kNA1, false>(x, b + idx * (size_t)wb, wb);
  } else {
#pragma unroll
    for (int k = 0; k < kNA1; k++) x[k] = c_fp.one[k];
  }
  mv_store<kNA1, 2>(dprod, 0, n, idx, x);
}

// element_cmp on wire bytes (canonical residues: equal elements <=> equal bytes): flags[i] = 1 if a[i] != b[i]
__global__ void k_bytes_cmp(uint8_t* __restrict__ flags, const uint8_t* __restrict__ a, const uint8_t* __restrict__ b,
                            size_t len, size_t n) {
  size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n) return;
  uint32_t diff = 0;
  for (size_t k = 0; k < len; k++) diff |= (uint32_t)(a[idx * len + k] ^ b[idx * len + k]);
  flags[idx] = diff ? 1 : 0;
}
// is_almost_coddh (ecc/pairing.c:15-33, ecc/d_param.c:739-784): 1 if t0 == t1 or t0 t1 == 1; t2 = t0 t1.
// The GT identity on the wire: the first coordinate is 1 (wb bytes, big-endian), every other one 0.
__global__ void k_coddh_flags(uint8_t* __restrict__ flags, const uint8_t* __restrict__ t0, const uint8_t* __restrict__ t1,
                              const uint8_t* __restrict__ t2, size_t len, size_t wb, size_t n) {
  size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n) return;
  uint32_t diff = 0, notone = 0;
  for (size_t k = 0; k < len; k++) {
    diff |= (uint32_t)(t0[idx * len + k] ^ t1[idx * len + k]);
    notone |= (uint32_t)(t2[idx * len + k] ^ (k == wb - 1 ? 1u : 0u));
  }
  flags[idx] = (!diff || !notone) ? 1 : 0;
}

// dependent chain of five-limb Montgomery multiplications (mode 0) / squarings (mode 1)
__global__ void k_fqmul_chain(uint32_t* __restrict__ out, const uint32_t* __restrict__ in, int iters, int mode) {
  size_t T = (size_t)gridDim.x * blockDim.x, t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  Fq a, b;
#pragma unroll
  for (int k = 0; k < kNS; k++) { a.v[k] = in[(2 * k) * T + t]; b.v[k] = in[(2 * k + 1) * T + t]; }
  if (mode == 0) for (int i = 0; i < iters; i++) fq_mul(a, a, b);
  else for (int i = 0; i < iters; i++) fq_sqr(a, a);
#pragma unroll
  for (int k = 0; k < kNS; k++) out[k * T + t] = a.v[k];
}
}  // namespace pbcb200

extern "C" int pbc_b200_fp_op(pbc_b200_pairing_t* p, int op, unsigned char* out,
                              const unsigned char* a, const unsigned char* b, size_t n) {
  if (!p || (n && (!out || !a))) return fail("null argument");
  if (n == 0) return 0;
  int dev = 0;
  CUDA_OK(cudaGetDevice(&dev));
  std::lock_guard<std::mutex> dev_lock(g_dev_mu[dev & 63]);
  if (ctx_prepare(p, dev)) return 1;
  size_t wb = (size_t)p->g1_len / 2;             // bytes per F_q coordinate: 64, 20, 19 or ceil(bits(p)/8)
  int wa = 1, wbn = 1, wo = 1;                   // coordinates per item (type a ops 8-14: see fp_op_widths)
  if (p->type == 'a') {
    if (op < 0 || op > 14) return fail("fp_op: type a has ops 0..14");
    fp_op_widths(op, &wa, &wbn, &wo);
  }
  if (wbn > 1 && !b) return fail("fp_op %d: needs b", op);
  DevBuf da, db, dout, dg;
  CUDA_OK(da.alloc(n * wb * wa));
  CUDA_OK(db.alloc(n * wb * wbn));
  CUDA_OK(dout.alloc(n * wb * wo));
  CUDA_OK(cudaMemcpy(da.p, a, n * wb * wa, cudaMemcpyHostToDevice));
  CUDA_OK(cudaMemcpy(db.p, b ? b : a, n * wb * wbn, cudaMemcpyHostToDevice));
  unsigned g = (unsigned)((n + 127) / 128);
  if (p->type == '1' || p->type == 'e') {
    k_a1_fp_op<kBlockA1Small><<<g, kBlockA1Small, (size_t)4 * kSlotA1 * kBlockA1Small>>>(op, dout.as<uint8_t>(), da.as<uint8_t>(), db.as<uint8_t>(), n);
  } else if (p->type == 'a' && op >= 8) {
    CUDA_OK(dg.alloc(n * wb));                   // b0 of ops 8 and 14 as a limb-major global array
    k_fp_slot_op<kNA, 64, 64><<<(unsigned)((n + 63) / 64), 64, 6 * 64 * 64>>>(op, dout.as<uint8_t>(), da.as<uint8_t>(),
                                                                          db.as<uint8_t>(), dg.as<uint4>(), n);
  } else if (p->type == 'a') {
    CUDA_OK(allow_smem(k_fp_op<kNA, true, 64, 128>, 4 * 64 * 128));
    k_fp_op<kNA, true, 64, 128><<<g, 128, 4 * 64 * 128>>>(op, dout.as<uint8_t>(), da.as<uint8_t>(), db.as<uint8_t>(), n);
  } else if (p->dwide) {
    pbcb200_dw::dw_fq_op(op, dout.as<uint8_t>(), da.as<uint8_t>(), db.as<uint8_t>(), n, 0);
  } else if (p->type == 'g') {
    k_fq_op<kWG><<<g, 128>>>(op, dout.as<uint8_t>(), da.as<uint8_t>(), db.as<uint8_t>(), n);
  } else {
    k_fq_op<kWS><<<g, 128>>>(op, dout.as<uint8_t>(), da.as<uint8_t>(), db.as<uint8_t>(), n);
  }
  LAUNCHED();
  CUDA_OK(cudaDeviceSynchronize());
  CUDA_OK(cudaMemcpy(out, dout.p, n * wb * wo, cudaMemcpyDeviceToHost));
  return 0;
}

/* GT-sized differential-test hook for the extension towers of types f, d and g (see k_f_tower_op,
 * k_d_tower_op, k_g_tower_op) and for the final stage of types a, a1 and e (op 3: enqueue_final on
 * Miller values made by k_a_mv_from_wire / k_e_mv_from_wire): operands and results in GT wire format. */
extern "C" int pbc_b200_tower_op(pbc_b200_pairing_t* p, int op, unsigned char* out,
                                 const unsigned char* a, const unsigned char* b, size_t n) {
  if (!p || (n && (!out || !a))) return fail("null argument");
  const bool batched_final = p->type == 'a' || p->type == '1' || p->type == 'e';
  if (!batched_final && p->type != 'f' && p->type != 'd' && p->type != 'g') return fail("tower_op: types a, a1, e, f, d and g only");
  if (batched_final && op != 3) return fail("tower_op: types a, a1 and e have op 3 only");
  if (n == 0) return 0;
  int dev = 0;
  CUDA_OK(cudaGetDevice(&dev));
  std::lock_guard<std::mutex> dev_lock(g_dev_mu[dev & 63]);
  if (ctx_prepare(p, dev)) return 1;
  size_t wb = (size_t)p->gt_len;
  DevBuf da, db, dout;
  if (batched_final) {
    // the final stage every pairing of these types takes (enqueue_final), on the caller's elements: they go
    // into the Miller-value layout first -- f and D = N(f) f0 f1 (a, a1), v and vd (e)
    const size_t el = p->type == 'a' ? (size_t)kNA * 4 : (size_t)kNA1 * 4;   // bytes per F_q element
    const size_t fw = p->type == 'e' ? 1 : 2;                                 // F_q elements per Miller value
    DevBuf ws;
    CUDA_OK(ws.alloc(n * el * (fw + 2)));
    uint8_t* f = ws.as<uint8_t>();
    uint8_t* dprod = f + fw * el * n;
    uint8_t* prefix = dprod + el * n;
    if (p->type == 'e' && b) {
      CUDA_OK(db.alloc(n * wb));
      CUDA_OK(cudaMemcpy(db.p, b, n * wb, cudaMemcpyHostToDevice));
    }
    CUDA_OK(da.alloc(n * wb));
    CUDA_OK(dout.alloc(n * wb));
    CUDA_OK(cudaMemcpy(da.p, a, n * wb, cudaMemcpyHostToDevice));
    unsigned g = (unsigned)((n + 127) / 128);
    if (p->type == 'a') k_a_mv_from_wire<kNA, true, 4><<<g, 128>>>(f, dprod, da.as<uint8_t>(), n, kWA);
    else if (p->type == '1') k_a_mv_from_wire<kNA1, false, 2><<<g, 128>>>(f, dprod, da.as<uint8_t>(), n, (int)(wb / 2));
    else k_e_mv_from_wire<<<g, 128>>>(f, dprod, da.as<uint8_t>(), db.as<uint8_t>(), n);
    LAUNCHED();
    if (enqueue_final(p, f, dprod, prefix, dout.as<uint8_t>(), n, 0, nullptr)) return 1;
    CUDA_OK(cudaGetLastError());
    CUDA_OK(cudaDeviceSynchronize());
    CUDA_OK(cudaMemcpy(out, dout.p, n * wb, cudaMemcpyDeviceToHost));
    return 0;
  }
  CUDA_OK(da.alloc(n * wb));
  CUDA_OK(db.alloc(n * wb));
  CUDA_OK(dout.alloc(n * wb));
  CUDA_OK(cudaMemcpy(da.p, a, n * wb, cudaMemcpyHostToDevice));
  CUDA_OK(cudaMemcpy(db.p, b ? b : a, n * wb, cudaMemcpyHostToDevice));
  unsigned g = (unsigned)((n + 63) / 64);
  if (op == 6 && p->type == 'f') {
    // the final exponentiation every type F pairing takes (k_f_finalexp_s), on the caller's elements: they
    // go into the Miller-value layout with their flags set, then the launch of enqueue_pairings
    if (!(p->f.slots_ok && p->f.bn))
      return fail("tower_op 6: the slot-machine final exponentiation needs the internal basis and a BN parameter");
    DevBuf ws;
    CUDA_OK(ws.alloc(n * 4 * ((size_t)kF12Words + 1 + (size_t)kFStashWords)));
    uint32_t* mv = ws.as<uint32_t>();
    uint32_t* flag = mv + (size_t)kF12Words * n;
    uint32_t* stash = flag + n;
    k_f_mv_from_wire<<<g, 64>>>(mv, flag, da.as<uint8_t>(), n);
    LAUNCHED();
    k_f_finalexp_s<kBlockFS><<<(unsigned)((n + kBlockFS - 1) / kBlockFS), kBlockFS, kSmemFFinalS>>>(mv, flag, dout.as<uint8_t>(), stash, n);
    LAUNCHED();
    CUDA_OK(cudaDeviceSynchronize());
    CUDA_OK(cudaMemcpy(out, dout.p, n * wb, cudaMemcpyDeviceToHost));
    return 0;
  }
  if (p->dwide) pbcb200_dw::dw_tower_op(op, dout.as<uint8_t>(), da.as<uint8_t>(), db.as<uint8_t>(), n, 0);
  else if (p->type == 'f') k_f_tower_op<<<g, 64>>>(op, dout.as<uint8_t>(), da.as<uint8_t>(), db.as<uint8_t>(), n);
  else if (p->type == 'g') k_g_tower_op<<<g, 64>>>(op, dout.as<uint8_t>(), da.as<uint8_t>(), db.as<uint8_t>(), n);
  else k_d_tower_op<<<g, 64>>>(op, dout.as<uint8_t>(), da.as<uint8_t>(), db.as<uint8_t>(), n);
  LAUNCHED();
  CUDA_OK(cudaDeviceSynchronize());
  CUDA_OK(cudaMemcpy(out, dout.p, n * wb, cudaMemcpyDeviceToHost));
  return 0;
}
