// limb_arith_host.cpp -- runs the limb-level field arithmetic of fp.cuh / fq_small.cuh on the CPU.
//
// TEST INFRASTRUCTURE.  Compiled against the header tests/host/make_host_fp.py generates (the
// device templates with their inline PTX routed through tests/host/ptx_emul.hpp).  One request per
// line on stdin:   N FULL op p a b c d      (hex, little-endian words are rebuilt here)
// one result per line on stdout (hex).  ops:
//   mul_os  mont_mul<N,FULL>(a, b)        mul_ps  mont_mul_ps<N,FULL>(a, b)     sqr_ps  mont_sqr_ps<N,FULL>(a)
//   add sub neg halve                      fp_add / fp_sub / fp_neg / fp_halve
//   fq_mul  fq_redc_call(fq_mulw_call(a, b))                       (N = kNS only)
//   fq_mul_os / fq_mac_os  the same through the inline operand-scanning product fqw_mul and fqw_redc2
//   fq_mul_rows / fq_mul_rows2 / fq_acc3 / fq_acc4  the accumulating products (FqAcc) and the row-wise reduction fqw_redc_os
//   fq_mac  fq_redc2_call(a b + c d)  fq_msb  fq_redc2_call(a b + (q R - c d))... see the test
#include HOST_FP_HEADER

#include <iostream>
#include <string>
#include <vector>

using namespace pbcb200;

static void from_hex(const std::string& s, uint32_t* w, int n) {
  for (int i = 0; i < n; i++) w[i] = 0;
  int bit = 0;
  for (size_t i = s.size(); i-- > 0;) {
    char c = s[i];
    uint32_t v = c <= '9' ? c - '0' : (c | 32) - 'a' + 10;
    if (bit / 32 < n) w[bit / 32] |= v << (bit % 32);
    bit += 4;
  }
}
static std::string to_hex(const uint32_t* w, int n) {
  std::string r;
  char buf[16];
  for (int i = n; i-- > 0;) { snprintf(buf, sizeof buf, "%08x", w[i]); r += buf; }
  return r;
}
static uint32_t neg_inv32(uint32_t p0) {
  uint32_t x = 1;
  for (int i = 0; i < 6; i++) x *= 2u - p0 * x;
  return 0u - x;
}

template <int N, bool FULL>
static std::string run(const std::string& op, const std::string& a_, const std::string& b_) {
  uint32_t a[N], b[N], r[N];
  from_hex(a_, a, N);
  from_hex(b_, b, N);
  if (op == "mul_os") { if constexpr (N % 2 == 0) mont_mul<N, FULL>(r, a, b); else return "odd"; }
  else if (op == "mul_ps") mont_mul_ps<N, FULL>(r, a, b);
  else if (op == "sqr_ps") mont_sqr_ps<N, FULL>(r, a);
  else if (op == "add") fp_add<N, FULL>(r, a, b);
  else if (op == "sub") fp_sub<N>(r, a, b);
  else if (op == "neg") fp_neg<N>(r, a);
  else if (op == "halve") fp_halve<N, FULL>(r, a);
  else return "?";
  return to_hex(r, N);
}

int main() {
  std::string sN, sF, op, p, a, b, c, d;
  while (std::cin >> sN >> sF >> op >> p >> a >> b >> c >> d) {
    int N = atoi(sN.c_str());
    bool full = sF == "1";
    memset(&c_fp, 0, sizeof c_fp);
    from_hex(p, c_fp.p, kMaxLimbs);
    c_fp.np0 = neg_inv32(c_fp.p[0]);
    c_fp.nlimbs = (uint32_t)N;
    std::string out = "?";
    if (op.rfind("fq_", 0) == 0) {
      if (N != kNS) { out = "kNS"; }
      else {
        Fq A, B, C, D;
        from_hex(a, A.v, kNS); from_hex(b, B.v, kNS); from_hex(c, C.v, kNS); from_hex(d, D.v, kNS);
        Fq R;
        if (op == "fq_wmul") { FqW t; fqw_mul(t, A, B); std::cout << to_hex(t.v, 2 * kNS) << "\n"; continue; }
        if (op == "fq_mul") R = fq_redc_call(fq_mulw_call(A, B));
        else if (op == "fq_mac") { FqW s, t = fq_mulw_call(A, B), u = fq_mulw_call(C, D); fqw_add(s, t, u); R = fq_redc2_call(s); }
        else if (op == "fq_mul_os") { FqW t; fqw_mul(t, A, B); fqw_redc2(R, t); }
        else if (op == "fq_mac_os") { FqW s, t, u; fqw_mul(t, A, B); fqw_mul(u, C, D); fqw_add(s, t, u); fqw_redc2(R, s); }
        else if (op == "fq_mul_rows") { fq_mul_os(R, A, B); }                                   // fqa_mul + fqa_merge + fqw_redc_os<false>
        else if (op == "fq_mul_rows2") { FqAcc g; FqW t; fqa_mul(g, A, B); fqa_merge<false>(t, g); fqw_redc_os<true>(R, t); }
        else if (op == "fq_acc3" || op == "fq_acc4") {
          // a b + c d + a d (+ c b), unmerged; printed as the 320-bit value
          FqAcc g; FqW t;
          fqa_mul(g, A, B); fqa_mac<true>(g, C, D); fqa_mac<false>(g, A, D);
          if (op == "fq_acc4") fqa_mac<false>(g, C, B);
          fqa_merge<true>(t, g);
          std::cout << to_hex(t.v, 2 * kNS) << "\n"; continue;
        }
        else if (op == "fq_mulcall") R = fq_mul_call(A, B);
        else if (op == "fq_sqrcall") R = fq_sqr_call(A);
        else { std::cout << "?" << "\n"; continue; }
        out = to_hex(R.v, kNS);
      }
    } else {
#define CASE(n, f) if (N == n && full == f) out = run<n, f>(op, a, b);
      CASE(5, false) CASE(6, false) CASE(16, true) CASE(16, false) CASE(34, false) CASE(34, true)
#undef CASE
    }
    std::cout << out << "\n";
  }
  fprintf(stderr, "ptx instructions interpreted: %llu\n", (unsigned long long)ptxemu::executed());
  return 0;
}
