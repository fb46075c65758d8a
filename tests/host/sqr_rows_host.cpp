// sqr_rows_host.cpp -- runs the row-wise squarer of fp.cuh (sqr_wide, mont_sqr_os) and the single-pass
// redc_wide on the CPU through the PTX interpreter.
//
// TEST INFRASTRUCTURE.  Compiled against the header tests/host/make_host_fp.py generates.  One request
// per line on stdin:   op n p a      (hex; n = limbs, decimal)     one result per line on stdout (hex):
//   wsqr    the exact 64 n-bit square of a          (n = 8 or 16)
//   sqr     a^2 / R mod p, mont_sqr_os              (n = 8 or 16)
//   fpsqr   a^2 / R mod p, fp_sqr<16, true>: the squarer the type A kernels call
//   redc1   a / R mod p for a < p R, redc_wide with one conditional subtraction (n = 16)
#include HOST_FP_HEADER

#include <iostream>
#include <string>

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

template <int N>
static std::string run(const std::string& op, const std::string& sa) {
  uint32_t a[N], r[N], t[2 * N + 1];
  from_hex(sa, a, N);
  if (op == "wsqr") { sqr_wide<N>(t, a); return to_hex(t, 2 * N); }
  if (op == "sqr") { mont_sqr_os<N>(r, a); return to_hex(r, N); }
  if (op == "redc1") { from_hex(sa, t, 2 * N + 1); redc_wide<N, 1>(r, t); return to_hex(r, N); }
  if constexpr (N == 16) {
    if (op == "fpsqr") { fp_sqr<16, true>(r, a); return to_hex(r, N); }
  }
  return "?";
}

int main() {
  std::string op, sp, sa;
  int n;
  while (std::cin >> op >> n >> sp >> sa) {
    memset(&c_fp, 0, sizeof c_fp);
    from_hex(sp, c_fp.p, kMaxLimbs);
    c_fp.np0 = neg_inv32(c_fp.p[0]);
    c_fp.nlimbs = n;
    std::cout << (n == 16 ? run<16>(op, sa) : n == 8 ? run<8>(op, sa) : std::string("?")) << "\n";
  }
  return 0;
}
