// lazy_redc_host.cpp -- runs the double-width primitives of fp.cuh (mul_wide, wide_add / wide_sub,
// wide_add_pR, wide_sub_pR_if_ge, redc_wide) on the CPU, N = 16, through the PTX interpreter.
//
// TEST INFRASTRUCTURE.  Compiled against the header tests/host/make_host_fp.py generates.  One request
// per line on stdin:   op p a b c d s      (hex)     one result per line on stdout (hex):
//   wmul    a b                          the 1024-bit product
//   redc    a (a value below 2 p R)      a / R mod p
//   sum     (a b + c d) / R              the Re l combination of the type A Miller step
//   kara0   (a b - c d + p R) / R  and  S' = a b + c d (- p R if >= p R), as "r s"
//   kara1   (a b - s + p R) / R
// Each combination follows Ops::lazy (slots.cuh) step for step.
#include HOST_FP_HEADER

#include <iostream>
#include <string>

using namespace pbcb200;

constexpr int N = 16;

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

int main() {
  std::string op, sp, sa, sb, sc, sd, ss;
  while (std::cin >> op >> sp >> sa >> sb >> sc >> sd >> ss) {
    memset(&c_fp, 0, sizeof c_fp);
    from_hex(sp, c_fp.p, kMaxLimbs);
    c_fp.np0 = neg_inv32(c_fp.p[0]);
    c_fp.nlimbs = N;
    uint32_t a[N], b[N], c[N], d[N], s[2 * N], acc[2 * N + 1] = {0}, p[2 * N], r[N];
    from_hex(sa, a, N); from_hex(sb, b, N); from_hex(sc, c, N); from_hex(sd, d, N); from_hex(ss, s, 2 * N);
    if (op == "wmul") {
      mul_wide<N>(p, a, b);
      std::cout << to_hex(p, 2 * N) << "\n";
    } else if (op == "redc") {
      from_hex(sa, acc, 2 * N + 1);
      redc_wide<N>(r, acc);
      std::cout << to_hex(r, N) << "\n";
    } else if (op == "sum") {
      mul_wide<N>(p, a, b); wide_add<N>(acc, p);
      mul_wide<N>(p, c, d); wide_add<N>(acc, p);
      redc_wide<N>(r, acc);
      std::cout << to_hex(r, N) << "\n";
    } else if (op == "kara0") {
      uint32_t t[2 * N + 1];
      mul_wide<N>(p, a, b); wide_add<N>(acc, p);
      mul_wide<N>(p, c, d);
      for (int k = 0; k <= 2 * N; k++) t[k] = acc[k];
      wide_add<N>(t, p);
      wide_sub_pR_if_ge<N>(t);
      wide_sub<N>(acc, p);
      wide_add_pR<N>(acc);
      redc_wide<N>(r, acc);
      std::cout << to_hex(r, N) << " " << to_hex(t, 2 * N + 1) << "\n";
    } else if (op == "kara1") {
      wide_sub<N>(acc, s);
      mul_wide<N>(p, a, b); wide_add<N>(acc, p);
      wide_add_pR<N>(acc);
      redc_wide<N>(r, acc);
      std::cout << to_hex(r, N) << "\n";
    } else {
      std::cout << "?\n";
    }
  }
  return 0;
}
