/* shim_test.c -- drop-in check through the reference's own API (pbc.h).
 *
 * TEST PROGRAM.  Links libpbc_b200_shim.so in front of the reference library, so
 * pairing_init_set_buf below is the interposed one and element_pairing /
 * element_prod_pairing / pairing_pp_apply run on the GPU; a second pairing_t initialised through
 * pairing_init_pbc_param (the reference's un-interposed initialiser) keeps the reference's CPU
 * vtable and serves as the checker.  Every comparison is on element_to_bytes output.
 *
 *   shim_test <param-file> [n_batch]
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <pbc.h>

void element_pairing_batch(element_t out[], element_t in1[], element_t in2[], int n);
void element_pow_zn_batch(element_t out[], element_t in[], element_t k[], int n);
void element_from_hash_batch(element_t out[], const void *data, int len, int n);
int pbc_b200_pairing_batch(pairing_t pairing, unsigned char *out, const unsigned char *in1,
                           const unsigned char *in2, size_t n);
int pbc_b200_prod_pairing_batch_v(pairing_t pairing, unsigned char *out, const unsigned char *in1,
                                  const unsigned char *in2, const size_t *offsets, size_t n_out);

static int same(element_t a, element_t b) {
  unsigned char x[1024], y[1024];
  int n = element_length_in_bytes(a);
  if (n != element_length_in_bytes(b) || n > 1024) return 0;
  element_to_bytes(x, a);
  element_to_bytes(y, b);
  return memcmp(x, y, n) == 0;
}
static void copy_elem(element_t dst, element_t src) {
  unsigned char x[1024];
  element_to_bytes(x, src);
  element_from_bytes(dst, x);
}

int main(int argc, char **argv) {
  static char param[16384];
  size_t len;
  FILE *fp;
  pairing_t gpu, cpu;
  pbc_param_t par;
  int i, n = argc > 2 ? atoi(argv[2]) : 256, bad = 0;
  if (argc < 2 || !(fp = fopen(argv[1], "r"))) { fprintf(stderr, "usage: shim_test <param-file> [n]\n"); return 2; }
  len = fread(param, 1, sizeof param - 1, fp);
  fclose(fp);
  param[len] = 0;
  if (pairing_init_set_buf(gpu, param, len)) { fprintf(stderr, "GPU-attached init failed\n"); return 1; }
  if (pbc_param_init_set_buf(par, param, len)) return 1;
  pairing_init_pbc_param(cpu, par);
  pbc_param_clear(par);
  pbc_random_set_deterministic(20260922);

  element_t *P = malloc(n * sizeof *P), *Q = malloc(n * sizeof *Q), *E = malloc(n * sizeof *E);
  element_t p2, q2, e2, ep;
  element_init_G1(p2, cpu); element_init_G2(q2, cpu); element_init_GT(e2, cpu); element_init_GT(ep, gpu);
  for (i = 0; i < n; i++) {
    element_init_G1(P[i], gpu); element_init_G2(Q[i], gpu); element_init_GT(E[i], gpu);
    element_random(P[i]); element_random(Q[i]);
  }
  /* 1. element_pairing, one at a time, GPU vs CPU vtable */
  for (i = 0; i < 4; i++) {
    element_pairing(E[i], P[i], Q[i]);
    copy_elem(p2, P[i]); copy_elem(q2, Q[i]);
    element_pairing(e2, p2, q2);
    if (!same(E[i], e2)) { printf("element_pairing mismatch at %d\n", i); bad++; }
  }
  /* 2. element_prod_pairing (n_prod = 4) */
  {
    element_t pc[4], qc[4];
    for (i = 0; i < 4; i++) { element_init_G1(pc[i], cpu); element_init_G2(qc[i], cpu); copy_elem(pc[i], P[i]); copy_elem(qc[i], Q[i]); }
    element_prod_pairing(ep, P, Q, 4);
    element_prod_pairing(e2, pc, qc, 4);
    if (!same(ep, e2)) { printf("element_prod_pairing mismatch\n"); bad++; }
    for (i = 0; i < 4; i++) { element_clear(pc[i]); element_clear(qc[i]); }
  }
  /* 2b. products with a pair count per output: segments of 1, 2 and 5 pairs (P[0..7]) in one call,
   * each against element_prod_pairing of the CPU vtable */
  {
    static const size_t off[4] = {0, 1, 3, 8};
    int l1 = pairing_length_in_bytes_G1(gpu), l2 = pairing_length_in_bytes_G2(gpu), lt = pairing_length_in_bytes_GT(gpu);
    unsigned char *b1 = malloc((size_t)8 * (l1 + l2) + (size_t)3 * lt), *b2 = b1 + (size_t)8 * l1, *bo = b2 + (size_t)8 * l2;
    element_t pc[5], qc[5];
    for (i = 0; i < 8; i++) { element_to_bytes(b1 + (size_t)i * l1, P[i]); element_to_bytes(b2 + (size_t)i * l2, Q[i]); }
    int rc = pbc_b200_prod_pairing_batch_v(gpu, bo, b1, b2, off, 3);
    if (rc) { printf("pbc_b200_prod_pairing_batch_v failed\n"); bad++; }
    for (i = 0; i < 5; i++) { element_init_G1(pc[i], cpu); element_init_G2(qc[i], cpu); }
    for (int s = 0; s < 3 && !rc; s++) {
      int len = (int)(off[s + 1] - off[s]);
      for (i = 0; i < len; i++) { copy_elem(pc[i], P[off[s] + i]); copy_elem(qc[i], Q[off[s] + i]); }
      element_prod_pairing(e2, pc, qc, len);
      element_from_bytes(ep, bo + (size_t)s * lt);
      if (!same(ep, e2)) { printf("pbc_b200_prod_pairing_batch_v mismatch in segment %d\n", s); bad++; }
    }
    for (i = 0; i < 5; i++) { element_clear(pc[i]); element_clear(qc[i]); }
    free(b1);
  }
  /* 3. pairing_pp_* */
  {
    pairing_pp_t pp;
    pairing_pp_init(pp, P[0], gpu);
    for (i = 0; i < 3; i++) {
      pairing_pp_apply(ep, Q[i], pp);
      copy_elem(p2, P[0]); copy_elem(q2, Q[i]);
      element_pairing(e2, p2, q2);
      if (!same(ep, e2)) { printf("pairing_pp_apply mismatch at %d\n", i); bad++; }
    }
    pairing_pp_clear(pp);
  }
  /* 4. identity semantics: e(O, Q) = 1 */
  element_set0(P[5]);
  element_pairing(ep, P[5], Q[5]);
  if (!element_is1(ep)) { printf("e(O,Q) != 1\n"); bad++; }
  /* 5. the batch entry point over element_t arrays (P[5] is O) */
  element_pairing_batch(E, P, Q, n);
  for (i = 0; i < n; i++) {
    if (element_is0(P[i])) { if (!element_is1(E[i])) { printf("batch identity mismatch at %d\n", i); bad++; } continue; }
    copy_elem(p2, P[i]); copy_elem(q2, Q[i]);
    element_pairing(e2, p2, q2);
    if (!same(E[i], e2)) { printf("batch mismatch at %d\n", i); bad++; if (bad > 8) break; }
  }
  /* 6. element_pow_zn over arrays, G1 and GT, GPU batch vs the reference's windowed power */
  {
    int m = n < 16 ? n : 16;
    element_t *K = malloc(m * sizeof *K), *R = malloc(m * sizeof *R), ref, kc;
    element_init_G1(ref, cpu); element_init_Zr(kc, cpu);
    for (i = 0; i < m; i++) { element_init_Zr(K[i], gpu); element_random(K[i]); element_init_G1(R[i], gpu); }
    element_pow_zn_batch(R, P + 6, K, m);
    for (i = 0; i < m; i++) {
      copy_elem(p2, P[6 + i]); copy_elem(kc, K[i]);
      element_pow_zn(ref, p2, kc);
      if (!same(R[i], ref)) { printf("G1 pow_zn batch mismatch at %d\n", i); bad++; }
    }
    element_pow_zn_batch(E + 6, E + 6, K, m);          /* in place on GT */
    for (i = 0; i < m; i++) {
      copy_elem(p2, P[6 + i]); copy_elem(q2, Q[6 + i]); copy_elem(kc, K[i]);
      element_pairing(e2, p2, q2);
      element_pow_zn(e2, e2, kc);
      if (!same(E[6 + i], e2)) { printf("GT pow_zn batch mismatch at %d\n", i); bad++; }
    }
    for (i = 0; i < m; i++) { element_clear(K[i]); element_clear(R[i]); }
    element_clear(ref); element_clear(kc);
  }
  {  /* element_from_hash_batch on G1 and G2 against element_from_hash of the CPU pairing */
    enum { H = 9, HL = 37 };
    unsigned char msg[H * HL];
    element_t G[H], ref1, ref2;
    for (i = 0; i < H * HL; i++) msg[i] = (unsigned char)(i * 131 + 7);
    element_init_G1(ref1, cpu); element_init_G2(ref2, cpu);
    for (i = 0; i < H; i++) element_init_G1(G[i], gpu);
    element_from_hash_batch(G, msg, HL, H);
    for (i = 0; i < H; i++) {
      element_from_hash(ref1, msg + i * HL, HL);
      if (!same(G[i], ref1) && !(element_is0(ref1) && element_is0(G[i]))) { printf("G1 from_hash batch mismatch at %d\n", i); bad++; }
      element_clear(G[i]);
      element_init_G2(G[i], gpu);
    }
    element_from_hash_batch(G, msg, HL, H);
    for (i = 0; i < H; i++) {
      element_from_hash(ref2, msg + i * HL, HL);
      if (!same(G[i], ref2)) { printf("G2 from_hash batch mismatch at %d\n", i); bad++; }
      element_clear(G[i]);
    }
    element_clear(ref1); element_clear(ref2);
  }
  printf("shim_test: %s (%d batch pairings, prod, ragged prod 1+2+5, pp, identity, pow_zn, from_hash G1 / G2; G1 %d B, G2 %d B, GT %d B)\n",
         bad ? "FAILED" : "OK", n, pairing_length_in_bytes_G1(gpu), pairing_length_in_bytes_G2(gpu),
         pairing_length_in_bytes_GT(gpu));
  for (i = 0; i < n; i++) { element_clear(P[i]); element_clear(Q[i]); element_clear(E[i]); }
  element_clear(p2); element_clear(q2); element_clear(e2); element_clear(ep);
  pairing_clear(gpu);
  pairing_clear(cpu);
  return bad ? 1 : 0;
}
