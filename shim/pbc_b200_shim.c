/* pbc_b200_shim.c -- the pbc.h surface over the GPU engine: host code in C.
 *
 * Built against the reference's own public headers (include/pbc.h, where they lie under the
 * reference tree -- nothing is copied) and linked with the reference library, this file puts
 * libpbc_b200.so behind the reference's plugin seam for the pairing hot path and nothing else:
 *
 *   pairing_init_set_buf / pairing_init_set_str   (ecc/pairing.c:88-102) -- interposed: run the
 *       reference initialisation (pbc_param_init_set_buf + pairing_init_pbc_param), then create a
 *       GPU handle from the same parameter text and re-point the vtable slots the hot path goes
 *       through (include/pbc_pairing.h:17-44):
 *         pairing->map            <- b200_map            (element_pairing / pairing_apply, :118-145)
 *         pairing->prod_pairings  <- b200_prod_pairings  (element_prod_pairing, :153-171)
 *         pairing->pp_init/apply/clear <- b200_pp_*      (pairing_pp_*, :54-89)
 *         pairing->clear_func     <- b200_clear          (releases the GPU handle, then the original)
 *       Everything else (element_t arithmetic, G1/G2/GT/Zr fields, finalpow, phi, I/O, RNG) stays
 *       the reference's.  A caller such as benchmark/benchmark.c compiles and links unchanged.
 *   pbc_b200_pairing_batch / pbc_b200_prod_pairing_batch -- the additive batch entry points
 *       (SURVEY 8b): n pairings in one call, reference wire format in and out.
 *   pbc_b200_prod_pairing_batch_v -- products with a pair count per output (offsets, host memory).
 *   element_pairing_batch -- the same over arrays of element_t.
 *
 * Elements cross the boundary as the bytes element_to_bytes() writes (include/pbc_field.h:475-484),
 * so the GPU result lands in the caller's element_t through element_from_bytes() and is
 * bit-identical to what the reference's own map() would have left there.
 *
 * There is no CPU fallback: if the GPU call fails the shim reports through pbc_die (the
 * reference's fatal-error convention, misc/utils.c:70-77).
 */
#include <pthread.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <pbc.h>

#include "../include/pbc_b200.h"

#define MAX_ATTACHED 64

struct attach_s {
  pairing_ptr pairing;
  pbc_b200_pairing_t *h;
  void (*orig_clear)(struct pairing_s *);
  int g1_len, g2_len, gt_len;
};
static struct attach_s g_attached[MAX_ATTACHED];
/* the table is shared by every pairing_t of the process: attach, detach and look-up take this lock
 * (the reference itself is used from one thread per pairing_t, SURVEY 8b; different pairings may
 * live on different threads) */
static pthread_mutex_t g_attach_mu = PTHREAD_MUTEX_INITIALIZER;

static struct attach_s *find_attach(pairing_ptr p) {
  int i;
  struct attach_s *a = NULL;
  pthread_mutex_lock(&g_attach_mu);
  for (i = 0; i < MAX_ATTACHED && !a; i++)
    if (g_attached[i].pairing == p) a = &g_attached[i];
  pthread_mutex_unlock(&g_attach_mu);
  if (!a) pbc_die("pbc_b200: pairing %p is not attached to a GPU handle", (void *)p);
  return a;
}

static void check(int rc, const char *what) {
  if (rc) pbc_die("pbc_b200: %s failed: %s", what, pbc_b200_last_error());
}

/* pairing->map: `out` is the inner F_q^k element (include/pbc_pairing.h:131-134) */
static void b200_map(element_ptr out, element_ptr in1, element_ptr in2, pairing_ptr pairing) {
  struct attach_s *a = find_attach(pairing);
  unsigned char buf[1024];
  unsigned char *b1 = buf, *b2 = b1 + a->g1_len, *bo = b2 + a->g2_len;
  element_to_bytes(b1, in1);
  element_to_bytes(b2, in2);
  check(pbc_b200_pairings_apply(a->h, bo, b1, b2, 1), "element_pairing");
  element_from_bytes(out, bo);
}

/* pairing->prod_pairings (include/pbc_pairing.h:153-171; infinite inputs were filtered by the caller) */
static void b200_prod_pairings(element_ptr out, element_t in1[], element_t in2[], int n_prod,
                               pairing_ptr pairing) {
  struct attach_s *a = find_attach(pairing);
  unsigned char *b1 = pbc_malloc((size_t)n_prod * (a->g1_len + a->g2_len) + a->gt_len);
  unsigned char *b2 = b1 + (size_t)n_prod * a->g1_len, *bo = b2 + (size_t)n_prod * a->g2_len;
  int i;
  for (i = 0; i < n_prod; i++) {
    element_to_bytes(b1 + (size_t)i * a->g1_len, in1[i]);
    element_to_bytes(b2 + (size_t)i * a->g2_len, in2[i]);
  }
  check(pbc_b200_prod_pairings_apply(a->h, bo, b1, b2, (size_t)n_prod, 1), "element_prod_pairing");
  element_from_bytes(out, bo);
  pbc_free(b1);
}

/* pairing_pp_init / apply / clear (include/pbc_pairing.h:54-89): p->data is the engine's
 * pbc_b200_pp_t -- the preprocessing (types a, a1: the line-coefficient table) is computed once here
 * and stays in device memory until pairing_pp_clear, as the reference keeps its table in p->data
 * (ecc/a_param.c:149-220) */
static void b200_pp_init(pairing_pp_t p, element_ptr in1, pairing_ptr pairing) {
  struct attach_s *a = find_attach(pairing);
  unsigned char buf[1024];
  pbc_b200_pp_t *pp = NULL;
  element_to_bytes(buf, in1);
  check(pbc_b200_pp_init(a->h, &pp, buf), "pairing_pp_init");
  p->data = pp;
}
static void b200_pp_apply(element_ptr out, element_ptr in2, pairing_pp_t p) {
  struct attach_s *a = find_attach(p->pairing);
  unsigned char buf[1024];
  unsigned char *b2 = buf, *bo = b2 + a->g2_len;
  element_to_bytes(b2, in2);
  check(pbc_b200_pp_apply((pbc_b200_pp_t *)p->data, bo, b2, 1), "pairing_pp_apply");
  element_from_bytes(out, bo);
}
static void b200_pp_clear(pairing_pp_t p) { pbc_b200_pp_clear((pbc_b200_pp_t *)p->data); }

static void b200_clear(pairing_ptr pairing) {
  struct attach_s *a = find_attach(pairing);
  void (*orig)(struct pairing_s *) = a->orig_clear;
  pbc_b200_pairing_clear(a->h);
  pthread_mutex_lock(&g_attach_mu);
  memset(a, 0, sizeof *a);
  pthread_mutex_unlock(&g_attach_mu);
  orig(pairing);
}

/* Attach a GPU handle to an initialised pairing_t.  Returns 0 on success, 1 on failure (the
 * reference's init convention); on failure the pairing is left as the reference set it up. */
int pbc_b200_attach(pairing_t pairing, const char *param, size_t len) {
  int i;
  struct attach_s *a = NULL, t;
  memset(&t, 0, sizeof t);
  if (!len) len = strlen(param);
  if (pbc_b200_pairing_init_set_buf(&t.h, param, len)) {
    pbc_error("pbc_b200: %s", pbc_b200_last_error());
    return 1;
  }
  t.g1_len = pbc_b200_pairing_length_in_bytes_G1(t.h);
  t.g2_len = pbc_b200_pairing_length_in_bytes_G2(t.h);
  t.gt_len = pbc_b200_pairing_length_in_bytes_GT(t.h);
  if (t.g1_len != pairing_length_in_bytes_G1(pairing) || t.g2_len != pairing_length_in_bytes_G2(pairing) ||
      t.gt_len != pairing_length_in_bytes_GT(pairing) || t.g1_len + t.g2_len + t.gt_len > 1024) {
    pbc_b200_pairing_clear(t.h);
    pbc_error("pbc_b200: element sizes disagree with the reference");
    return 1;
  }
  t.pairing = pairing;
  t.orig_clear = pairing->clear_func;
  pthread_mutex_lock(&g_attach_mu);
  for (i = 0; i < MAX_ATTACHED && !a; i++)
    if (!g_attached[i].pairing) a = &g_attached[i];
  if (a) *a = t;
  pthread_mutex_unlock(&g_attach_mu);
  if (!a) {
    pbc_b200_pairing_clear(t.h);
    pbc_error("pbc_b200: too many attached pairings");
    return 1;
  }
  pairing->map = b200_map;
  pairing->prod_pairings = b200_prod_pairings;
  pairing->pp_init = b200_pp_init;
  pairing->pp_apply = b200_pp_apply;
  pairing->pp_clear = b200_pp_clear;
  pairing->clear_func = b200_clear;
  return 0;
}

/* ecc/pairing.c:88-102, interposed (this library precedes the reference library at link time) */
int pairing_init_set_buf(pairing_t pairing, const char *input, size_t len) {
  pbc_param_t par;
  if (pbc_param_init_set_buf(par, input, len)) {
    pbc_error("error initializing pairing");
    return 1;
  }
  pairing_init_pbc_param(pairing, par);
  pbc_param_clear(par);
  if (pbc_b200_attach(pairing, input, len)) {
    pairing_clear(pairing);
    return 1;
  }
  return 0;
}
int pairing_init_set_str(pairing_t pairing, const char *s) { return pairing_init_set_buf(pairing, s, 0); }

/* ---- additive batch entry points (SURVEY 8b) ---------------------------------------------- */
int pbc_b200_pairing_batch(pairing_t pairing, unsigned char *out, const unsigned char *in1,
                           const unsigned char *in2, size_t n) {
  return pbc_b200_pairings_apply(find_attach(pairing)->h, out, in1, in2, n);
}
int pbc_b200_prod_pairing_batch(pairing_t pairing, unsigned char *out, const unsigned char *in1,
                                const unsigned char *in2, int n_prod, size_t n_out) {
  return pbc_b200_prod_pairings_apply(find_attach(pairing)->h, out, in1, in2, (size_t)n_prod, n_out);
}
/* out[i] = prod_{offsets[i] <= j < offsets[i+1]} e(in1[j], in2[j]): one GPU call for products of
 * different lengths (include/pbc_b200.h, pbc_b200_prod_pairings_apply_v) */
int pbc_b200_prod_pairing_batch_v(pairing_t pairing, unsigned char *out, const unsigned char *in1,
                                  const unsigned char *in2, const size_t *offsets, size_t n_out) {
  return pbc_b200_prod_pairings_apply_v(find_attach(pairing)->h, out, in1, in2, offsets, n_out);
}

/* out[i] = e(in1[i], in2[i]) for arrays of element_t: one GPU batch instead of n element_pairing
 * calls.  Infinite inputs give the identity, as pairing_apply does (include/pbc_pairing.h:123-130). */
void element_pairing_batch(element_t out[], element_t in1[], element_t in2[], int n) {
  if (n <= 0) return;
  pairing_ptr pairing = out[0]->field->pairing;
  struct attach_s *a = find_attach(pairing);
  size_t per = (size_t)a->g1_len + a->g2_len + a->gt_len;
  unsigned char *b1 = pbc_malloc(per * (size_t)n);
  unsigned char *b2 = b1 + (size_t)n * a->g1_len, *bo = b2 + (size_t)n * a->g2_len;
  int i;
  memset(b1, 0, per * (size_t)n);          /* slots of infinite inputs: result ignored below */
  for (i = 0; i < n; i++) {
    if (element_is0(in1[i]) || element_is0(in2[i])) continue;
    element_to_bytes(b1 + (size_t)i * a->g1_len, in1[i]);
    element_to_bytes(b2 + (size_t)i * a->g2_len, in2[i]);
  }
  check(pbc_b200_pairings_apply(a->h, bo, b1, b2, (size_t)n), "element_pairing_batch");
  for (i = 0; i < n; i++) {
    if (element_is0(in1[i]) || element_is0(in2[i])) element_set0(out[i]);
    else element_from_bytes((element_ptr)out[i]->data, bo + (size_t)i * a->gt_len);
  }
  pbc_free(b1);
}

/* out[i] = in[i]^k[i] (element_pow_zn, include/pbc_field.h:262-275) for arrays of G1 or GT elements
 * of an attached pairing: one GPU batch instead of n windowed powers on the CPU.  k[i] in Zr. */
void element_pow_zn_batch(element_t out[], element_t in[], element_t k[], int n) {
  if (n <= 0) return;
  pairing_ptr pairing = in[0]->field->pairing;
  struct attach_s *a = find_attach(pairing);
  int is_gt = in[0]->field == pairing->GT;
  if (!is_gt && in[0]->field != pairing->G1) pbc_die("pbc_b200: element_pow_zn_batch takes G1 or GT elements");
  size_t elen = is_gt ? a->gt_len : a->g1_len, zlen = pbc_b200_pairing_length_in_bytes_Zr(a->h);
  unsigned char *bi = pbc_malloc((2 * elen + zlen) * (size_t)n);
  unsigned char *bo = bi + (size_t)n * elen, *bk = bo + (size_t)n * elen;
  int i;
  memset(bi, 0, (2 * elen + zlen) * (size_t)n);
  for (i = 0; i < n; i++) {
    if (!element_is0(in[i])) element_to_bytes(bi + (size_t)i * elen, in[i]);
    element_to_bytes(bk + (size_t)i * zlen, k[i]);
  }
  check((is_gt ? pbc_b200_gt_pow_zn : pbc_b200_g1_pow_zn)(a->h, bo, bi, bk, (size_t)n), "element_pow_zn_batch");
  for (i = 0; i < n; i++) {
    if (element_is0(in[i]) || element_is0(k[i])) { element_set0(out[i]); continue; }
    element_from_bytes(out[i], bo + (size_t)i * elen);
  }
  pbc_free(bi);
}

/* out[i] = element_from_hash(out[i], data + i*len, len) (include/pbc_field.h:202-212 -> curve_from_hash,
 * ecc/curve.c:455-482) for arrays of G1 or G2 elements of an attached pairing: one GPU batch of n hashes
 * of len bytes each, back to back.  A G1 hash whose cofactor multiple is the point at infinity comes back
 * as zero bytes and is set to the identity. */
void element_from_hash_batch(element_t out[], const void *data, int len, int n) {
  if (n <= 0) return;
  pairing_ptr pairing = out[0]->field->pairing;
  struct attach_s *a = find_attach(pairing);
  int is_g1 = out[0]->field == pairing->G1;
  if (!is_g1 && out[0]->field != pairing->G2) pbc_die("pbc_b200: element_from_hash_batch takes G1 or G2 elements");
  if (len <= 0) pbc_die("pbc_b200: element_from_hash_batch needs len > 0");
  size_t elen = is_g1 ? a->g1_len : a->g2_len, k;
  unsigned char *bo = pbc_malloc(elen * (size_t)n);
  int i;
  check((is_g1 ? pbc_b200_g1_from_hash : pbc_b200_g2_from_hash)(a->h, bo, data, (size_t)len, (size_t)n),
        "element_from_hash_batch");
  for (i = 0; i < n; i++) {
    const unsigned char *e = bo + (size_t)i * elen;
    for (k = 0; k < elen && !e[k]; k++) {}
    if (k == elen) element_set0(out[i]);
    else element_from_bytes(out[i], (unsigned char *)e);
  }
  pbc_free(bo);
}
