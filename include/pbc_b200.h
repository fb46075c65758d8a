/* pbc_b200.h -- C ABI of the batched pairing engine for the H100 (libpbc_b200.so).
 *
 * This is the drop-in boundary for the pairing hot path of the PBC library: each entry point
 * below names the reference interface it stands in for (file:line under the reference tree).
 * Plain pointers and sizes only.  All element buffers use the reference *wire format*, i.e. the
 * bytes element_to_bytes() writes and element_from_bytes() reads (include/pbc_field.h:475-484):
 *
 *   type A  (param/a.param)     G1 128 B   G2 128 B   GT 128 B     x || y, 64-byte big-endian F_q
 *   type F  (param/f.param)     G1  40 B   G2  80 B   GT 240 B     20-byte big-endian F_q
 *   type D  (param/d159.param)  G1  40 B   G2 120 B   GT 120 B     20-byte big-endian F_q
 *   type D, 160..255-bit q      G1 2wb     G2 6wb     GT 6wb       wb = ceil(bits(q)/8) = 22..32-byte F_q;
 *                                                                  Zr ceil(bits(r)/8), r below 2^255:
 *     d277699-175-167.param     G1  44 B   G2 132 B   GT 132 B     Zr 21 B
 *     d278027-190-181.param     G1  48 B   G2 144 B   GT 144 B     Zr 23 B
 *     d105171-196-185.param     G1  50 B   G2 150 B   GT 150 B     Zr 24 B
 *     d201.param                G1  52 B   G2 156 B   GT 156 B     Zr 23 B
 *     d224.param                G1  56 B   G2 168 B   GT 168 B     Zr 28 B
 *     (type D q of 153..159 bits runs five-limb kernels, 160..255 bits eight-limb ones; other q are
 *     rejected at init)
 *   type G  (param/g149.param)  G1  38 B   G2 190 B   GT 190 B     19-byte big-endian F_q
 *   type A1 (param/a1.param)    G1 260 B   G2 260 B   GT 260 B     ceil(bits(p)/8) = 130-byte F_p; any
 *                                                                  p = l n - 1 below 2^1087 is accepted
 *   type E  (param/e.param)     G1 256 B   G2 256 B   GT 128 B     wb = ceil(bits(q)/8) = 128-byte F_q, Zr 20 B;
 *                                                                  G1 = G2 = 2wb, GT = wb (k = 1, GT in F_q^*):
 *                                                                  any q below 2^1087 with
 *                                                                  r = 2^exp2 + sign1 2^exp1 + sign0 dividing q - 1
 *
 * Semantics that are reproduced exactly:
 *   - bytes that do not decode to a point on the curve are the point at infinity
 *     (curve_from_bytes, ecc/curve.c:611-623);
 *   - e(O, Q) = e(P, O) = 1 (pairing_apply, include/pbc_pairing.h:118-135); in a product of
 *     pairings ANY infinite input makes the whole product 1 (element_prod_pairing, :153-171);
 *   - powers in G1 and G2 are the exact k P (k reduced mod r, mod n for type a1) for any point P on
 *     the curve, including points of small order and type a1's subgroup elements of order p1 or p2;
 *   - every output is bit-identical to the reference CPU path, including first and second arguments
 *     of small order (points of E(F_q) outside G1, twist points outside G2), second arguments drawn
 *     on the twist without cofactor multiplication, and twist points with y = 0 (types d, g: x a
 *     root of x^3 + a x + b) -- wherever the reference's own computation does not divide by zero.
 * One input is DEFINED here rather than copied: a first or second argument with y = 0 (type a, a1: the
 * 2-torsion point (0, 0); types d, g: a 2-torsion point of E(F_q) if the cofactor is even) lies on the
 * curve but outside the order-r groups and has no tangent line; the reference's projective doubling
 * inverts Z = 0 there and returns a by-product of that.  This library decodes such a point as the
 * point at infinity: the pairing is 1 (tests/test_gpu_edge_cases.py).
 * The other inputs on which the reference divides by zero (tests/test_gpu_small_order_pairings.py):
 *   - type a, a first argument of small order whose walk reaches O (the reference inverts Z = 0 in
 *     point_to_affine and goes on from the by-product) or whose last chord joins V to itself (the
 *     Miller value is 0 and the final exponentiation inverts it): the pairing is 1, and a product of
 *     pairings containing such a pair is 1, as for a Miller value with f0 f1 = 0;
 *   - type g, a pair whose Miller value lies in F_q^5 (a twist point of small order as the second
 *     argument, for one): the reference's Lucas step divides by P^2 - 4 = 0 and exits; the pairing is
 *     1, its exact value, and in a product the pair contributes 1;
 *   - types f, d, g, a first argument of small order whose walk reaches O: the reference's affine walk
 *     goes on from the stale coordinates of O and its final exponentiation inverts 0 and exits.  Here
 *     the next addition of +-P turns the Jacobian O into (0, 0, 0), after which every line is 0 (or a
 *     chord joins V to itself, which is 0 as well), so the Miller value is 0 and the output is the
 *     ZERO of F_q^k (all-zero bytes), which is not an element of GT: for the
 *     pairing, for pp one-shot and through a handle, and for every product holding such a pair (unless
 *     another input of that product is O, which makes it 1).  A caller that needs a GT element must
 *     keep such points out, e.g. by checking r P = O.
 * Type E (k = 1): e(P, Q) is bit-exact for P and Q in G1 (points of order r).  The Miller loop
 * evaluates at Q + R and at R, R a point outside E[r] that the library fixes at init
 * (pbc_b200_derived_constant "R", x then y); the reference draws its R at random per pairing_init.
 * For P in G1 the result does not depend on R, for other P it does, so neither library defines the
 * value for a first argument outside G1.  A second argument on the curve but outside G1 is bit-exact
 * too, except Q = R and every Q with Q + R in the group generated by P (Q = -R among them): there a
 * line of the loop vanishes at Q + R, or Q + R is O, and the value is unspecified.  Such Q can only be
 * built from the published R; no Q in G1 is one of them, since R is not in E[r].  Type E has no
 * element_from_hash and no compressed points here: those calls fail with a message.
 * There is no CPU fallback: without a CUDA device every compute entry point fails.
 *
 * Threading: like the reference (which is not thread-safe, SURVEY 8b) a handle is used by one thread
 * at a time; calls on DIFFERENT handles may come from different threads -- the blocking host-buffer
 * entry points serialise per device (the curve constants of one handle at a time are resident in
 * __constant__ memory).  With the asynchronous _device entry points keep one handle active per
 * device until its stream has drained.  The _device entry points of ONE handle share a per-device
 * workspace; the library orders its users with an event (each enqueue records it, the next enqueue's
 * stream waits for it), so calls of one handle on different streams serialise on the workspace
 * rather than overlap.
 *
 * Return convention: 0 on success, non-zero on failure (pairing_init_set_buf returns 1 on
 * failure, ecc/pairing.c:88-98); pbc_b200_last_error() gives the message the reference would
 * have sent to pbc_error().
 */
#ifndef PBC_B200_H
#define PBC_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct pbc_b200_pairing_s pbc_b200_pairing_t;

/* pairing_init_set_buf / pairing_init_set_str (ecc/pairing.c:88-102): parse "key value" parameter
 * text (ecc/param.c:42-111), derive the field constants (arith/montfp.c:533-600,
 * ecc/a_param.c:1431-1472 and :2230-2273, ecc/f_param.c:335-447, ecc/d_param.c:993-1095,
 * ecc/g_param.c:1258) and upload them.  Types a, a1, e, f, d (k = 6) and g are accepted.  Does not touch the GPU until the first compute call. */
int pbc_b200_pairing_init_set_buf(pbc_b200_pairing_t **out, const char *param, size_t len);
int pbc_b200_pairing_init_set_str(pbc_b200_pairing_t **out, const char *param);

/* pairing_clear (include/pbc_pairing.h:109-116) */
void pbc_b200_pairing_clear(pbc_b200_pairing_t *p);

/* pairing_length_in_bytes_G1 / _G2 / _GT (include/pbc_pairing.h:200-250); type letter 'a', 'e', 'f', 'd', 'g'; '1' for a1 */
int pbc_b200_pairing_length_in_bytes_G1(const pbc_b200_pairing_t *p);
int pbc_b200_pairing_length_in_bytes_G2(const pbc_b200_pairing_t *p);
int pbc_b200_pairing_length_in_bytes_GT(const pbc_b200_pairing_t *p);
int pbc_b200_pairing_type(const pbc_b200_pairing_t *p);

/* Batched element_pairing (include/pbc_pairing.h:141-145 -> pairing->map, ecc/a_param.c:1053,
 * ecc/f_param.c:289, ecc/d_param.c:570):  out[i] = e(in1[i], in2[i]),  i < n.
 * HOST buffers (pinned memory makes the copies asynchronous; pageable works).  The batch is cut
 * into contiguous slices, one per configured device (pbc_b200_set_devices), each slice is
 * streamed through its GPU in chunks; results land in `out` at the slice offset. */
int pbc_b200_pairings_apply(pbc_b200_pairing_t *p, unsigned char *out, const unsigned char *in1,
                            const unsigned char *in2, size_t n);

/* Same with DEVICE buffers on the current CUDA device, enqueued on `stream` (a cudaStream_t
 * passed as void*; NULL = default stream).  Asynchronous: returns after enqueueing.  Buffers
 * must be 4-byte aligned.  The workspace grows to the largest n seen (512 B per pairing). */
int pbc_b200_pairings_apply_device(pbc_b200_pairing_t *p, void *d_out, const void *d_in1,
                                   const void *d_in2, size_t n, void *stream);

/* Batched element_prod_pairing (include/pbc_pairing.h:153-171 -> pairing->prod_pairings,
 * ecc/a_param.c:1283-1383, ecc/d_param.c:710-736, ecc/pairing.c:35-46 for type F):
 *   out[i] = prod_{j<k} e(in1[i*k+j], in2[i*k+j]),  i < n_out.   One shared final
 * exponentiation per output. */
int pbc_b200_prod_pairings_apply(pbc_b200_pairing_t *p, unsigned char *out,
                                 const unsigned char *in1, const unsigned char *in2, size_t k,
                                 size_t n_out);
int pbc_b200_prod_pairings_apply_device(pbc_b200_pairing_t *p, void *d_out, const void *d_in1,
                                        const void *d_in2, size_t k, size_t n_out, void *stream);

/* Batched element_prod_pairing with a pair count per output (ragged batches, e.g. aggregate
 * signatures over different numbers of messages):
 *   out[i] = prod_{offsets[i] <= j < offsets[i+1]} e(in1[j], in2[j]),   i < n_out.
 * Each output is byte-identical to pbc_b200_prod_pairings_apply(k = its length, n_out = 1) on its
 * pairs, with the same rules (an O or off-curve input makes that output 1, and only that output).
 * offsets: n_out + 1 entries in HOST memory for both forms, offsets[0] = 0, strictly increasing (an
 * empty product is rejected, as k = 0 is above); the library has read them by the time the call
 * returns.  NULL offsets, offsets[0] != 0, a non-increasing entry (the message names its index) and a
 * byte count that overflows size_t fail before any CUDA call; n_out = 0 returns 0 and touches nothing.
 * Every pair runs its own Miller loop; the Miller values of each output are multiplied in passes of at
 * most 16 consecutive values per thread, so one long product costs log16(length) passes, not one
 * thread's serial loop.  The host form cuts the batch into chunks of whole outputs (multi-GPU: slices
 * of whole outputs balanced by pairs); the device form is asynchronous on `stream`, its workspace grows
 * to the largest call. */
int pbc_b200_prod_pairings_apply_v(pbc_b200_pairing_t *p, unsigned char *out, const unsigned char *in1,
                                   const unsigned char *in2, const size_t *offsets, size_t n_out);
int pbc_b200_prod_pairings_apply_v_device(pbc_b200_pairing_t *p, void *d_out, const void *d_in1,
                                          const void *d_in2, const size_t *offsets, size_t n_out, void *stream);

/* Batched pairing_pp_init + pairing_pp_apply (include/pbc_pairing.h:54-89,
 * ecc/a_param.c:149-220,317-360): one fixed first argument, n second arguments.
 *   out[i] = e(in1, in2[i]). */
int pbc_b200_pp_pairings_apply(pbc_b200_pairing_t *p, unsigned char *out, const unsigned char *in1,
                               const unsigned char *in2, size_t n);
int pbc_b200_pp_pairings_apply_device(pbc_b200_pairing_t *p, void *d_out, const void *d_in1,
                                      const void *d_in2, size_t n, void *stream);

/* pairing_pp_init / pairing_pp_apply / pairing_pp_clear (include/pbc_pairing.h:54-89 ->
 * a_pairing_pp_init/apply/clear ecc/a_param.c:149-220 and :317-360, a1: :1632-1818,
 * d_pairing_pp_* ecc/d_param.c:794-991): the preprocessing of one fixed first argument is done ONCE,
 * kept in device memory by the handle, and reused by every apply until clear -- what pairing_pp_t
 * is for.  Types a and a1 keep the table of line coefficients (160 / about 1 500 rows; an apply then
 * costs 7 instead of 17-19 multiplications per step); types f, d and g keep the decoded point.
 * The handle lives on the device that was current at init; apply switches to it.  As in the reference
 * (a pairing_pp_t points into its pairing_t), clear the pp handle before the pairing it belongs to. */
typedef struct pbc_b200_pp_s pbc_b200_pp_t;
int pbc_b200_pp_init(pbc_b200_pairing_t *p, pbc_b200_pp_t **pp, const unsigned char *in1);
int pbc_b200_pp_apply(pbc_b200_pp_t *pp, unsigned char *out, const unsigned char *in2, size_t n);
int pbc_b200_pp_apply_device(pbc_b200_pp_t *pp, void *d_out, const void *d_in2, size_t n, void *stream);
void pbc_b200_pp_clear(pbc_b200_pp_t *pp);

/* ---- the operations either side of the pairing (SURVEY 8f ranks 2 and 3) ---------------------
 * Batched element_pow_zn (include/pbc_field.h:262-275 -> arith/field.c:113-126):
 *   g1_pow_zn:  out[i] = k[i] * in[i]   in G1 (ecc/curve.c:455-482)
 *   g2_pow_zn:  the same in G2: the twist over F_q^2 (type f, ecc/f_param.c:367-378) or F_q^3
 *               (type d, ecc/d_param.c:1060-1070); type a: G2 = G1
 *   gt_pow_zn:  out[i] = in[i] ^ k[i]   in GT (ecc/pairing.c:199-231)
 * Elements in wire format; scalars are Zr wire bytes (pbc_b200_pairing_length_in_bytes_Zr = 20,
 * big-endian, reduced mod r as element_from_bytes does).  The point at infinity (k = 0 mod r, or an
 * input that is not on the curve) is written as all-zero bytes: the reference leaves stale
 * coordinates behind its infinity flag (ecc/curve.c:603-609), so there is nothing to match.
 * The _device forms take device pointers and enqueue on `stream`. */
int pbc_b200_pairing_length_in_bytes_Zr(const pbc_b200_pairing_t *p);
int pbc_b200_g1_pow_zn(pbc_b200_pairing_t *p, unsigned char *out, const unsigned char *in,
                       const unsigned char *k, size_t n);
int pbc_b200_gt_pow_zn(pbc_b200_pairing_t *p, unsigned char *out, const unsigned char *in,
                       const unsigned char *k, size_t n);
int pbc_b200_g2_pow_zn(pbc_b200_pairing_t *p, unsigned char *out, const unsigned char *in,
                       const unsigned char *k, size_t n);
int pbc_b200_g2_pow_zn_device(pbc_b200_pairing_t *p, void *d_out, const void *d_in, const void *d_k,
                              size_t n, void *stream);
int pbc_b200_g1_pow_zn_device(pbc_b200_pairing_t *p, void *d_out, const void *d_in, const void *d_k,
                              size_t n, void *stream);
int pbc_b200_gt_pow_zn_device(pbc_b200_pairing_t *p, void *d_out, const void *d_in, const void *d_k,
                              size_t n, void *stream);

/* The GT operations next to the pairing (SURVEY 8f rank 3), batched, host buffers:
 *   gt_mul:  out[i] = a[i] * b[i]      element_mul on GT (ecc/pairing.c:199-201 -> the F_q^k product:
 *            fi_mul arith/fieldquadratic.c:425-457 for types a / a1, polymod_mul arith/poly.c:932-1143 over
 *            fq_mul for f, the quadratic extensions of d / g)
 *   gt_cmp:  flags[i] = 1 if a[i] != b[i], else 0      element_cmp (include/pbc_field.h:334-339)
 *   is_almost_coddh (include/pbc_pairing.h:240-243 -> generic_is_almost_coddh ecc/pairing.c:15-33 for
 *            types a, a1, f; cc_is_almost_coddh ecc/d_param.c:739-784, ecc/g_param.c:560):
 *            flags[i] = 1 if e(a[i], d[i]) == e(b[i], c[i]) or e(a[i], d[i]) * e(b[i], c[i]) == 1, else 0;
 *            a, b in G1 and c, d in G2 (wire format).  Two batched pairings, one GT product, one compare. */
int pbc_b200_gt_mul(pbc_b200_pairing_t *p, unsigned char *out, const unsigned char *a,
                    const unsigned char *b, size_t n);
int pbc_b200_gt_cmp(pbc_b200_pairing_t *p, unsigned char *flags, const unsigned char *a,
                    const unsigned char *b, size_t n);
int pbc_b200_is_almost_coddh(pbc_b200_pairing_t *p, unsigned char *flags, const unsigned char *a,
                             const unsigned char *b, const unsigned char *c, const unsigned char *d,
                             size_t n);

/* Batched element_from_hash on G1 (include/pbc_field.h:202-212 -> curve_from_hash,
 * ecc/curve.c:455-482 with pbc_mpz_from_hash, arith/field.c:643-668): out[i] = the G1 element the
 * reference derives from the `len` bytes at data + i*len -- x from the hash, x <- x^2 + 1 until
 * x^3 + ax + b is a square, the odd square root, times the cofactor of G1.  Needs q = 3 mod 4 or
 * q = 5 mod 8 (a.param, f.param, d159.param all qualify); type D with 160..255-bit q takes any q
 * (Tonelli-Shanks where q = 1 mod 8: the four bundled sets other than d201).  Where the cofactor multiple
 * is the point at infinity (the point's order divides the cofactor: x = 1 on type a, for one) the
 * output is all-zero bytes, as for powers: the reference leaves stale coordinates there. */
int pbc_b200_g1_from_hash(pbc_b200_pairing_t *p, unsigned char *out, const unsigned char *data,
                          size_t len, size_t n);
int pbc_b200_g1_from_hash_device(pbc_b200_pairing_t *p, void *d_out, const void *d_data, size_t len,
                                 size_t n, void *stream);

/* Batched element_from_bytes_compressed on G1 (ecc/curve.c:762-813): each input is the x
 * coordinate in wire format followed by one byte, 1 when y is odd (fp_sgn_odd); output is the full
 * wire element x || y.  An x with no point on the curve gives zero bytes.  (Compression itself is
 * x plus the parity of y and needs no GPU; pbc_b200/pairing.py has it.) */
int pbc_b200_pairing_length_in_bytes_compressed_G1(const pbc_b200_pairing_t *p);
int pbc_b200_g1_from_bytes_compressed(pbc_b200_pairing_t *p, unsigned char *out, const unsigned char *in,
                                      size_t n);

/* Batched element_from_hash on G2 (curve_from_hash, ecc/curve.c:455-482, on the twist): out[i] = the
 * G2 element the reference derives from the `len` bytes at data + i*len.  The twist's field K sets x:
 * type f (K = F_q^2, fq_from_hash arith/fieldquadratic.c:311-316) hashes x0 from the first len/2 bytes
 * and x1 from the rest; types d and g (K = F_q^3, F_q^5, polymod_from_hash arith/poly.c:341-348) give
 * every coefficient the hash of the whole data.  Then x <- x^2 + 1 until x^3 + a'x + b' is a square of K
 * (zero counts as one in F_q^2, not in F_q^3 / F_q^5, as fq_is_sqr and polymod_is_sqr decide), y its
 * root with element_sign(y) >= 0 (fq_sign / polymod_sgn on the reference basis).  The twist has no
 * cofactor (ecc/f_param.c:383, ecc/d_param.c:1057, ecc/g_param.c:1319): the point found is the output
 * and usually lies outside the order-r subgroup, as in the reference.  Type f needs q = 3 mod 4; types d
 * and g take any q.  Types a and a1: G2 = G1, the calls give the bytes of pbc_b200_g1_from_hash.  Type e
 * fails with a message.  len is 1..2^20. */
int pbc_b200_g2_from_hash(pbc_b200_pairing_t *p, unsigned char *out, const unsigned char *data,
                          size_t len, size_t n);
int pbc_b200_g2_from_hash_device(pbc_b200_pairing_t *p, void *d_out, const void *d_data, size_t len,
                                 size_t n, void *stream);

/* Batched element_from_bytes_compressed on G2 (ecc/curve.c:762-813): each input is x in wire format
 * (pbc_b200_pairing_length_in_bytes_compressed_G2 - 1 bytes: 40 for f, 60 for d159, 95 for g149, 3 wb
 * for type d with wb-byte coordinates) followed by one byte; a non-zero byte selects the root y with
 * element_sign(y) > 0, zero the other one.  Coordinates >= q are reduced mod q, as element_from_bytes
 * does.  x^3 + a'x + b' = 0 gives (x, 0); an x with no point on the twist gives zero bytes.  Compression
 * is x || (1 if element_sign(y) > 0 else 0) and needs no GPU; pbc_b200/pairing.py has it.  Types a and a1
 * as G1, type e fails. */
int pbc_b200_pairing_length_in_bytes_compressed_G2(const pbc_b200_pairing_t *p);
int pbc_b200_g2_from_bytes_compressed(pbc_b200_pairing_t *p, unsigned char *out, const unsigned char *in,
                                      size_t n);

/* Multi-GPU fan-out for the host-buffer entry points: use devices [0, count).  count = 0 means
 * every visible device.  Default is 1 (the current device). */
int pbc_b200_set_devices(pbc_b200_pairing_t *p, int count);

/* Pinned host memory helpers (cudaHostAlloc / cudaFreeHost) so C callers can stage batches. */
void *pbc_b200_host_alloc(size_t bytes);
void pbc_b200_host_free(void *ptr);

/* Number of kernels this library has launched since it was loaded (bench.py: gpu_launches). */
uint64_t pbc_b200_kernel_launches(void);

/* Message of the last failure on this thread (pbc_error text, misc/utils.c:79-101). */
const char *pbc_b200_last_error(void);

/* ---- integer-pipe roofline probes (SURVEY 8d; bench.py) -------------------------------------
 * All return elapsed milliseconds (CUDA events on the launching stream) or a negative value.
 *   fpmul: every thread runs `iters` dependent Montgomery multiplications modulo this pairing's
 *          base-field prime; mode 0 = operand-scanning multiplier in registers, 1 = the multiplier
 *          the kernels use, through the shared-memory slot machine, 2 = product-scanning
 *          multiplier in registers, 3 = the squaring the kernels use, in registers, 6 (type a) = that
 *          squaring through the slot machine, 7 (type a) = the lazy two-product routine of the Miller
 *          step through the slot machine (two products, one reduction: about 1.5 multiplications'
 *          work).  muls = threads * iters.
 *   imad : IMAD.WIDE.U32 issue-rate probe, 32 * iters instructions per thread: the faster of two
 *          kernels, four independent carry chains of eight and eight carry-free chains of four
 *          (data-dependent multiplicands in both).
 *   fpmul_smem (type a): fpmul mode 1 with smem_bytes of dynamic shared memory per 128-thread block
 *          (at least the 16 KB it uses), so that it runs at the occupancy of a kernel with that
 *          footprint.  One full wave: *blocks_per_sm (the device's occupancy for that size) times the
 *          multiprocessor count blocks.  muls = blocks * 128 * iters. */
double pbc_b200_bench_fpmul(pbc_b200_pairing_t *p, int mode, int blocks, int iters, int reps);
double pbc_b200_bench_fpmul_smem(pbc_b200_pairing_t *p, int smem_bytes, int iters, int reps, int *blocks_per_sm);
double pbc_b200_bench_imad(int blocks, int threads, int iters, int reps);

/* Per-stage device timing of the device-buffer path (bench.py roofline): when enabled,
 * pbc_b200_pairings_apply_device records CUDA events on the launching stream around its three
 * kernels; after synchronising, pbc_b200_stage_times returns their durations in milliseconds
 * {main kernel (Miller loop), batch inversion, final exponentiation}. */
int pbc_b200_set_stage_profiling(pbc_b200_pairing_t *p, int on);
int pbc_b200_stage_times(pbc_b200_pairing_t *p, float *ms3);

/* Test hook for the one-time constant derivation (f_init_pairing ecc/f_param.c:408-444,
 * d_init_pairing ecc/d_param.c:1035-1049): writes the canonical residues of the named derived
 * constant, each as `width` big-endian bytes, and returns the byte count (negative on failure).
 * type f: xi, xi_inv, twist_b, xpowq2, xpowq6, xpowq8 (2 coordinates each), tateexp (1);
 * type d: xpwr3, xpwr4, xpowq, xpowq2 (3 each), nqrinv, nqrinv2, phikonr (1);
 * type e: R (2: the fixed point of the Miller loop, x then y), phikonr = (q - 1)/r (1).  Host only. */
int pbc_b200_derived_constant(const pbc_b200_pairing_t *p, const char *name, unsigned char *out,
                              size_t width, size_t cap);

/* F_p differential-test hook (guru/fp_test.c, guru/checkfp.c analogue): out[i] = a[i] op b[i]
 * in F_q on the device; operands and results are canonical big-endian F_q wire bytes.
 * op: 0 = mul, 1 = add, 2 = sub, 3 = invert a (b ignored), 4 = halve a, 5 = neg a,
 * 6 = square a, 7 = a*b - b.  Eight-limb type d: 8 = square root of a (q = 1 mod 8; zero for a
 * non-square), 9 = the lazy double-width product.  Type a, ops 8-14: the slot routines of the Miller
 * step with its mode flags, several coordinates per item -- (in a, in b, in out) =
 *   8 (2, 2, 1) a0 b0 + a1 b1 through lazy(LZ_TWO | LZ_GLOBAL_B), b0 read from a global array;
 *   9 (2, 2, 6) lazy(LZ_TWO | LZ_SUB | LZ_ADD_QR | LZ_KARATSUBA) then lazy(LZ_SUB_S | LZ_ADD_QR):
 *     a0 b0 - a1 b1, a0 b1 + a1 b0, the stored sum S' as two raw 64-byte words (low, high; not
 *     converted out of Montgomery form), a0 + a1, b0 + b1;
 *  10 (1, 1, 1) 2 a0^2 - b0;  11 (2, 2, 1) (a0 + a1)^2 - b0 - b1;  12 (2, 2, 1) (a0 + a1)(b0 + b1);
 *  13 (2, 2, 1) (a0 + a1)(b0 - b1);  14 (1, 1, 1) a0 b0, b0 read from a global array.
 * Item i's coordinates are consecutive: a holds n * (in a) coordinates, and so on. */
int pbc_b200_fp_op(pbc_b200_pairing_t *p, int op, unsigned char *out, const unsigned char *a,
                   const unsigned char *b, size_t n);

/* Extension-tower differential-test hook, GT wire format in and out.  Types f, d and g:
 * op 0 = a*b, 1 = a^2, 2 = 1/a, 3 = final exponentiation of a (f_tateexp ecc/f_param.c:250-283,
 * cc_tatepower ecc/d_param.c:505-564); type f: 4 = a times the sparse Miller line held in b's
 * coefficients 0, 3, 4, 6 = the final exponentiation the pairings run (the slot-machine kernel
 * k_f_finalexp_s; fails where the parameters do not allow it); type d: 5 = F_q^3 product of the real
 * halves, 6 = F_q^3 inverse.
 * Types a, a1 and e: op 3 only -- the final stage every pairing of these types runs (the batch
 * inversion and final-exponentiation kernels, with the pairings' launch configuration), on the
 * caller's Miller values.  Wire coordinates are reduced mod q, as element_from_bytes reduces them.
 *   a, a1: f = a[i] in F_q^2, out[i] = f^((q^2 - 1)/r), which is f^((p - 1) l) for a1; b is ignored.
 *     f with f0 f1 = 0 (f in F_q or in i F_q, zero included) gives the identity: the kernels take a
 *     shortcut there, exact for every such f but zero, which has no final exponentiation.
 *   e: out[i] = (v / vd)^((q - 1)/r) with v = a[i] and vd = b[i] (vd = 1 where b is NULL); vd = 0
 *     gives 1 and v = 0 with vd != 0 gives 0.
 * The reference divides by zero on those zero inputs; the values above are this hook's definition. */
int pbc_b200_tower_op(pbc_b200_pairing_t *p, int op, unsigned char *out, const unsigned char *a,
                      const unsigned char *b, size_t n);

#ifdef __cplusplus
}
#endif
#endif
