/* helib_b200.h -- C ABI of the H100-native DoubleCRT / NTT / key-switch engine.
 *
 * This is the drop-in boundary for HElib's hot path (SURVEY.md section 8b).  HElib itself has no
 * plugin/FFI seam above row granularity (src/intelExt.h:22-58 is per-row and CPU-only), so the
 * boundary sits at the helib::DoubleCRT method level: each entry point below replaces the body of
 * one DoubleCRT / Cmodulus / Ctxt method, cited as `reference: path:line` (paths relative to the
 * HElib source tree, v2.2.0).
 *
 * Conventions
 *  - Opaque handles.  The engine owns device memory; the caller owns host buffers.
 *  - Every function returns 0 on success or a negative HB_ERR_* code; nothing throws across the
 *    ABI.  hb_last_error() returns a thread-local message for the last failure.
 *  - A device polynomial (hb_poly) is a dense matrix uint64[nprimes][N]: the row of chain prime i
 *    holds canonical residues in [0, q_i) in HElib's evaluation order row[j] = f(psi_i^(2j+1))
 *    (reference: src/CModulus.cpp:392-426, src/PAlgebra.cpp:535-540).  Which rows are live is
 *    the caller's metadata (helib::IndexSet), passed to every call as an index list.
 *  - Host-side dense matrices use the same [nprimes][N] layout; only the rows named by the index
 *    list are read or written.
 *  - Calls are stream-ordered on the context's CUDA stream and asynchronous unless stated;
 *    hb_ctx_sync() or any download synchronises.  A context may be used by one host thread at a
 *    time (the reference's DoubleCRT has the same value-semantic rule).
 *  - There is no CPU fallback: without a CUDA device hb_ctx_create fails with HB_ERR_NO_DEVICE.
 */
#ifndef HELIB_B200_H
#define HELIB_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define HB_OK 0
#define HB_ERR_BAD_ARG (-1)      /* helib::InvalidArgument / LogicError */
#define HB_ERR_INDEX_SET (-2)    /* helib::RuntimeError: index-set precondition violated */
#define HB_ERR_NO_DEVICE (-3)
#define HB_ERR_CUDA (-4)
#define HB_ERR_OOM (-5)
#define HB_ERR_UNSUPPORTED (-6)

#define HB_OP_ADD 0
#define HB_OP_SUB 1
#define HB_OP_MUL 2
#define HB_OP_NEG 3
#define HB_OP_COPY 7

typedef struct hb_ctx hb_ctx;
typedef struct hb_poly hb_poly;

int hb_version(void);
const char* hb_last_error(void);
int hb_device_count(void);

/* ---- context: the device image of helib::Context's prime chain ---------------------------
 * reference: include/helib/Context.h:120-180 (moduli, smallPrimes/ctxtPrimes/specialPrimes,
 * digits), src/CModulus.cpp:62-135 (per-prime tables).  m must be a power of two (phi(m)=m/2);
 * q[i] are the chain primes in index order; psi[i] a primitive m-th root of unity mod q[i]
 * (i.e. 2N-th root, N = m/2), or psi == NULL to let the engine derive one deterministically
 * (smallest quadratic non-residue g, psi = g^((q-1)/m)). */
int hb_ctx_create(hb_ctx** out, int device, uint64_t m, int nprimes, const uint64_t* q, const uint64_t* psi);
void hb_ctx_destroy(hb_ctx* ctx);
/* digit_of[i] = digit number of ctxt prime i or -1; special = indices of the special primes.
 * reference: src/Context.cpp:902-928 (digits), :1014-1028 (special primes). */
int hb_ctx_set_chain(hb_ctx* ctx, const int32_t* digit_of, int ndigits, const int32_t* special, int nspecial);
int hb_ctx_get_psi(hb_ctx* ctx, uint64_t* psi_out);
int hb_ctx_sync(hb_ctx* ctx);
/* out[0] = exact-CRT fallback evaluations, out[1] = kernels launched, out[2] = bytes of device memory held */
int hb_ctx_stats(hb_ctx* ctx, uint64_t* out3);
int hb_ctx_reset_stats(hb_ctx* ctx);
/* Launch-timing hooks for bench.py: elapsed GPU milliseconds on the context's stream between the
 * two marks (CUDA events on the launching stream). */
int hb_ctx_mark_begin(hb_ctx* ctx);
int hb_ctx_mark_end(hb_ctx* ctx, float* ms_out);
/* Per-kernel profile for the roofline report: while enabled, every launch is bracketed by CUDA
 * events on the launching stream.  hb_ctx_profile_get(i, ...) returns HB_ERR_BAD_ARG past the end.
 * bytes = algorithmic HBM bytes (each row read once / written once) summed over the launches. */
int hb_ctx_profile(hb_ctx* ctx, int enable);
int hb_ctx_profile_get(hb_ctx* ctx, int i, char* name, int namelen, uint64_t* launches, double* ms, uint64_t* bytes);

/* ---- device polynomials (helib::DoubleCRT storage, include/helib/DoubleCRT.h:87-94) ---- */
int hb_poly_create(hb_ctx* ctx, hb_poly** out);          /* zero-filled [nprimes][N] */
void hb_poly_destroy(hb_poly* p);
int hb_poly_upload(hb_poly* p, const int32_t* idx, int n, const uint64_t* host_dense);
int hb_poly_download(hb_poly* p, const int32_t* idx, int n, uint64_t* host_dense);  /* synchronises */
int hb_poly_download_async(hb_poly* p, const int32_t* idx, int n, uint64_t* host_dense); /* stream-ordered; hb_ctx_sync() before reading */

/* Wire format (SURVEY 8f-3): byte-compatible with DoubleCRT::writeTo / read (src/DoubleCRT.cpp:1530-1561):
 * IndexSet (int64 card, int64 indices) then per row int32 length, int32 intSize(=8), little-endian int64 values
 * (src/binio.cpp:103-122).  hb_poly_deserialize also accepts intSize=4 rows and rejects residues outside [0,q). */
int hb_poly_serialized_size(hb_poly* p, int n, uint64_t* bytes);
int hb_poly_serialize(hb_poly* p, const int32_t* idx, int n, void* buf, uint64_t buflen);
int hb_poly_deserialize(hb_poly* p, const void* buf, uint64_t buflen, int32_t* idx_out, int* n_out);

/* Seeded uniform rows: NTL::SetSeed(ZZ seed) followed by polys[0].randomize(), polys[1].randomize(), ... over rows idx --
 * what SecKey::GenKeySWmatrix (src/keys.cpp:1189-1206) and Ctxt::keySwitchDigits (src/Ctxt.cpp:191-230) do to rebuild the
 * a_i of a key-switching matrix from its prgSeed, with DoubleCRT::randomize (src/DoubleCRT.cpp:1258-1378) per poly.
 * seed[0..seedlen) are the little-endian magnitude bytes of the ZZ, as write_raw_ZZ writes them (src/binio.cpp:180-203);
 * high-order zero bytes are ignored and seedlen == 0 is the seed 0.  The key is NTL's DeriveKey(32, bytes)
 * (HMAC-SHA256), the stream ChaCha20; each row consumes whole 2048-byte buffers, poly p+1 continues where poly p stopped.
 * idx must be strictly ascending; rows outside idx are not touched.  Expanded on the device: stream-ordered, no sync. */
int hb_poly_randomize(hb_poly* const* polys, int npolys, const int32_t* idx, int n, const uint8_t* seed, int seedlen);
/* Seeded polynomials: exactly the rows hb_poly_randomize(polys, npolys, idx, n, seed, seedlen) would write, held as the
 * seed plus a per-row schedule (first stream buffer of every row, exclusive row offset of every buffer) instead of rows in
 * device memory -- how HElib holds the a_i of a KeySwitch (b_i rows plus prgSeed, include/helib/keySwitching.h).
 * out[0..npolys) receive one handle per poly.  Runs the k_prg_count chain once and synchronises once.  Argument errors as
 * hb_poly_randomize (unsorted/duplicate idx, npolys <= 0, null seed with a length -> HB_ERR_BAD_ARG).
 * A seeded handle has no rows.  It is accepted in two places only: as an entry of evk_a of the key-switching entry points
 * (hb_keyswitch_digits, hb_keyswitch_digits_fused, hb_automorph_keyswitch_digits, hb_relinearize, hb_mul_relin_moddown,
 * hb_inner_product, hb_square_relin_moddown),
 * which regenerate the rows they read once per call into context scratch, and as `seeded` of hb_poly_expand.  Everything
 * else returns HB_ERR_BAD_ARG for it before launching anything; a key switch that needs a row outside the seeded set
 * returns HB_ERR_INDEX_SET.  hb_poly_destroy each handle; the shared schedule is freed with the last one and its bytes
 * count in hb_ctx_stats out[2]. */
int hb_poly_create_seeded(hb_ctx* ctx, int npolys, const int32_t* idx, int n, const uint8_t* seed, int seedlen, hb_poly** out);
/* Rows idx (a subset of the seeded set) of seeded[p] into the ordinary poly dst[p], all p in one k_prg_fill launch;
 * stream-ordered, no sync.  A row outside the seeded set -> HB_ERR_INDEX_SET. */
int hb_poly_expand(hb_poly* const* seeded, hb_poly* const* dst, int npolys, const int32_t* idx, int n);

/* ---- per-prime transforms: Cmodulus::FFT / iFFT (src/CModulus.cpp:362-429, 486-553) -----
 * In place on rows idx of each poly: coefficient rows (values in [0,q)) <-> evaluation rows. */
int hb_ntt_fwd(hb_poly* const* polys, int nitems, const int32_t* idx, int n);
int hb_ntt_inv(hb_poly* const* polys, int nitems, const int32_t* idx, int n);

/* ---- row-wise ring operations: DoubleCRT::Op<Add|Sub|Mul>, Negate, operator=
 * (src/DoubleCRT.cpp:216-384).  dst op= src on rows idx. */
int hb_pointwise(int op, hb_poly* const* dst, hb_poly* const* src, int nitems, const int32_t* idx, int n);
/* rows idx *= scalars[r] (already reduced mod q): DoubleCRT::Op(ZZ, MulFun) (src/DoubleCRT.cpp:339-361) */
int hb_scale_rows(hb_poly* const* polys, int nitems, const int32_t* idx, int n, const uint64_t* scalars);
/* rows idx *= prod(q_k : k in fidx) or its inverse: DoubleCRT::operator/= (src/DoubleCRT.cpp:1122-1139) */
int hb_scale_by_primes(hb_poly* const* polys, int nitems, const int32_t* idx, int n, const int32_t* fidx, int nf, int inverse);
int hb_zero_rows(hb_poly* const* polys, int nitems, const int32_t* idx, int n);

/* DoubleCRT::addPrimesAndScale (src/DoubleCRT.cpp:603-647) */
int hb_add_primes_and_scale(hb_poly* const* polys, int nitems, const int32_t* cur, int ncur, const int32_t* add, int nadd);
/* DoubleCRT::addPrimes (src/DoubleCRT.cpp:565-599): exact base extension of rows cur to rows add */
int hb_add_primes(hb_poly* const* polys, int nitems, const int32_t* cur, int ncur, const int32_t* add, int nadd);
/* DoubleCRT::scaleDownToSet (src/DoubleCRT.cpp:1464-1516): rows keep <- (x - delta)/P, rows cur\keep dropped
 * (left as garbage; the caller's index set shrinks).  ptxt_space = 1 for CKKS. */
int hb_scale_down(hb_poly* const* polys, int nitems, const int32_t* cur, int ncur, const int32_t* keep, int nkeep, uint64_t ptxt_space);
/* DoubleCRT::toPoly (src/DoubleCRT.cpp:925-1113): balanced (or positive) big integers,
 * out[N][Lout] little-endian two's-complement limbs.  Synchronises. */
int hb_to_poly(hb_poly* p, const int32_t* idx, int n, int positive, uint64_t* out_limbs, int Lout);
/* Tail of SecKey::Decrypt (src/keys.cpp:1381-1399): PolyRed(toPoly(ptxt), ptxt_space) times factor
 * (= (intFactor*Q)^-1 mod ptxt_space, or 1), out[N] in [0, ptxt_space).  The big integers stay on the device:
 * N words come back instead of N*(n+1).  ptxt_space >= 2, coprime to the primes in idx.  Synchronises. */
int hb_to_poly_mod_p(hb_poly* p, const int32_t* idx, int n, uint64_t ptxt_space, uint64_t factor, int64_t* out);
/* DoubleCRT(const zzX&, context, s) / FFT(const zzX&, s) (src/DoubleCRT.cpp:87-105, src/CModulus.cpp:339-356):
 * coeffs[nitems][N] signed 64-bit coefficients (|c| < 2^63) are copied once, reduced modulo every prime in idx
 * and transformed on the device.  Synchronises (the host buffer may be reused on return). */
int hb_poly_from_i64(hb_poly* const* polys, int nitems, const int32_t* idx, int n, const int64_t* coeffs);
/* DoubleCRT(const ZZX&, context, s) / FFT(const ZZX&, s) (src/DoubleCRT.cpp:68-85; the per-prime `convert`,
 * src/CModulus.cpp:453-457, timer FFT_remainder): limbs[nitems][N][L] little-endian two's-complement big
 * integers (the layout hb_to_poly produces).  Synchronises. */
int hb_poly_from_limbs(hb_poly* const* polys, int nitems, const int32_t* idx, int n, const uint64_t* limbs, int L);
/* dst += a * b row-wise: `key *= part; ptxt += key` of SecKey::Decrypt (src/keys.cpp:1373-1374) and
 * `parts[i] *= r; parts[i] += e` of PubKey::Encrypt (src/keys.cpp:416,443) in one pass. */
int hb_muladd(hb_poly* const* dst, hb_poly* const* a, hb_poly* const* b, int nitems, const int32_t* idx, int n);
/* ---- powerful basis and the recryption mod-switch (SURVEY 8f-4) ----
 * hb_ctx_set_powerful: PowerfulDCRT(context, mvec) (src/powerful.cpp:246-318): the factorisation of m into prime powers
 *   (what Context::buildRecryptData passes); optional -- without it the engine factors m itself on first use.
 * hb_ctx_powerful_info: number of factors, the factors, and to_poly[i] = cubeToPolyMap[shortToLongMap[i]], the exponent
 *   of X that powerful coefficient i is written to before the reduction modulo Phi_m (powerfulToPoly, src/powerful.cpp:223-244).
 * hb_dcrt_to_powerful: PowerfulDCRT::dcrtToPowerful (src/powerful.cpp:393-410): the balanced integers modulo Q of the
 *   powerful-basis coefficients, out[N][Lout] two's-complement limbs.
 * hb_raw_mod_switch: the per-part body of Ctxt::rawModSwitch (src/Ctxt.cpp:2976-3037): out[N] = the powerful-basis
 *   coefficients scaled by q/Q, rounded with the correction that keeps them = c*q*Q^-1 modulo ptxt_space, reduced
 *   symmetrically mod q (a tie of an even q is left at +-q/2; the reference flips a coin there). */
int hb_ctx_set_powerful(hb_ctx* ctx, const int64_t* mvec, int k);
int hb_ctx_powerful_info(hb_ctx* ctx, int32_t* nfactors, int64_t* mvec, int32_t* to_poly);
int hb_dcrt_to_powerful(hb_poly* p, const int32_t* idx, int n, uint64_t* out_limbs, int Lout);
int hb_raw_mod_switch(hb_poly* p, const int32_t* idx, int n, uint64_t q, uint64_t ptxt_space, int64_t* out);
/* DoubleCRT::breakIntoDigits (src/DoubleCRT.cpp:479-561).  src rows cur (ctxt primes only);
 * digits[item*maxdig + i] receives digit i over cur | special.  *ndig_out = number of digits. */
int hb_break_into_digits(hb_poly* const* src, int nitems, const int32_t* cur, int ncur, hb_poly* const* digits, int maxdig, int* ndig_out);
/* Ctxt::keySwitchDigits (src/Ctxt.cpp:191-230): out0 += sum_i D_i*b_i, out1 += sum_i D_i*a_i on rows idx.
 * evk_a[i]: the pseudo-random a_i, either expanded rows (e.g. by hb_poly_randomize) or seeded handles
 * (hb_poly_create_seeded), whose rows idx are regenerated on every call as the reference does from prgSeed
 * (src/Ctxt.cpp:196-206). */
int hb_keyswitch_digits(hb_poly* const* digits, int maxdig, int ndig, int nitems, const int32_t* idx, int n,
                        hb_poly* const* evk_a, hb_poly* const* evk_b, hb_poly* const* out0, hb_poly* const* out1);
/* The same inner product with the two passes around it folded in (what Ctxt::keySwitchPart + reLinearize do per part,
 * src/Ctxt.cpp:764-768,805-842):
 *   out0[r] = scal[r]*out0[r] + sum_i D_i[r]*b_i[r]   (same for out1 / a_i);  scal[r] == 0 => the row is a pure output
 *   (addPrimesAndScale: scal[r] = prod(special) mod q_r on the rows the part already has, 0 on the special rows);
 *   own / own_dig (optional): rows with own_dig[r] = i >= 0 take digit i from own[item] (the part being switched, whose rows
 *   ARE digit i's own rows) instead of digits[item*maxdig + i] -- no copies of the part into the digit polynomials.
 * Power-of-two m, at most 4 digits. */
int hb_keyswitch_digits_fused(hb_poly* const* digits, int maxdig, int ndig, int nitems, const int32_t* idx, int n,
                              hb_poly* const* evk_a, hb_poly* const* evk_b, hb_poly* const* out0, hb_poly* const* out1,
                              const uint64_t* scal, hb_poly* const* own, const int32_t* own_dig);
/* The mixed-radix step of DoubleCRT::breakIntoDigits (src/DoubleCRT.cpp:551-556) in one pass:
 * dst = (dst - src) / prod(q_f, f in fidx) on rows idx. */
int hb_sub_div_by_primes(hb_poly* const* dst, hb_poly* const* src, int nitems, const int32_t* idx, int n, const int32_t* fidx, int nf);
/* Hoisted automorphism + key switch (SURVEY 8f-1): BasicAutomorphPrecon::automorph (src/matmul.cpp:112-184),
 * the rotation path of Ctxt::smartAutomorph (src/Ctxt.cpp:2462-2515).  The digits of the s-part are computed once
 * with hb_break_into_digits; for each amount k (odd, < m) one launch applies sigma_k in the load stage:
 *   out0 = P*sigma_k(c0) + sum_i sigma_k(D_i)*b_i ,  out1 = sum_i sigma_k(D_i)*a_i     over S | special
 * (evk_a/evk_b: the matrix for s(X^k) -> s).  Outputs must not alias inputs.  Power-of-two m. */
int hb_automorph_keyswitch_digits(hb_poly* const* digits, int maxdig, int ndig, int nitems, const int32_t* S, int nS,
                                  hb_poly* const* c0, uint64_t k, hb_poly* const* evk_a, hb_poly* const* evk_b,
                                  hb_poly* const* out0, hb_poly* const* out1);
/* Hoisted linear map (SURVEY 8f-1): the loop body of MatMul1DExec::mul's native FULL branch (src/matmul.cpp:1226-1252) for
 * the amounts whose matrix is direct -- sum_j consts[j] * BasicAutomorphPrecon::automorph(k[j]) with the mod-down left lazy.
 * digits = hb_break_into_digits of c1 over S (maxdig, ndig as for hb_automorph_keyswitch_digits); c0, c1 over S;
 * consts[j] over S | special (evaluation form); evk_a/evk_b [namt*ndig], matrix j = entries j*ndig .. j*ndig+ndig-1, the
 * matrix for s(X^k[j]) -> s (ignored, and may be NULL, where k[j] == 1).  Over S | special, for every item:
 *   acc0 (+)= sum_j consts[j] * ( P*sigma_kj(c0) + [k_j != 1] sum_i sigma_kj(D_i)*b_{j,i} )
 *   acc1 (+)= sum_j consts[j] * ( [k_j == 1] P*c1  +  [k_j != 1] sum_i sigma_kj(D_i)*a_{j,i} )
 * P*x is addPrimesAndScale: x*P on the rows of S and 0 on the special rows.  accumulate = 0 overwrites acc0/acc1.
 * The items share k, consts and the matrices.  Power-of-two and general m.  One k_ks_linmap launch per group of up to 64
 * amounts (per item chunk and row chunk); seeded evk_a are regenerated a few matrices at a time, so the key scratch does
 * not grow with namt.  Errors, all reported before any launch: k[j] not in Z_m^*, S not within the ctxt primes, or a
 * seeded evk_a without a needed row -> HB_ERR_INDEX_SET; namt <= 0, ndig out of range, c1 NULL while some k[j] == 1, an
 * accumulator aliasing an input or another accumulator, or a seeded handle other than in evk_a -> HB_ERR_BAD_ARG.
 * Stream-ordered, no synchronisation; after the first call, a call of the same shape allocates nothing. */
int hb_hoisted_linear_map(hb_poly* const* digits, int maxdig, int ndig, int nitems, const int32_t* S, int nS,
                          hb_poly* const* c0, hb_poly* const* c1, int namt, const uint64_t* k, hb_poly* const* consts,
                          hb_poly* const* evk_a, hb_poly* const* evk_b, hb_poly* const* acc0, hb_poly* const* acc1,
                          int accumulate);
/* BSGS linear map (SURVEY 8f-1): the giant-step phase of MatMul1DExec::mul's non-iterative baby-step/giant-step branches
 * (src/matmul.cpp:1022-1057 native, 1097-1142 bad dimension with ALT_MATMUL).  The baby steps are inputs:
 * baby0/baby1[item*nbaby + j] are the two parts of baby step j of each item, over S (extended == 0: cleaned, the native
 * branch) or over S | special (extended == 1: not cleaned, the bad-dimension branch, whose baby steps j = 0 the caller first
 * brings to S | special with hb_add_primes_and_scale).  consts[t*nbaby + j] over the rows of the baby steps (NULL: a zero
 * diagonal, skipped as MulAdd skips it), kgiant[t] the amount of giant step t, scal[t] an integer factor (NULL: all 1).
 * For every item, with inner_t = scal[t] * sum_j consts[t*nbaby + j] * baby_j (both parts), over S | special:
 *   kgiant[t] == 1: term_t = P*inner_t (extended == 0, addPrimesAndScale) or inner_t (extended == 1)
 *   otherwise the steps of smartAutomorph(kgiant[t]) in HElib's order: sigma_k; if extended, the mod-down to S
 *     (scaleDownToSet with ptxt_space, as reLinearize's dropSmallAndSpecialPrimes); breakIntoDigits of part 1 over S; the
 *     key switch with matrix t: term_t = (P*c0' + sum_i D_i*b_{t,i}, sum_i D_i*a_{t,i})
 *   acc0/acc1 (+)= sum_t term_t                                  (accumulate = 0 overwrites)
 * scal[t] is relin_CKKS_adjust's factor, which HElib applies after the mod-down: it must be 1 when extended == 1.
 * evk_a/evk_b [ngiant*ndig_evk], matrix t = entries t*ndig_evk .. (ignored, and may be NULL, where kgiant[t] == 1); the
 * matrices need as many columns as S has digits.  ptxt_space = 1 for CKKS.  The items share the constants, amounts and
 * matrices.  Power-of-two and general m; expanded or seeded evk_a.  Work goes in groups of at most 32 (giant step, item)
 * pairs: one k_bsgs_mac pass per group and 8 pairs forms the rotated inner sums, the mod-down and digits run once per group
 * over all of its rotated sums, and one k_ks_giant pass per group sums the key switches into the accumulators.  The
 * scratch is min(32, nitems*ngiant)*(2 + ndig) polys whatever ngiant is.  Errors, all reported before any launch: kgiant[t] not in Z_m^*, S
 * not within the ctxt primes, or a seeded evk_a without a needed row -> HB_ERR_INDEX_SET; counts out of range, too few
 * matrix columns, scal != 1 in the extended form, an accumulator aliasing an input or another accumulator, or a seeded
 * handle other than in evk_a -> HB_ERR_BAD_ARG.  Stream-ordered, no synchronisation; after the first call, a call of the
 * same shape allocates nothing. */
int hb_bsgs_linear_map(hb_poly* const* baby0, hb_poly* const* baby1, int nbaby, int nitems,
                       const int32_t* S, int nS, int extended, uint64_t ptxt_space,
                       int ngiant, const uint64_t* kgiant, hb_poly* const* consts, const uint64_t* scal,
                       hb_poly* const* evk_a, hb_poly* const* evk_b, int ndig_evk,
                       hb_poly* const* acc0, hb_poly* const* acc1, int accumulate);
/* The same, returning the norms the noise bookkeeping of smartAutomorph needs for every rotated giant step:
 * norms[(item*ngiant + t)*(8 + 2) + i] = ln ||E_i|| of digit i (i < ndig; breakIntoDigits' norms), and at offsets 8 and 9 the
 * ||delta/P|| of parts 0 and 1 of the extended form's mod-down (hb_scale_down_norm).  Entries of unrotated giant steps are not
 * written.  Synchronises (host values). */
int hb_bsgs_linear_map_norm(hb_poly* const* baby0, hb_poly* const* baby1, int nbaby, int nitems,
                            const int32_t* S, int nS, int extended, uint64_t ptxt_space,
                            int ngiant, const uint64_t* kgiant, hb_poly* const* consts, const uint64_t* scal,
                            hb_poly* const* evk_a, hb_poly* const* evk_b, int ndig_evk,
                            hb_poly* const* acc0, hb_poly* const* acc1, int accumulate, double* norms);
/* Block linear map (SURVEY 8f-1): BlockMatMul1DExec::mul's non-iterative branches with one PartitionInfo interval
 * (src/matmul.cpp:1782-1868 native, 1869-1974 bad dimension), i.e. a GF(p)-linear map on slots of degree d.  digits =
 * hb_break_into_digits of c1 over S ([item*maxdig + i], maxdig at least the digits of S); c0, c1 over S.  Inner amounts
 * k0[i] (i < n0) with matrices evk0 (s(X^k0) -> s), outer amounts k1[j] (j < n1) with matrices evk1; consts[i*n1 + j] over
 * S | special (HElib's cache.multiplier[i*d1 + j]; NULL: a zero block, skipped as MulAdd skips it).  consts1 != NULL
 * selects the bad dimension: consts1 has the layout of consts, kfinal is genToPow(dim, -D) with matrix evkf.  For every
 * item, over S | special, in HElib's order of steps:
 *   r_i = BasicAutomorphPrecon::automorph(k0[i])   (k0[i] == 1: P*(c0, c1), addPrimesAndScale)
 *   a_j = sum_i consts[i*n1 + j] * r_i,  a1_j likewise with consts1
 *   term(x, k) = x for k == 1; otherwise smartAutomorph(k) in the extended form of hb_bsgs_linear_map: sigma_k, the mod-down
 *     to S (scaleDownToSet with ptxt_space), breakIntoDigits over S and the key switch
 *   acc0/acc1 (+)= sum_j term(a_j, k1[j])  [ + term( sum_j term(a1_j, k1[j]), kfinal ) ]      (accumulate = 0 overwrites)
 * evk*_a/evk*_b hold ndig_evk entries per matrix (matrix t = entries t*ndig_evk ..; evkf one matrix), ignored and may be
 * NULL where the amount is 1; they need as many columns as S has digits.  The items share everything but digits, c0, c1,
 * acc0 and acc1.  Power-of-two and general m; expanded or seeded evk_a.  Per chunk of items (at most 32) and group of
 * outputs ((j, set) pairs, at most 64 with the items): k_ks_hoist writes the rotations of at most 128/items inner amounts,
 * k_bsgs_mac folds them into the group's rotated sums, and the mod-down, digits and k_ks_giant follow as in
 * hb_bsgs_linear_map.  The scratch is at most 2*min(128, n0*ic) + min(64, nitems*n1*(bad ? 2 : 1))*(2 + ndig) + (bad ?
 * 2*ic : 0) polys, ic = min(32, nitems): it does not grow with n0 past 128/ic inner amounts, nor with n1.  Errors, all
 * reported before any launch: an amount not in Z_m^*, S not within the ctxt primes, or a seeded evk_a without a needed row
 * -> HB_ERR_INDEX_SET; n0, n1 or nitems <= 0, no amounts, too few digit slots or matrix columns, a missing matrix, an
 * accumulator aliasing an input or another accumulator, or a seeded handle other than in evk_a -> HB_ERR_BAD_ARG.
 * Stream-ordered, no synchronisation; after the first call, a call of the same shape allocates nothing. */
int hb_block_linear_map(hb_poly* const* digits, int maxdig, int nitems, const int32_t* S, int nS,
                        hb_poly* const* c0, hb_poly* const* c1, uint64_t ptxt_space,
                        int n0, const uint64_t* k0, hb_poly* const* evk0_a, hb_poly* const* evk0_b,
                        int n1, const uint64_t* k1, hb_poly* const* evk1_a, hb_poly* const* evk1_b,
                        hb_poly* const* consts, hb_poly* const* consts1, uint64_t kfinal,
                        hb_poly* const* evkf_a, hb_poly* const* evkf_b, int ndig_evk,
                        hb_poly* const* acc0, hb_poly* const* acc1, int accumulate);
/* The same, returning the norms the noise bookkeeping of smartAutomorph needs for every rotated term, in the layout of
 * hb_bsgs_linear_map_norm: with T = n1 (native) or 2*n1 + 1 (bad dimension), norms[(item*T + e)*(8 + 2) + i] = ln ||E_i||
 * of digit i (i < ndig), and at offsets 8 and 9 the ||delta/P|| of parts 0 and 1 of the mod-down.  Entry e = j is term
 * (a_j, k1[j]); in the bad dimension e = n1 + j is term (a1_j, k1[j]) and e = 2*n1 the final term (kfinal).  Entries of
 * unrotated terms are not written.  Synchronises (host values). */
int hb_block_linear_map_norm(hb_poly* const* digits, int maxdig, int nitems, const int32_t* S, int nS,
                             hb_poly* const* c0, hb_poly* const* c1, uint64_t ptxt_space,
                             int n0, const uint64_t* k0, hb_poly* const* evk0_a, hb_poly* const* evk0_b,
                             int n1, const uint64_t* k1, hb_poly* const* evk1_a, hb_poly* const* evk1_b,
                             hb_poly* const* consts, hb_poly* const* consts1, uint64_t kfinal,
                             hb_poly* const* evkf_a, hb_poly* const* evkf_b, int ndig_evk,
                             hb_poly* const* acc0, hb_poly* const* acc1, int accumulate, double* norms);
/* Full linear map leaves (SURVEY 8f-1): the last dimension of MatMulFullExec::rec_mul (src/matmul.cpp:2141-2148), every
 * leaf a hoisted MatMul1DExec::mul (:1226-1252 native, :1253-1283 bad dimension), all leaves of a ciphertext summed into
 * one accumulator.  Leaf l of item it is the two-part ciphertext (x0, x1)[it*nleaves + l]: over S | special when
 * ext[l] != 0 (a rotated leaf, not cleaned), over S otherwise (ext == NULL: every leaf over S).  Amounts k[t] (t < namt)
 * with matrices evk_a/evk_b (matrix t = entries t*ndig_evk .., ignored and may be NULL where k[t] == 1); constants
 * consts[l*namt + t] over S | special (HElib's cache.multiplier of leaf l; NULL: a zero diagonal, skipped as MulAdd skips
 * it).  consts1 != NULL selects a bad leaf dimension: consts1 has the layout of consts, kfinal is genToPow(dim, -D) with
 * matrix evkf.  For every item, over S | special, in HElib's order of steps:
 *   x_l <- cleanUp(x_l)      ext[l]: scaleDownToSet to S with ptxt_space (dropSmallAndSpecialPrimes)
 *   D_l  = breakIntoDigits(x_l.part1) over S
 *   r_{l,t} = BasicAutomorphPrecon(x_l).automorph(k[t])          (k[t] == 1: P*(c0, c1), addPrimesAndScale)
 *   acc0/acc1 (+)= sum_l sum_t consts[l*namt + t] * r_{l,t}  [ + sum_l term( sum_t consts1[l*namt + t] * r_{l,t}, kfinal ) ]
 * term(y, k) = y for k == 1, otherwise smartAutomorph(k) in the extended form of hb_bsgs_linear_map: sigma_k, the mod-down
 * to S, breakIntoDigits over S and the key switch.  accumulate = 0 overwrites.  The items share amounts, matrices and
 * constants; the inputs are read-only.  Power-of-two and general m; expanded or seeded evk_a.  Per chunk of at most 32
 * (item, leaf) pairs: the chunk's mod-downs and digits run in one batched launch each; one k_ks_leafmap pass per group of
 * at most 32 amounts sums every leaf's rotations into the accumulators (and the per-leaf sums of the bad dimension), its
 * matrices (seeded: regenerated once per chunk and group of amounts) read once for the up to 4 leaves a thread holds; in a bad
 * dimension sigma_kfinal, the mod-down, digits and k_ks_giant follow for the chunk's per-leaf sums.  The scratch is at most
 * min(32, nitems*nleaves)*(bad ? 4 + ndig : 2 + ndig) + (bad and evkf_a seeded ? ndig : 0) polys whatever nleaves and
 * namt are.  Errors, all reported before any launch: an amount not in Z_m^*, S not within the ctxt primes, or a seeded
 * evk_a without a needed row -> HB_ERR_INDEX_SET; nleaves, nitems or namt <= 0, ext not 0/1, no amounts, too few matrix
 * columns, S with more than 8 digits, a missing matrix, an accumulator aliasing an input or another accumulator, or a
 * seeded handle other than in evk_a -> HB_ERR_BAD_ARG.  Stream-ordered, no synchronisation; after the first call, a call
 * of the same shape allocates nothing. */
int hb_full_linear_map_leaves(hb_poly* const* x0, hb_poly* const* x1, int nleaves, int nitems, const int32_t* ext,
                              const int32_t* S, int nS, uint64_t ptxt_space, int namt, const uint64_t* k,
                              hb_poly* const* evk_a, hb_poly* const* evk_b, hb_poly* const* consts, hb_poly* const* consts1,
                              uint64_t kfinal, hb_poly* const* evkf_a, hb_poly* const* evkf_b, int ndig_evk,
                              hb_poly* const* acc0, hb_poly* const* acc1, int accumulate);
/* The same, returning the norms the noise bookkeeping of the leaves needs, in the layout of hb_block_linear_map_norm: with
 * T = nleaves (native) or 2*nleaves (bad dimension), norms[(item*T + e)*(8 + 2) + i].  Entry e = l is leaf l's cleanUp and
 * hoisting: ln ||E_i|| of its digit i (i < ndig, breakIntoDigits' norms) and, for ext[l] != 0, at offsets 8 and 9 the
 * ||delta/P|| of parts 0 and 1 of its mod-down (hb_scale_down_norm).  In the bad dimension entry nleaves + l is leaf l's
 * final term (kfinal): its digits' and mod-down's norms likewise.  Entries not computed are not written.  Synchronises. */
int hb_full_linear_map_leaves_norm(hb_poly* const* x0, hb_poly* const* x1, int nleaves, int nitems, const int32_t* ext,
                                   const int32_t* S, int nS, uint64_t ptxt_space, int namt, const uint64_t* k,
                                   hb_poly* const* evk_a, hb_poly* const* evk_b, hb_poly* const* consts, hb_poly* const* consts1,
                                   uint64_t kfinal, hb_poly* const* evkf_a, hb_poly* const* evkf_b, int ndig_evk,
                                   hb_poly* const* acc0, hb_poly* const* acc1, int accumulate, double* norms);
/* Ctxt::tensorProduct of two canonical 2-part ciphertexts (src/Ctxt.cpp:1563-1608) */
int hb_tensor(hb_poly* const* a0, hb_poly* const* a1, hb_poly* const* b0, hb_poly* const* b1,
              hb_poly* const* o0, hb_poly* const* o1, hb_poly* const* o2, int nitems, const int32_t* idx, int n);
/* The tensor products of npairs pairs per item, summed (Ctxt::multLowLvl's tensorProduct followed by innerProduct's +=,
 * src/Ctxt.cpp:2878-2893, for operands already at one prime set).  Pair j of item t is [t*npairs + j]; on rows idx:
 *   o0 (+)= sum_j a0_j*b0_j,  o1 (+)= sum_j (a0_j*b1_j + a1_j*b0_j),  o2 (+)= sum_j a1_j*b1_j   (mod q)
 * accumulate = 0 overwrites the outputs.  Inputs are read-only and may alias each other (a == b: sums of squares); on the
 * register path (power-of-two m, N a multiple of 512) they may be lazy below 8q + 2^32.  Outputs are canonical.
 * npairs or nitems <= 0, accumulate not 0/1, or an output aliasing an input or another output -> HB_ERR_BAD_ARG. */
int hb_tensor_sum(hb_poly* const* a0, hb_poly* const* a1, hb_poly* const* b0, hb_poly* const* b1, int npairs, int nitems,
                  const int32_t* idx, int n, hb_poly* const* o0, hb_poly* const* o1, hb_poly* const* o2, int accumulate);
/* Scaled sums of two-part ciphertexts: every simplePolyEval leaf of polyEval (src/polyEval.cpp:223-255) is
 * sum_i s_i * X^i + c on every row, with per-row integer scalars that the loop's multByConstant / modUpToSet / addCtxt /
 * addConstant arithmetic determines.  nitems items, each with nin inputs (in0, in1)[t*nin + i] and nout outputs
 * (out0, out1)[t*nout + j]; on every row r of U (sorted, no repeats, within the chain):
 *   out_k[t*nout + j] (+)= sum_i scal[(j*nin + i)*nU + r] * in_k[t*nin + i]   (mod q_{U[r]}, k = 0, 1)
 * plus cst[j*nU + r] on part 0 (cst may be NULL).  accumulate = 0 overwrites.  The items share scal and cst, which are
 * canonical residues; a zero scalar means that input row is not read.  Inputs may be any 64-bit words (reduced on load);
 * outputs are canonical.  Each input row is read once and each output row written once, for any nout (more than
 * HB_SSUM_MAXIN = 191 inputs run in groups, the later ones accumulating).  The tables are staged in context-owned device
 * memory in stream order: the call is asynchronous, the caller may free its arrays when it returns, and after the first
 * call a call of the same shape allocates nothing.  Counts <= 0, accumulate not 0/1, a scalar or constant not below its
 * prime, an output aliasing an input or another output, or a seeded handle -> HB_ERR_BAD_ARG; U unsorted, repeated or
 * outside the chain -> HB_ERR_INDEX_SET; all checked before any launch. */
int hb_ctxt_scaled_sums(hb_poly* const* in0, hb_poly* const* in1, int nin, hb_poly* const* out0, hb_poly* const* out1,
                        int nout, int nitems, const int32_t* U, int nU, const uint64_t* scal, const uint64_t* cst,
                        int accumulate);
/* DoubleCRT::automorph (src/DoubleCRT.cpp:1160-1202): dst[j] = src[idx(rep(j)*k mod m)], dst != src */
int hb_automorph(hb_poly* const* dst, hb_poly* const* src, int nitems, const int32_t* idx, int n, uint64_t k);

/* ---- noise metadata: canonical-embedding norms (embeddingLargestCoeff, src/norms.cpp:204-261,443-485),
 * computed in FP64 on the device from the coefficient data the conversion kernels already hold.
 * Same operations as above plus the norm outputs; these variants synchronise (they return host values).
 *  hb_add_primes_norm        : log_norms[item] = ln max_j |f(zeta^j)| of the balanced polynomial being extended
 *  hb_break_into_digits_norm : log_norms[item*maxdig+i] = ln ||E_i||  (breakIntoDigits returns their sum, src/DoubleCRT.cpp:542-545)
 *  hb_scale_down_norm        : norms[item] = ||delta/P||  (the fdelta norms of Ctxt::modDownToSet, src/Ctxt.cpp:476-505)
 * Precision: each coefficient enters as x/Q (x/P for the mod-down) taken from the conversion's 0.64 fixed-point sum over
 * the n source primes, with an absolute error of at most 4n*2^-64 in either direction.  The norm is therefore off by at
 * most 4n*N*2^-64*Q in absolute terms (Q: the product of cur for hb_add_primes_norm, of the digit's primes for
 * hb_break_into_digits_norm; 1 for hb_scale_down_norm, in delta/P units), above or below.  Polynomials whose coefficients
 * lie far below 2^-40*Q get about that floor instead of their norm; the zero polynomial over an empty set gives -inf.
 * The integer rows are exact whatever the norm's error. */
int hb_add_primes_norm(hb_poly* const* polys, int nitems, const int32_t* cur, int ncur, const int32_t* add, int nadd, double* log_norms);
int hb_break_into_digits_norm(hb_poly* const* src, int nitems, const int32_t* cur, int ncur, hb_poly* const* digits, int maxdig, int* ndig_out, double* log_norms);
int hb_scale_down_norm(hb_poly* const* polys, int nitems, const int32_t* cur, int ncur, const int32_t* keep, int nkeep, uint64_t ptxt_space, double* norms);

/* ---- prime-sharded base conversion (SURVEY.md 8e; one rank per GPU, rows sharded by prime index).
 * The exact conversion of hb_add_primes / hb_scale_down split where residues must cross shards:
 *   hb_conv_make_y : for the owned rows of the source set D: y_j = iNTT(row_j) * (Q_D/q_j)^-1 mod q_j,
 *                    written to ypolys rows `owned` in coefficient order (local work, no communication);
 *   [caller: all-gather of the y rows over NCCL/NVLink so that every rank holds all rows of D]
 *   hb_conv_from_y : exact CRT of the gathered y rows, reduction mod the target primes this rank owns,
 *                    forward transform into dst rows tgt.  mode 0: dst = x (addPrimes, src/DoubleCRT.cpp:565-599);
 *                    mode 1: dst = (dst - x) / Q_D with the BGV correction (scaleDownToSet, :1464-1516). */
int hb_conv_make_y(hb_poly* const* polys, int nitems, const int32_t* D, int nD, const int32_t* owned, int nOwned, hb_poly* const* ypolys);
int hb_conv_from_y(hb_poly* const* ypolys, int nitems, const int32_t* D, int nD, const int32_t* tgt, int nT,
                   uint64_t ptxt_space, hb_poly* const* dst, int mode);
/* Fused "make y + all-gather": like hb_conv_make_y, but the final kernel also stores the y rows into the
 * y buffers of up to 8 peer GPUs (peer_ypolys[p*nitems + item], obtained with hb_poly_ipc_open), so the rows
 * cross NVLink once, straight into place.  The caller orders a cross-rank barrier (e.g. a 1-element NCCL
 * all-reduce on the same stream) before hb_conv_from_y reads the buffers. */
int hb_conv_make_y_bcast(hb_poly* const* polys, int nitems, const int32_t* D, int nD, const int32_t* owned, int nOwned,
                         hb_poly* const* ypolys, hb_poly* const* peer_ypolys, int npeers);
/* CUDA IPC export / import of a polynomial's device buffer (one process per GPU; 64-byte handle). */
int hb_poly_ipc_export(hb_poly* p, void* handle64);
int hb_poly_ipc_open(hb_ctx* ctx, const void* handle64, hb_poly** out);
/* Alias caller-owned device memory (uint64[nprimes][N]) as a polynomial; hb_poly_destroy does not free it. */
int hb_poly_wrap(hb_ctx* ctx, void* device_ptr, hb_poly** out);
/* Issue the context's work on a caller-provided CUDA stream (cudaStream_t), e.g. the stream the caller's
 * NCCL collectives are ordered on. */
int hb_ctx_set_stream(hb_ctx* ctx, void* cuda_stream);

/* ---- fused ciphertext-level paths (host orchestration of Ctxt::reLinearize / keySwitchPart,
 * src/Ctxt.cpp:720-842, and Ctxt::multLowLvl + reLinearize + modDownToSet, src/Ctxt.cpp:393-562,
 * 1681-1774) with explicit prime sets (the noise-driven choice stays in the host Ctxt layer).
 * hb_relinearize: (c0,c1,c2) over ctxt primes S  ->  (c0,c1) over S | special   (c2 is consumed). */
int hb_relinearize(hb_poly* const* c0, hb_poly* const* c1, hb_poly* const* c2, int nitems,
                   const int32_t* S, int nS, hb_poly* const* evk_a, hb_poly* const* evk_b, int ndig_evk);
/* hb_mul_relin_moddown: operands (a0,a1),(b0,b1) over S_in; mod-down both to S (ptxt_space),
 * tensor, relinearise over S | special, mod-down the result to S.  Result in (a0,a1) rows S.
 * S is the common set of Ctxt::multiplyBy / multLowLvl (src/Ctxt.cpp:1700-1712) and must be a subset of S_in
 * (HB_ERR_INDEX_SET otherwise).  The 4*nitems operand polys must be distinct (HB_ERR_BAD_ARG before any launch): the
 * product is formed in place, so a ciphertext multiplied by itself needs a copy or hb_square_relin_moddown. */
int hb_mul_relin_moddown(hb_poly* const* a0, hb_poly* const* a1, hb_poly* const* b0, hb_poly* const* b1, int nitems,
                         const int32_t* S_in, int nS_in, const int32_t* S, int nS, uint64_t ptxt_space,
                         hb_poly* const* evk_a, hb_poly* const* evk_b, int ndig_evk);
/* hb_inner_product: innerProduct (src/Ctxt.cpp:2878-2893) of nitems vectors of npairs pairs, the batched form of
 * hb_mul_relin_moddown for sums: pair j of item t is (a0,a1),(b0,b1)[t*npairs + j], over S_in.  When S is a strict subset of
 * S_in every operand part is first brought to S (its rows overwritten, as hb_mul_relin_moddown's operands); then the summed
 * tensor products are relinearised once over S | special into (out0, out1), and with moddown = 1 modded down to S.  No
 * relin_CKKS_adjust (the Ctxt layer applies it).  npairs or nitems <= 0, moddown not 0/1, too few matrix columns, an output
 * aliasing an input, a key or another output, or a seeded handle other than in evk_a -> HB_ERR_BAD_ARG; S not within S_in
 * or not within the ctxt primes, or a seeded evk_a without a needed row -> HB_ERR_INDEX_SET; all checked before any launch.
 * Stream-ordered, no synchronisation; after the first call, a call of the same shape allocates nothing. */
int hb_inner_product(hb_poly* const* a0, hb_poly* const* a1, hb_poly* const* b0, hb_poly* const* b1, int npairs, int nitems,
                     const int32_t* S_in, int nS_in, const int32_t* S, int nS, uint64_t ptxt_space,
                     hb_poly* const* evk_a, hb_poly* const* evk_b, int ndig_evk, hb_poly* const* out0, hb_poly* const* out1, int moddown);
/* hb_square_tensor: the squaring branch of Ctxt::multLowLvl (src/Ctxt.cpp:1704-1708, 1748-1751) for nitems ciphertexts
 * (a0, a1) over S_in: both parts brought to S (bringToSet, S within S_in), then the self-tensor
 *   a0 <- a0^2,   a1 <- 2*a0*a1,   o2 <- a1^2   (mod q, canonical, rows S).
 * hb_square_tensor_norm also returns norms[2i + k] = ||delta/P||_canon of part k of item i, the double hb_scale_down_norm
 * returns for that part (0 when S == S_in).  nitems <= 0, an operand poly given twice, o2 aliasing an operand or another
 * output, a seeded handle, or a null norms -> HB_ERR_BAD_ARG; S not within S_in -> HB_ERR_INDEX_SET; all checked before
 * any launch. */
int hb_square_tensor(hb_poly* const* a0, hb_poly* const* a1, hb_poly* const* o2, int nitems, const int32_t* S_in, int nS_in,
                     const int32_t* S, int nS, uint64_t ptxt_space);
int hb_square_tensor_norm(hb_poly* const* a0, hb_poly* const* a1, hb_poly* const* o2, int nitems, const int32_t* S_in, int nS_in,
                          const int32_t* S, int nS, uint64_t ptxt_space, double* norms);
/* hb_square_relin_moddown: Ctxt::square (multiplyBy(*this)) of nitems ciphertexts, the fixed-set counterpart of
 * hb_mul_relin_moddown: (a0, a1) over S_in are brought to S, squared, relinearised over S | special and modded down to S;
 * the result is in (a0, a1) rows S, bit for bit what hb_mul_relin_moddown(x, copy of x) leaves.  No relin_CKKS_adjust (the
 * Ctxt layer applies it).  Errors as hb_square_tensor, and: no special primes, too few matrix columns, an operand aliasing
 * a key -> HB_ERR_BAD_ARG; S not within the ctxt primes, or a seeded evk_a without a needed row -> HB_ERR_INDEX_SET; all
 * checked before any launch.  Stream-ordered; after the first call, a call of the same shape allocates nothing. */
int hb_square_relin_moddown(hb_poly* const* a0, hb_poly* const* a1, int nitems, const int32_t* S_in, int nS_in,
                            const int32_t* S, int nS, uint64_t ptxt_space, hb_poly* const* evk_a, hb_poly* const* evk_b,
                            int ndig_evk);

#ifdef __cplusplus
}
#endif
#endif /* HELIB_B200_H */
