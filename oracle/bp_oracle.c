/* ORACLE — test infrastructure only.  Only tests/, __graft_entry__.smoke() and bench.py's
 * cpu_baseline / `--impl reference` legs may load this library; the product path never does.
 *
 * A CPU restatement of the Bulletproofs protocol layer of dalek-cryptography/bulletproofs v2.0.0
 * on top of the arithmetic in fe51.h / sc.h / ge.h / hashes.h.  The reference itself cannot be
 * compiled here (pure Rust, nightly-2019-07-31, un-vendored crates; see SURVEY.md section 8c), so
 * parity is pinned by the reference's own golden vectors: the 16 proofs and 8 commitments of
 * tests/range_proof.rs:15-95 (checked by tests/test_oracle_golden.py).
 * Unpinned by fixed vectors in the reference (round-trip tests only there): prover proof bytes,
 * reject side, stand-alone MSM — for those this oracle is "parity unpinned" and says so in DESIGN.md.
 *
 * Reference lines each function follows are cited at the function.
 */
#include <pthread.h>
#include <stdio.h>
#include "ge.h"
#include "hashes.h"

#define ORC_OK 0
#define ORC_VERIFICATION_ERROR 1      /* ProofError::VerificationError      errors.rs:16 */
#define ORC_FORMAT_ERROR 2            /* ProofError::FormatError            errors.rs:19 */
#define ORC_INVALID_BITSIZE 3         /* ProofError::InvalidBitsize         errors.rs:25 */
#define ORC_INVALID_GENS_LENGTH 4     /* ProofError::InvalidGeneratorsLength errors.rs:33 */
#define ORC_INVALID_AGGREGATION 5     /* ProofError::InvalidAggregation     errors.rs:29 */
#define ORC_INVALID_POINT 6           /* optional_multiscalar_mul -> None */
#define ORC_NONCANONICAL_SCALAR 7
#define ORC_MALICIOUS_DEALER 8        /* MPCError::MaliciousDealer party.rs:282-284 */

/* ------------------------------------------------------------------ generators.rs */
typedef struct { ge B, B_blinding; } pedersen_gens;
typedef struct { size_t gens_capacity, party_capacity; ge *G, *H; } bp_gens;   /* [party][i] row-major */

/* PedersenGens::default — generators.rs:44-53 */
static void pedersen_default(pedersen_gens *pc) {
    ge_init_constants();
    pc->B = GE_BASEPOINT;
    uint8_t enc[32], h[64];
    ge_encode(enc, &GE_BASEPOINT);
    sha3_512(h, enc, 32);
    ge_from_uniform_bytes(&pc->B_blinding, h);
}

/* GeneratorsChain::new + Iterator::next — generators.rs:62-104; labels per increase_capacity 179-204 */
static void gens_chain(ge *out, uint8_t tag, uint32_t party, size_t count) {
    sponge s; shake256_init(&s);
    uint8_t label[5] = { tag, (uint8_t)party, (uint8_t)(party >> 8), (uint8_t)(party >> 16), (uint8_t)(party >> 24) };
    sponge_absorb(&s, (const uint8_t *)"GeneratorsChain", 15);
    sponge_absorb(&s, label, 5);
    for (size_t i = 0; i < count; i++) { uint8_t u[64]; sponge_squeeze(&s, u, 64); ge_from_uniform_bytes(&out[i], u); }
}

void *orc_gens_new(size_t gens_capacity, size_t party_capacity) {
    ge_init_constants();
    bp_gens *g = malloc(sizeof *g);
    g->gens_capacity = gens_capacity; g->party_capacity = party_capacity;
    g->G = malloc(sizeof(ge) * gens_capacity * party_capacity);
    g->H = malloc(sizeof(ge) * gens_capacity * party_capacity);
    for (size_t p = 0; p < party_capacity; p++) {
        gens_chain(g->G + p * gens_capacity, 'G', (uint32_t)p, gens_capacity);
        gens_chain(g->H + p * gens_capacity, 'H', (uint32_t)p, gens_capacity);
    }
    return g;
}
void orc_gens_free(void *h) { bp_gens *g = h; free(g->G); free(g->H); free(g); }
void orc_gens_get(void *h, int which, size_t party, size_t idx, uint8_t out[32]) {
    bp_gens *g = h; ge_encode(out, &(which ? g->H : g->G)[party * g->gens_capacity + idx]);
}
void orc_pedersen_gens(uint8_t B[32], uint8_t Bb[32]) { pedersen_gens pc; pedersen_default(&pc); ge_encode(B, &pc.B); ge_encode(Bb, &pc.B_blinding); }
int orc_selfcheck(void) { ge_init_constants(); return ge_check_constants(); }

/* ------------------------------------------------------------------ transcript.rs */
static void t_rangeproof_domain_sep(merlin *t, uint64_t n, uint64_t m) {          /* transcript.rs:44-48 */
    merlin_append(t, "dom-sep", (const uint8_t *)"rangeproof v1", 13);
    merlin_append_u64(t, "n", n); merlin_append_u64(t, "m", m);
}
static void t_innerproduct_domain_sep(merlin *t, uint64_t n) {                      /* transcript.rs:50-53 */
    merlin_append(t, "dom-sep", (const uint8_t *)"ipp v1", 6);
    merlin_append_u64(t, "n", n);
}
static void t_append_scalar(merlin *t, const char *label, const sc *s) { uint8_t b[32]; sc_tobytes(b, s); merlin_append(t, label, b, 32); }
static void t_append_point(merlin *t, const char *label, const uint8_t p[32]) { merlin_append(t, label, p, 32); }
static int t_validate_and_append_point(merlin *t, const char *label, const uint8_t p[32]) {   /* transcript.rs:75-87 */
    uint8_t z = 0; for (int i = 0; i < 32; i++) z |= p[i];
    if (z == 0) return ORC_VERIFICATION_ERROR;
    merlin_append(t, label, p, 32); return ORC_OK;
}
static void t_challenge_scalar(merlin *t, const char *label, sc *out) {           /* transcript.rs:89-94 */
    uint8_t buf[64]; merlin_challenge(t, label, buf, 64); sc_from_bytes_wide(out, buf);
}
static void rng_scalar(chacha_rng *r, sc *out) { uint8_t b[64]; chacha_fill(r, b, 64); sc_from_bytes_wide(out, b); }  /* Scalar::random */

/* exported transcript helpers (opaque state = sizeof(merlin) <= 208 bytes) */
void orc_transcript_new(uint8_t *state, const uint8_t *label, size_t len) { merlin m; merlin_init(&m, label, len); memcpy(state, &m, sizeof m); }
void orc_transcript_append(uint8_t *state, const char *label, const uint8_t *msg, size_t len) { merlin m; memcpy(&m, state, sizeof m); merlin_append(&m, label, msg, len); memcpy(state, &m, sizeof m); }
void orc_transcript_challenge(uint8_t *state, const char *label, uint8_t *out, size_t len) { merlin m; memcpy(&m, state, sizeof m); merlin_challenge(&m, label, out, len); memcpy(state, &m, sizeof m); }
size_t orc_transcript_size(void) { return sizeof(merlin); }

/* ------------------------------------------------------------------ util.rs */
static void sc_one(sc *r) { sc_from_u64(r, 1); }
static void inner_product(sc *out, const sc *a, const sc *b, size_t n) {           /* inner_product_proof.rs:418-427 */
    sc acc, t; sc_zero(&acc);
    for (size_t i = 0; i < n; i++) { sc_mul(&t, &a[i], &b[i]); sc_add(&acc, &acc, &t); }
    *out = acc;
}
static void scalar_exp_vartime(sc *out, const sc *x, uint64_t n) {                 /* util.rs:222-234 */
    sc result, aux = *x; sc_one(&result);
    while (n > 0) { if (n & 1) sc_mul(&result, &result, &aux); n >>= 1; sc_mul(&aux, &aux, &aux); }
    *out = result;
}
static void sum_of_powers(sc *out, const sc *x, size_t n) {                        /* util.rs:240-262 */
    if (n & (n - 1)) { sc acc, p; sc_zero(&acc); sc_one(&p); for (size_t i = 0; i < n; i++) { sc_add(&acc, &acc, &p); sc_mul(&p, &p, x); } *out = acc; return; }
    if (n == 0 || n == 1) { sc_from_u64(out, n); return; }
    size_t m = n; sc result, factor = *x, t; sc_one(&result); sc_add(&result, &result, x);
    while (m > 2) { sc_mul(&factor, &factor, &factor); sc_mul(&t, &factor, &result); sc_add(&result, &result, &t); m /= 2; }
    *out = result;
}
/* delta(y,z) — range_proof/mod.rs:587-593 */
static void rp_delta(sc *out, size_t n, size_t m, const sc *y, const sc *z) {
    sc sum_y, sum_2, sum_z, two, zz, t, u;
    sc_from_u64(&two, 2);
    sum_of_powers(&sum_y, y, n * m); sum_of_powers(&sum_2, &two, n); sum_of_powers(&sum_z, z, m);
    sc_mul(&zz, z, z); sc_sub(&t, z, &zz); sc_mul(&t, &t, &sum_y);
    sc_mul(&u, &zz, z); sc_mul(&u, &u, &sum_2); sc_mul(&u, &u, &sum_z);
    sc_sub(out, &t, &u);
}

/* ------------------------------------------------------------------ inner_product_proof.rs */
static int is_pow2(size_t n) { return n && !(n & (n - 1)); }
static int lg2(size_t n) { int k = 0; while (((size_t)1 << k) < n) k++; return k; }

/* InnerProductProof::create — inner_product_proof.rs:38-193.  G,H,a,b are consumed (mutated).
 * Writes L_0,R_0,...,L_{k-1},R_{k-1},a,b (the to_bytes layout, :341-350) into out. */
static void ipp_create(merlin *t, const ge *Q, const sc *Gf, const sc *Hf, ge *G, ge *H, sc *a, sc *b, size_t n, uint8_t *out) {
    t_innerproduct_domain_sep(t, n);
    int first = 1; size_t round = 0;
    sc *ms = malloc(sizeof(sc) * (2 * n + 1)); ge *mp = malloc(sizeof(ge) * (2 * n + 1));
    while (n != 1) {
        n /= 2;
        sc *aL = a, *aR = a + n, *bL = b, *bR = b + n; ge *GL = G, *GR = G + n, *HL = H, *HR = H + n;
        sc cL, cR; inner_product(&cL, aL, bR, n); inner_product(&cR, aR, bL, n);
        ge Lp, Rp; uint8_t Lc[32], Rc[32];
        /* L = <a_L*g_R, G_R> + <b_R*h_L, H_L> + c_L Q   (:87-99 with factors, :153-157 without) */
        for (size_t i = 0; i < n; i++) {
            if (first) { sc_mul(&ms[i], &aL[i], &Gf[n + i]); sc_mul(&ms[n + i], &bR[i], &Hf[i]); } else { ms[i] = aL[i]; ms[n + i] = bR[i]; }
            mp[i] = GR[i]; mp[n + i] = HL[i];
        }
        ms[2 * n] = cL; mp[2 * n] = *Q;
        ge_msm_vartime(&Lp, ms, mp, 2 * n + 1); ge_encode(Lc, &Lp);
        /* R = <a_R*g_L, G_L> + <b_L*h_R, H_R> + c_R Q   (:101-113 / :159-163) */
        for (size_t i = 0; i < n; i++) {
            if (first) { sc_mul(&ms[i], &aR[i], &Gf[i]); sc_mul(&ms[n + i], &bL[i], &Hf[n + i]); } else { ms[i] = aR[i]; ms[n + i] = bL[i]; }
            mp[i] = GL[i]; mp[n + i] = HR[i];
        }
        ms[2 * n] = cR; mp[2 * n] = *Q;
        ge_msm_vartime(&Rp, ms, mp, 2 * n + 1); ge_encode(Rc, &Rp);
        memcpy(out + 64 * round, Lc, 32); memcpy(out + 64 * round + 32, Rc, 32); round++;
        t_append_point(t, "L", Lc); t_append_point(t, "R", Rc);
        sc u, ui; t_challenge_scalar(t, "u", &u); sc_invert(&ui, &u);
        for (size_t i = 0; i < n; i++) {                                             /* :124-135 / :174-179 */
            sc x, y2;
            sc_mul(&x, &aL[i], &u); sc_mul(&y2, &ui, &aR[i]); sc_add(&aL[i], &x, &y2);
            sc_mul(&x, &bL[i], &ui); sc_mul(&y2, &u, &bR[i]); sc_add(&bL[i], &x, &y2);
            sc s2[2]; ge p2[2], r;
            if (first) { sc_mul(&s2[0], &ui, &Gf[i]); sc_mul(&s2[1], &u, &Gf[n + i]); } else { s2[0] = ui; s2[1] = u; }
            p2[0] = GL[i]; p2[1] = GR[i]; ge_msm_vartime(&r, s2, p2, 2); GL[i] = r;
            if (first) { sc_mul(&s2[0], &u, &Hf[i]); sc_mul(&s2[1], &ui, &Hf[n + i]); } else { s2[0] = u; s2[1] = ui; }
            p2[0] = HL[i]; p2[1] = HR[i]; ge_msm_vartime(&r, s2, p2, 2); HL[i] = r;
        }
        first = 0;
    }
    sc_tobytes(out + 64 * round, &a[0]); sc_tobytes(out + 64 * round + 32, &b[0]);
    free(ms); free(mp);
}

typedef struct { int lg_n; const uint8_t *LR; sc a, b; } ipp_view;   /* LR: L_0,R_0,L_1,R_1,... */

/* InnerProductProof::from_bytes — inner_product_proof.rs:374-407 */
static int ipp_from_bytes(ipp_view *p, const uint8_t *s, size_t len) {
    if (len % 32) return ORC_FORMAT_ERROR;
    size_t ne = len / 32;
    if (ne < 2 || (ne - 2) % 2) return ORC_FORMAT_ERROR;
    size_t lg = (ne - 2) / 2;
    if (lg >= 32) return ORC_FORMAT_ERROR;
    p->lg_n = (int)lg; p->LR = s;
    if (!sc_from_canonical(&p->a, s + 64 * lg) || !sc_from_canonical(&p->b, s + 64 * lg + 32)) return ORC_FORMAT_ERROR;
    return ORC_OK;
}

/* InnerProductProof::verification_scalars — inner_product_proof.rs:198-253.
 * u_sq, u_inv_sq have lg_n entries, s has n entries. */
static int ipp_verification_scalars(const ipp_view *p, size_t n, merlin *t, sc *u_sq, sc *u_inv_sq, sc *s) {
    int lg_n = p->lg_n;
    if (lg_n >= 32) return ORC_VERIFICATION_ERROR;
    if (n != ((size_t)1 << lg_n)) return ORC_VERIFICATION_ERROR;
    t_innerproduct_domain_sep(t, n);
    sc ch[32], chi[32], allinv;
    for (int i = 0; i < lg_n; i++) {
        if (t_validate_and_append_point(t, "L", p->LR + 64 * i)) return ORC_VERIFICATION_ERROR;
        if (t_validate_and_append_point(t, "R", p->LR + 64 * i + 32)) return ORC_VERIFICATION_ERROR;
        t_challenge_scalar(t, "u", &ch[i]);
    }
    /* Scalar::batch_invert: each inverse + product of all inverses (:226-227), one field inversion (Montgomery's trick) */
    { sc pre[33], inv; sc_one(&pre[0]);
      for (int i = 0; i < lg_n; i++) sc_mul(&pre[i + 1], &pre[i], &ch[i]);
      sc_invert(&inv, &pre[lg_n]); allinv = inv;
      for (int i = lg_n - 1; i >= 0; i--) { sc_mul(&chi[i], &inv, &pre[i]); sc_mul(&inv, &inv, &ch[i]); } }
    for (int i = 0; i < lg_n; i++) { sc_mul(&u_sq[i], &ch[i], &ch[i]); sc_mul(&u_inv_sq[i], &chi[i], &chi[i]); }
    s[0] = allinv;
    for (size_t i = 1; i < n; i++) {
        int lg_i = 63 - __builtin_clzll((unsigned long long)i);
        size_t k = (size_t)1 << lg_i;
        sc_mul(&s[i], &s[i - k], &u_sq[(lg_n - 1) - lg_i]);
    }
    return ORC_OK;
}

/* InnerProductProof::verify — inner_product_proof.rs:260-326 */
static int ipp_verify(const ipp_view *p, size_t n, merlin *t, const sc *Gf, const sc *Hf, const ge *P, const ge *Q, const ge *G, const ge *H) {
    int k = p->lg_n;
    sc *s = malloc(sizeof(sc) * (n ? n : 1)); sc u_sq[32], u_inv_sq[32];
    int rc = ipp_verification_scalars(p, n, t, u_sq, u_inv_sq, s);
    if (rc) { free(s); return rc; }
    size_t nt = 1 + 2 * n + 2 * (size_t)k;
    sc *ms = malloc(sizeof(sc) * nt); ge *mp = malloc(sizeof(ge) * nt);
    sc_mul(&ms[0], &p->a, &p->b); mp[0] = *Q;
    for (size_t i = 0; i < n; i++) {
        sc x; sc_mul(&x, &p->a, &s[i]); sc_mul(&ms[1 + i], &x, &Gf[i]); mp[1 + i] = G[i];
        sc_mul(&x, &p->b, &s[n - 1 - i]); sc_mul(&ms[1 + n + i], &x, &Hf[i]); mp[1 + n + i] = H[i];
    }
    rc = ORC_OK;
    for (int i = 0; i < k; i++) {
        sc_neg(&ms[1 + 2 * n + i], &u_sq[i]); sc_neg(&ms[1 + 2 * n + k + i], &u_inv_sq[i]);
        if (!ge_decode(&mp[1 + 2 * n + i], p->LR + 64 * i) || !ge_decode(&mp[1 + 2 * n + k + i], p->LR + 64 * i + 32)) { rc = ORC_VERIFICATION_ERROR; break; }
    }
    if (!rc) { ge expect; ge_msm_vartime(&expect, ms, mp, nt); if (!ge_ristretto_eq(&expect, P)) rc = ORC_VERIFICATION_ERROR; }
    free(s); free(ms); free(mp);
    return rc;
}

/* ------------------------------------------------------------------ range_proof */
static int valid_bitsize(size_t n) { return n == 8 || n == 16 || n == 32 || n == 64; }

/* RangeProof::verify_multiple_with_rng — range_proof/mod.rs:345-452; from_bytes 497-538 */
/* the (scalar, point) terms of the mega-check in the reference's order (mod.rs:421-445): A, S, T_1, T_2, L.., R.., B~, B, G.., H.., V..;
 * *ms_out / *mp_out are malloc'ed (4 + 2k + 2 + 2N + m entries) when the return value is ORC_OK */
static int rp_verify_terms(const bp_gens *bg, const pedersen_gens *pc, merlin *t, const uint8_t *proof, size_t plen,
                           const uint8_t *V, size_t m, size_t n, chacha_rng *rng, sc **ms_out, ge **mp_out, size_t *nt_out, int *k_out) {
    if (plen % 32 || plen < 7 * 32) return ORC_FORMAT_ERROR;
    const uint8_t *A = proof, *S = proof + 32, *T1 = proof + 64, *T2 = proof + 96;
    sc t_x, t_x_bl, e_bl;
    if (!sc_from_canonical(&t_x, proof + 128) || !sc_from_canonical(&t_x_bl, proof + 160) || !sc_from_canonical(&e_bl, proof + 192)) return ORC_FORMAT_ERROR;
    ipp_view ipp; int rc = ipp_from_bytes(&ipp, proof + 224, plen - 224); if (rc) return rc;

    if (!valid_bitsize(n)) return ORC_INVALID_BITSIZE;
    if (bg->gens_capacity < n || bg->party_capacity < m) return ORC_INVALID_GENS_LENGTH;
    t_rangeproof_domain_sep(t, n, m);
    for (size_t j = 0; j < m; j++) t_append_point(t, "V", V + 32 * j);
    if (t_validate_and_append_point(t, "A", A) || t_validate_and_append_point(t, "S", S)) return ORC_VERIFICATION_ERROR;
    sc y, z, zz, minus_z, x, w, c;
    t_challenge_scalar(t, "y", &y); t_challenge_scalar(t, "z", &z);
    sc_mul(&zz, &z, &z); sc_neg(&minus_z, &z);
    if (t_validate_and_append_point(t, "T_1", T1) || t_validate_and_append_point(t, "T_2", T2)) return ORC_VERIFICATION_ERROR;
    t_challenge_scalar(t, "x", &x);
    t_append_scalar(t, "t_x", &t_x); t_append_scalar(t, "t_x_blinding", &t_x_bl); t_append_scalar(t, "e_blinding", &e_bl);
    t_challenge_scalar(t, "w", &w);
    rng_scalar(rng, &c);                                                               /* :396 */

    size_t N = n * m; int k = ipp.lg_n;
    sc *s = malloc(sizeof(sc) * (N ? N : 1)); sc u_sq[32], u_inv_sq[32];
    rc = ipp_verification_scalars(&ipp, N, t, u_sq, u_inv_sq, s);
    if (rc) { free(s); return rc; }
    size_t nt = 4 + 2 * (size_t)k + 2 + 2 * N + m;
    sc *ms = malloc(sizeof(sc) * nt); ge *mp = malloc(sizeof(ge) * nt);
    size_t o = 0; int bad = 0;
    sc cx; sc_mul(&cx, &c, &x);
    sc_one(&ms[0]); ms[1] = x; ms[2] = cx; sc_mul(&ms[3], &cx, &x);
    bad |= !ge_decode(&mp[0], A); bad |= !ge_decode(&mp[1], S); bad |= !ge_decode(&mp[2], T1); bad |= !ge_decode(&mp[3], T2);
    o = 4;
    for (int i = 0; i < k; i++) { ms[o + i] = u_sq[i]; bad |= !ge_decode(&mp[o + i], ipp.LR + 64 * i); }
    o += k;
    for (int i = 0; i < k; i++) { ms[o + i] = u_inv_sq[i]; bad |= !ge_decode(&mp[o + i], ipp.LR + 64 * i + 32); }
    o += k;
    { sc tt; sc_mul(&tt, &c, &t_x_bl); sc_add(&tt, &tt, &e_bl); sc_neg(&ms[o], &tt); mp[o] = pc->B_blinding; o++; }      /* -e~ - c t~ */
    { sc ab, d, t1, t2; sc_mul(&ab, &ipp.a, &ipp.b); sc_sub(&t1, &t_x, &ab); sc_mul(&t1, &w, &t1);
      rp_delta(&d, n, m, &y, &z); sc_sub(&t2, &d, &t_x); sc_mul(&t2, &c, &t2); sc_add(&ms[o], &t1, &t2); mp[o] = pc->B; o++; }
    /* g_i = -z - a s_i  (:415);  h_i = z + y^-i (zz z^j 2^i' - b s_{N-1-i})  (:416-419) */
    sc y_inv, exp_y_inv, exp_z, exp_2; sc_invert(&y_inv, &y); sc_one(&exp_y_inv); sc_one(&exp_z);
    for (size_t i = 0; i < N; i++) { sc tt; sc_mul(&tt, &ipp.a, &s[i]); sc_sub(&ms[o + i], &minus_z, &tt); mp[o + i] = bg->G[(i / n) * bg->gens_capacity + (i % n)]; }
    o += N;
    for (size_t j = 0; j < m; j++) {
        sc_one(&exp_2);
        for (size_t i = 0; i < n; i++) {
            size_t idx = j * n + i; sc z2, t1, t2;
            sc_mul(&z2, &exp_2, &exp_z);                    /* concat_z_and_2 */
            sc_mul(&t1, &zz, &z2); sc_mul(&t2, &ipp.b, &s[N - 1 - idx]); sc_sub(&t1, &t1, &t2);
            sc_mul(&t1, &exp_y_inv, &t1); sc_add(&ms[o + idx], &z, &t1);
            mp[o + idx] = bg->H[j * bg->gens_capacity + i];
            sc_mul(&exp_y_inv, &exp_y_inv, &y_inv); sc_add(&exp_2, &exp_2, &exp_2);
        }
        sc_mul(&exp_z, &exp_z, &z);
    }
    o += N;
    sc_one(&exp_z);
    for (size_t j = 0; j < m; j++) { sc tt; sc_mul(&tt, &c, &zz); sc_mul(&ms[o + j], &tt, &exp_z); bad |= !ge_decode(&mp[o + j], V + 32 * j); sc_mul(&exp_z, &exp_z, &z); }
    o += m;
    free(s);
    if (bad) { free(ms); free(mp); return ORC_VERIFICATION_ERROR; }                    /* :445 */
    *ms_out = ms; *mp_out = mp; *nt_out = nt; *k_out = k;
    return ORC_OK;
}
/* RangeProof::verify_multiple_with_rng — range_proof/mod.rs:345-452; from_bytes 497-538 */
static int rp_verify(const bp_gens *bg, const pedersen_gens *pc, merlin *t, const uint8_t *proof, size_t plen,
                     const uint8_t *V, size_t m, size_t n, chacha_rng *rng) {
    sc *ms; ge *mp; size_t nt; int k;
    int rc = rp_verify_terms(bg, pc, t, proof, plen, V, m, n, rng, &ms, &mp, &nt, &k);
    if (rc) return rc;
    ge mega; ge_msm_vartime(&mega, ms, mp, nt); if (!ge_is_identity(&mega)) rc = ORC_VERIFICATION_ERROR;   /* :447-451 */
    free(ms); free(mp);
    return rc;
}
/* Random-linear-combination batch on the CPU (SURVEY.md section 8a row A6 -- the reference has no batch verifier; this is the
 * apples-to-apples CPU line next to the GPU engine's batch path): every proof's mega-check is multiplied by its own random
 * 128-bit weight, the weighted scalars of the shared points B~, B, G.., H.. are summed, and ONE variable-time MSM over
 * 2 + 2N + count*(4 + 2k + m) terms (Pippenger, the dependency's dispatch) must give the identity.  Returns 1 when the whole
 * chunk is accepted, 0 when some proof is malformed or the combination does not vanish (callers then verify proof by proof). */
static int rp_verify_rlc_chunk(const bp_gens *bg, const pedersen_gens *pc, const uint8_t *tstate, const uint8_t *proofs, size_t plen,
                               const uint8_t *Vs, size_t m, size_t n, size_t count, chacha_rng *rng) {
    size_t N = n * m, S = 2 + 2 * N, cap = S, used = S;
    sc *as = calloc(S, sizeof(sc)); ge *ap = malloc(S * sizeof(ge));
    int ok = 1, have_static = 0;
    for (size_t i = 0; i < count && ok; i++) {
        merlin t; memcpy(&t, tstate, sizeof t);
        sc *ms; ge *mp; size_t nt; int k;
        if (rp_verify_terms(bg, pc, &t, proofs + i * plen, plen, Vs + 32 * m * i, m, n, rng, &ms, &mp, &nt, &k)) { ok = 0; break; }
        size_t D = 4 + 2 * (size_t)k + m, so = 4 + 2 * (size_t)k;       /* static block starts after A,S,T1,T2,L..,R.. */
        uint8_t wb[32] = {0}; chacha_fill(rng, wb, 16); wb[0] |= 1;       /* 128-bit non-zero weight */
        sc rho; sc_from_bytes_mod_order(&rho, wb);
        if (used + D > cap) { cap = 2 * cap + D; as = realloc(as, cap * sizeof(sc)); ap = realloc(ap, cap * sizeof(ge)); }
        if (!have_static) { for (size_t j = 0; j < S; j++) ap[j] = mp[so + j]; have_static = 1; }
        for (size_t j = 0; j < S; j++) { sc w; sc_mul(&w, &rho, &ms[so + j]); sc_add(&as[j], &as[j], &w); }
        for (size_t j = 0; j < so; j++) { sc_mul(&as[used], &rho, &ms[j]); ap[used++] = mp[j]; }
        for (size_t j = 0; j < m; j++) { sc_mul(&as[used], &rho, &ms[so + S + j]); ap[used++] = mp[so + S + j]; }
        free(ms); free(mp);
    }
    if (ok) { ge mega; ge_msm_vartime(&mega, as, ap, used); ok = ge_is_identity(&mega); }
    free(as); free(ap);
    return ok;
}

/* RangeProof::prove_multiple_with_rng — range_proof/mod.rs:234-288, restating the single-process
 * run of the MPC: party.rs:37-61,87-144,182-237,279-305 and dealer.rs:37-81,98-137,160-197,226-293. */
static int rp_prove(const bp_gens *bg, const pedersen_gens *pc, merlin *t, const uint64_t *values, const uint8_t *blindings,
                    size_t m, size_t n, chacha_rng *rng, uint8_t *proof_out, uint8_t *V_out) {
    if (!valid_bitsize(n)) return ORC_INVALID_BITSIZE;
    if (!is_pow2(m)) return ORC_INVALID_AGGREGATION;
    if (bg->gens_capacity < n || bg->party_capacity < m) return ORC_INVALID_GENS_LENGTH;
    size_t N = n * m; int k = lg2(N);
    sc *vb = malloc(sizeof(sc) * m), *a_bl = malloc(sizeof(sc) * m), *s_bl = malloc(sizeof(sc) * m);
    sc *sL = malloc(sizeof(sc) * N), *sR = malloc(sizeof(sc) * N);
    sc *l0 = malloc(sizeof(sc) * N), *l1 = malloc(sizeof(sc) * N), *r0 = malloc(sizeof(sc) * N), *r1 = malloc(sizeof(sc) * N);
    sc *t1b = malloc(sizeof(sc) * m), *t2b = malloc(sizeof(sc) * m), *ozz = malloc(sizeof(sc) * m);
    sc (*tp)[3] = malloc(sizeof(sc) * 3 * m);
    for (size_t j = 0; j < m; j++) if (!sc_from_canonical(&vb[j], blindings + 32 * j)) sc_from_bytes_mod_order(&vb[j], blindings + 32 * j);

    t_rangeproof_domain_sep(t, n, m);                                                  /* dealer.rs:70 */
    ge A, S; ge_identity(&A); ge_identity(&S);
    for (size_t j = 0; j < m; j++) {
        const ge *Gj = bg->G + j * bg->gens_capacity, *Hj = bg->H + j * bg->gens_capacity;
        ge Vp, tmp; sc v; sc_from_u64(&v, values[j]);
        { sc s2[2] = { v, vb[j] }; ge p2[2] = { pc->B, pc->B_blinding }; ge_msm_vartime(&Vp, s2, p2, 2); }   /* party.rs:51 */
        ge_encode(V_out + 32 * j, &Vp);
        rng_scalar(rng, &a_bl[j]);                                                     /* party.rs:98 */
        ge Aj; ge_scalarmult(&Aj, &a_bl[j], &pc->B_blinding);
        for (size_t i = 0; i < n; i++) {                                               /* party.rs:100-112 */
            if ((values[j] >> i) & 1) ge_add(&Aj, &Aj, &Gj[i]); else ge_sub(&Aj, &Aj, &Hj[i]);
        }
        rng_scalar(rng, &s_bl[j]);                                                     /* party.rs:114-116 */
        for (size_t i = 0; i < n; i++) rng_scalar(rng, &sL[j * n + i]);
        for (size_t i = 0; i < n; i++) rng_scalar(rng, &sR[j * n + i]);
        sc *ms = malloc(sizeof(sc) * (2 * n + 1)); ge *mp = malloc(sizeof(ge) * (2 * n + 1));     /* party.rs:119-124 */
        ms[0] = s_bl[j]; mp[0] = pc->B_blinding;
        for (size_t i = 0; i < n; i++) { ms[1 + i] = sL[j * n + i]; mp[1 + i] = Gj[i]; ms[1 + n + i] = sR[j * n + i]; mp[1 + n + i] = Hj[i]; }
        ge_msm_vartime(&tmp, ms, mp, 2 * n + 1);
        free(ms); free(mp);
        ge_add(&A, &A, &Aj); ge_add(&S, &S, &tmp);                                     /* dealer.rs:112-116 */
    }
    uint8_t Ac[32], Sc[32], T1c[32], T2c[32];
    for (size_t j = 0; j < m; j++) t_append_point(t, "V", V_out + 32 * j);             /* dealer.rs:107-109 */
    ge_encode(Ac, &A); ge_encode(Sc, &S); t_append_point(t, "A", Ac); t_append_point(t, "S", Sc);
    sc y, z, zz; t_challenge_scalar(t, "y", &y); t_challenge_scalar(t, "z", &z); sc_mul(&zz, &z, &z);

    ge T1, T2; ge_identity(&T1); ge_identity(&T2);
    sc one; sc_one(&one);
    for (size_t j = 0; j < m; j++) {                                                   /* party.rs:182-237 */
        sc offset_y, offset_z, exp_y, exp_2;
        scalar_exp_vartime(&offset_y, &y, (uint64_t)(j * n)); scalar_exp_vartime(&offset_z, &z, (uint64_t)j);
        sc_mul(&ozz[j], &zz, &offset_z); exp_y = offset_y; sc_one(&exp_2);
        for (size_t i = 0; i < n; i++) {
            size_t idx = j * n + i; sc aL, aR, t1, t2;
            sc_from_u64(&aL, (values[j] >> i) & 1); sc_sub(&aR, &aL, &one);
            sc_sub(&l0[idx], &aL, &z); l1[idx] = sL[idx];
            sc_add(&t1, &aR, &z); sc_mul(&t1, &exp_y, &t1); sc_mul(&t2, &ozz[j], &exp_2); sc_add(&r0[idx], &t1, &t2);
            sc_mul(&r1[idx], &exp_y, &sR[idx]);
            sc_mul(&exp_y, &exp_y, &y); sc_add(&exp_2, &exp_2, &exp_2);
        }
        /* VecPoly1::inner_product (Karatsuba) — util.rs:86-100 */
        sc t0, t2, t1, lsum, rsum, acc; inner_product(&t0, l0 + j * n, r0 + j * n, n); inner_product(&t2, l1 + j * n, r1 + j * n, n);
        sc_zero(&acc);
        for (size_t i = 0; i < n; i++) { sc pr; sc_add(&lsum, &l0[j * n + i], &l1[j * n + i]); sc_add(&rsum, &r0[j * n + i], &r1[j * n + i]); sc_mul(&pr, &lsum, &rsum); sc_add(&acc, &acc, &pr); }
        sc_sub(&t1, &acc, &t0); sc_sub(&t1, &t1, &t2);
        tp[j][0] = t0; tp[j][1] = t1; tp[j][2] = t2;
        rng_scalar(rng, &t1b[j]); rng_scalar(rng, &t2b[j]);                            /* party.rs:214-215 */
        ge T1j, T2j;
        { sc s2[2] = { t1, t1b[j] }; ge p2[2] = { pc->B, pc->B_blinding }; ge_msm_vartime(&T1j, s2, p2, 2); }
        { sc s2[2] = { t2, t2b[j] }; ge p2[2] = { pc->B, pc->B_blinding }; ge_msm_vartime(&T2j, s2, p2, 2); }
        ge_add(&T1, &T1, &T1j); ge_add(&T2, &T2, &T2j);                                /* dealer.rs:169-170 */
    }
    ge_encode(T1c, &T1); ge_encode(T2c, &T2); t_append_point(t, "T_1", T1c); t_append_point(t, "T_2", T2c);
    sc x; t_challenge_scalar(t, "x", &x);
    int rc = ORC_OK;
    if (sc_is_zero(&x)) rc = ORC_MALICIOUS_DEALER;                                     /* party.rs:282-284 */
    sc t_x, t_x_bl, e_bl; sc_zero(&t_x); sc_zero(&t_x_bl); sc_zero(&e_bl);
    sc *lv = malloc(sizeof(sc) * N), *rv = malloc(sizeof(sc) * N);
    for (size_t j = 0; j < m && !rc; j++) {                                            /* party.rs:279-305, dealer.rs:245-247 */
        sc e, u;
        sc_mul(&e, &x, &tp[j][2]); sc_add(&e, &e, &tp[j][1]); sc_mul(&e, &x, &e); sc_add(&e, &e, &tp[j][0]); sc_add(&t_x, &t_x, &e);
        sc_mul(&u, &ozz[j], &vb[j]);
        sc_mul(&e, &x, &t2b[j]); sc_add(&e, &e, &t1b[j]); sc_mul(&e, &x, &e); sc_add(&e, &e, &u); sc_add(&t_x_bl, &t_x_bl, &e);
        sc_mul(&e, &s_bl[j], &x); sc_add(&e, &e, &a_bl[j]); sc_add(&e_bl, &e_bl, &e);
        for (size_t i = 0; i < n; i++) { size_t idx = j * n + i; sc q; sc_mul(&q, &l1[idx], &x); sc_add(&lv[idx], &l0[idx], &q); sc_mul(&q, &r1[idx], &x); sc_add(&rv[idx], &r0[idx], &q); }
    }
    if (!rc) {
        t_append_scalar(t, "t_x", &t_x); t_append_scalar(t, "t_x_blinding", &t_x_bl); t_append_scalar(t, "e_blinding", &e_bl);
        sc w; t_challenge_scalar(t, "w", &w);
        ge Q; ge_scalarmult(&Q, &w, &pc->B);                                            /* dealer.rs:256 */
        sc *Gf = malloc(sizeof(sc) * N), *Hf = malloc(sizeof(sc) * N); sc y_inv, e; sc_invert(&y_inv, &y); sc_one(&e);
        for (size_t i = 0; i < N; i++) { sc_one(&Gf[i]); Hf[i] = e; sc_mul(&e, &e, &y_inv); }
        ge *G = malloc(sizeof(ge) * N), *H = malloc(sizeof(ge) * N);
        for (size_t i = 0; i < N; i++) { G[i] = bg->G[(i / n) * bg->gens_capacity + (i % n)]; H[i] = bg->H[(i / n) * bg->gens_capacity + (i % n)]; }
        memcpy(proof_out, Ac, 32); memcpy(proof_out + 32, Sc, 32); memcpy(proof_out + 64, T1c, 32); memcpy(proof_out + 96, T2c, 32);
        sc_tobytes(proof_out + 128, &t_x); sc_tobytes(proof_out + 160, &t_x_bl); sc_tobytes(proof_out + 192, &e_bl);
        ipp_create(t, &Q, Gf, Hf, G, H, lv, rv, N, proof_out + 224);
        free(Gf); free(Hf); free(G); free(H);
    }
    (void)k;
    free(vb); free(a_bl); free(s_bl); free(sL); free(sR); free(l0); free(l1); free(r0); free(r1); free(t1b); free(t2b); free(ozz); free(tp); free(lv); free(rv);
    return rc;
}

/* ------------------------------------------------------------------ exported protocol entry points */
static pedersen_gens g_pc; static int g_pc_ready = 0;
static const pedersen_gens *default_pc(void) { if (!g_pc_ready) { pedersen_default(&g_pc); g_pc_ready = 1; } return &g_pc; }
/* MSM backends: "u64" (serial 51-bit limbs, ge.h), "avx2", "ifma" (4-way vector, vec4_*.h), "auto" = fastest the CPU supports.
 * Returns 0, or -1 when the CPU lacks the instructions.  Not thread-safe: call before starting worker threads. */
void orc_vec_msm_avx2(ge *out, const sc *scalars, const ge *points, size_t n);
void orc_vec_msm_ifma(ge *out, const sc *scalars, const ge *points, size_t n);
int orc_vec_selftest_avx2(const uint8_t *pts, const uint8_t *rnd);
int orc_vec_selftest_ifma(const uint8_t *pts, const uint8_t *rnd);
const char *orc_vec_name_avx2(void);
const char *orc_vec_name_ifma(void);
static const char *g_backend_name = "u64 (5x 51-bit limbs, serial)";
static int cpu_has_avx2(void) { __builtin_cpu_init(); return __builtin_cpu_supports("avx2"); }
static int cpu_has_ifma(void) { __builtin_cpu_init(); return __builtin_cpu_supports("avx512ifma") && __builtin_cpu_supports("avx512vl") && __builtin_cpu_supports("avx2"); }
int orc_set_backend(const char *name) {
    ge_init_constants();
    ge one[1]; sc s1[1]; ge tmp; ge_identity(&one[0]); memset(s1, 0, sizeof s1);
    if (!strcmp(name, "auto")) name = cpu_has_ifma() ? "ifma" : cpu_has_avx2() ? "avx2" : "u64";
    if (!strcmp(name, "u64")) { ge_msm_backend = NULL; g_backend_name = "u64 (5x 51-bit limbs, serial)"; return 0; }
    if (!strcmp(name, "avx2")) { if (!cpu_has_avx2()) return -1; orc_vec_msm_avx2(&tmp, s1, one, 1); ge_msm_backend = orc_vec_msm_avx2; g_backend_name = orc_vec_name_avx2(); return 0; }
    if (!strcmp(name, "ifma")) { if (!cpu_has_ifma()) return -1; orc_vec_msm_ifma(&tmp, s1, one, 1); ge_msm_backend = orc_vec_msm_ifma; g_backend_name = orc_vec_name_ifma(); return 0; }
    return -2;
}
const char *orc_backend_name(void) { return g_backend_name; }
int orc_vec_selftest(const char *name, const uint8_t *pts, const uint8_t *rnd) {
    if (!strcmp(name, "avx2")) return cpu_has_avx2() ? orc_vec_selftest_avx2(pts, rnd) : -1;
    if (!strcmp(name, "ifma")) return cpu_has_ifma() ? orc_vec_selftest_ifma(pts, rnd) : -1;
    return -2;
}
void orc_init(void) { ge_init_constants(); default_pc(); }

int orc_rangeproof_verify(void *gens, const uint8_t *transcript_state, const uint8_t *proof, size_t plen,
                          const uint8_t *V, size_t m, size_t n, const uint8_t rng_seed[32]) {
    merlin t; memcpy(&t, transcript_state, sizeof t);
    chacha_rng rng; chacha_seed(&rng, rng_seed);
    return rp_verify(gens, default_pc(), &t, proof, plen, V, m, n, &rng);
}
int orc_rangeproof_prove(void *gens, const uint8_t *transcript_state, const uint64_t *values, const uint8_t *blindings,
                         size_t m, size_t n, const uint8_t rng_seed[32], uint8_t *proof_out, uint8_t *V_out) {
    merlin t; memcpy(&t, transcript_state, sizeof t);
    chacha_rng rng; chacha_seed(&rng, rng_seed);
    return rp_prove(gens, default_pc(), &t, values, blindings, m, n, &rng, proof_out, V_out);
}
/* ------------------------------------------------------------------ aggregated range-proof MPC messages (party.rs, dealer.rs, messages.rs) */
#include "mpc.h"
static int load_sc(sc *r, const uint8_t b[32]) { return sc_from_canonical(r, b); }
int orc_mpc_party_bit_commitment(void *gens, uint64_t v, const uint8_t v_blinding[32], size_t n, size_t j, const uint8_t seed[32], uint8_t out[96]) {
    sc vb; if (!load_sc(&vb, v_blinding)) return ORC_NONCANONICAL_SCALAR;
    return mpc_party_bit_commitment(gens, default_pc(), v, &vb, n, j, seed, out);
}
int orc_mpc_party_poly_commitment(void *gens, uint64_t v, size_t n, size_t j, const uint8_t seed[32], const uint8_t y[32], const uint8_t z[32], uint8_t out[64]) {
    sc ys, zs; if (!load_sc(&ys, y) || !load_sc(&zs, z)) return ORC_NONCANONICAL_SCALAR;
    return mpc_party_poly_commitment(gens, default_pc(), v, n, j, seed, &ys, &zs, out);
}
int orc_mpc_party_proof_share(void *gens, uint64_t v, const uint8_t v_blinding[32], size_t n, size_t j, const uint8_t seed[32], const uint8_t y[32], const uint8_t z[32],
                              const uint8_t x[32], uint8_t *out) {
    sc vb, ys, zs, xs; if (!load_sc(&vb, v_blinding) || !load_sc(&ys, y) || !load_sc(&zs, z) || !load_sc(&xs, x)) return ORC_NONCANONICAL_SCALAR;
    return mpc_party_proof_share(gens, v, &vb, n, j, seed, &ys, &zs, &xs, out);
}
int orc_mpc_dealer_bit_challenge(void *gens, uint8_t *tstate, size_t n, size_t m, const uint8_t *bitc, uint8_t y_out[32], uint8_t z_out[32]) {
    merlin t; memcpy(&t, tstate, sizeof t); sc y, z; uint8_t A[32], S[32];
    int rc = mpc_dealer_bit_challenge(gens, &t, n, m, bitc, &y, &z, A, S); if (rc) return rc;
    sc_tobytes(y_out, &y); sc_tobytes(z_out, &z); memcpy(tstate, &t, sizeof t); return ORC_OK;
}
int orc_mpc_dealer_poly_challenge(uint8_t *tstate, size_t m, const uint8_t *polyc, uint8_t x_out[32]) {
    merlin t; memcpy(&t, tstate, sizeof t); sc x; uint8_t T1[32], T2[32];
    int rc = mpc_dealer_poly_challenge(&t, m, polyc, &x, T1, T2); if (rc) return rc;
    sc_tobytes(x_out, &x); memcpy(tstate, &t, sizeof t); return ORC_OK;
}
int orc_mpc_dealer_run(void *gens, const uint8_t *initial_tstate, size_t n, size_t m, const uint8_t *bitc, const uint8_t *polyc, const uint8_t *shares, int trusted,
                       const uint8_t verify_seed[32], uint8_t *proof_out, uint8_t *bad) {
    merlin t; memcpy(&t, initial_tstate, sizeof t);
    return mpc_dealer_run(gens, default_pc(), &t, n, m, bitc, polyc, shares, trusted, verify_seed, proof_out, bad);
}
int orc_mpc_audit_share(void *gens, size_t n, size_t j, const uint8_t bitc[96], const uint8_t y[32], const uint8_t z[32], const uint8_t polyc[64], const uint8_t x[32], const uint8_t *share) {
    sc ys, zs, xs; if (!load_sc(&ys, y) || !load_sc(&zs, z) || !load_sc(&xs, x)) return ORC_NONCANONICAL_SCALAR;
    return mpc_audit_share(gens, default_pc(), n, j, bitc, &ys, &zs, polyc, &xs, share);
}

size_t orc_rangeproof_size(size_t n, size_t m) { return 32 * (9 + 2 * (size_t)lg2(n * m)); }

/* vartime_multiscalar_mul on compressed inputs; out = compressed result */
int orc_msm(const uint8_t *scalars, const uint8_t *points, size_t n, uint8_t out[32]) {
    ge_init_constants();
    sc *s = malloc(sizeof(sc) * (n ? n : 1)); ge *p = malloc(sizeof(ge) * (n ? n : 1)); int rc = ORC_OK;
    for (size_t i = 0; i < n && !rc; i++) {
        if (!sc_from_canonical(&s[i], scalars + 32 * i)) rc = ORC_NONCANONICAL_SCALAR;
        else if (!ge_decode(&p[i], points + 32 * i)) rc = ORC_INVALID_POINT;
    }
    if (!rc) { ge r; ge_msm_vartime(&r, s, p, n); ge_encode(out, &r); }
    free(s); free(p); return rc;
}
/* same sum by naive double-and-add per term (independent of Straus/Pippenger code) */
int orc_msm_naive(const uint8_t *scalars, const uint8_t *points, size_t n, uint8_t out[32]) {
    ge_init_constants();
    ge acc; ge_identity(&acc);
    for (size_t i = 0; i < n; i++) {
        sc s; ge p, r;
        if (!sc_from_canonical(&s, scalars + 32 * i)) return ORC_NONCANONICAL_SCALAR;
        if (!ge_decode(&p, points + 32 * i)) return ORC_INVALID_POINT;
        ge_scalarmult(&r, &s, &p); ge_add(&acc, &acc, &r);
    }
    ge_encode(out, &acc); return ORC_OK;
}
int orc_point_is_valid(const uint8_t p[32]) { ge_init_constants(); ge q; return ge_decode(&q, p); }
int orc_point_roundtrip(const uint8_t p[32], uint8_t out[32]) { ge_init_constants(); ge q; if (!ge_decode(&q, p)) return ORC_INVALID_POINT; ge_encode(out, &q); return ORC_OK; }
/* decode, then re-encode a different representative of the same coset (tests compress on Z != 1) */
int orc_point_double_encode(const uint8_t p[32], uint8_t out[32]) { ge_init_constants(); ge q; if (!ge_decode(&q, p)) return ORC_INVALID_POINT; ge_dbl(&q, &q); ge_encode(out, &q); return ORC_OK; }
int orc_point_add(const uint8_t a[32], const uint8_t b[32], uint8_t out[32]) { ge_init_constants(); ge p, q; if (!ge_decode(&p, a) || !ge_decode(&q, b)) return ORC_INVALID_POINT; ge_add(&p, &p, &q); ge_encode(out, &p); return ORC_OK; }
void orc_from_uniform_bytes(const uint8_t in[64], uint8_t out[32]) { ge_init_constants(); ge p; ge_from_uniform_bytes(&p, in); ge_encode(out, &p); }
void orc_scalar_from_wide(const uint8_t in[64], uint8_t out[32]) { sc s; sc_from_bytes_wide(&s, in); sc_tobytes(out, &s); }
void orc_scalar_mul(const uint8_t a[32], const uint8_t b[32], uint8_t out[32]) { sc x, y; sc_from_bytes_mod_order(&x, a); sc_from_bytes_mod_order(&y, b); sc_mul(&x, &x, &y); sc_tobytes(out, &x); }
void orc_scalar_invert(const uint8_t a[32], uint8_t out[32]) { sc x; sc_from_bytes_mod_order(&x, a); sc_invert(&x, &x); sc_tobytes(out, &x); }
/* count uniform scalars: consecutive 64-byte blocks of ChaCha20(seed) wide-reduced mod l (Scalar::random with a ChaChaRng), skipping `skip` scalars first */
void orc_scalars_from_chacha(const uint8_t seed[32], size_t skip, size_t count, uint8_t *out) {
    chacha_rng r; chacha_seed(&r, seed); uint8_t b[64]; sc s;
    for (size_t i = 0; i < skip; i++) chacha_fill(&r, b, 64);
    for (size_t i = 0; i < count; i++) { chacha_fill(&r, b, 64); sc_from_bytes_wide(&s, b); sc_tobytes(out + 32 * i, &s); }
}
void orc_chacha_fill(const uint8_t seed[32], uint8_t *out, size_t n) { chacha_rng r; chacha_seed(&r, seed); chacha_fill(&r, out, n); }
void orc_sha3_512(const uint8_t *in, size_t n, uint8_t out[64]) { sha3_512(out, in, n); }
void orc_shake256(const uint8_t *in, size_t n, uint8_t *out, size_t outlen) { sponge s; shake256_init(&s); sponge_absorb(&s, in, n); sponge_squeeze(&s, out, outlen); }

/* InnerProductProof::create on compressed inputs; proof_out has 32*(2 lg n + 2) bytes; transcript updated in place */
int orc_ipp_create(uint8_t *transcript_state, const uint8_t Q[32], const uint8_t *Gf, const uint8_t *Hf, const uint8_t *G, const uint8_t *H,
                   const uint8_t *a, const uint8_t *b, size_t n, uint8_t *proof_out) {
    ge_init_constants();
    if (!is_pow2(n)) return ORC_FORMAT_ERROR;
    merlin t; memcpy(&t, transcript_state, sizeof t);
    ge q; if (!ge_decode(&q, Q)) return ORC_INVALID_POINT;
    sc *gf = malloc(sizeof(sc) * n), *hf = malloc(sizeof(sc) * n), *av = malloc(sizeof(sc) * n), *bv = malloc(sizeof(sc) * n);
    ge *g = malloc(sizeof(ge) * n), *h = malloc(sizeof(ge) * n); int rc = ORC_OK;
    for (size_t i = 0; i < n && !rc; i++) {
        if (!sc_from_canonical(&gf[i], Gf + 32 * i) || !sc_from_canonical(&hf[i], Hf + 32 * i) || !sc_from_canonical(&av[i], a + 32 * i) || !sc_from_canonical(&bv[i], b + 32 * i)) rc = ORC_NONCANONICAL_SCALAR;
        else if (!ge_decode(&g[i], G + 32 * i) || !ge_decode(&h[i], H + 32 * i)) rc = ORC_INVALID_POINT;
    }
    if (!rc) { ipp_create(&t, &q, gf, hf, g, h, av, bv, n, proof_out); memcpy(transcript_state, &t, sizeof t); }
    free(gf); free(hf); free(av); free(bv); free(g); free(h); return rc;
}
int orc_ipp_verify(uint8_t *transcript_state, size_t n, const uint8_t *Gf, const uint8_t *Hf, const uint8_t P[32], const uint8_t Q[32],
                   const uint8_t *G, const uint8_t *H, const uint8_t *proof, size_t plen) {
    ge_init_constants();
    merlin t; memcpy(&t, transcript_state, sizeof t);
    ipp_view ipp; int rc = ipp_from_bytes(&ipp, proof, plen); if (rc) return rc;
    ge p, q; if (!ge_decode(&p, P) || !ge_decode(&q, Q)) return ORC_INVALID_POINT;
    sc *gf = malloc(sizeof(sc) * n), *hf = malloc(sizeof(sc) * n); ge *g = malloc(sizeof(ge) * n), *h = malloc(sizeof(ge) * n);
    for (size_t i = 0; i < n && !rc; i++) {
        if (!sc_from_canonical(&gf[i], Gf + 32 * i) || !sc_from_canonical(&hf[i], Hf + 32 * i)) rc = ORC_NONCANONICAL_SCALAR;
        else if (!ge_decode(&g[i], G + 32 * i) || !ge_decode(&h[i], H + 32 * i)) rc = ORC_INVALID_POINT;
    }
    if (!rc) { rc = ipp_verify(&ipp, n, &t, gf, hf, &p, &q, g, h); memcpy(transcript_state, &t, sizeof t); }
    free(gf); free(hf); free(g); free(h); return rc;
}

/* ------------------------------------------------------------------ linear_proof.rs (GHL'21 appendix E.3 argument)
 * LinearProof::create — linear_proof.rs:40-160; verify — :162-224; verification_scalars — :229-270;
 * subset_product — :272-284; wire format L_0,R_0,..,S,a,r — :291-336, from_bytes :351-397.  Round-trip tests only in the
 * reference (linear_proof.rs:413-487): parity unpinned. */
static int linear_create(merlin *t, chacha_rng *rng, const uint8_t C[32], sc r, sc *a, sc *b, ge *G, const ge *F, const ge *B, size_t n, uint8_t *out) {
    if (!is_pow2(n)) return ORC_FORMAT_ERROR;
    uint8_t enc[32];
    t_innerproduct_domain_sep(t, n);
    t_append_point(t, "C", C);
    for (size_t i = 0; i < n; i++) t_append_scalar(t, "b_i", &b[i]);
    for (size_t i = 0; i < n; i++) { ge_encode(enc, &G[i]); t_append_point(t, "G_i", enc); }
    ge_encode(enc, F); t_append_point(t, "F", enc); ge_encode(enc, B); t_append_point(t, "B", enc);
    size_t round = 0;
    sc *ms = malloc(sizeof(sc) * (n + 2)); ge *mp = malloc(sizeof(ge) * (n + 2));
    while (n != 1) {
        n /= 2;
        sc *aL = a, *aR = a + n, *bL = b, *bR = b + n; ge *GL = G, *GR = G + n;
        sc cL, cR, s_j, t_j; inner_product(&cL, aL, bR, n); inner_product(&cR, aR, bL, n);
        rng_scalar(rng, &s_j); rng_scalar(rng, &t_j);
        ge Lp, Rp; uint8_t Lc[32], Rc[32];
        for (size_t i = 0; i < n; i++) { ms[i] = aL[i]; mp[i] = GR[i]; }
        ms[n] = s_j; mp[n] = *B; ms[n + 1] = cL; mp[n + 1] = *F;
        ge_msm_vartime(&Lp, ms, mp, n + 2); ge_encode(Lc, &Lp);
        for (size_t i = 0; i < n; i++) { ms[i] = aR[i]; mp[i] = GL[i]; }
        ms[n] = t_j; mp[n] = *B; ms[n + 1] = cR; mp[n + 1] = *F;
        ge_msm_vartime(&Rp, ms, mp, n + 2); ge_encode(Rc, &Rp);
        memcpy(out + 64 * round, Lc, 32); memcpy(out + 64 * round + 32, Rc, 32); round++;
        t_append_point(t, "L", Lc); t_append_point(t, "R", Rc);
        sc x, xi, tmp; t_challenge_scalar(t, "x_j", &x); sc_invert(&xi, &x);
        for (size_t i = 0; i < n; i++) {
            sc_mul(&tmp, &xi, &aR[i]); sc_add(&aL[i], &aL[i], &tmp);
            sc_mul(&tmp, &x, &bR[i]); sc_add(&bL[i], &bL[i], &tmp);
            sc s2[2]; sc_one(&s2[0]); s2[1] = x; ge p2[2] = { GL[i], GR[i] }, g; ge_msm_vartime(&g, s2, p2, 2); GL[i] = g;
        }
        sc_mul(&tmp, &x, &s_j); sc_add(&r, &r, &tmp); sc_mul(&tmp, &xi, &t_j); sc_add(&r, &r, &tmp);
    }
    sc s_star, t_star, tmp; rng_scalar(rng, &s_star); rng_scalar(rng, &t_star);
    { sc s3[3]; ge p3[3] = { *B, *F, G[0] }, S; s3[0] = t_star; sc_mul(&s3[1], &s_star, &b[0]); s3[2] = s_star; ge_msm_vartime(&S, s3, p3, 3); ge_encode(enc, &S); }
    memcpy(out + 64 * round, enc, 32);
    t_append_point(t, "S", enc);
    sc x_star, a_star, r_star; t_challenge_scalar(t, "x_star", &x_star);
    sc_mul(&tmp, &x_star, &a[0]); sc_add(&a_star, &s_star, &tmp);
    sc_mul(&tmp, &x_star, &r); sc_add(&r_star, &t_star, &tmp);
    sc_tobytes(out + 64 * round + 32, &a_star); sc_tobytes(out + 64 * round + 64, &r_star);
    free(ms); free(mp);
    return ORC_OK;
}
static int linear_verify(merlin *t, const uint8_t *proof, size_t len, const uint8_t C[32], const ge *G, const ge *F, const ge *B, sc *b, size_t n) {
    if (len % 32) return ORC_FORMAT_ERROR;
    size_t ne = len / 32;
    if (ne < 3 || (ne - 3) % 2) return ORC_FORMAT_ERROR;
    size_t lg_n = (ne - 3) / 2;
    if (lg_n >= 32) return ORC_FORMAT_ERROR;
    const uint8_t *S = proof + 64 * lg_n; sc pa, pr;
    if (!sc_from_canonical(&pa, S + 32) || !sc_from_canonical(&pr, S + 64)) return ORC_FORMAT_ERROR;
    uint8_t enc[32];
    t_innerproduct_domain_sep(t, n);
    t_append_point(t, "C", C);
    for (size_t i = 0; i < n; i++) t_append_scalar(t, "b_i", &b[i]);
    for (size_t i = 0; i < n; i++) { ge_encode(enc, &G[i]); t_append_point(t, "G_i", enc); }
    ge_encode(enc, F); t_append_point(t, "F", enc); ge_encode(enc, B); t_append_point(t, "B", enc);
    if (n != ((size_t)1 << lg_n)) return ORC_VERIFICATION_ERROR;
    sc x[32], xi[32], tmp; size_t nm = n;
    for (size_t j = 0; j < lg_n; j++) {
        if (t_validate_and_append_point(t, "L", proof + 64 * j) || t_validate_and_append_point(t, "R", proof + 64 * j + 32)) return ORC_VERIFICATION_ERROR;
        t_challenge_scalar(t, "x_j", &x[j]);
        nm /= 2;
        for (size_t i = 0; i < nm; i++) { sc_mul(&tmp, &x[j], &b[nm + i]); sc_add(&b[i], &b[i], &tmp); }
    }
    for (size_t j = 0; j < lg_n; j++) sc_invert(&xi[j], &x[j]);
    t_append_point(t, "S", S);
    sc x_star; t_challenge_scalar(t, "x_star", &x_star);
    size_t nt = 3 + 2 * lg_n + n, q = 0; int bad = 0;
    sc *ms = malloc(sizeof(sc) * nt); ge *mp = malloc(sizeof(ge) * nt);
    ms[q] = pr; mp[q++] = *B;
    sc_mul(&ms[q], &pa, &b[0]); mp[q++] = *F;
    sc_neg(&ms[q], &x_star); bad |= !ge_decode(&mp[q++], C);
    for (size_t j = 0; j < lg_n; j++) { sc_mul(&tmp, &x_star, &x[j]); sc_neg(&ms[q], &tmp); bad |= !ge_decode(&mp[q++], proof + 64 * j); }
    for (size_t j = 0; j < lg_n; j++) { sc_mul(&tmp, &x_star, &xi[j]); sc_neg(&ms[q], &tmp); bad |= !ge_decode(&mp[q++], proof + 64 * j + 32); }
    sc *s = malloc(sizeof(sc) * n); sc_one(&s[0]);
    for (size_t i = 1; i < n; i++) { int lg_i = 63 - __builtin_clzll((unsigned long long)i); sc_mul(&s[i], &s[i - ((size_t)1 << lg_i)], &x[(lg_n - 1) - lg_i]); }
    for (size_t i = 0; i < n; i++) { sc_mul(&ms[q], &pa, &s[i]); mp[q++] = G[i]; }
    ge Sp, expect; bad |= !ge_decode(&Sp, S);
    int rc = ORC_OK;
    if (bad) rc = ORC_VERIFICATION_ERROR;
    else { ge_msm_vartime(&expect, ms, mp, nt); if (!ge_ristretto_eq(&expect, &Sp)) rc = ORC_VERIFICATION_ERROR; }
    free(ms); free(mp); free(s);
    return rc;
}
/* compressed-input wrappers: G = n points, F, B; a, b = n scalars; rng = ChaChaRng::from_seed(seed) */
int orc_linear_create(uint8_t *tstate, const uint8_t seed[32], const uint8_t C[32], const uint8_t r[32], const uint8_t *a, const uint8_t *b, const uint8_t *G,
                      const uint8_t F[32], const uint8_t B[32], size_t n, uint8_t *out) {
    ge_init_constants();
    merlin t; memcpy(&t, tstate, sizeof t); chacha_rng rng; chacha_seed(&rng, seed);
    sc rr, *av = malloc(sizeof(sc) * n), *bv = malloc(sizeof(sc) * n); ge *g = malloc(sizeof(ge) * n), f, bb; int rc = ORC_OK;
    if (!sc_from_canonical(&rr, r) || !ge_decode(&f, F) || !ge_decode(&bb, B)) rc = ORC_FORMAT_ERROR;
    for (size_t i = 0; i < n && !rc; i++) if (!sc_from_canonical(&av[i], a + 32 * i) || !sc_from_canonical(&bv[i], b + 32 * i) || !ge_decode(&g[i], G + 32 * i)) rc = ORC_FORMAT_ERROR;
    if (!rc) { rc = linear_create(&t, &rng, C, rr, av, bv, g, &f, &bb, n, out); memcpy(tstate, &t, sizeof t); }
    free(av); free(bv); free(g); return rc;
}
int orc_linear_verify(uint8_t *tstate, const uint8_t *proof, size_t len, const uint8_t C[32], const uint8_t *G, const uint8_t F[32], const uint8_t B[32], const uint8_t *b, size_t n) {
    ge_init_constants();
    merlin t; memcpy(&t, tstate, sizeof t);
    sc *bv = malloc(sizeof(sc) * (n ? n : 1)); ge *g = malloc(sizeof(ge) * (n ? n : 1)), f, bb; int rc = ORC_OK;
    if (!ge_decode(&f, F) || !ge_decode(&bb, B)) rc = ORC_FORMAT_ERROR;
    for (size_t i = 0; i < n && !rc; i++) if (!sc_from_canonical(&bv[i], b + 32 * i) || !ge_decode(&g[i], G + 32 * i)) rc = ORC_FORMAT_ERROR;
    if (!rc) { rc = linear_verify(&t, proof, len, C, g, &f, &bb, bv, n); memcpy(tstate, &t, sizeof t); }
    free(bv); free(g); return rc;
}

/* ------------------------------------------------------------------ R1CS (prover.rs / verifier.rs) with three gadgets */
#include "r1cs.h"

static int r1cs_build(r1_cs *cs, int gadget, size_t m, uint64_t param, uint64_t aux, r1_var *vars, shuffle_ctx *sctx) {
    if (gadget == 0) {                      /* shuffle: inputs then outputs (benches/r1cs.rs:98-120) */
        if (m < 2 || m % 2) return ORC_FORMAT_ERROR;
        sctx->k = m / 2; sctx->x = vars; sctx->y = vars + m / 2; shuffle_gadget(cs, sctx);
    } else if (gadget == 1) { if (m != 5) return ORC_FORMAT_ERROR; example_gadget(cs, vars, param); }
    else if (gadget == 2) { if (m != 1 || param > 64) return ORC_FORMAT_ERROR; range_gadget(cs, vars[0], aux, (size_t)param); }
    else return ORC_FORMAT_ERROR;
    return ORC_OK;
}
int orc_r1cs_prove(void *gens, const uint8_t *tstate, int gadget, const uint8_t *values, const uint8_t *blindings, size_t m, uint64_t param, uint64_t aux,
                   const uint8_t ext_seed[32], uint8_t *proof_out, size_t *proof_len, uint8_t *commitments_out) {
    merlin t; memcpy(&t, tstate, sizeof t);
    chacha_rng ext; chacha_seed(&ext, ext_seed);
    r1_cs cs; cs_init(&cs, 1, &t, default_pc());
    r1_var *vars = malloc(sizeof(r1_var) * (m ? m : 1)); shuffle_ctx sctx;
    for (size_t i = 0; i < m; i++) { sc v, b; sc_from_bytes_mod_order(&v, values + 32 * i); sc_from_bytes_mod_order(&b, blindings + 32 * i); vars[i] = cs_commit(&cs, &v, &b, NULL, commitments_out + 32 * i); }
    int rc = r1cs_build(&cs, gadget, m, param, aux, vars, &sctx);
    if (!rc) rc = r1cs_prove(&cs, gens, &ext, proof_out, proof_len);
    cs_free(&cs); free(vars); return rc;
}
int orc_r1cs_verify(void *gens, const uint8_t *tstate, int gadget, const uint8_t *commitments, size_t m, uint64_t param, const uint8_t *proof, size_t len, const uint8_t ext_seed[32]) {
    merlin t; memcpy(&t, tstate, sizeof t);
    chacha_rng ext; chacha_seed(&ext, ext_seed);
    r1_cs cs; cs_init(&cs, 0, &t, default_pc());
    r1_var *vars = malloc(sizeof(r1_var) * (m ? m : 1)); shuffle_ctx sctx;
    for (size_t i = 0; i < m; i++) vars[i] = cs_commit(&cs, NULL, NULL, commitments + 32 * i, NULL);
    int rc = r1cs_build(&cs, gadget, m, param, 0, vars, &sctx);
    if (!rc) rc = r1cs_verify(&cs, gens, proof, len, &ext);
    cs_free(&cs); free(vars); return rc;
}

/* ------------------------------------------------------------------ multi-threaded batch drivers
 * (CPU baseline: independent proofs, one per task — the reference has no batch verifier, so this
 *  is "verify_multiple per proof" on all host cores; BASELINE.md section 2.3) */
typedef struct {
    const bp_gens *bg; const uint8_t *tstate; const uint8_t *proofs; size_t plen; const uint8_t *Vs; size_t m, n, count;
    const uint64_t *values; const uint8_t *blindings; uint8_t *proofs_out, *Vs_out; const uint8_t *seeds; uint8_t *verdicts;
    int nthreads, tid, prove;
} batch_job;

static void *batch_worker(void *arg) {
    batch_job *j = arg;
    if (j->prove == 2) {        /* RLC batches: thread t takes the contiguous chunk t of the proofs, one combined MSM per chunk */
        size_t per = (j->count + (size_t)j->nthreads - 1) / (size_t)j->nthreads, a = (size_t)j->tid * per, b = a + per < j->count ? a + per : j->count;
        if (a >= b) return NULL;
        chacha_rng rng; chacha_seed(&rng, j->seeds); for (int q = 0; q < j->tid; q++) { uint8_t skip[64]; chacha_fill(&rng, skip, 64); }
        int ok = rp_verify_rlc_chunk(j->bg, default_pc(), j->tstate, j->proofs + a * j->plen, j->plen, j->Vs + 32 * j->m * a, j->m, j->n, b - a, &rng);
        for (size_t i = a; i < b; i++) {
            if (ok) { j->verdicts[i] = 0; continue; }
            merlin t; memcpy(&t, j->tstate, sizeof t);
            j->verdicts[i] = (uint8_t)rp_verify(j->bg, default_pc(), &t, j->proofs + i * j->plen, j->plen, j->Vs + 32 * i * j->m, j->m, j->n, &rng);
        }
        return NULL;
    }
    for (size_t i = (size_t)j->tid; i < j->count; i += (size_t)j->nthreads) {
        merlin t; memcpy(&t, j->tstate, sizeof t);
        chacha_rng rng; chacha_seed(&rng, j->seeds + 32 * i);
        if (j->prove)
            j->verdicts[i] = (uint8_t)rp_prove(j->bg, default_pc(), &t, j->values + i * j->m, j->blindings + 32 * i * j->m, j->m, j->n, &rng,
                                               j->proofs_out + i * j->plen, j->Vs_out + 32 * i * j->m);
        else
            j->verdicts[i] = (uint8_t)rp_verify(j->bg, default_pc(), &t, j->proofs + i * j->plen, j->plen, j->Vs + 32 * i * j->m, j->m, j->n, &rng);
    }
    return NULL;
}
static void run_batch(batch_job *proto, int nthreads) {
    if (nthreads < 1) nthreads = 1;
    pthread_t *th = malloc(sizeof(pthread_t) * nthreads); batch_job *jobs = malloc(sizeof(batch_job) * nthreads);
    default_pc();
    for (int i = 0; i < nthreads; i++) { jobs[i] = *proto; jobs[i].tid = i; jobs[i].nthreads = nthreads; pthread_create(&th[i], NULL, batch_worker, &jobs[i]); }
    for (int i = 0; i < nthreads; i++) pthread_join(th[i], NULL);
    free(th); free(jobs);
}
/* status[i] = per-proof verify status (0 = accept) */
void orc_rangeproof_verify_many(void *gens, const uint8_t *transcript_state, const uint8_t *proofs, size_t plen, const uint8_t *Vs,
                                size_t m, size_t n, size_t count, const uint8_t *seeds, int nthreads, uint8_t *status) {
    batch_job j = {0}; j.bg = gens; j.tstate = transcript_state; j.proofs = proofs; j.plen = plen; j.Vs = Vs; j.m = m; j.n = n; j.count = count;
    j.seeds = seeds; j.verdicts = status; j.prove = 0; run_batch(&j, nthreads);
}
/* same verdicts through the CPU random-linear-combination batch: nthreads chunks, one combined MSM each, per-proof recheck of a failing chunk */
void orc_rangeproof_verify_rlc(void *gens, const uint8_t *transcript_state, const uint8_t *proofs, size_t plen, const uint8_t *Vs,
                               size_t m, size_t n, size_t count, const uint8_t seed[32], int nthreads, uint8_t *status) {
    batch_job j = {0}; j.bg = gens; j.tstate = transcript_state; j.proofs = proofs; j.plen = plen; j.Vs = Vs; j.m = m; j.n = n; j.count = count;
    j.seeds = seed; j.verdicts = status; j.prove = 2; run_batch(&j, nthreads);
}
void orc_rangeproof_prove_many(void *gens, const uint8_t *transcript_state, const uint64_t *values, const uint8_t *blindings,
                               size_t m, size_t n, size_t count, const uint8_t *seeds, int nthreads, uint8_t *proofs_out, uint8_t *Vs_out, uint8_t *status) {
    batch_job j = {0}; j.bg = gens; j.tstate = transcript_state; j.values = values; j.blindings = blindings; j.m = m; j.n = n; j.count = count;
    j.plen = orc_rangeproof_size(n, m); j.proofs_out = proofs_out; j.Vs_out = Vs_out; j.seeds = seeds; j.verdicts = status; j.prove = 1; run_batch(&j, nthreads);
}
