/* ORACLE (test infrastructure only).
 *
 * Restatement of the R1CS proof system of the reference (feature `yoloproofs`, commented out in
 * Cargo.toml:43 but present in the tree):
 *   constraint system   src/r1cs/constraint_system.rs, linear_combination.rs
 *   Prover              src/r1cs/prover.rs:62-698
 *   Verifier            src/r1cs/verifier.rs:61-500
 *   R1CSProof wire form src/r1cs/proof.rs:71-204
 *   TranscriptRng       merlin 2.x (un-vendored): rekey_with_witness_bytes / finalize / fill_bytes
 * and of three gadgets used by the reference's tests and benches:
 *   shuffle  benches/r1cs.rs:34-67      (two-phase, randomized constraints)
 *   example  tests/r1cs.rs:225-236      ((a1+a2)(b1+b2) = c1+c2, constant term)
 *   range    tests/r1cs.rs:366-385      (allocate_multiplier, bit decomposition)
 * No fixed vectors exist in the reference for R1CS (round-trip tests only): parity unpinned; this
 * restatement is checked by prover<->verifier round trips and negative cases like the reference's.
 */
#ifndef ORACLE_R1CS_H
#define ORACLE_R1CS_H

enum { R1_COMMITTED = 0, R1_LEFT = 1, R1_RIGHT = 2, R1_OUT = 3, R1_ONE = 4 };
typedef struct { int kind; size_t idx; } r1_var;
typedef struct { r1_var v; sc c; } r1_term;
typedef struct { r1_term *t; size_t n, cap; } r1_lc;

struct r1_cs;
typedef int (*r1_deferred_fn)(struct r1_cs *, void *);
typedef struct r1_cs {
    int is_prover; merlin *tr; const pedersen_gens *pc;
    sc *aL, *aR, *aO; size_t nvars, vcap;          /* prover: assignments; verifier: only nvars */
    sc *v, *vbl; uint8_t *V; size_t m, mcap;         /* committed: prover values/blindings; both: compressed V */
    r1_lc *cons; size_t ncons, ccap;
    int pending; size_t pending_idx;
    r1_deferred_fn deferred[4]; void *dctx[4]; int ndef;
} r1_cs;

static r1_lc lc_empty(void) { r1_lc l = { NULL, 0, 0 }; return l; }
static void lc_push(r1_lc *l, r1_var v, const sc *c) {
    if (l->n == l->cap) { l->cap = l->cap ? 2 * l->cap : 4; l->t = realloc(l->t, l->cap * sizeof(r1_term)); }
    l->t[l->n].v = v; l->t[l->n].c = *c; l->n++;
}
static r1_var var_of(int kind, size_t idx) { r1_var v = { kind, idx }; return v; }
static void lc_push_i(r1_lc *l, r1_var v, int64_t c) {          /* small signed coefficient */
    sc s; sc_from_u64(&s, (uint64_t)(c < 0 ? -c : c)); if (c < 0) sc_neg(&s, &s); lc_push(l, v, &s);
}
static r1_lc lc_var(r1_var v) { r1_lc l = lc_empty(); lc_push_i(&l, v, 1); return l; }

static void cs_init(r1_cs *cs, int is_prover, merlin *tr, const pedersen_gens *pc) {
    memset(cs, 0, sizeof *cs); cs->is_prover = is_prover; cs->tr = tr; cs->pc = pc;
    merlin_append(tr, "dom-sep", (const uint8_t *)"r1cs v1", 7);                      /* transcript.rs:55-57 */
}
static void cs_free(r1_cs *cs) {
    for (size_t i = 0; i < cs->ncons; i++) free(cs->cons[i].t);
    free(cs->cons); free(cs->aL); free(cs->aR); free(cs->aO); free(cs->v); free(cs->vbl); free(cs->V);
}
static void cs_constrain(r1_cs *cs, r1_lc lc) {                                        /* takes ownership */
    if (cs->ncons == cs->ccap) { cs->ccap = cs->ccap ? 2 * cs->ccap : 16; cs->cons = realloc(cs->cons, cs->ccap * sizeof(r1_lc)); }
    cs->cons[cs->ncons++] = lc;
}
static size_t cs_new_var(r1_cs *cs) {
    if (cs->is_prover && cs->nvars == cs->vcap) {
        cs->vcap = cs->vcap ? 2 * cs->vcap : 16;
        cs->aL = realloc(cs->aL, cs->vcap * sizeof(sc)); cs->aR = realloc(cs->aR, cs->vcap * sizeof(sc)); cs->aO = realloc(cs->aO, cs->vcap * sizeof(sc));
    }
    return cs->nvars++;
}
static void cs_eval(const r1_cs *cs, const r1_lc *lc, sc *out) {                       /* prover.rs:340-356 */
    sc acc, t; sc_zero(&acc);
    for (size_t i = 0; i < lc->n; i++) {
        const sc *val; sc one; sc_one(&one);
        switch (lc->t[i].v.kind) {
            case R1_LEFT: val = &cs->aL[lc->t[i].v.idx]; break;
            case R1_RIGHT: val = &cs->aR[lc->t[i].v.idx]; break;
            case R1_OUT: val = &cs->aO[lc->t[i].v.idx]; break;
            case R1_COMMITTED: val = &cs->v[lc->t[i].v.idx]; break;
            default: val = &one;
        }
        sc_mul(&t, &lc->t[i].c, val); sc_add(&acc, &acc, &t);
    }
    *out = acc;
}
/* ConstraintSystem::multiply — prover.rs:73-103, verifier.rs:66-86; consumes left and right */
static void cs_multiply(r1_cs *cs, r1_lc left, r1_lc right, r1_var *l, r1_var *r, r1_var *o) {
    sc lv, rv; if (cs->is_prover) { cs_eval(cs, &left, &lv); cs_eval(cs, &right, &rv); }
    size_t i = cs_new_var(cs);
    if (cs->is_prover) { cs->aL[i] = lv; cs->aR[i] = rv; sc_mul(&cs->aO[i], &lv, &rv); }
    if (l) *l = var_of(R1_LEFT, i);
    if (r) *r = var_of(R1_RIGHT, i);
    if (o) *o = var_of(R1_OUT, i);
    lc_push_i(&left, var_of(R1_LEFT, i), -1); lc_push_i(&right, var_of(R1_RIGHT, i), -1);
    cs_constrain(cs, left); cs_constrain(cs, right);
}
/* allocate_multiplier — prover.rs:128-146, verifier.rs:104-115 */
static void cs_allocate_multiplier(r1_cs *cs, const sc *lv, const sc *rv, r1_var *l, r1_var *r, r1_var *o) {
    size_t i = cs_new_var(cs);
    if (cs->is_prover) { cs->aL[i] = *lv; cs->aR[i] = *rv; sc_mul(&cs->aO[i], lv, rv); }
    *l = var_of(R1_LEFT, i); *r = var_of(R1_RIGHT, i); *o = var_of(R1_OUT, i);
}
/* Prover::commit / Verifier::commit — prover.rs:278-288, verifier.rs:236-245 */
static r1_var cs_commit(r1_cs *cs, const sc *v, const sc *vbl, const uint8_t *V_in, uint8_t V_out[32]) {
    if (cs->m == cs->mcap) {
        cs->mcap = cs->mcap ? 2 * cs->mcap : 16;
        cs->V = realloc(cs->V, 32 * cs->mcap);
        if (cs->is_prover) { cs->v = realloc(cs->v, cs->mcap * sizeof(sc)); cs->vbl = realloc(cs->vbl, cs->mcap * sizeof(sc)); }
    }
    size_t i = cs->m++;
    if (cs->is_prover) {
        cs->v[i] = *v; cs->vbl[i] = *vbl;
        sc s2[2] = { *v, *vbl }; ge p2[2] = { cs->pc->B, cs->pc->B_blinding }, Vp;
        ge_msm_vartime(&Vp, s2, p2, 2); ge_encode(cs->V + 32 * i, &Vp);
    } else memcpy(cs->V + 32 * i, V_in, 32);
    if (V_out) memcpy(V_out, cs->V + 32 * i, 32);
    merlin_append(cs->tr, "V", cs->V + 32 * i, 32);
    return var_of(R1_COMMITTED, i);
}
static void cs_specify_randomized(r1_cs *cs, r1_deferred_fn fn, void *ctx) { cs->deferred[cs->ndef] = fn; cs->dctx[cs->ndef] = ctx; cs->ndef++; }
/* create_randomized_constraints — prover.rs:358-377, verifier.rs:302-321 */
static int cs_run_deferred(r1_cs *cs) {
    cs->pending = 0;
    if (cs->ndef == 0) { merlin_append(cs->tr, "dom-sep", (const uint8_t *)"r1cs-1phase", 11); return 0; }
    merlin_append(cs->tr, "dom-sep", (const uint8_t *)"r1cs-2phase", 11);
    int n = cs->ndef; cs->ndef = 0;
    for (int i = 0; i < n; i++) { int rc = cs->deferred[i](cs, cs->dctx[i]); if (rc) return rc; }
    return 0;
}
/* flattened_constraints — prover.rs:301-338, verifier.rs:260-298 */
static void cs_flatten(const r1_cs *cs, const sc *z, sc *wL, sc *wR, sc *wO, sc *wV, sc *wc) {
    size_t n = cs->nvars;
    for (size_t i = 0; i < n; i++) { sc_zero(&wL[i]); sc_zero(&wR[i]); sc_zero(&wO[i]); }
    for (size_t i = 0; i < cs->m; i++) sc_zero(&wV[i]);
    sc_zero(wc);
    sc exp_z = *z, t;
    for (size_t k = 0; k < cs->ncons; k++) {
        const r1_lc *lc = &cs->cons[k];
        for (size_t j = 0; j < lc->n; j++) {
            sc_mul(&t, &exp_z, &lc->t[j].c);
            size_t i = lc->t[j].v.idx;
            switch (lc->t[j].v.kind) {
                case R1_LEFT: sc_add(&wL[i], &wL[i], &t); break;
                case R1_RIGHT: sc_add(&wR[i], &wR[i], &t); break;
                case R1_OUT: sc_add(&wO[i], &wO[i], &t); break;
                case R1_COMMITTED: sc_sub(&wV[i], &wV[i], &t); break;
                default: sc_sub(wc, wc, &t);
            }
        }
        sc_mul(&exp_z, &exp_z, z);
    }
}

/* merlin TranscriptRng: clone, rekey with witness bytes, finalize with 32 external random bytes */
typedef struct { merlin m; } transcript_rng;
static void trng_begin(transcript_rng *r, const merlin *t) { r->m = *t; }
static void trng_rekey(transcript_rng *r, const char *label, const uint8_t *w, size_t len) {
    uint8_t l4[4] = { (uint8_t)len, (uint8_t)(len >> 8), (uint8_t)(len >> 16), (uint8_t)(len >> 24) };
    strobe_meta_ad(&r->m, (const uint8_t *)label, strlen(label), 0); strobe_meta_ad(&r->m, l4, 4, 1); strobe_key(&r->m, w, len, 0);
}
static void trng_finalize(transcript_rng *r, chacha_rng *ext) {
    uint8_t rb[32]; chacha_fill(ext, rb, 32);
    strobe_meta_ad(&r->m, (const uint8_t *)"rng", 3, 0); strobe_key(&r->m, rb, 32, 0);
}
static void trng_scalar(transcript_rng *r, sc *out) {                                  /* Scalar::random(&mut rng) */
    uint8_t l4[4] = { 64, 0, 0, 0 }, b[64];
    strobe_meta_ad(&r->m, l4, 4, 0); strobe_prf(&r->m, b, 64, 0); sc_from_bytes_wide(out, b);
}

static size_t next_pow2(size_t n) { size_t p = 1; while (p < n) p <<= 1; return p; }
static void msm_with_blinding(uint8_t out[32], const pedersen_gens *pc, const sc *bl, const sc *a, const ge *G, size_t na, const sc *b, const ge *H, size_t nb) {
    size_t n = 1 + na + nb; sc *s = malloc(n * sizeof(sc)); ge *p = malloc(n * sizeof(ge)), r;
    s[0] = *bl; p[0] = pc->B_blinding;
    for (size_t i = 0; i < na; i++) { s[1 + i] = a[i]; p[1 + i] = G[i]; }
    for (size_t i = 0; i < nb; i++) { s[1 + na + i] = b[i]; p[1 + na + i] = H[i]; }
    ge_msm_vartime(&r, s, p, n); ge_encode(out, &r); free(s); free(p);
}
static void commit_encode(uint8_t out[32], const pedersen_gens *pc, const sc *v, const sc *bl) {
    sc s2[2] = { *v, *bl }; ge p2[2] = { pc->B, pc->B_blinding }, r; ge_msm_vartime(&r, s2, p2, 2); ge_encode(out, &r);
}

/* Prover::prove — prover.rs:380-698.  Writes R1CSProof::to_bytes (proof.rs:83-112); returns 0 or an error code. */
static int r1cs_prove(r1_cs *cs, const bp_gens *bg, chacha_rng *ext, uint8_t *out, size_t *out_len) {
    merlin *t = cs->tr; const pedersen_gens *pc = cs->pc;
    merlin_append_u64(t, "m", (uint64_t)cs->m);
    transcript_rng rng; trng_begin(&rng, t);
    for (size_t i = 0; i < cs->m; i++) { uint8_t b[32]; sc_tobytes(b, &cs->vbl[i]); trng_rekey(&rng, "v_blinding", b, 32); }
    trng_finalize(&rng, ext);
    size_t n1 = cs->nvars;
    if (bg->gens_capacity < n1) return ORC_INVALID_GENS_LENGTH;
    const ge *G = bg->G, *H = bg->H;                                                    /* share(0) */
    sc i_bl1, o_bl1, s_bl1; trng_scalar(&rng, &i_bl1); trng_scalar(&rng, &o_bl1); trng_scalar(&rng, &s_bl1);
    sc *sL = malloc(sizeof(sc) * (n1 ? n1 : 1)), *sR = malloc(sizeof(sc) * (n1 ? n1 : 1));
    for (size_t i = 0; i < n1; i++) trng_scalar(&rng, &sL[i]);
    for (size_t i = 0; i < n1; i++) trng_scalar(&rng, &sR[i]);
    uint8_t A_I1[32], A_O1[32], S1[32], A_I2[32] = {0}, A_O2[32] = {0}, S2[32] = {0};
    msm_with_blinding(A_I1, pc, &i_bl1, cs->aL, G, n1, cs->aR, H, n1);
    msm_with_blinding(A_O1, pc, &o_bl1, cs->aO, G, n1, NULL, NULL, 0);
    msm_with_blinding(S1, pc, &s_bl1, sL, G, n1, sR, H, n1);
    merlin_append(t, "A_I1", A_I1, 32); merlin_append(t, "A_O1", A_O1, 32); merlin_append(t, "S1", S1, 32);
    int rc = cs_run_deferred(cs); if (rc) { free(sL); free(sR); return rc; }
    size_t n = cs->nvars, n2 = n - n1, padded_n = next_pow2(n);
    if (bg->gens_capacity < padded_n) { free(sL); free(sR); return ORC_INVALID_GENS_LENGTH; }
    sc i_bl2, o_bl2, s_bl2; sc_zero(&i_bl2); sc_zero(&o_bl2); sc_zero(&s_bl2);
    if (n2 > 0) { trng_scalar(&rng, &i_bl2); trng_scalar(&rng, &o_bl2); trng_scalar(&rng, &s_bl2); }
    sL = realloc(sL, sizeof(sc) * (n ? n : 1)); sR = realloc(sR, sizeof(sc) * (n ? n : 1));
    for (size_t i = n1; i < n; i++) trng_scalar(&rng, &sL[i]);
    for (size_t i = n1; i < n; i++) trng_scalar(&rng, &sR[i]);
    if (n2 > 0) {
        msm_with_blinding(A_I2, pc, &i_bl2, cs->aL + n1, G + n1, n2, cs->aR + n1, H + n1, n2);
        msm_with_blinding(A_O2, pc, &o_bl2, cs->aO + n1, G + n1, n2, NULL, NULL, 0);
        msm_with_blinding(S2, pc, &s_bl2, sL + n1, G + n1, n2, sR + n1, H + n1, n2);
    }
    merlin_append(t, "A_I2", A_I2, 32); merlin_append(t, "A_O2", A_O2, 32); merlin_append(t, "S2", S2, 32);
    sc y, z; t_challenge_scalar(t, "y", &y); t_challenge_scalar(t, "z", &z);
    sc *wL = malloc(sizeof(sc) * (n + 1)), *wR = malloc(sizeof(sc) * (n + 1)), *wO = malloc(sizeof(sc) * (n + 1)), *wV = malloc(sizeof(sc) * (cs->m + 1)), wc;
    cs_flatten(cs, &z, wL, wR, wO, wV, &wc);
    /* l(x) = l1 x + l2 x^2 + l3 x^3 ; r(x) = r0 + r1 x + r3 x^3   (prover.rs:556-573) */
    sc *l1 = malloc(sizeof(sc) * (n + 1)), *l2 = malloc(sizeof(sc) * (n + 1)), *l3 = malloc(sizeof(sc) * (n + 1));
    sc *r0 = malloc(sizeof(sc) * (n + 1)), *r1 = malloc(sizeof(sc) * (n + 1)), *r3 = malloc(sizeof(sc) * (n + 1));
    sc *exp_y_inv = malloc(sizeof(sc) * padded_n), y_inv, exp_y, tmp;
    sc_invert(&y_inv, &y); sc_one(&exp_y);
    { sc e; sc_one(&e); for (size_t i = 0; i < padded_n; i++) { exp_y_inv[i] = e; sc_mul(&e, &e, &y_inv); } }
    for (size_t i = 0; i < n; i++) {
        sc_mul(&tmp, &exp_y_inv[i], &wR[i]); sc_add(&l1[i], &cs->aL[i], &tmp);
        l2[i] = cs->aO[i]; l3[i] = sL[i];
        sc_sub(&r0[i], &wO[i], &exp_y);
        sc_mul(&tmp, &exp_y, &cs->aR[i]); sc_add(&r1[i], &tmp, &wL[i]);
        sc_mul(&r3[i], &exp_y, &sR[i]);
        sc_mul(&exp_y, &exp_y, &y);
    }
    /* VecPoly3::special_inner_product — util.rs:125-142 (l.0 = 0, r.2 = 0) */
    sc t1, t2, t3, t4, t5, t6, a, b;
    inner_product(&t1, l1, r0, n);
    inner_product(&a, l1, r1, n); inner_product(&b, l2, r0, n); sc_add(&t2, &a, &b);
    inner_product(&a, l2, r1, n); inner_product(&b, l3, r0, n); sc_add(&t3, &a, &b);
    inner_product(&a, l1, r3, n); inner_product(&b, l3, r1, n); sc_add(&t4, &a, &b);
    inner_product(&t5, l2, r3, n); inner_product(&t6, l3, r3, n);
    sc t1b, t3b, t4b, t5b, t6b;
    trng_scalar(&rng, &t1b); trng_scalar(&rng, &t3b); trng_scalar(&rng, &t4b); trng_scalar(&rng, &t5b); trng_scalar(&rng, &t6b);
    uint8_t T1[32], T3[32], T4[32], T5[32], T6[32];
    commit_encode(T1, pc, &t1, &t1b); commit_encode(T3, pc, &t3, &t3b); commit_encode(T4, pc, &t4, &t4b); commit_encode(T5, pc, &t5, &t5b); commit_encode(T6, pc, &t6, &t6b);
    merlin_append(t, "T_1", T1, 32); merlin_append(t, "T_3", T3, 32); merlin_append(t, "T_4", T4, 32); merlin_append(t, "T_5", T5, 32); merlin_append(t, "T_6", T6, 32);
    sc u, x; t_challenge_scalar(t, "u", &u); t_challenge_scalar(t, "x", &x);
    sc t2b; sc_zero(&t2b);
    for (size_t i = 0; i < cs->m; i++) { sc_mul(&tmp, &wV[i], &cs->vbl[i]); sc_add(&t2b, &t2b, &tmp); }
    /* Poly6::eval: x (t1 + x (t2 + x (t3 + x (t4 + x (t5 + x t6)))))  (util.rs:164-168) */
    sc t_x, t_x_bl;
    { const sc *c[6] = { &t1, &t2, &t3, &t4, &t5, &t6 }; sc acc = t6; for (int k = 4; k >= 0; k--) { sc_mul(&acc, &acc, &x); sc_add(&acc, &acc, c[k]); } sc_mul(&t_x, &acc, &x); }
    { const sc *c[6] = { &t1b, &t2b, &t3b, &t4b, &t5b, &t6b }; sc acc = t6b; for (int k = 4; k >= 0; k--) { sc_mul(&acc, &acc, &x); sc_add(&acc, &acc, c[k]); } sc_mul(&t_x_bl, &acc, &x); }
    sc *l_vec = malloc(sizeof(sc) * padded_n), *r_vec = malloc(sizeof(sc) * padded_n);
    for (size_t i = 0; i < n; i++) {                                                    /* VecPoly3::eval (util.rs:144-151) */
        sc acc; sc_mul(&acc, &l3[i], &x); sc_add(&acc, &acc, &l2[i]); sc_mul(&acc, &acc, &x); sc_add(&acc, &acc, &l1[i]); sc_mul(&l_vec[i], &acc, &x);
        sc_mul(&acc, &r3[i], &x); sc_mul(&acc, &acc, &x); sc_add(&acc, &acc, &r1[i]); sc_mul(&acc, &acc, &x); sc_add(&r_vec[i], &acc, &r0[i]);
    }
    for (size_t i = n; i < padded_n; i++) { sc_zero(&l_vec[i]); sc_neg(&r_vec[i], &exp_y); sc_mul(&exp_y, &exp_y, &y); }
    sc i_bl, o_bl, s_bl, e_bl;
    sc_mul(&tmp, &u, &i_bl2); sc_add(&i_bl, &i_bl1, &tmp); sc_mul(&tmp, &u, &o_bl2); sc_add(&o_bl, &o_bl1, &tmp); sc_mul(&tmp, &u, &s_bl2); sc_add(&s_bl, &s_bl1, &tmp);
    sc_mul(&e_bl, &x, &s_bl); sc_add(&e_bl, &e_bl, &o_bl); sc_mul(&e_bl, &e_bl, &x); sc_add(&e_bl, &e_bl, &i_bl); sc_mul(&e_bl, &e_bl, &x);
    t_append_scalar(t, "t_x", &t_x); t_append_scalar(t, "t_x_blinding", &t_x_bl); t_append_scalar(t, "e_blinding", &e_bl);
    sc w; t_challenge_scalar(t, "w", &w);
    ge Q; ge_scalarmult(&Q, &w, &pc->B);
    sc *Gf = malloc(sizeof(sc) * padded_n), *Hf = malloc(sizeof(sc) * padded_n);
    for (size_t i = 0; i < padded_n; i++) { if (i < n1) sc_one(&Gf[i]); else Gf[i] = u; sc_mul(&Hf[i], &exp_y_inv[i], &Gf[i]); }
    ge *Gv = malloc(sizeof(ge) * padded_n), *Hv = malloc(sizeof(ge) * padded_n);
    memcpy(Gv, G, sizeof(ge) * padded_n); memcpy(Hv, H, sizeof(ge) * padded_n);
    /* R1CSProof::to_bytes (proof.rs:83-112) */
    int two_phase = 0; for (int i = 0; i < 32; i++) two_phase |= A_I2[i] | A_O2[i] | S2[i];
    uint8_t *o = out;
    *o++ = two_phase ? 1 : 0;
    memcpy(o, A_I1, 32); o += 32; memcpy(o, A_O1, 32); o += 32; memcpy(o, S1, 32); o += 32;
    if (two_phase) { memcpy(o, A_I2, 32); o += 32; memcpy(o, A_O2, 32); o += 32; memcpy(o, S2, 32); o += 32; }
    memcpy(o, T1, 32); o += 32; memcpy(o, T3, 32); o += 32; memcpy(o, T4, 32); o += 32; memcpy(o, T5, 32); o += 32; memcpy(o, T6, 32); o += 32;
    sc_tobytes(o, &t_x); o += 32; sc_tobytes(o, &t_x_bl); o += 32; sc_tobytes(o, &e_bl); o += 32;
    ipp_create(t, &Q, Gf, Hf, Gv, Hv, l_vec, r_vec, padded_n, o);
    o += 32 * (2 * (size_t)lg2(padded_n) + 2);
    *out_len = (size_t)(o - out);
    free(sL); free(sR); free(wL); free(wR); free(wO); free(wV); free(l1); free(l2); free(l3); free(r0); free(r1); free(r3); free(exp_y_inv);
    free(l_vec); free(r_vec); free(Gf); free(Hf); free(Gv); free(Hv);
    return ORC_OK;
}

/* Verifier::verify — verifier.rs:329-500 on R1CSProof::from_bytes input (proof.rs:133-204) */
static int r1cs_verify(r1_cs *cs, const bp_gens *bg, const uint8_t *proof, size_t len, chacha_rng *ext) {
    merlin *t = cs->tr; const pedersen_gens *pc = cs->pc;
    if (len < 1) return ORC_FORMAT_ERROR;
    int version = proof[0]; const uint8_t *p = proof + 1; len -= 1;
    if (len % 32) return ORC_FORMAT_ERROR;
    size_t minlen = version == 0 ? 11 * 32 : version == 1 ? 14 * 32 : 0;
    if (!minlen || len < minlen) return ORC_FORMAT_ERROR;
    static const uint8_t ident[32] = {0};
    const uint8_t *A_I1 = p, *A_O1 = p + 32, *S1 = p + 64; p += 96;
    const uint8_t *A_I2 = ident, *A_O2 = ident, *S2 = ident;
    if (version == 1) { A_I2 = p; A_O2 = p + 32; S2 = p + 64; p += 96; }
    const uint8_t *T1 = p, *T3 = p + 32, *T4 = p + 64, *T5 = p + 96, *T6 = p + 128; p += 160;
    sc t_x, t_x_bl, e_bl;
    if (!sc_from_canonical(&t_x, p) || !sc_from_canonical(&t_x_bl, p + 32) || !sc_from_canonical(&e_bl, p + 64)) return ORC_FORMAT_ERROR;
    p += 96;
    ipp_view ipp; if (ipp_from_bytes(&ipp, p, (size_t)(proof + 1 + len - p))) return ORC_FORMAT_ERROR;

    merlin_append_u64(t, "m", (uint64_t)cs->m);
    size_t n1 = cs->nvars;
    if (t_validate_and_append_point(t, "A_I1", A_I1) || t_validate_and_append_point(t, "A_O1", A_O1) || t_validate_and_append_point(t, "S1", S1)) return ORC_VERIFICATION_ERROR;
    int rc = cs_run_deferred(cs); if (rc) return rc;
    size_t n = cs->nvars, n2 = n - n1, padded_n = next_pow2(n), pad = padded_n - n; (void)n2;
    if (bg->gens_capacity < padded_n) return ORC_INVALID_GENS_LENGTH;
    merlin_append(t, "A_I2", A_I2, 32); merlin_append(t, "A_O2", A_O2, 32); merlin_append(t, "S2", S2, 32);
    sc y, z, u, x, w; t_challenge_scalar(t, "y", &y); t_challenge_scalar(t, "z", &z);
    if (t_validate_and_append_point(t, "T_1", T1) || t_validate_and_append_point(t, "T_3", T3) || t_validate_and_append_point(t, "T_4", T4) ||
        t_validate_and_append_point(t, "T_5", T5) || t_validate_and_append_point(t, "T_6", T6)) return ORC_VERIFICATION_ERROR;
    t_challenge_scalar(t, "u", &u); t_challenge_scalar(t, "x", &x);
    t_append_scalar(t, "t_x", &t_x); t_append_scalar(t, "t_x_blinding", &t_x_bl); t_append_scalar(t, "e_blinding", &e_bl);
    t_challenge_scalar(t, "w", &w);
    sc *wL = malloc(sizeof(sc) * (n + 1)), *wR = malloc(sizeof(sc) * (n + 1)), *wO = malloc(sizeof(sc) * (n + 1)), *wV = malloc(sizeof(sc) * (cs->m + 1)), wc;
    cs_flatten(cs, &z, wL, wR, wO, wV, &wc);
    sc *s = malloc(sizeof(sc) * padded_n), u_sq[32], u_inv_sq[32];
    if (ipp_verification_scalars(&ipp, padded_n, t, u_sq, u_inv_sq, s)) { free(wL); free(wR); free(wO); free(wV); free(s); return ORC_VERIFICATION_ERROR; }
    int k = ipp.lg_n;
    sc y_inv, e, tmp; sc_invert(&y_inv, &y); sc_one(&e);
    sc *y_inv_vec = malloc(sizeof(sc) * padded_n), *yneg_wR = malloc(sizeof(sc) * padded_n);
    for (size_t i = 0; i < padded_n; i++) { y_inv_vec[i] = e; sc_mul(&e, &e, &y_inv); }
    for (size_t i = 0; i < padded_n; i++) { if (i < n) sc_mul(&yneg_wR[i], &wR[i], &y_inv_vec[i]); else sc_zero(&yneg_wR[i]); }
    sc delta; inner_product(&delta, yneg_wR, wL, n);
    transcript_rng rng; trng_begin(&rng, t); trng_finalize(&rng, ext);
    sc r; trng_scalar(&rng, &r);
    sc xx, rxx, xxx; sc_mul(&xx, &x, &x); sc_mul(&rxx, &r, &xx); sc_mul(&xxx, &x, &xx);
    size_t nt = 13 + cs->m + 2 * padded_n + 2 * (size_t)k, q = 0; int bad = 0;
    sc *ms = malloc(sizeof(sc) * nt); ge *mp = malloc(sizeof(ge) * nt);
    ms[q] = x; bad |= !ge_decode(&mp[q++], A_I1);
    ms[q] = xx; bad |= !ge_decode(&mp[q++], A_O1);
    ms[q] = xxx; bad |= !ge_decode(&mp[q++], S1);
    sc_mul(&ms[q], &u, &x); bad |= !ge_decode(&mp[q++], A_I2);
    sc_mul(&ms[q], &u, &xx); bad |= !ge_decode(&mp[q++], A_O2);
    sc_mul(&ms[q], &u, &xxx); bad |= !ge_decode(&mp[q++], S2);
    for (size_t i = 0; i < cs->m; i++) { sc_mul(&ms[q], &wV[i], &rxx); bad |= !ge_decode(&mp[q++], cs->V + 32 * i); }
    sc_mul(&ms[q], &r, &x); bad |= !ge_decode(&mp[q++], T1);
    sc_mul(&ms[q], &rxx, &x); bad |= !ge_decode(&mp[q++], T3);
    sc_mul(&ms[q], &rxx, &xx); bad |= !ge_decode(&mp[q++], T4);
    sc_mul(&ms[q], &rxx, &xxx); bad |= !ge_decode(&mp[q++], T5);
    sc_mul(&tmp, &rxx, &xx); sc_mul(&ms[q], &tmp, &xx); bad |= !ge_decode(&mp[q++], T6);
    { sc ab, a1, a2; sc_mul(&ab, &ipp.a, &ipp.b); sc_sub(&a1, &t_x, &ab); sc_mul(&a1, &w, &a1);
      sc_add(&a2, &wc, &delta); sc_mul(&a2, &xx, &a2); sc_sub(&a2, &a2, &t_x); sc_mul(&a2, &r, &a2); sc_add(&ms[q], &a1, &a2); mp[q++] = pc->B; }
    { sc_mul(&tmp, &r, &t_x_bl); sc_add(&tmp, &tmp, &e_bl); sc_neg(&ms[q], &tmp); mp[q++] = pc->B_blinding; }
    sc one; sc_one(&one);
    for (size_t i = 0; i < padded_n; i++) {                                              /* g_scalars (verifier.rs:428-432) */
        const sc *u1 = i < n1 ? &one : &u; sc a1, a2;
        sc_mul(&a1, &x, &yneg_wR[i]); sc_mul(&a2, &ipp.a, &s[i]); sc_sub(&a1, &a1, &a2); sc_mul(&ms[q], u1, &a1); mp[q++] = bg->G[i];
    }
    for (size_t i = 0; i < padded_n; i++) {                                              /* h_scalars (verifier.rs:434-442) */
        const sc *u1 = i < n1 ? &one : &u; sc a1, a2, zero; sc_zero(&zero);
        const sc *wLi = i < n ? &wL[i] : &zero, *wOi = i < n ? &wO[i] : &zero;
        sc_mul(&a1, &x, wLi); sc_add(&a1, &a1, wOi); sc_mul(&a2, &ipp.b, &s[padded_n - 1 - i]); sc_sub(&a1, &a1, &a2);
        sc_mul(&a1, &y_inv_vec[i], &a1); sc_sub(&a1, &a1, &one); sc_mul(&ms[q], u1, &a1); mp[q++] = bg->H[i];
    }
    for (int i = 0; i < k; i++) { ms[q] = u_sq[i]; bad |= !ge_decode(&mp[q++], ipp.LR + 64 * i); }
    for (int i = 0; i < k; i++) { ms[q] = u_inv_sq[i]; bad |= !ge_decode(&mp[q++], ipp.LR + 64 * i + 32); }
    rc = ORC_OK;
    if (bad) rc = ORC_VERIFICATION_ERROR;
    else { ge mega; ge_msm_vartime(&mega, ms, mp, nt); if (!ge_is_identity(&mega)) rc = ORC_VERIFICATION_ERROR; }
    (void)pad;
    free(wL); free(wR); free(wO); free(wV); free(s); free(y_inv_vec); free(yneg_wR); free(ms); free(mp);
    return rc;
}

/* ------------------------------------------------------------------ gadgets */
typedef struct { size_t k; r1_var *x, *y; } shuffle_ctx;
/* the deferred closure of ShuffleProof::gadget — benches/r1cs.rs:48-66 */
static int shuffle_deferred(r1_cs *cs, void *p) {
    shuffle_ctx *c = p; size_t k = c->k;
    sc z; t_challenge_scalar(cs->tr, "shuffle challenge", &z); sc mz; sc_neg(&mz, &z);
    r1_var one = var_of(R1_ONE, 0), o, prev;
    for (int side = 0; side < 2; side++) {
        const r1_var *v = side ? c->y : c->x;
        r1_lc a = lc_var(v[k - 1]), b = lc_var(v[k - 2]); lc_push(&a, one, &mz); lc_push(&b, one, &mz);
        cs_multiply(cs, a, b, NULL, NULL, &prev);
        for (size_t i = k - 2; i-- > 0;) { r1_lc l = lc_var(prev), r = lc_var(v[i]); lc_push(&r, one, &mz); cs_multiply(cs, l, r, NULL, NULL, &prev); }
        if (side == 0) o = prev;
        else { r1_lc d = lc_var(o); lc_push_i(&d, prev, -1); cs_constrain(cs, d); }
    }
    return 0;
}
static void shuffle_gadget(r1_cs *cs, shuffle_ctx *c) {                                /* benches/r1cs.rs:35-47 */
    if (c->k == 1) { r1_lc d = lc_var(c->y[0]); lc_push_i(&d, c->x[0], -1); cs_constrain(cs, d); return; }
    cs_specify_randomized(cs, shuffle_deferred, c);
}
/* example_gadget — tests/r1cs.rs:225-236: (a1 + a2) * (b1 + b2) = c1 + c2 with c2 a constant */
static void example_gadget(r1_cs *cs, const r1_var v[5], uint64_t c2) {
    r1_lc a = lc_var(v[0]), b = lc_var(v[2]); lc_push_i(&a, v[1], 1); lc_push_i(&b, v[3], 1);
    r1_var o; cs_multiply(cs, a, b, NULL, NULL, &o);
    r1_lc c = lc_var(v[4]); sc s; sc_from_u64(&s, c2); lc_push(&c, var_of(R1_ONE, 0), &s); lc_push_i(&c, o, -1);
    cs_constrain(cs, c);
}
/* range_proof gadget — tests/r1cs.rs:366-385 */
static void range_gadget(r1_cs *cs, r1_var vvar, uint64_t assignment, size_t n) {
    r1_lc v = lc_var(vvar); sc exp_2; sc_one(&exp_2);
    for (size_t i = 0; i < n; i++) {
        uint64_t bit = (assignment >> i) & 1; sc lv, rv; sc_from_u64(&lv, 1 - bit); sc_from_u64(&rv, bit);
        r1_var a, b, o; cs_allocate_multiplier(cs, &lv, &rv, &a, &b, &o);
        cs_constrain(cs, lc_var(o));
        r1_lc c = lc_var(a); lc_push_i(&c, b, 1); lc_push_i(&c, var_of(R1_ONE, 0), -1); cs_constrain(cs, c);
        sc neg; sc_neg(&neg, &exp_2); lc_push(&v, b, &neg);
        sc_add(&exp_2, &exp_2, &exp_2);
    }
    cs_constrain(cs, v);
}
#endif
