/* oracle/mpc.h — TEST INFRASTRUCTURE ONLY (see bp_oracle.c).  CPU restatement of the aggregated range-proof MPC messages:
 *   src/range_proof/party.rs    (Party::new :35-60, assign_position_with_rng :87-144,
 *                                                 apply_challenge_with_rng :182-237, apply_challenge :279-305)
 *   src/range_proof/dealer.rs   (Dealer::new :37-81, receive_bit_commitments :98-137,
 *                                                 receive_poly_commitments :160-197, assemble_shares :226-293,
 *                                                 receive_shares_with_rng :319-355)
 *   src/range_proof/messages.rs (ProofShare::check_size :56-81, audit_share :84-167)
 * Stateless form: a party is (v, v_blinding, n, j, rng seed); every stage replays the party's ChaCha stream in the
 * reference's draw order (a_blinding, s_blinding, s_L[n], s_R[n], t_1_blinding, t_2_blinding), so the three party
 * calls need no stored state.  Wire layouts: BitCommitment = V_j | A_j | S_j (96 B), PolyCommitment = T_1_j | T_2_j
 * (64 B), ProofShare = t_x | t_x_blinding | e_blinding | l_vec[n] | r_vec[n] (32*(3+2n) B).
 * Parity: unpinned by fixed vectors (the reference's MPC tests are randomised round-trips and negative tests,
 * src/range_proof/mod.rs tests); pinned transitively — the aggregated proof these shares assemble into must verify under
 * the golden-pinned verifier, and equals rp_prove's bytes when the parties share one RNG stream. */

#define ORC_WRONG_NUM_SHARES 9        /* MPCError::WrongNum{BitCommitments,PolyCommitments,ProofShares} */
#define ORC_MALFORMED_SHARES 10       /* MPCError::MalformedProofShares { bad_shares } */

typedef struct {
    sc a_bl, s_bl, t1_bl, t2_bl, t0, t1, t2, ozz;
    sc sL[64], sR[64], l0[64], l1[64], r0[64], r1[64];
} mpc_party;

/* stage 1 secrets (party.rs:98,114-116) */
static void mpc_party_draw_bits(mpc_party *p, chacha_rng *rng, size_t n) {
    rng_scalar(rng, &p->a_bl); rng_scalar(rng, &p->s_bl);
    for (size_t i = 0; i < n; i++) rng_scalar(rng, &p->sL[i]);
    for (size_t i = 0; i < n; i++) rng_scalar(rng, &p->sR[i]);
}
/* stage 2: l(x), r(x), t(x) and the T blindings (party.rs:182-237) */
static void mpc_party_poly(mpc_party *p, chacha_rng *rng, uint64_t v, size_t n, size_t j, const sc *y, const sc *z) {
    sc zz, offset_y, offset_z, exp_y, exp_2, one; sc_mul(&zz, z, z); sc_one(&one);
    scalar_exp_vartime(&offset_y, y, (uint64_t)(j * n)); scalar_exp_vartime(&offset_z, z, (uint64_t)j);
    sc_mul(&p->ozz, &zz, &offset_z); exp_y = offset_y; sc_one(&exp_2);
    for (size_t i = 0; i < n; i++) {
        sc aL, aR, u, w; sc_from_u64(&aL, (v >> i) & 1); sc_sub(&aR, &aL, &one);
        sc_sub(&p->l0[i], &aL, z); p->l1[i] = p->sL[i];
        sc_add(&u, &aR, z); sc_mul(&u, &exp_y, &u); sc_mul(&w, &p->ozz, &exp_2); sc_add(&p->r0[i], &u, &w);
        sc_mul(&p->r1[i], &exp_y, &p->sR[i]);
        sc_mul(&exp_y, &exp_y, y); sc_add(&exp_2, &exp_2, &exp_2);
    }
    sc acc, lsum, rsum; inner_product(&p->t0, p->l0, p->r0, n); inner_product(&p->t2, p->l1, p->r1, n); sc_zero(&acc);   /* util.rs:86-100 */
    for (size_t i = 0; i < n; i++) { sc pr; sc_add(&lsum, &p->l0[i], &p->l1[i]); sc_add(&rsum, &p->r0[i], &p->r1[i]); sc_mul(&pr, &lsum, &rsum); sc_add(&acc, &acc, &pr); }
    sc_sub(&p->t1, &acc, &p->t0); sc_sub(&p->t1, &p->t1, &p->t2);
    rng_scalar(rng, &p->t1_bl); rng_scalar(rng, &p->t2_bl);
}
static int mpc_party_check(const bp_gens *bg, size_t n, size_t j) {
    if (!valid_bitsize(n)) return ORC_INVALID_BITSIZE;                                   /* party.rs:43-45 */
    if (bg->gens_capacity < n) return ORC_INVALID_GENS_LENGTH;                           /* party.rs:46-48 */
    if (bg->party_capacity <= j) return ORC_INVALID_GENS_LENGTH;                         /* party.rs:93-95 */
    return ORC_OK;
}

/* Party::new + assign_position_with_rng -> BitCommitment */
static int mpc_party_bit_commitment(const bp_gens *bg, const pedersen_gens *pc, uint64_t v, const sc *v_bl, size_t n, size_t j, const uint8_t seed[32], uint8_t out[96]) {
    int rc = mpc_party_check(bg, n, j); if (rc) return rc;
    chacha_rng rng; chacha_seed(&rng, seed);
    mpc_party p; mpc_party_draw_bits(&p, &rng, n);
    const ge *Gj = bg->G + j * bg->gens_capacity, *Hj = bg->H + j * bg->gens_capacity;
    ge V, A, S; sc vs; sc_from_u64(&vs, v);
    { sc s2[2] = { vs, *v_bl }; ge p2[2] = { pc->B, pc->B_blinding }; ge_msm_vartime(&V, s2, p2, 2); }
    ge_scalarmult(&A, &p.a_bl, &pc->B_blinding);
    for (size_t i = 0; i < n; i++) { if ((v >> i) & 1) ge_add(&A, &A, &Gj[i]); else ge_sub(&A, &A, &Hj[i]); }
    sc ms[129]; ge mp[129]; ms[0] = p.s_bl; mp[0] = pc->B_blinding;
    for (size_t i = 0; i < n; i++) { ms[1 + i] = p.sL[i]; mp[1 + i] = Gj[i]; ms[1 + n + i] = p.sR[i]; mp[1 + n + i] = Hj[i]; }
    ge_msm_vartime(&S, ms, mp, 2 * n + 1);
    ge_encode(out, &V); ge_encode(out + 32, &A); ge_encode(out + 64, &S);
    return ORC_OK;
}
/* PartyAwaitingBitChallenge::apply_challenge_with_rng -> PolyCommitment */
static int mpc_party_poly_commitment(const bp_gens *bg, const pedersen_gens *pc, uint64_t v, size_t n, size_t j, const uint8_t seed[32], const sc *y, const sc *z, uint8_t out[64]) {
    int rc = mpc_party_check(bg, n, j); if (rc) return rc;
    chacha_rng rng; chacha_seed(&rng, seed);
    mpc_party p; mpc_party_draw_bits(&p, &rng, n); mpc_party_poly(&p, &rng, v, n, j, y, z);
    ge T1, T2;
    { sc s2[2] = { p.t1, p.t1_bl }; ge p2[2] = { pc->B, pc->B_blinding }; ge_msm_vartime(&T1, s2, p2, 2); }
    { sc s2[2] = { p.t2, p.t2_bl }; ge p2[2] = { pc->B, pc->B_blinding }; ge_msm_vartime(&T2, s2, p2, 2); }
    ge_encode(out, &T1); ge_encode(out + 32, &T2);
    return ORC_OK;
}
/* PartyAwaitingPolyChallenge::apply_challenge -> ProofShare */
static int mpc_party_proof_share(const bp_gens *bg, uint64_t v, const sc *v_bl, size_t n, size_t j, const uint8_t seed[32], const sc *y, const sc *z, const sc *x, uint8_t *out) {
    int rc = mpc_party_check(bg, n, j); if (rc) return rc;
    if (sc_is_zero(x)) return ORC_MALICIOUS_DEALER;                                      /* party.rs:282-284 */
    chacha_rng rng; chacha_seed(&rng, seed);
    mpc_party p; mpc_party_draw_bits(&p, &rng, n); mpc_party_poly(&p, &rng, v, n, j, y, z);
    sc t_x, t_x_bl, e_bl, e, u;
    sc_mul(&e, x, &p.t2); sc_add(&e, &e, &p.t1); sc_mul(&e, x, &e); sc_add(&t_x, &e, &p.t0);            /* t_poly.eval(x) */
    sc_mul(&u, &p.ozz, v_bl); sc_mul(&e, x, &p.t2_bl); sc_add(&e, &e, &p.t1_bl); sc_mul(&e, x, &e); sc_add(&t_x_bl, &e, &u);
    sc_mul(&e, &p.s_bl, x); sc_add(&e_bl, &e, &p.a_bl);
    sc_tobytes(out, &t_x); sc_tobytes(out + 32, &t_x_bl); sc_tobytes(out + 64, &e_bl);
    for (size_t i = 0; i < n; i++) {
        sc q, lv, rv; sc_mul(&q, &p.l1[i], x); sc_add(&lv, &p.l0[i], &q); sc_mul(&q, &p.r1[i], x); sc_add(&rv, &p.r0[i], &q);
        sc_tobytes(out + 96 + 32 * i, &lv); sc_tobytes(out + 96 + 32 * (n + i), &rv);
    }
    return ORC_OK;
}

/* ProofShare::audit_share (messages.rs:84-167); share = 32*(3+2n) bytes.  0 = Ok, 1 = Err */
static int mpc_audit_share(const bp_gens *bg, const pedersen_gens *pc, size_t n, size_t j, const uint8_t bitc[96], const sc *y, const sc *z,
                           const uint8_t polyc[64], const sc *x, const uint8_t *share) {
    if (n > bg->gens_capacity || j >= bg->party_capacity) return 1;                      /* check_size :56-81 (vector lengths are fixed by the wire layout) */
    sc t_x, t_x_bl, e_bl, l[64], r[64];
    if (!sc_from_canonical(&t_x, share) || !sc_from_canonical(&t_x_bl, share + 32) || !sc_from_canonical(&e_bl, share + 64)) return 1;
    for (size_t i = 0; i < n; i++) if (!sc_from_canonical(&l[i], share + 96 + 32 * i) || !sc_from_canonical(&r[i], share + 96 + 32 * (n + i))) return 1;
    ge A_j, S_j, V_j, T1_j, T2_j;
    if (!ge_decode(&A_j, bitc + 32) || !ge_decode(&S_j, bitc + 64) || !ge_decode(&T1_j, polyc) || !ge_decode(&T2_j, polyc + 32)) return 1;
    sc zz, minus_z, z_j, y_jn, y_jn_inv, y_inv, ip;
    sc_mul(&zz, z, z); sc_neg(&minus_z, z);
    scalar_exp_vartime(&z_j, z, (uint64_t)j); scalar_exp_vartime(&y_jn, y, (uint64_t)(j * n));
    sc_invert(&y_jn_inv, &y_jn); sc_invert(&y_inv, y);
    inner_product(&ip, l, r, n);
    if (!sc_eq(&t_x, &ip)) return 1;                                                     /* :112-114 */
    const ge *Gj = bg->G + j * bg->gens_capacity, *Hj = bg->H + j * bg->gens_capacity;
    sc ms[131]; ge mp[131]; size_t o = 0;
    sc_one(&ms[o]); mp[o++] = A_j; ms[o] = *x; mp[o++] = S_j; sc_neg(&ms[o], &e_bl); mp[o++] = pc->B_blinding;
    for (size_t i = 0; i < n; i++) { sc_sub(&ms[o], &minus_z, &l[i]); mp[o++] = Gj[i]; }               /* g :116 */
    sc exp_2, exp_y_inv, zzzj; sc_one(&exp_2); sc_one(&exp_y_inv); sc_mul(&zzzj, &zz, &z_j);
    for (size_t i = 0; i < n; i++) {                                                     /* h :117-125 */
        sc f, a, b, nr; sc_mul(&f, &exp_y_inv, &y_jn_inv); sc_neg(&nr, &r[i]);
        sc_mul(&a, &f, &nr); sc_mul(&b, &zzzj, &exp_2); sc_mul(&b, &f, &b);
        sc_add(&ms[o], z, &a); sc_add(&ms[o], &ms[o], &b); mp[o++] = Hj[i];
        sc_add(&exp_2, &exp_2, &exp_2); sc_mul(&exp_y_inv, &exp_y_inv, &y_inv);
    }
    ge P; ge_msm_vartime(&P, ms, mp, o);
    if (!ge_is_identity(&P)) return 1;                                                   /* :140-142 */
    if (!ge_decode(&V_j, bitc)) return 1;                                                /* :144 */
    sc sum_y, sum_2, two, delta, u, w; sc_from_u64(&two, 2);
    sum_of_powers(&sum_y, y, n); sum_of_powers(&sum_2, &two, n);
    sc_sub(&u, z, &zz); sc_mul(&u, &u, &sum_y); sc_mul(&u, &u, &y_jn);
    sc_mul(&w, z, &zz); sc_mul(&w, &w, &sum_2); sc_mul(&w, &w, &z_j); sc_sub(&delta, &u, &w);           /* :148 */
    sc ts[5]; ge tp[5] = { V_j, T1_j, T2_j, pc->B, pc->B_blinding };
    ts[0] = zzzj; ts[1] = *x; sc_mul(&ts[2], x, x); sc_sub(&ts[3], &delta, &t_x); sc_neg(&ts[4], &t_x_bl);
    ge Tc; ge_msm_vartime(&Tc, ts, tp, 5);
    return ge_is_identity(&Tc) ? 0 : 1;                                                  /* :162-166 */
}

/* Dealer::new + receive_bit_commitments: transcript in/out, -> y, z, A, S */
static int mpc_dealer_bit_challenge(const bp_gens *bg, merlin *t, size_t n, size_t m, const uint8_t *bitc, sc *y, sc *z, uint8_t A_out[32], uint8_t S_out[32]) {
    if (!valid_bitsize(n)) return ORC_INVALID_BITSIZE;                                   /* dealer.rs:44-55 */
    if (!is_pow2(m)) return ORC_INVALID_AGGREGATION;
    if (bg->gens_capacity < n || bg->party_capacity < m) return ORC_INVALID_GENS_LENGTH;
    t_rangeproof_domain_sep(t, n, m);                                                    /* dealer.rs:70 */
    ge A, S, q; ge_identity(&A); ge_identity(&S);
    for (size_t j = 0; j < m; j++) {
        t_append_point(t, "V", bitc + 96 * j);
        if (!ge_decode(&q, bitc + 96 * j + 32)) return ORC_INVALID_POINT;
        ge_add(&A, &A, &q);
        if (!ge_decode(&q, bitc + 96 * j + 64)) return ORC_INVALID_POINT;
        ge_add(&S, &S, &q);
    }
    ge_encode(A_out, &A); ge_encode(S_out, &S);
    t_append_point(t, "A", A_out); t_append_point(t, "S", S_out);
    t_challenge_scalar(t, "y", y); t_challenge_scalar(t, "z", z);
    return ORC_OK;
}
/* receive_poly_commitments: transcript in/out, -> x, T_1, T_2 */
static int mpc_dealer_poly_challenge(merlin *t, size_t m, const uint8_t *polyc, sc *x, uint8_t T1_out[32], uint8_t T2_out[32]) {
    ge T1, T2, q; ge_identity(&T1); ge_identity(&T2);
    for (size_t j = 0; j < m; j++) {
        if (!ge_decode(&q, polyc + 64 * j)) return ORC_INVALID_POINT;
        ge_add(&T1, &T1, &q);
        if (!ge_decode(&q, polyc + 64 * j + 32)) return ORC_INVALID_POINT;
        ge_add(&T2, &T2, &q);
    }
    ge_encode(T1_out, &T1); ge_encode(T2_out, &T2);
    t_append_point(t, "T_1", T1_out); t_append_point(t, "T_2", T2_out);
    t_challenge_scalar(t, "x", x);
    return ORC_OK;
}
/* The whole dealer run over collected messages: challenges, assemble_shares, verification with the initial transcript, audit on
 * failure.  trusted != 0 = receive_trusted_shares (no verification).  bad[j] = 1 for every share the audit rejects. */
static int mpc_dealer_run(const bp_gens *bg, const pedersen_gens *pc, const merlin *initial, size_t n, size_t m, const uint8_t *bitc, const uint8_t *polyc,
                          const uint8_t *shares, int trusted, const uint8_t verify_seed[32], uint8_t *proof_out, uint8_t *bad) {
    merlin t = *initial; sc y, z, x; uint8_t Ac[32], Sc[32], T1c[32], T2c[32];
    int rc = mpc_dealer_bit_challenge(bg, &t, n, m, bitc, &y, &z, Ac, Sc); if (rc) return rc;
    rc = mpc_dealer_poly_challenge(&t, m, polyc, &x, T1c, T2c); if (rc) return rc;
    size_t N = n * m, slen = 32 * (3 + 2 * n);
    memset(bad, 0, m);
    sc t_x, t_x_bl, e_bl; sc_zero(&t_x); sc_zero(&t_x_bl); sc_zero(&e_bl);
    sc *lv = malloc(sizeof(sc) * N), *rv = malloc(sizeof(sc) * N);
    int malformed = 0;
    for (size_t j = 0; j < m; j++) {                                                     /* assemble_shares :245-270; a non-canonical scalar cannot be a Scalar in the reference */
        const uint8_t *s = shares + slen * j; sc a, b, c;
        if (!sc_from_canonical(&a, s) || !sc_from_canonical(&b, s + 32) || !sc_from_canonical(&c, s + 64)) { bad[j] = 1; malformed = 1; continue; }
        sc_add(&t_x, &t_x, &a); sc_add(&t_x_bl, &t_x_bl, &b); sc_add(&e_bl, &e_bl, &c);
        for (size_t i = 0; i < n; i++)
            if (!sc_from_canonical(&lv[j * n + i], s + 96 + 32 * i) || !sc_from_canonical(&rv[j * n + i], s + 96 + 32 * (n + i))) { bad[j] = 1; malformed = 1; }
    }
    if (malformed) { free(lv); free(rv); return ORC_MALFORMED_SHARES; }
    t_append_scalar(&t, "t_x", &t_x); t_append_scalar(&t, "t_x_blinding", &t_x_bl); t_append_scalar(&t, "e_blinding", &e_bl);
    sc w; t_challenge_scalar(&t, "w", &w);
    ge Q; ge_scalarmult(&Q, &w, &pc->B);
    sc *Gf = malloc(sizeof(sc) * N), *Hf = malloc(sizeof(sc) * N); sc y_inv, e; sc_invert(&y_inv, &y); sc_one(&e);
    for (size_t i = 0; i < N; i++) { sc_one(&Gf[i]); Hf[i] = e; sc_mul(&e, &e, &y_inv); }
    ge *G = malloc(sizeof(ge) * N), *H = malloc(sizeof(ge) * N);
    for (size_t i = 0; i < N; i++) { G[i] = bg->G[(i / n) * bg->gens_capacity + (i % n)]; H[i] = bg->H[(i / n) * bg->gens_capacity + (i % n)]; }
    memcpy(proof_out, Ac, 32); memcpy(proof_out + 32, Sc, 32); memcpy(proof_out + 64, T1c, 32); memcpy(proof_out + 96, T2c, 32);
    sc_tobytes(proof_out + 128, &t_x); sc_tobytes(proof_out + 160, &t_x_bl); sc_tobytes(proof_out + 192, &e_bl);
    ipp_create(&t, &Q, Gf, Hf, G, H, lv, rv, N, proof_out + 224);
    free(Gf); free(Hf); free(G); free(H); free(lv); free(rv);
    if (trusted) return ORC_OK;
    uint8_t *Vs = malloc(32 * m);
    for (size_t j = 0; j < m; j++) memcpy(Vs + 32 * j, bitc + 96 * j, 32);
    merlin tv = *initial; chacha_rng vr; chacha_seed(&vr, verify_seed);
    rc = rp_verify(bg, pc, &tv, proof_out, 32 * (9 + 2 * (size_t)lg2(N)), Vs, m, n, &vr);               /* dealer.rs:330-337 */
    free(Vs);
    if (rc == ORC_OK) return ORC_OK;
    for (size_t j = 0; j < m; j++)                                                       /* dealer.rs:340-353 */
        bad[j] = (uint8_t)mpc_audit_share(bg, pc, n, j, bitc + 96 * j, &y, &z, polyc + 64 * j, &x, shares + slen * j);
    return ORC_MALFORMED_SHARES;
}
