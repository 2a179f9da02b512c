/* TEST-ONLY: the mock engine (mock_bpmsm.c, included whole) plus bp_r1cs_verify_batch, built as libmockbpmsm_r1cs.so by
 * build_mock_r1cs.py for tests/test_r1cs_batch.py's CPU run of its GPU tests and for the R1CS weights tests/test_batch_soundness.py reads back.  Like the rest of the mock this is not a check of the
 * engine: each proof gets its own mega-check, one oracle MSM, with no combination across proofs. */
#include "mock_bpmsm.c"

/* the dims and challenge arrays of the last bp_r1cs_verify_batch call, for tests that need each proof's weight rho (chal[7 j' + 5],
 * j' counting the 7 + lg(padded_n) scalars of the proofs before it) without a GPU */
static uint8_t *g_last_chal; static size_t g_last_chal_len;
static uint32_t *g_last_dims; static size_t g_last_n;
/* copies up to cap bytes of the last challenge array to out; returns its length in bytes */
size_t mock_r1cs_last_chal(uint8_t *out, size_t cap) { if (out) memcpy(out, g_last_chal, cap < g_last_chal_len ? cap : g_last_chal_len); return g_last_chal_len; }
/* copies up to cap dims words (4 per proof) to out; returns the number of proofs of the last call */
size_t mock_r1cs_last_dims(uint32_t *out, size_t cap) { if (out) memcpy(out, g_last_dims, 4 * (cap < 4 * g_last_n ? cap : 4 * g_last_n)); return g_last_n; }
static void keep_last_call(size_t n_proofs, const uint32_t *dims, const uint8_t *chal) {
    size_t nsc = 0;
    for (size_t j = 0; j < n_proofs; j++) { uint32_t N = dims[4 * j], k = 0; while (k < 32 && (1u << k) < N) k++; nsc += 7 + k; }
    free(g_last_chal); free(g_last_dims);
    g_last_chal = malloc(32 * nsc); memcpy(g_last_chal, chal, 32 * nsc); g_last_chal_len = 32 * nsc;
    g_last_dims = malloc(16 * n_proofs); memcpy(g_last_dims, dims, 16 * n_proofs); g_last_n = n_proofs;
}

/* ---- R1CS batch verification, literally: each proof's own mega-check (verifier.rs:459-491) as one MSM, with its G/H scalars written out
 * as verifier.rs:409-442 defines them; no combination across proofs */
int bp_r1cs_verify_batch(bp_ctx *c, bp_gens *gens, size_t n_proofs, const uint32_t *dims, const uint8_t *chal, const uint8_t *wL, const uint8_t *wR, const uint8_t *wO,
                         const uint8_t *scalars, const uint32_t *point_idx, const uint8_t *dyn_points, size_t n_dyn, uint8_t *verdicts) {
    if (!c || !gens || !dims || !chal || !verdicts || n_proofs == 0) return BP_ERR_INVALID_ARGUMENT;
    keep_last_call(n_proofs, dims, chal);
    TIMED_BEGIN;
    size_t co = 0, wo = 0, to = 0; int rc = BP_OK;
    sc one; sc_from_u64(&one, 1);
    for (size_t j = 0; j < n_proofs && rc == BP_OK; j++) {
        uint32_t N = dims[4 * j], n1 = dims[4 * j + 1], n = dims[4 * j + 2], nt = dims[4 * j + 3], k = 0;
        while (k < 32 && (1u << k) < N) k++;
        if (!N || (N & (N - 1)) || n > N || n1 > n || N > gens->cap) { snprintf(c->err, sizeof c->err, "bp_r1cs_verify_batch: inconsistent dims"); rc = BP_ERR_INVALID_ARGUMENT; break; }
        sc ch[7 + 32], t, t2;
        if ((rc = load_scalars(ch, chal + 32 * co, 7 + k)) != BP_OK) break;
        const sc *x = &ch[0], *yi = &ch[1], *u = &ch[2], *a = &ch[3], *b = &ch[4], *usq = &ch[7];
        size_t T = 2 * (size_t)N + nt;
        sc *s = malloc(T * sizeof(sc)), *sv = malloc(N * sizeof(sc)); ge *p = malloc(T * sizeof(ge));
        for (uint32_t i = 0; i < N; i++) { sv[i] = ch[6]; for (uint32_t bit = 0; bit < k; bit++) if ((i >> bit) & 1u) sc_mul(&sv[i], &sv[i], &usq[k - 1 - bit]); }
        sc ypow = one;
        for (uint32_t i = 0; i < N && rc == BP_OK; i++) {
            sc wl, wr, wo_, zero; sc_zero(&zero); wl = wr = wo_ = zero;
            if (i < n && (!sc_from_canonical(&wl, wL + 32 * (wo + i)) || !sc_from_canonical(&wr, wR + 32 * (wo + i)) || !sc_from_canonical(&wo_, wO + 32 * (wo + i)))) { rc = BP_ERR_NONCANONICAL_SCALAR; break; }
            const sc *u1 = i < n1 ? &one : u;
            sc_mul(&t, x, &ypow); sc_mul(&t, &t, &wr); sc_mul(&t2, a, &sv[i]); sc_sub(&t, &t, &t2); sc_mul(&s[i], u1, &t);                 /* u1 (x y^-i wR_i - a s_i) */
            sc_mul(&t, x, &wl); sc_add(&t, &t, &wo_); sc_mul(&t2, b, &sv[N - 1 - i]); sc_sub(&t, &t, &t2); sc_mul(&t, &ypow, &t); sc_sub(&t, &t, &one);
            sc_mul(&s[N + i], u1, &t);                                                                                                   /* u1 (y^-i (x wL_i + wO_i - b s_{N-1-i}) - 1) */
            p[i] = gens->tab[2 + i]; p[N + i] = gens->tab[2 + gens->parties * gens->cap + i];
            sc_mul(&ypow, &ypow, yi);
        }
        uint8_t verdict = BP_PROOF_OK;
        if (rc == BP_OK) rc = load_scalars(s + 2 * N, scalars + 32 * to, nt);
        for (uint32_t e = 0; e < nt && rc == BP_OK; e++) {
            uint32_t v = point_idx[to + e];
            if (v & BP_POINT_DYNAMIC) {
                uint32_t d = v & 0x7fffffffu;
                if (d >= n_dyn || !dyn_points) { rc = BP_ERR_INVALID_ARGUMENT; break; }
                if (!ge_decode(&p[2 * N + e], dyn_points + 32 * d)) verdict = BP_PROOF_VERIFICATION_ERROR;       /* optional_multiscalar_mul -> None */
            } else if (v >= gens->n_points) { rc = BP_ERR_INVALID_ARGUMENT; break; }
            else p[2 * N + e] = gens->tab[v];
        }
        if (rc == BP_OK && verdict == BP_PROOF_OK) {
            uint8_t out[32], z = 0; msm_ge(out, s, p, T);
            for (int i = 0; i < 32; i++) z |= out[i];
            verdict = z ? BP_PROOF_VERIFICATION_ERROR : BP_PROOF_OK;
        }
        verdicts[j] = verdict;
        free(s); free(sv); free(p);
        co += 7 + k; wo += n; to += nt;
    }
    TIMED_END; return rc;
}
