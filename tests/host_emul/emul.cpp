// TEST-ONLY host build of the device math headers (fe/ge/sc/merlin/rp/msm_common .cuh compiled
// with g++: the portable branches of the __host__ __device__ functions).  It lets the CPU-only
// test tier check the limb algorithms, point formulas, transcript replay, verification scalars and
// the Pippenger bookkeeping against the oracle without a GPU.  Nothing in the product links this.
#include <cstring>
#include <vector>
#include "../../bulletproofs_b200/csrc/ge.cuh"
#include "../../bulletproofs_b200/csrc/sc.cuh"
#include "../../bulletproofs_b200/csrc/merlin.cuh"
#include "../../bulletproofs_b200/csrc/rp.cuh"
#include "../../bulletproofs_b200/csrc/msm_common.cuh"

extern "C" {

void emul_fe_op(int op, const uint8_t *a, const uint8_t *b, uint8_t *out) {
    fe x = fe_frombytes_raw(a), y = fe_frombytes_raw(b), r;
    switch (op) {
        case 0: r = fe_add(x, y); break;
        case 1: r = fe_sub(x, y); break;
        case 2: r = fe_mul(x, y); break;
        case 3: r = fe_invert(x); break;
        case 4: r = fe_pow22523(x); break;
        case 5: r = fe_neg(x); break;
        default: r = fe_sq(x);
    }
    fe_tobytes(out, r);
}
int emul_point_roundtrip(const uint8_t *in, uint8_t *out) {
    fe x, y; if (!ge_decode(x, y, in)) return 0;
    ge_encode(out, ge_from_niels(ge_to_niels_affine(x, y))); return 1;
}
int emul_point_double_encode(const uint8_t *in, uint8_t *out) {
    fe x, y; if (!ge_decode(x, y, in)) return 0;
    ge_encode(out, ge_dbl(ge_from_niels(ge_to_niels_affine(x, y)))); return 1;
}
int emul_point_add(const uint8_t *a, const uint8_t *b, int sub, uint8_t *out) {
    fe x, y, x2, y2; if (!ge_decode(x, y, a) || !ge_decode(x2, y2, b)) return 0;
    ge_ext p = ge_from_niels(ge_to_niels_affine(x, y)); ge_niels q = ge_to_niels_affine(x2, y2);
    ge_ext r1 = sub ? ge_msub(p, q) : ge_madd(p, q);
    ge_ext r2 = sub ? ge_sub(p, ge_from_niels(q)) : ge_add(p, ge_from_niels(q));
    uint8_t o2[32]; ge_encode(out, r1); ge_encode(o2, r2);
    return memcmp(out, o2, 32) == 0 ? 1 : -1;
}
void emul_from_uniform(const uint8_t *in, uint8_t *out) { ge_encode(out, ge_from_uniform(in)); }
int emul_is_identity_of_diff(const uint8_t *a, const uint8_t *b) {   // a - b in the identity coset?
    fe x, y, x2, y2; if (!ge_decode(x, y, a) || !ge_decode(x2, y2, b)) return -1;
    return ge_is_identity(ge_msub(ge_from_niels(ge_to_niels_affine(x, y)), ge_to_niels_affine(x2, y2))) ? 1 : 0;
}

void emul_sc_mul(const uint8_t *a, const uint8_t *b, uint8_t *out) {
    sc x = sc_to_mont(sc_load(a)), y = sc_to_mont(sc_load(b)); sc_store(out, sc_from_mont(sc_mont_mul(x, y)));
}
// sum of n <= 32 products through the lazy-reduction accumulator (sc_wide_mac / sc_wide_redc), canonical bytes in and out
void emul_sc_sum_products(const uint8_t *a, const uint8_t *b, uint32_t n, uint8_t *out) {
    sc_wide acc = sc_wide_zero();
    for (uint32_t i = 0; i < n; i++) sc_wide_mac(acc, sc_to_mont(sc_load(a + 32 * i)), sc_to_mont(sc_load(b + 32 * i)));
    sc_store(out, sc_from_mont(sc_wide_redc(acc)));
}
void emul_sc_addsub(const uint8_t *a, const uint8_t *b, int sub, uint8_t *out) { sc x = sc_load(a), y = sc_load(b); sc_store(out, sub ? sc_sub(x, y) : sc_add(x, y)); }
void emul_sc_invert(const uint8_t *a, uint8_t *out) { sc_store(out, sc_from_mont(sc_mont_invert(sc_to_mont(sc_load(a))))); }
void emul_sc_from_wide(const uint8_t *in, uint8_t *out) { sc_store(out, sc_from_mont(sc_mont_from_wide(in))); }

void emul_transcript_new(const uint8_t *label, uint32_t len, uint8_t *ser) { alignas(8) uint8_t st[200]; merlin_t m; m.st = st; merlin_init(m, label, len); merlin_store(ser, m); }
void emul_transcript_append(uint8_t *ser, const char *label, const uint8_t *msg, uint32_t len) { alignas(8) uint8_t st[200]; merlin_t m; m.st = st; merlin_load(m, ser); merlin_append(m, label, msg, len); merlin_store(ser, m); }
void emul_transcript_challenge(uint8_t *ser, const char *label, uint8_t *out, uint32_t len) { alignas(8) uint8_t st[200]; merlin_t m; m.st = st; merlin_load(m, ser); merlin_challenge(m, label, out, len); merlin_store(ser, m); }

// full verification-scalar vector of one proof in the order [B~, B, G.., H.. | A,S,T1,T2,L..,R..,V..], canonical bytes
int emul_rp_scalars(const uint8_t *proof, uint32_t k, const uint8_t *V, uint32_t n, uint32_t m, const uint8_t *tstate, const uint8_t *seed, uint8_t *out) {
    static rp_head h; static rp_challenges ch; alignas(8) uint8_t st[200];
    rp_transcript(ch, proof, k, V, n, m, tstate, seed, st);
    if (ch.status) return (int)ch.status;
    std::vector<sc> tab(rp_tab_size(k, m)), pow2(64);
    for (int e = 0; e < 64; e++) pow2[e] = sc_mont_from_u64(1ULL << e);
    rp_scalars_head(h, tab.data(), pow2.data(), ch, proof, k, n, m);
    uint32_t N = n * m, S = 2 + 2 * N, D = 4 + 2 * k + m;
    sc_store(out, sc_from_mont(h.blinding_scalar)); sc_store(out + 32, sc_from_mont(h.basepoint_scalar));
    for (uint32_t i = 0; i < N; i++) { sc g, hh; rp_scalars_gh(h, tab.data(), i, k, g, hh); sc_store(out + 32 * (2 + i), sc_from_mont(g)); sc_store(out + 32 * (2 + N + i), sc_from_mont(hh)); }
    for (uint32_t i = 0; i < D; i++) sc_store(out + 32 * (S + i), sc_from_mont(rp_scalars_dynamic(h, i, k)));
    return 0;
}

int emul_pick_window(uint64_t avg_terms) { return msm_pick_window((size_t)avg_terms); }
int emul_num_windows(int c) { return msm_num_windows(c); }
// branch selection of a pipeline pass (msm_make_plan / msm_launch)
uint64_t emul_avg_terms(uint64_t T, uint32_t n_msm) { return msm_avg_terms((size_t)T, n_msm); }
uint32_t emul_heavy_min(uint64_t avg_terms, uint32_t nb) { return msm_heavy_min((size_t)avg_terms, nb); }
int emul_acc_split(uint64_t avg_terms, uint32_t nb, uint64_t n_buckets) { return msm_acc_split((size_t)avg_terms, nb, (size_t)n_buckets); }
int emul_use_combine4(uint32_t n_msm) { return msm_use_combine4(n_msm) ? 1 : 0; }
// the verifier's reject path (rp_verify_fallback): proofs per chunk, and whether so many failing chunks re-check the whole batch
int emul_rp_chunk(void) { return RP_CHUNK; }
int emul_rp_recheck_whole_batch(uint32_t failing_chunks) { return rp_recheck_whole_batch(failing_chunks) ? 1 : 0; }
// proofs per slice of the R1CS and LinearProof reject paths (recheck_slices in bpmsm.cu)
uint32_t emul_recheck_slice(uint32_t np, uint32_t entries_per_proof, uint32_t budget) { return bp_recheck_slice(np, entries_per_proof, budget); }
// the verification-scalar head's split of the k index bits: the low group has rp_kl(k) bits (TL = 2^kl generator indices)
uint32_t emul_rp_kl(uint32_t k) { return rp_kl(k); }
// bucket sizes of one MSM as k_msm_count makes them: counts[w * 2^(c-1) + b] += 1 for every term whose window-w digit is +-(b+1).
// counts = W * 2^(c-1) entries, zeroed by the caller; returns 3 on a non-canonical scalar (such a term is skipped by the kernels)
int emul_bucket_counts(const uint8_t *scalars, uint32_t n, int c, uint32_t *counts) {
    int W = msm_num_windows(c); uint32_t nb = 1u << (c - 1);
    for (uint32_t i = 0; i < n; i++) {
        sc s = sc_load(scalars + 32 * i); if (sc_geq_l(s)) return 3;
        msm_wide r = msm_recode(s.v, c, W);
        for (int w = 0; w < W; w++) { int d = msm_digit(r, w, c); if (d != 0) counts[(size_t)w * nb + (uint32_t)(d < 0 ? -d : d) - 1u]++; }
    }
    return 0;
}

// Pippenger bookkeeping exactly as the kernels do it (offset recoding, bucket sums, chunked suffix reduction, Horner)
int emul_msm(const uint8_t *scalars, const uint8_t *points, uint32_t n, int c, uint32_t nthreads, uint8_t *out) {
    int W = msm_num_windows(c); uint32_t nb = 1u << (c - 1);
    std::vector<ge_niels> pts(n);
    for (uint32_t i = 0; i < n; i++) { fe x, y; if (!ge_decode(x, y, points + 32 * i)) return 1; pts[i] = ge_to_niels_affine(x, y); }
    std::vector<ge_ext> wsum(W);
    for (int w = 0; w < W; w++) {
        std::vector<ge_ext> B(nb, ge_identity());
        for (uint32_t i = 0; i < n; i++) {
            sc s = sc_load(scalars + 32 * i); if (sc_geq_l(s)) return 3;
            msm_wide r = msm_recode(s.v, c, W); int d = msm_digit(r, w, c);
            if (d > 0) B[d - 1] = ge_madd(B[d - 1], pts[i]); else if (d < 0) B[-d - 1] = ge_msub(B[-d - 1], pts[i]);
        }
        uint32_t L = (nb + nthreads - 1) / nthreads;
        std::vector<ge_ext> S(nthreads, ge_identity()), acc(nthreads, ge_identity());
        for (uint32_t t = 0; t < nthreads; t++) { uint32_t lo = std::min(t * L, nb), hi = std::min(lo + L, nb); for (uint32_t j = lo; j < hi; j++) S[t] = ge_add(S[t], B[j]); }
        ge_ext total = ge_identity();
        for (int t = (int)nthreads - 1; t >= 0; t--) {
            uint32_t lo = std::min((uint32_t)t * L, nb), hi = std::min(lo + L, nb);
            ge_ext run = total;                                  // exclusive suffix
            for (uint32_t j = hi; j > lo; j--) { run = ge_add(run, B[j - 1]); acc[t] = ge_add(acc[t], run); }
            total = ge_add(total, S[t]);
        }
        ge_ext r = ge_identity(); for (uint32_t t = 0; t < nthreads; t++) r = ge_add(r, acc[t]);
        wsum[w] = r;
    }
    ge_ext a = wsum[W - 1];
    for (int w = W - 2; w >= 0; w--) { for (int i = 0; i < c; i++) a = ge_dbl(a); a = ge_add(a, wsum[w]); }
    ge_encode(out, a);
    return 0;
}
}
