// Per-proof verification scalars of an aggregated range proof, computed on the device.
//
// Restates RangeProof::verify_multiple_with_rng up to (not including) the mega-MSM:
//   src/range_proof/mod.rs:368-419 (transcript replay, scalar assembly),
//   src/inner_product_proof.rs:198-253 (verification_scalars),
//   src/range_proof/mod.rs:587-593 (delta),
// with two changes that do not alter any verdict:
//  (1) every scalar of proof i is multiplied by a per-proof random weight, so that a batch of
//      proofs is checked with one random-linear-combination MSM (SURVEY.md §8a row A6);
//  (2) the weight is rho * lambda with lambda = (prod u_j)^2 * y^(N-1).  Multiplying the whole
//      mega-check by lambda cancels every inverse the reference computes (y^-i, u_j^-2, the
//      batch_invert product), so no field inversion is needed on the device:
//        lambda * u_j^-2          = y^(N-1) * prod_{j' != j} u_j'^2
//        lambda * s_i             = U * y^(N-1) * prod_{bits set in i} u^2      (U = prod u_j)
//        lambda * y^-i * s_{N-1-i} = U * y^(N-1-i) * prod_{bits clear in i} u^2
//      lambda != 0 with overwhelming probability and rho is uniform, so rho*lambda is a uniform weight.
//
// The work is split in a transcript replay (one thread per proof: Keccak chain), a short
// sequential head (one thread: ~8k+30 products) and a data-parallel tail (one generator index per
// thread).  All scalars are in Montgomery form between the byte boundaries.
#pragma once
#include "sc.cuh"
#include "merlin.cuh"

// verdict codes, mirroring ProofError (src/errors.rs:12-54)
#define BP_PROOF_OK 0
#define BP_PROOF_VERIFICATION_ERROR 1
#define BP_PROOF_FORMAT_ERROR 2

#define BP_MAX_LG_N 20          // N = n*m up to 2^20 generator pairs per proof

// Reject path of a batch whose combined check failed (bpmsm.cu, rp_verify_fallback): one combined MSM per chunk of RP_CHUNK proofs
// (k_rp_scalars_sum keeps per-chunk partial sums), then the proofs of the failing chunks one by one -- or, when more than four
// chunks fail, every proof of the batch.  The second level runs the same kernels with chunks of one proof, whose sums
// k_rp_scalars_sum computes first.  Shared with the host-emulation tests.
#define RP_CHUNK 32
BP_HD bool rp_recheck_whole_batch(uint32_t failing_chunks) { return failing_chunks > 4; }

// out-of-line Montgomery product: one copy of the three-pass multiplier per kernel
BP_HDN sc sc_mm(const sc &a, const sc &b) { return sc_mont_mul(a, b); }

struct rp_challenges {          // Montgomery form
    sc y, z, x, w, c, rho;
    sc u[BP_MAX_LG_N];
    uint32_t status;
};

BP_HD bool bp_is_zero32(const uint8_t *p) { uint8_t z = 0; for (int i = 0; i < 32; i++) z |= p[i]; return z == 0; }
BP_HD sc rp_wide(const uint8_t buf[64]) { sc lo = sc_load(buf), hi = sc_load(buf + 32); return sc_add(sc_mm(lo, sc{SC_RR_LIMBS}), sc_mm(hi, sc{SC_RRR_LIMBS})); }
BP_HD sc rp_challenge(merlin_t &t, const char *label) { uint8_t buf[64]; merlin_challenge(t, label, buf, 64); return rp_wide(buf); }

// Transcript replay of one proof: pure hashing.  proof = 32*(9+2k) bytes, V = m*32 bytes, tstate = the serialized
// transcript the caller passed in, state200 = 200 bytes of 4-byte-aligned scratch for the STROBE state.
// Output: the 64-byte challenge outputs in the order y, z, x, w, c, rho (the batching weights), u_0..u_{k-1}
// -> raw[RP_RAW_U + j]; nothing the verifier hashes depends on a challenge, so the reduction mod l is left to the caller.
#define RP_RAW_Y 0
#define RP_RAW_Z 1
#define RP_RAW_X 2
#define RP_RAW_W 3
#define RP_RAW_C 4
#define RP_RAW_RHO 5
#define RP_RAW_U 6
BP_HD void rp_raw_challenge(merlin_t &t, const char *label, uint8_t *out64) { merlin_challenge(t, label, out64, 64); }
BP_HDN uint32_t rp_transcript_raw(uint8_t (*raw)[64], const uint8_t *proof, uint32_t k, const uint8_t *V, uint32_t n, uint32_t m,
                                  const uint8_t *tstate, const uint8_t *seed, uint8_t *state200) {
    const uint8_t *A = proof, *S = proof + 32, *T1 = proof + 64, *T2 = proof + 96;
    const uint8_t *LR = proof + 224, *ab = proof + 224 + 64 * k;
    // RangeProof::from_bytes / InnerProductProof::from_bytes canonicity (mod.rs:519-524, inner_product_proof.rs:399-404)
    if (sc_geq_l(sc_load(proof + 128)) || sc_geq_l(sc_load(proof + 160)) || sc_geq_l(sc_load(proof + 192)) || sc_geq_l(sc_load(ab)) || sc_geq_l(sc_load(ab + 32)))
        return BP_PROOF_FORMAT_ERROR;
    merlin_t t; t.st = state200; merlin_load(t, tstate);
    merlin_append(t, "dom-sep", (const uint8_t *)"rangeproof v1", 13);            // transcript.rs:44-48
    merlin_append_u64(t, "n", n); merlin_append_u64(t, "m", m);
    for (uint32_t j = 0; j < m; j++) merlin_append(t, "V", V + 32 * j, 32);         // mod.rs:370-374 (identity allowed)
    bool bad = bp_is_zero32(A) || bp_is_zero32(S);                                  // validate_and_append_point
    merlin_append(t, "A", A, 32); merlin_append(t, "S", S, 32);
    rp_raw_challenge(t, "y", raw[RP_RAW_Y]); rp_raw_challenge(t, "z", raw[RP_RAW_Z]);
    bad = bad || bp_is_zero32(T1) || bp_is_zero32(T2);
    merlin_append(t, "T_1", T1, 32); merlin_append(t, "T_2", T2, 32);
    rp_raw_challenge(t, "x", raw[RP_RAW_X]);
    merlin_append(t, "t_x", proof + 128, 32); merlin_append(t, "t_x_blinding", proof + 160, 32); merlin_append(t, "e_blinding", proof + 192, 32);
    rp_raw_challenge(t, "w", raw[RP_RAW_W]);
    merlin_append(t, "dom-sep", (const uint8_t *)"ipp v1", 6);                      // transcript.rs:50-53
    merlin_append_u64(t, "n", (uint64_t)n * m);
    for (uint32_t j = 0; j < k; j++) {                                              // inner_product_proof.rs:218-222
        bad = bad || bp_is_zero32(LR + 64 * j) || bp_is_zero32(LR + 64 * j + 32);
        merlin_append(t, "L", LR + 64 * j, 32); merlin_append(t, "R", LR + 64 * j + 32, 32);
        rp_raw_challenge(t, "u", raw[RP_RAW_U + j]);
    }
    // Batching weights c (mod.rs:396) and rho (row A6): bound to everything the proof's transcript has absorbed, the way
    // merlin's TranscriptRng binds a prover's randomness -- build_rng() (fork of the state), finalize(rng) = meta_ad("rng") +
    // KEY(32 bytes of the external RNG: the batch seed), fill_bytes(128) = meta_ad(LE32(128)) + PRF.  A caller that passes a
    // fixed or known seed therefore still gives a prover no knowledge of the weights before the proof bytes are fixed.
    strobe_begin_op(t, 16 | 2); strobe_absorb(t, (const uint8_t *)"rng", 3);
    strobe_begin_op(t, 2 | 4); strobe_overwrite(t, seed, 32);
    const uint8_t l128[4] = {128, 0, 0, 0};
    strobe_begin_op(t, 16 | 2); strobe_absorb(t, l128, 4);
    strobe_begin_op(t, 1 | 2 | 4); strobe_squeeze(t, raw[RP_RAW_C], 128);           // rows C and RHO are adjacent
    return bad ? BP_PROOF_VERIFICATION_ERROR : BP_PROOF_OK;
}
// Sequential form (host emulation, reference for the cooperative device head): replay + reduction of the challenges.
// seed = the batch's 32 bytes of external randomness (c and rho are derived from it and the proof's transcript).
BP_HDN void rp_transcript(rp_challenges &ch, const uint8_t *proof, uint32_t k, const uint8_t *V, uint32_t n, uint32_t m,
                         const uint8_t *tstate, const uint8_t *seed, uint8_t *state200) {
    uint8_t raw[RP_RAW_U + BP_MAX_LG_N][64];
    ch.status = rp_transcript_raw(raw, proof, k, V, n, m, tstate, seed, state200);
    if (ch.status != BP_PROOF_OK) return;
    ch.y = rp_wide(raw[RP_RAW_Y]); ch.z = rp_wide(raw[RP_RAW_Z]); ch.x = rp_wide(raw[RP_RAW_X]); ch.w = rp_wide(raw[RP_RAW_W]);
    for (uint32_t j = 0; j < k; j++) ch.u[j] = rp_wide(raw[RP_RAW_U + j]);
    // The device multiplies the proof's check by lambda = (prod u_j)^2 y^(N-1) (see the header).  A zero challenge would make
    // lambda vanish and the proof drop out of the combination, so it is rejected outright; the reference cannot verify such a
    // transcript either (u_j = 0 has no inverse), and an honest or dishonest prover hits it with probability ~2^-252 per hash.
    bool bad = sc_is_zero(ch.y);
    for (uint32_t j = 0; j < k; j++) bad = bad || sc_is_zero(ch.u[j]);
    if (bad) { ch.status = BP_PROOF_VERIFICATION_ERROR; return; }
    ch.c = rp_wide(raw[RP_RAW_C]); ch.rho = rp_wide(raw[RP_RAW_RHO]);
    if (sc_is_zero(ch.rho)) ch.rho = sc_mont_one();                  // a zero weight (probability 2^-252) would skip the proof
}

struct rp_head {                // Montgomery form; "L" = Lambda = rho * lambda
    uint32_t status, pad_[7];
    sc z, zz, L, zL, Lx, Lcx, Lcxx, Lczz, gA, hB, rhoY;
    sc u_sq[BP_MAX_LG_N], pre[BP_MAX_LG_N + 1], suf[BP_MAX_LG_N + 1];
    sc basepoint_scalar, blinding_scalar;
};

// Per-proof product tables (global memory, rp_tab_size() scalars per proof) that turn the tail into three products
// per generator index.  The k index bits are split in a low group of kl = ceil(k/2) bits (TL = 2^kl values) and a
// high group of kh = k - kl bits (TH = 2^kh values), i = hi*TL + lo, and ~v is the complement within the group:
//   s_lo[v] = prod_{b < kl, bit b of v} u_sq[k-1-b]           s_hi[v] = prod_{b < kh, bit b of v} u_sq[k-1-kl-b]
//   y_lo[v] = y^v                                               y_hi[v] = y^(v*TL)
//   A_hi[v] = gA * s_hi[v]
//   P_lo[v] = y_lo[~v] * F_lo(v)                                P_hi[v] = hA * y_hi[~v] * F_hi(v)
//   Q_lo[v] = y_lo[~v] * s_lo[~v]                               Q_hi[v] = hB * y_hi[~v] * s_hi[~v]
// with F(i) = 2^(i mod n) z^(i div n) = F_hi(hi) F_lo(lo) (n and TL are powers of two), so that
//   lambda-weighted  g_i = -zL - A_hi[hi] s_lo[lo],     h_i = zL + P_hi[hi] P_lo[lo] - Q_hi[hi] Q_lo[lo].
BP_HD uint32_t rp_kl(uint32_t k) { return (k + 1) / 2; }
BP_HD uint32_t rp_tab_size(uint32_t k, uint32_t m) { (void)m; uint32_t kl = rp_kl(k); return 4 * (1u << kl) + 5 * (1u << (k - kl)); }
struct rp_tabs { sc *s_lo, *A_hi, *P_lo, *P_hi, *Q_lo, *Q_hi, *s_hi, *y_lo, *y_hi; };
BP_HD rp_tabs rp_tab_ptrs(sc *tab, uint32_t k) {
    uint32_t kl = rp_kl(k), TL = 1u << kl, TH = 1u << (k - kl);
    rp_tabs t; t.s_lo = tab; t.A_hi = t.s_lo + TL; t.P_lo = t.A_hi + TH; t.P_hi = t.P_lo + TL; t.Q_lo = t.P_hi + TH; t.Q_hi = t.Q_lo + TL;
    t.s_hi = t.Q_hi + TH; t.y_lo = t.s_hi + TH; t.y_hi = t.y_lo + TL;
    return t;
}

BP_HD sc rp_pow_small(const sc &base0, uint32_t e) {                // base^e by square-and-multiply
    sc r = sc_mont_one(), base = base0;
    for (; e; e >>= 1) { if (e & 1u) r = sc_mm(r, base); if (e > 1) base = sc_mm(base, base); }
    return r;
}

// sum_{i<n} x^i for n a power of two (util.rs:240-256), Montgomery form
BP_HD sc rp_sum_of_powers_pow2(const sc &x, uint64_t n) {
    if (n == 1) return sc_mont_one();
    sc result = sc_add(sc_mont_one(), x), factor = x;
    for (uint64_t m = n; m > 2; m >>= 1) { factor = sc_mm(factor, factor); result = sc_add(result, sc_mm(factor, result)); }
    return result;
}

// table[v] for v in [0, 2^bits): product of f[b] over the set bits b of v; f(b) supplied by the caller
#define RP_BUILD_TABLE(tab, bits, FACTOR)                                                    \
    do {                                                                                     \
        (tab)[0] = sc_mont_one();                                                            \
        for (uint32_t b_ = 0; b_ < (bits); b_++) {                                           \
            const sc f_ = (FACTOR);                                                          \
            (tab)[1u << b_] = f_;                                                            \
            for (uint32_t v_ = 1; v_ < (1u << b_); v_++) (tab)[(1u << b_) + v_] = sc_mm((tab)[v_], f_); \
        }                                                                                    \
    } while (0)

// Sequential head: shared products and tables of one proof
BP_HDN void rp_scalars_head(rp_head &h, sc *tab, const sc *pow2, const rp_challenges &ch, const uint8_t *proof, uint32_t k, uint32_t n, uint32_t m) {
    const uint8_t *ab = proof + 224 + 64 * k;
    sc a = sc_to_mont(sc_load(ab)), b = sc_to_mont(sc_load(ab + 32));
    sc t_x = sc_to_mont(sc_load(proof + 128)), t_x_bl = sc_to_mont(sc_load(proof + 160)), e_bl = sc_to_mont(sc_load(proof + 192));
    h.z = ch.z; h.zz = sc_mm(ch.z, ch.z);
    uint32_t kl = rp_kl(k), kh = k - kl, TL = 1u << kl, TH = 1u << kh;
    rp_tabs T = rp_tab_ptrs(tab, k);
    sc U = sc_mont_one(), Y = sc_mont_one(), ypow2[BP_MAX_LG_N];
    h.pre[0] = sc_mont_one();
    for (uint32_t j = 0; j < k; j++) {
        h.u_sq[j] = sc_mm(ch.u[j], ch.u[j]); U = sc_mm(U, ch.u[j]);
        h.pre[j + 1] = sc_mm(h.pre[j], h.u_sq[j]);                  // prod_{j' <= j} u^2;  pre[k] = U^2
        ypow2[j] = j == 0 ? ch.y : sc_mm(ypow2[j - 1], ypow2[j - 1]);        // y^(2^j)
        Y = sc_mm(Y, ypow2[j]);                                     // ends as y^(N-1)
    }
    h.suf[k] = sc_mont_one();
    for (int j = (int)k - 1; j >= 0; j--) h.suf[j] = sc_mm(h.suf[j + 1], h.u_sq[j]);   // prod_{j' >= j} u^2
    // bit b of the index i <-> challenge k-1-b (inner_product_proof.rs:241-250)
    RP_BUILD_TABLE(T.s_lo, kl, h.u_sq[(k - 1) - b_]);
    RP_BUILD_TABLE(T.s_hi, kh, h.u_sq[(k - 1) - kl - b_]);
    RP_BUILD_TABLE(T.y_lo, kl, ypow2[b_]);
    RP_BUILD_TABLE(T.y_hi, kh, ypow2[kl + b_]);
    sc lambda = sc_mm(h.pre[k], Y);
    h.L = sc_mm(ch.rho, lambda); h.zL = sc_mm(ch.z, h.L);
    h.Lx = sc_mm(h.L, ch.x); h.Lcx = sc_mm(h.Lx, ch.c); h.Lcxx = sc_mm(h.Lcx, ch.x); h.Lczz = sc_mm(sc_mm(h.L, ch.c), h.zz);
    sc rhoU = sc_mm(ch.rho, U);
    h.gA = sc_mm(sc_mm(a, rhoU), Y);                                // a rho U y^(N-1)
    h.hB = sc_mm(b, rhoU);                                          // b rho U
    sc hA = sc_mm(sc_mm(rhoU, U), h.zz);                            // rho U^2 z^2
    // F(i) = 2^(i mod n) z^(i div n) split over the two index groups
    for (uint32_t v = 0; v < TL; v++) {
        sc F = sc_mm(pow2[v % n], rp_pow_small(ch.z, v / n));       // v < TL: (v mod n, v div n)
        T.P_lo[v] = sc_mm(T.y_lo[v ^ (TL - 1)], F);
        T.Q_lo[v] = sc_mm(T.y_lo[v ^ (TL - 1)], T.s_lo[v ^ (TL - 1)]);
    }
    for (uint32_t v = 0; v < TH; v++) {
        uint64_t idx = (uint64_t)v << kl;                           // i = v*TL: (i mod n, i div n)
        sc F = sc_mm(pow2[idx % n], rp_pow_small(ch.z, (uint32_t)(idx / n)));
        sc yc = T.y_hi[v ^ (TH - 1)];
        T.A_hi[v] = sc_mm(h.gA, T.s_hi[v]);
        T.P_hi[v] = sc_mm(sc_mm(hA, yc), F);
        T.Q_hi[v] = sc_mm(sc_mm(h.hB, yc), T.s_hi[v ^ (TH - 1)]);
    }
    h.rhoY = sc_mm(ch.rho, Y);
    // delta(y,z) = (z - z^2) sum y^i - z^3 (2^n - 1) sum z^j          (mod.rs:587-593)
    sc sum_y = rp_sum_of_powers_pow2(ch.y, (uint64_t)n * m), sum_z = rp_sum_of_powers_pow2(ch.z, m);
    sc sum_2 = sc_mont_from_u64(n == 64 ? ~0ULL : ((1ULL << n) - 1));
    sc delta = sc_sub(sc_mm(sc_sub(ch.z, h.zz), sum_y), sc_mm(sc_mm(sc_mm(h.zz, ch.z), sum_2), sum_z));
    // basepoint scalar w (t_x - a b) + c (delta - t_x)  (mod.rs:419);  blinding scalar -e~ - c t~  (mod.rs:430)
    sc bs = sc_add(sc_mm(ch.w, sc_sub(t_x, sc_mm(a, b))), sc_mm(ch.c, sc_sub(delta, t_x)));
    sc bl = sc_neg(sc_add(e_bl, sc_mm(ch.c, t_x_bl)));
    h.basepoint_scalar = sc_mm(h.L, bs); h.blinding_scalar = sc_mm(h.L, bl);
}

// Data-parallel tail: weighted g_i and h_i for generator pair i in [0, N) (mod.rs:415-417), Montgomery form.
// Three products per index (see the table definitions above).  The device sums these products over a chunk's proofs in
// k_rp_scalars_sum (kernels.cuh) and never calls this per-proof form; it is the reference the host-emulation tests check
// the scalar assembly with.
BP_HD void rp_scalars_gh(const rp_head &h, const sc *tab, uint32_t i, uint32_t k, sc &g, sc &hh) {
    uint32_t kl = rp_kl(k), TL = 1u << kl;
    rp_tabs T = rp_tab_ptrs(const_cast<sc *>(tab), k);
    uint32_t lo = i & (TL - 1), hi = i >> kl;
    g = sc_sub(sc_neg(h.zL), sc_mm(T.A_hi[hi], T.s_lo[lo]));
    hh = sc_sub(sc_add(h.zL, sc_mm(T.P_hi[hi], T.P_lo[lo])), sc_mm(T.Q_hi[hi], T.Q_lo[lo]));
}

// Per-proof ("dynamic") scalars in MSM order A, S, T_1, T_2, L_0..L_{k-1}, R_0..R_{k-1}, V_0..V_{m-1}
// (mod.rs:422-444 without the static B~, B, G, H block); idx in [0, 4+2k+m); Montgomery form
BP_HD sc rp_scalars_dynamic(const rp_head &h, uint32_t idx, uint32_t k) {
    if (idx == 0) return h.L;
    if (idx == 1) return h.Lx;
    if (idx == 2) return h.Lcx;
    if (idx == 3) return h.Lcxx;
    if (idx < 4 + k) return sc_mm(h.L, h.u_sq[idx - 4]);
    if (idx < 4 + 2 * k) { uint32_t j = idx - 4 - k; return sc_mm(h.rhoY, sc_mm(h.pre[j], h.suf[j + 1])); }
    return sc_mm(h.Lczz, rp_pow_small(h.z, idx - 4 - 2 * k));
}
