// Verification scalars of a batch of LinearProofs over one resident point set [B, F, G_0 .. G_{n-1}] (bp_linear_verify_batch),
// computed on the device.
//
// LinearProof::verify (src/linear_proof.rs:184-237) accepts when
//     S == r B + a b0 F - x* (C + sum_k x_k L_k + sum_k x_k^-1 R_k) + a sum_i s_i G_i,
// x_k the round challenges, x* the final one, s_i = prod_{bit b of i set} x_{lg n - 1 - b} (linear_proof.rs:272-284) and b0 the
// fold of the public vector b, which equals <b, s>.  Moved to one side and weighted by a per-proof random rho (from the proof's
// transcript, its a and r, and the batch seed: lin_transcript_raw), a batch is checked with one MSM that must vanish:
//     B: sum rho r     F: sum rho a b0     G_i: sum rho a s_i     C_j: -rho x*     L_{j,k}: -rho x* x_k     R_{j,k}: -rho x* x_k^-1     S_j: -rho
// The reject path runs the same code with rho = 1 and one proof per sum: each proof's own equation.
//
// The inverses x_k^-1 come from one Montgomery-trick inversion per proof.  A zero challenge has no inverse: such a proof is rejected
// outright with VerificationError, as rp.cuh rejects a zero u_j.  An honest or dishonest prover hits it with probability ~2^-252 per
// hash.
//
// The lg n index bits are split as in the range-proof head (rp.cuh): a low group of kl = rp_kl(k) bits (TL = 2^kl values) and a high
// group of kh = k - kl bits, i = hi*TL + lo, and each proof keeps the tables
//     slo[v] = prod_{b < kl, bit b of v} x_{k-1-b}        shi[v] = prod_{b < kh, bit b of v} x_{k-1-kl-b}
// so that s_i = shi[hi] slo[lo] costs one product.  Head, tables and the G sums are in Montgomery form; b, b0 and the B / F scalars
// are plain.  Shared with the host-emulation tests (tests/host_emul/emul_linear.cpp).
#pragma once
#include "rp.cuh"

// proofs per block of the combined G sum: their products are summed as 512-bit integers and reduced once (sc_wide, <= 32 products)
#define LIN_CHUNK 32
// per-proof points in MSM order: C, S, L_0 .. L_{k-1}, R_0 .. R_{k-1}
BP_HD uint32_t lin_dyn_terms(uint32_t k) { return 2 + 2 * k; }
// raw 64-byte challenge rows per proof: x_0 .. x_{k-1}, x*, rho
BP_HD uint32_t lin_raw_rows(uint32_t k) { return k + 2; }

// The reject path re-checks proofs in slices whose rows [B, F, G_0..G_{n-1} | C, S, L.., R..] of `row` terms each hold at most 2^20 terms
BP_HD uint32_t lin_recheck_slice(uint32_t np, uint32_t row) { return bp_recheck_slice(np, row, 1u << 20); }

// Reject path of a reserved device call (bp_linear_verify_device), one slice of P = lin_x_slice proofs per iteration of a WHILE node.
// The live count comes from the call's staged parameters and is clamped to the capacity, so a slice never indexes past the arenas; the
// loop runs lin_x_iters times (0 when the combined check passed), at most ceil(capacity / P), and each iteration adds one to its counter,
// so it ends by construction.
BP_HD uint32_t lin_x_slice(uint32_t capacity, uint32_t n, uint32_t k) { return lin_recheck_slice(capacity, n + 2 + lin_dyn_terms(k)); }
BP_HD uint32_t lin_x_clamp(uint32_t live, uint32_t capacity) { return live < capacity ? live : capacity; }
BP_HD uint32_t lin_x_iters(uint32_t live, uint32_t P, bool failed) { return failed ? live / P + (live % P ? 1u : 0u) : 0u; }
// proofs of iteration it that are live: [it P, min(it P + P, live))
BP_HD uint32_t lin_x_slice_live(uint32_t it, uint32_t P, uint32_t live) { const uint32_t p0 = it * P; return p0 >= live ? 0u : live - p0 < P ? live - p0 : P; }

BP_HD bool lin_b_canonical(const uint8_t *b, uint32_t n) {
    for (uint32_t i = 0; i < n; i++) if (sc_geq_l(sc_load(b + 32 * i))) return false;
    return true;
}

// Transcript replay of one proof: pure hashing.  proof = L_0 R_0 .. L_{k-1} R_{k-1} S a r (32*(2k+3) bytes, linear_proof.rs:322-334),
// b = its n public scalars, enc = the set's encodings [B, F, G_0 .. G_{n-1}], tstate = the proof's serialized transcript, state200 =
// 200 bytes of 4-byte-aligned scratch.  Output: the challenge rows x_0 .. x_{k-1}, x*, rho (raw[k + 1], the batching weight).  rho
// comes from a fork of the final state rekeyed with a || r (merlin_rng_rekey), then finalized with the seed: the check is linear in a
// and r, so a weight that did not depend on them would let two proofs with r + d and r - d cancel in the combination.
// A record that no Merlin transcript can hold between operations (pos at or beyond the STROBE rate, or pos_begin above pos) gives
// FormatError before anything is absorbed: with pos past the rate the absorb would never reach the permutation and would write beyond
// the 200-byte state.
#define LIN_WITNESS_LABEL "linear_a_r"
BP_HDN uint32_t lin_transcript_raw(uint8_t (*raw)[64], const uint8_t *proof, uint32_t k, uint32_t n, const uint8_t *C, const uint8_t *b,
                                   const uint8_t *enc, const uint8_t *tstate, const uint8_t *seed, uint8_t *state200) {
    const uint8_t *S = proof + 64 * k;
    if (sc_geq_l(sc_load(S + 32)) || sc_geq_l(sc_load(S + 64))) return BP_PROOF_FORMAT_ERROR;       // LinearProof::from_bytes
    if (tstate[200] >= BP_STROBE_R || tstate[201] > tstate[200]) return BP_PROOF_FORMAT_ERROR;
    merlin_t t; t.st = state200; merlin_load(t, tstate);
    merlin_append(t, "dom-sep", (const uint8_t *)"ipp v1", 6); merlin_append_u64(t, "n", n);           // innerproduct_domain_sep
    merlin_append(t, "C", C, 32);
    for (uint32_t i = 0; i < n; i++) merlin_append(t, "b_i", b + 32 * i, 32);
    for (uint32_t i = 0; i < n; i++) merlin_append(t, "G_i", enc + 64 + 32 * i, 32);
    merlin_append(t, "F", enc + 32, 32); merlin_append(t, "B", enc, 32);
    for (uint32_t j = 0; j < k; j++) {
        const uint8_t *L = proof + 64 * j, *R = L + 32;
        if (bp_is_zero32(L) || bp_is_zero32(R)) return BP_PROOF_VERIFICATION_ERROR;                 // validate_and_append_point
        merlin_append(t, "L", L, 32); merlin_append(t, "R", R, 32);
        merlin_challenge(t, "x_j", raw[j], 64);
    }
    merlin_append(t, "S", S, 32);
    merlin_challenge(t, "x_star", raw[k], 64);
    merlin_rng_rekey(t, LIN_WITNESS_LABEL, S + 32, 64);                                             // a || r: never absorbed
    merlin_rng_bytes(t, seed, raw[k + 1], 64);
    return BP_PROOF_OK;
}

struct lin_head {               // Montgomery form
    uint32_t status, pad_[7];
    sc rho, wa, xs;             // the weight (rho, or 1 on the reject path), rho a, x*
    sc x[BP_MAX_LG_N], xinv[BP_MAX_LG_N];
};

// head of one proof from its reduced round challenges x[0..k) and its raw x* and rho rows; weighted = the combined check.  Returns
// the proof's status (VerificationError for a zero challenge).
BP_HDN uint32_t lin_head_init(lin_head &h, const sc *x, uint32_t k, const uint8_t *raw_xs, const uint8_t *raw_rho, const uint8_t *proof, bool weighted) {
    bool bad = false;
    sc acc = sc_mont_one();
    for (uint32_t j = 0; j < k; j++) { bad = bad || sc_is_zero(x[j]); h.x[j] = x[j]; h.xinv[j] = acc; acc = sc_mm(acc, x[j]); }   // xinv: prefix products
    if (bad) { h.status = BP_PROOF_VERIFICATION_ERROR; return h.status; }
    sc inv = sc_mont_invert(acc);                                     // (prod x)^-1
    for (int j = (int)k - 1; j >= 0; j--) { h.xinv[j] = sc_mm(inv, h.xinv[j]); inv = sc_mm(inv, x[j]); }
    h.xs = rp_wide(raw_xs);
    sc rho = weighted ? rp_wide(raw_rho) : sc_mont_one();
    if (sc_is_zero(rho)) rho = sc_mont_one();                         // a zero weight (probability 2^-252) would skip the proof
    h.rho = rho;
    h.wa = sc_mm(rho, sc_to_mont(sc_load(proof + 64 * k + 32)));
    h.status = BP_PROOF_OK;
    return h.status;
}

BP_HD uint32_t lin_tab_size(uint32_t k) { const uint32_t kl = rp_kl(k); return (1u << kl) + (1u << (k - kl)); }
// table entry e of one proof (slo at e < TL, shi after it), computed on its own so that a block fills a proof's tables in parallel
BP_HD sc lin_tab_entry(const sc *x, uint32_t k, uint32_t e) {
    const uint32_t kl = rp_kl(k), TL = 1u << kl, hi = e >= TL ? 1u : 0u;
    const uint32_t v = hi ? e - TL : e, b0 = hi ? kl : 0u, bits = hi ? k - kl : kl;
    sc r = sc_mont_one();
    for (uint32_t b = 0; b < bits; b++) if ((v >> b) & 1u) r = sc_mm(r, x[k - 1 - b0 - b]);
    return r;
}
// proof's share of generator index i: acc += rho a s_i (the G sum); returns b_i s_i (plain, b_i plain)
BP_HD sc lin_acc_add(sc_wide &acc, const sc &wa, const sc *tab, uint32_t k, const sc &b_i, uint32_t i) {
    const uint32_t kl = rp_kl(k), TL = 1u << kl;
    const sc s = sc_mont_mul(tab[TL + (i >> kl)], tab[i & (TL - 1)]);       // inline: the G sum's inner loop
    sc_wide_mac(acc, wa, s);
    return sc_mont_mul(b_i, s);
}
// B and F scalars of one proof (plain): rho r and rho a b0, with b0 = <b, s> plain
BP_HD void lin_static_bf(const lin_head &h, const uint8_t *proof, uint32_t k, const sc &b0, sc &sB, sc &sF) {
    sB = sc_mm(h.rho, sc_load(proof + 64 * k + 64));
    sF = sc_mm(h.wa, b0);
}
// per-proof ("dynamic") scalar d in the order C, S, L_0.., R_0.. (plain)
BP_HD sc lin_dyn_scalar(const lin_head &h, uint32_t d, uint32_t k) {
    const sc rx = sc_mm(h.rho, h.xs);
    const sc v = d == 0 ? rx : d == 1 ? h.rho : d < 2 + k ? sc_mm(rx, h.x[d - 2]) : sc_mm(rx, h.xinv[d - 2 - k]);
    return sc_from_mont(sc_neg(v));
}
