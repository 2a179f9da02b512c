// Generator scalars of a batch of R1CS proofs (bp_r1cs_verify_batch), computed on the device.
//
// The mega-check of r1cs::Verifier::verify (src/r1cs/verifier.rs:398-497) weights generator pair i of a proof with
//     g_i = u1 (x y^-i wR_i - a s_i),      h_i = u1 (y^-i (x wL_i + wO_i - b s_{N-1-i}) - 1),
// u1 = 1 for i < n1 and u otherwise (the padding indices n <= i < N included), N = padded_n = 2^k, and s the vector of
// inner_product_proof.rs:227-251: s_i = s_0 prod_{bit b of i set} u_sq[k-1-b].  The host runs each proof's transcript, flattens
// its constraints and hands over x, y^-1, u, a, b, the batching weight rho, s_0 and u_sq (R1CS_CHAL_* below) with wL, wR, wO.
//
// The k index bits are split as in the range-proof head (rp.cuh): a low group of kl = rp_kl(k) bits (TL = 2^kl values) and a high
// group of kh = k - kl bits (TH = 2^kh values), i = hi*TL + lo, ~v = the complement within the group.  With W the proof's weight of
// index i (W = rho u1 in the combined check, u1 on the reject path), one table entry per group value turns every factor that depends
// on i alone into one product:
//   lo tables:  ylo[v] = y^-v                      slo[v] = prod_{b < kl, bit b of v} u_sq[k-1-b]      qlo[v] = y^-v slo[~v]
//   hi tables (one set for W = w_lo, i < n1, and one for W = w_hi, i >= n1):
//               Yhi[v] = W y^-(v TL)               AShi[v] = W a s_0 shi[v]                            Qhi[v] = W b s_0 y^-(v TL) shi[~v]
// with shi[v] = prod_{b < kh, bit b of v} u_sq[k-1-kl-b], so that
//   W g_i = Y x wR_i - AShi[hi] slo[lo],     W h_i = Y (x wL_i + wO_i) - Qhi[hi] qlo[lo] - W,     Y = Yhi[hi] ylo[lo] = W y^-i.
// The hi tables and ylo are in Montgomery form, slo and qlo and the wL/wR/wO inputs are plain, so every product of a Montgomery and a
// plain value is a plain value: the summed g_i and h_i come out as plain scalars, ready for the MSM.
//
// Shared with the host-emulation tests (tests/host_emul), which check the chunk sums against Python integers.
#pragma once
#include "rp.cuh"

// scalars of a proof's challenge block (ABI order), 32 bytes each, then u_sq[0..k)
#define R1CS_CHAL_X 0
#define R1CS_CHAL_YINV 1
#define R1CS_CHAL_U 2
#define R1CS_CHAL_A 3
#define R1CS_CHAL_B 4
#define R1CS_CHAL_RHO 5
#define R1CS_CHAL_S0 6
#define R1CS_CHAL_USQ 7

// proofs per block of the combined G/H sum: their products are summed as 512-bit integers and reduced once (sc_wide, <= 32 products)
#define R1CS_CHUNK 32

// The reject path holds the G/H sums of at most 2^22 generator indices at once (2*Nmax per re-checked proof): proofs per slice of np
// proofs whose largest padded_n is Nmax, by the shared slice rule
BP_HD uint32_t r1cs_recheck_slice(uint32_t np, uint32_t Nmax) { return bp_recheck_slice(np, 2 * Nmax, 1u << 22); }

// one proof of a batch: its dimensions and where its data start in the flat per-batch arrays
struct r1cs_proof {
    uint32_t padded_n, n1, n, k;
    uint32_t chal_off;       // first scalar of its challenge block (R1CS_CHAL_USQ + k scalars)
    uint32_t w_off;          // first of its n wL / wR / wO scalars
    uint32_t tab_off;        // first entry of its tables (r1cs_tab_size(k) scalars)
    uint32_t term_off;       // first of its other terms
};
// per-proof values the G/H sum reads besides the tables (written by the table builder)
struct r1cs_head {
    sc x;                    // Montgomery form
    sc w_lo, w_hi;           // plain: the weight W of indices i < n1 and i >= n1
};

BP_HD uint32_t r1cs_tab_size(uint32_t k) { uint32_t kl = rp_kl(k); return 3 * (1u << kl) + 6 * (1u << (k - kl)); }
struct r1cs_tabs { sc *ylo, *slo, *qlo; sc *Yhi[2], *AShi[2], *Qhi[2]; };
BP_HD r1cs_tabs r1cs_tab_ptrs(sc *tab, uint32_t k) {
    const uint32_t TL = 1u << rp_kl(k), TH = 1u << (k - rp_kl(k));
    r1cs_tabs t; t.ylo = tab; t.slo = tab + TL; t.qlo = tab + 2 * TL;
    for (int s = 0; s < 2; s++) { sc *b = tab + 3 * TL + 3 * s * TH; t.Yhi[s] = b; t.AShi[s] = b + TH; t.Qhi[s] = b + 2 * TH; }
    return t;
}

BP_HDN sc r1cs_chal(const uint8_t *chal, uint32_t j) { return sc_mm(sc_load(chal + 32 * j), sc{SC_RR_LIMBS}); }     // Montgomery form
// prod of u_sq[k-1-b0-b] over the set bits b of v (b < bits), Montgomery form
BP_HD sc r1cs_s_part(const uint8_t *chal, uint32_t k, uint32_t b0, uint32_t bits, uint32_t v) {
    sc r = sc_mont_one();
    for (uint32_t b = 0; b < bits; b++) if ((v >> b) & 1u) r = sc_mm(r, r1cs_chal(chal, R1CS_CHAL_USQ + (k - 1 - b0 - b)));
    return r;
}
// the proof's weights: weighted = the combined check (rho u1), otherwise the reject path's own mega-check (u1)
BP_HD void r1cs_weights(const uint8_t *chal, bool weighted, sc &w_lo, sc &w_hi) {
    const sc u = r1cs_chal(chal, R1CS_CHAL_U);
    w_lo = weighted ? r1cs_chal(chal, R1CS_CHAL_RHO) : sc_mont_one();
    w_hi = sc_mm(w_lo, u);
}
BP_HD void r1cs_head_init(r1cs_head &h, const uint8_t *chal, bool weighted) {
    sc w_lo, w_hi; r1cs_weights(chal, weighted, w_lo, w_hi);
    h.x = r1cs_chal(chal, R1CS_CHAL_X); h.w_lo = sc_from_mont(w_lo); h.w_hi = sc_from_mont(w_hi);
}
// table entry e (0 <= e < r1cs_tab_size(k)) of one proof, computed on its own so that a block fills a proof's tables in parallel
BP_HD void r1cs_tab_entry(sc *tab, const uint8_t *chal, uint32_t k, bool weighted, uint32_t e) {
    const uint32_t kl = rp_kl(k), kh = k - kl, TL = 1u << kl, TH = 1u << kh;
    if (e < 3 * TL) {
        const uint32_t which = e / TL, v = e % TL;
        sc r;
        if (which == 0) r = rp_pow_small(r1cs_chal(chal, R1CS_CHAL_YINV), v);                                                          // ylo, Montgomery
        else if (which == 1) r = sc_from_mont(r1cs_s_part(chal, k, 0, kl, v));                                                         // slo, plain
        else r = sc_from_mont(sc_mm(rp_pow_small(r1cs_chal(chal, R1CS_CHAL_YINV), v), r1cs_s_part(chal, k, 0, kl, v ^ (TL - 1))));     // qlo, plain
        tab[e] = r;
        return;
    }
    const uint32_t r0 = e - 3 * TL, set = r0 / (3 * TH), which = (r0 % (3 * TH)) / TH, v = r0 % TH;
    sc W = weighted ? r1cs_chal(chal, R1CS_CHAL_RHO) : sc_mont_one();
    if (set) W = sc_mm(W, r1cs_chal(chal, R1CS_CHAL_U));
    if (which != 1) W = sc_mm(W, rp_pow_small(r1cs_chal(chal, R1CS_CHAL_YINV), v << kl));                  // y^-(v TL)
    if (which == 0) { tab[e] = W; return; }                                                                 // Yhi
    W = sc_mm(sc_mm(W, r1cs_chal(chal, which == 1 ? R1CS_CHAL_A : R1CS_CHAL_B)), r1cs_chal(chal, R1CS_CHAL_S0));
    tab[e] = sc_mm(W, r1cs_s_part(chal, k, kl, kh, which == 1 ? v : v ^ (TH - 1)));                          // AShi, Qhi
}

// running sums of the weighted g_i and h_i of one generator index over the proofs of a chunk
struct r1cs_acc { sc_wide g, as, h, q; sc w; };
BP_HD void r1cs_acc_init(r1cs_acc &A) { A.g = sc_wide_zero(); A.as = sc_wide_zero(); A.h = sc_wide_zero(); A.q = sc_wide_zero(); A.w = sc_zero(); }
// add proof p's W g_i and W h_i (i < p.padded_n); wL / wR / wO: the proof's own n plain scalars
BP_HD void r1cs_acc_add(r1cs_acc &A, const r1cs_proof &p, const r1cs_head &h, const sc *tab, const sc *wL, const sc *wR, const sc *wO, uint32_t i) {
    const uint32_t kl = rp_kl(p.k), lo = i & ((1u << kl) - 1u), hi = i >> kl, set = i < p.n1 ? 0u : 1u;
    const r1cs_tabs T = r1cs_tab_ptrs(const_cast<sc *>(tab), p.k);
    sc_wide_mac(A.as, T.AShi[set][hi], T.slo[lo]);
    sc_wide_mac(A.q, T.Qhi[set][hi], T.qlo[lo]);
    A.w = sc_add(A.w, set ? h.w_hi : h.w_lo);
    if (i < p.n) {                                                   // wL = wR = wO = 0 on the padding indices
        const sc Y = sc_mm(T.Yhi[set][hi], T.ylo[lo]);
        sc_wide_mac(A.g, Y, sc_mm(h.x, wR[i]));
        sc_wide_mac(A.h, Y, sc_add(sc_mm(h.x, wL[i]), wO[i]));
    }
}
BP_HD void r1cs_acc_final(const r1cs_acc &A, sc &g, sc &hh) {
    g = sc_sub(sc_wide_redc(A.g), sc_wide_redc(A.as));
    hh = sc_sub(sc_sub(sc_wide_redc(A.h), sc_wide_redc(A.q)), A.w);
}
