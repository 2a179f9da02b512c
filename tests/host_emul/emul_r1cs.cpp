// TEST-ONLY host build of the R1CS batch verifier's scalar algebra (csrc/r1cs.cuh compiled with g++), linked into libemul.so beside
// emul.cpp.  It lets the CPU-only test tier check the weighted G/H sums against Python integers without a GPU.  Nothing in the
// product links this.
#include <algorithm>
#include <cstring>
#include <vector>
#include "../../bulletproofs_b200/csrc/r1cs.cuh"

extern "C" {

// the R1CS batch verifier's G/H sums (r1cs.cuh) as k_r1cs_tables + k_r1cs_gh_sum compute them: `count` proofs given as in
// bp_r1cs_verify_batch (dims 4 per proof, chal, wL / wR / wO), chunks of `chunk` proofs, W = rho u1 (weighted) or u1.
// out = ceil(count / chunk) rows of 2*Nmax canonical scalars: [sum W g_i, i < Nmax | sum W h_i, i < Nmax]
uint32_t emul_r1cs_tab_size(uint32_t k) { return r1cs_tab_size(k); }
void emul_r1cs_gh_sums(uint32_t count, const uint32_t *dims, const uint8_t *chal, const uint8_t *wL, const uint8_t *wR, const uint8_t *wO, int weighted, uint32_t chunk,
                       uint8_t *out) {
    std::vector<r1cs_proof> P(count); std::vector<r1cs_head> H(count);
    uint32_t chal_n = 0, w_n = 0, tab_n = 0, Nmax = 1;
    for (uint32_t j = 0; j < count; j++) {
        r1cs_proof &p = P[j];
        p.padded_n = dims[4 * j]; p.n1 = dims[4 * j + 1]; p.n = dims[4 * j + 2]; p.k = 0; while ((1u << p.k) < p.padded_n) p.k++;
        p.chal_off = chal_n; p.w_off = w_n; p.tab_off = tab_n; p.term_off = 0;
        chal_n += R1CS_CHAL_USQ + p.k; w_n += p.n; tab_n += r1cs_tab_size(p.k); Nmax = std::max(Nmax, p.padded_n);
    }
    std::vector<sc> tabs(tab_n), L(w_n), R(w_n), O(w_n);
    for (uint32_t i = 0; i < w_n; i++) { L[i] = sc_load(wL + 32 * i); R[i] = sc_load(wR + 32 * i); O[i] = sc_load(wO + 32 * i); }
    for (uint32_t j = 0; j < count; j++) {
        const uint8_t *c = chal + 32 * (size_t)P[j].chal_off;
        r1cs_head_init(H[j], c, weighted != 0);
        for (uint32_t e = 0; e < r1cs_tab_size(P[j].k); e++) r1cs_tab_entry(tabs.data() + P[j].tab_off, c, P[j].k, weighted != 0, e);
    }
    for (uint32_t ch = 0; ch * chunk < count; ch++)
        for (uint32_t i = 0; i < Nmax; i++) {
            r1cs_acc A; r1cs_acc_init(A);
            for (uint32_t q = ch * chunk; q < std::min(count, (ch + 1) * chunk); q++)
                if (i < P[q].padded_n) r1cs_acc_add(A, P[q], H[q], tabs.data() + P[q].tab_off, L.data() + P[q].w_off, R.data() + P[q].w_off, O.data() + P[q].w_off, i);
            sc g, h; r1cs_acc_final(A, g, h);
            sc_store(out + 32 * ((size_t)ch * 2 * Nmax + i), g); sc_store(out + 32 * ((size_t)ch * 2 * Nmax + Nmax + i), h);
        }
}
}
