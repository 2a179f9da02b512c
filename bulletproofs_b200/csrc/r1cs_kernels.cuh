// Kernels of the R1CS batch verifier (bp_r1cs_verify_batch in bpmsm.cu); the scalar algebra is in r1cs.cuh.
//
// Combined check, one MSM over the row
//     [sum_p W_p g_i (slot G[0][i]), i < Nmax | sum_p W_p h_i (slot H[0][i]), i < Nmax | rho_p x the other terms of every proof p]
// (Nmax = the largest padded_n; a proof contributes to its own indices only).  Reject path, the same kernels with chunks of one proof
// and W = u1: one MSM per proof over [g (padded_n) | h (padded_n) | its other terms], i.e. the proof's own mega-check.
#pragma once
#include "kernels.cuh"
#include "r1cs.cuh"

// per-proof heads and tables (r1cs.cuh): one block per proof, one table entry per thread
__global__ void __launch_bounds__(128) k_r1cs_tables(const r1cs_proof *__restrict__ proofs, const uint8_t *__restrict__ chal, int weighted,
                                                     r1cs_head *__restrict__ heads, sc *__restrict__ tabs) {
    const r1cs_proof p = proofs[blockIdx.x];
    const uint8_t *c = chal + (size_t)p.chal_off * 32;
    if (threadIdx.x == 0) r1cs_head_init(heads[blockIdx.x], c, weighted != 0);
    const uint32_t sz = r1cs_tab_size(p.k);
    for (uint32_t e = threadIdx.x; e < sz; e += blockDim.x) r1cs_tab_entry(tabs + p.tab_off, c, p.k, weighted != 0, e);
}
// G/H sum.  Block = (tile of blockDim generator indices, chunk of `chunk` proofs out of [p0, p0 + count)); thread = one index i.
// Writes part[ch * 2*Nmax + i] = sum W g_i and part[ch * 2*Nmax + Nmax + i] = sum W h_i over the chunk's proofs that are not excluded
// (plain scalars); a proof adds nothing at i >= its padded_n.
__global__ void __launch_bounds__(128) k_r1cs_gh_sum(const r1cs_proof *__restrict__ proofs, const r1cs_head *__restrict__ heads, const sc *__restrict__ tabs,
                                                     const sc *__restrict__ wL, const sc *__restrict__ wR, const sc *__restrict__ wO, const uint32_t *__restrict__ dec_bad,
                                                     uint32_t p0, uint32_t count, uint32_t chunk, uint32_t Nmax, sc *__restrict__ part) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x, ch = blockIdx.y;
    if (i >= Nmax) return;
    const uint32_t q0 = p0 + ch * chunk, q1 = min(p0 + count, q0 + chunk);
    r1cs_acc A; r1cs_acc_init(A);
    for (uint32_t q = q0; q < q1; q++) {
        const r1cs_proof p = proofs[q];
        if (i >= p.padded_n || dec_bad[q]) continue;
        r1cs_acc_add(A, p, heads[q], tabs + p.tab_off, wL + p.w_off, wR + p.w_off, wO + p.w_off, i);
    }
    sc g, h; r1cs_acc_final(A, g, h);
    sc *row = part + (size_t)ch * 2 * Nmax;
    row[i] = g; row[Nmax + i] = h;
}
// combined row, G/H part: add the chunks' partial sums (one thread per entry) and write the table slots
__global__ void __launch_bounds__(256) k_r1cs_gh_total(const sc *__restrict__ part, uint32_t nchunks, uint32_t Nmax, uint32_t gens_cap, uint32_t gens_parties,
                                                       uint8_t *__restrict__ scal, uint32_t *__restrict__ pidx) {
    const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= 2 * Nmax) return;
    sc acc = sc_zero();
    for (uint32_t c = 0; c < nchunks; c++) acc = sc_add(acc, part[(size_t)c * 2 * Nmax + e]);
    uint8_t b[32]; sc_store(b, acc); st32(scal + 32 * (size_t)e, b);
    pidx[e] = e < Nmax ? (uint32_t)bp_gens_slot(0, 0, e, gens_cap, gens_parties) : (uint32_t)bp_gens_slot(1, 0, e - Nmax, gens_cap, gens_parties);
}
// combined row, other terms: rho_p times each of proof p's other terms (zero for an excluded proof), after the 2*Nmax G/H entries
__global__ void __launch_bounds__(256) k_r1cs_other_terms(const uint32_t *__restrict__ term_off, uint32_t n_proofs, const uint8_t *__restrict__ chal,
                                                          const r1cs_proof *__restrict__ proofs, const uint32_t *__restrict__ dec_bad, const uint8_t *__restrict__ in_scal,
                                                          const uint32_t *__restrict__ in_pidx, uint32_t Nmax, uint8_t *__restrict__ scal, uint32_t *__restrict__ pidx) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= term_off[n_proofs]) return;
    const uint32_t q = msm_of_term(term_off, n_proofs, t);
    uint8_t b[32]; ld32(b, in_scal + 32 * (size_t)t);
    const sc v = dec_bad[q] ? sc_zero() : sc_mm(r1cs_chal(chal + (size_t)proofs[q].chal_off * 32, R1CS_CHAL_RHO), sc_load(b));   // Montgomery x plain = plain
    sc_store(b, v); st32(scal + 32 * ((size_t)2 * Nmax + t), b);
    pidx[2 * Nmax + t] = in_pidx[t];
}
// reject path: the rows [g (padded_n) | h (padded_n) | other terms, unweighted] of the proofs [p0, p0 + count), row q - p0 starting at
// row_off[q - p0]; part = the G/H sums of chunks of one proof with W = u1 (2*Nmax per proof)
__global__ void __launch_bounds__(256) k_r1cs_proof_rows(const uint32_t *__restrict__ row_off, uint32_t p0, uint32_t count, const r1cs_proof *__restrict__ proofs,
                                                         const sc *__restrict__ part, uint32_t Nmax, const uint8_t *__restrict__ in_scal, const uint32_t *__restrict__ in_pidx,
                                                         uint32_t gens_cap, uint32_t gens_parties, uint8_t *__restrict__ scal, uint32_t *__restrict__ pidx) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= row_off[count]) return;
    const uint32_t r = msm_of_term(row_off, count, t), e = t - row_off[r];
    const r1cs_proof p = proofs[p0 + r];
    uint8_t b[32]; uint32_t v;
    if (e < 2 * p.padded_n) {
        const bool isH = e >= p.padded_n; const uint32_t i = isH ? e - p.padded_n : e;
        sc_store(b, part[(size_t)r * 2 * Nmax + (isH ? Nmax : 0) + i]);
        v = (uint32_t)bp_gens_slot(isH ? 1 : 0, 0, i, gens_cap, gens_parties);
    } else {
        const uint32_t o = p.term_off + e - 2 * p.padded_n;
        ld32(b, in_scal + 32 * (size_t)o); v = in_pidx[o];
    }
    st32(scal + 32 * (size_t)t, b); pidx[t] = v;
}
