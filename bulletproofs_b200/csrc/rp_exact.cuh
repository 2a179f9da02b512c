// Device reject path of the exact range-proof entry points (bp_rangeproof_verify_group_device_exact*, bp_rangeproof_verify_mixed_device_exact*):
// the two levels of rp_verify_fallback (bpmsm.cu), driven on the device inside the exact graph (rp_exact_chain).  The pass arithmetic is in
// rp.cuh (rp_x_*).
//
// A group is the proofs of one geometry: the batches of a launch group (units b = 0..nbatch-1 of count proofs each, proof p = b count + q),
// or one class of a mix (one unit of `capacity` slots).  Level 1 builds one MSM row per chunk of RP_CHUNK proofs of every group, zero rows
// for the units whose own check passed, and checks them all in one multi-MSM pass; the live proofs of failing chunks go on the group's list.
// Level 2 runs on each group's list, P proofs per iteration of a WHILE node: their own static-term sums, their rows, one P-MSM pass and their
// verdicts.
#pragma once
#include "kernels.cuh"
#include "rp_mixed.cuh"

struct rp_xgroup {
    rp_geom g;                      // count = proofs per unit, nbatch = units
    const rp_params *par;           // the call's verdict address and live count
    const uint32_t *comb;           // per unit: its own combined check passed
    const uint32_t *status, *decbad;
    const rp_lean_head *chal;
    const sc *tabs, *part;          // head tables; chunk partial sums, S per chunk at (b nchunks + ch) S
    uint8_t *scal;                  // scalar array: proof p's dynamic scalars at scal + (S + p D) 32
    uint32_t dyn_base;              // dynamic point index of proof 0's first point
    uint32_t chunk0, row0;          // the group's first level-1 chunk and that chunk's first term
    uint32_t P;                     // level-2 proofs per iteration (rp_x_slice)
    uint32_t *list;                 // failing-proof list, capacity count nbatch
    uint32_t *ctr;                  // list length, iteration, iterations
    sc *part2;                      // level 2: the static-term sums of the iteration's proofs, S each
};
struct rp_xconds { cudaGraphConditionalHandle h[RP_MIXED_MAX_CLASSES]; };      // the WHILE node of each group

__device__ __forceinline__ uint32_t rp_x_group_live(const rp_xgroup &X) { return min(X.par->live, X.g.count * X.g.nbatch); }
__device__ __forceinline__ uint32_t rp_x_group_of(const rp_xgroup *G, uint32_t ng, uint32_t j) {
    uint32_t gi = 0;
    while (gi + 1 < ng && G[gi + 1].chunk0 <= j) gi++;
    return gi;
}

// After the plain chain: cond = some unit's own check failed; every list starts empty
__global__ void __launch_bounds__(32) k_rp_xprep(const rp_xgroup *__restrict__ G, uint32_t ng, cudaGraphConditionalHandle cond) {
    uint32_t any = 0;
    for (uint32_t gi = 0; gi < ng; gi++) {
        for (uint32_t b = threadIdx.x; b < G[gi].g.nbatch; b += 32) if (!G[gi].comb[b]) any = 1;
        if (threadIdx.x < 3) G[gi].ctr[threadIdx.x] = 0;
    }
    any = __any_sync(0xffffffffu, any);
    if (threadIdx.x == 0) cudaGraphSetConditional(cond, any);
}
// Level 1 rows, one block per chunk j: [S static | RP_CHUNK D dynamic] as k_rp_chunk_rows writes them, or zero scalars for a unit that passed
__global__ void __launch_bounds__(128) k_rp_xchunk_rows(const rp_xgroup *__restrict__ G, uint32_t ng, uint32_t gens_cap, uint32_t gens_parties,
                                                        uint8_t *__restrict__ out_scalars, uint32_t *__restrict__ out_pidx) {
    const uint32_t j = blockIdx.x;
    const rp_xgroup &X = G[rp_x_group_of(G, ng, j)];
    const rp_geom g = X.g;
    const uint32_t nch = (g.count + RP_CHUNK - 1) / RP_CHUNK, c = j - X.chunk0, b = c / nch, ch = c % nch, row = g.S + RP_CHUNK * g.D;
    const bool on = X.comb[b] == 0;
    const size_t base = (size_t)X.row0 + (size_t)c * row;
    for (uint32_t t = threadIdx.x; t < row; t += blockDim.x) {
        uint8_t v[32]; uint32_t idx = 0;
        for (int i = 0; i < 32; i++) v[i] = 0;
        if (on && t < g.S) {
            sc_store(v, sc_from_mont(X.part[((size_t)b * nch + ch) * g.S + t]));
            idx = rp_static_slot(g, t, gens_cap, gens_parties);
        } else if (on) {
            const uint32_t e = t - g.S, q = ch * RP_CHUNK + e / g.D;
            if (q < g.count) {
                const size_t d = (size_t)(b * g.count + q) * g.D + e % g.D;
                ld32(v, X.scal + (g.S + d) * 32);
                idx = BP_POINT_DYNAMIC | (uint32_t)(X.dyn_base + d);
            }
        }
        st32(out_scalars + 32 * (base + t), v); out_pidx[base + t] = idx;
    }
}
// Level 1 verdicts, one warp per chunk j, lane = proof of the chunk.  Units that passed are left alone.  A passing chunk's live proofs get
// their own codes; a failing chunk's live proofs keep VerificationError (or their own code) and go on the list.
__global__ void __launch_bounds__(32) k_rp_xchunk_verdicts(const rp_xgroup *__restrict__ G, uint32_t ng, const ge_ext *__restrict__ results) {
    const uint32_t j = blockIdx.x, lane = threadIdx.x;
    const rp_xgroup &X = G[rp_x_group_of(G, ng, j)];
    const uint32_t nch = (X.g.count + RP_CHUNK - 1) / RP_CHUNK, c = j - X.chunk0, b = c / nch, ch = c % nch;
    if (X.comb[b]) return;
    const bool ok = ge_is_identity(ld_ext(results + j));
    const uint32_t q = ch * RP_CHUNK + lane, p = b * X.g.count + q;
    const uint32_t unit_live = rp_x_unit_live(rp_x_group_live(X), X.g.count, b);
    const bool listed = rp_x_listed(q, unit_live, !ok);
    if (ok && q < unit_live) X.par->verdict[p] = rp_eff_status(X.status[p], X.decbad[p]);
    const uint32_t m = __ballot_sync(0xffffffffu, listed);
    if (!m) return;
    uint32_t at = 0;
    if (lane == 0) at = atomicAdd(X.ctr, __popc(m));
    at = __shfl_sync(0xffffffffu, at, 0);
    if (listed) X.list[at + __popc(m & ((1u << lane) - 1u))] = p;
}
// Before the level-2 loops: each group's list length clamped to its live proofs, its iteration count, and its WHILE condition
__global__ void __launch_bounds__(32) k_rp_xloop_init(const rp_xgroup *__restrict__ G, uint32_t ng, rp_xconds conds) {
    const uint32_t gi = threadIdx.x;
    if (gi >= ng) return;
    const rp_xgroup &X = G[gi];
    const uint32_t n = rp_x_clamp(X.ctr[0], rp_x_group_live(X)), iters = rp_x_iters(n, X.P);
    X.ctr[0] = n; X.ctr[1] = 0; X.ctr[2] = iters;
    cudaGraphSetConditional(conds.h[gi], iters ? 1u : 0u);
}
// Level 2, block i: the static-term sums of the i-th proof of this iteration, what k_rp_scalars_sum computes for a one-proof batch (the
// same products through rp_chunk_dot); a proof that failed or does not decode gets zero sums and zero dynamic scalars
__global__ void __launch_bounds__(128, 4) k_rp_xscalars(rp_xgroup X) {
    const uint32_t at = X.ctr[1] * X.P + blockIdx.x;
    if (at >= X.ctr[0]) return;
    const rp_geom g = X.g;
    const uint32_t p = X.list[at];
    const rp_lean_head &h = X.chal[p];
    const bool ok = h.status == BP_PROOF_OK && !X.decbad[p];
    const uint32_t mask = ok ? 1u : 0u, tsz = rp_tab_size(g.k, g.m);
    const sc zL = ok ? h.zL : sc_zero();
    sc *mine = X.part2 + (size_t)blockIdx.x * g.S;
    const uint32_t kl = rp_kl(g.k), TL = 1u << kl, TH = 1u << (g.k - kl);
    const uint32_t e_slo = 0, e_Ahi = TL, e_Plo = TL + TH, e_Phi = 2 * TL + TH, e_Qlo = 2 * TL + 2 * TH, e_Qhi = 3 * TL + 2 * TH;
    for (uint32_t i = threadIdx.x; i < g.N; i += blockDim.x) {
        const uint32_t lo = i & (TL - 1), hi = i >> kl;
        mine[2 + i] = sc_sub(sc_neg(zL), rp_chunk_dot(X.tabs, p, tsz, mask, e_Ahi + hi, e_slo + lo));
        const sc hP = sc_add(zL, rp_chunk_dot(X.tabs, p, tsz, mask, e_Phi + hi, e_Plo + lo));
        mine[2 + g.N + i] = sc_sub(hP, rp_chunk_dot(X.tabs, p, tsz, mask, e_Qhi + hi, e_Qlo + lo));
    }
    if (threadIdx.x < 2) mine[threadIdx.x] = ok ? (threadIdx.x == 0 ? h.blinding_scalar : h.basepoint_scalar) : sc_zero();
    if (ok) return;
    for (uint32_t e = threadIdx.x; e < g.D; e += blockDim.x) {
        uint4 *o = reinterpret_cast<uint4 *>(X.scal + (g.S + (size_t)p * g.D + e) * 32);
        o[0] = make_uint4(0, 0, 0, 0); o[1] = make_uint4(0, 0, 0, 0);
    }
}
// Level 2 rows: row i = [S static | D dynamic] of the iteration's i-th proof, zero scalars past the list's end
__global__ void __launch_bounds__(128) k_rp_xrows(rp_xgroup X, uint32_t gens_cap, uint32_t gens_parties, uint8_t *__restrict__ out_scalars, uint32_t *__restrict__ out_pidx) {
    const rp_geom g = X.g;
    const uint32_t row = g.S + g.D;
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)X.P * row) return;
    const uint32_t r = (uint32_t)(i / row), t = (uint32_t)(i % row), at = X.ctr[1] * X.P + r;
    uint8_t v[32]; uint32_t idx = 0;
    for (int k = 0; k < 32; k++) v[k] = 0;
    if (at < X.ctr[0]) {
        if (t < g.S) {
            sc_store(v, sc_from_mont(X.part2[(size_t)r * g.S + t]));
            idx = rp_static_slot(g, t, gens_cap, gens_parties);
        } else {
            const size_t d = (size_t)X.list[at] * g.D + (t - g.S);
            ld32(v, X.scal + (g.S + d) * 32);
            idx = BP_POINT_DYNAMIC | (uint32_t)(X.dyn_base + d);
        }
    }
    st32(out_scalars + 32 * i, v); out_pidx[i] = idx;
}
// Level 2 verdicts: a proof whose own MSM is the identity gets its own code; the others keep VerificationError
__global__ void __launch_bounds__(128) k_rp_xverdicts(rp_xgroup X, const ge_ext *__restrict__ results) {
    const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= X.P) return;
    const uint32_t at = X.ctr[1] * X.P + r;
    if (at >= X.ctr[0] || !ge_is_identity(ld_ext(results + r))) return;
    const uint32_t p = X.list[at];
    X.par->verdict[p] = rp_eff_status(X.status[p], X.decbad[p]);
}
// end of a level-2 iteration: the loop runs again while iterations are left (at most rp_x_iters of the clamped length)
__global__ void k_rp_xloop_next(uint32_t *__restrict__ ctr, cudaGraphConditionalHandle cond) {
    const uint32_t it = ++ctr[1];
    cudaGraphSetConditional(cond, it < ctr[2] ? 1u : 0u);
}
