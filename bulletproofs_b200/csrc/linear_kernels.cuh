// Kernels of the LinearProof batch verifier (bp_linear_verify_batch in bpmsm.cu); the scalar algebra is in linear.cuh.
//
// Combined check, one MSM over the row
//     [sum rho r (set point B) | sum rho a b0 (F) | sum rho a s_i (G_i), i < n | C, S, L.., R.. of every proof, weighted]
// whose first n + 2 terms use the set's resident points and the rest the batch's decompressed points.  Reject path: the same kernels
// with rho = 1 and chunks of one proof, then one MSM per proof over [B, F, G_0..G_{n-1} | C, S, L.., R..], its own equation.
#pragma once
#include "kernels.cuh"
#include "linear.cuh"

struct lin_geom { uint32_t n, k, count, proof_len, D; };      // D = lin_dyn_terms(k)
// per-call parameters on the device: the batch seed, the live count (proofs [live, count) are inert slots: no decompression, replay or
// table work, zero scalars, no verdict) and the flag of a b entry >= l
struct lin_params { uint8_t seed[32]; uint32_t live, noncanonical; };

// a proof's C, S, L and R, decompressed once: one thread per point.  A proof with a point that does not decode is a
// VerificationError and is left out of the combination (dec_bad).
__global__ void __launch_bounds__(128) k_lin_decompress(lin_geom g, const lin_params *__restrict__ par, const uint8_t *__restrict__ proofs, const uint8_t *__restrict__ C,
                                                        ge_niels *__restrict__ out, uint32_t *__restrict__ dec_bad) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)g.count * g.D) return;
    const uint32_t q = (uint32_t)(i / g.D), d = (uint32_t)(i % g.D);
    if (q >= par->live) return;
    const uint8_t *proof = proofs + (size_t)q * g.proof_len;
    const uint8_t *src = d == 0 ? C + 32 * (size_t)q : d == 1 ? proof + 64 * g.k : d < 2 + g.k ? proof + 64 * (d - 2) : proof + 64 * (d - 2 - g.k) + 32;
    uint8_t s[32]; ld32(s, src);
    fe x, y; const bool valid = ge_decode(x, y, s);
    st_niels(out + i, valid ? ge_to_niels_affine(x, y) : ge_niels_identity());
    if (!valid) dec_bad[q] = 1u;
}
// transcript replay, one thread per proof, with the byte-wise merlin_* functions on a STROBE state in the thread's own 204-byte shared-memory row.
// A proof with a b entry >= l raises par->noncanonical and gets status BP_VERDICT_NONCANONICAL_B without a replay; an inert slot gets
// VerificationError, so that every later kernel leaves both out of the combination.
#define LIN_TR_THREADS 32
__global__ void __launch_bounds__(LIN_TR_THREADS) k_lin_transcript(lin_geom g, lin_params *__restrict__ par, const uint8_t *__restrict__ tstates,
                                                                   const uint8_t *__restrict__ proofs, const uint8_t *__restrict__ C, const uint8_t *__restrict__ b,
                                                                   const uint8_t *__restrict__ enc, uint8_t *__restrict__ raw, uint32_t *__restrict__ status) {
    __shared__ __align__(16) uint8_t rows[LIN_TR_THREADS][204];
    const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= g.count) return;
    if (q >= par->live) { status[q] = BP_PROOF_VERIFICATION_ERROR; return; }
    const uint8_t *bq = b + (size_t)q * g.n * 32;
    if (!lin_b_canonical(bq, g.n)) { atomicOr(&par->noncanonical, 1u); status[q] = BP_VERDICT_NONCANONICAL_B; return; }
    uint8_t (*my)[64] = reinterpret_cast<uint8_t (*)[64]>(raw + (size_t)q * lin_raw_rows(g.k) * 64);
    status[q] = lin_transcript_raw(my, proofs + (size_t)q * g.proof_len, g.k, g.n, C + 32 * (size_t)q, bq, enc, tstates + (size_t)q * BP_TRANSCRIPT_BYTES, par->seed,
                                   rows[threadIdx.x]);
}
// The reduced round challenges of a block's proof, shared by k_lin_tables and k_linm_tables (linear_mixed.cuh).  One array at namespace
// scope: every call of lin_head_init passes the same array, so the compiler folds it into the function instead of passing a pointer.
__shared__ sc lin_xsh[BP_MAX_LG_N];
// per-proof head and tables (linear.cuh): one block per proof, one table entry per thread; weighted = combined check (rho), else rho = 1
__global__ void __launch_bounds__(128) k_lin_tables(lin_geom g, const uint8_t *__restrict__ raw, const uint8_t *__restrict__ proofs, int weighted,
                                                    uint32_t *__restrict__ status, lin_head *__restrict__ heads, sc *__restrict__ tabs) {
    sc *xsh = lin_xsh;
    const uint32_t q = blockIdx.x, st = status[q];
    if (st != BP_PROOF_OK) { if (threadIdx.x == 0) heads[q].status = st; return; }
    const uint8_t *rw = raw + (size_t)q * lin_raw_rows(g.k) * 64;
    for (uint32_t j = threadIdx.x; j < g.k; j += blockDim.x) xsh[j] = rp_wide(rw + 64 * j);
    __syncthreads();
    if (threadIdx.x == 0 && lin_head_init(heads[q], xsh, g.k, rw + 64 * g.k, rw + 64 * (g.k + 1), proofs + (size_t)q * g.proof_len, weighted != 0) != BP_PROOF_OK)
        status[q] = heads[q].status;
    const uint32_t tsz = lin_tab_size(g.k);
    for (uint32_t e = threadIdx.x; e < tsz; e += blockDim.x) tabs[(size_t)q * tsz + e] = lin_tab_entry(xsh, g.k, e);
}
// G sum.  Block = (tile of blockDim generator indices, chunk of `chunk` proofs out of [p0, p0 + count)); thread = one index i.
// part_g[ch * n + i] = sum over the chunk's included proofs of rho a s_i (Montgomery form); part_b0[tile * g.count + q] = proof q's
// <b, s> over the tile's indices (plain; the same on the combined and the reject pass, which writes it again).  ctr (the device reject
// path's counters: live, iteration, iterations) replaces p0 with iteration * count and stops the proofs at live; null elsewhere.
__global__ void __launch_bounds__(128) k_lin_g_sum(lin_geom g, const lin_head *__restrict__ heads, const sc *__restrict__ tabs, const uint8_t *__restrict__ b,
                                                   const uint32_t *__restrict__ dec_bad, uint32_t p0, uint32_t count, uint32_t chunk, const uint32_t *__restrict__ ctr,
                                                   sc *__restrict__ part_g, sc *__restrict__ part_b0) {
    __shared__ sc wsum[4][LIN_CHUNK];                 // per warp, per proof of the chunk
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x, ch = blockIdx.y, lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    if (ctr) p0 = ctr[1] * count;
    const uint32_t end = ctr ? p0 + lin_x_slice_live(ctr[1], count, ctr[0]) : p0 + count;
    const uint32_t q0 = p0 + ch * chunk, q1 = min(end, q0 + chunk), tsz = lin_tab_size(g.k);
    const bool in = i < g.n;
    sc_wide acc = sc_wide_zero();
    for (uint32_t q = q0; q < q1; q++) {
        if (heads[q].status != BP_PROOF_OK || dec_bad[q]) continue;          // the same for the whole block
        sc t = sc_zero();
        if (in) { uint8_t bb[32]; ld32(bb, b + ((size_t)q * g.n + i) * 32); t = lin_acc_add(acc, heads[q].wa, tabs + (size_t)q * tsz, g.k, sc_load(bb), i); }
        for (int d = 16; d >= 1; d >>= 1) {
            sc o; for (int w = 0; w < 8; w++) o.v[w] = __shfl_down_sync(0xffffffffu, t.v[w], d);
            t = sc_add(t, o);
        }
        if (lane == 0) wsum[warp][q - q0] = t;
    }
    if (in) part_g[(size_t)ch * g.n + i] = sc_wide_redc(acc);
    __syncthreads();
    if (q0 < q1 && threadIdx.x < q1 - q0) {
        const uint32_t q = q0 + threadIdx.x;
        sc s = sc_zero();
        if (heads[q].status == BP_PROOF_OK && !dec_bad[q]) for (uint32_t w = 0; w < blockDim.x / 32; w++) s = sc_add(s, wsum[w][threadIdx.x]);
        part_b0[(size_t)blockIdx.x * g.count + q] = s;
    }
}
// per proof: b0 from the tiles' partial sums, its B and F scalars (bf, plain) and its dynamic scalars and point map in the combined
// row, after the n + 2 static entries.  An excluded proof gets zero scalars.
__global__ void __launch_bounds__(128) k_lin_dynamic(lin_geom g, const lin_head *__restrict__ heads, const uint32_t *__restrict__ dec_bad, const sc *__restrict__ part_b0,
                                                     uint32_t tiles, const uint8_t *__restrict__ proofs, sc *__restrict__ bf, uint8_t *__restrict__ scal,
                                                     uint32_t *__restrict__ pidx) {
    const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= g.count) return;
    const bool ok = heads[q].status == BP_PROOF_OK && !dec_bad[q];
    sc sB = sc_zero(), sF = sc_zero();
    if (ok) {
        sc b0 = sc_zero();
        for (uint32_t t = 0; t < tiles; t++) b0 = sc_add(b0, part_b0[(size_t)t * g.count + q]);
        lin_static_bf(heads[q], proofs + (size_t)q * g.proof_len, g.k, b0, sB, sF);
    }
    bf[2 * (size_t)q] = sB; bf[2 * (size_t)q + 1] = sF;
    const size_t base = (size_t)g.n + 2 + (size_t)q * g.D;
    for (uint32_t d = 0; d < g.D; d++) {
        uint8_t bytes[32]; sc_store(bytes, ok ? lin_dyn_scalar(heads[q], d, g.k) : sc_zero());
        st32(scal + 32 * (base + d), bytes);
        pidx[base + d] = BP_POINT_DYNAMIC | (uint32_t)((size_t)q * g.D + d);
    }
}
// combined row, static part: one warp per entry e < n + 2 (B, F: the proofs' bf; G_i: the chunks' partial sums)
__global__ void __launch_bounds__(32) k_lin_g_total(lin_geom g, const sc *__restrict__ part_g, uint32_t nchunks, const sc *__restrict__ bf, uint8_t *__restrict__ scal,
                                                    uint32_t *__restrict__ pidx) {
    const uint32_t e = blockIdx.x;
    sc acc = sc_zero();
    if (e < 2) for (uint32_t q = threadIdx.x; q < g.count; q += 32) acc = sc_add(acc, bf[2 * (size_t)q + e]);
    else for (uint32_t c = threadIdx.x; c < nchunks; c += 32) acc = sc_add(acc, part_g[(size_t)c * g.n + e - 2]);
    for (int d = 16; d >= 1; d >>= 1) {
        sc o; for (int w = 0; w < 8; w++) o.v[w] = __shfl_down_sync(0xffffffffu, acc.v[w], d);
        acc = sc_add(acc, o);
    }
    if (threadIdx.x == 0) {
        uint8_t bytes[32]; sc_store(bytes, e < 2 ? acc : sc_from_mont(acc));
        st32(scal + 32 * (size_t)e, bytes); pidx[e] = e;
    }
}
// reject path: the rows [B, F, G_0..G_{n-1} | C, S, L.., R..] of the proofs [p0, p0 + cnt), n + 2 + D terms each; part_g = their own G
// scalars (chunks of one proof), dyn = the combined row, whose dynamic scalars k_lin_dynamic has rewritten with rho = 1.  ctr as for
// k_lin_g_sum: the rows of proofs at or past live get zero scalars.
__global__ void __launch_bounds__(256) k_lin_proof_rows(lin_geom g, uint32_t p0, uint32_t cnt, const uint32_t *__restrict__ ctr, const sc *__restrict__ part_g,
                                                        const sc *__restrict__ bf, const uint8_t *__restrict__ dyn, uint8_t *__restrict__ scal, uint32_t *__restrict__ pidx) {
    const uint32_t row = g.n + 2 + g.D;
    const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (size_t)cnt * row) return;
    const uint32_t r = (uint32_t)(t / row), e = (uint32_t)(t % row);
    if (ctr) p0 = ctr[1] * cnt;
    const uint32_t q = p0 + r;
    uint8_t bytes[32]; uint32_t v = e;
    if (ctr && r >= lin_x_slice_live(ctr[1], cnt, ctr[0])) { for (int j = 0; j < 32; j++) bytes[j] = 0; v = 0; }
    else if (e < 2) sc_store(bytes, bf[2 * (size_t)q + e]);
    else if (e < g.n + 2) sc_store(bytes, sc_from_mont(part_g[(size_t)r * g.n + e - 2]));
    else { const uint32_t o = e - g.n - 2; ld32(bytes, dyn + 32 * ((size_t)g.n + 2 + (size_t)q * g.D + o)); v = BP_POINT_DYNAMIC | (uint32_t)((size_t)q * g.D + o); }
    st32(scal + 32 * t, bytes); pidx[t] = v;
}

// ---------------------------------------------------------------------------------------------- reserved device calls
// (bp_linear_verify_device: the plain chain above at capacity, then these kernels inside the captured graph)
// Each live proof's verdict as combined_verdicts (bpmsm.cu) gives it: its own code when the front end rejected it (status, or
// VerificationError for a point that does not decode), else OK when the combined MSM vanished and VerificationError until the reject
// path decides it.  flag[0] = the combined check passed.
__global__ void __launch_bounds__(128) k_lin_verdicts(lin_geom g, const lin_params *__restrict__ par, const uint32_t *__restrict__ status,
                                                      const uint32_t *__restrict__ dec_bad, const ge_ext *__restrict__ combined, uint32_t *__restrict__ verdict,
                                                      uint32_t *__restrict__ flag) {
    const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
    const bool ok = ge_is_identity(ld_ext(combined));
    if (q == 0) flag[0] = ok ? 1u : 0u;
    if (q >= lin_x_clamp(par->live, g.count)) return;
    const uint32_t st = status[q];
    verdict[q] = st != BP_PROOF_OK ? st : dec_bad[q] ? (uint32_t)BP_PROOF_VERIFICATION_ERROR : ok ? (uint32_t)BP_PROOF_OK : (uint32_t)BP_PROOF_VERIFICATION_ERROR;
}
// Before the reject loop: ctr = (live, iteration 0, iterations) and the WHILE node's condition
__global__ void k_lin_xloop_init(const lin_params *__restrict__ par, uint32_t capacity, uint32_t P, const uint32_t *__restrict__ flag, uint32_t *__restrict__ ctr,
                                 cudaGraphConditionalHandle cond) {
    const uint32_t live = lin_x_clamp(par->live, capacity), iters = lin_x_iters(live, P, flag[0] == 0);
    ctr[0] = live; ctr[1] = 0; ctr[2] = iters;
    cudaGraphSetConditional(cond, iters ? 1u : 0u);
}
// One reject-path iteration's verdicts: a live proof the front end accepted is OK when its own MSM (results[r]) is the identity
__global__ void __launch_bounds__(128) k_lin_xverdicts(uint32_t P, const uint32_t *__restrict__ ctr, const uint32_t *__restrict__ status,
                                                       const uint32_t *__restrict__ dec_bad, const ge_ext *__restrict__ results, uint32_t *__restrict__ verdict) {
    const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= lin_x_slice_live(ctr[1], P, ctr[0])) return;
    const uint32_t q = ctr[1] * P + r;
    if (status[q] == BP_PROOF_OK && !dec_bad[q] && ge_is_identity(ld_ext(results + r))) verdict[q] = BP_PROOF_OK;
}
