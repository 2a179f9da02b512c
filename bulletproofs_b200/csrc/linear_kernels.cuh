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

// a proof's C, S, L and R, decompressed once: one thread per point.  A proof with a point that does not decode is a
// VerificationError and is left out of the combination (dec_bad).
__global__ void __launch_bounds__(128) k_lin_decompress(lin_geom g, const uint8_t *__restrict__ proofs, const uint8_t *__restrict__ C, ge_niels *__restrict__ out,
                                                        uint32_t *__restrict__ dec_bad) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)g.count * g.D) return;
    const uint32_t q = (uint32_t)(i / g.D), d = (uint32_t)(i % g.D);
    const uint8_t *proof = proofs + (size_t)q * g.proof_len;
    const uint8_t *src = d == 0 ? C + 32 * (size_t)q : d == 1 ? proof + 64 * g.k : d < 2 + g.k ? proof + 64 * (d - 2) : proof + 64 * (d - 2 - g.k) + 32;
    uint8_t s[32]; ld32(s, src);
    fe x, y; const bool valid = ge_decode(x, y, s);
    st_niels(out + i, valid ? ge_to_niels_affine(x, y) : ge_niels_identity());
    if (!valid) dec_bad[q] = 1u;
}
// transcript replay, one thread per proof, with the byte-wise merlin_* functions on a STROBE state in the thread's own 204-byte shared-memory row; also flags a b entry >= l
#define LIN_TR_THREADS 32
__global__ void __launch_bounds__(LIN_TR_THREADS) k_lin_transcript(lin_geom g, const uint8_t *__restrict__ tstates, const uint8_t *__restrict__ proofs,
                                                                   const uint8_t *__restrict__ C, const uint8_t *__restrict__ b, const uint8_t *__restrict__ enc,
                                                                   const uint8_t *__restrict__ seed, uint8_t *__restrict__ raw, uint32_t *__restrict__ status,
                                                                   uint32_t *__restrict__ noncanonical) {
    __shared__ __align__(16) uint8_t rows[LIN_TR_THREADS][204];
    const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= g.count) return;
    const uint8_t *bq = b + (size_t)q * g.n * 32;
    if (!lin_b_canonical(bq, g.n)) atomicOr(noncanonical, 1u);
    uint8_t (*my)[64] = reinterpret_cast<uint8_t (*)[64]>(raw + (size_t)q * lin_raw_rows(g.k) * 64);
    status[q] = lin_transcript_raw(my, proofs + (size_t)q * g.proof_len, g.k, g.n, C + 32 * (size_t)q, bq, enc, tstates + (size_t)q * BP_TRANSCRIPT_BYTES, seed,
                                   rows[threadIdx.x]);
}
// per-proof head and tables (linear.cuh): one block per proof, one table entry per thread; weighted = combined check (rho), else rho = 1
__global__ void __launch_bounds__(128) k_lin_tables(lin_geom g, const uint8_t *__restrict__ raw, const uint8_t *__restrict__ proofs, int weighted,
                                                    uint32_t *__restrict__ status, lin_head *__restrict__ heads, sc *__restrict__ tabs) {
    __shared__ sc xsh[BP_MAX_LG_N];
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
// <b, s> over the tile's indices (plain; the same on the combined and the reject pass, which writes it again).
__global__ void __launch_bounds__(128) k_lin_g_sum(lin_geom g, const lin_head *__restrict__ heads, const sc *__restrict__ tabs, const uint8_t *__restrict__ b,
                                                   const uint32_t *__restrict__ dec_bad, uint32_t p0, uint32_t count, uint32_t chunk, sc *__restrict__ part_g,
                                                   sc *__restrict__ part_b0) {
    __shared__ sc wsum[4][LIN_CHUNK];                 // per warp, per proof of the chunk
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x, ch = blockIdx.y, lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    const uint32_t q0 = p0 + ch * chunk, q1 = min(p0 + count, q0 + chunk), tsz = lin_tab_size(g.k);
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
    if (threadIdx.x < q1 - q0) {
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
// scalars (chunks of one proof), dyn = the combined row, whose dynamic scalars k_lin_dynamic has rewritten with rho = 1
__global__ void __launch_bounds__(256) k_lin_proof_rows(lin_geom g, uint32_t p0, uint32_t cnt, const sc *__restrict__ part_g, const sc *__restrict__ bf,
                                                        const uint8_t *__restrict__ dyn, uint8_t *__restrict__ scal, uint32_t *__restrict__ pidx) {
    const uint32_t row = g.n + 2 + g.D;
    const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (size_t)cnt * row) return;
    const uint32_t r = (uint32_t)(t / row), e = (uint32_t)(t % row), q = p0 + r;
    uint8_t bytes[32]; uint32_t v = e;
    if (e < 2) sc_store(bytes, bf[2 * (size_t)q + e]);
    else if (e < g.n + 2) sc_store(bytes, sc_from_mont(part_g[(size_t)r * g.n + e - 2]));
    else { const uint32_t o = e - g.n - 2; ld32(bytes, dyn + 32 * ((size_t)g.n + 2 + (size_t)q * g.D + o)); v = BP_POINT_DYNAMIC | (uint32_t)((size_t)q * g.D + o); }
    st32(scal + 32 * t, bytes); pidx[t] = v;
}
