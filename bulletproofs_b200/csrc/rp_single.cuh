// Fused single-proof range-proof verifier: one thread-block cluster per proof, one launch per call.
//
// The launch-group pipeline (kernels.cuh, range-proof section) spreads a batch over ~15 dependent launches, each nearly empty when the
// batch holds one proof.  Here a cluster of P.cl CTAs verifies its proof alone, with the proof's own check (mod.rs:421-447) weighted
// by rho * lambda as on the pipeline (rp.cuh header), so the verdict is exact and there is no reject path:
//   1. front end, in every CTA of the cluster: lane 0 replays the transcript (rp_transcript_proof) while warps 1.. decode the proof's
//      D points (ge_decode); thread 0 then runs the head (rp_head_lean), whose tables stay in shared memory;
//   2. the S = 2 + 2N static scalars (k_rp_scalars_sum's algebra for a chunk of one proof) and the D dynamic ones, recoded into
//      signed c-bit digits (msm_recode), one thread per term;
//   3. the MSM of S + D terms: CTA r of the cluster owns the windows [r wpc, (r+1) wpc), one thread per (window, bucket).  Each thread
//      lists the terms of its bucket (count, scan across the window's lanes, scatter), adds their points, and the window's lanes
//      reduce sum_b (b+1) B_b with shuffles; the window sums go to CTA 0 through distributed shared memory;
//   4. CTA 0 combines the W window sums (Horner, four lanes per point as k_msm_combine4) and writes the identity-coset verdict.
// The front end is computed redundantly by every CTA of the cluster: it is latency, and the copies run on different SMs, so only the
// window sums cross between CTAs.  The Horner chain of c (W - 1) ~ 253 doublings is the floor of the launch.
#pragma once
#include <cooperative_groups.h>
#include "kernels.cuh"

#define RP_SINGLE_THREADS 256
#define RP_SINGLE_MIN_K 3               // n >= 8
#define RP_SINGLE_MAX_K 10              // kernel instances; the routing rule (bpmsm.cu) may use fewer
#define RP_SINGLE_MAX_COUNT 64          // clusters of one launch the host path accepts (verdict staging)
#define RP_SINGLE_HDR 256               // device input block: caller transcript state (208 B) | seed (32 B) | pad, then proofs, commitments

// MSM plan of one proof's S + D terms: window size c, W windows of nb = 2^(c-1) buckets, cl CTAs per cluster, wpc windows per CTA
// (wpc * nb <= RP_SINGLE_THREADS, and nb divides 32, so a window's lanes never straddle a warp).  Shared with the host tests.
struct rp_single_plan { uint32_t c, W, nb, cl, wpc; };
BP_HD rp_single_plan rp_single_plan_of(uint32_t T) {
    rp_single_plan p;
    p.c = T <= 320 ? 5 : 6;
    p.cl = T <= 320 ? 4 : 8;
    p.W = (uint32_t)msm_num_windows((int)p.c); p.nb = 1u << (p.c - 1); p.wpc = (p.W + p.cl - 1) / p.cl;
    return p;
}
// byte offsets of the dynamic shared memory of one CTA
struct rp_single_smem { uint32_t wsum, niels, tabs, dyn, rec, lists, total; };
BP_HD rp_single_smem rp_single_layout(const rp_geom &g, const rp_single_plan &p) {
    const uint32_t T = g.S + g.D;
    rp_single_smem s; uint32_t o = 0;
    s.wsum = o; o += p.W * 128;                      // ge_ext window sums (CTA 0's are the ones read)
    s.niels = o; o += g.D * 96;                      // the proof's points, ge_niels
    s.tabs = o; o += rp_tab_size(g.k, g.m) * 32;     // the head's tables (stride 1)
    s.dyn = o; o += g.D * 32;                        // the head's dynamic scalars, canonical bytes
    s.rec = o; o += T * 36;                          // msm_wide recoding of every term
    s.lists = o; o += p.wpc * T * 2;                 // per window of the CTA: term ids of its buckets, bucket after bucket
    s.total = (o + 15) & ~15u;
    return s;
}
// bytes of one call's device input block for `count` proofs
BP_HD size_t rp_single_input_bytes(const rp_geom &g, uint32_t count) { return RP_SINGLE_HDR + (size_t)count * (g.proof_len + 32 * g.m); }

#ifdef __CUDACC__
// encoding of the proof's point idx in MSM order A, S, T_1, T_2, L.., R.., V..
__device__ __forceinline__ const uint8_t *rp_single_point(const uint8_t *proof, const uint8_t *V, uint32_t k, uint32_t idx) {
    if (idx < 4) return proof + 32 * idx;
    if (idx < 4 + k) return proof + 224 + 64 * (idx - 4);
    if (idx < 4 + 2 * k) return proof + 224 + 64 * (idx - 4 - k) + 32;
    return V + 32 * (idx - 4 - 2 * k);
}
__device__ __forceinline__ ge_ext rp_single_shfl_down(const ge_ext &p, uint32_t d, int width) {
    ge_ext r;
#pragma unroll
    for (int i = 0; i < 8; i++) {
        r.X.v[i] = __shfl_down_sync(0xffffffffu, p.X.v[i], d, width); r.Y.v[i] = __shfl_down_sync(0xffffffffu, p.Y.v[i], d, width);
        r.Z.v[i] = __shfl_down_sync(0xffffffffu, p.Z.v[i], d, width); r.T.v[i] = __shfl_down_sync(0xffffffffu, p.T.v[i], d, width);
    }
    return r;
}
// Horner combination of the window sums R[0..W) by one warp, four lanes per point (lane q holds coordinate q of X, Y, Z, T; the formulas
// of k_msm_combine4).  Every group of four lanes computes the same point; returns whether it lies in the identity coset (X == 0 or Y == 0).
__device__ __noinline__ bool rp_single_horner_is_identity(const ge_ext *R, int W, int c) {
    const uint32_t q = threadIdx.x & 3;
    const fe d2 = fe_const_d2();
    fe cur = ld_fe(&R[W - 1].X + q);
#pragma unroll 1
    for (int w = W - 2; w >= 0; w--) {
#pragma unroll 1
        for (int i = 0; i < c; i++) {
            fe x = shfl_fe4(cur, 0), y = shfl_fe4(cur, 1);
            fe sq = fe_sq(sel_fe(q == 3, cur, fe_add(x, y)));
            fe A = shfl_fe4(sq, 0), B = shfl_fe4(sq, 1), ZZ = shfl_fe4(sq, 2), D = shfl_fe4(sq, 3);
            fe H = fe_add(A, B), E = fe_sub(D, H), G = fe_sub(B, A), F = fe_sub(G, fe_dbl(ZZ)), Hn = fe_neg(H);
            fe o1 = sel_fe(q == 1, sel_fe(q == 2, E, F), G), o2 = sel_fe(q == 0, sel_fe(q == 2, Hn, G), F);
            cur = fe_mul(o1, o2);
        }
        const ge_ext *P2 = R + w;
        fe X2 = ld_fe(&P2->X), Y2 = ld_fe(&P2->Y), Z2 = ld_fe(&P2->Z), T2d = fe_mul(ld_fe(&P2->T), d2);
        fe x1 = shfl_fe4(cur, 0), y1 = shfl_fe4(cur, 1);
        fe a = sel_fe(q >= 2, sel_fe(q == 1, fe_sub(y1, x1), fe_add(y1, x1)), cur);
        fe b = sel_fe(q == 1, sel_fe(q == 2, sel_fe(q == 3, fe_sub(Y2, X2), T2d), Z2), fe_add(Y2, X2));
        fe pr = fe_mul(a, b);
        fe A = shfl_fe4(pr, 0), B = shfl_fe4(pr, 1), Dh = shfl_fe4(pr, 2), C = shfl_fe4(pr, 3);
        fe D = fe_dbl(Dh), E = fe_sub(B, A), F = fe_sub(D, C), G = fe_add(D, C), H = fe_add(B, A);
        fe o1 = sel_fe(q == 1, sel_fe(q == 2, E, F), G), o2 = sel_fe(q == 0, sel_fe(q == 2, H, G), F);
        cur = fe_mul(o1, o2);
    }
    const bool zero = fe_is_zero(cur);
    const uint32_t m = __ballot_sync(0xffffffffu, zero);
    return (m & 3u) != 0;                       // lane 0: X, lane 1: Y
}

// One CTA per SM is all a cluster launch of a few proofs fills, so the launch bounds ask for one: 138-148 registers and no spill (with the
// default bound ptxas holds 128 and spills up to 44 B).  One cluster per proof p = blockIdx.x / P.cl.  in = the call's input block (rp_single_input_bytes), raw = (RP_RAW_U + K) * 64 bytes of
// challenge rows per CTA, verdict[p] = the proof's ProofError code.
template <uint32_t K>
__global__ void __launch_bounds__(RP_SINGLE_THREADS, 1) k_rp_single(rp_geom g, rp_single_plan P, const uint8_t *__restrict__ in, const rp_tr_step *__restrict__ prog,
                                                                 uint32_t nsteps, const ge_niels *__restrict__ gens, uint32_t gens_cap, uint32_t gens_parties,
                                                                 const sc *__restrict__ pow2, uint8_t *__restrict__ raw_all, uint32_t *__restrict__ verdict) {
    namespace cg = cooperative_groups;
    cg::cluster_group cluster = cg::this_cluster();
    extern __shared__ __align__(128) uint8_t smem[];
    __shared__ rp_lean_head head;
    __shared__ uint32_t s_status, s_bad;
    const rp_single_smem L = rp_single_layout(g, P);
    const uint32_t tid = threadIdx.x, p = blockIdx.x / P.cl, rank = cluster.block_rank(), T = g.S + g.D;
    const uint8_t *proof = in + RP_SINGLE_HDR + (size_t)p * g.proof_len;
    const uint8_t *V = in + RP_SINGLE_HDR + (size_t)g.count * g.proof_len + (size_t)p * g.m * 32;
    uint8_t *raw = raw_all + (size_t)blockIdx.x * (RP_RAW_U + K) * 64;
    ge_ext *wsum = reinterpret_cast<ge_ext *>(smem + L.wsum);
    ge_niels *niels = reinterpret_cast<ge_niels *>(smem + L.niels);
    sc *tabs = reinterpret_cast<sc *>(smem + L.tabs);
    uint8_t *dyn = smem + L.dyn;
    msm_wide *rec = reinterpret_cast<msm_wide *>(smem + L.rec);
    uint16_t *lists = reinterpret_cast<uint16_t *>(smem + L.lists);

    // 1. front end
    if (tid == 0) s_bad = 0u;
    __syncthreads();
    if (tid == 0) {
        s_status = rp_transcript_proof(raw, proof, K, V, in, 0, 0, in + 208, prog, nsteps);
    } else if (tid >= 32) {
        for (uint32_t i = tid - 32; i < g.D; i += blockDim.x - 32) {
            uint8_t s[32]; ld32_any(s, rp_single_point(proof, V, K, i));
            fe x, y; const bool ok = ge_decode(x, y, s);
            st_niels(niels + i, ok ? ge_to_niels_affine(x, y) : ge_niels_identity());
            if (!ok) atomicOr(&s_bad, 1u);
        }
    }
    __syncthreads();
    if (tid == 0 && s_status == BP_PROOF_OK) s_status = rp_head_lean(head, tabs, dyn, pow2, raw, proof, K, g.n, g.m);
    // every CTA of the cluster has started (its shared memory may be written) once this returns
    cluster.sync();
    const bool live = s_status == BP_PROOF_OK && s_bad == 0u;
    if (live) {
        // 2. scalars of the S static terms [B_blinding, B, G(n, m).., H(n, m)..] and the D dynamic terms, recoded
        const uint32_t kl = rp_kl(K), TL = 1u << kl;
        const rp_tabs tb = rp_tab_ptrs(tabs, K);
        for (uint32_t t = tid; t < T; t += blockDim.x) {
            sc s;
            if (t < 2) s = rp_from_mont(t == 0 ? head.blinding_scalar : head.basepoint_scalar);
            else if (t < g.S) {
                const uint32_t i = (t - 2) % g.N, lo = i & (TL - 1), hi = i >> kl;
                if (t - 2 < g.N) s = sc_sub(sc_neg(head.zL), rp_mul(tb.A_hi[hi], tb.s_lo[lo]));                          // g_i
                else s = sc_sub(sc_add(head.zL, rp_mul(tb.P_hi[hi], tb.P_lo[lo])), rp_mul(tb.Q_hi[hi], tb.Q_lo[lo]));     // h_i
                s = rp_from_mont(s);
            } else s = sc_load(dyn + 32 * (t - g.S));
            rec[t] = msm_recode(s.v, (int)P.c, (int)P.W);
        }
        __syncthreads();
        // 3. this CTA's windows: thread (wl, b) owns bucket b of window rank * wpc + wl
        const uint32_t nb = P.nb, wl = tid / nb, b = tid % nb, w = rank * P.wpc + wl;
        const bool mine = wl < P.wpc && w < P.W;
        uint32_t cnt = 0;
        if (mine)
            for (uint32_t t = 0; t < T; t++) { const int d = msm_digit(rec[t], (int)w, (int)P.c); cnt += (uint32_t)(d == (int)b + 1 || d == -(int)b - 1); }
        uint32_t x = cnt;                          // exclusive scan of the counts over the window's nb lanes
        for (uint32_t d = 1; d < nb; d <<= 1) { const uint32_t o = __shfl_up_sync(0xffffffffu, x, d, (int)nb); if (b >= d) x += o; }
        const uint32_t start = x - cnt;
        uint16_t *lst = lists + (size_t)wl * T + start;
        if (mine) {
            uint32_t pos = 0;
            for (uint32_t t = 0; t < T; t++) {
                const int d = msm_digit(rec[t], (int)w, (int)P.c);
                if (d == (int)b + 1 || d == -(int)b - 1) lst[pos++] = (uint16_t)(t | (d < 0 ? 0x8000u : 0u));
            }
        }
        ge_ext acc = ge_identity();
        if (mine) {
#pragma unroll 1
            for (uint32_t e = 0; e < cnt; e++) {
                const uint32_t v = lst[e], t = v & 0x7fffu;
                const ge_niels q = t < g.S ? ldg_niels(gens + rp_static_slot(g, t, gens_cap, gens_parties)) : niels[t - g.S];
                acc = (v & 0x8000u) ? ge_msub(acc, q) : ge_madd(acc, q);
            }
        }
        // sum_b (b+1) B_b = sum_j (sum_{b >= j} B_b): suffix sums over the window's lanes, then their total
#pragma unroll 1
        for (uint32_t d = 1; d < nb; d <<= 1) { const ge_ext o = rp_single_shfl_down(acc, d, (int)nb); if (b + d < nb) acc = ge_add(acc, o); }
#pragma unroll 1
        for (uint32_t d = nb >> 1; d >= 1; d >>= 1) { const ge_ext o = rp_single_shfl_down(acc, d, (int)nb); acc = ge_add(acc, o); }
        if (mine && b == 0) *cluster.map_shared_rank(wsum + w, 0) = acc;
    }
    cluster.sync();
    // 4. the verdict
    if (rank != 0 || tid >= 32) return;
    if (!live) { if (tid == 0) verdict[p] = rp_eff_status(s_status, s_bad); return; }
    const bool ident = rp_single_horner_is_identity(wsum, (int)P.W, (int)P.c);
    if (tid == 0) verdict[p] = ident ? (uint32_t)BP_PROOF_OK : (uint32_t)BP_PROOF_VERIFICATION_ERROR;
}
typedef decltype(&k_rp_single<RP_SINGLE_MIN_K>) rp_single_fn;
template <uint32_t... I> static rp_single_fn rp_single_pick(uint32_t k, std::integer_sequence<uint32_t, I...>) {
    static const rp_single_fn fns[] = {&k_rp_single<RP_SINGLE_MIN_K + I>...};
    return fns[k - RP_SINGLE_MIN_K];
}
// the instance for k in [RP_SINGLE_MIN_K, RP_SINGLE_MAX_K]
static rp_single_fn rp_single_kernel(uint32_t k) { return rp_single_pick(k, std::make_integer_sequence<uint32_t, RP_SINGLE_MAX_K - RP_SINGLE_MIN_K + 1>()); }
#endif
