// The MSM of the fused single-proof verifiers (k_rp_single in rp_single.cuh, k_lin_single in linear_single.cuh): one thread-block
// cluster per proof, the proof's T recoded terms in shared memory, and a verdict that the sum lies in the identity coset.
//   - CTA r of the cluster owns the windows [r wpc, (r+1) wpc), one thread per (window, bucket).  Each thread lists the terms of its
//     bucket (count, scan across the window's lanes, scatter), adds their points, and the window's lanes reduce sum_b (b+1) B_b with
//     shuffles; the window sums go to CTA 0 through distributed shared memory;
//   - CTA 0 combines the W window sums (Horner, four lanes per point as k_msm_combine4).
// The Horner chain of c (W - 1) ~ 253 doublings is the floor of a launch.  The plan is host code, shared with the host tests.
#pragma once
#include "msm_common.cuh"

// MSM plan of one proof's T terms: window size c, W windows of nb = 2^(c-1) buckets, cl CTAs per cluster, wpc windows per CTA
// (wpc * nb <= RP_SINGLE_THREADS, and nb divides 32, so a window's lanes never straddle a warp).
#define RP_SINGLE_THREADS 256
struct rp_single_plan { uint32_t c, W, nb, cl, wpc; };
BP_HD rp_single_plan rp_single_plan_of(uint32_t T) {
    rp_single_plan p;
    p.c = T <= 320 ? 5 : 6;
    p.cl = T <= 320 ? 4 : 8;
    p.W = (uint32_t)msm_num_windows((int)p.c); p.nb = 1u << (p.c - 1); p.wpc = (p.W + p.cl - 1) / p.cl;
    return p;
}

#ifdef __CUDACC__
#include <cooperative_groups.h>
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

// The cluster MSM of the T terms recoded in rec (msm_recode with P.c, P.W), point of term t = load(t).  Every thread of every CTA of the
// cluster calls it; live (the same in every CTA) = the proof reached its MSM, else the call only joins the cluster barrier.  lists holds
// P.wpc * T term ids, wsum P.W window sums (CTA 0's are the ones read).  Returns, in warp 0 of CTA 0 of a live proof, whether the sum lies
// in the identity coset; false elsewhere.
template <class Load>
__device__ __forceinline__ bool single_msm_is_identity(cooperative_groups::cluster_group &cluster, const rp_single_plan &P, const msm_wide *rec, uint32_t T,
                                                       uint16_t *lists, ge_ext *wsum, bool live, Load load) {
    const uint32_t tid = threadIdx.x, rank = cluster.block_rank();
    if (live) {
        // thread (wl, b) owns bucket b of window rank * wpc + wl
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
                const uint32_t v = lst[e];
                const ge_niels q = load(v & 0x7fffu);
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
    if (!live || rank != 0 || tid >= 32) return false;
    return rp_single_horner_is_identity(wsum, (int)P.W, (int)P.c);
}
#endif
