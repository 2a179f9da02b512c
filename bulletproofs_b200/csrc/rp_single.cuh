// Fused single-proof range-proof verifier: one thread-block cluster per proof, one launch per call.
//
// The launch-group pipeline (kernels.cuh, range-proof section) spreads a batch over ~15 dependent launches, each nearly empty when the
// batch holds one proof.  Here a cluster of P.cl CTAs verifies its proof alone, with the proof's own check (mod.rs:421-447) weighted
// by rho * lambda as on the pipeline (rp.cuh header), so the verdict is exact and there is no reject path:
//   1. front end, in every CTA of the cluster: lane 0 replays the transcript (rp_transcript_proof) while warps 1.. decode the proof's
//      D points (ge_decode); thread 0 then runs the head (rp_head_lean), whose tables stay in shared memory;
//   2. the S = 2 + 2N static scalars (k_rp_scalars_sum's algebra for a chunk of one proof) and the D dynamic ones, recoded into
//      signed c-bit digits (msm_recode), one thread per term;
//   3. the MSM of S + D terms and 4. its identity-coset verdict on CTA 0: the cluster MSM of single_msm.cuh, static points from the
//      generator table, the proof's own from shared memory.
// The front end is computed redundantly by every CTA of the cluster: it is latency, and the copies run on different SMs, so only the
// window sums cross between CTAs.
#pragma once
#include "kernels.cuh"
#include "single_msm.cuh"

#define RP_SINGLE_MIN_K 3               // n >= 8
#define RP_SINGLE_MAX_K 10              // kernel instances; the routing rule (bpmsm.cu) may use fewer
#define RP_SINGLE_MAX_COUNT 64          // clusters of one launch the host path accepts (verdict staging)
#define RP_SINGLE_HDR 256               // device input block: caller transcript state (208 B) | seed (32 B) | pad, then proofs, commitments

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
    }
    // 3. the MSM (single_msm.cuh)
    const bool ident = single_msm_is_identity(cluster, P, rec, T, lists, wsum, live, [&](uint32_t t) {
        return t < g.S ? ldg_niels(gens + rp_static_slot(g, t, gens_cap, gens_parties)) : niels[t - g.S];
    });
    // 4. the verdict
    if (rank != 0 || tid >= 32) return;
    if (!live) { if (tid == 0) verdict[p] = rp_eff_status(s_status, s_bad); return; }
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
