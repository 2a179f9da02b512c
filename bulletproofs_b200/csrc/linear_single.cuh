// Fused LinearProof verifier for small calls (bp_linear_verify_batch and bp_linear_verify_mixed route to it, lin_single_routed): one
// thread-block cluster per proof, one launch per call.
//
// The pipeline (linear_kernels.cuh) spreads a call over ~15 dependent launches and replays every transcript byte by byte in one GPU
// thread.  Here the host replays each transcript (lin_transcript_raw, the same function the device replay runs) while the proofs are on
// their way to the device, and uploads the k + 2 challenge rows; then a cluster of P.cl CTAs checks its proof's own equation (rho = 1,
// linear.cuh), so the verdict is exact and there is no combined check and no reject path:
//   1. front end, in every CTA of the cluster: the block decodes C, S, L_j and R_j (2 + 2k points, ge_decode) into shared memory and
//      reduces the round challenges; thread 0 builds the head (lin_head_init, weighted = false); the block fills the s tables
//      (lin_tab_entry) and reduces b0 = <b, s>;
//   2. the n + 2 + 2 + 2k scalars in the batch verifier's term order [B: r | F: a b0 | G_i: a s_i | C, S, L.., R..: lin_dyn_scalar],
//      recoded into signed c-bit digits (msm_recode);
//   3. the cluster MSM and its identity-coset verdict (single_msm.cuh): B, F and G_i from the set's resident points (slots 0, 1, 2 + i),
//      the proof's own points from shared memory.
// Every cluster reads its own n and k from its descriptor, so one launch serves proofs of different lengths; the launch's plan and shared
// memory are those of its longest proof.  The host part is shared with the host tests (tests/host_emul/emul_linear_single.cpp).
#pragma once
#include "linear.cuh"
#include "single_msm.cuh"

#define LIN_SINGLE_MAX_COUNT 64         // clusters of one launch (verdict staging)
// the largest k whose layout fits the dynamic shared memory one CTA may hold (lin_single_layout: 205 KB at k = 12, 399 KB at k = 13)
#define LIN_SINGLE_MAX_K 12
#define LIN_SINGLE_SMEM_LIMIT (227u * 1024u - 4096u)      // 227 KB per block on sm_90, less room for the kernel's static shared memory
#define LIN_SINGLE_ALIGN 32             // every proof, C and b of the input block starts at a multiple of this

// One proof of a fused call: its n = 2^k, the host replay's status (BP_PROOF_OK: the device decides), and the byte offsets of its proof,
// C, b and k + 2 challenge rows (x_0 .. x_{k-1}, x*, rho) in the call's device input block
struct lin_single_desc {
    uint32_t n, k, status, pad_;
    uint64_t proof, C, b, raw;
};

// MSM terms of one proof: B, F, G_0 .. G_{n-1}, C, S, L.., R..
BP_HD uint32_t lin_single_terms(uint32_t k) { return (1u << k) + 2 + lin_dyn_terms(k); }
// byte offsets of the dynamic shared memory of one CTA for a proof of k rounds under plan p
struct lin_single_smem { uint32_t wsum, niels, tabs, rec, lists, total; };
BP_HD lin_single_smem lin_single_layout(uint32_t k, const rp_single_plan &p) {
    const uint32_t T = lin_single_terms(k);
    lin_single_smem s; uint32_t o = 0;
    s.wsum = o; o += p.W * 128;                      // ge_ext window sums (CTA 0's are the ones read)
    s.niels = o; o += lin_dyn_terms(k) * 96;         // the proof's points, ge_niels
    s.tabs = o; o += lin_tab_size(k) * 32;           // s tables: slo then shi (linear.cuh)
    s.rec = o; o += T * 36;                          // msm_wide recoding of every term
    s.lists = o; o += p.wpc * T * 2;                 // per window of the CTA: term ids of its buckets, bucket after bucket
    s.total = (o + 15) & ~15u;
    return s;
}
// the plan of a launch whose longest proof has k rounds; every shorter proof of the launch fits its layout
BP_HD rp_single_plan lin_single_plan(uint32_t kmax) { return rp_single_plan_of(lin_single_terms(kmax)); }

// Routing of bp_linear_verify_batch and bp_linear_verify_mixed: calls of at most LIN_ROUTE_MAX_COUNT admitted proofs, none longer than
// LIN_ROUTE_MAX_N, run the fused launch; every other call runs the pipeline.  Crossover measured on one H100 80GB HBM3 at a 700 W limit
// (benchmarks/linear_single.py, README.md "Results"), median wall time of a blocking call: at count 1 the fused launch wins at every n
// measured (n = 64: 866 us against 1781; n = 1024: 2.51 ms against 13.0); at n = 64 it wins up to 32 proofs (1.97 ms against 2.21) and
// at n = 1024 up to 16 (7.77 ms against 16.8) and loses at 32 (22.2 ms against 17.9).  Counts between 16 and 32 were not measured at
// n = 1024, so the rule stops at 16.
#define LIN_ROUTE_MAX_COUNT 16
#define LIN_ROUTE_MAX_N 1024
BP_HD bool lin_single_routed(size_t count, size_t nmax) { return count >= 1 && count <= LIN_ROUTE_MAX_COUNT && nmax <= LIN_ROUTE_MAX_N; }

#ifdef __CUDACC__
#include "linear_kernels.cuh"
// One CTA per SM is all a cluster launch of a few proofs fills, so the launch bounds ask for one.  One cluster per proof p = blockIdx.x /
// P.cl; in = the call's input block, desc = its descriptors, pts = the set's resident points [B, F, G_0 ..], verdict[p] = the proof's
// ProofError code.  heads[blockIdx.x] is the CTA's head, in global memory as the pipeline's are: lin_head_init then writes through a
// global pointer from every caller, and the pipeline's table kernels keep their code.
#define LIN_SINGLE_THREADS 256
__global__ void __launch_bounds__(LIN_SINGLE_THREADS, 1) k_lin_single(rp_single_plan P, const lin_single_desc *__restrict__ desc, const uint8_t *__restrict__ in,
                                                                   const ge_niels *__restrict__ pts, lin_head *__restrict__ heads, uint32_t *__restrict__ verdict) {
    namespace cg = cooperative_groups;
    cg::cluster_group cluster = cg::this_cluster();
    extern __shared__ __align__(128) uint8_t smem[];
    __shared__ sc s_red[LIN_SINGLE_THREADS / 32];
    __shared__ uint32_t s_bad;
    sc *xsh = lin_xsh;
    const uint32_t tid = threadIdx.x, p = blockIdx.x / P.cl;
    const lin_single_desc d = desc[p];
    lin_head &head = heads[blockIdx.x];
    const uint32_t n = d.n, k = d.k, D = lin_dyn_terms(k), T = n + 2 + D;
    const lin_single_smem L = lin_single_layout(k, P);
    const uint8_t *proof = in + d.proof, *raw = in + d.raw;
    ge_ext *wsum = reinterpret_cast<ge_ext *>(smem + L.wsum);
    ge_niels *niels = reinterpret_cast<ge_niels *>(smem + L.niels);
    sc *tabs = reinterpret_cast<sc *>(smem + L.tabs);
    msm_wide *rec = reinterpret_cast<msm_wide *>(smem + L.rec);
    uint16_t *lists = reinterpret_cast<uint16_t *>(smem + L.lists);

    // 1. front end: points and challenges, then the head and the tables
    const bool replayed = d.status == BP_PROOF_OK;
    if (tid == 0) s_bad = 0u;
    __syncthreads();
    if (replayed) {
        for (uint32_t j = tid; j < k; j += blockDim.x) xsh[j] = rp_wide(raw + 64 * j);
        for (uint32_t i = tid; i < D; i += blockDim.x) {
            const uint8_t *src = i == 0 ? in + d.C : i == 1 ? proof + 64 * k : i < 2 + k ? proof + 64 * (i - 2) : proof + 64 * (i - 2 - k) + 32;
            uint8_t s[32]; ld32(s, src);
            fe x, y; const bool ok = ge_decode(x, y, s);
            st_niels(niels + i, ok ? ge_to_niels_affine(x, y) : ge_niels_identity());
            if (!ok) atomicOr(&s_bad, 1u);
        }
    }
    __syncthreads();
    if (replayed) {
        if (tid == 0) lin_head_init(head, xsh, k, raw + 64 * k, raw + 64 * (k + 1), proof, false);
        for (uint32_t e = tid; e < lin_tab_size(k); e += blockDim.x) tabs[e] = lin_tab_entry(xsh, k, e);
    }
    // every CTA of the cluster has started (its shared memory may be written) once this returns
    cluster.sync();
    const bool live = replayed && s_bad == 0u && head.status == BP_PROOF_OK;
    if (live) {
        // 2. scalars, recoded: G_i and this thread's share of b0 = <b, s>, then the block's b0, B, F and the dynamic terms
        const uint32_t kl = rp_kl(k), TL = 1u << kl;
        const uint8_t *b = in + d.b;
        sc part = sc_zero();
        for (uint32_t i = tid; i < n; i += blockDim.x) {
            const sc s = sc_mont_mul(tabs[TL + (i >> kl)], tabs[i & (TL - 1)]);
            uint8_t bb[32]; ld32(bb, b + 32 * i);
            part = sc_add(part, sc_mont_mul(sc_load(bb), s));
            rec[2 + i] = msm_recode(sc_from_mont(sc_mm(head.wa, s)).v, (int)P.c, (int)P.W);
        }
        for (int o = 16; o >= 1; o >>= 1) {
            sc v; for (int w = 0; w < 8; w++) v.v[w] = __shfl_down_sync(0xffffffffu, part.v[w], o);
            part = sc_add(part, v);
        }
        if ((tid & 31u) == 0) s_red[tid >> 5] = part;
        for (uint32_t t = tid; t < D; t += blockDim.x) rec[n + 2 + t] = msm_recode(lin_dyn_scalar(head, t, k).v, (int)P.c, (int)P.W);
        __syncthreads();
        if (tid == 0) {
            sc b0 = sc_zero();
            for (uint32_t w = 0; w < blockDim.x / 32; w++) b0 = sc_add(b0, s_red[w]);
            sc sB, sF; lin_static_bf(head, proof, k, b0, sB, sF);
            rec[0] = msm_recode(sB.v, (int)P.c, (int)P.W); rec[1] = msm_recode(sF.v, (int)P.c, (int)P.W);
        }
        __syncthreads();
    }
    // 3. the MSM (single_msm.cuh)
    const bool ident = single_msm_is_identity(cluster, P, rec, T, lists, wsum, live, [&](uint32_t t) {
        return t < n + 2 ? ldg_niels(pts + t) : niels[t - n - 2];
    });
    if (cluster.block_rank() != 0 || tid != 0) return;
    verdict[p] = !replayed ? d.status : !live ? (uint32_t)BP_PROOF_VERIFICATION_ERROR : ident ? (uint32_t)BP_PROOF_OK : (uint32_t)BP_PROOF_VERIFICATION_ERROR;
}
#endif
