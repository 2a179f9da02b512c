// Device planning of a mixed-length LinearProof call whose inputs are device pointers (bp_linear_verify_mixed_device): the per-proof and
// per-block steps that place each proof in the reserved mix (linm_mix) without a host round trip.  The kernels below call these
// functions; the host-emulation tests run them block by block against the host plan (linm_make_plan).
//
// Placement, as for the range-proof mix (rp_mixed_device.cuh, whose generic helpers it uses): proof i is admitted when its offsets are in
// bounds and linm_param_verdict passes it; it then belongs to the mix class of its n, if the mix has one.  Within a class, proofs take
// the class's slots in input order up to its capacity: proof i's rank is the number of admitted proofs of its class before it (earlier
// blocks: an exclusive scan of per-block class counts; its own block: its rank among the same-class lanes of its warp plus the same-class
// lanes of the block's earlier warps).  A proof of no class, or ranked at or past the capacity, is unplaced.
#pragma once
#include "linear_mixed.cuh"
#include "rp_mixed_device.cuh"

static_assert(LINM_MAX_CLASSES <= RP_MIXED_MAX_CLASSES, "the per-warp class counts of rp_mix_rank_in_block");

// The reserved mix as the planner kernels see it (a kernel parameter): per class its n, capacity and first slot, and the set's size
struct linm_mix_classes {
    uint32_t C, set_n;
    uint32_t n[LINM_MAX_CLASSES], cap[LINM_MAX_CLASSES], first[LINM_MAX_CLASSES];
};
inline linm_mix_classes linm_mix_classes_of(const linm_plan &X, size_t set_n) {
    linm_mix_classes M{};
    M.C = (uint32_t)X.cls.size(); M.set_n = (uint32_t)set_n;
    for (uint32_t c = 0; c < M.C; c++) { M.n[c] = X.cls[c].n; M.cap[c] = X.cls[c].count; M.first[c] = X.cls[c].first; }
    return M;
}

// Proof i's bytes start at *po and its b at scalar *bo, or false when its offsets decrease or reach past proof_bytes / n_b (then none of
// its bytes may be read).  *len: its proof bytes, *n: its b scalars.
BP_HD bool linm_mix_bounds(const uint8_t *poff, const uint8_t *boff, uint64_t proof_bytes, uint64_t n_b, size_t i, uint64_t *po, uint64_t *len, uint64_t *bo,
                           uint64_t *n) {
    const uint64_t p0 = rp_ld_u64(poff + 8 * i), p1 = rp_ld_u64(poff + 8 * i + 8), b0 = rp_ld_u64(boff + 8 * i), b1 = rp_ld_u64(boff + 8 * i + 8);
    if (p1 < p0 || b1 < b0 || p1 > proof_bytes || b1 > n_b) return false;
    *po = p0; *len = p1 - p0; *bo = b0; *n = b1 - b0;
    return true;
}
// Admission of proof i as one word, code | class << 8 (the word of rp_mix_admit, so k_mix_verdicts reads it): its parameter code,
// linm_param_verdict's, with FormatError for offsets linm_mix_bounds refuses; its class of M, or RP_MIX_NO_CLASS when it is rejected or
// M lacks its n.
BP_HD uint32_t linm_mix_admit(const linm_mix_classes &M, const uint8_t *proofs, uint64_t proof_bytes, const uint8_t *poff, const uint8_t *boff, uint64_t n_b,
                              size_t i) {
    uint64_t po, len, bo, n;
    if (!linm_mix_bounds(poff, boff, proof_bytes, n_b, i, &po, &len, &bo, &n)) return BP_PROOF_FORMAT_ERROR | RP_MIX_NO_CLASS << 8;
    uint32_t k = 0;
    const uint8_t pv = linm_param_verdict(proofs + po, (size_t)len, (size_t)n, M.set_n, &k);
    if (pv != BP_PROOF_OK) return pv | RP_MIX_NO_CLASS << 8;
    uint32_t cls = RP_MIX_NO_CLASS;
    for (uint32_t c = 0; c < M.C; c++)
        if (M.n[c] == n) { cls = c; break; }
    return BP_PROOF_OK | cls << 8;
}
// The slot of rank `rank` in class c, or RP_MIX_NO_SLOT past its capacity
BP_HD uint32_t linm_mix_slot(const linm_mix_classes &M, uint32_t c, uint32_t rank) { return rank < M.cap[c] ? M.first[c] + rank : RP_MIX_NO_SLOT; }

#ifdef __CUDACC__
// Step 1, one thread per proof: code_cls[i] = its parameter code | its class << 8, rank[i] = its rank among the proofs of its class earlier
// in its block, hist[block][c] = the block's class-c proofs
__global__ void __launch_bounds__(RP_MIX_BLOCK) k_linm_admit(linm_mix_classes M, uint32_t count, const uint8_t *__restrict__ proofs, uint64_t proof_bytes,
                                                            const uint8_t *__restrict__ poff, const uint8_t *__restrict__ boff, uint64_t n_b,
                                                            uint32_t *__restrict__ code_cls, uint32_t *__restrict__ rank, uint32_t *__restrict__ hist) {
    __shared__ uint32_t s_wcnt[RP_MIX_WARPS][RP_MIXED_MAX_CLASSES];
    const uint32_t t = threadIdx.x, lane = t % 32, warp = t / 32, i = blockIdx.x * RP_MIX_BLOCK + t;
    for (uint32_t j = t; j < RP_MIX_WARPS * RP_MIXED_MAX_CLASSES; j += RP_MIX_BLOCK) s_wcnt[j / RP_MIXED_MAX_CLASSES][j % RP_MIXED_MAX_CLASSES] = 0;
    const uint32_t word = i < count ? linm_mix_admit(M, proofs, proof_bytes, poff, boff, n_b, i) : (uint32_t)RP_MIX_NO_CLASS << 8;
    if (i < count) code_cls[i] = word;
    const uint32_t cls = rp_mix_class(word);
    const uint32_t same = __match_any_sync(~0u, cls), wrank = __popc(same & ((1u << lane) - 1u));
    __syncthreads();
    if (cls != RP_MIX_NO_CLASS && wrank == 0) s_wcnt[warp][cls] = __popc(same);
    __syncthreads();
    if (cls != RP_MIX_NO_CLASS) rank[i] = rp_mix_rank_in_block(s_wcnt, warp, cls, wrank);
    if (t < M.C) hist[(size_t)blockIdx.x * M.C + t] = rp_mix_block_count(s_wcnt, t);
}
// Step 2, one block, warp c for class c: hist[b][c] becomes the class-c proofs of the blocks before b, and class c's live count,
// min(its proofs, its capacity), goes into the device class table (the front end's) and the class's parameters (its reject loop's)
__global__ void k_linm_scan(linm_mix_classes M, uint32_t nb, uint32_t *__restrict__ hist, linm_class *__restrict__ cls, lin_params *__restrict__ cpar) {
    const uint32_t c = threadIdx.x / 32, lane = threadIdx.x % 32;
    if (c >= M.C) return;
    uint32_t run = 0;
    for (uint32_t b0 = 0; b0 < nb; b0 += 32) {
        const uint32_t b = b0 + lane, v = b < nb ? hist[(size_t)b * M.C + c] : 0u;
        uint32_t x = v;
        for (uint32_t d = 1; d < 32; d *= 2) { const uint32_t y = __shfl_up_sync(~0u, x, d); if (lane >= d) x += y; }
        if (b < nb) hist[(size_t)b * M.C + c] = run + x - v;
        run += __shfl_sync(~0u, x, 31);
    }
    if (lane == 0) { const uint32_t live = min(run, M.cap[c]); cls[c].live = live; cpar[c].live = live; }
}
// Step 3, one thread per proof: slot[i] = proof i's slot (in place of its rank; RP_MIX_NO_SLOT when it has none) and, when placed, its
// gather entry at that slot.  Slots this call leaves inert keep stale entries, which k_linm_gather skips.
__global__ void __launch_bounds__(RP_MIX_BLOCK) k_linm_place(linm_mix_classes M, uint32_t count, const uint8_t *__restrict__ poff, const uint8_t *__restrict__ boff,
                                                            const uint32_t *__restrict__ code_cls, uint32_t *__restrict__ slot, const uint32_t *__restrict__ hist,
                                                            linm_gather *__restrict__ gather) {
    const uint32_t i = blockIdx.x * RP_MIX_BLOCK + threadIdx.x;
    if (i >= count) return;
    const uint32_t cls = rp_mix_class(code_cls[i]);
    uint32_t s = RP_MIX_NO_SLOT;
    if (cls != RP_MIX_NO_CLASS) {
        s = linm_mix_slot(M, cls, hist[(size_t)blockIdx.x * M.C + cls] + slot[i]);
        if (s != RP_MIX_NO_SLOT) {
            uint64_t po, len, bo, n;
            linm_mix_bounds(poff, boff, ~0ull, ~0ull, i, &po, &len, &bo, &n);        // admitted: in bounds
            gather[s] = linm_gather{po, bo, i, 0};
        }
    }
    slot[i] = s;
}
#endif
