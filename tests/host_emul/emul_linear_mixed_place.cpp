// TEST-ONLY host build of the device planner of a mixed-length LinearProof call on device inputs (linear_mixed_device.cuh): the per-proof
// and per-block steps of k_linm_admit, k_linm_scan and k_linm_place, run block by block of RP_MIX_BLOCK proofs, and the reserved mix
// (linm_mix) they place into.  The CPU tier runs them beside the host plan (linm_make_plan, emul_linear_mixed.cpp) on the same calls.
#include <algorithm>
#include "../../bulletproofs_b200/csrc/linear_mixed_device.cuh"

extern "C" {

// The mix of n_classes lengths: -1 when linm_mix refuses it, else C; first[C] (first slot of every class) and sums[2] = (slot total,
// combined-row terms)
int emul_linm_mix(size_t n_classes, const uint32_t *n, const uint32_t *capacity, size_t set_n, uint32_t *first, uint64_t *sums) {
    linm_plan X;
    if (linm_mix(n_classes, n, capacity, set_n, X)) return -1;
    for (size_t c = 0; c < X.cls.size(); c++) first[c] = X.cls[c].first;
    sums[0] = X.cls.back().first + X.cls.back().count; sums[1] = X.terms;
    return (int)X.cls.size();
}

// The device planner: codes[i] (parameter code), slot[i] (RP_MIX_NO_SLOT when rejected or unplaced), live[C] and, per slot of the mix,
// the gather entry a placed proof writes (gather[3 s ..]: proof byte offset, b scalar offset, input index; untouched for an empty slot).
// The offset arrays are byte buffers of any alignment, as on the device.  Returns -2 when the mix is refused, else 0.
int emul_linm_mixed_place(size_t n_classes, const uint32_t *mix_n, const uint32_t *capacity, size_t set_n, size_t count, const uint8_t *proofs,
                          uint64_t proof_bytes, const uint8_t *poff, const uint8_t *boff, uint64_t n_b, uint32_t *codes, uint32_t *slot, uint32_t *live,
                          uint64_t *gather) {
    linm_plan X;
    if (linm_mix(n_classes, mix_n, capacity, set_n, X)) return -2;
    const linm_mix_classes M = linm_mix_classes_of(X, set_n);
    const size_t nb = (count + RP_MIX_BLOCK - 1) / RP_MIX_BLOCK;
    std::vector<uint32_t> cls(count), rank(count), hist(nb * M.C, 0);
    for (size_t b = 0; b < nb; b++) {                     // k_linm_admit
        const size_t i0 = b * RP_MIX_BLOCK, lanes = std::min<size_t>(RP_MIX_BLOCK, count - i0);
        uint32_t wcnt[RP_MIX_WARPS][RP_MIXED_MAX_CLASSES] = {};
        std::vector<uint32_t> wrank(lanes);
        for (uint32_t t = 0; t < lanes; t++) {
            const uint32_t word = linm_mix_admit(M, proofs, proof_bytes, poff, boff, n_b, i0 + t);
            codes[i0 + t] = rp_mix_code(word);
            cls[i0 + t] = rp_mix_class(word);
        }
        for (uint32_t t = 0; t < lanes; t++) {            // __match_any_sync: the same-class lanes of t's warp before t
            const uint32_t c = cls[i0 + t];
            if (c == RP_MIX_NO_CLASS) continue;
            for (uint32_t j = t & ~31u; j < t; j++) wrank[t] += cls[i0 + j] == c ? 1u : 0u;
            wcnt[t / 32][c]++;
        }
        for (uint32_t t = 0; t < lanes; t++)
            if (cls[i0 + t] != RP_MIX_NO_CLASS) rank[i0 + t] = rp_mix_rank_in_block(wcnt, t / 32, cls[i0 + t], wrank[t]);
        for (uint32_t c = 0; c < M.C; c++) hist[b * M.C + c] = rp_mix_block_count(wcnt, c);
    }
    for (uint32_t c = 0; c < M.C; c++) {                  // k_linm_scan
        uint32_t run = 0;
        for (size_t b = 0; b < nb; b++) { const uint32_t v = hist[b * M.C + c]; hist[b * M.C + c] = run; run += v; }
        live[c] = std::min(run, M.cap[c]);
    }
    for (size_t i = 0; i < count; i++) {                  // k_linm_place
        slot[i] = cls[i] == RP_MIX_NO_CLASS ? RP_MIX_NO_SLOT : linm_mix_slot(M, cls[i], hist[(i / RP_MIX_BLOCK) * M.C + cls[i]] + rank[i]);
        if (slot[i] == RP_MIX_NO_SLOT) continue;
        uint64_t po, len, bo, n;
        linm_mix_bounds(poff, boff, ~0ull, ~0ull, i, &po, &len, &bo, &n);
        gather[3 * (size_t)slot[i]] = po; gather[3 * (size_t)slot[i] + 1] = bo; gather[3 * (size_t)slot[i] + 2] = i;
    }
    return 0;
}

}
