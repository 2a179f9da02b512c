// TEST-ONLY host build of the device planner of a mixed call on device inputs (rp_mixed_device.cuh): the per-proof and per-block steps
// of k_mix_admit, k_mix_scan and k_mix_place, run block by block of RP_MIX_BLOCK proofs, beside the host planner (rp_mixed_make_plan,
// rp_mixed_fit, rp_mixed_slots) on the same call.
#include <algorithm>
#include "../../bulletproofs_b200/csrc/rp_mixed_device.cuh"

extern "C" {

// The device planner: codes[i] (parameter code), slot[i] (RP_MIX_NO_SLOT when rejected or unplaced) and live[C].  The offset and n
// arrays are byte buffers of any alignment, as on the device.  Returns -2 when the mix is refused, else 0.
int emul_rp_mixed_place(size_t n_classes, const uint32_t *mix_n, const uint32_t *mix_m, const uint32_t *capacity, size_t count, const uint8_t *proofs,
                        uint64_t proof_bytes, const uint8_t *poff, const uint8_t *n, uint64_t n_commit, const uint8_t *coff, size_t gens_cap,
                        size_t gens_parties, uint32_t *codes, uint32_t *slot, uint32_t *live) {
    rp_mixed_plan X;
    if (rp_mixed_mix(n_classes, mix_n, mix_m, capacity, gens_cap, gens_parties, X)) return -2;
    const rp_mix_classes M = rp_mix_classes_of(X, gens_cap, gens_parties);
    const size_t nb = (count + RP_MIX_BLOCK - 1) / RP_MIX_BLOCK;
    std::vector<uint32_t> cls(count), rank(count), hist(nb * M.C, 0);
    for (size_t b = 0; b < nb; b++) {                     // k_mix_admit
        const size_t i0 = b * RP_MIX_BLOCK, lanes = std::min<size_t>(RP_MIX_BLOCK, count - i0);
        uint32_t wcnt[RP_MIX_WARPS][RP_MIXED_MAX_CLASSES] = {};
        std::vector<uint32_t> wrank(lanes);
        for (uint32_t t = 0; t < lanes; t++) {
            const uint32_t word = rp_mix_admit(M, proofs, proof_bytes, poff, n, n_commit, coff, i0 + t);
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
    for (uint32_t c = 0; c < M.C; c++) {                  // k_mix_scan
        uint32_t run = 0;
        for (size_t b = 0; b < nb; b++) { const uint32_t v = hist[b * M.C + c]; hist[b * M.C + c] = run; run += v; }
        live[c] = std::min(run, M.cap[c]);
    }
    for (size_t i = 0; i < count; i++)                    // k_mix_place
        slot[i] = cls[i] == RP_MIX_NO_CLASS ? RP_MIX_NO_SLOT : rp_mix_slot(M, cls[i], hist[(i / RP_MIX_BLOCK) * M.C + cls[i]] + rank[i]);
    return 0;
}

// The host planner on the same call (offsets starting at 0, u64 arrays): codes[i], and when the call fits the mix live[C] and the
// (input, slot) pair of every admitted proof (n_placed of them).  Returns -2 / -1 when the mix / the call is refused, 0 when the call
// does not fit, else 1.
int emul_rp_mixed_host_place(size_t n_classes, const uint32_t *mix_n, const uint32_t *mix_m, const uint32_t *capacity, size_t count, const uint8_t *proofs,
                             const uint64_t *poff, const uint32_t *n, const uint64_t *coff, size_t gens_cap, size_t gens_parties, uint32_t *codes,
                             uint32_t *live, uint32_t *src, uint32_t *slot, size_t *n_placed) {
    rp_mixed_plan X, P;
    if (rp_mixed_mix(n_classes, mix_n, mix_m, capacity, gens_cap, gens_parties, X)) return -2;
    if (rp_mixed_make_plan(count, proofs, poff, n, coff, gens_cap, gens_parties, P)) return -1;
    for (size_t i = 0; i < count; i++) codes[i] = P.codes[i];
    std::vector<uint32_t> lv;
    if (!rp_mixed_fit(P, X, lv)) return 0;
    std::copy(lv.begin(), lv.end(), live);
    const std::vector<std::pair<uint32_t, uint32_t>> s = rp_mixed_slots(P, X);
    for (size_t j = 0; j < s.size(); j++) { src[j] = s[j].first; slot[j] = s[j].second; }
    *n_placed = s.size();
    return 1;
}

}
