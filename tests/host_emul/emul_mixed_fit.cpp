// TEST-ONLY host build of the fit of a mixed-geometry call to a reserved mix (rp_mixed.cuh: rp_mixed_mix, rp_mixed_fit,
// rp_mixed_slots): the CPU tier checks which calls fit, each class's slot base and live count, and the gather table's slot order
// against a Python model.
#include "../../bulletproofs_b200/csrc/rp_mixed.cuh"

extern "C" {

// Returns -2 when the mix is refused, -1 when the call's plan is refused, 0 when the call does not fit the mix, else 1 with base[C] and
// live[C] per mix class and, per admitted proof in gather order, src[j] (its input index) and slot[j].  n_admitted receives their number.
int emul_rp_mixed_fit(size_t n_classes, const uint32_t *mix_n, const uint32_t *mix_m, const uint32_t *capacity, size_t count, const uint8_t *proofs,
                      const uint64_t *proof_offsets, const uint32_t *n, const uint64_t *commit_offsets, size_t gens_cap, size_t gens_parties,
                      uint32_t *base, uint32_t *live, uint32_t *src, uint32_t *slot, size_t *n_admitted) {
    rp_mixed_plan X, P;
    if (rp_mixed_mix(n_classes, mix_n, mix_m, capacity, gens_cap, gens_parties, X)) return -2;
    if (rp_mixed_make_plan(count, proofs, proof_offsets, n, commit_offsets, gens_cap, gens_parties, P)) return -1;
    std::vector<uint32_t> lv;
    if (!rp_mixed_fit(P, X, lv)) return 0;
    for (size_t c = 0; c < X.cls.size(); c++) { base[c] = X.cls[c].first; live[c] = lv[c]; }
    const std::vector<std::pair<uint32_t, uint32_t>> s = rp_mixed_slots(P, X);
    for (size_t j = 0; j < s.size(); j++) { src[j] = s[j].first; slot[j] = s[j].second; }
    *n_admitted = s.size();
    return 1;
}

}
