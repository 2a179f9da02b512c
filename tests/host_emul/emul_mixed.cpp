// TEST-ONLY host build of the plan of a mixed-geometry range-proof call (rp_mixed.cuh): the CPU tier checks the classes, segments,
// global dynamic indices and per-proof parameter codes against a Python model.
#include "../../bulletproofs_b200/csrc/rp_mixed.cuh"

extern "C" {

#define EMUL_MIXED_FIELDS 12
// Returns -1 when the call is refused, else the number of classes C.  codes[count]; order[number of admitted proofs]; cls[C * 12]: per
// class n, m, k, S, D, count, first, seg, dyn, proof_off, commit_off, part_off; sums[4]: terms, dynamic points, admitted proofs, T of
// the first class (0 without one).
int emul_rp_mixed_plan(size_t count, const uint8_t *proofs, const uint64_t *proof_offsets, const uint32_t *n, const uint64_t *commit_offsets,
                       size_t gens_cap, size_t gens_parties, uint8_t *codes, uint32_t *order, uint64_t *cls, uint64_t *sums) {
    rp_mixed_plan P;
    if (rp_mixed_make_plan(count, proofs, proof_offsets, n, commit_offsets, gens_cap, gens_parties, P)) return -1;
    for (size_t i = 0; i < count; i++) codes[i] = P.codes[i];
    for (size_t j = 0; j < P.order.size(); j++) order[j] = P.order[j];
    for (size_t c = 0; c < P.cls.size(); c++) {
        const rp_mixed_class &K = P.cls[c];
        const uint64_t f[EMUL_MIXED_FIELDS] = {K.g.n, K.g.m, K.g.k, K.g.S, K.g.D, K.g.count, K.first, K.seg, K.dyn, K.proof_off, K.commit_off, K.part_off};
        for (int j = 0; j < EMUL_MIXED_FIELDS; j++) cls[EMUL_MIXED_FIELDS * c + j] = f[j];
    }
    sums[0] = P.terms; sums[1] = P.dyn_points; sums[2] = P.order.size(); sums[3] = P.cls.empty() ? 0 : P.cls[0].g.T;
    return (int)P.cls.size();
}

}
