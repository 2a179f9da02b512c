// TEST-ONLY host build of the plan of a mixed-length LinearProof call (linear_mixed.cuh): the CPU tier checks the per-proof parameter codes,
// the classes, their arena offsets, the dynamic-term bases and the term count against a Python model.
#include "../../bulletproofs_b200/csrc/linear_mixed.cuh"

extern "C" {

#define EMUL_LINM_FIELDS 15
// one class as 15 words: n, k, first, count, proof_len, D, chunk0, tiles, proof_off, b_off, raw_off, tab_off, part_off, b0_off, dyn
static void emul_linm_class(const linm_class &K, uint64_t *out) {
    const uint64_t f[EMUL_LINM_FIELDS] = {K.n, K.k, K.first, K.count, K.proof_len, K.D, K.chunk0, K.tiles, K.proof_off, K.b_off, K.raw_off, K.tab_off,
                                          K.part_off, K.b0_off, K.dyn};
    for (int j = 0; j < EMUL_LINM_FIELDS; j++) out[j] = f[j];
}
// sums[10]: nmax, chunks, terms, dynamic points, proof bytes, b scalars, raw rows, table scalars, chunk-sum scalars, b0 scalars
static void emul_linm_sums(const linm_plan &P, uint64_t *sums) {
    const uint64_t f[10] = {P.nmax, P.chunks, P.terms, P.dyn_points, P.proof_bytes, P.b_scalars, P.raw_rows, P.tab_scalars, P.part_scalars, P.b0_scalars};
    for (int j = 0; j < 10; j++) sums[j] = f[j];
}

// Returns -1 when the call is refused, else the number of classes C.  codes[count]; order[admitted proofs]; cls[C * 15]; sums[10].
int emul_linm_plan(size_t count, const uint8_t *proofs, const uint64_t *proof_offsets, const uint64_t *b_offsets, size_t set_n, uint8_t *codes,
                   uint32_t *order, uint64_t *cls, uint64_t *sums) {
    linm_plan P;
    if (linm_make_plan(count, proofs, proof_offsets, b_offsets, set_n, P)) return -1;
    for (size_t i = 0; i < count; i++) codes[i] = P.codes[i];
    for (size_t j = 0; j < P.order.size(); j++) order[j] = P.order[j];
    for (size_t c = 0; c < P.cls.size(); c++) emul_linm_class(P.cls[c], cls + EMUL_LINM_FIELDS * c);
    emul_linm_sums(P, sums);
    return (int)P.cls.size();
}

// The layout of C classes of (n[c] = 2^k[c], count[c]) proofs alone, beyond what a call may hold: -1 when refused, else C
int emul_linm_layout(size_t C, const uint32_t *k, const uint32_t *count, uint64_t *cls, uint64_t *sums) {
    linm_plan P;
    for (size_t c = 0; c < C; c++) { linm_class K{}; K.k = k[c]; K.n = 1u << k[c]; K.count = count[c]; P.cls.push_back(K); }
    if (linm_layout(P)) return -1;
    for (size_t c = 0; c < C; c++) emul_linm_class(P.cls[c], cls + EMUL_LINM_FIELDS * c);
    emul_linm_sums(P, sums);
    return (int)C;
}

}
