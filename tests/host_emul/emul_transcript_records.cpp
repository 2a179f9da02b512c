// TEST-ONLY host build of k_rp_transcript's per-proof state load (rp_transcript_proof): the caller state of proof p at tstates + p * tstride,
// one state for every proof at stride 0, one checked record per proof otherwise.  Linked into libemul.so with emul.cpp.
#include <vector>
#include "../../bulletproofs_b200/csrc/rp.cuh"

extern "C" {

// Replays proof p of a launch whose states are at tstates with stride tstride; raw receives (6 + k) rows of 64 bytes.  Returns the verdict.
int emul_rp_transcript_proof(const uint8_t *proof, uint32_t k, const uint8_t *V, uint32_t n, uint32_t m, const uint8_t *tstates, uint64_t tstride, uint32_t p,
                             const uint8_t *seed, uint8_t *raw) {
    const std::vector<rp_tr_step> prog = rp_tr_program(n, m, k);
    return (int)rp_transcript_proof(raw, proof, k, V, tstates, tstride, p, seed, prog.data(), (uint32_t)prog.size());
}

}
