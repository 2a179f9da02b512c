// TEST-ONLY host build of the pass arithmetic of the device reject path (rp.cuh: rp_x_slice, rp_x_unit_live, rp_x_listed, rp_x_clamp,
// rp_x_iters): the CPU tier checks the failing-proof list, P and the level-2 iteration bound against a Python model.
#include "../../bulletproofs_b200/csrc/rp.cuh"

extern "C" {

uint32_t emul_rp_x_slice(uint32_t np, uint32_t S, uint32_t D) { return rp_x_slice(np, S, D); }
uint32_t emul_rp_x_clamp(uint32_t n, uint32_t live) { return rp_x_clamp(n, live); }
uint32_t emul_rp_x_iters(uint32_t n, uint32_t P) { return rp_x_iters(n, P); }

// The list k_rp_xchunk_verdicts builds for a group of nbatch units of count proofs, proofs [0, live) live: chunk_fail[b nch + ch] = 1 when
// chunk ch of unit b failed (nch = ceil(count / RP_CHUNK)).  Proof p = b count + q in chunk order (the device appends chunks in any order).
// Returns the list length.
uint32_t emul_rp_x_list(uint32_t count, uint32_t nbatch, uint32_t live, const uint8_t *chunk_fail, uint32_t *out) {
    const uint32_t nch = (count + RP_CHUNK - 1) / RP_CHUNK;
    uint32_t n = 0;
    for (uint32_t b = 0; b < nbatch; b++) {
        const uint32_t ul = rp_x_unit_live(live, count, b);
        for (uint32_t ch = 0; ch < nch; ch++)
            for (uint32_t lane = 0; lane < RP_CHUNK; lane++) {
                const uint32_t q = ch * RP_CHUNK + lane;
                if (rp_x_listed(q, ul, chunk_fail[b * nch + ch] != 0)) out[n++] = b * count + q;
            }
    }
    return n;
}

}
