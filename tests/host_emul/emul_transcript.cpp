// TEST-ONLY host build of the range-proof transcript replay in both forms: the byte-wise STROBE (rp_transcript_raw) and the
// scheduled word-wise replay the device runs (rp_transcript_sched over rp_tr_program).  Linked into libemul.so with emul.cpp.
#include <cstring>
#include <vector>
#include "../../bulletproofs_b200/csrc/rp.cuh"

extern "C" {

// Replays one proof both ways.  raw_b / raw_s receive (6 + k) rows of 64 bytes each; returns the two verdicts as st_b | st_s << 8.
int emul_rp_transcript_both(const uint8_t *proof, uint32_t k, const uint8_t *V, uint32_t n, uint32_t m, const uint8_t *tstate, const uint8_t *seed,
                            uint8_t *raw_b, uint8_t *raw_s) {
    alignas(8) uint8_t st[200], ts[208];
    memcpy(ts, tstate, BP_TRANSCRIPT_BYTES);
    uint32_t sb = rp_transcript_raw(reinterpret_cast<uint8_t (*)[64]>(raw_b), proof, k, V, n, m, ts, seed, st);
    const std::vector<rp_tr_step> prog = rp_tr_program(n, m, k);
    uint32_t ss = rp_transcript_sched(raw_s, proof, k, V, ts, seed, prog.data(), (uint32_t)prog.size());
    return (int)(sb | (ss << 8));
}

}
