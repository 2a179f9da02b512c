// TEST-ONLY host build of the LinearProof reserved device path's pass arithmetic (linear.cuh: lin_x_slice, lin_x_clamp, lin_x_iters,
// lin_x_slice_live) and of the record check of the shared transcript replay, lin_transcript_raw, on a caller-owned state buffer so that the
// CPU tier can see any byte written past the 200-byte state.
#include "../../bulletproofs_b200/csrc/linear.cuh"

extern "C" {

uint32_t emul_lin_x_slice(uint32_t capacity, uint32_t n, uint32_t k) { return lin_x_slice(capacity, n, k); }
uint32_t emul_lin_x_clamp(uint32_t live, uint32_t capacity) { return lin_x_clamp(live, capacity); }
uint32_t emul_lin_x_iters(uint32_t live, uint32_t P, int failed) { return lin_x_iters(live, P, failed != 0); }
uint32_t emul_lin_x_slice_live(uint32_t it, uint32_t P, uint32_t live) { return lin_x_slice_live(it, P, live); }

// lin_transcript_raw with the caller's state scratch (4-byte aligned, 200 bytes and whatever guard the caller puts after them)
uint32_t emul_lin_transcript_state(const uint8_t *proof, uint32_t k, uint32_t n, const uint8_t *C, const uint8_t *b, const uint8_t *enc,
                                   const uint8_t *tstate, const uint8_t *seed, uint8_t *raw, uint8_t *state) {
    return lin_transcript_raw(reinterpret_cast<uint8_t (*)[64]>(raw), proof, k, n, C, b, enc, tstate, seed, state);
}

}
