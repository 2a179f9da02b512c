// TEST-ONLY: the test hooks of include/bpmsm.h (bp_debug_fe_op, bp_debug_sc_op, bp_debug_ge_op) element for element on the host,
// through the same debug_ops.cuh the device hooks run, so that the CPU tier checks the portable branches on the operands the GPU
// tier feeds the PTX branches.  n pairs in, the hook's output bytes out.
#include "../../bulletproofs_b200/csrc/debug_ops.cuh"

extern "C" {

void emul_debug_fe_op(int op, const uint8_t *a, const uint8_t *b, uint64_t n, uint8_t *out) {
    for (uint64_t i = 0; i < n; i++) debug_fe_op(op, a + 32 * i, b + 32 * i, out + 32 * i);
}
void emul_debug_sc_op(int op, const uint8_t *a, const uint8_t *b, uint64_t n, uint8_t *out) {
    if (op == 8) { for (uint64_t i = 0; i < n / 32; i++) debug_sc_sum32(a + 1024 * i, b + 1024 * i, out + 32 * i); return; }
    for (uint64_t i = 0; i < n; i++) debug_sc_op(op, a + 32 * i, b + 32 * i, out + 32 * i);
}
void emul_debug_ge_op(int op, const uint8_t *a, const uint8_t *b, uint64_t n, uint8_t *out) {
    for (uint64_t i = 0; i < n; i++) debug_ge_op(op, a + 128 * i, b + 128 * i, out + 128 * i);
}
}
