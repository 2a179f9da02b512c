// The element-wise operations behind the test hooks of include/bpmsm.h (bp_debug_fe_op, bp_debug_sc_op, bp_debug_ge_op).  One
// definition serves both builds: bpmsm.cu runs it on the device (the PTX branches of fe.cuh / sc.cuh), tests/host_emul runs it on
// the host (the portable branches), so the two tiers of the suite check the same operation on the same bytes.  No product path
// calls anything here.
#pragma once
#include "ge.cuh"
#include "sc.cuh"
#include "rp.cuh"

#define BP_DEBUG_FE_OPS 11
#define BP_DEBUG_SC_OPS 9
#define BP_DEBUG_GE_OPS 4

// op 0 add, 1 sub, 2 mul, 3 invert(a), 4 a^((p-5)/8), 5 neg(a), 6 a^2, 7 (a+b)(a-b), 8 dbl(a): canonical bytes out.
// op 9: out[0] = fe_is_zero(a), out[1] = fe_is_negative(a), out[2] = fe_eq(a, b), the other bytes zero.
// op 10: fe_sqrt_ratio_i(a, b): the root r (canonical) with the was_square flag in bit 255.
BP_HD void debug_fe_op(int op, const uint8_t a[32], const uint8_t b[32], uint8_t out[32]) {
    fe x = fe_frombytes_raw(a), y = fe_frombytes_raw(b), r;
    bool flag = false;
    switch (op) {
        case 0: r = fe_add(x, y); break;
        case 1: r = fe_sub(x, y); break;
        case 2: r = fe_mul(x, y); break;
        case 3: r = fe_invert(x); break;
        case 4: r = fe_pow22523(x); break;
        case 5: r = fe_neg(x); break;
        case 6: r = fe_sq(x); break;
        case 7: r = fe_mul(fe_add(x, y), fe_sub(x, y)); break;      // chained, unreduced intermediates
        case 8: r = fe_dbl(x); break;
        case 9:
            for (int i = 0; i < 32; i++) out[i] = 0;
            out[0] = fe_is_zero(x); out[1] = fe_is_negative(x); out[2] = fe_eq(x, y);
            return;
        default: flag = fe_sqrt_ratio_i(r, x, y);
    }
    fe_tobytes(out, r);
    out[31] |= (uint8_t)(flag ? 0x80 : 0);
}

// ops 0-7 of bp_debug_sc_op on one pair; raw limbs in and out (a || b is the 64-byte input of ops 5 and 6)
BP_HD void debug_sc_op(int op, const uint8_t a[32], const uint8_t b[32], uint8_t out[32]) {
    uint8_t wide[64];
    for (int i = 0; i < 32; i++) { wide[i] = a[i]; wide[32 + i] = b[i]; }
    sc x = sc_load(a), y = sc_load(b), r;
    switch (op) {
        case 0: r = sc_mont_mul(x, y); break;
        case 1: r = sc_from_mont(sc_mont_mul(sc_to_mont(x), sc_to_mont(y))); break;
        case 2: r = sc_add(x, y); break;
        case 3: r = sc_sub(x, y); break;
        case 4: r = sc_neg(x); break;
        case 5: r = sc_mont_from_wide(wide); break;
        case 6: r = rp_wide(wide); break;
        default: r = sc_mont_invert(x);
    }
    sc_store(out, r);
}
// op 8 (sum32): (sum_{j<32} a_j*b_j)/R mod l through one lazy-reduction accumulator; a and b are 32 consecutive 32-byte values
BP_HD void debug_sc_sum32(const uint8_t *a, const uint8_t *b, uint8_t out[32]) {
    sc_wide acc = sc_wide_zero();
    for (int j = 0; j < 32; j++) sc_wide_mac(acc, sc_load(a + 32 * j), sc_load(b + 32 * j));
    sc_store(out, sc_wide_redc(acc));
}

// op 0 ge_add(a, b), 1 ge_madd(a, niels(b)), 2 ge_msub(a, niels(b)), 3 ge_dbl(a).  a and b are raw X|Y|Z|T limbs (4 x 32 bytes),
// loaded without reduction; for ops 1 and 2, b's first two coordinates are the affine (x, y) of the Niels point.  Canonical X|Y|Z|T out.
BP_HD void debug_ge_op(int op, const uint8_t a[128], const uint8_t b[128], uint8_t out[128]) {
    ge_ext p, q, r;
    p.X = fe_frombytes_raw(a); p.Y = fe_frombytes_raw(a + 32); p.Z = fe_frombytes_raw(a + 64); p.T = fe_frombytes_raw(a + 96);
    q.X = fe_frombytes_raw(b); q.Y = fe_frombytes_raw(b + 32); q.Z = fe_frombytes_raw(b + 64); q.T = fe_frombytes_raw(b + 96);
    switch (op) {
        case 0: r = ge_add(p, q); break;
        case 1: r = ge_madd(p, ge_to_niels_affine(q.X, q.Y)); break;
        case 2: r = ge_msub(p, ge_to_niels_affine(q.X, q.Y)); break;
        default: r = ge_dbl(p);
    }
    fe_tobytes(out, r.X); fe_tobytes(out + 32, r.Y); fe_tobytes(out + 64, r.Z); fe_tobytes(out + 96, r.T);
}
