// Scalars mod l = 2^252 + 27742317777372353535851937790883648493 for the device-side
// verification-scalar kernels (SURVEY.md §8(f) rank 1: verification_scalars and the g/h/delta
// assembly of src/range_proof/mod.rs:398-419,587-593 moved onto the GPU).
//
// Eight 32-bit limbs; products use Montgomery multiplication (R = 2^256, CIOS).  Kernels keep
// every scalar in Montgomery form and convert only at the byte boundaries, so the 32-byte
// little-endian canonical encodings match curve25519_dalek::scalar::Scalar bit for bit.
#pragma once
#include "fe.cuh"

struct sc { uint32_t v[8]; };

#define SC_L_LIMBS {0x5cf5d3edu, 0x5812631au, 0xa2f79cd6u, 0x14def9deu, 0x00000000u, 0x00000000u, 0x00000000u, 0x10000000u}
#define SC_LFACTOR 0x12547e1bu     // -l^-1 mod 2^32
#define SC_LPRIME_LIMBS {0x12547e1bu, 0xd2b51da3u, 0xfdba84ffu, 0xb1a206f2u, 0xffa36beau, 0x14e75438u, 0x6fe91836u, 0x9db6c6f2u}   // -l^-1 mod 2^256
#define SC_R_LIMBS {0x8d98951du, 0xd6ec3174u, 0x737dcf70u, 0xc6ef5bf4u, 0xfffffffeu, 0xffffffffu, 0xffffffffu, 0x0fffffffu}
#define SC_RR_LIMBS {0x449c0f01u, 0xa40611e3u, 0x68859347u, 0xd00e1ba7u, 0x17f5be65u, 0xceec73d2u, 0x7c309a3du, 0x0399411bu}
#define SC_RRR_LIMBS {0x7b83a2dbu, 0x2a9e4968u, 0xaef7f3ecu, 0x278324e6u, 0x04ec5b65u, 0x8065dc6cu, 0x3599cec7u, 0x0e530b77u}

BP_HD sc sc_zero() { sc r; for (int i = 0; i < 8; i++) r.v[i] = 0; return r; }
BP_HD sc sc_l() { return sc{SC_L_LIMBS}; }
BP_HD sc sc_mont_one() { return sc{SC_R_LIMBS}; }

BP_HD bool sc_geq_l(const sc &a) {
    const sc l = sc_l();
    for (int i = 7; i >= 0; i--) { if (a.v[i] > l.v[i]) return true; if (a.v[i] < l.v[i]) return false; }
    return true;
}
// a - l if a >= l (a < 2l)
BP_HD sc sc_cond_sub_l(const sc &a) {
    const sc l = sc_l(); sc d; int64_t c = 0;
    for (int i = 0; i < 8; i++) { c += (int64_t)a.v[i] - l.v[i]; d.v[i] = (uint32_t)c; c >>= 32; }
    uint32_t m = (uint32_t)c;            // all ones if a < l
    sc r; for (int i = 0; i < 8; i++) r.v[i] = (a.v[i] & m) | (d.v[i] & ~m);
    return r;
}
BP_HD sc sc_add(const sc &a, const sc &b) {       // inputs < l
    sc t; uint64_t c = 0;
    for (int i = 0; i < 8; i++) { c += (uint64_t)a.v[i] + b.v[i]; t.v[i] = (uint32_t)c; c >>= 32; }
    return sc_cond_sub_l(t);                      // a + b < 2l < 2^254: no carry out
}
BP_HD sc sc_sub(const sc &a, const sc &b) {       // inputs < l
    const sc l = sc_l(); sc t; int64_t c = 0;
    for (int i = 0; i < 8; i++) { c += (int64_t)a.v[i] - b.v[i]; t.v[i] = (uint32_t)c; c >>= 32; }
    uint32_t m = (uint32_t)c;                     // all ones on borrow: add l back
    uint64_t k = 0;
    for (int i = 0; i < 8; i++) { k += (uint64_t)t.v[i] + (l.v[i] & m); t.v[i] = (uint32_t)k; k >>= 32; }
    return t;
}
BP_HD sc sc_neg(const sc &a) { return sc_sub(sc_zero(), a); }
BP_HD bool sc_is_zero(const sc &a) { uint32_t z = 0; for (int i = 0; i < 8; i++) z |= a.v[i]; return z == 0; }

// Montgomery product a*b/R mod l; b < l, a < 2^256
BP_HD sc sc_mont_mul(const sc &a, const sc &b) {
#ifdef __CUDA_ARCH__
    // three passes through the PTX 8x8 multiplier of fe.cuh (high ILP, short carry chains):
    // t = a*b;  M = t_lo * (-l^-1) mod 2^256;  r = (t + M*l) / 2^256  (< 2l)
    fe fa, fb, fl = fe{SC_L_LIMBS}, flp = fe{SC_LPRIME_LIMBS};
    for (int i = 0; i < 8; i++) { fa.v[i] = a.v[i]; fb.v[i] = b.v[i]; }
    uint32_t t[16], q[16], u[16];
    fe_mul_wide(t, fa, fb);
    fe tl; for (int i = 0; i < 8; i++) tl.v[i] = t[i];
    fe_mul_wide(q, tl, flp);
    fe M; for (int i = 0; i < 8; i++) M.v[i] = q[i];
    fe_mul_wide(u, M, fl);
    // low halves cancel to zero mod 2^256 with a carry of (t_lo != 0)
    uint32_t nz = 0; for (int i = 0; i < 8; i++) nz |= t[i];
    uint64_t c = nz ? 1 : 0;
    sc r;
    for (int i = 0; i < 8; i++) { c += (uint64_t)t[8 + i] + u[8 + i]; r.v[i] = (uint32_t)c; c >>= 32; }
    return sc_cond_sub_l(r);                      // sum < 2l < 2^254: c is zero here
#elif defined(__SIZEOF_INT128__)
    // host (the C++ mirror's scalar arithmetic, the host-emulation tests): CIOS on four 64-bit limbs with 128-bit products
    typedef unsigned __int128 u128_;
    const uint64_t L64[4] = {0x5812631a5cf5d3edULL, 0x14def9dea2f79cd6ULL, 0, 0x1000000000000000ULL}, LF = 0xd2b51da312547e1bULL;     // l, -l^-1 mod 2^64
    uint64_t x[4], y[4], t[6] = {0, 0, 0, 0, 0, 0};
    for (int i = 0; i < 4; i++) { x[i] = (uint64_t)a.v[2 * i] | ((uint64_t)a.v[2 * i + 1] << 32); y[i] = (uint64_t)b.v[2 * i] | ((uint64_t)b.v[2 * i + 1] << 32); }
    for (int i = 0; i < 4; i++) {
        u128_ c = 0;
        for (int j = 0; j < 4; j++) { c += (u128_)x[j] * y[i] + t[j]; t[j] = (uint64_t)c; c >>= 64; }
        c += t[4]; t[4] = (uint64_t)c; t[5] = (uint64_t)(c >> 64);
        uint64_t m = t[0] * LF;
        c = (u128_)m * L64[0] + t[0]; c >>= 64;
        for (int j = 1; j < 4; j++) { c += (u128_)m * L64[j] + t[j]; t[j - 1] = (uint64_t)c; c >>= 64; }
        c += t[4]; t[3] = (uint64_t)c; t[4] = t[5] + (uint64_t)(c >> 64);
    }
    sc r; for (int i = 0; i < 4; i++) { r.v[2 * i] = (uint32_t)t[i]; r.v[2 * i + 1] = (uint32_t)(t[i] >> 32); }
    return sc_cond_sub_l(r);                      // t < 2l
#else
    const sc l = sc_l();
    uint32_t t[10];
    for (int i = 0; i < 10; i++) t[i] = 0;
    for (int i = 0; i < 8; i++) {
        uint64_t c = 0;
        for (int j = 0; j < 8; j++) { c += (uint64_t)a.v[j] * b.v[i] + t[j]; t[j] = (uint32_t)c; c >>= 32; }
        c += t[8]; t[8] = (uint32_t)c; t[9] = (uint32_t)(c >> 32);
        uint32_t m = t[0] * SC_LFACTOR;
        c = (uint64_t)m * l.v[0] + t[0]; c >>= 32;
        for (int j = 1; j < 8; j++) { c += (uint64_t)m * l.v[j] + t[j]; t[j - 1] = (uint32_t)c; c >>= 32; }
        c += t[8]; t[7] = (uint32_t)c; t[8] = t[9] + (uint32_t)(c >> 32);
    }
    sc r; for (int i = 0; i < 8; i++) r.v[i] = t[i];
    return sc_cond_sub_l(r);                      // t < 2l
#endif
}
// Lazy reduction for sums of products: acc (16 limbs) += a*b without reducing, then one Montgomery reduction of the sum.
// Up to 32 products of values < l fit: 32 l^2 < 2^512, and REDC(T) = (T + M l)/R < T/R + l < 3l for T < 32 l^2 (R = 2^256 ~ 16 l).
struct sc_wide { uint32_t v[16]; };
BP_HD sc_wide sc_wide_zero() { sc_wide r; for (int i = 0; i < 16; i++) r.v[i] = 0; return r; }
BP_HD void sc_wide_mac(sc_wide &acc, const sc &a, const sc &b) {
    fe fa, fb;
    for (int i = 0; i < 8; i++) { fa.v[i] = a.v[i]; fb.v[i] = b.v[i]; }
    uint32_t t[16];
    fe_mul_wide(t, fa, fb);
    uint64_t c = 0;
    for (int i = 0; i < 16; i++) { c += (uint64_t)acc.v[i] + t[i]; acc.v[i] = (uint32_t)c; c >>= 32; }
}
// T/R mod l for T < 32 l^2, result < l
BP_HD sc sc_wide_redc(const sc_wide &T) {
    fe fl = fe{SC_L_LIMBS}, flp = fe{SC_LPRIME_LIMBS}, tl;
    for (int i = 0; i < 8; i++) tl.v[i] = T.v[i];
    uint32_t q[16], u[16];
    fe_mul_wide(q, tl, flp);
    fe M; for (int i = 0; i < 8; i++) M.v[i] = q[i];
    fe_mul_wide(u, M, fl);
    uint32_t nz = 0; for (int i = 0; i < 8; i++) nz |= T.v[i];
    uint64_t c = nz ? 1 : 0;
    sc r;
    for (int i = 0; i < 8; i++) { c += (uint64_t)T.v[8 + i] + u[8 + i]; r.v[i] = (uint32_t)c; c >>= 32; }
    return sc_cond_sub_l(sc_cond_sub_l(r));       // < 3l before, c is zero (3l < 2^254)
}
BP_HD sc sc_to_mont(const sc &a) { return sc_mont_mul(a, sc{SC_RR_LIMBS}); }
BP_HD sc sc_from_mont(const sc &a) { sc one = sc_zero(); one.v[0] = 1; return sc_mont_mul(a, one); }
BP_HD sc sc_mont_from_u64(uint64_t x) { sc t = sc_zero(); t.v[0] = (uint32_t)x; t.v[1] = (uint32_t)(x >> 32); return sc_to_mont(t); }

BP_HD sc sc_load(const uint8_t b[32]) {
    sc r; for (int i = 0; i < 8; i++) r.v[i] = (uint32_t)b[4 * i] | ((uint32_t)b[4 * i + 1] << 8) | ((uint32_t)b[4 * i + 2] << 16) | ((uint32_t)b[4 * i + 3] << 24);
    return r;
}
BP_HD void sc_store(uint8_t b[32], const sc &a) {
    for (int i = 0; i < 8; i++) { b[4 * i] = (uint8_t)a.v[i]; b[4 * i + 1] = (uint8_t)(a.v[i] >> 8); b[4 * i + 2] = (uint8_t)(a.v[i] >> 16); b[4 * i + 3] = (uint8_t)(a.v[i] >> 24); }
}
// Scalar::from_bytes_mod_order_wide, result in Montgomery form
BP_HD sc sc_mont_from_wide(const uint8_t b[64]) {
    sc lo = sc_load(b), hi = sc_load(b + 32);
    return sc_add(sc_mont_mul(lo, sc{SC_RR_LIMBS}), sc_mont_mul(hi, sc{SC_RRR_LIMBS}));
}
// a^(l-2) in Montgomery form (variable time: the verifier's data are public)
BP_HDN sc sc_mont_invert(const sc &a) {
    // l - 2 = 2^252 + 0x14def9dea2f79cd65812631a5cf5d3eb
    const uint32_t e[4] = {0x5cf5d3ebu, 0x5812631au, 0xa2f79cd6u, 0x14def9deu};
    sc acc = a;                                   // bit 252
    for (int i = 251; i >= 128; i--) acc = sc_mont_mul(acc, acc);
    for (int i = 127; i >= 0; i--) {
        acc = sc_mont_mul(acc, acc);
        if ((e[i >> 5] >> (i & 31)) & 1u) acc = sc_mont_mul(acc, a);
    }
    return acc;
}
