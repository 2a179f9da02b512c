/* ORACLE (test infrastructure only).
 *
 * Scalars mod l = 2^252 + 27742317777372353535851937790883648493 as four 64-bit limbs.
 * Restates what the reference obtains from curve25519_dalek::scalar::Scalar (un-vendored
 * dependency, Cargo.toml:21): canonical 32-byte little-endian encodings,
 * `from_bytes_mod_order_wide` (used by challenge_scalar, src/transcript.rs:89-94),
 * `from_canonical_bytes` (src/range_proof/mod.rs:519-524), invert, batch_invert.
 * Reduction uses 2^252 = -c (mod l) folds, not dalek's Montgomery form; results are the same
 * canonical residues.
 */
#ifndef ORACLE_SC_H
#define ORACLE_SC_H
#include <stdint.h>
#include <string.h>

typedef unsigned __int128 sc_u128;
typedef struct { uint64_t v[4]; } sc;

static const uint64_t SC_L[4] = { 0x5812631a5cf5d3edULL, 0x14def9dea2f79cd6ULL, 0, 0x1000000000000000ULL };
static const uint64_t SC_C[2] = { 0x5812631a5cf5d3edULL, 0x14def9dea2f79cd6ULL };  /* l - 2^252 */

static inline int sc_geq_l(const uint64_t a[4]) {
    for (int i = 3; i >= 0; i--) { if (a[i] > SC_L[i]) return 1; if (a[i] < SC_L[i]) return 0; }
    return 1;
}
static inline uint64_t sc_add_raw(uint64_t r[4], const uint64_t a[4], const uint64_t b[4]) {
    sc_u128 c = 0;
    for (int i = 0; i < 4; i++) { c += (sc_u128)a[i] + b[i]; r[i] = (uint64_t)c; c >>= 64; }
    return (uint64_t)c;
}
static inline uint64_t sc_sub_raw(uint64_t r[4], const uint64_t a[4], const uint64_t b[4]) {
    uint64_t borrow = 0;
    for (int i = 0; i < 4; i++) {
        sc_u128 d = (sc_u128)a[i] - b[i] - borrow; r[i] = (uint64_t)d; borrow = (uint64_t)(d >> 64) & 1;
    }
    return borrow;
}

/* out[0..n+2) = in[0..n) * c */
static inline void sc_mul_c(uint64_t *out, const uint64_t *in, int n) {
    for (int i = 0; i < n + 2; i++) out[i] = 0;
    for (int i = 0; i < n; i++) {
        sc_u128 carry = 0;
        for (int j = 0; j < 2; j++) {
            carry += (sc_u128)in[i] * SC_C[j] + out[i + j]; out[i + j] = (uint64_t)carry; carry >>= 64;
        }
        int k = i + 2;
        while (carry && k < n + 2) { carry += out[k]; out[k] = (uint64_t)carry; carry >>= 64; k++; }
    }
}

/* split x (n limbs) at bit 252: lo = x mod 2^252 (4 limbs), hi = x >> 252 (n-3 limbs, caller sized) */
static inline void sc_split252(uint64_t lo[4], uint64_t *hi, const uint64_t *x, int n) {
    lo[0] = x[0]; lo[1] = x[1]; lo[2] = x[2]; lo[3] = x[3] & 0x0fffffffffffffffULL;
    for (int i = 3; i < n; i++) {
        uint64_t w = x[i] >> 60;
        if (i + 1 < n) w |= x[i + 1] << 4;
        hi[i - 3] = w;
    }
}

/* reduce a 512-bit little-endian limb array mod l */
static inline void sc_reduce512(sc *r, const uint64_t x[8]) {
    uint64_t x0[4], x1[5];            /* x = x0 + x1*2^252, x1 < 2^260 */
    sc_split252(x0, x1, x, 8);
    uint64_t t[7];                    /* t = x1*c < 2^385 */
    sc_mul_c(t, x1, 5);
    uint64_t t0[4], t1[4];            /* t1 < 2^133 */
    sc_split252(t0, t1, t, 7);
    uint64_t u[5];                    /* u = t1*c < 2^258 (t1 uses 3 limbs) */
    sc_mul_c(u, t1, 3);
    uint64_t u0[4], u1[2];
    sc_split252(u0, u1, u, 5);        /* u1 < 2^6 */
    uint64_t w[3];                    /* w = u1*c < 2^131 */
    sc_mul_c(w, u1, 1);
    uint64_t w4[4] = { w[0], w[1], w[2], 0 };
    /* x = x0 - t0 + u0 - w (mod l); every term < 2^252 < l.  acc = x0 + u0 + 2l - t0 - w > 0 */
    uint64_t acc[4], twol[4];
    sc_add_raw(twol, SC_L, SC_L);
    sc_add_raw(acc, x0, u0);
    sc_add_raw(acc, acc, twol);
    sc_sub_raw(acc, acc, t0);
    sc_sub_raw(acc, acc, w4);
    while (sc_geq_l(acc)) sc_sub_raw(acc, acc, SC_L);
    memcpy(r->v, acc, 32);
}

static inline void sc_from_bytes_wide(sc *r, const uint8_t b[64]) { uint64_t x[8]; memcpy(x, b, 64); sc_reduce512(r, x); }
static inline void sc_from_bytes_mod_order(sc *r, const uint8_t b[32]) {
    uint64_t x[8] = {0}; memcpy(x, b, 32); sc_reduce512(r, x);
}
/* returns 0 if the encoding is not canonical (>= l) */
static inline int sc_from_canonical(sc *r, const uint8_t b[32]) { memcpy(r->v, b, 32); return !sc_geq_l(r->v); }
static inline void sc_tobytes(uint8_t b[32], const sc *a) { memcpy(b, a->v, 32); }
static inline void sc_zero(sc *r) { memset(r, 0, sizeof *r); }
static inline void sc_from_u64(sc *r, uint64_t x) { sc_zero(r); r->v[0] = x; }
static inline int sc_is_zero(const sc *a) { return (a->v[0] | a->v[1] | a->v[2] | a->v[3]) == 0; }
static inline int sc_eq(const sc *a, const sc *b) { return memcmp(a, b, sizeof *a) == 0; }

static inline void sc_add(sc *r, const sc *a, const sc *b) {
    uint64_t t[4]; sc_add_raw(t, a->v, b->v);          /* < 2^254, no carry out */
    if (sc_geq_l(t)) sc_sub_raw(t, t, SC_L);
    memcpy(r->v, t, 32);
}
static inline void sc_sub(sc *r, const sc *a, const sc *b) {
    uint64_t t[4];
    if (sc_sub_raw(t, a->v, b->v)) sc_add_raw(t, t, SC_L);
    memcpy(r->v, t, 32);
}
static inline void sc_neg(sc *r, const sc *a) { sc z; sc_zero(&z); sc_sub(r, &z, a); }
static inline void sc_mul(sc *r, const sc *a, const sc *b) {
    uint64_t x[8] = {0};
    for (int i = 0; i < 4; i++) {
        sc_u128 carry = 0;
        for (int j = 0; j < 4; j++) {
            carry += (sc_u128)a->v[i] * b->v[j] + x[i + j]; x[i + j] = (uint64_t)carry; carry >>= 64;
        }
        x[i + 4] = (uint64_t)carry;
    }
    sc_reduce512(r, x);
}
static inline void sc_muladd(sc *r, const sc *a, const sc *b, const sc *c) { sc t; sc_mul(&t, a, b); sc_add(r, &t, c); }

/* a^(l-2) by square-and-multiply (variable time; oracle only) */
static inline void sc_invert(sc *r, const sc *a) {
    uint64_t e[4]; uint64_t two[4] = {2, 0, 0, 0};
    sc_sub_raw(e, SC_L, two);
    sc acc; sc_from_u64(&acc, 1);
    for (int i = 252; i >= 0; i--) {
        sc_mul(&acc, &acc, &acc);
        if ((e[i >> 6] >> (i & 63)) & 1) sc_mul(&acc, &acc, a);
    }
    *r = acc;
}
#endif
