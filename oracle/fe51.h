/* ORACLE (test infrastructure only — never linked into the product path).
 *
 * Field arithmetic mod p = 2^255 - 19 in five 51-bit limbs with 128-bit products:
 * a CPU restatement of the serial "u64 backend" that the reference selects through
 * `curve25519-dalek = { version = "2", features = ["u64_backend", ...] }`
 * (Cargo.toml:21).  That crate is NOT vendored in the reference repository,
 * so this file restates the published algorithm (radix-2^51 schoolbook multiply with
 * the 19-fold of the high half) rather than following reference lines.
 */
#ifndef ORACLE_FE51_H
#define ORACLE_FE51_H
#include <stdint.h>
#include <string.h>

typedef unsigned __int128 u128;
typedef struct { uint64_t v[5]; } fe;

#define FE_MASK51 ((1ULL << 51) - 1)

static inline void fe_0(fe *h) { memset(h, 0, sizeof *h); }
static inline void fe_1(fe *h) { fe_0(h); h->v[0] = 1; }
static inline void fe_copy(fe *h, const fe *f) { *h = *f; }

/* carry so that every limb < 2^51 + small */
static inline void fe_weak_reduce(fe *h) {
    uint64_t c;
    c = h->v[0] >> 51; h->v[0] &= FE_MASK51; h->v[1] += c;
    c = h->v[1] >> 51; h->v[1] &= FE_MASK51; h->v[2] += c;
    c = h->v[2] >> 51; h->v[2] &= FE_MASK51; h->v[3] += c;
    c = h->v[3] >> 51; h->v[3] &= FE_MASK51; h->v[4] += c;
    c = h->v[4] >> 51; h->v[4] &= FE_MASK51; h->v[0] += c * 19;
}

static inline void fe_add(fe *h, const fe *f, const fe *g) {
    for (int i = 0; i < 5; i++) h->v[i] = f->v[i] + g->v[i];
    fe_weak_reduce(h);
}

/* h = f - g, computed as f + 4p - g so no limb underflows (inputs < 2^52) */
static inline void fe_sub(fe *h, const fe *f, const fe *g) {
    h->v[0] = f->v[0] + 0x1fffffffffffb4ULL - g->v[0];   /* 4*(2^51-19) */
    h->v[1] = f->v[1] + 0x1ffffffffffffcULL - g->v[1];   /* 4*(2^51-1)  */
    h->v[2] = f->v[2] + 0x1ffffffffffffcULL - g->v[2];
    h->v[3] = f->v[3] + 0x1ffffffffffffcULL - g->v[3];
    h->v[4] = f->v[4] + 0x1ffffffffffffcULL - g->v[4];
    fe_weak_reduce(h);
}

static inline void fe_neg(fe *h, const fe *f) { fe z; fe_0(&z); fe_sub(h, &z, f); }

static inline void fe_mul(fe *h, const fe *f, const fe *g) {
    uint64_t f0 = f->v[0], f1 = f->v[1], f2 = f->v[2], f3 = f->v[3], f4 = f->v[4];
    uint64_t g0 = g->v[0], g1 = g->v[1], g2 = g->v[2], g3 = g->v[3], g4 = g->v[4];
    uint64_t g1_19 = g1 * 19, g2_19 = g2 * 19, g3_19 = g3 * 19, g4_19 = g4 * 19;
    u128 r0 = (u128)f0 * g0 + (u128)f1 * g4_19 + (u128)f2 * g3_19 + (u128)f3 * g2_19 + (u128)f4 * g1_19;
    u128 r1 = (u128)f0 * g1 + (u128)f1 * g0 + (u128)f2 * g4_19 + (u128)f3 * g3_19 + (u128)f4 * g2_19;
    u128 r2 = (u128)f0 * g2 + (u128)f1 * g1 + (u128)f2 * g0 + (u128)f3 * g4_19 + (u128)f4 * g3_19;
    u128 r3 = (u128)f0 * g3 + (u128)f1 * g2 + (u128)f2 * g1 + (u128)f3 * g0 + (u128)f4 * g4_19;
    u128 r4 = (u128)f0 * g4 + (u128)f1 * g3 + (u128)f2 * g2 + (u128)f3 * g1 + (u128)f4 * g0;
    uint64_t c;
    r1 += (uint64_t)(r0 >> 51); uint64_t h0 = (uint64_t)r0 & FE_MASK51;
    r2 += (uint64_t)(r1 >> 51); uint64_t h1 = (uint64_t)r1 & FE_MASK51;
    r3 += (uint64_t)(r2 >> 51); uint64_t h2 = (uint64_t)r2 & FE_MASK51;
    r4 += (uint64_t)(r3 >> 51); uint64_t h3 = (uint64_t)r3 & FE_MASK51;
    c = (uint64_t)(r4 >> 51);   uint64_t h4 = (uint64_t)r4 & FE_MASK51;
    h0 += c * 19;
    c = h0 >> 51; h0 &= FE_MASK51; h1 += c;
    h->v[0] = h0; h->v[1] = h1; h->v[2] = h2; h->v[3] = h3; h->v[4] = h4;
}

static inline void fe_sq(fe *h, const fe *f) {       /* 15 limb products instead of 25 */
    uint64_t f0 = f->v[0], f1 = f->v[1], f2 = f->v[2], f3 = f->v[3], f4 = f->v[4];
    uint64_t f0_2 = 2 * f0, f1_2 = 2 * f1, f3_19 = 19 * f3, f4_19 = 19 * f4;
    u128 r0 = (u128)f0 * f0 + (u128)(2 * f1) * f4_19 + (u128)(2 * f2) * f3_19;
    u128 r1 = (u128)f0_2 * f1 + (u128)(2 * f2) * f4_19 + (u128)f3 * f3_19;
    u128 r2 = (u128)f0_2 * f2 + (u128)f1 * f1 + (u128)(2 * f3) * f4_19;
    u128 r3 = (u128)f0_2 * f3 + (u128)f1_2 * f2 + (u128)f4 * f4_19;
    u128 r4 = (u128)f0_2 * f4 + (u128)f1_2 * f3 + (u128)f2 * f2;
    uint64_t c;
    r1 += (uint64_t)(r0 >> 51); uint64_t h0 = (uint64_t)r0 & FE_MASK51;
    r2 += (uint64_t)(r1 >> 51); uint64_t h1 = (uint64_t)r1 & FE_MASK51;
    r3 += (uint64_t)(r2 >> 51); uint64_t h2 = (uint64_t)r2 & FE_MASK51;
    r4 += (uint64_t)(r3 >> 51); uint64_t h3 = (uint64_t)r3 & FE_MASK51;
    c = (uint64_t)(r4 >> 51);   uint64_t h4 = (uint64_t)r4 & FE_MASK51;
    h0 += c * 19;
    c = h0 >> 51; h0 &= FE_MASK51; h1 += c;
    h->v[0] = h0; h->v[1] = h1; h->v[2] = h2; h->v[3] = h3; h->v[4] = h4;
}

static inline void fe_sqn(fe *h, const fe *f, int n) {
    fe_sq(h, f);
    for (int i = 1; i < n; i++) fe_sq(h, h);
}

static inline void fe_mul_small(fe *h, const fe *f, uint64_t s) { /* s < 2^12 */
    fe g; fe_0(&g); g.v[0] = s; fe_mul(h, f, &g);
}

/* canonical little-endian encoding */
static inline void fe_tobytes(uint8_t s[32], const fe *f) {
    fe t = *f;
    fe_weak_reduce(&t);
    fe_weak_reduce(&t);
    /* now t < 2p; compute q = (t + 19) >> 255 */
    uint64_t q = (t.v[0] + 19) >> 51;
    q = (t.v[1] + q) >> 51; q = (t.v[2] + q) >> 51; q = (t.v[3] + q) >> 51; q = (t.v[4] + q) >> 51;
    t.v[0] += 19 * q;
    uint64_t c;
    c = t.v[0] >> 51; t.v[0] &= FE_MASK51; t.v[1] += c;
    c = t.v[1] >> 51; t.v[1] &= FE_MASK51; t.v[2] += c;
    c = t.v[2] >> 51; t.v[2] &= FE_MASK51; t.v[3] += c;
    c = t.v[3] >> 51; t.v[3] &= FE_MASK51; t.v[4] += c;
    t.v[4] &= FE_MASK51;
    uint64_t w0 = t.v[0] | (t.v[1] << 51);
    uint64_t w1 = (t.v[1] >> 13) | (t.v[2] << 38);
    uint64_t w2 = (t.v[2] >> 26) | (t.v[3] << 25);
    uint64_t w3 = (t.v[3] >> 39) | (t.v[4] << 12);
    memcpy(s, &w0, 8); memcpy(s + 8, &w1, 8); memcpy(s + 16, &w2, 8); memcpy(s + 24, &w3, 8);
}

/* loads 255 bits; bit 255 is ignored (callers that need canonicity re-encode and compare) */
static inline void fe_frombytes(fe *h, const uint8_t s[32]) {
    uint64_t w0, w1, w2, w3;
    memcpy(&w0, s, 8); memcpy(&w1, s + 8, 8); memcpy(&w2, s + 16, 8); memcpy(&w3, s + 24, 8);
    h->v[0] = w0 & FE_MASK51;
    h->v[1] = ((w0 >> 51) | (w1 << 13)) & FE_MASK51;
    h->v[2] = ((w1 >> 38) | (w2 << 26)) & FE_MASK51;
    h->v[3] = ((w2 >> 25) | (w3 << 39)) & FE_MASK51;
    h->v[4] = (w3 >> 12) & FE_MASK51;
}

static inline int fe_is_negative(const fe *f) { uint8_t s[32]; fe_tobytes(s, f); return s[0] & 1; }
static inline int fe_is_zero(const fe *f) {
    uint8_t s[32]; fe_tobytes(s, f); uint8_t r = 0; for (int i = 0; i < 32; i++) r |= s[i]; return r == 0;
}
static inline int fe_eq(const fe *a, const fe *b) {
    uint8_t x[32], y[32]; fe_tobytes(x, a); fe_tobytes(y, b); return memcmp(x, y, 32) == 0;
}
static inline void fe_abs(fe *h, const fe *f) { if (fe_is_negative(f)) fe_neg(h, f); else *h = *f; }

/* z^(2^250 - 1) ladder shared by invert and pow22523; returns also z^11 */
static inline void fe_pow_2_250_1(fe *out, fe *z11, const fe *z) {
    fe t0, t1, t2, t3;
    fe_sq(&t0, z);                 /* 2 */
    fe_sqn(&t1, &t0, 2);           /* 8 */
    fe_mul(&t1, z, &t1);           /* 9 */
    fe_mul(&t0, &t0, &t1);         /* 11 */
    *z11 = t0;
    fe_sq(&t2, &t0);               /* 22 */
    fe_mul(&t1, &t1, &t2);         /* 31 = 2^5-1 */
    fe_sqn(&t2, &t1, 5);  fe_mul(&t1, &t2, &t1);   /* 2^10-1 */
    fe_sqn(&t2, &t1, 10); fe_mul(&t2, &t2, &t1);   /* 2^20-1 */
    fe_sqn(&t3, &t2, 20); fe_mul(&t2, &t3, &t2);   /* 2^40-1 */
    fe_sqn(&t2, &t2, 10); fe_mul(&t1, &t2, &t1);   /* 2^50-1 */
    fe_sqn(&t2, &t1, 50); fe_mul(&t2, &t2, &t1);   /* 2^100-1 */
    fe_sqn(&t3, &t2, 100); fe_mul(&t2, &t3, &t2);  /* 2^200-1 */
    fe_sqn(&t2, &t2, 50); fe_mul(out, &t2, &t1);   /* 2^250-1 */
}

static inline void fe_invert(fe *out, const fe *z) {   /* z^(p-2) = z^(2^255-21) */
    fe t, z11;
    fe_pow_2_250_1(&t, &z11, z);
    fe_sqn(&t, &t, 5);             /* 2^255 - 32 */
    fe_mul(out, &t, &z11);         /* 2^255 - 21 */
}

static inline void fe_pow22523(fe *out, const fe *z) { /* z^((p-5)/8) = z^(2^252-3) */
    fe t, z11;
    fe_pow_2_250_1(&t, &z11, z);
    fe_sqn(&t, &t, 2);             /* 2^252 - 4 */
    fe_mul(out, &t, z);            /* 2^252 - 3 */
}

/* parse a decimal literal (value < p) */
static inline void fe_from_decimal(fe *h, const char *dec) {
    fe ten, d; fe_0(h); fe_0(&ten); ten.v[0] = 10;
    for (; *dec; dec++) {
        fe_mul(h, h, &ten);
        fe_0(&d); d.v[0] = (uint64_t)(*dec - '0');
        fe_add(h, h, &d);
    }
}
#endif
