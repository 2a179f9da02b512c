/* ORACLE (test infrastructure only).
 *
 * Ristretto255 group on the twisted Edwards curve -x^2+y^2 = 1+d x^2 y^2 in extended
 * coordinates, plus the two variable-time multiscalar algorithms the reference reaches through
 * `RistrettoPoint::vartime_multiscalar_mul` / `optional_multiscalar_mul`
 * (src/inner_product_proof.rs:87,101,127,131,153,159,177,178,308;
 *  src/range_proof/mod.rs:421): Straus with width-5 NAF below 190 terms and
 * Pippenger (w = 6/7/8 by size, signed radix-2^w digits) from 190 terms up — the algorithm
 * selection of curve25519-dalek 2.x, an un-vendored dependency (Cargo.toml:21),
 * restated from its published design.  encode/decode/Elligator follow the ristretto255
 * specification as summarised in SURVEY.md section 8(c).
 */
#ifndef ORACLE_GE_H
#define ORACLE_GE_H
#include <stdlib.h>
#include "fe51.h"
#include "sc.h"

typedef struct { fe X, Y, Z, T; } ge;                 /* extended */
typedef struct { fe X, Y, Z; } ge_p2;                 /* projective */
typedef struct { fe X, Y, Z, T; } ge_p1p1;            /* completed */
typedef struct { fe YpX, YmX, Z, T2d; } ge_cached;    /* projective Niels */

static fe GE_D, GE_D2, GE_SQRT_M1, GE_SQRT_AD_MINUS_ONE, GE_INVSQRT_A_MINUS_D, GE_ONE_MINUS_D_SQ, GE_D_MINUS_ONE_SQ;
static ge GE_BASEPOINT;
static int ge_consts_ready = 0;

static void ge_identity(ge *p) { fe_0(&p->X); fe_1(&p->Y); fe_1(&p->Z); fe_0(&p->T); }

static void ge_to_cached(ge_cached *c, const ge *p) {
    fe_add(&c->YpX, &p->Y, &p->X); fe_sub(&c->YmX, &p->Y, &p->X); c->Z = p->Z; fe_mul(&c->T2d, &p->T, &GE_D2);
}
static void ge_cached_neg(ge_cached *r, const ge_cached *c) { r->YpX = c->YmX; r->YmX = c->YpX; r->Z = c->Z; fe_neg(&r->T2d, &c->T2d); }
static void ge_p1p1_to_p3(ge *r, const ge_p1p1 *p) {
    fe_mul(&r->X, &p->X, &p->T); fe_mul(&r->Y, &p->Y, &p->Z); fe_mul(&r->Z, &p->Z, &p->T); fe_mul(&r->T, &p->X, &p->Y);
}
static void ge_p1p1_to_p2(ge_p2 *r, const ge_p1p1 *p) {
    fe_mul(&r->X, &p->X, &p->T); fe_mul(&r->Y, &p->Y, &p->Z); fe_mul(&r->Z, &p->Z, &p->T);
}
/* r = p + q (q in cached form) */
static void ge_add_cached(ge_p1p1 *r, const ge *p, const ge_cached *q) {
    fe ypx, ymx, pp, mm, tt2d, zz, zz2;
    fe_add(&ypx, &p->Y, &p->X); fe_sub(&ymx, &p->Y, &p->X);
    fe_mul(&pp, &ypx, &q->YpX); fe_mul(&mm, &ymx, &q->YmX);
    fe_mul(&tt2d, &p->T, &q->T2d); fe_mul(&zz, &p->Z, &q->Z); fe_add(&zz2, &zz, &zz);
    fe_sub(&r->X, &pp, &mm); fe_add(&r->Y, &pp, &mm); fe_add(&r->Z, &zz2, &tt2d); fe_sub(&r->T, &zz2, &tt2d);
}
static void ge_sub_cached(ge_p1p1 *r, const ge *p, const ge_cached *q) { ge_cached n; ge_cached_neg(&n, q); ge_add_cached(r, p, &n); }
/* doubling of a projective point -> completed */
static void ge_p2_dbl(ge_p1p1 *r, const ge_p2 *p) {
    fe xx, yy, zz2, xpy, xpy2;
    fe_sq(&xx, &p->X); fe_sq(&yy, &p->Y); fe_sq(&zz2, &p->Z); fe_add(&zz2, &zz2, &zz2);
    fe_add(&xpy, &p->X, &p->Y); fe_sq(&xpy2, &xpy);
    fe_add(&r->Y, &yy, &xx);            /* Y3 = YY + XX */
    fe_sub(&r->Z, &yy, &xx);            /* Z3 = YY - XX */
    fe_sub(&r->X, &xpy2, &r->Y);        /* X3 = (X+Y)^2 - (YY+XX) */
    fe_sub(&r->T, &zz2, &r->Z);         /* T3 = 2ZZ - (YY-XX) */
}
static void ge_add(ge *r, const ge *p, const ge *q) { ge_cached c; ge_p1p1 t; ge_to_cached(&c, q); ge_add_cached(&t, p, &c); ge_p1p1_to_p3(r, &t); }
static void ge_sub(ge *r, const ge *p, const ge *q) { ge_cached c; ge_p1p1 t; ge_to_cached(&c, q); ge_sub_cached(&t, p, &c); ge_p1p1_to_p3(r, &t); }
static void ge_neg(ge *r, const ge *p) { fe_neg(&r->X, &p->X); r->Y = p->Y; r->Z = p->Z; fe_neg(&r->T, &p->T); }
static void ge_dbl(ge *r, const ge *p) { ge_p2 q = { p->X, p->Y, p->Z }; ge_p1p1 t; ge_p2_dbl(&t, &q); ge_p1p1_to_p3(r, &t); }

/* Ristretto equality and identity-coset test */
static int ge_ristretto_eq(const ge *a, const ge *b) {
    fe l, r; fe_mul(&l, &a->X, &b->Y); fe_mul(&r, &a->Y, &b->X); if (fe_eq(&l, &r)) return 1;
    fe_mul(&l, &a->Y, &b->Y); fe_mul(&r, &a->X, &b->X); return fe_eq(&l, &r);
}
static int ge_is_identity(const ge *a) { ge id; ge_identity(&id); return ge_ristretto_eq(a, &id); }

/* (was_square, r) with r = sqrt(u/v) or sqrt(i*u/v), r non-negative */
static int fe_sqrt_ratio_i(fe *r, const fe *u, const fe *v) {
    fe v3, v7, t, chk, neg_u, neg_u_i;
    fe_sq(&v3, v); fe_mul(&v3, &v3, v);
    fe_sq(&v7, &v3); fe_mul(&v7, &v7, v);
    fe_mul(&t, u, &v7); fe_pow22523(&t, &t);
    fe_mul(r, u, &v3); fe_mul(r, r, &t);
    fe_sq(&chk, r); fe_mul(&chk, &chk, v);
    fe_neg(&neg_u, u); fe_mul(&neg_u_i, &neg_u, &GE_SQRT_M1);
    int ok = fe_eq(&chk, u), flip = fe_eq(&chk, &neg_u), flip_i = fe_eq(&chk, &neg_u_i);
    if (flip || flip_i) fe_mul(r, r, &GE_SQRT_M1);
    fe_abs(r, r);
    return ok || flip;
}

/* returns 1 on success, 0 if the 32 bytes are not a valid canonical Ristretto encoding */
static int ge_decode(ge *p, const uint8_t s_bytes[32]) {
    fe s, ss, u1, u2, u2s, v, I, dx, dy, one, t;
    uint8_t chk[32];
    fe_frombytes(&s, s_bytes); fe_tobytes(chk, &s);
    if (memcmp(chk, s_bytes, 32) != 0) return 0;       /* non-canonical (>= p or bit 255 set) */
    if (s_bytes[0] & 1) return 0;                      /* negative */
    fe_1(&one);
    fe_sq(&ss, &s); fe_sub(&u1, &one, &ss); fe_add(&u2, &one, &ss); fe_sq(&u2s, &u2);
    fe_sq(&t, &u1); fe_mul(&t, &t, &GE_D); fe_neg(&t, &t); fe_sub(&v, &t, &u2s);   /* v = -d*u1^2 - u2^2 */
    fe_mul(&t, &v, &u2s);
    int ok = fe_sqrt_ratio_i(&I, &one, &t);
    fe_mul(&dx, &I, &u2); fe_mul(&dy, &I, &dx); fe_mul(&dy, &dy, &v);
    fe_add(&t, &s, &s); fe_mul(&p->X, &t, &dx); fe_abs(&p->X, &p->X);
    fe_mul(&p->Y, &u1, &dy); fe_1(&p->Z); fe_mul(&p->T, &p->X, &p->Y);
    if (!ok || fe_is_negative(&p->T) || fe_is_zero(&p->Y)) return 0;
    return 1;
}

static void ge_encode(uint8_t out[32], const ge *p) {
    fe u1, u2, t, I, d1, d2, zinv, ix, iy, ench, x, y, dinv, one, s;
    fe_add(&u1, &p->Z, &p->Y); fe_sub(&t, &p->Z, &p->Y); fe_mul(&u1, &u1, &t);
    fe_mul(&u2, &p->X, &p->Y);
    fe_sq(&t, &u2); fe_mul(&t, &t, &u1); fe_1(&one);
    fe_sqrt_ratio_i(&I, &one, &t);
    fe_mul(&d1, &I, &u1); fe_mul(&d2, &I, &u2);
    fe_mul(&zinv, &d1, &d2); fe_mul(&zinv, &zinv, &p->T);
    fe_mul(&ix, &p->X, &GE_SQRT_M1); fe_mul(&iy, &p->Y, &GE_SQRT_M1);
    fe_mul(&ench, &d1, &GE_INVSQRT_A_MINUS_D);
    fe_mul(&t, &p->T, &zinv);
    if (fe_is_negative(&t)) { x = iy; y = ix; dinv = ench; } else { x = p->X; y = p->Y; dinv = d2; }
    fe_mul(&t, &x, &zinv);
    if (fe_is_negative(&t)) fe_neg(&y, &y);
    fe_sub(&t, &p->Z, &y); fe_mul(&s, &dinv, &t); fe_abs(&s, &s);
    fe_tobytes(out, &s);
}

static void ge_elligator(ge *p, const fe *r0) {
    fe one, r, Ns, c, D, t, s, sp, Nt, ss; ge_p1p1 cp;
    fe_1(&one);
    fe_sq(&r, r0); fe_mul(&r, &r, &GE_SQRT_M1);
    fe_add(&Ns, &r, &one); fe_mul(&Ns, &Ns, &GE_ONE_MINUS_D_SQ);
    fe_neg(&c, &one);
    fe_mul(&t, &GE_D, &r); fe_sub(&D, &c, &t); fe_add(&t, &r, &GE_D); fe_mul(&D, &D, &t);
    int sq = fe_sqrt_ratio_i(&s, &Ns, &D);
    fe_mul(&sp, &s, r0); if (!fe_is_negative(&sp)) fe_neg(&sp, &sp);
    if (!sq) { s = sp; c = r; }
    fe_sub(&t, &r, &one); fe_mul(&Nt, &c, &t); fe_mul(&Nt, &Nt, &GE_D_MINUS_ONE_SQ); fe_sub(&Nt, &Nt, &D);
    fe_sq(&ss, &s);
    fe_add(&t, &s, &s); fe_mul(&cp.X, &t, &D);
    fe_mul(&cp.Z, &Nt, &GE_SQRT_AD_MINUS_ONE);
    fe_sub(&cp.Y, &one, &ss); fe_add(&cp.T, &one, &ss);
    ge_p1p1_to_p3(p, &cp);
}
static void ge_from_uniform_bytes(ge *p, const uint8_t b[64]) {
    fe r1, r2; ge p1, p2;
    fe_frombytes(&r1, b); fe_frombytes(&r2, b + 32);
    ge_elligator(&p1, &r1); ge_elligator(&p2, &r2); ge_add(p, &p1, &p2);
}

static void ge_init_constants(void) {
    if (ge_consts_ready) return;
    fe_from_decimal(&GE_D, "37095705934669439343138083508754565189542113879843219016388785533085940283555");
    fe_add(&GE_D2, &GE_D, &GE_D);
    fe_from_decimal(&GE_SQRT_M1, "19681161376707505956807079304988542015446066515923890162744021073123829784752");
    fe_from_decimal(&GE_SQRT_AD_MINUS_ONE, "25063068953384623474111414158702152701244531502492656460079210482610430750235");
    fe_from_decimal(&GE_INVSQRT_A_MINUS_D, "54469307008909316920995813868745141605393597292927456921205312896311721017578");
    fe_from_decimal(&GE_ONE_MINUS_D_SQ, "1159843021668779879193775521855586647937357759715417654439879720876111806838");
    fe_from_decimal(&GE_D_MINUS_ONE_SQ, "40440834346308536858101042469323190826248399146238708352240133220865137265952");
    /* ristretto255 basepoint = ed25519 basepoint: y = 4/5, x positive-even root */
    static const uint8_t bp[32] = { 0xe2, 0xf2, 0xae, 0x0a, 0x6a, 0xbc, 0x4e, 0x71, 0xa8, 0x84, 0xa9, 0x61, 0xc5, 0x00, 0x51, 0x5f,
                                    0x58, 0xe3, 0x0b, 0x6a, 0xa5, 0x82, 0xdd, 0x8d, 0xb6, 0xa6, 0x59, 0x45, 0xe0, 0x8d, 0x2d, 0x76 };
    ge_consts_ready = 1;
    ge_decode(&GE_BASEPOINT, bp);
}

/* returns 0 iff the algebraic identities defining the constants hold (self-check used by tests) */
static int ge_check_constants(void) {
    fe t, u, one, m1; fe_1(&one); fe_neg(&m1, &one);
    fe n, dnm; fe_0(&n); n.v[0] = 121665; fe_0(&dnm); dnm.v[0] = 121666;
    fe_mul(&t, &GE_D, &dnm); fe_add(&t, &t, &n); if (!fe_is_zero(&t)) return 1;          /* d*121666 = -121665 */
    fe_sq(&t, &GE_SQRT_M1); if (!fe_eq(&t, &m1)) return 2;
    fe_sq(&t, &GE_SQRT_AD_MINUS_ONE); fe_neg(&u, &GE_D); fe_sub(&u, &u, &one); if (!fe_eq(&t, &u)) return 3;   /* a*d-1 = -d-1 */
    fe_sq(&t, &GE_INVSQRT_A_MINUS_D); fe_mul(&t, &t, &u); if (!fe_eq(&t, &one)) return 4;                       /* a-d = -1-d */
    fe_sq(&t, &GE_D); fe_sub(&t, &one, &t); if (!fe_eq(&t, &GE_ONE_MINUS_D_SQ)) return 5;
    fe_sub(&t, &GE_D, &one); fe_sq(&t, &t); if (!fe_eq(&t, &GE_D_MINUS_ONE_SQ)) return 6;
    return 0;
}

/* ------------------------------------------------------------------ scalar multiplication */
static void ge_scalarmult(ge *r, const sc *s, const ge *p) {   /* plain double-and-add */
    ge acc; ge_identity(&acc);
    for (int i = 255; i >= 0; i--) {
        ge_dbl(&acc, &acc);
        if ((s->v[i >> 6] >> (i & 63)) & 1) ge_add(&acc, &acc, p);
    }
    *r = acc;
}

/* width-w non-adjacent form, 256 signed digits */
static void sc_naf(int8_t naf[256], const sc *s, int w) {
    uint64_t x[5] = { s->v[0], s->v[1], s->v[2], s->v[3], 0 };
    int width = 1 << w, window_mask = width - 1, pos = 0, carry = 0;
    memset(naf, 0, 256);
    while (pos < 256) {
        int idx = pos / 64, bit = pos % 64;
        uint64_t buf = bit < 64 - w ? x[idx] >> bit : (x[idx] >> bit) | (x[idx + 1] << (64 - bit));
        int window = carry + (int)(buf & window_mask);
        if ((window & 1) == 0) { pos += 1; continue; }
        if (window < width / 2) { carry = 0; naf[pos] = (int8_t)window; }
        else { carry = 1; naf[pos] = (int8_t)(window - width); }
        pos += w;
    }
}

/* Straus: shared doublings, per-point width-5 NAF tables of odd multiples */
static void ge_msm_straus(ge *out, const sc *scalars, const ge *points, size_t n) {
    int8_t (*nafs)[256] = malloc(n * 256);
    ge_cached (*tables)[8] = malloc(n * sizeof *tables);
    for (size_t k = 0; k < n; k++) {
        sc_naf(nafs[k], &scalars[k], 5);
        ge p2, cur = points[k]; ge_dbl(&p2, &points[k]);
        ge_to_cached(&tables[k][0], &cur);
        for (int j = 1; j < 8; j++) { ge_add(&cur, &cur, &p2); ge_to_cached(&tables[k][j], &cur); }
    }
    ge_p2 r = { {{0}}, {{1}}, {{1}} };
    ge_p1p1 t; ge r3;
    for (int i = 255; i >= 0; i--) {
        ge_p2_dbl(&t, &r);
        for (size_t k = 0; k < n; k++) {
            int d = nafs[k][i];
            if (d > 0) { ge_p1p1_to_p3(&r3, &t); ge_add_cached(&t, &r3, &tables[k][d / 2]); }
            else if (d < 0) { ge_p1p1_to_p3(&r3, &t); ge_sub_cached(&t, &r3, &tables[k][(-d) / 2]); }
        }
        ge_p1p1_to_p2(&r, &t);
    }
    ge_p1p1_to_p3(out, &t);   /* last completed point carries T */
    free(nafs); free(tables);
}

/* signed radix-2^w digits, digits in [-2^(w-1), 2^(w-1)) except the last which absorbs the carry */
static int sc_radix_2w(int8_t *digits, const sc *s, int w) {
    int count = (256 + w - 1) / w + (w == 8 ? 1 : 0);
    uint64_t x[5] = { s->v[0], s->v[1], s->v[2], s->v[3], 0 };
    int radix = 1 << w, mask = radix - 1, carry = 0, ndig = (256 + w - 1) / w;
    for (int i = 0; i < ndig; i++) {
        int bit_offset = i * w, idx = bit_offset / 64, bit = bit_offset % 64;
        uint64_t buf = bit < 64 - w ? x[idx] >> bit : (x[idx] >> bit) | (bit ? x[idx + 1] << (64 - bit) : 0);
        int coef = carry + (int)(buf & mask);
        carry = (coef + radix / 2) >> w;
        digits[i] = (int8_t)(coef - (carry << w));
    }
    if (w == 8) digits[ndig] = (int8_t)carry; else digits[ndig - 1] += (int8_t)(carry << w);
    return count;
}

static void ge_msm_pippenger(ge *out, const sc *scalars, const ge *points, size_t n) {
    int w = n < 500 ? 6 : n < 800 ? 7 : 8;
    int nb = 1 << (w - 1);
    int8_t (*digits)[44] = malloc(n * 44);
    ge_cached *cached = malloc(n * sizeof *cached);
    ge *buckets = malloc(nb * sizeof *buckets);
    int count = 0;
    for (size_t k = 0; k < n; k++) { memset(digits[k], 0, 44); count = sc_radix_2w(digits[k], &scalars[k], w); ge_to_cached(&cached[k], &points[k]); }
    ge total; ge_identity(&total);
    for (int col = count - 1; col >= 0; col--) {
        for (int b = 0; b < nb; b++) ge_identity(&buckets[b]);
        ge_p1p1 t;
        for (size_t k = 0; k < n; k++) {
            int d = digits[k][col];
            if (d > 0) { ge_add_cached(&t, &buckets[d - 1], &cached[k]); ge_p1p1_to_p3(&buckets[d - 1], &t); }
            else if (d < 0) { ge_sub_cached(&t, &buckets[-d - 1], &cached[k]); ge_p1p1_to_p3(&buckets[-d - 1], &t); }
        }
        ge run = buckets[nb - 1], sum = buckets[nb - 1];
        for (int b = nb - 2; b >= 0; b--) { ge_add(&run, &run, &buckets[b]); ge_add(&sum, &sum, &run); }
        for (int j = 0; j < w; j++) ge_dbl(&total, &total);
        ge_add(&total, &total, &sum);
    }
    *out = total;
    free(digits); free(cached); free(buckets);
}

/* optional vector backend (msm_avx2.c / msm_ifma.c), selected by orc_set_backend in bp_oracle.c; NULL = the serial u64 code below */
static void (*ge_msm_backend)(ge *out, const sc *scalars, const ge *points, size_t n) = NULL;

/* the dependency's dispatch: Straus below 190 terms, Pippenger from 190 up */
static void ge_msm_vartime(ge *out, const sc *scalars, const ge *points, size_t n) {
    if (ge_msm_backend) { ge_msm_backend(out, scalars, points, n); return; }
    if (n == 0) { ge_identity(out); return; }
    if (n < 190) ge_msm_straus(out, scalars, points, n); else ge_msm_pippenger(out, scalars, points, n);
}
#endif
