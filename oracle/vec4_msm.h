/* ORACLE (test infrastructure only — never linked into the product path).
 *
 * Variable-time multiscalar multiplication on top of a 4-way vector field backend (vec4_avx2.h or vec4_ifma.h, included
 * before this file).  Restates what the reference reaches through `RistrettoPoint::vartime_multiscalar_mul` /
 * `optional_multiscalar_mul` (src/range_proof/mod.rs:421, src/inner_product_proof.rs:87-178)
 * when curve25519-dalek runs one of its vector backends: extended points with the four coordinates (X, Y, Z, T) in the four
 * lanes of one vector element, the HWCD'08 section 3.1 parallel addition / doubling (two vector multiplications per addition,
 * one squaring + one multiplication per doubling), Straus with width-5 NAF tables below 190 terms and Pippenger from 190 up
 * (the same dispatch as ge.h).  Results are bit-identical to the scalar backend after encoding (unique canonical encodings).
 */
#include <stdlib.h>
#include "sc.h"

typedef struct { fe4 p; } gx;                    /* lanes (X, Y, Z, T) */
typedef struct { fe4 c; } gcv;                   /* cached: lanes (Y-X, Y+X, 2Z, 2dT), reduced */

static fe4 VEC_NAME(K_D2LANE);                   /* (1, 1, 1, 2d) */
static int VEC_NAME(k_ready) = 0;

static gx gx_from_ge(const ge *p) { gx r; r.p = fe4_pack(&p->X, &p->Y, &p->Z, &p->T); return r; }
static void gx_to_ge(ge *out, const gx *p) { fe t[4]; fe4_unpack(t, &p->p); out->X = t[0]; out->Y = t[1]; out->Z = t[2]; out->T = t[3]; }
static gx gx_identity(void) { ge id; ge_identity(&id); return gx_from_ge(&id); }

static gcv gx_to_cached(const gx *P) {
    fe4 A, B, s, d, t;
    fe4_perm(A, P->p, FE4_PERM_IMM(1, 1, 2, 3));          /* (Y, Y, Z, T) */
    fe4_perm(B, P->p, FE4_PERM_IMM(0, 0, 2, 3));          /* (X, X, Z, T) */
    s = fe4_add(A, B);                                     /* (., Y+X, 2Z, 2T) */
    d = fe4_sub(A, B);                                     /* (Y-X, ...) */
    fe4_blend(t, s, d, 1);
    t = fe4_reduce(t);
    gcv r; r.c = fe4_mul(t, VEC_NAME(K_D2LANE));           /* lane 3: 2T * d... K holds (1,1,1,d): 2dT */
    return r;
}
/* P + Q (neg = 0) or P - Q (neg = 1), Q cached */
static gx gx_add_cached(const gx *P, const gcv *Q, int neg) {
    fe4 A, B, s, d, S, M, P1, P2, U, V, sp, dp, q;
    fe4_perm(A, P->p, FE4_PERM_IMM(1, 1, 2, 3));
    fe4_perm(B, P->p, FE4_PERM_IMM(0, 0, 2, 3));
    s = fe4_add(A, B); d = fe4_sub(A, B);
    fe4_blend(S, P->p, d, 1); fe4_blend(S, S, s, 2);       /* (Y1-X1, Y1+X1, Z1, T1) */
    S = fe4_reduce(S);
    if (neg) { fe4_perm(q, Q->c, FE4_PERM_IMM(1, 0, 2, 3)); } else q = Q->c;     /* -Q swaps Y-X and Y+X (and negates 2dT: handled below) */
    M = fe4_mul(S, q);                                     /* (A', B', D', C') */
    fe4_perm(P1, M, FE4_PERM_IMM(1, 2, 2, 1));             /* (B', D', D', B') */
    fe4_perm(P2, M, FE4_PERM_IMM(0, 3, 3, 0));             /* (A', C', C', A') */
    s = fe4_reduce(fe4_add(P1, P2));                       /* add: (H, G, G, H)   sub: (H, F, F, H) */
    d = fe4_reduce(fe4_sub(P1, P2));                       /* add: (E, F, F, E)   sub: (E, G, G, E) */
    if (!neg) {
        fe4_blend(U, d, s, 2);                             /* (E, G, F, E) */
        fe4_perm(sp, s, FE4_PERM_IMM(0, 0, 2, 3)); fe4_perm(dp, d, FE4_PERM_IMM(1, 1, 1, 1));
        fe4_blend(V, sp, dp, 1);                           /* (F, H, G, H) */
    } else {
        fe4_blend(U, d, s, 4);                             /* (E, G, F, E) with F = D'+C', G = D'-C' */
        fe4_perm(sp, s, FE4_PERM_IMM(1, 0, 2, 3));         /* (F, H, F, H) */
        fe4_blend(V, sp, d, 4);                            /* (F, H, G, H) */
    }
    gx r; r.p = fe4_mul(U, V);                             /* (EF, GH, FG, EH) */
    return r;
}
static gx gx_dbl(const gx *P) {
    fe4 S, Yl, Q, t0, t1, Yb, Zb, W, W2, zz, sub, D, Dp, Tb, U, V, z = fe4_zero();
    fe4_perm(S, P->p, FE4_PERM_IMM(0, 1, 2, 0));
    fe4_perm(Yl, P->p, FE4_PERM_IMM(1, 1, 1, 1)); fe4_blend(Yl, z, Yl, 8);
    S = fe4_reduce(fe4_add(S, Yl));                        /* (X, Y, Z, X+Y) */
    Q = fe4_sq(S);                                         /* (XX, YY, ZZ, (X+Y)^2) */
    fe4_perm(t0, Q, FE4_PERM_IMM(0, 0, 0, 0)); fe4_perm(t1, Q, FE4_PERM_IMM(1, 1, 1, 1));
    Yb = fe4_reduce(fe4_add(t1, t0));                      /* YY + XX in every lane */
    Zb = fe4_reduce(fe4_sub(t1, t0));                      /* YY - XX */
    fe4_perm(W, Q, FE4_PERM_IMM(3, 3, 2, 2));              /* ((X+Y)^2, (X+Y)^2, ZZ, ZZ) */
    fe4_blend(zz, z, W, 12);
    W2 = fe4_add(W, zz);                                   /* (.., .., 2ZZ, 2ZZ) */
    fe4_blend(sub, Yb, Zb, 12);                            /* (Y3, Y3, Z3, Z3) completed coordinates */
    D = fe4_reduce(fe4_sub(W2, sub));                      /* (X3, X3, T3, T3) */
    fe4_perm(Dp, D, FE4_PERM_IMM(0, 0, 2, 0)); fe4_perm(Tb, D, FE4_PERM_IMM(2, 2, 2, 2));
    fe4_blend(U, Dp, Yb, 2); fe4_blend(U, U, Zb, 4);       /* (X3, Y3, Z3, X3) */
    fe4_blend(V, Tb, Zb, 2); fe4_blend(V, V, Yb, 8);       /* (T3, Z3, T3, Y3) */
    gx r; r.p = fe4_mul(U, V);                             /* (X3 T3, Y3 Z3, Z3 T3, X3 Y3) */
    return r;
}
static gx gx_add(const gx *P, const gx *Q) { gcv c = gx_to_cached(Q); return gx_add_cached(P, &c, 0); }

static void VEC_NAME(vec_init)(void) {
    if (VEC_NAME(k_ready)) return;
    ge_init_constants();
    fe one; fe_1(&one);
    VEC_NAME(K_D2LANE) = fe4_pack(&one, &one, &one, &GE_D);
    VEC_NAME(k_ready) = 1;
}

static gcv gcv_neg(const gcv *c) {                 /* (Y-X, Y+X, 2Z, 2dT) of -Q: swap the first two lanes, negate the last */
    fe4 sw, ng, r;
    fe4_perm(sw, c->c, FE4_PERM_IMM(1, 0, 2, 3));
    ng = fe4_sub(fe4_zero(), sw);
    fe4_blend(r, sw, ng, 8);
    gcv o; o.c = fe4_reduce(r); return o;
}
/* Straus (n < 190): per-point tables of the odd multiples +-P, +-3P, .., +-15P in cached form, width-5 NAF digits, shared
 * doublings.  One point addition is a single dependency chain of ~430 vector instructions, so the sum is kept in TWO
 * accumulators (even / odd non-zero digits of a bit position) whose additions and doublings are issued side by side: the
 * out-of-order core overlaps the two chains.  Signed table slots keep the paired additions free of data-dependent branches. */
static void VEC_NAME(msm_straus)(ge *out, const sc *scalars, const ge *points, size_t n) {
    int8_t (*nafs)[256] = malloc(n * 256);
    gcv (*tables)[16] = aligned_alloc(64, (n * sizeof *tables + 63) / 64 * 64);
    for (size_t k = 0; k < n; k++) {
        sc_naf(nafs[k], &scalars[k], 5);
        gx cur = gx_from_ge(&points[k]), p2 = gx_dbl(&cur);
        gcv c2 = gx_to_cached(&p2);
        tables[k][0] = gx_to_cached(&cur);
        for (int j = 1; j < 8; j++) { cur = gx_add_cached(&cur, &c2, 0); tables[k][j] = gx_to_cached(&cur); }
        for (int j = 0; j < 8; j++) tables[k][8 + j] = gcv_neg(&tables[k][j]);
    }
    gx r1 = gx_identity(), r2 = gx_identity();
    const gcv *todo[192];
    int started = 0;
    for (int i = 255; i >= 0; i--) {
        if (started) { gx d1 = gx_dbl(&r1), d2 = gx_dbl(&r2); r1 = d1; r2 = d2; }
        int m = 0;
        for (size_t k = 0; k < n; k++) { int d = nafs[k][i]; if (d) todo[m++] = &tables[k][d > 0 ? d / 2 : 8 + (-d) / 2]; }
        if (m) started = 1;
        int e = 0;
        for (; e + 1 < m; e += 2) { gx a1 = gx_add_cached(&r1, todo[e], 0), a2 = gx_add_cached(&r2, todo[e + 1], 0); r1 = a1; r2 = a2; }
        if (e < m) r1 = gx_add_cached(&r1, todo[e], 0);
    }
    r1 = gx_add(&r1, &r2);
    gx_to_ge(out, &r1);
    free(nafs); free(tables);
}

static void VEC_NAME(msm_pippenger)(ge *out, const sc *scalars, const ge *points, size_t n) {
    int w = n < 500 ? 6 : n < 800 ? 7 : 8;
    int nb = 1 << (w - 1);
    int8_t (*digits)[44] = malloc(n * 44);
    gcv *cached = aligned_alloc(64, (n * sizeof *cached + 63) / 64 * 64);
    gx *buckets = aligned_alloc(64, ((size_t)nb * sizeof *buckets + 63) / 64 * 64);
    int count = 0;
    for (size_t k = 0; k < n; k++) { memset(digits[k], 0, 44); count = sc_radix_2w(digits[k], &scalars[k], w); gx p = gx_from_ge(&points[k]); cached[k] = gx_to_cached(&p); }
    gx total = gx_identity();
    for (int col = count - 1; col >= 0; col--) {
        for (int b = 0; b < nb; b++) buckets[b] = gx_identity();
        for (size_t k = 0; k < n; k++) {
            int d = digits[k][col];
            if (d > 0) buckets[d - 1] = gx_add_cached(&buckets[d - 1], &cached[k], 0);
            else if (d < 0) buckets[-d - 1] = gx_add_cached(&buckets[-d - 1], &cached[k], 1);
        }
        gx run = buckets[nb - 1], sum = buckets[nb - 1];
        for (int b = nb - 2; b >= 0; b--) { run = gx_add(&run, &buckets[b]); sum = gx_add(&sum, &run); }
        for (int j = 0; j < w; j++) total = gx_dbl(&total);
        total = gx_add(&total, &sum);
    }
    gx_to_ge(out, &total);
    free(digits); free(cached); free(buckets);
}

/* exported entry: same contract as ge_msm_vartime (ge.h) */
void VEC_NAME(orc_vec_msm)(ge *out, const sc *scalars, const ge *points, size_t n) {
    VEC_NAME(vec_init)();
    if (n == 0) { ge_identity(out); return; }
    if (n < 190) VEC_NAME(msm_straus)(out, scalars, points, n); else VEC_NAME(msm_pippenger)(out, scalars, points, n);
}
const char *VEC_NAME(orc_vec_name)(void) { return VEC_BACKEND_NAME; }

/* self-test of the vector field and point operations against the scalar backend; returns 0 on success */
int VEC_NAME(orc_vec_selftest)(const uint8_t *seed_points /* 4 x 32 B compressed */, const uint8_t *rnd /* 8 x 32 B */) {
    VEC_NAME(vec_init)();
    fe a[4], b[4], r[4], e;
    for (int j = 0; j < 4; j++) { fe_frombytes(&a[j], rnd + 32 * j); fe_frombytes(&b[j], rnd + 32 * (4 + j)); }
    fe4 A = fe4_pack(&a[0], &a[1], &a[2], &a[3]), B = fe4_pack(&b[0], &b[1], &b[2], &b[3]), R;
    R = fe4_mul(A, B); fe4_unpack(r, &R);
    for (int j = 0; j < 4; j++) { fe_mul(&e, &a[j], &b[j]); if (!fe_eq(&e, &r[j])) return 1; }
    R = fe4_sq(A); fe4_unpack(r, &R);
    for (int j = 0; j < 4; j++) { fe_sq(&e, &a[j]); if (!fe_eq(&e, &r[j])) return 2; }
    R = fe4_reduce(fe4_add(A, B)); fe4_unpack(r, &R);
    for (int j = 0; j < 4; j++) { fe_add(&e, &a[j], &b[j]); if (!fe_eq(&e, &r[j])) return 3; }
    R = fe4_reduce(fe4_sub(A, B)); fe4_unpack(r, &R);
    for (int j = 0; j < 4; j++) { fe_sub(&e, &a[j], &b[j]); if (!fe_eq(&e, &r[j])) return 4; }
    R = fe4_mul(fe4_reduce(fe4_sub(A, B)), fe4_reduce(fe4_add(A, B))); fe4_unpack(r, &R);
    for (int j = 0; j < 4; j++) { fe s_, d_; fe_add(&s_, &a[j], &b[j]); fe_sub(&d_, &a[j], &b[j]); fe_mul(&e, &s_, &d_); if (!fe_eq(&e, &r[j])) return 5; }
    ge p[4];
    for (int j = 0; j < 4; j++) if (!ge_decode(&p[j], seed_points + 32 * j)) return 10;
    for (int j = 0; j < 4; j++) {
        gx P = gx_from_ge(&p[j]), Q = gx_from_ge(&p[(j + 1) & 3]);
        ge want, got; uint8_t w[32], g[32];
        gx D = gx_dbl(&P); gx_to_ge(&got, &D); ge_dbl(&want, &p[j]); ge_encode(w, &want); ge_encode(g, &got); if (memcmp(w, g, 32)) return 11;
        { fe t; fe_mul(&t, &got.X, &got.Y); fe u; fe_mul(&u, &got.Z, &got.T); if (!fe_eq(&t, &u)) return 12; }      /* T Z = X Y */
        gx S = gx_add(&P, &Q); gx_to_ge(&got, &S); ge_add(&want, &p[j], &p[(j + 1) & 3]); ge_encode(w, &want); ge_encode(g, &got); if (memcmp(w, g, 32)) return 13;
        gcv c = gx_to_cached(&Q); gx M = gx_add_cached(&P, &c, 1); gx_to_ge(&got, &M); ge_sub(&want, &p[j], &p[(j + 1) & 3]); ge_encode(w, &want); ge_encode(g, &got); if (memcmp(w, g, 32)) return 14;
        { fe t; fe_mul(&t, &got.X, &got.Y); fe u; fe_mul(&u, &got.Z, &got.T); if (!fe_eq(&t, &u)) return 15; }
        gx I = gx_identity(); gx Z = gx_add_cached(&I, &c, 0); gx_to_ge(&got, &Z); ge_encode(g, &got); ge_encode(w, &p[(j + 1) & 3]); if (memcmp(w, g, 32)) return 16;
    }
    return 0;
}
