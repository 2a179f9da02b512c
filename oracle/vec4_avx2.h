/* ORACLE (test infrastructure only — never linked into the product path).
 *
 * Four field elements mod p = 2^255 - 19 side by side in the 64-bit lanes of 256-bit vectors, ten limbs of alternately 26
 * and 25 bits (the classic radix-2^25.5 form), products with vpmuludq (32x32 -> 64 per lane).  This is the CPU restatement
 * of the 4-way AVX2 vector backend that the reference enables by default (`default = ["std", "avx2_backend"]`,
 * Cargo.toml:41-42; 1040 us vs 1490 us per 64-bit verification, README.md:76-77) through
 * curve25519-dalek (un-vendored dependency, Cargo.toml:21).  Published design: one vector operation works on the four
 * coordinates of an extended point (HWCD'08 section 3.1); the limb schedule below is written from scratch for this oracle
 * (one limb per vector, low 32 bits of each 64-bit lane used) rather than dalek's packed 5-vector layout.
 * Lane j of v[i] holds limb i of element j.
 *
 * Bounds: a "reduced" element has even limbs < 2^26 + 2^13 and odd limbs < 2^25 + 2^13.  fe4_mul / fe4_sq need limbs < 2^27
 * (19 * limb and 2 * limb must fit 32 bits; ten 64-bit products per column must not overflow): sums and differences go
 * through fe4_reduce first.
 */
#ifndef ORACLE_VEC4_AVX2_H
#define ORACLE_VEC4_AVX2_H
#include <immintrin.h>
#include "fe51.h"

#define VEC_NAME(x) x##_avx2
#define VEC_BACKEND_NAME "avx2 (4x 25.5-bit limbs, vpmuludq)"

typedef struct { __m256i v[10]; } fe4;

static inline fe4 fe4_pack(const fe *a, const fe *b, const fe *c, const fe *d) {
    fe4 r; const fe *e[4] = {a, b, c, d};
    uint64_t t[10][4];
    for (int j = 0; j < 4; j++) {
        fe w = *e[j]; fe_weak_reduce(&w);                                    /* limbs < 2^51 + small */
        for (int k = 0; k < 5; k++) { t[2 * k][j] = w.v[k] & ((1ULL << 26) - 1); t[2 * k + 1][j] = w.v[k] >> 26; }
    }
    for (int i = 0; i < 10; i++) r.v[i] = _mm256_loadu_si256((const __m256i *)t[i]);
    return r;
}
static inline void fe4_unpack(fe out[4], const fe4 *x) {
    uint64_t t[10][4];
    for (int i = 0; i < 10; i++) _mm256_storeu_si256((__m256i *)t[i], x->v[i]);
    for (int j = 0; j < 4; j++) {
        for (int k = 0; k < 5; k++) out[j].v[k] = t[2 * k][j] + (t[2 * k + 1][j] << 26);
        fe_weak_reduce(&out[j]);
    }
}
static inline fe4 fe4_add(fe4 a, fe4 b) { fe4 r; for (int i = 0; i < 10; i++) r.v[i] = _mm256_add_epi64(a.v[i], b.v[i]); return r; }
/* a + 2p - b (NOT reduced) */
static inline fe4 fe4_sub(fe4 a, fe4 b) {
    const __m256i p0 = _mm256_set1_epi64x(0x7ffffda), pe = _mm256_set1_epi64x(0x7fffffe), po = _mm256_set1_epi64x(0x3fffffe);   /* 2*(2^26-19), 2*(2^26-1), 2*(2^25-1) */
    fe4 r;
    r.v[0] = _mm256_sub_epi64(_mm256_add_epi64(a.v[0], p0), b.v[0]);
    for (int i = 1; i < 10; i++) r.v[i] = _mm256_sub_epi64(_mm256_add_epi64(a.v[i], (i & 1) ? po : pe), b.v[i]);
    return r;
}
static inline __m256i fe4_mul19(__m256i x) { return _mm256_add_epi64(_mm256_add_epi64(_mm256_slli_epi64(x, 4), _mm256_slli_epi64(x, 1)), x); }
/* PARALLEL carry passes (all ten carries taken at once; see vec4_ifma.h for why): one pass brings inputs < 2^37 to limbs
 * < 2^26 + 2^12; the 64-bit column sums of a product (< 2^63) need two */
static inline fe4 fe4_carry_pass(fe4 a) {
    const __m256i m26 = _mm256_set1_epi64x((1LL << 26) - 1), m25 = _mm256_set1_epi64x((1LL << 25) - 1);
    __m256i c[10];
    for (int i = 0; i < 10; i++) c[i] = _mm256_srli_epi64(a.v[i], (i & 1) ? 25 : 26);
    fe4 r;
    r.v[0] = _mm256_add_epi64(_mm256_and_si256(a.v[0], m26), fe4_mul19(c[9]));
    for (int i = 1; i < 10; i++) r.v[i] = _mm256_add_epi64(_mm256_and_si256(a.v[i], (i & 1) ? m25 : m26), c[i - 1]);
    return r;
}
static inline fe4 fe4_reduce(fe4 a) { return fe4_carry_pass(a); }                       /* after add / sub: inputs < 2^29 */
static inline fe4 fe4_reduce_wide(fe4 a) { return fe4_carry_pass(fe4_carry_pass(a)); }   /* product columns */
/* h_k = sum_{i+j=k} f_i g_j [x2 if i, j both odd] + 19 sum_{i+j=k+10} f_i g_j [x2 if both odd];  inputs: limbs < 2^27 */
static inline fe4 fe4_mul(fe4 f, fe4 g) {
    __m256i g19[10], f2[10], h[10];
    for (int j = 1; j < 10; j++) g19[j] = fe4_mul19(g.v[j]);
    for (int i = 1; i < 10; i += 2) f2[i] = _mm256_slli_epi64(f.v[i], 1);
    for (int k = 0; k < 10; k++) h[k] = _mm256_setzero_si256();
    for (int i = 0; i < 10; i++)
        for (int j = 0; j < 10; j++) {
            int k = i + j;
            __m256i a = ((i & 1) && (j & 1)) ? f2[i] : f.v[i];
            __m256i b = k >= 10 ? g19[j] : g.v[j];
            h[k >= 10 ? k - 10 : k] = _mm256_add_epi64(h[k >= 10 ? k - 10 : k], _mm256_mul_epu32(a, b));
        }
    fe4 r; for (int k = 0; k < 10; k++) r.v[k] = h[k];
    return fe4_reduce_wide(r);
}
static inline fe4 fe4_sq(fe4 f) {
    __m256i f19[10], f2[10], h[10];
    for (int j = 1; j < 10; j++) f19[j] = fe4_mul19(f.v[j]);
    for (int i = 0; i < 10; i++) f2[i] = _mm256_slli_epi64(f.v[i], 1);
    for (int k = 0; k < 10; k++) h[k] = _mm256_setzero_si256();
    for (int i = 0; i < 10; i++) {
        {   /* diagonal */
            int k = 2 * i;
            __m256i a = (i & 1) ? f2[i] : f.v[i];
            __m256i b = k >= 10 ? f19[i] : f.v[i];
            h[k >= 10 ? k - 10 : k] = _mm256_add_epi64(h[k >= 10 ? k - 10 : k], _mm256_mul_epu32(a, b));
        }
        for (int j = i + 1; j < 10; j++) {          /* off-diagonal, taken twice: 2 f_i (x2 again if both odd -> 4 f_i, via f2 on both sides) */
            int k = i + j;
            __m256i a = f2[i];
            __m256i b = k >= 10 ? f19[j] : f.v[j];
            if ((i & 1) && (j & 1)) b = _mm256_slli_epi64(b, 1);
            h[k >= 10 ? k - 10 : k] = _mm256_add_epi64(h[k >= 10 ? k - 10 : k], _mm256_mul_epu32(a, b));
        }
    }
    fe4 r; for (int k = 0; k < 10; k++) r.v[k] = h[k];
    return fe4_reduce_wide(r);
}
#define FE4_PERM_IMM(l0, l1, l2, l3) ((l0) | ((l1) << 2) | ((l2) << 4) | ((l3) << 6))
#define fe4_perm(r, a, imm) do { for (int i_ = 0; i_ < 10; i_++) (r).v[i_] = _mm256_permute4x64_epi64((a).v[i_], (imm)); } while (0)
#define FE4_BLEND_IMM(mask4) ((((mask4) & 1) ? 0x03 : 0) | (((mask4) & 2) ? 0x0c : 0) | (((mask4) & 4) ? 0x30 : 0) | (((mask4) & 8) ? 0xc0 : 0))
#define fe4_blend(r, a, b, mask4) do { for (int i_ = 0; i_ < 10; i_++) (r).v[i_] = _mm256_blend_epi32((a).v[i_], (b).v[i_], FE4_BLEND_IMM(mask4)); } while (0)
static inline fe4 fe4_zero(void) { fe4 r; for (int i = 0; i < 10; i++) r.v[i] = _mm256_setzero_si256(); return r; }
#define FE4_LIMBS 10
#endif
