/* ORACLE (test infrastructure only — never linked into the product path).
 *
 * Four field elements mod p = 2^255 - 19 side by side in the 64-bit lanes of 256-bit vectors, radix 2^51, products with
 * the AVX-512 IFMA instructions (vpmadd52luq / vpmadd52huq on ymm: AVX512IFMA + AVX512VL).  This is the CPU restatement of
 * the 4-way "ifma" vector backend that curve25519-dalek (un-vendored dependency, Cargo.toml:21,41-42; the
 * speed-up is quoted in README.md:82-84) selects on hosts with IFMA: the published design — one vector
 * operation works on the four coordinates of an extended point (HWCD'08 section 3.1, 4-processor formulas) — written from
 * scratch for this oracle.  Lane j of v[i] holds limb i of element j.
 *
 * Bounds: a "reduced" element has limbs < 2^51 + 2^15 (one parallel carry pass); vpmadd52 reads only the low 52 bits of its operands, so everything
 * fed to fe4_mul / fe4_sq must have limbs < 2^52: sums and differences are passed through fe4_reduce first.
 */
#ifndef ORACLE_VEC4_IFMA_H
#define ORACLE_VEC4_IFMA_H
#include <immintrin.h>
#include "fe51.h"

#define VEC_NAME(x) x##_ifma
#define VEC_BACKEND_NAME "avx512ifma (4x 51-bit limbs, vpmadd52)"

typedef struct { __m256i v[5]; } fe4;

static inline fe4 fe4_pack(const fe *a, const fe *b, const fe *c, const fe *d) {
    fe4 r;
    for (int i = 0; i < 5; i++) r.v[i] = _mm256_set_epi64x((long long)d->v[i], (long long)c->v[i], (long long)b->v[i], (long long)a->v[i]);
    return r;
}
static inline void fe4_unpack(fe out[4], const fe4 *x) {
    for (int i = 0; i < 5; i++) {
        uint64_t t[4]; _mm256_storeu_si256((__m256i *)t, x->v[i]);
        out[0].v[i] = t[0]; out[1].v[i] = t[1]; out[2].v[i] = t[2]; out[3].v[i] = t[3];
    }
}
static inline fe4 fe4_add(fe4 a, fe4 b) { fe4 r; for (int i = 0; i < 5; i++) r.v[i] = _mm256_add_epi64(a.v[i], b.v[i]); return r; }
/* a + 2p - b: limbs stay positive for reduced a, b; the result is NOT reduced */
static inline fe4 fe4_sub(fe4 a, fe4 b) {
    const __m256i p0 = _mm256_set1_epi64x(0xfffffffffffdaLL), pi = _mm256_set1_epi64x(0xffffffffffffeLL);   /* 2*(2^51-19), 2*(2^51-1) */
    fe4 r;
    r.v[0] = _mm256_sub_epi64(_mm256_add_epi64(a.v[0], p0), b.v[0]);
    for (int i = 1; i < 5; i++) r.v[i] = _mm256_sub_epi64(_mm256_add_epi64(a.v[i], pi), b.v[i]);
    return r;
}
static inline __m256i fe4_mul19(__m256i x) { return _mm256_add_epi64(_mm256_add_epi64(_mm256_slli_epi64(x, 4), _mm256_slli_epi64(x, 1)), x); }
/* one PARALLEL carry pass (all five carries taken at once: depth 3 instead of a 5-step ripple; the adds and the two vector
 * multiplications of a point addition form one long dependency chain, so latency is what matters): for inputs < 2^61 every
 * limb ends below 2^51 + 2^10 (limb 0: + 19 * 2^10 < 2^51 + 2^15) -- weakly reduced, which is all the callers need */
static inline fe4 fe4_reduce(fe4 a) {
    const __m256i mask = _mm256_set1_epi64x((1LL << 51) - 1);
    __m256i c0 = _mm256_srli_epi64(a.v[0], 51), c1 = _mm256_srli_epi64(a.v[1], 51), c2 = _mm256_srli_epi64(a.v[2], 51),
            c3 = _mm256_srli_epi64(a.v[3], 51), c4 = _mm256_srli_epi64(a.v[4], 51);
    fe4 r;
    r.v[0] = _mm256_add_epi64(_mm256_and_si256(a.v[0], mask), fe4_mul19(c4));
    r.v[1] = _mm256_add_epi64(_mm256_and_si256(a.v[1], mask), c0);
    r.v[2] = _mm256_add_epi64(_mm256_and_si256(a.v[2], mask), c1);
    r.v[3] = _mm256_add_epi64(_mm256_and_si256(a.v[3], mask), c2);
    r.v[4] = _mm256_add_epi64(_mm256_and_si256(a.v[4], mask), c3);
    return r;
}
/* columns col[0..9] of the 10-limb product -> 5 limbs: fold with 2^255 = 19, carry */
static inline fe4 fe4_fold(const __m256i lo[9], const __m256i hi[9]) {
    __m256i col[10];
    col[0] = lo[0];
    for (int k = 1; k < 9; k++) col[k] = _mm256_add_epi64(lo[k], _mm256_slli_epi64(hi[k - 1], 1));     /* hi parts weigh 2^52 = 2 * 2^51 */
    col[9] = _mm256_slli_epi64(hi[8], 1);
    fe4 r;
    for (int k = 0; k < 5; k++) r.v[k] = _mm256_add_epi64(col[k], fe4_mul19(col[k + 5]));
    return fe4_reduce(r);
}
/* inputs: limbs < 2^52; output reduced */
static inline fe4 fe4_mul(fe4 a, fe4 b) {
    __m256i lo[9], hi[9];
    const __m256i z = _mm256_setzero_si256();
    for (int k = 0; k < 9; k++) { lo[k] = z; hi[k] = z; }
    for (int i = 0; i < 5; i++)
        for (int j = 0; j < 5; j++) {
            lo[i + j] = _mm256_madd52lo_epu64(lo[i + j], a.v[i], b.v[j]);
            hi[i + j] = _mm256_madd52hi_epu64(hi[i + j], a.v[i], b.v[j]);
        }
    return fe4_fold(lo, hi);
}
static inline fe4 fe4_sq(fe4 a) {
    __m256i lo[9], hi[9], dl[9], dh[9];
    const __m256i z = _mm256_setzero_si256();
    for (int k = 0; k < 9; k++) { lo[k] = z; hi[k] = z; dl[k] = z; dh[k] = z; }
    for (int i = 0; i < 5; i++) {
        dl[2 * i] = _mm256_madd52lo_epu64(dl[2 * i], a.v[i], a.v[i]);
        dh[2 * i] = _mm256_madd52hi_epu64(dh[2 * i], a.v[i], a.v[i]);
        for (int j = i + 1; j < 5; j++) {
            lo[i + j] = _mm256_madd52lo_epu64(lo[i + j], a.v[i], a.v[j]);
            hi[i + j] = _mm256_madd52hi_epu64(hi[i + j], a.v[i], a.v[j]);
        }
    }
    for (int k = 0; k < 9; k++) { lo[k] = _mm256_add_epi64(_mm256_slli_epi64(lo[k], 1), dl[k]); hi[k] = _mm256_add_epi64(_mm256_slli_epi64(hi[k], 1), dh[k]); }
    return fe4_fold(lo, hi);
}
/* lane permutation / blend; PERM(a,b,c,d) = result lane 0 <- source lane a, ... */
#define FE4_PERM_IMM(l0, l1, l2, l3) ((l0) | ((l1) << 2) | ((l2) << 4) | ((l3) << 6))
#define fe4_perm(r, a, imm) do { for (int i_ = 0; i_ < 5; i_++) (r).v[i_] = _mm256_permute4x64_epi64((a).v[i_], (imm)); } while (0)
/* lanes with their bit set in mask4 come from b */
#define FE4_BLEND_IMM(mask4) ((((mask4) & 1) ? 0x03 : 0) | (((mask4) & 2) ? 0x0c : 0) | (((mask4) & 4) ? 0x30 : 0) | (((mask4) & 8) ? 0xc0 : 0))
#define fe4_blend(r, a, b, mask4) do { for (int i_ = 0; i_ < 5; i_++) (r).v[i_] = _mm256_blend_epi32((a).v[i_], (b).v[i_], FE4_BLEND_IMM(mask4)); } while (0)
static inline fe4 fe4_zero(void) { fe4 r; for (int i = 0; i < 5; i++) r.v[i] = _mm256_setzero_si256(); return r; }
#define FE4_LIMBS 5
#endif
