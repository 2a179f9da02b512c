/* ORACLE (test infrastructure only).
 *
 * Keccak-f[1600], SHAKE256, SHA3-512, the Merlin v1.0 transcript over STROBE-128, and the
 * ChaCha20 stream used as `rand_chacha::ChaChaRng`.  These live in un-vendored dependencies of
 * the reference (merlin = "2", sha3 = "0.8", rand_chacha = "0.2"; Cargo.toml:23,31,38);
 * this file restates the published constructions.  Call sites pinned:
 *   - SHAKE256 generator chain      src/generators.rs:62-104
 *   - SHA3-512 hash-to-group (B~)   src/generators.rs:44-53
 *   - Merlin labels / framing       src/transcript.rs:43-94
 *   - ChaChaRng::from_seed([24;32]) tests/range_proof.rs:108-113
 */
#ifndef ORACLE_HASHES_H
#define ORACLE_HASHES_H
#include <stdint.h>
#include <string.h>

static inline uint64_t rotl64(uint64_t x, int n) { return n ? (x << n) | (x >> (64 - n)) : x; }

static void keccak_f1600(uint64_t st[25]) {
    static const uint64_t RC[24] = {
        0x0000000000000001ULL, 0x0000000000008082ULL, 0x800000000000808aULL, 0x8000000080008000ULL,
        0x000000000000808bULL, 0x0000000080000001ULL, 0x8000000080008081ULL, 0x8000000000008009ULL,
        0x000000000000008aULL, 0x0000000000000088ULL, 0x0000000080008009ULL, 0x000000008000000aULL,
        0x000000008000808bULL, 0x800000000000008bULL, 0x8000000000008089ULL, 0x8000000000008003ULL,
        0x8000000000008002ULL, 0x8000000000000080ULL, 0x000000000000800aULL, 0x800000008000000aULL,
        0x8000000080008081ULL, 0x8000000000008080ULL, 0x0000000080000001ULL, 0x8000000080008008ULL };
    static const int ROT[25] = { 0, 1, 62, 28, 27, 36, 44, 6, 55, 20, 3, 10, 43, 25, 39,
                                 41, 45, 15, 21, 8, 18, 2, 61, 56, 14 };   /* index x + 5y */
    for (int round = 0; round < 24; round++) {
        uint64_t C[5], D[5], B[25];
        for (int x = 0; x < 5; x++) C[x] = st[x] ^ st[x + 5] ^ st[x + 10] ^ st[x + 15] ^ st[x + 20];
        for (int x = 0; x < 5; x++) D[x] = C[(x + 4) % 5] ^ rotl64(C[(x + 1) % 5], 1);
        for (int i = 0; i < 25; i++) st[i] ^= D[i % 5];
        /* rho + pi: B[y, 2x+3y] = rot(A[x,y]) */
        for (int x = 0; x < 5; x++)
            for (int y = 0; y < 5; y++)
                B[y + 5 * ((2 * x + 3 * y) % 5)] = rotl64(st[x + 5 * y], ROT[x + 5 * y]);
        for (int y = 0; y < 5; y++)
            for (int x = 0; x < 5; x++)
                st[x + 5 * y] = B[x + 5 * y] ^ (~B[(x + 1) % 5 + 5 * y] & B[(x + 2) % 5 + 5 * y]);
        st[0] ^= RC[round];
    }
}

/* generic sponge (byte-oriented, little-endian host assumed) */
typedef struct { uint64_t st[25]; int rate, pos; uint8_t pad; int squeezing; } sponge;

static inline void sponge_init(sponge *s, int rate, uint8_t pad) {
    memset(s, 0, sizeof *s); s->rate = rate; s->pad = pad;
}
static inline void sponge_absorb(sponge *s, const uint8_t *in, size_t len) {
    uint8_t *b = (uint8_t *)s->st;
    for (size_t i = 0; i < len; i++) {
        b[s->pos++] ^= in[i];
        if (s->pos == s->rate) { keccak_f1600(s->st); s->pos = 0; }
    }
}
static inline void sponge_squeeze(sponge *s, uint8_t *out, size_t len) {
    uint8_t *b = (uint8_t *)s->st;
    if (!s->squeezing) {
        b[s->pos] ^= s->pad; b[s->rate - 1] ^= 0x80;
        keccak_f1600(s->st); s->pos = 0; s->squeezing = 1;
    }
    for (size_t i = 0; i < len; i++) {
        if (s->pos == s->rate) { keccak_f1600(s->st); s->pos = 0; }
        out[i] = b[s->pos++];
    }
}
static inline void shake256_init(sponge *s) { sponge_init(s, 136, 0x1f); }
static inline void sha3_512(uint8_t out[64], const uint8_t *in, size_t len) {
    sponge s; sponge_init(&s, 72, 0x06); sponge_absorb(&s, in, len); sponge_squeeze(&s, out, 64);
}

/* ---------------- Merlin v1.0 over STROBE-128 (rate 166) ---------------- */
#define STROBE_R 166
enum { FLAG_I = 1, FLAG_A = 2, FLAG_C = 4, FLAG_T = 8, FLAG_M = 16, FLAG_K = 32 };
typedef struct { uint8_t st[200]; uint8_t pos, pos_begin, cur_flags; } merlin;

static inline void strobe_run_f(merlin *m) {
    m->st[m->pos] ^= m->pos_begin;
    m->st[m->pos + 1] ^= 0x04;
    m->st[STROBE_R + 1] ^= 0x80;
    uint64_t w[25]; memcpy(w, m->st, 200); keccak_f1600(w); memcpy(m->st, w, 200);
    m->pos = 0; m->pos_begin = 0;
}
static inline void strobe_absorb(merlin *m, const uint8_t *d, size_t n) {
    for (size_t i = 0; i < n; i++) { m->st[m->pos++] ^= d[i]; if (m->pos == STROBE_R) strobe_run_f(m); }
}
static inline void strobe_overwrite(merlin *m, const uint8_t *d, size_t n) {
    for (size_t i = 0; i < n; i++) { m->st[m->pos++] = d[i]; if (m->pos == STROBE_R) strobe_run_f(m); }
}
static inline void strobe_squeeze(merlin *m, uint8_t *d, size_t n) {
    for (size_t i = 0; i < n; i++) { d[i] = m->st[m->pos]; m->st[m->pos++] = 0; if (m->pos == STROBE_R) strobe_run_f(m); }
}
static inline void strobe_begin_op(merlin *m, uint8_t flags, int more) {
    if (more) return;
    uint8_t old = m->pos_begin;
    m->pos_begin = m->pos + 1;
    m->cur_flags = flags;
    uint8_t hdr[2] = { old, flags };
    strobe_absorb(m, hdr, 2);
    if ((flags & (FLAG_C | FLAG_K)) && m->pos != 0) strobe_run_f(m);
}
static inline void strobe_meta_ad(merlin *m, const uint8_t *d, size_t n, int more) { strobe_begin_op(m, FLAG_M | FLAG_A, more); strobe_absorb(m, d, n); }
static inline void strobe_ad(merlin *m, const uint8_t *d, size_t n, int more) { strobe_begin_op(m, FLAG_A, more); strobe_absorb(m, d, n); }
static inline void strobe_prf(merlin *m, uint8_t *d, size_t n, int more) { strobe_begin_op(m, FLAG_I | FLAG_A | FLAG_C, more); strobe_squeeze(m, d, n); }
static inline void strobe_key(merlin *m, const uint8_t *d, size_t n, int more) { strobe_begin_op(m, FLAG_A | FLAG_C, more); strobe_overwrite(m, d, n); }

static inline void merlin_append(merlin *m, const char *label, const uint8_t *msg, size_t len) {
    uint8_t l4[4] = { (uint8_t)len, (uint8_t)(len >> 8), (uint8_t)(len >> 16), (uint8_t)(len >> 24) };
    strobe_meta_ad(m, (const uint8_t *)label, strlen(label), 0);
    strobe_meta_ad(m, l4, 4, 1);
    strobe_ad(m, msg, len, 0);
}
static inline void merlin_init(merlin *m, const uint8_t *label, size_t len) {
    memset(m, 0, sizeof *m);
    static const uint8_t hdr[6] = { 1, STROBE_R + 2, 1, 0, 1, 96 };
    memcpy(m->st, hdr, 6); memcpy(m->st + 6, "STROBEv1.0.2", 12);
    uint64_t w[25]; memcpy(w, m->st, 200); keccak_f1600(w); memcpy(m->st, w, 200);
    strobe_meta_ad(m, (const uint8_t *)"Merlin v1.0", 11, 0);
    merlin_append(m, "dom-sep", label, len);
}
static inline void merlin_append_u64(merlin *m, const char *label, uint64_t x) {
    uint8_t b[8]; for (int i = 0; i < 8; i++) b[i] = (uint8_t)(x >> (8 * i));
    merlin_append(m, label, b, 8);
}
static inline void merlin_challenge(merlin *m, const char *label, uint8_t *out, size_t len) {
    uint8_t l4[4] = { (uint8_t)len, (uint8_t)(len >> 8), (uint8_t)(len >> 16), (uint8_t)(len >> 24) };
    strobe_meta_ad(m, (const uint8_t *)label, strlen(label), 0);
    strobe_meta_ad(m, l4, 4, 1);
    strobe_prf(m, out, len, 0);
}

/* ---------------- ChaCha20 keystream = rand_chacha ChaChaRng (64-bit counter, stream 0) -------- */
typedef struct { uint32_t key[8]; uint64_t counter; uint8_t buf[64]; int used; } chacha_rng;

static inline uint32_t rotl32(uint32_t x, int n) { return (x << n) | (x >> (32 - n)); }
#define CHACHA_QR(a, b, c, d) \
    a += b; d ^= a; d = rotl32(d, 16); c += d; b ^= c; b = rotl32(b, 12); \
    a += b; d ^= a; d = rotl32(d, 8);  c += d; b ^= c; b = rotl32(b, 7);
static inline void chacha_block(chacha_rng *r) {
    uint32_t in[16] = { 0x61707865, 0x3320646e, 0x79622d32, 0x6b206574 }, x[16];
    memcpy(in + 4, r->key, 32);
    in[12] = (uint32_t)r->counter; in[13] = (uint32_t)(r->counter >> 32); in[14] = 0; in[15] = 0;
    memcpy(x, in, 64);
    for (int i = 0; i < 10; i++) {
        CHACHA_QR(x[0], x[4], x[8], x[12]) CHACHA_QR(x[1], x[5], x[9], x[13])
        CHACHA_QR(x[2], x[6], x[10], x[14]) CHACHA_QR(x[3], x[7], x[11], x[15])
        CHACHA_QR(x[0], x[5], x[10], x[15]) CHACHA_QR(x[1], x[6], x[11], x[12])
        CHACHA_QR(x[2], x[7], x[8], x[13]) CHACHA_QR(x[3], x[4], x[9], x[14])
    }
    for (int i = 0; i < 16; i++) x[i] += in[i];
    memcpy(r->buf, x, 64); r->counter++; r->used = 0;
}
static inline void chacha_seed(chacha_rng *r, const uint8_t seed[32]) {
    memcpy(r->key, seed, 32); r->counter = 0; r->used = 64;
}
static inline void chacha_fill(chacha_rng *r, uint8_t *out, size_t n) {
    for (size_t i = 0; i < n; i++) { if (r->used == 64) chacha_block(r); out[i] = r->buf[r->used++]; }
}
#endif
