// Keccak-f[1600] and the Merlin v1.0 / STROBE-128 transcript for device-side Fiat-Shamir replay.
//
// The reference replays the transcript on the host for every proof
// (src/range_proof/mod.rs:368-393, src/inner_product_proof.rs:213-222,
//  labels in src/transcript.rs:43-94) through the un-vendored `merlin = "2"` crate.
// Here one thread replays one proof's transcript so that a batch of proofs needs no host work
// between the H2D copy and the MSM (SURVEY.md §8(f) rank 1, kernel K6).
#pragma once
#include "fe.cuh"

BP_HD uint64_t bp_rotl64(uint64_t x, int n) { return (x << n) | (x >> (64 - n)); }

#define BP_KECCAK_RC_INIT {                                                                                  \
        0x0000000000000001ULL, 0x0000000000008082ULL, 0x800000000000808aULL, 0x8000000080008000ULL,       \
        0x000000000000808bULL, 0x0000000080000001ULL, 0x8000000080008081ULL, 0x8000000000008009ULL,       \
        0x000000000000008aULL, 0x0000000000000088ULL, 0x0000000080008009ULL, 0x000000008000000aULL,       \
        0x000000008000808bULL, 0x800000000000008bULL, 0x8000000000008089ULL, 0x8000000000008003ULL,       \
        0x8000000000008002ULL, 0x8000000000000080ULL, 0x000000000000800aULL, 0x800000008000000aULL,       \
        0x8000000080008081ULL, 0x8000000000008080ULL, 0x0000000080000001ULL, 0x8000000080008008ULL }
// the 24 rounds with the round constants at RC
BP_HD void keccak_rounds(uint64_t s[25], const uint64_t *RC) {
    uint64_t a00 = s[0], a01 = s[1], a02 = s[2], a03 = s[3], a04 = s[4], a05 = s[5], a06 = s[6], a07 = s[7], a08 = s[8], a09 = s[9],
             a10 = s[10], a11 = s[11], a12 = s[12], a13 = s[13], a14 = s[14], a15 = s[15], a16 = s[16], a17 = s[17], a18 = s[18], a19 = s[19],
             a20 = s[20], a21 = s[21], a22 = s[22], a23 = s[23], a24 = s[24];
    for (int r = 0; r < 24; r++) {
        // theta
        uint64_t c0 = a00 ^ a05 ^ a10 ^ a15 ^ a20, c1 = a01 ^ a06 ^ a11 ^ a16 ^ a21, c2 = a02 ^ a07 ^ a12 ^ a17 ^ a22,
                 c3 = a03 ^ a08 ^ a13 ^ a18 ^ a23, c4 = a04 ^ a09 ^ a14 ^ a19 ^ a24;
        uint64_t d0 = c4 ^ bp_rotl64(c1, 1), d1 = c0 ^ bp_rotl64(c2, 1), d2 = c1 ^ bp_rotl64(c3, 1), d3 = c2 ^ bp_rotl64(c4, 1), d4 = c3 ^ bp_rotl64(c0, 1);
        a00 ^= d0; a05 ^= d0; a10 ^= d0; a15 ^= d0; a20 ^= d0;
        a01 ^= d1; a06 ^= d1; a11 ^= d1; a16 ^= d1; a21 ^= d1;
        a02 ^= d2; a07 ^= d2; a12 ^= d2; a17 ^= d2; a22 ^= d2;
        a03 ^= d3; a08 ^= d3; a13 ^= d3; a18 ^= d3; a23 ^= d3;
        a04 ^= d4; a09 ^= d4; a14 ^= d4; a19 ^= d4; a24 ^= d4;
        // rho + pi: B[y][2x+3y] = rot(A[x][y]);  b<xy> below is B at index x + 5y
        uint64_t b00 = a00,                 b10 = bp_rotl64(a01, 1),   b20 = bp_rotl64(a02, 62),  b05 = bp_rotl64(a03, 28),  b15 = bp_rotl64(a04, 27);
        uint64_t b16 = bp_rotl64(a05, 36),  b01 = bp_rotl64(a06, 44),  b11 = bp_rotl64(a07, 6),   b21 = bp_rotl64(a08, 55),  b06 = bp_rotl64(a09, 20);
        uint64_t b07 = bp_rotl64(a10, 3),   b17 = bp_rotl64(a11, 10),  b02 = bp_rotl64(a12, 43),  b12 = bp_rotl64(a13, 25),  b22 = bp_rotl64(a14, 39);
        uint64_t b23 = bp_rotl64(a15, 41),  b08 = bp_rotl64(a16, 45),  b18 = bp_rotl64(a17, 15),  b03 = bp_rotl64(a18, 21),  b13 = bp_rotl64(a19, 8);
        uint64_t b14 = bp_rotl64(a20, 18),  b24 = bp_rotl64(a21, 2),   b09 = bp_rotl64(a22, 61),  b19 = bp_rotl64(a23, 56),  b04 = bp_rotl64(a24, 14);
        // chi
        a00 = b00 ^ (~b01 & b02); a01 = b01 ^ (~b02 & b03); a02 = b02 ^ (~b03 & b04); a03 = b03 ^ (~b04 & b00); a04 = b04 ^ (~b00 & b01);
        a05 = b05 ^ (~b06 & b07); a06 = b06 ^ (~b07 & b08); a07 = b07 ^ (~b08 & b09); a08 = b08 ^ (~b09 & b05); a09 = b09 ^ (~b05 & b06);
        a10 = b10 ^ (~b11 & b12); a11 = b11 ^ (~b12 & b13); a12 = b12 ^ (~b13 & b14); a13 = b13 ^ (~b14 & b10); a14 = b14 ^ (~b10 & b11);
        a15 = b15 ^ (~b16 & b17); a16 = b16 ^ (~b17 & b18); a17 = b17 ^ (~b18 & b19); a18 = b18 ^ (~b19 & b15); a19 = b19 ^ (~b15 & b16);
        a20 = b20 ^ (~b21 & b22); a21 = b21 ^ (~b22 & b23); a22 = b22 ^ (~b23 & b24); a23 = b23 ^ (~b24 & b20); a24 = b24 ^ (~b20 & b21);
        a00 ^= RC[r];
    }
    s[0] = a00; s[1] = a01; s[2] = a02; s[3] = a03; s[4] = a04; s[5] = a05; s[6] = a06; s[7] = a07; s[8] = a08; s[9] = a09;
    s[10] = a10; s[11] = a11; s[12] = a12; s[13] = a13; s[14] = a14; s[15] = a15; s[16] = a16; s[17] = a17; s[18] = a18; s[19] = a19;
    s[20] = a20; s[21] = a21; s[22] = a22; s[23] = a23; s[24] = a24;
}
BP_HD void keccak_f1600(uint64_t s[25]) {
    const uint64_t RC[24] = BP_KECCAK_RC_INIT;
    keccak_rounds(s, RC);
}
#ifdef __CUDACC__
// The register-state replay's permutation reads the round constants from constant memory: its round loop is not unrolled, and a
// local array indexed by the round would sit in the kernel's stack frame.
__constant__ uint64_t bp_keccak_rc[24] = BP_KECCAK_RC_INIT;
#endif
BP_HD void keccak_f1600_reg(uint64_t s[25]) {
#ifdef __CUDA_ARCH__
    keccak_rounds(s, bp_keccak_rc);
#else
    keccak_f1600(s);
#endif
}

#define BP_STROBE_R 166
// Serialized transcript state = what crosses the C ABI: 200 state bytes, pos, pos_begin, cur_flags
#define BP_TRANSCRIPT_BYTES 203

// The 200 state bytes live wherever the caller puts them (a local array on the host, a padded
// shared-memory row on the device); st must be 4-byte aligned.
struct merlin_t { uint8_t *st; uint32_t pos, pos_begin, cur_flags; };

BP_HD void strobe_permute(merlin_t &m) {
    uint32_t *w32 = reinterpret_cast<uint32_t *>(m.st);
    uint64_t w[25];
    for (int i = 0; i < 25; i++) w[i] = (uint64_t)w32[2 * i] | ((uint64_t)w32[2 * i + 1] << 32);
    keccak_f1600(w);
    for (int i = 0; i < 25; i++) { w32[2 * i] = (uint32_t)w[i]; w32[2 * i + 1] = (uint32_t)(w[i] >> 32); }
}
BP_HD void merlin_load(merlin_t &m, const uint8_t *ser) {
    for (int i = 0; i < 200; i++) m.st[i] = ser[i];
    m.pos = ser[200]; m.pos_begin = ser[201]; m.cur_flags = ser[202];
}
BP_HD void merlin_store(uint8_t *ser, const merlin_t &m) {
    for (int i = 0; i < 200; i++) ser[i] = m.st[i];
    ser[200] = (uint8_t)m.pos; ser[201] = (uint8_t)m.pos_begin; ser[202] = (uint8_t)m.cur_flags;
}
BP_HDN void strobe_run_f(merlin_t &m) {
    m.st[m.pos] ^= (uint8_t)m.pos_begin;
    m.st[m.pos + 1] ^= 0x04;
    m.st[BP_STROBE_R + 1] ^= 0x80;
    strobe_permute(m);
    m.pos = 0; m.pos_begin = 0;
}
BP_HDN void strobe_absorb(merlin_t &m, const uint8_t *d, uint32_t n) {
    for (uint32_t i = 0; i < n; i++) { m.st[m.pos] ^= d[i]; if (++m.pos == BP_STROBE_R) strobe_run_f(m); }
}
BP_HDN void strobe_squeeze(merlin_t &m, uint8_t *d, uint32_t n) {
    for (uint32_t i = 0; i < n; i++) { d[i] = m.st[m.pos]; m.st[m.pos] = 0; if (++m.pos == BP_STROBE_R) strobe_run_f(m); }
}
BP_HDN void strobe_overwrite(merlin_t &m, const uint8_t *d, uint32_t n) {      // KEY operation (TranscriptRng rekeying)
    for (uint32_t i = 0; i < n; i++) { m.st[m.pos] = d[i]; if (++m.pos == BP_STROBE_R) strobe_run_f(m); }
}
BP_HD void strobe_begin_op(merlin_t &m, uint8_t flags) {
    uint8_t hdr[2] = { (uint8_t)m.pos_begin, flags };
    m.pos_begin = m.pos + 1; m.cur_flags = flags;
    strobe_absorb(m, hdr, 2);
    if ((flags & (4 | 32)) && m.pos != 0) strobe_run_f(m);       // C or K flag forces a permutation
}
// label must be a NUL-terminated ASCII string
BP_HDN void merlin_append(merlin_t &m, const char *label, const uint8_t *msg, uint32_t len) {
    uint32_t ll = 0; while (label[ll]) ll++;
    uint8_t l4[4] = { (uint8_t)len, (uint8_t)(len >> 8), (uint8_t)(len >> 16), (uint8_t)(len >> 24) };
    strobe_begin_op(m, 16 | 2); strobe_absorb(m, (const uint8_t *)label, ll);   // meta_ad(label)
    strobe_absorb(m, l4, 4);                                                     // meta_ad(len, more)
    strobe_begin_op(m, 2); strobe_absorb(m, msg, len);                           // ad(msg)
}
BP_HD void merlin_append_u64(merlin_t &m, const char *label, uint64_t x) {
    uint8_t b[8]; for (int i = 0; i < 8; i++) b[i] = (uint8_t)(x >> (8 * i));
    merlin_append(m, label, b, 8);
}
BP_HDN void merlin_challenge(merlin_t &m, const char *label, uint8_t *out, uint32_t len) {
    uint32_t ll = 0; while (label[ll]) ll++;
    uint8_t l4[4] = { (uint8_t)len, (uint8_t)(len >> 8), (uint8_t)(len >> 16), (uint8_t)(len >> 24) };
    strobe_begin_op(m, 16 | 2); strobe_absorb(m, (const uint8_t *)label, ll);
    strobe_absorb(m, l4, 4);
    strobe_begin_op(m, 1 | 2 | 4); strobe_squeeze(m, out, len);                  // prf
}
// A verifier's batching weights, derived the way merlin's TranscriptRng derives a prover's randomness: build_rng() (a fork of the
// state: the caller's t, which it no longer needs), rekey_with_witness_bytes(label, w) (merlin_rng_rekey) with every proof byte the
// transcript has not absorbed, finalize(rng) = meta_ad("rng") + KEY(32 bytes of the external RNG: the batch seed), then
// fill_bytes(len) = meta_ad(LE32(len)) + PRF.  The weights then depend on every byte of the proof, so two proofs that differ anywhere
// get independent weights, and a caller that passes a fixed or known seed still gives a prover no way to choose proofs whose errors
// cancel in the combination.
// rekey_with_witness_bytes: meta_ad(label), meta_ad(LE32(len), more), KEY(w)
BP_HDN void merlin_rng_rekey(merlin_t &t, const char *label, const uint8_t *w, uint32_t len) {
    uint32_t ll = 0; while (label[ll]) ll++;
    const uint8_t l4[4] = { (uint8_t)len, (uint8_t)(len >> 8), (uint8_t)(len >> 16), (uint8_t)(len >> 24) };
    strobe_begin_op(t, 16 | 2); strobe_absorb(t, (const uint8_t *)label, ll); strobe_absorb(t, l4, 4);
    strobe_begin_op(t, 2 | 4); strobe_overwrite(t, w, len);
}
BP_HDN void merlin_rng_bytes(merlin_t &t, const uint8_t *seed, uint8_t *out, uint32_t len) {
    strobe_begin_op(t, 16 | 2); strobe_absorb(t, (const uint8_t *)"rng", 3);
    strobe_begin_op(t, 2 | 4); strobe_overwrite(t, seed, 32);
    const uint8_t l4[4] = { (uint8_t)len, (uint8_t)(len >> 8), (uint8_t)(len >> 16), (uint8_t)(len >> 24) };
    strobe_begin_op(t, 16 | 2); strobe_absorb(t, l4, 4);
    strobe_begin_op(t, 1 | 2 | 4); strobe_squeeze(t, out, len);
}
// ------------------------------------------------------------------ word-wise STROBE on a register state
// The byte-wise functions above keep the state in memory and move one byte per step.  A transcript replay whose byte positions
// are the same for every thread of a warp (the range-proof replay: same labels, lengths and caller state for every proof of a
// call) runs instead on 25 words held in registers: each operation XORs a whole string of up to 40 bytes at the current position
// with funnel shifts, and the word it starts at is picked by a warp-uniform switch, so no state byte is ever addressed at run time.
struct strobe_w { uint64_t s[25]; uint32_t pos, pos_begin; };
#ifdef __CUDA_ARCH__
#define BP_UNROLL _Pragma("unroll")
#else
#define BP_UNROLL
#endif

BP_HD uint64_t sw_shl(uint64_t x, uint32_t sh) { return sh >= 64 ? 0 : x << sh; }
BP_HD uint64_t sw_shr(uint64_t x, uint32_t sh) { return sh >= 64 ? 0 : x >> sh; }
BP_HD uint64_t sw_keep(uint64_t x, int32_t nbytes) { return nbytes >= 8 ? x : nbytes <= 0 ? 0 : x & ((1ULL << (8 * nbytes)) - 1); }
// state bytes [p, p + 8*NW) ^= the NW little-endian words x (bytes beyond the caller's length already zero); p + 8*NW may pass 200
// only over zero bytes
template <int NW> BP_HD void sw_xor_at(strobe_w &t, uint32_t p, const uint64_t (&x)[NW]) {
    const uint32_t sh = 8 * (p & 7);
    uint64_t w[NW + 1];
    w[0] = x[0] << sh;
#pragma unroll
    for (int j = 1; j < NW; j++) w[j] = (x[j] << sh) | sw_shr(x[j - 1], 64 - sh);
    w[NW] = sw_shr(x[NW - 1], 64 - sh);
#define SW_CASE(c) case c: BP_UNROLL for (int j = 0; j <= NW; j++) if (c + j < 25) t.s[c + j] ^= w[j]; break;
    switch (p >> 3) {
        SW_CASE(0) SW_CASE(1) SW_CASE(2) SW_CASE(3) SW_CASE(4) SW_CASE(5) SW_CASE(6) SW_CASE(7) SW_CASE(8) SW_CASE(9) SW_CASE(10) SW_CASE(11)
        SW_CASE(12) SW_CASE(13) SW_CASE(14) SW_CASE(15) SW_CASE(16) SW_CASE(17) SW_CASE(18) SW_CASE(19) SW_CASE(20) default: break;
    }
#undef SW_CASE
}
// run_f at the current position (strobe_run_f)
BP_HD void sw_run_f(strobe_w &t) {
    const uint64_t pad[1] = { (uint64_t)(t.pos_begin & 0xff) | (0x04ULL << 8) };
    sw_xor_at<1>(t, t.pos, pad);
    t.s[(BP_STROBE_R + 1) / 8] ^= 0x80ULL << (8 * ((BP_STROBE_R + 1) % 8));
    keccak_f1600_reg(t.s);
    t.pos = 0; t.pos_begin = 0;
}
// begin_op(flags) followed by the absorption of len <= 38 bytes d (little-endian words, zero beyond len): one string
// [pos_begin, flags] || d, permuting once if it crosses the rate (at most once: the string is shorter than the rate)
BP_HD void sw_begin_absorb(strobe_w &t, uint8_t flags, const uint64_t (&d)[5], uint32_t len) {
    uint64_t x[5];
    x[0] = (uint64_t)(t.pos_begin & 0xff) | ((uint64_t)flags << 8) | (d[0] << 16);
#pragma unroll
    for (int j = 1; j < 5; j++) x[j] = (d[j] << 16) | (d[j - 1] >> 48);
    len += 2;
    t.pos_begin = t.pos + 1;
    const uint32_t a = len < BP_STROBE_R - t.pos ? len : BP_STROBE_R - t.pos;       // bytes before the rate boundary
    uint64_t head[5];
#pragma unroll
    for (int j = 0; j < 5; j++) head[j] = sw_keep(x[j], (int32_t)a - 8 * j);
    sw_xor_at<5>(t, t.pos, head);
    t.pos += a;
    if (t.pos == BP_STROBE_R) {
        sw_run_f(t);
        // the remaining len - a bytes start at state byte 0: x shifted right by a bytes, the whole words in three uniform stages
        // (constant indices only, so x stays in registers), then the bits
        const uint32_t q = a >> 3, r = 8 * (a & 7);
        if (q & 4) { x[0] = x[4]; x[1] = 0; x[2] = 0; x[3] = 0; x[4] = 0; }
        if (q & 2) { x[0] = x[2]; x[1] = x[3]; x[2] = x[4]; x[3] = 0; x[4] = 0; }
        if (q & 1) { x[0] = x[1]; x[1] = x[2]; x[2] = x[3]; x[3] = x[4]; x[4] = 0; }
#pragma unroll
        for (int j = 0; j < 5; j++)
            t.s[j] ^= sw_keep(sw_shr(x[j], r) | (j < 4 ? sw_shl(x[j < 4 ? j + 1 : j], 64 - r) : 0), (int32_t)(len - a) - 8 * j);
        t.pos = len - a;
    }
}

// Transcript::new(label): STROBE init, meta_ad("Merlin v1.0"), then append_message("dom-sep", label)
BP_HD void merlin_init(merlin_t &m, const uint8_t *label, uint32_t len) {
    for (int i = 0; i < 200; i++) m.st[i] = 0;
    const uint8_t hdr[18] = { 1, BP_STROBE_R + 2, 1, 0, 1, 96, 'S', 'T', 'R', 'O', 'B', 'E', 'v', '1', '.', '0', '.', '2' };
    for (int i = 0; i < 18; i++) m.st[i] = hdr[i];
    strobe_permute(m);
    m.pos = 0; m.pos_begin = 0; m.cur_flags = 0;
    const char proto[] = "Merlin v1.0";
    strobe_begin_op(m, 16 | 2); strobe_absorb(m, (const uint8_t *)proto, 11);
    merlin_append(m, "dom-sep", label, len);
}
