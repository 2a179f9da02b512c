// Per-proof verification scalars of an aggregated range proof, computed on the device.
//
// Restates RangeProof::verify_multiple_with_rng up to (not including) the mega-MSM:
//   src/range_proof/mod.rs:368-419 (transcript replay, scalar assembly),
//   src/inner_product_proof.rs:198-253 (verification_scalars),
//   src/range_proof/mod.rs:587-593 (delta),
// with two changes that do not alter any verdict:
//  (1) every scalar of proof i is multiplied by a per-proof random weight, so that a batch of
//      proofs is checked with one random-linear-combination MSM (SURVEY.md §8a row A6);
//  (2) the weight is rho * lambda with lambda = (prod u_j)^2 * y^(N-1).  Multiplying the whole
//      mega-check by lambda cancels every inverse the reference computes (y^-i, u_j^-2, the
//      batch_invert product), so no field inversion is needed on the device:
//        lambda * u_j^-2          = y^(N-1) * prod_{j' != j} u_j'^2
//        lambda * s_i             = U * y^(N-1) * prod_{bits set in i} u^2      (U = prod u_j)
//        lambda * y^-i * s_{N-1-i} = U * y^(N-1-i) * prod_{bits clear in i} u^2
//      lambda != 0 with overwhelming probability and rho is uniform, so rho*lambda is a uniform weight.
//
// The work is split in a transcript replay (one thread per proof: Keccak chain), a short
// sequential head (one thread: ~8k+30 products) and a data-parallel tail (one generator index per
// thread).  All scalars are in Montgomery form between the byte boundaries.
#pragma once
#include <cstring>
#include <vector>
#include "sc.cuh"
#include "merlin.cuh"

// verdict codes, mirroring ProofError (src/errors.rs:12-54)
#define BP_PROOF_OK 0
#define BP_PROOF_VERIFICATION_ERROR 1
#define BP_PROOF_FORMAT_ERROR 2

#define BP_MAX_LG_N 20          // N = n*m up to 2^20 generator pairs per proof

// geometry of a batch verification (kernels.cuh, range-proof section): D = 4+2k+m dynamic terms, S = 2+2N static terms per proof
struct rp_geom { uint32_t n, m, k, N, D, S; uint32_t proof_len; uint32_t count, nbatch, T; };

// Reject path of a batch whose combined check failed (bpmsm.cu, rp_verify_fallback): one combined MSM per chunk of RP_CHUNK proofs
// (k_rp_scalars_sum keeps per-chunk partial sums), then the proofs of the failing chunks one by one -- or, when more than four
// chunks fail, every proof of the batch.  The second level runs the same kernels with chunks of one proof, whose sums
// k_rp_scalars_sum computes first.  Shared with the host-emulation tests.
#define RP_CHUNK 32
BP_HD bool rp_recheck_whole_batch(uint32_t failing_chunks) { return failing_chunks > 4; }

// Shared-memory stage of k_rp_decompress (kernels.cuh).  A block of RP_DEC_THREADS threads decodes the points [i0, i0 + RP_DEC_THREADS)
// of the batch's total*D points (point idx of proof p is point p*D + idx; V_j is idx = 4+2k+j).  It stages the whole proofs it touches,
// at most RP_DEC_THREADS/D + 2 of them, and of the commitments only those of its own V points: V_j of proof p is commitment p*m + j,
// so a block's V points are consecutive commitments, at most RP_DEC_THREADS of them whatever m is.  The stage is bounded by the block.
// Shared with the host-emulation tests.
#define RP_DEC_THREADS 128
struct rp_dec_stage { uint32_t pf, np; uint64_t c0; uint32_t nc; };   // proofs [pf, pf+np), commitments [c0, c0+nc)
// the V points among points [0, i): the commitment index of point i when it is a V point
BP_HD uint64_t rp_dec_v_before(const rp_geom &g, uint64_t i) {
    const uint64_t p = i / g.D; const uint32_t idx = (uint32_t)(i % g.D), v0 = 4 + 2 * g.k;
    return p * g.m + (idx > v0 ? idx - v0 : 0u);
}
BP_HD rp_dec_stage rp_dec_block(const rp_geom &g, uint32_t total, uint64_t i0) {
    const uint64_t n_pts = (uint64_t)total * g.D, i1 = i0 + RP_DEC_THREADS < n_pts ? i0 + RP_DEC_THREADS : n_pts;
    rp_dec_stage s;
    s.pf = (uint32_t)(i0 / g.D); s.np = (uint32_t)((i1 - 1) / g.D) - s.pf + 1;
    s.c0 = rp_dec_v_before(g, i0); s.nc = (uint32_t)(rp_dec_v_before(g, i1) - s.c0);
    return s;
}
// bytes of the proof part of the stage (the commitments follow it); a multiple of 32, so the commitment part stays 16-byte aligned
BP_HD uint32_t rp_dec_proof_bytes(const rp_geom &g) { return (RP_DEC_THREADS / g.D + 2) * g.proof_len; }
// offset in the stage of point i's 32-byte encoding (i inside the block of s)
BP_HD uint32_t rp_dec_offset(const rp_geom &g, const rp_dec_stage &s, uint64_t i) {
    const uint32_t p = (uint32_t)(i / g.D) - s.pf, idx = (uint32_t)(i % g.D), proof = p * g.proof_len;
    if (idx < 4) return proof + 32 * idx;                                         // A, S, T_1, T_2
    if (idx < 4 + g.k) return proof + 224 + 64 * (idx - 4);                        // L_j
    if (idx < 4 + 2 * g.k) return proof + 224 + 64 * (idx - 4 - g.k) + 32;         // R_j
    return rp_dec_proof_bytes(g) + 32 * (uint32_t)(rp_dec_v_before(g, i) - s.c0); // V_j
}
// dynamic shared memory of one k_rp_decompress launch: the launch sites pass it, and bp_ctx_create raises the kernel's limit to
// rp_dec_smem_max, its largest value over the geometries rp_param_verdict admits
BP_HD uint32_t rp_dec_smem_bytes(const rp_geom &g) {
    const uint32_t np = RP_DEC_THREADS / g.D + 2, nv = np * g.m < RP_DEC_THREADS ? np * g.m : RP_DEC_THREADS;
    return rp_dec_proof_bytes(g) + 32 * nv;
}
inline uint32_t rp_dec_smem_max() {
    uint32_t mx = 0;
    for (uint32_t k = 3; k <= BP_MAX_LG_N; k++)
        for (uint32_t n = 8; n <= 64 && n <= (1u << k); n *= 2) {
            rp_geom g{};
            g.n = n; g.m = (1u << k) / n; g.k = k; g.D = 4 + 2 * k + g.m; g.proof_len = 32 * (9 + 2 * k);
            const uint32_t b = rp_dec_smem_bytes(g);
            mx = b > mx ? b : mx;
        }
    return mx;
}

// out-of-line Montgomery product: one copy of the three-pass multiplier per kernel
BP_HDN sc sc_mm(const sc &a, const sc &b) { return sc_mont_mul(a, b); }
// the same with operands and result passed by value, i.e. in registers: a caller whose scalars all live in registers keeps them
// there (with sc_mm every operand is spilled to an addressable stack slot).  Used by the range-proof head (rp_head_lean).
BP_HDN sc rp_mul(sc a, sc b) { return sc_mont_mul(a, b); }
BP_HD sc rp_to_mont(const sc &a) { return rp_mul(a, sc{SC_RR_LIMBS}); }
BP_HD sc rp_from_mont(const sc &a) { sc one = sc_zero(); one.v[0] = 1; return rp_mul(a, one); }

struct rp_challenges {          // Montgomery form
    sc y, z, x, w, c, rho;
    sc u[BP_MAX_LG_N];
    uint32_t status;
};

BP_HD bool bp_is_zero32(const uint8_t *p) { uint8_t z = 0; for (int i = 0; i < 32; i++) z |= p[i]; return z == 0; }
// proofs per slice of the R1CS and LinearProof reject paths (bpmsm.cu, recheck_slices) for np proofs of entries_per_proof entries each and
// `budget` entries per slice: at least one, at most 65535 (the grid's y extent in k_r1cs_gh_sum and k_lin_g_sum).  Shared with the tests.
BP_HD uint32_t bp_recheck_slice(uint32_t np, uint32_t entries_per_proof, uint32_t budget) {
    uint32_t per = budget / entries_per_proof;
    per = per < 1u ? 1u : per > 65535u ? 65535u : per;
    return per < np ? per : np;
}
BP_HD sc rp_wide(const uint8_t buf[64]) { sc lo = sc_load(buf), hi = sc_load(buf + 32); return sc_add(sc_mm(lo, sc{SC_RR_LIMBS}), sc_mm(hi, sc{SC_RRR_LIMBS})); }
BP_HD sc rp_challenge(merlin_t &t, const char *label) { uint8_t buf[64]; merlin_challenge(t, label, buf, 64); return rp_wide(buf); }

// Transcript replay of one proof: pure hashing.  proof = 32*(9+2k) bytes, V = m*32 bytes, tstate = the serialized
// transcript the caller passed in, state200 = 200 bytes of 4-byte-aligned scratch for the STROBE state.
// Output: the 64-byte challenge outputs in the order y, z, x, w, c, rho (the batching weights), u_0..u_{k-1}
// -> raw[RP_RAW_U + j]; nothing the verifier hashes depends on a challenge, so the reduction mod l is left to the caller.
#define RP_RAW_Y 0
#define RP_RAW_Z 1
#define RP_RAW_X 2
#define RP_RAW_W 3
#define RP_RAW_C 4
#define RP_RAW_RHO 5
#define RP_RAW_U 6
#define RP_WITNESS_LABEL "ipp_a_b"     // rekeying label of the weights' transcript fork (the 64 bytes a || b)
BP_HD void rp_raw_challenge(merlin_t &t, const char *label, uint8_t *out64) { merlin_challenge(t, label, out64, 64); }
BP_HDN uint32_t rp_transcript_raw(uint8_t (*raw)[64], const uint8_t *proof, uint32_t k, const uint8_t *V, uint32_t n, uint32_t m,
                                  const uint8_t *tstate, const uint8_t *seed, uint8_t *state200) {
    const uint8_t *A = proof, *S = proof + 32, *T1 = proof + 64, *T2 = proof + 96;
    const uint8_t *LR = proof + 224, *ab = proof + 224 + 64 * k;
    // RangeProof::from_bytes / InnerProductProof::from_bytes canonicity (mod.rs:519-524, inner_product_proof.rs:399-404)
    if (sc_geq_l(sc_load(proof + 128)) || sc_geq_l(sc_load(proof + 160)) || sc_geq_l(sc_load(proof + 192)) || sc_geq_l(sc_load(ab)) || sc_geq_l(sc_load(ab + 32)))
        return BP_PROOF_FORMAT_ERROR;
    merlin_t t; t.st = state200; merlin_load(t, tstate);
    merlin_append(t, "dom-sep", (const uint8_t *)"rangeproof v1", 13);            // transcript.rs:44-48
    merlin_append_u64(t, "n", n); merlin_append_u64(t, "m", m);
    for (uint32_t j = 0; j < m; j++) merlin_append(t, "V", V + 32 * j, 32);         // mod.rs:370-374 (identity allowed)
    bool bad = bp_is_zero32(A) || bp_is_zero32(S);                                  // validate_and_append_point
    merlin_append(t, "A", A, 32); merlin_append(t, "S", S, 32);
    rp_raw_challenge(t, "y", raw[RP_RAW_Y]); rp_raw_challenge(t, "z", raw[RP_RAW_Z]);
    bad = bad || bp_is_zero32(T1) || bp_is_zero32(T2);
    merlin_append(t, "T_1", T1, 32); merlin_append(t, "T_2", T2, 32);
    rp_raw_challenge(t, "x", raw[RP_RAW_X]);
    merlin_append(t, "t_x", proof + 128, 32); merlin_append(t, "t_x_blinding", proof + 160, 32); merlin_append(t, "e_blinding", proof + 192, 32);
    rp_raw_challenge(t, "w", raw[RP_RAW_W]);
    merlin_append(t, "dom-sep", (const uint8_t *)"ipp v1", 6);                      // transcript.rs:50-53
    merlin_append_u64(t, "n", (uint64_t)n * m);
    for (uint32_t j = 0; j < k; j++) {                                              // inner_product_proof.rs:218-222
        bad = bad || bp_is_zero32(LR + 64 * j) || bp_is_zero32(LR + 64 * j + 32);
        merlin_append(t, "L", LR + 64 * j, 32); merlin_append(t, "R", LR + 64 * j + 32, 32);
        rp_raw_challenge(t, "u", raw[RP_RAW_U + j]);
    }
    // batching weights c (mod.rs:396) and rho (row A6), from the transcript, the inner-product scalars a, b it never absorbs, and the
    // batch seed (merlin_rng_rekey, merlin_rng_bytes)
    merlin_rng_rekey(t, RP_WITNESS_LABEL, ab, 64);
    merlin_rng_bytes(t, seed, raw[RP_RAW_C], 128);                                  // rows C and RHO are adjacent
    return bad ? BP_PROOF_VERIFICATION_ERROR : BP_PROOF_OK;
}
// Scheduled form of rp_transcript_raw.  Every proof of a call absorbs the same labels and lengths in the same order from the same
// caller state, so the byte position of every absorbed field and every permutation point is the same for all proofs.  The op
// sequence of a geometry is a short program (rp_tr_program, built once per geometry on the host); rp_transcript_sched replays it
// on the word-wise register state of merlin.cuh, where only the 32-byte proof fields and the squeezed outputs differ per proof.
// Each step is one STROBE operation: begin_op(flags), then the step's bytes.
#define RP_TR_UNIFORM 0         // len <= 24 bytes held in the step (a label and its length, a u64, a domain separator)
#define RP_TR_PROOF 1           // the 32 proof bytes at offset arg; chk: a zero encoding makes the proof fail (validate_and_append_point)
#define RP_TR_V 2               // the 32 commitment bytes at offset arg
#define RP_TR_KEY 3             // KEY: the 32 bytes of the batch seed
#define RP_TR_PRF 4             // PRF: len bytes squeezed into raw row arg
#define RP_TR_KEY_PROOF 5       // KEY: the 64 proof bytes at offset arg (the inner-product scalars a || b)
struct rp_tr_step { uint8_t flags, kind, len, chk; uint32_t arg; uint64_t d[3]; };
static_assert(sizeof(rp_tr_step) == 32, "transcript step");

struct rp_tr_builder {             // host only
    std::vector<rp_tr_step> P;
    void push(uint8_t flags, uint8_t kind, const void *bytes, uint32_t len, uint32_t arg = 0, uint8_t chk = 0) {
        rp_tr_step s{}; s.flags = flags; s.kind = kind; s.len = (uint8_t)len; s.chk = chk; s.arg = arg;
        if (kind == RP_TR_UNIFORM) memcpy(s.d, bytes, len);             // little-endian words
        P.push_back(s);
    }
    void meta(const char *label, uint32_t len) {                        // meta_ad(label), meta_ad(LE32(len), more)
        uint8_t b[24]; uint32_t ll = (uint32_t)strlen(label);
        memcpy(b, label, ll); for (int i = 0; i < 4; i++) b[ll + i] = (uint8_t)(len >> (8 * i));
        push(16 | 2, RP_TR_UNIFORM, b, ll + 4);
    }
    void append(const char *label, const void *msg, uint32_t len) { meta(label, len); push(2, RP_TR_UNIFORM, msg, len); }
    void append_u64(const char *label, uint64_t x) { uint8_t b[8]; for (int i = 0; i < 8; i++) b[i] = (uint8_t)(x >> (8 * i)); append(label, b, 8); }
    void field(const char *label, uint8_t kind, uint32_t off, bool chk) { meta(label, 32); push(2, kind, nullptr, 32, off, chk ? 1 : 0); }
    void challenge(const char *label, uint32_t row) { meta(label, 64); push(1 | 2 | 4, RP_TR_PRF, nullptr, 64, row); }
};
// the op sequence of rp_transcript_raw for a geometry, step for step
inline std::vector<rp_tr_step> rp_tr_program(uint32_t n, uint32_t m, uint32_t k) {
    rp_tr_builder b;
    b.append("dom-sep", "rangeproof v1", 13);
    b.append_u64("n", n); b.append_u64("m", m);
    for (uint32_t j = 0; j < m; j++) b.field("V", RP_TR_V, 32 * j, false);
    b.field("A", RP_TR_PROOF, 0, true); b.field("S", RP_TR_PROOF, 32, true);
    b.challenge("y", RP_RAW_Y); b.challenge("z", RP_RAW_Z);
    b.field("T_1", RP_TR_PROOF, 64, true); b.field("T_2", RP_TR_PROOF, 96, true);
    b.challenge("x", RP_RAW_X);
    b.field("t_x", RP_TR_PROOF, 128, false); b.field("t_x_blinding", RP_TR_PROOF, 160, false); b.field("e_blinding", RP_TR_PROOF, 192, false);
    b.challenge("w", RP_RAW_W);
    b.append("dom-sep", "ipp v1", 6);
    b.append_u64("n", (uint64_t)n * m);
    for (uint32_t j = 0; j < k; j++) {
        b.field("L", RP_TR_PROOF, 224 + 64 * j, true); b.field("R", RP_TR_PROOF, 224 + 64 * j + 32, true);
        b.challenge("u", RP_RAW_U + j);
    }
    b.meta(RP_WITNESS_LABEL, 64); b.push(2 | 4, RP_TR_KEY_PROOF, nullptr, 0, 224 + 64 * k);     // merlin_rng_rekey(a || b)
    const uint8_t l4[4] = {128, 0, 0, 0};                                // merlin_rng_bytes(seed, 128): rows C and RHO
    b.push(16 | 2, RP_TR_UNIFORM, "rng", 3); b.push(2 | 4, RP_TR_KEY, nullptr, 32);
    b.push(16 | 2, RP_TR_UNIFORM, l4, 4); b.push(1 | 2 | 4, RP_TR_PRF, nullptr, 128, RP_RAW_C);
    return b.P;
}

BP_HD uint64_t rp_ld64(const uint8_t *p, bool aligned) {
#ifdef __CUDA_ARCH__
    if (aligned) return __ldg(reinterpret_cast<const unsigned long long *>(p));
#endif
    (void)aligned;
    uint64_t x = 0; for (int i = 0; i < 8; i++) x |= (uint64_t)p[i] << (8 * i);
    return x;
}
BP_HD void rp_st64(uint8_t *p, uint64_t x) {
#ifdef __CUDA_ARCH__
    *reinterpret_cast<uint64_t *>(p) = x;
#else
    for (int i = 0; i < 8; i++) p[i] = (uint8_t)(x >> (8 * i));
#endif
}
// Same outputs as rp_transcript_raw (raw rows, verdict) for the program of the geometry (n, m, k).  tstate = the serialized caller
// transcript, read with 8-byte loads when tstate_al says it is 8-byte aligned; seed = the batch seed; raw must be 8-byte aligned on the
// device.  check_tstate: a state no Merlin transcript can hold between operations (pos at or beyond the rate, or pos_begin above pos)
// gives BP_PROOF_FORMAT_ERROR before the replay indexes the state with pos.
BP_HD uint32_t rp_transcript_sched(uint8_t *raw, const uint8_t *proof, uint32_t k, const uint8_t *V, const uint8_t *tstate, const uint8_t *seed,
                                   const rp_tr_step *prog, uint32_t nsteps, bool tstate_al = true, bool check_tstate = false) {
    const uint8_t *ab = proof + 224 + 64 * k;
    if (sc_geq_l(sc_load(proof + 128)) || sc_geq_l(sc_load(proof + 160)) || sc_geq_l(sc_load(proof + 192)) || sc_geq_l(sc_load(ab)) || sc_geq_l(sc_load(ab + 32)))
        return BP_PROOF_FORMAT_ERROR;
    strobe_w t;
    t.pos = tstate[200]; t.pos_begin = tstate[201];
    if (check_tstate && (t.pos >= BP_STROBE_R || t.pos_begin > t.pos)) return BP_PROOF_FORMAT_ERROR;
    BP_UNROLL for (int i = 0; i < 25; i++) t.s[i] = rp_ld64(tstate + 8 * i, tstate_al);
    const bool al = (((uintptr_t)proof | (uintptr_t)V) & 7) == 0;      // the same for every proof of a call
    bool bad = false;
    for (uint32_t i = 0; i < nsteps; i++) {
        const rp_tr_step st = prog[i];
        uint64_t d[5] = {0, 0, 0, 0, 0};
        uint32_t len = 0;
        if (st.kind == RP_TR_UNIFORM) {
            d[0] = st.d[0]; d[1] = st.d[1]; d[2] = st.d[2]; len = st.len;
        } else if (st.kind <= RP_TR_V) {
            const uint8_t *src = (st.kind == RP_TR_V ? V : proof) + st.arg;
            BP_UNROLL for (int j = 0; j < 4; j++) d[j] = rp_ld64(src + 8 * j, al);
            if (st.chk) bad = bad || (d[0] | d[1] | d[2] | d[3]) == 0;
            len = 32;
        }
        sw_begin_absorb(t, st.flags, d, len);
        if (st.kind < RP_TR_KEY) continue;
        // KEY / PRF: the C or K flag permutes unless the header left the position at 0 (a header that ends on the rate boundary
        // permutes inside the absorption); either way the operation runs from state byte 0 with pos_begin 0
        if (t.pos != 0) sw_run_f(t);
        t.pos_begin = 0;
        if (st.kind == RP_TR_KEY) {
            for (int j = 0; j < 4; j++) t.s[j] = rp_ld64(seed + 8 * j, true);
            t.pos = 32;
        } else if (st.kind == RP_TR_KEY_PROOF) {
            BP_UNROLL for (int j = 0; j < 8; j++) t.s[j] = rp_ld64(proof + st.arg + 8 * j, al);
            t.pos = 64;
        } else {
            uint8_t *out = raw + 64 * (size_t)st.arg;
            BP_UNROLL for (int j = 0; j < 16; j++) if (8 * j < st.len) { rp_st64(out + 8 * j, t.s[j]); t.s[j] = 0; }
            t.pos = st.len;
        }
    }
    return bad ? BP_PROOF_VERIFICATION_ERROR : BP_PROOF_OK;
}
// The replay of proof p of a k_rp_transcript launch (rp_params: tstates, tstride).  Stride 0: every proof starts from the one state the
// caller passed, taken as it is.  Otherwise proof p starts from its own record at tstates + p * tstride, which is checked.  The 8-byte
// loads need the base and the stride both to be multiples of 8, so that the choice is the same for every thread; with 203-byte records
// back to back the state is read byte-wise.
BP_HD uint32_t rp_transcript_proof(uint8_t *raw, const uint8_t *proof, uint32_t k, const uint8_t *V, const uint8_t *tstates, uint64_t tstride, uint32_t p,
                                   const uint8_t *seed, const rp_tr_step *prog, uint32_t nsteps) {
    const bool al = (((uintptr_t)tstates | tstride) & 7) == 0;
    return rp_transcript_sched(raw, proof, k, V, tstates + p * tstride, seed, prog, nsteps, al, tstride != 0);
}

// Sequential form (host emulation, reference for the device head): the challenge rows reduced mod l (Montgomery form), with the
// zero-challenge and zero-weight rules of the verifier.
BP_HDN void rp_reduce_challenges(rp_challenges &ch, const uint8_t (*raw)[64], uint32_t k) {
    ch.status = BP_PROOF_OK;
    ch.y = rp_wide(raw[RP_RAW_Y]); ch.z = rp_wide(raw[RP_RAW_Z]); ch.x = rp_wide(raw[RP_RAW_X]); ch.w = rp_wide(raw[RP_RAW_W]);
    for (uint32_t j = 0; j < k; j++) ch.u[j] = rp_wide(raw[RP_RAW_U + j]);
    // The device multiplies the proof's check by lambda = (prod u_j)^2 y^(N-1) (see the header).  A zero challenge would make
    // lambda vanish and the proof drop out of the combination, so it is rejected outright; the reference cannot verify such a
    // transcript either (u_j = 0 has no inverse), and an honest or dishonest prover hits it with probability ~2^-252 per hash.
    bool bad = sc_is_zero(ch.y);
    for (uint32_t j = 0; j < k; j++) bad = bad || sc_is_zero(ch.u[j]);
    if (bad) { ch.status = BP_PROOF_VERIFICATION_ERROR; return; }
    ch.c = rp_wide(raw[RP_RAW_C]); ch.rho = rp_wide(raw[RP_RAW_RHO]);
    if (sc_is_zero(ch.rho)) ch.rho = sc_mont_one();                  // a zero weight (probability 2^-252) would skip the proof
}
// replay + reduction of the challenges.  seed = the batch's 32 bytes of external randomness (c and rho are derived from it and the
// proof's transcript).
BP_HDN void rp_transcript(rp_challenges &ch, const uint8_t *proof, uint32_t k, const uint8_t *V, uint32_t n, uint32_t m,
                         const uint8_t *tstate, const uint8_t *seed, uint8_t *state200) {
    uint8_t raw[RP_RAW_U + BP_MAX_LG_N][64];
    ch.status = rp_transcript_raw(raw, proof, k, V, n, m, tstate, seed, state200);
    if (ch.status == BP_PROOF_OK) rp_reduce_challenges(ch, raw, k);
}

struct rp_head {                // Montgomery form; "L" = Lambda = rho * lambda
    uint32_t status, pad_[7];
    sc z, zz, L, zL, Lx, Lcx, Lcxx, Lczz, gA, hB, rhoY;
    sc u_sq[BP_MAX_LG_N], pre[BP_MAX_LG_N + 1], suf[BP_MAX_LG_N + 1];
    sc basepoint_scalar, blinding_scalar;
};

// Per-proof product tables (global memory, rp_tab_size() scalars per proof) that turn the tail into three products
// per generator index.  The k index bits are split in a low group of kl = ceil(k/2) bits (TL = 2^kl values) and a
// high group of kh = k - kl bits (TH = 2^kh values), i = hi*TL + lo, and ~v is the complement within the group:
//   s_lo[v] = prod_{b < kl, bit b of v} u_sq[k-1-b]           s_hi[v] = prod_{b < kh, bit b of v} u_sq[k-1-kl-b]
//   y_lo[v] = y^v                                               y_hi[v] = y^(v*TL)
//   A_hi[v] = gA * s_hi[v]
//   P_lo[v] = y_lo[~v] * F_lo(v)                                P_hi[v] = hA * y_hi[~v] * F_hi(v)
//   Q_lo[v] = y_lo[~v] * s_lo[~v]                               Q_hi[v] = hB * y_hi[~v] * s_hi[~v]
// with F(i) = 2^(i mod n) z^(i div n) = F_hi(hi) F_lo(lo) (n and TL are powers of two), so that
//   lambda-weighted  g_i = -zL - A_hi[hi] s_lo[lo],     h_i = zL + P_hi[hi] P_lo[lo] - Q_hi[hi] Q_lo[lo].
BP_HD uint32_t rp_kl(uint32_t k) { return (k + 1) / 2; }
BP_HD uint32_t rp_tab_size(uint32_t k, uint32_t m) { (void)m; uint32_t kl = rp_kl(k); return 4 * (1u << kl) + 5 * (1u << (k - kl)); }
// A slice of proofs keeps its tables chunk-major: entry e of the proof at position q of its RP_CHUNK-proof chunk c is
// tab[(c tsz + e) RP_CHUNK + q], so a proof's entries lie RP_CHUNK scalars apart and the chunk's proofs share each entry's row.  The head
// (one lane per proof) then stores every entry as one contiguous row, and k_rp_scalars_sum reads the chunk's rows as one block.  A slice
// of count proofs holds whole chunks (rp_tab_slice); rp_tab_proof is entry 0 of its proof p.
#define RP_TAB_STRIDE RP_CHUNK
BP_HD uint64_t rp_tab_slice(uint64_t count, uint32_t k, uint32_t m) { return (count + RP_CHUNK - 1) / RP_CHUNK * RP_CHUNK * rp_tab_size(k, m); }
BP_HD size_t rp_tab_index(uint32_t p, uint32_t tsz) { return ((size_t)(p / RP_CHUNK) * tsz) * RP_CHUNK + p % RP_CHUNK; }
BP_HD sc *rp_tab_proof(sc *slice, uint32_t p, uint32_t tsz) { return slice + rp_tab_index(p, tsz); }
// the proofs block `block` of k_rp_scalars_sum sums: chunk ch of batch b, nq proofs from p0 (group index) on
struct rp_sum_block { uint32_t nchunks, b, ch, nq, p0; };
BP_HD rp_sum_block rp_sum_block_of(const rp_geom &g, uint32_t block) {
    rp_sum_block s;
    s.nchunks = (g.count + RP_CHUNK - 1) / RP_CHUNK; s.b = block / s.nchunks; s.ch = block % s.nchunks;
    const uint32_t q0 = s.ch * RP_CHUNK;
    s.nq = g.count - q0 < RP_CHUNK ? g.count - q0 : RP_CHUNK; s.p0 = s.b * g.count + q0;
    return s;
}
// one table of a proof: entry v at p[v * s] (s = RP_TAB_STRIDE in a slice, 1 for the host reference's contiguous tables)
struct rp_tab_col {
    sc *p; uint32_t s;
    BP_HD sc &operator[](uint32_t v) const { return p[v * s]; }
};
struct rp_tabs { rp_tab_col s_lo, A_hi, P_lo, P_hi, Q_lo, Q_hi, s_hi, y_lo, y_hi; };
// the tables of the proof whose entry 0 is tab, entries s apart; the six that k_rp_scalars_sum reads come first
BP_HD rp_tabs rp_tab_ptrs(sc *tab, uint32_t k, uint32_t s = 1) {
    const uint32_t kl = rp_kl(k), TL = 1u << kl, TH = 1u << (k - kl);
    rp_tabs t; uint32_t e = 0;
    t.s_lo = {tab + e * s, s}; e += TL; t.A_hi = {tab + e * s, s}; e += TH; t.P_lo = {tab + e * s, s}; e += TL; t.P_hi = {tab + e * s, s}; e += TH;
    t.Q_lo = {tab + e * s, s}; e += TL; t.Q_hi = {tab + e * s, s}; e += TH; t.s_hi = {tab + e * s, s}; e += TH; t.y_lo = {tab + e * s, s}; e += TL;
    t.y_hi = {tab + e * s, s};
    return t;
}

BP_HD sc rp_pow_small(const sc &base0, uint32_t e) {                // base^e by square-and-multiply
    sc r = sc_mont_one(), base = base0;
    for (; e; e >>= 1) { if (e & 1u) r = sc_mm(r, base); if (e > 1) base = sc_mm(base, base); }
    return r;
}

// sum_{i<n} x^i for n a power of two (util.rs:240-256), Montgomery form
BP_HD sc rp_sum_of_powers_pow2(const sc &x, uint64_t n) {
    if (n == 1) return sc_mont_one();
    sc result = sc_add(sc_mont_one(), x), factor = x;
    for (uint64_t m = n; m > 2; m >>= 1) { factor = rp_mul(factor, factor); result = sc_add(result, rp_mul(factor, result)); }
    return result;
}

#ifdef __CUDA_ARCH__
#define RP_ROLLED _Pragma("unroll 1")     // one call site per product in every instance: a constant k (k_rp_head_seq) unrolls nothing
#else
#define RP_ROLLED
#endif

// table[v] for v in [0, 2^bits): product of f[b] over the set bits b of v; f(b) supplied by the caller
#define RP_BUILD_TABLE(tab, bits, FACTOR)                                                    \
    do {                                                                                     \
        (tab)[0] = sc_mont_one();                                                            \
        RP_ROLLED for (uint32_t b_ = 0; b_ < (bits); b_++) {                                 \
            const sc f_ = (FACTOR);                                                          \
            (tab)[1u << b_] = f_;                                                            \
            RP_ROLLED for (uint32_t v_ = 1; v_ < (1u << b_); v_++) (tab)[(1u << b_) + v_] = rp_mul((tab)[v_], f_); \
        }                                                                                    \
    } while (0)

// Sequential head: shared products and tables of one proof
BP_HDN void rp_scalars_head(rp_head &h, sc *tab, const sc *pow2, const rp_challenges &ch, const uint8_t *proof, uint32_t k, uint32_t n, uint32_t m) {
    const uint8_t *ab = proof + 224 + 64 * k;
    sc a = sc_to_mont(sc_load(ab)), b = sc_to_mont(sc_load(ab + 32));
    sc t_x = sc_to_mont(sc_load(proof + 128)), t_x_bl = sc_to_mont(sc_load(proof + 160)), e_bl = sc_to_mont(sc_load(proof + 192));
    h.z = ch.z; h.zz = sc_mm(ch.z, ch.z);
    uint32_t kl = rp_kl(k), kh = k - kl, TL = 1u << kl, TH = 1u << kh;
    rp_tabs T = rp_tab_ptrs(tab, k);
    sc U = sc_mont_one(), Y = sc_mont_one(), ypow2[BP_MAX_LG_N];
    h.pre[0] = sc_mont_one();
    for (uint32_t j = 0; j < k; j++) {
        h.u_sq[j] = sc_mm(ch.u[j], ch.u[j]); U = sc_mm(U, ch.u[j]);
        h.pre[j + 1] = sc_mm(h.pre[j], h.u_sq[j]);                  // prod_{j' <= j} u^2;  pre[k] = U^2
        ypow2[j] = j == 0 ? ch.y : sc_mm(ypow2[j - 1], ypow2[j - 1]);        // y^(2^j)
        Y = sc_mm(Y, ypow2[j]);                                     // ends as y^(N-1)
    }
    h.suf[k] = sc_mont_one();
    for (int j = (int)k - 1; j >= 0; j--) h.suf[j] = sc_mm(h.suf[j + 1], h.u_sq[j]);   // prod_{j' >= j} u^2
    // bit b of the index i <-> challenge k-1-b (inner_product_proof.rs:241-250)
    RP_BUILD_TABLE(T.s_lo, kl, h.u_sq[(k - 1) - b_]);
    RP_BUILD_TABLE(T.s_hi, kh, h.u_sq[(k - 1) - kl - b_]);
    RP_BUILD_TABLE(T.y_lo, kl, ypow2[b_]);
    RP_BUILD_TABLE(T.y_hi, kh, ypow2[kl + b_]);
    sc lambda = sc_mm(h.pre[k], Y);
    h.L = sc_mm(ch.rho, lambda); h.zL = sc_mm(ch.z, h.L);
    h.Lx = sc_mm(h.L, ch.x); h.Lcx = sc_mm(h.Lx, ch.c); h.Lcxx = sc_mm(h.Lcx, ch.x); h.Lczz = sc_mm(sc_mm(h.L, ch.c), h.zz);
    sc rhoU = sc_mm(ch.rho, U);
    h.gA = sc_mm(sc_mm(a, rhoU), Y);                                // a rho U y^(N-1)
    h.hB = sc_mm(b, rhoU);                                          // b rho U
    sc hA = sc_mm(sc_mm(rhoU, U), h.zz);                            // rho U^2 z^2
    // F(i) = 2^(i mod n) z^(i div n) split over the two index groups
    for (uint32_t v = 0; v < TL; v++) {
        sc F = sc_mm(pow2[v % n], rp_pow_small(ch.z, v / n));       // v < TL: (v mod n, v div n)
        T.P_lo[v] = sc_mm(T.y_lo[v ^ (TL - 1)], F);
        T.Q_lo[v] = sc_mm(T.y_lo[v ^ (TL - 1)], T.s_lo[v ^ (TL - 1)]);
    }
    for (uint32_t v = 0; v < TH; v++) {
        uint64_t idx = (uint64_t)v << kl;                           // i = v*TL: (i mod n, i div n)
        sc F = sc_mm(pow2[idx % n], rp_pow_small(ch.z, (uint32_t)(idx / n)));
        sc yc = T.y_hi[v ^ (TH - 1)];
        T.A_hi[v] = sc_mm(h.gA, T.s_hi[v]);
        T.P_hi[v] = sc_mm(sc_mm(hA, yc), F);
        T.Q_hi[v] = sc_mm(sc_mm(h.hB, yc), T.s_hi[v ^ (TH - 1)]);
    }
    h.rhoY = sc_mm(ch.rho, Y);
    // delta(y,z) = (z - z^2) sum y^i - z^3 (2^n - 1) sum z^j          (mod.rs:587-593)
    sc sum_y = rp_sum_of_powers_pow2(ch.y, (uint64_t)n * m), sum_z = rp_sum_of_powers_pow2(ch.z, m);
    sc sum_2 = sc_mont_from_u64(n == 64 ? ~0ULL : ((1ULL << n) - 1));
    sc delta = sc_sub(sc_mm(sc_sub(ch.z, h.zz), sum_y), sc_mm(sc_mm(sc_mm(h.zz, ch.z), sum_2), sum_z));
    // basepoint scalar w (t_x - a b) + c (delta - t_x)  (mod.rs:419);  blinding scalar -e~ - c t~  (mod.rs:430)
    sc bs = sc_add(sc_mm(ch.w, sc_sub(t_x, sc_mm(a, b))), sc_mm(ch.c, sc_sub(delta, t_x)));
    sc bl = sc_neg(sc_add(e_bl, sc_mm(ch.c, t_x_bl)));
    h.basepoint_scalar = sc_mm(h.L, bs); h.blinding_scalar = sc_mm(h.L, bl);
}

// Data-parallel tail: weighted g_i and h_i for generator pair i in [0, N) (mod.rs:415-417), Montgomery form.
// Three products per index (see the table definitions above).  The device sums these products over a chunk's proofs in
// k_rp_scalars_sum (kernels.cuh) and never calls this per-proof form; it is the reference the host-emulation tests check
// the scalar assembly with.
BP_HD void rp_scalars_gh(const rp_head &h, const sc *tab, uint32_t i, uint32_t k, sc &g, sc &hh) {
    uint32_t kl = rp_kl(k), TL = 1u << kl;
    rp_tabs T = rp_tab_ptrs(const_cast<sc *>(tab), k);
    uint32_t lo = i & (TL - 1), hi = i >> kl;
    g = sc_sub(sc_neg(h.zL), sc_mm(T.A_hi[hi], T.s_lo[lo]));
    hh = sc_sub(sc_add(h.zL, sc_mm(T.P_hi[hi], T.P_lo[lo])), sc_mm(T.Q_hi[hi], T.Q_lo[lo]));
}

// Per-proof ("dynamic") scalars in MSM order A, S, T_1, T_2, L_0..L_{k-1}, R_0..R_{k-1}, V_0..V_{m-1}
// (mod.rs:422-444 without the static B~, B, G, H block); idx in [0, 4+2k+m); Montgomery form
BP_HD sc rp_scalars_dynamic(const rp_head &h, uint32_t idx, uint32_t k) {
    if (idx == 0) return h.L;
    if (idx == 1) return h.Lx;
    if (idx == 2) return h.Lcx;
    if (idx == 3) return h.Lcxx;
    if (idx < 4 + k) return sc_mm(h.L, h.u_sq[idx - 4]);
    if (idx < 4 + 2 * k) { uint32_t j = idx - 4 - k; return sc_mm(h.rhoY, sc_mm(h.pre[j], h.suf[j + 1])); }
    return sc_mm(h.Lczz, rp_pow_small(h.z, idx - 4 - 2 * k));
}

// ------------------------------------------------------------------ device head (k_rp_head_seq)
// The same products as rp_reduce_challenges + rp_scalars_head + rp_scalars_dynamic, for one thread per proof, with nothing indexed
// at run time in local memory: every challenge row is reduced where it is used; u_j^2 and y^(2^j) go straight into the table entry
// of their index bit (rp_usq_slot; y_lo[2^b] = y^(2^b), y_hi[2^b] = y^(2^(kl+b))), which is also where the L_j and R_j scalars read
// them back; and the product of every u^2 but u_j^2 that an R_j scalar needs is one entry of j's index group times the other group's
// full product, so no prefix or suffix array is kept.  Every product is rp_mul, whose operands stay in registers.

struct rp_lean_head {           // what k_rp_scalars_sum reads of a proof's head (Montgomery form)
    uint32_t status, pad_[7];
    sc zL, basepoint_scalar, blinding_scalar;
};

// challenge row of k_rp_transcript's output (8-byte aligned) reduced mod l, Montgomery form: rp_wide(row)
BP_HD sc rp_wide_row(const uint8_t *row) {
    sc lo, hi;
    BP_UNROLL for (int i = 0; i < 4; i++) {
        uint64_t a = rp_ld64(row + 8 * i, true), b = rp_ld64(row + 32 + 8 * i, true);
        lo.v[2 * i] = (uint32_t)a; lo.v[2 * i + 1] = (uint32_t)(a >> 32); hi.v[2 * i] = (uint32_t)b; hi.v[2 * i + 1] = (uint32_t)(b >> 32);
    }
    return sc_add(rp_mul(lo, sc{SC_RR_LIMBS}), rp_mul(hi, sc{SC_RRR_LIMBS}));
}
// the table entry that holds u_j^2: s_lo[2^b] for j = k-1-b (b < kl), s_hi[2^b] for j = k-1-kl-b (b < kh)
BP_HD sc *rp_usq_slot(const rp_tabs &T, uint32_t k, uint32_t j) {
    const uint32_t kh = k - rp_kl(k);
    return j >= kh ? &T.s_lo[1u << (k - 1 - j)] : &T.s_hi[1u << (kh - 1 - j)];
}
// canonical bytes of a Montgomery scalar into a 16-byte aligned MSM scalar slot
BP_HD void rp_put_scalar(uint8_t *dst, const sc &a) {
    const sc r = rp_from_mont(a);
#ifdef __CUDA_ARCH__
    uint4 *p = reinterpret_cast<uint4 *>(dst);
    p[0] = make_uint4(r.v[0], r.v[1], r.v[2], r.v[3]); p[1] = make_uint4(r.v[4], r.v[5], r.v[6], r.v[7]);
#else
    sc_store(dst, r);
#endif
}

// Head of one proof from its challenge rows raw (RP_RAW_U + k rows of 64 bytes, 8-byte aligned): the nine tables (rp_tab_size scalars
// from tab on, tab_stride apart: rp_tab_ptrs), h.zL and the two base-point scalars, and the D = 4 + 2k + m dynamic scalars in MSM order
// (rp_scalars_dynamic) as canonical bytes into dyn[32 d].  Returns BP_PROOF_VERIFICATION_ERROR for a zero y or u_j
// (rp_reduce_challenges), and then writes nothing but tables.  Force-inlined, so that a caller passing a constant k gets a head
// specialised to it.
BP_HD uint32_t rp_head_lean(rp_lean_head &h, sc *tab, uint8_t *dyn, const sc *pow2, const uint8_t *raw, const uint8_t *proof, uint32_t k,
                            uint32_t n, uint32_t m, uint32_t tab_stride = 1) {
    const uint32_t kl = rp_kl(k), kh = k - kl, TL = 1u << kl, TH = 1u << kh;
    const rp_tabs T = rp_tab_ptrs(tab, k, tab_stride);
    const sc one = sc_mont_one();
    sc U = one, yp = rp_wide_row(raw + 64 * RP_RAW_Y);
    bool bad = sc_is_zero(yp);
    RP_ROLLED for (uint32_t j = 0; j < k; j++) {
        const sc u = rp_wide_row(raw + 64 * (RP_RAW_U + j));
        bad = bad || sc_is_zero(u);
        U = rp_mul(U, u);
        *rp_usq_slot(T, k, j) = rp_mul(u, u);
        if (j) yp = rp_mul(yp, yp);                                    // y^(2^j)
        (j < kl ? T.y_lo[1u << j] : T.y_hi[1u << (j - kl)]) = yp;
    }
    if (bad) return BP_PROOF_VERIFICATION_ERROR;
    RP_BUILD_TABLE(T.s_lo, kl, T.s_lo[1u << b_]);
    RP_BUILD_TABLE(T.s_hi, kh, T.s_hi[1u << b_]);
    RP_BUILD_TABLE(T.y_lo, kl, T.y_lo[1u << b_]);
    RP_BUILD_TABLE(T.y_hi, kh, T.y_hi[1u << b_]);
    // Past this point only z, rho U and rho U^2 live across the stages (y^(N-1) = y_lo[TL-1] y_hi[TH-1] and (prod u_j)^2 =
    // s_lo[TL-1] s_hi[TH-1] are read back from the tables); each stage keeps its own factor and nothing else.
    const sc z = rp_wide_row(raw + 64 * RP_RAW_Z);
    sc rho = rp_wide_row(raw + 64 * RP_RAW_RHO);
    if (sc_is_zero(rho)) rho = one;
    const sc rhoU = rp_mul(rho, U), rhoUU = rp_mul(rhoU, U);
    {
        const sc Y = rp_mul(T.y_lo[TL - 1], T.y_hi[TH - 1]), rhoY = rp_mul(rho, Y);           // y^(N-1)
        const sc L = rp_mul(rhoUU, Y);                                                          // rho (prod u_j)^2 y^(N-1)
        h.zL = rp_mul(z, L);
        // L_j: L u_j^2;  R_j: rho y^(N-1) prod_{j' != j} u_j'^2 = (rho y^(N-1) x the other group's full product) x the entry of j's
        // group without bit j
        RP_ROLLED for (uint32_t j = 0; j < k; j++) rp_put_scalar(dyn + 32 * (4 + j), rp_mul(L, *rp_usq_slot(T, k, j)));
        sc R = rp_mul(rhoY, T.s_hi[TH - 1]);
        RP_ROLLED for (uint32_t j = kh; j < k; j++) rp_put_scalar(dyn + 32 * (4 + k + j), rp_mul(R, T.s_lo[(TL - 1) ^ (1u << (k - 1 - j))]));
        R = rp_mul(rhoY, T.s_lo[TL - 1]);
        RP_ROLLED for (uint32_t j = 0; j < kh; j++) rp_put_scalar(dyn + 32 * (4 + k + j), rp_mul(R, T.s_hi[(TH - 1) ^ (1u << (kh - 1 - j))]));
        // A, S, T_1, T_2: L, L x, L c x, L c x^2
        const sc c = rp_wide_row(raw + 64 * RP_RAW_C);
        {
            const sc x = rp_wide_row(raw + 64 * RP_RAW_X), Lx = rp_mul(L, x), Lcx = rp_mul(Lx, c);
            rp_put_scalar(dyn, L); rp_put_scalar(dyn + 32, Lx); rp_put_scalar(dyn + 64, Lcx); rp_put_scalar(dyn + 96, rp_mul(Lcx, x));
        }
        const sc zz = rp_mul(z, z);
        {   // V_j: L c z^2 z^j
            sc v = rp_mul(rp_mul(L, c), zz);
            RP_ROLLED for (uint32_t j = 0; j < m; j++) {
                rp_put_scalar(dyn + 32 * (4 + 2 * k + j), v);
                if (j + 1 < m) v = rp_mul(v, z);
            }
        }
        // delta(y,z) = (z - z^2) sum y^i - z^3 (2^n - 1) sum z^j  (mod.rs:587-593); base-point and blinding scalars (mod.rs:419,430)
        const sc sum_y = rp_sum_of_powers_pow2(T.y_lo[1], (uint64_t)n * m), sum_z = rp_sum_of_powers_pow2(z, m);     // y_lo[1] = y
        sc sum_2 = sc_zero(); sum_2.v[0] = n >= 32 ? ~0u : (1u << n) - 1; sum_2.v[1] = n == 64 ? ~0u : n > 32 ? (1u << (n - 32)) - 1 : 0;
        sum_2 = rp_to_mont(sum_2);                                                              // 2^n - 1
        const sc delta = sc_sub(rp_mul(sc_sub(z, zz), sum_y), rp_mul(rp_mul(rp_mul(zz, z), sum_2), sum_z));
        const sc t_x = rp_to_mont(sc_load(proof + 128)), ab = rp_mul(rp_to_mont(sc_load(proof + 224 + 64 * k)), rp_to_mont(sc_load(proof + 256 + 64 * k)));
        const sc bs = sc_add(rp_mul(rp_wide_row(raw + 64 * RP_RAW_W), sc_sub(t_x, ab)), rp_mul(c, sc_sub(delta, t_x)));
        h.basepoint_scalar = rp_mul(L, bs);
        const sc bl = sc_neg(sc_add(rp_to_mont(sc_load(proof + 192)), rp_mul(c, rp_to_mont(sc_load(proof + 160)))));
        h.blinding_scalar = rp_mul(L, bl);
    }
    // the tail's tables (their definitions above rp_tab_size)
    {
        const sc gA = rp_mul(rp_mul(rp_to_mont(sc_load(proof + 224 + 64 * k)), rhoU), rp_mul(T.y_lo[TL - 1], T.y_hi[TH - 1]));    // a rho U y^(N-1)
        RP_ROLLED for (uint32_t v = 0; v < TH; v++) T.A_hi[v] = rp_mul(gA, T.s_hi[v]);
    }
    {
        const sc hB = rp_mul(rp_to_mont(sc_load(proof + 256 + 64 * k)), rhoU);                 // b rho U
        RP_ROLLED for (uint32_t v = 0; v < TL; v++) T.Q_lo[v] = rp_mul(T.y_lo[v ^ (TL - 1)], T.s_lo[v ^ (TL - 1)]);
        RP_ROLLED for (uint32_t v = 0; v < TH; v++) T.Q_hi[v] = rp_mul(rp_mul(hB, T.y_hi[v ^ (TH - 1)]), T.s_hi[v ^ (TH - 1)]);
    }
    {
        // F(i) = 2^(i mod n) z^(i div n) over the two index groups; the power of z only grows with v (at most m - 1 products in all)
        sc zf = one; uint32_t ze = 0;
        RP_ROLLED for (uint32_t v = 0; v < TL; v++) {
            RP_ROLLED for (; ze < v / n; ze++) zf = rp_mul(zf, z);
            T.P_lo[v] = rp_mul(T.y_lo[v ^ (TL - 1)], rp_mul(pow2[v % n], zf));
        }
        const sc hA = rp_mul(rhoUU, rp_mul(z, z));                                              // rho U^2 z^2
        zf = one; ze = 0;
        RP_ROLLED for (uint32_t v = 0; v < TH; v++) {
            const uint64_t idx = (uint64_t)v << kl;
            RP_ROLLED for (; ze < idx / n; ze++) zf = rp_mul(zf, z);
            T.P_hi[v] = rp_mul(rp_mul(hA, T.y_hi[v ^ (TH - 1)]), rp_mul(pow2[idx % n], zf));
        }
    }
    return BP_PROOF_OK;
}
