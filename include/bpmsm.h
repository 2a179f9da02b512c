/* bpmsm.h — C ABI of the H100-native Ristretto255 multiscalar-multiplication engine.
 *
 * This is the drop-in boundary for the MSM-bound hot path of dalek-cryptography/bulletproofs.
 * The reference has no FFI; its only seam is the Rust trait surface of curve25519_dalek::traits
 * that the crate calls.  Each entry point below names the reference call site it replaces; the
 * Rust-side binding a maintainer would add is shown in INTEGRATION.md.
 *
 * Wire types (SURVEY.md §8b):
 *   scalar            32 bytes, little-endian, canonical (< l)          = curve25519_dalek::scalar::Scalar::as_bytes()
 *   compressed point  32 bytes, canonical Ristretto255 encoding         = CompressedRistretto::as_bytes()
 *   transcript        203 bytes: STROBE-128 state (200) ‖ pos ‖ pos_begin ‖ cur_flags  = merlin::Transcript fields
 *
 * Ownership: the caller owns every host buffer for the duration of the call; the library copies
 * in and out and retains nothing except the explicit handles (bp_ctx, bp_gens).
 * Threading: a bp_ctx is one device + one CUDA stream and is not thread-safe; different
 * contexts may be used concurrently.  There is no hidden global state and no CPU fallback:
 * every call fails with BP_ERR_CUDA when no sm_90 (H100) device is usable.
 * Timing: all work is variable-time (like the reference's vartime_* calls).  The reference's
 * constant-time `multiscalar_mul` sites (prover secrets) are served by the same variable-time
 * kernels; see DESIGN.md "constant-time policy".
 */
#ifndef BPMSM_H
#define BPMSM_H
#include <stddef.h>
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

/* call status */
#define BP_OK 0
#define BP_ERR_INVALID_POINT 1        /* a point failed to decompress: optional_multiscalar_mul -> None (range_proof/mod.rs:445) */
#define BP_ERR_LENGTH_MISMATCH 2      /* the reference panics (assert_eq!, inner_product_proof.rs:59-67) */
#define BP_ERR_NONCANONICAL_SCALAR 3  /* scalar bytes >= l: Scalar::from_canonical_bytes -> None */
#define BP_ERR_CUDA 4                 /* no device / launch failure; bp_last_error() has the text */
#define BP_ERR_INVALID_ARGUMENT 5

/* per-proof verdicts = ProofError variants (src/errors.rs:12-54) */
#define BP_PROOF_OK 0
#define BP_PROOF_VERIFICATION_ERROR 1
#define BP_PROOF_FORMAT_ERROR 2
#define BP_PROOF_INVALID_BITSIZE 3
#define BP_PROOF_INVALID_GENERATORS_LENGTH 4
#define BP_PROOF_INVALID_AGGREGATION 5

#define BP_TRANSCRIPT_BYTES 203

typedef struct bp_ctx bp_ctx;
typedef struct bp_gens bp_gens;

/* ---- context ------------------------------------------------------------------------------- */
/* stream: a cudaStream_t to run on (e.g. torch.cuda.current_stream().cuda_stream), or NULL to
 * create a private non-blocking stream. */
int bp_ctx_create(int device, void *stream, bp_ctx **out);
void bp_ctx_destroy(bp_ctx *ctx);
const char *bp_last_error(const bp_ctx *ctx);
/* number of kernels this context has launched so far (bench.py's gpu_launches) */
uint64_t bp_ctx_launch_count(const bp_ctx *ctx);
/* Pippenger window size (bits) of the generic MSM entry points on this context: 0 = chosen by terms per MSM (default), 2..18 = fixed.
 * Results do not depend on it; tests use it to cover every window geometry, benchmarks to tune. */
int bp_ctx_set_msm_window(bp_ctx *ctx, int window_bits);
/* block until all work queued on the context's stream is finished */
int bp_ctx_synchronize(bp_ctx *ctx);

/* ---- group primitives ---------------------------------------------------------------------- */
/* CompressedRistretto::decompress for n points: ok[i] = 1 if point i is a valid encoding.
 * Replaces the inline decompress() calls of range_proof/mod.rs:433-443. */
int bp_decompress_check_batch(bp_ctx *ctx, const uint8_t *points, size_t n, uint8_t *ok);
/* RistrettoPoint::from_uniform_bytes (generators.rs:94-99) for n 64-byte inputs -> n compressed points */
int bp_from_uniform_bytes_batch(bp_ctx *ctx, const uint8_t *uniform, size_t n, uint8_t *points_out);

/* ---- multiscalar multiplication ------------------------------------------------------------ */
/* RistrettoPoint::vartime_multiscalar_mul / optional_multiscalar_mul on wire types:
 *   out = compress( sum_i scalars[i] * decompress(points[i]) ).
 * Call sites replaced: inner_product_proof.rs:87,101,127,131,153,159,177,178,308;
 * range_proof/mod.rs:421; range_proof/messages.rs:128,149; generators.rs:40; range_proof/party.rs:119.
 * Returns BP_ERR_INVALID_POINT if any point does not decode (the reference's `None`). */
int bp_msm(bp_ctx *ctx, const uint8_t *scalars, const uint8_t *points, size_t n, uint8_t out[32]);
/* n_msm independent MSMs in one launch sequence: MSM j uses terms offsets[j] .. offsets[j+1]-1.
 * outs = n_msm x 32 bytes; status[j] = BP_OK / BP_ERR_INVALID_POINT / BP_ERR_NONCANONICAL_SCALAR. */
int bp_msm_batch(bp_ctx *ctx, const uint8_t *scalars, const uint8_t *points, const uint64_t *offsets,
                 size_t n_msm, uint8_t *outs, uint8_t *status);
/* Same with every array already resident in device memory; work is queued on the context's stream and the call returns without
 * synchronising.  d_scalars (total_terms x 32 B), d_points (total_terms x 32 B) and d_outs (n_msm x 32 B) must be 16-byte aligned,
 * d_offsets_u32 (n_msm + 1 words) 4-byte aligned; d_status (n_msm bytes, optional) may have any alignment.  A misaligned pointer
 * gives BP_ERR_INVALID_ARGUMENT with a message in bp_last_error(). */
int bp_msm_batch_device(bp_ctx *ctx, const void *d_scalars, const void *d_points, const void *d_offsets_u32,
                        size_t n_msm, size_t total_terms, void *d_outs, void *d_status);

/* MSMs whose points are generator-table entries and/or caller-supplied compressed points:
 * point_idx[t] < 2^31 selects table slot point_idx[t] of `gens` (layout of bp_gens_device_table: 0 = B_blinding,
 * 1 = B, 2 + party*cap + i = G[party][i], 2 + parties*cap + party*cap + i = H[party][i]); point_idx[t] = 2^31 | j
 * selects dyn_points[j].  This is how the prover-side constant-base call sites run without re-uploading the table:
 * PedersenGens::commit (generators.rs:39-41), A and S (range_proof/party.rs:100-124), T_1/T_2 (party.rs:216-217),
 * Q = w*B (dealer.rs:256), and the stand-alone IPP verification MSM (inner_product_proof.rs:308-319). */
int bp_msm_indexed_batch(bp_ctx *ctx, bp_gens *gens, const uint8_t *scalars, const uint32_t *point_idx,
                         const uint8_t *dyn_points, size_t n_dyn, const uint64_t *offsets, size_t n_msm,
                         uint8_t *outs, uint8_t *status);

/* ---- point values across the boundary ------------------------------------------------------- */
/* CompressedRistretto::decompress() -> Option<RistrettoPoint> for n points (call sites src/range_proof/mod.rs:433-443,
 * src/inner_product_proof.rs:296-306, src/r1cs/verifier.rs:482): xyzt_out[i] = the extended coordinates X | Y | Z | T of point i as
 * four canonical 32-byte field elements (Z = 1) -- an in-memory RistrettoPoint a host caller can keep; ok[i] = 0 where the
 * reference would return None (the slot then holds the identity).  bp_compress_batch is RistrettoPoint::compress()
 * (src/inner_product_proof.rs:99,113, src/range_proof/dealer.rs:113-116) on such values (any projective representative). */
int bp_decompress_batch(bp_ctx *ctx, const uint8_t *points, size_t n, uint8_t *xyzt_out, uint8_t *ok);
int bp_compress_batch(bp_ctx *ctx, const uint8_t *xyzt, size_t n, uint8_t *points_out);

/* ---- resident point sets ------------------------------------------------------------------- */
/* A vector of n points decompressed once and kept on the device (affine Niels form, 96 B/point): the bases of repeated MSMs
 * (`Vec<RistrettoPoint>` reused across vartime_multiscalar_mul calls, e.g. the generator vectors of inner_product_proof.rs:87-178).
 * BP_ERR_INVALID_POINT if any encoding is invalid.  Device form: d_points (n x 32 B compressed) must be 16-byte aligned, else
 * BP_ERR_INVALID_ARGUMENT. */
typedef struct bp_points bp_points;
int bp_points_create(bp_ctx *ctx, const uint8_t *points, size_t n, bp_points **out);
int bp_points_create_device(bp_ctx *ctx, const void *d_points, size_t n, bp_points **out);
void bp_points_destroy(bp_points *set);
size_t bp_points_count(const bp_points *set);
/* n_msm MSMs of `terms` terms each over the first `terms` points of the set; MSM j takes scalars[j*terms .. (j+1)*terms).
 * Device form: d_scalars / d_outs (n_msm x 32 B) / d_status (n_msm bytes, optional) are device pointers, nothing is synchronised;
 * d_scalars and d_outs must be 16-byte aligned (else BP_ERR_INVALID_ARGUMENT), d_status may have any alignment.
 * Host form: pinned memory recommended; synchronises. */
int bp_msm_points_device(bp_ctx *ctx, bp_points *set, const void *d_scalars, size_t n_msm, size_t terms, void *d_outs, void *d_status);
int bp_msm_points(bp_ctx *ctx, bp_points *set, const uint8_t *scalars, size_t n_msm, size_t terms, uint8_t *outs, uint8_t *status);

/* ---- inner-product prover, device-resident (no generator folding) ---------------------------- */
/* InnerProductProof::create (src/inner_product_proof.rs:38-193) for n_proofs proofs of the same length N side by side.  The vectors
 * a, b, G_factors, H_factors stay on the device; the points are never folded -- round j's L and R are MSMs of N + 1 terms over the
 * ORIGINAL generators with the accumulated challenge products as coefficients (same group elements, hence the same proof bytes, as
 * the reference's folded form :127-134,177-178) -- so a round is O(N) scalar products and one MSM launch chain for all proofs.
 * The host keeps the transcripts: round() returns L, R (:87-113,153-163), the caller appends them, draws u (:118-121,168-171) and
 * calls fold(u, u^-1) (:122-134,172-178); after lg N rounds finish() returns the final a, b (:187-192).
 *   begin        : G, H = BulletproofGens::G(n, m) / H(n, m) of the resident table, N = n*m
 *   begin_points : arbitrary G, H (N compressed points each)
 *   Q  : n_proofs x 32 B;  a, b : n_proofs x N canonical scalars;  G_factors / H_factors : likewise, or NULL for all ones. */
typedef struct bp_ippx bp_ippx;
int bp_ippx_begin(bp_ctx *ctx, bp_gens *gens, size_t n, size_t m, size_t n_proofs, const uint8_t *Q, const uint8_t *G_factors, const uint8_t *H_factors,
                  const uint8_t *a, const uint8_t *b, bp_ippx **out);
int bp_ippx_begin_points(bp_ctx *ctx, const uint8_t *G, const uint8_t *H, size_t N, size_t n_proofs, const uint8_t *Q, const uint8_t *G_factors, const uint8_t *H_factors,
                         const uint8_t *a, const uint8_t *b, bp_ippx **out);
size_t bp_ippx_current_len(const bp_ippx *sess);
int bp_ippx_round(bp_ippx *sess, uint8_t *LR_out /* n_proofs x 64 */);
int bp_ippx_fold(bp_ippx *sess, const uint8_t *u /* n_proofs x 32 */, const uint8_t *u_inv);
int bp_ippx_finish(bp_ippx *sess, uint8_t *ab_out /* n_proofs x 64 */);
void bp_ippx_end(bp_ippx *sess);

/* ---- generator tables ---------------------------------------------------------------------- */
/* BulletproofGens::new(gens_capacity, party_capacity) + PedersenGens::default()
 * (generators.rs:44-53,157-204): SHAKE256 expansion on the host, Elligator maps and the
 * table (affine Niels form, 96 B/point) on the device, where it stays resident. */
int bp_gens_create(bp_ctx *ctx, size_t gens_capacity, size_t party_capacity, bp_gens **out);
void bp_gens_destroy(bp_gens *gens);
/* compressed generator: which = 0 -> G, 1 -> H (party, index); 2 -> B; 3 -> B_blinding */
int bp_gens_get(bp_gens *gens, int which, size_t party, size_t index, uint8_t out[32]);
/* device pointer + size of the resident table, layout [B_blinding, B, G[party][i]..., H[party][i]...]:
 * this is the buffer broadcast once over NCCL at start-up (SURVEY.md §8e). */
int bp_gens_device_table(bp_gens *gens, void **d_table, size_t *bytes);
/* an uninitialised table of the same geometry, to be filled by a broadcast from rank 0 */
int bp_gens_create_empty(bp_ctx *ctx, size_t gens_capacity, size_t party_capacity, bp_gens **out);

/* ---- range proofs -------------------------------------------------------------------------- */
/* Batch verifier (SURVEY.md §8a row A6): `count` proofs with the same (n, m), each proof_len =
 * 32*(9 + 2*lg(n*m)) bytes as written by RangeProof::to_bytes (range_proof/mod.rs:487-499), each
 * with m commitments.  Every proof is checked exactly as RangeProof::verify_multiple
 * (range_proof/mod.rs:345-452) would: verdict[i] = BP_PROOF_OK iff the reference returns Ok(()).
 * All proofs start from the same transcript state (the *_transcripts forms below give each proof its own).  Internally one random-linear-combination
 * MSM covers the whole batch; if it does not vanish, every proof is re-checked on its own.  Small calls (at most 8 proofs with
 * lg(n*m) <= 6) are instead checked proof by proof in one launch, one thread-block cluster per proof with that proof's own MSM:
 * the same verdicts, with the latency of one launch rather than the pipeline's ~15.
 * When more than four chunks of 32 proofs fail, that re-check covers the whole batch at once with count*(S + D) terms
 * (S = 2 + 2nm, D = 4 + 2lg(nm) + m): beyond 2^31 terms the call returns BP_ERR_INVALID_ARGUMENT, which at n*m = 2^20 is
 * from about 1000 proofs, and it needs tens of GB of scratch well before that.
 * seed: 32 bytes of external randomness for the batching weights, or NULL to draw from the OS.  The weights of a proof
 * (the reference's `c = Scalar::random(rng)`, mod.rs:396, and the proof's weight in the combination) are squeezed from a fork
 * of that proof's final transcript state rekeyed with its inner-product scalars a || b (the proof bytes the transcript does not
 * absorb) and keyed with the seed -- merlin's `build_rng().rekey_with_witness_bytes(..).finalize(rng)` construction -- so they
 * depend on every proof byte even when the caller's seed is fixed or known.
 * Rejected parameters follow the reference's order, from_bytes (mod.rs:497-538) before verify_multiple's checks (mod.rs:358-366):
 * a proof_len that no proof can have gives every proof BP_PROOF_FORMAT_ERROR.  Otherwise, when n is not 8/16/32/64
 * (BP_PROOF_INVALID_BITSIZE), the generators are too few (BP_PROOF_INVALID_GENERATORS_LENGTH) or n*m differs from the 2^k the
 * length implies (BP_PROOF_VERIFICATION_ERROR), a proof whose t_x, t_x_blinding, e_blinding, a or b is not canonical gets
 * BP_PROOF_FORMAT_ERROR and every other proof gets that parameter code.  The device-resident entry points return
 * BP_ERR_INVALID_ARGUMENT for any rejected parameters instead. */
int bp_rangeproof_verify_batch(bp_ctx *ctx, bp_gens *gens, const uint8_t transcript[BP_TRANSCRIPT_BYTES],
                               const uint8_t *proofs, size_t proof_len, const uint8_t *commitments,
                               size_t n, size_t m, size_t count, const uint8_t seed[32], uint8_t *verdicts);
/* Asynchronous form for pipelining host buffers (pinned memory recommended): queues the H2D copies,
 * all kernels and the D2H copy of the verdicts on the context's stream; call
 * bp_rangeproof_verify_finish() to synchronise and run the rare per-proof fallback. */
int bp_rangeproof_verify_begin(bp_ctx *ctx, bp_gens *gens, const uint8_t transcript[BP_TRANSCRIPT_BYTES],
                               const uint8_t *proofs, size_t proof_len, const uint8_t *commitments,
                               size_t n, size_t m, size_t count, const uint8_t seed[32]);
int bp_rangeproof_verify_finish(bp_ctx *ctx, uint8_t *verdicts);
/* Device-resident form: proofs/commitments are device pointers; verdicts stay on the device
 * (count x uint32) and nothing is synchronised, so calls can be queued back to back on one context.
 * There is no per-proof recheck on this path: if the combined check fails, every well-formed proof of the
 * batch is marked BP_PROOF_VERIFICATION_ERROR and *h_batch_ok_pinned (optional, pinned) becomes 0 — rerun such a
 * batch through bp_rangeproof_verify_batch for per-proof verdicts.  Used for the HBM-resident throughput measurement.
 * d_proofs and d_commitments may have any alignment (16-byte aligned ones are read with bulk copies); d_verdicts_u32 must be
 * 4-byte aligned, else BP_ERR_INVALID_ARGUMENT. */
int bp_rangeproof_verify_batch_device(bp_ctx *ctx, bp_gens *gens, const uint8_t transcript[BP_TRANSCRIPT_BYTES],
                                      const void *d_proofs, size_t proof_len, const void *d_commitments,
                                      size_t n, size_t m, size_t count, const uint8_t seed[32], void *d_verdicts_u32,
                                      uint32_t *h_batch_ok_pinned);

/* Launch groups: `n_batches` (<= 256) independent batches of `count` proofs each in ONE launch sequence, so that the grids of a
 * group fill the 132 SMs of an H100 where a single 1024-proof batch gives most kernels less than one wave.  The group is checked
 * first with ONE random-linear-combination MSM over all of its proofs (every proof keeps its own independent weights).  When that
 * combination vanishes, every batch is accepted exactly as its own check would accept it.  Otherwise each batch's own combined MSM
 * runs on the device (no host round trip) and decides that batch's accept flag, and the per-proof fallback of the host path runs for
 * the failing batches only.  Verdicts and flags are the same as with one MSM per batch; a failing group costs one group MSM more.
 * proofs / commitments / verdicts are laid out batch after batch (n_batches*count entries); batch_ok (optional): n_batches flags,
 * 1 = every proof of that batch accepted.  The single-batch entry points above are the n_batches = 1 case. */
int bp_rangeproof_verify_group_begin(bp_ctx *ctx, bp_gens *gens, const uint8_t transcript[BP_TRANSCRIPT_BYTES],
                                     const uint8_t *proofs, size_t proof_len, const uint8_t *commitments,
                                     size_t n, size_t m, size_t count, size_t n_batches, const uint8_t seed[32]);
int bp_rangeproof_verify_group_finish(bp_ctx *ctx, uint8_t *verdicts, uint8_t *batch_ok);
/* Between *_begin and *_finish the context's arenas belong to the pending verification (its reject path reads them): every other
 * entry point on that context returns BP_ERR_INVALID_ARGUMENT with a message in bp_last_error(); use another context for concurrent work.
 * A failed *_begin leaves nothing pending. */
/* device-resident form (see bp_rangeproof_verify_batch_device, alignment rules included); h_batch_ok_pinned (optional, pinned):
 * n_batches x uint32 */
int bp_rangeproof_verify_group_device(bp_ctx *ctx, bp_gens *gens, const uint8_t transcript[BP_TRANSCRIPT_BYTES],
                                      const void *d_proofs, size_t proof_len, const void *d_commitments,
                                      size_t n, size_t m, size_t count, size_t n_batches, const uint8_t seed[32], void *d_verdicts_u32,
                                      uint32_t *h_batch_ok_pinned);
/* Reserve a geometry on a context: sizes every arena the verification of n_batches x count (n, m)-proofs touches, builds the
 * term->point maps, captures the launch sequence as a CUDA graph (two branches: decompression beside transcript replay) and runs
 * it once.  Afterwards no call with this geometry allocates, and each call costs one parameter upload + one graph launch.
 * Other geometries still work on the same context (direct launches, arenas grown on demand). */
int bp_rangeproof_verify_reserve(bp_ctx *ctx, bp_gens *gens, size_t n, size_t m, size_t count, size_t n_batches);
/* Proofs of any geometry in one call: RangeProof::from_bytes + verify_multiple(gens, pc_gens, transcript, value_commitments, n) for
 * each proof (mod.rs:345-452, 505-538), every proof from the same transcript state.  Proof i is the bytes
 * proofs[proof_offsets[i] .. proof_offsets[i+1]), its m_i = commit_offsets[i+1] - commit_offsets[i] value commitments start at
 * commitments + 32*commit_offsets[i], and n[i] is its bit size.  verdicts[i] is what bp_rangeproof_verify_batch returns for proof i
 * alone (count = 1, same transcript), parameter codes included: they apply per proof, and a rejected proof has no effect on the
 * others.  The admitted proofs are checked with one combined MSM; the batching weights are those of bp_rangeproof_verify_batch
 * (seed NULL: 32 bytes from the OS).  Synchronises.  BP_ERR_INVALID_ARGUMENT (message in bp_last_error) for a NULL argument,
 * count == 0, offsets that do not start at 0 or that decrease, 2^24 proofs or more, 2^31 MSM terms or more, or a pending
 * bp_rangeproof_verify_group_begin. */
int bp_rangeproof_verify_mixed(bp_ctx *ctx, bp_gens *gens, const uint8_t transcript[BP_TRANSCRIPT_BYTES], size_t count,
                               const uint8_t *proofs, const uint64_t *proof_offsets, const uint32_t *n,
                               const uint8_t *commitments, const uint64_t *commit_offsets, const uint8_t seed[32], uint8_t *verdicts);

/* Proofs that each start from their own transcript (RangeProof::verify_multiple with a `&mut Transcript` per proof, e.g. one bound to a
 * transaction hash or an output index).  Each mirrors the entry point of the same name without the suffix, `transcripts` in place of
 * `transcript`: one serialized state per proof (BP_TRANSCRIPT_BYTES each, back to back, any alignment), in proof order -- batch after
 * batch for the launch groups, input order for the mixed call; the layout of bp_linear_verify_batch's transcripts.  verdicts[i] is what
 * bp_rangeproof_verify_batch returns for proof i alone (count = 1) with record i as its transcript; parameter codes follow the same
 * rules and order.  A record that no Merlin transcript can hold between operations (pos >= 166, the STROBE-128 rate, or
 * pos_begin > pos) gives its proof BP_PROOF_FORMAT_ERROR; such a proof is left out of the combination like any rejected proof.  A call
 * on a geometry reserved with bp_rangeproof_verify_reserve replays the reserved graph and allocates nothing.
 *   _group_begin_transcripts: host buffers; collect the result with bp_rangeproof_verify_group_finish (n_batches = 1: one batch).
 *   _group_device_transcripts: d_transcripts is a device pointer (any alignment); nothing is synchronised; h_batch_ok_pinned as for
 *                              bp_rangeproof_verify_group_device.
 *   _mixed_transcripts: proofs of any geometry; synchronises. */
int bp_rangeproof_verify_group_begin_transcripts(bp_ctx *ctx, bp_gens *gens, const uint8_t *transcripts, const uint8_t *proofs, size_t proof_len,
                                                 const uint8_t *commitments, size_t n, size_t m, size_t count, size_t n_batches, const uint8_t seed[32]);
int bp_rangeproof_verify_group_device_transcripts(bp_ctx *ctx, bp_gens *gens, const void *d_transcripts, const void *d_proofs, size_t proof_len,
                                                  const void *d_commitments, size_t n, size_t m, size_t count, size_t n_batches, const uint8_t seed[32],
                                                  void *d_verdicts_u32, uint32_t *h_batch_ok_pinned);
int bp_rangeproof_verify_mixed_transcripts(bp_ctx *ctx, bp_gens *gens, const uint8_t *transcripts, size_t count, const uint8_t *proofs,
                                           const uint64_t *proof_offsets, const uint32_t *n, const uint8_t *commitments, const uint64_t *commit_offsets,
                                           const uint8_t seed[32], uint8_t *verdicts);

/* Reserve a mix on a context: n_classes (<= 24) classes of distinct (n[c], m[c]), each admitted by the generator table, with room for
 * capacity[c] > 0 proofs each.  Sizes every arena of the mix (its own, apart from those of the reserved geometry and of mixed calls that
 * do not fit), builds each class's term->point map and transcript step program once, captures the launch sequence as a CUDA graph and
 * runs it once.  BP_ERR_INVALID_ARGUMENT (message in bp_last_error) for a NULL argument, no class or more than 24, a duplicate class, a
 * class the generators reject, zero capacity, 2^24 proof slots or more, or 2^31 MSM terms or more.  Reserving again replaces the mix. */
int bp_rangeproof_verify_mixed_reserve(bp_ctx *ctx, bp_gens *gens, size_t n_classes, const uint32_t *n, const uint32_t *m, const uint32_t *capacity);
/* Asynchronous forms of bp_rangeproof_verify_mixed / _mixed_transcripts, same arguments without verdicts.  A call FITS the reserved mix
 * when gens is the reserved table, every admitted proof's (n, m) is a reserved class, no class receives more proofs than its capacity,
 * and the proof and commitment buffers are no larger than those of the mix filled to capacity (rejected proofs add bytes).  A fitting
 * call allocates nothing: it queues the H2D copies, one gather kernel, one graph launch and the D2H copies of verdicts and flags on the
 * context's stream and returns without synchronising; keep proofs, commitments and transcripts alive and unchanged until *_finish
 * (pinned memory recommended).  A class's slots beyond the proofs a call gives it are inert and cost no front-end work.  Any other call
 * (or a call while bp_prof_enable is on) runs the direct launches of bp_rangeproof_verify_mixed and synchronises inside *_begin.
 * bp_rangeproof_verify_mixed(_transcripts) are *_begin followed by *_finish, so they use the reserved graph too.  Pending rules as
 * for bp_rangeproof_verify_group_begin: until *_finish every other entry point on the context (group calls and their finish included)
 * returns BP_ERR_INVALID_ARGUMENT. */
int bp_rangeproof_verify_mixed_begin(bp_ctx *ctx, bp_gens *gens, const uint8_t transcript[BP_TRANSCRIPT_BYTES], size_t count,
                                     const uint8_t *proofs, const uint64_t *proof_offsets, const uint32_t *n,
                                     const uint8_t *commitments, const uint64_t *commit_offsets, const uint8_t seed[32]);
int bp_rangeproof_verify_mixed_begin_transcripts(bp_ctx *ctx, bp_gens *gens, const uint8_t *transcripts, size_t count, const uint8_t *proofs,
                                                 const uint64_t *proof_offsets, const uint32_t *n, const uint8_t *commitments,
                                                 const uint64_t *commit_offsets, const uint8_t seed[32]);
/* Synchronise, run the reject path of each class whose own check failed (its live proofs only) and write the count verdicts of the
 * pending mixed call in input order, parameter codes included.  BP_ERR_INVALID_ARGUMENT when no mixed call is pending. */
int bp_rangeproof_verify_mixed_finish(bp_ctx *ctx, uint8_t *verdicts);

/* Verdict of a proof that a device-resident mixed call admitted but could not place in the reserved mix (see below). */
#define BP_VERDICT_UNPLACED 0xFFFFFFFFu
/* Device-resident forms of the reserved mix: every input is already in device memory, the proofs are placed in the mix reserved with
 * bp_rangeproof_verify_mixed_reserve by device kernels, the mix's captured graph runs, and the verdicts stay on the device.  The host does
 * work in the number of classes only and does not synchronise (the exceptions are below), so calls can be queued back to back on one
 * context; each keeps its own parameters.  Proof i is d_proofs[d_proof_offsets[i] .. d_proof_offsets[i+1]) (u64 offsets, count + 1 of them, need not start at 0) out
 * of proof_bytes bytes, its m_i = d_commit_offsets[i+1] - d_commit_offsets[i] commitments start at commitment d_commit_offsets[i] of the
 * n_commitments at d_commitments, and d_n[i] (u32) is its bit size.  d_proofs, both offset arrays, d_n, d_commitments and d_transcripts
 * (one BP_TRANSCRIPT_BYTES record per proof, input order) may have any alignment; keep them unchanged until the call has run on the stream.
 *   - Parameter codes, per proof, on the device: those bp_rangeproof_verify_mixed gives (rejected proofs with a non-canonical scalar
 *     included).  A proof whose offsets decrease, or whose bytes lie beyond proof_bytes / n_commitments, gets BP_PROOF_FORMAT_ERROR and
 *     none of its bytes is read (the host forms refuse such a call as a whole instead).
 *   - Placement: each admitted proof goes to the mix class of its (n, m); within a class proofs take slots in input order up to the
 *     class's capacity.  An admitted proof whose class is not in the mix, or that comes after the first `capacity` proofs of its class,
 *     gets BP_VERDICT_UNPLACED: which proofs those are depends on the input only, so a caller can resubmit exactly them.
 *   - Verdicts: d_verdicts_u32[i] (4-byte aligned) receives proof i's code in input order.  As on the fixed-geometry device path there is
 *     no per-proof re-check on the device: a class whose own check fails marks each of its well-formed proofs BP_PROOF_VERIFICATION_ERROR,
 *     and h_class_ok_pinned (optional, pinned, one u32 per class of the mix in reservation order) receives 0 for it, 1 for a class that
 *     was accepted or had no proof.  Rerun the proofs of a flagged class through bp_rangeproof_verify_mixed for their own verdicts,
 *     or use the _exact forms below, which give them on the device.
 *   - Launches per call are constant (the planner kernels, one gather, one graph launch, one verdict kernel), whatever count and fill.
 *     No allocation, unless count exceeds every earlier call's and the number of slots of the mix: the planner's scratch then grows,
 *     which waits for the work already queued on the context.  Each call stages its parameter blocks in one of 8 pinned stages, used
 *     in turn: a call whose stage's previous upload (8 calls earlier) has not run yet waits on the host until it has, so at most 8
 *     calls' uploads are ever pending on a context.  While bp_prof_enable is on, the planner kernels are timed (k_mix_plan) and the
 *     graph is not.
 * BP_ERR_INVALID_ARGUMENT (message in bp_last_error), with nothing queued, when no mix is reserved on the context or gens is not the
 * table it was reserved on, for a NULL argument, count == 0, count >= 2^24, a misaligned d_verdicts_u32, or while a *_begin call is
 * pending on the context. */
int bp_rangeproof_verify_mixed_device(bp_ctx *ctx, bp_gens *gens, const uint8_t transcript[BP_TRANSCRIPT_BYTES], size_t count,
                                      const void *d_proofs, size_t proof_bytes, const void *d_proof_offsets, const void *d_n,
                                      const void *d_commitments, size_t n_commitments, const void *d_commit_offsets, const uint8_t seed[32],
                                      void *d_verdicts_u32, uint32_t *h_class_ok_pinned);
int bp_rangeproof_verify_mixed_device_transcripts(bp_ctx *ctx, bp_gens *gens, const void *d_transcripts, size_t count, const void *d_proofs,
                                                  size_t proof_bytes, const void *d_proof_offsets, const void *d_n, const void *d_commitments,
                                                  size_t n_commitments, const void *d_commit_offsets, const uint8_t seed[32], void *d_verdicts_u32,
                                                  uint32_t *h_class_ok_pinned);

/* Exact device-resident forms: the verdicts of the host forms, on the device, without a host round trip.
 *   _reserve_exact: everything bp_rangeproof_verify_reserve / bp_rangeproof_verify_mixed_reserve does (same arguments, same refusals; the
 *     plain graph is captured as before, so plain calls on the context still replay it), and in addition a second graph, the exact graph:
 *     the same launch sequence, then the reject path of the host forms run by the device (level 1: one MSM per chunk of 32 proofs of every
 *     failing batch or class, in one pass; level 2: one MSM per proof of every failing chunk, a bounded number of proofs per iteration of
 *     a conditional WHILE node).  Its scratch belongs to the reserved geometry or mix.  Runs the exact graph once.  A geometry whose
 *     reject path would need 2^31 MSM terms or more is refused with BP_ERR_INVALID_ARGUMENT.
 *   _device_exact(_transcripts): the arguments and alignment rules of the entry point without "_exact".  d_verdicts_u32[i] receives
 *     exactly the code the host form gives for proof i with the same seed (bp_rangeproof_verify_group_begin(_transcripts) +
 *     _group_finish; bp_rangeproof_verify_mixed(_transcripts)); in the mixed form an unplaced proof still gets BP_VERDICT_UNPLACED.
 *     h_batch_ok_pinned / h_class_ok_pinned receive what the plain call writes: they still tell which batch or class went through the
 *     reject path, and need no action.  No synchronisation and no allocation; calls queue back to back on one context, each with its own
 *     parameters (the staging rules of the plain forms).  Launches per call are the same whatever the number of bad proofs.  The one
 *     exception: while bp_prof_enable is on, the fixed-geometry forms launch directly and then run the host forms' reject path, which
 *     synchronises (the mixed forms launch the exact graph, untimed, as the plain ones do).
 * BP_ERR_INVALID_ARGUMENT (message in bp_last_error), with nothing queued, where the plain form refuses, when the geometry or mix was not
 * reserved with *_reserve_exact on this context and generator table (a later reservation that moves the verifier's scratch, or another
 * mix, ends an exact reservation), or while a *_begin call is pending on the context. */
int bp_rangeproof_verify_reserve_exact(bp_ctx *ctx, bp_gens *gens, size_t n, size_t m, size_t count, size_t n_batches);
int bp_rangeproof_verify_group_device_exact(bp_ctx *ctx, bp_gens *gens, const uint8_t transcript[BP_TRANSCRIPT_BYTES],
                                            const void *d_proofs, size_t proof_len, const void *d_commitments,
                                            size_t n, size_t m, size_t count, size_t n_batches, const uint8_t seed[32], void *d_verdicts_u32,
                                            uint32_t *h_batch_ok_pinned);
int bp_rangeproof_verify_group_device_exact_transcripts(bp_ctx *ctx, bp_gens *gens, const void *d_transcripts, const void *d_proofs, size_t proof_len,
                                                        const void *d_commitments, size_t n, size_t m, size_t count, size_t n_batches,
                                                        const uint8_t seed[32], void *d_verdicts_u32, uint32_t *h_batch_ok_pinned);
int bp_rangeproof_verify_mixed_reserve_exact(bp_ctx *ctx, bp_gens *gens, size_t n_classes, const uint32_t *n, const uint32_t *m, const uint32_t *capacity);
int bp_rangeproof_verify_mixed_device_exact(bp_ctx *ctx, bp_gens *gens, const uint8_t transcript[BP_TRANSCRIPT_BYTES], size_t count,
                                            const void *d_proofs, size_t proof_bytes, const void *d_proof_offsets, const void *d_n,
                                            const void *d_commitments, size_t n_commitments, const void *d_commit_offsets, const uint8_t seed[32],
                                            void *d_verdicts_u32, uint32_t *h_class_ok_pinned);
int bp_rangeproof_verify_mixed_device_exact_transcripts(bp_ctx *ctx, bp_gens *gens, const void *d_transcripts, size_t count, const void *d_proofs,
                                                        size_t proof_bytes, const void *d_proof_offsets, const void *d_n, const void *d_commitments,
                                                        size_t n_commitments, const void *d_commit_offsets, const uint8_t seed[32], void *d_verdicts_u32,
                                                        uint32_t *h_class_ok_pinned);

/* ---- R1CS proofs --------------------------------------------------------------------------- */
/* Batch verifier for r1cs::Verifier::verify (src/r1cs/verifier.rs:329-500, SURVEY.md §8a row A7): the mega-check MSM
 * (verifier.rs:398-497) of n_proofs proofs, each of its own circuit and size, after the host has run each proof's transcript phase
 * (verifier.rs:339-449: transcript, flattened constraints, verification scalars, r).  verdicts[j] = BP_PROOF_OK or
 * BP_PROOF_VERIFICATION_ERROR: exactly what proof j's own mega-check gives.  Internally one random-linear-combination MSM covers the
 * batch, with the G/H scalars summed over the proofs on the device; if it does not vanish every proof is re-checked on its own.
 * Inputs, flat, proofs back to back:
 *   dims       4 per proof: padded_n (a power of two, <= the generators' capacity), n1 (first-phase multipliers), n (multipliers),
 *              n_terms (other terms)
 *   chal       7 + lg(padded_n) scalars per proof: x, y^-1, u, a, b, rho, s_0 = prod u_j^-1, u_sq[0..lg padded_n).  rho is the
 *              proof's weight in the combination: uniformly random and bound to every byte of the proof (r1cs::verify_batch squeezes
 *              it from a TranscriptRng of the proof's transcript rekeyed with a || b).
 *   wL, wR, wO n scalars per proof (the flattened constraints, verifier.rs:260-298).  The device builds the G_i / H_i scalars
 *              u1 (x y^-i wR_i - a s_i) and u1 (y^-i (x wL_i + wO_i - b s_{N-1-i}) - 1), u1 = 1 for i < n1 and u otherwise, i < padded_n.
 *   scalars, point_idx   n_terms per proof: every other term of the mega-check (A_I1, A_O1, S1, A_I2, A_O2, S2, V, T_1, T_3..T_6,
 *              B, B_blinding, L, R), unweighted, point_idx encoded as for bp_msm_indexed_batch (dynamic indices address dyn_points).
 * A proof that uses an undecodable point gets BP_PROOF_VERIFICATION_ERROR (optional_multiscalar_mul -> None) and is left out of the
 * combination.  BP_ERR_INVALID_ARGUMENT (message in bp_last_error) for inconsistent dims, a slot or dynamic index out of range, or a
 * pending range-proof verification; BP_ERR_NONCANONICAL_SCALAR for a scalar >= l. */
int bp_r1cs_verify_batch(bp_ctx *ctx, bp_gens *gens, size_t n_proofs, const uint32_t *dims, const uint8_t *chal,
                         const uint8_t *wL, const uint8_t *wR, const uint8_t *wO, const uint8_t *scalars, const uint32_t *point_idx,
                         const uint8_t *dyn_points, size_t n_dyn, uint8_t *verdicts);

/* ---- linear proofs ------------------------------------------------------------------------- */
/* Batch verifier for LinearProof::verify (src/linear_proof.rs:184-237): `count` proofs of one length n over the same generators, held
 * as one resident point set `set` = [B, F, G_0 .. G_{n-1}, ...] (the order LinearProof::create builds).  Per proof j, back to back:
 * its serialized transcript (transcripts, count x BP_TRANSCRIPT_BYTES), its proof bytes (proofs, count x proof_len), its commitment C
 * (C, count x 32) and its public vector b (b, count x n x 32, canonical scalars).  verdicts[j] = what LinearProof::from_bytes + verify
 * return for proof j with G = set[2 .. n+2), F = set[1], B = set[0], checked in this order: BP_PROOF_FORMAT_ERROR for a proof_len no
 * proof can have (every proof) or a non-canonical a or r; BP_PROOF_INVALID_GENERATORS_LENGTH when the set has fewer than n + 2
 * points; BP_PROOF_VERIFICATION_ERROR when n is not 2^(rounds of proof_len), and otherwise BP_PROOF_OK or BP_PROOF_VERIFICATION_ERROR.
 * The transcripts are replayed on the device; one random-linear-combination MSM decides the batch (weights drawn from each proof's
 * transcript, its a || r and the seed, as for the range-proof batch; seed NULL = 32 bytes from the OS), and when it does not vanish every proof is
 * re-checked on its own.  A proof with a point that does not decode is rejected and left out of the combination.  Synchronises.
 * Small calls (at most 16 proofs of n <= 1024, whose parameters passed) take a fused path instead: the host replays each transcript
 * while the proofs are copied to the device, and one thread-block-cluster launch checks every proof's own equation; the returns and
 * verdicts are the same, and the seed is not used.
 * BP_ERR_NONCANONICAL_SCALAR for a b entry >= l; BP_ERR_INVALID_ARGUMENT (message in bp_last_error) for NULL arguments, count == 0,
 * more than 2^20 proofs, n above 2^20, a set of another context, or a pending range-proof verification. */
int bp_linear_verify_batch(bp_ctx *ctx, bp_points *set, size_t n, size_t count, const uint8_t *transcripts, const uint8_t *proofs,
                           size_t proof_len, const uint8_t *C, const uint8_t *b, const uint8_t seed[32], uint8_t *verdicts);

/* Device-resident LinearProof batches over a reservation.
 *   _reserve: reserve proofs of length n over `set`, at most `capacity` per call, on the context.  Sizes the reservation's own arenas
 *     (so a blocking bp_linear_verify_batch on the same context may grow its own without moving them), captures the verifier as a CUDA
 *     graph and runs it once.  Synchronises.  Reserving again replaces the reservation; bp_points_destroy of the reserved set ends it.
 *     BP_ERR_INVALID_ARGUMENT (message in bp_last_error) for a set of another context or with fewer than n + 2 points, n not a power of
 *     two or above 2^20, capacity 0 or above 2^20, 2^31 MSM terms or more, or a pending range-proof verification.
 *   _device: `count` proofs in device memory, in the layout of bp_linear_verify_batch (d_transcripts, d_proofs, d_C, d_b; any alignment;
 *     keep them unchanged until the call has run on the stream).  Stages the seed (NULL: 32 bytes from the OS) and count in one of 8 pinned
 *     slots used in turn (a call whose slot is still pending 8 calls later waits on the host), copies the inputs into the reservation,
 *     launches its graph and returns without synchronising: calls queue back to back, each with its own parameters, and launch the same
 *     kernels whatever the number of bad proofs.  d_verdicts_u32[j] (4-byte aligned) receives the code bp_linear_verify_batch gives proof
 *     j with the same seed, the reject path run on the device; a proof with a b entry >= l gets BP_VERDICT_NONCANONICAL_B and is left out
 *     of the combination (the blocking form refuses such a call as a whole).  *h_ok_pinned (optional, pinned) receives 1 when the combined
 *     check passed, 0 when the reject path ran.  BP_ERR_INVALID_ARGUMENT (message in bp_last_error), with nothing queued, when no
 *     reservation on the context matches set and n, for count 0 or above the capacity, a NULL argument, a misaligned d_verdicts_u32,
 *     proof_len != 32 (2 lg n + 3), or a pending range-proof verification. */
#define BP_VERDICT_NONCANONICAL_B 0xFFFFFFFEu
int bp_linear_verify_reserve(bp_ctx *ctx, bp_points *set, size_t n, size_t capacity);
int bp_linear_verify_device(bp_ctx *ctx, bp_points *set, size_t n, size_t count, const void *d_transcripts, const void *d_proofs,
                            size_t proof_len, const void *d_C, const void *d_b, const uint8_t seed[32], void *d_verdicts_u32,
                            uint32_t *h_ok_pinned);

/* LinearProofs of any lengths in one call, over one resident point set `set` = [B, F, G_0, G_1, ...].  Proof j is
 * proofs[proof_offsets[j] .. proof_offsets[j+1]); its public vector is the n_j = b_offsets[j+1] - b_offsets[j] scalars from
 * b + 32 b_offsets[j] on; its commitment is C + 32 j and its transcript record transcripts + BP_TRANSCRIPT_BYTES j; its generators are
 * G = set[2 .. n_j + 2), F = set[1], B = set[0].  verdicts[j] is the code bp_linear_verify_batch(ctx, set, n_j, 1, ...) gives proof j on
 * its own: its parameters are checked per proof, in the reference's order (a length no proof can have, then a non-canonical a or r:
 * BP_PROOF_FORMAT_ERROR; a set of fewer than n_j + 2 points: BP_PROOF_INVALID_GENERATORS_LENGTH; n_j not 2^(rounds), n_j = 0 included:
 * BP_PROOF_VERIFICATION_ERROR), and a proof they reject is left out of the combination.  Every admitted proof, whatever its length, is
 * checked by ONE random-linear-combination MSM over [B, F, G_0 .. G_{Nmax-1} | C, S, L.., R.. of every proof], Nmax the longest admitted
 * n_j, with each proof's weight drawn as in bp_linear_verify_batch (its transcript, its a || r and the seed; seed NULL = 32 bytes from the
 * OS).  When that MSM does not vanish, every admitted proof is re-checked by its own equation.  Synchronises.  A call of at most 16
 * admitted proofs, none longer than n = 1024, takes the fused path of bp_linear_verify_batch, with the same returns and verdicts.
 * BP_ERR_NONCANONICAL_SCALAR for a b entry >= l; BP_ERR_INVALID_ARGUMENT (message in bp_last_error) for NULL arguments, count == 0,
 * more than 2^20 proofs, offsets that do not start at 0 or that decrease, an n_j above 2^20, 2^31 MSM terms or more, a set of another
 * context, or a pending range-proof verification. */
int bp_linear_verify_mixed(bp_ctx *ctx, bp_points *set, size_t count, const uint8_t *transcripts, const uint8_t *proofs,
                           const uint64_t *proof_offsets, const uint8_t *C, const uint8_t *b, const uint64_t *b_offsets,
                           const uint8_t seed[32], uint8_t *verdicts);

/* Device-resident LinearProofs of mixed lengths over a reserved mix.
 *   _mixed_reserve: reserve n_classes lengths n[c] over `set`, at most capacity[c] proofs of each per call, on the context.  Sizes the
 *     mix's own arenas, laid out at capacity one class per n in reservation order (so the blocking calls and a bp_linear_verify_reserve
 *     reservation on the same context keep theirs), captures the verifier as a CUDA graph and runs it once.  Synchronises.  Reserving
 *     again replaces the mix; bp_points_destroy of its set ends it.  BP_ERR_INVALID_ARGUMENT (message in bp_last_error) for 0 classes or
 *     more than 21, a duplicate n, an n that is not a power of two or is above 2^20, a set with fewer than n + 2 points, a capacity of 0
 *     or above 2^20, 2^31 MSM terms or more (the combined row Nmax + 2 + sum capacity[c] (2 + 2 lg n[c]) and every class's reject-path
 *     rows), a NULL argument, a set of another context, or a pending range-proof verification.
 *   _mixed_device: `count` proofs in device memory, in the layout of bp_linear_verify_mixed: proof i is d_proofs[po[i] .. po[i+1]) out of
 *     proof_bytes bytes (po = d_proof_offsets, u64, count + 1 entries, need not start at 0), its b is the bo[i+1] - bo[i] scalars from
 *     scalar bo[i] of the n_b at d_b (bo = d_b_offsets, u64), its C is d_C + 32 i and its transcript record d_transcripts +
 *     BP_TRANSCRIPT_BYTES i.  Every input may have any alignment; keep them unchanged until the call has run on the stream.
 *     - Parameter codes, per proof, on the device: those bp_linear_verify_mixed gives.  A proof whose offsets decrease or reach past
 *       proof_bytes / n_b gets BP_PROOF_FORMAT_ERROR and none of its bytes is read (the blocking form refuses such a call as a whole).
 *     - Placement: each admitted proof goes to the class of its n; within a class proofs take slots in input order up to its capacity.
 *       An admitted proof of an n the mix lacks, or past its class's capacity, gets BP_VERDICT_UNPLACED: which proofs those are depends
 *       on the input only, so a caller can resubmit exactly them.  Slots a call leaves empty are inert.
 *     - Verdicts: d_verdicts_u32[i] (4-byte aligned) receives, in input order, the code bp_linear_verify_mixed gives proof i with the same
 *       seed, the reject path run on the device (one loop per class); a placed proof with a b entry >= l gets BP_VERDICT_NONCANONICAL_B
 *       and is left out of the combination.  *h_ok_pinned (optional, pinned) receives 1 when the combined check passed, 0 when the reject
 *       path ran.
 *     - Launches per call are constant (the planner kernels, one gather, one graph launch, one verdict kernel), whatever count, fill and
 *       the number of bad proofs.  No allocation, unless count exceeds every earlier call's and the number of slots of the mix: the
 *       planner's scratch then grows, which waits for the work already queued on the context.  The seed (NULL: 32 bytes from the OS) is
 *       staged in one of 8 pinned slots used in turn, as for bp_linear_verify_device; calls queue back to back, each with its own.
 *     BP_ERR_INVALID_ARGUMENT (message in bp_last_error), with nothing queued, when no mix is reserved on the context for this set, for a
 *     NULL argument, count == 0, count >= 2^24, a misaligned d_verdicts_u32, or a pending range-proof verification. */
int bp_linear_verify_mixed_reserve(bp_ctx *ctx, bp_points *set, size_t n_classes, const uint32_t *n, const uint32_t *capacity);
int bp_linear_verify_mixed_device(bp_ctx *ctx, bp_points *set, size_t count, const void *d_transcripts, const void *d_proofs, size_t proof_bytes,
                                  const void *d_proof_offsets, const void *d_C, const void *d_b, size_t n_b, const void *d_b_offsets,
                                  const uint8_t seed[32], void *d_verdicts_u32, uint32_t *h_ok_pinned);

/* D2D copy of the resident table to / from a caller-owned device buffer of bp_gens_device_table() bytes
 * (the Python harness broadcasts a torch tensor with NCCL and imports it on the other ranks); d_dst / d_src may have any alignment. */
int bp_gens_table_export(bp_gens *gens, void *d_dst);
int bp_gens_table_import(bp_gens *gens, const void *d_src);

/* ---- per-kernel timing (CUDA events on the launching stream; used by bench.py's roofline block) ---- */
int bp_prof_enable(bp_ctx *ctx, int on);
int bp_prof_kernel_count(void);
const char *bp_prof_kernel_name(int kernel_id);
int bp_prof_report(bp_ctx *ctx, double *ms, uint64_t *counts);
/* Per-launch records (kernel id, start, end in ms relative to the first record of `ref`, another context of the same device)
 * accumulated since profiling was enabled; does not clear them.  Diagnostic for multi-stream overlap (benchmarks/timeline.py). */
int bp_prof_timeline(bp_ctx *ctx, bp_ctx *ref, int *kernel_ids, double *start_ms, double *end_ms, size_t cap, size_t *n_out);

/* ---- host helpers -------------------------------------------------------------------------- */
/* merlin::Transcript for callers without the Rust crate (same framing as transcript.rs:43-94 expects):
 * Transcript::new(label), append_message, append_u64, challenge_bytes on the 203-byte wire state. */
void bp_transcript_new(const uint8_t *label, size_t len, uint8_t out[BP_TRANSCRIPT_BYTES]);
void bp_transcript_append_message(uint8_t state[BP_TRANSCRIPT_BYTES], const char *label, const uint8_t *msg, size_t len);
void bp_transcript_append_u64(uint8_t state[BP_TRANSCRIPT_BYTES], const char *label, uint64_t x);
void bp_transcript_challenge_bytes(uint8_t state[BP_TRANSCRIPT_BYTES], const char *label, uint8_t *out, size_t len);

/* ---- test hook ----------------------------------------------------------------------------- */
/* element-wise field operation on the device over n pairs of 32-byte little-endian values, loaded without reduction:
 * op 0 add, 1 sub, 2 mul, 3 invert(a), 4 a^((p-5)/8), 5 neg(a), 6 a^2, 7 (a+b)(a-b), 8 2a; canonical bytes out.
 * op 9: the predicates, out[0] = a == 0, out[1] = a is negative (odd canonical value), out[2] = a == b (mod p), other bytes zero.
 * op 10: sqrt_ratio_i(a, b) = the non-negative sqrt(a/b) or sqrt(i*a/b), canonical, with bit 255 set when a/b was square.
 * BP_ERR_INVALID_ARGUMENT for any other op. */
int bp_debug_fe_op(bp_ctx *ctx, int op, const uint8_t *a, const uint8_t *b, size_t n, uint8_t *out);
/* element-wise scalar operation (mod l) on the device over n pairs of 32-byte little-endian values, raw limbs in and out
 * (R = 2^256; Montgomery-form results are returned as they are, x*R mod l):
 *   op 0 sc_mont_mul(a, b) = a*b/R mod l (a any 256-bit value, b < l), 1 from_mont(to_mont(a) * to_mont(b)) = a*b mod l,
 *   2 a+b, 3 a-b, 4 -a (inputs < l), 5 sc_mont_from_wide(a || b) and 6 rp_wide(a || b) = (a + 2^256 b)*R mod l,
 *   7 sc_mont_invert(a) = a^(l-2) in Montgomery form, 8 sum32: out[i] = (sum_{j<32} a[32i+j]*b[32i+j])/R mod l through one
 *   lazy-reduction accumulator (inputs < l; n a multiple of 32, n/32 results) */
int bp_debug_sc_op(bp_ctx *ctx, int op, const uint8_t *a, const uint8_t *b, size_t n, uint8_t *out);
/* element-wise point operation on the device over n pairs of 128-byte points: raw X|Y|Z|T limbs (4 x 32 little-endian bytes, any
 * representative below 2^256, not reduced on load), canonical X|Y|Z|T out.  op 0 ge_add(a, b), 1 ge_madd(a, b) and 2 ge_msub(a, b)
 * with b's first 64 bytes taken as an affine (x, y) and turned into Niels form on the device, 3 ge_dbl(a) */
int bp_debug_ge_op(bp_ctx *ctx, int op, const uint8_t *a, const uint8_t *b, size_t n, uint8_t *out);
/* the fused single-proof path of bp_rangeproof_verify_batch (one thread-block cluster per proof, one launch) whatever the routing rule
 * says, so that a benchmark can time it where the rule sends calls to the pipeline: count <= 64 proofs with lg(n m) <= 10.  Same
 * arguments and verdicts as bp_rangeproof_verify_batch; BP_ERR_INVALID_ARGUMENT for anything outside those limits, a NULL argument,
 * parameters bp_rangeproof_verify_batch would give a verdict for, or a pending begin call. */
int bp_debug_rp_single_verify(bp_ctx *ctx, bp_gens *gens, const uint8_t transcript[BP_TRANSCRIPT_BYTES], const uint8_t *proofs, size_t proof_len,
                              const uint8_t *commitments, size_t n, size_t m, size_t count, const uint8_t seed[32], uint8_t *verdicts);
/* bp_linear_verify_batch down one path whatever its routing rule says, so that tests and benchmarks can compare the two on the same
 * inputs: path 1 the fused launch (count <= 64 proofs of lg n <= 12), path 2 the pipeline.  Same arguments, returns and verdicts as
 * bp_linear_verify_batch; BP_ERR_INVALID_ARGUMENT for any other path, or path 1 outside its limits once the parameters passed. */
int bp_debug_linear_verify_path(bp_ctx *ctx, bp_points *set, size_t n, size_t count, const uint8_t *transcripts, const uint8_t *proofs,
                                size_t proof_len, const uint8_t *C, const uint8_t *b, const uint8_t seed[32], uint8_t *verdicts, int path);

#ifdef __cplusplus
}
#endif
#endif
