// C++ mirror of the reference's public API for the MSM-bound path, above the C ABI of include/bpmsm.h.
//
// The reference is Rust (no rustc in this image), so the host side is C++ with the same names and
// argument meaning; every point operation goes through libbpmsm.so (sm_90a), the host only does
// transcripts (STROBE/Keccak byte shuffling) and scalar arithmetic mod l.
//   bulletproofs::Scalar            <- curve25519_dalek::scalar::Scalar
//   bulletproofs::Transcript        <- merlin::Transcript + TranscriptProtocol (src/transcript.rs:8-94)
//   bulletproofs::ChaChaRng         <- rand_chacha::ChaChaRng (tests/range_proof.rs:108)
//   bulletproofs::BulletproofGens / PedersenGens  (src/generators.rs:29-204), resident on the device
//   bulletproofs::InnerProductProof::{create, verify, to_bytes, from_bytes}   (src/inner_product_proof.rs:38-407)
//   bulletproofs::RangeProof::{prove_multiple_with_rng, verify_multiple, to_bytes, from_bytes}  (src/range_proof/mod.rs:234-538)
#pragma once
#include <atomic>
#include <exception>
#include <thread>
#include <sched.h>
#include <array>
#include <cstdint>
#include <cstring>
#include <stdexcept>
#include <string>
#include <vector>
#include "../../include/bpmsm.h"
#include "../csrc/merlin.cuh"
#include "../csrc/sc.cuh"

namespace bulletproofs {

enum class ProofError { Ok = 0, VerificationError = 1, FormatError = 2, InvalidBitsize = 3, InvalidGeneratorsLength = 4, InvalidAggregation = 5,
                        WrongNumBlindingFactors = 6, MaliciousDealer = 7, InvalidInputLength = 8 };

using Bytes32 = std::array<uint8_t, 32>;
using CompressedRistretto = Bytes32;

struct Rng { virtual void fill_bytes(uint8_t *out, size_t n) = 0; virtual ~Rng() {} };

// rand_chacha::ChaChaRng::from_seed: ChaCha20 keystream, 64-bit block counter from 0, stream 0
class ChaChaRng : public Rng {
    uint32_t key_[8]; uint64_t counter_ = 0; uint8_t buf_[64]; int used_ = 64;
    void block();
public:
    explicit ChaChaRng(const uint8_t seed[32]) { memcpy(key_, seed, 32); }
    void fill_bytes(uint8_t *out, size_t n) override;
};

// Scalar mod l, kept in Montgomery form (sc.cuh host path); to_bytes() is the canonical 32-byte encoding
class Scalar {
    sc m_;
    explicit Scalar(const sc &mont) : m_(mont) {}
public:
    Scalar() : m_(sc_zero()) {}
    static Scalar zero() { return Scalar(); }
    static Scalar one() { return Scalar(sc_mont_one()); }
    static Scalar from_u64(uint64_t x) { return Scalar(sc_mont_from_u64(x)); }
    static Scalar from_bytes_mod_order_wide(const uint8_t b[64]) { return Scalar(sc_mont_from_wide(b)); }
    static bool from_canonical_bytes(const uint8_t b[32], Scalar &out) { sc v = sc_load(b); if (sc_geq_l(v)) return false; out = Scalar(sc_to_mont(v)); return true; }
    static Scalar random(Rng &rng) { uint8_t b[64]; rng.fill_bytes(b, 64); return from_bytes_mod_order_wide(b); }
    Bytes32 to_bytes() const { Bytes32 o; sc_store(o.data(), sc_from_mont(m_)); return o; }
    void write(uint8_t *out) const { sc_store(out, sc_from_mont(m_)); }
    Scalar operator+(const Scalar &o) const { return Scalar(sc_add(m_, o.m_)); }
    Scalar operator-(const Scalar &o) const { return Scalar(sc_sub(m_, o.m_)); }
    Scalar operator*(const Scalar &o) const { return Scalar(sc_mont_mul(m_, o.m_)); }
    Scalar operator-() const { return Scalar(sc_neg(m_)); }
    Scalar &operator+=(const Scalar &o) { m_ = sc_add(m_, o.m_); return *this; }
    Scalar &operator*=(const Scalar &o) { m_ = sc_mont_mul(m_, o.m_); return *this; }
    bool is_zero() const { return sc_is_zero(m_); }
    Scalar invert() const { return Scalar(sc_mont_invert(m_)); }     // 0 -> 0, like dalek
};
// Host-side work of a batch (transcripts, scalar vectors, RNG draws) is independent per proof: spread it over the cores this process may use.
// Device calls stay on the calling thread.
template <class F> inline void parallel_for(size_t n, F fn) {
    cpu_set_t set; CPU_ZERO(&set);
    size_t cores = n > 1 && sched_getaffinity(0, sizeof set, &set) == 0 ? (size_t)CPU_COUNT(&set) : 1;     // no system call for one item (nested pack)
    size_t nt = std::min<size_t>(std::max<size_t>(cores, 1), n);
    if (nt <= 1) { for (size_t i = 0; i < n; i++) fn(i); return; }
    std::atomic<size_t> next{0}; std::exception_ptr err; std::atomic<bool> failed{false};
    std::vector<std::thread> th;
    for (size_t t = 0; t < nt; t++)
        th.emplace_back([&] {
            try { for (size_t i; (i = next++) < n;) fn(i); }
            catch (...) { if (!failed.exchange(true)) err = std::current_exception(); }
        });
    for (auto &x : th) x.join();
    if (failed) std::rethrow_exception(err);
}

inline void check(int rc, bp_ctx *ctx, const char *what) {
    if (rc != BP_OK) throw std::runtime_error(std::string(what) + " failed with code " + std::to_string(rc) + ": " + bp_last_error(ctx));
}
// canonical 32-byte encodings of v into out, over the host cores for long vectors (R1CS)
inline void pack(const std::vector<Scalar> &v, uint8_t *out) {
    const size_t CH = 8192, nch = (v.size() + CH - 1) / CH;
    parallel_for(nch, [&](size_t c) { for (size_t i = c * CH; i < std::min(v.size(), (c + 1) * CH); i++) v[i].write(out + 32 * i); });
}
inline std::vector<uint8_t> pack(const std::vector<Scalar> &v) { std::vector<uint8_t> o(32 * v.size()); pack(v, o.data()); return o; }
inline bool is_identity(const CompressedRistretto &p) { uint8_t z = 0; for (uint8_t b : p) z |= b; return z == 0; }     // the identity encodes as zeros
inline bool load_scalars(const uint8_t *b, size_t n, std::vector<Scalar> &out) { out.resize(n); for (size_t i = 0; i < n; i++) if (!Scalar::from_canonical_bytes(b + 32 * i, out[i])) return false; return true; }
inline std::vector<CompressedRistretto> load_points(const uint8_t *b, size_t n) { std::vector<CompressedRistretto> v(n); for (size_t i = 0; i < n; i++) memcpy(v[i].data(), b + 32 * i, 32); return v; }

Scalar inner_product(const std::vector<Scalar> &a, const std::vector<Scalar> &b);     // inner_product_proof.rs:418-427
Scalar scalar_exp_vartime(const Scalar &x, uint64_t n);                               // util.rs:222-234

class Transcript {
    alignas(8) uint8_t st_[200]; merlin_t m_;
public:
    Transcript() : st_{}, m_{st_, 0, 0, 0} {}                      // a zero state, for a member that is assigned before use
    explicit Transcript(const std::string &label) { m_.st = st_; merlin_init(m_, (const uint8_t *)label.data(), (uint32_t)label.size()); }
    explicit Transcript(const uint8_t wire[BP_TRANSCRIPT_BYTES]) { m_.st = st_; merlin_load(m_, wire); }
    Transcript(const Transcript &o) { memcpy(st_, o.st_, 200); m_ = o.m_; m_.st = st_; }
    Transcript &operator=(const Transcript &o) { memcpy(st_, o.st_, 200); m_ = o.m_; m_.st = st_; return *this; }
    void to_wire(uint8_t out[BP_TRANSCRIPT_BYTES]) const { merlin_store(out, m_); }
    void append_message(const char *label, const uint8_t *msg, size_t len) { merlin_append(m_, label, msg, (uint32_t)len); }
    void append_u64(const char *label, uint64_t x) { merlin_append_u64(m_, label, x); }
    // TranscriptProtocol (transcript.rs:43-94)
    void rangeproof_domain_sep(uint64_t n, uint64_t m) { append_message("dom-sep", (const uint8_t *)"rangeproof v1", 13); append_u64("n", n); append_u64("m", m); }
    void innerproduct_domain_sep(uint64_t n) { append_message("dom-sep", (const uint8_t *)"ipp v1", 6); append_u64("n", n); }
    void append_scalar(const char *label, const Scalar &s) { Bytes32 b = s.to_bytes(); append_message(label, b.data(), 32); }
    void append_point(const char *label, const CompressedRistretto &p) { append_message(label, p.data(), 32); }
    bool validate_and_append_point(const char *label, const CompressedRistretto &p) {
        if (is_identity(p)) return false;
        append_point(label, p); return true;
    }
    Scalar challenge_scalar(const char *label) { uint8_t buf[64]; merlin_challenge(m_, label, buf, 64); return Scalar::from_bytes_mod_order_wide(buf); }
};

// one device + stream (bp_ctx)
class Device {
public:
    bp_ctx *ctx;
    explicit Device(bp_ctx *borrowed) : ctx(borrowed) {}
};

// BulletproofGens::new + PedersenGens::default on the device (bp_gens); this class only borrows the handle
struct BulletproofGens {
    bp_gens *handle; size_t gens_capacity, party_capacity;
    // generator-table slots (layout of bp_gens_device_table)
    static uint32_t slot_B_blinding() { return 0; }
    static uint32_t slot_B() { return 1; }
    uint32_t slot_G(size_t party, size_t i) const { return (uint32_t)(2 + party * gens_capacity + i); }
    uint32_t slot_H(size_t party, size_t i) const { return (uint32_t)(2 + party_capacity * gens_capacity + party * gens_capacity + i); }
};

// Indexed MSMs for bp_msm_indexed_batch: each term is a scalar and a generator-table slot, or DYNAMIC | k for the k-th point of dyn;
// ends[i] is the end of MSM i in the term list.
struct MsmRequest {
    static constexpr uint32_t DYNAMIC = 0x80000000u;
    std::vector<Scalar> sc; std::vector<uint32_t> idx; std::vector<uint64_t> ends; std::vector<uint8_t> dyn;
    void term(const Scalar &s, uint32_t slot) { sc.push_back(s); idx.push_back(slot); }
    void dyn_term(const Scalar &s, const CompressedRistretto &p) { term(s, DYNAMIC | (uint32_t)(dyn.size() / 32)); dyn.insert(dyn.end(), p.begin(), p.end()); }
    void pedersen(const Scalar &v, const Scalar &v_blinding) { term(v, BulletproofGens::slot_B()); term(v_blinding, BulletproofGens::slot_B_blinding()); }  // generators.rs:39-41
    void end_msm() { ends.push_back(sc.size()); }
};
// The MSMs of reqs[0..count), in order, as one bp_msm_indexed_batch call (none if there are no MSMs): the outputs, and each MSM's
// BP_* status in *status if given.
std::vector<CompressedRistretto> run_msms(Device &dev, const BulletproofGens &gens, const MsmRequest *reqs, size_t count, std::vector<uint8_t> *status = nullptr);

struct InnerProductProof {
    std::vector<CompressedRistretto> L_vec, R_vec; Scalar a, b;
    // create over the generators G = gens.G(n, m), H = gens.H(n, m)  (the range-proof use, dealer.rs:272-281)
    static InnerProductProof create(Device &dev, const BulletproofGens &gens, size_t n, size_t m, Transcript &t, const CompressedRistretto &Q,
                                    const std::vector<Scalar> &G_factors, const std::vector<Scalar> &H_factors, std::vector<Scalar> a, std::vector<Scalar> b);
    // create over arbitrary vectors (inner_product_proof.rs:38-47)
    static InnerProductProof create(Device &dev, Transcript &t, const CompressedRistretto &Q, const std::vector<Scalar> &G_factors, const std::vector<Scalar> &H_factors,
                                    const std::vector<CompressedRistretto> &G, const std::vector<CompressedRistretto> &H, std::vector<Scalar> a, std::vector<Scalar> b);
    // B independent proofs over the same generators, all MSM launch chains shared (batched prover)
    static std::vector<InnerProductProof> create_many(Device &dev, const BulletproofGens &gens, size_t n, size_t m, std::vector<Transcript *> &ts, const std::vector<CompressedRistretto> &Qs,
                                                      const std::vector<std::vector<Scalar>> &G_factors, const std::vector<std::vector<Scalar>> &H_factors,
                                                      const std::vector<std::vector<Scalar>> &as, const std::vector<std::vector<Scalar>> &bs);
    // verification_scalars (inner_product_proof.rs:198-253)
    ProofError verification_scalars(size_t n, Transcript &t, std::vector<Scalar> &u_sq, std::vector<Scalar> &u_inv_sq, std::vector<Scalar> &s) const;
    // verify (inner_product_proof.rs:260-326)
    ProofError verify(Device &dev, size_t n, Transcript &t, const std::vector<Scalar> &G_factors, const std::vector<Scalar> &H_factors, const CompressedRistretto &P,
                      const CompressedRistretto &Q, const std::vector<CompressedRistretto> &G, const std::vector<CompressedRistretto> &H) const;
    std::vector<uint8_t> to_bytes() const;
    static ProofError from_bytes(const uint8_t *s, size_t len, InnerProductProof &out);
};

// src/linear_proof.rs:27-397 (GHL'21 appendix E.3): proves c = <a, b> for public b and committed a
struct LinearProof {
    std::vector<CompressedRistretto> L_vec, R_vec; CompressedRistretto S; Scalar a, r;
    static ProofError create(Device &dev, Transcript &t, Rng &rng, const CompressedRistretto &C, Scalar r, std::vector<Scalar> a_vec, std::vector<Scalar> b_vec,
                             const std::vector<CompressedRistretto> &G_vec, const CompressedRistretto &F, const CompressedRistretto &B, LinearProof &out);      // :40-160
    ProofError verify(Device &dev, Transcript &t, const CompressedRistretto &C, const std::vector<CompressedRistretto> &G, const CompressedRistretto &F,
                      const CompressedRistretto &B, std::vector<Scalar> b_vec) const;                                                                            // :162-224
    std::vector<uint8_t> to_bytes() const;                                            // :291-301
    static ProofError from_bytes(const uint8_t *s, size_t len, LinearProof &out);    // :351-397
};

struct RangeProof {
    CompressedRistretto A, S, T_1, T_2; Scalar t_x, t_x_blinding, e_blinding; InnerProductProof ipp_proof;
    // range_proof/mod.rs:234-288 (the MPC run with itself: party.rs / dealer.rs)
    static ProofError prove_multiple_with_rng(Device &dev, const BulletproofGens &gens, Transcript &t, const std::vector<uint64_t> &values,
                                              const std::vector<Scalar> &blindings, size_t n, Rng &rng, RangeProof &proof, std::vector<CompressedRistretto> &commitments);
    // B independent aggregated proofs (same n, same number of values m each): every proof runs the MPC dealer and party steps of
    // mpc.hpp, with their device calls merged across the proofs: one call for all V/A/S commitments, one for all T_1/T_2, one for all
    // Q, one device session for all inner-product arguments.  Same bytes as B calls of prove_multiple_with_rng with the same
    // transcripts and RNGs.
    static void prove_many(Device &dev, const BulletproofGens &gens, size_t n, std::vector<struct RangeProofJob> &jobs);
    // range_proof/mod.rs:345-452 through the batch verifier with count = 1
    ProofError verify_multiple(Device &dev, const BulletproofGens &gens, const Transcript &t, const std::vector<CompressedRistretto> &commitments, size_t n) const;
    std::vector<uint8_t> to_bytes() const;                                         // mod.rs:487-499
    static ProofError from_bytes(const uint8_t *s, size_t len, RangeProof &out);   // mod.rs:505-538
};

// one proof of a RangeProof::prove_many batch: inputs (transcript, values, blindings, rng) and outputs (proof, commitments, error)
struct RangeProofJob { Transcript *t; std::vector<uint64_t> values; std::vector<Scalar> blindings; Rng *rng; RangeProof proof; std::vector<CompressedRistretto> commitments; ProofError error = ProofError::Ok; };

}  // namespace bulletproofs
