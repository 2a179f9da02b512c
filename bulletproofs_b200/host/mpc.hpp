// Host mirror of the aggregated range-proof MPC API of the reference (src/range_proof/{party,dealer,messages}.rs): the
// typestate structs keep the reference's names and transitions; every point operation is a call into libbpmsm.so.
//   Party::new -> PartyAwaitingPosition --assign_position_with_rng--> (PartyAwaitingBitChallenge, BitCommitment)
//     --apply_challenge_with_rng(BitChallenge)--> (PartyAwaitingPolyChallenge, PolyCommitment) --apply_challenge(PolyChallenge)--> ProofShare
//   Dealer::new -> DealerAwaitingBitCommitments --receive_bit_commitments--> (DealerAwaitingPolyCommitments, BitChallenge)
//     --receive_poly_commitments--> (DealerAwaitingProofShares, PolyChallenge) --receive_shares / receive_trusted_shares--> RangeProof
// Rust moves (`self`) become plain structs passed by reference; Result<_, MPCError> becomes an MPCError return + out parameters.
#pragma once
#include "bulletproofs.hpp"

namespace bulletproofs {
namespace mpc {

// src/errors.rs:61-100.  Values shared with the oracle's ORC_* codes so the parity tests compare integers.
enum class MPCError { Ok = 0, InvalidBitsize = 3, InvalidGeneratorsLength = 4, InvalidAggregation = 5, MaliciousDealer = 8,
                      WrongNumBitCommitments = 9, MalformedProofShares = 10, WrongNumPolyCommitments = 11, WrongNumProofShares = 12 };

struct BitCommitment { CompressedRistretto V_j, A_j, S_j; };        // messages.rs:17-22 (A_j, S_j travel compressed here)
struct BitChallenge { Scalar y, z; };                                 // messages.rs:25-29
struct PolyCommitment { CompressedRistretto T_1_j, T_2_j; };         // messages.rs:32-36
struct PolyChallenge { Scalar x; };                                   // messages.rs:39-42

struct ProofShare {                                                   // messages.rs:45-53
    Scalar t_x, t_x_blinding, e_blinding; std::vector<Scalar> l_vec, r_vec;
    bool check_size(size_t expected_n, const BulletproofGens &gens, size_t j) const;                       // :56-81, true = Ok
    // :84-167: t_x == <l, r>, then two MSMs in one device call; true = Ok
    bool audit_share(Device &dev, const BulletproofGens &gens, size_t j, const BitCommitment &bit_commitment, const BitChallenge &bit_challenge,
                     const PolyCommitment &poly_commitment, const PolyChallenge &poly_challenge) const;
    std::vector<uint8_t> to_bytes() const;                            // t_x | t_x_blinding | e_blinding | l_vec | r_vec
    static bool from_bytes(const uint8_t *s, size_t n, ProofShare &out);
};

// Each party step is split in two: next_state does the RNG draws and the scalar algebra without a device call, and the *_terms
// functions append the party's terms of the message's points to an MSM request.  The *_with_rng / new_ steps run both, with one
// device call for their points; RangeProof::prove_many merges the terms of all parties and proofs into one call per step.
struct PartyAwaitingPolyChallenge {                                   // party.rs:240-250
    Scalar offset_zz; std::vector<Scalar> l0, l1, r0, r1; Scalar t0, t1, t2;
    Scalar v_blinding, a_blinding, s_blinding, t_1_blinding, t_2_blinding;
    void T_1_terms(MsmRequest &r) const { r.pedersen(t1, t_1_blinding); }                                  // :216
    void T_2_terms(MsmRequest &r) const { r.pedersen(t2, t_2_blinding); }                                  // :217
    MPCError apply_challenge(const PolyChallenge &pc, ProofShare &out) const;                              // :279-305
};
struct PartyAwaitingBitChallenge {                                    // party.rs:147-157
    Device *dev; const BulletproofGens *gens; size_t n; uint64_t v; Scalar v_blinding; size_t j;
    Scalar a_blinding, s_blinding; std::vector<Scalar> s_L, s_R;
    void A_terms(MsmRequest &r) const;                                                                     // :100-112
    void S_terms(MsmRequest &r) const;                                                                     // :119-124
    void next_state(const BitChallenge &vc, Rng &rng, PartyAwaitingPolyChallenge &next) const;            // :182-215
    void apply_challenge_with_rng(const BitChallenge &vc, Rng &rng, PartyAwaitingPolyChallenge &next, PolyCommitment &out) const;   // :182-237
};
struct PartyAwaitingPosition {                                        // party.rs:63-70
    Device *dev; const BulletproofGens *gens; size_t n; uint64_t v; Scalar v_blinding; CompressedRistretto V;
    void V_terms(MsmRequest &r) const { r.pedersen(Scalar::from_u64(v), v_blinding); }                   // :50
    MPCError next_state(size_t j, Rng &rng, PartyAwaitingBitChallenge &next) const;                        // :87-116
    MPCError assign_position_with_rng(size_t j, Rng &rng, PartyAwaitingBitChallenge &next, BitCommitment &out) const;               // :87-144
};
struct Party {
    static MPCError new_state(Device &dev, const BulletproofGens &gens, uint64_t v, const Scalar &v_blinding, size_t n, PartyAwaitingPosition &out);   // V not set
    static MPCError new_(Device &dev, const BulletproofGens &gens, uint64_t v, const Scalar &v_blinding, size_t n, PartyAwaitingPosition &out);   // party.rs:35-60
};

// The dealer steps likewise: next_state / share_sums / ipp_inputs are the transcript and scalar work, given the points the parties'
// messages sum to; the receive_* steps compute those sums (and Q = w B) on the device.
struct DealerAwaitingProofShares {                                    // dealer.rs:200-215
    Device *dev; const BulletproofGens *gens; size_t n, m; Transcript *transcript; Transcript initial_transcript;
    BitChallenge bit_challenge; std::vector<BitCommitment> bit_commitments; PolyChallenge poly_challenge; std::vector<PolyCommitment> poly_commitments;
    CompressedRistretto A, S, T_1, T_2;
    Scalar share_sums(const std::vector<ProofShare> &shares, RangeProof &proof) const;                                           // :245-256, returns w
    void ipp_inputs(const std::vector<ProofShare> &shares, std::vector<Scalar> &Gf, std::vector<Scalar> &Hf, std::vector<Scalar> &l, std::vector<Scalar> &r) const;   // :258-270
    MPCError assemble_shares(const std::vector<ProofShare> &shares, RangeProof &proof, std::vector<size_t> &bad_shares);           // :226-293
    MPCError receive_shares(const std::vector<ProofShare> &shares, RangeProof &proof, std::vector<size_t> &bad_shares);            // :319-355
    MPCError receive_trusted_shares(const std::vector<ProofShare> &shares, RangeProof &proof);                                     // :370-375
};
struct DealerAwaitingPolyCommitments {                                // dealer.rs:140-151
    Device *dev; const BulletproofGens *gens; size_t n, m; Transcript *transcript; Transcript initial_transcript;
    BitChallenge bit_challenge; std::vector<BitCommitment> bit_commitments; CompressedRistretto A, S;
    void next_state(const CompressedRistretto &T_1, const CompressedRistretto &T_2, DealerAwaitingProofShares &next, PolyChallenge &out) const;   // :172-196
    MPCError receive_poly_commitments(const std::vector<PolyCommitment> &pcs, DealerAwaitingProofShares &next, PolyChallenge &out) const;   // :160-197
};
struct DealerAwaitingBitCommitments {                                 // dealer.rs:84-94
    Device *dev; const BulletproofGens *gens; size_t n, m; Transcript *transcript; Transcript initial_transcript;
    void next_state(const std::vector<CompressedRistretto> &V, const CompressedRistretto &A, const CompressedRistretto &S, DealerAwaitingPolyCommitments &next,
                    BitChallenge &out) const;                                                                                        // :107-136
    MPCError receive_bit_commitments(const std::vector<BitCommitment> &bcs, DealerAwaitingPolyCommitments &next, BitChallenge &out) const;  // :98-137
};
struct Dealer {
    static MPCError new_(Device &dev, const BulletproofGens &gens, Transcript &transcript, size_t n, size_t m, DealerAwaitingBitCommitments &out);   // dealer.rs:37-81
};

}  // namespace mpc
}  // namespace bulletproofs
