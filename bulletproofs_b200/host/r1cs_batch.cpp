// r1cs::verify_batch (see r1cs.hpp) and its C shim: the host phase of many proofs, then one bp_r1cs_verify_batch call.
#include "r1cs.hpp"
#include <chrono>
#include <deque>

namespace bulletproofs {
namespace r1cs {

// the 32 bytes of the external RNG a proof of a batch finalises its TranscriptRng with
namespace {
class SlotRng : public Rng {
    const uint8_t *b_; size_t left_ = 32;
public:
    explicit SlotRng(const uint8_t *b) : b_(b) {}
    void fill_bytes(uint8_t *out, size_t n) override {
        if (n > left_) throw std::logic_error("r1cs::verify_batch: a proof drew more than its 32 external bytes");
        memcpy(out, b_, n); b_ += n; left_ -= n;
    }
};
double seconds_now() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); }
}  // namespace

std::vector<R1CSError> verify_batch(Device &dev, const BulletproofGens &gens, std::vector<Verifier *> &verifiers, const std::vector<const R1CSProof *> &proofs,
                                    Rng &external, R1CSBatchTiming *timing) {
    const size_t B = verifiers.size();
    if (proofs.size() != B) throw std::invalid_argument("r1cs::verify_batch: one proof per verifier");
    const double t0 = seconds_now();
    std::vector<uint8_t> ext(32 * B);
    for (size_t j = 0; j < B; j++) external.fill_bytes(ext.data() + 32 * j, 32);       // serially, in batch order
    std::vector<R1CSPrepared> P(B); std::vector<R1CSError> codes(B);
    parallel_for(B, [&](size_t j) { SlotRng r(ext.data() + 32 * j); codes[j] = verifiers[j]->prepare(*proofs[j], r, P[j], true); });
    // flat inputs of bp_r1cs_verify_batch for the proofs the host phase passed
    std::vector<size_t> sent;
    for (size_t j = 0; j < B; j++) if (codes[j] == R1CSError::Ok) sent.push_back(j);
    std::vector<uint32_t> dims, idx; std::vector<Scalar> chal, wL, wR, wO, sc; std::vector<uint8_t> dyn;
    for (size_t j : sent) {
        const R1CSPrepared &p = P[j];
        dims.insert(dims.end(), {(uint32_t)p.padded_n, (uint32_t)p.n1, (uint32_t)p.n, (uint32_t)p.terms.sc.size()});
        chal.insert(chal.end(), {p.x, p.y_inv, p.u, p.a, p.b, p.rho, p.s[0]});
        chal.insert(chal.end(), p.u_sq.begin(), p.u_sq.end());
        wL.insert(wL.end(), p.wL.begin(), p.wL.end()); wR.insert(wR.end(), p.wR.begin(), p.wR.end()); wO.insert(wO.end(), p.wO.begin(), p.wO.end());
        sc.insert(sc.end(), p.terms.sc.begin(), p.terms.sc.end());
        const uint32_t base = (uint32_t)(dyn.size() / 32);
        for (uint32_t v : p.terms.idx) idx.push_back(v & MsmRequest::DYNAMIC ? v + base : v);
        dyn.insert(dyn.end(), p.terms.dyn.begin(), p.terms.dyn.end());
    }
    std::vector<uint8_t> bchal = pack(chal), bwL = pack(wL), bwR = pack(wR), bwO = pack(wO), bsc = pack(sc);
    const double t1 = seconds_now();
    if (!sent.empty()) {
        std::vector<uint8_t> verdicts(sent.size());
        check(bp_r1cs_verify_batch(dev.ctx, gens.handle, sent.size(), dims.data(), bchal.data(), bwL.data(), bwR.data(), bwO.data(), bsc.data(), idx.data(),
                                   dyn.data(), dyn.size() / 32, verdicts.data()), dev.ctx, "r1cs batch mega-check");
        for (size_t q = 0; q < sent.size(); q++) codes[sent[q]] = verdicts[q] == BP_PROOF_OK ? R1CSError::Ok : R1CSError::VerificationError;
    }
    if (timing) { timing->prepare_s = t1 - t0; timing->engine_s = seconds_now() - t1; }
    return codes;
}

}  // namespace r1cs
}  // namespace bulletproofs

// ================================================================================================ C shim for the Python harness
using namespace bulletproofs;
using namespace bulletproofs::r1cs;
extern "C" {
// n proofs through r1cs::verify_batch: item j = transcript j (203 B), gadget j, param j, commitments [commit_off[j], commit_off[j+1]) (in
// points), proof bytes [proof_off[j], proof_off[j+1]).  codes[j] = what bph_r1cs_verify would return for item j.  timing (optional):
// seconds of the host phase and of the engine call.
int bph_r1cs_verify_batch(bp_ctx *ctx, bp_gens *gens, size_t gens_capacity, size_t party_capacity, size_t n, const uint8_t *transcripts, const int *gadgets,
                          const uint64_t *params, const uint8_t *commitments, const uint64_t *commit_off, const uint8_t *proofs, const uint64_t *proof_off,
                          const uint8_t ext_seed[32], int *codes, double *timing) {
    try {
        Device dev(ctx); BulletproofGens g{gens, gens_capacity, party_capacity}; ChaChaRng ext(ext_seed);
        std::deque<Transcript> ts; std::deque<Verifier> vs; std::deque<R1CSProof> ps;
        std::vector<Verifier *> batch_v; std::vector<const R1CSProof *> batch_p; std::vector<size_t> item;
        for (size_t j = 0; j < n; j++) {
            ps.emplace_back();
            R1CSError e = R1CSProof::from_bytes(proofs + proof_off[j], proof_off[j + 1] - proof_off[j], ps.back());
            if (e != R1CSError::Ok) { codes[j] = (int)e; continue; }
            ts.emplace_back(transcripts + BP_TRANSCRIPT_BYTES * j);
            vs.emplace_back(dev, g, ts.back());
            std::vector<Variable> vars;
            for (uint64_t i = commit_off[j]; i < commit_off[j + 1]; i++) { CompressedRistretto V; memcpy(V.data(), commitments + 32 * i, 32); vars.push_back(vs.back().commit(V)); }
            e = build_gadget(vs.back(), gadgets[j], vars, params[j], nullptr);
            if (e != R1CSError::Ok) { codes[j] = (int)e; continue; }
            batch_v.push_back(&vs.back()); batch_p.push_back(&ps.back()); item.push_back(j);
        }
        R1CSBatchTiming tm;
        std::vector<R1CSError> out = verify_batch(dev, g, batch_v, batch_p, ext, &tm);
        for (size_t q = 0; q < item.size(); q++) codes[item[q]] = (int)out[q];
        if (timing) { timing[0] = tm.prepare_s; timing[1] = tm.engine_s; }
        return 0;
    } catch (const std::exception &) { return -1; }
}
}
