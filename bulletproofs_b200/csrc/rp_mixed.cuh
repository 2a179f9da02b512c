// Host planning of range-proof verification: the parameter checks of one proof, and the layout of a call whose proofs have mixed
// geometries (bp_rangeproof_verify_mixed).  Host code apart from the two per-proof checks, which the device planner of
// rp_mixed_device.cuh calls as well; shared with the host-emulation tests.
#pragma once
#include <cstdint>
#include <map>
#include <utility>
#include <vector>
#include "../../include/bpmsm.h"
#include "rp.cuh"

// Parameter checks of verify_multiple_with_rng (mod.rs:358-366) and of from_bytes / verification_scalars that depend only on
// (proof_len, n, m) and the generator table's capacity: the verdict of every proof with these parameters, or BP_PROOF_OK to go on
// (and then *g describes the geometry; count, nbatch and T are left to the caller).
BP_HD uint8_t rp_param_verdict(size_t gens_cap, size_t gens_parties, size_t proof_len, size_t n, size_t m, rp_geom *g) {
    if (proof_len % 32 != 0 || proof_len < 7 * 32) return BP_PROOF_FORMAT_ERROR;                 // mod.rs:498-503
    size_t ne = (proof_len - 7 * 32) / 32;
    if (ne < 2 || (ne - 2) % 2 != 0 || (ne - 2) / 2 >= 32) return BP_PROOF_FORMAT_ERROR;         // inner_product_proof.rs:375-388
    size_t k = (ne - 2) / 2;
    if (!(n == 8 || n == 16 || n == 32 || n == 64)) return BP_PROOF_INVALID_BITSIZE;
    if (gens_cap < n || gens_parties < m) return BP_PROOF_INVALID_GENERATORS_LENGTH;
    if (m == 0 || n * m != ((size_t)1 << k) || k > BP_MAX_LG_N) return BP_PROOF_VERIFICATION_ERROR;   // inner_product_proof.rs:204-211
    g->n = (uint32_t)n; g->m = (uint32_t)m; g->k = (uint32_t)k; g->N = (uint32_t)(n * m);
    g->D = (uint32_t)(4 + 2 * k + m); g->S = 2 + 2 * g->N; g->proof_len = (uint32_t)proof_len;
    return BP_PROOF_OK;
}
// Verdict of one proof whose parameters rp_param_verdict rejected with `pv`.  The reference parses the proof
// (RangeProof::from_bytes, mod.rs:506-524) before it checks the parameters (mod.rs:359-365), so a proof with a non-canonical
// t_x, t_x_blinding, e_blinding, a or b gets FormatError whatever the parameters; a length-level FormatError covers every proof.
// The length passed rp_param_verdict's first checks whenever pv is not FormatError, so the offsets below lie inside the proof.
BP_HD uint8_t rp_rejected_proof_verdict(uint8_t pv, const uint8_t *proof, size_t proof_len) {
    if (pv == BP_PROOF_FORMAT_ERROR) return pv;
    const size_t k = (proof_len / 32 - 9) / 2, ab = 224 + 64 * k;
    const size_t offs[5] = {128, 160, 192, ab, ab + 32};
    for (size_t off : offs)
        if (sc_geq_l(sc_load(proof + off))) return BP_PROOF_FORMAT_ERROR;
    return pv;
}

// ---------------------------------------------------------------------------------------------- mixed geometries
// A call of proofs with any (n, m) verifies every admitted proof in ONE combined MSM.  The admitted proofs are grouped in classes of
// one (n, m) each, classes in the order of their first proof, proofs in input order within a class.  Class c is a batch of count_c
// proofs of geometry g (nbatch = 1), and owns one segment of the mixed scalar array, [S_c static | count_c * D_c dynamic], segments
// class after class.  Every per-proof array (status, head, verdict) is in class order; the decompressed per-proof points of all classes
// are one array, so the dynamic point index of a term is global: class c's points start at dyn.  The other fields are the class's
// offsets into the mixed arenas of the inputs, transcript rows, head tables, chunk partial sums and transcript step programs.
struct rp_mixed_class {
    rp_geom g;
    uint32_t first;                 // first proof of the class in class order
    uint64_t seg, dyn;              // first term of its segment; first dynamic point
    uint64_t proof_off, commit_off; // bytes into the gathered proofs / commitments
    uint64_t raw_off, tab_off, part_off, prog_off;      // bytes of challenge rows; scalars of head tables (whole chunks:
                                                        // rp_tab_slice); scalars of partial sums; steps
    uint32_t prog_steps;
};
struct rp_mixed_plan {
    std::vector<uint8_t> codes;     // per input proof: the parameter verdict (BP_PROOF_OK: admitted, the device decides)
    std::vector<uint32_t> order;    // input index of every admitted proof, in class order
    std::vector<rp_mixed_class> cls;
    uint64_t terms = 0, dyn_points = 0, proof_bytes = 0, commit_bytes = 0, raw_bytes = 0, tab_scalars = 0, part_scalars = 0, prog_steps = 0;
};
#define RP_MIXED_MAX_PROOFS (1u << 24)
#define RP_MIXED_MAX_TERMS (1u << 31)

// Offsets of every class of P (whose g.count is set) into the mixed arenas, class after class, and the totals.  Returns nullptr, or the
// reason the layout is refused (too many MSM terms).
inline const char *rp_mixed_layout(rp_mixed_plan &P) {
    uint32_t first = 0;
    for (rp_mixed_class &C : P.cls) {
        rp_geom &g = C.g;
        g.nbatch = 1;
        const uint64_t T = g.S + (uint64_t)g.count * g.D;
        if (P.terms + T >= RP_MIXED_MAX_TERMS) { P.cls.clear(); P.order.clear(); return "more than 2^31 MSM terms"; }
        g.T = (uint32_t)T;
        C.first = first;
        C.seg = P.terms; C.dyn = P.dyn_points; C.proof_off = P.proof_bytes; C.commit_off = P.commit_bytes;
        C.raw_off = P.raw_bytes; C.tab_off = P.tab_scalars; C.part_off = P.part_scalars; C.prog_off = P.prog_steps;
        C.prog_steps = (uint32_t)rp_tr_program(g.n, g.m, g.k).size();
        P.terms += T;
        P.dyn_points += (uint64_t)g.count * g.D;
        P.proof_bytes += (uint64_t)g.count * g.proof_len; P.commit_bytes += (uint64_t)g.count * g.m * 32;
        P.raw_bytes += (uint64_t)g.count * (RP_RAW_U + g.k) * 64; P.tab_scalars += rp_tab_slice(g.count, g.k, g.m);
        P.part_scalars += (uint64_t)((g.count + RP_CHUNK - 1) / RP_CHUNK) * g.S; P.prog_steps += C.prog_steps;
        first += g.count;
    }
    return nullptr;
}

// The plan of a mixed call.  Proof i is proofs[proof_offsets[i] .. proof_offsets[i+1]) with the commitment_offsets[i+1] -
// commitment_offsets[i] commitments from 32*commitment_offsets[i] on, verified with bit size n[i].  Returns nullptr, or the reason the
// call is refused (too many proofs, offsets that do not start at 0 or that decrease, too many MSM terms).
inline const char *rp_mixed_make_plan(size_t count, const uint8_t *proofs, const uint64_t *proof_offsets, const uint32_t *n,
                                      const uint64_t *commit_offsets, size_t gens_cap, size_t gens_parties, rp_mixed_plan &P) {
    P = rp_mixed_plan{};
    if (count == 0) return "no proofs";
    if (count >= RP_MIXED_MAX_PROOFS) return "more than 2^24 proofs";
    if (proof_offsets[0] != 0 || commit_offsets[0] != 0) return "proof and commitment offsets must start at 0";
    for (size_t i = 0; i < count; i++)
        if (proof_offsets[i + 1] < proof_offsets[i] || commit_offsets[i + 1] < commit_offsets[i]) return "proof and commitment offsets must not decrease";
    P.codes.resize(count);
    std::map<std::pair<uint32_t, uint32_t>, uint32_t> index;        // (n, m) -> class
    std::vector<std::vector<uint32_t>> members;
    for (size_t i = 0; i < count; i++) {
        const size_t len = proof_offsets[i + 1] - proof_offsets[i], m = commit_offsets[i + 1] - commit_offsets[i];
        rp_geom g{};
        uint8_t pv = rp_param_verdict(gens_cap, gens_parties, len, n[i], m, &g);
        P.codes[i] = pv == BP_PROOF_OK ? pv : rp_rejected_proof_verdict(pv, proofs + proof_offsets[i], len);
        if (pv != BP_PROOF_OK) continue;
        auto it = index.emplace(std::make_pair(g.n, g.m), (uint32_t)P.cls.size());
        if (it.second) { rp_mixed_class c{}; c.g = g; P.cls.push_back(c); members.emplace_back(); }
        members[it.first->second].push_back((uint32_t)i);
    }
    for (size_t c = 0; c < P.cls.size(); c++) P.cls[c].g.count = (uint32_t)members[c].size();
    if (const char *why = rp_mixed_layout(P)) return why;
    for (size_t c = 0; c < P.cls.size(); c++) P.order.insert(P.order.end(), members[c].begin(), members[c].end());
    return nullptr;
}

// ---------------------------------------------------------------------------------------------- reserved mixes
// A reserved mix (bp_rangeproof_verify_mixed_reserve) is the layout of a call with capacity_c proofs in each class c, classes in the
// order given: class c owns the proof slots [first_c, first_c + capacity_c) and every arena slice of that many proofs.  A later call
// fills a prefix of each class's slots (its live count); the rest are inert.
#define RP_MIXED_MAX_CLASSES 24
// The mix of n_classes classes (n[c], m[c], capacity[c]) as a layout (P.order and P.codes stay empty), or the reason it is refused.
inline const char *rp_mixed_mix(size_t n_classes, const uint32_t *n, const uint32_t *m, const uint32_t *capacity, size_t gens_cap, size_t gens_parties,
                                rp_mixed_plan &P) {
    P = rp_mixed_plan{};
    if (n_classes == 0 || n_classes > RP_MIXED_MAX_CLASSES) return "a mix holds 1 to 24 classes";
    uint64_t slots = 0;
    for (size_t c = 0; c < n_classes; c++) {
        for (size_t d = 0; d < c; d++)
            if (n[d] == n[c] && m[d] == m[c]) return "duplicate (n, m) class";
        if (capacity[c] == 0) return "zero capacity";
        size_t k = 0; while (((size_t)1 << k) < (size_t)n[c] * m[c]) k++;
        rp_mixed_class K{};
        if (rp_param_verdict(gens_cap, gens_parties, 32 * (9 + 2 * k), n[c], m[c], &K.g) != BP_PROOF_OK) return "a class's (n, m) is not admitted by the generators";
        K.g.count = capacity[c];
        slots += capacity[c];
        P.cls.push_back(K);
    }
    if (slots >= RP_MIXED_MAX_PROOFS) return "more than 2^24 proofs";
    return rp_mixed_layout(P);
}
// Where the admitted proofs of plan P go in the reserved mix X: live[c] = P's proofs of class c of X (0 for a class P lacks), or false
// when P does not fit (a class of P that X lacks, or more proofs than its capacity).
inline bool rp_mixed_fit(const rp_mixed_plan &P, const rp_mixed_plan &X, std::vector<uint32_t> &live) {
    live.assign(X.cls.size(), 0);
    for (const rp_mixed_class &K : P.cls) {
        size_t c = 0;
        while (c < X.cls.size() && (X.cls[c].g.n != K.g.n || X.cls[c].g.m != K.g.m)) c++;
        if (c == X.cls.size() || K.g.count > X.cls[c].g.count) return false;
        live[c] = K.g.count;
    }
    return true;
}
// The gather table of a fitting call in slot order: (input index, slot) of every admitted proof, class c's proofs in input order at
// slots first_c, first_c + 1, ...
inline std::vector<std::pair<uint32_t, uint32_t>> rp_mixed_slots(const rp_mixed_plan &P, const rp_mixed_plan &X) {
    std::vector<std::pair<uint32_t, uint32_t>> out;
    out.reserve(P.order.size());
    for (const rp_mixed_class &M : X.cls)
        for (const rp_mixed_class &K : P.cls)
            if (K.g.n == M.g.n && K.g.m == M.g.m)
                for (uint32_t q = 0; q < K.g.count; q++) out.emplace_back(P.order[K.first + q], M.first + q);
    return out;
}
