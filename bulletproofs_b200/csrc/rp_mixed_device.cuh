// Device planning of a mixed-geometry call whose inputs are device pointers (bp_rangeproof_verify_mixed_device): the per-proof and
// per-block steps that place each proof in a reserved mix without a host round trip.  The kernels of bpmsm.cu (k_mix_admit,
// k_mix_scan, k_mix_place, k_mix_verdicts) call these functions; the host-emulation tests run them block by block against the host
// planner (rp_mixed_make_plan, rp_mixed_fit, rp_mixed_slots).
//
// Placement: proof i is admitted when its offsets are in bounds and rp_param_verdict passes it; it then belongs to the mix class of its
// (n, m), if the mix has one.  Within a class, proofs take the class's slots in input order up to its capacity: proof i's rank is the
// number of admitted proofs of its class before it, the sum of (a) those in earlier blocks of RP_MIX_BLOCK proofs (an exclusive scan of
// the per-block class histograms) and (b) those earlier in its own block: its rank among the same-class lanes of its warp (one
// __match_any_sync on the device) plus the same-class lanes of the block's earlier warps (per-warp class counts).  A proof of no class,
// or ranked at or past the capacity, is unplaced.
#pragma once
#include "rp_mixed.cuh"

#define RP_MIX_BLOCK 256               // proofs per block of the planner kernels
#define RP_MIX_WARPS (RP_MIX_BLOCK / 32)
#define RP_MIX_NO_CLASS 0xFFu          // per-proof class byte: rejected, or admitted with an (n, m) the mix lacks
#define RP_MIX_NO_SLOT 0xFFFFFFFFu     // per-proof slot: unplaced (or rejected)

// bytes of one admitted proof of a mixed call: where its proof and commitments lie in the caller's buffers and in the class-ordered arenas
struct rp_gather { uint64_t src_p, src_c, dst_p, dst_c; uint32_t len_p, len_c; };

// The reserved mix as the planner kernels see it (a kernel parameter, under 1 KB): per class its (n, m), capacity, first slot, proof
// length and arena offsets, and the generator table's capacity for rp_param_verdict.
struct rp_mix_classes {
    uint32_t C, gens_cap, gens_parties;
    uint32_t n[RP_MIXED_MAX_CLASSES], m[RP_MIXED_MAX_CLASSES], cap[RP_MIXED_MAX_CLASSES], first[RP_MIXED_MAX_CLASSES], proof_len[RP_MIXED_MAX_CLASSES];
    uint64_t proof_off[RP_MIXED_MAX_CLASSES], commit_off[RP_MIXED_MAX_CLASSES];
};
inline rp_mix_classes rp_mix_classes_of(const rp_mixed_plan &X, size_t gens_cap, size_t gens_parties) {
    rp_mix_classes M{};
    M.C = (uint32_t)X.cls.size(); M.gens_cap = (uint32_t)gens_cap; M.gens_parties = (uint32_t)gens_parties;
    for (uint32_t c = 0; c < M.C; c++) {
        const rp_mixed_class &K = X.cls[c];
        M.n[c] = K.g.n; M.m[c] = K.g.m; M.cap[c] = K.g.count; M.first[c] = K.first; M.proof_len[c] = K.g.proof_len;
        M.proof_off[c] = K.proof_off; M.commit_off[c] = K.commit_off;
    }
    return M;
}

// little-endian words at any alignment (the caller's offset and n arrays)
BP_HD uint64_t rp_ld_u64(const uint8_t *p) { uint64_t v = 0; for (int b = 7; b >= 0; b--) v = (v << 8) | p[b]; return v; }
BP_HD uint32_t rp_ld_u32(const uint8_t *p) { return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24); }

// Proof i's bytes [*po, *po + len) and commitments [*co, *co + m), or false when its offsets decrease or reach past proof_bytes /
// n_commit (then none of its bytes may be read).
BP_HD bool rp_mix_bounds(const uint8_t *poff, const uint8_t *coff, uint64_t proof_bytes, uint64_t n_commit, size_t i, uint64_t *po, uint64_t *len,
                         uint64_t *co, uint64_t *m) {
    const uint64_t p0 = rp_ld_u64(poff + 8 * i), p1 = rp_ld_u64(poff + 8 * i + 8), c0 = rp_ld_u64(coff + 8 * i), c1 = rp_ld_u64(coff + 8 * i + 8);
    if (p1 < p0 || c1 < c0 || p1 > proof_bytes || c1 > n_commit) return false;
    *po = p0; *len = p1 - p0; *co = c0; *m = c1 - c0;
    return true;
}
// Admission of proof i as one word, code | class << 8: its parameter code, exactly bp_rangeproof_verify_mixed's (rp_param_verdict, then
// rp_rejected_proof_verdict), with FormatError for offsets rp_mix_bounds refuses; its class of M, or RP_MIX_NO_CLASS when it is rejected
// or M lacks its (n, m).
BP_HD uint32_t rp_mix_admit(const rp_mix_classes &M, const uint8_t *proofs, uint64_t proof_bytes, const uint8_t *poff, const uint8_t *n_arr, uint64_t n_commit,
                            const uint8_t *coff, size_t i) {
    uint64_t po, len, co, m;
    if (!rp_mix_bounds(poff, coff, proof_bytes, n_commit, i, &po, &len, &co, &m)) return BP_PROOF_FORMAT_ERROR | RP_MIX_NO_CLASS << 8;
    rp_geom g{};
    const uint8_t pv = rp_param_verdict(M.gens_cap, M.gens_parties, (size_t)len, rp_ld_u32(n_arr + 4 * i), (size_t)m, &g);
    if (pv != BP_PROOF_OK) return rp_rejected_proof_verdict(pv, proofs + po, (size_t)len) | RP_MIX_NO_CLASS << 8;
    uint32_t cls = RP_MIX_NO_CLASS;
    for (uint32_t c = 0; c < M.C; c++)
        if (M.n[c] == g.n && M.m[c] == g.m) { cls = c; break; }
    return BP_PROOF_OK | cls << 8;
}
BP_HD uint32_t rp_mix_code(uint32_t word) { return word & 0xFFu; }
BP_HD uint32_t rp_mix_class(uint32_t word) { return word >> 8; }
// The block's per-warp class counts: wcnt[w][c] = the class-c lanes of warp w.  Rank in the block of a class-c lane of warp `warp` whose
// rank among the class-c lanes of its own warp is wrank: wrank plus the class-c lanes of the earlier warps.
BP_HD uint32_t rp_mix_rank_in_block(const uint32_t (*wcnt)[RP_MIXED_MAX_CLASSES], uint32_t warp, uint32_t c, uint32_t wrank) {
    for (uint32_t w = 0; w < warp; w++) wrank += wcnt[w][c];
    return wrank;
}
// the block's class-c lanes
BP_HD uint32_t rp_mix_block_count(const uint32_t (*wcnt)[RP_MIXED_MAX_CLASSES], uint32_t c) { return rp_mix_rank_in_block(wcnt, RP_MIX_WARPS, c, 0); }
// The slot of rank `rank` in class c, or RP_MIX_NO_SLOT past its capacity
BP_HD uint32_t rp_mix_slot(const rp_mix_classes &M, uint32_t c, uint32_t rank) { return rank < M.cap[c] ? M.first[c] + rank : RP_MIX_NO_SLOT; }
// The gather entry of a proof placed at rank q of class c, from its bytes at po and commitments from commitment co on
BP_HD rp_gather rp_mix_gather_entry(const rp_mix_classes &M, uint32_t c, uint32_t q, uint64_t po, uint64_t co) {
    return rp_gather{po, 32 * co, M.proof_off[c] + (uint64_t)q * M.proof_len[c], M.commit_off[c] + (uint64_t)q * M.m[c] * 32, M.proof_len[c], M.m[c] * 32};
}
// Class of slot s (s below the slot total)
BP_HD uint32_t rp_mix_class_of_slot(const rp_mix_classes &M, uint32_t s) {
    uint32_t c = 0;
    while (c + 1 < M.C && s >= M.first[c + 1]) c++;
    return c;
}
