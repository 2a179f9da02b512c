// TEST-ONLY host build of the range-proof table layout (rp.cuh): the head writing one proof of a chunk-major slice, and the slots
// that the head, k_rp_scalars_sum (main and reject path) and the mixed layout give every (proof, entry) of their slices.
#include <utility>
#include <vector>
#include "../../bulletproofs_b200/csrc/rp_mixed.cuh"

typedef uint32_t (*lean_fn)(rp_lean_head &, sc *, uint8_t *, const sc *, const uint8_t *, const uint8_t *, uint32_t, uint32_t);
template <uint32_t K> static uint32_t lean_k(rp_lean_head &h, sc *tab, uint8_t *dyn, const sc *pow2, const uint8_t *raw, const uint8_t *proof, uint32_t n, uint32_t m) {
    return rp_head_lean(h, tab, dyn, pow2, raw, proof, K, n, m, RP_TAB_STRIDE);
}
template <uint32_t... I> static lean_fn lean_pick(uint32_t k, std::integer_sequence<uint32_t, I...>) {
    static const lean_fn fns[] = {&lean_k<3 + I>...};
    return fns[k - 3];
}

extern "C" {

// the head of one proof at slice index p of a slice of count proofs, as k_rp_head_seq runs it; writes [zL | base-point scalar |
// blinding scalar | D dynamic scalars | the nine tables read back through rp_tab_ptrs] as emul_rp_head_ref does.  Returns the status,
// or -2 when the head wrote a slot of the slice outside the proof's own entries.
int emul_rp_head_slice(const uint8_t *raw, const uint8_t *proof, uint32_t k, uint32_t n, uint32_t m, uint32_t count, uint32_t p, uint8_t *out) {
    if (k < 3 || k > BP_MAX_LG_N || p >= count) return -1;
    const uint32_t D = 4 + 2 * k + m, tsz = rp_tab_size(k, m);
    std::vector<sc> slice(rp_tab_slice(count, k, m)), pow2(64);
    const sc mark = sc_l();                                              // never a table value (every entry is < l)
    for (sc &s : slice) s = mark;
    for (int e = 0; e < 64; e++) pow2[e] = sc_mont_from_u64(1ULL << e);
    std::vector<uint64_t> rows((RP_RAW_U + k) * 8);
    memcpy(rows.data(), raw, (RP_RAW_U + k) * 64);
    rp_lean_head h{};
    sc *tab = rp_tab_proof(slice.data(), p, tsz);
    uint32_t st = lean_pick(k, std::make_integer_sequence<uint32_t, BP_MAX_LG_N - 2>())(h, tab, out + 96, pow2.data(), reinterpret_cast<const uint8_t *>(rows.data()),
                                                                                       proof, n, m);
    std::vector<bool> own(slice.size(), false);
    for (uint32_t e = 0; e < tsz; e++) own[rp_tab_index(p, tsz) + (size_t)e * RP_TAB_STRIDE] = true;
    for (size_t i = 0; i < slice.size(); i++)
        if (!own[i] && memcmp(&slice[i], &mark, sizeof mark) != 0) return -2;
    if (st) return (int)st;
    sc_store(out, sc_from_mont(h.zL)); sc_store(out + 32, sc_from_mont(h.basepoint_scalar)); sc_store(out + 64, sc_from_mont(h.blinding_scalar));
    const rp_tabs T = rp_tab_ptrs(tab, k, RP_TAB_STRIDE);
    const uint32_t kl = rp_kl(k), TL = 1u << kl, TH = 1u << (k - kl);
    uint8_t *o = out + 32 * (3 + D);
    for (const rp_tab_col *c : {&T.s_lo, &T.A_hi, &T.P_lo, &T.P_hi, &T.Q_lo, &T.Q_hi, &T.s_hi, &T.y_lo, &T.y_hi}) {
        const uint32_t len = (c == &T.s_lo || c == &T.P_lo || c == &T.Q_lo || c == &T.y_lo) ? TL : TH;
        for (uint32_t v = 0; v < len; v++, o += 32) sc_store(o, sc_from_mont((*c)[v]));
    }
    return 0;
}

uint64_t emul_rp_tab_slice(uint32_t count, uint32_t k, uint32_t m) { return rp_tab_slice(count, k, m); }
// slot of entry e of slice index p
uint64_t emul_rp_tab_slot(uint32_t p, uint32_t e, uint32_t k, uint32_t m) { return rp_tab_index(p, rp_tab_size(k, m)) + (uint64_t)e * RP_TAB_STRIDE; }

// The slice indices k_rp_scalars_sum reads on geometry (count, nbatch) with table index tab_p0 of its first proof: idx[block * RP_CHUNK
// + q] for q < the block's nq (RP_CHUNK * blocks entries; the rest are left alone).  Returns the number of blocks.
uint32_t emul_rp_sum_indices(uint32_t count, uint32_t nbatch, uint32_t tab_p0, uint32_t *idx) {
    rp_geom g{}; g.count = count; g.nbatch = nbatch;
    const uint32_t blocks = nbatch * ((count + RP_CHUNK - 1) / RP_CHUNK);
    for (uint32_t blk = 0; blk < blocks; blk++) {
        const rp_sum_block s = rp_sum_block_of(g, blk);
        for (uint32_t q = 0; q < s.nq; q++) idx[blk * RP_CHUNK + q] = tab_p0 + s.p0 + q;
    }
    return blocks;
}

// the table slices of a reserved mix of n_classes classes: off[c], len[c] (scalars), the proofs of class c and its tsz; returns the
// arena's scalars, or 0 when the mix is refused
uint64_t emul_rp_mix_tab_slices(uint32_t n_classes, const uint32_t *n, const uint32_t *m, const uint32_t *cap, uint64_t *off, uint64_t *len,
                                uint32_t *count, uint32_t *tsz) {
    rp_mixed_plan P;
    if (rp_mixed_mix(n_classes, n, m, cap, 64, 1u << 16, P)) return 0;
    for (uint32_t c = 0; c < n_classes; c++) {
        const rp_geom &g = P.cls[c].g;
        off[c] = P.cls[c].tab_off; len[c] = rp_tab_slice(g.count, g.k, g.m); count[c] = g.count; tsz[c] = rp_tab_size(g.k, g.m);
    }
    return P.tab_scalars;
}

}
