// TEST-ONLY host build of the range-proof head: the device's form (rp_head_lean, specialised to a constant k as k_rp_head_seq
// instantiates it) and the sequential reference (rp_reduce_challenges + rp_scalars_head + rp_scalars_dynamic) on the same challenge
// rows.  Both write [zL | base-point scalar | blinding scalar | D dynamic scalars | the nine tables] as canonical bytes.
#include <utility>
#include <vector>
#include "../../bulletproofs_b200/csrc/rp.cuh"

typedef uint32_t (*lean_fn)(rp_lean_head &, sc *, uint8_t *, const sc *, const uint8_t *, const uint8_t *, uint32_t, uint32_t);
template <uint32_t K> static uint32_t lean_k(rp_lean_head &h, sc *tab, uint8_t *dyn, const sc *pow2, const uint8_t *raw, const uint8_t *proof, uint32_t n, uint32_t m) {
    return rp_head_lean(h, tab, dyn, pow2, raw, proof, K, n, m);
}
template <uint32_t... I> static lean_fn lean_pick(uint32_t k, std::integer_sequence<uint32_t, I...>) {
    static const lean_fn fns[] = {&lean_k<3 + I>...};
    return fns[k - 3];
}

static std::vector<sc> pow2_table() {
    std::vector<sc> t(64);
    for (int e = 0; e < 64; e++) t[e] = sc_mont_from_u64(1ULL << e);
    return t;
}
static void put_tables(uint8_t *out, const std::vector<sc> &tab) {
    for (size_t i = 0; i < tab.size(); i++) sc_store(out + 32 * i, sc_from_mont(tab[i]));
}

extern "C" {

// raw = RP_RAW_U + k challenge rows of 64 bytes; k in [3, BP_MAX_LG_N]; returns the proof's status (outputs written when 0)
int emul_rp_head_lean(const uint8_t *raw, const uint8_t *proof, uint32_t k, uint32_t n, uint32_t m, uint8_t *out) {
    if (k < 3 || k > BP_MAX_LG_N) return -1;
    const uint32_t D = 4 + 2 * k + m;
    std::vector<sc> tab(rp_tab_size(k, m)), pow2 = pow2_table();
    std::vector<uint64_t> rows((RP_RAW_U + k) * 8);                  // 8-byte aligned, as the device's raw array
    memcpy(rows.data(), raw, (RP_RAW_U + k) * 64);
    rp_lean_head h{};
    uint32_t st = lean_pick(k, std::make_integer_sequence<uint32_t, BP_MAX_LG_N - 2>())(h, tab.data(), out + 96, pow2.data(),
                                                                                           reinterpret_cast<const uint8_t *>(rows.data()), proof, n, m);
    if (st) return (int)st;
    sc_store(out, sc_from_mont(h.zL)); sc_store(out + 32, sc_from_mont(h.basepoint_scalar)); sc_store(out + 64, sc_from_mont(h.blinding_scalar));
    put_tables(out + 32 * (3 + D), tab);
    return 0;
}
int emul_rp_head_ref(const uint8_t *raw, const uint8_t *proof, uint32_t k, uint32_t n, uint32_t m, uint8_t *out) {
    if (k < 3 || k > BP_MAX_LG_N) return -1;
    const uint32_t D = 4 + 2 * k + m;
    static rp_challenges ch; static rp_head h;
    rp_reduce_challenges(ch, reinterpret_cast<const uint8_t (*)[64]>(raw), k);
    if (ch.status) return (int)ch.status;
    std::vector<sc> tab(rp_tab_size(k, m)), pow2 = pow2_table();
    rp_scalars_head(h, tab.data(), pow2.data(), ch, proof, k, n, m);
    sc_store(out, sc_from_mont(h.zL)); sc_store(out + 32, sc_from_mont(h.basepoint_scalar)); sc_store(out + 64, sc_from_mont(h.blinding_scalar));
    for (uint32_t d = 0; d < D; d++) sc_store(out + 32 * (3 + d), sc_from_mont(rp_scalars_dynamic(h, d, k)));
    put_tables(out + 32 * (3 + D), tab);
    return 0;
}
uint32_t emul_rp_tab_size(uint32_t k, uint32_t m) { return rp_tab_size(k, m); }

}
