// TEST-ONLY host build of the LinearProof batch verifier's transcript replay and scalar algebra (csrc/linear.cuh compiled with g++),
// linked into libemul.so beside emul.cpp.  It lets the CPU-only test tier check the replayed challenges, the tables, b0 and the G sums
// against Python without a GPU.  Nothing in the product links this.
#include <algorithm>
#include <cstring>
#include <vector>
#include "../../bulletproofs_b200/csrc/linear.cuh"

extern "C" {

// lin_transcript_raw of one proof (k rounds, n = 2^k): raw = (k + 2) x 64 bytes (x_0 .., x*, rho); enc = [B, F, G_0 .. G_{n-1}]
uint32_t emul_lin_transcript(const uint8_t *proof, uint32_t k, uint32_t n, const uint8_t *C, const uint8_t *b, const uint8_t *enc, const uint8_t *tstate,
                             const uint8_t *seed, uint8_t *raw) {
    alignas(8) uint8_t st[200];
    return lin_transcript_raw(reinterpret_cast<uint8_t (*)[64]>(raw), proof, k, n, C, b, enc, tstate, seed, st);
}
// The batch's scalars as k_lin_tables, k_lin_g_sum and k_lin_dynamic compute them, from each proof's raw challenge rows: `count`
// proofs of n = 2^k, chunks of `chunk` proofs, rho from the rows (weighted) or 1.  Outputs, canonical scalars:
//   out_g  ceil(count / chunk) rows of n: sum over the chunk's proofs of rho a s_i
//   out_p  per proof: s_0 .. s_{n-1}, b0, B, F, then the 2 + 2k dynamic scalars C, S, L.., R..
//   status per proof (VerificationError for a zero challenge); a rejected proof adds nothing and gets zero scalars
void emul_lin_scalars(uint32_t count, uint32_t k, const uint8_t *raws, const uint8_t *proofs, uint32_t proof_len, const uint8_t *b, int weighted, uint32_t chunk,
                      uint8_t *out_g, uint8_t *out_p, uint32_t *status) {
    const uint32_t n = 1u << k, tsz = lin_tab_size(k), D = lin_dyn_terms(k), per = n + 3 + D;
    std::vector<lin_head> H(count); std::vector<sc> tabs((size_t)count * tsz), b0(count, sc_zero());
    for (uint32_t q = 0; q < count; q++) {
        const uint8_t *rw = raws + (size_t)q * lin_raw_rows(k) * 64, *proof = proofs + (size_t)q * proof_len;
        sc x[BP_MAX_LG_N];
        for (uint32_t j = 0; j < k; j++) x[j] = rp_wide(rw + 64 * j);
        status[q] = lin_head_init(H[q], x, k, rw + 64 * k, rw + 64 * (k + 1), proof, weighted != 0);
        for (uint32_t e = 0; e < tsz; e++) tabs[(size_t)q * tsz + e] = lin_tab_entry(x, k, e);
    }
    for (uint32_t ch = 0; ch * chunk < count; ch++)
        for (uint32_t i = 0; i < n; i++) {
            sc_wide acc = sc_wide_zero();
            for (uint32_t q = ch * chunk; q < std::min(count, (ch + 1) * chunk); q++) {
                if (status[q] != BP_PROOF_OK) continue;
                b0[q] = sc_add(b0[q], lin_acc_add(acc, H[q].wa, tabs.data() + (size_t)q * tsz, k, sc_load(b + ((size_t)q * n + i) * 32), i));
            }
            sc_store(out_g + 32 * ((size_t)ch * n + i), sc_from_mont(sc_wide_redc(acc)));
        }
    for (uint32_t q = 0; q < count; q++) {
        uint8_t *o = out_p + 32 * (size_t)q * per;
        const sc *tab = tabs.data() + (size_t)q * tsz; const uint32_t kl = rp_kl(k), TL = 1u << kl;
        for (uint32_t i = 0; i < n; i++) sc_store(o + 32 * i, sc_from_mont(sc_mm(tab[TL + (i >> kl)], tab[i & (TL - 1)])));
        const bool ok = status[q] == BP_PROOF_OK;
        sc sB = sc_zero(), sF = sc_zero();
        if (ok) lin_static_bf(H[q], proofs + (size_t)q * proof_len, k, b0[q], sB, sF);
        sc_store(o + 32 * n, b0[q]); sc_store(o + 32 * (n + 1), sB); sc_store(o + 32 * (n + 2), sF);
        for (uint32_t d = 0; d < D; d++) sc_store(o + 32 * (n + 3 + d), ok ? lin_dyn_scalar(H[q], d, k) : sc_zero());
    }
}
}
