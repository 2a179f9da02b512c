// TEST-ONLY host build of k_rp_decompress's staging arithmetic (rp_dec_block, rp_dec_offset, rp_dec_smem_bytes in rp.cuh): which
// proofs and commitments each block stages, and where in the stage each point's encoding lies, mapped back to the global buffers.
#include "../../bulletproofs_b200/csrc/rp.cuh"

static rp_geom dec_geom(uint32_t n, uint32_t m) {
    rp_geom g{};
    g.n = n; g.m = m; g.k = 0;
    while ((1u << g.k) < n * m) g.k++;
    g.N = n * m; g.D = 4 + 2 * g.k + m; g.S = 2 + 2 * g.N; g.proof_len = 32 * (9 + 2 * g.k);
    return g;
}

extern "C" {

uint32_t emul_rp_dec_smem(uint32_t n, uint32_t m) { return rp_dec_smem_bytes(dec_geom(n, m)); }
uint32_t emul_rp_dec_smem_max() { return rp_dec_smem_max(); }

// For every block of a launch over `count` proofs of (n, m): src[i] = where point i's 32 bytes come from, as a byte offset into the
// proof array, or into the commitment array with bit 63 set.  Returns the number of blocks whose stage breaks a bound: a read outside
// what the block copied, the proof part past rp_dec_proof_bytes, or the whole stage past rp_dec_smem_bytes.
uint32_t emul_rp_dec_sources(uint32_t n, uint32_t m, uint32_t count, uint64_t *src) {
    const rp_geom g = dec_geom(n, m);
    const uint64_t n_pts = (uint64_t)count * g.D, pb = rp_dec_proof_bytes(g);
    uint32_t bad = 0;
    for (uint64_t i0 = 0; i0 < n_pts; i0 += RP_DEC_THREADS) {
        const rp_dec_stage st = rp_dec_block(g, count, i0);
        const uint64_t a_bytes = (uint64_t)st.np * g.proof_len, b_bytes = 32ull * st.nc;
        bool ok = a_bytes <= pb && pb + b_bytes <= rp_dec_smem_bytes(g);
        for (uint64_t i = i0; i < i0 + RP_DEC_THREADS && i < n_pts; i++) {
            const uint64_t off = rp_dec_offset(g, st, i);
            if (off < pb) {
                ok = ok && off + 32 <= a_bytes;
                src[i] = (uint64_t)st.pf * g.proof_len + off;
            } else {
                ok = ok && off - pb + 32 <= b_bytes;
                src[i] = (1ull << 63) | (st.c0 * 32 + (off - pb));
            }
        }
        bad += ok ? 0 : 1;
    }
    return bad;
}

}
