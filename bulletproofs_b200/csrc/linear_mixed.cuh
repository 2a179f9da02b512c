// LinearProofs of different lengths in one call (bp_linear_verify_mixed): the host plan, and the class-aware front end on the device.
//
// Every proof over a set [B, F, G_0, G_1, ...] uses a prefix of it, so the proofs of every length share B, F and the low G_i, and ONE
// combined row checks them all:
//     [B | F | G_0 .. G_{Nmax-1} | C, S, L.., R.. of class 0's proofs | ... of class 1's proofs | ...]
// Nmax the longest admitted proof's n.  G_i's scalar sums rho a s_i over the proofs with n > i only.  The admitted proofs are grouped in
// classes of one n, classes in the order of their first proof, proofs in input order within a class ("class order"); every per-proof
// array (inputs, status, heads, verdicts) is in class order, and class c owns one slice of each arena, at the offsets of its linm_class.
// A G-sum chunk (LIN_CHUNK proofs) never crosses a class, so every block of k_linm_g_sum sums one n and one table layout.
// The host part is shared with the host-emulation tests (tests/host_emul/emul_linear_mixed.cpp).
#pragma once
#include <cstdint>
#include <map>
#include <vector>
#include "../../include/bpmsm.h"
#include "linear.cuh"

#define LINM_MAX_PROOFS (1u << 20)
#define LINM_MAX_N (1u << 20)
#define LINM_MAX_TERMS (1u << 31)
#define LINM_TILE 128           // generator indices per block of k_linm_g_sum: the tile of k_lin_g_sum at n >= 128

struct linm_class {
    uint32_t n, k, first, count;        // count proofs of n = 2^k, [first, first + count) in class order
    uint32_t proof_len, D, chunk0, tiles;   // D = lin_dyn_terms(k); first G-sum chunk; index tiles, ceil(n / LINM_TILE)
    uint64_t proof_off, b_off;          // bytes of gathered proofs; scalars of gathered b
    uint64_t raw_off, tab_off;          // 64-byte challenge rows; table scalars
    uint64_t part_off, b0_off;          // chunk sums: ceil(count / LIN_CHUNK) rows of n; b0 tile partials: tiles rows of count
    uint64_t dyn;                       // first dynamic point; its scalars are at Nmax + 2 + dyn in the combined row
    uint32_t live, pad_;                // proofs [first, first + live) are live, the rest inert slots (a reserved mix, live set per call)
};
struct linm_plan {
    std::vector<uint8_t> codes;         // per input proof: the parameter verdict (BP_PROOF_OK: admitted, the device decides)
    std::vector<uint32_t> order;        // input index of every admitted proof, in class order
    std::vector<linm_class> cls;
    uint32_t nmax = 0, chunks = 0;
    uint64_t terms = 0, dyn_points = 0, proof_bytes = 0, b_scalars = 0, raw_rows = 0, tab_scalars = 0, part_scalars = 0, b0_scalars = 0;
};

// The parameter checks of bp_linear_verify_batch for one proof of proof_len bytes and n public scalars over a set of set_n points, in
// the reference's order: LinearProof::from_bytes (a length no proof can have, then a non-canonical a or r: FormatError), the generators'
// length (InvalidGeneratorsLength), n = 2^(rounds) (VerificationError, n = 0 included).  BP_PROOF_OK, with *k the rounds, admits it.
// The host plan and the device planner of a reserved mix (linear_mixed_device.cuh) run the same code.
BP_HD uint8_t linm_param_verdict(const uint8_t *proof, size_t proof_len, size_t n, size_t set_n, uint32_t *k) {
    const size_t ne = proof_len / 32;
    if (proof_len % 32 != 0 || ne < 3 || (ne - 3) % 2 != 0 || (ne - 3) / 2 >= 32) return BP_PROOF_FORMAT_ERROR;
    *k = (uint32_t)((ne - 3) / 2);
    const uint8_t *ar = proof + 64 * (size_t)*k + 32;
    if (sc_geq_l(sc_load(ar)) || sc_geq_l(sc_load(ar + 32))) return BP_PROOF_FORMAT_ERROR;
    if (set_n < n + 2) return BP_PROOF_INVALID_GENERATORS_LENGTH;
    if (n != ((size_t)1 << *k)) return BP_PROOF_VERIFICATION_ERROR;
    return BP_PROOF_OK;
}

// Offsets of every class of P (n, k and count set) into the arenas, class after class, and the totals; every class's proofs live.  Returns
// nullptr, or the reason the layout is refused (2^31 MSM terms or more).
inline const char *linm_layout(linm_plan &P) {
    uint32_t first = 0;
    for (linm_class &K : P.cls) {
        K.proof_len = 32 * (2 * K.k + 3); K.D = lin_dyn_terms(K.k); K.tiles = (K.n + LINM_TILE - 1) / LINM_TILE;
        K.first = first; K.chunk0 = P.chunks;
        K.proof_off = P.proof_bytes; K.b_off = P.b_scalars; K.raw_off = P.raw_rows; K.tab_off = P.tab_scalars; K.part_off = P.part_scalars;
        K.b0_off = P.b0_scalars; K.dyn = P.dyn_points; K.live = K.count;
        const uint32_t nch = (K.count + LIN_CHUNK - 1) / LIN_CHUNK;
        P.proof_bytes += (uint64_t)K.count * K.proof_len; P.b_scalars += (uint64_t)K.count * K.n; P.raw_rows += (uint64_t)K.count * lin_raw_rows(K.k);
        P.tab_scalars += (uint64_t)K.count * lin_tab_size(K.k); P.part_scalars += (uint64_t)nch * K.n; P.b0_scalars += (uint64_t)K.tiles * K.count;
        P.dyn_points += (uint64_t)K.count * K.D;
        P.chunks += nch; first += K.count;
        if (K.n > P.nmax) P.nmax = K.n;
    }
    P.terms = P.cls.empty() ? 0 : P.nmax + 2 + P.dyn_points;
    if (P.terms >= LINM_MAX_TERMS) { P.cls.clear(); P.order.clear(); return "2^31 MSM terms or more"; }
    return nullptr;
}

// The plan of a call: proof j is proofs[proof_offsets[j] .. proof_offsets[j+1]) with the b_offsets[j+1] - b_offsets[j] scalars of b from
// b_offsets[j] on, over a set of set_n points.  Returns nullptr, or the reason the call is refused (no proof or more than 2^20, offsets
// that do not start at 0 or that decrease, an n above 2^20, 2^31 MSM terms or more).
inline const char *linm_make_plan(size_t count, const uint8_t *proofs, const uint64_t *proof_offsets, const uint64_t *b_offsets, size_t set_n, linm_plan &P) {
    P = linm_plan{};
    if (count == 0) return "no proofs";
    if (count > LINM_MAX_PROOFS) return "more than 2^20 proofs";
    if (proof_offsets[0] != 0 || b_offsets[0] != 0) return "proof and b offsets must start at 0";
    for (size_t j = 0; j < count; j++) {
        if (proof_offsets[j + 1] < proof_offsets[j] || b_offsets[j + 1] < b_offsets[j]) return "proof and b offsets must not decrease";
        if (b_offsets[j + 1] - b_offsets[j] > LINM_MAX_N) return "n above 2^20";
    }
    P.codes.resize(count);
    std::map<uint32_t, uint32_t> index;         // n -> class
    std::vector<std::vector<uint32_t>> members;
    for (size_t j = 0; j < count; j++) {
        const uint32_t n = (uint32_t)(b_offsets[j + 1] - b_offsets[j]);
        uint32_t k = 0;
        P.codes[j] = linm_param_verdict(proofs + proof_offsets[j], proof_offsets[j + 1] - proof_offsets[j], n, set_n, &k);
        if (P.codes[j] != BP_PROOF_OK) continue;
        auto it = index.emplace(n, (uint32_t)P.cls.size());
        if (it.second) { linm_class K{}; K.n = n; K.k = k; P.cls.push_back(K); members.emplace_back(); }
        members[it.first->second].push_back((uint32_t)j);
    }
    for (size_t c = 0; c < P.cls.size(); c++) P.cls[c].count = (uint32_t)members[c].size();
    if (const char *why = linm_layout(P)) return why;
    for (size_t c = 0; c < P.cls.size(); c++) P.order.insert(P.order.end(), members[c].begin(), members[c].end());
    return nullptr;
}

// A reserved mix (bp_linear_verify_mixed_reserve): n_classes lengths n[c], at most capacity[c] proofs each per call, over a set of set_n
// points, laid out at capacity, one class per n in reservation order (P.order and P.codes stay empty).  Returns nullptr, or the reason
// the mix is refused: no class or more than LINM_MAX_CLASSES, an n that is not a power of two up to 2^20 or repeats, a set shorter than
// n + 2, a capacity of 0 or above 2^20, or 2^31 MSM terms or more over the combined row and every class's reject-path slice.
#define LINM_MAX_CLASSES 21             // one per n = 2^0 .. 2^20
inline const char *linm_mix(size_t n_classes, const uint32_t *n, const uint32_t *capacity, size_t set_n, linm_plan &P) {
    P = linm_plan{};
    if (n_classes == 0 || n_classes > LINM_MAX_CLASSES) return "a mix holds 1 .. 21 lengths";
    for (size_t c = 0; c < n_classes; c++) {
        if (n[c] == 0 || (n[c] & (n[c] - 1)) || n[c] > LINM_MAX_N) return "every n must be a power of two up to 2^20";
        for (size_t j = 0; j < c; j++) if (n[j] == n[c]) return "duplicate n";
        if (set_n < (size_t)n[c] + 2) return "the point set has fewer than n + 2 points";
        if (capacity[c] == 0 || capacity[c] > LINM_MAX_PROOFS) return "capacity must be 1 .. 2^20";
        linm_class K{}; K.n = n[c]; K.count = capacity[c];
        while ((1u << K.k) < K.n) K.k++;
        P.cls.push_back(K);
    }
    if (const char *why = linm_layout(P)) return why;
    uint64_t terms = P.terms;
    for (const linm_class &K : P.cls) terms += (uint64_t)lin_x_slice(K.count, K.n, K.k) * (K.n + 2 + K.D);
    if (terms >= LINM_MAX_TERMS) { P.cls.clear(); return "2^31 MSM terms or more"; }
    return nullptr;
}

#ifdef __CUDACC__
#include "linear_kernels.cuh"
// ---------------------------------------------------------------------------------------------- kernels
// Each is the k_lin_* kernel of the same stage (linear_kernels.cuh) over every class at once: a thread or block finds its class in the
// table cls[0 .. C) (at most 21 classes, one per n = 2^0 .. 2^20) and works on that class's slices.

// the class whose range [start(c), start(c + 1)) holds v: the last one that starts at or below it
template <class Start>
__device__ __forceinline__ uint32_t linm_find(uint32_t C, uint64_t v, Start start) {
    uint32_t c = 0;
    while (c + 1 < C && start(c + 1) <= v) c++;
    return c;
}
__device__ __forceinline__ const linm_class &linm_of_proof(const linm_class *cls, uint32_t C, uint32_t q) {
    return cls[linm_find(C, q, [&](uint32_t c) { return (uint64_t)cls[c].first; })];
}

// where admitted proof q (class order) starts in the caller's buffers: proof bytes, b scalars, input index (transcript record and C)
struct linm_gather { uint64_t proof, b; uint32_t input, pad_; };
// the caller's inputs, uploaded as they are (or the caller's device buffers, at any alignment), gathered into class order: one block per
// admitted proof or slot; an inert slot copies nothing
__global__ void __launch_bounds__(128) k_linm_gather(const linm_class *__restrict__ cls, uint32_t C, const linm_gather *__restrict__ src,
                                                     const uint8_t *__restrict__ in_t, const uint8_t *__restrict__ in_p, const uint8_t *__restrict__ in_C,
                                                     const uint8_t *__restrict__ in_b, uint8_t *__restrict__ tstates, uint8_t *__restrict__ proofs,
                                                     uint8_t *__restrict__ Cs, uint8_t *__restrict__ b) {
    const uint32_t q = blockIdx.x;
    const linm_class &K = linm_of_proof(cls, C, q);
    const uint32_t r = q - K.first;
    if (r >= K.live) return;
    const linm_gather e = src[q];
    uint8_t *pd = proofs + K.proof_off + (size_t)r * K.proof_len;
    for (uint32_t i = threadIdx.x; i < K.proof_len; i += blockDim.x) pd[i] = in_p[e.proof + i];
    for (uint32_t i = threadIdx.x; i < BP_TRANSCRIPT_BYTES; i += blockDim.x) tstates[(size_t)q * BP_TRANSCRIPT_BYTES + i] = in_t[(size_t)e.input * BP_TRANSCRIPT_BYTES + i];
    if (threadIdx.x < 32) Cs[32 * (size_t)q + threadIdx.x] = in_C[32 * (size_t)e.input + threadIdx.x];
    const uint8_t *bsrc = in_b + 32 * e.b;
    uint8_t *bdst = b + 32 * (K.b_off + (size_t)r * K.n);                                       // 16-byte aligned: 32-byte scalars
    if (((uintptr_t)bsrc & 15u) == 0) {
        const uint4 *bs = reinterpret_cast<const uint4 *>(bsrc);
        uint4 *bd = reinterpret_cast<uint4 *>(bdst);
        for (uint32_t i = threadIdx.x; i < 2 * K.n; i += blockDim.x) bd[i] = bs[i];
    } else {
        for (uint32_t i = threadIdx.x; i < 32 * K.n; i += blockDim.x) bdst[i] = bsrc[i];
    }
}
// k_lin_decompress: one thread per dynamic point of every class; none for an inert slot
__global__ void __launch_bounds__(128) k_linm_decompress(const linm_class *__restrict__ cls, uint32_t C, uint64_t total, const uint8_t *__restrict__ proofs,
                                                         const uint8_t *__restrict__ Cs, ge_niels *__restrict__ out, uint32_t *__restrict__ dec_bad) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const linm_class &K = cls[linm_find(C, i, [&](uint32_t c) { return cls[c].dyn; })];
    const uint32_t k = K.k, r = (uint32_t)((i - K.dyn) / K.D), d = (uint32_t)((i - K.dyn) % K.D), q = K.first + r;
    if (r >= K.live) return;
    const uint8_t *proof = proofs + K.proof_off + (size_t)r * K.proof_len;
    const uint8_t *src = d == 0 ? Cs + 32 * (size_t)q : d == 1 ? proof + 64 * k : d < 2 + k ? proof + 64 * (d - 2) : proof + 64 * (d - 2 - k) + 32;
    uint8_t s[32]; ld32(s, src);
    fe x, y; const bool valid = ge_decode(x, y, s);
    st_niels(out + i, valid ? ge_to_niels_affine(x, y) : ge_niels_identity());
    if (!valid) dec_bad[q] = 1u;
}
// k_lin_transcript: one thread per proof; class order keeps a warp on one n, so its replays run the same number of absorbs.  An inert slot
// gets VerificationError, so that every later kernel leaves it out.
__global__ void __launch_bounds__(LIN_TR_THREADS) k_linm_transcript(const linm_class *__restrict__ cls, uint32_t C, uint32_t count, lin_params *__restrict__ par,
                                                                    const uint8_t *__restrict__ tstates, const uint8_t *__restrict__ proofs,
                                                                    const uint8_t *__restrict__ Cs, const uint8_t *__restrict__ b, const uint8_t *__restrict__ enc,
                                                                    uint8_t *__restrict__ raw, uint32_t *__restrict__ status) {
    __shared__ __align__(16) uint8_t rows[LIN_TR_THREADS][204];
    const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= count) return;
    const linm_class &K = linm_of_proof(cls, C, q);
    const uint32_t r = q - K.first;
    if (r >= K.live) { status[q] = BP_PROOF_VERIFICATION_ERROR; return; }
    const uint8_t *bq = b + 32 * (K.b_off + (size_t)r * K.n);
    if (!lin_b_canonical(bq, K.n)) { atomicOr(&par->noncanonical, 1u); status[q] = BP_VERDICT_NONCANONICAL_B; return; }
    uint8_t (*my)[64] = reinterpret_cast<uint8_t (*)[64]>(raw + 64 * (K.raw_off + (size_t)r * lin_raw_rows(K.k)));
    status[q] = lin_transcript_raw(my, proofs + K.proof_off + (size_t)r * K.proof_len, K.k, K.n, Cs + 32 * (size_t)q, bq, enc,
                                   tstates + (size_t)q * BP_TRANSCRIPT_BYTES, par->seed, rows[threadIdx.x]);
}
// k_lin_tables: one block per proof
__global__ void __launch_bounds__(128) k_linm_tables(const linm_class *__restrict__ cls, uint32_t C, const uint8_t *__restrict__ raw, const uint8_t *__restrict__ proofs,
                                                     int weighted, uint32_t *__restrict__ status, lin_head *__restrict__ heads, sc *__restrict__ tabs) {
    sc *xsh = lin_xsh;
    const uint32_t q = blockIdx.x, st = status[q];
    if (st != BP_PROOF_OK) { if (threadIdx.x == 0) heads[q].status = st; return; }
    const linm_class &K = linm_of_proof(cls, C, q);
    const uint32_t k = K.k, r = q - K.first, tsz = lin_tab_size(k);
    const uint8_t *rw = raw + 64 * (K.raw_off + (size_t)r * lin_raw_rows(k));
    for (uint32_t j = threadIdx.x; j < k; j += blockDim.x) xsh[j] = rp_wide(rw + 64 * j);
    __syncthreads();
    if (threadIdx.x == 0 && lin_head_init(heads[q], xsh, k, rw + 64 * k, rw + 64 * (k + 1), proofs + K.proof_off + (size_t)r * K.proof_len, weighted != 0) != BP_PROOF_OK)
        status[q] = heads[q].status;
    for (uint32_t e = threadIdx.x; e < tsz; e += blockDim.x) tabs[K.tab_off + (size_t)r * tsz + e] = lin_tab_entry(xsh, k, e);
}
// k_lin_g_sum over every class: block = (tile of LINM_TILE indices, global chunk); the chunk's class gives n, and a tile at or past n exits
// at once.  part_g[part_off + chunk * n + i] (Montgomery form) and part_b0[b0_off + tile * count + r] (plain) in the class's slices.  A
// chunk sums its live proofs only: one at or past the class's live count sums none, and writes zero G sums and no b0.
__global__ void __launch_bounds__(LINM_TILE) k_linm_g_sum(const linm_class *__restrict__ cls, uint32_t C, const lin_head *__restrict__ heads, const sc *__restrict__ tabs,
                                                          const uint8_t *__restrict__ b, const uint32_t *__restrict__ dec_bad, sc *__restrict__ part_g,
                                                          sc *__restrict__ part_b0) {
    __shared__ sc wsum[LINM_TILE / 32][LIN_CHUNK];
    const linm_class &K = cls[linm_find(C, blockIdx.y, [&](uint32_t c) { return (uint64_t)cls[c].chunk0; })];
    if (blockIdx.x >= K.tiles) return;                                      // the whole block
    const uint32_t n = K.n, k = K.k, tsz = lin_tab_size(k), lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    const uint32_t i = blockIdx.x * LINM_TILE + threadIdx.x, ch = blockIdx.y - K.chunk0;
    const uint32_t r0 = ch * LIN_CHUNK, r1 = max(r0, min(K.live, r0 + LIN_CHUNK));
    const uint32_t warps = min(LINM_TILE, n - blockIdx.x * LINM_TILE + 31u) / 32u;        // warps with an index below n
    const bool in = i < n;
    sc_wide acc = sc_wide_zero();
    if (warp < warps)
        for (uint32_t r = r0; r < r1; r++) {
            const uint32_t q = K.first + r;
            if (heads[q].status != BP_PROOF_OK || dec_bad[q]) continue;      // the same for the whole block
            sc t = sc_zero();
            if (in) { uint8_t bb[32]; ld32(bb, b + 32 * (K.b_off + (size_t)r * n + i)); t = lin_acc_add(acc, heads[q].wa, tabs + K.tab_off + (size_t)r * tsz, k, sc_load(bb), i); }
            for (int d = 16; d >= 1; d >>= 1) {
                sc o; for (int w = 0; w < 8; w++) o.v[w] = __shfl_down_sync(0xffffffffu, t.v[w], d);
                t = sc_add(t, o);
            }
            if (lane == 0) wsum[warp][r - r0] = t;
        }
    if (in) part_g[K.part_off + (size_t)ch * n + i] = sc_wide_redc(acc);
    __syncthreads();
    if (threadIdx.x < r1 - r0) {
        const uint32_t r = r0 + threadIdx.x, q = K.first + r;
        sc s = sc_zero();
        if (heads[q].status == BP_PROOF_OK && !dec_bad[q]) for (uint32_t w = 0; w < warps; w++) s = sc_add(s, wsum[w][threadIdx.x]);
        part_b0[K.b0_off + (size_t)blockIdx.x * K.count + r] = s;
    }
}
// k_lin_dynamic: per proof, b0 from its class's tile partials, its B and F scalars (bf) and its dynamic scalars and point map at its class's
// segment of the combined row
__global__ void __launch_bounds__(128) k_linm_dynamic(const linm_class *__restrict__ cls, uint32_t C, uint32_t count, uint32_t nmax, const lin_head *__restrict__ heads,
                                                      const uint32_t *__restrict__ dec_bad, const sc *__restrict__ part_b0, const uint8_t *__restrict__ proofs,
                                                      sc *__restrict__ bf, uint8_t *__restrict__ scal, uint32_t *__restrict__ pidx) {
    const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= count) return;
    const linm_class &K = linm_of_proof(cls, C, q);
    const uint32_t r = q - K.first, D = K.D;
    const bool ok = heads[q].status == BP_PROOF_OK && !dec_bad[q];
    sc sB = sc_zero(), sF = sc_zero();
    if (ok) {
        sc b0 = sc_zero();
        for (uint32_t t = 0; t < K.tiles; t++) b0 = sc_add(b0, part_b0[K.b0_off + (size_t)t * K.count + r]);
        lin_static_bf(heads[q], proofs + K.proof_off + (size_t)r * K.proof_len, K.k, b0, sB, sF);
    }
    bf[2 * (size_t)q] = sB; bf[2 * (size_t)q + 1] = sF;
    const uint64_t dyn = K.dyn + (uint64_t)r * D, base = (uint64_t)nmax + 2 + dyn;
    for (uint32_t d = 0; d < D; d++) {
        uint8_t bytes[32]; sc_store(bytes, ok ? lin_dyn_scalar(heads[q], d, K.k) : sc_zero());
        st32(scal + 32 * (base + d), bytes);
        pidx[base + d] = BP_POINT_DYNAMIC | (uint32_t)(dyn + d);
    }
}
// k_lin_g_total: one warp per static entry e < Nmax + 2.  B, F: every proof's bf; G_i: the chunk sums of every class with n > i.
__global__ void __launch_bounds__(32) k_linm_g_total(const linm_class *__restrict__ cls, uint32_t C, uint32_t count, const sc *__restrict__ part_g,
                                                     const sc *__restrict__ bf, uint8_t *__restrict__ scal, uint32_t *__restrict__ pidx) {
    const uint32_t e = blockIdx.x;
    sc acc = sc_zero();
    if (e < 2) for (uint32_t q = threadIdx.x; q < count; q += 32) acc = sc_add(acc, bf[2 * (size_t)q + e]);
    else
        for (uint32_t c = 0; c < C; c++) {
            const linm_class &K = cls[c];
            if (K.n <= e - 2) continue;
            const uint32_t nch = (K.count + LIN_CHUNK - 1) / LIN_CHUNK;
            for (uint32_t ch = threadIdx.x; ch < nch; ch += 32) acc = sc_add(acc, part_g[K.part_off + (size_t)ch * K.n + e - 2]);
        }
    for (int d = 16; d >= 1; d >>= 1) {
        sc o; for (int w = 0; w < 8; w++) o.v[w] = __shfl_down_sync(0xffffffffu, acc.v[w], d);
        acc = sc_add(acc, o);
    }
    if (threadIdx.x == 0) {
        uint8_t bytes[32]; sc_store(bytes, e < 2 ? acc : sc_from_mont(acc));
        st32(scal + 32 * (size_t)e, bytes); pidx[e] = e;
    }
}
#endif
