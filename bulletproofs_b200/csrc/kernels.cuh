// Device kernels of the MSM engine (sm_90a).  One thread = one independent point / bucket /
// scalar operation; a warp therefore carries 32 independent chains of the 8x32-bit-limb field
// arithmetic in fe.cuh.  The work is integer-pipe bound (IMAD.WIDE), not HBM bound: one 64-byte
// MSM term buys ~W mixed additions = W*7 field multiplications = W*7*72 wide multiplies.
#pragma once
#include <cuda_runtime.h>
#include <utility>
#include "ge.cuh"
#include "sc.cuh"
#include "merlin.cuh"
#include "rp.cuh"
#include "msm_common.cuh"

#define BP_POINT_DYNAMIC 0x80000000u     // point_idx flag: index into the per-call (dynamic) point array

// slot of G[party][index] (which = 0) or H[party][index] (which = 1) in the generator table [B_blinding, B, G[party][i].., H[party][i]..]
BP_HD size_t bp_gens_slot(size_t which, size_t party, size_t index, size_t cap, size_t parties) { return 2 + (which * parties + party) * cap + index; }

// ------------------------------------------------------------------ vector load/store helpers
__device__ __forceinline__ void ld32(uint8_t dst[32], const uint8_t *src) {       // 32 B, 16-B aligned
    const uint4 *p = reinterpret_cast<const uint4 *>(src);
    uint4 a = __ldg(p), b = __ldg(p + 1);
    uint32_t w[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
    memcpy(dst, w, 32);
}
__device__ __forceinline__ void ld32_any(uint8_t dst[32], const uint8_t *src) {   // any alignment (proof bytes)
    if ((reinterpret_cast<uintptr_t>(src) & 15) == 0) { ld32(dst, src); return; }
    if ((reinterpret_cast<uintptr_t>(src) & 3) == 0) { const uint32_t *p = reinterpret_cast<const uint32_t *>(src); uint32_t w[8]; for (int i = 0; i < 8; i++) w[i] = __ldg(p + i); memcpy(dst, w, 32); return; }
    for (int i = 0; i < 32; i++) dst[i] = src[i];
}
__device__ __forceinline__ void st32(uint8_t *dst, const uint8_t src[32]) {
    uint32_t w[8]; memcpy(w, src, 32);
    uint4 *p = reinterpret_cast<uint4 *>(dst);
    p[0] = make_uint4(w[0], w[1], w[2], w[3]); p[1] = make_uint4(w[4], w[5], w[6], w[7]);
}
__device__ __forceinline__ fe ld_fe(const fe *p) {
    const uint4 *q = reinterpret_cast<const uint4 *>(p); uint4 a = q[0], b = q[1];
    fe r; r.v[0] = a.x; r.v[1] = a.y; r.v[2] = a.z; r.v[3] = a.w; r.v[4] = b.x; r.v[5] = b.y; r.v[6] = b.z; r.v[7] = b.w; return r;
}
__device__ __forceinline__ fe ldg_fe(const fe *p) {
    const uint4 *q = reinterpret_cast<const uint4 *>(p); uint4 a = __ldg(q), b = __ldg(q + 1);
    fe r; r.v[0] = a.x; r.v[1] = a.y; r.v[2] = a.z; r.v[3] = a.w; r.v[4] = b.x; r.v[5] = b.y; r.v[6] = b.z; r.v[7] = b.w; return r;
}
__device__ __forceinline__ void st_fe(fe *p, const fe &v) {
    uint4 *q = reinterpret_cast<uint4 *>(p);
    q[0] = make_uint4(v.v[0], v.v[1], v.v[2], v.v[3]); q[1] = make_uint4(v.v[4], v.v[5], v.v[6], v.v[7]);
}
__device__ __forceinline__ ge_niels ldg_niels(const ge_niels *p) { ge_niels r; r.ypx = ldg_fe(&p->ypx); r.ymx = ldg_fe(&p->ymx); r.xy2d = ldg_fe(&p->xy2d); return r; }
__device__ __forceinline__ void st_niels(ge_niels *p, const ge_niels &v) { st_fe(&p->ypx, v.ypx); st_fe(&p->ymx, v.ymx); st_fe(&p->xy2d, v.xy2d); }
__device__ __forceinline__ ge_ext ld_ext(const ge_ext *p) { ge_ext r; r.X = ld_fe(&p->X); r.Y = ld_fe(&p->Y); r.Z = ld_fe(&p->Z); r.T = ld_fe(&p->T); return r; }
__device__ __forceinline__ void st_ext(ge_ext *p, const ge_ext &v) { st_fe(&p->X, v.X); st_fe(&p->Y, v.Y); st_fe(&p->Z, v.Z); st_fe(&p->T, v.T); }

__device__ __forceinline__ ge_ext shfl_down_ext(const ge_ext &p, int d) {
    ge_ext r;
#pragma unroll
    for (int i = 0; i < 8; i++) {
        r.X.v[i] = __shfl_down_sync(0xffffffffu, p.X.v[i], d); r.Y.v[i] = __shfl_down_sync(0xffffffffu, p.Y.v[i], d);
        r.Z.v[i] = __shfl_down_sync(0xffffffffu, p.Z.v[i], d); r.T.v[i] = __shfl_down_sync(0xffffffffu, p.T.v[i], d);
    }
    return r;
}

// ------------------------------------------------------------------ TMA staging of the streaming byte arrays
// The scalar and compressed-point arrays are read once, front to back.  Each block stages its contiguous tile
// (32 B per thread) into shared memory with ONE bulk asynchronous copy (cp.async.bulk: the TMA engine, SASS UBLKCP)
// signalled through an mbarrier, instead of one 2x128-bit global load pair per thread; threads then read their
// record from shared memory.  src must be 16-byte aligned, bytes a multiple of 16 (records are 32 B).
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void tma_stage_tile(void *smem_dst, const void *gsrc, uint32_t bytes, uint64_t *bar) {
    uint32_t b = smem_u32(bar);
    if (threadIdx.x == 0) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(b));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(b), "r"(bytes) : "memory");
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                     ::"r"(smem_u32(smem_dst)), "l"(gsrc), "r"(bytes), "r"(b) : "memory");
    }
    uint32_t done;
    do {
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], 0;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(done) : "r"(b) : "memory");
    } while (!done);
}
// Two-source form for the per-proof kernels: a block's slice of the proof array and of the commitment array (both contiguous,
// 16-byte aligned when the caller's buffers are) land in shared memory through two bulk copies signalled on one mbarrier; the
// threads then take their 32-byte fields -- at offsets that are not 16-byte aligned in general -- from shared memory.
// Falls back to a cooperative copy for buffers that are not 16-byte aligned.  bytes_b may be 0 (no second copy is issued).
__device__ __forceinline__ void tma_stage_two(uint8_t *dst_a, const uint8_t *src_a, uint32_t bytes_a, uint8_t *dst_b, const uint8_t *src_b, uint32_t bytes_b, uint64_t *bar) {
    const bool aligned = ((reinterpret_cast<uintptr_t>(src_a) | reinterpret_cast<uintptr_t>(src_b) | bytes_a | bytes_b) & 15) == 0;
    if (!aligned) {
        for (uint32_t i = threadIdx.x; i < bytes_a; i += blockDim.x) dst_a[i] = src_a[i];
        for (uint32_t i = threadIdx.x; i < bytes_b; i += blockDim.x) dst_b[i] = src_b[i];
        __syncthreads();
        return;
    }
    uint32_t b = smem_u32(bar);
    if (threadIdx.x == 0) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(b));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(b), "r"(bytes_a + bytes_b) : "memory");
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                     ::"r"(smem_u32(dst_a)), "l"(src_a), "r"(bytes_a), "r"(b) : "memory");
        if (bytes_b)
            asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                         ::"r"(smem_u32(dst_b)), "l"(src_b), "r"(bytes_b), "r"(b) : "memory");
    }
    uint32_t done;
    do {
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], 0;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(done) : "r"(b) : "memory");
    } while (!done);
}
__device__ __forceinline__ void lds32(uint8_t dst[32], const uint8_t *smem_src) {
    const uint4 *p = reinterpret_cast<const uint4 *>(smem_src);
    uint4 a = p[0], b = p[1];
    uint32_t w[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
    memcpy(dst, w, 32);
}

// ------------------------------------------------------------------ K1: batched Ristretto decompress
// in: n x 32 B compressed.  out: n affine-Niels points (identity when invalid), ok[i] in {0,1}.
__global__ void __launch_bounds__(128) k_decompress(const uint8_t *__restrict__ in, size_t n, ge_niels *__restrict__ out, uint8_t *__restrict__ ok) {
    __shared__ __align__(128) uint8_t tile[128 * 32];
    __shared__ __align__(8) uint64_t bar;
    size_t base = (size_t)blockIdx.x * blockDim.x, i = base + threadIdx.x;
    uint32_t cnt = (uint32_t)min((size_t)blockDim.x, n - base);
    tma_stage_tile(tile, in + 32 * base, 32u * cnt, &bar);
    if (i >= n) return;
    uint8_t s[32]; lds32(s, tile + 32 * threadIdx.x);
    fe x, y; bool valid = ge_decode(x, y, s);
    ge_niels q = valid ? ge_to_niels_affine(x, y) : ge_niels_identity();
    st_niels(out + i, q);
    if (ok) ok[i] = valid ? 1 : 0;
}

// ------------------------------------------------------------------ K3: batched compress / identity test
__global__ void __launch_bounds__(128) k_compress(const ge_ext *__restrict__ in, size_t n, uint8_t *__restrict__ out) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint8_t s[32]; ge_encode(s, ld_ext(in + i)); st32(out + 32 * i, s);
}

// ------------------------------------------------------------------ K7: from_uniform_bytes (generator chain)
// in: n x 64 B.  out: affine-Niels table entry and/or compressed bytes.
__global__ void __launch_bounds__(128) k_from_uniform(const uint8_t *__restrict__ in, size_t n, ge_niels *__restrict__ out_niels, uint8_t *__restrict__ out_comp) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint8_t u[64]; ld32(u, in + 64 * i); ld32(u + 32, in + 64 * i + 32);
    ge_ext p = ge_from_uniform(u);
    if (out_comp) { uint8_t s[32]; ge_encode(s, p); st32(out_comp + 32 * i, s); }
    if (out_niels) { fe zi = fe_invert(p.Z); st_niels(out_niels + i, ge_to_niels_affine(fe_mul(p.X, zi), fe_mul(p.Y, zi))); }
}
__global__ void __launch_bounds__(128) k_niels_to_compressed(const ge_niels *__restrict__ in, size_t n, uint8_t *__restrict__ out) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint8_t s[32]; ge_encode(s, ge_from_niels(ldg_niels(in + i))); st32(out + 32 * i, s);
}

// ------------------------------------------------------------------ K2: Pippenger bucket pipeline
// A batch of n_msm MSMs over a flat term array.  "segment" = (msm, window); every segment owns nb =
// 2^(c-1) buckets and a slice of `sorted` with room for all terms of its MSM:
//     seg = msm*W + w,   slice base = W*offsets[msm] + w*len,  len = offsets[msm+1]-offsets[msm].
// Buckets are accumulated by one thread each, except "heavy" ones (size >= heavy_min, chosen by the host as a multiple
// of the mean bucket size): k_msm_order lists those and k_msm_accumulate_heavy gives each a whole block.  Heavy buckets
// are not an adversarial corner only: scalars are < l ~ 2^252, so when c*(W-1) = 252 (c = 9, 12, ...) the top window
// holds nothing but the recoding carry and HALF of all terms land in its bucket 0.
// Every pass takes an optional `gate`: when it is given and *gate == 0 the whole grid returns at once (a launch group's per-batch
// pass on the direct-launch path, which only has work when the group's combined check failed).  nullptr = always run.
#define MSM_SKIP(gate) ((gate) != nullptr && *(gate) == 0u)
__device__ __forceinline__ size_t msm_slice_base(uint32_t o0, uint32_t len, uint32_t w, int W) {
    return (size_t)W * (size_t)o0 + (size_t)w * (size_t)len;
}
__device__ __forceinline__ uint32_t msm_of_term(const uint32_t *__restrict__ offsets, uint32_t n_msm, uint32_t t) {
    uint32_t lo = 0, hi = n_msm;            // largest j with offsets[j] <= t
    while (hi - lo > 1) { uint32_t mid = (lo + hi) >> 1; if (__ldg(offsets + mid) <= t) lo = mid; else hi = mid; }
    return lo;
}

// pass 1: histogram.  One thread per term; scalars are 32-byte canonical little-endian.
__global__ void __launch_bounds__(256) k_msm_count(const uint8_t *__restrict__ scalars, const uint32_t *__restrict__ offsets, uint32_t n_msm, uint32_t T,
                                                   int c, int W, uint32_t *__restrict__ counts, uint32_t *__restrict__ msm_err, const uint32_t *__restrict__ gate) {
    __shared__ __align__(128) uint8_t tile[256 * 32];
    __shared__ __align__(8) uint64_t bar;
    if (MSM_SKIP(gate)) return;
    uint32_t base = blockIdx.x * blockDim.x, t = base + threadIdx.x;
    tma_stage_tile(tile, scalars + 32 * (size_t)base, 32u * min(blockDim.x, T - base), &bar);
    if (t >= T) return;
    uint8_t sb[32]; lds32(sb, tile + 32 * threadIdx.x);
    sc s = sc_load(sb);
    uint32_t msm = n_msm == 1 ? 0u : msm_of_term(offsets, n_msm, t);
    if (sc_geq_l(s)) { if (msm_err) atomicOr(msm_err + msm, 2u); return; }       // non-canonical scalar
    msm_wide r = msm_recode(s.v, c, W);
    uint32_t nb = 1u << (c - 1);
    for (int w = 0; w < W; w++) {
        int d = msm_digit(r, w, c);
        if (d == 0) continue;
        uint32_t b = (uint32_t)(d < 0 ? -d : d) - 1u;
        atomicAdd(counts + ((size_t)msm * W + w) * nb + b, 1u);
    }
}
// pass 2: per-segment exclusive scan of the bucket counts (block per segment); cursor starts as a copy
#define MSM_SIZE_BINS 256        // bucket sizes are clamped to MSM_SIZE_BINS-1 for the load-balancing order
__global__ void __launch_bounds__(256) k_msm_scan(const uint32_t *__restrict__ counts, uint32_t nb, uint32_t *__restrict__ starts, uint32_t *__restrict__ cursor,
                                                  uint32_t *__restrict__ size_hist, const uint32_t *__restrict__ gate) {
    __shared__ uint32_t warp_sums[8];
    if (MSM_SKIP(gate)) return;
    __shared__ uint32_t hist[MSM_SIZE_BINS];
    for (uint32_t i = threadIdx.x; i < MSM_SIZE_BINS; i += blockDim.x) hist[i] = 0;
    __syncthreads();
    size_t seg = blockIdx.x;
    const uint32_t *cnt = counts + seg * nb; uint32_t *st = starts + seg * nb, *cu = cursor + seg * nb;
    uint32_t per = (nb + blockDim.x - 1) / blockDim.x;
    uint32_t lo = threadIdx.x * per, hi = min(lo + per, nb);
    uint32_t local = 0;
    for (uint32_t i = lo; i < hi; i++) local += cnt[i];
    // block exclusive scan of `local`
    uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5, v = local;
    for (int d = 1; d < 32; d <<= 1) { uint32_t o = __shfl_up_sync(0xffffffffu, v, d); if (lane >= (uint32_t)d) v += o; }
    if (lane == 31) warp_sums[wid] = v;
    __syncthreads();
    uint32_t base = 0;
    for (uint32_t k = 0; k < wid; k++) base += warp_sums[k];
    uint32_t run = base + v - local;
    for (uint32_t i = lo; i < hi; i++) { uint32_t c_ = cnt[i]; st[i] = run; cu[i] = run; run += c_; atomicAdd(&hist[MSM_SIZE_BINS - 1 - min(c_, (uint32_t)MSM_SIZE_BINS - 1)], 1u); }
    __syncthreads();
    for (uint32_t i = threadIdx.x; i < MSM_SIZE_BINS; i += blockDim.x) if (hist[i]) atomicAdd(size_hist + i, hist[i]);
}
// load-balancing order: bucket ids sorted by decreasing size (counting sort over the size histogram), so that the 32
// buckets a warp accumulates have (nearly) equal lengths and the longest buckets start first
__global__ void __launch_bounds__(256) k_msm_order(const uint32_t *__restrict__ counts, size_t n_buckets, const uint32_t *__restrict__ size_hist,
                                                   uint32_t *__restrict__ bin_cursor, uint32_t *__restrict__ order, uint32_t heavy_min,
                                                   uint32_t *__restrict__ heavy_n, uint32_t *__restrict__ heavy, const uint32_t *__restrict__ gate) {
    __shared__ uint32_t base[MSM_SIZE_BINS];
    if (MSM_SKIP(gate)) return;
    __shared__ uint32_t wsum[8];
    __shared__ uint32_t local[MSM_SIZE_BINS];          // this block's buckets per bin, then the block's base within the bin
    {   // exclusive scan of the 256-bin histogram, redundantly per block
        uint32_t v = size_hist[threadIdx.x], lane = threadIdx.x & 31, wid = threadIdx.x >> 5, x = v;
        for (int d = 1; d < 32; d <<= 1) { uint32_t o = __shfl_up_sync(0xffffffffu, x, d); if (lane >= (uint32_t)d) x += o; }
        if (lane == 31) wsum[wid] = x;
        local[threadIdx.x] = 0;
        __syncthreads();
        uint32_t b = 0; for (uint32_t k = 0; k < wid; k++) b += wsum[k];
        base[threadIdx.x] = b + x - v;
        __syncthreads();
    }
    // rank within (block, bin) through shared-memory atomics, then ONE global atomic per non-empty bin of the block: the buckets of a
    // window have nearly equal sizes, so per-bucket global atomics on a handful of bin cursors serialise (46 us for 786k buckets)
    size_t gb = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    bool live = gb < n_buckets;
    uint32_t cnt = live ? counts[gb] : 0;
    uint32_t bin = MSM_SIZE_BINS - 1 - min(cnt, (uint32_t)MSM_SIZE_BINS - 1);
    uint32_t rank = live ? atomicAdd(&local[bin], 1u) : 0;
    __syncthreads();
    { uint32_t mine = local[threadIdx.x]; __syncthreads(); local[threadIdx.x] = mine ? atomicAdd(bin_cursor + threadIdx.x, mine) : 0; }
    __syncthreads();
    if (!live) return;
    order[base[bin] + local[bin] + rank] = (uint32_t)gb;
    if (cnt >= heavy_min) heavy[atomicAdd(heavy_n, 1u)] = (uint32_t)gb;
}
// pass 3: scatter term ids (sign in bit 31) into their bucket's slice
__global__ void __launch_bounds__(256) k_msm_scatter(const uint8_t *__restrict__ scalars, const uint32_t *__restrict__ offsets, uint32_t n_msm, uint32_t T,
                                                     int c, int W, uint32_t *__restrict__ cursor, uint32_t *__restrict__ sorted, const uint32_t *__restrict__ gate) {
    __shared__ __align__(128) uint8_t tile[256 * 32];
    __shared__ __align__(8) uint64_t bar;
    if (MSM_SKIP(gate)) return;
    uint32_t base = blockIdx.x * blockDim.x, t = base + threadIdx.x;
    tma_stage_tile(tile, scalars + 32 * (size_t)base, 32u * min(blockDim.x, T - base), &bar);
    if (t >= T) return;
    uint8_t sb[32]; lds32(sb, tile + 32 * threadIdx.x);
    sc s = sc_load(sb);
    if (sc_geq_l(s)) return;
    uint32_t msm = n_msm == 1 ? 0u : msm_of_term(offsets, n_msm, t);
    uint32_t o0 = __ldg(offsets + msm), len = __ldg(offsets + msm + 1) - o0;
    msm_wide r = msm_recode(s.v, c, W);
    uint32_t nb = 1u << (c - 1);
    for (int w = 0; w < W; w++) {
        int d = msm_digit(r, w, c);
        if (d == 0) continue;
        uint32_t b = (uint32_t)(d < 0 ? -d : d) - 1u;
        uint32_t pos = atomicAdd(cursor + ((size_t)msm * W + w) * nb + b, 1u);
        sorted[msm_slice_base(o0, len, (uint32_t)w, W) + pos] = t | (d < 0 ? 0x80000000u : 0u);
    }
}
// heavy buckets (size >= heavy_min, listed by k_msm_order): one 128-thread block per bucket, grid-stride over the list: threads take
// strided entries, then a shuffle tree + one shared-memory round add the partial sums.  Runs in the first blocks of k_msm_accumulate's
// grid (a separate launch would wait for an SM with a free block slot behind the wide kernels of the other groups in flight).
#define MSM_ACC_THREADS 128
__device__ __noinline__ void msm_heavy_role(const uint32_t *__restrict__ starts, const uint32_t *__restrict__ ends, const uint32_t *__restrict__ sorted,
                                            const uint32_t *__restrict__ offsets, const uint32_t *__restrict__ heavy_n, const uint32_t *__restrict__ heavy, int W, uint32_t nb,
                                            const uint32_t *__restrict__ point_idx, const ge_niels *__restrict__ pts_static, const ge_niels *__restrict__ pts_dynamic,
                                            ge_ext *__restrict__ buckets, uint32_t first, uint32_t stride) {
    __shared__ ge_ext sm[MSM_ACC_THREADS / 32];
    uint32_t n_heavy = *heavy_n, lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    for (uint32_t h = first; h < n_heavy; h += stride) {
        size_t gb = heavy[h];
        size_t seg = gb / nb; uint32_t msm = (uint32_t)(seg / W), w = (uint32_t)(seg % W);
        uint32_t o0 = __ldg(offsets + msm), len = __ldg(offsets + msm + 1) - o0;
        const uint32_t *slice = sorted + msm_slice_base(o0, len, w, W);
        uint32_t lo = starts[gb], hi = ends[gb];
        ge_ext acc = ge_identity();
        for (uint32_t e = lo + threadIdx.x; e < hi; e += blockDim.x) {
            uint32_t v = __ldg(slice + e), t = v & 0x7fffffffu;
            uint32_t pi = point_idx ? __ldg(point_idx + t) : (t | BP_POINT_DYNAMIC);
            const ge_niels *src = (pi & BP_POINT_DYNAMIC) ? pts_dynamic + (pi & 0x7fffffffu) : pts_static + pi;
            ge_niels q = ldg_niels(src);
            if (v & 0x80000000u) q = ge_niels_neg(q);
            acc = ge_madd(acc, q);
        }
#pragma unroll 1
        for (int d = 16; d >= 1; d >>= 1) { ge_ext o = shfl_down_ext(acc, d); acc = ge_add(acc, o); }
        if (lane == 0) sm[wid] = acc;
        __syncthreads();
        if (wid == 0) {
            ge_ext r = lane < (blockDim.x >> 5) ? sm[lane] : ge_identity();
#pragma unroll 1
            for (int d = 2; d >= 1; d >>= 1) { ge_ext o = shfl_down_ext(r, d); r = ge_add(r, o); }
            if (lane == 0) st_ext(buckets + gb, r);
        }
        __syncthreads();
    }
}
// pass 4: bucket accumulation, SPLIT adjacent lanes per bucket: each sums every SPLIT-th +-point of the bucket's slice (mixed
// additions), a shuffle tree adds the partial sums.  SPLIT > 1 trades (SPLIT-1) full additions per bucket for SPLIT x more warps
// in flight and a SPLIT x shorter serial chain per thread.
template <int SPLIT>
__global__ void __launch_bounds__(128, 5) k_msm_accumulate(const uint32_t *__restrict__ starts, const uint32_t *__restrict__ ends, const uint32_t *__restrict__ sorted,
                                                        const uint32_t *__restrict__ offsets, const uint32_t *__restrict__ order, int W, uint32_t nb, size_t n_buckets,
                                                        const uint32_t *__restrict__ point_idx, const ge_niels *__restrict__ pts_static, const ge_niels *__restrict__ pts_dynamic,
                                                        ge_ext *__restrict__ buckets, uint32_t heavy_min, uint32_t n_light_blocks, const uint32_t *__restrict__ heavy_n, const uint32_t *__restrict__ heavy,
                                                        const uint32_t *__restrict__ gate) {
    if (MSM_SKIP(gate)) return;
    const uint32_t n_heavy_blocks = gridDim.x - n_light_blocks;
    if (blockIdx.x < n_heavy_blocks) {        // the grid's FIRST blocks own the heavy buckets (listed by k_msm_order), one block per bucket: the longest work starts first
        msm_heavy_role(starts, ends, sorted, offsets, heavy_n, heavy, W, nb, point_idx, pts_static, pts_dynamic, buckets, blockIdx.x, n_heavy_blocks);
        return;
    }
    size_t tid = (size_t)(blockIdx.x - n_heavy_blocks) * blockDim.x + threadIdx.x;
    size_t b = tid / SPLIT; uint32_t sub = (uint32_t)(tid % SPLIT);
    bool live = b < n_buckets;
    if (SPLIT == 1 && !live) return;
    size_t gb = live ? order[b] : 0;
    size_t seg = gb / nb; uint32_t msm = (uint32_t)(seg / W), w = (uint32_t)(seg % W);
    uint32_t o0 = __ldg(offsets + msm), len = __ldg(offsets + msm + 1) - o0;
    const uint32_t *slice = sorted + msm_slice_base(o0, len, w, W);
    uint32_t lo = starts[gb], hi = ends[gb];
    if (hi - lo >= heavy_min) live = false;     // k_msm_accumulate_heavy owns this bucket
    if (!live) { if (SPLIT == 1) return; lo = hi = 0; }
    ge_ext acc = ge_identity();
    for (uint32_t e = lo + sub; e < hi; e += SPLIT) {
        uint32_t v = __ldg(slice + e), t = v & 0x7fffffffu;
        uint32_t pi = point_idx ? __ldg(point_idx + t) : (t | BP_POINT_DYNAMIC);
        const ge_niels *src = (pi & BP_POINT_DYNAMIC) ? pts_dynamic + (pi & 0x7fffffffu) : pts_static + pi;
        ge_niels q = ldg_niels(src);
        if (v & 0x80000000u) q = ge_niels_neg(q);
        acc = ge_madd(acc, q);
    }
    if (SPLIT > 1) {
#pragma unroll 1
        for (int d = SPLIT / 2; d >= 1; d >>= 1) { ge_ext o = shfl_down_ext(acc, d); acc = ge_add(acc, o); }
    }
    if (live && sub == 0) st_ext(buckets + gb, acc);
}
// pass 5: bucket reduction  R = sum_j (j+1) B_j  per segment, one block per segment.
// Each thread owns a contiguous chunk; a warp-shuffle suffix scan over the chunk sums gives every
// thread the sum of all buckets above its chunk, then one running-sum pass finishes the chunk and
// a shuffle tree adds the per-thread results.
__global__ void __launch_bounds__(256) k_msm_reduce(const ge_ext *__restrict__ buckets, uint32_t nb, ge_ext *__restrict__ window_sums, const uint32_t *__restrict__ gate) {
    __shared__ ge_ext sm[8];
    if (MSM_SKIP(gate)) return;
    size_t seg = blockIdx.x;
    const ge_ext *B = buckets + seg * nb;
    uint32_t nthreads = blockDim.x, tid = threadIdx.x, lane = tid & 31, wid = tid >> 5, nwarps = nthreads >> 5;
    uint32_t L = (nb + nthreads - 1) / nthreads;
    uint32_t lo = min(tid * L, nb), hi = min(lo + L, nb);
    // 1. chunk sum
    ge_ext S = ge_identity();
    for (uint32_t j = lo; j < hi; j++) S = ge_add(S, ld_ext(B + j));
    // 2. inclusive suffix scan across the block
    ge_ext suf = S;
#pragma unroll 1
    for (int d = 1; d < 32; d <<= 1) { ge_ext o = shfl_down_ext(suf, d); if (lane + d < 32) suf = ge_add(suf, o); }
    if (lane == 0) sm[wid] = suf;               // total of this warp
    __syncthreads();
    ge_ext above = ge_identity();               // total of the warps holding higher buckets
#pragma unroll 1
    for (uint32_t k = wid + 1; k < nwarps; k++) above = ge_add(above, sm[k]);
    // exclusive suffix: everything strictly above this thread's chunk
    ge_ext next = shfl_down_ext(suf, 1);
    ge_ext run = lane == 31 ? above : ge_add(next, above);
    // 3. running-sum pass over the chunk, top bucket first
    ge_ext acc = ge_identity();
    for (uint32_t j = hi; j > lo; j--) { run = ge_add(run, ld_ext(B + j - 1)); acc = ge_add(acc, run); }
    // 4. block sum of acc
#pragma unroll 1
    for (int d = 16; d >= 1; d >>= 1) { ge_ext o = shfl_down_ext(acc, d); acc = ge_add(acc, o); }
    __syncthreads();
    if (lane == 0) sm[wid] = acc;
    __syncthreads();
    if (tid == 0) { ge_ext r = sm[0]; for (uint32_t k = 1; k < nwarps; k++) r = ge_add(r, sm[k]); st_ext(window_sums + seg, r); }
}
// pass 6: window combination (Horner with c doublings per window), one thread per MSM
__global__ void k_msm_combine(const ge_ext *__restrict__ window_sums, uint32_t n_msm, int c, int W, ge_ext *__restrict__ results, const uint32_t *__restrict__ gate) {
    if (MSM_SKIP(gate)) return;
    uint32_t m = blockIdx.x * blockDim.x + threadIdx.x;
    if (m >= n_msm) return;
    const ge_ext *R = window_sums + (size_t)m * W;
    ge_ext acc = ld_ext(R + W - 1);
#pragma unroll 1
    for (int w = W - 2; w >= 0; w--) {
#pragma unroll 1
        for (int i = 0; i < c; i++) acc = ge_dbl(acc);
        acc = ge_add(acc, ld_ext(R + w));
    }
    st_ext(results + m, acc);
}

// pass 6, latency-optimised form for few MSMs: four lanes per MSM, lane q holds coordinate q of the running point
// (X, Y, Z, T).  A doubling is then one squaring and one multiplication deep (the four squarings and the four products
// of the HWCD formulas run on the four lanes) plus two shuffle rounds, instead of eight field operations in sequence;
// the 253-doubling Horner chain is the longest dependency chain of a verified batch.
__device__ __forceinline__ fe shfl_fe4(const fe &v, int src) {
    fe r;
#pragma unroll
    for (int i = 0; i < 8; i++) r.v[i] = __shfl_sync(0xffffffffu, v.v[i], src, 4);
    return r;
}
__device__ __forceinline__ fe sel_fe(bool pick_b, const fe &a, const fe &b) { return fe_select(a, b, pick_b); }
__global__ void __launch_bounds__(32) k_msm_combine4(const ge_ext *__restrict__ window_sums, uint32_t n_msm, int c, int W, ge_ext *__restrict__ results, const uint32_t *__restrict__ gate) {
    if (MSM_SKIP(gate)) return;
    uint32_t lane = threadIdx.x & 31, q = lane & 3;
    uint32_t m = blockIdx.x * 8 + (lane >> 2);
    bool active = m < n_msm;
    const ge_ext *R = window_sums + (size_t)(active ? m : n_msm - 1) * W;       // idle groups shadow the last MSM (shuffles need every lane)
    const fe d2 = fe_const_d2();
    fe cur = ld_fe(&R[W - 1].X + q);
#pragma unroll 1
    for (int w = W - 2; w >= 0; w--) {
#pragma unroll 1
        for (int i = 0; i < c; i++) {
            // doubling: A = X^2, B = Y^2, ZZ = Z^2, D = (X+Y)^2 on lanes 0..3
            fe x = shfl_fe4(cur, 0), y = shfl_fe4(cur, 1);
            fe sq = fe_sq(sel_fe(q == 3, cur, fe_add(x, y)));
            fe A = shfl_fe4(sq, 0), B = shfl_fe4(sq, 1), ZZ = shfl_fe4(sq, 2), D = shfl_fe4(sq, 3);
            fe H = fe_add(A, B), E = fe_sub(D, H), G = fe_sub(B, A), F = fe_sub(G, fe_dbl(ZZ)), Hn = fe_neg(H);
            // X3 = E F, Y3 = G Hn, Z3 = F G, T3 = E Hn
            fe o1 = sel_fe(q == 1, sel_fe(q == 2, E, F), G), o2 = sel_fe(q == 0, sel_fe(q == 2, Hn, G), F);
            cur = fe_mul(o1, o2);
        }
        // addition of the window sum (extended, from memory): lanes compute (Y1-X1)(Y2-X2), (Y1+X1)(Y2+X2), Z1 Z2, T1 (2d T2)
        const ge_ext *P2 = R + w;
        fe X2 = ld_fe(&P2->X), Y2 = ld_fe(&P2->Y), Z2 = ld_fe(&P2->Z), T2d = fe_mul(ld_fe(&P2->T), d2);
        fe x1 = shfl_fe4(cur, 0), y1 = shfl_fe4(cur, 1);
        fe a = sel_fe(q >= 2, sel_fe(q == 1, fe_sub(y1, x1), fe_add(y1, x1)), cur);
        fe b = sel_fe(q == 1, sel_fe(q == 2, sel_fe(q == 3, fe_sub(Y2, X2), T2d), Z2), fe_add(Y2, X2));
        fe pr = fe_mul(a, b);
        fe A = shfl_fe4(pr, 0), B = shfl_fe4(pr, 1), Dh = shfl_fe4(pr, 2), C = shfl_fe4(pr, 3);
        fe D = fe_dbl(Dh), E = fe_sub(B, A), F = fe_sub(D, C), G = fe_add(D, C), H = fe_add(B, A);
        // X3 = E F, Y3 = G H, Z3 = F G, T3 = E H
        fe o1 = sel_fe(q == 1, sel_fe(q == 2, E, F), G), o2 = sel_fe(q == 0, sel_fe(q == 2, H, G), F);
        cur = fe_mul(o1, o2);
    }
    if (active) st_fe(&results[m].X + q, cur);
}

// ------------------------------------------------------------------ K4: inner-product prover without generator folding
// InnerProductProof::create (inner_product_proof.rs:69-185) folds G and H every round (N two-term scalar multiplications in total).
// The device session never folds points: after rounds with challenges u_1..u_j the folded generator at position i is the combination
//   G^(j)[i] = sum over original indices idx = i (mod n_j) of cG[idx] G[idx],   cG[idx] = G_factors[idx] * prod_r u_r^(+-1)
// (sign by the index bit the round consumed; H likewise with the signs swapped), so L_j and R_j are MSMs of N + 1 terms over the
// ORIGINAL resident points with scalars a_L[pos - h] * cG[idx] etc.; a round costs O(N) scalar products and one MSM launch chain.
// a, b are kept in Montgomery form, the coefficient vectors cG, cH in plain form, so that every product needed as an MSM scalar comes
// out of one Montgomery multiplication as a canonical value.  B proofs of the same length run side by side.
struct ippx_geom { uint32_t N, B, n; };        // N = original length, n = current length (power of two), B proofs
__global__ void __launch_bounds__(128) k_ippx_init(ippx_geom g, const uint8_t *__restrict__ a_in, const uint8_t *__restrict__ b_in, const uint8_t *__restrict__ Gf, const uint8_t *__restrict__ Hf,
                                                   sc *__restrict__ a, sc *__restrict__ b, sc *__restrict__ cG, sc *__restrict__ cH) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)g.B * g.N) return;
    a[i] = sc_to_mont(sc_load(a_in + 32 * i)); b[i] = sc_to_mont(sc_load(b_in + 32 * i));
    sc one = sc_zero(); one.v[0] = 1;
    cG[i] = Gf ? sc_load(Gf + 32 * i) : one; cH[i] = Hf ? sc_load(Hf + 32 * i) : one;
}
// c_L = <a_L, b_R>, c_R = <a_R, b_L> (inner_product_proof.rs:84-85,150-151): block (proof, which), canonical bytes into slot N of the proof's L / R scalar row
__global__ void __launch_bounds__(128) k_ippx_inner(ippx_geom g, const sc *__restrict__ a, const sc *__restrict__ b, uint8_t *__restrict__ scal) {
    __shared__ sc sm[4];
    const uint32_t p = blockIdx.x >> 1, which = blockIdx.x & 1, h = g.n >> 1;
    const sc *x = a + (size_t)p * g.N + (which ? h : 0), *y = b + (size_t)p * g.N + (which ? 0 : h);
    sc acc = sc_zero();
    for (uint32_t i0 = threadIdx.x * 16; i0 < h; i0 += blockDim.x * 16) {      // 16 products per lazy reduction
        sc_wide w = sc_wide_zero();
        for (uint32_t i = i0; i < min(i0 + 16, h); i++) sc_wide_mac(w, x[i], y[i]);
        acc = sc_add(acc, sc_wide_redc(w));
    }
    for (int d = 16; d >= 1; d >>= 1) { sc o; for (int i = 0; i < 8; i++) o.v[i] = __shfl_down_sync(0xffffffffu, acc.v[i], d); acc = sc_add(acc, o); }
    if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        for (uint32_t k = 1; k < (blockDim.x >> 5); k++) acc = sc_add(acc, sm[k]);
        uint8_t bytes[32]; sc_store(bytes, sc_from_mont(acc)); st32(scal + (((size_t)p * 2 + which) * (g.N + 1) + g.N) * 32, bytes);
    }
}
// MSM rows of the round: per proof an L row and an R row of N + 1 (scalar, point index) pairs.  gidx/hidx = table slots of the original G / H
// points, Q = dynamic point p.
__global__ void __launch_bounds__(128) k_ippx_rows(ippx_geom g, const sc *__restrict__ a, const sc *__restrict__ b, const sc *__restrict__ cG, const sc *__restrict__ cH,
                                                   const uint32_t *__restrict__ gidx, const uint32_t *__restrict__ hidx, uint8_t *__restrict__ scal, uint32_t *__restrict__ pidx) {
    size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (size_t)g.B * g.N) return;
    const uint32_t p = (uint32_t)(t / g.N), idx = (uint32_t)(t % g.N), h = g.n >> 1, pos = idx & (g.n - 1), blk = idx / g.n;
    const sc *ap = a + (size_t)p * g.N, *bp_ = b + (size_t)p * g.N;
    const size_t rowL = ((size_t)p * 2) * (g.N + 1), rowR = rowL + g.N + 1;
    uint8_t bytes[32];
    // G[idx]: right half -> L with a_L, left half -> R with a_R (inner_product_proof.rs:87-99,101-113)
    { bool right = pos >= h; uint32_t i = right ? pos - h : pos;
      sc v = sc_mont_mul(right ? ap[i] : ap[h + i], cG[t]);
      size_t slot = (right ? rowL : rowR) + blk * h + i;
      sc_store(bytes, v); st32(scal + slot * 32, bytes); pidx[slot] = gidx[idx]; }
    // H[idx]: left half -> L with b_R, right half -> R with b_L
    { bool left = pos < h; uint32_t i = left ? pos : pos - h;
      sc v = sc_mont_mul(left ? bp_[h + i] : bp_[i], cH[t]);
      size_t slot = (left ? rowL : rowR) + (g.N >> 1) + blk * h + i;
      sc_store(bytes, v); st32(scal + slot * 32, bytes); pidx[slot] = hidx[idx]; }
    if (idx == 0) { pidx[rowL + g.N] = BP_POINT_DYNAMIC | p; pidx[rowR + g.N] = BP_POINT_DYNAMIC | p; }
}
// apply the round's challenge: a' = a_L u + u^-1 a_R, b' = b_L u^-1 + u b_R (:125-126,175-176); cG *= u^-1 (left) / u (right), cH *= u / u^-1 (:127-134,177-178)
__global__ void __launch_bounds__(128) k_ippx_fold(ippx_geom g, const uint8_t *__restrict__ u_bytes, const uint8_t *__restrict__ uinv_bytes, sc *__restrict__ a, sc *__restrict__ b,
                                                   sc *__restrict__ cG, sc *__restrict__ cH) {
    size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (size_t)g.B * g.N) return;
    const uint32_t p = (uint32_t)(t / g.N), idx = (uint32_t)(t % g.N), h = g.n >> 1, pos = idx & (g.n - 1);
    const sc u = sc_to_mont(sc_load(u_bytes + 32 * p)), ui = sc_to_mont(sc_load(uinv_bytes + 32 * p));
    cG[t] = sc_mont_mul(cG[t], pos < h ? ui : u);
    cH[t] = sc_mont_mul(cH[t], pos < h ? u : ui);
    if (idx < h) {
        sc *ap = a + (size_t)p * g.N, *bp_ = b + (size_t)p * g.N;
        ap[idx] = sc_add(sc_mont_mul(ap[idx], u), sc_mont_mul(ui, ap[h + idx]));
        bp_[idx] = sc_add(sc_mont_mul(bp_[idx], ui), sc_mont_mul(u, bp_[h + idx]));
    }
}
__global__ void k_ippx_final(ippx_geom g, const sc *__restrict__ a, const sc *__restrict__ b, uint8_t *__restrict__ out) {
    uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= g.B) return;
    uint8_t bytes[32];
    sc_store(bytes, sc_from_mont(a[(size_t)p * g.N])); st32(out + 64 * p, bytes);
    sc_store(bytes, sc_from_mont(b[(size_t)p * g.N])); st32(out + 64 * p + 32, bytes);
}

// ------------------------------------------------------------------ range-proof batch verification kernels
// One launch group verifies `nbatch` independent batches of `count` proofs each; the per-proof kernels run over all nbatch*count
// proofs.  The group is checked first with ONE random-linear-combination MSM over the group scalar array
//     [S static (summed over every proof of the group) | D dynamic of proof 0 | ... | D dynamic of proof nbatch*count-1]
// (proof p = b*count + q; its dynamic scalars start at S + p*D).  When that combination lies in the identity coset every batch's
// own combination would too, and every batch is accepted.  Otherwise the per-batch pass runs: each batch's own MSM of
// T = S + count*D terms over rows [S static of batch b | the batch's count*D dynamic scalars], and its own accept flag.
// With nbatch == 1 the group array is the batch's row and there is no second pass.  (rp_geom: rp.cuh)

// generator-table slot of static term t of a row: B_blinding, B, then G(n, m) and H(n, m) in iterator order (generators.rs:207-259)
__device__ __forceinline__ uint32_t rp_static_slot(const rp_geom &g, uint32_t t, uint32_t gens_cap, uint32_t gens_parties) {
    if (t < 2) return t;
    const uint32_t which = t - 2 < g.N ? 0u : 1u, q = t - 2 - which * g.N;
    return (uint32_t)bp_gens_slot(which, q / g.n, q % g.n, gens_cap, gens_parties);
}

// Per-call parameter block, uploaded through a pinned staging ring; kernels read the input addresses from it so that the
// launch sequence itself is the same for every call on a reserved geometry (captured once as a CUDA graph).
struct rp_params {
    uint8_t tstate[208];                       // serialized transcript (BP_TRANSCRIPT_BYTES used)
    uint8_t seed[32];                          // external randomness of the batching weights
    const uint8_t *proofs, *commitments;       // device addresses: nbatch*count proofs / nbatch*count*m commitments
    uint32_t *verdict;                         // device address: nbatch*count verdict codes
    // device address of proof 0's caller state and the byte stride between proofs (rp_transcript_proof): the block's own tstate with
    // stride 0, or one BP_TRANSCRIPT_BYTES record per proof in proof order
    const uint8_t *tstates;
    uint64_t tstride;
    // proofs [0, live) are verified; the launch's slots from live on are inert: no decompression, replay or head, zero scalars and chunk
    // sums, no verdict.  count*nbatch on the fixed-geometry path; a reserved mixed class's fill on each call (its launches span the capacity)
    uint32_t live;
    uint8_t pad_[512 - 208 - 32 - 24 - 16 - 4];
};
static_assert(sizeof(rp_params) == 512, "parameter block");

__device__ __forceinline__ uint32_t rp_eff_status(uint32_t st, uint32_t dec_bad) {          // an undecodable point is a VerificationError (mod.rs:445)
    return st != BP_PROOF_OK ? st : (dec_bad ? (uint32_t)BP_PROOF_VERIFICATION_ERROR : (uint32_t)BP_PROOF_OK);
}

// K6: transcript replay (pure hashing).  One thread per proof (32 proofs per warp, every lane busy) replays the geometry's step program
// (rp_transcript_sched) with the Keccak state in registers; the step loads are warp-uniform, and so is every branch on a position when
// the proofs share one caller state.  Proofs with their own states may sit at different positions, and their lanes then diverge where
// a header crosses the rate.  The proof bytes are read straight from global memory a word at a time.
#define RP_TR_THREADS 32
__global__ void __launch_bounds__(RP_TR_THREADS) k_rp_transcript(const rp_params *__restrict__ par, rp_geom g, uint32_t total, const rp_tr_step *__restrict__ prog,
                                                                   uint32_t nsteps, uint8_t *__restrict__ raw, uint32_t *__restrict__ status) {
    uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= min(total, par->live)) return;
    const uint8_t *proof = par->proofs + (size_t)p * g.proof_len, *V = par->commitments + (size_t)p * g.m * 32;
    status[p] = rp_transcript_proof(raw + (size_t)p * (RP_RAW_U + g.k) * 64, proof, g.k, V, par->tstates, par->tstride, p, par->seed, prog, nsteps);
}
// Lean head: ONE thread per proof runs the sequential statement (rp_head_lean) -- ~8k+50 dependent Montgomery products -- and writes the
// proof's tables, its dynamic MSM scalars (group array slots S + p*D ..) and the few sums k_rp_scalars_sum needs.  Several groups are in
// flight, so a head's latency is hidden; what counts is its footprint (registers x time), taken from the MSM kernels beside it.  One
// instance per k = lg(n m) (rp_head_kernel), so that the index-group sizes and the table offsets are constants.
#define RP_HEAD_MIN_K 3         // n >= 8
template <uint32_t K>
__global__ void __launch_bounds__(32) k_rp_head_seq(const rp_params *__restrict__ par, rp_geom g, const uint8_t *__restrict__ raw, uint32_t total,
                                                    rp_lean_head *__restrict__ heads, sc *__restrict__ tabs, const sc *__restrict__ pow2, uint32_t *__restrict__ status,
                                                    uint8_t *__restrict__ scal) {
    uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= min(total, par->live)) return;
    uint32_t st = status[p];
    if (st == BP_PROOF_OK) {
        st = rp_head_lean(heads[p], tabs + (size_t)p * rp_tab_size(K, g.m), scal + (g.S + (size_t)p * g.D) * 32, pow2, raw + (size_t)p * (RP_RAW_U + K) * 64,
                          par->proofs + (size_t)p * g.proof_len, K, g.n, g.m);
        if (st != BP_PROOF_OK) status[p] = st;                  // zero challenge: see rp_reduce_challenges
    }
    heads[p].status = st;
}
typedef decltype(&k_rp_head_seq<RP_HEAD_MIN_K>) rp_head_fn;
template <uint32_t... I> static rp_head_fn rp_head_pick(uint32_t k, std::integer_sequence<uint32_t, I...>) {
    static const rp_head_fn fns[] = {&k_rp_head_seq<RP_HEAD_MIN_K + I>...};
    return fns[k - RP_HEAD_MIN_K];
}
// the instance for k in [RP_HEAD_MIN_K, BP_MAX_LG_N] (rp_param_verdict admits no other)
static rp_head_fn rp_head_kernel(uint32_t k) { return rp_head_pick(k, std::make_integer_sequence<uint32_t, BP_MAX_LG_N - RP_HEAD_MIN_K + 1>()); }
// K5 (combined check): verification scalars with the sum over the proofs taken in registers.  Block = (chunk of RP_CHUNK proofs of one
// batch); thread = generator index i: it walks the chunk's proofs and adds up their weighted g_i and h_i (three Montgomery products
// per proof and index), so no count x S per-proof array is written; k_rp_static_sum then adds the few per-chunk partial sums.  The
// head wrote each proof's per-proof ("dynamic") scalars into the MSM scalar array; this kernel, the first to see both the head's
// status and k_rp_decompress's dec_bad, zeroes those of the chunk's proofs that failed either, and those of inert proofs (index >= *live,
// whose head never ran: a chunk of them sums to zero).  The reject path launches it on a geometry with count = 1 to get each proof's own
// static-term scalars (one proof per block), with live = nullptr (every proof live).
__global__ void __launch_bounds__(128) k_rp_scalars_sum(rp_geom g, const rp_lean_head *__restrict__ heads, const sc *__restrict__ tabs, const uint32_t *__restrict__ dec_bad,
                                                        const uint32_t *__restrict__ live, sc *__restrict__ part, uint8_t *__restrict__ scal) {
    __shared__ uint32_t okmask;
    const uint32_t nchunks = (g.count + RP_CHUNK - 1) / RP_CHUNK, b = blockIdx.x / nchunks, ch = blockIdx.x % nchunks;
    const uint32_t q0 = ch * RP_CHUNK, nq = min((uint32_t)RP_CHUNK, g.count - q0), p0 = b * g.count + q0;
    const uint32_t nlive = live ? min(nq, *live > p0 ? *live - p0 : 0u) : nq;
    if (threadIdx.x < 32) {
        bool ok = threadIdx.x < nlive && heads[p0 + threadIdx.x].status == BP_PROOF_OK && !dec_bad[p0 + threadIdx.x];
        uint32_t m_ = __ballot_sync(0xffffffffu, ok);
        if (threadIdx.x == 0) okmask = m_;
    }
    __syncthreads();
    const uint32_t mask = okmask, tsz = rp_tab_size(g.k, g.m);
    sc *mine = part + ((size_t)b * nchunks + ch) * g.S;
    // weighted g_i = -zL - A_hi[hi] s_lo[lo],  h_i = zL + P_hi[hi] P_lo[lo] - Q_hi[hi] Q_lo[lo]  (rp_scalars_gh): the three products of the
    // chunk's proofs are summed as 512-bit integers and reduced once per chunk (RP_CHUNK <= 32 products fit), one third of the multiplies
    const uint32_t kl = rp_kl(g.k), TL = 1u << kl;
    for (uint32_t i = threadIdx.x; i < g.N; i += blockDim.x) {
        const uint32_t lo = i & (TL - 1), hi = i >> kl;
        sc zsum = sc_zero();
        sc_wide accA = sc_wide_zero(), accP = sc_wide_zero(), accQ = sc_wide_zero();
        for (uint32_t q = 0; q < nq; q++) {
            if (!((mask >> q) & 1u)) continue;
            rp_tabs T = rp_tab_ptrs(const_cast<sc *>(tabs) + (size_t)(p0 + q) * tsz, g.k);
            zsum = sc_add(zsum, heads[p0 + q].zL);
            sc_wide_mac(accA, T.A_hi[hi], T.s_lo[lo]); sc_wide_mac(accP, T.P_hi[hi], T.P_lo[lo]); sc_wide_mac(accQ, T.Q_hi[hi], T.Q_lo[lo]);
        }
        mine[2 + i] = sc_sub(sc_neg(zsum), sc_wide_redc(accA));
        mine[2 + g.N + i] = sc_sub(sc_add(zsum, sc_wide_redc(accP)), sc_wide_redc(accQ));
    }
    if (threadIdx.x < 2) {
        sc s0 = sc_zero();
        for (uint32_t q = 0; q < nq; q++) if ((mask >> q) & 1u) s0 = sc_add(s0, threadIdx.x == 0 ? heads[p0 + q].blinding_scalar : heads[p0 + q].basepoint_scalar);
        mine[threadIdx.x] = s0;
    }
    if (mask == (nq == 32 ? 0xffffffffu : (1u << nq) - 1u)) return;
    for (uint32_t e = threadIdx.x; e < nq * g.D; e += blockDim.x) {         // a proof that failed or does not decode gets zero scalars
        if ((mask >> (e / g.D)) & 1u) continue;
        uint4 *o = reinterpret_cast<uint4 *>(scal + (g.S + (size_t)p0 * g.D + e) * 32);
        o[0] = make_uint4(0, 0, 0, 0); o[1] = make_uint4(0, 0, 0, 0);
    }
}
// add the per-chunk partial sums of the static-term scalars: one warp per (static term, row).  Rows b < nbatch are the batches'
// own static rows (bstatic, b*S + s); with nbatch > 1 the extra row b = nbatch sums every chunk of every batch into the group
// array's static row (scal, s).  With nbatch == 1 the batch's row is the group row (grid.y = 1).
__global__ void __launch_bounds__(32) k_rp_static_sum(const sc *__restrict__ part, rp_geom g, uint8_t *__restrict__ scal, uint8_t *__restrict__ bstatic) {
    const uint32_t nchunks = (g.count + RP_CHUNK - 1) / RP_CHUNK, s = blockIdx.x, b = blockIdx.y;
    const bool grp = b == g.nbatch;
    const uint32_t c0 = grp ? 0u : b * nchunks, nc = grp ? g.nbatch * nchunks : nchunks;
    sc acc = sc_zero();
    for (uint32_t c = threadIdx.x; c < nc; c += 32) acc = sc_add(acc, part[((size_t)c0 + c) * g.S + s]);
    for (int d = 16; d >= 1; d >>= 1) {
        sc o; for (int i = 0; i < 8; i++) o.v[i] = __shfl_down_sync(0xffffffffu, acc.v[i], d);
        acc = sc_add(acc, o);
    }
    if (threadIdx.x == 0) {
        uint8_t bytes[32]; sc_store(bytes, sc_from_mont(acc));
        st32(grp || g.nbatch == 1 ? scal + (size_t)s * 32 : bstatic + ((size_t)b * g.S + s) * 32, bytes);
    }
}
// per-batch pass: gather the rows [S static of batch b | the batch's count*D dynamic scalars] (nbatch x T terms) out of the
// per-batch static rows and the group array
__global__ void __launch_bounds__(256) k_rp_batch_rows(const uint32_t *__restrict__ run, const uint8_t *__restrict__ bstatic, const uint8_t *__restrict__ scal, rp_geom g,
                                                       uint8_t *__restrict__ out) {
    if (run && !*run) return;
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)g.nbatch * g.T) return;
    uint32_t b = (uint32_t)(i / g.T), t = (uint32_t)(i % g.T);
    const uint8_t *src = t < g.S ? bstatic + ((size_t)b * g.S + t) * 32 : scal + (g.S + (size_t)b * g.count * g.D + (t - g.S)) * 32;
    const uint4 *s4 = reinterpret_cast<const uint4 *>(src); uint4 *o4 = reinterpret_cast<uint4 *>(out + 32 * i);
    o4[0] = __ldg(s4); o4[1] = __ldg(s4 + 1);
}
// decompress the per-proof points in MSM order A,S,T_1,T_2,L..,R..,V.. straight out of the proof bytes; independent of the
// transcript, so it runs beside k_rp_transcript / k_rp_head_seq (second branch of the launch graph).  The proofs a block's 128 points
// come from and the commitments of its own V points are contiguous (rp_dec_block, rp.cuh): they are staged with two TMA bulk copies into
// rp_dec_smem_bytes(g) of dynamic shared memory, at most RP_DEC_THREADS commitments whatever m is; the encodings are read from there.
__global__ void __launch_bounds__(RP_DEC_THREADS, 5) k_rp_decompress(const rp_params *__restrict__ par, rp_geom g, uint32_t total,
                                                                  ge_niels *__restrict__ out, uint32_t *__restrict__ dec_bad) {
    extern __shared__ __align__(128) uint8_t dec_smem[];
    __shared__ __align__(8) uint64_t bar;
    total = min(total, par->live);
    const size_t i0 = (size_t)blockIdx.x * blockDim.x, i = i0 + threadIdx.x, n_pts = (size_t)total * g.D;
    if (i0 >= n_pts) return;                    // a block of inert proofs only
    const rp_dec_stage st = rp_dec_block(g, total, i0);
    tma_stage_two(dec_smem, par->proofs + (size_t)st.pf * g.proof_len, st.np * g.proof_len, dec_smem + rp_dec_proof_bytes(g), par->commitments + st.c0 * 32,
                  st.nc * 32, &bar);
    if (i >= n_pts) return;
    uint8_t s[32]; lds32(s, dec_smem + rp_dec_offset(g, st, i));
    fe x, y; bool valid = ge_decode(x, y, s);
    st_niels(out + i, valid ? ge_to_niels_affine(x, y) : ge_niels_identity());
    if (!valid) dec_bad[i / g.D] = 1u;
}
// reject path: one combined MSM per chunk of `chunk` proofs out of the `count` re-checked proofs.  Rows are [S static | chunk*D dynamic]:
// the chunk's summed static-term scalars (part: S Montgomery scalars per chunk) and its proofs' dynamic scalars (dyn: from the first
// re-checked proof, whose points start at dynamic index dyn_base).  The tail of a short last chunk is padded with zero scalars (a zero
// scalar never touches its point).
__global__ void k_rp_chunk_rows(const sc *__restrict__ part, const uint8_t *__restrict__ dyn, rp_geom g, uint32_t count, uint32_t chunk, uint32_t gens_cap,
                                uint32_t gens_parties, uint32_t dyn_base, uint8_t *__restrict__ out_scalars, uint32_t *__restrict__ out_pidx) {
    const uint32_t nchunks = (count + chunk - 1) / chunk, row = g.S + chunk * g.D;
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)nchunks * row) return;
    uint32_t ch = (uint32_t)(i / row), t = (uint32_t)(i % row);
    uint8_t b[32]; uint32_t v;
    if (t < g.S) {
        sc_store(b, sc_from_mont(part[(size_t)ch * g.S + t]));
        v = rp_static_slot(g, t, gens_cap, gens_parties);
    } else {
        uint32_t e = t - g.S, q = ch * chunk + e / g.D;
        if (q < count) { ld32(b, dyn + ((size_t)q * g.D + e % g.D) * 32); v = BP_POINT_DYNAMIC | (dyn_base + q * g.D + e % g.D); }
        else { for (int j = 0; j < 32; j++) b[j] = 0; v = 0; }
    }
    st32(out_scalars + 32 * i, b); out_pidx[i] = v;
}
// reject path: verdicts of the `count` re-checked proofs (arrays point at the first one) from one MSM result per chunk of `chunk` proofs;
// chunk_ok[ch] = identity flags.  Only the proofs of passing chunks are written.  When the reject path starts, rp_verdict_rows has
// already given every well-formed proof of the failing batch VERIFICATION_ERROR and every other proof its own code, which is what a
// proof of a failing chunk keeps unless a finer re-check passes it.
__global__ void k_rp_verdict_chunks(const uint32_t *__restrict__ status, const uint32_t *__restrict__ dec_bad, const ge_ext *__restrict__ results, uint32_t count,
                                    uint32_t chunk, uint32_t *__restrict__ verdict, uint32_t *__restrict__ chunk_ok) {
    uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= count) return;
    uint32_t ch = q / chunk;
    bool ok = ge_is_identity(ld_ext(results + ch));
    if (q % chunk == 0) chunk_ok[ch] = ok ? 1u : 0u;
    if (ok) verdict[q] = rp_eff_status(status[q], dec_bad[q]);
}
// verdicts and flags of batch b once its combined check is decided (ok = the combination lies in the identity coset, mod.rs:447): every
// well-formed proof inherits that result, malformed ones keep their own code; batch_ok[b] = all accepted.  Block-wide; s_all = 1 on entry.
__device__ __forceinline__ void rp_verdict_rows(uint32_t b, uint32_t ok, const uint32_t *__restrict__ status, const uint32_t *__restrict__ dec_bad, const rp_geom &g,
                                                const rp_params *__restrict__ par, uint32_t *__restrict__ batch_ok, uint32_t *__restrict__ combined_ok, uint32_t *s_all) {
    uint32_t all = 1u;
    uint32_t *verdict = par->verdict;
    const uint32_t p_end = min(b * g.count + g.count, par->live);          // inert proofs get no verdict
    for (uint32_t q = threadIdx.x; b * g.count + q < p_end; q += blockDim.x) {
        uint32_t p = b * g.count + q;
        uint32_t st = rp_eff_status(status[p], dec_bad[p]);
        uint32_t v = st != BP_PROOF_OK ? st : (ok ? (uint32_t)BP_PROOF_OK : (uint32_t)BP_PROOF_VERIFICATION_ERROR);
        verdict[p] = v;
        if (v != BP_PROOF_OK) all = 0u;
    }
    if (!all) atomicExch(s_all, 0u);
    __syncthreads();
    if (threadIdx.x == 0) { batch_ok[b] = *s_all; combined_ok[b] = ok; }       // combined_ok = 0: the per-proof recheck has to find the offenders
}
// final verdicts of the per-batch pass, one block per batch (gated like the MSM passes: nothing to do when *run == 0)
__global__ void __launch_bounds__(256) k_rp_verdict_batch(const uint32_t *__restrict__ status, const uint32_t *__restrict__ dec_bad, const ge_ext *__restrict__ results,
                                                          rp_geom g, const rp_params *__restrict__ par, uint32_t *__restrict__ batch_ok, uint32_t *__restrict__ combined_ok,
                                                          const uint32_t *__restrict__ run) {
    __shared__ uint32_t s_ok, s_all;
    if (run && !*run) return;
    uint32_t b = blockIdx.x;
    if (threadIdx.x == 0) { s_ok = ge_is_identity(ld_ext(results + b)) ? 1u : 0u; s_all = 1u; }
    __syncthreads();
    rp_verdict_rows(b, s_ok, status, dec_bad, g, par, batch_ok, combined_ok, &s_all);
}
// verdict of the group check, one block per batch.  In the identity coset: every batch is accepted exactly as its own check would
// accept it (the verdicts and flags k_rp_verdict_batch would write), *run = 0.  Otherwise, with nbatch > 1: *run = 1 and nothing else
// is written (the per-batch pass decides); with nbatch == 1 the group check is the batch's check and its failure is final.
// set_cond: also hand the decision to the IF node of the captured graph that holds the per-batch pass.
__global__ void __launch_bounds__(256) k_rp_verdict_group(const uint32_t *__restrict__ status, const uint32_t *__restrict__ dec_bad, const ge_ext *__restrict__ result,
                                                          rp_geom g, const rp_params *__restrict__ par, uint32_t *__restrict__ batch_ok, uint32_t *__restrict__ combined_ok,
                                                          uint32_t *__restrict__ run, cudaGraphConditionalHandle cond, int set_cond) {
    __shared__ uint32_t s_ok, s_all;
    if (threadIdx.x == 0) { s_ok = ge_is_identity(ld_ext(result)) ? 1u : 0u; s_all = 1u; }
    __syncthreads();
    const uint32_t ok = s_ok, need_batches = !ok && g.nbatch > 1 ? 1u : 0u;
    if (blockIdx.x == 0 && threadIdx.x == 0) { *run = need_batches; if (set_cond) cudaGraphSetConditional(cond, need_batches); }
    if (need_batches) return;
    rp_verdict_rows(blockIdx.x, ok, status, dec_bad, g, par, batch_ok, combined_ok, &s_all);
}
