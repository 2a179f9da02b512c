// C ABI of the engine (include/bpmsm.h): context, scratch arenas, kernel orchestration.
// No CPU fallback: every entry point needs a usable CUDA device and fails with BP_ERR_CUDA otherwise.
#include <cuda_runtime.h>
#include <sys/random.h>
#include <cstdio>
#include <cstdlib>
#include <algorithm>
#include <cstring>
#include <string>
#include <vector>
#include "../../include/bpmsm.h"
#include "kernels.cuh"

static_assert(BP_TRANSCRIPT_BYTES == 203, "transcript wire size");

namespace {

struct DevBuf {
    void *p = nullptr; size_t cap = 0;
    cudaError_t ensure(size_t bytes) {
        if (bytes <= cap) return cudaSuccess;
        if (p) cudaFree(p);
        p = nullptr; cap = 0;
        size_t want = bytes + bytes / 4 + 256;
        cudaError_t e = cudaMalloc(&p, want);
        if (e == cudaSuccess) cap = want;
        return e;
    }
    void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
    template <class T> T *as() const { return reinterpret_cast<T *>(p); }
};

enum KernelId { KID_DECOMPRESS, KID_COMPRESS, KID_FROM_UNIFORM, KID_MSM_COUNT, KID_MSM_SCAN, KID_MSM_SCATTER, KID_MSM_ACCUMULATE, KID_MSM_REDUCE,
                KID_MSM_COMBINE, KID_RP_TRANSCRIPT, KID_RP_HEAD, KID_RP_SCALARS, KID_RP_DECOMPRESS, KID_RP_STATIC_REDUCE, KID_RP_VERDICT_GROUP, KID_RP_BATCH_ROWS,
                KID_RP_VERDICT_BATCH, KID_IPP_FOLD, KID_SMALL, KID_COUNT };
const char *const KERNEL_NAMES[KID_COUNT] = {"k_decompress", "k_compress", "k_from_uniform", "k_msm_count", "k_msm_scan", "k_msm_scatter", "k_msm_accumulate",
                                             "k_msm_reduce", "k_msm_combine", "k_rp_transcript", "k_rp_head", "k_rp_scalars_sum", "k_rp_decompress", "k_rp_static_reduce",
                                             "k_rp_verdict_group", "k_rp_batch_rows", "k_rp_verdict_batch", "k_ipp_fold", "small_kernels"};
struct ProfRec { int kid; cudaEvent_t a, b; };

struct VerifyState {          // what bp_rangeproof_verify_*begin leaves for *_finish
    bool active = false; rp_geom g{}; uint32_t total = 0, n_batches = 1; bp_gens *gens = nullptr; uint8_t param_verdict = 0;
    std::vector<uint8_t> param_codes;       // rejected parameters: every proof's verdict, decided on the host in *_begin
};
struct MsmArena { DevBuf counts, starts, cursor, order, sorted, buckets, wsums; };      // scratch of one Pippenger pipeline pass
struct MsmPlan { int c = 0, W = 0; uint32_t nb = 0, heavy_min = 0; size_t segs = 0, n_buckets = 0, heavy_cap = 0; uint32_t n_msm = 0, T = 0; };

}  // namespace

#define BP_MAX_GROUP_BATCHES 256

struct bp_ctx {
    int device = 0, sm_count = 132; cudaStream_t stream = nullptr; bool own_stream = false;
    cudaStream_t aux = nullptr; cudaEvent_t ev_fork = nullptr, ev_join = nullptr;    // second branch of the verifier's launch graph
    std::string err; uint64_t launches = 0;
    int msm_window = 0;                                       // 0 = by size (msm_pick_window); bp_ctx_set_msm_window pins it (tuning / tests)
    bool prof_on = false; std::vector<ProfRec> prof;          // per-kernel CUDA-event timing (bp_prof_*)
    // MSM scratch
    DevBuf in_scalars, in_points, in_offsets, niels, ok, msm_err, results, outs, flags, ix_pidx;
    MsmArena ar_gen;          // bp_msm*, indexed MSMs, IPP rounds, the verifier's reject path
    // range-proof scratch.  Everything the verifier's launch graph touches is private to it (rp_*, ar_rp): no other entry point can
    // regrow -- i.e. move -- a buffer whose address is baked into the captured graph.
    MsmArena ar_rp;
    DevBuf rp_niels, rp_results;
    DevBuf rp_chal, rp_raw, rp_tabs, pow2_tab, rp_proofs, rp_commit, rp_par, rp_part, rp_scalars, rp_status, rp_decbad, rp_pidx, rp_offsets, rp_verdict, rp_batch_ok, rp_combined;
    DevBuf rp_run, rp_bstatic, rp_bscal, rp_bpidx, rp_boffsets;     // launch groups: per-batch pass gate, static rows, scalar rows, point map, offsets
    cudaStream_t cap_body = nullptr;                                // captures the body of the verifier graph's conditional per-batch pass
    DevBuf fb_part, fb_scalars, fb_pidx, fb_offsets;                 // reject path: one-proof static sums, chunk rows, point map, offsets
    uint32_t *h_verdict = nullptr; size_t h_verdict_cap = 0;       // pinned
    uint32_t *h_flag = nullptr;                                      // pinned: combined_ok[BP_MAX_GROUP_BATCHES] | batch_ok[BP_MAX_GROUP_BATCHES]
    // pinned staging ring for the per-call parameter block of the verifier: a slot is reused only after the upload queued from it has
    // completed, so back-to-back device-path calls on one context never see each other's parameters
    static const int STAGE_SLOTS = 8;
    uint8_t *h_stage = nullptr; cudaEvent_t stage_ev[STAGE_SLOTS] = {}; unsigned stage_next = 0;
    VerifyState vs;
    size_t pidx_key[6] = {0, 0, 0, 0, 0, 0};                        // geometry the cached rp_pidx / rp_offsets were built for
    // reserved geometry: every arena sized, launch sequence captured as a CUDA graph
    cudaGraphExec_t graph = nullptr; size_t graph_key[6] = {0, 0, 0, 0, 0, 0}; uint64_t graph_launches = 0, graph_sig = 0;
};

struct bp_gens {
    bp_ctx *ctx = nullptr; size_t cap = 0, parties = 0, n_points = 0;
    ge_niels *d_table = nullptr;       // [B_blinding, B, G[party][i].., H[party][i]..]
};

namespace {

#define CK(ctx, call)                                                                                  \
    do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { (ctx)->err = std::string(#call) + ": " + cudaGetErrorString(e_); return BP_ERR_CUDA; } } while (0)
#define LAUNCH_CHECK(ctx)                                                                              \
    do { (ctx)->launches++; cudaError_t e_ = cudaGetLastError(); if (e_ != cudaSuccess) { (ctx)->err = std::string("kernel launch: ") + cudaGetErrorString(e_); return BP_ERR_CUDA; } } while (0)

// launch wrapper: counts the launch and, when profiling is enabled, brackets it with CUDA events on the launching stream
#define LAUNCH(ctx, kid, ...)                                                                          \
    do {                                                                                               \
        ProfRec pr_{(kid), nullptr, nullptr};                                                          \
        if ((ctx)->prof_on) { cudaEventCreate(&pr_.a); cudaEventCreate(&pr_.b); cudaEventRecord(pr_.a, (ctx)->stream); } \
        __VA_ARGS__;                                                                                   \
        if ((ctx)->prof_on) { cudaEventRecord(pr_.b, (ctx)->stream); (ctx)->prof.push_back(pr_); }     \
        LAUNCH_CHECK(ctx);                                                                             \
    } while (0)

// the fallback of a pending begin/finish verification reads the context's scratch arenas: other entry points must not run in between
#define BUSY_CHECK(c) do { if ((c)->vs.active) { (c)->err = "a range-proof verification is pending on this context: call bp_rangeproof_verify_group_finish first"; return BP_ERR_INVALID_ARGUMENT; } } while (0)

inline unsigned blocks_for(size_t n, unsigned threads) { return (unsigned)((n + threads - 1) / threads); }

// ---------------------------------------------------------------- host Keccak (SHAKE256 / SHA3-512) for the generator chain
struct HostSponge {
    uint64_t st[25]; unsigned rate, pos; uint8_t pad; bool squeezing;
    HostSponge(unsigned r, uint8_t p) : rate(r), pos(0), pad(p), squeezing(false) { memset(st, 0, sizeof st); }
    void xor_byte(unsigned i, uint8_t b) { st[i >> 3] ^= (uint64_t)b << (8 * (i & 7)); }
    uint8_t get_byte(unsigned i) const { return (uint8_t)(st[i >> 3] >> (8 * (i & 7))); }
    void absorb(const uint8_t *d, size_t n) { for (size_t i = 0; i < n; i++) { xor_byte(pos++, d[i]); if (pos == rate) { keccak_f1600(st); pos = 0; } } }
    void squeeze(uint8_t *o, size_t n) {
        if (!squeezing) { xor_byte(pos, pad); xor_byte(rate - 1, 0x80); keccak_f1600(st); pos = 0; squeezing = true; }
        for (size_t i = 0; i < n; i++) { if (pos == rate) { keccak_f1600(st); pos = 0; } o[i] = get_byte(pos++); }
    }
};

// ---------------------------------------------------------------- the Pippenger pipeline
struct MsmArgs {
    const uint8_t *d_scalars; const uint32_t *d_offsets; uint32_t n_msm, T;
    const uint32_t *d_point_idx; const ge_niels *d_static, *d_dynamic; uint32_t *d_err; int window;
    const uint32_t *run = nullptr;          // optional device gate: every pass returns at once when *run == 0 (see MSM_SKIP)
};

MsmPlan msm_make_plan(uint32_t T, uint32_t n_msm, int window) {
    MsmPlan p; p.T = T; p.n_msm = n_msm;
    size_t avg = msm_avg_terms(T, n_msm);
    p.c = window > 0 ? window : msm_pick_window(avg);
    p.W = msm_num_windows(p.c);
    p.nb = 1u << (p.c - 1);
    p.segs = (size_t)n_msm * p.W; p.n_buckets = p.segs * p.nb;
    // a heavy bucket holds >= heavy_min entries, so at most T*W/heavy_min of them exist
    p.heavy_min = msm_heavy_min(avg, p.nb);
    p.heavy_cap = std::min<size_t>(p.n_buckets, (size_t)T * p.W / p.heavy_min + 1);
    return p;
}
// arenas of one pipeline pass (grow-only; no CUDA call when they are already large enough, which is what lets a reserved
// geometry run under stream capture)
int msm_ensure(bp_ctx *ctx, MsmArena &ar, const MsmPlan &p) {
    // counts | size histogram | bin cursors share one allocation so a single memset clears them
    CK(ctx, ar.counts.ensure((p.n_buckets + 2 * MSM_SIZE_BINS + 4) * 4)); CK(ctx, ar.starts.ensure(p.n_buckets * 4)); CK(ctx, ar.cursor.ensure(p.n_buckets * 4));
    CK(ctx, ar.order.ensure((p.n_buckets + p.heavy_cap) * 4));
    CK(ctx, ar.sorted.ensure((size_t)p.T * p.W * 4)); CK(ctx, ar.buckets.ensure(p.n_buckets * sizeof(ge_ext))); CK(ctx, ar.wsums.ensure(p.segs * sizeof(ge_ext)));
    return BP_OK;
}
int msm_launch(bp_ctx *ctx, MsmArena &ar, const MsmArgs &a, const MsmPlan &p, ge_ext *d_results) {
    const int c = p.c, W = p.W; const uint32_t nb = p.nb, heavy_min = p.heavy_min; const size_t segs = p.segs, n_buckets = p.n_buckets;
    uint32_t *size_hist = ar.counts.as<uint32_t>() + n_buckets, *bin_cursor = size_hist + MSM_SIZE_BINS, *heavy_n = bin_cursor + MSM_SIZE_BINS;
    uint32_t *heavy = ar.order.as<uint32_t>() + n_buckets;
    cudaStream_t s = ctx->stream;
    CK(ctx, cudaMemsetAsync(ar.counts.p, 0, (n_buckets + 2 * MSM_SIZE_BINS + 4) * 4, s));
    LAUNCH(ctx, KID_MSM_COUNT, k_msm_count<<<blocks_for(a.T, 256), 256, 0, s>>>(a.d_scalars, a.d_offsets, a.n_msm, a.T, c, W, ar.counts.as<uint32_t>(), a.d_err, a.run));
    LAUNCH(ctx, KID_MSM_SCAN, k_msm_scan<<<(unsigned)segs, 256, 0, s>>>(ar.counts.as<uint32_t>(), nb, ar.starts.as<uint32_t>(), ar.cursor.as<uint32_t>(), size_hist, a.run));
    LAUNCH(ctx, KID_MSM_SCAN, k_msm_order<<<blocks_for(n_buckets, 256), 256, 0, s>>>(ar.counts.as<uint32_t>(), n_buckets, size_hist, bin_cursor, ar.order.as<uint32_t>(), heavy_min, heavy_n, heavy, a.run));
    LAUNCH(ctx, KID_MSM_SCATTER, k_msm_scatter<<<blocks_for(a.T, 256), 256, 0, s>>>(a.d_scalars, a.d_offsets, a.n_msm, a.T, c, W, ar.cursor.as<uint32_t>(), ar.sorted.as<uint32_t>(), a.run));
    const int acc_split = msm_acc_split(msm_avg_terms(a.T, a.n_msm), nb, n_buckets);
    const unsigned heavy_blocks = (unsigned)std::min<size_t>(p.heavy_cap, (size_t)ctx->sm_count);
#define ACC_LAUNCH(SP) do { unsigned light_ = blocks_for(n_buckets * SP, MSM_ACC_THREADS); \
        LAUNCH(ctx, KID_MSM_ACCUMULATE, k_msm_accumulate<SP><<<light_ + heavy_blocks, MSM_ACC_THREADS, 0, s>>>(ar.starts.as<uint32_t>(), ar.cursor.as<uint32_t>(), ar.sorted.as<uint32_t>(), \
        a.d_offsets, ar.order.as<uint32_t>(), W, nb, n_buckets, a.d_point_idx, a.d_static, a.d_dynamic, ar.buckets.as<ge_ext>(), heavy_min, light_, heavy_n, heavy, a.run)); } while (0)
    if (acc_split == 2) ACC_LAUNCH(2); else ACC_LAUNCH(1);
#undef ACC_LAUNCH
    // two warps per segment up to 2048 buckets (fewer scan / tree additions per useful bucket addition); eight for the wide windows of
    // large MSMs, where a segment's 16k-32k buckets would otherwise be 256-512 sequential additions per thread
    unsigned rthreads = nb >= 4096 ? 256 : nb >= 64 ? 64 : 32;
    LAUNCH(ctx, KID_MSM_REDUCE, k_msm_reduce<<<(unsigned)segs, rthreads, 0, s>>>(ar.buckets.as<ge_ext>(), nb, ar.wsums.as<ge_ext>(), a.run));
    if (msm_use_combine4(a.n_msm))      // few MSMs: the Horner chain is pure latency -> four cooperating lanes per MSM
        LAUNCH(ctx, KID_MSM_COMBINE, k_msm_combine4<<<blocks_for(a.n_msm, 8), 32, 0, s>>>(ar.wsums.as<ge_ext>(), a.n_msm, c, W, d_results, a.run));
    else
        LAUNCH(ctx, KID_MSM_COMBINE, k_msm_combine<<<blocks_for(a.n_msm, 32), 32, 0, s>>>(ar.wsums.as<ge_ext>(), a.n_msm, c, W, d_results, a.run));
    return BP_OK;
}
int msm_core(bp_ctx *ctx, const MsmArgs &a, ge_ext *d_results) {       // generic arena
    if (a.T == 0) return BP_ERR_INVALID_ARGUMENT;
    MsmPlan p = msm_make_plan(a.T, a.n_msm, a.window > 0 ? a.window : ctx->msm_window);
    int rc = msm_ensure(ctx, ctx->ar_gen, p);
    if (rc) return rc;
    return msm_launch(ctx, ctx->ar_gen, a, p, d_results);
}

__global__ void k_mark_invalid(const uint8_t *ok, const uint32_t *offsets, uint32_t n_msm, uint32_t T, uint32_t *msm_err) {
    uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= T || ok[t]) return;
    atomicOr(msm_err + (n_msm == 1 ? 0u : msm_of_term(offsets, n_msm, t)), 1u);
}
__global__ void k_msm_status(const uint32_t *msm_err, uint32_t n_msm, uint8_t *status) {
    uint32_t m = blockIdx.x * blockDim.x + threadIdx.x;
    if (m >= n_msm) return;
    uint32_t e = msm_err[m];
    status[m] = (e & 2u) ? BP_ERR_NONCANONICAL_SCALAR : (e & 1u) ? BP_ERR_INVALID_POINT : BP_OK;
}
enum RpLayout { RP_BATCH_ROWS, RP_GROUP_ROW };
__global__ void k_rp_point_idx(rp_geom g, uint32_t gens_cap, uint32_t gens_parties, int layout, uint32_t *out) {
    // RP_BATCH_ROWS, per batch: [S static | count*D dynamic] (g.nbatch batches);  RP_GROUP_ROW: [S static | g.nbatch*g.count*D dynamic].
    // Dynamic indices address the decompressed per-proof points: (first proof of the batch + q)*D + d.
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    size_t total = layout == RP_GROUP_ROW ? g.S + (size_t)g.nbatch * g.count * g.D : (size_t)g.nbatch * g.T;
    if (i >= total) return;
    uint32_t t, dyn;
    if (layout == RP_GROUP_ROW) { t = (uint32_t)min(i, (size_t)g.S); dyn = (uint32_t)(i - t); }
    else { uint32_t b = (uint32_t)(i / g.T); t = (uint32_t)(i % g.T); dyn = b * g.count * g.D + (t - g.S); if (t > g.S) t = g.S; }
    out[i] = t < g.S ? rp_static_slot(g, t, gens_cap, gens_parties) : BP_POINT_DYNAMIC | dyn;
}
// decompress to the four extended coordinates (X, Y, Z = 1, T), 4 x 32 canonical bytes per point: the in-memory RistrettoPoint
// a host caller keeps (bp_decompress_batch / bp_compress_batch)
__global__ void __launch_bounds__(128) k_decompress_xyzt(const uint8_t *__restrict__ in, size_t n, uint8_t *__restrict__ out, uint8_t *__restrict__ ok) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint8_t s[32]; ld32(s, in + 32 * i);
    fe x, y; bool valid = ge_decode(x, y, s);
    if (!valid) { x = fe_zero(); y = fe_one(); }
    uint8_t b[32];
    fe_tobytes(b, x); st32(out + 128 * i, b); fe_tobytes(b, y); st32(out + 128 * i + 32, b);
    fe_tobytes(b, fe_one()); st32(out + 128 * i + 64, b); fe_tobytes(b, fe_mul(x, y)); st32(out + 128 * i + 96, b);
    ok[i] = valid ? 1 : 0;
}
__global__ void __launch_bounds__(128) k_compress_xyzt(const uint8_t *__restrict__ in, size_t n, uint8_t *__restrict__ out) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    ge_ext p; uint8_t b[32];
    ld32(b, in + 128 * i); p.X = fe_frombytes_raw(b); ld32(b, in + 128 * i + 32); p.Y = fe_frombytes_raw(b);
    ld32(b, in + 128 * i + 64); p.Z = fe_frombytes_raw(b); ld32(b, in + 128 * i + 96); p.T = fe_frombytes_raw(b);
    uint8_t s[32]; ge_encode(s, p); st32(out + 32 * i, s);
}
// term -> point map of n_msm equal-length MSMs over the same resident point set: term t uses point t mod len
__global__ void k_iota_mod(uint32_t T, uint32_t len, uint32_t *out) {
    uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t < T) out[t] = t % len;
}
__global__ void k_fill_offsets(uint32_t n, uint32_t stride, uint32_t *out) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i <= n) out[i] = i * stride;
}

int lg2_exact(size_t v) { int k = 0; while (((size_t)1 << k) < v) k++; return ((size_t)1 << k) == v ? k : -1; }

}  // namespace

// ================================================================================================ C ABI
extern "C" {

int bp_ctx_create(int device, void *stream, bp_ctx **out) {
    if (!out) return BP_ERR_INVALID_ARGUMENT;
    *out = nullptr;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || device < 0 || device >= ndev) return BP_ERR_CUDA;
    if (cudaSetDevice(device) != cudaSuccess) return BP_ERR_CUDA;
    cudaDeviceProp prop;
    // the library holds sm_90a code only, which loads on compute capability 9.0 (H100) and nothing else
    if (cudaGetDeviceProperties(&prop, device) != cudaSuccess || prop.major != 9 || prop.minor != 0) return BP_ERR_CUDA;
    bp_ctx *c = new bp_ctx();
    c->device = device; c->sm_count = prop.multiProcessorCount > 0 ? prop.multiProcessorCount : 132;
    if (stream) { c->stream = (cudaStream_t)stream; c->own_stream = false; }
    else { if (cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking) != cudaSuccess) { delete c; return BP_ERR_CUDA; } c->own_stream = true; }
    if (cudaMallocHost((void **)&c->h_flag, 2 * BP_MAX_GROUP_BATCHES * 4) != cudaSuccess) { delete c; return BP_ERR_CUDA; }
    if (cudaMallocHost((void **)&c->h_stage, 512 * bp_ctx::STAGE_SLOTS) != cudaSuccess) { cudaFreeHost(c->h_flag); delete c; return BP_ERR_CUDA; }
    for (int i = 0; i < bp_ctx::STAGE_SLOTS; i++) cudaEventCreateWithFlags(&c->stage_ev[i], cudaEventDisableTiming);
    cudaStreamCreateWithFlags(&c->aux, cudaStreamNonBlocking);
    cudaStreamCreateWithFlags(&c->cap_body, cudaStreamNonBlocking);
    // k_rp_decompress stages the proofs its block touches in dynamic shared memory: up to 13 proofs of 32*(9+2*20) + 32*m bytes
    cudaFuncSetAttribute(k_rp_decompress, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024);
    cudaEventCreateWithFlags(&c->ev_fork, cudaEventDisableTiming); cudaEventCreateWithFlags(&c->ev_join, cudaEventDisableTiming);
    *out = c;
    return BP_OK;
}
void bp_ctx_destroy(bp_ctx *c) {
    if (!c) return;
    cudaSetDevice(c->device);
    cudaStreamSynchronize(c->stream);
    if (c->aux) cudaStreamSynchronize(c->aux);
    if (c->graph) cudaGraphExecDestroy(c->graph);
    DevBuf *bufs[] = {&c->in_scalars, &c->in_points, &c->in_offsets, &c->niels, &c->ok, &c->msm_err, &c->results, &c->outs, &c->flags, &c->ix_pidx, &c->rp_niels, &c->rp_results, &c->rp_chal, &c->rp_raw, &c->rp_tabs, &c->pow2_tab, &c->rp_proofs, &c->rp_commit, &c->rp_par, &c->rp_part, &c->rp_scalars,
                      &c->rp_status, &c->rp_decbad, &c->rp_pidx, &c->rp_offsets, &c->rp_verdict, &c->rp_batch_ok, &c->rp_combined, &c->fb_part, &c->fb_scalars, &c->fb_pidx, &c->fb_offsets,
                      &c->rp_run, &c->rp_bstatic, &c->rp_bscal, &c->rp_bpidx, &c->rp_boffsets};
    for (DevBuf *b : bufs) b->release();
    for (MsmArena *ar : {&c->ar_gen, &c->ar_rp}) for (DevBuf *b : {&ar->counts, &ar->starts, &ar->cursor, &ar->order, &ar->sorted, &ar->buckets, &ar->wsums}) b->release();
    if (c->h_verdict) cudaFreeHost(c->h_verdict);
    if (c->h_flag) cudaFreeHost(c->h_flag);
    if (c->h_stage) cudaFreeHost(c->h_stage);
    for (int i = 0; i < bp_ctx::STAGE_SLOTS; i++) if (c->stage_ev[i]) cudaEventDestroy(c->stage_ev[i]);
    if (c->ev_fork) cudaEventDestroy(c->ev_fork);
    if (c->ev_join) cudaEventDestroy(c->ev_join);
    if (c->aux) cudaStreamDestroy(c->aux);
    if (c->cap_body) cudaStreamDestroy(c->cap_body);
    if (c->own_stream) cudaStreamDestroy(c->stream);
    delete c;
}
const char *bp_last_error(const bp_ctx *c) { return c ? c->err.c_str() : "null context"; }
uint64_t bp_ctx_launch_count(const bp_ctx *c) { return c ? c->launches : 0; }
int bp_ctx_set_msm_window(bp_ctx *c, int window_bits) { if (!c || window_bits < 0 || window_bits > 18 || window_bits == 1) return BP_ERR_INVALID_ARGUMENT; c->msm_window = window_bits; return BP_OK; }
int bp_ctx_synchronize(bp_ctx *c) { if (!c) return BP_ERR_INVALID_ARGUMENT; CK(c, cudaSetDevice(c->device)); CK(c, cudaStreamSynchronize(c->stream)); return BP_OK; }

int bp_decompress_check_batch(bp_ctx *c, const uint8_t *points, size_t n, uint8_t *ok) {
    if (!c || !points || !ok) return BP_ERR_INVALID_ARGUMENT;
    BUSY_CHECK(c);
    if (n == 0) return BP_OK;
    CK(c, cudaSetDevice(c->device));
    CK(c, c->in_points.ensure(n * 32)); CK(c, c->niels.ensure(n * sizeof(ge_niels))); CK(c, c->ok.ensure(n));
    CK(c, cudaMemcpyAsync(c->in_points.p, points, n * 32, cudaMemcpyHostToDevice, c->stream));
    LAUNCH(c, KID_DECOMPRESS, k_decompress<<<blocks_for(n, 128), 128, 0, c->stream>>>(c->in_points.as<uint8_t>(), n, c->niels.as<ge_niels>(), c->ok.as<uint8_t>()));
    CK(c, cudaMemcpyAsync(ok, c->ok.p, n, cudaMemcpyDeviceToHost, c->stream));
    CK(c, cudaStreamSynchronize(c->stream));
    return BP_OK;
}

int bp_from_uniform_bytes_batch(bp_ctx *c, const uint8_t *uniform, size_t n, uint8_t *points_out) {
    if (!c || !uniform || !points_out) return BP_ERR_INVALID_ARGUMENT;
    BUSY_CHECK(c);
    if (n == 0) return BP_OK;
    CK(c, cudaSetDevice(c->device));
    CK(c, c->in_points.ensure(n * 64)); CK(c, c->outs.ensure(n * 32));
    CK(c, cudaMemcpyAsync(c->in_points.p, uniform, n * 64, cudaMemcpyHostToDevice, c->stream));
    LAUNCH(c, KID_FROM_UNIFORM, k_from_uniform<<<blocks_for(n, 128), 128, 0, c->stream>>>(c->in_points.as<uint8_t>(), n, nullptr, c->outs.as<uint8_t>()));
    CK(c, cudaMemcpyAsync(points_out, c->outs.p, n * 32, cudaMemcpyDeviceToHost, c->stream));
    CK(c, cudaStreamSynchronize(c->stream));
    return BP_OK;
}

int bp_msm_batch_device(bp_ctx *c, const void *d_scalars, const void *d_points, const void *d_offsets_u32, size_t n_msm, size_t total_terms,
                        void *d_outs, void *d_status) {
    if (!c || !d_scalars || !d_points || !d_offsets_u32 || !d_outs || n_msm == 0) return BP_ERR_INVALID_ARGUMENT;
    if (total_terms == 0 || total_terms >= (1u << 31) || n_msm >= (1u << 31)) return BP_ERR_INVALID_ARGUMENT;
    BUSY_CHECK(c);
    CK(c, cudaSetDevice(c->device));
    uint32_t T = (uint32_t)total_terms, M = (uint32_t)n_msm;
    CK(c, c->niels.ensure((size_t)T * sizeof(ge_niels))); CK(c, c->ok.ensure(T)); CK(c, c->msm_err.ensure((size_t)M * 4)); CK(c, c->results.ensure((size_t)M * sizeof(ge_ext)));
    cudaStream_t s = c->stream;
    CK(c, cudaMemsetAsync(c->msm_err.p, 0, (size_t)M * 4, s));
    LAUNCH(c, KID_DECOMPRESS, k_decompress<<<blocks_for(T, 128), 128, 0, s>>>((const uint8_t *)d_points, T, c->niels.as<ge_niels>(), c->ok.as<uint8_t>()));
    LAUNCH(c, KID_SMALL, k_mark_invalid<<<blocks_for(T, 256), 256, 0, s>>>(c->ok.as<uint8_t>(), (const uint32_t *)d_offsets_u32, M, T, c->msm_err.as<uint32_t>()));
    MsmArgs a{(const uint8_t *)d_scalars, (const uint32_t *)d_offsets_u32, M, T, nullptr, nullptr, c->niels.as<ge_niels>(), c->msm_err.as<uint32_t>(), 0};
    int rc = msm_core(c, a, c->results.as<ge_ext>());
    if (rc) return rc;
    LAUNCH(c, KID_COMPRESS, k_compress<<<blocks_for(M, 128), 128, 0, s>>>(c->results.as<ge_ext>(), M, (uint8_t *)d_outs));
    if (d_status) { LAUNCH(c, KID_SMALL, k_msm_status<<<blocks_for(M, 128), 128, 0, s>>>(c->msm_err.as<uint32_t>(), M, (uint8_t *)d_status)); }
    return BP_OK;
}

int bp_msm_batch(bp_ctx *c, const uint8_t *scalars, const uint8_t *points, const uint64_t *offsets, size_t n_msm, uint8_t *outs, uint8_t *status) {
    if (!c || !offsets || !outs || n_msm == 0) return BP_ERR_INVALID_ARGUMENT;
    size_t T = offsets[n_msm];
    if (offsets[0] != 0 || T >= (1u << 31)) return BP_ERR_INVALID_ARGUMENT;
    for (size_t j = 0; j < n_msm; j++) if (offsets[j + 1] < offsets[j]) return BP_ERR_LENGTH_MISMATCH;
    CK(c, cudaSetDevice(c->device));
    if (T == 0) {                      // every MSM empty: the identity encodes as 32 zero bytes
        memset(outs, 0, 32 * n_msm); if (status) memset(status, 0, n_msm); return BP_OK;
    }
    if (!scalars || !points) return BP_ERR_INVALID_ARGUMENT;
    std::vector<uint32_t> off32(n_msm + 1);
    for (size_t j = 0; j <= n_msm; j++) off32[j] = (uint32_t)offsets[j];
    CK(c, c->in_scalars.ensure(T * 32)); CK(c, c->in_points.ensure(T * 32)); CK(c, c->in_offsets.ensure((n_msm + 1) * 4));
    CK(c, c->outs.ensure(n_msm * 32)); CK(c, c->flags.ensure(n_msm));
    cudaStream_t s = c->stream;
    CK(c, cudaMemcpyAsync(c->in_scalars.p, scalars, T * 32, cudaMemcpyHostToDevice, s));
    CK(c, cudaMemcpyAsync(c->in_points.p, points, T * 32, cudaMemcpyHostToDevice, s));
    CK(c, cudaMemcpyAsync(c->in_offsets.p, off32.data(), (n_msm + 1) * 4, cudaMemcpyHostToDevice, s));
    int rc = bp_msm_batch_device(c, c->in_scalars.p, c->in_points.p, c->in_offsets.p, n_msm, T, c->outs.p, c->flags.p);
    if (rc) return rc;
    std::vector<uint8_t> st(n_msm);
    CK(c, cudaMemcpyAsync(outs, c->outs.p, n_msm * 32, cudaMemcpyDeviceToHost, s));
    CK(c, cudaMemcpyAsync(st.data(), c->flags.p, n_msm, cudaMemcpyDeviceToHost, s));
    CK(c, cudaStreamSynchronize(s));
    if (status) memcpy(status, st.data(), n_msm);
    return BP_OK;
}

int bp_msm(bp_ctx *c, const uint8_t *scalars, const uint8_t *points, size_t n, uint8_t out[32]) {
    uint64_t off[2] = {0, n}; uint8_t st = 0;
    int rc = bp_msm_batch(c, scalars, points, off, 1, out, &st);
    return rc ? rc : st;
}

// ---------------------------------------------------------------------------------------------- point values across the boundary
int bp_decompress_batch(bp_ctx *c, const uint8_t *points, size_t n, uint8_t *xyzt_out, uint8_t *ok) {
    if (!c || !points || !xyzt_out || !ok) return BP_ERR_INVALID_ARGUMENT;
    if (n == 0) return BP_OK;
    BUSY_CHECK(c);
    CK(c, cudaSetDevice(c->device));
    CK(c, c->in_points.ensure(n * 32)); CK(c, c->outs.ensure(n * 128)); CK(c, c->ok.ensure(n));
    CK(c, cudaMemcpyAsync(c->in_points.p, points, n * 32, cudaMemcpyHostToDevice, c->stream));
    LAUNCH(c, KID_DECOMPRESS, k_decompress_xyzt<<<blocks_for(n, 128), 128, 0, c->stream>>>(c->in_points.as<uint8_t>(), n, c->outs.as<uint8_t>(), c->ok.as<uint8_t>()));
    CK(c, cudaMemcpyAsync(xyzt_out, c->outs.p, n * 128, cudaMemcpyDeviceToHost, c->stream));
    CK(c, cudaMemcpyAsync(ok, c->ok.p, n, cudaMemcpyDeviceToHost, c->stream));
    CK(c, cudaStreamSynchronize(c->stream));
    return BP_OK;
}
int bp_compress_batch(bp_ctx *c, const uint8_t *xyzt, size_t n, uint8_t *points_out) {
    if (!c || !xyzt || !points_out) return BP_ERR_INVALID_ARGUMENT;
    if (n == 0) return BP_OK;
    BUSY_CHECK(c);
    CK(c, cudaSetDevice(c->device));
    CK(c, c->in_points.ensure(n * 128)); CK(c, c->outs.ensure(n * 32));
    CK(c, cudaMemcpyAsync(c->in_points.p, xyzt, n * 128, cudaMemcpyHostToDevice, c->stream));
    LAUNCH(c, KID_COMPRESS, k_compress_xyzt<<<blocks_for(n, 128), 128, 0, c->stream>>>(c->in_points.as<uint8_t>(), n, c->outs.as<uint8_t>()));
    CK(c, cudaMemcpyAsync(points_out, c->outs.p, n * 32, cudaMemcpyDeviceToHost, c->stream));
    CK(c, cudaStreamSynchronize(c->stream));
    return BP_OK;
}

// ---------------------------------------------------------------------------------------------- resident point sets (decompressed once, reused by many MSMs)
}  // extern "C"
struct bp_points { bp_ctx *ctx = nullptr; size_t n = 0; ge_niels *d_pts = nullptr; uint32_t *d_idx = nullptr; size_t idx_T = 0, idx_len = 0; };
extern "C" {
static int points_from_device(bp_ctx *c, const uint8_t *d_compressed, size_t n, bp_points **out) {
    bp_points *h = new bp_points(); h->ctx = c; h->n = n;
    cudaError_t e = cudaMalloc((void **)&h->d_pts, n * sizeof(ge_niels));
    if (e != cudaSuccess) { c->err = std::string("cudaMalloc(points): ") + cudaGetErrorString(e); delete h; return BP_ERR_CUDA; }
    int rc = [&]() -> int {
        CK(c, c->ok.ensure(n));
        LAUNCH(c, KID_DECOMPRESS, k_decompress<<<blocks_for(n, 128), 128, 0, c->stream>>>(d_compressed, n, h->d_pts, c->ok.as<uint8_t>()));
        std::vector<uint8_t> ok(n);
        CK(c, cudaMemcpyAsync(ok.data(), c->ok.p, n, cudaMemcpyDeviceToHost, c->stream)); CK(c, cudaStreamSynchronize(c->stream));
        for (uint8_t v : ok) if (!v) return BP_ERR_INVALID_POINT;
        return BP_OK;
    }();
    if (rc) { cudaFree(h->d_pts); delete h; return rc; }
    *out = h; return BP_OK;
}
int bp_points_create(bp_ctx *c, const uint8_t *points, size_t n, bp_points **out) {
    if (!c || !points || !out || n == 0 || n >= (1u << 31)) return BP_ERR_INVALID_ARGUMENT;
    BUSY_CHECK(c);
    CK(c, cudaSetDevice(c->device));
    CK(c, c->in_points.ensure(n * 32));
    CK(c, cudaMemcpyAsync(c->in_points.p, points, n * 32, cudaMemcpyHostToDevice, c->stream));
    return points_from_device(c, c->in_points.as<uint8_t>(), n, out);
}
int bp_points_create_device(bp_ctx *c, const void *d_points, size_t n, bp_points **out) {
    if (!c || !d_points || !out || n == 0 || n >= (1u << 31)) return BP_ERR_INVALID_ARGUMENT;
    BUSY_CHECK(c);
    CK(c, cudaSetDevice(c->device));
    return points_from_device(c, (const uint8_t *)d_points, n, out);
}
void bp_points_destroy(bp_points *h) { if (!h) return; cudaSetDevice(h->ctx->device); cudaStreamSynchronize(h->ctx->stream); cudaFree(h->d_pts); if (h->d_idx) cudaFree(h->d_idx); delete h; }
size_t bp_points_count(const bp_points *h) { return h ? h->n : 0; }

// n_msm MSMs of `terms` terms each over the first `terms` points of the set (MSM j uses scalars[j*terms .. (j+1)*terms)); device pointers,
// nothing synchronised.  No decompression on this path: 32 B of scalar per term is all that is read from the caller.
int bp_msm_points_device(bp_ctx *c, bp_points *h, const void *d_scalars, size_t n_msm, size_t terms, void *d_outs, void *d_status) {
    if (!c || !h || !d_scalars || !d_outs || n_msm == 0 || terms == 0 || terms > h->n || n_msm * terms >= (1u << 31)) return BP_ERR_INVALID_ARGUMENT;
    BUSY_CHECK(c);
    CK(c, cudaSetDevice(c->device));
    uint32_t T = (uint32_t)(n_msm * terms), M = (uint32_t)n_msm;
    cudaStream_t s = c->stream;
    if (h->idx_T < T || h->idx_len != terms) {
        CK(c, cudaStreamSynchronize(s));
        if (h->d_idx) cudaFree(h->d_idx);
        h->d_idx = nullptr; h->idx_T = 0;
        CK(c, cudaMalloc((void **)&h->d_idx, (size_t)T * 4));
        LAUNCH(c, KID_SMALL, k_iota_mod<<<blocks_for(T, 256), 256, 0, s>>>(T, (uint32_t)terms, h->d_idx));
        h->idx_T = T; h->idx_len = terms;
    }
    CK(c, c->in_offsets.ensure(((size_t)M + 1) * 4)); CK(c, c->msm_err.ensure((size_t)M * 4)); CK(c, c->results.ensure((size_t)M * sizeof(ge_ext)));
    LAUNCH(c, KID_SMALL, k_fill_offsets<<<blocks_for((size_t)M + 1, 256), 256, 0, s>>>(M, (uint32_t)terms, c->in_offsets.as<uint32_t>()));
    CK(c, cudaMemsetAsync(c->msm_err.p, 0, (size_t)M * 4, s));
    MsmArgs a{(const uint8_t *)d_scalars, c->in_offsets.as<uint32_t>(), M, T, h->d_idx, h->d_pts, nullptr, c->msm_err.as<uint32_t>(), 0};
    int rc = msm_core(c, a, c->results.as<ge_ext>());
    if (rc) return rc;
    LAUNCH(c, KID_COMPRESS, k_compress<<<blocks_for(M, 128), 128, 0, s>>>(c->results.as<ge_ext>(), M, (uint8_t *)d_outs));
    if (d_status) { LAUNCH(c, KID_SMALL, k_msm_status<<<blocks_for(M, 128), 128, 0, s>>>(c->msm_err.as<uint32_t>(), M, (uint8_t *)d_status)); }
    return BP_OK;
}
// host-buffer form (pinned memory recommended): H2D of the scalars, the MSMs, D2H of the 32-byte results; synchronises
int bp_msm_points(bp_ctx *c, bp_points *h, const uint8_t *scalars, size_t n_msm, size_t terms, uint8_t *outs, uint8_t *status) {
    if (!c || !h || !scalars || !outs || n_msm == 0 || terms == 0) return BP_ERR_INVALID_ARGUMENT;
    BUSY_CHECK(c);
    CK(c, cudaSetDevice(c->device));
    size_t T = n_msm * terms;
    CK(c, c->in_scalars.ensure(T * 32)); CK(c, c->outs.ensure(n_msm * 32)); CK(c, c->flags.ensure(n_msm));
    CK(c, cudaMemcpyAsync(c->in_scalars.p, scalars, T * 32, cudaMemcpyHostToDevice, c->stream));
    int rc = bp_msm_points_device(c, h, c->in_scalars.p, n_msm, terms, c->outs.p, c->flags.p);
    if (rc) return rc;
    std::vector<uint8_t> st(n_msm);
    CK(c, cudaMemcpyAsync(outs, c->outs.p, n_msm * 32, cudaMemcpyDeviceToHost, c->stream));
    CK(c, cudaMemcpyAsync(st.data(), c->flags.p, n_msm, cudaMemcpyDeviceToHost, c->stream));
    CK(c, cudaStreamSynchronize(c->stream));
    if (status) memcpy(status, st.data(), n_msm);
    return BP_OK;
}

// ---------------------------------------------------------------------------------------------- generators
static int gens_alloc(bp_ctx *c, size_t cap, size_t parties, bp_gens **out) {
    if (!c || !out || cap == 0 || parties == 0) return BP_ERR_INVALID_ARGUMENT;
    CK(c, cudaSetDevice(c->device));
    bp_gens *g = new bp_gens();
    g->ctx = c; g->cap = cap; g->parties = parties; g->n_points = 2 + 2 * cap * parties;
    cudaError_t e = cudaMalloc((void **)&g->d_table, g->n_points * sizeof(ge_niels));
    if (e != cudaSuccess) { c->err = std::string("cudaMalloc(gens): ") + cudaGetErrorString(e); delete g; return BP_ERR_CUDA; }
    *out = g;
    return BP_OK;
}
int bp_gens_create_empty(bp_ctx *c, size_t cap, size_t parties, bp_gens **out) { return gens_alloc(c, cap, parties, out); }

int bp_gens_create(bp_ctx *c, size_t cap, size_t parties, bp_gens **out) {
    int rc = gens_alloc(c, cap, parties, out);
    if (rc) return rc;
    bp_gens *g = *out;
    // ristretto255 basepoint, compressed (RISTRETTO_BASEPOINT_COMPRESSED)
    static const uint8_t BASEPOINT[32] = {0xe2, 0xf2, 0xae, 0x0a, 0x6a, 0xbc, 0x4e, 0x71, 0xa8, 0x84, 0xa9, 0x61, 0xc5, 0x00, 0x51, 0x5f,
                                          0x58, 0xe3, 0x0b, 0x6a, 0xa5, 0x82, 0xdd, 0x8d, 0xb6, 0xa6, 0x59, 0x45, 0xe0, 0x8d, 0x2d, 0x76};
    // uniform bytes: slot 0 = SHA3-512(B) for B_blinding (generators.rs:48-51); slot 1 unused (B is decompressed);
    // then the SHAKE256("GeneratorsChain" || tag || LE32(party)) streams (generators.rs:62-104,179-204)
    std::vector<uint8_t> uni(g->n_points * 64, 0);
    { HostSponge h(72, 0x06); h.absorb(BASEPOINT, 32); h.squeeze(uni.data(), 64); }
    for (int which = 0; which < 2; which++)
        for (size_t p = 0; p < parties; p++) {
            HostSponge h(136, 0x1f);
            uint8_t label[5] = {(uint8_t)(which ? 'H' : 'G'), (uint8_t)p, (uint8_t)(p >> 8), (uint8_t)(p >> 16), (uint8_t)(p >> 24)};
            h.absorb((const uint8_t *)"GeneratorsChain", 15); h.absorb(label, 5);
            h.squeeze(uni.data() + 64 * bp_gens_slot(which, p, 0, cap, parties), 64 * cap);
        }
    CK(c, c->in_points.ensure(uni.size())); CK(c, c->in_scalars.ensure(32));
    cudaStream_t s = c->stream;
    CK(c, cudaMemcpyAsync(c->in_points.p, uni.data(), uni.size(), cudaMemcpyHostToDevice, s));
    CK(c, cudaMemcpyAsync(c->in_scalars.p, BASEPOINT, 32, cudaMemcpyHostToDevice, s));
    LAUNCH(c, KID_FROM_UNIFORM, k_from_uniform<<<blocks_for(g->n_points, 128), 128, 0, s>>>(c->in_points.as<uint8_t>(), g->n_points, g->d_table, nullptr));
    LAUNCH(c, KID_DECOMPRESS, k_decompress<<<1, 128, 0, s>>>(c->in_scalars.as<uint8_t>(), 1, g->d_table + 1, nullptr));
    CK(c, cudaStreamSynchronize(s));
    return BP_OK;
}
void bp_gens_destroy(bp_gens *g) { if (!g) return; cudaSetDevice(g->ctx->device); cudaFree(g->d_table); delete g; }
int bp_gens_device_table(bp_gens *g, void **d_table, size_t *bytes) {
    if (!g || !d_table || !bytes) return BP_ERR_INVALID_ARGUMENT;
    *d_table = g->d_table; *bytes = g->n_points * sizeof(ge_niels); return BP_OK;
}
int bp_gens_get(bp_gens *g, int which, size_t party, size_t index, uint8_t out[32]) {
    if (!g || !out) return BP_ERR_INVALID_ARGUMENT;
    bp_ctx *c = g->ctx; size_t slot;
    if (which == 2) slot = 1; else if (which == 3) slot = 0;
    else if ((which == 0 || which == 1) && party < g->parties && index < g->cap) slot = bp_gens_slot(which, party, index, g->cap, g->parties);
    else return BP_ERR_INVALID_ARGUMENT;
    CK(c, cudaSetDevice(c->device)); CK(c, c->outs.ensure(32));
    LAUNCH(c, KID_SMALL, k_niels_to_compressed<<<1, 32, 0, c->stream>>>(g->d_table + slot, 1, c->outs.as<uint8_t>()));
    CK(c, cudaMemcpyAsync(out, c->outs.p, 32, cudaMemcpyDeviceToHost, c->stream));
    CK(c, cudaStreamSynchronize(c->stream));
    return BP_OK;
}
// table slots of BulletproofGens::G(n, m) followed by H(n, m), each in iterator order (generators.rs:207-259): 2*n*m entries
static std::vector<uint32_t> gens_nm_slots(const bp_gens *gens, size_t n, size_t m) {
    const size_t N = n * m;
    std::vector<uint32_t> idx(2 * N);
    for (size_t which = 0; which < 2; which++)
        for (size_t q = 0; q < N; q++) idx[which * N + q] = (uint32_t)bp_gens_slot(which, q / n, q % n, gens->cap, gens->parties);
    return idx;
}

// ---------------------------------------------------------------------------------------------- range proofs
// Parameter checks of verify_multiple_with_rng (mod.rs:358-366) and of from_bytes / verification_scalars
// that depend only on (proof_len, n, m): one verdict for the whole call, or BP_PROOF_OK to go on.
static uint8_t rp_param_verdict(const bp_gens *gens, size_t proof_len, size_t n, size_t m, rp_geom *g) {
    if (proof_len % 32 != 0 || proof_len < 7 * 32) return BP_PROOF_FORMAT_ERROR;                 // mod.rs:498-503
    size_t ne = (proof_len - 7 * 32) / 32;
    if (ne < 2 || (ne - 2) % 2 != 0 || (ne - 2) / 2 >= 32) return BP_PROOF_FORMAT_ERROR;         // inner_product_proof.rs:375-388
    size_t k = (ne - 2) / 2;
    if (!(n == 8 || n == 16 || n == 32 || n == 64)) return BP_PROOF_INVALID_BITSIZE;
    if (gens->cap < n || gens->parties < m) return BP_PROOF_INVALID_GENERATORS_LENGTH;
    if (m == 0 || n * m != ((size_t)1 << k) || k > BP_MAX_LG_N) return BP_PROOF_VERIFICATION_ERROR;   // inner_product_proof.rs:204-211
    g->n = (uint32_t)n; g->m = (uint32_t)m; g->k = (uint32_t)k; g->N = (uint32_t)(n * m);
    g->D = (uint32_t)(4 + 2 * k + m); g->S = 2 + 2 * g->N; g->proof_len = (uint32_t)proof_len;
    return BP_PROOF_OK;
}
// Verdict of one proof of a call whose parameters rp_param_verdict rejected with `pv`.  The reference parses the proof
// (RangeProof::from_bytes, mod.rs:506-524) before it checks the parameters (mod.rs:359-365), so a proof with a non-canonical
// t_x, t_x_blinding, e_blinding, a or b gets FormatError whatever the parameters; a length-level FormatError covers every proof.
// The length passed rp_param_verdict's first checks whenever pv is not FormatError, so the offsets below lie inside the proof.
static uint8_t rp_rejected_proof_verdict(uint8_t pv, const uint8_t *proof, size_t proof_len) {
    if (pv == BP_PROOF_FORMAT_ERROR) return pv;
    const size_t k = (proof_len / 32 - 9) / 2, ab = 224 + 64 * k;
    for (size_t off : {(size_t)128, (size_t)160, (size_t)192, ab, ab + 32})
        if (sc_geq_l(sc_load(proof + off))) return BP_PROOF_FORMAT_ERROR;
    return pv;
}
static bool rp_set_group(rp_geom *g, size_t count, size_t n_batches) {
    if (count == 0 || n_batches == 0 || n_batches > BP_MAX_GROUP_BATCHES || count >= (1u << 24)) return false;
    size_t T = (size_t)g->S + count * g->D;
    if (T * n_batches >= (1u << 31) || count * n_batches >= (1u << 24)) return false;
    g->count = (uint32_t)count; g->nbatch = (uint32_t)n_batches; g->T = (uint32_t)T;
    return true;
}

// terms of a launch group's combined MSM: [S static | nbatch*count*D dynamic] (kernels.cuh, range-proof section)
static uint32_t rp_group_terms(const rp_geom &g) { return g.S + g.nbatch * g.count * g.D; }
// block size of k_rp_scalars_sum: one thread per generator index, at least one warp
static unsigned rp_sum_threads(const rp_geom &g) { return std::min<uint32_t>(128, std::max<uint32_t>(32, g.N)); }
// every arena of one launch group (grow-only); after this nothing on the verification path allocates
static int rp_ensure(bp_ctx *c, const rp_geom &g) {
    size_t total = (size_t)g.count * g.nbatch, TT = (size_t)g.T * g.nbatch, TG = rp_group_terms(g);
    CK(c, c->rp_par.ensure(sizeof(rp_params)));
    CK(c, c->rp_scalars.ensure(TG * 32));
    CK(c, c->rp_part.ensure((size_t)g.nbatch * ((g.count + RP_CHUNK - 1) / RP_CHUNK) * g.S * sizeof(sc)));
    CK(c, c->rp_status.ensure(total * 4)); CK(c, c->rp_decbad.ensure(total * 4)); CK(c, c->rp_niels.ensure(total * g.D * sizeof(ge_niels)));
    CK(c, c->rp_pidx.ensure(TG * 4)); CK(c, c->rp_offsets.ensure(2 * 4)); CK(c, c->rp_results.ensure(((size_t)g.nbatch + 1) * sizeof(ge_ext))); CK(c, c->rp_run.ensure(4));
    CK(c, c->rp_batch_ok.ensure((size_t)g.nbatch * 4)); CK(c, c->rp_combined.ensure((size_t)g.nbatch * 4));
    CK(c, c->rp_chal.ensure(total * sizeof(rp_head))); CK(c, c->rp_tabs.ensure(total * rp_tab_size(g.k, g.m) * sizeof(sc)));
    CK(c, c->rp_raw.ensure(total * (RP_RAW_U + g.k) * 64));
    if (!c->h_verdict || c->h_verdict_cap < total) {
        if (c->h_verdict) cudaFreeHost(c->h_verdict);
        c->h_verdict = nullptr; c->h_verdict_cap = 0;
        CK(c, cudaMallocHost((void **)&c->h_verdict, total * 4));
        c->h_verdict_cap = total;
    }
    if (!c->pow2_tab.p) {            // 2^e (e < 64) in Montgomery form, computed once per context with the host build of sc.cuh
        std::vector<sc> tab(64);
        for (int e = 0; e < 64; e++) tab[e] = sc_mont_from_u64(1ULL << e);
        CK(c, c->pow2_tab.ensure(64 * sizeof(sc)));
        CK(c, cudaMemcpyAsync(c->pow2_tab.p, tab.data(), 64 * sizeof(sc), cudaMemcpyHostToDevice, c->stream)); CK(c, cudaStreamSynchronize(c->stream));
    }
    if (g.nbatch > 1) {       // the per-batch pass; its MSM shares the arena with the group MSM (they run one after the other)
        CK(c, c->rp_bstatic.ensure((size_t)g.nbatch * g.S * 32)); CK(c, c->rp_bscal.ensure(TT * 32)); CK(c, c->rp_bpidx.ensure(TT * 4));
        CK(c, c->rp_boffsets.ensure(((size_t)g.nbatch + 1) * 4));
        int rc = msm_ensure(c, c->ar_rp, msm_make_plan((uint32_t)TT, g.nbatch, 0));
        if (rc) return rc;
    }
    return msm_ensure(c, c->ar_rp, msm_make_plan((uint32_t)TG, 1, 0));
}
// signature of every device address the launch sequence of a group bakes into its graph: a regrown (moved) arena invalidates the graph
static uint64_t rp_ptr_signature(const bp_ctx *c) {
    const DevBuf *bufs[] = {&c->rp_par, &c->rp_part, &c->rp_scalars, &c->rp_status, &c->rp_decbad, &c->rp_niels, &c->rp_pidx, &c->rp_offsets, &c->rp_results, &c->rp_batch_ok, &c->rp_combined,
                            &c->rp_chal, &c->rp_tabs, &c->rp_raw, &c->pow2_tab, &c->rp_run, &c->rp_bstatic, &c->rp_bscal, &c->rp_bpidx, &c->rp_boffsets, &c->ar_rp.counts, &c->ar_rp.starts, &c->ar_rp.cursor, &c->ar_rp.order, &c->ar_rp.sorted, &c->ar_rp.buckets, &c->ar_rp.wsums};
    uint64_t h = 1469598103934665603ULL;
    for (const DevBuf *b : bufs) { h ^= (uint64_t)(uintptr_t)b->p; h *= 1099511628211ULL; }
    return h;
}
// term -> point maps and MSM offsets of the group MSM and of the per-batch MSMs: depend only on the geometry, rebuilt when it changes
static int rp_build_maps(bp_ctx *c, bp_gens *gens, const rp_geom &g) {
    size_t key[6] = {g.n, g.m, g.count, g.nbatch, gens->cap, gens->parties};
    if (memcmp(key, c->pidx_key, sizeof key) == 0) return BP_OK;
    cudaStream_t s = c->stream;
    const uint32_t TG = rp_group_terms(g);
    LAUNCH(c, KID_SMALL, k_rp_point_idx<<<blocks_for(TG, 256), 256, 0, s>>>(g, (uint32_t)gens->cap, (uint32_t)gens->parties, RP_GROUP_ROW, c->rp_pidx.as<uint32_t>()));
    LAUNCH(c, KID_SMALL, k_fill_offsets<<<1, 256, 0, s>>>(1, TG, c->rp_offsets.as<uint32_t>()));
    if (g.nbatch > 1) {
        LAUNCH(c, KID_SMALL, k_rp_point_idx<<<blocks_for((size_t)g.T * g.nbatch, 256), 256, 0, s>>>(g, (uint32_t)gens->cap, (uint32_t)gens->parties, RP_BATCH_ROWS,
                                                                                                    c->rp_bpidx.as<uint32_t>()));
        LAUNCH(c, KID_SMALL, k_fill_offsets<<<blocks_for((size_t)g.nbatch + 1, 256), 256, 0, s>>>(g.nbatch, g.T, c->rp_boffsets.as<uint32_t>()));
    }
    memcpy(c->pidx_key, key, sizeof key);
    return BP_OK;
}
// upload the per-call parameter block through the pinned staging ring, so that the asynchronous upload never reads caller
// memory after the entry point returns
static int rp_upload_params(bp_ctx *c, const uint8_t *h_transcript, const uint8_t *seed, const uint8_t *d_proofs, const uint8_t *d_commit, uint32_t *d_verdict) {
    unsigned slot = c->stage_next++ % bp_ctx::STAGE_SLOTS;
    CK(c, cudaEventSynchronize(c->stage_ev[slot]));                          // the upload that last used this slot is done
    rp_params *par = reinterpret_cast<rp_params *>(c->h_stage + 512 * slot);
    memset(par, 0, sizeof *par);
    memcpy(par->tstate, h_transcript, BP_TRANSCRIPT_BYTES);
    if (seed) memcpy(par->seed, seed, 32);
    else if (getrandom(par->seed, 32, 0) != 32) { c->err = "getrandom failed"; return BP_ERR_CUDA; }
    par->proofs = d_proofs; par->commitments = d_commit; par->verdict = d_verdict;
    CK(c, cudaMemcpyAsync(c->rp_par.p, par, sizeof *par, cudaMemcpyHostToDevice, c->stream));
    CK(c, cudaEventRecord(c->stage_ev[slot], c->stream));
    return BP_OK;
}

// Per-batch pass of a launch group whose combined check failed: every batch's own combined MSM and verdicts, as before the group
// check existed.  run = the device gate k_rp_verdict_group sets (direct launches: every kernel returns at once when the group
// passed), or nullptr inside the body of the captured graph's IF node, which runs only when the group failed.
static int rp_batch_pass(bp_ctx *c, bp_gens *gens, const rp_geom &g, const uint32_t *run) {
    cudaStream_t s = c->stream;
    const uint32_t TT = g.T * g.nbatch;
    LAUNCH(c, KID_RP_BATCH_ROWS, k_rp_batch_rows<<<blocks_for(TT, 256), 256, 0, s>>>(run, c->rp_bstatic.as<uint8_t>(), c->rp_scalars.as<uint8_t>(), g, c->rp_bscal.as<uint8_t>()));
    MsmArgs a{c->rp_bscal.as<uint8_t>(), c->rp_boffsets.as<uint32_t>(), g.nbatch, TT, c->rp_bpidx.as<uint32_t>(), gens->d_table, c->rp_niels.as<ge_niels>(), nullptr, 0, run};
    int rc = msm_launch(c, c->ar_rp, a, msm_make_plan(a.T, a.n_msm, 0), c->rp_results.as<ge_ext>());
    if (rc) return rc;
    LAUNCH(c, KID_RP_VERDICT_BATCH, k_rp_verdict_batch<<<g.nbatch, 256, 0, s>>>(c->rp_status.as<uint32_t>(), c->rp_decbad.as<uint32_t>(), c->rp_results.as<ge_ext>(), g, c->rp_par.as<rp_params>(),
                                                                                 c->rp_batch_ok.as<uint32_t>(), c->rp_combined.as<uint32_t>(), run));
    return BP_OK;
}

// The launch sequence of one group, launches only (no allocation, no synchronisation: capturable).  Two branches: the
// decompressions need nothing but the proof bytes and run beside the transcript replay and the head.  capture: the sequence is
// being captured into the verifier graph, whose per-batch pass goes under a conditional node.
static int rp_chain(bp_ctx *c, bp_gens *gens, const rp_geom &g, bool capture) {
    cudaStream_t s = c->stream, s2 = c->prof_on ? c->stream : c->aux;
    const uint32_t total = g.count * g.nbatch;
    const rp_params *par = c->rp_par.as<rp_params>();
    uint8_t *d_scal = c->rp_scalars.as<uint8_t>();
    if (s2 != s) { CK(c, cudaEventRecord(c->ev_fork, s)); CK(c, cudaStreamWaitEvent(s2, c->ev_fork, 0)); }
    CK(c, cudaMemsetAsync(c->rp_decbad.p, 0, (size_t)total * 4, s2));
    {   // branch 2
        cudaStream_t keep = c->stream; c->stream = s2;          // LAUNCH brackets its events on ctx->stream
        int rc = [&]() -> int {
            const size_t dec_smem = (size_t)(RP_DEC_THREADS / g.D + 2) * (g.proof_len + 32 * g.m);
            LAUNCH(c, KID_RP_DECOMPRESS, k_rp_decompress<<<blocks_for((size_t)total * g.D, RP_DEC_THREADS), RP_DEC_THREADS, dec_smem, s2>>>(par, g, total, c->rp_niels.as<ge_niels>(), c->rp_decbad.as<uint32_t>()));
            return BP_OK;
        }();
        c->stream = keep;
        if (rc) return rc;
    }
    if (s2 != s) CK(c, cudaEventRecord(c->ev_join, s2));
    LAUNCH(c, KID_RP_TRANSCRIPT, k_rp_transcript<<<blocks_for(total, RP_TR_THREADS), RP_TR_THREADS, 0, s>>>(par, g, total, c->rp_raw.as<uint8_t>(), c->rp_status.as<uint32_t>()));
    LAUNCH(c, KID_RP_HEAD, k_rp_head_seq<<<blocks_for(total, 32), 32, 0, s>>>(par, g, c->rp_raw.as<uint8_t>(), total, c->rp_chal.as<rp_head>(), c->rp_tabs.as<sc>(),
                                                                                  c->pow2_tab.as<sc>(), c->rp_status.as<uint32_t>()));
    if (s2 != s) CK(c, cudaStreamWaitEvent(s, c->ev_join, 0));
    const uint32_t nchunks = (g.count + RP_CHUNK - 1) / RP_CHUNK;
    LAUNCH(c, KID_RP_SCALARS, k_rp_scalars_sum<<<g.nbatch * nchunks, rp_sum_threads(g), 0, s>>>(g, c->rp_chal.as<rp_head>(), c->rp_tabs.as<sc>(),
                                                                                  c->rp_decbad.as<uint32_t>(), c->rp_part.as<sc>(), d_scal));
    LAUNCH(c, KID_RP_STATIC_REDUCE, k_rp_static_sum<<<dim3(g.S, g.nbatch > 1 ? g.nbatch + 1 : 1), 32, 0, s>>>(c->rp_part.as<sc>(), g, d_scal, c->rp_bstatic.as<uint8_t>()));
    // the group check: one MSM over every proof of the group (result in slot nbatch; the per-batch MSMs use slots 0..nbatch-1)
    ge_ext *d_group = c->rp_results.as<ge_ext>() + g.nbatch;
    MsmArgs a{d_scal, c->rp_offsets.as<uint32_t>(), 1, rp_group_terms(g), c->rp_pidx.as<uint32_t>(), gens->d_table, c->rp_niels.as<ge_niels>(), nullptr, 0};
    int rc = msm_launch(c, c->ar_rp, a, msm_make_plan(a.T, a.n_msm, 0), d_group);
    if (rc) return rc;
#define VERDICT_GROUP(COND, SET)                                                                                                                   \
    LAUNCH(c, KID_RP_VERDICT_GROUP, k_rp_verdict_group<<<g.nbatch, 256, 0, s>>>(c->rp_status.as<uint32_t>(), c->rp_decbad.as<uint32_t>(), d_group, g, par, \
                                                                                 c->rp_batch_ok.as<uint32_t>(), c->rp_combined.as<uint32_t>(), c->rp_run.as<uint32_t>(), COND, SET))
    if (g.nbatch == 1) { VERDICT_GROUP(0, 0); return BP_OK; }          // the group check is the batch's check
    if (!capture) { VERDICT_GROUP(0, 0); return rp_batch_pass(c, gens, g, c->rp_run.as<uint32_t>()); }
    // captured: the group verdict kernel sets the condition of an IF node whose body is the per-batch pass.  The handle resets to 0 at
    // every launch of the graph, so no call sees the decision of the one before.
    cudaStreamCaptureStatus cs; cudaGraph_t cg = nullptr; const cudaGraphNode_t *deps = nullptr; size_t nd = 0;
    cudaGraphConditionalHandle cond = 0;
    CK(c, cudaStreamGetCaptureInfo(s, &cs, nullptr, &cg, &deps, &nd));
    CK(c, cudaGraphConditionalHandleCreate(&cond, cg, 0, cudaGraphCondAssignDefault));
    VERDICT_GROUP(cond, 1);
#undef VERDICT_GROUP
    CK(c, cudaStreamGetCaptureInfo(s, &cs, nullptr, &cg, &deps, &nd));
    cudaGraphNodeParams np{};
    np.type = cudaGraphNodeTypeConditional; np.conditional.handle = cond; np.conditional.type = cudaGraphCondTypeIf; np.conditional.size = 1;
    cudaGraphNode_t node = nullptr;
    CK(c, cudaGraphAddNode(&node, cg, deps, nd, &np));
    CK(c, cudaStreamUpdateCaptureDependencies(s, &node, 1, cudaStreamSetCaptureDependencies));
    CK(c, cudaStreamBeginCaptureToGraph(c->cap_body, np.conditional.phGraph_out[0], nullptr, nullptr, 0, cudaStreamCaptureModeThreadLocal));
    c->stream = c->cap_body;                 // LAUNCH and msm_launch queue on ctx->stream
    rc = rp_batch_pass(c, gens, g, nullptr);
    c->stream = s;
    cudaGraph_t body = nullptr;
    cudaError_t e = cudaStreamEndCapture(c->cap_body, &body);
    if (rc) return rc;
    if (e != cudaSuccess) { c->err = std::string("cudaStreamEndCapture(per-batch pass): ") + cudaGetErrorString(e); return BP_ERR_CUDA; }
    return BP_OK;
}

static bool rp_graph_matches(const bp_ctx *c, const bp_gens *gens, const rp_geom &g) {
    size_t key[6] = {g.n, g.m, g.count, g.nbatch, (size_t)(uintptr_t)gens->d_table, g.proof_len};      // the table address is a kernel argument of the captured nodes
    return c->graph && memcmp(key, c->graph_key, sizeof key) == 0 && c->graph_sig == rp_ptr_signature(c);
}
// queue everything up to the verdicts; d_proofs / d_commitments are device pointers
static int rp_verify_queue(bp_ctx *c, bp_gens *gens, const rp_geom &g, const uint8_t *d_proofs, const uint8_t *d_commit,
                           const uint8_t *h_transcript, const uint8_t *seed, uint32_t *d_verdict) {
    const bool use_graph = !c->prof_on && rp_graph_matches(c, gens, g);
    if (!use_graph) { int rc = rp_ensure(c, g); if (rc) return rc; }
    int rc = rp_build_maps(c, gens, g);          // another geometry may have used the context since: the maps follow the key
    if (rc) return rc;
    rc = rp_upload_params(c, h_transcript, seed, d_proofs, d_commit, d_verdict);
    if (rc) return rc;
    if (use_graph) { CK(c, cudaGraphLaunch(c->graph, c->stream)); c->launches += c->graph_launches; return BP_OK; }
    return rp_chain(c, gens, g, false);
}

// Re-check of the proofs [p0, p0 + count) of a group in chunks of `chunk` proofs: one MSM per chunk over the row [S static | chunk*D
// dynamic], with part = the chunks' summed static-term scalars (Montgomery form, S per chunk).  Writes the verdicts of the proofs in
// passing chunks; chunk_ok (optional) receives the per-chunk pass flags, which synchronises.
static int rp_recheck(bp_ctx *c, bp_gens *gens, const rp_geom &g, const sc *part, uint32_t p0, uint32_t count, uint32_t chunk, uint32_t *d_verdict,
                      std::vector<uint32_t> *chunk_ok) {
    cudaStream_t s = c->stream;
    const uint32_t nch = (count + chunk - 1) / chunk, row = g.S + chunk * g.D;
    size_t T = (size_t)nch * row;
    if (T >= (1u << 31)) { c->err = "fallback batch too large"; return BP_ERR_INVALID_ARGUMENT; }
    CK(c, c->fb_scalars.ensure(T * 32)); CK(c, c->fb_pidx.ensure(T * 4)); CK(c, c->fb_offsets.ensure(((size_t)nch + 1) * 4));
    CK(c, c->results.ensure((size_t)nch * sizeof(ge_ext))); CK(c, c->flags.ensure((size_t)nch * 4));
    LAUNCH(c, KID_SMALL, k_rp_chunk_rows<<<blocks_for(T, 128), 128, 0, s>>>(part, c->rp_scalars.as<uint8_t>() + (g.S + (size_t)p0 * g.D) * 32, g, count, chunk,
                                                                              (uint32_t)gens->cap, (uint32_t)gens->parties, p0 * g.D, c->fb_scalars.as<uint8_t>(), c->fb_pidx.as<uint32_t>()));
    LAUNCH(c, KID_SMALL, k_fill_offsets<<<blocks_for((size_t)nch + 1, 256), 256, 0, s>>>(nch, row, c->fb_offsets.as<uint32_t>()));
    MsmArgs a{c->fb_scalars.as<uint8_t>(), c->fb_offsets.as<uint32_t>(), nch, (uint32_t)T, c->fb_pidx.as<uint32_t>(), gens->d_table, c->rp_niels.as<ge_niels>(), nullptr, 0};
    int rc = msm_core(c, a, c->results.as<ge_ext>());
    if (rc) return rc;
    LAUNCH(c, KID_SMALL, k_rp_verdict_chunks<<<blocks_for(count, 128), 128, 0, s>>>(c->rp_status.as<uint32_t>() + p0, c->rp_decbad.as<uint32_t>() + p0, c->results.as<ge_ext>(), count, chunk,
                                                                                    d_verdict + p0, c->flags.as<uint32_t>()));
    if (!chunk_ok) return BP_OK;
    chunk_ok->resize(nch);
    CK(c, cudaMemcpyAsync(chunk_ok->data(), c->flags.p, (size_t)nch * 4, cudaMemcpyDeviceToHost, s)); CK(c, cudaStreamSynchronize(s));
    return BP_OK;
}
// the proofs [p0, p0 + count) one by one (mod.rs:421-447 per proof): k_rp_scalars_sum on a geometry of one-proof batches gives each
// proof's own static-term scalars (and rewrites its dynamic scalars with the bytes the main pass wrote), then a re-check with chunk = 1
static int rp_recheck_proofs(bp_ctx *c, bp_gens *gens, const rp_geom &g, uint32_t p0, uint32_t count, uint32_t *d_verdict) {
    CK(c, c->fb_part.ensure((size_t)count * g.S * sizeof(sc)));
    rp_geom one = g; one.count = 1; one.nbatch = count;
    LAUNCH(c, KID_RP_SCALARS, k_rp_scalars_sum<<<count, rp_sum_threads(g), 0, c->stream>>>(one, c->rp_chal.as<rp_head>() + p0, c->rp_tabs.as<sc>() + (size_t)p0 * rp_tab_size(g.k, g.m),
                                                                                          c->rp_decbad.as<uint32_t>() + p0, c->fb_part.as<sc>(), c->rp_scalars.as<uint8_t>() + (size_t)p0 * g.D * 32));
    return rp_recheck(c, gens, g, c->fb_part.as<sc>(), p0, count, 1, d_verdict, nullptr);
}
// A batch whose combined check failed.  Level 1: one combined MSM per chunk of RP_CHUNK proofs, from the partial sums the main path
// already holds (one pipeline pass over the batch's ~T terms).  Level 2: the proofs of the failing chunks, each with its own MSM.
// One bad proof in 1024 costs two small passes instead of 1024 147-term MSMs.
static int rp_verify_fallback(bp_ctx *c, bp_gens *gens, const rp_geom &g, uint32_t batch, uint32_t *d_verdict) {
    const uint32_t nch = (g.count + RP_CHUNK - 1) / RP_CHUNK, p0 = batch * g.count;
    std::vector<uint32_t> ok;
    int rc = rp_recheck(c, gens, g, c->rp_part.as<sc>() + (size_t)batch * nch * g.S, p0, g.count, RP_CHUNK, d_verdict, &ok);
    if (rc) return rc;
    uint32_t nfail = 0; for (uint32_t v : ok) nfail += v ? 0 : 1;
    if (nfail == 0) return BP_OK;       // cannot happen when the batch's combination failed, short of a 2^-128 cancellation between chunk weights
    if (rp_recheck_whole_batch(nfail)) return rp_recheck_proofs(c, gens, g, p0, g.count, d_verdict);      // many bad chunks: one pass over the whole batch
    for (uint32_t ch = 0; ch < nch; ch++)
        if (!ok[ch]) { rc = rp_recheck_proofs(c, gens, g, p0 + ch * RP_CHUNK, std::min<uint32_t>(RP_CHUNK, g.count - ch * RP_CHUNK), d_verdict); if (rc) return rc; }
    return BP_OK;
}

int bp_rangeproof_verify_reserve(bp_ctx *c, bp_gens *gens, size_t n, size_t m, size_t count, size_t n_batches) {
    if (!c || !gens) return BP_ERR_INVALID_ARGUMENT;
    BUSY_CHECK(c);
    CK(c, cudaSetDevice(c->device));
    size_t k = 0; while (((size_t)1 << k) < n * m) k++;
    rp_geom g{};
    if (rp_param_verdict(gens, 32 * (9 + 2 * k), n, m, &g) != BP_PROOF_OK || !rp_set_group(&g, count, n_batches)) return BP_ERR_INVALID_ARGUMENT;
    CK(c, c->rp_proofs.ensure((size_t)g.count * g.nbatch * g.proof_len)); CK(c, c->rp_commit.ensure((size_t)g.count * g.nbatch * m * 32)); CK(c, c->rp_verdict.ensure((size_t)g.count * g.nbatch * 4));
    int rc = rp_ensure(c, g); if (rc) return rc;
    rc = rp_build_maps(c, gens, g); if (rc) return rc;
    CK(c, cudaStreamSynchronize(c->stream));
    if (c->graph) { cudaGraphExecDestroy(c->graph); c->graph = nullptr; }
    bool prof = c->prof_on; c->prof_on = false;
    uint64_t l0 = c->launches;
    cudaGraph_t graph = nullptr;
    CK(c, cudaStreamBeginCapture(c->stream, cudaStreamCaptureModeThreadLocal));
    rc = rp_chain(c, gens, g, true);
    cudaError_t e = cudaStreamEndCapture(c->stream, &graph);
    c->prof_on = prof;
    c->graph_launches = c->launches - l0; c->launches = l0;
    if (rc) { if (graph) cudaGraphDestroy(graph); return rc; }
    if (e != cudaSuccess) { c->err = std::string("cudaStreamEndCapture: ") + cudaGetErrorString(e); return BP_ERR_CUDA; }
    e = cudaGraphInstantiate(&c->graph, graph, 0);
    cudaGraphDestroy(graph);
    if (e != cudaSuccess) { c->graph = nullptr; c->err = std::string("cudaGraphInstantiate: ") + cudaGetErrorString(e); return BP_ERR_CUDA; }
    size_t key[6] = {g.n, g.m, g.count, g.nbatch, (size_t)(uintptr_t)gens->d_table, g.proof_len};      // the table address is a kernel argument of the captured nodes
    memcpy(c->graph_key, key, sizeof key); c->graph_sig = rp_ptr_signature(c);
    // one untimed pass so that the first real call finds module loading, the graph upload and the L2 working set done
    std::vector<uint8_t> zt(BP_TRANSCRIPT_BYTES, 0);
    CK(c, cudaMemsetAsync(c->rp_proofs.p, 0, (size_t)g.count * g.nbatch * g.proof_len, c->stream)); CK(c, cudaMemsetAsync(c->rp_commit.p, 0, (size_t)g.count * g.nbatch * m * 32, c->stream));
    rc = rp_verify_queue(c, gens, g, c->rp_proofs.as<uint8_t>(), c->rp_commit.as<uint8_t>(), zt.data(), nullptr, c->rp_verdict.as<uint32_t>());
    if (rc) return rc;
    CK(c, cudaStreamSynchronize(c->stream));
    return BP_OK;
}

int bp_rangeproof_verify_group_begin(bp_ctx *c, bp_gens *gens, const uint8_t *transcript, const uint8_t *proofs, size_t proof_len, const uint8_t *commitments,
                                     size_t n, size_t m, size_t count, size_t n_batches, const uint8_t *seed) {
    if (!c || !gens || !transcript || !proofs || !commitments || count == 0 || n_batches == 0) return BP_ERR_INVALID_ARGUMENT;
    if (c->vs.active) { c->err = "verify_begin called twice without verify_finish"; return BP_ERR_INVALID_ARGUMENT; }
    if (count * n_batches >= (1u << 24) || n_batches > BP_MAX_GROUP_BATCHES) return BP_ERR_INVALID_ARGUMENT;
    CK(c, cudaSetDevice(c->device));
    rp_geom g{};
    uint8_t pv = rp_param_verdict(gens, proof_len, n, m, &g);
    VerifyState vs; vs.total = (uint32_t)(count * n_batches); vs.n_batches = (uint32_t)n_batches; vs.gens = gens; vs.param_verdict = pv;
    if (pv != BP_PROOF_OK) {              // no kernel runs: _finish hands out these codes
        vs.param_codes.resize(vs.total);
        for (size_t i = 0; i < vs.total; i++) vs.param_codes[i] = rp_rejected_proof_verdict(pv, proofs + i * proof_len, proof_len);
        vs.active = true; c->vs = std::move(vs); return BP_OK;
    }
    if (!rp_set_group(&g, count, n_batches)) return BP_ERR_INVALID_ARGUMENT;
    vs.g = g;
    size_t total = vs.total;
    CK(c, c->rp_proofs.ensure(total * proof_len)); CK(c, c->rp_commit.ensure(total * m * 32)); CK(c, c->rp_verdict.ensure(total * 4));
    CK(c, cudaMemcpyAsync(c->rp_proofs.p, proofs, total * proof_len, cudaMemcpyHostToDevice, c->stream));
    CK(c, cudaMemcpyAsync(c->rp_commit.p, commitments, total * m * 32, cudaMemcpyHostToDevice, c->stream));
    int rc = rp_verify_queue(c, gens, g, c->rp_proofs.as<uint8_t>(), c->rp_commit.as<uint8_t>(), transcript, seed, c->rp_verdict.as<uint32_t>());
    if (rc) return rc;
    CK(c, cudaMemcpyAsync(c->h_verdict, c->rp_verdict.p, total * 4, cudaMemcpyDeviceToHost, c->stream));
    CK(c, cudaMemcpyAsync(c->h_flag, c->rp_combined.p, (size_t)g.nbatch * 4, cudaMemcpyDeviceToHost, c->stream));
    CK(c, cudaMemcpyAsync(c->h_flag + BP_MAX_GROUP_BATCHES, c->rp_batch_ok.p, (size_t)g.nbatch * 4, cudaMemcpyDeviceToHost, c->stream));
    vs.active = true; c->vs = vs;              // only a fully queued verification is pending
    return BP_OK;
}

int bp_rangeproof_verify_group_finish(bp_ctx *c, uint8_t *verdicts, uint8_t *batch_ok) {
    if (!c || !verdicts || !c->vs.active) return BP_ERR_INVALID_ARGUMENT;
    VerifyState vs = std::move(c->vs); c->vs = VerifyState{};
    if (vs.param_verdict != BP_PROOF_OK) { memcpy(verdicts, vs.param_codes.data(), vs.total); if (batch_ok) memset(batch_ok, 0, vs.n_batches); return BP_OK; }
    CK(c, cudaSetDevice(c->device));
    CK(c, cudaStreamSynchronize(c->stream));
    bool redo = false;
    for (uint32_t b = 0; b < vs.g.nbatch; b++)
        if (c->h_flag[b] == 0) {            // this batch's combined check failed: find the offenders (chunks of 32, then proof by proof)
            int rc = rp_verify_fallback(c, vs.gens, vs.g, b, c->rp_verdict.as<uint32_t>());
            if (rc) return rc;
            redo = true;
        }
    if (redo) {
        CK(c, cudaMemcpyAsync(c->h_verdict, c->rp_verdict.p, (size_t)vs.total * 4, cudaMemcpyDeviceToHost, c->stream));
        CK(c, cudaStreamSynchronize(c->stream));
    }
    for (uint32_t i = 0; i < vs.total; i++) verdicts[i] = (uint8_t)c->h_verdict[i];
    if (batch_ok) for (uint32_t b = 0; b < vs.g.nbatch; b++) batch_ok[b] = (uint8_t)c->h_flag[BP_MAX_GROUP_BATCHES + b];
    return BP_OK;
}

int bp_rangeproof_verify_group_device(bp_ctx *c, bp_gens *gens, const uint8_t *transcript, const void *d_proofs, size_t proof_len, const void *d_commitments,
                                      size_t n, size_t m, size_t count, size_t n_batches, const uint8_t *seed, void *d_verdicts_u32, uint32_t *h_batch_ok_pinned) {
    if (!c || !gens || !transcript || !d_proofs || !d_commitments || !d_verdicts_u32) return BP_ERR_INVALID_ARGUMENT;
    BUSY_CHECK(c);
    CK(c, cudaSetDevice(c->device));
    rp_geom g{};
    uint8_t pv = rp_param_verdict(gens, proof_len, n, m, &g);
    if (pv != BP_PROOF_OK || !rp_set_group(&g, count, n_batches)) return BP_ERR_INVALID_ARGUMENT;
    int rc = rp_verify_queue(c, gens, g, (const uint8_t *)d_proofs, (const uint8_t *)d_commitments, transcript, seed, (uint32_t *)d_verdicts_u32);
    if (rc) return rc;
    if (h_batch_ok_pinned) CK(c, cudaMemcpyAsync(h_batch_ok_pinned, c->rp_batch_ok.p, (size_t)g.nbatch * 4, cudaMemcpyDeviceToHost, c->stream));
    return BP_OK;
}

// single-batch forms
int bp_rangeproof_verify_begin(bp_ctx *c, bp_gens *gens, const uint8_t *transcript, const uint8_t *proofs, size_t proof_len, const uint8_t *commitments,
                               size_t n, size_t m, size_t count, const uint8_t *seed) {
    return bp_rangeproof_verify_group_begin(c, gens, transcript, proofs, proof_len, commitments, n, m, count, 1, seed);
}
int bp_rangeproof_verify_finish(bp_ctx *c, uint8_t *verdicts) { return bp_rangeproof_verify_group_finish(c, verdicts, nullptr); }
int bp_rangeproof_verify_batch(bp_ctx *c, bp_gens *gens, const uint8_t *transcript, const uint8_t *proofs, size_t proof_len, const uint8_t *commitments,
                               size_t n, size_t m, size_t count, const uint8_t *seed, uint8_t *verdicts) {
    int rc = bp_rangeproof_verify_begin(c, gens, transcript, proofs, proof_len, commitments, n, m, count, seed);
    if (rc) return rc;
    return bp_rangeproof_verify_finish(c, verdicts);
}
int bp_rangeproof_verify_batch_device(bp_ctx *c, bp_gens *gens, const uint8_t *transcript, const void *d_proofs, size_t proof_len, const void *d_commitments,
                                      size_t n, size_t m, size_t count, const uint8_t *seed, void *d_verdicts_u32, uint32_t *h_batch_ok_pinned) {
    return bp_rangeproof_verify_group_device(c, gens, transcript, d_proofs, proof_len, d_commitments, n, m, count, 1, seed, d_verdicts_u32, h_batch_ok_pinned);
}

// ---------------------------------------------------------------------------------------------- indexed MSMs and the IPP prover session
static int check_scalars_canonical(const uint8_t *s, size_t n) {
    for (size_t i = 0; i < n; i++) if (sc_geq_l(sc_load(s + 32 * i))) return BP_ERR_NONCANONICAL_SCALAR;
    return BP_OK;
}

int bp_msm_indexed_batch(bp_ctx *c, bp_gens *gens, const uint8_t *scalars, const uint32_t *point_idx, const uint8_t *dyn_points, size_t n_dyn,
                         const uint64_t *offsets, size_t n_msm, uint8_t *outs, uint8_t *status) {
    if (!c || !offsets || !outs || n_msm == 0) return BP_ERR_INVALID_ARGUMENT;
    size_t T = offsets[n_msm];
    if (offsets[0] != 0 || T == 0 || T >= (1u << 31) || !scalars || !point_idx) return BP_ERR_INVALID_ARGUMENT;
    BUSY_CHECK(c);
    CK(c, cudaSetDevice(c->device));
    for (size_t t = 0; t < T; t++) {
        uint32_t v = point_idx[t];
        if (v & BP_POINT_DYNAMIC) { if ((v & 0x7fffffffu) >= n_dyn || !dyn_points) return BP_ERR_INVALID_ARGUMENT; }
        else if (!gens || v >= gens->n_points) return BP_ERR_INVALID_ARGUMENT;
    }
    std::vector<uint32_t> off32(n_msm + 1);
    for (size_t j = 0; j <= n_msm; j++) { if (j && offsets[j] < offsets[j - 1]) return BP_ERR_LENGTH_MISMATCH; off32[j] = (uint32_t)offsets[j]; }
    cudaStream_t s = c->stream;
    uint32_t M = (uint32_t)n_msm;
    CK(c, c->in_scalars.ensure(T * 32)); CK(c, c->in_offsets.ensure((n_msm + 1) * 4)); CK(c, c->ix_pidx.ensure(T * 4));
    CK(c, c->outs.ensure(n_msm * 32)); CK(c, c->flags.ensure(n_msm)); CK(c, c->msm_err.ensure((size_t)M * 4)); CK(c, c->results.ensure((size_t)M * sizeof(ge_ext)));
    CK(c, cudaMemcpyAsync(c->in_scalars.p, scalars, T * 32, cudaMemcpyHostToDevice, s));
    CK(c, cudaMemcpyAsync(c->in_offsets.p, off32.data(), (n_msm + 1) * 4, cudaMemcpyHostToDevice, s));
    CK(c, cudaMemcpyAsync(c->ix_pidx.p, point_idx, T * 4, cudaMemcpyHostToDevice, s));
    CK(c, cudaMemsetAsync(c->msm_err.p, 0, (size_t)M * 4, s));
    std::vector<uint8_t> dyn_ok;
    if (n_dyn) {
        CK(c, c->in_points.ensure(n_dyn * 32)); CK(c, c->niels.ensure(n_dyn * sizeof(ge_niels))); CK(c, c->ok.ensure(n_dyn));
        CK(c, cudaMemcpyAsync(c->in_points.p, dyn_points, n_dyn * 32, cudaMemcpyHostToDevice, s));
        LAUNCH(c, KID_DECOMPRESS, k_decompress<<<blocks_for(n_dyn, 128), 128, 0, s>>>(c->in_points.as<uint8_t>(), n_dyn, c->niels.as<ge_niels>(), c->ok.as<uint8_t>()));
        dyn_ok.resize(n_dyn);
        CK(c, cudaMemcpyAsync(dyn_ok.data(), c->ok.p, n_dyn, cudaMemcpyDeviceToHost, s));
    }
    MsmArgs a{c->in_scalars.as<uint8_t>(), c->in_offsets.as<uint32_t>(), M, (uint32_t)T, c->ix_pidx.as<uint32_t>(), gens ? gens->d_table : nullptr, c->niels.as<ge_niels>(), c->msm_err.as<uint32_t>(), 0};
    int rc = msm_core(c, a, c->results.as<ge_ext>());
    if (rc) return rc;
    LAUNCH(c, KID_COMPRESS, k_compress<<<blocks_for(M, 128), 128, 0, s>>>(c->results.as<ge_ext>(), M, c->outs.as<uint8_t>()));
    LAUNCH(c, KID_SMALL, k_msm_status<<<blocks_for(M, 128), 128, 0, s>>>(c->msm_err.as<uint32_t>(), M, c->flags.as<uint8_t>()));
    std::vector<uint8_t> st(n_msm);
    CK(c, cudaMemcpyAsync(outs, c->outs.p, n_msm * 32, cudaMemcpyDeviceToHost, s));
    CK(c, cudaMemcpyAsync(st.data(), c->flags.p, n_msm, cudaMemcpyDeviceToHost, s));
    CK(c, cudaStreamSynchronize(s));
    // an undecodable caller-supplied point poisons the MSMs that use it (optional_multiscalar_mul -> None)
    if (n_dyn)
        for (size_t j = 0; j < n_msm; j++)
            for (size_t t = offsets[j]; t < offsets[j + 1]; t++)
                if ((point_idx[t] & BP_POINT_DYNAMIC) && !dyn_ok[point_idx[t] & 0x7fffffffu] && st[j] == BP_OK) st[j] = BP_ERR_INVALID_POINT;
    if (status) memcpy(status, st.data(), n_msm);
    return BP_OK;
}

}  // extern "C"

struct bp_ipp {
    bp_ctx *ctx = nullptr; uint32_t N = 0; ge_niels *pts = nullptr;     // [G (N) | H (N) | Q]
    DevBuf scal, idx, offs;
};

extern "C" {

static int ipp_alloc(bp_ctx *c, size_t N, bp_ipp **out) {
    if (!c || !out || N == 0 || (N & (N - 1)) || N >= (1u << 24)) return BP_ERR_INVALID_ARGUMENT;      // power of two (inner_product_proof.rs:67)
    CK(c, cudaSetDevice(c->device));
    bp_ipp *s = new bp_ipp(); s->ctx = c; s->N = (uint32_t)N;
    cudaError_t e = cudaMalloc((void **)&s->pts, (2 * N + 1) * sizeof(ge_niels));
    if (e != cudaSuccess) { c->err = std::string("cudaMalloc(ipp): ") + cudaGetErrorString(e); delete s; return BP_ERR_CUDA; }
    *out = s; return BP_OK;
}
int bp_ipp_begin(bp_ctx *c, bp_gens *gens, size_t n, size_t m, const uint8_t Q[32], bp_ipp **out) {
    if (!gens || !Q || n == 0 || m == 0 || n > gens->cap || m > gens->parties) return BP_ERR_INVALID_ARGUMENT;
    size_t N = n * m;
    int rc = ipp_alloc(c, N, out); if (rc) return rc;
    bp_ipp *s = *out;
    std::vector<uint32_t> idx = gens_nm_slots(gens, n, m);
    cudaStream_t st = c->stream;
    CK(c, s->idx.ensure(2 * N * 4)); CK(c, c->in_points.ensure(32)); CK(c, c->ok.ensure(1));
    CK(c, cudaMemcpyAsync(s->idx.p, idx.data(), 2 * N * 4, cudaMemcpyHostToDevice, st));
    CK(c, cudaMemcpyAsync(c->in_points.p, Q, 32, cudaMemcpyHostToDevice, st));
    LAUNCH(c, KID_SMALL, k_gather_niels<<<blocks_for(2 * N, 128), 128, 0, st>>>(gens->d_table, s->idx.as<uint32_t>(), (uint32_t)(2 * N), s->pts));
    LAUNCH(c, KID_DECOMPRESS, k_decompress<<<1, 128, 0, st>>>(c->in_points.as<uint8_t>(), 1, s->pts + 2 * N, c->ok.as<uint8_t>()));
    uint8_t ok = 0;
    CK(c, cudaMemcpyAsync(&ok, c->ok.p, 1, cudaMemcpyDeviceToHost, st)); CK(c, cudaStreamSynchronize(st));
    if (!ok) { cudaFree(s->pts); delete s; *out = nullptr; return BP_ERR_INVALID_POINT; }
    return BP_OK;
}
int bp_ipp_begin_points(bp_ctx *c, const uint8_t *G, const uint8_t *H, size_t N, const uint8_t Q[32], bp_ipp **out) {
    if (!G || !H || !Q) return BP_ERR_INVALID_ARGUMENT;
    int rc = ipp_alloc(c, N, out); if (rc) return rc;
    bp_ipp *s = *out; cudaStream_t st = c->stream;
    size_t n_pts = 2 * N + 1;
    CK(c, c->in_points.ensure(n_pts * 32)); CK(c, c->ok.ensure(n_pts));
    CK(c, cudaMemcpyAsync(c->in_points.p, G, N * 32, cudaMemcpyHostToDevice, st));
    CK(c, cudaMemcpyAsync(c->in_points.as<uint8_t>() + N * 32, H, N * 32, cudaMemcpyHostToDevice, st));
    CK(c, cudaMemcpyAsync(c->in_points.as<uint8_t>() + 2 * N * 32, Q, 32, cudaMemcpyHostToDevice, st));
    LAUNCH(c, KID_DECOMPRESS, k_decompress<<<blocks_for(n_pts, 128), 128, 0, st>>>(c->in_points.as<uint8_t>(), n_pts, s->pts, c->ok.as<uint8_t>()));
    std::vector<uint8_t> ok(n_pts);
    CK(c, cudaMemcpyAsync(ok.data(), c->ok.p, n_pts, cudaMemcpyDeviceToHost, st)); CK(c, cudaStreamSynchronize(st));
    for (uint8_t v : ok) if (!v) { cudaFree(s->pts); delete s; *out = nullptr; return BP_ERR_INVALID_POINT; }
    return BP_OK;
}
void bp_ipp_end(bp_ipp *s) { if (!s) return; cudaSetDevice(s->ctx->device); cudaStreamSynchronize(s->ctx->stream); cudaFree(s->pts); s->scal.release(); s->idx.release(); s->offs.release(); delete s; }

// one round's two MSMs: L = <sL[0..h), G_R> + <sL[h..2h), H_L> + sL[2h] Q ;  R = <sR[0..h), G_L> + <sR[h..2h), H_R> + sR[2h] Q
// (inner_product_proof.rs:87-113,153-163); h = n_half = current length / 2
int bp_ipp_lr(bp_ipp *s, size_t n_half, const uint8_t *scalars_L, const uint8_t *scalars_R, uint8_t L_out[32], uint8_t R_out[32]) {
    if (!s || !scalars_L || !scalars_R || !L_out || !R_out || n_half == 0 || 2 * n_half > s->N) return BP_ERR_INVALID_ARGUMENT;
    bp_ctx *c = s->ctx; BUSY_CHECK(c); CK(c, cudaSetDevice(c->device));
    size_t h = n_half, per = 2 * h + 1, N = s->N;
    if (check_scalars_canonical(scalars_L, per) || check_scalars_canonical(scalars_R, per)) return BP_ERR_NONCANONICAL_SCALAR;
    std::vector<uint32_t> idx(2 * per), offs = {0, (uint32_t)per, (uint32_t)(2 * per)};
    for (size_t i = 0; i < h; i++) {
        idx[i] = BP_POINT_DYNAMIC | (uint32_t)(h + i);              // G_R
        idx[h + i] = BP_POINT_DYNAMIC | (uint32_t)(N + i);          // H_L
        idx[per + i] = BP_POINT_DYNAMIC | (uint32_t)i;              // G_L
        idx[per + h + i] = BP_POINT_DYNAMIC | (uint32_t)(N + h + i);  // H_R
    }
    idx[2 * h] = idx[per + 2 * h] = BP_POINT_DYNAMIC | (uint32_t)(2 * N);   // Q
    cudaStream_t st = c->stream;
    CK(c, s->scal.ensure(2 * per * 32)); CK(c, s->idx.ensure(std::max<size_t>(2 * per, 2 * N) * 4)); CK(c, s->offs.ensure(16));
    CK(c, c->results.ensure(2 * sizeof(ge_ext))); CK(c, c->outs.ensure(64));
    CK(c, cudaMemcpyAsync(s->scal.p, scalars_L, per * 32, cudaMemcpyHostToDevice, st));
    CK(c, cudaMemcpyAsync(s->scal.as<uint8_t>() + per * 32, scalars_R, per * 32, cudaMemcpyHostToDevice, st));
    CK(c, cudaMemcpyAsync(s->idx.p, idx.data(), 2 * per * 4, cudaMemcpyHostToDevice, st));
    CK(c, cudaMemcpyAsync(s->offs.p, offs.data(), 12, cudaMemcpyHostToDevice, st));
    MsmArgs a{s->scal.as<uint8_t>(), s->offs.as<uint32_t>(), 2, (uint32_t)(2 * per), s->idx.as<uint32_t>(), nullptr, s->pts, nullptr, 0};
    int rc = msm_core(c, a, c->results.as<ge_ext>());
    if (rc) return rc;
    LAUNCH(c, KID_COMPRESS, k_compress<<<1, 128, 0, st>>>(c->results.as<ge_ext>(), 2, c->outs.as<uint8_t>()));
    uint8_t lr[64];
    CK(c, cudaMemcpyAsync(lr, c->outs.p, 64, cudaMemcpyDeviceToHost, st)); CK(c, cudaStreamSynchronize(st));
    memcpy(L_out, lr, 32); memcpy(R_out, lr + 32, 32);
    return BP_OK;
}
// G_L[i] = g_lo[i] G_L[i] + g_hi[i] G_R[i] ;  H_L[i] = h_lo[i] H_L[i] + h_hi[i] H_R[i]   (inner_product_proof.rs:124-135,174-179).
// per_index = 1: n_half scalars in each array (first round, factors folded in); 0: one scalar each (u^-1, u / u, u^-1).
int bp_ipp_fold(bp_ipp *s, size_t n_half, const uint8_t *g_lo, const uint8_t *g_hi, const uint8_t *h_lo, const uint8_t *h_hi, int per_index) {
    if (!s || !g_lo || !g_hi || !h_lo || !h_hi || n_half == 0 || 2 * n_half > s->N) return BP_ERR_INVALID_ARGUMENT;
    bp_ctx *c = s->ctx; BUSY_CHECK(c); CK(c, cudaSetDevice(c->device));
    size_t cnt = per_index ? n_half : 1, h = n_half;
    const uint8_t *arrs[4] = {g_lo, g_hi, h_lo, h_hi};
    for (auto a : arrs) if (check_scalars_canonical(a, cnt)) return BP_ERR_NONCANONICAL_SCALAR;
    cudaStream_t st = c->stream;
    CK(c, s->scal.ensure(4 * cnt * 32));
    for (int k = 0; k < 4; k++) CK(c, cudaMemcpyAsync(s->scal.as<uint8_t>() + (size_t)k * cnt * 32, arrs[k], cnt * 32, cudaMemcpyHostToDevice, st));
    uint32_t stride = per_index ? 32 : 0;
    const uint8_t *d = s->scal.as<uint8_t>();
    LAUNCH(c, KID_IPP_FOLD, k_ipp_fold<<<blocks_for(h, 64), 64, 0, st>>>(s->pts, (uint32_t)h, d, d + cnt * 32, stride));
    LAUNCH(c, KID_IPP_FOLD, k_ipp_fold<<<blocks_for(h, 64), 64, 0, st>>>(s->pts + s->N, (uint32_t)h, d + 2 * cnt * 32, d + 3 * cnt * 32, stride));
    CK(c, cudaStreamSynchronize(st));          // the scalar staging buffer is reused by the next round
    return BP_OK;
}

// ---------------------------------------------------------------------------------------------- inner-product prover, device-resident state
}  // extern "C"
struct bp_ippx {
    bp_ctx *ctx = nullptr; uint32_t N = 0, B = 0, n = 0;
    const ge_niels *d_static = nullptr; ge_niels *own_pts = nullptr;      // the gens table, or the session's own [G (N) | H (N)]
    ge_niels *d_q = nullptr;                                               // B points Q
    DevBuf a, b, cG, cH, gidx, hidx, scal, pidx, offs, in, outs;
};
extern "C" {
static void ippx_free(bp_ippx *s);
static int ippx_alloc(bp_ctx *c, size_t N, size_t B, bp_ippx **out) {
    if (!c || !out || N == 0 || (N & (N - 1)) || B == 0 || 2 * B * (N + 1) >= (1u << 31)) return BP_ERR_INVALID_ARGUMENT;      // power of two (inner_product_proof.rs:67)
    BUSY_CHECK(c);
    CK(c, cudaSetDevice(c->device));
    bp_ippx *s = new bp_ippx(); s->ctx = c; s->N = (uint32_t)N; s->B = (uint32_t)B; s->n = (uint32_t)N;
    size_t BN = B * N;
    cudaError_t e = cudaMalloc((void **)&s->d_q, B * sizeof(ge_niels));
    if (e != cudaSuccess) { c->err = std::string("cudaMalloc(ippx): ") + cudaGetErrorString(e); delete s; return BP_ERR_CUDA; }
    int rc = [&]() -> int {
        for (DevBuf *b : {&s->a, &s->b, &s->cG, &s->cH}) CK(c, b->ensure(BN * sizeof(sc)));
        CK(c, s->gidx.ensure(N * 4)); CK(c, s->hidx.ensure(N * 4)); CK(c, s->scal.ensure(2 * B * (N + 1) * 32)); CK(c, s->pidx.ensure(2 * B * (N + 1) * 4));
        CK(c, s->offs.ensure((2 * B + 1) * 4)); CK(c, s->in.ensure(std::max<size_t>(4 * BN * 32, 64 * B))); CK(c, s->outs.ensure(64 * B));
        return BP_OK;
    }();
    if (rc) { ippx_free(s); return rc; }
    *out = s; return BP_OK;
}
static void ippx_free(bp_ippx *s) {
    cudaFree(s->d_q); if (s->own_pts) cudaFree(s->own_pts);
    for (DevBuf *b : {&s->a, &s->b, &s->cG, &s->cH, &s->gidx, &s->hidx, &s->scal, &s->pidx, &s->offs, &s->in, &s->outs}) b->release();
    delete s;
}
// common tail of the two begin forms: Q points, scalar vectors (B x N canonical scalars each; Gf / Hf may be NULL = all ones)
static int ippx_load(bp_ippx *s, const uint8_t *Q, const uint8_t *Gf, const uint8_t *Hf, const uint8_t *a, const uint8_t *b) {
    bp_ctx *c = s->ctx; cudaStream_t st = c->stream; size_t BN = (size_t)s->B * s->N;
    for (const uint8_t *v : {a, b}) if (check_scalars_canonical(v, BN)) return BP_ERR_NONCANONICAL_SCALAR;
    for (const uint8_t *v : {Gf, Hf}) if (v && check_scalars_canonical(v, BN)) return BP_ERR_NONCANONICAL_SCALAR;
    uint8_t *din = s->in.as<uint8_t>();
    CK(c, cudaMemcpyAsync(din, a, BN * 32, cudaMemcpyHostToDevice, st)); CK(c, cudaMemcpyAsync(din + BN * 32, b, BN * 32, cudaMemcpyHostToDevice, st));
    if (Gf) CK(c, cudaMemcpyAsync(din + 2 * BN * 32, Gf, BN * 32, cudaMemcpyHostToDevice, st));
    if (Hf) CK(c, cudaMemcpyAsync(din + 3 * BN * 32, Hf, BN * 32, cudaMemcpyHostToDevice, st));
    ippx_geom g{s->N, s->B, s->n};
    LAUNCH(c, KID_SMALL, k_ippx_init<<<blocks_for(BN, 128), 128, 0, st>>>(g, din, din + BN * 32, Gf ? din + 2 * BN * 32 : nullptr, Hf ? din + 3 * BN * 32 : nullptr,
                                                                         s->a.as<sc>(), s->b.as<sc>(), s->cG.as<sc>(), s->cH.as<sc>()));
    CK(c, c->in_points.ensure((size_t)s->B * 32)); CK(c, c->ok.ensure(s->B));
    CK(c, cudaMemcpyAsync(c->in_points.p, Q, (size_t)s->B * 32, cudaMemcpyHostToDevice, st));
    LAUNCH(c, KID_DECOMPRESS, k_decompress<<<blocks_for(s->B, 128), 128, 0, st>>>(c->in_points.as<uint8_t>(), s->B, s->d_q, c->ok.as<uint8_t>()));
    std::vector<uint8_t> ok(s->B);
    CK(c, cudaMemcpyAsync(ok.data(), c->ok.p, s->B, cudaMemcpyDeviceToHost, st)); CK(c, cudaStreamSynchronize(st));
    for (uint8_t v : ok) if (!v) return BP_ERR_INVALID_POINT;
    LAUNCH(c, KID_SMALL, k_fill_offsets<<<blocks_for((size_t)2 * s->B + 1, 256), 256, 0, st>>>(2 * s->B, s->N + 1, s->offs.as<uint32_t>()));
    return BP_OK;
}
int bp_ippx_begin(bp_ctx *c, bp_gens *gens, size_t n, size_t m, size_t n_proofs, const uint8_t *Q, const uint8_t *Gf, const uint8_t *Hf, const uint8_t *a, const uint8_t *b, bp_ippx **out) {
    if (!gens || !Q || !a || !b || n == 0 || m == 0 || n > gens->cap || m > gens->parties) return BP_ERR_INVALID_ARGUMENT;
    size_t N = n * m;
    int rc = ippx_alloc(c, N, n_proofs, out); if (rc) return rc;
    bp_ippx *s = *out; s->d_static = gens->d_table;
    std::vector<uint32_t> idx = gens_nm_slots(gens, n, m);
    rc = [&]() -> int {
        CK(c, cudaMemcpyAsync(s->gidx.p, idx.data(), N * 4, cudaMemcpyHostToDevice, c->stream)); CK(c, cudaMemcpyAsync(s->hidx.p, idx.data() + N, N * 4, cudaMemcpyHostToDevice, c->stream));
        CK(c, cudaStreamSynchronize(c->stream));
        return ippx_load(s, Q, Gf, Hf, a, b);
    }();
    if (rc) { ippx_free(s); *out = nullptr; }
    return rc;
}
int bp_ippx_begin_points(bp_ctx *c, const uint8_t *G, const uint8_t *H, size_t N, size_t n_proofs, const uint8_t *Q, const uint8_t *Gf, const uint8_t *Hf, const uint8_t *a, const uint8_t *b, bp_ippx **out) {
    if (!G || !H || !Q || !a || !b) return BP_ERR_INVALID_ARGUMENT;
    int rc = ippx_alloc(c, N, n_proofs, out); if (rc) return rc;
    bp_ippx *s = *out; cudaStream_t st = c->stream;
    cudaError_t e = cudaMalloc((void **)&s->own_pts, 2 * N * sizeof(ge_niels));
    if (e != cudaSuccess) { c->err = std::string("cudaMalloc(ippx points): ") + cudaGetErrorString(e); ippx_free(s); *out = nullptr; return BP_ERR_CUDA; }
    s->d_static = s->own_pts;
    std::vector<uint8_t> ok(2 * N); std::vector<uint32_t> idx(2 * N);
    for (size_t q = 0; q < 2 * N; q++) idx[q] = (uint32_t)q;
    rc = [&]() -> int {
        CK(c, c->in_points.ensure(2 * N * 32)); CK(c, c->ok.ensure(2 * N));
        CK(c, cudaMemcpyAsync(c->in_points.p, G, N * 32, cudaMemcpyHostToDevice, st)); CK(c, cudaMemcpyAsync(c->in_points.as<uint8_t>() + N * 32, H, N * 32, cudaMemcpyHostToDevice, st));
        LAUNCH(c, KID_DECOMPRESS, k_decompress<<<blocks_for(2 * N, 128), 128, 0, st>>>(c->in_points.as<uint8_t>(), 2 * N, s->own_pts, c->ok.as<uint8_t>()));
        CK(c, cudaMemcpyAsync(ok.data(), c->ok.p, 2 * N, cudaMemcpyDeviceToHost, st));
        CK(c, cudaMemcpyAsync(s->gidx.p, idx.data(), N * 4, cudaMemcpyHostToDevice, st)); CK(c, cudaMemcpyAsync(s->hidx.p, idx.data() + N, N * 4, cudaMemcpyHostToDevice, st));
        CK(c, cudaStreamSynchronize(st));
        for (uint8_t v : ok) if (!v) return BP_ERR_INVALID_POINT;
        return ippx_load(s, Q, Gf, Hf, a, b);
    }();
    if (rc) { ippx_free(s); *out = nullptr; }
    return rc;
}
void bp_ippx_end(bp_ippx *s) { if (!s) return; cudaSetDevice(s->ctx->device); cudaStreamSynchronize(s->ctx->stream); ippx_free(s); }
size_t bp_ippx_current_len(const bp_ippx *s) { return s ? s->n : 0; }
// L and R of the current round for every proof (inner_product_proof.rs:87-113 / 153-163): LR_out = n_proofs x (L | R) compressed; synchronises
int bp_ippx_round(bp_ippx *s, uint8_t *LR_out) {
    if (!s || !LR_out || s->n < 2) return BP_ERR_INVALID_ARGUMENT;
    bp_ctx *c = s->ctx; BUSY_CHECK(c); CK(c, cudaSetDevice(c->device));
    cudaStream_t st = c->stream; ippx_geom g{s->N, s->B, s->n};
    uint32_t M = 2 * s->B, T = M * (s->N + 1);
    LAUNCH(c, KID_SMALL, k_ippx_inner<<<M, 128, 0, st>>>(g, s->a.as<sc>(), s->b.as<sc>(), s->scal.as<uint8_t>()));
    LAUNCH(c, KID_SMALL, k_ippx_rows<<<blocks_for((size_t)s->B * s->N, 128), 128, 0, st>>>(g, s->a.as<sc>(), s->b.as<sc>(), s->cG.as<sc>(), s->cH.as<sc>(), s->gidx.as<uint32_t>(), s->hidx.as<uint32_t>(),
                                                                                          s->scal.as<uint8_t>(), s->pidx.as<uint32_t>()));
    CK(c, c->results.ensure((size_t)M * sizeof(ge_ext)));
    MsmArgs a{s->scal.as<uint8_t>(), s->offs.as<uint32_t>(), M, T, s->pidx.as<uint32_t>(), s->d_static, s->d_q, nullptr, 0};
    int rc = msm_core(c, a, c->results.as<ge_ext>());
    if (rc) return rc;
    LAUNCH(c, KID_COMPRESS, k_compress<<<blocks_for(M, 128), 128, 0, st>>>(c->results.as<ge_ext>(), M, s->outs.as<uint8_t>()));
    CK(c, cudaMemcpyAsync(LR_out, s->outs.p, (size_t)M * 32, cudaMemcpyDeviceToHost, st)); CK(c, cudaStreamSynchronize(st));
    return BP_OK;
}
// apply the challenges u (and their inverses), one pair per proof; halves the current length
int bp_ippx_fold(bp_ippx *s, const uint8_t *u, const uint8_t *u_inv) {
    if (!s || !u || !u_inv || s->n < 2) return BP_ERR_INVALID_ARGUMENT;
    bp_ctx *c = s->ctx; BUSY_CHECK(c); CK(c, cudaSetDevice(c->device));
    if (check_scalars_canonical(u, s->B) || check_scalars_canonical(u_inv, s->B)) return BP_ERR_NONCANONICAL_SCALAR;
    cudaStream_t st = c->stream; ippx_geom g{s->N, s->B, s->n};
    uint8_t *din = s->in.as<uint8_t>();
    CK(c, cudaMemcpyAsync(din, u, (size_t)s->B * 32, cudaMemcpyHostToDevice, st)); CK(c, cudaMemcpyAsync(din + (size_t)s->B * 32, u_inv, (size_t)s->B * 32, cudaMemcpyHostToDevice, st));
    LAUNCH(c, KID_IPP_FOLD, k_ippx_fold<<<blocks_for((size_t)s->B * s->N, 128), 128, 0, st>>>(g, din, din + (size_t)s->B * 32, s->a.as<sc>(), s->b.as<sc>(), s->cG.as<sc>(), s->cH.as<sc>()));
    CK(c, cudaStreamSynchronize(st));          // the staging buffer is reused by the next call
    s->n >>= 1;
    return BP_OK;
}
// the final a, b (inner_product_proof.rs:187-192): ab_out = n_proofs x (a | b)
int bp_ippx_finish(bp_ippx *s, uint8_t *ab_out) {
    if (!s || !ab_out || s->n != 1) return BP_ERR_INVALID_ARGUMENT;
    bp_ctx *c = s->ctx; BUSY_CHECK(c); CK(c, cudaSetDevice(c->device));
    ippx_geom g{s->N, s->B, s->n};
    LAUNCH(c, KID_SMALL, k_ippx_final<<<blocks_for(s->B, 128), 128, 0, c->stream>>>(g, s->a.as<sc>(), s->b.as<sc>(), s->outs.as<uint8_t>()));
    CK(c, cudaMemcpyAsync(ab_out, s->outs.p, (size_t)s->B * 64, cudaMemcpyDeviceToHost, c->stream)); CK(c, cudaStreamSynchronize(c->stream));
    return BP_OK;
}

// ---------------------------------------------------------------------------------------------- per-kernel timing
int bp_prof_enable(bp_ctx *c, int on) {
    if (!c) return BP_ERR_INVALID_ARGUMENT;
    for (ProfRec &r : c->prof) { cudaEventDestroy(r.a); cudaEventDestroy(r.b); }
    c->prof.clear(); c->prof_on = on != 0; return BP_OK;
}
int bp_prof_kernel_count(void) { return KID_COUNT; }
const char *bp_prof_kernel_name(int kid) { return kid >= 0 && kid < KID_COUNT ? KERNEL_NAMES[kid] : ""; }
// synchronises the stream, adds up the CUDA-event durations recorded since the last report; ms/counts have bp_prof_kernel_count() entries
int bp_prof_report(bp_ctx *c, double *ms, uint64_t *counts) {
    if (!c || !ms || !counts) return BP_ERR_INVALID_ARGUMENT;
    CK(c, cudaSetDevice(c->device)); CK(c, cudaStreamSynchronize(c->stream));
    for (int i = 0; i < KID_COUNT; i++) { ms[i] = 0; counts[i] = 0; }
    for (ProfRec &r : c->prof) { float t = 0; if (cudaEventElapsedTime(&t, r.a, r.b) == cudaSuccess) { ms[r.kid] += t; counts[r.kid]++; } cudaEventDestroy(r.a); cudaEventDestroy(r.b); }
    c->prof.clear();
    return BP_OK;
}
// per-launch records since the last report/enable: start and end in ms relative to the first record of `ref` (a context of the
// same device whose profiling was enabled first); synchronises both streams.  Diagnostic for multi-stream overlap.
int bp_prof_timeline(bp_ctx *c, bp_ctx *ref, int *kernel_ids, double *start_ms, double *end_ms, size_t cap, size_t *n_out) {
    if (!c || !ref || !kernel_ids || !start_ms || !end_ms || !n_out) return BP_ERR_INVALID_ARGUMENT;
    CK(c, cudaSetDevice(c->device)); CK(c, cudaStreamSynchronize(c->stream)); CK(c, cudaStreamSynchronize(ref->stream));
    if (ref->prof.empty()) return BP_ERR_INVALID_ARGUMENT;
    size_t n = 0;
    for (ProfRec &r : c->prof) {
        if (n >= cap) break;
        float a = 0, b = 0;
        if (cudaEventElapsedTime(&a, ref->prof[0].a, r.a) != cudaSuccess || cudaEventElapsedTime(&b, ref->prof[0].a, r.b) != cudaSuccess) continue;
        kernel_ids[n] = r.kid; start_ms[n] = a; end_ms[n] = b; n++;
    }
    *n_out = n;
    return BP_OK;
}
// copy the resident generator table to / from another device buffer (e.g. a torch tensor used for the NCCL broadcast)
int bp_gens_table_export(bp_gens *g, void *d_dst) {
    if (!g || !d_dst) return BP_ERR_INVALID_ARGUMENT;
    bp_ctx *c = g->ctx; CK(c, cudaSetDevice(c->device));
    CK(c, cudaMemcpyAsync(d_dst, g->d_table, g->n_points * sizeof(ge_niels), cudaMemcpyDeviceToDevice, c->stream)); CK(c, cudaStreamSynchronize(c->stream)); return BP_OK;
}
int bp_gens_table_import(bp_gens *g, const void *d_src) {
    if (!g || !d_src) return BP_ERR_INVALID_ARGUMENT;
    bp_ctx *c = g->ctx; CK(c, cudaSetDevice(c->device));
    CK(c, cudaMemcpyAsync(g->d_table, d_src, g->n_points * sizeof(ge_niels), cudaMemcpyDeviceToDevice, c->stream)); CK(c, cudaStreamSynchronize(c->stream)); return BP_OK;
}

// ---------------------------------------------------------------------------------------------- host helpers
// merlin::Transcript for hosts that do not have the Rust crate (the Python harness, C++ callers):
// same STROBE code the device kernels use, compiled for the host.  Pure byte shuffling, no curve math.
void bp_transcript_new(const uint8_t *label, size_t len, uint8_t out[BP_TRANSCRIPT_BYTES]) { alignas(8) uint8_t st[200]; merlin_t m; m.st = st; merlin_init(m, label, (uint32_t)len); merlin_store(out, m); }
void bp_transcript_append_message(uint8_t state[BP_TRANSCRIPT_BYTES], const char *label, const uint8_t *msg, size_t len) {
    alignas(8) uint8_t st[200]; merlin_t m; m.st = st; merlin_load(m, state); merlin_append(m, label, msg, (uint32_t)len); merlin_store(state, m);
}
void bp_transcript_append_u64(uint8_t state[BP_TRANSCRIPT_BYTES], const char *label, uint64_t x) { alignas(8) uint8_t st[200]; merlin_t m; m.st = st; merlin_load(m, state); merlin_append_u64(m, label, x); merlin_store(state, m); }
void bp_transcript_challenge_bytes(uint8_t state[BP_TRANSCRIPT_BYTES], const char *label, uint8_t *out, size_t len) {
    alignas(8) uint8_t st[200]; merlin_t m; m.st = st; merlin_load(m, state); merlin_challenge(m, label, out, (uint32_t)len); merlin_store(state, m);
}

// test hook: element-wise field operation on the device (pins the PTX carry chains of fe.cuh)
__global__ void k_debug_fe(int op, const uint8_t *a, const uint8_t *b, size_t n, uint8_t *out) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint8_t ab[32], bb[32]; ld32(ab, a + 32 * i); ld32(bb, b + 32 * i);
    fe x = fe_frombytes_raw(ab), y = fe_frombytes_raw(bb), r;
    switch (op) {
        case 0: r = fe_add(x, y); break;
        case 1: r = fe_sub(x, y); break;
        case 2: r = fe_mul(x, y); break;
        case 3: r = fe_invert(x); break;
        case 4: r = fe_pow22523(x); break;
        case 5: r = fe_neg(x); break;
        case 7: r = fe_mul(fe_add(x, y), fe_sub(x, y)); break;      // chained, unreduced intermediates
        default: r = fe_sq(x);
    }
    uint8_t o[32]; fe_tobytes(o, r); st32(out + 32 * i, o);
}
int bp_debug_fe_op(bp_ctx *c, int op, const uint8_t *a, const uint8_t *b, size_t n, uint8_t *out) {
    if (!c || !a || !b || !out || n == 0) return BP_ERR_INVALID_ARGUMENT;
    CK(c, cudaSetDevice(c->device));
    CK(c, c->in_scalars.ensure(n * 32)); CK(c, c->in_points.ensure(n * 32)); CK(c, c->outs.ensure(n * 32));
    CK(c, cudaMemcpyAsync(c->in_scalars.p, a, n * 32, cudaMemcpyHostToDevice, c->stream));
    CK(c, cudaMemcpyAsync(c->in_points.p, b, n * 32, cudaMemcpyHostToDevice, c->stream));
    LAUNCH(c, KID_SMALL, k_debug_fe<<<blocks_for(n, 128), 128, 0, c->stream>>>(op, c->in_scalars.as<uint8_t>(), c->in_points.as<uint8_t>(), n, c->outs.as<uint8_t>()));
    CK(c, cudaMemcpyAsync(out, c->outs.p, n * 32, cudaMemcpyDeviceToHost, c->stream));
    CK(c, cudaStreamSynchronize(c->stream));
    return BP_OK;
}

// test hook: element-wise scalar operation on the device (pins the device branch of sc_mont_mul and the lazy reduction of sc.cuh).
// Raw limbs in and out: no conversion is added around the operation under test.
__global__ void k_debug_sc(int op, const uint8_t *a, const uint8_t *b, size_t n, uint8_t *out) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (op == 8) {                                                  // sum32: one accumulator per 32 consecutive pairs
        if (i >= n / 32) return;
        sc_wide acc = sc_wide_zero();
        for (size_t j = 32 * i; j < 32 * i + 32; j++) { uint8_t x[32], y[32]; ld32(x, a + 32 * j); ld32(y, b + 32 * j); sc_wide_mac(acc, sc_load(x), sc_load(y)); }
        uint8_t o[32]; sc_store(o, sc_wide_redc(acc)); st32(out + 32 * i, o);
        return;
    }
    if (i >= n) return;
    uint8_t wide[64]; ld32(wide, a + 32 * i); ld32(wide + 32, b + 32 * i);
    sc x = sc_load(wide), y = sc_load(wide + 32), r;
    switch (op) {
        case 0: r = sc_mont_mul(x, y); break;
        case 1: r = sc_from_mont(sc_mont_mul(sc_to_mont(x), sc_to_mont(y))); break;
        case 2: r = sc_add(x, y); break;
        case 3: r = sc_sub(x, y); break;
        case 4: r = sc_neg(x); break;
        case 5: r = sc_mont_from_wide(wide); break;
        case 6: r = rp_wide(wide); break;
        default: r = sc_mont_invert(x);
    }
    uint8_t o[32]; sc_store(o, r); st32(out + 32 * i, o);
}
int bp_debug_sc_op(bp_ctx *c, int op, const uint8_t *a, const uint8_t *b, size_t n, uint8_t *out) {
    if (!c || !a || !b || !out || n == 0 || op < 0 || op > 8 || (op == 8 && n % 32 != 0)) return BP_ERR_INVALID_ARGUMENT;
    BUSY_CHECK(c);
    CK(c, cudaSetDevice(c->device));
    const size_t n_out = op == 8 ? n / 32 : n;
    CK(c, c->in_scalars.ensure(n * 32)); CK(c, c->in_points.ensure(n * 32)); CK(c, c->outs.ensure(n_out * 32));
    CK(c, cudaMemcpyAsync(c->in_scalars.p, a, n * 32, cudaMemcpyHostToDevice, c->stream));
    CK(c, cudaMemcpyAsync(c->in_points.p, b, n * 32, cudaMemcpyHostToDevice, c->stream));
    LAUNCH(c, KID_SMALL, k_debug_sc<<<blocks_for(n_out, 128), 128, 0, c->stream>>>(op, c->in_scalars.as<uint8_t>(), c->in_points.as<uint8_t>(), n, c->outs.as<uint8_t>()));
    CK(c, cudaMemcpyAsync(out, c->outs.p, n_out * 32, cudaMemcpyDeviceToHost, c->stream));
    CK(c, cudaStreamSynchronize(c->stream));
    return BP_OK;
}

}  // extern "C"
