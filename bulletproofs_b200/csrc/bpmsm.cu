// C ABI of the engine (include/bpmsm.h): context, scratch arenas, kernel orchestration.
// No CPU fallback: every entry point needs a usable CUDA device and fails with BP_ERR_CUDA otherwise.
#include <cuda_runtime.h>
#include <sys/random.h>
#include <cstdio>
#include <cstdlib>
#include <algorithm>
#include <array>
#include <cstring>
#include <memory>
#include <string>
#include <vector>
#include "../../include/bpmsm.h"
#include "kernels.cuh"
#include "r1cs_kernels.cuh"
#include "linear_kernels.cuh"
#include "linear_mixed.cuh"
#include "linear_mixed_device.cuh"
#include "rp_mixed_device.cuh"
#include "rp_single.cuh"
#include "rp_exact.cuh"

static_assert(BP_TRANSCRIPT_BYTES == 203, "transcript wire size");

namespace {

// One device allocation, freed with its owner.
struct DevBuf {
    void *p = nullptr; size_t cap = 0;
    uint64_t *moves = nullptr;      // optional: counts every (re)allocation, i.e. every change of p (RpScratch)
    DevBuf() = default;
    explicit DevBuf(uint64_t *m) : moves(m) {}
    DevBuf(DevBuf &&o) noexcept : p(o.p), cap(o.cap), moves(o.moves) { o.p = nullptr; o.cap = 0; }      // move-only: no copy is declared
    ~DevBuf() { if (p) cudaFree(p); }
    // grow-only, with headroom: the scratch of a context
    // s: the stream of the owning context, the only stream whose work reads the buffer (the verifier's second branch joins it again)
    cudaError_t ensure(size_t bytes, cudaStream_t s) {
        if (bytes <= cap) return cudaSuccess;
        // Work queued earlier (the device-resident entry points return without synchronising) may still read the old buffer, and
        // cudaFree is documented only as "may perform implicit synchronization": wait for that work explicitly.  Only this context's
        // stream, so that other contexts and their graph captures are not touched.  Buffers only grow, so this runs when a context
        // first meets a larger size, never in a steady stream of calls of one geometry.
        if (p) { cudaError_t e = cudaStreamSynchronize(s); if (e != cudaSuccess) return e; cudaFree(p); p = nullptr; cap = 0; }
        return alloc(bytes + bytes / 4 + 256);
    }
    // exactly `bytes`, into an empty buffer: the fixed allocations of a handle, which would otherwise carry ensure's 25 % headroom
    // (about 25 MB on a 2^20-point set)
    cudaError_t alloc(size_t bytes) {
        if (moves) ++*moves;
        cudaError_t e = cudaMalloc(&p, bytes);
        if (e == cudaSuccess) cap = bytes; else p = nullptr;
        return e;
    }
    template <class T> T *as() const { return reinterpret_cast<T *>(p); }
};
// One pinned host allocation, freed with its owner.  Grow-only; the old buffer is freed when it grows, so its owner must know that no
// queued copy still reads or writes it.
struct PinnedBuf {
    void *p = nullptr; size_t cap = 0;
    PinnedBuf() = default;
    PinnedBuf(const PinnedBuf &) = delete;
    ~PinnedBuf() { if (p) cudaFreeHost(p); }
    cudaError_t ensure(size_t bytes) {
        if (bytes <= cap) return cudaSuccess;
        if (p) cudaFreeHost(p);
        p = nullptr; cap = 0;
        cudaError_t e = cudaMallocHost(&p, bytes);
        if (e == cudaSuccess) cap = bytes; else p = nullptr;
        return e;
    }
    template <class T> T *as() const { return reinterpret_cast<T *>(p); }
};
// Pinned staging slots for per-call uploads: acquire() waits for the upload last queued from its slot, record() follows the new one, so
// queued calls on one context never see each other's data and no upload reads caller memory after the entry point returns.
struct StageRing {
    static const int SLOTS = 8;
    PinnedBuf buf; size_t slot_bytes = 0; cudaEvent_t ev[SLOTS] = {}; unsigned next = 0, cur = 0;
    ~StageRing() { for (cudaEvent_t e : ev) if (e) cudaEventDestroy(e); }
    cudaError_t init(size_t bytes) {
        slot_bytes = bytes;
        cudaError_t e = buf.ensure(SLOTS * bytes);
        for (cudaEvent_t &v : ev) if (e == cudaSuccess) e = cudaEventCreateWithFlags(&v, cudaEventDisableTiming);
        return e;
    }
    template <class T> cudaError_t acquire(T *&slot) {
        cur = next++ % SLOTS;
        slot = reinterpret_cast<T *>(buf.as<uint8_t>() + cur * slot_bytes);
        return cudaEventSynchronize(ev[cur]);
    }
    cudaError_t record(cudaStream_t s) { return cudaEventRecord(ev[cur], s); }
};

// profiling label of every kernel id, in id order
#define BP_KERNELS(X)                                                                                                                        \
    X(DECOMPRESS, "k_decompress") X(COMPRESS, "k_compress") X(FROM_UNIFORM, "k_from_uniform") X(MSM_COUNT, "k_msm_count")                  \
    X(MSM_SCAN, "k_msm_scan") X(MSM_SCATTER, "k_msm_scatter") X(MSM_ACCUMULATE, "k_msm_accumulate") X(MSM_REDUCE, "k_msm_reduce")         \
    X(MSM_COMBINE, "k_msm_combine") X(RP_TRANSCRIPT, "k_rp_transcript") X(RP_HEAD, "k_rp_head") X(RP_SCALARS, "k_rp_scalars_sum")          \
    X(RP_DECOMPRESS, "k_rp_decompress") X(RP_STATIC_REDUCE, "k_rp_static_reduce") X(RP_VERDICT_GROUP, "k_rp_verdict_group")                \
    X(RP_BATCH_ROWS, "k_rp_batch_rows") X(RP_VERDICT_BATCH, "k_rp_verdict_batch") X(IPPX_FOLD, "k_ippx_fold") X(SMALL, "small_kernels")    \
    X(R1CS_TABLES, "k_r1cs_tables") X(R1CS_GH_SUM, "k_r1cs_gh_sum") X(R1CS_ROWS, "k_r1cs_rows")                                          \
    X(LIN_DECOMPRESS, "k_lin_decompress") X(LIN_TRANSCRIPT, "k_lin_transcript") X(LIN_TABLES, "k_lin_tables") X(LIN_G_SUM, "k_lin_g_sum")   \
    X(LIN_DYNAMIC, "k_lin_dynamic") X(LIN_G_TOTAL, "k_lin_g_total") X(LIN_ROWS, "k_lin_proof_rows") X(MIX_PLAN, "k_mix_plan")     \
    X(RP_SINGLE, "k_rp_single") X(LINM_GATHER, "k_linm_gather") X(LINM_DECOMPRESS, "k_linm_decompress") X(LINM_TRANSCRIPT, "k_linm_transcript")          \
    X(LINM_TABLES, "k_linm_tables") X(LINM_G_SUM, "k_linm_g_sum") X(LINM_DYNAMIC, "k_linm_dynamic") X(LINM_G_TOTAL, "k_linm_g_total")
#define KID_ENUM(id, name) KID_##id,
enum KernelId { BP_KERNELS(KID_ENUM) KID_COUNT };
#define KID_NAME(id, name) name,
const char *const KERNEL_NAMES[KID_COUNT] = {BP_KERNELS(KID_NAME)};
struct ProfRec { int kid; cudaEvent_t a, b; };

struct VerifyState {          // what bp_rangeproof_verify_*begin leaves for *_finish
    bool active = false; rp_geom g{}; uint32_t total = 0, n_batches = 1; bp_gens *gens = nullptr; uint8_t param_verdict = 0;
    std::vector<uint8_t> param_codes;       // rejected parameters: every proof's verdict, decided on the host in *_begin
};
struct MsmArena {             // scratch of one Pippenger pipeline pass; `moves` as in DevBuf
    uint64_t *moves = nullptr;
    DevBuf counts{moves}, starts{moves}, cursor{moves}, order{moves}, sorted{moves}, buckets{moves}, wsums{moves};
};
// Scratch of the device reject path of an exact graph (rp_exact.cuh): the group table, the MSM rows of either level, the MSM offsets (level
// 1, then each group's level 2), their results, the failing-proof lists, three counters per group and the level-2 static-term sums.
// `moves` as in DevBuf.
struct XScratch {
    uint64_t *moves = nullptr;
    DevBuf grp{moves}, scal{moves}, pidx{moves}, offsets{moves}, results{moves}, list{moves}, ctr{moves}, part2{moves};
};
// Everything the verifier's launch graph bakes into its nodes.  Private to the verifier: no other entry point regrows -- i.e. moves --
// one of these buffers.  Each counts its reallocations in `moves`; a captured graph is replayed only while the count it was captured
// at still holds.
struct RpScratch {
    uint64_t moves = 0;
    MsmArena ar{&moves};
    DevBuf niels{&moves}, results{&moves}, chal{&moves}, raw{&moves}, tabs{&moves}, pow2_tab{&moves}, par{&moves}, part{&moves}, scalars{&moves},
        status{&moves}, decbad{&moves}, pidx{&moves}, offsets{&moves}, batch_ok{&moves}, combined{&moves};
    DevBuf run{&moves}, bstatic{&moves}, bscal{&moves}, bpidx{&moves}, boffsets{&moves};  // launch groups: per-batch pass gate, static rows, scalar rows, point map, offsets
    DevBuf prog{&moves}; uint32_t prog_steps = 0;            // transcript step program of the geometry in pidx_key (rp_tr_program)
    XScratch xs{&moves};                                     // the exact graph's reject path (bp_rangeproof_verify_reserve_exact)
};
// Arenas of bp_rangeproof_verify_mixed (layout: rp_mixed.cuh), apart from RpScratch: a mixed call never moves or overwrites what the
// verifier graph and the cached maps of the fixed-geometry path point at.
struct MixScratch {
    MsmArena ar;
    DevBuf in_proofs, in_commit, gather, proofs, commit, par, prog, raw, status, decbad, chal, tabs, part, scalars, pidx, offsets, niels, verdict, flags,
        results, pow2_tab, tstates;
};
// A reserved mix (bp_rangeproof_verify_mixed_reserve): its layout, its own arenas and pinned staging, and its captured graph.  Only
// bp_rangeproof_verify_mixed_reserve moves these buffers, and it captures the graph again, so the graph never meets a moved one.
struct MixReserve {
    rp_mixed_plan X;                                   // the classes at capacity (rp_mixed_mix): slots, segments and arena slices
    MixScratch x;
    // pinned, written on the host by each fitting call and read by its uploads: rp_params[C] | rp_gather[A] | transcript records[A];
    // the uploads complete before the call's finish returns, and no other call on the context runs in between
    PinnedBuf h_stage;
    PinnedBuf h_verdict, h_flag;                       // A verdicts in slot order, C combined flags
    cudaGraphExec_t graph = nullptr; uint64_t graph_launches = 0;
    // bp_rangeproof_verify_mixed_reserve_exact: the exact graph (the same sequence, then the device reject path on xs); null otherwise
    XScratch xs; cudaGraphExec_t xgraph = nullptr; uint64_t xgraph_launches = 0;
    const void *gens_table = nullptr; size_t gens_cap = 0, gens_parties = 0;      // the generator table the graph reads
    // calls on device inputs (bp_rangeproof_verify_mixed_device*): the mix as the planner kernels see it, a staging ring of the C parameter
    // blocks (so queued calls never see each other's blocks, and h_stage above is not touched), and the planner's per-input scratch:
    // code | class, rank then slot, per-block class counts
    rp_mix_classes M{};
    StageRing dstage;
    DevBuf pl_code, pl_slot, pl_hist;
    ~MixReserve() { if (graph) cudaGraphExecDestroy(graph); if (xgraph) cudaGraphExecDestroy(xgraph); }
    size_t slots() const { return X.cls.empty() ? 0 : X.cls.back().first + X.cls.back().g.count; }
};
struct MixedState {           // what bp_rangeproof_verify_mixed_begin* leaves for *_finish
    bool active = false, reserved = false;     // reserved: queued on the reserved mix's graph; else verdicts already holds every verdict
    bp_gens *gens = nullptr;
    std::vector<uint8_t> verdicts;             // input order; the parameter codes until finish
    std::vector<uint32_t> live;                // per class of the mix
    std::vector<std::pair<uint32_t, uint32_t>> slots;      // (input index, slot) of every admitted proof
};
// Scratch of the fused single-proof path (rp_single.cuh), apart from RpScratch and the mixed arenas, so that a reserved verifier graph
// or a reserved mix on the same context never meets a buffer this path moved.  h_io (pinned): verdicts (RP_SINGLE_MAX_COUNT words), then
// the call's input block as it is uploaded.
struct SingleScratch {
    DevBuf in, raw, verdict, prog, pow2_tab;
    uint32_t prog_steps = 0; uint32_t prog_key[2] = {0, 0};       // (n, m) of the cached transcript step program
    PinnedBuf h_io;
    uint32_t smem_set = 0;                                          // bit k - RP_SINGLE_MIN_K: k_rp_single<k>'s shared-memory limit is raised
};
struct MsmPlan { int c = 0, W = 0; uint32_t nb = 0, heavy_min = 0; size_t segs = 0, n_buckets = 0, heavy_cap = 0; uint32_t n_msm = 0, T = 0; };
// A reserved LinearProof geometry (bp_linear_verify_reserve): n over one point set, up to g.count = capacity proofs per call.  Every buffer
// its graph reads is its own and only bp_linear_verify_reserve sizes them, so the blocking bp_linear_verify_batch may regrow the context's
// ln_* arenas, niels and MSM arena without moving anything the graph bakes in.  Inputs (aligned copies of the caller's), the front end's
// scratch as in bp_linear_verify_batch, the combined row, the reject path's rows, its MSM results (the combined one at 0), the verdicts
// and ctr = live, iteration, iterations, combined-check flag.  stage: the seed and live count of each call.
struct LinReserve {
    const bp_points *set = nullptr;
    lin_geom g{}; uint32_t tiles = 0, nch = 0, P = 0, T = 0;
    DevBuf tstate, proofs, C, b, par, raw, status, decbad, heads, tabs, part_g, part_b0, bf, scal, pidx, offsets, niels, rscal, rpidx, roffsets, results,
        verdict, ctr;
    MsmArena ar;
    StageRing stage;
    cudaGraphExec_t graph = nullptr; uint64_t graph_launches = 0;
    ~LinReserve() { if (graph) cudaGraphExecDestroy(graph); }
};
// A reserved mix of LinearProof lengths (bp_linear_verify_mixed_reserve) over one point set: X, the classes at capacity (linm_mix), and
// M, the mix as the planner kernels see it.  As with LinReserve, every buffer its graph reads is its own and only the reserve sizes them,
// apart from the planner's per-input scratch pl_*, which the graph never reads.  The device class table cls (each call's planner sets its
// live counts), the per-class parameters cpar (the live count of each class's reject loop), the gather table (slot order), the front
// end's arenas laid out as in bp_linear_verify_mixed, the combined row, the reject path's rows (the largest class slice), every class's
// MSM offsets (from roff[c] on), the MSM results (the combined one at 0), the verdicts in slot order, and ctr: (live, iteration,
// iterations, -) per class, then the combined-check flag.  stage: the seed of each call.
struct LinMixReserve {
    const bp_points *set = nullptr;
    linm_plan X; linm_mix_classes M{};
    std::vector<uint32_t> P, roff;                     // per class: proofs per reject-loop iteration, its first MSM offset in roffsets
    uint32_t T = 0;
    DevBuf cls, cpar, gather, tstate, proofs, C, b, par, raw, status, decbad, heads, tabs, part_g, part_b0, bf, scal, pidx, offsets, niels, rscal, rpidx,
        roffsets, results, verdict, ctr;
    DevBuf pl_code, pl_slot, pl_hist;                  // planner: code | class, rank then slot, per-block class counts
    MsmArena ar;
    StageRing stage;
    cudaGraphExec_t graph = nullptr; uint64_t graph_launches = 0;
    ~LinMixReserve() { if (graph) cudaGraphExecDestroy(graph); }
    uint32_t slots() const { return X.cls.back().first + X.cls.back().count; }
};

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
    // range-proof scratch: the verifier graph's own, and the host forms' copies of proofs, commitments and verdicts, which the graph
    // reads only through the parameter block
    RpScratch rp;
    DevBuf rp_proofs, rp_commit, rp_verdict, rp_tstates;           // rp_tstates: the per-proof transcript records of *_transcripts calls
    cudaStream_t cap_body = nullptr;                                // captures the body of the verifier graph's conditional per-batch pass
    DevBuf fb_part;                                                  // range-proof reject path: one-proof static sums
    SingleScratch sp;                                                // bp_rangeproof_verify_batch's fused single-proof path
    MixScratch mx;                                                   // bp_rangeproof_verify_mixed, calls that do not fit the reserved mix
    std::unique_ptr<MixReserve> mix;                                 // bp_rangeproof_verify_mixed_reserve
    std::unique_ptr<LinReserve> lin;                                 // bp_linear_verify_reserve
    std::unique_ptr<LinMixReserve> linm;                             // bp_linear_verify_mixed_reserve
    MixedState ms;
    // R1CS batches (bp_r1cs_verify_batch): inputs, per-proof heads and tables, G/H partial sums, combined row
    DevBuf r1_proofs, r1_term_off, r1_chal, r1_w, r1_in_scal, r1_in_pidx, r1_decbad, r1_heads, r1_tabs, r1_part, r1_scal, r1_pidx;
    // LinearProof batches (bp_linear_verify_batch): inputs, challenge rows, per-proof heads and tables, partial sums, combined row
    DevBuf ln_tstate, ln_proofs, ln_C, ln_b, ln_seed, ln_raw, ln_status, ln_decbad, ln_heads, ln_tabs, ln_part_g, ln_part_b0, ln_bf, ln_scal, ln_pidx;
    // bp_linear_verify_mixed, which lays its class-ordered proofs out on the ln_* arenas: the caller's buffers as they are (b | C | proofs |
    // transcript records) and the class and gather tables
    DevBuf lm_in, lm_meta;
    // MSM rows of every reject path: scalars, point map, offsets.  Shared: the R1CS and LinearProof entry points synchronise before they
    // return, and the range-proof re-check runs inside *_finish, while BUSY_CHECK keeps every other entry point out from *_begin on.
    DevBuf rk_scal, rk_pidx, rk_offsets;
    PinnedBuf h_verdict;                                             // the verdicts of a pending begin
    PinnedBuf h_flag;                                                // combined_ok[BP_MAX_GROUP_BATCHES] | batch_ok[BP_MAX_GROUP_BATCHES]
    StageRing stage;                                                 // the verifier's per-call parameter blocks
    VerifyState vs;
    size_t pidx_key[6] = {0, 0, 0, 0, 0, 0};                        // geometry the cached rp.pidx / rp.offsets were built for
    // reserved geometry: every arena sized, launch sequence captured as a CUDA graph, at rp.moves == graph_moves
    cudaGraphExec_t graph = nullptr; std::array<size_t, 6> graph_key{}; uint64_t graph_launches = 0, graph_moves = 0;
    // geometry reserved with bp_rangeproof_verify_reserve_exact: the exact graph (the launch sequence, then the device reject path), kept
    // like the graph above
    cudaGraphExec_t xgraph = nullptr; std::array<size_t, 6> xgraph_key{}; uint64_t xgraph_launches = 0, xgraph_moves = 0;
    ~bp_ctx() {                       // bp_ctx_destroy synchronises first; the members free the buffers after this
        if (graph) cudaGraphExecDestroy(graph);
        if (xgraph) cudaGraphExecDestroy(xgraph);
        if (ev_fork) cudaEventDestroy(ev_fork);
        if (ev_join) cudaEventDestroy(ev_join);
        if (aux) cudaStreamDestroy(aux);
        if (cap_body) cudaStreamDestroy(cap_body);
        if (own_stream) cudaStreamDestroy(stream);
    }
};

struct bp_gens {
    bp_ctx *ctx = nullptr; size_t cap = 0, parties = 0, n_points = 0;
    DevBuf d_table;                    // ge_niels [B_blinding, B, G[party][i].., H[party][i]..]
};

namespace {

#define CK(ctx, call)                                                                                  \
    do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { (ctx)->err = std::string(#call) + ": " + cudaGetErrorString(e_); return BP_ERR_CUDA; } } while (0)
// One kernel launch on stream s: launch() issues it and returns its error, which becomes "<what><error text>".  Counts the launch and,
// when profiling is enabled, brackets it with CUDA events on s.  LAUNCH(ctx, kid, kernel, grid, block, smem, stream, args...) is
// kernel<<<grid, block, smem, stream>>>(args...) through it.
template <class Launch>
int launch_profiled(bp_ctx *c, int kid, cudaStream_t s, const char *what, Launch launch) {
    ProfRec pr{kid, nullptr, nullptr};
    if (c->prof_on) { cudaEventCreate(&pr.a); cudaEventCreate(&pr.b); cudaEventRecord(pr.a, s); }
    cudaError_t e = launch();
    if (c->prof_on) { cudaEventRecord(pr.b, s); c->prof.push_back(pr); }
    c->launches++;
    if (e != cudaSuccess) { c->err = std::string(what) + cudaGetErrorString(e); return BP_ERR_CUDA; }
    return BP_OK;
}
#define LAUNCH(ctx, kid, kernel, grid, block, smem, stream, ...)                                       \
    do {                                                                                               \
        int lrc_ = launch_profiled((ctx), (kid), (stream), "kernel launch: ", [&] {                    \
            kernel<<<(grid), (block), (smem), (stream)>>>(__VA_ARGS__); return cudaGetLastError(); }); \
        if (lrc_) return lrc_;                                                                         \
    } while (0)

// the fallback of a pending begin/finish verification reads the context's scratch arenas: other entry points must not run in between
#define BUSY_CHECK(c) do { if ((c)->vs.active || (c)->ms.active) { (c)->err = (c)->vs.active ? "a range-proof verification is pending on this context: call bp_rangeproof_verify_group_finish first" \
    : "a mixed range-proof verification is pending on this context: call bp_rangeproof_verify_mixed_finish first"; return BP_ERR_INVALID_ARGUMENT; } } while (0)

inline unsigned blocks_for(size_t n, unsigned threads) { return (unsigned)((n + threads - 1) / threads); }
// block size of k_rp_scalars_sum, k_r1cs_gh_sum and k_lin_g_sum over n generator indices: one thread per index, at least one warp
inline unsigned sum_threads(uint32_t n) { return std::min<uint32_t>(128, std::max<uint32_t>(32, n)); }

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
    CK(ctx, ar.counts.ensure((p.n_buckets + 2 * MSM_SIZE_BINS + 4) * 4, ctx->stream)); CK(ctx, ar.starts.ensure(p.n_buckets * 4, ctx->stream)); CK(ctx, ar.cursor.ensure(p.n_buckets * 4, ctx->stream));
    CK(ctx, ar.order.ensure((p.n_buckets + p.heavy_cap) * 4, ctx->stream));
    CK(ctx, ar.sorted.ensure((size_t)p.T * p.W * 4, ctx->stream)); CK(ctx, ar.buckets.ensure(p.n_buckets * sizeof(ge_ext), ctx->stream)); CK(ctx, ar.wsums.ensure(p.segs * sizeof(ge_ext), ctx->stream));
    return BP_OK;
}
int msm_launch(bp_ctx *ctx, MsmArena &ar, const MsmArgs &a, const MsmPlan &p, ge_ext *d_results, cudaStream_t s) {
    const int c = p.c, W = p.W; const uint32_t nb = p.nb, heavy_min = p.heavy_min; const size_t segs = p.segs, n_buckets = p.n_buckets;
    uint32_t *size_hist = ar.counts.as<uint32_t>() + n_buckets, *bin_cursor = size_hist + MSM_SIZE_BINS, *heavy_n = bin_cursor + MSM_SIZE_BINS;
    uint32_t *heavy = ar.order.as<uint32_t>() + n_buckets;
    CK(ctx, cudaMemsetAsync(ar.counts.p, 0, (n_buckets + 2 * MSM_SIZE_BINS + 4) * 4, s));
    LAUNCH(ctx, KID_MSM_COUNT, k_msm_count, blocks_for(a.T, 256), 256, 0, s, a.d_scalars, a.d_offsets, a.n_msm, a.T, c, W, ar.counts.as<uint32_t>(), a.d_err, a.run);
    LAUNCH(ctx, KID_MSM_SCAN, k_msm_scan, (unsigned)segs, 256, 0, s, ar.counts.as<uint32_t>(), nb, ar.starts.as<uint32_t>(), ar.cursor.as<uint32_t>(), size_hist, a.run);
    LAUNCH(ctx, KID_MSM_SCAN, k_msm_order, blocks_for(n_buckets, 256), 256, 0, s, ar.counts.as<uint32_t>(), n_buckets, size_hist, bin_cursor, ar.order.as<uint32_t>(), heavy_min, heavy_n, heavy, a.run);
    LAUNCH(ctx, KID_MSM_SCATTER, k_msm_scatter, blocks_for(a.T, 256), 256, 0, s, a.d_scalars, a.d_offsets, a.n_msm, a.T, c, W, ar.cursor.as<uint32_t>(), ar.sorted.as<uint32_t>(), a.run);
    const int acc_split = msm_acc_split(msm_avg_terms(a.T, a.n_msm), nb, n_buckets);
    const unsigned heavy_blocks = (unsigned)std::min<size_t>(p.heavy_cap, (size_t)ctx->sm_count);
#define ACC_LAUNCH(SP) do { unsigned light_ = blocks_for(n_buckets * SP, MSM_ACC_THREADS); \
        LAUNCH(ctx, KID_MSM_ACCUMULATE, k_msm_accumulate<SP>, light_ + heavy_blocks, MSM_ACC_THREADS, 0, s, ar.starts.as<uint32_t>(), ar.cursor.as<uint32_t>(), ar.sorted.as<uint32_t>(), \
        a.d_offsets, ar.order.as<uint32_t>(), W, nb, n_buckets, a.d_point_idx, a.d_static, a.d_dynamic, ar.buckets.as<ge_ext>(), heavy_min, light_, heavy_n, heavy, a.run); } while (0)
    if (acc_split == 2) ACC_LAUNCH(2); else ACC_LAUNCH(1);
#undef ACC_LAUNCH
    // two warps per segment up to 2048 buckets (fewer scan / tree additions per useful bucket addition); eight for the wide windows of
    // large MSMs, where a segment's 16k-32k buckets would otherwise be 256-512 sequential additions per thread
    unsigned rthreads = nb >= 4096 ? 256 : nb >= 64 ? 64 : 32;
    LAUNCH(ctx, KID_MSM_REDUCE, k_msm_reduce, (unsigned)segs, rthreads, 0, s, ar.buckets.as<ge_ext>(), nb, ar.wsums.as<ge_ext>(), a.run);
    if (msm_use_combine4(a.n_msm))      // few MSMs: the Horner chain is pure latency -> four cooperating lanes per MSM
        LAUNCH(ctx, KID_MSM_COMBINE, k_msm_combine4, blocks_for(a.n_msm, 8), 32, 0, s, ar.wsums.as<ge_ext>(), a.n_msm, c, W, d_results, a.run);
    else
        LAUNCH(ctx, KID_MSM_COMBINE, k_msm_combine, blocks_for(a.n_msm, 32), 32, 0, s, ar.wsums.as<ge_ext>(), a.n_msm, c, W, d_results, a.run);
    return BP_OK;
}
int msm_core(bp_ctx *ctx, const MsmArgs &a, ge_ext *d_results) {       // generic arena
    if (a.T == 0) return BP_ERR_INVALID_ARGUMENT;
    MsmPlan p = msm_make_plan(a.T, a.n_msm, a.window > 0 ? a.window : ctx->msm_window);
    int rc = msm_ensure(ctx, ctx->ar_gen, p);
    if (rc) return rc;
    return msm_launch(ctx, ctx->ar_gen, a, p, d_results, ctx->stream);
}

// An undecodable point poisons the MSM that uses it (optional_multiscalar_mul -> None): flags[the MSM of t] |= 1 for every term t < T
// whose point did not decode.  That is ok[t] when pidx is null (one point per term), else ok[pidx[t] & 0x7fffffff] for the terms with
// BP_POINT_DYNAMIC set.  k_msm_status ranks the flag below a non-canonical scalar's.
__global__ void __launch_bounds__(256) k_flag_undecodable(const uint8_t *__restrict__ ok, const uint32_t *__restrict__ pidx, const uint32_t *__restrict__ offsets,
                                                          uint32_t n_msm, uint32_t T, uint32_t *__restrict__ flags) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= T) return;
    uint32_t i = t;
    if (pidx) { const uint32_t v = pidx[t]; if (!(v & BP_POINT_DYNAMIC)) return; i = v & 0x7fffffffu; }
    if (!ok[i]) atomicOr(flags + msm_of_term(offsets, n_msm, t), 1u);
}
__global__ void k_msm_status(const uint32_t *msm_err, uint32_t n_msm, uint8_t *status) {
    uint32_t m = blockIdx.x * blockDim.x + threadIdx.x;
    if (m >= n_msm) return;
    uint32_t e = msm_err[m];
    status[m] = (e & 2u) ? BP_ERR_NONCANONICAL_SCALAR : (e & 1u) ? BP_ERR_INVALID_POINT : BP_OK;
}
enum RpLayout { RP_BATCH_ROWS, RP_GROUP_ROW };
__global__ void k_rp_point_idx(rp_geom g, uint32_t gens_cap, uint32_t gens_parties, int layout, uint32_t dyn_base, uint32_t *out) {
    // RP_BATCH_ROWS, per batch: [S static | count*D dynamic] (g.nbatch batches);  RP_GROUP_ROW: [S static | g.nbatch*g.count*D dynamic].
    // Dynamic indices address the decompressed per-proof points: dyn_base + (first proof of the batch + q)*D + d (dyn_base: the first
    // point of a class of a mixed call, 0 otherwise).
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    size_t total = layout == RP_GROUP_ROW ? g.S + (size_t)g.nbatch * g.count * g.D : (size_t)g.nbatch * g.T;
    if (i >= total) return;
    uint32_t t, dyn;
    if (layout == RP_GROUP_ROW) { t = (uint32_t)min(i, (size_t)g.S); dyn = (uint32_t)(i - t); }
    else { uint32_t b = (uint32_t)(i / g.T); t = (uint32_t)(i % g.T); dyn = b * g.count * g.D + (t - g.S); if (t > g.S) t = g.S; }
    out[i] = t < g.S ? rp_static_slot(g, t, gens_cap, gens_parties) : BP_POINT_DYNAMIC | (dyn_base + dyn);
}
// one block per proof: the caller's offsets may have any alignment, so the copy is bytewise (a few MB per call)
__global__ void __launch_bounds__(128) k_rp_gather(const uint8_t *__restrict__ in_p, const uint8_t *__restrict__ in_c, const rp_gather *__restrict__ tab,
                                                  uint8_t *__restrict__ out_p, uint8_t *__restrict__ out_c) {
    const rp_gather e = tab[blockIdx.x];
    for (uint32_t b = threadIdx.x; b < e.len_p; b += blockDim.x) out_p[e.dst_p + b] = in_p[e.src_p + b];
    for (uint32_t b = threadIdx.x; b < e.len_c; b += blockDim.x) out_c[e.dst_c + b] = in_c[e.src_c + b];
}
// The device planner of a mixed call on device inputs (rp_mixed_device.cuh).  Step 1, one thread per proof: code_cls[i] = its parameter
// code | its class << 8, rank[i] = its rank among the proofs of its class earlier in its block, hist[block][c] = the block's class-c proofs.
__global__ void __launch_bounds__(RP_MIX_BLOCK) k_mix_admit(rp_mix_classes M, uint32_t count, const uint8_t *__restrict__ proofs, uint64_t proof_bytes,
                                                           const uint8_t *__restrict__ poff, const uint8_t *__restrict__ n_arr, uint64_t n_commit,
                                                           const uint8_t *__restrict__ coff, uint32_t *__restrict__ code_cls, uint32_t *__restrict__ rank,
                                                           uint32_t *__restrict__ hist) {
    __shared__ uint32_t s_wcnt[RP_MIX_WARPS][RP_MIXED_MAX_CLASSES];
    const uint32_t t = threadIdx.x, lane = t % 32, warp = t / 32, i = blockIdx.x * RP_MIX_BLOCK + t;
    for (uint32_t j = t; j < RP_MIX_WARPS * RP_MIXED_MAX_CLASSES; j += RP_MIX_BLOCK) s_wcnt[j / RP_MIXED_MAX_CLASSES][j % RP_MIXED_MAX_CLASSES] = 0;
    const uint32_t word = i < count ? rp_mix_admit(M, proofs, proof_bytes, poff, n_arr, n_commit, coff, i) : (uint32_t)RP_MIX_NO_CLASS << 8;
    if (i < count) code_cls[i] = word;
    const uint32_t cls = rp_mix_class(word);
    const uint32_t same = __match_any_sync(~0u, cls), wrank = __popc(same & ((1u << lane) - 1u));     // same-class lanes of this warp, those before it
    __syncthreads();
    if (cls != RP_MIX_NO_CLASS && wrank == 0) s_wcnt[warp][cls] = __popc(same);
    __syncthreads();
    if (cls != RP_MIX_NO_CLASS) rank[i] = rp_mix_rank_in_block(s_wcnt, warp, cls, wrank);
    if (t < M.C) hist[(size_t)blockIdx.x * M.C + t] = rp_mix_block_count(s_wcnt, t);
}
// Step 2, one block, warp c for class c: hist[b][c] becomes the class-c proofs of the blocks before b (exclusive scan over the nb blocks),
// and class c's live count, min(its proofs, its capacity), goes into its parameter block (uploaded before this kernel).
__global__ void k_mix_scan(rp_mix_classes M, uint32_t nb, uint32_t *__restrict__ hist, rp_params *__restrict__ par) {
    const uint32_t c = threadIdx.x / 32, lane = threadIdx.x % 32;
    if (c >= M.C) return;
    uint32_t run = 0;
    for (uint32_t b0 = 0; b0 < nb; b0 += 32) {
        const uint32_t b = b0 + lane, v = b < nb ? hist[(size_t)b * M.C + c] : 0u;
        uint32_t x = v;
        for (uint32_t d = 1; d < 32; d *= 2) { const uint32_t y = __shfl_up_sync(~0u, x, d); if (lane >= d) x += y; }
        if (b < nb) hist[(size_t)b * M.C + c] = run + x - v;
        run += __shfl_sync(~0u, x, 31);
    }
    if (lane == 0) par[c].live = min(run, M.cap[c]);
}
// Step 3, one thread per proof and per slot: slot[i] = proof i's slot (in place of its rank; RP_MIX_NO_SLOT when it has none), its gather
// entry and, with per-proof transcripts, its record at its slot of the mix's records.  Every slot this call leaves inert gets an empty
// gather entry, so that the gather copies nothing into it.
__global__ void __launch_bounds__(RP_MIX_BLOCK) k_mix_place(rp_mix_classes M, uint32_t count, uint32_t slots, const uint8_t *__restrict__ poff,
                                                           const uint8_t *__restrict__ coff, const uint8_t *__restrict__ records, const uint32_t *__restrict__ code_cls,
                                                           uint32_t *__restrict__ slot, const uint32_t *__restrict__ hist, const rp_params *__restrict__ par,
                                                           rp_gather *__restrict__ gather, uint8_t *__restrict__ tstates) {
    const uint32_t i = blockIdx.x * RP_MIX_BLOCK + threadIdx.x;
    if (i < slots) {
        const uint32_t c = rp_mix_class_of_slot(M, i);
        if (i - M.first[c] >= par[c].live) gather[i] = rp_gather{0, 0, 0, 0, 0, 0};
    }
    if (i >= count) return;
    const uint32_t cls = rp_mix_class(code_cls[i]);
    uint32_t s = RP_MIX_NO_SLOT;
    if (cls != RP_MIX_NO_CLASS) {
        const uint32_t q = hist[(size_t)blockIdx.x * M.C + cls] + slot[i];
        s = rp_mix_slot(M, cls, q);
        if (s != RP_MIX_NO_SLOT) {
            uint64_t po, len, co, m;
            rp_mix_bounds(poff, coff, ~0ull, ~0ull, i, &po, &len, &co, &m);        // admitted: in bounds
            gather[s] = rp_mix_gather_entry(M, cls, q, po, co);
            if (records)
                for (uint32_t b = 0; b < BP_TRANSCRIPT_BYTES; b++) tstates[(size_t)s * BP_TRANSCRIPT_BYTES + b] = records[(size_t)i * BP_TRANSCRIPT_BYTES + b];
        }
    }
    slot[i] = s;
}
// after the mix's graph: every proof's verdict in input order, its parameter code, its slot's verdict or BP_VERDICT_UNPLACED
__global__ void __launch_bounds__(RP_MIX_BLOCK) k_mix_verdicts(uint32_t count, const uint32_t *__restrict__ code_cls, const uint32_t *__restrict__ slot,
                                                              const uint32_t *__restrict__ verdict, uint32_t *__restrict__ out) {
    const uint32_t i = blockIdx.x * RP_MIX_BLOCK + threadIdx.x;
    if (i >= count) return;
    const uint32_t code = rp_mix_code(code_cls[i]), s = slot[i];
    out[i] = code != BP_PROOF_OK ? code : s == RP_MIX_NO_SLOT ? (uint32_t)BP_VERDICT_UNPLACED : verdict[s];
}
// condition of the class pass of a reserved mix's graph: set when the combined check's result is not the identity
__global__ void k_set_cond_unless_identity(const ge_ext *__restrict__ result, cudaGraphConditionalHandle cond) {
    cudaGraphSetConditional(cond, ge_is_identity(ld_ext(result)) ? 0u : 1u);
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

// the MSMs of `a` into ctx->results, then the outputs: M compressed results, and the per-MSM status when d_status is set
int msm_to_outputs(bp_ctx *ctx, const MsmArgs &a, uint8_t *d_outs, uint8_t *d_status) {
    int rc = msm_core(ctx, a, ctx->results.as<ge_ext>());
    if (rc) return rc;
    const uint32_t M = a.n_msm;
    LAUNCH(ctx, KID_COMPRESS, k_compress, blocks_for(M, 128), 128, 0, ctx->stream, ctx->results.as<ge_ext>(), M, d_outs);
    if (d_status) LAUNCH(ctx, KID_SMALL, k_msm_status, blocks_for(M, 128), 128, 0, ctx->stream, ctx->msm_err.as<uint32_t>(), M, d_status);
    return BP_OK;
}
// tail of the host-buffer MSM forms: download the n_msm outputs and, when status is set, their status, and synchronise
int msm_download(bp_ctx *ctx, size_t n_msm, uint8_t *outs, uint8_t *status) {
    CK(ctx, cudaMemcpyAsync(outs, ctx->outs.p, n_msm * 32, cudaMemcpyDeviceToHost, ctx->stream));
    if (status) CK(ctx, cudaMemcpyAsync(status, ctx->flags.p, n_msm, cudaMemcpyDeviceToHost, ctx->stream));
    CK(ctx, cudaStreamSynchronize(ctx->stream));
    return BP_OK;
}
// decompress n points from device memory into out and fail with BP_ERR_INVALID_POINT unless every one decodes; synchronises
int decompress_all(bp_ctx *ctx, const uint8_t *d_compressed, size_t n, ge_niels *out) {
    CK(ctx, ctx->ok.ensure(n, ctx->stream));
    LAUNCH(ctx, KID_DECOMPRESS, k_decompress, blocks_for(n, 128), 128, 0, ctx->stream, d_compressed, n, out, ctx->ok.as<uint8_t>());
    std::vector<uint8_t> ok(n);
    CK(ctx, cudaMemcpyAsync(ok.data(), ctx->ok.p, n, cudaMemcpyDeviceToHost, ctx->stream)); CK(ctx, cudaStreamSynchronize(ctx->stream));
    for (uint8_t v : ok) if (!v) return BP_ERR_INVALID_POINT;
    return BP_OK;
}

// what the first invalid point index of caller terms fails (a generator-table slot, or BP_POINT_DYNAMIC | an index below n_dyn), or nullptr
const char *point_index_error(const uint32_t *point_idx, size_t T, const bp_gens *gens, const uint8_t *dyn_points, size_t n_dyn) {
    for (size_t t = 0; t < T; t++) {
        const uint32_t v = point_idx[t];
        if (v & BP_POINT_DYNAMIC) { if ((v & 0x7fffffffu) >= n_dyn || !dyn_points) return "dynamic point index out of range"; }
        else if (!gens || v >= gens->n_points) return "generator-table slot out of range";
    }
    return nullptr;
}
// upload the n_dyn caller-supplied points and decompress them into c->niels, with c->ok[i] = whether point i decodes
int upload_dyn_points(bp_ctx *c, const uint8_t *dyn_points, size_t n_dyn) {
    CK(c, c->in_points.ensure(n_dyn * 32, c->stream)); CK(c, c->niels.ensure(n_dyn * sizeof(ge_niels), c->stream)); CK(c, c->ok.ensure(n_dyn, c->stream));
    CK(c, cudaMemcpyAsync(c->in_points.p, dyn_points, n_dyn * 32, cudaMemcpyHostToDevice, c->stream));
    LAUNCH(c, KID_DECOMPRESS, k_decompress, blocks_for(n_dyn, 128), 128, 0, c->stream, c->in_points.as<uint8_t>(), n_dyn, c->niels.as<ge_niels>(), c->ok.as<uint8_t>());
    return BP_OK;
}
// Reject path, `per` proofs at a time: rows(p0, cnt, a) sizes rk_scal / rk_pidx, queues the kernels that write the MSM rows of the proofs
// [p0, p0 + cnt) and sets `a` to their MSMs.  A proof that pre (its verdict before them) rejects keeps its code.  Synchronises.
template <class Rows>
int recheck_slices(bp_ctx *c, uint32_t np, uint32_t per, const std::vector<uint8_t> &pre, uint8_t *verdicts, Rows rows) {
    for (uint32_t p0 = 0; p0 < np; p0 += per) {
        const uint32_t cnt = std::min(per, np - p0);
        CK(c, c->rk_offsets.ensure(((size_t)cnt + 1) * 4, c->stream)); CK(c, c->results.ensure((size_t)cnt * sizeof(ge_ext), c->stream)); CK(c, c->outs.ensure((size_t)cnt * 32, c->stream));
        MsmArgs a{};
        int rc = rows(p0, cnt, a);
        if (rc) return rc;
        rc = msm_to_outputs(c, a, c->outs.as<uint8_t>(), nullptr);
        if (rc) return rc;
        std::vector<uint8_t> out((size_t)cnt * 32);
        CK(c, cudaMemcpyAsync(out.data(), c->outs.p, (size_t)cnt * 32, cudaMemcpyDeviceToHost, c->stream)); CK(c, cudaStreamSynchronize(c->stream));
        for (uint32_t r = 0; r < cnt; r++) verdicts[p0 + r] = pre[p0 + r] != BP_PROOF_OK ? pre[p0 + r] : bp_is_zero32(out.data() + 32 * r) ? BP_PROOF_OK : BP_PROOF_VERIFICATION_ERROR;
    }
    return BP_OK;
}
// Verdicts of a batch from its combined MSM's compressed result: the identity accepts every proof in the combination, so each proof
// gets its verdict before the MSM, pre (which rejects a proof left out of it); otherwise recheck() decides every proof by its own MSM.
template <class Recheck>
int combined_verdicts(const uint8_t combined[32], const std::vector<uint8_t> &pre, uint8_t *verdicts, Recheck recheck) {
    if (bp_is_zero32(combined)) { memcpy(verdicts, pre.data(), pre.size()); return BP_OK; }
    return recheck();
}
// Caller-owned device buffers.  The MSM kernels stage scalars and compressed points with one bulk copy per block (tma_stage_tile),
// which needs a 16-byte-aligned source, and write 32-byte results with 16-byte stores (st32); offsets and range-proof verdicts are
// 32-bit words.  A misaligned buffer would fault on the device and lose the context, so the entry points refuse it instead.
inline bool is_aligned(const void *p, uintptr_t a) { return ((uintptr_t)p & (a - 1)) == 0; }
// the batching-weight seed of a verifier call: the caller's 32 bytes, or 32 fresh ones from the OS when seed is null
int draw_seed(bp_ctx *c, const uint8_t *seed, uint8_t out[32]) {
    if (seed) memcpy(out, seed, 32);
    else if (getrandom(out, 32, 0) != 32) { c->err = "getrandom failed"; return BP_ERR_CUDA; }
    return BP_OK;
}
// Capture what launch() queues on c->stream into *exec, replacing its graph, with profiling off (graph nodes are not timed); *launches
// gets the launches it counted.  c->prof_on and c->launches are left as they were, whether or not the capture succeeds.
template <class Launch>
int graph_capture(bp_ctx *c, cudaGraphExec_t *exec, uint64_t *launches, Launch launch) {
    if (*exec) { cudaGraphExecDestroy(*exec); *exec = nullptr; }
    CK(c, cudaStreamBeginCapture(c->stream, cudaStreamCaptureModeThreadLocal));
    const bool prof = c->prof_on; const uint64_t l0 = c->launches;
    c->prof_on = false;
    const int rc = launch();
    cudaGraph_t graph = nullptr;
    cudaError_t e = cudaStreamEndCapture(c->stream, &graph);
    c->prof_on = prof;
    *launches = c->launches - l0; c->launches = l0;
    if (rc) { if (graph) cudaGraphDestroy(graph); return rc; }
    if (e != cudaSuccess) { c->err = std::string("cudaStreamEndCapture: ") + cudaGetErrorString(e); return BP_ERR_CUDA; }
    e = cudaGraphInstantiate(exec, graph, 0);
    cudaGraphDestroy(graph);
    if (e != cudaSuccess) { *exec = nullptr; c->err = std::string("cudaGraphInstantiate: ") + cudaGetErrorString(e); return BP_ERR_CUDA; }
    return BP_OK;
}
// A conditional node (IF or WHILE) in the graph being captured on c->stream, in two steps.  graph_cond creates its handle, for a kernel the
// caller then queues to set it; graph_body adds the node after that kernel and captures body(c->cap_body) into it ("what" names the body in
// the error text).  The handle resets to 0 at every launch of the graph, so no call sees the decision of the one before.
int graph_cond(bp_ctx *c, cudaGraphConditionalHandle *cond) {
    cudaStreamCaptureStatus cs; cudaGraph_t cg = nullptr; const cudaGraphNode_t *deps = nullptr; size_t nd = 0;
    CK(c, cudaStreamGetCaptureInfo(c->stream, &cs, nullptr, &cg, &deps, &nd));
    CK(c, cudaGraphConditionalHandleCreate(cond, cg, 0, cudaGraphCondAssignDefault));
    return BP_OK;
}
template <class Body>
int graph_body(bp_ctx *c, cudaGraphConditionalHandle cond, cudaGraphConditionalNodeType type, const char *what, Body body) {
    cudaStreamCaptureStatus cs; cudaGraph_t cg = nullptr; const cudaGraphNode_t *deps = nullptr; size_t nd = 0;
    CK(c, cudaStreamGetCaptureInfo(c->stream, &cs, nullptr, &cg, &deps, &nd));
    cudaGraphNodeParams np{};
    np.type = cudaGraphNodeTypeConditional; np.conditional.handle = cond; np.conditional.type = type; np.conditional.size = 1;
    cudaGraphNode_t node = nullptr;
    CK(c, cudaGraphAddNode(&node, cg, deps, nd, &np));
    CK(c, cudaStreamUpdateCaptureDependencies(c->stream, &node, 1, cudaStreamSetCaptureDependencies));
    CK(c, cudaStreamBeginCaptureToGraph(c->cap_body, np.conditional.phGraph_out[0], nullptr, nullptr, 0, cudaStreamCaptureModeThreadLocal));
    const int rc = body(c->cap_body);
    cudaGraph_t g = nullptr;
    cudaError_t e = cudaStreamEndCapture(c->cap_body, &g);
    if (rc) return rc;
    if (e != cudaSuccess) { c->err = std::string("cudaStreamEndCapture(") + what + "): " + cudaGetErrorString(e); return BP_ERR_CUDA; }
    return BP_OK;
}

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
    std::unique_ptr<bp_ctx> c(new bp_ctx());          // a failure below releases what was made so far
    c->device = device; c->sm_count = prop.multiProcessorCount > 0 ? prop.multiProcessorCount : 132;
    if (stream) c->stream = (cudaStream_t)stream;
    else { if (cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking) != cudaSuccess) return BP_ERR_CUDA; c->own_stream = true; }
    if (c->h_flag.ensure(2 * BP_MAX_GROUP_BATCHES * 4) != cudaSuccess || c->stage.init(sizeof(rp_params)) != cudaSuccess ||
        cudaStreamCreateWithFlags(&c->aux, cudaStreamNonBlocking) != cudaSuccess || cudaStreamCreateWithFlags(&c->cap_body, cudaStreamNonBlocking) != cudaSuccess ||
        cudaEventCreateWithFlags(&c->ev_fork, cudaEventDisableTiming) != cudaSuccess || cudaEventCreateWithFlags(&c->ev_join, cudaEventDisableTiming) != cudaSuccess)
        return BP_ERR_CUDA;
    // k_rp_decompress stages the whole proofs its block touches and the commitments of its own points, at most RP_DEC_THREADS of them
    // (rp_dec_smem_bytes, rp.cuh): at most 8 KB over every geometry rp_param_verdict admits, whatever m is
    cudaFuncSetAttribute(k_rp_decompress, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)rp_dec_smem_max());
    *out = c.release();
    return BP_OK;
}
void bp_ctx_destroy(bp_ctx *c) {
    if (!c) return;
    cudaSetDevice(c->device);
    cudaStreamSynchronize(c->stream);
    if (c->aux) cudaStreamSynchronize(c->aux);
    delete c;                   // frees every buffer, event and stream it owns
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
    int rc = upload_dyn_points(c, points, n);
    if (rc) return rc;
    CK(c, cudaMemcpyAsync(ok, c->ok.p, n, cudaMemcpyDeviceToHost, c->stream));
    CK(c, cudaStreamSynchronize(c->stream));
    return BP_OK;
}

int bp_from_uniform_bytes_batch(bp_ctx *c, const uint8_t *uniform, size_t n, uint8_t *points_out) {
    if (!c || !uniform || !points_out) return BP_ERR_INVALID_ARGUMENT;
    BUSY_CHECK(c);
    if (n == 0) return BP_OK;
    CK(c, cudaSetDevice(c->device));
    CK(c, c->in_points.ensure(n * 64, c->stream)); CK(c, c->outs.ensure(n * 32, c->stream));
    CK(c, cudaMemcpyAsync(c->in_points.p, uniform, n * 64, cudaMemcpyHostToDevice, c->stream));
    LAUNCH(c, KID_FROM_UNIFORM, k_from_uniform, blocks_for(n, 128), 128, 0, c->stream, c->in_points.as<uint8_t>(), n, nullptr, c->outs.as<uint8_t>());
    CK(c, cudaMemcpyAsync(points_out, c->outs.p, n * 32, cudaMemcpyDeviceToHost, c->stream));
    CK(c, cudaStreamSynchronize(c->stream));
    return BP_OK;
}

int bp_msm_batch_device(bp_ctx *c, const void *d_scalars, const void *d_points, const void *d_offsets_u32, size_t n_msm, size_t total_terms,
                        void *d_outs, void *d_status) {
    if (!c || !d_scalars || !d_points || !d_offsets_u32 || !d_outs || n_msm == 0) return BP_ERR_INVALID_ARGUMENT;
    if (total_terms == 0 || total_terms >= (1u << 31) || n_msm >= (1u << 31)) return BP_ERR_INVALID_ARGUMENT;
    if (!is_aligned(d_scalars, 16) || !is_aligned(d_points, 16) || !is_aligned(d_outs, 16) || !is_aligned(d_offsets_u32, 4)) {
        c->err = "bp_msm_batch_device: d_scalars, d_points and d_outs must be 16-byte aligned, d_offsets_u32 4-byte aligned"; return BP_ERR_INVALID_ARGUMENT;
    }
    BUSY_CHECK(c);
    CK(c, cudaSetDevice(c->device));
    uint32_t T = (uint32_t)total_terms, M = (uint32_t)n_msm;
    CK(c, c->niels.ensure((size_t)T * sizeof(ge_niels), c->stream)); CK(c, c->ok.ensure(T, c->stream)); CK(c, c->msm_err.ensure((size_t)M * 4, c->stream)); CK(c, c->results.ensure((size_t)M * sizeof(ge_ext), c->stream));
    cudaStream_t s = c->stream;
    CK(c, cudaMemsetAsync(c->msm_err.p, 0, (size_t)M * 4, s));
    LAUNCH(c, KID_DECOMPRESS, k_decompress, blocks_for(T, 128), 128, 0, s, (const uint8_t *)d_points, T, c->niels.as<ge_niels>(), c->ok.as<uint8_t>());
    LAUNCH(c, KID_SMALL, k_flag_undecodable, blocks_for(T, 256), 256, 0, s, c->ok.as<uint8_t>(), nullptr, (const uint32_t *)d_offsets_u32, M, T, c->msm_err.as<uint32_t>());
    MsmArgs a{(const uint8_t *)d_scalars, (const uint32_t *)d_offsets_u32, M, T, nullptr, nullptr, c->niels.as<ge_niels>(), c->msm_err.as<uint32_t>(), 0};
    return msm_to_outputs(c, a, (uint8_t *)d_outs, (uint8_t *)d_status);
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
    if (!scalars || !points || n_msm >= (1u << 31)) return BP_ERR_INVALID_ARGUMENT;
    BUSY_CHECK(c);
    std::vector<uint32_t> off32(n_msm + 1);
    for (size_t j = 0; j <= n_msm; j++) off32[j] = (uint32_t)offsets[j];
    CK(c, c->in_scalars.ensure(T * 32, c->stream)); CK(c, c->in_points.ensure(T * 32, c->stream)); CK(c, c->in_offsets.ensure((n_msm + 1) * 4, c->stream));
    CK(c, c->outs.ensure(n_msm * 32, c->stream)); CK(c, c->flags.ensure(n_msm, c->stream));
    cudaStream_t s = c->stream;
    CK(c, cudaMemcpyAsync(c->in_scalars.p, scalars, T * 32, cudaMemcpyHostToDevice, s));
    CK(c, cudaMemcpyAsync(c->in_points.p, points, T * 32, cudaMemcpyHostToDevice, s));
    CK(c, cudaMemcpyAsync(c->in_offsets.p, off32.data(), (n_msm + 1) * 4, cudaMemcpyHostToDevice, s));
    int rc = bp_msm_batch_device(c, c->in_scalars.p, c->in_points.p, c->in_offsets.p, n_msm, T, c->outs.p, c->flags.p);
    if (rc) return rc;
    return msm_download(c, n_msm, outs, status);
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
    CK(c, c->in_points.ensure(n * 32, c->stream)); CK(c, c->outs.ensure(n * 128, c->stream)); CK(c, c->ok.ensure(n, c->stream));
    CK(c, cudaMemcpyAsync(c->in_points.p, points, n * 32, cudaMemcpyHostToDevice, c->stream));
    LAUNCH(c, KID_DECOMPRESS, k_decompress_xyzt, blocks_for(n, 128), 128, 0, c->stream, c->in_points.as<uint8_t>(), n, c->outs.as<uint8_t>(), c->ok.as<uint8_t>());
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
    CK(c, c->in_points.ensure(n * 128, c->stream)); CK(c, c->outs.ensure(n * 32, c->stream));
    CK(c, cudaMemcpyAsync(c->in_points.p, xyzt, n * 128, cudaMemcpyHostToDevice, c->stream));
    LAUNCH(c, KID_COMPRESS, k_compress_xyzt, blocks_for(n, 128), 128, 0, c->stream, c->in_points.as<uint8_t>(), n, c->outs.as<uint8_t>());
    CK(c, cudaMemcpyAsync(points_out, c->outs.p, n * 32, cudaMemcpyDeviceToHost, c->stream));
    CK(c, cudaStreamSynchronize(c->stream));
    return BP_OK;
}

// ---------------------------------------------------------------------------------------------- resident point sets (decompressed once, reused by many MSMs)
}  // extern "C"
struct bp_points {
    bp_ctx *ctx = nullptr; size_t n = 0;
    DevBuf d_pts;                       // ge_niels [n]
    DevBuf d_enc;                       // the n x 32 B encodings it was created from: canonical, as every point decoded
    DevBuf d_idx; size_t idx_T = 0, idx_len = 0;         // term -> point map of the last geometry (k_iota_mod)
};
extern "C" {
static int points_from_device(bp_ctx *c, const uint8_t *d_compressed, size_t n, bp_points **out) {
    std::unique_ptr<bp_points> h(new bp_points()); h->ctx = c; h->n = n;
    CK(c, h->d_pts.alloc(n * sizeof(ge_niels))); CK(c, h->d_enc.alloc(n * 32));
    CK(c, cudaMemcpyAsync(h->d_enc.p, d_compressed, n * 32, cudaMemcpyDeviceToDevice, c->stream));     // decompress_all synchronises
    int rc = decompress_all(c, d_compressed, n, h->d_pts.as<ge_niels>());
    if (rc) return rc;
    *out = h.release(); return BP_OK;
}
int bp_points_create(bp_ctx *c, const uint8_t *points, size_t n, bp_points **out) {
    if (!c || !points || !out || n == 0 || n >= (1u << 31)) return BP_ERR_INVALID_ARGUMENT;
    BUSY_CHECK(c);
    CK(c, cudaSetDevice(c->device));
    CK(c, c->in_points.ensure(n * 32, c->stream));
    CK(c, cudaMemcpyAsync(c->in_points.p, points, n * 32, cudaMemcpyHostToDevice, c->stream));
    return points_from_device(c, c->in_points.as<uint8_t>(), n, out);
}
int bp_points_create_device(bp_ctx *c, const void *d_points, size_t n, bp_points **out) {
    if (!c || !d_points || !out || n == 0 || n >= (1u << 31)) return BP_ERR_INVALID_ARGUMENT;
    if (!is_aligned(d_points, 16)) { c->err = "bp_points_create_device: d_points must be 16-byte aligned"; return BP_ERR_INVALID_ARGUMENT; }
    BUSY_CHECK(c);
    CK(c, cudaSetDevice(c->device));
    return points_from_device(c, (const uint8_t *)d_points, n, out);
}
// destroying the set of a LinearProof reservation or mix ends it, so that no later call replays a graph that reads the freed points
void bp_points_destroy(bp_points *h) {
    if (!h) return;
    cudaSetDevice(h->ctx->device); cudaStreamSynchronize(h->ctx->stream);
    if (h->ctx->lin && h->ctx->lin->set == h) h->ctx->lin.reset();
    if (h->ctx->linm && h->ctx->linm->set == h) h->ctx->linm.reset();
    delete h;
}
size_t bp_points_count(const bp_points *h) { return h ? h->n : 0; }

// n_msm MSMs of `terms` terms each over the first `terms` points of the set (MSM j uses scalars[j*terms .. (j+1)*terms)); device pointers,
// nothing synchronised.  No decompression on this path: 32 B of scalar per term is all that is read from the caller.
int bp_msm_points_device(bp_ctx *c, bp_points *h, const void *d_scalars, size_t n_msm, size_t terms, void *d_outs, void *d_status) {
    if (!c || !h || !d_scalars || !d_outs || n_msm == 0 || terms == 0 || terms > h->n || n_msm * terms >= (1u << 31)) return BP_ERR_INVALID_ARGUMENT;
    if (!is_aligned(d_scalars, 16) || !is_aligned(d_outs, 16)) { c->err = "bp_msm_points_device: d_scalars and d_outs must be 16-byte aligned"; return BP_ERR_INVALID_ARGUMENT; }
    BUSY_CHECK(c);
    CK(c, cudaSetDevice(c->device));
    uint32_t T = (uint32_t)(n_msm * terms), M = (uint32_t)n_msm;
    cudaStream_t s = c->stream;
    if (h->idx_T < T || h->idx_len != terms) {
        h->idx_T = 0;
        CK(c, h->d_idx.ensure((size_t)T * 4, s));
        LAUNCH(c, KID_SMALL, k_iota_mod, blocks_for(T, 256), 256, 0, s, T, (uint32_t)terms, h->d_idx.as<uint32_t>());
        h->idx_T = T; h->idx_len = terms;
    }
    CK(c, c->in_offsets.ensure(((size_t)M + 1) * 4, c->stream)); CK(c, c->msm_err.ensure((size_t)M * 4, c->stream)); CK(c, c->results.ensure((size_t)M * sizeof(ge_ext), c->stream));
    LAUNCH(c, KID_SMALL, k_fill_offsets, blocks_for((size_t)M + 1, 256), 256, 0, s, M, (uint32_t)terms, c->in_offsets.as<uint32_t>());
    CK(c, cudaMemsetAsync(c->msm_err.p, 0, (size_t)M * 4, s));
    MsmArgs a{(const uint8_t *)d_scalars, c->in_offsets.as<uint32_t>(), M, T, h->d_idx.as<uint32_t>(), h->d_pts.as<ge_niels>(), nullptr, c->msm_err.as<uint32_t>(), 0};
    return msm_to_outputs(c, a, (uint8_t *)d_outs, (uint8_t *)d_status);
}
// host-buffer form (pinned memory recommended): H2D of the scalars, the MSMs, D2H of the 32-byte results; synchronises
int bp_msm_points(bp_ctx *c, bp_points *h, const uint8_t *scalars, size_t n_msm, size_t terms, uint8_t *outs, uint8_t *status) {
    if (!c || !h || !scalars || !outs || n_msm == 0 || terms == 0 || terms > h->n || n_msm * terms >= (1u << 31)) return BP_ERR_INVALID_ARGUMENT;
    BUSY_CHECK(c);
    CK(c, cudaSetDevice(c->device));
    size_t T = n_msm * terms;
    CK(c, c->in_scalars.ensure(T * 32, c->stream)); CK(c, c->outs.ensure(n_msm * 32, c->stream)); CK(c, c->flags.ensure(n_msm, c->stream));
    CK(c, cudaMemcpyAsync(c->in_scalars.p, scalars, T * 32, cudaMemcpyHostToDevice, c->stream));
    int rc = bp_msm_points_device(c, h, c->in_scalars.p, n_msm, terms, c->outs.p, c->flags.p);
    if (rc) return rc;
    return msm_download(c, n_msm, outs, status);
}

// ---------------------------------------------------------------------------------------------- generators
static int gens_alloc(bp_ctx *c, size_t cap, size_t parties, bp_gens **out) {
    if (!c || !out || cap == 0 || parties == 0) return BP_ERR_INVALID_ARGUMENT;
    CK(c, cudaSetDevice(c->device));
    std::unique_ptr<bp_gens> g(new bp_gens());
    g->ctx = c; g->cap = cap; g->parties = parties; g->n_points = 2 + 2 * cap * parties;
    CK(c, g->d_table.alloc(g->n_points * sizeof(ge_niels)));
    *out = g.release();
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
    CK(c, c->in_points.ensure(uni.size(), c->stream)); CK(c, c->in_scalars.ensure(32, c->stream));
    cudaStream_t s = c->stream;
    CK(c, cudaMemcpyAsync(c->in_points.p, uni.data(), uni.size(), cudaMemcpyHostToDevice, s));
    CK(c, cudaMemcpyAsync(c->in_scalars.p, BASEPOINT, 32, cudaMemcpyHostToDevice, s));
    LAUNCH(c, KID_FROM_UNIFORM, k_from_uniform, blocks_for(g->n_points, 128), 128, 0, s, c->in_points.as<uint8_t>(), g->n_points, g->d_table.as<ge_niels>(), nullptr);
    LAUNCH(c, KID_DECOMPRESS, k_decompress, 1, 128, 0, s, c->in_scalars.as<uint8_t>(), 1, g->d_table.as<ge_niels>() + 1, nullptr);
    CK(c, cudaStreamSynchronize(s));
    return BP_OK;
}
void bp_gens_destroy(bp_gens *g) { if (!g) return; cudaSetDevice(g->ctx->device); delete g; }
int bp_gens_device_table(bp_gens *g, void **d_table, size_t *bytes) {
    if (!g || !d_table || !bytes) return BP_ERR_INVALID_ARGUMENT;
    *d_table = g->d_table.p; *bytes = g->n_points * sizeof(ge_niels); return BP_OK;
}
int bp_gens_get(bp_gens *g, int which, size_t party, size_t index, uint8_t out[32]) {
    if (!g || !out) return BP_ERR_INVALID_ARGUMENT;
    bp_ctx *c = g->ctx; size_t slot;
    if (which == 2) slot = 1; else if (which == 3) slot = 0;
    else if ((which == 0 || which == 1) && party < g->parties && index < g->cap) slot = bp_gens_slot(which, party, index, g->cap, g->parties);
    else return BP_ERR_INVALID_ARGUMENT;
    CK(c, cudaSetDevice(c->device)); CK(c, c->outs.ensure(32, c->stream));
    LAUNCH(c, KID_SMALL, k_niels_to_compressed, 1, 32, 0, c->stream, g->d_table.as<ge_niels>() + slot, 1, c->outs.as<uint8_t>());
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
static bool rp_set_group(rp_geom *g, size_t count, size_t n_batches) {
    if (count == 0 || n_batches == 0 || n_batches > BP_MAX_GROUP_BATCHES || count >= (1u << 24)) return false;
    size_t T = (size_t)g->S + count * g->D;
    if (T * n_batches >= (1u << 31) || count * n_batches >= (1u << 24)) return false;
    g->count = (uint32_t)count; g->nbatch = (uint32_t)n_batches; g->T = (uint32_t)T;
    return true;
}

// terms of a launch group's combined MSM: [S static | nbatch*count*D dynamic] (kernels.cuh, range-proof section)
static uint32_t rp_group_terms(const rp_geom &g) { return g.S + g.nbatch * g.count * g.D; }
// 2^e (e < 64) in Montgomery form, the head's pow2 argument: computed once per buffer with the host build of sc.cuh
static int rp_pow2_table(bp_ctx *c, DevBuf &tab_buf) {
    if (tab_buf.p) return BP_OK;
    std::vector<sc> tab(64);
    for (int e = 0; e < 64; e++) tab[e] = sc_mont_from_u64(1ULL << e);
    CK(c, tab_buf.ensure(64 * sizeof(sc), c->stream));
    CK(c, cudaMemcpyAsync(tab_buf.p, tab.data(), 64 * sizeof(sc), cudaMemcpyHostToDevice, c->stream)); CK(c, cudaStreamSynchronize(c->stream));
    return BP_OK;
}
// geometry g's transcript step program into buf (grown to fit) and its step count into *steps; synchronises, so that the host copy may go
static int rp_upload_program(bp_ctx *c, DevBuf &buf, const rp_geom &g, uint32_t *steps) {
    const std::vector<rp_tr_step> prog = rp_tr_program(g.n, g.m, g.k);
    CK(c, buf.ensure(prog.size() * sizeof(rp_tr_step), c->stream));
    CK(c, cudaMemcpyAsync(buf.p, prog.data(), prog.size() * sizeof(rp_tr_step), cudaMemcpyHostToDevice, c->stream)); CK(c, cudaStreamSynchronize(c->stream));
    *steps = (uint32_t)prog.size();
    return BP_OK;
}
// every arena of one launch group but the step program (rp_build_maps), grow-only; after these nothing on the verification path allocates
static int rp_ensure(bp_ctx *c, const rp_geom &g) {
    size_t total = (size_t)g.count * g.nbatch, TT = (size_t)g.T * g.nbatch, TG = rp_group_terms(g);
    RpScratch &r = c->rp;
    CK(c, r.par.ensure(sizeof(rp_params), c->stream));
    CK(c, r.scalars.ensure(TG * 32, c->stream));
    CK(c, r.part.ensure((size_t)g.nbatch * ((g.count + RP_CHUNK - 1) / RP_CHUNK) * g.S * sizeof(sc), c->stream));
    CK(c, r.status.ensure(total * 4, c->stream)); CK(c, r.decbad.ensure(total * 4, c->stream)); CK(c, r.niels.ensure(total * g.D * sizeof(ge_niels), c->stream));
    CK(c, r.pidx.ensure(TG * 4, c->stream)); CK(c, r.offsets.ensure(2 * 4, c->stream)); CK(c, r.results.ensure(((size_t)g.nbatch + 1) * sizeof(ge_ext), c->stream)); CK(c, r.run.ensure(4, c->stream));
    CK(c, r.batch_ok.ensure((size_t)g.nbatch * 4, c->stream)); CK(c, r.combined.ensure((size_t)g.nbatch * 4, c->stream));
    CK(c, r.chal.ensure(total * sizeof(rp_lean_head), c->stream)); CK(c, r.tabs.ensure(rp_tab_slice(total, g.k, g.m) * sizeof(sc), c->stream));
    CK(c, r.raw.ensure(total * (RP_RAW_U + g.k) * 64, c->stream));
    CK(c, c->h_verdict.ensure(total * 4));
    int rc = rp_pow2_table(c, r.pow2_tab);
    if (rc) return rc;
    if (g.nbatch > 1) {       // the per-batch pass; its MSM shares the arena with the group MSM (they run one after the other)
        CK(c, r.bstatic.ensure((size_t)g.nbatch * g.S * 32, c->stream)); CK(c, r.bscal.ensure(TT * 32, c->stream)); CK(c, r.bpidx.ensure(TT * 4, c->stream));
        CK(c, r.boffsets.ensure(((size_t)g.nbatch + 1) * 4, c->stream));
        rc = msm_ensure(c, r.ar, msm_make_plan((uint32_t)TT, g.nbatch, 0));
        if (rc) return rc;
    }
    return msm_ensure(c, r.ar, msm_make_plan((uint32_t)TG, 1, 0));
}
// term -> point maps and MSM offsets of the group MSM and of the per-batch MSMs, and the transcript step program: depend only on the
// geometry, rebuilt when it changes
static int rp_build_maps(bp_ctx *c, bp_gens *gens, const rp_geom &g) {
    size_t key[6] = {g.n, g.m, g.count, g.nbatch, gens->cap, gens->parties};
    if (memcmp(key, c->pidx_key, sizeof key) == 0) return BP_OK;
    cudaStream_t s = c->stream;
    int rc = rp_upload_program(c, c->rp.prog, g, &c->rp.prog_steps);
    if (rc) return rc;
    const uint32_t TG = rp_group_terms(g);
    LAUNCH(c, KID_SMALL, k_rp_point_idx, blocks_for(TG, 256), 256, 0, s, g, (uint32_t)gens->cap, (uint32_t)gens->parties, RP_GROUP_ROW, 0u, c->rp.pidx.as<uint32_t>());
    LAUNCH(c, KID_SMALL, k_fill_offsets, 1, 256, 0, s, 1, TG, c->rp.offsets.as<uint32_t>());
    if (g.nbatch > 1) {
        LAUNCH(c, KID_SMALL, k_rp_point_idx, blocks_for((size_t)g.T * g.nbatch, 256), 256, 0, s, g, (uint32_t)gens->cap, (uint32_t)gens->parties, RP_BATCH_ROWS,
               0u, c->rp.bpidx.as<uint32_t>());
        LAUNCH(c, KID_SMALL, k_fill_offsets, blocks_for((size_t)g.nbatch + 1, 256), 256, 0, s, g.nbatch, g.T, c->rp.boffsets.as<uint32_t>());
    }
    memcpy(c->pidx_key, key, sizeof key);
    return BP_OK;
}
// a parameter block for device address d_block; exactly one of h_transcript (every proof's tstate) and d_records (one per proof) is set
static void rp_fill_params(rp_params &pa, const rp_params *d_block, const uint8_t *h_transcript, const uint8_t *d_records, const uint8_t seed[32],
                           const uint8_t *d_proofs, const uint8_t *d_commit, uint32_t *d_verdict, uint32_t live) {
    memset(&pa, 0, sizeof pa);
    if (h_transcript) memcpy(pa.tstate, h_transcript, BP_TRANSCRIPT_BYTES);
    pa.tstates = d_records ? d_records : reinterpret_cast<const uint8_t *>(d_block) + offsetof(rp_params, tstate);
    pa.tstride = d_records ? BP_TRANSCRIPT_BYTES : 0;
    memcpy(pa.seed, seed, 32);
    pa.proofs = d_proofs; pa.commitments = d_commit; pa.verdict = d_verdict; pa.live = live;
}

// Per-batch pass of a launch group whose combined check failed: every batch's own combined MSM and verdicts, as before the group
// check existed.  run = the device gate k_rp_verdict_group sets (direct launches: every kernel returns at once when the group
// passed), or nullptr inside the body of the captured graph's IF node, which runs only when the group failed.
static int rp_batch_pass(bp_ctx *c, bp_gens *gens, const rp_geom &g, const uint32_t *run, cudaStream_t s) {
    RpScratch &r = c->rp;
    const uint32_t TT = g.T * g.nbatch;
    LAUNCH(c, KID_RP_BATCH_ROWS, k_rp_batch_rows, blocks_for(TT, 256), 256, 0, s, run, r.bstatic.as<uint8_t>(), r.scalars.as<uint8_t>(), g, r.bscal.as<uint8_t>());
    MsmArgs a{r.bscal.as<uint8_t>(), r.boffsets.as<uint32_t>(), g.nbatch, TT, r.bpidx.as<uint32_t>(), gens->d_table.as<ge_niels>(), r.niels.as<ge_niels>(), nullptr, 0, run};
    int rc = msm_launch(c, r.ar, a, msm_make_plan(a.T, a.n_msm, 0), r.results.as<ge_ext>(), s);
    if (rc) return rc;
    LAUNCH(c, KID_RP_VERDICT_BATCH, k_rp_verdict_batch, g.nbatch, 256, 0, s, r.status.as<uint32_t>(), r.decbad.as<uint32_t>(), r.results.as<ge_ext>(), g, r.par.as<rp_params>(),
           r.batch_ok.as<uint32_t>(), r.combined.as<uint32_t>(), run);
    return BP_OK;
}

// What the front end and the reject path use of one verified geometry: its scalar array (static row first), per-proof status, dec_bad
// and heads from its first proof on, head tables, chunk partial sums and decompressed per-proof points (dynamic index 0 = its first
// proof's first point).  The fixed-geometry verifier passes its own scratch (rp_view); a mixed call passes one class's slices.
struct RpView { uint8_t *scalars; uint32_t *status, *decbad; rp_lean_head *chal; sc *tabs, *part; ge_niels *niels; };
static RpView rp_view(RpScratch &r) {
    return {r.scalars.as<uint8_t>(), r.status.as<uint32_t>(), r.decbad.as<uint32_t>(), r.chal.as<rp_lean_head>(), r.tabs.as<sc>(), r.part.as<sc>(), r.niels.as<ge_niels>()};
}
// One segment of the front end: `count` proofs of geometry g (count = g.count * g.nbatch) read through parameter block par, with their
// transcript rows, step program and, with more than one batch, the per-batch static rows
struct RpSegment { const rp_params *par; rp_geom g; uint32_t count; RpView v; uint8_t *raw; const rp_tr_step *prog; uint32_t steps; uint8_t *bstatic; };
// The front end over segments whose dec_bad flags lie back to back from the first segment's on, up to the scalar array; launches only
// (no allocation, no synchronisation: capturable).  Two branches: the decompressions need nothing but the proof bytes and run beside
// the transcript replays and the heads.
static int rp_front_end(bp_ctx *c, const std::vector<RpSegment> &seg, const sc *pow2_tab) {
    cudaStream_t s = c->stream, s2 = c->prof_on ? c->stream : c->aux;
    size_t total = 0;
    for (const RpSegment &x : seg) total += x.count;
    if (s2 != s) { CK(c, cudaEventRecord(c->ev_fork, s)); CK(c, cudaStreamWaitEvent(s2, c->ev_fork, 0)); }
    CK(c, cudaMemsetAsync(seg[0].v.decbad, 0, total * 4, s2));
    for (const RpSegment &x : seg)                // branch 2
        LAUNCH(c, KID_RP_DECOMPRESS, k_rp_decompress, blocks_for((size_t)x.count * x.g.D, RP_DEC_THREADS), RP_DEC_THREADS, rp_dec_smem_bytes(x.g), s2, x.par, x.g,
               x.count, x.v.niels, x.v.decbad);
    if (s2 != s) CK(c, cudaEventRecord(c->ev_join, s2));
    for (const RpSegment &x : seg) {
        LAUNCH(c, KID_RP_TRANSCRIPT, k_rp_transcript, blocks_for(x.count, RP_TR_THREADS), RP_TR_THREADS, 0, s, x.par, x.g, x.count, x.prog, x.steps, x.raw, x.v.status);
        LAUNCH(c, KID_RP_HEAD, rp_head_kernel(x.g.k), blocks_for(x.count, 32), 32, 0, s, x.par, x.g, x.raw, x.count, x.v.chal, x.v.tabs, pow2_tab, x.v.status,
               x.v.scalars);
    }
    if (s2 != s) CK(c, cudaStreamWaitEvent(s, c->ev_join, 0));
    for (const RpSegment &x : seg) {
        LAUNCH(c, KID_RP_SCALARS, k_rp_scalars_sum, x.g.nbatch * ((x.g.count + RP_CHUNK - 1) / RP_CHUNK), sum_threads(x.g.N), 0, s, x.g, x.v.chal, x.v.tabs, 0u,
               x.v.decbad, &x.par->live, x.v.part, x.v.scalars);
        LAUNCH(c, KID_RP_STATIC_REDUCE, k_rp_static_sum, dim3(x.g.S, x.g.nbatch > 1 ? x.g.nbatch + 1 : 1), 32, 0, s, x.v.part, x.g, x.v.scalars, x.bstatic);
    }
    return BP_OK;
}

// The launch sequence of one group, launches only (capturable): the front end as one segment, the group check and its verdicts.
// capture: the sequence is being captured into the verifier graph, whose per-batch pass goes under a conditional node.
static int rp_chain(bp_ctx *c, bp_gens *gens, const rp_geom &g, bool capture) {
    cudaStream_t s = c->stream;
    RpScratch &r = c->rp;
    const rp_params *par = r.par.as<rp_params>();
    int rc = rp_front_end(c, {{par, g, g.count * g.nbatch, rp_view(r), r.raw.as<uint8_t>(), r.prog.as<rp_tr_step>(), r.prog_steps, r.bstatic.as<uint8_t>()}},
                          r.pow2_tab.as<sc>());
    if (rc) return rc;
    // the group check: one MSM over every proof of the group (result in slot nbatch; the per-batch MSMs use slots 0..nbatch-1)
    ge_ext *d_group = r.results.as<ge_ext>() + g.nbatch;
    MsmArgs a{r.scalars.as<uint8_t>(), r.offsets.as<uint32_t>(), 1, rp_group_terms(g), r.pidx.as<uint32_t>(), gens->d_table.as<ge_niels>(), r.niels.as<ge_niels>(), nullptr, 0};
    rc = msm_launch(c, r.ar, a, msm_make_plan(a.T, a.n_msm, 0), d_group, s);
    if (rc) return rc;
    // with one batch the group check is the batch's check; captured, the group verdict kernel sets the condition of an IF node whose body
    // is the per-batch pass
    const bool gated = capture && g.nbatch > 1;
    cudaGraphConditionalHandle cond = 0;
    if (gated) { rc = graph_cond(c, &cond); if (rc) return rc; }
    LAUNCH(c, KID_RP_VERDICT_GROUP, k_rp_verdict_group, g.nbatch, 256, 0, s, r.status.as<uint32_t>(), r.decbad.as<uint32_t>(), d_group, g, par,
           r.batch_ok.as<uint32_t>(), r.combined.as<uint32_t>(), r.run.as<uint32_t>(), cond, gated ? 1 : 0);
    if (g.nbatch == 1) return BP_OK;
    if (!gated) return rp_batch_pass(c, gens, g, r.run.as<uint32_t>(), s);
    return graph_body(c, cond, cudaGraphCondTypeIf, "per-batch pass", [&](cudaStream_t body) { return rp_batch_pass(c, gens, g, nullptr, body); });
}

// what a captured graph depends on besides the verifier's scratch: the geometry, and the generator table, whose address is a kernel
// argument of the captured nodes
static std::array<size_t, 6> rp_graph_key(const bp_gens *gens, const rp_geom &g) {
    return {g.n, g.m, g.count, g.nbatch, (size_t)(uintptr_t)gens->d_table.p, g.proof_len};
}
static bool rp_graph_matches(const bp_ctx *c, const bp_gens *gens, const rp_geom &g) {
    return c->graph && c->graph_key == rp_graph_key(gens, g) && c->graph_moves == c->rp.moves;
}
static bool rp_xgraph_matches(const bp_ctx *c, const bp_gens *gens, const rp_geom &g) {
    return c->xgraph && c->xgraph_key == rp_graph_key(gens, g) && c->xgraph_moves == c->rp.moves;
}
static int rp_verify_fallback(bp_ctx *c, bp_gens *gens, const rp_geom &g, const RpView &v, uint32_t batch, uint32_t *d_verdict);
// queue everything up to the verdicts; d_proofs / d_commitments (and d_tstates, when the proofs have their own transcripts) are device
// pointers.  exact: the exact graph, which the caller has checked (rp_xgraph_matches); under profiling, the direct launches and then the
// host-driven reject path, which synchronises.
static int rp_verify_queue(bp_ctx *c, bp_gens *gens, const rp_geom &g, const uint8_t *d_proofs, const uint8_t *d_commit,
                           const uint8_t *h_transcript, const uint8_t *d_tstates, const uint8_t *seed, uint32_t *d_verdict, bool exact = false) {
    const bool use_graph = !c->prof_on && (exact ? rp_xgraph_matches(c, gens, g) : rp_graph_matches(c, gens, g));
    if (!use_graph) { int rc = rp_ensure(c, g); if (rc) return rc; }
    int rc = rp_build_maps(c, gens, g);          // another geometry may have used the context since: the maps follow the key
    if (rc) return rc;
    // the per-call parameter block, through the context's staging ring
    rp_params *par = nullptr;
    CK(c, c->stage.acquire(par));
    uint8_t sd[32];
    rc = draw_seed(c, seed, sd);
    if (rc) return rc;
    rp_fill_params(*par, c->rp.par.as<rp_params>(), h_transcript, d_tstates, sd, d_proofs, d_commit, d_verdict, g.count * g.nbatch);
    CK(c, cudaMemcpyAsync(c->rp.par.p, par, sizeof *par, cudaMemcpyHostToDevice, c->stream));
    CK(c, c->stage.record(c->stream));
    if (use_graph) {
        CK(c, cudaGraphLaunch(exact ? c->xgraph : c->graph, c->stream));
        c->launches += exact ? c->xgraph_launches : c->graph_launches;
        return BP_OK;
    }
    rc = rp_chain(c, gens, g, false);
    if (rc || !exact) return rc;
    std::vector<uint32_t> comb(g.nbatch);
    CK(c, cudaMemcpyAsync(comb.data(), c->rp.combined.p, (size_t)g.nbatch * 4, cudaMemcpyDeviceToHost, c->stream)); CK(c, cudaStreamSynchronize(c->stream));
    for (uint32_t b = 0; b < g.nbatch; b++)
        if (!comb[b]) { rc = rp_verify_fallback(c, gens, g, rp_view(c->rp), b, d_verdict); if (rc) return rc; }
    return BP_OK;
}

// Re-check of the proofs [p0, p0 + count) of a group in chunks of `chunk` proofs: one MSM per chunk over the row [S static | chunk*D
// dynamic], with part = the chunks' summed static-term scalars (Montgomery form, S per chunk).  Writes the verdicts of the proofs in
// passing chunks; chunk_ok (optional) receives the per-chunk pass flags, which synchronises.
static int rp_recheck(bp_ctx *c, bp_gens *gens, const rp_geom &g, const RpView &v, const sc *part, uint32_t p0, uint32_t count, uint32_t chunk,
                      uint32_t *d_verdict, std::vector<uint32_t> *chunk_ok) {
    cudaStream_t s = c->stream;
    const uint32_t nch = (count + chunk - 1) / chunk, row = g.S + chunk * g.D;
    size_t T = (size_t)nch * row;
    if (T >= (1u << 31)) { c->err = "fallback batch too large"; return BP_ERR_INVALID_ARGUMENT; }
    CK(c, c->rk_scal.ensure(T * 32, c->stream)); CK(c, c->rk_pidx.ensure(T * 4, c->stream)); CK(c, c->rk_offsets.ensure(((size_t)nch + 1) * 4, c->stream));
    CK(c, c->results.ensure((size_t)nch * sizeof(ge_ext), c->stream)); CK(c, c->flags.ensure((size_t)nch * 4, c->stream));
    LAUNCH(c, KID_SMALL, k_rp_chunk_rows, blocks_for(T, 128), 128, 0, s, part, v.scalars + (g.S + (size_t)p0 * g.D) * 32, g, count, chunk,
           (uint32_t)gens->cap, (uint32_t)gens->parties, p0 * g.D, c->rk_scal.as<uint8_t>(), c->rk_pidx.as<uint32_t>());
    LAUNCH(c, KID_SMALL, k_fill_offsets, blocks_for((size_t)nch + 1, 256), 256, 0, s, nch, row, c->rk_offsets.as<uint32_t>());
    MsmArgs a{c->rk_scal.as<uint8_t>(), c->rk_offsets.as<uint32_t>(), nch, (uint32_t)T, c->rk_pidx.as<uint32_t>(), gens->d_table.as<ge_niels>(), v.niels, nullptr, 0};
    int rc = msm_core(c, a, c->results.as<ge_ext>());
    if (rc) return rc;
    LAUNCH(c, KID_SMALL, k_rp_verdict_chunks, blocks_for(count, 128), 128, 0, s, v.status + p0, v.decbad + p0, c->results.as<ge_ext>(), count, chunk,
           d_verdict + p0, c->flags.as<uint32_t>());
    if (!chunk_ok) return BP_OK;
    chunk_ok->resize(nch);
    CK(c, cudaMemcpyAsync(chunk_ok->data(), c->flags.p, (size_t)nch * 4, cudaMemcpyDeviceToHost, s)); CK(c, cudaStreamSynchronize(s));
    return BP_OK;
}
// the proofs [p0, p0 + count) one by one (mod.rs:421-447 per proof): k_rp_scalars_sum on a geometry of one-proof batches gives each
// proof's own static-term scalars (the dynamic ones are where the head and the main pass left them: it only zeroes again those of
// proofs that failed), then a re-check with chunk = 1
static int rp_recheck_proofs(bp_ctx *c, bp_gens *gens, const rp_geom &g, const RpView &v, uint32_t p0, uint32_t count, uint32_t *d_verdict) {
    CK(c, c->fb_part.ensure((size_t)count * g.S * sizeof(sc), c->stream));
    rp_geom one = g; one.count = 1; one.nbatch = count;
    LAUNCH(c, KID_RP_SCALARS, k_rp_scalars_sum, count, sum_threads(g.N), 0, c->stream, one, v.chal + p0, v.tabs, p0,
           v.decbad + p0, nullptr, c->fb_part.as<sc>(), v.scalars + (size_t)p0 * g.D * 32);
    return rp_recheck(c, gens, g, v, c->fb_part.as<sc>(), p0, count, 1, d_verdict, nullptr);
}
// A batch whose combined check failed.  Level 1: one combined MSM per chunk of RP_CHUNK proofs, from the partial sums the main path
// already holds (one pipeline pass over the batch's ~T terms).  Level 2: the proofs of the failing chunks, each with its own MSM.
// One bad proof in 1024 costs two small passes instead of 1024 147-term MSMs.
static int rp_verify_fallback(bp_ctx *c, bp_gens *gens, const rp_geom &g, const RpView &v, uint32_t batch, uint32_t *d_verdict) {
    const uint32_t nch = (g.count + RP_CHUNK - 1) / RP_CHUNK, p0 = batch * g.count;
    std::vector<uint32_t> ok;
    int rc = rp_recheck(c, gens, g, v, v.part + (size_t)batch * nch * g.S, p0, g.count, RP_CHUNK, d_verdict, &ok);
    if (rc) return rc;
    uint32_t nfail = 0; for (uint32_t f : ok) nfail += f ? 0 : 1;
    if (nfail == 0) return BP_OK;       // cannot happen when the batch's combination failed, short of a 2^-128 cancellation between chunk weights
    if (rp_recheck_whole_batch(nfail)) return rp_recheck_proofs(c, gens, g, v, p0, g.count, d_verdict);      // many bad chunks: one pass over the whole batch
    for (uint32_t ch = 0; ch < nch; ch++)
        if (!ok[ch]) { rc = rp_recheck_proofs(c, gens, g, v, p0 + ch * RP_CHUNK, std::min<uint32_t>(RP_CHUNK, g.count - ch * RP_CHUNK), d_verdict); if (rc) return rc; }
    return BP_OK;
}

// ---------------------------------------------------------------------------------------------- device reject path (exact graphs)
// The groups of an exact graph (rp_exact.cuh) and the sizes of its passes: nct level-1 chunks over t1 terms; group gi's level-2 offsets
// start at offsets[off2[gi]]
struct XPlan { std::vector<rp_xgroup> G; uint32_t nct = 0, t1 = 0; std::vector<uint32_t> off2; };
// group of the proofs of view v: geometry g (count proofs per unit, nbatch units), their parameter block and per-unit combined flags, their
// points from dynamic index dyn_base on
static rp_xgroup rp_xgroup_of(const rp_geom &g, const RpView &v, const rp_params *par, const uint32_t *comb, uint32_t dyn_base) {
    rp_xgroup G{};
    G.g = g; G.par = par; G.comb = comb; G.status = v.status; G.decbad = v.decbad; G.chal = v.chal; G.tabs = v.tabs; G.part = v.part; G.scal = v.scalars;
    G.dyn_base = dyn_base;
    return G;
}
// Lays out the reject path of X.G (geometry and views set) on xs: every group's level-1 chunks, P, list, counters and level-2 sums; uploads
// the group table and the MSM offsets and sizes arena ar for every pass.  Synchronises; runs before the graphs that read these buffers are
// captured, so that nothing they bake in moves afterwards.
static int rp_exact_prepare(bp_ctx *c, XScratch &xs, MsmArena &ar, XPlan &X) {
    size_t nct = 0, t1 = 0, lists = 0, part2 = 0, t2max = 0, pmax = 0, noff = 0;
    for (rp_xgroup &G : X.G) {
        const rp_geom &g = G.g;
        const size_t nch = (size_t)(g.count + RP_CHUNK - 1) / RP_CHUNK * g.nbatch;
        G.P = rp_x_slice(g.count * g.nbatch, g.S, g.D);
        nct += nch; t1 += nch * (g.S + RP_CHUNK * g.D); lists += (size_t)g.count * g.nbatch; part2 += (size_t)G.P * g.S;
        t2max = std::max<size_t>(t2max, (size_t)G.P * (g.S + g.D)); pmax = std::max<size_t>(pmax, G.P); noff += G.P + 1;
    }
    if (t1 >= (1u << 31)) { c->err = "the device reject path of this geometry or mix needs 2^31 MSM terms or more"; return BP_ERR_INVALID_ARGUMENT; }
    noff += nct + 1;
    const size_t ng = X.G.size();
    CK(c, xs.grp.ensure(ng * sizeof(rp_xgroup), c->stream)); CK(c, xs.scal.ensure(std::max(t1, t2max) * 32, c->stream));
    CK(c, xs.pidx.ensure(std::max(t1, t2max) * 4, c->stream)); CK(c, xs.offsets.ensure(noff * 4, c->stream));
    CK(c, xs.results.ensure(std::max(nct, pmax) * sizeof(ge_ext), c->stream)); CK(c, xs.list.ensure(lists * 4, c->stream));
    CK(c, xs.ctr.ensure(ng * 3 * 4, c->stream)); CK(c, xs.part2.ensure(part2 * sizeof(sc), c->stream));
    std::vector<uint32_t> off;
    off.reserve(noff);
    X.nct = (uint32_t)nct; X.t1 = (uint32_t)t1; X.off2.assign(ng, 0);
    size_t chunk = 0, term = 0, list = 0, sums = 0;
    for (size_t gi = 0; gi < ng; gi++) {
        rp_xgroup &G = X.G[gi];
        const rp_geom &g = G.g;
        const uint32_t nch = (g.count + RP_CHUNK - 1) / RP_CHUNK * g.nbatch, row = g.S + RP_CHUNK * g.D;
        G.chunk0 = (uint32_t)chunk; G.row0 = (uint32_t)term;
        for (uint32_t j = 0; j < nch; j++) off.push_back((uint32_t)(term + (size_t)j * row));
        chunk += nch; term += (size_t)nch * row;
        G.list = xs.list.as<uint32_t>() + list; list += (size_t)g.count * g.nbatch;
        G.ctr = xs.ctr.as<uint32_t>() + 3 * gi;
        G.part2 = xs.part2.as<sc>() + sums; sums += (size_t)G.P * g.S;
    }
    off.push_back((uint32_t)t1);
    for (size_t gi = 0; gi < ng; gi++) {
        const rp_xgroup &G = X.G[gi];
        X.off2[gi] = (uint32_t)off.size();
        for (uint32_t i = 0; i <= G.P; i++) off.push_back(i * (G.g.S + G.g.D));
    }
    CK(c, cudaMemcpyAsync(xs.grp.p, X.G.data(), ng * sizeof(rp_xgroup), cudaMemcpyHostToDevice, c->stream));
    CK(c, cudaMemcpyAsync(xs.offsets.p, off.data(), off.size() * 4, cudaMemcpyHostToDevice, c->stream));
    CK(c, cudaStreamSynchronize(c->stream));
    int rc = msm_ensure(c, ar, msm_make_plan(X.t1, X.nct, 0));
    for (const rp_xgroup &G : X.G)
        if (!rc) rc = msm_ensure(c, ar, msm_make_plan(G.P * (G.g.S + G.g.D), G.P, 0));
    return rc;
}
// The device reject path, captured after a verifier's launch sequence (whose per-unit combined flags it reads), launches only.  An IF node
// runs level 1 when some unit failed; then each group's WHILE node runs level 2 on its list, one iteration per P listed proofs.  niels: the
// dynamic points the groups' dyn_base index.
static int rp_exact_chain(bp_ctx *c, bp_gens *gens, XScratch &xs, MsmArena &ar, const XPlan &X, const ge_niels *niels) {
    cudaStream_t s = c->stream;
    const rp_xgroup *dG = xs.grp.as<rp_xgroup>();
    const uint32_t ng = (uint32_t)X.G.size(), cap = (uint32_t)gens->cap, parties = (uint32_t)gens->parties;
    uint8_t *scal = xs.scal.as<uint8_t>(); uint32_t *pidx = xs.pidx.as<uint32_t>(), *off = xs.offsets.as<uint32_t>();
    ge_ext *res = xs.results.as<ge_ext>();
    const ge_niels *table = gens->d_table.as<ge_niels>();
    cudaGraphConditionalHandle any = 0;
    int rc = graph_cond(c, &any);
    if (rc) return rc;
    LAUNCH(c, KID_SMALL, k_rp_xprep, 1, 32, 0, s, dG, ng, any);
    rc = graph_body(c, any, cudaGraphCondTypeIf, "level-1 re-check", [&](cudaStream_t b) {
        LAUNCH(c, KID_SMALL, k_rp_xchunk_rows, X.nct, 128, 0, b, dG, ng, cap, parties, scal, pidx);
        MsmArgs a{scal, off, X.nct, X.t1, pidx, table, niels, nullptr, 0};
        int r = msm_launch(c, ar, a, msm_make_plan(a.T, a.n_msm, 0), res, b);
        if (r) return r;
        LAUNCH(c, KID_SMALL, k_rp_xchunk_verdicts, X.nct, 32, 0, b, dG, ng, res);
        return BP_OK;
    });
    if (rc) return rc;
    rp_xconds conds{};
    for (uint32_t gi = 0; gi < ng; gi++) { rc = graph_cond(c, &conds.h[gi]); if (rc) return rc; }
    LAUNCH(c, KID_SMALL, k_rp_xloop_init, 1, 32, 0, s, dG, ng, conds);
    for (uint32_t gi = 0; gi < ng; gi++) {
        const rp_xgroup &G = X.G[gi];
        const uint32_t T2 = G.P * (G.g.S + G.g.D);
        rc = graph_body(c, conds.h[gi], cudaGraphCondTypeWhile, "level-2 re-check", [&](cudaStream_t b) {
            LAUNCH(c, KID_RP_SCALARS, k_rp_xscalars, G.P, sum_threads(G.g.N), 0, b, G);
            LAUNCH(c, KID_SMALL, k_rp_xrows, blocks_for(T2, 128), 128, 0, b, G, cap, parties, scal, pidx);
            MsmArgs a{scal, off + X.off2[gi], G.P, T2, pidx, table, niels, nullptr, 0};
            int r = msm_launch(c, ar, a, msm_make_plan(a.T, a.n_msm, 0), res, b);
            if (r) return r;
            LAUNCH(c, KID_SMALL, k_rp_xverdicts, blocks_for(G.P, 128), 128, 0, b, G, res);
            LAUNCH(c, KID_SMALL, k_rp_xloop_next, 1, 1, 0, b, G.ctr, conds.h[gi]);
            return BP_OK;
        });
        if (rc) return rc;
    }
    return BP_OK;
}

// ---------------------------------------------------------------------------------------------- fused single-proof path
// Routing of bp_rangeproof_verify_batch: calls of at most RP_ROUTE_MAX_COUNT proofs with lg(n m) <= RP_ROUTE_MAX_K run k_rp_single, one
// cluster per proof in one launch; every other call runs the launch-group pipeline.  Crossover measured on one H100 SXM 80GB at a 700 W
// limit (benchmarks/single_proof.py, README.md "Results"), median wall time of a blocking call: at count 1 the fused launch wins up to
// lg(nm) = 6 (e.g. (8,1) 544 us against 618, (64,1) 721 against 732; (8,8) ties, 738 against 737) and loses from 7 on ((64,2) 956
// against 870); at (64,1) it wins up to 16 proofs (count 8: 720 against 786) and loses at 32 (1200 against 860).  Counts above 1 were
// measured at few geometries, so the rule stops at 8.
#define RP_ROUTE_MAX_COUNT 8
#define RP_ROUTE_MAX_K 6
static bool rp_single_routed(size_t count, size_t proof_len, size_t n, size_t m) {
    if (count < 1 || count > RP_ROUTE_MAX_COUNT || n == 0 || n > 64 || m == 0 || m > (1u << RP_ROUTE_MAX_K)) return false;
    size_t k = 0; while (((size_t)1 << k) < n * m) k++;
    return k <= RP_ROUTE_MAX_K && proof_len == 32 * (9 + 2 * k);
}
// One launch of k_rp_single over `count` proofs of geometry g (rp_param_verdict passed), then the verdicts.  Synchronises.
static int rp_single_verify(bp_ctx *c, bp_gens *gens, const rp_geom &g, const uint8_t *transcript, const uint8_t *proofs, const uint8_t *commitments,
                            const uint8_t *seed, uint8_t *verdicts) {
    if (g.k < RP_SINGLE_MIN_K || g.k > RP_SINGLE_MAX_K || g.count == 0 || g.count > RP_SINGLE_MAX_COUNT) return BP_ERR_INVALID_ARGUMENT;
    CK(c, cudaSetDevice(c->device));
    SingleScratch &x = c->sp;
    cudaStream_t s = c->stream;
    const rp_single_plan P = rp_single_plan_of(g.S + g.D);
    const rp_single_smem L = rp_single_layout(g, P);
    const size_t in_bytes = rp_single_input_bytes(g, g.count), io_bytes = RP_SINGLE_MAX_COUNT * 4 + in_bytes;
    CK(c, x.in.ensure(in_bytes, s)); CK(c, x.verdict.ensure(RP_SINGLE_MAX_COUNT * 4, s));
    CK(c, x.raw.ensure((size_t)g.count * P.cl * (RP_RAW_U + g.k) * 64, s));
    int rc = rp_pow2_table(c, x.pow2_tab);
    if (rc) return rc;
    if (x.prog_key[0] != g.n || x.prog_key[1] != g.m) {      // every call synchronises before it returns: no launch reads the old program
        rc = rp_upload_program(c, x.prog, g, &x.prog_steps);
        if (rc) return rc;
        x.prog_key[0] = g.n; x.prog_key[1] = g.m;
    }
    if (x.h_io.cap < io_bytes) CK(c, x.h_io.ensure(io_bytes + io_bytes / 4));      // likewise, nothing reads the old buffer
    uint8_t *h_in = x.h_io.as<uint8_t>() + RP_SINGLE_MAX_COUNT * 4;
    memset(h_in, 0, RP_SINGLE_HDR);
    memcpy(h_in, transcript, BP_TRANSCRIPT_BYTES);
    rc = draw_seed(c, seed, h_in + 208);
    if (rc) return rc;
    memcpy(h_in + RP_SINGLE_HDR, proofs, (size_t)g.count * g.proof_len);
    memcpy(h_in + RP_SINGLE_HDR + (size_t)g.count * g.proof_len, commitments, (size_t)g.count * g.m * 32);
    CK(c, cudaMemcpyAsync(x.in.p, h_in, in_bytes, cudaMemcpyHostToDevice, s));
    const rp_single_fn fn = rp_single_kernel(g.k);
    const uint32_t bit = 1u << (g.k - RP_SINGLE_MIN_K);
    if (!(x.smem_set & bit)) {
        size_t mx = 0;                                      // the largest layout of this k over the admitted (n, m)
        for (uint32_t n = 8; n <= 64 && n <= (1u << g.k); n *= 2) {
            rp_geom h{}; h.n = n; h.m = (1u << g.k) / n; h.k = g.k; h.N = 1u << g.k; h.D = 4 + 2 * g.k + h.m; h.S = 2 + 2 * h.N;
            mx = std::max<size_t>(mx, rp_single_layout(h, rp_single_plan_of(h.S + h.D)).total);
        }
        CK(c, cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)mx));
        CK(c, cudaFuncSetAttribute(fn, cudaFuncAttributeNonPortableClusterSizeAllowed, 0));
        x.smem_set |= bit;
    }
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(g.count * P.cl); cfg.blockDim = dim3(RP_SINGLE_THREADS); cfg.dynamicSmemBytes = L.total; cfg.stream = s;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension; attr[0].val.clusterDim.x = P.cl; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr; cfg.numAttrs = 1;
    rc = launch_profiled(c, KID_RP_SINGLE, s, "k_rp_single launch: ", [&] {
        return cudaLaunchKernelEx(&cfg, fn, g, P, x.in.as<const uint8_t>(), x.prog.as<const rp_tr_step>(), x.prog_steps, gens->d_table.as<const ge_niels>(),
                                  (uint32_t)gens->cap, (uint32_t)gens->parties, x.pow2_tab.as<const sc>(), x.raw.as<uint8_t>(), x.verdict.as<uint32_t>());
    });
    if (rc) return rc;
    uint32_t *h_v = x.h_io.as<uint32_t>();
    CK(c, cudaMemcpyAsync(h_v, x.verdict.p, (size_t)g.count * 4, cudaMemcpyDeviceToHost, s));
    CK(c, cudaStreamSynchronize(s));
    for (uint32_t i = 0; i < g.count; i++) verdicts[i] = (uint8_t)h_v[i];
    return BP_OK;
}

// bp_rangeproof_verify_reserve and, with exact, bp_rangeproof_verify_reserve_exact
static int rp_reserve(bp_ctx *c, bp_gens *gens, size_t n, size_t m, size_t count, size_t n_batches, bool exact) {
    if (!c || !gens) return BP_ERR_INVALID_ARGUMENT;
    BUSY_CHECK(c);
    CK(c, cudaSetDevice(c->device));
    size_t k = 0; while (((size_t)1 << k) < n * m) k++;
    rp_geom g{};
    if (rp_param_verdict(gens->cap, gens->parties, 32 * (9 + 2 * k), n, m, &g) != BP_PROOF_OK || !rp_set_group(&g, count, n_batches)) return BP_ERR_INVALID_ARGUMENT;
    CK(c, c->rp_proofs.ensure((size_t)g.count * g.nbatch * g.proof_len, c->stream)); CK(c, c->rp_commit.ensure((size_t)g.count * g.nbatch * m * 32, c->stream)); CK(c, c->rp_verdict.ensure((size_t)g.count * g.nbatch * 4, c->stream));
    CK(c, c->rp_tstates.ensure((size_t)g.count * g.nbatch * BP_TRANSCRIPT_BYTES, c->stream));
    int rc = rp_ensure(c, g); if (rc) return rc;
    XPlan X;
    if (exact) {                  // every buffer either graph bakes in is sized before the first capture
        c->xgraph_key = {};
        RpScratch &r = c->rp;
        X.G = {rp_xgroup_of(g, rp_view(r), r.par.as<rp_params>(), r.combined.as<uint32_t>(), 0)};
        rc = rp_exact_prepare(c, r.xs, r.ar, X); if (rc) return rc;
    }
    rc = rp_build_maps(c, gens, g); if (rc) return rc;
    CK(c, cudaStreamSynchronize(c->stream));
    rc = graph_capture(c, &c->graph, &c->graph_launches, [&] { return rp_chain(c, gens, g, true); });
    if (rc) return rc;
    c->graph_key = rp_graph_key(gens, g); c->graph_moves = c->rp.moves;
    if (exact) {
        rc = graph_capture(c, &c->xgraph, &c->xgraph_launches, [&] {
            const int r = rp_chain(c, gens, g, true);
            return r ? r : rp_exact_chain(c, gens, c->rp.xs, c->rp.ar, X, c->rp.niels.as<ge_niels>());
        });
        if (rc) return rc;
        c->xgraph_key = rp_graph_key(gens, g); c->xgraph_moves = c->rp.moves;
    }
    // one untimed pass so that the first real call finds module loading, the graph upload and the L2 working set done
    std::vector<uint8_t> zt(BP_TRANSCRIPT_BYTES, 0);
    CK(c, cudaMemsetAsync(c->rp_proofs.p, 0, (size_t)g.count * g.nbatch * g.proof_len, c->stream)); CK(c, cudaMemsetAsync(c->rp_commit.p, 0, (size_t)g.count * g.nbatch * m * 32, c->stream));
    rc = rp_verify_queue(c, gens, g, c->rp_proofs.as<uint8_t>(), c->rp_commit.as<uint8_t>(), zt.data(), nullptr, nullptr, c->rp_verdict.as<uint32_t>());
    if (rc) return rc;
    if (exact) {
        rc = rp_verify_queue(c, gens, g, c->rp_proofs.as<uint8_t>(), c->rp_commit.as<uint8_t>(), zt.data(), nullptr, nullptr, c->rp_verdict.as<uint32_t>(), true);
        if (rc) return rc;
    }
    CK(c, cudaStreamSynchronize(c->stream));
    return BP_OK;
}
int bp_rangeproof_verify_reserve(bp_ctx *c, bp_gens *gens, size_t n, size_t m, size_t count, size_t n_batches) {
    return rp_reserve(c, gens, n, m, count, n_batches, false);
}
int bp_rangeproof_verify_reserve_exact(bp_ctx *c, bp_gens *gens, size_t n, size_t m, size_t count, size_t n_batches) {
    return rp_reserve(c, gens, n, m, count, n_batches, true);
}

// bp_rangeproof_verify_group_begin (transcript: one state for every proof) and *_begin_transcripts (transcripts: one record per proof)
static int rp_group_begin(bp_ctx *c, bp_gens *gens, const uint8_t *transcript, const uint8_t *transcripts, const uint8_t *proofs, size_t proof_len,
                          const uint8_t *commitments, size_t n, size_t m, size_t count, size_t n_batches, const uint8_t *seed) {
    if (!c || !gens || !(transcript || transcripts) || !proofs || !commitments || count == 0 || n_batches == 0) return BP_ERR_INVALID_ARGUMENT;
    if (c->vs.active) { c->err = "verify_begin called twice without verify_finish"; return BP_ERR_INVALID_ARGUMENT; }
    BUSY_CHECK(c);
    if (count * n_batches >= (1u << 24) || n_batches > BP_MAX_GROUP_BATCHES) return BP_ERR_INVALID_ARGUMENT;
    CK(c, cudaSetDevice(c->device));
    rp_geom g{};
    uint8_t pv = rp_param_verdict(gens->cap, gens->parties, proof_len, n, m, &g);
    VerifyState vs; vs.total = (uint32_t)(count * n_batches); vs.n_batches = (uint32_t)n_batches; vs.gens = gens; vs.param_verdict = pv;
    if (pv != BP_PROOF_OK) {              // no kernel runs: _finish hands out these codes
        vs.param_codes.resize(vs.total);
        for (size_t i = 0; i < vs.total; i++) vs.param_codes[i] = rp_rejected_proof_verdict(pv, proofs + i * proof_len, proof_len);
        vs.active = true; c->vs = std::move(vs); return BP_OK;
    }
    if (!rp_set_group(&g, count, n_batches)) return BP_ERR_INVALID_ARGUMENT;
    vs.g = g;
    size_t total = vs.total;
    CK(c, c->rp_proofs.ensure(total * proof_len, c->stream)); CK(c, c->rp_commit.ensure(total * m * 32, c->stream)); CK(c, c->rp_verdict.ensure(total * 4, c->stream));
    CK(c, cudaMemcpyAsync(c->rp_proofs.p, proofs, total * proof_len, cudaMemcpyHostToDevice, c->stream));
    CK(c, cudaMemcpyAsync(c->rp_commit.p, commitments, total * m * 32, cudaMemcpyHostToDevice, c->stream));
    if (transcripts) {
        CK(c, c->rp_tstates.ensure(total * BP_TRANSCRIPT_BYTES, c->stream));
        CK(c, cudaMemcpyAsync(c->rp_tstates.p, transcripts, total * BP_TRANSCRIPT_BYTES, cudaMemcpyHostToDevice, c->stream));
    }
    int rc = rp_verify_queue(c, gens, g, c->rp_proofs.as<uint8_t>(), c->rp_commit.as<uint8_t>(), transcript, transcripts ? c->rp_tstates.as<uint8_t>() : nullptr, seed,
                             c->rp_verdict.as<uint32_t>());
    if (rc) return rc;
    CK(c, cudaMemcpyAsync(c->h_verdict.p, c->rp_verdict.p, total * 4, cudaMemcpyDeviceToHost, c->stream));
    CK(c, cudaMemcpyAsync(c->h_flag.p, c->rp.combined.p, (size_t)g.nbatch * 4, cudaMemcpyDeviceToHost, c->stream));
    CK(c, cudaMemcpyAsync(c->h_flag.as<uint32_t>() + BP_MAX_GROUP_BATCHES, c->rp.batch_ok.p, (size_t)g.nbatch * 4, cudaMemcpyDeviceToHost, c->stream));
    vs.active = true; c->vs = vs;              // only a fully queued verification is pending
    return BP_OK;
}
int bp_rangeproof_verify_group_begin(bp_ctx *c, bp_gens *gens, const uint8_t *transcript, const uint8_t *proofs, size_t proof_len, const uint8_t *commitments,
                                     size_t n, size_t m, size_t count, size_t n_batches, const uint8_t *seed) {
    return rp_group_begin(c, gens, transcript, nullptr, proofs, proof_len, commitments, n, m, count, n_batches, seed);
}
int bp_rangeproof_verify_group_begin_transcripts(bp_ctx *c, bp_gens *gens, const uint8_t *transcripts, const uint8_t *proofs, size_t proof_len,
                                                 const uint8_t *commitments, size_t n, size_t m, size_t count, size_t n_batches, const uint8_t *seed) {
    return rp_group_begin(c, gens, nullptr, transcripts, proofs, proof_len, commitments, n, m, count, n_batches, seed);
}

int bp_rangeproof_verify_group_finish(bp_ctx *c, uint8_t *verdicts, uint8_t *batch_ok) {
    if (!c || !verdicts || !c->vs.active) return BP_ERR_INVALID_ARGUMENT;
    VerifyState vs = std::move(c->vs); c->vs = VerifyState{};
    if (vs.param_verdict != BP_PROOF_OK) { memcpy(verdicts, vs.param_codes.data(), vs.total); if (batch_ok) memset(batch_ok, 0, vs.n_batches); return BP_OK; }
    CK(c, cudaSetDevice(c->device));
    CK(c, cudaStreamSynchronize(c->stream));
    const uint32_t *h_verdict = c->h_verdict.as<uint32_t>(), *h_flag = c->h_flag.as<uint32_t>();
    bool redo = false;
    for (uint32_t b = 0; b < vs.g.nbatch; b++)
        if (h_flag[b] == 0) {               // this batch's combined check failed: find the offenders (chunks of 32, then proof by proof)
            int rc = rp_verify_fallback(c, vs.gens, vs.g, rp_view(c->rp), b, c->rp_verdict.as<uint32_t>());
            if (rc) return rc;
            redo = true;
        }
    if (redo) {
        CK(c, cudaMemcpyAsync(c->h_verdict.p, c->rp_verdict.p, (size_t)vs.total * 4, cudaMemcpyDeviceToHost, c->stream));
        CK(c, cudaStreamSynchronize(c->stream));
    }
    for (uint32_t i = 0; i < vs.total; i++) verdicts[i] = (uint8_t)h_verdict[i];
    if (batch_ok) for (uint32_t b = 0; b < vs.g.nbatch; b++) batch_ok[b] = (uint8_t)h_flag[BP_MAX_GROUP_BATCHES + b];
    return BP_OK;
}

// bp_rangeproof_verify_group_device (transcript: one host state for every proof) and *_device_transcripts (d_transcripts: one device
// record per proof); exact: their *_exact forms, on the exact graph of a geometry reserved with bp_rangeproof_verify_reserve_exact
static int rp_group_device(bp_ctx *c, bp_gens *gens, const uint8_t *transcript, const void *d_transcripts, const void *d_proofs, size_t proof_len,
                           const void *d_commitments, size_t n, size_t m, size_t count, size_t n_batches, const uint8_t *seed, void *d_verdicts_u32,
                           uint32_t *h_batch_ok_pinned, bool exact = false) {
    if (!c || !gens || !(transcript || d_transcripts) || !d_proofs || !d_commitments || !d_verdicts_u32) return BP_ERR_INVALID_ARGUMENT;
    if (!is_aligned(d_verdicts_u32, 4)) { c->err = "bp_rangeproof_verify_group_device: d_verdicts_u32 must be 4-byte aligned"; return BP_ERR_INVALID_ARGUMENT; }
    BUSY_CHECK(c);
    CK(c, cudaSetDevice(c->device));
    rp_geom g{};
    uint8_t pv = rp_param_verdict(gens->cap, gens->parties, proof_len, n, m, &g);
    if (pv != BP_PROOF_OK || !rp_set_group(&g, count, n_batches)) return BP_ERR_INVALID_ARGUMENT;
    if (exact && !rp_xgraph_matches(c, gens, g)) {
        c->err = "bp_rangeproof_verify_group_device_exact: this geometry is not reserved with bp_rangeproof_verify_reserve_exact on this context and generator table";
        return BP_ERR_INVALID_ARGUMENT;
    }
    int rc = rp_verify_queue(c, gens, g, (const uint8_t *)d_proofs, (const uint8_t *)d_commitments, transcript, (const uint8_t *)d_transcripts, seed,
                             (uint32_t *)d_verdicts_u32, exact);
    if (rc) return rc;
    if (h_batch_ok_pinned) CK(c, cudaMemcpyAsync(h_batch_ok_pinned, c->rp.batch_ok.p, (size_t)g.nbatch * 4, cudaMemcpyDeviceToHost, c->stream));
    return BP_OK;
}
int bp_rangeproof_verify_group_device(bp_ctx *c, bp_gens *gens, const uint8_t *transcript, const void *d_proofs, size_t proof_len, const void *d_commitments,
                                      size_t n, size_t m, size_t count, size_t n_batches, const uint8_t *seed, void *d_verdicts_u32, uint32_t *h_batch_ok_pinned) {
    return rp_group_device(c, gens, transcript, nullptr, d_proofs, proof_len, d_commitments, n, m, count, n_batches, seed, d_verdicts_u32, h_batch_ok_pinned);
}
int bp_rangeproof_verify_group_device_transcripts(bp_ctx *c, bp_gens *gens, const void *d_transcripts, const void *d_proofs, size_t proof_len,
                                                  const void *d_commitments, size_t n, size_t m, size_t count, size_t n_batches, const uint8_t *seed,
                                                  void *d_verdicts_u32, uint32_t *h_batch_ok_pinned) {
    return rp_group_device(c, gens, nullptr, d_transcripts, d_proofs, proof_len, d_commitments, n, m, count, n_batches, seed, d_verdicts_u32, h_batch_ok_pinned);
}
int bp_rangeproof_verify_group_device_exact(bp_ctx *c, bp_gens *gens, const uint8_t *transcript, const void *d_proofs, size_t proof_len, const void *d_commitments,
                                            size_t n, size_t m, size_t count, size_t n_batches, const uint8_t *seed, void *d_verdicts_u32, uint32_t *h_batch_ok_pinned) {
    return rp_group_device(c, gens, transcript, nullptr, d_proofs, proof_len, d_commitments, n, m, count, n_batches, seed, d_verdicts_u32, h_batch_ok_pinned, true);
}
int bp_rangeproof_verify_group_device_exact_transcripts(bp_ctx *c, bp_gens *gens, const void *d_transcripts, const void *d_proofs, size_t proof_len,
                                                        const void *d_commitments, size_t n, size_t m, size_t count, size_t n_batches, const uint8_t *seed,
                                                        void *d_verdicts_u32, uint32_t *h_batch_ok_pinned) {
    return rp_group_device(c, gens, nullptr, d_transcripts, d_proofs, proof_len, d_commitments, n, m, count, n_batches, seed, d_verdicts_u32, h_batch_ok_pinned, true);
}

// single-batch forms
int bp_rangeproof_verify_begin(bp_ctx *c, bp_gens *gens, const uint8_t *transcript, const uint8_t *proofs, size_t proof_len, const uint8_t *commitments,
                               size_t n, size_t m, size_t count, const uint8_t *seed) {
    return bp_rangeproof_verify_group_begin(c, gens, transcript, proofs, proof_len, commitments, n, m, count, 1, seed);
}
int bp_rangeproof_verify_finish(bp_ctx *c, uint8_t *verdicts) { return bp_rangeproof_verify_group_finish(c, verdicts, nullptr); }
int bp_rangeproof_verify_batch(bp_ctx *c, bp_gens *gens, const uint8_t *transcript, const uint8_t *proofs, size_t proof_len, const uint8_t *commitments,
                               size_t n, size_t m, size_t count, const uint8_t *seed, uint8_t *verdicts) {
    // Small calls go to the fused kernel once every check of the pipeline's begin would pass (any refusal or parameter verdict is left
    // to it, with its messages and order); the verdicts are the same, each proof checked on its own.
    rp_geom g{};
    if (c && gens && transcript && proofs && commitments && verdicts && !c->vs.active && !c->ms.active && rp_single_routed(count, proof_len, n, m)
        && rp_param_verdict(gens->cap, gens->parties, proof_len, n, m, &g) == BP_PROOF_OK && rp_set_group(&g, count, 1))
        return rp_single_verify(c, gens, g, transcript, proofs, commitments, seed, verdicts);
    int rc = bp_rangeproof_verify_begin(c, gens, transcript, proofs, proof_len, commitments, n, m, count, seed);
    if (rc) return rc;
    return bp_rangeproof_verify_finish(c, verdicts);
}
int bp_rangeproof_verify_batch_device(bp_ctx *c, bp_gens *gens, const uint8_t *transcript, const void *d_proofs, size_t proof_len, const void *d_commitments,
                                      size_t n, size_t m, size_t count, const uint8_t *seed, void *d_verdicts_u32, uint32_t *h_batch_ok_pinned) {
    return bp_rangeproof_verify_group_device(c, gens, transcript, d_proofs, proof_len, d_commitments, n, m, count, 1, seed, d_verdicts_u32, h_batch_ok_pinned);
}

// Proofs of any geometry in one call (layout: rp_mixed.cuh).  Each class runs the fixed-geometry front end on its slices of the mixed
// arenas; one MSM then checks every admitted proof.  When it fails, one pipeline pass over the same array with an MSM per class segment
// finds the failing classes, and each of those runs the fixed-geometry reject path on its own slices.  A call that fits the context's
// reserved mix runs this sequence as the mix's captured graph on the mix's own arenas; any other call launches it directly on MixScratch.

// every arena of a mixed call of layout P (grow-only): in_p / in_c bytes of caller proofs / commitments, records: per-proof transcripts
static int mix_ensure(bp_ctx *c, MixScratch &x, const rp_mixed_plan &P, uint64_t in_p, uint64_t in_c, bool records) {
    const size_t C = P.cls.size(), A = P.cls.back().first + P.cls.back().g.count;
    CK(c, x.in_proofs.ensure(in_p, c->stream)); CK(c, x.in_commit.ensure(in_c, c->stream)); CK(c, x.gather.ensure(A * sizeof(rp_gather), c->stream));
    CK(c, x.proofs.ensure(P.proof_bytes, c->stream)); CK(c, x.commit.ensure(P.commit_bytes, c->stream)); CK(c, x.par.ensure(C * sizeof(rp_params), c->stream));
    CK(c, x.prog.ensure(P.prog_steps * sizeof(rp_tr_step), c->stream)); CK(c, x.raw.ensure(P.raw_bytes, c->stream));
    CK(c, x.status.ensure(A * 4, c->stream)); CK(c, x.decbad.ensure(A * 4, c->stream)); CK(c, x.verdict.ensure(A * 4, c->stream));
    CK(c, x.chal.ensure(A * sizeof(rp_lean_head), c->stream)); CK(c, x.tabs.ensure(P.tab_scalars * sizeof(sc), c->stream));
    CK(c, x.part.ensure(P.part_scalars * sizeof(sc), c->stream)); CK(c, x.scalars.ensure(P.terms * 32, c->stream)); CK(c, x.pidx.ensure(P.terms * 4, c->stream));
    CK(c, x.offsets.ensure((C + 3) * 4, c->stream)); CK(c, x.niels.ensure(P.dyn_points * sizeof(ge_niels), c->stream));
    CK(c, x.flags.ensure(3 * C * 4, c->stream)); CK(c, x.results.ensure((C + 1) * sizeof(ge_ext), c->stream));
    if (records) CK(c, x.tstates.ensure(A * BP_TRANSCRIPT_BYTES, c->stream));
    int rc = rp_pow2_table(c, x.pow2_tab);
    if (rc) return rc;
    return msm_ensure(c, x.ar, msm_make_plan((uint32_t)P.terms, 1, 0));
}
// the transcript step programs and the MSM offsets of layout P (the combined MSM, then the class segments), queued from host vectors
// that the caller keeps until the stream has read them
static int mix_upload_layout(bp_ctx *c, MixScratch &x, const rp_mixed_plan &P, std::vector<rp_tr_step> &hprog, std::vector<uint32_t> &hoff) {
    const uint32_t C = (uint32_t)P.cls.size();
    hprog.clear(); hprog.reserve(P.prog_steps);
    hoff.assign(C + 3, 0);
    hoff[1] = (uint32_t)P.terms;
    for (uint32_t k = 0; k < C; k++) {
        const rp_geom &g = P.cls[k].g;
        const std::vector<rp_tr_step> prog = rp_tr_program(g.n, g.m, g.k);
        hprog.insert(hprog.end(), prog.begin(), prog.end());
        hoff[2 + k] = (uint32_t)P.cls[k].seg;
    }
    hoff[2 + C] = (uint32_t)P.terms;
    CK(c, cudaMemcpyAsync(x.prog.p, hprog.data(), hprog.size() * sizeof(rp_tr_step), cudaMemcpyHostToDevice, c->stream));
    CK(c, cudaMemcpyAsync(x.offsets.p, hoff.data(), hoff.size() * 4, cudaMemcpyHostToDevice, c->stream));
    return BP_OK;
}
// the slices of class K: the front end and the reject path run on them as on a fixed-geometry batch
static RpView mix_view(MixScratch &x, const rp_mixed_class &K) {
    return RpView{x.scalars.as<uint8_t>() + K.seg * 32, x.status.as<uint32_t>() + K.first, x.decbad.as<uint32_t>() + K.first, x.chal.as<rp_lean_head>() + K.first,
                  x.tabs.as<sc>() + K.tab_off, x.part.as<sc>() + K.part_off, x.niels.as<ge_niels>() + K.dyn};
}
// class k's point map: its segment of the term -> point map
static int mix_point_map(bp_ctx *c, bp_gens *gens, MixScratch &x, const rp_mixed_class &K, cudaStream_t s) {
    LAUNCH(c, KID_SMALL, k_rp_point_idx, blocks_for(K.g.T, 256), 256, 0, s, K.g, (uint32_t)gens->cap, (uint32_t)gens->parties, RP_GROUP_ROW, (uint32_t)K.dyn,
           x.pidx.as<uint32_t>() + K.seg);
    return BP_OK;
}
// The launches of a mixed call of layout P, after the parameter blocks, gathered inputs and point maps: the front end with one segment
// per class, the combined check and each class's verdicts from it.  Launches only: capturable.
static int mix_chain(bp_ctx *c, bp_gens *gens, MixScratch &x, const rp_mixed_plan &P) {
    const uint32_t C = (uint32_t)P.cls.size();
    const rp_params *d_par = x.par.as<rp_params>();
    cudaStream_t s = c->stream;
    std::vector<RpSegment> seg;
    for (uint32_t k = 0; k < C; k++) {
        const rp_mixed_class &K = P.cls[k];
        seg.push_back({d_par + k, K.g, K.g.count, mix_view(x, K), x.raw.as<uint8_t>() + K.raw_off, x.prog.as<rp_tr_step>() + K.prog_off, K.prog_steps, nullptr});
    }
    int rc = rp_front_end(c, seg, x.pow2_tab.as<sc>());
    if (rc) return rc;
    // the combined check over every class (result slot 0; the per-class MSMs use slots 1..C)
    uint32_t *batch_ok = x.flags.as<uint32_t>(), *combined = batch_ok + C, *run = combined + C;
    MsmArgs a{x.scalars.as<uint8_t>(), x.offsets.as<uint32_t>(), 1, (uint32_t)P.terms, x.pidx.as<uint32_t>(), gens->d_table.as<ge_niels>(), x.niels.as<ge_niels>(), nullptr, 0};
    rc = msm_launch(c, x.ar, a, msm_make_plan(a.T, 1, 0), x.results.as<ge_ext>(), s);
    if (rc) return rc;
    for (uint32_t k = 0; k < C; k++) {
        const RpView v = mix_view(x, P.cls[k]);
        LAUNCH(c, KID_RP_VERDICT_GROUP, k_rp_verdict_group, 1, 256, 0, s, v.status, v.decbad, x.results.as<ge_ext>(), P.cls[k].g, d_par + k, batch_ok + k, combined + k,
               run + k, (cudaGraphConditionalHandle)0, 0);
    }
    return BP_OK;
}
// the pass that decides the classes once the combined check failed: one MSM per class segment over the same array, then each class's
// verdicts and combined flag from its own MSM (with one class the combined check already was its MSM)
static int mix_class_pass(bp_ctx *c, bp_gens *gens, MixScratch &x, const rp_mixed_plan &P, cudaStream_t s) {
    const uint32_t C = (uint32_t)P.cls.size();
    uint32_t *batch_ok = x.flags.as<uint32_t>(), *combined = batch_ok + C;
    MsmArgs b{x.scalars.as<uint8_t>(), x.offsets.as<uint32_t>() + 2, C, (uint32_t)P.terms, x.pidx.as<uint32_t>(), gens->d_table.as<ge_niels>(), x.niels.as<ge_niels>(), nullptr, 0};
    int rc = msm_launch(c, x.ar, b, msm_make_plan(b.T, C, 0), x.results.as<ge_ext>() + 1, s);
    if (rc) return rc;
    for (uint32_t k = 0; k < C; k++) {
        const RpView v = mix_view(x, P.cls[k]);
        LAUNCH(c, KID_RP_VERDICT_BATCH, k_rp_verdict_batch, 1, 256, 0, s, v.status, v.decbad, x.results.as<ge_ext>() + 1 + k, P.cls[k].g, x.par.as<rp_params>() + k,
               batch_ok + k, combined + k, nullptr);
    }
    return BP_OK;
}
// the reject path of every class whose own check failed (comb[k] == 0), over its live[k] proofs; d_verdict gets their verdicts.  Synchronises.
static int mix_reject(bp_ctx *c, bp_gens *gens, MixScratch &x, const rp_mixed_plan &P, const uint32_t *live, const uint32_t *comb, bool *redo) {
    for (size_t k = 0; k < P.cls.size(); k++)
        if (!comb[k] && live[k]) {
            const rp_mixed_class &K = P.cls[k];
            rp_geom g = K.g; g.count = live[k]; g.T = g.S + g.count * g.D;
            int rc = rp_verify_fallback(c, gens, g, mix_view(x, K), 0, x.verdict.as<uint32_t>() + K.first);
            if (rc) return rc;
            *redo = true;
        }
    return BP_OK;
}
// class k's parameter block with live proofs; records: the proofs' transcripts are the records at the class's slots of x.tstates
static void mix_params(rp_params &pa, const rp_mixed_class &K, MixScratch &x, uint32_t k, const uint8_t *transcript, bool records, const uint8_t seed[32], uint32_t live) {
    rp_fill_params(pa, x.par.as<rp_params>() + k, transcript, records ? x.tstates.as<uint8_t>() + (size_t)K.first * BP_TRANSCRIPT_BYTES : nullptr, seed,
                   x.proofs.as<uint8_t>() + K.proof_off, x.commit.as<uint8_t>() + K.commit_off, x.verdict.as<uint32_t>() + K.first, live);
}
// The host side of a call's placement in layout X: class k's parameter block with live[k] proofs into hpar[k]; for the j-th (input index,
// slot) pair, in slot order, that input's gather entry into hg[j] and, with per-proof transcripts, its record at its slot of hts
static void mix_place(const rp_mixed_plan &X, MixScratch &x, const uint8_t *transcript, const uint8_t *transcripts, const uint8_t seed[32], const uint32_t *live,
                      const std::vector<std::pair<uint32_t, uint32_t>> &slots, const uint64_t *proof_offsets, const uint64_t *commit_offsets, rp_params *hpar,
                      rp_gather *hg, uint8_t *hts) {
    for (uint32_t k = 0; k < X.cls.size(); k++) mix_params(hpar[k], X.cls[k], x, k, transcript, transcripts != nullptr, seed, live[k]);
    uint32_t k = 0;
    for (size_t j = 0; j < slots.size(); j++) {
        const uint32_t i = slots[j].first, slot = slots[j].second;
        while (slot >= X.cls[k].first + X.cls[k].g.count) k++;
        const rp_mixed_class &K = X.cls[k];
        hg[j] = rp_gather_entry(proof_offsets[i], commit_offsets[i], K.proof_off, K.commit_off, K.g.proof_len, K.g.m, slot - K.first);
        if (transcripts) memcpy(hts + (size_t)slot * BP_TRANSCRIPT_BYTES, transcripts + (size_t)i * BP_TRANSCRIPT_BYTES, BP_TRANSCRIPT_BYTES);
    }
}

// A call that does not fit the reserved mix: plan P laid out on MixScratch, every launch direct, synchronised; verdicts in input order
static int rp_mixed_direct(bp_ctx *c, bp_gens *gens, const uint8_t *transcript, const uint8_t *transcripts, size_t count, const uint8_t *proofs,
                           const uint64_t *proof_offsets, const uint8_t *commitments, const uint64_t *commit_offsets, const uint8_t seed[32],
                           const rp_mixed_plan &P, uint8_t *verdicts) {
    MixScratch &x = c->mx;
    const uint32_t C = (uint32_t)P.cls.size(), A = (uint32_t)P.order.size();
    const uint64_t in_p = proof_offsets[count], in_c = 32 * commit_offsets[count];
    int rc = mix_ensure(c, x, P, in_p, in_c, transcripts != nullptr);
    if (rc) return rc;
    // every admitted proof at its own slot of P, in class order
    std::vector<uint32_t> live(C);
    for (uint32_t k = 0; k < C; k++) live[k] = P.cls[k].g.count;
    std::vector<std::pair<uint32_t, uint32_t>> slots(A);
    for (uint32_t j = 0; j < A; j++) slots[j] = {P.order[j], j};
    std::vector<rp_params> hpar(C);
    std::vector<rp_gather> hg(A);
    std::vector<uint8_t> hts(transcripts ? (size_t)A * BP_TRANSCRIPT_BYTES : 0);
    mix_place(P, x, transcript, transcripts, seed, live.data(), slots, proof_offsets, commit_offsets, hpar.data(), hg.data(), hts.data());
    cudaStream_t s = c->stream;
    // the caller's buffers as they are, then gathered into class order on the device
    CK(c, cudaMemcpyAsync(x.in_proofs.p, proofs, in_p, cudaMemcpyHostToDevice, s)); CK(c, cudaMemcpyAsync(x.in_commit.p, commitments, in_c, cudaMemcpyHostToDevice, s));
    CK(c, cudaMemcpyAsync(x.gather.p, hg.data(), (size_t)A * sizeof(rp_gather), cudaMemcpyHostToDevice, s));
    LAUNCH(c, KID_SMALL, k_rp_gather, A, 128, 0, s, x.in_proofs.as<uint8_t>(), x.in_commit.as<uint8_t>(), x.gather.as<rp_gather>(), x.proofs.as<uint8_t>(),
           x.commit.as<uint8_t>());
    CK(c, cudaMemcpyAsync(x.par.p, hpar.data(), (size_t)C * sizeof(rp_params), cudaMemcpyHostToDevice, s));
    if (transcripts) CK(c, cudaMemcpyAsync(x.tstates.p, hts.data(), hts.size(), cudaMemcpyHostToDevice, s));
    std::vector<rp_tr_step> hprog; std::vector<uint32_t> hoff;
    rc = mix_upload_layout(c, x, P, hprog, hoff);
    if (rc) return rc;
    for (const rp_mixed_class &K : P.cls) { rc = mix_point_map(c, gens, x, K, s); if (rc) return rc; }
    rc = mix_chain(c, gens, x, P);
    if (rc) return rc;
    const uint32_t *combined = x.flags.as<uint32_t>() + C;
    std::vector<uint32_t> hverd(A), hcomb(C);
    CK(c, cudaMemcpyAsync(hverd.data(), x.verdict.p, (size_t)A * 4, cudaMemcpyDeviceToHost, s));
    CK(c, cudaMemcpyAsync(hcomb.data(), combined, (size_t)C * 4, cudaMemcpyDeviceToHost, s));
    CK(c, cudaStreamSynchronize(s));
    if (!hcomb[0]) {
        if (C > 1) {
            rc = msm_ensure(c, x.ar, msm_make_plan((uint32_t)P.terms, C, 0));
            if (rc) return rc;
            rc = mix_class_pass(c, gens, x, P, s);
            if (rc) return rc;
            CK(c, cudaMemcpyAsync(hcomb.data(), combined, (size_t)C * 4, cudaMemcpyDeviceToHost, s));
            CK(c, cudaStreamSynchronize(s));
        }
        bool redo = false;
        rc = mix_reject(c, gens, x, P, live.data(), hcomb.data(), &redo);
        if (rc) return rc;
        CK(c, cudaMemcpyAsync(hverd.data(), x.verdict.p, (size_t)A * 4, cudaMemcpyDeviceToHost, s));
        CK(c, cudaStreamSynchronize(s));
    }
    for (uint32_t j = 0; j < A; j++) verdicts[P.order[j]] = (uint8_t)hverd[j];
    return BP_OK;
}

// the launch sequence of the reserved mix R, captured: mix_chain on the mix at capacity and, with more than one class, the class pass under
// an IF node whose condition is the combined check's failure
static int mix_capture(bp_ctx *c, bp_gens *gens, MixReserve &R) {
    const rp_mixed_plan &X = R.X;
    int rc = mix_chain(c, gens, R.x, X);
    if (rc) return rc;
    if (X.cls.size() == 1) return BP_OK;
    cudaGraphConditionalHandle cond = 0;
    rc = graph_cond(c, &cond);
    if (rc) return rc;
    LAUNCH(c, KID_SMALL, k_set_cond_unless_identity, 1, 32, 0, c->stream, R.x.results.as<ge_ext>(), cond);
    return graph_body(c, cond, cudaGraphCondTypeIf, "class pass", [&](cudaStream_t body) { return mix_class_pass(c, gens, R.x, X, body); });
}

// a fitting call (live: its proofs per class of the mix): stage the parameter blocks, gather table and records, queue the uploads, the
// gather, the graph and the downloads of verdicts and flags.  No allocation, no synchronisation.
static int mix_queue(bp_ctx *c, const uint8_t *transcript, const uint8_t *transcripts, size_t count, const uint8_t *proofs, const uint64_t *proof_offsets,
                     const uint8_t *commitments, const uint64_t *commit_offsets, const uint8_t seed[32], const std::vector<uint32_t> &live,
                     const std::vector<std::pair<uint32_t, uint32_t>> &slots) {
    MixReserve &R = *c->mix; MixScratch &x = R.x; const rp_mixed_plan &X = R.X;
    const uint32_t C = (uint32_t)X.cls.size(), A = (uint32_t)slots.size();
    rp_params *hpar = R.h_stage.as<rp_params>();
    rp_gather *hg = reinterpret_cast<rp_gather *>(hpar + C);
    uint8_t *hts = reinterpret_cast<uint8_t *>(hg + R.slots());
    mix_place(X, x, transcript, transcripts, seed, live.data(), slots, proof_offsets, commit_offsets, hpar, hg, hts);
    cudaStream_t s = c->stream;
    CK(c, cudaMemcpyAsync(x.in_proofs.p, proofs, proof_offsets[count], cudaMemcpyHostToDevice, s));
    CK(c, cudaMemcpyAsync(x.in_commit.p, commitments, 32 * commit_offsets[count], cudaMemcpyHostToDevice, s));
    CK(c, cudaMemcpyAsync(x.gather.p, hg, (size_t)A * sizeof(rp_gather), cudaMemcpyHostToDevice, s));
    CK(c, cudaMemcpyAsync(x.par.p, hpar, (size_t)C * sizeof(rp_params), cudaMemcpyHostToDevice, s));
    if (transcripts)
        for (uint32_t j = 0; j < C; j++)
            if (live[j]) {
                const size_t off = (size_t)X.cls[j].first * BP_TRANSCRIPT_BYTES;
                CK(c, cudaMemcpyAsync(x.tstates.as<uint8_t>() + off, hts + off, (size_t)live[j] * BP_TRANSCRIPT_BYTES, cudaMemcpyHostToDevice, s));
            }
    LAUNCH(c, KID_SMALL, k_rp_gather, A, 128, 0, s, x.in_proofs.as<uint8_t>(), x.in_commit.as<uint8_t>(), x.gather.as<rp_gather>(), x.proofs.as<uint8_t>(),
           x.commit.as<uint8_t>());
    CK(c, cudaGraphLaunch(R.graph, s));
    c->launches += R.graph_launches;
    CK(c, cudaMemcpyAsync(R.h_verdict.p, x.verdict.p, R.slots() * 4, cudaMemcpyDeviceToHost, s));
    CK(c, cudaMemcpyAsync(R.h_flag.p, x.flags.as<uint32_t>() + C, (size_t)C * 4, cudaMemcpyDeviceToHost, s));
    return BP_OK;
}

// bp_rangeproof_verify_mixed_begin (transcript: one state for every proof) and *_begin_transcripts (transcripts: one record per proof, in
// input order)
static int rp_mixed_begin(bp_ctx *c, bp_gens *gens, const uint8_t *transcript, const uint8_t *transcripts, size_t count, const uint8_t *proofs,
                          const uint64_t *proof_offsets, const uint32_t *n, const uint8_t *commitments, const uint64_t *commit_offsets, const uint8_t *seed) {
    if (!c) return BP_ERR_INVALID_ARGUMENT;
    if (!gens || !(transcript || transcripts) || !proofs || !proof_offsets || !n || !commitments || !commit_offsets || count == 0) {
        c->err = "bp_rangeproof_verify_mixed: null argument or no proofs"; return BP_ERR_INVALID_ARGUMENT;
    }
    BUSY_CHECK(c);
    rp_mixed_plan P;
    if (const char *why = rp_mixed_make_plan(count, proofs, proof_offsets, n, commit_offsets, gens->cap, gens->parties, P)) {
        c->err = std::string("bp_rangeproof_verify_mixed: ") + why; return BP_ERR_INVALID_ARGUMENT;
    }
    MixedState ms; ms.gens = gens; ms.verdicts = P.codes;
    if (P.cls.empty()) { ms.active = true; c->ms = std::move(ms); return BP_OK; }      // every proof's parameters are rejected: no kernel runs
    CK(c, cudaSetDevice(c->device));
    uint8_t seed_bytes[32];
    int rc = draw_seed(c, seed, seed_bytes);
    if (rc) return rc;
    MixReserve *R = c->mix.get();
    // profiling times each kernel: the graph's nodes are not timed, so a profiled call takes the direct path
    const bool fits = R && R->graph && !c->prof_on && R->gens_table == gens->d_table.p && R->gens_cap == gens->cap && R->gens_parties == gens->parties &&
                      proof_offsets[count] <= R->x.in_proofs.cap && 32 * commit_offsets[count] <= R->x.in_commit.cap && rp_mixed_fit(P, R->X, ms.live);
    if (fits) {
        ms.slots = rp_mixed_slots(P, R->X);
        rc = mix_queue(c, transcript, transcripts, count, proofs, proof_offsets, commitments, commit_offsets, seed_bytes, ms.live, ms.slots);
        if (rc) return rc;
        ms.reserved = true;
    } else {
        rc = rp_mixed_direct(c, gens, transcript, transcripts, count, proofs, proof_offsets, commitments, commit_offsets, seed_bytes, P, ms.verdicts.data());
        if (rc) return rc;
    }
    ms.active = true; c->ms = std::move(ms);          // only a fully queued verification is pending
    return BP_OK;
}
int bp_rangeproof_verify_mixed_begin(bp_ctx *c, bp_gens *gens, const uint8_t *transcript, size_t count, const uint8_t *proofs, const uint64_t *proof_offsets,
                                     const uint32_t *n, const uint8_t *commitments, const uint64_t *commit_offsets, const uint8_t *seed) {
    return rp_mixed_begin(c, gens, transcript, nullptr, count, proofs, proof_offsets, n, commitments, commit_offsets, seed);
}
int bp_rangeproof_verify_mixed_begin_transcripts(bp_ctx *c, bp_gens *gens, const uint8_t *transcripts, size_t count, const uint8_t *proofs,
                                                 const uint64_t *proof_offsets, const uint32_t *n, const uint8_t *commitments, const uint64_t *commit_offsets,
                                                 const uint8_t *seed) {
    return rp_mixed_begin(c, gens, nullptr, transcripts, count, proofs, proof_offsets, n, commitments, commit_offsets, seed);
}
int bp_rangeproof_verify_mixed_finish(bp_ctx *c, uint8_t *verdicts) {
    if (!c || !verdicts) return BP_ERR_INVALID_ARGUMENT;
    if (!c->ms.active) { c->err = "bp_rangeproof_verify_mixed_finish: no mixed verification is pending"; return BP_ERR_INVALID_ARGUMENT; }
    MixedState ms = std::move(c->ms); c->ms = MixedState{};
    if (ms.reserved) {
        MixReserve &R = *c->mix;
        CK(c, cudaSetDevice(c->device));
        CK(c, cudaStreamSynchronize(c->stream));
        bool redo = false;
        int rc = mix_reject(c, ms.gens, R.x, R.X, ms.live.data(), R.h_flag.as<uint32_t>(), &redo);
        if (rc) return rc;
        if (redo) {
            CK(c, cudaMemcpyAsync(R.h_verdict.p, R.x.verdict.p, R.slots() * 4, cudaMemcpyDeviceToHost, c->stream));
            CK(c, cudaStreamSynchronize(c->stream));
        }
        for (const auto &e : ms.slots) ms.verdicts[e.first] = (uint8_t)R.h_verdict.as<uint32_t>()[e.second];
    }
    memcpy(verdicts, ms.verdicts.data(), ms.verdicts.size());
    return BP_OK;
}
int bp_rangeproof_verify_mixed(bp_ctx *c, bp_gens *gens, const uint8_t *transcript, size_t count, const uint8_t *proofs, const uint64_t *proof_offsets,
                               const uint32_t *n, const uint8_t *commitments, const uint64_t *commit_offsets, const uint8_t *seed, uint8_t *verdicts) {
    if (c && !verdicts) { c->err = "bp_rangeproof_verify_mixed: null argument or no proofs"; return BP_ERR_INVALID_ARGUMENT; }
    int rc = bp_rangeproof_verify_mixed_begin(c, gens, transcript, count, proofs, proof_offsets, n, commitments, commit_offsets, seed);
    return rc ? rc : bp_rangeproof_verify_mixed_finish(c, verdicts);
}
int bp_rangeproof_verify_mixed_transcripts(bp_ctx *c, bp_gens *gens, const uint8_t *transcripts, size_t count, const uint8_t *proofs, const uint64_t *proof_offsets,
                                           const uint32_t *n, const uint8_t *commitments, const uint64_t *commit_offsets, const uint8_t *seed, uint8_t *verdicts) {
    if (c && !verdicts) { c->err = "bp_rangeproof_verify_mixed: null argument or no proofs"; return BP_ERR_INVALID_ARGUMENT; }
    int rc = bp_rangeproof_verify_mixed_begin_transcripts(c, gens, transcripts, count, proofs, proof_offsets, n, commitments, commit_offsets, seed);
    return rc ? rc : bp_rangeproof_verify_mixed_finish(c, verdicts);
}

// A reserve refused with BP_ERR_INVALID_ARGUMENT (a NULL argument, a call pending, or a mix rp_mixed_mix refuses: no class or more than
// 24, a duplicate class, zero capacity, a class the generators reject, too many slots or MSM terms) changes nothing: the context keeps the
// mix it had, and fitting calls still replay that mix's graph.  Once the arguments are accepted the old mix is dropped, so a BP_ERR_CUDA
// while sizing or capturing the new one leaves the context with no mix.
// bp_rangeproof_verify_mixed_reserve and, with exact, bp_rangeproof_verify_mixed_reserve_exact
static int rp_mixed_reserve(bp_ctx *c, bp_gens *gens, size_t n_classes, const uint32_t *n, const uint32_t *m, const uint32_t *capacity, bool exact) {
    if (!c) return BP_ERR_INVALID_ARGUMENT;
    if (!gens || !n || !m || !capacity) { c->err = "bp_rangeproof_verify_mixed_reserve: null argument"; return BP_ERR_INVALID_ARGUMENT; }
    BUSY_CHECK(c);
    auto R = std::make_unique<MixReserve>();
    if (const char *why = rp_mixed_mix(n_classes, n, m, capacity, gens->cap, gens->parties, R->X)) {
        c->err = std::string("bp_rangeproof_verify_mixed_reserve: ") + why; return BP_ERR_INVALID_ARGUMENT;
    }
    CK(c, cudaSetDevice(c->device));
    CK(c, cudaStreamSynchronize(c->stream));
    c->mix.reset();                                   // reserving again replaces the mix (a failure below leaves none)
    const rp_mixed_plan &X = R->X;
    const size_t C = X.cls.size(), A = R->slots();
    MixScratch &x = R->x;
    int rc = mix_ensure(c, x, X, X.proof_bytes, X.commit_bytes, true);
    if (rc) return rc;
    rc = msm_ensure(c, x.ar, msm_make_plan((uint32_t)X.terms, (uint32_t)C, 0));
    if (rc) return rc;
    XPlan XP;
    if (exact) {                  // one group per class, each class one unit
        const uint32_t *comb = x.flags.as<uint32_t>() + C;
        for (size_t k = 0; k < C; k++) XP.G.push_back(rp_xgroup_of(X.cls[k].g, mix_view(x, X.cls[k]), x.par.as<rp_params>() + k, comb + k, (uint32_t)X.cls[k].dyn));
        rc = rp_exact_prepare(c, R->xs, x.ar, XP);
        if (rc) return rc;
    }
    CK(c, R->h_stage.ensure(C * sizeof(rp_params) + A * (sizeof(rp_gather) + BP_TRANSCRIPT_BYTES)));
    CK(c, R->h_verdict.ensure(A * 4)); CK(c, R->h_flag.ensure(C * 4));
    CK(c, R->dstage.init(C * sizeof(rp_params)));
    R->M = rp_mix_classes_of(X, gens->cap, gens->parties);
    // the device planner's scratch for calls of up to one proof per slot; larger calls grow it
    CK(c, R->pl_code.ensure(A * 4, c->stream)); CK(c, R->pl_slot.ensure(A * 4, c->stream));
    CK(c, R->pl_hist.ensure((size_t)blocks_for(A, RP_MIX_BLOCK) * C * 4, c->stream));
    // built once: the step programs, the MSM offsets and every class's point map
    std::vector<rp_tr_step> hprog; std::vector<uint32_t> hoff;
    rc = mix_upload_layout(c, x, X, hprog, hoff);
    if (rc) return rc;
    for (const rp_mixed_class &K : X.cls) { rc = mix_point_map(c, gens, x, K, c->stream); if (rc) return rc; }
    // no call has filled a slot yet: zero inputs and empty classes for the warm pass below
    CK(c, cudaMemsetAsync(x.proofs.p, 0, X.proof_bytes, c->stream)); CK(c, cudaMemsetAsync(x.commit.p, 0, X.commit_bytes, c->stream));
    CK(c, cudaStreamSynchronize(c->stream));
    rc = graph_capture(c, &R->graph, &R->graph_launches, [&] { return mix_capture(c, gens, *R); });
    if (rc) return rc;
    if (exact) {
        rc = graph_capture(c, &R->xgraph, &R->xgraph_launches, [&] {
            const int r = mix_capture(c, gens, *R);
            return r ? r : rp_exact_chain(c, gens, R->xs, x.ar, XP, x.niels.as<ge_niels>());
        });
        if (rc) return rc;
    }
    R->gens_table = gens->d_table.p; R->gens_cap = gens->cap; R->gens_parties = gens->parties;
    // one pass with every class at capacity, so that the first real call finds module loading, the graph upload and the L2 working set done
    rp_params *hpar = R->h_stage.as<rp_params>();
    const uint8_t zero[BP_TRANSCRIPT_BYTES] = {};
    for (size_t k = 0; k < C; k++) mix_params(hpar[k], X.cls[k], x, (uint32_t)k, zero, false, zero, X.cls[k].g.count);
    CK(c, cudaMemcpyAsync(x.par.p, hpar, C * sizeof(rp_params), cudaMemcpyHostToDevice, c->stream));
    CK(c, cudaGraphLaunch(R->graph, c->stream));
    if (exact) CK(c, cudaGraphLaunch(R->xgraph, c->stream));
    CK(c, cudaStreamSynchronize(c->stream));
    c->mix = std::move(R);
    return BP_OK;
}
int bp_rangeproof_verify_mixed_reserve(bp_ctx *c, bp_gens *gens, size_t n_classes, const uint32_t *n, const uint32_t *m, const uint32_t *capacity) {
    return rp_mixed_reserve(c, gens, n_classes, n, m, capacity, false);
}
int bp_rangeproof_verify_mixed_reserve_exact(bp_ctx *c, bp_gens *gens, size_t n_classes, const uint32_t *n, const uint32_t *m, const uint32_t *capacity) {
    return rp_mixed_reserve(c, gens, n_classes, n, m, capacity, true);
}

// bp_rangeproof_verify_mixed_device (transcript: one host state for every proof) and *_device_transcripts (d_records: one device record
// per proof, in input order).  Every input is a device pointer; the planner kernels place the proofs in the reserved mix, the mix's graph
// runs unchanged on its arenas, and one kernel writes the verdicts in input order.  Nothing synchronises, unless a call of more proofs than
// the planner's scratch holds grows it.  exact: the *_exact forms, on the exact graph of a mix reserved with bp_rangeproof_verify_mixed_reserve_exact.
static int rp_mixed_device(bp_ctx *c, bp_gens *gens, const uint8_t *transcript, const void *d_records, size_t count, const void *d_proofs, size_t proof_bytes,
                           const void *d_proof_offsets, const void *d_n, const void *d_commitments, size_t n_commitments, const void *d_commit_offsets,
                           const uint8_t *seed, void *d_verdicts_u32, uint32_t *h_class_ok_pinned, bool exact = false) {
    if (!c) return BP_ERR_INVALID_ARGUMENT;
    if (!gens || !(transcript || d_records) || !d_proofs || !d_proof_offsets || !d_n || !d_commitments || !d_commit_offsets || !d_verdicts_u32 || count == 0) {
        c->err = "bp_rangeproof_verify_mixed_device: null argument or no proofs"; return BP_ERR_INVALID_ARGUMENT;
    }
    if (count >= RP_MIXED_MAX_PROOFS) { c->err = "bp_rangeproof_verify_mixed_device: more than 2^24 proofs"; return BP_ERR_INVALID_ARGUMENT; }
    if (!is_aligned(d_verdicts_u32, 4)) { c->err = "bp_rangeproof_verify_mixed_device: d_verdicts_u32 must be 4-byte aligned"; return BP_ERR_INVALID_ARGUMENT; }
    BUSY_CHECK(c);
    MixReserve *R = c->mix.get();
    if (!R || !R->graph || R->gens_table != gens->d_table.p || R->gens_cap != gens->cap || R->gens_parties != gens->parties) {
        c->err = "bp_rangeproof_verify_mixed_device: no mix is reserved on this context for this generator table"; return BP_ERR_INVALID_ARGUMENT;
    }
    if (exact && !R->xgraph) {
        c->err = "bp_rangeproof_verify_mixed_device_exact: the mix on this context is not reserved with bp_rangeproof_verify_mixed_reserve_exact"; return BP_ERR_INVALID_ARGUMENT;
    }
    CK(c, cudaSetDevice(c->device));
    MixScratch &x = R->x; const rp_mixed_plan &X = R->X; const rp_mix_classes &M = R->M;
    const uint32_t C = M.C, A = (uint32_t)R->slots(), n = (uint32_t)count, nb = blocks_for(count, RP_MIX_BLOCK);
    cudaStream_t s = c->stream;
    CK(c, R->pl_code.ensure((size_t)n * 4, s)); CK(c, R->pl_slot.ensure((size_t)n * 4, s)); CK(c, R->pl_hist.ensure((size_t)nb * C * 4, s));
    uint8_t seed_bytes[32];
    int rc = draw_seed(c, seed, seed_bytes);
    if (rc) return rc;
    // the parameter blocks with live = 0; k_mix_scan sets each class's live count on the device
    rp_params *hpar = nullptr;
    CK(c, R->dstage.acquire(hpar));
    for (uint32_t k = 0; k < C; k++) mix_params(hpar[k], X.cls[k], x, k, transcript, d_records != nullptr, seed_bytes, 0);
    CK(c, cudaMemcpyAsync(x.par.p, hpar, (size_t)C * sizeof(rp_params), cudaMemcpyHostToDevice, s));
    CK(c, R->dstage.record(s));
    const uint8_t *proofs = (const uint8_t *)d_proofs, *poff = (const uint8_t *)d_proof_offsets, *coff = (const uint8_t *)d_commit_offsets;
    uint32_t *code_cls = R->pl_code.as<uint32_t>(), *slot = R->pl_slot.as<uint32_t>(), *hist = R->pl_hist.as<uint32_t>();
    LAUNCH(c, KID_MIX_PLAN, k_mix_admit, nb, RP_MIX_BLOCK, 0, s, M, n, proofs, (uint64_t)proof_bytes, poff, (const uint8_t *)d_n, (uint64_t)n_commitments, coff,
           code_cls, slot, hist);
    LAUNCH(c, KID_MIX_PLAN, k_mix_scan, 1, 32 * C, 0, s, M, nb, hist, x.par.as<rp_params>());
    LAUNCH(c, KID_MIX_PLAN, k_mix_place, blocks_for(std::max(n, A), RP_MIX_BLOCK), RP_MIX_BLOCK, 0, s, M, n, A, poff, coff, (const uint8_t *)d_records, code_cls,
           slot, hist, x.par.as<rp_params>(), x.gather.as<rp_gather>(), x.tstates.as<uint8_t>());
    LAUNCH(c, KID_SMALL, k_rp_gather, A, 128, 0, s, proofs, (const uint8_t *)d_commitments, x.gather.as<rp_gather>(), x.proofs.as<uint8_t>(), x.commit.as<uint8_t>());
    CK(c, cudaGraphLaunch(exact ? R->xgraph : R->graph, s));
    c->launches += exact ? R->xgraph_launches : R->graph_launches;
    LAUNCH(c, KID_MIX_PLAN, k_mix_verdicts, nb, RP_MIX_BLOCK, 0, s, n, code_cls, slot, x.verdict.as<uint32_t>(), (uint32_t *)d_verdicts_u32);
    if (h_class_ok_pinned) CK(c, cudaMemcpyAsync(h_class_ok_pinned, x.flags.as<uint32_t>() + C, (size_t)C * 4, cudaMemcpyDeviceToHost, s));
    return BP_OK;
}
int bp_rangeproof_verify_mixed_device(bp_ctx *c, bp_gens *gens, const uint8_t *transcript, size_t count, const void *d_proofs, size_t proof_bytes,
                                      const void *d_proof_offsets, const void *d_n, const void *d_commitments, size_t n_commitments, const void *d_commit_offsets,
                                      const uint8_t *seed, void *d_verdicts_u32, uint32_t *h_class_ok_pinned) {
    return rp_mixed_device(c, gens, transcript, nullptr, count, d_proofs, proof_bytes, d_proof_offsets, d_n, d_commitments, n_commitments, d_commit_offsets, seed,
                           d_verdicts_u32, h_class_ok_pinned);
}
int bp_rangeproof_verify_mixed_device_transcripts(bp_ctx *c, bp_gens *gens, const void *d_transcripts, size_t count, const void *d_proofs, size_t proof_bytes,
                                                  const void *d_proof_offsets, const void *d_n, const void *d_commitments, size_t n_commitments,
                                                  const void *d_commit_offsets, const uint8_t *seed, void *d_verdicts_u32, uint32_t *h_class_ok_pinned) {
    return rp_mixed_device(c, gens, nullptr, d_transcripts, count, d_proofs, proof_bytes, d_proof_offsets, d_n, d_commitments, n_commitments, d_commit_offsets, seed,
                           d_verdicts_u32, h_class_ok_pinned);
}
int bp_rangeproof_verify_mixed_device_exact(bp_ctx *c, bp_gens *gens, const uint8_t *transcript, size_t count, const void *d_proofs, size_t proof_bytes,
                                            const void *d_proof_offsets, const void *d_n, const void *d_commitments, size_t n_commitments, const void *d_commit_offsets,
                                            const uint8_t *seed, void *d_verdicts_u32, uint32_t *h_class_ok_pinned) {
    return rp_mixed_device(c, gens, transcript, nullptr, count, d_proofs, proof_bytes, d_proof_offsets, d_n, d_commitments, n_commitments, d_commit_offsets, seed,
                           d_verdicts_u32, h_class_ok_pinned, true);
}
int bp_rangeproof_verify_mixed_device_exact_transcripts(bp_ctx *c, bp_gens *gens, const void *d_transcripts, size_t count, const void *d_proofs, size_t proof_bytes,
                                                        const void *d_proof_offsets, const void *d_n, const void *d_commitments, size_t n_commitments,
                                                        const void *d_commit_offsets, const uint8_t *seed, void *d_verdicts_u32, uint32_t *h_class_ok_pinned) {
    return rp_mixed_device(c, gens, nullptr, d_transcripts, count, d_proofs, proof_bytes, d_proof_offsets, d_n, d_commitments, n_commitments, d_commit_offsets, seed,
                           d_verdicts_u32, h_class_ok_pinned, true);
}

// ---------------------------------------------------------------------------------------------- indexed MSMs and the IPP prover session
static int check_scalars_canonical(const uint8_t *s, size_t n) {
    for (size_t i = 0; i < n; i++) if (sc_geq_l(sc_load(s + 32 * i))) return BP_ERR_NONCANONICAL_SCALAR;
    return BP_OK;
}

// Indexed MSMs over device inputs: scalars, term -> point map and offsets.  The n_dyn dynamic points are in c->niels, decompressed by
// upload_dyn_points, which left c->ok for k_flag_undecodable.  Nothing synchronised.
static int msm_indexed_device(bp_ctx *c, const bp_gens *gens, const uint8_t *d_scalars, const uint32_t *d_pidx, const uint32_t *d_offsets, uint32_t M, uint32_t T,
                              size_t n_dyn, uint8_t *d_outs, uint8_t *d_status) {
    CK(c, c->msm_err.ensure((size_t)M * 4, c->stream)); CK(c, c->results.ensure((size_t)M * sizeof(ge_ext), c->stream));
    CK(c, cudaMemsetAsync(c->msm_err.p, 0, (size_t)M * 4, c->stream));
    if (n_dyn) LAUNCH(c, KID_SMALL, k_flag_undecodable, blocks_for(T, 256), 256, 0, c->stream, c->ok.as<uint8_t>(), d_pidx, d_offsets, M, T, c->msm_err.as<uint32_t>());
    MsmArgs a{d_scalars, d_offsets, M, T, d_pidx, gens ? gens->d_table.as<ge_niels>() : nullptr, c->niels.as<ge_niels>(), c->msm_err.as<uint32_t>(), 0};
    return msm_to_outputs(c, a, d_outs, d_status);
}

int bp_msm_indexed_batch(bp_ctx *c, bp_gens *gens, const uint8_t *scalars, const uint32_t *point_idx, const uint8_t *dyn_points, size_t n_dyn,
                         const uint64_t *offsets, size_t n_msm, uint8_t *outs, uint8_t *status) {
    if (!c || !offsets || !outs || n_msm == 0) return BP_ERR_INVALID_ARGUMENT;
    size_t T = offsets[n_msm];
    if (offsets[0] != 0 || T == 0 || T >= (1u << 31) || !scalars || !point_idx) return BP_ERR_INVALID_ARGUMENT;
    BUSY_CHECK(c);
    CK(c, cudaSetDevice(c->device));
    if (point_index_error(point_idx, T, gens, dyn_points, n_dyn)) return BP_ERR_INVALID_ARGUMENT;
    std::vector<uint32_t> off32(n_msm + 1);
    for (size_t j = 0; j <= n_msm; j++) { if (j && offsets[j] < offsets[j - 1]) return BP_ERR_LENGTH_MISMATCH; off32[j] = (uint32_t)offsets[j]; }
    cudaStream_t s = c->stream;
    CK(c, c->in_scalars.ensure(T * 32, c->stream)); CK(c, c->in_offsets.ensure((n_msm + 1) * 4, c->stream)); CK(c, c->ix_pidx.ensure(T * 4, c->stream));
    CK(c, c->outs.ensure(n_msm * 32, c->stream)); CK(c, c->flags.ensure(n_msm, c->stream));
    CK(c, cudaMemcpyAsync(c->in_scalars.p, scalars, T * 32, cudaMemcpyHostToDevice, s));
    CK(c, cudaMemcpyAsync(c->in_offsets.p, off32.data(), (n_msm + 1) * 4, cudaMemcpyHostToDevice, s));
    CK(c, cudaMemcpyAsync(c->ix_pidx.p, point_idx, T * 4, cudaMemcpyHostToDevice, s));
    if (n_dyn) { int rc = upload_dyn_points(c, dyn_points, n_dyn); if (rc) return rc; }
    int rc = msm_indexed_device(c, gens, c->in_scalars.as<uint8_t>(), c->ix_pidx.as<uint32_t>(), c->in_offsets.as<uint32_t>(), (uint32_t)n_msm, (uint32_t)T, n_dyn,
                                c->outs.as<uint8_t>(), c->flags.as<uint8_t>());
    if (rc) return rc;
    return msm_download(c, n_msm, outs, status);
}

// ---------------------------------------------------------------------------------------------- R1CS and LinearProof batches
#define BP_MAX_BATCH_PROOFS (1u << 20)          // largest batch of bp_r1cs_verify_batch and bp_linear_verify_batch
// Reject path of an R1CS batch: every proof's own mega-check.  The same table and G/H sum kernels run with W = u1 and chunks of one
// proof, then one MSM launch over the rows [g | h | other terms] of a slice of proofs.
static int r1cs_recheck(bp_ctx *c, bp_gens *gens, const std::vector<r1cs_proof> &P, const std::vector<uint32_t> &term_off, uint32_t Nmax,
                        const sc *d_wL, const sc *d_wR, const sc *d_wO, const std::vector<uint8_t> &pre, uint8_t *verdicts) {
    cudaStream_t s = c->stream;
    const uint32_t np = (uint32_t)P.size();
    LAUNCH(c, KID_R1CS_TABLES, k_r1cs_tables, np, 128, 0, s, c->r1_proofs.as<r1cs_proof>(), c->r1_chal.as<uint8_t>(), 0, c->r1_heads.as<r1cs_head>(), c->r1_tabs.as<sc>());
    const unsigned thr = sum_threads(Nmax);
    return recheck_slices(c, np, r1cs_recheck_slice(np, Nmax), pre, verdicts, [&](uint32_t p0, uint32_t cnt, MsmArgs &a) {
        std::vector<uint32_t> row_off(cnt + 1, 0);
        for (uint32_t r = 0; r < cnt; r++) row_off[r + 1] = row_off[r] + 2 * P[p0 + r].padded_n + (term_off[p0 + r + 1] - term_off[p0 + r]);
        const uint32_t T = row_off[cnt];
        CK(c, c->r1_part.ensure((size_t)cnt * 2 * Nmax * sizeof(sc), c->stream)); CK(c, c->rk_scal.ensure((size_t)T * 32, c->stream)); CK(c, c->rk_pidx.ensure((size_t)T * 4, c->stream));
        CK(c, cudaMemcpyAsync(c->rk_offsets.p, row_off.data(), ((size_t)cnt + 1) * 4, cudaMemcpyHostToDevice, s));
        LAUNCH(c, KID_R1CS_GH_SUM, k_r1cs_gh_sum, dim3(blocks_for(Nmax, thr), cnt), thr, 0, s, c->r1_proofs.as<r1cs_proof>(), c->r1_heads.as<r1cs_head>(), c->r1_tabs.as<sc>(),
            d_wL, d_wR, d_wO, c->r1_decbad.as<uint32_t>(), p0, cnt, 1, Nmax, c->r1_part.as<sc>());
        LAUNCH(c, KID_R1CS_ROWS, k_r1cs_proof_rows, blocks_for(T, 256), 256, 0, s, c->rk_offsets.as<uint32_t>(), p0, cnt, c->r1_proofs.as<r1cs_proof>(), c->r1_part.as<sc>(), Nmax,
            c->r1_in_scal.as<uint8_t>(), c->r1_in_pidx.as<uint32_t>(), (uint32_t)gens->cap, (uint32_t)gens->parties, c->rk_scal.as<uint8_t>(), c->rk_pidx.as<uint32_t>());
        a = MsmArgs{c->rk_scal.as<uint8_t>(), c->rk_offsets.as<uint32_t>(), cnt, T, c->rk_pidx.as<uint32_t>(), gens->d_table.as<ge_niels>(), c->niels.as<ge_niels>(), nullptr, 0};
        return BP_OK;
    });
}

int bp_r1cs_verify_batch(bp_ctx *c, bp_gens *gens, size_t n_proofs, const uint32_t *dims, const uint8_t *chal, const uint8_t *wL, const uint8_t *wR, const uint8_t *wO,
                         const uint8_t *scalars, const uint32_t *point_idx, const uint8_t *dyn_points, size_t n_dyn, uint8_t *verdicts) {
    if (!c) return BP_ERR_INVALID_ARGUMENT;
    auto reject = [c](const std::string &m) { c->err = "bp_r1cs_verify_batch: " + m; return BP_ERR_INVALID_ARGUMENT; };
    if (!gens || !dims || !chal || !verdicts || n_proofs == 0) return reject("null argument or empty batch");
    if (n_proofs > BP_MAX_BATCH_PROOFS) return reject("more than 2^20 proofs");
    BUSY_CHECK(c);
    // per-proof layout of the flat inputs, and the argument checks
    std::vector<r1cs_proof> P(n_proofs); std::vector<uint32_t> term_off(n_proofs + 1, 0);
    size_t chal_n = 0, w_n = 0, tab_n = 0, terms = 0; uint32_t Nmax = 1;
    for (size_t j = 0; j < n_proofs; j++) {
        const uint32_t pn = dims[4 * j], n1 = dims[4 * j + 1], n = dims[4 * j + 2], nt = dims[4 * j + 3];
        if (pn == 0 || (pn & (pn - 1)) || n > pn || n1 > n) return reject("proof " + std::to_string(j) + ": inconsistent dims (padded_n a power of two, n1 <= n <= padded_n)");
        if (pn > gens->cap) return reject("proof " + std::to_string(j) + ": padded_n above the generators' capacity");
        r1cs_proof &p = P[j];
        p.padded_n = pn; p.n1 = n1; p.n = n; p.k = (uint32_t)lg2_exact(pn);
        p.chal_off = (uint32_t)chal_n; p.w_off = (uint32_t)w_n; p.tab_off = (uint32_t)tab_n; p.term_off = (uint32_t)terms;
        chal_n += R1CS_CHAL_USQ + p.k; w_n += n; tab_n += r1cs_tab_size(p.k); terms += nt;
        if (terms >= (1u << 30)) return reject("batch too large");
        term_off[j + 1] = (uint32_t)terms;
        Nmax = std::max(Nmax, pn);
    }
    if (2 * (size_t)Nmax + terms >= (1u << 31) || w_n >= (1u << 28) || tab_n >= (1u << 28)) return reject("batch too large");
    if ((w_n && (!wL || !wR || !wO)) || (terms && (!scalars || !point_idx))) return reject("null argument");
    if (const char *e = point_index_error(point_idx, terms, gens, dyn_points, n_dyn)) return reject(e);
    if (check_scalars_canonical(chal, chal_n) || (w_n && (check_scalars_canonical(wL, w_n) || check_scalars_canonical(wR, w_n) || check_scalars_canonical(wO, w_n))) ||
        (terms && check_scalars_canonical(scalars, terms))) { c->err = "bp_r1cs_verify_batch: non-canonical scalar"; return BP_ERR_NONCANONICAL_SCALAR; }
    CK(c, cudaSetDevice(c->device));
    cudaStream_t s = c->stream;
    const uint32_t np = (uint32_t)n_proofs, nch = (np + R1CS_CHUNK - 1) / R1CS_CHUNK, T = 2 * Nmax + (uint32_t)terms;
    CK(c, c->r1_proofs.ensure(n_proofs * sizeof(r1cs_proof), c->stream)); CK(c, c->r1_term_off.ensure((n_proofs + 1) * 4, c->stream)); CK(c, c->r1_chal.ensure(chal_n * 32, c->stream));
    CK(c, c->r1_w.ensure(3 * w_n * 32 + 32, c->stream)); CK(c, c->r1_in_scal.ensure(terms * 32 + 32, c->stream)); CK(c, c->r1_in_pidx.ensure(terms * 4 + 4, c->stream)); CK(c, c->r1_decbad.ensure(n_proofs * 4, c->stream));
    CK(c, c->r1_heads.ensure(n_proofs * sizeof(r1cs_head), c->stream)); CK(c, c->r1_tabs.ensure(tab_n * sizeof(sc), c->stream)); CK(c, c->r1_part.ensure((size_t)nch * 2 * Nmax * sizeof(sc), c->stream));
    CK(c, c->r1_scal.ensure((size_t)T * 32, c->stream)); CK(c, c->r1_pidx.ensure((size_t)T * 4, c->stream)); CK(c, c->in_offsets.ensure(8, c->stream));
    CK(c, c->results.ensure(sizeof(ge_ext), c->stream)); CK(c, c->outs.ensure(32, c->stream));
    sc *d_wL = c->r1_w.as<sc>(), *d_wR = d_wL + w_n, *d_wO = d_wR + w_n;        // wL | wR | wO
    CK(c, cudaMemcpyAsync(c->r1_proofs.p, P.data(), n_proofs * sizeof(r1cs_proof), cudaMemcpyHostToDevice, s));
    CK(c, cudaMemcpyAsync(c->r1_term_off.p, term_off.data(), (n_proofs + 1) * 4, cudaMemcpyHostToDevice, s));
    CK(c, cudaMemcpyAsync(c->r1_chal.p, chal, chal_n * 32, cudaMemcpyHostToDevice, s));
    if (w_n) {
        CK(c, cudaMemcpyAsync(d_wL, wL, w_n * 32, cudaMemcpyHostToDevice, s)); CK(c, cudaMemcpyAsync(d_wR, wR, w_n * 32, cudaMemcpyHostToDevice, s));
        CK(c, cudaMemcpyAsync(d_wO, wO, w_n * 32, cudaMemcpyHostToDevice, s));
    }
    if (terms) {
        CK(c, cudaMemcpyAsync(c->r1_in_scal.p, scalars, terms * 32, cudaMemcpyHostToDevice, s)); CK(c, cudaMemcpyAsync(c->r1_in_pidx.p, point_idx, terms * 4, cudaMemcpyHostToDevice, s));
    }
    CK(c, cudaMemsetAsync(c->r1_decbad.p, 0, n_proofs * 4, s));
    // 1. the dynamic points, decompressed once; a proof that uses an undecodable one is a VerificationError and is left out of the combination
    if (n_dyn) {
        int rc = upload_dyn_points(c, dyn_points, n_dyn);
        if (rc) return rc;
        if (terms) LAUNCH(c, KID_SMALL, k_flag_undecodable, blocks_for(terms, 256), 256, 0, s, c->ok.as<uint8_t>(), c->r1_in_pidx.as<uint32_t>(), c->r1_term_off.as<uint32_t>(),
                          np, (uint32_t)terms, c->r1_decbad.as<uint32_t>());
    }
    // 2. per-proof tables with W = rho u1;  3. G/H sums over chunks of R1CS_CHUNK proofs, then over the chunks;  4. the combined row, one MSM
    LAUNCH(c, KID_R1CS_TABLES, k_r1cs_tables, np, 128, 0, s, c->r1_proofs.as<r1cs_proof>(), c->r1_chal.as<uint8_t>(), 1, c->r1_heads.as<r1cs_head>(), c->r1_tabs.as<sc>());
    const unsigned thr = sum_threads(Nmax);
    LAUNCH(c, KID_R1CS_GH_SUM, k_r1cs_gh_sum, dim3(blocks_for(Nmax, thr), nch), thr, 0, s, c->r1_proofs.as<r1cs_proof>(), c->r1_heads.as<r1cs_head>(), c->r1_tabs.as<sc>(),
        d_wL, d_wR, d_wO, c->r1_decbad.as<uint32_t>(), 0, np, R1CS_CHUNK, Nmax, c->r1_part.as<sc>());
    LAUNCH(c, KID_R1CS_ROWS, k_r1cs_gh_total, blocks_for(2 * Nmax, 256), 256, 0, s, c->r1_part.as<sc>(), nch, Nmax, (uint32_t)gens->cap, (uint32_t)gens->parties,
        c->r1_scal.as<uint8_t>(), c->r1_pidx.as<uint32_t>());
    if (terms) LAUNCH(c, KID_R1CS_ROWS, k_r1cs_other_terms, blocks_for(terms, 256), 256, 0, s, c->r1_term_off.as<uint32_t>(), np, c->r1_chal.as<uint8_t>(), c->r1_proofs.as<r1cs_proof>(),
        c->r1_decbad.as<uint32_t>(), c->r1_in_scal.as<uint8_t>(), c->r1_in_pidx.as<uint32_t>(), Nmax, c->r1_scal.as<uint8_t>(), c->r1_pidx.as<uint32_t>());
    LAUNCH(c, KID_SMALL, k_fill_offsets, 1, 32, 0, s, 1, T, c->in_offsets.as<uint32_t>());
    MsmArgs a{c->r1_scal.as<uint8_t>(), c->in_offsets.as<uint32_t>(), 1, T, c->r1_pidx.as<uint32_t>(), gens->d_table.as<ge_niels>(), c->niels.as<ge_niels>(), nullptr, 0};
    int rc = msm_to_outputs(c, a, c->outs.as<uint8_t>(), nullptr);
    if (rc) return rc;
    uint8_t combined[32]; std::vector<uint32_t> dec_bad(n_proofs);
    CK(c, cudaMemcpyAsync(combined, c->outs.p, 32, cudaMemcpyDeviceToHost, s));
    CK(c, cudaMemcpyAsync(dec_bad.data(), c->r1_decbad.p, n_proofs * 4, cudaMemcpyDeviceToHost, s));
    CK(c, cudaStreamSynchronize(s));
    std::vector<uint8_t> pre(n_proofs);
    for (size_t j = 0; j < n_proofs; j++) pre[j] = dec_bad[j] ? BP_PROOF_VERIFICATION_ERROR : BP_PROOF_OK;
    // 5. when the combination fails, every proof is decided by its own mega-check
    return combined_verdicts(combined, pre, verdicts, [&] { return r1cs_recheck(c, gens, P, term_off, Nmax, d_wL, d_wR, d_wO, pre, verdicts); });
}

// Reject path of a LinearProof batch: every proof's own equation.  The same table and G sum kernels run with rho = 1 and chunks of one
// proof, then one MSM launch over the rows [B, F, G.. | C, S, L.., R..] of a slice of proofs.
static int lin_recheck(bp_ctx *c, bp_points *set, const lin_geom &g, uint32_t tiles, const std::vector<uint8_t> &pre, uint8_t *verdicts) {
    cudaStream_t s = c->stream;
    const uint32_t row = g.n + 2 + g.D;
    LAUNCH(c, KID_LIN_TABLES, k_lin_tables, g.count, 128, 0, s, g, c->ln_raw.as<uint8_t>(), c->ln_proofs.as<uint8_t>(), 0, c->ln_status.as<uint32_t>(),
           c->ln_heads.as<lin_head>(), c->ln_tabs.as<sc>());
    LAUNCH(c, KID_LIN_DYNAMIC, k_lin_dynamic, blocks_for(g.count, 128), 128, 0, s, g, c->ln_heads.as<lin_head>(), c->ln_decbad.as<uint32_t>(), c->ln_part_b0.as<sc>(), tiles,
           c->ln_proofs.as<uint8_t>(), c->ln_bf.as<sc>(), c->ln_scal.as<uint8_t>(), c->ln_pidx.as<uint32_t>());
    const unsigned thr = sum_threads(g.n);
    return recheck_slices(c, g.count, lin_recheck_slice(g.count, row), pre, verdicts, [&](uint32_t p0, uint32_t cnt, MsmArgs &a) {
        const uint32_t T = cnt * row;
        CK(c, c->ln_part_g.ensure((size_t)cnt * g.n * sizeof(sc), s)); CK(c, c->rk_scal.ensure((size_t)T * 32, s)); CK(c, c->rk_pidx.ensure((size_t)T * 4, s));
        LAUNCH(c, KID_LIN_G_SUM, k_lin_g_sum, dim3(tiles, cnt), thr, 0, s, g, c->ln_heads.as<lin_head>(), c->ln_tabs.as<sc>(), c->ln_b.as<uint8_t>(), c->ln_decbad.as<uint32_t>(),
               p0, cnt, 1, nullptr, c->ln_part_g.as<sc>(), c->ln_part_b0.as<sc>());
        LAUNCH(c, KID_LIN_ROWS, k_lin_proof_rows, blocks_for(T, 256), 256, 0, s, g, p0, cnt, nullptr, c->ln_part_g.as<sc>(), c->ln_bf.as<sc>(), c->ln_scal.as<uint8_t>(),
               c->rk_scal.as<uint8_t>(), c->rk_pidx.as<uint32_t>());
        LAUNCH(c, KID_SMALL, k_fill_offsets, blocks_for((size_t)cnt + 1, 256), 256, 0, s, cnt, row, c->rk_offsets.as<uint32_t>());
        a = MsmArgs{c->rk_scal.as<uint8_t>(), c->rk_offsets.as<uint32_t>(), cnt, T, c->rk_pidx.as<uint32_t>(), set->d_pts.as<ge_niels>(), c->niels.as<ge_niels>(), nullptr, 0};
        return BP_OK;
    });
}

int bp_linear_verify_batch(bp_ctx *c, bp_points *set, size_t n, size_t count, const uint8_t *transcripts, const uint8_t *proofs, size_t proof_len, const uint8_t *C,
                           const uint8_t *b, const uint8_t seed[32], uint8_t *verdicts) {
    if (!c) return BP_ERR_INVALID_ARGUMENT;
    auto reject = [c](const std::string &m) { c->err = "bp_linear_verify_batch: " + m; return BP_ERR_INVALID_ARGUMENT; };
    if (!set || !transcripts || !proofs || !C || !verdicts || count == 0 || (n && !b)) return reject("null argument or empty batch");
    if (count > BP_MAX_BATCH_PROOFS) return reject("more than 2^20 proofs");
    if (set->ctx != c) return reject("the point set belongs to another context");
    BUSY_CHECK(c);
    // LinearProof::from_bytes (linear_proof.rs:339-356), the generators' length and verification_scalars' length check: when one of
    // them fails for the whole call, every proof is decided here (a proof whose a or r is not canonical still gets FormatError)
    const size_t ne = proof_len / 32;
    uint8_t pv = BP_PROOF_OK; size_t k = 0;
    if (proof_len % 32 != 0 || ne < 3 || (ne - 3) % 2 != 0 || (ne - 3) / 2 >= 32) {
        pv = BP_PROOF_FORMAT_ERROR;
    } else {
        k = (ne - 3) / 2;
        if (set->n < n + 2) pv = BP_PROOF_INVALID_GENERATORS_LENGTH;
        else if (n != ((size_t)1 << k)) pv = BP_PROOF_VERIFICATION_ERROR;
    }
    if (pv != BP_PROOF_OK) {
        if (n && check_scalars_canonical(b, count * n)) { c->err = "bp_linear_verify_batch: non-canonical b"; return BP_ERR_NONCANONICAL_SCALAR; }
        for (size_t q = 0; q < count; q++) {
            const uint8_t *ar = proofs + q * proof_len + 64 * k + 32;
            verdicts[q] = pv != BP_PROOF_FORMAT_ERROR && (sc_geq_l(sc_load(ar)) || sc_geq_l(sc_load(ar + 32))) ? (uint8_t)BP_PROOF_FORMAT_ERROR : pv;
        }
        return BP_OK;
    }
    if (k > BP_MAX_LG_N) return reject("n above 2^20");
    CK(c, cudaSetDevice(c->device));
    cudaStream_t s = c->stream;
    const lin_geom g{(uint32_t)n, (uint32_t)k, (uint32_t)count, (uint32_t)proof_len, lin_dyn_terms((uint32_t)k)};
    const uint32_t thr = sum_threads(g.n), tiles = blocks_for(g.n, thr), nch = (g.count + LIN_CHUNK - 1) / LIN_CHUNK, T = g.n + 2 + g.count * g.D;
    CK(c, c->ln_tstate.ensure(count * BP_TRANSCRIPT_BYTES, s)); CK(c, c->ln_proofs.ensure(count * proof_len, s)); CK(c, c->ln_C.ensure(count * 32, s));
    CK(c, c->ln_b.ensure(count * n * 32, s)); CK(c, c->ln_seed.ensure(sizeof(lin_params), s)); CK(c, c->ln_raw.ensure(count * lin_raw_rows(g.k) * 64, s));
    CK(c, c->ln_status.ensure(count * 4, s)); CK(c, c->ln_decbad.ensure(count * 4, s)); CK(c, c->ln_heads.ensure(count * sizeof(lin_head), s));
    CK(c, c->ln_tabs.ensure(count * lin_tab_size(g.k) * sizeof(sc), s)); CK(c, c->ln_part_g.ensure((size_t)nch * n * sizeof(sc), s));
    CK(c, c->ln_part_b0.ensure((size_t)tiles * count * sizeof(sc), s)); CK(c, c->ln_bf.ensure(2 * count * sizeof(sc), s));
    CK(c, c->ln_scal.ensure((size_t)T * 32, s)); CK(c, c->ln_pidx.ensure((size_t)T * 4, s)); CK(c, c->in_offsets.ensure(8, s));
    CK(c, c->niels.ensure(count * g.D * sizeof(ge_niels), s)); CK(c, c->results.ensure(sizeof(ge_ext), s)); CK(c, c->outs.ensure(32, s));
    lin_params hp{};
    hp.live = g.count;                      // every slot live
    int rc = draw_seed(c, seed, hp.seed);
    if (rc) return rc;
    lin_params *d_par = c->ln_seed.as<lin_params>();
    CK(c, cudaMemcpyAsync(c->ln_tstate.p, transcripts, count * BP_TRANSCRIPT_BYTES, cudaMemcpyHostToDevice, s));
    CK(c, cudaMemcpyAsync(c->ln_proofs.p, proofs, count * proof_len, cudaMemcpyHostToDevice, s));
    CK(c, cudaMemcpyAsync(c->ln_C.p, C, count * 32, cudaMemcpyHostToDevice, s));
    CK(c, cudaMemcpyAsync(c->ln_b.p, b, count * n * 32, cudaMemcpyHostToDevice, s));
    CK(c, cudaMemcpyAsync(d_par, &hp, sizeof hp, cudaMemcpyHostToDevice, s));
    CK(c, cudaMemsetAsync(c->ln_decbad.p, 0, count * 4, s));
    // 1. the proofs' points, decompressed once;  2. transcript replay;  3. heads and tables with the weights rho;  4. G sums over chunks
    // of LIN_CHUNK proofs and b0 over tiles of indices;  5. per-proof scalars, then the static ones;  6. one MSM
    LAUNCH(c, KID_LIN_DECOMPRESS, k_lin_decompress, blocks_for((size_t)count * g.D, 128), 128, 0, s, g, d_par, c->ln_proofs.as<uint8_t>(), c->ln_C.as<uint8_t>(),
           c->niels.as<ge_niels>(), c->ln_decbad.as<uint32_t>());
    LAUNCH(c, KID_LIN_TRANSCRIPT, k_lin_transcript, blocks_for(count, LIN_TR_THREADS), LIN_TR_THREADS, 0, s, g, d_par, c->ln_tstate.as<uint8_t>(), c->ln_proofs.as<uint8_t>(),
           c->ln_C.as<uint8_t>(), c->ln_b.as<uint8_t>(), set->d_enc.as<uint8_t>(), c->ln_raw.as<uint8_t>(), c->ln_status.as<uint32_t>());
    LAUNCH(c, KID_LIN_TABLES, k_lin_tables, g.count, 128, 0, s, g, c->ln_raw.as<uint8_t>(), c->ln_proofs.as<uint8_t>(), 1, c->ln_status.as<uint32_t>(),
           c->ln_heads.as<lin_head>(), c->ln_tabs.as<sc>());
    LAUNCH(c, KID_LIN_G_SUM, k_lin_g_sum, dim3(tiles, nch), thr, 0, s, g, c->ln_heads.as<lin_head>(), c->ln_tabs.as<sc>(), c->ln_b.as<uint8_t>(), c->ln_decbad.as<uint32_t>(),
           0, g.count, LIN_CHUNK, nullptr, c->ln_part_g.as<sc>(), c->ln_part_b0.as<sc>());
    LAUNCH(c, KID_LIN_DYNAMIC, k_lin_dynamic, blocks_for(count, 128), 128, 0, s, g, c->ln_heads.as<lin_head>(), c->ln_decbad.as<uint32_t>(), c->ln_part_b0.as<sc>(), tiles,
           c->ln_proofs.as<uint8_t>(), c->ln_bf.as<sc>(), c->ln_scal.as<uint8_t>(), c->ln_pidx.as<uint32_t>());
    LAUNCH(c, KID_LIN_G_TOTAL, k_lin_g_total, g.n + 2, 32, 0, s, g, c->ln_part_g.as<sc>(), nch, c->ln_bf.as<sc>(), c->ln_scal.as<uint8_t>(), c->ln_pidx.as<uint32_t>());
    LAUNCH(c, KID_SMALL, k_fill_offsets, 1, 32, 0, s, 1, T, c->in_offsets.as<uint32_t>());
    MsmArgs a{c->ln_scal.as<uint8_t>(), c->in_offsets.as<uint32_t>(), 1, T, c->ln_pidx.as<uint32_t>(), set->d_pts.as<ge_niels>(), c->niels.as<ge_niels>(), nullptr, 0};
    rc = msm_to_outputs(c, a, c->outs.as<uint8_t>(), nullptr);
    if (rc) return rc;
    uint8_t combined[32]; uint32_t noncanon = 0; std::vector<uint32_t> status(count), dec_bad(count);
    CK(c, cudaMemcpyAsync(combined, c->outs.p, 32, cudaMemcpyDeviceToHost, s));
    CK(c, cudaMemcpyAsync(&noncanon, &d_par->noncanonical, 4, cudaMemcpyDeviceToHost, s));
    CK(c, cudaMemcpyAsync(status.data(), c->ln_status.p, count * 4, cudaMemcpyDeviceToHost, s));
    CK(c, cudaMemcpyAsync(dec_bad.data(), c->ln_decbad.p, count * 4, cudaMemcpyDeviceToHost, s));
    CK(c, cudaStreamSynchronize(s));
    if (noncanon) { c->err = "bp_linear_verify_batch: non-canonical b"; return BP_ERR_NONCANONICAL_SCALAR; }
    std::vector<uint8_t> pre(count);
    for (size_t q = 0; q < count; q++) pre[q] = status[q] != BP_PROOF_OK ? (uint8_t)status[q] : dec_bad[q] ? (uint8_t)BP_PROOF_VERIFICATION_ERROR : (uint8_t)BP_PROOF_OK;
    // 7. when the combination fails, every proof is decided by its own equation
    return combined_verdicts(combined, pre, verdicts, [&] { return lin_recheck(c, set, g, tiles, pre, verdicts); });
}

// The graph of a reserved LinearProof geometry, launches only: the chain of bp_linear_verify_batch at capacity, the verdicts, then the reject
// path of lin_recheck run by the device: an IF node (the combined MSM is not the identity) recomputes the tables and scalars with rho = 1,
// and a WHILE node checks P proofs per iteration by their own MSMs (lin_x_iters iterations; none when the combined check passed).
static int lin_chain(bp_ctx *c, const bp_points *set, LinReserve &R) {
    cudaStream_t s = c->stream;
    const lin_geom &g = R.g;
    const uint32_t thr = sum_threads(g.n), row = g.n + 2 + g.D, T2 = R.P * row;
    lin_params *par = R.par.as<lin_params>();
    uint32_t *status = R.status.as<uint32_t>(), *decbad = R.decbad.as<uint32_t>(), *verdict = R.verdict.as<uint32_t>(), *ctr = R.ctr.as<uint32_t>();
    lin_head *heads = R.heads.as<lin_head>();
    ge_ext *res = R.results.as<ge_ext>();
    CK(c, cudaMemsetAsync(R.decbad.p, 0, (size_t)g.count * 4, s));
    LAUNCH(c, KID_LIN_DECOMPRESS, k_lin_decompress, blocks_for((size_t)g.count * g.D, 128), 128, 0, s, g, par, R.proofs.as<uint8_t>(), R.C.as<uint8_t>(),
           R.niels.as<ge_niels>(), decbad);
    LAUNCH(c, KID_LIN_TRANSCRIPT, k_lin_transcript, blocks_for(g.count, LIN_TR_THREADS), LIN_TR_THREADS, 0, s, g, par, R.tstate.as<uint8_t>(), R.proofs.as<uint8_t>(),
           R.C.as<uint8_t>(), R.b.as<uint8_t>(), set->d_enc.as<uint8_t>(), R.raw.as<uint8_t>(), status);
    LAUNCH(c, KID_LIN_TABLES, k_lin_tables, g.count, 128, 0, s, g, R.raw.as<uint8_t>(), R.proofs.as<uint8_t>(), 1, status, heads, R.tabs.as<sc>());
    LAUNCH(c, KID_LIN_G_SUM, k_lin_g_sum, dim3(R.tiles, R.nch), thr, 0, s, g, heads, R.tabs.as<sc>(), R.b.as<uint8_t>(), decbad, 0, g.count, LIN_CHUNK, nullptr,
           R.part_g.as<sc>(), R.part_b0.as<sc>());
    LAUNCH(c, KID_LIN_DYNAMIC, k_lin_dynamic, blocks_for(g.count, 128), 128, 0, s, g, heads, decbad, R.part_b0.as<sc>(), R.tiles, R.proofs.as<uint8_t>(), R.bf.as<sc>(),
           R.scal.as<uint8_t>(), R.pidx.as<uint32_t>());
    LAUNCH(c, KID_LIN_G_TOTAL, k_lin_g_total, g.n + 2, 32, 0, s, g, R.part_g.as<sc>(), R.nch, R.bf.as<sc>(), R.scal.as<uint8_t>(), R.pidx.as<uint32_t>());
    MsmArgs a{R.scal.as<uint8_t>(), R.offsets.as<uint32_t>(), 1, R.T, R.pidx.as<uint32_t>(), set->d_pts.as<ge_niels>(), R.niels.as<ge_niels>(), nullptr, 0};
    int rc = msm_launch(c, R.ar, a, msm_make_plan(a.T, 1, 0), res, s);
    if (rc) return rc;
    LAUNCH(c, KID_SMALL, k_lin_verdicts, blocks_for(g.count, 128), 128, 0, s, g, par, status, decbad, res, verdict, ctr + 3);
    cudaGraphConditionalHandle failed = 0, loop = 0;
    rc = graph_cond(c, &failed);
    if (rc) return rc;
    LAUNCH(c, KID_SMALL, k_set_cond_unless_identity, 1, 32, 0, s, res, failed);
    rc = graph_body(c, failed, cudaGraphCondTypeIf, "LinearProof re-check tables", [&](cudaStream_t b) {
        LAUNCH(c, KID_LIN_TABLES, k_lin_tables, g.count, 128, 0, b, g, R.raw.as<uint8_t>(), R.proofs.as<uint8_t>(), 0, status, heads, R.tabs.as<sc>());
        LAUNCH(c, KID_LIN_DYNAMIC, k_lin_dynamic, blocks_for(g.count, 128), 128, 0, b, g, heads, decbad, R.part_b0.as<sc>(), R.tiles, R.proofs.as<uint8_t>(),
               R.bf.as<sc>(), R.scal.as<uint8_t>(), R.pidx.as<uint32_t>());
        return BP_OK;
    });
    if (rc) return rc;
    rc = graph_cond(c, &loop);
    if (rc) return rc;
    LAUNCH(c, KID_SMALL, k_lin_xloop_init, 1, 1, 0, s, par, g.count, R.P, ctr + 3, ctr, loop);
    return graph_body(c, loop, cudaGraphCondTypeWhile, "LinearProof re-check slices", [&](cudaStream_t b) {
        LAUNCH(c, KID_LIN_G_SUM, k_lin_g_sum, dim3(R.tiles, R.P), thr, 0, b, g, heads, R.tabs.as<sc>(), R.b.as<uint8_t>(), decbad, 0, R.P, 1, ctr, R.part_g.as<sc>(),
               R.part_b0.as<sc>());
        LAUNCH(c, KID_LIN_ROWS, k_lin_proof_rows, blocks_for(T2, 256), 256, 0, b, g, 0, R.P, ctr, R.part_g.as<sc>(), R.bf.as<sc>(), R.scal.as<uint8_t>(),
               R.rscal.as<uint8_t>(), R.rpidx.as<uint32_t>());
        MsmArgs ra{R.rscal.as<uint8_t>(), R.roffsets.as<uint32_t>(), R.P, T2, R.rpidx.as<uint32_t>(), set->d_pts.as<ge_niels>(), R.niels.as<ge_niels>(), nullptr, 0};
        int r = msm_launch(c, R.ar, ra, msm_make_plan(ra.T, ra.n_msm, 0), res, b);
        if (r) return r;
        LAUNCH(c, KID_SMALL, k_lin_xverdicts, blocks_for(R.P, 128), 128, 0, b, R.P, ctr, status, decbad, res, verdict);
        LAUNCH(c, KID_SMALL, k_rp_xloop_next, 1, 1, 0, b, ctr, loop);
        return BP_OK;
    });
}

int bp_linear_verify_reserve(bp_ctx *c, bp_points *set, size_t n, size_t capacity) {
    if (!c) return BP_ERR_INVALID_ARGUMENT;
    auto reject = [c](const std::string &m) { c->err = "bp_linear_verify_reserve: " + m; return BP_ERR_INVALID_ARGUMENT; };
    if (!set || set->ctx != c) return reject("the point set is null or belongs to another context");
    if (n == 0 || (n & (n - 1)) || n > ((size_t)1 << BP_MAX_LG_N)) return reject("n must be a power of two up to 2^20");
    if (set->n < n + 2) return reject("the point set has fewer than n + 2 points");
    if (capacity == 0 || capacity > BP_MAX_BATCH_PROOFS) return reject("capacity must be 1 .. 2^20");
    const uint32_t k = (uint32_t)lg2_exact(n), D = lin_dyn_terms(k);
    if (n + 2 + capacity * D >= ((size_t)1 << 31)) return reject("2^31 MSM terms or more");
    BUSY_CHECK(c);
    CK(c, cudaSetDevice(c->device));
    CK(c, cudaStreamSynchronize(c->stream));
    c->lin.reset();                                   // reserving again replaces the reservation (a failure below leaves none)
    auto R = std::make_unique<LinReserve>();
    cudaStream_t s = c->stream;
    lin_geom &g = R->g;
    g = lin_geom{(uint32_t)n, k, (uint32_t)capacity, 32 * (2 * k + 3), D};
    const uint32_t thr = sum_threads(g.n), row = g.n + 2 + D;
    R->tiles = blocks_for(g.n, thr); R->nch = (g.count + LIN_CHUNK - 1) / LIN_CHUNK; R->P = lin_x_slice(g.count, g.n, k); R->T = g.n + 2 + g.count * D;
    const size_t cap = capacity, T2 = (size_t)R->P * row;
    CK(c, R->tstate.alloc(cap * BP_TRANSCRIPT_BYTES)); CK(c, R->proofs.alloc(cap * g.proof_len)); CK(c, R->C.alloc(cap * 32)); CK(c, R->b.alloc(cap * n * 32));
    CK(c, R->par.alloc(sizeof(lin_params))); CK(c, R->raw.alloc(cap * lin_raw_rows(k) * 64)); CK(c, R->status.alloc(cap * 4)); CK(c, R->decbad.alloc(cap * 4));
    CK(c, R->heads.alloc(cap * sizeof(lin_head))); CK(c, R->tabs.alloc(cap * lin_tab_size(k) * sizeof(sc)));
    CK(c, R->part_g.alloc((size_t)std::max(R->nch, R->P) * n * sizeof(sc))); CK(c, R->part_b0.alloc((size_t)R->tiles * cap * sizeof(sc)));
    CK(c, R->bf.alloc(2 * cap * sizeof(sc))); CK(c, R->scal.alloc((size_t)R->T * 32)); CK(c, R->pidx.alloc((size_t)R->T * 4)); CK(c, R->offsets.alloc(8));
    CK(c, R->niels.alloc(cap * D * sizeof(ge_niels))); CK(c, R->rscal.alloc(T2 * 32)); CK(c, R->rpidx.alloc(T2 * 4)); CK(c, R->roffsets.alloc(((size_t)R->P + 1) * 4));
    CK(c, R->results.alloc((size_t)R->P * sizeof(ge_ext))); CK(c, R->verdict.alloc(cap * 4)); CK(c, R->ctr.alloc(4 * 4));
    int rc = msm_ensure(c, R->ar, msm_make_plan(R->T, 1, 0));
    if (!rc) rc = msm_ensure(c, R->ar, msm_make_plan((uint32_t)T2, R->P, 0));
    if (rc) return rc;
    CK(c, R->stage.init(sizeof(lin_params)));
    LAUNCH(c, KID_SMALL, k_fill_offsets, 1, 32, 0, s, 1, R->T, R->offsets.as<uint32_t>());
    LAUNCH(c, KID_SMALL, k_fill_offsets, blocks_for((size_t)R->P + 1, 256), 256, 0, s, R->P, row, R->roffsets.as<uint32_t>());
    // no call has filled a slot yet: zero inputs for the warm pass below
    for (DevBuf *z : {&R->tstate, &R->proofs, &R->C, &R->b, &R->niels}) CK(c, cudaMemsetAsync(z->p, 0, z->cap, s));
    CK(c, cudaStreamSynchronize(s));
    R->set = set;
    rc = graph_capture(c, &R->graph, &R->graph_launches, [&] { return lin_chain(c, set, *R); });
    if (rc) return rc;
    // one pass with every slot live, so that the first real call finds module loading, the graph upload and the L2 working set done
    lin_params hp{};
    hp.live = g.count;
    CK(c, cudaMemcpyAsync(R->par.p, &hp, sizeof hp, cudaMemcpyHostToDevice, s));
    CK(c, cudaGraphLaunch(R->graph, s));
    CK(c, cudaStreamSynchronize(s));
    c->lin = std::move(R);
    return BP_OK;
}

int bp_linear_verify_device(bp_ctx *c, bp_points *set, size_t n, size_t count, const void *d_transcripts, const void *d_proofs, size_t proof_len, const void *d_C,
                            const void *d_b, const uint8_t seed[32], void *d_verdicts_u32, uint32_t *h_ok_pinned) {
    if (!c) return BP_ERR_INVALID_ARGUMENT;
    auto reject = [c](const std::string &m) { c->err = "bp_linear_verify_device: " + m; return BP_ERR_INVALID_ARGUMENT; };
    if (!set || !d_transcripts || !d_proofs || !d_C || !d_b || !d_verdicts_u32) return reject("null argument");
    if (!is_aligned(d_verdicts_u32, 4)) return reject("d_verdicts_u32 must be 4-byte aligned");
    BUSY_CHECK(c);
    LinReserve *R = c->lin.get();
    if (!R || R->set != set || R->g.n != n) return reject("no LinearProof verification is reserved on this context for this point set and n");
    if (count == 0 || count > R->g.count) return reject("count must be 1 .. the reserved capacity");
    if (proof_len != R->g.proof_len) return reject("proof_len is not 32 (2 lg n + 3)");
    CK(c, cudaSetDevice(c->device));
    cudaStream_t s = c->stream;
    lin_params *hp = nullptr;
    CK(c, R->stage.acquire(hp));
    memset(hp, 0, sizeof *hp);
    hp->live = (uint32_t)count;
    int rc = draw_seed(c, seed, hp->seed);
    if (rc) return rc;
    CK(c, cudaMemcpyAsync(R->par.p, hp, sizeof *hp, cudaMemcpyHostToDevice, s));
    CK(c, R->stage.record(s));
    CK(c, cudaMemcpyAsync(R->tstate.p, d_transcripts, count * BP_TRANSCRIPT_BYTES, cudaMemcpyDeviceToDevice, s));
    CK(c, cudaMemcpyAsync(R->proofs.p, d_proofs, count * proof_len, cudaMemcpyDeviceToDevice, s));
    CK(c, cudaMemcpyAsync(R->C.p, d_C, count * 32, cudaMemcpyDeviceToDevice, s));
    CK(c, cudaMemcpyAsync(R->b.p, d_b, count * n * 32, cudaMemcpyDeviceToDevice, s));
    CK(c, cudaGraphLaunch(R->graph, s));
    c->launches += R->graph_launches;
    CK(c, cudaMemcpyAsync(d_verdicts_u32, R->verdict.p, count * 4, cudaMemcpyDeviceToDevice, s));
    if (h_ok_pinned) CK(c, cudaMemcpyAsync(h_ok_pinned, R->ctr.as<uint32_t>() + 3, 4, cudaMemcpyDeviceToHost, s));
    return BP_OK;
}

// Reject path of a mixed LinearProof call (layout P: linear_mixed.cuh): every admitted proof's own equation.  The tables and scalars run
// again with rho = 1 over every class; then each class is re-checked as lin_recheck re-checks a batch of its n, on its own slices of the
// arenas, with its dynamic scalars read from its segment of the combined row.  pre and verdicts in class order.
static int linm_recheck(bp_ctx *c, bp_points *set, const linm_plan &P, const std::vector<uint8_t> &pre, uint8_t *verdicts) {
    cudaStream_t s = c->stream;
    const uint32_t A = (uint32_t)P.order.size(), NC = (uint32_t)P.cls.size();
    const linm_class *d_cls = c->lm_meta.as<linm_class>();
    LAUNCH(c, KID_LINM_TABLES, k_linm_tables, A, 128, 0, s, d_cls, NC, c->ln_raw.as<uint8_t>(), c->ln_proofs.as<uint8_t>(), 0, c->ln_status.as<uint32_t>(),
           c->ln_heads.as<lin_head>(), c->ln_tabs.as<sc>());
    LAUNCH(c, KID_LINM_DYNAMIC, k_linm_dynamic, blocks_for(A, 128), 128, 0, s, d_cls, NC, A, P.nmax, c->ln_heads.as<lin_head>(), c->ln_decbad.as<uint32_t>(),
           c->ln_part_b0.as<sc>(), c->ln_proofs.as<uint8_t>(), c->ln_bf.as<sc>(), c->ln_scal.as<uint8_t>(), c->ln_pidx.as<uint32_t>());
    for (const linm_class &K : P.cls) {
        const lin_geom g{K.n, K.k, K.count, K.proof_len, K.D};
        const uint32_t row = g.n + 2 + g.D, thr = sum_threads(g.n), tiles = blocks_for(g.n, thr);
        const std::vector<uint8_t> pre_k(pre.begin() + K.first, pre.begin() + K.first + K.count);
        int rc = recheck_slices(c, K.count, lin_recheck_slice(K.count, row), pre_k, verdicts + K.first, [&](uint32_t p0, uint32_t cnt, MsmArgs &a) {
            const uint32_t T = cnt * row;
            CK(c, c->ln_part_g.ensure((size_t)cnt * g.n * sizeof(sc), s)); CK(c, c->rk_scal.ensure((size_t)T * 32, s)); CK(c, c->rk_pidx.ensure((size_t)T * 4, s));
            LAUNCH(c, KID_LIN_G_SUM, k_lin_g_sum, dim3(tiles, cnt), thr, 0, s, g, c->ln_heads.as<lin_head>() + K.first, c->ln_tabs.as<sc>() + K.tab_off,
                   c->ln_b.as<uint8_t>() + 32 * K.b_off, c->ln_decbad.as<uint32_t>() + K.first, p0, cnt, 1, nullptr, c->ln_part_g.as<sc>(), c->ln_part_b0.as<sc>() + K.b0_off);
            // k_lin_proof_rows reads proof r's dynamic scalars at g.n + 2 + r D; the class's are at Nmax + 2 + dyn + r D
            LAUNCH(c, KID_LIN_ROWS, k_lin_proof_rows, blocks_for(T, 256), 256, 0, s, g, p0, cnt, nullptr, c->ln_part_g.as<sc>(), c->ln_bf.as<sc>() + 2 * (size_t)K.first,
                   c->ln_scal.as<uint8_t>() + 32 * ((size_t)P.nmax + K.dyn - K.n), c->rk_scal.as<uint8_t>(), c->rk_pidx.as<uint32_t>());
            LAUNCH(c, KID_SMALL, k_fill_offsets, blocks_for((size_t)cnt + 1, 256), 256, 0, s, cnt, row, c->rk_offsets.as<uint32_t>());
            a = MsmArgs{c->rk_scal.as<uint8_t>(), c->rk_offsets.as<uint32_t>(), cnt, T, c->rk_pidx.as<uint32_t>(), set->d_pts.as<ge_niels>(),
                        c->niels.as<ge_niels>() + K.dyn, nullptr, 0};
            return BP_OK;
        });
        if (rc) return rc;
    }
    return BP_OK;
}

int bp_linear_verify_mixed(bp_ctx *c, bp_points *set, size_t count, const uint8_t *transcripts, const uint8_t *proofs, const uint64_t *proof_offsets,
                           const uint8_t *C, const uint8_t *b, const uint64_t *b_offsets, const uint8_t seed[32], uint8_t *verdicts) {
    if (!c) return BP_ERR_INVALID_ARGUMENT;
    auto reject = [c](const std::string &m) { c->err = "bp_linear_verify_mixed: " + m; return BP_ERR_INVALID_ARGUMENT; };
    if (!set || !transcripts || !proofs || !proof_offsets || !C || !b || !b_offsets || !verdicts || count == 0) return reject("null argument or empty batch");
    if (set->ctx != c) return reject("the point set belongs to another context");
    BUSY_CHECK(c);
    linm_plan P;
    if (const char *why = linm_make_plan(count, proofs, proof_offsets, b_offsets, set->n, P)) return reject(why);
    // b of a proof rejected on its parameters is checked here, as bp_linear_verify_batch checks it; the device checks the admitted ones
    for (size_t j = 0; j < count; j++)
        if (P.codes[j] != BP_PROOF_OK && check_scalars_canonical(b + 32 * b_offsets[j], b_offsets[j + 1] - b_offsets[j])) {
            c->err = "bp_linear_verify_mixed: non-canonical b"; return BP_ERR_NONCANONICAL_SCALAR;
        }
    if (P.cls.empty()) { memcpy(verdicts, P.codes.data(), count); return BP_OK; }
    CK(c, cudaSetDevice(c->device));
    cudaStream_t s = c->stream;
    const uint32_t A = (uint32_t)P.order.size(), NC = (uint32_t)P.cls.size(), T = (uint32_t)P.terms;
    // the caller's buffers as they are: b | C | proofs | transcript records, b and C at 32-byte offsets
    const size_t nb = 32 * b_offsets[count], oc = nb, op = oc + 32 * count, ot = op + proof_offsets[count], in_bytes = ot + count * BP_TRANSCRIPT_BYTES;
    std::vector<linm_gather> hg(A);
    for (uint32_t q = 0; q < A; q++) { const uint32_t j = P.order[q]; hg[q] = linm_gather{proof_offsets[j], b_offsets[j], j, 0}; }
    const size_t cls_bytes = (size_t)NC * sizeof(linm_class);
    CK(c, c->lm_in.ensure(in_bytes, s)); CK(c, c->lm_meta.ensure(cls_bytes + (size_t)A * sizeof(linm_gather), s));
    CK(c, c->ln_tstate.ensure((size_t)A * BP_TRANSCRIPT_BYTES, s)); CK(c, c->ln_proofs.ensure(P.proof_bytes, s)); CK(c, c->ln_C.ensure((size_t)A * 32, s));
    CK(c, c->ln_b.ensure(P.b_scalars * 32, s)); CK(c, c->ln_seed.ensure(sizeof(lin_params), s)); CK(c, c->ln_raw.ensure(P.raw_rows * 64, s));
    CK(c, c->ln_status.ensure((size_t)A * 4, s)); CK(c, c->ln_decbad.ensure((size_t)A * 4, s)); CK(c, c->ln_heads.ensure((size_t)A * sizeof(lin_head), s));
    CK(c, c->ln_tabs.ensure(P.tab_scalars * sizeof(sc), s)); CK(c, c->ln_part_g.ensure(P.part_scalars * sizeof(sc), s));
    CK(c, c->ln_part_b0.ensure(P.b0_scalars * sizeof(sc), s)); CK(c, c->ln_bf.ensure(2 * (size_t)A * sizeof(sc), s));
    CK(c, c->ln_scal.ensure((size_t)T * 32, s)); CK(c, c->ln_pidx.ensure((size_t)T * 4, s)); CK(c, c->in_offsets.ensure(8, s));
    CK(c, c->niels.ensure(P.dyn_points * sizeof(ge_niels), s)); CK(c, c->results.ensure(sizeof(ge_ext), s)); CK(c, c->outs.ensure(32, s));
    lin_params hp{};
    hp.live = A;
    int rc = draw_seed(c, seed, hp.seed);
    if (rc) return rc;
    lin_params *d_par = c->ln_seed.as<lin_params>();
    const linm_class *d_cls = c->lm_meta.as<linm_class>();
    uint8_t *in = c->lm_in.as<uint8_t>();
    if (nb) CK(c, cudaMemcpyAsync(in, b, nb, cudaMemcpyHostToDevice, s));
    CK(c, cudaMemcpyAsync(in + oc, C, 32 * count, cudaMemcpyHostToDevice, s));
    if (proof_offsets[count]) CK(c, cudaMemcpyAsync(in + op, proofs, proof_offsets[count], cudaMemcpyHostToDevice, s));
    CK(c, cudaMemcpyAsync(in + ot, transcripts, count * BP_TRANSCRIPT_BYTES, cudaMemcpyHostToDevice, s));
    CK(c, cudaMemcpyAsync(c->lm_meta.p, P.cls.data(), cls_bytes, cudaMemcpyHostToDevice, s));
    CK(c, cudaMemcpyAsync(c->lm_meta.as<uint8_t>() + cls_bytes, hg.data(), (size_t)A * sizeof(linm_gather), cudaMemcpyHostToDevice, s));
    CK(c, cudaMemcpyAsync(d_par, &hp, sizeof hp, cudaMemcpyHostToDevice, s));
    CK(c, cudaMemsetAsync(c->ln_decbad.p, 0, (size_t)A * 4, s));
    // 0. the admitted proofs gathered into class order, then the stages of bp_linear_verify_batch, one launch each over every class:
    // 1. decompression;  2. transcript replay;  3. heads and tables;  4. G sums over (tile, chunk) and b0;  5. per-proof scalars, then the
    // static ones;  6. one MSM over the combined row
    LAUNCH(c, KID_LINM_GATHER, k_linm_gather, A, 128, 0, s, d_cls, NC, reinterpret_cast<const linm_gather *>(c->lm_meta.as<uint8_t>() + cls_bytes), in + ot, in + op,
           in + oc, in, c->ln_tstate.as<uint8_t>(), c->ln_proofs.as<uint8_t>(), c->ln_C.as<uint8_t>(), c->ln_b.as<uint8_t>());
    LAUNCH(c, KID_LINM_DECOMPRESS, k_linm_decompress, blocks_for(P.dyn_points, 128), 128, 0, s, d_cls, NC, P.dyn_points, c->ln_proofs.as<uint8_t>(), c->ln_C.as<uint8_t>(),
           c->niels.as<ge_niels>(), c->ln_decbad.as<uint32_t>());
    LAUNCH(c, KID_LINM_TRANSCRIPT, k_linm_transcript, blocks_for(A, LIN_TR_THREADS), LIN_TR_THREADS, 0, s, d_cls, NC, A, d_par, c->ln_tstate.as<uint8_t>(),
           c->ln_proofs.as<uint8_t>(), c->ln_C.as<uint8_t>(), c->ln_b.as<uint8_t>(), set->d_enc.as<uint8_t>(), c->ln_raw.as<uint8_t>(), c->ln_status.as<uint32_t>());
    LAUNCH(c, KID_LINM_TABLES, k_linm_tables, A, 128, 0, s, d_cls, NC, c->ln_raw.as<uint8_t>(), c->ln_proofs.as<uint8_t>(), 1, c->ln_status.as<uint32_t>(),
           c->ln_heads.as<lin_head>(), c->ln_tabs.as<sc>());
    LAUNCH(c, KID_LINM_G_SUM, k_linm_g_sum, dim3(blocks_for(P.nmax, LINM_TILE), P.chunks), LINM_TILE, 0, s, d_cls, NC, c->ln_heads.as<lin_head>(), c->ln_tabs.as<sc>(),
           c->ln_b.as<uint8_t>(), c->ln_decbad.as<uint32_t>(), c->ln_part_g.as<sc>(), c->ln_part_b0.as<sc>());
    LAUNCH(c, KID_LINM_DYNAMIC, k_linm_dynamic, blocks_for(A, 128), 128, 0, s, d_cls, NC, A, P.nmax, c->ln_heads.as<lin_head>(), c->ln_decbad.as<uint32_t>(),
           c->ln_part_b0.as<sc>(), c->ln_proofs.as<uint8_t>(), c->ln_bf.as<sc>(), c->ln_scal.as<uint8_t>(), c->ln_pidx.as<uint32_t>());
    LAUNCH(c, KID_LINM_G_TOTAL, k_linm_g_total, P.nmax + 2, 32, 0, s, d_cls, NC, A, c->ln_part_g.as<sc>(), c->ln_bf.as<sc>(), c->ln_scal.as<uint8_t>(),
           c->ln_pidx.as<uint32_t>());
    LAUNCH(c, KID_SMALL, k_fill_offsets, 1, 32, 0, s, 1, T, c->in_offsets.as<uint32_t>());
    MsmArgs a{c->ln_scal.as<uint8_t>(), c->in_offsets.as<uint32_t>(), 1, T, c->ln_pidx.as<uint32_t>(), set->d_pts.as<ge_niels>(), c->niels.as<ge_niels>(), nullptr, 0};
    rc = msm_to_outputs(c, a, c->outs.as<uint8_t>(), nullptr);
    if (rc) return rc;
    uint8_t combined[32]; uint32_t noncanon = 0; std::vector<uint32_t> status(A), dec_bad(A);
    CK(c, cudaMemcpyAsync(combined, c->outs.p, 32, cudaMemcpyDeviceToHost, s));
    CK(c, cudaMemcpyAsync(&noncanon, &d_par->noncanonical, 4, cudaMemcpyDeviceToHost, s));
    CK(c, cudaMemcpyAsync(status.data(), c->ln_status.p, (size_t)A * 4, cudaMemcpyDeviceToHost, s));
    CK(c, cudaMemcpyAsync(dec_bad.data(), c->ln_decbad.p, (size_t)A * 4, cudaMemcpyDeviceToHost, s));
    CK(c, cudaStreamSynchronize(s));
    if (noncanon) { c->err = "bp_linear_verify_mixed: non-canonical b"; return BP_ERR_NONCANONICAL_SCALAR; }
    std::vector<uint8_t> pre(A), vq(A);
    for (uint32_t q = 0; q < A; q++) pre[q] = status[q] != BP_PROOF_OK ? (uint8_t)status[q] : dec_bad[q] ? (uint8_t)BP_PROOF_VERIFICATION_ERROR : (uint8_t)BP_PROOF_OK;
    // 7. when the combination fails, every admitted proof is decided by its own equation
    rc = combined_verdicts(combined, pre, vq.data(), [&] { return linm_recheck(c, set, P, pre, vq.data()); });
    if (rc) return rc;
    memcpy(verdicts, P.codes.data(), count);
    for (uint32_t q = 0; q < A; q++) verdicts[P.order[q]] = vq[q];
    return BP_OK;
}

// The graph of a reserved mix, launches only: the front end of bp_linear_verify_mixed over every slot of the mix (inert slots past each
// class's live count), one combined MSM and the verdicts, then the reject path of linm_recheck run by the device: an IF node (the combined
// MSM is not the identity) recomputes the tables and scalars with rho = 1, and one WHILE node per class checks R.P[c] of its proofs per
// iteration by their own MSMs, on the class's slices, as lin_chain does for a fixed geometry.
static int linm_chain(bp_ctx *c, const bp_points *set, LinMixReserve &R) {
    cudaStream_t s = c->stream;
    const linm_plan &X = R.X;
    const uint32_t A = R.slots(), NC = (uint32_t)X.cls.size();
    const linm_class *cls = R.cls.as<linm_class>();
    lin_params *par = R.par.as<lin_params>();
    uint32_t *status = R.status.as<uint32_t>(), *decbad = R.decbad.as<uint32_t>(), *verdict = R.verdict.as<uint32_t>(), *ctr = R.ctr.as<uint32_t>(), *flag = ctr + 4 * NC;
    lin_head *heads = R.heads.as<lin_head>();
    ge_ext *res = R.results.as<ge_ext>();
    CK(c, cudaMemsetAsync(R.decbad.p, 0, (size_t)A * 4, s));
    LAUNCH(c, KID_LINM_DECOMPRESS, k_linm_decompress, blocks_for(X.dyn_points, 128), 128, 0, s, cls, NC, X.dyn_points, R.proofs.as<uint8_t>(), R.C.as<uint8_t>(),
           R.niels.as<ge_niels>(), decbad);
    LAUNCH(c, KID_LINM_TRANSCRIPT, k_linm_transcript, blocks_for(A, LIN_TR_THREADS), LIN_TR_THREADS, 0, s, cls, NC, A, par, R.tstate.as<uint8_t>(), R.proofs.as<uint8_t>(),
           R.C.as<uint8_t>(), R.b.as<uint8_t>(), set->d_enc.as<uint8_t>(), R.raw.as<uint8_t>(), status);
    LAUNCH(c, KID_LINM_TABLES, k_linm_tables, A, 128, 0, s, cls, NC, R.raw.as<uint8_t>(), R.proofs.as<uint8_t>(), 1, status, heads, R.tabs.as<sc>());
    LAUNCH(c, KID_LINM_G_SUM, k_linm_g_sum, dim3(blocks_for(X.nmax, LINM_TILE), X.chunks), LINM_TILE, 0, s, cls, NC, heads, R.tabs.as<sc>(), R.b.as<uint8_t>(), decbad,
           R.part_g.as<sc>(), R.part_b0.as<sc>());
    LAUNCH(c, KID_LINM_DYNAMIC, k_linm_dynamic, blocks_for(A, 128), 128, 0, s, cls, NC, A, X.nmax, heads, decbad, R.part_b0.as<sc>(), R.proofs.as<uint8_t>(),
           R.bf.as<sc>(), R.scal.as<uint8_t>(), R.pidx.as<uint32_t>());
    LAUNCH(c, KID_LINM_G_TOTAL, k_linm_g_total, X.nmax + 2, 32, 0, s, cls, NC, A, R.part_g.as<sc>(), R.bf.as<sc>(), R.scal.as<uint8_t>(), R.pidx.as<uint32_t>());
    MsmArgs a{R.scal.as<uint8_t>(), R.offsets.as<uint32_t>(), 1, R.T, R.pidx.as<uint32_t>(), set->d_pts.as<ge_niels>(), R.niels.as<ge_niels>(), nullptr, 0};
    int rc = msm_launch(c, R.ar, a, msm_make_plan(a.T, 1, 0), res, s);
    if (rc) return rc;
    // every slot's verdict (par->live = the slot total; an inert slot's is never read)
    LAUNCH(c, KID_SMALL, k_lin_verdicts, blocks_for(A, 128), 128, 0, s, lin_geom{0, 0, A, 0, 0}, par, status, decbad, res, verdict, flag);
    cudaGraphConditionalHandle failed = 0;
    rc = graph_cond(c, &failed);
    if (rc) return rc;
    LAUNCH(c, KID_SMALL, k_set_cond_unless_identity, 1, 32, 0, s, res, failed);
    rc = graph_body(c, failed, cudaGraphCondTypeIf, "LinearProof mix re-check tables", [&](cudaStream_t b) {
        LAUNCH(c, KID_LINM_TABLES, k_linm_tables, A, 128, 0, b, cls, NC, R.raw.as<uint8_t>(), R.proofs.as<uint8_t>(), 0, status, heads, R.tabs.as<sc>());
        LAUNCH(c, KID_LINM_DYNAMIC, k_linm_dynamic, blocks_for(A, 128), 128, 0, b, cls, NC, A, X.nmax, heads, decbad, R.part_b0.as<sc>(), R.proofs.as<uint8_t>(),
               R.bf.as<sc>(), R.scal.as<uint8_t>(), R.pidx.as<uint32_t>());
        return BP_OK;
    });
    if (rc) return rc;
    for (uint32_t ci = 0; ci < NC; ci++) {
        const linm_class &K = X.cls[ci];
        const lin_geom g{K.n, K.k, K.count, K.proof_len, K.D};
        const uint32_t P = R.P[ci], row = g.n + 2 + g.D, T2 = P * row, thr = sum_threads(g.n), tiles = blocks_for(g.n, thr);
        uint32_t *cc = ctr + 4 * ci;
        cudaGraphConditionalHandle loop = 0;
        rc = graph_cond(c, &loop);
        if (rc) return rc;
        LAUNCH(c, KID_SMALL, k_lin_xloop_init, 1, 1, 0, s, R.cpar.as<lin_params>() + ci, g.count, P, flag, cc, loop);
        rc = graph_body(c, loop, cudaGraphCondTypeWhile, "LinearProof mix re-check slices", [&](cudaStream_t b) {
            LAUNCH(c, KID_LIN_G_SUM, k_lin_g_sum, dim3(tiles, P), thr, 0, b, g, heads + K.first, R.tabs.as<sc>() + K.tab_off, R.b.as<uint8_t>() + 32 * K.b_off,
                   decbad + K.first, 0, P, 1, cc, R.part_g.as<sc>(), R.part_b0.as<sc>() + K.b0_off);
            // k_lin_proof_rows reads proof r's dynamic scalars at g.n + 2 + r D; the class's are at Nmax + 2 + dyn + r D
            LAUNCH(c, KID_LIN_ROWS, k_lin_proof_rows, blocks_for(T2, 256), 256, 0, b, g, 0, P, cc, R.part_g.as<sc>(), R.bf.as<sc>() + 2 * (size_t)K.first,
                   R.scal.as<uint8_t>() + 32 * ((size_t)X.nmax + K.dyn - K.n), R.rscal.as<uint8_t>(), R.rpidx.as<uint32_t>());
            MsmArgs ra{R.rscal.as<uint8_t>(), R.roffsets.as<uint32_t>() + R.roff[ci], P, T2, R.rpidx.as<uint32_t>(), set->d_pts.as<ge_niels>(),
                       R.niels.as<ge_niels>() + K.dyn, nullptr, 0};
            int r = msm_launch(c, R.ar, ra, msm_make_plan(ra.T, ra.n_msm, 0), res, b);
            if (r) return r;
            LAUNCH(c, KID_SMALL, k_lin_xverdicts, blocks_for(P, 128), 128, 0, b, P, cc, status + K.first, decbad + K.first, res, verdict + K.first);
            LAUNCH(c, KID_SMALL, k_rp_xloop_next, 1, 1, 0, b, cc, loop);
            return BP_OK;
        });
        if (rc) return rc;
    }
    return BP_OK;
}

int bp_linear_verify_mixed_reserve(bp_ctx *c, bp_points *set, size_t n_classes, const uint32_t *n, const uint32_t *capacity) {
    if (!c) return BP_ERR_INVALID_ARGUMENT;
    auto reject = [c](const std::string &m) { c->err = "bp_linear_verify_mixed_reserve: " + m; return BP_ERR_INVALID_ARGUMENT; };
    if (!set || set->ctx != c) return reject("the point set is null or belongs to another context");
    if (!n || !capacity) return reject("null argument");
    BUSY_CHECK(c);
    auto R = std::make_unique<LinMixReserve>();
    const linm_plan &X = R->X;
    if (const char *why = linm_mix(n_classes, n, capacity, set->n, R->X)) return reject(why);
    CK(c, cudaSetDevice(c->device));
    CK(c, cudaStreamSynchronize(c->stream));
    c->linm.reset();                                  // reserving again replaces the mix (a failure below leaves none)
    cudaStream_t s = c->stream;
    const uint32_t NC = (uint32_t)X.cls.size(), A = R->slots();
    R->M = linm_mix_classes_of(X, set->n);
    R->T = (uint32_t)X.terms;
    size_t part_g = X.part_scalars, T2max = 0, noff = 0, Pmax = 1;
    for (const linm_class &K : X.cls) {
        const uint32_t P = lin_x_slice(K.count, K.n, K.k);
        R->P.push_back(P); R->roff.push_back((uint32_t)noff);
        noff += P + 1; Pmax = std::max<size_t>(Pmax, P);
        part_g = std::max(part_g, (size_t)P * K.n); T2max = std::max(T2max, (size_t)P * (K.n + 2 + K.D));
    }
    const size_t cap = A;
    CK(c, R->cls.alloc(NC * sizeof(linm_class))); CK(c, R->cpar.alloc(NC * sizeof(lin_params))); CK(c, R->gather.alloc(cap * sizeof(linm_gather)));
    CK(c, R->tstate.alloc(cap * BP_TRANSCRIPT_BYTES)); CK(c, R->proofs.alloc(X.proof_bytes)); CK(c, R->C.alloc(cap * 32)); CK(c, R->b.alloc(X.b_scalars * 32));
    CK(c, R->par.alloc(sizeof(lin_params))); CK(c, R->raw.alloc(X.raw_rows * 64)); CK(c, R->status.alloc(cap * 4)); CK(c, R->decbad.alloc(cap * 4));
    CK(c, R->heads.alloc(cap * sizeof(lin_head))); CK(c, R->tabs.alloc(X.tab_scalars * sizeof(sc))); CK(c, R->part_g.alloc(part_g * sizeof(sc)));
    CK(c, R->part_b0.alloc(X.b0_scalars * sizeof(sc))); CK(c, R->bf.alloc(2 * cap * sizeof(sc))); CK(c, R->scal.alloc((size_t)R->T * 32));
    CK(c, R->pidx.alloc((size_t)R->T * 4)); CK(c, R->offsets.alloc(8)); CK(c, R->niels.alloc(X.dyn_points * sizeof(ge_niels)));
    CK(c, R->rscal.alloc(T2max * 32)); CK(c, R->rpidx.alloc(T2max * 4)); CK(c, R->roffsets.alloc(noff * 4)); CK(c, R->results.alloc(Pmax * sizeof(ge_ext)));
    CK(c, R->verdict.alloc(cap * 4)); CK(c, R->ctr.alloc((4 * (size_t)NC + 4) * 4));
    // one arena for every MSM of the graph: they run one after another
    int rc = msm_ensure(c, R->ar, msm_make_plan(R->T, 1, 0));
    for (uint32_t ci = 0; ci < NC && !rc; ci++) {
        const linm_class &K = X.cls[ci];
        rc = msm_ensure(c, R->ar, msm_make_plan(R->P[ci] * (K.n + 2 + K.D), R->P[ci], 0));
    }
    if (rc) return rc;
    CK(c, R->stage.init(sizeof(lin_params)));
    // the planner's scratch for calls of up to one proof per slot; larger calls grow it
    CK(c, R->pl_code.ensure(cap * 4, s)); CK(c, R->pl_slot.ensure(cap * 4, s)); CK(c, R->pl_hist.ensure((size_t)blocks_for(cap, RP_MIX_BLOCK) * NC * 4, s));
    // the class table with every slot live, and the per-class parameters to match, for the warm pass below
    std::vector<lin_params> cp(NC);
    for (uint32_t ci = 0; ci < NC; ci++) { memset(&cp[ci], 0, sizeof(lin_params)); cp[ci].live = X.cls[ci].count; }
    CK(c, cudaMemcpyAsync(R->cls.p, X.cls.data(), NC * sizeof(linm_class), cudaMemcpyHostToDevice, s));
    CK(c, cudaMemcpyAsync(R->cpar.p, cp.data(), NC * sizeof(lin_params), cudaMemcpyHostToDevice, s));
    LAUNCH(c, KID_SMALL, k_fill_offsets, 1, 32, 0, s, 1, R->T, R->offsets.as<uint32_t>());
    for (uint32_t ci = 0; ci < NC; ci++) {
        const linm_class &K = X.cls[ci];
        LAUNCH(c, KID_SMALL, k_fill_offsets, blocks_for((size_t)R->P[ci] + 1, 256), 256, 0, s, R->P[ci], K.n + 2 + K.D, R->roffsets.as<uint32_t>() + R->roff[ci]);
    }
    // no call has filled a slot yet: zero inputs for the warm pass
    for (DevBuf *z : {&R->tstate, &R->proofs, &R->C, &R->b, &R->niels}) CK(c, cudaMemsetAsync(z->p, 0, z->cap, s));
    CK(c, cudaStreamSynchronize(s));
    R->set = set;
    rc = graph_capture(c, &R->graph, &R->graph_launches, [&] { return linm_chain(c, set, *R); });
    if (rc) return rc;
    // one pass with every slot live, so that the first real call finds module loading, the graph upload and the L2 working set done
    lin_params hp{};
    hp.live = A;
    CK(c, cudaMemcpyAsync(R->par.p, &hp, sizeof hp, cudaMemcpyHostToDevice, s));
    CK(c, cudaGraphLaunch(R->graph, s));
    CK(c, cudaStreamSynchronize(s));
    c->linm = std::move(R);
    return BP_OK;
}

// Every input is a device pointer; the planner kernels place the proofs in the reserved mix and set each class's live count, the gather
// copies the placed proofs into slot order, the mix's graph runs, and k_mix_verdicts writes the verdicts in input order.  Nothing
// synchronises, unless a call of more proofs than the planner's scratch holds grows it.
int bp_linear_verify_mixed_device(bp_ctx *c, bp_points *set, size_t count, const void *d_transcripts, const void *d_proofs, size_t proof_bytes,
                                  const void *d_proof_offsets, const void *d_C, const void *d_b, size_t n_b, const void *d_b_offsets, const uint8_t seed[32],
                                  void *d_verdicts_u32, uint32_t *h_ok_pinned) {
    if (!c) return BP_ERR_INVALID_ARGUMENT;
    auto reject = [c](const std::string &m) { c->err = "bp_linear_verify_mixed_device: " + m; return BP_ERR_INVALID_ARGUMENT; };
    if (!set || !d_transcripts || !d_proofs || !d_proof_offsets || !d_C || !d_b || !d_b_offsets || !d_verdicts_u32 || count == 0)
        return reject("null argument or no proofs");
    if (count >= RP_MIXED_MAX_PROOFS) return reject("2^24 proofs or more");
    if (!is_aligned(d_verdicts_u32, 4)) return reject("d_verdicts_u32 must be 4-byte aligned");
    BUSY_CHECK(c);
    LinMixReserve *R = c->linm.get();
    if (!R || R->set != set) return reject("no LinearProof mix is reserved on this context for this point set");
    CK(c, cudaSetDevice(c->device));
    cudaStream_t s = c->stream;
    const linm_mix_classes &M = R->M;
    const uint32_t NC = M.C, A = R->slots(), n = (uint32_t)count, nb = blocks_for(count, RP_MIX_BLOCK);
    CK(c, R->pl_code.ensure((size_t)n * 4, s)); CK(c, R->pl_slot.ensure((size_t)n * 4, s)); CK(c, R->pl_hist.ensure((size_t)nb * NC * 4, s));
    lin_params *hp = nullptr;
    CK(c, R->stage.acquire(hp));
    memset(hp, 0, sizeof *hp);
    hp->live = A;                                     // every slot; each class's live count is set on the device by k_linm_scan
    int rc = draw_seed(c, seed, hp->seed);
    if (rc) return rc;
    CK(c, cudaMemcpyAsync(R->par.p, hp, sizeof *hp, cudaMemcpyHostToDevice, s));
    CK(c, R->stage.record(s));
    const uint8_t *poff = (const uint8_t *)d_proof_offsets, *boff = (const uint8_t *)d_b_offsets;
    uint32_t *code_cls = R->pl_code.as<uint32_t>(), *slot = R->pl_slot.as<uint32_t>(), *hist = R->pl_hist.as<uint32_t>();
    LAUNCH(c, KID_MIX_PLAN, k_linm_admit, nb, RP_MIX_BLOCK, 0, s, M, n, (const uint8_t *)d_proofs, (uint64_t)proof_bytes, poff, boff, (uint64_t)n_b, code_cls, slot, hist);
    LAUNCH(c, KID_MIX_PLAN, k_linm_scan, 1, 32 * NC, 0, s, M, nb, hist, R->cls.as<linm_class>(), R->cpar.as<lin_params>());
    LAUNCH(c, KID_MIX_PLAN, k_linm_place, nb, RP_MIX_BLOCK, 0, s, M, n, poff, boff, code_cls, slot, hist, R->gather.as<linm_gather>());
    LAUNCH(c, KID_LINM_GATHER, k_linm_gather, A, 128, 0, s, R->cls.as<linm_class>(), NC, R->gather.as<linm_gather>(), (const uint8_t *)d_transcripts,
           (const uint8_t *)d_proofs, (const uint8_t *)d_C, (const uint8_t *)d_b, R->tstate.as<uint8_t>(), R->proofs.as<uint8_t>(), R->C.as<uint8_t>(),
           R->b.as<uint8_t>());
    CK(c, cudaGraphLaunch(R->graph, s));
    c->launches += R->graph_launches;
    LAUNCH(c, KID_MIX_PLAN, k_mix_verdicts, nb, RP_MIX_BLOCK, 0, s, n, code_cls, slot, R->verdict.as<uint32_t>(), (uint32_t *)d_verdicts_u32);
    if (h_ok_pinned) CK(c, cudaMemcpyAsync(h_ok_pinned, R->ctr.as<uint32_t>() + 4 * NC, 4, cudaMemcpyDeviceToHost, s));
    return BP_OK;
}

// ---------------------------------------------------------------------------------------------- inner-product prover, device-resident state
}  // extern "C"
struct bp_ippx {
    bp_ctx *ctx = nullptr; uint32_t N = 0, B = 0, n = 0;
    const ge_niels *d_static = nullptr; DevBuf own_pts;      // the gens table, or the session's own ge_niels [G (N) | H (N)]
    DevBuf d_q;                                              // ge_niels [B]: the points Q
    DevBuf a, b, cG, cH, gidx, hidx, scal, pidx, offs, in, outs;
};
extern "C" {
static int ippx_alloc(bp_ctx *c, size_t N, size_t B, bp_ippx **out) {
    if (!c || !out || N == 0 || (N & (N - 1)) || B == 0 || 2 * B * (N + 1) >= (1u << 31)) return BP_ERR_INVALID_ARGUMENT;      // power of two (inner_product_proof.rs:67)
    BUSY_CHECK(c);
    CK(c, cudaSetDevice(c->device));
    std::unique_ptr<bp_ippx> s(new bp_ippx()); s->ctx = c; s->N = (uint32_t)N; s->B = (uint32_t)B; s->n = (uint32_t)N;
    size_t BN = B * N;
    CK(c, s->d_q.alloc(B * sizeof(ge_niels)));
    for (DevBuf *b : {&s->a, &s->b, &s->cG, &s->cH}) CK(c, b->ensure(BN * sizeof(sc), c->stream));
    CK(c, s->gidx.ensure(N * 4, c->stream)); CK(c, s->hidx.ensure(N * 4, c->stream)); CK(c, s->scal.ensure(2 * B * (N + 1) * 32, c->stream)); CK(c, s->pidx.ensure(2 * B * (N + 1) * 4, c->stream));
    CK(c, s->offs.ensure((2 * B + 1) * 4, c->stream)); CK(c, s->in.ensure(std::max<size_t>(4 * BN * 32, 64 * B), c->stream)); CK(c, s->outs.ensure(64 * B, c->stream));
    *out = s.release(); return BP_OK;
}
// common tail of the two begin forms: Q points, scalar vectors (B x N canonical scalars each; Gf / Hf may be NULL = all ones); hands
// the session out in *out once it is loaded
static int ippx_load(std::unique_ptr<bp_ippx> s, const uint8_t *Q, const uint8_t *Gf, const uint8_t *Hf, const uint8_t *a, const uint8_t *b, bp_ippx **out) {
    bp_ctx *c = s->ctx; cudaStream_t st = c->stream; size_t BN = (size_t)s->B * s->N;
    for (const uint8_t *v : {a, b}) if (check_scalars_canonical(v, BN)) return BP_ERR_NONCANONICAL_SCALAR;
    for (const uint8_t *v : {Gf, Hf}) if (v && check_scalars_canonical(v, BN)) return BP_ERR_NONCANONICAL_SCALAR;
    uint8_t *din = s->in.as<uint8_t>();
    CK(c, cudaMemcpyAsync(din, a, BN * 32, cudaMemcpyHostToDevice, st)); CK(c, cudaMemcpyAsync(din + BN * 32, b, BN * 32, cudaMemcpyHostToDevice, st));
    if (Gf) CK(c, cudaMemcpyAsync(din + 2 * BN * 32, Gf, BN * 32, cudaMemcpyHostToDevice, st));
    if (Hf) CK(c, cudaMemcpyAsync(din + 3 * BN * 32, Hf, BN * 32, cudaMemcpyHostToDevice, st));
    ippx_geom g{s->N, s->B, s->n};
    LAUNCH(c, KID_SMALL, k_ippx_init, blocks_for(BN, 128), 128, 0, st, g, din, din + BN * 32, Gf ? din + 2 * BN * 32 : nullptr, Hf ? din + 3 * BN * 32 : nullptr,
           s->a.as<sc>(), s->b.as<sc>(), s->cG.as<sc>(), s->cH.as<sc>());
    CK(c, c->in_points.ensure((size_t)s->B * 32, c->stream));
    CK(c, cudaMemcpyAsync(c->in_points.p, Q, (size_t)s->B * 32, cudaMemcpyHostToDevice, st));
    int rc = decompress_all(c, c->in_points.as<uint8_t>(), s->B, s->d_q.as<ge_niels>());
    if (rc) return rc;
    LAUNCH(c, KID_SMALL, k_fill_offsets, blocks_for((size_t)2 * s->B + 1, 256), 256, 0, st, 2 * s->B, s->N + 1, s->offs.as<uint32_t>());
    *out = s.release(); return BP_OK;
}
int bp_ippx_begin(bp_ctx *c, bp_gens *gens, size_t n, size_t m, size_t n_proofs, const uint8_t *Q, const uint8_t *Gf, const uint8_t *Hf, const uint8_t *a, const uint8_t *b, bp_ippx **out) {
    if (!gens || !Q || !a || !b || n == 0 || m == 0 || n > gens->cap || m > gens->parties) return BP_ERR_INVALID_ARGUMENT;
    size_t N = n * m;
    int rc = ippx_alloc(c, N, n_proofs, out); if (rc) return rc;
    std::unique_ptr<bp_ippx> s(*out); *out = nullptr;        // handed out once loaded
    s->d_static = gens->d_table.as<ge_niels>();
    std::vector<uint32_t> idx = gens_nm_slots(gens, n, m);
    CK(c, cudaMemcpyAsync(s->gidx.p, idx.data(), N * 4, cudaMemcpyHostToDevice, c->stream)); CK(c, cudaMemcpyAsync(s->hidx.p, idx.data() + N, N * 4, cudaMemcpyHostToDevice, c->stream));
    CK(c, cudaStreamSynchronize(c->stream));
    return ippx_load(std::move(s), Q, Gf, Hf, a, b, out);
}
int bp_ippx_begin_points(bp_ctx *c, const uint8_t *G, const uint8_t *H, size_t N, size_t n_proofs, const uint8_t *Q, const uint8_t *Gf, const uint8_t *Hf, const uint8_t *a, const uint8_t *b, bp_ippx **out) {
    if (!G || !H || !Q || !a || !b) return BP_ERR_INVALID_ARGUMENT;
    int rc = ippx_alloc(c, N, n_proofs, out); if (rc) return rc;
    std::unique_ptr<bp_ippx> s(*out); *out = nullptr;        // handed out once loaded
    cudaStream_t st = c->stream;
    CK(c, s->own_pts.alloc(2 * N * sizeof(ge_niels)));
    s->d_static = s->own_pts.as<ge_niels>();
    std::vector<uint32_t> idx(2 * N);
    for (size_t q = 0; q < 2 * N; q++) idx[q] = (uint32_t)q;
    CK(c, c->in_points.ensure(2 * N * 32, c->stream));
    CK(c, cudaMemcpyAsync(c->in_points.p, G, N * 32, cudaMemcpyHostToDevice, st)); CK(c, cudaMemcpyAsync(c->in_points.as<uint8_t>() + N * 32, H, N * 32, cudaMemcpyHostToDevice, st));
    CK(c, cudaMemcpyAsync(s->gidx.p, idx.data(), N * 4, cudaMemcpyHostToDevice, st)); CK(c, cudaMemcpyAsync(s->hidx.p, idx.data() + N, N * 4, cudaMemcpyHostToDevice, st));
    rc = decompress_all(c, c->in_points.as<uint8_t>(), 2 * N, s->own_pts.as<ge_niels>());        // its synchronisation covers the index upload
    if (rc) return rc;
    return ippx_load(std::move(s), Q, Gf, Hf, a, b, out);
}
void bp_ippx_end(bp_ippx *s) { if (!s) return; cudaSetDevice(s->ctx->device); cudaStreamSynchronize(s->ctx->stream); delete s; }
size_t bp_ippx_current_len(const bp_ippx *s) { return s ? s->n : 0; }
// L and R of the current round for every proof (inner_product_proof.rs:87-113 / 153-163): LR_out = n_proofs x (L | R) compressed; synchronises
int bp_ippx_round(bp_ippx *s, uint8_t *LR_out) {
    if (!s || !LR_out || s->n < 2) return BP_ERR_INVALID_ARGUMENT;
    bp_ctx *c = s->ctx; BUSY_CHECK(c); CK(c, cudaSetDevice(c->device));
    cudaStream_t st = c->stream; ippx_geom g{s->N, s->B, s->n};
    uint32_t M = 2 * s->B, T = M * (s->N + 1);
    LAUNCH(c, KID_SMALL, k_ippx_inner, M, 128, 0, st, g, s->a.as<sc>(), s->b.as<sc>(), s->scal.as<uint8_t>());
    LAUNCH(c, KID_SMALL, k_ippx_rows, blocks_for((size_t)s->B * s->N, 128), 128, 0, st, g, s->a.as<sc>(), s->b.as<sc>(), s->cG.as<sc>(), s->cH.as<sc>(), s->gidx.as<uint32_t>(), s->hidx.as<uint32_t>(),
           s->scal.as<uint8_t>(), s->pidx.as<uint32_t>());
    CK(c, c->results.ensure((size_t)M * sizeof(ge_ext), c->stream));
    MsmArgs a{s->scal.as<uint8_t>(), s->offs.as<uint32_t>(), M, T, s->pidx.as<uint32_t>(), s->d_static, s->d_q.as<ge_niels>(), nullptr, 0};
    int rc = msm_to_outputs(c, a, s->outs.as<uint8_t>(), nullptr);
    if (rc) return rc;
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
    LAUNCH(c, KID_IPPX_FOLD, k_ippx_fold, blocks_for((size_t)s->B * s->N, 128), 128, 0, st, g, din, din + (size_t)s->B * 32, s->a.as<sc>(), s->b.as<sc>(), s->cG.as<sc>(), s->cH.as<sc>());
    CK(c, cudaStreamSynchronize(st));          // the staging buffer is reused by the next call
    s->n >>= 1;
    return BP_OK;
}
// the final a, b (inner_product_proof.rs:187-192): ab_out = n_proofs x (a | b)
int bp_ippx_finish(bp_ippx *s, uint8_t *ab_out) {
    if (!s || !ab_out || s->n != 1) return BP_ERR_INVALID_ARGUMENT;
    bp_ctx *c = s->ctx; BUSY_CHECK(c); CK(c, cudaSetDevice(c->device));
    ippx_geom g{s->N, s->B, s->n};
    LAUNCH(c, KID_SMALL, k_ippx_final, blocks_for(s->B, 128), 128, 0, c->stream, g, s->a.as<sc>(), s->b.as<sc>(), s->outs.as<uint8_t>());
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
    CK(c, cudaMemcpyAsync(d_dst, g->d_table.p, g->n_points * sizeof(ge_niels), cudaMemcpyDeviceToDevice, c->stream)); CK(c, cudaStreamSynchronize(c->stream)); return BP_OK;
}
int bp_gens_table_import(bp_gens *g, const void *d_src) {
    if (!g || !d_src) return BP_ERR_INVALID_ARGUMENT;
    bp_ctx *c = g->ctx; CK(c, cudaSetDevice(c->device));
    CK(c, cudaMemcpyAsync(g->d_table.p, d_src, g->n_points * sizeof(ge_niels), cudaMemcpyDeviceToDevice, c->stream)); CK(c, cudaStreamSynchronize(c->stream)); return BP_OK;
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

// test hooks: the element-wise operations of debug_ops.cuh on the device (they pin the PTX carry chains of fe.cuh, the device branch
// of sc_mont_mul and the lazy reduction of sc.cuh, and the point formulas of ge.cuh on any representative)
}  // extern "C"
#include "debug_ops.cuh"
extern "C" {
__global__ void k_debug_fe(int op, const uint8_t *a, const uint8_t *b, size_t n, uint8_t *out) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint8_t ab[32], bb[32], o[32]; ld32(ab, a + 32 * i); ld32(bb, b + 32 * i);
    debug_fe_op(op, ab, bb, o); st32(out + 32 * i, o);
}
// the fused single-proof path of bp_rangeproof_verify_batch whatever its routing rule says, for count <= RP_SINGLE_MAX_COUNT and
// lg(n m) <= RP_SINGLE_MAX_K (benchmarks/single_proof.py measures the crossover that sets the rule with it)
int bp_debug_rp_single_verify(bp_ctx *c, bp_gens *gens, const uint8_t *transcript, const uint8_t *proofs, size_t proof_len, const uint8_t *commitments,
                              size_t n, size_t m, size_t count, const uint8_t *seed, uint8_t *verdicts) {
    if (!c || !gens || !transcript || !proofs || !commitments || !verdicts) return BP_ERR_INVALID_ARGUMENT;
    BUSY_CHECK(c);
    rp_geom g{};
    if (rp_param_verdict(gens->cap, gens->parties, proof_len, n, m, &g) != BP_PROOF_OK || !rp_set_group(&g, count, 1)) return BP_ERR_INVALID_ARGUMENT;
    return rp_single_verify(c, gens, g, transcript, proofs, commitments, seed, verdicts);
}
int bp_debug_fe_op(bp_ctx *c, int op, const uint8_t *a, const uint8_t *b, size_t n, uint8_t *out) {
    if (!c || !a || !b || !out || n == 0 || op < 0 || op >= BP_DEBUG_FE_OPS) return BP_ERR_INVALID_ARGUMENT;
    BUSY_CHECK(c);
    CK(c, cudaSetDevice(c->device));
    CK(c, c->in_scalars.ensure(n * 32, c->stream)); CK(c, c->in_points.ensure(n * 32, c->stream)); CK(c, c->outs.ensure(n * 32, c->stream));
    CK(c, cudaMemcpyAsync(c->in_scalars.p, a, n * 32, cudaMemcpyHostToDevice, c->stream));
    CK(c, cudaMemcpyAsync(c->in_points.p, b, n * 32, cudaMemcpyHostToDevice, c->stream));
    LAUNCH(c, KID_SMALL, k_debug_fe, blocks_for(n, 128), 128, 0, c->stream, op, c->in_scalars.as<uint8_t>(), c->in_points.as<uint8_t>(), n, c->outs.as<uint8_t>());
    CK(c, cudaMemcpyAsync(out, c->outs.p, n * 32, cudaMemcpyDeviceToHost, c->stream));
    CK(c, cudaStreamSynchronize(c->stream));
    return BP_OK;
}

// raw limbs in and out: no conversion is added around the operation under test
__global__ void k_debug_sc(int op, const uint8_t *a, const uint8_t *b, size_t n, uint8_t *out) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (op == 8) {                                                  // sum32: one accumulator per 32 consecutive pairs
        if (i >= n / 32) return;
        uint8_t o[32]; debug_sc_sum32(a + 1024 * i, b + 1024 * i, o); st32(out + 32 * i, o);
        return;
    }
    if (i >= n) return;
    uint8_t ab[32], bb[32], o[32]; ld32(ab, a + 32 * i); ld32(bb, b + 32 * i);
    debug_sc_op(op, ab, bb, o); st32(out + 32 * i, o);
}
int bp_debug_sc_op(bp_ctx *c, int op, const uint8_t *a, const uint8_t *b, size_t n, uint8_t *out) {
    if (!c || !a || !b || !out || n == 0 || op < 0 || op >= BP_DEBUG_SC_OPS || (op == 8 && n % 32 != 0)) return BP_ERR_INVALID_ARGUMENT;
    BUSY_CHECK(c);
    CK(c, cudaSetDevice(c->device));
    const size_t n_out = op == 8 ? n / 32 : n;
    CK(c, c->in_scalars.ensure(n * 32, c->stream)); CK(c, c->in_points.ensure(n * 32, c->stream)); CK(c, c->outs.ensure(n_out * 32, c->stream));
    CK(c, cudaMemcpyAsync(c->in_scalars.p, a, n * 32, cudaMemcpyHostToDevice, c->stream));
    CK(c, cudaMemcpyAsync(c->in_points.p, b, n * 32, cudaMemcpyHostToDevice, c->stream));
    LAUNCH(c, KID_SMALL, k_debug_sc, blocks_for(n_out, 128), 128, 0, c->stream, op, c->in_scalars.as<uint8_t>(), c->in_points.as<uint8_t>(), n, c->outs.as<uint8_t>());
    CK(c, cudaMemcpyAsync(out, c->outs.p, n_out * 32, cudaMemcpyDeviceToHost, c->stream));
    CK(c, cudaStreamSynchronize(c->stream));
    return BP_OK;
}

__global__ void k_debug_ge(int op, const uint8_t *a, const uint8_t *b, size_t n, uint8_t *out) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint8_t ab[128], bb[128], o[128];
    for (int k = 0; k < 4; k++) { ld32(ab + 32 * k, a + 128 * i + 32 * k); ld32(bb + 32 * k, b + 128 * i + 32 * k); }
    debug_ge_op(op, ab, bb, o);
    for (int k = 0; k < 4; k++) st32(out + 128 * i + 32 * k, o + 32 * k);
}
int bp_debug_ge_op(bp_ctx *c, int op, const uint8_t *a, const uint8_t *b, size_t n, uint8_t *out) {
    if (!c || !a || !b || !out || n == 0 || op < 0 || op >= BP_DEBUG_GE_OPS) return BP_ERR_INVALID_ARGUMENT;
    BUSY_CHECK(c);
    CK(c, cudaSetDevice(c->device));
    CK(c, c->in_scalars.ensure(n * 128, c->stream)); CK(c, c->in_points.ensure(n * 128, c->stream)); CK(c, c->outs.ensure(n * 128, c->stream));
    CK(c, cudaMemcpyAsync(c->in_scalars.p, a, n * 128, cudaMemcpyHostToDevice, c->stream));
    CK(c, cudaMemcpyAsync(c->in_points.p, b, n * 128, cudaMemcpyHostToDevice, c->stream));
    LAUNCH(c, KID_SMALL, k_debug_ge, blocks_for(n, 128), 128, 0, c->stream, op, c->in_scalars.as<uint8_t>(), c->in_points.as<uint8_t>(), n, c->outs.as<uint8_t>());
    CK(c, cudaMemcpyAsync(out, c->outs.p, n * 128, cudaMemcpyDeviceToHost, c->stream));
    CK(c, cudaStreamSynchronize(c->stream));
    return BP_OK;
}

}  // extern "C"
