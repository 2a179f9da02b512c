// Shared (host+device) pieces of the Pippenger pipeline: window geometry and signed-digit recoding.
#pragma once
#include "fe.cuh"

// Number of c-bit windows needed for scalars < 2^253 with the offset recoding below:
// s + K must fit in c*W bits where K = sum_w 2^(c*w + c - 1), which holds when c*W >= 255.
BP_HD int msm_num_windows(int c) { return (255 + c - 1) / c; }

// 288-bit little-endian integer big enough for s + K (c*W <= 255 + c - 1 <= 271 bits)
struct msm_wide { uint32_t v[9]; };

// s + K: after this every window's signed digit is independent of the others:
//   digit_w = window_w(s + K) - 2^(c-1)  in [-2^(c-1), 2^(c-1)),   sum_w digit_w 2^(c w) = s
BP_HD msm_wide msm_recode(const uint32_t s[8], int c, int W) {
    msm_wide k; for (int i = 0; i < 9; i++) k.v[i] = 0;
    for (int w = 0; w < W; w++) { int bit = c * w + c - 1; k.v[bit >> 5] |= 1u << (bit & 31); }
    msm_wide r; uint64_t carry = 0;
    for (int i = 0; i < 9; i++) { carry += (uint64_t)(i < 8 ? s[i] : 0u) + k.v[i]; r.v[i] = (uint32_t)carry; carry >>= 32; }
    return r;
}
BP_HD int msm_digit(const msm_wide &r, int w, int c) {
    int bit = c * w, idx = bit >> 5, sh = bit & 31;
    uint64_t two = (uint64_t)r.v[idx] | ((uint64_t)(idx + 1 < 9 ? r.v[idx + 1] : 0u) << 32);
    uint32_t raw = (uint32_t)(two >> sh) & ((1u << c) - 1u);
    return (int)raw - (1 << (c - 1));
}
// window size by terms per MSM (bench.py --workload msm --window c measures the alternatives).  Scalars are < l ~ 2^252, so a window size c that divides 252 leaves the
// top window nothing but the recoding carry: HALF of all terms land in its bucket 0 (one thread -- or one heavy-bucket block -- adds
// n/2 points while the other buckets hold n/2^(c-1)).  From 17 terms up the table therefore only uses c in {5, 8, 10, 11, 13, 15, 16}.
BP_HD int msm_pick_window(size_t avg_terms) {
    if (avg_terms <= 8) return 3;
    if (avg_terms <= 16) return 4;
    if (avg_terms <= 384) return 5;
    if (avg_terms <= 2560) return 8;
    if (avg_terms <= 8192) return 10;
    if (avg_terms <= 49152) return 11;
    if (avg_terms <= 262144) return 13;
    if (avg_terms <= 1572864) return 15;
    return 16;
}

// Branch selection of one pipeline pass (msm_make_plan / msm_launch), shared with the host-emulation tests so that a test can
// show its inputs reach the branch it is about.  avg_terms = ceil(T / n_msm), nb = 2^(c-1) buckets per window.
BP_HD size_t msm_avg_terms(size_t T, uint32_t n_msm) { return (T + n_msm - 1) / n_msm; }
// heavy-bucket threshold: far above the mean bucket size, and large enough that a block per bucket pays off.  A bucket of
// >= heavy_min entries is summed by a whole block (k_msm_order lists it, k_msm_accumulate leaves it to the heavy blocks).
BP_HD uint32_t msm_heavy_min(size_t avg_terms, uint32_t nb) {
    size_t h = 8 * (avg_terms / nb + 1);
    return (uint32_t)(h > 256 ? h : 256);
}
// lanes per light bucket in k_msm_accumulate: two once buckets hold >= 8 terms on average (half the serial chain per thread and
// twice the warps in flight for one extra addition per bucket)
BP_HD int msm_acc_split(size_t avg_terms, uint32_t nb, size_t n_buckets) { return avg_terms / nb >= 8 && n_buckets < 65536 ? 2 : 1; }
// window combination: up to this many MSMs the Horner chain is pure latency and k_msm_combine4 gives each MSM four lanes;
// more MSMs take k_msm_combine, one thread per MSM
#define MSM_COMBINE4_MAX_MSMS 256
BP_HD bool msm_use_combine4(uint32_t n_msm) { return n_msm <= MSM_COMBINE4_MAX_MSMS; }
