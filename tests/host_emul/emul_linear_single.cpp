// TEST-ONLY host build of the host part of the fused LinearProof path (linear_single.cuh): the CPU tier checks the shared-memory layout of
// every k against the per-block limit, the plan, and the routing rule at its edges.
#include "../../bulletproofs_b200/csrc/linear_single.cuh"

extern "C" {

// LIN_SINGLE_MAX_K, LIN_SINGLE_MAX_COUNT, LIN_SINGLE_SMEM_LIMIT, LIN_ROUTE_MAX_COUNT, LIN_ROUTE_MAX_N, RP_SINGLE_THREADS
void emul_lin_single_consts(uint64_t out[6]) {
    const uint64_t f[6] = {LIN_SINGLE_MAX_K, LIN_SINGLE_MAX_COUNT, LIN_SINGLE_SMEM_LIMIT, LIN_ROUTE_MAX_COUNT, LIN_ROUTE_MAX_N, RP_SINGLE_THREADS};
    for (int j = 0; j < 6; j++) out[j] = f[j];
}
// the plan of a launch whose longest proof has kmax rounds (c, W, nb, cl, wpc), and the layout of a proof of k rounds under it
// (wsum, niels, tabs, rec, lists, total); returns the proof's MSM terms
uint32_t emul_lin_single_layout(uint32_t k, uint32_t kmax, uint32_t plan[5], uint32_t lay[6]) {
    const rp_single_plan P = lin_single_plan(kmax);
    const uint32_t p[5] = {P.c, P.W, P.nb, P.cl, P.wpc};
    for (int j = 0; j < 5; j++) plan[j] = p[j];
    const lin_single_smem L = lin_single_layout(k, P);
    const uint32_t l[6] = {L.wsum, L.niels, L.tabs, L.rec, L.lists, L.total};
    for (int j = 0; j < 6; j++) lay[j] = l[j];
    return lin_single_terms(k);
}
int emul_lin_single_routed(size_t count, size_t nmax) { return lin_single_routed(count, nmax) ? 1 : 0; }

}
