/* TEST-ONLY: the entry points of include/bpmsm.h the host mirror never calls, so that the Python binding's symbol check passes on the
 * mock engine (see mock_bpmsm.c).  Every one of them fails like the real library does without a device. */
#include <stddef.h>
#define BP_ERR_CUDA 4
#define STUB(name) int name(void) { return BP_ERR_CUDA; }
STUB(bp_from_uniform_bytes_batch) STUB(bp_msm_batch_device) STUB(bp_decompress_batch) STUB(bp_compress_batch) STUB(bp_points_create_device)
STUB(bp_msm_points_device) STUB(bp_gens_device_table) STUB(bp_gens_create_empty) STUB(bp_rangeproof_verify_begin) STUB(bp_rangeproof_verify_finish)
STUB(bp_rangeproof_verify_batch_device) STUB(bp_rangeproof_verify_group_begin) STUB(bp_rangeproof_verify_group_finish) STUB(bp_rangeproof_verify_group_device)
STUB(bp_rangeproof_verify_reserve) STUB(bp_gens_table_export) STUB(bp_gens_table_import) STUB(bp_prof_enable) STUB(bp_prof_report) STUB(bp_prof_timeline) STUB(bp_debug_fe_op)
STUB(bp_debug_sc_op)
int bp_prof_kernel_count(void) { return 0; }
const char *bp_prof_kernel_name(int i) { (void)i; return ""; }
