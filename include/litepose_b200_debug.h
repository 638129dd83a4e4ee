/*
 * litepose_b200 -- library state for tests and debugging, bound by litepose_b200/_lib.py (DEBUG_SIGNATURES).  Same
 * library as include/litepose_b200.h; nothing here launches device work.
 *
 * SM limit: the SM count the persistent kernels size their grids from (lp_pw1x1_f16, lp_fusion_deconv_f16 /
 * _act_f16, lp_head_pw_dual_f16, lp_dw7_project_f16, lp_head_fused_f16, lp_block_s1_f16, lp_block_s2_f16,
 * lp_stem_fused_f16, lp_bn_apply_f16).  It runs the partition an H100 PCIe, a MIG slice or a single SM would run.
 *   lp_set_sm_limit: n > 0 caps the count at n; n <= 0 restores the device's count; a cap above the device's count
 *     has no effect.  Process-wide: every thread's launches follow it.
 *   lp_get_sm_limit: the effective count for the current device.
 * Results do not depend on it: every output is the same bits at any grid.  A grid is fixed when its kernel is
 * launched, so a CUDA graph captured before the call keeps its old grids; build engines and capture graphs after
 * setting it.
 */
#ifndef LITEPOSE_B200_DEBUG_H
#define LITEPOSE_B200_DEBUG_H

#ifdef __cplusplus
extern "C" {
#endif

void lp_set_sm_limit(int n);
int lp_get_sm_limit(void);

#ifdef __cplusplus
}
#endif
#endif /* LITEPOSE_B200_DEBUG_H */
