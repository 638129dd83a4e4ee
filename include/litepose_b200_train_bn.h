/*
 * litepose_b200 -- C ABI of the train-mode BatchNorm kernels: NCHW batch-norm forward and backward with the ReLU /
 * ReLU6 that follows it fused (csrc/bn_nchw_train.cu), bound by litepose_b200/_lib.py (TRAIN_BN_SIGNATURES) and used
 * by litepose_b200.train_bn.  Same library and the same conventions as include/litepose_b200.h (device pointers,
 * caller-owned buffers, work on `stream`, LP_OK or an error code with lp_last_error()); LP_DT_* as in
 * include/litepose_b200_train.h.
 *
 *   lp_bn_nchw_*         <- nn.BatchNorm2d(C) in training mode (+ nn.ReLU / nn.ReLU6), forward and backward
 *                           (every BatchNorm of pose_mobilenet / pose_simplenet; SuperBatchNorm2d of
 *                           pose_supermobilenet on the leading C channels)
 */
#ifndef LITEPOSE_B200_TRAIN_BN_H
#define LITEPOSE_B200_TRAIN_BN_H

#include "litepose_b200_train.h"

#ifdef __cplusplus
extern "C" {
#endif

/* ---- NCHW train-mode BatchNorm (litepose_b200.train_bn) -------------------------
 * x / y / dy / dx NCHW [N,C,H,W], dtype LP_DT_F32 or LP_DT_F16 for all four; gamma, beta, running_mean, running_var,
 * dgamma, dbeta [C] fp32; saved [4][C] fp32 = (mean, invstd, scale, shift) of the forward, read by the backward.
 * act LP_ACT_NONE, LP_ACT_RELU or LP_ACT_RELU6 (the activation applied after the normalisation; NaN passes through).
 * N >= 1, C >= 0, H, W >= 1, N*H*W >= 2 (one value per channel is refused, as by F.batch_norm); C == 0 launches
 * nothing.  Pointers aligned to their element; workspace of lp_bn_nchw_workspace_bytes(N, C, H, W) bytes (0 for bad
 * arguments), 8-byte aligned.  Sums are fp64 over pixel ranges fixed by the shape, merged in a fixed order: the same
 * bits on every run and device (bn_nchw_train.cu states the arithmetic in full).
 * lp_bn_nchw_fwd: y = act(BN(x)) with the batch statistics (biased variance); running_mean / running_var are updated
 *                 in place to (1 - momentum) * running + momentum * batch statistic (unbiased variance).
 *                 0 <= momentum <= 1, eps >= 0.
 * lp_bn_nchw_bwd: for the incoming dy of y: dx, dgamma, dbeta, each optional (NULL: not computed); the activation's
 *                 mask is the forward's, recomputed from x and saved. */
size_t lp_bn_nchw_workspace_bytes(int N, int C, int H, int W);
int lp_bn_nchw_fwd(const void* x, const float* gamma, const float* beta, float* running_mean, float* running_var,
                   double momentum, double eps, void* y, float* saved, int N, int C, int H, int W, int act, int dtype,
                   void* workspace, size_t workspace_bytes, lp_stream_t stream);
int lp_bn_nchw_bwd(const void* x, const void* dy, const float* gamma, const float* saved, void* dx, float* dgamma,
                   float* dbeta, int N, int C, int H, int W, int act, int dtype, void* workspace, size_t workspace_bytes,
                   lp_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* LITEPOSE_B200_TRAIN_BN_H */
