/*
 * litepose_b200 -- C ABI of the training kernels: NCHW depthwise convolution forward, input gradient and weight
 * gradient (csrc/dw_train.cu), bound by litepose_b200/_lib.py (TRAIN_SIGNATURES) and used by litepose_b200.train_dw.
 * Same library and the same conventions as include/litepose_b200.h (device pointers, caller-owned buffers, work on
 * `stream`, LP_OK or an error code with lp_last_error()); the tensors here are NCHW as the module tree trains them.
 *
 *   lp_dw_nchw_*         <- nn.Conv2d(C, C, k, stride, k // 2, groups=C, bias=False) forward and backward
 *                           (InvBottleneck.depth_conv, SepConv2d and the stem's depthwise of pose_mobilenet /
 *                           pose_simplenet; SuperSepConv2d and SuperInvBottleneck of pose_supermobilenet)
 */
#ifndef LITEPOSE_B200_TRAIN_H
#define LITEPOSE_B200_TRAIN_H

#include "litepose_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* ---- NCHW depthwise convolution for training (litepose_b200.train_dw) -----------
 * The depthwise convs of the module tree (nn.Conv2d, groups == C, no bias) in the layout it trains in:
 * x / dx NCHW [N,C,H,W], y / dy [N,C,Ho,Wo] with Ho = (H-1)/stride + 1, Wo likewise, w / dw [C][k][k];
 * k in {3, 5, 7}, stride 1 or 2, padding k/2, dilation 1.  dtype LP_DT_F32 or LP_DT_F16 for every tensor of a call;
 * pointers aligned to their element.  Any N, C >= 0 and H, W >= 1; N*C == 0 launches nothing (wgrad then writes
 * dw = +0 when C > 0).  Arithmetic (dw_train.cu states it in full): fp32 fmaf chains over the taps in a fixed order,
 * padding as +0 inputs; fp16 operands are converted exactly and the result is rounded once to fp16.
 * lp_dw_nchw_fwd:   y  = conv(x, w).
 * lp_dw_nchw_dgrad: dx = the input gradient of conv for dy (H, W are those of dx).
 * lp_dw_nchw_wgrad: dw = the weight gradient for x, dy: fp32 partials over fixed pixel ranges (the same bits on every
 *                   run and device), merged in fp64 in range order, rounded to fp32 (then fp16); workspace of
 *                   lp_dw_nchw_wgrad_workspace_bytes(...) bytes, 4-byte aligned (0 bytes for bad arguments). */
enum { LP_DT_F32 = 0, LP_DT_F16 = 1 };
int lp_dw_nchw_fwd(const void* x, const void* w, void* y, int N, int C, int H, int W, int k, int stride, int dtype,
                   lp_stream_t stream);
int lp_dw_nchw_dgrad(const void* dy, const void* w, void* dx, int N, int C, int H, int W, int k, int stride, int dtype,
                     lp_stream_t stream);
size_t lp_dw_nchw_wgrad_workspace_bytes(int N, int C, int H, int W, int k, int stride);
int lp_dw_nchw_wgrad(const void* x, const void* dy, void* dw, int N, int C, int H, int W, int k, int stride, int dtype,
                     void* workspace, size_t workspace_bytes, lp_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* LITEPOSE_B200_TRAIN_H */
