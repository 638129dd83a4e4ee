/*
 * litepose_b200 -- C ABI of the H100 (sm_90a) LitePose inference kernels.
 *
 * The reference (mit-han-lab/litepose) is a pure Python/PyTorch project; its hot
 * path has no FFI of its own.  This header is the boundary a maintainer binds
 * with ctypes (see INTEGRATION.md) to replace, function by function:
 *
 *   lp_stem_*            <- LitePose.first            lib/models/pose_mobilenet.py:36-41
 *   lp_pw1x1_* / lp_dwconv_*
 *                        <- InvBottleneck.forward     lib/models/layers/layers.py:90-118
 *   lp_fusion_deconv_*   <- deconv_refined/raw + BN + ReLU
 *                                                     lib/models/pose_mobilenet.py:102-135,146-149
 *   lp_bn_*              <- train-mode BatchNorm2d (the super-network's BN recalibration,
 *                           calibrate_test.py:58-61; lib/models/layers/super_layers.py:19-28)
 *   lp_head_*            <- final_refined/final_raw (SepConv2d)
 *                                                     lib/models/pose_mobilenet.py:86-100,151-154
 *                                                     lib/models/layers/layers.py:120-133
 *   lp_nms_topk_*        <- HeatmapParser.nms/top_k   lib/core/group.py:131-176
 *   lp_tag_match_*       <- match_by_tag/py_max_match lib/core/group.py:19-97
 *   lp_adjust_refine_*   <- HeatmapParser.adjust/refine + scores
 *                                                     lib/core/group.py:178-291
 *   lp_glue_*            <- get_multi_stage_outputs/aggregate_results
 *                                                     lib/core/inference.py:75-208
 *
 * Conventions (modelled on the reference's own native plugin convention,
 * nano_demo/fast_utils/plugins.cpp: caller-allocated *_out buffers, raw pointers):
 *   - every pointer is a DEVICE pointer on the current CUDA device unless the
 *     parameter is documented as host memory (weight packing helpers);
 *   - the caller owns all inputs, outputs and workspaces; the library never
 *     allocates device memory, never frees and never retains a pointer;
 *   - work is enqueued on `stream` (a cudaStream_t); no hidden synchronisation;
 *   - every entry point returns LP_OK or an error code, never aborts;
 *     lp_last_error() gives a thread-local message for the last failure;
 *   - activations are NHWC fp16 between kernels; the stem reads the reference's
 *     NCHW input, the heads write the reference's NCHW fp32 outputs;
 *   - re-entrant per device/stream: no unguarded global state.
 */
#ifndef LITEPOSE_B200_H
#define LITEPOSE_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef void* lp_stream_t; /* cudaStream_t */

enum {
    LP_OK = 0,
    LP_ERR_BAD_ARG = 1,   /* shape / value out of the supported range */
    LP_ERR_ALIGN = 2,     /* pointer or stride not sufficiently aligned */
    LP_ERR_ARCH = 3,      /* device is not sm_90 */
    LP_ERR_CUDA = 4,      /* CUDA runtime / driver failure (launch, tensor map ...) */
    LP_ERR_CAPACITY = 5   /* workspace or output capacity too small */
};

enum { LP_ACT_NONE = 0, LP_ACT_RELU = 1, LP_ACT_RELU6 = 2 };

/* ---- library state ------------------------------------------------------ */
int lp_version(void);
const char* lp_last_error(void);
/* LP_OK iff the current device is compute capability 9.x */
int lp_device_check(void);
/* number of kernels this library launched (process-wide counter) */
uint64_t lp_launch_count(void);
void lp_reset_launch_count(void);

/* ---- M1: stem conv3x3 stride 2 (3 -> 32) + bias + ReLU6 ------------------
 * x: NCHW [N,3,H,W], fp32 (x_is_fp32 != 0) or fp16;  w: fp16 [32][27] (co, ci*9+ky*3+kx)
 * BN-folded;  bias: fp32 [32];  y: NHWC fp16 [N,H/2,W/2,32].  H, W even.
 * flip_x != 0 reads the image mirrored along W, i.e. computes the stem of
 * torch.flip(x, [3]) (the flip-test pass, lib/core/inference.py:120) without a copy. */
int lp_stem_conv3x3_s2(const void* x, int x_is_fp32, int flip_x, const void* w, const float* bias,
                       void* y, int N, int H, int W, lp_stream_t stream);
/* The same with the activation chosen: act LP_ACT_RELU6 (lp_stem_conv3x3_s2) or LP_ACT_NONE (bias may be NULL: the
 * raw convolution, rounded once to fp16, that the BN recalibration pass takes batch statistics of). */
int lp_stem_conv3x3_s2_act(const void* x, int x_is_fp32, int flip_x, const void* w, const float* bias,
                           void* y, int N, int H, int W, int act, lp_stream_t stream);

/* ---- M1 fused: the whole stem (conv3x3 s2 + BN + ReLU6 -> dw3x3 + BN + ReLU6 -> 1x1 + BN) in ONE kernel ----------
 * reference lib/models/pose_mobilenet.py:36-41.  x NCHW fp32/fp16 as above (flip_x = mirrored pass); w1_packed [32][64]
 * fp16: row co = the 27 BN-folded taps of output channel co (k = c*9 + ky*3 + kx), zero padded; w_dw [9][32] tap-major;
 * w_pw_packed / b_pw_packed from lp_pw1x1_pack(K = 32, N = C0); out [N,H/2,W/2,C0] fp16 NHWC.  flip_x must be 0 or 1
 * (LP_ERR_BAD_ARG otherwise).  The two 32-channel half-resolution intermediates never reach HBM.
 * An fp32 image is rounded to fp16 (round to nearest even) as it is loaded: the output for an fp32 x equals, bit for
 * bit, the output for x converted to fp16.  (lp_stem_conv3x3_s2 does not round: it convolves the fp32 values.)
 * lp_stem_fused_supported: H even, W % 4 == 0, C0 % 8 == 0, C0 <= 32. */
int lp_stem_fused_supported(int H, int W, int C0);
int lp_stem_fused_f16(const void* x, int x_is_fp32, int flip_x, const void* w1_packed, const float* b1, const void* w_dw,
                      const float* b_dw, const void* w_pw_packed, const float* b_pw_packed, void* out, int N, int H, int W,
                      int C0, lp_stream_t stream);

/* ---- M1/M2/M4: depthwise k x k (k in {3,5,7}), stride 1|2, pad k/2 ---------
 * x: NHWC fp16 [N,H,W,C];  w: fp16 [k*k][C] (tap-major, BN-folded);  bias fp32 [C];
 * y: NHWC fp16 [N,H/stride,W/stride,C].  C % 8 == 0; H, W even when stride == 2. */
int lp_dwconv_f16(const void* x, const void* w, const float* bias, void* y, int N, int C, int H,
                  int W, int k, int stride, int act, lp_stream_t stream);
/* Depthwise arithmetic of lp_dwconv_f16: 0 = every product accumulated in fp32, 1 = the k taps of one kernel
 * row accumulated in packed fp16 (HFMA2), row sums in fp32, 2 = fully packed fp16 (chains of two kernel rows folded
 * into a running fp16 total - the arithmetic of the fused block kernels).  Any other value (and the initial state)
 * selects the default: 2 for k = 7 and k = 3 (backbone, stem), 0 for k = 5 (heads).  Process-wide; set before
 * building engines / capturing graphs. */
void lp_set_dw_precision(int prec);
int lp_get_dw_precision(void);
/* The SM limit the persistent kernels size their grids from (a test and debug seam) is declared in
 * include/litepose_b200_debug.h. */

/* ---- M1/M2: pointwise 1x1 as a wgmma GEMM ---------------------------------
 * out[M,N] = act(a[M,K] * W^T + bias) (+ residual[M,N]);  a/out/residual fp16 row-major
 * (NHWC activations flattened, M = batch*H*W);  K % 8 == 0, N % 8 == 0.
 * Weights must be packed once (host memory in, host memory out): */
size_t lp_pw1x1_packed_elems(int K, int N);        /* fp16 elements */
size_t lp_pw1x1_packed_bias_elems(int N);          /* fp32 elements */
int lp_pw1x1_pack(const uint16_t* w_f16 /*[N][K] host*/, const float* bias /*[N] host or NULL*/,
                  int K, int N, uint16_t* w_packed /*host*/, float* bias_packed /*host*/);
int lp_pw1x1_f16(const void* a, const void* w_packed, const float* bias_packed, const void* residual,
                 void* out, int M, int K, int N, int act, lp_stream_t stream);

/* ---- M2 fused: depthwise 7x7 stride 1 (+bias +ReLU6) -> pointwise projection (+bias)(+residual)
 * (InvBottleneck.depth_conv + point_conv + identity add, lib/models/layers/layers.py:100-118) in one
 * kernel: the expanded depthwise output stays in shared memory as the wgmma A operand.
 * x [N,H,W,Ce] NHWC fp16; w_dw fp16 [49][Ce]; b_dw fp32 [Ce]; w_proj_packed / b_proj_packed from
 * lp_pw1x1_pack(K = Ce, N = Co); residual/out [N,H,W,Co] fp16.  Ce % 8 == 0, Co % 8 == 0, Co <= 160. */
int lp_dw7_project_f16(const void* x, const void* w_dw, const float* b_dw, const void* w_proj_packed,
                       const float* b_proj_packed, const void* residual, void* out, int N, int H, int W,
                       int Ce, int Co, lp_stream_t stream);

/* ---- M2 block-fused: one stride-1 InvBottleneck in ONE kernel ---------------------------------
 * reference lib/models/layers/layers.py:90-118 (inv -> depth_conv -> point_conv -> + identity).  The narrow haloed
 * input tile is expanded on the tensor cores inside the kernel; the 6x tensor never reaches HBM.
 * x [N,H,W,Cin] fp16 NHWC; w_exp_packed from lp_block_s1_pack_wexp ([Ce][Cin] BN-folded); b_exp [Ce];
 * w_dw tap-major [49][Ce]; b_dw [Ce]; w_proj_packed / b_proj_packed from lp_pw1x1_pack(K = Ce, N = Co);
 * identity != 0 adds x (Cin == Co).  Shapes the kernel can hold on chip: lp_block_s1_supported() (Cin <= 64, Co <= 64,
 * shared-memory budget on Ce); callers fall back to lp_pw1x1_f16 + lp_dw7_project_f16 otherwise. */
int lp_block_s1_supported(int Cin, int Ce, int Co);
size_t lp_block_s1_wexp_elems(int Cin, int Ce);     /* fp16 elements */
int lp_block_s1_pack_wexp(const uint16_t* w_f16 /*[Ce][Cin] host*/, int Cin, int Ce, uint16_t* out /*host*/);
int lp_block_s1_f16(const void* x, const void* w_exp_packed, const float* b_exp, const void* w_dw, const float* b_dw,
                    const void* w_proj_packed, const float* b_proj_packed, int identity, void* out, int N, int H, int W,
                    int Cin, int Ce, int Co, lp_stream_t stream);

/* ---- M2 block-fused: one stride-2 InvBottleneck (k = 7, no identity) in ONE kernel ------------------------------
 * Same arithmetic as lp_pw1x1_f16 (ReLU6) -> lp_dwconv_f16 (k7, stride 2, ReLU6, packed fp16) -> lp_pw1x1_f16, values
 * equal; the 6x tensor never reaches HBM.  x [N,H,W,Cin] fp16 NHWC, H and W even; out [N,H/2,W/2,Co].  Weights as for
 * lp_block_s1_f16 (w_exp_packed from lp_block_s1_pack_wexp).  Shapes: lp_block_s2_supported() (Cin 8 or 16, Co <= 64,
 * shared-memory budget on Ce); callers run the three-kernel chain otherwise. */
int lp_block_s2_supported(int Cin, int Ce, int Co);
int lp_block_s2_f16(const void* x, const void* w_exp_packed, const float* b_exp, const void* w_dw, const float* b_dw,
                    const void* w_proj_packed, const float* b_proj_packed, void* out, int N, int H, int W, int Cin,
                    int Ce, int Co, lp_stream_t stream);

/* ---- M3: fusion deconv level ----------------------------------------------
 * out = ReLU(ConvT4x4s2p1(refined) + ConvT4x4s2p1(raw) + bias), one kernel.
 * refined NHWC fp16 [N,H,W,Cr], raw [N,H,W,Cw], out [N,2H,2W,Co].
 * w_refined/w_raw: BN-scaled fp16 in the reference layout [Cin][Co][4][4] (host).
 * Single branch (pose_simplenet's deconv_bnrelu(deconv_refined(refined)), no deconv_raw): Cw == 0 with
 * w_raw / raw NULL; the K program then holds the refined channels only (row kernel: K = Cr rounded up to
 * 16, taken for Cr <= 64).  Every Cw > 0 call and its packed layout are those of the two-branch form. */
size_t lp_deconv_packed_elems(int Cr, int Cw, int Co);
size_t lp_deconv_packed_bias_elems(int Co);
int lp_deconv_pack(const uint16_t* w_refined, const uint16_t* w_raw, const float* bias, int Cr, int Cw,
                   int Co, uint16_t* w_packed, float* bias_packed);
int lp_fusion_deconv_f16(const void* refined, const void* raw, const void* w_packed,
                         const float* bias_packed, void* out, int N, int H, int W, int Cr, int Cw,
                         int Co, lp_stream_t stream);
/* The same with the activation chosen: act LP_ACT_RELU (lp_fusion_deconv_f16) or LP_ACT_NONE (the raw sum of both
 * branches + bias, for the BN recalibration pass).  Same kernel selection and accumulation order. */
int lp_fusion_deconv_act_f16(const void* refined, const void* raw, const void* w_packed,
                             const float* bias_packed, void* out, int N, int H, int W, int Cr, int Cw,
                             int Co, int act, lp_stream_t stream);

/* ---- train-mode BatchNorm (BN recalibration) -------------------------------
 * lp_bn_stats_f16: batch statistics of x NHWC fp16 [M, C] (M = N*H*W pixels) and, per channel c,
 *   scale[c] = gamma / sqrt(var + eps), shift[c] = beta - mean * scale (var the biased variance),
 *   new_mean[c] = (1 - momentum) * running_mean + momentum * mean,
 *   new_var[c]  = (1 - momentum) * running_var + momentum * var * M / (M - 1);
 * sets *nonfinite = 1 (and leaves it otherwise) when one of those values is not finite.  gamma, beta, running_*, scale,
 * shift, new_* fp32 [C].  Sums in fp64 over fixed pixel ranges, merged in a fixed order (bn_train.cu states it): the
 * result is the same bits on every run.  M >= 2, C % 8 == 0; workspace of lp_bn_stats_workspace_bytes(M, C) bytes,
 * x and workspace 16-byte aligned.
 * lp_bn_apply_f16: y = act(fmaf(x, scale, shift)) (+ residual) in fp32, one rounding to fp16; x, residual, y [M, C];
 * y may be x.  ReLU maps v to (v > 0 ? v : +0), ReLU6 then to min(v, 6).  C % 8 == 0, 16-byte aligned pointers. */
size_t lp_bn_stats_workspace_bytes(int M, int C);
int lp_bn_stats_f16(const void* x, int M, int C, const float* gamma, const float* beta, const float* running_mean,
                    const float* running_var, double momentum, double eps, float* scale, float* shift, float* new_mean,
                    float* new_var, int* nonfinite, void* workspace, size_t workspace_bytes, lp_stream_t stream);
int lp_bn_apply_f16(const void* x, const float* scale, const float* shift, const void* residual, void* y, int M, int C,
                    int act, lp_stream_t stream);

/* ---- M4: head pointwise pair ------------------------------------------------
 * out_nchw[N,Co,H,W] = a1[N,H,W,C1] * W1^T + a2[N,H,W,C2] * W2^T  (no bias, no act);
 * out is fp32 (out_fp32 != 0; what the reference hands to the glue after tofp32) or fp16;
 * a1/a2 are the ReLU'd depthwise-5x5 outputs (lp_dwconv_f16).  w1 [Co][C1], w2 [Co][C2] host fp16.
 * Single branch: C2 == 0 with a2 / w2 NULL, out = a1 * W1^T. */
size_t lp_head_packed_elems(int C1, int C2, int Co);
int lp_head_pack(const uint16_t* w1, const uint16_t* w2, int C1, int C2, int Co, uint16_t* w_packed);
int lp_head_pw_dual_f16(const void* a1, const void* a2, const void* w_packed, void* out_nchw,
                        int out_fp32, int N, int H, int W, int C1, int C2, int Co, lp_stream_t stream);

/* ---- M4 fused: both SepConv2d heads of one level in ONE kernel -------------------
 * out_nchw[N,Co,H,W] = W1 * relu(dw5x5(a1) + b1) + W2 * relu(dw5x5(a2) + b2)
 * (final_refined[i](refined) + final_raw[i](raw), lib/models/pose_mobilenet.py:151-154,
 * lib/models/layers/layers.py:120-133): depthwise 5x5 on the CUDA cores, result kept in shared
 * memory as the wgmma A operand, bias-free 1x1 on the tensor cores, NCHW fp32/fp16 store.
 * Pack (host memory): dw1/dw2 tap-major [25][C] BN-folded fp16 + fp32 biases, w1 [Co][C1], w2 [Co][C2].
 * Single branch (pose_simplenet's final_refined[i](refined) alone): C2 == 0 with dw2, bdw2, w2 and a2 NULL;
 * the slabs all come from a1 and the packed buffers carry none for the missing branch. */
size_t lp_head_fused_dw_elems(int C1, int C2);           /* fp16 elements of dw_cat; bias: /25 fp32 */
size_t lp_head_fused_pw_elems(int C1, int C2, int Co);   /* fp16 elements of pw_packed */
int lp_head_fused_pack(const uint16_t* dw1, const float* bdw1, const uint16_t* dw2, const float* bdw2,
                       const uint16_t* w1, const uint16_t* w2, int C1, int C2, int Co, uint16_t* dw_cat,
                       float* bdw_cat, uint16_t* pw_packed);
int lp_head_fused_f16(const void* a1, const void* a2, const void* dw_cat, const float* bdw_cat,
                      const void* pw_packed, void* out_nchw, int out_fp32, int N, int H, int W, int C1,
                      int C2, int Co, lp_stream_t stream);

/* Largest K (= MAX_NUM_PEOPLE) the evaluation parser takes: top-K slots per (image, joint) plane and the side of
 * the matcher's cost matrices.  K <= 64 runs on per-warp lists and one warp per image; 64 < K <= 256 on per-CTA
 * candidate buffers and one CTA per image with its cost matrices in the caller's workspace.  The uniform entry
 * points lp_nms_topk_f32 / lp_tag_match_f32 keep K <= 64; K up to LP_PARSER_MAX_PEOPLE goes through the ragged
 * entry points (a uniform batch is N equal lp_map_desc_t entries, with the same results per image). */
#define LP_PARSER_MAX_PEOPLE 256

/* ---- G1+G2: NMS (k x k window max, -inf padding) + top-K per (n,j) plane -----
 * det fp32 [N,J,H,W]; tag fp32 [N,J,H,W,T].  Order: value desc, flat index asc over
 * NMS survivors with value > 0; unused slots are (0.0f, index 0).  NaN never takes a slot, and
 * a NaN anywhere in a pixel's window suppresses it (the reference's max-pool propagates NaN).
 * nms_kernel odd, 1..9.  Width bound (one fp32 strip buffer of at most 200 KB in shared memory):
 * W <= 51200 / (nms_kernel + 1), e.g. 8533 at kernel 5; wider maps return LP_ERR_BAD_ARG.
 * Any height is accepted.
 * val_k [N,J,K] f32; ind_k [N,J,K] i32 (flat y*W+x); tag_k [N,J,K,T] f32.  K <= 64
 * (lp_nms_topk_ragged_f32: K <= LP_PARSER_MAX_PEOPLE).
 * min_value (double, compared as the reference does: float32 value widened to double): only survivors
 * with value > max(min_value, 0) are reported.  0 reproduces top_k as the
 * reference computes it; the full parse passes DETECTION_THRESHOLD, because match_by_tag drops every
 * candidate with val <= DETECTION_THRESHOLD before it looks at anything else (group.py:43-45), so the
 * keypoints are unchanged while background pixels never reach the NMS window test. */
size_t lp_nms_topk_workspace_bytes(int N, int J, int H, int W, int K);
int lp_nms_topk_f32(const float* det, const float* tag, int N, int J, int H, int W, int T,
                    int nms_kernel, int K, double min_value, float* val_k, int32_t* ind_k, float* tag_k,
                    void* workspace, size_t workspace_bytes, lp_stream_t stream);

/* ---- G3: tag matching (match_by_tag + Munkres), one image per CTA -----------
 * joint_order: int32 [J] device.  ans [N,pcap,J,3+T] f32 (x,y,val,tags), rows in
 * person-creation order; num_people [N] i32 (true count, may exceed pcap ->
 * LP_ERR_CAPACITY is NOT raised on the device; the caller compares against pcap;
 * pcap = J*K can never overflow).  Thresholds are doubles because the reference
 * compares float64 joint rows against Python floats (group.py:38-41,84).
 * K <= 64 (lp_tag_match_ragged_f32: K <= LP_PARSER_MAX_PEOPLE).  K <= 64: max_num_people <= 64, one warp
 * per image (one cost-matrix column per lane up to 32, two above).  K > 64 (ragged entry): max_num_people <= K, one 256-thread CTA per image; its two fp64
 * K x K matrices (costs, distances) live in the workspace, which lp_tag_match_workspace_bytes sizes from K. */
size_t lp_tag_match_workspace_bytes(int N, int J, int K, int T, int pcap);
int lp_tag_match_f32(const float* val_k, const int32_t* ind_k, const float* tag_k, int N, int J,
                     int K, int T, int W, const int32_t* joint_order, double det_threshold,
                     double tag_threshold, int use_detection_val, int ignore_too_much,
                     int max_num_people, int pcap, float* ans, int32_t* num_people,
                     void* workspace, size_t workspace_bytes, lp_stream_t stream);

/* ---- G4+G5+G6: adjust, scores, refine ---------------------------------------
 * In-place on ans [N,pcap,J,3+T]; scores [N,pcap] f32 = mean joint value after adjust
 * and before refine (group.py:275).  det/tag as for lp_nms_topk_f32 (un-NMS'd det). */
size_t lp_adjust_refine_workspace_bytes(int N, int J, int pcap);
int lp_adjust_refine_f32(const float* det, const float* tag, int N, int J, int H, int W, int T,
                         int pcap, float* ans, const int32_t* num_people, float* scores,
                         int do_adjust, int do_refine, void* workspace, size_t workspace_bytes,
                         lp_stream_t stream);

/* ---- pre-processing ("next" row 3, pre side) -------------------------------------
 * resize_align_multi_scale's image warp (lib/utils/transforms.py:183-192:
 * cv2.warpAffine(image, trans, size), INTER_LINEAR, BORDER_CONSTANT 0) restated exactly in
 * OpenCV's fixed-point arithmetic, optionally followed by torchvision ToTensor + Normalize
 * (valid.py:172-186,212) in IEEE float32.  img: N x [H][W][3] uint8 (device); minv [N,6]
 * float64 (device) = the INVERTED 2x3 matrices (dst -> src), inverted on
 * the host in OpenCV's operation order (litepose_b200.lib.utils.transforms.invert_affine);
 * mean/std: 3 floats each (HOST pointers, read at call time).
 * out_mode 0: uint8 [N][out_h][out_w][3]; 1: float32 [N,3,out_h,out_w]; 2: float16 NCHW. */
int lp_warp_affine_normalize_u8(const uint8_t* img, int N, int H, int W, const double* minv,
                                int out_w, int out_h, const float* mean, const float* std, void* out,
                                int out_mode, lp_stream_t stream);

/* Ragged form: N images of different sizes in ONE launch.  img is one byte buffer holding every
 * image's [src_h][src_w][3] pixels at its src_offset; desc [N] (device) gives per image the
 * source size, the inverted matrix (as minv above) and its output slot: dst_offset elements
 * (of the out_mode's element type) into out, an [out_h][out_w][3] (mode 0) or [3][out_h][out_w]
 * block.  max_out_w / max_out_h bound every out_w / out_h (they size the grid).  Per image the
 * result is bit-identical to lp_warp_affine_normalize_u8 on that image alone (same device code). */
typedef struct {
    int64_t src_offset;      /* bytes */
    int32_t src_h, src_w;
    double minv[6];
    int64_t dst_offset;      /* elements */
    int32_t out_h, out_w;
} lp_warp_desc_t;
int lp_warp_affine_normalize_ragged_u8(const uint8_t* img, int N, const lp_warp_desc_t* desc,
                                       int max_out_w, int max_out_h, const float* mean,
                                       const float* std, void* out, int out_mode, lp_stream_t stream);

/* ---- ragged parser: the G1-G6 chain on a det/tag arena of differently sized maps ----------
 * det holds image n's [J,h,w] block at desc[n].det_offset, tag its [J,h,w,T] block at
 * desc[n].tag_offset (elements).  hw_host [N][2] (HOST memory) lists the same (h, w) pairs as
 * desc (device); it sizes the grids and the workspaces.  Outputs keep the uniform layouts
 * (val_k [N,J,K], ans [N,pcap,J,3+T], ...) and per image equal, bit for bit, the uniform entry
 * points run on that image alone: they share the device code, a uniform call derives the
 * offsets from N, H, W, a ragged call reads them from desc.  Tag matching and adjust/refine
 * need the workspaces of lp_tag_match_workspace_bytes / lp_adjust_refine_workspace_bytes. */
typedef struct {
    int32_t h, w;
    int64_t det_offset;      /* elements */
    int64_t tag_offset;      /* elements */
} lp_map_desc_t;
size_t lp_nms_topk_ragged_workspace_bytes(int N, const int32_t* hw_host, int J, int K);
int lp_nms_topk_ragged_f32(const float* det, const float* tag, int N, const int32_t* hw_host,
                           const lp_map_desc_t* desc, int J, int T, int nms_kernel, int K,
                           double min_value, float* val_k, int32_t* ind_k, float* tag_k,
                           void* workspace, size_t workspace_bytes, lp_stream_t stream);
int lp_tag_match_ragged_f32(const float* val_k, const int32_t* ind_k, const float* tag_k, int N,
                            int J, int K, int T, const lp_map_desc_t* desc,
                            const int32_t* joint_order, double det_threshold,
                            double tag_threshold, int use_detection_val, int ignore_too_much,
                            int max_num_people, int pcap, float* ans, int32_t* num_people,
                            void* workspace, size_t workspace_bytes, lp_stream_t stream);
int lp_adjust_refine_ragged_f32(const float* det, const float* tag, int N, const int32_t* hw_host,
                                const lp_map_desc_t* desc, int J, int T, int pcap, float* ans,
                                const int32_t* num_people, float* scores, int do_adjust,
                                int do_refine, void* workspace, size_t workspace_bytes,
                                lp_stream_t stream);

/* ---- final predictions ("next" row 3, post-processing side) ----------------------
 * get_final_preds (lib/utils/transforms.py:195-202): in place, x and y of every keypoint of
 * the first min(num_people[n], pcap) persons of image n go through trans[n] (row-major 2x3
 * float64, get_affine_transform(center, scale, 0, heatmap_size, inv=1)) in float64 and are
 * stored back as float32.  ans [N,pcap,J,row] f32 (row >= 2: x, y, ...). */
int lp_transform_preds_f32(float* ans, const int32_t* num_people, const double* trans, int N,
                           int pcap, int J, int row, lp_stream_t stream);

/* ---- fast_utils plugin on the GPU ("next" row 2) -------------------------------
 * The reference's own native grouping for its "fast inference" demo parser
 * (nano_demo/fast_utils/group.py:38-47), batched over N images.
 *
 * lp_find_peaks_f32 replaces find_peaks_out_nchw (nano_demo/fast_utils/parse/find_peaks.cpp:80-97,
 * bound by plugins.cpp:9-29): per (image, joint) plane the first M pixels in scan order with
 * value >= threshold and no strictly larger value in the window_size x window_size
 * neighbourhood.  input, tmap [N,C,H,W] f32; count [N,C] i32, val/tag [N,C,M] f32,
 * ind [N,C,M,2] i32 = (x, y).  Entries past count are left untouched (the reference's
 * allocate-and-return variant zero-fills first, plugins.cpp:52-56).
 *
 * lp_assign_f32 replaces assign_out (assign.cpp:68-122, bound by plugins.cpp:66-82) for every
 * image: persons are built joint by joint in joint_order (i32 [C]) with the reference's
 * slack-array KM (assign.cpp:15-66), same float arithmetic and visiting order.
 * ans [N,M,C,4] f32 = (x, y, val, tag), untouched where nothing is assigned;
 * num_person [N] i32; status [N] i32: 0, or 1 when KM hit the round cap (the reference has no
 * cap and would not return).  M <= 32 (LP_ERR_CAPACITY above; the reference's arrays hold 10). */
int lp_find_peaks_f32(const float* input, const float* tmap, int N, int C, int H, int W, int M,
                      float threshold, int window_size, int32_t* count, float* val, float* tag,
                      int32_t* ind, lp_stream_t stream);
int lp_assign_f32(const int32_t* count, const float* val, const float* tag, const int32_t* ind,
                  const int32_t* joint_order, int N, int C, int M, float threshold,
                  int32_t* num_person, float* ans, int32_t* status, lp_stream_t stream);

/* lp_find_peaks_f32 on the maps as the glue writes them, uniform or ragged, in ONE launch
 * (the pipeline's fast grouping mode).  det [N,J,H,W] f32, or image n's [J,h,w] block at
 * desc[n].det_offset; the tag of a peak is read IN PLACE at channel 0 of the interleaved
 * [N,tag_planes,H,W,T] map (or image n's [tag_planes,h,w,T] block at desc[n].tag_offset).
 * tag_planes: J, or 1 = one map shared by every joint (MODEL.TAG_PER_JOINT off).
 * Uniform: hw_host = desc = NULL.  Ragged: hw_host [N][2] (HOST) = the (h, w) of desc (device),
 * H and W are ignored.  One CTA per (image, joint) plane, N*J planes.  Outputs as for
 * lp_find_peaks_f32 (count [N,J], val/tag_out [N,J,M], ind [N,J,M,2]; entries past count
 * untouched) and per image bit-identical to lp_find_peaks_f32 on det[n] and
 * tag[n,...,0].contiguous(): the same device code. */
int lp_find_peaks_maps_f32(const float* det, const float* tag, int N, int H, int W,
                           const int32_t* hw_host, const lp_map_desc_t* desc, int J, int T,
                           int tag_planes, int M, float threshold, int window_size,
                           int32_t* count, float* val, float* tag_out, int32_t* ind,
                           lp_stream_t stream);

/* ---- glue ("next" row 1): fused flip/upsample/average/project ----------------
 * From the two forward passes' outputs (plain: o0 [N,2J,h,w], o1 [N,J,2h,2w]; flipped
 * pass: f0, f1, NULL when flip == 0) produce det [N,J,Hd,Wd] and tag [N,J,Hd,Wd,T]
 * (T = 2 with flip else 1) exactly as get_multi_stage_outputs + aggregate_results do for
 * SCALE_FACTOR [1], WITH_HEATMAPS (1,1), WITH_AE (1,0).  (Hd,Wd) == (2h,2w): no
 * projection; otherwise PROJECT2IMAGE to size_projected = (Wd,Hd).  flip_index: int32 [J]. */
int lp_glue_f32(const float* o0, const float* o1, const float* f0, const float* f1,
                const int32_t* flip_index, int N, int J, int h, int w, int flip, int Hd, int Wd,
                float* det, float* tag, lp_stream_t stream);

/* General form of the glue (every cfg branch of lib/core/inference.py:75-208 for the LitePose head
 * layout) and one scale of the multi-scale test (reference valid.py:205-225 + aggregate_results,
 * inference.py:176-208).
 *   model_joints: DATASET.NUM_JOINTS = heat channels of o0 / o1 (it counts the centre joint when
 *     DATASET.WITH_CENTER is on, lib/config/default.py:175-177); J <= model_joints joints are
 *     written (J = model_joints - 1 with TEST.IGNORE_CENTER, inference.py:147-150); flip_index
 *     has model_joints entries.
 *   tag_shared: MODEL.TAG_PER_JOINT off - o0 = [model_joints heat | ONE tag map], the tag map is
 *     not permuted in the flip pass (inference.py:141-144) and tag is [N,1,Hd,Wd,T].
 *   Multi-scale: ONE call per scale, largest scale first, on that scale's network outputs (h, w
 *     follow the scale; Hd, Wd are the common size: base_size with PROJECT2IMAGE, else the size of
 *     the first scale's heat-maps).  The scale's flip-averaged heat-map, resampled to (Hd,Wd), is
 *     stored (accumulate == 0: first scale) or added to det (`final_heatmaps += ...`); divide_by
 *     != 1 divides the sum afterwards (`final_heatmaps / len(SCALE_FACTOR)`, valid.py:223: pass
 *     it with the last scale).  tag is written (resampled to (Hd,Wd)) only by the scale == 1
 *     call; pass NULL for the other scales (inference.py:179-190).
 * Single scale: accumulate 0, divide_by 1.  Projection ratios down to a 4.6x shrink. */
int lp_glue_scale_f32(const float* o0, const float* o1, const float* f0, const float* f1,
                      const int32_t* flip_index, int N, int J, int model_joints, int tag_shared,
                      int h, int w, int flip, int Hd, int Wd, int accumulate, float divide_by,
                      float* det, float* tag, lp_stream_t stream);

/* ---- per-step host payload ------------------------------------------------------
 * What HeatmapParser.parse hands back to valid.py:227 (lib/core/group.py:269-291), for a whole
 * batch, as one fixed-size row per image that a single D2H copy / NCCL gather carries:
 *   packed [N, keep*row + keep + 1] f32 = keep persons x row (= J*(3+T)) keypoint floats |
 *   keep scores | person count.  ans [N,pcap,J,3+T], scores [N,pcap], num_people [N] are the
 * parser's result buffers; keep <= pcap.  The count is the TRUE count (it may exceed keep: the
 * caller then fetches the image from the parser's buffers - nothing is clipped silently). */
int lp_pack_payload_f32(const float* ans, const int32_t* num_people, const float* scores, int N,
                        int pcap, int row, int keep, float* packed, lp_stream_t stream);
/* The fast grouping's row per image: packed [N, M*C*4 + 2] f32 = ans [N,M,C,4] of
 * lp_assign_f32 (every person: M <= 32) | person count | KM status (0 ok, 1 round cap hit). */
int lp_pack_fast_payload_f32(const float* ans, const int32_t* num_person, const int32_t* status,
                             int N, int M, int C, float* packed, lp_stream_t stream);

/* ---- synthetic workload: planted persons (bench / tests only) --------------------
 * A random-weight network detects nobody, so the benchmark plants persons between glue and
 * parser: det[det_index[i]] = max(det[..], det_value[i]) (atomic, order independent) and
 * tag[tag_index[i]] = tag_value[i] (indices unique).  Flat element indices, int64 device. */
int lp_plant_crowd_f32(float* det, const int64_t* det_index, const float* det_value,
                       int64_t n_det, float* tag, const int64_t* tag_index,
                       const float* tag_value, int64_t n_tag, lp_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* LITEPOSE_B200_H */
