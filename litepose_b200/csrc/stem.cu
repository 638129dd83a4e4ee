// Stem: conv3x3 stride 2 (3 -> 32) + folded-BN bias + ReLU6 (or no activation: the raw convolution the BN
// recalibration pass takes its batch statistics of, lp_stem_conv3x3_s2_act); reads the reference's NCHW input
// (fp32, or fp16 under network_to_half) and writes the NHWC fp16 activation layout used by all
// later kernels.  Reference: convbnrelu(3, 32, ker=3, stride=2), lib/models/pose_mobilenet.py:37,
// lib/models/layers/layers.py:18-24.
//
// CTA = 64 x 8 output pixels; the 3-channel haloed input patch is staged in shared memory as
// fp32 (16-byte global vector loads, all of a thread's loads in flight at once).  Each thread computes two x-adjacent output pixels x 32 channels;
// weights are read as warp-uniform float4 broadcasts from shared memory (1 LDS.128 per 8 FFMA).
// Output: 64 B contiguous per pixel (4 x 16-byte stores).
#include "common.cuh"

namespace lp {

constexpr int ST_TW = 64, ST_TH = 8;                          // output tile; each thread owns 2 x-adjacent pixels
constexpr int ST_IW = ST_TW * 2 + 1, ST_IH = ST_TH * 2 + 1;   // 129 x 17 input patch (stride 2, pad 1)
constexpr int ST_PAD = 3;                                      // patch column c lives at s_in[..][ST_PAD + c]: the 128 columns
                                                               // right of the halo column start 16-byte aligned
constexpr int ST_IWP = 136;                                    // row pitch in floats (3 pad + 129, rounded; 136 % 32 = 8)

template <typename TIn> struct StemVec;
template <> struct StemVec<__half> { static constexpr int N = 8; };   // 16-byte global vectors
template <> struct StemVec<float> { static constexpr int N = 4; };

template <int ACT>
__device__ __forceinline__ float stem_act(float v) {
    return ACT == LP_ACT_RELU6 ? fminf(fmaxf(v, 0.f), 6.f) : v;
}

template <typename TIn, bool VEC, int ACT>
__global__ void __launch_bounds__(256)
stem_kernel(const TIn* __restrict__ x, const __half* __restrict__ w, const float* __restrict__ bias,
            __half* __restrict__ y, int H, int W, int flip_x) {
    __shared__ __align__(16) float s_in[3][ST_IH][ST_IWP];
    __shared__ __align__(16) float s_w[27][32];   // [tap][co]
    __shared__ __align__(16) float s_b[32];
    const int Ho = H / 2, Wo = W / 2;
    const int n = blockIdx.z;
    const int ox0 = blockIdx.x * ST_TW, oy0 = blockIdx.y * ST_TH;
    const int ix0 = ox0 * 2 - 1, iy0 = oy0 * 2 - 1;

    for (int i = threadIdx.x; i < 27 * 32; i += 256) {
        const int co = i & 31, t = i >> 5;
        s_w[t][co] = __half2float(w[co * 27 + t]);
    }
    if (threadIdx.x < 32) s_b[threadIdx.x] = bias ? bias[threadIdx.x] : 0.f;
    const TIn* xn = x + (size_t)n * 3 * H * W;
    if (VEC) {
        // Patch columns 1..128 (image columns 2*ox0 .. 2*ox0+127) are 16-byte aligned in global memory when W is a
        // multiple of the vector width: one 16-byte load per vector, all loads of a thread in flight together; the
        // halo column (image column 2*ox0-1) is a scalar load.  With flip_x the mirrored vector is loaded and reversed.
        constexpr int VN = StemVec<TIn>::N;
        constexpr int VPR = 128 / VN;                     // vectors per patch row
        constexpr int NV = 3 * ST_IH * VPR;               // vectors per patch
        constexpr int PER = (NV + 255) / 256;
        uint4 tmp[PER];
#pragma unroll
        for (int u = 0; u < PER; ++u) {
            const int i = threadIdx.x + u * 256;
            tmp[u] = make_uint4(0u, 0u, 0u, 0u);
            if (i < NV) {
                const int v = i % VPR, rr = i / VPR;
                const int r = rr % ST_IH, c = rr / ST_IH;
                const int gy = iy0 + r, gx = ix0 + 1 + v * VN;
                if (gy >= 0 && gy < H && gx < W) {
                    const int sx = flip_x ? W - VN - gx : gx;
                    tmp[u] = *reinterpret_cast<const uint4*>(xn + ((size_t)c * H + gy) * W + sx);
                }
            }
        }
        float halo = 0.f;
        int hrow = -1;
        if (threadIdx.x < 3 * ST_IH) {
            hrow = threadIdx.x;
            const int r = hrow % ST_IH, c = hrow / ST_IH;
            const int gy = iy0 + r;
            if (gy >= 0 && gy < H && ix0 >= 0) halo = (float)xn[((size_t)c * H + gy) * W + (flip_x ? W - 1 - ix0 : ix0)];
        }
#pragma unroll
        for (int u = 0; u < PER; ++u) {
            const int i = threadIdx.x + u * 256;
            if (i < NV) {
                const int v = i % VPR, rr = i / VPR;
                const int r = rr % ST_IH, c = rr / ST_IH;
                float f[VN];
                if (VN == 8) {
                    const __half2* h = reinterpret_cast<const __half2*>(&tmp[u]);
#pragma unroll
                    for (int k = 0; k < 4; ++k) {
                        const float2 t = __half22float2(h[k]);
                        f[2 * k] = t.x;
                        f[2 * k + 1] = t.y;
                    }
                } else {
                    const float* t = reinterpret_cast<const float*>(&tmp[u]);
#pragma unroll
                    for (int k = 0; k < VN; ++k) f[k] = t[k];
                }
                float4* dst = reinterpret_cast<float4*>(&s_in[c][r][ST_PAD + 1 + v * VN]);
#pragma unroll
                for (int k = 0; k < VN / 4; ++k) {
                    dst[k] = flip_x ? make_float4(f[VN - 1 - 4 * k], f[VN - 2 - 4 * k], f[VN - 3 - 4 * k], f[VN - 4 - 4 * k])
                                    : make_float4(f[4 * k], f[4 * k + 1], f[4 * k + 2], f[4 * k + 3]);
                }
            }
        }
        if (hrow >= 0) s_in[hrow / ST_IH][hrow % ST_IH][ST_PAD] = halo;
    } else {
        // generic path (W not a multiple of the vector width or unaligned base): scalar loads, 8 in flight per thread
        constexpr int NELEM = 3 * ST_IH * ST_IW;
        for (int i0 = threadIdx.x; i0 < NELEM; i0 += 256 * 8) {
            float tmp[8];
#pragma unroll
            for (int u = 0; u < 8; ++u) {
                const int i = i0 + u * 256;
                float v = 0.f;
                if (i < NELEM) {
                    const int c = i / (ST_IH * ST_IW);
                    const int rem = i - c * (ST_IH * ST_IW);
                    const int r = rem / ST_IW, col = rem - r * ST_IW;
                    const int gy = iy0 + r, gx = ix0 + col;
                    if (gy >= 0 && gy < H && gx >= 0 && gx < W)
                        v = (float)xn[((size_t)c * H + gy) * W + (flip_x ? W - 1 - gx : gx)];
                }
                tmp[u] = v;
            }
#pragma unroll
            for (int u = 0; u < 8; ++u) {
                const int i = i0 + u * 256;
                if (i < NELEM) {
                    const int c = i / (ST_IH * ST_IW);
                    const int rem = i - c * (ST_IH * ST_IW);
                    const int r = rem / ST_IW, col = rem - r * ST_IW;
                    s_in[c][r][ST_PAD + col] = tmp[u];
                }
            }
        }
    }
    __syncthreads();

    const int lx = threadIdx.x & 31, ly = threadIdx.x >> 5;    // pixels (2*lx, 2*lx+1) of row ly
    float acc0[32], acc1[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) acc0[i] = acc1[i] = s_b[i];
#pragma unroll
    for (int c = 0; c < 3; ++c)
#pragma unroll
        for (int ky = 0; ky < 3; ++ky) {
            // the two pixels need patch columns 4*lx .. 4*lx+4 (stored at ST_PAD + column: the float4 is aligned)
            const float* row = &s_in[c][2 * ly + ky][ST_PAD + 4 * lx];
            const float e = row[0];
            const float4 a = *reinterpret_cast<const float4*>(row + 1);
            const float in0[3] = {e, a.x, a.y};
            const float in1[3] = {a.y, a.z, a.w};
#pragma unroll
            for (int kx = 0; kx < 3; ++kx) {
                const float4* wr = reinterpret_cast<const float4*>(s_w[c * 9 + ky * 3 + kx]);
#pragma unroll
                for (int g = 0; g < 8; ++g) {
                    const float4 wv = wr[g];
                    acc0[4 * g + 0] = fmaf(in0[kx], wv.x, acc0[4 * g + 0]);
                    acc0[4 * g + 1] = fmaf(in0[kx], wv.y, acc0[4 * g + 1]);
                    acc0[4 * g + 2] = fmaf(in0[kx], wv.z, acc0[4 * g + 2]);
                    acc0[4 * g + 3] = fmaf(in0[kx], wv.w, acc0[4 * g + 3]);
                    acc1[4 * g + 0] = fmaf(in1[kx], wv.x, acc1[4 * g + 0]);
                    acc1[4 * g + 1] = fmaf(in1[kx], wv.y, acc1[4 * g + 1]);
                    acc1[4 * g + 2] = fmaf(in1[kx], wv.z, acc1[4 * g + 2]);
                    acc1[4 * g + 3] = fmaf(in1[kx], wv.w, acc1[4 * g + 3]);
                }
            }
        }
    const int oy = oy0 + ly;
    if (oy < Ho) {
#pragma unroll
        for (int p = 0; p < 2; ++p) {
            const int ox = ox0 + 2 * lx + p;
            if (ox >= Wo) continue;
            const float* acc = p ? acc1 : acc0;
            uint4* op = reinterpret_cast<uint4*>(y + (((size_t)n * Ho + oy) * Wo + ox) * 32);
#pragma unroll
            for (int g = 0; g < 4; ++g) {
                uint4 o;
                __half2* h = reinterpret_cast<__half2*>(&o);
#pragma unroll
                for (int i = 0; i < 4; ++i)
                    h[i] = __floats2half2_rn(stem_act<ACT>(acc[8 * g + 2 * i]), stem_act<ACT>(acc[8 * g + 2 * i + 1]));
                op[g] = o;
            }
        }
    }
}

}  // namespace lp

using namespace lp;

template <int ACT>
static void stem_launch(const void* x, int x_is_fp32, int flip_x, const __half* wh, const float* bias, __half* yh, int N,
                        int H, int W, cudaStream_t st) {
    dim3 grid((W / 2 + ST_TW - 1) / ST_TW, (H / 2 + ST_TH - 1) / ST_TH, N);
    const bool aligned = (reinterpret_cast<uintptr_t>(x) & 15) == 0;
    if (x_is_fp32) {
        const float* xf = reinterpret_cast<const float*>(x);
        if (aligned && W % 4 == 0) stem_kernel<float, true, ACT><<<grid, 256, 0, st>>>(xf, wh, bias, yh, H, W, flip_x);
        else stem_kernel<float, false, ACT><<<grid, 256, 0, st>>>(xf, wh, bias, yh, H, W, flip_x);
    } else {
        const __half* xh = reinterpret_cast<const __half*>(x);
        if (aligned && W % 8 == 0) stem_kernel<__half, true, ACT><<<grid, 256, 0, st>>>(xh, wh, bias, yh, H, W, flip_x);
        else stem_kernel<__half, false, ACT><<<grid, 256, 0, st>>>(xh, wh, bias, yh, H, W, flip_x);
    }
}

extern "C" int lp_stem_conv3x3_s2_act(const void* x, int x_is_fp32, int flip_x, const void* w, const float* bias,
                                      void* y, int N, int H, int W, int act, lp_stream_t stream) {
    LP_CHECK_ARG(x && w && y, "lp_stem_conv3x3_s2: null pointer");
    LP_CHECK_ARG(N > 0 && N <= 65535 && H > 0 && W > 0 && H % 2 == 0 && W % 2 == 0,
                 "lp_stem_conv3x3_s2: bad shape N=%d H=%d W=%d (H, W even)", N, H, W);
    LP_CHECK_ARG(act == LP_ACT_RELU6 || act == LP_ACT_NONE, "lp_stem_conv3x3_s2_act: act %d (ReLU6 or none)", act);
    if (reinterpret_cast<uintptr_t>(y) & 15) {
        set_error("lp_stem_conv3x3_s2: y must be 16-byte aligned");
        return LP_ERR_ALIGN;
    }
    const __half* wh = reinterpret_cast<const __half*>(w);
    __half* yh = reinterpret_cast<__half*>(y);
    cudaStream_t st = (cudaStream_t)stream;
    if (act == LP_ACT_RELU6) stem_launch<LP_ACT_RELU6>(x, x_is_fp32, flip_x, wh, bias, yh, N, H, W, st);
    else stem_launch<LP_ACT_NONE>(x, x_is_fp32, flip_x, wh, bias, yh, N, H, W, st);
    LP_LAUNCH_CHECK("stem_kernel");
    return LP_OK;
}

extern "C" int lp_stem_conv3x3_s2(const void* x, int x_is_fp32, int flip_x, const void* w, const float* bias, void* y,
                                  int N, int H, int W, lp_stream_t stream) {
    return lp_stem_conv3x3_s2_act(x, x_is_fp32, flip_x, w, bias, y, N, H, W, LP_ACT_RELU6, stream);
}
