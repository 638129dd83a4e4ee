// Pre-processing of the evaluation loop on the device (SURVEY.md 8(f) row 3, pre side): the reference's
// resize_align_multi_scale (lib/utils/transforms.py:183-192) = cv2.warpAffine(image, trans, size) with the defaults
// INTER_LINEAR / BORDER_CONSTANT(0), followed by torchvision ToTensor + Normalize (valid.py:172-186,212).
//
// cv2.warpAffine on 8-bit images is integer arithmetic end to end and is restated exactly (OpenCV imgwarp.cpp,
// WarpAffineInvoker + remapBilinear with the fixed-point table): the 2x3 matrix is inverted in double (host side, same
// operation order), source coordinates are AB_BITS=10 fixed point with INTER_BITS=5 sub-pixel positions,
// adelta[x] = round(M0*x*1024), X0 = round((M1*y+M2)*1024) + 16, X = (X0 + adelta[x]) >> 5, the four bilinear weights
// are (32-fy)(32-fx)*32 ... (exact products, they always sum to 1<<15, so OpenCV's table fix-up never fires) and the
// pixel is (sum + (1<<14)) >> 15; neighbours outside the image read the border value 0.
// ToTensor / Normalize are IEEE float32 divisions and a subtraction, reproduced with round-to-nearest intrinsics.
#include "common.cuh"

namespace lp {

// One output pixel (x, y) of one image: src = its [H][W][3] uint8 pixels, M = its inverted 2x3 matrix, out = the first
// element of its output block ([out_h][out_w][3] for MODE 0, [3][out_h][out_w] else).  MODE 0: uint8 HWC (the warped
// image itself), 1: float32 NCHW normalised, 2: float16 NCHW normalised.  Shared by the uniform and the ragged kernel.
template <int MODE>
__device__ __forceinline__ void warp_affine_pixel(const uint8_t* __restrict__ src, int H, int W, const double* M, int x,
                                                  int y, int out_w, int out_h, float m0, float m1, float m2, float s0,
                                                  float s1, float s2, void* __restrict__ out) {
    // saturate_cast<int>(double) == cvRound: round half to even
    const int adelta = __double2int_rn(__dmul_rn(__dmul_rn(M[0], (double)x), 1024.0));
    const int bdelta = __double2int_rn(__dmul_rn(__dmul_rn(M[3], (double)x), 1024.0));
    const int X0 = __double2int_rn(__dmul_rn(__dadd_rn(__dmul_rn(M[1], (double)y), M[2]), 1024.0)) + 16;
    const int Y0 = __double2int_rn(__dmul_rn(__dadd_rn(__dmul_rn(M[4], (double)y), M[5]), 1024.0)) + 16;
    const int X = (X0 + adelta) >> 5, Y = (Y0 + bdelta) >> 5;
    // OpenCV stores the integer part as short (saturated); image sizes here are far below 32768
    const int sx = max(min(X >> 5, 32767), -32768), sy = max(min(Y >> 5, 32767), -32768);
    const int fx = X & 31, fy = Y & 31;
    const int w00 = (32 - fy) * (32 - fx) * 32, w01 = (32 - fy) * fx * 32, w10 = fy * (32 - fx) * 32, w11 = fy * fx * 32;
    const bool x0ok = sx >= 0 && sx < W, x1ok = sx + 1 >= 0 && sx + 1 < W;
    const bool y0ok = sy >= 0 && sy < H, y1ok = sy + 1 >= 0 && sy + 1 < H;
    int v[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const int p00 = (x0ok && y0ok) ? src[((size_t)sy * W + sx) * 3 + c] : 0;
        const int p01 = (x1ok && y0ok) ? src[((size_t)sy * W + sx + 1) * 3 + c] : 0;
        const int p10 = (x0ok && y1ok) ? src[((size_t)(sy + 1) * W + sx) * 3 + c] : 0;
        const int p11 = (x1ok && y1ok) ? src[((size_t)(sy + 1) * W + sx + 1) * 3 + c] : 0;
        v[c] = (p00 * w00 + p01 * w01 + p10 * w10 + p11 * w11 + (1 << 14)) >> 15;     // <= 255 by construction
    }
    if (MODE == 0) {
        uint8_t* o = reinterpret_cast<uint8_t*>(out) + ((size_t)y * out_w + x) * 3;
        o[0] = (uint8_t)v[0];
        o[1] = (uint8_t)v[1];
        o[2] = (uint8_t)v[2];
    } else {
        const float mean[3] = {m0, m1, m2}, sd[3] = {s0, s1, s2};
        const size_t plane = (size_t)out_h * out_w;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const float t = __fdiv_rn((float)v[c], 255.f);                               // ToTensor
            const float r = __fdiv_rn(__fsub_rn(t, mean[c]), sd[c]);                     // Normalize
            const size_t o = (size_t)c * plane + (size_t)y * out_w + x;
            if (MODE == 1) reinterpret_cast<float*>(out)[o] = r;
            else reinterpret_cast<__half*>(out)[o] = __float2half_rn(r);
        }
    }
}

template <int MODE>
__global__ void __launch_bounds__(256)
warp_affine_kernel(const uint8_t* __restrict__ img, int H, int W, const double* __restrict__ minv, int out_w, int out_h,
                   float m0, float m1, float m2, float s0, float s1, float s2, void* __restrict__ out) {
    const int n = blockIdx.z;
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y;
    if (x >= out_w) return;
    const size_t esz = MODE == 0 ? 1 : (MODE == 1 ? 4 : 2);
    warp_affine_pixel<MODE>(img + (size_t)n * H * W * 3, H, W, minv + (size_t)n * 6, x, y, out_w, out_h, m0, m1, m2, s0,
                            s1, s2, reinterpret_cast<uint8_t*>(out) + (size_t)n * 3 * out_h * out_w * esz);
}

// Ragged batch: image n = blockIdx.z has its own source size, matrix and output slot (lp_warp_desc_t); the grid covers
// the largest output, blocks outside an image's output return at once.
template <int MODE>
__global__ void __launch_bounds__(256)
warp_affine_ragged_kernel(const uint8_t* __restrict__ img, const lp_warp_desc_t* __restrict__ desc, float m0, float m1,
                          float m2, float s0, float s1, float s2, void* __restrict__ out) {
    const lp_warp_desc_t& d = desc[blockIdx.z];
    const int out_w = d.out_w, out_h = d.out_h;
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y;
    if (x >= out_w || y >= out_h) return;
    const size_t esz = MODE == 0 ? 1 : (MODE == 1 ? 4 : 2);
    warp_affine_pixel<MODE>(img + d.src_offset, d.src_h, d.src_w, d.minv, x, y, out_w, out_h, m0, m1, m2, s0, s1, s2,
                            reinterpret_cast<uint8_t*>(out) + (size_t)d.dst_offset * esz);
}

}  // namespace lp

extern "C" int lp_warp_affine_normalize_u8(const uint8_t* img, int N, int H, int W, const double* minv, int out_w, int out_h,
                                           const float* mean, const float* std, void* out, int out_mode,
                                           lp_stream_t stream) {
    LP_CHECK_ARG(img && minv && out, "lp_warp_affine_normalize_u8: null pointer");
    LP_CHECK_ARG(N > 0 && N <= 65535 && H > 0 && W > 0 && H < 32768 && W < 32768 && out_w > 0 && out_h > 0 && out_h <= 65535,
                 "lp_warp_affine_normalize_u8: bad shape N=%d H=%d W=%d out=%dx%d", N, H, W, out_w, out_h);
    LP_CHECK_ARG(out_mode >= 0 && out_mode <= 2, "lp_warp_affine_normalize_u8: out_mode %d (0 u8 HWC, 1 f32 NCHW, 2 f16 NCHW)",
                 out_mode);
    LP_CHECK_ARG(out_mode == 0 || (mean && std), "lp_warp_affine_normalize_u8: mean/std required for normalised output");
    dim3 grid((out_w + 255) / 256, out_h, N);
    cudaStream_t s = (cudaStream_t)stream;
    const float m0 = mean ? mean[0] : 0.f, m1 = mean ? mean[1] : 0.f, m2 = mean ? mean[2] : 0.f;
    const float s0 = std ? std[0] : 1.f, s1 = std ? std[1] : 1.f, s2 = std ? std[2] : 1.f;
    if (out_mode == 0) lp::warp_affine_kernel<0><<<grid, 256, 0, s>>>(img, H, W, minv, out_w, out_h, m0, m1, m2, s0, s1, s2, out);
    else if (out_mode == 1) lp::warp_affine_kernel<1><<<grid, 256, 0, s>>>(img, H, W, minv, out_w, out_h, m0, m1, m2, s0, s1, s2, out);
    else lp::warp_affine_kernel<2><<<grid, 256, 0, s>>>(img, H, W, minv, out_w, out_h, m0, m1, m2, s0, s1, s2, out);
    LP_LAUNCH_CHECK("warp_affine_kernel");
    return LP_OK;
}

extern "C" int lp_warp_affine_normalize_ragged_u8(const uint8_t* img, int N, const lp_warp_desc_t* desc, int max_out_w,
                                                  int max_out_h, const float* mean, const float* std, void* out,
                                                  int out_mode, lp_stream_t stream) {
    LP_CHECK_ARG(img && desc && out, "lp_warp_affine_normalize_ragged_u8: null pointer");
    LP_CHECK_ARG(N > 0 && N <= 65535 && max_out_w > 0 && max_out_h > 0 && max_out_h <= 65535,
                 "lp_warp_affine_normalize_ragged_u8: bad shape N=%d max out=%dx%d", N, max_out_w, max_out_h);
    LP_CHECK_ARG(out_mode >= 0 && out_mode <= 2,
                 "lp_warp_affine_normalize_ragged_u8: out_mode %d (0 u8 HWC, 1 f32 NCHW, 2 f16 NCHW)", out_mode);
    LP_CHECK_ARG(out_mode == 0 || (mean && std), "lp_warp_affine_normalize_ragged_u8: mean/std required for normalised output");
    dim3 grid((max_out_w + 255) / 256, max_out_h, N);
    cudaStream_t s = (cudaStream_t)stream;
    const float m0 = mean ? mean[0] : 0.f, m1 = mean ? mean[1] : 0.f, m2 = mean ? mean[2] : 0.f;
    const float s0 = std ? std[0] : 1.f, s1 = std ? std[1] : 1.f, s2 = std ? std[2] : 1.f;
    if (out_mode == 0) lp::warp_affine_ragged_kernel<0><<<grid, 256, 0, s>>>(img, desc, m0, m1, m2, s0, s1, s2, out);
    else if (out_mode == 1) lp::warp_affine_ragged_kernel<1><<<grid, 256, 0, s>>>(img, desc, m0, m1, m2, s0, s1, s2, out);
    else lp::warp_affine_ragged_kernel<2><<<grid, 256, 0, s>>>(img, desc, m0, m1, m2, s0, s1, s2, out);
    LP_LAUNCH_CHECK("warp_affine_ragged_kernel");
    return LP_OK;
}
