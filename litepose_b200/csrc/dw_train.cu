// NCHW depthwise convolution for training: forward, input gradient (dgrad) and weight gradient (wgrad), fp32 or fp16,
// kernel k in {3, 5, 7}, stride s in {1, 2}, padding p = k / 2, no bias.  These are the depthwise convs of
// pose_mobilenet, pose_simplenet and pose_supermobilenet in the layout the module tree trains in (litepose_b200.train_dw).
//
// Arithmetic (tests/dw_train_emul.py restates it bit for bit).  Operands are converted exactly to fp32 and every sum
// is an fp32 fmaf chain that starts from +0; an fp16 result is that fp32 value rounded once to fp16, so an fp16 call
// returns the fp32 call's result on the up-converted inputs, rounded to fp16.
//   forward  y[n,c,oy,ox]: taps ky = 0 .. k-1 (outer), kx = 0 .. k-1 (inner), acc = fmaf(x[oy*s+ky-p, ox*s+kx-p],
//            w[c,ky,kx], acc); an input outside the plane is +0 (it still multiplies the weight: an inf or NaN weight
//            poisons the sum, as under F.conv2d's zero padding).
//   dgrad    dx[n,c,iy,ix]: taps ky = k-1 .. 0 (outer), kx = k-1 .. 0 (inner) whose (iy+p-ky) and (ix+p-kx) are
//            multiples of s (at s = 2 the other taps are skipped), acc = fmaf(dy[(iy+p-ky)/s, (ix+p-kx)/s], w[c,ky,kx],
//            acc), dy outside the output plane +0.  At s = 1 this is the forward kernel on dy with the flipped weights.
//   wgrad    dw[c,ky,kx] = sum over n, oy, ox of x[n,c,oy*s+ky-p, ox*s+kx-p] * dy[n,c,oy,ox], in two kernels:
//            dw_wgrad_partial: a range is the output pixels [oy0, oy0 + 128) x [ox0, ox0 + 32) of one image (ranges
//              numbered (n * ranges_y + ry) * ranges_x + rx; they depend on the shape only).  Thread (tx, ty) of its
//              256 (tx = lane, ty = warp) takes the pixels (oy0 + 32q + 4ty + r, ox0 + tx), q = 0..3 (outer), r = 0..3
//              (inner), those inside the plane only, and keeps one fmaf chain per tap from +0.  Each warp then folds
//              its lanes with the butterfly v += shfl_xor(v, 16, 8, 4, 2, 1) (lane 0's value is taken), and the eight
//              warp sums are added in warp order from warp 0's, all in fp32: part[range][c][tap].
//            dw_wgrad_merge: per (c, tap), the partials are added in fp64 in range order from range 0's and the sum
//              is rounded to fp32 (then to fp16 for an fp16 weight).
// Everything is a fixed function of the shape and the inputs: no atomics, no dependence on the SM count.
#include "common.cuh"
#include "../../include/litepose_b200_train.h"

namespace lp {

constexpr int DWT_THREADS = 256;
constexpr int DWT_TILE = 32;                 // output tile 32 x 32: 32 columns (lanes) x 8 warps x 4 rows
constexpr int DWT_ROWS = 4;                  // output rows per thread
constexpr int DWT_WG_PASSES = 4;             // wgrad range: 4 tiles down, 128 x 32 output pixels
constexpr int DWT_DG2_W = 64;                // stride-2 dgrad tile: 32 rows x 64 columns of dx

__device__ __forceinline__ float ld_f(const float* p) { return __ldg(p); }
__device__ __forceinline__ float ld_f(const __half* p) { return __half2float(__ldg(p)); }
__device__ __forceinline__ void st_f(float* p, float v) { *p = v; }
__device__ __forceinline__ void st_f(__half* p, float v) { *p = __float2half_rn(v); }

// rows x cols of plane src [H][W] from (y0, x0) into dst (leading dimension ld) as fp32, +0 outside the plane
template <typename T>
__device__ __forceinline__ void stage_plane(float* dst, int rows, int cols, int ld, const T* __restrict__ src, int H,
                                            int W, int y0, int x0) {
    for (int i = threadIdx.x; i < rows * cols; i += DWT_THREADS) {
        const int r = i / cols, cc = i - r * cols;
        const int gy = y0 + r, gx = x0 + cc;
        dst[r * ld + cc] = (gy >= 0 && gy < H && gx >= 0 && gx < W) ? ld_f(src + (size_t)gy * W + gx) : 0.f;
    }
}

// Forward (and, with flip = 1 at S = 1, dgrad: the weights read flipped).  CTA = one (n, c) plane's 32 x 32 output
// tile; thread (lane, warp) computes rows 4 * warp + r of column lane, reading each staged input row once for the
// four outputs whose windows hold it.
template <typename T, int K, int S>
__global__ void __launch_bounds__(DWT_THREADS)
dw_fwd_kernel(const T* __restrict__ x, const T* __restrict__ w, T* __restrict__ y, int C, int H, int W, int Ho, int Wo,
              int flip) {
    constexpr int P = K / 2, R = DWT_ROWS;
    constexpr int IW = (DWT_TILE - 1) * S + K, IH = (DWT_TILE - 1) * S + K;
    __shared__ float tile[IH * IW];
    const size_t plane = blockIdx.x;
    const int c = (int)(plane % (size_t)C);
    const int oy0 = blockIdx.y * DWT_TILE, ox0 = blockIdx.z * DWT_TILE;
    stage_plane(tile, IH, IW, IW, x + plane * H * W, H, W, oy0 * S - P, ox0 * S - P);
    float wr[K * K];
#pragma unroll
    for (int i = 0; i < K * K; ++i) wr[i] = ld_f(w + (size_t)c * K * K + (flip ? K * K - 1 - i : i));
    __syncthreads();
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    float acc[R];
#pragma unroll
    for (int r = 0; r < R; ++r) acc[r] = 0.f;
#pragma unroll
    for (int j = 0; j < (R - 1) * S + K; ++j) {
        const float* row = tile + (ty * R * S + j) * IW + tx * S;
        float v[K];
#pragma unroll
        for (int kx = 0; kx < K; ++kx) v[kx] = row[kx];
#pragma unroll
        for (int r = 0; r < R; ++r) {
            const int ky = j - r * S;
            if (ky >= 0 && ky < K) {
#pragma unroll
                for (int kx = 0; kx < K; ++kx) acc[r] = fmaf(v[kx], wr[ky * K + kx], acc[r]);
            }
        }
    }
    const int ox = ox0 + tx;
    if (ox >= Wo) return;
    T* yp = y + plane * Ho * Wo;
#pragma unroll
    for (int r = 0; r < R; ++r) {
        const int oy = oy0 + ty * R + r;
        if (oy < Ho) st_f(yp + (size_t)oy * Wo + ox, acc[r]);
    }
}

// Stride-2 dgrad, the gather form.  CTA = one plane's 32 x 64 dx tile; warp w takes the columns of parity PX = w & 1
// (so a warp never diverges on which kx taps apply), rows 8 * (w >> 1) + r; the row parity follows r.
template <typename T, int K, int PX>
__device__ __forceinline__ void dgrad_s2_body(const float* tile, const float (&wr)[K * K], T* dxp, int iy0, int ix0,
                                              int H, int W, int tx, int rg) {
    constexpr int P = K / 2, DW = DWT_DG2_W / 2 + P + 1, B = (P + 1) / 2;
    const int ix = ix0 + 2 * tx + PX;
#pragma unroll
    for (int r = 0; r < 8; ++r) {
        float acc = 0.f;
#pragma unroll
        for (int ky = K - 1; ky >= 0; --ky) {
            if (((r + P - ky) & 1) != 0) continue;
            const float* row = tile + (rg * 4 + (r + P - ky) / 2 + B) * DW + tx + B;
#pragma unroll
            for (int kx = K - 1; kx >= 0; --kx) {
                if (((PX + P - kx) & 1) != 0) continue;
                acc = fmaf(row[(PX + P - kx) / 2], wr[ky * K + kx], acc);
            }
        }
        const int iy = iy0 + rg * 8 + r;
        if (iy < H && ix < W) st_f(dxp + (size_t)iy * W + ix, acc);
    }
}

template <typename T, int K>
__global__ void __launch_bounds__(DWT_THREADS)
dw_dgrad_s2_kernel(const T* __restrict__ dy, const T* __restrict__ w, T* __restrict__ dx, int C, int H, int W, int Ho,
                   int Wo) {
    constexpr int P = K / 2, DH = DWT_TILE / 2 + P + 1, DW = DWT_DG2_W / 2 + P + 1, B = (P + 1) / 2;
    __shared__ float tile[DH * DW];
    const size_t plane = blockIdx.x;
    const int c = (int)(plane % (size_t)C);
    const int iy0 = blockIdx.y * DWT_TILE, ix0 = blockIdx.z * DWT_DG2_W;
    // dy rows / columns iy0 / 2 - B ...: every (iy + p - ky) / 2 of the tile's rows, and likewise for the columns
    stage_plane(tile, DH, DW, DW, dy + plane * Ho * Wo, Ho, Wo, iy0 / 2 - B, ix0 / 2 - B);
    float wr[K * K];
#pragma unroll
    for (int i = 0; i < K * K; ++i) wr[i] = ld_f(w + (size_t)c * K * K + i);
    __syncthreads();
    const int tx = threadIdx.x & 31, wq = threadIdx.x >> 5;
    T* dxp = dx + plane * H * W;
    if (wq & 1) dgrad_s2_body<T, K, 1>(tile, wr, dxp, iy0, ix0, H, W, tx, wq >> 1);
    else dgrad_s2_body<T, K, 0>(tile, wr, dxp, iy0, ix0, H, W, tx, wq >> 1);
}

// wgrad partials: CTA = (channel c, range); see the file comment for the order.
template <typename T, int K, int S>
__global__ void __launch_bounds__(DWT_THREADS)
dw_wgrad_partial(const T* __restrict__ x, const T* __restrict__ dy, float* __restrict__ part, int C, int H, int W,
                 int Ho, int Wo, int ranges_y, int ranges_x) {
    constexpr int P = K / 2, R = DWT_ROWS, KK = K * K;
    constexpr int IW = (DWT_TILE - 1) * S + K, IH = (DWT_TILE - 1) * S + K;
    __shared__ float xt[IH * IW];
    __shared__ float dt[DWT_TILE * DWT_TILE];
    __shared__ float red[DWT_THREADS / 32][KK];
    const size_t b = blockIdx.x;
    const int c = (int)(b % (size_t)C);
    const size_t rg = b / (size_t)C;
    const int rx = (int)(rg % (size_t)ranges_x);
    const int ry = (int)((rg / (size_t)ranges_x) % (size_t)ranges_y);
    const size_t n = rg / ((size_t)ranges_x * ranges_y);
    const size_t plane = n * C + c;
    const T* xp = x + plane * H * W;
    const T* dp = dy + plane * Ho * Wo;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    const int ox0 = rx * DWT_TILE;
    const bool col_ok = ox0 + tx < Wo;
    float acc[KK];
#pragma unroll
    for (int i = 0; i < KK; ++i) acc[i] = 0.f;
    for (int q = 0; q < DWT_WG_PASSES; ++q) {
        const int oy0 = (ry * DWT_WG_PASSES + q) * DWT_TILE;
        if (oy0 >= Ho) break;                      // uniform over the CTA
        if (q) __syncthreads();
        stage_plane(xt, IH, IW, IW, xp, H, W, oy0 * S - P, ox0 * S - P);
        stage_plane(dt, DWT_TILE, DWT_TILE, DWT_TILE, dp, Ho, Wo, oy0, ox0);
        __syncthreads();
        float d[R];
        bool ok[R];
#pragma unroll
        for (int r = 0; r < R; ++r) {
            d[r] = dt[(ty * R + r) * DWT_TILE + tx];
            ok[r] = col_ok && oy0 + ty * R + r < Ho;
        }
#pragma unroll
        for (int j = 0; j < (R - 1) * S + K; ++j) {
            const float* row = xt + (ty * R * S + j) * IW + tx * S;
            float v[K];
#pragma unroll
            for (int kx = 0; kx < K; ++kx) v[kx] = row[kx];
#pragma unroll
            for (int r = 0; r < R; ++r) {
                const int ky = j - r * S;
                if (ky >= 0 && ky < K && ok[r]) {
#pragma unroll
                    for (int kx = 0; kx < K; ++kx) acc[ky * K + kx] = fmaf(v[kx], d[r], acc[ky * K + kx]);
                }
            }
        }
    }
#pragma unroll
    for (int i = 0; i < KK; ++i) {
        float v = acc[i];
#pragma unroll
        for (int o = 16; o >= 1; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if (tx == 0) red[ty][i] = v;
    }
    __syncthreads();
    if (threadIdx.x < KK) {
        float s = red[0][threadIdx.x];
#pragma unroll
        for (int wq = 1; wq < DWT_THREADS / 32; ++wq) s += red[wq][threadIdx.x];
        part[(rg * C + c) * KK + threadIdx.x] = s;
    }
}

template <typename T>
__global__ void __launch_bounds__(128)
dw_wgrad_merge(const float* __restrict__ part, size_t nranges, int CKK, T* __restrict__ dw) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= CKK) return;
    double s = part[i];
    for (size_t r = 1; r < nranges; ++r) s = __dadd_rn(s, (double)part[r * CKK + i]);
    st_f(dw + i, __double2float_rn(s));
}

struct DwtShape {
    int Ho, Wo, ry, rx;
    size_t ranges;
};

static int dwt_check(const char* fn, int N, int C, int H, int W, int k, int stride, int dtype, DwtShape* sh) {
    LP_CHECK_ARG(k == 3 || k == 5 || k == 7, "%s: kernel size %d (3, 5 or 7)", fn, k);
    LP_CHECK_ARG(stride == 1 || stride == 2, "%s: stride %d (1 or 2)", fn, stride);
    LP_CHECK_ARG(dtype == LP_DT_F32 || dtype == LP_DT_F16, "%s: dtype %d (LP_DT_F32 or LP_DT_F16)", fn, dtype);
    LP_CHECK_ARG(N >= 0 && C >= 0 && H >= 1 && W >= 1, "%s: bad shape N=%d C=%d H=%d W=%d", fn, N, C, H, W);
    sh->Ho = (H - 1) / stride + 1;
    sh->Wo = (W - 1) / stride + 1;
    sh->ry = (sh->Ho + DWT_TILE * DWT_WG_PASSES - 1) / (DWT_TILE * DWT_WG_PASSES);
    sh->rx = (sh->Wo + DWT_TILE - 1) / DWT_TILE;
    sh->ranges = (size_t)N * sh->ry * sh->rx;
    LP_CHECK_ARG((size_t)N * C <= 0x7fffffffu && (H + DWT_TILE - 1) / DWT_TILE <= 65535 &&
                 (W + DWT_TILE - 1) / DWT_TILE <= 65535 && sh->ranges * C <= 0x7fffffffu,
                 "%s: shape N=%d C=%d H=%d W=%d exceeds the launch grid", fn, N, C, H, W);
    return LP_OK;
}

}  // namespace lp

using namespace lp;

#define LP_DWT_DISPATCH(k, stride, F)                               \
    switch (k * 10 + stride) {                                      \
        case 31: F(3, 1); break;                                    \
        case 32: F(3, 2); break;                                    \
        case 51: F(5, 1); break;                                    \
        case 52: F(5, 2); break;                                    \
        case 71: F(7, 1); break;                                    \
        default: F(7, 2); break;                                    \
    }

template <typename T>
static void dwt_fwd_launch(const void* x, const void* w, void* y, int N, int C, int H, int W, int Ho, int Wo, int k,
                           int stride, int flip, cudaStream_t st) {
    const dim3 grid((unsigned)((size_t)N * C), (Ho + DWT_TILE - 1) / DWT_TILE, (Wo + DWT_TILE - 1) / DWT_TILE);
    const T* xt = reinterpret_cast<const T*>(x);
    const T* wt = reinterpret_cast<const T*>(w);
    T* yt = reinterpret_cast<T*>(y);
#define LP_DWT_FWD(K_, S_) dw_fwd_kernel<T, K_, S_><<<grid, DWT_THREADS, 0, st>>>(xt, wt, yt, C, H, W, Ho, Wo, flip)
    LP_DWT_DISPATCH(k, stride, LP_DWT_FWD)
#undef LP_DWT_FWD
}

extern "C" int lp_dw_nchw_fwd(const void* x, const void* w, void* y, int N, int C, int H, int W, int k, int stride,
                              int dtype, lp_stream_t stream) {
    DwtShape sh;
    const int rc = dwt_check("lp_dw_nchw_fwd", N, C, H, W, k, stride, dtype, &sh);
    if (rc != LP_OK) return rc;
    if ((size_t)N * C == 0) return LP_OK;
    LP_CHECK_ARG(x && w && y, "lp_dw_nchw_fwd: null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    if (dtype == LP_DT_F32) dwt_fwd_launch<float>(x, w, y, N, C, H, W, sh.Ho, sh.Wo, k, stride, 0, st);
    else dwt_fwd_launch<__half>(x, w, y, N, C, H, W, sh.Ho, sh.Wo, k, stride, 0, st);
    LP_LAUNCH_CHECK("dw_fwd_kernel");
    return LP_OK;
}

template <typename T>
static void dwt_dgrad_s2_launch(const void* dy, const void* w, void* dx, int N, int C, int H, int W, int Ho, int Wo,
                                int k, cudaStream_t st) {
    const dim3 grid((unsigned)((size_t)N * C), (H + DWT_TILE - 1) / DWT_TILE, (W + DWT_DG2_W - 1) / DWT_DG2_W);
    const T* dt = reinterpret_cast<const T*>(dy);
    const T* wt = reinterpret_cast<const T*>(w);
    T* xt = reinterpret_cast<T*>(dx);
    if (k == 3) dw_dgrad_s2_kernel<T, 3><<<grid, DWT_THREADS, 0, st>>>(dt, wt, xt, C, H, W, Ho, Wo);
    else if (k == 5) dw_dgrad_s2_kernel<T, 5><<<grid, DWT_THREADS, 0, st>>>(dt, wt, xt, C, H, W, Ho, Wo);
    else dw_dgrad_s2_kernel<T, 7><<<grid, DWT_THREADS, 0, st>>>(dt, wt, xt, C, H, W, Ho, Wo);
}

extern "C" int lp_dw_nchw_dgrad(const void* dy, const void* w, void* dx, int N, int C, int H, int W, int k, int stride,
                                int dtype, lp_stream_t stream) {
    DwtShape sh;
    const int rc = dwt_check("lp_dw_nchw_dgrad", N, C, H, W, k, stride, dtype, &sh);
    if (rc != LP_OK) return rc;
    if ((size_t)N * C == 0) return LP_OK;
    LP_CHECK_ARG(dy && w && dx, "lp_dw_nchw_dgrad: null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    if (stride == 1) {
        // the forward kernel on dy (H x W at stride 1) with the weights flipped: the same taps in the same order
        if (dtype == LP_DT_F32) dwt_fwd_launch<float>(dy, w, dx, N, C, H, W, H, W, k, 1, 1, st);
        else dwt_fwd_launch<__half>(dy, w, dx, N, C, H, W, H, W, k, 1, 1, st);
        LP_LAUNCH_CHECK("dw_fwd_kernel (dgrad)");
        return LP_OK;
    }
    if (dtype == LP_DT_F32) dwt_dgrad_s2_launch<float>(dy, w, dx, N, C, H, W, sh.Ho, sh.Wo, k, st);
    else dwt_dgrad_s2_launch<__half>(dy, w, dx, N, C, H, W, sh.Ho, sh.Wo, k, st);
    LP_LAUNCH_CHECK("dw_dgrad_s2_kernel");
    return LP_OK;
}

extern "C" size_t lp_dw_nchw_wgrad_workspace_bytes(int N, int C, int H, int W, int k, int stride) {
    DwtShape sh;
    if (dwt_check("lp_dw_nchw_wgrad_workspace_bytes", N, C, H, W, k, stride, LP_DT_F32, &sh) != LP_OK) return 0;
    return sh.ranges * C * k * k * sizeof(float);
}

template <typename T>
static void dwt_wgrad_launch(const void* x, const void* dy, void* dw, float* part, int N, int C, int H, int W,
                             const DwtShape& sh, int k, int stride, cudaStream_t st) {
    const unsigned grid = (unsigned)(sh.ranges * C);
    const T* xt = reinterpret_cast<const T*>(x);
    const T* dt = reinterpret_cast<const T*>(dy);
#define LP_DWT_WG(K_, S_) \
    dw_wgrad_partial<T, K_, S_><<<grid, DWT_THREADS, 0, st>>>(xt, dt, part, C, H, W, sh.Ho, sh.Wo, sh.ry, sh.rx)
    LP_DWT_DISPATCH(k, stride, LP_DWT_WG)
#undef LP_DWT_WG
}

extern "C" int lp_dw_nchw_wgrad(const void* x, const void* dy, void* dw, int N, int C, int H, int W, int k, int stride,
                                int dtype, void* workspace, size_t workspace_bytes, lp_stream_t stream) {
    DwtShape sh;
    const int rc = dwt_check("lp_dw_nchw_wgrad", N, C, H, W, k, stride, dtype, &sh);
    if (rc != LP_OK) return rc;
    if ((size_t)C == 0) return LP_OK;
    LP_CHECK_ARG(dw, "lp_dw_nchw_wgrad: null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    const int CKK = C * k * k;
    if (N == 0) {   // no pixels: the gradient is +0
        LP_CUDA(cudaMemsetAsync(dw, 0, (size_t)CKK * (dtype == LP_DT_F32 ? 4 : 2), st));
        return LP_OK;
    }
    LP_CHECK_ARG(x && dy && workspace, "lp_dw_nchw_wgrad: null pointer");
    const size_t need = lp_dw_nchw_wgrad_workspace_bytes(N, C, H, W, k, stride);
    if (workspace_bytes < need) {
        set_error("lp_dw_nchw_wgrad: workspace of %zu bytes, %zu needed", workspace_bytes, need);
        return LP_ERR_CAPACITY;
    }
    if (reinterpret_cast<uintptr_t>(workspace) & 3) {
        set_error("lp_dw_nchw_wgrad: workspace must be 4-byte aligned");
        return LP_ERR_ALIGN;
    }
    float* part = reinterpret_cast<float*>(workspace);
    if (dtype == LP_DT_F32) dwt_wgrad_launch<float>(x, dy, dw, part, N, C, H, W, sh, k, stride, st);
    else dwt_wgrad_launch<__half>(x, dy, dw, part, N, C, H, W, sh, k, stride, st);
    LP_LAUNCH_CHECK("dw_wgrad_partial");
    const int blocks = (CKK + 127) / 128;
    if (dtype == LP_DT_F32) dw_wgrad_merge<float><<<blocks, 128, 0, st>>>(part, sh.ranges, CKK, (float*)dw);
    else dw_wgrad_merge<__half><<<blocks, 128, 0, st>>>(part, sh.ranges, CKK, (__half*)dw);
    LP_LAUNCH_CHECK("dw_wgrad_merge");
    return LP_OK;
}
