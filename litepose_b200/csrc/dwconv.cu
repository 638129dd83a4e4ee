// Depthwise k x k convolution (+ folded-BN bias + activation), NHWC fp16, sm_90a.
// Reference op: nn.Conv2d(C, C, k, stride, k//2, groups=C) + BatchNorm2d + ReLU6/ReLU
//   (reference lib/models/layers/layers.py:100-104 depth_conv k=7; :123-127 SepConv2d k=5;
//    lib/models/pose_mobilenet.py:38 stem dw3x3).
//
// HBM-bound design: one CTA owns a (TH x TW) output tile of a 32-channel slab.  The haloed
// input tile is staged in shared memory by ONE TMA tensor copy (cp.async.bulk.tensor.4d) whose
// out-of-bounds zero fill implements the conv padding and every image/channel border, so the
// compute loop has no boundary branches.  Each thread owns one channel PAIR (half2) and walks
// 4x4 output micro-blocks with the k*k half2 weights held in registers, accumulating in fp32.
// Algorithmic bytes per launch: 2*(N*C*Hin*Win + N*C*Hout*Wout + C*k*k) (+4*C bias).
#include "common.cuh"

namespace lp {

constexpr int DW_CB = 32;        // channels per CTA slab
constexpr int DW_THREADS = 256;  // 16 channel pairs x 16 micro-block slots
constexpr int BY = 4, BX = 4;    // outputs per thread micro-block

template <int K, int S>
struct DwCfg {
    static constexpr int TH = (S == 1) ? 32 : 16;          // output tile
    static constexpr int TW = (S == 1) ? 32 : 16;
    static constexpr int IH = (TH - 1) * S + K;             // input tile incl. halo
    static constexpr int IW = (TW - 1) * S + K;
    static constexpr int IR = (BY - 1) * S + K;             // input rows / cols per micro-block
    static constexpr int IC = (BX - 1) * S + K;
    static constexpr int SMEM = IH * IW * DW_CB * 2 + 128 + 64;
};

// fp16 x fp16 + fp32 -> fp32 with one rounding: the fp16 -> fp32 conversions are exact, so the fp32 FMA of the
// converted operands gives the same result as a mixed-precision FMA.
__device__ __forceinline__ float fhfma(unsigned short a, unsigned short b, float c) {
    return __fmaf_rn(__half2float(__ushort_as_half(a)), __half2float(__ushort_as_half(b)), c);
}
__device__ __forceinline__ float fhadd(unsigned short a, float c) { return __fadd_rn(__half2float(__ushort_as_half(a)), c); }
__device__ __forceinline__ unsigned short lo16(__half2 v) { return __half_as_ushort(__low2half(v)); }
__device__ __forceinline__ unsigned short hi16(__half2 v) { return __half_as_ushort(__high2half(v)); }

// PREC 0: every product accumulated in fp32 (fhfma).  PREC 1: the K taps of one kernel row are accumulated with
// packed HFMA2 in fp16 (2 channels per instruction), each row sum is then added into the fp32 accumulator (fhadd).
template <int K, int S, int PREC>
__global__ void __launch_bounds__(DW_THREADS, 2)
dwconv_kernel(const __grid_constant__ CUtensorMap map_x, const __half* __restrict__ w, const float* __restrict__ bias,
              __half* __restrict__ y, int C, int Hout, int Wout, int tiles_x, int act) {
    using Cfg = DwCfg<K, S>;
    extern __shared__ __align__(1024) uint8_t smem[];
    uint64_t* bar = reinterpret_cast<uint64_t*>(smem + Cfg::IH * Cfg::IW * DW_CB * 2);

    const int tile = blockIdx.x;
    const int tx = tile % tiles_x, ty = tile / tiles_x;
    const int c0 = blockIdx.y * DW_CB;
    const int n = blockIdx.z;
    const int ox0 = tx * Cfg::TW, oy0 = ty * Cfg::TH;

    pdl_launch_dependents();
    if (threadIdx.x == 0) {
        mbar_init(bar, 1);
        fence_barrier_init();
        pdl_wait();           // input activations complete (weights below are static and may be read earlier)
        mbar_expect_tx(bar, Cfg::IH * Cfg::IW * DW_CB * 2);
        tma_load_4d(smem, &map_x, bar, c0, ox0 * S - K / 2, oy0 * S - K / 2, n);
    }

    const int cp = threadIdx.x & 15;           // channel pair inside the slab
    const int sub = (threadIdx.x >> 4) & 1;    // half-warp: second half works on the x-adjacent micro-block ...
    const int wid = threadIdx.x >> 5;
    // ... in MIRRORED column order (stride 1), so the two half-warps always touch pixels of opposite parity
    // (64 B per pixel = 16 banks): conflict-free LDS.  Mirrored data needs mirrored weights and mirrored stores.
    const bool mir = (S == 1) && sub;
    const int ch = c0 + 2 * cp;
    const bool ch_ok = ch < C;

    __half2 wreg[K * K];   // tap-major weights [k*k][C] -> this thread's channel pair
#pragma unroll
    for (int ky = 0; ky < K; ++ky)
#pragma unroll
        for (int kx = 0; kx < K; ++kx) {
            const int t = ky * K + (mir ? K - 1 - kx : kx);
            wreg[ky * K + kx] = ch_ok ? *reinterpret_cast<const __half2*>(w + (size_t)t * C + ch) : __floats2half2_rn(0.f, 0.f);
        }
    float2 b2 = make_float2(0.f, 0.f);
    if (ch_ok && bias) b2 = make_float2(bias[ch], bias[ch + 1]);

    __syncthreads();          // barrier init visible to all waiters
    pdl_wait();               // also orders this kernel's output writes after the previous kernel's reads
    mbar_wait(bar, 0);

    const __half2* tile_in = reinterpret_cast<const __half2*>(smem);   // [IH][IW][16 pairs]
    constexpr int PAIRS_X = Cfg::TW / (2 * BX);
    constexpr int NPAIRS = (Cfg::TH / BY) * PAIRS_X;
    const int cstep = mir ? -(DW_CB / 2) : (DW_CB / 2);

#pragma unroll 1
    for (int q = wid; q < NPAIRS; q += DW_THREADS / 32) {
        const int by = q / PAIRS_X, bx = (q % PAIRS_X) * 2 + sub;
        const int oy = by * BY, ox = bx * BX;           // tile-local output origin
        if (oy0 + oy >= Hout || ox0 + ox >= Wout) continue;   // micro-block fully outside
        float2 acc[BY][BX];
        __half2 acch[BY][BX], part[BY][BX];      // PREC 2: running fp16 total + current two-row chain
        const __half2 bh = __float22half2_rn(b2);
#pragma unroll
        for (int i = 0; i < BY; ++i)
#pragma unroll
            for (int j = 0; j < BX; ++j) {
                acc[i][j] = b2;
                acch[i][j] = bh;
            }

        // slot c of a row holds input column (ox*S + c), or (ox*S + IC-1-c) when mirrored
        const __half2* base = tile_in + ((oy * S) * Cfg::IW + ox * S + (mir ? Cfg::IC - 1 : 0)) * (DW_CB / 2) + cp;
#pragma unroll
        for (int r = 0; r < Cfg::IR; ++r) {
            __half2 in[Cfg::IC];
#pragma unroll
            for (int c = 0; c < Cfg::IC; ++c) in[c] = base[r * Cfg::IW * (DW_CB / 2) + c * cstep];
#pragma unroll
            for (int i = 0; i < BY; ++i) {
                const int ky = r - i * S;
                if (ky >= 0 && ky < K) {
                    if (PREC == 0) {
#pragma unroll
                        for (int kx = 0; kx < K; ++kx) {
                            const __half2 wv = wreg[ky * K + kx];
#pragma unroll
                            for (int j = 0; j < BX; ++j) {
                                acc[i][j].x = fhfma(lo16(in[j * S + kx]), lo16(wv), acc[i][j].x);
                                acc[i][j].y = fhfma(hi16(in[j * S + kx]), hi16(wv), acc[i][j].y);
                            }
                        }
                    } else if (PREC == 2) {
                        // fully packed: chains of two kernel rows folded into a running fp16 total (dw_inner.cuh)
#pragma unroll
                        for (int kx = 0; kx < K; ++kx) {
                            const __half2 wv = wreg[ky * K + kx];
#pragma unroll
                            for (int j = 0; j < BX; ++j) {
                                if ((ky & 1) == 0 && kx == 0) part[i][j] = __hmul2(in[j * S + kx], wv);
                                else part[i][j] = __hfma2(in[j * S + kx], wv, part[i][j]);
                            }
                        }
                        if ((ky & 1) || ky == K - 1) {
#pragma unroll
                            for (int j = 0; j < BX; ++j) acch[i][j] = __hadd2(acch[i][j], part[i][j]);
                        }
                    } else {
#pragma unroll
                        for (int j = 0; j < BX; ++j) {
                            __half2 sacc = __hmul2(in[j * S], wreg[ky * K]);
#pragma unroll
                            for (int kx = 1; kx < K; ++kx) sacc = __hfma2(in[j * S + kx], wreg[ky * K + kx], sacc);
                            acc[i][j].x = fhadd(lo16(sacc), acc[i][j].x);
                            acc[i][j].y = fhadd(hi16(sacc), acc[i][j].y);
                        }
                    }
                }
            }
        }
        if (ch_ok) {
            const int gy0 = oy0 + oy, gx0 = ox0 + ox;
            // one 64-bit base per micro-block; every pixel is base + (i*Wout + jj)*C elements
            __half* ybase = y + (((size_t)n * Hout + gy0) * Wout + gx0) * C + ch;
            const bool full = (gy0 + BY <= Hout) && (gx0 + BX <= Wout);
#pragma unroll
            for (int i = 0; i < BY; ++i) {
#pragma unroll
                for (int j = 0; j < BX; ++j) {
                    const int jj = mir ? BX - 1 - j : j;
                    if (full || (gy0 + i < Hout && gx0 + jj < Wout)) {
                        __half2 o;
                        if (PREC == 2) {
                            o = acch[i][j];
                            if (act != LP_ACT_NONE) o = __hmax2(o, __floats2half2_rn(0.f, 0.f));
                            if (act == LP_ACT_RELU6) o = __hmin2(o, __floats2half2_rn(6.f, 6.f));
                        } else {
                            o = __floats2half2_rn(act_apply(acc[i][j].x, act), act_apply(acc[i][j].y, act));
                        }
                        *reinterpret_cast<__half2*>(ybase + ((size_t)i * Wout + jj) * C) = o;
                    }
                }
            }
        }
    }
}

// Depthwise arithmetic of this (unfused) kernel: 0 = fp32 accumulation, 1 = packed fp16 row sums added in fp32,
// 2 = fully packed fp16 (grouped chains, like the fused block kernels).  Default: 2 for the backbone / stem kernels
// k = 7 and k = 3, 0 for k = 5 (the SepConv heads feed the network outputs directly).
static int g_dw_prec = -2;   // -2: per-kernel-size default
static int dw_prec(int k) {
    if (g_dw_prec == -2) return k == 5 ? 0 : 2;
    return g_dw_prec;
}

template <int K, int S, int PREC>
static int launch_dw(const void* x, const void* w, const float* bias, void* y, int N, int C, int H, int W, int act,
                     cudaStream_t stream) {
    using Cfg = DwCfg<K, S>;
    const int Hout = H / S, Wout = W / S;
    CUtensorMap map;
    uint64_t dims[4] = {(uint64_t)C, (uint64_t)W, (uint64_t)H, (uint64_t)N};
    uint64_t strides[3] = {(uint64_t)C * 2, (uint64_t)W * C * 2, (uint64_t)H * W * C * 2};
    uint32_t box[4] = {(uint32_t)DW_CB, (uint32_t)Cfg::IW, (uint32_t)Cfg::IH, 1u};
    int rc = make_tmap(&map, x, 4, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_NONE);
    if (rc) return rc;
    cudaError_t e = cudaFuncSetAttribute((const void*)dwconv_kernel<K, S, PREC>,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM);
    if (e != cudaSuccess) return cuda_fail(e, "cudaFuncSetAttribute(dwconv)");
    const int tiles_x = (Wout + Cfg::TW - 1) / Cfg::TW, tiles_y = (Hout + Cfg::TH - 1) / Cfg::TH;
    dim3 grid(tiles_x * tiles_y, (C + DW_CB - 1) / DW_CB, N);
    cudaError_t le = launch_pdl(dwconv_kernel<K, S, PREC>, grid, dim3(DW_THREADS), (size_t)Cfg::SMEM, stream, map,
                                reinterpret_cast<const __half*>(w), bias, reinterpret_cast<__half*>(y), C, Hout, Wout,
                                tiles_x, act);
    if (le != cudaSuccess) return cuda_fail(le, "launch dwconv_kernel");
    LP_LAUNCH_CHECK("dwconv_kernel");
    return LP_OK;
}

}  // namespace lp

using namespace lp;

extern "C" void lp_set_dw_precision(int prec) { lp::g_dw_prec = (prec >= 0 && prec <= 2) ? prec : -2; }
extern "C" int lp_get_dw_precision(void) { return lp::dw_prec(7); }

extern "C" int lp_dwconv_f16(const void* x, const void* w, const float* bias, void* y, int N, int C, int H, int W, int k,
                             int stride, int act, lp_stream_t stream) {
    LP_CHECK_ARG(x && w && y, "lp_dwconv_f16: null pointer");
    LP_CHECK_ARG(N > 0 && N <= 65535 && C > 0 && C % 8 == 0 && H > 0 && W > 0,
                 "lp_dwconv_f16: bad shape N=%d C=%d H=%d W=%d", N, C, H, W);
    LP_CHECK_ARG((k == 3 || k == 5 || k == 7) && (stride == 1 || stride == 2), "lp_dwconv_f16: k=%d stride=%d unsupported",
                 k, stride);
    LP_CHECK_ARG(stride == 1 || (H % 2 == 0 && W % 2 == 0), "lp_dwconv_f16: stride 2 needs even H, W (%d, %d)", H, W);
    LP_CHECK_ARG(act >= LP_ACT_NONE && act <= LP_ACT_RELU6, "lp_dwconv_f16: bad act %d", act);
    if ((reinterpret_cast<uintptr_t>(x) & 15) || (reinterpret_cast<uintptr_t>(y) & 3) || (reinterpret_cast<uintptr_t>(w) & 3)) {
        set_error("lp_dwconv_f16: x must be 16-byte aligned, w/y 4-byte aligned");
        return LP_ERR_ALIGN;
    }
    cudaStream_t s = (cudaStream_t)stream;
    const int prec = dw_prec(k);
#define LP_DW(KK, SS)                                                                      \
    if (k == KK && stride == SS)                                                           \
        return prec == 2 ? launch_dw<KK, SS, 2>(x, w, bias, y, N, C, H, W, act, s)         \
             : prec == 1 ? launch_dw<KK, SS, 1>(x, w, bias, y, N, C, H, W, act, s)         \
                         : launch_dw<KK, SS, 0>(x, w, bias, y, N, C, H, W, act, s);
    LP_DW(7, 1) LP_DW(7, 2) LP_DW(5, 1) LP_DW(5, 2) LP_DW(3, 1) LP_DW(3, 2)
#undef LP_DW
    return LP_ERR_BAD_ARG;
}
