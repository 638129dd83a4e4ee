// The whole stem in ONE kernel (reference lib/models/pose_mobilenet.py:36-41, lib/models/layers/layers.py:18-24):
//   convbnrelu(3, 32, ker=3, stride=2) -> convbnrelu(32, 32, ker=3, stride=1, groups=32) -> Conv2d(32, C0, 1) + BN
// reading the reference's NCHW image (fp32, or fp16 under network_to_half; optionally mirrored = the flip pass) and
// writing the NHWC fp16 tensor x0 [N, H/2, W/2, C0] the backbone starts from.  Unfused, the two 32-channel
// half-resolution intermediates (134 MB each at batch 32 / 512^2) are written and read back; here they stay on chip:
// HBM traffic = the image once + x0 once.
//
// Per 16 x 8 output tile (persistent 128-thread CTAs, 3 per SM so that one CTA's barriers and MMA round trips hide
// behind the others; the next tile's image patch is prefetched into registers):
//   P0  haloed 3 x 21 x 40 image patch -> shared memory (fp16), 8/16-byte vector loads, zero outside the image
//   P1  im2col of the 18 x 10 conv1 outputs the depthwise needs (27 taps, K padded to 32) -> 128B-swizzled K-major A1
//   P2  wgmma        D1[192 px x 32] = A1 x W1^T            (the CTA is one warpgroup; fp32 accumulators in registers)
//   P3  + bias -> ReLU6 -> fp16, ZERO outside the image (the depthwise pads conv1's OUTPUT with zeros)
//       -> chunk-major tile [4 x 8ch][180 px][16 B] (conflict-free stores and loads, see dwblock.cu)
//   P4  depthwise 3x3 on the CUDA cores (register-blocked HFMA2 loop of dw_inner.cuh), + bias, ReLU6
//       -> 128B-swizzled K-major A2 [128 px x 32]
//   P5  wgmma        D2[128 px x C0] = A2 x W3^T
//   P6  + bias (no activation) -> fp16 -> NHWC rows
#include "common.cuh"
#include "dw_inner.cuh"

namespace lp {

// Geometry: 16 x 8 output tile = 8 micro-blocks of 4 x 4 pixels x 16 channel pairs = 128 threads for the depthwise (the
// register-blocked loop of dw_inner.cuh: 36 LDS.32 per 16 outputs instead of 36 LDS.128 per output); the 18 x 10 conv1
// outputs it needs are the first three 64-row blocks of the im2col A tile.  Small CTAs (128 threads = one warpgroup,
// ~58 KB) so that three are resident per SM and one CTA's barriers / wgmma waits hide behind the others; the next
// tile's image patch is prefetched into registers.
constexpr int SF_TW = 16, SF_TH = 8;                 // output tile (pixels of the H/2 x W/2 grid)
constexpr int SF_CW = SF_TW + 2, SF_CH = SF_TH + 2;  // conv1 outputs needed: 18 x 10
constexpr int SF_CPIX = SF_CW * SF_CH;               // 180
constexpr int SF_PH = 2 * SF_CH + 1;                 // image patch rows: 21
constexpr int SF_PW = 40;                            // image patch columns (37 used, first = 2*ox0 - 4)
constexpr int SF_PV = SF_PW / 4;                     // 4-pixel vectors per patch row
constexpr int SF_NV = 3 * SF_PH * SF_PV;             // 630 vectors per patch
constexpr int SF_THREADS = 128;
constexpr int SF_PER = (SF_NV + SF_THREADS - 1) / SF_THREADS;   // 5 vectors per thread
constexpr int SF_A = 2 * 128 * 128;                  // A1 (im2col, two M-tiles); its first half holds A2 once conv1 has retired
constexpr int SF_B = 32 * 128;                       // weight tiles: up to 32 rows x 128 B
constexpr int SF_TCHUNK = 2976;                      // chunk pitch of the conv1 tile: 180 * 16 + 96 (pitch = 32 mod 128)
constexpr int SF_T = 4 * SF_TCHUNK;

struct SfParams {
    int N, H, W, Ho, Wo, C0, n_tile;
    int tiles_x, tiles_y, num_tiles;
    int flip_x, x_is_fp32;    // flip_x: 0 plain, 1 mirrored
    const void* x;
    const float* b1;        // [32]
    const __half* w_dw;     // [9][32] tap-major
    const float* b_dw;      // [32]
    const float* b_pw;      // packed, n_tile
    __half* out;            // [N, Ho, Wo, C0]
};

struct SfSmem {
    alignas(1024) uint8_t a[SF_A];
    alignas(1024) uint8_t b1[SF_B];
    alignas(1024) uint8_t b2[SF_B];
    alignas(16) uint8_t t[SF_T];
    alignas(16) __half patch[3][SF_PH][SF_PW];
    alignas(16) __half wdw[9][32];
    float bias1[32], biasdw[32], biaspw[32];
    uint64_t w_full;
};

// one 4-pixel vector of the image patch of tile t, RAW (zero outside the image): the load must not be consumed before
// the patch is written to shared memory one tile later, or the prefetch stalls on the spot (the first version applied
// the mirror permutation here and spent 26 % of its stall samples on it)
template <bool FP32>
__device__ __forceinline__ uint4 sf_load_vec(const SfParams& p, int t, int i) {
    const int tx = t % p.tiles_x, ty = (t / p.tiles_x) % p.tiles_y, n = t / (p.tiles_x * p.tiles_y);
    const int v = i % SF_PV, rr = i / SF_PV;
    const int r = rr % SF_PH, c = rr / SF_PH;
    const int gy = 2 * ty * SF_TH - 3 + r, gx = 2 * tx * SF_TW - 4 + 4 * v;
    uint4 o = make_uint4(0u, 0u, 0u, 0u);
    if (gy >= 0 && gy < p.H && gx >= 0 && gx < p.W) {       // gx % 4 == 0 and W % 4 == 0: all four or none inside
        const int sx = p.flip_x ? p.W - 4 - gx : gx;
        const size_t off = (((size_t)n * 3 + c) * p.H + gy) * p.W + sx;
        if (FP32) {
            o = __ldg(reinterpret_cast<const uint4*>(reinterpret_cast<const float*>(p.x) + off));
        } else {
            const uint2 q = __ldg(reinterpret_cast<const uint2*>(reinterpret_cast<const __half*>(p.x) + off));
            o.x = q.x;
            o.y = q.y;
        }
    }
    return o;
}
// raw vector -> four fp16 pixels in patch order (mirrored for the flip pass)
template <bool FP32>
__device__ __forceinline__ uint2 sf_pack_vec(uint4 raw, int flip_x) {
    __half2 lo, hi;
    if (FP32) {
        const float f0 = __uint_as_float(raw.x), f1 = __uint_as_float(raw.y), f2 = __uint_as_float(raw.z),
                    f3 = __uint_as_float(raw.w);
        if (flip_x) { lo = __floats2half2_rn(f3, f2); hi = __floats2half2_rn(f1, f0); }
        else { lo = __floats2half2_rn(f0, f1); hi = __floats2half2_rn(f2, f3); }
    } else {
        const __half2 a = *reinterpret_cast<const __half2*>(&raw.x), b = *reinterpret_cast<const __half2*>(&raw.y);
        if (flip_x) { lo = __lowhigh2highlow(b); hi = __lowhigh2highlow(a); }
        else { lo = a; hi = b; }
    }
    uint2 o;
    o.x = *reinterpret_cast<const uint32_t*>(&lo);
    o.y = *reinterpret_cast<const uint32_t*>(&hi);
    return o;
}

template <bool FP32>
__global__ void __launch_bounds__(SF_THREADS, 3)
stem_fused_kernel(const __grid_constant__ CUtensorMap map_w1, const __grid_constant__ CUtensorMap map_w3,
                  const __grid_constant__ SfParams p) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    SfSmem& sm = *reinterpret_cast<SfSmem*>(smem_raw);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&map_w1);
        tma_prefetch_desc(&map_w3);
        mbar_init(&sm.w_full, 1);
        fence_barrier_init();
    }
    for (int i = threadIdx.x; i < 9 * 32; i += SF_THREADS) sm.wdw[i / 32][i % 32] = p.w_dw[i];
    if (threadIdx.x < 32) {
        sm.bias1[threadIdx.x] = p.b1 ? p.b1[threadIdx.x] : 0.f;
        sm.biasdw[threadIdx.x] = p.b_dw ? p.b_dw[threadIdx.x] : 0.f;
        sm.biaspw[threadIdx.x] = (p.b_pw && threadIdx.x < p.n_tile) ? p.b_pw[threadIdx.x] : 0.f;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        mbar_expect_tx(&sm.w_full, (uint32_t)(SF_B + p.n_tile * 128));
        tma_load_2d(sm.b1, &map_w1, &sm.w_full, 0, 0);
        tma_load_2d(sm.b2, &map_w3, &sm.w_full, 0, 0);
    }
    const __half2 zero2 = __floats2half2_rn(0.f, 0.f);

    // image patch of the first tile -> registers
    uint4 pre[SF_PER];
#pragma unroll
    for (int u = 0; u < SF_PER; ++u) {
        const int i = threadIdx.x + u * SF_THREADS;
        pre[u] = make_uint4(0u, 0u, 0u, 0u);
        if (i < SF_NV && (int)blockIdx.x < p.num_tiles) pre[u] = sf_load_vec<FP32>(p, blockIdx.x, i);
    }

    int it = 0;
    for (int t = blockIdx.x; t < p.num_tiles; t += gridDim.x, ++it) {
        const int tx = t % p.tiles_x, ty = (t / p.tiles_x) % p.tiles_y, n = t / (p.tiles_x * p.tiles_y);
        const int ox0 = tx * SF_TW, oy0 = ty * SF_TH;

        // ---- P0: prefetched patch registers -> shared memory; then start fetching the next tile's patch
#pragma unroll
        for (int u = 0; u < SF_PER; ++u) {
            const int i = threadIdx.x + u * SF_THREADS;
            if (i < SF_NV) {
                const int v = i % SF_PV, rr = i / SF_PV;
                *reinterpret_cast<uint2*>(&sm.patch[rr / SF_PH][rr % SF_PH][4 * v]) =
                    sf_pack_vec<FP32>(pre[u], p.flip_x);
            }
        }
        __syncthreads();
        {
            const int tn = t + gridDim.x;
#pragma unroll
            for (int u = 0; u < SF_PER; ++u) {
                const int i = threadIdx.x + u * SF_THREADS;
                if (i < SF_NV && tn < p.num_tiles) pre[u] = sf_load_vec<FP32>(p, tn, i);
            }
        }

        // ---- P1: im2col rows of the 18 x 10 conv1 outputs (row r = y1l * 18 + x1l): k = c*9 + ky*3 + kx, K padded to 32
#pragma unroll 1
        for (int r = threadIdx.x; r < SF_CPIX; r += SF_THREADS) {
            const int y1l = r / SF_CW, x1l = r - y1l * SF_CW;
            __half v[32];
#pragma unroll
            for (int c = 0; c < 3; ++c)
#pragma unroll
                for (int ky = 0; ky < 3; ++ky)
#pragma unroll
                    for (int kx = 0; kx < 3; ++kx) v[c * 9 + ky * 3 + kx] = sm.patch[c][2 * y1l + ky][1 + 2 * x1l + kx];
#pragma unroll
            for (int k = 27; k < 32; ++k) v[k] = __float2half(0.f);
            uint8_t* row = sm.a + (r >> 7) * 16384 + (r & 127) * 128;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                uint4 q;
                __half* qh = reinterpret_cast<__half*>(&q);
#pragma unroll
                for (int e = 0; e < 8; ++e) qh[e] = v[8 * j + e];
                *reinterpret_cast<uint4*>(row + ((j ^ (r & 7)) << 4)) = q;
            }
        }
        fence_proxy_async();
        __syncthreads();

        // ---- P2: conv1 on the tensor cores: conv1 rows 0..179 lie in the first three 64-row blocks of A1
        if (it == 0) mbar_wait(&sm.w_full, 0);
        float acc1[3][2][8];
#pragma unroll
        for (int b = 0; b < 3; ++b)
#pragma unroll
            for (int c = 0; c < 2; ++c)
#pragma unroll
                for (int i = 0; i < 8; ++i) acc1[b][c][i] = 0.f;
        wg_fence();
#pragma unroll
        for (int b = 0; b < 3; ++b)
#pragma unroll
            for (int k = 0; k < 2; ++k)
                wg_mma_chunks<2>(acc1[b], 0, 2, smem_u32(sm.a) + b * 8192 + k * 32, smem_u32(sm.b1) + k * 32);
        wg_commit();
        wg_wait0();

        // ---- P3: conv1 epilogue -> chunk-major fp16 tile (zero outside the image: the depthwise pads conv1's output)
#pragma unroll
        for (int b = 0; b < 3; ++b)
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int r = b * 64 + frag_row(warp, lane, i);
                if (r < SF_CPIX) {
                    const int y1l = r / SF_CW, x1l = r - y1l * SF_CW;
                    const int y1 = oy0 - 1 + y1l, x1 = ox0 - 1 + x1l;
                    const bool in = y1 >= 0 && y1 < p.Ho && x1 >= 0 && x1 < p.Wo;
#pragma unroll
                    for (int c = 0; c < 2; ++c) {
                        const int ch = c * 16 + frag_col(lane, i);
                        __half2 h = zero2;
                        if (in) h = expand_relu6(acc1[b][c][2 * i] + sm.bias1[ch], acc1[b][c][2 * i + 1] + sm.bias1[ch + 1]);
                        *reinterpret_cast<__half2*>(sm.t + (ch >> 3) * SF_TCHUNK + r * 16 + (ch & 7) * 2) = h;
                    }
                }
            }
        __syncthreads();

        // ---- P4: depthwise 3x3 (+ bias, ReLU6) on the CUDA cores: thread = channel pair x 4x4 micro-block, packed fp16
        {
            const int cp = threadIdx.x & 15, sub = (threadIdx.x >> 4) & 1;
            const bool mir = sub != 0;
            const int blk = (warp << 1) | sub;              // 8 micro-blocks: 2 rows x 4 columns of 4x4 pixels
            const int oy = (blk >> 2) * 4, ox = (blk & 3) * 4;
            const __half2 bh = __floats2half2_rn(sm.biasdw[2 * cp], sm.biasdw[2 * cp + 1]);
            const __half2* tile_in = reinterpret_cast<const __half2*>(sm.t + (cp >> 2) * SF_TCHUNK) + (cp & 3);
            __half2 acc[4][4];
            dw_slab_hfma2<3, 4, SF_CW, 32, 4>(tile_in, reinterpret_cast<const __half2*>(&sm.wdw[0][0]), cp, mir, oy, ox, bh, acc);
            // A1 is dead (conv1 retired): the first M-tile of its buffer now holds A2 (128 pixels x 32 channels)
            dw_relu6(acc);
            dw_store_a<4>(sm.a, 16384, acc, oy, ox, mir, cp >> 2, cp);
        }
        fence_proxy_async();
        __syncthreads();

        // ---- P5: stem 1x1 on the tensor cores
        float acc2[2][2][8];
#pragma unroll
        for (int b = 0; b < 2; ++b)
#pragma unroll
            for (int c = 0; c < 2; ++c)
#pragma unroll
                for (int i = 0; i < 8; ++i) acc2[b][c][i] = 0.f;
        wg_fence();
#pragma unroll
        for (int b = 0; b < 2; ++b)
#pragma unroll
            for (int k = 0; k < 2; ++k)
                wg_mma_chunks<2>(acc2[b], 0, p.n_tile >> 4, smem_u32(sm.a) + b * 8192 + k * 32, smem_u32(sm.b2) + k * 32);
        wg_commit();
        wg_wait0();

        // ---- P6: output rows (no activation after the stem's 1x1 + BN)
#pragma unroll
        for (int b = 0; b < 2; ++b)
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int pix = b * 64 + frag_row(warp, lane, i);
                const int oy = oy0 + (pix >> 4), ox = ox0 + (pix & 15);
                if (oy < p.Ho && ox < p.Wo)
                    proj_store_row<2>(p.out, nullptr, (((size_t)n * p.Ho + oy) * p.Wo + ox) * p.C0, p.C0, acc2[b], i, sm.biaspw,
                                      lane);
            }
        __syncthreads();      // the A buffer, the conv1 tile and the patch are free for the next tile
    }
}

}  // namespace lp

using namespace lp;

// 1 when lp_stem_fused_f16 handles this shape (else the caller runs lp_stem_conv3x3_s2 + lp_dwconv_f16 + lp_pw1x1_f16)
extern "C" int lp_stem_fused_supported(int H, int W, int C0) {
    return (H > 0 && W > 0 && H % 2 == 0 && W % 4 == 0 && C0 >= 8 && C0 % 8 == 0 && C0 <= 32) ? 1 : 0;
}

// w1_packed: [32][64] fp16, row co = the 27 BN-folded taps (k = c*9 + ky*3 + kx) of output channel co, zero padded.
// w_dw: [9][32] tap-major BN-folded depthwise weights.  w_pw_packed / b_pw_packed: lp_pw1x1_pack(K = 32, N = C0).
extern "C" int lp_stem_fused_f16(const void* x, int x_is_fp32, int flip_x, const void* w1_packed, const float* b1,
                                 const void* w_dw, const float* b_dw, const void* w_pw_packed, const float* b_pw_packed,
                                 void* out, int N, int H, int W, int C0, lp_stream_t stream) {
    LP_CHECK_ARG(x && w1_packed && w_dw && w_pw_packed && out, "lp_stem_fused_f16: null pointer");
    LP_CHECK_ARG(N > 0 && lp_stem_fused_supported(H, W, C0),
                 "lp_stem_fused_f16: unsupported shape N=%d H=%d W=%d C0=%d (H even, W %% 4 == 0, C0 %% 8 == 0, C0 <= 32)", N,
                 H, W, C0);
    LP_CHECK_ARG(flip_x == 0 || flip_x == 1, "lp_stem_fused_f16: flip_x=%d (0 plain, 1 mirrored)", flip_x);
    if ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(out) | reinterpret_cast<uintptr_t>(w1_packed) |
         reinterpret_cast<uintptr_t>(w_pw_packed)) & 15) {
        set_error("lp_stem_fused_f16: pointers must be 16-byte aligned");
        return LP_ERR_ALIGN;
    }
    SfParams p;
    memset(&p, 0, sizeof(p));
    p.N = N; p.H = H; p.W = W; p.Ho = H / 2; p.Wo = W / 2; p.C0 = C0;
    p.n_tile = (C0 + 15) / 16 * 16;
    p.tiles_x = (p.Wo + SF_TW - 1) / SF_TW;
    p.tiles_y = (p.Ho + SF_TH - 1) / SF_TH;
    p.num_tiles = p.tiles_x * p.tiles_y * N;
    p.flip_x = flip_x; p.x_is_fp32 = x_is_fp32;
    p.x = x; p.b1 = b1; p.w_dw = reinterpret_cast<const __half*>(w_dw); p.b_dw = b_dw; p.b_pw = b_pw_packed;
    p.out = reinterpret_cast<__half*>(out);
    CUtensorMap m1, m3;
    int rc = make_tmap_rows64(&m1, w1_packed, 32, 64, 32, CU_TENSOR_MAP_SWIZZLE_128B);
    if (rc) return rc;
    rc = make_tmap_rows64(&m3, w_pw_packed, p.n_tile, 64, p.n_tile, CU_TENSOR_MAP_SWIZZLE_128B);
    if (rc) return rc;
    const int smem = (int)sizeof(SfSmem);      // ~58 KB: three CTAs per SM
    int grid = 3 * num_sms();
    if (grid > p.num_tiles) grid = p.num_tiles;
    cudaError_t e;
    if (x_is_fp32) {
        e = cudaFuncSetAttribute((const void*)stem_fused_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        if (e != cudaSuccess) return cuda_fail(e, "cudaFuncSetAttribute(stem_fused)");
        stem_fused_kernel<true><<<grid, SF_THREADS, smem, (cudaStream_t)stream>>>(m1, m3, p);
    } else {
        e = cudaFuncSetAttribute((const void*)stem_fused_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        if (e != cudaSuccess) return cuda_fail(e, "cudaFuncSetAttribute(stem_fused)");
        stem_fused_kernel<false><<<grid, SF_THREADS, smem, (cudaStream_t)stream>>>(m1, m3, p);
    }
    LP_LAUNCH_CHECK("stem_fused_kernel");
    return LP_OK;
}
