// Fused depthwise 7x7 (stride 1) + ReLU6 + pointwise projection (+ residual) of an inverted-residual block
// (reference lib/models/layers/layers.py:100-118: depth_conv -> point_conv -> optional identity add).
//
// Unfused, the 6x-expanded tensor is written by the depthwise kernel and read back by the projection GEMM; here it
// never leaves the SM.  Projections up to 64 channels (and the heads) run dw_project_kernel; wider block projections run
// dw_project_wide_kernel further below.  dw_project_kernel, per CTA (persistent over 16x16-pixel output tiles):
//   warp 16 (1 thread) TMA producer: haloed 22x22x32-channel input slabs (hardware zero fill = conv padding) into a
//                      4-deep ring, projection-weight K blocks into a 2-deep ring
//   warps 0-15         depthwise on the CUDA cores, two groups of 8 warps working on the two 32-channel halves of a
//                      64-channel K block: one 4x4 micro-block x channel pair per thread per slab, with the arithmetic
//                      of dw_inner.cuh: blocks (HEAD = 0) its packed-fp16 chains (dw_slab_hfma2), heads (HEAD = 1) its
//                      fp32 accumulation (dw_ffma); results written as fp16 straight into the 128B-swizzled K-major
//                      A-operand tiles (dw_store_a)
//   warps 0-15         as four warpgroups, one per 64 pixels: wgmma D[64 px x Co] += A[64 x 64 ch] * Wp^T per
//                      64-channel K block, fp32 accumulators in registers; then the epilogue from the accumulator
//                      fragments: + folded-BN bias (+ residual), fp16 NHWC (proj_store_row; heads: NCHW fp32/fp16
//                      planes)
// HBM traffic per block: read N*H*W*Ce*2 (+ N*H*W*Co*2 residual), write N*H*W*Co*2  -- the depthwise output
// (N*H*W*Ce*2 written + read again) is gone; the kernel is bound by the FMA pipe (2*49 flop per expanded element).
#include "common.cuh"
#include "dw_inner.cuh"

namespace lp {

constexpr int FP_T = 16;                         // output tile side
constexpr int FP_CB = 32;                        // channels per slab
template <int K> struct FpCfg {
    static constexpr int I = FP_T + K - 1;                       // haloed input side (22 for k = 7, 20 for k = 5)
    static constexpr int IN_BYTES = I * I * FP_CB * 2;           // 30976 / 25600
    static constexpr int W_BYTES = K * K * FP_CB * 2;            // depthwise weights of one slab: 3136 / 1600 B
};
constexpr int FP_IN_STRIDE = 35840;                           // ring pitch: input tile + weight slab (multiple of 1024)
constexpr int FP_W_OFF = 31744;                               // weights inside a ring stage (128-byte aligned)
constexpr int FP_NIN = 4;                                      // slab ring: even slabs use stages 0/2, odd 1/3
constexpr int FP_A_TILE = 128 * 64 * 2;                       // one M-tile x one 64-channel K block, 16 KiB
constexpr int FP_NB = 2;
constexpr int FP_B_BYTES = 160 * 64 * 2;                      // Co <= 160
constexpr int FP_DW_WARPS = 16;                                // two groups of 8: even / odd 32-channel slabs
constexpr int FP_THREADS = (FP_DW_WARPS + 4) * 32;   // + one producer warpgroup (one thread of it works)
// registers: 20 warps leave 96 per thread at launch (5 warps per SM sub-partition); the producer warpgroup gives up
// 72 of them so that the four compute warpgroups, which hold up to 64 accumulators each, run with 112
constexpr int FP_REGS_PRODUCER = 24, FP_REGS_COMPUTE = 112;
// setmaxnreg.inc only draws on what setmaxnreg.dec released in the CTA: 128 x (96 - 24) >= 512 x (112 - 96)
static_assert(128 * (96 - FP_REGS_PRODUCER) >= 512 * (FP_REGS_COMPUTE - 96), "register hand-over exceeds the released pool");
static_assert(FP_W_OFF >= FpCfg<7>::IN_BYTES && FP_W_OFF + FpCfg<7>::W_BYTES <= FP_IN_STRIDE, "ring stage layout");
constexpr int FP_MAX_CE = 1024;
constexpr size_t FP_SMEM = (size_t)FP_NIN * FP_IN_STRIDE + 2 * FP_A_TILE + FP_NB * FP_B_BYTES + 1024 + FP_MAX_CE * 4 + 1024;

struct FpBars {
    uint64_t in_full[FP_NIN], in_empty[FP_NIN];
    uint64_t b_full[FP_NB], b_empty[FP_NB];
};

struct FpParams {
    int N, H, W, Ce, Co, n_tile;      // n_tile = round_up(Co, 16)
    int tiles_x, tiles_y, num_tiles;
    int nslabs, nkb;
    int ns0;                          // slabs taken from the first source (HEAD mode: the rest come from the second)
    int out_fp32;                     // HEAD mode: NCHW output dtype
    const __half* w_dw;               // [k*k][Ce]
    const float* b_dw;                // [Ce] (HEAD mode: padded per slab, nslabs*32)
    const float* b_pj;                // packed, n_tile
    const __half* residual;           // [N,H,W,Co] or null
    void* out;                        // [N,H,W,Co] fp16 (HEAD: [N,Co,H,W] fp32/fp16)
};

// HEAD = 0: block projection (ReLU6 after the depthwise, NHWC fp16 output with bias and optional residual).
// HEAD = 1: output head (two sources, ReLU after the depthwise, bias-free 1x1, NCHW fp32/fp16 output).
// NC: 16-column accumulator chunks held per thread (>= n_tile / 16).
__device__ __forceinline__ void fp_dw_sync() { asm volatile("bar.sync 1, 512;" ::: "memory"); }

template <int K, int HEAD, int NC>
__global__ void __launch_bounds__(FP_THREADS, 1)
dw_project_kernel(const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_x1,
                  const __grid_constant__ CUtensorMap map_w, const __grid_constant__ CUtensorMap map_dw,
                  const __grid_constant__ FpParams p) {
    using Cfg = FpCfg<K>;
    constexpr int FP_I = Cfg::I;
    extern __shared__ __align__(1024) uint8_t smem[];
    uint8_t* sIn = smem;                                         // FP_NIN x [22][22][32] fp16
    uint8_t* sA = smem + FP_NIN * FP_IN_STRIDE;                  // [mtile 2] x 16 KiB, 128B-swizzled
    uint8_t* sB = sA + 2 * FP_A_TILE;                            // FP_NB x [n_tile][64] fp16, 128B-swizzled
    float* sBias = reinterpret_cast<float*>(sB + FP_NB * FP_B_BYTES);    // projection bias (<= 160)
    float* sBdw = sBias + 192;                                            // depthwise bias (<= FP_MAX_CE)
    FpBars* bars = reinterpret_cast<FpBars*>(sBdw + FP_MAX_CE);

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&map_x);
        if (HEAD) tma_prefetch_desc(&map_x1);
        tma_prefetch_desc(&map_w);
        tma_prefetch_desc(&map_dw);
        for (int i = 0; i < FP_NIN; ++i) { mbar_init(&bars->in_full[i], 1); mbar_init(&bars->in_empty[i], 8); }
        for (int i = 0; i < FP_NB; ++i) { mbar_init(&bars->b_full[i], 1); mbar_init(&bars->b_empty[i], FP_DW_WARPS); }
        fence_barrier_init();
    }
    for (int i = threadIdx.x; i < p.n_tile; i += FP_THREADS) sBias[i] = p.b_pj ? p.b_pj[i] : 0.f;
    for (int i = threadIdx.x; i < p.nslabs * FP_CB; i += FP_THREADS)
        sBdw[i] = (p.b_dw && (HEAD || i < p.Ce)) ? p.b_dw[i] : 0.f;
    pdl_launch_dependents();
    __syncthreads();
    pdl_wait();                   // the expanded input of this block is complete from here on

    if (warp >= FP_DW_WARPS) {
        // ------------------------------------------------------------------ TMA producer
        regs_dec<FP_REGS_PRODUCER>();
        if (warp == FP_DW_WARPS && lane == 0) {
            uint32_t iu[2] = {0, 0}, bs = 0, bph = 0;
            for (int t = blockIdx.x; t < p.num_tiles; t += gridDim.x) {
                const int tx = t % p.tiles_x, ty = (t / p.tiles_x) % p.tiles_y, n = t / (p.tiles_x * p.tiles_y);
                for (int s = 0; s < p.nslabs; ++s) {
                    if ((s & 1) == 0) {   // projection weights of K block s/2
                        mbar_wait_backoff(&bars->b_empty[bs], bph ^ 1);
                        mbar_expect_tx(&bars->b_full[bs], p.n_tile * 128);
                        tma_load_2d(sB + bs * FP_B_BYTES, &map_w, &bars->b_full[bs], 0, (s >> 1) * p.n_tile);
                        if (++bs == FP_NB) { bs = 0; bph ^= 1; }
                    }
                    const int g = s & 1;                              // even / odd slab group, stages g and g+2
                    const uint32_t is = 2 * (iu[g] & 1) + g;
                    mbar_wait_backoff(&bars->in_empty[is], ((iu[g] >> 1) & 1) ^ 1);
                    mbar_expect_tx(&bars->in_full[is], Cfg::IN_BYTES + Cfg::W_BYTES);
                    const bool second = HEAD && s >= p.ns0;
                    tma_load_4d(sIn + is * FP_IN_STRIDE, second ? &map_x1 : &map_x, &bars->in_full[is],
                                (second ? s - p.ns0 : s) * FP_CB, tx * FP_T - K / 2, ty * FP_T - K / 2, n);
                    tma_load_2d(sIn + is * FP_IN_STRIDE + FP_W_OFF, &map_dw, &bars->in_full[is], s * FP_CB, 0);
                    ++iu[g];
                }
            }
        }
    } else {
        // ------------------------------------------------------------------ depthwise warps + epilogue
        regs_inc<FP_REGS_COMPUTE>();
        const int cp = threadIdx.x & 15;
        const int sub = (threadIdx.x >> 4) & 1;
        const bool mir = sub != 0;
        const int grp = warp >> 3;                         // 0: even slabs (channels 0-31 of a K block), 1: odd slabs
        const int gw = warp & 7;
        const int blk = (gw << 1) | sub;                   // 16 micro-blocks: 4 x 4 of 4x4 pixels
        const int by = blk >> 2, bx = blk & 3;
        const int oy = by * 4, ox = bx * 4;
        uint32_t iu = 0;                                  // slabs consumed by this group
        // ---- MMA warpgroup wg = warp / 4 owns pixels 64*wg .. 64*wg+63 of the 256-pixel tile (M-tile wg / 2)
        const int wg = warp >> 2, wq = warp & 3;
        const int nch = p.n_tile >> 4;
        const uint32_t a_wg = smem_u32(sA + (wg >> 1) * FP_A_TILE) + (wg & 1) * 8192;
        uint32_t bs = 0, bph = 0;
        float pacc[NC][8];
        auto epilogue = [&](int te) {
            const int tx = te % p.tiles_x, ty = (te / p.tiles_x) % p.tiles_y, n = te / (p.tiles_x * p.tiles_y);
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int row = (wg & 1) * 64 + frag_row(wq, lane, i);    // pixel inside M-tile wg / 2
                const int py = (wg >> 1) * 8 + (row >> 4), px = row & 15;
                const int gy = ty * FP_T + py, gx = tx * FP_T + px;
                if (gy >= p.H || gx >= p.W) continue;
                if constexpr (HEAD) {
#pragma unroll
                    for (int c = 0; c < NC; ++c) {
                        const int co = c * 16 + frag_col(lane, i);
                        if (co >= p.Co) continue;
                        const float v0 = pacc[c][2 * i], v1 = pacc[c][2 * i + 1];
                        const size_t plane = (size_t)p.H * p.W;
                        const size_t o = ((size_t)n * p.Co + co) * plane + (size_t)gy * p.W + gx;
                        if (p.out_fp32) {
                            float* op = reinterpret_cast<float*>(p.out) + o;
                            op[0] = v0;
                            if (co + 1 < p.Co) op[plane] = v1;
                        } else {
                            __half* op = reinterpret_cast<__half*>(p.out) + o;
                            op[0] = __float2half_rn(v0);
                            if (co + 1 < p.Co) op[plane] = __float2half_rn(v1);
                        }
                    }
                } else {
                    proj_store_row<NC>(reinterpret_cast<__half*>(p.out), p.residual, (((size_t)n * p.H + gy) * p.W + gx) * p.Co,
                                       p.Co, pacc, i, sBias, lane);
                }
            }
        };
        int it = 0;
        for (int t = blockIdx.x; t < p.num_tiles; t += gridDim.x, ++it) {
#pragma unroll
            for (int c = 0; c < NC; ++c)
#pragma unroll
                for (int i = 0; i < 8; ++i) pacc[c][i] = 0.f;
            for (int kb = 0; kb < p.nkb; ++kb) {
                // (Splitting an odd last slab by rows between the two groups - each on its own M-tile, 2x4 micro-blocks -
                // was measured in round 2: 12 % slower.  The FMA pipe, not the idle group, bounds the kernel, and the
                // smaller micro-blocks need more LDS per MAC.)
                const int s = 2 * kb + grp;
                const bool have = s < p.nslabs;            // the last K block may hold a single slab
                // Depthwise (dw_inner.cuh): blocks (HEAD = 0) run the packed-fp16 chains; the heads (HEAD = 1) feed the
                // network outputs directly and keep fp32 accumulation.  The slab's weights are TMA-staged next to its
                // input tile ([K*K][32] fp16; channels beyond Ce are zero-filled by the tensor map).
                float2 acc[4][4];
                __half2 acch[4][4];
                if (have) {
                    const float2 b2 = *reinterpret_cast<const float2*>(sBdw + s * FP_CB + 2 * cp);
                    const uint32_t is = 2 * (iu & 1) + grp;          // this group's stages: grp, grp+2
                    mbar_wait(&bars->in_full[is], (iu >> 1) & 1);
                    const __half2* tile_in = reinterpret_cast<const __half2*>(sIn + is * FP_IN_STRIDE) + cp;
                    const __half2* wslab = reinterpret_cast<const __half2*>(sIn + is * FP_IN_STRIDE + FP_W_OFF);
                    if constexpr (HEAD) {
                        __half2 wreg[K * K];
                        dw_load_wslab<K, FP_CB>(wslab, cp, mir, wreg);
                        dw_ffma<K, 4, FP_I, FP_CB / 2>(tile_in, wreg, mir, oy, ox, b2, acc);
                    } else {
                        dw_slab_hfma2<K, 4, FP_I, FP_CB>(tile_in, wslab, cp, mir, oy, ox, __float22half2_rn(b2), acch);
                    }
                    __syncwarp();
                    if (lane == 0) mbar_arrive(&bars->in_empty[is]);
                    ++iu;
                }
                // the single A buffer is free once every warpgroup's MMAs of the previous K block have retired
                fp_dw_sync();
                if (have) {
                    if constexpr (HEAD) {
                        // ReLU in fp32, then one rounding (a packed hmax after rounding could turn +0 into -0)
#pragma unroll
                        for (int i = 0; i < 4; ++i)
#pragma unroll
                            for (int j = 0; j < 4; ++j)
                                acch[i][j] = __floats2half2_rn(fmaxf(acc[i][j].x, 0.f), fmaxf(acc[i][j].y, 0.f));
                    } else {
                        dw_relu6(acch);
                    }
                    dw_store_a<4>(sA, FP_A_TILE, acch, oy, ox, mir, (grp << 2) | (cp >> 2), cp);
                    fence_proxy_async();
                }
                fp_dw_sync();                              // A tile complete
                // projection of this K block: 32 channels per slab present
                const int k16 = 2 * min(2, p.nslabs - 2 * kb);
                mbar_wait(&bars->b_full[bs], bph);
                const uint32_t b_base = smem_u32(sB + bs * FP_B_BYTES);
                wg_fence();
                for (int k = 0; k < k16; ++k) wg_mma_chunks<NC>(pacc, 0, nch, a_wg + k * 32, b_base + k * 32);
                wg_commit();
                wg_wait0();
                __syncwarp();
                if (lane == 0) mbar_arrive(&bars->b_empty[bs]);
                if (++bs == FP_NB) { bs = 0; bph ^= 1; }
            }
            epilogue(t);
        }
    }
}

// Instantiations by accumulator width: n_tile <= 16 * NC.
template <int K, int HEAD, int NC>
static int launch_dw_project_nc(const CUtensorMap& m0, const CUtensorMap& m1, const CUtensorMap& mw, const CUtensorMap& md,
                                const FpParams& p, cudaStream_t stream) {
    auto kern = dw_project_kernel<K, HEAD, NC>;
    cudaError_t e = cudaFuncSetAttribute((const void*)kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)FP_SMEM);
    if (e != cudaSuccess) return cuda_fail(e, "cudaFuncSetAttribute(dw_project_kernel)");
    const int grid = p.num_tiles < num_sms() ? p.num_tiles : num_sms();
    cudaError_t le = launch_pdl(kern, dim3(grid), dim3(FP_THREADS), FP_SMEM, stream, m0, m1, mw, md, p);
    if (le != cudaSuccess) return cuda_fail(le, HEAD ? "launch dw_project_kernel<5,1>" : "launch dw_project_kernel<7,0>");
    LP_LAUNCH_CHECK(HEAD ? "dw_project_kernel<5,1>" : "dw_project_kernel<7,0>");
    return LP_OK;
}

template <int K, int HEAD>
static int launch_dw_project(const CUtensorMap& m0, const CUtensorMap& m1, const CUtensorMap& mw, const CUtensorMap& md,
                             const FpParams& p, cudaStream_t stream) {
    if (p.n_tile <= 32) return launch_dw_project_nc<K, HEAD, 2>(m0, m1, mw, md, p, stream);
    if constexpr (!HEAD) {
        return launch_dw_project_nc<K, HEAD, 4>(m0, m1, mw, md, p, stream);     // blocks: Co <= 64 (wider: below)
    } else {
        if (p.n_tile <= 64) return launch_dw_project_nc<K, HEAD, 4>(m0, m1, mw, md, p, stream);
        return launch_dw_project_nc<K, HEAD, 8>(m0, m1, mw, md, p, stream);     // heads: Co <= 128
    }
}

// ------------------------------------------------------------------ wide projections (block Co 65..160)
// dw_project_kernel keeps its projection accumulators live through the depthwise loop; at Co > 64 they no longer fit
// beside the loop's ~95 registers and ptxas spills inside it.  This kernel gives the two jobs to different warps:
//   warps 0-7   (2 warpgroups) depthwise, two groups of 4 warps on the even / odd 32-channel slabs of a K block: one
//               4x4 micro-block x channel pair per thread (dw_inner.cuh, the same packed-fp16 chain as above), ReLU6'd
//               fp16 results into a 2-deep ring of 128B-swizzled A tiles (full / empty mbarriers)
//   warps 8-15  (2 warpgroups) projection: wgmma m64 x n(16 NC) x k16 over 64 pixels each, fp32 accumulators in
//               registers; every K block is committed and the previous one waited for (wait_group 1), so the MMAs of
//               K block kb run under the depthwise of kb + 1; then the bias / residual / NHWC epilogue, which runs
//               under the depthwise of the next tile
// There is no producer warp: the first thread of each depthwise group issues the TMA loads of its group's haloed
// 22x14x32 input slabs + depthwise weights (two ring stages per group, the slab after next is loaded when the slab
// before is released), the first MMA thread those of the projection-weight K blocks (two-slot ring).  ptxas compiles
// a kernel for one register budget, whatever setmaxnreg does at run time; with 16 warps that budget is 128, enough for
// the 80 accumulators of NC = 10 and for the depthwise loop (a 17th warp would count as 20 and leave 96).
// Tiles are 16 x 8 pixels (one 128-row M-tile): more tiles per persistent CTA than 16 x 16, so that the epilogue and
// pipeline fill of one tile hide under the next.
constexpr int FW_TX = 16, FW_TY = 8;                              // output tile
constexpr int FW_IX = FW_TX + 6, FW_IY = FW_TY + 6;               // haloed input slab: 22 x 14 pixels
constexpr int FW_IN_BYTES = FW_IX * FW_IY * FP_CB * 2;            // 19712
constexpr int FW_W_OFF = FW_IN_BYTES;                             // depthwise weights of the slab (128-byte aligned)
constexpr int FW_IN_STRIDE = 23552;                               // ring pitch (multiple of 1024)
constexpr int FW_NIN = 4;                                         // slab ring: group g uses stages g and g + 2
constexpr int FW_NA = 2, FW_NB = 2;                               // A-tile ring, projection-weight ring
constexpr int FW_DW_WARPS = 8, FW_MMA_WARPS = 8;
constexpr int FW_THREADS = (FW_DW_WARPS + FW_MMA_WARPS) * 32;
static_assert(FW_W_OFF % 128 == 0 && FW_W_OFF + FpCfg<7>::W_BYTES <= FW_IN_STRIDE, "ring stage layout");
constexpr size_t FW_SMEM = (size_t)FW_NIN * FW_IN_STRIDE + FW_NA * FP_A_TILE + FW_NB * FP_B_BYTES + 1024 + FP_MAX_CE * 4 + 1024;

struct FwBars {
    uint64_t in_full[FW_NIN], in_empty[FW_NIN];
    uint64_t a_full[FW_NA], a_empty[FW_NA];
    uint64_t b_full[FW_NB], b_empty[FW_NB];
};

// NC = n_tile / 16 exactly: every K=16 slice of the projection is one straight-line m64n(16 NC)k16.
template <int NC>
__global__ void __launch_bounds__(FW_THREADS, 1)
dw_project_wide_kernel(const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_w,
                       const __grid_constant__ CUtensorMap map_dw, const __grid_constant__ FpParams p) {
    extern __shared__ __align__(1024) uint8_t smem[];
    uint8_t* sIn = smem;                                          // FW_NIN x ([14][22][32] fp16 + [49][32] fp16)
    uint8_t* sA = smem + FW_NIN * FW_IN_STRIDE;                   // FW_NA x [128 px][64 ch], 128B-swizzled
    uint8_t* sB = sA + FW_NA * FP_A_TILE;                         // FW_NB x [n_tile][64] fp16, 128B-swizzled
    float* sBias = reinterpret_cast<float*>(sB + FW_NB * FP_B_BYTES);     // projection bias (<= 160)
    float* sBdw = sBias + 192;                                             // depthwise bias (<= FP_MAX_CE)
    FwBars* bars = reinterpret_cast<FwBars*>(sBdw + FP_MAX_CE);

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t my_tiles = (p.num_tiles - blockIdx.x + gridDim.x - 1) / gridDim.x;   // grid <= num_tiles

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&map_x);
        tma_prefetch_desc(&map_w);
        tma_prefetch_desc(&map_dw);
        for (int i = 0; i < FW_NIN; ++i) { mbar_init(&bars->in_full[i], 1); mbar_init(&bars->in_empty[i], FW_DW_WARPS / 2); }
        for (int i = 0; i < FW_NA; ++i) { mbar_init(&bars->a_full[i], FW_DW_WARPS); mbar_init(&bars->a_empty[i], FW_MMA_WARPS); }
        for (int i = 0; i < FW_NB; ++i) { mbar_init(&bars->b_full[i], 1); mbar_init(&bars->b_empty[i], FW_MMA_WARPS); }
        fence_barrier_init();
    }
    for (int i = threadIdx.x; i < p.n_tile; i += FW_THREADS) sBias[i] = p.b_pj ? p.b_pj[i] : 0.f;
    for (int i = threadIdx.x; i < p.nslabs * FP_CB; i += FW_THREADS) sBdw[i] = (p.b_dw && i < p.Ce) ? p.b_dw[i] : 0.f;
    // The projection always runs all four K=16 slices of a K block.  In the half K block of an odd slab count the A
    // channels 32..63 hold zeros (or ReLU6 outputs of an earlier K block) against zero-padded weights: exact zero
    // products, which leave the fp32 accumulators unchanged.
    for (int i = threadIdx.x; i < FW_NA * FP_A_TILE / 16; i += FW_THREADS) reinterpret_cast<uint4*>(sA)[i] = make_uint4(0, 0, 0, 0);
    fence_proxy_async();
    pdl_launch_dependents();
    __syncthreads();
    pdl_wait();                   // the expanded input of this block is complete from here on

    if (warp < FW_DW_WARPS) {
        // ------------------------------------------------------------------ depthwise warps
        const int cp = threadIdx.x & 15;
        const bool mir = ((threadIdx.x >> 4) & 1) != 0;
        const int grp = warp >> 2;                         // 0: even slabs (channels 0-31 of a K block), 1: odd slabs
        const int blk = ((warp & 3) << 1) | (int)mir;      // 8 micro-blocks: 2 x 4 of 4x4 pixels
        const int oy = (blk >> 2) * 4, ox = (blk & 3) * 4;
        const int jch = (grp << 2) | (cp >> 2);
        const bool loader = (warp & 3) == 0 && lane == 0;
        const uint32_t ng = (p.nslabs - grp + 1) >> 1;    // slabs of this group per tile
        const uint32_t nj = ng * my_tiles;
        // slab j of this group's sequence (tile j / ng of the CTA, its K block j % ng) -> stage 2 (j & 1) + grp
        auto load_slab = [&](uint32_t j) {
            const int t = blockIdx.x + (int)(j / ng) * gridDim.x, s = 2 * (int)(j % ng) + grp;
            const int tx = t % p.tiles_x, ty = (t / p.tiles_x) % p.tiles_y, n = t / (p.tiles_x * p.tiles_y);
            const uint32_t is = 2 * (j & 1) + grp;
            mbar_expect_tx(&bars->in_full[is], FW_IN_BYTES + FpCfg<7>::W_BYTES);
            tma_load_4d(sIn + is * FW_IN_STRIDE, &map_x, &bars->in_full[is], s * FP_CB, tx * FW_TX - 3, ty * FW_TY - 3, n);
            tma_load_2d(sIn + is * FW_IN_STRIDE + FW_W_OFF, &map_dw, &bars->in_full[is], s * FP_CB, 0);
        };
        if (loader) {
            if (nj > 0) load_slab(0);
            if (nj > 1) load_slab(1);
        }
        uint32_t iu = 0, au = 0;                           // slabs consumed by this group, K blocks handed over
        for (int t = blockIdx.x; t < p.num_tiles; t += gridDim.x) {
            for (int kb = 0; kb < p.nkb; ++kb, ++au) {
                const int s = 2 * kb + grp;
                const bool have = s < p.nslabs;            // the last K block may hold a single slab
                __half2 acch[4][4];
                if (have) {
                    const uint32_t is = 2 * (iu & 1) + grp;
                    if (loader && iu >= 1 && iu + 1 < nj) {
                        // the other stage of the group: slab iu - 1 is released by all four warps -> slab iu + 1
                        mbar_wait(&bars->in_empty[is ^ 2], ((iu - 1) >> 1) & 1);
                        load_slab(iu + 1);
                    }
                    const __half2 bh = __float22half2_rn(*reinterpret_cast<const float2*>(sBdw + s * FP_CB + 2 * cp));
                    mbar_wait(&bars->in_full[is], (iu >> 1) & 1);
                    const uint8_t* st = sIn + is * FW_IN_STRIDE;
                    dw_slab_hfma2<7, 4, FW_IX, FP_CB>(reinterpret_cast<const __half2*>(st) + cp,
                                                      reinterpret_cast<const __half2*>(st + FW_W_OFF), cp, mir, oy, ox, bh, acch);
                    __syncwarp();
                    if (lane == 0) mbar_arrive(&bars->in_empty[is]);
                    ++iu;
                }
                const uint32_t q = au & 1;
                mbar_wait(&bars->a_empty[q], ((au >> 1) & 1) ^ 1);
                if (have) {
                    dw_relu6(acch);
                    dw_store_a<4>(sA + q * FP_A_TILE, FP_A_TILE, acch, oy, ox, mir, jch, cp);
                    fence_proxy_async();
                }
                __syncwarp();
                if (lane == 0) mbar_arrive(&bars->a_full[q]);
            }
        }
    } else {
        // ------------------------------------------------------------------ projection MMAs + epilogue
        const int wg = (warp - FW_DW_WARPS) >> 2, wq = warp & 3;        // rows 64 wg .. 64 wg + 63 of the tile
        const bool loader = warp == FW_DW_WARPS && lane == 0;
        const uint32_t nu = my_tiles * p.nkb;
        auto load_w = [&](uint32_t v) {                                 // K block v % nkb -> slot v & 1
            const uint32_t q = v & 1;
            mbar_expect_tx(&bars->b_full[q], p.n_tile * 128);
            tma_load_2d(sB + q * FP_B_BYTES, &map_w, &bars->b_full[q], 0, (int)(v % p.nkb) * p.n_tile);
        };
        // K block v has retired in this warp: release its A tile and weight slot; the loader refills the slot with v + 2
        auto release = [&](uint32_t v) {
            __syncwarp();
            if (lane == 0) { mbar_arrive(&bars->a_empty[v & 1]); mbar_arrive(&bars->b_empty[v & 1]); }
            if (loader && v + 2 < nu) {
                mbar_wait(&bars->b_empty[v & 1], (v >> 1) & 1);
                load_w(v + 2);
            }
        };
        if (loader) {
            load_w(0);
            if (nu > 1) load_w(1);
        }
        uint32_t u = 0;                                                 // K blocks consumed (A and B rings alike)
        float pacc[NC][8];
        for (int t = blockIdx.x; t < p.num_tiles; t += gridDim.x) {
            for (int kb = 0; kb < p.nkb; ++kb, ++u) {
                const uint32_t q = u & 1, ph = (u >> 1) & 1;
                mbar_wait(&bars->a_full[q], ph);
                mbar_wait(&bars->b_full[q], ph);
                const uint32_t a_base = smem_u32(sA + q * FP_A_TILE) + wg * 8192, b_base = smem_u32(sB + q * FP_B_BYTES);
                wg_fence();
#pragma unroll
                for (int k = 0; k < 4; ++k) wg_mma_n<NC>(pacc, a_base + k * 32, b_base + k * 32, kb | k);
                wg_commit();
                if (kb > 0) {
                    wg_wait1();
                    release(u - 1);
                }
            }
            wg_wait0();
            release(u - 1);
            // epilogue: accumulator row = pixel of the 16 x 8 tile
            const int tx = t % p.tiles_x, ty = (t / p.tiles_x) % p.tiles_y, n = t / (p.tiles_x * p.tiles_y);
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int row = wg * 64 + frag_row(wq, lane, i);
                const int gy = ty * FW_TY + (row >> 4), gx = tx * FW_TX + (row & 15);
                if (gy >= p.H || gx >= p.W) continue;
                proj_store_row<NC>(reinterpret_cast<__half*>(p.out), p.residual, (((size_t)n * p.H + gy) * p.W + gx) * p.Co, p.Co,
                                   pacc, i, sBias, lane);
            }
        }
    }
}

template <int NC>
static int launch_dw_project_wide_nc(const CUtensorMap& mx, const CUtensorMap& mw, const CUtensorMap& md, const FpParams& p,
                                     cudaStream_t stream) {
    auto kern = dw_project_wide_kernel<NC>;
    cudaError_t e = cudaFuncSetAttribute((const void*)kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)FW_SMEM);
    if (e != cudaSuccess) return cuda_fail(e, "cudaFuncSetAttribute(dw_project_wide_kernel)");
    const int grid = p.num_tiles < num_sms() ? p.num_tiles : num_sms();
    cudaError_t le = launch_pdl(kern, dim3(grid), dim3(FW_THREADS), FW_SMEM, stream, mx, mw, md, p);
    if (le != cudaSuccess) return cuda_fail(le, "launch dw_project_wide_kernel");
    LP_LAUNCH_CHECK("dw_project_wide_kernel");
    return LP_OK;
}

static int launch_dw_project_wide(const CUtensorMap& mx, const CUtensorMap& mw, const CUtensorMap& md, const FpParams& p,
                                  cudaStream_t stream) {
    switch (p.n_tile / 16) {
        case 5: return launch_dw_project_wide_nc<5>(mx, mw, md, p, stream);
        case 6: return launch_dw_project_wide_nc<6>(mx, mw, md, p, stream);
        case 7: return launch_dw_project_wide_nc<7>(mx, mw, md, p, stream);
        case 8: return launch_dw_project_wide_nc<8>(mx, mw, md, p, stream);
        case 9: return launch_dw_project_wide_nc<9>(mx, mw, md, p, stream);
        default: return launch_dw_project_wide_nc<10>(mx, mw, md, p, stream);
    }
}

}  // namespace lp

using namespace lp;

// Fused depthwise-7x7(stride 1, +bias +ReLU6) -> pointwise projection (+bias, +residual).
// x [N,H,W,Ce] fp16 NHWC; w_dw tap-major [49][Ce]; w_proj_packed / b_proj_packed from lp_pw1x1_pack(K=Ce, N=Co);
// out [N,H,W,Co].  Ce % 8 == 0, Co % 8 == 0, Co <= 160.
extern "C" int lp_dw7_project_f16(const void* x, const void* w_dw, const float* b_dw, const void* w_proj_packed,
                                  const float* b_proj_packed, const void* residual, void* out, int N, int H, int W,
                                  int Ce, int Co, lp_stream_t stream) {
    LP_CHECK_ARG(x && w_dw && w_proj_packed && out, "lp_dw7_project_f16: null pointer");
    LP_CHECK_ARG(N > 0 && H > 0 && W > 0 && Ce >= 8 && Ce % 8 == 0 && Ce <= FP_MAX_CE - FP_CB && Co >= 8 && Co % 8 == 0 &&
                     Co <= 160,
                 "lp_dw7_project_f16: bad shape N=%d H=%d W=%d Ce=%d Co=%d (Ce <= 992, Co <= 160)", N, H, W, Ce, Co);
    if ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(out) | reinterpret_cast<uintptr_t>(w_proj_packed) |
         reinterpret_cast<uintptr_t>(residual) | reinterpret_cast<uintptr_t>(w_dw)) & 15) {
        set_error("lp_dw7_project_f16: pointers must be 16-byte aligned");
        return LP_ERR_ALIGN;
    }
    FpParams p;
    memset(&p, 0, sizeof(p));
    p.N = N; p.H = H; p.W = W; p.Ce = Ce; p.Co = Co;
    p.n_tile = (Co + 15) / 16 * 16;
    const bool wide = p.n_tile > 64;                  // dw_project_wide_kernel, 16 x 8 tiles
    const int tw = wide ? FW_TX : FP_T, th = wide ? FW_TY : FP_T;
    p.tiles_x = (W + tw - 1) / tw;
    p.tiles_y = (H + th - 1) / th;
    p.num_tiles = p.tiles_x * p.tiles_y * N;
    p.nslabs = (Ce + FP_CB - 1) / FP_CB;
    p.nkb = (Ce + 63) / 64;
    p.w_dw = reinterpret_cast<const __half*>(w_dw);
    p.b_dw = b_dw;
    p.b_pj = b_proj_packed;
    p.residual = reinterpret_cast<const __half*>(residual);
    p.out = out;
    p.ns0 = p.nslabs;
    CUtensorMap mx, mw, md;
    int rc = make_tmap_nhwc(&mx, x, N, H, W, Ce, FP_CB, wide ? FW_IX : FpCfg<7>::I, wide ? FW_IY : FpCfg<7>::I,
                            CU_TENSOR_MAP_SWIZZLE_NONE);
    if (rc) return rc;
    // packed projection weights: [kb][n_tile][64] (lp_pw1x1_pack with a single N chunk since Co <= 160)
    rc = make_tmap_rows64(&mw, w_proj_packed, p.nkb * p.n_tile, 64, p.n_tile, CU_TENSOR_MAP_SWIZZLE_128B);
    if (rc) return rc;
    rc = make_tmap_taps(&md, w_dw, 49, Ce);
    if (rc) return rc;
    if (wide) return launch_dw_project_wide(mx, mw, md, p, (cudaStream_t)stream);
    return launch_dw_project<7, 0>(mx, mx, mw, md, p, (cudaStream_t)stream);
}

// ------------------------------------------------------------------ fused output head (M4)
static int head_slabs(int C) { return (C + FP_CB - 1) / FP_CB; }

extern "C" size_t lp_head_fused_dw_elems(int C1, int C2) { return (size_t)25 * (head_slabs(C1) + head_slabs(C2)) * FP_CB; }
extern "C" size_t lp_head_fused_pw_elems(int C1, int C2, int Co) {
    const int ns = head_slabs(C1) + head_slabs(C2);
    return (size_t)((ns + 1) / 2) * ((Co + 15) / 16 * 16) * 64;
}
// dw1/dw2: tap-major [25][C] BN-folded depthwise weights, bdw1/bdw2 their biases; w1 [Co][C1], w2 [Co][C2].
// Outputs (host): dw_cat [25][ns*32] fp16, bdw_cat [ns*32] fp32, pw_packed [kb][n_tile][64] fp16 in slab order.
extern "C" int lp_head_fused_pack(const uint16_t* dw1, const float* bdw1, const uint16_t* dw2, const float* bdw2,
                                  const uint16_t* w1, const uint16_t* w2, int C1, int C2, int Co, uint16_t* dw_cat,
                                  float* bdw_cat, uint16_t* pw_packed) {
    LP_CHECK_ARG(dw1 && dw2 && w1 && w2 && dw_cat && bdw_cat && pw_packed && C1 > 0 && C2 > 0 && Co > 0,
                 "lp_head_fused_pack: bad args");
    const int s1 = head_slabs(C1), s2 = head_slabs(C2), ns = s1 + s2, CP = ns * FP_CB;
    const int nt = (Co + 15) / 16 * 16, nkb = (ns + 1) / 2;
    for (int t = 0; t < 25; ++t)
        for (int c = 0; c < CP; ++c) {
            const bool second = c >= s1 * FP_CB;
            const int cc = second ? c - s1 * FP_CB : c;
            const int C = second ? C2 : C1;
            dw_cat[(size_t)t * CP + c] = cc < C ? (second ? dw2 : dw1)[(size_t)t * C + cc] : (uint16_t)0;
        }
    for (int c = 0; c < CP; ++c) {
        const bool second = c >= s1 * FP_CB;
        const int cc = second ? c - s1 * FP_CB : c;
        const float* b = second ? bdw2 : bdw1;
        bdw_cat[c] = (b && cc < (second ? C2 : C1)) ? b[cc] : 0.f;
    }
    for (int kb = 0; kb < nkb; ++kb)
        for (int r = 0; r < nt; ++r)
            for (int kk = 0; kk < 64; ++kk) {
                const int c = kb * 64 + kk;                    // padded concatenated channel
                uint16_t v = 0;
                if (r < Co && c < CP) {
                    const bool second = c >= s1 * FP_CB;
                    const int cc = second ? c - s1 * FP_CB : c;
                    if (cc < (second ? C2 : C1)) v = (second ? w2 : w1)[(size_t)r * (second ? C2 : C1) + cc];
                }
                pw_packed[((size_t)kb * nt + r) * 64 + kk] = v;
            }
    return LP_OK;
}

// out[N,Co,H,W] = W1 * relu(dw5(a1) + b1) + W2 * relu(dw5(a2) + b2): both SepConv2d heads of one level in ONE kernel
// (reference lib/models/pose_mobilenet.py:151-154, lib/models/layers/layers.py:120-133).
extern "C" int lp_head_fused_f16(const void* a1, const void* a2, const void* dw_cat, const float* bdw_cat,
                                 const void* pw_packed, void* out_nchw, int out_fp32, int N, int H, int W, int C1, int C2,
                                 int Co, lp_stream_t stream) {
    LP_CHECK_ARG(a1 && a2 && dw_cat && bdw_cat && pw_packed && out_nchw, "lp_head_fused_f16: null pointer");
    LP_CHECK_ARG(N > 0 && H > 0 && W > 0 && C1 % 8 == 0 && C2 % 8 == 0 && C1 > 0 && C2 > 0 && Co > 0 && Co <= 128,
                 "lp_head_fused_f16: bad shape N=%d H=%d W=%d C1=%d C2=%d Co=%d", N, H, W, C1, C2, Co);
    if ((reinterpret_cast<uintptr_t>(a1) | reinterpret_cast<uintptr_t>(a2) | reinterpret_cast<uintptr_t>(dw_cat) |
         reinterpret_cast<uintptr_t>(pw_packed)) & 15) {
        set_error("lp_head_fused_f16: pointers must be 16-byte aligned");
        return LP_ERR_ALIGN;
    }
    FpParams p;
    memset(&p, 0, sizeof(p));
    p.N = N; p.H = H; p.W = W; p.Co = Co;
    p.ns0 = head_slabs(C1);
    p.nslabs = p.ns0 + head_slabs(C2);
    p.Ce = p.nslabs * FP_CB;
    LP_CHECK_ARG(p.Ce <= FP_MAX_CE, "lp_head_fused_f16: too many channels");
    p.nkb = (p.nslabs + 1) / 2;
    p.n_tile = (Co + 15) / 16 * 16;
    p.tiles_x = (W + FP_T - 1) / FP_T;
    p.tiles_y = (H + FP_T - 1) / FP_T;
    p.num_tiles = p.tiles_x * p.tiles_y * N;
    p.w_dw = reinterpret_cast<const __half*>(dw_cat);
    p.b_dw = bdw_cat;
    p.out = out_nchw;
    p.out_fp32 = out_fp32;
    CUtensorMap m0, m1, mw, md;
    int rc = make_tmap_nhwc(&m0, a1, N, H, W, C1, FP_CB, FpCfg<5>::I, FpCfg<5>::I, CU_TENSOR_MAP_SWIZZLE_NONE);
    if (rc) return rc;
    rc = make_tmap_nhwc(&m1, a2, N, H, W, C2, FP_CB, FpCfg<5>::I, FpCfg<5>::I, CU_TENSOR_MAP_SWIZZLE_NONE);
    if (rc) return rc;
    rc = make_tmap_rows64(&mw, pw_packed, p.nkb * p.n_tile, 64, p.n_tile, CU_TENSOR_MAP_SWIZZLE_128B);
    if (rc) return rc;
    rc = make_tmap_taps(&md, dw_cat, 25, p.Ce);
    if (rc) return rc;
    return launch_dw_project<5, 1>(m0, m1, mw, md, p, (cudaStream_t)stream);
}
