// One stride-1 inverted-residual block in ONE kernel (reference lib/models/layers/layers.py:90-118:
//   inv (1x1 expand + BN + ReLU6) -> depth_conv (7x7 depthwise + BN + ReLU6) -> point_conv (1x1 + BN) -> (+ identity)).
//
// The 6x-expanded tensor never exists in HBM: per 16x16-pixel output tile the CTA
//   * TMA-loads the NARROW haloed input tile X [22x22 px][Cin <= 64] (hardware zero fill = image border) as a
//     128B-swizzled K-major operand (484 rows of 128 B, channels beyond Cin zero-filled by the tensor map),
//   * expands it 32 channels at a time on the tensor cores: E[px, 32] = X[px, Cin] * We[32, Cin]^T, run by the two
//     warpgroups of the slab's group as wgmma (M=64, N=32) over 256 haloed pixels each (halo recompute factor 1.89 -
//     the tensor pipe is otherwise idle), fp32 accumulators in registers,
//   * the same warps turn the accumulators (+bias -> ReLU6 -> zero outside the image -> fp16) into the [22][22][32ch]
//     slab layout of the depthwise loop (the "epilogue" of the expansion),
//   * run the packed-fp16 7x7 depthwise on the slab (same HFMA2 loop as dwpw.cu), write ReLU6'd fp16 results into
//     the swizzled K-major A tile; the four warpgroups then run the projection wgmma on 64 pixels each (fp32
//     accumulators in registers for the whole tile),
//   * all 16 depthwise warps finish the tile from their accumulators: + bias, + identity row (read back from
//     global/L2), fp16 stores.
// Warp roles: 0-15 depthwise + MMA (two groups of 8 = even / odd 32-channel slabs), 16 TMA producer.
// HBM traffic of a block: read N*H*W*Cin*2 (x1.9 halo, L2 hits) + identity row, write N*H*W*Co*2.
#include "common.cuh"
#include "dw_inner.cuh"

namespace lp {

constexpr int BK_T = 16;                          // output tile side
constexpr int BK_I = BK_T + 6;                    // haloed side (22)
constexpr int BK_PIX = BK_I * BK_I;               // 484 haloed pixels = rows of X
constexpr int BK_CB = 32;                         // channels per slab
constexpr int BK_X_BYTES = 512 * 128;             // 4 M-tiles of 128 rows x 128 B (TMA fills the first 484 rows)
constexpr int BK_X_TX = BK_PIX * 128;             // bytes the TMA box delivers
constexpr int BK_WE_SLAB = BK_CB * 128;           // expansion weights of one slab: 32 rows x 128 B
constexpr int BK_CHUNK = 7840;                    // chunk-major slab: [4 chunks of 8 ch][484 px][16 B], chunk pitch = 7744 + 96
                                                  // (pitch = 32 mod 128: the 4 chunks of a pixel and the pixel of the mirrored
                                                  // half-warp fall into 8 different 16-byte bank groups -> conflict-free LDS;
                                                  // consecutive pixels of a chunk are contiguous -> conflict-free 16-byte STS)
constexpr int BK_SLAB = 31744;                    // 4 * 7840 = 31360 B, padded
constexpr int BK_DW_BYTES = 49 * BK_CB * 2;       // depthwise weights of one slab (tap-major [49][32]) = 3136 B
constexpr int BK_DW_SLAB = 3200;                 // their pitch in shared memory (TMA destinations are 128-byte aligned)
constexpr int BK_A_TILE = 128 * 64 * 2;
constexpr int BK_DW_WARPS = 16;
constexpr int BK_THREADS = (BK_DW_WARPS + 4) * 32;   // + one producer warpgroup (one thread of it works)
// registers: 20 warps leave 96 per thread at launch; the producer warpgroup hands 72 of them to the compute warpgroups
constexpr int BK_REGS_PRODUCER = 24, BK_REGS_COMPUTE = 112;
// setmaxnreg.inc only draws on what setmaxnreg.dec released in the CTA: 128 x (96 - 24) >= 512 x (112 - 96)
static_assert(128 * (96 - BK_REGS_PRODUCER) >= 512 * (BK_REGS_COMPUTE - 96), "register hand-over exceeds the released pool");
constexpr int BK_MAX_CE = 416;

struct BkBars {
    uint64_t w_full;
    // streaming mode (the three weight sets do not fit beside X and the slabs): two-slot rings
    uint64_t we_full[2], we_empty[2];          // expansion weights of a slab: producer -> the group that expands it
    uint64_t dw_full[2][2], dw_empty[2][2];    // depthwise weights of a slab, per group: producer -> the group's warps
    uint64_t wp_full[2], wp_empty[2];          // projection weights of a K block: producer -> all depthwise warps
    uint64_t x_full, x_empty;
};

struct BkParams {
    int N, H, W, Cin, Ce, Co, n_tile;
    int tiles_x, tiles_y, num_tiles;
    int nslabs, nkb, k16;             // k16 = K=16 MMA steps that carry input channels (ceil(Cin/16))
    int off_we, off_slab, off_dww, off_a, off_wp, off_bias;   // shared-memory layout (bytes)
    int wp_stage;                     // streaming mode: bytes of one projection-weight ring slot
    const float* b_exp;               // [Ce]
    const float* b_dw;                // [Ce]
    const float* b_pj;                // packed, n_tile
    const __half* residual;           // = x when the block has an identity connection, else null
    __half* out;                      // [N,H,W,Co]
};

// STREAM = 0: all weights of the block resident in shared memory; STREAM = 1: expansion / depthwise / projection weights
// travel through two-slot rings (blocks with Ce up to 288 at Cin = 48: stage 2 of LitePose-S).
// K16 = ceil(Cin / 16) K=16 steps of the expansion, NC = n_tile / 16 projection chunks: compile-time widths, so that every
// wgmma is issued straight-line (one m64n32k16 per expansion slice, one m64n(16 NC)k16 per projection slice).
template <int STREAM, int K16, int NC>
__global__ void __launch_bounds__(BK_THREADS, 1)
block_s1_kernel(const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_we,
                const __grid_constant__ CUtensorMap map_dw, const __grid_constant__ CUtensorMap map_wp,
                const __grid_constant__ BkParams p) {
    constexpr int K = 7;
    extern __shared__ __align__(1024) uint8_t smem[];
    uint8_t* sX = smem;
    uint8_t* sWe = smem + p.off_we;
    uint8_t* sSlab = smem + p.off_slab;
    uint8_t* sDww = smem + p.off_dww;
    uint8_t* sA = smem + p.off_a;
    uint8_t* sWp = smem + p.off_wp;
    float* sBexp = reinterpret_cast<float*>(smem + p.off_bias);
    float* sBdw = sBexp + BK_MAX_CE;
    float* sBpj = sBdw + BK_MAX_CE;
    BkBars* bars = reinterpret_cast<BkBars*>(sBpj + 64);

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&map_x);
        tma_prefetch_desc(&map_we);
        tma_prefetch_desc(&map_dw);
        tma_prefetch_desc(&map_wp);
        mbar_init(&bars->w_full, 1);
        for (int i = 0; i < 2; ++i) {
            mbar_init(&bars->we_full[i], 1);
            mbar_init(&bars->we_empty[i], BK_DW_WARPS / 2);
            mbar_init(&bars->wp_full[i], 1);
            mbar_init(&bars->wp_empty[i], BK_DW_WARPS);
            for (int g = 0; g < 2; ++g) { mbar_init(&bars->dw_full[g][i], 1); mbar_init(&bars->dw_empty[g][i], BK_DW_WARPS / 2); }
        }
        mbar_init(&bars->x_full, 1);
        mbar_init(&bars->x_empty, BK_DW_WARPS);
        fence_barrier_init();
    }
    for (int i = threadIdx.x; i < p.nslabs * BK_CB; i += BK_THREADS) {
        sBexp[i] = (i < p.Ce && p.b_exp) ? p.b_exp[i] : 0.f;
        sBdw[i] = (i < p.Ce && p.b_dw) ? p.b_dw[i] : 0.f;
    }
    for (int i = threadIdx.x; i < p.n_tile; i += BK_THREADS) sBpj[i] = p.b_pj ? p.b_pj[i] : 0.f;
    // The projection always runs all four K=16 slices of a K block.  In the half K block of an odd slab count the A
    // channels 32..63 hold zeros (or the ReLU6 outputs of an earlier K block) against zero-padded weights: exact zero
    // products, which leave the fp32 accumulators unchanged.
    for (int i = threadIdx.x; i < 2 * BK_A_TILE / 16; i += BK_THREADS) reinterpret_cast<uint4*>(sA)[i] = make_uint4(0, 0, 0, 0);
    fence_proxy_async();
    pdl_launch_dependents();
    __syncthreads();

    if (warp >= BK_DW_WARPS) {
        // ------------------------------------------------------------------ TMA producer
        regs_dec<BK_REGS_PRODUCER>();
        if (warp == BK_DW_WARPS && lane == 0) {
            if (!STREAM) {
                // weights are static: they may be fetched before the previous kernel of the stream has finished
                mbar_expect_tx(&bars->w_full, (uint32_t)(p.nslabs * (BK_WE_SLAB + BK_DW_BYTES) + p.nkb * p.n_tile * 128));
                for (int s = 0; s < p.nslabs; ++s) {
                    tma_load_2d(sWe + s * BK_WE_SLAB, &map_we, &bars->w_full, 0, s * BK_CB);
                    tma_load_2d(sDww + s * BK_DW_SLAB, &map_dw, &bars->w_full, s * BK_CB, 0);
                }
                for (int kb = 0; kb < p.nkb; ++kb)
                    tma_load_2d(sWp + kb * p.n_tile * 128, &map_wp, &bars->w_full, 0, kb * p.n_tile);
            }
            pdl_wait();               // the block input is complete from here on
            uint32_t we_n = 0, wp_n = 0, dw_n[2] = {0, 0};
            int it = 0;
            for (int t = blockIdx.x; t < p.num_tiles; t += gridDim.x, ++it) {
                const int tx = t % p.tiles_x, ty = (t / p.tiles_x) % p.tiles_y, n = t / (p.tiles_x * p.tiles_y);
                mbar_wait_backoff(&bars->x_empty, (it & 1) ^ 1);
                mbar_expect_tx(&bars->x_full, BK_X_TX);
                tma_load_4d(sX, &map_x, &bars->x_full, 0, tx * BK_T - 3, ty * BK_T - 3, n);
                if (STREAM) {
                    // the tile's weights in the order their consumers want them: per K block the expansion weights of its
                    // slabs (MMA issuer, slab order), their depthwise weights (the group that runs the slab), then the
                    // projection weights of the K block; two-slot rings keep the producer about one K block ahead
                    const int sw = (p.nslabs & 1) ? (it & 1) : 0;
                    for (int kb = 0; kb < p.nkb; ++kb) {
                        for (int s = 2 * kb; s < 2 * kb + 2 && s < p.nslabs; ++s) {
                            const uint32_t q = we_n & 1;
                            mbar_wait_backoff(&bars->we_empty[q], ((we_n >> 1) & 1) ^ 1);
                            mbar_expect_tx(&bars->we_full[q], BK_WE_SLAB);
                            tma_load_2d(sWe + q * BK_WE_SLAB, &map_we, &bars->we_full[q], 0, s * BK_CB);
                            ++we_n;
                        }
                        for (int s = 2 * kb; s < 2 * kb + 2 && s < p.nslabs; ++s) {
                            const int g = (s & 1) ^ sw;
                            const uint32_t q = dw_n[g] & 1;
                            mbar_wait_backoff(&bars->dw_empty[g][q], ((dw_n[g] >> 1) & 1) ^ 1);
                            mbar_expect_tx(&bars->dw_full[g][q], BK_DW_BYTES);
                            tma_load_2d(sDww + (g * 2 + q) * BK_DW_SLAB, &map_dw, &bars->dw_full[g][q], s * BK_CB, 0);
                            ++dw_n[g];
                        }
                        {
                            const uint32_t q = wp_n & 1;
                            mbar_wait_backoff(&bars->wp_empty[q], ((wp_n >> 1) & 1) ^ 1);
                            mbar_expect_tx(&bars->wp_full[q], (uint32_t)p.n_tile * 128);
                            tma_load_2d(sWp + q * p.wp_stage, &map_wp, &bars->wp_full[q], 0, kb * p.n_tile);
                            ++wp_n;
                        }
                    }
                }
            }
        }
    } else {
        // ------------------------------------------------------------------ depthwise warps (+ MMAs and both epilogues)
        regs_inc<BK_REGS_COMPUTE>();
        const int cp = threadIdx.x & 15;
        const int sub = (threadIdx.x >> 4) & 1;
        const bool mir = sub != 0;
        const int grp = warp >> 3;                         // 0: even slabs, 1: odd slabs
        const int gw = warp & 7;
        const int wq = warp & 3;                           // warp inside its warpgroup
        const int wg = warp >> 2;                          // projection: pixels 64*wg .. of the 256-pixel tile
        const int ewg = wg & 1;                            // expansion: haloed pixels 256*ewg .. of the group's slab
        const int blk = (gw << 1) | sub;
        const int by = blk >> 2, bx = blk & 3;
        const int oy = by * 4, ox = bx * 4;
        uint8_t* slab = sSlab + grp * BK_SLAB;
        const uint32_t a_wg = smem_u32(sA + (wg >> 1) * BK_A_TILE) + (wg & 1) * 8192;
        const __half2 zero2 = __floats2half2_rn(0.f, 0.f), six2 = __floats2half2_rn(6.f, 6.f);
        uint32_t ec = 0;                                   // slabs expanded by this group
        int it = 0;
        float pacc[NC][8];                                 // projection accumulators
        if (!STREAM) mbar_wait(&bars->w_full, 0);           // weights resident
        pdl_wait();                                        // the identity rows are read from global memory
        for (int t = blockIdx.x; t < p.num_tiles; t += gridDim.x, ++it) {
            const int tx = t % p.tiles_x, ty = (t / p.tiles_x) % p.tiles_y, n = t / (p.tiles_x * p.tiles_y);
            // Odd slab counts (Ce = 96: 3 slabs) leave one group idle in the last round of a tile; the groups therefore swap
            // roles on odd tiles (group 0 takes the odd slabs), so that over two tiles each group runs the same number of
            // slabs.
            const int vg = grp ^ ((p.nslabs & 1) ? (it & 1) : 0);      // which slab parity this group runs in this tile
            const int last_kb = (p.nslabs - 1 - vg) >> 1;               // this group's last K block with a slab (-1: none)
            if (last_kb < 0) {
                __syncwarp();
                if (lane == 0) mbar_arrive(&bars->x_empty);
            }
#pragma unroll
            for (int c = 0; c < NC; ++c)
#pragma unroll
                for (int i = 0; i < 8; ++i) pacc[c][i] = 0.f;
            // which of the thread's 8 haloed pixels (expansion rows (ewg * 4 + j) * 64 + frag_row(wq, lane, 0 / 1), j = 0..3)
            // lie inside the image: the same for every slab of the tile
            uint32_t in_img = 0;
#pragma unroll
            for (int j = 0; j < 4; ++j)
#pragma unroll
                for (int i = 0; i < 2; ++i) {
                    const int pi = (ewg * 4 + j) * 64 + frag_row(wq, lane, i);
                    const int yy = pi / BK_I, xx = pi - yy * BK_I;
                    const int gy = ty * BK_T - 3 + yy, gx = tx * BK_T - 3 + xx;
                    if (pi < BK_PIX && gy >= 0 && gy < p.H && gx >= 0 && gx < p.W) in_img |= 1u << (j * 2 + i);
                }
            for (int kb = 0; kb < p.nkb; ++kb) {
                const int s = 2 * kb + vg;
                const bool have = s < p.nslabs;
                __half2 acch[4][4];
                if (have) {
                    if (grp) asm volatile("bar.sync 2, 256;" ::: "memory");     // previous slab fully consumed
                    else asm volatile("bar.sync 1, 256;" ::: "memory");
                    // ---- expansion of slab s: this warpgroup's 256 haloed pixels x 32 channels, in two halves of 128
                    if (s == vg) mbar_wait(&bars->x_full, it & 1);
                    uint32_t b_base = smem_u32(sWe + s * BK_WE_SLAB);
                    const uint32_t we_i = (uint32_t)(it * p.nslabs + s);       // STREAM: position in the slab sequence
                    if (STREAM) {
                        mbar_wait(&bars->we_full[we_i & 1], (we_i >> 1) & 1);
                        b_base = smem_u32(sWe + (we_i & 1) * BK_WE_SLAB);
                    }
                    float be[2][2][2];
#pragma unroll
                    for (int i = 0; i < 2; ++i)
#pragma unroll
                        for (int c = 0; c < 2; ++c) {
                            const int ch = c * 16 + frag_col(lane, 2 * i);
                            be[i][c][0] = sBexp[s * BK_CB + ch];
                            be[i][c][1] = sBexp[s * BK_CB + ch + 1];
                        }
#pragma unroll
                    for (int hb = 0; hb < 2; ++hb) {
                        float eacc[2][2][8];                 // written by the first K=16 slice (scale-d = 0)
                        const uint32_t x_base = smem_u32(sX) + (ewg * 4 + hb * 2) * 8192;
                        wg_fence();
#pragma unroll
                        for (int b = 0; b < 2; ++b)
#pragma unroll
                            for (int k = 0; k < K16; ++k) wg_mma_n<2>(eacc[b], x_base + b * 8192 + k * 32, b_base + k * 32, k);
                        wg_commit();
                        wg_wait0();
                        // + bias in fp32, round to fp16, ReLU6 on the packed halves (clamping commutes with rounding),
                        // zero outside the image; chunk-major slab layout
#pragma unroll
                        for (int b = 0; b < 2; ++b)
#pragma unroll
                            for (int i = 0; i < 4; ++i) {
                                const int pi = (ewg * 4 + hb * 2 + b) * 64 + frag_row(wq, lane, i);
                                if (pi >= BK_PIX) continue;
                                const bool in = (in_img >> ((hb * 2 + b) * 2 + (i & 1))) & 1;
#pragma unroll
                                for (int c = 0; c < 2; ++c) {
                                    const int ch = c * 16 + frag_col(lane, i);
                                    __half2 h = zero2;
                                    if (in)
                                        h = __hmin2(__hmax2(__floats2half2_rn(eacc[b][c][2 * i] + be[i >> 1][c][0],
                                                                              eacc[b][c][2 * i + 1] + be[i >> 1][c][1]),
                                                            zero2),
                                                    six2);
                                    *reinterpret_cast<__half2*>(slab + (ch >> 3) * BK_CHUNK + pi * 16 + (ch & 7) * 2) = h;
                                }
                            }
                    }
                    __syncwarp();
                    if (STREAM && lane == 0) mbar_arrive(&bars->we_empty[we_i & 1]);
                    if (kb == last_kb && lane == 0) mbar_arrive(&bars->x_empty);   // X may be overwritten
                    ++ec;
                    if (grp) asm volatile("bar.sync 2, 256;" ::: "memory");     // slab complete
                    else asm volatile("bar.sync 1, 256;" ::: "memory");

                    // ---- depthwise 7x7 on the slab: packed fp16 (dw_inner.cuh), chunk-major slab addressing
                    const int ch = s * BK_CB + 2 * cp;
                    const __half2 bh = __float22half2_rn(*reinterpret_cast<const float2*>(sBdw + ch));
                    const __half2* tile_in = reinterpret_cast<const __half2*>(slab + (cp >> 2) * BK_CHUNK) + (cp & 3);
                    if (STREAM) {
                        // this slab's depthwise weights arrive through the group's ring (slot = slabs run by the group so far)
                        const uint32_t q = (ec - 1) & 1;
                        mbar_wait(&bars->dw_full[grp][q], ((ec - 1) >> 1) & 1);
                        dw_slab_hfma2<K, 4, BK_I, BK_CB, 4>(tile_in, reinterpret_cast<const __half2*>(sDww + (grp * 2 + q) * BK_DW_SLAB),
                                                            cp, mir, oy, ox, bh, acch);
                        __syncwarp();
                        if (lane == 0) mbar_arrive(&bars->dw_empty[grp][q]);
                    } else {
                        dw_slab_hfma2<K, 4, BK_I, BK_CB, 4>(tile_in, reinterpret_cast<const __half2*>(sDww + s * BK_DW_SLAB), cp, mir,
                                                            oy, ox, bh, acch);
                    }
                }
                // the single A buffer is free once every warpgroup's projection MMAs of the previous K block retired
                asm volatile("bar.sync 3, 512;" ::: "memory");
                if (have) {
                    dw_store_a<4>(sA, BK_A_TILE, acch, oy, ox, mir, (vg << 2) | (cp >> 2), cp);
                    fence_proxy_async();
                }
                asm volatile("bar.sync 3, 512;" ::: "memory");                  // A tile complete
                // ---- projection of K block kb
                const uint32_t wp_i = (uint32_t)(it * p.nkb + kb);
                uint32_t b_base = smem_u32(sWp + kb * p.n_tile * 128);
                if (STREAM) {
                    mbar_wait(&bars->wp_full[wp_i & 1], (wp_i >> 1) & 1);
                    b_base = smem_u32(sWp + (wp_i & 1) * p.wp_stage);
                }
                wg_fence();
#pragma unroll
                for (int k = 0; k < 4; ++k) wg_mma_n<NC>(pacc, a_wg + k * 32, b_base + k * 32);
                wg_commit();
                wg_wait0();
                if (STREAM) {
                    __syncwarp();
                    if (lane == 0) mbar_arrive(&bars->wp_empty[wp_i & 1]);
                }
            }
            // ---- final epilogue: accumulator row = pixel of M-tile wg / 2
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int row = (wg & 1) * 64 + frag_row(wq, lane, i);
                const int py = (wg >> 1) * 8 + (row >> 4), px = row & 15;
                const int gy = ty * BK_T + py, gx = tx * BK_T + px;
                if (gy >= p.H || gx >= p.W) continue;
                const size_t off = (((size_t)n * p.H + gy) * p.W + gx) * p.Co;
#pragma unroll
                for (int c = 0; c < NC; ++c) {
                    const int co = c * 16 + frag_col(lane, i);
                    if (co >= p.Co) continue;
                    float2 v = make_float2(pacc[c][2 * i] + sBpj[co], pacc[c][2 * i + 1] + sBpj[co + 1]);
                    if (p.residual) {
                        const float2 f = __half22float2(*reinterpret_cast<const __half2*>(p.residual + off + co));
                        v.x += f.x;
                        v.y += f.y;
                    }
                    *reinterpret_cast<__half2*>(p.out + off + co) = __float22half2_rn(v);
                }
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// One stride-2 inverted-residual block (k = 7, Cin <= 16, no identity) in ONE kernel: the same arithmetic as
// lp_pw1x1_f16 (ReLU6) -> lp_dwconv_f16 (k7, s2, ReLU6, packed fp16) -> lp_pw1x1_f16, without the 6x tensor in HBM.
// Per 16x8-pixel output tile (one 128-row projection M-tile pair) the CTA
//   * TMA-loads the haloed input X [21 rows][37 px][16 ch] at its real width: 777 rows of 32 B, 32B-swizzled, channels
//     beyond Cin and pixels outside the image zero-filled by the tensor map,
//   * per 32-channel slab: expands X on the tensor cores (14 x wgmma m64n32k16, one K=16 slice), + bias -> fp16 -> ReLU6,
//     zero outside the image, into a pixel-major [777 px][32 ch] slab with a 72-byte pixel pitch, then runs the packed
//     fp16 7x7 stride-2 depthwise of dw_inner.cuh on it (thread = channel pair x 4x4 output micro-block) and writes the
//     ReLU6'd results into the slab's 64B-swizzled A tile [128 px][32 ch],
//   * projects all slabs at once: warpgroup w runs output rows 4w..4w+3 (M = 64) over every K=16 slice in channel order,
//     4 slices per 64-channel K block like lp_pw1x1_f16 (the slices past Ce read zero A rows against zero weights),
//     fp32 accumulators, + bias, one rounding to fp16.
// Warp roles: two warpgroups, each expands and convolves its own slabs (s = wg, wg + 2, ...) with its own slab buffer;
// an odd last slab is shared (expansion by M-tile halves, depthwise on 4x2 micro-blocks, both in warpgroup 0's buffer),
// and named barrier, so one warpgroup's expansion epilogue overlaps the other's depthwise loop.  Thread 0 also issues
// the TMA loads: the next tile's X as soon as every warp has expanded its last slab of the current tile.
// Bank conflicts: the two half-warps of a warp convolve x-adjacent micro-blocks, i.e. read pixels 8 apart; with
// 72-byte pixels those are 144 words apart (= 16 mod 32 banks), so the 16 + 16 words of one LDS fall into 32 banks.
// HBM traffic: read N*H*W*Cin*2 (plus halo re-reads, L2 hits), write N*H/2*W/2*Co*2.
constexpr int S2_TW = 16, S2_TH = 8;                       // output tile
constexpr int S2_IW = 2 * S2_TW + 5, S2_IH = 2 * S2_TH + 5; // haloed input tile: 37 x 21
constexpr int S2_PIX = S2_IW * S2_IH;                       // 777 rows of X / pixels of a slab
constexpr int S2_X_BYTES = 14 * 64 * 32;                    // 14 M-tiles of 64 rows x 32 B (TMA fills the first 777 rows)
constexpr int S2_X_TX = S2_PIX * 32;
constexpr int S2_PP = 18;                                   // slab pixel pitch in half2 (72 B)
constexpr int S2_SLAB = (S2_PIX * S2_PP * 4 + 127) & ~127;  // 56064 B
constexpr int S2_WE_SLAB = 32 * 32;                         // expansion weights of a slab: 32 rows x 32 B
constexpr int S2_A_SLAB = 128 * 64;                         // A tile of a slab: 128 px x 64 B
constexpr int S2_THREADS = 256;

struct S2Bars {
    uint64_t w_full, x_full, x_empty;
};

struct S2Params {
    int N, H, W, Cin, Ce, Co, Hout, Wout, n_tile;
    int tiles_x, tiles_y, num_tiles;
    int nslabs, nkb;
    int off_we, off_a, off_wp, off_slab, off_dww, off_bias;
    const float* b_exp;               // [Ce]
    const float* b_dw;                // [Ce]
    const float* b_pj;                // packed, n_tile
    __half* out;                      // [N,H/2,W/2,Co]
};

// next tile's haloed input into sX, once every warp has expanded its last slab of tile `it`
__device__ __forceinline__ void s2_load_next_x(const CUtensorMap* map_x, S2Bars* bars, uint8_t* sX, const S2Params& p, int t2,
                                               int it) {
    if (t2 >= p.num_tiles) return;
    const int tx = t2 % p.tiles_x, ty = (t2 / p.tiles_x) % p.tiles_y, n = t2 / (p.tiles_x * p.tiles_y);
    mbar_wait(&bars->x_empty, it & 1);
    mbar_expect_tx(&bars->x_full, S2_X_TX);
    tma_load_4d(sX, map_x, &bars->x_full, 0, tx * 2 * S2_TW - 3, ty * 2 * S2_TH - 3, n);
}

// expansion of slab s into `slab` for haloed pixels of M-tiles 2 mp0 .. 2 mp1 - 1 (one warpgroup, two M-tiles per
// wgmma batch): + bias in fp32, round to fp16, ReLU6 (clamping commutes with rounding), zero outside the image
__device__ __forceinline__ void s2_expand(uint8_t* slab, const uint8_t* sX, const uint8_t* sWe, const float* sBexp, int s,
                                          int mp0, int mp1, uint32_t in_img, int wq, int lane) {
    const __half2 zero2 = __floats2half2_rn(0.f, 0.f), six2 = __floats2half2_rn(6.f, 6.f);
    float be[2][2][2];
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int c = 0; c < 2; ++c) {
            const int ch = c * 16 + frag_col(lane, 2 * i);
            be[i][c][0] = sBexp[s * BK_CB + ch];
            be[i][c][1] = sBexp[s * BK_CB + ch + 1];
        }
    const uint64_t bdesc = wg_desc_sw32(smem_u32(sWe + s * S2_WE_SLAB));
#pragma unroll 1
    for (int mp = mp0; mp < mp1; ++mp) {
        float eacc[2][2][8];
        wg_fence();
#pragma unroll
        for (int b = 0; b < 2; ++b) wg_mma_nd<2>(eacc[b], wg_desc_sw32(smem_u32(sX) + (mp * 2 + b) * 2048), bdesc, 0);
        wg_commit();
        wg_wait0();
#pragma unroll
        for (int b = 0; b < 2; ++b)
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int pi = (mp * 2 + b) * 64 + frag_row(wq, lane, i);
                if (pi >= S2_PIX) continue;
                const bool in = (in_img >> ((mp * 2 + b) * 2 + (i & 1))) & 1;
#pragma unroll
                for (int c = 0; c < 2; ++c) {
                    const int ch = c * 16 + frag_col(lane, i);
                    __half2 h = zero2;
                    if (in)
                        h = __hmin2(__hmax2(__floats2half2_rn(eacc[b][c][2 * i] + be[i >> 1][c][0],
                                                              eacc[b][c][2 * i + 1] + be[i >> 1][c][1]),
                                            zero2),
                                    six2);
                    *reinterpret_cast<__half2*>(slab + pi * (S2_PP * 4) + ch * 2) = h;
                }
            }
    }
}

// depthwise 7x7 stride 2 of slab s (dw_inner.cuh) for the thread's channel pair and 4-wide x BY-tall micro-block at
// (oy, ox) of the output tile, ReLU6, into the slab's 64B-swizzled A tile (row = pixel of the 16x8 tile)
template <int BY>
__device__ __forceinline__ void s2_depthwise(const uint8_t* slab, const uint8_t* sDww, const float* sBdw, uint8_t* sA, int s,
                                             int cp, int oy, int ox) {
    const __half2 zero2 = __floats2half2_rn(0.f, 0.f), six2 = __floats2half2_rn(6.f, 6.f);
    __half2 acch[BY][4];
    const __half2 bh = __float22half2_rn(*reinterpret_cast<const float2*>(sBdw + s * BK_CB + 2 * cp));
    dw_slab_hfma2<7, BY, S2_IW, BK_CB, S2_PP, 2>(reinterpret_cast<const __half2*>(slab) + cp,
                                                 reinterpret_cast<const __half2*>(sDww + s * BK_DW_SLAB), cp, false, oy, ox,
                                                 bh, acch);
    uint8_t* a_s = sA + s * S2_A_SLAB;
#pragma unroll
    for (int i = 0; i < BY; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int r = (oy + i) * S2_TW + ox + j;
            const __half2 v = __hmin2(__hmax2(acch[i][j], zero2), six2);
            *reinterpret_cast<__half2*>(a_s + r * 64 + (((cp >> 2) ^ ((r >> 1) & 3)) << 4) + ((cp & 3) << 2)) = v;
        }
}

// NC = n_tile / 16 projection chunks (one m64n(16 NC)k16 per K=16 slice)
template <int NC>
__global__ void __launch_bounds__(S2_THREADS, 1)
block_s2_kernel(const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_we,
                const __grid_constant__ CUtensorMap map_dw, const __grid_constant__ CUtensorMap map_wp,
                const __grid_constant__ S2Params p) {
    extern __shared__ __align__(1024) uint8_t smem[];
    uint8_t* sX = smem;
    uint8_t* sWe = smem + p.off_we;
    uint8_t* sA = smem + p.off_a;
    uint8_t* sWp = smem + p.off_wp;
    uint8_t* sDww = smem + p.off_dww;
    float* sBexp = reinterpret_cast<float*>(smem + p.off_bias);
    float* sBdw = sBexp + p.nslabs * 32;
    float* sBpj = sBdw + p.nslabs * 32;
    S2Bars* bars = reinterpret_cast<S2Bars*>(sBpj + 64);

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int wg = warp >> 2, wq = warp & 3;
    uint8_t* slab = smem + p.off_slab + wg * S2_SLAB;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&map_x);
        tma_prefetch_desc(&map_we);
        tma_prefetch_desc(&map_dw);
        tma_prefetch_desc(&map_wp);
        mbar_init(&bars->w_full, 1);
        mbar_init(&bars->x_full, 1);
        mbar_init(&bars->x_empty, S2_THREADS / 32);
        fence_barrier_init();
    }
    for (int i = threadIdx.x; i < p.nslabs * 32; i += S2_THREADS) {
        sBexp[i] = (i < p.Ce && p.b_exp) ? p.b_exp[i] : 0.f;
        sBdw[i] = (i < p.Ce && p.b_dw) ? p.b_dw[i] : 0.f;
    }
    for (int i = threadIdx.x; i < p.n_tile; i += S2_THREADS) sBpj[i] = p.b_pj ? p.b_pj[i] : 0.f;
    // A tiles of the slabs past the last one (the rest of the last K block) stay zero
    for (int i = p.nslabs * S2_A_SLAB / 16 + threadIdx.x; i < 2 * p.nkb * S2_A_SLAB / 16; i += S2_THREADS)
        reinterpret_cast<uint4*>(sA)[i] = make_uint4(0, 0, 0, 0);
    fence_proxy_async();
    pdl_launch_dependents();
    __syncthreads();

    if (threadIdx.x == 0) {
        // weights are static: they may be fetched before the previous kernel of the stream has finished
        mbar_expect_tx(&bars->w_full, (uint32_t)(p.nslabs * (S2_WE_SLAB + BK_DW_BYTES) + p.nkb * p.n_tile * 128));
        for (int s = 0; s < p.nslabs; ++s) {
            tma_load_2d(sWe + s * S2_WE_SLAB, &map_we, &bars->w_full, 0, s * BK_CB);
            tma_load_2d(sDww + s * BK_DW_SLAB, &map_dw, &bars->w_full, s * BK_CB, 0);
        }
        for (int kb = 0; kb < p.nkb; ++kb) tma_load_2d(sWp + kb * p.n_tile * 128, &map_wp, &bars->w_full, 0, kb * p.n_tile);
    }
    pdl_wait();                       // the block input is complete from here on (and the output no longer read)
    if (threadIdx.x == 0 && (int)blockIdx.x < p.num_tiles) {
        const int t = blockIdx.x;
        const int tx = t % p.tiles_x, ty = (t / p.tiles_x) % p.tiles_y, n = t / (p.tiles_x * p.tiles_y);
        mbar_expect_tx(&bars->x_full, S2_X_TX);
        tma_load_4d(sX, &map_x, &bars->x_full, 0, tx * 2 * S2_TW - 3, ty * 2 * S2_TH - 3, n);
    }
    mbar_wait(&bars->w_full, 0);

    const int cp = threadIdx.x & 15;
    const int blk = (wq << 1) | ((threadIdx.x >> 4) & 1);       // micro-block of the 4 x 2 grid of 4x4 blocks
    const int oy = (blk >> 2) * 4, ox = (blk & 3) * 4;
    const int nk16 = 4 * p.nkb;
    float pacc[NC][8];
    int it = 0;
    for (int t = blockIdx.x; t < p.num_tiles; t += gridDim.x, ++it) {
        const int tx = t % p.tiles_x, ty = (t / p.tiles_x) % p.tiles_y, n = t / (p.tiles_x * p.tiles_y);
        // which of the thread's 28 expansion rows (M-tile m, rows frag_row(wq, lane, 0 / 1)) lie inside the image
        uint32_t in_img = 0;
#pragma unroll
        for (int m = 0; m < 14; ++m)
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                const int pi = m * 64 + frag_row(wq, lane, i);
                const int yy = pi / S2_IW, xx = pi - yy * S2_IW;
                const int gy = ty * 2 * S2_TH - 3 + yy, gx = tx * 2 * S2_TW - 3 + xx;
                if (pi < S2_PIX && gy >= 0 && gy < p.H && gx >= 0 && gx < p.W) in_img |= 1u << (m * 2 + i);
            }
        mbar_wait(&bars->x_full, it & 1);
        // Slabs 0 .. nfull-1 alternate between the warpgroups; an odd last slab is split between both (expansion by
        // M-tile halves, depthwise on 4x2 micro-blocks), so that neither warpgroup idles for a whole slab.
        const int nfull = p.nslabs & ~1;
        for (int s = wg; s < nfull; s += 2) {
            asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory");   // the previous slab is fully consumed
            s2_expand(slab, sX, sWe, sBexp, s, 0, 7, in_img, wq, lane);
            const bool last = s + 2 >= nfull && nfull == p.nslabs;
            if (last) {
                __syncwarp();
                if (lane == 0) mbar_arrive(&bars->x_empty);                   // X may be overwritten
            }
            asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory");   // slab complete
            if (last && threadIdx.x == 0) s2_load_next_x(&map_x, bars, sX, p, t + gridDim.x, it);
            s2_depthwise<4>(slab, sDww, sBdw, sA, s, cp, oy, ox);
        }
        if (nfull < p.nslabs) {
            const int s = nfull;
            uint8_t* slab0 = smem + p.off_slab;
            asm volatile("bar.sync 3, 256;" ::: "memory");                  // warpgroup 0's slab buffer is free
            s2_expand(slab0, sX, sWe, sBexp, s, wg ? 4 : 0, wg ? 7 : 4, in_img, wq, lane);
            __syncwarp();
            if (lane == 0) mbar_arrive(&bars->x_empty);
            asm volatile("bar.sync 3, 256;" ::: "memory");                  // slab complete
            if (threadIdx.x == 0) s2_load_next_x(&map_x, bars, sX, p, t + gridDim.x, it);
            const int b16 = (wg << 3) | blk;                                // 16 micro-blocks of 4 x 2 rows
            s2_depthwise<2>(slab0, sDww, sBdw, sA, s, cp, (b16 >> 2) * 2, (b16 & 3) * 4);
        }
        fence_proxy_async();
        __syncthreads();                                                     // A complete
        // ---- projection: warpgroup wg = output rows 4 wg .. 4 wg + 3, every K=16 slice in channel order
        const uint32_t a_base = smem_u32(sA) + wg * 64 * 64;
        const uint32_t b_base = smem_u32(sWp);
        wg_fence();
        for (int k = 0; k < nk16; ++k)
            wg_mma_nd<NC>(pacc, wg_desc_sw64(a_base + (k >> 1) * S2_A_SLAB + (k & 1) * 32),
                          wg_desc_sw128(b_base + (k >> 2) * p.n_tile * 128 + (k & 3) * 32), k);
        wg_commit();
        wg_wait0();
        __syncthreads();                                                     // A may be overwritten
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int row = wg * 64 + frag_row(wq, lane, i);
            const int gy = ty * S2_TH + (row >> 4), gx = tx * S2_TW + (row & 15);
            if (gy >= p.Hout || gx >= p.Wout) continue;
            const size_t off = (((size_t)n * p.Hout + gy) * p.Wout + gx) * p.Co;
#pragma unroll
            for (int c = 0; c < NC; ++c) {
                const int co = c * 16 + frag_col(lane, i);
                if (co >= p.Co) continue;
                *reinterpret_cast<__half2*>(p.out + off + co) =
                    __float22half2_rn(make_float2(pacc[c][2 * i] + sBpj[co], pacc[c][2 * i + 1] + sBpj[co + 1]));
            }
        }
    }
}

static size_t s2_layout(S2Params& p) {
    size_t off = S2_X_BYTES;                                                  // 1024-aligned (28 KiB)
    p.off_we = (int)off;    off += ((size_t)p.nslabs * S2_WE_SLAB + 1023) & ~(size_t)1023;
    p.off_a = (int)off;     off += (size_t)2 * p.nkb * S2_A_SLAB;            // 8 KiB per slab, 1024-aligned
    p.off_wp = (int)off;    off += ((size_t)p.nkb * p.n_tile * 128 + 1023) & ~(size_t)1023;
    p.off_slab = (int)off;  off += 2 * S2_SLAB;
    p.off_dww = (int)off;   off += ((size_t)p.nslabs * BK_DW_SLAB + 127) & ~(size_t)127;
    p.off_bias = (int)off;  off += ((size_t)2 * p.nslabs * 32 + 64) * 4 + sizeof(S2Bars) + 64;
    return off + 1024;                                                        // alignment slack of the dynamic base
}

static size_t bk_layout(BkParams& p, int stream) {
    size_t off = BK_X_BYTES;
    const int n_we = stream ? 2 : p.nslabs, n_dw = stream ? 4 : p.nslabs;
    p.wp_stage = (p.n_tile * 128 + 1023) & ~1023;
    p.off_we = (int)off;                       off += (size_t)n_we * BK_WE_SLAB;             // 1024-aligned (4 KiB slabs)
    p.off_a = (int)off;                        off += 2 * BK_A_TILE;                          // 1024-aligned
    p.off_wp = (int)off;                       off += stream ? (size_t)2 * p.wp_stage : (((size_t)p.nkb * p.n_tile * 128 + 1023) & ~(size_t)1023);
    p.off_slab = (int)off;                     off += 2 * BK_SLAB;
    p.off_dww = (int)off;                      off += ((size_t)n_dw * BK_DW_SLAB + 127) & ~(size_t)127;
    p.off_bias = (int)off;                     off += (2 * BK_MAX_CE + 64) * 4 + sizeof(BkBars) + 64;
    return off + 1024;                         // alignment slack of the dynamic shared-memory base
}

}  // namespace lp

using namespace lp;

static int bk_shape_ok(int Cin, int Ce, int Co, BkParams* out, int* stream_out = nullptr) {
    if (Cin < 8 || Cin > 64 || Cin % 8 || Ce < 8 || Ce % 8 || Ce > BK_MAX_CE - BK_CB || Co < 8 || Co % 8 || Co > 64) return 0;
    BkParams p;
    memset(&p, 0, sizeof(p));
    p.Cin = Cin; p.Ce = Ce; p.Co = Co;
    p.n_tile = (Co + 15) / 16 * 16;
    p.nslabs = (Ce + BK_CB - 1) / BK_CB;
    p.nkb = (Ce + 63) / 64;
    p.k16 = (Cin + 15) / 16;
    int stream = 0;
    size_t need = bk_layout(p, 0);               // everything resident when it fits (no ring hand-overs)
    if (need > 232448) {                         // 227 KiB of dynamic shared memory per CTA on sm_90
        stream = 1;
        need = bk_layout(p, 1);
        if (need > 232448) return 0;
    }
    if (out) *out = p;
    if (stream_out) *stream_out = stream;
    return (int)need;
}

// 1 when lp_block_s1_f16 can run this block shape (shared-memory budget), else 0
extern "C" int lp_block_s1_supported(int Cin, int Ce, int Co) { return bk_shape_ok(Cin, Ce, Co, nullptr) > 0; }

extern "C" size_t lp_block_s1_wexp_elems(int Cin, int Ce) { return (size_t)((Ce + BK_CB - 1) / BK_CB) * BK_CB * 64; }

// w_exp [Ce][Cin] fp16 (BN folded) -> [nslabs*32][64] K-major rows (zero padded), what map_we loads
extern "C" int lp_block_s1_pack_wexp(const uint16_t* w, int Cin, int Ce, uint16_t* out) {
    LP_CHECK_ARG(w && out && Cin > 0 && Cin <= 64 && Ce > 0, "lp_block_s1_pack_wexp: bad args");
    const int rows = (Ce + BK_CB - 1) / BK_CB * BK_CB;
    for (int r = 0; r < rows; ++r)
        for (int k = 0; k < 64; ++k) out[(size_t)r * 64 + k] = (r < Ce && k < Cin) ? w[(size_t)r * Cin + k] : (uint16_t)0;
    return LP_OK;
}

// x [N,H,W,Cin] fp16 NHWC -> out [N,H,W,Co]: relu6(x We^T + be) -> dw7x7 (+bd, relu6) -> Wp (+bp) (+ x when identity)
extern "C" int lp_block_s1_f16(const void* x, const void* w_exp_packed, const float* b_exp, const void* w_dw,
                               const float* b_dw, const void* w_proj_packed, const float* b_proj_packed, int identity,
                               void* out, int N, int H, int W, int Cin, int Ce, int Co, lp_stream_t stream) {
    LP_CHECK_ARG(x && w_exp_packed && w_dw && w_proj_packed && out, "lp_block_s1_f16: null pointer");
    BkParams p;
    int stream_mode = 0;
    const int need = bk_shape_ok(Cin, Ce, Co, &p, &stream_mode);
    LP_CHECK_ARG(N > 0 && H > 0 && W > 0 && need > 0,
                 "lp_block_s1_f16: unsupported shape N=%d H=%d W=%d Cin=%d Ce=%d Co=%d (see lp_block_s1_supported)", N, H, W,
                 Cin, Ce, Co);
    LP_CHECK_ARG(!identity || Cin == Co, "lp_block_s1_f16: identity needs Cin == Co");
    if ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(out) | reinterpret_cast<uintptr_t>(w_proj_packed) |
         reinterpret_cast<uintptr_t>(w_exp_packed) | reinterpret_cast<uintptr_t>(w_dw)) & 15) {
        set_error("lp_block_s1_f16: pointers must be 16-byte aligned");
        return LP_ERR_ALIGN;
    }
    p.N = N; p.H = H; p.W = W;
    p.tiles_x = (W + BK_T - 1) / BK_T;
    p.tiles_y = (H + BK_T - 1) / BK_T;
    p.num_tiles = p.tiles_x * p.tiles_y * N;
    p.b_exp = b_exp;
    p.b_dw = b_dw;
    p.b_pj = b_proj_packed;
    p.residual = identity ? reinterpret_cast<const __half*>(x) : nullptr;
    p.out = reinterpret_cast<__half*>(out);
    CUtensorMap mx, mwe, mdw, mwp;
    {
        uint64_t dims[4] = {(uint64_t)Cin, (uint64_t)W, (uint64_t)H, (uint64_t)N};
        uint64_t strides[3] = {(uint64_t)Cin * 2, (uint64_t)W * Cin * 2, (uint64_t)H * W * Cin * 2};
        uint32_t box[4] = {64u, (uint32_t)BK_I, (uint32_t)BK_I, 1u};
        int rc = make_tmap(&mx, x, 4, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B);
        if (rc) return rc;
        uint64_t d2[2] = {64u, (uint64_t)p.nslabs * BK_CB};
        uint64_t s2[1] = {128u};
        uint32_t b2[2] = {64u, (uint32_t)BK_CB};
        rc = make_tmap(&mwe, w_exp_packed, 2, d2, s2, b2, CU_TENSOR_MAP_SWIZZLE_128B);
        if (rc) return rc;
        uint64_t d3[2] = {(uint64_t)Ce, 49u};
        uint64_t s3[1] = {(uint64_t)Ce * 2};
        uint32_t b3[2] = {(uint32_t)BK_CB, 49u};
        rc = make_tmap(&mdw, w_dw, 2, d3, s3, b3, CU_TENSOR_MAP_SWIZZLE_NONE);
        if (rc) return rc;
        uint64_t d4[2] = {64u, (uint64_t)p.nkb * p.n_tile};
        uint64_t s4[1] = {128u};
        uint32_t b4[2] = {64u, (uint32_t)p.n_tile};
        rc = make_tmap(&mwp, w_proj_packed, 2, d4, s4, b4, CU_TENSOR_MAP_SWIZZLE_128B);
        if (rc) return rc;
    }
    const int grid = p.num_tiles < num_sms() ? p.num_tiles : num_sms();
    const int nc = p.n_tile / 16;
    using Kern = void (*)(const CUtensorMap, const CUtensorMap, const CUtensorMap, const CUtensorMap, const BkParams);
    // [layout][k16 - 1][nc - 1]
    static const Kern kernels[2][4][4] = {
        {{block_s1_kernel<0, 1, 1>, block_s1_kernel<0, 1, 2>, block_s1_kernel<0, 1, 3>, block_s1_kernel<0, 1, 4>},
         {block_s1_kernel<0, 2, 1>, block_s1_kernel<0, 2, 2>, block_s1_kernel<0, 2, 3>, block_s1_kernel<0, 2, 4>},
         {block_s1_kernel<0, 3, 1>, block_s1_kernel<0, 3, 2>, block_s1_kernel<0, 3, 3>, block_s1_kernel<0, 3, 4>},
         {block_s1_kernel<0, 4, 1>, block_s1_kernel<0, 4, 2>, block_s1_kernel<0, 4, 3>, block_s1_kernel<0, 4, 4>}},
        {{block_s1_kernel<1, 1, 1>, block_s1_kernel<1, 1, 2>, block_s1_kernel<1, 1, 3>, block_s1_kernel<1, 1, 4>},
         {block_s1_kernel<1, 2, 1>, block_s1_kernel<1, 2, 2>, block_s1_kernel<1, 2, 3>, block_s1_kernel<1, 2, 4>},
         {block_s1_kernel<1, 3, 1>, block_s1_kernel<1, 3, 2>, block_s1_kernel<1, 3, 3>, block_s1_kernel<1, 3, 4>},
         {block_s1_kernel<1, 4, 1>, block_s1_kernel<1, 4, 2>, block_s1_kernel<1, 4, 3>, block_s1_kernel<1, 4, 4>}},
    };
    const Kern k = kernels[stream_mode][p.k16 - 1][nc - 1];
    cudaError_t e = cudaFuncSetAttribute((const void*)k, cudaFuncAttributeMaxDynamicSharedMemorySize, need);
    if (e != cudaSuccess) return cuda_fail(e, "cudaFuncSetAttribute(block_s1)");
    e = launch_pdl(k, dim3(grid), dim3(BK_THREADS), (size_t)need, (cudaStream_t)stream, mx, mwe, mdw, mwp, p);
    if (e != cudaSuccess) return cuda_fail(e, "launch block_s1_kernel");
    LP_LAUNCH_CHECK("block_s1_kernel");
    return LP_OK;
}

static int s2_shape_ok(int Cin, int Ce, int Co, S2Params* out) {
    if (Cin < 8 || Cin > 16 || Cin % 8 || Ce < 8 || Ce % 8 || Co < 8 || Co % 8 || Co > 64) return 0;
    S2Params p;
    memset(&p, 0, sizeof(p));
    p.Cin = Cin; p.Ce = Ce; p.Co = Co;
    p.n_tile = (Co + 15) / 16 * 16;
    p.nslabs = (Ce + BK_CB - 1) / BK_CB;
    p.nkb = (Ce + 63) / 64;
    const size_t need = s2_layout(p);
    if (need > 232448) return 0;                 // 227 KiB of dynamic shared memory per CTA on sm_90
    if (out) *out = p;
    return (int)need;
}

// 1 when lp_block_s2_f16 can run this block shape (Cin <= 16, Co <= 64, shared-memory budget on Ce), else 0
extern "C" int lp_block_s2_supported(int Cin, int Ce, int Co) { return s2_shape_ok(Cin, Ce, Co, nullptr) > 0; }

// x [N,H,W,Cin] fp16 NHWC -> out [N,H/2,W/2,Co]: relu6(x We^T + be) -> dw7x7 stride 2 (+bd, relu6) -> Wp (+bp)
extern "C" int lp_block_s2_f16(const void* x, const void* w_exp_packed, const float* b_exp, const void* w_dw,
                               const float* b_dw, const void* w_proj_packed, const float* b_proj_packed, void* out, int N,
                               int H, int W, int Cin, int Ce, int Co, lp_stream_t stream) {
    LP_CHECK_ARG(x && w_exp_packed && w_dw && w_proj_packed && out, "lp_block_s2_f16: null pointer");
    S2Params p;
    const int need = s2_shape_ok(Cin, Ce, Co, &p);
    LP_CHECK_ARG(N > 0 && H > 0 && W > 0 && H % 2 == 0 && W % 2 == 0 && need > 0,
                 "lp_block_s2_f16: unsupported shape N=%d H=%d W=%d Cin=%d Ce=%d Co=%d (even H, W; see "
                 "lp_block_s2_supported)", N, H, W, Cin, Ce, Co);
    if ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(out) | reinterpret_cast<uintptr_t>(w_proj_packed) |
         reinterpret_cast<uintptr_t>(w_exp_packed) | reinterpret_cast<uintptr_t>(w_dw)) & 15) {
        set_error("lp_block_s2_f16: pointers must be 16-byte aligned");
        return LP_ERR_ALIGN;
    }
    p.N = N; p.H = H; p.W = W;
    p.Hout = H / 2; p.Wout = W / 2;
    p.tiles_x = (p.Wout + S2_TW - 1) / S2_TW;
    p.tiles_y = (p.Hout + S2_TH - 1) / S2_TH;
    p.num_tiles = p.tiles_x * p.tiles_y * N;
    p.b_exp = b_exp;
    p.b_dw = b_dw;
    p.b_pj = b_proj_packed;
    p.out = reinterpret_cast<__half*>(out);
    CUtensorMap mx, mwe, mdw, mwp;
    {
        uint64_t dims[4] = {(uint64_t)Cin, (uint64_t)W, (uint64_t)H, (uint64_t)N};
        uint64_t strides[3] = {(uint64_t)Cin * 2, (uint64_t)W * Cin * 2, (uint64_t)H * W * Cin * 2};
        uint32_t box[4] = {16u, (uint32_t)S2_IW, (uint32_t)S2_IH, 1u};
        int rc = make_tmap(&mx, x, 4, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_32B);
        if (rc) return rc;
        // the K = 16 slice (columns 0..15) of lp_block_s1_pack_wexp's [nslabs*32][64] rows
        uint64_t d2[2] = {64u, (uint64_t)p.nslabs * BK_CB};
        uint64_t s2[1] = {128u};
        uint32_t b2[2] = {16u, (uint32_t)BK_CB};
        rc = make_tmap(&mwe, w_exp_packed, 2, d2, s2, b2, CU_TENSOR_MAP_SWIZZLE_32B);
        if (rc) return rc;
        uint64_t d3[2] = {(uint64_t)Ce, 49u};
        uint64_t s3[1] = {(uint64_t)Ce * 2};
        uint32_t b3[2] = {(uint32_t)BK_CB, 49u};
        rc = make_tmap(&mdw, w_dw, 2, d3, s3, b3, CU_TENSOR_MAP_SWIZZLE_NONE);
        if (rc) return rc;
        uint64_t d4[2] = {64u, (uint64_t)p.nkb * p.n_tile};
        uint64_t s4[1] = {128u};
        uint32_t b4[2] = {64u, (uint32_t)p.n_tile};
        rc = make_tmap(&mwp, w_proj_packed, 2, d4, s4, b4, CU_TENSOR_MAP_SWIZZLE_128B);
        if (rc) return rc;
    }
    const int grid = p.num_tiles < num_sms() ? p.num_tiles : num_sms();
    using Kern = void (*)(const CUtensorMap, const CUtensorMap, const CUtensorMap, const CUtensorMap, const S2Params);
    static const Kern kernels[4] = {block_s2_kernel<1>, block_s2_kernel<2>, block_s2_kernel<3>, block_s2_kernel<4>};
    const Kern k = kernels[p.n_tile / 16 - 1];
    cudaError_t e = cudaFuncSetAttribute((const void*)k, cudaFuncAttributeMaxDynamicSharedMemorySize, need);
    if (e != cudaSuccess) return cuda_fail(e, "cudaFuncSetAttribute(block_s2)");
    e = launch_pdl(k, dim3(grid), dim3(S2_THREADS), (size_t)need, (cudaStream_t)stream, mx, mwe, mdw, mwp, p);
    if (e != cudaSuccess) return cuda_fail(e, "launch block_s2_kernel");
    LP_LAUNCH_CHECK("block_s2_kernel");
    return LP_OK;
}
