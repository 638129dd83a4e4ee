// wgmma tensor-core contraction kernel for the fusion deconv and the unfused heads of LitePose on sm_90a.
// The 1x1 convolutions run their own kernel (pw_gemm.cu).
//
// One persistent, warp-specialised kernel covers the two spatial contractions of the network
// (reference lib/models/pose_mobilenet.py:102-154):
//   MODE_DECONV fusion deconv level: 4 sub-pixel phases, each a K = 4*(Cr+Cw) contraction, both branches,
//               folded-BN bias + ReLU, written interleaved into the 2x up-sampled NHWC output
//   MODE_HEAD   head pair:  out_nchw_f32 = A1 W1^T + A2 W2^T
//
// Structure per CTA (384 threads, 1 CTA/SM, grid = min(#tiles, #SMs)):
//   warp 0 lane 0 : TMA producer  (cp.async.bulk.tensor -> 128B-swizzled smem ring)
//   warps 4..11   : two consumer warpgroups, one per 64-row half of the 128-row tile: wgmma m64n16k16 from the ring
//                   into fp32 register accumulators (up to 256 columns), then the epilogue straight from the
//                   accumulator fragments (direct stores).  The producer runs up to a ring ahead, so the next tile's
//                   loads overlap the epilogue.
// A "step" is one 128-row x 64-channel activation tile (one TMA box; spatially shifted boxes with hardware
// zero fill implement the deconv taps and all image borders) multiplied against 1..4 weight sub-tiles.
#include "common.cuh"

namespace lp {

constexpr int BM = 128;
constexpr int BK = 64;
constexpr int A_BYTES = BM * BK * 2;    // 16 KiB
constexpr int B_BYTES = 256 * BK * 2;   // 32 KiB
constexpr int STAGES = 4;
constexpr int MAX_STEPS = 48;
constexpr int GEMM_THREADS = 384;   // warpgroup 0: TMA (warp 0), warpgroups 1, 2: MMA + epilogue
constexpr int CONS_WARPS = 8;
constexpr int ACC_CHUNKS = 16;      // 256 accumulator columns per tile
constexpr int MAX_BIAS = 1024;

enum { MODE_DECONV = 1, MODE_HEAD = 2 };

struct Step {
    int16_t kc;       // channel offset of this 64-wide K block inside its source tensor
    int8_t dx, dy;    // spatial shift of the activation box (deconv taps)
    uint8_t map;      // activation source (0/1)
    uint8_t nb;       // weight sub-tiles multiplied against this activation tile (1..4)
    uint8_t k16;      // number of K=16 MMAs that carry data in this block (1..4)
    uint8_t pad;
    uint8_t acc[4];   // accumulator index per sub-tile
    uint16_t bt0;     // first weight sub-tile index (rows bt*n_tile of the packed weight matrix)
    uint16_t pad2;
};

struct GemmParams {
    int num_tiles;
    int n_chunks;
    int n_tile;        // MMA N (multiple of 16, <= 256)
    int num_steps;
    int total_bt;      // weight sub-tiles per chunk
    int N;             // Co
    int act;
    int H, W, TH, TW, tiles_x, tiles_y;
    const float* bias;       // packed, n_chunks*n_tile (may be null)
    void* out;
    Step steps[MAX_STEPS];
};

struct __align__(8) GemmBarriers {
    uint64_t full[STAGES];
    uint64_t empty[STAGES];
};

constexpr size_t GEMM_SMEM = 1024 /*align slack*/ + (size_t)STAGES * (A_BYTES + B_BYTES) + MAX_BIAS * 4 + 256;

template <int MODE>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap mapA0, const __grid_constant__ CUtensorMap mapA1,
               const __grid_constant__ CUtensorMap mapB, const __grid_constant__ GemmParams p) {
    extern __shared__ __align__(1024) uint8_t smem[];
    uint8_t* sA = smem;
    uint8_t* sB = smem + STAGES * A_BYTES;
    float* sBias = reinterpret_cast<float*>(smem + STAGES * (A_BYTES + B_BYTES));
    GemmBarriers* bars = reinterpret_cast<GemmBarriers*>(sBias + MAX_BIAS);

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;

    if (warp == 0 && lane == 0) {
        tma_prefetch_desc(&mapA0);
        tma_prefetch_desc(&mapA1);
        tma_prefetch_desc(&mapB);
        for (int i = 0; i < STAGES; ++i) {
            mbar_init(&bars->full[i], 1);
            mbar_init(&bars->empty[i], CONS_WARPS);
        }
        fence_barrier_init();
    }
    {
        const int nb = p.n_chunks * p.n_tile;
        for (int i = threadIdx.x; i < nb && i < MAX_BIAS; i += GEMM_THREADS) sBias[i] = p.bias ? p.bias[i] : 0.f;
    }
    pdl_launch_dependents();      // the next kernel may start its own prologue
    __syncthreads();
    pdl_wait();                   // activations written by the previous kernel are complete and visible from here on

    // Work distribution: item t -> (m-tile t / n_chunks, chunk t %% n_chunks), strided over the grid.
    if (warp == 0) {
        // ------------------------------------------------------------ TMA producer
        if (lane == 0) {
            uint32_t stage = 0, phase = 0;
            for (int t = blockIdx.x; t < p.num_tiles; t += gridDim.x) {
                const int chunk = t % p.n_chunks;
                const int mt = t / p.n_chunks;
                const int tx = mt % p.tiles_x;
                const int ty = (mt / p.tiles_x) % p.tiles_y;
                const int n = mt / (p.tiles_x * p.tiles_y);
                for (int s = 0; s < p.num_steps; ++s) {
                    const Step& st = p.steps[s];
                    mbar_wait_backoff(&bars->empty[stage], phase ^ 1);
                    const uint32_t bytes = A_BYTES + (uint32_t)st.nb * p.n_tile * (BK * 2);
                    mbar_expect_tx(&bars->full[stage], bytes);
                    tma_load_4d(sA + stage * A_BYTES, st.map ? &mapA1 : &mapA0, &bars->full[stage], st.kc,
                                tx * p.TW + st.dx, ty * p.TH + st.dy, n);
                    uint8_t* b_dst = sB + stage * B_BYTES;
                    for (int j = 0; j < st.nb; ++j) {
                        tma_load_2d(b_dst + j * p.n_tile * (BK * 2), &mapB, &bars->full[stage], 0,
                                    (chunk * p.total_bt + st.bt0 + j) * p.n_tile);
                    }
                    if (++stage == STAGES) { stage = 0; phase ^= 1; }
                }
            }
        }
    } else if (warp >= 4) {
        // ------------------------------------------------------------ consumer warpgroups: MMA + epilogue
        const int wg = (warp >> 2) - 1;            // 64-row half of the tile
        const int wq = warp & 3;
        const int nch = p.n_tile >> 4;
        uint32_t stage = 0, phase = 0;
        for (int t = blockIdx.x; t < p.num_tiles; t += gridDim.x) {
            const int mt = t / p.n_chunks;
            float acc[ACC_CHUNKS][8];
#pragma unroll
            for (int c = 0; c < ACC_CHUNKS; ++c)
#pragma unroll
                for (int i = 0; i < 8; ++i) acc[c][i] = 0.f;
            for (int s = 0; s < p.num_steps; ++s) {
                const Step& st = p.steps[s];
                mbar_wait(&bars->full[stage], phase);
                const uint32_t a_base = smem_u32(sA + stage * A_BYTES) + wg * 8192;
                const uint32_t b_base = smem_u32(sB + stage * B_BYTES);
                wg_fence();
                for (int j = 0; j < st.nb; ++j) {
                    const uint32_t bj = b_base + j * p.n_tile * (BK * 2);
                    for (int k = 0; k < st.k16; ++k)
                        wg_mma_chunks<ACC_CHUNKS>(acc, st.acc[j] * nch, nch, a_base + k * 32, bj + k * 32);
                }
                wg_commit();
                wg_wait0();
                __syncwarp();
                if (lane == 0) mbar_arrive(&bars->empty[stage]);
                if (++stage == STAGES) { stage = 0; phase ^= 1; }
            }
            const int rbase = wg * 64;
            const int tx = mt % p.tiles_x;
            const int ty = (mt / p.tiles_x) % p.tiles_y;
            const int n = mt / (p.tiles_x * p.tiles_y);
            const int Co = p.N;
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int row = rbase + frag_row(wq, lane, i);
                const int ly = row / p.TW, lx = row % p.TW;
                const int y = ty * p.TH + ly, x = tx * p.TW + lx;
                if (y >= p.H || x >= p.W) continue;
                if (MODE == MODE_DECONV) {
                    __half* out = reinterpret_cast<__half*>(p.out);
#pragma unroll
                    for (int c = 0; c < ACC_CHUNKS; ++c) {
                        if (c < 4 * nch) {
                            const int ph = c / nch;                       // sub-pixel phase = accumulator index
                            const int co = (c - ph * nch) * 16 + frag_col(lane, i);
                            if (co < Co) {
                                const int a = ph >> 1, b = ph & 1;
                                __half* op = out + ((((long long)n * 2 * p.H + 2 * y + a) * (2 * p.W)) + 2 * x + b) * Co + co;
                                *reinterpret_cast<__half2*>(op) =
                                    __floats2half2_rn(fmaxf(acc[c][2 * i] + sBias[co], 0.f),
                                                      fmaxf(acc[c][2 * i + 1] + sBias[co + 1], 0.f));
                            }
                        }
                    }
                } else {  // MODE_HEAD: NCHW, fp32 (act == 1) or fp16 (act == 0)
                    const long long plane = (long long)p.H * p.W;
                    const long long off = (long long)n * Co * plane + (long long)y * p.W + x;
                    float* op32 = reinterpret_cast<float*>(p.out) + off;
                    __half* op16 = reinterpret_cast<__half*>(p.out) + off;
#pragma unroll
                    for (int c = 0; c < ACC_CHUNKS; ++c) {
                        if (c < nch) {
                            const int co = c * 16 + frag_col(lane, i);
#pragma unroll
                            for (int e = 0; e < 2; ++e) {
                                if (co + e < Co) {
                                    if (p.act) op32[(long long)(co + e) * plane] = acc[c][2 * i + e];
                                    else op16[(long long)(co + e) * plane] = __float2half_rn(acc[c][2 * i + e]);
                                }
                            }
                        }
                    }
                }
            }
        }
    }
}

// ------------------------------------------------------------------ host side
static inline int round_up(int a, int b) { return (a + b - 1) / b * b; }

static int set_smem_attr_once(const void* fn) {
    // cudaFuncSetAttribute is per-device state; cheap enough to set on every call
    cudaError_t e = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)GEMM_SMEM);
    if (e != cudaSuccess) return cuda_fail(e, "cudaFuncSetAttribute(gemm_tc)");
    return LP_OK;
}

static void pick_spatial_tile(int H, int W, int* TH, int* TW) {
    int best = -1, bw = 32;
    const int cands[3] = {32, 16, 8};
    for (int i = 0; i < 3; ++i) {
        const int tw = cands[i], th = BM / tw;
        const int cover = round_up(W, tw) * round_up(H, th);
        if (best < 0 || cover < best) { best = cover; bw = tw; }
    }
    *TW = bw;
    *TH = BM / bw;
}

template <int MODE>
static int launch_gemm(const CUtensorMap& a0, const CUtensorMap& a1, const CUtensorMap& b, const GemmParams& p,
                       cudaStream_t stream) {
    int rc = set_smem_attr_once((const void*)gemm_tc_kernel<MODE>);
    if (rc) return rc;
    const int grid = p.num_tiles < num_sms() ? p.num_tiles : num_sms();
    if (grid < 1) return LP_OK;
    cudaError_t le = launch_pdl(gemm_tc_kernel<MODE>, dim3(grid), dim3(GEMM_THREADS), GEMM_SMEM, stream, a0, a1, b, p);
    if (le != cudaSuccess) return cuda_fail(le, "launch gemm_tc_kernel");
    LP_LAUNCH_CHECK("gemm_tc_kernel");
    return LP_OK;
}

}  // namespace lp

using namespace lp;

// ------------------------------------------------------------------ fusion deconv
// Two kernels share one packed-weight buffer: [tiled-kernel weights | row-kernel weights (when the channels qualify)].
// Wide maps run the row-streaming kernel (deconv_rows.cu), the others the tiled MODE_DECONV kernel above.
namespace lp {
bool deconv_rows_channels_ok(int Cr, int Cw, int Co);
bool deconv_rows_shape_ok(int W);
size_t deconv_rows_packed_elems(int Cr, int Cw, int Co);
void deconv_rows_pack(const uint16_t* wr, const uint16_t* ww, int Cr, int Cw, int Co, uint16_t* wp);
int launch_deconv_rows(const void* refined, const void* raw, const void* w_rows, const float* bias_packed, void* out, int N,
                       int H, int W, int Cr, int Cw, int Co, cudaStream_t stream);
}  // namespace lp

static int deconv_ntile(int Co) { return round_up(Co, 16); }

// enumerate steps; optionally emit packed weights
static int deconv_program(int Cr, int Cw, int Co, Step* steps, int* total_bt, const uint16_t* wr, const uint16_t* ww,
                          uint16_t* wp) {
    const int nt = deconv_ntile(Co);
    int s = 0, bt = 0;
    for (int br = 0; br < 2; ++br) {
        const int C = br ? Cw : Cr;
        const uint16_t* w = br ? ww : wr;
        for (int kb = 0; kb * BK < C; ++kb) {
            const int kv = (C - kb * BK) < BK ? (C - kb * BK) : BK;
            for (int di = -1; di <= 1; ++di)
                for (int dj = -1; dj <= 1; ++dj) {
                    if (s >= MAX_STEPS) return -1;
                    Step st;
                    memset(&st, 0, sizeof(st));
                    st.kc = (int16_t)(kb * BK);
                    st.dx = (int8_t)dj;
                    st.dy = (int8_t)di;
                    st.map = (uint8_t)br;
                    st.k16 = (uint8_t)((kv + 15) / 16);
                    st.bt0 = (uint16_t)bt;
                    int nb = 0;
                    for (int a = 0; a < 2; ++a) {
                        int ki;
                        if (a == 0) { if (di == 0) ki = 1; else if (di == -1) ki = 3; else continue; }
                        else        { if (di == 0) ki = 2; else if (di == 1) ki = 0; else continue; }
                        for (int b = 0; b < 2; ++b) {
                            int kj;
                            if (b == 0) { if (dj == 0) kj = 1; else if (dj == -1) kj = 3; else continue; }
                            else        { if (dj == 0) kj = 2; else if (dj == 1) kj = 0; else continue; }
                            st.acc[nb] = (uint8_t)(a * 2 + b);
                            if (wp) {
                                uint16_t* dst = wp + (size_t)(bt + nb) * nt * BK;
                                for (int co = 0; co < nt; ++co)
                                    for (int kk = 0; kk < BK; ++kk) {
                                        const int ci = kb * BK + kk;
                                        dst[(size_t)co * BK + kk] =
                                            (co < Co && ci < C) ? w[(((size_t)ci * Co + co) * 4 + ki) * 4 + kj] : (uint16_t)0;
                                    }
                            }
                            ++nb;
                        }
                    }
                    st.nb = (uint8_t)nb;
                    bt += nb;
                    if (steps) steps[s] = st;
                    ++s;
                }
        }
    }
    *total_bt = bt;
    return s;
}

extern "C" size_t lp_deconv_packed_elems(int Cr, int Cw, int Co) {
    int bt = 0;
    if (deconv_program(Cr, Cw, Co, nullptr, &bt, nullptr, nullptr, nullptr) < 0) return 0;
    return (size_t)bt * deconv_ntile(Co) * BK + deconv_rows_packed_elems(Cr, Cw, Co);
}
extern "C" size_t lp_deconv_packed_bias_elems(int Co) { return (size_t)deconv_ntile(Co); }
extern "C" int lp_deconv_pack(const uint16_t* wr, const uint16_t* ww, const float* bias, int Cr, int Cw, int Co,
                              uint16_t* wp, float* bp) {
    // Cw == 0: single branch (no raw deconv); deconv_program and dr_pack never read w_raw then
    LP_CHECK_ARG(wr && (ww || Cw == 0) && wp && bp, "lp_deconv_pack: null pointer");
    LP_CHECK_ARG(Cr % 8 == 0 && Cw % 8 == 0 && Co % 8 == 0 && Co <= 64, "lp_deconv_pack: bad channels %d %d %d", Cr, Cw, Co);
    int bt = 0;
    LP_CHECK_ARG(deconv_program(Cr, Cw, Co, nullptr, &bt, wr, ww, wp) > 0, "lp_deconv_pack: too many K blocks");
    if (deconv_rows_channels_ok(Cr, Cw, Co)) deconv_rows_pack(wr, ww, Cr, Cw, Co, wp + (size_t)bt * deconv_ntile(Co) * BK);
    for (int i = 0; i < deconv_ntile(Co); ++i) bp[i] = (bias && i < Co) ? bias[i] : 0.f;
    return LP_OK;
}

extern "C" int lp_fusion_deconv_f16(const void* refined, const void* raw, const void* w_packed, const float* bias_packed,
                                    void* out, int N, int H, int W, int Cr, int Cw, int Co, lp_stream_t stream) {
    LP_CHECK_ARG(refined && (raw || Cw == 0) && w_packed && out, "lp_fusion_deconv_f16: null pointer");
    LP_CHECK_ARG(N > 0 && H > 0 && W > 0 && Cr % 8 == 0 && Cw % 8 == 0 && Co % 8 == 0 && Co >= 8 && Co <= 64,
                 "lp_fusion_deconv_f16: bad shape N=%d H=%d W=%d Cr=%d Cw=%d Co=%d (Co<=64)", N, H, W, Cr, Cw, Co);
    GemmParams p;
    memset(&p, 0, sizeof(p));
    p.n_chunks = 1;
    p.n_tile = deconv_ntile(Co);
    p.num_steps = deconv_program(Cr, Cw, Co, p.steps, &p.total_bt, nullptr, nullptr, nullptr);
    LP_CHECK_ARG(p.num_steps > 0, "lp_fusion_deconv_f16: too many K blocks");
    if ((reinterpret_cast<uintptr_t>(refined) | reinterpret_cast<uintptr_t>(raw) | reinterpret_cast<uintptr_t>(out) |
         reinterpret_cast<uintptr_t>(w_packed)) & 15) {
        set_error("lp_fusion_deconv_f16: pointers must be 16-byte aligned");
        return LP_ERR_ALIGN;
    }
    if (deconv_rows_channels_ok(Cr, Cw, Co) && deconv_rows_shape_ok(W)) {
        const uint16_t* w_rows = reinterpret_cast<const uint16_t*>(w_packed) + (size_t)p.total_bt * p.n_tile * BK;
        return launch_deconv_rows(refined, raw, w_rows, bias_packed, out, N, H, W, Cr, Cw, Co, (cudaStream_t)stream);
    }
    pick_spatial_tile(H, W, &p.TH, &p.TW);
    p.tiles_x = (W + p.TW - 1) / p.TW;
    p.tiles_y = (H + p.TH - 1) / p.TH;
    p.num_tiles = p.tiles_x * p.tiles_y * N;
    p.H = H;
    p.W = W;
    p.N = Co;
    p.act = LP_ACT_RELU;
    p.bias = bias_packed;
    p.out = out;
    CUtensorMap m0, m1, mb;
    int rc = make_tmap_nhwc(&m0, refined, N, H, W, Cr, BK, p.TW, p.TH, CU_TENSOR_MAP_SWIZZLE_128B);
    if (rc) return rc;
    if (Cw > 0) {
        rc = make_tmap_nhwc(&m1, raw, N, H, W, Cw, BK, p.TW, p.TH, CU_TENSOR_MAP_SWIZZLE_128B);
        if (rc) return rc;
    } else {
        m1 = m0;      // single branch: no step selects map 1
    }
    rc = make_tmap_rows64(&mb, w_packed, p.total_bt * p.n_tile, BK, p.n_tile, CU_TENSOR_MAP_SWIZZLE_128B);
    if (rc) return rc;
    return launch_gemm<MODE_DECONV>(m0, m1, mb, p, (cudaStream_t)stream);
}

// ------------------------------------------------------------------ heads
extern "C" size_t lp_head_packed_elems(int C1, int C2, int Co) {
    return (size_t)((C1 + BK - 1) / BK + (C2 + BK - 1) / BK) * round_up(Co, 16) * BK;
}
extern "C" int lp_head_pack(const uint16_t* w1, const uint16_t* w2, int C1, int C2, int Co, uint16_t* wp) {
    LP_CHECK_ARG(w1 && (w2 || C2 == 0) && wp && C1 > 0 && C2 >= 0 && Co > 0, "lp_head_pack: bad args");
    const int nt = round_up(Co, 16);
    int bt = 0;
    for (int br = 0; br < 2; ++br) {
        const int C = br ? C2 : C1;
        const uint16_t* w = br ? w2 : w1;
        for (int kb = 0; kb * BK < C; ++kb, ++bt)
            for (int co = 0; co < nt; ++co)
                for (int kk = 0; kk < BK; ++kk) {
                    const int ci = kb * BK + kk;
                    wp[((size_t)bt * nt + co) * BK + kk] = (co < Co && ci < C) ? w[(size_t)co * C + ci] : (uint16_t)0;
                }
    }
    return LP_OK;
}

extern "C" int lp_head_pw_dual_f16(const void* a1, const void* a2, const void* w_packed, void* out_nchw, int out_fp32,
                                   int N, int H, int W, int C1, int C2, int Co, lp_stream_t stream) {
    LP_CHECK_ARG(a1 && (a2 || C2 == 0) && w_packed && out_nchw, "lp_head_pw_dual_f16: null pointer");
    LP_CHECK_ARG(N > 0 && H > 0 && W > 0 && C1 % 8 == 0 && C2 % 8 == 0 && C2 >= 0 && Co > 0 && Co <= 256,
                 "lp_head_pw_dual_f16: bad shape N=%d H=%d W=%d C1=%d C2=%d Co=%d", N, H, W, C1, C2, Co);
    GemmParams p;
    memset(&p, 0, sizeof(p));
    p.n_chunks = 1;
    p.n_tile = round_up(Co, 16);
    int s = 0;
    for (int br = 0; br < 2; ++br) {
        const int C = br ? C2 : C1;
        for (int kb = 0; kb * BK < C; ++kb, ++s) {
            LP_CHECK_ARG(s < MAX_STEPS, "lp_head_pw_dual_f16: too many K blocks");
            Step& st = p.steps[s];
            st.kc = (int16_t)(kb * BK);
            st.map = (uint8_t)br;
            st.nb = 1;
            const int kv = (C - kb * BK) < BK ? (C - kb * BK) : BK;
            st.k16 = (uint8_t)((kv + 15) / 16);
            st.bt0 = (uint16_t)s;
        }
    }
    p.num_steps = s;
    p.total_bt = s;
    p.TW = 32;
    p.TH = 4;
    if (W < 32) pick_spatial_tile(H, W, &p.TH, &p.TW);
    p.tiles_x = (W + p.TW - 1) / p.TW;
    p.tiles_y = (H + p.TH - 1) / p.TH;
    p.num_tiles = p.tiles_x * p.tiles_y * N;
    p.H = H;
    p.W = W;
    p.N = Co;
    p.act = out_fp32 ? 1 : 0;   // MODE_HEAD reuses `act` as the output-dtype flag
    p.out = out_nchw;
    CUtensorMap m0, m1, mb;
    int rc = make_tmap_nhwc(&m0, a1, N, H, W, C1, BK, p.TW, p.TH, CU_TENSOR_MAP_SWIZZLE_128B);
    if (rc) return rc;
    if (C2 > 0) {
        rc = make_tmap_nhwc(&m1, a2, N, H, W, C2, BK, p.TW, p.TH, CU_TENSOR_MAP_SWIZZLE_128B);
        if (rc) return rc;
    } else {
        m1 = m0;      // single branch: no step selects map 1
    }
    rc = make_tmap_rows64(&mb, w_packed, p.total_bt * p.n_tile, BK, p.n_tile, CU_TENSOR_MAP_SWIZZLE_128B);
    if (rc) return rc;
    return launch_gemm<MODE_HEAD>(m0, m1, mb, p, (cudaStream_t)stream);
}
