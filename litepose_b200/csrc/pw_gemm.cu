// Pointwise (1x1) convolution on sm_90a: out[M,N] = act(A[M,K] W^T + b) (+ residual), fp16 in/out, fp32 accumulation
// (reference lib/models/layers/layers.py:95-108: InvBottleneck inv/point_conv, stem 1x1).
//
// Every 1x1 layer of the network has K <= 192 and N <= 720, so it does at most ~110 FLOP per byte moved: the kernel is
// bound by HBM bandwidth and is built to keep loads and stores in flight, not to maximise MMA rate.
//
// pw_gemm_kernel<NC> (384 threads, 1 CTA/SM, persistent):
//   warps 0, 1 (lane 0) : TMA producers, one per consumer warpgroup, each running its warpgroup's A ring up to nst
//                         stages ahead
//   warps 4..11         : two consumer warpgroups.  Each owns its own stream of 64-row tiles, its own A ring and
//                         mbarriers and TWO output staging slots, so one warpgroup's epilogue and TMA store run while
//                         the other's MMAs run, and a tile's store drains while the next tile is computed.
// Each K=16 slice is ONE straight-line wgmma m64n(16 NC)k16 (NC = n_tile / 16, 1..10); the first slice of a tile
// overwrites the accumulators (scale-d = 0).  Every K block runs all four slices: past K, the A columns are TMA zero
// fill and the packed weights are zero, so those products are exact zeros that leave the fp32 accumulators unchanged,
// and no slice count depends on a run-time value (which makes ptxas fence and serialise the wgmma issue).  Weight layout (lp_pw1x1_pack): N <= 160 is one chunk of round_up(N, 16)
// rows, wider N is cut into 128-row chunks; per chunk, K blocks of [n_tile][64] fp16 rows, zero padded.
// Resident-weights mode: a CTA keeps one N chunk for its life and loads that chunk's weights once; the CTAs sharing a
// chunk split its m-tiles, so the CTAs of the different chunks walk the same rows together and A is read from HBM once
// (the other chunks' reads hit L2).  Shapes whose weights do not fit stream a weight block with every A block.
#include "common.cuh"

namespace lp {

namespace {

constexpr int PW_BM = 64;                       // rows per tile (one warpgroup)
constexpr int PW_BK = 64;                       // K block: one 128-byte swizzle row of fp16
constexpr int PW_A_BYTES = PW_BM * PW_BK * 2;   // 8 KiB
constexpr int PW_OUT_SUB = PW_BM * 64 * 2;      // one 64-row x 64-column fp16 output box (128B-swizzled), 8 KiB
constexpr int PW_MAX_STAGES = 16;               // A ring stages per warpgroup
constexpr int PW_MIN_RES_STAGES = 4;            // resident-weights mode needs this many A stages per warpgroup
constexpr int PW_MAX_KB = 48;
constexpr int PW_MAX_BIAS = 1024;
constexpr int PW_THREADS = 384;
constexpr int PW_SMEM = 227 * 1024;             // the sm_90 per-block maximum; the host carves it per launch
constexpr int PW_FIXED = 1024 /*align slack*/ + PW_MAX_BIAS * 4 + 1024 /*barriers*/;

struct PwParams {
    int M, N, act;
    int n_chunks, n_tile;   // N chunks of n_tile = 16 NC weight rows
    int kb;                 // K blocks of 64
    int m_tiles;            // 64-row tiles
    int resident;           // one chunk's weights stay in shared memory, only A streams
    int nst;                // A ring stages per warpgroup
    int stage_bytes;        // A block (+ its weight block when not resident)
    int slot_bytes;         // one output staging slot: ceil(n_tile / 64) boxes
    int bres_bytes;         // resident weights
    const float* bias;      // packed, n_chunks * n_tile (may be null)
    const __half* residual; // [M, N] (may be null)
};

struct __align__(8) PwBars {
    uint64_t full[2][PW_MAX_STAGES];
    uint64_t empty[2][PW_MAX_STAGES];
    uint64_t res_full[2][2];
    uint64_t bres_full;
};
static_assert(sizeof(PwBars) <= 1024, "barrier area");

// Named barrier of the 128 threads of consumer warpgroup wg (id 0 is __syncthreads).
__device__ __forceinline__ void wg_sync(int wg) { asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory"); }

// Tile sequence of warpgroup wg of this CTA (the same for its producer and its consumers).
struct PwWork {
    int t0, step, end;
    __device__ PwWork(const PwParams& p, int wg) {
        if (p.resident) {   // item = m-tile of the CTA's chunk
            t0 = (int)(blockIdx.x / p.n_chunks) * 2 + wg;
            step = 2 * (int)(gridDim.x / p.n_chunks);
            end = p.m_tiles;
        } else {            // item = (m-tile, chunk)
            t0 = (int)blockIdx.x * 2 + wg;
            step = 2 * (int)gridDim.x;
            end = p.m_tiles * p.n_chunks;
        }
    }
};
__device__ __forceinline__ void pw_item(const PwParams& p, int t, int* mt, int* chunk) {
    if (p.resident) {
        *mt = t;
        *chunk = (int)blockIdx.x % p.n_chunks;
    } else {
        *mt = t / p.n_chunks;
        *chunk = t % p.n_chunks;
    }
}

// Epilogue of one 64-row tile, columns [0, ncols) of its chunk: acc + bias -> activation (-> + residual, read from the
// slot) -> fp16 into the 128B-swizzled staging slot.  The activation and the residual switch are template arguments so
// that the per-element code has no branches.
template <int NC, int ACT, bool RES>
__device__ __forceinline__ void pw_epilogue(const float (&acc)[NC][8], uint8_t* sSlot, const float* bias, int ncols,
                                            int wq, int lane) {
#pragma unroll
    for (int c = 0; c < NC; ++c) {
        if (c * 16 < ncols) {
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int row = frag_row(wq, lane, i);
                const int col = c * 16 + frag_col(lane, i);
                const float2 b = *reinterpret_cast<const float2*>(bias + col);
                float v0 = acc[c][2 * i] + b.x, v1 = acc[c][2 * i + 1] + b.y;
                v0 = act_apply(v0, ACT);
                v1 = act_apply(v1, ACT);
                __half2* d = reinterpret_cast<__half2*>(sSlot + (col >> 6) * PW_OUT_SUB + row * 128 +
                                                        ((((col & 63) >> 3) ^ (row & 7)) << 4) + (col & 7) * 2);
                if (RES) {
                    const float2 f = __half22float2(*d);
                    v0 += f.x;
                    v1 += f.y;
                }
                *d = __floats2half2_rn(v0, v1);
            }
        }
    }
}

template <int NC>
__global__ void __launch_bounds__(PW_THREADS, 1)
pw_gemm_kernel(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapB,
               const __grid_constant__ CUtensorMap mapOut, const __grid_constant__ CUtensorMap mapRes,
               const __grid_constant__ PwParams p) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    // [4 output slots: wg 0 slot 0, 1, wg 1 slot 0, 1][resident weights][A ring wg 0][A ring wg 1] ... [bias][barriers]
    uint8_t* sOut = smem;
    uint8_t* sW = sOut + 4 * p.slot_bytes;
    uint8_t* sRing = sW + p.bres_bytes;
    float* sBias = reinterpret_cast<float*>(smem + (PW_SMEM - PW_FIXED));
    PwBars* bars = reinterpret_cast<PwBars*>(sBias + PW_MAX_BIAS);

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&mapA);
        tma_prefetch_desc(&mapB);
        tma_prefetch_desc(&mapOut);
        if (p.residual) tma_prefetch_desc(&mapRes);
        for (int g = 0; g < 2; ++g) {
            for (int i = 0; i < PW_MAX_STAGES; ++i) {
                mbar_init(&bars->full[g][i], 1);
                mbar_init(&bars->empty[g][i], 4);   // one arrival per consumer warp
            }
            mbar_init(&bars->res_full[g][0], 1);
            mbar_init(&bars->res_full[g][1], 1);
        }
        mbar_init(&bars->bres_full, 1);
        fence_barrier_init();
    }
    for (int i = threadIdx.x; i < p.n_chunks * p.n_tile; i += PW_THREADS) sBias[i] = p.bias ? p.bias[i] : 0.f;
    pdl_launch_dependents();      // the next kernel may start its own prologue
    __syncthreads();
    pdl_wait();                   // activations written by the previous kernel are complete and visible from here on

    const int b_bytes = p.n_tile * (PW_BK * 2);   // one K block of one chunk's weights
    if (warp < 2) {
        // ------------------------------------------------------------ TMA producer of warpgroup `warp`
        if (lane == 0) {
            const int wg = warp;
            uint8_t* ring = sRing + wg * p.nst * p.stage_bytes;
            if (p.resident && wg == 0) {
                const int chunk = (int)blockIdx.x % p.n_chunks;
                mbar_expect_tx(&bars->bres_full, (uint32_t)(p.kb * b_bytes));
                for (int s = 0; s < p.kb; ++s)
                    tma_load_2d(sW + s * b_bytes, &mapB, &bars->bres_full, 0, (chunk * p.kb + s) * p.n_tile);
            }
            const PwWork w(p, wg);
            const uint32_t bytes = PW_A_BYTES + (p.resident ? 0 : b_bytes);
            uint32_t stage = 0, phase = 0;
            for (int t = w.t0; t < w.end; t += w.step) {
                int mt, chunk;
                pw_item(p, t, &mt, &chunk);
                for (int s = 0; s < p.kb; ++s) {
                    mbar_wait_backoff(&bars->empty[wg][stage], phase ^ 1);
                    mbar_expect_tx(&bars->full[wg][stage], bytes);
                    uint8_t* dst = ring + stage * p.stage_bytes;
                    tma_load_2d(dst, &mapA, &bars->full[wg][stage], s * PW_BK, mt * PW_BM);
                    if (!p.resident)
                        tma_load_2d(dst + PW_A_BYTES, &mapB, &bars->full[wg][stage], 0, (chunk * p.kb + s) * p.n_tile);
                    if (++stage == (uint32_t)p.nst) { stage = 0; phase ^= 1; }
                }
            }
        }
    } else if (warp >= 4) {
        // ------------------------------------------------------------ consumer warpgroups: MMA + epilogue
        const int wg = (warp >> 2) - 1;
        const int wq = warp & 3;
        const bool issuer = (threadIdx.x & 127) == 0;   // residual loads and output stores of this warpgroup
        uint8_t* ring = sRing + wg * p.nst * p.stage_bytes;
        const PwWork w(p, wg);
        uint32_t stage = 0, phase = 0;
        if (p.resident) mbar_wait(&bars->bres_full, 0);
        float acc[NC][8];
        int it = 0;
        for (int t = w.t0; t < w.end; t += w.step, ++it) {
            int mt, chunk;
            pw_item(p, t, &mt, &chunk);
            const int ncols = min(p.n_tile, p.N - chunk * p.n_tile);   // valid columns of this chunk
            const int nsub = (ncols + 63) >> 6;
            const int slot = it & 1;
            uint8_t* sSlot = sOut + (2 * wg + slot) * p.slot_bytes;
            // The slot is free once the store of tile it - 2 has read it; tile it - 1's store may still be draining.
            // The residual tile is fetched into the slot while this tile's MMAs run.
            if (issuer) asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");
            if (p.residual && issuer) {
                mbar_expect_tx(&bars->res_full[wg][slot], nsub * PW_OUT_SUB);
                for (int g = 0; g < nsub; ++g)
                    tma_load_2d(sSlot + g * PW_OUT_SUB, &mapRes, &bars->res_full[wg][slot], chunk * p.n_tile + g * 64,
                                mt * PW_BM);
            }
            uint32_t prev = 0;
            for (int s = 0; s < p.kb; ++s) {
                mbar_wait(&bars->full[wg][stage], phase);
                const uint32_t a_base = smem_u32(ring + stage * p.stage_bytes);
                const uint32_t b_base = p.resident ? smem_u32(sW + s * b_bytes) : a_base + PW_A_BYTES;
                wg_fence();
#pragma unroll
                for (int k = 0; k < 4; ++k) wg_mma_n<NC>(acc, a_base + k * 32, b_base + k * 32, s | k);
                wg_commit();
                if (s > 0) {   // K block s - 1 has retired: release its stage
                    wg_wait1();
                    __syncwarp();
                    if (lane == 0) mbar_arrive(&bars->empty[wg][prev]);
                }
                prev = stage;
                if (++stage == (uint32_t)p.nst) { stage = 0; phase ^= 1; }
            }
            wg_wait0();
            __syncwarp();
            if (lane == 0) mbar_arrive(&bars->empty[wg][prev]);

            // Epilogue: bias, activation, residual into the 128B-swizzled slot; TMA stores clip rows/columns at M/N.
            const float* bias = sBias + chunk * p.n_tile;
            if (p.residual) {
                mbar_wait(&bars->res_full[wg][slot], (it >> 1) & 1);
                switch (p.act) {
                    case LP_ACT_RELU: pw_epilogue<NC, LP_ACT_RELU, true>(acc, sSlot, bias, ncols, wq, lane); break;
                    case LP_ACT_RELU6: pw_epilogue<NC, LP_ACT_RELU6, true>(acc, sSlot, bias, ncols, wq, lane); break;
                    default: pw_epilogue<NC, LP_ACT_NONE, true>(acc, sSlot, bias, ncols, wq, lane); break;
                }
            } else {
                wg_sync(wg);   // the issuer has seen the slot free
                switch (p.act) {
                    case LP_ACT_RELU: pw_epilogue<NC, LP_ACT_RELU, false>(acc, sSlot, bias, ncols, wq, lane); break;
                    case LP_ACT_RELU6: pw_epilogue<NC, LP_ACT_RELU6, false>(acc, sSlot, bias, ncols, wq, lane); break;
                    default: pw_epilogue<NC, LP_ACT_NONE, false>(acc, sSlot, bias, ncols, wq, lane); break;
                }
            }
            fence_proxy_async();
            wg_sync(wg);
            if (issuer) {
                for (int g = 0; g < nsub; ++g) {
                    asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(
                                     reinterpret_cast<uint64_t>(&mapOut)),
                                 "r"(smem_u32(sSlot + g * PW_OUT_SUB)), "r"(chunk * p.n_tile + g * 64), "r"(mt * PW_BM)
                                 : "memory");
                }
                asm volatile("cp.async.bulk.commit_group;" ::: "memory");
            }
        }
        if (issuer) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
    }
}

template <int NC>
int launch_pw_nc(const CUtensorMap& ma, const CUtensorMap& mb, const CUtensorMap& mo, const CUtensorMap& mr,
                 const PwParams& p, int grid, cudaStream_t stream) {
    auto kern = pw_gemm_kernel<NC>;
    cudaError_t e = cudaFuncSetAttribute((const void*)kern, cudaFuncAttributeMaxDynamicSharedMemorySize, PW_SMEM);
    if (e != cudaSuccess) return cuda_fail(e, "cudaFuncSetAttribute(pw_gemm_kernel)");
    cudaError_t le = launch_pdl(kern, dim3(grid), dim3(PW_THREADS), (size_t)PW_SMEM, stream, ma, mb, mo, mr, p);
    if (le != cudaSuccess) return cuda_fail(le, "launch pw_gemm_kernel");
    LP_LAUNCH_CHECK("pw_gemm_kernel");
    return LP_OK;
}

int launch_pw(const CUtensorMap& ma, const CUtensorMap& mb, const CUtensorMap& mo, const CUtensorMap& mr,
              const PwParams& p, int grid, cudaStream_t stream) {
    switch (p.n_tile / 16) {
        case 1: return launch_pw_nc<1>(ma, mb, mo, mr, p, grid, stream);
        case 2: return launch_pw_nc<2>(ma, mb, mo, mr, p, grid, stream);
        case 3: return launch_pw_nc<3>(ma, mb, mo, mr, p, grid, stream);
        case 4: return launch_pw_nc<4>(ma, mb, mo, mr, p, grid, stream);
        case 5: return launch_pw_nc<5>(ma, mb, mo, mr, p, grid, stream);
        case 6: return launch_pw_nc<6>(ma, mb, mo, mr, p, grid, stream);
        case 7: return launch_pw_nc<7>(ma, mb, mo, mr, p, grid, stream);
        case 8: return launch_pw_nc<8>(ma, mb, mo, mr, p, grid, stream);
        case 9: return launch_pw_nc<9>(ma, mb, mo, mr, p, grid, stream);
        default: return launch_pw_nc<10>(ma, mb, mo, mr, p, grid, stream);
    }
}

// N <= 160 (every projection, incl. the fused depthwise+projection kernel's single-chunk layout): one chunk of
// round_up(N,16) MMA columns.  Wider layers (the 6x expansions) are cut into 128-column chunks: a multiple of the
// 64-column TMA store box, so stores of neighbouring chunks never overlap.
void pw_tiling(int N, int* n_chunks, int* n_tile) {
    const int np = (N + 15) / 16 * 16;
    if (np <= 160) {
        *n_chunks = 1;
        *n_tile = np;
        return;
    }
    *n_chunks = (np + 127) / 128;
    *n_tile = 128;
}

}  // namespace

}  // namespace lp

using namespace lp;

extern "C" size_t lp_pw1x1_packed_elems(int K, int N) {
    int nc, nt;
    pw_tiling(N, &nc, &nt);
    return (size_t)nc * ((K + PW_BK - 1) / PW_BK) * nt * PW_BK;
}
extern "C" size_t lp_pw1x1_packed_bias_elems(int N) {
    int nc, nt;
    pw_tiling(N, &nc, &nt);
    return (size_t)nc * nt;
}
extern "C" int lp_pw1x1_pack(const uint16_t* w, const float* bias, int K, int N, uint16_t* wp, float* bp) {
    LP_CHECK_ARG(w && wp && bp && K > 0 && N > 0, "lp_pw1x1_pack: null pointer or bad shape K=%d N=%d", K, N);
    int nc, nt;
    pw_tiling(N, &nc, &nt);
    const int kb = (K + PW_BK - 1) / PW_BK;
    for (int c = 0; c < nc; ++c)
        for (int s = 0; s < kb; ++s)
            for (int r = 0; r < nt; ++r) {
                const int n = c * nt + r;
                uint16_t* dst = wp + (((size_t)c * kb + s) * nt + r) * PW_BK;
                for (int kk = 0; kk < PW_BK; ++kk) {
                    const int k = s * PW_BK + kk;
                    dst[kk] = (n < N && k < K) ? w[(size_t)n * K + k] : (uint16_t)0;
                }
            }
    for (int i = 0; i < nc * nt; ++i) bp[i] = (bias && i < N) ? bias[i] : 0.f;
    return LP_OK;
}

extern "C" int lp_pw1x1_f16(const void* a, const void* w_packed, const float* bias_packed, const void* residual,
                            void* out, int M, int K, int N, int act, lp_stream_t stream) {
    LP_CHECK_ARG(a && w_packed && out, "lp_pw1x1_f16: null pointer");
    LP_CHECK_ARG(M > 0 && K >= 8 && N >= 8 && K % 8 == 0 && N % 8 == 0,
                 "lp_pw1x1_f16: need M>0, K%%8==0, N%%8==0 (M=%d K=%d N=%d)", M, K, N);
    LP_CHECK_ARG(act >= LP_ACT_NONE && act <= LP_ACT_RELU6, "lp_pw1x1_f16: bad act %d", act);
    if ((reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(out) | reinterpret_cast<uintptr_t>(w_packed) |
         reinterpret_cast<uintptr_t>(residual)) & 15) {
        set_error("lp_pw1x1_f16: pointers must be 16-byte aligned");
        return LP_ERR_ALIGN;
    }
    PwParams p;
    memset(&p, 0, sizeof(p));
    pw_tiling(N, &p.n_chunks, &p.n_tile);
    p.kb = (K + PW_BK - 1) / PW_BK;
    LP_CHECK_ARG(p.kb <= PW_MAX_KB && p.n_chunks * p.n_tile <= PW_MAX_BIAS, "lp_pw1x1_f16: K=%d or N=%d too large", K, N);
    p.m_tiles = (M + PW_BM - 1) / PW_BM;
    p.M = M;
    p.N = N;
    p.act = act;
    p.bias = bias_packed;
    p.residual = reinterpret_cast<const __half*>(residual);

    // Shared memory: 4 output slots, then either one chunk's weights and 2 x nst A stages, or 2 x nst (A + weight
    // block) stages.  Resident when the weights leave room for PW_MIN_RES_STAGES A stages per warpgroup.
    const int sms = num_sms();
    const int b_bytes = p.n_tile * PW_BK * 2;
    p.slot_bytes = (p.n_tile + 63) / 64 * PW_OUT_SUB;
    const int avail = PW_SMEM - PW_FIXED - 4 * p.slot_bytes;
    const int bres = p.kb * b_bytes;
    const int nst_res = (avail - bres) / (2 * PW_A_BYTES);
    if (nst_res >= PW_MIN_RES_STAGES && p.n_chunks <= sms) {
        p.resident = 1;
        p.bres_bytes = bres;
        p.stage_bytes = PW_A_BYTES;
        p.nst = nst_res;
    } else {
        p.stage_bytes = PW_A_BYTES + b_bytes;
        p.nst = avail / (2 * p.stage_bytes);
    }
    if (p.nst > PW_MAX_STAGES) p.nst = PW_MAX_STAGES;
    LP_CHECK_ARG(p.nst >= 2, "lp_pw1x1_f16: N=%d leaves no room for the A ring", N);

    int grid;
    if (p.resident) {
        // a multiple of n_chunks CTAs, at most one per SM, and no more warpgroups per chunk than m-tiles
        int cpc = sms / p.n_chunks;
        if (cpc > (p.m_tiles + 1) / 2) cpc = (p.m_tiles + 1) / 2;
        grid = cpc * p.n_chunks;
    } else {
        const int items = p.m_tiles * p.n_chunks;
        grid = (items + 1) / 2 < sms ? (items + 1) / 2 : sms;
    }

    CUtensorMap ma, mb, mo, mr;
    {
        uint64_t dims[2] = {(uint64_t)K, (uint64_t)M};
        uint64_t strides[1] = {(uint64_t)K * 2};
        uint32_t box[2] = {(uint32_t)PW_BK, (uint32_t)PW_BM};
        int rc = make_tmap(&ma, a, 2, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B);
        if (rc) return rc;
    }
    {
        int rc = make_tmap_rows64(&mb, w_packed, p.n_chunks * p.kb * p.n_tile, PW_BK, p.n_tile, CU_TENSOR_MAP_SWIZZLE_128B);
        if (rc) return rc;
    }
    {
        uint64_t dims[2] = {(uint64_t)N, (uint64_t)M};
        uint64_t strides[1] = {(uint64_t)N * 2};
        uint32_t box[2] = {64u, (uint32_t)PW_BM};
        int rc = make_tmap(&mo, out, 2, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B);
        if (rc) return rc;
        mr = mo;
        if (residual) {
            rc = make_tmap(&mr, residual, 2, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B);
            if (rc) return rc;
        }
    }
    return launch_pw(ma, mb, mo, mr, p, grid, (cudaStream_t)stream);
}
