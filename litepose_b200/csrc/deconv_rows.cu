// Fusion-deconv level as a row-streaming wgmma kernel (large maps: the last, HBM-heaviest levels).
//
// Reference: lib/models/pose_mobilenet.py:102-135,146-150 - ReLU(BN(ConvT(refined) + ConvT(raw))), k4 s2 p1.
// Sub-pixel form: output pixel (2y+a, 2x+b) is a contraction over the 2x2 input neighbourhood selected by (a, b) and
// over the concatenated channels [refined | raw]; the 4 phases share the 3x3 input neighbourhood of (y, x).
//
// One persistent CTA walks DOWN consecutive image rows of a 128-pixel wide strip, so every input row is fetched once
// per strip (plus one halo row at the start of a run) instead of 9 shifted boxes per tile:
//   warps 0..3    : producers - 16-byte cp.async copies of one input row (130 px: 128 + x halo) of BOTH branches into a
//                   128B-swizzled K-major slot [px][refined ch | raw ch | 0], zero filled outside the image
//   warps 4..11   : two consumer warpgroups, 64 strip pixels each.  MMA: the 9 (dy, dx) taps are 9 operand views of three
//                   resident row slots: the A descriptor start address moves by (dx+1) pixel rows (128 B) inside the
//                   slot (the 128B swizzle is a function of the absolute shared-memory address, so a row-shifted view
//                   stays consistent); the weights of all 16 (tap, phase) sub-tiles stay resident in shared memory;
//                   the 4 phase accumulators (fp32, <= 256 columns) live in registers.  Epilogue from the accumulator
//                   fragments: bias + ReLU, fp16, staged in shared memory so that each of the two output rows of the
//                   tile leaves as fully contiguous 16-byte stores
#include "common.cuh"

namespace lp {

constexpr int DR_TW = 128;                 // strip width (MMA M)
constexpr int DR_SLOT_PX = DR_TW + 2;      // with x halo
constexpr int DR_SLOT_BYTES = 17 * 1024;   // 130 px x 128 B rounded up to the swizzle period
constexpr int DR_NS = 5;                   // row slots in the ring
constexpr int DR_PROD_WARPS = 4;           // warps 0..3 producers, warps 4..11 MMA + epilogue
constexpr int DR_EPI_WARP0 = DR_PROD_WARPS;
constexpr int DR_EPI_THREADS = 256;
constexpr int DR_THREADS = (DR_EPI_WARP0 + 8) * 32;
constexpr int DR_MAX_NT = 64;

// The k4 s2 p1 transposed convolution in sub-pixel form: phase (a, b) of output pixel (2y+a, 2x+b) sums, over the taps
// (dy, dx) with dy in {0, a ? +1 : -1}, dx in {0, b ? +1 : -1}, input pixel (y+dy, x+dx) times kernel element
// (ki, kj), ki = dy == 0 ? 1 + a : (a ? 0 : 3), kj likewise.  Accumulator columns are ordered (0,0) (0,1) (1,1) (1,0)
// so that the phases sharing a tap are neighbours wherever possible: 10 MMA groups (N = 1, 2 or 4 phases) per K=16
// slice instead of 16.  Group g multiplies the slot view shifted by (DY, DX) with LEN consecutive weight sub-tiles
// starting at BT into accumulator positions POS .. POS+LEN-1.
constexpr int DR_G = 10;
#define DR_TABLE(name, ...) \
    __host__ __device__ constexpr int name(int i) { constexpr int t[] = {__VA_ARGS__}; return t[i]; }
DR_TABLE(dr_g_dy, 0, -1, 1, 0, 0, 0, -1, -1, 1, 1)
DR_TABLE(dr_g_dx, 0, 0, 0, 1, -1, -1, -1, 1, 1, -1)
DR_TABLE(dr_g_pos, 0, 0, 2, 1, 0, 3, 0, 1, 2, 3)
DR_TABLE(dr_g_len, 4, 2, 2, 2, 1, 1, 1, 1, 1, 1)
DR_TABLE(dr_g_bt, 0, 4, 6, 8, 10, 11, 12, 13, 14, 15)
DR_TABLE(dr_pos_a, 0, 0, 1, 1)   // accumulator position -> phase
DR_TABLE(dr_pos_b, 0, 1, 1, 0)
#undef DR_TABLE

struct DrParams {
    const __half* refined;
    const __half* raw;
    const float* bias;       // n_tile floats
    __half* out;
    int N, H, W, Cr, Cw, Co;
    int n_tile;              // round_up(Co, 16)
    int nch;                 // 16-byte channel chunks per pixel = (Cr + Cw) / 8
    int k16;                 // K=16 MMAs per group = ceil(nch / 2)
    int strips;              // ceil(W / 128)
    int items;               // strips * N * H
    int pair_pitch;          // staging bytes per output pixel pair: 4*Co + 16
};

struct __align__(8) DrBarriers {
    uint64_t full[DR_NS];
    uint64_t empty[DR_NS];
    uint64_t w_full;
};

__device__ __forceinline__ void cp_async16_zfill(uint32_t dst, const void* src, bool valid) {
    const int sz = valid ? 16 : 0;
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(sz) : "memory");
}

// Items are ordered strip-major, then image, then row, so a CTA's contiguous item range walks down the rows of a strip.
struct DrCursor {
    int sx, n, y;
    __device__ __forceinline__ void init(const DrParams& p, int item) {
        const int per_strip = p.N * p.H;
        sx = item / per_strip;
        const int g = item - sx * per_strip;
        n = g / p.H;
        y = g - n * p.H;
    }
    // advance to the next item; returns true when it continues the row run (same strip and image, next row)
    __device__ __forceinline__ bool next(const DrParams& p) {
        if (++y < p.H) return true;
        y = 0;
        if (++n == p.N) { n = 0; ++sx; }
        return false;
    }
};

// all MMAs of one tile for one warpgroup (10 groups x K16 slices), fully unrolled: group g multiplies the row view
// shifted by (dy, dx) with dr_g_len(g) consecutive weight sub-tiles into accumulator positions dr_g_pos(g) ...
template <int K16, int NCH>
__device__ __forceinline__ void dr_mma_tile(float (&acc)[4 * NCH][8], const uint32_t (&slot)[3], uint32_t w, uint32_t nt) {
#pragma unroll
    for (int g = 0; g < DR_G; ++g) {
        const uint32_t a = slot[dr_g_dy(g) + 1] + (dr_g_dx(g) + 1) * 128;   // (dx+1) pixel rows of 128 B
        const uint32_t b = w + dr_g_bt(g) * nt * 128;
#pragma unroll
        for (int k = 0; k < K16; ++k) wg_mma_chunks<4 * NCH>(acc, dr_g_pos(g) * NCH, dr_g_len(g) * NCH, a + 32 * k, b + 32 * k);
    }
}

template <int NCH>
__global__ void __launch_bounds__(DR_THREADS, 1)
deconv_rows_kernel(const __grid_constant__ CUtensorMap mapW, const __grid_constant__ DrParams p) {
    extern __shared__ __align__(1024) uint8_t smem[];
    const int w_bytes = 16 * p.n_tile * 128;
    const int stage_bytes = 2 * DR_TW * p.pair_pitch;           // two output rows of the tile
    uint8_t* sW = smem;
    uint8_t* sSlot = smem + w_bytes;                            // w_bytes is a multiple of 2048
    uint8_t* sStage = sSlot + DR_NS * DR_SLOT_BYTES;
    float* sBias = reinterpret_cast<float*>(sStage + 2 * stage_bytes);
    DrBarriers* bars = reinterpret_cast<DrBarriers*>(sBias + DR_MAX_NT);

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&mapW);
        for (int i = 0; i < DR_NS; ++i) { mbar_init(&bars->full[i], DR_PROD_WARPS); mbar_init(&bars->empty[i], DR_EPI_THREADS / 32); }
        mbar_init(&bars->w_full, 1);
        fence_barrier_init();
    }
    for (int i = threadIdx.x; i < DR_MAX_NT; i += DR_THREADS) sBias[i] = (p.bias && i < p.n_tile) ? p.bias[i] : 0.f;
    // K padding chunks of every slot pixel are zero for the whole kernel (the copies never touch them)
    for (int i = threadIdx.x; i < DR_NS * DR_SLOT_PX * 8; i += DR_THREADS) {
        const int c = i & 7, px = (i >> 3) % DR_SLOT_PX, s = (i >> 3) / DR_SLOT_PX;
        if (c >= p.nch)
            *reinterpret_cast<uint4*>(sSlot + s * DR_SLOT_BYTES + px * 128 + ((c ^ (px & 7)) << 4)) = make_uint4(0, 0, 0, 0);
    }
    fence_proxy_async();
    pdl_launch_dependents();
    __syncthreads();
    pdl_wait();

    // contiguous item range of this CTA
    const int per = p.items / (int)gridDim.x, extra = p.items % (int)gridDim.x;
    const int it_begin = (int)blockIdx.x * per + min((int)blockIdx.x, extra);
    const int n_items = per + ((int)blockIdx.x < extra ? 1 : 0);
    DrCursor cur;
    cur.init(p, it_begin);

    if (warp < DR_PROD_WARPS) {
        // ------------------------------------------------------------ producers: weights once, then input rows
        if (threadIdx.x == 0) {
            mbar_expect_tx(&bars->w_full, (uint32_t)w_bytes);
            for (int j = 0; j < 16; ++j) tma_load_2d(sW + j * p.n_tile * 128, &mapW, &bars->w_full, 0, j * p.n_tile);
        }
        // thread -> (channel chunk, pixel phase): 8 chunk lanes x 16 pixels per pass, 9 passes cover the 130 slot pixels
        const int t = threadIdx.x;
        const int ch = t & 7, px0 = t >> 3;
        const int nr = p.Cr >> 3;
        const bool active = ch < p.nch;
        const __half* bptr = (ch < nr) ? p.refined + ch * 8 : p.raw + (ch - nr) * 8;
        const int cstride = (ch < nr) ? p.Cr : p.Cw;
        int load = 0;          // running row-load index
        int pending = -1;      // load whose copies are issued but not yet published
        bool cont = false;
        for (int k = 0; k < n_items; ++k) {
            const int x0 = cur.sx * DR_TW, n = cur.n, y = cur.y;
            for (int r = cont ? y + 1 : y - 1; r <= y + 1; ++r, ++load) {
                const int slot = load % DR_NS;
                if (lane == 0) mbar_wait_backoff(&bars->empty[slot], ((load / DR_NS) & 1) ^ 1);
                __syncwarp();
                if (active) {
                    const uint32_t sbase = smem_u32(sSlot + slot * DR_SLOT_BYTES);
                    const bool rv = (r >= 0) && (r < p.H);
                    const size_t rowpix = ((size_t)n * p.H + (rv ? r : 0)) * p.W;
#pragma unroll
                    for (int q = 0; q < (DR_SLOT_PX + 15) / 16; ++q) {
                        const int px = px0 + 16 * q;
                        if (px < DR_SLOT_PX) {
                            const int x = x0 - 1 + px;
                            const bool v = rv && x >= 0 && x < p.W;
                            const __half* src = v ? bptr + (rowpix + x) * cstride : bptr;
                            cp_async16_zfill(sbase + px * 128 + ((ch ^ (px & 7)) << 4), src, v);
                        }
                    }
                }
                asm volatile("cp.async.commit_group;" ::: "memory");
                if (pending >= 0) {
                    // the previous row has landed once at most one group (the one just issued) is outstanding
                    asm volatile("cp.async.wait_group 1;" ::: "memory");
                    fence_proxy_async();
                    __syncwarp();
                    if (lane == 0) mbar_arrive(&bars->full[pending % DR_NS]);
                }
                pending = load;
            }
            cont = cur.next(p);
        }
        if (pending >= 0) {
            asm volatile("cp.async.wait_group 0;" ::: "memory");
            fence_proxy_async();
            __syncwarp();
            if (lane == 0) mbar_arrive(&bars->full[pending % DR_NS]);
        }
    } else {
        // ------------------------------------------------------------ consumer warpgroups: MMA + epilogue
        const int wg = (warp - DR_EPI_WARP0) >> 2;     // strip pixels 64*wg .. 64*wg+63
        const int wq = warp & 3;
        const int et = threadIdx.x - DR_EPI_WARP0 * 32;   // 0..255
        const int Co = p.Co;
        const int cpp = Co >> 2;                  // 16-byte chunks per output pixel pair
        const uint32_t nt = (uint32_t)p.n_tile;
        const uint32_t w_base = smem_u32(sW);
        const uint32_t slot_base = smem_u32(sSlot) + wg * 64 * 128;
        mbar_wait(&bars->w_full, 0);
        int load = 0, base = 0;
        bool cont = false;
        float acc[4 * NCH][8];
        for (int it = 0; it < n_items; ++it) {
            const int x0 = cur.sx * DR_TW, n = cur.n, y = cur.y;
            const int vw = min(DR_TW, p.W - x0);
            if (cont) { base += 1; load += 1; } else { base = load; load += 3; }
            const bool next_cont = cur.next(p) && (it + 1 < n_items);
            // rows base, base+1 were waited for by the previous tile of the run
            for (int d = cont ? 2 : 0; d < 3; ++d) mbar_wait(&bars->full[(base + d) % DR_NS], ((base + d) / DR_NS) & 1);
            uint32_t slot[3];
#pragma unroll
            for (int d = 0; d < 3; ++d) slot[d] = slot_base + (uint32_t)((base + d) % DR_NS) * DR_SLOT_BYTES;
#pragma unroll
            for (int c = 0; c < 4 * NCH; ++c)
#pragma unroll
                for (int i = 0; i < 8; ++i) acc[c][i] = 0.f;
            wg_fence();
            switch (p.k16) {
                case 1: dr_mma_tile<1, NCH>(acc, slot, w_base, nt); break;
                case 2: dr_mma_tile<2, NCH>(acc, slot, w_base, nt); break;
                case 3: dr_mma_tile<3, NCH>(acc, slot, w_base, nt); break;
                default: dr_mma_tile<4, NCH>(acc, slot, w_base, nt); break;
            }
            wg_commit();
            wg_wait0();
            // rows no later tile needs go back to the producers
            __syncwarp();
            if (lane == 0) {
                mbar_arrive(&bars->empty[base % DR_NS]);
                if (!next_cont) {
                    mbar_arrive(&bars->empty[(base + 1) % DR_NS]);
                    mbar_arrive(&bars->empty[(base + 2) % DR_NS]);
                }
            }
            cont = next_cont;
            uint8_t* st = sStage + (it & 1) * stage_bytes;
#pragma unroll
            for (int c = 0; c < 4 * NCH; ++c) {
                const int pos = c / NCH;
                const int a = dr_pos_a(pos), b = dr_pos_b(pos);
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const int px = wg * 64 + frag_row(wq, lane, i);
                    const int co = (c - pos * NCH) * 16 + frag_col(lane, i);
                    if (co < Co)
                        *reinterpret_cast<__half2*>(st + a * (DR_TW * p.pair_pitch) + px * p.pair_pitch + b * (Co * 2) + co * 2) =
                            __floats2half2_rn(fmaxf(acc[c][2 * i] + sBias[co], 0.f), fmaxf(acc[c][2 * i + 1] + sBias[co + 1], 0.f));
                }
            }
            asm volatile("bar.sync 1, 256;" ::: "memory");
            // copy-out: output rows 2y, 2y+1, pixels 2*x0 .. 2*(x0+vw)-1, each row one contiguous run
            const int per_row = vw * cpp;
            uint4* orow0 = reinterpret_cast<uint4*>(p.out + (((size_t)n * 2 * p.H + 2 * y) * (2 * p.W) + 2 * x0) * Co);
            const size_t row_stride16 = ((size_t)2 * p.W * Co) >> 3;     // one output row in 16-byte units
            // up to 1024 16-byte chunks per output row: all loads of a row first, then its stores
#pragma unroll
            for (int a = 0; a < 2; ++a) {
                const uint8_t* srow = st + a * (DR_TW * p.pair_pitch);
                uint4* orow = orow0 + a * row_stride16;
                uint4 v[4];
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    const int i = et + u * DR_EPI_THREADS;
                    if (i < per_row) {
                        int pair, c;
                        if (cpp == 8) { pair = i >> 3; c = i & 7; }
                        else { pair = i / cpp; c = i - pair * cpp; }
                        v[u] = *reinterpret_cast<const uint4*>(srow + pair * p.pair_pitch + c * 16);
                    }
                }
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    const int i = et + u * DR_EPI_THREADS;
                    if (i < per_row) orow[i] = v[u];
                }
            }
        }
    }
}

// ------------------------------------------------------------------ host side
static inline int dr_round_up(int a, int b) { return (a + b - 1) / b * b; }

static size_t dr_smem_bytes(int Co) {
    const int nt = dr_round_up(Co, 16);
    return 1024 + (size_t)16 * nt * 128 + (size_t)DR_NS * DR_SLOT_BYTES + (size_t)2 * 2 * DR_TW * (4 * Co + 16) +
           DR_MAX_NT * 4 + sizeof(DrBarriers) + 64;
}

// packed weights [sub-tile (group order, accumulator order inside a group)][co (n_tile)][64]:
// K index kk < Cr -> refined channel kk, Cr <= kk < Cr+Cw -> raw channel kk-Cr, else 0
static void dr_pack(int Cr, int Cw, int Co, const uint16_t* wr, const uint16_t* ww, uint16_t* wp) {
    const int nt = dr_round_up(Co, 16);
    for (int g = 0; g < DR_G; ++g)
        for (int l = 0; l < dr_g_len(g); ++l) {
            const int pos = dr_g_pos(g) + l;
            const int a = dr_pos_a(pos), b = dr_pos_b(pos);
            const int dy = dr_g_dy(g), dx = dr_g_dx(g);
            const int ki = dy == 0 ? 1 + a : (a ? 0 : 3);
            const int kj = dx == 0 ? 1 + b : (b ? 0 : 3);
            uint16_t* dst = wp + (size_t)(dr_g_bt(g) + l) * nt * 64;
            for (int co = 0; co < nt; ++co)
                for (int kk = 0; kk < 64; ++kk) {
                    uint16_t v = 0;
                    if (co < Co) {
                        if (kk < Cr) v = wr[(((size_t)kk * Co + co) * 4 + ki) * 4 + kj];
                        else if (kk < Cr + Cw) v = ww[(((size_t)(kk - Cr) * Co + co) * 4 + ki) * 4 + kj];
                    }
                    dst[(size_t)co * 64 + kk] = v;
                }
        }
}

// channel eligibility (decides whether the packed buffer carries the row-kernel weights)
bool deconv_rows_channels_ok(int Cr, int Cw, int Co) {
    return Cr % 8 == 0 && Cw % 8 == 0 && Co % 8 == 0 && Cr + Cw <= 64 && Co <= DR_MAX_NT && dr_smem_bytes(Co) <= 227 * 1024;
}
size_t deconv_rows_packed_elems(int Cr, int Cw, int Co) {
    return deconv_rows_channels_ok(Cr, Cw, Co) ? (size_t)16 * dr_round_up(Co, 16) * 64 : 0;
}
void deconv_rows_pack(const uint16_t* wr, const uint16_t* ww, int Cr, int Cw, int Co, uint16_t* wp) {
    dr_pack(Cr, Cw, Co, wr, ww, wp);
}
// the row kernel pays off on wide maps (a strip is 128 pixels); narrow levels keep the tiled kernel
bool deconv_rows_shape_ok(int W) { return W >= 64; }

int launch_deconv_rows(const void* refined, const void* raw, const void* w_rows, const float* bias_packed, void* out, int N,
                       int H, int W, int Cr, int Cw, int Co, cudaStream_t stream) {
    DrParams p;
    memset(&p, 0, sizeof(p));
    p.refined = reinterpret_cast<const __half*>(refined);
    p.raw = reinterpret_cast<const __half*>(raw);
    p.bias = bias_packed;
    p.out = reinterpret_cast<__half*>(out);
    p.N = N; p.H = H; p.W = W; p.Cr = Cr; p.Cw = Cw; p.Co = Co;
    p.n_tile = dr_round_up(Co, 16);
    p.nch = (Cr + Cw) / 8;
    p.k16 = (p.nch + 1) / 2;
    p.strips = (W + DR_TW - 1) / DR_TW;
    const long long items = (long long)p.strips * N * H;
    LP_CHECK_ARG(items < (1ll << 31), "lp_fusion_deconv_f16: too many rows");
    p.items = (int)items;
    p.pair_pitch = 4 * Co + 16;
    CUtensorMap mw;
    {
        uint64_t dims[2] = {64, (uint64_t)16 * p.n_tile};
        uint64_t strides[1] = {128};
        uint32_t box[2] = {64, (uint32_t)p.n_tile};
        int rc = make_tmap(&mw, w_rows, 2, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B);
        if (rc) return rc;
    }
    const size_t smem = dr_smem_bytes(Co);
    // accumulator width: 4 phases x n_tile columns, 16 per chunk
    auto kern = p.n_tile <= 16 ? deconv_rows_kernel<1> : p.n_tile <= 32 ? deconv_rows_kernel<2>
              : p.n_tile <= 48 ? deconv_rows_kernel<3> : deconv_rows_kernel<4>;
    cudaError_t e = cudaFuncSetAttribute((const void*)kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return cuda_fail(e, "cudaFuncSetAttribute(deconv_rows)");
    int grid = p.items < num_sms() ? p.items : num_sms();
    cudaError_t le = launch_pdl(kern, dim3(grid), dim3(DR_THREADS), smem, stream, mw, p);
    if (le != cudaSuccess) return cuda_fail(le, "launch deconv_rows_kernel");
    LP_LAUNCH_CHECK("deconv_rows_kernel");
    return LP_OK;
}

}  // namespace lp
