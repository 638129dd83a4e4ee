// The depthwise arithmetic of every kernel (dwconv.cu, dwpw.cu, dwblock.cu, stem_fused.cu), once: one thread = one
// channel PAIR x a BY x 4 micro-block of output pixels of an fp16 slab in shared memory.  One function per precision
// mode of lp_set_dw_precision, each restated bit for bit by tests/dw_emul.py's dwconv(..., prec):
//   prec 2  dw_hfma2    packed fp16 (HFMA2): two MACs per lane per instruction, where fp32 accumulation needs a
//                       conversion and an FMA per MAC-lane and leaves fewer issue slots for the LDS/STS of the loop.  The
//                       K*K taps are accumulated as chains of two kernel rows folded into a running fp16 total seeded
//                       with the fp16 bias (<= 2K roundings at partial magnitude per chain).  The fused block kernels and
//                       the unfused k = 3, 7 default.
//   prec 0  dw_ffma     every product accumulated in fp32 (fhfma).  The heads, which feed the network outputs directly.
//   prec 1  dw_rowsum   the K taps of one kernel row accumulated with packed HFMA2, each row sum added in fp32.
// With the packed chains the network's outputs stay at 0.27-0.34 of the parity tolerance for XS/S and 0.67 for M 512,
// against 0.25-0.30 and 0.62 with an fp32 depthwise (error budget dominated by the fp16 activation storage;
// tests/emulate_dw_precision.py measures this with the emulator, tests/test_gpu_dw_exact.py holds the kernels to it).
//
// Weights: wreg[K*K] in registers, tap-major, kernel rows already reversed for mirrored lanes (dw_load_wslab reads them
// from a TMA-staged slab; dwconv.cu loads its own from global memory).
// Bank conflicts: a half-warp (16 channel pairs) reads the 64 contiguous bytes of ONE pixel; the other half-warp works
// on the x-adjacent micro-block in MIRRORED column order, so the two pixels always have opposite parity (the other 16
// banks).  Mirrored data needs mirrored weights and mirrored stores (dw_store_a, dwconv.cu).
#pragma once
#include "common.cuh"

namespace lp {

// fp16 x fp16 + fp32 -> fp32 with one rounding: the fp16 -> fp32 conversions are exact, so the fp32 FMA of the
// converted operands gives the same result as a mixed-precision FMA.
__device__ __forceinline__ float fhfma(__half a, __half b, float c) { return __fmaf_rn(__half2float(a), __half2float(b), c); }

// The thread's weights from a TMA-staged tap-major [K*K][CB] fp16 slab; mirrored lanes read kx reversed.
template <int K, int CB>
__device__ __forceinline__ void dw_load_wslab(const __half2* __restrict__ wslab, int cp, bool mir, __half2 (&wreg)[K * K]) {
    constexpr int HP = CB / 2;           // half2 per tap
    const __half2* ws = wslab + cp + (mir ? (K - 1) * HP : 0);
    const int wstep = mir ? -HP : HP;
#pragma unroll
    for (int ky = 0; ky < K; ++ky)
#pragma unroll
        for (int kx = 0; kx < K; ++kx) wreg[ky * K + kx] = ws[ky * K * HP + kx * wstep];
}

// The input walk of every mode.  tile_in = the thread's channel pair in the slab (the caller offsets it); PP = pixel
// pitch in half2 units (CB/2 for a pixel-major [I][I][CB] slab, 4 for the chunk-major slabs of dwblock.cu and
// stem_fused.cu), I = row pitch in pixels.  S = stride: output (oy + i, ox + j) reads input (S (oy + i) + ky,
// S (ox + j) + kx) of the slab.  Stride 2 has no mirrored lanes (mir must be false).  Row r of the micro-block's input
// window is loaded into in[] (slot c = input column c, or IRX-1-c when mirrored) and handed to op(i, ky, in) for every
// output row i whose kernel row ky it is.
template <int K, int BY, int I, int PP, int S, typename Op>
__device__ __forceinline__ void dw_walk(const __half2* __restrict__ tile_in, bool mir, int oy, int ox, Op&& op) {
    constexpr int IRX = 3 * S + K;          // input columns of a micro-block
    constexpr int IRY = (BY - 1) * S + K;   // input rows
    const int cstep = mir ? -PP : PP;
    const __half2* base = tile_in + (S * (oy * I + ox) + (mir ? IRX - 1 : 0)) * PP;
#pragma unroll
    for (int r = 0; r < IRY; ++r) {
        __half2 in[IRX];
#pragma unroll
        for (int c = 0; c < IRX; ++c) in[c] = base[r * I * PP + c * cstep];
#pragma unroll
        for (int i = 0; i < BY; ++i) {
            const int ky = r - i * S;
            if (ky >= 0 && ky < K) op(i, ky, in);
        }
    }
}

// prec 2: chains of two kernel rows (hmul2 at even ky, kx = 0, then hfma2) folded into the fp16 total with hadd2 after
// an odd ky or the last one: chains of <= 2K roundings at partial magnitude instead of K*K at full magnitude.
template <int K, int BY, int I, int PP, int S = 1>
__device__ __forceinline__ void dw_hfma2(const __half2* __restrict__ tile_in, const __half2 (&wreg)[K * K], bool mir, int oy,
                                         int ox, __half2 bias, __half2 (&acc)[BY][4]) {
    __half2 part[BY][4];
#pragma unroll
    for (int i = 0; i < BY; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = bias;
    dw_walk<K, BY, I, PP, S>(tile_in, mir, oy, ox, [&](int i, int ky, const auto& in) {
#pragma unroll
        for (int kx = 0; kx < K; ++kx) {
            const __half2 wv = wreg[ky * K + kx];
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                if ((ky & 1) == 0 && kx == 0) part[i][j] = __hmul2(in[j * S + kx], wv);     // a new two-row chain
                else part[i][j] = __hfma2(in[j * S + kx], wv, part[i][j]);
            }
        }
        if ((ky & 1) || ky == K - 1) {
#pragma unroll
            for (int j = 0; j < 4; ++j) acc[i][j] = __hadd2(acc[i][j], part[i][j]);
        }
    });
}

// prec 0: acc = bias, then every tap in kernel-row order acc = fhfma(x, w, acc) per lane.
template <int K, int BY, int I, int PP, int S = 1>
__device__ __forceinline__ void dw_ffma(const __half2* __restrict__ tile_in, const __half2 (&wreg)[K * K], bool mir, int oy,
                                        int ox, float2 bias, float2 (&acc)[BY][4]) {
#pragma unroll
    for (int i = 0; i < BY; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = bias;
    dw_walk<K, BY, I, PP, S>(tile_in, mir, oy, ox, [&](int i, int ky, const auto& in) {
#pragma unroll
        for (int kx = 0; kx < K; ++kx) {
            const __half2 wv = wreg[ky * K + kx];
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                acc[i][j].x = fhfma(__low2half(in[j * S + kx]), __low2half(wv), acc[i][j].x);
                acc[i][j].y = fhfma(__high2half(in[j * S + kx]), __high2half(wv), acc[i][j].y);
            }
        }
    });
}

// prec 1: per kernel row an fp16 chain (hmul2 on the first tap, hfma2 on the rest), its sum added to the fp32 acc.
template <int K, int BY, int I, int PP, int S = 1>
__device__ __forceinline__ void dw_rowsum(const __half2* __restrict__ tile_in, const __half2 (&wreg)[K * K], bool mir, int oy,
                                          int ox, float2 bias, float2 (&acc)[BY][4]) {
#pragma unroll
    for (int i = 0; i < BY; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = bias;
    dw_walk<K, BY, I, PP, S>(tile_in, mir, oy, ox, [&](int i, int ky, const auto& in) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            __half2 s = __hmul2(in[j * S], wreg[ky * K]);
#pragma unroll
            for (int kx = 1; kx < K; ++kx) s = __hfma2(in[j * S + kx], wreg[ky * K + kx], s);
            acc[i][j].x = __fadd_rn(__half2float(__low2half(s)), acc[i][j].x);
            acc[i][j].y = __fadd_rn(__half2float(__high2half(s)), acc[i][j].y);
        }
    });
}

// prec 2 on a TMA-staged [K*K][CB] weight slab: the fused kernels' depthwise.
template <int K, int BY, int I, int CB, int PP = CB / 2, int S = 1>
__device__ __forceinline__ void dw_slab_hfma2(const __half2* __restrict__ tile_in, const __half2* __restrict__ wslab, int cp,
                                              bool mir, int oy, int ox, __half2 bias, __half2 (&acc)[BY][4]) {
    __half2 wreg[K * K];
    dw_load_wslab<K, CB>(wslab, cp, mir, wreg);
    dw_hfma2<K, BY, I, PP, S>(tile_in, wreg, mir, oy, ox, bias, acc);
}

// ReLU6 of a micro-block's packed results (see relu6_h2)
template <int BY>
__device__ __forceinline__ void dw_relu6(__half2 (&v)[BY][4]) {
#pragma unroll
    for (int i = 0; i < BY; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) v[i][j] = relu6_h2(v[i][j]);
}

// Activated fp16 results of a micro-block -> 128B-swizzled K-major A tile(s) of the projection: row = pixel of the
// 16x16 tile (two M-tiles of 8 rows x 16 px), 16-byte chunk jch = channels 8*jch.. of the 64-channel K block.
template <int BY>
__device__ __forceinline__ void dw_store_a(uint8_t* sA, int a_tile_bytes, const __half2 (&v)[BY][4], int oy, int ox, bool mir,
                                           int jch, int cp) {
    uint8_t* a_mt = sA + (oy >> 3) * a_tile_bytes;      // a micro-block never straddles the two M-tiles (oy % BY == 0)
#pragma unroll
    for (int i = 0; i < BY; ++i) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int r = ((oy + i) & 7) * 16 + ox + (mir ? 3 - j : j);     // row inside the M-tile
            *reinterpret_cast<__half2*>(a_mt + r * 128 + ((jch ^ (r & 7)) << 4) + ((cp & 3) << 2)) = v[i][j];
        }
    }
}

}  // namespace lp
