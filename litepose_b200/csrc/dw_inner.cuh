// Inner loop of the fused depthwise kernels (dwpw.cu, dwblock.cu): one thread = one channel PAIR x a BY x 4 micro-block
// of output pixels of a [I][I][32-channel] fp16 slab in shared memory.
//
// Arithmetic: packed fp16 (HFMA2): two MACs per lane per instruction, where fp32 accumulation needs a conversion and an
// FMA per MAC-lane and leaves fewer issue slots for the LDS/STS of the loop.  The K*K taps are accumulated as chains of two kernel rows folded into
// a running fp16 total seeded with the fp16 bias (<= 2K roundings at partial magnitude per chain).  The network's outputs
// stay at 0.27-0.34 of the parity tolerance for XS/S and 0.67 for M 512, against 0.25-0.30 and 0.62 with an fp32
// depthwise (error budget dominated by the fp16 activation storage; tests/emulate_dw_precision.py runs the bit-exact
// emulator of this arithmetic, tests/dw_emul.py, which tests/test_gpu_dw_exact.py holds the kernels to).
//
// Bank conflicts: a half-warp (16 channel pairs) reads the 64 contiguous bytes of ONE pixel; the other half-warp works
// on the x-adjacent micro-block in MIRRORED column order, so the two pixels always have opposite parity (the other 16
// banks).  Mirrored data needs mirrored weights (read with a negative tap stride) and mirrored stores (caller).
#pragma once
#include <cuda_fp16.h>

namespace lp {

// PP = pixel pitch of the slab in half2 units: CB/2 for the pixel-major [I][I][CB] slab the TMA delivers (dwpw.cu,
// tile_in already offset by the thread's channel pair), 4 for the chunk-major slab of dwblock.cu
// ([4 chunks of 8 channels][I*I pixels][16 B], tile_in offset by chunk base + pair inside the chunk), any other pitch
// with tile_in offset by the pair.  I = row pitch of the slab in pixels.  S = stride: output (oy + i, ox + j) reads
// input (S (oy + i) + ky, S (ox + j) + kx) of the slab.  Stride 2 has no mirrored lanes (mir must be false).
template <int K, int BY, int I, int CB, int PP = CB / 2, int S = 1>
__device__ __forceinline__ void dw_slab_hfma2(const __half2* __restrict__ tile_in, const __half2* __restrict__ wslab, int cp,
                                              bool mir, int oy, int ox, __half2 bias, __half2 (&acc)[BY][4]) {
    constexpr int IRX = 3 * S + K;       // input columns of a micro-block
    constexpr int IRY = (BY - 1) * S + K;   // input rows
    constexpr int HP = CB / 2;           // half2 per pixel of the weight slab
    const int cstep = mir ? -PP : PP;
    __half2 part[BY][4];
#pragma unroll
    for (int i = 0; i < BY; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = bias;
    __half2 wreg[K * K];
    {
        const __half2* ws = wslab + cp + (mir ? (K - 1) * HP : 0);
        const int wstep = mir ? -HP : HP;
#pragma unroll
        for (int ky = 0; ky < K; ++ky)
#pragma unroll
            for (int kx = 0; kx < K; ++kx) wreg[ky * K + kx] = ws[ky * K * HP + kx * wstep];
    }
    const __half2* base = tile_in + (S * (oy * I + ox) + (mir ? IRX - 1 : 0)) * PP + (PP == HP ? cp : 0);
#pragma unroll
    for (int r = 0; r < IRY; ++r) {
        __half2 in[IRX];
#pragma unroll
        for (int c = 0; c < IRX; ++c) in[c] = base[r * I * PP + c * cstep];
#pragma unroll
        for (int i = 0; i < BY; ++i) {
            const int ky = r - i * S;
            if (ky >= 0 && ky < K) {
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
            }
        }
    }
}

// ReLU6'd results of a micro-block -> 128B-swizzled K-major A tile(s) of the projection: row = pixel of the 16x16 tile
// (two M-tiles of 8 rows x 16 px), 16-byte chunk jch = channels 8*jch.. of the 64-channel K block.
template <int BY>
__device__ __forceinline__ void dw_store_a(uint8_t* sA, int a_tile_bytes, const __half2 (&acc)[BY][4], int oy, int ox, bool mir,
                                           int jch, int cp) {
    const __half2 zero2 = __floats2half2_rn(0.f, 0.f), six2 = __floats2half2_rn(6.f, 6.f);
    uint8_t* a_mt = sA + (oy >> 3) * a_tile_bytes;      // a micro-block never straddles the two M-tiles (oy % BY == 0)
#pragma unroll
    for (int i = 0; i < BY; ++i) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int r = ((oy + i) & 7) * 16 + ox + (mir ? 3 - j : j);     // row inside the M-tile
            const __half2 v = __hmin2(__hmax2(acc[i][j], zero2), six2);
            *reinterpret_cast<__half2*>(a_mt + r * 128 + ((jch ^ (r & 7)) << 4) + ((cp & 3) << 2)) = v;
        }
    }
}

}  // namespace lp
