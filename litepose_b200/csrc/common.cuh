// Common device/host helpers for the LitePose sm_90a kernels.
// PTX wrappers: mbarrier, TMA (cp.async.bulk.tensor), wgmma.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "../../include/litepose_b200.h"

namespace lp {

// ---------------------------------------------------------------- error state
void set_error(const char* fmt, ...);
int cuda_fail(cudaError_t e, const char* what);

#define LP_CHECK_ARG(cond, ...)                 \
    do {                                        \
        if (!(cond)) {                          \
            lp::set_error(__VA_ARGS__);         \
            return LP_ERR_BAD_ARG;              \
        }                                       \
    } while (0)

#define LP_CUDA(call)                                              \
    do {                                                           \
        cudaError_t _e = (call);                                   \
        if (_e != cudaSuccess) return lp::cuda_fail(_e, #call);    \
    } while (0)

#define LP_LAUNCH_CHECK(name)                                      \
    do {                                                           \
        cudaError_t _e = cudaGetLastError();                       \
        if (_e != cudaSuccess) return lp::cuda_fail(_e, name);     \
        lp::count_launch();                                        \
    } while (0)

void count_launch();

// Build a tiled tensor map (driver entry point resolved at run time; no libcuda link).
// dims/strides innermost first; strides in bytes for dims 1..rank-1.
int make_tmap(CUtensorMap* map, const void* base, int rank, const uint64_t* dims,
              const uint64_t* strides_bytes, const uint32_t* box, CUtensorMapSwizzle swz,
              CUtensorMapDataType dt = CU_TENSOR_MAP_DATA_TYPE_FLOAT16);
// The fp16 layouts the kernels load:
//   NHWC activation [N][H][W][C], box (box_c channels x box_w x box_h pixels) of one image
int make_tmap_nhwc(CUtensorMap* map, const void* x, int N, int H, int W, int C, int box_c, int box_w, int box_h,
                   CUtensorMapSwizzle swz);
//   packed K-major weights [rows][64] (lp_pw1x1_pack and its kin), box (box_k columns x box_rows rows)
int make_tmap_rows64(CUtensorMap* map, const void* w, int rows, int box_k, int box_rows, CUtensorMapSwizzle swz);
//   tap-major depthwise weights [taps][C], box = every tap of one 32-channel slab, unswizzled
int make_tmap_taps(CUtensorMap* map, const void* w, int taps, int C);

int num_sms();

// Programmatic dependent launch (PDL): kernels launched through launch_pdl() may start their prologue (barrier init,
// descriptor prefetch, weight staging) while the previous kernel of the stream drains; they call
// pdl_wait() before touching any activation memory.

#ifdef __CUDACC__
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                              Args&&... args) {
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}
#endif

// ---------------------------------------------------------------- device side
#ifdef __CUDACC__

__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    while (!mbar_try_wait(bar, parity)) {
    }
}
// Wait used by the single-thread producer / MMA roles: back off with nanosleep so that the spinning warp does not
// take issue slots from the compute warps of its SM sub-partition (the warp scheduler favours high warp ids).
__device__ __forceinline__ void mbar_wait_backoff(uint64_t* bar, uint32_t parity) {
    while (!mbar_try_wait(bar, parity)) __nanosleep(128);
}

__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
        ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
        : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2,
                                            int c3) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, "
        "%6}], [%2];" ::"r"(smem_u32(dst)),
        "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
        : "memory");
}

// ---- wgmma (Hopper warpgroup MMA): D[64 x 16 per call] (+)= A[smem] * B[smem]^T, fp16 in, fp32 accumulators in the
// registers of the issuing warpgroup.  Every thread of the four warps of a warpgroup executes these together.
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_wait0() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
__device__ __forceinline__ void wg_wait1() { asm volatile("wgmma.wait_group.sync.aligned 1;" ::: "memory"); }
__device__ __forceinline__ void wg_mma16(float (&d)[8], uint64_t adesc, uint64_t bdesc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
        : "l"(adesc), "l"(bdesc)
        : "memory");
}

// Per-warpgroup register budget (all four warps of a warpgroup execute it): the producer warpgroup of the fused kernels
// hands registers to the compute warpgroups, whose wgmma accumulators stay live across the depthwise work.
template <int N> __device__ __forceinline__ void regs_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N> __device__ __forceinline__ void regs_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }

// K-major, 128B-swizzled shared-memory matrix descriptor (sm_90 wgmma): 8-row x 128-byte swizzle atoms stacked along
// M/N every 1024 bytes; a K=16 slice starts 32 bytes further into the atom.
__device__ __forceinline__ uint64_t wg_desc_sw128(uint32_t smem_addr) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);   // start address  [0,14)
    d |= (uint64_t)1 << 16;                        // LBO (unused for swizzled K-major)
    d |= (uint64_t)(1024 >> 4) << 32;              // SBO = 1024 B   [32,46)
    d |= (uint64_t)1 << 62;                        // SWIZZLE_128B
    return d;
}

// acc[c] += A[64 rows at a_addr, K=16] x B[rows 16*(c - c0) .. +15 at b_addr, K=16]^T for c0 <= c < c0 + nc: one K=16
// slice against nc 16-column chunks.  NC bounds the accumulator array; the chunk range is uniform over the warpgroup.
template <int NC>
__device__ __forceinline__ void wg_mma_chunks(float (&acc)[NC][8], int c0, int nc, uint32_t a_addr, uint32_t b_addr) {
    const uint64_t ad = wg_desc_sw128(a_addr);
#pragma unroll
    for (int c = 0; c < NC; ++c)
        if (c >= c0 && c < c0 + nc) wg_mma16(acc[c], ad, wg_desc_sw128(b_addr + (uint32_t)(c - c0) * 2048u));
}

// The same for operands whose rows are 32 or 64 bytes wide: 8-row swizzle atoms of 256 / 512 bytes stacked along M/N
// (the layout a TMA box with CU_TENSOR_MAP_SWIZZLE_32B / _64B writes when its inner extent is the row width).
__device__ __forceinline__ uint64_t wg_desc_sw32(uint32_t smem_addr) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);
    d |= (uint64_t)1 << 16;
    d |= (uint64_t)(256 >> 4) << 32;               // SBO = 256 B
    d |= (uint64_t)3 << 62;                        // SWIZZLE_32B
    return d;
}
__device__ __forceinline__ uint64_t wg_desc_sw64(uint32_t smem_addr) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);
    d |= (uint64_t)1 << 16;
    d |= (uint64_t)(512 >> 4) << 32;               // SBO = 512 B
    d |= (uint64_t)2 << 62;                        // SWIZZLE_64B
    return d;
}

// acc[0..NC) (+)= A[64 rows at a_addr, K=16] x B[16*NC rows at b_addr, K=16]^T as ONE wgmma m64n(16*NC)k16.  The m64nN
// accumulator fragment is the n16 fragments of its 16-column chunks concatenated in register order (frag_row / frag_col
// hold per chunk), and the B rows are contiguous 1024-byte swizzle atoms, so this computes what wg_mma_chunks<NC>(acc,
// 0, NC, ...) does with one A read instead of NC.  accumulate = 0 overwrites acc with the product (scale-d = 0): the
// accumulators then need no zeroing by ordinary instructions, which would make ptxas fence (and serialise) the wgmma
// issue when it sits on a data-dependent path.  wg_mma_nd takes the two matrix descriptors (any swizzle mode);
// wg_mma_n builds 128B-swizzle descriptors from shared-memory addresses.
template <int NC> __device__ __forceinline__ void wg_mma_nd(float (&acc)[NC][8], uint64_t adesc, uint64_t bdesc, int accumulate);
template <> __device__ __forceinline__ void wg_mma_nd<1>(float (&d)[1][8], uint64_t adesc, uint64_t bdesc, int accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0][0]), "+f"(d[0][1]), "+f"(d[0][2]), "+f"(d[0][3]), "+f"(d[0][4]), "+f"(d[0][5]), "+f"(d[0][6]), "+f"(d[0][7])
        : "l"(adesc), "l"(bdesc), "r"(accumulate)
        : "memory");
}
template <> __device__ __forceinline__ void wg_mma_nd<2>(float (&d)[2][8], uint64_t adesc, uint64_t bdesc, int accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 "
        "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0][0]), "+f"(d[0][1]), "+f"(d[0][2]), "+f"(d[0][3]), "+f"(d[0][4]), "+f"(d[0][5]), "+f"(d[0][6]), "+f"(d[0][7]),
          "+f"(d[1][0]), "+f"(d[1][1]), "+f"(d[1][2]), "+f"(d[1][3]), "+f"(d[1][4]), "+f"(d[1][5]), "+f"(d[1][6]), "+f"(d[1][7])
        : "l"(adesc), "l"(bdesc), "r"(accumulate)
        : "memory");
}
template <> __device__ __forceinline__ void wg_mma_nd<3>(float (&d)[3][8], uint64_t adesc, uint64_t bdesc, int accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %26, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n48k16.f32.f16.f16 "
        "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23}, %24, %25, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0][0]), "+f"(d[0][1]), "+f"(d[0][2]), "+f"(d[0][3]), "+f"(d[0][4]), "+f"(d[0][5]), "+f"(d[0][6]), "+f"(d[0][7]),
          "+f"(d[1][0]), "+f"(d[1][1]), "+f"(d[1][2]), "+f"(d[1][3]), "+f"(d[1][4]), "+f"(d[1][5]), "+f"(d[1][6]), "+f"(d[1][7]),
          "+f"(d[2][0]), "+f"(d[2][1]), "+f"(d[2][2]), "+f"(d[2][3]), "+f"(d[2][4]), "+f"(d[2][5]), "+f"(d[2][6]), "+f"(d[2][7])
        : "l"(adesc), "l"(bdesc), "r"(accumulate)
        : "memory");
}
template <> __device__ __forceinline__ void wg_mma_nd<4>(float (&d)[4][8], uint64_t adesc, uint64_t bdesc, int accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
        "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,"
        "%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0][0]), "+f"(d[0][1]), "+f"(d[0][2]), "+f"(d[0][3]), "+f"(d[0][4]), "+f"(d[0][5]), "+f"(d[0][6]), "+f"(d[0][7]),
          "+f"(d[1][0]), "+f"(d[1][1]), "+f"(d[1][2]), "+f"(d[1][3]), "+f"(d[1][4]), "+f"(d[1][5]), "+f"(d[1][6]), "+f"(d[1][7]),
          "+f"(d[2][0]), "+f"(d[2][1]), "+f"(d[2][2]), "+f"(d[2][3]), "+f"(d[2][4]), "+f"(d[2][5]), "+f"(d[2][6]), "+f"(d[2][7]),
          "+f"(d[3][0]), "+f"(d[3][1]), "+f"(d[3][2]), "+f"(d[3][3]), "+f"(d[3][4]), "+f"(d[3][5]), "+f"(d[3][6]), "+f"(d[3][7])
        : "l"(adesc), "l"(bdesc), "r"(accumulate)
        : "memory");
}

// m64n80k16 .. m64n160k16: the projection widths of the wide depthwise+projection kernel (dwpw.cu, Co 65..160)
template <> __device__ __forceinline__ void wg_mma_nd<5>(float (&d)[5][8], uint64_t adesc, uint64_t bdesc, int accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %42, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n80k16.f32.f16.f16 "
        "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,"
        "%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39}, %40, %41, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0][0]), "+f"(d[0][1]), "+f"(d[0][2]), "+f"(d[0][3]), "+f"(d[0][4]), "+f"(d[0][5]), "+f"(d[0][6]), "+f"(d[0][7]),
          "+f"(d[1][0]), "+f"(d[1][1]), "+f"(d[1][2]), "+f"(d[1][3]), "+f"(d[1][4]), "+f"(d[1][5]), "+f"(d[1][6]), "+f"(d[1][7]),
          "+f"(d[2][0]), "+f"(d[2][1]), "+f"(d[2][2]), "+f"(d[2][3]), "+f"(d[2][4]), "+f"(d[2][5]), "+f"(d[2][6]), "+f"(d[2][7]),
          "+f"(d[3][0]), "+f"(d[3][1]), "+f"(d[3][2]), "+f"(d[3][3]), "+f"(d[3][4]), "+f"(d[3][5]), "+f"(d[3][6]), "+f"(d[3][7]),
          "+f"(d[4][0]), "+f"(d[4][1]), "+f"(d[4][2]), "+f"(d[4][3]), "+f"(d[4][4]), "+f"(d[4][5]), "+f"(d[4][6]), "+f"(d[4][7])
        : "l"(adesc), "l"(bdesc), "r"(accumulate)
        : "memory");
}
template <> __device__ __forceinline__ void wg_mma_nd<6>(float (&d)[6][8], uint64_t adesc, uint64_t bdesc, int accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %50, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n96k16.f32.f16.f16 "
        "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,"
        "%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47}, %48, %49, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0][0]), "+f"(d[0][1]), "+f"(d[0][2]), "+f"(d[0][3]), "+f"(d[0][4]), "+f"(d[0][5]), "+f"(d[0][6]), "+f"(d[0][7]),
          "+f"(d[1][0]), "+f"(d[1][1]), "+f"(d[1][2]), "+f"(d[1][3]), "+f"(d[1][4]), "+f"(d[1][5]), "+f"(d[1][6]), "+f"(d[1][7]),
          "+f"(d[2][0]), "+f"(d[2][1]), "+f"(d[2][2]), "+f"(d[2][3]), "+f"(d[2][4]), "+f"(d[2][5]), "+f"(d[2][6]), "+f"(d[2][7]),
          "+f"(d[3][0]), "+f"(d[3][1]), "+f"(d[3][2]), "+f"(d[3][3]), "+f"(d[3][4]), "+f"(d[3][5]), "+f"(d[3][6]), "+f"(d[3][7]),
          "+f"(d[4][0]), "+f"(d[4][1]), "+f"(d[4][2]), "+f"(d[4][3]), "+f"(d[4][4]), "+f"(d[4][5]), "+f"(d[4][6]), "+f"(d[4][7]),
          "+f"(d[5][0]), "+f"(d[5][1]), "+f"(d[5][2]), "+f"(d[5][3]), "+f"(d[5][4]), "+f"(d[5][5]), "+f"(d[5][6]), "+f"(d[5][7])
        : "l"(adesc), "l"(bdesc), "r"(accumulate)
        : "memory");
}
template <> __device__ __forceinline__ void wg_mma_nd<7>(float (&d)[7][8], uint64_t adesc, uint64_t bdesc, int accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %58, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n112k16.f32.f16.f16 "
        "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,"
        "%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,"
        "%48,%49,%50,%51,%52,%53,%54,%55}, %56, %57, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0][0]), "+f"(d[0][1]), "+f"(d[0][2]), "+f"(d[0][3]), "+f"(d[0][4]), "+f"(d[0][5]), "+f"(d[0][6]), "+f"(d[0][7]),
          "+f"(d[1][0]), "+f"(d[1][1]), "+f"(d[1][2]), "+f"(d[1][3]), "+f"(d[1][4]), "+f"(d[1][5]), "+f"(d[1][6]), "+f"(d[1][7]),
          "+f"(d[2][0]), "+f"(d[2][1]), "+f"(d[2][2]), "+f"(d[2][3]), "+f"(d[2][4]), "+f"(d[2][5]), "+f"(d[2][6]), "+f"(d[2][7]),
          "+f"(d[3][0]), "+f"(d[3][1]), "+f"(d[3][2]), "+f"(d[3][3]), "+f"(d[3][4]), "+f"(d[3][5]), "+f"(d[3][6]), "+f"(d[3][7]),
          "+f"(d[4][0]), "+f"(d[4][1]), "+f"(d[4][2]), "+f"(d[4][3]), "+f"(d[4][4]), "+f"(d[4][5]), "+f"(d[4][6]), "+f"(d[4][7]),
          "+f"(d[5][0]), "+f"(d[5][1]), "+f"(d[5][2]), "+f"(d[5][3]), "+f"(d[5][4]), "+f"(d[5][5]), "+f"(d[5][6]), "+f"(d[5][7]),
          "+f"(d[6][0]), "+f"(d[6][1]), "+f"(d[6][2]), "+f"(d[6][3]), "+f"(d[6][4]), "+f"(d[6][5]), "+f"(d[6][6]), "+f"(d[6][7])
        : "l"(adesc), "l"(bdesc), "r"(accumulate)
        : "memory");
}
template <> __device__ __forceinline__ void wg_mma_nd<8>(float (&d)[8][8], uint64_t adesc, uint64_t bdesc, int accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
        "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,"
        "%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,"
        "%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0][0]), "+f"(d[0][1]), "+f"(d[0][2]), "+f"(d[0][3]), "+f"(d[0][4]), "+f"(d[0][5]), "+f"(d[0][6]), "+f"(d[0][7]),
          "+f"(d[1][0]), "+f"(d[1][1]), "+f"(d[1][2]), "+f"(d[1][3]), "+f"(d[1][4]), "+f"(d[1][5]), "+f"(d[1][6]), "+f"(d[1][7]),
          "+f"(d[2][0]), "+f"(d[2][1]), "+f"(d[2][2]), "+f"(d[2][3]), "+f"(d[2][4]), "+f"(d[2][5]), "+f"(d[2][6]), "+f"(d[2][7]),
          "+f"(d[3][0]), "+f"(d[3][1]), "+f"(d[3][2]), "+f"(d[3][3]), "+f"(d[3][4]), "+f"(d[3][5]), "+f"(d[3][6]), "+f"(d[3][7]),
          "+f"(d[4][0]), "+f"(d[4][1]), "+f"(d[4][2]), "+f"(d[4][3]), "+f"(d[4][4]), "+f"(d[4][5]), "+f"(d[4][6]), "+f"(d[4][7]),
          "+f"(d[5][0]), "+f"(d[5][1]), "+f"(d[5][2]), "+f"(d[5][3]), "+f"(d[5][4]), "+f"(d[5][5]), "+f"(d[5][6]), "+f"(d[5][7]),
          "+f"(d[6][0]), "+f"(d[6][1]), "+f"(d[6][2]), "+f"(d[6][3]), "+f"(d[6][4]), "+f"(d[6][5]), "+f"(d[6][6]), "+f"(d[6][7]),
          "+f"(d[7][0]), "+f"(d[7][1]), "+f"(d[7][2]), "+f"(d[7][3]), "+f"(d[7][4]), "+f"(d[7][5]), "+f"(d[7][6]), "+f"(d[7][7])
        : "l"(adesc), "l"(bdesc), "r"(accumulate)
        : "memory");
}
template <> __device__ __forceinline__ void wg_mma_nd<9>(float (&d)[9][8], uint64_t adesc, uint64_t bdesc, int accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %74, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n144k16.f32.f16.f16 "
        "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,"
        "%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,"
        "%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63,%64,%65,%66,%67,%68,%69,%70,%71}, %72, %73, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0][0]), "+f"(d[0][1]), "+f"(d[0][2]), "+f"(d[0][3]), "+f"(d[0][4]), "+f"(d[0][5]), "+f"(d[0][6]), "+f"(d[0][7]),
          "+f"(d[1][0]), "+f"(d[1][1]), "+f"(d[1][2]), "+f"(d[1][3]), "+f"(d[1][4]), "+f"(d[1][5]), "+f"(d[1][6]), "+f"(d[1][7]),
          "+f"(d[2][0]), "+f"(d[2][1]), "+f"(d[2][2]), "+f"(d[2][3]), "+f"(d[2][4]), "+f"(d[2][5]), "+f"(d[2][6]), "+f"(d[2][7]),
          "+f"(d[3][0]), "+f"(d[3][1]), "+f"(d[3][2]), "+f"(d[3][3]), "+f"(d[3][4]), "+f"(d[3][5]), "+f"(d[3][6]), "+f"(d[3][7]),
          "+f"(d[4][0]), "+f"(d[4][1]), "+f"(d[4][2]), "+f"(d[4][3]), "+f"(d[4][4]), "+f"(d[4][5]), "+f"(d[4][6]), "+f"(d[4][7]),
          "+f"(d[5][0]), "+f"(d[5][1]), "+f"(d[5][2]), "+f"(d[5][3]), "+f"(d[5][4]), "+f"(d[5][5]), "+f"(d[5][6]), "+f"(d[5][7]),
          "+f"(d[6][0]), "+f"(d[6][1]), "+f"(d[6][2]), "+f"(d[6][3]), "+f"(d[6][4]), "+f"(d[6][5]), "+f"(d[6][6]), "+f"(d[6][7]),
          "+f"(d[7][0]), "+f"(d[7][1]), "+f"(d[7][2]), "+f"(d[7][3]), "+f"(d[7][4]), "+f"(d[7][5]), "+f"(d[7][6]), "+f"(d[7][7]),
          "+f"(d[8][0]), "+f"(d[8][1]), "+f"(d[8][2]), "+f"(d[8][3]), "+f"(d[8][4]), "+f"(d[8][5]), "+f"(d[8][6]), "+f"(d[8][7])
        : "l"(adesc), "l"(bdesc), "r"(accumulate)
        : "memory");
}
template <> __device__ __forceinline__ void wg_mma_nd<10>(float (&d)[10][8], uint64_t adesc, uint64_t bdesc, int accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %82, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n160k16.f32.f16.f16 "
        "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,"
        "%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,"
        "%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63,%64,%65,%66,%67,%68,%69,%70,%71,"
        "%72,%73,%74,%75,%76,%77,%78,%79}, %80, %81, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0][0]), "+f"(d[0][1]), "+f"(d[0][2]), "+f"(d[0][3]), "+f"(d[0][4]), "+f"(d[0][5]), "+f"(d[0][6]), "+f"(d[0][7]),
          "+f"(d[1][0]), "+f"(d[1][1]), "+f"(d[1][2]), "+f"(d[1][3]), "+f"(d[1][4]), "+f"(d[1][5]), "+f"(d[1][6]), "+f"(d[1][7]),
          "+f"(d[2][0]), "+f"(d[2][1]), "+f"(d[2][2]), "+f"(d[2][3]), "+f"(d[2][4]), "+f"(d[2][5]), "+f"(d[2][6]), "+f"(d[2][7]),
          "+f"(d[3][0]), "+f"(d[3][1]), "+f"(d[3][2]), "+f"(d[3][3]), "+f"(d[3][4]), "+f"(d[3][5]), "+f"(d[3][6]), "+f"(d[3][7]),
          "+f"(d[4][0]), "+f"(d[4][1]), "+f"(d[4][2]), "+f"(d[4][3]), "+f"(d[4][4]), "+f"(d[4][5]), "+f"(d[4][6]), "+f"(d[4][7]),
          "+f"(d[5][0]), "+f"(d[5][1]), "+f"(d[5][2]), "+f"(d[5][3]), "+f"(d[5][4]), "+f"(d[5][5]), "+f"(d[5][6]), "+f"(d[5][7]),
          "+f"(d[6][0]), "+f"(d[6][1]), "+f"(d[6][2]), "+f"(d[6][3]), "+f"(d[6][4]), "+f"(d[6][5]), "+f"(d[6][6]), "+f"(d[6][7]),
          "+f"(d[7][0]), "+f"(d[7][1]), "+f"(d[7][2]), "+f"(d[7][3]), "+f"(d[7][4]), "+f"(d[7][5]), "+f"(d[7][6]), "+f"(d[7][7]),
          "+f"(d[8][0]), "+f"(d[8][1]), "+f"(d[8][2]), "+f"(d[8][3]), "+f"(d[8][4]), "+f"(d[8][5]), "+f"(d[8][6]), "+f"(d[8][7]),
          "+f"(d[9][0]), "+f"(d[9][1]), "+f"(d[9][2]), "+f"(d[9][3]), "+f"(d[9][4]), "+f"(d[9][5]), "+f"(d[9][6]), "+f"(d[9][7])
        : "l"(adesc), "l"(bdesc), "r"(accumulate)
        : "memory");
}

template <int NC>
__device__ __forceinline__ void wg_mma_n(float (&acc)[NC][8], uint32_t a_addr, uint32_t b_addr, int accumulate = 1) {
    wg_mma_nd<NC>(acc, wg_desc_sw128(a_addr), wg_desc_sw128(b_addr), accumulate);
}

// Accumulator fragment of m64n16 per thread (warp w = warp % 4 of the warpgroup): value pair i (0..3) of chunk c is
// acc[c][2i], acc[c][2i+1] at row 16w + lane/4 + 8*(i&1), columns 16c + 8*(i>>1) + 2*(lane&3) + {0,1}.
__device__ __forceinline__ int frag_row(int wq, int lane, int i) { return 16 * wq + (lane >> 2) + 8 * (i & 1); }
__device__ __forceinline__ int frag_col(int lane, int i) { return 8 * (i >> 1) + 2 * (lane & 3); }

// Projection epilogue of value pairs i of the NC chunks of an accumulator fragment (one pixel, NHWC element offset
// off): out = fp16(acc + bias (+ residual)), the bias and residual added in fp32 and one rounding at the end.
template <int NC>
__device__ __forceinline__ void proj_store_row(__half* out, const __half* residual, size_t off, int Co,
                                               const float (&acc)[NC][8], int i, const float* bias, int lane) {
#pragma unroll
    for (int c = 0; c < NC; ++c) {
        const int co = c * 16 + frag_col(lane, i);
        if (co >= Co) continue;
        float2 v = make_float2(acc[c][2 * i] + bias[co], acc[c][2 * i + 1] + bias[co + 1]);
        if (residual) {
            const float2 f = __half22float2(*reinterpret_cast<const __half2*>(residual + off + co));
            v.x += f.x;
            v.y += f.y;
        }
        *reinterpret_cast<__half2*>(out + off + co) = __float22half2_rn(v);
    }
}

__device__ __forceinline__ __half2 relu6_h2(__half2 v) {
    return __hmin2(__hmax2(v, __floats2half2_rn(0.f, 0.f)), __floats2half2_rn(6.f, 6.f));
}

// Expansion epilogue: relu6(fp16(v)) for v = acc + bias in fp32.  The clamp runs on the rounded, packed pair and is
// exact: rounding to fp16 is monotonic and 0 and 6 are fp16 values, so clamping commutes with it.
__device__ __forceinline__ __half2 expand_relu6(float v0, float v1) { return relu6_h2(__floats2half2_rn(v0, v1)); }

__device__ __forceinline__ float act_apply(float v, int act) {
    if (act == LP_ACT_RELU) return fmaxf(v, 0.f);
    if (act == LP_ACT_RELU6) return fminf(fmaxf(v, 0.f), 6.f);
    return v;
}

// Fusion-deconv epilogue activation (both deconv kernels): ReLU in the network, none for the raw sums the BN
// recalibration pass takes its batch statistics of.
template <int ACT>
__device__ __forceinline__ float deconv_act(float v) {
    return ACT == LP_ACT_RELU ? fmaxf(v, 0.f) : v;
}

#endif  // __CUDACC__
}  // namespace lp
