// Library state of the C ABI: thread-local error string, launch counter, device check, SM count and its limit,
// tensor-map construction through the driver entry point (no link-time libcuda dependency).
#include <atomic>
#include <cstdarg>
#include <cstring>
#include <mutex>

#include "common.cuh"
#include "../../include/litepose_b200_debug.h"

namespace lp {

static thread_local char g_err[512] = "";
static std::atomic<uint64_t> g_launches{0};

void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

int cuda_fail(cudaError_t e, const char* what) {
    set_error("CUDA error %d (%s) in %s", (int)e, cudaGetErrorString(e), what);
    return LP_ERR_CUDA;
}

void count_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode() {
    static PFN_encodeTiled fn = nullptr;
    static std::once_flag once;
    std::call_once(once, [] {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<PFN_encodeTiled>(p);
    });
    return fn;
}

int make_tmap(CUtensorMap* map, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
              const uint32_t* box, CUtensorMapSwizzle swz, CUtensorMapDataType dt) {
    PFN_encodeTiled enc = get_encode();
    if (!enc) {
        set_error("cuTensorMapEncodeTiled entry point unavailable (driver too old?)");
        return LP_ERR_CUDA;
    }
    // cuTensorMapEncodeTiled is a DRIVER entry point: it needs a context current on the calling thread.  A thread that
    // has not made a runtime call yet (an nn.DataParallel worker whose device is already the current one, so torch never
    // calls cudaSetDevice in it) has none and the encode fails with CUDA_ERROR_INVALID_CONTEXT: bind the primary context
    // of the current device once per thread.
    static thread_local bool ctx_bound = false;
    if (!ctx_bound) {
        cudaFree(nullptr);
        ctx_bound = true;
    }
    if (reinterpret_cast<uintptr_t>(base) & 15) {
        set_error("tensor map base address must be 16-byte aligned");
        return LP_ERR_ALIGN;
    }
    cuuint64_t gd[5];
    cuuint64_t gs[4];
    cuuint32_t bx[5], es[5];
    for (int i = 0; i < rank; ++i) {
        gd[i] = dims[i];
        bx[i] = box[i];
        es[i] = 1;
    }
    for (int i = 0; i < rank - 1; ++i) {
        gs[i] = strides_bytes[i];
        if (gs[i] & 15) {
            set_error("tensor map stride %d (%llu bytes) must be a multiple of 16", i, (unsigned long long)gs[i]);
            return LP_ERR_ALIGN;
        }
    }
    CUresult r = enc(map, dt, (cuuint32_t)rank, const_cast<void*>(base), gd, gs, bx, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     swz, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r == CUDA_ERROR_INVALID_CONTEXT) {       // e.g. the thread's context was popped by another library: bind and retry
        cudaFree(nullptr);
        r = enc(map, dt, (cuuint32_t)rank, const_cast<void*>(base), gd, gs, bx, es, CU_TENSOR_MAP_INTERLEAVE_NONE, swz,
                CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    }
    if (r != CUDA_SUCCESS) {
        set_error("cuTensorMapEncodeTiled failed (CUresult %d): rank %d dims [%llu,%llu,%llu,%llu] box [%u,%u,%u,%u]",
                  (int)r, rank, (unsigned long long)gd[0], (unsigned long long)(rank > 1 ? gd[1] : 0),
                  (unsigned long long)(rank > 2 ? gd[2] : 0), (unsigned long long)(rank > 3 ? gd[3] : 0), bx[0],
                  rank > 1 ? bx[1] : 0, rank > 2 ? bx[2] : 0, rank > 3 ? bx[3] : 0);
        return LP_ERR_CUDA;
    }
    return LP_OK;
}

int make_tmap_nhwc(CUtensorMap* map, const void* x, int N, int H, int W, int C, int box_c, int box_w, int box_h,
                   CUtensorMapSwizzle swz) {
    uint64_t dims[4] = {(uint64_t)C, (uint64_t)W, (uint64_t)H, (uint64_t)N};
    uint64_t strides[3] = {(uint64_t)C * 2, (uint64_t)W * C * 2, (uint64_t)H * W * C * 2};
    uint32_t box[4] = {(uint32_t)box_c, (uint32_t)box_w, (uint32_t)box_h, 1u};
    return make_tmap(map, x, 4, dims, strides, box, swz);
}

int make_tmap_rows64(CUtensorMap* map, const void* w, int rows, int box_k, int box_rows, CUtensorMapSwizzle swz) {
    uint64_t dims[2] = {64u, (uint64_t)rows};
    uint64_t strides[1] = {128u};
    uint32_t box[2] = {(uint32_t)box_k, (uint32_t)box_rows};
    return make_tmap(map, w, 2, dims, strides, box, swz);
}

int make_tmap_taps(CUtensorMap* map, const void* w, int taps, int C) {
    uint64_t dims[2] = {(uint64_t)C, (uint64_t)taps};
    uint64_t strides[1] = {(uint64_t)C * 2};
    uint32_t box[2] = {32u, (uint32_t)taps};
    return make_tmap(map, w, 2, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_NONE);
}

// lp_set_sm_limit: 0 = no limit.  Process-wide, so a pipeline's worker threads size their grids from the same count.
static std::atomic<int> g_sm_limit{0};

int num_sms() {
    static thread_local int cached_dev = -1;
    static thread_local int cached = 0;
    int dev = 0;
    int v = 132;
    if (cudaGetDevice(&dev) == cudaSuccess) {
        if (dev != cached_dev) {
            int a = 0;
            if (cudaDeviceGetAttribute(&a, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || a <= 0) a = 132;
            cached = a;
            cached_dev = dev;
        }
        v = cached;
    }
    const int limit = g_sm_limit.load(std::memory_order_relaxed);
    return limit > 0 && limit < v ? limit : v;
}

}  // namespace lp

extern "C" int lp_version(void) { return 100; }

extern "C" const char* lp_last_error(void) { return lp::g_err; }

extern "C" int lp_device_check(void) {
    int dev = 0, major = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return lp::cuda_fail(e, "cudaGetDevice");
    e = cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev);
    if (e != cudaSuccess) return lp::cuda_fail(e, "cudaDeviceGetAttribute");
    if (major != 9) {
        lp::set_error("litepose_b200 kernels are built for sm_90a only; device %d has compute capability major %d", dev,
                      major);
        return LP_ERR_ARCH;
    }
    return LP_OK;
}

extern "C" uint64_t lp_launch_count(void) { return lp::g_launches.load(); }
extern "C" void lp_reset_launch_count(void) { lp::g_launches.store(0); }

extern "C" void lp_set_sm_limit(int n) { lp::g_sm_limit.store(n > 0 ? n : 0, std::memory_order_relaxed); }
extern "C" int lp_get_sm_limit(void) { return lp::num_sms(); }
