// Train-mode BatchNorm2d on NCHW activations, with the ReLU / ReLU6 that follows it fused: forward (batch statistics,
// running-statistics update, normalise + activation) and backward (dx, dgamma, dbeta), x / y / dy / dx fp32 or fp16,
// gamma, beta, the running and the saved statistics fp32.  These are the BatchNorms of pose_mobilenet, pose_simplenet
// and pose_supermobilenet in the layout the module tree trains in (litepose_b200.train_bn).
//
// Arithmetic (tests/bn_nchw_train_emul.py restates it bit for bit).  M = N * H * W values per channel; channel c's
// values are numbered j = n * HW + p (image n, pixel p of the plane).
//   reduction  bnt_partial: CTA (range r, channel c) takes j in [r * BNT_RANGE, (r + 1) * BNT_RANGE), those below M.
//              Thread t adds the values j = r * BNT_RANGE + t + 256 i, i = 0, 1, ..., in fp64 from +0 (a pair of sums);
//              each warp folds its lanes with the butterfly v += shfl_xor(v, 16, 8, 4, 2, 1) (lane 0's value is
//              taken) and the eight warp sums are added in warp order from warp 0's, in fp64:
//              part[2 * (r * C + c) + {0, 1}].  The ranges depend on the shape only.
//     forward:  the pair is (x, x * x); an fp32 value and its square are exact in fp64.
//     backward: v = fmaf(x, scale, shift) (the forward's pre-activation, bit for bit), the mask m(v) is ReLU:
//               !(v <= 0), ReLU6: !(v <= 0) && !(v >= 6), none: 1; g = m ? dy : +0 (a masked NaN gradient is 0, as
//               threshold_backward / hardtanh_backward select it); xhat = fp32(fp32(x - mean) * invstd); the pair is
//               (g, g * xhat), the product exact in fp64.
//   forward merge (bnt_fwd_merge): per channel, bn_merge_channel (bn_merge.cuh, shared with lp_bn_stats_f16) adds the
//              ranges in order and derives mean, invstd, scale, shift and the new running statistics; the running
//              statistics are updated in place and saved[4][C] = (mean, invstd, scale, shift).  A channel whose mean
//              is not finite (it holds an inf or NaN) gets NaN invstd, scale, shift and new running variance, as
//              F.batch_norm's variance is NaN there.
//   forward apply: y = act(fmaf(x, scale, shift)) in fp32, rounded once to y's dtype.  act keeps NaN: ReLU is
//              (v <= 0 ? +0 : v), ReLU6 then (v >= 6 ? 6 : v), so a NaN stays NaN as under F.relu / F.relu6.
//   backward merge (bnt_bwd_merge): per channel, in fp64 in range order: Sg = sum g, Sgx = sum g * xhat;
//              dbeta = fp32(Sg), dgamma = fp32(Sgx), mg = fp32(Sg / M), mgx = fp32(Sgx / M),
//              k = fp32(gamma * invstd) (exact product, one rounding).
//   backward apply: dx = k * fmaf(-xhat, mgx, g - mg): d = fp32(g - mg), d = fmaf(-xhat, mgx, d), dx = fp32(k * d),
//              rounded once more to dx's dtype (PyTorch's train-mode gamma * invstd * (g - mean(g) - xhat * mean(g xhat))).
// Everything is a fixed function of the shape and the inputs: no atomics, no dependence on the SM count.
#include "bn_merge.cuh"
#include "../../include/litepose_b200_train_bn.h"

namespace lp {

constexpr int BNT_THREADS = 256;
constexpr int BNT_RANGE = 8192;             // values of one channel per reduction CTA (32 per thread)
constexpr int BNT_APPLY = BNT_THREADS * 4;  // pixels of one plane per apply CTA (4 per thread)

__device__ __forceinline__ float bnt_ld(const float* p) { return __ldg(p); }
__device__ __forceinline__ float bnt_ld(const __half* p) { return __half2float(__ldg(p)); }
__device__ __forceinline__ void bnt_st(float* p, float v) { *p = v; }
__device__ __forceinline__ void bnt_st(__half* p, float v) { *p = __float2half_rn(v); }

template <int ACT>
__device__ __forceinline__ float bnt_act(float v) {
    if (ACT != LP_ACT_NONE) v = v <= 0.f ? 0.f : v;
    if (ACT == LP_ACT_RELU6) v = v >= 6.f ? 6.f : v;
    return v;
}

template <int ACT>
__device__ __forceinline__ bool bnt_mask(float v) {
    if (ACT == LP_ACT_RELU) return !(v <= 0.f);
    if (ACT == LP_ACT_RELU6) return !(v <= 0.f) && !(v >= 6.f);
    return true;
}

// GRAD = false: sums of (x, x^2).  GRAD = true: sums of (g, g * xhat); saved = [mean, invstd, scale, shift][C].
template <typename T, bool GRAD, int ACT>
__global__ void __launch_bounds__(BNT_THREADS)
bnt_partial(const T* __restrict__ x, const T* __restrict__ dy, const float* __restrict__ saved, int C, int HW,
            long long M, double* __restrict__ part) {
    __shared__ double red[BNT_THREADS / 32][2];
    const int c = (int)(blockIdx.x % (unsigned)C);
    const long long r = blockIdx.x / (unsigned)C;
    float mean = 0.f, invstd = 0.f, scale = 0.f, shift = 0.f;
    if (GRAD) {
        mean = saved[c];
        invstd = saved[C + c];
        scale = saved[2 * C + c];
        shift = saved[3 * C + c];
    }
    const long long j0 = r * BNT_RANGE + threadIdx.x;
    const long long j1 = min(r * BNT_RANGE + BNT_RANGE, M);
    // (n, p) of j, stepped by BNT_THREADS without a division per value
    long long n = j0 / HW;
    int p = (int)(j0 - n * HW);
    const int dn = BNT_THREADS / HW, dp = BNT_THREADS % HW;
    const size_t cs = (size_t)C * HW;
    double a1 = 0.0, a2 = 0.0;
    constexpr int U = 8;                     // loads in flight; the additions stay in j order
    for (long long j = j0; j < j1; j += U * BNT_THREADS) {
        float va[U], vd[U];
        bool in[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
            in[u] = j + (long long)u * BNT_THREADS < j1;
            const size_t o = (size_t)n * cs + (size_t)c * HW + p;
            va[u] = in[u] ? bnt_ld(x + o) : 0.f;
            if (GRAD) vd[u] = in[u] ? bnt_ld(dy + o) : 0.f;
            n += dn;
            p += dp;
            if (p >= HW) {
                p -= HW;
                ++n;
            }
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
            if (!in[u]) continue;
            if (GRAD) {
                const float g = bnt_mask<ACT>(fmaf(va[u], scale, shift)) ? vd[u] : 0.f;
                const float xh = __fmul_rn(__fsub_rn(va[u], mean), invstd);
                a1 = __dadd_rn(a1, (double)g);
                a2 = __dadd_rn(a2, __dmul_rn((double)g, (double)xh));
            } else {
                const double d = va[u];
                a1 = __dadd_rn(a1, d);
                a2 = __dadd_rn(a2, __dmul_rn(d, d));
            }
        }
    }
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) {
        a1 = __dadd_rn(a1, __shfl_xor_sync(0xffffffffu, a1, o));
        a2 = __dadd_rn(a2, __shfl_xor_sync(0xffffffffu, a2, o));
    }
    const int lane = threadIdx.x & 31, wq = threadIdx.x >> 5;
    if (lane == 0) {
        red[wq][0] = a1;
        red[wq][1] = a2;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        double t1 = red[0][0], t2 = red[0][1];
#pragma unroll
        for (int w = 1; w < BNT_THREADS / 32; ++w) {
            t1 = __dadd_rn(t1, red[w][0]);
            t2 = __dadd_rn(t2, red[w][1]);
        }
        const size_t o = (size_t)r * C + c;
        part[2 * o] = t1;
        part[2 * o + 1] = t2;
    }
}

__global__ void __launch_bounds__(128)
bnt_fwd_merge(const double* __restrict__ part, int nparts, long long M, int C, const float* __restrict__ gamma,
              const float* __restrict__ beta, float* running_mean, float* running_var, double momentum, double eps,
              float* __restrict__ saved) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C) return;
    BnMerged r = bn_merge_channel(part, nparts, M, C, c, gamma[c], beta[c], running_mean[c], running_var[c],
                                  momentum, eps);
    if (!isfinite(r.mean)) {
        // an inf or NaN in the channel: F.batch_norm's variance is NaN there, so the whole channel is NaN and so is
        // the new running variance (bn_merge_channel's max(var, 0) would turn that NaN into 0)
        r.invstd = r.scale = r.shift = r.new_var = __int_as_float(0x7fffffff);
    }
    running_mean[c] = r.new_mean;
    running_var[c] = r.new_var;
    saved[c] = r.mean;
    saved[C + c] = r.invstd;
    saved[2 * C + c] = r.scale;
    saved[3 * C + c] = r.shift;
}

// coef[3][C] = (k, mg, mgx) for the apply pass; dgamma / dbeta may be null (not needed)
__global__ void __launch_bounds__(128)
bnt_bwd_merge(const double* __restrict__ part, int nparts, long long M, int C, const float* __restrict__ gamma,
              const float* __restrict__ saved, float* __restrict__ dgamma, float* __restrict__ dbeta,
              float* __restrict__ coef) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C) return;
    double t1 = part[2 * c], t2 = part[2 * c + 1];
    for (int i = 1; i < nparts; ++i) {
        const size_t o = (size_t)i * C + c;
        t1 = __dadd_rn(t1, part[2 * o]);
        t2 = __dadd_rn(t2, part[2 * o + 1]);
    }
    if (dbeta) dbeta[c] = __double2float_rn(t1);
    if (dgamma) dgamma[c] = __double2float_rn(t2);
    const double m = (double)M;
    coef[c] = __double2float_rn(__dmul_rn((double)gamma[c], (double)saved[C + c]));
    coef[C + c] = __double2float_rn(__ddiv_rn(t1, m));
    coef[2 * C + c] = __double2float_rn(__ddiv_rn(t2, m));
}

// CTA (plane n * C + c, chunk): pixels chunk * BNT_APPLY + t + 256 i, i = 0..3
template <typename T, int ACT>
__global__ void __launch_bounds__(BNT_THREADS)
bnt_fwd_apply(const T* __restrict__ x, const float* __restrict__ saved, T* __restrict__ y, int C, int HW) {
    const size_t plane = blockIdx.x;
    const int c = (int)(plane % (size_t)C);
    const float scale = saved[2 * C + c], shift = saved[3 * C + c];
    const T* xp = x + plane * HW;
    T* yp = y + plane * HW;
    const int p0 = blockIdx.y * BNT_APPLY + threadIdx.x;
    float v[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int p = p0 + i * BNT_THREADS;
        v[i] = p < HW ? bnt_ld(xp + p) : 0.f;
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int p = p0 + i * BNT_THREADS;
        if (p < HW) bnt_st(yp + p, bnt_act<ACT>(fmaf(v[i], scale, shift)));
    }
}

template <typename T, int ACT>
__global__ void __launch_bounds__(BNT_THREADS)
bnt_bwd_apply(const T* __restrict__ x, const T* __restrict__ dy, const float* __restrict__ saved,
              const float* __restrict__ coef, T* __restrict__ dx, int C, int HW) {
    const size_t plane = blockIdx.x;
    const int c = (int)(plane % (size_t)C);
    const float mean = saved[c], invstd = saved[C + c], scale = saved[2 * C + c], shift = saved[3 * C + c];
    const float k = coef[c], mg = coef[C + c], mgx = coef[2 * C + c];
    const size_t base = plane * HW;
    const int p0 = blockIdx.y * BNT_APPLY + threadIdx.x;
    float vx[4], vd[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int p = p0 + i * BNT_THREADS;
        vx[i] = p < HW ? bnt_ld(x + base + p) : 0.f;
        vd[i] = p < HW ? bnt_ld(dy + base + p) : 0.f;
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int p = p0 + i * BNT_THREADS;
        if (p >= HW) continue;
        const float g = bnt_mask<ACT>(fmaf(vx[i], scale, shift)) ? vd[i] : 0.f;
        const float xh = __fmul_rn(__fsub_rn(vx[i], mean), invstd);
        float d = __fsub_rn(g, mg);
        d = __fmaf_rn(-xh, mgx, d);
        bnt_st(dx + base + p, __fmul_rn(k, d));
    }
}

struct BntShape {
    long long M;
    int HW, nparts, chunks;
};

static int bnt_check(const char* fn, int N, int C, int H, int W, int act, int dtype, BntShape* sh) {
    LP_CHECK_ARG(dtype == LP_DT_F32 || dtype == LP_DT_F16, "%s: dtype %d (LP_DT_F32 or LP_DT_F16)", fn, dtype);
    LP_CHECK_ARG(act >= LP_ACT_NONE && act <= LP_ACT_RELU6, "%s: act %d (LP_ACT_NONE, LP_ACT_RELU or LP_ACT_RELU6)", fn,
                 act);
    LP_CHECK_ARG(N >= 1 && C >= 0 && H >= 1 && W >= 1, "%s: bad shape N=%d C=%d H=%d W=%d", fn, N, C, H, W);
    LP_CHECK_ARG((long long)H * W <= 0x7fffffffLL, "%s: plane %d x %d too large", fn, H, W);
    sh->HW = H * W;
    sh->M = (long long)N * sh->HW;
    LP_CHECK_ARG(sh->M >= 2, "%s: one value per channel (N*H*W = %lld): train-mode BatchNorm needs more than one", fn,
                 sh->M);
    const long long nparts = (sh->M + BNT_RANGE - 1) / BNT_RANGE;
    sh->nparts = (int)(nparts < 0x7fffffffLL ? nparts : 0x7fffffffLL);
    sh->chunks = (sh->HW + BNT_APPLY - 1) / BNT_APPLY;
    LP_CHECK_ARG((long long)N * C <= 0x7fffffffLL && nparts * C <= 0x7fffffffLL && sh->chunks <= 65535,
                 "%s: shape N=%d C=%d H=%d W=%d exceeds the launch grid", fn, N, C, H, W);
    return LP_OK;
}

static size_t bnt_ws_bytes(const BntShape& sh, int C) {
    return (size_t)sh.nparts * C * 2 * sizeof(double) + (size_t)3 * C * sizeof(float);
}

static int bnt_check_ws(const char* fn, const BntShape& sh, int C, const void* ws, size_t bytes) {
    LP_CHECK_ARG(ws, "%s: null workspace", fn);
    if (bytes < bnt_ws_bytes(sh, C)) {
        set_error("%s: workspace of %zu bytes, %zu needed", fn, bytes, bnt_ws_bytes(sh, C));
        return LP_ERR_CAPACITY;
    }
    if (reinterpret_cast<uintptr_t>(ws) & 7) {
        set_error("%s: workspace must be 8-byte aligned", fn);
        return LP_ERR_ALIGN;
    }
    return LP_OK;
}

static bool bnt_misaligned(const void* p, size_t a) { return (reinterpret_cast<uintptr_t>(p) & (a - 1)) != 0; }

}  // namespace lp

using namespace lp;

#define LP_BNT_ACT(act, F)                      \
    switch (act) {                              \
        case LP_ACT_RELU: F(LP_ACT_RELU); break;   \
        case LP_ACT_RELU6: F(LP_ACT_RELU6); break; \
        default: F(LP_ACT_NONE); break;         \
    }

extern "C" size_t lp_bn_nchw_workspace_bytes(int N, int C, int H, int W) {
    BntShape sh;
    if (bnt_check("lp_bn_nchw_workspace_bytes", N, C, H, W, LP_ACT_NONE, LP_DT_F32, &sh) != LP_OK) return 0;
    return bnt_ws_bytes(sh, C);
}

template <typename T>
static void bnt_stats_launch(const void* x, double* part, const BntShape& sh, int C, cudaStream_t st) {
    bnt_partial<T, false, LP_ACT_NONE><<<(unsigned)((size_t)sh.nparts * C), BNT_THREADS, 0, st>>>(
        reinterpret_cast<const T*>(x), nullptr, nullptr, C, sh.HW, sh.M, part);
}

template <typename T>
static void bnt_apply_fwd_launch(const void* x, void* y, const float* saved, const BntShape& sh, int N, int C,
                                 int act, cudaStream_t st) {
    const dim3 grid((unsigned)((size_t)N * C), (unsigned)sh.chunks);
    const T* xt = reinterpret_cast<const T*>(x);
    T* yt = reinterpret_cast<T*>(y);
#define LP_BNT_FA(A) bnt_fwd_apply<T, A><<<grid, BNT_THREADS, 0, st>>>(xt, saved, yt, C, sh.HW)
    LP_BNT_ACT(act, LP_BNT_FA)
#undef LP_BNT_FA
}

extern "C" int lp_bn_nchw_fwd(const void* x, const float* gamma, const float* beta, float* running_mean,
                              float* running_var, double momentum, double eps, void* y, float* saved, int N, int C,
                              int H, int W, int act, int dtype, void* workspace, size_t workspace_bytes,
                              lp_stream_t stream) {
    const char* fn = "lp_bn_nchw_fwd";
    BntShape sh;
    int rc = bnt_check(fn, N, C, H, W, act, dtype, &sh);
    if (rc != LP_OK) return rc;
    LP_CHECK_ARG(momentum >= 0.0 && momentum <= 1.0 && eps >= 0.0, "%s: bad momentum %g / eps %g", fn, momentum, eps);
    if (C == 0) return LP_OK;
    LP_CHECK_ARG(x && gamma && beta && running_mean && running_var && y && saved, "%s: null pointer", fn);
    rc = bnt_check_ws(fn, sh, C, workspace, workspace_bytes);
    if (rc != LP_OK) return rc;
    const size_t el = dtype == LP_DT_F32 ? 4 : 2;
    if (bnt_misaligned(x, el) || bnt_misaligned(y, el) || bnt_misaligned(gamma, 4) || bnt_misaligned(beta, 4) ||
        bnt_misaligned(running_mean, 4) || bnt_misaligned(running_var, 4) || bnt_misaligned(saved, 4)) {
        set_error("%s: pointers must be aligned to their element", fn);
        return LP_ERR_ALIGN;
    }
    cudaStream_t st = (cudaStream_t)stream;
    double* part = reinterpret_cast<double*>(workspace);
    if (dtype == LP_DT_F32) bnt_stats_launch<float>(x, part, sh, C, st);
    else bnt_stats_launch<__half>(x, part, sh, C, st);
    LP_LAUNCH_CHECK("bnt_partial");
    bnt_fwd_merge<<<(C + 127) / 128, 128, 0, st>>>(part, sh.nparts, sh.M, C, gamma, beta, running_mean, running_var,
                                                   momentum, eps, saved);
    LP_LAUNCH_CHECK("bnt_fwd_merge");
    if (dtype == LP_DT_F32) bnt_apply_fwd_launch<float>(x, y, saved, sh, N, C, act, st);
    else bnt_apply_fwd_launch<__half>(x, y, saved, sh, N, C, act, st);
    LP_LAUNCH_CHECK("bnt_fwd_apply");
    return LP_OK;
}

template <typename T>
static void bnt_grad_sums_launch(const void* x, const void* dy, const float* saved, double* part, const BntShape& sh,
                                 int C, int act, cudaStream_t st) {
    const unsigned grid = (unsigned)((size_t)sh.nparts * C);
    const T* xt = reinterpret_cast<const T*>(x);
    const T* dt = reinterpret_cast<const T*>(dy);
#define LP_BNT_BP(A) bnt_partial<T, true, A><<<grid, BNT_THREADS, 0, st>>>(xt, dt, saved, C, sh.HW, sh.M, part)
    LP_BNT_ACT(act, LP_BNT_BP)
#undef LP_BNT_BP
}

template <typename T>
static void bnt_apply_bwd_launch(const void* x, const void* dy, const float* saved, const float* coef, void* dx,
                                 const BntShape& sh, int N, int C, int act, cudaStream_t st) {
    const dim3 grid((unsigned)((size_t)N * C), (unsigned)sh.chunks);
    const T* xt = reinterpret_cast<const T*>(x);
    const T* dt = reinterpret_cast<const T*>(dy);
    T* xo = reinterpret_cast<T*>(dx);
#define LP_BNT_BA(A) bnt_bwd_apply<T, A><<<grid, BNT_THREADS, 0, st>>>(xt, dt, saved, coef, xo, C, sh.HW)
    LP_BNT_ACT(act, LP_BNT_BA)
#undef LP_BNT_BA
}

extern "C" int lp_bn_nchw_bwd(const void* x, const void* dy, const float* gamma, const float* saved, void* dx,
                              float* dgamma, float* dbeta, int N, int C, int H, int W, int act, int dtype,
                              void* workspace, size_t workspace_bytes, lp_stream_t stream) {
    const char* fn = "lp_bn_nchw_bwd";
    BntShape sh;
    int rc = bnt_check(fn, N, C, H, W, act, dtype, &sh);
    if (rc != LP_OK) return rc;
    if (C == 0 || !(dx || dgamma || dbeta)) return LP_OK;
    LP_CHECK_ARG(x && dy && gamma && saved, "%s: null pointer", fn);
    rc = bnt_check_ws(fn, sh, C, workspace, workspace_bytes);
    if (rc != LP_OK) return rc;
    const size_t el = dtype == LP_DT_F32 ? 4 : 2;
    if (bnt_misaligned(x, el) || bnt_misaligned(dy, el) || bnt_misaligned(dx, el) || bnt_misaligned(gamma, 4) ||
        bnt_misaligned(saved, 4) || bnt_misaligned(dgamma, 4) || bnt_misaligned(dbeta, 4)) {
        set_error("%s: pointers must be aligned to their element", fn);
        return LP_ERR_ALIGN;
    }
    cudaStream_t st = (cudaStream_t)stream;
    double* part = reinterpret_cast<double*>(workspace);
    float* coef = reinterpret_cast<float*>(part + (size_t)sh.nparts * C * 2);
    if (dtype == LP_DT_F32) bnt_grad_sums_launch<float>(x, dy, saved, part, sh, C, act, st);
    else bnt_grad_sums_launch<__half>(x, dy, saved, part, sh, C, act, st);
    LP_LAUNCH_CHECK("bnt_partial (backward)");
    bnt_bwd_merge<<<(C + 127) / 128, 128, 0, st>>>(part, sh.nparts, sh.M, C, gamma, saved, dgamma, dbeta, coef);
    LP_LAUNCH_CHECK("bnt_bwd_merge");
    if (!dx) return LP_OK;
    if (dtype == LP_DT_F32) bnt_apply_bwd_launch<float>(x, dy, saved, coef, dx, sh, N, C, act, st);
    else bnt_apply_bwd_launch<__half>(x, dy, saved, coef, dx, sh, N, C, act, st);
    LP_LAUNCH_CHECK("bnt_bwd_apply");
    return LP_OK;
}
