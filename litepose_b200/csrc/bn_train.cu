// Training-mode BatchNorm on NHWC fp16 activations: batch statistics and the normalise + activation pass of the
// super-network's BN recalibration (reference calibrate_test.py:58-61: model.train(); model(images)).
//
// lp_bn_stats_f16 reduces an [M, C] tensor in two kernels, with no atomics, so the result is the same bits on every run:
//   bn_stats_partial  CTA (r, t) takes pixels [r * BN_ROWS, (r + 1) * BN_ROWS) and channel vectors [t * VT, t * VT + VT)
//                     (VT = min(C / 8, 32) vectors of 8 channels).  Thread lane l = threadIdx.x / VT accumulates the
//                     pixels r * BN_ROWS + l + k * RL, k = 0, 1, ... (RL = 256 / VT lanes) in fp64, sum and sum of squares
//                     from +0; the lanes are then added in lane order 0, 1, ..., RL - 1, starting from lane 0's sums.
//   bn_stats_merge    one thread per channel adds the CTA partials in pixel-range order r = 0, 1, ..., starting from
//                     range 0's, then derives in fp64, every operation rounded once (no contraction), as
//                     bn_merge_channel (bn_merge.cuh) states:
//                       mean = S1 / M, var = max(S2 / M - mean * mean, 0), var_unbiased = var * M / (M - 1),
//                       s = gamma / sqrt(var + eps), scale = fp32(s), shift = fp32(beta - mean * s),
//                       new running = fp32((1 - momentum) * running + momentum * stat) for (mean, var_unbiased),
//                     and sets *nonfinite to 1 when one of scale, shift or the new running values is not finite.
// fp16 values and their squares are exact in fp64, so each addition is the only rounding of its step.
//
// lp_bn_apply_f16: y = act(fmaf(x, scale, shift)) (+ residual) in fp32, one rounding to fp16, 8 channels per 16-byte
// vector.  act: ReLU is (v > 0 ? v : +0), ReLU6 then (v < 6 ? v : 6); y may alias x.
#include "bn_merge.cuh"

namespace lp {

constexpr int BN_ROWS = 2048;      // pixels per statistics CTA
constexpr int BN_THREADS = 256;
constexpr int BN_MAX_VT = 32;      // channel vectors (of 8) per statistics CTA

__device__ __forceinline__ void unpack8(const uint4& v, float (&f)[8]) {
    const __half2* h = reinterpret_cast<const __half2*>(&v);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const float2 t = __half22float2(h[k]);
        f[2 * k] = t.x;
        f[2 * k + 1] = t.y;
    }
}

__global__ void __launch_bounds__(BN_THREADS)
bn_stats_partial(const __half* __restrict__ x, long long M, int C, int VT, double* __restrict__ part) {
    __shared__ double s1[BN_THREADS * 8], s2[BN_THREADS * 8];
    const int RL = BN_THREADS / VT;
    const int V = C >> 3;
    const int lane = threadIdx.x / VT, tv = threadIdx.x - lane * VT;
    const int cv = blockIdx.y * VT + tv;
    const long long r0 = (long long)blockIdx.x * BN_ROWS;
    const long long r1 = min(r0 + BN_ROWS, M);
    double a1[8], a2[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) a1[j] = a2[j] = 0.0;
    if (lane < RL && cv < V) {
        const uint4* src = reinterpret_cast<const uint4*>(x) + cv;
        long long r = r0 + lane;
        // two loads in flight per iteration; the additions stay in pixel order
        for (; r + RL < r1; r += 2 * RL) {
            const uint4 va = src[r * V], vb = src[(r + RL) * V];
            float fa[8], fb[8];
            unpack8(va, fa);
            unpack8(vb, fb);
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const double da = fa[j], db = fb[j];
                a1[j] = __dadd_rn(a1[j], da);
                a2[j] = __dadd_rn(a2[j], __dmul_rn(da, da));
                a1[j] = __dadd_rn(a1[j], db);
                a2[j] = __dadd_rn(a2[j], __dmul_rn(db, db));
            }
        }
        if (r < r1) {
            float fa[8];
            unpack8(src[r * V], fa);
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const double da = fa[j];
                a1[j] = __dadd_rn(a1[j], da);
                a2[j] = __dadd_rn(a2[j], __dmul_rn(da, da));
            }
        }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        s1[threadIdx.x * 8 + j] = a1[j];
        s2[threadIdx.x * 8 + j] = a2[j];
    }
    __syncthreads();
    // thread t < 8 * VT owns channel 8 * (tile start) + t: adds the lanes in order
    if (threadIdx.x < 8 * VT) {
        const int tvc = threadIdx.x >> 3, j = threadIdx.x & 7;
        const int c = (blockIdx.y * VT + tvc) * 8 + j;
        if (c < C) {
            double t1 = s1[tvc * 8 + j], t2 = s2[tvc * 8 + j];
            for (int l = 1; l < RL; ++l) {
                t1 = __dadd_rn(t1, s1[(l * VT + tvc) * 8 + j]);
                t2 = __dadd_rn(t2, s2[(l * VT + tvc) * 8 + j]);
            }
            const size_t o = (size_t)blockIdx.x * C + c;
            part[2 * o] = t1;
            part[2 * o + 1] = t2;
        }
    }
}

__global__ void __launch_bounds__(128)
bn_stats_merge(const double* __restrict__ part, int nparts, long long M, int C, const float* __restrict__ gamma,
               const float* __restrict__ beta, const float* __restrict__ rmean, const float* __restrict__ rvar,
               double momentum, double eps, float* __restrict__ scale, float* __restrict__ shift,
               float* __restrict__ new_mean, float* __restrict__ new_var, int* __restrict__ nonfinite) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C) return;
    const BnMerged r = bn_merge_channel(part, nparts, M, C, c, gamma[c], beta[c], rmean[c], rvar[c], momentum, eps);
    scale[c] = r.scale;
    shift[c] = r.shift;
    new_mean[c] = r.new_mean;
    new_var[c] = r.new_var;
    if (!(isfinite(r.scale) && isfinite(r.shift) && isfinite(r.new_mean) && isfinite(r.new_var))) *nonfinite = 1;
}

template <int ACT>
__device__ __forceinline__ float bn_act(float v) {
    if (ACT != LP_ACT_NONE) v = v > 0.f ? v : 0.f;
    if (ACT == LP_ACT_RELU6) v = v < 6.f ? v : 6.f;
    return v;
}

template <int ACT, bool RES>
__global__ void __launch_bounds__(256)
bn_apply_kernel(const __half* x, const float* __restrict__ scale, const float* __restrict__ shift,
                const __half* __restrict__ res, __half* y, long long nvec, int V) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += (long long)gridDim.x * blockDim.x) {
        const int c0 = (int)(i % V) * 8;
        float f[8], r[8];
        unpack8(reinterpret_cast<const uint4*>(x)[i], f);
        if (RES) unpack8(reinterpret_cast<const uint4*>(res)[i], r);
        const float4 sa = *reinterpret_cast<const float4*>(scale + c0), sb = *reinterpret_cast<const float4*>(scale + c0 + 4);
        const float4 ba = *reinterpret_cast<const float4*>(shift + c0), bb = *reinterpret_cast<const float4*>(shift + c0 + 4);
        const float s[8] = {sa.x, sa.y, sa.z, sa.w, sb.x, sb.y, sb.z, sb.w};
        const float b[8] = {ba.x, ba.y, ba.z, ba.w, bb.x, bb.y, bb.z, bb.w};
        uint4 o;
        __half2* h = reinterpret_cast<__half2*>(&o);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            float v0 = bn_act<ACT>(fmaf(f[2 * k], s[2 * k], b[2 * k]));
            float v1 = bn_act<ACT>(fmaf(f[2 * k + 1], s[2 * k + 1], b[2 * k + 1]));
            if (RES) {
                v0 = __fadd_rn(v0, r[2 * k]);
                v1 = __fadd_rn(v1, r[2 * k + 1]);
            }
            h[k] = __floats2half2_rn(v0, v1);
        }
        reinterpret_cast<uint4*>(y)[i] = o;
    }
}

static int bn_vt(int C) { return (C / 8) < BN_MAX_VT ? (C / 8) : BN_MAX_VT; }

}  // namespace lp

using namespace lp;

extern "C" size_t lp_bn_stats_workspace_bytes(int M, int C) {
    if (M <= 0 || C <= 0) return 0;
    return (size_t)((M + BN_ROWS - 1) / BN_ROWS) * C * 2 * sizeof(double);
}

extern "C" int lp_bn_stats_f16(const void* x, int M, int C, const float* gamma, const float* beta,
                               const float* running_mean, const float* running_var, double momentum, double eps,
                               float* scale, float* shift, float* new_mean, float* new_var, int* nonfinite,
                               void* workspace, size_t workspace_bytes, lp_stream_t stream) {
    LP_CHECK_ARG(x && gamma && beta && running_mean && running_var && scale && shift && new_mean && new_var && nonfinite &&
                 workspace, "lp_bn_stats_f16: null pointer");
    LP_CHECK_ARG(M >= 2 && C >= 8 && C % 8 == 0, "lp_bn_stats_f16: bad shape M=%d C=%d (M >= 2, C %% 8 == 0)", M, C);
    LP_CHECK_ARG(eps >= 0.0 && momentum >= 0.0 && momentum <= 1.0, "lp_bn_stats_f16: bad momentum %g / eps %g",
                 momentum, eps);
    if (workspace_bytes < lp_bn_stats_workspace_bytes(M, C)) {
        set_error("lp_bn_stats_f16: workspace of %zu bytes, %zu needed", workspace_bytes, lp_bn_stats_workspace_bytes(M, C));
        return LP_ERR_CAPACITY;
    }
    if ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(workspace)) & 15) {
        set_error("lp_bn_stats_f16: x and workspace must be 16-byte aligned");
        return LP_ERR_ALIGN;
    }
    const int VT = bn_vt(C);
    const int nparts = (M + BN_ROWS - 1) / BN_ROWS;
    const dim3 grid(nparts, (C / 8 + VT - 1) / VT);
    double* part = reinterpret_cast<double*>(workspace);
    cudaStream_t st = (cudaStream_t)stream;
    bn_stats_partial<<<grid, BN_THREADS, 0, st>>>(reinterpret_cast<const __half*>(x), M, C, VT, part);
    LP_LAUNCH_CHECK("bn_stats_partial");
    bn_stats_merge<<<(C + 127) / 128, 128, 0, st>>>(part, nparts, M, C, gamma, beta, running_mean, running_var, momentum,
                                                   eps, scale, shift, new_mean, new_var, nonfinite);
    LP_LAUNCH_CHECK("bn_stats_merge");
    return LP_OK;
}

extern "C" int lp_bn_apply_f16(const void* x, const float* scale, const float* shift, const void* residual, void* y,
                               int M, int C, int act, lp_stream_t stream) {
    LP_CHECK_ARG(x && scale && shift && y, "lp_bn_apply_f16: null pointer");
    LP_CHECK_ARG(M > 0 && C >= 8 && C % 8 == 0, "lp_bn_apply_f16: bad shape M=%d C=%d (C %% 8 == 0)", M, C);
    LP_CHECK_ARG(act >= LP_ACT_NONE && act <= LP_ACT_RELU6, "lp_bn_apply_f16: bad act %d", act);
    if ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y) | reinterpret_cast<uintptr_t>(residual) |
         reinterpret_cast<uintptr_t>(scale) | reinterpret_cast<uintptr_t>(shift)) & 15) {
        set_error("lp_bn_apply_f16: pointers must be 16-byte aligned");
        return LP_ERR_ALIGN;
    }
    const long long nvec = (long long)M * (C / 8);
    const long long want = (nvec + 255) / 256;
    const int grid = (int)(want < 8LL * num_sms() ? want : 8LL * num_sms());
    const __half* xh = reinterpret_cast<const __half*>(x);
    const __half* rh = reinterpret_cast<const __half*>(residual);
    __half* yh = reinterpret_cast<__half*>(y);
    cudaStream_t st = (cudaStream_t)stream;
#define LP_BN_APPLY(A)                                                                                    \
    if (residual) bn_apply_kernel<A, true><<<grid, 256, 0, st>>>(xh, scale, shift, rh, yh, nvec, C / 8);  \
    else bn_apply_kernel<A, false><<<grid, 256, 0, st>>>(xh, scale, shift, rh, yh, nvec, C / 8);
    if (act == LP_ACT_RELU) { LP_BN_APPLY(LP_ACT_RELU) }
    else if (act == LP_ACT_RELU6) { LP_BN_APPLY(LP_ACT_RELU6) }
    else { LP_BN_APPLY(LP_ACT_NONE) }
#undef LP_BN_APPLY
    LP_LAUNCH_CHECK("bn_apply_kernel");
    return LP_OK;
}
