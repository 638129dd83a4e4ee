// The per-channel merge of train-mode BatchNorm statistics, shared by the NHWC fp16 recalibration (bn_train.cu,
// lp_bn_stats_f16) and the NCHW training forward (bn_nchw_train.cu, lp_bn_nchw_fwd).  Both reduction kernels leave
// the per-range fp64 (sum, sum of squares) of channel c at part[2 * (r * C + c)], part[2 * (r * C + c) + 1].
#pragma once
#include "common.cuh"

namespace lp {

struct BnMerged {
    float scale, shift;          // the apply pass's y = fmaf(x, scale, shift)
    float mean, invstd;          // saved for the backward pass
    float new_mean, new_var;     // the momentum update of the running statistics
};

// Adds the ranges in order r = 0, 1, ..., starting from range 0's, then derives in fp64, every operation rounded once:
//   mean = S1 / M, var = max(S2 / M - mean * mean, 0), var_unbiased = var * M / (M - 1),
//   s = gamma / sqrt(var + eps), scale = fp32(s), shift = fp32(beta - mean * s), invstd = fp32(1 / sqrt(var + eps)),
//   new running = fp32((1 - momentum) * running + momentum * stat) for (mean, var_unbiased).
__device__ __forceinline__ BnMerged bn_merge_channel(const double* __restrict__ part, int nparts, long long M, int C,
                                                     int c, float gamma, float beta, float rmean, float rvar,
                                                     double momentum, double eps) {
    double t1 = part[2 * c], t2 = part[2 * c + 1];
    for (int i = 1; i < nparts; ++i) {
        const size_t o = (size_t)i * C + c;
        t1 = __dadd_rn(t1, part[2 * o]);
        t2 = __dadd_rn(t2, part[2 * o + 1]);
    }
    const double m = (double)M;
    const double mean = __ddiv_rn(t1, m);
    double var = __dsub_rn(__ddiv_rn(t2, m), __dmul_rn(mean, mean));
    var = var > 0.0 ? var : 0.0;
    const double var_u = __ddiv_rn(__dmul_rn(var, m), __dsub_rn(m, 1.0));
    const double sd = __dsqrt_rn(__dadd_rn(var, eps));
    const double s = __ddiv_rn((double)gamma, sd);
    const double keep = __dsub_rn(1.0, momentum);
    BnMerged r;
    r.scale = __double2float_rn(s);
    r.shift = __double2float_rn(__dsub_rn((double)beta, __dmul_rn(mean, s)));
    r.mean = __double2float_rn(mean);
    r.invstd = __double2float_rn(__ddiv_rn(1.0, sd));
    r.new_mean = __double2float_rn(__dadd_rn(__dmul_rn(keep, (double)rmean), __dmul_rn(momentum, mean)));
    r.new_var = __double2float_rn(__dadd_rn(__dmul_rn(keep, (double)rvar), __dmul_rn(momentum, var_u)));
    return r;
}

}  // namespace lp
