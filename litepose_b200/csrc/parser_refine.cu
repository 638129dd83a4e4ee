// G4+G5+G6: adjust, per-person scores, refine on the device (reference lib/core/group.py:178-291).
//   adjust : quarter-pixel shift toward the larger 4-neighbour (strict >), then +0.5   (:178-197)
//   scores : mean joint value per person after adjust, before refine                     (:275)
//   refine : per person, prev_tag = mean tag over detected joints; for every joint the arg-max over the
//            whole map of det - round(||tag - prev_tag||); fills only undetected joints    (:199-267)
// The reference runs refine once per person with ~10 dense passes each (P x 44 MB at 512^2, T=2).  Here ONE
// pass over det+tag serves all persons: algorithmic bytes 4*N*J*H*W*(1+T), and only (person, joint) pairs that
// are actually missing are evaluated.  Results are reduced with warp shuffles -> shared atomics -> one global
// 64-bit atomicMax per (CTA, person); key = (orderable score bits << 32) | ~flat_index so that ties resolve to
// the first (lowest) index like torch.argmax on the CPU.
#include "common.cuh"

namespace lp {

constexpr int RF_THREADS = 256;
constexpr int RF_PIX = 8;                       // pixels per thread
constexpr int RF_CHUNK = RF_THREADS * RF_PIX;   // pixels per CTA
constexpr int RF_PB = 32;                       // persons per shared-memory batch
constexpr int RF_TMAX = 4;

struct RefineWs {
    float* prev;                  // [N][pcap][RF_TMAX]
    int32_t* miss_cnt;            // [N][J]
    int32_t* miss_list;           // [N][J][pcap]
    unsigned long long* best;     // [N][pcap][J]
};

// Maps of image n.  Uniform call (desc == nullptr): [N,J,H,W] det and [N,J,H,W,T] tag.  Ragged call: desc[n] gives the
// size and the offsets of the image's blocks in the det / tag arena.
struct ImageMaps {
    int H, W;
    size_t det_off, tag_off;
};

__device__ __forceinline__ ImageMaps image_maps(const lp_map_desc_t* desc, int n, int J, int H, int W, int T) {
    ImageMaps m;
    if (desc == nullptr) {
        m.H = H;
        m.W = W;
        m.det_off = (size_t)n * J * H * W;
        m.tag_off = (size_t)n * J * H * W * T;
    } else {
        m.H = desc[n].h;
        m.W = desc[n].w;
        m.det_off = (size_t)desc[n].det_offset;
        m.tag_off = (size_t)desc[n].tag_offset;
    }
    return m;
}

__device__ __forceinline__ float np_mean_pairwise(const float* a, int n, int stride) {
    // numpy add.reduce (pairwise, 8 accumulators) / n for n < 128
    float res;
    if (n < 8) {
        res = 0.f;
        for (int i = 0; i < n; ++i) res = __fadd_rn(res, a[i * stride]);
    } else {
        float r[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) r[j] = a[j * stride];
        int i = 8;
        for (; i < n - (n % 8); i += 8)
#pragma unroll
            for (int j = 0; j < 8; ++j) r[j] = __fadd_rn(r[j], a[(i + j) * stride]);
        res = __fadd_rn(__fadd_rn(__fadd_rn(r[0], r[1]), __fadd_rn(r[2], r[3])),
                        __fadd_rn(__fadd_rn(r[4], r[5]), __fadd_rn(r[6], r[7])));
        for (; i < n; ++i) res = __fadd_rn(res, a[i * stride]);
    }
    return __fdiv_rn(res, (float)n);
}

// one CTA per image
__global__ void __launch_bounds__(128)
adjust_scores_kernel(const float* __restrict__ det, const float* __restrict__ tag, const lp_map_desc_t* __restrict__ desc,
                     int J, int H_u, int W_u, int T, int pcap, float* __restrict__ ans_all,
                     const int32_t* __restrict__ num_people, float* __restrict__ scores_all, int do_adjust, int do_refine,
                     RefineWs ws) {
    const int n = blockIdx.x;
    const int D = 3 + T;
    const int P = min(num_people[n], pcap);
    const ImageMaps im = image_maps(desc, n, J, H_u, W_u, T);
    const int H = im.H, W = im.W;
    float* ans = ans_all + (size_t)n * pcap * J * D;
    const float* detn = det + im.det_off;
    const float* tagn = tag + im.tag_off;

    if (do_refine) {
        for (int i = threadIdx.x; i < J; i += blockDim.x) ws.miss_cnt[(size_t)n * J + i] = 0;
        for (int i = threadIdx.x; i < P * J; i += blockDim.x) ws.best[(size_t)n * pcap * J + i] = 0ull;
    }
    if (do_adjust) {
        for (int e = threadIdx.x; e < P * J; e += blockDim.x) {
            const int j = e % J;
            float* kp = ans + (size_t)e * D;
            if (kp[2] > 0.f) {
                float x = kp[0], y = kp[1];
                const int xi = (int)x, yi = (int)y;
                const float* tmp = detn + (size_t)j * H * W;
                x += (tmp[yi * W + min(xi + 1, W - 1)] > tmp[yi * W + max(xi - 1, 0)]) ? 0.25f : -0.25f;
                y += (tmp[min(yi + 1, H - 1) * W + xi] > tmp[max(yi - 1, 0) * W + xi]) ? 0.25f : -0.25f;
                kp[0] = x + 0.5f;
                kp[1] = y + 0.5f;
            }
        }
    }
    __syncthreads();
    for (int p = threadIdx.x; p < P; p += blockDim.x) {
        const float* kp = ans + (size_t)p * J * D;
        scores_all[(size_t)n * pcap + p] = np_mean_pairwise(kp + 2, J, D);
        if (!do_refine) continue;
        // prev_tag = torch.mean over detected joints (ATen CPU order: columns in groups of 4 sequentially,
        // left-over columns with 4 interleaved partial sums; see oracle/group_ref.py::_mean_f32_rows)
        float sum[RF_TMAX];
        float part[RF_TMAX][4];
        for (int t = 0; t < T; ++t) {
            sum[t] = 0.f;
            part[t][0] = part[t][1] = part[t][2] = part[t][3] = 0.f;
        }
        int m = 0;
        for (int j = 0; j < J; ++j) m += kp[(size_t)j * D + 2] > 0.f;
        const int full_cols = (T / 4) * 4;
        const int groups = m / 4;
        int q = 0;
        for (int j = 0; j < J; ++j) {
            const float* k = kp + (size_t)j * D;
            if (k[2] > 0.f) {
                const int x = (int)k[0], y = (int)k[1];
                const float* tp = tagn + (((size_t)j * H + y) * W + x) * T;
                for (int t = 0; t < T; ++t) {
                    const float v = tp[t];
                    if (t < full_cols) sum[t] = __fadd_rn(sum[t], v);
                    else if (q < groups * 4) part[t][q & 3] = __fadd_rn(part[t][q & 3], v);
                    else part[t][0] = __fadd_rn(part[t][0], v);
                }
                ++q;
            } else {
                const int slot = atomicAdd(&ws.miss_cnt[(size_t)n * J + j], 1);
                ws.miss_list[((size_t)n * J + j) * pcap + slot] = p;
            }
        }
        for (int t = 0; t < T; ++t) {
            float s = sum[t];
            if (t >= full_cols)
                s = __fadd_rn(__fadd_rn(__fadd_rn(part[t][0], part[t][1]), part[t][2]), part[t][3]);
            ws.prev[((size_t)n * pcap + p) * RF_TMAX + t] = __fdiv_rn(s, (float)m);
        }
    }
}

__device__ __forceinline__ unsigned order_f32(float f) {
    const unsigned b = __float_as_uint(f);
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

__device__ __forceinline__ unsigned long long warp_max_u64(unsigned long long v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const unsigned long long other = __shfl_xor_sync(0xffffffffu, v, o);
        v = other > v ? other : v;
    }
    return v;
}

template <int T>
__global__ void __launch_bounds__(RF_THREADS)
refine_argmax_kernel(const float* __restrict__ det, const float* __restrict__ tag, const lp_map_desc_t* __restrict__ desc,
                     int J, int H_u, int W_u, int pcap, RefineWs ws) {
    const int n = blockIdx.z, j = blockIdx.y;
    const ImageMaps im = image_maps(desc, n, J, H_u, W_u, T);
    const int HW = im.H * im.W;
    const int pix0 = blockIdx.x * RF_CHUNK;
    if (pix0 >= HW) return;                        // ragged: the grid covers the largest map
    const int cnt = ws.miss_cnt[(size_t)n * J + j];
    if (cnt == 0) return;
    __shared__ unsigned long long s_best[RF_PB];
    __shared__ float s_prev[RF_PB][RF_TMAX];
    __shared__ int s_pid[RF_PB];
    const size_t plane = (size_t)n * J + j;
    const float* dp = det + im.det_off + (size_t)j * HW;
    const float* tp = tag + im.tag_off + (size_t)j * HW * T;
    float d[RF_PIX], tg[RF_PIX][T];
#pragma unroll
    for (int k = 0; k < RF_PIX; ++k) {
        const int i = pix0 + threadIdx.x + k * RF_THREADS;
        if (i < HW) {
            d[k] = __ldg(dp + i);
#pragma unroll
            for (int t = 0; t < T; ++t) tg[k][t] = __ldg(tp + (size_t)i * T + t);
        } else {
            d[k] = 0.f;
#pragma unroll
            for (int t = 0; t < T; ++t) tg[k][t] = 0.f;
        }
    }
    const int32_t* list = ws.miss_list + plane * pcap;
    for (int q0 = 0; q0 < cnt; q0 += RF_PB) {
        const int nb = min(RF_PB, cnt - q0);
        __syncthreads();
        if (threadIdx.x < nb) {
            const int p = list[q0 + threadIdx.x];
            s_pid[threadIdx.x] = p;
            s_best[threadIdx.x] = 0ull;
            for (int t = 0; t < T; ++t) s_prev[threadIdx.x][t] = ws.prev[((size_t)n * pcap + p) * RF_TMAX + t];
        }
        __syncthreads();
        for (int q = 0; q < nb; ++q) {
            float pv[T];
#pragma unroll
            for (int t = 0; t < T; ++t) pv[t] = s_prev[q][t];
            unsigned long long best = 0ull;
#pragma unroll
            for (int k = 0; k < RF_PIX; ++k) {
                const int i = pix0 + threadIdx.x + k * RF_THREADS;
                float s = 0.f;
#pragma unroll
                for (int t = 0; t < T; ++t) {
                    const float df = __fsub_rn(tg[k][t], pv[t]);
                    const float sq = __fmul_rn(df, df);
                    s = (t == 0) ? sq : __fadd_rn(s, sq);
                }
                const float tt = __fsqrt_rn(s);
                const float score = __fadd_rn(__fsub_rn(d[k], rintf(tt)), 0.0f);   // +0.0f canonicalises -0.0
                const unsigned long long key =
                    ((unsigned long long)order_f32(score) << 32) | (unsigned long long)(0xffffffffu - (unsigned)i);
                if (i < HW && key > best) best = key;
            }
            best = warp_max_u64(best);
            if ((threadIdx.x & 31) == 0 && best) atomicMax(&s_best[q], best);
        }
        __syncthreads();
        if (threadIdx.x < nb && s_best[threadIdx.x])
            atomicMax(&ws.best[((size_t)n * pcap + s_pid[threadIdx.x]) * J + j], s_best[threadIdx.x]);
    }
}

__global__ void __launch_bounds__(128)
refine_finalize_kernel(const float* __restrict__ det, const lp_map_desc_t* __restrict__ desc, int J, int H_u, int W_u,
                       int T, int pcap, float* __restrict__ ans_all, RefineWs ws) {
    const int n = blockIdx.y, j = blockIdx.x;
    const int cnt = ws.miss_cnt[(size_t)n * J + j];
    const int D = 3 + T;
    const ImageMaps im = image_maps(desc, n, J, H_u, W_u, T);
    const int H = im.H, W = im.W;
    const float* tmp = det + im.det_off + (size_t)j * H * W;
    for (int q = threadIdx.x; q < cnt; q += blockDim.x) {
        const int p = ws.miss_list[((size_t)n * J + j) * pcap + q];
        const unsigned long long key = ws.best[((size_t)n * pcap + p) * J + j];
        if (!key) continue;
        const int idx = (int)(0xffffffffu - (unsigned)(key & 0xffffffffu));
        const int yy = idx / W, xx = idx % W;
        const float val = tmp[idx];
        if (val > 0.f) {
            float x = (float)xx + 0.5f, y = (float)yy + 0.5f;
            x += (tmp[yy * W + min(xx + 1, W - 1)] > tmp[yy * W + max(xx - 1, 0)]) ? 0.25f : -0.25f;
            y += (tmp[min(yy + 1, H - 1) * W + xx] > tmp[max(yy - 1, 0) * W + xx]) ? 0.25f : -0.25f;
            float* kp = ans_all + (((size_t)n * pcap + p) * J + j) * D;
            kp[0] = x;
            kp[1] = y;
            kp[2] = val;
        }
    }
}

}  // namespace lp

using namespace lp;

static size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

extern "C" size_t lp_adjust_refine_workspace_bytes(int N, int J, int pcap) {
    if (N <= 0 || J <= 0 || pcap <= 0) return 0;
    size_t b = 0;
    b += align_up((size_t)N * pcap * RF_TMAX * sizeof(float), 256);
    b += align_up((size_t)N * J * sizeof(int32_t), 256);
    b += align_up((size_t)N * J * pcap * sizeof(int32_t), 256);
    b += align_up((size_t)N * pcap * J * sizeof(unsigned long long), 256);
    return b;
}

// Both entry points: uniform (hw_host == nullptr, every map H x W) or ragged (per-image sizes, device desc).
static int adjust_refine_launch(const float* det, const float* tag, int N, const int32_t* hw_host, const lp_map_desc_t* desc,
                                int J, int H, int W, int T, int pcap, float* ans, const int32_t* num_people, float* scores,
                                int do_adjust, int do_refine, void* workspace, size_t workspace_bytes, lp_stream_t stream,
                                const char* name) {
    LP_CHECK_ARG(det && tag && ans && num_people && scores && workspace, "%s: null pointer", name);
    LP_CHECK_ARG(N > 0 && N <= 65535 && J > 0 && J <= 65535 && pcap > 0, "%s: bad shape N=%d J=%d pcap=%d", name, N, J, pcap);
    LP_CHECK_ARG(T >= 1 && T <= RF_TMAX, "%s: T=%d unsupported (1..%d)", name, T, RF_TMAX);
    long long max_hw = 0;
    for (int n = 0; n < (hw_host ? N : 1); ++n) {
        const int h = hw_host ? hw_host[2 * n] : H, w = hw_host ? hw_host[2 * n + 1] : W;
        LP_CHECK_ARG(h > 0 && w > 0 && (long long)h * w < (1ll << 31), "%s: bad map size %dx%d (image %d)", name, h, w, n);
        max_hw = (long long)h * w > max_hw ? (long long)h * w : max_hw;
    }
    const size_t need = lp_adjust_refine_workspace_bytes(N, J, pcap);
    if (workspace_bytes < need) {
        set_error("%s: workspace %zu < required %zu bytes", name, workspace_bytes, need);
        return LP_ERR_CAPACITY;
    }
    if (reinterpret_cast<uintptr_t>(workspace) & 255) {
        set_error("%s: workspace must be 256-byte aligned", name);
        return LP_ERR_ALIGN;
    }
    RefineWs ws;
    uint8_t* b = reinterpret_cast<uint8_t*>(workspace);
    ws.prev = reinterpret_cast<float*>(b);
    b += align_up((size_t)N * pcap * RF_TMAX * sizeof(float), 256);
    ws.miss_cnt = reinterpret_cast<int32_t*>(b);
    b += align_up((size_t)N * J * sizeof(int32_t), 256);
    ws.miss_list = reinterpret_cast<int32_t*>(b);
    b += align_up((size_t)N * J * pcap * sizeof(int32_t), 256);
    ws.best = reinterpret_cast<unsigned long long*>(b);
    cudaStream_t s = (cudaStream_t)stream;
    adjust_scores_kernel<<<N, 128, 0, s>>>(det, tag, desc, J, H, W, T, pcap, ans, num_people, scores, do_adjust, do_refine,
                                           ws);
    LP_LAUNCH_CHECK("adjust_scores_kernel");
    if (do_refine) {
        dim3 grid((unsigned)((max_hw + RF_CHUNK - 1) / RF_CHUNK), J, N);
        switch (T) {
            case 1: refine_argmax_kernel<1><<<grid, RF_THREADS, 0, s>>>(det, tag, desc, J, H, W, pcap, ws); break;
            case 2: refine_argmax_kernel<2><<<grid, RF_THREADS, 0, s>>>(det, tag, desc, J, H, W, pcap, ws); break;
            case 3: refine_argmax_kernel<3><<<grid, RF_THREADS, 0, s>>>(det, tag, desc, J, H, W, pcap, ws); break;
            default: refine_argmax_kernel<4><<<grid, RF_THREADS, 0, s>>>(det, tag, desc, J, H, W, pcap, ws); break;
        }
        LP_LAUNCH_CHECK("refine_argmax_kernel");
        dim3 g2(J, N);
        refine_finalize_kernel<<<g2, 128, 0, s>>>(det, desc, J, H, W, T, pcap, ans, ws);
        LP_LAUNCH_CHECK("refine_finalize_kernel");
    }
    return LP_OK;
}

extern "C" int lp_adjust_refine_f32(const float* det, const float* tag, int N, int J, int H, int W, int T, int pcap,
                                    float* ans, const int32_t* num_people, float* scores, int do_adjust, int do_refine,
                                    void* workspace, size_t workspace_bytes, lp_stream_t stream) {
    LP_CHECK_ARG(H > 0 && W > 0, "lp_adjust_refine_f32: bad shape N=%d J=%d H=%d W=%d pcap=%d", N, J, H, W, pcap);
    return adjust_refine_launch(det, tag, N, nullptr, nullptr, J, H, W, T, pcap, ans, num_people, scores, do_adjust,
                                do_refine, workspace, workspace_bytes, stream, "lp_adjust_refine_f32");
}

extern "C" int lp_adjust_refine_ragged_f32(const float* det, const float* tag, int N, const int32_t* hw_host,
                                           const lp_map_desc_t* desc, int J, int T, int pcap, float* ans,
                                           const int32_t* num_people, float* scores, int do_adjust, int do_refine,
                                           void* workspace, size_t workspace_bytes, lp_stream_t stream) {
    LP_CHECK_ARG(hw_host && desc, "lp_adjust_refine_ragged_f32: null pointer");
    return adjust_refine_launch(det, tag, N, hw_host, desc, J, 0, 0, T, pcap, ans, num_people, scores, do_adjust,
                                do_refine, workspace, workspace_bytes, stream, "lp_adjust_refine_ragged_f32");
}

// ---------------------------------------------------------------------------------------------- final predictions
// get_final_preds (reference lib/utils/transforms.py:195-202 -> transform_preds :50-57 -> affine_transform :101-104):
// x, y of every keypoint of every found person go through the image's inverse affine (2x3, float64) and are stored
// back as float32.  np.dot(t, [x, y, 1.]) on the reference's host evaluates each row as fma(t0, x, t1*y) + t2
// (OpenBLAS dgemv, determined against numpy in the build container); the same order is used here.
namespace lp {
__global__ void transform_preds_kernel(float* __restrict__ ans, const int* __restrict__ num, const double* __restrict__ trans,
                                       int pcap, int J, int row) {
    const int n = blockIdx.y;
    const int np_ = min(num[n], pcap);
    const int i = blockIdx.x * blockDim.x + threadIdx.x;      // (person, joint)
    if (i >= np_ * J) return;
    const double* t = trans + (size_t)n * 6;
    float* p = ans + ((size_t)n * pcap * J + i) * row;
    const double x = (double)p[0], y = (double)p[1];
    const double nx = __dadd_rn(__fma_rn(t[0], x, __dmul_rn(t[1], y)), t[2]);
    const double ny = __dadd_rn(__fma_rn(t[3], x, __dmul_rn(t[4], y)), t[5]);
    p[0] = __double2float_rn(nx);
    p[1] = __double2float_rn(ny);
}
}  // namespace lp

extern "C" int lp_transform_preds_f32(float* ans, const int32_t* num_people, const double* trans, int N, int pcap, int J,
                                      int row, lp_stream_t stream) {
    LP_CHECK_ARG(ans && num_people && trans, "lp_transform_preds_f32: null pointer");
    LP_CHECK_ARG(N > 0 && N <= 65535 && pcap > 0 && J > 0 && row >= 2, "lp_transform_preds_f32: bad shape N=%d pcap=%d J=%d row=%d",
                 N, pcap, J, row);
    dim3 grid((pcap * J + 127) / 128, N);
    lp::transform_preds_kernel<<<grid, 128, 0, (cudaStream_t)stream>>>(ans, num_people, trans, pcap, J, row);
    LP_LAUNCH_CHECK("transform_preds_kernel");
    return LP_OK;
}
