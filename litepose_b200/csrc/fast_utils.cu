// "Fast inference" grouping of the reference's nano demo on the GPU (SURVEY.md 8(f) row 2): the reference's only
// native code, nano_demo/fast_utils/parse/find_peaks.cpp:9-97 and assign.cpp:11-122, exported by plugins.cpp:9-116 as
// find_peaks[_out] / assign[_out] and driven by nano_demo/fast_utils/group.py:38-47.
//
//   find_peaks : one CTA per (image, joint) plane; pixels are visited in scan order 1024 at a time, every candidate
//                (value >= threshold, no strictly larger value in the window) gets its scan-order rank from a
//                ballot-free block prefix sum, the first M ranks are written - the same set and order as the
//                reference's sequential scan with its early exit.
//   assign     : one warp per image; lane i owns column / row i of the reference's KM state (slack-array Hungarian
//                variant), the augmenting DFS runs as an explicit stack with ballot / ffs column scans - same visiting
//                order, same float arithmetic (IEEE single ops, no contraction), same number of label-update rounds
//                (the reference walks towards a padded column in steps of the smallest slack, typically thousands of
//                rounds), including its `abs(t) < 1e-2` which binds to int abs(int) with its includes: trunc(t) == 0.
// The reference's [10] stack arrays (assign.cpp:46-48,79-80) are lifted to 32 entries; its unbounded KM loop is capped
// (status 1 is reported where the reference would not return).
#include "common.cuh"

namespace lp {

constexpr int FU_MAXP = 32;
constexpr int FU_MAXPAIRS = 256;
constexpr int FU_MAX_ROUNDS = 1 << 20;   // per KM row; the reference needs ~1e4/|d| rounds to reach a padded column
constexpr int FP_THREADS = 256;
constexpr int FP_PPT = 4;

__device__ __forceinline__ bool fu_is_peak(const float* __restrict__ in, int idx, int H, int W, float thr, int win) {
    const float hval = in[idx];
    if (hval < thr) return false;
    const int i = idx / W, j = idx - i * W;
    const int ii0 = max(i - win, 0), jj0 = max(j - win, 0);
    const int ii1 = min(i + win + 1, H), jj1 = min(j + win + 1, W);
    bool peak = true;
    for (int ii = ii0; ii < ii1; ++ii)
        for (int jj = jj0; jj < jj1; ++jj)
            if (in[ii * W + jj] > hval) peak = false;
    return peak;
}

// One (image, joint) plane, one CTA: `in` is the H x W heat-map, the tag of pixel idx is tm[idx * tstride] (1: a plain
// [H,W] map; T: channel 0 of an interleaved [H,W,T] map).  Writes count[0] and the first min(count, M) entries of
// pv / pt / pi; entries past the count are not written.
__device__ __forceinline__ void fu_find_peaks_plane(const float* __restrict__ in, const float* __restrict__ tm, int H, int W,
                                                    int tstride, int M, float thr, int window_size, int* __restrict__ count,
                                                    float* __restrict__ pv, float* __restrict__ pt, int* __restrict__ pi) {
    __shared__ int s_warp[FP_THREADS / 32];
    const int HW = H * W;
    const int win = window_size / 2;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int base = 0;     // peaks found before this chunk (identical in every thread)
    for (int start = 0; start < HW && base < M; start += FP_THREADS * FP_PPT) {
        const int idx0 = start + threadIdx.x * FP_PPT;
        unsigned flags = 0;
#pragma unroll
        for (int k = 0; k < FP_PPT; ++k) {
            const int idx = idx0 + k;
            if (idx < HW && fu_is_peak(in, idx, H, W, thr, win)) flags |= 1u << k;
        }
        const int c = __popc(flags);
        int incl = c;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int v = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += v;
        }
        if (lane == 31) s_warp[warp] = incl;
        __syncthreads();
        int woff = 0, total = 0;
#pragma unroll
        for (int w = 0; w < FP_THREADS / 32; ++w) {
            const int v = s_warp[w];
            if (w < warp) woff += v;
            total += v;
        }
        int r = base + woff + incl - c;
#pragma unroll
        for (int k = 0; k < FP_PPT; ++k)
            if (flags & (1u << k)) {
                if (r < M) {
                    const int idx = idx0 + k;
                    const int i = idx / W;
                    pi[2 * r] = idx - i * W;
                    pi[2 * r + 1] = i;
                    pv[r] = in[idx];
                    pt[r] = tm[(size_t)idx * tstride];
                }
                ++r;
            }
        base += total;
        __syncthreads();
    }
    if (threadIdx.x == 0) *count = min(base, M);
}

__global__ void __launch_bounds__(FP_THREADS)
find_peaks_kernel(const float* __restrict__ input, const float* __restrict__ tmap, int H, int W, int M, float thr,
                  int window_size, int* __restrict__ count, float* __restrict__ val, float* __restrict__ tag,
                  int* __restrict__ ind) {
    const int plane = blockIdx.x;
    const size_t HW = (size_t)H * W;
    fu_find_peaks_plane(input + plane * HW, tmap + plane * HW, H, W, 1, M, thr, window_size, count + plane,
                        val + (size_t)plane * M, tag + (size_t)plane * M, ind + (size_t)plane * M * 2);
}

// The same planes read where the pipeline's glue leaves them: det [N,J,H,W] (or image n's [J,h,w] block at
// desc[n].det_offset), tag [N,tag_planes,H,W,T] (or [tag_planes,h,w,T] at desc[n].tag_offset) read in place at channel
// 0; tag_planes == 1 serves every joint from the one shared map.  Outputs in the layouts of find_peaks_kernel.
// (The minimum of 4 resident CTAs lifts ptxas' default 32-register budget, which spills the tag stride here.)
__global__ void __launch_bounds__(FP_THREADS, 4)
find_peaks_maps_kernel(const float* __restrict__ det, const float* __restrict__ tmap, const lp_map_desc_t* __restrict__ desc,
                       int J, int H, int W, int T, int tag_planes, int M, float thr, int window_size,
                       int* __restrict__ count, float* __restrict__ val, float* __restrict__ tag, int* __restrict__ ind) {
    const int plane = blockIdx.x;
    const int n = plane / J, j = plane - n * J;
    const int tj = tag_planes == 1 ? 0 : j;
    int h = H, w = W;
    size_t det_off, tag_off;
    if (desc == nullptr) {
        det_off = (size_t)plane * H * W;
        tag_off = ((size_t)n * tag_planes + tj) * H * W * T;
    } else {
        h = desc[n].h;
        w = desc[n].w;
        det_off = (size_t)desc[n].det_offset + (size_t)j * h * w;
        tag_off = (size_t)desc[n].tag_offset + (size_t)tj * h * w * T;
    }
    fu_find_peaks_plane(det + det_off, tmap + tag_off, h, w, T, M, thr, window_size, count + plane,
                        val + (size_t)plane * M, tag + (size_t)plane * M, ind + (size_t)plane * M * 2);
}

// ---------------------------------------------------------------------------------------------- assign
// One warp per image.  Lane i owns column i (Ly, slack, mat) and row i (Lx) of the KM state; the S / T sets are
// warp-uniform bit masks; the gain matrix lives in shared memory (row u is read by all lanes, conflict free).
struct FuShared {
    float G[FU_MAXP][FU_MAXP + 1];
    float diff[FU_MAXP][FU_MAXP + 1];
    float sum[FU_MAXP];
    int ch[FU_MAXP], nj[FU_MAXP];
    int npairs;
    unsigned short pairs[FU_MAXPAIRS];     // fast-forward: row | column << 5 | tree-edge flag << 10
};

struct FuKm {
    float Lx, Ly, slack;
    int mat;
    unsigned S, T;
    unsigned ev, tr;     // per column lane: rows whose pair with this column the last search evaluated as non-tight / took as tree edge
};

__device__ __forceinline__ float fu_min(float a, float b) { return a < b ? a : b; }   // the reference's MIN macro

// assign.cpp:15-31.  The recursion becomes an explicit stack (frame k lives in lane k: row u and the column to resume
// at); inside a frame the reference's column scan is done for all columns at once: the columns before the first
// "tight" one (trunc(t) == 0, see the file header) take the slack update, the tight column is visited (T), and either
// ends the search (free column) or pushes the row it is matched to - the same visiting order and side effects as the
// sequential scan, because t of a frame does not change while its callees run and T is re-read on every re-entry.
__device__ bool fu_match(const FuShared& s, FuKm& k, int n, int u0, int lane) {
    int sp = 0;
    int fr_u = 0, fr_pos = 0;           // this lane's frame (valid for lane <= sp)
    if (lane == 0) { fr_u = u0; fr_pos = 0; }
    k.S |= 1u << u0;
    for (;;) {
        const int u = __shfl_sync(0xffffffffu, fr_u, sp);
        const int pos = __shfl_sync(0xffffffffu, fr_pos, sp);
        const float lxu = __shfl_sync(0xffffffffu, k.Lx, u);
        const float t = __fsub_rn(__fadd_rn(lxu, k.Ly), s.G[u][lane]);
        const bool active = lane < n && lane >= pos && !((k.T >> lane) & 1u);
        const unsigned eq = __ballot_sync(0xffffffffu, active && __float2int_rz(t) == 0);
        if (eq == 0) {
            if (active) {
                k.slack = fu_min(k.slack, t);
                k.ev |= 1u << u;
            }
            if (sp == 0) return false;
            --sp;                         // the caller resumes behind the column it descended from
            continue;
        }
        const int e = __ffs(eq) - 1;
        if (active && lane < e) {
            k.slack = fu_min(k.slack, t);
            k.ev |= 1u << u;
        }
        if (lane == e) k.tr |= 1u << u;
        k.T |= 1u << e;
        const int m = __shfl_sync(0xffffffffu, k.mat, e);
        if (m == -1) {
            if (lane == e) k.mat = u;     // success: every caller takes the column it descended from
            for (int f = sp - 1; f >= 0; --f) {
                const int fu = __shfl_sync(0xffffffffu, fr_u, f);
                const int fc = __shfl_sync(0xffffffffu, fr_pos, f) - 1;
                if (lane == fc) k.mat = fu;
            }
            return true;
        }
        if (lane == sp) fr_pos = e + 1;
        ++sp;
        if (lane == sp) { fr_u = m; fr_pos = 0; }
        k.S |= 1u << m;
    }
}

// assign.cpp:45-66; false when the round cap is hit (the reference has none)
__device__ bool fu_km(FuShared& s, int n, int lane) {
    FuKm k;
    k.Lx = -1e6f;
    if (lane < n)
        for (int j = 0; j < n; ++j) k.Lx = k.Lx > s.G[lane][j] ? k.Lx : s.G[lane][j];
    k.Ly = 0.f;
    k.mat = -1;
    k.slack = 1e6f;
    for (int i = 0; i < n; ++i) {
        k.slack = 1e6f;
        int rounds = 0;
        unsigned prevS = 0xffffffffu, prevT = 0xffffffffu;
        for (;;) {
            k.S = 0;
            k.T = 0;
            k.ev = 0;
            k.tr = 0;
            if (fu_match(s, k, n, i, lane)) break;
            if (++rounds >= FU_MAX_ROUNDS) return false;
            float d = lane < n ? fu_min(1e8f, k.slack) : 1e8f;           // assign.cpp:33-43
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) d = fu_min(d, __shfl_xor_sync(0xffffffffu, d, o));
            if ((k.S >> lane) & 1u) k.Lx = __fsub_rn(k.Lx, d);
            if ((k.T >> lane) & 1u) k.Ly = __fadd_rn(k.Ly, d);

            // ---- fast-forward of a label walk (round 2).  d often stems from a pair whose column has been visited since
            // (slack is only reset per row), while the only unvisited columns left are far away (a padded -1e4 column):
            // the labels then crawl for thousands of rounds with the SAME failed search.  A round can be skipped - its label
            // update applied without running the search - iff the search would evaluate the same pairs with the same
            // tight / non-tight outcome.  The search consults only the pairs it evaluated last time (ev: non-tight, feeds
            // slack; tr: tree edge, tight), so:
            //   * pairs with a visited column only drift by rounding: they are re-evaluated EXACTLY every skipped round
            //     (same fp32 expression), their minimum keeps the running slack minimum exact (only the minimum over all
            //     columns is ever consumed), a status flip ends the walk before that round is skipped;
            //   * pairs with an unvisited column drop by at most d + DELTA per round: a conservative bound on the number of
            //     rounds for which they stay non-tight and >= d is computed once.
            const bool walk = (k.S == prevS) && (k.T == prevT) && d > 0.f;
            prevS = k.S;
            prevT = k.T;
            if (walk) {
                constexpr float DELTA = 0.008f;           // rounding drift bound per round for |labels| < 1e5
                const bool inS = (k.S >> lane) & 1u, inT = (k.T >> lane) & 1u;
                // (1) conservative round bound from the evaluated pairs with an unvisited column
                float rl = (lane >= n || (fabsf(k.Lx) < 1e5f && fabsf(k.Ly) < 1e5f)) ? 1e9f : 0.f;
                for (unsigned sb = k.S; sb; sb &= sb - 1) {
                    const int u = __ffs(sb) - 1;
                    const float lxu = __shfl_sync(0xffffffffu, k.Lx, u);
                    if (lane < n && !inT && ((k.ev >> u) & 1u)) {
                        const float t = __fsub_rn(__fadd_rn(lxu, k.Ly), s.G[u][lane]);
                        const float x = (t - fmaxf(1.f, d) - 2.f * DELTA) / (d + DELTA);
                        rl = fu_min(rl, x >= 0.f ? floorf(x) + 1.f : 0.f);
                    }
                }
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) rl = fu_min(rl, __shfl_xor_sync(0xffffffffu, rl, o));
                int rmax = rl > 1e6f ? 1000000 : (int)rl;
                if (rmax > FU_MAX_ROUNDS - 1 - rounds) rmax = FU_MAX_ROUNDS - 1 - rounds;
                // (2) list of the pairs that are tracked exactly: visited column, evaluated (type 0) or tree edge (type 1)
                if (lane == 0) s.npairs = 0;
                __syncwarp();
                if (lane < n && inT) {
                    for (unsigned m = k.ev | k.tr; m; m &= m - 1) {
                        const int u = __ffs(m) - 1;
                        const int q = atomicAdd(&s.npairs, 1);
                        if (q < FU_MAXPAIRS) s.pairs[q] = (unsigned short)(u | (lane << 5) | (((k.tr >> u) & 1u) << 10));
                    }
                }
                __syncwarp();
                const int np = s.npairs;
                if (np <= FU_MAXPAIRS) {
                    float gmin = d;                       // running minimum of slack over all columns (== d after the reduction)
                    // the first 32 tracked pairs live in registers (pair q <-> lane q); more (rare) are re-read from smem
                    const unsigned e0 = lane < np ? s.pairs[lane] : 0u;
                    const int u0 = e0 & 31, v0 = (e0 >> 5) & 31;
                    const float g0 = s.G[u0][v0];
                    const bool have0 = lane < np, tree0 = (e0 >> 10) & 1u;
                    for (int j = 0; j < rmax; ++j) {
                        // the search on the current labels: exact re-evaluation of the tracked pairs
                        float tmin = 1e30f;
                        bool flip = false;
                        {
                            const float lxu = __shfl_sync(0xffffffffu, k.Lx, u0);
                            const float lyv = __shfl_sync(0xffffffffu, k.Ly, v0);
                            const float t = __fsub_rn(__fadd_rn(lxu, lyv), g0);
                            const bool tight = __float2int_rz(t) == 0;
                            if (have0) {
                                flip = tree0 ? !tight : tight;
                                if (!tree0) tmin = t;
                            }
                        }
                        for (int q0 = 32; q0 < np; q0 += 32) {
                            const int q = q0 + lane;
                            const unsigned e = q < np ? s.pairs[q] : 0u;
                            const int u = e & 31, v = (e >> 5) & 31;
                            const float lxu = __shfl_sync(0xffffffffu, k.Lx, u);
                            const float lyv = __shfl_sync(0xffffffffu, k.Ly, v);
                            if (q < np) {
                                const float t = __fsub_rn(__fadd_rn(lxu, lyv), s.G[u][v]);
                                const bool tight = __float2int_rz(t) == 0;
                                if ((e >> 10) & 1u) flip |= !tight;
                                else {
                                    flip |= tight;
                                    tmin = fu_min(tmin, t);
                                }
                            }
                        }
                        if (__any_sync(0xffffffffu, flip)) break;      // this state needs the real search
#pragma unroll
                        for (int o = 16; o > 0; o >>= 1) tmin = fu_min(tmin, __shfl_xor_sync(0xffffffffu, tmin, o));
                        if (tmin <= 0.f) break;
                        gmin = fu_min(gmin, tmin);
                        ++rounds;
                        if (inS) k.Lx = __fsub_rn(k.Lx, gmin);
                        if (inT) k.Ly = __fadd_rn(k.Ly, gmin);
                    }
                    if (lane == 0) k.slack = fu_min(k.slack, gmin);     // only the minimum over the columns is ever consumed
                }
            }
        }
    }
    if (lane < n) s.ch[k.mat] = lane;
    __syncwarp();
    return true;
}

__global__ void __launch_bounds__(32)
assign_kernel(const int* __restrict__ count, const float* __restrict__ val, const float* __restrict__ tag,
              const int* __restrict__ ind, const int* __restrict__ joint_order, int C, int M, float threshold,
              int* __restrict__ num_person, float* __restrict__ ans, int* __restrict__ status) {
    __shared__ FuShared s;
    const int img = blockIdx.x, lane = threadIdx.x;
    const int* cnt = count + (size_t)img * C;
    const float* v = val + (size_t)img * C * M;
    const float* tg = tag + (size_t)img * C * M;
    const int* id2 = ind + (size_t)img * C * M * 2;
    float* a = ans + (size_t)img * M * C * 4;
    int num = 0, st = 0;
    for (int idj = 0; idj < C && st == 0; ++idj) {
        const int i = joint_order[idj];
        const int ci = cnt[i];
        if (ci == 0) continue;
        if (num == 0) {
            num = ci;
            if (lane < num) {
                const int p = i * M + lane, q = (lane * C + i) << 2;
                a[q] = (float)id2[p << 1];
                a[q | 1] = (float)id2[(p << 1) | 1];
                a[q | 2] = v[p];
                a[q | 3] = tg[p];
                s.nj[lane] = 1;
                s.sum[lane] = tg[p];
            }
            __syncwarp();
            continue;
        }
        const int n = max(num, ci);
        // lanes = candidates k, loop over persons j (assign.cpp:92-98)
        for (int j = 0; j < n; ++j) {
            if (lane < n) {
                float df = 1e4f, g = -1e4f;
                if (j < num && lane < ci) {
                    const int pre = i * M + lane;
                    // `1.0 * sum[j] / nj[j]`: double quotient narrowed to dist()'s float parameter
                    const float mean = __double2float_rn(__ddiv_rn((double)s.sum[j], (double)s.nj[j]));
                    const float dd = __fsub_rn(mean, tg[pre]);
                    df = __fsqrt_rn(__fmul_rn(dd, dd));
                    g = -__fsub_rn(__fmul_rn(df, 100.f), v[pre]);
                }
                s.diff[j][lane] = df;
                s.G[j][lane] = g;
            }
        }
        __syncwarp();
        if (!fu_km(s, n, lane)) {
            st = 1;
            break;
        }
        if (lane == 0) {      // assign.cpp:100-120: order dependent (new persons are appended as they appear)
            const int old_num = num;
            for (int j = 0; j < n; ++j) {
                const int c = s.ch[j];
                if (c >= ci) continue;
                const int p = i * M + c;
                int row;
                if (j < old_num && s.diff[j][c] < threshold) {
                    row = j;
                    s.nj[j]++;
                    s.sum[j] = __fadd_rn(s.sum[j], tg[p]);
                } else {
                    if (num == M) continue;
                    row = num;
                    s.nj[num] = 1;
                    s.sum[num] = tg[p];
                    num++;
                }
                const int q = (row * C + i) << 2;
                a[q] = (float)id2[p << 1];
                a[q | 1] = (float)id2[(p << 1) | 1];
                a[q | 2] = v[p];
                a[q | 3] = tg[p];
            }
        }
        num = __shfl_sync(0xffffffffu, num, 0);
        __syncwarp();
    }
    if (lane == 0) {
        num_person[img] = num;
        status[img] = st;
    }
}

}  // namespace lp

using namespace lp;

extern "C" int lp_find_peaks_f32(const float* input, const float* tmap, int N, int C, int H, int W, int M,
                                 float threshold, int window_size, int* count, float* val, float* tag, int* ind,
                                 lp_stream_t stream) {
    LP_CHECK_ARG(input && tmap && count && val && tag && ind, "lp_find_peaks_f32: null pointer");
    LP_CHECK_ARG(N > 0 && C > 0 && H > 0 && W > 0 && M > 0 && window_size >= 0 && (long long)N * C <= 0x7fffffffll &&
                     (long long)H * W <= 0x7fffffffll,
                 "lp_find_peaks_f32: bad shape N=%d C=%d H=%d W=%d M=%d window=%d", N, C, H, W, M, window_size);
    find_peaks_kernel<<<N * C, FP_THREADS, 0, (cudaStream_t)stream>>>(input, tmap, H, W, M, threshold, window_size, count,
                                                                      val, tag, ind);
    LP_LAUNCH_CHECK("find_peaks_kernel");
    return LP_OK;
}

extern "C" int lp_find_peaks_maps_f32(const float* det, const float* tag, int N, int H, int W, const int32_t* hw_host,
                                      const lp_map_desc_t* desc, int J, int T, int tag_planes, int M, float threshold,
                                      int window_size, int32_t* count, float* val, float* tag_out, int32_t* ind,
                                      lp_stream_t stream) {
    LP_CHECK_ARG(det && tag && count && val && tag_out && ind, "lp_find_peaks_maps_f32: null pointer");
    LP_CHECK_ARG((hw_host == nullptr) == (desc == nullptr), "lp_find_peaks_maps_f32: hw_host and desc go together");
    LP_CHECK_ARG(N > 0 && J > 0 && T > 0 && M > 0 && window_size >= 0 && (tag_planes == 1 || tag_planes == J) &&
                     (long long)N * J <= 0x7fffffffll,
                 "lp_find_peaks_maps_f32: bad shape N=%d J=%d T=%d tag_planes=%d M=%d window=%d", N, J, T, tag_planes, M,
                 window_size);
    // one CTA per plane whatever its size: the host sizes only validate the planes
    for (int n = 0; n < (hw_host ? N : 1); ++n) {
        const int h = hw_host ? hw_host[2 * n] : H, w = hw_host ? hw_host[2 * n + 1] : W;
        LP_CHECK_ARG(h > 0 && w > 0 && (long long)h * w <= 0x7fffffffll, "lp_find_peaks_maps_f32: bad map size %dx%d "
                     "(image %d)", h, w, n);
    }
    find_peaks_maps_kernel<<<N * J, FP_THREADS, 0, (cudaStream_t)stream>>>(det, tag, desc, J, H, W, T, tag_planes, M,
                                                                           threshold, window_size, count, val, tag_out,
                                                                           ind);
    LP_LAUNCH_CHECK("find_peaks_maps_kernel");
    return LP_OK;
}

extern "C" int lp_assign_f32(const int* count, const float* val, const float* tag, const int* ind, const int* joint_order,
                             int N, int C, int M, float threshold, int* num_person, float* ans, int* status,
                             lp_stream_t stream) {
    LP_CHECK_ARG(count && val && tag && ind && joint_order && num_person && ans && status, "lp_assign_f32: null pointer");
    LP_CHECK_ARG(N > 0 && C > 0 && M > 0, "lp_assign_f32: bad shape N=%d C=%d M=%d", N, C, M);
    if (M > FU_MAXP) {
        set_error("lp_assign_f32: max_count %d exceeds the %d candidates/persons this build holds per joint", M, FU_MAXP);
        return LP_ERR_CAPACITY;
    }
    assign_kernel<<<N, 32, 0, (cudaStream_t)stream>>>(count, val, tag, ind, joint_order, C, M, threshold, num_person, ans,
                                                     status);
    LP_LAUNCH_CHECK("assign_kernel");
    return LP_OK;
}
