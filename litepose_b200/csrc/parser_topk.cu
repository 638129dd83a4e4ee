// G1+G2: heat-map NMS + top-K peak pick on the device (reference lib/core/group.py:131-176).
//   nms:   det * (maxpool_kxk(det) == det), -inf padding                  (group.py:131-135)
//   top_k: K largest of the H*W NMS'd values per (n, j), tags gathered     (group.py:141-176)
// Canonical order (torch.topk's tie order is unspecified): value desc, flat index asc over
// survivors with value > 0; unused slots are (0.0f, index 0)  -- same rule as oracle/group_ref.py.
//
// HBM-bound: det is read once (algorithmic bytes 4*N*J*H*W).  Kernel 1: one CTA per band of rows of one
// plane keeps a running sorted top-K of 64-bit keys (value bits << 32 | ~index); the window maximum is
// evaluated only for pixels that reach the current K-th value; candidates are compacted with warp
// ballots and merged by one warp.  Kernel 2: one warp per plane merges the per-band lists and gathers tags.
#include <math.h>

#include "common.cuh"

namespace lp {

constexpr int TK_THREADS = 256;
constexpr int TK_MAXK = 64;

__device__ __forceinline__ unsigned long long shfl_max_u64(unsigned long long v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        unsigned long long other = __shfl_xor_sync(0xffffffffu, v, o);
        v = other > v ? other : v;
    }
    return v;
}

__host__ __device__ inline int strip_rows(int W) {
    // keep both shared planes (rows + halo) under ~96 KB
    int sr = 16;
    while (sr > 2 && (size_t)(sr + 8) * W * 8 > 96 * 1024) sr >>= 1;
    return sr;
}

constexpr int TK_SPB = 4;        // strips walked sequentially by one CTA (a "band")

__host__ __device__ inline int plane_bands(int H, int W) {
    const int sr = strip_rows(W);
    return ((H + sr - 1) / sr + TK_SPB - 1) / TK_SPB;
}

// Sorted insert of `key` into the descending list s_top[0..ntop) (capacity K <= 64) by one warp.
__device__ __forceinline__ int topk_insert(unsigned long long* s_top, int ntop, int K, unsigned long long key, int lane) {
    const unsigned long long a = lane < ntop ? s_top[lane] : 0ull;
    const unsigned long long b = (lane + 32) < ntop ? s_top[lane + 32] : 0ull;
    const int pos = __popc(__ballot_sync(0xffffffffu, a > key)) + __popc(__ballot_sync(0xffffffffu, b > key));
    if (pos >= K) return ntop;
    const int nnew = ntop < K ? ntop + 1 : K;
    // shift [pos, nnew-1) right by one: element i takes old element i-1
    const unsigned long long pa = __shfl_up_sync(0xffffffffu, a, 1);
    unsigned long long pb = __shfl_up_sync(0xffffffffu, b, 1);
    const unsigned long long a31 = __shfl_sync(0xffffffffu, a, 31);
    if (lane == 0) pb = a31;
    __syncwarp();
    if (lane > pos && lane < nnew) s_top[lane] = pa;
    if (lane + 32 > pos && lane + 32 < nnew) s_top[lane + 32] = pb;
    if (lane == 0) s_top[pos] = key;
    __syncwarp();
    return nnew;
}

constexpr int TK_WARPS = TK_THREADS / 32;

// Geometry of one (image, joint) plane.  Uniform call (desc == nullptr): every plane is H x W, planes are adjacent, the
// per-warp candidate lists of plane p start at p * nbands * TK_WARPS * K.  Ragged call: image n = plane / J has its own
// size and det / tag offsets (desc[n]); its lists follow those of images 0..n-1 (prefix sum over the images).
struct PlaneGeom {
    int H, W, SR, nbands;
    size_t det_off, tag_off, list_off;
};

__device__ __forceinline__ PlaneGeom plane_geom(const lp_map_desc_t* desc, int plane, int J, int H, int W, int T, int K) {
    PlaneGeom g;
    if (desc == nullptr) {
        g.H = H;
        g.W = W;
        g.SR = strip_rows(W);
        g.nbands = plane_bands(H, W);
        g.det_off = (size_t)plane * H * W;
        g.tag_off = (size_t)plane * H * W * T;
        g.list_off = (size_t)plane * g.nbands * TK_WARPS * K;
        return g;
    }
    const int n = plane / J, j = plane - n * J;
    size_t lists = 0;
    for (int i = 0; i < n; ++i) lists += (size_t)J * plane_bands(desc[i].h, desc[i].w) * TK_WARPS * K;
    g.H = desc[n].h;
    g.W = desc[n].w;
    g.SR = strip_rows(g.W);
    g.nbands = plane_bands(g.H, g.W);
    g.det_off = (size_t)desc[n].det_offset + (size_t)j * g.H * g.W;
    g.tag_off = (size_t)desc[n].tag_offset + (size_t)j * g.H * g.W * T;
    g.list_off = lists + (size_t)j * g.nbands * TK_WARPS * K;
    return g;
}

// partial: per plane [bands * TK_WARPS][K] keys (PlaneGeom::list_off) (sorted, 0 = empty); plane_thr: [N*J] running lower bound of the plane's
// K-th key (zero-initialised by the caller).  One CTA walks TK_SPB strips of SR rows of one plane; inside a strip every
// warp owns the rows r == warp (mod 8) and keeps its OWN sorted top-K list (no block barriers, no serial merge).  A pixel
// can only matter if its key reaches the best known K-th key -- the maximum over all warps of the CTA (shared memory)
// and over all CTAs of the plane (global memory) of their local K-th keys, each a valid lower bound of the plane's
// K-th key -- so the k x k window maximum (the NMS test) is evaluated for a vanishing fraction of pixels and the
// kernel streams at memory speed.  The per-warp lists are merged by topk_merge_kernel.
__global__ void __launch_bounds__(TK_THREADS)
nms_topk_strip_kernel(const float* __restrict__ det, const lp_map_desc_t* __restrict__ desc, int J, int H_u, int W_u,
                      int R /*window radius*/, int K, float floor_v, unsigned long long* __restrict__ partial,
                      unsigned long long* __restrict__ plane_thr) {
    extern __shared__ __align__(16) float sm[];
    const int plane = blockIdx.y;
    const PlaneGeom geo = plane_geom(desc, plane, J, H_u, W_u, 1, K);
    const int band = blockIdx.x;
    if (band >= geo.nbands) return;                // ragged: the grid covers the image with the most bands
    const int H = geo.H, W = geo.W, SR = geo.SR;
    float* s_val = sm;                             // [SR+2R][W] raw values (out-of-image rows hold -inf)
    __shared__ unsigned long long s_top[TK_WARPS][TK_MAXK];
    __shared__ unsigned long long s_thr;           // CTA-wide lower bound of the K-th key
    const float* p = det + geo.det_off;
    const float NEG_INF = __int_as_float(0xff800000);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int i = lane; i < TK_MAXK; i += 32) s_top[warp][i] = 0ull;
    if (threadIdx.x == 0) s_thr = 0ull;
    int ntop = 0;
    unsigned long long* mytop = s_top[warp];
    const bool vec = (W & 3) == 0 && ((reinterpret_cast<uintptr_t>(p) & 15) == 0);

    for (int st = 0; st < TK_SPB; ++st) {
        const int y0 = (band * TK_SPB + st) * SR;
        if (y0 >= H) break;
        const int rows = min(SR, H - y0);
        const int hrows = rows + 2 * R;
        __syncthreads();                           // previous strip fully consumed
        if (vec) {
            const int w4 = W >> 2;
            for (int i = threadIdx.x; i < hrows * w4; i += TK_THREADS * 4) {
                float4 tmp[4];
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    const int q = i + u * TK_THREADS;
                    const int r = q / w4, c = q - r * w4;
                    const int gy = y0 - R + r;
                    tmp[u] = (q < hrows * w4 && gy >= 0 && gy < H)
                                 ? __ldg(reinterpret_cast<const float4*>(p + (size_t)gy * W) + c)
                                 : make_float4(NEG_INF, NEG_INF, NEG_INF, NEG_INF);
                }
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    const int q = i + u * TK_THREADS;
                    if (q < hrows * w4) reinterpret_cast<float4*>(s_val)[q] = tmp[u];
                }
            }
        } else {
            for (int i = threadIdx.x; i < hrows * W; i += TK_THREADS) {
                const int r = i / W, x = i - r * W;
                const int gy = y0 - R + r;
                s_val[i] = (gy >= 0 && gy < H) ? __ldg(p + (size_t)gy * W + x) : NEG_INF;
            }
        }
        __syncthreads();
        // refresh the bound with what the other CTAs of this plane have found so far
        unsigned long long thr = s_thr;
        {
            const unsigned long long g = *reinterpret_cast<volatile unsigned long long*>(plane_thr + plane);
            thr = g > thr ? g : thr;
        }
        // Test of one pixel that passed the cheap value test: NMS window maximum, then the key (0 = no candidate).
        auto pixel_key = [&](int r, int x, float v) -> unsigned long long {
            const float* c = s_val + (r + R) * W + x;
            // cheap reject first: most pixels lose against a direct neighbour
            const float l = x > 0 ? c[-1] : NEG_INF, rr = x < W - 1 ? c[1] : NEG_INF;
            if (R > 0 && !(v >= l && v >= rr && v >= c[-W] && v >= c[W])) return 0ull;
            float m = NEG_INF;
            const int xa = max(x - R, 0), xb = min(x + R, W - 1);
            for (int d = 0; d <= 2 * R; ++d)
                for (int xx = xa; xx <= xb; ++xx) m = fmaxf(m, s_val[(r + d) * W + xx]);
            if (v != m) return 0ull;
            const unsigned idx = (unsigned)((y0 + r) * W + x);
            return ((unsigned long long)__float_as_uint(v) << 32) | (0xffffffffu - idx);
        };
        // Warp-wide insertion of the lanes' keys (ascending lane order) into this warp's list; refreshes the bound.
        auto insert_keys = [&](unsigned long long key) {
            unsigned bal = __ballot_sync(0xffffffffu, key > thr);
            if (!bal) return;
            while (bal) {
                const int src = __ffs(bal) - 1;
                bal &= bal - 1;
                const unsigned long long k2 = __shfl_sync(0xffffffffu, key, src);
                ntop = topk_insert(mytop, ntop, K, k2, lane);
            }
            if (ntop >= K) {
                const unsigned long long kth = mytop[K - 1];
                if (kth > thr) {
                    if (lane == 0) atomicMax(&s_thr, kth);
                    thr = kth;
                }
            }
        };
        for (int r = warp; r < rows; r += TK_WARPS) {
            if (vec) {
                // 4 pixels per lane (one 16-byte shared load), 128 per warp step; the slow path runs per sub-pixel
                for (int x0 = 0; x0 < W; x0 += 128) {
                    const int x = x0 + 4 * lane;
                    const float thr_v = __uint_as_float((unsigned)(thr >> 32));      // 0 while no list is full
                    float4 q = make_float4(0.f, 0.f, 0.f, 0.f);
                    if (x < W) q = *reinterpret_cast<const float4*>(s_val + (r + R) * W + x);
                    const float vv[4] = {q.x, q.y, q.z, q.w};
                    bool c4[4];
                    bool any4 = false;
#pragma unroll
                    for (int u = 0; u < 4; ++u) {
                        c4[u] = vv[u] > floor_v && vv[u] >= thr_v;
                        any4 |= c4[u];
                    }
                    if (__any_sync(0xffffffffu, any4)) {
#pragma unroll
                        for (int u = 0; u < 4; ++u) {
                            if (!__any_sync(0xffffffffu, c4[u])) continue;
                            insert_keys(c4[u] ? pixel_key(r, x + u, vv[u]) : 0ull);
                        }
                    }
                    // pick up the bound published by the other warps
                    const unsigned long long sh = *reinterpret_cast<volatile unsigned long long*>(&s_thr);
                    thr = sh > thr ? sh : thr;
                }
            } else {
                for (int x0 = 0; x0 < W; x0 += 32) {
                    const int x = x0 + lane;
                    const float thr_v = __uint_as_float((unsigned)(thr >> 32));
                    const float v = x < W ? s_val[(r + R) * W + x] : 0.f;
                    const bool cand = v > floor_v && v >= thr_v;
                    if (__any_sync(0xffffffffu, cand)) insert_keys(cand ? pixel_key(r, x, v) : 0ull);
                    const unsigned long long sh = *reinterpret_cast<volatile unsigned long long*>(&s_thr);
                    thr = sh > thr ? sh : thr;
                }
            }
        }
        // publish this CTA's bound to the plane
        __syncwarp();
        if (lane == 0 && thr) atomicMax(plane_thr + plane, thr);
    }
    __syncwarp();
    unsigned long long* out = partial + geo.list_off + ((size_t)band * TK_WARPS + warp) * K;
    for (int k = lane; k < K; k += 32) out[k] = k < ntop ? mytop[k] : 0ull;
}

// one warp per plane
__global__ void __launch_bounds__(32)
topk_merge_kernel(const unsigned long long* __restrict__ partial, const float* __restrict__ tag,
                  const lp_map_desc_t* __restrict__ desc, int J, int H_u, int W_u, int T, int K, float* __restrict__ val_k,
                  int32_t* __restrict__ ind_k, float* __restrict__ tag_k) {
    const int plane = blockIdx.x;
    const int lane = threadIdx.x;
    const PlaneGeom geo = plane_geom(desc, plane, J, H_u, W_u, T, K);
    const int nstrips = geo.nbands * TK_WARPS;
    const unsigned long long* pl = partial + geo.list_off;
    const float* tg = tag + geo.tag_off;
    // each lane owns strips lane, lane+32, ...; head[] = cursor into each sorted strip list
    constexpr int MAXS = 8;   // up to 256 strips
    int head[MAXS];
#pragma unroll
    for (int i = 0; i < MAXS; ++i) head[i] = 0;
    for (int k = 0; k < K; ++k) {
        unsigned long long best = 0ull;
        int bi = -1;
#pragma unroll
        for (int i = 0; i < MAXS; ++i) {
            const int s = lane + 32 * i;
            if (s < nstrips && head[i] < K) {
                const unsigned long long v = pl[(size_t)s * K + head[i]];
                if (v > best) { best = v; bi = i; }
            }
        }
        const unsigned long long win = shfl_max_u64(best);
        if (win != 0ull && best == win) {   // keys are unique (index part), exactly one lane matches
#pragma unroll
            for (int i = 0; i < MAXS; ++i)
                if (i == bi) head[i]++;
        }
        if (lane == 0) {
            float v = 0.f;
            int idx = 0;
            if (win != 0ull) {
                v = __uint_as_float((unsigned)(win >> 32));
                idx = (int)(0xffffffffu - (unsigned)(win & 0xffffffffu));
            }
            val_k[(size_t)plane * K + k] = v;
            ind_k[(size_t)plane * K + k] = idx;
            for (int t = 0; t < T; ++t)
                tag_k[((size_t)plane * K + k) * T + t] = __ldg(tg + (size_t)idx * T + t);
        }
    }
}

}  // namespace lp

using namespace lp;

static size_t topk_list_bytes(int J, int H, int W, int K) {
    return (size_t)J * plane_bands(H, W) * TK_WARPS * K * sizeof(unsigned long long);
}

// floor_v: (double)v > min_value  <=>  v > floor_v with floor_v = min_value rounded DOWN to float (the reference compares
// the float32 values with a Python float, i.e. in double: group.py:43)
static float topk_floor(double min_value) {
    float floor_v = 0.f;
    if (min_value > 0.0) {
        floor_v = (float)min_value;
        if ((double)floor_v > min_value) floor_v = nextafterf(floor_v, 0.f);
    }
    return floor_v;
}

// Both entry points: validate, then the strip kernel over (max bands, N*J planes) and one merge warp per plane.
static int topk_launch(const float* det, const float* tag, int N, const int32_t* hw_host, const lp_map_desc_t* desc,
                       int J, int H, int W, int T, int nms_kernel, int K, double min_value, float* val_k, int32_t* ind_k,
                       float* tag_k, void* workspace, size_t workspace_bytes, size_t need, lp_stream_t stream,
                       const char* name) {
    LP_CHECK_ARG(det && tag && val_k && ind_k && tag_k && workspace, "%s: null pointer", name);
    LP_CHECK_ARG(K > 0 && K <= TK_MAXK, "%s: K=%d out of range (1..%d)", name, K, TK_MAXK);
    LP_CHECK_ARG(nms_kernel >= 1 && nms_kernel <= 9 && (nms_kernel & 1), "%s: NMS kernel %d must be odd, <= 9", name,
                 nms_kernel);
    LP_CHECK_ARG((long long)N * J <= 65535, "%s: N*J=%lld exceeds the grid limit 65535", name, (long long)N * J);
    const int R = nms_kernel / 2;
    int max_bands = 0;
    size_t smem = 0;
    for (int n = 0; n < (hw_host ? N : 1); ++n) {
        const int h = hw_host ? hw_host[2 * n] : H, w = hw_host ? hw_host[2 * n + 1] : W;
        LP_CHECK_ARG(h > 0 && w > 0 && (long long)h * w < (1ll << 31), "%s: bad map size %dx%d (image %d)", name, h, w, n);
        const int nb = plane_bands(h, w);
        LP_CHECK_ARG(nb * TK_WARPS <= 256, "%s: plane too large (H=%d W=%d)", name, h, w);
        const size_t sm = (size_t)(strip_rows(w) + 2 * R) * w * sizeof(float);
        LP_CHECK_ARG(sm <= 200 * 1024, "%s: W=%d too wide for the strip buffers", name, w);
        max_bands = nb > max_bands ? nb : max_bands;
        smem = sm > smem ? sm : smem;
    }
    if (workspace_bytes < need) {
        set_error("%s: workspace %zu < required %zu bytes", name, workspace_bytes, need);
        return LP_ERR_CAPACITY;
    }
    cudaError_t e = cudaFuncSetAttribute((const void*)nms_topk_strip_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)smem);
    if (e != cudaSuccess) return cuda_fail(e, "cudaFuncSetAttribute(nms_topk)");
    cudaStream_t s = (cudaStream_t)stream;
    const size_t planes = (size_t)N * J;
    unsigned long long* lists = reinterpret_cast<unsigned long long*>(workspace);
    unsigned long long* plane_thr = lists + (need - planes * sizeof(unsigned long long)) / sizeof(unsigned long long);
    cudaError_t em = cudaMemsetAsync(plane_thr, 0, planes * sizeof(unsigned long long), s);
    if (em != cudaSuccess) return cuda_fail(em, "cudaMemsetAsync(plane_thr)");
    dim3 grid(max_bands, N * J);
    nms_topk_strip_kernel<<<grid, TK_THREADS, smem, s>>>(det, desc, J, H, W, R, K, topk_floor(min_value), lists, plane_thr);
    LP_LAUNCH_CHECK("nms_topk_strip_kernel");
    topk_merge_kernel<<<N * J, 32, 0, s>>>(lists, tag, desc, J, H, W, T, K, val_k, ind_k, tag_k);
    LP_LAUNCH_CHECK("topk_merge_kernel");
    return LP_OK;
}

extern "C" size_t lp_nms_topk_workspace_bytes(int N, int J, int H, int W, int K) {
    if (N <= 0 || J <= 0 || H <= 0 || W <= 0 || K <= 0) return 0;
    // per-warp candidate lists + one running threshold per plane
    return (size_t)N * topk_list_bytes(J, H, W, K) + (size_t)N * J * sizeof(unsigned long long);
}

extern "C" int lp_nms_topk_f32(const float* det, const float* tag, int N, int J, int H, int W, int T, int nms_kernel,
                               int K, double min_value, float* val_k, int32_t* ind_k, float* tag_k, void* workspace,
                               size_t workspace_bytes, lp_stream_t stream) {
    LP_CHECK_ARG(N > 0 && J > 0 && H > 0 && W > 0 && T > 0 && (long long)H * W < (1ll << 31),
                 "lp_nms_topk_f32: bad shape N=%d J=%d H=%d W=%d T=%d", N, J, H, W, T);
    return topk_launch(det, tag, N, nullptr, nullptr, J, H, W, T, nms_kernel, K, min_value, val_k, ind_k, tag_k, workspace,
                       workspace_bytes, lp_nms_topk_workspace_bytes(N, J, H, W, K), stream, "lp_nms_topk_f32");
}

extern "C" size_t lp_nms_topk_ragged_workspace_bytes(int N, const int32_t* hw_host, int J, int K) {
    if (N <= 0 || !hw_host || J <= 0 || K <= 0) return 0;
    size_t b = (size_t)N * J * sizeof(unsigned long long);
    for (int n = 0; n < N; ++n) {
        if (hw_host[2 * n] <= 0 || hw_host[2 * n + 1] <= 0) return 0;
        b += topk_list_bytes(J, hw_host[2 * n], hw_host[2 * n + 1], K);
    }
    return b;
}

extern "C" int lp_nms_topk_ragged_f32(const float* det, const float* tag, int N, const int32_t* hw_host,
                                      const lp_map_desc_t* desc, int J, int T, int nms_kernel, int K, double min_value,
                                      float* val_k, int32_t* ind_k, float* tag_k, void* workspace, size_t workspace_bytes,
                                      lp_stream_t stream) {
    LP_CHECK_ARG(hw_host && desc, "lp_nms_topk_ragged_f32: null pointer");
    LP_CHECK_ARG(N > 0 && J > 0 && T > 0, "lp_nms_topk_ragged_f32: bad shape N=%d J=%d T=%d", N, J, T);
    return topk_launch(det, tag, N, hw_host, desc, J, 0, 0, T, nms_kernel, K, min_value, val_k, ind_k, tag_k, workspace,
                       workspace_bytes, lp_nms_topk_ragged_workspace_bytes(N, hw_host, J, K), stream,
                       "lp_nms_topk_ragged_f32");
}
