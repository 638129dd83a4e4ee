// G3: tag-distance grouping on the device -- match_by_tag + Munkres
// (reference lib/core/group.py:19-97; third-party `munkres` package restated in
// oracle/munkres_ref.py, SURVEY.md Appendix A.7/A.8).
//
// One warp per image (images are independent, SURVEY H5); joints are processed sequentially in
// joint_order like the reference, the inner searches/reductions run across the 32 lanes
// (lane <-> cost-matrix column).  Bit-exact requirements reproduced here:
//   * joints rows are float64 in the reference: the threshold tests run in double;
//   * running person tag = np.mean(list of f32 vectors, axis=0): sequential f32 sum / count for
//     T >= 2, numpy's 8-accumulator pairwise sum for T == 1 (measured, see oracle/group_ref.py);
//   * cost = rint(||dtag||_2) * 100 - val in double, no FMA contraction; 1e10 padding columns;
//   * the exact Munkres step sequence (cyclic scan, LAST zero of the first row that has one);
//   * person identity = float32 tag[0] with dict semantics (equal keys collide, insertion order).
#include <cstdlib>

#include "common.cuh"

namespace lp {

constexpr int MM = 32;   // max matrix side == warp width

struct MatchSmem {
    double C[MM][MM + 1];
    double saved[MM][MM + 1];
    float ct[MM][8];        // candidate tags (T <= 8)
    float mean[MM][8];
    float cv[MM];
    int cx[MM], cy[MM];
    int star_col[MM], star_row[MM], prime_col[MM];
    int P;
};

__device__ __forceinline__ double warp_min_d(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const double other = __shfl_xor_sync(0xffffffffu, v, o);
        v = other < v ? other : v;
    }
    return v;
}

// Munkres on the n x n matrix S.C (n <= 32); result in S.star_col[row]
__device__ void munkres_warp(MatchSmem& S, const int n, const int lane) {
    const double INF = __longlong_as_double(0x7ff0000000000000ll);
    const bool act = lane < n;
    // step 1
    for (int i = 0; i < n; ++i) {
        const double v = act ? S.C[i][lane] : INF;
        const double m = warp_min_d(v);
        if (act) S.C[i][lane] = v - m;
    }
    if (lane < MM) { S.star_col[lane] = -1; S.star_row[lane] = -1; S.prime_col[lane] = -1; }
    __syncwarp();
    // step 2
    unsigned col_cov = 0, row_cov = 0;
    for (int i = 0; i < n; ++i) {
        const unsigned z = __ballot_sync(0xffffffffu, act && S.C[i][lane] == 0.0 && !((col_cov >> lane) & 1u));
        if (z) {
            const int j = __ffs(z) - 1;
            if (lane == 0) { S.star_col[i] = j; S.star_row[j] = i; }
            col_cov |= 1u << j;
        }
    }
    __syncwarp();
    for (;;) {
        // step 3
        col_cov = __ballot_sync(0xffffffffu, act && S.star_row[lane] >= 0);
        row_cov = 0;
        if (__popc(col_cov) >= n) break;
        // step 4 (+ step 6 when no uncovered zero is left)
        int row = 0, col = 0;
        int z0r = -1, z0c = -1;
        for (;;) {
            int fr = -1, fc = -1;
            for (int ii = 0; ii < n; ++ii) {
                int i = row + ii;
                if (i >= n) i -= n;
                if ((row_cov >> i) & 1u) continue;
                const unsigned z = __ballot_sync(0xffffffffu, act && S.C[i][lane] == 0.0 && !((col_cov >> lane) & 1u));
                if (z) {
                    const unsigned low = z & ((1u << col) - 1u);   // columns scanned after the wrap-around
                    fc = low ? (31 - __clz(low)) : (31 - __clz(z));
                    fr = i;
                    break;
                }
            }
            if (fr < 0) {
                // step 6
                double m = INF;
                if (act && !((col_cov >> lane) & 1u))
                    for (int i = 0; i < n; ++i)
                        if (!((row_cov >> i) & 1u)) { const double v = S.C[i][lane]; m = v < m ? v : m; }
                m = warp_min_d(m);
                if (act) {
                    const bool cu = !((col_cov >> lane) & 1u);
                    for (int i = 0; i < n; ++i) {
                        double v = S.C[i][lane];
                        if ((row_cov >> i) & 1u) v = __dadd_rn(v, m);
                        if (cu) v = __dsub_rn(v, m);
                        S.C[i][lane] = v;
                    }
                }
                __syncwarp();
                row = 0;
                col = 0;
                continue;
            }
            if (lane == 0) S.prime_col[fr] = fc;
            const int sc = S.star_col[fr];
            __syncwarp();
            if (sc >= 0) {
                row = fr;
                col = sc;
                row_cov |= 1u << fr;
                col_cov &= ~(1u << sc);
            } else {
                z0r = fr;
                z0c = fc;
                break;
            }
        }
        // step 5
        if (lane == 0) {
            int r = z0r, c = z0c;
            for (;;) {
                const int sr = S.star_row[c];
                S.star_row[c] = r;
                S.star_col[r] = c;
                if (sr < 0) break;
                r = sr;
                c = S.prime_col[sr];
            }
        }
        __syncwarp();
        if (lane < MM) S.prime_col[lane] = -1;
        __syncwarp();
    }
}

// numpy add.reduce order for a contiguous 1-D float32 run of n < 128 elements
__device__ float np_pairwise_sum_f32(const float* a, int n, int stride) {
    if (n < 8) {
        float r = 0.f;
        for (int i = 0; i < n; ++i) r = __fadd_rn(r, a[i * stride]);
        return r;
    }
    float r[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) r[j] = a[j * stride];
    int i = 8;
    for (; i < n - (n % 8); i += 8)
#pragma unroll
        for (int j = 0; j < 8; ++j) r[j] = __fadd_rn(r[j], a[(i + j) * stride]);
    float res = __fadd_rn(__fadd_rn(__fadd_rn(r[0], r[1]), __fadd_rn(r[2], r[3])),
                          __fadd_rn(__fadd_rn(r[4], r[5]), __fadd_rn(r[6], r[7])));
    for (; i < n; ++i) res = __fadd_rn(res, a[i * stride]);
    return res;
}

struct MatchArgs {
    const float* val_k; const int32_t* ind_k; const float* tag_k;
    int N, J, K, T, W;
    const lp_map_desc_t* desc;                   // ragged call: per-image map width desc[n].w (else W)
    const int32_t* joint_order;
    double det_thr, tag_thr;
    int use_det_val, ignore_too_much, max_people, pcap;
    float* ans; int32_t* num_people;
    float* pkey; int32_t* ptagn; float* ptags;   // workspace
};

__device__ int find_person(const MatchArgs& a, const float* pkey, int P, float key, int lane) {
    const int lim = P < a.pcap ? P : a.pcap;
    for (int p0 = 0; p0 < lim; p0 += 32) {
        const int p = p0 + lane;
        const unsigned m = __ballot_sync(0xffffffffu, p < lim && pkey[p] == key);
        if (m) return p0 + __ffs(m) - 1;
    }
    return -1;
}

__global__ void __launch_bounds__(32)
tag_match_kernel(const MatchArgs a) {
    __shared__ MatchSmem S;
    const int n = blockIdx.x;
    const int lane = threadIdx.x;
    const int J = a.J, K = a.K, T = a.T, D = 3 + a.T;
    const int W = a.desc ? a.desc[n].w : a.W;
    float* ans = a.ans + (size_t)n * a.pcap * J * D;
    float* pkey = a.pkey + (size_t)n * a.pcap;
    int32_t* ptagn = a.ptagn + (size_t)n * a.pcap;
    float* ptags = a.ptags + (size_t)n * a.pcap * J * T;
    int P = 0;

    // setdefault(key, zeros)[idx] = joint ; tag_dict[key] = [tag]
    auto new_or_reset = [&](int r, int idx) {
        const float key = S.ct[r][0];
        int p = find_person(a, pkey, P, key, lane);
        if (p < 0) {
            p = P++;
            if (p < a.pcap) {
                for (int e = lane; e < J * D; e += 32) ans[(size_t)p * J * D + e] = 0.f;
                if (lane == 0) pkey[p] = key;
            }
        }
        __syncwarp();
        if (p < a.pcap) {
            float* row = ans + ((size_t)p * J + idx) * D;
            if (lane == 0) {
                row[0] = (float)S.cx[r];
                row[1] = (float)S.cy[r];
                row[2] = S.cv[r];
                ptagn[p] = 1;
            }
            if (lane < T) {
                row[3 + lane] = S.ct[r][lane];
                ptags[((size_t)p * J + 0) * T + lane] = S.ct[r][lane];
            }
        }
        __syncwarp();
    };

    for (int ji = 0; ji < J; ++ji) {
        const int idx = a.joint_order[ji];
        const size_t base = ((size_t)n * J + idx) * K;
        float v = 0.f;
        bool ok = false;
        if (lane < K) {
            v = a.val_k[base + lane];
            ok = (double)v > a.det_thr;
        }
        const unsigned mask = __ballot_sync(0xffffffffu, ok);
        const int rows = __popc(mask);
        if (rows == 0) continue;
        if (ok) {
            const int r = __popc(mask & ((1u << lane) - 1u));
            const int ind = a.ind_k[base + lane];
            S.cx[r] = ind % W;
            S.cy[r] = ind / W;
            S.cv[r] = v;
            for (int t = 0; t < T; ++t) S.ct[r][t] = a.tag_k[(base + lane) * T + t];
        }
        __syncwarp();

        if (ji == 0 || P == 0) {
            for (int r = 0; r < rows; ++r) new_or_reset(r, idx);
            continue;
        }
        const int G = P < a.max_people ? P : a.max_people;
        if (a.ignore_too_much && G == a.max_people) continue;
        // running mean tag of each grouped person
        if (lane < G) {
            const int cnt = ptagn[lane];
            const float* tl = ptags + (size_t)lane * J * T;
            for (int t = 0; t < T; ++t) {
                float s;
                if (T == 1) {
                    s = np_pairwise_sum_f32(tl, cnt, 1);
                } else {
                    s = tl[t];
                    for (int q = 1; q < cnt; ++q) s = __fadd_rn(s, tl[q * T + t]);
                }
                S.mean[lane][t] = __fdiv_rn(s, (float)cnt);
            }
        }
        __syncwarp();
        const int nn = rows > G ? rows : G;
        for (int r = 0; r < nn; ++r) {
            if (lane < nn) {
                double c;
                if (r >= rows) {
                    c = 0.0;                       // Munkres pads missing rows with 0
                } else if (lane < G) {
                    double d2 = 0.0;
                    for (int t = 0; t < T; ++t) {
                        const double dd = __dsub_rn((double)S.ct[r][t], (double)S.mean[lane][t]);
                        const double sq = __dmul_rn(dd, dd);
                        d2 = (t == 0) ? sq : __dadd_rn(d2, sq);
                    }
                    const double d = sqrt(d2);
                    S.saved[r][lane] = d;
                    c = a.use_det_val ? __dsub_rn(__dmul_rn(rint(d), 100.0), (double)S.cv[r]) : d;
                } else {
                    c = 1e10;                      // reference pads columns with 1e10 when rows > cols
                }
                S.C[r][lane] = c;
            }
        }
        __syncwarp();
        munkres_warp(S, nn, lane);
        __syncwarp();
        for (int r = 0; r < rows; ++r) {
            const int c = S.star_col[r];
            const bool accept = (c >= 0) && (c < G) && (S.saved[r][c] < a.tag_thr);
            if (accept) {
                const int cnt = ptagn[c];
                float* row = ans + ((size_t)c * J + idx) * D;
                __syncwarp();
                if (lane == 0) {
                    row[0] = (float)S.cx[r];
                    row[1] = (float)S.cy[r];
                    row[2] = S.cv[r];
                    ptagn[c] = cnt + 1;
                }
                if (lane < T) {
                    row[3 + lane] = S.ct[r][lane];
                    if (cnt < J) ptags[((size_t)c * J + cnt) * T + lane] = S.ct[r][lane];
                }
                __syncwarp();
            } else {
                new_or_reset(r, idx);
            }
        }
    }
    if (lane == 0) a.num_people[n] = P;
}


// ---- wide variant: 32 < MAX_NUM_PEOPLE <= 64 (the reference has no limit, lib/config/default.py MAX_NUM_PEOPLE) ------
// Same algorithm, same scan orders and the same IEEE operations as above; lane l owns the cost-matrix columns l and
// l + 32, the cover sets are 64-bit masks built from two ballots.  Shared memory (two 64 x 65 double matrices) is
// dynamic.  LP_MATCH_WIDE=1 routes every call through this kernel (the tests run the goldens through both).
constexpr int MW = 64;

struct MatchSmemW {
    double C[MW][MW + 1];
    double saved[MW][MW + 1];
    float ct[MW][8];
    float mean[MW][8];
    float cv[MW];
    int cx[MW], cy[MW];
    int star_col[MW], star_row[MW], prime_col[MW];
};

typedef unsigned long long u64;

__device__ __forceinline__ u64 ballot64(bool p_lo, bool p_hi) {
    const unsigned lo = __ballot_sync(0xffffffffu, p_lo);
    const unsigned hi = __ballot_sync(0xffffffffu, p_hi);
    return (u64)lo | ((u64)hi << 32);
}
__device__ __forceinline__ bool bit64(u64 m, int i) { return (m >> i) & 1ull; }

// Munkres on the n x n matrix S.C (n <= 64); result in S.star_col[row]
__device__ void munkres_warp_wide(MatchSmemW& S, const int n, const int lane) {
    const double INF = __longlong_as_double(0x7ff0000000000000ll);
    const int c0 = lane, c1 = lane + 32;
    const bool act0 = c0 < n, act1 = c1 < n;
    // step 1
    for (int i = 0; i < n; ++i) {
        const double v0 = act0 ? S.C[i][c0] : INF;
        const double v1 = act1 ? S.C[i][c1] : INF;
        const double m = warp_min_d(v1 < v0 ? v1 : v0);
        if (act0) S.C[i][c0] = v0 - m;
        if (act1) S.C[i][c1] = v1 - m;
    }
    S.star_col[c0] = -1; S.star_row[c0] = -1; S.prime_col[c0] = -1;
    S.star_col[c1] = -1; S.star_row[c1] = -1; S.prime_col[c1] = -1;
    __syncwarp();
    // step 2
    u64 col_cov = 0, row_cov = 0;
    for (int i = 0; i < n; ++i) {
        const u64 z = ballot64(act0 && S.C[i][c0] == 0.0 && !bit64(col_cov, c0),
                               act1 && S.C[i][c1] == 0.0 && !bit64(col_cov, c1));
        if (z) {
            const int j = __ffsll((long long)z) - 1;
            if (lane == 0) { S.star_col[i] = j; S.star_row[j] = i; }
            col_cov |= 1ull << j;
        }
    }
    __syncwarp();
    for (;;) {
        // step 3
        col_cov = ballot64(act0 && S.star_row[c0] >= 0, act1 && S.star_row[c1] >= 0);
        row_cov = 0;
        if (__popcll(col_cov) >= n) break;
        // step 4 (+ step 6 when no uncovered zero is left)
        int row = 0, col = 0;
        int z0r = -1, z0c = -1;
        for (;;) {
            int fr = -1, fc = -1;
            for (int ii = 0; ii < n; ++ii) {
                int i = row + ii;
                if (i >= n) i -= n;
                if (bit64(row_cov, i)) continue;
                const u64 z = ballot64(act0 && S.C[i][c0] == 0.0 && !bit64(col_cov, c0),
                                       act1 && S.C[i][c1] == 0.0 && !bit64(col_cov, c1));
                if (z) {
                    const u64 low = z & ((1ull << col) - 1ull);   // columns scanned after the wrap-around (col < 64)
                    fc = low ? (63 - __clzll((long long)low)) : (63 - __clzll((long long)z));
                    fr = i;
                    break;
                }
            }
            if (fr < 0) {
                // step 6
                double m = INF;
                for (int s = 0; s < 2; ++s) {
                    const int c = lane + 32 * s;
                    if (c < n && !bit64(col_cov, c))
                        for (int i = 0; i < n; ++i)
                            if (!bit64(row_cov, i)) { const double v = S.C[i][c]; m = v < m ? v : m; }
                }
                m = warp_min_d(m);
                for (int s = 0; s < 2; ++s) {
                    const int c = lane + 32 * s;
                    if (c < n) {
                        const bool cu = !bit64(col_cov, c);
                        for (int i = 0; i < n; ++i) {
                            double v = S.C[i][c];
                            if (bit64(row_cov, i)) v = __dadd_rn(v, m);
                            if (cu) v = __dsub_rn(v, m);
                            S.C[i][c] = v;
                        }
                    }
                }
                __syncwarp();
                row = 0;
                col = 0;
                continue;
            }
            if (lane == 0) S.prime_col[fr] = fc;
            const int sc = S.star_col[fr];
            __syncwarp();
            if (sc >= 0) {
                row = fr;
                col = sc;
                row_cov |= 1ull << fr;
                col_cov &= ~(1ull << sc);
            } else {
                z0r = fr;
                z0c = fc;
                break;
            }
        }
        // step 5
        if (lane == 0) {
            int r = z0r, c = z0c;
            for (;;) {
                const int sr = S.star_row[c];
                S.star_row[c] = r;
                S.star_col[r] = c;
                if (sr < 0) break;
                r = sr;
                c = S.prime_col[sr];
            }
        }
        __syncwarp();
        S.prime_col[c0] = -1;
        S.prime_col[c1] = -1;
        __syncwarp();
    }
}

__global__ void __launch_bounds__(32)
tag_match_wide_kernel(const MatchArgs a) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    MatchSmemW& S = *reinterpret_cast<MatchSmemW*>(smem_raw);
    const int n = blockIdx.x;
    const int lane = threadIdx.x;
    const int J = a.J, K = a.K, T = a.T, D = 3 + a.T;
    const int W = a.desc ? a.desc[n].w : a.W;
    float* ans = a.ans + (size_t)n * a.pcap * J * D;
    float* pkey = a.pkey + (size_t)n * a.pcap;
    int32_t* ptagn = a.ptagn + (size_t)n * a.pcap;
    float* ptags = a.ptags + (size_t)n * a.pcap * J * T;
    int P = 0;

    auto new_or_reset = [&](int r, int idx) {
        const float key = S.ct[r][0];
        int p = find_person(a, pkey, P, key, lane);
        if (p < 0) {
            p = P++;
            if (p < a.pcap) {
                for (int e = lane; e < J * D; e += 32) ans[(size_t)p * J * D + e] = 0.f;
                if (lane == 0) pkey[p] = key;
            }
        }
        __syncwarp();
        if (p < a.pcap) {
            float* row = ans + ((size_t)p * J + idx) * D;
            if (lane == 0) {
                row[0] = (float)S.cx[r];
                row[1] = (float)S.cy[r];
                row[2] = S.cv[r];
                ptagn[p] = 1;
            }
            if (lane < T) {
                row[3 + lane] = S.ct[r][lane];
                ptags[((size_t)p * J + 0) * T + lane] = S.ct[r][lane];
            }
        }
        __syncwarp();
    };

    for (int ji = 0; ji < J; ++ji) {
        const int idx = a.joint_order[ji];
        const size_t base = ((size_t)n * J + idx) * K;
        float v[2] = {0.f, 0.f};
        bool ok[2] = {false, false};
        for (int s = 0; s < 2; ++s) {
            const int k = lane + 32 * s;
            if (k < K) {
                v[s] = a.val_k[base + k];
                ok[s] = (double)v[s] > a.det_thr;
            }
        }
        const u64 mask = ballot64(ok[0], ok[1]);
        const int rows = __popcll(mask);
        if (rows == 0) continue;
        for (int s = 0; s < 2; ++s) {
            const int k = lane + 32 * s;
            if (ok[s]) {
                const int r = __popcll(mask & ((1ull << k) - 1ull));
                const int ind = a.ind_k[base + k];
                S.cx[r] = ind % W;
                S.cy[r] = ind / W;
                S.cv[r] = v[s];
                for (int t = 0; t < T; ++t) S.ct[r][t] = a.tag_k[(base + k) * T + t];
            }
        }
        __syncwarp();

        if (ji == 0 || P == 0) {
            for (int r = 0; r < rows; ++r) new_or_reset(r, idx);
            continue;
        }
        const int G = P < a.max_people ? P : a.max_people;
        if (a.ignore_too_much && G == a.max_people) continue;
        // running mean tag of each grouped person
        for (int g = lane; g < G; g += 32) {
            const int cnt = ptagn[g];
            const float* tl = ptags + (size_t)g * J * T;
            for (int t = 0; t < T; ++t) {
                float sum;
                if (T == 1) {
                    sum = np_pairwise_sum_f32(tl, cnt, 1);
                } else {
                    sum = tl[t];
                    for (int q = 1; q < cnt; ++q) sum = __fadd_rn(sum, tl[q * T + t]);
                }
                S.mean[g][t] = __fdiv_rn(sum, (float)cnt);
            }
        }
        __syncwarp();
        const int nn = rows > G ? rows : G;
        for (int r = 0; r < nn; ++r) {
            for (int c = lane; c < nn; c += 32) {
                double cst;
                if (r >= rows) {
                    cst = 0.0;                     // Munkres pads missing rows with 0
                } else if (c < G) {
                    double d2 = 0.0;
                    for (int t = 0; t < T; ++t) {
                        const double dd = __dsub_rn((double)S.ct[r][t], (double)S.mean[c][t]);
                        const double sq = __dmul_rn(dd, dd);
                        d2 = (t == 0) ? sq : __dadd_rn(d2, sq);
                    }
                    const double d = sqrt(d2);
                    S.saved[r][c] = d;
                    cst = a.use_det_val ? __dsub_rn(__dmul_rn(rint(d), 100.0), (double)S.cv[r]) : d;
                } else {
                    cst = 1e10;                    // reference pads columns with 1e10 when rows > cols
                }
                S.C[r][c] = cst;
            }
        }
        __syncwarp();
        munkres_warp_wide(S, nn, lane);
        __syncwarp();
        for (int r = 0; r < rows; ++r) {
            const int c = S.star_col[r];
            const bool accept = (c >= 0) && (c < G) && (S.saved[r][c] < a.tag_thr);
            if (accept) {
                const int cnt = ptagn[c];
                float* row = ans + ((size_t)c * J + idx) * D;
                __syncwarp();
                if (lane == 0) {
                    row[0] = (float)S.cx[r];
                    row[1] = (float)S.cy[r];
                    row[2] = S.cv[r];
                    ptagn[c] = cnt + 1;
                }
                if (lane < T) {
                    row[3 + lane] = S.ct[r][lane];
                    if (cnt < J) ptags[((size_t)c * J + cnt) * T + lane] = S.ct[r][lane];
                }
                __syncwarp();
            } else {
                new_or_reset(r, idx);
            }
        }
    }
    if (lane == 0) a.num_people[n] = P;
}

}  // namespace lp

using namespace lp;

extern "C" size_t lp_tag_match_workspace_bytes(int N, int J, int K, int T, int pcap) {
    (void)K;
    if (N <= 0 || J <= 0 || T <= 0 || pcap <= 0) return 0;
    return (size_t)N * pcap * (sizeof(float) + sizeof(int32_t) + (size_t)J * T * sizeof(float));
}

// Both entry points: W > 0 (uniform) or desc != nullptr (ragged).
static int tag_match_launch(const float* val_k, const int32_t* ind_k, const float* tag_k, int N, int J, int K, int T,
                            int W, const lp_map_desc_t* desc, const int32_t* joint_order, double det_threshold,
                            double tag_threshold, int use_detection_val, int ignore_too_much, int max_num_people, int pcap,
                            float* ans, int32_t* num_people, void* workspace, size_t workspace_bytes, lp_stream_t stream,
                            const char* name) {
    LP_CHECK_ARG(val_k && ind_k && tag_k && joint_order && ans && num_people && workspace, "%s: null pointer", name);
    LP_CHECK_ARG(N > 0 && J > 0 && J <= 32 && K > 0 && K <= MW && T > 0 && T < 8 && (W > 0 || desc),
                 "%s: bad shape N=%d J=%d K=%d T=%d (J<=32, K<=64, T<8)", name, N, J, K, T);
    LP_CHECK_ARG(max_num_people > 0 && max_num_people <= MW, "%s: max_num_people=%d out of range (1..64)", name,
                 max_num_people);
    LP_CHECK_ARG(pcap >= max_num_people, "%s: pcap=%d must be >= max_num_people=%d", name, pcap, max_num_people);
    LP_CHECK_ARG(det_threshold >= 0.0, "%s: detection threshold must be >= 0", name);
    const size_t need = lp_tag_match_workspace_bytes(N, J, K, T, pcap);
    if (workspace_bytes < need) {
        set_error("%s: workspace %zu < required %zu bytes", name, workspace_bytes, need);
        return LP_ERR_CAPACITY;
    }
    MatchArgs a;
    a.val_k = val_k; a.ind_k = ind_k; a.tag_k = tag_k;
    a.N = N; a.J = J; a.K = K; a.T = T; a.W = W; a.desc = desc;
    a.joint_order = joint_order;
    a.det_thr = det_threshold; a.tag_thr = tag_threshold;
    a.use_det_val = use_detection_val; a.ignore_too_much = ignore_too_much;
    a.max_people = max_num_people; a.pcap = pcap;
    a.ans = ans; a.num_people = num_people;
    uint8_t* ws = reinterpret_cast<uint8_t*>(workspace);
    a.pkey = reinterpret_cast<float*>(ws);
    a.ptagn = reinterpret_cast<int32_t*>(ws + (size_t)N * pcap * sizeof(float));
    a.ptags = reinterpret_cast<float*>(ws + (size_t)N * pcap * (sizeof(float) + sizeof(int32_t)));
    const char* env_wide = getenv("LP_MATCH_WIDE");       // read per call: the tests flip it inside one process
    const bool force_wide = env_wide && env_wide[0] == '1';
    if (K > MM || max_num_people > MM || force_wide) {
        // cost matrices up to 64 x 64: two columns per lane, 70 KB of dynamic shared memory
        const cudaError_t attr = cudaFuncSetAttribute((const void*)tag_match_wide_kernel,
                                                      cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(MatchSmemW));
        if (attr != cudaSuccess) return cuda_fail(attr, "cudaFuncSetAttribute(tag_match_wide)");
        tag_match_wide_kernel<<<N, 32, sizeof(MatchSmemW), (cudaStream_t)stream>>>(a);
        LP_LAUNCH_CHECK("tag_match_wide_kernel");
        return LP_OK;
    }
    tag_match_kernel<<<N, 32, 0, (cudaStream_t)stream>>>(a);
    LP_LAUNCH_CHECK("tag_match_kernel");
    return LP_OK;
}

extern "C" int lp_tag_match_f32(const float* val_k, const int32_t* ind_k, const float* tag_k, int N, int J, int K, int T,
                                int W, const int32_t* joint_order, double det_threshold, double tag_threshold,
                                int use_detection_val, int ignore_too_much, int max_num_people, int pcap, float* ans,
                                int32_t* num_people, void* workspace, size_t workspace_bytes, lp_stream_t stream) {
    LP_CHECK_ARG(W > 0, "lp_tag_match_f32: bad shape W=%d", W);
    return tag_match_launch(val_k, ind_k, tag_k, N, J, K, T, W, nullptr, joint_order, det_threshold, tag_threshold,
                            use_detection_val, ignore_too_much, max_num_people, pcap, ans, num_people, workspace,
                            workspace_bytes, stream, "lp_tag_match_f32");
}

extern "C" int lp_tag_match_ragged_f32(const float* val_k, const int32_t* ind_k, const float* tag_k, int N, int J, int K,
                                       int T, const lp_map_desc_t* desc, const int32_t* joint_order, double det_threshold,
                                       double tag_threshold, int use_detection_val, int ignore_too_much,
                                       int max_num_people, int pcap, float* ans, int32_t* num_people, void* workspace,
                                       size_t workspace_bytes, lp_stream_t stream) {
    LP_CHECK_ARG(desc, "lp_tag_match_ragged_f32: null pointer");
    return tag_match_launch(val_k, ind_k, tag_k, N, J, K, T, 0, desc, joint_order, det_threshold, tag_threshold,
                            use_detection_val, ignore_too_much, max_num_people, pcap, ans, num_people, workspace,
                            workspace_bytes, stream, "lp_tag_match_ragged_f32");
}
