// Fixed-size host payload of one step + the synthetic benchmark's planted persons.
//
// lp_pack_payload_f32: what leaves the GPU per step is one row per image:
//   [ keep persons x J x (3+T) keypoints | keep scores | person count ]
// gathered from the parser's result buffers (ans [N,pcap,J,3+T], scores [N,pcap], num_people [N]) - the tensors that
// HeatmapParser.parse returns to valid.py:227 (reference lib/core/group.py:269-291) in a form one D2H copy / one NCCL
// gather can carry.  One launch instead of three strided torch copies.
//
// lp_pack_fast_payload_f32: the same for the fast grouping (find_peaks + KM assign, fast_utils.cu): every one of the
// at most M <= 32 persons (ans [N,M,C,4]), the person count and the KM status - no overflow path is needed.
//
// lp_plant_crowd_f32: a random-weight network detects nobody (SURVEY H8), so the benchmark plants persons into the
// projected maps between glue and parser: Gaussian patches max-composited into det (order independent), tag patches
// overwriting tag.  Index / value lists are built once on the host (litepose_b200.pipeline.PlantedCrowd).
#include "common.cuh"

namespace lp {

__global__ void __launch_bounds__(256)
pack_payload_kernel(const float* __restrict__ ans, const int32_t* __restrict__ num, const float* __restrict__ scores,
                    int pcap, int row, int keep, float* __restrict__ packed) {
    const int n = blockIdx.y;
    const int width = keep * row + keep + 1;
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= width) return;
    float v;
    if (e < keep * row) v = ans[(size_t)n * pcap * row + e];               // persons are contiguous rows of `row` floats
    else if (e < keep * row + keep) v = scores[(size_t)n * pcap + (e - keep * row)];
    else v = (float)num[n];
    packed[(size_t)n * width + e] = v;
}

// the fast grouping's row: M*C*4 keypoint floats | person count | KM status
__global__ void __launch_bounds__(256)
pack_fast_payload_kernel(const float* __restrict__ ans, const int32_t* __restrict__ num,
                         const int32_t* __restrict__ status, int kp, float* __restrict__ packed) {
    const int n = blockIdx.y;
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= kp + 2) return;
    float v;
    if (e < kp) v = ans[(size_t)n * kp + e];
    else if (e == kp) v = (float)num[n];
    else v = (float)status[n];
    packed[(size_t)n * (kp + 2) + e] = v;
}

__device__ __forceinline__ void atomic_max_f32(float* addr, float v) {
    // IEEE ordering through the integer views: non-negative floats order like signed ints, negative ones inversely
    // like unsigned ints (no NaNs here)
    if (v >= 0.f) atomicMax(reinterpret_cast<int*>(addr), __float_as_int(v));
    else atomicMin(reinterpret_cast<unsigned int*>(addr), __float_as_uint(v));
}

__global__ void __launch_bounds__(256)
plant_crowd_kernel(float* __restrict__ det, const long long* __restrict__ didx, const float* __restrict__ dval,
                   long long nd, float* __restrict__ tag, const long long* __restrict__ tidx,
                   const float* __restrict__ tval, long long nt) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < nd) atomic_max_f32(det + didx[i], dval[i]);
    if (i < nt) tag[tidx[i]] = tval[i];
}

}  // namespace lp

using namespace lp;

extern "C" int lp_pack_payload_f32(const float* ans, const int32_t* num_people, const float* scores, int N, int pcap,
                                   int row, int keep, float* packed, lp_stream_t stream) {
    LP_CHECK_ARG(ans && num_people && scores && packed, "lp_pack_payload_f32: null pointer");
    LP_CHECK_ARG(N > 0 && N <= 65535 && pcap > 0 && row > 0 && keep > 0 && keep <= pcap,
                 "lp_pack_payload_f32: bad shape N=%d pcap=%d row=%d keep=%d (1 <= keep <= pcap)", N, pcap, row, keep);
    const long long width = (long long)keep * row + keep + 1;
    LP_CHECK_ARG(width < (1ll << 30), "lp_pack_payload_f32: payload row too large");
    dim3 grid((unsigned)((width + 255) / 256), N);
    pack_payload_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(ans, num_people, scores, pcap, row, keep, packed);
    LP_LAUNCH_CHECK("pack_payload_kernel");
    return LP_OK;
}

extern "C" int lp_pack_fast_payload_f32(const float* ans, const int32_t* num_person, const int32_t* status, int N, int M,
                                        int C, float* packed, lp_stream_t stream) {
    LP_CHECK_ARG(ans && num_person && status && packed, "lp_pack_fast_payload_f32: null pointer");
    LP_CHECK_ARG(N > 0 && N <= 65535 && M > 0 && C > 0 && (long long)M * C * 4 + 2 < (1ll << 30),
                 "lp_pack_fast_payload_f32: bad shape N=%d M=%d C=%d", N, M, C);
    const int kp = M * C * 4;
    dim3 grid((unsigned)((kp + 2 + 255) / 256), N);
    pack_fast_payload_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(ans, num_person, status, kp, packed);
    LP_LAUNCH_CHECK("pack_fast_payload_kernel");
    return LP_OK;
}

extern "C" int lp_plant_crowd_f32(float* det, const int64_t* det_index, const float* det_value, int64_t n_det, float* tag,
                                  const int64_t* tag_index, const float* tag_value, int64_t n_tag, lp_stream_t stream) {
    LP_CHECK_ARG(det && tag, "lp_plant_crowd_f32: null pointer");
    LP_CHECK_ARG(n_det >= 0 && n_tag >= 0 && (n_det == 0 || (det_index && det_value)) &&
                     (n_tag == 0 || (tag_index && tag_value)),
                 "lp_plant_crowd_f32: bad index lists");
    const long long m = n_det > n_tag ? n_det : n_tag;
    if (m == 0) return LP_OK;
    LP_CHECK_ARG(m < (1ll << 38), "lp_plant_crowd_f32: list too long");
    plant_crowd_kernel<<<(unsigned)((m + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
        det, reinterpret_cast<const long long*>(det_index), det_value, n_det, tag,
        reinterpret_cast<const long long*>(tag_index), tag_value, n_tag);
    LP_LAUNCH_CHECK("plant_crowd_kernel");
    return LP_OK;
}
