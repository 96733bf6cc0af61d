// Kernels around a training pass over the samples an occupancy grid keeps (ops.mlp_forward_grid): the compaction writes
// K, the kept count, to device memory, and every kernel here reads it there, so that a pass makes no host round trip and
// can be captured into a CUDA graph.  Kept sample k < K of a batch is sample idx[k] = r * S + j of the dense [R, S]
// layout; the idx are increasing, so the kept samples of one ray are consecutive.
//   scatter: the compacted rows into their dense places;
//   gather:  the dense rows at the kept samples (upstream gradients, density noise);
//   ray sum: per ray, the sum of its kept rows (the rays' origin and direction gradients), sequential in k: no atomics,
//            the same bits on every run.
#include "common.cuh"

namespace sparf {
namespace {

constexpr int kThreads = 256;

// dst[idx[k] * width + c] = src[k * width + c] for k < *K.  SPAN: for k in [*begin, *K), at most C of them
template <bool SPAN = false>
__global__ void __launch_bounds__(kThreads) scatter_kernel(long long C, const int64_t* __restrict__ K,
                                                           const int64_t* __restrict__ idx, int width,
                                                           const float* __restrict__ src, float* __restrict__ dst,
                                                           const int64_t* __restrict__ begin) {
  const long long i = (long long)blockIdx.x * kThreads + threadIdx.x, j = i / width, k = SPAN ? *begin + j : j;
  if (j >= C || k >= *K) return;
  dst[idx[k] * width + i % width] = src[SPAN ? k * width + i % width : i];
}

// dst[k * width + c] = src[idx[k] * width + c] for k < *K.  SPAN: for k in [*begin, *K), at most C of them
template <bool SPAN = false>
__global__ void __launch_bounds__(kThreads) gather_kernel(long long C, const int64_t* __restrict__ K,
                                                          const int64_t* __restrict__ idx, int width,
                                                          const float* __restrict__ src, float* __restrict__ dst,
                                                          const int64_t* __restrict__ begin) {
  const long long i = (long long)blockIdx.x * kThreads + threadIdx.x, j = i / width, k = SPAN ? *begin + j : j;
  if (j >= C || k >= *K) return;
  dst[SPAN ? k * width + i % width : i] = src[idx[k] * width + i % width];
}

// dst[r * width + c] = sum over k < *K with idx[k] / S == r of src[k * width + c], in increasing k; one thread per ray
__global__ void __launch_bounds__(kThreads) ray_sum_kernel(long long R, int S, long long C, const int64_t* __restrict__ K,
                                                           const int64_t* __restrict__ idx, int width,
                                                           const float* __restrict__ src, float* __restrict__ dst) {
  const long long r = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (r >= R) return;
  const long long k = *K, n = k < C ? k : C, first = r * S, last = first + S;
  long long lo = 0, hi = n;      // the first kept row at or past sample r * S
  while (lo < hi) {
    const long long mid = (lo + hi) / 2;
    if (idx[mid] < first) lo = mid + 1;
    else hi = mid;
  }
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  for (long long k = lo; k < n && idx[k] < last; ++k)
    for (int c = 0; c < width; ++c) acc[c] += src[k * width + c];
  for (int c = 0; c < width; ++c) dst[r * width + c] = acc[c];
}

// ray_sum_kernel over W appended segments: rows [ends[w], ends[w + 1]) hold window w's kept samples, idx increasing within
// a segment but not across segments.  Per ray, a search in each segment, in window order: the ray's rows are then added
// in increasing sample order from 0, as ray_sum_kernel adds them
__global__ void __launch_bounds__(kThreads) ray_sum_segments_kernel(long long R, int S, int W, const int64_t* __restrict__ ends,
                                                                    const int64_t* __restrict__ idx, int width,
                                                                    const float* __restrict__ src, float* __restrict__ dst) {
  const long long r = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (r >= R) return;
  const long long first = r * S, last = first + S;
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  for (int w = 0; w < W; ++w) {
    long long lo = ends[w], hi = ends[w + 1];
    const long long end = hi;
    while (lo < hi) {           // the segment's first row at or past sample r * S
      const long long mid = (lo + hi) / 2;
      if (idx[mid] < first) lo = mid + 1;
      else hi = mid;
    }
    for (long long k = lo; k < end && idx[k] < last; ++k)
      for (int c = 0; c < width; ++c) acc[c] += src[k * width + c];
  }
  for (int c = 0; c < width; ++c) dst[r * width + c] = acc[c];
}

}  // namespace
}  // namespace sparf

using namespace sparf;

extern "C" int sparf_compact_scatter(int64_t C, const int64_t* K, const int64_t* sample_idx, int32_t width,
                                     const float* src, float* dst, sparf_stream_t stream) {
  SPARF_REQUIRE(C >= 0 && width >= 1 && width <= 4, "compact_scatter: C=%lld width=%d", (long long)C, width);
  if (C == 0) return SPARF_OK;
  SPARF_REQUIRE(K && sample_idx && src && dst, "compact_scatter: NULL tensor");
  scatter_kernel<<<ceil_div(C * width, kThreads), kThreads, 0, (cudaStream_t)stream>>>(C, K, sample_idx, width, src, dst,
                                                                                      nullptr);
  SPARF_CHECK_LAUNCH("scatter_kernel");
  return SPARF_OK;
}

extern "C" int sparf_compact_gather(int64_t C, const int64_t* K, const int64_t* sample_idx, int32_t width, const float* src,
                                    float* dst, sparf_stream_t stream) {
  SPARF_REQUIRE(C >= 0 && width >= 1 && width <= 4, "compact_gather: C=%lld width=%d", (long long)C, width);
  if (C == 0) return SPARF_OK;
  SPARF_REQUIRE(K && sample_idx && src && dst, "compact_gather: NULL tensor");
  gather_kernel<<<ceil_div(C * width, kThreads), kThreads, 0, (cudaStream_t)stream>>>(C, K, sample_idx, width, src, dst,
                                                                                     nullptr);
  SPARF_CHECK_LAUNCH("gather_kernel");
  return SPARF_OK;
}

extern "C" int sparf_compact_ray_sum(int64_t R, int32_t S, int64_t C, const int64_t* K, const int64_t* sample_idx,
                                     int32_t width, const float* src, float* dst, sparf_stream_t stream) {
  SPARF_REQUIRE(R >= 0 && S >= 1 && C >= 0 && width >= 1 && width <= 4, "compact_ray_sum: R=%lld S=%d C=%lld width=%d",
                (long long)R, S, (long long)C, width);
  if (R == 0) return SPARF_OK;
  SPARF_REQUIRE(K && dst && (C == 0 || (sample_idx && src)), "compact_ray_sum: NULL tensor");
  ray_sum_kernel<<<ceil_div(R, kThreads), kThreads, 0, (cudaStream_t)stream>>>(R, S, C, K, sample_idx, width, src, dst);
  SPARF_CHECK_LAUNCH("ray_sum_kernel");
  return SPARF_OK;
}

// the span movers: rows [ends[w], ends[w + 1]) of the compacted buffers, at most C (a window's capacity) of them
extern "C" int sparf_compact_scatter_span(int64_t C, const int64_t* ends, int32_t w, const int64_t* sample_idx,
                                          int32_t width, const float* src, float* dst, sparf_stream_t stream) {
  SPARF_REQUIRE(C >= 0 && w >= 0 && width >= 1 && width <= 4, "compact_scatter_span: C=%lld w=%d width=%d", (long long)C,
                w, width);
  if (C == 0) return SPARF_OK;
  SPARF_REQUIRE(ends && sample_idx && src && dst, "compact_scatter_span: NULL tensor");
  scatter_kernel<true><<<ceil_div(C * width, kThreads), kThreads, 0, (cudaStream_t)stream>>>(C, ends + w + 1, sample_idx,
                                                                                            width, src, dst, ends + w);
  SPARF_CHECK_LAUNCH("scatter_kernel<span>");
  return SPARF_OK;
}

extern "C" int sparf_compact_gather_span(int64_t C, const int64_t* ends, int32_t w, const int64_t* sample_idx,
                                         int32_t width, const float* src, float* dst, sparf_stream_t stream) {
  SPARF_REQUIRE(C >= 0 && w >= 0 && width >= 1 && width <= 4, "compact_gather_span: C=%lld w=%d width=%d", (long long)C,
                w, width);
  if (C == 0) return SPARF_OK;
  SPARF_REQUIRE(ends && sample_idx && src && dst, "compact_gather_span: NULL tensor");
  gather_kernel<true><<<ceil_div(C * width, kThreads), kThreads, 0, (cudaStream_t)stream>>>(C, ends + w + 1, sample_idx,
                                                                                           width, src, dst, ends + w);
  SPARF_CHECK_LAUNCH("gather_kernel<span>");
  return SPARF_OK;
}

extern "C" int sparf_compact_ray_sum_segments(int64_t R, int32_t S, int32_t W, const int64_t* ends,
                                              const int64_t* sample_idx, int32_t width, const float* src, float* dst,
                                              sparf_stream_t stream) {
  SPARF_REQUIRE(R >= 0 && S >= 1 && W >= 1 && width >= 1 && width <= 4,
                "compact_ray_sum_segments: R=%lld S=%d W=%d width=%d", (long long)R, S, W, width);
  if (R == 0) return SPARF_OK;
  SPARF_REQUIRE(ends && sample_idx && src && dst, "compact_ray_sum_segments: NULL tensor");
  ray_sum_segments_kernel<<<ceil_div(R, kThreads), kThreads, 0, (cudaStream_t)stream>>>(R, S, W, ends, sample_idx, width,
                                                                                       src, dst);
  SPARF_CHECK_LAUNCH("ray_sum_segments_kernel");
  return SPARF_OK;
}
