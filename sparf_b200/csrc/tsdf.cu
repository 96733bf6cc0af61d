// TSDF fusion: depth and colour maps integrated into a truncated signed distance volume on BARF's lattice
// (sparf_b200/tsdf.py).  One thread per lattice point loops over the views in order, keeps the point's state in
// registers and writes it once: no atomics, so the result is deterministic and the call capturable.  The projection
// and the update are written with rounded intrinsics (no FMA contraction) so that tests/tsdf_oracle.py can restate
// them bit for bit; the rules are in include/sparf_b200.h.
#include <cmath>

#include "common.cuh"

namespace sparf {
namespace {

constexpr int kTsdfThreads = 256;
constexpr int kViewFloats = 12 + 6;      // pose_w2c [3,4] and the first two rows of K
constexpr int kViewsPerStage = 128;      // views staged in shared memory at a time

__global__ void __launch_bounds__(kTsdfThreads)
    tsdf_integrate_kernel(const float* __restrict__ axis, int n, float trunc, int B, int H, int W,
                          const float* __restrict__ pose, const float* __restrict__ intr,
                          const float* __restrict__ depth, const float* __restrict__ rgb,
                          const uint8_t* __restrict__ valid, float* __restrict__ tsdf, float* __restrict__ weight,
                          float* __restrict__ color) {
  __shared__ float cam[kViewsPerStage * kViewFloats];
  const long long nn = (long long)n * n, npts = nn * n;
  const long long p = (long long)blockIdx.x * kTsdfThreads + threadIdx.x;
  const bool live = p < npts;
  float px = 0.f, py = 0.f, pz = 0.f, T = 1.f, Wt = 0.f, c0 = 0.f, c1 = 0.f, c2 = 0.f;
  if (live) {
    const long long i = p / nn, r = p - i * nn, j = r / n, k = r - j * n;
    px = __ldg(axis + i);
    py = __ldg(axis + j);
    pz = __ldg(axis + k);
    T = tsdf[p];
    Wt = weight[p];
    if (rgb) {
      c0 = color[3 * p];
      c1 = color[3 * p + 1];
      c2 = color[3 * p + 2];
    }
  }
  const float fW = (float)W, fH = (float)H;
  for (int b0 = 0; b0 < B; b0 += kViewsPerStage) {
    const int nb = min(kViewsPerStage, B - b0);
    __syncthreads();  // the previous stage is read by every thread
    for (int q = threadIdx.x; q < nb * kViewFloats; q += kTsdfThreads) {
      const int v = q / kViewFloats, e = q - v * kViewFloats;
      cam[q] = e < 12 ? pose[(long long)(b0 + v) * 12 + e] : intr[(long long)(b0 + v) * 9 + (e - 12)];
    }
    __syncthreads();
    if (!live) continue;
    for (int v = 0; v < nb; ++v) {
      const float* P = cam + v * kViewFloats;
      const float x = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(P[0], px), __fmul_rn(P[1], py)), __fmul_rn(P[2], pz)), P[3]);
      const float y = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(P[4], px), __fmul_rn(P[5], py)), __fmul_rn(P[6], pz)), P[7]);
      const float z = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(P[8], px), __fmul_rn(P[9], py)), __fmul_rn(P[10], pz)), P[11]);
      if (!(z > 0.f)) continue;
      const float* K = P + 12;
      const float u = __fdiv_rn(__fadd_rn(__fadd_rn(__fmul_rn(K[0], x), __fmul_rn(K[1], y)), __fmul_rn(K[2], z)), z);
      const float w = __fdiv_rn(__fadd_rn(__fadd_rn(__fmul_rn(K[3], x), __fmul_rn(K[4], y)), __fmul_rn(K[5], z)), z);
      if (!(u >= 0.f && u < fW && w >= 0.f && w < fH)) continue;   // also rejects NaN
      const long long pix = ((long long)(b0 + v) * H + (int)w) * W + (int)u;   // u, w >= 0: truncation is floor
      if (valid && !__ldg(valid + pix)) continue;
      const float d = __ldg(depth + pix);
      if (!(isfinite(d) && d > 0.f)) continue;
      const float s = __fsub_rn(d, z);
      if (s < -trunc) continue;
      const float f = fminf(1.f, __fdiv_rn(s, trunc));
      // (W tsdf + f) / (W + 1) written as tsdf + (f - tsdf) / (W + 1): a constant observation leaves the value exact
      Wt = __fadd_rn(Wt, 1.f);
      T = __fadd_rn(T, __fdiv_rn(__fsub_rn(f, T), Wt));
      if (rgb) {
        const float* c = rgb + 3 * pix;
        c0 = __fadd_rn(c0, __fdiv_rn(__fsub_rn(__ldg(c), c0), Wt));
        c1 = __fadd_rn(c1, __fdiv_rn(__fsub_rn(__ldg(c + 1), c1), Wt));
        c2 = __fadd_rn(c2, __fdiv_rn(__fsub_rn(__ldg(c + 2), c2), Wt));
      }
    }
  }
  if (live) {
    tsdf[p] = T;
    weight[p] = Wt;
    if (rgb) {
      color[3 * p] = c0;
      color[3 * p + 1] = c1;
      color[3 * p + 2] = c2;
    }
  }
}

}  // namespace
}  // namespace sparf

using namespace sparf;

extern "C" int sparf_tsdf_integrate(const float* axis, int32_t n, float trunc, int32_t B, int32_t H, int32_t W,
                                    const float* pose_w2c, const float* intr, const float* depth, const float* rgb,
                                    const uint8_t* valid, float* tsdf, float* weight, float* color,
                                    sparf_stream_t stream) {
  long long npts = 0, npix = 0;
  SPARF_REQUIRE(n >= 2 && !__builtin_mul_overflow((long long)n, (long long)n, &npts) &&
                    !__builtin_mul_overflow(npts, (long long)n, &npts) && npts <= (1ll << 38),
                "tsdf_integrate: n = %d (>= 2, at most 2^38 lattice points)", (int)n);
  SPARF_REQUIRE(trunc > 0.f && std::isfinite(trunc), "tsdf_integrate: trunc %g (finite, > 0)", (double)trunc);
  SPARF_REQUIRE(B >= 1 && H >= 1 && W >= 1 && H <= (1 << 24) && W <= (1 << 24) &&
                    !__builtin_mul_overflow((long long)B, (long long)H, &npix) &&
                    !__builtin_mul_overflow(npix, (long long)W, &npix) && npix <= (1ll << 60),
                "tsdf_integrate: views %d x %d x %d (each >= 1, H and W at most 2^24)", (int)B, (int)H, (int)W);
  SPARF_REQUIRE(axis && pose_w2c && intr && depth && tsdf && weight && (color || !rgb), "tsdf_integrate: NULL pointer");
  const long long blocks = (npts + kTsdfThreads - 1) / kTsdfThreads;
  tsdf_integrate_kernel<<<(unsigned)blocks, kTsdfThreads, 0, (cudaStream_t)stream>>>(
      axis, n, trunc, B, H, W, pose_w2c, intr, depth, rgb, valid, tsdf, weight, color);
  SPARF_CHECK_LAUNCH("tsdf_integrate_kernel");
  return SPARF_OK;
}
