// The sample compaction shared by the occupancy grid (occupancy.cu) and early ray termination (termination.cu): the
// occupancy lookups (box and contracted), a block scan, the tile-total scan and the workspace layout of a count / scan /
// emit over n samples.
//   count: 4 consecutive samples per thread; a block scan writes each thread's tile-local offset and each 2048-sample
//          tile writes its total;
//   scan:  one CTA turns the tile totals into 64-bit tile bases and writes K;
//   emit:  repeats the test and writes each kept sample at its offset.
// Workspace: 4 B per 4 samples + 8 B per 2048 samples.
#pragma once
#include "common.cuh"

namespace sparf {
namespace {

constexpr int kOcThreads = 512;
constexpr int kOcItems = 4;                      // consecutive samples per thread
constexpr int kOcTile = kOcThreads * kOcItems;   // samples per tile (one CTA)
constexpr int kScanThreads = 1024;

struct Lookup {
  const float *o, *d, *t;
  const uint32_t* bits;
  long long n;        // R * S
  int S, res;
  float r0, r1, fres;
  // sample m is evaluated: outside [r0, r1]^3 (or NaN) or in an occupied cell
  __device__ __forceinline__ bool kept(long long m) const {
    const long long r = m / S;
    const float tm = __ldg(t + m);
    long long cell = 0;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      const float x = add_rn(__ldg(o + 3 * r + a), mul_rn(__ldg(d + 3 * r + a), tm));   // encode_xyz_kernel's x
      const float u = __fmul_rn(__fdiv_rn(__fsub_rn(x, r0), __fsub_rn(r1, r0)), fres);
      if (!(u >= 0.f && u < fres)) return true;                                           // outside or NaN
      cell = cell * res + (int)u;
    }
    return __ldg(bits + (cell >> 5)) >> (cell & 31) & 1u;
  }
};

// The contracted grid's lookup (include/sparf_b200.h): y = (x - center) / radius, v = y where ||y||_inf <= 1 and
// y / m * (2 - 1 / m) with m = ||y||_inf beyond, so every finite x lands in the cube [-2, 2]^3 of res^3 cells.
struct ContractedLookup {
  const float *o, *d, *t;
  const uint32_t* bits;
  int S, res;
  float c0, c1, c2, radius, fres;
  // sample m is evaluated: a u outside [0, res) (NaN, infinite or |v| rounded to 2) or an occupied cell
  __device__ __forceinline__ bool kept(long long m) const {
    const long long r = m / S;
    const float tm = __ldg(t + m);
    const float c[3] = {c0, c1, c2};
    float v[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      const float x = add_rn(__ldg(o + 3 * r + a), mul_rn(__ldg(d + 3 * r + a), tm));   // encode_xyz_kernel's x
      v[a] = __fdiv_rn(__fsub_rn(x, c[a]), radius);
    }
    // fmaxf drops a NaN |y_a|, but that axis's u is NaN on either branch, so the sample is kept all the same
    const float n = fmaxf(fmaxf(fabsf(v[0]), fabsf(v[1])), fabsf(v[2]));
    if (n > 1.f) {
      const float q = __fdiv_rn(1.f, n), s = __fsub_rn(2.f, q);
#pragma unroll
      for (int a = 0; a < 3; ++a) v[a] = __fmul_rn(__fmul_rn(v[a], q), s);
    }
    long long cell = 0;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      const float u = __fmul_rn(__fmul_rn(__fadd_rn(v[a], 2.f), 0.25f), fres);
      if (!(u >= 0.f && u < fres)) return true;                                           // NaN, inf or u = res
      cell = cell * res + (int)u;
    }
    return __ldg(bits + (cell >> 5)) >> (cell & 31) & 1u;
  }
};

// exclusive block scan of one value per thread; total = the block's sum
template <typename T, int THREADS>
__device__ __forceinline__ void block_scan(T& x, T& total) {
  constexpr int NW = THREADS / 32;
  __shared__ T sx[NW];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  T ix = x;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const T u = __shfl_up_sync(0xffffffffu, ix, d);
    if (lane >= d) ix += u;
  }
  if (lane == 31) sx[w] = ix;
  __syncthreads();
  if (w == 0) {
    T v = lane < NW ? sx[lane] : T(0);
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const T u = __shfl_up_sync(0xffffffffu, v, d);
      if (lane >= d) v += u;
    }
    if (lane < NW) sx[lane] = v;
  }
  __syncthreads();
  total = sx[NW - 1];
  x = (w ? sx[w - 1] : T(0)) + ix - x;
  __syncthreads();  // the next call reuses sx
}

// the body of a one-CTA (kScanThreads) scan kernel: tile totals -> exclusive 64-bit tile bases (in place); *K = the sum.
// APPEND: the bases start at *start instead of 0 (the emit then writes after the rows already there), and *K = *start
// + the sum
template <bool APPEND = false>
__device__ __forceinline__ void scan_tiles(long long* __restrict__ tiles, long long ntiles, int64_t* __restrict__ K,
                                           const int64_t* __restrict__ start = nullptr) {
  long long carry = APPEND ? *start : 0;
  for (long long base = 0; base < ntiles; base += (long long)kScanThreads * kOcItems) {
    const long long t0 = base + (long long)threadIdx.x * kOcItems;
    long long e[kOcItems], s = 0;
#pragma unroll
    for (int u = 0; u < kOcItems; ++u) {
      e[u] = t0 + u < ntiles ? tiles[t0 + u] : 0;
      s += e[u];
    }
    long long total;
    block_scan<long long, kScanThreads>(s, total);
    s += carry;
#pragma unroll
    for (int u = 0; u < kOcItems; ++u) {
      if (t0 + u < ntiles) tiles[t0 + u] = s;
      s += e[u];
    }
    carry += total;
  }
  if (threadIdx.x == 0) *K = carry;
}

bool sizes_ok(int64_t R, int32_t S) {
  // at most 2^58 samples: every byte count stays inside 64 bits
  long long n = 0;
  return R >= 0 && S >= 1 && !__builtin_mul_overflow((long long)R, (long long)S, &n) && n <= (1ll << 58);
}

bool res_ok(int32_t res) { return res >= 1 && res <= 4096; }

struct Carve {
  uint32_t* local;
  long long* tiles;
  long long ntiles;
};

// the workspace of a compaction over n = R * S samples
size_t carve(int64_t R, int32_t S, void* ws, Carve* c) {
  const long long ntiles = ((long long)R * S + kOcTile - 1) / kOcTile;
  WsCarver w(ws);
  const Carve k{w.take<uint32_t>(ntiles * kOcThreads), w.take<long long>(ntiles), ntiles};
  if (c) *c = k;
  return w.end;
}

Lookup make_lookup(int64_t R, int32_t S, const float* origins, const float* dirs, const float* t, const uint32_t* bits,
                   int32_t res, float r0, float r1) {
  return Lookup{origins, dirs, t, bits, (long long)R * S, S, res, r0, r1, (float)res};
}

ContractedLookup make_contracted_lookup(int32_t S, const float* origins, const float* dirs, const float* t,
                                        const uint32_t* bits, int32_t res, const float* center, float radius) {
  return ContractedLookup{origins, dirs, t, bits, S, res, center[0], center[1], center[2], radius, (float)res};
}

}  // namespace
}  // namespace sparf
