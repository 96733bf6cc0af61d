// The sample compaction shared by the occupancy grid (occupancy.cu) and early ray termination (termination.cu): the
// occupancy lookup, a block scan, the tile-total scan and the workspace layout of a count / scan / emit over n samples.
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

// the body of a one-CTA (kScanThreads) scan kernel: tile totals -> exclusive 64-bit tile bases (in place); *K = the sum
__device__ __forceinline__ void scan_tiles(long long* __restrict__ tiles, long long ntiles, int64_t* __restrict__ K) {
  long long carry = 0;
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
  const size_t a = align_up((size_t)ntiles * kOcThreads * 4, 256);
  char* b = (char*)ws;
  if (c) *c = Carve{(uint32_t*)b, (long long*)(b + a), ntiles};
  return a + (size_t)ntiles * sizeof(long long);
}

Lookup make_lookup(int64_t R, int32_t S, const float* origins, const float* dirs, const float* t, const uint32_t* bits,
                   int32_t res, float r0, float r1) {
  return Lookup{origins, dirs, t, bits, (long long)R * S, S, res, r0, r1, (float)res};
}

}  // namespace
}  // namespace sparf
