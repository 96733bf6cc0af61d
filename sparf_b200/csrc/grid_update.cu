// Updating an occupancy grid on the device inside a training step (sparf_b200/occupancy.py update_): each cell keeps a
// decaying density, a fixed budget of random cells is re-sampled, and the bits are re-thresholded.  Every size is fixed
// by the budget, so the update can be captured in a CUDA graph.
//   count:  one thread per 4 consecutive bit words: the occupied interior cells of each word (popcount of the bits
//           under the interior mask); a block scan writes each word's tile-local prefix and each 2048-word tile its
//           total;
//   scan:   one CTA turns the tile totals into 64-bit tile bases and writes K, the occupied interior count;
//   sample: one thread per sample: the drawn interior cell (directly for the uniform half, by a binary search over the
//           word prefixes and a select within the word for the occupied half) and its jittered point in fp64;
//   ema:    after the density query, a scatter-max of the samples' sigma into a scratch array (float atomicMax on the
//           int bit pattern, valid for values >= 0), then one thread per 32-cell word: decay, max and threshold, writing
//           whole bit words.  max is exact and order-independent: the result is deterministic.
// Semantics in include/sparf_b200.h ("occupancy grid update").
#include <cfloat>
#include <cmath>

#include "compaction.cuh"

namespace sparf {
namespace {

constexpr int kGuThreads = 256;

struct GridShape {
  int res;
  bool contracted;   // interior = every index in [2, res-3]; otherwise every cell
  long long ncell;

  // bit b of word w is an interior cell
  __device__ __forceinline__ uint32_t interior_mask(long long w) const {
    uint32_t m = 0;
    for (int b = 0; b < 32; ++b) {
      const long long c = w * 32 + b;
      if (c >= ncell) break;
      if (contracted) {
        const int i = (int)(c / ((long long)res * res)), j = (int)(c / res % res), k = (int)(c % res);
        if (i < 2 || i > res - 3 || j < 2 || j > res - 3 || k < 2 || k > res - 3) continue;
      }
      m |= 1u << b;
    }
    return m;
  }
};

GridShape make_shape(int32_t res, bool contracted) {
  return GridShape{res, contracted, (long long)res * res * res};
}

long long interior_count(int32_t res, bool contracted) {
  const long long m = contracted ? res - 4 : res;
  return m * m * m;
}

struct SampleCarve {
  uint32_t* local;    // [words] tile-local exclusive prefix of the occupied interior counts
  long long* tiles;   // [ntiles] tile totals, then exclusive tile bases
  int64_t* K;         // the occupied interior count
  long long words, ntiles;
};

// the sample's part of the workspace; the ema's part is the scratch [res^3] at offset 0 (the two calls share it)
size_t sample_carve(int32_t res, void* ws, SampleCarve* c) {
  const long long words = ((long long)res * res * res + 31) / 32;
  const long long ntiles = (words + kOcTile - 1) / kOcTile;
  WsCarver w(ws);
  const SampleCarve k{w.take<uint32_t>(words), w.take<long long>(ntiles), w.take<int64_t>(1), words, ntiles};
  if (c) *c = k;
  return w.end;
}

size_t ema_bytes(int32_t res) { return (size_t)res * res * res * 4; }

__global__ void __launch_bounds__(kOcThreads) grid_count_kernel(GridShape G, const uint32_t* __restrict__ bits,
                                                                 long long words, uint32_t* __restrict__ local,
                                                                 long long* __restrict__ tiles) {
  const long long w0 = (long long)blockIdx.x * kOcTile + (long long)threadIdx.x * kOcItems;
  int c[kOcItems], s = 0;
#pragma unroll
  for (int u = 0; u < kOcItems; ++u) {
    c[u] = w0 + u < words ? __popc(__ldg(bits + w0 + u) & G.interior_mask(w0 + u)) : 0;
    s += c[u];
  }
  int total;
  block_scan<int, kOcThreads>(s, total);
#pragma unroll
  for (int u = 0; u < kOcItems; ++u) {
    if (w0 + u < words) local[w0 + u] = (uint32_t)s;
    s += c[u];
  }
  if (threadIdx.x == 0) tiles[blockIdx.x] = total;
}

__global__ void __launch_bounds__(kScanThreads) grid_scan_kernel(long long* __restrict__ tiles, long long ntiles,
                                                                 int64_t* __restrict__ K) {
  scan_tiles(tiles, ntiles, K);
}

// min(floor((double)u * n), n - 1), clamped at 0 (n >= 1)
__device__ __forceinline__ long long pick(float u, long long n) {
  const long long j = (long long)floor(__dmul_rn((double)u, (double)n));
  return j < 0 ? 0 : (j > n - 1 ? n - 1 : j);
}

struct SampleArgs {
  GridShape G;
  const uint32_t* bits;
  const uint32_t* local;
  const long long* tiles;
  const int64_t* K;
  long long words, n_interior, n_uniform, n;
  double r0, r1, c[3], radius;   // box [r0, r1]^3, or the contraction (center, radius)
  const float *u_cell, *u_jit;
  int64_t* cells;
  float* points;
};

__global__ void __launch_bounds__(kGuThreads) grid_sample_kernel(SampleArgs A) {
  const long long i = (long long)blockIdx.x * kGuThreads + threadIdx.x;
  if (i >= A.n) return;
  const int res = A.G.res;
  const long long K = *A.K;
  const float u = __ldg(A.u_cell + i);
  long long cell;
  if (i < A.n_uniform || K == 0) {                      // interior cell number j in increasing linear index
    const long long j = pick(u, A.n_interior);
    if (A.G.contracted) {
      const long long m = res - 4;
      cell = ((2 + j / (m * m)) * res + (2 + j / m % m)) * res + (2 + j % m);
    } else {
      cell = j;
    }
  } else {                                               // the j-th occupied interior cell
    const long long j = pick(u, K);
    long long lo = 0, hi = A.words - 1;                  // the last word whose prefix is <= j
    while (lo < hi) {
      const long long mid = (lo + hi + 1) >> 1;
      if (A.tiles[mid / kOcTile] + A.local[mid] <= j) lo = mid;
      else hi = mid - 1;
    }
    const uint32_t m = __ldg(A.bits + lo) & A.G.interior_mask(lo);
    int r = (int)(j - (A.tiles[lo / kOcTile] + A.local[lo])), b = 0;
    for (; b < 31; ++b)                                  // the r-th set bit of m
      if ((m >> b & 1u) && r-- == 0) break;
    cell = lo * 32 + b;
  }
  A.cells[i] = cell;
  const long long ci[3] = {cell / ((long long)res * res), cell / res % res, cell % res};
  double v[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const double x = __dadd_rn((double)ci[a], (double)__ldg(A.u_jit + 3 * i + a));
    v[a] = A.G.contracted ? __dadd_rn(-2.0, __ddiv_rn(__dmul_rn(x, 4.0), (double)res))
                          : __dadd_rn(A.r0, __ddiv_rn(__dmul_rn(x, __dsub_rn(A.r1, A.r0)), (double)res));
  }
  if (A.G.contracted) {                                  // occupancy.contracted_warp: center + radius * y
    const double n = fmax(fmax(fabs(v[0]), fabs(v[1])), fabs(v[2]));
    const double den = n <= 1.0 ? 1.0 : __dmul_rn(n, __dsub_rn(2.0, n));
#pragma unroll
    for (int a = 0; a < 3; ++a) v[a] = __dadd_rn(A.c[a], __dmul_rn(A.radius, __ddiv_rn(v[a], den)));
  }
#pragma unroll
  for (int a = 0; a < 3; ++a) A.points[3 * i + a] = __double2float_rn(v[a]);
}

__global__ void __launch_bounds__(kGuThreads) grid_scatter_max_kernel(long long n, long long ncell,
                                                                      const int64_t* __restrict__ cells,
                                                                      const float* __restrict__ sigma,
                                                                      int* __restrict__ smax) {
  const long long i = (long long)blockIdx.x * kGuThreads + threadIdx.x;
  if (i >= n) return;
  const long long c = __ldg(cells + i);
  if (c < 0 || c >= ncell) return;
  float s = __ldg(sigma + i);
  if (!(s <= FLT_MAX)) s = FLT_MAX;                      // NaN and +inf
  atomicMax(smax + c, __float_as_int(s));               // the int order is the float order for s >= 0
}

__global__ void __launch_bounds__(kGuThreads) grid_ema_kernel(GridShape G, long long words, float decay, float thres,
                                                              const int* __restrict__ smax, float* __restrict__ density,
                                                              uint32_t* __restrict__ bits) {
  const long long w = (long long)blockIdx.x * kGuThreads + threadIdx.x;
  if (w >= words) return;
  const uint32_t interior = G.interior_mask(w);
  uint32_t word = 0;
  for (int b = 0; b < 32; ++b) {
    const long long c = w * 32 + b;
    if (c >= G.ncell) break;
    if (!(interior >> b & 1u)) {                         // the contracted shell: untouched, always occupied
      word |= 1u << b;
      continue;
    }
    const float d = fmaxf(__fmul_rn(decay, density[c]), __int_as_float(__ldg(smax + c)));
    density[c] = d;
    word |= (uint32_t)!(d < thres) << b;
  }
  bits[w] = word;
}

}  // namespace
}  // namespace sparf

using namespace sparf;

extern "C" size_t sparf_occupancy_sample_workspace_bytes(int32_t res) {
  if (!res_ok(res)) return 0;
  const size_t s = sample_carve(res, nullptr, nullptr), e = ema_bytes(res);
  return s > e ? s : e;
}

extern "C" int sparf_occupancy_sample(int32_t res, const uint32_t* bits, float r0, float r1, const float* center,
                                      float radius, int64_t n_uniform, int64_t n_occupied, const float* u_cell,
                                      const float* u_jit, int64_t* cells, float* points, void* workspace,
                                      size_t workspace_bytes, sparf_stream_t stream) {
  const bool contracted = center != nullptr;
  SPARF_REQUIRE(res_ok(res), "occupancy_sample: res %d (1 ... 4096)", (int)res);
  SPARF_REQUIRE(!contracted || res >= 8, "occupancy_sample: a contracted grid needs res >= 8 (res %d)", (int)res);
  SPARF_REQUIRE(n_uniform >= 0 && n_occupied >= 0 && n_uniform <= (1ll << 30) && n_occupied <= (1ll << 30),
                "occupancy_sample: budgets %lld, %lld (0 ... 2^30)", (long long)n_uniform, (long long)n_occupied);
  if (contracted) {
    SPARF_REQUIRE(std::isfinite(center[0]) && std::isfinite(center[1]) && std::isfinite(center[2]) &&
                      std::isfinite(radius) && radius > 0.f,
                  "occupancy_sample: contraction center (%g, %g, %g), radius %g (finite, radius > 0)", (double)center[0],
                  (double)center[1], (double)center[2], (double)radius);
  } else {
    SPARF_REQUIRE(std::isfinite(r0) && std::isfinite(r1) && r1 > r0, "occupancy_sample: box [%g, %g]", (double)r0,
                  (double)r1);
  }
  const long long n = n_uniform + n_occupied;
  if (n == 0) return SPARF_OK;
  SPARF_REQUIRE(bits && u_cell && u_jit && cells && points && workspace, "occupancy_sample: NULL pointer");
  SampleCarve c;
  SPARF_TRY(check_workspace("occupancy_sample", workspace, workspace_bytes, sample_carve(res, workspace, &c)));
  cudaStream_t s = (cudaStream_t)stream;
  const GridShape G = make_shape(res, contracted);
  grid_count_kernel<<<(unsigned)c.ntiles, kOcThreads, 0, s>>>(G, bits, c.words, c.local, c.tiles);
  SPARF_CHECK_LAUNCH("grid_count_kernel");
  grid_scan_kernel<<<1, kScanThreads, 0, s>>>(c.tiles, c.ntiles, c.K);
  SPARF_CHECK_LAUNCH("grid_scan_kernel");
  SampleArgs A{G, bits, c.local, c.tiles, c.K, c.words, interior_count(res, contracted), n_uniform, n,
               r0, r1, {0.0, 0.0, 0.0}, (double)radius, u_cell, u_jit, cells, points};
  if (contracted)
    for (int a = 0; a < 3; ++a) A.c[a] = center[a];
  grid_sample_kernel<<<(unsigned)((n + kGuThreads - 1) / kGuThreads), kGuThreads, 0, s>>>(A);
  SPARF_CHECK_LAUNCH("grid_sample_kernel");
  return SPARF_OK;
}

extern "C" int sparf_occupancy_ema(int32_t res, int32_t contracted, int64_t n, const int64_t* cells, const float* sigma,
                                   float decay, float thres, float* density, uint32_t* bits, void* workspace,
                                   size_t workspace_bytes, sparf_stream_t stream) {
  SPARF_REQUIRE(res_ok(res), "occupancy_ema: res %d (1 ... 4096)", (int)res);
  SPARF_REQUIRE(!contracted || res >= 8, "occupancy_ema: a contracted grid needs res >= 8 (res %d)", (int)res);
  SPARF_REQUIRE(n >= 0 && n <= (1ll << 31), "occupancy_ema: n %lld (0 ... 2^31)", (long long)n);
  SPARF_REQUIRE(decay > 0.f && decay <= 1.f, "occupancy_ema: decay %g (0 < decay <= 1)", (double)decay);
  SPARF_REQUIRE(density && bits && workspace && (n == 0 || (cells && sigma)), "occupancy_ema: NULL pointer");
  SPARF_TRY(check_workspace("occupancy_ema", workspace, workspace_bytes, ema_bytes(res)));
  cudaStream_t s = (cudaStream_t)stream;
  const GridShape G = make_shape(res, contracted != 0);
  int* smax = (int*)workspace;
  SPARF_CHECK_CUDA(cudaMemsetAsync(smax, 0, ema_bytes(res), s));   // 0.0f: max(decayed >= 0, 0) = decayed
  if (n > 0) {
    grid_scatter_max_kernel<<<(unsigned)((n + kGuThreads - 1) / kGuThreads), kGuThreads, 0, s>>>(n, G.ncell, cells,
                                                                                              sigma, smax);
    SPARF_CHECK_LAUNCH("grid_scatter_max_kernel");
  }
  const long long words = (G.ncell + 31) / 32;
  grid_ema_kernel<<<(unsigned)((words + kGuThreads - 1) / kGuThreads), kGuThreads, 0, s>>>(G, words, decay, thres, smax,
                                                                                           density, bits);
  SPARF_CHECK_LAUNCH("grid_ema_kernel");
  return SPARF_OK;
}
