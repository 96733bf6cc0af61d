// Early ray termination for inference renders: the samples of one window [k0, k1) of every ray are evaluated while the
// ray is alive, and a ray dies once the optical depth tau it has accumulated shows it opaque (tau > tau_max).
//   count / scan / emit: the compaction of occupancy.cu (compaction.cuh) over the R * (k1 - k0) window samples; kept =
//          alive[r] (NULL: every ray) and, with a grid, the occupancy lookup: the box grid's (sparf_termination_*) or
//          the contracted grid's (sparf_contracted_*, which with alive = NULL and [0, S) is the plain grid
//          compaction).  The kernels are templated on the lookup.  Output in increasing order of r * S + k;
//   update: one thread per alive ray adds the window's sd_k = sigma_k * (gap_k * len) to tau in sample order, with
//          explicit rounding (include/sparf_b200.h states the op order), and clears alive[r] when tau > tau_max.
//   append: (training, sparf_*_append) count / scan / emit with the scan's bases starting at ends[w] instead of 0, so
//          that window w's samples land after the earlier windows' in one compacted set, and ends[w + 1] written.
// Deterministic (no atomics).  Workspace: that of a compaction over R * (k1 - k0) samples.
#include <cmath>

#include "compaction.cuh"

namespace sparf {
namespace {

constexpr int kUpdateThreads = 256;

// Lk: Lookup (the box grid) or ContractedLookup (the contracted grid)
template <class Lk>
struct Window {
  Lk Q;                   // o, d, t [R,S]; Q.bits NULL = no grid
  const uint8_t* alive;   // [R]; NULL = every ray alive
  long long n;            // R * W
  int W, k0;
  __device__ __forceinline__ long long sample(long long m) const { return m / W * Q.S + k0 + m % W; }
  __device__ __forceinline__ bool kept(long long m) const {
    if (alive && !__ldg(alive + m / W)) return false;
    return !Q.bits || Q.kept(sample(m));
  }
};

template <class Lk>
__global__ void __launch_bounds__(kOcThreads) termination_count_kernel(Window<Lk> Wn, uint32_t* __restrict__ local,
                                                                       long long* __restrict__ tiles) {
  const long long m0 = (long long)blockIdx.x * kOcTile + (long long)threadIdx.x * kOcItems;
  int c = 0;
#pragma unroll
  for (int u = 0; u < kOcItems; ++u)
    if (m0 + u < Wn.n) c += Wn.kept(m0 + u);
  int total;
  block_scan<int, kOcThreads>(c, total);
  local[(long long)blockIdx.x * kOcThreads + threadIdx.x] = (uint32_t)c;
  if (threadIdx.x == 0) tiles[blockIdx.x] = total;
}

// APPEND (training termination, sparf_*_append): the window's rows go after those of the windows before it, from
// K[-1] = ends[w] on, and K = ends[w + 1] = ends[w] + the window's count
template <bool APPEND = false>
__global__ void __launch_bounds__(kScanThreads) termination_scan_kernel(long long* __restrict__ tiles, long long ntiles,
                                                                        int64_t* __restrict__ K) {
  scan_tiles<APPEND>(tiles, ntiles, K, APPEND ? K - 1 : nullptr);
}

template <class Lk>
__global__ void __launch_bounds__(kOcThreads) termination_emit_kernel(Window<Lk> Wn, const uint32_t* __restrict__ local,
                                                                      const long long* __restrict__ tiles,
                                                                      int64_t* __restrict__ sample_idx,
                                                                      float* __restrict__ origins_k,
                                                                      float* __restrict__ dirs_k,
                                                                      float* __restrict__ t_k) {
  const long long m0 = (long long)blockIdx.x * kOcTile + (long long)threadIdx.x * kOcItems;
  if (m0 >= Wn.n) return;
  long long id = tiles[blockIdx.x] + local[(long long)blockIdx.x * kOcThreads + threadIdx.x];
  for (int u = 0; u < kOcItems; ++u) {
    const long long m = m0 + u;
    if (m >= Wn.n) break;
    if (!Wn.kept(m)) continue;
    const long long r = m / Wn.W, g = Wn.sample(m);
    sample_idx[id] = g;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      origins_k[3 * id + a] = Wn.Q.o[3 * r + a];
      dirs_k[3 * id + a] = Wn.Q.d[3 * r + a];
    }
    t_k[id] = Wn.Q.t[g];
    ++id;
  }
}

// tau[r] += sum over k in [k0, k1) of sigma[r,k] * (gap_k * len), in k order, each op rounded; then alive[r] = 0 when
// tau[r] > tau_max (a NaN tau stays alive)
__global__ void __launch_bounds__(kUpdateThreads) termination_update_kernel(long long R, int S, int k0, int k1,
                                                                            const float* __restrict__ sigma,
                                                                            const float* __restrict__ t,
                                                                            const float* __restrict__ dirs,
                                                                            float tau_max, float* __restrict__ tau,
                                                                            uint8_t* __restrict__ alive) {
  const long long r = (long long)blockIdx.x * kUpdateThreads + threadIdx.x;
  if (r >= R || !alive[r]) return;
  const float dx = dirs[3 * r], dy = dirs[3 * r + 1], dz = dirs[3 * r + 2];
  const float len = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz)));
  const float* sg = sigma + r * S;
  const float* tt = t + r * S;
  float acc = tau[r];
  for (int k = k0; k < k1; ++k) {
    const float gap = k + 1 < S ? __fsub_rn(tt[k + 1], tt[k]) : 1e10f;
    acc = __fadd_rn(acc, __fmul_rn(sg[k], __fmul_rn(gap, len)));
  }
  tau[r] = acc;
  if (acc > tau_max) alive[r] = 0;
}

bool window_ok(int32_t S, int32_t k0, int32_t k1) { return k0 >= 0 && k0 < k1 && k1 <= S; }

}  // namespace
}  // namespace sparf

using namespace sparf;

extern "C" size_t sparf_termination_workspace_bytes(int64_t R, int32_t window) {
  return sizes_ok(R, window) ? carve(R, window, nullptr, nullptr) : 0;
}

// the checks and the workspace carve count and emit share, with the grid's own checks (grid_ok) after the sizes'; fills
// every field of *wn but the lookup.  R == 0 returns before the pointers are checked (nothing to launch)
template <class Lk, class GridCheck>
static int window_setup(const char* name, int64_t R, int32_t S, int32_t k0, int32_t k1, GridCheck grid_ok,
                        const float* origins, const float* dirs, const float* t, const uint8_t* alive, void* workspace,
                        size_t workspace_bytes, Window<Lk>* wn, Carve* c) {
  SPARF_REQUIRE(sizes_ok(R, S), "%s: R %lld, S %d (R >= 0, S >= 1, R * S <= 2^58)", name, (long long)R, (int)S);
  SPARF_REQUIRE(window_ok(S, k0, k1), "%s: window [%d, %d) of S %d (0 <= k0 < k1 <= S)", name, (int)k0, (int)k1, (int)S);
  SPARF_TRY(grid_ok());
  if (R == 0) return SPARF_OK;
  SPARF_REQUIRE(origins && dirs && t && workspace, "%s: NULL pointer", name);
  SPARF_TRY(check_workspace(name, workspace, workspace_bytes, carve(R, k1 - k0, workspace, c)));
  SPARF_REQUIRE(c->ntiles < (1ll << 31), "%s: too many samples", name);
  wn->alive = alive;
  wn->n = (long long)R * (k1 - k0);
  wn->W = k1 - k0;
  wn->k0 = k0;
  return SPARF_OK;
}

// count: K = 0 for R == 0, else the count and scan kernels.  APPEND: K = ends + w + 1, and the count starts at K[-1]
template <bool APPEND = false, class Lk>
static int launch_count(int64_t R, const Window<Lk>& wn, const Carve& c, int64_t* K, cudaStream_t s) {
  if (R == 0) {
    if (APPEND) SPARF_CHECK_CUDA(cudaMemcpyAsync(K, K - 1, sizeof(int64_t), cudaMemcpyDeviceToDevice, s));
    else SPARF_CHECK_CUDA(cudaMemsetAsync(K, 0, sizeof(int64_t), s));
    return SPARF_OK;
  }
  termination_count_kernel<<<(unsigned)c.ntiles, kOcThreads, 0, s>>>(wn, c.local, c.tiles);
  SPARF_CHECK_LAUNCH("termination_count_kernel");
  termination_scan_kernel<APPEND><<<1, kScanThreads, 0, s>>>(c.tiles, c.ntiles, K);
  SPARF_CHECK_LAUNCH("termination_scan_kernel");
  return SPARF_OK;
}

template <class Lk>
static int launch_emit(int64_t R, const Window<Lk>& wn, const Carve& c, int64_t* sample_idx, float* origins_k,
                       float* dirs_k, float* t_k, cudaStream_t s) {
  if (R == 0) return SPARF_OK;
  termination_emit_kernel<<<(unsigned)c.ntiles, kOcThreads, 0, s>>>(wn, c.local, c.tiles, sample_idx, origins_k, dirs_k,
                                                                   t_k);
  SPARF_CHECK_LAUNCH("termination_emit_kernel");
  return SPARF_OK;
}

// the box grid's window (bits NULL: no grid)
static int termination_setup(const char* name, int64_t R, int32_t S, int32_t k0, int32_t k1, const float* origins,
                             const float* dirs, const float* t, const uint8_t* alive, const uint32_t* bits, int32_t res,
                             float r0, float r1, void* workspace, size_t workspace_bytes, Window<Lookup>* wn, Carve* c) {
  auto grid_ok = [&]() -> int {
    if (bits) {
      SPARF_REQUIRE(res_ok(res), "%s: res %d (1 ... 4096)", name, (int)res);
      SPARF_REQUIRE(r1 > r0, "%s: empty box [%g, %g]", name, (double)r0, (double)r1);
    }
    return SPARF_OK;
  };
  SPARF_TRY(window_setup(name, R, S, k0, k1, grid_ok, origins, dirs, t, alive, workspace, workspace_bytes, wn, c));
  if (R > 0) wn->Q = make_lookup(R, S, origins, dirs, t, bits, bits ? res : 1, r0, r1);
  return SPARF_OK;
}

// the contracted grid's window (bits required; center: host float[3])
static int contracted_setup(const char* name, int64_t R, int32_t S, int32_t k0, int32_t k1, const float* origins,
                            const float* dirs, const float* t, const uint8_t* alive, const uint32_t* bits, int32_t res,
                            const float* center, float radius, void* workspace, size_t workspace_bytes,
                            Window<ContractedLookup>* wn, Carve* c) {
  auto grid_ok = [&]() -> int {
    SPARF_REQUIRE(res_ok(res), "%s: res %d (1 ... 4096)", name, (int)res);
    SPARF_REQUIRE(center, "%s: NULL center", name);
    SPARF_REQUIRE(std::isfinite(center[0]) && std::isfinite(center[1]) && std::isfinite(center[2]),
                  "%s: center (%g, %g, %g) is not finite", name, (double)center[0], (double)center[1],
                  (double)center[2]);
    SPARF_REQUIRE(radius > 0.f && std::isfinite(radius), "%s: radius %g (finite, > 0)", name, (double)radius);
    return SPARF_OK;
  };
  SPARF_TRY(window_setup(name, R, S, k0, k1, grid_ok, origins, dirs, t, alive, workspace, workspace_bytes, wn, c));
  if (R == 0) return SPARF_OK;
  SPARF_REQUIRE(bits, "%s: NULL bits", name);
  wn->Q = make_contracted_lookup(S, origins, dirs, t, bits, res, center, radius);
  return SPARF_OK;
}

extern "C" int sparf_termination_count(int64_t R, int32_t S, int32_t k0, int32_t k1, const float* origins,
                                       const float* dirs, const float* t, const uint8_t* alive, const uint32_t* bits,
                                       int32_t res, float r0, float r1, int64_t* K, void* workspace,
                                       size_t workspace_bytes, sparf_stream_t stream) {
  SPARF_REQUIRE(K, "termination_count: NULL pointer");
  Window<Lookup> wn;
  Carve c;
  SPARF_TRY(termination_setup("termination_count", R, S, k0, k1, origins, dirs, t, alive, bits, res, r0, r1, workspace,
                              workspace_bytes, &wn, &c));
  return launch_count(R, wn, c, K, (cudaStream_t)stream);
}

extern "C" int sparf_termination_emit(int64_t R, int32_t S, int32_t k0, int32_t k1, const float* origins,
                                      const float* dirs, const float* t, const uint8_t* alive, const uint32_t* bits,
                                      int32_t res, float r0, float r1, int64_t* sample_idx, float* origins_k,
                                      float* dirs_k, float* t_k, void* workspace, size_t workspace_bytes,
                                      sparf_stream_t stream) {
  Window<Lookup> wn;
  Carve c;
  SPARF_TRY(termination_setup("termination_emit", R, S, k0, k1, origins, dirs, t, alive, bits, res, r0, r1, workspace,
                              workspace_bytes, &wn, &c));
  return launch_emit(R, wn, c, sample_idx, origins_k, dirs_k, t_k, (cudaStream_t)stream);
}

extern "C" int sparf_contracted_count(int64_t R, int32_t S, int32_t k0, int32_t k1, const float* origins,
                                      const float* dirs, const float* t, const uint8_t* alive, const uint32_t* bits,
                                      int32_t res, const float* center, float radius, int64_t* K, void* workspace,
                                      size_t workspace_bytes, sparf_stream_t stream) {
  SPARF_REQUIRE(K, "contracted_count: NULL pointer");
  Window<ContractedLookup> wn;
  Carve c;
  SPARF_TRY(contracted_setup("contracted_count", R, S, k0, k1, origins, dirs, t, alive, bits, res, center, radius,
                             workspace, workspace_bytes, &wn, &c));
  return launch_count(R, wn, c, K, (cudaStream_t)stream);
}

extern "C" int sparf_contracted_emit(int64_t R, int32_t S, int32_t k0, int32_t k1, const float* origins,
                                     const float* dirs, const float* t, const uint8_t* alive, const uint32_t* bits,
                                     int32_t res, const float* center, float radius, int64_t* sample_idx,
                                     float* origins_k, float* dirs_k, float* t_k, void* workspace,
                                     size_t workspace_bytes, sparf_stream_t stream) {
  Window<ContractedLookup> wn;
  Carve c;
  SPARF_TRY(contracted_setup("contracted_emit", R, S, k0, k1, origins, dirs, t, alive, bits, res, center, radius,
                             workspace, workspace_bytes, &wn, &c));
  return launch_emit(R, wn, c, sample_idx, origins_k, dirs_k, t_k, (cudaStream_t)stream);
}

// the appending compaction of window w: count, scan from ends[w] (writing ends[w + 1]) and emit, on one workspace
template <class Lk>
static int launch_append(int64_t R, const Window<Lk>& wn, const Carve& c, int64_t* ends, int32_t w, int64_t* sample_idx,
                         float* origins_k, float* dirs_k, float* t_k, cudaStream_t s) {
  SPARF_TRY(launch_count<true>(R, wn, c, ends + w + 1, s));
  return launch_emit(R, wn, c, sample_idx, origins_k, dirs_k, t_k, s);
}

extern "C" int sparf_termination_append(int64_t R, int32_t S, int32_t k0, int32_t k1, const float* origins,
                                        const float* dirs, const float* t, const uint8_t* alive, const uint32_t* bits,
                                        int32_t res, float r0, float r1, int64_t* ends, int32_t w, int64_t* sample_idx,
                                        float* origins_k, float* dirs_k, float* t_k, void* workspace,
                                        size_t workspace_bytes, sparf_stream_t stream) {
  SPARF_REQUIRE(ends && w >= 0, "termination_append: NULL ends or w %d < 0", (int)w);
  Window<Lookup> wn;
  Carve c;
  SPARF_TRY(termination_setup("termination_append", R, S, k0, k1, origins, dirs, t, alive, bits, res, r0, r1, workspace,
                              workspace_bytes, &wn, &c));
  return launch_append(R, wn, c, ends, w, sample_idx, origins_k, dirs_k, t_k, (cudaStream_t)stream);
}

extern "C" int sparf_contracted_append(int64_t R, int32_t S, int32_t k0, int32_t k1, const float* origins,
                                       const float* dirs, const float* t, const uint8_t* alive, const uint32_t* bits,
                                       int32_t res, const float* center, float radius, int64_t* ends, int32_t w,
                                       int64_t* sample_idx, float* origins_k, float* dirs_k, float* t_k, void* workspace,
                                       size_t workspace_bytes, sparf_stream_t stream) {
  SPARF_REQUIRE(ends && w >= 0, "contracted_append: NULL ends or w %d < 0", (int)w);
  Window<ContractedLookup> wn;
  Carve c;
  SPARF_TRY(contracted_setup("contracted_append", R, S, k0, k1, origins, dirs, t, alive, bits, res, center, radius,
                             workspace, workspace_bytes, &wn, &c));
  return launch_append(R, wn, c, ends, w, sample_idx, origins_k, dirs_k, t_k, (cudaStream_t)stream);
}

extern "C" int sparf_termination_update(int64_t R, int32_t S, int32_t k0, int32_t k1, const float* sigma,
                                        const float* t, const float* dirs, float tau_max, float* tau, uint8_t* alive,
                                        sparf_stream_t stream) {
  SPARF_REQUIRE(sizes_ok(R, S), "termination_update: R %lld, S %d (R >= 0, S >= 1, R * S <= 2^58)", (long long)R,
                (int)S);
  SPARF_REQUIRE(window_ok(S, k0, k1), "termination_update: window [%d, %d) of S %d (0 <= k0 < k1 <= S)", (int)k0,
                (int)k1, (int)S);
  SPARF_REQUIRE(!(tau_max != tau_max), "termination_update: tau_max is NaN");
  if (R == 0) return SPARF_OK;
  SPARF_REQUIRE(sigma && t && dirs && tau && alive, "termination_update: NULL pointer");
  const long long blocks = (R + kUpdateThreads - 1) / kUpdateThreads;
  SPARF_REQUIRE(blocks < (1ll << 31), "termination_update: too many rays");
  termination_update_kernel<<<(unsigned)blocks, kUpdateThreads, 0, (cudaStream_t)stream>>>(R, S, k0, k1, sigma, t, dirs,
                                                                                          tau_max, tau, alive);
  SPARF_CHECK_LAUNCH("termination_update_kernel");
  return SPARF_OK;
}
