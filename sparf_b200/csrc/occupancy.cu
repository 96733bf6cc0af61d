// Occupancy grid for skipping empty space in inference renders: a bitfield of res^3 cells built from the density
// lattice sigma [res+1]^3 (mesh.density_grid), and a per-sample lookup that compacts the samples to evaluate.
//   build: one thread per 32 cells (one bitfield word); a cell is occupied if a lattice point within one cell of it
//          (indices [c-1, c+2] per axis, clipped) has !(sigma < thres): sigma >= thres or NaN;
//   count: per sample x = o + t d (the MLP encoder's op order) and its cell; kept = outside the box or in an occupied
//          cell.  4 consecutive samples per thread; a block scan writes each thread's tile-local offset and each
//          2048-sample tile writes its total;
//   scan:  one CTA turns the tile totals into 64-bit tile bases and writes K;
//   emit:  repeats the lookup and writes each kept sample's index and the MLP's inputs (o, d, t) at its offset.
// Deterministic (no atomics), ordered by sample index r * S + k.  Workspace: 4 B per 4 samples + 8 B per 2048 samples.
// The lookup, the scans and the workspace layout are in compaction.cuh (termination.cu shares them).
#include "compaction.cuh"

namespace sparf {
namespace {

constexpr int kBuildThreads = 256;

__global__ void __launch_bounds__(kBuildThreads) occupancy_build_kernel(const float* __restrict__ sigma, int res,
                                                                         float thres, uint32_t* __restrict__ bits) {
  const long long n = res + 1, ncell = (long long)res * res * res;
  const long long w = (long long)blockIdx.x * kBuildThreads + threadIdx.x;
  if (w * 32 >= ncell) return;
  uint32_t word = 0;
  for (int b = 0; b < 32; ++b) {
    const long long c = w * 32 + b;
    if (c >= ncell) break;
    const int i = (int)(c / ((long long)res * res)), j = (int)(c / res % res), k = (int)(c % res);
    bool occ = false;
    for (int a = max(i - 1, 0); a <= min(i + 2, res) && !occ; ++a)
      for (int bb = max(j - 1, 0); bb <= min(j + 2, res) && !occ; ++bb) {
        const float* row = sigma + ((long long)a * n + bb) * n;
        for (int cc = max(k - 1, 0); cc <= min(k + 2, res); ++cc) occ |= !(__ldg(row + cc) < thres);   // NaN: occupied
      }
    word |= (uint32_t)occ << b;
  }
  bits[w] = word;
}

__global__ void __launch_bounds__(kOcThreads) occupancy_count_kernel(Lookup Q, uint32_t* __restrict__ local,
                                                                     long long* __restrict__ tiles) {
  const long long m0 = (long long)blockIdx.x * kOcTile + (long long)threadIdx.x * kOcItems;
  int c = 0;
#pragma unroll
  for (int u = 0; u < kOcItems; ++u)
    if (m0 + u < Q.n) c += Q.kept(m0 + u);
  int total;
  block_scan<int, kOcThreads>(c, total);
  local[(long long)blockIdx.x * kOcThreads + threadIdx.x] = (uint32_t)c;
  if (threadIdx.x == 0) tiles[blockIdx.x] = total;
}

// tile totals -> exclusive 64-bit tile bases (in place); *K = the sum
__global__ void __launch_bounds__(kScanThreads) occupancy_scan_kernel(long long* __restrict__ tiles, long long ntiles,
                                                                      int64_t* __restrict__ K) {
  scan_tiles(tiles, ntiles, K);
}

__global__ void __launch_bounds__(kOcThreads) occupancy_emit_kernel(Lookup Q, const uint32_t* __restrict__ local,
                                                                    const long long* __restrict__ tiles,
                                                                    int64_t* __restrict__ sample_idx,
                                                                    float* __restrict__ origins_k,
                                                                    float* __restrict__ dirs_k, float* __restrict__ t_k) {
  const long long m0 = (long long)blockIdx.x * kOcTile + (long long)threadIdx.x * kOcItems;
  if (m0 >= Q.n) return;
  long long id = tiles[blockIdx.x] + local[(long long)blockIdx.x * kOcThreads + threadIdx.x];
  for (int u = 0; u < kOcItems; ++u) {
    const long long m = m0 + u;
    if (m >= Q.n) break;
    if (!Q.kept(m)) continue;
    const long long r = m / Q.S;
    sample_idx[id] = m;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      origins_k[3 * id + a] = Q.o[3 * r + a];
      dirs_k[3 * id + a] = Q.d[3 * r + a];
    }
    t_k[id] = Q.t[m];
    ++id;
  }
}

}  // namespace
}  // namespace sparf

using namespace sparf;

extern "C" int sparf_occupancy_build(const float* sigma, int32_t res, float thres, uint32_t* bits, sparf_stream_t stream) {
  SPARF_REQUIRE(res_ok(res), "occupancy_build: res %d (1 ... 4096)", (int)res);
  SPARF_REQUIRE(sigma && bits, "occupancy_build: NULL pointer");
  const long long words = ((long long)res * res * res + 31) / 32;
  occupancy_build_kernel<<<ceil_div(words, kBuildThreads), kBuildThreads, 0, (cudaStream_t)stream>>>(sigma, res, thres,
                                                                                                     bits);
  SPARF_CHECK_LAUNCH("occupancy_build_kernel");
  return SPARF_OK;
}

extern "C" size_t sparf_occupancy_workspace_bytes(int64_t R, int32_t S) {
  return sizes_ok(R, S) ? carve(R, S, nullptr, nullptr) : 0;
}

extern "C" int sparf_occupancy_count(int64_t R, int32_t S, const float* origins, const float* dirs, const float* t,
                                     const uint32_t* bits, int32_t res, float r0, float r1, int64_t* K, void* workspace,
                                     size_t workspace_bytes, sparf_stream_t stream) {
  SPARF_REQUIRE(sizes_ok(R, S), "occupancy_count: R %lld, S %d (R >= 0, S >= 1, R * S <= 2^58)", (long long)R, (int)S);
  SPARF_REQUIRE(res_ok(res), "occupancy_count: res %d (1 ... 4096)", (int)res);
  SPARF_REQUIRE(r1 > r0, "occupancy_count: empty box [%g, %g]", (double)r0, (double)r1);
  SPARF_REQUIRE(K && (R == 0 || (origins && dirs && t && bits && workspace)), "occupancy_count: NULL pointer");
  cudaStream_t s = (cudaStream_t)stream;
  if (R == 0) {
    SPARF_CHECK_CUDA(cudaMemsetAsync(K, 0, sizeof(int64_t), s));
    return SPARF_OK;
  }
  Carve c;
  SPARF_TRY(check_workspace("occupancy_count", workspace, workspace_bytes, carve(R, S, workspace, &c)));
  SPARF_REQUIRE(c.ntiles < (1ll << 31), "occupancy_count: too many samples");
  const Lookup Q = make_lookup(R, S, origins, dirs, t, bits, res, r0, r1);
  occupancy_count_kernel<<<(unsigned)c.ntiles, kOcThreads, 0, s>>>(Q, c.local, c.tiles);
  SPARF_CHECK_LAUNCH("occupancy_count_kernel");
  occupancy_scan_kernel<<<1, kScanThreads, 0, s>>>(c.tiles, c.ntiles, K);
  SPARF_CHECK_LAUNCH("occupancy_scan_kernel");
  return SPARF_OK;
}

extern "C" int sparf_occupancy_emit(int64_t R, int32_t S, const float* origins, const float* dirs, const float* t,
                                    const uint32_t* bits, int32_t res, float r0, float r1, int64_t* sample_idx,
                                    float* origins_k, float* dirs_k, float* t_k, void* workspace, size_t workspace_bytes,
                                    sparf_stream_t stream) {
  SPARF_REQUIRE(sizes_ok(R, S), "occupancy_emit: R %lld, S %d (R >= 0, S >= 1, R * S <= 2^58)", (long long)R, (int)S);
  SPARF_REQUIRE(res_ok(res), "occupancy_emit: res %d (1 ... 4096)", (int)res);
  SPARF_REQUIRE(r1 > r0, "occupancy_emit: empty box [%g, %g]", (double)r0, (double)r1);
  if (R == 0) return SPARF_OK;
  SPARF_REQUIRE(origins && dirs && t && bits && workspace, "occupancy_emit: NULL pointer");
  Carve c;
  SPARF_TRY(check_workspace("occupancy_emit", workspace, workspace_bytes, carve(R, S, workspace, &c)));
  SPARF_REQUIRE(c.ntiles < (1ll << 31), "occupancy_emit: too many samples");
  occupancy_emit_kernel<<<(unsigned)c.ntiles, kOcThreads, 0, (cudaStream_t)stream>>>(
      make_lookup(R, S, origins, dirs, t, bits, res, r0, r1), c.local, c.tiles, sample_idx, origins_k, dirs_k, t_k);
  SPARF_CHECK_LAUNCH("occupancy_emit_kernel");
  return SPARF_OK;
}
