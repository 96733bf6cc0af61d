// Marching cubes over a dense fp32 volume: a vertex-deduplicated triangle mesh in index space, deterministic (no
// atomics decide any order).  Two passes over the lattice with one hand-written exclusive scan between them:
//   count: per lattice point, its owned crossing edges (a 3-bit mask) and, at a cell origin, the cell's triangle count;
//          a block scan turns both into tile-local offsets, and each 2048-point tile writes its two totals;
//   scan:  one CTA turns the tile totals into 64-bit tile bases and writes the mesh totals V, F;
//   emit:  per point its vertices, per cell its triangles; a cell edge's vertex id is its owner point's offset plus
//          the rank of the edge's axis among that point's crossing axes.
// Workspace: per point one uint32 (local vertex offset << 3 | crossing mask) and one uint32 (local triangle offset),
// per tile two int64: 8 B per point + 16 B per 2048 points.
// The masked mode (kMasked) of both passes drops the cells with a non-finite corner, and with them every crossing edge
// that no remaining cell has; the same passes then renumber what is left.
#include <cstring>

#include "common.cuh"

namespace sparf {
namespace {

constexpr int kMcThreads = 512;
constexpr int kMcItems = 4;                         // consecutive points per thread
constexpr int kMcTile = kMcThreads * kMcItems;      // points per tile (one CTA)
constexpr int kMcRow = 3 * SPARF_MCUBES_MAX_TRIS;
constexpr int kScanThreads = 1024;

// row c: the triangles of case c as cell-edge ids (see sparf_mcubes_table), padded with -1
const signed char kTableHost[256][kMcRow] = {
#include "mcubes_table.cuh"
};
__device__ const signed char kTableDev[256][kMcRow] = {
#include "mcubes_table.cuh"
};

struct Vol {
  const float* v;
  long long nx, ny, nz, nyz, n;
  float iso;
  __device__ __forceinline__ bool in(long long p) const { return __ldg(v + p) >= iso; }   // NaN: outside
};

// linear index -> (i, j, k)
__device__ __forceinline__ void unravel(const Vol& V, long long p, long long& i, long long& j, long long& k) {
  i = p / V.nyz;
  const long long r = p - i * V.nyz;
  j = r / V.nz;
  k = r - j * V.nz;
}

// case index of the cell with origin p: bit c = corner (c & 1, c >> 1 & 1, c >> 2 & 1) is inside
__device__ __forceinline__ int cell_case(const Vol& V, long long p) {
  int c = 0;
#pragma unroll
  for (int q = 0; q < 8; ++q) c |= (int)V.in(p + (q & 1) * V.nyz + ((q >> 1) & 1) * V.nz + ((q >> 2) & 1)) << q;
  return c;
}

// bit a set: the lattice edge from (i,j,k) along axis a crosses the iso value
__device__ __forceinline__ int edge_mask(const Vol& V, long long p, long long i, long long j, long long k, bool in0) {
  int m = 0;
  if (i + 1 < V.nx) m |= (int)(V.in(p + V.nyz) != in0);
  if (j + 1 < V.ny) m |= (int)(V.in(p + V.nz) != in0) << 1;
  if (k + 1 < V.nz) m |= (int)(V.in(p + 1) != in0) << 2;
  return m;
}

// every corner of the cell with origin p is finite
__device__ __forceinline__ bool cell_finite(const Vol& V, long long p) {
  bool ok = true;
#pragma unroll
  for (int q = 0; q < 8; ++q) ok &= isfinite(__ldg(V.v + p + (q & 1) * V.nyz + ((q >> 1) & 1) * V.nz + ((q >> 2) & 1)));
  return ok;
}

// bits of mask m (edge_mask at (i,j,k)) whose lattice edge lies in a cell with finite corners.  The cells of the edge
// along a have origin p - d e_b - d' e_b' (d, d' in {0, 1}) for the two other axes b < b'.  A cell of the table uses
// every crossing edge it has, so these are the edges of the triangles kept.
__device__ __forceinline__ int finite_cell_edges(const Vol& V, long long p, long long i, long long j, long long k, int m) {
  const long long c[3] = {i, j, k}, n[3] = {V.nx, V.ny, V.nz}, stride[3] = {V.nyz, V.nz, 1};
  int out = 0;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    if (!(m >> a & 1)) continue;
    const int b = a == 0 ? 1 : 0, b2 = a == 2 ? 1 : 2;
    bool used = false;
#pragma unroll
    for (int q = 0; q < 4 && !used; ++q) {
      const long long ob = c[b] - (q & 1), ob2 = c[b2] - (q >> 1);
      if (ob >= 0 && ob + 1 < n[b] && ob2 >= 0 && ob2 + 1 < n[b2])
        used = cell_finite(V, p - (q & 1) * stride[b] - (q >> 1) * stride[b2]);
    }
    out |= (int)used << a;
  }
  return out;
}

__device__ __forceinline__ void advance(const Vol& V, long long& i, long long& j, long long& k) {
  if (++k == V.nz) {
    k = 0;
    if (++j == V.ny) {
      j = 0;
      ++i;
    }
  }
}

// exclusive block scan of two values per thread; tx, ty = the block's totals.  Each TAG has its own shared arrays, so
// that no two kernels share them and each kernel's shared layout is its own.
template <typename T, int THREADS, int TAG = 0>
__device__ __forceinline__ void block_scan2(T& x, T& y, T& tx, T& ty) {
  constexpr int NW = THREADS / 32;
  __shared__ T sx[NW], sy[NW];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  T ix = x, iy = y;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const T ux = __shfl_up_sync(0xffffffffu, ix, d), uy = __shfl_up_sync(0xffffffffu, iy, d);
    if (lane >= d) {
      ix += ux;
      iy += uy;
    }
  }
  if (lane == 31) {
    sx[w] = ix;
    sy[w] = iy;
  }
  __syncthreads();
  if (w == 0) {
    T vx = lane < NW ? sx[lane] : T(0), vy = lane < NW ? sy[lane] : T(0);
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const T ux = __shfl_up_sync(0xffffffffu, vx, d), uy = __shfl_up_sync(0xffffffffu, vy, d);
      if (lane >= d) {
        vx += ux;
        vy += uy;
      }
    }
    if (lane < NW) {
      sx[lane] = vx;
      sy[lane] = vy;
    }
  }
  __syncthreads();
  tx = sx[NW - 1];
  ty = sy[NW - 1];
  x = (w ? sx[w - 1] : T(0)) + ix - x;
  y = (w ? sy[w - 1] : T(0)) + iy - y;
  __syncthreads();  // the next call reuses sx, sy
}

// the count pass of one tile; ntri [256] = the triangle count of each case.  The kernels below own the shared table
// (a template kernel would place it after block_scan2's arrays).
template <bool kMasked>
__device__ __forceinline__ void count_tile(Vol V, const unsigned char* ntri, uint32_t* __restrict__ vpack,
                                           uint32_t* __restrict__ tloc, longlong2* __restrict__ tiles) {
  const long long p0 = (long long)blockIdx.x * kMcTile + (long long)threadIdx.x * kMcItems;
  int mask[kMcItems], nt[kMcItems];
  int sv = 0, st = 0;
  if (p0 < V.n) {
    long long i, j, k;
    unravel(V, p0, i, j, k);
#pragma unroll
    for (int u = 0; u < kMcItems; ++u) {
      const long long p = p0 + u;
      mask[u] = nt[u] = 0;
      if (p < V.n) {
        mask[u] = edge_mask(V, p, i, j, k, V.in(p));
        if constexpr (kMasked) mask[u] = finite_cell_edges(V, p, i, j, k, mask[u]);
        if (i + 1 < V.nx && j + 1 < V.ny && k + 1 < V.nz && (!kMasked || cell_finite(V, p))) nt[u] = ntri[cell_case(V, p)];
        advance(V, i, j, k);
      }
      sv += __popc(mask[u]);
      st += nt[u];
    }
  }
  int tv, tt;
  block_scan2<int, kMcThreads, kMasked>(sv, st, tv, tt);
  if (p0 < V.n) {
#pragma unroll
    for (int u = 0; u < kMcItems; ++u) {
      const long long p = p0 + u;
      if (p < V.n) {
        vpack[p] = ((uint32_t)sv << 3) | (uint32_t)mask[u];
        tloc[p] = (uint32_t)st;
      }
      sv += __popc(mask[u]);
      st += nt[u];
    }
  }
  if (threadIdx.x == 0) tiles[blockIdx.x] = make_longlong2(tv, tt);
}

__device__ __forceinline__ void fill_ntri(unsigned char* ntri) {
  if (threadIdx.x < 256) {
    int n = 0;
    while (n < SPARF_MCUBES_MAX_TRIS && kTableDev[threadIdx.x][3 * n] >= 0) ++n;
    ntri[threadIdx.x] = (unsigned char)n;
  }
  __syncthreads();
}

__global__ void __launch_bounds__(kMcThreads) mcubes_count_kernel(Vol V, uint32_t* __restrict__ vpack,
                                                                  uint32_t* __restrict__ tloc,
                                                                  longlong2* __restrict__ tiles) {
  __shared__ unsigned char ntri[256];
  fill_ntri(ntri);
  count_tile<false>(V, ntri, vpack, tloc, tiles);
}

__global__ void __launch_bounds__(kMcThreads) mcubes_count_masked_kernel(Vol V, uint32_t* __restrict__ vpack,
                                                                         uint32_t* __restrict__ tloc,
                                                                         longlong2* __restrict__ tiles) {
  __shared__ unsigned char ntri[256];
  fill_ntri(ntri);
  count_tile<true>(V, ntri, vpack, tloc, tiles);
}

// tile totals -> exclusive 64-bit tile bases (in place); totals = {V, F}
__global__ void __launch_bounds__(kScanThreads) mcubes_scan_kernel(longlong2* __restrict__ tiles, long long ntiles,
                                                                   int64_t* __restrict__ totals) {
  long long cv = 0, ct = 0;
  for (long long base = 0; base < ntiles; base += (long long)kScanThreads * kMcItems) {
    const long long t0 = base + (long long)threadIdx.x * kMcItems;
    longlong2 e[kMcItems];
    long long sv = 0, st = 0;
#pragma unroll
    for (int u = 0; u < kMcItems; ++u) {
      e[u] = t0 + u < ntiles ? tiles[t0 + u] : make_longlong2(0, 0);
      sv += e[u].x;
      st += e[u].y;
    }
    long long tv, tt;
    block_scan2<long long, kScanThreads>(sv, st, tv, tt);
    sv += cv;
    st += ct;
#pragma unroll
    for (int u = 0; u < kMcItems; ++u) {
      if (t0 + u < ntiles) tiles[t0 + u] = make_longlong2(sv, st);
      sv += e[u].x;
      st += e[u].y;
    }
    cv += tv;
    ct += tt;
  }
  if (threadIdx.x == 0) {
    totals[0] = cv;
    totals[1] = ct;
  }
}

template <bool kMasked>
__global__ void __launch_bounds__(kMcThreads) mcubes_emit_kernel(Vol V, const uint32_t* __restrict__ vpack,
                                                                 const uint32_t* __restrict__ tloc,
                                                                 const longlong2* __restrict__ tiles,
                                                                 float* __restrict__ verts, int64_t* __restrict__ faces) {
  __shared__ signed char tab[256 * kMcRow];
  for (int q = threadIdx.x; q < 256 * kMcRow; q += kMcThreads) tab[q] = (&kTableDev[0][0])[q];
  __syncthreads();
  const long long p0 = (long long)blockIdx.x * kMcTile + (long long)threadIdx.x * kMcItems;
  if (p0 >= V.n) return;
  const longlong2 base = tiles[blockIdx.x];
  long long i, j, k;
  unravel(V, p0, i, j, k);
  for (int u = 0; u < kMcItems; ++u) {
    const long long p = p0 + u;
    if (p >= V.n) break;
    const uint32_t vp = vpack[p];
    if (vp & 7u) {
      const float v0 = __ldg(V.v + p);
      long long id = base.x + (vp >> 3);
      const float c[3] = {(float)i, (float)j, (float)k};
      const long long stride[3] = {V.nyz, V.nz, 1};
#pragma unroll
      for (int a = 0; a < 3; ++a) {
        if (!(vp >> a & 1u)) continue;
        const float v1 = __ldg(V.v + p + stride[a]);
        const float s = __fdiv_rn(__fsub_rn(V.iso, v0), __fsub_rn(v1, v0));
        float* o = verts + 3 * id++;
        o[0] = a == 0 ? __fadd_rn(c[0], s) : c[0];
        o[1] = a == 1 ? __fadd_rn(c[1], s) : c[1];
        o[2] = a == 2 ? __fadd_rn(c[2], s) : c[2];
      }
    }
    if (i + 1 < V.nx && j + 1 < V.ny && k + 1 < V.nz && (!kMasked || cell_finite(V, p))) {
      const signed char* row = tab + cell_case(V, p) * kMcRow;
      int64_t* f = faces + 3 * (base.y + tloc[p]);
      for (int q = 0; q < kMcRow && row[q] >= 0; ++q) {
        // edge e = 4a + m: along axis a from the corner whose offsets on the other two axes b < b' are (m & 1, m >> 1)
        const int e = row[q], a = e >> 2, m = e & 3;
        const int oi = a == 0 ? 0 : (m & 1), oj = a == 1 ? 0 : (a == 0 ? (m & 1) : (m >> 1)), ok = a == 2 ? 0 : (m >> 1);
        const long long owner = p + oi * V.nyz + oj * V.nz + ok;
        const uint32_t ov = vpack[owner];
        f[q] = tiles[owner / kMcTile].x + (ov >> 3) + __popc(ov & 7u & ((1u << a) - 1u));
      }
    }
    advance(V, i, j, k);
  }
}

bool extents_ok(int64_t nx, int64_t ny, int64_t nz) {
  // at most 2^58 points: every byte count stays inside 64 bits
  long long n = 0;
  return nx >= 2 && ny >= 2 && nz >= 2 && !__builtin_mul_overflow((long long)nx, (long long)ny, &n) &&
         !__builtin_mul_overflow(n, (long long)nz, &n) && n <= (1ll << 58);
}

struct Carve {
  uint32_t *vpack, *tloc;
  longlong2* tiles;
  long long ntiles;
};

size_t carve(int64_t nx, int64_t ny, int64_t nz, void* ws, Carve* c) {
  const long long n = (long long)nx * ny * nz;
  const long long ntiles = (n + kMcTile - 1) / kMcTile;
  WsCarver w(ws);
  const Carve k{w.take<uint32_t>(n), w.take<uint32_t>(n), w.take<longlong2>(ntiles), ntiles};
  if (c) *c = k;
  return w.end;
}

Vol make_vol(const float* vol, int64_t nx, int64_t ny, int64_t nz, float iso) {
  return Vol{vol, nx, ny, nz, (long long)ny * nz, (long long)nx * ny * nz, iso};
}

template <bool kMasked>
int mcubes_count(const char* what, const float* vol, int64_t nx, int64_t ny, int64_t nz, float iso, int64_t* totals,
                 void* workspace, size_t workspace_bytes, sparf_stream_t stream) {
  SPARF_REQUIRE(extents_ok(nx, ny, nz), "%s: extents %lld x %lld x %lld (each >= 2, at most 2^58 points)", what,
                (long long)nx, (long long)ny, (long long)nz);
  SPARF_REQUIRE(vol && totals && workspace, "%s: NULL pointer", what);
  Carve c;
  SPARF_TRY(check_workspace(what, workspace, workspace_bytes, carve(nx, ny, nz, workspace, &c)));
  SPARF_REQUIRE(c.ntiles < (1ll << 31), "%s: volume too large", what);
  cudaStream_t s = (cudaStream_t)stream;
  const Vol V = make_vol(vol, nx, ny, nz, iso);
  (kMasked ? mcubes_count_masked_kernel : mcubes_count_kernel)<<<(unsigned)c.ntiles, kMcThreads, 0, s>>>(
      V, c.vpack, c.tloc, c.tiles);
  SPARF_CHECK_LAUNCH(kMasked ? "mcubes_count_masked_kernel" : "mcubes_count_kernel");
  mcubes_scan_kernel<<<1, kScanThreads, 0, s>>>(c.tiles, c.ntiles, totals);
  SPARF_CHECK_LAUNCH("mcubes_scan_kernel");
  return SPARF_OK;
}

template <bool kMasked>
int mcubes_emit(const char* what, const float* vol, int64_t nx, int64_t ny, int64_t nz, float iso, float* verts,
                int64_t* faces, void* workspace, size_t workspace_bytes, sparf_stream_t stream) {
  SPARF_REQUIRE(extents_ok(nx, ny, nz), "%s: extents %lld x %lld x %lld (each >= 2, at most 2^58 points)", what,
                (long long)nx, (long long)ny, (long long)nz);
  SPARF_REQUIRE(vol && workspace, "%s: NULL pointer", what);
  Carve c;
  SPARF_TRY(check_workspace(what, workspace, workspace_bytes, carve(nx, ny, nz, workspace, &c)));
  SPARF_REQUIRE(c.ntiles < (1ll << 31), "%s: volume too large", what);
  mcubes_emit_kernel<kMasked><<<(unsigned)c.ntiles, kMcThreads, 0, (cudaStream_t)stream>>>(
      make_vol(vol, nx, ny, nz, iso), c.vpack, c.tloc, c.tiles, verts, faces);
  SPARF_CHECK_LAUNCH(kMasked ? "mcubes_emit_kernel<true>" : "mcubes_emit_kernel<false>");
  return SPARF_OK;
}

}  // namespace
}  // namespace sparf

using namespace sparf;

extern "C" size_t sparf_mcubes_workspace_bytes(int64_t nx, int64_t ny, int64_t nz) {
  return extents_ok(nx, ny, nz) ? carve(nx, ny, nz, nullptr, nullptr) : 0;
}

extern "C" int sparf_mcubes_count(const float* vol, int64_t nx, int64_t ny, int64_t nz, float iso, int64_t* totals,
                                  void* workspace, size_t workspace_bytes, sparf_stream_t stream) {
  return mcubes_count<false>("mcubes_count", vol, nx, ny, nz, iso, totals, workspace, workspace_bytes, stream);
}

extern "C" int sparf_mcubes_emit(const float* vol, int64_t nx, int64_t ny, int64_t nz, float iso, float* verts,
                                 int64_t* faces, void* workspace, size_t workspace_bytes, sparf_stream_t stream) {
  return mcubes_emit<false>("mcubes_emit", vol, nx, ny, nz, iso, verts, faces, workspace, workspace_bytes, stream);
}

extern "C" int sparf_mcubes_count_masked(const float* vol, int64_t nx, int64_t ny, int64_t nz, float iso,
                                         int64_t* totals, void* workspace, size_t workspace_bytes,
                                         sparf_stream_t stream) {
  return mcubes_count<true>("mcubes_count_masked", vol, nx, ny, nz, iso, totals, workspace, workspace_bytes, stream);
}

extern "C" int sparf_mcubes_emit_masked(const float* vol, int64_t nx, int64_t ny, int64_t nz, float iso, float* verts,
                                        int64_t* faces, void* workspace, size_t workspace_bytes, sparf_stream_t stream) {
  return mcubes_emit<true>("mcubes_emit_masked", vol, nx, ny, nz, iso, verts, faces, workspace, workspace_bytes, stream);
}

extern "C" int sparf_mcubes_table(int8_t* table) {
  SPARF_REQUIRE(table, "mcubes_table: NULL pointer");
  memcpy(table, kTableHost, sizeof(kTableHost));
  return SPARF_OK;
}
