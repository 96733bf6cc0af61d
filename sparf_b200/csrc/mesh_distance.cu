// Exact closest-point queries against a triangle mesh or a point cloud over a uniform grid.  Semantics in
// include/sparf_b200.h.
//   count:  the target's bounding box (order-independent float min / max atomics), the grid (grid_setup_kernel: box,
//           padding and cells per axis), per primitive the number of cells its box overlaps, an exclusive int64 scan,
//           and the totals {entries, cells};
//   fill:   the counts and the scan again (a pure function of the grid), the (cell, primitive) pairs at the scanned
//           offsets in primitive order, one stable radix sort by cell (so each cell lists its primitives in increasing
//           id), and cell_start by a binary search per cell;
//   query:  one thread per point walks Chebyshev shells of cells around the point's (clamped) cell, and stops once the
//           planes bounding the visited box lie farther than the best distance or max_dist.
// Every point-primitive distance is one fp32 function of (point, primitive) with each operation rounded on its own, so
// the minimum (ties to the smaller id) is the same bytes for every grid.
// Workspace: 8 B per primitive (counts, scanned in place) + 12 B per entry (keys in / out, ids in) + scan / sort
// scratch.
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include "distance_grid.cuh"

namespace sparf {
namespace {

constexpr int kMdThreads = 256;
constexpr int kQueryThreads = 128;
constexpr long long kMaxCells = 1ll << 24;

__device__ __forceinline__ V3 axpy(float t, V3 d, V3 a) {   // a + t d
  return {__fadd_rn(a.x, __fmul_rn(t, d.x)), __fadd_rn(a.y, __fmul_rn(t, d.y)), __fadd_rn(a.z, __fmul_rn(t, d.z))};
}
__device__ __forceinline__ float dot(V3 a, V3 b) {
  return __fadd_rn(__fadd_rn(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)), __fmul_rn(a.z, b.z));
}
__device__ __forceinline__ V3 cross(V3 a, V3 b) {
  return {__fsub_rn(__fmul_rn(a.y, b.z), __fmul_rn(a.z, b.y)), __fsub_rn(__fmul_rn(a.z, b.x), __fmul_rn(a.x, b.z)),
          __fsub_rn(__fmul_rn(a.x, b.y), __fmul_rn(a.y, b.x))};
}
// a d - b c within 1.5 ulps (Kahan's difference of products with one FMA correction)
__device__ __forceinline__ float diff_of_products(float a, float d, float b, float c) {
  const float w = __fmul_rn(b, c);
  return __fadd_rn(__fmaf_rn(a, d, -w), __fmaf_rn(-b, c, w));
}
// The face normal: a plain fp32 cross product of a sliver's edges cancels down to a few bits, which turns its direction
// by ~2^-24 / sin(angle) and moves a distant query's foot point sideways by that times the distance.
__device__ __forceinline__ V3 cross_accurate(V3 a, V3 b) {
  return {diff_of_products(a.y, b.z, a.z, b.y), diff_of_products(a.z, b.x, a.x, b.z),
          diff_of_products(a.x, b.y, a.y, b.x)};
}
__device__ __forceinline__ float dist2(V3 a, V3 b) {
  const V3 d = sub(a, b);
  return dot(d, d);
}

// the closest point of the segment a -> b to p: the projection's parameter clamped to [0, 1] (0 when a = b)
__device__ __forceinline__ V3 closest_on_segment(V3 p, V3 a, V3 b) {
  const V3 ab = sub(b, a);
  const float l = dot(ab, ab);
  float t = 0.f;
  if (l > 0.f) t = fminf(fmaxf(__fdiv_rn(dot(sub(p, a), ab), l), 0.f), 1.f);
  return axpy(t, ab, a);
}

// The closest point of triangle abc to p, by its Voronoi regions: the projection onto the plane when it lies inside
// the triangle (face region; only when the normal n = ab x ac is nonzero), and the nearest of the three edges, whose
// clamped parameters cover the vertex regions.  All four candidates are compared, so a zero-area, collinear or
// repeated-vertex triangle is the union of its edges and a sliver's rounded face test cannot lose the minimum.  Ties go
// to the face, then the edges ab, bc, ca.  *d2 = |p - q|^2.
__device__ __forceinline__ V3 closest_on_triangle(V3 p, V3 a, V3 b, V3 c, float* d2) {
  V3 q = closest_on_segment(p, a, b);
  float best = dist2(p, q);
  const V3 q1 = closest_on_segment(p, b, c);
  const float e1 = dist2(p, q1);
  if (e1 < best) best = e1, q = q1;
  const V3 q2 = closest_on_segment(p, c, a);
  const float e2 = dist2(p, q2);
  if (e2 < best) best = e2, q = q2;
  const V3 ab = sub(b, a), ac = sub(c, a), ap = sub(p, a);
  const V3 n = cross_accurate(ab, ac);
  const float nn = dot(n, n);
  if (nn > 0.f && dot(n, cross(ab, ap)) >= 0.f && dot(n, cross(sub(c, b), sub(p, b))) >= 0.f &&
      dot(n, cross(sub(a, c), sub(p, c))) >= 0.f) {
    const V3 qf = axpy(-__fdiv_rn(dot(n, ap), nn), n, p);
    const float ef = dist2(p, qf);
    if (ef <= best) best = ef, q = qf;
  }
  *d2 = best;
  return q;
}

// float <-> int keys whose int order is the float order (atomicMin / atomicMax on floats; NaN is never stored)
__device__ __forceinline__ int fkey(float f) {
  const int i = __float_as_int(f);
  return i >= 0 ? i : i ^ 0x7fffffff;
}
__device__ __forceinline__ float fkey_inv(int k) { return __int_as_float(k >= 0 ? k : k ^ 0x7fffffff); }

struct Target {
  const float* verts;
  const int64_t* faces;     // NULL: a point target
  long long n_verts, n_prims;
};

// the cell range [lo, hi] per axis of primitive i; false for a face with an id outside [0, V)
__device__ __forceinline__ bool prim_cells(const Target& T, const SparfDistanceGrid& g, long long i, int* lo, int* hi) {
  V3 mn, mx;
  if (!T.faces) {
    mn = mx = load3(T.verts, i);
  } else {
    long long id[3];
    if (!tri_ids(T.faces, i, T.n_verts, id)) return false;
    const V3 a = load3(T.verts, id[0]), b = load3(T.verts, id[1]), c = load3(T.verts, id[2]);
    mn = {fminf(a.x, fminf(b.x, c.x)), fminf(a.y, fminf(b.y, c.y)), fminf(a.z, fminf(b.z, c.z))};
    mx = {fmaxf(a.x, fmaxf(b.x, c.x)), fmaxf(a.y, fmaxf(b.y, c.y)), fmaxf(a.z, fmaxf(b.z, c.z))};
  }
  const float mns[3] = {mn.x, mn.y, mn.z}, mxs[3] = {mx.x, mx.y, mx.z};
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    lo[a] = cell_of(mns[a], g.lo[a], g.cell[a], g.dims[a]);
    hi[a] = cell_of(mxs[a], g.lo[a], g.cell[a], g.dims[a]);
    if (hi[a] < lo[a]) hi[a] = lo[a];   // a NaN coordinate
  }
  return true;
}

__device__ __forceinline__ long long prim_count(const Target& T, const SparfDistanceGrid& g, long long i) {
  int lo[3], hi[3];
  if (!prim_cells(T, g, i, lo, hi)) return 0;
  return (long long)(hi[0] - lo[0] + 1) * (hi[1] - lo[1] + 1) * (hi[2] - lo[2] + 1);
}

// box[0..2] = fkey(min), box[3..5] = fkey(max) over the finite-or-infinite (non-NaN) vertex coordinates
__global__ void __launch_bounds__(kMdThreads) bbox_kernel(const float* __restrict__ verts, long long n_verts,
                                                          int* __restrict__ box) {
  float mn[3] = {INFINITY, INFINITY, INFINITY}, mx[3] = {-INFINITY, -INFINITY, -INFINITY};
  for (long long v = thread_index(); v < n_verts; v += (long long)gridDim.x * blockDim.x) {
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      const float x = verts[3 * v + a];
      mn[a] = fminf(mn[a], x);    // fminf / fmaxf skip NaN
      mx[a] = fmaxf(mx[a], x);
    }
  }
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    for (int o = 16; o > 0; o >>= 1) {
      mn[a] = fminf(mn[a], __shfl_xor_sync(0xffffffffu, mn[a], o));
      mx[a] = fmaxf(mx[a], __shfl_xor_sync(0xffffffffu, mx[a], o));
    }
  }
  if ((threadIdx.x & 31) == 0) {
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      atomicMin(box + a, fkey(mn[a]));
      atomicMax(box + 3 + a, fkey(mx[a]));
    }
  }
}

// The grid: the box padded by 1e-3 of its largest extent + 1e-6 of its largest |coordinate| (at least 1e-20), and
// either the given cells per axis or the automatic policy of the header.  totals[1] = the number of cells.
__global__ void grid_setup_kernel(const int* __restrict__ box, long long n_prims, int cx, int cy, int cz,
                                  SparfDistanceGrid* __restrict__ g, int64_t* __restrict__ totals) {
  float mn[3], mx[3];
  for (int a = 0; a < 3; ++a) {
    mn[a] = fkey_inv(box[a]);
    mx[a] = fkey_inv(box[3 + a]);
    if (!(mn[a] <= mx[a])) mn[a] = mx[a] = 0.f;     // no non-NaN coordinate
  }
  double L = 0.0, M = 0.0;
  for (int a = 0; a < 3; ++a) {
    L = fmax(L, (double)mx[a] - (double)mn[a]);
    M = fmax(M, fmax(fabs((double)mn[a]), fabs((double)mx[a])));
  }
  const double pad = fmax(fmax(1e-3 * L, 1e-6 * M), 1e-20);
  double ext[3];
  for (int a = 0; a < 3; ++a) {
    g->lo[a] = (float)((double)mn[a] - pad);
    ext[a] = (double)mx[a] + pad - (double)g->lo[a];
  }
  int n[3] = {cx, cy, cz};
  if (cx == 0) {
    const double target = fmin((double)kMaxCells, fmax(1.0, pow((double)n_prims, 1.5)));
    double h = cbrt(ext[0] * ext[1] * ext[2] / target);
    while (true) {
      long long total = 1;
      for (int a = 0; a < 3; ++a) {
        n[a] = (int)fmin(fmax(ceil(ext[a] / h), 1.0), (double)kMaxCells);
        total *= n[a];
        if (total > kMaxCells) break;
      }
      if (total <= kMaxCells) break;
      h *= 1.25;
    }
  }
  for (int a = 0; a < 3; ++a) {
    g->dims[a] = n[a];
    g->cell[a] = (float)(ext[a] / n[a]);
  }
  g->reserved = 0;
  totals[1] = (int64_t)n[0] * n[1] * n[2];
}

__global__ void __launch_bounds__(kMdThreads) count_kernel(Target T, const SparfDistanceGrid* __restrict__ g,
                                                           long long* __restrict__ counts) {
  const long long i = thread_index();
  if (i < T.n_prims) counts[i] = prim_count(T, *g, i);
}

// totals[0] = the entries: the last scanned offset + the last count
__global__ void entries_kernel(Target T, const SparfDistanceGrid* __restrict__ g, const long long* __restrict__ offs,
                               int64_t* __restrict__ totals) {
  totals[0] = offs[T.n_prims - 1] + prim_count(T, *g, T.n_prims - 1);
}

__global__ void __launch_bounds__(kMdThreads) emit_kernel(Target T, const SparfDistanceGrid* __restrict__ g,
                                                          const long long* __restrict__ offs, int* __restrict__ keys,
                                                          int* __restrict__ ids) {
  const long long i = thread_index();
  if (i >= T.n_prims) return;
  const SparfDistanceGrid G = *g;
  int lo[3], hi[3];
  if (!prim_cells(T, G, i, lo, hi)) return;
  long long o = offs[i];
  for (int x = lo[0]; x <= hi[0]; ++x)
    for (int y = lo[1]; y <= hi[1]; ++y)
      for (int z = lo[2]; z <= hi[2]; ++z, ++o) {
        keys[o] = (x * G.dims[1] + y) * G.dims[2] + z;
        ids[o] = (int)i;
      }
}

// cell_start[c] = the first entry whose cell is >= c, for c in [0, n_cells]
__global__ void __launch_bounds__(kMdThreads) cell_start_kernel(const int* __restrict__ keys, int n_entries,
                                                                int n_cells, int* __restrict__ cell_start) {
  const long long c = thread_index();
  if (c > n_cells) return;
  int lo = 0, hi = n_entries;
  while (lo < hi) {
    const int mid = (int)(((unsigned)lo + (unsigned)hi) >> 1);
    if (keys[mid] < c) lo = mid + 1;
    else hi = mid;
  }
  cell_start[c] = lo;
}

struct Query {
  Target T;
  const SparfDistanceGrid* grid;
  const int* cell_start;
  const int* prims;
  const float* points;
  long long n_points;
  float max_dist;
  float* dist;
  int64_t* index;
  float* closest;
};

__device__ __forceinline__ void visit(const Query& Q, V3 p, int cell, float* best_d2, int* best_id, V3* best_q) {
  const int e1 = Q.cell_start[cell + 1];
  for (int e = Q.cell_start[cell]; e < e1; ++e) {
    const int id = Q.prims[e];
    float d2;
    V3 q;
    if (!Q.T.faces) {
      q = load3(Q.T.verts, id);
      d2 = dist2(p, q);
    } else {
      const int64_t* f = Q.T.faces + 3 * (long long)id;
      q = closest_on_triangle(p, load3(Q.T.verts, f[0]), load3(Q.T.verts, f[1]), load3(Q.T.verts, f[2]), &d2);
    }
    if (d2 < *best_d2 || (d2 == *best_d2 && id < *best_id)) {
      *best_d2 = d2;
      *best_id = id;
      *best_q = q;
    }
  }
}

__global__ void __launch_bounds__(kQueryThreads) query_kernel(Query Q) {
  const long long i = thread_index();
  if (i >= Q.n_points) return;
  const SparfDistanceGrid G = *Q.grid;
  const V3 p = load3(Q.points, i);
  const float ps[3] = {p.x, p.y, p.z};
  int c[3];
  float M = 0.f, pm = 0.f;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    c[a] = cell_of(ps[a], G.lo[a], G.cell[a], G.dims[a]);
    M = fmaxf(M, fmaxf(fabsf(G.lo[a]), fabsf(G.lo[a] + G.cell[a] * G.dims[a])));
    pm = fmaxf(pm, fabsf(ps[a]));
  }
  // the bound below must stay under every computed distance of a primitive beyond a plane of the visited box: cell
  // assignment, plane positions and the distance itself each round within a few ulps of the coordinates' magnitude
  const float slop = 0x1p-18f * (pm + M);
  float best_d2 = INFINITY;
  int best_id = INT_MAX;
  V3 best_q = {NAN, NAN, NAN};
  for (int r = 0;; ++r) {
    int lo[3], hi[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      lo[a] = max(c[a] - r, 0);
      hi[a] = min(c[a] + r, G.dims[a] - 1);
    }
    for (int x = lo[0]; x <= hi[0]; ++x) {
      for (int y = lo[1]; y <= hi[1]; ++y) {
        const int row = (x * G.dims[1] + y) * G.dims[2];
        if (x == c[0] - r || x == c[0] + r || y == c[1] - r || y == c[1] + r) {
          for (int z = lo[2]; z <= hi[2]; ++z) visit(Q, p, row + z, &best_d2, &best_id, &best_q);
        } else {
          if (c[2] - r >= 0) visit(Q, p, row + c[2] - r, &best_d2, &best_id, &best_q);
          if (r > 0 && c[2] + r < G.dims[2]) visit(Q, p, row + c[2] + r, &best_d2, &best_id, &best_q);
        }
      }
    }
    // every unvisited primitive lies beyond one of the box's inner planes: its distance is at least the nearest one's
    float b = INFINITY;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      if (lo[a] > 0) b = fminf(b, ps[a] - (G.lo[a] + G.cell[a] * lo[a]));
      if (hi[a] < G.dims[a] - 1) b = fminf(b, (G.lo[a] + G.cell[a] * (hi[a] + 1)) - ps[a]);
    }
    if (b == INFINITY) break;       // the whole grid is visited
    b = (b - slop) * (1.f - 0x1p-20f);
    // strictly greater: an unvisited primitive at the same distance may have a smaller id
    if (b > fminf(sqrtf(best_d2), Q.max_dist)) break;
  }
  const float d = sqrtf(best_d2);
  const bool hit = best_id != INT_MAX && d <= Q.max_dist;
  Q.dist[i] = hit ? d : INFINITY;
  Q.index[i] = hit ? (int64_t)best_id : -1;
  Q.closest[3 * i] = hit ? best_q.x : NAN;
  Q.closest[3 * i + 1] = hit ? best_q.y : NAN;
  Q.closest[3 * i + 2] = hit ? best_q.z : NAN;
}

__global__ void __launch_bounds__(kMdThreads) miss_kernel(long long n, float* dist, int64_t* index, float* closest) {
  const long long i = thread_index();
  if (i >= n) return;
  dist[i] = INFINITY;
  index[i] = -1;
  closest[3 * i] = closest[3 * i + 1] = closest[3 * i + 2] = NAN;
}

// V, F in [0, INT32_MAX]; F = -1 is a point target; triangles need vertices
bool sizes_ok(int64_t n_verts, int64_t n_faces) {
  return n_verts >= 0 && n_verts <= INT32_MAX && n_faces >= -1 && n_faces <= INT32_MAX && (n_verts > 0 || n_faces <= 0);
}

long long prims_of(int64_t n_verts, int64_t n_faces) { return n_faces < 0 ? n_verts : n_faces; }

int sort_bits(long long n_cells) {
  int b = 0;
  while (b < 31 && (1ll << b) < n_cells) ++b;
  return b;
}

struct Ws {
  int* box;
  long long* offs;
  int *keys_in, *keys, *ids_in;
  void* tmp;
  size_t tmp_bytes;
};

// 0 when cub cannot size its scratch (no current device)
size_t carve(long long n_prims, long long n_entries, void* ws, Ws* out) {
  CubScratch tmp;
  if (n_prims > 0)
    tmp.add([&](size_t& b) {
      return cub::DeviceScan::ExclusiveSum(nullptr, b, (long long*)nullptr, (long long*)nullptr, (int)n_prims);
    });
  if (n_entries > 0)
    tmp.add([&](size_t& b) {
      return cub::DeviceRadixSort::SortPairs(nullptr, b, (int*)nullptr, (int*)nullptr, (int*)nullptr, (int*)nullptr,
                                             (int)n_entries, 0, 24);
    });
  if (!tmp.ok) return 0;
  WsCarver c(ws);
  const Ws w{c.take<int>(6), c.take<long long>(n_prims), c.take<int>(n_entries), c.take<int>(n_entries),
             c.take<int>(n_entries), c.take<char>(tmp.bytes > 0 ? tmp.bytes : 1), tmp.bytes};
  if (out) *out = w;
  return c.end;
}

// the per-primitive counts of the grid g, scanned in place into w.offs
int count_and_scan(const Target& T, const SparfDistanceGrid* g, const Ws& w, cudaStream_t s) {
  count_kernel<<<grid_of(T.n_prims, kMdThreads), kMdThreads, 0, s>>>(T, g, w.offs);
  SPARF_CHECK_LAUNCH("count_kernel");
  size_t t = w.tmp_bytes;
  SPARF_CHECK_CUDA(cub::DeviceScan::ExclusiveSum(w.tmp, t, w.offs, w.offs, (int)T.n_prims, s));
  return SPARF_OK;
}

#define SPARF_MD_REQUIRE_SIZES(what, V, F)                                                                          \
  SPARF_REQUIRE(sizes_ok(V, F), "%s: %lld vertices, %lld faces (each in [0, 2^31 - 1], faces -1 for points; faces " \
                "need vertices)", what, (long long)(V), (long long)(F))

}  // namespace
}  // namespace sparf

using namespace sparf;

extern "C" size_t sparf_distance_grid_workspace_bytes(int64_t n_prims, int64_t n_entries) {
  if (n_prims < 0 || n_prims > INT32_MAX || n_entries < 0 || n_entries > INT32_MAX) return 0;
  return carve(n_prims, n_entries, nullptr, nullptr);
}

extern "C" int sparf_distance_grid_count(const float* vertices, int64_t n_verts, const int64_t* faces, int64_t n_faces,
                                         int32_t cells_x, int32_t cells_y, int32_t cells_z, SparfDistanceGrid* grid,
                                         int64_t* totals, void* workspace, size_t workspace_bytes,
                                         sparf_stream_t stream) {
  const char* what = "distance_grid_count";
  SPARF_MD_REQUIRE_SIZES(what, n_verts, n_faces);
  const bool autoc = cells_x == 0 && cells_y == 0 && cells_z == 0;
  SPARF_REQUIRE(autoc || (cells_x >= 1 && cells_y >= 1 && cells_z >= 1 &&
                          (long long)cells_x * cells_y * cells_z <= kMaxCells),
                "%s: cells per axis %d x %d x %d (all 0, or each >= 1 with at most 2^24 cells)", what, cells_x,
                cells_y, cells_z);
  const long long P = prims_of(n_verts, n_faces);
  SPARF_REQUIRE(grid && totals && (n_verts == 0 || vertices) && (n_faces <= 0 || faces), "%s: NULL pointer", what);
  cudaStream_t s = (cudaStream_t)stream;
  if (P == 0) {     // an empty target: one cell, no entries
    SPARF_CHECK_CUDA(cudaMemsetAsync(grid, 0, sizeof(SparfDistanceGrid), s));
    SPARF_CHECK_CUDA(cudaMemsetAsync(totals, 0, 2 * sizeof(int64_t), s));
    return SPARF_OK;
  }
  Ws w;
  SPARF_TRY(check_workspace(what, workspace, workspace_bytes, carve(P, 0, workspace, &w)));
  SPARF_CHECK_CUDA(cudaMemsetAsync(w.box, 0x7f, 3 * sizeof(int), s));     // fkey(3.4e38)
  SPARF_CHECK_CUDA(cudaMemsetAsync(w.box + 3, 0x80, 3 * sizeof(int), s)); // fkey(-3.4e38)
  const unsigned nb = min(grid_of(n_verts, kMdThreads), 4u * (unsigned)num_sms());
  bbox_kernel<<<nb, kMdThreads, 0, s>>>(vertices, n_verts, w.box);
  SPARF_CHECK_LAUNCH("bbox_kernel");
  grid_setup_kernel<<<1, 1, 0, s>>>(w.box, P, cells_x, cells_y, cells_z, grid, totals);
  SPARF_CHECK_LAUNCH("grid_setup_kernel");
  const Target T{vertices, n_faces < 0 ? nullptr : faces, n_verts, P};
  SPARF_TRY(count_and_scan(T, grid, w, s));
  entries_kernel<<<1, 1, 0, s>>>(T, grid, w.offs, totals);
  SPARF_CHECK_LAUNCH("entries_kernel");
  return SPARF_OK;
}

extern "C" int sparf_distance_grid_fill(const float* vertices, int64_t n_verts, const int64_t* faces, int64_t n_faces,
                                        const SparfDistanceGrid* grid, int64_t n_cells, int64_t n_entries,
                                        int32_t* cell_start, int32_t* prims, void* workspace, size_t workspace_bytes,
                                        sparf_stream_t stream) {
  const char* what = "distance_grid_fill";
  SPARF_MD_REQUIRE_SIZES(what, n_verts, n_faces);
  const long long P = prims_of(n_verts, n_faces);
  SPARF_REQUIRE(n_cells >= 0 && n_cells <= kMaxCells && (n_cells > 0 || P == 0) && n_entries >= 0 &&
                    n_entries <= INT32_MAX && (n_entries == 0 || P > 0),
                "%s: %lld cells (at most 2^24), %lld entries (at most 2^31 - 1) of %lld primitives", what,
                (long long)n_cells, (long long)n_entries, P);
  SPARF_REQUIRE(grid && cell_start && (n_entries == 0 || prims) && (n_verts == 0 || vertices) &&
                    (n_faces <= 0 || faces),
                "%s: NULL pointer", what);
  cudaStream_t s = (cudaStream_t)stream;
  if (P == 0) {
    SPARF_CHECK_CUDA(cudaMemsetAsync(cell_start, 0, sizeof(int32_t) * (size_t)(n_cells + 1), s));
    return SPARF_OK;
  }
  Ws w;
  SPARF_TRY(check_workspace(what, workspace, workspace_bytes, carve(P, n_entries, workspace, &w)));
  const Target T{vertices, n_faces < 0 ? nullptr : faces, n_verts, P};
  if (n_entries > 0) {
    SPARF_TRY(count_and_scan(T, grid, w, s));
    emit_kernel<<<grid_of(P, kMdThreads), kMdThreads, 0, s>>>(T, grid, w.offs, w.keys_in, w.ids_in);
    SPARF_CHECK_LAUNCH("emit_kernel");
    size_t t = w.tmp_bytes;
    SPARF_CHECK_CUDA(cub::DeviceRadixSort::SortPairs(w.tmp, t, w.keys_in, w.keys, w.ids_in, prims, (int)n_entries, 0,
                                                     sort_bits(n_cells), s));
  }
  cell_start_kernel<<<grid_of(n_cells + 1, kMdThreads), kMdThreads, 0, s>>>(w.keys, (int)n_entries, (int)n_cells,
                                                                             cell_start);
  SPARF_CHECK_LAUNCH("cell_start_kernel");
  return SPARF_OK;
}

extern "C" int sparf_distance_query(const float* vertices, int64_t n_verts, const int64_t* faces, int64_t n_faces,
                                    const SparfDistanceGrid* grid, const int32_t* cell_start, const int32_t* prims,
                                    const float* points, int64_t n_points, float max_dist, float* dist,
                                    int64_t* index, float* closest, sparf_stream_t stream) {
  const char* what = "distance_query";
  SPARF_MD_REQUIRE_SIZES(what, n_verts, n_faces);
  SPARF_REQUIRE(n_points >= 0 && n_points <= INT32_MAX, "%s: %lld points (at most 2^31 - 1)", what,
                (long long)n_points);
  SPARF_REQUIRE(max_dist >= 0.f, "%s: max_dist %g (must be >= 0 or +inf)", what, (double)max_dist);
  if (n_points == 0) return SPARF_OK;
  SPARF_REQUIRE(points && dist && index && closest, "%s: NULL pointer", what);
  cudaStream_t s = (cudaStream_t)stream;
  const long long P = prims_of(n_verts, n_faces);
  if (P == 0) {
    miss_kernel<<<grid_of(n_points, kMdThreads), kMdThreads, 0, s>>>(n_points, dist, index, closest);
    SPARF_CHECK_LAUNCH("miss_kernel");
    return SPARF_OK;
  }
  SPARF_REQUIRE(grid && cell_start && vertices && (n_faces < 0 || faces), "%s: NULL pointer", what);
  const Query Q{{vertices, n_faces < 0 ? nullptr : faces, n_verts, P}, grid, cell_start, prims, points, n_points,
                max_dist, dist, index, closest};
  query_kernel<<<grid_of(n_points, kQueryThreads), kQueryThreads, 0, s>>>(Q);
  SPARF_CHECK_LAUNCH("query_kernel");
  return SPARF_OK;
}
