// First hits of rays on a triangle mesh over the uniform grid of csrc/mesh_distance.cu.  Semantics in
// include/sparf_b200.h (mesh ray cast).
//   hit test: the watertight ray/triangle test of Woop, Benthin and Wald (JCGT 2013): the vertices relative to the
//             origin, permuted so that the dominant axis of d is z and sheared so that d becomes (0, 0, 1); the edge
//             functions U, V, W of the sheared triangle (recomputed in fp64 when one is exactly 0), a hit when they
//             share a sign and det = U + V + W != 0, t = (U Az + V Bz + W Cz) / det.  Every fp32 operation is rounded on
//             its own, so a shared edge gives exactly opposite edge functions in its two triangles.
//   walk:     one thread per ray takes the slabs of cells perpendicular to the dominant axis k of d in ray order and
//             visits, in each, the cells its segment in the slab covers, padded by a rounding slop; it stops once the
//             slab's far plane, shrunk for rounding, lies strictly beyond the best hit.  DESIGN §3.1.15 gives the
//             argument that no grid changes the result.
// No workspace.
#include "distance_grid.cuh"

namespace sparf {
namespace {

constexpr int kRcThreads = 128;
constexpr int kMissThreads = 256;

__device__ __forceinline__ float comp(V3 v, int a) { return a == 0 ? v.x : (a == 1 ? v.y : v.z); }
// element a of a per-axis array by selects (a runtime index would put the array in local memory)
template <typename T>
__device__ __forceinline__ T pick(const T (&v)[3], int a) { return a == 0 ? v[0] : (a == 1 ? v[1] : v[2]); }

// the ray in the sheared frame of the watertight test
struct Shear {
  V3 o;
  int kx, ky, kz;
  float sx, sy, sz;
};

struct Sheared {
  float x, y, z;    // z still unscaled: A[kz]
};

__device__ __forceinline__ Sheared shear(const Shear& S, V3 v) {
  const V3 a = sub(v, S.o);
  const float az = comp(a, S.kz);
  return {__fsub_rn(comp(a, S.kx), __fmul_rn(S.sx, az)), __fsub_rn(comp(a, S.ky), __fmul_rn(S.sy, az)), az};
}

__device__ __forceinline__ float edge32(Sheared p, Sheared q) { return __fsub_rn(__fmul_rn(p.x, q.y), __fmul_rn(p.y, q.x)); }
// the products of two fp32 values are exact in fp64, so the sign of the fp64 difference is the exact sign
__device__ __forceinline__ double edge64(Sheared p, Sheared q) {
  return __dsub_rn(__dmul_rn((double)p.x, (double)q.y), __dmul_rn((double)p.y, (double)q.x));
}

// true when (b - a) x (c - a) is exactly 0: fp32 differences and products are exact in fp64 for coordinates within
// 2^29 of each other's magnitude, and so is the test
__device__ __forceinline__ bool zero_area(V3 a, V3 b, V3 c) {
  const double ux = (double)b.x - a.x, uy = (double)b.y - a.y, uz = (double)b.z - a.z;
  const double vx = (double)c.x - a.x, vy = (double)c.y - a.y, vz = (double)c.z - a.z;
  return uy * vz - uz * vy == 0.0 && uz * vx - ux * vz == 0.0 && ux * vy - uy * vx == 0.0;
}

struct Cast {
  const float* verts;
  const int64_t* faces;
  long long n_verts;
  const SparfDistanceGrid* grid;
  const int* cell_start;
  const int* prims;
  const float* origins;
  const float* dirs;
  long long n_rays;
  float t_min, t_max;
  float* t;
  int64_t* face;
  float* bary;
};

struct Best {
  float t;
  int id;
  float u, v, w;
};

// the hit of triangle id, if any, replaces *B when (t, id) is smaller
__device__ __forceinline__ void test_triangle(const Cast& C, const Shear& S, int id, Best* B) {
  long long ix[3];
  if (!tri_ids(C.faces, id, C.n_verts, ix)) return;
  const V3 a = load3(C.verts, ix[0]), b = load3(C.verts, ix[1]), c = load3(C.verts, ix[2]);
  const Sheared A = shear(S, a), Bv = shear(S, b), Cv = shear(S, c);
  float U = edge32(Cv, Bv), V = edge32(A, Cv), W = edge32(Bv, A);
  if (U == 0.f || V == 0.f || W == 0.f) {
    const double U64 = edge64(Cv, Bv), V64 = edge64(A, Cv), W64 = edge64(Bv, A);
    if ((U64 < 0.0 || V64 < 0.0 || W64 < 0.0) && (U64 > 0.0 || V64 > 0.0 || W64 > 0.0)) return;
    U = (float)U64, V = (float)V64, W = (float)W64;
  } else if ((U < 0.f || V < 0.f || W < 0.f) && (U > 0.f || V > 0.f || W > 0.f)) {
    return;
  }
  const float det = __fadd_rn(__fadd_rn(U, V), W);
  if (det == 0.f) return;
  const float T = __fadd_rn(__fadd_rn(__fmul_rn(U, __fmul_rn(S.sz, A.z)), __fmul_rn(V, __fmul_rn(S.sz, Bv.z))),
                            __fmul_rn(W, __fmul_rn(S.sz, Cv.z)));
  const float t = __fdiv_rn(T, det);
  if (!(t >= C.t_min && t <= C.t_max)) return;
  if (!(t < B->t || (t == B->t && id < B->id))) return;
  if (zero_area(a, b, c)) return;
  *B = {t, id, __fdiv_rn(U, det), __fdiv_rn(V, det), __fdiv_rn(W, det)};
}

__device__ __forceinline__ void visit(const Cast& C, const Shear& S, int cell, Best* B) {
  const int e1 = C.cell_start[cell + 1];
  for (int e = C.cell_start[cell]; e < e1; ++e) test_triangle(C, S, C.prims[e], B);
}

__device__ __forceinline__ float t_at(float plane, float o, float d) { return __fdiv_rn(__fsub_rn(plane, o), d); }
__device__ __forceinline__ float x_at(float o, float t, float d) { return __fadd_rn(o, __fmul_rn(t, d)); }

__global__ void __launch_bounds__(kRcThreads) raycast_kernel(Cast C) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= C.n_rays) return;
  const SparfDistanceGrid G = *C.grid;
  const V3 o = load3(C.origins, i), d = load3(C.dirs, i);
  Best B = {INFINITY, INT_MAX, NAN, NAN, NAN};
  bool ok = true;
  int k = 0;
  float hi[3], M = 0.f, om = 0.f;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    ok = ok && isfinite(comp(o, a)) && isfinite(comp(d, a));
    if (fabsf(comp(d, a)) > fabsf(comp(d, k))) k = a;
    hi[a] = __fadd_rn(pick(G.lo, a), __fmul_rn(pick(G.cell, a), (float)pick(G.dims, a)));
    M = fmaxf(M, fmaxf(fabsf(pick(G.lo, a)), fabsf(hi[a])));
    om = fmaxf(om, fabsf(comp(o, a)));
  }
  ok = ok && comp(d, k) != 0.f;
  // Coordinates along the ray, plane positions and cell assignment each round within a few ulps of the scale: slop
  // pads the cells a slab visits and the box; stop_slop (coordinates along k) also covers the rounding of a hit's t.
  const float scale = __fadd_rn(om, M);
  const float slop = 0x1p-18f * scale, stop_slop = 0x1p-14f * scale;
  float t0 = C.t_min, t1 = C.t_max;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const float lo = __fsub_rn(pick(G.lo, a), slop), up = __fadd_rn(hi[a], slop);
    if (comp(d, a) == 0.f) {
      ok = ok && comp(o, a) >= lo && comp(o, a) <= up;
    } else {
      const float ta = t_at(lo, comp(o, a), comp(d, a)), tb = t_at(up, comp(o, a), comp(d, a));
      t0 = fmaxf(t0, fminf(ta, tb));
      t1 = fminf(t1, fmaxf(ta, tb));
    }
  }
  const float dk = comp(d, k), o_k = comp(o, k), adk = fabsf(dk);
  const float widen = __fdiv_rn(stop_slop, adk);
  t0 = __fsub_rn(__fsub_rn(t0, __fmul_rn(fabsf(t0), 0x1p-20f)), widen);
  t1 = __fadd_rn(__fadd_rn(t1, __fmul_rn(fabsf(t1), 0x1p-20f)), widen);
  if (ok && t0 <= t1) {
    const int i1 = k == 0 ? 1 : 0, i2 = k == 2 ? 1 : 2;   // the two other axes
    Shear S;
    S.o = o;
    S.kz = k;
    S.kx = (k + 1) % 3;
    S.ky = (k + 2) % 3;
    S.sx = __fdiv_rn(comp(d, S.kx), dk);
    S.sy = __fdiv_rn(comp(d, S.ky), dk);
    S.sz = __fdiv_rn(1.f, dk);
    const int n = pick(G.dims, k), dir = dk > 0.f ? 1 : -1;
    const float sg = dir > 0 ? slop : -slop;
    const int s_first = cell_of(__fsub_rn(x_at(o_k, t0, dk), sg), pick(G.lo, k), pick(G.cell, k), n);
    const int s_last = cell_of(__fadd_rn(x_at(o_k, t1, dk), sg), pick(G.lo, k), pick(G.cell, k), n);
    const int stride_k = k == 0 ? G.dims[1] * G.dims[2] : (k == 1 ? G.dims[2] : 1);
    const int stride_1 = i1 == 0 ? G.dims[1] * G.dims[2] : (i1 == 1 ? G.dims[2] : 1);
    const int stride_2 = i2 == 1 ? G.dims[2] : 1;
    for (int s = s_first;; s += dir) {
      // the slab's planes in ray order; the grid's first and last slabs reach to the ends of the walk (cell_of clamps)
      const int p_near = dir > 0 ? s : s + 1, p_far = dir > 0 ? s + 1 : s;
      const float P_near = __fadd_rn(pick(G.lo, k), __fmul_rn(pick(G.cell, k), (float)p_near));
      const float P_far = __fadd_rn(pick(G.lo, k), __fmul_rn(pick(G.cell, k), (float)p_far));
      const float ta = (p_near == 0 || p_near == n) ? t0 : fmaxf(t0, t_at(__fsub_rn(P_near, sg), o_k, dk));
      const float tb = (p_far == 0 || p_far == n) ? t1 : fminf(t1, t_at(__fadd_rn(P_far, sg), o_k, dk));
      if (ta <= tb) {
        int c_lo[2], c_hi[2];
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          const int a = j == 0 ? i1 : i2;
          const float xa = x_at(comp(o, a), ta, comp(d, a)), xb = x_at(comp(o, a), tb, comp(d, a));
          c_lo[j] = cell_of(__fsub_rn(fminf(xa, xb), slop), pick(G.lo, a), pick(G.cell, a), pick(G.dims, a));
          c_hi[j] = cell_of(__fadd_rn(fmaxf(xa, xb), slop), pick(G.lo, a), pick(G.cell, a), pick(G.dims, a));
        }
        for (int u = c_lo[0]; u <= c_hi[0]; ++u)
          for (int v = c_lo[1]; v <= c_hi[1]; ++v) visit(C, S, s * stride_k + u * stride_1 + v * stride_2, &B);
      }
      if (s == s_last) break;
      // every hit not yet visited lies beyond the far plane (its cell along k comes later in ray order); strictly
      // greater: a later triangle at the same t may have a smaller id
      float nb = t_at(__fsub_rn(P_far, dir > 0 ? stop_slop : -stop_slop), o_k, dk);
      nb = __fsub_rn(nb, __fmul_rn(fabsf(nb), 0x1p-20f));
      if (nb > B.t) break;
    }
  }
  const bool hit = B.id != INT_MAX;
  C.t[i] = hit ? B.t : INFINITY;
  C.face[i] = hit ? (int64_t)B.id : -1;
  C.bary[3 * i] = B.u;      // NaN on a miss
  C.bary[3 * i + 1] = B.v;
  C.bary[3 * i + 2] = B.w;
}

__global__ void __launch_bounds__(kMissThreads) miss_kernel(long long n, float* t, int64_t* face, float* bary) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  t[i] = INFINITY;
  face[i] = -1;
  bary[3 * i] = bary[3 * i + 1] = bary[3 * i + 2] = NAN;
}

}  // namespace
}  // namespace sparf

using namespace sparf;

extern "C" int sparf_raycast(const float* vertices, int64_t n_verts, const int64_t* faces, int64_t n_faces,
                             const SparfDistanceGrid* grid, const int32_t* cell_start, const int32_t* prims,
                             const float* origins, const float* dirs, int64_t n_rays, float t_min, float t_max,
                             float* t, int64_t* face, float* bary, sparf_stream_t stream) {
  const char* what = "raycast";
  SPARF_REQUIRE(n_verts >= 0 && n_verts <= INT32_MAX && n_faces >= 0 && n_faces <= INT32_MAX &&
                    (n_verts > 0 || n_faces == 0),
                "%s: %lld vertices, %lld faces (each in [0, 2^31 - 1]; faces need vertices)", what,
                (long long)n_verts, (long long)n_faces);
  SPARF_REQUIRE(n_rays >= 0 && n_rays <= INT32_MAX, "%s: %lld rays (at most 2^31 - 1)", what, (long long)n_rays);
  SPARF_REQUIRE(t_min >= 0.f && t_max >= t_min, "%s: t_min %g, t_max %g (need 0 <= t_min <= t_max, +inf allowed)",
                what, (double)t_min, (double)t_max);
  if (n_rays == 0) return SPARF_OK;
  SPARF_REQUIRE(origins && dirs && t && face && bary, "%s: NULL pointer", what);
  cudaStream_t s = (cudaStream_t)stream;
  if (n_faces == 0) {
    miss_kernel<<<grid_of(n_rays, kMissThreads), kMissThreads, 0, s>>>(n_rays, t, face, bary);
    SPARF_CHECK_LAUNCH("miss_kernel");
    return SPARF_OK;
  }
  SPARF_REQUIRE(grid && cell_start && vertices && faces, "%s: NULL pointer", what);
  const Cast C{vertices, faces, n_verts, grid, cell_start, prims, origins, dirs, n_rays, t_min, t_max, t, face, bary};
  raycast_kernel<<<grid_of(n_rays, kRcThreads), kRcThreads, 0, s>>>(C);
  SPARF_CHECK_LAUNCH("raycast_kernel");
  return SPARF_OK;
}
