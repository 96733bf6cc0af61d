// The device code of the uniform grid that mesh_distance.cu builds and queries and mesh_raycast.cu walks: fp32 points,
// face ids and the cell of a coordinate.  The ray walk finds every hit only because it assigns a coordinate to the same
// cell as the build (DESIGN §3.1.15): both take cell_of from here.
#pragma once
#include "common.cuh"

namespace sparf {
namespace {

struct V3 {
  float x, y, z;
};

__device__ __forceinline__ V3 sub(V3 a, V3 b) { return {__fsub_rn(a.x, b.x), __fsub_rn(a.y, b.y), __fsub_rn(a.z, b.z)}; }
__device__ __forceinline__ V3 load3(const float* v, long long i) { return {v[3 * i], v[3 * i + 1], v[3 * i + 2]}; }

// the vertex ids of face f; false when one lies outside [0, n_verts)
__device__ __forceinline__ bool tri_ids(const int64_t* faces, long long f, long long n_verts, long long* id) {
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    id[c] = faces[3 * f + c];
    if (id[c] < 0 || id[c] >= n_verts) return false;
  }
  return true;
}

__device__ __forceinline__ int cell_of(float x, float lo, float h, int n) {
  const float t = floorf(__fdiv_rn(__fsub_rn(x, lo), h));
  return (int)fminf(fmaxf(t, 0.f), (float)(n - 1));    // NaN -> 0
}

}  // namespace
}  // namespace sparf
