// Connected components of a vertex-welded triangle mesh, and the selection of a subset of them (floater removal).
// Semantics in include/sparf_b200.h.  Labelling is a lock-free union-find over the faces, then compact labels:
//   init:     parent[v] = v;
//   hook:     per face (a, b, c), union(a, b) and union(a, c): the larger root is linked under the smaller one with a
//             CAS, and find halves the path on its way.  So parent[x] <= x for every x, with equality iff x is a root,
//             and the root of a class is its smallest vertex id whatever the schedule;
//   compress: parent[v] = root(v), and rank[v] = (v is a root);
//   scan:     an in-place exclusive cub scan of rank: rank[r] = the number of roots below r;
//   label:    labels[v] = rank[parent[v]], and C = the number of roots.
// parent lives in the caller's labels buffer.  The face counts are integer atomics, aggregated per warp.  Selection:
// per vertex and per face a kept flag, two in-place scans into output offsets, then a scatter.
// Workspace: 4 B per vertex (rank, later the vertex offsets) + 4 B per face (the face offsets) + the scan scratch.
#include <cub/device/device_scan.cuh>

#include "common.cuh"

namespace sparf {
namespace {

constexpr int kCcThreads = 256;

// parent is written concurrently during the hook and compress passes: it is read and written through volatile
// accesses only.  A load through the non-coherent read-only path could return a stale root forever and livelock the
// hook loop.
__device__ __forceinline__ int ld_parent(const int* parent, int v) { return *(const volatile int*)(parent + v); }

// the root of v, pointing each vertex on the way at its grandparent (path halving).  A halving store only targets a
// non-root (which never becomes a root again; hooks CAS roots only) and stores one of its ancestors, so concurrent
// halvings and hooks keep every path valid.
__device__ __forceinline__ int find_root(int* parent, int v) {
  int p = ld_parent(parent, v);
  while (p != v) {
    const int g = ld_parent(parent, p);
    if (g != p) *(volatile int*)(parent + v) = g;
    v = g;
    p = ld_parent(parent, v);
  }
  return v;
}

__device__ __forceinline__ void unite(int* parent, int a, int b) {
  while (true) {
    a = find_root(parent, a);
    b = find_root(parent, b);
    if (a == b) return;
    const int lo = a < b ? a : b, hi = a < b ? b : a;
    const int old = atomicCAS(parent + hi, hi, lo);
    if (old == hi) return;
    // hi was linked by another thread meanwhile: go on from its new parent
    a = lo;
    b = old;
  }
}

__device__ __forceinline__ bool id_ok(long long x, long long n) { return x >= 0 && x < n; }

__global__ void __launch_bounds__(kCcThreads) cc_init_kernel(int n_verts, int* __restrict__ parent) {
  const long long v = thread_index();
  if (v < n_verts) parent[v] = (int)v;
}

// faces with an id outside [0, V) are skipped: no out-of-bounds access, the labels are then unspecified
__global__ void __launch_bounds__(kCcThreads) cc_hook_kernel(const int64_t* __restrict__ faces, long long n_faces,
                                                             int n_verts, int* parent) {
  const long long f = thread_index();
  if (f >= n_faces) return;
  const long long a = faces[3 * f], b = faces[3 * f + 1], c = faces[3 * f + 2];
  if (!id_ok(a, n_verts) || !id_ok(b, n_verts) || !id_ok(c, n_verts)) return;
  unite(parent, (int)a, (int)b);
  unite(parent, (int)a, (int)c);
}

// The walk does not halve: a halving store of another thread could land on parent[v] after v's own thread stored the
// root there, and leave a non-root in it.  So thread v is the only writer of parent[v], and every entry ends at its
// root.  The stores of other threads only shorten the paths a walk takes.
__global__ void __launch_bounds__(kCcThreads) cc_compress_kernel(int n_verts, int* parent, int* __restrict__ rank) {
  const long long v = thread_index();
  if (v >= n_verts) return;
  int r = (int)v, p = ld_parent(parent, r);
  while (p != r) {
    r = p;
    p = ld_parent(parent, r);
  }
  *(volatile int*)(parent + v) = r;
  rank[v] = r == (int)v;
}

// labels (= parent, compressed) -> the compact labels; the last vertex's thread writes C
__global__ void __launch_bounds__(kCcThreads) cc_label_kernel(int n_verts, int* __restrict__ labels,
                                                              const int* __restrict__ rank,
                                                              int64_t* __restrict__ n_components) {
  const long long v = thread_index();
  if (v >= n_verts) return;
  const int r = labels[v];
  labels[v] = rank[r];
  if (v == n_verts - 1) *n_components = (int64_t)rank[v] + (r == (int)v);
}

// face_counts[labels[first vertex]] += 1, one atomic per distinct label of a warp (neighbouring faces mostly share one)
__global__ void __launch_bounds__(kCcThreads) cc_face_count_kernel(const int64_t* __restrict__ faces, long long n_faces,
                                                                   long long n_verts, const int* __restrict__ labels,
                                                                   long long n_components,
                                                                   unsigned long long* __restrict__ counts) {
  const long long f = thread_index();
  int lab = -1;
  if (f < n_faces) {
    const long long a = faces[3 * f];
    if (id_ok(a, n_verts)) {
      const int l = labels[a];
      if (id_ok(l, n_components)) lab = l;
    }
  }
  const unsigned peers = __match_any_sync(0xffffffffu, lab);
  if (lab >= 0 && (threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(counts + lab, (unsigned long long)__popc(peers));
}

struct Select {
  const int64_t* faces;
  long long n_faces, n_verts;
  const int* labels;
  const uint8_t* keep;
  long long n_components;
  int *voff, *foff;         // kept flags, scanned in place into output offsets
};

__device__ __forceinline__ int vert_kept(const Select& S, long long v) {
  const int l = S.labels[v];
  return id_ok(l, S.n_components) && S.keep[l] != 0;
}

// a face is kept with the component of its first vertex (all three share it); one with an id outside [0, V) never is
__device__ __forceinline__ int face_kept(const Select& S, long long f) {
  const long long a = S.faces[3 * f], b = S.faces[3 * f + 1], c = S.faces[3 * f + 2];
  return id_ok(a, S.n_verts) && id_ok(b, S.n_verts) && id_ok(c, S.n_verts) && vert_kept(S, a);
}

// thread i: the kept flag of vertex i and of face i
__global__ void __launch_bounds__(kCcThreads) select_flag_kernel(Select S) {
  const long long i = thread_index();
  if (i < S.n_verts) S.voff[i] = vert_kept(S, i);
  if (i < S.n_faces) S.foff[i] = face_kept(S, i);
}

// totals = {V', F'}: the last offsets plus the last flags
__global__ void select_totals_kernel(Select S, int64_t* __restrict__ totals) {
  const long long v = S.n_verts - 1, f = S.n_faces - 1;
  totals[0] = (int64_t)S.voff[v] + vert_kept(S, v);
  totals[1] = f < 0 ? 0 : (int64_t)S.foff[f] + face_kept(S, f);
}

__global__ void __launch_bounds__(kCcThreads) select_emit_kernel(Select S, int64_t* __restrict__ vert_ids,
                                                                 int64_t* __restrict__ faces_out) {
  const long long i = thread_index();
  if (i < S.n_verts && vert_kept(S, i)) vert_ids[S.voff[i]] = i;
  if (i < S.n_faces && face_kept(S, i)) {
    int64_t* o = faces_out + 3 * (long long)S.foff[i];
#pragma unroll
    for (int c = 0; c < 3; ++c) o[c] = S.voff[S.faces[3 * i + c]];
  }
}

bool sizes_ok(int64_t n_verts, int64_t n_faces) {
  return n_verts >= 0 && n_verts <= INT32_MAX && n_faces >= 0 && n_faces <= INT32_MAX && (n_verts > 0 || n_faces == 0);
}

struct Carve {
  int *rank, *foff;         // rank doubles as the vertex offsets of the selection
  void* tmp;
  size_t tmp_bytes;
};

size_t carve(int64_t n_verts, int64_t n_faces, void* ws, Carve* c) {
  CubScratch tmp;
  if (n_verts > 0)
    tmp.add([&](size_t& b) { return cub::DeviceScan::ExclusiveSum(nullptr, b, (int*)nullptr, (int)n_verts); });
  if (n_faces > 0)
    tmp.add([&](size_t& b) { return cub::DeviceScan::ExclusiveSum(nullptr, b, (int*)nullptr, (int)n_faces); });
  if (!tmp.ok) return 0;
  WsCarver w(ws);
  const Carve k{w.take<int>(n_verts), w.take<int>(n_faces), w.take<char>(tmp.bytes > 0 ? tmp.bytes : 1), tmp.bytes};
  if (c) *c = k;
  return w.end;
}

#define SPARF_CC_REQUIRE_SIZES(what, V, F)                                                                        \
  SPARF_REQUIRE(sizes_ok(V, F), "%s: %lld vertices, %lld faces (each in [0, 2^31 - 1]; faces need vertices)", \
                what, (long long)(V), (long long)(F))

}  // namespace
}  // namespace sparf

using namespace sparf;

extern "C" size_t sparf_mesh_components_workspace_bytes(int64_t n_verts, int64_t n_faces) {
  return sizes_ok(n_verts, n_faces) ? carve(n_verts, n_faces, nullptr, nullptr) : 0;
}

extern "C" int sparf_mesh_components(const int64_t* faces, int64_t n_faces, int64_t n_verts, int32_t* labels,
                                     int64_t* n_components, void* workspace, size_t workspace_bytes,
                                     sparf_stream_t stream) {
  SPARF_CC_REQUIRE_SIZES("mesh_components", n_verts, n_faces);
  SPARF_REQUIRE(n_components && (n_faces == 0 || faces) && (n_verts == 0 || labels), "mesh_components: NULL pointer");
  cudaStream_t s = (cudaStream_t)stream;
  if (n_verts == 0) {
    SPARF_CHECK_CUDA(cudaMemsetAsync(n_components, 0, sizeof(int64_t), s));
    return SPARF_OK;
  }
  Carve c;
  SPARF_TRY(check_workspace("mesh_components", workspace, workspace_bytes, carve(n_verts, n_faces, workspace, &c)));
  const int V = (int)n_verts;
  cc_init_kernel<<<grid_of(V, kCcThreads), kCcThreads, 0, s>>>(V, labels);
  SPARF_CHECK_LAUNCH("cc_init_kernel");
  if (n_faces > 0) {
    cc_hook_kernel<<<grid_of(n_faces, kCcThreads), kCcThreads, 0, s>>>(faces, n_faces, V, labels);
    SPARF_CHECK_LAUNCH("cc_hook_kernel");
  }
  cc_compress_kernel<<<grid_of(V, kCcThreads), kCcThreads, 0, s>>>(V, labels, c.rank);
  SPARF_CHECK_LAUNCH("cc_compress_kernel");
  size_t t = c.tmp_bytes;
  SPARF_CHECK_CUDA(cub::DeviceScan::ExclusiveSum(c.tmp, t, c.rank, V, s));
  cc_label_kernel<<<grid_of(V, kCcThreads), kCcThreads, 0, s>>>(V, labels, c.rank, n_components);
  SPARF_CHECK_LAUNCH("cc_label_kernel");
  return SPARF_OK;
}

extern "C" int sparf_mesh_component_faces(const int64_t* faces, int64_t n_faces, int64_t n_verts, const int32_t* labels,
                                          int64_t n_components, int64_t* face_counts, sparf_stream_t stream) {
  SPARF_CC_REQUIRE_SIZES("mesh_component_faces", n_verts, n_faces);
  SPARF_REQUIRE(n_components >= 0 && n_components <= n_verts, "mesh_component_faces: %lld components of %lld vertices",
                (long long)n_components, (long long)n_verts);
  SPARF_REQUIRE((n_faces == 0 || (faces && labels)) && (n_components == 0 || face_counts),
                "mesh_component_faces: NULL pointer");
  if (n_components == 0) return SPARF_OK;
  cudaStream_t s = (cudaStream_t)stream;
  SPARF_CHECK_CUDA(cudaMemsetAsync(face_counts, 0, sizeof(int64_t) * (size_t)n_components, s));
  if (n_faces == 0) return SPARF_OK;
  cc_face_count_kernel<<<grid_of(n_faces, kCcThreads), kCcThreads, 0, s>>>(faces, n_faces, n_verts, labels,
                                                                           n_components,
                                                                           (unsigned long long*)face_counts);
  SPARF_CHECK_LAUNCH("cc_face_count_kernel");
  return SPARF_OK;
}

namespace {
int select_args(const char* what, const int64_t* faces, int64_t n_faces, int64_t n_verts, const int32_t* labels,
                const uint8_t* keep, int64_t n_components) {
  SPARF_CC_REQUIRE_SIZES(what, n_verts, n_faces);
  SPARF_REQUIRE(n_components >= 0 && n_components <= n_verts, "%s: %lld components of %lld vertices", what,
                (long long)n_components, (long long)n_verts);
  SPARF_REQUIRE((n_faces == 0 || faces) && (n_verts == 0 || labels) && (n_components == 0 || keep),
                "%s: NULL pointer", what);
  return SPARF_OK;
}
}  // namespace

extern "C" int sparf_mesh_select_count(const int64_t* faces, int64_t n_faces, int64_t n_verts, const int32_t* labels,
                                       const uint8_t* keep, int64_t n_components, int64_t* totals, void* workspace,
                                       size_t workspace_bytes, sparf_stream_t stream) {
  SPARF_TRY(select_args("mesh_select_count", faces, n_faces, n_verts, labels, keep, n_components));
  SPARF_REQUIRE(totals, "mesh_select_count: NULL pointer");
  cudaStream_t s = (cudaStream_t)stream;
  if (n_verts == 0) {
    SPARF_CHECK_CUDA(cudaMemsetAsync(totals, 0, 2 * sizeof(int64_t), s));
    return SPARF_OK;
  }
  Carve c;
  SPARF_TRY(check_workspace("mesh_select_count", workspace, workspace_bytes, carve(n_verts, n_faces, workspace, &c)));
  const Select S{faces, n_faces, n_verts, labels, keep, n_components, c.rank, c.foff};
  select_flag_kernel<<<grid_of(n_verts > n_faces ? n_verts : n_faces, kCcThreads), kCcThreads, 0, s>>>(S);
  SPARF_CHECK_LAUNCH("select_flag_kernel");
  size_t t = c.tmp_bytes;
  SPARF_CHECK_CUDA(cub::DeviceScan::ExclusiveSum(c.tmp, t, c.rank, (int)n_verts, s));
  if (n_faces > 0) {
    t = c.tmp_bytes;
    SPARF_CHECK_CUDA(cub::DeviceScan::ExclusiveSum(c.tmp, t, c.foff, (int)n_faces, s));
  }
  select_totals_kernel<<<1, 1, 0, s>>>(S, totals);
  SPARF_CHECK_LAUNCH("select_totals_kernel");
  return SPARF_OK;
}

extern "C" int sparf_mesh_select_emit(const int64_t* faces, int64_t n_faces, int64_t n_verts, const int32_t* labels,
                                      const uint8_t* keep, int64_t n_components, int64_t* vert_ids, int64_t* faces_out,
                                      void* workspace, size_t workspace_bytes, sparf_stream_t stream) {
  SPARF_TRY(select_args("mesh_select_emit", faces, n_faces, n_verts, labels, keep, n_components));
  if (n_verts == 0) return SPARF_OK;
  Carve c;
  SPARF_TRY(check_workspace("mesh_select_emit", workspace, workspace_bytes, carve(n_verts, n_faces, workspace, &c)));
  const Select S{faces, n_faces, n_verts, labels, keep, n_components, c.rank, c.foff};
  select_emit_kernel<<<grid_of(n_verts > n_faces ? n_verts : n_faces, kCcThreads), kCcThreads, 0,
                       (cudaStream_t)stream>>>(S, vert_ids, faces_out);
  SPARF_CHECK_LAUNCH("select_emit_kernel");
  return SPARF_OK;
}
