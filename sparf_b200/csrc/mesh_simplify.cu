// Mesh simplification by quadric error metrics (Garland-Heckbert) in parallel rounds of independent edge collapses.
// Semantics in include/sparf_b200.h; tests/simplify_oracle.py restates them in NumPy.  One round:
//   build:    per live face i, three half-edge entries (lo << nb | hi, i) and three vertex entries (v, i);
//   sort:     two stable cub radix sorts: the edges (unique edges = runs, a run's values = the edge's faces) and the
//             vertices (a run = the vertex's live faces in increasing order, vstart by binary search);
//   edges:    head flags, an inclusive scan -> edge ids, estart[e] = first entry of edge e, E on the device;
//   classify: per edge its face count flags its endpoints boundary (1) or locked (>= 3); a face with repeated ids locks
//             its vertices (during build);
//   key:      per edge collapsible + link condition + v* + fold check -> key = cost bits << 32 | e, or ~0 if not valid;
//   select:   the k-th smallest key by an 8-pass radix select (256-bin histograms over the keys, one digit a pass);
//   claim:    every candidate (key <= k-th, valid) atomicMin's its key onto the vertices of the faces around a and b;
//   win:      a candidate holding every one of them collapses at once (the regions of winners are disjoint);
//   compact:  dead faces dropped, ids renamed through ren, flags scanned, the kept faces written in their order.
// All fp64 arithmetic of the quadric, position and cost path goes through rounded intrinsics (no FMA contraction), so
// the NumPy oracle, whose scalar operations round the same way, reproduces every bit.
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include "common.cuh"

namespace sparf {
namespace {

constexpr int kMsThreads = 256;
constexpr unsigned long long kNoKey = ~0ull;
constexpr int64_t kMaxFaces = INT32_MAX / 3;    // 3 F half-edge entries are counted in int (cub's item count)

__device__ __forceinline__ double ad(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double sb(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double ml(double a, double b) { return __dmul_rn(a, b); }

struct V3 {
  double x, y, z;
};

__device__ __forceinline__ V3 load3(const float* p, int v) {
  return V3{(double)p[3 * v], (double)p[3 * v + 1], (double)p[3 * v + 2]};
}
__device__ __forceinline__ V3 sub3(V3 a, V3 b) { return V3{sb(a.x, b.x), sb(a.y, b.y), sb(a.z, b.z)}; }
__device__ __forceinline__ double dot3(V3 a, V3 b) { return ad(ad(ml(a.x, b.x), ml(a.y, b.y)), ml(a.z, b.z)); }
// (p1 - p0) x (p2 - p0)
__device__ __forceinline__ V3 tri_cross(V3 p0, V3 p1, V3 p2) {
  const V3 u = sub3(p1, p0), w = sub3(p2, p0);
  return V3{sb(ml(u.y, w.z), ml(u.z, w.y)), sb(ml(u.z, w.x), ml(u.x, w.z)), sb(ml(u.x, w.y), ml(u.y, w.x))};
}
__device__ __forceinline__ V3 round_f32(V3 a) {
  return V3{(double)__double2float_rn(a.x), (double)__double2float_rn(a.y), (double)__double2float_rn(a.z)};
}

// the area-weighted plane quadric of a face: q_ij = (w n_i) n_j over (i, j) = 00 01 02 03 11 12 13 22 23 33,
// n4 = (c / |c|, -n . p0), w = |c| / 2; a zero-area face gives 0
__device__ void face_quadric(V3 p0, V3 p1, V3 p2, double q[10]) {
  const V3 c = tri_cross(p0, p1, p2);
  const double len = __dsqrt_rn(dot3(c, c));
  if (!(len > 0.0)) {
#pragma unroll
    for (int i = 0; i < 10; ++i) q[i] = 0.0;
    return;
  }
  const V3 n{__ddiv_rn(c.x, len), __ddiv_rn(c.y, len), __ddiv_rn(c.z, len)};
  const double n4[4] = {n.x, n.y, n.z, -dot3(n, p0)};
  const double w = ml(len, 0.5);
  int k = 0;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const double wn = ml(w, n4[i]);
#pragma unroll
    for (int j = i; j < 4; ++j) q[k++] = ml(wn, n4[j]);
  }
}

// v^T Q v with v = (x, y, z, 1), in this order
__device__ double quad_eval(const double q[10], V3 v) {
  double r = ml(ml(q[0], v.x), v.x);
  r = ad(r, ml(2.0, ml(ml(q[1], v.x), v.y)));
  r = ad(r, ml(2.0, ml(ml(q[2], v.x), v.z)));
  r = ad(r, ml(2.0, ml(q[3], v.x)));
  r = ad(r, ml(ml(q[4], v.y), v.y));
  r = ad(r, ml(2.0, ml(ml(q[5], v.y), v.z)));
  r = ad(r, ml(2.0, ml(q[6], v.y)));
  r = ad(r, ml(ml(q[7], v.z), v.z));
  r = ad(r, ml(2.0, ml(q[8], v.z)));
  return ad(r, q[9]);
}

__device__ __forceinline__ double det3(double a00, double a01, double a02, double a10, double a11, double a12,
                                       double a20, double a21, double a22) {
  return ad(sb(ml(a00, sb(ml(a11, a22), ml(a12, a21))), ml(a01, sb(ml(a10, a22), ml(a12, a20)))),
            ml(a02, sb(ml(a10, a21), ml(a11, a20))));
}

struct Collapse {
  V3 v;            // v* (fp32 values)
  double cost;     // quadric of Q[a] + Q[b] at v*
  int s;           // the survivor
};

// v* and its cost for the edge (a, b), a < b (header: "position v*")
__device__ Collapse place(const float* pos, const double* Q, const uint8_t* bnd, int a, int b) {
  double q[10];
#pragma unroll
  for (int i = 0; i < 10; ++i) q[i] = ad(Q[10 * (size_t)a + i], Q[10 * (size_t)b + i]);
  const V3 pa = load3(pos, a), pb = load3(pos, b);
  if (bnd[a] || bnd[b]) {
    const int s = bnd[a] ? a : b;
    const V3 v = bnd[a] ? pa : pb;
    return Collapse{v, quad_eval(q, v), s};
  }
  const double det = det3(q[0], q[1], q[2], q[1], q[4], q[5], q[2], q[5], q[7]);
  const double tr = ad(ad(q[0], q[4]), q[7]);
  if (fabs(det) > ml(1e-10, ml(ml(tr, tr), tr))) {
    const double b0 = -q[3], b1 = -q[6], b2 = -q[8];
    const V3 x = round_f32(V3{__ddiv_rn(det3(b0, q[1], q[2], b1, q[4], q[5], b2, q[5], q[7]), det),
                              __ddiv_rn(det3(q[0], b0, q[2], q[1], b1, q[5], q[2], b2, q[7]), det),
                              __ddiv_rn(det3(q[0], q[1], b0, q[1], q[4], b1, q[2], q[5], b2), det)});
    const V3 mid{ml(ad(pa.x, pb.x), 0.5), ml(ad(pa.y, pb.y), 0.5), ml(ad(pa.z, pb.z), 0.5)};
    const V3 dm = sub3(x, mid), ab = sub3(pb, pa);
    if (dot3(dm, dm) <= dot3(ab, ab)) return Collapse{x, quad_eval(q, x), a};
  }
  const V3 mid = round_f32(V3{ml(ad(pa.x, pb.x), 0.5), ml(ad(pa.y, pb.y), 0.5), ml(ad(pa.z, pb.z), 0.5)});
  Collapse best{pa, quad_eval(q, pa), a};
  const double cb = quad_eval(q, pb), cm = quad_eval(q, mid);
  if (cb < best.cost) best = Collapse{pb, cb, a};
  if (cm < best.cost) best = Collapse{mid, cm, a};
  return best;
}

// the round's state, carved from the workspace (see carve for the layout and the aliases)
struct Ws {
  float *pos, *attrs;
  double* q;
  int* ren;                         // ren[r] = s once r is removed, else r
  uint8_t *bnd, *lock;
  unsigned long long* claim;
  int* vstart;                      // [V + 1]
  int* faces;                       // [F][3] live faces, int32
  uint8_t* dead;                    // [F]
  unsigned long long *ekeys_in, *ekeys;
  int *evals_in, *evals, *vkeys_in, *vkeys, *vvals_in, *vvals;
  int* estart;                      // [3F + 1]
  unsigned long long* ckey;         // = ekeys_in  (per-edge keys, after the sorts)
  int* eid;                         // = evals_in  (scanned head flags)
  int* faces_tmp;                   // = vkeys_in  (the compacted faces)
  int* foff;                        // = vvals_in  (face offsets; vertex offsets in emit)
  unsigned long long* sel;          // {prefix, thresh, rank, done, E}
  unsigned* hist;                   // [256]
  void* tmp;
  size_t tmp_bytes;
};

__device__ __forceinline__ long long thread_index() { return (long long)blockIdx.x * blockDim.x + threadIdx.x; }
unsigned grid_of(long long n) { return (unsigned)((n + kMsThreads - 1) / kMsThreads); }

int id_bits(int64_t n_verts) {
  int nb = 1;
  while (nb < 31 && ((int64_t)1 << nb) < n_verts) ++nb;
  return nb;
}

__global__ void __launch_bounds__(kMsThreads) ms_init_kernel(const int64_t* __restrict__ faces, int n_faces,
                                                             int n_verts, Ws w, int64_t* __restrict__ counts) {
  const long long i = thread_index();
  if (i < 3ll * n_faces) w.faces[i] = (int)faces[i];
  if (i < n_verts) w.ren[i] = (int)i;
  if (i == 0) {
    counts[0] = n_faces;
    counts[1] = 0;
  }
}

// the entries of the two sorts; a face with repeated ids locks its vertices
__global__ void __launch_bounds__(kMsThreads) ms_build_kernel(int n_live, int nb, Ws w) {
  const long long i = thread_index();
  if (i >= n_live) return;
  const int f[3] = {w.faces[3 * i], w.faces[3 * i + 1], w.faces[3 * i + 2]};
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const int u = f[c], v = f[c == 2 ? 0 : c + 1];
    const unsigned long long lo = u < v ? u : v, hi = u < v ? v : u;
    w.ekeys_in[3 * i + c] = lo << nb | hi;
    w.evals_in[3 * i + c] = (int)i;
    w.vkeys_in[3 * i + c] = u;
    w.vvals_in[3 * i + c] = (int)i;
  }
  if (f[0] == f[1] || f[1] == f[2] || f[0] == f[2]) w.lock[f[0]] = w.lock[f[1]] = w.lock[f[2]] = 1;
}

// vstart[v] = the first sorted vertex entry >= v (v in [0, V])
__global__ void __launch_bounds__(kMsThreads) ms_vstart_kernel(int n_verts, int n_entries, Ws w) {
  const long long v = thread_index();
  if (v > n_verts) return;
  int lo = 0, hi = n_entries;
  while (lo < hi) {
    const int m = (lo + hi) >> 1;
    if (w.vkeys[m] < v) lo = m + 1;
    else hi = m;
  }
  w.vstart[v] = lo;
}

// Q[v] = the sum of the quadrics of v's faces in increasing face id (a face with repeated ids adds 0, its area)
__global__ void __launch_bounds__(kMsThreads) ms_quadric_kernel(int n_verts, Ws w) {
  const long long v = thread_index();
  if (v >= n_verts) return;
  double q[10] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
  for (int j = w.vstart[v]; j < w.vstart[v + 1]; ++j) {
    const int* f = w.faces + 3 * (size_t)w.vvals[j];
    double fq[10];
    face_quadric(load3(w.pos, f[0]), load3(w.pos, f[1]), load3(w.pos, f[2]), fq);
#pragma unroll
    for (int i = 0; i < 10; ++i) q[i] = ad(q[i], fq[i]);
  }
#pragma unroll
  for (int i = 0; i < 10; ++i) w.q[10 * v + i] = q[i];
}

__global__ void ms_round_begin_kernel(Ws w, long long k, int64_t* __restrict__ counts) {
  w.sel[0] = 0;           // prefix
  w.sel[1] = kNoKey;      // thresh
  w.sel[2] = (unsigned long long)k;
  w.sel[3] = 0;           // done
  for (int d = 0; d < 256; ++d) w.hist[d] = 0;
  counts[1] = 0;
}

__global__ void __launch_bounds__(kMsThreads) ms_head_kernel(int n_entries, Ws w) {
  const long long i = thread_index();
  if (i < n_entries) w.eid[i] = i == 0 || w.ekeys[i] != w.ekeys[i - 1];
}

// heads of the sorted edge entries: estart[edge id] = first entry; the last thread writes E and estart[E]
__global__ void __launch_bounds__(kMsThreads) ms_edge_start_kernel(int n_entries, Ws w) {
  const long long i = thread_index();
  if (i >= n_entries) return;
  if (i == 0 || w.ekeys[i] != w.ekeys[i - 1]) w.estart[w.eid[i] - 1] = (int)i;
  if (i == n_entries - 1) {
    w.estart[w.eid[i]] = n_entries;
    w.sel[4] = (unsigned long long)w.eid[i];
  }
}

__device__ __forceinline__ void edge_ends(const Ws& w, int nb, int e, int* a, int* b) {
  const unsigned long long key = w.ekeys[w.estart[e]];
  *a = (int)(key >> nb);
  *b = (int)(key & ((1ull << nb) - 1));
}

__global__ void __launch_bounds__(kMsThreads) ms_classify_kernel(int nb, Ws w) {
  const long long e = thread_index();
  if (e >= (long long)w.sel[4]) return;
  const int n = w.estart[e + 1] - w.estart[e];
  if (n == 2) return;
  int a, b;
  edge_ends(w, nb, (int)e, &a, &b);
  uint8_t* flag = n == 1 ? w.bnd : w.lock;
  flag[a] = flag[b] = 1;
}

__device__ __forceinline__ bool has(const int* f, int x) { return f[0] == x || f[1] == x || f[2] == x; }
__device__ __forceinline__ int third(const int* f, int a, int b) {
  return f[0] != a && f[0] != b ? f[0] : f[1] != a && f[1] != b ? f[1] : f[2];
}

// Lk(a) n Lk(b) = Lk(ab) for the interior edge (a, b) with faces abc, abd: c != d, no common neighbour but c and d,
// and not both acd and bcd (a tetrahedron)
__device__ bool link_ok(const Ws& w, int a, int b, int c, int d) {
  if (c == d) return false;
  bool acd = false, bcd = false;
  for (int j = w.vstart[a]; j < w.vstart[a + 1]; ++j) {
    const int* fa = w.faces + 3 * (size_t)w.vvals[j];
    acd = acd || (has(fa, c) && has(fa, d));
    for (int t = 0; t < 3; ++t) {
      const int x = fa[t];
      if (x == a || x == b || x == c || x == d) continue;
      for (int i = w.vstart[b]; i < w.vstart[b + 1]; ++i)
        if (has(w.faces + 3 * (size_t)w.vvals[i], x)) return false;
    }
  }
  for (int i = w.vstart[b]; i < w.vstart[b + 1] && !bcd; ++i) {
    const int* fb = w.faces + 3 * (size_t)w.vvals[i];
    bcd = has(fb, c) && has(fb, d);
  }
  return !(acd && bcd);
}

// every live face around v that does not hold both a and b and has a nonzero normal keeps a positive dot of its new and
// old normals
__device__ bool no_fold(const Ws& w, int v, int a, int b, V3 vs) {
  for (int j = w.vstart[v]; j < w.vstart[v + 1]; ++j) {
    const int* f = w.faces + 3 * (size_t)w.vvals[j];
    if (has(f, a) && has(f, b)) continue;
    const V3 p[3] = {load3(w.pos, f[0]), load3(w.pos, f[1]), load3(w.pos, f[2])};
    const V3 n_old = tri_cross(p[0], p[1], p[2]);
    if (n_old.x == 0.0 && n_old.y == 0.0 && n_old.z == 0.0) continue;    // no orientation to keep
    const V3 n_new = tri_cross(f[0] == v ? vs : p[0], f[1] == v ? vs : p[1], f[2] == v ? vs : p[2]);
    if (!(dot3(n_new, n_old) > 0.0)) return false;
  }
  return true;
}

__global__ void __launch_bounds__(kMsThreads) ms_key_kernel(int nb, Ws w) {
  const long long e = thread_index();
  if (e >= (long long)w.sel[4]) return;
  unsigned long long key = kNoKey;
  const int e0 = w.estart[e];
  int a, b;
  edge_ends(w, nb, (int)e, &a, &b);
  if (w.estart[e + 1] - e0 == 2 && !w.lock[a] && !w.lock[b] && !(w.bnd[a] && w.bnd[b])) {
    const int c = third(w.faces + 3 * (size_t)w.evals[e0], a, b);
    const int d = third(w.faces + 3 * (size_t)w.evals[e0 + 1], a, b);
    if (link_ok(w, a, b, c, d)) {
      const Collapse k = place(w.pos, w.q, w.bnd, a, b);
      if (no_fold(w, a, a, b, k.v) && no_fold(w, b, a, b, k.v)) {
        const float cost = __double2float_rn(k.cost > 0.0 ? k.cost : 0.0);
        key = (unsigned long long)__float_as_uint(cost) << 32 | (unsigned long long)e;
      }
    }
  }
  w.ckey[e] = key;
}

// radix select, pass p: the histogram of digit p (bits 56 - 8p ..) over the keys that match the prefix above it
__global__ void __launch_bounds__(kMsThreads) ms_hist_kernel(int pass, Ws w) {
  if (w.sel[3]) return;
  __shared__ unsigned h[256];
  h[threadIdx.x] = 0;
  __syncthreads();
  const int shift = 56 - 8 * pass;
  const unsigned long long high = pass == 0 ? 0 : ~0ull << (shift + 8), prefix = w.sel[0];
  const long long n = (long long)w.sel[4];
  for (long long i = thread_index(); i < n; i += (long long)gridDim.x * blockDim.x) {
    const unsigned long long key = w.ckey[i];
    if (((key ^ prefix) & high) == 0) atomicAdd(&h[(key >> shift) & 255], 1u);
  }
  __syncthreads();
  if (h[threadIdx.x]) atomicAdd(&w.hist[threadIdx.x], h[threadIdx.x]);
}

// the digit that holds the rank-th key; when fewer keys match than the rank, every valid key is a candidate
__global__ void ms_pick_kernel(int pass, Ws w) {
  if (w.sel[3]) return;
  const int shift = 56 - 8 * pass;
  unsigned long long cum = 0, rank = w.sel[2];
  int d = 0;
  for (; d < 256; ++d) {
    const unsigned long long h = w.hist[d];
    if (cum + h >= rank) break;
    cum += h;
  }
  for (int i = 0; i < 256; ++i) w.hist[i] = 0;
  if (d == 256) {
    w.sel[1] = kNoKey;
    w.sel[3] = 1;
    return;
  }
  w.sel[0] |= (unsigned long long)d << shift;
  w.sel[2] = rank - cum;
  if (pass == 7) w.sel[1] = w.sel[0];
}

__device__ __forceinline__ bool candidate(const Ws& w, long long e, unsigned long long* key) {
  *key = w.ckey[e];
  return *key != kNoKey && *key <= w.sel[1];
}

__global__ void __launch_bounds__(kMsThreads) ms_claim_kernel(int nb, Ws w) {
  const long long e = thread_index();
  unsigned long long key;
  if (e >= (long long)w.sel[4] || !candidate(w, e, &key)) return;
  int ab[2];
  edge_ends(w, nb, (int)e, &ab[0], &ab[1]);
  for (int t = 0; t < 2; ++t)
    for (int j = w.vstart[ab[t]]; j < w.vstart[ab[t] + 1]; ++j) {
      const int* f = w.faces + 3 * (size_t)w.vvals[j];
      for (int c = 0; c < 3; ++c) atomicMin(w.claim + f[c], key);
    }
}

// a candidate that holds all of its vertices collapses: pos, Q and attrs of the survivor, ren of the removed vertex,
// its two faces dead.  Winners' regions are disjoint, and nothing else reads pos, Q or attrs here.
__global__ void __launch_bounds__(kMsThreads) ms_win_kernel(int nb, int n_attrs, Ws w, int64_t* __restrict__ counts) {
  const long long e = thread_index();
  unsigned long long key;
  if (e >= (long long)w.sel[4] || !candidate(w, e, &key)) return;
  int a, b;
  edge_ends(w, nb, (int)e, &a, &b);
  const int ab[2] = {a, b};
  for (int t = 0; t < 2; ++t)
    for (int j = w.vstart[ab[t]]; j < w.vstart[ab[t] + 1]; ++j) {
      const int* f = w.faces + 3 * (size_t)w.vvals[j];
      for (int c = 0; c < 3; ++c)
        if (w.claim[f[c]] != key) return;
    }
  const Collapse k = place(w.pos, w.q, w.bnd, a, b);
  const int s = k.s, r = s == a ? b : a;
  const V3 pa = load3(w.pos, a), pb = load3(w.pos, b), ab3 = sub3(pb, pa);
  const double den = dot3(ab3, ab3);
  double t = den > 0.0 ? __ddiv_rn(dot3(sub3(k.v, pa), ab3), den) : 0.0;
  t = t < 0.0 ? 0.0 : t > 1.0 ? 1.0 : t;
  for (int i = 0; i < n_attrs; ++i) {
    const double xa = w.attrs[(size_t)a * n_attrs + i], xb = w.attrs[(size_t)b * n_attrs + i];
    w.attrs[(size_t)s * n_attrs + i] = __double2float_rn(ad(xa, ml(t, sb(xb, xa))));
  }
#pragma unroll
  for (int i = 0; i < 10; ++i) w.q[10 * (size_t)s + i] = ad(w.q[10 * (size_t)s + i], w.q[10 * (size_t)r + i]);
  w.pos[3 * (size_t)s] = (float)k.v.x;
  w.pos[3 * (size_t)s + 1] = (float)k.v.y;
  w.pos[3 * (size_t)s + 2] = (float)k.v.z;
  w.ren[r] = s;
  const int e0 = w.estart[e];
  w.dead[w.evals[e0]] = w.dead[w.evals[e0 + 1]] = 1;
  atomicAdd((unsigned long long*)counts + 1, 1ull);
}

__global__ void __launch_bounds__(kMsThreads) ms_face_flag_kernel(int n_live, Ws w) {
  const long long i = thread_index();
  if (i < n_live) w.foff[i] = !w.dead[i];
}

__global__ void __launch_bounds__(kMsThreads) ms_face_emit_kernel(int n_live, Ws w, int64_t* __restrict__ counts) {
  const long long i = thread_index();
  if (i >= n_live) return;
  if (!w.dead[i]) {
    int* o = w.faces_tmp + 3 * (size_t)w.foff[i];
#pragma unroll
    for (int c = 0; c < 3; ++c) o[c] = w.ren[w.faces[3 * i + c]];
  }
  if (i == n_live - 1) counts[0] = (int64_t)w.foff[i] + !w.dead[i];
}

// emit: vertex kept flags (ren[v] == v) -> offsets; then the vertices, their attributes and ids, and the faces
__global__ void __launch_bounds__(kMsThreads) ms_vert_flag_kernel(int n_verts, Ws w) {
  const long long v = thread_index();
  if (v < n_verts) w.foff[v] = w.ren[v] == (int)v;
}

__global__ void __launch_bounds__(kMsThreads) ms_emit_kernel(int n_verts, int n_live, int n_attrs, Ws w,
                                                             float* __restrict__ vertices, float* __restrict__ attrs,
                                                             int64_t* __restrict__ vert_ids, int64_t* __restrict__ faces) {
  const long long i = thread_index();
  if (i < n_verts && w.ren[i] == (int)i) {
    const int o = w.foff[i];
    vert_ids[o] = i;
    for (int c = 0; c < 3; ++c) vertices[3 * (size_t)o + c] = w.pos[3 * i + c];
    for (int c = 0; c < n_attrs; ++c) attrs[(size_t)o * n_attrs + c] = w.attrs[i * n_attrs + c];
  }
  if (i < n_live)
    for (int c = 0; c < 3; ++c) faces[3 * i + c] = w.foff[w.faces[3 * i + c]];
}

bool sizes_ok(int64_t n_verts, int64_t n_faces, int32_t n_attrs) {
  return n_verts >= 0 && n_verts <= INT32_MAX && n_faces >= 0 && n_faces <= kMaxFaces &&
         (n_verts > 0 || n_faces == 0) && n_attrs >= 0;
}

size_t take(char** p, size_t bytes) {
  const size_t a = align_up(bytes, 256);
  *p += a;
  return a;
}

// Layout (bytes): per vertex pos 12, attrs 4A, Q 80, ren 4, boundary and locked flags 2, claim 8, vstart 4 (+4);
// per face the live faces 12 and the dead flags 1; per half-edge entry (3 per face) the two sorts' keys and values in
// and out (8 + 8 + 4 + 4 and 4 + 4 + 4 + 4) and estart 4 (+4).  The sort inputs are dead once both sorts ran: the
// edge keys in hold the per-edge keys, the edge values in the scanned head flags, the vertex keys in the compacted
// faces and the vertex values in the face (emit: vertex) offsets.  So 110 + 4A B per vertex, 145 B per face, plus the
// largest cub scratch of the sorts and scans over 3F entries.
size_t carve(int64_t n_verts, int64_t n_faces, int32_t n_attrs, void* ws, Ws* out) {
  const int n3 = (int)(3 * n_faces), nv = (int)n_verts;
  size_t t_sort = 0, t_vsort = 0, t_scan = 0, t_vscan = 0;
  bool ok = true;
  if (n3 > 0) {
    ok = cub::DeviceRadixSort::SortPairs(nullptr, t_sort, (unsigned long long*)nullptr, (unsigned long long*)nullptr,
                                         (int*)nullptr, (int*)nullptr, n3) == cudaSuccess;
    ok = ok && cub::DeviceRadixSort::SortPairs(nullptr, t_vsort, (int*)nullptr, (int*)nullptr, (int*)nullptr,
                                               (int*)nullptr, n3) == cudaSuccess;
    ok = ok && cub::DeviceScan::InclusiveSum(nullptr, t_scan, (int*)nullptr, n3) == cudaSuccess;
  }
  if (nv > 0) ok = ok && cub::DeviceScan::ExclusiveSum(nullptr, t_vscan, (int*)nullptr, nv) == cudaSuccess;
  if (!ok) {
    cudaGetLastError();
    return 0;
  }
  size_t tmp = t_sort;
  for (size_t t : {t_vsort, t_scan, t_vscan}) tmp = t > tmp ? t : tmp;
  char* base = (char*)ws;
  char* p = base;
  const size_t V = (size_t)n_verts, F = (size_t)n_faces, H = 3 * F;
  Ws w;
  w.pos = (float*)p;                 take(&p, 12 * V);
  w.attrs = (float*)p;               take(&p, 4 * (size_t)n_attrs * V);
  w.q = (double*)p;                  take(&p, 80 * V);
  w.ren = (int*)p;                   take(&p, 4 * V);
  w.bnd = (uint8_t*)p;               take(&p, V);
  w.lock = (uint8_t*)p;              take(&p, V);
  w.claim = (unsigned long long*)p;  take(&p, 8 * V);
  w.vstart = (int*)p;                take(&p, 4 * (V + 1));
  w.faces = (int*)p;                 take(&p, 12 * F);
  w.dead = (uint8_t*)p;              take(&p, F);
  w.ekeys_in = (unsigned long long*)p;  take(&p, 8 * H);
  w.ekeys = (unsigned long long*)p;     take(&p, 8 * H);
  w.evals_in = (int*)p;              take(&p, 4 * H);
  w.evals = (int*)p;                 take(&p, 4 * H);
  w.vkeys_in = (int*)p;              take(&p, 4 * (H > V ? H : V));   // faces_tmp / vertex offsets
  w.vkeys = (int*)p;                 take(&p, 4 * H);
  w.vvals_in = (int*)p;              take(&p, 4 * (H > V ? H : V));   // face / vertex offsets
  w.vvals = (int*)p;                 take(&p, 4 * H);
  w.estart = (int*)p;                take(&p, 4 * (H + 1));
  w.sel = (unsigned long long*)p;    take(&p, 8 * 5);
  w.hist = (unsigned*)p;             take(&p, 4 * 256);
  w.tmp = p;
  w.tmp_bytes = tmp;
  w.ckey = w.ekeys_in;
  w.eid = w.evals_in;
  w.faces_tmp = w.vkeys_in;
  w.foff = w.vvals_in;
  if (out) *out = w;
  return (size_t)(p - base) + (tmp > 0 ? tmp : 1);
}

int check_ws(const char* what, int64_t n_verts, int64_t n_faces, int32_t n_attrs, void* ws, size_t ws_bytes, Ws* w) {
  SPARF_REQUIRE(ws, "%s: NULL workspace", what);
  const size_t need = carve(n_verts, n_faces, n_attrs, ws, w);
  if (need == 0) {
    set_error("%s: no current CUDA device to size the sort and scan scratch for", what);
    return SPARF_ERR_CUDA;
  }
  if (ws_bytes < need) {
    set_error("%s: workspace %zu B < %zu B", what, ws_bytes, need);
    return SPARF_ERR_WORKSPACE;
  }
  return SPARF_OK;
}

// the vertex CSR of the live faces (sorted vertex entries, vstart); build must have run
int vertex_csr(Ws& w, int n_live, int n_verts, int nb, cudaStream_t s) {
  size_t t = w.tmp_bytes;
  SPARF_CHECK_CUDA(cub::DeviceRadixSort::SortPairs(w.tmp, t, w.vkeys_in, w.vkeys, w.vvals_in, w.vvals, 3 * n_live, 0,
                                                   nb, s));
  ms_vstart_kernel<<<grid_of(n_verts + 1), kMsThreads, 0, s>>>(n_verts, 3 * n_live, w);
  SPARF_CHECK_LAUNCH("ms_vstart_kernel");
  return SPARF_OK;
}

#define SPARF_MS_REQUIRE_SIZES(what, V, F, A)                                                                       \
  SPARF_REQUIRE(sizes_ok(V, F, A), "%s: %lld vertices, %lld faces, %d attributes (V <= 2^31 - 1, F <= %lld, A >= 0; " \
                "faces need vertices)", what, (long long)(V), (long long)(F), (int)(A), (long long)kMaxFaces)

}  // namespace
}  // namespace sparf

using namespace sparf;

extern "C" size_t sparf_mesh_simplify_workspace_bytes(int64_t n_verts, int64_t n_faces, int32_t n_attrs) {
  return sizes_ok(n_verts, n_faces, n_attrs) ? carve(n_verts, n_faces, n_attrs, nullptr, nullptr) : 0;
}

extern "C" int sparf_mesh_simplify_init(const float* vertices, const int64_t* faces, const float* attrs,
                                        int64_t n_verts, int64_t n_faces, int32_t n_attrs, int64_t* counts,
                                        void* workspace, size_t workspace_bytes, sparf_stream_t stream) {
  SPARF_MS_REQUIRE_SIZES("mesh_simplify_init", n_verts, n_faces, n_attrs);
  SPARF_REQUIRE(counts && (n_verts == 0 || vertices) && (n_faces == 0 || faces) &&
                    (n_verts == 0 || n_attrs == 0 || attrs),
                "mesh_simplify_init: NULL pointer");
  cudaStream_t s = (cudaStream_t)stream;
  if (n_verts == 0) {
    SPARF_CHECK_CUDA(cudaMemsetAsync(counts, 0, 2 * sizeof(int64_t), s));
    return SPARF_OK;
  }
  Ws w;
  SPARF_TRY(check_ws("mesh_simplify_init", n_verts, n_faces, n_attrs, workspace, workspace_bytes, &w));
  const int V = (int)n_verts, F = (int)n_faces;
  SPARF_CHECK_CUDA(cudaMemcpyAsync(w.pos, vertices, 12 * (size_t)V, cudaMemcpyDeviceToDevice, s));
  if (n_attrs > 0)
    SPARF_CHECK_CUDA(cudaMemcpyAsync(w.attrs, attrs, 4 * (size_t)n_attrs * V, cudaMemcpyDeviceToDevice, s));
  ms_init_kernel<<<grid_of(3ll * F > V ? 3ll * F : V), kMsThreads, 0, s>>>(faces, F, V, w, counts);
  SPARF_CHECK_LAUNCH("ms_init_kernel");
  const int nb = id_bits(V);
  if (F > 0) {
    ms_build_kernel<<<grid_of(F), kMsThreads, 0, s>>>(F, nb, w);
    SPARF_CHECK_LAUNCH("ms_build_kernel");
    SPARF_TRY(vertex_csr(w, F, V, nb, s));
  } else {
    SPARF_CHECK_CUDA(cudaMemsetAsync(w.vstart, 0, 4 * ((size_t)V + 1), s));
  }
  ms_quadric_kernel<<<grid_of(V), kMsThreads, 0, s>>>(V, w);
  SPARF_CHECK_LAUNCH("ms_quadric_kernel");
  return SPARF_OK;
}

extern "C" int sparf_mesh_simplify_round(int64_t n_verts, int64_t n_faces, int32_t n_attrs, int64_t n_live, int64_t k,
                                         int64_t* counts, void* workspace, size_t workspace_bytes,
                                         sparf_stream_t stream) {
  SPARF_MS_REQUIRE_SIZES("mesh_simplify_round", n_verts, n_faces, n_attrs);
  SPARF_REQUIRE(n_live >= 0 && n_live <= n_faces && k >= 1, "mesh_simplify_round: %lld live faces of %lld, k = %lld",
                (long long)n_live, (long long)n_faces, (long long)k);
  SPARF_REQUIRE(counts, "mesh_simplify_round: NULL pointer");
  cudaStream_t s = (cudaStream_t)stream;
  if (n_live == 0) {
    SPARF_CHECK_CUDA(cudaMemsetAsync(counts, 0, 2 * sizeof(int64_t), s));
    return SPARF_OK;
  }
  Ws w;
  SPARF_TRY(check_ws("mesh_simplify_round", n_verts, n_faces, n_attrs, workspace, workspace_bytes, &w));
  const int V = (int)n_verts, n = (int)n_live, H = 3 * n, nb = id_bits(V);
  SPARF_CHECK_CUDA(cudaMemsetAsync(w.bnd, 0, (size_t)V, s));
  SPARF_CHECK_CUDA(cudaMemsetAsync(w.lock, 0, (size_t)V, s));
  SPARF_CHECK_CUDA(cudaMemsetAsync(w.claim, 0xff, 8 * (size_t)V, s));
  SPARF_CHECK_CUDA(cudaMemsetAsync(w.dead, 0, (size_t)n, s));
  ms_round_begin_kernel<<<1, 1, 0, s>>>(w, k, counts);
  SPARF_CHECK_LAUNCH("ms_round_begin_kernel");
  ms_build_kernel<<<grid_of(n), kMsThreads, 0, s>>>(n, nb, w);
  SPARF_CHECK_LAUNCH("ms_build_kernel");
  size_t t = w.tmp_bytes;
  SPARF_CHECK_CUDA(cub::DeviceRadixSort::SortPairs(w.tmp, t, w.ekeys_in, w.ekeys, w.evals_in, w.evals, H, 0, 2 * nb, s));
  SPARF_TRY(vertex_csr(w, n, V, nb, s));
  ms_head_kernel<<<grid_of(H), kMsThreads, 0, s>>>(H, w);
  SPARF_CHECK_LAUNCH("ms_head_kernel");
  t = w.tmp_bytes;
  SPARF_CHECK_CUDA(cub::DeviceScan::InclusiveSum(w.tmp, t, w.eid, w.eid, H, s));
  ms_edge_start_kernel<<<grid_of(H), kMsThreads, 0, s>>>(H, w);
  SPARF_CHECK_LAUNCH("ms_edge_start_kernel");
  // the kernels over edges run over H >= E threads and read E on the device
  ms_classify_kernel<<<grid_of(H), kMsThreads, 0, s>>>(nb, w);
  SPARF_CHECK_LAUNCH("ms_classify_kernel");
  ms_key_kernel<<<grid_of(H), kMsThreads, 0, s>>>(nb, w);
  SPARF_CHECK_LAUNCH("ms_key_kernel");
  const unsigned hist_grid = grid_of(H) < 1024 ? grid_of(H) : 1024;
  for (int pass = 0; pass < 8; ++pass) {
    ms_hist_kernel<<<hist_grid, kMsThreads, 0, s>>>(pass, w);
    SPARF_CHECK_LAUNCH("ms_hist_kernel");
    ms_pick_kernel<<<1, 1, 0, s>>>(pass, w);
    SPARF_CHECK_LAUNCH("ms_pick_kernel");
  }
  ms_claim_kernel<<<grid_of(H), kMsThreads, 0, s>>>(nb, w);
  SPARF_CHECK_LAUNCH("ms_claim_kernel");
  ms_win_kernel<<<grid_of(H), kMsThreads, 0, s>>>(nb, n_attrs, w, counts);
  SPARF_CHECK_LAUNCH("ms_win_kernel");
  ms_face_flag_kernel<<<grid_of(n), kMsThreads, 0, s>>>(n, w);
  SPARF_CHECK_LAUNCH("ms_face_flag_kernel");
  t = w.tmp_bytes;
  SPARF_CHECK_CUDA(cub::DeviceScan::ExclusiveSum(w.tmp, t, w.foff, w.foff, n, s));
  ms_face_emit_kernel<<<grid_of(n), kMsThreads, 0, s>>>(n, w, counts);
  SPARF_CHECK_LAUNCH("ms_face_emit_kernel");
  SPARF_CHECK_CUDA(cudaMemcpyAsync(w.faces, w.faces_tmp, 12 * (size_t)n, cudaMemcpyDeviceToDevice, s));
  return SPARF_OK;
}

extern "C" int sparf_mesh_simplify_emit(int64_t n_verts, int64_t n_faces, int32_t n_attrs, int64_t n_live,
                                        float* vertices, float* attrs, int64_t* vert_ids, int64_t* faces,
                                        void* workspace, size_t workspace_bytes, sparf_stream_t stream) {
  SPARF_MS_REQUIRE_SIZES("mesh_simplify_emit", n_verts, n_faces, n_attrs);
  SPARF_REQUIRE(n_live >= 0 && n_live <= n_faces, "mesh_simplify_emit: %lld live faces of %lld", (long long)n_live,
                (long long)n_faces);
  SPARF_REQUIRE((n_verts == 0 || (vertices && vert_ids && (n_attrs == 0 || attrs))) && (n_live == 0 || faces),
                "mesh_simplify_emit: NULL pointer");
  if (n_verts == 0) return SPARF_OK;
  Ws w;
  SPARF_TRY(check_ws("mesh_simplify_emit", n_verts, n_faces, n_attrs, workspace, workspace_bytes, &w));
  cudaStream_t s = (cudaStream_t)stream;
  const int V = (int)n_verts, n = (int)n_live;
  ms_vert_flag_kernel<<<grid_of(V), kMsThreads, 0, s>>>(V, w);
  SPARF_CHECK_LAUNCH("ms_vert_flag_kernel");
  size_t t = w.tmp_bytes;
  SPARF_CHECK_CUDA(cub::DeviceScan::ExclusiveSum(w.tmp, t, w.foff, w.foff, V, s));
  ms_emit_kernel<<<grid_of(V > n ? V : n), kMsThreads, 0, s>>>(V, n, n_attrs, w, vertices, attrs, vert_ids, faces);
  SPARF_CHECK_LAUNCH("ms_emit_kernel");
  return SPARF_OK;
}
