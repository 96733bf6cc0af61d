// Sparse marching cubes over 8^3-cell blocks of a [res+1]^3 lattice (include/sparf_b200.h, "sparse marching cubes"):
// the mesh of the dense extractor (mcubes.cu) restricted to the cells of the active blocks, without the dense volume.
//   classify: per block, its coarse window's verdict (flag); a device scan gives each active block its rank (slot);
//   blocks:   the active block ids in linear order, scattered from the slots;
//   points:   the 729 lattice points of a range of active blocks, gathered from the axis;
//   count:    one CTA per active block over its sigma [9][9][9]: the crossing edges it owns (a shared edge belongs to the
//             active block of smallest linear index that contains it, so every vertex is counted once) and per segment
//             (8 cells along k) the triangle count, written at the segment's place in global cell order; two scans;
//   emit:     the same pass writes owned vertices as (key (linear p) * 3 + a, position) and each segment's triangles,
//             over vertex keys, straight into their final rows; a radix sort of the keys gives the vertex order, and a
//             binary search turns each triangle's keys into vertex ids.
// No atomics decide any order; the output is deterministic.
#include <cub/block/block_scan.cuh>
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include "common.cuh"

namespace sparf {
namespace {

constexpr int kB = SPARF_MCUBES_BLOCK;            // cells per block edge
constexpr int kP = kB + 1;                          // lattice points per block edge
constexpr int kBlockPoints = kP * kP * kP;          // 729
constexpr int kCells = kB * kB * kB;                // 512: one thread per cell
constexpr int kSegs = kB * kB;                      // 64 segments (u, v) of kB cells along k
constexpr int kRow = 3 * SPARF_MCUBES_MAX_TRIS;
constexpr int kMaxRes = 8192;
constexpr int kFlat = 256;

__device__ const signed char kTableDev[256][kRow] = {
#include "mcubes_table.cuh"
};

bool res_ok(int32_t res) { return res >= kB && res <= kMaxRes && res % kB == 0; }

// ---------------------------------------------------------------- classification
__global__ void sparse_flag_kernel(const float* __restrict__ coarse, int nb, float iso, int* __restrict__ flag) {
  const long long b = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long nblocks = (long long)nb * nb * nb;
  if (b >= nblocks) return;
  const int bi = (int)(b / ((long long)nb * nb)), bj = (int)(b / nb % nb), bk = (int)(b % nb);
  const int n = nb + 1;
  bool in = false, out = false;
  for (int i = max(bi - 1, 0); i <= min(bi + 2, nb); ++i)
    for (int j = max(bj - 1, 0); j <= min(bj + 2, nb); ++j)
      for (int k = max(bk - 1, 0); k <= min(bk + 2, nb); ++k) {
        const float s = __ldg(coarse + ((long long)i * n + j) * n + k);
        if (s != s) {
          flag[b] = 1;
          return;
        }
        if (s >= iso) in = true;
        else out = true;
      }
  flag[b] = in && out;
}

// slots hold the exclusive scan of the flags: inactive blocks get -1; the last thread writes the active count
__global__ void sparse_slot_kernel(const int* __restrict__ flag, long long nblocks, int* __restrict__ slots,
                                   int64_t* __restrict__ n_active) {
  const long long b = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= nblocks) return;
  const int r = slots[b];
  if (b == nblocks - 1) *n_active = (int64_t)r + flag[b];
  if (!flag[b]) slots[b] = -1;
}

__global__ void sparse_blocks_kernel(const int* __restrict__ slots, long long nblocks, int64_t* __restrict__ block_ids) {
  const long long b = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (b < nblocks && slots[b] >= 0) block_ids[slots[b]] = b;
}

__global__ void sparse_points_kernel(const float* __restrict__ axis, int nb, const int64_t* __restrict__ block_ids,
                                     long long b0, long long npts, float* __restrict__ points) {
  const long long x = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (x >= npts) return;
  const long long b = block_ids[b0 + x / kBlockPoints];
  const int q = (int)(x % kBlockPoints);
  const long long bi = b / ((long long)nb * nb), bj = b / nb % nb, bk = b % nb;
  points[3 * x + 0] = __ldg(axis + kB * bi + q / (kP * kP));
  points[3 * x + 1] = __ldg(axis + kB * bj + q / kP % kP);
  points[3 * x + 2] = __ldg(axis + kB * bk + q % kP);
}

// ---------------------------------------------------------------- marching cubes over the blocks
struct Sparse {
  const float* sigma;         // [n_active][9][9][9]
  const int* slots;           // [nb^3]
  const int64_t* block_ids;   // [n_active]
  long long n_active;
  int nb;
  long long n;                // res + 1
  float iso;
};

struct Counts {
  int64_t *vcnt, *voff;       // [n_active]: owned vertices per block, their exclusive scan
  int64_t *scnt, *soff;       // [64 n_active] in global segment order: triangles per segment, their exclusive scan
  int64_t* totals;            // {V, F}
};

struct Emit {
  int64_t* keys;              // [max_verts] vertex keys of the owned vertices (unsorted); padded with 3 (res+1)^3, above every key
  int64_t* idx;               // [max_verts] 0, 1, 2, ...: the sort's payload
  float* pos;                 // [max_verts][3]
  int64_t* faces;             // [max_faces][3] vertex keys, then ids
  long long max_verts, max_faces;
};

__device__ __forceinline__ long long lower_bound(const int64_t* a, long long n, long long key) {
  long long lo = 0, hi = n;
  while (lo < hi) {
    const long long mid = (lo + hi) >> 1;
    if (a[mid] < key) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}

// the edge from local point (u, v, w) of block (bi, bj, bk) along axis a (inside the block) belongs to this block
// unless an active block of smaller linear index contains it too: one that differs by -1 on a non-a axis where the
// point is at local 0, or by +1 where it is at local kB, with a negative first nonzero difference
__device__ __forceinline__ bool owns_edge(const Sparse& S, const int blk[3], const int loc[3], int a) {
  int lo[3], hi[3];
#pragma unroll
  for (int x = 0; x < 3; ++x) {
    lo[x] = (x != a && loc[x] == 0 && blk[x] > 0) ? -1 : 0;
    hi[x] = (x != a && loc[x] == kB && blk[x] < S.nb - 1) ? 1 : 0;
  }
  for (int di = lo[0]; di <= hi[0]; ++di)
    for (int dj = lo[1]; dj <= hi[1]; ++dj)
      for (int dk = lo[2]; dk <= hi[2]; ++dk) {
        const int first = di ? di : (dj ? dj : dk);
        if (first >= 0) continue;
        const long long nbr = ((long long)(blk[0] + di) * S.nb + (blk[1] + dj)) * S.nb + (blk[2] + dk);
        if (__ldg(S.slots + nbr) >= 0) return false;
      }
  return true;
}

template <bool EMIT>
__global__ void __launch_bounds__(kCells) sparse_mc_kernel(Sparse S, Counts C, Emit E) {
  using BlockScan = cub::BlockScan<int, kCells>;
  __shared__ typename BlockScan::TempStorage scan_tmp;
  __shared__ float s[kBlockPoints];
  __shared__ unsigned char ntri[256];
  __shared__ long long span[4];      // P0, NP, R0, NR: first index and count of the block's plane and row
  const long long r = blockIdx.x;
  const long long b = S.block_ids[r];
  const long long nb = S.nb;
  const int blk[3] = {(int)(b / (nb * nb)), (int)(b / nb % nb), (int)(b % nb)};
  const float* sig = S.sigma + r * kBlockPoints;
  for (int q = threadIdx.x; q < kBlockPoints; q += kCells) s[q] = __ldg(sig + q);
  if (threadIdx.x < 256) {
    int n = 0;
    while (n < SPARF_MCUBES_MAX_TRIS && kTableDev[threadIdx.x][3 * n] >= 0) ++n;
    ntri[threadIdx.x] = (unsigned char)n;
  }
  if (threadIdx.x == 0) {
    const long long plane = blk[0] * nb * nb, row = plane + blk[1] * nb;
    const long long p0 = lower_bound(S.block_ids, S.n_active, plane);
    const long long r0 = lower_bound(S.block_ids, S.n_active, row);
    span[0] = p0;
    span[1] = lower_bound(S.block_ids, S.n_active, plane + nb * nb) - p0;
    span[2] = r0;
    span[3] = lower_bound(S.block_ids, S.n_active, row + nb) - r0;
  }
  __syncthreads();

  // vertices: points q = tid and tid + kCells, a 3-bit mask of owned crossing edges each
  int mask[2] = {0, 0};
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int q = threadIdx.x + h * kCells;
    if (q >= kBlockPoints) continue;
    const int loc[3] = {q / (kP * kP), q / kP % kP, q % kP};
    const bool in0 = s[q] >= S.iso;
    const int stride[3] = {kP * kP, kP, 1};
#pragma unroll
    for (int a = 0; a < 3; ++a)
      if (loc[a] < kB && (s[q + stride[a]] >= S.iso) != in0 && owns_edge(S, blk, loc, a)) mask[h] |= 1 << a;
  }
  int nv = __popc(mask[0]) + __popc(mask[1]), vex, vtot;
  BlockScan(scan_tmp).ExclusiveSum(nv, vex, vtot);

  // cells: thread = (u, v, w), w fastest, so a segment (u, v) is 8 consecutive lanes
  const int cu = threadIdx.x >> 6, cv = (threadIdx.x >> 3) & 7, cw = threadIdx.x & 7;
  const int c0 = (cu * kP + cv) * kP + cw;
  int cs = 0;
#pragma unroll
  for (int q = 0; q < 8; ++q) cs |= (int)(s[c0 + (q & 1) * kP * kP + ((q >> 1) & 1) * kP + ((q >> 2) & 1)] >= S.iso) << q;
  const int nt = ntri[cs];
  int incl = nt;
#pragma unroll
  for (int d = 1; d < kB; d <<= 1) {
    const int y = __shfl_up_sync(0xffffffffu, incl, d, kB);
    if (cw >= d) incl += y;
  }
  const int seg_total = __shfl_sync(0xffffffffu, incl, kB - 1, kB);
  // global cell order is (i, j, k): by plane bi, then u, then row bj, then v, then bk
  const long long P0 = span[0], NP = span[1], R0 = span[2], NR = span[3];
  const long long seg = kSegs * P0 + cu * kB * NP + kB * (R0 - P0) + cv * NR + (r - R0);

  if constexpr (!EMIT) {
    if (threadIdx.x == 0) C.vcnt[r] = vtot;
    if (cw == 0) C.scnt[seg] = seg_total;
  } else {
    // owned vertices at their block offset, positions as the dense extractor computes them
    long long id = C.voff[r] + vex;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int q = threadIdx.x + h * kCells;
      if (!mask[h]) continue;
      const long long p[3] = {kB * blk[0] + q / (kP * kP), kB * blk[1] + q / kP % kP, kB * blk[2] + q % kP};
      const long long lin = (p[0] * S.n + p[1]) * S.n + p[2];
      const float v0 = s[q];
      const int stride[3] = {kP * kP, kP, 1};
#pragma unroll
      for (int a = 0; a < 3; ++a) {
        if (!(mask[h] >> a & 1)) continue;
        const float sa = __fdiv_rn(__fsub_rn(S.iso, v0), __fsub_rn(s[q + stride[a]], v0));
        if (id < E.max_verts) {
          E.keys[id] = lin * 3 + a;
          float* o = E.pos + 3 * id;
          o[0] = a == 0 ? __fadd_rn((float)p[0], sa) : (float)p[0];
          o[1] = a == 1 ? __fadd_rn((float)p[1], sa) : (float)p[1];
          o[2] = a == 2 ? __fadd_rn((float)p[2], sa) : (float)p[2];
        }
        ++id;
      }
    }
    // this cell's triangles over vertex keys, at the segment's offset + the earlier cells' triangles
    long long f = C.soff[seg] + (incl - nt);
    const long long ci = kB * blk[0] + cu, cj = kB * blk[1] + cv, ck = kB * blk[2] + cw;
    for (int t = 0; t < nt; ++t, ++f) {
      if (f >= E.max_faces) break;
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        // edge e = 4a + m: along axis a from the corner whose offsets on the other two axes b < b' are (m & 1, m >> 1)
        const int e = kTableDev[cs][3 * t + c], a = e >> 2, m = e & 3;
        const int oi = a == 0 ? 0 : (m & 1), oj = a == 1 ? 0 : (a == 0 ? (m & 1) : (m >> 1)), ok = a == 2 ? 0 : (m >> 1);
        E.faces[3 * f + c] = (((ci + oi) * S.n + (cj + oj)) * S.n + (ck + ok)) * 3 + a;
      }
    }
  }
}

__global__ void sparse_totals_kernel(Counts C, long long n_active) {
  const long long last = n_active - 1, slast = kSegs * n_active - 1;
  C.totals[0] = C.voff[last] + C.vcnt[last];
  C.totals[1] = C.soff[slast] + C.scnt[slast];
}

// keys past V get the padding key (above every real key) so that the sort leaves them at the end
__global__ void sparse_pad_kernel(int64_t* __restrict__ keys, int64_t* __restrict__ idx, long long max_verts,
                                  const int64_t* __restrict__ totals, long long pad) {
  const long long x = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (x >= max_verts) return;
  idx[x] = x;
  if (x >= totals[0]) keys[x] = pad;
}

__global__ void sparse_gather_kernel(const int64_t* __restrict__ idx, const float* __restrict__ pos,
                                     const int64_t* __restrict__ totals, long long max_verts, float* __restrict__ verts) {
  const long long x = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (x >= max_verts || x >= totals[0]) return;
  const long long i = idx[x];
  verts[3 * x + 0] = pos[3 * i + 0];
  verts[3 * x + 1] = pos[3 * i + 1];
  verts[3 * x + 2] = pos[3 * i + 2];
}

__global__ void sparse_ids_kernel(const int64_t* __restrict__ sorted_keys, const int64_t* __restrict__ totals,
                                  long long max_verts, long long max_faces, int64_t* __restrict__ faces) {
  const long long x = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long F = min((long long)totals[1], max_faces);
  if (x >= 3 * F) return;
  faces[x] = lower_bound(sorted_keys, min((long long)totals[0], max_verts), faces[x]);
}

// ---------------------------------------------------------------- workspace
int key_bits(int32_t res) {
  const long long n = res + 1;
  const long long pad = n * n * n * 3;    // one past the largest key
  int bits = 1;
  while (bits < 63 && (pad >> bits)) ++bits;
  return bits;
}

struct Carve {
  int* flag;                 // classification: [nb^3]
  void* tmp;                 // device-wide scan / sort scratch
  size_t tmp_bytes;
  Counts C;
  Emit E;
  int64_t *keys_out, *idx_out;
};

// layout: counts (n_active), sort buffers (max_verts), then scratch; classification's flags share offset 0 with the
// counts, and the scratch starts after the larger of the two
size_t carve(int32_t res, long long n_active, long long max_verts, void* ws, Carve* c) {
  const long long nb = res / kB, nblocks = nb * nb * nb;
  CubScratch tmp;
  tmp.add([&](size_t& b) {
    return cub::DeviceScan::ExclusiveSum(nullptr, b, (const int*)nullptr, (int*)nullptr, (int)nblocks);
  });
  if (n_active > 0) {
    tmp.add([&](size_t& b) {
      return cub::DeviceScan::ExclusiveSum(nullptr, b, (const int64_t*)nullptr, (int64_t*)nullptr, (int)n_active);
    });
    tmp.add([&](size_t& b) {
      return cub::DeviceScan::ExclusiveSum(nullptr, b, (const int64_t*)nullptr, (int64_t*)nullptr,
                                           (int)(kSegs * n_active));
    });
  }
  if (max_verts > 0)
    tmp.add([&](size_t& b) {
      return cub::DeviceRadixSort::SortPairs(nullptr, b, (const int64_t*)nullptr, (int64_t*)nullptr,
                                             (const int64_t*)nullptr, (int64_t*)nullptr, (int)max_verts, 0,
                                             key_bits(res));
    });
  if (!tmp.ok) return 0;
  Carve k{};
  WsCarver cls(ws), w(ws);
  k.flag = cls.take<int>(nblocks);
  k.C.vcnt = w.take<int64_t>(n_active);
  k.C.voff = w.take<int64_t>(n_active);
  k.C.scnt = w.take<int64_t>(kSegs * n_active);
  k.C.soff = w.take<int64_t>(kSegs * n_active);
  k.C.totals = w.take<int64_t>(2);
  k.E.keys = w.take<int64_t>(max_verts);
  k.keys_out = w.take<int64_t>(max_verts);
  k.E.idx = w.take<int64_t>(max_verts);
  k.idx_out = w.take<int64_t>(max_verts);
  k.E.pos = w.take<float>(3 * max_verts);
  k.E.max_verts = max_verts;
  w.end = w.end > cls.end ? w.end : cls.end;
  k.tmp_bytes = tmp.bytes;
  k.tmp = w.take<char>(tmp.bytes);
  if (c) *c = k;
  return w.end;
}

// every scanned or sorted length fits cub's int item count
bool sizes_ok(int32_t res, int64_t n_active, int64_t max_verts) {
  if (!res_ok(res)) return false;
  const long long nb = res / kB;
  return n_active >= 0 && n_active <= nb * nb * nb && kSegs * n_active < (1ll << 31) && max_verts >= 0 &&
         max_verts < (1ll << 31);
}

// count and emit share this: the per-block pass and the two scans
int count_pass(const Sparse& S, const Carve& c, cudaStream_t s) {
  sparse_mc_kernel<false><<<(unsigned)S.n_active, kCells, 0, s>>>(S, c.C, c.E);
  SPARF_CHECK_LAUNCH("sparse_mc_kernel<count>");
  size_t t = c.tmp_bytes;
  SPARF_CHECK_CUDA(cub::DeviceScan::ExclusiveSum(c.tmp, t, c.C.vcnt, c.C.voff, (int)S.n_active, s));
  t = c.tmp_bytes;
  SPARF_CHECK_CUDA(cub::DeviceScan::ExclusiveSum(c.tmp, t, c.C.scnt, c.C.soff, (int)(kSegs * S.n_active), s));
  sparse_totals_kernel<<<1, 1, 0, s>>>(c.C, S.n_active);
  SPARF_CHECK_LAUNCH("sparse_totals_kernel");
  return SPARF_OK;
}

}  // namespace
}  // namespace sparf

using namespace sparf;

extern "C" size_t sparf_mcubes_sparse_workspace_bytes(int32_t res, int64_t n_active, int64_t max_verts) {
  return sizes_ok(res, n_active, max_verts) ? carve(res, n_active, max_verts, nullptr, nullptr) : 0;
}

extern "C" int sparf_mcubes_sparse_classify(const float* coarse, int32_t res, float iso, int32_t* slots,
                                            int64_t* n_active, void* workspace, size_t workspace_bytes,
                                            sparf_stream_t stream) {
  SPARF_REQUIRE(res_ok(res), "mcubes_sparse_classify: res %d (a multiple of %d in [%d, %d])", res, kB, kB, kMaxRes);
  SPARF_REQUIRE(coarse && slots && n_active && workspace, "mcubes_sparse_classify: NULL pointer");
  Carve c;
  SPARF_TRY(check_workspace("mcubes_sparse_classify", workspace, workspace_bytes, carve(res, 0, 0, workspace, &c)));
  cudaStream_t s = (cudaStream_t)stream;
  const int nb = res / kB;
  const long long nblocks = (long long)nb * nb * nb;
  sparse_flag_kernel<<<grid_of(nblocks, kFlat), kFlat, 0, s>>>(coarse, nb, iso, c.flag);
  SPARF_CHECK_LAUNCH("sparse_flag_kernel");
  size_t t = c.tmp_bytes;
  SPARF_CHECK_CUDA(cub::DeviceScan::ExclusiveSum(c.tmp, t, c.flag, slots, (int)nblocks, s));
  sparse_slot_kernel<<<grid_of(nblocks, kFlat), kFlat, 0, s>>>(c.flag, nblocks, slots, n_active);
  SPARF_CHECK_LAUNCH("sparse_slot_kernel");
  return SPARF_OK;
}

extern "C" int sparf_mcubes_sparse_blocks(const int32_t* slots, int32_t res, int64_t* block_ids, sparf_stream_t stream) {
  SPARF_REQUIRE(res_ok(res), "mcubes_sparse_blocks: res %d (a multiple of %d in [%d, %d])", res, kB, kB, kMaxRes);
  SPARF_REQUIRE(slots && block_ids, "mcubes_sparse_blocks: NULL pointer");
  const long long nb = res / kB, nblocks = nb * nb * nb;
  sparse_blocks_kernel<<<grid_of(nblocks, kFlat), kFlat, 0, (cudaStream_t)stream>>>(slots, nblocks, block_ids);
  SPARF_CHECK_LAUNCH("sparse_blocks_kernel");
  return SPARF_OK;
}

extern "C" int sparf_mcubes_sparse_points(const float* axis, int32_t res, const int64_t* block_ids, int64_t b0,
                                          int64_t n_blocks, float* points, sparf_stream_t stream) {
  SPARF_REQUIRE(res_ok(res), "mcubes_sparse_points: res %d (a multiple of %d in [%d, %d])", res, kB, kB, kMaxRes);
  SPARF_REQUIRE(b0 >= 0 && n_blocks >= 0, "mcubes_sparse_points: blocks [%lld, +%lld)", (long long)b0,
                (long long)n_blocks);
  if (n_blocks == 0) return SPARF_OK;
  SPARF_REQUIRE(axis && block_ids && points, "mcubes_sparse_points: NULL pointer");
  const long long npts = (long long)n_blocks * kBlockPoints;
  sparse_points_kernel<<<grid_of(npts, kFlat), kFlat, 0, (cudaStream_t)stream>>>(axis, res / kB, block_ids, b0, npts,
                                                                                points);
  SPARF_CHECK_LAUNCH("sparse_points_kernel");
  return SPARF_OK;
}

extern "C" int sparf_mcubes_sparse_count(const float* sigma_blocks, int32_t res, const int32_t* slots,
                                         const int64_t* block_ids, int64_t n_active, float iso, int64_t* totals,
                                         void* workspace, size_t workspace_bytes, sparf_stream_t stream) {
  SPARF_REQUIRE(sizes_ok(res, n_active, 0), "mcubes_sparse_count: res %d, %lld active blocks", res, (long long)n_active);
  SPARF_REQUIRE(totals && workspace, "mcubes_sparse_count: NULL pointer");
  cudaStream_t s = (cudaStream_t)stream;
  if (n_active == 0) {
    SPARF_CHECK_CUDA(cudaMemsetAsync(totals, 0, 2 * sizeof(int64_t), s));
    return SPARF_OK;
  }
  SPARF_REQUIRE(sigma_blocks && slots && block_ids, "mcubes_sparse_count: NULL pointer");
  Carve c;
  SPARF_TRY(check_workspace("mcubes_sparse_count", workspace, workspace_bytes, carve(res, n_active, 0, workspace, &c)));
  const Sparse S{sigma_blocks, slots, block_ids, n_active, res / kB, res + 1, iso};
  c.C.totals = totals;
  return count_pass(S, c, s);
}

extern "C" int sparf_mcubes_sparse_emit(const float* sigma_blocks, int32_t res, const int32_t* slots,
                                        const int64_t* block_ids, int64_t n_active, float iso, int64_t max_verts,
                                        int64_t max_faces, float* verts, int64_t* faces, void* workspace,
                                        size_t workspace_bytes, sparf_stream_t stream) {
  // a block has at most kCells * SPARF_MCUBES_MAX_TRIS triangles: a larger capacity is a caller's error
  SPARF_REQUIRE(sizes_ok(res, n_active, max_verts) && max_faces >= 0 &&
                    max_faces <= (long long)kCells * SPARF_MCUBES_MAX_TRIS * n_active,
                "mcubes_sparse_emit: res %d, %lld active blocks, capacity %lld vertices / %lld faces", res,
                (long long)n_active, (long long)max_verts, (long long)max_faces);
  if (n_active == 0) return SPARF_OK;
  SPARF_REQUIRE(sigma_blocks && slots && block_ids && workspace && (verts || !max_verts) && (faces || !max_faces),
                "mcubes_sparse_emit: NULL pointer");
  Carve c;
  SPARF_TRY(check_workspace("mcubes_sparse_emit", workspace, workspace_bytes,
                            carve(res, n_active, max_verts, workspace, &c)));
  cudaStream_t s = (cudaStream_t)stream;
  const Sparse S{sigma_blocks, slots, block_ids, n_active, res / kB, res + 1, iso};
  SPARF_TRY(count_pass(S, c, s));
  c.E.faces = faces;
  c.E.max_faces = max_faces;
  sparse_mc_kernel<true><<<(unsigned)n_active, kCells, 0, s>>>(S, c.C, c.E);
  SPARF_CHECK_LAUNCH("sparse_mc_kernel<emit>");
  if (max_verts > 0) {
    const long long n = res + 1;
    sparse_pad_kernel<<<grid_of(max_verts, kFlat), kFlat, 0, s>>>(c.E.keys, c.E.idx, max_verts, c.C.totals, n * n * n * 3);
    SPARF_CHECK_LAUNCH("sparse_pad_kernel");
    size_t t = c.tmp_bytes;
    SPARF_CHECK_CUDA(cub::DeviceRadixSort::SortPairs(c.tmp, t, c.E.keys, c.keys_out, c.E.idx, c.idx_out, (int)max_verts,
                                                     0, key_bits(res), s));
    sparse_gather_kernel<<<grid_of(max_verts, kFlat), kFlat, 0, s>>>(c.idx_out, c.E.pos, c.C.totals, max_verts, verts);
    SPARF_CHECK_LAUNCH("sparse_gather_kernel");
  }
  if (max_faces > 0) {
    sparse_ids_kernel<<<grid_of(3 * max_faces, kFlat), kFlat, 0, s>>>(c.keys_out, c.C.totals, max_verts, max_faces,
                                                                       faces);
    SPARF_CHECK_LAUNCH("sparse_ids_kernel");
  }
  return SPARF_OK;
}
