// wgmma GEMMs of the tensor-core MLP engines (SPARF_ENGINE_TC_3X / TC_1X / TC_3X_W1), sm_90a.
//
// The GEMMs read both operands as images: 16-bit (hi, lo) halves in [128 rows x 32 K] tiles, each tile already in the
// canonical no-swizzle K-major shared-memory layout (8 x 8 core matrices of 128 contiguous bytes, core matrices adjacent
// in K 128 B apart = leading byte offset, 8-row groups 512 B apart = stride byte offset), hi and lo halves of a tile
// adjacent (16 KB).
//   pack: splits an fp32 operand (with the GEMM's own indexing: transposes, per-ray rows, bounds) into an image; the
//     weights and the encodings take this path;
//   head backward: the colour head's narrow layer, whose gradient it writes straight into its two images;
//   feature backward: the last trunk layer's gradient of a density query, (feat > 0) * d_feat, likewise;
//   gemm: persistent, one CTA per SM walking 128 x 128 output tiles (the weight gradient: tiles x k-ranges).  A
//     producer thread streams the tiles of both operands with cp.async.bulk into a STAGES-deep ring of shared-memory
//     stages that runs on across tiles, each stage completing on its "full" mbarrier (complete_tx); two consumer
//     warpgroups wait on it, issue wgmma.m64n128k16 (register accumulators) and hand the stage back on its "empty"
//     mbarrier once the MMAs that read it have retired.  So the next tile's first stages load during an epilogue.  The
//     epilogue can write the output's own images (row and transposed) for the next GEMMs, so trunk activations and
//     gradients are never packed from fp32;
//   staged weight-gradient gemm: the same walk, ring and MMAs, with B read as fp32 rows by bulk copies and split in
//     shared memory by a fourth (converter) warpgroup, so the weight gradient's activation operand is never packed.
//   trunk chain: the trunk forward at width 256 in one persistent kernel.  A tile of 128 rows goes through every layer
//     with its activations in shared memory (each layer's epilogue splits its output over its input), each consumer
//     warpgroup on its own 64 rows, a quarter of the columns at a time; only the weights stream through the ring, one
//     stage feeding both warpgroups, and global memory gets the fp32 activations that are asked for and the last
//     layer's row image.  Same MMA order and epilogue arithmetic per output element as the gemm, so the same bytes.
#include <cuda_bf16.h>
#include <cudaTypedefs.h>
#include <cuda_fp16.h>

#include <algorithm>
#include <type_traits>

#include "gemm_wgmma.cuh"

namespace sparf {
namespace {

constexpr int TM = 128, TN = 128, TK = 32;
constexpr int TILE_ELEMS = TM * TK;          // one [128 x 32] 16-bit operand tile, 8 KB

struct __align__(128) WgSmem {
  uint16_t a[2][TILE_ELEMS];   // hi, lo
  uint16_t b[2][TILE_ELEMS];
};

__device__ __forceinline__ int sw_off(int r, int k) { return (((r >> 3) * (TK / 8) + (k >> 3)) << 6) + ((r & 7) << 3) + (k & 7); }

__device__ __forceinline__ uint64_t smem_desc(const void* p) {
  uint32_t a = static_cast<uint32_t>(__cvta_generic_to_shared(p));
  uint64_t d = (uint64_t)((a & 0x3FFFF) >> 4);
  d |= (uint64_t)(128 >> 4) << 16;            // leading byte offset: next core matrix along K
  d |= (uint64_t)(512 >> 4) << 32;            // stride byte offset: next 8-row group
  return d;                                   // base offset 0, no swizzle
}

#define SPARF_WG_D64                                                                                                        \
  "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),   \
      "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]),  \
      "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]),  \
      "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]),  \
      "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]),  \
      "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]),  \
      "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
#define SPARF_WG_REGS                                                                                                       \
  "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31," \
  "%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,"    \
  "%61,%62,%63}"

// D[64 x 128] += A[64 x 16] B[128 x 16]^T, both K-major in shared memory
template <bool F16>
__device__ __forceinline__ void wgmma_m64n128k16(float (&d)[64], uint64_t da, uint64_t db) {
  if constexpr (F16) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 " SPARF_WG_REGS ", %64, %65, p, 1, 1, 0, 0;\n}\n"
                 : SPARF_WG_D64
                 : "l"(da), "l"(db), "r"(1));
  } else {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 " SPARF_WG_REGS ", %64, %65, p, 1, 1, 0, 0;\n}\n"
                 : SPARF_WG_D64
                 : "l"(da), "l"(db), "r"(1));
  }
}

#define SPARF_WG_D32                                                                                                        \
  "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),   \
      "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]),  \
      "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]),  \
      "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
#define SPARF_WG_REGS32                                                                                                     \
  "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}"

// D[64 x 64] += A[64 x 16] B[64 x 16]^T, both K-major in shared memory (the fused trunk chains' column quarters)
template <bool F16>
__device__ __forceinline__ void wgmma_m64n64k16(float (&d)[32], uint64_t da, uint64_t db) {
  if constexpr (F16) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 " SPARF_WG_REGS32 ", %32, %33, p, 1, 1, 0, 0;\n}\n"
                 : SPARF_WG_D32
                 : "l"(da), "l"(db), "r"(1));
  } else {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 " SPARF_WG_REGS32 ", %32, %33, p, 1, 1, 0, 0;\n}\n"
                 : SPARF_WG_D32
                 : "l"(da), "l"(db), "r"(1));
  }
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;\n" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;\n" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;\n" ::: "memory"); }

// the lo halves are stored scaled by 2^LO_SHIFT (exact) so that they stay clear of the fp16 subnormal range; the products
// that carry one lo factor accumulate separately and are scaled back once at the end
constexpr int LO_SHIFT = 11;

// x 2^-LO_SHIFT, rounded once as ldexpf(x, -LO_SHIFT) is (exact unless the result is subnormal); __fmul_rn keeps the
// multiply out of an FMA with the add that follows it, which would skip that rounding
__device__ __forceinline__ float lo_unscale(float x) { return __fmul_rn(x, 1.f / (1 << LO_SHIFT)); }

template <bool F16>
__device__ __forceinline__ void split16(float x, uint16_t& hi, uint16_t& lo) {
  if constexpr (F16) {
    __half h = __float2half_rn(x);
    __half l = __float2half_rn(ldexpf(x - __half2float(h), LO_SHIFT));
    hi = __half_as_ushort(h);
    lo = __half_as_ushort(l);
  } else {
    __nv_bfloat16 h = __float2bfloat16_rn(x);
    __nv_bfloat16 l = __float2bfloat16_rn(ldexpf(x - __bfloat162float(h), LO_SHIFT));
    hi = __bfloat16_as_ushort(h);
    lo = __bfloat16_as_ushort(l);
  }
}

constexpr int TILE_BYTES = TILE_ELEMS * 2;        // one 16-bit half of a tile
constexpr int STAGES = 6;
constexpr int STAGE_BYTES = 4 * TILE_BYTES;       // A hi, A lo, B hi, B lo
constexpr int CONSUMERS = 256;                    // two MMA warpgroups (warps 0-7)
constexpr int GEMM_THREADS = CONSUMERS + 128;     // + the producer warpgroup (one thread issues the copies)
constexpr int RED_BYTES = 8 * TN * 4;             // column-sum reduction, [8 warps][128 columns] fp32
constexpr int GEMM_SMEM = STAGES * STAGE_BYTES + RED_BYTES + 2 * STAGES * 8;

// element i of this thread's share of a [128 x 32] tile: KFAST = consecutive threads along K (operand contiguous in K
// in global memory), else consecutive threads along the 128 rows
template <bool KFAST>
__device__ __forceinline__ void tile_pos(int i, int& r, int& k) {
  const int idx = threadIdx.x + 256 * i;
  if (KFAST) { r = idx >> 5; k = idx & 31; }
  else { r = idx & 127; k = idx >> 7; }
}

// ---- operand views: f(k-step, row, k within the step) -> fp32 element (0 outside the operand)
struct Rows {   // X[m / div][k]
  const float* X;
  int ldx, K, div, M;
  __device__ float operator()(int kt, int m, int kk) const {
    const int k = kt * TK + kk;
    return (m < M && k < K) ? X[(size_t)(m / div) * ldx + k] : 0.f;
  }
};
struct NtB {    // W[n][k] (first source), W[n][wcol2 + k] (second source)
  const float* W;
  int ldw, wcol2, K1v, K2v, N, s1;
  __device__ float operator()(int kt, int n, int kk) const {
    const bool two = kt >= s1;
    const int k = (two ? kt - s1 : kt) * TK + kk;
    if (n >= N || k >= (two ? K2v : K1v)) return 0.f;
    return W[(size_t)n * ldw + (two ? wcol2 : 0) + k];
  }
};
struct NnB {    // W[n][wcol + k] as rows k, contraction over n
  const float* W;
  int ldw, wcol, Kv, N;
  __device__ float operator()(int kt, int k, int nn) const {
    const int n = kt * TK + nn;
    return (n < N && k < Kv) ? W[(size_t)n * ldw + wcol + k] : 0.f;
  }
};
struct Cols {   // X[m][n] as rows n, contraction over m
  const float* X;
  int ldx, M, N;
  __device__ float operator()(int kt, int n, int mm) const {
    const int m = kt * TK + mm;
    return (m < M && n < N) ? X[(size_t)m * ldx + n] : 0.f;
  }
};
// X[m / div][k] as rows k, contraction over m.  bits (may be NULL): pack_kernel also writes bits[m][k >> 5] bit k & 31
// = X[m / div][k] > 0 (kw = ceil(K / 32) words per row), the ReLU mask of the same layer's input gradient.
struct TnB {
  const float* X;
  int ldx, div, M, K;
  uint32_t* bits;
  int kw;
  __device__ float operator()(int kt, int k, int mm) const {
    const int m = kt * TK + mm;
    return (m < M && k < K) ? X[(size_t)(m / div) * ldx + k] : 0.f;
  }
};

// image tile (row tile rt, k-step kt) at ((rt * ksteps + kt) * 2 + half) * TILE_ELEMS.  Loads follow the operand's
// contiguous dimension (KFAST); the split tile is assembled in shared memory and leaves in 16-byte vectors.
// DYN (Rows only): f.M is a capacity, of which live_rows rows are packed; row tiles past them are not written.  f.X's
// rows start at row_start (the span forward's global rows); the image's at 0.
// QUARTERS (the fused trunk chains' weight images): the image is laid out per 64-row quarter instead, 4 KB [64 x 32]
// blocks at ((quarter * ksteps + kt) * PASSES' halves + half) * 2048 elements, so that a quarter's k-steps are contiguous.
template <bool F16, int PASSES, bool KFAST, class F, bool DYN = false, bool QUARTERS = false>
__global__ void __launch_bounds__(256) pack_kernel(F f, int ksteps, uint16_t* __restrict__ img, RowCount rc) {
  __shared__ __align__(16) uint16_t t[2 * TILE_ELEMS];
  const int kt = blockIdx.x, rt = blockIdx.y;
  if constexpr (DYN) {
    f.M = (int)live_rows<true>(f.M, rc);
    if (rt * TM >= f.M) return;
    f.X += row_start<true>(rc) * f.ldx;
  }
  float v[16];
#pragma unroll
  for (int i = 0; i < 16; ++i) {     // all loads first
    int r, k;
    tile_pos<KFAST>(i, r, k);
    v[i] = f(kt, rt * TM + r, k);
  }
  if constexpr (std::is_same<F, TnB>::value) {
    // warp w holds rows r = 32 (w % 4) + lane (one bit word) of k-columns mm = w / 4 + 2 i: a ballot per i makes word
    // (m = kt * 32 + mm, rt * 4 + w % 4), which lane i stores; every word is written by one block
    if (f.bits) {
      const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
      uint32_t word = 0;
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        const uint32_t b = __ballot_sync(0xffffffffu, v[i] > 0.f);
        if (lane == i) word = b;
      }
      const int m = kt * TK + (w >> 2) + 2 * lane, c = rt * (TM / 32) + (w & 3);
      if (lane < 16 && m < f.M && c < f.kw) f.bits[(size_t)m * f.kw + c] = word;
    }
  }
#pragma unroll
  for (int i = 0; i < 16; ++i) {
    int r, k;
    tile_pos<KFAST>(i, r, k);
    uint16_t hi, lo;
    split16<F16>(v[i], hi, lo);
    const int o = sw_off(r, k);
    t[o] = hi;
    if (PASSES == 3) t[TILE_ELEMS + o] = lo;
  }
  __syncthreads();
  const uint4* src = reinterpret_cast<const uint4*>(t);
  constexpr int HB = PASSES == 3 ? 2 : 1;
  constexpr int NV = HB * TILE_ELEMS * 2 / 16;
  if constexpr (QUARTERS) {
    constexpr int QV = TILE_ELEMS / 16;     // 16-byte vectors of a [64 x 32] half: rows 0-63 of a tile half come first
    uint4* dst = reinterpret_cast<uint4*>(img);
#pragma unroll
    for (int i = threadIdx.x; i < NV; i += 256) {
      const int h = i / (2 * QV), v = i % (2 * QV);
      dst[(((size_t)(2 * rt + v / QV) * ksteps + kt) * HB + h) * QV + v % QV] = src[i];
    }
  } else {
    uint4* dst = reinterpret_cast<uint4*>(img + ((size_t)rt * ksteps + kt) * 2 * TILE_ELEMS);
#pragma unroll
    for (int i = threadIdx.x; i < NV; i += 256) dst[i] = src[i];
  }
}

// The colour-head backward of the tensor-core engines, one CTA per 128-row tile (rows m0 + r):
//   gpre[m][j] = d_rgb[m][j] c (1 - c), c = rgb[m][j];  graw[m] = d_sigma[m] softplus'(raw[m])      (as head_grad_kernel)
//   Ghid[m][n] = (hid[m][n] > 0) * sum_j gpre[m][j] W9[j][n]                                          (as narrow_dgrad_kernel)
// Ghid never goes to HBM in fp32: it leaves as its row image (dgrad passes) and its transposed image (wgrad passes),
// split from the same fp32 values as pack_kernel would split them, zero past M and HW.  Per CTA, one atomic per output:
// db_hid += the column sums of Ghid, dW9[j] += gpre_j^T hid, db9[j] += sum gpre_j, db_raw += sum graw.
struct HeadBwd {
  int M, HW;
  const float *d_rgb, *rgb, *d_sigma, *raw, *hid, *W9;
  float* graw;
  uint16_t *row, *tr;       // images, row_ks = ceil(HW / 32) and tr_ks = ceil(M / 32) k-steps per row tile
  int row_ks, tr_ks;
  float *dW9, *db9, *db_hid, *db_raw;
};

constexpr int HB_LD = TN + 1;       // Ghid tile in shared memory, [128 rows][128 columns + 1]: conflict-free both ways
constexpr int HEAD_SMEM = (TM * HB_LD + 8 * 16 * 32 + TM * 4 + 3 * TN + 4 * 4) * 4;

// eight consecutive k of one image row -> their bf16 hi halves and lo halves, 16 bytes each
__device__ __forceinline__ void split8(const float (&v)[8], uint4& hi, uint4& lo) {
  uint16_t h[8], l[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) split16<false>(v[e], h[e], l[e]);
  hi = make_uint4(h[0] | (uint32_t)h[1] << 16, h[2] | (uint32_t)h[3] << 16, h[4] | (uint32_t)h[5] << 16, h[6] | (uint32_t)h[7] << 16);
  lo = make_uint4(l[0] | (uint32_t)l[1] << 16, l[2] | (uint32_t)l[3] << 16, l[4] | (uint32_t)l[5] << 16, l[6] | (uint32_t)l[7] << 16);
}

// The images of the column block n0 of a 128-row tile (rows blockIdx.x * 128 + r) whose fp32 values are in V
// [TM][HB_LD]: row image (rows m, k = n, ROWP passes) and transposed image (rows n, k = m, TRP passes).  16-byte chunk c
// of a tile half is row c & 7 of core matrix c >> 3 (eight consecutive k), so consecutive threads write consecutive 16
// bytes.
template <int ROWP, int TRP>
__device__ __forceinline__ void store_block_images(const float* V, int n0, uint16_t* row, int row_ks, uint16_t* tr,
                                                   int tr_ks) {
  const int tid = threadIdx.x;
#pragma unroll
  for (int kq = 0; kq < 4; ++kq) {
    const int kt = (n0 >> 5) + kq;      // row image: rows m, k = n
    if (kt >= row_ks) break;
    uint16_t* t = row + ((size_t)blockIdx.x * row_ks + kt) * 2 * TILE_ELEMS;
#pragma unroll
    for (int s = 0; s < 2; ++s) {
      const int c = tid + 256 * s, core = c >> 3, r = (core >> 2) * 8 + (c & 7), k = kq * 32 + (core & 3) * 8;
      float v[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) v[e] = V[r * HB_LD + k + e];
      uint4 hi, lo;
      split8(v, hi, lo);
      reinterpret_cast<uint4*>(t)[c] = hi;
      if (ROWP == 3) reinterpret_cast<uint4*>(t + TILE_ELEMS)[c] = lo;
    }
  }
#pragma unroll
  for (int kq = 0; kq < 4; ++kq) {
    const int kt = blockIdx.x * (TM / TK) + kq;   // transposed image: rows n (row tile n0 / 128), k = m
    if (kt >= tr_ks) break;
    uint16_t* t = tr + ((size_t)(n0 / TN) * tr_ks + kt) * 2 * TILE_ELEMS;
#pragma unroll
    for (int s = 0; s < 2; ++s) {
      const int c = tid + 256 * s, core = c >> 3, r = (core >> 2) * 8 + (c & 7), k = kq * 32 + (core & 3) * 8;
      float v[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) v[e] = V[(k + e) * HB_LD + r];
      uint4 hi, lo;
      split8(v, hi, lo);
      reinterpret_cast<uint4*>(t)[c] = hi;
      if (TRP == 3) reinterpret_cast<uint4*>(t + TILE_ELEMS)[c] = lo;
    }
  }
}

// DYN: p.M is a capacity, of which live_rows rows are processed; CTAs past them return at once.
template <int ROWP, int TRP, bool DYN = false>
__global__ void __launch_bounds__(256) head_bwd_kernel(const HeadBwd p, RowCount rc) {
  extern __shared__ __align__(16) float hsm[];
  float* V = hsm;                           // [TM][HB_LD] Ghid of this tile's rows, one column block at a time
  float* red = V + TM * HB_LD;              // [8 warps][16 sums][32 lanes]
  float* g = red + 8 * 16 * 32;             // [TM][4]: gpre 0..2, graw
  float* w9 = g + TM * 4;                   // [3][TN]: this column block of W9
  float* rsum = w9 + 3 * TN;                // [4 warps][4]: sums of gpre 0..2 and graw
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int m0 = blockIdx.x * TM;
  const int M = (int)live_rows<DYN, false>(p.M, rc);
  if (DYN && m0 >= M) return;
  if (tid < TM) {
    const int m = m0 + tid;
    float s[4] = {0.f, 0.f, 0.f, 0.f};
    if (m < M) {
#pragma unroll
      for (int j = 0; j < 3; ++j) {
        const float c = p.rgb[(size_t)m * 3 + j];
        s[j] = p.d_rgb[(size_t)m * 3 + j] * c * (1.f - c);
      }
      s[3] = p.d_sigma[m] * softplus_grad_f(p.raw[m]);
      p.graw[m] = s[3];
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) g[tid * 4 + j] = s[j];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) s[j] += __shfl_xor_sync(0xffffffffu, s[j], o);
      if (lane == 0) rsum[warp * 4 + j] = s[j];
    }
  }
  for (int n0 = 0; n0 < p.HW; n0 += TN) {
    __syncthreads();                        // g and rsum written; the previous column block's V and red read
    if (n0 == 0 && tid < 4) {
      const float s = rsum[tid] + rsum[4 + tid] + rsum[8 + tid] + rsum[12 + tid];
      atomicAdd(tid < 3 ? p.db9 + tid : p.db_raw, s);
    }
    for (int i = tid; i < 3 * TN; i += 256) {
      const int n = n0 + i % TN;
      w9[i] = n < p.HW ? p.W9[(size_t)(i / TN) * p.HW + n] : 0.f;
    }
    __syncthreads();
    // columns n0 + 4 c4 + q of rows warp + 8 i: hid in 16-byte loads, all issued first
    const int c4 = lane, n = n0 + 4 * c4;
    float4 x[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const int m = m0 + warp + 8 * i;
      x[i] = m < M && n < p.HW ? *reinterpret_cast<const float4*>(p.hid + (size_t)m * p.HW + n) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
    float cs[4] = {0.f, 0.f, 0.f, 0.f}, dw[3][4];
#pragma unroll
    for (int j = 0; j < 3; ++j)
#pragma unroll
      for (int q = 0; q < 4; ++q) dw[j][q] = 0.f;
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const int r = warp + 8 * i;
      const float h[4] = {x[i].x, x[i].y, x[i].z, x[i].w};
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        float v = 0.f;
#pragma unroll
        for (int j = 0; j < 3; ++j) v = fmaf(g[r * 4 + j], w9[j * TN + 4 * c4 + q], v);
        v = h[q] > 0.f ? v : 0.f;
        V[r * HB_LD + 4 * c4 + q] = v;
        cs[q] += v;
#pragma unroll
        for (int j = 0; j < 3; ++j) dw[j][q] = fmaf(g[r * 4 + j], h[q], dw[j][q]);
      }
    }
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      red[(warp * 16 + q) * 32 + lane] = cs[q];
#pragma unroll
      for (int j = 0; j < 3; ++j) red[(warp * 16 + 4 + 4 * j + q) * 32 + lane] = dw[j][q];
    }
    __syncthreads();
#pragma unroll
    for (int s = 0; s < 2; ++s) {           // sum k of lane l's columns: k = 0..3 Ghid column q = k, 4 + 4 j + q: dW9[j]
      const int idx = tid + 256 * s, k = idx >> 5, l = idx & 31, col = n0 + 4 * l + (k & 3);
      float v = 0.f;
#pragma unroll
      for (int w = 0; w < 8; ++w) v += red[(w * 16 + k) * 32 + l];
      if (col < p.HW) atomicAdd(k < 4 ? p.db_hid + col : p.dW9 + (size_t)((k - 4) >> 2) * p.HW + col, v);
    }
    store_block_images<ROWP, TRP>(V, n0, p.row, p.row_ks, p.tr, p.tr_ks);
  }
}

// The last trunk layer's gradient when the caller gives it (sparf_density_backward), one CTA per 128-row tile:
//   G[m][n] = (feat[m][n] > 0) * d_feat[m][n]      (d_feat NULL: G = 0)
// G leaves only as its row image (dgrad passes) and its transposed image (wgrad passes), split from the same fp32 values
// as pack_kernel would split them, zero past M and W.  Per CTA, one atomic per output: db_feat += the column sums of G,
// db_raw[0] += sum d_raw (d_raw may be NULL).
struct FeatBwd {
  int M, W;
  const float *d_raw, *d_feat, *feat;
  uint16_t *row, *tr;
  int row_ks, tr_ks;
  float *db_raw, *db_feat;
  bool vec;                 // d_feat 16-byte aligned: 16-byte loads
};

constexpr int FEAT_SMEM = (TM * HB_LD + 8 * 4 * 32 + 4) * 4;

template <int ROWP, int TRP>
__global__ void __launch_bounds__(256) feat_bwd_kernel(const FeatBwd p) {
  extern __shared__ __align__(16) float fsm[];
  float* V = fsm;                           // [TM][HB_LD] G of this tile's rows, one column block at a time
  float* red = V + TM * HB_LD;              // [8 warps][4 columns per lane][32 lanes]
  float* rsum = red + 8 * 4 * 32;           // [4 warps]: sums of d_raw
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int m0 = blockIdx.x * TM;
  if (p.d_raw && tid < TM) {
    float s = m0 + tid < p.M ? p.d_raw[m0 + tid] : 0.f;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) rsum[warp] = s;
  }
  for (int n0 = 0; n0 < p.W; n0 += TN) {
    __syncthreads();                        // rsum written; the previous column block's V and red read
    if (n0 == 0 && tid == 0 && p.d_raw) atomicAdd(p.db_raw, rsum[0] + rsum[1] + rsum[2] + rsum[3]);
    // columns n0 + 4 c4 + q of rows warp + 8 i, all loads issued first
    const int c4 = lane, n = n0 + 4 * c4;
    float4 x[16], g[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const int m = m0 + warp + 8 * i;
      const bool in = p.d_feat && m < p.M && n < p.W;
      const size_t o = (size_t)m * p.W + n;
      x[i] = in ? *reinterpret_cast<const float4*>(p.feat + o) : make_float4(0.f, 0.f, 0.f, 0.f);
      g[i] = !in ? make_float4(0.f, 0.f, 0.f, 0.f)
                 : p.vec ? *reinterpret_cast<const float4*>(p.d_feat + o)
                         : make_float4(p.d_feat[o], p.d_feat[o + 1], p.d_feat[o + 2], p.d_feat[o + 3]);
    }
    float cs[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const int r = warp + 8 * i;
      const float h[4] = {x[i].x, x[i].y, x[i].z, x[i].w}, d[4] = {g[i].x, g[i].y, g[i].z, g[i].w};
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float v = h[q] > 0.f ? d[q] : 0.f;
        V[r * HB_LD + 4 * c4 + q] = v;
        cs[q] += v;
      }
    }
#pragma unroll
    for (int q = 0; q < 4; ++q) red[(warp * 4 + q) * 32 + lane] = cs[q];
    __syncthreads();
    if (p.d_feat && tid < TM) {             // column n0 + 4 l + q, q = tid / 32, l = tid % 32
      const int q = tid >> 5, col = n0 + 4 * lane + q;
      float v = 0.f;
#pragma unroll
      for (int w = 0; w < 8; ++w) v += red[(w * 4 + q) * 32 + lane];
      if (col < p.W) atomicAdd(p.db_feat + col, v);
    }
    store_block_images<ROWP, TRP>(V, n0, p.row, p.row_ks, p.tr, p.tr_ks);
  }
}

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }
__device__ __forceinline__ void mbar_init(uint64_t* b, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" ::"r"(smem_u32(b)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* b, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" ::"r"(smem_u32(b)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* b) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];\n" ::"r"(smem_u32(b)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* b, uint32_t parity) {
  asm volatile("{\n.reg .pred P;\nSPARF_WAIT_%=:\n"
               "mbarrier.try_wait.parity.shared::cta.b64 P, [%0], %1;\n"
               "@!P bra SPARF_WAIT_%=;\n}\n" ::"r"(smem_u32(b)), "r"(parity) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];\n"
               ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
// a box of a 2D tensor map at column c0, row r0 (elements), zeros where it leaves the tensor
__device__ __forceinline__ void tensor_g2s(void* dst, const CUtensorMap* map, int c0, int r0, uint64_t* bar) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];\n"
               ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(r0), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void wgmma_wait_1() { asm volatile("wgmma.wait_group.sync.aligned 1;\n" ::: "memory"); }

// A GEMM operand as images: k-steps [0, ks0) of each row tile from image p0 (ks0 k-steps per row tile), the rest from
// p1 (ks1 k-steps per row tile), e.g. [H3 | enc] at the skip layer
struct Opnd {
  const uint16_t *p0, *p1;
  int ks0, ks1;
  __device__ const uint16_t* tile(int rt, int kt) const {
    return kt < ks0 ? p0 + ((size_t)rt * ks0 + kt) * 2 * TILE_ELEMS : p1 + ((size_t)rt * ks1 + kt - ks0) * 2 * TILE_ELEMS;
  }
};

struct Epi {
  int kind;                 // 0: Y = act(acc + bias) ; 1: D (=|+=) mask * (acc + r1_vec r1_row) ; 2: dW += acc (atomic)
  int M, N, act;            // output rows / columns
  const float* bias;
  float* out;
  int ldo, col_off, Kv;
  union {
    const float* mask;          // kind 1, ldbits == 0: keep = mask[m][n] > 0
    const uint32_t* mask_bits;  // kind 1, ldbits > 0: keep = bit n & 31 of word [m][n >> 5], ldbits words per row
  };
  const float *r1_vec, *r1_row;
  int ldmask, accumulate;
  float* colsum;            // kind 1: += column sums of the output
  float* r1_wgrad;          // kind 1 with mask and r1_vec: += sum_m r1_vec[m] mask[m][n] (the density row's gradient)
  uint16_t *row, *tr;      // output images, row_ks / tr_ks k-steps per row tile
  int row_ks, tr_ks;
  int pairs;                // N even, out and mask 8-byte aligned with even leading dimensions (kinds 0 and 1)
  // Last, in what was padding: the kernels' code is sensitive to the size of this parameter (a larger Epi made ptxas
  // build the forward GEMM's epilogue differently, and that GEMM ran about 10 % slower).
  int ldbits;
};

// The work units of a persistent GEMM: unit u = output tile u % tiles (B row tile t % rtb, A row tile t / rtb: the B
// tiles of one A row tile are consecutive units, so they read that A row tile from L2 at about the same time) over
// k-range u / tiles of nsplit, the ranges as even as possible.  CTA c takes units c, c + gridDim.x, ...
struct Units {
  int rtb, tiles, nsplit, nk;
  __device__ void get(int u, int& bx, int& by, int& kt0, int& nku) const {
    const int t = u % tiles, s = u / tiles;
    bx = t % rtb;
    by = t / rtb;
    kt0 = s * nk / nsplit;
    nku = (s + 1) * nk / nsplit - kt0;
  }
};

// The producer (one thread): the A and B tiles of every k-step of the CTA's units, in order, into a ring of STAGES
// stages that runs on across units.  Stage s is refilled once the consumers' 8 warps have arrived on empty[s] (the
// first pass finds every stage free), and completes on full[s] with the copies' bytes.
template <int PASSES>
__device__ __forceinline__ void produce(const Opnd& a, const Opnd& b, const Units& w, uint64_t* full, uint64_t* empty) {
  extern __shared__ __align__(1024) uint8_t smem[];
  const uint32_t bytes = PASSES == 3 ? 2 * TILE_BYTES : TILE_BYTES;
  int it = 0;
  for (int u = blockIdx.x; u < w.tiles * w.nsplit; u += gridDim.x) {
    int bx, by, kt0, nk;
    w.get(u, bx, by, kt0, nk);
    for (int j = 0; j < nk; ++j, ++it) {
      const int s = it % STAGES;
      mbar_wait(&empty[s], ((it / STAGES) & 1) ^ 1);
      uint8_t* st = smem + s * STAGE_BYTES;
      mbar_expect_tx(&full[s], 2 * bytes);
      bulk_g2s(st, a.tile(by, kt0 + j), bytes, &full[s]);
      bulk_g2s(st + 2 * TILE_BYTES, b.tile(bx, kt0 + j), bytes, &full[s]);
    }
  }
}

// The MMAs of one unit of nk k-steps, ring position it on entry (advanced by nk).  acc[64] of this thread = its
// fragment of the warpgroup's [64 x 128] block: acc[4 j + 2 h + c] is row 16 warp + lane/4 + 8 h, column
// 8 j + 2 (lane % 4) + c.  One MMA group stays in flight: each warp releases a stage once the group that read it has
// retired.  CONV (the staged weight-gradient GEMM): a stage is ready once its copies are complete (full) and its B
// operand has been split in place (conv).  NST: the ring's depth in stages.
template <bool F16, int PASSES, bool CONV = false, int NST = STAGES>
__device__ __forceinline__ void mma_unit(float (&acc)[64], int nk, int& it, uint64_t* full, uint64_t* empty,
                                         uint64_t* conv = nullptr) {
  extern __shared__ __align__(1024) uint8_t smem[];
  const int wg = threadIdx.x >> 7, lane = threadIdx.x & 31;
  float acc_lo[PASSES == 3 ? 64 : 1];
#pragma unroll
  for (int i = 0; i < 64; ++i) acc[i] = 0.f;
#pragma unroll
  for (int i = 0; i < (PASSES == 3 ? 64 : 1); ++i) acc_lo[i] = 0.f;
  if (nk <= 0) return;
  for (int j = 0; j < nk; ++j, ++it) {
    const int s = it % NST;
    mbar_wait(&full[s], (it / NST) & 1);
    if constexpr (CONV) mbar_wait(&conv[s], (it / NST) & 1);
    const uint8_t* st = smem + s * STAGE_BYTES;
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < TK / 16; ++ks) {
      const int ao = wg * (64 / 8) * 512 + ks * 256;   // this warpgroup's 64 rows, K16 sub-step (bytes)
      const int bo = ks * 256;
      const uint64_t ahi = smem_desc(st + ao), bhi = smem_desc(st + 2 * TILE_BYTES + bo);
      if constexpr (PASSES == 3) {
        wgmma_m64n128k16<F16>(acc_lo, smem_desc(st + TILE_BYTES + ao), bhi);
        wgmma_m64n128k16<F16>(acc_lo, ahi, smem_desc(st + 3 * TILE_BYTES + bo));
      }
      wgmma_m64n128k16<F16>(acc, ahi, bhi);
    }
    wgmma_commit();
    wgmma_wait_1();               // the MMAs of the previous k-step are done: its stage is free
    if (j > 0 && lane == 0) mbar_arrive(&empty[(it + NST - 1) % NST]);
  }
  wgmma_wait_all();
  if (lane == 0) mbar_arrive(&empty[(it + NST - 1) % NST]);
  if constexpr (PASSES == 3) {
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] += lo_unscale(acc_lo[i]);
  }
}

__device__ __forceinline__ int frag_row(int i) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;   // w = 4 * warpgroup + warp in warpgroup
  return w * 16 + (lane >> 2) + ((i >> 1) & 1) * 8;
}
__device__ __forceinline__ int frag_col(int i) { return (i >> 2) * 8 + (threadIdx.x & 3) * 2 + (i & 1); }

// two fp32 values of adjacent columns -> their hi halves and their lo halves, each pair in 32 bits (first column low)
template <bool F16>
__device__ __forceinline__ void split2(float x0, float x1, uint32_t& hi, uint32_t& lo) {
  uint16_t h0, l0, h1, l1;
  split16<F16>(x0, h0, l0);
  split16<F16>(x1, h1, l1);
  hi = h0 | (uint32_t)h1 << 16;
  lo = l0 | (uint32_t)l1 << 16;
}

// this lane's 32 bits of the transpose of the warp's 8 x 8 16-bit matrix (same fragment layout)
__device__ __forceinline__ uint32_t movmatrix_trans(uint32_t x) {
  uint32_t y;
  asm volatile("movmatrix.sync.aligned.m8n8.trans.b16 %0, %1;\n" : "=r"(y) : "r"(x));
  return y;
}


static bool pair_aligned(const float* p, int ld) { return !p || (!(reinterpret_cast<uintptr_t>(p) & 7) && ld % 2 == 0); }

// columns n, n + 1 of one row (n even; two: column n + 1 exists): one 8-byte access when every such pair of the
// matrix is 8-byte aligned and complete (PAIRS).  The choice is made once per tile, not per pair: a branch per access
// would keep the compiler from issuing the tile's loads together.
template <bool PAIRS>
__device__ __forceinline__ float2 ld2(const float* p, bool two) {
  if (PAIRS) return *reinterpret_cast<const float2*>(p);
  return make_float2(p[0], two ? p[1] : 0.f);
}
template <bool PAIRS>
__device__ __forceinline__ void st2(float* p, float x, float y, bool two) {
  if (PAIRS) {
    *reinterpret_cast<float2*>(p) = make_float2(x, y);
  } else {
    p[0] = x;
    if (two) p[1] = y;
  }
}

// the consumer warpgroups only (the producer warpgroup never joins)
__device__ __forceinline__ void consumer_sync() { asm volatile("bar.sync 1, %0;\n" ::"n"(CONSUMERS) : "memory"); }
// the 4 warps of this consumer warpgroup (barriers 3 and 4)
__device__ __forceinline__ void warpgroup_sync() { asm volatile("bar.sync %0, 128;\n" ::"r"(3 + (threadIdx.x >> 7)) : "memory"); }

// dst[n0 + c] += column c of the tile summed over its rows, from part[2 j + c'] = this thread's share of column
// 8 j + 2 (lane % 4) + c' (its two rows): over the 16 rows of each warp (shuffles), the 8 warps (the 4 KB of shared
// memory after the ring), the CTAs (one atomic per column)
__device__ __forceinline__ void tile_colsum(const float (&part)[32], int n0, int N, float* dst) {
  extern __shared__ __align__(1024) uint8_t smem[];
  float* red = reinterpret_cast<float*>(smem + STAGES * STAGE_BYTES);   // [8][128]
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  consumer_sync();              // the previous sums have been read
#pragma unroll
  for (int j = 0; j < 16; ++j)
#pragma unroll
    for (int c = 0; c < 2; ++c) {
      float s = part[2 * j + c];
#pragma unroll
      for (int o = 4; o < 32; o <<= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
      if (lane < 4) red[w * TN + 8 * j + 2 * lane + c] = s;
    }
  consumer_sync();
  if (threadIdx.x < TN && n0 + (int)threadIdx.x < N) {
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) s += red[i * TN + threadIdx.x];
    atomicAdd(dst + n0 + threadIdx.x, s);
  }
}

// The epilogue of output tile (B row tile bx, A row tile by).  It writes, each only when its template flag is set: the
// fp32 output (F32), a row image of the output (rows = output rows, K = output columns) and a transposed image (rows =
// output columns, K = output rows), with ROWP / TRP passes (3: hi and lo halves, 1: hi only) in the GEMM's 16-bit type.
// An image holds the split of the very fp32 value the output gets, zero past M and N, so it is bit-identical to what
// pack_kernel would make of the fp32 output.  Images and column sums take the full k-range and no accumulate.
// the fp32 values of the tile (kinds of Epi), stored when F32; acc = the values the images take, 0 past M and N
template <bool F32, bool PAIRS>
__device__ __forceinline__ void epilogue_values(float (&acc)[64], int m0, int n0, const Epi e) {
  // The mask loads come first, in a loop of their own, and leave one bit per value (acc[i] is kept iff bit i of keep).
  // Issued pair by pair inside the loop below, behind its branches, each would wait out its own memory latency (a mask
  // tile is 64 KB from HBM).
  // The density row's weight gradient (r1_wgrad) is summed from the same mask values: there the mask source is the
  // layer's input.  Only the input-gradient GEMMs that write images (no fp32 output) carry that code; it would change
  // how the compiler builds the other instantiations' epilogues.
  uint64_t keep = ~0ull;
  if (!F32 && e.kind == 1 && e.ldbits > 0) {
    // the same bits as one word per 32 columns: this thread's two rows of the tile's four words (2 KB per tile).  Like
    // r1_wgrad, only the image-writing input gradients carry this code, so that the other instantiations keep theirs.
    uint32_t wd[2][TN / 32];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int m = m0 + frag_row(2 * h);
#pragma unroll
      for (int q = 0; q < TN / 32; ++q) {
        const int c = (n0 >> 5) + q;
        wd[h][q] = m < e.M && c < e.ldbits ? e.mask_bits[(size_t)m * e.ldbits + c] : 0u;
      }
    }
    keep = 0;
#pragma unroll
    for (int i = 0; i < 64; i += 2) {     // columns n0 + 8 j + 2 (lane % 4) + {0, 1}, j = i / 4
      const int j = i >> 2, b = 8 * (j & 3) + 2 * (threadIdx.x & 3);
      keep |= (uint64_t)(wd[(i >> 1) & 1][j >> 2] >> b & 3u) << i;
    }
  } else if (e.kind == 1 && e.mask) {
    // e.mask shares its storage with e.mask_bits: this branch may read it as fp32 only because a bit mask never reaches
    // it.  The branch above takes every bit mask of the !F32 instantiations, and tc_gemm_nn refuses a bit mask with an
    // fp32 output D, so the F32 instantiations are never given one.
    float rv[2] = {0.f, 0.f}, part[32];
    if constexpr (!F32) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int m = m0 + frag_row(2 * h);
        if (e.r1_wgrad && m < e.M) rv[h] = e.r1_vec[m];
      }
    }
#pragma unroll
    for (int i = 0; i < 64; i += 2) {
      const int m = m0 + frag_row(i), n = n0 + frag_col(i);
      const float2 mk = m < e.M && n < e.N ? ld2<PAIRS>(e.mask + (size_t)m * e.ldmask + n, n + 1 < e.N) : make_float2(0.f, 0.f);
      keep &= ~((uint64_t)!(mk.x > 0.f) << i | (uint64_t)!(mk.y > 0.f) << (i + 1));
      if constexpr (!F32) {
        const int h = (i >> 1) & 1, p = 2 * (i >> 2);
        part[p] = h ? fmaf(rv[1], mk.x, part[p]) : rv[0] * mk.x;
        part[p + 1] = h ? fmaf(rv[1], mk.y, part[p + 1]) : rv[0] * mk.y;
      }
    }
    if constexpr (!F32) {
      if (e.r1_wgrad) tile_colsum(part, n0, e.N, e.r1_wgrad);
    }
  }
#pragma unroll
  for (int i = 0; i < 64; i += 2) {     // the pair acc[i], acc[i + 1]: columns n, n + 1 of row m
    const int m = m0 + frag_row(i), n = n0 + frag_col(i);
    if (m >= e.M || n >= e.N) {
      acc[i] = acc[i + 1] = 0.f;
      continue;
    }
    const bool two = n + 1 < e.N;
    if (e.kind == 0) {
      // two 4-byte loads: the last trunk layer's bias starts one float into its buffer (after the density row's)
      const float2 bv = e.bias ? make_float2(e.bias[n], two ? e.bias[n + 1] : 0.f) : make_float2(0.f, 0.f);
      float v0 = acc[i] + bv.x, v1 = acc[i + 1] + bv.y;
      if (e.act == 1) {
        v0 = fmaxf(v0, 0.f);
        v1 = fmaxf(v1, 0.f);
      }
      if (F32) st2<PAIRS>(e.out + (size_t)m * e.ldo + n, v0, v1, two);
      acc[i] = v0;
      acc[i + 1] = v1;
    } else if (e.kind == 1) {
      float v0 = acc[i], v1 = acc[i + 1];
      if (e.r1_vec && n < e.Kv) v0 = fmaf(e.r1_vec[m], e.r1_row[n], v0);
      if (e.r1_vec && two && n + 1 < e.Kv) v1 = fmaf(e.r1_vec[m], e.r1_row[n + 1], v1);
      if (!(keep >> i & 1)) v0 = 0.f;
      if (!(keep >> (i + 1) & 1)) v1 = 0.f;
      if (F32) {
        float* d = e.out + (size_t)m * e.ldo + n;
        if (e.accumulate) {
          const float2 o = ld2<PAIRS>(d, two);
          st2<PAIRS>(d, o.x + v0, o.y + v1, two);
        } else {
          st2<PAIRS>(d, v0, v1, two);
        }
      }
      acc[i] = v0;
      acc[i + 1] = v1;
    } else if (F32) {
      float* d = e.out + (size_t)m * e.ldo + e.col_off + n;
      if (n < e.Kv) atomicAdd(d, acc[i]);
      if (two && n + 1 < e.Kv) atomicAdd(d + 1, acc[i + 1]);
    }
    if (!two) acc[i + 1] = 0.f;
  }
}

template <bool F16, bool F32, int ROWP, int TRP>
__device__ __forceinline__ void epilogue(float (&acc)[64], int bx, int by, const Epi e) {
  const int m0 = by * TM, n0 = bx * TN;
  if (e.pairs) epilogue_values<F32, true>(acc, m0, n0, e);
  else epilogue_values<F32, false>(acc, m0, n0, e);
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  if (e.colsum) {
    float part[32];
#pragma unroll
    for (int j = 0; j < 16; ++j)
#pragma unroll
      for (int c = 0; c < 2; ++c) part[2 * j + c] = acc[4 * j + c] + acc[4 * j + 2 + c];
    tile_colsum(part, n0, e.N, e.colsum);
  }
  // The fragment of (j, h) is an 8 x 8 block: lane holds its row lane / 4, columns 2 (lane % 4) + {0, 1}.  In an image
  // that block is one core matrix (sw_off) and the lane's two values are its 32-bit word `lane`: a warp stores 128
  // contiguous bytes per half.
  if constexpr (ROWP > 0) {     // image row m, k n: tile (by, n / 32)
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const int kt = (n0 >> 5) + (j >> 2);
      if (kt >= e.row_ks) break;
      uint16_t* t = e.row + ((size_t)by * e.row_ks + kt) * 2 * TILE_ELEMS;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        uint32_t hi, lo;
        split2<F16>(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1], hi, lo);
        const int core = (2 * w + h) * (TK / 8) + (j & 3);
        reinterpret_cast<uint32_t*>(t + core * 64)[lane] = hi;
        if (ROWP == 3) reinterpret_cast<uint32_t*>(t + TILE_ELEMS + core * 64)[lane] = lo;
      }
    }
  }
  if constexpr (TRP > 0) {      // image row n, k m: tile (bx, m / 32); each block is transposed in registers first
    const int kt = (m0 >> 5) + (w >> 1);
    if (kt < e.tr_ks) {
      uint16_t* t = e.tr + ((size_t)bx * e.tr_ks + kt) * 2 * TILE_ELEMS;
#pragma unroll
      for (int j = 0; j < 16; ++j)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          uint32_t hi, lo;
          split2<F16>(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1], hi, lo);
          const int core = j * (TK / 8) + 2 * (w & 1) + h;
          reinterpret_cast<uint32_t*>(t + core * 64)[lane] = movmatrix_trans(hi);
          if (TRP == 3) reinterpret_cast<uint32_t*>(t + TILE_ELEMS + core * 64)[lane] = movmatrix_trans(lo);
        }
    }
  }
}

// Persistent, warp-specialized GEMM: each CTA walks its units (Units); thread 256 streams their tiles into the ring while
// warps 0-7 (two warpgroups, 64 output rows each) run the MMAs and epilogue of one unit after another, so the next
// unit's first stages load during an epilogue.  Registers are handed out per warpgroup: the producer warpgroup gives
// its share back (setmaxnreg), so that the consumers get 232 each (128 x 40 + 256 x 232 <= 64 K) and the epilogue,
// with its loads issued together, does not spill.
// DYN (output tiles only, nsplit = 1): e.M is a capacity, of which live_rows rows are computed; the units of A row
// tiles past them are skipped.  SPAN (with DYN and F32; the span forward): the fp32 output's rows start at row_start, the
// images' at 0; without it rc.start is never read.
template <bool F16, int PASSES, bool F32, int ROWP, int TRP, bool DYN = false, bool SPAN = false>
__global__ void __launch_bounds__(GEMM_THREADS, 1) wg_gemm_kernel(Opnd a, Opnd b, Units w, Epi e, RowCount rc) {
  extern __shared__ __align__(1024) uint8_t smem[];
  if constexpr (DYN) {
    e.M = (int)live_rows<true, SPAN>(e.M, rc);
    if (e.M == 0) return;
    w.tiles = (e.M + TM - 1) / TM * w.rtb;
    if constexpr (SPAN) e.out += row_start<true>(rc) * e.ldo;
  }
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + STAGES * STAGE_BYTES + RED_BYTES);
  uint64_t* empty = full + STAGES;
  if (threadIdx.x == 0) {
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], CONSUMERS / 32);
    }
    asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
  }
  __syncthreads();
  if (threadIdx.x >= CONSUMERS) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;\n" ::: "memory");
    if (threadIdx.x == CONSUMERS) produce<PASSES>(a, b, w, full, empty);
    return;
  }
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;\n" ::: "memory");
  int it = 0;
  for (int u = blockIdx.x; u < w.tiles * w.nsplit; u += gridDim.x) {
    int bx, by, kt0, nk;
    w.get(u, bx, by, kt0, nk);
    float acc[64];
    mma_unit<F16, PASSES>(acc, nk, it, full, empty);
    epilogue<F16, F32, ROWP, TRP>(acc, bx, by, e);
  }
}

// The weight gradient's B operand straight from fp32, X[m / div][k] as rows k, contraction over m (TnB's values): X 16-byte
// aligned, ldx and K multiples of 4 floats, so that every row of a k-step is one bulk copy.  bits (may be NULL) as TnB.
struct Staged {
  const float* X;
  int ldx, div, M, K;
  uint32_t* bits;
  int kw;
};

constexpr int STAGED_THREADS = CONSUMERS + 256;   // + the converter warpgroup (8-11) + the producer warpgroup (12-15)
constexpr int STAGED_STAGES = 5;                  // one stage fewer than the other GEMMs: room for the partial tile
constexpr int PART_BYTES = TM * TN * 4;           // the partial tile, [128 x 128] fp32
constexpr int STAGED_SMEM = STAGED_STAGES * STAGE_BYTES + PART_BYTES + 3 * STAGED_STAGES * 8;

// split8 with the lo half's scaling by 2^LO_SHIFT as a multiply: the same bytes (the scaling of the residual is exact,
// it overflows to the same infinity, and NaN stays NaN), without the special-case code of ldexpf, which made up most of
// the converter's instructions
__device__ __forceinline__ void split8_mul(const float (&v)[8], uint4& hi, uint4& lo) {
  uint16_t h[8], l[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    const __nv_bfloat16 b = __float2bfloat16_rn(v[e]);
    h[e] = __bfloat16_as_ushort(b);
    l[e] = __bfloat16_as_ushort(__float2bfloat16_rn((v[e] - __bfloat162float(b)) * (float)(1 << LO_SHIFT)));
  }
  hi = make_uint4(h[0] | (uint32_t)h[1] << 16, h[2] | (uint32_t)h[3] << 16, h[4] | (uint32_t)h[5] << 16, h[6] | (uint32_t)h[7] << 16);
  lo = make_uint4(l[0] | (uint32_t)l[1] << 16, l[2] | (uint32_t)l[3] << 16, l[4] | (uint32_t)l[5] << 16, l[6] | (uint32_t)l[7] << 16);
}

__device__ __forceinline__ void converter_sync() { asm volatile("bar.sync 2, 128;\n" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory"); }

// The producer warp: per k-step, the A tile with one copy and the 32 rows m of B (X[m / div][128 bx, 128 bx + 128) in
// fp32, 512 bytes per row at most) into the stage's 16 KB of B halves, row m at 512 (m - m0) bytes.  With div = 1 the
// rows are one box of the tensor map xmap (zeros past M and K), so a k-step is two copies; the time of a k-step's
// copies followed their count more than their bytes.  Per-ray rows (div > 1) take one copy per lane; rows at or past M
// are not copied and the bytes past K of a row not written.  The converter reads neither.
template <int PASSES, int NST = STAGES>
__device__ __forceinline__ void produce_staged(const Opnd& a, const Staged& x, const CUtensorMap* xmap, const Units& w,
                                               uint64_t* full, uint64_t* empty) {
  extern __shared__ __align__(1024) uint8_t smem[];
  const int lane = threadIdx.x & 31;
  const uint32_t abytes = PASSES == 3 ? 2 * TILE_BYTES : TILE_BYTES;
  int it = 0;
  for (int u = blockIdx.x; u < w.tiles * w.nsplit; u += gridDim.x) {
    int bx, by, kt0, nk;
    w.get(u, bx, by, kt0, nk);
    const int k0 = bx * TM;
    const uint32_t rbytes = 4 * min(TM, x.K - k0);
    for (int j = 0; j < nk; ++j, ++it) {
      const int s = it % NST, m0 = (kt0 + j) * TK;
      mbar_wait(&empty[s], ((it / NST) & 1) ^ 1);
      uint8_t* st = smem + s * STAGE_BYTES;
      if (x.div == 1) {
        if (lane == 0) {
          mbar_expect_tx(&full[s], abytes + TK * TM * 4);
          bulk_g2s(st, a.tile(by, kt0 + j), abytes, &full[s]);
          tensor_g2s(st + 2 * TILE_BYTES, xmap, k0, m0, &full[s]);
        }
        continue;
      }
      if (lane == 0) {
        mbar_expect_tx(&full[s], abytes + min(TK, x.M - m0) * rbytes);
        bulk_g2s(st, a.tile(by, kt0 + j), abytes, &full[s]);
      }
      __syncwarp();             // the expected bytes are set before any row copy can complete
      const int m = m0 + lane;
      if (m < x.M) bulk_g2s(st + 2 * TILE_BYTES + lane * (TM * 4), x.X + (size_t)(m / x.div) * x.ldx + k0, rbytes, &full[s]);
    }
  }
}

// The converter warpgroup: thread t takes column k = 128 bx + t of a staged k-step, reads its 32 values m (lane = k: no
// bank conflicts), zero at or past M and K, and once the warpgroup has read the whole tile writes them in place as the
// K-major image pack_kernel<TnB> makes (four 16-byte core-matrix rows per half), then hands the stage to the consumers
// on conv[s].  Its warps also write the ReLU bits of units with by == 0 (one per (bx, k-step)): a ballot per row m.
template <int PASSES, int NST = STAGES>
__device__ __forceinline__ void convert_staged(const Staged& x, const Units& w, uint64_t* full, uint64_t* conv) {
  extern __shared__ __align__(1024) uint8_t smem[];
  const int t = threadIdx.x - CONSUMERS, lane = t & 31;
  int it = 0;
  for (int u = blockIdx.x; u < w.tiles * w.nsplit; u += gridDim.x) {
    int bx, by, kt0, nk;
    w.get(u, bx, by, kt0, nk);
    const bool kin = bx * TM + t < x.K, bits = x.bits && by == 0;
    const int bword = bx * (TM / 32) + (t >> 5);
    for (int j = 0; j < nk; ++j, ++it) {
      const int s = it % NST, m0 = (kt0 + j) * TK;
      mbar_wait(&full[s], (it / NST) & 1);
      uint8_t* st = smem + s * STAGE_BYTES + 2 * TILE_BYTES;
      const float* src = reinterpret_cast<const float*>(st);
      float v[TK];
      if (kin && m0 + TK <= x.M) {
#pragma unroll
        for (int r = 0; r < TK; ++r) v[r] = src[r * TM + t];
      } else {
#pragma unroll
        for (int r = 0; r < TK; ++r) v[r] = kin && m0 + r < x.M ? src[r * TM + t] : 0.f;
      }
      if (bits) {
        uint32_t word = 0;
#pragma unroll
        for (int r = 0; r < TK; ++r) {
          const uint32_t b = __ballot_sync(0xffffffffu, v[r] > 0.f);
          if (lane == r) word = b;
        }
        if (m0 + lane < x.M && bword < x.kw) x.bits[(size_t)(m0 + lane) * x.kw + bword] = word;
      }
      converter_sync();         // the whole tile has been read before it is overwritten
      uint16_t* img = reinterpret_cast<uint16_t*>(st);
#pragma unroll
      for (int o = 0; o < TK / 8; ++o) {
        float e8[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) e8[e] = v[8 * o + e];
        uint4 hi, lo;
        split8_mul(e8, hi, lo);
        const int off = sw_off(t, 8 * o);
        *reinterpret_cast<uint4*>(img + off) = hi;
        if (PASSES == 3) *reinterpret_cast<uint4*>(img + TILE_ELEMS + off) = lo;
      }
      fence_proxy_async();      // the image is visible to the MMAs; the reads above precede the stage's next copies
      __syncwarp();
      if (lane == 0) mbar_arrive(&conv[s]);
    }
  }
}

// Element (r, c) of the staged GEMM's partial tile, [128 rows x 128 columns] fp32 after the ring: the 8-column groups of
// row r are permuted by r % 8, so that a warp's fragment stores (8 rows x one column group) and the flush's reads (32
// columns of one row) are free of bank conflicts.
__device__ __forceinline__ int part_off(int r, int c) { return r * TN + (((c >> 3) ^ (r & 7)) << 3) + (c & 7); }

// The staged GEMM's epilogue of unit (bx, by).  A CTA's consecutive units of one output tile (with a grid that is a
// multiple of the tile count, all of its units) sum their partial tiles in shared memory, in unit order, and the last
// of them adds the sum to dW with one atomic per element: a warp's atomics cover 128 contiguous bytes of a row.  The
// first unit stores its partial instead of adding it to zeros, which would turn -0 into +0.  Each warp stores, adds and
// flushes the 16 rows of its own fragments, so only its own lanes share them.
__device__ __forceinline__ void presum_epilogue(const float (&acc)[64], float* part, bool first, bool flush, int bx, int by,
                                                const Epi& e) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
  for (int i = 0; i < 64; i += 2) {
    float2* p = reinterpret_cast<float2*>(part + part_off(frag_row(i), frag_col(i)));
    if (first) {
      *p = make_float2(acc[i], acc[i + 1]);
    } else {
      const float2 o = *p;
      *p = make_float2(o.x + acc[i], o.y + acc[i + 1]);
    }
  }
  if (!flush) return;
  __syncwarp();
  const int m0 = by * TM, n0 = bx * TN;
  float* out = e.out + e.col_off + n0;
  for (int i = 0; i < 16; ++i) {
    const int r = 16 * w + i, m = m0 + r;
    if (m >= e.M) continue;
#pragma unroll
    for (int q = 0; q < TN / 32; ++q) {
      const int c = 32 * q + lane, n = n0 + c;
      if (n < e.N && n < e.Kv) atomicAdd(out + (size_t)m * e.ldo + c, part[part_off(r, c)]);
    }
  }
  __syncwarp();                 // the tile has been read before the next unit's partial overwrites it
}

// The weight-gradient GEMM dW += G^T X with B read as fp32 (Staged): wg_gemm_kernel's units and MMAs on a ring of
// STAGED_STAGES, with a fourth warpgroup that splits each stage's B in place between its copies and its MMAs, so no pack
// kernel writes and no GEMM reads an image of X, and an epilogue that adds each CTA's partials of one tile once
// (presum_epilogue).  Registers: producer 40, converter 64, consumers 200 (<= 64 K).  xmap: X as a tensor of x.M rows
// (the capacity with DYN) by x.K columns, read where div = 1 (produce_staged).
// DYN: x.M is a capacity, of which live_rows rows are summed; the k-range split is gemm_units' for that count, computed
// here from ctas (the CTAs gemm_units was given).
template <int PASSES, bool DYN = false>
__global__ void __launch_bounds__(STAGED_THREADS, 1) wg_gemm_staged_kernel(Opnd a, Staged x, Units w, Epi e, RowCount rc,
                                                                           int ctas, const __grid_constant__ CUtensorMap xmap) {
  extern __shared__ __align__(1024) uint8_t smem[];
  if constexpr (DYN) {
    x.M = (int)live_rows<true, false>(x.M, rc);
    if (x.M == 0) return;
    w.nk = (x.M + TK - 1) / TK;
    w.nsplit = max(1, min(w.nk, (ctas + w.tiles - 1) / w.tiles * ((w.nk + 1023) / 1024)));
  }
  float* part = reinterpret_cast<float*>(smem + STAGED_STAGES * STAGE_BYTES);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + STAGED_STAGES * STAGE_BYTES + PART_BYTES);
  uint64_t* empty = full + STAGED_STAGES;
  uint64_t* conv = empty + STAGED_STAGES;
  if (threadIdx.x == 0) {
    for (int i = 0; i < STAGED_STAGES; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], CONSUMERS / 32);
      mbar_init(&conv[i], 4);
    }
    asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
  }
  __syncthreads();
  if (threadIdx.x >= CONSUMERS + 128) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;\n" ::: "memory");
    if (threadIdx.x < CONSUMERS + 128 + 32) produce_staged<PASSES, STAGED_STAGES>(a, x, &xmap, w, full, empty);
    return;
  }
  if (threadIdx.x >= CONSUMERS) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 64;\n" ::: "memory");
    convert_staged<PASSES, STAGED_STAGES>(x, w, full, conv);
    return;
  }
  asm volatile("setmaxnreg.inc.sync.aligned.u32 200;\n" ::: "memory");
  const int units = w.tiles * w.nsplit, grid = gridDim.x;
  int it = 0;
  for (int u = blockIdx.x; u < units; u += grid) {
    int bx, by, kt0, nk;
    w.get(u, bx, by, kt0, nk);
    float acc[64];
    mma_unit<false, PASSES, true, STAGED_STAGES>(acc, nk, it, full, empty, conv);
    const int t = u % w.tiles;
    const bool first = u < grid || (u - grid) % w.tiles != t;
    const bool flush = u + grid >= units || (u + grid) % w.tiles != t;
    presum_epilogue(acc, part, first, flush, bx, by, e);
  }
}

// ---- The fused trunk forward: one tile of 128 rows goes through every trunk layer without leaving the SM.
constexpr int CH_W = 256;                     // the trunk width it is built for
constexpr int CH_M = TM;                      // rows per tile: 64 per consumer warpgroup
constexpr int CH_KS = CH_W / TK;              // k-steps of a layer's activation input
constexpr int CH_ENC_KS = 2;                  // k-steps of the encoding at most (64 columns)
constexpr int CH_Q = 4;                       // a layer's output columns are computed in quarters of 64
constexpr int CH_QHALF = CH_W / CH_Q * TK * 2;             // one 16-bit half of a quarter's k-step of B, [64 x 32], 4 KB
constexpr int CH_STAGE_KS = 2;                // weight ring: per stage two k-steps of one quarter (hi, lo each), 16 KB
constexpr int CH_STAGE = CH_STAGE_KS * 2 * CH_QHALF;
constexpr int CH_STAGES = 4;
constexpr int CH_ENC = CH_KS * 2 * TILE_BYTES;            // byte offsets in shared memory: activations at 0 (128 KB),
constexpr int CH_RING = CH_ENC + CH_ENC_KS * 2 * TILE_BYTES;  // the encoding (32 KB), the ring (64 KB),
constexpr int CH_BAR = CH_RING + CH_STAGES * CH_STAGE;    // full[4], empty[4], enc_full, enc_empty
constexpr int CH_SMEM = CH_BAR + (2 * CH_STAGES + 2) * 8;
static_assert(CH_SMEM <= 232448, "the fused chains' shared memory exceeds an H100 SM's 227 KB");

// Its own parameter struct (not Epi: see the note there).  Layer l < nl computes H[l] = relu(in_l W_l^T + bias[l]), in_0 =
// enc, in_l = H[l-1] ( | enc at l == skip), from the weight image w[l] (256 rows, chain_ks(l) k-steps, as tc_pack_nt
// makes it: per quarter).  H[l] == NULL: not written to global memory.  last (may be NULL): the row image of H[nl-1].
// bits[l] (may be NULL): the ReLU mask H[l] > 0, 8 words per row (trunk_chain_kernel's BITS instantiations only).
struct Chain {
  int M, nl, skip, enc_ks;
  const uint16_t* enc;
  const uint16_t* w[SPARF_MAX_TRUNK];
  const float* bias[SPARF_MAX_TRUNK];
  float* H[SPARF_MAX_TRUNK];
  uint16_t* last;
  uint32_t* bits[SPARF_MAX_TRUNK];
};

__host__ __device__ __forceinline__ int chain_ks(int l, int skip, int enc_ks) {
  return l == 0 ? enc_ks : CH_KS + (l == skip ? enc_ks : 0);
}

// The weight stages of one layer of nk k-steps into the ring (position it, advanced): per quarter its k-steps,
// CH_STAGE_KS to a stage (the last one of an odd count alone), each stage one copy, since the image holds a quarter's
// k-steps one after another.
template <int PASSES>
__device__ __forceinline__ void chain_stream(const uint16_t* w, int nk, int& it, uint64_t* full, uint64_t* empty) {
  extern __shared__ __align__(1024) uint8_t smem[];
  constexpr int HB = PASSES == 3 ? 2 : 1;     // halves copied
  for (int q = 0; q < CH_Q; ++q)
    for (int j0 = 0; j0 < nk; j0 += CH_STAGE_KS, ++it) {
      const int s = it % CH_STAGES;
      mbar_wait(&empty[s], ((it / CH_STAGES) & 1) ^ 1);
      const uint32_t bytes = (nk - j0 < CH_STAGE_KS ? nk - j0 : CH_STAGE_KS) * HB * CH_QHALF;
      mbar_expect_tx(&full[s], bytes);
      bulk_g2s(smem + CH_RING + s * CH_STAGE, w + ((size_t)q * nk + j0) * HB * (CH_QHALF / 2), bytes, &full[s]);
    }
}

// A 128-row tile of a row image (row tile t, ks k-steps) into shared memory at dst, one copy per k-step and half
template <int PASSES>
__device__ __forceinline__ void chain_load_rows(uint8_t* dst, const uint16_t* img, int t, int ks, uint64_t* bar) {
  constexpr int HB = PASSES == 3 ? 2 : 1;
  mbar_expect_tx(bar, ks * HB * TILE_BYTES);
  for (int kt = 0; kt < ks; ++kt)
    for (int h = 0; h < HB; ++h)
      bulk_g2s(dst + (kt * 2 + h) * TILE_BYTES, img + (((size_t)t * ks + kt) * 2 + h) * TILE_ELEMS, TILE_BYTES, bar);
}

// The producer (one thread) walks (tile, layer, quarter, k-step): the tile's rows of the encoding image once per tile
// (they stay for layer 0 and the skip layer; the buffer is free once the previous tile's last reader has retired), and
// the layers' weights into a ring that runs on across quarters, layers and tiles.
template <int PASSES>
__device__ __forceinline__ void chain_produce(const Chain& c, int tiles, uint64_t* full, uint64_t* empty, uint64_t* enc_full,
                                              uint64_t* enc_empty) {
  extern __shared__ __align__(1024) uint8_t smem[];
  int it = 0, n = 0;
  for (int t = blockIdx.x; t < tiles; t += gridDim.x) {
    mbar_wait(enc_empty, (n & 1) ^ 1);
    ++n;
    chain_load_rows<PASSES>(smem + CH_ENC, c.enc, t, c.enc_ks, enc_full);
    for (int l = 0; l < c.nl; ++l) chain_stream<PASSES>(c.w[l], chain_ks(l, c.skip, c.enc_ks), it, full, empty);
  }
}

// The MMAs of one quarter of a layer for this warpgroup's 64 rows of the tile: nk k-steps of A, the first na (0 or
// CH_KS) from the activation buffer and the rest from the encoding's (the skip layer; the encoding alone at layer 0), B
// the quarter's k-steps from the ring.  Per k-step mma_unit's instruction sequence, so every output element sums in the
// same order as the GEMMs'.  Warpgroup g's A is rows [64 g, 64 g + 64) of each [128 x 32] k-step, its second 4 KB.  One
// MMA group (a stage) stays in flight; each warp releases a stage once the group that read it has retired.
template <bool F16, int PASSES>
__device__ __forceinline__ void chain_mma(float (&acc)[32], int nk, int na, int& it, uint64_t* full, uint64_t* empty) {
  extern __shared__ __align__(1024) uint8_t smem[];
  constexpr int HB = PASSES == 3 ? 2 : 1;
  const int wg = threadIdx.x >> 7, lane = threadIdx.x & 31;
  float acc_lo[PASSES == 3 ? 32 : 1];
#pragma unroll
  for (int i = 0; i < 32; ++i) acc[i] = 0.f;
#pragma unroll
  for (int i = 0; i < (PASSES == 3 ? 32 : 1); ++i) acc_lo[i] = 0.f;
  for (int j0 = 0; j0 < nk; j0 += CH_STAGE_KS, ++it) {
    const int s = it % CH_STAGES;
    mbar_wait(&full[s], (it / CH_STAGES) & 1);
    const uint8_t* st = smem + CH_RING + s * CH_STAGE;
    wgmma_fence();
#pragma unroll
    for (int jj = 0; jj < CH_STAGE_KS; ++jj) {
      const int j = j0 + jj;
      if (j >= nk) break;
      const uint8_t* a = (j < na ? smem + j * 2 * TILE_BYTES : smem + CH_ENC + (j - na) * 2 * TILE_BYTES) + wg * (TILE_BYTES / 2);
      const uint8_t* b = st + jj * HB * CH_QHALF;
#pragma unroll
      for (int ks = 0; ks < TK / 16; ++ks) {
        const uint64_t ahi = smem_desc(a + ks * 256), bhi = smem_desc(b + ks * 256);
        if constexpr (PASSES == 3) {
          wgmma_m64n64k16<F16>(acc_lo, smem_desc(a + TILE_BYTES + ks * 256), bhi);
          wgmma_m64n64k16<F16>(acc_lo, ahi, smem_desc(b + CH_QHALF + ks * 256));
        }
        wgmma_m64n64k16<F16>(acc, ahi, bhi);
      }
    }
    wgmma_commit();
    wgmma_wait_1();             // the stages before this one have retired
    if (j0 > 0 && lane == 0) mbar_arrive(&empty[(it + CH_STAGES - 1) % CH_STAGES]);
  }
  wgmma_wait_all();
  if (lane == 0) mbar_arrive(&empty[(it + CH_STAGES - 1) % CH_STAGES]);
  if constexpr (PASSES == 3) {
#pragma unroll
    for (int i = 0; i < 32; ++i) acc[i] += lo_unscale(acc_lo[i]);
  }
}

// A quarter's fragment: acc[4 j + 2 h + c] is row 64 wg + 16 wq + lane / 4 + 8 h of the tile, column 64 q + 8 j +
// 2 (lane % 4) + c of the layer.
__device__ __forceinline__ int chain_row(int t, int h) {
  return t * CH_M + (threadIdx.x >> 5) * 16 + ((threadIdx.x & 31) >> 2) + 8 * h;
}

// The split of a quarter's values (split2: the bytes a row image holds of them): s[2 j + h] the hi pair of (j, h), the
// lo pair 16 words further on (PASSES == 3)
template <int PASSES>
using ChainSplit = uint32_t[PASSES == 3 ? 32 : 16];

template <bool F16, int PASSES>
__device__ __forceinline__ void chain_split(const float (&acc)[32], ChainSplit<PASSES>& s) {
#pragma unroll
  for (int j = 0; j < 8; ++j)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      uint32_t hi, lo;
      split2<F16>(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1], hi, lo);
      s[2 * j + h] = hi;
      if (PASSES == 3) s[16 + 2 * j + h] = lo;
    }
}

// quarter q's split as part of a 128-row tile of a row image at img (k-step stride kstride, the lo half lo_off after
// the hi half, 16-bit elements): the fragment of (j, h) is one core matrix, this lane's pair its 32-bit word `lane`
template <int PASSES>
__device__ __forceinline__ void chain_put(const ChainSplit<PASSES>& s, int q, uint16_t* img, int kstride, int lo_off) {
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    uint16_t* kt = img + (size_t)(2 * q + (j >> 2)) * kstride;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int core = (2 * w + h) * (TK / 8) + (j & 3);
      reinterpret_cast<uint32_t*>(kt + core * 64)[lane] = s[2 * j + h];
      if (PASSES == 3) reinterpret_cast<uint32_t*>(kt + lo_off + core * 64)[lane] = s[16 + 2 * j + h];
    }
  }
}

// this thread's bias pairs of quarter q of layer l, columns 64 q + 8 j + 2 (lane % 4) + {0, 1}; loaded before the
// quarter's MMAs.  Two scalar loads per pair: a bias in a flat parameter bank may start at an odd float.
__device__ __forceinline__ void chain_bias(float2 (&bv)[8], const float* bias, int q) {
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const float* b = bias + q * 64 + j * 8 + (lane & 3) * 2;
    bv[j] = make_float2(b[0], b[1]);
  }
}

// The bias and ReLU of a quarter as epilogue_values kind 0: acc becomes the layer's output, zero past M.
__device__ __forceinline__ void chain_bias_relu(float (&acc)[32], const float2 (&bv)[8], int M, int t) {
#pragma unroll
  for (int i = 0; i < 32; i += 2) {
    if (chain_row(t, (i >> 1) & 1) >= M) {
      acc[i] = acc[i + 1] = 0.f;
      continue;
    }
    acc[i] = fmaxf(acc[i] + bv[i >> 2].x, 0.f);
    acc[i + 1] = fmaxf(acc[i + 1] + bv[i >> 2].y, 0.f);
  }
}

// The fp32 output of quarter q (acc after chain_bias_relu) to H[l].  Quarter 3's runs after the proxy fence that follows
// the stores into the activation buffer: a fence issued behind these global stores waits for them too, once per layer
// with no MMA in flight; issued after it, they drain while the next layer's MMAs run.
__device__ __forceinline__ void chain_store(const float (&acc)[32], float* H, int M, int t, int q) {
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int i = 0; i < 32; i += 2) {
    const int m = chain_row(t, (i >> 1) & 1), n = q * 64 + (i >> 2) * 8 + (lane & 3) * 2;
    if (m < M) *reinterpret_cast<float2*>(H + (size_t)m * CH_W + n) = make_float2(acc[i], acc[i + 1]);
  }
}

// The ReLU mask of quarter q as tc_gemm_tn writes it, bit n & 31 of word [m][n >> 5] = H[m][n] > 0 (the predicate the
// fp32 mask applies, so NaN and -0 give 0): a lane's 8 values of a 32-column word (4 j x 2 columns) go to its bits
// 2 (lane % 4) + 8 (j % 4) + {0, 1}, the quad ORs them together, and lanes with lane % 4 < 2 store word lane % 4 of the
// quarter's two.  Like chain_store, quarter 3's runs after the proxy fence.
__device__ __forceinline__ void chain_store_bits(const float (&acc)[32], uint32_t* bits, int M, int t, int q) {
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    uint32_t mine = 0;
#pragma unroll
    for (int wd = 0; wd < 2; ++wd) {
      uint32_t w = 0;
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) {
        const int i = 4 * (4 * wd + jj) + 2 * h, b = 8 * jj + 2 * (lane & 3);
        w |= (uint32_t)(acc[i] > 0.f) << b | (uint32_t)(acc[i + 1] > 0.f) << (b + 1);
      }
      w |= __shfl_xor_sync(0xffffffffu, w, 1);
      w |= __shfl_xor_sync(0xffffffffu, w, 2);
      if ((lane & 3) == wd) mine = w;
    }
    const int m = chain_row(t, h);
    if (m < M && (lane & 3) < 2) bits[(size_t)m * (CH_W / 32) + 2 * q + (lane & 3)] = mine;
  }
}

// Persistent and warp-specialized like wg_gemm_kernel (thread 256 produces, warps 0-7 consume, the same register
// hand-back), on tiles of 128 rows: warpgroup g computes every column of rows [64 g, 64 g + 64) of the tile, a quarter
// of 64 columns at a time, and never reads the other warpgroup's rows; the two share only the weight ring, each stage of
// which both consume.  A quarter's split stays in registers until the layer's last quarter has retired its MMAs; then
// the warpgroup overwrites its rows of the layer's input in the activation buffer with all four (the same split2 as a
// row image's), fences them for the async proxy and meets its own 4 warps at a named barrier before the next layer's
// MMAs.  The last layer's split goes to its row image in global memory instead, where asked.
// Tiles: ceil(M / 128), so that the last image's 128-row tiles are written whole; a warpgroup whose rows all lie past M
// still runs (and releases) every stage, and its epilogue zeroes them.  DYN: c.M is a capacity, of which live_rows rows
// (M) are computed.  SPAN (with DYN; the span forward): H and bits take their rows from row_start on (the last image's
// rows start at 0); without it rc.start is never read.  BITS: c.bits[l] are written where not NULL (the other
// instantiations never read them).
template <bool F16, int PASSES, bool DYN = false, bool BITS = false, bool SPAN = false>
__global__ void __launch_bounds__(GEMM_THREADS, 1) trunk_chain_kernel(const Chain c, RowCount rc) {
  extern __shared__ __align__(1024) uint8_t smem[];
  const int M = (int)live_rows<DYN, SPAN>(c.M, rc);
  if (DYN && M == 0) return;
  const int tiles = (M + CH_M - 1) / CH_M;
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + CH_BAR);
  uint64_t* empty = full + CH_STAGES;
  uint64_t* enc_full = empty + CH_STAGES;
  uint64_t* enc_empty = enc_full + 1;
  if (threadIdx.x == 0) {
    for (int i = 0; i < CH_STAGES; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], CONSUMERS / 32);
    }
    mbar_init(enc_full, 1);
    mbar_init(enc_empty, CONSUMERS / 32);
    asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
  }
  __syncthreads();
  if (threadIdx.x >= CONSUMERS) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;\n" ::: "memory");
    if (threadIdx.x == CONSUMERS) chain_produce<PASSES>(c, tiles, full, empty, enc_full, enc_empty);
    return;
  }
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;\n" ::: "memory");
  const int enc_last = c.skip > 0 && c.skip < c.nl ? c.skip : 0;   // the last layer that reads the encoding
  const long long s0 = row_start<SPAN>(rc);   // the span forward: H and bits at global rows s0 + m; 0 otherwise
  int it = 0, n = 0;
  for (int t = blockIdx.x; t < tiles; t += gridDim.x) {
    mbar_wait(enc_full, n & 1);
    ++n;
    for (int l = 0; l < c.nl; ++l) {
      const int nk = chain_ks(l, c.skip, c.enc_ks), na = l == 0 ? 0 : CH_KS;
      ChainSplit<PASSES> held[CH_Q - 1];
#pragma unroll
      for (int q = 0; q < CH_Q; ++q) {
        float2 bv[8];
        chain_bias(bv, c.bias[l], q);
        float acc[32];
        chain_mma<F16, PASSES>(acc, nk, na, it, full, empty);
        if (q == CH_Q - 1 && l == enc_last && (threadIdx.x & 31) == 0) mbar_arrive(enc_empty);
        chain_bias_relu(acc, bv, M, t);
        if (l + 1 < c.nl) {
          if (q < CH_Q - 1) {
            chain_split<F16, PASSES>(acc, held[q]);
          } else {      // every MMA on this warpgroup's rows of the layer's input has retired
            ChainSplit<PASSES> s;
            chain_split<F16, PASSES>(acc, s);
            uint16_t* buf = reinterpret_cast<uint16_t*>(smem);
#pragma unroll
            for (int p = 0; p < CH_Q - 1; ++p) chain_put<PASSES>(held[p], p, buf, 2 * TILE_ELEMS, TILE_ELEMS);
            chain_put<PASSES>(s, CH_Q - 1, buf, 2 * TILE_ELEMS, TILE_ELEMS);
            fence_proxy_async();      // the stores into the activation buffer, before the MMAs that read them
            warpgroup_sync();
          }
        } else if (c.last) {
          ChainSplit<PASSES> s;
          chain_split<F16, PASSES>(acc, s);
          chain_put<PASSES>(s, q, c.last + (size_t)t * CH_KS * 2 * TILE_ELEMS, 2 * TILE_ELEMS, TILE_ELEMS);
        }
        if (c.H[l]) chain_store(acc, c.H[l] + s0 * CH_W, M, t, q);
        if (BITS && c.bits[l]) chain_store_bits(acc, c.bits[l] + s0 * (CH_W / 32), M, t, q);
      }
    }
  }
}

template <bool F16, int PASSES>
static int launch_chain(const Chain& c, int ctas, RowCount rc, cudaStream_t st) {
  bool bits = false;
  for (int l = 0; l < c.nl; ++l) bits |= c.bits[l] != nullptr;
  auto kernel = bits ? (rc.rows ? trunk_chain_kernel<F16, PASSES, true, true> : trunk_chain_kernel<F16, PASSES, false, true>)
                     : (rc.rows ? trunk_chain_kernel<F16, PASSES, true> : trunk_chain_kernel<F16, PASSES>);
  if (rc.start) {       // the span forward: a taped forward, which keeps the mask bits
    if (!bits) {
      set_error("trunk_chain: a row start needs the mask bits (taped forward)");
      return SPARF_ERR_UNSUPPORTED;
    }
    kernel = trunk_chain_kernel<F16, PASSES, true, true, true>;
  }
  SPARF_CHECK_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, CH_SMEM));
  kernel<<<std::min(ceil_div(c.M, CH_M), ctas), GEMM_THREADS, CH_SMEM, st>>>(c, rc);
  SPARF_CHECK_LAUNCH("trunk_chain_kernel");
  return SPARF_OK;
}

// ---- The trunk backward's input gradients in one persistent kernel, the same walk as trunk_chain_kernel.  Layer l
// (top >= l >= 1) computes G[l-1] = mask_l * (G[l] W_l), W_l's [256 x 256] part over H[l-1], from its weight image w[l]
// (256 rows, CH_KS k-steps, as tc_pack_nn packs it: per quarter); mask_l = bits[l] (H[l-1] > 0, 8 words per row).
// G[top] comes in as its row image, and a tile's gradient stays in the activation buffer from layer to layer.  G[l-1]
// leaves as its transposed image tr[l] (tr_ks k-steps per row tile), its column sums (db[l] +=) and, where row[l] is not
// NULL, its row image.  Shared memory as trunk_chain_kernel's, with the column sums' partials where the encoding would be.
struct DgChain {
  int M, top, tr_ks;
  const uint16_t* in;
  const uint16_t* w[SPARF_MAX_TRUNK];
  const uint32_t* bits[SPARF_MAX_TRUNK];
  float* db[SPARF_MAX_TRUNK];
  uint16_t* tr[SPARF_MAX_TRUNK];
  uint16_t* row[SPARF_MAX_TRUNK];
};

// The producer (one thread) walks (tile, layer, quarter, k-step): the tile's rows of the input image once per tile,
// once the previous tile's last MMAs have retired (act_empty), and the weights as chain_produce streams them.
template <int DP>
__device__ __forceinline__ void dg_produce(const DgChain& c, int tiles, uint64_t* full, uint64_t* empty, uint64_t* act_full,
                                           uint64_t* act_empty) {
  extern __shared__ __align__(1024) uint8_t smem[];
  int it = 0, n = 0;
  for (int t = blockIdx.x; t < tiles; t += gridDim.x) {
    mbar_wait(act_empty, (n & 1) ^ 1);
    ++n;
    chain_load_rows<DP>(smem, c.in, t, CH_KS, act_full);
    for (int l = c.top; l >= 1; --l) chain_stream<DP>(c.w[l], CH_KS, it, full, empty);
  }
}

// this thread's two rows' mask words of quarter q (one 8-byte load each); rows past M get none, so they are zero
__device__ __forceinline__ void dg_mask_words(uint2 (&wd)[2], const uint32_t* bits, int M, int t, int q) {
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int m = chain_row(t, h);
    wd[h] = m < M ? *reinterpret_cast<const uint2*>(bits + (size_t)m * (CH_W / 32) + 2 * q) : make_uint2(0, 0);
  }
}

// quarter q's split as the transposed image's (epilogue<..., TRP>'s): rows n (row tile q / 2), k = m (k-step 4 t + m / 32
// of the tile's rows); each 8 x 8 block is transposed in registers
template <int TP, int DP>
__device__ __forceinline__ void dg_put_tr(const ChainSplit<DP>& s, int q, uint16_t* tr, int tr_ks, int t) {
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int kt = 4 * t + (w >> 1);
  if (kt >= tr_ks) return;
  uint16_t* tp = tr + ((size_t)(q >> 1) * tr_ks + kt) * 2 * TILE_ELEMS;
#pragma unroll
  for (int j = 0; j < 8; ++j)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int core = (8 * (q & 1) + j) * (TK / 8) + 2 * (w & 1) + h;
      reinterpret_cast<uint32_t*>(tp + core * 64)[lane] = movmatrix_trans(s[2 * j + h]);
      if (TP == 3) reinterpret_cast<uint32_t*>(tp + TILE_ELEMS + core * 64)[lane] = movmatrix_trans(s[16 + 2 * j + h]);
    }
}

// Persistent and warp-specialized as trunk_chain_kernel (128-row tiles, each warpgroup on its own 64 rows a quarter of
// the columns at a time, the ring, register hand-back), with a quarter's mask words loaded before its MMAs.  Per quarter:
// MMAs (tc_gemm_nn's per output element), the mask (rows past M have no bits, so they are zero), the column sums'
// per-warp partials, the split, and from it the transposed image and the row image, which drain while the next
// quarter's MMAs run.  After quarter 3 the warpgroup writes the four splits over its rows of the layer's input in the
// activation buffer (not after layer 1), fences them and meets its own 4 warps at a named barrier; then come the column
// sums' atomics (one per column per 64 rows) and quarter 3's global stores.  The values and the images' bytes are
// tc_gemm_nn's; the column sums add 64-row blocks instead of 128-row tiles.
// DP: the activation buffer's and row images' passes (the input gradients'), TP: the transposed images' (the weight
// gradients'), TP <= DP.  DYN: c.M is a capacity, of which live_rows rows are computed.
template <int DP, int TP, bool DYN = false>
__global__ void __launch_bounds__(GEMM_THREADS, 1) dgrad_chain_kernel(const DgChain c, RowCount rc) {
  static_assert(TP <= DP, "the transposed images are written from the activation buffer's split");
  extern __shared__ __align__(1024) uint8_t smem[];
  const int M = (int)live_rows<DYN, false>(c.M, rc);
  if (DYN && M == 0) return;
  const int tiles = (M + CH_M - 1) / CH_M;
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + CH_BAR);
  uint64_t* empty = full + CH_STAGES;
  uint64_t* act_full = empty + CH_STAGES;
  uint64_t* act_empty = act_full + 1;
  // [2][8 warps][256 columns]: a layer's partials go to the other buffer than the previous layer's, so a warp that is
  // ahead never overwrites partials that the rest of its warpgroup has still to read
  float* red = reinterpret_cast<float*>(smem + CH_ENC);
  if (threadIdx.x == 0) {
    for (int i = 0; i < CH_STAGES; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], CONSUMERS / 32);
    }
    mbar_init(act_full, 1);
    mbar_init(act_empty, CONSUMERS / 32);
    asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
  }
  __syncthreads();
  if (threadIdx.x >= CONSUMERS) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;\n" ::: "memory");
    if (threadIdx.x == CONSUMERS) dg_produce<DP>(c, tiles, full, empty, act_full, act_empty);
    return;
  }
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;\n" ::: "memory");
  const int wg = threadIdx.x >> 7, w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // r: layers run, for the column sums' buffer
  int it = 0, n = 0, r = 0;
  for (int t = blockIdx.x; t < tiles; t += gridDim.x) {
    mbar_wait(act_full, n & 1);
    ++n;
    for (int l = c.top; l >= 1; --l, ++r) {
      float* rb = red + (r & 1) * (CONSUMERS / 32) * CH_W;
      uint16_t* row = c.row[l] ? c.row[l] + (size_t)t * CH_KS * 2 * TILE_ELEMS : nullptr;
      ChainSplit<DP> held[CH_Q - 1];
#pragma unroll
      for (int q = 0; q < CH_Q; ++q) {
        uint2 wd[2];
        dg_mask_words(wd, c.bits[l], M, t, q);
        float acc[32];
        chain_mma<false, DP>(acc, CH_KS, CH_KS, it, full, empty);
        if (q == CH_Q - 1 && l == 1 && lane == 0) mbar_arrive(act_empty);
        const uint32_t wds[2][2] = {{wd[0].x, wd[0].y}, {wd[1].x, wd[1].y}};
#pragma unroll
        for (int i = 0; i < 32; i += 2) {     // columns 8 j + 2 (lane % 4) + {0, 1} of word j / 4, j = i / 4
          const int j = i >> 2;
          const uint32_t k = wds[(i >> 1) & 1][j >> 2] >> (8 * (j & 3) + 2 * (lane & 3));
          if (!(k & 1)) acc[i] = 0.f;
          if (!(k & 2)) acc[i + 1] = 0.f;
        }
        // column sums as tile_colsum's: over the 16 rows of each warp (shuffles), then its warpgroup's 4 warps
#pragma unroll
        for (int j = 0; j < 8; ++j)
#pragma unroll
          for (int cc = 0; cc < 2; ++cc) {
            float s = acc[4 * j + cc] + acc[4 * j + 2 + cc];
#pragma unroll
            for (int o = 4; o < 32; o <<= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
            if (lane < 4) rb[w * CH_W + q * 64 + 8 * j + 2 * lane + cc] = s;
          }
        ChainSplit<DP> s;
        chain_split<false, DP>(acc, s);
        if (q == CH_Q - 1) {    // every MMA on this warpgroup's rows of G[l] has retired
          if (l > 1) {
            uint16_t* buf = reinterpret_cast<uint16_t*>(smem);
#pragma unroll
            for (int p = 0; p < CH_Q - 1; ++p) chain_put<DP>(held[p], p, buf, 2 * TILE_ELEMS, TILE_ELEMS);
            chain_put<DP>(s, q, buf, 2 * TILE_ELEMS, TILE_ELEMS);
            fence_proxy_async();
          }
          warpgroup_sync();     // the warpgroup's partials are in rb, its split in the activation buffer
#pragma unroll
          for (int i = 0; i < CH_W / 128; ++i) {
            const int col = (threadIdx.x & 127) + 128 * i;
            float sum = 0.f;
#pragma unroll
            for (int k = 0; k < 4; ++k) sum += rb[(4 * wg + k) * CH_W + col];
            atomicAdd(c.db[l] + col, sum);
          }
        } else if (l > 1) {
#pragma unroll
          for (int i = 0; i < (DP == 3 ? 32 : 16); ++i) held[q][i] = s[i];
        }
        dg_put_tr<TP, DP>(s, q, c.tr[l], c.tr_ks, t);
        if (row) chain_put<DP>(s, q, row, 2 * TILE_ELEMS, TILE_ELEMS);
      }
    }
  }
}

template <int DP, int TP>
static int launch_dgrad_chain(const DgChain& c, int ctas, RowCount rc, cudaStream_t st) {
  auto kernel = rc.rows ? dgrad_chain_kernel<DP, TP, true> : dgrad_chain_kernel<DP, TP>;
  SPARF_CHECK_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, CH_SMEM));
  kernel<<<std::min(ceil_div(c.M, CH_M), ctas), GEMM_THREADS, CH_SMEM, st>>>(c, rc);
  SPARF_CHECK_LAUNCH("dgrad_chain_kernel");
  return SPARF_OK;
}

template <bool F16, int PASSES, bool KFAST, class F, bool DYN = false, bool QUARTERS = false>
static int launch_pack(F f, int rtiles, int ksteps, uint16_t* img, cudaStream_t st, RowCount rc = {nullptr, 0}) {
  pack_kernel<F16, PASSES, KFAST, F, DYN, QUARTERS><<<dim3(ksteps, rtiles), 256, 0, st>>>(f, ksteps, img, rc);
  SPARF_CHECK_LAUNCH("pack_kernel");
  return SPARF_OK;
}

// a fused chain's weight image: CH_W rows of B in quarters (pack_kernel's QUARTERS layout)
template <bool KFAST, class F>
static int pack_chain_weights(const TcPrec& p, F f, int ksteps, uint16_t* img, cudaStream_t st) {
  constexpr int RT = CH_W / TM;
  return p.f16 ? (p.passes == 3 ? launch_pack<true, 3, KFAST, F, false, true>(f, RT, ksteps, img, st)
                                : launch_pack<true, 1, KFAST, F, false, true>(f, RT, ksteps, img, st))
               : (p.passes == 3 ? launch_pack<false, 3, KFAST, F, false, true>(f, RT, ksteps, img, st)
                                : launch_pack<false, 1, KFAST, F, false, true>(f, RT, ksteps, img, st));
}

template <bool F16, int PASSES, bool F32, int ROWP, int TRP>
static int launch_gemm(const Opnd& a, const Opnd& b, const Units& w, int ctas, const Epi& e, RowCount rc, cudaStream_t st) {
  auto kernel = rc.rows ? wg_gemm_kernel<F16, PASSES, F32, ROWP, TRP, true> : wg_gemm_kernel<F16, PASSES, F32, ROWP, TRP>;
  if (rc.start) {       // the span forward: only GEMMs with an fp32 output (into the tape) take global rows
    if constexpr (F32) {
      kernel = wg_gemm_kernel<F16, PASSES, F32, ROWP, TRP, true, true>;
    } else {
      set_error("a GEMM without an fp32 output takes no row start");
      return SPARF_ERR_UNSUPPORTED;
    }
  }
  SPARF_CHECK_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, GEMM_SMEM));
  kernel<<<std::min(w.tiles * w.nsplit, ctas), GEMM_THREADS, GEMM_SMEM, st>>>(a, b, w, e, rc);
  SPARF_CHECK_LAUNCH("wg_gemm_kernel");
  return SPARF_OK;
}

static int gemm_ctas(const TcPrec& p) { return p.max_ctas > 0 ? std::min(p.max_ctas, num_sms()) : num_sms(); }  // one CTA fills an SM

// The units of a GEMM over (B row tiles x A row tiles) output tiles.  split_k: each output tile's k-steps are shared out
// in about ceil(CTAs / output tiles) ranges per 1024 k-steps (32 768 rows; atomic epilogues only), so every CTA does one
// long reduction per 32 768 rows: no accumulator chain gets longer than at 32 768 rows, whatever the chunk size, so the
// rounding of the sums does not grow with it.
static Units gemm_units(int rta, int rtb, int ksteps, bool split_k, int ctas) {
  Units w{rtb, rta * rtb, 1, ksteps};
  if (split_k) w.nsplit = std::max(1, std::min(ksteps, ceil_div(ctas, w.tiles) * ceil_div(ksteps, 1024)));
  return w;
}

// pack B into p.pack_b, then the persistent GEMM over its units (gemm_units) with the epilogue outputs e asks for: fp32
// (e.out), a row image (row image passes = the GEMM's), a transposed image
template <bool F16, int PASSES, bool BK, class FB>
static int run(const TcPrec& p, const Opnd& a, int a_rows, FB fb, int b_rows, int ksteps, bool split_k, const Epi& e,
               int row_passes, int tr_passes, cudaStream_t st) {
  const int rta = ceil_div(a_rows, TM), rtb = ceil_div(b_rows, TM);
  SPARF_REQUIRE(p.pack_b && (size_t)rtb * ksteps * 2 * TILE_ELEMS <= p.pack_elems,
                "tc gemm: B operand image needs %zu 16-bit elements, have %zu", (size_t)rtb * ksteps * 2 * TILE_ELEMS,
                p.pack_elems);
  SPARF_TRY((launch_pack<F16, PASSES, BK>(fb, rtb, ksteps, p.pack_b, st)));
  const Opnd b{p.pack_b, nullptr, ksteps, 0};
  const int ctas = gemm_ctas(p);
  const Units w = gemm_units(rta, rtb, ksteps, split_k, ctas);
  const bool f32 = e.out != nullptr;
  const RowCount rc = p.rows;
  SPARF_REQUIRE(!rc.rows || !split_k, "tc gemm: a device row count needs the staged weight-gradient GEMM");
  if (f32 && !row_passes && !tr_passes) return launch_gemm<F16, PASSES, true, 0, 0>(a, b, w, ctas, e, rc, st);
  if (f32 && row_passes == PASSES && !tr_passes) return launch_gemm<F16, PASSES, true, PASSES, 0>(a, b, w, ctas, e, rc, st);
  if (!f32 && row_passes == PASSES && tr_passes == 3) return launch_gemm<F16, PASSES, false, PASSES, 3>(a, b, w, ctas, e, rc, st);
  if (!f32 && row_passes == PASSES && tr_passes == 1) return launch_gemm<F16, PASSES, false, PASSES, 1>(a, b, w, ctas, e, rc, st);
  SPARF_REQUIRE(false, "tc gemm: no kernel for fp32 output %d, row image %d passes, transposed image %d passes", (int)f32,
                row_passes, tr_passes);
}

// X (div = 1) as a 2D tensor of x.M rows by x.K fp32 columns, row pitch ldx, read in boxes of one k-step's 32 rows by
// 128 columns; zeros outside the tensor
static int staged_tensor_map(const Staged& x, CUtensorMap* map) {
  static PFN_cuTensorMapEncodeTiled_v12000 encode = nullptr;
  if (!encode) {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult q;
    SPARF_CHECK_CUDA(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q));
    SPARF_REQUIRE(fn && q == cudaDriverEntryPointSuccess, "tc_gemm_tn: the driver has no cuTensorMapEncodeTiled");
    encode = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(fn);
  }
  const cuuint64_t dims[2] = {(cuuint64_t)x.K, (cuuint64_t)x.M}, pitch[1] = {(cuuint64_t)x.ldx * 4};
  const cuuint32_t box[2] = {TM, TK}, step[2] = {1, 1};
  const CUresult r = encode(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(x.X), dims, pitch, box, step,
                            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  SPARF_REQUIRE(r == CUDA_SUCCESS, "tc_gemm_tn: cuTensorMapEncodeTiled failed (%d)", (int)r);
  return SPARF_OK;
}

// the weight-gradient GEMM with B = x read as fp32 (no pack), N output rows, over the k-steps of gt
template <int PASSES>
static int run_staged(const TcPrec& p, const Opnd& gt, int N, const Staged& x, int ksteps, const Epi& e, cudaStream_t st) {
  CUtensorMap xmap{};
  if (x.div == 1 && x.M > 0) SPARF_TRY(staged_tensor_map(x, &xmap));
  const int ctas = gemm_ctas(p);
  const Units w = gemm_units(ceil_div(N, TM), ceil_div(x.K, TM), ksteps, true, ctas);
  auto kernel = p.rows.rows ? wg_gemm_staged_kernel<PASSES, true> : wg_gemm_staged_kernel<PASSES>;
  SPARF_CHECK_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, STAGED_SMEM));
  kernel<<<std::min(w.tiles * w.nsplit, ctas), STAGED_THREADS, STAGED_SMEM, st>>>(gt, x, w, e, p.rows, ctas, xmap);
  SPARF_CHECK_LAUNCH("wg_gemm_staged_kernel");
  return SPARF_OK;
}

static Opnd opnd(const TcImage& x, const TcImage& y = TcImage{}) { return Opnd{x.p, y.p, x.ks, y.ks}; }

// the image outputs of an epilogue; they need the full k-range and no accumulation
static int set_images(Epi& e, const TcOut& o, int M, int N) {
  SPARF_REQUIRE(!e.accumulate || (!o.row_passes && !o.tr_passes), "tc gemm: images of an accumulated output");
  SPARF_REQUIRE(!o.row_passes || (o.row.p && o.row.ks == ceil_div(N, TK)), "tc gemm: row image needs %d k-steps",
                ceil_div(N, TK));
  SPARF_REQUIRE(!o.tr_passes || (o.tr.p && o.tr.ks == ceil_div(M, TK)), "tc gemm: transposed image needs %d k-steps",
                ceil_div(M, TK));
  e.row = o.row.p; e.row_ks = o.row.ks;
  e.tr = o.tr.p; e.tr_ks = o.tr.ks;
  return SPARF_OK;
}

}  // namespace

#define SPARF_WG_RUN(BK, ...)                                                                   \
  (p.f16 ? (p.passes == 3 ? run<true, 3, BK>(__VA_ARGS__) : run<true, 1, BK>(__VA_ARGS__))       \
         : (p.passes == 3 ? run<false, 3, BK>(__VA_ARGS__) : run<false, 1, BK>(__VA_ARGS__)))
#define SPARF_WG_PACK(KFAST, ...)                                                                                 \
  (p.f16 ? (p.passes == 3 ? launch_pack<true, 3, KFAST>(__VA_ARGS__) : launch_pack<true, 1, KFAST>(__VA_ARGS__)) \
         : (p.passes == 3 ? launch_pack<false, 3, KFAST>(__VA_ARGS__) : launch_pack<false, 1, KFAST>(__VA_ARGS__)))

size_t tc_image_elems(int rows, int cols) { return (size_t)ceil_div(rows, TM) * ceil_div(cols, TK) * 2 * TILE_ELEMS; }

size_t tc_pack_elems(int rows, int ksteps_rows, int cols) {
  // an image of max(rows, cols) rounded to row tiles x ksteps_rows k-steps (callers pass their largest GEMM)
  return (size_t)ceil_div(std::max(rows, cols), TM) * ksteps_rows * 2 * TILE_ELEMS;
}

int tc_pack_rows(TcPrec p, int M, int K, const float* X, int ldx, int div, TcImage img, cudaStream_t st) {
  SPARF_REQUIRE((p.passes == 1 || p.passes == 3) && img.p && img.ks == ceil_div(K, TK), "tc_pack_rows: passes=%d ks=%d K=%d",
                p.passes, img.ks, K);
  if (p.rows.rows) {
    const Rows f{X, ldx, K, div, M};
    return p.f16 ? (p.passes == 3 ? launch_pack<true, 3, true, Rows, true>(f, ceil_div(M, TM), img.ks, img.p, st, p.rows)
                                  : launch_pack<true, 1, true, Rows, true>(f, ceil_div(M, TM), img.ks, img.p, st, p.rows))
                 : (p.passes == 3 ? launch_pack<false, 3, true, Rows, true>(f, ceil_div(M, TM), img.ks, img.p, st, p.rows)
                                  : launch_pack<false, 1, true, Rows, true>(f, ceil_div(M, TM), img.ks, img.p, st, p.rows));
  }
  return SPARF_WG_PACK(true, Rows{X, ldx, K, div, M}, ceil_div(M, TM), img.ks, img.p, st);
}

int tc_pack_cols(TcPrec p, int M, int N, const float* X, int ldx, TcImage img, cudaStream_t st) {
  SPARF_REQUIRE((p.passes == 1 || p.passes == 3) && img.p && img.ks == ceil_div(M, TK), "tc_pack_cols: passes=%d ks=%d M=%d",
                p.passes, img.ks, M);
  return SPARF_WG_PACK(false, Cols{X, ldx, M, N}, ceil_div(N, TM), img.ks, img.p, st);
}

int tc_gemm_nt(TcPrec p, int act, int M, int N, TcImage a1, int K1v, TcImage a2, int K2v, const float* W, int ldw, int wcol2,
               const float* bias, float* Y, int ldy, const TcOut& out, cudaStream_t st) {
  SPARF_REQUIRE((p.passes == 1 || p.passes == 3) && (act == 0 || act == 1) && Y, "tc_gemm_nt: passes=%d act=%d", p.passes, act);
  const int ks = a1.ks + (a2.p ? a2.ks : 0);
  Epi e{};
  e.kind = 0; e.M = M; e.N = N; e.act = act; e.bias = bias; e.out = Y; e.ldo = ldy;
  e.pairs = N % 2 == 0 && pair_aligned(Y, ldy);
  SPARF_TRY(set_images(e, out, M, N));
  return SPARF_WG_RUN(true, p, opnd(a1, a2.p ? a2 : TcImage{}), M, NtB{W, ldw, wcol2, K1v, K2v, N, a1.ks}, N, ks, false, e,
                      out.row_passes, out.tr_passes, st);
}

bool tc_chain_supported(int W, int E3p, int nt, int skip) {
  return W == CH_W && E3p <= CH_ENC_KS * TK && nt >= 3 && nt <= SPARF_MAX_TRUNK && skip != 0 && skip < nt;
}

int tc_chain_ksteps(int l, int skip, int E3p) { return chain_ks(l, skip, ceil_div(E3p, TK)); }

int tc_pack_nt(TcPrec p, int N, int ks1, int K1v, int ks2, int K2v, const float* W, int ldw, int wcol2, TcImage img,
               cudaStream_t st) {
  SPARF_REQUIRE((p.passes == 1 || p.passes == 3) && N == CH_W && img.p && img.ks == ks1 + ks2,
                "tc_pack_nt: passes=%d N=%d ks=%d, %d + %d k-steps", p.passes, N, img.ks, ks1, ks2);
  return pack_chain_weights<true>(p, NtB{W, ldw, wcol2, K1v, K2v, N, ks1}, img.ks, img.p, st);
}

int tc_pack_nn(TcPrec p, int Kout, int N, int Kv, const float* W, int ldw, int wcol, TcImage img, cudaStream_t st) {
  SPARF_REQUIRE((p.passes == 1 || p.passes == 3) && Kout == CH_W && img.p && img.ks == ceil_div(N, TK),
                "tc_pack_nn: passes=%d Kout=%d ks=%d N=%d", p.passes, Kout, img.ks, N);
  return pack_chain_weights<false>(p, NnB{W, ldw, wcol, Kv, N}, img.ks, img.p, st);
}

int tc_dgrad_chain(TcPrec dg, TcPrec wg, int M, int W, int top, TcImage in, const TcImage* wimg, const uint32_t* const* bits,
                   float* const* db, const TcImage* tr, const TcImage* row, cudaStream_t st) {
  SPARF_REQUIRE(!dg.f16 && !wg.f16 && M >= 1 && W == CH_W && top >= 1 && top < SPARF_MAX_TRUNK && in.p && in.ks == CH_KS,
                "tc_dgrad_chain: bf16 images, M=%d W=%d top=%d, input row image of %d k-steps", M, W, top, CH_KS);
  DgChain c{};
  c.M = M; c.top = top; c.tr_ks = ceil_div(M, TK); c.in = in.p;
  for (int l = 1; l <= top; ++l) {
    SPARF_REQUIRE(wimg[l].p && wimg[l].ks == CH_KS && bits[l] && !(reinterpret_cast<uintptr_t>(bits[l]) & 15) && db[l] &&
                      tr[l].p && tr[l].ks == c.tr_ks && (!row[l].p || row[l].ks == CH_KS),
                  "tc_dgrad_chain: layer %d: weight image of %d k-steps, 16-byte aligned mask bits, column sums, transposed "
                  "image of %d k-steps, row image of %d",
                  l, CH_KS, c.tr_ks, CH_KS);
    c.w[l] = wimg[l].p; c.bits[l] = bits[l]; c.db[l] = db[l]; c.tr[l] = tr[l].p; c.row[l] = row[l].p;
  }
  const int ctas = gemm_ctas(dg);
  if (dg.passes == 3 && wg.passes == 3) return launch_dgrad_chain<3, 3>(c, ctas, dg.rows, st);
  if (dg.passes == 3 && wg.passes == 1) return launch_dgrad_chain<3, 1>(c, ctas, dg.rows, st);
  if (dg.passes == 1 && wg.passes == 1) return launch_dgrad_chain<1, 1>(c, ctas, dg.rows, st);
  SPARF_REQUIRE(false, "tc_dgrad_chain: no kernel for %d-pass row and %d-pass transposed images", dg.passes, wg.passes);
}

int tc_trunk_chain(TcPrec p, int M, int W, int nt, int skip, TcImage enc, const TcImage* wimg, const float* const* bias,
                   float* const* H, uint32_t* const* bits, const TcOut& last, cudaStream_t st) {
  SPARF_REQUIRE((p.passes == 1 || p.passes == 3) && M >= 1 && enc.p && tc_chain_supported(W, enc.ks * TK, nt, skip),
                "tc_trunk_chain: passes=%d M=%d W=%d nt=%d skip=%d encoding k-steps %d", p.passes, M, W, nt, skip, enc.ks);
  Chain c{};
  c.M = M; c.skip = skip; c.enc_ks = enc.ks; c.enc = enc.p;
  c.nl = H[nt - 1] ? nt : nt - 1;       // without the last layer's output the chain ends at the density row's input
  SPARF_REQUIRE(H[c.nl - 1], "tc_trunk_chain: no output asked for");
  for (int l = 0; l < c.nl; ++l) {
    SPARF_REQUIRE(wimg[l].p && wimg[l].ks == chain_ks(l, skip, enc.ks) && bias[l] && !(reinterpret_cast<uintptr_t>(H[l]) & 7),
                  "tc_trunk_chain: layer %d: weight image of %d k-steps, bias, 8-byte aligned output", l,
                  chain_ks(l, skip, enc.ks));
    c.w[l] = wimg[l].p; c.bias[l] = bias[l]; c.H[l] = H[l];
    c.bits[l] = bits ? bits[l] : nullptr;
  }
  if (last.row_passes) {
    SPARF_REQUIRE(c.nl == nt && last.row_passes == p.passes && !last.tr_passes && last.row.p && last.row.ks == CH_KS,
                  "tc_trunk_chain: the last layer's row image takes the chain's passes and %d k-steps", CH_KS);
    c.last = last.row.p;
  }
  const int ctas = gemm_ctas(p);
  return p.f16 ? (p.passes == 3 ? launch_chain<true, 3>(c, ctas, p.rows, st) : launch_chain<true, 1>(c, ctas, p.rows, st))
               : (p.passes == 3 ? launch_chain<false, 3>(c, ctas, p.rows, st) : launch_chain<false, 1>(c, ctas, p.rows, st));
}

int tc_gemm_nn(TcPrec p, int M, int N, int Kout, int Kv, TcImage g, const float* W, int ldw, int wcol, const float* mask_src,
               int ldmask, const uint32_t* mask_bits, const float* r1_vec, const float* r1_row, float* D, int ldd,
               int accumulate, const TcOut& out, float* db, float* r1_wgrad, cudaStream_t st) {
  SPARF_REQUIRE((p.passes == 1 || p.passes == 3) && g.ks == ceil_div(N, TK), "tc_gemm_nn: passes=%d ks=%d N=%d", p.passes,
                g.ks, N);
  SPARF_REQUIRE(!r1_wgrad || (mask_src && r1_vec && !D), "tc_gemm_nn: r1_wgrad needs the mask source, r1_vec, no fp32 D");
  SPARF_REQUIRE(!mask_src || !mask_bits, "tc_gemm_nn: an fp32 mask or a bit mask, not both");
  SPARF_REQUIRE(!mask_bits || !D, "tc_gemm_nn: a bit mask needs image outputs only (no fp32 D)");
  Epi e{};
  e.kind = 1; e.M = M; e.N = Kout; e.out = D; e.ldo = ldd; e.Kv = Kv; e.mask = mask_src; e.ldmask = ldmask;
  if (mask_bits) {
    e.mask_bits = mask_bits;
    e.ldbits = ceil_div(Kout, 32);
  }
  e.r1_vec = r1_vec; e.r1_row = r1_row; e.accumulate = accumulate; e.colsum = db; e.r1_wgrad = r1_wgrad;
  e.pairs = Kout % 2 == 0 && pair_aligned(D, ldd) && pair_aligned(mask_src, ldmask);
  SPARF_REQUIRE(!db || !accumulate, "tc_gemm_nn: column sums of an accumulated output");
  SPARF_TRY(set_images(e, out, M, Kout));
  return SPARF_WG_RUN(false, p, opnd(g), M, NnB{W, ldw, wcol, Kv, N}, Kout, g.ks, false, e, out.row_passes, out.tr_passes, st);
}

int tc_gemm_tn(TcPrec p, int M, int N, int K, int Kv, TcImage gt, const float* X, int ldx, int div, float* dW, int ldw,
               int wcol, uint32_t* bits, cudaStream_t st) {
  SPARF_REQUIRE((p.passes == 1 || p.passes == 3) && gt.ks == ceil_div(M, TK), "tc_gemm_tn: passes=%d ks=%d", p.passes, gt.ks);
  Epi e{};
  e.kind = 2; e.M = N; e.N = K; e.out = dW; e.ldo = ldw; e.col_off = wcol; e.Kv = Kv;
  // rows of X that bulk copies can read (16-byte aligned), which every engine call has: B is split inside the GEMM
  if (!(reinterpret_cast<uintptr_t>(X) & 15) && ldx % 4 == 0 && K % 4 == 0) {
    SPARF_REQUIRE(!p.f16, "tc_gemm_tn: bf16 halves only");
    const Staged x{X, ldx, div, M, K, bits, ceil_div(K, 32)};
    return p.passes == 3 ? run_staged<3>(p, opnd(gt), N, x, gt.ks, e, st) : run_staged<1>(p, opnd(gt), N, x, gt.ks, e, st);
  }
  SPARF_REQUIRE(!p.rows.rows, "tc_gemm_tn: a device row count needs X 16-byte aligned with ldx and K multiples of 4");
  return SPARF_WG_RUN(false, p, opnd(gt), N, TnB{X, ldx, div, M, K, bits, ceil_div(K, 32)}, K, gt.ks, true, e, 0, 0, st);
}

template <int ROWP, int TRP>
static int launch_head_bwd(const HeadBwd& h, RowCount rc, cudaStream_t st) {
  auto kernel = rc.rows ? head_bwd_kernel<ROWP, TRP, true> : head_bwd_kernel<ROWP, TRP>;
  SPARF_CHECK_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, HEAD_SMEM));
  kernel<<<ceil_div(h.M, TM), 256, HEAD_SMEM, st>>>(h, rc);
  SPARF_CHECK_LAUNCH("head_bwd_kernel");
  return SPARF_OK;
}

int tc_head_backward(TcPrec dg, TcPrec wg, int M, int HW, const float* d_rgb, const float* rgb, const float* d_sigma,
                     const float* raw, const float* hid, const float* W9, float* graw, TcImage row, TcImage tr, float* dW9,
                     float* db9, float* db_hid, float* db_raw, cudaStream_t st) {
  SPARF_REQUIRE(!dg.f16 && !wg.f16 && (dg.passes == 1 || dg.passes == 3) && (wg.passes == 1 || wg.passes == 3),
                "tc_head_backward: bf16 1- or 3-pass images only");
  SPARF_REQUIRE(M >= 1 && HW % 4 == 0 && !(reinterpret_cast<uintptr_t>(hid) & 15), "tc_head_backward: M=%d HW=%d", M, HW);
  SPARF_REQUIRE(row.p && row.ks == ceil_div(HW, TK) && tr.p && tr.ks == ceil_div(M, TK),
                "tc_head_backward: images need %d and %d k-steps", ceil_div(HW, TK), ceil_div(M, TK));
  const HeadBwd h{M, HW, d_rgb, rgb, d_sigma, raw, hid, W9, graw, row.p, tr.p, row.ks, tr.ks, dW9, db9, db_hid, db_raw};
  if (dg.passes == 3 && wg.passes == 3) return launch_head_bwd<3, 3>(h, dg.rows, st);
  if (dg.passes == 3 && wg.passes == 1) return launch_head_bwd<3, 1>(h, dg.rows, st);
  if (dg.passes == 1 && wg.passes == 1) return launch_head_bwd<1, 1>(h, dg.rows, st);
  SPARF_REQUIRE(false, "tc_head_backward: no kernel for %d-pass row and %d-pass transposed images", dg.passes, wg.passes);
}

template <int ROWP, int TRP>
static int launch_feat_bwd(const FeatBwd& f, cudaStream_t st) {
  auto kernel = feat_bwd_kernel<ROWP, TRP>;
  SPARF_CHECK_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, FEAT_SMEM));
  kernel<<<ceil_div(f.M, TM), 256, FEAT_SMEM, st>>>(f);
  SPARF_CHECK_LAUNCH("feat_bwd_kernel");
  return SPARF_OK;
}

int tc_feat_backward(TcPrec dg, TcPrec wg, int M, int W, const float* d_raw, const float* d_feat, const float* feat,
                     TcImage row, TcImage tr, float* db_raw, float* db_feat, cudaStream_t st) {
  SPARF_REQUIRE(!dg.f16 && !wg.f16 && (dg.passes == 1 || dg.passes == 3) && (wg.passes == 1 || wg.passes == 3),
                "tc_feat_backward: bf16 1- or 3-pass images only");
  SPARF_REQUIRE(M >= 1 && W % 4 == 0 && (!d_feat || (feat && !(reinterpret_cast<uintptr_t>(feat) & 15))),
                "tc_feat_backward: M=%d W=%d", M, W);
  SPARF_REQUIRE(row.p && row.ks == ceil_div(W, TK) && tr.p && tr.ks == ceil_div(M, TK),
                "tc_feat_backward: images need %d and %d k-steps", ceil_div(W, TK), ceil_div(M, TK));
  const FeatBwd f{M, W, d_raw, d_feat, feat, row.p, tr.p, row.ks, tr.ks, db_raw, db_feat,
                  !(reinterpret_cast<uintptr_t>(d_feat) & 15)};
  if (dg.passes == 3 && wg.passes == 3) return launch_feat_bwd<3, 3>(f, st);
  if (dg.passes == 3 && wg.passes == 1) return launch_feat_bwd<3, 1>(f, st);
  if (dg.passes == 1 && wg.passes == 1) return launch_feat_bwd<1, 1>(f, st);
  SPARF_REQUIRE(false, "tc_feat_backward: no kernel for %d-pass row and %d-pass transposed images", dg.passes, wg.passes);
}

}  // namespace sparf

using namespace sparf;

// scratch operand images for the self-tests (diagnostics only: allocated and freed on the stream)
static int alloc_images(size_t elems, cudaStream_t st, TcPrec& p) {
  SPARF_CHECK_CUDA(cudaMallocAsync(reinterpret_cast<void**>(&p.pack_a), elems * 2, st));
  SPARF_CHECK_CUDA(cudaMallocAsync(reinterpret_cast<void**>(&p.pack_b), elems * 2, st));
  p.pack_elems = elems;
  return SPARF_OK;
}

static void free_images(TcPrec& p, cudaStream_t st) {
  cudaFreeAsync(p.pack_a, st);
  cudaFreeAsync(p.pack_b, st);
}

// Exact-integer checks of the operand images, descriptors, the copy ring and the fragment mapping (small integers are
// exact in bf16 and their dot products exact in fp32).  A [128,K], B [128,K] fp32 row-major, K in {64,...,256}: D = A B^T.
extern "C" int sparf_tc_selftest(const float* A, const float* B, int32_t K, void* packed, float* D, sparf_stream_t stream) {
  (void)packed;
  SPARF_REQUIRE(K % 64 == 0 && K >= 64 && K <= 256, "tc_selftest: K=%d", K);
  cudaStream_t st = (cudaStream_t)stream;
  TcPrec p{false, 1};
  SPARF_TRY(alloc_images(tc_pack_elems(128, K / 32, 128), st, p));
  const TcImage a{p.pack_a, K / 32};
  int rc = tc_pack_rows(p, 128, K, A, K, 1, a, st);
  if (!rc) rc = tc_gemm_nt(p, 0, 128, 128, a, K, TcImage{}, 0, B, K, 0, nullptr, D, 128, TcOut{}, st);
  free_images(p, st);
  return rc;
}

// D[128,128] = G^T X, G and X [rows, 128] fp32 row-major (the weight-gradient contraction over rows)
extern "C" int sparf_tc_selftest_tn(const float* G, const float* X, int32_t rows, float* D, sparf_stream_t stream) {
  SPARF_REQUIRE(rows == 64 || rows == 128, "tc_selftest_tn: rows=%d", rows);
  cudaStream_t st = (cudaStream_t)stream;
  SPARF_CHECK_CUDA(cudaMemsetAsync(D, 0, 128 * 128 * sizeof(float), st));
  TcPrec p{false, 1};
  SPARF_TRY(alloc_images(tc_pack_elems(128, rows / 32, 128), st, p));
  const TcImage gt{p.pack_a, rows / 32};
  int rc = tc_pack_cols(p, rows, 128, G, 128, gt, st);
  if (!rc) rc = tc_gemm_tn(p, rows, 128, 128, 128, gt, X, 128, 1, D, 128, 0, nullptr, st);
  free_images(p, st);
  return rc;
}

// The epilogue images, chained through three 3-pass bf16 GEMMs (exact on small integers):
//   D = X W1 (X [M,128], W1 [128,96]; the input-gradient GEMM), written only as a row image, a transposed image and its
//       column sums db[96];
//   Y = [D | E] W2^T (E [M,40], W2 [128,136]): the row image as the first segment of a two-segment A operand;
//   Z = D^T X [96,128]: the transposed image as the weight-gradient A operand, its rows split into k-ranges.
// The image buffers start as NaN, so a k-step past M that is not zero-padded shows in Z.  max_ctas > 0 caps the GEMM
// grids (else they take one CTA per SM), so that CTAs take several units and the copy ring wraps across them.
static int selftest_images(const float* X, const float* W1, const float* E, const float* W2, int M, float* Y, float* Z,
                           float* db, int max_ctas, cudaStream_t st) {
  SPARF_REQUIRE(M >= 1 && M <= 1024, "tc_selftest_images: M=%d", M);
  const int N = 128, K = 96, KE = 40;
  TcPrec q{false, 3};
  q.max_ctas = max_ctas;
  const TcImage x{nullptr, N / TK}, d{nullptr, K / TK}, e{nullptr, ceil_div(KE, TK)}, dt{nullptr, ceil_div(M, TK)};
  const size_t nx = tc_image_elems(M, N), nd = tc_image_elems(M, K), ne = tc_image_elems(M, KE), ndt = tc_image_elems(K, M);
  SPARF_TRY(alloc_images(nx + nd + ne + ndt + tc_pack_elems(std::max(M, N), ceil_div(K + KE, TK), 0), st, q));
  TcImage xi = x, di = d, ei = e, dti = dt;
  xi.p = q.pack_a; di.p = xi.p + nx; ei.p = di.p + nd; dti.p = ei.p + ne;
  SPARF_CHECK_CUDA(cudaMemsetAsync(q.pack_a, 0xFF, (nx + nd + ne + ndt) * 2, st));
  SPARF_CHECK_CUDA(cudaMemsetAsync(db, 0, K * sizeof(float), st));
  SPARF_CHECK_CUDA(cudaMemsetAsync(Z, 0, K * N * sizeof(float), st));
  TcOut o;
  o.row = di; o.row_passes = 3;
  o.tr = dti; o.tr_passes = 3;
  int rc = tc_pack_rows(q, M, N, X, N, 1, xi, st);
  if (!rc)
    rc = tc_gemm_nn(q, M, N, K, K, xi, W1, K, 0, nullptr, 0, nullptr, nullptr, nullptr, nullptr, 0, 0, o, db, nullptr, st);
  if (!rc) rc = tc_pack_rows(q, M, KE, E, KE, 1, ei, st);
  if (!rc) rc = tc_gemm_nt(q, 0, M, 128, di, K, ei, KE, W2, K + KE, K, nullptr, Y, 128, TcOut{}, st);
  if (!rc) rc = tc_gemm_tn(q, M, K, N, N, dti, X, N, 1, Z, N, 0, nullptr, st);
  free_images(q, st);
  return rc;
}

extern "C" int sparf_tc_selftest_images(const float* X, const float* W1, const float* E, const float* W2, int32_t M, float* Y,
                                        float* Z, float* db, sparf_stream_t stream) {
  return selftest_images(X, W1, E, W2, M, Y, Z, db, 0, (cudaStream_t)stream);
}

static int selftest_wgrad(const float* G, const float* X, int M, int N, int K, int Kv, int ldx, int div, int passes,
                          int max_ctas, const int64_t* rows, float* dW, uint32_t* bits, cudaStream_t st) {
  SPARF_REQUIRE(M >= 1 && M <= (1 << 20) && N >= 1 && N <= 512 && K >= 1 && K <= 512 && Kv >= 0 && Kv <= K && ldx >= K &&
                    div >= 1 && (passes == 1 || passes == 3),
                "tc_selftest_wgrad: M=%d N=%d K=%d Kv=%d ldx=%d div=%d passes=%d", M, N, K, Kv, ldx, div, passes);
  SPARF_REQUIRE(G && X && dW, "tc_selftest_wgrad: NULL tensor");
  SPARF_CHECK_CUDA(cudaMemsetAsync(dW, 0, (size_t)N * K * sizeof(float), st));
  TcPrec p{false, passes};
  p.max_ctas = max_ctas;
  SPARF_TRY(alloc_images(std::max(tc_image_elems(N, M), tc_pack_elems(K, ceil_div(M, TK), 0)), st, p));
  const TcImage gt{p.pack_a, ceil_div(M, TK)};
  int rc = tc_pack_cols(p, M, N, G, N, gt, st);
  p.rows = RowCount{rows, 0};
  if (!rc) rc = tc_gemm_tn(p, M, N, K, Kv, gt, X, ldx, div, dW, K, 0, bits, st);
  free_images(p, st);
  return rc;
}

extern "C" int sparf_tc_selftest_wgrad(const float* G, const float* X, int32_t M, int32_t N, int32_t K, int32_t Kv, int32_t ldx,
                                       int32_t div, int32_t passes, int32_t max_ctas, float* dW, uint32_t* bits,
                                       sparf_stream_t stream) {
  return selftest_wgrad(G, X, M, N, K, Kv, ldx, div, passes, max_ctas, nullptr, dW, bits, (cudaStream_t)stream);
}

extern "C" int sparf_tc_selftest_wgrad_rows(const float* G, const float* X, int32_t M, int32_t N, int32_t K, int32_t Kv,
                                            int32_t ldx, int32_t div, int32_t passes, int32_t max_ctas, const int64_t* rows,
                                            float* dW, uint32_t* bits, sparf_stream_t stream) {
  SPARF_REQUIRE(rows, "tc_selftest_wgrad_rows: NULL row count");
  return selftest_wgrad(G, X, M, N, K, Kv, ldx, div, passes, max_ctas, rows, dW, bits, (cudaStream_t)stream);
}

extern "C" int sparf_tc_selftest_mask_bits(const float* G, const float* W, const float* X, int32_t M, int32_t N, int32_t K,
                                           int32_t max_ctas, uint16_t* img, sparf_stream_t stream) {
  SPARF_REQUIRE(M >= 1 && M <= (1 << 20) && N >= 1 && N <= 512 && K >= 2 && K <= 512 && K % 2 == 0,
                "tc_selftest_mask_bits: M=%d N=%d K=%d", M, N, K);
  SPARF_REQUIRE(G && W && X && img, "tc_selftest_mask_bits: NULL tensor");
  cudaStream_t st = (cudaStream_t)stream;
  TcPrec p{false, 3};
  p.max_ctas = max_ctas;
  const size_t ng = tc_image_elems(M, N), ngt = tc_image_elems(N, M);
  const size_t nrow = tc_image_elems(M, K), ntr = tc_image_elems(K, M);
  SPARF_TRY(alloc_images(ng + ngt + tc_pack_elems(K, ceil_div(M, TK) + ceil_div(N, TK), 0), st, p));
  uint32_t* bits = nullptr;
  float* dW = nullptr;
  const size_t nbits = (size_t)M * ceil_div(K, 32);
  SPARF_CHECK_CUDA(cudaMallocAsync(reinterpret_cast<void**>(&bits), nbits * 4 + (size_t)N * K * sizeof(float), st));
  dW = reinterpret_cast<float*>(bits + nbits);
  SPARF_CHECK_CUDA(cudaMemsetAsync(dW, 0, (size_t)N * K * sizeof(float), st));
  SPARF_CHECK_CUDA(cudaMemsetAsync(img, 0xFF, 2 * (nrow + ntr) * sizeof(uint16_t), st));
  const TcImage g{p.pack_a, ceil_div(N, TK)}, gt{p.pack_a + ng, ceil_div(M, TK)};
  TcOut o[2];
  for (int i = 0; i < 2; ++i) {
    o[i].row = TcImage{img + i * (nrow + ntr), ceil_div(K, TK)};
    o[i].tr = TcImage{img + i * (nrow + ntr) + nrow, ceil_div(M, TK)};
    o[i].row_passes = o[i].tr_passes = 3;
  }
  int rc = tc_pack_rows(p, M, N, G, N, 1, g, st);
  if (!rc) rc = tc_pack_cols(p, M, N, G, N, gt, st);
  if (!rc) rc = tc_gemm_tn(p, M, N, K, K, gt, X, K, 1, dW, K, 0, bits, st);
  if (!rc)
    rc = tc_gemm_nn(p, M, N, K, K, g, W, K, 0, X, K, nullptr, nullptr, nullptr, nullptr, 0, 0, o[0], nullptr, nullptr, st);
  if (!rc)
    rc = tc_gemm_nn(p, M, N, K, K, g, W, K, 0, nullptr, 0, bits, nullptr, nullptr, nullptr, 0, 0, o[1], nullptr, nullptr, st);
  cudaFreeAsync(bits, st);
  free_images(p, st);
  return rc;
}

extern "C" int sparf_tc_selftest_persistent(const float* X, const float* W1, const float* E, const float* W2, int32_t M,
                                            float* Y, float* Z, float* db, int32_t max_ctas, sparf_stream_t stream) {
  return selftest_images(X, W1, E, W2, M, Y, Z, db, max_ctas, (cudaStream_t)stream);
}

// The fused trunk forward (chain != 0) or the same layers through tc_gemm_nt chained by row images (chain == 0), width
// 256, on the same inputs: enc [M, E3p] (E3p = E3 rounded up to 32, zero padded), W = the layers' [256, ldw_l] weights one
// after another (ldw_l = (l == 0 ? E3 : 256) + (l == skip ? E3 : 0)), bias [nt, 256].  H [nt, M, 256]: layer l is written
// iff bit l of outputs; without bit nt-1 the last layer is not computed.  last (may be NULL): the last layer's row image.
// rows (may be NULL): M is a capacity, *rows the rows computed.  The two runs must give the same bytes.  bits (may be
// NULL; the chain only): [nt - 2][M][8] ReLU masks of layers 0 ... nt-3.
static int selftest_chain(const float* enc, int M, int E3, int nt, int skip, const float* W, const float* bias, int passes,
                          int f16, int max_ctas, int chain, uint32_t outputs, const int64_t* rows, float* H, uint16_t* last,
                          uint32_t* bits, cudaStream_t st) {
  SPARF_REQUIRE(enc && W && bias && H && M >= 1 && M <= (1 << 20) && E3 >= 1 && (passes == 1 || passes == 3),
                "tc_selftest_chain: M=%d E3=%d passes=%d", M, E3, passes);
  const int E3p = ceil_div(E3, TK) * TK, eks = E3p / TK;
  SPARF_REQUIRE(tc_chain_supported(CH_W, E3p, nt, skip) && (outputs >> (nt - 2) & 1), "tc_selftest_chain: nt=%d skip=%d", nt, skip);
  SPARF_REQUIRE(!bits || chain, "tc_selftest_chain: mask bits come from the chain only");
  TcPrec p{f16 != 0, passes};
  p.max_ctas = max_ctas;
  p.rows = RowCount{rows, 0};
  const bool feat = outputs >> (nt - 1) & 1;
  size_t wel = 0;
  for (int l = 0; l < nt; ++l) wel += tc_image_elems(CH_W, chain_ks(l, skip, eks) * TK);
  const size_t ne = tc_image_elems(M, E3p), nh = tc_image_elems(M, CH_W);
  SPARF_TRY(alloc_images(std::max(ne + 2 * nh, wel), st, p));
  float* scratch = nullptr;
  SPARF_CHECK_CUDA(cudaMallocAsync(reinterpret_cast<void**>(&scratch), (size_t)M * CH_W * sizeof(float), st));
  const TcImage ei{p.pack_a, eks}, himg[2] = {{p.pack_a + ne, CH_KS}, {p.pack_a + ne + nh, CH_KS}};
  TcOut lo;
  if (feat && last) {
    lo.row = TcImage{last, CH_KS};
    lo.row_passes = passes;
  }
  int rc = tc_pack_rows(p, M, E3p, enc, E3p, 1, ei, st);
  const float* Wl[SPARF_MAX_TRUNK];
  const float* bl[SPARF_MAX_TRUNK];
  float* Hl[SPARF_MAX_TRUNK];
  uint32_t* bl_bits[SPARF_MAX_TRUNK] = {};
  TcImage wimg[SPARF_MAX_TRUNK];
  size_t wo = 0, io = 0;
  for (int l = 0; l < nt; ++l) {
    Wl[l] = W + wo;
    bl[l] = bias + (size_t)l * CH_W;
    Hl[l] = outputs >> l & 1 ? H + (size_t)l * M * CH_W : nullptr;
    if (bits && l < nt - 2) bl_bits[l] = bits + (size_t)l * M * (CH_W / 32);
    wimg[l] = TcImage{p.pack_b + io, chain_ks(l, skip, eks)};
    wo += (size_t)CH_W * ((l == 0 ? E3 : CH_W) + (l == skip ? E3 : 0));
    io += tc_image_elems(CH_W, wimg[l].ks * TK);
  }
  if (chain) {
    for (int l = 0; l < nt && !rc; ++l)
      rc = tc_pack_nt(p, CH_W, l == 0 ? eks : CH_KS, l == 0 ? E3 : CH_W, l == skip ? eks : 0, E3, Wl[l],
                      (l == 0 ? E3 : CH_W) + (l == skip ? E3 : 0), CH_W, wimg[l], st);
    if (!rc) rc = tc_trunk_chain(p, M, CH_W, nt, skip, ei, wimg, bl, Hl, bl_bits, lo, st);
  } else {
    for (int l = 0; l < (feat ? nt : nt - 1) && !rc; ++l) {
      TcOut o;
      if (l < nt - 1) {
        o.row = himg[l & 1];
        o.row_passes = passes;
      } else {
        o = lo;
      }
      rc = tc_gemm_nt(p, 1, M, CH_W, l == 0 ? ei : himg[(l - 1) & 1], l == 0 ? E3 : CH_W, l == skip ? ei : TcImage{}, E3, Wl[l],
                      (l == 0 ? E3 : CH_W) + (l == skip ? E3 : 0), CH_W, bl[l], Hl[l] ? Hl[l] : scratch, CH_W, o, st);
    }
  }
  cudaFreeAsync(scratch, st);
  free_images(p, st);
  return rc;
}

extern "C" int sparf_tc_selftest_chain(const float* enc, int32_t M, int32_t E3, int32_t nt, int32_t skip, const float* W,
                                       const float* bias, int32_t passes, int32_t f16, int32_t max_ctas, int32_t chain,
                                       uint32_t outputs, const int64_t* rows, float* H, uint16_t* last,
                                       sparf_stream_t stream) {
  return selftest_chain(enc, M, E3, nt, skip, W, bias, passes, f16, max_ctas, chain, outputs, rows, H, last, nullptr,
                        (cudaStream_t)stream);
}

// The fused trunk forward with every output and the ReLU masks of layers 0 ... nt-3, bits [nt - 2][M][8]
extern "C" int sparf_tc_selftest_chain_bits(const float* enc, int32_t M, int32_t E3, int32_t nt, int32_t skip, const float* W,
                                            const float* bias, int32_t passes, int32_t f16, int32_t max_ctas,
                                            const int64_t* rows, float* H, uint32_t* bits, sparf_stream_t stream) {
  SPARF_REQUIRE(bits && nt >= 3 && nt <= SPARF_MAX_TRUNK, "tc_selftest_chain_bits: nt=%d, bits", nt);
  return selftest_chain(enc, M, E3, nt, skip, W, bias, passes, f16, max_ctas, 1, (1u << nt) - 1, rows, H, nullptr, bits,
                        (cudaStream_t)stream);
}

// The trunk backward's input gradients of layers nt-2 ... 1 through dgrad_chain_kernel (chain != 0) or layer by layer
// through tc_gemm_nn with bit masks (chain == 0), width 256, on the same inputs: G [M, 256] = G[nt-2] in fp32 (packed
// into its row image first), W as sparf_tc_selftest_chain's, bits [nt-2][M][8] the masks of H[0] ... H[nt-3].  Outputs:
// tr [nt-2] the transposed images of G[0] ... G[nt-3] (wg_passes), db [nt-2][256] their column sums, row (may be NULL)
// [2] the row images of G[0] and G[skip] (skip <= nt-3).  rows as sparf_tc_selftest_chain's.  The images must be the
// same bytes.
extern "C" int sparf_tc_selftest_dgrad_chain(const float* G, int32_t M, int32_t E3, int32_t nt, int32_t skip, const float* W,
                                             const uint32_t* bits, int32_t dg_passes, int32_t wg_passes, int32_t max_ctas,
                                             int32_t chain, const int64_t* rows, uint16_t* tr, uint16_t* row, float* db,
                                             sparf_stream_t stream) {
  SPARF_REQUIRE(G && W && bits && tr && db && M >= 1 && M <= (1 << 20) && E3 >= 1 && nt >= 3 && nt <= SPARF_MAX_TRUNK &&
                    skip > 0 && skip < nt && (!row || skip <= nt - 3),
                "tc_selftest_dgrad_chain: M=%d E3=%d nt=%d skip=%d", M, E3, nt, skip);
  cudaStream_t st = (cudaStream_t)stream;
  TcPrec dg{false, dg_passes}, wg{false, wg_passes};
  dg.max_ctas = wg.max_ctas = max_ctas;
  dg.rows = wg.rows = RowCount{rows, 0};
  const int top = nt - 2;
  const size_t nh = tc_image_elems(M, CH_W), ntr = tc_image_elems(CH_W, M), nw = tc_image_elems(CH_W, CH_W);
  SPARF_TRY(alloc_images(std::max(3 * nh, (top + 1) * nw), st, dg));
  SPARF_CHECK_CUDA(cudaMemsetAsync(db, 0, (size_t)top * CH_W * sizeof(float), st));
  const TcImage gin{dg.pack_a, CH_KS}, scratch[2] = {{dg.pack_a + nh, CH_KS}, {dg.pack_a + 2 * nh, CH_KS}};
  const float* Wl[SPARF_MAX_TRUNK];
  int ldw[SPARF_MAX_TRUNK];
  size_t wo = 0;
  for (int l = 0; l < nt; ++l) {
    Wl[l] = W + wo;
    ldw[l] = (l == 0 ? E3 : CH_W) + (l == skip ? E3 : 0);
    wo += (size_t)CH_W * ldw[l];
  }
  TcImage trl[SPARF_MAX_TRUNK], rowl[SPARF_MAX_TRUNK], wimg[SPARF_MAX_TRUNK];
  const uint32_t* bl[SPARF_MAX_TRUNK] = {};
  float* dbl[SPARF_MAX_TRUNK] = {};
  for (int l = 1; l <= top; ++l) {
    trl[l] = TcImage{tr + (size_t)(l - 1) * ntr, ceil_div(M, TK)};
    if (row && (l == 1 || l - 1 == skip)) rowl[l] = TcImage{row + (l == 1 ? 0 : nh), CH_KS};
    bl[l] = bits + (size_t)(l - 1) * M * (CH_W / 32);
    dbl[l] = db + (size_t)(l - 1) * CH_W;
    wimg[l] = TcImage{dg.pack_b + (size_t)l * nw, CH_KS};
  }
  int rc = tc_pack_rows(dg, M, CH_W, G, CH_W, 1, gin, st);
  if (chain) {
    for (int l = 1; l <= top && !rc; ++l) rc = tc_pack_nn(dg, CH_W, CH_W, CH_W, Wl[l], ldw[l], 0, wimg[l], st);
    if (!rc) rc = tc_dgrad_chain(dg, wg, M, CH_W, top, gin, wimg, bl, dbl, trl, rowl, st);
  } else {
    TcImage g = gin;
    for (int l = top; l >= 1 && !rc; --l) {
      TcOut o;
      o.row = rowl[l].p ? rowl[l] : scratch[l & 1];
      o.tr = trl[l];
      o.row_passes = dg_passes;
      o.tr_passes = wg_passes;
      rc = tc_gemm_nn(dg, M, CH_W, CH_W, CH_W, g, Wl[l], ldw[l], 0, nullptr, 0, bl[l], nullptr, nullptr, nullptr, 0, 0, o,
                      dbl[l], nullptr, st);
      g = o.row;
    }
  }
  free_images(dg, st);
  return rc;
}
