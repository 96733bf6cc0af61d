// wgmma GEMMs of the tensor-core MLP engines (SPARF_ENGINE_TC_3X / TC_1X / TC_3X_W1), sm_90a.
//
// Two kernels per GEMM:
//   pack: the fp32 operands (with the GEMM's own indexing: concatenated sources, transposes, per-ray rows, bounds) are
//     split once into 16-bit (hi, lo) halves and written as an image of [128 rows x 32 K] tiles, each tile already in the
//     canonical no-swizzle K-major shared-memory layout (8 x 8 core matrices of 128 contiguous bytes, core matrices
//     adjacent in K 128 B apart = leading byte offset, 8-row groups 512 B apart = stride byte offset), hi and lo halves of
//     a tile adjacent (16 KB);
//   gemm: one CTA = two warpgroups = one 128 x 128 output tile; one thread streams the tiles of both operands with
//     cp.async.bulk into a STAGES-deep ring of shared-memory stages, each completing on its own mbarrier (complete_tx);
//     both warpgroups wait on the stage's barrier and issue wgmma.m64n128k16 (register accumulators); one MMA group stays
//     in flight while the stage consumed before it is refilled, so STAGES - 1 tile copies overlap the MMAs.
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include <algorithm>

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

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;\n" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;\n" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;\n" ::: "memory"); }

// the lo halves are stored scaled by 2^LO_SHIFT (exact) so that they stay clear of the fp16 subnormal range; the products
// that carry one lo factor accumulate separately and are scaled back once at the end
constexpr int LO_SHIFT = 11;

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
constexpr int STAGES = 4;
constexpr int STAGE_BYTES = 4 * TILE_BYTES;       // A hi, A lo, B hi, B lo
constexpr int GEMM_SMEM = STAGES * STAGE_BYTES + STAGES * 8;

// element i of this thread's share of a [128 x 32] tile: KFAST = consecutive threads along K (operand contiguous in K
// in global memory), else consecutive threads along the 128 rows
template <bool KFAST>
__device__ __forceinline__ void tile_pos(int i, int& r, int& k) {
  const int idx = threadIdx.x + 256 * i;
  if (KFAST) { r = idx >> 5; k = idx & 31; }
  else { r = idx & 127; k = idx >> 7; }
}

// ---- operand views: f(k-step, row, k within the step) -> fp32 element (0 outside the operand)
struct NtA {    // X1[m][k] for k-steps < s1, then X2[m / div2][k]
  const float *X1, *X2;
  int ld1, K1, ld2, K2, div2, M, s1;
  __device__ float operator()(int kt, int m, int kk) const {
    const bool two = kt >= s1;
    const int k = (two ? kt - s1 : kt) * TK + kk;
    if (m >= M || k >= (two ? K2 : K1)) return 0.f;
    return two ? X2[(size_t)(m / div2) * ld2 + k] : X1[(size_t)m * ld1 + k];
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
struct NnA {    // G[m][n], contraction over n
  const float* G;
  int ldg, M, N;
  __device__ float operator()(int kt, int m, int nn) const {
    const int n = kt * TK + nn;
    return (m < M && n < N) ? G[(size_t)m * ldg + n] : 0.f;
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
struct TnA {    // G[m][n] as rows n, contraction over m
  const float* G;
  int ldg, M, N;
  __device__ float operator()(int kt, int n, int mm) const {
    const int m = kt * TK + mm;
    return (m < M && n < N) ? G[(size_t)m * ldg + n] : 0.f;
  }
};
struct TnB {    // X[m / div][k] as rows k, contraction over m
  const float* X;
  int ldx, div, M, K;
  __device__ float operator()(int kt, int k, int mm) const {
    const int m = kt * TK + mm;
    return (m < M && k < K) ? X[(size_t)(m / div) * ldx + k] : 0.f;
  }
};

// image tile (row tile rt, k-step kt) at ((rt * ksteps + kt) * 2 + half) * TILE_ELEMS.  Loads follow the operand's
// contiguous dimension (KFAST); the split tile is assembled in shared memory and leaves in 16-byte vectors.
template <bool F16, int PASSES, bool KFAST, class F>
__global__ void __launch_bounds__(256) pack_kernel(F f, int ksteps, uint16_t* __restrict__ img) {
  __shared__ __align__(16) uint16_t t[2 * TILE_ELEMS];
  const int kt = blockIdx.x, rt = blockIdx.y;
  float v[16];
#pragma unroll
  for (int i = 0; i < 16; ++i) {     // all loads first
    int r, k;
    tile_pos<KFAST>(i, r, k);
    v[i] = f(kt, rt * TM + r, k);
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
  uint4* dst = reinterpret_cast<uint4*>(img + ((size_t)rt * ksteps + kt) * 2 * TILE_ELEMS);
  const uint4* src = reinterpret_cast<const uint4*>(t);
  constexpr int NV = (PASSES == 3 ? 2 : 1) * TILE_ELEMS * 2 / 16;
#pragma unroll
  for (int i = threadIdx.x; i < NV; i += 256) dst[i] = src[i];
}

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }
__device__ __forceinline__ void mbar_init(uint64_t* b, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" ::"r"(smem_u32(b)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* b, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" ::"r"(smem_u32(b)), "r"(bytes) : "memory");
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
__device__ __forceinline__ void wgmma_wait_1() { asm volatile("wgmma.wait_group.sync.aligned 1;\n" ::: "memory"); }

// acc[64] of this thread = its fragment of the warpgroup's [64 x 128] block: acc[4 j + 2 h + c] is
// row 16 warp + lane/4 + 8 h, column 8 j + 2 (lane % 4) + c.  Operands: A image row tile blockIdx.y, B image row tile
// blockIdx.x, k-steps [kt0, kt0 + nk) of images with a_ks / b_ks k-steps per row tile.
template <bool F16, int PASSES>
__device__ __forceinline__ void wg_pipeline(float (&acc)[64], const uint16_t* __restrict__ pa, int a_ks,
                                            const uint16_t* __restrict__ pb, int b_ks, int kt0, int nk) {
  extern __shared__ __align__(1024) uint8_t smem[];
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + STAGES * STAGE_BYTES);
  const int tid = threadIdx.x, wg = tid >> 7;
  float acc_lo[PASSES == 3 ? 64 : 1];
#pragma unroll
  for (int i = 0; i < 64; ++i) acc[i] = 0.f;
#pragma unroll
  for (int i = 0; i < (PASSES == 3 ? 64 : 1); ++i) acc_lo[i] = 0.f;
  if (tid == 0) {
    for (int i = 0; i < STAGES; ++i) mbar_init(&full[i], 1);
    asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
  }
  __syncthreads();
  if (nk <= 0) return;
  const uint32_t bytes = PASSES == 3 ? 2 * TILE_BYTES : TILE_BYTES;
  const uint16_t* a0 = pa + ((size_t)blockIdx.y * a_ks + kt0) * 2 * TILE_ELEMS;
  const uint16_t* b0 = pb + ((size_t)blockIdx.x * b_ks + kt0) * 2 * TILE_ELEMS;
  auto issue = [&](int j) {       // k-step j of this CTA -> stage j % STAGES
    uint8_t* st = smem + (j % STAGES) * STAGE_BYTES;
    uint64_t* bar = &full[j % STAGES];
    mbar_expect_tx(bar, 2 * bytes);
    bulk_g2s(st, a0 + (size_t)j * 2 * TILE_ELEMS, bytes, bar);
    bulk_g2s(st + 2 * TILE_BYTES, b0 + (size_t)j * 2 * TILE_ELEMS, bytes, bar);
  };
  if (tid == 0)
    for (int j = 0; j < STAGES - 1 && j < nk; ++j) issue(j);
  for (int j = 0; j < nk; ++j) {
    mbar_wait(&full[j % STAGES], (j / STAGES) & 1);
    const uint8_t* st = smem + (j % STAGES) * STAGE_BYTES;
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
    wgmma_wait_1();               // the MMAs of k-step j - 1 are done (this warpgroup) ...
    __syncthreads();              // ... in both warpgroups: its stage is free
    if (tid == 0 && j + STAGES - 1 < nk) issue(j + STAGES - 1);
  }
  wgmma_wait_all();
  if constexpr (PASSES == 3) {
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] += ldexpf(acc_lo[i], -LO_SHIFT);
  }
}

__device__ __forceinline__ int frag_row(int i) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;   // w = 4 * warpgroup + warp in warpgroup
  return w * 16 + (lane >> 2) + ((i >> 1) & 1) * 8;
}
__device__ __forceinline__ int frag_col(int i) { return (i >> 2) * 8 + (threadIdx.x & 3) * 2 + (i & 1); }

struct Epi {
  int kind;                 // 0: Y = act(acc + bias) ; 1: D (=|+=) mask * (acc + r1_vec r1_row) ; 2: dW += acc (atomic)
  int M, N, act;            // output rows / columns
  const float* bias;
  float* out;
  int ldo, col_off, Kv;
  const float *mask, *r1_vec, *r1_row;
  int ldmask, accumulate;
};

template <bool F16, int PASSES>
__global__ void __launch_bounds__(256) wg_gemm_kernel(const uint16_t* __restrict__ pa, int a_ks, const uint16_t* __restrict__ pb,
                                                      int b_ks, int nk_total, int nk_slab, Epi e) {
  const int kt0 = blockIdx.z * nk_slab;
  float acc[64];
  wg_pipeline<F16, PASSES>(acc, pa, a_ks, pb, b_ks, kt0, min(nk_slab, nk_total - kt0));
  const int m0 = blockIdx.y * TM, n0 = blockIdx.x * TN;
#pragma unroll
  for (int i = 0; i < 64; ++i) {
    const int m = m0 + frag_row(i), n = n0 + frag_col(i);
    if (m >= e.M || n >= e.N) continue;
    if (e.kind == 0) {
      float v = acc[i] + (e.bias ? e.bias[n] : 0.f);
      if (e.act == 1) v = fmaxf(v, 0.f);
      e.out[(size_t)m * e.ldo + n] = v;
    } else if (e.kind == 1) {
      float v = acc[i];
      if (e.r1_vec && n < e.Kv) v = fmaf(e.r1_vec[m], e.r1_row[n], v);
      if (e.mask && !(e.mask[(size_t)m * e.ldmask + n] > 0.f)) v = 0.f;
      float* d = e.out + (size_t)m * e.ldo + n;
      *d = e.accumulate ? (*d + v) : v;
    } else if (n < e.Kv) {
      atomicAdd(e.out + (size_t)m * e.ldo + e.col_off + n, acc[i]);
    }
  }
}

template <bool F16, int PASSES, bool KFAST, class F>
static int launch_pack(F f, int rtiles, int ksteps, uint16_t* img, cudaStream_t st) {
  pack_kernel<F16, PASSES, KFAST, F><<<dim3(ksteps, rtiles), 256, 0, st>>>(f, ksteps, img);
  SPARF_CHECK_LAUNCH("pack_kernel");
  return SPARF_OK;
}

// pack A and B, then the pipelined GEMM over grid (B row tiles, A row tiles, slabs of nk_slab k-steps)
template <bool F16, int PASSES, bool AK, bool BK, class FA, class FB>
static int run(const TcPrec& p, FA fa, int a_rows, FB fb, int b_rows, int ksteps, int nk_slab, const Epi& e, cudaStream_t st) {
  const int rta = ceil_div(a_rows, TM), rtb = ceil_div(b_rows, TM);
  const size_t need = (size_t)std::max(rta, rtb) * ksteps * 2 * TILE_ELEMS;
  SPARF_REQUIRE(p.pack_a && p.pack_b && need <= p.pack_elems, "tc gemm: operand images need %zu 16-bit elements, have %zu",
                need, p.pack_elems);
  int rc = launch_pack<F16, PASSES, AK>(fa, rta, ksteps, p.pack_a, st);
  if (rc) return rc;
  rc = launch_pack<F16, PASSES, BK>(fb, rtb, ksteps, p.pack_b, st);
  if (rc) return rc;
  SPARF_CHECK_CUDA(cudaFuncSetAttribute(wg_gemm_kernel<F16, PASSES>, cudaFuncAttributeMaxDynamicSharedMemorySize, GEMM_SMEM));
  wg_gemm_kernel<F16, PASSES><<<dim3(rtb, rta, ceil_div(ksteps, nk_slab)), 256, GEMM_SMEM, st>>>(p.pack_a, ksteps, p.pack_b,
                                                                                               ksteps, ksteps, nk_slab, e);
  SPARF_CHECK_LAUNCH("wg_gemm_kernel");
  return SPARF_OK;
}

}  // namespace

#define SPARF_WG_RUN(AK, BK, ...)                                              \
  (p.f16 ? (p.passes == 3 ? run<true, 3, AK, BK>(__VA_ARGS__) : run<true, 1, AK, BK>(__VA_ARGS__))     \
         : (p.passes == 3 ? run<false, 3, AK, BK>(__VA_ARGS__) : run<false, 1, AK, BK>(__VA_ARGS__)))

size_t tc_pack_elems(int rows, int ksteps_rows, int cols) {
  // an image of max(rows, cols) rounded to row tiles x ksteps_rows k-steps (callers pass their largest GEMM)
  return (size_t)ceil_div(std::max(rows, cols), TM) * ksteps_rows * 2 * TILE_ELEMS;
}

int tc_gemm_nt(TcPrec p, int act, int M, int N, const float* X1, int ld1, int K1, int K1v, const float* X2, int ld2, int K2,
               int K2v, int div2, const float* W, int ldw, int wcol2, const float* bias, float* Y, int ldy, cudaStream_t st) {
  SPARF_REQUIRE((p.passes == 1 || p.passes == 3) && (act == 0 || act == 1), "tc_gemm_nt: passes=%d act=%d", p.passes, act);
  const int s1 = ceil_div(K1, TK), ks = s1 + (X2 ? ceil_div(K2, TK) : 0);
  Epi e{};
  e.kind = 0; e.M = M; e.N = N; e.act = act; e.bias = bias; e.out = Y; e.ldo = ldy;
  return SPARF_WG_RUN(true, true, p, NtA{X1, X2, ld1, K1, ld2, K2, div2, M, s1}, M, NtB{W, ldw, wcol2, K1v, K2v, N, s1}, N,
                      ks, ks, e, st);
}

int tc_gemm_nn(TcPrec p, int M, int N, int Kout, int Kv, const float* G, int ldg, const float* W, int ldw, int wcol,
               const float* mask_src, int ldmask, const float* r1_vec, const float* r1_row, float* D, int ldd, int accumulate,
               cudaStream_t st) {
  SPARF_REQUIRE(p.passes == 1 || p.passes == 3, "tc_gemm_nn: passes=%d", p.passes);
  const int ks = ceil_div(N, TK);
  Epi e{};
  e.kind = 1; e.M = M; e.N = Kout; e.out = D; e.ldo = ldd; e.Kv = Kv; e.mask = mask_src; e.ldmask = ldmask;
  e.r1_vec = r1_vec; e.r1_row = r1_row; e.accumulate = accumulate;
  return SPARF_WG_RUN(true, false, p, NnA{G, ldg, M, N}, M, NnB{W, ldw, wcol, Kv, N}, Kout, ks, ks, e, st);
}

int tc_gemm_tn(TcPrec p, int M, int N, int K, int Kv, int rows_per_slab, const float* G, int ldg, const float* X, int ldx,
               int div, float* dW, int ldw, int wcol, cudaStream_t st) {
  SPARF_REQUIRE((p.passes == 1 || p.passes == 3) && rows_per_slab % TK == 0, "tc_gemm_tn: passes=%d slab=%d", p.passes,
                rows_per_slab);
  const int ks = ceil_div(M, TK);
  Epi e{};
  e.kind = 2; e.M = N; e.N = K; e.out = dW; e.ldo = ldw; e.col_off = wcol; e.Kv = Kv;
  return SPARF_WG_RUN(false, false, p, TnA{G, ldg, M, N}, N, TnB{X, ldx, div, M, K}, K, ks, rows_per_slab / TK, e, st);
}

}  // namespace sparf

using namespace sparf;

// scratch operand images for the self-tests (diagnostics only: allocated and freed on the stream)
static int with_images(size_t elems, cudaStream_t st, TcPrec& p) {
  SPARF_CHECK_CUDA(cudaMallocAsync(reinterpret_cast<void**>(&p.pack_a), elems * 2, st));
  SPARF_CHECK_CUDA(cudaMallocAsync(reinterpret_cast<void**>(&p.pack_b), elems * 2, st));
  p.pack_elems = elems;
  return SPARF_OK;
}

// Exact-integer checks of the operand images, descriptors, the copy ring and the fragment mapping (small integers are
// exact in bf16 and their dot products exact in fp32).  A [128,K], B [128,K] fp32 row-major, K in {64,...,256}: D = A B^T.
extern "C" int sparf_tc_selftest(const float* A, const float* B, int32_t K, void* packed, float* D, sparf_stream_t stream) {
  (void)packed;
  SPARF_REQUIRE(K % 64 == 0 && K >= 64 && K <= 256, "tc_selftest: K=%d", K);
  cudaStream_t st = (cudaStream_t)stream;
  TcPrec p{false, 1};
  int rc = with_images(tc_pack_elems(128, K / 32, 128), st, p);
  if (rc) return rc;
  rc = tc_gemm_nt(p, 0, 128, 128, A, K, K, K, nullptr, 0, 0, 0, 1, B, K, 0, nullptr, D, 128, st);
  cudaFreeAsync(p.pack_a, st);
  cudaFreeAsync(p.pack_b, st);
  return rc;
}

// D[128,128] = G^T X, G and X [rows, 128] fp32 row-major (the weight-gradient contraction over rows)
extern "C" int sparf_tc_selftest_tn(const float* G, const float* X, int32_t rows, float* D, sparf_stream_t stream) {
  SPARF_REQUIRE(rows == 64 || rows == 128, "tc_selftest_tn: rows=%d", rows);
  cudaStream_t st = (cudaStream_t)stream;
  SPARF_CHECK_CUDA(cudaMemsetAsync(D, 0, 128 * 128 * sizeof(float), st));
  TcPrec p{false, 1};
  int rc = with_images(tc_pack_elems(128, rows / 32, 128), st, p);
  if (rc) return rc;
  rc = tc_gemm_tn(p, rows, 128, 128, 128, rows, G, 128, X, 128, 1, D, 128, 0, st);
  cudaFreeAsync(p.pack_a, st);
  cudaFreeAsync(p.pack_b, st);
  return rc;
}
