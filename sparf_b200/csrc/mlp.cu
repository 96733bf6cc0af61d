// Layer-by-layer engines for the NeRF MLP, activations in a caller-provided HBM workspace, processed in row chunks so
// memory stays bounded.  Works for any width that is a multiple of 8 and any L_xyz/L_view <= 16.
//   SPARF_ENGINE_SIMT_FP32: CUDA-core FFMA GEMMs, the bit-level twin of the reference's fp32 path (same per-element
//     arithmetic, fp32 accumulate): the exact engine and the on-device cross-check of the tensor-core engines.
//   SPARF_ENGINE_TC_3X / TC_1X / TC_3X_W1: the same orchestration with every wide GEMM on Hopper tensor cores
//     (gemm_wgmma.cu); encoders, narrow layers and reductions are the shared CUDA-core kernels below.
// The C-ABI entry points of the MLP (sparf_mlp_*) and of the density queries (sparf_density_*) are at the end; the
// density queries run the same trunk code at arbitrary points, without the colour head.
//
// Reference: NeRF.compute_raw_density / NeRF.forward (source/models/frequency_nerf.py:149-227),
// FrequencyEmbedder (:47-69), positional_encoding (:229-258).
#include <algorithm>

#include "common.cuh"
#include "gemm_wgmma.cuh"

namespace sparf {

// ------------------------------------------------------------------------------------------------
// encoders
// ------------------------------------------------------------------------------------------------
__global__ void c2f_weights_kernel(C2F c, int L_xyz, int L_view, float* __restrict__ wts /*[32]*/) {
  int j = threadIdx.x;
  if (j < 16) wts[j] = j < L_xyz ? band_weight(c, L_xyz, j) : 0.f;
  else if (j < 32) wts[j] = (j - 16) < L_view ? band_weight(c, L_view, j - 16) : 0.f;
}

// enc[m][0:3] = x = o + t*d ; enc[m][3 + c*2L + {0,L} + j] = w_j * {sin,cos}(x_c * 2^j pi) ; zero pad to E3p
// dirs == NULL: the origins are the points themselves, x = o (S = 1; the value o + 0*d takes)
// DYN (S = 1): total / E3p rows is a capacity, of which live_rows are encoded (the same for every kernel below with DYN);
// the rows of the global buffers start at row_start (RowCount)
template <bool DYN = false>
__global__ void encode_xyz_kernel(long long total, int S, int L, int E3p, const float* __restrict__ origins,
                                  const float* __restrict__ dirs, const float* __restrict__ t,
                                  const float* __restrict__ wts, float* __restrict__ enc, RowCount rc) {
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (DYN ? live_rows<DYN>(total / E3p, rc) * E3p : total)) return;
  if constexpr (DYN) {
    const long long s0 = row_start<true>(rc);
    origins += s0 * 3;
    if (dirs) dirs += s0 * 3;
    t += s0;
    enc += s0 * E3p;
  }
  int col = (int)(idx % E3p);
  long long m = idx / E3p;
  long long r = m / S;
  float val = 0.f;
  if (col < 3 + 6 * L) {
    int c = col < 3 ? col : (col - 3) / (2 * L);
    float x = dirs ? add_rn(origins[r * 3 + c], mul_rn(dirs[r * 3 + c], t[m])) : origins[r * 3 + c];  // camera.py:433-435
    if (col < 3) {
      val = x;
    } else {
      int rem = (col - 3) - c * 2 * L;
      int is_cos = rem >= L;
      int j = rem - is_cos * L;
      float arg = mul_rn(x, band_freq(j));
      val = mul_rn(is_cos ? cosf(arg) : sinf(arg), wts[j]);
    }
  }
  enc[idx] = val;
}

// per-ray view-direction encoding: unit = d / max(|d|, 1e-12) (F.normalize), same layout as above
template <bool DYN = false>
__global__ void encode_dir_kernel(int total, int L, int Evp, const float* __restrict__ dirs,
                                  const float* __restrict__ wts_view, float* __restrict__ denc, RowCount rc) {
  int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (DYN ? (int)live_rows<DYN>(total / Evp, rc) * Evp : total)) return;
  if constexpr (DYN) {
    const long long s0 = row_start<true>(rc);
    dirs += s0 * 3;
    denc += s0 * Evp;
  }
  int col = idx % Evp, r = idx / Evp;
  float val = 0.f;
  if (col < 3 + 6 * L) {
    float dx = dirs[r * 3], dy = dirs[r * 3 + 1], dz = dirs[r * 3 + 2];
    float len = fmaxf(sqrtf(dx * dx + dy * dy + dz * dz), 1e-12f);
    int c = col < 3 ? col : (col - 3) / (2 * L);
    float u = __fdiv_rn(c == 0 ? dx : (c == 1 ? dy : dz), len);
    if (col < 3) {
      val = u;
    } else {
      int rem = (col - 3) - c * 2 * L;
      int is_cos = rem >= L;
      int j = rem - is_cos * L;
      float arg = mul_rn(u, band_freq(j));
      val = mul_rn(is_cos ? cosf(arg) : sinf(arg), wts_view[j]);
    }
  }
  denc[idx] = val;
}

// ------------------------------------------------------------------------------------------------
// 128x128x8 SGEMM family.  256 threads, 8x8 outputs per thread laid out as 2x2 blocks of 4x4 so that
// shared-memory reads are conflict-free float4s.
// ------------------------------------------------------------------------------------------------
constexpr int BM = 128, BN = 128, BK = 8;

struct Frag {
  float acc[8][8];
  __device__ __forceinline__ void zero() {
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
  }
  __device__ __forceinline__ void mma(const float (*As)[BM], const float (*Bs)[BN], int ty, int tx) {
#pragma unroll
    for (int kk = 0; kk < BK; ++kk) {
      float4 a0 = *reinterpret_cast<const float4*>(&As[kk][ty * 4]);
      float4 a1 = *reinterpret_cast<const float4*>(&As[kk][64 + ty * 4]);
      float4 b0 = *reinterpret_cast<const float4*>(&Bs[kk][tx * 4]);
      float4 b1 = *reinterpret_cast<const float4*>(&Bs[kk][64 + tx * 4]);
      float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      float b[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
  }
};
__device__ __forceinline__ int frag_row(int ty, int i) { return (i < 4 ? 0 : 64) + ty * 4 + (i & 3); }
__device__ __forceinline__ int frag_col(int tx, int j) { return (j < 4 ? 0 : 64) + tx * 4 + (j & 3); }

// ---- NT:  Y[m][n] = relu( sum_k X1[m][k] W[n][k] + sum_k X2[m/div2][k] W[n][wcol2+k] + bias[n] )
__global__ void __launch_bounds__(256) gemm_nt_kernel(int M, int N, const float* __restrict__ X1, int ld1, int K1,
                                                      int K1v, const float* __restrict__ X2, int ld2, int K2, int K2v,
                                                      int div2, const float* __restrict__ W, int ldw, int wcol2,
                                                      const float* __restrict__ bias, float* __restrict__ Y, int ldy) {
  __shared__ __align__(16) float As[BK][BM];
  __shared__ __align__(16) float Bs[BK][BN];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;
  const int lrow = tid >> 1, lk = (tid & 1) * 4;
  Frag f;
  f.zero();
  for (int src = 0; src < 2; ++src) {
    const float* X = src == 0 ? X1 : X2;
    if (!X) continue;
    const int ld = src == 0 ? ld1 : ld2, K = src == 0 ? K1 : K2, Kv = src == 0 ? K1v : K2v;
    const int wc = src == 0 ? 0 : wcol2, dv = src == 0 ? 1 : div2;
    for (int k0 = 0; k0 < K; k0 += BK) {
      float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
      int m = m0 + lrow;
      if (m < M) a = *reinterpret_cast<const float4*>(X + (size_t)(m / dv) * ld + k0 + lk);
      As[lk + 0][lrow] = a.x; As[lk + 1][lrow] = a.y; As[lk + 2][lrow] = a.z; As[lk + 3][lrow] = a.w;
      int n = n0 + lrow;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        int k = k0 + lk + i;
        Bs[lk + i][lrow] = (n < N && k < Kv) ? W[(size_t)n * ldw + wc + k] : 0.f;
      }
      __syncthreads();
      f.mma(As, Bs, ty, tx);
      __syncthreads();
    }
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    int m = m0 + frag_row(ty, i);
    if (m >= M) continue;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      int n = n0 + frag_col(tx, j);
      if (n >= N) continue;
      float v = f.acc[i][j] + (bias ? bias[n] : 0.f);
      v = fmaxf(v, 0.f);
      Y[(size_t)m * ldy + n] = v;
    }
  }
}

// ---- NN (dgrad):  D[m][k] = mask(m,k) * ( sum_n G[m][n] W[n][wcol+k] + r1_vec[m]*r1_row[k] )  (= or +=)
__global__ void __launch_bounds__(256) gemm_nn_kernel(int M, int N, int Kout, int Kv, const float* __restrict__ G, int ldg,
                                                      const float* __restrict__ W, int ldw, int wcol,
                                                      const float* __restrict__ mask_src, int ldmask,
                                                      const float* __restrict__ r1_vec, const float* __restrict__ r1_row,
                                                      float* __restrict__ D, int ldd, int accumulate) {
  __shared__ __align__(16) float As[BK][BM];
  __shared__ __align__(16) float Bs[BK][BN];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int m0 = blockIdx.y * BM, c0 = blockIdx.x * BN;
  const int lrow = tid >> 1, lk = (tid & 1) * 4;
  const int bn = tid >> 5, bc = (tid & 31) * 4;
  Frag f;
  f.zero();
  for (int nk0 = 0; nk0 < N; nk0 += BK) {
    float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
    int m = m0 + lrow;
    if (m < M && nk0 + lk < N) a = *reinterpret_cast<const float4*>(G + (size_t)m * ldg + nk0 + lk);  // N % 4 == 0
    As[lk + 0][lrow] = a.x; As[lk + 1][lrow] = a.y; As[lk + 2][lrow] = a.z; As[lk + 3][lrow] = a.w;
    int n = nk0 + bn;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      int k = c0 + bc + i;
      Bs[bn][bc + i] = (n < N && k < Kv) ? W[(size_t)n * ldw + wcol + k] : 0.f;
    }
    __syncthreads();
    f.mma(As, Bs, ty, tx);
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    int m = m0 + frag_row(ty, i);
    if (m >= M) continue;
    float rv = r1_vec ? r1_vec[m] : 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      int k = c0 + frag_col(tx, j);
      if (k >= Kout) continue;
      float v = f.acc[i][j];
      if (r1_vec && k < Kv) v = fmaf(rv, r1_row[k], v);
      if (mask_src && !(mask_src[(size_t)m * ldmask + k] > 0.f)) v = 0.f;
      float* d = D + (size_t)m * ldd + k;
      *d = accumulate ? (*d + v) : v;
    }
  }
}

// ---- TN (wgrad):  dW[n][wcol+k] += sum_{m in slab} G[m][n] X[m/div][k]      (atomic over slabs)
__global__ void __launch_bounds__(256) gemm_tn_kernel(int M, int N, int K, int Kv, int rows_per_slab,
                                                      const float* __restrict__ G, int ldg, const float* __restrict__ X,
                                                      int ldx, int div, float* __restrict__ dW, int ldw, int wcol) {
  __shared__ __align__(16) float As[BK][BM];
  __shared__ __align__(16) float Bs[BK][BN];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int n0 = blockIdx.y * BM, c0 = blockIdx.x * BN;
  const int m_begin = blockIdx.z * rows_per_slab, m_end = min(M, m_begin + rows_per_slab);
  const int lm = tid >> 5, lc = (tid & 31) * 4;
  Frag f;
  f.zero();
  for (int mm0 = m_begin; mm0 < m_end; mm0 += BK) {
    int m = mm0 + lm;
    float4 a = make_float4(0.f, 0.f, 0.f, 0.f), b = make_float4(0.f, 0.f, 0.f, 0.f);
    if (m < m_end) {
      if (n0 + lc < N) a = *reinterpret_cast<const float4*>(G + (size_t)m * ldg + n0 + lc);  // N % 4 == 0
      if (c0 + lc < K) b = *reinterpret_cast<const float4*>(X + (size_t)(m / div) * ldx + c0 + lc);  // K % 4 == 0
    }
    *reinterpret_cast<float4*>(&As[lm][lc]) = a;
    *reinterpret_cast<float4*>(&Bs[lm][lc]) = b;
    __syncthreads();
    f.mma(As, Bs, ty, tx);
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    int n = n0 + frag_row(ty, i);
    if (n >= N) continue;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      int k = c0 + frag_col(tx, j);
      if (k >= Kv) continue;
      atomicAdd(dW + (size_t)n * ldw + wcol + k, f.acc[i][j]);
    }
  }
}

// launchers of the CUDA-core GEMMs (the tensor-core engines call gemm_wgmma.cu instead)
static int gemm_nt(int M, int N, const float* X1, int ld1, int K1, int K1v, const float* X2, int ld2, int K2, int K2v,
                   int div2, const float* W, int ldw, int wcol2, const float* bias, float* Y, int ldy, cudaStream_t st) {
  gemm_nt_kernel<<<dim3(ceil_div(N, BN), ceil_div(M, BM)), 256, 0, st>>>(M, N, X1, ld1, K1, K1v, X2, ld2, K2, K2v, div2, W, ldw,
                                                                        wcol2, bias, Y, ldy);
  SPARF_CHECK_LAUNCH("gemm_nt_kernel");
  return SPARF_OK;
}

static int gemm_nn(int M, int N, int Kout, int Kv, const float* G, int ldg, const float* W, int ldw, int wcol,
                   const float* mask_src, int ldmask, const float* r1_vec, const float* r1_row, float* D, int ldd, int accumulate,
                   cudaStream_t st) {
  gemm_nn_kernel<<<dim3(ceil_div(Kout, BN), ceil_div(M, BM)), 256, 0, st>>>(M, N, Kout, Kv, G, ldg, W, ldw, wcol, mask_src,
                                                                           ldmask, r1_vec, r1_row, D, ldd, accumulate);
  SPARF_CHECK_LAUNCH("gemm_nn_kernel");
  return SPARF_OK;
}

static int gemm_tn(int M, int N, int K, int Kv, int rows_per_slab, const float* G, int ldg, const float* X, int ldx,
                   int div, float* dW, int ldw, int wcol, cudaStream_t st) {
  gemm_tn_kernel<<<dim3(ceil_div(K, BN), ceil_div(N, BM), ceil_div(M, rows_per_slab)), 256, 0, st>>>(
      M, N, K, Kv, rows_per_slab, G, ldg, X, ldx, div, dW, ldw, wcol);
  SPARF_CHECK_LAUNCH("gemm_tn_kernel");
  return SPARF_OK;
}

// GEMM precision per role: forward, input gradient (dgrad), weight gradient (wgrad); passes 0 on the SIMT engine
struct EnginePrec {
  TcPrec fwd, dgrad, wgrad;
};

static EnginePrec engine_prec(int engine) {
  const TcPrec fp32{false, 0}, f16x3{true, 3}, f16x1{true, 1}, bf16x3{false, 3}, bf16x1{false, 1};
  switch (engine) {
    case SPARF_ENGINE_TC_3X: return EnginePrec{f16x3, bf16x3, bf16x3};
    case SPARF_ENGINE_TC_1X: return EnginePrec{f16x1, bf16x1, bf16x1};
    case SPARF_ENGINE_TC_3X_W1: return EnginePrec{f16x3, bf16x3, bf16x1};
    default: return EnginePrec{fp32, fp32, fp32};
  }
}

// ------------------------------------------------------------------------------------------------
// narrow layers (1 or 3 outputs): one warp per row
// ------------------------------------------------------------------------------------------------
// MODE 0: density row:  raw = X.W[0] + b ; z = raw + noise ; raw_out[m] = z ; sigma[m] = softplus(z)
// MODE 1: colour head:  rgb[m][j] = sigmoid(X.W[j] + b[j]), j < 3
template <int MODE, bool DYN = false>
__global__ void rowdot_kernel(long long M, int K, const float* __restrict__ X, int ldx, const float* __restrict__ W,
                              int ldw, const float* __restrict__ bias, const float* __restrict__ noise,
                              float* __restrict__ raw_out, float* __restrict__ out, RowCount rc) {
  const int lane = threadIdx.x & 31;
  long long m = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (m >= live_rows<DYN>(M, rc)) return;
  if constexpr (DYN) {
    const long long s0 = row_start<true>(rc);
    X += s0 * ldx;
    if (noise) noise += s0;
    if (raw_out) raw_out += s0;
    if (out) out += s0 * (MODE == 0 ? 1 : 3);
  }
  constexpr int NS = MODE == 0 ? 1 : 3;
  float acc[NS];
#pragma unroll
  for (int j = 0; j < NS; ++j) acc[j] = 0.f;
  const float* x = X + (size_t)m * ldx;
  for (int k = lane; k < K; k += 32) {
    float xv = x[k];
#pragma unroll
    for (int j = 0; j < NS; ++j) acc[j] = fmaf(xv, W[(size_t)j * ldw + k], acc[j]);
  }
#pragma unroll
  for (int j = 0; j < NS; ++j)
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) acc[j] += __shfl_xor_sync(0xffffffffu, acc[j], s);
  if (lane == 0) {
    if (MODE == 0) {
      float raw = acc[0] + bias[0];
      float z = noise ? add_rn(raw, noise[m]) : raw;
      if (raw_out) raw_out[m] = z;     // the softplus argument, what the backward needs
      if (out) out[m] = softplus_f(z);
    } else {
#pragma unroll
      for (int j = 0; j < NS; ++j) out[m * 3 + j] = sigmoid_f(acc[j] + bias[j]);
    }
  }
}

// g_pre[m][j] = d_rgb[m][j] * c (1-c) ;  g_raw[m] = d_sigma[m] * softplus'(raw)   (raw: the softplus argument, noise added)
__global__ void head_grad_kernel(long long M, const float* __restrict__ d_rgb, const float* __restrict__ rgbv,
                                 const float* __restrict__ d_sigma, const float* __restrict__ raw,
                                 float* __restrict__ g_pre /*[M,4]*/, float* __restrict__ g_raw) {
  long long m = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= M) return;
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    float c = rgbv[m * 3 + j];
    g_pre[m * 4 + j] = d_rgb[m * 3 + j] * c * (1.f - c);
  }
  g_pre[m * 4 + 3] = 0.f;
  g_raw[m] = d_sigma[m] * softplus_grad_f(raw[m]);
}

// dW[j][k] += sum_m g[m*gs + j] X[m][k] ; db[j] += sum_m g[m*gs+j]   (NS <= 3 narrow outputs)
template <int NS>
__global__ void narrow_wgrad_kernel(long long M, int K, int rows_per_block, const float* __restrict__ g, int gs,
                                    const float* __restrict__ X, int ldx, float* __restrict__ dW, int ldw,
                                    float* __restrict__ db) {
  long long m_begin = (long long)blockIdx.x * rows_per_block;
  long long m_end = m_begin + rows_per_block < M ? m_begin + rows_per_block : M;
  for (int k = threadIdx.x; k < K + 1; k += blockDim.x) {
    float acc[NS];
#pragma unroll
    for (int j = 0; j < NS; ++j) acc[j] = 0.f;
    for (long long m = m_begin; m < m_end; ++m) {
      float xv = k < K ? X[(size_t)m * ldx + k] : 1.f;  // column K = the bias
#pragma unroll
      for (int j = 0; j < NS; ++j) acc[j] = fmaf(g[m * gs + j], xv, acc[j]);
    }
#pragma unroll
    for (int j = 0; j < NS; ++j) {
      if (k < K) atomicAdd(dW + (size_t)j * ldw + k, acc[j]);
      else atomicAdd(db + j, acc[j]);
    }
  }
}

// Ghid[m][k] = (hid[m][k] > 0) * sum_j g_pre[m][j] W9[j][k]
__global__ void narrow_dgrad_kernel(long long total, int K, const float* __restrict__ g_pre, const float* __restrict__ W,
                                    int ldw, const float* __restrict__ hid, float* __restrict__ out) {
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  int k = (int)(idx % K);
  long long m = idx / K;
  float v = 0.f;
#pragma unroll
  for (int j = 0; j < 3; ++j) v = fmaf(g_pre[m * 4 + j], W[(size_t)j * ldw + k], v);
  out[idx] = hid[idx] > 0.f ? v : 0.f;
}

// db[n] += sum_m G[m][n]
__global__ void colsum_kernel(long long M, int N, int rows_per_block, const float* __restrict__ G, int ldg,
                              float* __restrict__ db) {
  __shared__ float red[8][33];
  int cx = threadIdx.x & 31, ry = threadIdx.x >> 5;
  int n = blockIdx.x * 32 + cx;
  long long m_begin = (long long)blockIdx.y * rows_per_block;
  long long m_end = m_begin + rows_per_block < M ? m_begin + rows_per_block : M;
  float acc = 0.f;
  if (n < N)
    for (long long m = m_begin + ry; m < m_end; m += 8) acc += G[(size_t)m * ldg + n];
  red[ry][cx] = acc;
  __syncthreads();
  if (ry == 0 && n < N) {
    float v = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) v += red[i][cx];
    atomicAdd(db + n, v);
  }
}

// out[i] = v: the density row's upstream gradient of the point-gradient query (d raw / d raw = 1)
__global__ void fill_kernel(long long n, float v, float* __restrict__ out) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = v;
}

// G[i] = (feat[i] > 0) * d_feat[i]: the last trunk layer's gradient when the caller gives it (density backward)
__global__ void relu_mask_kernel(long long total, const float* __restrict__ feat, const float* __restrict__ d_feat,
                                 float* __restrict__ G) {
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  G[idx] = feat[idx] > 0.f ? d_feat[idx] : 0.f;
}

// out[r][c] = sum_{k<S} in[(r*S+k)][c]
template <bool DYN = false>
__global__ void ray_reduce_kernel(int nrays, int S, int C, const float* __restrict__ in, float* __restrict__ out,
                                  RowCount rc) {
  int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (int)live_rows<DYN, false>(nrays, rc) * C) return;
  int c = idx % C, r = idx / C;
  float acc = 0.f;
  for (int k = 0; k < S; ++k) acc += in[((size_t)r * S + k) * C + c];
  out[idx] = acc;
}

// positional-encoding backward + reduction over the ray:  d_o += sum_k g_x ; d_d += sum_k t_k g_x
// d/dx [w sin(f x)] = f * (w cos(f x)) = f * enc_cos ; d/dx [w cos(f x)] = -f * enc_sin.  One warp per ray.
// t == NULL (with d_d == NULL): the encoding of points (encode_xyz_kernel without dirs), d_o = the points' gradient.
template <bool DYN = false>
__global__ void posenc_bwd_kernel(int nrays, int S, int L, int E3p, const float* __restrict__ enc,
                                  const float* __restrict__ Genc, const float* __restrict__ t,
                                  float* __restrict__ d_o, float* __restrict__ d_d, RowCount rc) {
  const int lane = threadIdx.x & 31;
  int r = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (r >= (int)live_rows<DYN, false>(nrays, rc)) return;
  float so[3] = {0.f, 0.f, 0.f}, sd[3] = {0.f, 0.f, 0.f};
  for (int k = lane; k < S; k += 32) {
    size_t m = (size_t)r * S + k;
    const float* e = enc + m * E3p;
    const float* g = Genc + m * E3p;
    float tk = t ? t[m] : 0.f;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      float gx = g[c];
      for (int j = 0; j < L; ++j) {
        float f = band_freq(j);
        int is = 3 + c * 2 * L + j, ic = is + L;
        gx += f * (g[is] * e[ic] - g[ic] * e[is]);
      }
      so[c] += gx;
      sd[c] += tk * gx;
    }
  }
#pragma unroll
  for (int c = 0; c < 3; ++c) {
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) {
      so[c] += __shfl_xor_sync(0xffffffffu, so[c], s);
      sd[c] += __shfl_xor_sync(0xffffffffu, sd[c], s);
    }
  }
  if (lane == 0) {
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      if (d_o) d_o[r * 3 + c] += so[c];
      if (d_d) d_d[r * 3 + c] += sd[c];
    }
  }
}

// view-direction encoding backward: g_unit from Gdenc, then through unit = d/|d|
template <bool DYN = false>
__global__ void direnc_bwd_kernel(int nrays, int L, int Evp, const float* __restrict__ denc,
                                  const float* __restrict__ Gdenc, const float* __restrict__ dirs,
                                  float* __restrict__ d_d, RowCount rc) {
  int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= (int)live_rows<DYN, false>(nrays, rc)) return;
  const float* e = denc + (size_t)r * Evp;
  const float* g = Gdenc + (size_t)r * Evp;
  float gu[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    float gx = g[c];
    for (int j = 0; j < L; ++j) {
      float f = band_freq(j);
      int is = 3 + c * 2 * L + j, ic = is + L;
      gx += f * (g[is] * e[ic] - g[ic] * e[is]);
    }
    gu[c] = gx;
  }
  float dx = dirs[r * 3], dy = dirs[r * 3 + 1], dz = dirs[r * 3 + 2];
  float len = fmaxf(sqrtf(dx * dx + dy * dy + dz * dz), 1e-12f);
  float ux = dx / len, uy = dy / len, uz = dz / len;
  float dot = gu[0] * ux + gu[1] * uy + gu[2] * uz;
  d_d[r * 3] += (gu[0] - ux * dot) / len;
  d_d[r * 3 + 1] += (gu[1] - uy * dot) / len;
  d_d[r * 3 + 2] += (gu[2] - uz * dot) / len;
}

// ------------------------------------------------------------------------------------------------
// host orchestration
// ------------------------------------------------------------------------------------------------
static inline int pad8(int x) { return (x + 7) / 8 * 8; }

struct MlpDims {
  int E3, E3p, Ev, Evp, W, HW, nt, skip;
};

static MlpDims mlp_dims(const SparfMLP* mlp) {
  MlpDims d;
  d.E3 = 3 + 6 * mlp->L_xyz;
  d.Ev = 3 + 6 * mlp->L_view;
  d.E3p = pad8(d.E3);
  d.Evp = pad8(d.Ev);
  d.W = mlp->width;
  d.HW = mlp->head_width;
  d.nt = mlp->n_trunk;
  d.skip = mlp->skip_layer;
  return d;
}

// the trunk's fields (density calls); validate_mlp: these and the colour head's (MLP calls)
static int validate_trunk(const SparfMLP* mlp) {
  SPARF_REQUIRE(mlp != nullptr, "mlp is NULL");
  SPARF_REQUIRE(mlp->n_trunk >= 2 && mlp->n_trunk <= SPARF_MAX_TRUNK, "n_trunk=%d unsupported", mlp->n_trunk);
  SPARF_REQUIRE(mlp->width % 8 == 0 && mlp->width >= 8, "width=%d must be a multiple of 8", mlp->width);
  SPARF_REQUIRE(mlp->L_xyz >= 1 && mlp->L_xyz <= SPARF_MAX_L && mlp->L_view >= 1 && mlp->L_view <= SPARF_MAX_L,
                "L_xyz=%d / L_view=%d unsupported", mlp->L_xyz, mlp->L_view);
  SPARF_REQUIRE(mlp->skip_layer < mlp->n_trunk && mlp->skip_layer != 0, "skip_layer=%d unsupported", mlp->skip_layer);
  SPARF_REQUIRE(!mlp->use_c2f || mlp->progress, "use_c2f needs the progress pointer");
  for (int i = 0; i < mlp->n_trunk; ++i)
    SPARF_REQUIRE(mlp->trunk_w[i] && mlp->trunk_b[i], "trunk layer %d has NULL tensors", i);
  return SPARF_OK;
}

static int validate_mlp(const SparfMLP* mlp) {
  SPARF_TRY(validate_trunk(mlp));
  SPARF_REQUIRE(mlp->head_width % 8 == 0 && mlp->head_width >= 8, "head_width=%d must be a multiple of 8", mlp->head_width);
  SPARF_REQUIRE(mlp->head_w[0] && mlp->head_b[0] && mlp->head_w[1] && mlp->head_b[1], "head has NULL tensors");
  return SPARF_OK;
}

// The passes of the MLP calls.  The taped forward writes the activations to a caller-held tape that the taped backward
// reads; the recompute backward recomputes them chunk by chunk.  The density calls run kForward and kRecomputeBackward,
// and kGradient: the recompute backward of the points' gradient alone, without weight gradients.
enum class Pass { kForward, kTapedForward, kRecomputeBackward, kTapedBackward, kGradient };

// Rows per chunk: the recompute backward keeps every trunk activation of its chunk, so it takes the smallest chunks; the
// taped passes keep only a chunk's images and gradients (about 1 GB at 131072 rows of the default net) and take the
// largest, so that weight packs, GEMM ramp-ups and small kernels repeat as seldom as possible.
static int chunk_rows(Pass pass) {
  switch (pass) {
    case Pass::kForward: return 65536;
    case Pass::kRecomputeBackward:
    case Pass::kGradient: return 32768;
    default: return 131072;
  }
}

// whole rays of S samples per chunk, at least one
static int chunk_rays(int S, Pass pass) { return std::max(1, chunk_rows(pass) / S); }

struct Carver {
  char* p;
  size_t used;
  float* take(size_t nfloats) {
    size_t bytes = align_up(nfloats * sizeof(float), 256);
    float* r = reinterpret_cast<float*>(p + used);
    used += bytes;
    return r;
  }
  TcImage image(int rows, int cols) {   // operand image of a [rows x cols] matrix
    return TcImage{reinterpret_cast<uint16_t*>(take((tc_image_elems(rows, cols) + 1) / 2)), ceil_div(cols, 32)};
  }
};

// The forward's activations that the backward reads: the encodings, the nt trunk activations, the colour-head
// activations and the softplus argument of the density (noise added).  A taped forward keeps them for the whole batch in
// the tape; the workspace holds one chunk's (its trunk activations ping-pong in a plain forward).  With the fused trunk
// (trunk_chained) the taped and recompute forwards also keep the ReLU masks of H[0] ... H[nt-3] as bits (8 words per row
// of width 256; in the tape after everything else): the chained input gradients read them, since they all run before
// the weight gradients that would otherwise write them.
struct Tape {
  float *enc, *denc, *hid, *raw;
  float* H[SPARF_MAX_TRUNK];
  uint32_t* bits[SPARF_MAX_TRUNK];
};

// Whether the trunk forward runs as one fused kernel (tc_trunk_chain), and the input gradients of layers nt-2 ... 1 as
// another (tc_dgrad_chain), from the shape alone: a tensor-core engine and a trunk the kernels are built for.  Other
// shapes go layer by layer through tc_gemm_nt and tc_gemm_nn.
static bool trunk_chained(const MlpDims& d, bool tc) { return tc && tc_chain_supported(d.W, d.E3p, d.nt, d.skip); }

static size_t tape_layout(const MlpDims& d, bool tc, int R, int S, char* base, Tape* tp) {
  const size_t M = (size_t)R * S;
  Carver cv{base, 0};
  Tape t{};
  t.enc = cv.take(M * d.E3p);
  t.denc = cv.take((size_t)R * d.Evp);
  t.hid = cv.take(M * d.HW);
  t.raw = cv.take(M);
  for (int l = 0; l < d.nt; ++l) t.H[l] = cv.take(M * d.W);
  for (int l = 0; trunk_chained(d, tc) && l < d.nt - 2; ++l) t.bits[l] = reinterpret_cast<uint32_t*>(cv.take(M * (d.W / 32)));
  if (tp) *tp = t;
  return cv.used + 256;
}

constexpr size_t kMaxTapeBytes = (size_t)16 << 30;   // larger batches take the recompute backward

// the slice of a whole-batch tape that holds the chunk starting at ray r0
static Tape tape_chunk(const Tape& t, const MlpDims& d, int r0, int S) {
  const size_t m0 = (size_t)r0 * S;
  Tape c{};
  c.enc = t.enc + m0 * d.E3p;
  c.denc = t.denc + (size_t)r0 * d.Evp;
  c.hid = t.hid + m0 * d.HW;
  c.raw = t.raw + m0;
  for (int l = 0; l < d.nt; ++l) {
    c.H[l] = t.H[l] + m0 * d.W;
    c.bits[l] = t.bits[l] ? t.bits[l] + m0 * (d.W / 32) : nullptr;
  }
  return c;
}

// Workspace of one call, per chunk of nrc rays.  Tensor-core engines keep their GEMM operands as images: the forward's
// encodings and ping-pong trunk activations (fused trunk: the last layer's only, and every trunk weight), the backward's
// trunk gradients (a row image for the next input gradient, a transposed one for the weight gradient; no fp32 copy; see
// grad_row), the colour-head gradient's two images (no fp32 copy either), the ReLU mask bits of one layer input (written
// by its weight-gradient GEMM, read by its input-gradient GEMM), and a buffer for the weight operand packed per GEMM.
// head = false (density calls, S = 1): no colour-head or view-direction buffer.  kGradient takes no more than
// kRecomputeBackward: it keeps no last-layer features and no mask bits, and its transposed gradient images, which no
// weight gradient reads, share one buffer; it adds a row of ones and, on the tensor cores, one row of bias sums.
struct Ws {
  float *wts, *rgbv, *G0, *G1, *Genc, *Ghid, *gpre, *graw, *Gdtmp, *Gdenc;
  float *ones, *colsum_sink;    // kGradient: the density row's upstream gradient (1 per row); bias sums nobody reads
  Tape act;     // the forward's activations of one chunk (forward and recompute backward)
  TcImage encimg, dencimg, Himg[2], Grow[2], Gtr[SPARF_MAX_TRUNK - 1], ghid_row, ghid_tr;
  TcImage wimg[SPARF_MAX_TRUNK];   // fused trunk forward: every trunk layer's weight image, alive at once
  TcImage nnimg[SPARF_MAX_TRUNK];  // chained input gradients: the weight images of layers 1 ... nt-2, alive at once
  uint32_t* mask_bits;   // [Mc x ceil(W / 32)]
  uint16_t* pack_b;
  size_t pack_elems;
};

static size_t carve(const MlpDims& d, bool tc, int nrc, int S, Pass pass, bool head, char* base, Ws* out) {
  const size_t Mc = (size_t)nrc * S;
  const bool grad_only = pass == Pass::kGradient;
  const bool fwd_here = pass == Pass::kForward || pass == Pass::kRecomputeBackward || grad_only;   // not taped
  const bool bwd = pass == Pass::kRecomputeBackward || pass == Pass::kTapedBackward || grad_only;
  const bool chain = trunk_chained(d, tc);
  Carver cv{base, 0};
  Ws w{};
  w.wts = cv.take(32);
  if (fwd_here) {
    w.act.enc = cv.take(Mc * d.E3p);
    if (head) {
      w.act.denc = cv.take((size_t)nrc * d.Evp);
      w.act.hid = cv.take(Mc * d.HW);
      w.act.raw = cv.take(Mc);
      w.rgbv = cv.take(Mc * 3);
    }
    // the backward keeps every layer; the forward ping-pongs, or keeps the last two only (the density row's input and
    // the colour head's) when the fused trunk leaves the others on the SM
    const int nH = pass == Pass::kForward ? 2 : grad_only ? d.nt - 1 : d.nt;
    if (chain && pass == Pass::kForward) {
      for (int l = d.nt - 2; l < d.nt; ++l) w.act.H[l] = cv.take(Mc * d.W);
    } else {
      for (int l = 0; l < nH; ++l) w.act.H[l] = cv.take(Mc * d.W);
      for (int l = nH; l < d.nt; ++l) w.act.H[l] = w.act.H[l & 1];
    }
    if (grad_only) w.act.H[d.nt - 1] = nullptr;     // the point gradient needs no last-layer features
    for (int l = 0; chain && bwd && l < d.nt - 2; ++l) w.act.bits[l] = reinterpret_cast<uint32_t*>(cv.take(Mc * (d.W / 32)));
  }
  if (bwd && !tc) {
    w.G0 = cv.take(Mc * d.W);
    w.G1 = cv.take(Mc * d.W);
  }
  if (bwd) {
    w.Genc = cv.take(Mc * d.E3p);
    if (grad_only) w.ones = cv.take(Mc);
    if (!tc && head) {
      w.Ghid = cv.take(Mc * d.HW);
      w.gpre = cv.take(Mc * 4);
    }
    if (head) {
      w.graw = cv.take(Mc);
      w.Gdtmp = cv.take(Mc * d.Evp);
      w.Gdenc = cv.take((size_t)nrc * d.Evp);
    }
  }
  if (tc && pass != Pass::kTapedBackward) {
    w.encimg = cv.image((int)Mc, d.E3p);
    if (head) w.dencimg = cv.image((int)Mc, d.Evp);
    if (chain) {    // only the last layer's image (the colour head reads it) and the weight images
      if (head) w.Himg[(d.nt - 1) & 1] = cv.image((int)Mc, d.W);
      for (int l = 0; l < d.nt; ++l) w.wimg[l] = cv.image(d.W, tc_chain_ksteps(l, d.skip, d.E3p) * 32);
    } else {
      for (TcImage& h : w.Himg) h = cv.image((int)Mc, d.W);
    }
  }
  if (tc && bwd) {
    for (TcImage& g : w.Grow) g = cv.image((int)Mc, d.W);
    const int ntr = chain ? d.nt - 1 : 2;
    for (int i = 0; i < (grad_only ? 1 : ntr); ++i) w.Gtr[i] = cv.image(d.W, (int)Mc);
    for (int i = 1; grad_only && i < ntr; ++i) w.Gtr[i] = w.Gtr[0];
    for (int l = 1; chain && l <= d.nt - 2; ++l) w.nnimg[l] = cv.image(d.W, d.W);
    if (head) {
      w.ghid_row = cv.image((int)Mc, d.HW);
      w.ghid_tr = cv.image(d.HW, (int)Mc);
    }
    if (grad_only) w.colsum_sink = cv.take(d.W);
    else w.mask_bits = reinterpret_cast<uint32_t*>(cv.take(Mc * ceil_div(d.W, 32)));
  }
  if (tc) {     // largest B operand image: a weight [width x (W + encoding)] (the weight gradients read theirs as fp32)
    const int HW = head ? d.HW : 0, Evp = head ? d.Evp : 0;
    const int wmax = std::max(std::max(d.W, HW), std::max(d.E3p, Evp));
    w.pack_elems = tc_pack_elems(wmax, ceil_div(wmax, 32) + ceil_div(std::max(d.E3p, Evp), 32), 0);
    w.pack_b = reinterpret_cast<uint16_t*>(cv.take((w.pack_elems + 1) / 2));
  }
  if (out) *out = w;
  return cv.used + 256;
}

// The workspace a call of `pass` over R rays of S samples (density: M points) checks for.  The two MLP forwards are
// given one size, the larger of the two (sparf_mlp_workspace_bytes with backward = 0), and the plain forward checks
// for that one.
static size_t workspace_need(const MlpDims& d, bool tc, long long R, int S, Pass pass, bool head) {
  auto bytes = [&](Pass p) {
    return carve(d, tc, (int)std::min<long long>(R, chunk_rays(S, p)), S, p, head, nullptr, nullptr);
  };
  return head && pass == Pass::kForward ? std::max(bytes(Pass::kForward), bytes(Pass::kTapedForward)) : bytes(pass);
}

// What the chunk loop of an MLP or density call works with
struct Call {
  MlpDims d;
  bool tc;          // the wide GEMMs run on the tensor cores (gemm_wgmma.cu), else the FFMA kernels above
  int nrc;          // rays (density: points) per chunk
  Ws w;             // the workspace, carved for one chunk
  EnginePrec ep;    // with the workspace's buffer for packed weights
  Tape tape;        // the whole batch's tape (taped passes)
  RowCount rc{nullptr, 0};   // rc.rows != NULL (the *_rows calls, S = 1): the rows are a capacity, *rc.rows live

  // the chunk starting at row m0: the kernels' and GEMMs' live rows are counted from there
  void at(long long m0) {
    if (!rc.rows) return;
    rc.m0 = m0;
    for (TcPrec* p : {&ep.fwd, &ep.dgrad, &ep.wgrad}) p->rows = rc;
  }
};

// The steps every MLP and density call starts with: resolve the engine, validate the network (head: with the colour
// head), check the tape (taped passes: tape != NULL) and the workspace against the pass's sizes, carve the workspace for
// one chunk, and give the GEMMs its pack buffer.  who: the entry point, for the error text.
static int begin_call(const char* who, const SparfMLP* mlp, int engine, long long R, int S, Pass pass, bool head, void* tape,
                      size_t tape_bytes, void* workspace, size_t workspace_bytes, Call* c, long long tape_R = -1) {
  const int e = resolve_engine(engine);
  if (e < 0) {
    set_error("%s: engine %d not available in this build", who, engine);
    return SPARF_ERR_UNSUPPORTED;
  }
  SPARF_TRY(head ? validate_mlp(mlp) : validate_trunk(mlp));
  c->d = mlp_dims(mlp);
  c->tc = is_tc(e);
  if (tape_R < 0) tape_R = R;     // the span forward's tape holds more rows (its capacity) than one call processes
  if (tape) {
    SPARF_REQUIRE(tape_bytes >= tape_layout(c->d, c->tc, (int)tape_R, S, nullptr, nullptr), "%s: tape %zu bytes too small",
                  who, tape_bytes);
    tape_layout(c->d, c->tc, (int)tape_R, S, reinterpret_cast<char*>(align_up(reinterpret_cast<size_t>(tape), 256)),
                &c->tape);
  }
  const size_t need = workspace_need(c->d, c->tc, R, S, pass, head);
  if (workspace_bytes < need) {
    set_error("%s: workspace %zu < %zu bytes", who, workspace_bytes, need);
    return SPARF_ERR_WORKSPACE;
  }
  c->nrc = (int)std::min<long long>(R, chunk_rays(S, pass));
  carve(c->d, c->tc, c->nrc, S, pass, head, reinterpret_cast<char*>(workspace), &c->w);
  c->ep = engine_prec(e);
  for (TcPrec* p : {&c->ep.fwd, &c->ep.dgrad, &c->ep.wgrad}) {
    p->pack_b = c->w.pack_b;
    p->pack_elems = c->w.pack_elems;
  }
  return SPARF_OK;
}

static inline int trunk_in_main(const MlpDims& d, int l) { return l == 0 ? d.E3p : d.W; }
static inline int trunk_in_main_valid(const MlpDims& d, int l) { return l == 0 ? d.E3 : d.W; }
static inline int trunk_ldw(const MlpDims& d, int l) {
  return (l == 0 ? d.E3 : d.W) + (l == d.skip ? d.E3 : 0);
}

// c2f weights and the point encoding of one chunk of Mc rows (rows r * S + k; dirs == NULL: origins are the points,
// S = 1), and on the tensor cores its operand image
static int chunk_encode_xyz(const SparfMLP* mlp, const Call& c, long long Mc, int S, const float* origins,
                            const float* dirs, const float* t, float* enc, cudaStream_t st) {
  const MlpDims& d = c.d;
  C2F c2f{mlp->use_c2f, mlp->c2f_start, mlp->c2f_range, mlp->progress};
  c2f_weights_kernel<<<1, 32, 0, st>>>(c2f, mlp->L_xyz, mlp->L_view, c.w.wts);
  SPARF_CHECK_LAUNCH("c2f_weights_kernel");
  if (c.rc.rows)
    encode_xyz_kernel<true><<<ceil_div(Mc * d.E3p, 256), 256, 0, st>>>(Mc * d.E3p, S, mlp->L_xyz, d.E3p, origins, dirs, t,
                                                                       c.w.wts, enc, c.rc);
  else
    encode_xyz_kernel<<<ceil_div(Mc * d.E3p, 256), 256, 0, st>>>(Mc * d.E3p, S, mlp->L_xyz, d.E3p, origins, dirs, t, c.w.wts,
                                                                 enc, c.rc);
  SPARF_CHECK_LAUNCH("encode_xyz_kernel");
  if (c.tc) SPARF_TRY(tc_pack_rows(c.ep.fwd, (int)Mc, d.E3p, enc, d.E3p, 1, c.w.encimg, st));
  return SPARF_OK;
}

// trunk layers 0 ... nt-1 of one chunk from its encoding.  H: array of nt activation buffers (may alias in pairs);
// H[nt-1] == NULL skips the last layer's feature GEMM (the density row reads H[nt-2] only).  raw (the softplus argument,
// noise added) and sigma may be NULL; both NULL skips the density row.  The tensor-core engines run the layers in one
// fused kernel where trunk_chained says so (H[l] == NULL then means layer l's activation is not kept; bits[l] != NULL
// keeps its ReLU mask), else chain them through the row images their epilogues write (the workspace's image buffers);
// last_image: the last layer's row image is written too (the colour head reads it).
static int chunk_trunk(const SparfMLP* mlp, const Call& c, long long Mc, const float* enc, float* const* H,
                       uint32_t* const* bits, const float* noise, float* raw, float* sigma, bool last_image, cudaStream_t st) {
  const MlpDims& d = c.d;
  const Ws& w = c.w;
  const float* in = enc;
  const bool chained = trunk_chained(d, c.tc);
  if (chained) {
    // the weights as the GEMMs would pack them one by one, then every layer in one launch; H[l] == NULL stays on the SM
    const float* bias[SPARF_MAX_TRUNK];
    for (int l = 0; l < d.nt; ++l) {
      const bool last = l == d.nt - 1;
      bias[l] = mlp->trunk_b[l] + (last ? 1 : 0);
      if (last && !H[l]) break;
      const int ldw = trunk_ldw(d, l);
      SPARF_TRY(tc_pack_nt(c.ep.fwd, d.W, ceil_div(trunk_in_main(d, l), 32), trunk_in_main_valid(d, l),
                           l == d.skip ? w.encimg.ks : 0, d.E3, mlp->trunk_w[l] + (last ? ldw : 0), ldw, d.W, w.wimg[l], st));
    }
    TcOut o;
    if (last_image) {
      o.row = w.Himg[(d.nt - 1) & 1];
      o.row_passes = c.ep.fwd.passes;
    }
    SPARF_TRY(tc_trunk_chain(c.ep.fwd, (int)Mc, d.W, d.nt, d.skip, w.encimg, w.wimg, bias, H, bits, o, st));
  }
  for (int l = 0; l < d.nt; ++l) {
    const bool last = l == d.nt - 1;
    const int ldw = trunk_ldw(d, l);
    const float* Wl = mlp->trunk_w[l] + (last ? ldw : 0);  // last layer: row 0 is the density row
    const float* bl = mlp->trunk_b[l] + (last ? 1 : 0);
    const bool sk = l == d.skip;
    if (chained) {
      // done above
    } else if (c.tc && H[l]) {
      TcOut o;
      if (!last || last_image) {
        o.row = w.Himg[l & 1];
        o.row_passes = c.ep.fwd.passes;
      }
      SPARF_TRY(tc_gemm_nt(c.ep.fwd, 1, (int)Mc, d.W, l == 0 ? w.encimg : w.Himg[(l - 1) & 1], trunk_in_main_valid(d, l),
                           sk ? w.encimg : TcImage{}, d.E3, Wl, ldw, d.W, bl, H[l], d.W, o, st));
    } else if (H[l]) {
      SPARF_TRY(gemm_nt((int)Mc, d.W, in, trunk_in_main(d, l), trunk_in_main(d, l), trunk_in_main_valid(d, l),
                        sk ? enc : nullptr, d.E3p, d.E3p, d.E3, 1, Wl, ldw, d.W, bl, H[l], d.W, st));
    }
    if (last && (raw || sigma)) {
      if (c.rc.rows)
        rowdot_kernel<0, true><<<ceil_div(Mc, 8), 256, 0, st>>>(Mc, d.W, in, d.W, mlp->trunk_w[l], ldw, mlp->trunk_b[l], noise,
                                                                raw, sigma, c.rc);
      else
        rowdot_kernel<0><<<ceil_div(Mc, 8), 256, 0, st>>>(Mc, d.W, in, d.W, mlp->trunk_w[l], ldw, mlp->trunk_b[l], noise, raw,
                                                         sigma, c.rc);
      SPARF_CHECK_LAUNCH("rowdot_kernel<0>");
    }
    in = H[l];
  }
  return SPARF_OK;
}

// forward through the MLP for one chunk of nr rays into the activations v (v.raw may be NULL); sigma may be NULL.  The
// tensor-core engines pack the encodings once.
static int chunk_forward(const SparfMLP* mlp, const Call& c, int nr, int S, const float* origins, const float* dirs,
                         const float* t, const float* noise, const Tape& v, float* sigma, float* rgb, cudaStream_t st) {
  const MlpDims& d = c.d;
  const long long Mc = (long long)nr * S;
  SPARF_TRY(chunk_encode_xyz(mlp, c, Mc, S, origins, dirs, t, v.enc, st));
  if (c.rc.rows)
    encode_dir_kernel<true><<<ceil_div((long long)nr * d.Evp, 256), 256, 0, st>>>(nr * d.Evp, mlp->L_view, d.Evp, dirs,
                                                                                  c.w.wts + 16, v.denc, c.rc);
  else
    encode_dir_kernel<<<ceil_div((long long)nr * d.Evp, 256), 256, 0, st>>>(nr * d.Evp, mlp->L_view, d.Evp, dirs, c.w.wts + 16,
                                                                            v.denc, c.rc);
  SPARF_CHECK_LAUNCH("encode_dir_kernel");
  if (c.tc) SPARF_TRY(tc_pack_rows(c.ep.fwd, (int)Mc, d.Evp, v.denc, d.Evp, S, c.w.dencimg, st));
  SPARF_TRY(chunk_trunk(mlp, c, Mc, v.enc, v.H, v.bits, noise, v.raw, sigma, true, st));
  if (c.tc)
    SPARF_TRY(tc_gemm_nt(c.ep.fwd, 1, (int)Mc, d.HW, c.w.Himg[(d.nt - 1) & 1], d.W, c.w.dencimg, d.Ev, mlp->head_w[0],
                         d.W + d.Ev, d.W, mlp->head_b[0], v.hid, d.HW, TcOut{}, st));
  else
    SPARF_TRY(gemm_nt((int)Mc, d.HW, v.H[d.nt - 1], d.W, d.W, d.W, v.denc, d.Evp, d.Evp, d.Ev, S, mlp->head_w[0], d.W + d.Ev,
                      d.W, mlp->head_b[0], v.hid, d.HW, st));
  if (c.rc.rows)
    rowdot_kernel<1, true><<<ceil_div(Mc, 8), 256, 0, st>>>(Mc, d.HW, v.hid, d.HW, mlp->head_w[1], d.HW, mlp->head_b[1], nullptr,
                                                            nullptr, rgb, c.rc);
  else
    rowdot_kernel<1><<<ceil_div(Mc, 8), 256, 0, st>>>(Mc, d.HW, v.hid, d.HW, mlp->head_w[1], d.HW, mlp->head_b[1], nullptr,
                                                     nullptr, rgb, c.rc);
  SPARF_CHECK_LAUNCH("rowdot_kernel<1>");
  return SPARF_OK;
}

// The taped calls with a device row count (sparf_mlp_*_tape_rows, sparf_mlp_forward_tape_span): tensor-core engines and
// one-sample rays only.  start (span forward only; may be NULL): the device row the call's rows start at.
static int rows_call(const char* who, Call* c, int S, const int64_t* rows, const int64_t* start = nullptr) {
  if (!rows) return SPARF_OK;
  if (!c->tc) {
    set_error("%s: a device row count needs a tensor-core engine (tc_3x, tc_1x or tc_3x_w1)", who);
    return SPARF_ERR_UNSUPPORTED;
  }
  SPARF_REQUIRE(S == 1, "%s: a device row count needs S = 1 (one-sample rays), got S = %d", who, S);
  c->rc.rows = rows;
  c->rc.start = start;
  return SPARF_OK;
}

// The MLP forward, chunk by chunk.  tape == NULL: the activations stay in the workspace; else they go straight into the
// tape.  rows != NULL (taped, S = 1): R is a capacity, *rows the rays evaluated.  start != NULL as well (the span
// forward): the rows [*start, *rows) of the global buffers, at most R of them, and the tape holds tape_R rows.
static int mlp_forward(const SparfMLP* mlp, int engine, int R, int S, const float* origins, const float* dirs, const float* t,
                       const float* noise, float* sigma, float* rgb, void* tape, size_t tape_bytes, void* workspace,
                       size_t workspace_bytes, cudaStream_t st, const int64_t* rows = nullptr,
                       const int64_t* start = nullptr, long long tape_R = -1) {
  Call c;
  const char* who = start ? "mlp_forward_tape_span" : rows ? "mlp_forward_tape_rows" : tape ? "mlp_forward_tape" : "mlp_forward";
  SPARF_TRY(begin_call(who, mlp, engine, R, S, tape ? Pass::kTapedForward : Pass::kForward, true, tape, tape_bytes, workspace,
                       workspace_bytes, &c, tape_R));
  SPARF_TRY(rows_call(who, &c, S, rows, start));
  Tape v = c.w.act;
  v.raw = nullptr;      // the plain forward does not keep the softplus argument
  for (int r0 = 0; r0 < R; r0 += c.nrc) {
    const int nr = std::min(c.nrc, R - r0);
    c.at(r0);
    const size_t m0 = (size_t)r0 * S;
    SPARF_TRY(chunk_forward(mlp, c, nr, S, origins + (size_t)r0 * 3, dirs + (size_t)r0 * 3, t + m0, noise ? noise + m0 : nullptr,
                            tape ? tape_chunk(c.tape, c.d, r0, S) : v, sigma + m0, rgb + m0 * 3, st));
  }
  return SPARF_OK;
}

constexpr int kSimtSlab = 2048;   // rows per SIMT wgrad slab (the tensor-core GEMMs choose their own k-ranges)

// tensor cores: the trunk gradients G leave each input-gradient GEMM as images, in ping-pong buffer i: a row image (the
// next input gradient's A operand) and a transposed one (K = this chunk's Mc rows; the weight gradient's A operand)
static TcImage grad_tr(const Ws& w, int i, long long Mc) { return TcImage{w.Gtr[i].p, ceil_div(Mc, 32)}; }
static TcOut grad_images(const Call& c, int i, long long Mc) {
  TcOut o;
  o.row = c.w.Grow[i];
  o.tr = grad_tr(c.w, i, Mc);
  o.row_passes = c.ep.dgrad.passes;
  o.tr_passes = c.ep.wgrad.passes;
  return o;
}

// Colour-head backward of one chunk of Mc rows (S samples per ray) from d_rgb, d_sigma and the forward's rgbv and
// activations v, on the CUDA cores.  Leaves the density row's gradient in w.graw, the last trunk layer's feature gradient
// in w.G0 and, when dir_grad, the gradient of each row's view-direction encoding in w.Gdtmp.
static int head_backward_simt(const SparfMLP* mlp, const Call& c, long long Mc, int S, const float* d_rgb, const float* rgbv,
                              const float* d_sigma, const Tape& v, const SparfMLPGrad* grad, bool dir_grad, cudaStream_t st) {
  const MlpDims& d = c.d;
  const Ws& w = c.w;
  const int ldw8 = d.W + d.Ev;
  const float* feat = v.H[d.nt - 1];
  head_grad_kernel<<<ceil_div(Mc, 256), 256, 0, st>>>(Mc, d_rgb, rgbv, d_sigma, v.raw, w.gpre, w.graw);
  SPARF_CHECK_LAUNCH("head_grad_kernel");
  // colour head, layer 1 (HW -> 3)
  narrow_wgrad_kernel<3><<<ceil_div(Mc, 512), 128, 0, st>>>(Mc, d.HW, 512, w.gpre, 4, v.hid, d.HW, grad->head_w[1], d.HW,
                                                             grad->head_b[1]);
  SPARF_CHECK_LAUNCH("narrow_wgrad_kernel<3>");
  narrow_dgrad_kernel<<<ceil_div(Mc * d.HW, 256), 256, 0, st>>>(Mc * d.HW, d.HW, w.gpre, mlp->head_w[1], d.HW, v.hid, w.Ghid);
  SPARF_CHECK_LAUNCH("narrow_dgrad_kernel");
  // colour head, layer 0 ([feat | denc] -> HW)
  SPARF_TRY(gemm_tn((int)Mc, d.HW, d.W, d.W, kSimtSlab, w.Ghid, d.HW, feat, d.W, 1, grad->head_w[0], ldw8, 0, st));
  SPARF_TRY(gemm_tn((int)Mc, d.HW, d.Evp, d.Ev, kSimtSlab, w.Ghid, d.HW, v.denc, d.Evp, S, grad->head_w[0], ldw8, d.W, st));
  colsum_kernel<<<dim3(ceil_div(d.HW, 32), ceil_div(Mc, 1024)), 256, 0, st>>>(Mc, d.HW, 1024, w.Ghid, d.HW, grad->head_b[0]);
  SPARF_CHECK_LAUNCH("colsum_kernel(head)");
  SPARF_TRY(gemm_nn((int)Mc, d.HW, d.W, d.W, w.Ghid, d.HW, mlp->head_w[0], ldw8, 0, feat, d.W, nullptr, nullptr, w.G0, d.W, 0, st));
  if (dir_grad)
    SPARF_TRY(gemm_nn((int)Mc, d.HW, d.Evp, d.Ev, w.Ghid, d.HW, mlp->head_w[0], ldw8, d.W, nullptr, 0, nullptr, nullptr, w.Gdtmp,
                      d.Evp, 0, st));
  return SPARF_OK;
}

// The same on the tensor cores: layer 1 (HW -> 3) and the head's gradients in one kernel that writes Ghid as images,
// then layer 0 ([feat | denc] -> HW), whose input gradient leaves as image pair 0 of the trunk gradients, with the bias
// gradient of the last trunk layer.
static int head_backward_tc(const SparfMLP* mlp, const Call& c, long long Mc, int S, const float* d_rgb, const float* rgbv,
                            const float* d_sigma, const Tape& v, const SparfMLPGrad* grad, bool dir_grad, cudaStream_t st) {
  const MlpDims& d = c.d;
  const Ws& w = c.w;
  const EnginePrec& ep = c.ep;
  const int ldw8 = d.W + d.Ev;
  const float* feat = v.H[d.nt - 1];
  const TcImage ghid_t{w.ghid_tr.p, ceil_div(Mc, 32)}, ghid = w.ghid_row;
  SPARF_TRY(tc_head_backward(ep.dgrad, ep.wgrad, (int)Mc, d.HW, d_rgb, rgbv, d_sigma, v.raw, v.hid, mlp->head_w[1], w.graw, ghid,
                             ghid_t, grad->head_w[1], grad->head_b[1], grad->head_b[0], grad->trunk_b[d.nt - 1], st));
  // the weight gradient of feat writes its ReLU mask bits, the input gradient of feat reads them
  SPARF_TRY(tc_gemm_tn(ep.wgrad, (int)Mc, d.HW, d.W, d.W, ghid_t, feat, d.W, 1, grad->head_w[0], ldw8, 0, w.mask_bits, st));
  SPARF_TRY(tc_gemm_tn(ep.wgrad, (int)Mc, d.HW, d.Evp, d.Ev, ghid_t, v.denc, d.Evp, S, grad->head_w[0], ldw8, d.W, nullptr, st));
  SPARF_TRY(tc_gemm_nn(ep.dgrad, (int)Mc, d.HW, d.W, d.W, ghid, mlp->head_w[0], ldw8, 0, nullptr, 0, w.mask_bits, nullptr,
                       nullptr, nullptr, 0, 0, grad_images(c, 0, Mc), grad->trunk_b[d.nt - 1] + 1, nullptr, st));
  if (dir_grad)
    SPARF_TRY(tc_gemm_nn(ep.dgrad, (int)Mc, d.HW, d.Evp, d.Ev, ghid, mlp->head_w[0], ldw8, d.W, nullptr, 0, nullptr, nullptr,
                         nullptr, w.Gdtmp, d.Evp, 0, TcOut{}, nullptr, nullptr, st));
  return SPARF_OK;
}

// Backward through trunk layers nt-1 ... 0 of one chunk of Mc rows on the CUDA cores, from the gradient of the last
// layer's features in w.G0 and of its density row, graw (may be NULL: zero).  H: the chunk's nt-1 first trunk
// activations, enc its encoding.  Parameter gradients +=, the encoding's gradient into w.Genc when enc_grad.
// grad == NULL: no weight or bias gradient, only the input gradients (the point gradient of sparf_density_gradient).
static int trunk_backward_simt(const SparfMLP* mlp, const Call& c, long long Mc, const float* enc, float* const* H,
                               const float* graw, const SparfMLPGrad* grad, bool enc_grad, cudaStream_t st) {
  const MlpDims& d = c.d;
  float* G = c.w.G0;
  float* Gn = c.w.G1;
  bool genc_written = false;
  for (int l = d.nt - 1; l >= 0; --l) {
    const bool last = l == d.nt - 1;
    const bool r1 = last && graw;       // the density row's rank-1 term: z = [raw | feat_pre]
    const int ldw = trunk_ldw(d, l);
    const float* in = l == 0 ? enc : H[l - 1];
    const int Kin = trunk_in_main(d, l), Kinv = trunk_in_main_valid(d, l);
    const int rowoff = last ? 1 : 0;
    const float* Wl = mlp->trunk_w[l] + (size_t)rowoff * ldw;
    if (grad) {
      float* dWl = grad->trunk_w[l] + (size_t)rowoff * ldw;
      SPARF_TRY(gemm_tn((int)Mc, d.W, Kin, Kinv, kSimtSlab, G, d.W, in, Kin, 1, dWl, ldw, 0, st));
      if (l == d.skip) SPARF_TRY(gemm_tn((int)Mc, d.W, d.E3p, d.E3, kSimtSlab, G, d.W, enc, d.E3p, 1, dWl, ldw, d.W, st));
      colsum_kernel<<<dim3(ceil_div(d.W, 32), ceil_div(Mc, 1024)), 256, 0, st>>>(Mc, d.W, 1024, G, d.W, grad->trunk_b[l] + rowoff);
      SPARF_CHECK_LAUNCH("colsum_kernel(trunk)");
      if (r1) {
        narrow_wgrad_kernel<1><<<ceil_div(Mc, 512), 128, 0, st>>>(Mc, d.W, 512, graw, 1, in, d.W, grad->trunk_w[l], ldw,
                                                                   grad->trunk_b[l]);
        SPARF_CHECK_LAUNCH("narrow_wgrad_kernel<1>");
      }
    }
    if (l > 0)
      SPARF_TRY(gemm_nn((int)Mc, d.W, d.W, d.W, G, d.W, Wl, ldw, 0, in, d.W, r1 ? graw : nullptr, r1 ? mlp->trunk_w[l] : nullptr,
                        Gn, d.W, 0, st));
    if (enc_grad && (l == d.skip || l == 0)) {
      SPARF_TRY(gemm_nn((int)Mc, d.W, d.E3p, d.E3, G, d.W, Wl, ldw, l == 0 ? 0 : d.W, nullptr, 0, nullptr, nullptr, c.w.Genc,
                        d.E3p, genc_written ? 1 : 0, st));
      genc_written = true;
    }
    std::swap(G, Gn);
  }
  return SPARF_OK;
}

// The image buffers of G_l, the gradient of trunk layer l's output (G_{nt-1} is buffer 0, the head's or the caller's).
// Layer by layer they ping-pong.  With the chained input gradients every transposed image of G_{nt-2} ... G_0 is alive
// until the weight gradients that follow the chain, G_0's in G_{nt-1}'s buffer (whose weight gradient ran before the
// chain); the chain's input is G_{nt-2}'s row image, and the row images it writes for the encoding's gradient go to the
// two row buffers: G_0's over G_{nt-1}'s, G_skip's over G_{nt-2}'s, each 128-row tile of which is read only by the CTA
// that writes it there afterwards.
static int grad_tr_buf(const MlpDims& d, bool chained, int l) { return chained ? (l ? d.nt - 1 - l : 0) : (d.nt - 1 - l) & 1; }
static int grad_row(const MlpDims& d, bool chained, int l) {
  return chained ? (l == 0 || l == d.nt - 1 ? 0 : 1) : (d.nt - 1 - l) & 1;
}

// The input gradients of layers nt-2 ... 1 in one launch (tc_dgrad_chain), from G_{nt-2}'s row image and the masks the
// fused forward kept (bits[l - 1] = H_{l-1} > 0), into the transposed images of G_{nt-3} ... G_0, the bias gradients of
// layers nt-3 ... 0 and, with enc_grad, the row images of G_skip and G_0.
static int chunk_dgrad_chain(const SparfMLP* mlp, const Call& c, long long Mc, uint32_t* const* bits, const SparfMLPGrad* grad,
                             bool enc_grad, cudaStream_t st) {
  const MlpDims& d = c.d;
  const int top = d.nt - 2;
  const uint32_t* mask[SPARF_MAX_TRUNK] = {};
  float* db[SPARF_MAX_TRUNK] = {};
  TcImage tr[SPARF_MAX_TRUNK], row[SPARF_MAX_TRUNK];
  for (int l = top; l >= 1; --l) {
    SPARF_TRY(tc_pack_nn(c.ep.dgrad, d.W, d.W, d.W, mlp->trunk_w[l], trunk_ldw(d, l), 0, c.w.nnimg[l], st));
    mask[l] = bits[l - 1];
    db[l] = grad ? grad->trunk_b[l - 1] : c.w.colsum_sink;    // the chain always sums its columns
    tr[l] = grad_tr(c.w, grad_tr_buf(d, true, l - 1), Mc);
    if (enc_grad && (l - 1 == 0 || l - 1 == d.skip)) row[l] = c.w.Grow[grad_row(d, true, l - 1)];
  }
  return tc_dgrad_chain(c.ep.dgrad, c.ep.wgrad, (int)Mc, d.W, top, c.w.Grow[grad_row(d, true, top)], c.w.nnimg, mask, db, tr,
                        row, st);
}

// The same on the tensor cores, from the last layer's feature gradient as image pair 0.  The last layer's bias gradient
// is the caller's: the kernel that made image pair 0 adds it (the SIMT path adds the column sums of G0).  The last layer's
// input-gradient epilogue also sums the density row's weight gradient.
// bits: the fused forward's ReLU masks of H_0 ... H_{nt-3} (trunk_chained: the input gradients of layers nt-2 ... 1 run
// as one chain once layer nt-1 is done, and the weight gradients of the layers below it after that).
// grad == NULL: no weight gradient GEMM; every input gradient reads its mask from the fp32 H_{l-1}, the chain's bias sums
// go to w.colsum_sink and the transposed images, which only weight gradients read, to one shared buffer.
static int trunk_backward_tc(const SparfMLP* mlp, const Call& c, long long Mc, const float* enc, float* const* H,
                             uint32_t* const* bits, const float* graw, const SparfMLPGrad* grad, bool enc_grad, cudaStream_t st) {
  const MlpDims& d = c.d;
  const EnginePrec& ep = c.ep;
  const bool chained = trunk_chained(d, true);
  bool genc_written = false;
  for (int l = d.nt - 1; l >= 0; --l) {
    const bool last = l == d.nt - 1;
    const bool r1 = last && graw;       // the density row's rank-1 term: z = [raw | feat_pre]
    const int ldw = trunk_ldw(d, l);
    const float* in = l == 0 ? enc : H[l - 1];
    const int Kin = trunk_in_main(d, l), Kinv = trunk_in_main_valid(d, l);
    const int rowoff = last ? 1 : 0;
    const float* Wl = mlp->trunk_w[l] + (size_t)rowoff * ldw;
    const int gi = (d.nt - 1 - l) & 1;   // layer by layer: the layer's output gradient is image pair gi
    const bool nn = l > 0 && (!chained || last);   // the input gradient is a GEMM of its own
    // The input gradient's ReLU mask is H_{l-1} > 0: as bits that the weight gradient writes while it reads H_{l-1} anyway,
    // except with the density row's rank-1 term, whose weight gradient (r1_wgrad) the epilogue sums from the fp32 values
    // of H_{l-1}: that layer reads them as its mask.
    uint32_t* wbits = grad && nn && !r1 ? c.w.mask_bits : nullptr;
    if (grad) {
      float* dWl = grad->trunk_w[l] + (size_t)rowoff * ldw;
      const TcImage gt = grad_tr(c.w, grad_tr_buf(d, chained, l), Mc);
      SPARF_TRY(tc_gemm_tn(ep.wgrad, (int)Mc, d.W, Kin, Kinv, gt, in, Kin, 1, dWl, ldw, 0, wbits, st));
      if (l == d.skip) SPARF_TRY(tc_gemm_tn(ep.wgrad, (int)Mc, d.W, d.E3p, d.E3, gt, enc, d.E3p, 1, dWl, ldw, d.W, nullptr, st));
    }
    if (nn)
      SPARF_TRY(tc_gemm_nn(ep.dgrad, (int)Mc, d.W, d.W, d.W, c.w.Grow[gi], Wl, ldw, 0, wbits ? nullptr : in, d.W, wbits,
                           r1 ? graw : nullptr, r1 ? mlp->trunk_w[l] : nullptr, nullptr, 0, 0, grad_images(c, gi ^ 1, Mc),
                           grad ? grad->trunk_b[l - 1] : nullptr, grad && r1 ? grad->trunk_w[l] : nullptr, st));
    if (enc_grad && (l == d.skip || l == 0)) {
      SPARF_TRY(tc_gemm_nn(ep.dgrad, (int)Mc, d.W, d.E3p, d.E3, c.w.Grow[grad_row(d, chained, l)], Wl, ldw, l == 0 ? 0 : d.W,
                           nullptr, 0, nullptr, nullptr, nullptr, c.w.Genc, d.E3p, genc_written ? 1 : 0, TcOut{}, nullptr,
                           nullptr, st));
      genc_written = true;
    }
    if (chained && last) SPARF_TRY(chunk_dgrad_chain(mlp, c, Mc, bits, grad, enc_grad, st));
  }
  return SPARF_OK;
}

// The MLP backward, chunk by chunk.  tape == NULL: recompute each chunk's forward in the workspace (noise as in the
// forward call); else read the activations from the tape and the colour output from rgb_fwd, the forward's.  rows: as
// in mlp_forward.
static int mlp_backward(const SparfMLP* mlp, int engine, int R, int S, const float* origins, const float* dirs, const float* t,
                        const float* noise, const float* rgb_fwd, void* tape, size_t tape_bytes, const float* d_sigma,
                        const float* d_rgb, const SparfMLPGrad* grad, float* d_origins, float* d_dirs, void* workspace,
                        size_t workspace_bytes, cudaStream_t st, const int64_t* rows = nullptr) {
  Call c;
  const char* who = rows ? "mlp_backward_tape_rows" : tape ? "mlp_backward_tape" : "mlp_backward";
  SPARF_TRY(begin_call(who, mlp, engine, R, S, tape ? Pass::kTapedBackward : Pass::kRecomputeBackward, true, tape, tape_bytes,
                       workspace, workspace_bytes, &c));
  SPARF_TRY(rows_call(who, &c, S, rows));
  const MlpDims& d = c.d;
  const Ws& w = c.w;
  const bool need_rays = d_origins != nullptr || d_dirs != nullptr;
  for (int r0 = 0; r0 < R; r0 += c.nrc) {
    const int nr = std::min(c.nrc, R - r0);
    c.at(r0);
    const long long Mc = (long long)nr * S;
    const size_t m0 = (size_t)r0 * S;
    const float* d_c = dirs + (size_t)r0 * 3;
    const Tape v = tape ? tape_chunk(c.tape, d, r0, S) : w.act;
    const float* rgbv = tape ? rgb_fwd + m0 * 3 : w.rgbv;
    if (!tape)
      SPARF_TRY(chunk_forward(mlp, c, nr, S, origins + (size_t)r0 * 3, d_c, t + m0, noise ? noise + m0 : nullptr, v, nullptr,
                              w.rgbv, st));
    SPARF_TRY(c.tc ? head_backward_tc(mlp, c, Mc, S, d_rgb + m0 * 3, rgbv, d_sigma + m0, v, grad, d_dirs != nullptr, st)
                   : head_backward_simt(mlp, c, Mc, S, d_rgb + m0 * 3, rgbv, d_sigma + m0, v, grad, d_dirs != nullptr, st));
    if (d_dirs) {
      if (c.rc.rows) {
        ray_reduce_kernel<true><<<ceil_div((long long)nr * d.Evp, 256), 256, 0, st>>>(nr, S, d.Evp, w.Gdtmp, w.Gdenc, c.rc);
        SPARF_CHECK_LAUNCH("ray_reduce_kernel");
        direnc_bwd_kernel<true><<<ceil_div(nr, 128), 128, 0, st>>>(nr, mlp->L_view, d.Evp, v.denc, w.Gdenc, d_c,
                                                                   d_dirs + (size_t)r0 * 3, c.rc);
      } else {
        ray_reduce_kernel<<<ceil_div((long long)nr * d.Evp, 256), 256, 0, st>>>(nr, S, d.Evp, w.Gdtmp, w.Gdenc, c.rc);
        SPARF_CHECK_LAUNCH("ray_reduce_kernel");
        direnc_bwd_kernel<<<ceil_div(nr, 128), 128, 0, st>>>(nr, mlp->L_view, d.Evp, v.denc, w.Gdenc, d_c, d_dirs + (size_t)r0 * 3,
                                                             c.rc);
      }
      SPARF_CHECK_LAUNCH("direnc_bwd_kernel");
    }
    SPARF_TRY(c.tc ? trunk_backward_tc(mlp, c, Mc, v.enc, v.H, v.bits, w.graw, grad, need_rays, st)
                   : trunk_backward_simt(mlp, c, Mc, v.enc, v.H, w.graw, grad, need_rays, st));
    if (need_rays) {
      float* d_o = d_origins ? d_origins + (size_t)r0 * 3 : nullptr;
      float* d_d = d_dirs ? d_dirs + (size_t)r0 * 3 : nullptr;
      if (c.rc.rows)
        posenc_bwd_kernel<true><<<ceil_div(nr, 4), 128, 0, st>>>(nr, S, mlp->L_xyz, d.E3p, v.enc, w.Genc, t + m0, d_o, d_d, c.rc);
      else
        posenc_bwd_kernel<<<ceil_div(nr, 4), 128, 0, st>>>(nr, S, mlp->L_xyz, d.E3p, v.enc, w.Genc, t + m0, d_o, d_d, c.rc);
      SPARF_CHECK_LAUNCH("posenc_bwd_kernel");
    }
  }
  return SPARF_OK;
}

// tc_feat_backward and the path it stands for (relu_mask_kernel's fp32 G, then tc_pack_rows / tc_pack_cols and
// colsum_kernel) on the same inputs; scratch = G [M x W]
static int selftest_featgrad(const float* d_raw, const float* d_feat, const float* feat, int M, int W, TcPrec dg, TcPrec wg,
                             uint16_t* img, float* sums, float* scratch, cudaStream_t st) {
  const size_t nrow = tc_image_elems(M, W), ntr = tc_image_elems(W, M);
  const TcImage row{img, ceil_div(W, 32)}, tr{img + nrow, ceil_div(M, 32)};
  const TcImage row_ref{img + nrow + ntr, row.ks}, tr_ref{img + 2 * nrow + ntr, tr.ks};
  float* ref = sums + W + 1;
  SPARF_CHECK_CUDA(cudaMemsetAsync(img, 0xFF, 2 * (nrow + ntr) * sizeof(uint16_t), st));
  SPARF_CHECK_CUDA(cudaMemsetAsync(sums, 0, 2 * (W + 1) * sizeof(float), st));
  SPARF_TRY(tc_feat_backward(dg, wg, M, W, d_raw, d_feat, feat, row, tr, sums, sums + 1, st));
  relu_mask_kernel<<<ceil_div((long long)M * W, 256), 256, 0, st>>>((long long)M * W, feat, d_feat, scratch);
  SPARF_CHECK_LAUNCH("relu_mask_kernel");
  colsum_kernel<<<dim3(ceil_div(W, 32), ceil_div(M, 1024)), 256, 0, st>>>(M, W, 1024, scratch, W, ref + 1);
  SPARF_CHECK_LAUNCH("colsum_kernel");
  colsum_kernel<<<dim3(1, ceil_div(M, 1024)), 256, 0, st>>>(M, 1, 1024, d_raw, 1, ref);
  SPARF_CHECK_LAUNCH("colsum_kernel");
  SPARF_TRY(tc_pack_rows(dg, M, W, scratch, W, 1, row_ref, st));
  return tc_pack_cols(wg, M, W, scratch, W, tr_ref, st);
}

// tc_head_backward and the path it replaced (head_grad_kernel, narrow_dgrad_kernel's fp32 Ghid, then tc_pack_rows /
// tc_pack_cols) on the same inputs; scratch = Ghid [M x HW], gpre [M x 4], the fused kernel's sums [4 HW + 4]
static int selftest_head(const float* d_rgb, const float* rgb, const float* d_sigma, const float* raw, const float* hid,
                         const float* W9, int M, int HW, TcPrec dg, TcPrec wg, uint16_t* img, float* graw, float* scratch,
                         cudaStream_t st) {
  const size_t nrow = tc_image_elems(M, HW), ntr = tc_image_elems(HW, M);
  const TcImage row{img, ceil_div(HW, 32)}, tr{img + nrow, ceil_div(M, 32)};
  const TcImage row_ref{img + nrow + ntr, row.ks}, tr_ref{img + 2 * nrow + ntr, tr.ks};
  float *Ghid = scratch, *gpre = Ghid + (size_t)M * HW, *sums = gpre + (size_t)M * 4;
  SPARF_CHECK_CUDA(cudaMemsetAsync(img, 0xFF, 2 * (nrow + ntr) * sizeof(uint16_t), st));
  SPARF_CHECK_CUDA(cudaMemsetAsync(sums, 0, (4 * HW + 4) * sizeof(float), st));
  SPARF_TRY(tc_head_backward(dg, wg, M, HW, d_rgb, rgb, d_sigma, raw, hid, W9, graw, row, tr, sums, sums + 3 * HW,
                             sums + 3 * HW + 3, sums + 4 * HW + 3, st));
  head_grad_kernel<<<ceil_div(M, 256), 256, 0, st>>>(M, d_rgb, rgb, d_sigma, raw, gpre, graw + M);
  SPARF_CHECK_LAUNCH("head_grad_kernel");
  narrow_dgrad_kernel<<<ceil_div((long long)M * HW, 256), 256, 0, st>>>((long long)M * HW, HW, gpre, W9, HW, hid, Ghid);
  SPARF_CHECK_LAUNCH("narrow_dgrad_kernel");
  SPARF_TRY(tc_pack_rows(dg, M, HW, Ghid, HW, 1, row_ref, st));
  return tc_pack_cols(wg, M, HW, Ghid, HW, tr_ref, st);
}

}  // namespace sparf

using namespace sparf;

// ------------------------------------------------------------------------------------------------
// C ABI: the MLP calls, and the density queries (the trunk alone at arbitrary points, NeRF.compute_raw_density; rows =
// points, S = 1, without the colour head's buffers)
// ------------------------------------------------------------------------------------------------
extern "C" size_t sparf_mlp_workspace_bytes(const SparfMLP* mlp, int32_t R, int32_t S, int32_t backward, int32_t engine) {
  if (!mlp || R <= 0 || S <= 0) return 0;
  const int e = resolve_engine(engine);
  if (e < 0 || backward < 0 || backward > 2) return 0;
  const Pass pass = backward == 0 ? Pass::kForward : backward == 1 ? Pass::kRecomputeBackward : Pass::kTapedBackward;
  return workspace_need(mlp_dims(mlp), is_tc(e), R, S, pass, true);
}

extern "C" int sparf_mlp_forward(const SparfMLP* mlp, int32_t engine, int32_t R, int32_t S, const float* origins,
                                 const float* dirs, const float* t, const float* noise, float* sigma, float* rgb,
                                 void* workspace, size_t workspace_bytes, sparf_stream_t stream) {
  SPARF_REQUIRE(mlp && R >= 0 && S > 0, "mlp_forward: bad arguments");
  SPARF_REQUIRE(origins && dirs && t && sigma && rgb, "mlp_forward: NULL tensor");
  if (R == 0) return SPARF_OK;
  return mlp_forward(mlp, engine, R, S, origins, dirs, t, noise, sigma, rgb, nullptr, 0, workspace, workspace_bytes,
                     (cudaStream_t)stream);
}

extern "C" int sparf_mlp_backward(const SparfMLP* mlp, int32_t engine, int32_t R, int32_t S, const float* origins,
                                  const float* dirs, const float* t, const float* noise, const float* d_sigma,
                                  const float* d_rgb, const SparfMLPGrad* grad, float* d_origins, float* d_dirs,
                                  void* workspace, size_t workspace_bytes, sparf_stream_t stream) {
  SPARF_REQUIRE(mlp && R >= 0 && S > 0, "mlp_backward: bad arguments");
  SPARF_REQUIRE(origins && dirs && t && d_sigma && d_rgb && grad, "mlp_backward: NULL tensor");
  if (R == 0) return SPARF_OK;
  return mlp_backward(mlp, engine, R, S, origins, dirs, t, noise, nullptr, nullptr, 0, d_sigma, d_rgb, grad, d_origins, d_dirs,
                      workspace, workspace_bytes, (cudaStream_t)stream);
}

// tape variants: the training forward keeps what the backward needs, so that the backward does not recompute the forward
extern "C" size_t sparf_mlp_tape_bytes(const SparfMLP* mlp, int32_t engine, int32_t R, int32_t S) {
  if (!mlp || R <= 0 || S <= 0 || resolve_engine(engine) < 0 || validate_mlp(mlp)) return 0;
  const size_t n = tape_layout(mlp_dims(mlp), is_tc(resolve_engine(engine)), R, S, nullptr, nullptr);
  return n <= kMaxTapeBytes ? n : 0;
}

extern "C" int sparf_mlp_forward_tape(const SparfMLP* mlp, int32_t engine, int32_t R, int32_t S, const float* origins,
                                      const float* dirs, const float* t, const float* noise, float* sigma, float* rgb,
                                      void* tape, size_t tape_bytes, void* workspace, size_t workspace_bytes,
                                      sparf_stream_t stream) {
  SPARF_REQUIRE(mlp && R > 0 && S > 0 && origins && dirs && t && sigma && rgb && tape, "mlp_forward_tape: bad arguments");
  return mlp_forward(mlp, engine, R, S, origins, dirs, t, noise, sigma, rgb, tape, tape_bytes, workspace, workspace_bytes,
                     (cudaStream_t)stream);
}

extern "C" int sparf_mlp_backward_tape(const SparfMLP* mlp, int32_t engine, int32_t R, int32_t S, const float* origins,
                                       const float* dirs, const float* t, const float* sigma, const float* rgb,
                                       const float* d_sigma, const float* d_rgb, const SparfMLPGrad* grad,
                                       float* d_origins, float* d_dirs, void* tape, size_t tape_bytes, void* workspace,
                                       size_t workspace_bytes, sparf_stream_t stream) {
  SPARF_REQUIRE(mlp && R > 0 && S > 0 && origins && dirs && t && sigma && rgb && d_sigma && d_rgb && grad && tape,
                "mlp_backward_tape: bad arguments");
  return mlp_backward(mlp, engine, R, S, origins, dirs, t, nullptr, rgb, tape, tape_bytes, d_sigma, d_rgb, grad, d_origins,
                      d_dirs, workspace, workspace_bytes, (cudaStream_t)stream);
}

// the taped pair with a device row count: R = C is the capacity, *rows = K the rows evaluated
extern "C" int sparf_mlp_forward_tape_rows(const SparfMLP* mlp, int32_t engine, int32_t R, int32_t S, const int64_t* rows,
                                           const float* origins, const float* dirs, const float* t, const float* noise,
                                           float* sigma, float* rgb, void* tape, size_t tape_bytes, void* workspace,
                                           size_t workspace_bytes, sparf_stream_t stream) {
  SPARF_REQUIRE(mlp && R > 0 && S > 0 && rows && origins && dirs && t && sigma && rgb && tape,
                "mlp_forward_tape_rows: bad arguments");
  return mlp_forward(mlp, engine, R, S, origins, dirs, t, noise, sigma, rgb, tape, tape_bytes, workspace, workspace_bytes,
                     (cudaStream_t)stream, rows);
}

// the taped forward over the device-side row span [*begin, min(*end, *begin + cap)) of capacity-C buffers and tape
extern "C" int sparf_mlp_forward_tape_span(const SparfMLP* mlp, int32_t engine, int32_t C, int32_t cap, const int64_t* begin,
                                           const int64_t* end, const float* origins, const float* dirs, const float* t,
                                           const float* noise, float* sigma, float* rgb, void* tape, size_t tape_bytes,
                                           void* workspace, size_t workspace_bytes, sparf_stream_t stream) {
  SPARF_REQUIRE(mlp && C > 0 && cap > 0 && cap <= C && begin && end && origins && dirs && t && sigma && rgb && tape,
                "mlp_forward_tape_span: bad arguments");
  return mlp_forward(mlp, engine, cap, 1, origins, dirs, t, noise, sigma, rgb, tape, tape_bytes, workspace, workspace_bytes,
                     (cudaStream_t)stream, end, begin, C);
}

extern "C" int sparf_mlp_backward_tape_rows(const SparfMLP* mlp, int32_t engine, int32_t R, int32_t S, const int64_t* rows,
                                            const float* origins, const float* dirs, const float* t, const float* sigma,
                                            const float* rgb, const float* d_sigma, const float* d_rgb,
                                            const SparfMLPGrad* grad, float* d_origins, float* d_dirs, void* tape,
                                            size_t tape_bytes, void* workspace, size_t workspace_bytes,
                                            sparf_stream_t stream) {
  SPARF_REQUIRE(mlp && R > 0 && S > 0 && rows && origins && dirs && t && sigma && rgb && d_sigma && d_rgb && grad && tape,
                "mlp_backward_tape_rows: bad arguments");
  return mlp_backward(mlp, engine, R, S, origins, dirs, t, nullptr, rgb, tape, tape_bytes, d_sigma, d_rgb, grad, d_origins,
                      d_dirs, workspace, workspace_bytes, (cudaStream_t)stream, rows);
}

extern "C" size_t sparf_density_workspace_bytes(const SparfMLP* mlp, int64_t M, int32_t backward, int32_t engine) {
  if (!mlp || M <= 0) return 0;
  const int e = resolve_engine(engine);
  if (e < 0 || backward < 0 || backward > 2) return 0;
  const Pass pass = backward == 0 ? Pass::kForward : backward == 1 ? Pass::kRecomputeBackward : Pass::kGradient;
  return workspace_need(mlp_dims(mlp), is_tc(e), M, 1, pass, false);
}

extern "C" int sparf_density_forward(const SparfMLP* mlp, int32_t engine, int64_t M, const float* points, float* raw,
                                     float* feat, void* workspace, size_t workspace_bytes, sparf_stream_t stream) {
  SPARF_REQUIRE(mlp && M >= 0, "density_forward: bad arguments");
  if (M == 0) return SPARF_OK;
  SPARF_REQUIRE(points && raw, "density_forward: NULL tensor");
  Call c;
  SPARF_TRY(begin_call("density_forward", mlp, engine, M, 1, Pass::kForward, false, nullptr, 0, workspace, workspace_bytes, &c));
  const cudaStream_t st = (cudaStream_t)stream;
  const MlpDims& d = c.d;
  Tape v = c.w.act;
  for (long long p0 = 0; p0 < M; p0 += c.nrc) {
    const int n = (int)std::min<long long>(c.nrc, M - p0);
    v.H[d.nt - 1] = feat ? feat + (size_t)p0 * d.W : nullptr;     // the features go straight to the caller, or nowhere
    SPARF_TRY(chunk_encode_xyz(mlp, c, n, 1, points + (size_t)p0 * 3, nullptr, nullptr, v.enc, st));
    SPARF_TRY(chunk_trunk(mlp, c, n, v.enc, v.H, nullptr, nullptr, raw + p0, nullptr, false, st));
  }
  return SPARF_OK;
}

// recomputes the forward per chunk, then the last layer's gradient from the caller's (tensor cores: tc_feat_backward,
// straight into image pair 0; SIMT: the masked d_feat in G0) and the trunk backward with d_raw as the density row's
extern "C" int sparf_density_backward(const SparfMLP* mlp, int32_t engine, int64_t M, const float* points, const float* d_raw,
                                      const float* d_feat, const SparfMLPGrad* grad, float* d_points, void* workspace,
                                      size_t workspace_bytes, sparf_stream_t stream) {
  SPARF_REQUIRE(mlp && M >= 0, "density_backward: bad arguments");
  if (M == 0) return SPARF_OK;
  SPARF_REQUIRE(points && grad, "density_backward: NULL tensor");
  Call c;
  SPARF_TRY(begin_call("density_backward", mlp, engine, M, 1, Pass::kRecomputeBackward, false, nullptr, 0, workspace,
                       workspace_bytes, &c));
  const cudaStream_t st = (cudaStream_t)stream;
  const MlpDims& d = c.d;
  float* db = grad->trunk_b[d.nt - 1];
  Tape v = c.w.act;
  if (!d_feat) v.H[d.nt - 1] = nullptr;   // the features are needed only as the mask of d_feat
  for (long long p0 = 0; p0 < M; p0 += c.nrc) {
    const int n = (int)std::min<long long>(c.nrc, M - p0);
    const float* dr = d_raw ? d_raw + p0 : nullptr;
    const float* df = d_feat ? d_feat + (size_t)p0 * d.W : nullptr;
    SPARF_TRY(chunk_encode_xyz(mlp, c, n, 1, points + (size_t)p0 * 3, nullptr, nullptr, v.enc, st));
    SPARF_TRY(chunk_trunk(mlp, c, n, v.enc, v.H, v.bits, nullptr, nullptr, nullptr, false, st));
    if (c.tc) {
      SPARF_TRY(tc_feat_backward(c.ep.dgrad, c.ep.wgrad, n, d.W, dr, df, v.H[d.nt - 1], c.w.Grow[0], grad_tr(c.w, 0, n), db,
                                 db + 1, st));
    } else if (df) {
      relu_mask_kernel<<<ceil_div((long long)n * d.W, 256), 256, 0, st>>>((long long)n * d.W, v.H[d.nt - 1], df, c.w.G0);
      SPARF_CHECK_LAUNCH("relu_mask_kernel");
    } else {
      SPARF_CHECK_CUDA(cudaMemsetAsync(c.w.G0, 0, (size_t)n * d.W * sizeof(float), st));
    }
    SPARF_TRY(c.tc ? trunk_backward_tc(mlp, c, n, v.enc, v.H, v.bits, dr, grad, d_points != nullptr, st)
                   : trunk_backward_simt(mlp, c, n, v.enc, v.H, dr, grad, d_points != nullptr, st));
    if (d_points) {
      posenc_bwd_kernel<<<ceil_div(n, 4), 128, 0, st>>>(n, 1, mlp->L_xyz, d.E3p, v.enc, c.w.Genc, nullptr,
                                                       d_points + (size_t)p0 * 3, nullptr, c.rc);
      SPARF_CHECK_LAUNCH("posenc_bwd_kernel");
    }
  }
  return SPARF_OK;
}

// sparf_density_backward's input-gradient path with d_raw = 1 and d_feat = NULL (G_{nt-1} = 0), without the weight
// gradients; grad_points is written
extern "C" int sparf_density_gradient(const SparfMLP* mlp, int32_t engine, int64_t M, const float* points, float* grad_points,
                                      void* workspace, size_t workspace_bytes, sparf_stream_t stream) {
  SPARF_REQUIRE(mlp && M >= 0, "density_gradient: bad arguments");
  if (M == 0) return SPARF_OK;
  SPARF_REQUIRE(points && grad_points, "density_gradient: NULL tensor");
  Call c;
  SPARF_TRY(begin_call("density_gradient", mlp, engine, M, 1, Pass::kGradient, false, nullptr, 0, workspace, workspace_bytes,
                       &c));
  const cudaStream_t st = (cudaStream_t)stream;
  const MlpDims& d = c.d;
  const Tape& v = c.w.act;
  fill_kernel<<<ceil_div(c.nrc, 256), 256, 0, st>>>(c.nrc, 1.f, c.w.ones);
  SPARF_CHECK_LAUNCH("fill_kernel");
  for (long long p0 = 0; p0 < M; p0 += c.nrc) {
    const int n = (int)std::min<long long>(c.nrc, M - p0);
    float* gp = grad_points + (size_t)p0 * 3;
    SPARF_CHECK_CUDA(cudaMemsetAsync(gp, 0, (size_t)n * 3 * sizeof(float), st));   // posenc_bwd_kernel adds
    SPARF_TRY(chunk_encode_xyz(mlp, c, n, 1, points + (size_t)p0 * 3, nullptr, nullptr, v.enc, st));
    SPARF_TRY(chunk_trunk(mlp, c, n, v.enc, v.H, v.bits, nullptr, nullptr, nullptr, false, st));
    // the last layer's feature gradient is 0: the images tc_feat_backward writes for d_feat = NULL, or G0
    if (c.tc)
      SPARF_CHECK_CUDA(cudaMemsetAsync(c.w.Grow[0].p, 0, tc_image_elems(n, d.W) * sizeof(uint16_t), st));
    else
      SPARF_CHECK_CUDA(cudaMemsetAsync(c.w.G0, 0, (size_t)n * d.W * sizeof(float), st));
    SPARF_TRY(c.tc ? trunk_backward_tc(mlp, c, n, v.enc, v.H, v.bits, c.w.ones, nullptr, true, st)
                   : trunk_backward_simt(mlp, c, n, v.enc, v.H, c.w.ones, nullptr, true, st));
    posenc_bwd_kernel<<<ceil_div(n, 4), 128, 0, st>>>(n, 1, mlp->L_xyz, d.E3p, v.enc, c.w.Genc, nullptr, gp, nullptr, c.rc);
    SPARF_CHECK_LAUNCH("posenc_bwd_kernel");
  }
  return SPARF_OK;
}

extern "C" int sparf_tc_selftest_head(const float* d_rgb, const float* rgb, const float* d_sigma, const float* raw,
                                      const float* hid, const float* W9, int32_t M, int32_t HW, int32_t row_passes,
                                      int32_t tr_passes, uint16_t* img, float* graw, sparf_stream_t stream) {
  SPARF_REQUIRE(M >= 1 && M <= (1 << 20) && HW >= 8 && HW <= 512 && HW % 8 == 0, "tc_selftest_head: M=%d HW=%d", M, HW);
  cudaStream_t st = (cudaStream_t)stream;
  float* scratch = nullptr;
  SPARF_CHECK_CUDA(cudaMallocAsync(reinterpret_cast<void**>(&scratch), ((size_t)M * (HW + 4) + 4 * HW + 4) * sizeof(float), st));
  const int rc = selftest_head(d_rgb, rgb, d_sigma, raw, hid, W9, M, HW, TcPrec{false, row_passes}, TcPrec{false, tr_passes},
                               img, graw, scratch, st);
  cudaFreeAsync(scratch, st);
  return rc;
}

extern "C" int sparf_tc_selftest_featgrad(const float* d_raw, const float* d_feat, const float* feat, int32_t M, int32_t W,
                                          int32_t row_passes, int32_t tr_passes, uint16_t* img, float* sums,
                                          sparf_stream_t stream) {
  SPARF_REQUIRE(M >= 1 && M <= (1 << 20) && W >= 8 && W <= 512 && W % 8 == 0, "tc_selftest_featgrad: M=%d W=%d", M, W);
  SPARF_REQUIRE(d_raw && d_feat && feat && img && sums, "tc_selftest_featgrad: NULL tensor");
  cudaStream_t st = (cudaStream_t)stream;
  float* scratch = nullptr;
  SPARF_CHECK_CUDA(cudaMallocAsync(reinterpret_cast<void**>(&scratch), (size_t)M * W * sizeof(float), st));
  const int rc = selftest_featgrad(d_raw, d_feat, feat, M, W, TcPrec{false, row_passes}, TcPrec{false, tr_passes}, img, sums,
                                   scratch, st);
  cudaFreeAsync(scratch, st);
  return rc;
}
