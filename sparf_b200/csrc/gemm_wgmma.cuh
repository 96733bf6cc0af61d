// Hopper (sm_90a) tensor-core GEMMs of the layer-by-layer MLP engine: the same three contractions as the CUDA-core
// FFMA kernels of mlp_simt.cu (NT forward, NN input gradient, TN weight gradient, same arguments and epilogues), on
// wgmma with 16-bit operands and fp32 accumulation.  passes = 3 splits both fp32 operands into (hi, lo) 16-bit halves and
// accumulates x_lo*w_hi + x_hi*w_lo (in a second accumulator) + x_hi*w_hi (fp32-level products); passes = 1 multiplies the hi halves only.
#pragma once
#include "common.cuh"

namespace sparf {

struct TcPrec {
  bool f16;     // fp16 halves (forward: 11-bit mantissas) or bf16 halves (gradients: fp32 exponent range)
  int passes;   // 3 or 1; 0 = CUDA-core FFMA kernels instead of tensor cores
  // two caller-owned buffers of pack_elems 16-bit elements each for the pre-split operand images (tensor cores only)
  uint16_t* pack_a = nullptr;
  uint16_t* pack_b = nullptr;
  size_t pack_elems = 0;
};

// 16-bit elements of one operand image buffer for GEMMs whose operands have at most max(rows, cols) rows and ksteps
// 32-wide k-steps
size_t tc_pack_elems(int rows, int ksteps, int cols);

// Y[m][n] = act( sum_k X1[m][k] W[n][k] + sum_k X2[m/div2][k] W[n][wcol2+k] + bias[n] ),  act: 0 none, 1 ReLU
int tc_gemm_nt(TcPrec p, int act, int M, int N, const float* X1, int ld1, int K1, int K1v, const float* X2, int ld2, int K2,
               int K2v, int div2, const float* W, int ldw, int wcol2, const float* bias, float* Y, int ldy, cudaStream_t st);
// D[m][k] = mask(m,k) * ( sum_n G[m][n] W[n][wcol+k] + r1_vec[m]*r1_row[k] )   (= or +=)
int tc_gemm_nn(TcPrec p, int M, int N, int Kout, int Kv, const float* G, int ldg, const float* W, int ldw, int wcol,
               const float* mask_src, int ldmask, const float* r1_vec, const float* r1_row, float* D, int ldd, int accumulate,
               cudaStream_t st);
// dW[n][wcol+k] += sum_m G[m][n] X[m/div][k]   (atomic over slabs of rows_per_slab rows)
int tc_gemm_tn(TcPrec p, int M, int N, int K, int Kv, int rows_per_slab, const float* G, int ldg, const float* X, int ldx,
               int div, float* dW, int ldw, int wcol, cudaStream_t st);

}  // namespace sparf
