// Hopper (sm_90a) tensor-core GEMMs of the layer-by-layer MLP engine: the same three contractions as the CUDA-core
// FFMA kernels of mlp_simt.cu (NT forward, NN input gradient, TN weight gradient, same epilogues), on wgmma with 16-bit
// operands and fp32 accumulation.  passes = 3 splits both fp32 operands into (hi, lo) 16-bit halves and accumulates
// x_lo*w_hi + x_hi*w_lo (in a second accumulator) + x_hi*w_hi (fp32-level products); passes = 1 multiplies the hi halves only.
//
// The activation / gradient operand (A) is given as an operand image: either the image a GEMM epilogue wrote of its
// output, or one packed from fp32 (tc_pack_rows / tc_pack_cols).  The weight operand (B) is packed by each call.
#pragma once
#include "common.cuh"

namespace sparf {

struct TcPrec {
  bool f16;     // fp16 halves (forward: 11-bit mantissas) or bf16 halves (gradients: fp32 exponent range)
  int passes;   // 3 or 1; 0 = CUDA-core FFMA kernels instead of tensor cores
  // caller-owned buffer of pack_elems 16-bit elements for the packed B operand (tensor cores only); pack_a, as large,
  // is the caller's scratch image for A operands that no epilogue writes
  uint16_t* pack_a = nullptr;
  uint16_t* pack_b = nullptr;
  size_t pack_elems = 0;
  int max_ctas = 0;   // > 0: at most this many CTAs per GEMM (self-tests of the persistent loop); else one per SM
};

// An operand image of a [rows x K] matrix: split 16-bit halves in [128 rows x 32 K] tiles of wgmma's shared-memory
// layout, tile (row tile rt, k-step kt), half h at ((rt * ks + kt) * 2 + h) * 4096 elements, zero past rows and K.
struct TcImage {
  uint16_t* p = nullptr;
  int ks = 0;   // k-steps of 32 per row tile = ceil(K / 32)
};

// images a GEMM epilogue writes of its output D [M x N], in the GEMM's 16-bit type: row (rows m, K = n; its passes must
// be the GEMM's) and transposed (rows n, K = m); passes 3 = hi and lo halves, 1 = hi only, 0 = not written
struct TcOut {
  TcImage row, tr;
  int row_passes = 0, tr_passes = 0;
};

// 16-bit elements of the image of a [rows x cols] matrix
size_t tc_image_elems(int rows, int cols);
// 16-bit elements of one B operand image buffer for GEMMs whose operands have at most max(rows, cols) rows and ksteps
// 32-wide k-steps
size_t tc_pack_elems(int rows, int ksteps, int cols);

// img = the [M x K] matrix X[m / div][k]
int tc_pack_rows(TcPrec p, int M, int K, const float* X, int ldx, int div, TcImage img, cudaStream_t st);
// img = the [N x M] matrix X[m][n] (the transpose of X [M x N])
int tc_pack_cols(TcPrec p, int M, int N, const float* X, int ldx, TcImage img, cudaStream_t st);

// Y[m][n] = act( sum_k A1[m][k] W[n][k] + sum_k A2[m][k] W[n][wcol2+k] + bias[n] ),  act: 0 none, 1 ReLU.  A1 has K1v
// valid columns, A2 (a2.p may be NULL) K2v.  out: images of Y.
int tc_gemm_nt(TcPrec p, int act, int M, int N, TcImage a1, int K1v, TcImage a2, int K2v, const float* W, int ldw, int wcol2,
               const float* bias, float* Y, int ldy, const TcOut& out, cudaStream_t st);
// D[m][k] = mask(m,k) * ( sum_n G[m][n] W[n][wcol+k] + r1_vec[m]*r1_row[k] )   (= or +=), G [M x N] as its row image.
// D may be NULL when out writes images; db (may be NULL) += the column sums of D.
int tc_gemm_nn(TcPrec p, int M, int N, int Kout, int Kv, TcImage g, const float* W, int ldw, int wcol, const float* mask_src,
               int ldmask, const float* r1_vec, const float* r1_row, float* D, int ldd, int accumulate, const TcOut& out,
               float* db, cudaStream_t st);
// dW[n][wcol+k] += sum_m G[m][n] X[m/div][k]   (atomic over k-ranges of the rows, about one CTA per SM in all), G [M x N]
// as its transposed image
int tc_gemm_tn(TcPrec p, int M, int N, int K, int Kv, TcImage gt, const float* X, int ldx, int div, float* dW, int ldw,
               int wcol, cudaStream_t st);

}  // namespace sparf
