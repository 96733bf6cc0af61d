// Hopper (sm_90a) tensor-core GEMMs of the layer-by-layer MLP engine: the same three contractions as the CUDA-core
// FFMA kernels of mlp.cu (NT forward, NN input gradient, TN weight gradient, same epilogues), on wgmma with 16-bit
// operands and fp32 accumulation.  passes = 3 splits both fp32 operands into (hi, lo) 16-bit halves and accumulates
// x_lo*w_hi + x_hi*w_lo (in a second accumulator) + x_hi*w_hi (fp32-level products); passes = 1 multiplies the hi halves only.
//
// The activation / gradient operand (A) is given as an operand image: either the image a GEMM epilogue wrote of its
// output, or one packed from fp32 (tc_pack_rows / tc_pack_cols).  The B operand (a weight) is packed by each call; the
// weight gradient's activation operand is read as fp32 and split inside the GEMM.
#pragma once
#include "common.cuh"

namespace sparf {

struct TcPrec {
  bool f16;     // fp16 halves (forward: 11-bit mantissas) or bf16 halves (gradients: fp32 exponent range)
  int passes;   // 3 or 1; 0 = CUDA-core FFMA kernels instead of tensor cores
  // caller-owned buffer of pack_elems 16-bit elements for the packed B operand (tensor cores only); pack_a, as large,
  // is the self-tests' scratch image for A operands
  uint16_t* pack_a = nullptr;
  uint16_t* pack_b = nullptr;
  size_t pack_elems = 0;
  int max_ctas = 0;   // > 0: at most this many CTAs per GEMM (self-tests of the persistent loop); else one per SM
  // rows.rows != NULL: the row count M of a call (the rows of A and of an NT / NN output, the contraction of a TN) is a
  // capacity, of which the kernels process min(M, max(0, *rows.rows - rows.m0)) rows, read on the device.  The TN
  // GEMM's k-range split is then computed in the kernel from that count, as the host computes it from M.
  RowCount rows{nullptr, 0};
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
// 16-bit elements of one B operand image buffer for GEMMs whose B operands have at most max(rows, cols) rows and ksteps
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
// The fused trunk forward (trunk_chain_kernel): layers l = 0 ... nt-1 of width W, H[l] = relu(in_l W_l^T + bias[l]) with
// in_0 = enc, in_l = H[l-1], [H[l-1] | enc] at l == skip, in one launch that keeps a 128-row tile's activations in shared
// memory from layer to layer.  Every H[l], and the last layer's row image, is bit-identical to what the same layers give
// through tc_gemm_nt chained by row images.
// Whether the kernel is built for a trunk of this shape (width 256, an encoding of at most 64 padded columns, at least 3 layers):
bool tc_chain_supported(int W, int E3p, int nt, int skip);
// k-steps of layer l's weight image
int tc_chain_ksteps(int l, int skip, int E3p);
// img = the fused forward's weight image of W (N = 256 rows): the values tc_gemm_nt packs, ks1 k-steps of W[n][k], k < K1v,
// then ks2 of W[n][wcol2 + k], k < K2v, in the chains' layout: per quarter of 64 rows its k-steps one after another
int tc_pack_nt(TcPrec p, int N, int ks1, int K1v, int ks2, int K2v, const float* W, int ldw, int wcol2, TcImage img,
               cudaStream_t st);
// wimg[l]: layer l's weight image (tc_pack_nt, tc_chain_ksteps(l) k-steps), all alive at once.  H[l] == NULL: that
// layer's fp32 output is not written; H[nt-1] == NULL ends the chain after layer nt-2.  bits (may be NULL; else bits[l]
// may be NULL): the ReLU mask H[l] > 0 of layer l as tc_gemm_tn writes it ([M x 8] words), for tc_dgrad_chain.  last: the
// last layer's row image (row_passes = p.passes, or 0: none).  p.rows as for the GEMMs.
int tc_trunk_chain(TcPrec p, int M, int W, int nt, int skip, TcImage enc, const TcImage* wimg, const float* const* bias,
                   float* const* H, uint32_t* const* bits, const TcOut& last, cudaStream_t st);
// img = the fused input gradients' weight image of W (Kout = 256 rows k, contraction over N): the values tc_gemm_nn packs,
// W[n][wcol + k], k < Kv, in the chains' layout (as tc_pack_nt's)
int tc_pack_nn(TcPrec p, int Kout, int N, int Kv, const float* W, int ldw, int wcol, TcImage img, cudaStream_t st);
// The trunk backward's input gradients in one launch (dgrad_chain_kernel), width W = 256, for layers l = top ... 1:
//   G[l-1] = (bit k of bits[l][m]) * sum_n G[l][m][n] W_l[n][k],  db[l][k] += sum_m G[l-1][m][k]
// from G[top] as its row image `in` (dg passes) and wimg[l] (tc_pack_nn of W_l's first 256 columns, dg passes), keeping a
// 128-row tile's gradient in shared memory from layer to layer.  G[l-1] leaves as its transposed image tr[l] (wg passes)
// and, where row[l].p is not NULL, its row image (dg passes).  Values and images are bit-identical to tc_gemm_nn's with
// the same bit masks (bf16 halves); the column sums add 64-row blocks.  dg.rows as for the GEMMs.
int tc_dgrad_chain(TcPrec dg, TcPrec wg, int M, int W, int top, TcImage in, const TcImage* wimg, const uint32_t* const* bits,
                   float* const* db, const TcImage* tr, const TcImage* row, cudaStream_t st);
// D[m][k] = mask(m,k) * ( sum_n G[m][n] W[n][wcol+k] + r1_vec[m]*r1_row[k] )   (= or +=), G [M x N] as its row image.
// mask(m,k) = mask_src[m][k] > 0, or bit k & 31 of mask_bits[m][k >> 5] (ceil(Kout / 32) words per row, as tc_gemm_tn
// writes them; only with D NULL), or 1 when both are NULL.  D may be NULL when out writes images; db (may be NULL) +=
// the column sums of D; r1_wgrad (may be NULL; needs mask_src and r1_vec) += sum_m r1_vec[m] mask_src[m][k], the weight
// gradient of the rank-1 row when mask_src is the layer input.
int tc_gemm_nn(TcPrec p, int M, int N, int Kout, int Kv, TcImage g, const float* W, int ldw, int wcol, const float* mask_src,
               int ldmask, const uint32_t* mask_bits, const float* r1_vec, const float* r1_row, float* D, int ldd,
               int accumulate, const TcOut& out, float* db, float* r1_wgrad, cudaStream_t st);
// dW[n][wcol+k] += sum_m G[m][n] X[m/div][k]   (atomic over k-ranges of the rows, about one per SM per 32 768 rows), G [M x N]
// as its transposed image.  bits (may be NULL) [M x ceil(K / 32)]: bit k & 31 of word [m][k >> 5] = X[m/div][k] > 0, the
// ReLU mask of the input gradient of the layer whose input X is, written while X is split.  X is read as fp32 inside the
// GEMM when X is 16-byte aligned and ldx and K are multiples of 4 (bf16 only); otherwise it is packed into p.pack_b
// first ([ceil(K / 128) * 128 x ceil(M / 32) * 32] image).
int tc_gemm_tn(TcPrec p, int M, int N, int K, int Kv, TcImage gt, const float* X, int ldx, int div, float* dW, int ldw,
               int wcol, uint32_t* bits, cudaStream_t st);

// The colour-head backward in one kernel (bf16 images): from the upstream d_rgb [M,3], d_sigma [M], the forward's rgb
// [M,3], raw [M] (softplus argument) and hid [M,HW], and the head's output layer W9 [3,HW]:
//   graw[m] = d_sigma[m] softplus'(raw[m]);  gpre[m][j] = d_rgb[m][j] rgb (1 - rgb);  Ghid = (hid > 0) * gpre W9,
// Ghid written only as its row image (dg passes) and its transposed image (wg passes), bit-identical to tc_pack_rows /
// tc_pack_cols of the fp32 Ghid; and dW9 [3,HW] += gpre^T hid, db9[3] += sum gpre, db_hid[HW] += the column sums of
// Ghid, db_raw[0] += sum graw.
int tc_head_backward(TcPrec dg, TcPrec wg, int M, int HW, const float* d_rgb, const float* rgb, const float* d_sigma,
                     const float* raw, const float* hid, const float* W9, float* graw, TcImage row, TcImage tr, float* dW9,
                     float* db9, float* db_hid, float* db_raw, cudaStream_t st);

// The last trunk layer's gradient from the caller's d_raw [M] and d_feat [M,W] (each may be NULL: a zero gradient) and
// the recomputed features feat [M,W] (16-byte aligned; may be NULL when d_feat is):  G = (feat > 0) * d_feat, written only
// as its row image (dg passes) and its transposed image (wg passes), bit-identical to tc_pack_rows / tc_pack_cols of the
// fp32 G; and db_feat[W] += the column sums of G, db_raw[0] += sum d_raw.
int tc_feat_backward(TcPrec dg, TcPrec wg, int M, int W, const float* d_raw, const float* d_feat, const float* feat,
                     TcImage row, TcImage tr, float* db_raw, float* db_feat, cudaStream_t st);

}  // namespace sparf
