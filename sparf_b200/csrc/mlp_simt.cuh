// Internal interface of the layer-by-layer MLP engines (mlp_simt.cu).
#pragma once
#include "common.cuh"
#include "gemm_wgmma.cuh"

namespace sparf {

struct SimtDims {
  int E3, E3p, Ev, Evp, W, HW, nt, skip;
};

// GEMM precision per role: forward, input gradient (dgrad), weight gradient (wgrad)
struct EnginePrec {
  TcPrec fwd, dgrad, wgrad;
};
EnginePrec engine_prec(int engine);

SimtDims simt_dims(const SparfMLP* mlp);
// the trunk's fields (density calls); simt_validate: these and the colour head's (MLP calls)
int simt_validate_trunk(const SparfMLP* mlp);
int simt_validate(const SparfMLP* mlp);
// mode 0: forward, 1: backward (recompute), 2: backward from a tape, 3: taped forward
size_t simt_workspace_bytes(const SparfMLP* mlp, int R, int S, int mode, int engine);
int simt_mlp_forward(const SparfMLP* mlp, int engine, int R, int S, const float* origins, const float* dirs, const float* t,
                     const float* noise, float* sigma, float* rgb, void* workspace, size_t workspace_bytes,
                     cudaStream_t st);
size_t simt_tape_bytes(const SparfMLP* mlp, int R, int S);
int simt_mlp_forward_tape(const SparfMLP* mlp, int engine, int R, int S, const float* origins, const float* dirs,
                          const float* t, const float* noise, float* sigma, float* rgb, void* tape, size_t tape_bytes,
                          void* workspace, size_t workspace_bytes, cudaStream_t st);
int simt_mlp_backward_tape(const SparfMLP* mlp, int engine, int R, int S, const float* origins, const float* dirs,
                           const float* t, const float* rgb, const float* d_sigma, const float* d_rgb, const SparfMLPGrad* grad,
                           float* d_origins, float* d_dirs, void* tape, size_t tape_bytes, void* workspace,
                           size_t workspace_bytes, cudaStream_t st);
int simt_mlp_backward(const SparfMLP* mlp, int engine, int R, int S, const float* origins, const float* dirs, const float* t,
                      const float* noise, const float* d_sigma, const float* d_rgb, const SparfMLPGrad* grad,
                      float* d_origins, float* d_dirs, void* workspace, size_t workspace_bytes, cudaStream_t st);
// trunk-only density queries at M points: mode 0 forward, 1 backward (recomputes the forward)
size_t simt_density_workspace_bytes(const SparfMLP* mlp, long long M, int mode, int engine);
int simt_density_forward(const SparfMLP* mlp, int engine, long long M, const float* points, float* raw, float* feat,
                         void* workspace, size_t workspace_bytes, cudaStream_t st);
int simt_density_backward(const SparfMLP* mlp, int engine, long long M, const float* points, const float* d_raw,
                          const float* d_feat, const SparfMLPGrad* grad, float* d_points, void* workspace,
                          size_t workspace_bytes, cudaStream_t st);

}  // namespace sparf
