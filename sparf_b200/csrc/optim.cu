// Fused parameter update of one optimiser group over flat fp32 buffers (SURVEY.md §8f.1): what the reference does
// with check_invalid_gradients + clip_grad_norm_ + torch.optim.Adam.step + ExponentialLR.step (+ linear LR warm-up
// for the poses) -- source/training/engine/iter_based_trainer.py:128-147, nerf_trainer.py:181-204,
// joint_pose_nerf_trainer.py:513-549 -- as two kernels with the step counter in device memory, so the update can sit
// in the same CUDA graph as the render step.
#include "common.cuh"

namespace sparf {
namespace {

// scratch[0] = sum g^2 (double), scratch[1] = non-finite flag (as double), both zeroed by the second kernel
__global__ void __launch_bounds__(256) grad_stats_kernel(long long n, const float* __restrict__ g, double* __restrict__ scratch) {
  double acc = 0.0;
  int bad = 0;
  for (long long i = blockIdx.x * 256LL + threadIdx.x; i < n; i += (long long)gridDim.x * 256) {
    const float v = g[i];
    if (!isfinite(v)) bad = 1;
    acc += (double)v * (double)v;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    acc += __shfl_xor_sync(0xffffffffu, acc, o);
    bad |= __shfl_xor_sync(0xffffffffu, bad, o);
  }
  __shared__ double s_acc[8];
  __shared__ int s_bad[8];
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  if (l == 0) { s_acc[w] = acc; s_bad[w] = bad; }
  __syncthreads();
  if (threadIdx.x == 0) {
    double a = 0.0;
    int b = 0;
    for (int i = 0; i < 8; ++i) { a += s_acc[i]; b |= s_bad[i]; }
    atomicAdd(&scratch[0], a);
    if (b) atomicAdd(&scratch[1], 1.0);
  }
}

struct AdamArgs {
  long long n;
  float* param;
  float* grad;
  float* exp_avg;
  float* exp_avg_sq;
  long long* step;        // device: step[0] = Adam updates taken (bias correction), step[1] = iterations seen (LR schedule)
  double* scratch;
  double lr0, gamma, warmup, beta1, beta2, eps, max_norm;
};

// torch.optim.Adam (single-tensor path, amsgrad=False, weight_decay=0, maximize=False):
//   exp_avg.lerp_(g, 1 - b1); exp_avg_sq.mul_(b2).addcmul_(g, g, value=1 - b2)
//   denom = (exp_avg_sq.sqrt() / sqrt(1 - b2^t)).add_(eps); param.addcdiv_(exp_avg, denom, value=-lr / (1 - b1^t))
// Scalars are formed in double and rounded to fp32 where torch hands them to an fp32 kernel.
__global__ void __launch_bounds__(256) adam_kernel(AdamArgs a) {
  const double sumsq = a.scratch[0];
  const bool bad = a.scratch[1] != 0.0;
  const long long t = a.step[0] + 1;    // this update's number (torch: state["step"])
  const long long k = a.step[1] + 1;    // this iteration's number (the schedulers advance even when an update is skipped)
  // clip_grad_norm_: coef = max_norm / (norm + 1e-6), clamped to 1
  float coef = 1.f;
  if (a.max_norm > 0.0) {
    const float norm = sqrtf((float)sumsq);
    coef = fminf((float)a.max_norm / (norm + 1e-6f), 1.f);
  }
  // ExponentialLR: lr of iteration k is lr0 * gamma^(k-1); warm-up multiplies by min(1, k / warmup)
  double lr = a.lr0 * pow(a.gamma, (double)(k - 1));
  if (a.warmup > 0.0) lr *= fmin(1.0, (double)k / a.warmup);
  const double bc1 = 1.0 - pow(a.beta1, (double)t), bc2 = 1.0 - pow(a.beta2, (double)t);
  const float step_size = (float)(lr / bc1);
  const float bc2_sqrt = (float)sqrt(bc2);
  const float w1 = (float)(1.0 - a.beta1), b2 = (float)a.beta2, w2 = (float)(1.0 - a.beta2), eps = (float)a.eps;
  if (!bad) {   // a non-finite gradient skips the update (iter_based_trainer.py:129, joint_pose_nerf_trainer.py:541)
    for (long long i = blockIdx.x * 256LL + threadIdx.x; i < a.n; i += (long long)gridDim.x * 256) {
      float g = a.grad[i];
      if (coef != 1.f) { g = __fmul_rn(g, coef); a.grad[i] = g; }      // clip_grad_norm_ scales .grad in place
      float m = a.exp_avg[i], v = a.exp_avg_sq[i];
      m = w1 < 0.5f ? __fadd_rn(m, __fmul_rn(w1, __fsub_rn(g, m)))                       // Tensor.lerp_, both branches
                    : __fsub_rn(g, __fmul_rn(__fsub_rn(g, m), __fsub_rn(1.f, w1)));
      v = __fadd_rn(__fmul_rn(v, b2), __fmul_rn(w2, __fmul_rn(g, g))); // mul_ then addcmul_
      const float denom = __fadd_rn(__fdiv_rn(__fsqrt_rn(v), bc2_sqrt), eps);
      a.param[i] = __fadd_rn(a.param[i], __fmul_rn(-step_size, __fdiv_rn(m, denom)));
      a.exp_avg[i] = m;
      a.exp_avg_sq[i] = v;
    }
  }
  // last block out resets the scratch and advances the counter for the next update
  __shared__ bool last;
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned int done = atomicAdd(reinterpret_cast<unsigned int*>(&a.scratch[2]), 1u);
    last = done == gridDim.x - 1;
  }
  __syncthreads();
  if (last && threadIdx.x == 0) {
    a.scratch[0] = 0.0;
    a.scratch[1] = 0.0;
    reinterpret_cast<unsigned int*>(&a.scratch[2])[0] = 0u;
    if (!bad) a.step[0] = t;
    a.step[1] = k;
  }
}

}  // namespace
}  // namespace sparf

using namespace sparf;

extern "C" int sparf_adam_step(int64_t n, float* param, float* grad, float* exp_avg, float* exp_avg_sq, int64_t* step,
                               double* scratch, double lr0, double gamma, double warmup_steps, double beta1,
                               double beta2, double eps, double max_norm, sparf_stream_t stream) {
  SPARF_REQUIRE(n >= 0 && param && grad && exp_avg && exp_avg_sq && step && scratch, "adam_step: null argument");
  SPARF_REQUIRE(lr0 >= 0 && gamma > 0 && beta1 >= 0 && beta1 < 1 && beta2 >= 0 && beta2 < 1 && eps >= 0,
                "adam_step: bad hyper-parameters");
  if (n == 0) return SPARF_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const int blocks = (int)std::min<long long>((n + 255) / 256, (long long)num_sms() * 8);
  grad_stats_kernel<<<blocks, 256, 0, st>>>(n, grad, scratch);
  SPARF_CHECK_LAUNCH("grad_stats_kernel");
  AdamArgs a;
  a.n = n; a.param = param; a.grad = grad; a.exp_avg = exp_avg; a.exp_avg_sq = exp_avg_sq;
  a.step = reinterpret_cast<long long*>(step); a.scratch = scratch;
  a.lr0 = lr0; a.gamma = gamma; a.warmup = warmup_steps; a.beta1 = beta1; a.beta2 = beta2; a.eps = eps; a.max_norm = max_norm;
  adam_kernel<<<blocks, 256, 0, st>>>(a);
  SPARF_CHECK_LAUNCH("adam_kernel");
  return SPARF_OK;
}

// ------------------------------------------------------------------------------------------------
// mip-NeRF-360 distortion regulariser (source/training/core/regularization_losses.py:20-48; called with the
// renderer's `t` and `weights`, base_losses.py:166-172).  The reference builds the [S-1, S-1] matrix |u_i - u_j| per
// ray; along a ray the mid-points u are monotone, so the pair sum collapses to prefix sums:
//   sum_ij a_i a_j |u_i - u_j| = 2 sum_i a_i (u_i A_i - M_i),  A_i = sum_{j<i} a_j,  M_i = sum_{j<i} a_j u_j
// with a_i = w_{i+1}, u_i = (t_{i+1} + t_i) / 2, i = 0..S-2; plus sum_i a_i^2 (t_{i+1} - t_i) / 3.
// The terms u_i A_i and M_i cancel when the weight mass sits far from u = 0 compared with its spread (a far scene, or
// fine samples clustered at a surface): in fp32 that costs up to 10-50x the literal form's error
// (tests/test_distortion_fp64.py).  The pair term is invariant under u -> u - c, so every pass after the first works on
// mid-points centred at the ray's weighted mean c = sum a u / sum a (u_0 when sum a = 0), formed as
// ((t_{i+1} - c) + (t_i - c)) / 2 so the shift is exact for t near c.  c is a constant of the formula, not a function
// of the inputs: d_w and d_t are those of the uncentred sums.
// One warp per ray, shuffle scans (like compositing).  loss += scale * mean over rays; d_w, d_t are written.
// ------------------------------------------------------------------------------------------------
namespace sparf {
namespace {

__device__ __forceinline__ float warp_excl_scan(float v, int lane, float& total) {
  float x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    float y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  total = __shfl_sync(0xffffffffu, x, 31);
  float e = __shfl_up_sync(0xffffffffu, x, 1);
  return lane == 0 ? 0.f : e;
}

__global__ void __launch_bounds__(128) distortion_kernel(int R, int S, const float* __restrict__ t, const float* __restrict__ w,
                                                         float scale, float* __restrict__ loss, float* __restrict__ d_w,
                                                         float* __restrict__ d_t) {
  const int lane = threadIdx.x & 31;
  const int r = blockIdx.x * 4 + (threadIdx.x >> 5);
  if (r >= R) return;
  const float* tr = t + (size_t)r * S;
  const float* wr = w + (size_t)r * S;
  const int n = S - 1;
  // orientation: inverse-depth samples decrease along the ray; the pair term only needs monotone mid-points
  const float sgn = tr[S - 1] >= tr[0] ? 1.f : -1.f;
  // pass 0: the centre c (in t, unoriented)
  float A_tot = 0.f, M_tot = 0.f;
  for (int i0 = 0; i0 < n; i0 += 32) {
    const int i = i0 + lane;
    const float a = i < n ? wr[i + 1] : 0.f;
    const float m = i < n ? 0.5f * (tr[i + 1] + tr[i]) : 0.f;
    float sa = a, sm = a * m;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { sa += __shfl_xor_sync(0xffffffffu, sa, o); sm += __shfl_xor_sync(0xffffffffu, sm, o); }
    A_tot += sa; M_tot += sm;
  }
  const float c = A_tot > 0.f ? M_tot / A_tot : 0.5f * (tr[1] + tr[0]);
  // pass 1: totals (for the suffix sums) and the loss
  A_tot = 0.f; M_tot = 0.f;
  for (int i0 = 0; i0 < n; i0 += 32) {
    const int i = i0 + lane;
    const float a = i < n ? wr[i + 1] : 0.f;
    const float u = i < n ? sgn * 0.5f * ((tr[i + 1] - c) + (tr[i] - c)) : 0.f;
    float sa = a, sm = a * u;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { sa += __shfl_xor_sync(0xffffffffu, sa, o); sm += __shfl_xor_sync(0xffffffffu, sm, o); }
    A_tot += sa; M_tot += sm;
  }
  float A_run = 0.f, M_run = 0.f, acc = 0.f;
  const float gs = scale / (float)R;
  for (int i0 = 0; i0 < n; i0 += 32) {
    const int i = i0 + lane;
    const bool ok = i < n;
    const float a = ok ? wr[i + 1] : 0.f;
    const float t0 = ok ? tr[i] : 0.f, t1 = ok ? tr[i + 1] : 0.f;
    const float u = sgn * 0.5f * ((t1 - c) + (t0 - c)), dt = t1 - t0;
    float ta, tm;
    const float A = A_run + warp_excl_scan(a, lane, ta);
    const float M = M_run + warp_excl_scan(a * u, lane, tm);
    A_run += ta; M_run += tm;
    if (ok) {
      const float A_gt = A_tot - A - a, M_gt = M_tot - M - a * u;          // sums over j > i
      acc += 2.f * a * (u * A - M) + a * a * dt * (1.f / 3.f);
      // d/da_i = 2 sum_j a_j |u_i - u_j| + 2 a_i dt_i / 3
      d_w[(size_t)r * S + i + 1] = gs * (2.f * ((u * A - M) + (M_gt - u * A_gt)) + 2.f * a * dt * (1.f / 3.f));
      if (d_t) {
        const float du = gs * sgn * 2.f * a * (A - A_gt);                     // d/du_i (in the original orientation)
        const float dd = gs * a * a * (1.f / 3.f);                            // d/d(dt_i)
        // t_i receives (du_i / 2 - dd_i) from interval i and (du_{i-1} / 2 + dd_{i-1}) from interval i - 1
        atomicAdd(d_t + (size_t)r * S + i, 0.5f * du - dd);
        atomicAdd(d_t + (size_t)r * S + i + 1, 0.5f * du + dd);
      }
    }
  }
  if (lane == 0) d_w[(size_t)r * S] = 0.f;        // w_0 never enters (regularization_losses.py:41)
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if (lane == 0) atomicAdd(loss, gs * acc);
}

}  // namespace
}  // namespace sparf

extern "C" int sparf_distortion_fwd_bwd(int32_t R, int32_t S, const float* t, const float* w, float scale, float* loss,
                                        float* d_w, float* d_t, sparf_stream_t stream) {
  SPARF_REQUIRE(R >= 0 && S >= 2 && t && w && loss && d_w, "distortion: bad arguments R=%d S=%d", R, S);
  if (R == 0) return SPARF_OK;
  cudaStream_t st = (cudaStream_t)stream;
  if (d_t) SPARF_CHECK_CUDA(cudaMemsetAsync(d_t, 0, (size_t)R * S * sizeof(float), st));
  distortion_kernel<<<ceil_div(R, 4), 128, 0, st>>>(R, S, t, w, scale, loss, d_w, d_t);
  SPARF_CHECK_LAUNCH("distortion_kernel");
  return SPARF_OK;
}
