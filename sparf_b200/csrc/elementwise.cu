// Ray generation, depth sampling, hierarchical resampling, alpha compositing and the photometric
// Huber loss: the HBM-light stages around the MLP.  One warp per ray for everything that scans a ray.
#include "common.cuh"

namespace sparf {

// ------------------------------------------------------------------------------------------------
// rays: camera.get_center_and_ray[_at_pixels]  (source/utils/camera.py:347-416)
// ------------------------------------------------------------------------------------------------
struct PixelSrc {
  const int64_t* ray_idx;
  const float* pixels;
  int per_image, W, n;
  __device__ __forceinline__ void get(int b, int i, float& u, float& v) const {
    if (pixels) {
      const float* p = pixels + (per_image ? ((size_t)b * n + i) * 2 : (size_t)i * 2);
      u = p[0];
      v = p[1];
    } else {
      long long idx = ray_idx[per_image ? (size_t)b * n + i : (size_t)i];
      int y = (int)(idx / W), x = (int)(idx - (long long)y * W);
      u = (float)x + 0.5f;  // camera.py:365-366
      v = (float)y + 0.5f;
    }
  }
};

__global__ void raygen_fwd_kernel(int n, const float* __restrict__ pose, const float* __restrict__ kinv,
                                  PixelSrc src, float* __restrict__ origins, float* __restrict__ dirs) {
  int b = blockIdx.y, i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float* P = pose + b * 12;
  const float* K = kinv + b * 9;
  float u, v;
  src.get(b, i, u, v);
  // p = K^-1 [u,v,1]^T  (camera.py:318-319)
  float p[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) p[c] = fmaf(K[c * 3 + 1], v, K[c * 3 + 0] * u) + K[c * 3 + 2];
  // c2w = [R^T | -R^T t]  (camera.py:92-98); centre = tc ; ray = (Rc p + tc) - tc  (camera.py:372-379)
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    float tc = -(P[0 * 4 + c] * P[0 * 4 + 3]) - P[1 * 4 + c] * P[1 * 4 + 3] - P[2 * 4 + c] * P[2 * 4 + 3];
    float w = fmaf(P[2 * 4 + c], p[2], fmaf(P[1 * 4 + c], p[1], P[0 * 4 + c] * p[0])) + tc;
    size_t o = ((size_t)b * n + i) * 3 + c;
    origins[o] = tc;
    dirs[o] = w - tc;
  }
}

// d(pose_w2c)[b] += sum over the image's rays.  o_c = -sum_j R[j][c] t_j ; d_c = sum_j R[j][c] p_j.
__global__ void raygen_bwd_kernel(int n, const float* __restrict__ pose, const float* __restrict__ kinv,
                                  PixelSrc src, const float* __restrict__ g_o, const float* __restrict__ g_d,
                                  float* __restrict__ d_pose, float* __restrict__ d_pixels) {
  int b = blockIdx.y, i = blockIdx.x * blockDim.x + threadIdx.x;
  const float* P = pose + b * 12;
  const float* K = kinv + b * 9;
  float acc[12];
#pragma unroll
  for (int q = 0; q < 12; ++q) acc[q] = 0.f;
  if (i < n) {
    float u, v, p[3];
    src.get(b, i, u, v);
#pragma unroll
    for (int c = 0; c < 3; ++c) p[c] = fmaf(K[c * 3 + 1], v, K[c * 3 + 0] * u) + K[c * 3 + 2];
    size_t o = ((size_t)b * n + i) * 3;
    float go[3] = {0.f, 0.f, 0.f}, gd[3] = {0.f, 0.f, 0.f};
    if (g_o) { go[0] = g_o[o]; go[1] = g_o[o + 1]; go[2] = g_o[o + 2]; }
    if (g_d) { gd[0] = g_d[o]; gd[1] = g_d[o + 1]; gd[2] = g_d[o + 2]; }
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      float gt = 0.f;
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        acc[j * 4 + c] = gd[c] * p[j] - go[c] * P[j * 4 + 3];
        gt -= go[c] * P[j * 4 + c];
      }
      acc[j * 4 + 3] = gt;
    }
    // float pixel locations are differentiable in the reference (camera.py:400-416: ray = R^T K^-1 [u,v,1]): the
    // depth-consistency loss renders at pixels projected from a rendered depth (depth_cons_loss.py:247-283)
    if (d_pixels) {
      float du = 0.f, dv = 0.f;
#pragma unroll
      for (int c = 0; c < 3; ++c) {
#pragma unroll
        for (int j = 0; j < 3; ++j) {
          du = fmaf(gd[c] * P[j * 4 + c], K[j * 3 + 0], du);
          dv = fmaf(gd[c] * P[j * 4 + c], K[j * 3 + 1], dv);
        }
      }
      if (src.per_image) {
        d_pixels[((size_t)b * n + i) * 2] = du;
        d_pixels[((size_t)b * n + i) * 2 + 1] = dv;
      } else {   // one pixel list shared by every image: the gradients of the B images add up
        atomicAdd(d_pixels + (size_t)i * 2, du);
        atomicAdd(d_pixels + (size_t)i * 2 + 1, dv);
      }
    }
  }
  __shared__ float red[12][8];
  int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int q = 0; q < 12; ++q) {
    float v = acc[q];
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) v += __shfl_xor_sync(0xffffffffu, v, s);
    if (lane == 0) red[q][warp] = v;
  }
  __syncthreads();
  if (threadIdx.x < 12) {
    float v = 0.f;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) v += red[threadIdx.x][w];
    atomicAdd(d_pose + b * 12 + threadIdx.x, v);
  }
}

// ------------------------------------------------------------------------------------------------
// depth samples: Graph.sample_depth / sample_depth_diff_max_range_per_ray (renderer.py:383-419, 595-624)
// ------------------------------------------------------------------------------------------------
__global__ void sample_depth_kernel(long long total, int S, float near, float range, int inverse,
                                    const float* __restrict__ rand, const float* __restrict__ far_per_ray,
                                    float* __restrict__ t) {
  long long m = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= total) return;
  int k = (int)(m % S);
  long long r = m / S;
  float u = far_per_ray ? 1.0f : (rand ? rand[m] : 0.5f);
  float rg = far_per_ray ? __fsub_rn(far_per_ray[r], near) : range;
  float v = add_rn(mul_rn(__fdiv_rn(add_rn(u, (float)k), (float)S), rg), near);
  if (inverse) v = __fdiv_rn(1.0f, add_rn(v, 1e-8f));
  t[m] = v;
}

// ------------------------------------------------------------------------------------------------
// hierarchical resampling: Graph.sample_depth_from_pdf + cat + sort (renderer.py:421-456, 334-336)
// one 128-thread block per ray; S + S_fine <= 4096 (the sort buffer and the cdf live in shared memory)
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float linspace_at(float a, float b, float step, int steps, int i) {
  // torch.linspace: symmetric evaluation from both ends
  return (i < steps / 2) ? add_rn(a, mul_rn(step, (float)i)) : __fsub_rn(b, mul_rn(step, (float)(steps - i - 1)));
}

__global__ void __launch_bounds__(128) sample_pdf_merge_kernel(int S, int Sf, float near, float far,
                                                               const float* __restrict__ weights,
                                                               const float* __restrict__ t_coarse,
                                                               const float* __restrict__ u_mid,
                                                               float* __restrict__ t_fine,
                                                               float* __restrict__ t_all, int npow2) {
  extern __shared__ float sm[];
  float* cdf = sm;             // S+1
  float* buf = sm + (S + 1);   // npow2
  __shared__ float s_red[4];
  const int r = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float* w = weights + (size_t)r * S;

  // sum of weights
  float part = 0.f;
  for (int k = tid; k < S; k += 128) part += w[k];
#pragma unroll
  for (int s = 16; s > 0; s >>= 1) part += __shfl_xor_sync(0xffffffffu, part, s);
  if (lane == 0) s_red[warp] = part;
  __syncthreads();
  const float denom = add_rn(s_red[0] + s_red[1] + s_red[2] + s_red[3], 1e-6f);

  // cdf = [0, cumsum(w / denom)]: warp 0 scans 32 at a time with a running carry
  if (warp == 0) {
    float carry = 0.f;
    if (lane == 0) cdf[0] = 0.f;
    for (int k0 = 0; k0 < S; k0 += 32) {
      int k = k0 + lane;
      float v = k < S ? __fdiv_rn(w[k], denom) : 0.f;
#pragma unroll
      for (int s = 1; s < 32; s <<= 1) {
        float o = __shfl_up_sync(0xffffffffu, v, s);
        if (lane >= s) v += o;
      }
      v += carry;
      if (k < S) cdf[k + 1] = v;
      carry = __shfl_sync(0xffffffffu, v, 31);
    }
  }
  __syncthreads();

  const float step = __fdiv_rn(__fsub_rn(far, near), (float)S);  // linspace(near, far, S+1)
  for (int i = tid; i < Sf; i += 128) {
    float u = u_mid[i];
    // searchsorted(cdf, u, right=True): first index with cdf[idx] > u, in [0, S+1]
    int lo = 0, hi = S + 1;
    while (lo < hi) {
      int mid = (lo + hi) >> 1;
      if (cdf[mid] <= u) lo = mid + 1; else hi = mid;
    }
    int il = max(lo - 1, 0), ih = min(lo, S);
    float cl = cdf[il], ch = cdf[ih];
    float bl = linspace_at(near, far, step, S + 1, il), bh = linspace_at(near, far, step, S + 1, ih);
    float frac = __fdiv_rn(__fsub_rn(u, cl), add_rn(__fsub_rn(ch, cl), 1e-8f));
    float tf = add_rn(bl, mul_rn(frac, __fsub_rn(bh, bl)));
    buf[S + i] = tf;
    if (t_fine) t_fine[(size_t)r * Sf + i] = tf;
  }
  for (int k = tid; k < S; k += 128) buf[k] = t_coarse[(size_t)r * S + k];
  for (int k = S + Sf + tid; k < npow2; k += 128) buf[k] = __int_as_float(0x7f800000);
  __syncthreads();
  // bitonic sort (ascending) of npow2 values in shared memory
  for (int size = 2; size <= npow2; size <<= 1) {
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      for (int i = tid; i < npow2 / 2; i += 128) {
        int lo_i = 2 * i - (i & (stride - 1));
        int hi_i = lo_i + stride;
        bool up = ((lo_i & size) == 0);
        float a = buf[lo_i], b = buf[hi_i];
        if ((a > b) == up) { buf[lo_i] = b; buf[hi_i] = a; }
      }
      __syncthreads();
    }
  }
  for (int k = tid; k < S + Sf; k += 128) t_all[(size_t)r * (S + Sf) + k] = buf[k];
}

// ------------------------------------------------------------------------------------------------
// compositing: NeRF.composite (frequency_nerf.py:283-343).  One warp per ray.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int s = 16; s > 0; s >>= 1) v += __shfl_xor_sync(0xffffffffu, v, s);
  return v;
}
__device__ __forceinline__ float warp_incl_scan(float v, int lane) {
#pragma unroll
  for (int s = 1; s < 32; s <<= 1) {
    float o = __shfl_up_sync(0xffffffffu, v, s);
    if (lane >= s) v += o;
  }
  return v;
}

__global__ void composite_fwd_kernel(int R, int S, const float* __restrict__ sigma, const float* __restrict__ rgb,
                                     const float* __restrict__ t, const float* __restrict__ dirs, int white_bg,
                                     float* __restrict__ rgb_map, float* __restrict__ depth,
                                     float* __restrict__ opacity, float* __restrict__ depth_var,
                                     float* __restrict__ rgb_var, float* __restrict__ weights,
                                     float* __restrict__ all_cum) {
  const int lane = threadIdx.x & 31;
  const int r = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (r >= R) return;
  const float dx = dirs[r * 3], dy = dirs[r * 3 + 1], dz = dirs[r * 3 + 2];
  const float len = sqrtf(dx * dx + dy * dy + dz * dz);
  const float* sg = sigma + (size_t)r * S;
  const float* tt = t + (size_t)r * S;
  const float* cc = rgb + (size_t)r * S * 3;
  float* ww = weights + (size_t)r * S;
  float carry = 0.f, a_r = 0.f, a_g = 0.f, a_b = 0.f, a_d = 0.f, a_o = 0.f;
  for (int k0 = 0; k0 < S; k0 += 32) {
    int k = k0 + lane;
    float sd = 0.f, tk = 0.f;
    if (k < S) {
      tk = tt[k];
      float gap = (k + 1 < S) ? __fsub_rn(tt[k + 1], tk) : 1e10f;
      sd = mul_rn(sg[k], mul_rn(gap, len));
    }
    float incl = warp_incl_scan(sd, lane);
    // exclusive prefix by SHIFTING the inclusive scan: (incl - sd) would cancel catastrophically on the
    // last sample, whose sd ~ 1e10 (frequency_nerf.py:304)
    float prev = __shfl_up_sync(0xffffffffu, incl, 1);
    float excl = carry + (lane == 0 ? 0.f : prev);
    carry += __shfl_sync(0xffffffffu, incl, 31);
    if (k < S) {
      float T = expf(-excl);
      float w = T * (1.f - expf(-sd));
      ww[k] = w;
      a_r += w * cc[k * 3];
      a_g += w * cc[k * 3 + 1];
      a_b += w * cc[k * 3 + 2];
      a_d += w * tk;
      a_o += w;
      if (k == S - 2) all_cum[r] = T;
    }
  }
  a_r = warp_sum(a_r); a_g = warp_sum(a_g); a_b = warp_sum(a_b); a_d = warp_sum(a_d); a_o = warp_sum(a_o);
  // second pass over the weights this lane just wrote: variances around the composited values
  float v_d = 0.f, v_c = 0.f;
  for (int k = lane; k < S; k += 32) {
    float w = ww[k];
    float dd = tt[k] - a_d;
    v_d += w * dd * dd;
    v_c += w * ((cc[k * 3] - a_r) + (cc[k * 3 + 1] - a_g) + (cc[k * 3 + 2] - a_b));
  }
  v_d = warp_sum(v_d);
  v_c = warp_sum(v_c);
  if (lane == 0) {
    float bg = white_bg ? (1.f - a_o) : 0.f;
    rgb_map[r * 3] = a_r + bg;
    rgb_map[r * 3 + 1] = a_g + bg;
    rgb_map[r * 3 + 2] = a_b + bg;
    depth[r] = a_d;
    opacity[r] = a_o;
    depth_var[r] = v_d;
    rgb_var[r] = v_c;
  }
}

// Backward.  With sd_k = sigma_k*gap_k*len, T_k = exp(-sum_{j<k} sd_j), w_k = T_k (1 - e^{-sd_k}) and
// G_k = dL/dw_k:   dL/dsd_k = G_k T_k e^{-sd_k} - sum_{j>k} G_j w_j.
// Dynamic smem: 2*S floats per warp (A_k = G_k w_k and B_k = G_k T_k e^{-sd_k}).
__global__ void composite_bwd_kernel(int R, int S, const float* __restrict__ sigma, const float* __restrict__ rgb,
                                     const float* __restrict__ t, const float* __restrict__ dirs, int white_bg,
                                     const float* __restrict__ g_rgb, const float* __restrict__ g_depth,
                                     const float* __restrict__ g_opacity, const float* __restrict__ g_weights,
                                     float* __restrict__ d_sigma, float* __restrict__ d_rgb,
                                     float* __restrict__ d_dirs) {
  extern __shared__ float sm[];
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const int r = blockIdx.x * (blockDim.x >> 5) + wib;
  if (r >= R) return;
  float* A = sm + (size_t)wib * 2 * S;
  float* Bv = A + S;
  const float dx = dirs[r * 3], dy = dirs[r * 3 + 1], dz = dirs[r * 3 + 2];
  const float len = sqrtf(dx * dx + dy * dy + dz * dz);
  const float* sg = sigma + (size_t)r * S;
  const float* tt = t + (size_t)r * S;
  const float* cc = rgb + (size_t)r * S * 3;
  const float gr = g_rgb ? g_rgb[r * 3] : 0.f, gg = g_rgb ? g_rgb[r * 3 + 1] : 0.f, gb = g_rgb ? g_rgb[r * 3 + 2] : 0.f;
  const float gd = g_depth ? g_depth[r] : 0.f;
  float go = g_opacity ? g_opacity[r] : 0.f;
  if (white_bg) go -= (gr + gg + gb);
  float carry = 0.f;
  for (int k0 = 0; k0 < S; k0 += 32) {
    int k = k0 + lane;
    float sd = 0.f, tk = 0.f;
    if (k < S) {
      tk = tt[k];
      float gap = (k + 1 < S) ? __fsub_rn(tt[k + 1], tk) : 1e10f;
      sd = mul_rn(sg[k], mul_rn(gap, len));
    }
    float incl = warp_incl_scan(sd, lane);
    // exclusive prefix by SHIFTING the inclusive scan: (incl - sd) would cancel catastrophically on the
    // last sample, whose sd ~ 1e10 (frequency_nerf.py:304)
    float prev = __shfl_up_sync(0xffffffffu, incl, 1);
    float excl = carry + (lane == 0 ? 0.f : prev);
    carry += __shfl_sync(0xffffffffu, incl, 31);
    if (k < S) {
      float T = expf(-excl), e = expf(-sd);
      float w = T * (1.f - e);
      float c0 = cc[k * 3], c1 = cc[k * 3 + 1], c2 = cc[k * 3 + 2];
      float G = gr * c0 + gg * c1 + gb * c2 + gd * tk + go;
      if (g_weights) G += g_weights[(size_t)r * S + k];
      A[k] = G * w;
      Bv[k] = G * T * e;
      float* dc = d_rgb + ((size_t)r * S + k) * 3;
      dc[0] = w * gr; dc[1] = w * gg; dc[2] = w * gb;
    }
  }
  __syncwarp();
  // reverse pass: suffix sums of A
  float suf_carry = 0.f, dlen = 0.f;
  int nchunks = (S + 31) / 32;
  for (int c = nchunks - 1; c >= 0; --c) {
    int k = c * 32 + (31 - lane);  // lane 0 handles the LAST sample of the chunk
    float a = k < S ? A[k] : 0.f;
    float incl = warp_incl_scan(a, lane);  // sum over samples >= k within the chunk
    float prev = __shfl_up_sync(0xffffffffu, incl, 1);
    float suf = suf_carry + (lane == 0 ? 0.f : prev);  // strictly after k
    suf_carry += __shfl_sync(0xffffffffu, incl, 31);
    if (k < S) {
      float dsd = Bv[k] - suf;
      float gapl = (k + 1 < S) ? __fsub_rn(tt[k + 1], tt[k]) : 1e10f;
      float s = sg[k];
      d_sigma[(size_t)r * S + k] = dsd * mul_rn(gapl, len);
      dlen += dsd * s * gapl;
    }
  }
  dlen = warp_sum(dlen);
  if (lane == 0 && d_dirs) {
    float inv = dlen / len;
    d_dirs[r * 3] += inv * dx;
    d_dirs[r * 3 + 1] += inv * dy;
    d_dirs[r * 3 + 2] += inv * dz;
  }
}

// ------------------------------------------------------------------------------------------------
// 2 * mean Huber(delta = 0.5)  (base_losses.py:155-156) with its gradient
// ------------------------------------------------------------------------------------------------
__global__ void huber2_kernel(long long n, const float* __restrict__ pred, const float* __restrict__ target,
                              float scale, float* __restrict__ loss, float* __restrict__ d_pred) {
  const float delta = 0.5f;
  float acc = 0.f;
  const float norm = 2.f * scale / (float)n;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    float z = pred[i] - target[i], az = fabsf(z);
    acc += az < delta ? 0.5f * z * z : delta * (az - 0.5f * delta);
    // torch's clamp form: a NaN residual keeps a NaN gradient (a copysign of delta would hide it), +-inf gives +-delta
    if (d_pred) d_pred[i] = norm * (z < -delta ? -delta : (z > delta ? delta : z));
  }
  acc = warp_sum(acc);
  __shared__ float red[32];
  int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) red[warp] = acc;
  __syncthreads();
  if (warp == 0) {
    float v = lane < (int)(blockDim.x >> 5) ? red[lane] : 0.f;
    v = warp_sum(v);
    if (lane == 0 && loss) atomicAdd(loss, v * norm);
  }
}

}  // namespace sparf

using namespace sparf;

namespace sparf {
// ------------------------------------------------------------------------------------------------
// stand-alone positional encoding (FrequencyEmbedder.__call__ + NeRF.positional_encoding, frequency_nerf.py:47-69,
// 229-258): out[n][c*2L + {0, L} + j] = w_j * {sin, cos}(x[n][c] * 2^j pi).  The MLP kernels fuse this; the tensor op
// exists so that the mirrored methods are callable on their own.
// ------------------------------------------------------------------------------------------------
__global__ void posenc_fwd_kernel(long long n, int C, int L, const float* __restrict__ x, C2F c2f, float* __restrict__ out) {
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int width = 2 * C * L;
  if (idx >= n * width) return;
  const int col = (int)(idx % width);
  const long long row = idx / width;
  const int c = col / (2 * L), rem = col - c * 2 * L, is_cos = rem >= L, j = rem - is_cos * L;
  const float arg = mul_rn(x[row * C + c], band_freq(j));
  out[idx] = mul_rn(is_cos ? cosf(arg) : sinf(arg), band_weight(c2f, L, j));
}

// d_x[n][c] = sum_j f_j w_j (g_sin cos(arg) - g_cos sin(arg))
__global__ void posenc_bwd_kernel2(long long n, int C, int L, const float* __restrict__ x, C2F c2f,
                                   const float* __restrict__ g_out, float* __restrict__ d_x) {
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n * C) return;
  const int c = (int)(idx % C);
  const long long row = idx / C;
  const float* g = g_out + row * 2 * C * L + c * 2 * L;
  float acc = 0.f;
  for (int j = 0; j < L; ++j) {
    const float f = band_freq(j), arg = mul_rn(x[idx], f);
    acc += f * band_weight(c2f, L, j) * (g[j] * cosf(arg) - g[L + j] * sinf(arg));
  }
  d_x[idx] = acc;
}

}  // namespace sparf
using namespace sparf;

extern "C" int sparf_posenc_forward(int64_t n, int32_t channels, int32_t L, const float* x, int32_t use_c2f, float c2f_start,
                                    float c2f_range, const float* progress, float* out, sparf_stream_t stream) {
  SPARF_REQUIRE(n >= 0 && channels > 0 && L > 0 && L <= 16, "posenc: bad sizes n=%lld C=%d L=%d", (long long)n, channels, L);
  if (n == 0) return SPARF_OK;
  C2F c2f{use_c2f, c2f_start, c2f_range, progress};
  const long long total = n * 2 * channels * L;
  posenc_fwd_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(n, channels, L, x, c2f, out);
  SPARF_CHECK_LAUNCH("posenc_fwd_kernel");
  return SPARF_OK;
}

extern "C" int sparf_posenc_backward(int64_t n, int32_t channels, int32_t L, const float* x, int32_t use_c2f, float c2f_start,
                                     float c2f_range, const float* progress, const float* d_out, float* d_x,
                                     sparf_stream_t stream) {
  SPARF_REQUIRE(n >= 0 && channels > 0 && L > 0 && L <= 16, "posenc: bad sizes n=%lld C=%d L=%d", (long long)n, channels, L);
  if (n == 0) return SPARF_OK;
  C2F c2f{use_c2f, c2f_start, c2f_range, progress};
  const long long total = n * channels;
  posenc_bwd_kernel2<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(n, channels, L, x, c2f, d_out, d_x);
  SPARF_CHECK_LAUNCH("posenc_bwd_kernel2");
  return SPARF_OK;
}

extern "C" int sparf_raygen_forward(int32_t B, int32_t n, int32_t W, const float* pose_w2c, const float* intr_inv,
                                    const int64_t* ray_idx, const float* pixels, int32_t per_image,
                                    float* origins, float* dirs, sparf_stream_t stream) {
  SPARF_REQUIRE(B > 0 && n >= 0, "raygen: bad sizes B=%d n=%d", B, n);
  SPARF_REQUIRE((ray_idx != nullptr) != (pixels != nullptr), "raygen: exactly one of ray_idx / pixels must be given");
  if (n == 0) return SPARF_OK;
  PixelSrc src{ray_idx, pixels, per_image, W, n};
  dim3 grid(ceil_div(n, 128), B);
  raygen_fwd_kernel<<<grid, 128, 0, (cudaStream_t)stream>>>(n, pose_w2c, intr_inv, src, origins, dirs);
  SPARF_CHECK_LAUNCH("raygen_fwd_kernel");
  return SPARF_OK;
}

extern "C" int sparf_raygen_backward(int32_t B, int32_t n, int32_t W, const float* pose_w2c, const float* intr_inv,
                                     const int64_t* ray_idx, const float* pixels, int32_t per_image,
                                     const float* d_origins, const float* d_dirs, float* d_pose_w2c,
                                     float* d_pixels, sparf_stream_t stream) {
  SPARF_REQUIRE(B > 0 && n >= 0, "raygen: bad sizes B=%d n=%d", B, n);
  SPARF_REQUIRE((ray_idx != nullptr) != (pixels != nullptr), "raygen: exactly one of ray_idx / pixels must be given");
  if (n == 0) return SPARF_OK;
  PixelSrc src{ray_idx, pixels, per_image, W, n};
  dim3 grid(ceil_div(n, 256), B);
  SPARF_REQUIRE(d_pixels == nullptr || pixels != nullptr, "raygen: d_pixels needs the float-pixel path");
  raygen_bwd_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(n, pose_w2c, intr_inv, src, d_origins, d_dirs, d_pose_w2c, d_pixels);
  SPARF_CHECK_LAUNCH("raygen_bwd_kernel");
  return SPARF_OK;
}

extern "C" int sparf_sample_depth(int32_t R, int32_t S, float near, float range, int32_t inverse, const float* rand,
                                  const float* far_per_ray, float* t, sparf_stream_t stream) {
  SPARF_REQUIRE(R >= 0 && S > 0, "sample_depth: bad sizes R=%d S=%d", R, S);
  long long total = (long long)R * S;
  if (total == 0) return SPARF_OK;
  sample_depth_kernel<<<ceil_div(total, 256), 256, 0, (cudaStream_t)stream>>>(total, S, near, range, inverse, rand,
                                                                              far_per_ray, t);
  SPARF_CHECK_LAUNCH("sample_depth_kernel");
  return SPARF_OK;
}

extern "C" int sparf_sample_pdf_merge(int32_t R, int32_t S, int32_t S_fine, float near, float far,
                                      const float* weights, const float* t_coarse, const float* u, float* t_fine,
                                      float* t_all, sparf_stream_t stream) {
  SPARF_REQUIRE(R >= 0 && S > 0 && S_fine > 0, "sample_pdf: bad sizes R=%d S=%d Sf=%d", R, S, S_fine);
  SPARF_REQUIRE(S <= 4096 - S_fine, "sample_pdf: S + S_fine = %lld exceeds the limit S + S_fine <= 4096",
                (long long)S + S_fine);
  if (R == 0) return SPARF_OK;
  int npow2 = 1;
  while (npow2 < S + S_fine) npow2 <<= 1;
  size_t smem = (size_t)(S + 1 + npow2) * sizeof(float);
  sample_pdf_merge_kernel<<<R, 128, smem, (cudaStream_t)stream>>>(S, S_fine, near, far, weights, t_coarse, u, t_fine,
                                                                  t_all, npow2);
  SPARF_CHECK_LAUNCH("sample_pdf_merge_kernel");
  return SPARF_OK;
}

extern "C" int sparf_composite_forward(int32_t R, int32_t S, const float* sigma, const float* rgb, const float* t,
                                       const float* dirs, int32_t white_bg, float* rgb_map, float* depth,
                                       float* opacity, float* depth_var, float* rgb_var, float* weights,
                                       float* all_cumulated, sparf_stream_t stream) {
  SPARF_REQUIRE(R >= 0 && S >= 2, "composite: bad sizes R=%d S=%d", R, S);
  if (R == 0) return SPARF_OK;
  composite_fwd_kernel<<<ceil_div(R, 4), 128, 0, (cudaStream_t)stream>>>(R, S, sigma, rgb, t, dirs, white_bg, rgb_map,
                                                                         depth, opacity, depth_var, rgb_var, weights,
                                                                         all_cumulated);
  SPARF_CHECK_LAUNCH("composite_fwd_kernel");
  return SPARF_OK;
}

extern "C" int sparf_composite_backward(int32_t R, int32_t S, const float* sigma, const float* rgb, const float* t,
                                        const float* dirs, int32_t white_bg, const float* g_rgb_map,
                                        const float* g_depth, const float* g_opacity, const float* g_weights,
                                        float* d_sigma, float* d_rgb, float* d_dirs, sparf_stream_t stream) {
  SPARF_REQUIRE(R >= 0 && S >= 2, "composite: bad sizes R=%d S=%d", R, S);
  SPARF_REQUIRE(S <= 4096, "composite_backward: S = %d exceeds the limit S <= 4096 (2*S floats of shared memory per ray)", S);
  if (R == 0) return SPARF_OK;
  size_t smem = (size_t)4 * 2 * S * sizeof(float);
  if (smem > 48 * 1024) {
    SPARF_CHECK_CUDA(cudaFuncSetAttribute(composite_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  }
  composite_bwd_kernel<<<ceil_div(R, 4), 128, smem, (cudaStream_t)stream>>>(R, S, sigma, rgb, t, dirs, white_bg,
                                                                            g_rgb_map, g_depth, g_opacity, g_weights,
                                                                            d_sigma, d_rgb, d_dirs);
  SPARF_CHECK_LAUNCH("composite_bwd_kernel");
  return SPARF_OK;
}

extern "C" int sparf_huber2_fwd_bwd(int64_t n, const float* pred, const float* target, float scale, float* loss,
                                    float* d_pred, sparf_stream_t stream) {
  SPARF_REQUIRE(n >= 0, "huber2: bad n");
  if (n == 0) return SPARF_OK;
  int blocks = (int)((n + 255) / 256);
  if (blocks > 1024) blocks = 1024;
  huber2_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(n, pred, target, scale, loss, d_pred);
  SPARF_CHECK_LAUNCH("huber2_kernel");
  return SPARF_OK;
}
