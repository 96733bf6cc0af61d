// C-ABI entry points that dispatch between MLP engines, plus library-level bookkeeping.
#include <cstring>

#include "common.cuh"
#include "mlp_simt.cuh"

namespace sparf {

static thread_local char g_err[512] = "";
unsigned long long g_launch_count = 0;

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int num_sms() {
  static int cache[64] = {};
  int dev = 0;
  cudaGetDevice(&dev);
  int& n = cache[dev & 63];           // per device ordinal (several devices in one process)
  if (n == 0) {
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (n <= 0) n = 132;
  }
  return n;
}

// the wgmma kernels exist for sm_90a only
static bool device_is_sm90() {
  int dev = 0, major = 0, minor = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return false;
  cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev);
  cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev);
  return major == 9 && minor == 0;
}

static bool is_tc(int engine) { return engine == SPARF_ENGINE_TC_3X || engine == SPARF_ENGINE_TC_1X || engine == SPARF_ENGINE_TC_3X_W1; }

// AUTO -> the 3-pass tensor-core engine; both AUTO choices are parity engines
static int resolve_engine(const SparfMLP*, int engine) {
  if (engine == SPARF_ENGINE_AUTO) return device_is_sm90() ? SPARF_ENGINE_TC_3X : SPARF_ENGINE_SIMT_FP32;
  if (engine == SPARF_ENGINE_SIMT_FP32) return engine;
  return is_tc(engine) && device_is_sm90() ? engine : -1;
}

}  // namespace sparf

using namespace sparf;

extern "C" int sparf_version(void) { return SPARF_B200_VERSION; }
extern "C" const char* sparf_last_error(void) { return g_err; }
extern "C" uint64_t sparf_launch_count(void) { return g_launch_count; }

extern "C" int sparf_engine_available(int engine) {
  if (engine == SPARF_ENGINE_SIMT_FP32) return 1;
  if (is_tc(engine)) return device_is_sm90() ? 1 : 0;
  return 0;
}

extern "C" size_t sparf_mlp_workspace_bytes(const SparfMLP* mlp, int32_t R, int32_t S, int32_t backward, int32_t engine) {
  if (!mlp || R <= 0 || S <= 0) return 0;
  const int e = resolve_engine(mlp, engine);
  if (e < 0 || backward < 0 || backward > 2) return 0;
  return simt_workspace_bytes(mlp, R, S, backward, e);
}

extern "C" int sparf_mlp_forward(const SparfMLP* mlp, int32_t engine, int32_t R, int32_t S, const float* origins,
                                 const float* dirs, const float* t, const float* noise, float* sigma, float* rgb,
                                 void* workspace, size_t workspace_bytes, sparf_stream_t stream) {
  SPARF_REQUIRE(mlp && R >= 0 && S > 0, "mlp_forward: bad arguments");
  SPARF_REQUIRE(origins && dirs && t && sigma && rgb, "mlp_forward: NULL tensor");
  if (R == 0) return SPARF_OK;
  const int e = resolve_engine(mlp, engine);
  if (e < 0) {
    set_error("mlp_forward: engine %d not available in this build", engine);
    return SPARF_ERR_UNSUPPORTED;
  }
  return simt_mlp_forward(mlp, e, R, S, origins, dirs, t, noise, sigma, rgb, workspace, workspace_bytes, (cudaStream_t)stream);
}

extern "C" int sparf_mlp_backward(const SparfMLP* mlp, int32_t engine, int32_t R, int32_t S, const float* origins,
                                  const float* dirs, const float* t, const float* noise, const float* d_sigma,
                                  const float* d_rgb, const SparfMLPGrad* grad, float* d_origins, float* d_dirs,
                                  void* workspace, size_t workspace_bytes, sparf_stream_t stream) {
  SPARF_REQUIRE(mlp && R >= 0 && S > 0, "mlp_backward: bad arguments");
  SPARF_REQUIRE(origins && dirs && t && d_sigma && d_rgb && grad, "mlp_backward: NULL tensor");
  if (R == 0) return SPARF_OK;
  const int e = resolve_engine(mlp, engine);
  if (e < 0) {
    set_error("mlp_backward: engine %d not available in this build", engine);
    return SPARF_ERR_UNSUPPORTED;
  }
  return simt_mlp_backward(mlp, e, R, S, origins, dirs, t, noise, d_sigma, d_rgb, grad, d_origins, d_dirs, workspace,
                           workspace_bytes, (cudaStream_t)stream);
}

// ---------------------------------------------------------------- density queries: the trunk alone at arbitrary points
extern "C" size_t sparf_density_workspace_bytes(const SparfMLP* mlp, int64_t M, int32_t backward, int32_t engine) {
  if (!mlp || M <= 0) return 0;
  const int e = resolve_engine(mlp, engine);
  if (e < 0 || backward < 0 || backward > 1) return 0;
  return simt_density_workspace_bytes(mlp, M, backward, e);
}

extern "C" int sparf_density_forward(const SparfMLP* mlp, int32_t engine, int64_t M, const float* points, float* raw,
                                     float* feat, void* workspace, size_t workspace_bytes, sparf_stream_t stream) {
  SPARF_REQUIRE(mlp && M >= 0, "density_forward: bad arguments");
  if (M == 0) return SPARF_OK;
  SPARF_REQUIRE(points && raw, "density_forward: NULL tensor");
  const int e = resolve_engine(mlp, engine);
  if (e < 0) {
    set_error("density_forward: engine %d not available in this build", engine);
    return SPARF_ERR_UNSUPPORTED;
  }
  return simt_density_forward(mlp, e, M, points, raw, feat, workspace, workspace_bytes, (cudaStream_t)stream);
}

extern "C" int sparf_density_backward(const SparfMLP* mlp, int32_t engine, int64_t M, const float* points, const float* d_raw,
                                      const float* d_feat, const SparfMLPGrad* grad, float* d_points, void* workspace,
                                      size_t workspace_bytes, sparf_stream_t stream) {
  SPARF_REQUIRE(mlp && M >= 0, "density_backward: bad arguments");
  if (M == 0) return SPARF_OK;
  SPARF_REQUIRE(points && grad, "density_backward: NULL tensor");
  const int e = resolve_engine(mlp, engine);
  if (e < 0) {
    set_error("density_backward: engine %d not available in this build", engine);
    return SPARF_ERR_UNSUPPORTED;
  }
  return simt_density_backward(mlp, e, M, points, d_raw, d_feat, grad, d_points, workspace, workspace_bytes,
                               (cudaStream_t)stream);
}

// ---------------------------------------------------------------- tape variants: the training forward keeps what the
// backward needs, so that the backward does not recompute the forward
extern "C" size_t sparf_mlp_tape_bytes(const SparfMLP* mlp, int32_t engine, int32_t R, int32_t S) {
  if (!mlp || R <= 0 || S <= 0 || resolve_engine(mlp, engine) < 0) return 0;
  return simt_tape_bytes(mlp, R, S);
}

extern "C" int sparf_mlp_forward_tape(const SparfMLP* mlp, int32_t engine, int32_t R, int32_t S, const float* origins,
                                      const float* dirs, const float* t, const float* noise, float* sigma, float* rgb,
                                      void* tape, size_t tape_bytes, void* workspace, size_t workspace_bytes,
                                      sparf_stream_t stream) {
  SPARF_REQUIRE(mlp && R > 0 && S > 0 && origins && dirs && t && sigma && rgb && tape, "mlp_forward_tape: bad arguments");
  const int e = resolve_engine(mlp, engine);
  if (e < 0) {
    set_error("mlp_forward_tape: engine %d not available", engine);
    return SPARF_ERR_UNSUPPORTED;
  }
  return simt_mlp_forward_tape(mlp, e, R, S, origins, dirs, t, noise, sigma, rgb, tape, tape_bytes, workspace, workspace_bytes,
                               (cudaStream_t)stream);
}

extern "C" int sparf_mlp_backward_tape(const SparfMLP* mlp, int32_t engine, int32_t R, int32_t S, const float* origins,
                                       const float* dirs, const float* t, const float* sigma, const float* rgb,
                                       const float* d_sigma, const float* d_rgb, const SparfMLPGrad* grad,
                                       float* d_origins, float* d_dirs, void* tape, size_t tape_bytes, void* workspace,
                                       size_t workspace_bytes, sparf_stream_t stream) {
  SPARF_REQUIRE(mlp && R > 0 && S > 0 && origins && dirs && t && sigma && rgb && d_sigma && d_rgb && grad && tape,
                "mlp_backward_tape: bad arguments");
  const int e = resolve_engine(mlp, engine);
  if (e < 0) {
    set_error("mlp_backward_tape: engine %d not available", engine);
    return SPARF_ERR_UNSUPPORTED;
  }
  return simt_mlp_backward_tape(mlp, e, R, S, origins, dirs, t, rgb, d_sigma, d_rgb, grad, d_origins, d_dirs, tape, tape_bytes,
                                workspace, workspace_bytes, (cudaStream_t)stream);
}
