// Shared helpers for the sparf_b200 CUDA sources (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <cstdarg>
#include <cstdint>
#include <cstdio>

#include "../../include/sparf_b200.h"

namespace sparf {

// thread-local error text behind sparf_last_error()
void set_error(const char* fmt, ...);

#define SPARF_CHECK_CUDA(expr)                                                                   \
  do {                                                                                           \
    cudaError_t _e = (expr);                                                                     \
    if (_e != cudaSuccess) {                                                                     \
      ::sparf::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
      return SPARF_ERR_CUDA;                                                                     \
    }                                                                                            \
  } while (0)

// every kernel launch of the library goes through this macro: it also feeds sparf_launch_count()
extern unsigned long long g_launch_count;
#define SPARF_CHECK_LAUNCH(name)                                                                 \
  do {                                                                                           \
    ++::sparf::g_launch_count;                                                                   \
    cudaError_t _e = cudaGetLastError();                                                         \
    if (_e != cudaSuccess) {                                                                     \
      ::sparf::set_error("launch of %s failed: %s (%s:%d)", name, cudaGetErrorString(_e), __FILE__, __LINE__); \
      return SPARF_ERR_CUDA;                                                                     \
    }                                                                                            \
  } while (0)

#define SPARF_REQUIRE(cond, ...)                 \
  do {                                           \
    if (!(cond)) {                               \
      ::sparf::set_error(__VA_ARGS__);           \
      return SPARF_ERR_INVALID;                  \
    }                                            \
  } while (0)

// returns the status of a call that fails with a nonzero SPARF_ERR_*
#define SPARF_TRY(expr)      \
  do {                       \
    int _rc = (expr);        \
    if (_rc) return _rc;     \
  } while (0)

static inline int ceil_div(long long a, long long b) { return (int)((a + b - 1) / b); }
static inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// the blocks of `threads` threads that cover n items, and the item of the calling thread
static inline unsigned grid_of(long long n, int threads) { return (unsigned)((n + threads - 1) / threads); }
__device__ __forceinline__ long long thread_index() { return (long long)blockIdx.x * blockDim.x + threadIdx.x; }

// The layout of a caller's workspace: each take<T>(count) starts at the next multiple of 256 B and returns a typed
// pointer (NULL when the base is NULL: the carve only measures).  end = the last piece's offset plus its size.
struct WsCarver {
  char* base;
  size_t end = 0;
  explicit WsCarver(void* ws) : base((char*)ws) {}
  template <typename T>
  T* take(size_t count) {
    const size_t o = align_up(end, 256);
    end = o + count * sizeof(T);
    return base ? (T*)(base + o) : nullptr;
  }
};

// The largest scratch of a set of cub size queries.  cub sizes its scratch for the current device: without one a query
// fails, its error is cleared, ok turns false and the later queries are skipped.
struct CubScratch {
  size_t bytes = 0;
  bool ok = true;
  // query: cudaError_t (size_t& bytes), one cub call with a NULL scratch pointer
  template <typename Query>
  void add(Query query) {
    if (!ok) return;
    size_t b = 0;
    if (query(b) != cudaSuccess) {
      cudaGetLastError();
      ok = false;
    } else if (b > bytes) {
      bytes = b;
    }
  }
};

// A call's workspace ws of `have` bytes against the `need` bytes its carve measured: SPARF_ERR_INVALID for a NULL ws,
// SPARF_ERR_CUDA for need = 0 (cub could not size its scratch), SPARF_ERR_WORKSPACE when have < need.
static inline int check_workspace(const char* what, const void* ws, size_t have, size_t need) {
  SPARF_REQUIRE(ws, "%s: NULL workspace", what);
  if (need == 0) {
    set_error("%s: no current CUDA device to size the cub scratch for", what);
    return SPARF_ERR_CUDA;
  }
  if (have < need) {
    set_error("%s: workspace %zu B < %zu B", what, have, need);
    return SPARF_ERR_WORKSPACE;
  }
  return SPARF_OK;
}

// A row count read on the device (the *_rows and *_span MLP entry points): of the cap rows a kernel is sized for,
// starting at row m0 of the call, it processes min(cap, max(0, *rows - s - m0)), s = *start (start NULL: s = 0).  The
// span forward (start != NULL) adds s to the row of every global input, output and tape buffer it touches; workspace
// buffers stay call-local.  Kernels take it behind a template flag DYN; without it they process cap rows and never touch
// `rows` or `start`.
struct RowCount {
  const int64_t* rows;
  long long m0;
  const int64_t* start;
};
template <bool DYN>
__device__ __forceinline__ long long row_start(const RowCount& rc) {
  if constexpr (DYN) return rc.start ? *rc.start : 0;
  else return 0;
}
// START = false: the kernel is never given a start (the backward's kernels; the large GEMM and trunk-chain kernels take
// the span forward's rows through instantiations of their own), so its code stays that of the *_rows calls
template <bool DYN, bool START = true>
__device__ __forceinline__ long long live_rows(long long cap, const RowCount& rc) {
  if constexpr (DYN) {
    const long long k = *rc.rows - (START ? row_start<true>(rc) : 0) - rc.m0;
    return k < 0 ? 0 : (k < cap ? k : cap);
  } else {
    return cap;
  }
}

// number of SMs of the current device (cached)
int num_sms();

// the MLP engines that run their wide GEMMs on the tensor cores (gemm_wgmma.cu)
static inline bool is_tc(int engine) {
  return engine == SPARF_ENGINE_TC_3X || engine == SPARF_ENGINE_TC_1X || engine == SPARF_ENGINE_TC_3X_W1;
}
// the engine an MLP or density call runs on: AUTO resolved, -1 when the engine is not available on this device
int resolve_engine(int engine);

// ---- arithmetic that must round exactly like the reference's separate fp32 torch ops (no FMA
// contraction): the 2^9*pi positional-encoding band amplifies a 1-ulp difference in x by ~1e3.
__device__ __forceinline__ float mul_rn(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float add_rn(float a, float b) { return __fadd_rn(a, b); }

// torch.nn.functional.softplus (beta=1, threshold=20) and its derivative
__device__ __forceinline__ float softplus_f(float z) { return z > 20.f ? z : log1pf(expf(z)); }
__device__ __forceinline__ float softplus_grad_f(float z) {
  if (z > 20.f) return 1.f;
  float e = expf(z);
  return e / (e + 1.f);
}
__device__ __forceinline__ float sigmoid_f(float z) { return 1.f / (1.f + expf(-z)); }

// BARF coarse-to-fine weight of frequency band j (frequency_nerf.py:248-253), fp32 op-for-op:
//   alpha = (progress - start) / (end - start) * L ; w = (1 - cos(pi * clamp(alpha - j, 0, 1))) / 2
__device__ __forceinline__ float c2f_weight(float progress, float start, float den, int L, int j) {
  float alpha = mul_rn(__fdiv_rn(__fsub_rn(progress, start), den), (float)L);
  float x = fminf(fmaxf(__fsub_rn(alpha, (float)j), 0.f), 1.f);
  float c = cosf(mul_rn(x, 3.14159274101257324f));
  return __fdiv_rn(__fsub_rn(1.f, c), 2.f);
}

struct C2F {
  int enabled;
  float start, den;
  const float* progress;
};

__device__ __forceinline__ float band_weight(const C2F& c, int L, int j) {
  if (!c.enabled) return 1.f;
  return c2f_weight(*c.progress, c.start, c.den, L, j);
}

// frequency of band j: 2^j * float(pi) (exact scaling of the fp32 constant), frequency_nerf.py:52
__device__ __forceinline__ float band_freq(int j) { return ldexpf(3.14159274101257324f, j); }

}  // namespace sparf
