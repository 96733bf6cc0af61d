// Library-level bookkeeping: the error text, the launch counter, device queries and engine resolution.
#include "common.cuh"

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

// AUTO -> the 3-pass tensor-core engine; both AUTO choices are parity engines
int resolve_engine(int engine) {
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
