// dalm_b200 — C-ABI plumbing shared by all translation units: error string, launch counter, version, device probe.
#include "common.cuh"
#include <stdarg.h>
#include <atomic>

namespace dalm {
static thread_local char g_err[1024] = "";
static std::atomic<long long> g_launches{0};

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
int check_launch(const char* what) {
  cudaError_t e = cudaPeekAtLastError();
  if (e != cudaSuccess) {
    set_error("%s: launch failed: %s", what, cudaGetErrorString(e));
    (void)cudaGetLastError();
    return 3;
  }
  return 0;
}
void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }
static int device_attr(cudaDeviceAttr a, int fallback) {
  int dev = 0, v = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&v, a, dev) != cudaSuccess || v <= 0) return fallback;
  return v;
}
int num_sms() {
  static const int n = device_attr(cudaDevAttrMultiProcessorCount, 132);
  return n;
}
long long l2_bytes() {
  static const long long n = device_attr(cudaDevAttrL2CacheSize, 50 << 20);
  return n;
}
}  // namespace dalm

extern "C" const char* dalm_b200_last_error() { return dalm::g_err; }
extern "C" const char* dalm_b200_version() { return "dalm_b200 0.1.0 (sm_90a)"; }
extern "C" long long dalm_b200_launch_count() { return dalm::g_launches.load(); }
extern "C" void dalm_b200_reset_launch_count() { dalm::g_launches.store(0); }

// 0 if the current device is a compute-capability 9.0 part (H100); non-zero + message otherwise.
extern "C" int dalm_b200_probe_device() {
  int dev = 0;
  DALM_CUDA(cudaGetDevice(&dev));
  cudaDeviceProp prop;
  DALM_CUDA(cudaGetDeviceProperties(&prop, dev));
  DALM_REQUIRE(prop.major == 9 && prop.minor == 0, "dalm_b200 is built for sm_90a only; device %d is sm_%d%d (%s)", dev, prop.major,
               prop.minor, prop.name);
  return 0;
}
