// C-ABI plumbing: error string, version, device query.
#include <stdarg.h>
#include <stdlib.h>
#include <mutex>
#include <map>
#include <utility>
#include "common.cuh"

namespace lavb {
static thread_local char g_err[512] = "";
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

// SM count of the current device (cached per ordinal): persistent kernels size their grids from it.
// LAVB_NUM_SMS (read once) caps it: persistent CTAs with ~200 KB of shared memory leave no room for another stream's small
// kernels on their SMs, so a cap of e.g. 116 keeps 16 SMs free for the latency-bound chains of a second agent group.
int num_sms() {
  static int cache[64];
  static int cap = -1;
  if (cap < 0) { const char* e = getenv("LAVB_NUM_SMS"); cap = e ? atoi(e) : 0; }
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) { cudaGetLastError(); return kNumSMsH100; }
  if (dev >= 0 && dev < 64 && cache[dev] > 0) return cache[dev];
  int n = 0;
  if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) { cudaGetLastError(); return kNumSMsH100; }
  if (cap > 0 && cap < n) n = cap;
  if (dev >= 0 && dev < 64) cache[dev] = n;
  return n;
}

// cudaFuncAttributeMaxDynamicSharedMemorySize is a per-DEVICE attribute: set it per (kernel, device ordinal) whenever a launch
// needs more than the largest size set so far (erf_nb16's footprint grows with the image width, so a narrow first call must not
// cap later wide ones), under a lock (several host threads may drive their own pipelines).  Callers warm up before any stream
// capture.
cudaError_t ensure_dyn_smem(const void* kernel, int bytes) {
  static std::mutex mu;
  static std::map<std::pair<const void*, int>, int> largest;
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  std::lock_guard<std::mutex> lock(mu);
  auto it = largest.find({kernel, dev});
  if (it != largest.end() && it->second >= bytes) return cudaSuccess;
  e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  if (e == cudaSuccess) largest[{kernel, dev}] = bytes;
  return e;
}
}  // namespace lavb

extern "C" int lavb_abi_version(void) { return LAVB_ABI_VERSION; }
extern "C" int lavb_h16_dtype(void) { return LAVB_H16; }
extern "C" const char* lavb_last_error(void) { return lavb::g_err; }
extern "C" int lavb_device_cc(void) {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) { cudaGetLastError(); return -1; }
  cudaDeviceProp p;
  if (cudaGetDeviceProperties(&p, dev) != cudaSuccess) { cudaGetLastError(); return -1; }
  return p.major * 10 + p.minor;
}
