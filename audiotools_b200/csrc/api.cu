// api.cu -- version, thread-local error message and kernel launch count of libb2a.so (include/b2a.h), and the SM
// count the persistent grids are sized by.
#include <atomic>

#include "b2a_common.h"

namespace b2a {
int num_sms() {
  constexpr int MAX_DEVICES = 64;
  static std::atomic<int> cached[MAX_DEVICES];  // 0: not queried yet
  int dev = 0, n = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return B2A_NUM_SMS;
  const bool cacheable = dev >= 0 && dev < MAX_DEVICES;
  if (cacheable && (n = cached[dev].load(std::memory_order_relaxed)) > 0) return n;
  if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = B2A_NUM_SMS;
  if (cacheable) cached[dev].store(n, std::memory_order_relaxed);
  return n;
}

char* err_buf() {
  static thread_local char buf[512] = {0};
  return buf;
}
int fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(err_buf(), 512, fmt, ap);
  va_end(ap);
  return code;
}
}  // namespace b2a

int64_t b2a_kernel_launches = 0;  // C linkage from its declaration in b2a.h

extern "C" int b2a_version(void) { return B2A_VERSION; }
extern "C" const char* b2a_last_error(void) { return b2a::err_buf(); }
