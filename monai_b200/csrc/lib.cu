// Library-level entry points of the C ABI (include/monai_b200.h): version, error string, launch counter.
#include "common.cuh"
#include "../../include/monai_b200.h"
#include <atomic>
#include <cstdarg>

namespace b200 {

static thread_local char t_err[1024] = "";
static std::atomic<long long> g_launches{0};

char* err_buf() { return t_err; }

int set_err(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(t_err, sizeof(t_err), fmt, ap);
  va_end(ap);
  return code;
}

void note_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }

int num_sms() {
  static int cached = 0;
  if (cached == 0) {
    int dev = 0, n = 0;
    if (cudaGetDevice(&dev) == cudaSuccess &&
        cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess && n > 0)
      cached = n;
    else
      cached = 132;   // H100 SXM
  }
  return cached;
}

}  // namespace b200

extern "C" int b200_abi_version(void) { return B200_ABI_VERSION; }
extern "C" const char* b200_last_error(void) { return b200::err_buf(); }
extern "C" long long b200_launch_count(void) { return b200::g_launches.load(); }
