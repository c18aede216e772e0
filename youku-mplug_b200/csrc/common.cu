#include "common.h"

#include <string.h>

namespace ymp {

static thread_local char g_err[512] = "";
std::atomic<uint64_t> g_launches{0};
thread_local int g_pdl = 0;

int set_error(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}

int num_sms() {
  static int cached[64] = {0};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
  if (cached[dev] == 0) {
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0)
      n = 132;
    cached[dev] = n;
  }
  return cached[dev];
}

}  // namespace ymp

extern "C" {
const char* ymp_last_error(void) { return ymp::g_err; }
int ymp_abi_version(void) { return 3; }
uint64_t ymp_launch_count(void) { return ymp::g_launches.load(std::memory_order_relaxed); }
int ymp_set_pdl(int on) { const int prev = ymp::g_pdl; ymp::g_pdl = on ? 1 : 0; return prev; }
}
