// Host-side helpers shared by every translation unit of libymp_b200.so.
#pragma once
#include <cuda_runtime.h>
#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>

#include <atomic>

#include "../../include/ymp.h"

namespace ymp {

int set_error(int code, const char* fmt, ...);
extern std::atomic<uint64_t> g_launches;
inline void count_launch(uint64_t n = 1) { g_launches.fetch_add(n, std::memory_order_relaxed); }
int num_sms();  // SM count of the current device (cached)

// Deterministic mode (ymp_set_deterministic, process-wide): the launchers of the four order-dependent sums (split-K
// GEMM, LayerNorm gamma/beta gradients, column sums, sum of squares) then write one partial per CTA to a caller-provided
// workspace and add the partials to the output in index order (ordered_sum below) instead of by atomics.  Read when a
// call is launched, so a captured CUDA graph keeps the mode it was captured under.
extern int g_deterministic;

// out[r * ld_out + c] = ((out + parts[0]) + parts[1]) + ... + parts[nparts - 1], part k of element (r, c) at
// parts[k * part_stride + r * ld_parts + c]; r < rows, c < cols (one fixed order, whatever the launch).  With out2 set,
// the same launch also sums parts2 into out2 (same geometry).
int ordered_sum(float* out, long ld_out, const float* parts, long ld_parts, long part_stride, int rows, int cols,
                int nparts, cudaStream_t st, float* out2 = nullptr, const float* parts2 = nullptr);

#define YMP_CHECK_ARG(cond, ...)                                   \
  do {                                                             \
    if (!(cond)) return ymp::set_error(YMP_EINVAL, __VA_ARGS__);   \
  } while (0)

#define YMP_CUDA(expr)                                                                  \
  do {                                                                                  \
    cudaError_t _e = (expr);                                                            \
    if (_e != cudaSuccess)                                                              \
      return ymp::set_error(YMP_ECUDA, "%s failed: %s (%s:%d)", #expr,                  \
                            cudaGetErrorString(_e), __FILE__, __LINE__);                \
  } while (0)

#define YMP_LAUNCH_CHECK()                                                              \
  do {                                                                                  \
    cudaError_t _e = cudaPeekAtLastError();                                             \
    if (_e != cudaSuccess) {                                                            \
      cudaGetLastError();                                                               \
      return ymp::set_error(YMP_ECUDA, "kernel launch failed: %s (%s:%d)",              \
                            cudaGetErrorString(_e), __FILE__, __LINE__);                \
    }                                                                                   \
    ymp::count_launch();                                                                \
  } while (0)

// Per-device "done once" flag for cudaFuncSetAttribute (function attributes belong to the device's context: a process
// that drives several GPUs must set them on each).  Usage: static DeviceOnce once; if (once.first()) { ...set... }
struct DeviceOnce {
  bool done[64] = {};
  bool first() {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return true;
    if (done[dev]) return false;
    done[dev] = true;
    return true;
  }
};

// Per-device running maximum (dynamic shared-memory opt-in that grows with the problem size).
struct DeviceMax {
  int cur[64] = {};
  bool raise(int v) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return true;
    if (v <= cur[dev]) return false;
    cur[dev] = v;
    return true;
  }
};

static inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

}  // namespace ymp
