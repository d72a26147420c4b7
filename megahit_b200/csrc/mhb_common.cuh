// mhb_common.cuh -- helpers shared by the CUDA translation units of libmhb (not part of the C ABI).
#pragma once
#include <cuda_runtime.h>

#include "mhb.h"
#include "mhb_internal.h"

#define CK(call)                                                                                   \
  do {                                                                                             \
    cudaError_t e_ = (call);                                                                       \
    if (e_ != cudaSuccess)                                                                         \
      return mhb_set_error(MHB_ERR_CUDA, "%s failed at %s:%d: %s", #call, __FILE__, __LINE__,      \
                           cudaGetErrorString(e_));                                                \
  } while (0)
// every kernel launch site of the library goes through CK_LAUNCH(): the counter behind mhb_launch_count()
extern unsigned long long g_mhb_launches;
#define CK_LAUNCH()          \
  do {                       \
    ++g_mhb_launches;        \
    CK(cudaGetLastError());  \
  } while (0)

#define MHB_FOR_W(M) M(1) M(2) M(3) M(4) M(5) M(6) M(7) M(8) M(9) M(10) M(11) M(12) M(13) M(14) M(15) M(16)
#define MHB_FOR_WR(M) MHB_FOR_W(M) M(17)

// SM count of the device this process is bound to (mhb_device.cu)
int mhb_sm_count();
static inline int sm_count() { return mhb_sm_count(); }

// blocks for n items of per_block items each, at most blocks_per_sm per SM, at least 1
static inline unsigned grid_cap(uint64_t n, uint64_t per_block, unsigned blocks_per_sm) {
  const uint64_t g = std::min((n + per_block - 1) / per_block, (uint64_t)sm_count() * blocks_per_sm);
  return (unsigned)std::max<uint64_t>(g, 1);
}

// ms between start() and stop() on one stream, from two CUDA events (stop waits for the stream to reach it)
struct EventTimer {
  cudaEvent_t a, b;
  cudaStream_t st;
  explicit EventTimer(cudaStream_t s = 0) : st(s) {
    cudaEventCreate(&a);
    cudaEventCreate(&b);
  }
  EventTimer(const EventTimer &) = delete;
  EventTimer &operator=(const EventTimer &) = delete;
  ~EventTimer() {
    cudaEventDestroy(a);
    cudaEventDestroy(b);
  }
  void start() { cudaEventRecord(a, st); }
  double stop() {
    cudaEventRecord(b, st);
    cudaEventSynchronize(b);
    float ms = 0;
    cudaEventElapsedTime(&ms, a, b);
    return ms;
  }
};
