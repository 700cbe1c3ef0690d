// Library-wide state of libb200vq.so (error text, launch counter, SM count, SM limit) and the entry points that report or
// set it.  Every other b200vq_* entry point is defined in the kernel file that implements it.
#include "../../include/b200vq.h"

#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>

#include "common.cuh"

namespace b200 {

static thread_local char g_err[512] = "";
std::atomic<long long> g_launches{0};

int set_error(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}

void count_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }

int current_device() {
  int dev = -1;
  return cudaGetDevice(&dev) == cudaSuccess ? dev : -1;
}

int num_sms() {
  static PerDevice cache;
  const int dev = current_device();
  if (dev < 0 || dev >= kMaxDevices) return 132;
  if (!cache.done[dev]) {
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
    cache.value[dev] = n;
    cache.done[dev] = true;
  }
  return cache.value[dev];
}

static std::atomic<int> g_sm_limit{-1};
int sm_limit() {
  int v = g_sm_limit.load(std::memory_order_relaxed);
  if (v < 0) {
    const char* e = getenv("B200VQ_SM_LIMIT");
    v = e ? atoi(e) : 0;
    if (v < 0) v = 0;
    g_sm_limit.store(v);
  }
  return v;
}

}  // namespace b200

using namespace b200;

extern "C" {

int b200vq_version(void) { return B200VQ_VERSION; }
const char* b200vq_last_error(void) { return g_err; }
const char* b200vq_arch(void) { return "sm_90a"; }
long long b200vq_launch_count(void) { return g_launches.load(); }

int b200vq_set_sm_limit(int n) { g_sm_limit.store(n < 0 ? 0 : n); return 0; }

}  // extern "C"
