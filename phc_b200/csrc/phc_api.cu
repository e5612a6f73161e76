// Error reporting / version entry points of libphc_b200.so (include/phc_b200.h).
#include <cuda_runtime.h>
#include <stdio.h>
#include <string.h>

#include "../../include/phc_b200.h"

static thread_local char g_err[512] = "";

extern "C" void phc_set_error(const char* msg) {
  strncpy(g_err, msg ? msg : "", sizeof(g_err) - 1);
  g_err[sizeof(g_err) - 1] = 0;
}

static unsigned long long g_launches = 0;   // kernels launched through this library (bench.py: gpu_launches)

extern "C" int phc_check_cuda(cudaError_t e, const char* what) {
  if (e == cudaSuccess) return PHC_OK;
  snprintf(g_err, sizeof(g_err), "%s: %s (%s)", what, cudaGetErrorString(e), cudaGetErrorName(e));
  return PHC_ERR_CUDA;
}

extern "C" void phc_count_launches(int n) { __atomic_fetch_add(&g_launches, (unsigned long long)n, __ATOMIC_RELAXED); }
extern "C" void phc_launch_count_add(int64_t n) { if (n > 0) __atomic_fetch_add(&g_launches, (unsigned long long)n, __ATOMIC_RELAXED); }
extern "C" int64_t phc_launch_count(void) { return (int64_t)__atomic_load_n(&g_launches, __ATOMIC_RELAXED); }
extern "C" const char* phc_last_error(void) { return g_err; }
extern "C" int phc_version(void) { return 200; }   /* 0.2.0 */
extern "C" int phc_compiled_sm(void) { return 90; }
