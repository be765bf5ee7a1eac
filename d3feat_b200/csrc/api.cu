// Error state and launch counter shared by every entry point of libd3feat_b200.so, and the entry points that read
// them. Each op's entry point is defined in the file that implements it.
#include <stdarg.h>

#include "common.cuh"

namespace d3f {

static thread_local char g_err[512] = "";
static thread_local long long g_launches = 0;

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int cuda_fail(cudaError_t e, const char* what) {
  set_error("CUDA error %d (%s) at %s", (int)e, cudaGetErrorString(e), what);
  return D3F_ERR_CUDA;
}

void count_launch(int n) { g_launches += n; }

}  // namespace d3f

using namespace d3f;

extern "C" {

int d3f_version(void) { return 100; }

const char* d3f_last_error(void) { return g_err; }

long long d3f_launch_count(void) { return g_launches; }

}  // extern "C"
