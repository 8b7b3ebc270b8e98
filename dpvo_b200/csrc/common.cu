// Error text, launch counter and version for the C-ABI (include/dpvo_b200.h).
#include "common.cuh"
#include <stdarg.h>

namespace dpvo {
static thread_local char g_err[512] = "";
std::atomic<long long> g_launches{0};

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
}  // namespace dpvo

extern "C" const char* dpvo_version(void) { return "dpvo_b200 0.1 (sm_90a)"; }
extern "C" const char* dpvo_last_error(void) { return dpvo::g_err; }
extern "C" int64_t dpvo_launch_count(void) { return (int64_t)dpvo::g_launches.load(); }
