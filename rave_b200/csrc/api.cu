// Library-level entry points: version, last-error string, launch counter.
#include <stdarg.h>

#include <atomic>

#include "common.cuh"

namespace rave {
static thread_local char g_err[512] = "";
static std::atomic<unsigned long long> g_launches{0};

void set_error(const char *fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
void count_launch(int n) { g_launches.fetch_add((unsigned long long)n, std::memory_order_relaxed); }
}  // namespace rave

extern "C" int rave_b200_version(void) { return 105; }
extern "C" const char *rave_b200_last_error(void) { return rave::g_err; }
extern "C" unsigned long long rave_b200_launch_count(void) {
  return rave::g_launches.load(std::memory_order_relaxed);
}
