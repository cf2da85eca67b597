// Thread-local error string + build info for the C ABI.
#include "common.cuh"
#include <stdarg.h>
#include <atomic>

namespace lvg {
static thread_local char g_err[512] = "";

static std::atomic<long long> g_launches{0};
void count_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }
long long launches() { return g_launches.load(std::memory_order_relaxed); }

void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}
}  // namespace lvg

namespace lvg { long long launches(); }
extern "C" int64_t lvg_launch_count(void) { return (int64_t)lvg::launches(); }
extern "C" int lvg_abi_version(void) { return LVG_ABI_VERSION; }
extern "C" const char* lvg_last_error(void) { return lvg::g_err; }
extern "C" const char* lvg_build_info(void) {
    return "liblvg_ops sm_90a nvcc " __DATE__;
}
