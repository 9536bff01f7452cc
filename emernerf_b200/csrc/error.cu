#include <stdarg.h>
#include <string.h>

#include "common.cuh"

namespace emer {
static thread_local char g_err[512] = "";
void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

// Per-device facts, cached (cudaGetDevice is a thread-local read; the attribute query runs once per device).
static int g_sm_count[64] = {0};
int current_device() {
    int dev = 0;
    cudaGetDevice(&dev);
    return (dev >= 0 && dev < 64) ? dev : 0;
}
int sm_count() {
    const int dev = current_device();
    if (g_sm_count[dev] == 0) {
        int n = 0;
        if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;   // H100 SXM
        g_sm_count[dev] = n;
    }
    return g_sm_count[dev];
}
}  // namespace emer

extern "C" const char* emer_last_error(void) { return emer::g_err; }
extern "C" int emer_version(void) { return 1; }
