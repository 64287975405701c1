// supir_b200 — library-level C ABI: error string, version, launch counter; the per-device plumbing of common.cuh.
#include "common.cuh"
#include "supir_b200.h"

#include <atomic>
#include <cstdarg>
#include <cstdio>

namespace supir {

static thread_local char g_err[1024] = "";
std::atomic<long long> g_launches{0};

int set_error(int code, const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return code;
}

void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }

// current device, clamped into the per-device caches (function attributes and SM counts are per device)
int current_device_slot() {
    int dev = 0;
    cudaGetDevice(&dev);
    return dev < 0 ? 0 : (dev > 63 ? 63 : dev);
}

int device_sm_count() {
    static int sms[64] = {};
    const int d = current_device_slot();
    if (sms[d] == 0) {
        cudaDeviceGetAttribute(&sms[d], cudaDevAttrMultiProcessorCount, d);
        if (sms[d] <= 0) sms[d] = 132;
    }
    return sms[d];
}

}  // namespace supir

extern "C" const char* supir_last_error(void) { return supir::g_err; }
extern "C" int supir_version(void) { return 100; }
extern "C" long long supir_launch_count(void) { return supir::g_launches.load(); }
extern "C" void supir_reset_launch_count(void) { supir::g_launches.store(0); }
