// C-ABI plumbing: version, error reporting, device probe.
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>

#include "cb_common.cuh"

namespace cb {

static thread_local char g_err[1024] = {0};

void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

int check_cuda(cudaError_t e, const char* what) {
    if (e == cudaSuccess) return 0;
    set_error("%s: %s (%d)", what, cudaGetErrorString(e), (int)e);
    return (int)e;
}

int device_sm_count() {
    static int n = 0;
    if (n == 0) {
        int dev = 0;
        if (cudaGetDevice(&dev) != cudaSuccess) return 132;
        if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
    }
    return n;
}

bool pdl_enabled() {
    static const bool on = !(getenv("CB_PDL") && atoi(getenv("CB_PDL")) == 0);
    return on;
}

static unsigned long long g_launches = 0;
void count_launches(int n) { __atomic_fetch_add(&g_launches, (unsigned long long)n, __ATOMIC_RELAXED); }
unsigned long long get_launches() { return __atomic_load_n(&g_launches, __ATOMIC_RELAXED); }

}  // namespace cb

extern "C" unsigned long long cb_launch_count(void) { return cb::get_launches(); }

extern "C" int cb_abi_version(void) { return CB_ABI_VERSION; }

extern "C" const char* cb_last_error(void) { return cb::g_err; }

extern "C" int cb_device_ok(void) {
    int dev = 0, major = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) {
        cudaGetLastError();
        return 0;
    }
    if (cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev) != cudaSuccess) {
        cudaGetLastError();
        return 0;
    }
    int minor = 0;
    if (cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev) != cudaSuccess) {
        cudaGetLastError();
        return 0;
    }
    return (major == 9 && minor == 0) ? 1 : 0;   // sm_90a code runs on compute capability 9.0 only
}
