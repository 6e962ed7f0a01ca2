// Error plumbing, device queries.
#include <stdarg.h>
#include <string.h>

#include "common.cuh"

namespace anysd {

static thread_local char g_err[512] = "";

void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

int check_launch(const char* what) {
    cudaError_t e = cudaPeekAtLastError();
    if (e != cudaSuccess) {
        cudaGetLastError();
        set_error("%s: CUDA error %d (%s)", what, (int)e, cudaGetErrorString(e));
        return ANYSD_ECUDA;
    }
    return ANYSD_OK;
}

int sm_count() {
    static thread_local int cached_dev = -1, cached = 0;
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 132;
    if (dev != cached_dev) {
        cudaDeviceGetAttribute(&cached, cudaDevAttrMultiProcessorCount, dev);
        cached_dev = dev;
    }
    return cached > 0 ? cached : 132;
}

}  // namespace anysd

extern "C" {

const char* anysd_last_error(void) { return anysd::g_err; }

int anysd_version(void) { return 100; }

int anysd_device_info(int* sms, int* cc_major, int* cc_minor) {
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) {
        anysd::set_error("cudaGetDevice failed: %s (no CUDA device; there is no CPU fallback)", cudaGetErrorString(e));
        return ANYSD_ECUDA;
    }
    int a = 0, b = 0, c = 0;
    cudaDeviceGetAttribute(&a, cudaDevAttrMultiProcessorCount, dev);
    cudaDeviceGetAttribute(&b, cudaDevAttrComputeCapabilityMajor, dev);
    cudaDeviceGetAttribute(&c, cudaDevAttrComputeCapabilityMinor, dev);
    if (sms) *sms = a;
    if (cc_major) *cc_major = b;
    if (cc_minor) *cc_minor = c;
    return ANYSD_OK;
}
}
