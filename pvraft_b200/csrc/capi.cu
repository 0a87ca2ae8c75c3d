// Error plumbing + device queries of the C ABI (include/pvraft_b200.h).
#include <stdarg.h>
#include <string.h>

#include "common.cuh"

namespace pvraft {

static thread_local char g_err[512] = "";

void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

int fail(int code, const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return code;
}

int check_launch(const char* what) {
    const cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) return 0;
    return fail((int)e, "%s: launch failed: %s", what, cudaGetErrorString(e));
}

int sm_count() {
    static thread_local int cached_dev = -1, cached = 0;
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 132;
    if (dev != cached_dev) {
        int n = 0;
        if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
        cached = n;
        cached_dev = dev;
    }
    return cached;
}

}  // namespace pvraft

extern "C" int pvraft_version(void) { return PVRAFT_VERSION; }

extern "C" const char* pvraft_last_error_string(void) { return pvraft::g_err; }

extern "C" int pvraft_device_info(int* sm, int* smem_optin) {
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return pvraft::fail((int)e, "device_info: %s", cudaGetErrorString(e));
    int n = 0, s = 0;
    e = cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (e == cudaSuccess) e = cudaDeviceGetAttribute(&s, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
    if (e != cudaSuccess) return pvraft::fail((int)e, "device_info: %s", cudaGetErrorString(e));
    if (sm) *sm = n;
    if (smem_optin) *smem_optin = s;
    return 0;
}

extern "C" int pvraft_sizeof(int which) {
    switch (which) {
        case 0: return (int)sizeof(pvraft_linear_args);
        case 1: return (int)sizeof(pvraft_corrfeat_args);
        case 2: return (int)sizeof(pvraft_gru_args);
        case 3: return (int)sizeof(pvraft_flowout_args);
        case 4: return (int)sizeof(pvraft_tc_linear_args);
        case 5: return (int)sizeof(pvraft_knn_branch_args);
        default: return -1;
    }
}
