// Error plumbing + device queries of the C ABI (include/pvraft_b200.h), and the tensor-map encoder of the TMA kernels.
#include <stdarg.h>
#include <string.h>

#include "tma.cuh"

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

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// a 2-D row-major tensor [rows, cols] with row stride ld (elements), loaded as boxes of [box_rows, 32] elements
static int encode_2d(CUtensorMap* map, CUtensorMapDataType dtype, int esize, CUtensorMapSwizzle swizzle, const void* base, long long rows,
                     int cols, long long ld, int box_rows, const char* op) {
    // through the driver entry point (no link-time dependency on libcuda), looked up once: the initialisation of a
    // function-local static is thread-safe, and the library is called from several host threads (nn.DataParallel)
    static const EncodeTiledFn encode = []() -> EncodeTiledFn {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
            return reinterpret_cast<EncodeTiledFn>(p);
        return nullptr;
    }();
    if (!encode) return fail(PVRAFT_ERR_UNSUPPORTED, "%s: cuTensorMapEncodeTiled is not available from this driver", op);
    const cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
    const cuuint64_t strides[1] = {(cuuint64_t)ld * esize};
    const cuuint32_t box[2] = {32, (cuuint32_t)box_rows};
    const cuuint32_t estr[2] = {1, 1};
    const CUresult r = encode(map, dtype, 2, const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle,
                              CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return fail(PVRAFT_ERR_UNSUPPORTED, "%s: cuTensorMapEncodeTiled failed (%d)", op, (int)r);
    return 0;
}

int make_tensor_map(CUtensorMap* map, const float* base, long long rows, int cols, long long ld, int box_rows, const char* op) {
    return encode_2d(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, CU_TENSOR_MAP_SWIZZLE_128B, base, rows, cols, ld, box_rows, op);
}

int make_tensor_map_bf16(CUtensorMap* map, const uint16_t* base, long long rows, int cols, long long ld, int box_rows, const char* op) {
    return encode_2d(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, CU_TENSOR_MAP_SWIZZLE_64B, base, rows, cols, ld, box_rows, op);
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
        case 6: return (int)sizeof(pvraft_update_chain_args);
        default: return -1;
    }
}
