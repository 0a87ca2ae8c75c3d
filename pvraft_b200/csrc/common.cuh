// Shared device/host helpers for the pvraft_b200 kernels (sm_90a).
#pragma once
#include <cstdlib>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/pvraft_b200.h"

namespace pvraft {

constexpr int kWarp = 32;
constexpr unsigned kFull = 0xffffffffu;
constexpr int kSmemBudget = 227 * 1024;  // opt-in dynamic shared memory per CTA on sm_90 (H100)

// ---- host side error plumbing (definitions in capi.cu) -------------------------------------------
void set_error(const char* fmt, ...);
int fail(int code, const char* fmt, ...);
int check_launch(const char* what);
int sm_count();

template <typename Kernel>
inline int opt_in_smem(Kernel k, size_t bytes) {
    if (bytes > (size_t)kSmemBudget) return fail(PVRAFT_ERR_SMEM, "kernel needs %zu B of shared memory (> %d)", bytes, kSmemBudget);
    cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
    if (e != cudaSuccess) return fail((int)e, "cudaFuncSetAttribute(smem=%zu): %s", bytes, cudaGetErrorString(e));
    return 0;
}

// ---- device helpers -------------------------------------------------------------------------------
__device__ __forceinline__ int lane_id() { return threadIdx.x & 31; }
__device__ __forceinline__ int warp_id() { return threadIdx.x >> 5; }

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(kFull, v, o));
    return v;
}
__device__ __forceinline__ float warp_min(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fminf(v, __shfl_xor_sync(kFull, v, o));
    return v;
}
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(kFull, v, o);
    return v;
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(kFull, v, o);
    return v;
}

// float -> uint key with the same order, for atomicMin / atomicMax and radix selects on floats: negatives get every bit
// flipped, the rest the sign bit set (-0 orders below +0; a NaN with the sign bit clear above +inf); ord_float inverts it
__device__ __forceinline__ unsigned ord_key(float f) {
    const unsigned u = __float_as_uint(f);
    return u ^ ((unsigned)((int)u >> 31) | 0x80000000u);
}
__device__ __forceinline__ float ord_float(unsigned k) { return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k); }

// streaming (read-once) 128-bit loads that do not pollute L1
__device__ __forceinline__ float4 ld_stream_f4(const float4* p) {
    float4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
    return r;
}
__device__ __forceinline__ int4 ld_stream_i4(const int4* p) {
    int4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.s32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
    return r;
}

// GroupNorm scale/shift for one channel from raw double sums: y = x*scale + shift
struct GnAffine {
    float scale, shift;
};
__device__ __forceinline__ GnAffine gn_affine(const double* stats_bg /* (sum,sumsq) of the group */, double count,
                                              float gamma, float beta) {
    const double mean = stats_bg[0] / count;
    double var = stats_bg[1] / count - mean * mean;
    var = var < 0.0 ? 0.0 : var;
    const double rstd = rsqrt(var + 1e-5);
    GnAffine a;
    a.scale = (float)(rstd * (double)gamma);
    a.shift = (float)((double)beta - mean * rstd * (double)gamma);
    return a;
}

// GroupNorm raw sums of n fp32 values y without the fp32 error that gn_affine's var = sum y^2 / n - mean^2 would expose:
// plain fp32 partials of y^2 carry ~2^-24 mean^2, which stays standing next to the variance (a relative 2^-24 r^2 for a
// group whose mean is r times its spread).  So sum y^2 is formed from the fp32 sum of squares about a pivot p, one of the
// values, whose error is ~2^-24 of the spread: sum y^2 = sum (y - p)^2 + p (2 sum y - n p), in double (pivot_sumsq).  sum y
// itself comes from a compensated fp32 sum (kahan_add: the pair s - err holds it to ~2^-48), so that the mean is as exact as
// double accumulation would make it.
__device__ __forceinline__ void kahan_add(float& s, float& err, float y) {
    const float v = y - err, t = s + v;
    err = (t - s) - v;
    s = t;
}
__device__ __forceinline__ double kahan_value(float s, float err) { return (double)s - (double)err; }
__device__ __forceinline__ double pivot_sumsq(double sum_y, float p, float sdd, int n) {
    const double dp = p;
    return fma(dp, 2.0 * sum_y - (double)n * dp, (double)sdd);
}

__device__ __forceinline__ float apply_act(float x, int act, float slope) {
    if (act == PVRAFT_ACT_RELU) return fmaxf(x, 0.f);
    if (act == PVRAFT_ACT_LRELU) return x >= 0.f ? x : slope * x;
    return x;
}

// Branch-free form of apply_act for latency-critical single-warp code paths (a taken branch costs a warp ~25 cycles):
// y = max(x, lo) + slope * min(x, 0) with (lo, slope) = (-inf, 0) none, (0, 0) ReLU, (0, s) LeakyReLU -- exact in all three.
struct ActCoef {
    float lo, slope;
};
__device__ __forceinline__ ActCoef act_coef(int act, float slope) {
    ActCoef c;
    c.lo = act == PVRAFT_ACT_NONE ? -INFINITY : 0.f;
    c.slope = act == PVRAFT_ACT_LRELU ? slope : 0.f;
    return c;
}
__device__ __forceinline__ float apply_act(float x, const ActCoef& c) { return fmaf(c.slope, fminf(x, 0.f), fmaxf(x, c.lo)); }

// prologue of four consecutive channels: the folded GroupNorm affine, then the activation
__device__ __forceinline__ float4 tc_gn_act4(float4 x, const float4& sc, const float4& sh, const ActCoef& act) {
    x.x = apply_act(fmaf(x.x, sc.x, sh.x), act);
    x.y = apply_act(fmaf(x.y, sc.y, sh.y), act);
    x.z = apply_act(fmaf(x.z, sc.z, sh.z), act);
    x.w = apply_act(fmaf(x.w, sc.w, sh.w), act);
    return x;
}

// ConvGRU gates of the tensor-core kernels (tc_linear.cu, update_chain.cu)
__device__ __forceinline__ float tsigmoid(float x) { return 1.f / (1.f + expf(-x)); }
// ConvGRU state update h' = (1 - z) h + z tanh(q) (model/update.py:37-39); one definition for every kernel that applies it, so
// that the multiply-add contraction is the same everywhere
__device__ __forceinline__ float tgru_blend(float z, float h, float q_pre) { return (1.f - z) * h + z * tanhf(q_pre); }

// Contiguous split of `total` items over `parts` workers: worker w gets [begin, end).
__host__ __device__ __forceinline__ void split_range(long long total, int parts, int w, long long& begin, long long& end) {
    const long long per = (total + parts - 1) / parts;
    begin = per * w;
    end = begin + per;
    if (begin > total) begin = total;
    if (end > total) end = total;
}

// Launch with programmatic stream serialization (PDL): the grid may be scheduled while the previous kernel of the stream
// drains.  The kernel MUST execute pdl_wait() before its first global access (and may call pdl_trigger() at entry so that
// its own successor can be staged early).
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), int grid, int block, size_t smem, cudaStream_t stream, Args... args) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3((unsigned)grid);
    cfg.blockDim = dim3((unsigned)block);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, kernel, KArgs(args)...);
}

}  // namespace pvraft
