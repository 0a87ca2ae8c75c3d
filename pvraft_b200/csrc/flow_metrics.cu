// Training extras on the device (SURVEY.md section 8f, row f3): the masked L1 flow loss of tools/loss.py:16-40 and the
// end-point-error statistics of tools/metric.py:6-79, one pass over the points each, accumulated in double; the loss's
// backward needs no host synchronisation (the point count and the incoming gradient are read from device memory).
#include "fixed_point.cuh"

namespace pvraft {

// acc[0] = sum over valid points of |ex|+|ey|+|ez|     acc[1] = number of valid points (mask > 0)
// acc[2] = sum of the end-point errors ||e||            acc[3..5] = points with (epe < .05 or rel < .05), (epe < .1 or rel < .1),
//                                                                  (epe > .3 or rel > .1), rel = epe / (||gt|| + 1e-4)   (metric.py:66-77)
// DET: the grid is capped by a constant, so each warp's sums cover the same points on every GPU; they enter the [6]
// fixed-point workspace `acc` points at then (fixed_point.cuh)
template <bool DET>
__global__ void __launch_bounds__(256) k_flow_metrics(const float* __restrict__ est, const float* __restrict__ gt, const float* __restrict__ mask,
                                                      long long points, double* __restrict__ acc) {
    __shared__ double s_acc[6];
    if (threadIdx.x < 6) s_acc[threadIdx.x] = 0.0;
    __syncthreads();
    float v[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < points; p += (long long)gridDim.x * blockDim.x) {
        if (mask && !(__ldg(mask + p) > 0.f)) continue;
        const float gx = __ldg(gt + 3 * p), gy = __ldg(gt + 3 * p + 1), gz = __ldg(gt + 3 * p + 2);
        const float ex = __ldg(est + 3 * p) - gx, ey = __ldg(est + 3 * p + 1) - gy, ez = __ldg(est + 3 * p + 2) - gz;
        const float epe = sqrtf(ex * ex + ey * ey + ez * ez);
        const float rel = epe / (sqrtf(gx * gx + gy * gy + gz * gz) + 1e-4f);
        v[0] += fabsf(ex) + fabsf(ey) + fabsf(ez);
        v[1] += 1.f;
        v[2] += epe;
        v[3] += (epe < 0.05f || rel < 0.05f) ? 1.f : 0.f;
        v[4] += (epe < 0.1f || rel < 0.1f) ? 1.f : 0.f;
        v[5] += (epe > 0.3f || rel > 0.1f) ? 1.f : 0.f;
    }
#pragma unroll
    for (int i = 0; i < 6; ++i) {
        const float s = warp_sum(v[i]);
        if constexpr (DET) {
            if (lane_id() == 0 && s != 0.f) fx_atomic(reinterpret_cast<unsigned long long*>(acc) + i * kFxWords, (double)s);
        } else {
            if (lane_id() == 0 && s != 0.f) atomicAdd(&s_acc[i], (double)s);
        }
    }
    if constexpr (DET) return;
    __syncthreads();
    if (threadIdx.x < 6 && s_acc[threadIdx.x] != 0.0) atomicAdd(acc + threadIdx.x, s_acc[threadIdx.x]);
}

// d/d est of  weight * mean_{valid points, 3 components} |est - gt|  times the upstream gradient g (device scalar)
__global__ void __launch_bounds__(256) k_flow_l1_bwd(const float* __restrict__ est, const float* __restrict__ gt, const float* __restrict__ mask,
                                                     long long points, const double* __restrict__ acc, const float* __restrict__ g, float weight,
                                                     float* __restrict__ d_est) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= points * 3) return;
    const long long p = i / 3;
    const double cnt = acc[1];
    const float scale = cnt > 0.0 ? (float)((double)(__ldg(g) * weight) / (3.0 * cnt)) : 0.f;
    const float e = __ldg(est + i) - __ldg(gt + i);
    const bool ok = !mask || __ldg(mask + p) > 0.f;
    d_est[i] = ok ? (e > 0.f ? scale : (e < 0.f ? -scale : 0.f)) : 0.f;
}

}  // namespace pvraft

using namespace pvraft;

extern "C" int pvraft_flow_metrics_fwd(const float* est, const float* gt, const float* mask, int64_t points, double* acc, void* det_workspace,
                                       void* stream) {
    if (!est || !gt || !acc || points <= 0) return fail(PVRAFT_ERR_BAD_ARG, "flow_metrics: bad argument");
    long long blocks = (points + 255) / 256;
    const long long cap = det_workspace ? kDetCtas : (long long)sm_count() * 8;
    if (blocks > cap) blocks = cap;
    cudaStream_t st = (cudaStream_t)stream;
    if (!det_workspace) {
        k_flow_metrics<false><<<(unsigned)blocks, 256, 0, st>>>(est, gt, mask, points, acc);
        return check_launch("flow_metrics");
    }
    k_flow_metrics<true><<<(unsigned)blocks, 256, 0, st>>>(est, gt, mask, points, static_cast<double*>(det_workspace));
    const int rc = check_launch("flow_metrics");
    if (rc) return rc;
    return fx_flush_f64(static_cast<const unsigned long long*>(det_workspace), 1, 6, 6, 0, acc, st);
}

extern "C" int64_t pvraft_flow_metrics_det_workspace_bytes(void) { return 6 * kFxWords * 8; }

extern "C" int pvraft_flow_l1_bwd(const float* est, const float* gt, const float* mask, int64_t points, const double* acc, const float* g,
                                  float weight, float* d_est, void* stream) {
    if (!est || !gt || !acc || !g || !d_est || points <= 0) return fail(PVRAFT_ERR_BAD_ARG, "flow_l1_bwd: bad argument");
    const long long total = (long long)points * 3;
    k_flow_l1_bwd<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(est, gt, mask, points, acc, g, weight, d_est);
    return check_launch("flow_l1_bwd");
}
