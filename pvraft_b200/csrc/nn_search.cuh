// The distance of the brute-force nearest-neighbour searches that rank points by their own coordinates rather than by the
// kNN graph's expanded form |q|^2 + |x|^2 - 2 q.x (self_supervised.cu, flow_propagate.cu).
#pragma once
#include "common.cuh"

namespace pvraft {

// the squared length of the fp32 difference q - p, (dx*dx + dy*dy) + dz*dz rounded to nearest at every step, with no FMA
// contraction
__device__ __forceinline__ float diff_sq(float qx, float qy, float qz, const float4& p) {
    const float dx = __fsub_rn(qx, p.x), dy = __fsub_rn(qy, p.y), dz = __fsub_rn(qz, p.z);
    return __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
}

}  // namespace pvraft
