// The distance of the brute-force nearest-neighbour searches that rank points by their own coordinates rather than by the
// kNN graph's expanded form |q|^2 + |x|^2 - 2 q.x (self_supervised.cu, flow_propagate.cu, laplacian.cu), and the sorted
// k-best list of the k-nearest searches.
#pragma once
#include "common.cuh"

namespace pvraft {

// the squared length of the fp32 difference q - p, (dx*dx + dy*dy) + dz*dz rounded to nearest at every step, with no FMA
// contraction
__device__ __forceinline__ float diff_sq(float qx, float qy, float qz, const float4& p) {
    const float dx = __fsub_rn(qx, p.x), dy = __fsub_rn(qy, p.y), dz = __fsub_rn(qz, p.z);
    return __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
}

// insert (d, j) into the ascending list best / arg of length K; the caller has checked d < best[K - 1].  Candidates that
// arrive in ascending index order keep the list ordered on (distance, index).
template <int K>
__device__ __forceinline__ void kbest_insert(float (&best)[K], int (&arg)[K], float d, int j) {
#pragma unroll
    for (int i = K - 1; i > 0; --i) {
        if (best[i - 1] > d) {
            best[i] = best[i - 1];
            arg[i] = arg[i - 1];
        } else if (best[i] > d) {
            best[i] = d;
            arg[i] = j;
        }
    }
    if (best[0] > d) {
        best[0] = d;
        arg[0] = j;
    }
}

}  // namespace pvraft
