// The inverse-squared-distance interpolation of a field on the searched cloud at a query point, and its backward, shared by
// the Laplacian term (laplacian.cu: the field is P2's Laplacian) and the forward-backward consistency term
// (flow_consistency.cu: the field is the reverse flow).
//
//   Fhat = sum_r w_r F[j_r] / sum_r w_r,  w_r = 1 / (d_r + 1e-8),  d_r the squared distance of the r-th nearest, nearest first
//
// Backward, for the upstream gradient e of Fhat, with the neighbours held fixed:
//   dFhat/dF[j_m] = w_m / sum w, and dFhat/dd_m = -(w_m^2 / sum w) (F_m - Fhat) = -(w_m / sum w)^2 sum_r w_r (F_m - F_r).
//   Evaluating F_m - Fhat as that weighted sum of differences keeps it accurate when one weight dominates (a duplicated
//   point: d = 0, w = 1e8), where Fhat and F_m agree to nearly every bit and their difference, multiplied by
//   w_m^2 / sum w ~ 1e8, would be rounding noise.  dd_m/dq = 2 (q - P_m) = -dd_m/dP_m.
#pragma once
#include "fixed_point.cuh"

namespace pvraft {

constexpr int kIdwMaxK = 8;                            // interpolation neighbours at most

// From the K nearest (nd, nx) of a query, nearest first, among M points: write their ids to nn_row (an unfilled slot, only
// possible when non-finite coordinates leave fewer than K comparable points, contributes nothing and reads back as -1) and
// return the weighted sums (sum w F.x, sum w F.y, sum w F.z, sum w) of the field f, in fp32 nearest first.  Fhat is the
// first three over the fourth.
template <int K>
__device__ __forceinline__ float4 idw_sums(const float (&nd)[K], const int (&nx)[K], const float* f, int M, int32_t* nn_row) {
    float sw = 0.f, sx = 0.f, sy = 0.f, sz = 0.f;
#pragma unroll
    for (int r = 0; r < K; ++r) {
        const int j = nx[r];
        const bool ok = j < M;
        nn_row[r] = ok ? j : -1;
        if (!ok) continue;
        const float wr = __fdiv_rn(1.f, __fadd_rn(nd[r], 1e-8f));
        sx = __fadd_rn(sx, __fmul_rn(wr, __ldg(f + 3ll * j)));
        sy = __fadd_rn(sy, __fmul_rn(wr, __ldg(f + 3ll * j + 1)));
        sz = __fadd_rn(sz, __fmul_rn(wr, __ldg(f + 3ll * j + 2)));
        sw = __fadd_rn(sw, wr);
    }
    return make_float4(sx, sy, sz, sw);
}

// The backward of Fhat at the query q = (qx, qy, qz) for its upstream gradient e.  The neighbours are the k (<= kIdwMaxK)
// slots of row `row` of nn_idx, -1 for none.  Neighbour j is row pb M + j of the searched cloud p and row fb M + j of the field
// f (pb, fb: their sample).  (ox, oy, oz) += the gradient of q (the distance terms); d_p -= it at each neighbour's row of p
// (skipped when d_p is null); d_f += (w_r / sum w) e at its row of f (skipped when null).
template <bool DET>
__device__ __forceinline__ void idw_bwd(float qx, float qy, float qz, const float* p, const float* f, const int32_t* nn_idx, long long row,
                                        int k, int pb, int fb, int M, float ex, float ey, float ez, float& ox, float& oy, float& oz,
                                        Acc<DET> d_p, Acc<DET> d_f) {
    int jj[kIdwMaxK];
    float wt[kIdwMaxK], dx[kIdwMaxK], dy[kIdwMaxK], dz[kIdwMaxK], lx[kIdwMaxK], ly[kIdwMaxK], lz[kIdwMaxK];
    float sw = 0.f;
#pragma unroll
    for (int r = 0; r < kIdwMaxK; ++r) {
        jj[r] = r < k ? __ldg(nn_idx + row * k + r) : -1;
        wt[r] = dx[r] = dy[r] = dz[r] = lx[r] = ly[r] = lz[r] = 0.f;
        if (jj[r] < 0) continue;
        const long long m = 3 * ((long long)pb * M + jj[r]), mf = 3 * ((long long)fb * M + jj[r]);
        dx[r] = __fsub_rn(qx, __ldg(p + m));
        dy[r] = __fsub_rn(qy, __ldg(p + m + 1));
        dz[r] = __fsub_rn(qz, __ldg(p + m + 2));
        lx[r] = __ldg(f + mf);
        ly[r] = __ldg(f + mf + 1);
        lz[r] = __ldg(f + mf + 2);
        const float d = __fadd_rn(__fadd_rn(__fmul_rn(dx[r], dx[r]), __fmul_rn(dy[r], dy[r])), __fmul_rn(dz[r], dz[r]));
        wt[r] = __fdiv_rn(1.f, __fadd_rn(d, 1e-8f));   // the forward's weight, bit for bit
        sw = __fadd_rn(sw, wt[r]);
    }
#pragma unroll
    for (int m = 0; m < kIdwMaxK; ++m) {
        if (jj[m] < 0) continue;
        float tx = 0.f, ty = 0.f, tz = 0.f;   // sum_r w_r (F_m - F_r) = sum w (F_m - Fhat)
#pragma unroll
        for (int r = 0; r < kIdwMaxK; ++r) {
            tx += wt[r] * (lx[m] - lx[r]);
            ty += wt[r] * (ly[m] - ly[r]);
            tz += wt[r] * (lz[m] - lz[r]);
        }
        const float om = __fdiv_rn(wt[m], sw);
        const float gd = -2.f * om * om * ((ex * tx + ey * ty) + ez * tz);   // d/dd_m times dd_m/d(q - P_m) = 2 (q - P_m)
        const float vx = gd * dx[m], vy = gd * dy[m], vz = gd * dz[m];
        ox += vx;
        oy += vy;
        oz += vz;
        const long long r = 3 * ((long long)pb * M + jj[m]), rf = 3 * ((long long)fb * M + jj[m]);
        if (d_p) {
            add(d_p, r, -vx);
            add(d_p, r + 1, -vy);
            add(d_p, r + 2, -vz);
        }
        if (d_f) {
            add(d_f, rf, om * ex);
            add(d_f, rf + 1, om * ey);
            add(d_f, rf + 2, om * ez);
        }
    }
}

}  // namespace pvraft
