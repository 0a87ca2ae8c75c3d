// Point-to-plane ICP of rigid fits against the second scan, every segment of every sample in one launch sequence, with no
// host synchronisation (the rule is stated in include/pvraft_b200.h, pvraft_rigid_refine_fwd):
//
//   k_rf_stage     a target takes part when target_mask allows it and its coordinates are finite (takes_part): staged as
//                  it is, any other point as NaN, so the index's bounds ignore it and no distance to it compares <= r2
//   (index)        grid_index_build on the staged targets
//   k_rf_normals   one warp per target: its k_normal nearest targets (grid_knn_diff, on (diff_sq, id)), their covariance
//                  about their mean in double, the eigenvector of its smallest eigenvalue (cyclic Jacobi); a target whose
//                  normal is not valid is staged as NaN in place (each warp writes its own target only)
//   (index)        grid_index_build again, over the targets with a valid normal: the only ones a source point can match
//   (grouping)     O > 1 only: rm_group (rigid_segments.cuh), the moment windows of each segment (with O = 1 window c
//                  of a sample is its item c, and membership is labels == 0)
//   k_rf_members   over the windows: (n, sum x) of the members, then sum |x - c_x|^2 about their centroid (k_rf_setup)
//   per iteration  k_icp_step (the hot path: move, exact fixed-radius nearest search, the 6x6 point-to-plane normal
//                  equations summed per window) and k_icp_solve (one thread per segment: the degeneracy-aware solve)
//   k_rf_write     the refined R and t, and what the last iteration saw
#include "grid_index.cuh"
#include "rigid_segments.cuh"

namespace pvraft {

constexpr int kRfMaxIterations = 64;
constexpr int kRfMinK = 3, kRfMaxK = 32;
constexpr double kNormalKappa = 0.25;   // a normal is valid when lambda0 < kNormalKappa lambda1
constexpr double kRankTol = 1e-4;       // an eigen-direction of the scaled system is solved for when lambda > kRankTol lambda_max
constexpr double kConvergedStep = 1e-6; // metres: rho |omega| + |dt| at or below it ends a segment's iterations
constexpr int kRfMinMatches = 6;
constexpr int kRfMom = 29;              // per segment and iteration: upper JtJ (21, row-major), Jt r (6), count, sum r^2
constexpr int kRfMemb = 5;              // per segment: n, sum x (3), sum |x - c_x|^2
constexpr int kRfState = 21;            // doubles per segment: R (9), c_y (3), c_x (3), rho, steps, done, rank, matched, sse
constexpr int kRfHist = 12;             // R (9), c_y (3)
constexpr int kRfNormalWarps = 8;

__global__ void __launch_bounds__(256) k_rf_stage(const float* __restrict__ xyz2, const uint8_t* __restrict__ mask, long long points,
                                                  float* __restrict__ staged) {
    const long long p = (long long)blockIdx.x * 256 + threadIdx.x;
    if (p >= points) return;
    const float x = xyz2[3 * p], y = xyz2[3 * p + 1], z = xyz2[3 * p + 2];
    const bool on = takes_part(mask, p, x, y, z);
    staged[3 * p] = on ? x : NAN;
    staged[3 * p + 1] = on ? y : NAN;
    staged[3 * p + 2] = on ? z : NAN;
}

// One warp per target (kRfNormalWarps per CTA): normals [B,M] float4 (n, 1) when valid, (0, 0, 0, 0) otherwise, also into
// normals_out when given; nbr_out [B,M,k] (when given) the neighbour ids, nearest first, -1 for a slot no target filled or
// a point that is no target; staged[target] becomes NaN unless the normal is valid.
__global__ void __launch_bounds__(kRfNormalWarps * kWarp) k_rf_normals(const float* __restrict__ xyz2, int M, long long points, int k,
                                                                       GridIndex ix, float* __restrict__ staged, float4* __restrict__ normals,
                                                                       float4* __restrict__ normals_out, int32_t* __restrict__ nbr_out) {
    const long long q = (long long)blockIdx.x * kRfNormalWarps + warp_id();
    if (q >= points) return;
    const int s = (int)(q / M), lane = lane_id();
    const float qx = staged[3 * q], qy = staged[3 * q + 1], qz = staged[3 * q + 2];
    bool valid = false;
    double nv[3] = {0.0, 0.0, 0.0};
    if (qx != qx && nbr_out && lane < k) nbr_out[q * k + lane] = -1;
    if (qx == qx) {   // a target (NaN staged otherwise): uniform over the warp
        const long long base = (long long)s * M;
        float bd;
        int bi;
        grid_knn_diff(ix.pts + base, ix.ids + base, ix.cell_start + (long long)s * (ix.cells + 1), ix.params[s], qx, qy, qz, k, bd, bi);
        const bool full = __shfl_sync(kFull, bi, k - 1) < kGridNone;   // k targets found
        if (nbr_out && lane < k) nbr_out[q * k + lane] = bi < kGridNone ? bi : -1;
        if (full) {
            // differences from the target, exact in double: coordinates of any size do not cancel
            double d[3] = {0.0, 0.0, 0.0};
            if (lane < k) {
                const long long o = (base + bi) * 3;
                d[0] = (double)__ldg(xyz2 + o) - (double)qx;
                d[1] = (double)__ldg(xyz2 + o + 1) - (double)qy;
                d[2] = (double)__ldg(xyz2 + o + 2) - (double)qz;
            }
            double mean[3];
#pragma unroll
            for (int a = 0; a < 3; ++a) mean[a] = warp_sum(d[a]) / (double)k;
            double e[3];
#pragma unroll
            for (int a = 0; a < 3; ++a) e[a] = lane < k ? d[a] - mean[a] : 0.0;
            double C[3][3];
#pragma unroll
            for (int a = 0; a < 3; ++a)
#pragma unroll
                for (int b = a; b < 3; ++b) C[a][b] = C[b][a] = warp_sum(e[a] * e[b]);
            double V[3][3];
            jacobi_sym<3>(C, V);
            const double l0 = C[0][0], l1 = C[1][1], l2 = C[2][2];
            const int lo = l0 <= l1 ? (l0 <= l2 ? 0 : 2) : (l1 <= l2 ? 1 : 2);   // the smallest, lowest index on ties
            const double lmin = lo == 0 ? l0 : (lo == 1 ? l1 : l2);
            const double lmid = lo == 0 ? fmin(l1, l2) : (lo == 1 ? fmin(l0, l2) : fmin(l0, l1));
            valid = lmin < kNormalKappa * lmid;
            const double n0 = V[0][lo], n1 = V[1][lo], n2 = V[2][lo];
            const double nn = sqrt(n0 * n0 + n1 * n1 + n2 * n2);
            nv[0] = n0 / nn;
            nv[1] = n1 / nn;
            nv[2] = n2 / nn;
        }
    }
    if (lane != 0) return;
    const float4 out = valid ? make_float4((float)nv[0], (float)nv[1], (float)nv[2], 1.f) : make_float4(0.f, 0.f, 0.f, 0.f);
    normals[q] = out;
    if (normals_out) normals_out[q] = out;
    if (!valid) staged[3 * q] = staged[3 * q + 1] = staged[3 * q + 2] = NAN;
}

// A source point takes part in segment (s, o) when labels[s, i] == o (every point with labels NULL) and its coordinates are
// finite.  pass 0: (1, x) into acc slots 0..3; pass 1: |x - c_x|^2 into slot 4, c_x from the state.
template <bool DET>
__global__ void __launch_bounds__(kMomThreads) k_rf_members(const float* __restrict__ x, const int32_t* __restrict__ labels,
                                                            const int32_t* __restrict__ items, const int32_t* __restrict__ nitems,
                                                            int per, int N, int pass, const double* __restrict__ state,
                                                            Acc<DET, double> acc) {
    __shared__ double part[kMomThreads / kWarp][kRfMemb];
    const int s = blockIdx.y;
    const int n_items = items ? nitems[s] : 1;
    for (int it = items ? (int)blockIdx.x : 0; it < n_items; it += gridDim.x) {
        const SegItem w = seg_item(items, s, per, N, items ? it : (int)blockIdx.x);
        const int i = w.c * kMomThreads + threadIdx.x;
        double v[kRfMemb] = {0.0, 0.0, 0.0, 0.0, 0.0};
        if (i < N) {
            const long long p = (long long)s * N + i;
            const float x0 = __ldg(x + 3 * p), x1 = __ldg(x + 3 * p + 1), x2 = __ldg(x + 3 * p + 2);
            if ((!labels || labels[p] == w.o) && finite3(x0, x1, x2)) {
                if (pass == 0) {
                    v[0] = 1.0;
                    v[1] = x0;
                    v[2] = x1;
                    v[3] = x2;
                } else {
                    const double* cx = state + (long long)w.g * kRfState + 12;
                    const double d0 = (double)x0 - cx[0], d1 = (double)x1 - cx[1], d2 = (double)x2 - cx[2];
                    v[4] = d0 * d0 + d1 * d1 + d2 * d2;
                }
            }
        }
        window_add<kRfMemb>(v, part, acc, w.g);
    }
}

// the fp32 model of the step kernel from the double state: R, c_x, c_y rounded once; flag 1 while the segment iterates
__device__ __forceinline__ void rf_model(const double* st, bool live, float* m) {
#pragma unroll
    for (int k = 0; k < 9; ++k) m[k] = (float)st[k];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        m[kModelCx + c] = (float)st[12 + c];
        m[kModelCy + c] = (float)st[9 + c];
    }
    m[kModelFlag] = live ? 1.f : 0.f;
}

__device__ __forceinline__ void rf_history(double* hist, int g, int iterations, int k, const double* st) {
    if (!hist) return;
    double* h = hist + ((long long)g * (iterations + 1) + k) * kRfHist;
#pragma unroll
    for (int j = 0; j < kRfHist; ++j) h[j] = st[j];
}

// One thread per segment: c_x from the member sums, c_y = R c_x + t from the input fit, history entry 0 and the model.
template <bool DET>
__global__ void __launch_bounds__(64) k_rf_setup(const double* __restrict__ memb, FxSlots slots, int G, int iterations,
                                                 const float* __restrict__ R_in, const float* __restrict__ t_in, double* __restrict__ state,
                                                 float* __restrict__ model, double* __restrict__ hist) {
    const int g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= G) return;
    const double n = acc_read<DET>(memb, slots, (long long)g * kRfMemb);
    double* st = state + (long long)g * kRfState;
#pragma unroll
    for (int k = 0; k < kRfState; ++k) st[k] = 0.0;
    double cx[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) cx[c] = n > 0.0 ? acc_read<DET>(memb, slots, (long long)g * kRfMemb + 1 + c) / n : 0.0;
#pragma unroll
    for (int k = 0; k < 9; ++k) st[k] = (double)R_in[9ll * g + k];
#pragma unroll
    for (int r = 0; r < 3; ++r) {
        st[9 + r] = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(st[3 * r], cx[0]), __dmul_rn(st[3 * r + 1], cx[1])), __dmul_rn(st[3 * r + 2], cx[2])),
                              (double)t_in[3ll * g + r]);
        st[12 + r] = cx[r];
    }
    rf_history(hist, g, iterations, 0, st);
    rf_model(st, n > 0.0, model + (long long)g * kModel);
}

// The hot path, one iteration over the windows of every live segment.  Per member i with finite x:
//   move    p = R (x - c_x) + c_y in fp32 (p_k = (R (x - c_x))_k + c_y_k, model_rotate, each operation rounded, none
//           contracted), R, c_x, c_y the model's fp32 values;
//   match   the nearest target q of the second index on (diff_sq(p, q), id) with diff_sq <= r2, found by
//           grid_radius_visit (exact for the fp32 predicate; a non-finite p matches nothing) -> corr (id or -1);
//   sum     r = n . (p - q), J = [(p - c_y) x n, n] in double from the fp32 values: upper J J^T (21), J r (6), 1, r^2,
//           summed by window_add into acc [G,kRfMom].
template <bool DET>
__global__ void __launch_bounds__(kMomThreads) k_icp_step(const float* __restrict__ x, const int32_t* __restrict__ labels,
                                                          const int32_t* __restrict__ items, const int32_t* __restrict__ nitems,
                                                          int per, int N, int M, float r2, const float* __restrict__ model, GridIndex ix,
                                                          const float4* __restrict__ normals, int32_t* __restrict__ corr,
                                                          Acc<DET, double> acc) {
    __shared__ double part[kMomThreads / kWarp][kRfMom];
    const int s = blockIdx.y;
    const int n_items = items ? nitems[s] : 1;
    const long long tbase = (long long)s * M;
    const float4* P = ix.pts + tbase;
    const int32_t* I = ix.ids + tbase;
    const int32_t* CS = ix.cell_start + (long long)s * (ix.cells + 1);
    for (int it = items ? (int)blockIdx.x : 0; it < n_items; it += gridDim.x) {
        const SegItem w = seg_item(items, s, per, N, items ? it : (int)blockIdx.x);
        const float* m = model + (long long)w.g * kModel;
        if (m[kModelFlag] == 0.f) continue;   // converged or empty: uniform over the CTA
        const int i = w.c * kMomThreads + threadIdx.x;
        double v[kRfMom];
#pragma unroll
        for (int k = 0; k < kRfMom; ++k) v[k] = 0.0;
        const long long p = (long long)s * N + i;
        float x0 = 0.f, x1 = 0.f, x2 = 0.f;
        bool member = false;
        if (i < N) {
            x0 = __ldg(x + 3 * p), x1 = __ldg(x + 3 * p + 1), x2 = __ldg(x + 3 * p + 2);
            member = !labels || labels[p] == w.o;
        }
        if (member) {
            int best = -1;
            if (finite3(x0, x1, x2)) {
                float q[3];
                model_rotate(m, x0, x1, x2, q);
                const float p0 = __fadd_rn(q[0], m[kModelCy]), p1 = __fadd_rn(q[1], m[kModelCy + 1]), p2 = __fadd_rn(q[2], m[kModelCy + 2]);
                if (finite3(p0, p1, p2)) {
                    float bd = INFINITY;
                    int bk = -1;
                    grid_radius_visit(CS, ix.params[s], p0, p1, p2, r2, [&](int begin, int end) {
                        for (int k = begin; k < end; ++k) {
                            const float d = diff_sq(p0, p1, p2, __ldg(P + k));
                            if (!(d <= r2)) continue;
                            const int id = __ldg(I + k);
                            if (d < bd || (d == bd && id < best)) {
                                bd = d;
                                best = id;
                                bk = k;
                            }
                        }
                    });
                    if (best >= 0) {
                        const float4 q = __ldg(P + bk);
                        const float4 nq = __ldg(normals + tbase + best);
                        const double n[3] = {nq.x, nq.y, nq.z};
                        const double e[3] = {(double)p0 - (double)q.x, (double)p1 - (double)q.y, (double)p2 - (double)q.z};
                        const double a[3] = {(double)p0 - (double)m[kModelCy], (double)p1 - (double)m[kModelCy + 1],
                                             (double)p2 - (double)m[kModelCy + 2]};
                        const double r = n[0] * e[0] + n[1] * e[1] + n[2] * e[2];
                        const double J[6] = {a[1] * n[2] - a[2] * n[1], a[2] * n[0] - a[0] * n[2], a[0] * n[1] - a[1] * n[0], n[0], n[1], n[2]};
                        int u = 0;
#pragma unroll
                        for (int j = 0; j < 6; ++j)
#pragma unroll
                            for (int l = j; l < 6; ++l) v[u++] = J[j] * J[l];
#pragma unroll
                        for (int j = 0; j < 6; ++j) v[21 + j] = J[j] * r;
                        v[27] = 1.0;
                        v[28] = r * r;
                    }
                }
            }
            if (corr) corr[p] = best;
        }
        window_add<kRfMom>(v, part, acc, w.g);
    }
}

// R <- exp([w]x) R (Rodrigues in double: E = I + a K + b K^2, a = sin(th) / th, b = 2 sin^2(th / 2) / th^2, th = |w|)
__device__ __forceinline__ void rf_rotate(double* R, const double (&w)[3]) {
    const double th = sqrt(w[0] * w[0] + w[1] * w[1] + w[2] * w[2]);
    const double a = th > 0.0 ? sin(th) / th : 1.0;
    const double sh = th > 0.0 ? sin(0.5 * th) / th : 0.5;
    const double b = 2.0 * sh * sh;
    const double K[9] = {0.0, -w[2], w[1], w[2], 0.0, -w[0], -w[1], w[0], 0.0};
    double E[9];
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const double k2 = K[3 * r] * K[c] + K[3 * r + 1] * K[3 + c] + K[3 * r + 2] * K[6 + c];
            E[3 * r + c] = (r == c ? 1.0 : 0.0) + a * K[3 * r + c] + b * k2;
        }
    double out[9];
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c) out[3 * r + c] = E[3 * r] * R[c] + E[3 * r + 1] * R[3 + c] + E[3 * r + 2] * R[6 + c];
#pragma unroll
    for (int k = 0; k < 9; ++k) R[k] = out[k];
}

// One thread per segment after iteration `iter`'s sums: with >= kRfMinMatches correspondences, the system scaled by rho
// (rotation unknowns rho w) is decomposed by Jacobi and solved along the eigen-directions with lambda > kRankTol lambda_max;
// R <- exp([w]x) R, c_y <- c_y + dt; the segment stops after a step with rho |w| + |dt| <= kConvergedStep.
template <bool DET>
__global__ void __launch_bounds__(64) k_icp_solve(const double* __restrict__ mom, const double* __restrict__ memb, FxSlots slots,
                                                  FxSlots mslots, int G, int iter, int iterations, double* __restrict__ state,
                                                  float* __restrict__ model, double* __restrict__ hist) {
    const int g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= G) return;
    double* st = state + (long long)g * kRfState;
    float* m = model + (long long)g * kModel;
    if (m[kModelFlag] != 0.f) {
        const long long b0 = (long long)g * kRfMom;
        const double cnt = acc_read<DET>(mom, slots, b0 + 27);
        st[19] = cnt;
        st[20] = acc_read<DET>(mom, slots, b0 + 28);
        st[18] = 0.0;
        if (cnt >= (double)kRfMinMatches) {
            const double n = acc_read<DET>(memb, mslots, (long long)g * kRfMemb);
            double rho = sqrt(acc_read<DET>(memb, mslots, (long long)g * kRfMemb + 4) / n);
            if (!(rho > 0.0)) rho = 1.0;
            st[15] = rho;
            double A[6][6], V[6][6], y[6];
            int u = 0;
#pragma unroll
            for (int j = 0; j < 6; ++j) {
                const double sj = j < 3 ? 1.0 / rho : 1.0;
#pragma unroll
                for (int l = j; l < 6; ++l) {
                    const double sl = l < 3 ? 1.0 / rho : 1.0;
                    A[j][l] = A[l][j] = acc_read<DET>(mom, slots, b0 + u++) * sj * sl;
                }
                y[j] = acc_read<DET>(mom, slots, b0 + 21 + j) * sj;
            }
            jacobi_sym<6>(A, V);
            double lmax = A[0][0];
#pragma unroll
            for (int j = 1; j < 6; ++j) lmax = fmax(lmax, A[j][j]);
            double z[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
            int rank = 0;
#pragma unroll
            for (int j = 0; j < 6; ++j) {
                const double lj = A[j][j];
                if (!(lj > kRankTol * lmax) || !(lj > 0.0)) continue;
                ++rank;
                double c = 0.0;
#pragma unroll
                for (int k = 0; k < 6; ++k) c += V[k][j] * y[k];
                c /= lj;
#pragma unroll
                for (int k = 0; k < 6; ++k) z[k] -= c * V[k][j];
            }
            const double w[3] = {z[0] / rho, z[1] / rho, z[2] / rho};
            rf_rotate(st, w);
#pragma unroll
            for (int c = 0; c < 3; ++c) st[9 + c] += z[3 + c];
            st[16] += 1.0;
            st[18] = rank;
            const double step = sqrt(z[0] * z[0] + z[1] * z[1] + z[2] * z[2]) + sqrt(z[3] * z[3] + z[4] * z[4] + z[5] * z[5]);
            if (step <= kConvergedStep) st[17] = 1.0;
            rf_model(st, st[17] == 0.0, m);
        }
    }
    rf_history(hist, g, iterations, iter + 1, st);
}

// One thread per segment: R, t (t = c_y - R c_x in double; the input's R and t where no step was taken), degenerate =
// input degenerate AND rank < 6, matched, rmse = sqrt(sum r^2 / matched), rank, steps
__global__ void __launch_bounds__(64) k_rf_write(const double* __restrict__ state, int G, const float* __restrict__ R_in,
                                                 const float* __restrict__ t_in, const uint8_t* __restrict__ deg_in, float* __restrict__ R,
                                                 float* __restrict__ t, uint8_t* __restrict__ degenerate, int32_t* __restrict__ matched,
                                                 float* __restrict__ rmse, int32_t* __restrict__ rank, int32_t* __restrict__ steps) {
    const int g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= G) return;
    const double* st = state + (long long)g * kRfState;
    const bool moved = st[16] > 0.0;
#pragma unroll
    for (int k = 0; k < 9; ++k) R[9ll * g + k] = moved ? (float)st[k] : R_in[9ll * g + k];
#pragma unroll
    for (int r = 0; r < 3; ++r) {
        const double rc = __dadd_rn(__dadd_rn(__dmul_rn(st[3 * r], st[12]), __dmul_rn(st[3 * r + 1], st[13])), __dmul_rn(st[3 * r + 2], st[14]));
        t[3ll * g + r] = moved ? (float)__dsub_rn(st[9 + r], rc) : t_in[3ll * g + r];
    }
    const int rk = (int)st[18], cnt = (int)st[19];
    degenerate[g] = deg_in[g] && rk < 6;
    matched[g] = cnt;
    rmse[g] = cnt > 0 ? (float)sqrt(st[20] / (double)cnt) : 0.f;
    rank[g] = rk;
    steps[g] = (int)st[16];
}

// workspace: grid index over M | staged [B,M,3] f32 | normals [B,M] float4 | the grouping (RmGroupWs, O > 1 only) | model [G,16] f32 |
// state [G,kRfState] f64 | memb [G,kRfMemb] f64 | mom [iterations,G,kRfMom] f64, each range 16-byte aligned
struct RefineWs {
    void* index;
    float* staged;
    float4* normals;
    RmGroupWs grp;
    float* model;
    double *state, *memb, *mom;
    int64_t bytes;
};
static RefineWs refine_ws(void* ws, int B, int N, int M, int O, int iterations) {
    ByteCarve w(ws);
    const long long G = (long long)B * O, tm = (long long)B * M;
    RefineWs L;
    L.index = w.take<void>(grid_index_bytes(B, M));
    L.staged = w.take<float>(12 * tm);
    L.normals = w.take<float4>(16 * tm);
    L.grp = O > 1 ? rm_group_carve(w, B, N, O) : RmGroupWs{};
    L.model = w.take<float>(4 * G * kModel);
    L.state = w.take<double>(8 * G * kRfState);
    L.memb = w.take<double>(8 * G * kRfMemb);
    L.mom = w.take<double>(8 * iterations * G * kRfMom);
    L.bytes = w.bytes;
    return L;
}

static bool bad_sizes(int B, int N, int M, int O, int iterations) {
    return B < 1 || N < 1 || M < 1 || O < 1 || O > kMaxObjects || iterations < 1 || iterations > kRfMaxIterations ||
           (long long)B * N > 0x7fffffffll || (long long)B * M > 0x7fffffffll || (long long)B * O > 65535;
}

}  // namespace pvraft

using namespace pvraft;

extern "C" int64_t pvraft_rigid_refine_workspace_bytes(int B, int N, int M, int O, int iterations) {
    return bad_sizes(B, N, M, O, iterations) ? 0 : refine_ws(nullptr, B, N, M, O, iterations).bytes;
}

extern "C" int64_t pvraft_rigid_refine_det_workspace_bytes(int B, int O, int iterations) {
    return B < 1 || O < 1 || O > kMaxObjects || iterations < 1 || iterations > kRfMaxIterations || (long long)B * O > 65535
               ? 0
               : fx_bytes((long long)B * O * (kRfMemb + (long long)iterations * kRfMom));
}

extern "C" int pvraft_rigid_refine_fwd(const float* xyz1, const float* xyz2, const int32_t* labels, const uint8_t* target_mask,
                                       const float* R_in, const float* t_in, const uint8_t* degenerate_in, int B, int N, int M, int O,
                                       int iterations, float max_distance, int k_normal, float* R, float* t, uint8_t* degenerate,
                                       int32_t* matched, float* rmse, int32_t* rank, int32_t* steps, double* history, int32_t* corr,
                                       float* normals, int32_t* neighbours, void* workspace, void* det_workspace, void* stream) {
    if (!xyz1 || !xyz2 || (!labels && O != 1) || !R_in || !t_in || !degenerate_in || !R || !t || !degenerate || !matched || !rmse ||
        !rank || !steps || !workspace || bad_sizes(B, N, M, O, iterations) || !(max_distance > 0.f) || isinf(max_distance) ||
        isinf(max_distance * max_distance) || k_normal < kRfMinK || k_normal > kRfMaxK || k_normal > M)
        return fail(PVRAFT_ERR_BAD_ARG, "rigid_refine_fwd: bad argument");
    if (reinterpret_cast<uintptr_t>(workspace) & 15) return fail(PVRAFT_ERR_BAD_ARG, "rigid_refine_fwd: workspace not 16-byte aligned");
    cudaStream_t st = (cudaStream_t)stream;
    const RefineWs L = refine_ws(workspace, B, N, M, O, iterations);
    const int G = B * O;
    const long long tpts = (long long)B * M;
    const float r2 = max_distance * max_distance;
    int rc;
    cudaError_t e = cudaSuccess;
    if (!det_workspace) {   // memb | mom, the whole carved span (the 16-byte padding between the ranges included)
        const char* end = reinterpret_cast<const char*>(L.mom + (size_t)iterations * G * kRfMom);
        e = cudaMemsetAsync(L.memb, 0, (size_t)(end - reinterpret_cast<const char*>(L.memb)), st);
    }
    if (e == cudaSuccess && corr) e = cudaMemsetAsync(corr, 0xff, 4 * (size_t)B * N, st);   // -1 off the members
    if (e != cudaSuccess) return fail((int)e, "rigid_refine_fwd: memset failed: %s", cudaGetErrorString(e));
    // the targets, their normals, and the index of the targets with a valid normal
    k_rf_stage<<<(unsigned)((tpts + 255) / 256), 256, 0, st>>>(xyz2, target_mask, tpts, L.staged);
    if ((rc = check_launch("rigid_refine_fwd stage"))) return rc;
    GridIndex ix;
    if ((rc = grid_index_build(L.staged, nullptr, B, M, L.index, st, &ix))) return rc;
    k_rf_normals<<<(unsigned)((tpts + kRfNormalWarps - 1) / kRfNormalWarps), kRfNormalWarps * kWarp, 0, st>>>(
        xyz2, M, tpts, k_normal, ix, L.staged, L.normals, reinterpret_cast<float4*>(normals), neighbours);
    if ((rc = check_launch("rigid_refine_fwd normals"))) return rc;
    if ((rc = grid_index_build(L.staged, nullptr, B, M, L.index, st, &ix))) return rc;
    // the segments: with O = 1 window c of sample s is item c and membership is read from labels, so only O > 1 groups
    if (O > 1 && (rc = rm_group(labels, B, N, O, L.grp, st))) return rc;
    const int32_t* items = O > 1 ? L.grp.mitems : nullptr;
    const int32_t* nitems = O > 1 ? L.grp.nm : nullptr;
    const int windows = (N + kMomThreads - 1) / kMomThreads;   // with O > 1 the items cover them, plus one per segment
    const dim3 wgrid((unsigned)(windows + (O > 1 ? O : 0)), (unsigned)B);
    const unsigned sblocks = (unsigned)((G + 63) / 64);
    const FxSlots mslots = det_workspace ? fx_slots(det_workspace) : FxSlots{};
    if (det_workspace) {
        k_rf_members<true><<<wgrid, kMomThreads, 0, st>>>(xyz1, labels, items, nitems, O, N, 0, L.state, mslots);
        k_rf_setup<true><<<sblocks, 64, 0, st>>>(L.memb, mslots, G, iterations, R_in, t_in, L.state, L.model, history);
        k_rf_members<true><<<wgrid, kMomThreads, 0, st>>>(xyz1, labels, items, nitems, O, N, 1, L.state, mslots);
    } else {
        k_rf_members<false><<<wgrid, kMomThreads, 0, st>>>(xyz1, labels, items, nitems, O, N, 0, L.state, L.memb);
        k_rf_setup<false><<<sblocks, 64, 0, st>>>(L.memb, FxSlots{}, G, iterations, R_in, t_in, L.state, L.model, history);
        k_rf_members<false><<<wgrid, kMomThreads, 0, st>>>(xyz1, labels, items, nitems, O, N, 1, L.state, L.memb);
    }
    for (int k = 0; k < iterations; ++k) {
        double* mom = L.mom + (long long)k * G * kRfMom;
        if (det_workspace) {
            const FxSlots slots = mslots + (long long)G * kRfMemb + (long long)k * G * kRfMom;
            k_icp_step<true><<<wgrid, kMomThreads, 0, st>>>(xyz1, labels, items, nitems, O, N, M, r2, L.model, ix, L.normals, corr, slots);
            k_icp_solve<true><<<sblocks, 64, 0, st>>>(mom, L.memb, slots, mslots, G, k, iterations, L.state, L.model, history);
        } else {
            k_icp_step<false><<<wgrid, kMomThreads, 0, st>>>(xyz1, labels, items, nitems, O, N, M, r2, L.model, ix, L.normals, corr, mom);
            k_icp_solve<false><<<sblocks, 64, 0, st>>>(mom, L.memb, FxSlots{}, FxSlots{}, G, k, iterations, L.state, L.model, history);
        }
    }
    k_rf_write<<<sblocks, 64, 0, st>>>(L.state, G, R_in, t_in, degenerate_in, R, t, degenerate, matched, rmse, rank, steps);
    return check_launch("rigid_refine_fwd");
}
