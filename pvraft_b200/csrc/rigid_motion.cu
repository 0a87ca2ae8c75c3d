// A robust rigid fit of a scene flow (the sensor's ego-motion, and which points move with it): RANSAC over minimal samples
// with a Horn/Kabsch refit, forward and backward, with no host synchronisation.  y = x + f is formed in fp32 (one rounded add
// per coordinate) everywhere below.
//
//   sampling   hypothesis h draws r = 0, 1, 2: j_r = splitmix64((seed << 32) | (h << 2) | r) mod n_allowed, an index into the
//              segment's ascending member list (the identity without labels).  The key leaves out the sample and the
//              segment, so a segment's result does not depend on the rest of the batch.  A triple is rejected, never
//              redrawn (triple_rejected, in double, every operation rounded and none contracted).
//   minimal    Horn's closed form about the triple's own centroids (horn_fit: the top eigenvector of the 4x4 N(S) by cyclic
//              Jacobi sweeps in double), stored as (R, c_x, c_y) in fp32; the residual is R (x - c_x) - (y - c_y) (residual2).
//   score      k_rigid_score: every (hypothesis, member) pair, ||residual||^2 <= threshold^2 in fp32, counted with
//              ballots into integers, so the counts and the selection (k_rigid_select: most inliers, lowest h on ties) are
//              the same bits in any mode.
//   refit      `rounds` times: k_rigid_moments takes (count, sum dx, sum dy, sum dx dy^T) in double about the current
//              model's (c_x, c_y) over the members within the threshold of it (DET: fixed-point slots), and
//              k_rigid_solve (one thread per segment) runs the same Horn solve; its (R, x-bar, y-bar) is the next round's model.
//   degenerate count < 3, or an eigen-gap lambda0 - lambda1 <= kGapTol lambda0: R = I, t = y-bar - x-bar.  A sample none of
//              whose hypotheses is accepted takes every allowed point as its inliers in every round and is degenerate.
//
// A fit is O SEGMENTS per sample: segment (b, o) is the points with labels[b, i] == o, or, with labels NULL (O = 1), every
// point of the sample.  rigid_motion is O = 1 (labels = where(mask, 0, -1), or NULL without a mask), rigid_objects one
// segment per object.  The grouping (k_rigid_allowed for O = 1, k_ro_group_* otherwise) gives both the same RmSegs, and
// every kernel after it has one form.
//
// Backward (k_rigid_bwd, one thread per point, each gradient written once): the inlier set held fixed, from the per-segment
// double state the forward saves (eigenvectors, eigenvalues, centroids, count):
//   dt -> d y-bar += dt, d x-bar -= R^T dt, dR -= dt x-bar^T;  dR -> dq through R(q);  dq -> dN = sym(sum_{j>=1} v_j v_j^T dq
//   v_0^T / (lambda0 - lambda_j));  dN -> dS;  dx_i = dS (y_i - y-bar) + d x-bar / n, dy_i = dS^T (x_i - x-bar) + d y-bar / n.
#include "fixed_point.cuh"

namespace pvraft {

constexpr int kRmState = 32;          // doubles per segment in the saved state
constexpr int kRmModel = 16;          // floats per model: R (9, row-major), c_x (3), c_y (3), flag
constexpr int kRmMoments = 16;        // n, sum dx (3), sum dy (3), sum dx dy^T (9, row-major)
constexpr int kRmMaxH = 4096;
constexpr int kRmMaxRounds = 8;
constexpr double kCollinearTol = 1e-6;
constexpr double kGapTol = 1e-5;
constexpr int kJacobiSweeps = 12;

__host__ __device__ __forceinline__ unsigned long long splitmix64(unsigned long long z) {
    z += 0x9e3779b97f4a7c15ull;
    z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
    z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
    return z ^ (z >> 31);
}

// Horn's N(S) for S = sum (x_i - x-bar)(y_i - y-bar)^T (row-major): its top unit eigenvector q gives the rotation R(q) that
// maximises sum (y_i - y-bar) . R (x_i - x-bar).
__device__ __forceinline__ void horn_matrix(const double (&S)[9], double (&a)[4][4]) {
    const double xx = S[0], xy = S[1], xz = S[2], yx = S[3], yy = S[4], yz = S[5], zx = S[6], zy = S[7], zz = S[8];
    a[0][0] = xx + yy + zz;
    a[1][1] = xx - yy - zz;
    a[2][2] = -xx + yy - zz;
    a[3][3] = -xx - yy + zz;
    a[0][1] = a[1][0] = yz - zy;
    a[0][2] = a[2][0] = zx - xz;
    a[0][3] = a[3][0] = xy - yx;
    a[1][2] = a[2][1] = xy + yx;
    a[1][3] = a[3][1] = zx + xz;
    a[2][3] = a[3][2] = yz + zy;
}

// Cyclic Jacobi on a symmetric 4x4 matrix: a becomes diagonal (the eigenvalues), column j of v the eigenvector of a[j][j].
__device__ __forceinline__ void jacobi4(double (&a)[4][4], double (&v)[4][4]) {
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) v[i][j] = i == j ? 1.0 : 0.0;
    for (int sweep = 0; sweep < kJacobiSweeps; ++sweep) {
        const double off = fabs(a[0][1]) + fabs(a[0][2]) + fabs(a[0][3]) + fabs(a[1][2]) + fabs(a[1][3]) + fabs(a[2][3]);
        if (off == 0.0) break;
#pragma unroll
        for (int p = 0; p < 3; ++p)
#pragma unroll
            for (int q = p + 1; q < 4; ++q) {
                const double apq = a[p][q];
                if (apq == 0.0) continue;
                const double theta = (a[q][q] - a[p][p]) / (2.0 * apq);
                const double t = fabs(theta) > 1e150 ? 0.5 / theta : copysign(1.0, theta) / (fabs(theta) + sqrt(theta * theta + 1.0));
                const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
                a[p][p] -= t * apq;
                a[q][q] += t * apq;
                a[p][q] = a[q][p] = 0.0;
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    if (k != p && k != q) {
                        const double akp = a[k][p], akq = a[k][q];
                        a[k][p] = a[p][k] = c * akp - s * akq;
                        a[k][q] = a[q][k] = s * akp + c * akq;
                    }
                    const double vkp = v[k][p], vkq = v[k][q];
                    v[k][p] = c * vkp - s * vkq;
                    v[k][q] = s * vkp + c * vkq;
                }
            }
    }
}

__device__ __forceinline__ void quat_rot(const double (&q)[4], double (&R)[9]) {
    const double w = q[0], x = q[1], y = q[2], z = q[3];
    R[0] = w * w + x * x - y * y - z * z;
    R[1] = 2.0 * (x * y - w * z);
    R[2] = 2.0 * (x * z + w * y);
    R[3] = 2.0 * (x * y + w * z);
    R[4] = w * w - x * x + y * y - z * z;
    R[5] = 2.0 * (y * z - w * x);
    R[6] = 2.0 * (x * z - w * y);
    R[7] = 2.0 * (y * z + w * x);
    R[8] = w * w - x * x - y * y + z * z;
}

// The solve: S -> the eigen-decomposition of N(S), ordered so that column 0 of V and lam[0] are the top pair, and R(q) for
// q = column 0 (normalised).  Returns true when the fit is proper: lam[0] - (the next largest) > kGapTol lam[0].
__device__ __forceinline__ bool horn_fit(const double (&S)[9], double (&V)[4][4], double (&lam)[4], double (&R)[9]) {
    double a[4][4];
    horn_matrix(S, a);
    jacobi4(a, V);
    double l[4] = {a[0][0], a[1][1], a[2][2], a[3][3]};
    int top = 0;
    double lmax = l[0];
#pragma unroll
    for (int j = 1; j < 4; ++j)
        if (l[j] > lmax) {
            lmax = l[j];
            top = j;
        }
    // swap the top pair into slot 0 (a permutation of columns; the others keep their order)
#pragma unroll
    for (int j = 1; j < 4; ++j)
        if (j == top) {
            const double t = l[0]; l[0] = l[j]; l[j] = t;
#pragma unroll
            for (int k = 0; k < 4; ++k) { const double u = V[k][0]; V[k][0] = V[k][j]; V[k][j] = u; }
        }
    double second = l[1];
#pragma unroll
    for (int j = 2; j < 4; ++j) second = fmax(second, l[j]);
    double q[4] = {V[0][0], V[1][0], V[2][0], V[3][0]};
    const double qn = sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
#pragma unroll
    for (int k = 0; k < 4; ++k) q[k] /= qn;
    quat_rot(q, R);
#pragma unroll
    for (int j = 0; j < 4; ++j) lam[j] = l[j];
    return l[0] - second > kGapTol * l[0];
}

// ||R (x - c_x) - (y - c_y)||^2 in fp32: d = x - c_x, e = y - c_y; r_k = ((R_k0 d_0 + R_k1 d_1) + R_k2 d_2) - e_k;
// (r_0^2 + r_1^2) + r_2^2; every operation rounded to nearest, none contracted
__device__ __forceinline__ float residual2(const float* m, float x0, float x1, float x2, float y0, float y1, float y2) {
    const float d0 = __fsub_rn(x0, m[9]), d1 = __fsub_rn(x1, m[10]), d2 = __fsub_rn(x2, m[11]);
    const float e0 = __fsub_rn(y0, m[12]), e1 = __fsub_rn(y1, m[13]), e2 = __fsub_rn(y2, m[14]);
    const float r0 = __fsub_rn(__fadd_rn(__fadd_rn(__fmul_rn(m[0], d0), __fmul_rn(m[1], d1)), __fmul_rn(m[2], d2)), e0);
    const float r1 = __fsub_rn(__fadd_rn(__fadd_rn(__fmul_rn(m[3], d0), __fmul_rn(m[4], d1)), __fmul_rn(m[5], d2)), e1);
    const float r2 = __fsub_rn(__fadd_rn(__fadd_rn(__fmul_rn(m[6], d0), __fmul_rn(m[7], d1)), __fmul_rn(m[8], d2)), e2);
    return __fadd_rn(__fadd_rn(__fmul_rn(r0, r0), __fmul_rn(r1, r1)), __fmul_rn(r2, r2));
}

__device__ __forceinline__ double dot3(double a0, double a1, double a2, double b0, double b1, double b2) {
    return __dadd_rn(__dadd_rn(__dmul_rn(a0, b0), __dmul_rn(a1, b1)), __dmul_rn(a2, b2));
}

// The rejection tests of a triple with distinct indices (x, y [3][3] as doubles of the fp32 values): near-collinear unless
// |a x b|^2 > 1e-6 |a|^2 |b|^2 (a = x1 - x0, b = x2 - x0), or a pairwise distance (0-1, 0-2, 1-2) that changes by more than
// 2 threshold between x and y; in double, each operation rounded, none contracted
__device__ __forceinline__ bool triple_rejected(const double (&x)[3][3], const double (&y)[3][3], double thr) {
    const double a0 = __dsub_rn(x[1][0], x[0][0]), a1 = __dsub_rn(x[1][1], x[0][1]), a2 = __dsub_rn(x[1][2], x[0][2]);
    const double b0 = __dsub_rn(x[2][0], x[0][0]), b1 = __dsub_rn(x[2][1], x[0][1]), b2 = __dsub_rn(x[2][2], x[0][2]);
    const double c0 = __dsub_rn(__dmul_rn(a1, b2), __dmul_rn(a2, b1));
    const double c1 = __dsub_rn(__dmul_rn(a2, b0), __dmul_rn(a0, b2));
    const double c2 = __dsub_rn(__dmul_rn(a0, b1), __dmul_rn(a1, b0));
    if (!(dot3(c0, c1, c2, c0, c1, c2) > __dmul_rn(__dmul_rn(kCollinearTol, dot3(a0, a1, a2, a0, a1, a2)), dot3(b0, b1, b2, b0, b1, b2))))
        return true;
    const int P[3][2] = {{0, 1}, {0, 2}, {1, 2}};
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const int i = P[k][0], j = P[k][1];
        const double u0 = __dsub_rn(x[i][0], x[j][0]), u1 = __dsub_rn(x[i][1], x[j][1]), u2 = __dsub_rn(x[i][2], x[j][2]);
        const double w0 = __dsub_rn(y[i][0], y[j][0]), w1 = __dsub_rn(y[i][1], y[j][1]), w2 = __dsub_rn(y[i][2], y[j][2]);
        const double dx = __dsqrt_rn(dot3(u0, u1, u2, u0, u1, u2)), dy = __dsqrt_rn(dot3(w0, w1, w2, w0, w1, w2));
        if (!(fabs(__dsub_rn(dx, dy)) <= __dmul_rn(2.0, thr))) return true;
    }
    return false;
}

// The O = 1 grouping: the members (labels == 0) of each sample in ascending order -> list [B,N] (the first n[s] entries of
// row s), one CTA of kRmScan threads per sample
constexpr int kRmScan = 1024;
__global__ void __launch_bounds__(kRmScan) k_rigid_allowed(const int32_t* __restrict__ labels, int N, int32_t* __restrict__ list,
                                                           int32_t* __restrict__ nmem) {
    __shared__ int warp_tot[kRmScan / kWarp];
    __shared__ int base_sh;
    const int s = blockIdx.x, lane = lane_id(), wid = warp_id();
    const int32_t* l = labels + (long long)s * N;
    int32_t* out = list + (long long)s * N;
    if (threadIdx.x == 0) base_sh = 0;
    for (int c0 = 0; c0 < N; c0 += kRmScan) {
        const int i = c0 + threadIdx.x;
        const bool on = i < N && l[i] == 0;
        const unsigned bal = __ballot_sync(kFull, on);
        __syncthreads();   // base_sh of the previous chunk is final; warp_tot free
        if (lane == 0) warp_tot[wid] = __popc(bal);
        __syncthreads();
        int before = base_sh;
        for (int w = 0; w < wid; ++w) before += warp_tot[w];
        if (on) out[before + __popc(bal & ((1u << lane) - 1u))] = i;
        __syncthreads();
        if (threadIdx.x == 0) {
            int tot = 0;
            for (int w = 0; w < kRmScan / kWarp; ++w) tot += warp_tot[w];
            base_sh += tot;
        }
    }
    __syncthreads();
    if (threadIdx.x == 0) nmem[s] = base_sh;
}

// The segments of one fit: segment g is a subset of sample g / per, and its members, ascending, are list[first(g), first(g) +
// count(g)), first(g) = start[g] (g N with start NULL: k_rigid_allowed) -- or, with list NULL (no labels), all N points of
// the sample.
struct RmSegs {
    const int32_t* list;    // [B,N] member ids, or NULL
    const int32_t* start;   // [G] offset of each segment's members in list, or NULL
    const int32_t* n;       // [G] member counts (read with list only)
    int N, per;
    __device__ __forceinline__ int count(int g) const { return list ? n[g] : N; }
    __device__ __forceinline__ long long first(int g) const { return start ? (long long)start[g] : (long long)g * N; }
    __device__ __forceinline__ int member(int g, long long j) const { return list ? __ldg(list + first(g) + j) : (int)j; }
};

// One thread per (segment, hypothesis): draw, test and fit the triple -> hyp [G,H,kRmModel] (flag 1: accepted, 0: rejected),
// hcnt [G,H] zeroed, triples [G,H,3] (or NULL: the drawn point indices, -1 with no member)
__global__ void __launch_bounds__(128) k_rigid_hypotheses(const float* __restrict__ x, const float* __restrict__ f, RmSegs sg, int H,
                                                          unsigned long long seed, float thr, float* __restrict__ hyp,
                                                          int32_t* __restrict__ hcnt, int32_t* __restrict__ triples) {
    const int g = blockIdx.y, h = blockIdx.x * blockDim.x + threadIdx.x;
    if (h >= H) return;
    const int s = g / sg.per, N = sg.N;
    const long long hs = (long long)g * H + h;
    const int n_al = sg.count(g);
    int idx[3];
    unsigned long long j[3];
#pragma unroll
    for (int r = 0; r < 3; ++r) {
        j[r] = n_al > 0 ? splitmix64((seed << 32) | ((unsigned long long)h << 2) | (unsigned long long)r) % (unsigned long long)n_al : 0ull;
        idx[r] = n_al <= 0 ? -1 : sg.member(g, (long long)j[r]);
        if (triples) triples[hs * 3 + r] = idx[r];
    }
    hcnt[hs] = 0;
    float* m = hyp + hs * kRmModel;
    bool rejected = n_al <= 0 || j[0] == j[1] || j[0] == j[2] || j[1] == j[2];
    double xd[3][3], yd[3][3];
    if (!rejected) {
#pragma unroll
        for (int r = 0; r < 3; ++r)
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                const long long o = ((long long)s * N + idx[r]) * 3 + c;
                const float xv = __ldg(x + o);
                xd[r][c] = xv;
                yd[r][c] = __fadd_rn(xv, __ldg(f + o));
            }
        rejected = triple_rejected(xd, yd, (double)thr);
    }
    if (rejected) {
        m[15] = 0.f;
        return;
    }
    double cx[3], cy[3], S[9];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        cx[c] = (xd[0][c] + xd[1][c] + xd[2][c]) / 3.0;
        cy[c] = (yd[0][c] + yd[1][c] + yd[2][c]) / 3.0;
    }
#pragma unroll
    for (int k = 0; k < 3; ++k)
#pragma unroll
        for (int l = 0; l < 3; ++l) {
            double acc = 0.0;
#pragma unroll
            for (int r = 0; r < 3; ++r) acc += (xd[r][k] - cx[k]) * (yd[r][l] - cy[l]);
            S[3 * k + l] = acc;
        }
    double V[4][4], lam[4], R[9];
    horn_fit(S, V, lam, R);
#pragma unroll
    for (int k = 0; k < 9; ++k) m[k] = (float)R[k];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        m[9 + c] = (float)cx[c];
        m[12 + c] = (float)cy[c];
    }
    m[15] = 1.f;
}

// Inlier counts of every (hypothesis, member) pair.  A CTA holds kScHyp hypotheses in shared memory (read as broadcasts) and
// kScPer members per thread in registers; per hypothesis and warp a ballot and a popcount, lane j of each warp keeps
// hypothesis j's count, then one shared and one global integer atomic.  Without `items` (one segment per sample): grid
// (ceil(N / kScPoints), ceil(H / kScHyp), B), CTA x takes members [x kScPoints, (x + 1) kScPoints) of segment s.  With items
// [B,stride] (nitems [B] of them per sample): grid (stride, ceil(H / kScHyp), B), CTA x takes item x = (j << 8) | o --
// members [j kScPoints, (j + 1) kScPoints) of segment (sample, o) -- so the work is the members' number times H.
constexpr int kScThreads = 256, kScPer = 4, kScPoints = kScThreads * kScPer, kScHyp = 32;
__global__ void __launch_bounds__(kScThreads) k_rigid_score(const float* __restrict__ x, const float* __restrict__ f, RmSegs sg,
                                                            const int32_t* __restrict__ items, const int32_t* __restrict__ nitems,
                                                            int stride, int H, float thr2, const float* __restrict__ hyp,
                                                            int32_t* __restrict__ hcnt) {
    __shared__ float sh[kScHyp][kRmModel];
    __shared__ int cnt[kScHyp];
    const int s = blockIdx.z, h0 = blockIdx.y * kScHyp, lane = lane_id(), N = sg.N;
    int g = s, base = blockIdx.x * kScPoints;
    if (items) {
        if ((int)blockIdx.x >= nitems[s]) return;   // uniform over the CTA
        const int w = items[(long long)s * stride + blockIdx.x];
        g = s * sg.per + (w & 255);
        base = (w >> 8) * kScPoints;
    }
    const int n_g = sg.count(g);
    if (base >= n_g) return;   // no member left: uniform over the CTA
    for (int i = threadIdx.x; i < kScHyp * kRmModel; i += kScThreads) {
        const int hh = h0 + i / kRmModel;
        sh[i / kRmModel][i % kRmModel] = hh < H ? __ldg(hyp + ((long long)g * H + h0) * kRmModel + i) : 0.f;
    }
    if (threadIdx.x < kScHyp) cnt[threadIdx.x] = 0;
    float px[kScPer][3], py[kScPer][3];
    bool ok[kScPer];
#pragma unroll
    for (int k = 0; k < kScPer; ++k) {
        const int j = base + k * kScThreads + threadIdx.x;
        const int i = j < n_g ? sg.member(g, j) : 0;
        ok[k] = j < n_g;
        const long long o = ((long long)s * N + i) * 3;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            px[k][c] = ok[k] ? __ldg(x + o + c) : 0.f;
            py[k][c] = ok[k] ? __fadd_rn(px[k][c], __ldg(f + o + c)) : 0.f;
        }
    }
    __syncthreads();
    int mine = 0;
    for (int j = 0; j < kScHyp; ++j) {
        const float* m = sh[j];
        if (m[15] == 0.f) continue;   // rejected or past H: uniform over the CTA
        int c = 0;
#pragma unroll
        for (int k = 0; k < kScPer; ++k)
            c += __popc(__ballot_sync(kFull, ok[k] && residual2(m, px[k][0], px[k][1], px[k][2], py[k][0], py[k][1], py[k][2]) <= thr2));
        if (lane == j) mine += c;
    }
    if (mine) atomicAdd(cnt + lane, mine);
    __syncthreads();
    if (threadIdx.x < kScHyp && h0 + threadIdx.x < H && cnt[threadIdx.x]) atomicAdd(hcnt + (long long)g * H + h0 + threadIdx.x, cnt[threadIdx.x]);
}

// One CTA per segment: the accepted hypothesis with the most inliers (lowest h on ties) -> model [G,kRmModel] (flag 1), or,
// with none accepted, R = I about the first member (flag 0: every member an inlier); hyp_count [G,H] (or NULL: the counts,
// -1 for a rejected hypothesis); the segment's moment accumulators of every round zeroed
constexpr int kSelThreads = 256;
__global__ void __launch_bounds__(kSelThreads) k_rigid_select(const float* __restrict__ x, const float* __restrict__ f, RmSegs sg, int H,
                                                              int B, int rounds, const float* __restrict__ hyp,
                                                              const int32_t* __restrict__ hcnt, float* __restrict__ model,
                                                              double* __restrict__ mom, int32_t* __restrict__ hyp_count) {
    __shared__ long long best_w[kSelThreads / kWarp];
    const int s = blockIdx.x, smp = s / sg.per, N = sg.N;   // s: the segment; B: the number of segments
    long long best = -1;   // (count << 32) | (H - 1 - h): the largest wins
    for (int h = threadIdx.x; h < H; h += kSelThreads) {
        const long long hs = (long long)s * H + h;
        const bool acc = hyp[hs * kRmModel + 15] != 0.f;
        const int c = hcnt[hs];
        if (hyp_count) hyp_count[hs] = acc ? c : -1;
        if (acc) best = max(best, ((long long)c << 32) | (long long)(H - 1 - h));
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) best = max(best, __shfl_xor_sync(kFull, best, o));
    if (lane_id() == 0) best_w[warp_id()] = best;
    for (int i = threadIdx.x; i < rounds * kRmMoments; i += kSelThreads)
        mom[((long long)(i / kRmMoments) * B + s) * kRmMoments + i % kRmMoments] = 0.0;
    __syncthreads();
    if (threadIdx.x != 0) return;
    for (int w = 0; w < kSelThreads / kWarp; ++w) best = max(best, best_w[w]);
    float* m = model + (long long)s * kRmModel;
    if (best >= 0) {
        const int h = H - 1 - (int)(best & 0xffffffffll);
        const float* src = hyp + ((long long)s * H + h) * kRmModel;
        for (int k = 0; k < kRmModel; ++k) m[k] = src[k];
        return;
    }
    const int n_al = sg.count(s);
    const int i0 = n_al <= 0 ? -1 : sg.member(s, 0);
    for (int k = 0; k < 9; ++k) m[k] = k % 4 == 0 ? 1.f : 0.f;
    for (int c = 0; c < 3; ++c) {
        const float xv = i0 < 0 ? 0.f : x[((long long)smp * N + i0) * 3 + c];
        m[9 + c] = xv;
        m[12 + c] = i0 < 0 ? 0.f : __fadd_rn(xv, f[((long long)smp * N + i0) * 3 + c]);
    }
    m[15] = 0.f;
}

// One refit round's moments over windows of kMomThreads consecutive point ids: point i of sample s is an inlier of segment g
// when it is a member and (flag 0, or residual2 under g's model <= thr2); (1, dx, dy, dx dy^T) with dx = x - c_x, dy = y - c_y
// in double summed per warp (xor butterfly), then over the CTA's warps in order, and added once per (window, segment) into
// acc [G,kRmMoments] (DET: fixed-point slots).  Without `items` (one segment per sample): grid (ceil(N / kMomThreads), B),
// membership labels == 0 (every point with labels NULL), inliers [B,N] written for every point.  With items [B,N] (nitems
// [B] per sample; item (c << 8) | o: the window c of point ids [c kMomThreads, (c + 1) kMomThreads), of segment (sample, o),
// membership labels == o): grid (any, B), each CTA taking items x, x + gridDim.x, ...; inliers written for members only.
// A window's partial sum is the same value either way, so in the DET form a segment's moments are those of the one-segment
// launch with labels = where(labels == o, 0, -1).
constexpr int kMomThreads = 256;
template <bool DET>
__global__ void __launch_bounds__(kMomThreads) k_rigid_moments(const float* __restrict__ x, const float* __restrict__ f,
                                                               const int32_t* __restrict__ labels, const int32_t* __restrict__ items,
                                                               const int32_t* __restrict__ nitems, int per, int N, float thr2,
                                                               const float* __restrict__ model, uint8_t* __restrict__ inliers,
                                                               Acc<DET, double> acc) {
    __shared__ double part[kMomThreads / kWarp][kRmMoments];
    const int s = blockIdx.y;
    const int n_items = items ? nitems[s] : 1;
    for (int it = items ? (int)blockIdx.x : 0; it < n_items; it += gridDim.x) {
        int g = s, o = 0, c = blockIdx.x;
        if (items) {
            const int w = items[(long long)s * N + it];
            o = w & 255;
            g = s * per + o;
            c = w >> 8;
        }
        const int i = c * kMomThreads + threadIdx.x;
        const float* m = model + (long long)g * kRmModel;
        double v[kRmMoments];
#pragma unroll
        for (int k = 0; k < kRmMoments; ++k) v[k] = 0.0;
        if (i < N) {
            const long long p = (long long)s * N + i;
            const bool member = !labels || labels[p] == o;
            const float x0 = __ldg(x + 3 * p), x1 = __ldg(x + 3 * p + 1), x2 = __ldg(x + 3 * p + 2);
            const float y0 = __fadd_rn(x0, __ldg(f + 3 * p)), y1 = __fadd_rn(x1, __ldg(f + 3 * p + 1)), y2 = __fadd_rn(x2, __ldg(f + 3 * p + 2));
            const bool in = member && (m[15] == 0.f || residual2(m, x0, x1, x2, y0, y1, y2) <= thr2);
            if (!items || member) inliers[p] = in;
            if (in) {
                const double d[3] = {(double)x0 - (double)m[9], (double)x1 - (double)m[10], (double)x2 - (double)m[11]};
                const double e[3] = {(double)y0 - (double)m[12], (double)y1 - (double)m[13], (double)y2 - (double)m[14]};
                v[0] = 1.0;
#pragma unroll
                for (int k = 0; k < 3; ++k) {
                    v[1 + k] = d[k];
                    v[4 + k] = e[k];
                }
#pragma unroll
                for (int k = 0; k < 3; ++k)
#pragma unroll
                    for (int l = 0; l < 3; ++l) v[7 + 3 * k + l] = d[k] * e[l];
            }
        }
#pragma unroll
        for (int k = 0; k < kRmMoments; ++k) v[k] = warp_sum(v[k]);
        if (lane_id() == 0)
#pragma unroll
            for (int k = 0; k < kRmMoments; ++k) part[warp_id()][k] = v[k];
        __syncthreads();
        if (threadIdx.x < kRmMoments) {
            double t = 0.0;
            for (int w = 0; w < kMomThreads / kWarp; ++w) t += part[w][threadIdx.x];
            if (t != 0.0) add(acc, (long long)g * kRmMoments + threadIdx.x, t);
        }
        __syncthreads();   // part is reused by the next item
    }
}

// One thread per segment: the Horn solve of one round's moments -> R [G,3,3], t [G,3], count [G], degenerate [G], state
// [G,kRmState] and the next round's model.  DET: the moments are read from the fixed-point slots.
template <bool DET>
__global__ void __launch_bounds__(64) k_rigid_solve(const double* __restrict__ mom, FxSlots slots, int B, float* __restrict__ model,
                                                    float* __restrict__ Rout, float* __restrict__ tout, int32_t* __restrict__ count,
                                                    uint8_t* __restrict__ degenerate, double* __restrict__ state) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= B) return;
    double mo[kRmMoments];
#pragma unroll
    for (int k = 0; k < kRmMoments; ++k) {
        const long long i = (long long)s * kRmMoments + k;
        mo[k] = DET ? fx_value(slots.base + i * kFxWords) : mom[i];
    }
    float* m = model + (long long)s * kRmModel;
    const bool sampled = m[15] != 0.f;
    const double n = mo[0];
    double xb[3], yb[3], mdx[3], mdy[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        mdx[c] = n > 0.0 ? mo[1 + c] / n : 0.0;
        mdy[c] = n > 0.0 ? mo[4 + c] / n : 0.0;
        xb[c] = n > 0.0 ? (double)m[9 + c] + mdx[c] : 0.0;
        yb[c] = n > 0.0 ? (double)m[12 + c] + mdy[c] : 0.0;
    }
    double S[9];
#pragma unroll
    for (int k = 0; k < 3; ++k)
#pragma unroll
        for (int l = 0; l < 3; ++l) S[3 * k + l] = mo[7 + 3 * k + l] - n * mdx[k] * mdy[l];
    double V[4][4], lam[4], R[9];
    const bool proper = horn_fit(S, V, lam, R) && n >= 3.0 && sampled;
    if (!proper)
#pragma unroll
        for (int k = 0; k < 9; ++k) R[k] = k % 4 == 0 ? 1.0 : 0.0;
    double* st = state + (long long)s * kRmState;
#pragma unroll
    for (int k = 0; k < 4; ++k)
#pragma unroll
        for (int j = 0; j < 4; ++j) st[4 * j + k] = V[k][j];   // eigenvector j at [4 j, 4 j + 4)
#pragma unroll
    for (int j = 0; j < 4; ++j) st[16 + j] = lam[j];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        st[20 + c] = xb[c];
        st[23 + c] = yb[c];
    }
    st[26] = n;
    st[27] = proper ? 0.0 : 1.0;
    for (int k = 28; k < kRmState; ++k) st[k] = 0.0;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const double t = yb[k] - (R[3 * k] * xb[0] + R[3 * k + 1] * xb[1] + R[3 * k + 2] * xb[2]);
        tout[s * 3 + k] = (float)t;
    }
#pragma unroll
    for (int k = 0; k < 9; ++k) {
        Rout[s * 9 + k] = (float)R[k];
        m[k] = (float)R[k];
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        m[9 + c] = (float)xb[c];
        m[12 + c] = (float)yb[c];
    }
    count[s] = (int32_t)n;
    degenerate[s] = !proper;
}

// One thread per point: d_xyz1 and d_flow [B,N,3], every element written once (zero off the inliers).  The point's segment:
// (sample, labels[p]) with `per` segments per sample, or its sample with labels NULL; the state, dR and dt are per segment.
__global__ void __launch_bounds__(256) k_rigid_bwd(const float* __restrict__ x, const float* __restrict__ f,
                                                   const uint8_t* __restrict__ inliers, const int32_t* __restrict__ labels, int per,
                                                   const double* __restrict__ state, const float* __restrict__ dR,
                                                   const float* __restrict__ dt, int N, long long points, float* __restrict__ d_x,
                                                   float* __restrict__ d_f) {
    for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < points; p += (long long)gridDim.x * blockDim.x) {
        const int lab = labels ? labels[p] : 0;
        const bool in = inliers[p] && lab >= 0 && lab < per;
        const int s = (int)(p / N) * per + (in ? lab : 0);
        const double* st = state + (long long)s * kRmState;
        const double n = st[26];
        double gx[3] = {0.0, 0.0, 0.0}, gy[3] = {0.0, 0.0, 0.0};
        if (in && n > 0.0) {
            const double* xb = st + 20;
            const double* yb = st + 23;
            double g[3];
#pragma unroll
            for (int c = 0; c < 3; ++c) g[c] = (double)__ldg(dt + 3 * s + c);
            double dS[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
            double dxb[3], dyb[3] = {g[0], g[1], g[2]};
            if (st[27] != 0.0) {
#pragma unroll
                for (int c = 0; c < 3; ++c) dxb[c] = -g[c];
            } else {
                const double q[4] = {st[0], st[1], st[2], st[3]};
                double R[9];
                quat_rot(q, R);
                double D[9];
#pragma unroll
                for (int k = 0; k < 3; ++k) {
                    dxb[k] = -(R[k] * g[0] + R[3 + k] * g[1] + R[6 + k] * g[2]);
#pragma unroll
                    for (int l = 0; l < 3; ++l) D[3 * k + l] = (double)__ldg(dR + 9 * s + 3 * k + l) - g[k] * xb[l];
                }
                const double w = q[0], qx = q[1], qy = q[2], qz = q[3];
                const double dq[4] = {
                    2.0 * (w * (D[0] + D[4] + D[8]) + qz * (D[3] - D[1]) + qy * (D[2] - D[6]) + qx * (D[7] - D[5])),
                    2.0 * (qx * (D[0] - D[4] - D[8]) + qy * (D[1] + D[3]) + qz * (D[2] + D[6]) + w * (D[7] - D[5])),
                    2.0 * (qy * (-D[0] + D[4] - D[8]) + qx * (D[1] + D[3]) + qz * (D[5] + D[7]) + w * (D[2] - D[6])),
                    2.0 * (qz * (-D[0] - D[4] + D[8]) + qx * (D[2] + D[6]) + qy * (D[5] + D[7]) + w * (D[3] - D[1]))};
                // X = sum_{j>=1} (v_j . dq) / (lam0 - lam_j) v_j v0^T, G = (X + X^T) / 2
                double X[4][4];
#pragma unroll
                for (int a = 0; a < 4; ++a)
#pragma unroll
                    for (int b = 0; b < 4; ++b) X[a][b] = 0.0;
#pragma unroll
                for (int j = 1; j < 4; ++j) {
                    const double* vj = st + 4 * j;
                    const double c = (vj[0] * dq[0] + vj[1] * dq[1] + vj[2] * dq[2] + vj[3] * dq[3]) / (st[16] - st[16 + j]);
#pragma unroll
                    for (int a = 0; a < 4; ++a)
#pragma unroll
                        for (int b = 0; b < 4; ++b) X[a][b] += c * vj[a] * q[b];
                }
                double G[4][4];
#pragma unroll
                for (int a = 0; a < 4; ++a)
#pragma unroll
                    for (int b = 0; b < 4; ++b) G[a][b] = 0.5 * (X[a][b] + X[b][a]);
                dS[0] = G[0][0] + G[1][1] - G[2][2] - G[3][3];                        // xx
                dS[4] = G[0][0] - G[1][1] + G[2][2] - G[3][3];                        // yy
                dS[8] = G[0][0] - G[1][1] - G[2][2] + G[3][3];                        // zz
                dS[5] = 2.0 * (G[0][1] + G[2][3]);                                    // yz
                dS[7] = 2.0 * (-G[0][1] + G[2][3]);                                   // zy
                dS[6] = 2.0 * (G[0][2] + G[1][3]);                                    // zx
                dS[2] = 2.0 * (-G[0][2] + G[1][3]);                                   // xz
                dS[1] = 2.0 * (G[0][3] + G[1][2]);                                    // xy
                dS[3] = 2.0 * (-G[0][3] + G[1][2]);                                   // yx
            }
            const float x0 = __ldg(x + 3 * p), x1 = __ldg(x + 3 * p + 1), x2 = __ldg(x + 3 * p + 2);
            const double a[3] = {(double)x0 - xb[0], (double)x1 - xb[1], (double)x2 - xb[2]};
            const double b[3] = {(double)__fadd_rn(x0, __ldg(f + 3 * p)) - yb[0], (double)__fadd_rn(x1, __ldg(f + 3 * p + 1)) - yb[1],
                                 (double)__fadd_rn(x2, __ldg(f + 3 * p + 2)) - yb[2]};
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                gx[k] = dS[3 * k] * b[0] + dS[3 * k + 1] * b[1] + dS[3 * k + 2] * b[2] + dxb[k] / n;
                gy[k] = dS[k] * a[0] + dS[3 + k] * a[1] + dS[6 + k] * a[2] + dyb[k] / n;
            }
        }
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            d_f[3 * p + c] = (float)gy[c];
            d_x[3 * p + c] = (float)(gx[c] + gy[c]);
        }
    }
}

// ---- the grouping for O > 1 ------------------------------------------------------------------------------------------------
// The points of each sample grouped stably by label (labels [B,N], -1 or out of [0, O): no segment) in windows of kRoChunk
// point ids, with integer counts only:
//   k_ro_group_count    per window, the number of points of each object -> cnt [B,C,O] (C = ceil(N / kRoChunk))
//   k_ro_group_scan     one CTA per sample, thread o per object: n[g] and start[g] = s N + (members of the objects before
//                       o); pre [B,C,O] = where window c's members of o go in the sample's list; the moment items (c << 8) | o of every window
//                       holding a member of o, and the score items (j << 8) | o of every kScPoints members of o
//   k_ro_group_scatter  per window, each point's rank among the window's points of its object (warp match, then the warps
//                       before it): list[pre + rank] = i, so each object's members are ascending
constexpr int kRoChunk = 256;
constexpr int kRoMaxObjects = 256;
static_assert(kRoChunk == kMomThreads, "the moment items are the grouping's windows");

__global__ void __launch_bounds__(kRoChunk) k_ro_group_count(const int32_t* __restrict__ labels, int N, int O, int C,
                                                             int32_t* __restrict__ cnt) {
    __shared__ int c_sh[kRoMaxObjects];
    const int s = blockIdx.y, c = blockIdx.x, i = c * kRoChunk + threadIdx.x;
    if (threadIdx.x < O) c_sh[threadIdx.x] = 0;
    __syncthreads();
    const int l = i < N ? labels[(long long)s * N + i] : -1;
    if (l >= 0 && l < O) atomicAdd(c_sh + l, 1);
    __syncthreads();
    if (threadIdx.x < O) cnt[((long long)s * C + c) * O + threadIdx.x] = c_sh[threadIdx.x];
}

__device__ __forceinline__ int cta_exclusive_scan(int v, int* sh, int& total) {
    sh[threadIdx.x] = v;
    __syncthreads();
    if (threadIdx.x == 0) {
        int run = 0;
        for (int k = 0; k < (int)blockDim.x; ++k) {
            const int u = sh[k];
            sh[k] = run;
            run += u;
        }
        sh[blockDim.x] = run;
    }
    __syncthreads();
    const int r = sh[threadIdx.x];
    total = sh[blockDim.x];
    __syncthreads();
    return r;
}

__global__ void __launch_bounds__(kRoMaxObjects) k_ro_group_scan(const int32_t* __restrict__ cnt, int N, int O, int C, int sstride,
                                                                 int32_t* __restrict__ pre, int32_t* __restrict__ start,
                                                                 int32_t* __restrict__ nseg, int32_t* __restrict__ mitems,
                                                                 int32_t* __restrict__ nmitems, int32_t* __restrict__ sitems,
                                                                 int32_t* __restrict__ nsitems) {
    __shared__ int sh[kRoMaxObjects + 1];
    const int s = blockIdx.x, o = threadIdx.x;
    const bool on = o < O;
    const int32_t* cs = cnt + (long long)s * C * O;
    int n = 0, nw = 0;
    if (on)
        for (int c = 0; c < C; ++c) {
            const int v = __ldg(cs + (long long)c * O + o);
            n += v;
            nw += v != 0;
        }
    const int ns = (n + kScPoints - 1) / kScPoints;
    int tn, tw, ts;
    const int bn = cta_exclusive_scan(n, sh, tn);
    int bw = cta_exclusive_scan(nw, sh, tw);
    const int bs = cta_exclusive_scan(ns, sh, ts);
    if (on) {
        const long long g = (long long)s * O + o;
        start[g] = (int32_t)((long long)s * N + bn);
        nseg[g] = n;
        int run = bn;   // within the sample
        int32_t* ps = pre + (long long)s * C * O;
        for (int c = 0; c < C; ++c) {
            const int v = __ldg(cs + (long long)c * O + o);
            ps[(long long)c * O + o] = run;
            if (v) mitems[(long long)s * N + bw++] = (c << 8) | o;
            run += v;
        }
        for (int j = 0; j < ns; ++j) sitems[(long long)s * sstride + bs + j] = (j << 8) | o;
    }
    if (threadIdx.x == 0) {
        nmitems[s] = tw;
        nsitems[s] = ts;
    }
}

__global__ void __launch_bounds__(kRoChunk) k_ro_group_scatter(const int32_t* __restrict__ labels, int N, int O, int C,
                                                               const int32_t* __restrict__ pre, int32_t* __restrict__ list) {
    __shared__ int wc[kRoChunk / kWarp][kRoMaxObjects];
    const int s = blockIdx.y, c = blockIdx.x, i = c * kRoChunk + threadIdx.x, lane = lane_id(), warp = warp_id();
    for (int k = threadIdx.x; k < (kRoChunk / kWarp) * kRoMaxObjects; k += kRoChunk) (&wc[0][0])[k] = 0;
    __syncthreads();
    int l = i < N ? labels[(long long)s * N + i] : -1;
    if (l < 0 || l >= O) l = -1;
    const unsigned peers = __match_any_sync(kFull, l);
    const int rank = __popc(peers & ((1u << lane) - 1u));
    if (l >= 0 && rank == 0) wc[warp][l] = __popc(peers);
    __syncthreads();
    if (l < 0) return;
    int before = rank;
    for (int w = 0; w < warp; ++w) before += wc[w][l];
    list[(long long)s * N + __ldg(pre + ((long long)s * C + c) * O + l) + before] = i;
}

// the forward's workspace: list [B,N] | start [G] | n [G] | cnt [B,C,O] | pre [B,C,O] | moment items [B,N] | nm [B] |
// score items [B,S] | ns [B] | hyp [G,H,16] f32 | hcnt [G,H] | model [G,16] f32 | mom [rounds,G,16] f64, each range 16-byte
// aligned (O = 1 uses list and n only of the grouping's ranges)
struct FitWs {
    int32_t *list, *start, *n, *cnt, *pre, *mitems, *nm, *sitems, *ns;
    float* hyp;
    int32_t* hcnt;
    float* model;
    double* mom;
    int C, S;
    int64_t bytes;
};
static FitWs fit_ws(void* ws, int B, int N, int O, int H, int rounds) {
    char* base = static_cast<char*>(ws);
    int64_t off = 0;
    auto take = [&](int64_t bytes) {
        char* p = base ? base + off : nullptr;
        off += (bytes + 15) / 16 * 16;
        return p;
    };
    FitWs L;
    const long long G = (long long)B * O;
    L.C = (N + kRoChunk - 1) / kRoChunk;
    L.S = (N + kScPoints - 1) / kScPoints + O;
    L.list = reinterpret_cast<int32_t*>(take(4ll * B * N));
    L.start = reinterpret_cast<int32_t*>(take(4 * G));
    L.n = reinterpret_cast<int32_t*>(take(4 * G));
    L.cnt = reinterpret_cast<int32_t*>(take(4ll * B * L.C * O));
    L.pre = reinterpret_cast<int32_t*>(take(4ll * B * L.C * O));
    L.mitems = reinterpret_cast<int32_t*>(take(4ll * B * N));
    L.nm = reinterpret_cast<int32_t*>(take(4ll * B));
    L.sitems = reinterpret_cast<int32_t*>(take(4ll * B * L.S));
    L.ns = reinterpret_cast<int32_t*>(take(4ll * B));
    L.hyp = reinterpret_cast<float*>(take(4 * G * H * kRmModel));
    L.hcnt = reinterpret_cast<int32_t*>(take(4 * G * H));
    L.model = reinterpret_cast<float*>(take(4 * G * kRmModel));
    L.mom = reinterpret_cast<double*>(take(8 * rounds * G * kRmMoments));
    L.bytes = off;
    return L;
}

static bool bad_sizes(int B, int N, int O, int H, int rounds) {
    return B < 1 || N < 1 || O < 1 || O > kRoMaxObjects || H < 1 || H > kRmMaxH || rounds < 1 || rounds > kRmMaxRounds ||
           (long long)B * N > 0x7fffffffll;
}

}  // namespace pvraft

using namespace pvraft;

extern "C" int64_t pvraft_rigid_objects_workspace_bytes(int B, int N, int O, int H, int rounds) {
    return bad_sizes(B, N, O, H, rounds) ? 0 : fit_ws(nullptr, B, N, O, H, rounds).bytes;
}

extern "C" int64_t pvraft_rigid_objects_fwd_det_workspace_bytes(int B, int O, int rounds) {
    return B < 1 || O < 1 || O > kRoMaxObjects || rounds < 1 || rounds > kRmMaxRounds ? 0 : fx_bytes((long long)rounds * B * O * kRmMoments);
}

extern "C" int pvraft_rigid_objects_fwd(const float* xyz1, const float* flow, const int32_t* labels, int B, int N, int O, float threshold,
                                        int H, int rounds, int seed, float* R, float* t, uint8_t* inliers, int32_t* count,
                                        uint8_t* degenerate, double* state, int32_t* triples, int32_t* hyp_count, void* workspace,
                                        void* det_workspace, void* stream) {
    if (!xyz1 || !flow || (!labels && O != 1) || !R || !t || !inliers || !count || !degenerate || !state || !workspace ||
        bad_sizes(B, N, O, H, rounds) || !(threshold > 0.f) || isinf(threshold) || seed < 0)
        return fail(PVRAFT_ERR_BAD_ARG, "rigid_objects_fwd: bad argument");
    if ((long long)B * O > 65535) return fail(PVRAFT_ERR_UNSUPPORTED, "rigid_objects_fwd: B * O = %lld fits (at most 65535)", (long long)B * O);
    cudaStream_t st = (cudaStream_t)stream;
    const FitWs L = fit_ws(workspace, B, N, O, H, rounds);
    const int G = B * O;
    const float thr2 = threshold * threshold;
    // O = 1: the member list in one launch (none without labels), and the score and moment kernels' one-segment grids;
    // O > 1: the stable grouping, and work items that cover each segment's members
    const int32_t *sitems = nullptr, *nsitems = nullptr, *mitems = nullptr, *nmitems = nullptr;
    unsigned score_x = (unsigned)((N + kScPoints - 1) / kScPoints), mom_x = (unsigned)L.C;
    if (O == 1) {
        if (labels) k_rigid_allowed<<<B, kRmScan, 0, st>>>(labels, N, L.list, L.n);
    } else {
        cudaError_t e = cudaMemsetAsync(inliers, 0, (size_t)B * N, st);   // the moments write the members' inliers only
        if (e != cudaSuccess) return fail((int)e, "rigid_objects_fwd: memset failed: %s", cudaGetErrorString(e));
        k_ro_group_count<<<dim3((unsigned)L.C, (unsigned)B), kRoChunk, 0, st>>>(labels, N, O, L.C, L.cnt);
        k_ro_group_scan<<<B, kRoMaxObjects, 0, st>>>(L.cnt, N, O, L.C, L.S, L.pre, L.start, L.n, L.mitems, L.nm, L.sitems, L.ns);
        k_ro_group_scatter<<<dim3((unsigned)L.C, (unsigned)B), kRoChunk, 0, st>>>(labels, N, O, L.C, L.pre, L.list);
        sitems = L.sitems, nsitems = L.ns, mitems = L.mitems, nmitems = L.nm;
        score_x = (unsigned)L.S;
        mom_x += (unsigned)O;
    }
    const RmSegs sg{labels ? L.list : nullptr, O > 1 ? L.start : nullptr, L.n, N, O};
    k_rigid_hypotheses<<<dim3((unsigned)((H + 127) / 128), (unsigned)G), 128, 0, st>>>(xyz1, flow, sg, H, (unsigned long long)seed,
                                                                                      threshold, L.hyp, L.hcnt, triples);
    k_rigid_score<<<dim3(score_x, (unsigned)((H + kScHyp - 1) / kScHyp), (unsigned)B), kScThreads, 0, st>>>(
        xyz1, flow, sg, sitems, nsitems, L.S, H, thr2, L.hyp, L.hcnt);
    k_rigid_select<<<G, kSelThreads, 0, st>>>(xyz1, flow, sg, H, G, rounds, L.hyp, L.hcnt, L.model, L.mom, hyp_count);
    const unsigned sblocks = (unsigned)((G + 63) / 64);
    for (int r = 0; r < rounds; ++r) {
        double* mom = L.mom + (long long)r * G * kRmMoments;
        if (det_workspace) {
            const FxSlots slots = fx_slots(det_workspace) + (long long)r * G * kRmMoments;
            k_rigid_moments<true><<<dim3(mom_x, (unsigned)B), kMomThreads, 0, st>>>(xyz1, flow, labels, mitems, nmitems, O, N, thr2, L.model,
                                                                                  inliers, slots);
            k_rigid_solve<true><<<sblocks, 64, 0, st>>>(mom, slots, G, L.model, R, t, count, degenerate, state);
        } else {
            k_rigid_moments<false><<<dim3(mom_x, (unsigned)B), kMomThreads, 0, st>>>(xyz1, flow, labels, mitems, nmitems, O, N, thr2, L.model,
                                                                                   inliers, mom);
            k_rigid_solve<false><<<sblocks, 64, 0, st>>>(mom, FxSlots{}, G, L.model, R, t, count, degenerate, state);
        }
    }
    return check_launch("rigid_objects_fwd");
}

extern "C" int pvraft_rigid_objects_bwd(const float* xyz1, const float* flow, const int32_t* labels, const uint8_t* inliers,
                                        const double* state, const float* dR, const float* dt, int B, int N, int O, float* d_xyz1,
                                        float* d_flow, void* stream) {
    if (!xyz1 || !flow || (!labels && O != 1) || !inliers || !state || !dR || !dt || !d_xyz1 || !d_flow || B < 1 || N < 1 || O < 1 ||
        O > kRoMaxObjects || (long long)B * N > 0x7fffffffll)
        return fail(PVRAFT_ERR_BAD_ARG, "rigid_objects_bwd: bad argument");
    const long long points = (long long)B * N;
    const unsigned blocks = (unsigned)scatter_blocks(points, false);
    k_rigid_bwd<<<blocks, 256, 0, (cudaStream_t)stream>>>(xyz1, flow, inliers, labels, O, state, dR, dt, N, points, d_xyz1, d_flow);
    return check_launch("rigid_objects_bwd");
}
