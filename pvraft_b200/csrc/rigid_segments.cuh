// What the rigid fit (rigid_motion.cu) and its refinement against the second scan (rigid_refine.cu) share: the segments of
// a fit -- the member lists the grouping writes -- and the cyclic Jacobi eigen-solve in double.
//
// A fit is O SEGMENTS per sample: segment (b, o) is the points with labels[b, i] == o, or, with labels NULL (O = 1), every
// point of the sample.  rm_group (rigid_motion.cu) groups the points: with O = 1 one launch of k_rigid_allowed compacts the
// members (labels == 0); with O > 1 the three k_ro_group_* launches group the points stably by label and list the moment
// items (c << 8) | o, one per window c of kMomThreads point ids that holds a member of object o.  Both give each segment
// an ascending member list, so every kernel after the grouping has one form.
#pragma once
#include "fixed_point.cuh"

namespace pvraft {

constexpr int kJacobiSweeps = 12;
constexpr int kMomThreads = 256;      // the moment windows: point ids [c kMomThreads, (c + 1) kMomThreads)
constexpr int kRoChunk = 256;         // the grouping's windows (O > 1)
constexpr int kRoMaxObjects = 256;
static_assert(kRoChunk == kMomThreads, "the moment items are the grouping's windows");

// Cyclic Jacobi on a symmetric D x D matrix: a becomes diagonal (the eigenvalues), column j of v the eigenvector of
// a[j][j].  Pairs (p, q), p < q, in row order; at most kJacobiSweeps sweeps, stopping early once a is diagonal.
template <int D>
__device__ __forceinline__ void jacobi_sym(double (&a)[D][D], double (&v)[D][D]) {
#pragma unroll
    for (int i = 0; i < D; ++i)
#pragma unroll
        for (int j = 0; j < D; ++j) v[i][j] = i == j ? 1.0 : 0.0;
    for (int sweep = 0; sweep < kJacobiSweeps; ++sweep) {
        double off = fabs(a[0][1]);   // the off-diagonal magnitudes summed in pair order
#pragma unroll
        for (int p = 0; p < D - 1; ++p)
#pragma unroll
            for (int q = p + 1; q < D; ++q)
                if (p > 0 || q > 1) off += fabs(a[p][q]);
        if (off == 0.0) break;
#pragma unroll
        for (int p = 0; p < D - 1; ++p)
#pragma unroll
            for (int q = p + 1; q < D; ++q) {
                const double apq = a[p][q];
                if (apq == 0.0) continue;
                const double theta = (a[q][q] - a[p][p]) / (2.0 * apq);
                const double t = fabs(theta) > 1e150 ? 0.5 / theta : copysign(1.0, theta) / (fabs(theta) + sqrt(theta * theta + 1.0));
                const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
                a[p][p] -= t * apq;
                a[q][q] += t * apq;
                a[p][q] = a[q][p] = 0.0;
#pragma unroll
                for (int k = 0; k < D; ++k) {
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

// The grouping's workspace ranges: list [B,N] | start [G] | n [G] | cnt [B,C,O] | pre [B,C,O] | moment items [B,N] | nm [B]
// | score items [B,S] | ns [B], C = ceil(N / kRoChunk), S = ceil(N / kScPoints) + O, each range 16-byte aligned (O = 1
// uses list and n only).  rm_group_carve takes them from base + off (base NULL: only counts) and advances off.
struct RmGroupWs {
    int32_t *list, *start, *n, *cnt, *pre, *mitems, *nm, *sitems, *ns;
    int C, S;
};
RmGroupWs rm_group_carve(char* base, int64_t& off, int B, int N, int O);

// Group the points of labels [B,N] (NULL only with O = 1: no launch, every point a member) into L.  The moment items and
// their counts per sample are L.mitems and L.nm with O > 1; with O = 1 window c of sample s is item c.  -> 0, or the
// check_launch code of a failed launch.
int rm_group(const int32_t* labels, int B, int N, int O, const RmGroupWs& L, cudaStream_t st);

// The segments rm_group wrote.
inline RmSegs rm_segs(const int32_t* labels, int N, int O, const RmGroupWs& L) {
    return RmSegs{labels ? L.list : nullptr, O > 1 ? L.start : nullptr, L.n, N, O};
}

}  // namespace pvraft
