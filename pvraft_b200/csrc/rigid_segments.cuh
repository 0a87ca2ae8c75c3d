// What the rigid family (rigid_motion.cu, rigid_refine.cu, clusters.cu, tracks.cu) shares: the segments of a fit -- the
// member lists the grouping writes, its work items and the walk and sum over them --, the fp32 model, which points take
// part, the object limit, and the small device helpers (dot3, the block scan, the cyclic Jacobi eigen-solve in double).
//
// A fit is O SEGMENTS per sample: segment (b, o) is the points with labels[b, i] == o, or, with labels NULL (O = 1), every
// point of the sample.  rm_group (rigid_motion.cu) groups the points whenever labels are given: the three k_ro_group_*
// launches group them stably by label, so each segment has an ascending member list, and list the work items
// (c << 8) | o (seg_item_code): the moment items, one per window c of kMomThreads point ids that holds a member of object
// o, and the score items, one per kScPoints members of o.  Every kernel after the grouping has one form.
#pragma once
#include "fixed_point.cuh"

namespace pvraft {

constexpr int kJacobiSweeps = 12;
constexpr int kMomThreads = 256;      // the moment windows: point ids [c kMomThreads, (c + 1) kMomThreads)
constexpr int kRoChunk = 256;         // the grouping's windows
constexpr int kMaxObjects = 256;      // segments per sample of a fit, objects of a clustering or a tracking step
static_assert(kRoChunk == kMomThreads, "the moment items are the grouping's windows");

// The fp32 model of a segment: R (9, row-major), c_x (3), c_y (3), flag
constexpr int kModel = 16, kModelCx = 9, kModelCy = 12, kModelFlag = 15;

__device__ __forceinline__ bool finite3(float x, float y, float z) { return isfinite(x) && isfinite(y) && isfinite(z); }

// Whether point p (coordinates x, y, z) takes part in a clustering or as a target: mask (or NULL: every point) allows it
// and its coordinates are finite.  The callers stage any other point as NaN.
__device__ __forceinline__ bool takes_part(const uint8_t* mask, long long p, float x, float y, float z) {
    return (!mask || mask[p] != 0) && finite3(x, y, z);
}

// r_k = (R (x - c_x))_k under model m in fp32: d = x - c_x; ((R_k0 d_0 + R_k1 d_1) + R_k2 d_2), every operation rounded to
// nearest, none contracted
__device__ __forceinline__ void model_rotate(const float* m, float x0, float x1, float x2, float (&r)[3]) {
    const float d0 = __fsub_rn(x0, m[kModelCx]), d1 = __fsub_rn(x1, m[kModelCx + 1]), d2 = __fsub_rn(x2, m[kModelCx + 2]);
#pragma unroll
    for (int k = 0; k < 3; ++k) r[k] = __fadd_rn(__fadd_rn(__fmul_rn(m[3 * k], d0), __fmul_rn(m[3 * k + 1], d1)), __fmul_rn(m[3 * k + 2], d2));
}

// (a0 b0 + a1 b1) + a2 b2 in double, every operation rounded to nearest, none contracted
__device__ __forceinline__ double dot3(double a0, double a1, double a2, double b0, double b1, double b2) {
    return __dadd_rn(__dadd_rn(__dmul_rn(a0, b0), __dmul_rn(a1, b1)), __dmul_rn(a2, b2));
}

// An exclusive scan of v over the CTA's T threads (warp shuffles, then the warp totals); total: the sum.  Ends with a
// barrier, so it can be called again at once.
template <int T>
__device__ __forceinline__ int block_exclusive_scan(int v, int& total) {
    __shared__ int wsum[T / kWarp];
    const int lane = lane_id(), warp = warp_id();
    int x = v;
#pragma unroll
    for (int o = 1; o < kWarp; o <<= 1) {
        const int y = __shfl_up_sync(kFull, x, o);
        if (lane >= o) x += y;
    }
    if (lane == kWarp - 1) wsum[warp] = x;
    __syncthreads();
    int before = 0;
    total = 0;
#pragma unroll
    for (int w = 0; w < T / kWarp; ++w) {
        const int s = wsum[w];
        before += w < warp ? s : 0;
        total += s;
    }
    __syncthreads();
    return before + x - v;
}

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

// The segments of one fit: segment g is a subset of sample g / per, and its members, ascending, are list[start[g], start[g] +
// n[g]) -- or, with list NULL (no labels), all N points of the sample.
struct RmSegs {
    const int32_t* list;    // [B,N] member ids, or NULL
    const int32_t* start;   // [G] offset of each segment's members in list (read with list only)
    const int32_t* n;       // [G] member counts (read with list only)
    int N, per;
    __device__ __forceinline__ int count(int g) const { return list ? n[g] : N; }
    __device__ __forceinline__ int member(int g, long long j) const { return list ? __ldg(list + start[g] + j) : (int)j; }
};

// A work item (c << 8) | o: chunk c of segment (sample, o) -- a window of kMomThreads point ids for the moments, kScPoints
// members for the score
constexpr int kItemObjectBits = 8;
static_assert(kMaxObjects <= 1 << kItemObjectBits, "an item's object field holds every object");
__device__ __forceinline__ int32_t seg_item_code(int c, int o) { return (c << kItemObjectBits) | o; }

// Item `it` of sample s, from items [B,stride]; without items (one segment per sample) item it is chunk it of segment s.
struct SegItem {
    int g, o, c;   // the segment, its object, the chunk
};
__device__ __forceinline__ SegItem seg_item(const int32_t* items, int s, int per, long long stride, int it) {
    if (!items) return SegItem{s, 0, it};
    const int w = items[(long long)s * stride + it];
    const int o = w & ((1 << kItemObjectBits) - 1);
    return SegItem{s * per + o, o, w >> kItemObjectBits};
}

// The window walk that k_rigid_moments, k_rf_members and k_icp_step run over the moment windows, grid (x, B), sample
// s = blockIdx.y:
//     for (int it = items ? (int)blockIdx.x : 0; it < (items ? nitems[s] : 1); it += gridDim.x)
//         seg_item(items, s, per, N, items ? it : (int)blockIdx.x)
// with items [B,N] (nitems [B] per sample) CTA x takes items x, x + gridDim.x, ...; without, CTA x is window x of segment
// (sample, 0).

// Sum v[0..K) over the CTA's warps in order (warp xor butterfly, then warp 0, 1, ...) and add it once into acc slot
// g * K + k.  part: [kMomThreads / kWarp][K] shared.
template <int K, class A>
__device__ __forceinline__ void window_add(double (&v)[K], double (*part)[K], A acc, long long g) {
#pragma unroll
    for (int k = 0; k < K; ++k) v[k] = warp_sum(v[k]);
    if (lane_id() == 0)
#pragma unroll
        for (int k = 0; k < K; ++k) part[warp_id()][k] = v[k];
    __syncthreads();
    if (threadIdx.x < K) {
        double t = 0.0;
        for (int w = 0; w < kMomThreads / kWarp; ++w) t += part[w][threadIdx.x];
        if (t != 0.0) add(acc, g * K + threadIdx.x, t);
    }
    __syncthreads();   // part is reused by the next item
}

// Accumulator slot i, summed by window_add in either mode: the default mode's doubles, or (DET) the fixed-point slots
template <bool DET>
__device__ __forceinline__ double acc_read(const double* acc, FxSlots slots, long long i) {
    return DET ? fx_value(slots.base + i * kFxWords) : acc[i];
}

// The grouping's workspace ranges: list [B,N] | start [G] | n [G] | cnt [B,C,O] | pre [B,C,O] | moment items [B,N] | nm [B]
// | score items [B,S] | ns [B], C = ceil(N / kRoChunk), S = ceil(N / kScPoints) + O, each range 16-byte aligned, taken
// from w.
struct RmGroupWs {
    int32_t *list, *start, *n, *cnt, *pre, *mitems, *nm, *sitems, *ns;
    int C, S;
};
RmGroupWs rm_group_carve(ByteCarve& w, int B, int N, int O);

// Group the points of labels [B,N] (NULL only with O = 1: no launch, every point a member) into L.  -> 0, or the
// check_launch code of a failed launch.
int rm_group(const int32_t* labels, int B, int N, int O, const RmGroupWs& L, cudaStream_t st);

// The segments rm_group wrote.
inline RmSegs rm_segs(const int32_t* labels, int N, int O, const RmGroupWs& L) {
    return RmSegs{labels ? L.list : nullptr, L.start, L.n, N, O};
}

}  // namespace pvraft
