// A uniform-grid index of point clouds of any size, and the exact k-nearest search on it in the difference form.
//
// The index of S clouds of N points (grid_index_build, csrc/grid_index.cu) is what k_knn_grid reads: per sample the points
// as float4 (x, y, z, |p|^2) sorted by linear cell id (x fastest), their original ids, cell_start[c] = number of points in
// cells < c, and GridParams.  k_grid_sort (knn.cu) builds the same layout in shared memory for N <= 16384; this one is a
// multi-CTA counting sort for any N.
#pragma once
#include "nn_search.cuh"

namespace pvraft {

struct GridParams {      // one per sample
    float gmin[3], h[3], inv_h[3];
    int G[3];
    float margin;        // absolute safety margin of the face-distance bound (cell assignment is done in fp32)
    float max_norm;      // largest |p|^2 of the sample (rounding slack of the expanded distance form)
};

__device__ __forceinline__ float sqnorm(float x, float y, float z) {
    return __fadd_rn(__fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y)), __fmul_rn(z, z));
}

__device__ __forceinline__ int cell_coord(float v, float gmin, float inv_h, int G) {
    const int c = (int)floorf((v - gmin) * inv_h);
    return c < 0 ? 0 : (c >= G ? G - 1 : c);
}

// (distance, id) ordering: smaller distance first, ties -> smaller id first
__device__ __forceinline__ bool worse(float d1, int i1, float d2, int i2) { return d1 > d2 || (d1 == d2 && i1 > i2); }

// The warp keeps its current k best SORTED across the lanes (lane i = i-th best, lanes >= k hold +inf sentinels), so an
// insertion is one ballot + one shuffle-up instead of a full warp reduction for the new k-th distance.
// insert the candidates flagged in `cand` (one per lane: d, id); tau / tau_i = the current k-th (distance, id)
__device__ __forceinline__ void insert_candidates(unsigned cand, float d, int id, float& bd, int& bi, float& tau, int& tau_i, int k) {
    const int lane = lane_id();
    while (cand) {
        const int src = __ffs(cand) - 1;
        cand &= cand - 1;
        const float cd = __shfl_sync(kFull, d, src);
        const int cid = __shfl_sync(kFull, id, src);
        if (worse(cd, cid, tau, tau_i)) continue;   // tau may have tightened since the ballot
        const unsigned behind = __ballot_sync(kFull, worse(bd, bi, cd, cid));   // a suffix of the lanes: they move up by one
        const float nd = __shfl_up_sync(kFull, bd, 1);
        const int ni = __shfl_up_sync(kFull, bi, 1);
        if ((behind >> lane) & 1u) {
            const bool first = lane == 0 || !((behind >> (lane - 1)) & 1u);
            bd = first ? cd : nd;
            bi = first ? cid : ni;
        }
        tau = __shfl_sync(kFull, bd, k - 1);
        tau_i = __shfl_sync(kFull, bi, k - 1);
    }
}

// ---- the index of S clouds ----------------------------------------------------------------------------------------------
struct GridIndex {
    float4* pts;           // [S,N] (x, y, z, |p|^2) in cell order
    int32_t* ids;          // [S,N] original id of each sorted point
    int32_t* cell_start;   // [S, cells + 1]
    GridParams* params;    // [S]
    int cells;             // cell budget of every sample: the row stride of cell_start is cells + 1
};

// Cells per sample: at most max(kGridMinCells, kGridCellsPerPoint * N), and at most kGridMaxDim along an axis.  The cell edge
// aims at kGridOcc points per cell of the bounding box, as k_grid_sort's does; the budget only binds for boxes much longer
// along one axis than the others, and keeps cell_start at 4 bytes per point.
constexpr int kGridMinCells = 32768;
constexpr int kGridCellsPerPoint = 1;
constexpr int kGridMaxDim = 1024;
constexpr float kGridOcc = 3.0f;

int grid_index_cells(int N);
int64_t grid_index_bytes(int S, int N);
GridIndex grid_index_carve(void* workspace, int S, int N);
// Build the index of xyz [S,N,3] (+ offset [S,N,3], one fp32 add per coordinate, when offset != NULL) in `workspace`
// (grid_index_bytes(S, N) bytes, 16-byte aligned).  No host synchronisation: capturable into a CUDA graph.
int grid_index_build(const float* xyz, const float* offset, int S, int N, void* workspace, cudaStream_t st, GridIndex* ix);

// ---- the k-nearest search in the difference form --------------------------------------------------------------------------
constexpr int kGridNone = 0x7fffff00;   // ids of the list's unfilled slots (kGridNone + lane): larger than any point id

// score the sorted range [begin, end) of the index against q (one warp), for grid_knn_diff
__device__ __forceinline__ void grid_scan_diff(const float4* __restrict__ P, const int32_t* __restrict__ I, int begin, int end, float qx, float qy,
                                               float qz, int k, float& bd, int& bi, float& tau, int& tau_i) {
    const int lane = lane_id();
    for (int i0 = begin; i0 < end; i0 += 32) {
        const int i = i0 + lane;
        float d = INFINITY;
        int id = 0x7fffffff;
        if (i < end) {
            d = diff_sq(qx, qy, qz, __ldg(P + i));
            id = __ldg(I + i);
        }
        const unsigned cand = __ballot_sync(kFull, i < end && d < INFINITY && !worse(d, id, tau, tau_i));
        insert_candidates(cand, d, id, bd, bi, tau, tau_i, k);
    }
}

// One warp finds the k (<= 32) nearest points of q in one sample of the index, ranked on (diff_sq(q, p), id) -- the order of
// the brute-force searches of nn_search.cuh, whatever order the points are visited in.  Only finite distances enter the list
// (the brute-force searches admit a point only below a finite or infinite running k-th distance, which +inf and NaN never
// are).  On return lane r < k holds the r-th nearest (bd, bi); a slot no point filled holds (+inf, kGridNone + r).
//
// The visit is k_knn_grid's: shells of cells of growing Chebyshev radius r around q's cell.  The stopping rule must be exact
// for the computed fp32 distance.  After shell r, every unvisited point p lies outside the box of cells [c - r, c + r], so on
// some axis a, |q_a - p_a| >= bound, the distance from q to the nearest face of the box with cells behind it; `margin`
// covers the fp32 error of the face position and of the cell assignment (k_knn_grid), so b = bound - margin is a lower
// bound on |q_a - p_a| in exact arithmetic.  Rounding to nearest is monotone, and b is an fp32 number, so the computed
// |dx_a| = fl(|q_a - p_a|) >= b and fl(dx_a * dx_a) >= fl(b * b).  Every other term of diff_sq is >= 0 and each rounded sum
// of non-negative terms is >= each of its terms, so the computed distance of p is >= fl(b * b): the bound carries the
// rounding of all three products and both sums with no slack term.  The search stops when fl(b * b) > tau, STRICTLY: every
// unvisited point then has a distance above the k-th, so none can enter, not even on an equal distance with a lower id.
__device__ __forceinline__ void grid_knn_diff(const float4* __restrict__ P, const int32_t* __restrict__ I, const int32_t* __restrict__ CS,
                                              const GridParams& gp, float qx, float qy, float qz, int k, float& bd, int& bi) {
    const int lane = lane_id();
    const float qv[3] = {qx, qy, qz};
    int c[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) c[a] = cell_coord(qv[a], gp.gmin[a], gp.inv_h[a], gp.G[a]);
    bd = INFINITY;                 // sorted list of (distance, id): +inf sentinels with ascending ids
    bi = kGridNone + lane;
    float tau = INFINITY;
    int tau_i = kGridNone + k - 1;
    auto scan = [&](int begin, int end) {   // score the sorted range [begin, end)
        grid_scan_diff(P, I, begin, end, qx, qy, qz, k, bd, bi, tau, tau_i);
    };
    const int rmax = max(max(gp.G[0], gp.G[1]), gp.G[2]);
    for (int r = 0; r < rmax; ++r) {
        const int x0 = max(c[0] - r, 0), x1 = min(c[0] + r, gp.G[0] - 1);
        for (int z = max(c[2] - r, 0); z <= min(c[2] + r, gp.G[2] - 1); ++z) {
            const bool z_face = (z == c[2] - r) || (z == c[2] + r);
            for (int y = max(c[1] - r, 0); y <= min(c[1] + r, gp.G[1] - 1); ++y) {
                const int row = (z * gp.G[1] + y) * gp.G[0];
                if (z_face || y == c[1] - r || y == c[1] + r) {
                    scan(__ldg(CS + row + x0), __ldg(CS + row + x1 + 1));   // the whole run along x is new
                } else {   // only the two end cells of the run are on the shell
                    if (c[0] - r >= 0) scan(__ldg(CS + row + c[0] - r), __ldg(CS + row + c[0] - r + 1));
                    if (c[0] + r < gp.G[0] && r > 0) scan(__ldg(CS + row + c[0] + r), __ldg(CS + row + c[0] + r + 1));
                }
            }
        }
        float bound = INFINITY;
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            if (c[a] - r > 0) bound = fminf(bound, qv[a] - (gp.gmin[a] + (float)(c[a] - r) * gp.h[a]));
            if (c[a] + r < gp.G[a] - 1) bound = fminf(bound, (gp.gmin[a] + (float)(c[a] + r + 1) * gp.h[a]) - qv[a]);
        }
        if (bound == INFINITY) break;                 // the box covers the whole grid
        const float b = bound - gp.margin;
        if (b > 0.f && __fmul_rn(b, b) > tau) break;
    }
}

}  // namespace pvraft

namespace pvraft {

// The grid forms of the fused search kernels (k_chamfer_grid, k_laplacian_grid, k_flow_propagate_grid): one warp per query,
// each warp taking kGqPerWarp consecutive queries in order, so what a warp sums is a function of the shapes.
constexpr int kGqWarps = 8;
constexpr int kGqThreads = kGqWarps * kWarp;
constexpr int kGqPerWarp = 8;
constexpr int kGqPerCta = kGqWarps * kGqPerWarp;

}  // namespace pvraft
