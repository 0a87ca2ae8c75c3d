// The uniform-grid index of grid_index.cuh for any N and any number of samples, built on the device in one launch sequence
// with no host synchronisation (the searches run inside CUDA-graph capture):
//
//   k_gi_bounds   per sample: bounding box and largest |p|^2, CTA reductions merged with atomics on order-preserving keys
//   k_gi_params   one thread per sample: cell edge and grid dimensions, as k_grid_sort, but with a cell budget that grows with N
//   k_gi_count    cell id of every point and its rank among its cell's points (an atomic histogram of cell ids)
//   k_gi_scan     one CTA per sample: exclusive scan of the histogram -> cell_start
//   k_gi_scatter  point (x, y, z, |p|^2) and id to cell_start[cell] + rank
//
// The ranks come from atomics, so the order of the points WITHIN a cell can differ from run to run.  That is allowed only
// because every search on the index ranks candidates on (distance, original id) and visits a cell's points as a set: the
// result does not depend on the order inside a cell, and is bitwise the same from run to run.
#include "fixed_point.cuh"
#include "grid_index.cuh"

namespace pvraft {

constexpr int kGiThreads = 256;
constexpr int kGiScanThreads = 1024;
constexpr int kGiBoundCtas = 64;   // CTAs per sample of the bounds reduction

__device__ __forceinline__ void load_point(const float* __restrict__ xyz, const float* __restrict__ off, long long p, float& x, float& y,
                                           float& z) {
    x = __ldg(xyz + 3 * p);
    y = __ldg(xyz + 3 * p + 1);
    z = __ldg(xyz + 3 * p + 2);
    if (off) {   // W = P + offset, the add of k_flow_propagate's staging
        x = __fadd_rn(x, __ldg(off + 3 * p));
        y = __fadd_rn(y, __ldg(off + 3 * p + 1));
        z = __fadd_rn(z, __ldg(off + 3 * p + 2));
    }
}

// lo [S,4] (memset 0xff) and hi [S,4] (memset 0) as ord_key: lo = (min x, min y, min z, -), hi = (max x, max y, max z, max |p|^2).
// NaN coordinates are ignored, as by k_grid_sort's fminf / fmaxf.
__global__ void __launch_bounds__(kGiThreads) k_gi_bounds(const float* __restrict__ xyz, const float* __restrict__ off, int N,
                                                          unsigned* __restrict__ lo_key, unsigned* __restrict__ hi_key) {
    const int s = blockIdx.y;
    float lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY}, mx = 0.f;
    for (int i = blockIdx.x * kGiThreads + threadIdx.x; i < N; i += gridDim.x * kGiThreads) {
        float x, y, z;
        load_point(xyz, off, (long long)s * N + i, x, y, z);
        lo[0] = fminf(lo[0], x); lo[1] = fminf(lo[1], y); lo[2] = fminf(lo[2], z);
        hi[0] = fmaxf(hi[0], x); hi[1] = fmaxf(hi[1], y); hi[2] = fmaxf(hi[2], z);
        mx = fmaxf(mx, sqnorm(x, y, z));
    }
#pragma unroll
    for (int a = 0; a < 3; ++a) { lo[a] = -warp_max(-lo[a]); hi[a] = warp_max(hi[a]); }
    mx = warp_max(mx);
    if (lane_id() == 0) {
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            atomicMin(lo_key + 4 * s + a, ord_key(lo[a]));
            atomicMax(hi_key + 4 * s + a, ord_key(hi[a]));
        }
        atomicMax(hi_key + 4 * s + 3, ord_key(mx));
    }
}

// The cell edge of k_grid_sort (~kGridOcc points per cell of the bounding box, the thin axis of a flat cloud one cell),
// enlarged until the grid has at most `cells` cells and at most kGridMaxDim along every axis.
__global__ void k_gi_params(const unsigned* __restrict__ lo_key, const unsigned* __restrict__ hi_key, int S, int N, int cells,
                            GridParams* __restrict__ params) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= S) return;
    float lo[3], hi[3];
    for (int a = 0; a < 3; ++a) {
        lo[a] = ord_float(lo_key[4 * s + a]);
        hi[a] = ord_float(hi_key[4 * s + a]);
    }
    const float mx = ord_float(hi_key[4 * s + 3]);
    GridParams gp;
    float ext[3], vol = 1.f, big = 0.f, amax = 0.f;
    for (int a = 0; a < 3; ++a) {
        ext[a] = fmaxf(hi[a] - lo[a], 0.f);
        big = fmaxf(big, ext[a]);
        amax = fmaxf(amax, fmaxf(fabsf(lo[a]), fabsf(hi[a])));
    }
    for (int a = 0; a < 3; ++a) vol *= fmaxf(ext[a], 1e-3f * big + 1e-20f);
    float h = cbrtf(kGridOcc * vol / (float)N);
    h = fmaxf(h, big / (float)kGridMaxDim + 1e-30f);
    for (;;) {
        long long n = 1;
        for (int a = 0; a < 3; ++a) { gp.G[a] = max(1, min(kGridMaxDim, (int)ceilf(ext[a] / h))); n *= gp.G[a]; }
        if (n <= cells) break;
        h *= 1.26f;
    }
    for (int a = 0; a < 3; ++a) { gp.gmin[a] = lo[a]; gp.h[a] = h; gp.inv_h[a] = 1.f / h; }
    gp.margin = 1e-5f * (amax + big) + 1e-30f;
    gp.max_norm = mx;
    params[s] = gp;
}

// key[s,i] = linear cell id of point i, rank[s,i] = its slot among the points of that cell; hist [S, cells + 1] zeroed
__global__ void __launch_bounds__(kGiThreads) k_gi_count(const float* __restrict__ xyz, const float* __restrict__ off, int N, int cells,
                                                         const GridParams* __restrict__ params, int32_t* __restrict__ hist,
                                                         int32_t* __restrict__ key, int32_t* __restrict__ rank) {
    const int s = blockIdx.y;
    const int i = blockIdx.x * kGiThreads + threadIdx.x;
    if (i >= N) return;
    const GridParams gp = params[s];
    const long long p = (long long)s * N + i;
    float x, y, z;
    load_point(xyz, off, p, x, y, z);
    const int cx = cell_coord(x, gp.gmin[0], gp.inv_h[0], gp.G[0]);
    const int cy = cell_coord(y, gp.gmin[1], gp.inv_h[1], gp.G[1]);
    const int cz = cell_coord(z, gp.gmin[2], gp.inv_h[2], gp.G[2]);
    const int c = (cz * gp.G[1] + cy) * gp.G[0] + cx;
    key[p] = c;
    rank[p] = atomicAdd(hist + (long long)s * (cells + 1) + c, 1);
}

// in place: cs[s, c] = sum of the counts of cells < c, for c in [0, cells]; each thread scans one contiguous chunk
__global__ void __launch_bounds__(kGiScanThreads) k_gi_scan(int32_t* __restrict__ cs, int cells) {
    __shared__ int s_warp[kGiScanThreads / 32];
    int32_t* c = cs + (long long)blockIdx.x * (cells + 1);
    const int n = cells + 1;
    const int per = (n + kGiScanThreads - 1) / kGiScanThreads;
    const int lo = min(n, (int)threadIdx.x * per), hi = min(n, lo + per);
    int sum = 0;
    for (int i = lo; i < hi; ++i) sum += c[i];
    const int lane = lane_id(), warp = warp_id();
    int incl = sum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int v = __shfl_up_sync(kFull, incl, o);
        if (lane >= o) incl += v;
    }
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    if (warp == 0) {
        int v = s_warp[lane];
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int u = __shfl_up_sync(kFull, v, o);
            if (lane >= o) v += u;
        }
        s_warp[lane] = v;
    }
    __syncthreads();
    int run = incl - sum + (warp ? s_warp[warp - 1] : 0);
    for (int i = lo; i < hi; ++i) {
        const int v = c[i];
        c[i] = run;
        run += v;
    }
}

__global__ void __launch_bounds__(kGiThreads) k_gi_scatter(const float* __restrict__ xyz, const float* __restrict__ off, int N, int cells,
                                                           const int32_t* __restrict__ cs, const int32_t* __restrict__ key,
                                                           const int32_t* __restrict__ rank, float4* __restrict__ pts, int32_t* __restrict__ ids) {
    const int s = blockIdx.y;
    const int i = blockIdx.x * kGiThreads + threadIdx.x;
    if (i >= N) return;
    const long long p = (long long)s * N + i;
    float x, y, z;
    load_point(xyz, off, p, x, y, z);
    const long long dst = (long long)s * N + __ldg(cs + (long long)s * (cells + 1) + __ldg(key + p)) + __ldg(rank + p);
    pts[dst] = make_float4(x, y, z, sqnorm(x, y, z));
    ids[dst] = i;
}

int grid_index_cells(int N) {
    const long long c = (long long)kGridCellsPerPoint * N;
    return (int)(c < kGridMinCells ? kGridMinCells : (c > (1 << 28) ? (1 << 28) : c));
}

// workspace: float4 pts[S*N] | int32 ids[S*N] | int32 key[S*N] | int32 rank[S*N] | int32 cell_start[S*(cells+1)] |
//            GridParams[S] | unsigned lo[S*4] | unsigned hi[S*4], every block 16-byte aligned
struct GiWs {
    float4* pts;
    int32_t *ids, *key, *rank, *cell_start;
    GridParams* params;
    unsigned *lo, *hi;
    int64_t bytes;
};
static GiWs gi_ws(void* ws, int S, int N) {
    ByteCarve w(ws);
    const long long sn = (long long)S * N;
    GiWs L;
    L.pts = w.take<float4>(sn * (long long)sizeof(float4));
    L.ids = w.take<int32_t>(4 * sn);
    L.key = w.take<int32_t>(4 * sn);
    L.rank = w.take<int32_t>(4 * sn);
    L.cell_start = w.take<int32_t>(4ll * S * (grid_index_cells(N) + 1));
    L.params = w.take<GridParams>((long long)S * (long long)sizeof(GridParams));
    L.lo = w.take<unsigned>(16ll * S);
    L.hi = w.take<unsigned>(16ll * S);
    L.bytes = w.bytes;
    return L;
}

int64_t grid_index_bytes(int S, int N) { return S < 1 || N < 1 ? 0 : gi_ws(nullptr, S, N).bytes; }

GridIndex grid_index_carve(void* workspace, int S, int N) {
    const GiWs L = gi_ws(workspace, S, N);
    return GridIndex{L.pts, L.ids, L.cell_start, L.params, grid_index_cells(N)};
}

int grid_index_build(const float* xyz, const float* offset, int S, int N, void* workspace, cudaStream_t st, GridIndex* ix) {
    if (!xyz || !workspace || S < 1 || N < 1) return fail(PVRAFT_ERR_BAD_ARG, "grid_index: bad argument");
    if (S > 65535) return fail(PVRAFT_ERR_UNSUPPORTED, "grid_index: S = %d samples (at most 65535)", S);
    if (reinterpret_cast<uintptr_t>(workspace) & 15) return fail(PVRAFT_ERR_BAD_ARG, "grid_index: workspace not 16-byte aligned");
    const GiWs L = gi_ws(workspace, S, N);
    *ix = grid_index_carve(workspace, S, N);
    const int cells = ix->cells;
    cudaError_t e = cudaMemsetAsync(L.lo, 0xff, (size_t)S * 16, st);
    if (e == cudaSuccess) e = cudaMemsetAsync(L.hi, 0, (size_t)S * 16, st);
    if (e == cudaSuccess) e = cudaMemsetAsync(ix->cell_start, 0, (size_t)S * (cells + 1) * 4, st);
    if (e != cudaSuccess) return fail((int)e, "grid_index: memset failed: %s", cudaGetErrorString(e));
    const int per_sample = (N + kGiThreads - 1) / kGiThreads;
    int rc;
    k_gi_bounds<<<dim3(min(per_sample, kGiBoundCtas), S), kGiThreads, 0, st>>>(xyz, offset, N, L.lo, L.hi);
    if ((rc = check_launch("grid_index bounds"))) return rc;
    k_gi_params<<<(S + 31) / 32, 32, 0, st>>>(L.lo, L.hi, S, N, cells, ix->params);
    if ((rc = check_launch("grid_index params"))) return rc;
    k_gi_count<<<dim3(per_sample, S), kGiThreads, 0, st>>>(xyz, offset, N, cells, ix->params, ix->cell_start, L.key, L.rank);
    if ((rc = check_launch("grid_index count"))) return rc;
    k_gi_scan<<<S, kGiScanThreads, 0, st>>>(ix->cell_start, cells);
    if ((rc = check_launch("grid_index scan"))) return rc;
    k_gi_scatter<<<dim3(per_sample, S), kGiThreads, 0, st>>>(xyz, offset, N, cells, ix->cell_start, L.key, L.rank, ix->pts, ix->ids);
    return check_launch("grid_index scatter");
}

}  // namespace pvraft

using namespace pvraft;

extern "C" int64_t pvraft_grid_index_workspace_bytes(int S, int N) { return grid_index_bytes(S, N); }

extern "C" int pvraft_grid_index_fwd(const float* xyz, const float* offset, int S, int N, void* workspace, void* stream) {
    GridIndex ix;
    return grid_index_build(xyz, offset, S, N, workspace, (cudaStream_t)stream, &ix);
}
