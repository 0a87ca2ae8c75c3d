// k-nearest-neighbour search: backs knn_point (reference model/pointconv.py:28-39) and the adjacency of
// Graph.construct_graph (reference model/flot/graph.py:53-60, which sorts a full N x N distance matrix to keep
// 32 columns).
//
// Kernels:
//   k_grid_sort   one CTA per sample: bounding box -> uniform grid (~3 points per cell), points sorted by cell id with a
//                 bitonic sort in shared memory -> float4 (x,y,z,|p|^2) in cell order + original ids
//   k_grid_cells  cell_start[c] by binary search in the sorted cell ids
//   k_knn_grid    one warp per query: grid_knn (grid_index.cuh), shells of cells of growing radius around the query's cell; the
//                 warp keeps the current k best as one (distance, id) pair per lane plus the running k-th distance tau, a
//                 candidate enters only if it beats tau, and the search stops once the unvisited space is farther than tau plus
//                 the rounding slack of the distance formula: a few hundred candidates are scored per query instead of the
//                 whole cloud.
// Distances reproduce the reference's expanded form bit-for-bit on the CPU oracle: |q|^2 and |x|^2 as
// (x*x+y*y)+z*z, q.x as fma(z,z',fma(y,y',x*x')); ranking is on (distance, original id), so the result does not
// depend on the visiting order.  Clouds too large for the shared-memory sort get the same index from the multi-CTA counting
// sort of grid_index.cu, and the same k_knn_grid searches it.
#include "grid_index.cuh"

namespace pvraft {

constexpr int kKnnThreads = 256;
constexpr int kKnnTile = 2048;      // candidates per shared-memory tile of the brute-force kernel
constexpr int kSortMaxN = 16384;    // (key, id) pairs of the in-smem sort: 8 B * 16384 = 128 KB

__device__ __forceinline__ float ref_distance(int mode, float qx, float qy, float qz, float qn, const float4 p) {
    const float dot = __fmaf_rn(qz, p.z, __fmaf_rn(qy, p.y, __fmul_rn(qx, p.x)));
    if (mode == 0) return __fsub_rn(__fadd_rn(qn, p.w), __fmul_rn(2.f, dot));   // graph.py:53-57
    return __fadd_rn(__fadd_rn(__fmul_rn(-2.f, dot), qn), p.w);                  // pointconv.py:21-24
}

// The distance form (grid_index.cuh) of the kNN graph: ref_distance, every candidate not worse than the k-th admitted (NaN
// included; k_knn uses the same dist and admitted), and a stop once bound^2 exceeds the k-th distance by more than the
// rounding slack of the expanded form, which depends on |q|^2 and the sample's largest |p|^2.
struct ExpandedForm {
    int mode;
    float qn;
    float slack;
    __device__ __forceinline__ float dist(float qx, float qy, float qz, const float4& p) const { return ref_distance(mode, qx, qy, qz, qn, p); }
    static constexpr bool kFiniteOnly = false;
    __device__ __forceinline__ bool stop(float b, float tau) const { return b * b > tau + slack; }
};

__device__ __forceinline__ void write_result(const float* __restrict__ X, float qx, float qy, float qz, int lane, int k, int bi,
                                             size_t out_row, int32_t* __restrict__ out, float* __restrict__ rel) {
    if (lane < k) {
        const size_t o = out_row * k + lane;
        out[o] = bi;
        if (rel) {   // edge feature of Graph.construct_graph: neighbour - centre (graph.py:69-74)
            rel[o * 3 + 0] = __fsub_rn(__ldg(X + (size_t)bi * 3 + 0), qx);
            rel[o * 3 + 1] = __fsub_rn(__ldg(X + (size_t)bi * 3 + 1), qy);
            rel[o * 3 + 2] = __fsub_rn(__ldg(X + (size_t)bi * 3 + 2), qz);
        }
    }
}

// ---------------------------------------------------------------------------------------------------------
// brute force (any N)
// ---------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kKnnThreads) k_knn(const float* __restrict__ xyz, const float* __restrict__ query, int N, int S,
                                                     int k, int mode, int32_t* __restrict__ out, float* __restrict__ rel) {
    __shared__ float4 s_pts[kKnnTile];
    const int b = blockIdx.y;
    const int lane = lane_id(), w = warp_id();
    const int q = blockIdx.x * (kKnnThreads / 32) + w;
    const bool live = q < S;
    const float* X = xyz + (size_t)b * N * 3;
    float qx = 0.f, qy = 0.f, qz = 0.f;
    if (live) {
        const float* Q = query + ((size_t)b * S + q) * 3;
        qx = __ldg(Q); qy = __ldg(Q + 1); qz = __ldg(Q + 2);
    }
    const ExpandedForm form{mode, sqnorm(qx, qy, qz), 0.f};   // no stopping test: every point is scored
    float bd = INFINITY;                 // sorted list of (distance, id): +inf sentinels with ascending ids
    int bi = kGridNone + lane;
    float tau = INFINITY;
    int tau_i = kGridNone + k - 1;
    for (int base = 0; base < N; base += kKnnTile) {
        const int cnt = min(kKnnTile, N - base);
        __syncthreads();
        for (int i = threadIdx.x; i < cnt; i += kKnnThreads) {
            const float x = __ldg(X + (size_t)(base + i) * 3), y = __ldg(X + (size_t)(base + i) * 3 + 1), z = __ldg(X + (size_t)(base + i) * 3 + 2);
            s_pts[i] = make_float4(x, y, z, sqnorm(x, y, z));
        }
        __syncthreads();
        if (!live) continue;
        for (int i0 = 0; i0 < cnt; i0 += 32) {
            const int i = i0 + lane;
            float d = INFINITY;
            const int id = base + i;
            if (i < cnt) d = form.dist(qx, qy, qz, s_pts[i]);
            const unsigned cand = admitted<ExpandedForm>(i < cnt, d, id, tau, tau_i);
            insert_candidates(cand, d, id, bd, bi, tau, tau_i, k);
        }
    }
    if (live) write_result(X, qx, qy, qz, lane, k, bi, (size_t)b * S + q, out, rel);
}

// ---------------------------------------------------------------------------------------------------------
// uniform grid (N <= kSortMaxN)
// ---------------------------------------------------------------------------------------------------------
// Per sample: bounding box -> G[0] x G[1] x G[2] cells of edge h ~ cbrt(kCellOcc * volume / N) (at most kMaxCells cells),
// points sorted by linear cell id (x fastest) with the in-shared-memory bitonic sort, and cell_start[c] = number of
// points in cells < c.  A run of cells along x is therefore one contiguous range of the sorted array.
constexpr int kMaxCells = 32768;
constexpr int kMaxGridDim = 64;
constexpr float kCellOcc = 3.0f;   // (the time is flat between 1.5 and 16 points per cell: insertions dominate, not the scan)

// `morton` != 0: the sort key is the Morton (Z-order) interleave of the cell coordinates instead of the linear cell id, and only
// `ids` (the permutation) is of interest to the caller: a spatially coherent point order (pvraft_point_order_fwd).
__global__ void __launch_bounds__(1024) k_grid_sort(const float* __restrict__ xyz, int N, int NP /*pow2 >= N*/, float occ, int morton, GridParams* __restrict__ params,
                                                     float4* __restrict__ sorted, int32_t* __restrict__ ids, unsigned* __restrict__ keys) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    unsigned long long* s = reinterpret_cast<unsigned long long*>(smem_raw);   // (cell id << 32) | point id
    __shared__ float s_red[32][7];
    __shared__ GridParams s_gp;
    const int b = blockIdx.x;
    const float* X = xyz + (size_t)b * N * 3;
    // ---- bounding box and largest norm ----
    float lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY}, mx = 0.f;
    for (int i = threadIdx.x; i < N; i += blockDim.x) {
        const float x = __ldg(X + (size_t)i * 3), y = __ldg(X + (size_t)i * 3 + 1), z = __ldg(X + (size_t)i * 3 + 2);
        lo[0] = fminf(lo[0], x); lo[1] = fminf(lo[1], y); lo[2] = fminf(lo[2], z);
        hi[0] = fmaxf(hi[0], x); hi[1] = fmaxf(hi[1], y); hi[2] = fmaxf(hi[2], z);
        mx = fmaxf(mx, sqnorm(x, y, z));
    }
#pragma unroll
    for (int a = 0; a < 3; ++a) { lo[a] = -warp_max(-lo[a]); hi[a] = warp_max(hi[a]); }
    mx = warp_max(mx);
    if ((threadIdx.x & 31) == 0) {
        float* r = s_red[threadIdx.x >> 5];
        r[0] = lo[0]; r[1] = lo[1]; r[2] = lo[2]; r[3] = hi[0]; r[4] = hi[1]; r[5] = hi[2]; r[6] = mx;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        const int nw = blockDim.x >> 5;
        for (int w = 1; w < nw; ++w) {
            for (int a = 0; a < 3; ++a) { s_red[0][a] = fminf(s_red[0][a], s_red[w][a]); s_red[0][3 + a] = fmaxf(s_red[0][3 + a], s_red[w][3 + a]); }
            s_red[0][6] = fmaxf(s_red[0][6], s_red[w][6]);
        }
        GridParams gp;
        float ext[3], vol = 1.f, big = 0.f, amax = 0.f;
        for (int a = 0; a < 3; ++a) {
            ext[a] = fmaxf(s_red[0][3 + a] - s_red[0][a], 0.f);
            big = fmaxf(big, ext[a]);
            amax = fmaxf(amax, fmaxf(fabsf(s_red[0][a]), fabsf(s_red[0][3 + a])));
        }
        for (int a = 0; a < 3; ++a) vol *= fmaxf(ext[a], 1e-3f * big + 1e-20f);   // flat clouds: the thin axis gets one cell
        float h = cbrtf(occ * vol / (float)N);
        h = fmaxf(h, big / (float)kMaxGridDim + 1e-30f);
        for (;;) {   // respect the cell budget
            long long cells = 1;
            for (int a = 0; a < 3; ++a) { gp.G[a] = max(1, min(kMaxGridDim, (int)ceilf(ext[a] / h))); cells *= gp.G[a]; }
            if (cells <= kMaxCells) break;
            h *= 1.26f;
        }
        for (int a = 0; a < 3; ++a) { gp.gmin[a] = s_red[0][a]; gp.h[a] = h; gp.inv_h[a] = 1.f / h; }
        gp.margin = 1e-5f * (amax + big) + 1e-30f;
        gp.max_norm = s_red[0][6];
        s_gp = gp;
        params[b] = gp;
    }
    __syncthreads();
    const GridParams gp = s_gp;
    // ---- sort by cell id ----
    for (int i = threadIdx.x; i < NP; i += blockDim.x) {
        unsigned long long e = 0xFFFFFFFFFFFFFFFFull;   // pads sort to the end
        if (i < N) {
            const int cx = cell_coord(__ldg(X + (size_t)i * 3), gp.gmin[0], gp.inv_h[0], gp.G[0]);
            const int cy = cell_coord(__ldg(X + (size_t)i * 3 + 1), gp.gmin[1], gp.inv_h[1], gp.G[1]);
            const int cz = cell_coord(__ldg(X + (size_t)i * 3 + 2), gp.gmin[2], gp.inv_h[2], gp.G[2]);
            unsigned key = (unsigned)((cz * gp.G[1] + cy) * gp.G[0] + cx);
            if (morton) {   // cell coordinates are < 64: spread 6 bits each over every third bit
                key = 0u;
#pragma unroll
                for (int bit = 0; bit < 6; ++bit)
                    key |= (((unsigned)cx >> bit) & 1u) << (3 * bit) | (((unsigned)cy >> bit) & 1u) << (3 * bit + 1) | (((unsigned)cz >> bit) & 1u) << (3 * bit + 2);
            }
            e = ((unsigned long long)key << 32) | (unsigned)i;
        }
        s[i] = e;
    }
    __syncthreads();
    for (int size = 2; size <= NP; size <<= 1) {
        for (int stride = size >> 1; stride > 0; stride >>= 1) {
            for (int t = threadIdx.x; t < NP / 2; t += blockDim.x) {
                const int l = (t / stride) * (stride << 1) + (t % stride);
                const int u = l + stride;
                const bool asc = ((l & size) == 0);
                const unsigned long long a = s[l], c = s[u];
                if ((a > c) == asc) { s[l] = c; s[u] = a; }
            }
            __syncthreads();
        }
    }
    for (int i = threadIdx.x; i < N; i += blockDim.x) {
        const int id = (int)(s[i] & 0xFFFFFFFFull);
        const float x = __ldg(X + (size_t)id * 3), y = __ldg(X + (size_t)id * 3 + 1), z = __ldg(X + (size_t)id * 3 + 2);
        sorted[(size_t)b * N + i] = make_float4(x, y, z, sqnorm(x, y, z));
        ids[(size_t)b * N + i] = id;
        keys[(size_t)b * N + i] = (unsigned)(s[i] >> 32);
    }
}

// cell_start[b][c] = number of points of sample b whose cell id is < c, for c in [0, kMaxCells]
__global__ void k_grid_cells(const unsigned* __restrict__ keys, int N, int32_t* __restrict__ cell_start) {
    const int b = blockIdx.y;
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c > kMaxCells) return;
    const unsigned* K = keys + (size_t)b * N;
    int lo = 0, hi = N;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (__ldg(K + mid) < (unsigned)c) lo = mid + 1; else hi = mid;
    }
    cell_start[(size_t)b * (kMaxCells + 1) + c] = lo;
}

// One warp per query on the index `ix` of xyz (B samples): grid_knn in the expanded form.
__global__ void __launch_bounds__(kKnnThreads) k_knn_grid(const float* __restrict__ xyz, GridIndex ix, const float* __restrict__ query,
                                                          int N, int S, int k, int mode, int32_t* __restrict__ out, float* __restrict__ rel) {
    const int b = blockIdx.y;
    const int q = blockIdx.x * (kKnnThreads / 32) + warp_id();
    if (q >= S) return;
    const float4* P = ix.pts + (size_t)b * N;
    const int32_t* I = ix.ids + (size_t)b * N;
    const int32_t* CS = ix.cell_start + b * (ix.cells + 1ll);
    const GridParams gp = ix.params[b];
    const float* Q = query + ((size_t)b * S + q) * 3;
    const float qv[3] = {__ldg(Q), __ldg(Q + 1), __ldg(Q + 2)};
    const float qn = sqnorm(qv[0], qv[1], qv[2]);
    const ExpandedForm form{mode, qn, 4e-6f * (qn + gp.max_norm) + 1e-30f};
    float bd;
    int bi;
    grid_knn(form, P, I, CS, gp, qv[0], qv[1], qv[2], k, bd, bi);
    write_result(xyz + (size_t)b * N * 3, qv[0], qv[1], qv[2], lane_id(), k, bi, (size_t)b * S + q, out, rel);
}

// The index of k_grid_sort in `workspace` (pvraft_knn_workspace_bytes): float4 sorted[B*N] | int32 ids[B*N] | uint32 keys[B*N]
// | int32 cell_start[B*(kMaxCells+1)] | GridParams[B] (16-byte aligned).  `keys` is k_grid_sort's sort key of each point.
static GridIndex knn_index_carve(void* workspace, int B, int N, unsigned*& keys) {
    GridIndex ix;
    ix.pts = reinterpret_cast<float4*>(workspace);
    ix.ids = reinterpret_cast<int32_t*>(ix.pts + (size_t)B * N);
    keys = reinterpret_cast<unsigned*>(ix.ids + (size_t)B * N);
    ix.cell_start = reinterpret_cast<int32_t*>(keys + (size_t)B * N);
    ix.params = reinterpret_cast<GridParams*>((reinterpret_cast<uintptr_t>(ix.cell_start + (size_t)B * (kMaxCells + 1)) + 15) & ~(uintptr_t)15);
    ix.cells = kMaxCells;
    return ix;
}

}  // namespace pvraft

using namespace pvraft;

extern "C" int64_t pvraft_knn_workspace_bytes(int B, int N) {
    if (B <= 0 || N <= 0) return 0;
    if (N > kSortMaxN) return grid_index_bytes(B, N);
    return (int64_t)B * N * (int64_t)(sizeof(float4) + sizeof(int32_t) + sizeof(unsigned)) +
           (int64_t)B * (kMaxCells + 1) * (int64_t)sizeof(int32_t) + (int64_t)B * (int64_t)sizeof(GridParams) + 512;
}

extern "C" int pvraft_knn_fwd(const float* xyz, const float* query, int B, int N, int S, int k, int mode, int32_t* idx,
                              float* rel, void* workspace, void* stream) {
    if (!xyz || !query || !idx) return fail(PVRAFT_ERR_BAD_ARG, "knn: null pointer");
    if (B <= 0 || N <= 0 || S <= 0) return fail(PVRAFT_ERR_BAD_ARG, "knn: bad shape");
    if (k < 1 || k > 32 || k > N) return fail(PVRAFT_ERR_UNSUPPORTED, "knn: k=%d (need 1 <= k <= min(32, N=%d))", k, N);
    if (mode != 0 && mode != 1) return fail(PVRAFT_ERR_BAD_ARG, "knn: mode=%d", mode);
    if (B > 65535) return fail(PVRAFT_ERR_UNSUPPORTED, "knn: B=%d", B);
    cudaStream_t st = (cudaStream_t)stream;
    dim3 grid((S + kKnnThreads / 32 - 1) / (kKnnThreads / 32), B);
    GridIndex ix;
    int rc;
    if (workspace && N <= kSortMaxN && N >= 64) {
        int NP = 1;
        while (NP < N) NP <<= 1;
        unsigned* keys;
        ix = knn_index_carve(workspace, B, N, keys);
        const size_t smem = (size_t)NP * sizeof(unsigned long long);
        if ((rc = opt_in_smem(k_grid_sort, smem))) return rc;
        k_grid_sort<<<B, 1024, smem, st>>>(xyz, N, NP, kCellOcc, 0, ix.params, ix.pts, ix.ids, keys);
        if ((rc = check_launch("knn grid sort"))) return rc;
        k_grid_cells<<<dim3((kMaxCells + 1 + 255) / 256, B), 256, 0, st>>>(keys, N, ix.cell_start);
        if ((rc = check_launch("knn grid cells"))) return rc;
    } else if (workspace && N > kSortMaxN) {
        if ((rc = grid_index_build(xyz, nullptr, B, N, workspace, st, &ix))) return rc;
    } else {
        k_knn<<<grid, kKnnThreads, 0, st>>>(xyz, query, N, S, k, mode, idx, rel);
        return check_launch("knn");
    }
    k_knn_grid<<<grid, kKnnThreads, 0, st>>>(xyz, ix, query, N, S, k, mode, idx, rel);
    return check_launch("knn grid");
}

extern "C" int pvraft_point_order_fwd(const float* xyz, int B, int N, int32_t* perm, void* workspace, void* stream) {
    if (!xyz || !perm || !workspace) return fail(PVRAFT_ERR_BAD_ARG, "point_order: null pointer");
    if (B <= 0 || N < 64 || N > kSortMaxN || B > 65535) return fail(PVRAFT_ERR_UNSUPPORTED, "point_order: B=%d, N=%d (64 <= N <= %d)", B, N, kSortMaxN);
    cudaStream_t st = (cudaStream_t)stream;
    int NP = 1;
    while (NP < N) NP <<= 1;
    unsigned* keys;
    const GridIndex ix = knn_index_carve(workspace, B, N, keys);   // the permutation is the `ids` array of the sort
    const size_t smem = (size_t)NP * sizeof(unsigned long long);
    int rc;
    if ((rc = opt_in_smem(k_grid_sort, smem))) return rc;
    k_grid_sort<<<B, 1024, smem, st>>>(xyz, N, NP, kCellOcc, 1, ix.params, ix.pts, ix.ids, keys);
    if ((rc = check_launch("point order sort"))) return rc;
    const cudaError_t e = cudaMemcpyAsync(perm, ix.ids, (size_t)B * N * sizeof(int32_t), cudaMemcpyDeviceToDevice, st);
    if (e != cudaSuccess) return fail((int)e, "point_order: copy failed: %s", cudaGetErrorString(e));
    return 0;
}
