// Flow propagation along a scan sequence (no counterpart in the reference): a flow defined on one cloud, flow_prev on
// xyz_prev, is carried onto the points of another cloud xyz under a constant-velocity assumption.  The previous points
// moved by their flow, W = xyz_prev + flow_prev (one fp32 add per coordinate, formed while staging, never stored), are
// searched for the k nearest of every query q of xyz, and q takes their inverse-distance-weighted mean flow.
//
// The search is brute force in the difference form of nn_search.cuh, ranked on (distance, index): the lowest index wins an
// exact tie.  Each CTA keeps kPrPerCta queries in registers (kPrQueries per lane, the same queries in every warp) while W
// streams through double-buffered shared-memory tiles; warp w searches the w-th slice of every tile, so the eight warps
// split the searched cloud and a CTA covers only 64 queries, which fills the SMs at the model's sizes (N = 8192, B = 1:
// 128 CTAs).  Each lane keeps a sorted k-best list per query in registers; within a warp candidates arrive in ascending
// index order, so a strict comparison keeps the (distance, index) order.  At the end the eight lists of a query are merged
// on (distance, index) in shared memory by one thread, which also forms the weighted mean, nearest first.  There are no
// atomics and no reduction whose order depends on timing: the result is a function of the inputs.
#include "grid_index.cuh"

namespace pvraft {

constexpr int kPrWarps = 8;
constexpr int kPrThreads = kPrWarps * kWarp;
constexpr int kPrQueries = 2;                          // queries per lane, held in registers
constexpr int kPrPerCta = kWarp * kPrQueries;          // queries per CTA, searched by every warp
constexpr int kPrTile = 256;                           // warped points per shared-memory tile (two tiles)
constexpr int kPrSlice = kPrTile / kPrWarps;           // points of a tile each warp searches
constexpr int kPrMaxK = 8;
constexpr int kPrNone = 0x7fffffff;                    // index of an unfilled slot: loses every (distance, index) tie
static_assert(kPrTile == kPrThreads, "each thread stages one point per tile");

// The per-query step after the search, shared by k_flow_propagate and k_flow_propagate_grid: from the k nearest (nd, nx) of
// a query, nearest first, write its flow and neighbours at row `row`.
// w_j = 1 / (sqrt(d_j) + 1e-8); flow = sum_j w_j flow_prev[j] / sum_j w_j, summed nearest first.  An unfilled slot (only
// possible when non-finite coordinates leave fewer than K comparable points) contributes nothing and reads back as -1.
template <int K>
__device__ __forceinline__ void propagate_point(const float (&nd)[K], const int (&nx)[K], const float* fp, int M, long long row,
                                                float* flow_out, int32_t* idx_out) {
    float sw = 0.f, sx = 0.f, sy = 0.f, sz = 0.f;
#pragma unroll
    for (int r = 0; r < K; ++r) {
        const int j = nx[r];
        const bool ok = j < M;
        if (idx_out) idx_out[row * K + r] = ok ? j : -1;
        if (!ok) continue;
        const float w = __fdiv_rn(1.f, __fadd_rn(__fsqrt_rn(nd[r]), 1e-8f));
        sx = __fadd_rn(sx, __fmul_rn(w, __ldg(fp + 3ll * j)));
        sy = __fadd_rn(sy, __fmul_rn(w, __ldg(fp + 3ll * j + 1)));
        sz = __fadd_rn(sz, __fmul_rn(w, __ldg(fp + 3ll * j + 2)));
        sw = __fadd_rn(sw, w);
    }
    flow_out[3 * row] = __fdiv_rn(sx, sw);
    flow_out[3 * row + 1] = __fdiv_rn(sy, sw);
    flow_out[3 * row + 2] = __fdiv_rn(sz, sw);
}

// xyz_prev, flow_prev [B,M,3], xyz [B,N,3] -> flow_out [B,N,3], idx_out [B,N,K] (or NULL); grid (ceil(N / kPrPerCta), B)
template <int K>
__global__ void __launch_bounds__(kPrThreads) k_flow_propagate(const float* __restrict__ xyz_prev, const float* __restrict__ flow_prev,
                                                                const float* __restrict__ xyz, int M, int N, float* __restrict__ flow_out,
                                                                int32_t* __restrict__ idx_out) {
    __shared__ float4 tile[2][kPrTile];
    __shared__ float md[kPrWarps][K][kPrPerCta];       // every warp's k-best lists, [warp][rank][query]
    __shared__ int mi[kPrWarps][K][kPrPerCta];
    const int b = blockIdx.y;
    const float* pp = xyz_prev + (long long)b * M * 3;
    const float* fp = flow_prev + (long long)b * M * 3;
    const float* qp = xyz + (long long)b * N * 3;
    const int q0 = blockIdx.x * kPrPerCta;
    const int lane = lane_id(), warp = warp_id();

    float qx[kPrQueries], qy[kPrQueries], qz[kPrQueries], best[kPrQueries][K];
    int arg[kPrQueries][K];
#pragma unroll
    for (int i = 0; i < kPrQueries; ++i) {
        const int q = q0 + i * kWarp + lane;
        const bool ok = q < N;
        qx[i] = ok ? __ldg(qp + 3ll * q) : 0.f;
        qy[i] = ok ? __ldg(qp + 3ll * q + 1) : 0.f;
        qz[i] = ok ? __ldg(qp + 3ll * q + 2) : 0.f;
#pragma unroll
        for (int r = 0; r < K; ++r) {
            best[i][r] = INFINITY;
            arg[i][r] = kPrNone;
        }
    }

    // the next tile is fetched (and warped) into registers while the current one is searched; points past the end read as
    // NaN, whose distance never compares below a list entry
    float st[3];
    auto fetch = [&](int t) {
        const int p = t * kPrTile + threadIdx.x;
        const bool ok = p < M;
#pragma unroll
        for (int c = 0; c < 3; ++c) st[c] = ok ? __fadd_rn(__ldg(pp + 3ll * p + c), __ldg(fp + 3ll * p + c)) : NAN;
    };
    auto store = [&](int buf) { tile[buf][threadIdx.x] = make_float4(st[0], st[1], st[2], 0.f); };

    const int tiles = (M + kPrTile - 1) / kPrTile;
    fetch(0);
    store(0);
    __syncthreads();
    for (int t = 0; t < tiles; ++t) {
        const bool more = t + 1 < tiles;
        if (more) fetch(t + 1);
        const float4* tl = tile[t & 1] + warp * kPrSlice;
        const int base = t * kPrTile + warp * kPrSlice;
#pragma unroll 8
        for (int j = 0; j < kPrSlice; ++j) {
            const float4 p = tl[j];   // the same address in every lane: a broadcast
#pragma unroll
            for (int i = 0; i < kPrQueries; ++i) {
                const float d = diff_sq(qx[i], qy[i], qz[i], p);
                if (d < best[i][K - 1]) kbest_insert<K>(best[i], arg[i], d, base + j);
            }
        }
        if (more) store((t + 1) & 1);   // the buffer searched in iteration t - 1, released by its barrier
        __syncthreads();
    }

#pragma unroll
    for (int i = 0; i < kPrQueries; ++i)
#pragma unroll
        for (int r = 0; r < K; ++r) {
            md[warp][r][i * kWarp + lane] = best[i][r];
            mi[warp][r][i * kWarp + lane] = arg[i][r];
        }
    __syncthreads();
    const int t = threadIdx.x, q = q0 + t;
    if (t >= kPrPerCta || q >= N) return;

    // merge the warps' lists: each is ascending in (distance, index), so K times the least head wins
    float hd[kPrWarps];
    int hx[kPrWarps], pos[kPrWarps];
#pragma unroll
    for (int w = 0; w < kPrWarps; ++w) {
        pos[w] = 0;
        hd[w] = md[w][0][t];
        hx[w] = mi[w][0][t];
    }
    float nd[K];
    int nx[K];
#pragma unroll
    for (int r = 0; r < K; ++r) {
        int bw = 0;
        float bd = hd[0];
        int bx = hx[0];
#pragma unroll
        for (int w = 1; w < kPrWarps; ++w)
            if (hd[w] < bd || (hd[w] == bd && hx[w] < bx)) {
                bw = w;
                bd = hd[w];
                bx = hx[w];
            }
        nd[r] = bd;
        nx[r] = bx;
#pragma unroll
        for (int w = 0; w < kPrWarps; ++w)
            if (w == bw) {
                ++pos[w];
                hd[w] = pos[w] < K ? md[w][pos[w]][t] : INFINITY;
                hx[w] = pos[w] < K ? mi[w][pos[w]][t] : kPrNone;
            }
    }

    propagate_point<K>(nd, nx, fp, M, (long long)b * N + q, flow_out, idx_out);
}

template <int K>
static void launch_propagate(dim3 grid, cudaStream_t st, const float* xyz_prev, const float* flow_prev, const float* xyz, int M, int N,
                             float* flow_out, int32_t* idx_out) {
    k_flow_propagate<K><<<grid, kPrThreads, 0, st>>>(xyz_prev, flow_prev, xyz, M, N, flow_out, idx_out);
}

// The grid form of k_flow_propagate: the same search on the index `ix` of W = xyz_prev + flow_prev (built with flow_prev as
// its offset, the same fp32 add), the same propagate_point.  One warp per query, kGqPerWarp consecutive queries per warp.
template <int K>
__global__ void __launch_bounds__(kGqThreads) k_flow_propagate_grid(const float* __restrict__ flow_prev, const float* __restrict__ xyz, int M, int N,
                                                                     GridIndex ix, float* __restrict__ flow_out, int32_t* __restrict__ idx_out) {
    const int b = blockIdx.y;
    const int q0 = (blockIdx.x * kGqWarps + warp_id()) * kGqPerWarp;
    if (q0 >= N) return;   // uniform over the warp; no barrier follows
    const float* fp = flow_prev + (long long)b * M * 3;
    const float* qp = xyz + (long long)b * N * 3;
    const float4* P = ix.pts + (long long)b * M;
    const int32_t* I = ix.ids + (long long)b * M;
    const int32_t* CS = ix.cell_start + (long long)b * (ix.cells + 1);
    const GridParams gp = ix.params[b];
    for (int q = q0; q < min(q0 + kGqPerWarp, N); ++q) {
        float bd;
        int bi;
        grid_knn_diff(P, I, CS, gp, __ldg(qp + 3ll * q), __ldg(qp + 3ll * q + 1), __ldg(qp + 3ll * q + 2), K, bd, bi);
        float nd[K];
        int nx[K];
#pragma unroll
        for (int r = 0; r < K; ++r) {
            nd[r] = __shfl_sync(kFull, bd, r);
            nx[r] = __shfl_sync(kFull, bi, r);
        }
        if (lane_id() == 0) propagate_point<K>(nd, nx, fp, M, (long long)b * N + q, flow_out, idx_out);
    }
}

template <int K>
static void launch_propagate_grid(dim3 grid, cudaStream_t st, const float* flow_prev, const float* xyz, int M, int N, const GridIndex& ix,
                                  float* flow_out, int32_t* idx_out) {
    k_flow_propagate_grid<K><<<grid, kGqThreads, 0, st>>>(flow_prev, xyz, M, N, ix, flow_out, idx_out);
}

}  // namespace pvraft

using namespace pvraft;

extern "C" int pvraft_flow_propagate_fwd(const float* xyz_prev, const float* flow_prev, const float* xyz, int B, int M, int N, int k,
                                         float* flow_out, int32_t* idx_out, void* stream) {
    if (!xyz_prev || !flow_prev || !xyz || !flow_out || B < 1 || M < 1 || N < 1 || k < 1 || k > kPrMaxK || k > M)
        return fail(PVRAFT_ERR_BAD_ARG, "flow_propagate_fwd: bad argument");
    if (B > 65535) return fail(PVRAFT_ERR_UNSUPPORTED, "flow_propagate_fwd: B = %d samples (at most 65535)", B);
    const dim3 grid((unsigned)((N + kPrPerCta - 1) / kPrPerCta), (unsigned)B);
    cudaStream_t st = (cudaStream_t)stream;
    switch (k) {
        case 1: launch_propagate<1>(grid, st, xyz_prev, flow_prev, xyz, M, N, flow_out, idx_out); break;
        case 2: launch_propagate<2>(grid, st, xyz_prev, flow_prev, xyz, M, N, flow_out, idx_out); break;
        case 3: launch_propagate<3>(grid, st, xyz_prev, flow_prev, xyz, M, N, flow_out, idx_out); break;
        case 4: launch_propagate<4>(grid, st, xyz_prev, flow_prev, xyz, M, N, flow_out, idx_out); break;
        case 5: launch_propagate<5>(grid, st, xyz_prev, flow_prev, xyz, M, N, flow_out, idx_out); break;
        case 6: launch_propagate<6>(grid, st, xyz_prev, flow_prev, xyz, M, N, flow_out, idx_out); break;
        case 7: launch_propagate<7>(grid, st, xyz_prev, flow_prev, xyz, M, N, flow_out, idx_out); break;
        default: launch_propagate<8>(grid, st, xyz_prev, flow_prev, xyz, M, N, flow_out, idx_out); break;
    }
    return check_launch("flow_propagate_fwd");
}

extern "C" int pvraft_flow_propagate_grid_fwd(const float* xyz_prev, const float* flow_prev, const float* xyz, int B, int M, int N, int k,
                                              float* flow_out, int32_t* idx_out, void* workspace, void* stream) {
    if (!xyz_prev || !flow_prev || !xyz || !flow_out || !workspace || B < 1 || M < 1 || N < 1 || k < 1 || k > kPrMaxK || k > M)
        return fail(PVRAFT_ERR_BAD_ARG, "flow_propagate_grid_fwd: bad argument");
    if (B > 65535) return fail(PVRAFT_ERR_UNSUPPORTED, "flow_propagate_grid_fwd: B = %d samples (at most 65535)", B);
    cudaStream_t st = (cudaStream_t)stream;
    GridIndex ix;
    const int rc = grid_index_build(xyz_prev, flow_prev, B, M, workspace, st, &ix);
    if (rc) return rc;
    const dim3 grid((unsigned)((N + kGqPerCta - 1) / kGqPerCta), (unsigned)B);
    switch (k) {
        case 1: launch_propagate_grid<1>(grid, st, flow_prev, xyz, M, N, ix, flow_out, idx_out); break;
        case 2: launch_propagate_grid<2>(grid, st, flow_prev, xyz, M, N, ix, flow_out, idx_out); break;
        case 3: launch_propagate_grid<3>(grid, st, flow_prev, xyz, M, N, ix, flow_out, idx_out); break;
        case 4: launch_propagate_grid<4>(grid, st, flow_prev, xyz, M, N, ix, flow_out, idx_out); break;
        case 5: launch_propagate_grid<5>(grid, st, flow_prev, xyz, M, N, ix, flow_out, idx_out); break;
        case 6: launch_propagate_grid<6>(grid, st, flow_prev, xyz, M, N, ix, flow_out, idx_out); break;
        case 7: launch_propagate_grid<7>(grid, st, flow_prev, xyz, M, N, ix, flow_out, idx_out); break;
        default: launch_propagate_grid<8>(grid, st, flow_prev, xyz, M, N, ix, flow_out, idx_out); break;
    }
    return check_launch("flow_propagate_grid_fwd");
}
