// Flow propagation along a scan sequence (no counterpart in the reference): a flow defined on one cloud, flow_prev on
// xyz_prev, is carried onto the points of another cloud xyz under a constant-velocity assumption.  The previous points
// moved by their flow, W = xyz_prev + flow_prev (one fp32 add per coordinate, formed while staging, never stored), are
// searched for the k nearest of every query q of xyz, and q takes their inverse-distance-weighted mean flow.
//
// The search is the tiled brute-force K-best search of nn_search.cuh (tiled_kbest), in its difference form ranked on
// (distance, index): the lowest index wins an exact tie.  W is formed while staging the tiles.  The thread that owns a query
// then forms the weighted mean, nearest first.  There are no atomics: the result is a function of the inputs.
#include "grid_index.cuh"

namespace pvraft {

constexpr int kPrMaxK = 8;

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

// xyz_prev, flow_prev [B,M,3], xyz [B,N,3] -> flow_out [B,N,3], idx_out [B,N,K] (or NULL); grid (ceil(N / kKbPerCta), B)
template <int K>
__global__ void __launch_bounds__(kKbThreads) k_flow_propagate(const float* __restrict__ xyz_prev, const float* __restrict__ flow_prev,
                                                                const float* __restrict__ xyz, int M, int N, float* __restrict__ flow_out,
                                                                int32_t* __restrict__ idx_out) {
    const int b = blockIdx.y;
    const float* fp = flow_prev + (long long)b * M * 3;
    float nd[K];
    int nx[K];
    if (!tiled_kbest<K, true>(xyz + (long long)b * N * 3, N, xyz_prev + (long long)b * M * 3, fp, M, nd, nx)) return;
    const int q = blockIdx.x * kKbPerCta + threadIdx.x;
    if (q < N) propagate_point<K>(nd, nx, fp, M, (long long)b * N + q, flow_out, idx_out);
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

}  // namespace pvraft

using namespace pvraft;

extern "C" int pvraft_flow_propagate_fwd(const float* xyz_prev, const float* flow_prev, const float* xyz, int B, int M, int N, int k,
                                         float* flow_out, int32_t* idx_out, void* stream) {
    if (!xyz_prev || !flow_prev || !xyz || !flow_out || B < 1 || M < 1 || N < 1 || k < 1 || k > kPrMaxK || k > M)
        return fail(PVRAFT_ERR_BAD_ARG, "flow_propagate_fwd: bad argument");
    if (B > 65535) return fail(PVRAFT_ERR_UNSUPPORTED, "flow_propagate_fwd: B = %d samples (at most 65535)", B);
    const dim3 grid((unsigned)((N + kKbPerCta - 1) / kKbPerCta), (unsigned)B);
    cudaStream_t st = (cudaStream_t)stream;
    dispatch_k<kPrMaxK>(k, [&](auto kc) {
        k_flow_propagate<decltype(kc)::value><<<grid, kKbThreads, 0, st>>>(xyz_prev, flow_prev, xyz, M, N, flow_out, idx_out);
    });
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
    dispatch_k<kPrMaxK>(k, [&](auto kc) {
        k_flow_propagate_grid<decltype(kc)::value><<<grid, kGqThreads, 0, st>>>(flow_prev, xyz, M, N, ix, flow_out, idx_out);
    });
    return check_launch("flow_propagate_grid_fwd");
}
