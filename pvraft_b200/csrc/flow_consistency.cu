// The forward-backward consistency of a pair of flows (UnFlow's term and occlusion test, applied to scene flow): a point of
// P1 moved by the forward flow, W = P1 + f12, should be carried back to where it started by the reverse flow f21 found there.
//
//   bhat_i = sum_r w_r f21[j_r] / sum_r w_r,  w_r = 1 / (d_r + 1e-8)   j_r the k nearest of W_i in P2[s % B], d_r the squared
//            distance: the Laplacian term's interpolation (idw.cuh), bit for bit, with the reverse flow as its field
//   r_i    = f12_i + bhat_i                                             the round trip's residual
//   ok_i   = ||r_i||^2 < alpha (||f12_i||^2 + ||bhat_i||^2) + beta       UnFlow's criterion, in double on the fp32 vectors
//   F_s    = (1/N) sum_i ||r_i||^2
//
// k_flow_consistency_fwd searches P2 with the tiled brute-force K-best search (tiled_kbest), k_flow_consistency_grid with the
// grid shell walk (grid_knn_diff) on an index of P2; both return the same neighbours, so the same bits.  The thread that owns
// a query writes its neighbours, r_i and ok_i and adds ||r_i||^2 (in double) to the sample's sum; DET: into the fixed-point
// workspace, each warp's sum being a function of the shapes.
//
// Backward, with the neighbours held fixed: e_i = dF/dr_i = 2 g_s / N r_i.
//   d_f12_i = e_i, and d_W_i the distance terms of bhat (idw_bwd): both written once per point;
//   d_P2 the negated distance terms and d_f21[s, j_r] += (w_r / sum w) e_i, accumulated.
#include "grid_index.cuh"
#include "idw.cuh"

namespace pvraft {

// The per-query step after the search, shared by both forward kernels: from the k nearest (nd, nx) of w_q, nearest first,
// write nn_idx, res and ok of row `row` and return ||r||^2 in double.  fb is the reverse flow of the query's sample.
template <int K>
__device__ __forceinline__ double consistency_point(const float (&nd)[K], const int (&nx)[K], const float* f12, const float* fb, int M,
                                                    float alpha, float beta, long long row, int32_t* nn_idx, float* res, uint8_t* ok) {
    const float4 t = idw_sums<K>(nd, nx, fb, M, nn_idx + row * K);
    const float bx = __fdiv_rn(t.x, t.w), by = __fdiv_rn(t.y, t.w), bz = __fdiv_rn(t.z, t.w);
    const float fx = __ldg(f12 + 3 * row), fy = __ldg(f12 + 3 * row + 1), fz = __ldg(f12 + 3 * row + 2);
    const float rx = __fadd_rn(fx, bx), ry = __fadd_rn(fy, by), rz = __fadd_rn(fz, bz);
    res[3 * row] = rx;
    res[3 * row + 1] = ry;
    res[3 * row + 2] = rz;
    const double rr = ((double)rx * (double)rx + (double)ry * (double)ry) + (double)rz * (double)rz;
    const double ff = ((double)fx * (double)fx + (double)fy * (double)fy) + (double)fz * (double)fz;
    const double bb = ((double)bx * (double)bx + (double)by * (double)by) + (double)bz * (double)bz;
    ok[row] = rr < (double)alpha * (ff + bb) + (double)beta;
    return rr;
}

// w, f12 [S,N,3], p2 [B,M,3], f21 [S,M,3] (sample s searches entry s % B) -> nn_idx [S,N,K], res [S,N,3], ok [S,N],
// acc[s] += sum_i ||res_i||^2; grid (ceil(N / kKbPerCta), S).  DET: acc is the [S] fixed-point workspace.
template <int K, bool DET>
__global__ void __launch_bounds__(kKbThreads) k_flow_consistency_fwd(const float* __restrict__ w, const float* __restrict__ f12,
                                                                     const float* __restrict__ p2, const float* __restrict__ f21, int B,
                                                                     int N, int M, float alpha, float beta, int32_t* __restrict__ nn_idx,
                                                                     float* __restrict__ res, uint8_t* __restrict__ ok,
                                                                     Acc<DET, double> acc) {
    const int s = blockIdx.y, b = s % B;
    float nd[K];
    int nx[K];
    if (!tiled_kbest<K, false>(w + (long long)s * N * 3, N, p2 + (long long)b * M * 3, nullptr, M, nd, nx)) return;   // whole warps
    const int q = blockIdx.x * kKbPerCta + threadIdx.x;
    double part = 0.0;
    if (q < N) part = consistency_point<K>(nd, nx, f12, f21 + (long long)s * M * 3, M, alpha, beta, (long long)s * N + q, nn_idx, res, ok);
    part = warp_sum(part);
    if (lane_id() == 0 && part != 0.0) add(acc, s, part);
}

// The grid form: the same search on the index `ix` of p2 (B samples), the same consistency_point.  One warp per query
// (kGqPerWarp consecutive queries per warp); lane 0 forms each query's result and sums its queries' terms in order.
template <int K, bool DET>
__global__ void __launch_bounds__(kGqThreads) k_flow_consistency_grid(const float* __restrict__ w, const float* __restrict__ f12,
                                                                      const float* __restrict__ f21, int B, int N, int M, float alpha,
                                                                      float beta, GridIndex ix, int32_t* __restrict__ nn_idx,
                                                                      float* __restrict__ res, uint8_t* __restrict__ ok,
                                                                      Acc<DET, double> acc) {
    const int s = blockIdx.y, b = s % B;
    const int lane = lane_id();
    const int q0 = (blockIdx.x * kGqWarps + warp_id()) * kGqPerWarp;
    if (q0 >= N) return;   // uniform over the warp; no barrier follows
    const float* ws = w + (long long)s * N * 3;
    const float* fb = f21 + (long long)s * M * 3;
    const float4* P = ix.pts + (long long)b * M;
    const int32_t* I = ix.ids + (long long)b * M;
    const int32_t* CS = ix.cell_start + (long long)b * (ix.cells + 1);
    const GridParams gp = ix.params[b];
    double part = 0.0;
    for (int q = q0; q < min(q0 + kGqPerWarp, N); ++q) {
        float bd;
        int bi;
        grid_knn_diff(P, I, CS, gp, __ldg(ws + 3ll * q), __ldg(ws + 3ll * q + 1), __ldg(ws + 3ll * q + 2), K, bd, bi);
        float nd[K];
        int nx[K];
#pragma unroll
        for (int r = 0; r < K; ++r) {
            nd[r] = __shfl_sync(kFull, bd, r);
            nx[r] = __shfl_sync(kFull, bi, r);
        }
        if (lane == 0) part += consistency_point<K>(nd, nx, f12, fb, M, alpha, beta, (long long)s * N + q, nn_idx, res, ok);
    }
    if (lane == 0 && part != 0.0) add(acc, s, part);
}

// One thread per point (s, i): d_w and d_f12 [S,N,3] written, d_p2 [B,M,3] (or NULL) and d_f21 [S,M,3] accumulated, for the
// upstream gradient g [S] on the device.  k slots of nn_idx per point; a slot of -1 contributes nothing.  DET: d_p2 and d_f21
// are fixed-point workspaces.
template <bool DET>
__global__ void __launch_bounds__(256) k_flow_consistency_bwd(const float* __restrict__ w, const float* __restrict__ p2,
                                                              const float* __restrict__ f21, const int32_t* __restrict__ nn_idx,
                                                              const float* __restrict__ res, const float* __restrict__ g, int B, int N,
                                                              int M, int k, long long points, float* __restrict__ d_w,
                                                              float* __restrict__ d_f12, Acc<DET> d_p2, Acc<DET> d_f21) {
    for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < points; p += (long long)gridDim.x * blockDim.x) {
        const int s = (int)(p / N), b = s % B;
        const float c = 2.f * __ldg(g + s) / (float)N;
        const float ex = c * __ldg(res + 3 * p), ey = c * __ldg(res + 3 * p + 1), ez = c * __ldg(res + 3 * p + 2);
        d_f12[3 * p] = ex;
        d_f12[3 * p + 1] = ey;
        d_f12[3 * p + 2] = ez;
        float ox = 0.f, oy = 0.f, oz = 0.f;
        idw_bwd<DET>(__ldg(w + 3 * p), __ldg(w + 3 * p + 1), __ldg(w + 3 * p + 2), p2, f21, nn_idx, p, k, b, s, M, ex, ey, ez, ox, oy, oz,
                     d_p2, d_f21);
        d_w[3 * p] = ox;
        d_w[3 * p + 1] = oy;
        d_w[3 * p + 2] = oz;
    }
}

static bool bad_term(int S, int B, int N, int M, int k) {
    return S < 1 || B < 1 || S % B != 0 || N < 1 || M < 1 || k < 1 || k > kIdwMaxK || k > M;
}

static bool bad_criterion(float alpha, float beta) { return !(alpha >= 0.f) || !(beta >= 0.f) || isinf(alpha) || isinf(beta); }

// flow_consistency_bwd's workspace: [3 B M] slots for d_p2 | [3 S M] for d_f21
struct ConsistencyBwdWs {
    FxSlots d_p2, d_f21;
    int64_t bytes;
};
static ConsistencyBwdWs consistency_bwd_ws(void* ws, int S, int B, int M) {
    FxCarve c(ws);
    return {c.take(3ll * B * M), c.take(3ll * S * M), c.bytes()};
}

}  // namespace pvraft

using namespace pvraft;

extern "C" int pvraft_flow_consistency_fwd(const float* w, const float* f12, const float* p2, const float* f21, int S, int B, int N, int M,
                                           int k, float alpha, float beta, int32_t* nn_idx, float* res, uint8_t* ok, double* acc,
                                           void* det_workspace, void* stream) {
    if (!w || !f12 || !p2 || !f21 || !nn_idx || !res || !ok || !acc || bad_term(S, B, N, M, k) || bad_criterion(alpha, beta))
        return fail(PVRAFT_ERR_BAD_ARG, "flow_consistency_fwd: bad argument");
    if (S > 65535) return fail(PVRAFT_ERR_UNSUPPORTED, "flow_consistency_fwd: S = %d samples (at most 65535)", S);
    const dim3 grid((unsigned)((N + kKbPerCta - 1) / kKbPerCta), (unsigned)S);
    cudaStream_t st = (cudaStream_t)stream;
    const bool det = det_workspace != nullptr;
    dispatch_k<kIdwMaxK>(k, [&](auto kc) {
        constexpr int K = decltype(kc)::value;
        if (det) k_flow_consistency_fwd<K, true><<<grid, kKbThreads, 0, st>>>(w, f12, p2, f21, B, N, M, alpha, beta, nn_idx, res, ok,
                                                                               fx_slots(det_workspace));
        else k_flow_consistency_fwd<K, false><<<grid, kKbThreads, 0, st>>>(w, f12, p2, f21, B, N, M, alpha, beta, nn_idx, res, ok, acc);
    });
    const int rc = check_launch("flow_consistency_fwd");
    return rc || !det ? rc : fx_flush(fx_slots(det_workspace), S, acc, st);
}

extern "C" int64_t pvraft_flow_consistency_fwd_det_workspace_bytes(int S) { return S < 1 ? 0 : fx_bytes(S); }

extern "C" int pvraft_flow_consistency_grid_fwd(const float* w, const float* f12, const float* p2, const float* f21, int S, int B, int N,
                                                int M, int k, float alpha, float beta, int32_t* nn_idx, float* res, uint8_t* ok,
                                                double* acc, void* workspace, void* det_workspace, void* stream) {
    if (!w || !f12 || !p2 || !f21 || !nn_idx || !res || !ok || !acc || !workspace || bad_term(S, B, N, M, k) || bad_criterion(alpha, beta))
        return fail(PVRAFT_ERR_BAD_ARG, "flow_consistency_grid_fwd: bad argument");
    if (S > 65535) return fail(PVRAFT_ERR_UNSUPPORTED, "flow_consistency_grid_fwd: S = %d samples (at most 65535)", S);
    cudaStream_t st = (cudaStream_t)stream;
    GridIndex ix;
    int rc = grid_index_build(p2, nullptr, B, M, workspace, st, &ix);
    if (rc) return rc;
    const dim3 grid((unsigned)((N + kGqPerCta - 1) / kGqPerCta), (unsigned)S);
    const bool det = det_workspace != nullptr;
    dispatch_k<kIdwMaxK>(k, [&](auto kc) {
        constexpr int K = decltype(kc)::value;
        if (det) k_flow_consistency_grid<K, true><<<grid, kGqThreads, 0, st>>>(w, f12, f21, B, N, M, alpha, beta, ix, nn_idx, res, ok,
                                                                                fx_slots(det_workspace));
        else k_flow_consistency_grid<K, false><<<grid, kGqThreads, 0, st>>>(w, f12, f21, B, N, M, alpha, beta, ix, nn_idx, res, ok, acc);
    });
    rc = check_launch("flow_consistency_grid_fwd");
    return rc || !det ? rc : fx_flush(fx_slots(det_workspace), S, acc, st);
}

extern "C" int pvraft_flow_consistency_bwd(const float* w, const float* p2, const float* f21, const int32_t* nn_idx, const float* res,
                                           const float* g, int S, int B, int N, int M, int k, float* d_w, float* d_f12, float* d_p2,
                                           float* d_f21, void* det_workspace, void* stream) {
    if (!w || !p2 || !f21 || !nn_idx || !res || !g || !d_w || !d_f12 || !d_f21 || bad_term(S, B, N, M, k))
        return fail(PVRAFT_ERR_BAD_ARG, "flow_consistency_bwd: bad argument");
    const long long points = (long long)S * N;
    const bool det = det_workspace != nullptr;
    const unsigned blocks = (unsigned)scatter_blocks(points, det);
    cudaStream_t st = (cudaStream_t)stream;
    if (!det) {
        k_flow_consistency_bwd<false><<<blocks, 256, 0, st>>>(w, p2, f21, nn_idx, res, g, B, N, M, k, points, d_w, d_f12, d_p2, d_f21);
        return check_launch("flow_consistency_bwd");
    }
    const ConsistencyBwdWs L = consistency_bwd_ws(det_workspace, S, B, M);
    k_flow_consistency_bwd<true><<<blocks, 256, 0, st>>>(w, p2, f21, nn_idx, res, g, B, N, M, k, points, d_w, d_f12,
                                                         d_p2 ? L.d_p2 : FxSlots{}, L.d_f21);
    int rc = check_launch("flow_consistency_bwd");
    if (!rc && d_p2) rc = fx_flush(L.d_p2, 3ll * B * M, d_p2, st);
    if (!rc) rc = fx_flush(L.d_f21, 3ll * S * M, d_f21, st);
    return rc;
}

extern "C" int64_t pvraft_flow_consistency_bwd_det_workspace_bytes(int S, int B, int M) {
    return S < 1 || B < 1 || M < 1 ? 0 : consistency_bwd_ws(nullptr, S, B, M).bytes;
}
