// Self-supervised scene-flow losses on the device (the PointPWC-Net family of objectives, for scans without ground truth):
// the Chamfer distance between the first cloud moved by the flow, W = P1 + f, and the second cloud P2, and the smoothness of
// the flow over the first cloud's kNN graph.  Forward and backward, no host synchronisation inside a step (the upstream
// gradient is read from device memory), a DET form of every reduction (fixed_point.cuh).
//
// k_chamfer_nn is a brute-force nearest-neighbour search in the DIFFERENCE form, d = (dx*dx + dy*dy) + dz*dz of the fp32
// difference vector, rounded to nearest at every step and never contracted into an FMA; ties go to the lowest index.  Why
// not pvraft_knn_fwd with k = 1: that kernel ranks by the graph's expanded form |q|^2 + |x|^2 - 2 q.x (model/flot/graph.py:53-57,
// which it must reproduce).  For a LiDAR scan tens of metres from the origin the three terms are ~1e3 and cancel down to an
// error of ~1e-4, comparable to the squared nearest-neighbour distances the Chamfer term sums; its warp-per-query sorted
// list is also built for k = 32, not for one neighbour.  Here each thread keeps several queries and their running minimum
// and argmin in registers while the other cloud streams through shared memory in double-buffered tiles; one launch searches
// both directions (blockIdx.z) for every prediction of a sequence (blockIdx.y = sample s, which searches b[s % B]).
#include "fixed_point.cuh"
#include "grid_index.cuh"

namespace pvraft {

constexpr int kNnThreads = 128;
constexpr int kNnQueries = 4;                          // queries per thread, held in registers
constexpr int kNnPerCta = kNnThreads * kNnQueries;
constexpr int kNnTile = 256;                           // searched points per shared-memory tile (two tiles)
constexpr int kNnStage = kNnTile / kNnThreads;         // points each thread stages per tile

// a [S,N,3], b [B,M,3].  z = 0: every a-point of sample s queries b[s % B] -> nn_ab [S,N], acc[2s] += sum of the minima;
// z = 1: every b-point queries a[s] -> nn_ba [S,M], acc[2s + 1].  DET: acc is the [2S] fixed-point workspace.  What a warp
// sums (its lanes' kNnQueries minima) is fixed by the shapes.
template <bool DET>
__global__ void __launch_bounds__(kNnThreads) k_chamfer_nn(const float* __restrict__ a, const float* __restrict__ b, int B, int N, int M,
                                                          int32_t* __restrict__ nn_ab, int32_t* __restrict__ nn_ba, double* __restrict__ acc) {
    __shared__ float4 tile[2][kNnTile];
    const int s = blockIdx.y, dir = blockIdx.z;
    const float* pa = a + (long long)s * N * 3;
    const float* pb = b + (long long)(s % B) * M * 3;
    const float* qry = dir ? pb : pa;
    const float* cld = dir ? pa : pb;
    const int nq = dir ? M : N, nc = dir ? N : M;
    int32_t* out = dir ? nn_ba + (long long)s * M : nn_ab + (long long)s * N;
    const int q0 = blockIdx.x * kNnPerCta;
    if (q0 >= nq) return;   // uniform over the CTA, before any barrier

    float qx[kNnQueries], qy[kNnQueries], qz[kNnQueries], best[kNnQueries];
    int arg[kNnQueries];
#pragma unroll
    for (int k = 0; k < kNnQueries; ++k) {
        const int q = q0 + k * kNnThreads + threadIdx.x;
        const bool ok = q < nq;
        qx[k] = ok ? __ldg(qry + 3ll * q) : 0.f;
        qy[k] = ok ? __ldg(qry + 3ll * q + 1) : 0.f;
        qz[k] = ok ? __ldg(qry + 3ll * q + 2) : 0.f;
        best[k] = INFINITY;
        arg[k] = 0;
    }

    // the next tile is fetched into registers while the current one is searched; points past the end read as NaN, whose
    // distance never compares below the running minimum
    float st[kNnStage][3];
    auto fetch = [&](int t) {
#pragma unroll
        for (int r = 0; r < kNnStage; ++r) {
            const int p = t * kNnTile + r * kNnThreads + threadIdx.x;
            const bool ok = p < nc;
            st[r][0] = ok ? __ldg(cld + 3ll * p) : NAN;
            st[r][1] = ok ? __ldg(cld + 3ll * p + 1) : NAN;
            st[r][2] = ok ? __ldg(cld + 3ll * p + 2) : NAN;
        }
    };
    auto store = [&](int buf) {
#pragma unroll
        for (int r = 0; r < kNnStage; ++r) tile[buf][r * kNnThreads + threadIdx.x] = make_float4(st[r][0], st[r][1], st[r][2], 0.f);
    };

    const int tiles = (nc + kNnTile - 1) / kNnTile;
    fetch(0);
    store(0);
    __syncthreads();
    for (int t = 0; t < tiles; ++t) {
        const bool more = t + 1 < tiles;
        if (more) fetch(t + 1);
        const float4* tl = tile[t & 1];
        const int base = t * kNnTile;
#pragma unroll 8
        for (int j = 0; j < kNnTile; ++j) {
            const float4 p = tl[j];   // the same address in every lane: a broadcast
#pragma unroll
            for (int k = 0; k < kNnQueries; ++k) {
                const float d = diff_sq(qx[k], qy[k], qz[k], p);
                if (d < best[k]) {   // strict: candidates arrive in ascending index order, so ties keep the lowest
                    best[k] = d;
                    arg[k] = base + j;
                }
            }
        }
        if (more) store((t + 1) & 1);   // the buffer searched in iteration t - 1, released by its barrier
        __syncthreads();
    }

    double sum = 0.0;
#pragma unroll
    for (int k = 0; k < kNnQueries; ++k) {
        const int q = q0 + k * kNnThreads + threadIdx.x;
        if (q < nq) {
            out[q] = arg[k];
            sum += (double)best[k];
        }
    }
    sum = warp_sum(sum);
    if (lane_id() == 0 && sum != 0.0) {
        if constexpr (DET) fx_atomic(reinterpret_cast<unsigned long long*>(acc) + (2ll * s + dir) * kFxWords, sum);
        else atomicAdd(acc + 2 * s + dir, sum);
    }
}

// The grid form of k_chamfer_nn: the same nn_ab, nn_ba and minima, searched on the index ib of b (B samples) for z = 0 and
// the index ia of a (S samples) for z = 1.  One warp per query, kGqPerWarp consecutive queries per warp; lane 0 sums the
// warp's minima in query order, so what a warp sums is fixed by the shapes.  A query with no finite distance gets index 0
// and an infinite minimum, as in k_chamfer_nn.
template <bool DET>
__global__ void __launch_bounds__(kGqThreads) k_chamfer_grid(const float* __restrict__ a, const float* __restrict__ b, int B, int N, int M,
                                                              GridIndex ib, GridIndex ia, int32_t* __restrict__ nn_ab, int32_t* __restrict__ nn_ba,
                                                              double* __restrict__ acc) {
    const int s = blockIdx.y, dir = blockIdx.z;
    const int nq = dir ? M : N, nc = dir ? N : M;
    const int q0 = (blockIdx.x * kGqWarps + warp_id()) * kGqPerWarp;
    if (q0 >= nq) return;   // uniform over the warp; no barrier follows
    const float* qry = dir ? b + (long long)(s % B) * M * 3 : a + (long long)s * N * 3;
    int32_t* out = dir ? nn_ba + (long long)s * M : nn_ab + (long long)s * N;
    const int t = dir ? s : s % B;   // the searched sample of its index
    const float4* P = (dir ? ia.pts : ib.pts) + (long long)t * nc;
    const int32_t* I = (dir ? ia.ids : ib.ids) + (long long)t * nc;
    const int32_t* CS = (dir ? ia.cell_start : ib.cell_start) + (long long)t * ((dir ? ia.cells : ib.cells) + 1);
    const GridParams gp = (dir ? ia.params : ib.params)[t];
    double sum = 0.0;
    for (int q = q0; q < min(q0 + kGqPerWarp, nq); ++q) {
        float bd;
        int bi;
        grid_knn_diff(P, I, CS, gp, __ldg(qry + 3ll * q), __ldg(qry + 3ll * q + 1), __ldg(qry + 3ll * q + 2), 1, bd, bi);
        if (lane_id() == 0) {
            out[q] = bi < nc ? bi : 0;
            sum += (double)bd;
        }
    }
    if (lane_id() == 0 && sum != 0.0) {
        if constexpr (DET) fx_atomic(reinterpret_cast<unsigned long long*>(acc) + (2ll * s + dir) * kFxWords, sum);
        else atomicAdd(acc + 2 * s + dir, sum);
    }
}

// Items [0, S*N): d_a[s,i] += v, d_b[s%B, nn_ab] -= v with v = 2 g_s / N (a_i - b_nn); items [S*N, S*N + S*M):
// d_a[s, nn_ba] += v, d_b[s%B, j] -= v with v = 2 g_s / M (a_nn - b_j).  d_b may be NULL.  DET: d_a and d_b are the
// fixed-point workspaces; every value added is one item's.
template <bool DET>
__global__ void __launch_bounds__(256) k_chamfer_bwd(const float* __restrict__ a, const float* __restrict__ b, const int32_t* __restrict__ nn_ab,
                                                     const int32_t* __restrict__ nn_ba, const float* __restrict__ g, int B, int N, int M,
                                                     long long items_a, long long items, float* __restrict__ d_a, float* __restrict__ d_b) {
    for (long long it = (long long)blockIdx.x * blockDim.x + threadIdx.x; it < items; it += (long long)gridDim.x * blockDim.x) {
        long long ia, ib;
        float c;
        if (it < items_a) {
            const int s = (int)(it / N);
            ia = it;
            ib = (long long)(s % B) * M + __ldg(nn_ab + it);
            c = 2.f * __ldg(g + s) / (float)N;
        } else {
            const long long r = it - items_a;
            const int s = (int)(r / M);
            ib = (long long)(s % B) * M + (r - (long long)s * M);
            ia = (long long)s * N + __ldg(nn_ba + r);
            c = 2.f * __ldg(g + s) / (float)M;
        }
#pragma unroll
        for (int x = 0; x < 3; ++x) {
            const float v = c * (__ldg(a + 3 * ia + x) - __ldg(b + 3 * ib + x));
            scatter_add<DET>(d_a, 3 * ia + x, v);
            if (d_b) scatter_add<DET>(d_b, 3 * ib + x, -v);
        }
    }
}

// f [S,N,3], nbr [B,N,k] (sample s uses nbr[s % B]) -> acc[s] += sum_i sum_e ||f[nbr[i,e]] - f[i]||, grid (x, S).  A point's
// k lengths are summed in double in edge order; DET: acc is the [S] fixed-point workspace and the grid's x extent is
// capped by a constant, so what a warp sums is fixed by the shapes.
template <bool DET>
__global__ void __launch_bounds__(256) k_flow_smooth_fwd(const float* __restrict__ f, const int32_t* __restrict__ nbr, int B, int N, int k,
                                                         double* __restrict__ acc) {
    const int s = blockIdx.y;
    const float* fs = f + (long long)s * N * 3;
    const int32_t* ns = nbr + (long long)(s % B) * N * k;
    double sum = 0.0;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < N; i += gridDim.x * blockDim.x) {
        const float fx = __ldg(fs + 3ll * i), fy = __ldg(fs + 3ll * i + 1), fz = __ldg(fs + 3ll * i + 2);
        for (int e = 0; e < k; ++e) {
            const long long j = __ldg(ns + (long long)i * k + e);
            const float4 d = make_float4(__ldg(fs + 3 * j), __ldg(fs + 3 * j + 1), __ldg(fs + 3 * j + 2), 0.f);
            sum += (double)sqrtf(diff_sq(fx, fy, fz, d));
        }
    }
    sum = warp_sum(sum);
    if (lane_id() == 0 && sum != 0.0) {
        if constexpr (DET) fx_atomic(reinterpret_cast<unsigned long long*>(acc) + (long long)s * kFxWords, sum);
        else atomicAdd(acc + s, sum);
    }
}

// d_f[s,j] += u, d_f[s,i] -= u for every edge (i, j = nbr[i,e]), u = g_s / (N k) (f_j - f_i) / ||f_j - f_i|| (0 where f_j = f_i,
// self edges included).  One thread per point: the scattered +u per edge, then the point's own -sum_e u (edge order).
template <bool DET>
__global__ void __launch_bounds__(256) k_flow_smooth_bwd(const float* __restrict__ f, const int32_t* __restrict__ nbr, const float* __restrict__ g,
                                                         int B, int N, int k, long long points, float* __restrict__ d_f) {
    for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < points; p += (long long)gridDim.x * blockDim.x) {
        const int s = (int)(p / N);
        const long long i = p - (long long)s * N;
        const long long row = (long long)s * N;
        const int32_t* ni = nbr + ((long long)(s % B) * N + i) * k;
        const float scale = __ldg(g + s) / ((float)N * (float)k);
        const float fx = __ldg(f + 3 * p), fy = __ldg(f + 3 * p + 1), fz = __ldg(f + 3 * p + 2);
        float ox = 0.f, oy = 0.f, oz = 0.f;
        for (int e = 0; e < k; ++e) {
            const long long j = row + __ldg(ni + e);
            const float dx = __ldg(f + 3 * j) - fx, dy = __ldg(f + 3 * j + 1) - fy, dz = __ldg(f + 3 * j + 2) - fz;
            const float n2 = __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
            if (!(n2 > 0.f)) continue;
            const float r = scale / sqrtf(n2);
            const float ux = dx * r, uy = dy * r, uz = dz * r;
            scatter_add<DET>(d_f, 3 * j, ux);
            scatter_add<DET>(d_f, 3 * j + 1, uy);
            scatter_add<DET>(d_f, 3 * j + 2, uz);
            ox -= ux;
            oy -= uy;
            oz -= uz;
        }
        scatter_add<DET>(d_f, 3 * p, ox);
        scatter_add<DET>(d_f, 3 * p + 1, oy);
        scatter_add<DET>(d_f, 3 * p + 2, oz);
    }
}

static bool bad_batch(int S, int B, int N) { return S < 1 || B < 1 || S % B != 0 || N < 1; }

}  // namespace pvraft

using namespace pvraft;

extern "C" int pvraft_chamfer_fwd(const float* a, const float* b, int S, int B, int N, int M, int32_t* nn_ab, int32_t* nn_ba, double* acc,
                                  void* det_workspace, void* stream) {
    if (!a || !b || !nn_ab || !nn_ba || !acc || bad_batch(S, B, N) || M < 1) return fail(PVRAFT_ERR_BAD_ARG, "chamfer_fwd: bad argument");
    if (S > 65535) return fail(PVRAFT_ERR_UNSUPPORTED, "chamfer_fwd: S = %d samples (at most 65535)", S);
    const int nmax = N > M ? N : M;
    const dim3 grid((unsigned)((nmax + kNnPerCta - 1) / kNnPerCta), (unsigned)S, 2);
    cudaStream_t st = (cudaStream_t)stream;
    if (!det_workspace) {
        k_chamfer_nn<false><<<grid, kNnThreads, 0, st>>>(a, b, B, N, M, nn_ab, nn_ba, acc);
        return check_launch("chamfer_fwd");
    }
    k_chamfer_nn<true><<<grid, kNnThreads, 0, st>>>(a, b, B, N, M, nn_ab, nn_ba, static_cast<double*>(det_workspace));
    const int rc = check_launch("chamfer_fwd");
    if (rc) return rc;
    return fx_flush_f64(static_cast<const unsigned long long*>(det_workspace), 1, 2ll * S, 2ll * S, 0, acc, st);
}

extern "C" int64_t pvraft_chamfer_fwd_det_workspace_bytes(int S) { return S < 1 ? 0 : 2ll * S * kFxWords * 8; }

extern "C" int64_t pvraft_chamfer_grid_workspace_bytes(int S, int B, int N, int M) {
    if (S < 1 || B < 1 || N < 1 || M < 1) return 0;
    return grid_index_bytes(B, M) + grid_index_bytes(S, N);
}

extern "C" int pvraft_chamfer_grid_fwd(const float* a, const float* b, int S, int B, int N, int M, int32_t* nn_ab, int32_t* nn_ba, double* acc,
                                       void* workspace, void* det_workspace, void* stream) {
    if (!a || !b || !nn_ab || !nn_ba || !acc || !workspace || bad_batch(S, B, N) || M < 1)
        return fail(PVRAFT_ERR_BAD_ARG, "chamfer_grid_fwd: bad argument");
    if (S > 65535) return fail(PVRAFT_ERR_UNSUPPORTED, "chamfer_grid_fwd: S = %d samples (at most 65535)", S);
    cudaStream_t st = (cudaStream_t)stream;
    GridIndex ib, ia;
    int rc = grid_index_build(b, nullptr, B, M, workspace, st, &ib);
    if (!rc) rc = grid_index_build(a, nullptr, S, N, static_cast<char*>(workspace) + grid_index_bytes(B, M), st, &ia);
    if (rc) return rc;
    const int nmax = N > M ? N : M;
    const dim3 grid((unsigned)((nmax + kGqPerCta - 1) / kGqPerCta), (unsigned)S, 2);
    if (!det_workspace) {
        k_chamfer_grid<false><<<grid, kGqThreads, 0, st>>>(a, b, B, N, M, ib, ia, nn_ab, nn_ba, acc);
        return check_launch("chamfer_grid_fwd");
    }
    k_chamfer_grid<true><<<grid, kGqThreads, 0, st>>>(a, b, B, N, M, ib, ia, nn_ab, nn_ba, static_cast<double*>(det_workspace));
    rc = check_launch("chamfer_grid_fwd");
    if (rc) return rc;
    return fx_flush_f64(static_cast<const unsigned long long*>(det_workspace), 1, 2ll * S, 2ll * S, 0, acc, st);
}

extern "C" int pvraft_chamfer_bwd(const float* a, const float* b, const int32_t* nn_ab, const int32_t* nn_ba, const float* g, int S, int B,
                                  int N, int M, float* d_a, float* d_b, void* det_workspace, void* stream) {
    if (!a || !b || !nn_ab || !nn_ba || !g || !d_a || bad_batch(S, B, N) || M < 1) return fail(PVRAFT_ERR_BAD_ARG, "chamfer_bwd: bad argument");
    const long long items_a = (long long)S * N, items = items_a + (long long)S * M;
    const bool det = det_workspace != nullptr;
    const unsigned blocks = (unsigned)scatter_blocks(items, det);
    cudaStream_t st = (cudaStream_t)stream;
    if (!det) {
        k_chamfer_bwd<false><<<blocks, 256, 0, st>>>(a, b, nn_ab, nn_ba, g, B, N, M, items_a, items, d_a, d_b);
        return check_launch("chamfer_bwd");
    }
    const long long na = 3 * items_a, nb = 3ll * B * M;
    float* ws_a = static_cast<float*>(det_workspace);
    float* ws_b = reinterpret_cast<float*>(static_cast<unsigned long long*>(det_workspace) + na * kFxWords);
    k_chamfer_bwd<true><<<blocks, 256, 0, st>>>(a, b, nn_ab, nn_ba, g, B, N, M, items_a, items, ws_a, d_b ? ws_b : nullptr);
    int rc = check_launch("chamfer_bwd");
    if (rc) return rc;
    rc = fx_flush_f32(reinterpret_cast<const unsigned long long*>(ws_a), 1, na, na, 0, d_a, st);
    if (rc || !d_b) return rc;
    return fx_flush_f32(reinterpret_cast<const unsigned long long*>(ws_b), 1, nb, nb, 0, d_b, st);
}

extern "C" int64_t pvraft_chamfer_bwd_det_workspace_bytes(int S, int B, int N, int M) {
    if (S < 1 || B < 1 || N < 1 || M < 1) return 0;
    return (3ll * S * N + 3ll * B * M) * kFxWords * 8;
}

extern "C" int pvraft_flow_smooth_fwd(const float* f, const int32_t* nbr, int S, int B, int N, int k, double* acc, void* det_workspace,
                                      void* stream) {
    if (!f || !nbr || !acc || bad_batch(S, B, N) || k < 1 || k > 32) return fail(PVRAFT_ERR_BAD_ARG, "flow_smooth_fwd: bad argument");
    if (S > 65535) return fail(PVRAFT_ERR_UNSUPPORTED, "flow_smooth_fwd: S = %d samples (at most 65535)", S);
    long long bx = (N + 255) / 256;
    if (bx > kDetCtas) bx = kDetCtas;   // a constant in both forms
    const dim3 grid((unsigned)bx, (unsigned)S);
    cudaStream_t st = (cudaStream_t)stream;
    if (!det_workspace) {
        k_flow_smooth_fwd<false><<<grid, 256, 0, st>>>(f, nbr, B, N, k, acc);
        return check_launch("flow_smooth_fwd");
    }
    k_flow_smooth_fwd<true><<<grid, 256, 0, st>>>(f, nbr, B, N, k, static_cast<double*>(det_workspace));
    const int rc = check_launch("flow_smooth_fwd");
    if (rc) return rc;
    return fx_flush_f64(static_cast<const unsigned long long*>(det_workspace), 1, S, S, 0, acc, st);
}

extern "C" int64_t pvraft_flow_smooth_fwd_det_workspace_bytes(int S) { return S < 1 ? 0 : (int64_t)S * kFxWords * 8; }

extern "C" int pvraft_flow_smooth_bwd(const float* f, const int32_t* nbr, const float* g, int S, int B, int N, int k, float* d_f,
                                      void* det_workspace, void* stream) {
    if (!f || !nbr || !g || !d_f || bad_batch(S, B, N) || k < 1 || k > 32) return fail(PVRAFT_ERR_BAD_ARG, "flow_smooth_bwd: bad argument");
    const long long points = (long long)S * N;
    const bool det = det_workspace != nullptr;
    const unsigned blocks = (unsigned)scatter_blocks(points, det);
    cudaStream_t st = (cudaStream_t)stream;
    if (!det) {
        k_flow_smooth_bwd<false><<<blocks, 256, 0, st>>>(f, nbr, g, B, N, k, points, d_f);
        return check_launch("flow_smooth_bwd");
    }
    k_flow_smooth_bwd<true><<<blocks, 256, 0, st>>>(f, nbr, g, B, N, k, points, static_cast<float*>(det_workspace));
    const int rc = check_launch("flow_smooth_bwd");
    if (rc) return rc;
    return fx_flush_f32(static_cast<const unsigned long long*>(det_workspace), 1, 3 * points, 3 * points, 0, d_f, st);
}

extern "C" int64_t pvraft_flow_smooth_bwd_det_workspace_bytes(int S, int N) { return S < 1 || N < 1 ? 0 : 3ll * S * N * kFxWords * 8; }
