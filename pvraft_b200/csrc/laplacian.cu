// The Laplacian regularity term of the self-supervised loss (PointPWC-Net's third term): the local shape of the first cloud
// moved by the flow, W = P1 + f, should match the local shape of the second cloud P2 around the same place.
//
//   L(X)_i = sum_{j in G(i)} (X_j - X_i) / (k_lap - 1)   over a kNN graph G that contains the point itself (contributing 0)
//   L2     = L(P2) over G2 = knn(P2, P2, k_lap)          once per call, shared by every prediction of batch entry b
//   Lhat_i = sum_r w_r L2[j_r] / sum_r w_r,  w_r = 1 / (d_r + 1e-8)   j_r the k_int nearest of W_i in P2[s % B], d_r the
//            squared distance (the weighting of PointPWC-Net's curvature interpolation; not k_flow_propagate's 1/(sqrt(d)+1e-8))
//   R_s    = (1/N) sum_i ||Lhat_i - L(W)_i||^2,  L(W) over G1 = knn(P1, P1, k_lap): neighbours of the un-moved cloud, values of W
//
// k_laplacian_fwd does the search in the structure of k_flow_propagate: the difference form of nn_search.cuh ranked on
// (distance, index), kLpPerCta queries per CTA held in registers by every warp while P2 streams through double-buffered
// shared-memory tiles, warp w searching the w-th slice of each tile with a sorted K-best list per query, and the eight lists
// merged on (distance, index) in shared memory at the end.  The thread that owns a query then interpolates L2, gathers L(W)_i
// over G1, writes the residual Lhat_i - L(W)_i and its neighbours for the backward pass, and adds its squared length (in
// double) to the sample's sum; DET: into the fixed-point workspace, each warp's sum being a function of the shapes.
//
// Backward, with the neighbours held fixed: e_i = dR/d(residual_i) = 2 g_s / N (Lhat_i - L(W)_i).
//   through L(W):  -e_i / (k_lap - 1) at every neighbour j != i of G1(i), +e_i / (k_lap - 1) per such edge at i;
//   through Lhat:  dLhat/dL2[j_m] = w_m / sum w, and dLhat/dd_m = -(w_m^2 / sum w) (L2_m - Lhat) = -(w_m / sum w)^2 sum_r w_r
//                  (L2_m - L2_r).  Evaluating L2_m - Lhat as that weighted sum of differences keeps it accurate when one
//                  weight dominates (a duplicated point: d = 0, w = 1e8), where Lhat and L2_m agree to nearly every bit and
//                  their difference, multiplied by w_m^2 / sum w ~ 1e8, would be rounding noise.
//                  dd_m/dW_i = 2 (W_i - P2_m) = -dd_m/dP2_m.
//   k_cloud_laplacian_bwd carries dL2 into P2 over G2.
#include "fixed_point.cuh"
#include "grid_index.cuh"

namespace pvraft {

constexpr int kLpWarps = 8;
constexpr int kLpThreads = kLpWarps * kWarp;
constexpr int kLpQueries = 2;                          // queries per lane, held in registers
constexpr int kLpPerCta = kWarp * kLpQueries;          // queries per CTA, searched by every warp
constexpr int kLpTile = 256;                           // searched points per shared-memory tile (two tiles)
constexpr int kLpSlice = kLpTile / kLpWarps;           // points of a tile each warp searches
constexpr int kLpMaxK = 8;                             // interpolation neighbours k_int
constexpr int kLpMaxGraph = 32;                        // graph neighbours k_lap (the kNN kernel's limit)
constexpr int kLpNone = 0x7fffffff;                    // index of an unfilled slot: loses every (distance, index) tie
static_assert(kLpTile == kLpThreads, "each thread stages one point per tile");
static_assert(kLpPerCta % kWarp == 0, "the merging threads are whole warps");

// L(x)_i over the graph row nbr_i (k ids into x): the fp32 differences summed in edge order, then divided by k - 1.  A self
// edge adds an exact zero.
__device__ __forceinline__ float3 laplacian_at(const float* __restrict__ x, const int32_t* __restrict__ nbr_i, int k, long long i) {
    const float xi = __ldg(x + 3 * i), yi = __ldg(x + 3 * i + 1), zi = __ldg(x + 3 * i + 2);
    float sx = 0.f, sy = 0.f, sz = 0.f;
    for (int e = 0; e < k; ++e) {
        const long long j = __ldg(nbr_i + e);
        sx = __fadd_rn(sx, __fsub_rn(__ldg(x + 3 * j), xi));
        sy = __fadd_rn(sy, __fsub_rn(__ldg(x + 3 * j + 1), yi));
        sz = __fadd_rn(sz, __fsub_rn(__ldg(x + 3 * j + 2), zi));
    }
    const float den = (float)(k - 1);
    return make_float3(__fdiv_rn(sx, den), __fdiv_rn(sy, den), __fdiv_rn(sz, den));
}

// x [B,N,3], nbr [B,N,k] -> out [B,N,3] = L(x); one thread per point, every output written once
__global__ void __launch_bounds__(256) k_cloud_laplacian(const float* __restrict__ x, const int32_t* __restrict__ nbr, int N, int k,
                                                         long long points, float* __restrict__ out) {
    for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < points; p += (long long)gridDim.x * blockDim.x) {
        const long long b = p / N;
        const float3 l = laplacian_at(x + b * N * 3, nbr + p * k, k, p - b * N);
        out[3 * p] = l.x;
        out[3 * p + 1] = l.y;
        out[3 * p + 2] = l.z;
    }
}

// d_x [B,N,3] += the gradient of L(x) for the upstream gradient g_l [B,N,3]: c = g_l[i] / (k - 1) at every neighbour j != i,
// -c per such edge at i.  DET: d_x is the fixed-point workspace.
template <bool DET>
__global__ void __launch_bounds__(256) k_cloud_laplacian_bwd(const float* __restrict__ g_l, const int32_t* __restrict__ nbr, int N, int k,
                                                             long long points, float* __restrict__ d_x) {
    const float den = (float)(k - 1);
    for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < points; p += (long long)gridDim.x * blockDim.x) {
        const long long b = p / N, i = p - b * N;
        const float cx = __fdiv_rn(__ldg(g_l + 3 * p), den), cy = __fdiv_rn(__ldg(g_l + 3 * p + 1), den),
                    cz = __fdiv_rn(__ldg(g_l + 3 * p + 2), den);
        float ox = 0.f, oy = 0.f, oz = 0.f;
        for (int e = 0; e < k; ++e) {
            const long long j = __ldg(nbr + p * k + e);
            if (j == i) continue;
            const long long r = 3 * (b * N + j);
            scatter_add<DET>(d_x, r, cx);
            scatter_add<DET>(d_x, r + 1, cy);
            scatter_add<DET>(d_x, r + 2, cz);
            ox -= cx;
            oy -= cy;
            oz -= cz;
        }
        scatter_add<DET>(d_x, 3 * p, ox);
        scatter_add<DET>(d_x, 3 * p + 1, oy);
        scatter_add<DET>(d_x, 3 * p + 2, oz);
    }
}

// The per-query step of k_laplacian_grid after its search, the same formula, order and rounding as k_laplacian_fwd's (which
// keeps its own copy, so that its machine code is unchanged): from the k_int nearest (nd, nx) of w_q, nearest first, write
// nn_idx and the residual of row `row` and return its squared length in double.
// Lhat = sum_r w_r L2[j_r] / sum_r w_r, summed in fp32 nearest first.  An unfilled slot (only possible when non-finite
// coordinates leave fewer than K comparable points) contributes nothing and reads back as -1.
template <int K>
__device__ __forceinline__ double laplacian_point(const float (&nd)[K], const int (&nx)[K], const float* ws,
                                                  const float* lp, const int32_t* g1_q, int kl, int M, long long row,
                                                  int q, int32_t* nn_idx, float* res) {
    float sw = 0.f, sx = 0.f, sy = 0.f, sz = 0.f;
#pragma unroll
    for (int r = 0; r < K; ++r) {
        const int j = nx[r];
        const bool ok = j < M;
        nn_idx[row * K + r] = ok ? j : -1;
        if (!ok) continue;
        const float wr = __fdiv_rn(1.f, __fadd_rn(nd[r], 1e-8f));
        sx = __fadd_rn(sx, __fmul_rn(wr, __ldg(lp + 3ll * j)));
        sy = __fadd_rn(sy, __fmul_rn(wr, __ldg(lp + 3ll * j + 1)));
        sz = __fadd_rn(sz, __fmul_rn(wr, __ldg(lp + 3ll * j + 2)));
        sw = __fadd_rn(sw, wr);
    }
    const float3 lw = laplacian_at(ws, g1_q, kl, q);
    const float rx = __fsub_rn(__fdiv_rn(sx, sw), lw.x), ry = __fsub_rn(__fdiv_rn(sy, sw), lw.y),
                rz = __fsub_rn(__fdiv_rn(sz, sw), lw.z);
    res[3 * row] = rx;
    res[3 * row + 1] = ry;
    res[3 * row + 2] = rz;
    return ((double)rx * (double)rx + (double)ry * (double)ry) + (double)rz * (double)rz;
}

// w [S,N,3], p2 and l2 [B,M,3], g1 [B,N,kl] (sample s uses entry s % B) -> nn_idx [S,N,K], res [S,N,3] = Lhat - L(w),
// acc[s] += sum_i ||res_i||^2; grid (ceil(N / kLpPerCta), S).  DET: acc is the [S] fixed-point workspace.
template <int K, bool DET>
__global__ void __launch_bounds__(kLpThreads) k_laplacian_fwd(const float* __restrict__ w, const float* __restrict__ p2, const float* __restrict__ l2,
                                                               const int32_t* __restrict__ g1, int B, int N, int M, int kl,
                                                               int32_t* __restrict__ nn_idx, float* __restrict__ res, double* __restrict__ acc) {
    __shared__ float4 tile[2][kLpTile];
    __shared__ float md[kLpWarps][K][kLpPerCta];       // every warp's k-best lists, [warp][rank][query]
    __shared__ int mi[kLpWarps][K][kLpPerCta];
    const int s = blockIdx.y, b = s % B;
    const float* ws = w + (long long)s * N * 3;
    const float* cp = p2 + (long long)b * M * 3;
    const float* lp = l2 + (long long)b * M * 3;
    const int q0 = blockIdx.x * kLpPerCta;
    const int lane = lane_id(), warp = warp_id();

    float qx[kLpQueries], qy[kLpQueries], qz[kLpQueries], best[kLpQueries][K];
    int arg[kLpQueries][K];
#pragma unroll
    for (int i = 0; i < kLpQueries; ++i) {
        const int q = q0 + i * kWarp + lane;
        const bool ok = q < N;
        qx[i] = ok ? __ldg(ws + 3ll * q) : 0.f;
        qy[i] = ok ? __ldg(ws + 3ll * q + 1) : 0.f;
        qz[i] = ok ? __ldg(ws + 3ll * q + 2) : 0.f;
#pragma unroll
        for (int r = 0; r < K; ++r) {
            best[i][r] = INFINITY;
            arg[i][r] = kLpNone;
        }
    }

    // the next tile is fetched into registers while the current one is searched; points past the end read as NaN, whose
    // distance never compares below a list entry
    float st[3];
    auto fetch = [&](int t) {
        const int p = t * kLpTile + threadIdx.x;
        const bool ok = p < M;
#pragma unroll
        for (int c = 0; c < 3; ++c) st[c] = ok ? __ldg(cp + 3ll * p + c) : NAN;
    };
    auto store = [&](int buf) { tile[buf][threadIdx.x] = make_float4(st[0], st[1], st[2], 0.f); };

    const int tiles = (M + kLpTile - 1) / kLpTile;
    fetch(0);
    store(0);
    __syncthreads();
    for (int t = 0; t < tiles; ++t) {
        const bool more = t + 1 < tiles;
        if (more) fetch(t + 1);
        const float4* tl = tile[t & 1] + warp * kLpSlice;
        const int base = t * kLpTile + warp * kLpSlice;
#pragma unroll 8
        for (int j = 0; j < kLpSlice; ++j) {
            const float4 p = tl[j];   // the same address in every lane: a broadcast
#pragma unroll
            for (int i = 0; i < kLpQueries; ++i) {
                const float d = diff_sq(qx[i], qy[i], qz[i], p);
                if (d < best[i][K - 1]) kbest_insert<K>(best[i], arg[i], d, base + j);
            }
        }
        if (more) store((t + 1) & 1);   // the buffer searched in iteration t - 1, released by its barrier
        __syncthreads();
    }

#pragma unroll
    for (int i = 0; i < kLpQueries; ++i)
#pragma unroll
        for (int r = 0; r < K; ++r) {
            md[warp][r][i * kWarp + lane] = best[i][r];
            mi[warp][r][i * kWarp + lane] = arg[i][r];
        }
    __syncthreads();
    const int t = threadIdx.x, q = q0 + t;
    if (t >= kLpPerCta) return;   // whole warps; the rest stay for the warp sum

    double part = 0.0;
    if (q < N) {
        // merge the warps' lists: each is ascending in (distance, index), so K times the least head wins
        float hd[kLpWarps];
        int hx[kLpWarps], pos[kLpWarps];
#pragma unroll
        for (int v = 0; v < kLpWarps; ++v) {
            pos[v] = 0;
            hd[v] = md[v][0][t];
            hx[v] = mi[v][0][t];
        }
        float nd[K];
        int nx[K];
#pragma unroll
        for (int r = 0; r < K; ++r) {
            int bw = 0;
            float bd = hd[0];
            int bx = hx[0];
#pragma unroll
            for (int v = 1; v < kLpWarps; ++v)
                if (hd[v] < bd || (hd[v] == bd && hx[v] < bx)) {
                    bw = v;
                    bd = hd[v];
                    bx = hx[v];
                }
            nd[r] = bd;
            nx[r] = bx;
#pragma unroll
            for (int v = 0; v < kLpWarps; ++v)
                if (v == bw) {
                    ++pos[v];
                    hd[v] = pos[v] < K ? md[v][pos[v]][t] : INFINITY;
                    hx[v] = pos[v] < K ? mi[v][pos[v]][t] : kLpNone;
                }
        }

        // Lhat = sum_r w_r L2[j_r] / sum_r w_r, summed in fp32 nearest first.  An unfilled slot (only possible when
        // non-finite coordinates leave fewer than K comparable points) contributes nothing and reads back as -1.
        float sw = 0.f, sx = 0.f, sy = 0.f, sz = 0.f;
        const long long row = (long long)s * N + q;
#pragma unroll
        for (int r = 0; r < K; ++r) {
            const int j = nx[r];
            const bool ok = j < M;
            nn_idx[row * K + r] = ok ? j : -1;
            if (!ok) continue;
            const float wr = __fdiv_rn(1.f, __fadd_rn(nd[r], 1e-8f));
            sx = __fadd_rn(sx, __fmul_rn(wr, __ldg(lp + 3ll * j)));
            sy = __fadd_rn(sy, __fmul_rn(wr, __ldg(lp + 3ll * j + 1)));
            sz = __fadd_rn(sz, __fmul_rn(wr, __ldg(lp + 3ll * j + 2)));
            sw = __fadd_rn(sw, wr);
        }
        const float3 lw = laplacian_at(ws, g1 + ((long long)b * N + q) * kl, kl, q);
        const float rx = __fsub_rn(__fdiv_rn(sx, sw), lw.x), ry = __fsub_rn(__fdiv_rn(sy, sw), lw.y),
                    rz = __fsub_rn(__fdiv_rn(sz, sw), lw.z);
        res[3 * row] = rx;
        res[3 * row + 1] = ry;
        res[3 * row + 2] = rz;
        part = ((double)rx * (double)rx + (double)ry * (double)ry) + (double)rz * (double)rz;
    }
    part = warp_sum(part);
    if (lane == 0 && part != 0.0) {
        if constexpr (DET) fx_atomic(reinterpret_cast<unsigned long long*>(acc) + (long long)s * kFxWords, part);
        else atomicAdd(acc + s, part);
    }
}

// The grid form of k_laplacian_fwd: the same search on the index `ix` of p2 (B samples), the same laplacian_point.  One warp
// per query (kGqPerWarp consecutive queries per warp); lane 0 forms each query's result and sums its queries' terms in order.
template <int K, bool DET>
__global__ void __launch_bounds__(kGqThreads) k_laplacian_grid(const float* __restrict__ w, const float* __restrict__ l2,
                                                                const int32_t* __restrict__ g1, int B, int N, int M, int kl, GridIndex ix,
                                                                int32_t* __restrict__ nn_idx, float* __restrict__ res, double* __restrict__ acc) {
    const int s = blockIdx.y, b = s % B;
    const int lane = lane_id();
    const int q0 = (blockIdx.x * kGqWarps + warp_id()) * kGqPerWarp;
    if (q0 >= N) return;   // uniform over the warp; no barrier follows
    const float* ws = w + (long long)s * N * 3;
    const float* lp = l2 + (long long)b * M * 3;
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
        if (lane == 0) part += laplacian_point<K>(nd, nx, ws, lp, g1 + ((long long)b * N + q) * kl, kl, M, (long long)s * N + q, q, nn_idx, res);
    }
    if (lane == 0 && part != 0.0) {
        if constexpr (DET) fx_atomic(reinterpret_cast<unsigned long long*>(acc) + (long long)s * kFxWords, part);
        else atomicAdd(acc + s, part);
    }
}

// One thread per point (s, i) of W: d_w [S,N,3] (over G1 and at i), d_p2 [B,M,3] (the distance part; or NULL) and
// d_l2 [B,M,3] (or NULL), all accumulated, for the upstream gradient g [S] on the device.  k (<= kLpMaxK) slots of nn_idx
// per point; a slot of -1 contributes nothing.  DET: the destinations are fixed-point workspaces.
template <bool DET>
__global__ void __launch_bounds__(256) k_laplacian_bwd(const float* __restrict__ w, const float* __restrict__ p2, const float* __restrict__ l2,
                                                       const int32_t* __restrict__ g1, const int32_t* __restrict__ nn_idx,
                                                       const float* __restrict__ res, const float* __restrict__ g, int B, int N, int M,
                                                       int kl, int k, long long points, float* __restrict__ d_w, float* __restrict__ d_p2,
                                                       float* __restrict__ d_l2) {
    const float den = (float)(kl - 1);
    for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < points; p += (long long)gridDim.x * blockDim.x) {
        const int s = (int)(p / N), b = s % B;
        const long long i = p - (long long)s * N;
        const float c = 2.f * __ldg(g + s) / (float)N;
        const float ex = c * __ldg(res + 3 * p), ey = c * __ldg(res + 3 * p + 1), ez = c * __ldg(res + 3 * p + 2);

        // through L(W)_i
        const float cx = __fdiv_rn(ex, den), cy = __fdiv_rn(ey, den), cz = __fdiv_rn(ez, den);
        float ox = 0.f, oy = 0.f, oz = 0.f;
        const int32_t* ni = g1 + ((long long)b * N + i) * kl;
        for (int e = 0; e < kl; ++e) {
            const long long j = __ldg(ni + e);
            if (j == i) continue;
            const long long r = 3 * ((long long)s * N + j);
            scatter_add<DET>(d_w, r, -cx);
            scatter_add<DET>(d_w, r + 1, -cy);
            scatter_add<DET>(d_w, r + 2, -cz);
            ox += cx;
            oy += cy;
            oz += cz;
        }

        // through Lhat_i
        const float wx = __ldg(w + 3 * p), wy = __ldg(w + 3 * p + 1), wz = __ldg(w + 3 * p + 2);
        int jj[kLpMaxK];
        float wt[kLpMaxK], dx[kLpMaxK], dy[kLpMaxK], dz[kLpMaxK], lx[kLpMaxK], ly[kLpMaxK], lz[kLpMaxK];
        float sw = 0.f;
#pragma unroll
        for (int r = 0; r < kLpMaxK; ++r) {
            jj[r] = r < k ? __ldg(nn_idx + p * k + r) : -1;
            wt[r] = dx[r] = dy[r] = dz[r] = lx[r] = ly[r] = lz[r] = 0.f;
            if (jj[r] < 0) continue;
            const long long m = 3 * ((long long)b * M + jj[r]);
            dx[r] = __fsub_rn(wx, __ldg(p2 + m));
            dy[r] = __fsub_rn(wy, __ldg(p2 + m + 1));
            dz[r] = __fsub_rn(wz, __ldg(p2 + m + 2));
            lx[r] = __ldg(l2 + m);
            ly[r] = __ldg(l2 + m + 1);
            lz[r] = __ldg(l2 + m + 2);
            const float d = __fadd_rn(__fadd_rn(__fmul_rn(dx[r], dx[r]), __fmul_rn(dy[r], dy[r])), __fmul_rn(dz[r], dz[r]));
            wt[r] = __fdiv_rn(1.f, __fadd_rn(d, 1e-8f));   // the forward's weight, bit for bit
            sw = __fadd_rn(sw, wt[r]);
        }
#pragma unroll
        for (int m = 0; m < kLpMaxK; ++m) {
            if (jj[m] < 0) continue;
            float tx = 0.f, ty = 0.f, tz = 0.f;   // sum_r w_r (L2_m - L2_r) = sum w (L2_m - Lhat)
#pragma unroll
            for (int r = 0; r < kLpMaxK; ++r) {
                tx += wt[r] * (lx[m] - lx[r]);
                ty += wt[r] * (ly[m] - ly[r]);
                tz += wt[r] * (lz[m] - lz[r]);
            }
            const float om = __fdiv_rn(wt[m], sw);
            const float gd = -2.f * om * om * ((ex * tx + ey * ty) + ez * tz);   // dR/dd_m times dd_m/d(W_i - P2_m) = 2 (W_i - P2_m)
            const float vx = gd * dx[m], vy = gd * dy[m], vz = gd * dz[m];
            ox += vx;
            oy += vy;
            oz += vz;
            const long long r = 3 * ((long long)b * M + jj[m]);
            if (d_p2) {
                scatter_add<DET>(d_p2, r, -vx);
                scatter_add<DET>(d_p2, r + 1, -vy);
                scatter_add<DET>(d_p2, r + 2, -vz);
            }
            if (d_l2) {
                scatter_add<DET>(d_l2, r, om * ex);
                scatter_add<DET>(d_l2, r + 1, om * ey);
                scatter_add<DET>(d_l2, r + 2, om * ez);
            }
        }
        scatter_add<DET>(d_w, 3 * p, ox);
        scatter_add<DET>(d_w, 3 * p + 1, oy);
        scatter_add<DET>(d_w, 3 * p + 2, oz);
    }
}

template <int K>
static void launch_fwd(dim3 grid, cudaStream_t st, bool det, const float* w, const float* p2, const float* l2, const int32_t* g1, int B,
                       int N, int M, int kl, int32_t* nn_idx, float* res, double* acc) {
    if (det) k_laplacian_fwd<K, true><<<grid, kLpThreads, 0, st>>>(w, p2, l2, g1, B, N, M, kl, nn_idx, res, acc);
    else k_laplacian_fwd<K, false><<<grid, kLpThreads, 0, st>>>(w, p2, l2, g1, B, N, M, kl, nn_idx, res, acc);
}

template <int K>
static void launch_grid(dim3 grid, cudaStream_t st, bool det, const float* w, const float* l2, const int32_t* g1, int B, int N, int M, int kl,
                        const GridIndex& ix, int32_t* nn_idx, float* res, double* acc) {
    if (det) k_laplacian_grid<K, true><<<grid, kGqThreads, 0, st>>>(w, l2, g1, B, N, M, kl, ix, nn_idx, res, acc);
    else k_laplacian_grid<K, false><<<grid, kGqThreads, 0, st>>>(w, l2, g1, B, N, M, kl, ix, nn_idx, res, acc);
}

static bool bad_graph(int k, int n) { return k < 2 || k > kLpMaxGraph || k > n; }

static bool bad_term(int S, int B, int N, int M, int k_lap, int k_int) {
    return S < 1 || B < 1 || S % B != 0 || N < 1 || M < 1 || bad_graph(k_lap, N) || k_int < 1 || k_int > kLpMaxK || k_int > M;
}

}  // namespace pvraft

using namespace pvraft;

extern "C" int pvraft_cloud_laplacian_fwd(const float* x, const int32_t* nbr, int B, int N, int k, float* out, void* stream) {
    if (!x || !nbr || !out || B < 1 || N < 1 || bad_graph(k, N)) return fail(PVRAFT_ERR_BAD_ARG, "cloud_laplacian_fwd: bad argument");
    const long long points = (long long)B * N;
    k_cloud_laplacian<<<(unsigned)scatter_blocks(points, false), 256, 0, (cudaStream_t)stream>>>(x, nbr, N, k, points, out);
    return check_launch("cloud_laplacian_fwd");
}

extern "C" int pvraft_cloud_laplacian_bwd(const float* g_l, const int32_t* nbr, int B, int N, int k, float* d_x, void* det_workspace,
                                          void* stream) {
    if (!g_l || !nbr || !d_x || B < 1 || N < 1 || bad_graph(k, N)) return fail(PVRAFT_ERR_BAD_ARG, "cloud_laplacian_bwd: bad argument");
    const long long points = (long long)B * N;
    const bool det = det_workspace != nullptr;
    const unsigned blocks = (unsigned)scatter_blocks(points, det);
    cudaStream_t st = (cudaStream_t)stream;
    if (!det) {
        k_cloud_laplacian_bwd<false><<<blocks, 256, 0, st>>>(g_l, nbr, N, k, points, d_x);
        return check_launch("cloud_laplacian_bwd");
    }
    k_cloud_laplacian_bwd<true><<<blocks, 256, 0, st>>>(g_l, nbr, N, k, points, static_cast<float*>(det_workspace));
    const int rc = check_launch("cloud_laplacian_bwd");
    if (rc) return rc;
    return fx_flush_f32(static_cast<const unsigned long long*>(det_workspace), 1, 3 * points, 3 * points, 0, d_x, st);
}

extern "C" int64_t pvraft_cloud_laplacian_bwd_det_workspace_bytes(int B, int N) { return B < 1 || N < 1 ? 0 : 3ll * B * N * kFxWords * 8; }

extern "C" int pvraft_laplacian_fwd(const float* w, const float* p2, const float* l2, const int32_t* g1, int S, int B, int N, int M, int k_lap,
                                    int k_int, int32_t* nn_idx, float* res, double* acc, void* det_workspace, void* stream) {
    if (!w || !p2 || !l2 || !g1 || !nn_idx || !res || !acc || bad_term(S, B, N, M, k_lap, k_int))
        return fail(PVRAFT_ERR_BAD_ARG, "laplacian_fwd: bad argument");
    if (S > 65535) return fail(PVRAFT_ERR_UNSUPPORTED, "laplacian_fwd: S = %d samples (at most 65535)", S);
    const dim3 grid((unsigned)((N + kLpPerCta - 1) / kLpPerCta), (unsigned)S);
    cudaStream_t st = (cudaStream_t)stream;
    const bool det = det_workspace != nullptr;
    double* sums = det ? static_cast<double*>(det_workspace) : acc;
    switch (k_int) {
        case 1: launch_fwd<1>(grid, st, det, w, p2, l2, g1, B, N, M, k_lap, nn_idx, res, sums); break;
        case 2: launch_fwd<2>(grid, st, det, w, p2, l2, g1, B, N, M, k_lap, nn_idx, res, sums); break;
        case 3: launch_fwd<3>(grid, st, det, w, p2, l2, g1, B, N, M, k_lap, nn_idx, res, sums); break;
        case 4: launch_fwd<4>(grid, st, det, w, p2, l2, g1, B, N, M, k_lap, nn_idx, res, sums); break;
        case 5: launch_fwd<5>(grid, st, det, w, p2, l2, g1, B, N, M, k_lap, nn_idx, res, sums); break;
        case 6: launch_fwd<6>(grid, st, det, w, p2, l2, g1, B, N, M, k_lap, nn_idx, res, sums); break;
        case 7: launch_fwd<7>(grid, st, det, w, p2, l2, g1, B, N, M, k_lap, nn_idx, res, sums); break;
        default: launch_fwd<8>(grid, st, det, w, p2, l2, g1, B, N, M, k_lap, nn_idx, res, sums); break;
    }
    const int rc = check_launch("laplacian_fwd");
    if (rc || !det) return rc;
    return fx_flush_f64(static_cast<const unsigned long long*>(det_workspace), 1, S, S, 0, acc, st);
}

extern "C" int64_t pvraft_laplacian_fwd_det_workspace_bytes(int S) { return S < 1 ? 0 : (int64_t)S * kFxWords * 8; }

extern "C" int pvraft_laplacian_grid_fwd(const float* w, const float* p2, const float* l2, const int32_t* g1, int S, int B, int N, int M,
                                         int k_lap, int k_int, int32_t* nn_idx, float* res, double* acc, void* workspace, void* det_workspace,
                                         void* stream) {
    if (!w || !p2 || !l2 || !g1 || !nn_idx || !res || !acc || !workspace || bad_term(S, B, N, M, k_lap, k_int))
        return fail(PVRAFT_ERR_BAD_ARG, "laplacian_grid_fwd: bad argument");
    if (S > 65535) return fail(PVRAFT_ERR_UNSUPPORTED, "laplacian_grid_fwd: S = %d samples (at most 65535)", S);
    cudaStream_t st = (cudaStream_t)stream;
    GridIndex ix;
    int rc = grid_index_build(p2, nullptr, B, M, workspace, st, &ix);
    if (rc) return rc;
    const dim3 grid((unsigned)((N + kGqPerCta - 1) / kGqPerCta), (unsigned)S);
    const bool det = det_workspace != nullptr;
    double* sums = det ? static_cast<double*>(det_workspace) : acc;
    switch (k_int) {
        case 1: launch_grid<1>(grid, st, det, w, l2, g1, B, N, M, k_lap, ix, nn_idx, res, sums); break;
        case 2: launch_grid<2>(grid, st, det, w, l2, g1, B, N, M, k_lap, ix, nn_idx, res, sums); break;
        case 3: launch_grid<3>(grid, st, det, w, l2, g1, B, N, M, k_lap, ix, nn_idx, res, sums); break;
        case 4: launch_grid<4>(grid, st, det, w, l2, g1, B, N, M, k_lap, ix, nn_idx, res, sums); break;
        case 5: launch_grid<5>(grid, st, det, w, l2, g1, B, N, M, k_lap, ix, nn_idx, res, sums); break;
        case 6: launch_grid<6>(grid, st, det, w, l2, g1, B, N, M, k_lap, ix, nn_idx, res, sums); break;
        case 7: launch_grid<7>(grid, st, det, w, l2, g1, B, N, M, k_lap, ix, nn_idx, res, sums); break;
        default: launch_grid<8>(grid, st, det, w, l2, g1, B, N, M, k_lap, ix, nn_idx, res, sums); break;
    }
    rc = check_launch("laplacian_grid_fwd");
    if (rc || !det) return rc;
    return fx_flush_f64(static_cast<const unsigned long long*>(det_workspace), 1, S, S, 0, acc, st);
}

extern "C" int pvraft_laplacian_bwd(const float* w, const float* p2, const float* l2, const int32_t* g1, const int32_t* nn_idx, const float* res,
                                    const float* g, int S, int B, int N, int M, int k_lap, int k_int, float* d_w, float* d_p2, float* d_l2,
                                    void* det_workspace, void* stream) {
    if (!w || !p2 || !l2 || !g1 || !nn_idx || !res || !g || !d_w || bad_term(S, B, N, M, k_lap, k_int))
        return fail(PVRAFT_ERR_BAD_ARG, "laplacian_bwd: bad argument");
    const long long points = (long long)S * N;
    const bool det = det_workspace != nullptr;
    const unsigned blocks = (unsigned)scatter_blocks(points, det);
    cudaStream_t st = (cudaStream_t)stream;
    if (!det) {
        k_laplacian_bwd<false><<<blocks, 256, 0, st>>>(w, p2, l2, g1, nn_idx, res, g, B, N, M, k_lap, k_int, points, d_w, d_p2, d_l2);
        return check_launch("laplacian_bwd");
    }
    // workspace: [3 S N | 3 B M | 3 B M] slots for d_w, d_p2, d_l2
    const long long nw = 3 * points, nb = 3ll * B * M;
    unsigned long long* ws = static_cast<unsigned long long*>(det_workspace);
    float* ws_w = reinterpret_cast<float*>(ws);
    float* ws_p2 = reinterpret_cast<float*>(ws + nw * kFxWords);
    float* ws_l2 = reinterpret_cast<float*>(ws + (nw + nb) * kFxWords);
    k_laplacian_bwd<true><<<blocks, 256, 0, st>>>(w, p2, l2, g1, nn_idx, res, g, B, N, M, k_lap, k_int, points, ws_w, d_p2 ? ws_p2 : nullptr,
                                                  d_l2 ? ws_l2 : nullptr);
    int rc = check_launch("laplacian_bwd");
    if (rc) return rc;
    rc = fx_flush_f32(ws, 1, nw, nw, 0, d_w, st);
    if (!rc && d_p2) rc = fx_flush_f32(reinterpret_cast<const unsigned long long*>(ws_p2), 1, nb, nb, 0, d_p2, st);
    if (!rc && d_l2) rc = fx_flush_f32(reinterpret_cast<const unsigned long long*>(ws_l2), 1, nb, nb, 0, d_l2, st);
    return rc;
}

extern "C" int64_t pvraft_laplacian_bwd_det_workspace_bytes(int S, int B, int N, int M) {
    if (S < 1 || B < 1 || N < 1 || M < 1) return 0;
    return (3ll * S * N + 6ll * B * M) * kFxWords * 8;
}
