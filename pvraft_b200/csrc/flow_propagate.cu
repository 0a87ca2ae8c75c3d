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
#include "nn_search.cuh"

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

// insert (d, j) into the ascending list best / arg of length K; the caller has checked d < best[K - 1]
template <int K>
__device__ __forceinline__ void kbest_insert(float (&best)[K], int (&arg)[K], float d, int j) {
#pragma unroll
    for (int i = K - 1; i > 0; --i) {
        if (best[i - 1] > d) {
            best[i] = best[i - 1];
            arg[i] = arg[i - 1];
        } else if (best[i] > d) {
            best[i] = d;
            arg[i] = j;
        }
    }
    if (best[0] > d) {
        best[0] = d;
        arg[0] = j;
    }
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

    // w_j = 1 / (sqrt(d_j) + 1e-8); flow = sum_j w_j flow_prev[j] / sum_j w_j, summed nearest first.  An unfilled slot (only
    // possible when non-finite coordinates leave fewer than K comparable points) contributes nothing and reads back as -1.
    float sw = 0.f, sx = 0.f, sy = 0.f, sz = 0.f;
    const long long row = (long long)b * N + q;
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

template <int K>
static void launch_propagate(dim3 grid, cudaStream_t st, const float* xyz_prev, const float* flow_prev, const float* xyz, int M, int N,
                             float* flow_out, int32_t* idx_out) {
    k_flow_propagate<K><<<grid, kPrThreads, 0, st>>>(xyz_prev, flow_prev, xyz, M, N, flow_out, idx_out);
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
