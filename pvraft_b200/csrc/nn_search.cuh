// The distance of the brute-force nearest-neighbour searches that rank points by their own coordinates rather than by the
// kNN graph's expanded form |q|^2 + |x|^2 - 2 q.x (self_supervised.cu, flow_propagate.cu, laplacian.cu), the sorted k-best
// list of the k-nearest searches, and the tiled brute-force K-best search of k_flow_propagate and k_laplacian_fwd.
#pragma once
#include <type_traits>
#include "common.cuh"

namespace pvraft {

// the squared length of the fp32 difference q - p, (dx*dx + dy*dy) + dz*dz rounded to nearest at every step, with no FMA
// contraction
__device__ __forceinline__ float diff_sq(float qx, float qy, float qz, const float4& p) {
    const float dx = __fsub_rn(qx, p.x), dy = __fsub_rn(qy, p.y), dz = __fsub_rn(qz, p.z);
    return __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
}

// insert (d, j) into the ascending list best / arg of length K; the caller has checked d < best[K - 1].  Candidates that
// arrive in ascending index order keep the list ordered on (distance, index).
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

// f(std::integral_constant<int, K>()) with K = k, for the k-best kernels instantiated at K = 1..kMax; the caller has checked
// 1 <= k <= kMax.
template <int kMax, class F>
void dispatch_k(int k, F&& f) {
    if constexpr (kMax > 1)
        if (k < kMax) return dispatch_k<kMax - 1>(k, f);
    f(std::integral_constant<int, kMax>());
}

// ---- the tiled brute-force K-best search ----------------------------------------------------------------------------------
// Each CTA keeps kKbPerCta queries in registers (kKbQueries per lane, the same queries in every warp) while the searched
// cloud streams through double-buffered shared-memory tiles; warp w searches the w-th slice of every tile, so the eight warps
// split the searched cloud and a CTA covers only 64 queries, which fills the SMs at the model's sizes (N = 8192, B = 1: 128
// CTAs).  Each lane keeps a sorted K-best list per query in registers; within a warp candidates arrive in ascending index
// order, so a strict comparison keeps the (distance, index) order.  At the end the eight lists of a query are merged on
// (distance, index) in shared memory by one thread.  There are no atomics and no reduction whose order depends on timing.
constexpr int kKbWarps = 8;
constexpr int kKbThreads = kKbWarps * kWarp;
constexpr int kKbQueries = 2;                          // queries per lane, held in registers
constexpr int kKbPerCta = kWarp * kKbQueries;          // queries per CTA, searched by every warp
constexpr int kKbTile = 256;                           // searched points per shared-memory tile (two tiles)
constexpr int kKbSlice = kKbTile / kKbWarps;           // points of a tile each warp searches
constexpr int kKbNone = 0x7fffffff;                    // index of an unfilled slot: loses every (distance, index) tie
static_assert(kKbTile == kKbThreads, "each thread stages one point per tile");
static_assert(kKbPerCta % kWarp == 0, "the merging threads are whole warps");

// The K nearest, on (diff_sq, index), of the CTA's queries qp[blockIdx.x * kKbPerCta + t] (t < kKbPerCta, rows past N read as
// the origin) among the M points of cp, each plus off (one fp32 add per coordinate while staging) when OFFSET.  Launched with
// kKbThreads threads; every thread must call it.  Returns t < kKbPerCta, with that thread's query's K nearest in (nd, nx),
// nearest first; a slot no point filled (only possible when non-finite coordinates leave fewer than K comparable points)
// holds (+inf, kKbNone).
template <int K, bool OFFSET>
__device__ __forceinline__ bool tiled_kbest(const float* __restrict__ qp, int N, const float* __restrict__ cp, const float* __restrict__ off,
                                            int M, float (&nd)[K], int (&nx)[K]) {
    __shared__ float4 tile[2][kKbTile];
    __shared__ float md[kKbWarps][K][kKbPerCta];       // every warp's k-best lists, [warp][rank][query]
    __shared__ int mi[kKbWarps][K][kKbPerCta];
    const int q0 = blockIdx.x * kKbPerCta;
    const int lane = lane_id(), warp = warp_id();

    float qx[kKbQueries], qy[kKbQueries], qz[kKbQueries], best[kKbQueries][K];
    int arg[kKbQueries][K];
#pragma unroll
    for (int i = 0; i < kKbQueries; ++i) {
        const int q = q0 + i * kWarp + lane;
        const bool ok = q < N;
        qx[i] = ok ? __ldg(qp + 3ll * q) : 0.f;
        qy[i] = ok ? __ldg(qp + 3ll * q + 1) : 0.f;
        qz[i] = ok ? __ldg(qp + 3ll * q + 2) : 0.f;
#pragma unroll
        for (int r = 0; r < K; ++r) {
            best[i][r] = INFINITY;
            arg[i][r] = kKbNone;
        }
    }

    // the next tile is fetched (and offset) into registers while the current one is searched; points past the end read as
    // NaN, whose distance never compares below a list entry
    float st[3];
    auto fetch = [&](int t) {
        const int p = t * kKbTile + threadIdx.x;
        const bool ok = p < M;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            if constexpr (OFFSET) st[c] = ok ? __fadd_rn(__ldg(cp + 3ll * p + c), __ldg(off + 3ll * p + c)) : NAN;
            else st[c] = ok ? __ldg(cp + 3ll * p + c) : NAN;
        }
    };
    auto store = [&](int buf) { tile[buf][threadIdx.x] = make_float4(st[0], st[1], st[2], 0.f); };

    const int tiles = (M + kKbTile - 1) / kKbTile;
    fetch(0);
    store(0);
    __syncthreads();
    for (int t = 0; t < tiles; ++t) {
        const bool more = t + 1 < tiles;
        if (more) fetch(t + 1);
        const float4* tl = tile[t & 1] + warp * kKbSlice;
        const int base = t * kKbTile + warp * kKbSlice;
#pragma unroll 8
        for (int j = 0; j < kKbSlice; ++j) {
            const float4 p = tl[j];   // the same address in every lane: a broadcast
#pragma unroll
            for (int i = 0; i < kKbQueries; ++i) {
                const float d = diff_sq(qx[i], qy[i], qz[i], p);
                if (d < best[i][K - 1]) kbest_insert<K>(best[i], arg[i], d, base + j);
            }
        }
        if (more) store((t + 1) & 1);   // the buffer searched in iteration t - 1, released by its barrier
        __syncthreads();
    }

#pragma unroll
    for (int i = 0; i < kKbQueries; ++i)
#pragma unroll
        for (int r = 0; r < K; ++r) {
            md[warp][r][i * kWarp + lane] = best[i][r];
            mi[warp][r][i * kWarp + lane] = arg[i][r];
        }
    __syncthreads();
    const int t = threadIdx.x;
    if (t >= kKbPerCta) return false;

    // merge the warps' lists: each is ascending in (distance, index), so K times the least head wins
    float hd[kKbWarps];
    int hx[kKbWarps], pos[kKbWarps];
#pragma unroll
    for (int w = 0; w < kKbWarps; ++w) {
        pos[w] = 0;
        hd[w] = md[w][0][t];
        hx[w] = mi[w][0][t];
    }
#pragma unroll
    for (int r = 0; r < K; ++r) {
        int bw = 0;
        float bd = hd[0];
        int bx = hx[0];
#pragma unroll
        for (int w = 1; w < kKbWarps; ++w)
            if (hd[w] < bd || (hd[w] == bd && hx[w] < bx)) {
                bw = w;
                bd = hd[w];
                bx = hx[w];
            }
        nd[r] = bd;
        nx[r] = bx;
#pragma unroll
        for (int w = 0; w < kKbWarps; ++w)
            if (w == bw) {
                ++pos[w];
                hd[w] = pos[w] < K ? md[w][pos[w]][t] : INFINITY;
                hx[w] = pos[w] < K ? mi[w][pos[w]][t] : kKbNone;
            }
    }
    return true;
}

}  // namespace pvraft
