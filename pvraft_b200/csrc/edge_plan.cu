// The gather plan of the SetConv edge kernel (layout in edge_plan.cuh): one CTA per tile deduplicates the tile's neighbour
// and centre ids in a shared-memory hash (a Morton tile of 32 points makes ~1000 references to ~200 distinct rows) and
// writes the distinct ids in slot order and each reference's slot.  Built once per graph; every edge launch on the graph,
// whatever its channel count, then only copies rows.
#include "edge_plan.cuh"

namespace pvraft {

constexpr int kPlanWarps = 8;                                       // 4 neighbour lists per lane, + the centres in warp 0
constexpr int kEdgeHashBits = 11, kEdgeHash = 1 << kEdgeHashBits;   // > kEdgeRefs: linear probing always reaches an empty key

struct PlanSmem {
    int key[kEdgeHash];      // row id, -1 = empty
    short slot[kEdgeHash];   // slot of key[h]
    int count;               // distinct rows so far
};

// warp-collective: puts the rows id[0..K) of every lane (-1: nothing) into the tile's hash, returns their key indices in h and
// writes each new row's id at its slot of `ids`.  The K compare-and-swaps of a lane are in flight together; each round's new
// keys take the next slots (one warp scan, one shared atomic).
template <int K>
__device__ __forceinline__ void edge_insert(const int (&id)[K], int (&h)[K], PlanSmem& s, int32_t* ids) {
    const int lane = lane_id();
    unsigned pending = 0;
#pragma unroll
    for (int m = 0; m < K; ++m) {
        h[m] = (int)(((unsigned)id[m] * 0x9E3779B1u) >> (32 - kEdgeHashBits));
        if (id[m] >= 0) pending |= 1u << m;
    }
    while (__any_sync(kFull, pending)) {
        int old[K];
#pragma unroll
        for (int m = 0; m < K; ++m)
            if (pending >> m & 1u) old[m] = atomicCAS(&s.key[h[m]], -1, id[m]);
        unsigned fresh = 0;
#pragma unroll
        for (int m = 0; m < K; ++m)
            if (pending >> m & 1u) {
                if (old[m] == -1) fresh |= 1u << m;
                if (old[m] == -1 || old[m] == id[m]) pending &= ~(1u << m);
                else h[m] = (h[m] + 1) & (kEdgeHash - 1);
            }
        const int nf = __popc(fresh);
        int incl = nf;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int v = __shfl_up_sync(kFull, incl, o);
            if (lane >= o) incl += v;
        }
        const int total = __shfl_sync(kFull, incl, 31);
        if (total) {
            int first = 0;
            if (lane == 31) first = atomicAdd(&s.count, total);
            int sl = __shfl_sync(kFull, first, 31) + incl - nf;
#pragma unroll
            for (int m = 0; m < K; ++m)
                if (fresh >> m & 1u) {
                    s.slot[h[m]] = (short)sl;
                    ids[sl] = id[m];
                    ++sl;
                }
        }
    }
}

__global__ void __launch_bounds__(kPlanWarps * 32) k_edge_plan(const int32_t* __restrict__ nbr, const int32_t* __restrict__ order, int N,
                                                              unsigned char* __restrict__ plan) {
    __shared__ PlanSmem s;
    const int lane = lane_id(), w = warp_id();
    const int tps = edge_tiles_per_sample(N);
    const long long t = blockIdx.x;
    const int b = (int)(t / tps), start = (int)(t - (long long)b * tps) * kEdgeTile, len = min(kEdgeTile, N - start);
    unsigned char* rec = plan + t * kEdgePlanBytes;
    int32_t* ids = reinterpret_cast<int32_t*>(rec);
    uint16_t* slots = reinterpret_cast<uint16_t*>(rec + kEdgePlanSlots);
    // this thread's references: neighbour `lane` of the points w, w + 8, ..., and (warp 0) the centre of point `lane`
    constexpr int M = kEdgeTile / kPlanWarps;
    const long long s0 = (long long)b * N;
    int id[M + 1], h[M + 1];
#pragma unroll
    for (int m = 0; m < M; ++m) {
        const int p = w + kPlanWarps * m;
        id[m] = p < len ? (order ? __ldg(order + s0 + start + p) : start + p) : -1;
    }
    id[M] = w == 0 && lane < len ? (order ? __ldg(order + s0 + start + lane) : start + lane) : -1;
#pragma unroll
    for (int m = 0; m < M; ++m)
        if (id[m] >= 0) id[m] = __ldg(nbr + (s0 + id[m]) * 32 + lane);
    for (int j = threadIdx.x; j < kEdgeHash; j += kPlanWarps * 32) s.key[j] = -1;
    if (threadIdx.x == 0) s.count = 0;
    __syncthreads();
    edge_insert<M + 1>(id, h, s, ids);
    __syncthreads();   // every slot is in place
#pragma unroll
    for (int m = 0; m < M; ++m) slots[(w + kPlanWarps * m) * 32 + lane] = id[m] >= 0 ? (uint16_t)s.slot[h[m]] : 0;
    if (w == 0) slots[kEdgeTile * 32 + lane] = id[M] >= 0 ? (uint16_t)s.slot[h[M]] : 0;
    if (threadIdx.x == 0) *reinterpret_cast<int32_t*>(rec + kEdgePlanCount) = s.count;
}

}  // namespace pvraft

using namespace pvraft;

extern "C" int64_t pvraft_edge_plan_bytes(int B, int N) {
    if (B <= 0 || N <= 0) return 0;
    return (int64_t)B * edge_tiles_per_sample(N) * kEdgePlanBytes;
}

extern "C" int pvraft_edge_plan_fwd(const int32_t* nbr, const int32_t* order, int B, int N, void* plan, void* stream) {
    if (!nbr || !plan) return fail(PVRAFT_ERR_BAD_ARG, "edge_plan: null pointer");
    if (B <= 0 || N <= 0) return fail(PVRAFT_ERR_BAD_ARG, "edge_plan: bad shape");
    if (reinterpret_cast<uintptr_t>(plan) % 16) return fail(PVRAFT_ERR_BAD_ARG, "edge_plan: plan must be 16-byte aligned");
    const long long tiles = (long long)B * edge_tiles_per_sample(N);
    if (tiles > 0x7fffffffLL) return fail(PVRAFT_ERR_UNSUPPORTED, "edge_plan: %lld tiles", tiles);
    k_edge_plan<<<(unsigned)tiles, kPlanWarps * 32, 0, (cudaStream_t)stream>>>(nbr, order, N, static_cast<unsigned char*>(plan));
    return check_launch("edge_plan");
}
