// Euclidean clustering of a point cloud on the device (single linkage: the connected components of the fixed-radius graph),
// the objects of pvraft_b200.rigid_objects.  Every decision is an integer one, so the labels are the same bits in any mode
// and from run to run (the rule is stated in include/pvraft_b200.h, pvraft_euclidean_clusters_fwd):
//
//   k_cc_stage    a point takes part when allowed (mask) and finite (takes_part): its coordinates are staged as they are,
//                 any other point's as NaN, so the index's bounds ignore it and no distance to it compares <= r2; parent[i] = i
//   (index)       grid_index_build on the staged cloud
//   k_cc_edges    one warp per query: grid_radius_visit (grid_index.cuh, exact for the fp32 predicate); every edge (i, j) with
//                 j < i is united: the two roots are found (path halving) and the larger is hooked under the smaller with an
//                 atomicCAS, retried from the value the CAS returns.  parent[v] <= v always, so a tree's root is its smallest
//                 id, and once every edge has been united the root of a component is its smallest point id, whatever order
//                 the unions ran in
//   k_cc_flatten  root of every taking-part point (into labels), component sizes by integer atomics at the roots
//   k_cc_rank     one CTA per sample: the components of >= min_points points, keyed (size << 32) | ~root (unique); the O-th
//                 largest key by an 8-bit radix select, then each kept key's rank among the kept (a count) is its object
//   k_cc_label    labels[i] = the object of i's root, or -1
#include "grid_index.cuh"
#include "rigid_segments.cuh"

namespace pvraft {

constexpr int kCcThreads = 256;
constexpr int kCcWarps = kCcThreads / kWarp;
constexpr int kCcRankThreads = 1024;

__global__ void __launch_bounds__(kCcThreads) k_cc_stage(const float* __restrict__ xyz, const uint8_t* __restrict__ mask, int N,
                                                         long long points, float* __restrict__ staged, int32_t* __restrict__ parent,
                                                         int32_t* __restrict__ size, int32_t* __restrict__ objmap) {
    const long long p = (long long)blockIdx.x * kCcThreads + threadIdx.x;
    if (p >= points) return;
    const float x = xyz[3 * p], y = xyz[3 * p + 1], z = xyz[3 * p + 2];
    const bool on = takes_part(mask, p, x, y, z);
    staged[3 * p] = on ? x : NAN;
    staged[3 * p + 1] = on ? y : NAN;
    staged[3 * p + 2] = on ? z : NAN;
    parent[p] = on ? (int32_t)(p % N) : -1;
    size[p] = 0;
    objmap[p] = -1;
}

// the root of x in a sample's forest par (parent[v] <= v); path halving, racing writes only ever store an ancestor
__device__ __forceinline__ int uf_find(int32_t* par, int x) {
    for (;;) {
        const int p = __ldcg(par + x);
        if (p == x) return x;
        const int q = __ldcg(par + p);
        if (q == p) return p;
        __stcg(par + x, q);
        x = q;
    }
}

__device__ __forceinline__ void uf_unite(int32_t* par, int a, int b) {
    for (;;) {
        a = uf_find(par, a);
        b = uf_find(par, b);
        if (a == b) return;
        if (a > b) {
            const int t = a;
            a = b;
            b = t;
        }
        const int old = atomicCAS(par + b, b, a);   // hook the larger root under the smaller
        if (old == b) return;
        b = old;                                    // b was hooked meanwhile: continue from its new parent
    }
}

// one warp per (sample, point) query, kCcWarps queries per CTA
__global__ void __launch_bounds__(kCcThreads) k_cc_edges(const float* __restrict__ staged, const float* __restrict__ flow, int N,
                                                         long long points, float r2, float fr2, GridIndex ix, int32_t* __restrict__ parent) {
    const long long q = (long long)blockIdx.x * kCcWarps + warp_id();
    if (q >= points) return;
    const int s = (int)(q / N), i = (int)(q % N), lane = lane_id();
    const float qx = staged[3 * q], qy = staged[3 * q + 1], qz = staged[3 * q + 2];
    if (qx != qx) return;   // not taking part (NaN staged): uniform over the warp
    const long long base = (long long)s * N;
    const float4* P = ix.pts + base;
    const int32_t* I = ix.ids + base;
    const int32_t* CS = ix.cell_start + (long long)s * (ix.cells + 1);
    const GridParams gp = ix.params[s];
    float fx = 0.f, fy = 0.f, fz = 0.f;
    if (flow) {
        fx = flow[3 * q];
        fy = flow[3 * q + 1];
        fz = flow[3 * q + 2];
    }
    int32_t* par = parent + base;
    grid_radius_visit(CS, gp, qx, qy, qz, r2, [&](int begin, int end) {
        for (int k = begin + lane; k < end; k += kWarp) {
            const int j = __ldg(I + k);
            if (j >= i || !(diff_sq(qx, qy, qz, __ldg(P + k)) <= r2)) continue;
            if (flow) {
                const long long pj = base + j;
                if (!(diff_sq(fx, fy, fz, make_float4(flow[3 * pj], flow[3 * pj + 1], flow[3 * pj + 2], 0.f)) <= fr2)) continue;
            }
            uf_unite(par, i, j);
        }
    });
}

// labels[p] = the root of a taking-part point (-1 otherwise); size[root] counts its component
__global__ void __launch_bounds__(kCcThreads) k_cc_flatten(int N, long long points, int32_t* __restrict__ parent, int32_t* __restrict__ size,
                                                           int32_t* __restrict__ labels) {
    const long long p = (long long)blockIdx.x * kCcThreads + threadIdx.x;
    if (p >= points) return;
    const long long base = p - p % N;
    int root = -1;
    if (parent[p] >= 0) {
        root = uf_find(parent + base, (int)(p - base));
        atomicAdd(size + base + root, 1);
    }
    labels[p] = root;
}

// one CTA per sample: objmap[root] = object id of the kept components, counts [B,O], num_objects [B]; cand [B,N] u64 scratch
__global__ void __launch_bounds__(kCcRankThreads) k_cc_rank(const int32_t* __restrict__ size, int N, int O, int min_points,
                                                            unsigned long long* __restrict__ cand, int32_t* __restrict__ objmap,
                                                            int32_t* __restrict__ counts, int32_t* __restrict__ num_objects) {
    __shared__ int n_sh, nsel_sh, hist[256];
    __shared__ unsigned long long sel[kMaxObjects];
    __shared__ unsigned long long prefix_sh;
    const int s = blockIdx.x;
    const int32_t* sz = size + (long long)s * N;
    unsigned long long* cd = cand + (long long)s * N;
    if (threadIdx.x == 0) {
        n_sh = 0;
        nsel_sh = 0;
        prefix_sh = 0ull;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < N; i += kCcRankThreads) {
        const int v = sz[i];
        if (v >= min_points) cd[atomicAdd(&n_sh, 1)] = ((unsigned long long)v << 32) | (unsigned long long)(0xffffffffu - (unsigned)i);
    }
    __syncthreads();
    const int n = n_sh;
    // the O-th largest key: digits from the top, each the largest whose bucket still holds the rank sought
    unsigned long long pmask = 0ull;
    int need = O;
    if (n > O)
        for (int shift = 56; shift >= 0; shift -= 8) {
            for (int d = threadIdx.x; d < 256; d += kCcRankThreads) hist[d] = 0;
            __syncthreads();
            const unsigned long long pre = prefix_sh;
            for (int k = threadIdx.x; k < n; k += kCcRankThreads) {
                const unsigned long long key = cd[k];
                if ((key & pmask) == pre) atomicAdd(hist + (int)((key >> shift) & 255ull), 1);
            }
            __syncthreads();
            if (threadIdx.x == 0) {
                int cum = 0, d = 255;
                for (; d > 0; --d) {
                    if (cum + hist[d] >= need) break;
                    cum += hist[d];
                }
                need -= cum;
                prefix_sh = pre | ((unsigned long long)d << shift);
            }
            pmask |= 255ull << shift;
            __syncthreads();
        }
    const unsigned long long thr = n > O ? prefix_sh : 0ull;
    for (int k = threadIdx.x; k < n; k += kCcRankThreads) {
        const unsigned long long key = cd[k];
        if (key >= thr) sel[atomicAdd(&nsel_sh, 1)] = key;
    }
    __syncthreads();
    const int nsel = nsel_sh;
    if (threadIdx.x < nsel) {
        const unsigned long long key = sel[threadIdx.x];
        int rank = 0;
        for (int k = 0; k < nsel; ++k) rank += sel[k] > key;
        const int root = (int)(0xffffffffu - (unsigned)(key & 0xffffffffull));
        objmap[(long long)s * N + root] = rank;
        counts[(long long)s * O + rank] = (int32_t)(key >> 32);
    }
    for (int o = nsel + threadIdx.x; o < O; o += kCcRankThreads) counts[(long long)s * O + o] = 0;
    if (threadIdx.x == 0) num_objects[s] = nsel;
}

__global__ void __launch_bounds__(kCcThreads) k_cc_label(int N, long long points, const int32_t* __restrict__ objmap,
                                                         int32_t* __restrict__ labels) {
    const long long p = (long long)blockIdx.x * kCcThreads + threadIdx.x;
    if (p >= points) return;
    const int root = labels[p];
    labels[p] = root < 0 ? -1 : objmap[p - p % N + root];
}

// workspace: grid index | staged [B,N,3] f32 | parent [B,N] | size [B,N] | objmap [B,N] | cand [B,N] u64, 16-byte aligned
struct ClusterWs {
    void* index;
    float* staged;
    int32_t *parent, *size, *objmap;
    unsigned long long* cand;
    int64_t bytes;
};
static ClusterWs cluster_ws(void* ws, int B, int N) {
    ByteCarve w(ws);
    const long long pts = (long long)B * N;
    ClusterWs L;
    L.index = w.take<void>(grid_index_bytes(B, N));
    L.staged = w.take<float>(12 * pts);
    L.parent = w.take<int32_t>(4 * pts);
    L.size = w.take<int32_t>(4 * pts);
    L.objmap = w.take<int32_t>(4 * pts);
    L.cand = w.take<unsigned long long>(8 * pts);
    L.bytes = w.bytes;
    return L;
}

static bool bad_radius(float r) { return !(r > 0.f) || isinf(r) || isinf(r * r); }

}  // namespace pvraft

using namespace pvraft;

extern "C" int64_t pvraft_euclidean_clusters_workspace_bytes(int B, int N) {
    return B < 1 || N < 1 || (long long)B * N > 0x7fffffffll ? 0 : cluster_ws(nullptr, B, N).bytes;
}

extern "C" int pvraft_euclidean_clusters_fwd(const float* xyz, const float* flow, const uint8_t* mask, int B, int N, float radius,
                                             float flow_radius, int min_points, int max_objects, int32_t* labels,
                                             int32_t* num_objects, int32_t* counts, void* workspace, void* stream) {
    if (!xyz || !labels || !num_objects || !counts || !workspace || B < 1 || N < 1 || (long long)B * N > 0x7fffffffll ||
        bad_radius(radius) || (flow && bad_radius(flow_radius)) || min_points < 1 || max_objects < 1 || max_objects > kMaxObjects)
        return fail(PVRAFT_ERR_BAD_ARG, "euclidean_clusters_fwd: bad argument");
    if (B > 65535) return fail(PVRAFT_ERR_UNSUPPORTED, "euclidean_clusters_fwd: B = %d samples (at most 65535)", B);
    if (reinterpret_cast<uintptr_t>(workspace) & 15) return fail(PVRAFT_ERR_BAD_ARG, "euclidean_clusters_fwd: workspace not 16-byte aligned");
    cudaStream_t st = (cudaStream_t)stream;
    const ClusterWs L = cluster_ws(workspace, B, N);
    const long long points = (long long)B * N;
    const unsigned blocks = (unsigned)((points + kCcThreads - 1) / kCcThreads);
    k_cc_stage<<<blocks, kCcThreads, 0, st>>>(xyz, mask, N, points, L.staged, L.parent, L.size, L.objmap);
    int rc = check_launch("euclidean_clusters_fwd stage");
    if (rc) return rc;
    GridIndex ix;
    if ((rc = grid_index_build(L.staged, nullptr, B, N, L.index, st, &ix))) return rc;
    k_cc_edges<<<(unsigned)((points + kCcWarps - 1) / kCcWarps), kCcThreads, 0, st>>>(L.staged, flow, N, points, radius * radius,
                                                                                       flow ? flow_radius * flow_radius : 0.f, ix, L.parent);
    k_cc_flatten<<<blocks, kCcThreads, 0, st>>>(N, points, L.parent, L.size, labels);
    k_cc_rank<<<B, kCcRankThreads, 0, st>>>(L.size, N, max_objects, min_points, L.cand, L.objmap, counts, num_objects);
    k_cc_label<<<blocks, kCcThreads, 0, st>>>(N, points, L.objmap, labels);
    return check_launch("euclidean_clusters_fwd");
}
