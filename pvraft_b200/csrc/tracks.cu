// Multi-object tracking from scene flow (no counterpart in the reference): the objects of one pair of a scan sequence are
// associated with those of the previous pair by the votes of their points, and each object's identity, age and rigid
// motion since it was born are carried forward (pvraft_b200.track.ObjectTracker; the rule is stated in include/pvraft_b200.h,
// pvraft_track_objects_fwd).  The nearest moved previous point of every current point is an input: it is the propagation
// search's neighbour (pvraft_flow_propagate_fwd or its grid form with k = 1), so there is no search loop here.
//
//   k_track_votes   one thread per current point: its object c and, through its nearest moved previous point W_i (within
//                   the gate), the previous object a it votes for; the lanes of a warp that share a counter are counted with
//                   one match and one integer atomic (members [B,O], overlap [B,O,O_prev], cleared on the stream first).
//                   Integer counts: the result does not depend on the order of the atomics
//   k_track_assign  one CTA per sample: the eligible pairs (c, a) compacted into shared memory as 64-bit keys whose
//                   ascending order is the greedy order (larger overlap, lower c, lower a), a bitonic sort, one thread's
//                   greedy pass, a block scan that numbers the new tracks, and one thread per slot for its track, match, age
//                   and pose (composed in double)
#include "nn_search.cuh"
#include "rigid_segments.cuh"

namespace pvraft {

constexpr int kTvThreads = 256;
constexpr int kTaThreads = 256;
constexpr int kTaMaxPairs = 16 * kMaxObjects;   // min_overlap >= 1/16: at most 16 eligible previous objects per slot
static_assert(kTaThreads == kMaxObjects, "one assigning thread per slot");

// members[b,c] and overlap[b,c,a] (both zeroed on the stream first); grid (ceil(N / kTvThreads), B)
__global__ void __launch_bounds__(kTvThreads) k_track_votes(const float* __restrict__ xyz_prev, const float* __restrict__ flow_prev,
                                                            const int32_t* __restrict__ labels_prev, const int32_t* __restrict__ track_prev,
                                                            const float* __restrict__ xyz, const int32_t* __restrict__ labels,
                                                            const int32_t* __restrict__ num_objects, const int32_t* __restrict__ nn, int M,
                                                            int N, int O_prev, int O, float g2, int32_t* __restrict__ overlap,
                                                            int32_t* __restrict__ members) {
    const int b = blockIdx.y, j = blockIdx.x * kTvThreads + threadIdx.x, lane = lane_id();
    int c = -1, a = -1;
    if (j < N) {
        const long long p = (long long)b * N + j;
        c = __ldg(labels + p);
        if (c < 0 || c >= min(__ldg(num_objects + b), O)) c = -1;
        const int i = c >= 0 && M > 0 ? __ldg(nn + p) : -1;
        if (i >= 0 && i < M) {
            const long long q = (long long)b * M + i;
            const int s = __ldg(labels_prev + q);
            if (s >= 0 && s < O_prev && __ldg(track_prev + (long long)b * O_prev + s) >= 0) {
                // W_i = X_i + G_i, the same fp32 add the search staged, and the distance it ranked on
                const float4 w = make_float4(__fadd_rn(__ldg(xyz_prev + 3 * q), __ldg(flow_prev + 3 * q)),
                                             __fadd_rn(__ldg(xyz_prev + 3 * q + 1), __ldg(flow_prev + 3 * q + 1)),
                                             __fadd_rn(__ldg(xyz_prev + 3 * q + 2), __ldg(flow_prev + 3 * q + 2)), 0.f);
                if (diff_sq(__ldg(xyz + 3 * p), __ldg(xyz + 3 * p + 1), __ldg(xyz + 3 * p + 2), w) <= g2) a = s;
            }
        }
    }
    // every lane of the warp takes part in both matches (no lane has returned); the lowest lane of a group adds its size
    const unsigned below = (1u << lane) - 1u;
    const unsigned pc = __match_any_sync(kFull, c);
    if (c >= 0 && !(pc & below)) atomicAdd(members + (long long)b * O + c, __popc(pc));
    const int key = a < 0 ? -1 : c * O_prev + a;   // < 256 * 256
    const unsigned pa = __match_any_sync(kFull, key);
    if (key >= 0 && !(pa & below)) atomicAdd(overlap + (long long)b * O * O_prev + key, __popc(pa));
}

// one CTA per sample; a matched slot's pose is R = Ra Rp, t = Ra tp + ta in double, each entry a dot3
__global__ void __launch_bounds__(kTaThreads) k_track_assign(const int32_t* __restrict__ overlap, const int32_t* __restrict__ members,
                                                             const int32_t* __restrict__ num_objects, const int32_t* __restrict__ track_prev,
                                                             const int32_t* __restrict__ age_prev, const double* __restrict__ pose_prev,
                                                             const float* __restrict__ R_prev, const float* __restrict__ t_prev, int O_prev,
                                                             int O, double min_overlap, int32_t* __restrict__ next_id,
                                                             int32_t* __restrict__ match, int32_t* __restrict__ track,
                                                             int32_t* __restrict__ age, double* __restrict__ pose) {
    __shared__ unsigned long long keys[kTaMaxPairs];
    __shared__ int mem_sh[kMaxObjects];
    __shared__ int match_sh[kMaxObjects];
    __shared__ unsigned char taken_sh[kMaxObjects];
    __shared__ int count_sh;
    const int b = blockIdx.x, c = threadIdx.x;
    const int nb = max(0, min(num_objects[b], O));
    const int base_id = next_id[b];   // read by every thread before thread 0 writes it back, after the scan's barrier
    if (c == 0) count_sh = 0;
    mem_sh[c] = c < O ? members[(long long)b * O + c] : 0;
    match_sh[c] = -1;
    taken_sh[c] = 0;
    __syncthreads();

    // the eligible pairs: key (0x7fffffff - overlap) << 16 | c << 8 | a, ascending = larger overlap, lower c, lower a
    const int32_t* ov = overlap + (long long)b * O * O_prev;
    for (int e = threadIdx.x; e < nb * O_prev; e += kTaThreads) {
        const int v = ov[e];
        const int ec = e / O_prev, ea = e - ec * O_prev;
        if (v >= 1 && (double)v >= min_overlap * (double)mem_sh[ec]) {
            const int slot = atomicAdd(&count_sh, 1);
            if (slot < kTaMaxPairs)   // always: the votes of one slot are disjoint, so it has at most 1 / min_overlap such pairs
                keys[slot] = ((unsigned long long)(0x7fffffffu - (unsigned)v) << 16) | ((unsigned long long)ec << 8) | (unsigned long long)ea;
        }
    }
    __syncthreads();
    const int count = min(count_sh, kTaMaxPairs);
    int n2 = 1;
    while (n2 < count) n2 <<= 1;
    for (int k = count + threadIdx.x; k < n2; k += kTaThreads) keys[k] = ~0ull;
    __syncthreads();
    // bitonic sort, ascending
    for (int k = 2; k <= n2; k <<= 1)
        for (int h = k >> 1; h > 0; h >>= 1) {
            for (int i = threadIdx.x; i < n2; i += kTaThreads) {
                const int l = i ^ h;
                if (l > i) {
                    const unsigned long long x = keys[i], y = keys[l];
                    if ((x > y) == ((i & k) == 0)) {
                        keys[i] = y;
                        keys[l] = x;
                    }
                }
            }
            __syncthreads();
        }
    // the greedy matching: a pair is accepted when neither its slot nor its previous object is taken
    if (threadIdx.x == 0)
        for (int k = 0; k < count; ++k) {
            const unsigned long long key = keys[k];
            const int kc = (int)((key >> 8) & 255ull), ka = (int)(key & 255ull);
            if (match_sh[kc] < 0 && !taken_sh[ka]) {
                match_sh[kc] = ka;
                taken_sh[ka] = 1;
            }
        }
    __syncthreads();

    const bool live = c < nb;
    const int a = live ? match_sh[c] : -1;
    int born_total;
    const int rank = block_exclusive_scan<kTaThreads>(live && a < 0 ? 1 : 0, born_total);
    if (threadIdx.x == 0) next_id[b] = base_id + born_total;
    if (c >= O) return;
    const long long r = (long long)b * O + c;
    double P[12] = {1.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0};
    match[r] = a;
    if (!live) {
        track[r] = -1;
        age[r] = -1;
    } else if (a < 0) {
        track[r] = base_id + rank;
        age[r] = 0;
    } else {
        const long long pa = (long long)b * O_prev + a;
        track[r] = track_prev[pa];
        age[r] = age_prev[pa] + 1;
        const float* Ra = R_prev + 9 * pa;
        const float* ta = t_prev + 3 * pa;
        const double* Q = pose_prev + 12 * pa;
#pragma unroll
        for (int i = 0; i < 3; ++i) {
            const double x0 = Ra[3 * i], x1 = Ra[3 * i + 1], x2 = Ra[3 * i + 2];
#pragma unroll
            for (int k = 0; k < 3; ++k) P[3 * i + k] = dot3(x0, x1, x2, Q[k], Q[3 + k], Q[6 + k]);
            P[9 + i] = __dadd_rn(dot3(x0, x1, x2, Q[9], Q[10], Q[11]), (double)ta[i]);
        }
    }
#pragma unroll
    for (int k = 0; k < 12; ++k) pose[12 * r + k] = P[k];
}

static bool bad_gate(float g) { return !(g > 0.f) || isinf(g) || isinf(g * g); }

}  // namespace pvraft

using namespace pvraft;

extern "C" int pvraft_track_objects_fwd(const float* xyz_prev, const float* flow_prev, const int32_t* labels_prev, const int32_t* track_prev,
                                        const int32_t* age_prev, const double* pose_prev, const float* R_prev, const float* t_prev,
                                        const float* xyz, const int32_t* labels, const int32_t* num_objects, const int32_t* nn, int B, int M,
                                        int N, int O_prev, int O, float gate, double min_overlap, int32_t* next_id, int32_t* overlap,
                                        int32_t* members, int32_t* match, int32_t* track, int32_t* age, double* pose, void* stream) {
    if (!xyz || !labels || !num_objects || !next_id || !members || !match || !track || !age || !pose || B < 1 || N < 1 || M < 0 ||
        O < 1 || O > kMaxObjects || O_prev < 0 || O_prev > kMaxObjects || (M == 0 && O_prev != 0) ||
        (M > 0 && (!xyz_prev || !flow_prev || !labels_prev || !nn)) ||
        (O_prev > 0 && (!track_prev || !age_prev || !pose_prev || !R_prev || !t_prev || !overlap)) || bad_gate(gate) ||
        !(min_overlap >= 1.0 / 16.0 && min_overlap <= 1.0))
        return fail(PVRAFT_ERR_BAD_ARG, "track_objects_fwd: bad argument");
    if (B > 65535) return fail(PVRAFT_ERR_UNSUPPORTED, "track_objects_fwd: B = %d samples (at most 65535)", B);
    cudaStream_t st = (cudaStream_t)stream;
    cudaError_t e = cudaMemsetAsync(members, 0, sizeof(int32_t) * (size_t)B * O, st);
    if (e == cudaSuccess && O_prev > 0) e = cudaMemsetAsync(overlap, 0, sizeof(int32_t) * (size_t)B * O * O_prev, st);
    if (e != cudaSuccess) return fail((int)e, "track_objects_fwd: cudaMemsetAsync: %s", cudaGetErrorString(e));
    k_track_votes<<<dim3((unsigned)((N + kTvThreads - 1) / kTvThreads), (unsigned)B), kTvThreads, 0, st>>>(
        xyz_prev, flow_prev, labels_prev, track_prev, xyz, labels, num_objects, nn, M, N, O_prev, O, gate * gate, overlap, members);
    k_track_assign<<<B, kTaThreads, 0, st>>>(overlap, members, num_objects, track_prev, age_prev, pose_prev, R_prev, t_prev, O_prev, O,
                                             min_overlap, next_id, match, track, age, pose);
    return check_launch("track_objects_fwd");
}
