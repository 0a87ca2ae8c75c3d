// An oriented box for every segment of a clustering -- its extent, heading and displacement over the pair -- in one launch
// sequence with no host synchronisation (the rule is stated in include/pvraft_b200.h, pvraft_object_boxes_fwd):
//
//   (grouping)      rm_group (rigid_segments.cuh): the moment windows of each segment
//   k_box_clear     the extent keys to the identities of min / max (ord_key of +inf / -inf), the counts to 0
//   k_box_extents   over the windows: the window's members (P, Q, H) staged in shared memory, thread a < A projects them
//                   onto direction a; one atomicMin / atomicMax per item, angle and extent on order-preserving keys, the
//                   height extent and the member count once per item
//   k_box_finalize  one warp per segment: lanes stride over the angles, a warp argmin on (area, a), lane 0 writes the box
//
// Every extent is an exact fp32 minimum or maximum, so no result depends on the order of the atomics: there is no
// det_workspace, and a batched call equals per-sample calls bit for bit.
#include "rigid_segments.cuh"

namespace pvraft {

constexpr int kBoxMaxAngles = 256;
constexpr int kBoxWarps = 8;   // segments per CTA of k_box_finalize
static_assert(kBoxMaxAngles <= kMomThreads, "one thread of k_box_extents per angle");

// (c_a, s_a): the fp32 roundings of the double cos and sin of a pi / (2 A)
__device__ __forceinline__ void box_dir(int a, int A, float& c, float& s) {
    double sd, cd;
    sincospi(a / (2.0 * A), &sd, &cd);
    c = (float)cd;
    s = (float)sd;
}

// component k of (x0, x1, x2), k = p, q or up known at run time only: selects, not an indexed local array
__device__ __forceinline__ float pick(float x0, float x1, float x2, int k) { return k == 0 ? x0 : (k == 1 ? x1 : x2); }
__device__ __forceinline__ double pick(double x0, double x1, double x2, int k) { return k == 0 ? x0 : (k == 1 ? x1 : x2); }

// keys [G,A,4] (umin, umax, vmin, vmax), hkeys [G,2] (hmin, hmax) as ord_key, cnt [G]
__global__ void __launch_bounds__(256) k_box_clear(unsigned* __restrict__ keys, unsigned* __restrict__ hkeys, int32_t* __restrict__ cnt,
                                                   long long G, int A) {
    const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
    const unsigned lo = ord_key(INFINITY), hi = ord_key(-INFINITY);
    if (i < G * A * 4) keys[i] = (i & 1) ? hi : lo;
    if (i < G * 2) hkeys[i] = (i & 1) ? hi : lo;
    if (i < G) cnt[i] = 0;
}

// The window walk of rigid_segments.cuh over the moment items.  Member: labels == o and three finite coordinates; P = x_p,
// Q = x_q, H = x_up.  Thread a < A: u = fl(fl(c P) + fl(s Q)), v = fl(fl(c Q) - fl(s P)) of every staged member, their
// minima and maxima.
__global__ void __launch_bounds__(kMomThreads) k_box_extents(const float* __restrict__ x, const int32_t* __restrict__ labels,
                                                             const int32_t* __restrict__ items, const int32_t* __restrict__ nitems,
                                                             int per, int N, int up, int A, unsigned* __restrict__ keys,
                                                             unsigned* __restrict__ hkeys, int32_t* __restrict__ cnt) {
    __shared__ float sp[kMomThreads], sq[kMomThreads];
    __shared__ float hlo[kMomThreads / kWarp], hhi[kMomThreads / kWarp];
    const int s = blockIdx.y, a = threadIdx.x;
    const int ip = up == 2 ? 0 : up + 1, iq = up == 0 ? 2 : up - 1;   // p = (up + 1) % 3, q = (up + 2) % 3
    float c = 0.f, sn = 0.f;
    if (a < A) box_dir(a, A, c, sn);
    for (int it = blockIdx.x; it < nitems[s]; it += gridDim.x) {
        const SegItem w = seg_item(items, s, per, N, it);
        const int i = w.c * kMomThreads + threadIdx.x;
        bool member = false;
        float P = 0.f, Q = 0.f, H = 0.f;
        if (i < N) {
            const long long p = (long long)s * N + i;
            const float x0 = __ldg(x + 3 * p), x1 = __ldg(x + 3 * p + 1), x2 = __ldg(x + 3 * p + 2);
            member = labels[p] == w.o && finite3(x0, x1, x2);
            P = pick(x0, x1, x2, ip);
            Q = pick(x0, x1, x2, iq);
            H = pick(x0, x1, x2, up);
        }
        const float lo = warp_min(member ? H : INFINITY), hi = warp_max(member ? H : -INFINITY);
        if (lane_id() == 0) {
            hlo[warp_id()] = lo;
            hhi[warp_id()] = hi;
        }
        int m;
        const int at = block_exclusive_scan<kMomThreads>(member ? 1 : 0, m);   // its barriers publish hlo / hhi
        if (member) {
            sp[at] = P;
            sq[at] = Q;
        }
        __syncthreads();
        if (m > 0) {   // uniform over the CTA
            if (threadIdx.x == 0) {
                float l = hlo[0], h = hhi[0];
                for (int k = 1; k < kMomThreads / kWarp; ++k) {
                    l = fminf(l, hlo[k]);
                    h = fmaxf(h, hhi[k]);
                }
                atomicMin(hkeys + 2ll * w.g, ord_key(l));
                atomicMax(hkeys + 2ll * w.g + 1, ord_key(h));
                atomicAdd(cnt + w.g, m);
            }
            if (a < A) {
                float umin = INFINITY, umax = -INFINITY, vmin = INFINITY, vmax = -INFINITY;
                for (int j = 0; j < m; ++j) {
                    const float pj = sp[j], qj = sq[j];
                    const float u = __fadd_rn(__fmul_rn(c, pj), __fmul_rn(sn, qj));
                    const float v = __fsub_rn(__fmul_rn(c, qj), __fmul_rn(sn, pj));
                    umin = fminf(umin, u);
                    umax = fmaxf(umax, u);
                    vmin = fminf(vmin, v);
                    vmax = fmaxf(vmax, v);
                }
                unsigned* k = keys + ((long long)w.g * A + a) * 4;
                atomicMin(k, ord_key(umin));
                atomicMax(k + 1, ord_key(umax));
                atomicMin(k + 2, ord_key(vmin));
                atomicMax(k + 3, ord_key(vmax));
            }
        }
        __syncthreads();   // sp, sq, hlo, hhi are reused by the next item
    }
}

// One warp per segment g = (b, o): area_a = (umax - umin)(vmax - vmin) in double (a NaN area counts as +inf), a* the lowest
// a of the least area; lane 0 writes the box.  extents [G,A,4] and dirs [A,2] when given (dirs by segment 0's warp).
__global__ void __launch_bounds__(kBoxWarps * kWarp) k_box_finalize(
    const unsigned* __restrict__ keys, const unsigned* __restrict__ hkeys, const int32_t* __restrict__ cnt, const float* __restrict__ R_o,
    const float* __restrict__ t_o, const float* __restrict__ R_e, const float* __restrict__ t_e, const uint8_t* __restrict__ ego_degenerate,
    int G, int O, int up, int A, float* __restrict__ center, float* __restrict__ size, float* __restrict__ yaw, float* __restrict__ rotation,
    float* __restrict__ displacement, int32_t* __restrict__ count, float* __restrict__ extents, float* __restrict__ dirs) {
    const int g = blockIdx.x * kBoxWarps + warp_id(), lane = lane_id();
    if (g >= G) return;
    const int ip = up == 2 ? 0 : up + 1, iq = up == 0 ? 2 : up - 1;
    const unsigned* kg = keys + (long long)g * A * 4;
    double best = INFINITY;
    int besta = 0x7fffffff;
    for (int a = lane; a < A; a += kWarp) {
        const float e[4] = {ord_float(kg[4 * a]), ord_float(kg[4 * a + 1]), ord_float(kg[4 * a + 2]), ord_float(kg[4 * a + 3])};
        if (extents) {
#pragma unroll
            for (int k = 0; k < 4; ++k) extents[((long long)g * A + a) * 4 + k] = e[k];
        }
        if (dirs && g == 0) box_dir(a, A, dirs[2 * a], dirs[2 * a + 1]);
        double area = __dmul_rn(__dsub_rn((double)e[1], (double)e[0]), __dsub_rn((double)e[3], (double)e[2]));
        if (area != area) area = INFINITY;
        if (area < best || (area == best && a < besta)) {
            best = area;
            besta = a;
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const double ob = __shfl_xor_sync(kFull, best, o);
        const int oa = __shfl_xor_sync(kFull, besta, o);
        if (ob < best || (ob == best && oa < besta)) {
            best = ob;
            besta = oa;
        }
    }
    if (lane != 0) return;
    const int n = cnt[g];
    count[g] = n;
    float* cg = center + 3ll * g;
    float* sg = size + 3ll * g;
    float* dg = displacement + 3ll * g;
    float* rg = rotation + 9ll * g;
    if (n == 0) {   // an empty slot: zeros and the basis (e_p, e_q, e_up)
#pragma unroll
        for (int k = 0; k < 3; ++k) cg[k] = sg[k] = dg[k] = 0.f;
#pragma unroll
        for (int k = 0; k < 9; ++k) rg[k] = 0.f;
        rg[3 * ip] = rg[3 * iq + 1] = rg[3 * up + 2] = 1.f;
        yaw[g] = 0.f;
        return;
    }
    const int a = besta;
    const float umin = ord_float(kg[4 * a]), umax = ord_float(kg[4 * a + 1]), vmin = ord_float(kg[4 * a + 2]), vmax = ord_float(kg[4 * a + 3]);
    const float hmin = ord_float(hkeys[2ll * g]), hmax = ord_float(hkeys[2ll * g + 1]);
    float cf, sf;
    box_dir(a, A, cf, sf);
    const double c = cf, s = sf;
    const double du = __dsub_rn((double)umax, (double)umin), dv = __dsub_rn((double)vmax, (double)vmin);
    double phi = M_PI * (a / (2.0 * A));
    if (!(du >= dv)) phi += M_PI / 2;
    sg[0] = (float)fmax(du, dv);
    sg[1] = (float)fmin(du, dv);
    sg[2] = (float)__dsub_rn((double)hmax, (double)hmin);
    // the centre from the fp32 (c, s), in double, rounded once
    const double mu = __dmul_rn(__dadd_rn((double)umin, (double)umax), 0.5), mv = __dmul_rn(__dadd_rn((double)vmin, (double)vmax), 0.5);
    const float Pc = (float)__dsub_rn(__dmul_rn(c, mu), __dmul_rn(s, mv)), Qc = (float)__dadd_rn(__dmul_rn(s, mu), __dmul_rn(c, mv));
    const float Hc = (float)__dmul_rn(__dadd_rn((double)hmin, (double)hmax), 0.5);
    const float c0 = up == 0 ? Hc : (ip == 0 ? Pc : Qc), c1 = up == 1 ? Hc : (ip == 1 ? Pc : Qc), c2 = up == 2 ? Hc : (ip == 2 ? Pc : Qc);
    // the displacement: y = R_o c + t_o, d = y - c, or with a proper ego fit d = R_e^T (y - t_e) - c
    const float* R = R_o + 9ll * g;
    const float* t = t_o + 3ll * g;
    const int b = g / O;
    const bool ego = R_e && !ego_degenerate[b];
    double y0 = __dadd_rn(dot3(R[0], R[1], R[2], c0, c1, c2), (double)t[0]);
    double y1 = __dadd_rn(dot3(R[3], R[4], R[5], c0, c1, c2), (double)t[1]);
    double y2 = __dadd_rn(dot3(R[6], R[7], R[8], c0, c1, c2), (double)t[2]);
    if (ego) {
        const float* Re = R_e + 9ll * b;
        const float* te = t_e + 3ll * b;
        const double w0 = __dsub_rn(y0, (double)te[0]), w1 = __dsub_rn(y1, (double)te[1]), w2 = __dsub_rn(y2, (double)te[2]);
        y0 = dot3(Re[0], Re[3], Re[6], w0, w1, w2);
        y1 = dot3(Re[1], Re[4], Re[7], w0, w1, w2);
        y2 = dot3(Re[2], Re[5], Re[8], w0, w1, w2);
    }
    const double d0 = __dsub_rn(y0, (double)c0), d1 = __dsub_rn(y1, (double)c1), d2 = __dsub_rn(y2, (double)c2);
    // the heading: the length axis points the way the centre moves
    if (__dadd_rn(__dmul_rn(pick(d0, d1, d2, ip), cos(phi)), __dmul_rn(pick(d0, d1, d2, iq), sin(phi))) < 0.0) phi += M_PI;
    if (phi > M_PI) phi -= 2 * M_PI;
    const double cp = cos(phi), sp = sin(phi);
    cg[0] = c0;
    cg[1] = c1;
    cg[2] = c2;
    dg[0] = (float)d0;
    dg[1] = (float)d1;
    dg[2] = (float)d2;
    yaw[g] = (float)phi;
#pragma unroll
    for (int k = 0; k < 9; ++k) rg[k] = 0.f;
    rg[3 * ip] = (float)cp;
    rg[3 * iq] = (float)sp;
    rg[3 * ip + 1] = (float)-sp;
    rg[3 * iq + 1] = (float)cp;
    rg[3 * up + 2] = 1.f;
}

// workspace: the grouping (RmGroupWs) | keys [G,A,4] u32 | hkeys [G,2] u32 | cnt [G] i32, each range 16-byte aligned
struct BoxWs {
    RmGroupWs grp;
    unsigned *keys, *hkeys;
    int32_t* cnt;
    int64_t bytes;
};
static BoxWs box_ws(void* ws, int B, int N, int O, int A) {
    ByteCarve w(ws);
    const long long G = (long long)B * O;
    BoxWs L;
    L.grp = rm_group_carve(w, B, N, O);
    L.keys = w.take<unsigned>(16 * G * A);
    L.hkeys = w.take<unsigned>(8 * G);
    L.cnt = w.take<int32_t>(4 * G);
    L.bytes = w.bytes;
    return L;
}

static bool bad_sizes(int B, int N, int O, int A) {
    return B < 1 || N < 1 || (long long)B * N > 0x7fffffffll || O < 1 || O > kMaxObjects || A < 1 || A > kBoxMaxAngles;
}

}  // namespace pvraft

using namespace pvraft;

extern "C" int64_t pvraft_object_boxes_workspace_bytes(int B, int N, int O, int A) {
    return bad_sizes(B, N, O, A) || (long long)B * O > 65535 ? 0 : box_ws(nullptr, B, N, O, A).bytes;
}

extern "C" int pvraft_object_boxes_fwd(const float* xyz, const int32_t* labels, const float* R_o, const float* t_o, const float* R_e,
                                       const float* t_e, const uint8_t* ego_degenerate, int B, int N, int O, int up, int A, float* center,
                                       float* size, float* yaw, float* rotation, float* displacement, int32_t* count, float* extents,
                                       float* dirs, void* workspace, void* stream) {
    if (!xyz || !labels || !R_o || !t_o || !R_e != !t_e || !R_e != !ego_degenerate || !center || !size || !yaw || !rotation ||
        !displacement || !count || !workspace || bad_sizes(B, N, O, A) || up < 0 || up > 2)
        return fail(PVRAFT_ERR_BAD_ARG, "object_boxes_fwd: bad argument");
    if (reinterpret_cast<uintptr_t>(workspace) & 15) return fail(PVRAFT_ERR_BAD_ARG, "object_boxes_fwd: workspace not 16-byte aligned");
    if ((long long)B * O > 65535) return fail(PVRAFT_ERR_UNSUPPORTED, "object_boxes_fwd: B O = %lld > 65535", (long long)B * O);
    cudaStream_t st = (cudaStream_t)stream;
    const BoxWs L = box_ws(workspace, B, N, O, A);
    const int G = B * O;
    int rc;
    if ((rc = rm_group(labels, B, N, O, L.grp, st))) return rc;
    const long long words = (long long)G * A * 4;
    k_box_clear<<<(unsigned)((words + 255) / 256), 256, 0, st>>>(L.keys, L.hkeys, L.cnt, G, A);
    const int windows = (N + kMomThreads - 1) / kMomThreads;
    k_box_extents<<<dim3((unsigned)(windows + O), (unsigned)B), kMomThreads, 0, st>>>(xyz, labels, L.grp.mitems, L.grp.nm, O, N, up, A,
                                                                                      L.keys, L.hkeys, L.cnt);
    k_box_finalize<<<(unsigned)((G + kBoxWarps - 1) / kBoxWarps), kBoxWarps * kWarp, 0, st>>>(
        L.keys, L.hkeys, L.cnt, R_o, t_o, R_e, t_e, ego_degenerate, G, O, up, A, center, size, yaw, rotation, displacement, count,
        extents, dirs);
    return check_launch("object_boxes_fwd");
}
