// SetConv edge stage (reference model/flot/gconv.py:65-80): the gather over the 32-NN graph, fc1 on
// [x_j - x_i, rel_xyz], the statistics of gn1 and the max-pool over neighbours, without ever
// materialising the reference's [B, C+3, 32, N] edge tensor.
//
// fc1 is linear and bias-free, so  W.[x_j - x_i, e] = P_j - P_i + W_e.e  with  P = W[:, :cin].x  computed
// once per point by pvraft_linear_fwd; this kernel only gathers the 32 rows P_j (L2-resident table).
// GroupNorm + LeakyReLU is monotone per channel, so max_e lrelu(GN(y_e)) = lrelu(GN(max_e y_e)) when the
// folded GN scale is >= 0 and lrelu(GN(min_e y_e)) otherwise: the kernel emits both the per-channel max
// and min of the raw y, plus the double-precision (sum, sum^2) of all N*32*C raw values per group.
//
// One warp per point; lane l owns the adjacent channel pairs (2l, 2l+1) + 64q: a neighbour row is one 8-byte load per lane
// and pair, and the per-edge scalars (neighbour id, edge vector) are read back as ONE broadcast 16-byte shared-memory load.
#include "fixed_point.cuh"

namespace pvraft {

constexpr int kEdgeThreads = 256;

// elementwise arithmetic on channel pairs held as one 64-bit value: each component is one IEEE round-to-nearest operation
// (the _rn intrinsics are never contracted into an FMA)
__device__ __forceinline__ unsigned long long pk(float lo, float hi) {
    unsigned long long r;
    asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(lo), "f"(hi));
    return r;
}
__device__ __forceinline__ float2 upk(unsigned long long v) {
    float2 d;
    asm("mov.b64 {%0, %1}, %2;" : "=f"(d.x), "=f"(d.y) : "l"(v));
    return d;
}
__device__ __forceinline__ unsigned long long fma2(unsigned long long a, unsigned long long b, unsigned long long c) {
    const float2 x = upk(a), y = upk(b), z = upk(c);
    return pk(__fmaf_rn(x.x, y.x, z.x), __fmaf_rn(x.y, y.y, z.y));
}
__device__ __forceinline__ unsigned long long mul2(unsigned long long a, unsigned long long b) {
    const float2 x = upk(a), y = upk(b);
    return pk(__fmul_rn(x.x, y.x), __fmul_rn(x.y, y.y));
}
__device__ __forceinline__ unsigned long long add2(unsigned long long a, unsigned long long b) {
    const float2 x = upk(a), y = upk(b);
    return pk(__fadd_rn(x.x, y.x), __fadd_rn(x.y, y.y));
}
__device__ __forceinline__ unsigned long long sub2(unsigned long long a, unsigned long long b) {
    const float2 x = upk(a), y = upk(b);
    return pk(__fsub_rn(x.x, y.x), __fsub_rn(x.y, y.y));
}

// DET: every point's per-channel (sum, sum^2) over its 32 edges enters a per-lane fixed-point register sum, and those enter the
// [B,16] fixed-point workspace `stats` points at then (fixed_point.cuh): the sums do not depend on which CTA took which points
template <int PAIRS, bool DET>
__global__ void __launch_bounds__(kEdgeThreads, DET ? 2 : (PAIRS == 1 ? 6 : 4)) k_setconv_edge_pairs(const float* __restrict__ fc1p, const int32_t* __restrict__ nbr,
                                                                     const float* __restrict__ edge_feats, const float* __restrict__ w_fc1,
                                                                     int cin, int B, int N, int C, float* __restrict__ ymax,
                                                                     float* __restrict__ ymin, double* __restrict__ stats,
                                                                     const int32_t* __restrict__ order) {
    __shared__ double s_part[kEdgeThreads / 32][128][2];
    __shared__ __align__(16) float4 s_edge[kEdgeThreads / 32][32];   // (neighbour id bits, ex, ey, ez) of the warp's point
    pdl_trigger();   // the next kernel may be staged while this one drains
    pdl_wait();      // (launched with PDL: nothing above touches global memory)
    const int lane = lane_id(), w = warp_id(), nwarps = kEdgeThreads / 32;
    const int ld = cin + 3;
    float2 wx[PAIRS], wy[PAIRS], wz[PAIRS];
#pragma unroll
    for (int q = 0; q < PAIRS; ++q) {
        const int c = min(2 * lane + 64 * q, C - 2);   // (lanes past C replicate the last pair; their results are dropped)
        wx[q] = make_float2(__ldg(w_fc1 + (size_t)c * ld + cin + 0), __ldg(w_fc1 + (size_t)(c + 1) * ld + cin + 0));
        wy[q] = make_float2(__ldg(w_fc1 + (size_t)c * ld + cin + 1), __ldg(w_fc1 + (size_t)(c + 1) * ld + cin + 1));
        wz[q] = make_float2(__ldg(w_fc1 + (size_t)c * ld + cin + 2), __ldg(w_fc1 + (size_t)(c + 1) * ld + cin + 2));
    }
    unsigned long long wx2[PAIRS], wy2[PAIRS], wz2[PAIRS];
#pragma unroll
    for (int q = 0; q < PAIRS; ++q) { wx2[q] = pk(wx[q].x, wx[q].y); wy2[q] = pk(wy[q].x, wy[q].y); wz2[q] = pk(wz[q].x, wz[q].y); }
    const long long total = (long long)B * N;
    long long pt_begin, pt_end;
    split_range(total, gridDim.x, blockIdx.x, pt_begin, pt_end);   // (handing SM-mates adjacent ranges was measured: no gain)
    long long seg = pt_begin;
    while (seg < pt_end) {
        const int b = (int)(seg / N);
        long long seg_end = (long long)(b + 1) * N;
        if (seg_end > pt_end) seg_end = pt_end;
        double dS[PAIRS][2], dSS[PAIRS][2];
#pragma unroll
        for (int q = 0; q < PAIRS; ++q) { dS[q][0] = dS[q][1] = 0.0; dSS[q][0] = dSS[q][1] = 0.0; }
        Fx fS[PAIRS][2], fSS[PAIRS][2];
        if constexpr (DET) {
#pragma unroll
            for (int q = 0; q < PAIRS; ++q)
#pragma unroll
                for (int h = 0; h < 2; ++h) fS[q][h] = fSS[q][h] = Fx{0ull, 0ull, 0u};
        }
        bool on[PAIRS];   // C need not fill the last group of 64 channels (encoder layers: 16, 48, 96)
        int coff[PAIRS];
#pragma unroll
        for (int q = 0; q < PAIRS; ++q) { on[q] = 2 * lane + 64 * q < C; coff[q] = on[q] ? 2 * lane + 64 * q : 0; }
        const float* P = fc1p + (size_t)b * N * C;
        for (long long r = seg + w; r < seg_end; r += nwarps) {
            // processing order: with `order` (a space-filling-curve rank -> point table) the 8 warps of a CTA work on spatial
            // neighbours at the same time, whose 32-neighbourhoods overlap: their gathers hit the same rows in L1
            const int i = order ? __ldg(order + r) : (int)(r - (long long)b * N);
            const long long pt = (long long)b * N + i;
            // lane e parks neighbour e: id and edge feature x_j - x_i (graph.edge_feats, gconv.py:66)
            const float* ef = edge_feats + ((size_t)pt * 32 + lane) * 3;
            __syncwarp();
            s_edge[w][lane] = make_float4(__int_as_float(__ldg(nbr + pt * 32 + lane) * C), __ldg(ef), __ldg(ef + 1), __ldg(ef + 2));
            __syncwarp();
            unsigned long long pi[PAIRS], s1[PAIRS], s2[PAIRS];
            float2 mx[PAIRS], mn[PAIRS];
#pragma unroll
            for (int q = 0; q < PAIRS; ++q) {
                const float2 t = __ldg(reinterpret_cast<const float2*>(P + (size_t)i * C + coff[q]));
                pi[q] = pk(t.x, t.y);
                mx[q] = make_float2(-INFINITY, -INFINITY); mn[q] = make_float2(INFINITY, INFINITY);
                s1[q] = pk(0.f, 0.f); s2[q] = pk(0.f, 0.f);
            }
#pragma unroll 8
            for (int e = 0; e < 32; ++e) {
                const float4 ed = s_edge[w][e];
                const float* row = P + __float_as_int(ed.x);
                const unsigned long long ex = pk(ed.y, ed.y), ey = pk(ed.z, ed.z), ez = pk(ed.w, ed.w);
#pragma unroll
                for (int q = 0; q < PAIRS; ++q) {
                    const float2 pj = __ldg(reinterpret_cast<const float2*>(row + coff[q]));
                    // y = (P_j - P_i) + fma(w_z, e_z, fma(w_y, e_y, w_x * e_x)), both channels of the pair at once
                    const unsigned long long t = fma2(wz2[q], ez, fma2(wy2[q], ey, mul2(wx2[q], ex)));
                    const unsigned long long y2 = add2(sub2(pk(pj.x, pj.y), pi[q]), t);
                    const float2 y = upk(y2);
                    mx[q].x = fmaxf(mx[q].x, y.x); mx[q].y = fmaxf(mx[q].y, y.y);
                    mn[q].x = fminf(mn[q].x, y.x); mn[q].y = fminf(mn[q].y, y.y);
                    s1[q] = add2(s1[q], y2);
                    s2[q] = fma2(y2, y2, s2[q]);
                }
            }
#pragma unroll
            for (int q = 0; q < PAIRS; ++q) {
                const size_t o = (size_t)pt * C + coff[q];
                if (on[q]) {
                    *reinterpret_cast<float2*>(ymax + o) = mx[q];
                    *reinterpret_cast<float2*>(ymin + o) = mn[q];
                }
                const float2 a1 = upk(s1[q]), a2 = upk(s2[q]);
                if constexpr (DET) {
                    fx_add(fS[q][0], fx_from((double)a1.x)); fx_add(fS[q][1], fx_from((double)a1.y));
                    fx_add(fSS[q][0], fx_from((double)a2.x)); fx_add(fSS[q][1], fx_from((double)a2.y));
                } else {
                dS[q][0] += (double)a1.x; dS[q][1] += (double)a1.y;
                dSS[q][0] += (double)a2.x; dSS[q][1] += (double)a2.y;
                }
            }
        }
        if constexpr (DET) {   // lanes -> the CTA's shared slots -> one global addition per (group, moment)
            __shared__ unsigned long long s_fx[16 * kFxWords];
            __syncthreads();
            if (threadIdx.x < 16 * kFxWords) s_fx[threadIdx.x] = 0ull;
            __syncthreads();
            const int gsz = C / PVRAFT_GN_GROUPS;
#pragma unroll
            for (int q = 0; q < PAIRS; ++q)
#pragma unroll
                for (int h = 0; h < 2; ++h)
                    if (on[q]) {
                        const int g = (2 * lane + 64 * q + h) / gsz;
                        fx_atomic(s_fx + (g * 2) * kFxWords, fS[q][h]);
                        fx_atomic(s_fx + (g * 2 + 1) * kFxWords, fSS[q][h]);
                    }
            __syncthreads();
            if (threadIdx.x < 16) {
                const Fx v{s_fx[threadIdx.x * kFxWords], s_fx[threadIdx.x * kFxWords + 1], (unsigned)s_fx[threadIdx.x * kFxWords + 2]};
                fx_atomic(reinterpret_cast<unsigned long long*>(stats) + ((size_t)b * 16 + threadIdx.x) * kFxWords, v);
            }
            seg = seg_end;
            continue;
        }
        // block reduction of the per-channel partials -> per-group sums -> one atomic per (group, moment)
        __syncthreads();
#pragma unroll
        for (int q = 0; q < PAIRS; ++q) {
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                if (on[q]) {
                    s_part[w][2 * lane + 64 * q + h][0] = dS[q][h];
                    s_part[w][2 * lane + 64 * q + h][1] = dSS[q][h];
                }
            }
        }
        __syncthreads();
        if (threadIdx.x < 16) {
            const int g = threadIdx.x >> 1, m = threadIdx.x & 1, gsz = C / PVRAFT_GN_GROUPS;
            double acc = 0.0;
            for (int c = g * gsz; c < (g + 1) * gsz; ++c)
                for (int ww = 0; ww < nwarps; ++ww) acc += s_part[ww][c][m];
            if (acc != 0.0) atomicAdd(stats + (size_t)b * 16 + threadIdx.x, acc);
        }
        seg = seg_end;
    }
}

}  // namespace pvraft

using namespace pvraft;

template <bool DET>
static int setconv_edge_fwd(const float* fc1p, const int32_t* nbr, const float* edge_feats, const float* w_fc1, int cin, int B, int N, int C,
                            float* ymax, float* ymin, double* stats, const int32_t* order, void* ws, void* stream) {
    if (!fc1p || !nbr || !edge_feats || !w_fc1 || !ymax || !ymin || !stats) return fail(PVRAFT_ERR_BAD_ARG, "setconv_edge: null pointer");
    if (B <= 0 || N <= 0 || cin <= 0) return fail(PVRAFT_ERR_BAD_ARG, "setconv_edge: bad shape");
    if (C <= 0 || C > 128 || C % PVRAFT_GN_GROUPS) return fail(PVRAFT_ERR_UNSUPPORTED, "setconv_edge: C=%d (multiple of 8, <= 128)", C);
    const long long total = (long long)B * N;
    long long g = (long long)sm_count() * 8;
    const long long need = (total + (kEdgeThreads / 32) - 1) / (kEdgeThreads / 32);
    if (g > need) g = need;
    const int grid = (int)(g < 1 ? 1 : g);
    cudaStream_t st = (cudaStream_t)stream;
    double* kstats = DET ? static_cast<double*>(ws) : stats;
    if (C <= 64) launch_pdl(k_setconv_edge_pairs<1, DET>, grid, kEdgeThreads, 0, st, fc1p, nbr, edge_feats, w_fc1, cin, B, N, C, ymax, ymin, kstats, order);
    else launch_pdl(k_setconv_edge_pairs<2, DET>, grid, kEdgeThreads, 0, st, fc1p, nbr, edge_feats, w_fc1, cin, B, N, C, ymax, ymin, kstats, order);
    const int rc = check_launch("setconv_edge");
    if (rc || !DET) return rc;
    return fx_flush_f64(static_cast<const unsigned long long*>(ws), 1, (long long)B * 16, (long long)B * 16, 0, stats, st);
}

extern "C" int pvraft_setconv_edge_fwd(const float* fc1p, const int32_t* nbr, const float* edge_feats, const float* w_fc1, int cin,
                                       int B, int N, int C, float* ymax, float* ymin, double* stats, const int32_t* order,
                                       void* det_workspace, void* stream) {
    auto f = det_workspace ? setconv_edge_fwd<true> : setconv_edge_fwd<false>;
    return f(fc1p, nbr, edge_feats, w_fc1, cin, B, N, C, ymax, ymin, stats, order, det_workspace, stream);
}

extern "C" int64_t pvraft_setconv_edge_det_workspace_bytes(int B) { return (int64_t)B * 16 * kFxWords * 8; }
