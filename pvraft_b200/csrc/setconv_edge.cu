// SetConv edge stage (reference model/flot/gconv.py:65-80): the gather over the 32-NN graph, fc1 on
// [x_j - x_i, rel_xyz], the statistics of gn1 and the max-pool over neighbours, without ever
// materialising the reference's [B, C+3, 32, N] edge tensor.
//
// fc1 is linear and bias-free, so  W.[x_j - x_i, e] = P_j - P_i + W_e.e  with  P = W[:, :cin].x  computed
// once per point by pvraft_linear_fwd; this kernel only gathers the 32 rows P_j.
// GroupNorm + LeakyReLU is monotone per channel, so max_e lrelu(GN(y_e)) = lrelu(GN(max_e y_e)) when the
// folded GN scale is >= 0 and lrelu(GN(min_e y_e)) otherwise: the kernel emits both the per-channel max
// and min of the raw y, plus the double-precision (sum, sum^2) of all N*32*C raw values per group (each point's 32 edges
// summed in fp32 about its first edge's value and converted exactly: pivot_sumsq, csrc/common.cuh).
//
// Persistent and warp-specialised, one CTA per SM.  A CTA walks tiles of kEdgeTile consecutive positions of the processing
// order (edge_plan.cuh), driven by the graph's gather plan (edge_plan.cu): the producer warps bulk-copy tile t + 1's row ids
// and reference slots, then its distinct rows P_j, into the idle half of a double-buffered table while the consumer warps
// compute tile t.  The consumers run one warp per point exactly as a plain gather would: lane l owns the adjacent channel
// pairs (2l, 2l+1) + 64q, a neighbour row is one 8-byte shared-memory load per lane and pair, and the per-edge scalars (row
// offset, edge vector) are read back as ONE broadcast 16-byte shared-memory load.  A tile with more distinct rows than the
// table holds is gathered from global memory instead (an unordered cloud), with the same arithmetic: the results never
// depend on the order nor on the plan.
#include "edge_plan.cuh"
#include "fixed_point.cuh"
#include "tma.cuh"

namespace pvraft {

// Warps per role and form, within the register budget of one CTA per SM and without spills (registers: DESIGN 4.2).  Four
// producer warps issue a tile's row copies, where the budget has room for them beside the consumers; points are dealt to
// the consumers round-robin across tiles, so a count that does not divide kEdgeTile still balances.
constexpr int kEdgeConsumerWarps = 24;                         // at most
__host__ __device__ constexpr int edge_consumer_warps(int pairs, bool det) { return pairs == 1 ? (det ? 16 : 24) : (det ? 8 : 12); }
constexpr int kEdgeProducerWarps = 4;
__host__ __device__ constexpr int edge_threads(int pairs, bool det) { return (edge_consumer_warps(pairs, det) + kEdgeProducerWarps) * 32; }
constexpr int kEdgeTableFloats = 22528;                        // one table buffer: rows = min(kEdgeRefs, this / C)
// named barriers (0 is __syncthreads): the consumers among themselves, "buffer free" (consumers arrive, the producers wait)
constexpr int kBarConsumers = 1, kBarEmpty = 2;


inline int edge_table_rows(int C) { return kEdgeTableFloats / C < kEdgeRefs ? kEdgeTableFloats / C : kEdgeRefs; }

// shared memory after the two table buffers [2][rows][C]
struct EdgeSmem {
    alignas(16) int row[2][kEdgeRefs];     // row id of table slot r (the plan's ids)
    alignas(16) uint16_t slot[2][kEdgeRefs];   // table slot of each reference (the plan's slots)
    unsigned long long meta[2];            // mbarrier: the tile's ids and slots are in place
    unsigned long long full[2];            // mbarrier: the tile's rows are in place
    float4 edge[kEdgeConsumerWarps][32];   // (row offset bits, ex, ey, ez) of a consumer warp's point
    double part[kEdgeConsumerWarps][16];   // per-warp GroupNorm partials (group, moment)
    unsigned long long fx[16 * kFxWords];  // DET: the CTA's fixed-point (group, moment) sums
};

__device__ __forceinline__ void cp_async16(void* dst, const void* src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(dst)), "l"(src) : "memory");
}
// one arrival on the mbarrier once every cp.async this thread has issued so far has landed
__device__ __forceinline__ void cp_async_arrive(void* bar) {
    asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void bar_sync(int id, int n) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory"); }
__device__ __forceinline__ void bar_arrive(int id, int n) { asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(n) : "memory"); }

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

template <bool TABLE>
__device__ __forceinline__ float2 ld_row(const float* p) {
    if constexpr (TABLE) return *reinterpret_cast<const float2*>(p);   // LDS.64 from the shared table
    else return __ldg(reinterpret_cast<const float2*>(p));
}

// y = (P_j - P_i) + fma(w_z, e_z, fma(w_y, e_y, w_x * e_x)) of one edge, both channels of a pair at once.  ed: the edge's
// (row offset, edge vector); pi: the centre's pair
template <bool TABLE>
__device__ __forceinline__ unsigned long long edge_y2(const float* rows, const float4& ed, int coff, unsigned long long pi,
                                                      unsigned long long wx2, unsigned long long wy2, unsigned long long wz2) {
    const float2 pj = ld_row<TABLE>(rows + __float_as_int(ed.x) + coff);
    const unsigned long long t = fma2(wz2, pk(ed.w, ed.w), fma2(wy2, pk(ed.z, ed.z), mul2(wx2, pk(ed.y, ed.y))));
    return add2(sub2(pk(pj.x, pj.y), pi), t);
}

// one point: y_e = (P_j - P_i) + W_e.e over the 32 edges in order 0..31 -> per-channel max, min, and the sum and sum of
// squares of y_e - piv with the pivot piv = y_0 (pivot_sumsq).  The sum is of y_e - piv too, uncompensated: a compensated
// sum does not fit the register budget of the one-pair form (it spills), so a point's mean carries ~2^-24 of its spread.
// rows: the shared table (TABLE) or the sample's P; se: the warp's (row offset, edge vector) list; ctr: the centre row P_i
template <int PAIRS, bool TABLE>
__device__ __forceinline__ void edge_point(const float* rows, const float4* se, const float* ctr, const int (&coff)[PAIRS],
                                           const unsigned long long (&wx2)[PAIRS], const unsigned long long (&wy2)[PAIRS],
                                           const unsigned long long (&wz2)[PAIRS], float2 (&mx)[PAIRS], float2 (&mn)[PAIRS],
                                           unsigned long long (&piv)[PAIRS], unsigned long long (&s1)[PAIRS],
                                           unsigned long long (&s2)[PAIRS]) {
    unsigned long long pi[PAIRS];
#pragma unroll
    for (int q = 0; q < PAIRS; ++q) {
        const float2 t = ld_row<TABLE>(ctr + coff[q]);
        pi[q] = pk(t.x, t.y);
        piv[q] = edge_y2<TABLE>(rows, se[0], coff[q], pi[q], wx2[q], wy2[q], wz2[q]);
        mx[q] = make_float2(-INFINITY, -INFINITY); mn[q] = make_float2(INFINITY, INFINITY);
        s1[q] = pk(0.f, 0.f); s2[q] = pk(0.f, 0.f);
    }
#pragma unroll 8
    for (int e = 0; e < 32; ++e) {
        const float4 ed = se[e];
#pragma unroll
        for (int q = 0; q < PAIRS; ++q) {
            const unsigned long long y2 = edge_y2<TABLE>(rows, ed, coff[q], pi[q], wx2[q], wy2[q], wz2[q]);
            const float2 y = upk(y2);
            mx[q].x = fmaxf(mx[q].x, y.x); mx[q].y = fmaxf(mx[q].y, y.y);
            mn[q].x = fminf(mn[q].x, y.x); mn[q].y = fminf(mn[q].y, y.y);
            const unsigned long long d2 = sub2(y2, piv[q]);
            s1[q] = add2(s1[q], d2);
            s2[q] = fma2(d2, d2, s2[q]);
        }
    }
}

// DET: every point's per-channel (sum, sum^2) over its 32 edges enters a per-lane fixed-point register sum, and those enter the
// [B,16] fixed-point workspace `stats` points at then (fixed_point.cuh): the sums do not depend on which CTA took which points
template <int PAIRS, bool DET>
__global__ void __launch_bounds__(edge_threads(PAIRS, DET), 1) k_setconv_edge_pairs(const float* __restrict__ fc1p, const int32_t* __restrict__ nbr,
                                                                     const float* __restrict__ edge_feats, const float* __restrict__ w_fc1,
                                                                     int cin, int B, int N, int C, float* __restrict__ ymax,
                                                                     float* __restrict__ ymin, Acc<DET, double> stats,
                                                                     const int32_t* __restrict__ order, const unsigned char* __restrict__ plan,
                                                                     int rows) {
    constexpr int CW = edge_consumer_warps(PAIRS, DET), kConsumers = CW * 32, kThreads = edge_threads(PAIRS, DET);
    constexpr int PW = kEdgeProducerWarps;
    static_assert(CW <= kEdgeConsumerWarps, "work split");
    extern __shared__ __align__(128) unsigned char smem[];
    float* tables = reinterpret_cast<float*>(smem);   // [2][rows][C]
    EdgeSmem& s = *reinterpret_cast<EdgeSmem*>(smem + (size_t)2 * rows * C * sizeof(float));
    pdl_trigger();   // the next kernel may be staged while this one drains
    if (threadIdx.x == 0) {
        for (int i = 0; i < 2; ++i) {
            mbar_init(&s.meta[i], 1);    // the producer's expect_tx, then the bulk copies' bytes
            mbar_init(&s.full[i], PW * 32);   // per producer thread: the landing of its row copies
        }
        fence_mbarrier_init();
    }
    __syncthreads();
    pdl_wait();      // (launched with PDL: nothing above touches global memory; P is the previous launch's output)
    const int lane = lane_id(), w = warp_id();
    const int tps = edge_tiles_per_sample(N);
    long long t_begin, t_end;
    split_range((long long)B * tps, gridDim.x, blockIdx.x, t_begin, t_end);
    const int ntiles = (int)(t_end - t_begin);

    if (w >= CW) {   // ---- producers: tile k into buffer k & 1 ----
        const int pw = w - CW;
        const int chunks = C / 4, rows_per_copy = 32 / chunks, copy_row = lane / chunks, copy_chunk = lane - copy_row * chunks;
        const int* count = reinterpret_cast<const int*>(plan + kEdgePlanCount);   // (of tile t at t * kEdgePlanBytes / 4)
        int n = ntiles > 0 ? __ldg(count + t_begin * (kEdgePlanBytes / 4)) : 0;
        for (int k = 0; k < ntiles; ++k) {
            const int buf = k & 1;
            const long long t = t_begin + k;
            const int b = (int)(t / tps);
            const unsigned char* rec = plan + t * kEdgePlanBytes;
            const bool in_table = n <= rows;   // an overflowing tile copies no rows (its consumers gather from global memory)
            if (k >= 2) bar_sync(kBarEmpty + buf, kThreads);   // the consumers are done with tile k - 2
            if (pw == 0 && lane == 0) {
                const unsigned id_bytes = in_table ? (unsigned)(n * 4 + 15) & ~15u : 0u;
                mbar_expect_tx(&s.meta[buf], id_bytes + kEdgeRefs * 2);
                if (id_bytes) bulk_g2s(s.row[buf], rec, id_bytes, &s.meta[buf]);
                bulk_g2s(s.slot[buf], rec + kEdgePlanSlots, kEdgeRefs * 2, &s.meta[buf]);
            }
            if (in_table && copy_row < rows_per_copy) {
                // the distinct rows -> the table: a warp copies rows_per_copy rows of C / 4 16-byte chunks per instruction
                mbar_wait(&s.meta[buf], (unsigned)(k >> 1) & 1u);
                const float* P = fc1p + (size_t)b * N * C + 4 * copy_chunk;
                float* table = tables + (size_t)buf * rows * C + 4 * copy_chunk;
#pragma unroll 1
                for (int r = pw * rows_per_copy + copy_row; r < n; r += PW * rows_per_copy)
                    cp_async16(table + (size_t)r * C, P + (size_t)s.row[buf][r] * C);
            }
            cp_async_arrive(&s.full[buf]);   // (when this thread's copies have landed)
            if (k + 1 < ntiles) n = __ldg(count + (t + 1) * (kEdgePlanBytes / 4));
        }
        return;
    }

    // ---- consumers: one warp per point ----
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
    bool on[PAIRS];   // C need not fill the last group of 64 channels (encoder layers: 16, 48, 96)
    int coff[PAIRS];
#pragma unroll
    for (int q = 0; q < PAIRS; ++q) { on[q] = 2 * lane + 64 * q < C; coff[q] = on[q] ? 2 * lane + 64 * q : 0; }
    const int gsz = C / PVRAFT_GN_GROUPS;
    double dS[PAIRS][2], dSS[PAIRS][2];
    Fx fS[PAIRS][2], fSS[PAIRS][2];
    auto reset = [&]() {
#pragma unroll
        for (int q = 0; q < PAIRS; ++q)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                dS[q][h] = dSS[q][h] = 0.0;
                if constexpr (DET) fS[q][h] = fSS[q][h] = Fx{0ull, 0ull, 0u};
            }
    };
    // the consumers' partials of sample b -> one global addition per (group, moment) and CTA
    auto flush = [&](int b) {
        if constexpr (DET) {
            const FxSlots sfx{s.fx};
            bar_sync(kBarConsumers, kConsumers);
            fx_stage_zero(sfx, 16, kConsumers);
            bar_sync(kBarConsumers, kConsumers);
#pragma unroll
            for (int q = 0; q < PAIRS; ++q)
#pragma unroll
                for (int h = 0; h < 2; ++h)
                    if (on[q]) {
                        const int g = (2 * lane + 64 * q + h) / gsz;
                        add(sfx, g * 2, fS[q][h]);
                        add(sfx, g * 2 + 1, fSS[q][h]);
                    }
            bar_sync(kBarConsumers, kConsumers);
            fx_stage_flush(sfx, 16, stats + b * 16, kConsumers);
        } else {
            bar_sync(kBarConsumers, kConsumers);   // (the previous flush has read s.part)
#pragma unroll
            for (int g = 0; g < PVRAFT_GN_GROUPS; ++g) {
                double a = 0.0, a2 = 0.0;
#pragma unroll
                for (int q = 0; q < PAIRS; ++q)
#pragma unroll
                    for (int h = 0; h < 2; ++h)
                        if (on[q] && (2 * lane + 64 * q + h) / gsz == g) { a += dS[q][h]; a2 += dSS[q][h]; }
#pragma unroll
                for (int o = 16; o; o >>= 1) { a += __shfl_xor_sync(kFull, a, o); a2 += __shfl_xor_sync(kFull, a2, o); }
                if (lane == 0) { s.part[w][2 * g] = a; s.part[w][2 * g + 1] = a2; }
            }
            bar_sync(kBarConsumers, kConsumers);
            if (threadIdx.x < 16) {
                double acc = 0.0;
                for (int ww = 0; ww < CW; ++ww) acc += s.part[ww][threadIdx.x];
                if (acc != 0.0) atomicAdd(stats + (size_t)b * 16 + threadIdx.x, acc);
            }
        }
        reset();
    };
    reset();
    int cur = -1;   // the sample whose partials the registers hold
    int deal = 0;   // the consumer warp that takes the next point: points are dealt round-robin across tiles
    for (int k = 0; k < ntiles; ++k) {
        const int buf = k & 1;
        const long long t = t_begin + k;
        const int b = (int)(t / tps), start = (int)(t - (long long)b * tps) * kEdgeTile, len = min(kEdgeTile, N - start);
        if (b != cur) {
            if (cur >= 0) flush(cur);
            cur = b;
        }
        const int p0 = w >= deal ? w - deal : w - deal + CW;   // this warp's first point of the tile
        deal = (deal + len) % CW;
        // the global reads that do not need the table, issued before waiting for it: the ids and edge vectors of the warp's points
        constexpr int U = (kEdgeTile + CW - 1) / CW;
        int pid[U];
        float3 pe[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const int p = p0 + u * CW;
            pid[u] = p < len ? (order ? __ldg(order + (long long)b * N + start + p) : start + p) : 0;
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
            // lane e parks neighbour e: its row offset and edge feature x_j - x_i (graph.edge_feats, gconv.py:66)
            const float* ef = edge_feats + (((size_t)b * N + pid[u]) * 32 + lane) * 3;
            pe[u] = p0 + u * CW < len ? make_float3(__ldg(ef), __ldg(ef + 1), __ldg(ef + 2)) : make_float3(0.f, 0.f, 0.f);
        }
        const bool in_table = __ldg(reinterpret_cast<const int*>(plan + t * kEdgePlanBytes + kEdgePlanCount)) <= rows;
        mbar_wait(&s.meta[buf], (unsigned)(k >> 1) & 1u);
        mbar_wait(&s.full[buf], (unsigned)(k >> 1) & 1u);
        const float* P = fc1p + (size_t)b * N * C;
        const float* table = tables + (size_t)buf * rows * C;
#pragma unroll 1
        for (int p = p0; p < len; p += CW) {
            const int i = pid[0];
            const float3 e = pe[0];
#pragma unroll
            for (int u = 0; u + 1 < U; ++u) { pid[u] = pid[u + 1]; pe[u] = pe[u + 1]; }
            const long long pt = (long long)b * N + i;
            const int off = (in_table ? (int)s.slot[buf][p * 32 + lane] : __ldg(nbr + pt * 32 + lane)) * C;
            __syncwarp();
            s.edge[w][lane] = make_float4(__int_as_float(off), e.x, e.y, e.z);
            __syncwarp();
            float2 mx[PAIRS], mn[PAIRS];
            unsigned long long piv[PAIRS], s1[PAIRS], s2[PAIRS];
            if (in_table)
                edge_point<PAIRS, true>(table, s.edge[w], table + s.slot[buf][kEdgeTile * 32 + p] * C, coff, wx2, wy2, wz2, mx, mn, piv, s1, s2);
            else
                edge_point<PAIRS, false>(P, s.edge[w], P + (size_t)i * C, coff, wx2, wy2, wz2, mx, mn, piv, s1, s2);
#pragma unroll
            for (int q = 0; q < PAIRS; ++q) {
                const size_t o = (size_t)pt * C + coff[q];
                if (on[q]) {
                    *reinterpret_cast<float2*>(ymax + o) = mx[q];
                    *reinterpret_cast<float2*>(ymin + o) = mn[q];
                }
                const float2 pv = upk(piv[q]), a1 = upk(s1[q]), a2 = upk(s2[q]);
                const double t1[2] = {fma(32.0, (double)pv.x, (double)a1.x), fma(32.0, (double)pv.y, (double)a1.y)};
                const double t2[2] = {pivot_sumsq(t1[0], pv.x, a2.x, 32), pivot_sumsq(t1[1], pv.y, a2.y, 32)};
                if constexpr (DET) {
                    fx_add(fS[q][0], fx_from(t1[0])); fx_add(fS[q][1], fx_from(t1[1]));
                    fx_add(fSS[q][0], fx_from(t2[0])); fx_add(fSS[q][1], fx_from(t2[1]));
                } else {
                    dS[q][0] += t1[0]; dS[q][1] += t1[1];
                    dSS[q][0] += t2[0]; dSS[q][1] += t2[1];
                }
            }
        }
        if (k + 2 < ntiles) bar_arrive(kBarEmpty + buf, kThreads);   // the producers may refill this buffer with tile k + 2
    }
    if (cur >= 0) flush(cur);
}

}  // namespace pvraft

using namespace pvraft;

template <bool DET>
static int setconv_edge_fwd(const float* fc1p, const int32_t* nbr, const float* edge_feats, const float* w_fc1, int cin, int B, int N, int C,
                            float* ymax, float* ymin, double* stats, const int32_t* order, const void* plan, void* ws, void* stream) {
    if (!fc1p || !nbr || !edge_feats || !w_fc1 || !ymax || !ymin || !stats || !plan) return fail(PVRAFT_ERR_BAD_ARG, "setconv_edge: null pointer");
    if (B <= 0 || N <= 0 || cin <= 0) return fail(PVRAFT_ERR_BAD_ARG, "setconv_edge: bad shape");
    if (C <= 0 || C > 128 || C % PVRAFT_GN_GROUPS) return fail(PVRAFT_ERR_UNSUPPORTED, "setconv_edge: C=%d (multiple of 8, <= 128)", C);
    if (reinterpret_cast<uintptr_t>(fc1p) % 16) return fail(PVRAFT_ERR_BAD_ARG, "setconv_edge: fc1p must be 16-byte aligned (rows are bulk-copied)");
    if (reinterpret_cast<uintptr_t>(plan) % 16) return fail(PVRAFT_ERR_BAD_ARG, "setconv_edge: plan must be 16-byte aligned");
    const int rows = edge_table_rows(C);
    const size_t smem = (size_t)2 * rows * C * sizeof(float) + sizeof(EdgeSmem);
    const long long tiles = (long long)B * edge_tiles_per_sample(N);
    long long g = sm_count();
    if (g > tiles) g = tiles;
    const int grid = (int)g;
    cudaStream_t st = (cudaStream_t)stream;
    Acc<DET, double> kstats;   // DET: the [B,16] workspace
    if constexpr (DET) kstats = fx_slots(ws);
    else kstats = stats;
    const auto kernel = C <= 64 ? k_setconv_edge_pairs<1, DET> : k_setconv_edge_pairs<2, DET>;
    int rc;
    if ((rc = opt_in_smem(kernel, smem))) return rc;
    launch_pdl(kernel, grid, edge_threads(C <= 64 ? 1 : 2, DET), smem, st, fc1p, nbr, edge_feats, w_fc1, cin, B, N, C, ymax, ymin, kstats, order,
               static_cast<const unsigned char*>(plan), rows);
    rc = check_launch("setconv_edge");
    if (rc || !DET) return rc;
    return gn_stats_flush(ws, B, stats, st);
}

extern "C" int pvraft_setconv_edge_fwd(const float* fc1p, const int32_t* nbr, const float* edge_feats, const float* w_fc1, int cin,
                                       int B, int N, int C, float* ymax, float* ymin, double* stats, const int32_t* order,
                                       const void* plan, void* det_workspace, void* stream) {
    auto f = det_workspace ? setconv_edge_fwd<true> : setconv_edge_fwd<false>;
    return f(fc1p, nbr, edge_feats, w_fc1, cin, B, N, C, ymax, ymin, stats, order, plan, det_workspace, stream);
}

extern "C" int64_t pvraft_setconv_edge_det_workspace_bytes(int B) { return gn_stats_ws_bytes(B); }
