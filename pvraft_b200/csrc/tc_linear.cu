// Per-point linear layers on the Hopper tensor cores (wgmma), fp32-accurate (3xTF32), with the GroupNorm / activation
// prologue and the bias / activation / residual / GroupNorm-statistics / GRU-gate epilogues fused around the MMA.
//
//   out[M x N] = epilogue( prologue(A)[M x K] . W[N x K]^T )          M = B*Npts points, N = cout, K = cin
//
// Persistent kernel, one CTA (17 warps) per SM, tiles of 128 consecutive points, 32-channel k-blocks:
//   warp 16      TMA producer: raw fp32 activation boxes [128 x 32] (SWIZZLE_128B; up to three source tensors concatenated
//                along K, e.g. [h | inp | motion] for the GRU) into a ring of 2..6 stages; the pre-split weight boxes
//                W_hi, W_lo once per CTA when they fit next to the ring, else with every k-block
//   warps 8-15   two warpgroups, one per 64-row half of the tile.  Each transforms its rows of the raw box in place: every
//                16-byte chunk gets the folded GroupNorm affine + activation of its channels (optionally choosing the max or
//                the min input by the sign of the scale), is split into hi = tf32(x), lo = tf32(x - hi) and written AT THE
//                SAME swizzled offset (the split is elementwise); fence.proxy.async; then it issues A_hi.W_hi + A_lo.W_hi +
//                A_hi.W_lo = 3 x 4 wgmma.m64nNk8.tf32 and transforms the next k-block while they run.  At the end of a tile
//                the accumulator registers go to a shared-memory tile [128 rows][N] and the warpgroup moves on
//   warps 0-7    epilogue, two per 32-row lane quadrant, one tile behind the MMA: thread = row reads its accumulator row ->
//                bias / activation / residual -> transpose through shared memory -> coalesced stores; GroupNorm (sum,
//                sum^2) of the output combined across the warps into one double atomic per (group, moment) and tile;
//                ConvGRU-gate, cat-tail and flow-head (64 -> 3 + RAFT coordinate update) variants
// Launched with programmatic stream serialization: the prologue overlaps the previous kernel's tail (griddepcontrol.wait
// precedes the first global read).  Replaces the k_linear / k_gru / k_corrfeat / k_flowout CUDA-core kernels whenever
// Npts % 128 == 0 and every source has a multiple of 32 channels.
#include <cuda.h>
#include <stdlib.h>

#include "fixed_point.cuh"
#include "wgmma.cuh"

namespace pvraft {

constexpr int kTcThreads = 544;   // 8 epilogue warps | 2 transform + MMA warpgroups | TMA producer
constexpr int kTcEpiThreads = 256, kTcProducerWarp = 16;
constexpr int kTcM = 128, kTcKB = 32;
constexpr int kTcABytes = kTcM * kTcKB * 4;   // 16 KB: one activation box
constexpr int kTcMaxStages = 6;

// In-kernel timeline of CTA 0 (how the pipeline was tuned, tools/tc_clock.py): compiled in only with -DPVRAFT_TC_TIMELINE
// and then recorded when PVRAFT_TC_DBG=1; the product build carries none of it.
#ifdef PVRAFT_TC_TIMELINE
__device__ unsigned long long g_tc_clock[64];
__device__ __forceinline__ unsigned long long gtimer() { unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); return t; }
#define TC_MARK(cond, slot) do { if (clk && (cond)) g_tc_clock[(slot)] = gtimer(); } while (0)
#else
#define TC_MARK(cond, slot) do { } while (0)
#endif

enum TcEpilogue { TC_EPI_PLAIN = 0, TC_EPI_GRU_ZR = 1, TC_EPI_GRU_Q = 2, TC_EPI_FLOW = 3 };

struct TcParams {
    // prologue (per input channel, per sample): x = act(raw * scale + shift); raw = max or min input by sign(scale)
    const double* in_stats;   // [B,8,2] or null (plain)
    const float* in_gamma;
    const float* in_beta;
    double in_count;
    int in_act;
    float in_slope;
    int minmax;               // 1: second raw source holds the per-channel minima
    // epilogue
    int epi;
    const float* bias;        // [N] or null
    const float* bias2;       // GRU_ZR: bias of r
    int out_act;
    const float* residual;    // [M,N] or null
    float* out;               // [M,N]   (GRU_ZR: z [M,64]; GRU_Q: new hidden state [M,64])
    float* out2;              // GRU_ZR: r*h [M,64]
    const float* h;           // GRU: previous hidden state [M,64]
    const float* z;           // GRU_Q: update gate [M,64]
    double* out_stats;        // [B,8,2] or null
    int M, N, K, cout, pts_per_sample;
    const float* src[3];      // activation sources [M, 32*seg_kb[i]] row-major
    const float* src_min;     // per-channel minima paired with src[0] (minmax prologue)
    int seg_kb[3];            // k-blocks contributed by each activation source
    int stages;               // depth of the shared-memory ring (1..4)
    int w_resident;           // 1: all weight boxes are loaded once per CTA and stay in shared memory
    int settled;              // 1: weights / biases may be read before griddepcontrol.wait
    int dbg;                  // 1: CTA 0 records a globaltimer timeline into g_tc_clock
    int gn_kb;                // k-blocks (from the start: source 0) that go through the GroupNorm prologue
    int out_ld;               // row stride of `out` in floats (cout, or cout + 3 with a tail)
    const float* tail;        // [M,3] copied into output columns cout..cout+2, or nullptr
    const float *w3, *b3, *coords1, *coords2;   // FLOW epilogue
    float *coords2_out, *flow_out;
};

__device__ __forceinline__ unsigned tsu32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void tmbar_init(void* bar, unsigned count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(tsu32(bar)), "r"(count));
}
__device__ __forceinline__ void tmbar_expect_tx(void* bar, unsigned bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(tsu32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tmbar_arrive(void* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(tsu32(bar)) : "memory");
}
__device__ __forceinline__ void tmbar_wait(void* bar, unsigned parity) {
    asm volatile(
        "{\n\t.reg .pred P1;\n\t"
        "WAIT_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n\t"
        "@P1 bra DONE_%=;\n\t"
        "bra WAIT_%=;\n\t"
        "DONE_%=:\n\t}" ::"r"(tsu32(bar)),
        "r"(parity)
        : "memory");
}
__device__ __forceinline__ void ttma_load_2d(void* dst, const CUtensorMap* map, void* bar, int c0, int c1) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(tsu32(dst)),
                 "l"(map), "r"(tsu32(bar)), "r"(c0), "r"(c1)
                 : "memory");
}
// round-to-nearest (ties away from zero) to the 10-bit TF32 mantissa with two full-rate integer ops; identical to
// cvt.rna.tf32.f32 for finite values (the conversion instruction runs at a fraction of the ALU rate)
__device__ __forceinline__ float tf32_rna(float x) {
    return __uint_as_float((__float_as_uint(x) + 0x1000u) & 0xFFFFE000u);
}
// row `arow` of the shared accumulator tile, W consecutive columns, as raw bits (thread = row)
template <int W>
__device__ __forceinline__ void acc_ld(const float* arow, unsigned (&v)[W]) {
#pragma unroll
    for (int q = 0; q < W / 4; ++q) {
        const uint4 u = *reinterpret_cast<const uint4*>(arow + 4 * q);
        v[4 * q + 0] = u.x; v[4 * q + 1] = u.y; v[4 * q + 2] = u.z; v[4 * q + 3] = u.w;
    }
}
// thread-per-row values of a [32 rows x 16 columns] block -> shared-memory transpose -> stores of 8 rows x 64 B per instruction
// (thread-per-row stores would scatter 32 half-filled sectors per instruction).  stg: this warp's [32][20] staging tile.
constexpr int kTcPitch16 = 20;
__device__ __forceinline__ void stage_store16(float* __restrict__ stg, int lane, const float (&y)[16], float* __restrict__ gbase, int ld) {
    __syncwarp();
#pragma unroll
    for (int q = 0; q < 4; ++q) *reinterpret_cast<float4*>(stg + lane * kTcPitch16 + q * 4) = make_float4(y[q * 4], y[q * 4 + 1], y[q * 4 + 2], y[q * 4 + 3]);
    __syncwarp();
    const int rsub = lane >> 2, cq = lane & 3;
    float4 o[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) o[j] = *reinterpret_cast<const float4*>(stg + (j * 8 + rsub) * kTcPitch16 + cq * 4);
#pragma unroll
    for (int j = 0; j < 4; ++j) *reinterpret_cast<float4*>(gbase + (size_t)(j * 8 + rsub) * ld + cq * 4) = o[j];
}
// the inverse: a [32 rows x 16 columns] block of a row-major global tensor, loaded as 8 rows x 64 B per instruction and handed
// to the thread that owns each row (thread-per-row loads would touch 32 sectors per instruction)
// COHERENT: the operand is written by the previous launch, which may still run when this one starts (programmatic dependent
// launch), so it is not read-only over this kernel's lifetime: ld.global.cg (L2) instead of the non-coherent path.
template <bool COHERENT = false>
__device__ __forceinline__ void stage_load16(float* __restrict__ stg, int lane, const float* gbase, int ld, float (&x)[16]) {
    const int rsub = lane >> 2, cq = lane & 3;
    float4 o[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const float4* src = reinterpret_cast<const float4*>(gbase + (size_t)(j * 8 + rsub) * ld + cq * 4);
        o[j] = COHERENT ? __ldcg(src) : __ldg(src);
    }
    __syncwarp();
#pragma unroll
    for (int j = 0; j < 4; ++j) *reinterpret_cast<float4*>(stg + (j * 8 + rsub) * kTcPitch16 + cq * 4) = o[j];
    __syncwarp();
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        const float4 v = *reinterpret_cast<const float4*>(stg + lane * kTcPitch16 + q * 4);
        x[q * 4 + 0] = v.x; x[q * 4 + 1] = v.y; x[q * 4 + 2] = v.z; x[q * 4 + 3] = v.w;
    }
}
__device__ __forceinline__ float tsigmoid(float x) { return 1.f / (1.f + expf(-x)); }
// ConvGRU state update h' = (1 - z) h + z tanh(q) (model/update.py:37-39); one definition for every kernel that applies it, so
// that the multiply-add contraction is the same everywhere
__device__ __forceinline__ float tgru_blend(float z, float h, float q_pre) { return (1.f - z) * h + z * tanhf(q_pre); }

// epilogue of the accumulator tile s_acc [128 rows][pitch]: thread = point (row quad * 32 + lane)
// DET: the tile's (sum, sum^2) per group -- fixed-order sums over its 128 rows -- enter p.out_stats, which then points at the
// [B,16] fixed-point workspace (fixed_point.cuh), as exact additions
template <bool DET>
__device__ __forceinline__ void tc_epilogue(const TcParams& p, float* __restrict__ s_acc, int pitch, int quad, int half, int lane, int row0,
                                            int sample, const float* __restrict__ s_bias, float* __restrict__ s_stage, float* __restrict__ s_part) {
    const int row = row0 + quad * 32 + lane;
    const int gsz = p.cout / PVRAFT_GN_GROUPS;
    const float* arow = s_acc + (size_t)(quad * 32 + lane) * pitch;
    if (p.epi == TC_EPI_PLAIN) {
        // Every tile is full (M is a multiple of 128).  This code runs on one warp per scheduler, so it is written for
        // latency: no per-element branches, addresses hoisted, loads batched ahead of their consumers.
        const bool vec = (p.out_ld & 3) == 0;
        const ActCoef oact = act_coef(p.out_act, 0.f);
        const int rsub = lane >> 3, cq = lane & 7;
        float* obase = p.out + (size_t)(row0 + quad * 32 + rsub) * p.out_ld + cq * 4;
        const size_t ostep = (size_t)4 * p.out_ld;
        const bool want_stats = p.out_stats != nullptr;
        for (int c0 = half * 32; c0 < p.N; c0 += 64) {
            unsigned v[32];
            acc_ld(arow + c0, v);
            float* stg = s_acc + (size_t)(quad * 32) * pitch + c0;   // this warp's [32 rows][32 columns]: staged in place
            float y[32];
#pragma unroll
            for (int q = 0; q < 8; ++q) {
                const float4 bv = *reinterpret_cast<const float4*>(s_bias + c0 + q * 4);
                y[q * 4 + 0] = apply_act(__uint_as_float(v[q * 4 + 0]) + bv.x, oact);
                y[q * 4 + 1] = apply_act(__uint_as_float(v[q * 4 + 1]) + bv.y, oact);
                y[q * 4 + 2] = apply_act(__uint_as_float(v[q * 4 + 2]) + bv.z, oact);
                y[q * 4 + 3] = apply_act(__uint_as_float(v[q * 4 + 3]) + bv.w, oact);
            }
            if (p.residual != nullptr) {   // (rare: FlotRefine.fc) thread-per-row loads, before the statistics
#pragma unroll
                for (int i = 0; i < 32; ++i)
                    if (c0 + i < p.cout) y[i] += __ldg(p.residual + (size_t)row * p.cout + c0 + i);
            }
            if (p.tail != nullptr && c0 + 32 == p.out_ld) {   // last three columns of the row carry the tail (cat([out, flow]))
                const float* tp = p.tail + (size_t)row * 3;
                y[29] = __ldg(tp); y[30] = __ldg(tp + 1); y[31] = __ldg(tp + 2);
            }
            if (vec) {
                // transpose through shared memory so that a store instruction writes 4 rows x 128 contiguous bytes
                // (thread-per-row stores would scatter 32 half-filled sectors per instruction)
                __syncwarp();
#pragma unroll
                for (int q = 0; q < 8; ++q)
                    *reinterpret_cast<float4*>(stg + lane * pitch + q * 4) = make_float4(y[q * 4], y[q * 4 + 1], y[q * 4 + 2], y[q * 4 + 3]);
                __syncwarp();
                float4 t[8];
#pragma unroll
                for (int i = 0; i < 8; ++i) t[i] = *reinterpret_cast<const float4*>(stg + (i * 4 + rsub) * pitch + cq * 4);
                if (c0 + cq * 4 < p.out_ld) {
#pragma unroll
                    for (int i = 0; i < 8; ++i) *reinterpret_cast<float4*>(obase + i * ostep + c0) = t[i];
                }
                if (want_stats) {
                    // lane = column: (sum, sum^2) of this warp's 32 rows, read down the staged tile (conflict-free)
                    float s1 = 0.f, s2 = 0.f;
#pragma unroll
                    for (int r = 0; r < 32; ++r) {
                        const float a = stg[r * pitch + lane];
                        s1 += a;
                        s2 = fmaf(a, a, s2);
                    }
                    *reinterpret_cast<float2*>(s_part + (size_t)(quad * 128 + c0 + lane) * 2) = make_float2(s1, s2);
                }
            } else {
                float* o = p.out + (size_t)row * p.out_ld + c0;
#pragma unroll
                for (int i = 0; i < 32; ++i) {
                    if (c0 + i < p.out_ld) o[i] = y[i];
                }
            }
        }
        if (want_stats) {
            // combine the 4 epilogue warps and the columns of each GroupNorm group: thread t owns column t
            asm volatile("bar.sync 3, 256;" ::: "memory");
            const int t = (half * 4 + quad) * 32 + lane;   // 0..255; threads 0..N-1 own one column each
            double a1 = 0.0, a2 = 0.0;
            if (t < p.N) {
#pragma unroll
                for (int w = 0; w < 4; ++w) {
                    const float2 pr = *reinterpret_cast<const float2*>(s_part + (size_t)(w * 128 + t) * 2);
                    a1 += (double)pr.x;
                    a2 += (double)pr.y;
                }
            }
            if ((gsz & (gsz - 1)) == 0 && gsz <= 32) {   // groups are aligned runs of gsz lanes
                for (int o = gsz >> 1; o > 0; o >>= 1) {
                    a1 += __shfl_xor_sync(kFull, a1, o);
                    a2 += __shfl_xor_sync(kFull, a2, o);
                }
                if ((t & (gsz - 1)) == 0 && t < p.cout) {
                    if constexpr (DET) {
                        unsigned long long* fx = reinterpret_cast<unsigned long long*>(p.out_stats) + ((size_t)sample * 16 + (t / gsz) * 2) * kFxWords;
                        fx_atomic(fx, a1);
                        fx_atomic(fx + kFxWords, a2);
                    } else {
                    atomicAdd(p.out_stats + (size_t)sample * 16 + (t / gsz) * 2 + 0, a1);
                    atomicAdd(p.out_stats + (size_t)sample * 16 + (t / gsz) * 2 + 1, a2);
                    }
                }
            } else if (DET && t < p.cout) {
                unsigned long long* fx = reinterpret_cast<unsigned long long*>(p.out_stats) + ((size_t)sample * 16 + (t / gsz) * 2) * kFxWords;
                fx_atomic(fx, a1);
                fx_atomic(fx + kFxWords, a2);
            } else if (t < p.cout) {
                atomicAdd(p.out_stats + (size_t)sample * 16 + (t / gsz) * 2 + 0, a1);
                atomicAdd(p.out_stats + (size_t)sample * 16 + (t / gsz) * 2 + 1, a2);
            }
            asm volatile("bar.sync 3, 256;" ::: "memory");
        }
    } else if (p.epi == TC_EPI_GRU_ZR) {
        // accumulator columns 0..63 = z pre-activation, 64..127 = r pre-activation (model/update.py:34-35)
        float* stg = s_stage + (size_t)(half * 4 + quad) * 32 * kTcPitch16;
        for (int c = half * 32; c < half * 32 + 32; c += 16) {
            unsigned vz[16], vr[16];
            acc_ld(arow + c, vz);
            acc_ld(arow + 64 + c, vr);
            float z[16], rh[16], hh[16];
            stage_load16(stg, lane, p.h + (size_t)(row0 + quad * 32) * 64 + c, 64, hh);
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const float4 hv = make_float4(hh[q * 4], hh[q * 4 + 1], hh[q * 4 + 2], hh[q * 4 + 3]);
                float4 bz = *reinterpret_cast<const float4*>(s_bias + c + q * 4);
                float4 br = *reinterpret_cast<const float4*>(s_bias + p.N + c + q * 4);
                if (p.residual != nullptr) {   // per-point pre-activation term [M,128] = [z | r] (the constant context part)
                    const float4 az = __ldg(reinterpret_cast<const float4*>(p.residual + (size_t)row * 128 + c + q * 4));
                    const float4 ar = __ldg(reinterpret_cast<const float4*>(p.residual + (size_t)row * 128 + 64 + c + q * 4));
                    bz.x += az.x; bz.y += az.y; bz.z += az.z; bz.w += az.w;
                    br.x += ar.x; br.y += ar.y; br.z += ar.z; br.w += ar.w;
                }
                z[q * 4 + 0] = tsigmoid(__uint_as_float(vz[q * 4 + 0]) + bz.x); z[q * 4 + 1] = tsigmoid(__uint_as_float(vz[q * 4 + 1]) + bz.y);
                z[q * 4 + 2] = tsigmoid(__uint_as_float(vz[q * 4 + 2]) + bz.z); z[q * 4 + 3] = tsigmoid(__uint_as_float(vz[q * 4 + 3]) + bz.w);
                rh[q * 4 + 0] = tsigmoid(__uint_as_float(vr[q * 4 + 0]) + br.x) * hv.x; rh[q * 4 + 1] = tsigmoid(__uint_as_float(vr[q * 4 + 1]) + br.y) * hv.y;
                rh[q * 4 + 2] = tsigmoid(__uint_as_float(vr[q * 4 + 2]) + br.z) * hv.z; rh[q * 4 + 3] = tsigmoid(__uint_as_float(vr[q * 4 + 3]) + br.w) * hv.w;
            }
            stage_store16(stg, lane, z, p.out + (size_t)(row0 + quad * 32) * 64 + c, 64);
            stage_store16(stg, lane, rh, p.out2 + (size_t)(row0 + quad * 32) * 64 + c, 64);
        }
    } else if (p.epi == TC_EPI_FLOW) {
        // y = relu(acc + b) (flow_head.out_conv.0/1); delta = w3 . y + b3 (out_conv.2); RAFT update of the coordinates.
        // The two warps of a lane quadrant hold 32 of the 64 columns each: half 1 parks its partial dot products.
        const float* s_w3 = s_part + 512;   // [3][64], staged at kernel start; s_part[0..511] = [128 rows][4] exchange
        unsigned v[32];
        const int c0 = half * 32;
        acc_ld(arow + c0, v);
        float d0 = 0.f, d1 = 0.f, d2 = 0.f;
#pragma unroll
        for (int q = 0; q < 8; ++q) {
            const float4 bv = *reinterpret_cast<const float4*>(s_bias + c0 + q * 4);
            const float4 wa = *reinterpret_cast<const float4*>(s_w3 + 0 * 64 + c0 + q * 4);
            const float4 wb = *reinterpret_cast<const float4*>(s_w3 + 1 * 64 + c0 + q * 4);
            const float4 wc = *reinterpret_cast<const float4*>(s_w3 + 2 * 64 + c0 + q * 4);
            const float y0 = fmaxf(__uint_as_float(v[q * 4 + 0]) + bv.x, 0.f), y1 = fmaxf(__uint_as_float(v[q * 4 + 1]) + bv.y, 0.f);
            const float y2 = fmaxf(__uint_as_float(v[q * 4 + 2]) + bv.z, 0.f), y3 = fmaxf(__uint_as_float(v[q * 4 + 3]) + bv.w, 0.f);
            d0 = fmaf(wa.w, y3, fmaf(wa.z, y2, fmaf(wa.y, y1, fmaf(wa.x, y0, d0))));
            d1 = fmaf(wb.w, y3, fmaf(wb.z, y2, fmaf(wb.y, y1, fmaf(wb.x, y0, d1))));
            d2 = fmaf(wc.w, y3, fmaf(wc.z, y2, fmaf(wc.y, y1, fmaf(wc.x, y0, d2))));
        }
        float* xch = s_part + (size_t)(quad * 32 + lane) * 4;
        if (half == 1) *reinterpret_cast<float4*>(xch) = make_float4(d0, d1, d2, 0.f);
        asm volatile("bar.sync 3, 256;" ::: "memory");
        if (half == 0) {
            const float4 o = *reinterpret_cast<const float4*>(xch);
            const float dd[3] = {(d0 + o.x) + s_bias[p.N + 0], (d1 + o.y) + s_bias[p.N + 1], (d2 + o.z) + s_bias[p.N + 2]};
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                const size_t g = (size_t)row * 3 + k;
                p.out[g] = dd[k];
                if (p.coords2_out != nullptr) {
                    const float c2 = p.coords2[g] + dd[k];   // RAFTSceneFlow.py:45
                    p.coords2_out[g] = c2;
                    if (p.flow_out != nullptr) {
                        const float fl = c2 - __ldg(p.coords1 + g);   // RAFTSceneFlow.py:46
                        p.flow_out[g] = fl;
                    }
                }
            }
        }
        asm volatile("bar.sync 3, 256;" ::: "memory");   // the exchange buffer is free for the next tile
    } else {
        // q = tanh(acc + b); h' = (1 - z) h + z q   (model/update.py:37-39)
        float* stg = s_stage + (size_t)(half * 4 + quad) * 32 * kTcPitch16;
        for (int c = half * 32; c < half * 32 + 32; c += 16) {
            unsigned vq[16];
            acc_ld(arow + c, vq);
            float o[16], hh[16], zz[16];
            stage_load16(stg, lane, p.h + (size_t)(row0 + quad * 32) * 64 + c, 64, hh);
            stage_load16<true>(stg, lane, p.z + (size_t)(row0 + quad * 32) * 64 + c, 64, zz);   // z comes from the launch before
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const float4 hv = make_float4(hh[q * 4], hh[q * 4 + 1], hh[q * 4 + 2], hh[q * 4 + 3]);
                const float4 zv = make_float4(zz[q * 4], zz[q * 4 + 1], zz[q * 4 + 2], zz[q * 4 + 3]);
                float4 bq = *reinterpret_cast<const float4*>(s_bias + c + q * 4);
                if (p.residual != nullptr) {   // per-point pre-activation term [M,64]
                    const float4 aq = __ldg(reinterpret_cast<const float4*>(p.residual + (size_t)row * 64 + c + q * 4));
                    bq.x += aq.x; bq.y += aq.y; bq.z += aq.z; bq.w += aq.w;
                }
                o[q * 4 + 0] = tgru_blend(zv.x, hv.x, __uint_as_float(vq[q * 4 + 0]) + bq.x);
                o[q * 4 + 1] = tgru_blend(zv.y, hv.y, __uint_as_float(vq[q * 4 + 1]) + bq.y);
                o[q * 4 + 2] = tgru_blend(zv.z, hv.z, __uint_as_float(vq[q * 4 + 2]) + bq.z);
                o[q * 4 + 3] = tgru_blend(zv.w, hv.w, __uint_as_float(vq[q * 4 + 3]) + bq.w);
            }
            stage_store16(stg, lane, o, p.out + (size_t)(row0 + quad * 32) * 64 + c, 64);
        }
    }
}

// A CTA walks tiles blockIdx.x, +gridDim.x, ...; the operand ring runs across tile boundaries.

// Position of one pipeline role in the (tile, k-block) walk and in the operand ring; advanced without divisions (a
// runtime integer division is a ~100-cycle dependent chain, paid per step by warps that have nothing to hide it behind)
struct TcCursor {
    int ti = 0, kb = 0, s = 0;
    unsigned phase = 0;
    __device__ __forceinline__ void next(int num_kb, int S) {
        if (++kb == num_kb) { kb = 0; ++ti; }
        if (++s == S) { s = 0; phase ^= 1u; }
    }
};

// one k-block (32 channels) of a warpgroup's 64 x N accumulator: 3xTF32, four K = 8 slices
template <int N>
__device__ __forceinline__ void tc_mma_kblock(float (&acc)[64], unsigned long long a_hi, unsigned long long a_lo, unsigned long long b_hi,
                                              unsigned long long b_lo, int kb) {
#pragma unroll
    for (int k = 0; k < kTcKB / 8; ++k) {
        wgmma_tf32<N>(acc, wgmma_desc_k(a_hi, k), wgmma_desc_k(b_hi, k), (kb | k) != 0);
        wgmma_tf32<N>(acc, wgmma_desc_k(a_lo, k), wgmma_desc_k(b_hi, k), 1);
        wgmma_tf32<N>(acc, wgmma_desc_k(a_hi, k), wgmma_desc_k(b_lo, k), 1);
    }
}
// prologue of four consecutive channels: the folded GroupNorm affine, then the activation
__device__ __forceinline__ float4 tc_gn_act4(float4 x, const float4& sc, const float4& sh, const ActCoef& act) {
    x.x = apply_act(fmaf(x.x, sc.x, sh.x), act);
    x.y = apply_act(fmaf(x.y, sc.y, sh.y), act);
    x.z = apply_act(fmaf(x.z, sc.z, sh.z), act);
    x.w = apply_act(fmaf(x.w, sc.w, sh.w), act);
    return x;
}
// 3xTF32 operand split of one 16-byte chunk at byte offset `off` of an operand stage: hi = tf32(x) at stage + off, lo =
// tf32(x - hi) at the same offset of the lo box behind it
__device__ __forceinline__ void tc_split_store(unsigned char* stage, int off, const float4& x) {
    float4 hi, lo;
    hi.x = tf32_rna(x.x); hi.y = tf32_rna(x.y); hi.z = tf32_rna(x.z); hi.w = tf32_rna(x.w);
    lo.x = tf32_rna(x.x - hi.x); lo.y = tf32_rna(x.y - hi.y); lo.z = tf32_rna(x.z - hi.z); lo.w = tf32_rna(x.w - hi.w);
    *reinterpret_cast<float4*>(stage + off) = hi;
    *reinterpret_cast<float4*>(stage + kTcABytes + off) = lo;
}
// row pitch (floats) of the shared accumulator tile: whole 32-column epilogue chunks plus 4, so that thread-per-row 16-byte
// accesses of 8 consecutive rows fall into distinct bank groups
__host__ __device__ __forceinline__ int tc_acc_pitch(int n) { return ((n + 31) & ~31) + 4; }

// NT = p.N (the padded cout): the wgmma shape is part of the instruction
template <int NT, bool DET>
__global__ void __launch_bounds__(kTcThreads, 1)
k_tc_linear(const __grid_constant__ CUtensorMap map_w_hi, const __grid_constant__ CUtensorMap map_w_lo,
            const __grid_constant__ CUtensorMap map_a0, const __grid_constant__ CUtensorMap map_a1,
            const __grid_constant__ CUtensorMap map_a2, const __grid_constant__ CUtensorMap map_min, const TcParams p) {
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    // 1024-byte alignment by pointer arithmetic on the shared array: an integer round trip would lose the address space
    // and turn every shared-memory access below into a generic LD/ST
    unsigned char* tiles = smem_raw + ((1024u - ((unsigned)__cvta_generic_to_shared(smem_raw) & 1023u)) & 1023u);
    // stage layout: [A hi 16K][A lo 16K][W hi N*128][W lo N*128, only when the weights are streamed];
    // resident weights live behind the ring as num_kb x [W hi][W lo]
    const int w_bytes = p.N * kTcKB * 4;
    const int w_off = 2 * kTcABytes;
    const int stage_bytes = w_off + (p.w_resident ? 0 : 2 * w_bytes);
    const int S = p.stages;
    const int num_kb = p.K / kTcKB;
    const int acc_pitch = tc_acc_pitch(NT);
    unsigned char* w_res = tiles + (size_t)S * stage_bytes;
    float* s_scale = reinterpret_cast<float*>(w_res + (p.w_resident ? (size_t)num_kb * 2 * w_bytes : 0));   // [2 groups][scale K | shift K]
    float* s_bias = s_scale + 4 * p.K;                                            // [2 * N]
    float* s_acc = s_bias + 2 * p.N;                                              // [128 rows][acc_pitch] accumulator tile
    float* s_estage = s_acc + (size_t)kTcM * acc_pitch;                           // GRU epilogues: [8 warps][32][20] staging
    float* s_part = s_estage + (p.epi == TC_EPI_GRU_ZR || p.epi == TC_EPI_GRU_Q ? 8 * 32 * kTcPitch16 : 0);   // [4 warps][128 columns][2]
    __shared__ __align__(8) unsigned long long s_full[kTcMaxStages], s_empty[kTcMaxStages];
    __shared__ __align__(8) unsigned long long s_acc_full, s_acc_empty, s_w_full;
    const int warp = warp_id(), lane = lane_id();
    const int n_tiles = (p.M + kTcM - 1) / kTcM;
    const int my_tiles = blockIdx.x < n_tiles ? (n_tiles - 1 - blockIdx.x) / gridDim.x + 1 : 0;
    const int total_steps = my_tiles * num_kb;
#ifdef PVRAFT_TC_TIMELINE
    const bool clk = p.dbg && blockIdx.x == 0;
#endif
    TC_MARK(threadIdx.x == 0, 0);

    if (warp == kTcProducerWarp && lane == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_w_hi) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_w_lo) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_a0) : "memory");
        for (int s = 0; s < S; ++s) { tmbar_init(&s_full[s], 1); tmbar_init(&s_empty[s], 8); }   // 8 MMA warps release a stage
        tmbar_init(&s_acc_full, 8);     // 8 MMA warps deposit the accumulator tile
        tmbar_init(&s_acc_empty, 8);    // 8 epilogue warps have consumed it
        tmbar_init(&s_w_full, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    // Programmatic dependent launch: everything above (shared-memory carve-up, barrier init, descriptor prefetch) may
    // overlap the tail of the previous kernel on this stream.  The layer's PARAMETERS (hi/lo weights, biases) are fetched
    // in that window too when the caller vouches that they are settled (p.settled: last written several launches ago --
    // the steady state of a forward, whose weights are split once): the SMs that finished the previous kernel early then
    // hold their weights when the dependency resolves.  Every read of an ACTIVATION is below the wait.
    auto load_weights = [&]() {   // the whole weight matrix (hi and lo) once per CTA
        tmbar_expect_tx(&s_w_full, (unsigned)(num_kb * 2 * w_bytes));
        for (int kb = 0; kb < num_kb; ++kb) {
            ttma_load_2d(w_res + (size_t)kb * 2 * w_bytes, &map_w_hi, &s_w_full, kb * kTcKB, 0);
            ttma_load_2d(w_res + (size_t)kb * 2 * w_bytes + w_bytes, &map_w_lo, &s_w_full, kb * kTcKB, 0);
        }
    };
    auto load_bias = [&]() {   // by the epilogue threads 0..255
        for (int c = threadIdx.x; c < p.N; c += kTcEpiThreads) {
            s_bias[c] = (p.bias != nullptr && c < p.cout) ? __ldg(p.bias + c) : 0.f;
            s_bias[p.N + c] = (p.bias2 != nullptr && c < p.cout) ? __ldg(p.bias2 + c) : 0.f;
        }
        if (p.epi == TC_EPI_FLOW) {   // out_conv.2: weights behind the exchange buffer, bias in the bias2 slots
            for (int i = threadIdx.x; i < 192; i += kTcEpiThreads) s_part[512 + i] = __ldg(p.w3 + i);
            if (threadIdx.x < 3) s_bias[p.N + threadIdx.x] = __ldg(p.b3 + threadIdx.x);
        }
    };
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    __syncthreads();   // barrier init visible to every role
    if (p.settled) {
        if (warp == kTcProducerWarp && lane == 0 && p.w_resident) load_weights();
        if (warp < 8) load_bias();
    }
    asm volatile("griddepcontrol.wait;" ::: "memory");
    if (!p.settled && warp < 8) load_bias();
    __syncthreads();

    if (warp == kTcProducerWarp) {
        // ===== TMA producer: raw activation boxes (and the weights) =====
        if (lane == 0) {
            if (p.w_resident && !p.settled) load_weights();
            const unsigned tx = (unsigned)(kTcABytes * (p.minmax ? 2 : 1) + (p.w_resident ? 0 : 2 * w_bytes));
            TcCursor cw;
            for (int step = 0; step < total_steps; ++step, cw.next(num_kb, S)) {
                const int s = cw.s, kb = cw.kb;
                const int row0 = (blockIdx.x + cw.ti * gridDim.x) * kTcM;
                tmbar_wait(&s_empty[s], cw.phase ^ 1u);   // the MMAs that read this stage last time have retired
                unsigned char* st = tiles + (size_t)s * stage_bytes;
                tmbar_expect_tx(&s_full[s], tx);
                // raw fp32 rows of the source this k-block belongs to land where the hi operand will be (the transform works
                // in place); the min array of a (max, min) pair lands in the lo half
                if (kb < p.seg_kb[0]) ttma_load_2d(st, &map_a0, &s_full[s], kb * kTcKB, row0);
                else if (kb < p.seg_kb[0] + p.seg_kb[1]) ttma_load_2d(st, &map_a1, &s_full[s], (kb - p.seg_kb[0]) * kTcKB, row0);
                else ttma_load_2d(st, &map_a2, &s_full[s], (kb - p.seg_kb[0] - p.seg_kb[1]) * kTcKB, row0);
                if (p.minmax) ttma_load_2d(st + kTcABytes, &map_min, &s_full[s], kb * kTcKB, row0);
                if (!p.w_resident) {
                    ttma_load_2d(st + w_off, &map_w_hi, &s_full[s], kb * kTcKB, 0);
                    ttma_load_2d(st + w_off + w_bytes, &map_w_lo, &s_full[s], kb * kTcKB, 0);
                }
            }
        }
    } else if (warp >= 8) {
        // ===== transform + MMA: warpgroup grp owns rows [64 grp, 64 grp + 64) of every tile =====
        // raw fp32 box -> GroupNorm affine + activation -> tf32 hi/lo operand tiles, in place; then the wgmma of this k-block
        // run asynchronously while the next k-block is transformed.  Each group keeps its own copy of the per-sample
        // GroupNorm table.
        const int grp = (warp >> 2) - 2;
        const int t = threadIdx.x & 127;   // chunk c = t + 128*i, i < 4, of the group's 512 16-byte chunks of a k-block
        const int a_off = grp * 64 * 128;  // byte offset of the group's rows in an activation box (1024-aligned)
        float* g_scale = s_scale + grp * 2 * p.K;
        float* g_shift = g_scale + p.K;
        const ActCoef iact = act_coef(p.in_act, p.in_slope);
        TcCursor cp;
        const int tiles_per_sample = p.pts_per_sample / kTcM;
        int table_first = -1, table_end = -1;   // tile range [first, end) of the sample whose table this group holds
        if (p.w_resident) tmbar_wait(&s_w_full, 0u);
        float acc[64];
        int prev_s = -1;
        for (int ti = 0; ti < my_tiles; ++ti) {
          for (int kb = 0; kb < num_kb; ++kb) {
            const int s = cp.s;
            auto gn_table = [&]() {
                const int tile = blockIdx.x + cp.ti * gridDim.x;
                if (tile < table_first || tile >= table_end) {   // folded GroupNorm affine of every input channel of this sample
                    const int sample = tile / tiles_per_sample;
                    table_first = sample * tiles_per_sample;
                    table_end = table_first + tiles_per_sample;
                    asm volatile("bar.sync %0, 128;" ::"r"(1 + grp) : "memory");   // the group is done with the previous table
                    const int gn_k = p.gn_kb * kTcKB, gsz = gn_k / PVRAFT_GN_GROUPS;
                    for (int k = t; k < gn_k; k += 128) {
                        const double* sp = p.in_stats + (size_t)sample * 16 + (k / gsz) * 2;
                        const double st[2] = {__ldcg(sp), __ldcg(sp + 1)};   // (written by the launch before: L2, not the nc path)
                        const GnAffine af = gn_affine(st, p.in_count, __ldg(p.in_gamma + k), __ldg(p.in_beta + k));
                        g_scale[k] = af.scale;
                        g_shift[k] = af.shift;
                    }
                    asm volatile("bar.sync %0, 128;" ::"r"(1 + grp) : "memory");
                }
            };
            // the sums are complete once the previous launch is: the table is built before the box wait, under the TMA latency
            if (p.in_stats != nullptr) gn_table();
            tmbar_wait(&s_full[s], cp.phase);   // the raw box(es) of this k-block have landed
            unsigned char* st = tiles + (size_t)s * stage_bytes;
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int c = t + i * 128, r = grp * 64 + (c >> 3), lc = c & 7;
                // K-major SWIZZLE_128B: 16-byte chunk lc of row r lives at chunk (lc ^ (r & 7)) of the row's 128 bytes
                const int off = r * 128 + ((lc ^ (r & 7)) << 4);
                float4 x = *reinterpret_cast<const float4*>(st + off);
                if (kb < p.gn_kb) {
                    const int k = kb * kTcKB + lc * 4;
                    const float4 sc = *reinterpret_cast<const float4*>(g_scale + k);
                    const float4 sh = *reinterpret_cast<const float4*>(g_shift + k);
                    if (p.minmax) {
                        const float4 mn = *reinterpret_cast<const float4*>(st + kTcABytes + off);
                        x.x = sc.x < 0.f ? mn.x : x.x; x.y = sc.y < 0.f ? mn.y : x.y;
                        x.z = sc.z < 0.f ? mn.z : x.z; x.w = sc.w < 0.f ? mn.w : x.w;
                    }
                    x.x = apply_act(fmaf(x.x, sc.x, sh.x), iact);
                    x.y = apply_act(fmaf(x.y, sc.y, sh.y), iact);
                    x.z = apply_act(fmaf(x.z, sc.z, sh.z), iact);
                    x.w = apply_act(fmaf(x.w, sc.w, sh.w), iact);
                }
                float4 hi, lo;
                hi.x = tf32_rna(x.x); hi.y = tf32_rna(x.y); hi.z = tf32_rna(x.z); hi.w = tf32_rna(x.w);
                lo.x = tf32_rna(x.x - hi.x); lo.y = tf32_rna(x.y - hi.y); lo.z = tf32_rna(x.z - hi.z); lo.w = tf32_rna(x.w - hi.w);
                *reinterpret_cast<float4*>(st + off) = hi;   // in place: raw -> hi; the lo half of the stage held the min array
                *reinterpret_cast<float4*>(st + kTcABytes + off) = lo;
            }
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy writes -> visible to wgmma (async proxy)
            asm volatile("bar.sync %0, 128;" ::"r"(1 + grp) : "memory");   // the group's 64 rows are in place
            TC_MARK(t == 0 && ti * num_kb + kb < 8, 8 + ti * num_kb + kb);
            const unsigned char* wb = p.w_resident ? w_res + (size_t)kb * 2 * w_bytes : st + w_off;
            wgmma_fence_regs(acc);
            wgmma_fence();
            tc_mma_kblock<NT>(acc, wgmma_desc(st + a_off), wgmma_desc(st + kTcABytes + a_off), wgmma_desc(wb), wgmma_desc(wb + w_bytes), kb);
            wgmma_commit();
            wgmma_wait<1>();   // the previous k-block's MMAs have retired: its stage may be refilled
            if (prev_s >= 0 && lane == 0) tmbar_arrive(&s_empty[prev_s]);
            prev_s = s;
            cp.next(num_kb, S);
          }
          wgmma_wait<0>();
          wgmma_fence_regs(acc);
          if (lane == 0) tmbar_arrive(&s_empty[prev_s]);
          prev_s = -1;
          TC_MARK(t == 0 && ti < 8, 16 + ti);
          tmbar_wait(&s_acc_empty, ((unsigned)ti & 1u) ^ 1u);   // the epilogue has consumed the previous tile
          // accumulator fragment -> rows 64 grp + 16 (warp % 4) + lane / 4 (+8), columns 8 j + 2 (lane % 4) (+1)
          float* a0 = s_acc + (size_t)(grp * 64 + (warp & 3) * 16 + (lane >> 2)) * acc_pitch + 2 * (lane & 3);
#pragma unroll
          for (int j = 0; j < NT / 8; ++j) {
              *reinterpret_cast<float2*>(a0 + 8 * j) = make_float2(acc[4 * j + 0], acc[4 * j + 1]);
              *reinterpret_cast<float2*>(a0 + (size_t)8 * acc_pitch + 8 * j) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
          }
          __syncwarp();
          if (lane == 0) tmbar_arrive(&s_acc_full);
        }
    } else {
        // ===== epilogue: accumulator tile -> registers -> global, one tile behind the MMA =====
        const int quad = warp & 3;   // rows 32 quad .. +31 of the tile
        const int half = warp >> 2;  // two warps per quadrant: 32-column chunks c0 = 32*half, +64, ...
        for (int ti = 0; ti < my_tiles; ++ti) {
            const int row0 = (blockIdx.x + ti * gridDim.x) * kTcM;
            tmbar_wait(&s_acc_full, (unsigned)ti & 1u);
            TC_MARK(threadIdx.x == 0 && ti < 4, 24 + ti);
            const int sample = row0 / p.pts_per_sample;
            tc_epilogue<DET>(p, s_acc, acc_pitch, quad, half, lane, row0, sample, s_bias, s_estage, s_part);
            __syncwarp();
            if (lane == 0) tmbar_arrive(&s_acc_empty);   // one arrival per epilogue warp
            TC_MARK(threadIdx.x == 0 && ti < 4, 28 + ti);
        }
    }
    TC_MARK(threadIdx.x == 256, 1);
}

// ===== the update chain: MotionEncoder, ConvGRU and the flow-head fc1 pre-transform of one RAFT iteration in one launch =====
//   L0 cc     = relu(W_cc [lrelu(GN(y1)) | kfeat] + b_cc)        K 192, N 64   (corr.py fold_corr_motion)
//   L1 motion = [relu(W_m [cc | cflow] + b_m) (61) | flow (3)]   K 128, N 64
//   L2 [z|r]  = sigmoid(W_zr [net | inp | motion] + b_zr)        K 192, N 128;  z stays in registers, r*net -> X
//   L3 net'   = (1 - z) net + z tanh(W_q [r*net | inp | motion] + b_q)   K 192, N 64  -> HBM and X
//   L4 P      = W_fc1[:, :64] net'                               K 64,  N 64   -> HBM
// Each layer runs exactly the k-block sequence, transform, 3xTF32 wgmma order and epilogue formula of its k_tc_linear
// launch, so the results are the same bits.  Warp 8 streams, per k-block, the weight boxes (hi, lo) of every layer and the
// raw activation box of the k-blocks read from HBM (y1, kfeat, cflow, net, inp).  Warpgroup grp (warps 4 grp .. +3) owns
// rows 64 grp .. +63 of every tile from operand to output: it transforms its rows of a box, issues the wgmma, and at the end
// of a layer applies the epilogue to its accumulator registers, writing the activation either to HBM (net', P) or as raw
// fp32 into an on-chip [128 x 64] buffer laid out like two TMA boxes (X: cc, then r*net, then net'; Y: motion).  A k-block
// read from a buffer is split from there into the ring stage instead of in place.  Nothing crosses the two warpgroups but
// the ring, so a layer boundary costs a warpgroup only its own epilogue.
constexpr int kChThreads = 288;   // 2 transform + MMA + epilogue warpgroups | TMA producer
constexpr int kChProducerWarp = 8;
constexpr int kChStages = 2;
constexpr int kChWBytes = 128 * kTcKB * 4;                   // one weight box of the widest layer (N = 128)
constexpr int kChStageBytes = 2 * kTcABytes + 2 * kChWBytes;  // [A hi][A lo][W hi][W lo] = 64 KB
constexpr int kChBufBytes = 2 * kTcABytes;                    // [128 rows x 64 channels] as two swizzled boxes
constexpr int kChSteps = 24;                                  // k-blocks per tile over the five layers
enum ChSrc { CH_Y1 = 0, CH_KFEAT, CH_CFLOW, CH_NET, CH_INP, CH_X, CH_Y };

struct ChainParams {
    const double* y1_stats;   // [B,8,2]: GroupNorm sums of y1
    const float *gn_gamma, *gn_beta;
    double gn_count;
    float gn_slope;           // PReLU slope of the y1 prologue
    const float *flow, *net;  // [M,3], [M,64]
    const float *b_cc, *b_m, *b_z, *b_r, *b_q;
    float *net_out, *p_out;   // [M,64] each
    int M, pts_per_sample;
};
struct ChainMaps {
    CUtensorMap a[5];         // y1, kfeat, cflow, net, inp: [M, C] boxes of [128 x 32]
    CUtensorMap w_hi[5], w_lo[5];
};

// step i of a tile: layer, source, k-block within the source; a layer's k-blocks are consecutive
__device__ __forceinline__ int ch_layer(int i) { return i < 6 ? 0 : i < 10 ? 1 : i < 16 ? 2 : i < 22 ? 3 : 4; }
__device__ __forceinline__ int ch_src(int i) {
    // from step 6 on, sources come in pairs of k-blocks: X, cflow | net, inp, Y | X, inp, Y | X  (a nibble each)
    constexpr unsigned long long pairs = (unsigned long long)CH_X | (unsigned long long)CH_CFLOW << 4 | (unsigned long long)CH_NET << 8 |
                                         (unsigned long long)CH_INP << 12 | (unsigned long long)CH_Y << 16 | (unsigned long long)CH_X << 20 |
                                         (unsigned long long)CH_INP << 24 | (unsigned long long)CH_Y << 28 | (unsigned long long)CH_X << 32;
    return i < 4 ? CH_Y1 : i < 6 ? CH_KFEAT : (int)((pairs >> (4 * ((i - 6) >> 1))) & 15u);
}
__device__ __forceinline__ int ch_skb(int i) {   // y1 has four k-blocks, every other source two
    return i < 4 ? i : (i < 6 ? i - 4 : (i - 6) & 1);
}
__device__ __forceinline__ int ch_first(int layer) { return layer == 0 ? 0 : layer == 1 ? 6 : layer == 2 ? 10 : layer == 3 ? 16 : 22; }
__device__ __forceinline__ int ch_w_bytes(int layer) { return (layer == 2 ? 128 : 64) * kTcKB * 4; }

// raw fp32 value pair (columns c, c + 1; c even) of tile row r into an on-chip [128 x 64] buffer in the TMA box layout
__device__ __forceinline__ void ch_buf_store2(unsigned char* buf, int r, int c, float v0, float v1) {
    const int lc = (c & 31) >> 2;
    *reinterpret_cast<float2*>(buf + (c >> 5) * kTcABytes + r * 128 + ((lc ^ (r & 7)) << 4) + (c & 3) * 4) = make_float2(v0, v1);
}

// the MMA warpgroup's part of one tile step: wait for the stage, transform its rows of the k-block (from the stage in place,
// or from an on-chip buffer), issue the 3xTF32 wgmma and release the stage
template <int N>
__device__ __forceinline__ void ch_kblock(float (&acc)[64], int kb, int src, int skb, unsigned char* tiles, unsigned char* buf_x,
                                          unsigned char* buf_y, const float* g_scale, const float* g_shift, const ActCoef& iact,
                                          unsigned long long* s_full, unsigned long long* s_empty, TcCursor& cp, int grp, int t,
                                          int lane) {
    const int s = cp.s;
    tmbar_wait(&s_full[s], cp.phase);
    unsigned char* st = tiles + (size_t)s * kChStageBytes;
    const unsigned char* from = src == CH_X ? buf_x + skb * kTcABytes : src == CH_Y ? buf_y + skb * kTcABytes : st;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int c = t + i * 128, r = grp * 64 + (c >> 3), lc = c & 7;
        const int off = r * 128 + ((lc ^ (r & 7)) << 4);
        float4 x = *reinterpret_cast<const float4*>(from + off);
        if (src == CH_Y1) {
            const int k = skb * kTcKB + lc * 4;
            x = tc_gn_act4(x, *reinterpret_cast<const float4*>(g_scale + k), *reinterpret_cast<const float4*>(g_shift + k), iact);
        }
        tc_split_store(st, off, x);
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    asm volatile("bar.sync %0, 128;" ::"r"(1 + grp) : "memory");
    const unsigned char* wb = st + 2 * kTcABytes;
    wgmma_fence_regs(acc);
    wgmma_fence();
    tc_mma_kblock<N>(acc, wgmma_desc(st + grp * 64 * 128), wgmma_desc(st + kTcABytes + grp * 64 * 128), wgmma_desc(wb),
                     wgmma_desc(wb + N * kTcKB * 4), kb);
    wgmma_commit();
    // retire this k-block before the next transform: with two stages the refill of this one then overlaps the whole next
    // step (waiting one k-block later would start each refill only once the next box had landed, exposing every load)
    wgmma_wait<0>();
    if (lane == 0) tmbar_arrive(&s_empty[s]);
    cp.next(kChSteps, kChStages);
}
// all k-blocks of one layer (steps i0 .. i0 + nkb - 1), then the accumulator is final in registers
template <int N>
__device__ __forceinline__ void ch_layer_mma(float (&acc)[64], int i0, int nkb, unsigned char* tiles, unsigned char* buf_x,
                                             unsigned char* buf_y, const float* g_scale, const float* g_shift, const ActCoef& iact,
                                             unsigned long long* s_full, unsigned long long* s_empty, TcCursor& cp, int grp, int t,
                                             int lane) {
    for (int kb = 0; kb < nkb; ++kb)
        ch_kblock<N>(acc, kb, ch_src(i0 + kb), ch_skb(i0 + kb), tiles, buf_x, buf_y, g_scale, g_shift, iact, s_full, s_empty, cp, grp, t, lane);
    wgmma_fence_regs(acc);
}

__global__ void __launch_bounds__(kChThreads, 1)
k_update_chain(const __grid_constant__ ChainMaps maps, const ChainParams p) {
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    unsigned char* tiles = smem_raw + ((1024u - ((unsigned)__cvta_generic_to_shared(smem_raw) & 1023u)) & 1023u);
    unsigned char* buf_x = tiles + (size_t)kChStages * kChStageBytes;
    unsigned char* buf_y = buf_x + kChBufBytes;
    float* s_scale = reinterpret_cast<float*>(buf_y + kChBufBytes);   // [2 groups][scale 128 | shift 128]
    float* s_bias = s_scale + 2 * 256;                                 // cc 64 | m 64 | z 64 | r 64 | q 64
    __shared__ __align__(8) unsigned long long s_full[kChStages], s_empty[kChStages];
    const int warp = warp_id(), lane = lane_id();
    const int n_tiles = p.M / kTcM;
    const int my_tiles = blockIdx.x < n_tiles ? (n_tiles - 1 - blockIdx.x) / gridDim.x + 1 : 0;
    if (warp == kChProducerWarp && lane == 0) {
        for (int i = 0; i < 5; ++i) {
            asm volatile("prefetch.tensormap [%0];" ::"l"(&maps.a[i]) : "memory");
            asm volatile("prefetch.tensormap [%0];" ::"l"(&maps.w_hi[i]) : "memory");
            asm volatile("prefetch.tensormap [%0];" ::"l"(&maps.w_lo[i]) : "memory");
        }
        for (int s = 0; s < kChStages; ++s) { tmbar_init(&s_full[s], 1); tmbar_init(&s_empty[s], 8); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    __syncthreads();
    asm volatile("griddepcontrol.wait;" ::: "memory");   // every global read below
    if (threadIdx.x < 64) {
        const int c = threadIdx.x;
        s_bias[c] = __ldg(p.b_cc + c);
        s_bias[64 + c] = c < 61 ? __ldg(p.b_m + c) : 0.f;
        s_bias[128 + c] = __ldg(p.b_z + c);
        s_bias[192 + c] = __ldg(p.b_r + c);
        s_bias[256 + c] = __ldg(p.b_q + c);
    }
    __syncthreads();

    if (warp == kChProducerWarp) {
        if (lane == 0) {
            TcCursor cw;
            for (int step = 0; step < my_tiles * kChSteps; ++step, cw.next(kChSteps, kChStages)) {
                const int i = cw.kb, layer = ch_layer(i), src = ch_src(i);
                const int row0 = (blockIdx.x + cw.ti * gridDim.x) * kTcM;
                const int wb = ch_w_bytes(layer);
                const int lkb = i - ch_first(layer), skb = ch_skb(i);   // k-block of the layer's weights, of the source
                tmbar_wait(&s_empty[cw.s], cw.phase ^ 1u);
                unsigned char* st = tiles + (size_t)cw.s * kChStageBytes;
                tmbar_expect_tx(&s_full[cw.s], (unsigned)((src < CH_X ? kTcABytes : 0) + 2 * wb));
                if (src < CH_X) ttma_load_2d(st, &maps.a[src], &s_full[cw.s], skb * kTcKB, row0);
                ttma_load_2d(st + 2 * kTcABytes, &maps.w_hi[layer], &s_full[cw.s], lkb * kTcKB, 0);
                ttma_load_2d(st + 2 * kTcABytes + wb, &maps.w_lo[layer], &s_full[cw.s], lkb * kTcKB, 0);
            }
        }
        return;
    }

    const int grp = warp >> 2, t = threadIdx.x & 127;
    float* g_scale = s_scale + grp * 256;
    float* g_shift = g_scale + 128;
    const ActCoef iact = act_coef(PVRAFT_ACT_LRELU, p.gn_slope);
    const ActCoef relu = act_coef(PVRAFT_ACT_RELU, 0.f), none = act_coef(PVRAFT_ACT_NONE, 0.f);
    const int tiles_per_sample = p.pts_per_sample / kTcM;
    const int rq = (warp & 3) * 16 + (lane >> 2);   // accumulator rows rq, rq + 8 of the group's 64; columns 8 j + cq, + 1
    const int cq = 2 * (lane & 3);
    int table_sample = -1;
    TcCursor cp;
    float acc[64], z[32];
    for (int ti = 0; ti < my_tiles; ++ti) {
        const int tile = blockIdx.x + ti * gridDim.x;
        const int row0 = tile * kTcM;
        const int sample = tile / tiles_per_sample;
        if (sample != table_sample) {   // folded GroupNorm affine of the 128 channels of y1 for this sample
            table_sample = sample;
            asm volatile("bar.sync %0, 128;" ::"r"(1 + grp) : "memory");
            const double* sp = p.y1_stats + (size_t)sample * 16 + (t / 16) * 2;
            const double st[2] = {__ldcg(sp), __ldcg(sp + 1)};
            const GnAffine af = gn_affine(st, p.gn_count, __ldg(p.gn_gamma + t), __ldg(p.gn_beta + t));
            g_scale[t] = af.scale;
            g_shift[t] = af.shift;
            asm volatile("bar.sync %0, 128;" ::"r"(1 + grp) : "memory");
        }
        const int r_lo = grp * 64 + rq;   // tile rows of acc[4 j + 0, 1] and (+ 8) acc[4 j + 2, 3]
        // L0: cc -> X
        ch_layer_mma<64>(acc, 0, 6, tiles, buf_x, buf_y, g_scale, g_shift, iact, s_full, s_empty, cp, grp, t, lane);
#pragma unroll
        for (int j = 0; j < 8; ++j)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int c = 8 * j + cq;
                ch_buf_store2(buf_x, r_lo + 8 * h, c, apply_act(acc[4 * j + 2 * h] + s_bias[c], relu), apply_act(acc[4 * j + 2 * h + 1] + s_bias[c + 1], relu));
            }
        asm volatile("bar.sync %0, 128;" ::"r"(1 + grp) : "memory");
        // L1: motion = [relu(.) | flow] -> Y
        ch_layer_mma<64>(acc, 6, 4, tiles, buf_x, buf_y, g_scale, g_shift, iact, s_full, s_empty, cp, grp, t, lane);
#pragma unroll
        for (int j = 0; j < 8; ++j)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int c = 8 * j + cq, r = r_lo + 8 * h;
                float v0 = apply_act(acc[4 * j + 2 * h] + s_bias[64 + c], relu), v1 = apply_act(acc[4 * j + 2 * h + 1] + s_bias[64 + c + 1], relu);
                if (c >= 60) {   // columns 61..63 carry the flow (cat([out, flow]), model/update.py:20)
                    const float* fl = p.flow + (size_t)(row0 + r) * 3;
                    if (c == 62) { v0 = __ldcg(fl + 1); v1 = __ldcg(fl + 2); } else { v1 = __ldcg(fl); }
                }
                ch_buf_store2(buf_y, r, c, v0, v1);
            }
        asm volatile("bar.sync %0, 128;" ::"r"(1 + grp) : "memory");
        // L2: z (registers), r * net -> X
        ch_layer_mma<128>(acc, 10, 6, tiles, buf_x, buf_y, g_scale, g_shift, iact, s_full, s_empty, cp, grp, t, lane);
#pragma unroll
        for (int j = 0; j < 8; ++j)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int c = 8 * j + cq, r = r_lo + 8 * h;
                const float2 hv = __ldcg(reinterpret_cast<const float2*>(p.net + (size_t)(row0 + r) * 64 + c));
                z[4 * j + 2 * h] = tsigmoid(acc[4 * j + 2 * h] + s_bias[128 + c]);
                z[4 * j + 2 * h + 1] = tsigmoid(acc[4 * j + 2 * h + 1] + s_bias[128 + c + 1]);
                ch_buf_store2(buf_x, r, c, tsigmoid(acc[32 + 4 * j + 2 * h] + s_bias[192 + c]) * hv.x,
                              tsigmoid(acc[32 + 4 * j + 2 * h + 1] + s_bias[192 + c + 1]) * hv.y);
            }
        asm volatile("bar.sync %0, 128;" ::"r"(1 + grp) : "memory");
        // L3: net' -> HBM and X
        ch_layer_mma<64>(acc, 16, 6, tiles, buf_x, buf_y, g_scale, g_shift, iact, s_full, s_empty, cp, grp, t, lane);
#pragma unroll
        for (int j = 0; j < 8; ++j)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int c = 8 * j + cq, r = r_lo + 8 * h;
                const size_t g = (size_t)(row0 + r) * 64 + c;
                const float2 hv = __ldcg(reinterpret_cast<const float2*>(p.net + g));
                const float o0 = tgru_blend(z[4 * j + 2 * h], hv.x, acc[4 * j + 2 * h] + s_bias[256 + c]);
                const float o1 = tgru_blend(z[4 * j + 2 * h + 1], hv.y, acc[4 * j + 2 * h + 1] + s_bias[256 + c + 1]);
                *reinterpret_cast<float2*>(p.net_out + g) = make_float2(o0, o1);
                ch_buf_store2(buf_x, r, c, o0, o1);
            }
        asm volatile("bar.sync %0, 128;" ::"r"(1 + grp) : "memory");
        // L4: P = W_fc1 net' -> HBM (no bias)
        ch_layer_mma<64>(acc, 22, 2, tiles, buf_x, buf_y, g_scale, g_shift, iact, s_full, s_empty, cp, grp, t, lane);
#pragma unroll
        for (int j = 0; j < 8; ++j)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int c = 8 * j + cq, r = r_lo + 8 * h;
                *reinterpret_cast<float2*>(p.p_out + (size_t)(row0 + r) * 64 + c) =
                    make_float2(apply_act(acc[4 * j + 2 * h] + 0.f, none), apply_act(acc[4 * j + 2 * h + 1] + 0.f, none));
            }
    }
}

// hi = tf32(w), lo = tf32(w - hi) of a [rows, ld] weight window [rows, cols] written as [rows_pad, cols_pad] (zero padded)
__global__ void k_weight_split(const float* __restrict__ w, int rows, int cols, int ld, int col0, int rows_pad, int cols_pad,
                               float* __restrict__ hi, float* __restrict__ lo) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= rows_pad * cols_pad) return;
    const int r = i / cols_pad, c = i - r * cols_pad;
    float x = 0.f;
    if (r < rows && c < cols) x = __ldg(w + (size_t)r * ld + col0 + c);
    const float h = tf32_rna(x);
    hi[i] = h;
    lo[i] = tf32_rna(x - h);
}

typedef CUresult (*TcEncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                               const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                               CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static TcEncodeFn tc_encode_fn() {
    static TcEncodeFn fn = nullptr;
    if (!fn) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<TcEncodeFn>(p);
    }
    return fn;
}
// [rows, cols] fp32 row-major (row stride ld floats), box = box_rows x 32 columns, 128-byte swizzle
static int tc_make_map(CUtensorMap* m, const float* base, long long rows, int cols, long long ld, int box_rows) {
    TcEncodeFn fn = tc_encode_fn();
    if (!fn) return fail(PVRAFT_ERR_UNSUPPORTED, "tc_linear: cuTensorMapEncodeTiled is not available from this driver");
    const cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
    const cuuint64_t strides[1] = {(cuuint64_t)ld * sizeof(float)};
    const cuuint32_t box[2] = {(cuuint32_t)kTcKB, (cuuint32_t)box_rows};
    const cuuint32_t estr[2] = {1, 1};
    const CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(base), dims, strides, box, estr,
                          CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                          CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return fail(PVRAFT_ERR_UNSUPPORTED, "tc_linear: cuTensorMapEncodeTiled failed (%d)", (int)r);
    return 0;
}

}  // namespace pvraft

using namespace pvraft;

#ifdef PVRAFT_TC_TIMELINE
extern "C" __attribute__((visibility("default"))) int pvraft_tc_debug_clock(unsigned long long* host64) {
    return (int)cudaMemcpyFromSymbol(host64, g_tc_clock, sizeof(unsigned long long) * 64);
}
#endif

extern "C" int pvraft_tc_weight_split(const float* w, int rows, int cols, int ld, int col0, int rows_pad, int cols_pad, float* hi,
                                      float* lo, void* stream) {
    if (!w || !hi || !lo || rows <= 0 || cols <= 0 || rows_pad < rows || cols_pad < cols) return fail(PVRAFT_ERR_BAD_ARG, "tc_weight_split: bad argument");
    const int n = rows_pad * cols_pad;
    k_weight_split<<<(n + 255) / 256, 256, 0, (cudaStream_t)stream>>>(w, rows, cols, ld > 0 ? ld : cols, col0, rows_pad, cols_pad, hi, lo);
    return check_launch("tc_weight_split");
}

template <bool DET>
static int tc_linear_fwd(const pvraft_tc_linear_args* a, void* ws, void* stream) {
    if (!a || !a->in[0] || !a->w_hi || !a->w_lo || !a->out) return fail(PVRAFT_ERR_BAD_ARG, "tc_linear: null pointer");
    if (a->B <= 0 || a->N <= 0 || a->n_pad < 16 || a->n_pad > 128 || a->n_pad % 16) return fail(PVRAFT_ERR_BAD_ARG, "tc_linear: bad shape (n_pad=%d)", a->n_pad);
    if (a->N % kTcM) return fail(PVRAFT_ERR_UNSUPPORTED, "tc_linear: points per sample (%d) must be a multiple of 128", a->N);
    int K = 0;
    for (int s = 0; s < 3; ++s) {
        if (a->in[s] && (a->in_channels[s] <= 0 || a->in_channels[s] % kTcKB)) return fail(PVRAFT_ERR_UNSUPPORTED, "tc_linear: source %d has %d channels (multiple of 32 needed)", s, a->in_channels[s]);
        if (a->in[s]) K += a->in_channels[s];
    }
    if (K <= 0 || K > 512) return fail(PVRAFT_ERR_UNSUPPORTED, "tc_linear: K=%d", K);
    if (a->in_stats && (a->in_channels[0] % PVRAFT_GN_GROUPS || !a->in_gamma || !a->in_beta)) return fail(PVRAFT_ERR_BAD_ARG, "tc_linear: GroupNorm prologue needs gamma, beta and in_channels[0] %% 8 == 0");
    if (a->tail && (a->epilogue != TC_EPI_PLAIN || a->cout + 3 != a->n_pad || a->n_pad % 32 || a->residual || a->out_stats)) return fail(PVRAFT_ERR_BAD_ARG, "tc_linear: a tail needs the plain epilogue and cout + 3 == n_pad (multiple of 32)");
    if (a->in_min && !a->in_stats) return fail(PVRAFT_ERR_BAD_ARG, "tc_linear: in_min needs the GroupNorm prologue");
    if (a->out_stats && (a->epilogue != TC_EPI_PLAIN || a->cout % PVRAFT_GN_GROUPS || (a->cout / PVRAFT_GN_GROUPS) % 4)) return fail(PVRAFT_ERR_UNSUPPORTED, "tc_linear: out_stats needs a GroupNorm group size that is a multiple of 4 (cout=%d)", a->cout);
    if (a->epilogue < TC_EPI_PLAIN || a->epilogue > TC_EPI_FLOW) return fail(PVRAFT_ERR_BAD_ARG, "tc_linear: unknown epilogue %d", a->epilogue);
    if ((a->epilogue == TC_EPI_GRU_ZR || a->epilogue == TC_EPI_GRU_Q) && (a->cout != 64 || !a->h || (!a->bias && !a->residual))) return fail(PVRAFT_ERR_BAD_ARG, "tc_linear: GRU epilogues need cout=64, h and a bias or a pre-activation term");
    if (a->epilogue == TC_EPI_FLOW && (a->cout != 64 || a->n_pad != 64 || !a->bias || !a->w3 || !a->b3 || (a->coords2_out && !a->coords2) || (a->flow_out && (!a->coords2_out || !a->coords1)))) return fail(PVRAFT_ERR_BAD_ARG, "tc_linear: flow epilogue needs cout = n_pad = 64, bias, w3, b3 and consistent coordinate pointers");
    if (a->epilogue == TC_EPI_GRU_ZR && (a->n_pad != 128 || (!a->bias2 && !a->residual) || !a->out2)) return fail(PVRAFT_ERR_BAD_ARG, "tc_linear: GRU zr epilogue needs n_pad=128, bias2, out2");
    if (a->epilogue == TC_EPI_GRU_Q && (a->n_pad != 64 || !a->z)) return fail(PVRAFT_ERR_BAD_ARG, "tc_linear: GRU q epilogue needs n_pad=64 and z");
    const long long M = (long long)a->B * a->N;
    TcParams p{};
    p.in_stats = a->in_stats; p.in_gamma = a->in_gamma; p.in_beta = a->in_beta; p.in_count = a->in_count; p.in_act = a->in_act;
    p.in_slope = a->in_slope; p.minmax = a->in_min != nullptr;
    p.epi = a->epilogue; p.bias = a->bias; p.bias2 = a->bias2; p.out_act = a->out_act; p.residual = a->residual; p.out = a->out;
    p.out2 = a->out2; p.h = a->h; p.z = a->z; p.out_stats = DET && a->out_stats ? static_cast<double*>(ws) : a->out_stats;
    p.M = (int)M; p.N = a->n_pad; p.K = K; p.cout = a->cout; p.pts_per_sample = a->N;
    CUtensorMap mw_hi, mw_lo;
    int rc;
    for (int s = 0; s < 3; ++s) {
        p.src[s] = a->in[s];
        p.seg_kb[s] = a->in[s] ? a->in_channels[s] / kTcKB : 0;
    }
    p.src_min = a->in_min;
    p.gn_kb = a->in_stats ? a->in_channels[0] / kTcKB : 0;
    p.tail = a->tail;
    p.w3 = a->w3; p.b3 = a->b3; p.coords1 = a->coords1; p.coords2 = a->coords2; p.coords2_out = a->coords2_out; p.flow_out = a->flow_out;
    p.out_ld = a->tail ? a->cout + 3 : a->cout;
    p.settled = a->params_settled ? 1 : 0;
    if ((rc = tc_make_map(&mw_hi, a->w_hi, a->n_pad, K, K, a->n_pad)) || (rc = tc_make_map(&mw_lo, a->w_lo, a->n_pad, K, K, a->n_pad))) return rc;
    CUtensorMap ma[3], mmin;
    for (int s = 0; s < 3; ++s) {   // unused slots repeat source 0 (a tensor map must be valid even if never dereferenced)
        const int q = a->in[s] ? s : 0;
        if ((rc = tc_make_map(&ma[s], a->in[q], M, a->in_channels[q], a->in_channels[q], kTcM))) return rc;
    }
    if ((rc = tc_make_map(&mmin, a->in_min ? a->in_min : a->in[0], M, a->in_channels[0], a->in_channels[0], kTcM))) return rc;
    const size_t a_stage = (size_t)2 * kTcABytes;
    const size_t w_all = (size_t)(K / kTcKB) * 2 * a->n_pad * kTcKB * 4;          // hi + lo of the whole weight matrix
    const bool gru = a->epilogue == TC_EPI_GRU_ZR || a->epilogue == TC_EPI_GRU_Q;
    const size_t fixed = (size_t)(4 * K + 2 * a->n_pad + kTcM * tc_acc_pitch(a->n_pad) + (gru ? 8 * 32 * kTcPitch16 : 0) + 4 * 128 * 2) * sizeof(float) + 1024 + 64;
    const size_t budget = (size_t)kSmemBudget - 2048 /* static barriers */ - fixed;
    // Weights stay resident in shared memory when that still leaves a ring of >= 3 activation stages (re-streaming the
    // same few KB per tile from every SM hot-spots a handful of L2 slices); otherwise they travel with the k-blocks.
    const size_t w_kb = (size_t)2 * a->n_pad * kTcKB * 4;
    const int stages_res = w_all < budget ? (int)((budget - w_all) / a_stage) : 0;
    const int stages_str = (int)(budget / (a_stage + w_kb));
    p.w_resident = (stages_res >= 3 || stages_res >= stages_str) ? 1 : 0;
    int stages = p.w_resident ? stages_res : stages_str;
    stages = stages < 1 ? 1 : (stages > kTcMaxStages ? kTcMaxStages : stages);
    const size_t stage = a_stage + (p.w_resident ? 0 : w_kb);
    if (stages < 2) return fail(PVRAFT_ERR_SMEM, "tc_linear: K=%d, n_pad=%d leave room for only %d operand stage(s) (2 needed)", K, a->n_pad, stages);
    p.stages = stages;
    if (const char* e = getenv("PVRAFT_TC_DBG")) p.dbg = atoi(e);
    const size_t smem = stages * stage + (p.w_resident ? w_all : 0) + fixed;
    decltype(&k_tc_linear<16, DET>) kernel = nullptr;
    switch (a->n_pad) {
        case 16: kernel = k_tc_linear<16, DET>; break;
        case 32: kernel = k_tc_linear<32, DET>; break;
        case 48: kernel = k_tc_linear<48, DET>; break;
        case 64: kernel = k_tc_linear<64, DET>; break;
        case 80: kernel = k_tc_linear<80, DET>; break;
        case 96: kernel = k_tc_linear<96, DET>; break;
        case 112: kernel = k_tc_linear<112, DET>; break;
        default: kernel = k_tc_linear<128, DET>; break;
    }
    if ((rc = opt_in_smem(kernel, smem))) return rc;
    const long long n_tiles = (M + kTcM - 1) / kTcM;
    const int grid = (int)(n_tiles < sm_count() ? n_tiles : sm_count());
    // launched with programmatic stream serialization: the kernel's prologue may start while the previous kernel drains
    const cudaError_t le = launch_pdl(kernel, grid, kTcThreads, smem, (cudaStream_t)stream, mw_hi, mw_lo, ma[0], ma[1], ma[2], mmin, p);
    if (le != cudaSuccess) return fail((int)le, "tc_linear: launch failed: %s", cudaGetErrorString(le));
    rc = check_launch("tc_linear");
    if (rc || !DET || !a->out_stats) return rc;
    return fx_flush_f64(static_cast<const unsigned long long*>(ws), 1, (long long)a->B * 16, (long long)a->B * 16, 0, a->out_stats, (cudaStream_t)stream);
}

extern "C" int pvraft_tc_linear_fwd(const pvraft_tc_linear_args* a, void* det_workspace, void* stream) {
    return det_workspace ? tc_linear_fwd<true>(a, det_workspace, stream) : tc_linear_fwd<false>(a, nullptr, stream);
}

extern "C" int64_t pvraft_tc_linear_det_workspace_bytes(int B) { return (int64_t)B * 16 * kFxWords * 8; }

extern "C" int pvraft_update_chain_fwd(const pvraft_update_chain_args* a, void* stream) {
    if (!a || !a->y1 || !a->y1_stats || !a->gn_gamma || !a->gn_beta || !a->kfeat || !a->cflow || !a->flow || !a->net || !a->inp ||
        !a->b_cc || !a->b_m || !a->b_z || !a->b_r || !a->b_q || !a->net_out || !a->p_out)
        return fail(PVRAFT_ERR_BAD_ARG, "update_chain: null pointer");
    for (int l = 0; l < 5; ++l)
        if (!a->w_hi[l] || !a->w_lo[l]) return fail(PVRAFT_ERR_BAD_ARG, "update_chain: null weight of layer %d", l);
    if (a->B <= 0 || a->N <= 0) return fail(PVRAFT_ERR_BAD_ARG, "update_chain: bad shape (B=%d, N=%d)", a->B, a->N);
    if (a->N % kTcM) return fail(PVRAFT_ERR_UNSUPPORTED, "update_chain: points per sample (%d) must be a multiple of 128", a->N);
    if (a->hidden != 64 || a->context != 64 || a->y1_channels != 128)
        return fail(PVRAFT_ERR_UNSUPPORTED, "update_chain: built for hidden = context = 64 and 128 lookup features (got %d, %d, %d)",
                    a->hidden, a->context, a->y1_channels);
    if (a->net_out == a->net) return fail(PVRAFT_ERR_BAD_ARG, "update_chain: net_out must not alias net");
    const long long M = (long long)a->B * a->N;
    ChainMaps maps;
    const float* src[5] = {a->y1, a->kfeat, a->cflow, a->net, a->inp};
    const int width[5] = {128, 64, 64, 64, 64};
    const int n_pad[5] = {64, 64, 128, 64, 64}, k[5] = {192, 128, 192, 192, 64};
    int rc;
    for (int i = 0; i < 5; ++i) {
        if ((rc = tc_make_map(&maps.a[i], src[i], M, width[i], width[i], kTcM))) return rc;
        if ((rc = tc_make_map(&maps.w_hi[i], a->w_hi[i], n_pad[i], k[i], k[i], n_pad[i])) ||
            (rc = tc_make_map(&maps.w_lo[i], a->w_lo[i], n_pad[i], k[i], k[i], n_pad[i])))
            return rc;
    }
    ChainParams p{};
    p.y1_stats = a->y1_stats; p.gn_gamma = a->gn_gamma; p.gn_beta = a->gn_beta; p.gn_count = a->gn_count; p.gn_slope = a->gn_slope;
    p.flow = a->flow; p.net = a->net;
    p.b_cc = a->b_cc; p.b_m = a->b_m; p.b_z = a->b_z; p.b_r = a->b_r; p.b_q = a->b_q;
    p.net_out = a->net_out; p.p_out = a->p_out;
    p.M = (int)M; p.pts_per_sample = a->N;
    const size_t smem = (size_t)kChStages * kChStageBytes + 2 * kChBufBytes + (2 * 256 + 5 * 64) * sizeof(float) + 1024;
    if ((rc = opt_in_smem(k_update_chain, smem))) return rc;
    const long long n_tiles = M / kTcM;
    const int grid = (int)(n_tiles < sm_count() ? n_tiles : sm_count());
    const cudaError_t le = launch_pdl(k_update_chain, grid, kChThreads, smem, (cudaStream_t)stream, maps, p);
    if (le != cudaSuccess) return fail((int)le, "update_chain: launch failed: %s", cudaGetErrorString(le));
    return check_launch("update_chain");
}
