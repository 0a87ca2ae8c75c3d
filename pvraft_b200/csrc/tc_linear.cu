// Per-point linear layers on the Hopper tensor cores (wgmma), fp32-accurate (3xTF32) or on bf16 operands, with the GroupNorm / activation
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
// BF16 (the 'bf16-compute' mode of the RAFT loop): the transformed activations are rounded to bf16 (nearest even) and stored
// in the lo half of the stage, one 64-row tile per warpgroup at the group's offset; the weights arrive as bf16 boxes
// [N x 32] (SWIZZLE_64B, pvraft_tc_weight_bf16); 2 x wgmma.m64nNk16.bf16 per k-block, fp32 accumulation and epilogues.
// Launched with programmatic stream serialization: the prologue overlaps the previous kernel's tail (griddepcontrol.wait
// precedes the first global read).  Replaces the k_linear / k_gru / k_corrfeat / k_flowout CUDA-core kernels whenever
// Npts % 128 == 0 and every source has a multiple of 32 channels.
#include "fixed_point.cuh"
#include "tma.cuh"
#include "wgmma.cuh"

namespace pvraft {

constexpr int kTcThreads = 544;   // 8 epilogue warps | 2 transform + MMA warpgroups | TMA producer
constexpr int kTcEpiThreads = 256, kTcProducerWarp = 16;
constexpr int kTcMaxStages = 6;

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
    int gn_kb;                // k-blocks (from the start: source 0) that go through the GroupNorm prologue
    int out_ld;               // row stride of `out` in floats (cout, or cout + 3 with a tail)
    const float* tail;        // [M,3] copied into output columns cout..cout+2, or nullptr
    const float *w3, *b3, *coords1, *coords2;   // FLOW epilogue
    float *coords2_out, *flow_out;
};

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
                    // lane = column: (sum, sum^2) of this warp's 32 rows, read down the staged tile (conflict-free): the
                    // compensated sum, the squares about the column's first row (pivot_sumsq); the double sums then
                    // replace the block's first four rows
                    const float piv = stg[lane];
                    float s1 = 0.f, e1 = 0.f, s2 = 0.f;
#pragma unroll
                    for (int r = 0; r < 32; ++r) {
                        const float a = stg[r * pitch + lane], d = a - piv;
                        kahan_add(s1, e1, a);
                        s2 = fmaf(d, d, s2);
                    }
                    const double a1 = kahan_value(s1, e1), a2 = pivot_sumsq(a1, piv, s2, 32);
                    __syncwarp();
                    *reinterpret_cast<double2*>(stg + (lane >> 3) * pitch + (lane & 7) * 4) = make_double2(a1, a2);
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
                // column t's partial of the warp of lane quadrant w: in that warp's staged block of chunk t & ~31
                const float* part = s_acc + (size_t)((t & 31) >> 3) * pitch + (t & ~31) + (t & 7) * 4;
#pragma unroll
                for (int w = 0; w < 4; ++w) {
                    const double2 pr = *reinterpret_cast<const double2*>(part + (size_t)w * 32 * pitch);
                    a1 += pr.x;
                    a2 += pr.y;
                }
            }
            if ((gsz & (gsz - 1)) == 0 && gsz <= 32) {   // groups are aligned runs of gsz lanes
                for (int o = gsz >> 1; o > 0; o >>= 1) {
                    a1 += __shfl_xor_sync(kFull, a1, o);
                    a2 += __shfl_xor_sync(kFull, a2, o);
                }
                if ((t & (gsz - 1)) == 0 && t < p.cout) {
                    if constexpr (DET) {
                        const FxSlots fx = fx_slots(p.out_stats) + (sample * 16 + (t / gsz) * 2);
                        add(fx, 0, a1);
                        add(fx, 1, a2);
                    } else {
                    atomicAdd(p.out_stats + (size_t)sample * 16 + (t / gsz) * 2 + 0, a1);
                    atomicAdd(p.out_stats + (size_t)sample * 16 + (t / gsz) * 2 + 1, a2);
                    }
                }
            } else if (DET && t < p.cout) {
                const FxSlots fx = fx_slots(p.out_stats) + (sample * 16 + (t / gsz) * 2);
                add(fx, 0, a1);
                add(fx, 1, a2);
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

// row pitch (floats) of the shared accumulator tile: whole 32-column epilogue chunks plus 4, so that thread-per-row 16-byte
// accesses of 8 consecutive rows fall into distinct bank groups
__host__ __device__ __forceinline__ int tc_acc_pitch(int n) { return ((n + 31) & ~31) + 4; }

// A CTA walks tiles blockIdx.x, +gridDim.x, ...; the operand ring runs across tile boundaries.
// NT = p.N (the padded cout): the wgmma shape is part of the instruction.  BF16: bf16 operands (map_w_hi holds the bf16
// weights, map_w_lo is not read)
template <int NT, bool DET, bool BF16>
__global__ void __launch_bounds__(kTcThreads, 1)
k_tc_linear(const __grid_constant__ CUtensorMap map_w_hi, const __grid_constant__ CUtensorMap map_w_lo,
            const __grid_constant__ CUtensorMap map_a0, const __grid_constant__ CUtensorMap map_a1,
            const __grid_constant__ CUtensorMap map_a2, const __grid_constant__ CUtensorMap map_min, const TcParams p) {
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    unsigned char* tiles = SMEM_ALIGN_1024(smem_raw);
    // stage layout: [A hi 16K][A lo 16K][W hi N*128][W lo N*128, only when the weights are streamed];
    // resident weights live behind the ring as num_kb x [W hi][W lo].
    // BF16: [A raw 16K][A bf16: 4K at the start of each group's 8K of the lo half][W N*64, only when streamed]
    constexpr int w_boxes = BF16 ? 1 : 2;
    const int w_bytes = p.N * kTcKB * (BF16 ? 2 : 4);
    const int w_off = 2 * kTcABytes;
    const int stage_bytes = w_off + (p.w_resident ? 0 : w_boxes * w_bytes);
    const int S = p.stages;
    const int num_kb = p.K / kTcKB;
    const int acc_pitch = tc_acc_pitch(NT);
    unsigned char* w_res = tiles + (size_t)S * stage_bytes;
    float* s_scale = reinterpret_cast<float*>(w_res + (p.w_resident ? (size_t)num_kb * w_boxes * w_bytes : 0));   // [2 groups][scale K | shift K]
    float* s_bias = s_scale + 4 * p.K;                                            // [2 * N]
    float* s_acc = s_bias + 2 * p.N;                                              // [128 rows][acc_pitch] accumulator tile
    float* s_estage = s_acc + (size_t)kTcM * acc_pitch;                           // GRU epilogues: [8 warps][32][20] staging
    float* s_part = s_estage + (p.epi == TC_EPI_GRU_ZR || p.epi == TC_EPI_GRU_Q ? 8 * 32 * kTcPitch16 : 0);   // FLOW: [128 rows][4] exchange | w3
    __shared__ __align__(8) unsigned long long s_full[kTcMaxStages], s_empty[kTcMaxStages];
    __shared__ __align__(8) unsigned long long s_acc_full, s_acc_empty, s_w_full;
    const int warp = warp_id(), lane = lane_id();
    const int n_tiles = (p.M + kTcM - 1) / kTcM;
    const int my_tiles = blockIdx.x < n_tiles ? (n_tiles - 1 - blockIdx.x) / gridDim.x + 1 : 0;
    const int total_steps = my_tiles * num_kb;

    if (warp == kTcProducerWarp && lane == 0) {
        prefetch_tensormap(&map_w_hi);
        if constexpr (!BF16) prefetch_tensormap(&map_w_lo);
        prefetch_tensormap(&map_a0);
        for (int s = 0; s < S; ++s) { mbar_init(&s_full[s], 1); mbar_init(&s_empty[s], 8); }   // 8 MMA warps release a stage
        mbar_init(&s_acc_full, 8);     // 8 MMA warps deposit the accumulator tile
        mbar_init(&s_acc_empty, 8);    // 8 epilogue warps have consumed it
        mbar_init(&s_w_full, 1);
        fence_mbarrier_init();
    }
    // Programmatic dependent launch: everything above (shared-memory carve-up, barrier init, descriptor prefetch) may
    // overlap the tail of the previous kernel on this stream.  The layer's PARAMETERS (hi/lo weights, biases) are fetched
    // in that window too when the caller vouches that they are settled (p.settled: last written several launches ago --
    // the steady state of a forward, whose weights are split once): the SMs that finished the previous kernel early then
    // hold their weights when the dependency resolves.  Every read of an ACTIVATION is below the wait.
    auto load_weights = [&]() {   // the whole weight matrix (hi and lo) once per CTA
        mbar_expect_tx(&s_w_full, (unsigned)(num_kb * w_boxes * w_bytes));
        for (int kb = 0; kb < num_kb; ++kb) {
            tma_load_2d(w_res + (size_t)kb * w_boxes * w_bytes, &map_w_hi, &s_w_full, kb * kTcKB, 0);
            if constexpr (!BF16) tma_load_2d(w_res + (size_t)kb * 2 * w_bytes + w_bytes, &map_w_lo, &s_w_full, kb * kTcKB, 0);
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
            const unsigned tx = (unsigned)(kTcABytes * (p.minmax ? 2 : 1) + (p.w_resident ? 0 : w_boxes * w_bytes));
            TcCursor cw;
            for (int step = 0; step < total_steps; ++step, cw.next(num_kb, S)) {
                const int s = cw.s, kb = cw.kb;
                const int row0 = (blockIdx.x + cw.ti * gridDim.x) * kTcM;
                mbar_wait(&s_empty[s], cw.phase ^ 1u);   // the MMAs that read this stage last time have retired
                unsigned char* st = tiles + (size_t)s * stage_bytes;
                mbar_expect_tx(&s_full[s], tx);
                // raw fp32 rows of the source this k-block belongs to land where the hi operand will be (the transform works
                // in place); the min array of a (max, min) pair lands in the lo half
                if (kb < p.seg_kb[0]) tma_load_2d(st, &map_a0, &s_full[s], kb * kTcKB, row0);
                else if (kb < p.seg_kb[0] + p.seg_kb[1]) tma_load_2d(st, &map_a1, &s_full[s], (kb - p.seg_kb[0]) * kTcKB, row0);
                else tma_load_2d(st, &map_a2, &s_full[s], (kb - p.seg_kb[0] - p.seg_kb[1]) * kTcKB, row0);
                if (p.minmax) tma_load_2d(st + kTcABytes, &map_min, &s_full[s], kb * kTcKB, row0);
                if (!p.w_resident) {
                    tma_load_2d(st + w_off, &map_w_hi, &s_full[s], kb * kTcKB, 0);
                    if constexpr (!BF16) tma_load_2d(st + w_off + w_bytes, &map_w_lo, &s_full[s], kb * kTcKB, 0);
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
        if (p.w_resident) mbar_wait(&s_w_full, 0u);
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
            mbar_wait(&s_full[s], cp.phase);   // the raw box(es) of this k-block have landed
            unsigned char* st = tiles + (size_t)s * stage_bytes;
            float4 xb[4];   // BF16: the transformed chunks, stored once the group has read the whole box
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
                if constexpr (BF16) {
                    xb[i] = x;
                    continue;
                }
                float4 hi, lo;
                hi.x = tf32_rna(x.x); hi.y = tf32_rna(x.y); hi.z = tf32_rna(x.z); hi.w = tf32_rna(x.w);
                lo.x = tf32_rna(x.x - hi.x); lo.y = tf32_rna(x.y - hi.y); lo.z = tf32_rna(x.z - hi.z); lo.w = tf32_rna(x.w - hi.w);
                *reinterpret_cast<float4*>(st + off) = hi;   // in place: raw -> hi; the lo half of the stage held the min array
                *reinterpret_cast<float4*>(st + kTcABytes + off) = lo;
            }
            if constexpr (BF16) {
                // the bf16 tile overwrites min-array rows of this group that its other threads may not have read yet
                if (p.minmax) asm volatile("bar.sync %0, 128;" ::"r"(1 + grp) : "memory");
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const int c = t + i * 128;
                    tc_bf16_store(st + kTcABytes + a_off, c >> 3, c & 7, xb[i]);
                }
            }
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy writes -> visible to wgmma (async proxy)
            asm volatile("bar.sync %0, 128;" ::"r"(1 + grp) : "memory");   // the group's 64 rows are in place
            const unsigned char* wb = p.w_resident ? w_res + (size_t)kb * w_boxes * w_bytes : st + w_off;
            wgmma_fence_regs(acc);
            wgmma_fence();
            if constexpr (BF16) tc_mma_kblock_bf16<NT>(acc, wgmma_desc_bf16(st + kTcABytes + a_off), wgmma_desc_bf16(wb), kb);
            else tc_mma_kblock<NT>(acc, wgmma_desc(st + a_off), wgmma_desc(st + kTcABytes + a_off), wgmma_desc(wb), wgmma_desc(wb + w_bytes), kb);
            wgmma_commit();
            wgmma_wait<1>();   // the previous k-block's MMAs have retired: its stage may be refilled
            if (prev_s >= 0 && lane == 0) mbar_arrive(&s_empty[prev_s]);
            prev_s = s;
            cp.next(num_kb, S);
          }
          wgmma_wait<0>();
          wgmma_fence_regs(acc);
          if (lane == 0) mbar_arrive(&s_empty[prev_s]);
          prev_s = -1;
          mbar_wait(&s_acc_empty, ((unsigned)ti & 1u) ^ 1u);   // the epilogue has consumed the previous tile
          // accumulator fragment -> rows 64 grp + 16 (warp % 4) + lane / 4 (+8), columns 8 j + 2 (lane % 4) (+1)
          float* a0 = s_acc + (size_t)(grp * 64 + (warp & 3) * 16 + (lane >> 2)) * acc_pitch + 2 * (lane & 3);
#pragma unroll
          for (int j = 0; j < NT / 8; ++j) {
              *reinterpret_cast<float2*>(a0 + 8 * j) = make_float2(acc[4 * j + 0], acc[4 * j + 1]);
              *reinterpret_cast<float2*>(a0 + (size_t)8 * acc_pitch + 8 * j) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
          }
          __syncwarp();
          if (lane == 0) mbar_arrive(&s_acc_full);
        }
    } else {
        // ===== epilogue: accumulator tile -> registers -> global, one tile behind the MMA =====
        const int quad = warp & 3;   // rows 32 quad .. +31 of the tile
        const int half = warp >> 2;  // two warps per quadrant: 32-column chunks c0 = 32*half, +64, ...
        for (int ti = 0; ti < my_tiles; ++ti) {
            const int row0 = (blockIdx.x + ti * gridDim.x) * kTcM;
            mbar_wait(&s_acc_full, (unsigned)ti & 1u);
            const int sample = row0 / p.pts_per_sample;
            tc_epilogue<DET>(p, s_acc, acc_pitch, quad, half, lane, row0, sample, s_bias, s_estage, s_part);
            __syncwarp();
            if (lane == 0) mbar_arrive(&s_acc_empty);   // one arrival per epilogue warp
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

// bf16(w) (round to nearest even) of a [rows, ld] weight window [rows, cols] written as [rows_pad, cols_pad] (zero padded)
__global__ void k_weight_bf16(const float* __restrict__ w, int rows, int cols, int ld, int col0, int rows_pad, int cols_pad,
                              __nv_bfloat16* __restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= rows_pad * cols_pad) return;
    const int r = i / cols_pad, c = i - r * cols_pad;
    float x = 0.f;
    if (r < rows && c < cols) x = __ldg(w + (size_t)r * ld + col0 + c);
    out[i] = __float2bfloat16_rn(x);
}

}  // namespace pvraft

using namespace pvraft;

extern "C" int pvraft_tc_weight_split(const float* w, int rows, int cols, int ld, int col0, int rows_pad, int cols_pad, float* hi,
                                      float* lo, void* stream) {
    if (!w || !hi || !lo || rows <= 0 || cols <= 0 || rows_pad < rows || cols_pad < cols) return fail(PVRAFT_ERR_BAD_ARG, "tc_weight_split: bad argument");
    const int n = rows_pad * cols_pad;
    k_weight_split<<<(n + 255) / 256, 256, 0, (cudaStream_t)stream>>>(w, rows, cols, ld > 0 ? ld : cols, col0, rows_pad, cols_pad, hi, lo);
    return check_launch("tc_weight_split");
}

extern "C" int pvraft_tc_weight_bf16(const float* w, int rows, int cols, int ld, int col0, int rows_pad, int cols_pad, uint16_t* out,
                                     void* stream) {
    if (!w || !out || rows <= 0 || cols <= 0 || rows_pad < rows || cols_pad < cols) return fail(PVRAFT_ERR_BAD_ARG, "tc_weight_bf16: bad argument");
    const int n = rows_pad * cols_pad;
    k_weight_bf16<<<(n + 255) / 256, 256, 0, (cudaStream_t)stream>>>(w, rows, cols, ld > 0 ? ld : cols, col0, rows_pad, cols_pad,
                                                                      reinterpret_cast<__nv_bfloat16*>(out));
    return check_launch("tc_weight_bf16");
}

template <bool DET, bool BF16>
static int tc_linear_fwd(const pvraft_tc_linear_args* a, void* ws, void* stream) {
    if (!a || !a->in[0] || !a->out) return fail(PVRAFT_ERR_BAD_ARG, "tc_linear: null pointer");
    if (BF16 ? (a->w_hi || a->w_lo) : (!a->w_hi || !a->w_lo))
        return fail(PVRAFT_ERR_BAD_ARG, "tc_linear: pass either w_hi and w_lo (3xTF32) or w_bf16 (bf16), not both");
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
    if (BF16) {   // the unused lo slot repeats the bf16 map (a tensor map must be valid even if never dereferenced)
        if ((rc = make_tensor_map_bf16(&mw_hi, a->w_bf16, a->n_pad, K, K, a->n_pad, "tc_linear"))) return rc;
        mw_lo = mw_hi;
    } else if ((rc = make_tensor_map(&mw_hi, a->w_hi, a->n_pad, K, K, a->n_pad, "tc_linear")) ||
               (rc = make_tensor_map(&mw_lo, a->w_lo, a->n_pad, K, K, a->n_pad, "tc_linear"))) {
        return rc;
    }
    CUtensorMap ma[3], mmin;
    for (int s = 0; s < 3; ++s) {   // unused slots repeat source 0 (a tensor map must be valid even if never dereferenced)
        const int q = a->in[s] ? s : 0;
        if ((rc = make_tensor_map(&ma[s], a->in[q], M, a->in_channels[q], a->in_channels[q], kTcM, "tc_linear"))) return rc;
    }
    if ((rc = make_tensor_map(&mmin, a->in_min ? a->in_min : a->in[0], M, a->in_channels[0], a->in_channels[0], kTcM, "tc_linear"))) return rc;
    const size_t a_stage = (size_t)2 * kTcABytes;
    const size_t w_kb = (size_t)(BF16 ? 2 : 8) * a->n_pad * kTcKB;               // one k-block of weights: hi + lo, or bf16
    const size_t w_all = (size_t)(K / kTcKB) * w_kb;                               // the whole weight matrix
    const bool gru = a->epilogue == TC_EPI_GRU_ZR || a->epilogue == TC_EPI_GRU_Q;
    const size_t fixed = (size_t)(4 * K + 2 * a->n_pad + kTcM * tc_acc_pitch(a->n_pad) + (gru ? 8 * 32 * kTcPitch16 : 0) + 4 * 128 * 2) * sizeof(float) + 1024 + 64;
    const size_t budget = (size_t)kSmemBudget - 2048 /* static barriers */ - fixed;
    // Weights stay resident in shared memory when that still leaves a ring of >= 3 activation stages (re-streaming the
    // same few KB per tile from every SM hot-spots a handful of L2 slices); otherwise they travel with the k-blocks.
    const int stages_res = w_all < budget ? (int)((budget - w_all) / a_stage) : 0;
    const int stages_str = (int)(budget / (a_stage + w_kb));
    p.w_resident = (stages_res >= 3 || stages_res >= stages_str) ? 1 : 0;
    int stages = p.w_resident ? stages_res : stages_str;
    stages = stages < 1 ? 1 : (stages > kTcMaxStages ? kTcMaxStages : stages);
    const size_t stage = a_stage + (p.w_resident ? 0 : w_kb);
    if (stages < 2) return fail(PVRAFT_ERR_SMEM, "tc_linear: K=%d, n_pad=%d leave room for only %d operand stage(s) (2 needed)", K, a->n_pad, stages);
    p.stages = stages;
    const size_t smem = stages * stage + (p.w_resident ? w_all : 0) + fixed;
    decltype(&k_tc_linear<16, DET, BF16>) kernel = nullptr;
    switch (a->n_pad) {
        case 16: kernel = k_tc_linear<16, DET, BF16>; break;
        case 32: kernel = k_tc_linear<32, DET, BF16>; break;
        case 48: kernel = k_tc_linear<48, DET, BF16>; break;
        case 64: kernel = k_tc_linear<64, DET, BF16>; break;
        case 80: kernel = k_tc_linear<80, DET, BF16>; break;
        case 96: kernel = k_tc_linear<96, DET, BF16>; break;
        case 112: kernel = k_tc_linear<112, DET, BF16>; break;
        default: kernel = k_tc_linear<128, DET, BF16>; break;
    }
    if ((rc = opt_in_smem(kernel, smem))) return rc;
    const long long n_tiles = (M + kTcM - 1) / kTcM;
    const int grid = (int)(n_tiles < sm_count() ? n_tiles : sm_count());
    // launched with programmatic stream serialization: the kernel's prologue may start while the previous kernel drains
    const cudaError_t le = launch_pdl(kernel, grid, kTcThreads, smem, (cudaStream_t)stream, mw_hi, mw_lo, ma[0], ma[1], ma[2], mmin, p);
    if (le != cudaSuccess) return fail((int)le, "tc_linear: launch failed: %s", cudaGetErrorString(le));
    rc = check_launch("tc_linear");
    if (rc || !DET || !a->out_stats) return rc;
    return gn_stats_flush(ws, a->B, a->out_stats, (cudaStream_t)stream);
}

extern "C" int pvraft_tc_linear_fwd(const pvraft_tc_linear_args* a, void* det_workspace, void* stream) {
    if (a && a->w_bf16)
        return det_workspace ? tc_linear_fwd<true, true>(a, det_workspace, stream) : tc_linear_fwd<false, true>(a, nullptr, stream);
    return det_workspace ? tc_linear_fwd<true, false>(a, det_workspace, stream) : tc_linear_fwd<false, false>(a, nullptr, stream);
}

extern "C" int64_t pvraft_tc_linear_det_workspace_bytes(int B) { return gn_stats_ws_bytes(B); }
