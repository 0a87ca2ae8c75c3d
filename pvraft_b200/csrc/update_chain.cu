// The update chain: MotionEncoder, ConvGRU and the flow-head fc1 pre-transform of one RAFT iteration in one launch, on the
// Hopper tensor cores (wgmma), fp32-accurate (3xTF32) or on bf16 operands.
//   L0 cc     = relu(W_cc [lrelu(GN(y1)) | kfeat] + b_cc)        K 192, N 64   (corr.py fold_corr_motion)
//   L1 motion = [relu(W_m [cc | cflow] + b_m) (61) | flow (3)]   K 128, N 64
//   L2 [z|r]  = sigmoid(W_zr [net | inp | motion] + b_zr)        K 192, N 128;  z stays in registers, r*net -> X
//   L3 net'   = (1 - z) net + z tanh(W_q [r*net | inp | motion] + b_q)   K 192, N 64  -> HBM and X
//   L4 P      = W_fc1[:, :64] net'                               K 64,  N 64   -> HBM
// Each layer runs exactly the k-block sequence, transform, 3xTF32 wgmma order and epilogue formula of its k_tc_linear
// launch (tc_linear.cu), so the results are the same bits.  Warp 8 streams, per k-block, the weight boxes (hi, lo) of every
// layer and the raw activation box of the k-blocks read from HBM (y1, kfeat, cflow, net, inp).  Warpgroup grp (warps 4 grp
// .. +3) owns rows 64 grp .. +63 of every tile from operand to output: it transforms its rows of a box, issues the wgmma, and
// at the end of a layer applies the epilogue to its accumulator registers, writing the activation either to HBM (net', P) or
// as raw fp32 into an on-chip [128 x 64] buffer laid out like two TMA boxes (X: cc, then r*net, then net'; Y: motion).  A
// k-block read from a buffer is split from there into the ring stage instead of in place.  Nothing crosses the two
// warpgroups but the ring, so a layer boundary costs a warpgroup only its own epilogue.
// BF16 (the 'bf16-compute' mode of the RAFT loop): the bf16 form of the five k_tc_linear launches, with their k-block order,
// bf16 rounding, two wgmma.m64nNk16.bf16 per k-block and epilogues, so again the same bits.  A stage holds the bf16 operand
// tile of the two warpgroups (4 KB each) and one bf16 weight box instead of hi and lo: 32 KB instead of 64, so the ring is
// four stages deep instead of two.
#include "tma.cuh"
#include "wgmma.cuh"

namespace pvraft {

constexpr int kChThreads = 288;   // 2 transform + MMA + epilogue warpgroups | TMA producer
constexpr int kChProducerWarp = 8;
constexpr int kChWBytes = 128 * kTcKB * 4;                   // one weight box of the widest layer (N = 128)
// ring depth and stage layout: [A hi][A lo][W hi][W lo] = 64 KB; BF16: [A raw 16 KB][A bf16, 4 KB per group][W 8 KB] = 32 KB
template <bool BF16> struct ChRing {
    static constexpr int stages = BF16 ? 4 : 2;
    static constexpr int w_off = BF16 ? kTcABytes + 2 * kTcABf16Bytes : 2 * kTcABytes;
    static constexpr int stage_bytes = BF16 ? w_off + kChWBytes / 2 : w_off + 2 * kChWBytes;
};
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
__device__ __forceinline__ int ch_w_bytes(int layer, bool bf16) { return (layer == 2 ? 128 : 64) * kTcKB * (bf16 ? 2 : 4); }

// raw fp32 value pair (columns c, c + 1; c even) of tile row r into an on-chip [128 x 64] buffer in the TMA box layout
__device__ __forceinline__ void ch_buf_store2(unsigned char* buf, int r, int c, float v0, float v1) {
    const int lc = (c & 31) >> 2;
    *reinterpret_cast<float2*>(buf + (c >> 5) * kTcABytes + r * 128 + ((lc ^ (r & 7)) << 4) + (c & 3) * 4) = make_float2(v0, v1);
}

// the MMA warpgroup's part of one tile step: wait for the stage, transform its rows of the k-block (from the stage in place,
// or from an on-chip buffer), issue the 3xTF32 (or bf16) wgmma and release the stage
template <int N, bool BF16>
__device__ __forceinline__ void ch_kblock(float (&acc)[64], int kb, int src, int skb, unsigned char* tiles, unsigned char* buf_x,
                                          unsigned char* buf_y, const float* g_scale, const float* g_shift, const ActCoef& iact,
                                          unsigned long long* s_full, unsigned long long* s_empty, TcCursor& cp, int grp, int t,
                                          int lane) {
    const int s = cp.s;
    mbar_wait(&s_full[s], cp.phase);
    unsigned char* st = tiles + (size_t)s * ChRing<BF16>::stage_bytes;
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
        if constexpr (BF16) tc_bf16_store(st + kTcABytes + grp * kTcABf16Bytes, c >> 3, lc, x);
        else tc_split_store(st, off, x);
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    asm volatile("bar.sync %0, 128;" ::"r"(1 + grp) : "memory");
    const unsigned char* wb = st + ChRing<BF16>::w_off;
    wgmma_fence_regs(acc);
    wgmma_fence();
    if constexpr (BF16) tc_mma_kblock_bf16<N>(acc, wgmma_desc_bf16(st + kTcABytes + grp * kTcABf16Bytes), wgmma_desc_bf16(wb), kb);
    else tc_mma_kblock<N>(acc, wgmma_desc(st + grp * 64 * 128), wgmma_desc(st + kTcABytes + grp * 64 * 128), wgmma_desc(wb),
                          wgmma_desc(wb + N * kTcKB * 4), kb);
    wgmma_commit();
    // retire this k-block before the next transform: with two stages the refill of this one then overlaps the whole next
    // step (waiting one k-block later would start each refill only once the next box had landed, exposing every load)
    wgmma_wait<0>();
    if (lane == 0) mbar_arrive(&s_empty[s]);
    cp.next(kChSteps, ChRing<BF16>::stages);
}
// all k-blocks of one layer (steps i0 .. i0 + nkb - 1), then the accumulator is final in registers
template <int N, bool BF16>
__device__ __forceinline__ void ch_layer_mma(float (&acc)[64], int i0, int nkb, unsigned char* tiles, unsigned char* buf_x,
                                             unsigned char* buf_y, const float* g_scale, const float* g_shift, const ActCoef& iact,
                                             unsigned long long* s_full, unsigned long long* s_empty, TcCursor& cp, int grp, int t,
                                             int lane) {
    for (int kb = 0; kb < nkb; ++kb)
        ch_kblock<N, BF16>(acc, kb, ch_src(i0 + kb), ch_skb(i0 + kb), tiles, buf_x, buf_y, g_scale, g_shift, iact, s_full, s_empty, cp, grp, t, lane);
    wgmma_fence_regs(acc);
}

// BF16: maps.w_hi hold the bf16 weights, maps.w_lo are not read
template <bool BF16>
__global__ void __launch_bounds__(kChThreads, 1)
k_update_chain(const __grid_constant__ ChainMaps maps, const ChainParams p) {
    constexpr int kChStages = ChRing<BF16>::stages, kChStageBytes = ChRing<BF16>::stage_bytes;
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    unsigned char* tiles = SMEM_ALIGN_1024(smem_raw);
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
            prefetch_tensormap(&maps.a[i]);
            prefetch_tensormap(&maps.w_hi[i]);
            if constexpr (!BF16) prefetch_tensormap(&maps.w_lo[i]);
        }
        for (int s = 0; s < kChStages; ++s) { mbar_init(&s_full[s], 1); mbar_init(&s_empty[s], 8); }
        fence_mbarrier_init();
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
                const int wb = ch_w_bytes(layer, BF16);
                const int lkb = i - ch_first(layer), skb = ch_skb(i);   // k-block of the layer's weights, of the source
                mbar_wait(&s_empty[cw.s], cw.phase ^ 1u);
                unsigned char* st = tiles + (size_t)cw.s * kChStageBytes;
                mbar_expect_tx(&s_full[cw.s], (unsigned)((src < CH_X ? kTcABytes : 0) + (BF16 ? 1 : 2) * wb));
                if (src < CH_X) tma_load_2d(st, &maps.a[src], &s_full[cw.s], skb * kTcKB, row0);
                tma_load_2d(st + ChRing<BF16>::w_off, &maps.w_hi[layer], &s_full[cw.s], lkb * kTcKB, 0);
                if constexpr (!BF16) tma_load_2d(st + ChRing<BF16>::w_off + wb, &maps.w_lo[layer], &s_full[cw.s], lkb * kTcKB, 0);
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
        ch_layer_mma<64, BF16>(acc, 0, 6, tiles, buf_x, buf_y, g_scale, g_shift, iact, s_full, s_empty, cp, grp, t, lane);
#pragma unroll
        for (int j = 0; j < 8; ++j)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int c = 8 * j + cq;
                ch_buf_store2(buf_x, r_lo + 8 * h, c, apply_act(acc[4 * j + 2 * h] + s_bias[c], relu), apply_act(acc[4 * j + 2 * h + 1] + s_bias[c + 1], relu));
            }
        asm volatile("bar.sync %0, 128;" ::"r"(1 + grp) : "memory");
        // L1: motion = [relu(.) | flow] -> Y
        ch_layer_mma<64, BF16>(acc, 6, 4, tiles, buf_x, buf_y, g_scale, g_shift, iact, s_full, s_empty, cp, grp, t, lane);
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
        ch_layer_mma<128, BF16>(acc, 10, 6, tiles, buf_x, buf_y, g_scale, g_shift, iact, s_full, s_empty, cp, grp, t, lane);
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
        ch_layer_mma<64, BF16>(acc, 16, 6, tiles, buf_x, buf_y, g_scale, g_shift, iact, s_full, s_empty, cp, grp, t, lane);
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
        ch_layer_mma<64, BF16>(acc, 22, 2, tiles, buf_x, buf_y, g_scale, g_shift, iact, s_full, s_empty, cp, grp, t, lane);
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

}  // namespace pvraft

using namespace pvraft;

extern "C" int pvraft_update_chain_fwd(const pvraft_update_chain_args* a, void* stream) {
    if (!a || !a->y1 || !a->y1_stats || !a->gn_gamma || !a->gn_beta || !a->kfeat || !a->cflow || !a->flow || !a->net || !a->inp ||
        !a->b_cc || !a->b_m || !a->b_z || !a->b_r || !a->b_q || !a->net_out || !a->p_out)
        return fail(PVRAFT_ERR_BAD_ARG, "update_chain: null pointer");
    const bool bf16 = a->w_bf16[0] != nullptr;
    for (int l = 0; l < 5; ++l) {
        if (bf16 ? (!a->w_bf16[l] || a->w_hi[l] || a->w_lo[l]) : (!a->w_hi[l] || !a->w_lo[l] || a->w_bf16[l]))
            return fail(PVRAFT_ERR_BAD_ARG, "update_chain: layer %d needs w_hi and w_lo (3xTF32) or w_bf16 (bf16), as every other layer", l);
    }
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
        if ((rc = make_tensor_map(&maps.a[i], src[i], M, width[i], width[i], kTcM, "update_chain"))) return rc;
        if (bf16) {   // the unused lo slots repeat the bf16 maps (a tensor map must be valid even if never dereferenced)
            if ((rc = make_tensor_map_bf16(&maps.w_hi[i], a->w_bf16[i], n_pad[i], k[i], k[i], n_pad[i], "update_chain"))) return rc;
            maps.w_lo[i] = maps.w_hi[i];
        } else if ((rc = make_tensor_map(&maps.w_hi[i], a->w_hi[i], n_pad[i], k[i], k[i], n_pad[i], "update_chain")) ||
                   (rc = make_tensor_map(&maps.w_lo[i], a->w_lo[i], n_pad[i], k[i], k[i], n_pad[i], "update_chain"))) {
            return rc;
        }
    }
    ChainParams p{};
    p.y1_stats = a->y1_stats; p.gn_gamma = a->gn_gamma; p.gn_beta = a->gn_beta; p.gn_count = a->gn_count; p.gn_slope = a->gn_slope;
    p.flow = a->flow; p.net = a->net;
    p.b_cc = a->b_cc; p.b_m = a->b_m; p.b_z = a->b_z; p.b_r = a->b_r; p.b_q = a->b_q;
    p.net_out = a->net_out; p.p_out = a->p_out;
    p.M = (int)M; p.pts_per_sample = a->N;
    const size_t ring = bf16 ? (size_t)ChRing<true>::stages * ChRing<true>::stage_bytes : (size_t)ChRing<false>::stages * ChRing<false>::stage_bytes;
    const size_t smem = ring + 2 * kChBufBytes + (2 * 256 + 5 * 64) * sizeof(float) + 1024;
    const auto kernel = bf16 ? k_update_chain<true> : k_update_chain<false>;
    if ((rc = opt_in_smem(kernel, smem))) return rc;
    const long long n_tiles = M / kTcM;
    const int grid = (int)(n_tiles < sm_count() ? n_tiles : sm_count());
    const cudaError_t le = launch_pdl(kernel, grid, kChThreads, smem, (cudaStream_t)stream, maps, p);
    if (le != cudaSuccess) return fail((int)le, "update_chain: launch failed: %s", cudaGetErrorString(le));
    return check_launch("update_chain");
}
