// All-pairs feature correlation on the Hopper tensor cores (wgmma + TMA), fp32-accurate.
//
// Replaces CorrBlock.calculate_corr (reference model/corr.py:95-100):  corr[b,i,j] = <fmap1[b,:,i], fmap2[b,:,j]> / sqrt(C).
// This is the one large dense contraction of the model (2*N*N*C = 17.2 GFLOP per sample at N=8192).
//
// The operands are point-major [B,N,C] (K-major for the MMA).  To keep fp32 parity on a TF32 datapath every
// operand is split once into hi = tf32(x) and lo = tf32(x - hi) (k_tf32_split) and each product is evaluated as
// hi*hi + lo*hi + hi*lo (the classic 3xTF32 scheme, error ~2^-21 relative per product; the dropped lo*lo term is
// ~2^-22).  The kernel is persistent (one CTA per SM walks 128 x 128 output tiles); roles and pipeline are described at
// k_corr_gemm below.  The division by sqrt(C) is a true division, as on the reference's CPU path.
#include "tma.cuh"
#include "wgmma.cuh"

namespace pvraft {

constexpr int kGemmThreads = 384;   // warpgroup 0: TMA producer (one thread) | warpgroups 1, 2: MMA + epilogue
constexpr int kTileM = 128, kTileN = 128, kBlockK = 32;     // 32 tf32 = one 128-byte swizzle row
constexpr int kOperandBytes = kTileM * kBlockK * 4;         // 16 KB
constexpr int kStageBytes = 4 * kOperandBytes;              // A_hi, A_lo, B_hi, B_lo
constexpr int kStages = 3;
constexpr int kConsumerWarps = 8;

struct GemmParams {
    float* corr;   // [B, tiles_m * 128, ldc]: rows [r0, r0 + 128 tiles_m) x columns [c0, c0 + 128 tiles_n) of every sample
    int N, M, C;   // rows per sample of operand A (fmap1) and of operand B (fmap2), channels
    float scale;   // sqrt(C): the divisor of model/corr.py:99
    float rscale;  // RN(1 / scale)
    int r0, c0;    // first row of fmap1 / of fmap2 (multiples of 128)
    int tiles_m, tiles_n;   // 128-row / 128-column tiles of the window
    long long ldc;          // output row stride in floats
    long long n_tiles;      // B * tiles_m * tiles_n
};

// x / s, correctly rounded, from r = RN(1/s) (Markstein): q0 = x r; q = q0 + (x - q0 s) r.  Three instructions instead of
// the ~10 of the generic division, bit-identical to it (checked against true division on 1.3e8 values, see DESIGN.md).
__device__ __forceinline__ float div_by_const(float x, float s, float r) {
    const float q0 = x * r;
    return fmaf(fmaf(-q0, s, x), r, q0);
}

// Persistent kernel, one CTA per SM, tiles t = blockIdx.x + i * gridDim.x with the column tile fastest (neighbouring CTAs
// share the A row-panel in L2):
//   warp 0          TMA producer: four 128 x 32 boxes (A hi/lo, B hi/lo) per k-block into a 3-stage ring; it runs up to
//                   three k-blocks ahead, across tile boundaries, so the next tile's operands land during the epilogue
//   warpgroups 1-2  rows [64 (g - 1), +64) of the tile: 3 x 4 wgmma.m64n128k8 per k-block (the stage is released once
//                   the next k-block's group is in flight), then the epilogue straight from the accumulator registers:
//                   exact division by sqrt(C), each store instruction writes 8 rows x 32 contiguous bytes
__global__ void __launch_bounds__(kGemmThreads, 1)
k_corr_gemm(const __grid_constant__ CUtensorMap map_a_hi, const __grid_constant__ CUtensorMap map_a_lo,
            const __grid_constant__ CUtensorMap map_b_hi, const __grid_constant__ CUtensorMap map_b_lo, const GemmParams p) {
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    unsigned char* tiles = SMEM_ALIGN_1024(smem_raw);
    __shared__ __align__(8) unsigned long long s_full[kStages], s_empty[kStages];
    const int warp = warp_id(), lane = lane_id();
    const int num_kb = p.C / kBlockK;
    const long long my_tiles = blockIdx.x < p.n_tiles ? (p.n_tiles - 1 - blockIdx.x) / gridDim.x + 1 : 0;

    if (warp == 0 && lane == 0) {
        prefetch_tensormap(&map_a_hi);
        prefetch_tensormap(&map_a_lo);
        prefetch_tensormap(&map_b_hi);
        prefetch_tensormap(&map_b_lo);
        for (int s = 0; s < kStages; ++s) { mbar_init(&s_full[s], 1); mbar_init(&s_empty[s], kConsumerWarps); }
        fence_mbarrier_init();
    }
    __syncthreads();
    const int tiles_per_batch = p.tiles_m * p.tiles_n;

    if (warp < 4) {
        // ===== TMA producer =====
        if (warp == 0 && lane == 0) {
            int s = 0;
            unsigned phase = 0;
            for (long long i = 0; i < my_tiles; ++i) {
                const long long t = blockIdx.x + i * gridDim.x;
                const int b = (int)(t / tiles_per_batch), r = (int)(t - (long long)b * tiles_per_batch);
                const int tile_m = r / p.tiles_n, tile_n = r - tile_m * p.tiles_n;
                const int row_a = b * p.N + p.r0 + tile_m * kTileM, row_b = b * p.M + p.c0 + tile_n * kTileN;
                for (int kb = 0; kb < num_kb; ++kb) {
                    mbar_wait(&s_empty[s], phase ^ 1u);
                    unsigned char* st = tiles + (size_t)s * kStageBytes;
                    mbar_expect_tx(&s_full[s], kStageBytes);
                    tma_load_2d(st + 0 * kOperandBytes, &map_a_hi, &s_full[s], kb * kBlockK, row_a);
                    tma_load_2d(st + 1 * kOperandBytes, &map_a_lo, &s_full[s], kb * kBlockK, row_a);
                    tma_load_2d(st + 2 * kOperandBytes, &map_b_hi, &s_full[s], kb * kBlockK, row_b);
                    tma_load_2d(st + 3 * kOperandBytes, &map_b_lo, &s_full[s], kb * kBlockK, row_b);
                    if (++s == kStages) { s = 0; phase ^= 1u; }
                }
            }
        }
        return;
    }
    // ===== MMA + epilogue, one warpgroup per 64-row half of the tile =====
    const int half = (warp >> 2) - 1;             // 0 | 1
    const int wq = warp & 3;                       // warp within the warpgroup: rows 16 wq .. +15 of the half
    const int a_off = half * 64 * 128;             // byte offset of the half's rows inside an A box (1024-aligned)
    float acc[64];
    int s = 0, prev_s = -1;
    unsigned phase = 0;
    for (long long i = 0; i < my_tiles; ++i) {
        const long long t = blockIdx.x + i * gridDim.x;
        const int b = (int)(t / tiles_per_batch), r = (int)(t - (long long)b * tiles_per_batch);
        const int tile_m = r / p.tiles_n, tile_n = r - tile_m * p.tiles_n;
        for (int kb = 0; kb < num_kb; ++kb) {
            mbar_wait(&s_full[s], phase);
            unsigned char* st = tiles + (size_t)s * kStageBytes;
            const unsigned long long a_hi = wgmma_desc(st + 0 * kOperandBytes + a_off), a_lo = wgmma_desc(st + 1 * kOperandBytes + a_off);
            const unsigned long long b_hi = wgmma_desc(st + 2 * kOperandBytes), b_lo = wgmma_desc(st + 3 * kOperandBytes);
            wgmma_fence_regs(acc);
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < kBlockK / 8; ++k) {
                wgmma_tf32<kTileN>(acc, wgmma_desc_k(a_hi, k), wgmma_desc_k(b_hi, k), (kb | k) != 0);
                wgmma_tf32<kTileN>(acc, wgmma_desc_k(a_lo, k), wgmma_desc_k(b_hi, k), 1);
                wgmma_tf32<kTileN>(acc, wgmma_desc_k(a_hi, k), wgmma_desc_k(b_lo, k), 1);
            }
            wgmma_commit();
            wgmma_wait<1>();                       // the previous k-block's MMAs have retired: its stage may be refilled
            if (prev_s >= 0 && lane == 0) mbar_arrive(&s_empty[prev_s]);
            prev_s = s;
            if (++s == kStages) { s = 0; phase ^= 1u; }
        }
        wgmma_wait<0>();
        wgmma_fence_regs(acc);
        if (lane == 0) mbar_arrive(&s_empty[prev_s]);
        prev_s = -1;
        // corr / sqrt(C) as a true (correctly rounded) division (model/corr.py:99)
        const int row = tile_m * kTileM + half * 64 + wq * 16 + (lane >> 2);
        float* o = p.corr + ((size_t)b * p.tiles_m * kTileM + row) * (size_t)p.ldc + (size_t)tile_n * kTileN + 2 * (lane & 3);
        const size_t down8 = (size_t)8 * p.ldc;
#pragma unroll
        for (int j = 0; j < kTileN / 8; ++j) {
            *reinterpret_cast<float2*>(o + 8 * j) = make_float2(div_by_const(acc[4 * j + 0], p.scale, p.rscale), div_by_const(acc[4 * j + 1], p.scale, p.rscale));
            *reinterpret_cast<float2*>(o + down8 + 8 * j) = make_float2(div_by_const(acc[4 * j + 2], p.scale, p.rscale), div_by_const(acc[4 * j + 3], p.scale, p.rscale));
        }
    }
}

// hi = tf32(x) (round to nearest), lo = tf32(x - hi)
__global__ void k_tf32_split(const float* __restrict__ x, long long n, float* __restrict__ hi, float* __restrict__ lo) {
    const long long i = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * 4;
    if (i >= n) return;
    const float4 v = *reinterpret_cast<const float4*>(x + i);
    float h[4], l[4];
    const float in[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        unsigned hb, lb;
        asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(hb) : "f"(in[q]));
        h[q] = __uint_as_float(hb);
        asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(lb) : "f"(in[q] - h[q]));
        l[q] = __uint_as_float(lb);
    }
    *reinterpret_cast<float4*>(hi + i) = make_float4(h[0], h[1], h[2], h[3]);
    *reinterpret_cast<float4*>(lo + i) = make_float4(l[0], l[1], l[2], l[3]);
}

// Rows [r0, r0 + 128 tiles_m) x columns [c0, c0 + 128 tiles_n) of every sample, from split operands A [B*N, C] and
// B [B*M, C] (hi/lo of both maps), into corr [B, 128 tiles_m, ldc]
static int launch_gemm(const float* a_hi, const float* a_lo, const float* b_hi, const float* b_lo, int B, int N, int M, int C, int r0,
                       int tiles_m, int c0, int tiles_n, float* corr, long long ldc, cudaStream_t st) {
    int rc;
    CUtensorMap ma_hi, ma_lo, mb_hi, mb_lo;
    const long long rows_a = (long long)B * N, rows_b = (long long)B * M;
    if ((rc = make_tensor_map(&ma_hi, a_hi, rows_a, C, C, kTileM, "corr_matmul")) ||
        (rc = make_tensor_map(&ma_lo, a_lo, rows_a, C, C, kTileM, "corr_matmul")) ||
        (rc = make_tensor_map(&mb_hi, b_hi, rows_b, C, C, kTileN, "corr_matmul")) ||
        (rc = make_tensor_map(&mb_lo, b_lo, rows_b, C, C, kTileN, "corr_matmul")))
        return rc;
    GemmParams p{};
    p.corr = corr; p.N = N; p.M = M; p.C = C;
    p.scale = sqrtf((float)C);
    p.rscale = (float)(1.0 / (double)p.scale);
    p.r0 = r0; p.c0 = c0;
    p.tiles_m = tiles_m; p.tiles_n = tiles_n;
    p.ldc = ldc;
    p.n_tiles = (long long)B * tiles_m * tiles_n;
    const size_t smem = (size_t)kStages * kStageBytes + 1024;
    if ((rc = opt_in_smem(k_corr_gemm, smem))) return rc;
    const int grid = (int)(p.n_tiles < sm_count() ? p.n_tiles : sm_count());
    k_corr_gemm<<<grid, kGemmThreads, smem, st>>>(ma_hi, ma_lo, mb_hi, mb_lo, p);
    return check_launch("corr_gemm");
}

static void launch_split(const float* x, long long n, float* hi, float* lo, cudaStream_t st) {
    k_tf32_split<<<(unsigned)((n / 4 + 255) / 256), 256, 0, st>>>(x, n, hi, lo);
}

}  // namespace pvraft

using namespace pvraft;

extern "C" int64_t pvraft_corr_matmul_workspace_bytes(int B, int N, int M, int C) {
    if (B <= 0 || N <= 0 || M <= 0 || C <= 0) return 0;
    return (int64_t)2 * B * ((int64_t)N + M) * C * (int64_t)sizeof(float);   // hi/lo copies of both feature maps
}

extern "C" int pvraft_corr_matmul_fwd(const float* fmap1, const float* fmap2, int B, int N, int M, int C, float* corr, void* workspace,
                                      void* stream) {
    if (!fmap1 || !fmap2 || !corr || !workspace) return fail(PVRAFT_ERR_BAD_ARG, "corr_matmul: null pointer");
    if (B <= 0 || N <= 0 || M <= 0 || C <= 0) return fail(PVRAFT_ERR_BAD_ARG, "corr_matmul: bad shape");
    if (N % kTileM || M % kTileN || C % kBlockK)
        return fail(PVRAFT_ERR_UNSUPPORTED, "corr_matmul: N=%d and M=%d must be multiples of 128 and C=%d of 32", N, M, C);
    if (B > 65535 || N / kTileM > 65535 || M / kTileN > 65535) return fail(PVRAFT_ERR_UNSUPPORTED, "corr_matmul: grid too large");
    cudaStream_t st = (cudaStream_t)stream;
    const long long na = (long long)B * N * C, nb = (long long)B * M * C;
    float* a_hi = reinterpret_cast<float*>(workspace);
    float* a_lo = a_hi + na;
    float* b_hi = a_lo + na;
    float* b_lo = b_hi + nb;
    launch_split(fmap1, na, a_hi, a_lo, st);
    launch_split(fmap2, nb, b_hi, b_lo, st);
    const int rc = check_launch("tf32_split");
    if (rc) return rc;
    return launch_gemm(a_hi, a_lo, b_hi, b_lo, B, N, M, C, 0, N / kTileM, 0, M / kTileN, corr, M, st);
}

extern "C" int pvraft_tf32_split_fwd(const float* x, int64_t n, float* hi, float* lo, void* stream) {
    if (!x || !hi || !lo || n <= 0) return fail(PVRAFT_ERR_BAD_ARG, "tf32_split: bad argument");
    if (n % 4 || ((uintptr_t)x | (uintptr_t)hi | (uintptr_t)lo) % 16)
        return fail(PVRAFT_ERR_UNSUPPORTED, "tf32_split: n=%lld must be a multiple of 4 and the buffers 16-byte aligned", (long long)n);
    launch_split(x, n, hi, lo, (cudaStream_t)stream);
    return check_launch("tf32_split");
}

extern "C" int pvraft_corr_matmul_window_fwd(const float* a_hi, const float* a_lo, const float* b_hi, const float* b_lo, int B, int N,
                                             int M, int C, int r0, int rows, int c0, int cols, float* corr, int64_t ldc, void* stream) {
    if (!a_hi || !a_lo || !b_hi || !b_lo || !corr) return fail(PVRAFT_ERR_BAD_ARG, "corr_matmul_window: null pointer");
    if (B <= 0 || N <= 0 || M <= 0 || C <= 0 || rows <= 0 || cols <= 0 || r0 < 0 || c0 < 0)
        return fail(PVRAFT_ERR_BAD_ARG, "corr_matmul_window: bad shape");
    if (N % kTileM || M % kTileN || C % kBlockK || r0 % kTileM || c0 % kTileN)
        return fail(PVRAFT_ERR_UNSUPPORTED, "corr_matmul_window: N=%d, M=%d, r0=%d and c0=%d must be multiples of 128 and C=%d of 32", N,
                    M, r0, c0, C);
    const int tiles_m = (rows + kTileM - 1) / kTileM, tiles_n = (cols + kTileN - 1) / kTileN;
    if (rows > N - r0 || cols > M - c0 || r0 + tiles_m * kTileM > N || c0 + tiles_n * kTileN > M)
        return fail(PVRAFT_ERR_UNSUPPORTED, "corr_matmul_window: rows [%d, %d) x columns [%d, %d), whole tiles, exceed N=%d x M=%d", r0,
                    r0 + tiles_m * kTileM, c0, c0 + tiles_n * kTileN, N, M);
    if (ldc < (int64_t)tiles_n * kTileN || ldc % 4)
        return fail(PVRAFT_ERR_UNSUPPORTED, "corr_matmul_window: ldc=%lld (need a multiple of 4, >= %d)", (long long)ldc, tiles_n * kTileN);
    if ((long long)B * N > 0x7fffffffLL || (long long)B * M > 0x7fffffffLL)
        return fail(PVRAFT_ERR_UNSUPPORTED, "corr_matmul_window: B*N=%lld / B*M=%lld operand rows", (long long)B * N, (long long)B * M);
    return launch_gemm(a_hi, a_lo, b_hi, b_lo, B, N, M, C, r0, tiles_m, c0, tiles_n, corr, ldc, (cudaStream_t)stream);
}
