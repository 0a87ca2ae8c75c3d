// Weight gradient of a per-point 1x1 convolution on the Hopper tensor cores (wgmma) with bf16 operands: the backward of the
// loop layers in the 'bf16-mixed' training mode (pvraft_b200/train.py, LinearFn).
//
//   dW[o,i] += sum_r bf16(dy[r,o]) . bf16(x[r,i])   (fp32 accumulation)      db[o] += sum_r dy[r,o]   (fp32, unrounded dy)
//
// The contraction runs over the rows r, so both point-major operands are MN-major for the MMA.  The threads that load them
// transpose them instead: D[i,o] = (x^T)[i,:] . (dy^T)[o,:] with A = x^T (64 input channels of the CTA, wgmma M) and
// B = dy^T (all cout output channels, wgmma N), both written K-major in the bf16 SWIZZLE_64B layout of the 'bf16-compute'
// k_tc_linear (wgmma.cuh: tc_bf16_store, wgmma_desc_bf16).  One CTA = one warpgroup; grid = (row slabs, ceil(cin / 64)).
// A CTA walks its slab 32 rows at a time: every thread loads 4 consecutive rows of one channel (lanes = consecutive channels,
// so each load instruction reads contiguous bytes of a row; rows past the end and channels past cin read as zero), rounds
// them to bf16 and stores them as one 8-byte chunk of the operand tile; two wgmma.m64nNk16 per 32 rows run while the next
// rows are loaded (double-buffered tiles).  The [64 x cout] partial stays in registers across the whole slab and is reduced
// once at the end: fp32 atomics into dW, or (DET) exact fixed-point additions into the caller's workspace.  The slab count
// follows from the shapes and is capped by a constant, so what each CTA adds is a function of the shapes.
#include "fixed_point.cuh"
#include "tma.cuh"
#include "wgmma.cuh"

namespace pvraft {

constexpr int kWgTcThreads = 128;     // one warpgroup
constexpr int kWgTcRows = 32;         // rows per step: one bf16 k-block (two K = 16 slices)
constexpr int kWgTcSlabRows = 256;    // target rows per CTA: the atomics of the final reduction stay small next to the loads
constexpr int kWgTcMaxSlabs = 128;    // cap of the slab count (a constant: the rows a CTA sums depend on the shapes only)

// NT = cout (32, 64, 96 or 128): the wgmma width
template <int NT, bool DET>
__global__ void __launch_bounds__(kWgTcThreads) k_tc_wgrad(const float* __restrict__ x, const float* __restrict__ dy, long long rows,
                                                            int cin, long long slab_rows, Acc<DET> dW, int dw_ld, Acc<DET> db) {
    constexpr int kA = 64 * kWgTcRows * 2;        // bf16 x^T tile [64 channels][32 rows]
    constexpr int kB = NT * kWgTcRows * 2;        // bf16 dy^T tile [NT channels][32 rows]
    constexpr int kChans = 64 + NT;               // channels a step loads: the CTA's 64 of x, then all NT of dy
    constexpr int kUnits = (kWgTcRows / 4) * kChans;   // (4-row group, channel) pairs of a step
    constexpr int kPerThread = (kUnits + kWgTcThreads - 1) / kWgTcThreads;
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    unsigned char* tiles = SMEM_ALIGN_1024(smem_raw);   // 2 x [A | B], each tile 512-byte aligned
    float* s_db = reinterpret_cast<float*>(tiles + 2 * (kA + kB));   // [8 row groups][NT] partial column sums of dy
    const int t = threadIdx.x;
    const int c0 = blockIdx.y * 64;               // first input channel of this CTA
    const bool bias_cta = db && blockIdx.y == 0;
    const long long r_begin = (long long)blockIdx.x * slab_rows;
    const long long r_end = min(rows, r_begin + slab_rows);
    const int steps = r_end > r_begin ? (int)((r_end - r_begin + kWgTcRows - 1) / kWgTcRows) : 0;

    float acc[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0.f;
    float bsum[kPerThread];
#pragma unroll
    for (int j = 0; j < kPerThread; ++j) bsum[j] = 0.f;

    for (int s = 0; s < steps; ++s) {
        const long long r0 = r_begin + (long long)s * kWgTcRows;
        float4 v[kPerThread];
#pragma unroll
        for (int j = 0; j < kPerThread; ++j) {   // global -> registers (all loads of the step in flight together)
            const int u = t + j * kWgTcThreads;
            const int ch = u % kChans, g = u / kChans;
            float e[4] = {0.f, 0.f, 0.f, 0.f};
            if (u < kUnits) {
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    const long long r = r0 + g * 4 + q;
                    if (r < r_end) {
                        if (ch < 64) {
                            if (c0 + ch < cin) e[q] = __ldg(x + r * cin + c0 + ch);
                        } else {
                            e[q] = __ldg(dy + r * NT + ch - 64);
                        }
                    }
                }
            }
            v[j] = make_float4(e[0], e[1], e[2], e[3]);
        }
        unsigned char* a_tile = tiles + (s & 1) * (kA + kB);
        unsigned char* b_tile = a_tile + kA;
        wgmma_wait<1>();   // this warp's MMAs of step s - 2, which read these tiles, have retired ...
        __syncthreads();   // ... and every other warp's
#pragma unroll
        for (int j = 0; j < kPerThread; ++j) {   // registers -> bf16 K-major tiles (row = channel, k = row of the slab)
            const int u = t + j * kWgTcThreads;
            if (u >= kUnits) continue;
            const int ch = u % kChans, g = u / kChans;
            if (ch < 64) {
                tc_bf16_store(a_tile, ch, g, v[j]);
            } else {
                tc_bf16_store(b_tile, ch - 64, g, v[j]);
                if (bias_cta) bsum[j] += (v[j].x + v[j].y) + (v[j].z + v[j].w);
            }
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy writes -> visible to wgmma
        __syncthreads();
        wgmma_fence_regs(acc);
        wgmma_fence();
        const unsigned long long da = wgmma_desc_bf16(a_tile), dbd = wgmma_desc_bf16(b_tile);
#pragma unroll
        for (int k = 0; k < kWgTcRows / 16; ++k) wgmma_bf16<NT>(acc, wgmma_desc_k(da, k), wgmma_desc_k(dbd, k), 1);
        wgmma_commit();
    }
    wgmma_wait<0>();
    wgmma_fence_regs(acc);

    // dW: accumulator fragment -> (input channel i = c0 + 16 warp + lane / 4 (+8), output channel o = 8 j + 2 (lane % 4) (+1))
    const int warp = warp_id(), lane = lane_id();
    const int i0 = c0 + warp * 16 + (lane >> 2);
#pragma unroll
    for (int j = 0; j < NT / 8; ++j) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const int i = i0 + (e >> 1) * 8, o = 8 * j + 2 * (lane & 3) + (e & 1);
            const float a = acc[4 * j + e];
            if (i < cin && a != 0.f) add(dW, (size_t)o * dw_ld + i, a);
        }
    }
    if (!bias_cta) return;
    // db: the per-thread sums of every (row group, output channel) pair -- each pair belongs to exactly one thread --
    // combined in a fixed order (row group 0..7)
#pragma unroll
    for (int j = 0; j < kPerThread; ++j) {
        const int u = t + j * kWgTcThreads;
        const int ch = u % kChans, g = u / kChans;
        if (u < kUnits && ch >= 64) s_db[g * NT + ch - 64] = bsum[j];
    }
    __syncthreads();
    if (t < NT) {
        float b = 0.f;
#pragma unroll
        for (int g = 0; g < 8; ++g) b += s_db[g * NT + t];
        if (b != 0.f) add(db, t, b);
    }
}

}  // namespace pvraft

using namespace pvraft;

template <bool DET>
static int tc_wgrad(const float* x, const float* dy, int64_t rows, int cin, int cout, float* dW, int dw_ld, float* db, void* ws, void* stream) {
    if (!x || !dy || !dW || rows <= 0 || dw_ld < 0 || (dw_ld > 0 && dw_ld < cin)) return fail(PVRAFT_ERR_BAD_ARG, "tc_wgrad_bf16: bad argument");
    if (cin < 32 || cin > 192 || cin % 32 || cout < 32 || cout > 128 || cout % 32)
        return fail(PVRAFT_ERR_UNSUPPORTED, "tc_wgrad_bf16: cin=%d cout=%d (multiples of 32, cin <= 192, cout <= 128)", cin, cout);
    const int steps = (int)((rows + kWgTcRows - 1) / kWgTcRows);
    long long slabs = (rows + kWgTcSlabRows - 1) / kWgTcSlabRows;
    if (slabs > kWgTcMaxSlabs) slabs = kWgTcMaxSlabs;
    const long long slab_rows = (long long)((steps + slabs - 1) / slabs) * kWgTcRows;
    slabs = (rows + slab_rows - 1) / slab_rows;
    const dim3 grid((unsigned)slabs, (unsigned)((cin + 63) / 64));
    const size_t smem = 1024 + 2 * (size_t)(64 + cout) * kWgTcRows * 2 + (size_t)8 * cout * sizeof(float);
    const int ld = dw_ld > 0 ? dw_ld : cin;
    cudaStream_t st = (cudaStream_t)stream;
    const WgradWs L = wgrad_ws(ws, cin, cout);
    Acc<DET> out_w, out_b;   // DET: the weight slots are [cout][cin], leading dimension cin
    int out_ld = ld;
    if constexpr (DET) { out_w = L.w; out_b = db ? L.b : FxSlots{}; out_ld = cin; }
    else { out_w = dW; out_b = db; }
    decltype(&k_tc_wgrad<32, DET>) kernel = nullptr;
    switch (cout) {
        case 32: kernel = k_tc_wgrad<32, DET>; break;
        case 64: kernel = k_tc_wgrad<64, DET>; break;
        case 96: kernel = k_tc_wgrad<96, DET>; break;
        default: kernel = k_tc_wgrad<128, DET>; break;
    }
    int rc;
    if ((rc = opt_in_smem(kernel, smem))) return rc;
    kernel<<<grid, kWgTcThreads, smem, st>>>(x, dy, rows, cin, slab_rows, out_w, out_ld, out_b);
    if ((rc = check_launch("tc_wgrad_bf16")) || !DET) return rc;
    return wgrad_flush(L, cin, cout, ld, dW, db, st);
}

extern "C" int pvraft_tc_wgrad_bf16(const float* x, const float* dy, int64_t rows, int cin, int cout, float* dW, int dw_ld, float* db,
                                    void* det_workspace, void* stream) {
    auto f = det_workspace ? tc_wgrad<true> : tc_wgrad<false>;
    return f(x, dy, rows, cin, cout, dW, dw_ld, db, det_workspace, stream);
}

extern "C" int64_t pvraft_tc_wgrad_bf16_det_workspace_bytes(int cin, int cout) { return wgrad_ws(nullptr, cin, cout).bytes; }
