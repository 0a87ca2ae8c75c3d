// Backward kernels (and the few layer-wise forward kernels the inference path fuses away) behind the gradient contract of
// SURVEY.md section 8b: everything tools/engine.py:131-147 differentiates through when it calls loss.backward() on the
// flows of RSF.forward -- the truncated correlation (model/corr.py:31-42), the voxel / kNN lookup (corr.py:47-93), the
// 1x1 convolutions and GroupNorms of the update block (model/update.py) and the SetConvs (model/flot/gconv.py:58-85).
//
// The training path runs layer by layer (pvraft_b200/train.py wraps each entry point in a torch.autograd.Function); every
// arithmetic step of forward and backward is one of the kernels of this library.  Layout conventions as in the forward
// kernels: per-point features point-major [B,rows,C]; "rows" is N for per-point layers and N*32 for per-edge layers.
// Reductions into parameter gradients use fp32 / fp64 atomics (order-nondeterministic, like ATen's own CUDA backward) in
// the default instantiations.  The DET instantiations (what an entry point runs when given a det_workspace) add exact
// fixed-point values instead (fixed_point.cuh) and size their grids from the shapes alone, so their results are bitwise
// reproducible; their accumulator arguments then point at the caller's fixed-point workspace.
#include "fixed_point.cuh"

namespace pvraft {

// ---------------------------------------------------------------------------------------------------------------------
// 1x1 convolution, weight / bias gradient:  dW[o,i] += sum_r dY[r,o] X[r,i],  db[o] += sum_r dY[r,o]
// (the data gradient dX = dY W is pvraft_linear_fwd with the transposed weight).
// grid = (row workers, ceil(cout/32)); a CTA stages 64-row tiles of X (all cin columns) and of its 32 dY columns and keeps a
// 4x4 register tile per thread and (o-block, i-block) pair across ALL its row tiles; one atomicAdd pass at the end.
// ---------------------------------------------------------------------------------------------------------------------
constexpr int kWgRows = 64;
constexpr int kWgThreads = 256;

template <bool DET>
__global__ void __launch_bounds__(kWgThreads) k_linear_wgrad(const float* __restrict__ x, const float* __restrict__ dy, long long rows,
                                                             int cin, int cout, float* __restrict__ dW, int dw_ld, float* __restrict__ db) {
    extern __shared__ __align__(16) float smem_wg[];
    const int cin_p = (cin + 3) & ~3;
    const int xs_ld = cin_p + 4;                 // +4 floats: consecutive rows start in different bank groups
    float* xs = smem_wg;                         // [64][xs_ld]
    float* ds = smem_wg + kWgRows * xs_ld;       // [64][36]
    const int o0 = blockIdx.y * 32;
    const int ib_n = cin_p >> 2;                 // 4-column blocks of X
    const int tiles = 8 * ib_n;                  // (o-block, i-block) pairs of this CTA
    float acc[2][16];
    float accb[2][4];
#pragma unroll
    for (int t = 0; t < 2; ++t) {
#pragma unroll
        for (int q = 0; q < 16; ++q) acc[t][q] = 0.f;
#pragma unroll
        for (int q = 0; q < 4; ++q) accb[t][q] = 0.f;
    }
    for (long long r0 = (long long)blockIdx.x * kWgRows; r0 < rows; r0 += (long long)gridDim.x * kWgRows) {
        const int nr = (int)min((long long)kWgRows, rows - r0);
        __syncthreads();
        for (int i = threadIdx.x; i < kWgRows * cin_p; i += kWgThreads) {
            const int r = i / cin_p, c = i - r * cin_p;
            xs[r * xs_ld + c] = (r < nr && c < cin) ? __ldg(x + (r0 + r) * cin + c) : 0.f;
        }
        for (int i = threadIdx.x; i < kWgRows * 32; i += kWgThreads) {
            const int r = i >> 5, c = i & 31;
            ds[r * 36 + c] = (r < nr && o0 + c < cout) ? __ldg(dy + (r0 + r) * cout + o0 + c) : 0.f;
        }
        __syncthreads();
#pragma unroll
        for (int t = 0; t < 2; ++t) {
            const int tile = threadIdx.x + t * kWgThreads;
            if (tile < tiles) {
                const int ob = tile / ib_n, ib = tile - ob * ib_n;
                const float* xp = xs + ib * 4;
                const float* dp = ds + ob * 4;
#pragma unroll 4
                for (int r = 0; r < kWgRows; ++r) {
                    const float4 xv = *reinterpret_cast<const float4*>(xp + r * xs_ld);
                    const float4 dv = *reinterpret_cast<const float4*>(dp + r * 36);
                    const float dvv[4] = {dv.x, dv.y, dv.z, dv.w};
#pragma unroll
                    for (int o = 0; o < 4; ++o) {
                        acc[t][o * 4 + 0] = fmaf(dvv[o], xv.x, acc[t][o * 4 + 0]);
                        acc[t][o * 4 + 1] = fmaf(dvv[o], xv.y, acc[t][o * 4 + 1]);
                        acc[t][o * 4 + 2] = fmaf(dvv[o], xv.z, acc[t][o * 4 + 2]);
                        acc[t][o * 4 + 3] = fmaf(dvv[o], xv.w, acc[t][o * 4 + 3]);
                        if (ib == 0) accb[t][o] += dvv[o];
                    }
                }
            }
        }
    }
#pragma unroll
    for (int t = 0; t < 2; ++t) {
        const int tile = threadIdx.x + t * kWgThreads;
        if (tile < tiles) {
            const int ob = tile / ib_n, ib = tile - ob * ib_n;
#pragma unroll
            for (int o = 0; o < 4; ++o) {
                const int oo = o0 + ob * 4 + o;
                if (oo >= cout) continue;
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const int ii = ib * 4 + i;
                    if (ii < cin && acc[t][o * 4 + i] != 0.f) {
                        if constexpr (DET) fx_atomic(reinterpret_cast<unsigned long long*>(dW) + ((size_t)oo * cin + ii) * kFxWords, (double)acc[t][o * 4 + i]);
                        else atomicAdd(dW + (size_t)oo * dw_ld + ii, acc[t][o * 4 + i]);
                    }
                }
                if (db && ib == 0 && accb[t][o] != 0.f) {
                    if constexpr (DET) fx_atomic(reinterpret_cast<unsigned long long*>(db) + (size_t)oo * kFxWords, (double)accb[t][o]);
                    else atomicAdd(db + oo, accb[t][o]);
                }
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// Backward of a linear layer with a tiny input width (cin <= 4: the SetConv edge term W_e e over [dx,dy,dz] and the
// knn_conv over [corr, dx, dy, dz]; rows = B*N*32).  ONE pass over dy [rows, cout] gives dW, db and (if asked) dx -- the
// generic pair (k_linear with the transposed weight + k_linear_wgrad) reads dy twice and keeps 8 of 256 threads busy in
// the weight-gradient tile loop at this shape.  LPR lanes share a row, 16 output channels each (cout = 16 * LPR).
// ---------------------------------------------------------------------------------------------------------------------
template <int LPR, bool DET>
__global__ void __launch_bounds__(256) k_linear_bwd_small(const float* __restrict__ x, const float* __restrict__ dy, const float* __restrict__ W,
                                                          long long rows, int cin, int w_ld, float* __restrict__ dW, int dw_ld,
                                                          float* __restrict__ db, float* __restrict__ dx) {
    constexpr int COUT = 16 * LPR, RPW = 32 / LPR;   // LPR = 3 or 6 leaves two lanes of the warp idle
    __shared__ float4 s_w[COUT];
    __shared__ float s_acc[COUT][5];
    const int lane = lane_id(), w = warp_id(), q = lane % LPR, rr = lane / LPR;
    const bool active = rr < RPW;
    for (int i = threadIdx.x; i < COUT; i += blockDim.x) {
        float v[4] = {0.f, 0.f, 0.f, 0.f};
        for (int k = 0; k < cin; ++k) v[k] = __ldg(W + (size_t)i * w_ld + k);
        s_w[i] = make_float4(v[0], v[1], v[2], v[3]);
        for (int k = 0; k < 5; ++k) s_acc[i][k] = 0.f;
    }
    __syncthreads();
    float acc[16][4], accb[16];
#pragma unroll
    for (int o = 0; o < 16; ++o) { accb[o] = 0.f; acc[o][0] = acc[o][1] = acc[o][2] = acc[o][3] = 0.f; }
    const long long stride = (long long)gridDim.x * 8 * RPW;
    long long r = ((long long)blockIdx.x * 8 + w) * RPW + rr;
    float4 d4[4];
    float xv[4];
    auto fetch = [&](long long row) {
        if (active && row < rows) {
            const float4* dp = reinterpret_cast<const float4*>(dy + (size_t)row * COUT + q * 16);
#pragma unroll
            for (int k = 0; k < 4; ++k) d4[k] = __ldg(dp + k);
            if (cin == 4) {
                const float4 t = __ldg(reinterpret_cast<const float4*>(x + (size_t)row * 4));
                xv[0] = t.x; xv[1] = t.y; xv[2] = t.z; xv[3] = t.w;
            } else {
#pragma unroll
                for (int k = 0; k < 4; ++k) xv[k] = k < cin ? __ldg(x + (size_t)row * cin + k) : 0.f;
            }
        } else {
#pragma unroll
            for (int k = 0; k < 4; ++k) { d4[k] = make_float4(0.f, 0.f, 0.f, 0.f); xv[k] = 0.f; }
        }
    };
    fetch(r);
    // every lane of a warp runs the same number of passes (the dx reduction below shuffles across the row's lanes)
    const long long r_warp = ((long long)blockIdx.x * 8 + w) * RPW;
    for (long long rw = r_warp; rw < rows; rw += stride, r += stride) {
        const float d[16] = {d4[0].x, d4[0].y, d4[0].z, d4[0].w, d4[1].x, d4[1].y, d4[1].z, d4[1].w,
                             d4[2].x, d4[2].y, d4[2].z, d4[2].w, d4[3].x, d4[3].y, d4[3].z, d4[3].w};
        const float xc[4] = {xv[0], xv[1], xv[2], xv[3]};
        fetch(r + stride);   // next pass in flight while this one is consumed
        float sx[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int o = 0; o < 16; ++o) {
            accb[o] += d[o];
#pragma unroll
            for (int k = 0; k < 4; ++k) acc[o][k] = fmaf(d[o], xc[k], acc[o][k]);
            if (dx) {
                const float4 wv = s_w[q * 16 + o];
                sx[0] = fmaf(d[o], wv.x, sx[0]); sx[1] = fmaf(d[o], wv.y, sx[1]);
                sx[2] = fmaf(d[o], wv.z, sx[2]); sx[3] = fmaf(d[o], wv.w, sx[3]);
            }
        }
        if (dx) {
            float tot[4] = {0.f, 0.f, 0.f, 0.f};
            const int row_lane0 = (active ? rr : 0) * LPR;
#pragma unroll
            for (int m = 0; m < LPR; ++m) {
#pragma unroll
                for (int k = 0; k < 4; ++k) tot[k] += __shfl_sync(0xffffffffu, sx[k], row_lane0 + m);
            }
            if (active && q == 0 && r < rows) {
                if (cin == 4) {
                    *reinterpret_cast<float4*>(dx + (size_t)r * 4) = make_float4(tot[0], tot[1], tot[2], tot[3]);
                } else {
                    for (int k = 0; k < cin; ++k) dx[(size_t)r * cin + k] = tot[k];
                }
            }
        }
    }
    // rows of the warp -> its first row's lanes (a shuffle tree over the row index; idle lanes hold zeros), then the CTA's
    // 8 warps -> shared -> one global atomic per entry and CTA
#pragma unroll
    for (int o = 0; o < 16; ++o) {
#pragma unroll
        for (int m = 1; m < RPW; m <<= 1) {
            const bool take = lane + m * LPR < 32;
            const float t = __shfl_down_sync(0xffffffffu, accb[o], m * LPR);
            accb[o] += take ? t : 0.f;
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const float u = __shfl_down_sync(0xffffffffu, acc[o][k], m * LPR);
                acc[o][k] += take ? u : 0.f;
            }
        }
        if (rr == 0) {
            if constexpr (DET) {   // every warp's sums straight into the fixed-point slots [COUT][cin] | [COUT]
                unsigned long long* fx = reinterpret_cast<unsigned long long*>(dW);
#pragma unroll
                for (int k = 0; k < 4; ++k)
                    if (k < cin) fx_atomic(fx + ((size_t)(q * 16 + o) * cin + k) * kFxWords, (double)acc[o][k]);
                if (db) fx_atomic(reinterpret_cast<unsigned long long*>(db) + (size_t)(q * 16 + o) * kFxWords, (double)accb[o]);
            } else {
#pragma unroll
                for (int k = 0; k < 4; ++k) atomicAdd(&s_acc[q * 16 + o][k], acc[o][k]);
                atomicAdd(&s_acc[q * 16 + o][4], accb[o]);
            }
        }
    }
    if constexpr (DET) return;
    __syncthreads();
    for (int i = threadIdx.x; i < COUT * 5; i += blockDim.x) {
        const int o = i / 5, k = i - o * 5;
        const float v = s_acc[o][k];
        if (v == 0.f) continue;
        if (k < 4) { if (k < cin) atomicAdd(dW + (size_t)o * dw_ld + k, v); }
        else if (db) atomicAdd(db + o, v);
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// GroupNorm(8 groups) + activation, backward.   y = act(xh * gamma + beta), xh = (x - mean) * rstd   (per sample, group)
//   g   = dy * act'(.)                                 dgamma[c] += sum g * xh,   dbeta[c] += sum g
//   dxh = g * gamma                                    dslope    += sum_{t<0} dy * t   (t = xh*gamma+beta; PReLU only)
//   dx  = rstd * (dxh - mean_g(dxh) - xh * mean_g(dxh * xh))
// pass 1 (k_gn_bwd_reduce) accumulates the per-(sample, group) sums and the parameter gradients in double; pass 2
// (k_gn_bwd_apply) writes dx.  A thread keeps one channel (blockDim = C * rows-per-pass), so its group is fixed.
// ---------------------------------------------------------------------------------------------------------------------
struct GnBwdParams {
    const float* x;
    const float* dy;
    const double* stats;   // [B,8,2] raw sums of x
    const float* gamma;
    const float* beta;
    double count;
    int act;
    float slope;
    long long rows;        // rows per sample
    int B, C;
    double* gsum;          // [B,8,2]: sum dxh, sum dxh*xh
    double* dgamma;        // [C]
    double* dbeta;         // [C]
    double* dslope;        // [1] or null
    float* dx;
    const float* slope_dev;   // device copy of the slope (PReLU weight) or null
    const uint8_t* arg;       // null: dy is [B,rows,C].  Else the activation was followed by a max over each point's 32 consecutive rows:
                              // dy is [B,rows/32,C] and reaches only row (32*point + arg[point,c]) of column c
};

__device__ __forceinline__ void gn_mean_rstd(const double* st, double count, float& mean, float& rstd) {
    const double m = st[0] / count;
    double var = st[1] / count - m * m;
    var = var < 0.0 ? 0.0 : var;
    mean = (float)m;
    rstd = (float)rsqrt(var + 1e-5);
}

// DET: a CTA's fixed-point slots -> the workspace [B*16 gsum | C dgamma | C dbeta | 1 dslope] (p.gsum points at it)
__device__ __forceinline__ void gn_bwd_flush_fx(const GnBwdParams& p, const unsigned long long* s_fx, int b) {
    unsigned long long* ws = reinterpret_cast<unsigned long long*>(p.gsum);
    for (int i = threadIdx.x; i < 16 + 2 * p.C + 1; i += blockDim.x) {
        const Fx v{s_fx[i * kFxWords], s_fx[i * kFxWords + 1], (unsigned)s_fx[i * kFxWords + 2]};
        if (!v.lo && !v.hi && !v.bad) continue;
        fx_atomic(ws + (size_t)(i < 16 ? b * 16 + i : p.B * 16 + (i - 16)) * kFxWords, v);
    }
}

template <bool DET>
__global__ void __launch_bounds__(256) k_gn_bwd_reduce(const GnBwdParams pp) {
    GnBwdParams p = pp;
    if (p.slope_dev) p.slope = __ldg(p.slope_dev);
    __shared__ double s_g[8][2];
    __shared__ double s_par[3];   // unused slots keep the layout simple
    __shared__ double s_ch[2][256];   // dgamma | dbeta of this CTA: ONE global atomic per channel and CTA
    unsigned long long* s_fx = nullptr;   // DET: [16 gsum | C dgamma | C dbeta | dslope] fixed-point slots of this CTA
    if constexpr (DET) { __shared__ unsigned long long s_fx_[(16 + 2 * 256 + 1) * kFxWords]; s_fx = s_fx_; }
    const int b = blockIdx.y;
    const int C = p.C, gsz = C / PVRAFT_GN_GROUPS;
    const int rpp = blockDim.x / C;   // rows per pass
    const int c = threadIdx.x % C, rl = threadIdx.x / C;
    const bool live = rl < rpp;
    if (threadIdx.x < 16) (&s_g[0][0])[threadIdx.x] = 0.0;
    if (threadIdx.x < 3) s_par[threadIdx.x] = 0.0;
    s_ch[0][threadIdx.x] = 0.0;
    s_ch[1][threadIdx.x] = 0.0;
    if constexpr (DET)
        for (int i = threadIdx.x; i < (16 + 2 * C + 1) * kFxWords; i += blockDim.x) s_fx[i] = 0ull;
    __syncthreads();
    const int g = c / gsz;
    float mean, rstd;
    gn_mean_rstd(p.stats + ((size_t)b * 8 + g) * 2, p.count, mean, rstd);
    const float ga = __ldg(p.gamma + c), be = __ldg(p.beta + c);
    double a0 = 0.0, a1 = 0.0, dg = 0.0, dbt = 0.0, dsl = 0.0;
    float f0 = 0.f, f1 = 0.f, fg = 0.f, fb = 0.f, fs = 0.f;
    int pend = 0;
    if (live) {
        const long long base = (long long)b * p.rows;
        for (long long r = (long long)blockIdx.x * rpp + rl; r < p.rows; r += (long long)gridDim.x * rpp) {
            const size_t at = (size_t)(base + r) * C + c;
            const float xh = (__ldg(p.x + at) - mean) * rstd;
            const float t = fmaf(xh, ga, be);
            const float d = __ldg(p.dy + at);
            float gq = d;
            if (p.act == PVRAFT_ACT_RELU) gq = t > 0.f ? d : 0.f;
            else if (p.act == PVRAFT_ACT_LRELU) { gq = t >= 0.f ? d : d * p.slope; if (t < 0.f) fs += d * t; }
            const float dxh = gq * ga;
            f0 += dxh; f1 += dxh * xh; fg += gq * xh; fb += gq;
            if (++pend == 32) { a0 += f0; a1 += f1; dg += fg; dbt += fb; dsl += fs; f0 = f1 = fg = fb = fs = 0.f; pend = 0; }
        }
        a0 += f0; a1 += f1; dg += fg; dbt += fb; dsl += fs;
        if constexpr (DET) {
            fx_atomic(s_fx + (g * 2) * kFxWords, a0);
            fx_atomic(s_fx + (g * 2 + 1) * kFxWords, a1);
            fx_atomic(s_fx + (16 + c) * kFxWords, dg);
            fx_atomic(s_fx + (16 + C + c) * kFxWords, dbt);
            if (p.dslope && dsl != 0.0) fx_atomic(s_fx + (16 + 2 * C) * kFxWords, dsl);
        } else {
        atomicAdd(&s_g[g][0], a0);
        atomicAdd(&s_g[g][1], a1);
        atomicAdd(&s_ch[0][c], dg);
        atomicAdd(&s_ch[1][c], dbt);
        if (p.dslope && dsl != 0.0) atomicAdd(&s_par[0], dsl);
        }
    }
    __syncthreads();
    if constexpr (DET) {
        gn_bwd_flush_fx(p, s_fx, b);
        return;
    }
    if (threadIdx.x < 16) {
        const double v = (&s_g[0][0])[threadIdx.x];
        if (v != 0.0) atomicAdd(p.gsum + (size_t)b * 16 + threadIdx.x, v);
    }
    if (threadIdx.x < C) {
        if (s_ch[0][threadIdx.x] != 0.0) atomicAdd(p.dgamma + threadIdx.x, s_ch[0][threadIdx.x]);
        if (s_ch[1][threadIdx.x] != 0.0) atomicAdd(p.dbeta + threadIdx.x, s_ch[1][threadIdx.x]);
    }
    if (threadIdx.x == 0 && p.dslope && s_par[0] != 0.0) atomicAdd(p.dslope, s_par[0]);
}

__global__ void __launch_bounds__(256) k_gn_bwd_apply(const GnBwdParams pp) {
    GnBwdParams p = pp;
    if (p.slope_dev) p.slope = __ldg(p.slope_dev);
    const int b = blockIdx.y;
    const int C = p.C, gsz = C / PVRAFT_GN_GROUPS;
    const int rpp = blockDim.x / C;
    const int c = threadIdx.x % C, rl = threadIdx.x / C;
    if (rl >= rpp) return;
    const int g = c / gsz;
    float mean, rstd;
    gn_mean_rstd(p.stats + ((size_t)b * 8 + g) * 2, p.count, mean, rstd);
    const float ga = __ldg(p.gamma + c), be = __ldg(p.beta + c);
    const float m0 = (float)(p.gsum[((size_t)b * 8 + g) * 2] / p.count), m1 = (float)(p.gsum[((size_t)b * 8 + g) * 2 + 1] / p.count);
    const long long base = (long long)b * p.rows;
    for (long long r = (long long)blockIdx.x * rpp + rl; r < p.rows; r += (long long)gridDim.x * rpp) {
        const size_t at = (size_t)(base + r) * C + c;
        const float xh = (__ldg(p.x + at) - mean) * rstd;
        const float t = fmaf(xh, ga, be);
        const float d = __ldg(p.dy + at);
        float gq = d;
        if (p.act == PVRAFT_ACT_RELU) gq = t > 0.f ? d : 0.f;
        else if (p.act == PVRAFT_ACT_LRELU) gq = t >= 0.f ? d : d * p.slope;
        p.dx[at] = rstd * (gq * ga - m0 - xh * m1);
    }
}

// The same two passes when the activation was followed by a max over each point's 32 consecutive rows (GnActMaxFn): only the
// arg-max row of a (point, channel) carries gradient, so pass 1 gathers ONE x per (point, channel) -- 1/32 of the tensor -- and
// pass 2 streams x -> dx in 16-byte pieces with the point's (arg, dy) held in registers across its 32 rows.
template <bool DET>
__global__ void __launch_bounds__(256) k_gn_bwd_reduce_arg(const GnBwdParams pp) {
    GnBwdParams p = pp;
    if (p.slope_dev) p.slope = __ldg(p.slope_dev);
    __shared__ double s_g[8][2];
    __shared__ double s_par;
    __shared__ double s_ch[2][256];
    unsigned long long* s_fx = nullptr;   // DET: as in k_gn_bwd_reduce
    if constexpr (DET) { __shared__ unsigned long long s_fx_[(16 + 2 * 256 + 1) * kFxWords]; s_fx = s_fx_; }
    const int b = blockIdx.y;
    const int C = p.C, gsz = C / PVRAFT_GN_GROUPS;
    const int ppp = blockDim.x / C;   // points per pass
    const int c = threadIdx.x % C, rl = threadIdx.x / C;
    if (threadIdx.x < 16) (&s_g[0][0])[threadIdx.x] = 0.0;
    if (threadIdx.x == 0) s_par = 0.0;
    s_ch[0][threadIdx.x] = 0.0;
    s_ch[1][threadIdx.x] = 0.0;
    if constexpr (DET)
        for (int i = threadIdx.x; i < (16 + 2 * C + 1) * kFxWords; i += blockDim.x) s_fx[i] = 0ull;
    __syncthreads();
    const int g = c / gsz;
    float mean, rstd;
    gn_mean_rstd(p.stats + ((size_t)b * 8 + g) * 2, p.count, mean, rstd);
    const float ga = __ldg(p.gamma + c), be = __ldg(p.beta + c);
    if (rl < ppp) {
        double a0 = 0.0, a1 = 0.0, dg = 0.0, dbt = 0.0, dsl = 0.0;
        float f0 = 0.f, f1 = 0.f, fg = 0.f, fb = 0.f, fs = 0.f;
        int pend = 0;
        const long long pts = p.rows >> 5, pbase = (long long)b * pts;
        for (long long pt = (long long)blockIdx.x * ppp + rl; pt < pts; pt += (long long)gridDim.x * ppp) {
            const size_t pc = (size_t)(pbase + pt) * C + c;
            const int a = __ldg(p.arg + pc);
            const float d = __ldg(p.dy + pc);
            const float xh = (__ldg(p.x + ((size_t)(pbase + pt) * PVRAFT_KNN + a) * C + c) - mean) * rstd;
            const float t = fmaf(xh, ga, be);
            float gq = d;
            if (p.act == PVRAFT_ACT_RELU) gq = t > 0.f ? d : 0.f;
            else if (p.act == PVRAFT_ACT_LRELU) { gq = t >= 0.f ? d : d * p.slope; if (t < 0.f) fs += d * t; }
            const float dxh = gq * ga;
            f0 += dxh; f1 += dxh * xh; fg += gq * xh; fb += gq;
            if (++pend == 32) { a0 += f0; a1 += f1; dg += fg; dbt += fb; dsl += fs; f0 = f1 = fg = fb = fs = 0.f; pend = 0; }
        }
        a0 += f0; a1 += f1; dg += fg; dbt += fb; dsl += fs;
        if constexpr (DET) {
            fx_atomic(s_fx + (g * 2) * kFxWords, a0);
            fx_atomic(s_fx + (g * 2 + 1) * kFxWords, a1);
            fx_atomic(s_fx + (16 + c) * kFxWords, dg);
            fx_atomic(s_fx + (16 + C + c) * kFxWords, dbt);
            if (p.dslope && dsl != 0.0) fx_atomic(s_fx + (16 + 2 * C) * kFxWords, dsl);
        } else {
        atomicAdd(&s_g[g][0], a0);
        atomicAdd(&s_g[g][1], a1);
        atomicAdd(&s_ch[0][c], dg);
        atomicAdd(&s_ch[1][c], dbt);
        if (p.dslope && dsl != 0.0) atomicAdd(&s_par, dsl);
        }
    }
    __syncthreads();
    if constexpr (DET) {
        gn_bwd_flush_fx(p, s_fx, b);
        return;
    }
    if (threadIdx.x < 16) {
        const double v = (&s_g[0][0])[threadIdx.x];
        if (v != 0.0) atomicAdd(p.gsum + (size_t)b * 16 + threadIdx.x, v);
    }
    if (threadIdx.x < C) {
        if (s_ch[0][threadIdx.x] != 0.0) atomicAdd(p.dgamma + threadIdx.x, s_ch[0][threadIdx.x]);
        if (s_ch[1][threadIdx.x] != 0.0) atomicAdd(p.dbeta + threadIdx.x, s_ch[1][threadIdx.x]);
    }
    if (threadIdx.x == 0 && p.dslope && s_par != 0.0) atomicAdd(p.dslope, s_par);
}

__global__ void __launch_bounds__(256) k_gn_bwd_apply_arg(const GnBwdParams pp) {
    GnBwdParams p = pp;
    if (p.slope_dev) p.slope = __ldg(p.slope_dev);
    const int b = blockIdx.y;
    const int C = p.C, C4 = C >> 2, gsz = C / PVRAFT_GN_GROUPS;
    const int ppp = blockDim.x / C4;
    const int c4 = threadIdx.x % C4, rl = threadIdx.x / C4;
    if (rl >= ppp) return;
    float mean[4], rstd[4], ga[4], be[4], m0[4], m1[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        const int c = c4 * 4 + q, g = c / gsz;
        gn_mean_rstd(p.stats + ((size_t)b * 8 + g) * 2, p.count, mean[q], rstd[q]);
        ga[q] = __ldg(p.gamma + c);
        be[q] = __ldg(p.beta + c);
        m0[q] = (float)(p.gsum[((size_t)b * 8 + g) * 2] / p.count);
        m1[q] = (float)(p.gsum[((size_t)b * 8 + g) * 2 + 1] / p.count);
    }
    const long long pts = p.rows >> 5, pbase = (long long)b * pts;
    for (long long pt = (long long)blockIdx.x * ppp + rl; pt < pts; pt += (long long)gridDim.x * ppp) {
        const size_t pc = (size_t)(pbase + pt) * C + c4 * 4;
        const uchar4 a4 = __ldg(reinterpret_cast<const uchar4*>(p.arg + pc));
        const float4 d4 = __ldg(reinterpret_cast<const float4*>(p.dy + pc));
        const int a[4] = {a4.x, a4.y, a4.z, a4.w};
        const float d[4] = {d4.x, d4.y, d4.z, d4.w};
        const float4* xp = reinterpret_cast<const float4*>(p.x + (size_t)(pbase + pt) * PVRAFT_KNN * C) + c4;
        float4* op = reinterpret_cast<float4*>(p.dx + (size_t)(pbase + pt) * PVRAFT_KNN * C) + c4;
#pragma unroll 8
        for (int j = 0; j < PVRAFT_KNN; ++j) {
            const float4 x4 = __ldg(xp + (size_t)j * C4);
            const float xv[4] = {x4.x, x4.y, x4.z, x4.w};
            float o[4];
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const float xh = (xv[q] - mean[q]) * rstd[q];
                const float t = fmaf(xh, ga[q], be[q]);
                const float dd = a[q] == j ? d[q] : 0.f;
                float gq = dd;
                if (p.act == PVRAFT_ACT_RELU) gq = t > 0.f ? dd : 0.f;
                else if (p.act == PVRAFT_ACT_LRELU) gq = t >= 0.f ? dd : dd * p.slope;
                o[q] = rstd[q] * (gq * ga[q] - m0[q] - xh * m1[q]);
            }
            op[(size_t)j * C4] = make_float4(o[0], o[1], o[2], o[3]);
        }
    }
}

// GroupNorm + activation + max over each point's 32 consecutive rows in one pass (model/flot/gconv.py:76-80, model/corr.py:87-92):
// the normalised [B,N*32,C] tensor is never written.  One thread per (point, channel); arg = first row attaining the maximum.
__global__ void __launch_bounds__(256) k_gn_act_maxk(const float* __restrict__ x, const double* __restrict__ stats, const float* __restrict__ gamma,
                                                     const float* __restrict__ beta, double count, int act, float slope, int B, long long pts_per_sample,
                                                     int C, float* __restrict__ y, uint8_t* __restrict__ arg, const float* __restrict__ slope_dev) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)B * pts_per_sample * C) return;
    if (slope_dev) slope = __ldg(slope_dev);
    const long long pt = i / C;
    const int c = (int)(i - pt * C), b = (int)(pt / pts_per_sample);
    float mean, rstd;
    gn_mean_rstd(stats + ((size_t)b * 8 + c / (C / PVRAFT_GN_GROUPS)) * 2, count, mean, rstd);
    const float sc = rstd * __ldg(gamma + c), sh = __ldg(beta + c) - mean * rstd * __ldg(gamma + c);
    const float* xp = x + (size_t)pt * PVRAFT_KNN * C + c;
    float m = -INFINITY;
    int a = 0;
#pragma unroll 8
    for (int j = 0; j < PVRAFT_KNN; ++j) {
        float t = fmaf(__ldg(xp + (size_t)j * C), sc, sh);
        if (act == PVRAFT_ACT_RELU) t = fmaxf(t, 0.f);
        else if (act == PVRAFT_ACT_LRELU) t = t >= 0.f ? t : slope * t;
        if (t > m) { m = t; a = j; }
    }
    y[i] = m;
    arg[i] = (uint8_t)a;
}

// ---------------------------------------------------------------------------------------------------------------------
// SetConv edge stage, layer-wise (model/flot/gconv.py:65-73 with fc1 factorised: W [x_j - x_i, e] = P_j - P_i + W_e e):
//   forward   T[b,n,j,:] = P[b,nbr[b,n,j],:] - P[b,n,:] + E[b,n,j,:]   in place on E, GroupNorm sums of T accumulated
//   backward  dP[b,nbr,:] += dT[b,n,j,:],  dP[b,n,:] -= sum_j dT[b,n,j,:]   (dE = dT)
// One warp per point; lanes stride over the channels.
// ---------------------------------------------------------------------------------------------------------------------
template <bool DET>
__global__ void __launch_bounds__(256) k_edge_fwd(const float* __restrict__ P, const int32_t* __restrict__ nbr, float* __restrict__ E,
                                                  int B, int N, int C, double* __restrict__ stats) {
    __shared__ double s_g[16];
    const int lane = lane_id(), w = warp_id();
    const long long pt = (long long)blockIdx.x * 8 + w;
    const int b0 = (int)(((long long)blockIdx.x * 8) / N);   // a CTA's 8 points may straddle two samples
    unsigned long long* s_fx = nullptr;   // DET: fixed-point [16] of the CTA's first sample; `stats` is the [B,16] workspace
    if constexpr (DET) { __shared__ unsigned long long s_fx_[16 * kFxWords]; s_fx = s_fx_; }
    if (threadIdx.x < 16) s_g[threadIdx.x] = 0.0;
    if constexpr (DET)
        if (threadIdx.x < 16 * kFxWords) s_fx[threadIdx.x] = 0ull;
    __syncthreads();
    const int gsz = C / PVRAFT_GN_GROUPS;
    if (pt < (long long)B * N) {
        const int b = (int)(pt / N);
        const float* Pb = P + (size_t)b * N * C;
        const float* pc = P + (size_t)pt * C;
        for (int c = lane; c < C; c += 32) {
            const float ctr = __ldg(pc + c);
            float s = 0.f, ss = 0.f;
            for (int j = 0; j < PVRAFT_KNN; ++j) {
                const int nb = __ldg(nbr + pt * PVRAFT_KNN + j);
                float* e = E + ((size_t)pt * PVRAFT_KNN + j) * C + c;
                const float t = (__ldg(Pb + (size_t)nb * C + c) - ctr) + *e;
                *e = t;
                s += t;
                ss += t * t;
            }
            if (DET && stats) {   // one (point, channel) sum of 32 neighbours per contribution
                unsigned long long* gfx = reinterpret_cast<unsigned long long*>(stats) + (size_t)b * 16 * kFxWords;
                unsigned long long* dst = b == b0 ? s_fx : gfx;
                fx_atomic(dst + ((c / gsz) * 2) * kFxWords, (double)s);
                fx_atomic(dst + ((c / gsz) * 2 + 1) * kFxWords, (double)ss);
            } else if (stats) {
                if (b == b0) {
                    atomicAdd(&s_g[(c / gsz) * 2], (double)s);
                    atomicAdd(&s_g[(c / gsz) * 2 + 1], (double)ss);
                } else {
                    atomicAdd(stats + (size_t)b * 16 + (c / gsz) * 2, (double)s);
                    atomicAdd(stats + (size_t)b * 16 + (c / gsz) * 2 + 1, (double)ss);
                }
            }
        }
    }
    __syncthreads();
    if constexpr (DET) {
        if (stats && threadIdx.x < 16) {
            const Fx v{s_fx[threadIdx.x * kFxWords], s_fx[threadIdx.x * kFxWords + 1], (unsigned)s_fx[threadIdx.x * kFxWords + 2]};
            fx_atomic(reinterpret_cast<unsigned long long*>(stats) + ((size_t)b0 * 16 + threadIdx.x) * kFxWords, v);
        }
        return;
    }
    if (stats && threadIdx.x < 16 && s_g[threadIdx.x] != 0.0) atomicAdd(stats + (size_t)b0 * 16 + threadIdx.x, s_g[threadIdx.x]);
}

template <bool DET>
__global__ void __launch_bounds__(256) k_edge_bwd(const float* __restrict__ dT, const int32_t* __restrict__ nbr, int B, int N, int C,
                                                  float* __restrict__ dP) {
    const int lane = lane_id(), w = warp_id();
    const long long pt = (long long)blockIdx.x * 8 + w;
    if (pt >= (long long)B * N) return;
    const int b = (int)(pt / N);
    float* dPb = dP + (size_t)b * N * C;
    for (int c = lane; c < C; c += 32) {
        float s = 0.f;
        for (int j = 0; j < PVRAFT_KNN; ++j) {
            const int nb = __ldg(nbr + pt * PVRAFT_KNN + j);
            const float g = __ldg(dT + ((size_t)pt * PVRAFT_KNN + j) * C + c);
            s += g;
            if constexpr (DET) fx_atomic(reinterpret_cast<unsigned long long*>(dP) + ((size_t)b * N * C + (size_t)nb * C + c) * kFxWords, (double)g);
            else atomicAdd(dPb + (size_t)nb * C + c, g);
        }
        if constexpr (DET) fx_atomic(reinterpret_cast<unsigned long long*>(dP) + ((size_t)pt * C + c) * kFxWords, -(double)s);
        else atomicAdd(dP + (size_t)pt * C + c, -s);
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// max over the 32 neighbours (gconv.py:80, corr.py:92): y[b,n,c] = max_j x[b,n,j,c], arg = first j attaining it.
// ---------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_maxk_fwd(const float* __restrict__ x, long long pts, int C, float* __restrict__ y,
                                                  uint8_t* __restrict__ arg) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= pts * C) return;
    const long long pt = i / C;
    const int c = (int)(i - pt * C);
    const float* xp = x + (size_t)pt * PVRAFT_KNN * C + c;
    float m = __ldg(xp);
    int a = 0;
    for (int j = 1; j < PVRAFT_KNN; ++j) {
        const float v = __ldg(xp + (size_t)j * C);
        if (v > m) { m = v; a = j; }
    }
    y[i] = m;
    arg[i] = (uint8_t)a;
}

__global__ void __launch_bounds__(256) k_maxk_bwd(const float* __restrict__ dy, const uint8_t* __restrict__ arg, long long pts, int C,
                                                  float* __restrict__ dx) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;   // over pts * 32 * C
    if (i >= pts * PVRAFT_KNN * C) return;
    const long long pt = i / ((long long)PVRAFT_KNN * C);
    const int rem = (int)(i - pt * PVRAFT_KNN * C);
    const int j = rem / C, c = rem - j * C;
    dx[i] = arg[pt * C + c] == j ? __ldg(dy + pt * C + c) : 0.f;
}

// ---------------------------------------------------------------------------------------------------------------------
// Correlation lookup, backward w.r.t. the truncated correlation values (model/corr.py:47-66 and :84; the index math is
// under no_grad in the reference, corr.py:52-62, and the query coordinates are detached, RAFTSceneFlow.py:41):
//   d corr[b,n,k] = sum_levels valid_l(k) * g_vox[b,n,l*27+cell_l(k)] / clamp(count_l[cell], 1, N)  +  [k selected as j-th nn] g_sel[b,n,j,0]
// (N = query points; the table holds the M points of the second cloud)
// One warp per point; cells are re-derived with the forward's arithmetic (cell edge by true division or exact reciprocal).
// ---------------------------------------------------------------------------------------------------------------------
struct LookupBwdParams {
    const int32_t* corr_idx;
    const float4* tab;         // [B,M]
    const float* coords;
    const int32_t* knn_slot;   // [B,N,32]
    const float* g_vox;        // [B,N,vox_ld]
    const float* g_sel;        // [B,N,32,4]
    float* d_corr;             // [B,N,K]
    int B, N, K, levels, vox_ld;
    float r[4], inv_r[4];
    int pow2;
    int M;
};

__global__ void __launch_bounds__(256) k_lookup_bwd(const LookupBwdParams p) {
    __shared__ int s_cnt[8][4 * 27];
    __shared__ float s_g[8][4 * 27];
    const int lane = lane_id(), w = warp_id();
    const long long pt = (long long)blockIdx.x * 8 + w;
    if (pt >= (long long)p.B * p.N) return;
    const int b = (int)(pt / p.N);
    const int L = p.levels, nvox = L * 27;
    for (int i = lane; i < 4 * 27; i += 32) {
        s_cnt[w][i] = 0;
        s_g[w][i] = i < nvox ? __ldg(p.g_vox + pt * p.vox_ld + i) : 0.f;
    }
    __syncwarp();
    const float cx = __ldg(p.coords + pt * 3), cy = __ldg(p.coords + pt * 3 + 1), cz = __ldg(p.coords + pt * 3 + 2);
    const float4* tab = p.tab + (size_t)b * p.M;
    const int32_t* ri = p.corr_idx + pt * p.K;
    float* dr = p.d_corr + pt * p.K;
    // pass 1: counts per (level, cell)
    for (int k = lane; k < p.K; k += 32) {
        const float4 q = __ldg(tab + __ldg(ri + k));
        const float dx = __fsub_rn(q.x, cx), dy = __fsub_rn(q.y, cy), dz = __fsub_rn(q.z, cz);
        for (int l = 0; l < L; ++l) {
            const float qx = rintf(p.pow2 ? __fmul_rn(dx, p.inv_r[l]) : __fdiv_rn(dx, p.r[l]));
            const float qy = rintf(p.pow2 ? __fmul_rn(dy, p.inv_r[l]) : __fdiv_rn(dy, p.r[l]));
            const float qz = rintf(p.pow2 ? __fmul_rn(dz, p.inv_r[l]) : __fdiv_rn(dz, p.r[l]));
            if (fmaxf(fmaxf(fabsf(qx), fabsf(qy)), fabsf(qz)) <= 1.f) atomicAdd(&s_cnt[w][l * 27 + (int)fmaf(qx, 9.f, fmaf(qy, 3.f, qz + 13.f))], 1);
        }
    }
    __syncwarp();
    // pass 2: the gradient of every candidate's correlation through the means
    for (int k = lane; k < p.K; k += 32) {
        const float4 q = __ldg(tab + __ldg(ri + k));
        const float dx = __fsub_rn(q.x, cx), dy = __fsub_rn(q.y, cy), dz = __fsub_rn(q.z, cz);
        float g = 0.f;
        for (int l = 0; l < L; ++l) {
            const float qx = rintf(p.pow2 ? __fmul_rn(dx, p.inv_r[l]) : __fdiv_rn(dx, p.r[l]));
            const float qy = rintf(p.pow2 ? __fmul_rn(dy, p.inv_r[l]) : __fdiv_rn(dy, p.r[l]));
            const float qz = rintf(p.pow2 ? __fmul_rn(dz, p.inv_r[l]) : __fdiv_rn(dz, p.r[l]));
            if (fmaxf(fmaxf(fabsf(qx), fabsf(qy)), fabsf(qz)) <= 1.f) {
                const int cell = l * 27 + (int)fmaf(qx, 9.f, fmaf(qy, 3.f, qz + 13.f));
                g += s_g[w][cell] / (float)min(s_cnt[w][cell], p.N);
            }
        }
        dr[k] = g;
    }
    __syncwarp();
    __threadfence_block();
    // the 32 selected neighbours (distinct slots): + d/d(corr channel of the kNN 4-vector)
    const int slot = __ldg(p.knn_slot + pt * PVRAFT_KNN + lane);
    dr[slot] += __ldg(p.g_sel + (pt * PVRAFT_KNN + lane) * 4);
}

// ---------------------------------------------------------------------------------------------------------------------
// Truncated correlation, backward (model/corr.py:95-100 then the top-k gather of :37-38), sparse: only the K kept entries
// of a row carry gradient, so the dense N x M gradient of the reference is never formed (f2, d_f2: M rows per sample):
//   d f1[b,n,:] = (1/sqrt(C)) sum_k g[b,n,k] f2[b,idx[b,n,k],:]      d f2[b,m,:] += (1/sqrt(C)) g[b,n,k] f1[b,n,:]  (m = idx[b,n,k])
// One warp per row; lanes own C/32 (<= 8) consecutive channels.
// ---------------------------------------------------------------------------------------------------------------------
template <int CPL, bool DET>
__global__ void __launch_bounds__(256) k_corr_init_bwd(const float* __restrict__ g, const int32_t* __restrict__ idx, const float* __restrict__ f1,
                                                       const float* __restrict__ f2, int B, int N, int M, int K, float scale,
                                                       float* __restrict__ d_f1, float* __restrict__ d_f2) {
    constexpr int C = CPL * 32;
    const int lane = lane_id(), w = warp_id();
    const long long row = (long long)blockIdx.x * 8 + w;
    if (row >= (long long)B * N) return;
    const int b = (int)(row / N);
    const float* f2b = f2 + (size_t)b * M * C;
    float* d2b = d_f2 + (size_t)b * M * C;
    float a[CPL], acc[CPL];
#pragma unroll
    for (int i = 0; i < CPL; ++i) { a[i] = __ldg(f1 + row * C + lane * CPL + i) * scale; acc[i] = 0.f; }
    for (int k0 = 0; k0 < K; k0 += 32) {
        const float gk = k0 + lane < K ? __ldg(g + row * K + k0 + lane) : 0.f;
        const int ik = k0 + lane < K ? __ldg(idx + row * K + k0 + lane) : 0;
        const int n = min(32, K - k0);
        for (int j = 0; j < n; ++j) {
            const float gj = __shfl_sync(kFull, gk, j);
            const int m = __shfl_sync(kFull, ik, j);
            if (gj == 0.f) continue;
            if constexpr (DET) {   // d_f2 is the fixed-point workspace [B,M,C]
                unsigned long long* fx = reinterpret_cast<unsigned long long*>(d_f2) + ((size_t)b * M + m) * C * kFxWords;
#pragma unroll
                for (int i = 0; i < CPL; ++i) {
                    acc[i] = fmaf(gj, __ldg(f2b + (size_t)m * C + lane * CPL + i), acc[i]);
                    fx_atomic(fx + (size_t)(lane * CPL + i) * kFxWords, (double)(gj * a[i]));
                }
            } else if constexpr (CPL == 4) {   // the model's C = 128: one 128-bit load and one vector reduction per lane
                const float4 v = __ldg(reinterpret_cast<const float4*>(f2b + (size_t)m * C) + lane);
                acc[0] = fmaf(gj, v.x, acc[0]); acc[1] = fmaf(gj, v.y, acc[1]); acc[2] = fmaf(gj, v.z, acc[2]); acc[3] = fmaf(gj, v.w, acc[3]);
                atomicAdd(reinterpret_cast<float4*>(d2b + (size_t)m * C) + lane, make_float4(gj * a[0], gj * a[1], gj * a[2], gj * a[3]));
            } else {
#pragma unroll
                for (int i = 0; i < CPL; ++i) {
                    acc[i] = fmaf(gj, __ldg(f2b + (size_t)m * C + lane * CPL + i), acc[i]);
                    atomicAdd(d2b + (size_t)m * C + lane * CPL + i, gj * a[i]);
                }
            }
        }
    }
#pragma unroll
    for (int i = 0; i < CPL; ++i) d_f1[row * C + lane * CPL + i] = acc[i] * scale;
}

}  // namespace pvraft

using namespace pvraft;

template <bool DET>
static int linear_wgrad(const float* x, const float* dy, int64_t rows, int cin, int cout, float* dW, int dw_ld, float* db, void* ws,
                        void* stream) {
    if (!x || !dy || !dW || rows <= 0 || cin <= 0 || cout <= 0) return fail(PVRAFT_ERR_BAD_ARG, "linear_wgrad: bad argument");
    if (cin > 256 || cout > 128) return fail(PVRAFT_ERR_UNSUPPORTED, "linear_wgrad: cin=%d cout=%d (max 256/128)", cin, cout);
    const int cin_p = (cin + 3) & ~3;
    if (8 * (cin_p >> 2) > 2 * kWgThreads) return fail(PVRAFT_ERR_UNSUPPORTED, "linear_wgrad: cin=%d", cin);
    const size_t smem = sizeof(float) * ((size_t)kWgRows * (cin_p + 4) + (size_t)kWgRows * 36);
    int rc;
    if ((rc = opt_in_smem(k_linear_wgrad<DET>, smem))) return rc;
    long long workers = (rows + kWgRows - 1) / kWgRows;
    const long long cap = DET ? kDetCtas : (long long)sm_count() * 2;
    if (workers > cap) workers = cap;
    dim3 grid((unsigned)workers, (unsigned)((cout + 31) / 32));
    const int ld = dw_ld > 0 ? dw_ld : cin;
    cudaStream_t st = (cudaStream_t)stream;
    if constexpr (DET) {
        unsigned long long* fx = static_cast<unsigned long long*>(ws);
        unsigned long long* fxb = fx + (size_t)cout * cin * kFxWords;
        k_linear_wgrad<true><<<grid, kWgThreads, smem, st>>>(x, dy, rows, cin, cout, reinterpret_cast<float*>(fx), ld,
                                                             db ? reinterpret_cast<float*>(fxb) : nullptr);
        if ((rc = check_launch("linear_wgrad"))) return rc;
        if ((rc = fx_flush_f32(fx, cout, cin, cin, ld, dW, st))) return rc;
        return db ? fx_flush_f32(fxb, 1, cout, cout, cout, db, st) : 0;
    }
    k_linear_wgrad<false><<<grid, kWgThreads, smem, st>>>(x, dy, rows, cin, cout, dW, ld, db);
    return check_launch("linear_wgrad");
}

extern "C" int pvraft_linear_wgrad(const float* x, const float* dy, int64_t rows, int cin, int cout, float* dW, int dw_ld, float* db,
                                   void* det_workspace, void* stream) {
    auto f = det_workspace ? linear_wgrad<true> : linear_wgrad<false>;
    return f(x, dy, rows, cin, cout, dW, dw_ld, db, det_workspace, stream);
}

extern "C" int64_t pvraft_linear_wgrad_det_workspace_bytes(int cin, int cout) {
    return (int64_t)((int64_t)cout * cin + cout) * kFxWords * 8;
}

template <bool DET>
static int linear_bwd_small(const float* x, const float* dy, const float* W, int64_t rows, int cin, int cout, int w_ld, float* dW, int dw_ld,
                            float* db, float* dx, void* ws, void* stream) {
    if (!x || !dy || !W || !dW || rows <= 0) return fail(PVRAFT_ERR_BAD_ARG, "linear_bwd_small: bad argument");
    const int lpr = cout / 16;
    if (cin < 1 || cin > 4 || cout % 16 || !(lpr == 1 || lpr == 2 || lpr == 3 || lpr == 4 || lpr == 6 || lpr == 8))
        return fail(PVRAFT_ERR_UNSUPPORTED, "linear_bwd_small: cin=%d cout=%d (cin <= 4, cout in {16,32,48,64,96,128})", cin, cout);
    if ((reinterpret_cast<uintptr_t>(dy) & 15) || (cin == 4 && ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(dx)) & 15)))
        return fail(PVRAFT_ERR_BAD_ARG, "linear_bwd_small: dy (and x, dx when cin == 4) must be 16-byte aligned");
    const int rpc = 8 * (32 / lpr);
    long long ctas = (rows + rpc - 1) / rpc;
    const long long cap = DET ? kDetCtas / 2 : (long long)sm_count();   // 152 registers x 256 threads: one resident CTA per SM
    if (ctas > cap) ctas = cap;
    const int wl = w_ld > 0 ? w_ld : cin, dl = dw_ld > 0 ? dw_ld : cin;
    cudaStream_t st = (cudaStream_t)stream;
    unsigned long long* fx = static_cast<unsigned long long*>(ws);
    unsigned long long* fxb = DET ? fx + (size_t)cout * cin * kFxWords : nullptr;
    float* kdW = DET ? reinterpret_cast<float*>(fx) : dW;
    float* kdb = DET ? (db ? reinterpret_cast<float*>(fxb) : nullptr) : db;
#define PVRAFT_LBS(L) k_linear_bwd_small<L, DET><<<(unsigned)ctas, 256, 0, st>>>(x, dy, W, rows, cin, wl, kdW, dl, kdb, dx)
    switch (lpr) {
        case 1: PVRAFT_LBS(1); break;
        case 2: PVRAFT_LBS(2); break;
        case 3: PVRAFT_LBS(3); break;
        case 4: PVRAFT_LBS(4); break;
        case 6: PVRAFT_LBS(6); break;
        default: PVRAFT_LBS(8); break;
    }
#undef PVRAFT_LBS
    int rc = check_launch("linear_bwd_small");
    if (rc || !DET) return rc;
    if ((rc = fx_flush_f32(fx, cout, cin, cin, dl, dW, st))) return rc;
    return db ? fx_flush_f32(fxb, 1, cout, cout, cout, db, st) : 0;
}

extern "C" int pvraft_linear_bwd_small(const float* x, const float* dy, const float* W, int64_t rows, int cin, int cout, int w_ld, float* dW,
                                       int dw_ld, float* db, float* dx, void* det_workspace, void* stream) {
    auto f = det_workspace ? linear_bwd_small<true> : linear_bwd_small<false>;
    return f(x, dy, W, rows, cin, cout, w_ld, dW, dw_ld, db, dx, det_workspace, stream);
}

extern "C" int64_t pvraft_linear_bwd_small_det_workspace_bytes(int cin, int cout) {
    return (int64_t)((int64_t)cout * cin + cout) * kFxWords * 8;
}

template <bool DET>
static int gn_act_bwd(const float* x, const float* dy, const double* stats, const float* gamma, const float* beta, double count, int act,
                      float slope, int B, int64_t rows, int C, double* gsum, double* dgamma, double* dbeta, double* dslope, float* dx,
                      const float* slope_dev, const uint8_t* arg, void* ws, void* stream) {
    if (!x || !dy || !stats || !gamma || !beta || !gsum || !dgamma || !dbeta || !dx) return fail(PVRAFT_ERR_BAD_ARG, "gn_act_bwd: null pointer");
    if (C > 256 || C % PVRAFT_GN_GROUPS || B <= 0 || rows <= 0) return fail(PVRAFT_ERR_UNSUPPORTED, "gn_act_bwd: C=%d", C);
    if (arg && rows % PVRAFT_KNN) return fail(PVRAFT_ERR_BAD_ARG, "gn_act_bwd: the max-pooled form needs rows %% 32 == 0");
    GnBwdParams p{x, dy, stats, gamma, beta, count, act, slope, (long long)rows, B, C, gsum, dgamma, dbeta, dslope, dx, slope_dev, arg};
    GnBwdParams pr = p;   // the reducing pass: DET accumulates into the fixed-point workspace, flushed before the apply pass
    if (DET) pr.gsum = static_cast<double*>(ws);
    const long long cap = ((DET ? kDetCtas * 4 : (long long)sm_count() * 8) + B - 1) / B;
    cudaStream_t st = (cudaStream_t)stream;
    auto flush = [&]() -> int {
        if (!DET) return 0;
        const unsigned long long* fx = static_cast<const unsigned long long*>(ws);
        int rc;
        if ((rc = fx_flush_f64(fx, 1, (long long)B * 16, (long long)B * 16, 0, gsum, st))) return rc;
        fx += (size_t)B * 16 * kFxWords;
        if ((rc = fx_flush_f64(fx, 1, C, C, 0, dgamma, st))) return rc;
        if ((rc = fx_flush_f64(fx + (size_t)C * kFxWords, 1, C, C, 0, dbeta, st))) return rc;
        return dslope ? fx_flush_f64(fx + (size_t)2 * C * kFxWords, 1, 1, 1, 0, dslope, st) : 0;
    };
    if (arg) {
        const long long pts = rows / PVRAFT_KNN;
        const int ppp_r = 256 / C, ppp_a = 256 / (C / 4);
        long long wr = (pts + ppp_r * 16 - 1) / (ppp_r * 16), wa = (pts + ppp_a - 1) / ppp_a;   // >= 16 points per reducing thread
        if (wr > cap) wr = cap;
        if (wa > cap) wa = cap;
        k_gn_bwd_reduce_arg<DET><<<dim3((unsigned)wr, (unsigned)B), 256, 0, st>>>(pr);
        int rc = check_launch("gn_bwd_reduce_arg");
        if (rc || (rc = flush())) return rc;
        k_gn_bwd_apply_arg<<<dim3((unsigned)wa, (unsigned)B), 256, 0, st>>>(p);
        return check_launch("gn_bwd_apply_arg");
    }
    const int rpp = 256 / C;
    long long workers = (rows + rpp - 1) / rpp, wr = (rows + rpp * 16 - 1) / (rpp * 16);   // >= 16 rows per reducing thread
    if (workers > cap) workers = cap;
    if (wr > cap) wr = cap;
    dim3 grid((unsigned)workers, (unsigned)B);
    k_gn_bwd_reduce<DET><<<dim3((unsigned)wr, (unsigned)B), 256, 0, st>>>(pr);
    int rc = check_launch("gn_bwd_reduce");
    if (rc || (rc = flush())) return rc;
    k_gn_bwd_apply<<<grid, 256, 0, st>>>(p);
    return check_launch("gn_bwd_apply");
}

extern "C" int pvraft_gn_act_bwd(const float* x, const float* dy, const double* stats, const float* gamma, const float* beta, double count,
                                 int act, float slope, int B, int64_t rows, int C, double* gsum, double* dgamma, double* dbeta,
                                 double* dslope, float* dx, const float* slope_dev, const uint8_t* arg, void* det_workspace, void* stream) {
    auto f = det_workspace ? gn_act_bwd<true> : gn_act_bwd<false>;
    return f(x, dy, stats, gamma, beta, count, act, slope, B, rows, C, gsum, dgamma, dbeta, dslope, dx, slope_dev, arg, det_workspace, stream);
}

extern "C" int64_t pvraft_gn_act_bwd_det_workspace_bytes(int B, int C) {
    return (int64_t)((int64_t)B * 16 + 2 * (int64_t)C + 1) * kFxWords * 8;
}

extern "C" int pvraft_gn_act_maxk_fwd(const float* x, const double* stats, const float* gamma, const float* beta, double count, int act,
                                      float slope, int B, int64_t pts_per_sample, int C, float* y, uint8_t* arg, const float* slope_dev,
                                      void* stream) {
    if (!x || !stats || !gamma || !beta || !y || !arg || B <= 0 || pts_per_sample <= 0) return fail(PVRAFT_ERR_BAD_ARG, "gn_act_maxk: bad argument");
    if (C > 256 || C % PVRAFT_GN_GROUPS) return fail(PVRAFT_ERR_UNSUPPORTED, "gn_act_maxk: C=%d", C);
    const long long total = (long long)B * pts_per_sample * C;
    k_gn_act_maxk<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(x, stats, gamma, beta, count, act, slope, B,
                                                                                      (long long)pts_per_sample, C, y, arg, slope_dev);
    return check_launch("gn_act_maxk");
}

extern "C" int pvraft_edge_fwd(const float* P, const int32_t* nbr, float* E, int B, int N, int C, double* stats, void* det_workspace,
                               void* stream) {
    if (!P || !nbr || !E || B <= 0 || N <= 0 || C <= 0) return fail(PVRAFT_ERR_BAD_ARG, "edge_fwd: bad argument");
    if (stats && C % PVRAFT_GN_GROUPS) return fail(PVRAFT_ERR_BAD_ARG, "edge_fwd: statistics need C %% 8 == 0");
    const unsigned blocks = (unsigned)(((long long)B * N + 7) / 8);
    cudaStream_t st = (cudaStream_t)stream;
    if (!det_workspace) {
        k_edge_fwd<false><<<blocks, 256, 0, st>>>(P, nbr, E, B, N, C, stats);
        return check_launch("edge_fwd");
    }
    k_edge_fwd<true><<<blocks, 256, 0, st>>>(P, nbr, E, B, N, C, stats ? static_cast<double*>(det_workspace) : nullptr);
    const int rc = check_launch("edge_fwd");
    if (rc || !stats) return rc;
    return fx_flush_f64(static_cast<const unsigned long long*>(det_workspace), 1, (long long)B * 16, (long long)B * 16, 0, stats, st);
}

extern "C" int64_t pvraft_edge_fwd_det_workspace_bytes(int B) { return (int64_t)B * 16 * kFxWords * 8; }

extern "C" int pvraft_edge_bwd(const float* dT, const int32_t* nbr, int B, int N, int C, float* dP, void* det_workspace, void* stream) {
    if (!dT || !nbr || !dP || B <= 0 || N <= 0 || C <= 0) return fail(PVRAFT_ERR_BAD_ARG, "edge_bwd: bad argument");
    const long long pts = (long long)B * N;
    const unsigned blocks = (unsigned)((pts + 7) / 8);
    cudaStream_t st = (cudaStream_t)stream;
    if (!det_workspace) {
        k_edge_bwd<false><<<blocks, 256, 0, st>>>(dT, nbr, B, N, C, dP);
        return check_launch("edge_bwd");
    }
    k_edge_bwd<true><<<blocks, 256, 0, st>>>(dT, nbr, B, N, C, static_cast<float*>(det_workspace));
    const int rc = check_launch("edge_bwd");
    if (rc) return rc;
    return fx_flush_f32(static_cast<const unsigned long long*>(det_workspace), 1, pts * C, pts * C, 0, dP, st);
}

extern "C" int64_t pvraft_edge_bwd_det_workspace_bytes(int B, int N, int C) { return (int64_t)B * N * C * kFxWords * 8; }

extern "C" int pvraft_maxk_fwd(const float* x, int64_t pts, int C, float* y, uint8_t* arg, void* stream) {
    if (!x || !y || !arg || pts <= 0 || C <= 0) return fail(PVRAFT_ERR_BAD_ARG, "maxk_fwd: bad argument");
    const long long total = (long long)pts * C;
    k_maxk_fwd<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(x, pts, C, y, arg);
    return check_launch("maxk_fwd");
}

extern "C" int pvraft_maxk_bwd(const float* dy, const uint8_t* arg, int64_t pts, int C, float* dx, void* stream) {
    if (!dy || !arg || !dx || pts <= 0 || C <= 0) return fail(PVRAFT_ERR_BAD_ARG, "maxk_bwd: bad argument");
    const long long total = (long long)pts * PVRAFT_KNN * C;
    if ((total + 255) / 256 > 0x7fffffffLL) return fail(PVRAFT_ERR_UNSUPPORTED, "maxk_bwd: too many elements");
    k_maxk_bwd<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(dy, arg, pts, C, dx);
    return check_launch("maxk_bwd");
}

extern "C" int pvraft_corr_lookup_bwd(const int32_t* corr_idx, const float* xyz2_pad, const float* coords, const int32_t* knn_slot,
                                      const float* g_vox, int vox_ld, const float* g_sel, int B, int N, int M, int K, int levels,
                                      float base_scale, float* d_corr, void* stream) {
    if (!corr_idx || !xyz2_pad || !coords || !knn_slot || !g_vox || !g_sel || !d_corr) return fail(PVRAFT_ERR_BAD_ARG, "corr_lookup_bwd: null pointer");
    if (B <= 0 || N <= 0 || M <= 0 || K < 32 || levels < 1 || levels > 4 || vox_ld < levels * 27)
        return fail(PVRAFT_ERR_BAD_ARG, "corr_lookup_bwd: bad shape");
    LookupBwdParams p{};
    p.corr_idx = corr_idx; p.tab = reinterpret_cast<const float4*>(xyz2_pad); p.coords = coords; p.knn_slot = knn_slot;
    p.g_vox = g_vox; p.g_sel = g_sel; p.d_corr = d_corr;
    p.B = B; p.N = N; p.M = M; p.K = K; p.levels = levels; p.vox_ld = vox_ld;
    p.pow2 = 1;
    for (int l = 0; l < 4; ++l) {
        const float r = (float)((double)base_scale * (double)(1 << l));   // as pvraft_corr_lookup_fwd
        p.r[l] = r;
        p.inv_r[l] = 1.0f / r;
        int e;
        if (l < levels && !(r > 0.f && frexpf(r, &e) == 0.5f)) p.pow2 = 0;
    }
    const long long pts = (long long)B * N;
    k_lookup_bwd<<<(unsigned)((pts + 7) / 8), 256, 0, (cudaStream_t)stream>>>(p);
    return check_launch("corr_lookup_bwd");
}

template <bool DET>
static int corr_init_bwd(const float* g, const int32_t* idx, const float* fmap1, const float* fmap2, int B, int N, int M, int C, int K,
                         float* d_fmap1, float* d_fmap2, void* ws, void* stream) {
    if (!g || !idx || !fmap1 || !fmap2 || !d_fmap1 || !d_fmap2 || B <= 0 || N <= 0 || M <= 0 || K <= 0)
        return fail(PVRAFT_ERR_BAD_ARG, "corr_init_bwd: bad argument");
    float* kd2 = DET ? static_cast<float*>(ws) : d_fmap2;
    const long long rows = (long long)B * N;
    const unsigned blocks = (unsigned)((rows + 7) / 8);
    const float scale = 1.0f / sqrtf((float)C);
    cudaStream_t st = (cudaStream_t)stream;
    switch (C) {
        case 32: k_corr_init_bwd<1, DET><<<blocks, 256, 0, st>>>(g, idx, fmap1, fmap2, B, N, M, K, scale, d_fmap1, kd2); break;
        case 64: k_corr_init_bwd<2, DET><<<blocks, 256, 0, st>>>(g, idx, fmap1, fmap2, B, N, M, K, scale, d_fmap1, kd2); break;
        case 128: k_corr_init_bwd<4, DET><<<blocks, 256, 0, st>>>(g, idx, fmap1, fmap2, B, N, M, K, scale, d_fmap1, kd2); break;
        case 256: k_corr_init_bwd<8, DET><<<blocks, 256, 0, st>>>(g, idx, fmap1, fmap2, B, N, M, K, scale, d_fmap1, kd2); break;
        default: return fail(PVRAFT_ERR_UNSUPPORTED, "corr_init_bwd: C=%d (32, 64, 128, 256)", C);
    }
    int rc = check_launch("corr_init_bwd");
    if (rc || !DET) return rc;
    const long long rows2 = (long long)B * M;
    return fx_flush_f32(static_cast<const unsigned long long*>(ws), 1, rows2 * C, rows2 * C, 0, d_fmap2, st);
}

extern "C" int pvraft_corr_init_bwd(const float* g, const int32_t* idx, const float* fmap1, const float* fmap2, int B, int N, int M, int C,
                                    int K, float* d_fmap1, float* d_fmap2, void* det_workspace, void* stream) {
    auto f = det_workspace ? corr_init_bwd<true> : corr_init_bwd<false>;
    return f(g, idx, fmap1, fmap2, B, N, M, C, K, d_fmap1, d_fmap2, det_workspace, stream);
}

extern "C" int64_t pvraft_corr_init_bwd_det_workspace_bytes(int B, int M, int C) { return (int64_t)B * M * C * kFxWords * 8; }
