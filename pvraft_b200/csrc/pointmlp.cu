// Dense per-point kernels of the PV-RAFT iteration (fp32, CUDA-core register-tiled GEMMs with the
// weights resident in shared memory of persistent CTAs):
//   k_linear   generic  [GroupNorm -> act ->] 1x1 conv [-> bias][-> ReLU] with output GN statistics
//   k_gn_act   trailing GroupNorm + activation (optionally writing channel-major)
//   k_corrfeat CorrBlock feature head (+ optional MotionEncoder)    reference model/corr.py:17-29,91-93,45
//                                                                   reference model/update.py:15-21
//   k_gru      ConvGRU                                              reference model/update.py:31-40
//   k_flowout  FlowHead tail + coordinate update                    reference model/update.py:69-72,
//                                                                   model/RAFTSceneFlow.py:45-46
// GroupNorm needs statistics over all points of a sample, so every GroupNorm is a kernel boundary:
// the producer accumulates double-precision (sum, sum^2) per (sample, group) with atomics and the
// consumer folds mean/rstd/gamma/beta into one FMA per element while staging its input tile.
#include "fixed_point.cuh"
#include "tile_gemm.cuh"

namespace pvraft {

// ---------------------------------------------------------------------------------------------------
// tile scheduling: tiles never straddle samples; CTA `blockIdx.x` owns a contiguous run of tiles
// ---------------------------------------------------------------------------------------------------
struct TileIter {
    long long t, t_end;
    int tiles_per_sample, N;
    __device__ TileIter(int B, int N_) : N(N_) {
        tiles_per_sample = (N_ + kTP - 1) / kTP;
        split_range((long long)B * tiles_per_sample, gridDim.x, blockIdx.x, t, t_end);
    }
    __device__ bool valid() const { return t < t_end; }
    __device__ int sample() const { return (int)(t / tiles_per_sample); }
    __device__ int p0() const { return (int)(t % tiles_per_sample) * kTP; }
    __device__ int npts() const { const int r = N - p0(); return r < kTP ? r : kTP; }
};

template <typename Kernel>
static int tile_grid(Kernel k, int B, int N, size_t smem) {
    const long long tiles = (long long)B * ((N + kTP - 1) / kTP);
    int occ = 1;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k, kMlpThreads, smem) != cudaSuccess) occ = 1;
    occ = occ < 1 ? 1 : (occ > 4 ? 4 : occ);
    // persistent CTAs, as many per SM as shared memory allows (<= 4): a CTA alternates between a load phase and
    // a GEMM phase, so co-resident CTAs are what overlaps the two
    long long g = (long long)sm_count() * occ;
    if (g > tiles) g = tiles;
    return (int)(g < 1 ? 1 : g);
}

// flush per-thread double partial sums of a (channel -> group) statistic into global [8][2]
__device__ __forceinline__ void flush_stats(double* s_g /*[16] smem*/, double* gstats /*[8][2] of the sample*/,
                                            const double* dS, const double* dSS, const int* ch, int n, int cout) {
    __syncthreads();
    if (threadIdx.x < 16) s_g[threadIdx.x] = 0.0;
    __syncthreads();
    const int gsz = cout / PVRAFT_GN_GROUPS;
    for (int i = 0; i < n; ++i) {
        if (ch[i] < cout && (dS[i] != 0.0 || dSS[i] != 0.0)) {
            const int g = ch[i] / gsz;
            atomicAdd(&s_g[g * 2 + 0], dS[i]);
            atomicAdd(&s_g[g * 2 + 1], dSS[i]);
        }
    }
    __syncthreads();
    if (threadIdx.x < 16 && s_g[threadIdx.x] != 0.0) atomicAdd(gstats + threadIdx.x, s_g[threadIdx.x]);
}

// DET form (fixed_point.cuh): after every tile, each thread's sums over its points of the tile enter the CTA's fixed-point
// slots s_fx [16]; when the CTA leaves a sample these are added to the sample's slots of the [B,16] workspace
__device__ __forceinline__ void tile_stats_fx(unsigned long long* s_fx, double* dS, double* dSS, const int* ch, int n, int cout) {
    const int gsz = cout / PVRAFT_GN_GROUPS;
    for (int i = 0; i < n; ++i) {
        if (ch[i] < cout && (dS[i] != 0.0 || dSS[i] != 0.0)) {
            const int g = ch[i] / gsz;
            fx_atomic(s_fx + (g * 2) * kFxWords, dS[i]);
            fx_atomic(s_fx + (g * 2 + 1) * kFxWords, dSS[i]);
        }
        dS[i] = 0.0;
        dSS[i] = 0.0;
    }
}

__device__ __forceinline__ void flush_stats_fx(unsigned long long* s_fx, unsigned long long* gfx /*[16] slots of the sample*/) {
    __syncthreads();
    if (threadIdx.x < 16) {
        const Fx v{s_fx[threadIdx.x * kFxWords], s_fx[threadIdx.x * kFxWords + 1], (unsigned)s_fx[threadIdx.x * kFxWords + 2]};
        fx_atomic(gfx + threadIdx.x * kFxWords, v);
    }
    __syncthreads();
    if (threadIdx.x < 16 * kFxWords) s_fx[threadIdx.x] = 0ull;
}

// ---------------------------------------------------------------------------------------------------
// k_linear
// ---------------------------------------------------------------------------------------------------
struct LinearParams {
    pvraft_linear_args a;
    int KD, WS, CP, AS, passes;
};

template <int CM4>
__device__ __forceinline__ void linear_compute(const LinearParams& P, const float* s_act, const float* s_w, const float* s_bias,
                                               size_t row0, int npts, double (&dS)[8], double (&dSS)[8]) {
    const pvraft_linear_args& a = P.a;
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    float acc[4][CM4 * 4];
#pragma unroll
    for (int p = 0; p < 4; ++p)
#pragma unroll
        for (int c = 0; c < CM4 * 4; ++c) acc[p][c] = 0.f;
    tile_gemm<CM4>(s_act, P.AS, s_w, P.WS, P.KD, acc);
#pragma unroll
    for (int pass = 0; pass < CM4; ++pass) {
        const int c0 = pass * 64 + tx * 4;
        const float4 bv = *reinterpret_cast<const float4*>(s_bias + c0);
#pragma unroll
        for (int p = 0; p < 4; ++p) {
            const int pp = ty * 4 + p;
            float y[4] = {acc[p][pass * 4 + 0] + bv.x, acc[p][pass * 4 + 1] + bv.y, acc[p][pass * 4 + 2] + bv.z,
                          acc[p][pass * 4 + 3] + bv.w};
#pragma unroll
            for (int c = 0; c < 4; ++c) y[c] = apply_act(y[c], a.out_act, 0.f);
            if (pp < npts) {
                float* o = a.out + (row0 + pp) * a.cout + c0;
                if (a.residual) {
                    const float* rs = a.residual + (row0 + pp) * a.cout + c0;
#pragma unroll
                    for (int c = 0; c < 4; ++c)
                        if (c0 + c < a.cout) y[c] += __ldg(rs + c);
                }
                if ((a.cout & 3) == 0 && c0 + 3 < a.cout) {
                    *reinterpret_cast<float4*>(o) = make_float4(y[0], y[1], y[2], y[3]);
                } else {
#pragma unroll
                    for (int c = 0; c < 4; ++c)
                        if (c0 + c < a.cout) o[c] = y[c];
                }
                if (a.out_stats) {
#pragma unroll
                    for (int c = 0; c < 4; ++c) {
                        const double v = (double)y[c];
                        dS[pass * 4 + c] += v;
                        dSS[pass * 4 + c] += v * v;
                    }
                }
            }
        }
    }
}

template <bool DET>
__global__ void __launch_bounds__(kMlpThreads, 2) k_linear(const LinearParams P) {
    const pvraft_linear_args& a = P.a;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float* s_w = reinterpret_cast<float*>(smem_raw);
    float* s_bias = s_w + P.KD * P.WS;
    float* s_scale = s_bias + P.CP;
    float* s_shift = s_scale + P.KD;
    float* s_act = s_shift + P.KD;
    double* s_g = reinterpret_cast<double*>(s_act + kTP * P.AS);   // [16]  (DET: [16] fixed-point slots; a.out_stats is the workspace)
    unsigned long long* s_fx = reinterpret_cast<unsigned long long*>(s_g);
    if constexpr (DET)
        if (threadIdx.x < 16 * kFxWords) s_fx[threadIdx.x] = 0ull;
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;

    const int w_cin = a.w_cin > 0 ? a.w_cin : a.cin;
    stage_weight(s_w, P.KD, P.WS, P.CP, a.weight, a.cout, a.w_ld > 0 ? a.w_ld : w_cin, 0, w_cin);
    stage_vector(s_bias, P.CP, a.bias, a.cout);

    double dS[8], dSS[8];
    int ch[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) { dS[i] = 0.0; dSS[i] = 0.0; ch[i] = (i >> 2) * 64 + tx * 4 + (i & 3); }
    int cur_b = -1;
    const bool vec4 = (a.cin & 3) == 0;

    for (TileIter it(a.B, a.N); it.valid(); ++it.t) {
        const int b = it.sample(), p0 = it.p0(), npts = it.npts();
        if (b != cur_b) {
            if constexpr (DET) {
                if (a.out_stats && cur_b >= 0) flush_stats_fx(s_fx, reinterpret_cast<unsigned long long*>(a.out_stats) + (size_t)cur_b * 16 * kFxWords);
            } else {
            if (a.out_stats && cur_b >= 0) flush_stats(s_g, a.out_stats + (size_t)cur_b * 16, dS, dSS, ch, P.passes * 4, a.cout);
            }
            if (cur_b >= 0) {
#pragma unroll
                for (int i = 0; i < 8; ++i) { dS[i] = 0.0; dSS[i] = 0.0; }
            }
            __syncthreads();
            if (a.in_mode != PVRAFT_IN_PLAIN) {
                const int gsz = a.cin / PVRAFT_GN_GROUPS;
                for (int k = tid; k < P.KD; k += blockDim.x) {
                    GnAffine af{0.f, 0.f};
                    if (k < a.cin) af = gn_affine(a.in_stats + (size_t)b * 16 + (k / gsz) * 2, a.in_count, __ldg(a.in_gamma + k), __ldg(a.in_beta + k));
                    s_scale[k] = af.scale;
                    s_shift[k] = af.shift;
                }
            }
            cur_b = b;
        }
        __syncthreads();   // previous tile's GEMM readers done; scale/shift visible
        // ---- stage the activation tile (GroupNorm + activation folded in) ----------------------------
        const size_t row0 = (size_t)b * a.N + p0;
        if (vec4) {
            const int c4 = a.cin >> 2;
            for (int i = tid; i < kTP * (P.KD >> 2); i += blockDim.x) {
                const int p = i / (P.KD >> 2), k4 = i - p * (P.KD >> 2);
                float4 x = make_float4(0.f, 0.f, 0.f, 0.f);
                if (p < npts && k4 < c4) {
                    const size_t g = (row0 + p) * a.cin + k4 * 4;
                    x = *reinterpret_cast<const float4*>(a.in + g);
                    if (a.in_mode != PVRAFT_IN_PLAIN) {
                        const float4 sc = *reinterpret_cast<const float4*>(s_scale + k4 * 4);
                        const float4 sh = *reinterpret_cast<const float4*>(s_shift + k4 * 4);
                        if (a.in_mode == PVRAFT_IN_GN_MINMAX) {
                            const float4 mn = *reinterpret_cast<const float4*>(a.in_min + g);
                            x.x = sc.x < 0.f ? mn.x : x.x; x.y = sc.y < 0.f ? mn.y : x.y;
                            x.z = sc.z < 0.f ? mn.z : x.z; x.w = sc.w < 0.f ? mn.w : x.w;
                        }
                        x.x = apply_act(fmaf(x.x, sc.x, sh.x), a.in_act, a.in_slope);
                        x.y = apply_act(fmaf(x.y, sc.y, sh.y), a.in_act, a.in_slope);
                        x.z = apply_act(fmaf(x.z, sc.z, sh.z), a.in_act, a.in_slope);
                        x.w = apply_act(fmaf(x.w, sc.w, sh.w), a.in_act, a.in_slope);
                    }
                }
                *reinterpret_cast<float4*>(s_act + p * P.AS + k4 * 4) = x;
            }
        } else {
            for (int i = tid; i < kTP * P.KD; i += blockDim.x) {
                const int p = i / P.KD, k = i - p * P.KD;
                float x = 0.f;
                if (p < npts && k < a.cin) {
                    const size_t g = (row0 + p) * a.cin + k;
                    x = __ldg(a.in + g);
                    if (a.in_mode != PVRAFT_IN_PLAIN) {
                        const float sc = s_scale[k];
                        if (a.in_mode == PVRAFT_IN_GN_MINMAX && sc < 0.f) x = __ldg(a.in_min + g);
                        x = apply_act(fmaf(x, sc, s_shift[k]), a.in_act, a.in_slope);
                    }
                }
                s_act[p * P.AS + k] = x;
            }
        }
        __syncthreads();
        // ---- GEMM: all (<= 128) output channels in one sweep over the activations + epilogue ------------------
        if (P.passes == 2) linear_compute<2>(P, s_act, s_w, s_bias, row0, npts, dS, dSS);
        else linear_compute<1>(P, s_act, s_w, s_bias, row0, npts, dS, dSS);
        if constexpr (DET)
            if (a.out_stats) tile_stats_fx(s_fx, dS, dSS, ch, P.passes * 4, a.cout);
    }
    if constexpr (DET) {
        if (a.out_stats && cur_b >= 0) flush_stats_fx(s_fx, reinterpret_cast<unsigned long long*>(a.out_stats) + (size_t)cur_b * 16 * kFxWords);
        return;
    }
    if (a.out_stats && cur_b >= 0) flush_stats(s_g, a.out_stats + (size_t)cur_b * 16, dS, dSS, ch, P.passes * 4, a.cout);
}

// ---------------------------------------------------------------------------------------------------
// k_gn_act: out = act(GN(in)), optional transpose to channel-major [B,C,N]
// ---------------------------------------------------------------------------------------------------
__global__ void k_gn_act(const float* __restrict__ in, const double* __restrict__ stats, const float* __restrict__ gamma,
                         const float* __restrict__ beta, double count, int act, float slope, int B, int N, int C,
                         int transpose_out, float* __restrict__ out, const float* __restrict__ slope_dev) {
    if (slope_dev) slope = __ldg(slope_dev);   // a learnable PReLU slope read on the device (no host read-back per optimizer step)
    __shared__ float s_scale[256], s_shift[256];
    __shared__ float s_tile[32][33];
    const int b = blockIdx.z;
    const int gsz = C / PVRAFT_GN_GROUPS;
    for (int k = threadIdx.y * 32 + threadIdx.x; k < C; k += 256) {
        const GnAffine af = gn_affine(stats + (size_t)b * 16 + (k / gsz) * 2, count, gamma[k], beta[k]);
        s_scale[k] = af.scale;
        s_shift[k] = af.shift;
    }
    __syncthreads();
    const int n0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
    // block (32 x 8) handles a 32 points x 32 channels patch
    for (int r = threadIdx.y; r < 32; r += 8) {
        const int n = n0 + r, c = c0 + threadIdx.x;
        float v = 0.f;
        if (n < N && c < C) v = apply_act(fmaf(in[((size_t)b * N + n) * C + c], s_scale[c], s_shift[c]), act, slope);
        if (!transpose_out) {
            if (n < N && c < C) out[((size_t)b * N + n) * C + c] = v;
        } else {
            s_tile[r][threadIdx.x] = v;
        }
    }
    if (transpose_out) {
        __syncthreads();
        for (int r = threadIdx.y; r < 32; r += 8) {
            const int c = c0 + r, n = n0 + threadIdx.x;
            if (n < N && c < C) out[((size_t)b * C + c) * N + n] = s_tile[threadIdx.x][r];
        }
    }
}

// [B,R,C] -> [B,C,R]
__global__ void k_transpose(const float* __restrict__ in, int R, int C, float* __restrict__ out) {
    __shared__ float s_tile[32][33];
    const int b = blockIdx.z, r0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
    for (int i = threadIdx.y; i < 32; i += 8) {
        const int r = r0 + i, c = c0 + threadIdx.x;
        if (r < R && c < C) s_tile[i][threadIdx.x] = in[((size_t)b * R + r) * C + c];
    }
    __syncthreads();
    for (int i = threadIdx.y; i < 32; i += 8) {
        const int c = c0 + i, r = r0 + threadIdx.x;
        if (r < R && c < C) out[((size_t)b * C + c) * R + r] = s_tile[threadIdx.x][i];
    }
}

// ---------------------------------------------------------------------------------------------------
// k_corrfeat: correlation feature head (+ optional motion encoder)
// ---------------------------------------------------------------------------------------------------
struct CorrFeatSmem {
    // offsets in floats
    int w_out, b_out, w_knn, b_knn, w_kout, b_kout, g1_scale, g1_shift, wk_eff, bk_eff;
    int w_cc, b_cc, w_cf, b_cf, w_cm, b_cm;
    int r1, sel, r3, total;
};
constexpr int kAS128 = 132, kAS64 = 68;
constexpr int kWS64 = 68, kWS128 = 132;   // wstride(64), wstride(128)

__host__ __device__ inline CorrFeatSmem corrfeat_layout() {
    CorrFeatSmem L{};
    int o = 0;
    auto take = [&](int n) { int r = o; o += (n + 3) & ~3; return r; };
    L.w_out = take(128 * kWS64); L.b_out = take(64);
    L.w_knn = take(4 * 64); L.b_knn = take(64);
    L.w_kout = take(64 * kWS64); L.b_kout = take(64);
    L.g1_scale = take(128); L.g1_shift = take(128);
    L.wk_eff = take(4 * 64); L.bk_eff = take(64);
    L.w_cc = take(64 * kWS64); L.b_cc = take(64);
    L.w_cf = take(4 * 64); L.b_cf = take(64);
    L.w_cm = take(128 * kWS64); L.b_cm = take(64);
    L.r1 = take(kTP * kAS128);      // GN'd y1 tile, later [cor | flo]
    L.sel = take(kTP * 32 * 4);     // kNN 4-vectors
    L.r3 = take(kTP * kAS64);       // kNN pooled feature, later the correlation feature
    L.total = o;
    return L;
}

__global__ void __launch_bounds__(kMlpThreads, 1) k_corrfeat(const pvraft_corrfeat_args a) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float* S = reinterpret_cast<float*>(smem_raw);
    const CorrFeatSmem L = corrfeat_layout();
    __shared__ double s_kn[64 * 2];   // per-channel (sum, sumsq) of the knn_conv output from the moments
    __shared__ float s_flow[kTP * 4];
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    const bool do_feat = a.y1 != nullptr;
    const bool do_motion = a.motion != nullptr;

    if (do_feat) {
        stage_weight(S + L.w_out, 128, kWS64, 64, a.w_out, 64, 128, 0, 128);
        stage_vector(S + L.b_out, 64, a.b_out, 64);
        stage_weight(S + L.w_knn, 4, 64, 64, a.w_knn, 64, 4, 0, 4);
        stage_vector(S + L.b_knn, 64, a.b_knn, 64);
        stage_weight(S + L.w_kout, 64, kWS64, 64, a.w_kout, 64, 64, 0, 64);
        stage_vector(S + L.b_kout, 64, a.b_kout, 64);
    }
    if (do_motion) {
        stage_weight(S + L.w_cc, 64, kWS64, 64, a.w_cc, 64, 64, 0, 64);
        stage_vector(S + L.b_cc, 64, a.b_cc, 64);
        stage_weight(S + L.w_cf, 4, 64, 64, a.w_cf, 64, 3, 0, 3);
        stage_vector(S + L.b_cf, 64, a.b_cf, 64);
        stage_weight(S + L.w_cm, 128, kWS64, 64, a.w_cm, 61, 128, 0, 128);
        stage_vector(S + L.b_cm, 64, a.b_cm, 61);
    }
    const float slope1 = do_feat ? __ldg(a.prelu1) : 0.f;
    const float slopek = do_feat ? __ldg(a.preluk) : 0.f;
    int cur_b = -1;

    for (TileIter it(a.B, a.N); it.valid(); ++it.t) {
        const int b = it.sample(), p0 = it.p0(), npts = it.npts();
        const size_t row0 = (size_t)b * a.N + p0;
        __syncthreads();
        if (do_feat && b != cur_b) {
            // GroupNorm(8,128) affine of out_conv[1] from the accumulated sums of y1
            if (tid < 128) {
                const GnAffine af = gn_affine(a.y1_stats + (size_t)b * 16 + (tid / 16) * 2, (double)a.N * 16.0,
                                              __ldg(a.gn1_gamma + tid), __ldg(a.gn1_beta + tid));
                S[L.g1_scale + tid] = af.scale;
                S[L.g1_shift + tid] = af.shift;
            }
            // statistics of t_c = w_c . f + b_c over all edges from the moments of f (see corr_lookup.cu)
            if (tid < 64) {
                const double* m = a.moments + (size_t)b * PVRAFT_MOMENTS;
                const double w0 = S[L.w_knn + 0 * 64 + tid], w1 = S[L.w_knn + 1 * 64 + tid];
                const double w2 = S[L.w_knn + 2 * 64 + tid], w3 = S[L.w_knn + 3 * 64 + tid];
                const double bc = S[L.b_knn + tid], cnt = m[14];
                const double lin = w0 * m[0] + w1 * m[1] + w2 * m[2] + w3 * m[3];
                const double quad = w0 * w0 * m[4] + w1 * w1 * m[8] + w2 * w2 * m[11] + w3 * w3 * m[13] +
                                    2.0 * (w0 * w1 * m[5] + w0 * w2 * m[6] + w0 * w3 * m[7] + w1 * w2 * m[9] +
                                           w1 * w3 * m[10] + w2 * w3 * m[12]);
                s_kn[tid * 2 + 0] = lin + cnt * bc;
                s_kn[tid * 2 + 1] = quad + 2.0 * bc * lin + cnt * bc * bc;
            }
            __syncthreads();
            if (tid < 64) {
                const int g = tid / 8;
                double st[2] = {0.0, 0.0};
                for (int c = g * 8; c < g * 8 + 8; ++c) { st[0] += s_kn[c * 2]; st[1] += s_kn[c * 2 + 1]; }
                const double cnt = a.moments[(size_t)b * PVRAFT_MOMENTS + 14] * 8.0;
                const GnAffine af = gn_affine(st, cnt, __ldg(a.gnk_gamma + tid), __ldg(a.gnk_beta + tid));
                // fold the GroupNorm affine into the 4->64 conv: t_norm = (scale*w).f + (scale*b + shift)
                for (int i = 0; i < 4; ++i) S[L.wk_eff + i * 64 + tid] = af.scale * S[L.w_knn + i * 64 + tid];
                S[L.bk_eff + tid] = fmaf(af.scale, S[L.b_knn + tid], af.shift);
            }
            cur_b = b;
            __syncthreads();
        }
        float corr[4][4];
        if (do_feat) {
            // ---- stage GN+PReLU(y1) and the kNN 4-vectors ------------------------------------------
            for (int i = tid; i < kTP * 32; i += blockDim.x) {
                const int p = i >> 5, k4 = i & 31;
                float4 x = make_float4(0.f, 0.f, 0.f, 0.f);
                if (p < npts) {
                    x = *reinterpret_cast<const float4*>(a.y1 + (row0 + p) * 128 + k4 * 4);
                    const float4 sc = *reinterpret_cast<const float4*>(S + L.g1_scale + k4 * 4);
                    const float4 sh = *reinterpret_cast<const float4*>(S + L.g1_shift + k4 * 4);
                    x.x = fmaf(x.x, sc.x, sh.x); x.y = fmaf(x.y, sc.y, sh.y); x.z = fmaf(x.z, sc.z, sh.z); x.w = fmaf(x.w, sc.w, sh.w);
                    x.x = x.x >= 0.f ? x.x : slope1 * x.x; x.y = x.y >= 0.f ? x.y : slope1 * x.y;
                    x.z = x.z >= 0.f ? x.z : slope1 * x.z; x.w = x.w >= 0.f ? x.w : slope1 * x.w;
                }
                *reinterpret_cast<float4*>(S + L.r1 + p * kAS128 + k4 * 4) = x;
            }
            for (int i = tid; i < kTP * 32; i += blockDim.x) {
                const int p = i >> 5;
                float4 x = make_float4(0.f, 0.f, 0.f, 0.f);
                if (p < npts) x = *reinterpret_cast<const float4*>(a.knn_sel + (row0 * 32 + i) * 4);
                *reinterpret_cast<float4*>(S + L.sel + i * 4) = x;
            }
            __syncthreads();
            // ---- voxel branch: Conv1d 128->64 ---------------------------------------------------------
            float vf[4][4];
#pragma unroll
            for (int p = 0; p < 4; ++p)
#pragma unroll
                for (int c = 0; c < 4; ++c) vf[p][c] = 0.f;
            tile_gemm<1>(S + L.r1, kAS128, S + L.w_out, kWS64, 128, vf);
            // ---- kNN branch: (GN-folded) 4->64 conv, PReLU, max over the 32 neighbours -----------------
            {
                float4 wk[4];
#pragma unroll
                for (int i = 0; i < 4; ++i) wk[i] = *reinterpret_cast<const float4*>(S + L.wk_eff + i * 64 + tx * 4);
                const float4 bk = *reinterpret_cast<const float4*>(S + L.bk_eff + tx * 4);
#pragma unroll
                for (int p = 0; p < 4; ++p) {
                    float m[4] = {-INFINITY, -INFINITY, -INFINITY, -INFINITY};
                    const float4* fp = reinterpret_cast<const float4*>(S + L.sel) + (ty * 4 + p) * 32;
#pragma unroll 4
                    for (int e = 0; e < 32; ++e) {
                        const float4 f = fp[e];
                        float t0 = fmaf(wk[3].x, f.w, fmaf(wk[2].x, f.z, fmaf(wk[1].x, f.y, fmaf(wk[0].x, f.x, bk.x))));
                        float t1 = fmaf(wk[3].y, f.w, fmaf(wk[2].y, f.z, fmaf(wk[1].y, f.y, fmaf(wk[0].y, f.x, bk.y))));
                        float t2 = fmaf(wk[3].z, f.w, fmaf(wk[2].z, f.z, fmaf(wk[1].z, f.y, fmaf(wk[0].z, f.x, bk.z))));
                        float t3 = fmaf(wk[3].w, f.w, fmaf(wk[2].w, f.z, fmaf(wk[1].w, f.y, fmaf(wk[0].w, f.x, bk.w))));
                        t0 = t0 >= 0.f ? t0 : slopek * t0; t1 = t1 >= 0.f ? t1 : slopek * t1;
                        t2 = t2 >= 0.f ? t2 : slopek * t2; t3 = t3 >= 0.f ? t3 : slopek * t3;
                        m[0] = fmaxf(m[0], t0); m[1] = fmaxf(m[1], t1); m[2] = fmaxf(m[2], t2); m[3] = fmaxf(m[3], t3);
                    }
                    *reinterpret_cast<float4*>(S + L.r3 + (ty * 4 + p) * kAS64 + tx * 4) = make_float4(m[0], m[1], m[2], m[3]);
                }
            }
            __syncthreads();
            float kf[4][4];
#pragma unroll
            for (int p = 0; p < 4; ++p)
#pragma unroll
                for (int c = 0; c < 4; ++c) kf[p][c] = 0.f;
            tile_gemm<1>(S + L.r3, kAS64, S + L.w_kout, kWS64, 64, kf);
            const float4 bo = *reinterpret_cast<const float4*>(S + L.b_out + tx * 4);
            const float4 bko = *reinterpret_cast<const float4*>(S + L.b_kout + tx * 4);
#pragma unroll
            for (int p = 0; p < 4; ++p) {
                corr[p][0] = (vf[p][0] + bo.x) + (kf[p][0] + bko.x);
                corr[p][1] = (vf[p][1] + bo.y) + (kf[p][1] + bko.y);
                corr[p][2] = (vf[p][2] + bo.z) + (kf[p][2] + bko.z);
                corr[p][3] = (vf[p][3] + bo.w) + (kf[p][3] + bko.w);
                const int pp = ty * 4 + p;
                if (a.corr_feat && pp < npts)
                    *reinterpret_cast<float4*>(a.corr_feat + (row0 + pp) * 64 + tx * 4) = make_float4(corr[p][0], corr[p][1], corr[p][2], corr[p][3]);
            }
            __syncthreads();   // r3 readers (kNN GEMM) done before it is reused below
        } else {
#pragma unroll
            for (int p = 0; p < 4; ++p) {
                const int pp = ty * 4 + p;
                float4 x = make_float4(0.f, 0.f, 0.f, 0.f);
                if (pp < npts) x = *reinterpret_cast<const float4*>(a.corr_in + (row0 + pp) * 64 + tx * 4);
                corr[p][0] = x.x; corr[p][1] = x.y; corr[p][2] = x.z; corr[p][3] = x.w;
            }
        }
        if (do_motion) {
            // ---- MotionEncoder: relu(conv_corr), relu(conv_flow), relu(conv([cor,flo])), ++ flow -----
#pragma unroll
            for (int p = 0; p < 4; ++p)
                *reinterpret_cast<float4*>(S + L.r3 + (ty * 4 + p) * kAS64 + tx * 4) = make_float4(corr[p][0], corr[p][1], corr[p][2], corr[p][3]);
            if (tid < kTP) {
                float4 f = make_float4(0.f, 0.f, 0.f, 0.f);
                if (tid < npts) {
                    const float* fl = a.flow + (row0 + tid) * 3;
                    f = make_float4(fl[0], fl[1], fl[2], 0.f);
                }
                *reinterpret_cast<float4*>(s_flow + tid * 4) = f;
            }
            __syncthreads();
            float cor[4][4];
#pragma unroll
            for (int p = 0; p < 4; ++p)
#pragma unroll
                for (int c = 0; c < 4; ++c) cor[p][c] = 0.f;
            tile_gemm<1>(S + L.r3, kAS64, S + L.w_cc, kWS64, 64, cor);
            const float4 bcc = *reinterpret_cast<const float4*>(S + L.b_cc + tx * 4);
            const float4 bcf = *reinterpret_cast<const float4*>(S + L.b_cf + tx * 4);
            float4 wf[3];
#pragma unroll
            for (int i = 0; i < 3; ++i) wf[i] = *reinterpret_cast<const float4*>(S + L.w_cf + i * 64 + tx * 4);
#pragma unroll
            for (int p = 0; p < 4; ++p) {
                const int pp = ty * 4 + p;
                const float4 f = *reinterpret_cast<const float4*>(s_flow + pp * 4);
                float4 c4 = make_float4(fmaxf(cor[p][0] + bcc.x, 0.f), fmaxf(cor[p][1] + bcc.y, 0.f),
                                        fmaxf(cor[p][2] + bcc.z, 0.f), fmaxf(cor[p][3] + bcc.w, 0.f));
                float4 f4;
                f4.x = fmaxf(fmaf(wf[2].x, f.z, fmaf(wf[1].x, f.y, fmaf(wf[0].x, f.x, bcf.x))), 0.f);
                f4.y = fmaxf(fmaf(wf[2].y, f.z, fmaf(wf[1].y, f.y, fmaf(wf[0].y, f.x, bcf.y))), 0.f);
                f4.z = fmaxf(fmaf(wf[2].z, f.z, fmaf(wf[1].z, f.y, fmaf(wf[0].z, f.x, bcf.z))), 0.f);
                f4.w = fmaxf(fmaf(wf[2].w, f.z, fmaf(wf[1].w, f.y, fmaf(wf[0].w, f.x, bcf.w))), 0.f);
                *reinterpret_cast<float4*>(S + L.r1 + pp * kAS128 + tx * 4) = c4;
                *reinterpret_cast<float4*>(S + L.r1 + pp * kAS128 + 64 + tx * 4) = f4;
            }
            __syncthreads();
            float mo[4][4];
#pragma unroll
            for (int p = 0; p < 4; ++p)
#pragma unroll
                for (int c = 0; c < 4; ++c) mo[p][c] = 0.f;
            tile_gemm<1>(S + L.r1, kAS128, S + L.w_cm, kWS64, 128, mo);
            const float4 bcm = *reinterpret_cast<const float4*>(S + L.b_cm + tx * 4);
#pragma unroll
            for (int p = 0; p < 4; ++p) {
                const int pp = ty * 4 + p;
                float y[4] = {fmaxf(mo[p][0] + bcm.x, 0.f), fmaxf(mo[p][1] + bcm.y, 0.f),
                              fmaxf(mo[p][2] + bcm.z, 0.f), fmaxf(mo[p][3] + bcm.w, 0.f)};
                if (tx == 15) {   // channels 60..63: 60 is learned, 61..63 carry the flow (update.py:20)
                    const float4 f = *reinterpret_cast<const float4*>(s_flow + pp * 4);
                    y[1] = f.x; y[2] = f.y; y[3] = f.z;
                }
                if (pp < npts) *reinterpret_cast<float4*>(a.motion + (row0 + pp) * 64 + tx * 4) = make_float4(y[0], y[1], y[2], y[3]);
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------------
// k_gru: ConvGRU over [h | inp | motion]
// ---------------------------------------------------------------------------------------------------
constexpr int kAS192 = 196;
struct GruSmem { int w_zr, w_qx, w_qh, b_z, b_r, b_q, act, rh, total; };
__host__ __device__ inline GruSmem gru_layout() {
    GruSmem L{};
    int o = 0;
    auto take = [&](int n) { int r = o; o += (n + 3) & ~3; return r; };
    L.w_zr = take(192 * kWS128); L.w_qx = take(128 * kWS64); L.w_qh = take(64 * kWS64);
    L.b_z = take(64); L.b_r = take(64); L.b_q = take(64);
    L.act = take(kTP * kAS192); L.rh = take(kTP * kAS64);
    L.total = o;
    return L;
}

__device__ __forceinline__ float sigmoid_f(float x) { return 1.f / (1.f + expf(-x)); }

__global__ void __launch_bounds__(kMlpThreads, 1) k_gru(const pvraft_gru_args a) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float* S = reinterpret_cast<float*>(smem_raw);
    const GruSmem L = gru_layout();
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    // [z | r] weights side by side, k-major [192][128 (+4)]
    stage_weight(S + L.w_zr, 192, kWS128, 64, a.w_z, 64, 192, 0, 192);
    stage_weight(S + L.w_zr + 64, 192, kWS128, 64, a.w_r, 64, 192, 0, 192);
    stage_weight(S + L.w_qx, 128, kWS64, 64, a.w_q, 64, 192, 64, 128);   // columns 64..191 act on x = [inp, motion]
    stage_weight(S + L.w_qh, 64, kWS64, 64, a.w_q, 64, 192, 0, 64);      // columns 0..63 act on r*h
    stage_vector(S + L.b_z, 64, a.b_z, 64);
    stage_vector(S + L.b_r, 64, a.b_r, 64);
    stage_vector(S + L.b_q, 64, a.b_q, 64);

    // the next tile's [h | inp | motion] rows are fetched into registers while the current tile is in the GEMMs
    float4 pf[12];
    auto fetch = [&](const TileIter& t) {
        const size_t r0 = (size_t)t.sample() * a.N + t.p0();
        const int np = t.npts();
#pragma unroll
        for (int q = 0; q < 12; ++q) {
            const int i = tid + q * kMlpThreads, p = i / 48, k4 = i - p * 48;
            pf[q] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (p < np) {
                const float* src = k4 < 16 ? a.net : (k4 < 32 ? a.inp : a.motion);
                pf[q] = __ldg(reinterpret_cast<const float4*>(src + (r0 + p) * 64 + (k4 & 15) * 4));
            }
        }
    };
    TileIter it(a.B, a.N);
    if (it.valid()) fetch(it);
    for (; it.valid(); ++it.t) {
        const int p0 = it.p0(), npts = it.npts();
        const size_t row0 = (size_t)it.sample() * a.N + p0;
        __syncthreads();
#pragma unroll
        for (int q = 0; q < 12; ++q) {
            const int i = tid + q * kMlpThreads, p = i / 48, k4 = i - p * 48;
            *reinterpret_cast<float4*>(S + L.act + p * kAS192 + k4 * 4) = pf[q];
        }
        __syncthreads();
        {
            TileIter nx = it;
            ++nx.t;
            if (nx.valid()) fetch(nx);
        }
        float zr[4][8];
#pragma unroll
        for (int p = 0; p < 4; ++p)
#pragma unroll
            for (int c = 0; c < 8; ++c) zr[p][c] = 0.f;
        tile_gemm<2>(S + L.act, kAS192, S + L.w_zr, kWS128, 192, zr);
        const float4 bz = *reinterpret_cast<const float4*>(S + L.b_z + tx * 4);
        const float4 br = *reinterpret_cast<const float4*>(S + L.b_r + tx * 4);
        float z[4][4], h[4][4];
#pragma unroll
        for (int p = 0; p < 4; ++p) {
            const int pp = ty * 4 + p;
            const float4 hv = *reinterpret_cast<const float4*>(S + L.act + pp * kAS192 + tx * 4);
            h[p][0] = hv.x; h[p][1] = hv.y; h[p][2] = hv.z; h[p][3] = hv.w;
            z[p][0] = sigmoid_f(zr[p][0] + bz.x); z[p][1] = sigmoid_f(zr[p][1] + bz.y);
            z[p][2] = sigmoid_f(zr[p][2] + bz.z); z[p][3] = sigmoid_f(zr[p][3] + bz.w);
            const float r0 = sigmoid_f(zr[p][4] + br.x), r1 = sigmoid_f(zr[p][5] + br.y);
            const float r2 = sigmoid_f(zr[p][6] + br.z), r3 = sigmoid_f(zr[p][7] + br.w);
            *reinterpret_cast<float4*>(S + L.rh + pp * kAS64 + tx * 4) = make_float4(r0 * hv.x, r1 * hv.y, r2 * hv.z, r3 * hv.w);
        }
        __syncthreads();
        float q[4][4];
#pragma unroll
        for (int p = 0; p < 4; ++p)
#pragma unroll
            for (int c = 0; c < 4; ++c) q[p][c] = 0.f;
        tile_gemm<1>(S + L.rh, kAS64, S + L.w_qh, kWS64, 64, q);
        tile_gemm<1>(S + L.act + 64, kAS192, S + L.w_qx, kWS64, 128, q);
        const float4 bq = *reinterpret_cast<const float4*>(S + L.b_q + tx * 4);
#pragma unroll
        for (int p = 0; p < 4; ++p) {
            const int pp = ty * 4 + p;
            const float q0 = tanhf(q[p][0] + bq.x), q1 = tanhf(q[p][1] + bq.y), q2 = tanhf(q[p][2] + bq.z), q3 = tanhf(q[p][3] + bq.w);
            float4 o;
            o.x = (1.f - z[p][0]) * h[p][0] + z[p][0] * q0;
            o.y = (1.f - z[p][1]) * h[p][1] + z[p][1] * q1;
            o.z = (1.f - z[p][2]) * h[p][2] + z[p][2] * q2;
            o.w = (1.f - z[p][3]) * h[p][3] + z[p][3] * q3;
            if (pp < npts) *reinterpret_cast<float4*>(a.net_out + (row0 + pp) * 64 + tx * 4) = o;
        }
    }
}

// ---------------------------------------------------------------------------------------------------
// k_flowout: GN3+LReLU(setconv) ++ conv1(net) -> Conv1d 128->64, ReLU, Conv1d 64->3; coords update
// ---------------------------------------------------------------------------------------------------
struct FlowOutSmem { int w_c1, b_c1, w_o0, b_o0, w_o2, b_o2, scale, shift, cat, tmp, total; };
__host__ __device__ inline FlowOutSmem flowout_layout() {
    FlowOutSmem L{};
    int o = 0;
    auto take = [&](int n) { int r = o; o += (n + 3) & ~3; return r; };
    L.w_c1 = take(64 * kWS64); L.b_c1 = take(64);
    L.w_o0 = take(128 * kWS64); L.b_o0 = take(64);
    L.w_o2 = take(64 * 4); L.b_o2 = take(4);
    L.scale = take(64); L.shift = take(64);
    L.cat = take(kTP * kAS128); L.tmp = take(kTP * kAS64);
    L.total = o;
    return L;
}

__global__ void __launch_bounds__(kMlpThreads, 2) k_flowout(const pvraft_flowout_args a) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float* S = reinterpret_cast<float*>(smem_raw);
    const FlowOutSmem L = flowout_layout();
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    stage_weight(S + L.w_c1, 64, kWS64, 64, a.w_c1, 64, 64, 0, 64);
    stage_vector(S + L.b_c1, 64, a.b_c1, 64);
    stage_weight(S + L.w_o0, 128, kWS64, 64, a.w_o0, 64, 128, 0, 128);
    stage_vector(S + L.b_o0, 64, a.b_o0, 64);
    stage_weight(S + L.w_o2, 64, 4, 4, a.w_o2, 3, 64, 0, 64);
    stage_vector(S + L.b_o2, 4, a.b_o2, 3);
    int cur_b = -1;
    for (TileIter it(a.B, a.N); it.valid(); ++it.t) {
        const int b = it.sample(), p0 = it.p0(), npts = it.npts();
        const size_t row0 = (size_t)b * a.N + p0;
        __syncthreads();
        if (b != cur_b) {
            if (tid < 64) {
                const GnAffine af = gn_affine(a.z3_stats + (size_t)b * 16 + (tid / 8) * 2, (double)a.N * 8.0,
                                              __ldg(a.gn3_gamma + tid), __ldg(a.gn3_beta + tid));
                S[L.scale + tid] = af.scale;
                S[L.shift + tid] = af.shift;
            }
            cur_b = b;
            __syncthreads();
        }
        // cat[:, 0:64] = LeakyReLU(GN3(z3)) (gconv.py:82-83);  tmp = net tile (input of conv1)
        for (int i = tid; i < kTP * 16; i += blockDim.x) {
            const int p = i >> 4, k4 = i & 15;
            float4 s = make_float4(0.f, 0.f, 0.f, 0.f), n = s;
            if (p < npts) {
                s = *reinterpret_cast<const float4*>(a.z3 + (row0 + p) * 64 + k4 * 4);
                n = *reinterpret_cast<const float4*>(a.net + (row0 + p) * 64 + k4 * 4);
                const float4 sc = *reinterpret_cast<const float4*>(S + L.scale + k4 * 4);
                const float4 sh = *reinterpret_cast<const float4*>(S + L.shift + k4 * 4);
                s.x = fmaf(s.x, sc.x, sh.x); s.y = fmaf(s.y, sc.y, sh.y); s.z = fmaf(s.z, sc.z, sh.z); s.w = fmaf(s.w, sc.w, sh.w);
                s.x = s.x >= 0.f ? s.x : 0.1f * s.x; s.y = s.y >= 0.f ? s.y : 0.1f * s.y;
                s.z = s.z >= 0.f ? s.z : 0.1f * s.z; s.w = s.w >= 0.f ? s.w : 0.1f * s.w;
            }
            *reinterpret_cast<float4*>(S + L.cat + p * kAS128 + k4 * 4) = s;
            *reinterpret_cast<float4*>(S + L.tmp + p * kAS64 + k4 * 4) = n;
        }
        __syncthreads();
        float c1[4][4];
#pragma unroll
        for (int p = 0; p < 4; ++p)
#pragma unroll
            for (int c = 0; c < 4; ++c) c1[p][c] = 0.f;
        tile_gemm<1>(S + L.tmp, kAS64, S + L.w_c1, kWS64, 64, c1);
        const float4 bc1 = *reinterpret_cast<const float4*>(S + L.b_c1 + tx * 4);
#pragma unroll
        for (int p = 0; p < 4; ++p)
            *reinterpret_cast<float4*>(S + L.cat + (ty * 4 + p) * kAS128 + 64 + tx * 4) =
                make_float4(c1[p][0] + bc1.x, c1[p][1] + bc1.y, c1[p][2] + bc1.z, c1[p][3] + bc1.w);
        __syncthreads();
        float o0[4][4];
#pragma unroll
        for (int p = 0; p < 4; ++p)
#pragma unroll
            for (int c = 0; c < 4; ++c) o0[p][c] = 0.f;
        tile_gemm<1>(S + L.cat, kAS128, S + L.w_o0, kWS64, 128, o0);
        const float4 bo0 = *reinterpret_cast<const float4*>(S + L.b_o0 + tx * 4);
#pragma unroll
        for (int p = 0; p < 4; ++p)
            *reinterpret_cast<float4*>(S + L.tmp + (ty * 4 + p) * kAS64 + tx * 4) =
                make_float4(fmaxf(o0[p][0] + bo0.x, 0.f), fmaxf(o0[p][1] + bo0.y, 0.f), fmaxf(o0[p][2] + bo0.z, 0.f), fmaxf(o0[p][3] + bo0.w, 0.f));
        __syncthreads();
        if (tid < kTP * 3) {
            const int p = tid / 3, c = tid - p * 3;
            if (p < npts) {
                float acc = S[L.b_o2 + c];
                const float* t = S + L.tmp + p * kAS64;
#pragma unroll 8
                for (int k = 0; k < 64; ++k) acc = fmaf(t[k], S[L.w_o2 + k * 4 + c], acc);
                const size_t g = (row0 + p) * 3 + c;
                if (a.delta) a.delta[g] = acc;
                if (a.coords2_out) {
                    const float c2 = a.coords2[g] + acc;               // RAFTSceneFlow.py:45
                    a.coords2_out[g] = c2;
                    if (a.flow_out) a.flow_out[g] = c2 - a.coords1[g]; // RAFTSceneFlow.py:46
                }
            }
        }
    }
}

}  // namespace pvraft

using namespace pvraft;

template <bool DET>
static int linear_fwd(const pvraft_linear_args* a, void* ws, void* stream) {
    if (!a || !a->in || !a->weight || !a->out) return fail(PVRAFT_ERR_BAD_ARG, "linear: null pointer");
    if (a->B <= 0 || a->N <= 0 || a->cin <= 0 || a->cout <= 0) return fail(PVRAFT_ERR_BAD_ARG, "linear: bad shape");
    if (a->cout > 128 || a->cin > 256) return fail(PVRAFT_ERR_UNSUPPORTED, "linear: cin=%d cout=%d (max 256/128)", a->cin, a->cout);
    if (a->in_mode != PVRAFT_IN_PLAIN) {
        if (!a->in_stats || !a->in_gamma || !a->in_beta || a->cin % PVRAFT_GN_GROUPS) return fail(PVRAFT_ERR_BAD_ARG, "linear: GroupNorm input needs stats/gamma/beta and cin %% 8 == 0");
        if (a->in_mode == PVRAFT_IN_GN_MINMAX && !a->in_min) return fail(PVRAFT_ERR_BAD_ARG, "linear: in_min missing");
    }
    if (a->out_stats && a->cout % PVRAFT_GN_GROUPS) return fail(PVRAFT_ERR_BAD_ARG, "linear: out_stats needs cout %% 8 == 0");
    LinearParams P{};
    P.a = *a;
    if (DET && a->out_stats) P.a.out_stats = static_cast<double*>(ws);
    P.KD = pad4(a->cin);
    P.CP = pad64(a->cout);
    P.WS = wstride(P.CP);
    P.AS = act_stride(P.KD);
    P.passes = P.CP / 64;
    const size_t smem = sizeof(float) * ((size_t)P.KD * P.WS + P.CP + 2 * P.KD + (size_t)kTP * P.AS) + 16 * (DET ? kFxWords * 8 : sizeof(double)) + 16;
    int rc;
    if ((rc = opt_in_smem(k_linear<DET>, smem))) return rc;
    k_linear<DET><<<tile_grid(k_linear<DET>, a->B, a->N, smem), kMlpThreads, smem, (cudaStream_t)stream>>>(P);
    rc = check_launch("linear");
    if (rc || !DET || !a->out_stats) return rc;
    return fx_flush_f64(static_cast<const unsigned long long*>(ws), 1, (long long)a->B * 16, (long long)a->B * 16, 0, a->out_stats, (cudaStream_t)stream);
}

extern "C" int pvraft_linear_fwd(const pvraft_linear_args* a, void* det_workspace, void* stream) {
    return det_workspace ? linear_fwd<true>(a, det_workspace, stream) : linear_fwd<false>(a, nullptr, stream);
}

extern "C" int64_t pvraft_linear_det_workspace_bytes(int B) { return (int64_t)B * 16 * kFxWords * 8; }

extern "C" int pvraft_gn_act_fwd(const float* in, const double* stats, const float* gamma, const float* beta, double count,
                                 int act, float slope, int B, int N, int C, int transpose_out, float* out, const float* slope_dev,
                                 void* stream) {
    if (!in || !stats || !gamma || !beta || !out) return fail(PVRAFT_ERR_BAD_ARG, "gn_act: null pointer");
    if (C > 256 || C % PVRAFT_GN_GROUPS) return fail(PVRAFT_ERR_UNSUPPORTED, "gn_act: C=%d", C);
    dim3 grid((N + 31) / 32, (C + 31) / 32, B), block(32, 8);
    k_gn_act<<<grid, block, 0, (cudaStream_t)stream>>>(in, stats, gamma, beta, count, act, slope, B, N, C, transpose_out, out, slope_dev);
    return check_launch("gn_act");
}

extern "C" int pvraft_transpose_fwd(const float* in, int B, int R, int C, float* out, void* stream) {
    if (!in || !out || B <= 0 || R <= 0 || C <= 0) return fail(PVRAFT_ERR_BAD_ARG, "transpose: bad argument");
    dim3 grid((R + 31) / 32, (C + 31) / 32, B), block(32, 8);
    k_transpose<<<grid, block, 0, (cudaStream_t)stream>>>(in, R, C, out);
    return check_launch("transpose");
}

extern "C" int pvraft_corr_feature_fwd(const pvraft_corrfeat_args* a, void* stream) {
    if (!a || a->B <= 0 || a->N <= 0) return fail(PVRAFT_ERR_BAD_ARG, "corr_feature: bad argument");
    const bool feat = a->y1 != nullptr, motion = a->motion != nullptr;
    if (!feat && !motion) return fail(PVRAFT_ERR_BAD_ARG, "corr_feature: nothing to do");
    if (feat && (!a->y1_stats || !a->gn1_gamma || !a->gn1_beta || !a->prelu1 || !a->w_out || !a->b_out || !a->knn_sel ||
                 !a->moments || !a->w_knn || !a->b_knn || !a->gnk_gamma || !a->gnk_beta || !a->preluk || !a->w_kout || !a->b_kout))
        return fail(PVRAFT_ERR_BAD_ARG, "corr_feature: null pointer in the feature stage");
    if (!feat && !a->corr_in) return fail(PVRAFT_ERR_BAD_ARG, "corr_feature: corr_in required without y1");
    if (motion && (!a->flow || !a->w_cc || !a->b_cc || !a->w_cf || !a->b_cf || !a->w_cm || !a->b_cm))
        return fail(PVRAFT_ERR_BAD_ARG, "corr_feature: null pointer in the motion stage");
    const size_t smem = (size_t)corrfeat_layout().total * sizeof(float);
    int rc;
    if ((rc = opt_in_smem(k_corrfeat, smem))) return rc;
    k_corrfeat<<<tile_grid(k_corrfeat, a->B, a->N, smem), kMlpThreads, smem, (cudaStream_t)stream>>>(*a);
    return check_launch("corr_feature");
}

extern "C" int pvraft_gru_fwd(const pvraft_gru_args* a, void* stream) {
    if (!a || !a->net || !a->inp || !a->motion || !a->w_z || !a->b_z || !a->w_r || !a->b_r || !a->w_q || !a->b_q || !a->net_out)
        return fail(PVRAFT_ERR_BAD_ARG, "gru: null pointer");
    if (a->B <= 0 || a->N <= 0) return fail(PVRAFT_ERR_BAD_ARG, "gru: bad shape");
    const size_t smem = (size_t)gru_layout().total * sizeof(float);
    int rc;
    if ((rc = opt_in_smem(k_gru, smem))) return rc;
    k_gru<<<tile_grid(k_gru, a->B, a->N, smem), kMlpThreads, smem, (cudaStream_t)stream>>>(*a);
    return check_launch("gru");
}

extern "C" int pvraft_flow_out_fwd(const pvraft_flowout_args* a, void* stream) {
    if (!a || !a->z3 || !a->z3_stats || !a->gn3_gamma || !a->gn3_beta || !a->net || !a->w_c1 || !a->b_c1 || !a->w_o0 ||
        !a->b_o0 || !a->w_o2 || !a->b_o2)
        return fail(PVRAFT_ERR_BAD_ARG, "flow_out: null pointer");
    if (a->coords2_out && (!a->coords2 || (a->flow_out && !a->coords1))) return fail(PVRAFT_ERR_BAD_ARG, "flow_out: coords missing");
    if (a->B <= 0 || a->N <= 0) return fail(PVRAFT_ERR_BAD_ARG, "flow_out: bad shape");
    const size_t smem = (size_t)flowout_layout().total * sizeof(float);
    int rc;
    if ((rc = opt_in_smem(k_flowout, smem))) return rc;
    k_flowout<<<tile_grid(k_flowout, a->B, a->N, smem), kMlpThreads, smem, (cudaStream_t)stream>>>(*a);
    return check_launch("flow_out");
}
