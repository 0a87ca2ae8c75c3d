// kNN branch of the correlation feature head + the flow embedding of the MotionEncoder, for the tensor-core path.
//
//   kfeat[b,n,c] = max_e PReLU(GN(knn_conv.0(f_e)))      reference model/corr.py:86-92 (knn_conv, then max over dim 3)
//   cflow[b,n,c] = relu(conv_flow(flow))                 reference model/update.py:17
//
// f_e = (corr, dx, dy, dz) of the 32 selected candidates (knn_sel from the lookup kernel).  The GroupNorm statistics of the
// [B,64,N,32] tensor follow analytically from the per-sample moments of f that the lookup accumulated, so the affine is
// folded into the 4->64 convolution and the whole branch is one pass: 4 FMA + max + min per (candidate, channel).
// PReLU with slope <= 1 is convex, so max_e PReLU(t_e) = max(PReLU(max_e t_e), PReLU(min_e t_e)) exactly; a learned slope
// above 1 takes the per-candidate path.
//
// Thread layout: 256 threads = 16 (channel quads) x 16 (point quads) over a tile of 64 points whose 32x4 candidate
// vectors are staged in shared memory (32 KB); several CTAs share an SM.
#include "common.cuh"

namespace pvraft {

constexpr int kKbThreads = 256;
constexpr int kKbTile = 64;

// two IEEE fma.rn over a candidate pair
__device__ __forceinline__ float2 fma2(float2 a, float2 b, float2 c) {
    return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y));
}

template <bool CONVEX>
__global__ void __launch_bounds__(kKbThreads) k_knn_branch(const pvraft_knn_branch_args a) {
    __shared__ __align__(16) float s_sel[kKbTile * 32 * 4];
    __shared__ __align__(16) float s_w[4 * 64];      // folded weights, [i][c]
    __shared__ __align__(16) float s_b[64];
    __shared__ __align__(16) float s_wf[4 * 64];     // conv_flow, [i][c] (i < 3)
    __shared__ __align__(16) float s_bf[64];
    __shared__ double s_kn[64 * 2];
    pdl_trigger();   // the next kernel may be staged while this one drains
    pdl_wait();      // (launched with PDL: nothing above touches global memory)
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    const int tiles_per_sample = (a.N + kKbTile - 1) / kKbTile;
    const int n_tiles = a.B * tiles_per_sample;
    const float slope = __ldg(a.preluk);
    if (a.cflow != nullptr && tid < 64) {
        s_wf[0 * 64 + tid] = __ldg(a.w_cf + tid * 3 + 0);
        s_wf[1 * 64 + tid] = __ldg(a.w_cf + tid * 3 + 1);
        s_wf[2 * 64 + tid] = __ldg(a.w_cf + tid * 3 + 2);
        s_bf[tid] = __ldg(a.b_cf + tid);
    }
    int cur_b = -1;
    for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const int b = tile / tiles_per_sample, p0 = (tile - b * tiles_per_sample) * kKbTile;
        const int npts = min(kKbTile, a.N - p0);
        const size_t row0 = (size_t)b * a.N + p0;
        __syncthreads();   // previous tile's readers are done with s_sel (and with the folded weights)
        if (b != cur_b) {
            // per-channel (sum, sum^2) of t_c = w_c . f + b_c over all N*32 candidate vectors, from the moments of f
            if (tid < 64) {
                const double* m = a.moments + (size_t)b * PVRAFT_MOMENTS;
                const double w0 = __ldg(a.w_knn + tid * 4 + 0), w1 = __ldg(a.w_knn + tid * 4 + 1);
                const double w2 = __ldg(a.w_knn + tid * 4 + 2), w3 = __ldg(a.w_knn + tid * 4 + 3);
                const double bc = __ldg(a.b_knn + tid), cnt = m[14];
                const double lin = w0 * m[0] + w1 * m[1] + w2 * m[2] + w3 * m[3];
                const double quad = w0 * w0 * m[4] + w1 * w1 * m[8] + w2 * w2 * m[11] + w3 * w3 * m[13] +
                                    2.0 * (w0 * w1 * m[5] + w0 * w2 * m[6] + w0 * w3 * m[7] + w1 * w2 * m[9] + w1 * w3 * m[10] + w2 * w3 * m[12]);
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
                // GroupNorm affine folded into the convolution: t_norm = (scale*w).f + (scale*b + shift)
                for (int i = 0; i < 4; ++i) s_w[i * 64 + tid] = af.scale * __ldg(a.w_knn + tid * 4 + i);
                s_b[tid] = fmaf(af.scale, __ldg(a.b_knn + tid), af.shift);
            }
            cur_b = b;
        }
        // staged per point as four arrays of 32 (corr, dx, dy, dz): a 128-bit load yields one component of 4 candidates,
        // i.e. two operand pairs for the packed FMA
        for (int i = tid; i < kKbTile * 32; i += kKbThreads) {
            float4 x = make_float4(0.f, 0.f, 0.f, 0.f);
            if ((i >> 5) < npts) x = __ldg(reinterpret_cast<const float4*>(a.knn_sel) + row0 * 32 + i);
            float* dst = s_sel + (i >> 5) * 128 + (i & 31);
            dst[0] = x.x; dst[32] = x.y; dst[64] = x.z; dst[96] = x.w;
        }
        __syncthreads();
        float wk[4][4], bk[4];   // [input i][channel c]
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const float4 t4 = *reinterpret_cast<const float4*>(s_w + i * 64 + tx * 4);
            wk[i][0] = t4.x; wk[i][1] = t4.y; wk[i][2] = t4.z; wk[i][3] = t4.w;
        }
        {
            const float4 t4 = *reinterpret_cast<const float4*>(s_b + tx * 4);
            bk[0] = t4.x; bk[1] = t4.y; bk[2] = t4.z; bk[3] = t4.w;
        }
#pragma unroll
        for (int p = 0; p < 4; ++p) {
            const int pp = ty * 4 + p;
            const float* fp = s_sel + pp * 128;
            float hi[4] = {-INFINITY, -INFINITY, -INFINITY, -INFINITY};
            float lo[4] = {INFINITY, INFINITY, INFINITY, INFINITY};
#pragma unroll 2
            for (int e = 0; e < 32; e += 4) {
                const float4 f0 = *reinterpret_cast<const float4*>(fp + e);        // corr of candidates e..e+3
                const float4 f1 = *reinterpret_cast<const float4*>(fp + 32 + e);   // dx
                const float4 f2 = *reinterpret_cast<const float4*>(fp + 64 + e);   // dy
                const float4 f3 = *reinterpret_cast<const float4*>(fp + 96 + e);   // dz
#pragma unroll
                for (int c = 0; c < 4; ++c) {
                    // t_e = fma(w3, dz, fma(w2, dy, fma(w1, dx, fma(w0, corr, b)))) for two candidates per instruction
                    const float2 b2 = make_float2(bk[c], bk[c]);
                    float2 ta = fma2(make_float2(wk[0][c], wk[0][c]), make_float2(f0.x, f0.y), b2);
                    float2 tb = fma2(make_float2(wk[0][c], wk[0][c]), make_float2(f0.z, f0.w), b2);
                    ta = fma2(make_float2(wk[1][c], wk[1][c]), make_float2(f1.x, f1.y), ta);
                    tb = fma2(make_float2(wk[1][c], wk[1][c]), make_float2(f1.z, f1.w), tb);
                    ta = fma2(make_float2(wk[2][c], wk[2][c]), make_float2(f2.x, f2.y), ta);
                    tb = fma2(make_float2(wk[2][c], wk[2][c]), make_float2(f2.z, f2.w), tb);
                    ta = fma2(make_float2(wk[3][c], wk[3][c]), make_float2(f3.x, f3.y), ta);
                    tb = fma2(make_float2(wk[3][c], wk[3][c]), make_float2(f3.z, f3.w), tb);
                    if (!CONVEX) {
                        ta.x = ta.x >= 0.f ? ta.x : slope * ta.x; ta.y = ta.y >= 0.f ? ta.y : slope * ta.y;
                        tb.x = tb.x >= 0.f ? tb.x : slope * tb.x; tb.y = tb.y >= 0.f ? tb.y : slope * tb.y;
                    }
                    hi[c] = fmaxf(fmaxf(hi[c], fmaxf(ta.x, ta.y)), fmaxf(tb.x, tb.y));
                    if (CONVEX) lo[c] = fminf(fminf(lo[c], fminf(ta.x, ta.y)), fminf(tb.x, tb.y));
                }
            }
            if (CONVEX) {
#pragma unroll
                for (int c = 0; c < 4; ++c) {
                    const float u = hi[c] >= 0.f ? hi[c] : slope * hi[c];
                    const float v = lo[c] >= 0.f ? lo[c] : slope * lo[c];
                    hi[c] = fmaxf(u, v);
                }
            }
            if (pp < npts) {
                *reinterpret_cast<float4*>(a.kfeat + (row0 + pp) * 64 + tx * 4) = make_float4(hi[0], hi[1], hi[2], hi[3]);
                if (a.cflow != nullptr) {
                    const float* fl = a.flow + (row0 + pp) * 3;
                    const float fx = __ldg(fl), fy = __ldg(fl + 1), fz = __ldg(fl + 2);
                    const float4 w0 = *reinterpret_cast<const float4*>(s_wf + 0 * 64 + tx * 4);
                    const float4 w1 = *reinterpret_cast<const float4*>(s_wf + 1 * 64 + tx * 4);
                    const float4 w2 = *reinterpret_cast<const float4*>(s_wf + 2 * 64 + tx * 4);
                    const float4 bf = *reinterpret_cast<const float4*>(s_bf + tx * 4);
                    float4 o;
                    o.x = fmaxf(fmaf(w2.x, fz, fmaf(w1.x, fy, fmaf(w0.x, fx, bf.x))), 0.f);
                    o.y = fmaxf(fmaf(w2.y, fz, fmaf(w1.y, fy, fmaf(w0.y, fx, bf.y))), 0.f);
                    o.z = fmaxf(fmaf(w2.z, fz, fmaf(w1.z, fy, fmaf(w0.z, fx, bf.z))), 0.f);
                    o.w = fmaxf(fmaf(w2.w, fz, fmaf(w1.w, fy, fmaf(w0.w, fx, bf.w))), 0.f);
                    *reinterpret_cast<float4*>(a.cflow + (row0 + pp) * 64 + tx * 4) = o;
                }
            }
        }
    }
}

}  // namespace pvraft

using namespace pvraft;

extern "C" int pvraft_knn_branch_fwd(const pvraft_knn_branch_args* a, void* stream) {
    if (!a || !a->knn_sel || !a->moments || !a->w_knn || !a->b_knn || !a->gnk_gamma || !a->gnk_beta || !a->preluk || !a->kfeat)
        return fail(PVRAFT_ERR_BAD_ARG, "knn_branch: null pointer");
    if ((a->cflow != nullptr) != (a->flow != nullptr) || (a->cflow && (!a->w_cf || !a->b_cf)))
        return fail(PVRAFT_ERR_BAD_ARG, "knn_branch: flow, w_cf, b_cf and cflow go together");
    if (a->B <= 0 || a->N <= 0) return fail(PVRAFT_ERR_BAD_ARG, "knn_branch: bad shape");
    // the convexity shortcut needs the (learned) PReLU slope on the host
    float slope = a->preluk_host;
    if (slope != slope) {
        cudaError_t e = cudaMemcpyAsync(&slope, a->preluk, sizeof(float), cudaMemcpyDeviceToHost, (cudaStream_t)stream);
        if (e == cudaSuccess) e = cudaStreamSynchronize((cudaStream_t)stream);
        if (e != cudaSuccess) return fail((int)e, "knn_branch: reading the PReLU slope failed: %s", cudaGetErrorString(e));
    }
    const long long n_tiles = (long long)a->B * ((a->N + kKbTile - 1) / kKbTile);
    int per_sm = 0;
    if (slope <= 1.f) cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_knn_branch<true>, kKbThreads, 0);
    else cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_knn_branch<false>, kKbThreads, 0);
    const long long cap = (long long)sm_count() * (per_sm > 0 ? per_sm : 1);
    const int grid = (int)(n_tiles < cap ? n_tiles : cap);
    if (slope <= 1.f) launch_pdl(k_knn_branch<true>, grid, kKbThreads, 0, (cudaStream_t)stream, *a);
    else launch_pdl(k_knn_branch<false>, grid, kKbThreads, 0, (cudaStream_t)stream, *a);
    return check_launch("knn_branch");
}
