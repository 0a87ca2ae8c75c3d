// Per-row top-K of the dense correlation matrix: the truncation step of CorrBlock.init_module
// (reference model/corr.py:37-40, torch.topk(corr, k, dim=2, sorted=True)).
//
// One CTA per row.  The row is staged once in shared memory as order-preserving uint32 keys (one pad word
// per 32 so that a thread can later walk its own 32-key segment without bank conflicts); the K-th largest
// key is found by a 4-pass (8 bits per pass) radix select on shared-memory histograms; then every thread
// counts the survivors of its segment, one block scan gives it its output offset, and the K survivors are
// written in ASCENDING COLUMN order (ties at the threshold: lowest columns win).  The reference sorts the K
// values descending; nothing downstream depends on that order (pvraft_corr_reorder rearranges every row
// anyway), so the sort is not done here -- CorrBlock.truncated_corr sorts on demand for API parity.
// The same kernels run the two steps of the windowed build of large clouds (pvraft_corr_topk_window_fwd): the top-K of
// each column window of a slab, and the merge of a row's per-window candidate lists through their stored column ids.
#include "common.cuh"

namespace pvraft {

constexpr int kTopkThreads = 256;

__device__ __forceinline__ int padded(int i) { return i + (i >> 5); }

// Both kernels read M columns of row r at corr + r * ld and write its K survivors to val / idx + r * ld_out; the id of column j
// is ids[r * ld + j] when an id map is given (a candidate list), col_base + j otherwise.
__global__ void __launch_bounds__(kTopkThreads) k_corr_topk(const float* __restrict__ corr, int M, long long ld, int K,
                                                            float* __restrict__ val, int32_t* __restrict__ idx, long long ld_out,
                                                            int col_base, const int32_t* __restrict__ ids) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    unsigned* s_key = reinterpret_cast<unsigned*>(smem_raw);   // [padded(M)]
    __shared__ int s_hist[256];
    __shared__ unsigned s_prefix, s_need;
    __shared__ unsigned s_warp[kTopkThreads / 32];
    const size_t row = blockIdx.x;
    const float* src = corr + row * (size_t)ld;
    const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
    for (int i = tid; i < M; i += kTopkThreads) s_key[padded(i)] = ord_key(__ldg(src + i));
    if (tid == 0) { s_prefix = 0u; s_need = (unsigned)K; }
    // ---- radix select: after pass p the top 8*(p+1) bits of the K-th largest key are known --------------
    for (int pass = 0; pass < 4; ++pass) {
        const int shift = 24 - 8 * pass;
        s_hist[tid] = 0;
        __syncthreads();
        const unsigned prefix = s_prefix;
        const unsigned mask = pass == 0 ? 0u : (0xFFFFFFFFu << (shift + 8));
        for (int i = tid; i < M; i += kTopkThreads) {
            const unsigned k = s_key[padded(i)];
            if ((k & mask) == prefix) atomicAdd(&s_hist[(k >> shift) & 0xFF], 1);
        }
        __syncthreads();
        if (w == 0) {
            // lane l owns bins 8l .. 8l+7; suffix sums locate the bin holding the `need`-th largest key
            int h[8], mine = 0;
#pragma unroll
            for (int q = 0; q < 8; ++q) { h[q] = s_hist[lane * 8 + q]; mine += h[q]; }
            int above = mine;   // inclusive suffix sum over lanes >= l
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const int a = __shfl_down_sync(kFull, above, o);
                if (lane + o < 32) above += a;
            }
            const int need = (int)s_need;
            const int higher = above - mine;   // keys in bins owned by higher lanes
            const bool here = higher < need && above >= need;
            if (here) {
                int acc = higher, bin = 7;
                for (; bin > 0; --bin) {
                    if (acc + h[bin] >= need) break;
                    acc += h[bin];
                }
                s_need = (unsigned)(need - acc);          // rank of the target inside the chosen bin
                s_prefix = prefix | ((unsigned)(lane * 8 + bin) << shift);
            }
        }
        __syncthreads();
    }
    const unsigned T = s_prefix;       // exact K-th largest key
    const int need_eq = (int)s_need;   // how many keys == T belong to the top-K (lowest columns first)
    // ---- ordered compaction: thread t owns columns [t*seg, (t+1)*seg) ----------------------------------------
    const int seg = (M + kTopkThreads - 1) / kTopkThreads;
    const int c0 = tid * seg, c1 = min(M, c0 + seg);
    unsigned n_gt = 0, n_eq = 0;
    for (int i = c0; i < c1; ++i) {
        const unsigned k = s_key[padded(i)];
        n_gt += k > T ? 1u : 0u;
        n_eq += k == T ? 1u : 0u;
    }
    // block exclusive scan of (n_gt | n_eq << 16): M <= 49152 keeps both fields below 65536
    unsigned packed = n_gt | (n_eq << 16), incl = packed;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const unsigned a = __shfl_up_sync(kFull, incl, o);
        if (lane >= o) incl += a;
    }
    if (lane == 31) s_warp[w] = incl;
    __syncthreads();
    unsigned base = 0;
    for (int q = 0; q < w; ++q) base += s_warp[q];
    const unsigned excl = base + incl - packed;
    const int gt_before = (int)(excl & 0xFFFFu), eq_before = (int)(excl >> 16);
    // output position = (# kept elements in lower columns) = gt_before + min(eq_before, need_eq)
    int pos = gt_before + min(eq_before, need_eq);
    int eq_seen = eq_before;
    for (int i = c0; i < c1; ++i) {
        const unsigned k = s_key[padded(i)];
        bool keep = k > T;
        if (k == T) { keep = eq_seen < need_eq; ++eq_seen; }
        if (keep) {
            val[row * ld_out + pos] = ord_float(k);
            idx[row * ld_out + pos] = ids ? __ldg(ids + row * ld + i) : col_base + i;
            ++pos;
        }
    }
}

// ---------------------------------------------------------------------------------------------------------
// Variant for M <= 8192, M % 4 == 0 (the model's case).  The row is staged once as order-preserving keys, 16 bytes per
// thread and step (thread t owns the float4 columns j*256 + t: coalesced global loads, conflict-free 128-bit shared
// loads); the K-th largest key is found with three radix passes (11 + 11 + 10 bits) of which only the first counts every
// key; the ordered compaction scans packed per-chunk counts (11-bit fields) across the block.
// ---------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kTopkThreads) k_corr_topk_vec(const float* __restrict__ corr, int M, long long ld, int K,
                                                                float* __restrict__ val, int32_t* __restrict__ idx, long long ld_out,
                                                                int col_base, const int32_t* __restrict__ ids) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    uint4* s_key = reinterpret_cast<uint4*>(smem_raw);   // [8 * 256]
    constexpr int kCand = 1024;                          // capacity of the candidate list of the second and third pass
    __shared__ int s_hist[2048 + kTopkThreads];          // 2048 bins + one private sink per thread (see below)
    __shared__ unsigned s_cand[kCand];
    __shared__ int s_wsum[kTopkThreads / 32];
    __shared__ unsigned s_scan[kTopkThreads / 32][7];
    __shared__ unsigned s_prefix;
    __shared__ int s_need;
    const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
    const size_t row = blockIdx.x;
    const float4* src = reinterpret_cast<const float4*>(corr + row * (size_t)ld);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const int c4 = j * kTopkThreads + tid;
        uint4 kk = make_uint4(0u, 0u, 0u, 0u);   // padding: below every real key, never selected (K <= M)
        if (c4 * 4 < M) {
            const float4 v = __ldg(src + c4);
            kk = make_uint4(ord_key(v.x), ord_key(v.y), ord_key(v.z), ord_key(v.w));
        }
        s_key[c4] = kk;
    }
    // ---- radix select, 11 + 11 + 10 bits (each thread only ever reads the keys it wrote) ----
    // Only the first pass looks at every key.  Its increments are UNCONDITIONAL shared-memory atomics -- keys that do not take
    // part add to the thread's private sink bin instead of being skipped, because an `if` around a shared-memory atomic
    // compiles to a branch + reconvergence per key.  The keys that fall into the bin of the K-th largest (a few hundred of
    // 8192) are then collected once, and the second and third pass run over that list; a list overflow (more than 1024
    // keys share their top 11 bits: near-constant rows) falls back to scanning the row again.
    const int sink = 2048 + tid;
    // locate, with block-wide suffix sums over the 2048 bins, the bin holding the need-th largest counted key
    auto find_bin = [&](unsigned prefix, int shift, int need) {
        int h[8], mine = 0;   // thread t owns bins 8t .. 8t+7
#pragma unroll
        for (int q = 0; q < 8; ++q) { h[q] = s_hist[tid * 8 + q]; mine += h[q]; }
        int incl = mine;   // inclusive suffix sum over the lanes >= lane of this warp
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int a = __shfl_down_sync(kFull, incl, o);
            if (lane + o < 32) incl += a;
        }
        if (lane == 0) s_wsum[w] = incl;
        __syncthreads();
        int above = incl;
        for (int ww = w + 1; ww < kTopkThreads / 32; ++ww) above += s_wsum[ww];
        const int higher = above - mine;   // keys in bins owned by higher threads
        if (higher < need && above >= need) {
            int acc = higher, bin = 7;
            for (; bin > 0; --bin) {
                if (acc + h[bin] >= need) break;
                acc += h[bin];
            }
            s_need = need - acc;   // rank of the target inside the chosen bin
            s_prefix = prefix | ((unsigned)(tid * 8 + bin) << shift);
        }
        __syncthreads();
    };
    for (int i = tid; i < 2048; i += kTopkThreads) s_hist[i] = 0;
    __syncthreads();
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const uint4 kk = s_key[j * kTopkThreads + tid];
        atomicAdd(&s_hist[kk.x >> 21], 1);
        atomicAdd(&s_hist[kk.y >> 21], 1);
        atomicAdd(&s_hist[kk.z >> 21], 1);
        atomicAdd(&s_hist[kk.w >> 21], 1);
    }
    __syncthreads();
    find_bin(0u, 21, K);
    unsigned prefix = s_prefix;
    int need = s_need;
    int ncand = 0;
    {   // candidates of the remaining passes: keys whose top 11 bits equal the chosen bin
        // (count, block scan, predicated stores: a per-key `if { atomicAdd; store }` costs a divergent branch per key)
        const unsigned top = prefix >> 21;
        int mine = 0;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const uint4 kk = s_key[j * kTopkThreads + tid];
            mine += ((kk.x >> 21) == top) + ((kk.y >> 21) == top) + ((kk.z >> 21) == top) + ((kk.w >> 21) == top);
        }
        int incl = mine;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int a = __shfl_up_sync(kFull, incl, o);
            if (lane >= o) incl += a;
        }
        if (lane == 31) s_wsum[w] = incl;
        __syncthreads();
        int at = incl - mine, total = 0;
        for (int ww = 0; ww < kTopkThreads / 32; ++ww) {
            const int a = s_wsum[ww];
            total += a;
            if (ww < w) at += a;
        }
        ncand = total;   // (the same value in every thread)
        if (total <= kCand && mine > 0) {
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const uint4 kk = s_key[j * kTopkThreads + tid];
                const unsigned ke[4] = {kk.x, kk.y, kk.z, kk.w};
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const bool hit = (ke[e] >> 21) == top;
                    if (hit) s_cand[at] = ke[e];
                    at += hit ? 1 : 0;
                }
            }
        }
    }
    __syncthreads();
#pragma unroll 1
    for (int pass = 1; pass < 3; ++pass) {
        const int shift = pass == 1 ? 10 : 0;
        const unsigned digit_mask = pass == 1 ? 0x7FFu : 0x3FFu;
        const unsigned hi_mask = 0xFFFFFFFFu << (shift + (pass == 1 ? 11 : 10));
        for (int i = tid; i < 2048; i += kTopkThreads) s_hist[i] = 0;
        __syncthreads();
        if (ncand <= kCand) {
            for (int i = tid; i < ncand; i += kTopkThreads) {
                const unsigned k = s_cand[i];
                atomicAdd(&s_hist[(k & hi_mask) == prefix ? (int)((k >> shift) & digit_mask) : sink], 1);
            }
        } else {
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const uint4 kk = s_key[j * kTopkThreads + tid];
                atomicAdd(&s_hist[(kk.x & hi_mask) == prefix ? (int)((kk.x >> shift) & digit_mask) : sink], 1);
                atomicAdd(&s_hist[(kk.y & hi_mask) == prefix ? (int)((kk.y >> shift) & digit_mask) : sink], 1);
                atomicAdd(&s_hist[(kk.z & hi_mask) == prefix ? (int)((kk.z >> shift) & digit_mask) : sink], 1);
                atomicAdd(&s_hist[(kk.w & hi_mask) == prefix ? (int)((kk.w >> shift) & digit_mask) : sink], 1);
            }
        }
        __syncthreads();
        find_bin(prefix, shift, need);
        prefix = s_prefix;
        need = s_need;
    }
    const unsigned T = prefix;   // exact K-th largest key
    const int need_eq = need;    // how many keys == T belong to the top-K (lowest columns first)
    // ---- ordered compaction: chunk j = columns [1024 j, 1024 j + 1024), inside a chunk thread order = column order ----
    // words 0-2: keys > T per chunk in 11-bit fields (at most K - 1 <= 1023 keys exceed T, so no field overflows);
    // words 3-6: keys == T per chunk in 16-bit fields (a whole 1024-key chunk may tie with T: 11 bits at shift 22 would wrap)
    unsigned cnt[7] = {0u, 0u, 0u, 0u, 0u, 0u, 0u};
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const uint4 kk = s_key[j * kTopkThreads + tid];
        const unsigned g = (kk.x > T) + (kk.y > T) + (kk.z > T) + (kk.w > T);
        const unsigned q = (kk.x == T) + (kk.y == T) + (kk.z == T) + (kk.w == T);
        cnt[j / 3] += g << (11 * (j % 3));
        cnt[3 + j / 2] += q << (16 * (j % 2));
    }
    unsigned inc[7];
#pragma unroll
    for (int i = 0; i < 7; ++i) inc[i] = cnt[i];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
#pragma unroll
        for (int i = 0; i < 7; ++i) {
            const unsigned a = __shfl_up_sync(kFull, inc[i], o);
            if (lane >= o) inc[i] += a;
        }
    }
    if (lane == 31) {
#pragma unroll
        for (int i = 0; i < 7; ++i) s_scan[w][i] = inc[i];
    }
    __syncthreads();
    unsigned tot[7] = {0u, 0u, 0u, 0u, 0u, 0u, 0u}, before[7];
#pragma unroll
    for (int i = 0; i < 7; ++i) before[i] = inc[i] - cnt[i];   // exclusive within the warp
    for (int ww = 0; ww < kTopkThreads / 32; ++ww) {
#pragma unroll
        for (int i = 0; i < 7; ++i) {
            const unsigned a = s_scan[ww][i];
            tot[i] += a;
            if (ww < w) before[i] += a;
        }
    }
    // Only ~K/M of the keys are kept: a float4 group without any key >= T (3 in 4 groups at K/M = 1/16) is skipped on its
    // packed counts alone, and the surviving groups store through a per-row base pointer.
    // The kept keys go to their output position in a shared-memory staging row first (the candidate list and the histogram
    // are dead by now) and leave with coalesced stores; the scattered 4-byte global stores this replaces cost ~25
    // instructions per kept key.
    __syncthreads();
    unsigned* s_oval = s_cand;                                  // [K <= 1024] keys
    int* s_oidx = s_hist;                                       // [K <= 1024] columns
    int base_gt = 0, base_eq = 0;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const int sh = 11 * (j % 3), sq = 16 * (j % 2);
        int gt_before = base_gt + (int)((before[j / 3] >> sh) & 0x7FFu);
        int eq_before = base_eq + (int)((before[3 + j / 2] >> sq) & 0xFFFFu);
        base_gt += (int)((tot[j / 3] >> sh) & 0x7FFu);
        base_eq += (int)((tot[3 + j / 2] >> sq) & 0xFFFFu);
        const unsigned mine = ((cnt[j / 3] >> sh) & 0x7FFu) | ((cnt[3 + j / 2] >> sq) & 0xFFFFu);   // any key >= T in this group?
        if (mine == 0u) continue;
        const int col = (j * kTopkThreads + tid) * 4;
        const uint4 kk = s_key[j * kTopkThreads + tid];
        const unsigned ke[4] = {kk.x, kk.y, kk.z, kk.w};
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const unsigned key = ke[e];
            const bool gt = key > T, eq = key == T;
            if (gt || (eq && eq_before < need_eq)) {
                const int pos = gt_before + min(eq_before, need_eq);
                s_oval[pos] = key;
                s_oidx[pos] = col + e;
            }
            gt_before += gt ? 1 : 0;
            eq_before += eq ? 1 : 0;
        }
    }
    __syncthreads();
    float* vrow = val + row * (size_t)ld_out;
    int32_t* irow = idx + row * (size_t)ld_out;
    const int32_t* idrow = ids ? ids + row * (size_t)ld : nullptr;
    for (int i = tid; i < K; i += kTopkThreads) {
        vrow[i] = ord_float(s_oval[i]);
        irow[i] = idrow ? __ldg(idrow + s_oidx[i]) : col_base + s_oidx[i];
    }
}

static int launch_topk(const float* corr, long long rows, int M, long long ld, int K, int col_base, const int32_t* ids, float* val,
                       int32_t* idx, long long ld_out, cudaStream_t st) {
    if (M <= 8192 && M % 4 == 0 && ld % 4 == 0 && (uintptr_t)corr % 16 == 0) {
        k_corr_topk_vec<<<(unsigned)rows, kTopkThreads, 8 * kTopkThreads * sizeof(uint4), st>>>(corr, M, ld, K, val, idx, ld_out, col_base, ids);
        return check_launch("corr_topk");
    }
    const size_t smem = (size_t)(M + (M >> 5) + 4) * 4;
    int rc;
    if ((rc = opt_in_smem(k_corr_topk, smem))) return rc;
    k_corr_topk<<<(unsigned)rows, kTopkThreads, smem, st>>>(corr, M, ld, K, val, idx, ld_out, col_base, ids);
    return check_launch("corr_topk");
}

}  // namespace pvraft

using namespace pvraft;

extern "C" int pvraft_corr_topk_fwd(const float* corr, int B, int N, int M, int K, float* val, int32_t* idx, void* stream) {
    if (!corr || !val || !idx) return fail(PVRAFT_ERR_BAD_ARG, "corr_topk: null pointer");
    if (B <= 0 || N <= 0 || M <= 0) return fail(PVRAFT_ERR_BAD_ARG, "corr_topk: bad shape");
    if (K < 1 || K > M || K > 1024) return fail(PVRAFT_ERR_UNSUPPORTED, "corr_topk: K=%d with M=%d (need 1 <= K <= min(M,1024))", K, M);
    if (M > 49152) return fail(PVRAFT_ERR_UNSUPPORTED, "corr_topk: M=%d columns (max 49152)", M);
    const long long rows = (long long)B * N;
    if (rows > 0x7fffffffLL) return fail(PVRAFT_ERR_UNSUPPORTED, "corr_topk: too many rows");
    return launch_topk(corr, rows, M, M, K, 0, nullptr, val, idx, K, (cudaStream_t)stream);
}

extern "C" int pvraft_corr_topk_window_fwd(const float* corr, int rows, int cols, int64_t ld, int K, int col_base, const int32_t* cand_ids,
                                           float* val, int32_t* idx, int64_t ld_out, void* stream) {
    if (!corr || !val || !idx) return fail(PVRAFT_ERR_BAD_ARG, "corr_topk_window: null pointer");
    if (rows <= 0 || cols <= 0 || ld < cols || col_base < 0) return fail(PVRAFT_ERR_BAD_ARG, "corr_topk_window: bad shape");
    if (K < 1 || K > cols || K > 1024 || ld_out < K)
        return fail(PVRAFT_ERR_UNSUPPORTED, "corr_topk_window: K=%d with cols=%d, ld_out=%lld (need 1 <= K <= min(cols,1024), ld_out >= K)", K,
                    cols, (long long)ld_out);
    if (cols > 49152) return fail(PVRAFT_ERR_UNSUPPORTED, "corr_topk_window: cols=%d (max 49152)", cols);
    if (!cand_ids && (long long)col_base + cols > 0x7fffffffLL) return fail(PVRAFT_ERR_UNSUPPORTED, "corr_topk_window: column ids overflow");
    return launch_topk(corr, rows, cols, ld, K, col_base, cand_ids, val, idx, ld_out, (cudaStream_t)stream);
}
