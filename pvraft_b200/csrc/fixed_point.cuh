// Exact fixed-point accumulation for the deterministic instantiations of the reducing kernels (the library's form of
// torch.use_deterministic_algorithms(True); include/pvraft_b200.h, "Deterministic mode").
//
// A slot holds a signed Q64.64 number -- value = (hi * 2^64 + lo) * 2^-64 in 128-bit two's complement -- plus a flag word:
// three 64-bit words.  A contribution enters as fx_from(v): |v| truncated toward zero to a multiple of 2^-64.  From then on
// every addition is an integer addition (the low word's carry is propagated with the returned old value), which is exact,
// so the final bits do not depend on the order of the additions: not on the grid size, the SM count, which warp claimed
// which point, or timing.  What the kernels must keep fixed is only WHAT enters: each contribution is a value whose own
// floating-point evaluation order is a function of the shapes (one point, one 128-point tile, one warp's rows, ...).
//
// Error.  The bound is ABSOLUTE, not relative: every contribution is truncated toward zero to a multiple of 2^-64 (5.4e-20),
// so a term smaller than that vanishes and a sum of n terms can be off by up to n * 2^-64 -- which is large relative to a
// sum of tiny terms (gradients of ~1e-15 summed over ~1e6 terms), and negligible for the magnitudes this model produces.
// fx_value then rounds the exact 128-bit sum to double once (round to nearest even); the flush adds that double to the
// destination, which rounds once more (in fp32 for fp32 destinations).  The range is |sum| < 2^63; a contribution that is
// not finite or has |v| >= 2^62 sets the flag, and the slot reads back as NaN.
//
// The shared code every reducing kernel uses:
//   FxSlots, Acc<DET, T>  a typed destination: a kernel declares its accumulating parameters Acc<DET, T> -- T* in the default
//                         instantiation, FxSlots (slots of the caller's workspace) in the DET one -- and adds with add(dst, i, v),
//                         an atomicAdd or an exact fixed-point addition.  Structs whose layout the default kernels share carry
//                         the workspace in their T* field and convert it with fx_slots().
//   fx_stage_zero/flush   a CTA's slots staged in shared memory: zeroed, and later added into the global slots (empty ones
//                         skipped), by the CTA or by the first `nt` threads of it.
//   FxCarve               the host's description of a workspace as consecutive named slot ranges; the size query of an entry
//                         point and its launcher run the same description.  fx_flush adds the slots into the real destination.
#pragma once
#include <type_traits>
#include "common.cuh"

namespace pvraft {

constexpr int kFxWords = 3;   // lo, hi, flag

struct Fx {
    unsigned long long lo, hi;
    unsigned bad;
};

__device__ __forceinline__ Fx fx_from(double v) {
    Fx r{0ull, 0ull, 0u};
    const double a = fabs(v);
    if (!(a < 0x1p62)) { r.bad = 1u; return r; }   // also catches NaN
    const double ip = floor(a);
    r.hi = (unsigned long long)ip;
    r.lo = (unsigned long long)((a - ip) * 0x1p64);   // a - ip is exact and < 1
    if (v < 0.0) {
        r.lo = ~r.lo + 1ull;
        r.hi = ~r.hi + (r.lo == 0ull ? 1ull : 0ull);
    }
    return r;
}

__device__ __forceinline__ void fx_add(Fx& a, const Fx& b) {
    const unsigned long long lo = a.lo + b.lo;
    a.hi += b.hi + (lo < a.lo ? 1ull : 0ull);
    a.lo = lo;
    a.bad |= b.bad;
}

// slot: kFxWords words in shared or global memory
__device__ __forceinline__ void fx_atomic(unsigned long long* slot, const Fx& v) {
    unsigned long long carry = 0ull;
    if (v.lo) {
        const unsigned long long old = atomicAdd(slot, v.lo);
        carry = old + v.lo < old ? 1ull : 0ull;
    }
    const unsigned long long h = v.hi + carry;
    if (h) atomicAdd(slot + 1, h);
    if (v.bad) atomicOr(slot + 2, 1ull);
}

__device__ __forceinline__ void fx_atomic(unsigned long long* slot, double v) { fx_atomic(slot, fx_from(v)); }

__device__ __forceinline__ Fx fx_load(const unsigned long long* slot) { return Fx{slot[0], slot[1], (unsigned)slot[2]}; }

// kFxWords-word slots in global or shared memory: slot i starts at base + i * kFxWords
struct FxSlots {
    unsigned long long* base;
    __host__ __device__ explicit operator bool() const { return base != nullptr; }
};
__host__ __device__ __forceinline__ FxSlots operator+(FxSlots s, long long i) { return FxSlots{s.base + i * kFxWords}; }
// the workspace carried in a T* field of a struct that the default instantiation shares
__host__ __device__ __forceinline__ FxSlots fx_slots(const void* ws) {
    return FxSlots{static_cast<unsigned long long*>(const_cast<void*>(ws))};
}

// an accumulating parameter: the real destination, or (DET) slots of the fixed-point workspace
template <bool DET, typename T = float>
using Acc = std::conditional_t<DET, FxSlots, T* __restrict__>;

// dst[i] += v: an atomic, or an exact addition into slot i
__device__ __forceinline__ void add(float* dst, long long i, float v) { atomicAdd(dst + i, v); }
__device__ __forceinline__ void add(double* dst, long long i, double v) { atomicAdd(dst + i, v); }
__device__ __forceinline__ void add(FxSlots dst, long long i, double v) { fx_atomic(dst.base + i * kFxWords, v); }
__device__ __forceinline__ void add(FxSlots dst, long long i, const Fx& v) { fx_atomic(dst.base + i * kFxWords, v); }

// a CTA's n slots staged in shared memory (s), handled by its threads below nt: zero them before the first shared add, and
// add them into the n global slots g, skipping empty ones, after the last (each behind a barrier of those threads)
__device__ __forceinline__ void fx_stage_zero(FxSlots s, int n, int nt = blockDim.x) {
    for (int i = threadIdx.x; i < n * kFxWords; i += nt) s.base[i] = 0ull;
}
__device__ __forceinline__ void fx_stage_flush(FxSlots s, int n, FxSlots g, int nt = blockDim.x) {
    for (int i = threadIdx.x; i < n; i += nt) {
        const Fx v = fx_load(s.base + i * kFxWords);
        if (v.lo || v.hi || v.bad) fx_atomic(g.base + i * kFxWords, v);
    }
}

__device__ __forceinline__ double fx_value(const unsigned long long* slot) {
    if (slot[2]) return __longlong_as_double(0x7ff8000000000000ll);
    unsigned long long lo = slot[0], hi = slot[1];
    const bool neg = (long long)hi < 0;
    if (neg) {
        lo = ~lo + 1ull;
        hi = ~hi + (lo == 0ull ? 1ull : 0ull);
    }
    double r;
    if (hi == 0ull) {
        r = __ull2double_rn(lo) * 0x1p-64;   // one rounding; the power-of-two scale is exact
    } else {
        // the top 64 bits of the 128-bit magnitude, with every bit below them folded into bit 0 (a sticky bit: the 11 bits
        // a 64 -> 53-bit rounding drops decide the rounding, and a nonzero remainder must break a tie upward), then one rounding
        const int s = __clzll((long long)hi);
        const unsigned long long top = s ? (hi << s) | (lo >> (64 - s)) : hi;
        const unsigned long long rest = s ? lo << s : lo;
        r = ldexp(__ull2double_rn(top | (rest != 0ull ? 1ull : 0ull)), -s);   // top * 2^(64 - s) * 2^-64
    }
    return neg ? -r : r;
}

// out[r * ld + c] += value of slot (r * acc_ld + c), for r < rows, c < cols (a separate launch after the accumulating kernel)
int fx_flush(FxSlots acc, long long rows, long long cols, long long acc_ld, long long ld, double* out, cudaStream_t st);
int fx_flush(FxSlots acc, long long rows, long long cols, long long acc_ld, long long ld, float* out, cudaStream_t st);
// out[i] += value of slot i, for i < n
template <typename T>
inline int fx_flush(FxSlots acc, long long n, T* out, cudaStream_t st) { return fx_flush(acc, 1, n, n, 0, out, st); }

inline int64_t fx_bytes(long long slots) { return slots * kFxWords * 8; }

// Host: a workspace carved into consecutive slot ranges, in the order of the take() calls.  Carving a null workspace only
// counts, so that an entry point's size query and its launcher share one description.
struct FxCarve {
    unsigned long long* base;
    long long slots = 0;
    explicit FxCarve(void* ws) : base(static_cast<unsigned long long*>(ws)) {}
    FxSlots take(long long n) {
        const FxSlots r{base ? base + slots * kFxWords : nullptr};
        slots += n;
        return r;
    }
    int64_t bytes() const { return fx_bytes(slots); }
};

// Host: a workspace carved into consecutive byte ranges, each starting 16-byte aligned, in the order of the take() calls;
// a null base only counts (bytes: the size so far)
struct ByteCarve {
    char* base;
    int64_t bytes = 0;
    explicit ByteCarve(void* ws) : base(static_cast<char*>(ws)) {}
    template <typename T>
    T* take(int64_t n) {
        T* r = reinterpret_cast<T*>(base ? base + bytes : nullptr);
        bytes += (n + 15) / 16 * 16;
        return r;
    }
};

// The [B,16] GroupNorm statistics (slot b * 16 + 2 * group + moment) of k_linear, k_tc_linear, k_setconv_edge_pairs and
// k_edge_fwd
inline int64_t gn_stats_ws_bytes(int B) { return fx_bytes(16ll * B); }
inline int gn_stats_flush(void* ws, int B, double* stats, cudaStream_t st) { return fx_flush(fx_slots(ws), 16ll * B, stats, st); }

// The weight gradients of k_linear_wgrad, k_linear_bwd_small and k_tc_wgrad: [cout][cin] weight slots | [cout] bias slots
struct WgradWs {
    FxSlots w, b;
    int64_t bytes;
};
inline WgradWs wgrad_ws(void* ws, int cin, int cout) {
    FxCarve c(ws);
    return {c.take((long long)cout * cin), c.take(cout), c.bytes()};
}
// dW[o * ld + i] += slot (o, i), db[o] += slot o (db may be null)
inline int wgrad_flush(const WgradWs& L, int cin, int cout, int ld, float* dW, float* db, cudaStream_t st) {
    const int rc = fx_flush(L.w, cout, cin, cin, ld, dW, st);
    return rc || !db ? rc : fx_flush(L.b, cout, db, st);
}
// grid caps of the deterministic instantiations: constants, so that the rows a CTA or thread sums depend on the shapes only
constexpr long long kDetCtas = 256;

// CTAs of 256 threads for a grid-stride scatter over `items`: capped by kDetCtas in the deterministic form, by 8 per SM
// otherwise
inline long long scatter_blocks(long long items, bool det) {
    long long blocks = (items + 255) / 256;
    const long long cap = det ? kDetCtas : (long long)sm_count() * 8;
    return blocks > cap ? cap : blocks;
}

}  // namespace pvraft
