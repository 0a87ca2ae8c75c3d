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
#pragma once
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

// dst[i] += v: an fp32 atomic, or (DET) an exact addition into slot i of the fixed-point workspace dst
template <bool DET>
__device__ __forceinline__ void scatter_add(float* dst, long long i, float v) {
    if constexpr (DET) fx_atomic(reinterpret_cast<unsigned long long*>(dst) + i * kFxWords, (double)v);
    else atomicAdd(dst + i, v);
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
int fx_flush_f64(const unsigned long long* acc, long long rows, long long cols, long long acc_ld, long long ld, double* out, cudaStream_t st);
int fx_flush_f32(const unsigned long long* acc, long long rows, long long cols, long long acc_ld, long long ld, float* out, cudaStream_t st);

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
