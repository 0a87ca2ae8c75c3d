// Read-out of the fixed-point accumulators (fixed_point.cuh): one thread per slot, a single writer per output entry.
#include "fixed_point.cuh"

namespace pvraft {

template <typename T>
__global__ void k_fx_flush(const unsigned long long* __restrict__ acc, long long rows, long long cols, long long acc_ld, long long ld,
                           T* __restrict__ out) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= rows * cols) return;
    const long long r = i / cols, c = i - r * cols;
    T* o = out + r * ld + c;
    *o = *o + (T)fx_value(acc + (r * acc_ld + c) * kFxWords);
}

template <typename T>
static int flush(const unsigned long long* acc, long long rows, long long cols, long long acc_ld, long long ld, T* out, cudaStream_t st) {
    const long long n = rows * cols;
    if (n <= 0) return PVRAFT_OK;
    k_fx_flush<T><<<(unsigned)((n + 255) / 256), 256, 0, st>>>(acc, rows, cols, acc_ld, ld, out);
    return check_launch("fx_flush");
}

int fx_flush(FxSlots acc, long long rows, long long cols, long long acc_ld, long long ld, double* out, cudaStream_t st) {
    return flush(acc.base, rows, cols, acc_ld, ld, out, st);
}

int fx_flush(FxSlots acc, long long rows, long long cols, long long acc_ld, long long ld, float* out, cudaStream_t st) {
    return flush(acc.base, rows, cols, acc_ld, ld, out, st);
}

}  // namespace pvraft
