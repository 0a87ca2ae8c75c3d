// TMA engine and mbarrier primitives of the Hopper kernels (corr_gemm.cu, corr_lookup.cu, tc_linear.cu, update_chain.cu),
// and the host encoder of their tensor maps.
#pragma once
#include <cuda.h>

#include "common.cuh"

namespace pvraft {

// ---- host -----------------------------------------------------------------------------------------------
// [rows, cols] fp32 row-major (row stride ld floats) -> `map`: boxes of box_rows x 32 columns (one 128-byte swizzle row),
// SWIZZLE_128B.  Error messages start with `op` (definition in capi.cu).
int make_tensor_map(CUtensorMap* map, const float* base, long long rows, int cols, long long ld, int box_rows, const char* op);
// the same for a bf16 tensor (row stride ld elements): boxes of box_rows x 32 columns (one 64-byte swizzle row), SWIZZLE_64B
int make_tensor_map_bf16(CUtensorMap* map, const uint16_t* base, long long rows, int cols, long long ld, int box_rows, const char* op);

// ---- device ---------------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }

// the dynamic shared array rounded up to the 1024-byte alignment of SWIZZLE_128B tiles, by pointer arithmetic on the shared
// array: an integer round trip would lose the address space and turn every shared-memory access into a generic LD/ST.
// A macro: as an inline function, the same expression changes the machine code of the kernels that use it.
#define SMEM_ALIGN_1024(smem_raw) ((smem_raw) + ((1024u - ((unsigned)__cvta_generic_to_shared(smem_raw) & 1023u)) & 1023u))

__device__ __forceinline__ void mbar_init(void* bar, unsigned count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
// makes the barrier initialisations above visible to the other threads and to the TMA engine
__device__ __forceinline__ void fence_mbarrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(void* bar, unsigned bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(void* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// spins until the phase with parity `parity` of the barrier has completed
__device__ __forceinline__ void mbar_wait(void* bar, unsigned parity) {
    asm volatile(
        "{\n\t.reg .pred P1;\n\t"
        "WAIT_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n\t"
        "@P1 bra DONE_%=;\n\t"
        "bra WAIT_%=;\n\t"
        "DONE_%=:\n\t}" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}

__device__ __forceinline__ void prefetch_tensormap(const CUtensorMap* map) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(map) : "memory");
}
// the box at (column c0, row c1) of a 2-D tensor map -> dst, its bytes counted as transactions on bar
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* map, void* bar, int c0, int c1) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(smem_u32(dst)),
                 "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
                 : "memory");
}
// `bytes` (a multiple of 16) contiguous bytes global -> shared by the bulk-copy engine, counted as transactions on bar
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, unsigned bytes, void* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)),
                 "l"(src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}

// Position of one pipeline role in the (tile, k-block) walk and in the operand ring; advanced without divisions (a
// runtime integer division is a ~100-cycle dependent chain, paid per step by warps that have nothing to hide it behind)
struct TcCursor {
    int ti = 0, kb = 0, s = 0;
    unsigned phase = 0;
    __device__ __forceinline__ void next(int num_kb, int S) {
        if (++kb == num_kb) { kb = 0; ++ti; }
        if (++s == S) { s = 0; phase ^= 1u; }
    }
};

}  // namespace pvraft
