// Shared device helpers for libgptq_b200 (sm_90a only).
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "gptq_b200.h"

#ifndef __CUDA_ARCH__
#define GPTQ_HOST_ONLY 1
#endif

namespace gptq {

constexpr int kNumSMs = 132;  // H100 SXM

__host__ __device__ constexpr int ceil_div(int a, int b) { return (a + b - 1) / b; }

// ---------------------------------------------------------------------------------------------
// Bit-field extraction.  A "run" is 32 consecutive values = BITS consecutive 32-bit words.
// bits 2/4/8: value j at bit BITS*(j % ipb) of word j / ipb  (quant/quant_linear.py:103,124-127)
// bits 3    : value j at bit 3*j of the 96-bit little-endian stream formed by the 3 words.
// ---------------------------------------------------------------------------------------------
template <int BITS>
__device__ __forceinline__ int extract_field(const uint32_t* run, int j) {
    if constexpr (BITS == 3) {
        const int bit = 3 * j;
        const int wi = bit >> 5, sh = bit & 31;
        uint32_t v = run[wi] >> sh;
        if (sh > 29) v |= run[wi + 1] << (32 - sh);
        return int(v & 7u);
    } else {
        constexpr int ipb = 32 / BITS;
        constexpr uint32_t maxq = (1u << BITS) - 1u;
        return int((run[j / ipb] >> ((j % ipb) * BITS)) & maxq);
    }
}

// Zero point of column n in one qzeros row (stored minus one; the +1 is NOT masked,
// quant/quant_linear.py:120-121), read straight from global memory.
template <int BITS>
__device__ __forceinline__ int load_zero(const int32_t* __restrict__ qzeros_row, int n) {
    const uint32_t* p = reinterpret_cast<const uint32_t*>(qzeros_row) + (n >> 5) * BITS;
    const int j = n & 31;
    if constexpr (BITS == 3) {
        const int bit = 3 * j;
        const int wi = bit >> 5, sh = bit & 31;
        uint32_t v = __ldg(p + wi) >> sh;
        if (sh > 29) v |= __ldg(p + wi + 1) << (32 - sh);
        return int(v & 7u) + 1;
    } else {
        constexpr int ipb = 32 / BITS;
        constexpr uint32_t maxq = (1u << BITS) - 1u;
        return int((__ldg(p + j / ipb) >> ((j % ipb) * BITS)) & maxq) + 1;
    }
}

// The reference's dequantised weight: (w - z) converted to fp16 (exact) times the fp16 scale,
// rounded once to fp16 (int32 * fp16 -> fp16 in quant/quant_linear.py:128).
__device__ __forceinline__ __half dequant_one(int w, int z, __half s) { return __hmul(__int2half_rn(w - z), s); }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// silu(a) * b on fp32 accumulators (quant/fused_mlp.py:163-164, :170-172)
__device__ __forceinline__ float swiglu(float a, float b) { return (a * (1.0f / (1.0f + expf(-a)))) * b; }

}  // namespace gptq
