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

// ---- host: alignment, scratch carving, launches ------------------------------------------------------------------------------
inline bool aligned(const void* p, size_t a) { return (reinterpret_cast<uintptr_t>(p) & (a - 1)) == 0; }
inline size_t align256(size_t v) { return (v + 255) & ~(size_t)255; }
// the next buffer of a scratch region whose first `end` bytes are taken: its offset; every buffer starts on a 256-byte boundary
inline size_t carve(size_t& end, size_t bytes) {
    const size_t o = end;
    end += align256(bytes);
    return o;
}

// Launches `kernel`, first opting it in to `smem` bytes of dynamic shared memory when that is more than the default 48 KB.  pdl:
// programmatic dependent launch, the kernel may start while its predecessor on the stream drains; such a kernel calls
// grid_dependency_wait() before it touches anything another kernel produces or still reads.
template <typename... KArgs, typename... Args>
cudaError_t launch_kernel(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, bool pdl, Args&&... args) {
    if (smem > 48 * 1024) {
        const cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
    }
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = pdl ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

// the device side of programmatic dependent launch
__device__ __forceinline__ void grid_dependency_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void grid_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

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

// ---- RoPE (rotate_half_kernel, quant/fused_attn.py:8-58) --------------------------------------------------------------------
// Both decode engines and gptq_rope_inplace(_freq) rotate with these, so their q and k agree bit for bit.
inline float rope_inv_base(float base, int head_dim) { return (float)(-2.0 * log((double)base) / (double)head_dim); }  // :91
inline float attn_scale(int head_dim) { return 1.0f / sqrtf((float)head_dim); }                                        // SDPA's head_dim^-0.5

// The frequencies of one rotation, carried by value in the launch parameters (a captured graph replays them without a device buffer).
// table == 0: pair i turns by exp(i * inv_base), the unscaled rule.  table == 1: by f[i], a host table of head_dim / 2 values (a scaled
// rotation such as LLaMA-3.1's llama3 rule, computed by the host bit for bit as HF computes it; gptq_b200.ops.rope_inv_freq).
constexpr int kRopeMaxPairs = 64;  // head_dim 128
struct RopeFreqs {
    float inv_base;
    int table;
    float f[kRopeMaxPairs];
};
// host: the rule of a call; inv_freq (HOST, head_dim / 2 entries, checked by rope_table_ok) or nullptr for the unscaled rule at `base`
inline RopeFreqs rope_freqs(float base, int head_dim, const float* inv_freq) {
    RopeFreqs r{};
    r.inv_base = rope_inv_base(base, head_dim);
    r.table = inv_freq != nullptr;
    for (int i = 0; inv_freq != nullptr && i < head_dim / 2; ++i) r.f[i] = inv_freq[i];
    return r;
}
// host: every entry of a table finite and > 0 (a frequency the angle rule below can use)
inline bool rope_table_ok(const float* inv_freq, int n) {
    for (int i = 0; i < n; ++i)
        if (!(inv_freq[i] > 0.f) || !isfinite(inv_freq[i])) return false;
    return true;
}
// The frequency of pair i; times the position, rounded once in fp32, it is the angle (then its cosf and sinf).  The unscaled rule is fp32
// with the accurate expf (the reference insists on libdevice exp, :42-43).
__device__ __forceinline__ float rope_inv_freq(int i, const RopeFreqs& r) { return r.table ? r.f[i] : expf((float)i * r.inv_base); }
// x' = x c - y s ; y' = x s + y c, y at +head_dim/2 (:52-57): the reference's operation order, no FMA contraction (two roundings per term)
__device__ __forceinline__ float rope_x(float x, float y, float c, float s) { return __fsub_rn(__fmul_rn(x, c), __fmul_rn(y, s)); }
__device__ __forceinline__ float rope_y(float x, float y, float c, float s) { return __fadd_rn(__fmul_rn(x, s), __fmul_rn(y, c)); }

// ---- RMSNorm (rms_norm_fwd_fused, quant/triton_norm.py:21-39) ----------------------------------------------------------------
// Every kernel keeps its own order for the sum of squares; the scale and the apply step are these.
__device__ __forceinline__ float rms_rstd(float sumsq, int n, float eps) { return 1.0f / sqrtf(sumsq / (float)n + eps); }
// fp16((x * rstd) * w) of two elements: two fp32 roundings, one fp16 rounding (:30-38)
__device__ __forceinline__ __half2 rms_apply2(float2 x, float rstd, float2 w) {
    return __floats2half2_rn(__fmul_rn(__fmul_rn(x.x, rstd), w.x), __fmul_rn(__fmul_rn(x.y, rstd), w.y));
}

// ---- greedy argmax: the larger value wins, the lower id wins a tie -----------------------------------------------------------
// Macros, not functions: the compiler optimises a branching __forceinline__ function on its own before it inlines it, and the
// persistent kernel's code around the call would change with it.
#define GPTQ_ARGMAX_BEATS(v, i, best, idx) ((v) > (best) || ((v) == (best) && (i) < (idx)))
// every lane ends with the warp's (best, idx)
#define GPTQ_WARP_ARGMAX(best, idx)                                    \
    _Pragma("unroll") for (int o_ = 16; o_ > 0; o_ >>= 1) {           \
        const float ov_ = __shfl_xor_sync(0xffffffffu, best, o_);     \
        const int oi_ = __shfl_xor_sync(0xffffffffu, idx, o_);        \
        if (GPTQ_ARGMAX_BEATS(ov_, oi_, best, idx)) {                  \
            best = ov_;                                                \
            idx = oi_;                                                 \
        }                                                              \
    }

}  // namespace gptq
