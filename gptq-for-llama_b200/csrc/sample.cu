// sample.cu -- the next token of each sequence drawn from the fp16 logits of a decode step (gptq_sample_tokens): eos suppression below a
// minimum length, temperature, top-k, top-p and one Philox4x32-10 draw, or the argmax at temperature <= 0.  The rule is stated in
// include/gptq_b200.h; oracle/sampling.py restates it in numpy float64.
//
// One CTA of 1024 threads per row; thread t owns the contiguous ids [t*C, t*C + C), C = ceil(V / 1024), and every pass walks them in
// ascending order.  Thresholds are found on 16-bit order-preserving keys of the fp16 logits, so no decision depends on the order of a
// float sum: top-k by a two-level radix select over integer shared-memory histograms, the top-p boundary by a binary search over the keys
// whose every step sums the weights above a candidate in fp64 -- per thread in id order, then over the threads in a fixed tree.  The draw
// scans the same per-thread sums.  No float atomics, no workspace: a row's token depends on its logits, its parameters and its position.
#include <cstdint>

#include "common.cuh"
#include "kernels.h"

namespace gptq {
namespace {

constexpr int kThreads = 1024, kWarps = kThreads / 32;
constexpr uint32_t kKeyNegInf = 0x03FF;  // key of -inf (+inf is 0xFC00); the keys NaN bits would have lie outside [0x03FF, 0xFC00]

// fp16 bits -> key whose unsigned order is the order of the values: -0 is +0, NaN is -inf.
__device__ __forceinline__ uint32_t half_key(uint32_t bits) {
    if ((bits & 0x7C00u) == 0x7C00u && (bits & 0x03FFu) != 0) return kKeyNegInf;
    if (bits == 0x8000u) bits = 0;
    return (bits & 0x8000u) ? (~bits & 0xFFFFu) : (bits ^ 0x8000u);
}

__device__ __forceinline__ float key_value(uint32_t key) {
    const uint32_t bits = (key & 0x8000u) ? (key ^ 0x8000u) : (~key & 0xFFFFu);
    return __half2float(__ushort_as_half((unsigned short)bits));
}

// Random123's Philox4x32-10
__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint32_t k0, uint32_t k1) {
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        if (r) {
            k0 += 0x9E3779B9u;
            k1 += 0xBB67AE85u;
        }
        const uint32_t hi0 = __umulhi(0xD2511F53u, c.x), lo0 = 0xD2511F53u * c.x;
        const uint32_t hi1 = __umulhi(0xCD9E8D57u, c.z), lo1 = 0xCD9E8D57u * c.z;
        c = make_uint4(hi1 ^ c.y ^ k0, lo1, hi0 ^ c.w ^ k1, lo0);
    }
    return c;
}

// Every thread gets op over the block's values; the order of the combination is fixed.  `sh` holds kWarps entries.
template <class T, class Op>
__device__ __forceinline__ T block_reduce(T v, Op op, T* sh) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = op(v, __shfl_xor_sync(0xffffffffu, v, o));
    __syncthreads();  // sh is free again after its previous use
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
    __syncthreads();
    T r = sh[0];
#pragma unroll 1
    for (int w = 1; w < kWarps; ++w) r = op(r, sh[w]);
    return r;
}

// Exclusive prefix sum of one fp64 value per thread in thread order, fixed tree; *total gets the sum of all.
__device__ __forceinline__ double block_exclusive_scan(double v, double* sh, double* total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    double inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const double n = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += n;
    }
    __syncthreads();
    if (lane == 31) sh[warp] = inc;
    __syncthreads();
    double before = 0.0, all = 0.0;
#pragma unroll 1
    for (int w = 0; w < kWarps; ++w) {
        if (w == warp) before = all;
        all += sh[w];
    }
    *total = all;
    return before + inc - v;
}

__global__ void __launch_bounds__(kThreads) sample_kernel(const __half* __restrict__ logits, int64_t ld, int V, const int32_t* __restrict__ positions,
                                                          gptq_sampling prm, int32_t* __restrict__ next_tokens) {
    const int b = blockIdx.x, tid = threadIdx.x;
    const unsigned short* row = reinterpret_cast<const unsigned short*>(logits) + (size_t)b * ld;
    const int pos = positions[b];
    const float T = prm.temperature[b];
    const int eos = prm.eos_token[b];
    const int drop = (eos >= 0 && eos < V && (int64_t)pos + 1 < (int64_t)prm.min_length[b]) ? eos : -1;  // HF MinLengthLogitsProcessor
    const int C = ceil_div(V, kThreads), i0 = min(V, tid * C), i1 = min(V, i0 + C);
    auto key_at = [&](int i) -> uint32_t { return i == drop ? kKeyNegInf : half_key(row[i]); };

    __shared__ double shd[kWarps];
    __shared__ unsigned long long shu[kWarps];
    __shared__ int shi[kWarps];
    __shared__ unsigned hist[256];
    __shared__ uint32_t sel[2];

    // largest key, lowest id on ties: the argmax of argmax_row / argmax_kernel (float compare: -0 == +0)
    unsigned long long best = 0;
    for (int i = i0; i < i1; ++i) best = max(best, ((unsigned long long)key_at(i) << 32) | (uint32_t)(0x7fffffff - i));
    best = block_reduce(best, [](unsigned long long a, unsigned long long c) { return max(a, c); }, shu);
    const uint32_t kmax = (uint32_t)(best >> 32);
    if (!(T > 0.f)) {  // greedy
        if (tid == 0) next_tokens[b] = 0x7fffffff - (int)(uint32_t)best;
        return;
    }
    auto z_of = [&](uint32_t key) { return __fdiv_rn(key_value(key), T); };  // HF TemperatureLogitsWarper: fp32 logits / T
    const float zmax = z_of(kmax);
    if (zmax == -INFINITY) {  // nothing above -inf
        if (tid == 0) next_tokens[b] = 0;
        return;
    }

    // top-k: the k-th largest key counted with multiplicity; keep z >= z of it (ties at the k-th value are kept)
    const int k = prm.top_k[b];
    uint32_t kth = kKeyNegInf;
    if (k > 0 && k < V) {
        uint32_t prefix = 0, need = (uint32_t)k;
#pragma unroll 1
        for (int level = 0; level < 2; ++level) {
            for (int j = tid; j < 256; j += kThreads) hist[j] = 0;
            __syncthreads();
            for (int i = i0; i < i1; ++i) {
                const uint32_t key = key_at(i);
                if (level == 0) atomicAdd(&hist[key >> 8], 1u);
                else if ((key >> 8) == prefix) atomicAdd(&hist[key & 255u], 1u);
            }
            __syncthreads();
            if (tid == 0) {
                uint32_t acc = 0;
                int j = 255;
                for (; j > 0 && acc + hist[j] < need; --j) acc += hist[j];
                sel[0] = level == 0 ? (uint32_t)j : (prefix << 8) | (uint32_t)j;
                sel[1] = need - acc;
            }
            __syncthreads();
            prefix = sel[0];
            need = sel[1];
        }
        kth = prefix;
    }
    const float zth = z_of(kth);
    const bool inf_mode = zmax == INFINITY;  // +inf entries share all the mass
    auto weight = [&](float z) -> double { return inf_mode ? (z == INFINITY ? 1.0 : 0.0) : exp((double)z - (double)zmax); };
    auto topk_weight = [&](int i) -> double {
        const float z = z_of(key_at(i));
        return z >= zth ? weight(z) : 0.0;
    };
    auto sum = [](double a, double c) { return a + c; };

    // top-p: keep v iff (top-k mass with z > z_v) < top_p * (top-k mass).  The test is monotone in the key, so the kept set is every key
    // at or above the smallest key that passes; the largest key always passes.  Keys below the top-k threshold never pass.
    const float p = prm.top_p[b];
    uint32_t tp_key = kKeyNegInf;
    if (p < 1.f) {
        double w_all = 0.0;
        for (int i = i0; i < i1; ++i) w_all += topk_weight(i);
        const double bound = (double)p * block_reduce(w_all, sum, shd);
        uint32_t lo = max(kth, kKeyNegInf), hi = kmax;
#pragma unroll 1
        while (lo < hi) {
            const uint32_t mid = (lo + hi) >> 1;
            const float zm = z_of(mid);
            double above = 0.0;
            for (int i = i0; i < i1; ++i) {
                const float z = z_of(key_at(i));
                if (z >= zth && z > zm) above += weight(z);
            }
            if (block_reduce(above, sum, shd) < bound) hi = mid;
            else lo = mid + 1;
        }
        tp_key = hi;
    }

    // draw: the first kept token, in id order, whose inclusive running weight exceeds u * W
    double mine = 0.0;
    int last = -1;
    for (int i = i0; i < i1; ++i) {
        const uint32_t key = key_at(i);
        if (key < tp_key) continue;
        const float z = z_of(key);
        if (z < zth) continue;
        mine += weight(z);
        last = i;
    }
    double W;
    const double before = block_exclusive_scan(mine, shd, &W);
    const uint64_t seed = prm.seed[b];
    const uint4 x = philox4x32_10(make_uint4((uint32_t)pos, 0u, 0u, 0u), (uint32_t)seed, (uint32_t)(seed >> 32));
    const double target = ((double)(x.x >> 5) * 67108864.0 + (double)(x.y >> 6)) * 0x1p-53 * W;
    const int last_kept = block_reduce(last, [](int a, int c) { return max(a, c); }, shi);
    const int owner = block_reduce(last >= 0 && before + mine > target ? tid : kThreads, [](int a, int c) { return min(a, c); }, shi);
    if (owner == kThreads) {  // rounding left none
        if (tid == 0) next_tokens[b] = last_kept;
    } else if (tid == owner) {
        double run = before;
        int tok = last;
        for (int i = i0; i < i1; ++i) {
            const uint32_t key = key_at(i);
            if (key < tp_key) continue;
            const float z = z_of(key);
            if (z < zth) continue;
            run += weight(z);
            if (run > target) {
                tok = i;
                break;
            }
        }
        next_tokens[b] = tok;
    }
}

}  // namespace

cudaError_t launch_sample_tokens(const void* logits, int64_t ld, int batch, int vocab, const int32_t* positions, const gptq_sampling& params,
                                 int32_t* next_tokens, cudaStream_t stream) {
    sample_kernel<<<batch, kThreads, 0, stream>>>(reinterpret_cast<const __half*>(logits), ld, vocab, positions, params, next_tokens);
    return cudaGetLastError();
}

}  // namespace gptq
