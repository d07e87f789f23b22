// RoPE (in place) and RMSNorm: the two HBM/launch-bound elementwise ops on the path.
#include "common.cuh"
#include "kernels.h"

namespace gptq {
namespace {

// rotate_half_kernel (quant/fused_attn.py:8-58): one block per token, threads over (row, i); fp32 math (common.cuh), fp16 store.
__global__ void rope_kernel(__half* __restrict__ qk, int64_t token_stride, const int64_t* __restrict__ position_ids, int64_t pos_batch_stride, int seq,
                            int rows, int head_dim, float inv_base) {
    const int token = blockIdx.x;
    const int b = token / seq, s = token % seq;
    const float pos = (float)__ldg(position_ids + (size_t)b * pos_batch_stride + s);
    const int half_dim = head_dim >> 1;
    __half* base = qk + (size_t)token * token_stride;
    // 2 elements (i, i+1) per thread so loads/stores are 32-bit
    const int pairs_per_row = half_dim >> 1;
    for (int idx = threadIdx.x; idx < rows * pairs_per_row; idx += blockDim.x) {
        const int row = idx / pairs_per_row;
        const int i = (idx - row * pairs_per_row) * 2;
        const float f0 = rope_inv_freq(i, inv_base) * pos, f1 = rope_inv_freq(i + 1, inv_base) * pos;
        const float c0 = cosf(f0), s0 = sinf(f0), c1 = cosf(f1), s1 = sinf(f1);
        __half2* px = reinterpret_cast<__half2*>(base + (size_t)row * head_dim + i);
        __half2* py = reinterpret_cast<__half2*>(base + (size_t)row * head_dim + half_dim + i);
        const float2 xv = __half22float2(*px), yv = __half22float2(*py);
        const float ox0 = rope_x(xv.x, yv.x, c0, s0), ox1 = rope_x(xv.y, yv.y, c1, s1);
        const float oy0 = rope_y(xv.x, yv.x, c0, s0), oy1 = rope_y(xv.y, yv.y, c1, s1);
        *px = __floats2half2_rn(ox0, ox1);
        *py = __floats2half2_rn(oy0, oy1);
    }
}

// rms_norm_fwd_fused (quant/triton_norm.py:7-39): one block per row; variance in fp32, y = fp16((x * rstd) * w) (common.cuh).
template <int THREADS>
__global__ void __launch_bounds__(THREADS) rmsnorm_kernel(const __half* __restrict__ x, int64_t ldx, const __half* __restrict__ w, __half* __restrict__ y,
                                                          int64_t ldy, int N, float eps) {
    const int row = blockIdx.x;
    const __half2* xr = reinterpret_cast<const __half2*>(x + (size_t)row * ldx);
    const __half2* wr = reinterpret_cast<const __half2*>(w);
    __half2* yr = reinterpret_cast<__half2*>(y + (size_t)row * ldy);
    const int n2 = N >> 1;
    float ss = 0.f;
    for (int i = threadIdx.x; i < n2; i += THREADS) {
        const float2 v = __half22float2(xr[i]);
        ss = fmaf(v.x, v.x, ss);
        ss = fmaf(v.y, v.y, ss);
    }
    ss = warp_sum(ss);
    __shared__ float part[THREADS / 32];
    __shared__ float rstd_s;
    if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = ss;
    __syncthreads();
    if (threadIdx.x < 32) {
        float t = threadIdx.x < THREADS / 32 ? part[threadIdx.x] : 0.f;
        t = warp_sum(t);
        if (threadIdx.x == 0) rstd_s = rms_rstd(t, N, eps);
    }
    __syncthreads();
    const float rstd = rstd_s;
    for (int i = threadIdx.x; i < n2; i += THREADS) {
        yr[i] = rms_apply2(__half22float2(xr[i]), rstd, __half22float2(__ldg(wr + i)));
    }
}

}  // namespace

cudaError_t launch_rope(void* qk, int64_t token_stride, const int64_t* position_ids, int64_t pos_batch_stride, int bsz, int seq, int rows, int head_dim,
                        float base, cudaStream_t stream) {
    const int work = rows * (head_dim / 4);
    const int threads = work >= 256 ? 256 : ((work + 31) / 32) * 32;
    rope_kernel<<<bsz * seq, threads, 0, stream>>>(reinterpret_cast<__half*>(qk), token_stride, position_ids, pos_batch_stride, seq, rows, head_dim,
                                                    rope_inv_base(base, head_dim));
    return cudaGetLastError();
}

cudaError_t launch_rmsnorm(const void* x, int64_t ldx, const void* weight, void* y, int64_t ldy, int M, int N, float eps, cudaStream_t stream) {
    const __half* xp = reinterpret_cast<const __half*>(x);
    const __half* wp = reinterpret_cast<const __half*>(weight);
    __half* yp = reinterpret_cast<__half*>(y);
    if (N >= 2048)
        rmsnorm_kernel<256><<<M, 256, 0, stream>>>(xp, ldx, wp, yp, ldy, N, eps);
    else
        rmsnorm_kernel<64><<<M, 64, 0, stream>>>(xp, ldx, wp, yp, ldy, N, eps);
    return cudaGetLastError();
}

}  // namespace gptq
