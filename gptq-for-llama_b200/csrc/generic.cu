// Generic CUDA-core kernels: every bit width in {2,3,4,8}, arbitrary g_idx (act-order), any M.
// They are the correctness backbone (and the only path for shapes the tuned kernels reject);
// the tuned int4 matvec / wgmma GEMM live in their own files and are dispatched from capi.cu.
//
// Arithmetic follows matmul_248_kernel (quant/quant_linear.py:84-137 of the reference):
//   W[k,n] = fp16( fp16(q[k,n] - (z[g_idx[k],n] + 1)) * s[g_idx[k],n] ),  out = fp16( sum_k fp32(x*W) ) (+ bias in fp16)
#include "common.cuh"
#include "kernels.h"

namespace gptq {

namespace {

constexpr int kGenWarps = 8;

template <int BITS>
struct WeightCursor {
    const uint32_t* __restrict__ qweight;
    const __half* __restrict__ scales;
    const int32_t* __restrict__ qzeros;
    int N;
    int zstride;  // words per qzeros row
    int cur_g = -1;
    __half s;
    int z;
    uint32_t run[BITS];

    __device__ __forceinline__ void init(const gptq_qweight& w) {
        qweight = reinterpret_cast<const uint32_t*>(w.qweight);
        scales = reinterpret_cast<const __half*>(w.scales);
        qzeros = w.qzeros;
        N = w.N;
        zstride = w.N / 32 * BITS;
    }
    __device__ __forceinline__ void load_run(int r, int n) {
#pragma unroll
        for (int i = 0; i < BITS; ++i) run[i] = __ldg(qweight + (size_t)(r * BITS + i) * N + n);
    }
    __device__ __forceinline__ void set_group(int g, int n) {
        if (g != cur_g) {
            cur_g = g;
            s = __ldg(scales + (size_t)g * N + n);
            z = load_zero<BITS>(qzeros + (size_t)g * zstride, n);
        }
    }
    __device__ __forceinline__ float weight(int j) const { return __half2float(dequant_one(extract_field<BITS>(run, j), z, s)); }
};

// grid (N/32, ceil(M/MB)); block 32 x kGenWarps: lane = output column, warps split K, shuffle-free
// column ownership + one shared-memory cross-warp reduction.
template <int BITS, int MB, bool DUAL>
__global__ void __launch_bounds__(32 * kGenWarps) qlinear_generic_kernel(const __half* __restrict__ x, int64_t ldx, gptq_qweight w1, gptq_qweight w2,
                                                                         const __half* __restrict__ bias, __half* __restrict__ out, int64_t ldo, int M) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int n = blockIdx.x * 32 + lane;
    const int m0 = blockIdx.y * MB;
    const int K = w1.K;
    const bool gather = w1.groupsize <= 0;
    const int gs = gather ? 1 : w1.groupsize;

    WeightCursor<BITS> c1, c2;
    c1.init(w1);
    if constexpr (DUAL) c2.init(w2);

    float acc1[MB], acc2[MB];
#pragma unroll
    for (int m = 0; m < MB; ++m) acc1[m] = acc2[m] = 0.f;

    const __half* xr[MB];
#pragma unroll
    for (int m = 0; m < MB; ++m) xr[m] = x + (size_t)min(m0 + m, M - 1) * ldx;

    for (int r = warp; r < K / 32; r += kGenWarps) {
        c1.load_run(r, n);
        if constexpr (DUAL) c2.load_run(r, n);
#pragma unroll
        for (int j = 0; j < 32; ++j) {
            const int k = r * 32 + j;
            const int g1 = gather ? __ldg(w1.g_idx + k) : k / gs;
            c1.set_group(g1, n);
            const float wv1 = c1.weight(j);
            float wv2 = 0.f;
            if constexpr (DUAL) {
                const int g2 = gather ? __ldg(w2.g_idx + k) : k / gs;
                c2.set_group(g2, n);
                wv2 = c2.weight(j);
            }
#pragma unroll
            for (int m = 0; m < MB; ++m) {
                const float xv = __half2float(__ldg(xr[m] + k));
                acc1[m] = fmaf(xv, wv1, acc1[m]);
                if constexpr (DUAL) acc2[m] = fmaf(xv, wv2, acc2[m]);
            }
        }
    }

    constexpr int NACC = DUAL ? 2 * MB : MB;
    __shared__ float red[kGenWarps][NACC][32];
#pragma unroll
    for (int m = 0; m < MB; ++m) {
        red[warp][m][lane] = acc1[m];
        if constexpr (DUAL) red[warp][MB + m][lane] = acc2[m];
    }
    __syncthreads();
    if (warp == 0) {
#pragma unroll
        for (int m = 0; m < MB; ++m) {
            float a = 0.f, b = 0.f;
#pragma unroll
            for (int wv = 0; wv < kGenWarps; ++wv) {
                a += red[wv][m][lane];
                if constexpr (DUAL) b += red[wv][MB + m][lane];
            }
            if (m0 + m < M) {
                __half o;
                if constexpr (DUAL) {
                    o = __float2half_rn(swiglu(a, b));
                } else {
                    o = __float2half_rn(a);
                    if (bias != nullptr) o = __hadd(o, bias[n]);  // fp16 add after the store rounding (quant_linear.py:376)
                }
                out[(size_t)(m0 + m) * ldo + n] = o;
            }
        }
    }
}

// out[M,K] = g[M,N] . W^T.  grid (K/32, ceil(M/MB)); block: lanes stride over n, warps split N.
template <int BITS, int MB>
__global__ void __launch_bounds__(32 * kGenWarps) qlinear_transpose_generic_kernel(const __half* __restrict__ gin, int64_t ldg, gptq_qweight w,
                                                                                   __half* __restrict__ out, int64_t ldo, int M) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int r = blockIdx.x;
    const int m0 = blockIdx.y * MB;
    const bool gather = w.groupsize <= 0;
    const int gs = gather ? 1 : w.groupsize;
    const int N = w.N;
    const __half* scales = reinterpret_cast<const __half*>(w.scales);
    const int zstride = N / 32 * BITS;

    int grp[32];
#pragma unroll
    for (int j = 0; j < 32; ++j) {
        const int k = r * 32 + j;
        grp[j] = gather ? __ldg(w.g_idx + k) : k / gs;
    }

    float acc[MB][32];
#pragma unroll
    for (int m = 0; m < MB; ++m)
#pragma unroll
        for (int j = 0; j < 32; ++j) acc[m][j] = 0.f;

    for (int n = warp * 32 + lane; n < N; n += 32 * kGenWarps) {
        uint32_t run[BITS];
#pragma unroll
        for (int i = 0; i < BITS; ++i) run[i] = __ldg(reinterpret_cast<const uint32_t*>(w.qweight) + (size_t)(r * BITS + i) * N + n);
        float gv[MB];
#pragma unroll
        for (int m = 0; m < MB; ++m) gv[m] = __half2float(__ldg(gin + (size_t)min(m0 + m, M - 1) * ldg + n));
        int cur = -1, z = 0;
        __half s = __float2half(0.f);
#pragma unroll
        for (int j = 0; j < 32; ++j) {
            if (grp[j] != cur) {
                cur = grp[j];
                s = __ldg(scales + (size_t)cur * N + n);
                z = load_zero<BITS>(w.qzeros + (size_t)cur * zstride, n);
            }
            const float wv = __half2float(dequant_one(extract_field<BITS>(run, j), z, s));
#pragma unroll
            for (int m = 0; m < MB; ++m) acc[m][j] = fmaf(gv[m], wv, acc[m][j]);
        }
    }

    __shared__ float red[kGenWarps][MB][32];
#pragma unroll
    for (int m = 0; m < MB; ++m)
#pragma unroll
        for (int j = 0; j < 32; ++j) {
            const float v = warp_sum(acc[m][j]);
            if (lane == j) red[warp][m][j] = v;
        }
    __syncthreads();
    if (warp == 0) {
#pragma unroll
        for (int m = 0; m < MB; ++m) {
            float a = 0.f;
#pragma unroll
            for (int wv = 0; wv < kGenWarps; ++wv) a += red[wv][m][lane];
            if (m0 + m < M) out[(size_t)(m0 + m) * ldo + r * 32 + lane] = __float2half_rn(a);
        }
    }
}

template <int BITS>
__global__ void dequant_kernel(gptq_qweight w, __half* __restrict__ out, int64_t ldo) {
    const int n = blockIdx.x * blockDim.x + threadIdx.x;
    const int r = blockIdx.y;
    if (n >= w.N) return;
    const bool gather = w.groupsize <= 0;
    const int gs = gather ? 1 : w.groupsize;
    WeightCursor<BITS> c;
    c.init(w);
    c.load_run(r, n);
#pragma unroll
    for (int j = 0; j < 32; ++j) {
        const int k = r * 32 + j;
        c.set_group(gather ? __ldg(w.g_idx + k) : k / gs, n);
        out[(size_t)k * ldo + n] = dequant_one(extract_field<BITS>(c.run, j), c.z, c.s);
    }
}

template <int BITS, bool DUAL>
cudaError_t launch_generic_bits(const QLinearArgs& a) {
    const dim3 block(32 * kGenWarps);
    const __half* x = reinterpret_cast<const __half*>(a.x);
    const __half* bias = reinterpret_cast<const __half*>(a.bias);
    __half* out = reinterpret_cast<__half*>(a.out);
    if (a.M == 1) {
        qlinear_generic_kernel<BITS, 1, DUAL><<<dim3(a.w.N / 32, 1), block, 0, a.stream>>>(x, a.ldx, a.w, a.w2, bias, out, a.ldo, a.M);
    } else if (a.M == 2) {
        qlinear_generic_kernel<BITS, 2, DUAL><<<dim3(a.w.N / 32, 1), block, 0, a.stream>>>(x, a.ldx, a.w, a.w2, bias, out, a.ldo, a.M);
    } else {
        // gridDim.y is limited to 65535
        constexpr int MB = 4;
        for (int m0 = 0; m0 < a.M; m0 += 65535 * MB) {
            const int rows = min(a.M - m0, 65535 * MB);
            qlinear_generic_kernel<BITS, MB, DUAL><<<dim3(a.w.N / 32, ceil_div(rows, MB)), block, 0, a.stream>>>(x + (size_t)m0 * a.ldx, a.ldx, a.w, a.w2, bias,
                                                                                                                  out + (size_t)m0 * a.ldo, a.ldo, rows);
        }
    }
    return cudaGetLastError();
}

template <bool DUAL>
cudaError_t launch_generic_dual(const QLinearArgs& a) {
    switch (a.w.bits) {
        case 2: return launch_generic_bits<2, DUAL>(a);
        case 3: return launch_generic_bits<3, DUAL>(a);
        case 4: return launch_generic_bits<4, DUAL>(a);
        case 8: return launch_generic_bits<8, DUAL>(a);
    }
    return cudaErrorInvalidValue;
}

}  // namespace

cudaError_t launch_qlinear_generic(const QLinearArgs& a) { return a.dual ? launch_generic_dual<true>(a) : launch_generic_dual<false>(a); }

cudaError_t launch_qlinear_transpose_generic(const void* g, int64_t ldg, const gptq_qweight& w, void* out, int64_t ldo, int M, cudaStream_t stream) {
    constexpr int MB = 2;
    const __half* gp = reinterpret_cast<const __half*>(g);
    __half* op = reinterpret_cast<__half*>(out);
    for (int m0 = 0; m0 < M; m0 += 65535 * MB) {
        const int rows = min(M - m0, 65535 * MB);
        const dim3 grid(w.K / 32, ceil_div(rows, MB)), block(32 * kGenWarps);
        const __half* gi = gp + (size_t)m0 * ldg;
        __half* oi = op + (size_t)m0 * ldo;
        switch (w.bits) {
            case 2: qlinear_transpose_generic_kernel<2, MB><<<grid, block, 0, stream>>>(gi, ldg, w, oi, ldo, rows); break;
            case 3: qlinear_transpose_generic_kernel<3, MB><<<grid, block, 0, stream>>>(gi, ldg, w, oi, ldo, rows); break;
            case 4: qlinear_transpose_generic_kernel<4, MB><<<grid, block, 0, stream>>>(gi, ldg, w, oi, ldo, rows); break;
            case 8: qlinear_transpose_generic_kernel<8, MB><<<grid, block, 0, stream>>>(gi, ldg, w, oi, ldo, rows); break;
            default: return cudaErrorInvalidValue;
        }
    }
    return cudaGetLastError();
}

cudaError_t launch_dequant(const gptq_qweight& w, void* out, int64_t ldo, cudaStream_t stream) {
    const dim3 block(128), grid(ceil_div(w.N, 128), w.K / 32);
    __half* o = reinterpret_cast<__half*>(out);
    switch (w.bits) {
        case 2: dequant_kernel<2><<<grid, block, 0, stream>>>(w, o, ldo); break;
        case 3: dequant_kernel<3><<<grid, block, 0, stream>>>(w, o, ldo); break;
        case 4: dequant_kernel<4><<<grid, block, 0, stream>>>(w, o, ldo); break;
        case 8: dequant_kernel<8><<<grid, block, 0, stream>>>(w, o, ldo); break;
        default: return cudaErrorInvalidValue;
    }
    return cudaGetLastError();
}

}  // namespace gptq
