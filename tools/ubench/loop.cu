// Microbenchmark of the decode matvec's per-stage inner loop on sm_90a: 16 warps per CTA (4 per scheduler), one CTA per SM,
// every warp runs `iters` stages of 4 k-steps from shared memory.  Prints cycles per stage per warp for a few instruction mixes.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o loop loop.cu
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>

__device__ __forceinline__ uint4 lds128(uint32_t a) {
    uint4 r;
    asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "r"(a));
    return r;
}
__device__ __forceinline__ void mma_f16(float (&d)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void mma_f8(float (&d)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k32.row.col.f32.e4m3.e4m3.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void mma_i8(int (&d)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k32.row.col.s32.u8.s8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3])
                 : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}
__device__ __forceinline__ uint2 lds64(uint32_t a) {
    uint2 r;
    asm volatile("ld.shared.v2.u32 {%0,%1}, [%2];" : "=r"(r.x), "=r"(r.y) : "r"(a));
    return r;
}
__device__ __forceinline__ uint32_t mulhi(uint32_t q, uint32_t m) {
    uint32_t r;
    asm("mul.hi.u32 %0, %1, %2;" : "=r"(r) : "r"(q), "r"(m));
    return r;
}

// V: 0 fp16 imm masks + mul.hi | 1 fp16 register masks + mul.hi | 2 as 0 without the MMAs | 3 MMAs only | 4 fp8 imm masks | 5 fp8 register masks
//    6 fp16 imm masks + SHF | 7 fp8 without the MMAs | 8 fp8 MMAs only
template <int V>
__global__ void __launch_bounds__(512, 1) k_loop(float* out, long long* cyc, int iters, uint32_t m_lo, uint32_t m_hi, uint32_t m_f8) {
    extern __shared__ __align__(16) uint8_t smem[];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
    for (int i = tid; i < 40960 / 4; i += 512) reinterpret_cast<uint32_t*>(smem)[i] = i * 2654435761u;
    __syncthreads();
    uint32_t sbase;
    asm("{ .reg .u64 a; cvta.to.shared.u64 a, %1; cvt.u32.u64 %0, a; }" : "=r"(sbase) : "l"(smem));
    const uint32_t wbase = sbase + (warp & 7) * 128 + t * 1056 + g * 16, xbase = sbase + 36864 + t * 16;
    float acc0[4] = {0, 0, 0, 0}, acc1[4] = {0, 0, 0, 0};
    uint32_t sink = 0;
    float tot = 0.f;
    const long long t0 = clock64();
#pragma unroll 1
    for (int it = 0; it < iters; ++it) {
        uint4 q[4], xf[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) q[j] = lds128(wbase + j * 4224 + (it & 1) * 16896);
#pragma unroll
        for (int j = 0; j < 4; ++j) xf[j] = lds128(xbase + j * 64 + (it & 7) * 256);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const uint32_t w[4] = {q[j].x, q[j].y, q[j].z, q[j].w};
            if (V == 3) {
                mma_f16(acc0, w[0], w[1], w[2], w[3], xf[j].x, xf[j].y);
                mma_f16(acc1, w[1], w[2], w[3], w[0], xf[j].x, xf[j].y);
                mma_f16(acc0, w[2], w[3], w[0], w[1], xf[j].z, xf[j].w);
                mma_f16(acc1, w[3], w[0], w[1], w[2], xf[j].z, xf[j].w);
            } else if (V == 8) {
                mma_f8(acc0, w[0], w[1], w[2], w[3], xf[j].x, xf[j].y);
                mma_f8(acc1, w[2], w[3], w[0], w[1], xf[j].z, xf[j].w);
            } else if (V == 4 || V == 5 || V == 7) {
                uint32_t a[4][2];
#pragma unroll
                for (int c = 0; c < 4; ++c) {
                    const uint32_t q4 = mulhi(w[c], 0x10000000u);
                    if (V == 5) {
                        a[c][0] = w[c] & m_f8;
                        a[c][1] = q4 & m_f8;
                    } else {
                        a[c][0] = w[c] & 0x0f0f0f0fu;
                        a[c][1] = q4 & 0x0f0f0f0fu;
                    }
                }
                if (V == 7) {
                    sink ^= a[0][0] ^ a[1][0] ^ a[0][1] ^ a[1][1] ^ a[2][0] ^ a[3][0] ^ a[2][1] ^ a[3][1];
                } else {
                    mma_f8(acc0, a[0][0], a[1][0], a[0][1], a[1][1], xf[j].x, xf[j].y);
                    mma_f8(acc1, a[2][0], a[3][0], a[2][1], a[3][1], xf[j].x, xf[j].y);
                }
            } else {
                uint32_t a[4][4];
#pragma unroll
                for (int c = 0; c < 4; ++c) {
                    const uint32_t q8 = (V == 6) ? (w[c] >> 8) : mulhi(w[c], 0x01000000u);
                    if (V == 1) {
                        a[c][0] = w[c] & m_lo; a[c][1] = w[c] & m_hi; a[c][2] = q8 & m_lo; a[c][3] = q8 & m_hi;
                    } else {
                        a[c][0] = w[c] & 0x000f000fu; a[c][1] = w[c] & 0x00f000f0u; a[c][2] = q8 & 0x000f000fu; a[c][3] = q8 & 0x00f000f0u;
                    }
                }
                if (V == 2) {
#pragma unroll
                    for (int c = 0; c < 4; ++c) sink ^= a[c][0] ^ a[c][1] ^ a[c][2] ^ a[c][3];
                } else {
                    mma_f16(acc0, a[0][0], a[1][0], a[0][1], a[1][1], xf[j].x, xf[j].y);
                    mma_f16(acc1, a[2][0], a[3][0], a[2][1], a[3][1], xf[j].x, xf[j].y);
                    mma_f16(acc0, a[0][2], a[1][2], a[0][3], a[1][3], xf[j].z, xf[j].w);
                    mma_f16(acc1, a[2][2], a[3][2], a[2][3], a[3][3], xf[j].z, xf[j].w);
                }
            }
        }
        tot += acc0[0] + acc1[2];
    }
    const long long t1 = clock64();
    out[blockIdx.x * 512 + tid] = tot + acc0[1] + acc1[3] + (float)sink;
    if (tid == 0) cyc[blockIdx.x] = t1 - t0;
}

// int8 path: A = u8 nibbles (2 LOP3 + 1 SHF per packed word), B = x as s8 digits, IMMA.16832, int32 accumulators
// V: 0 full | 1 dequant only | 2 IMMA only
template <int V>
__global__ void __launch_bounds__(512, 1) k_loop_i8(float* out, long long* cyc, int iters) {
    extern __shared__ __align__(16) uint8_t smem[];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
    for (int i = tid; i < 40960 / 4; i += 512) reinterpret_cast<uint32_t*>(smem)[i] = i * 2654435761u;
    __syncthreads();
    uint32_t sbase;
    asm("{ .reg .u64 a; cvta.to.shared.u64 a, %1; cvt.u32.u64 %0, a; }" : "=r"(sbase) : "l"(smem));
    const uint32_t wbase = sbase + (warp & 7) * 128 + t * 1056 + g * 16, xbase = sbase + 36864 + (g & 3) * 1024 + t * 8;
    int acc0[4] = {0, 0, 0, 0}, acc1[4] = {0, 0, 0, 0};
    uint32_t sink = 0;
    float tot = 0.f;
    const long long t0 = clock64();
#pragma unroll 1
    for (int it = 0; it < iters; ++it) {
        uint4 q[4];
        uint2 xf[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) q[j] = lds128(wbase + j * 4224 + (it & 1) * 16896);
#pragma unroll
        for (int j = 0; j < 4; ++j) xf[j] = lds64(xbase + j * 32 + (it & 7) * 128);
#pragma unroll
        for (int c = 0; c < 4; ++c) acc0[c] = acc1[c] = 0;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const uint32_t w[4] = {q[j].x, q[j].y, q[j].z, q[j].w};
            if (V == 2) {
                mma_i8(acc0, w[0], w[1], w[2], w[3], xf[j].x, xf[j].y);
                mma_i8(acc1, w[2], w[3], w[0], w[1], xf[j].x, xf[j].y);
            } else {
                uint32_t a[4][2];
#pragma unroll
                for (int c = 0; c < 4; ++c) {
                    a[c][0] = w[c] & 0x0f0f0f0fu;
                    a[c][1] = (w[c] >> 4) & 0x0f0f0f0fu;
                }
                if (V == 1) {
                    sink ^= a[0][0] ^ a[1][0] ^ a[0][1] ^ a[1][1] ^ a[2][0] ^ a[3][0] ^ a[2][1] ^ a[3][1];
                } else {
                    mma_i8(acc0, a[0][0], a[1][0], a[0][1], a[1][1], xf[j].x, xf[j].y);
                    mma_i8(acc1, a[2][0], a[3][0], a[2][1], a[3][1], xf[j].x, xf[j].y);
                }
            }
        }
        // group epilogue of the two lanes that hold digits: 4 columns x (2 conversions + 2 fma)
        tot = fmaf((float)acc0[0], 256.f, tot) + (float)acc0[1];
        tot = fmaf((float)acc0[2], 256.f, tot) + (float)acc0[3];
        tot = fmaf((float)acc1[0], 256.f, tot) + (float)acc1[1];
        tot = fmaf((float)acc1[2], 256.f, tot) + (float)acc1[3];
    }
    const long long t1 = clock64();
    out[blockIdx.x * 512 + tid] = tot + (float)sink;
    if (tid == 0) cyc[blockIdx.x] = t1 - t0;
}

template <int V>
void run_i8(const char* name, float* out, long long* cyc, int nb) {
    const int iters = 2000;
    cudaFuncSetAttribute(k_loop_i8<V>, cudaFuncAttributeMaxDynamicSharedMemorySize, 40960);
    k_loop_i8<V><<<nb, 512, 40960>>>(out, cyc, 10);
    k_loop_i8<V><<<nb, 512, 40960>>>(out, cyc, iters);
    cudaDeviceSynchronize();
    long long h[1024];
    cudaMemcpy(h, cyc, nb * sizeof(long long), cudaMemcpyDeviceToHost);
    double s = 0;
    for (int i = 0; i < nb; ++i) s += (double)h[i];
    printf("%-58s %8.1f cycles per stage per warp (16 warps/SM)   err=%s\n", name, s / nb / iters, cudaGetErrorString(cudaGetLastError()));
}

template <int V>
void run(const char* name, float* out, long long* cyc, int nb) {
    const int iters = 2000;
    cudaFuncSetAttribute(k_loop<V>, cudaFuncAttributeMaxDynamicSharedMemorySize, 40960);
    k_loop<V><<<nb, 512, 40960>>>(out, cyc, 10, 0x000f000fu, 0x00f000f0u, 0x0f0f0f0fu);
    k_loop<V><<<nb, 512, 40960>>>(out, cyc, iters, 0x000f000fu, 0x00f000f0u, 0x0f0f0f0fu);
    cudaDeviceSynchronize();
    long long h[1024];
    cudaMemcpy(h, cyc, nb * sizeof(long long), cudaMemcpyDeviceToHost);
    double s = 0;
    for (int i = 0; i < nb; ++i) s += (double)h[i];
    printf("%-58s %8.1f cycles per stage per warp (16 warps/SM)   err=%s\n", name, s / nb / iters, cudaGetErrorString(cudaGetLastError()));
}

int main() {
    int nb = 132;
    cudaDeviceProp pr;
    cudaGetDeviceProperties(&pr, 0);
    nb = pr.multiProcessorCount;
    float* out;
    long long* cyc;
    cudaMalloc(&out, nb * 512 * 4);
    cudaMalloc(&cyc, nb * 8);
    run<0>("fp16 subnormal, immediate masks, mul.hi shift (current)", out, cyc, nb);
    run<1>("fp16 subnormal, register masks, mul.hi shift", out, cyc, nb);
    run<6>("fp16 subnormal, immediate masks, SHF shift", out, cyc, nb);
    run<2>("  the same dequant without the MMAs", out, cyc, nb);
    run<3>("  16 HMMA.16816 per stage only (+LDS)", out, cyc, nb);
    run<4>("fp8 e4m3 nibbles, immediate masks, mul.hi shift", out, cyc, nb);
    run<5>("fp8 e4m3 nibbles, register masks, mul.hi shift", out, cyc, nb);
    run<7>("  the same dequant without the MMAs", out, cyc, nb);
    run<8>("  8 QMMA.16832 per stage only (+LDS)", out, cyc, nb);
    run_i8<0>("int8: u8 nibbles (2 LOP3 + SHF), 8 IMMA.16832 + epilogue", out, cyc, nb);
    run_i8<1>("  the same dequant without the MMAs", out, cyc, nb);
    run_i8<2>("  8 IMMA.16832 per stage only (+LDS, epilogue)", out, cyc, nb);
    return 0;
}
