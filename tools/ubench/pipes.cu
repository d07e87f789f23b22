// Issue-rate / latency microbenchmark for the instruction mix of the int4 decode matvec on sm_90a:
// legacy HMMA.16816 (mma.sync), HFMA2, LOP3.  Prints cycles per warp-instruction per SM sub-partition.
#include <cstdio>
#include <cstdint>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

template <int CHAINS>
__global__ void k_hmma(float* out, long long* cyc, int iters) {
    float acc[CHAINS][4];
#pragma unroll
    for (int c = 0; c < CHAINS; ++c)
        for (int i = 0; i < 4; ++i) acc[c][i] = 0.f;
    uint32_t a0 = threadIdx.x, a1 = threadIdx.x * 3, a2 = 7, a3 = 9, b0 = 0x3c003c00, b1 = 0x3c003c00;
    __syncthreads();
    const long long t0 = clock64();
    for (int it = 0; it < iters; ++it) {
#pragma unroll
        for (int c = 0; c < CHAINS; ++c)
            asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                         : "+f"(acc[c][0]), "+f"(acc[c][1]), "+f"(acc[c][2]), "+f"(acc[c][3])
                         : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
    }
    const long long t1 = clock64();
    float s = 0.f;
#pragma unroll
    for (int c = 0; c < CHAINS; ++c) s += acc[c][0] + acc[c][1] + acc[c][2] + acc[c][3];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
    if (threadIdx.x == 0) cyc[blockIdx.x] = t1 - t0;
}

template <int CHAINS>
__global__ void k_hfma2(float* out, long long* cyc, int iters) {
    __half2 acc[CHAINS];
#pragma unroll
    for (int c = 0; c < CHAINS; ++c) acc[c] = __float2half2_rn((float)threadIdx.x * 1e-3f + c);
    const __half2 m = __float2half2_rn(0.999f), a = __float2half2_rn(1e-3f);
    __syncthreads();
    const long long t0 = clock64();
    for (int it = 0; it < iters; ++it) {
#pragma unroll
        for (int c = 0; c < CHAINS; ++c) acc[c] = __hfma2(acc[c], m, a);
    }
    const long long t1 = clock64();
    float s = 0.f;
#pragma unroll
    for (int c = 0; c < CHAINS; ++c) s += __low2float(acc[c]) + __high2float(acc[c]);
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
    if (threadIdx.x == 0) cyc[blockIdx.x] = t1 - t0;
}

template <int CHAINS>
__global__ void k_lop3(float* out, long long* cyc, int iters) {
    uint32_t acc[CHAINS];
#pragma unroll
    for (int c = 0; c < CHAINS; ++c) acc[c] = threadIdx.x * 2654435761u + c;
    __syncthreads();
    const long long t0 = clock64();
    for (int it = 0; it < iters; ++it) {
#pragma unroll
        for (int c = 0; c < CHAINS; ++c) asm volatile("lop3.b32 %0, %0, %1, 0x64006400, 0x6a;" : "+r"(acc[c]) : "r"(acc[(c + 1) % CHAINS] | 1u));
    }
    const long long t1 = clock64();
    uint32_t s = 0;
#pragma unroll
    for (int c = 0; c < CHAINS; ++c) s ^= acc[c];
    out[blockIdx.x * blockDim.x + threadIdx.x] = (float)s;
    if (threadIdx.x == 0) cyc[blockIdx.x] = t1 - t0;
}

// Mixed streams: do the half-rate pipes overlap?  8 independent HFMA2 chains + 8 independent chains of a second kind per iteration.
template <int MODE>
__global__ void k_mix(float* out, long long* cyc, int iters) {
    __half2 h[8];
    uint32_t a[8];
    float acc[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
#pragma unroll
    for (int c = 0; c < 8; ++c) {
        h[c] = __float2half2_rn((float)threadIdx.x * 1e-3f + c);
        a[c] = threadIdx.x * 2654435761u + c;
    }
    const __half2 m = __float2half2_rn(0.999f), ad = __float2half2_rn(1e-3f);
    const uint32_t k1 = threadIdx.x | 1u;
    __syncthreads();
    const long long t0 = clock64();
    for (int it = 0; it < iters; ++it) {
#pragma unroll
        for (int c = 0; c < 8; ++c) {
            if (MODE != 2) h[c] = __hfma2(h[c], m, ad);
            if (MODE == 0) asm volatile("lop3.b32 %0, %0, %1, 0x64006400, 0x6a;" : "+r"(a[c]) : "r"(k1));
            if (MODE == 1) asm volatile("add.u32 %0, %0, %1;" : "+r"(a[c]) : "r"(k1));
            if (MODE == 2) {
                asm volatile("lop3.b32 %0, %0, %1, 0x64006400, 0x6a;" : "+r"(a[c]) : "r"(k1));
                asm volatile("shr.u32 %0, %0, 1;" : "+r"(a[(c + 4) & 7]));
            }
        }
        if (MODE == 3) {
#pragma unroll
            for (int c = 0; c < 2; ++c)
                asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                             : "+f"(acc[c][0]), "+f"(acc[c][1]), "+f"(acc[c][2]), "+f"(acc[c][3])
                             : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(a[4]), "r"(a[5]));
        }
    }
    const long long t1 = clock64();
    float s = acc[0][0] + acc[1][0];
#pragma unroll
    for (int c = 0; c < 8; ++c) s += __low2float(h[c]) + (float)a[c];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
    if (threadIdx.x == 0) cyc[blockIdx.x] = t1 - t0;
}

template <typename K>
void run_mix(const char* name, K kern, int threads, int iters, float* out, long long* cyc) {
    kern<<<132, threads>>>(out, cyc, iters);
    kern<<<132, threads>>>(out, cyc, iters);
    cudaDeviceSynchronize();
    long long h[132];
    cudaMemcpy(h, cyc, sizeof(h), cudaMemcpyDeviceToHost);
    double avg = 0;
    for (int i = 0; i < 132; ++i) avg += (double)h[i];
    avg /= 132;
    const int wps = threads / 128;
    printf("MIX %-34s warps/SMSP %d: %.1f cycles per iteration per warp -> %.1f per SMSP per warp-iteration (%s)\n", name, wps, avg / iters, avg / iters / wps,
           cudaGetErrorString(cudaGetLastError()));
}

template <typename K>
void run(const char* name, K kern, int chains, int threads, int iters, float* out, long long* cyc) {
    kern<<<132, threads>>>(out, cyc, iters);
    kern<<<132, threads>>>(out, cyc, iters);
    cudaDeviceSynchronize();
    long long h[132];
    cudaMemcpy(h, cyc, sizeof(h), cudaMemcpyDeviceToHost);
    double avg = 0;
    for (int i = 0; i < 132; ++i) avg += (double)h[i];
    avg /= 132;
    const int warps_per_smsp = threads / 32 / 4 > 0 ? threads / 32 / 4 : 1;
    const double per_warp_instr = avg / ((double)iters * chains);
    printf("%-8s chains %d warps/SMSP %d%s: %.2f cycles per warp-instr per warp -> %.2f cycles per instr per SMSP (%s)\n", name, chains, warps_per_smsp,
           threads < 128 ? " (1 warp only)" : "", per_warp_instr, per_warp_instr / (threads >= 128 ? warps_per_smsp : 1), cudaGetErrorString(cudaGetLastError()));
}

int main() {
    float* out;
    long long* cyc;
    cudaMalloc(&out, 132 * 1024 * 4);
    cudaMalloc(&cyc, 132 * 8);
    const int it = 4096;
    run("HMMA", k_hmma<1>, 1, 32, it, out, cyc);   // latency (1 dependent chain, 1 warp)
    run("HMMA", k_hmma<2>, 2, 32, it, out, cyc);
    run("HMMA", k_hmma<4>, 4, 32, it, out, cyc);
    run("HMMA", k_hmma<8>, 8, 32, it, out, cyc);
    run("HMMA", k_hmma<4>, 4, 128, it, out, cyc);  // 1 warp per SMSP
    run("HMMA", k_hmma<4>, 4, 512, it, out, cyc);  // 4 warps per SMSP
    run("HMMA", k_hmma<2>, 2, 512, it, out, cyc);
    run("HFMA2", k_hfma2<1>, 1, 32, it, out, cyc);
    run("HFMA2", k_hfma2<8>, 8, 32, it, out, cyc);
    run("HFMA2", k_hfma2<8>, 8, 512, it, out, cyc);
    run("LOP3", k_lop3<1>, 1, 32, it, out, cyc);
    run("LOP3", k_lop3<8>, 8, 32, it, out, cyc);
    run("LOP3", k_lop3<8>, 8, 512, it, out, cyc);
    run_mix("8 HFMA2 + 8 LOP3", k_mix<0>, 512, it, out, cyc);   // 16 if the pipes overlap, 32 if they serialise
    run_mix("8 HFMA2 + 8 IADD", k_mix<1>, 512, it, out, cyc);
    run_mix("8 LOP3 + 8 SHR (both integer)", k_mix<2>, 512, it, out, cyc);
    run_mix("8 HFMA2 + 2 HMMA", k_mix<3>, 512, it, out, cyc);
    run_mix("8 HFMA2 + 8 LOP3", k_mix<0>, 128, it, out, cyc);
    return 0;
}
