// Grid-barrier latency on H100 under HBM load: one CTA per SM, thread 0 of every CTA synchronises ROUNDS times; the other
// warps stream a large buffer (background traffic like the decode kernel's weight stream).  Per variant: time from the LAST
// arrival to the median / last release, in ns (globaltimer).
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o barrier barrier.cu
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <vector>
#include <cuda_runtime.h>

constexpr int ROUNDS = 64;

__device__ __forceinline__ unsigned long long gtime() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
    return t;
}

// V: 0 red.release + ld.acquire poll | 1 same + nanosleep(100) | 2 relaxed poll + fence.acquire once | 3 two-level (groups of 16 CTAs)
template <int V, bool LOAD>
__global__ void __launch_bounds__(576, 1) k_bar(unsigned long long* bar, unsigned long long* tarr, unsigned long long* tpass, const uint4* big, size_t big_n, float* sink,
                                                volatile int* stop) {
    const int tid = threadIdx.x;
    if (tid >= 32) {
        if (!LOAD) return;
        // background: every warp streams its own region until thread 0 of CTA 0 raises the stop flag
        uint4 acc = make_uint4(0, 0, 0, 0);
        size_t i = ((size_t)blockIdx.x * 544 + (tid - 32)) * 64 % big_n;
        while (*stop == 0) {
#pragma unroll
            for (int u = 0; u < 8; ++u) {
                uint4 v;
                asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(big + (i + u * 544 * 132) % big_n));
                acc.x ^= v.x; acc.y ^= v.y; acc.z ^= v.z; acc.w ^= v.w;
            }
            i = (i + 8ull * 544 * 132 + 1) % big_n;
        }
        if (acc.x == 0x12345) sink[tid] = (float)acc.y;
        return;
    }
    if (tid != 0) return;
    unsigned long long target = 0;
    const unsigned nb = gridDim.x;
    for (int r = 0; r < ROUNDS; ++r) {
        // a "phase": ~3 us of nothing, slightly different per CTA
        const unsigned long long t0 = gtime();
        while (gtime() - t0 < 3000 + (blockIdx.x * 37 % 500)) {}
        tarr[r * nb + blockIdx.x] = gtime();
        if (V == 3) {
            const unsigned grp = blockIdx.x / 16, ngrp = (nb + 15) / 16, gsize = min(16u, nb - grp * 16);
            unsigned long long* gc = bar + 32 + grp * 32;  // one 256-byte line per group counter
            unsigned long long old;
            asm volatile("atom.acq_rel.gpu.global.add.u64 %0, [%1], 1;" : "=l"(old) : "l"(gc) : "memory");
            target += ngrp;
            if ((old + 1) % gsize == 0) asm volatile("red.release.gpu.global.add.u64 [%0], 1;" ::"l"(bar) : "memory");
            unsigned long long v;
            do {
                asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(bar) : "memory");
            } while (v < target);
        } else {
            target += nb;
            asm volatile("red.release.gpu.global.add.u64 [%0], 1;" ::"l"(bar) : "memory");
            unsigned long long v;
            if (V == 2) {
                do {
                    asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(bar) : "memory");
                } while (v < target);
                asm volatile("fence.acq_rel.gpu;" ::: "memory");
            } else {
                do {
                    asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(bar) : "memory");
                    if (V == 1 && v < target) __nanosleep(100);
                } while (v < target);
            }
        }
        tpass[r * nb + blockIdx.x] = gtime();
    }
    if (blockIdx.x == 0) *stop = 1;
}

template <int V, bool LOAD>
void run(const char* name, int nb, unsigned long long* bar, unsigned long long* tarr, unsigned long long* tpass, const uint4* big, size_t big_n, float* sink, int* stop) {
    cudaMemset(bar, 0, 65536);
    cudaMemset(stop, 0, 4);
    void* args[] = {&bar, &tarr, &tpass, (void*)&big, &big_n, &sink, &stop};
    cudaError_t e = cudaLaunchCooperativeKernel((void*)k_bar<V, LOAD>, dim3(nb), dim3(576), args, 0, 0);
    cudaDeviceSynchronize();
    std::vector<unsigned long long> a(ROUNDS * nb), p(ROUNDS * nb);
    cudaMemcpy(a.data(), tarr, a.size() * 8, cudaMemcpyDeviceToHost);
    cudaMemcpy(p.data(), tpass, p.size() * 8, cudaMemcpyDeviceToHost);
    std::vector<double> med, last;
    for (int r = 8; r < ROUNDS; ++r) {
        const unsigned long long la = *std::max_element(a.begin() + r * nb, a.begin() + (r + 1) * nb);
        std::vector<unsigned long long> pp(p.begin() + r * nb, p.begin() + (r + 1) * nb);
        std::sort(pp.begin(), pp.end());
        med.push_back((double)pp[nb / 2] - (double)la);
        last.push_back((double)pp[nb - 1] - (double)la);
    }
    std::sort(med.begin(), med.end());
    std::sort(last.begin(), last.end());
    printf("%-62s load=%d  last arrival -> median release %6.0f ns, -> last release %6.0f ns   (%s)\n", name, (int)LOAD, med[med.size() / 2], last[last.size() / 2],
           cudaGetErrorString(e == cudaSuccess ? cudaGetLastError() : e));
}

int main() {
    cudaDeviceProp pr;
    cudaGetDeviceProperties(&pr, 0);
    const int nb = pr.multiProcessorCount;
    unsigned long long *bar, *tarr, *tpass;
    float* sink;
    int* stop;
    uint4* big;
    const size_t big_n = (size_t)1 << 27;  // 2 GiB of uint4
    cudaMalloc(&bar, 65536);
    cudaMalloc(&tarr, ROUNDS * nb * 8);
    cudaMalloc(&tpass, ROUNDS * nb * 8);
    cudaMalloc(&sink, 4096);
    cudaMalloc(&stop, 4);
    cudaMalloc(&big, big_n * 16);
    cudaMemset(big, 1, big_n * 16);
    run<0, false>("red.release + ld.acquire poll (the kernel's barrier)", nb, bar, tarr, tpass, big, big_n, sink, stop);
    run<0, true>("red.release + ld.acquire poll (the kernel's barrier)", nb, bar, tarr, tpass, big, big_n, sink, stop);
    run<1, true>("  + nanosleep(100) between polls", nb, bar, tarr, tpass, big, big_n, sink, stop);
    run<2, true>("relaxed poll + one fence.acq_rel at the end", nb, bar, tarr, tpass, big, big_n, sink, stop);
    run<2, false>("relaxed poll + one fence.acq_rel at the end", nb, bar, tarr, tpass, big, big_n, sink, stop);
    run<3, true>("two-level: groups of 16 CTAs (atom), top-level counter polled", nb, bar, tarr, tpass, big, big_n, sink, stop);
    run<3, false>("two-level: groups of 16 CTAs (atom), top-level counter polled", nb, bar, tarr, tpass, big, big_n, sink, stop);
    return 0;
}
