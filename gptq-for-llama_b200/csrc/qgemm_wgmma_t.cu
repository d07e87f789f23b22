// Transposed quantized GEMM on the Hopper tensor cores: out[M,K] = g[M,N] . deq(W)^T, int4, M > 8.
//
// The gradient of a quantized linear with respect to its input (QuantLinearFunction.backward): what fine-tuning adapters over a frozen
// 4-bit model spends its backward pass on.  Replaces transpose_matmul_248_kernel (quant/quant_linear.py:191-258 of the reference; there:
// mma.sync tiles chosen by an autotuner) with one static configuration, the mirror image of qgemm_wgmma.cu.  The reduction runs over N
// (the columns of the packed weight); the output feature is k.
//
//   CTA = 2 consumer warpgroups, tile (128 * WT) rows x 128 output features, reduction step 64 columns of N, S-stage shared-memory ring
//   A (gradients)    : reduction-contiguous, so a K-major TMA tile exactly like x in the forward kernel: box 64 (n) x 128 rows,
//                      SWIZZLE_128B; issued by one thread S-2 steps ahead.  Rows past M arrive as zeros; their stores are guarded.
//   B (weights)      : one packed int32 = 8 consecutive k of one column n.  Here k is the OUTPUT dimension, so the 8 dequantised halves are
//                      one 16 B chunk of an MN-major B tile (feature-contiguous): reduction row n at n * 128 B inside a box of 64 features
//                      (8 KB; two boxes per tile), chunk c at c ^ (n & 7).  wgmma reads it with the transpose-B immediate (smem_desc_mn,
//                      LBO = 8 KB between the boxes, SBO = 1 KB between 8-row groups).  A warp reads 32 consecutive n of one packed row (one
//                      coalesced 128 B load) and its 32 16-byte stores of a chunk column are bank-conflict free under the swizzle.
//                      A thread owns column n of the step and 4 consecutive packed rows = 32 consecutive k: one scale and one zero per
//                      thread and step (groupsize % 32 == 0), loaded with the packed words kAhead + 1 steps before they are needed.
//                      Step it+1 is dequantised while the wgmmas of step it run; the dequantised tile never touches HBM.
//   MMA              : wgmma.mma_async m64n128k16 (f16 x f16 -> f32), A K-major and B MN-major from shared-memory descriptors
//   epilogue         : registers -> fp16 -> global
//
// Numerics: fp16 operands identical to the reference's (exact dequant, int4_core.cuh), fp32 accumulation, one fp16 rounding.  No atomics,
// no workspace, nothing shared between CTAs: a row's result does not depend on the other rows of the call and is the same from run to run.
#include "common.cuh"
#include "int4_core.cuh"
#include "kernels.h"
#include "wgmma.cuh"

namespace gptq {
namespace {

using namespace int4;

constexpr int BF = 128, BR = kWgmmaBK;     // output features (k) per CTA; reduction columns (n) per step
constexpr int kTileBytes = 128 * BR * 2;   // 16 KB: 128 rows of A x 64 n, or 64 n x 128 features of B
constexpr int kBoxBytes = BR * 128;        // 8 KB: 64 reduction rows x 64 features (one swizzle-atom column of the B tile)
constexpr int kGemmTThreads = 256;         // two warpgroups: B dequantisation, wgmma, epilogue
constexpr int kAhead = 2;                  // packed words are requested kAhead + 1 steps before they are dequantised

struct GemmTParams {
    const uint32_t* qw;
    const __half* sc;
    const uint32_t* qz;
    __half* out;
    int64_t ldo;
    int M, K, N, groupsize;
};

struct PackedCol {  // one thread's share of a step: 4 packed rows (32 k) of one column, with the column's scale and zeros word
    uint32_t q[4];
    uint32_t z;
    __half s;
};

// WT: 64-row M tiles per warpgroup (1 or 2); S: ring stages (the TMA of A runs S - 2 steps ahead), as in qgemm_wgmma_kernel.
template <int WT, int S>
__global__ void __launch_bounds__(kGemmTThreads, 1) qgemm_wgmma_t_kernel(const __grid_constant__ CUtensorMap tmG, const GemmTParams p) {
    constexpr int kATile = WT * kTileBytes;  // 128 * WT rows
    constexpr int kAhead2 = S - 2;
    extern __shared__ __align__(16) uint8_t smem_raw[];
    __shared__ __align__(8) unsigned long long full[S];  // A of the stage has landed (TMA complete_tx)
    const int tid = threadIdx.x, wg = tid >> 7, warp = (tid & 127) >> 5, lane = tid & 31;
    const int m0 = blockIdx.y * (128 * WT), k0 = blockIdx.x * BF;
    const uint32_t sbase = (smem_u32(smem_raw) + 1023u) & ~1023u;  // SWIZZLE_128B atoms need 1024 B alignment
    uint8_t* sptr = smem_raw + (sbase - smem_u32(smem_raw));
    const uint32_t a_s = sbase, b_s = sbase + S * kATile;  // A tiles: [stage][128 * WT rows]; B tiles: [stage]
    uint8_t* b_ptr = sptr + S * kATile;
    const uint32_t full0 = smem_u32(&full[0]);
    const int nsteps = p.N / BR;

    auto load_a = [&](int it) {
        const int s = it % S;
        mbar_expect_tx(full0 + s * 8, kATile);
#pragma unroll
        for (int r = 0; r < WT; ++r) tma_load_2d(a_s + s * kATile + r * kTileBytes, &tmG, it * BR, m0 + 128 * r, full0 + s * 8);
    };
    if (tid == 0) {
        for (int i = 0; i < S; ++i) mbar_init(full0 + i * 8, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        for (int it = 0; it < kAhead2 && it < nsteps; ++it) load_a(it);
    }

    // ---- B producer role: reduction row bn = column n of the step, packed rows pr0 .. pr0 + 3 of the tile (32 consecutive k) ---------
    const int bn = ((tid >> 5) & 1) * 32 + lane, pr0 = (tid >> 6) * 4;
    const int zshift = (bn & 7) * 4;
    const int grp = (k0 + pr0 * 8) / p.groupsize;  // groupsize % 32 == 0: the thread's 32 k share a group, the same one at every step
    const uint32_t* qwp = p.qw + (size_t)(k0 / 8 + pr0) * p.N + bn;
    const __half* scp = p.sc + (size_t)grp * p.N + bn;
    const uint32_t* qzp = p.qz + (size_t)grp * (p.N >> 3) + (bn >> 3);
    uint8_t* b_dst = b_ptr + (pr0 >> 3) * kBoxBytes + bn * 128;  // the thread's row of its 64-feature box
    PackedCol bq[kAhead + 1] = {};  // steps j .. j + kAhead (a register ring, rotated every step)
    auto load_b = [&](int it, PackedCol& dst) {
        const int n = it * BR;
#pragma unroll
        for (int i = 0; i < 4; ++i) dst.q[i] = __ldg(qwp + (size_t)i * p.N + n);
        dst.s = __ldg(scp + n);
        dst.z = __ldg(qzp + (n >> 3));
    };
    // dequantise step j (held in bq[0]) into its stage, then rotate the ring and request step j + kAhead + 1
    auto produce_b = [&](int j) {
        const int s = j % S;
        __half2 za, zb;
        zero_consts(bq[0].z, zshift, za, zb);
        const __half2 sc2 = __half2half2(bq[0].s);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int c = (pr0 & 7) + i;
            *reinterpret_cast<uint4*>(b_dst + s * kTileBytes + ((c ^ (bn & 7)) << 4)) = dequant_chunk(bq[0].q[i], za, zb, sc2);
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic-proxy writes -> visible to wgmma (async proxy)
#pragma unroll
        for (int d = 0; d < kAhead; ++d) bq[d] = bq[d + 1];
        if (j + kAhead + 1 < nsteps) load_b(j + kAhead + 1, bq[kAhead]);
    };
#pragma unroll
    for (int d = 0; d <= kAhead; ++d)
        if (d < nsteps) load_b(d, bq[d]);
    produce_b(0);

    float acc[WT][64];
#pragma unroll
    for (int t = 0; t < WT; ++t)
#pragma unroll
        for (int i = 0; i < 64; ++i) acc[t][i] = 0.f;

#pragma unroll 1
    for (int it = 0; it < nsteps; ++it) {
        const int s = it % S;
        // B of step it is complete in both warpgroups' halves, and both warpgroups retired the wgmmas of step it - 2
        __syncthreads();
        if (tid == 0 && it + kAhead2 < nsteps) load_a(it + kAhead2);  // its stage was last read by step it - 2
        mbar_wait(full0 + s * 8, (it / S) & 1u);
        wgmma_fence();
        const uint64_t bd = smem_desc_mn(b_s + s * kTileBytes, kBoxBytes);
#pragma unroll
        for (int t = 0; t < WT; ++t) {
            const uint64_t ad = smem_desc(a_s + s * kATile + (wg * WT + t) * (kTileBytes / 2));  // 64 rows = 8 KB
#pragma unroll
            for (int k = 0; k < BR / 16; ++k) wgmma_m64n128k16_tn(acc[t], ad + 2 * k, bd + k * (16 * 128 >> 4));  // 16 reduction rows of 128 B
        }
        wgmma_commit();
        // while the tensor cores work: the B tile of step it + 1 (its stage was last read by step it + 1 - S <= it - 3)
        if (it + 1 < nsteps) produce_b(it + 1);
#pragma unroll
        for (int t = 0; t < WT; ++t) pin(acc[t]);
        wgmma_wait<1>();
    }
    wgmma_wait<0>();
#pragma unroll
    for (int t = 0; t < WT; ++t) pin(acc[t]);

    // ---- epilogue: accumulator fragment (row 16 warp + lane / 4 [+ 8], feature 8 j + 2 (lane % 4) [+ 1]) -> fp16 -> global ----
#pragma unroll
    for (int t = 0; t < WT; ++t) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int row = m0 + 64 * (wg * WT + t) + 16 * warp + (lane >> 2) + 8 * h;
            if (row >= p.M) continue;
            __half* orow = p.out + (size_t)row * p.ldo + k0 + 2 * (lane & 3);
#pragma unroll
            for (int j = 0; j < BF / 8; ++j)
                *reinterpret_cast<__half2*>(orow + 8 * j) = __floats2half2_rn(acc[t][4 * j + 2 * h], acc[t][4 * j + 2 * h + 1]);
        }
    }
}

}  // namespace

bool gemm_t_tc_supported(const void* g, int64_t ldg, const gptq_qweight& w, const void* out, int64_t ldo, int M) {
    if (w.bits != 4 || M <= 8) return false;
    if (w.groupsize <= 0 || w.groupsize % 32 != 0) return false;  // a thread's 32 consecutive k share one scale and zero
    if (w.K % BF != 0 || w.N % BR != 0) return false;
    if (!aligned(g, 16) || ldg % 8 != 0 || !aligned(out, 16) || ldo % 8 != 0) return false;  // TMA rows of g, paired fp16 stores of out
    if (ceil_div(M, 128) > 65535) return false;                                                 // gridDim.y
    return true;
}

cudaError_t launch_qlinear_transpose_tc(const void* g, int64_t ldg, const gptq_qweight& w, void* out, int64_t ldo, int M, cudaStream_t stream) {
    CUtensorMap tmG;
    if (!make_kmajor_tensor_map(&tmG, g, M, w.N, ldg)) return cudaErrorNotSupported;
    GemmTParams p{};
    p.qw = reinterpret_cast<const uint32_t*>(w.qweight);
    p.sc = reinterpret_cast<const __half*>(w.scales);
    p.qz = reinterpret_cast<const uint32_t*>(w.qzeros);
    p.out = reinterpret_cast<__half*>(out);
    p.ldo = ldo;
    p.M = M; p.K = w.K; p.N = w.N; p.groupsize = w.groupsize;
    // 256-row tiles above 128 rows; stages fill ~192 KB of the 227 KB a block may use: 48 KB per stage -> 4, 32 KB -> 6
    const int wt = M > 128 ? 2 : 1;
    const int stages = wt == 2 ? 4 : 6;
    const size_t smem = 1024 + (size_t)(wt + 1) * stages * kTileBytes;
    return launch_kernel(wt == 2 ? qgemm_wgmma_t_kernel<2, 4> : qgemm_wgmma_t_kernel<1, 6>, dim3(w.K / BF, ceil_div(M, 128 * wt)), dim3(kGemmTThreads), smem,
                         stream, false, tmG, p);
}

}  // namespace gptq
