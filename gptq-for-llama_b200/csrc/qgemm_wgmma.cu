// Batched (prefill) quantized GEMM on the Hopper tensor cores: out[M,N] = x[M,K] . deq(W), int4, M > 8.
//
// This path IS a dense contraction (2*M flop per 0.53 B of weight: compute-bound above M ~ 70), so unlike the decode
// matvec it belongs on wgmma.  Replaces matmul_248_kernel for large M (quant/quant_linear.py:72-137 of the reference;
// there: mma.sync tiles chosen by an autotuner) with one static configuration:
//
//   CTA = 2 consumer warpgroups, tile (128 * WT) rows x 128 columns, K step 64, S-stage shared-memory ring
//   A (activations)  : TMA (cp.async.bulk.tensor.2d), box 64 (k) x 128 rows, SWIZZLE_128B = the canonical K-major layout
//                      (row r at r*128 B, 16-byte chunk c at c ^ (r & 7)); issued by one thread S-2 K steps ahead
//   B (weights)      : each thread dequantises packed words -- one int32 = 8 consecutive k of one column = exactly one 16 B
//                      chunk of the K-major B tile -- with the reference-exact fp16 arithmetic (int4_core.cuh) and stores it
//                      swizzled; the dequantised tile never touches HBM.  Step it+1 is dequantised while the wgmmas of step it run.
//   MMA              : each warpgroup issues wgmma.mma_async m64n128k16 (f16 x f16 -> f32) on its WT x 64 rows from shared-memory
//                      descriptors; fp32 accumulators in registers
//   epilogue         : registers -> fp16 (+ bias) -> global
//
// Numerics: fp16 operands identical to the reference's (exact dequant), fp32 accumulation, one fp16 rounding.
#include "common.cuh"
#include "int4_core.cuh"
#include "kernels.h"
#include "wgmma.cuh"

namespace gptq {
namespace {

using namespace int4;

constexpr int BN = 128, BK = kWgmmaBK;
constexpr int kTileBytes = 128 * BK * 2;  // 16 KB: 128 rows (of A) or 128 columns (of B) x 64 k
constexpr int kGemmThreads = 256;         // two warpgroups: B dequantisation, wgmma, epilogue
constexpr int kAhead = 2;                 // packed words are requested kAhead + 1 K steps before they are dequantised

struct GemmParams {
    const __half* x;
    int64_t ldx;
    const uint32_t* qw[2];  // [1]: second weight of the fused SwiGLU MLP (DUAL)
    const __half* sc[2];
    const uint32_t* qz[2];
    const __half* bias;
    __half* out;
    int64_t ldo;
    int M, K, N, groupsize;
};

// DUAL: out = silu(x.Wg) * (x.Wu) with both fp32 accumulators in registers (fusedmatmul_248_kernel, quant/fused_mlp.py:84-168)
// WT: 64-row M tiles per warpgroup (1 or 2).  With WT = 2 every dequantised B tile feeds 256 rows, which halves the CUDA-core
// dequant work per tensor-core flop.  DUAL uses WT = 1: its two accumulators already take 128 registers per thread.
// S: ring stages; the TMA of A runs S - 2 steps ahead (a stage is rewritten once both warpgroups retired the wgmmas that read it).
template <bool DUAL, int WT, int S>
__global__ void __launch_bounds__(kGemmThreads, 1) qgemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmA, const GemmParams p) {
    constexpr int NW = DUAL ? 2 : 1;
    constexpr int kATile = WT * kTileBytes;  // 128 * WT rows
    constexpr int kAhead2 = S - 2;
    extern __shared__ __align__(16) uint8_t smem_raw[];
    __shared__ __align__(8) unsigned long long full[S];  // A of the stage has landed (TMA complete_tx)
    const int tid = threadIdx.x, wg = tid >> 7, wt = tid & 127, warp = wt >> 5, lane = tid & 31;
    const int m0 = blockIdx.y * (128 * WT), n0 = blockIdx.x * BN;
    const uint32_t sbase = (smem_u32(smem_raw) + 1023u) & ~1023u;  // SWIZZLE_128B atoms need 1024 B alignment
    uint8_t* sptr = smem_raw + (sbase - smem_u32(smem_raw));
    const uint32_t a_s = sbase, b_s = sbase + S * kATile;  // A tiles: [stage][128 * WT rows]; B tiles: [stage][weight]
    uint8_t* b_ptr = sptr + S * kATile;
    const uint32_t full0 = smem_u32(&full[0]);
    const int nkb = p.K / BK;

    auto load_a = [&](int it) {
        const int s = it % S;
        mbar_expect_tx(full0 + s * 8, kATile);
#pragma unroll
        for (int r = 0; r < WT; ++r)
            asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(
                             a_s + s * kATile + r * kTileBytes),
                         "l"(&tmA), "r"(it * BK), "r"(m0 + 128 * r), "r"(full0 + s * 8)
                         : "memory");
    };
    if (tid == 0) {
        for (int i = 0; i < S; ++i) mbar_init(full0 + i * 8, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        for (int it = 0; it < kAhead2 && it < nkb; ++it) load_a(it);
    }

    // ---- B producer role: column n = tid & 127, k-chunks c = (tid >> 7) + 2 i ------------------------------------------------
    const int bn = tid & 127, bc0 = tid >> 7;
    const int col = n0 + bn;
    const int zshift = (col & 7) * 4;
    uint32_t bq[kAhead + 1][NW][4];  // packed words of K steps j .. j + kAhead (a register ring, rotated every step)
    auto load_b = [&](int it, uint32_t (&dst)[NW][4]) {
        const int kr0 = it * (BK / 8);
#pragma unroll
        for (int w = 0; w < NW; ++w)
#pragma unroll
            for (int i = 0; i < 4; ++i) dst[w][i] = __ldg(p.qw[w] + col + (size_t)(kr0 + bc0 + 2 * i) * p.N);
    };
    int cur_grp = -1;
    __half2 za[NW], zb[NW], sc2[NW];
    // dequantise step j (held in bq[0]) into its stage, then rotate the ring and request step j + kAhead + 1
    auto produce_b = [&](int j) {
        const int s = j % S;
        const int grp = (j * BK) / p.groupsize;
        if (grp != cur_grp) {
            cur_grp = grp;
#pragma unroll
            for (int w = 0; w < NW; ++w) {
                const __half sv = __ldg(p.sc[w] + (size_t)grp * p.N + col);
                zero_consts(__ldg(p.qz[w] + (size_t)grp * (p.N >> 3) + (col >> 3)), zshift, za[w], zb[w]);
                sc2[w] = __half2half2(sv);
            }
        }
#pragma unroll
        for (int w = 0; w < NW; ++w) {
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int c = bc0 + 2 * i;
                *reinterpret_cast<uint4*>(b_ptr + (s * NW + w) * kTileBytes + bn * 128 + ((c ^ (bn & 7)) << 4)) =
                    dequant_chunk(bq[0][w][i], za[w], zb[w], sc2[w]);
            }
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic-proxy writes -> visible to wgmma (async proxy)
#pragma unroll
        for (int d = 0; d < kAhead; ++d)
#pragma unroll
            for (int w = 0; w < NW; ++w)
#pragma unroll
                for (int i = 0; i < 4; ++i) bq[d][w][i] = bq[d + 1][w][i];
        if (j + kAhead + 1 < nkb) load_b(j + kAhead + 1, bq[kAhead]);
    };
#pragma unroll
    for (int d = 0; d <= kAhead; ++d)
        if (d < nkb) load_b(d, bq[d]);
    produce_b(0);

    float acc[NW][WT][64];
#pragma unroll
    for (int w = 0; w < NW; ++w)
#pragma unroll
        for (int t = 0; t < WT; ++t)
#pragma unroll
            for (int i = 0; i < 64; ++i) acc[w][t][i] = 0.f;

#pragma unroll 1
    for (int it = 0; it < nkb; ++it) {
        const int s = it % S;
        // B of step it is complete in both warpgroups' halves, and both warpgroups retired the wgmmas of step it - 2
        __syncthreads();
        if (tid == 0 && it + kAhead2 < nkb) load_a(it + kAhead2);  // its stage was last read by step it - 2
        mbar_wait(full0 + s * 8, (it / S) & 1u);
        wgmma_fence();
#pragma unroll
        for (int w = 0; w < NW; ++w) {
            const uint64_t bd = smem_desc(b_s + (s * NW + w) * kTileBytes);
#pragma unroll
            for (int t = 0; t < WT; ++t) {
                const uint64_t ad = smem_desc(a_s + s * kATile + (wg * WT + t) * (kTileBytes / 2));  // 64 rows = 8 KB
#pragma unroll
                for (int k = 0; k < BK / 16; ++k) wgmma_m64n128k16(acc[w][t], ad + 2 * k, bd + 2 * k);
            }
        }
        wgmma_commit();
        // while the tensor cores work: the B tile of step it + 1 (its stage was last read by step it + 1 - S <= it - 3)
        if (it + 1 < nkb) produce_b(it + 1);
#pragma unroll
        for (int w = 0; w < NW; ++w)
#pragma unroll
            for (int t = 0; t < WT; ++t) pin(acc[w][t]);
        wgmma_wait<1>();
    }
    wgmma_wait<0>();
#pragma unroll
    for (int w = 0; w < NW; ++w)
#pragma unroll
        for (int t = 0; t < WT; ++t) pin(acc[w][t]);

    // ---- epilogue: accumulator fragment (row 16 warp + lane / 4 [+ 8], column 8 j + 2 (lane % 4) [+ 1]) -> fp16 (+bias) -> global ----
#pragma unroll
    for (int t = 0; t < WT; ++t) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int row = m0 + 64 * (wg * WT + t) + 16 * warp + (lane >> 2) + 8 * h;
            if (row >= p.M) continue;
            __half* orow = p.out + (size_t)row * p.ldo + n0 + 2 * (lane & 3);
#pragma unroll
            for (int j = 0; j < BN / 8; ++j) {
                float v0 = acc[0][t][4 * j + 2 * h], v1 = acc[0][t][4 * j + 2 * h + 1];
                if constexpr (DUAL) {  // silu(gate) * up on the fp32 accumulators, one rounding (quant/fused_mlp.py:163-165)
                    v0 = swiglu(v0, acc[NW - 1][t][4 * j + 2 * h]);
                    v1 = swiglu(v1, acc[NW - 1][t][4 * j + 2 * h + 1]);
                }
                __half h0 = __float2half_rn(v0), h1 = __float2half_rn(v1);
                if (p.bias != nullptr) {
                    const int c = n0 + 8 * j + 2 * (lane & 3);
                    h0 = __hadd(h0, p.bias[c]);
                    h1 = __hadd(h1, p.bias[c + 1]);
                }
                *reinterpret_cast<__half2*>(orow + 8 * j) = __halves2half2(h0, h1);
            }
        }
    }
}

}  // namespace

bool gemm_tc_supported(const QLinearArgs& a) {
    const gptq_qweight& w = a.w;
    if (w.bits != 4 || a.M <= 8) return false;
    if (a.dual && (!aligned(a.w2.qweight, 4))) return false;
    if (w.groupsize <= 0 || w.groupsize % BK != 0) return false;
    if (w.N % BN != 0 || w.K % BK != 0) return false;
    if (!aligned(a.x, 16) || a.ldx % 8 != 0 || !aligned(a.out, 16) || a.ldo % 8 != 0) return false;
    if (a.norm_w != nullptr || a.residual != nullptr) return false;
    return true;
}

cudaError_t launch_qlinear_gemm_tc(const QLinearArgs& a) {
    CUtensorMap tmA;
    if (!make_kmajor_tensor_map(&tmA, a.x, a.M, a.w.K, a.ldx)) return cudaErrorNotSupported;
    GemmParams p{};
    p.x = reinterpret_cast<const __half*>(a.x);
    p.ldx = a.ldx;
    p.qw[0] = reinterpret_cast<const uint32_t*>(a.w.qweight);
    p.sc[0] = reinterpret_cast<const __half*>(a.w.scales);
    p.qz[0] = reinterpret_cast<const uint32_t*>(a.w.qzeros);
    if (a.dual) {
        p.qw[1] = reinterpret_cast<const uint32_t*>(a.w2.qweight);
        p.sc[1] = reinterpret_cast<const __half*>(a.w2.scales);
        p.qz[1] = reinterpret_cast<const uint32_t*>(a.w2.qzeros);
    }
    p.bias = reinterpret_cast<const __half*>(a.bias);
    p.out = reinterpret_cast<__half*>(a.out);
    p.ldo = a.ldo;
    p.M = a.M; p.K = a.w.K; p.N = a.w.N; p.groupsize = a.w.groupsize;
    // 256-row tiles above 128 rows (single weight); stages fill ~192 KB of the 227 KB a block may use: 48 KB per stage -> 4, 32 KB -> 6
    const int wt = (!a.dual && a.M > 128) ? 2 : 1;
    const int nw = a.dual ? 2 : 1;
    const int stages = (wt + nw == 2) ? 6 : 4;
    const size_t smem = 1024 + (size_t)(wt + nw) * stages * kTileBytes;
    const auto kernel = a.dual ? qgemm_wgmma_kernel<true, 1, 4> : wt == 2 ? qgemm_wgmma_kernel<false, 2, 4> : qgemm_wgmma_kernel<false, 1, 6>;
    return launch_kernel(kernel, dim3(a.w.N / BN, ceil_div(a.M, 128 * wt)), dim3(kGemmThreads), smem, a.stream, false, tmA, p);
}

}  // namespace gptq
