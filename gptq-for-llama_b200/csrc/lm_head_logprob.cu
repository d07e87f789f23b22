// Per-token log-likelihood through the fp16 lm_head: logprob[m] = l[m, t_m] - logsumexp_v l[m, v], l = fp16(x . W^T), without ever
// writing the [M, V] logits (the scoring / perplexity path of the engine; the reference materialises them, llama.py:246-256).
//
//   CTA = 2 consumer warpgroups, tile 256 rows of x x 128 vocabulary rows of W, K step 64, 4-stage shared-memory ring
//   x, W             : both K-major fp16 (W [V, K] as nn.Linear stores it), both by TMA (cp.async.bulk.tensor.2d, box 64 (k) x 128 rows,
//                      SWIZZLE_128B), issued by one thread two K steps ahead; rows past M or V arrive as zeros
//   MMA              : each warpgroup issues wgmma.mma_async m64n128k16 (f16 x f16 -> f32) on its 128 rows; fp32 accumulators in registers
//   ring depth       : a stage is 256 x 64 + 128 x 64 halves = 48 KB, so 4 stages (192 KB + 1 KB of alignment slack) fit the 227 KB a block may
//                      use and 5 do not.  As in qgemm_wgmma.cu a stage is rewritten once both warpgroups retired the wgmmas that read it (one
//                      block barrier per K step, wgmma.wait_group 1), so the TMA runs S - 2 = 2 K steps ahead.
//   epilogue         : per (row, vocabulary tile): every accumulator rounded to fp16 and back (the reference's lm_head output is fp16),
//                      columns >= V masked, row max and sum exp(l - max) over the tile with quad shuffles -> one float2 partial; the lane
//                      holding column t_m writes the target logit
//   combine          : one warp per row merges the row's ceil(V / 128) partials in a fixed order (lane i: tiles i, i + 32, ...; then a
//                      butterfly), so a row's result depends on nothing but its own x row, W and target; it zeroes the partials it read
//
// Numerics: fp32 accumulation, one fp16 rounding per logit, fp32 log-softmax on the fp16 logits.
#include "common.cuh"
#include "int4_core.cuh"
#include "kernels.h"
#include "wgmma.cuh"

namespace gptq {
namespace {

using int4::mbar_expect_tx;
using int4::mbar_init;
using int4::mbar_wait;
using int4::smem_u32;

constexpr int BM = 256, BN = 128, BK = kWgmmaBK;
constexpr int kTileBytes = 128 * BK * 2;       // 16 KB: 128 rows x 64 k
constexpr int kStageBytes = 3 * kTileBytes;    // x rows 0..127 | x rows 128..255 | W rows n0..n0+127
constexpr int kStages = 4;
constexpr int kThreads = 256;
constexpr size_t kSmemBytes = 1024 + (size_t)kStages * kStageBytes;
constexpr int kCombineWarps = 8;
constexpr int kGroupM = 8;

struct LogprobParams {
    const int32_t* targets;
    float2* part;   // [M, ntiles] (max, sum exp(l - max)) per row and vocabulary tile
    float* tlogit;  // [M] logit of the target
    int M, K, V, ntiles, mtiles;
};

__global__ void __launch_bounds__(kThreads, 1) lm_head_logprob_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmW,
                                                                      const LogprobParams p) {
    extern __shared__ __align__(16) uint8_t smem_raw[];
    __shared__ __align__(8) unsigned long long full[kStages];  // the stage has landed (TMA complete_tx)
    const int tid = threadIdx.x, wg = tid >> 7, warp = (tid & 127) >> 5, lane = tid & 31;
    // grouped raster: kGroupM row tiles walk the vocabulary together, so that their x rows (kGroupM x 2 MB at K = 4096) and the W tiles in
    // flight stay in L2, and W is streamed from HBM once per kGroupM row tiles
    const int per_group = kGroupM * p.ntiles, grp = blockIdx.x / per_group, r = blockIdx.x % per_group;
    const int gm = min(kGroupM, p.mtiles - grp * kGroupM);
    const int m0 = (grp * kGroupM + r % gm) * BM, tile = r / gm, n0 = tile * BN;
    const uint32_t sbase = (smem_u32(smem_raw) + 1023u) & ~1023u;  // SWIZZLE_128B atoms need 1024 B alignment
    const uint32_t full0 = smem_u32(&full[0]);
    const int nkb = p.K / BK;

    auto load = [&](int it) {
        const int s = it % kStages;
        const uint32_t st = sbase + s * kStageBytes, bar = full0 + s * 8;
        mbar_expect_tx(bar, kStageBytes);
        tma_load_2d(st, &tmX, it * BK, m0, bar);
        tma_load_2d(st + kTileBytes, &tmX, it * BK, m0 + 128, bar);
        tma_load_2d(st + 2 * kTileBytes, &tmW, it * BK, n0, bar);
    };
    if (tid == 0) {
        for (int i = 0; i < kStages; ++i) mbar_init(full0 + i * 8, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        for (int it = 0; it < kStages - 2 && it < nkb; ++it) load(it);
    }

    float acc[2][64];
#pragma unroll
    for (int t = 0; t < 2; ++t)
#pragma unroll
        for (int i = 0; i < 64; ++i) acc[t][i] = 0.f;

#pragma unroll 1
    for (int it = 0; it < nkb; ++it) {
        const int s = it % kStages;
        // both warpgroups retired the wgmmas of step it - 2, whose stage the next load rewrites
        __syncthreads();
        if (tid == 0 && it + kStages - 2 < nkb) load(it + kStages - 2);
        mbar_wait(full0 + s * 8, (it / kStages) & 1u);
        wgmma_fence();
        const uint32_t st = sbase + s * kStageBytes;
        const uint64_t bd = smem_desc(st + 2 * kTileBytes);
#pragma unroll
        for (int t = 0; t < 2; ++t) {
            const uint64_t ad = smem_desc(st + (wg * 2 + t) * (kTileBytes / 2));  // 64 rows = 8 KB
#pragma unroll
            for (int k = 0; k < BK / 16; ++k) wgmma_m64n128k16(acc[t], ad + 2 * k, bd + 2 * k);
        }
        wgmma_commit();
        pin(acc[0]);
        pin(acc[1]);
        wgmma_wait<1>();
    }
    wgmma_wait<0>();
    pin(acc[0]);
    pin(acc[1]);

    // ---- epilogue: accumulator fragment (row 16 warp + lane / 4 [+ 8], column 8 j + 2 (lane % 4) [+ 1]); the four lanes of a quad hold one row ----
    // Rows past M hold zeros and are reduced like the others (every lane must take part in the shuffles); only their stores are skipped.
#pragma unroll
    for (int t = 0; t < 2; ++t) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int row = m0 + 64 * (wg * 2 + t) + 16 * warp + (lane >> 2) + 8 * h;
            const int tgt = row < p.M ? __ldg(p.targets + row) : -1;
            const int c0 = n0 + 2 * (lane & 3);
            float mx = -INFINITY, tl = 0.f;
            bool has_t = false;
#pragma unroll
            for (int j = 0; j < BN / 8; ++j)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int c = c0 + 8 * j + e;
                    const float l = __half2float(__float2half_rn(acc[t][4 * j + 2 * h + e]));
                    if (c < p.V) mx = fmaxf(mx, l);
                    if (c == tgt) tl = l, has_t = true;
                }
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));  // finite: column n0 < V lies in every row's quad
            float sum = 0.f;
#pragma unroll
            for (int j = 0; j < BN / 8; ++j)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int c = c0 + 8 * j + e;
                    if (c < p.V) sum += expf(__half2float(__float2half_rn(acc[t][4 * j + 2 * h + e])) - mx);
                }
            sum += __shfl_xor_sync(0xffffffffu, sum, 1);
            sum += __shfl_xor_sync(0xffffffffu, sum, 2);
            if (row < p.M) {
                if ((lane & 3) == 0) p.part[(size_t)row * p.ntiles + tile] = make_float2(mx, sum);
                if (has_t) p.tlogit[row] = tl;  // a target >= V can only meet a masked column: the combine ignores its logit
            }
        }
    }
}

// (m, s) <- (m, s) merged with (mo, so): max and sum exp(l - max) of the union.  Commutative bit for bit (fmaxf, and a + b == b + a).
__device__ __forceinline__ void lse_merge(float& m, float& s, float mo, float so) {
    if (mo == -INFINITY) return;
    if (m == -INFINITY) {
        m = mo, s = so;
        return;
    }
    const float mn = fmaxf(m, mo);
    s = s * expf(m - mn) + so * expf(mo - mn);
    m = mn;
}

__global__ void __launch_bounds__(32 * kCombineWarps) lm_head_logprob_combine_kernel(const LogprobParams p, float* __restrict__ out) {
    const int row = blockIdx.x * kCombineWarps + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (row >= p.M) return;
    float2* part = p.part + (size_t)row * p.ntiles;
    float m = -INFINITY, s = 0.f;
    for (int i = lane; i < p.ntiles; i += 32) {
        const float2 q = part[i];
        part[i] = make_float2(0.f, 0.f);  // the workspace is left zeroed
        lse_merge(m, s, q.x, q.y);
    }
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const float mo = __shfl_xor_sync(0xffffffffu, m, o), so = __shfl_xor_sync(0xffffffffu, s, o);
        lse_merge(m, s, mo, so);
    }
    if (lane == 0) {
        const int t = p.targets[row];
        const float tl = p.tlogit[row];
        p.tlogit[row] = 0.f;
        // a target outside [0, V) has no logit (the host rejects it before the launch): NaN, nothing read out of bounds
        out[row] = (t >= 0 && t < p.V) ? tl - (m + logf(s)) : __int_as_float(0x7fc00000);
    }
}

}  // namespace

size_t lm_head_logprob_workspace_bytes(int M, int V) {
    if (M <= 0 || V <= 0) return 0;
    const size_t part = (size_t)M * ceil_div(V, BN) * sizeof(float2);
    return align256(part + (size_t)M * sizeof(float));
}

cudaError_t launch_lm_head_logprob(const void* x, int64_t ldx, const void* w, int64_t ldw, int M, int K, int V, const int32_t* targets, float* logprob,
                                   void* workspace, cudaStream_t stream) {
    CUtensorMap tmX, tmW;
    if (!make_kmajor_tensor_map(&tmX, x, M, K, ldx) || !make_kmajor_tensor_map(&tmW, w, V, K, ldw)) return cudaErrorNotSupported;
    LogprobParams p{};
    p.targets = targets;
    p.ntiles = ceil_div(V, BN);
    p.part = reinterpret_cast<float2*>(workspace);
    p.tlogit = reinterpret_cast<float*>(p.part + (size_t)M * p.ntiles);
    p.mtiles = ceil_div(M, BM);
    p.M = M, p.K = K, p.V = V;
    const cudaError_t e = launch_kernel(lm_head_logprob_kernel, dim3(p.mtiles * p.ntiles), dim3(kThreads), kSmemBytes, stream, false, tmX, tmW, p);
    if (e != cudaSuccess) return e;
    lm_head_logprob_combine_kernel<<<ceil_div(M, kCombineWarps), 32 * kCombineWarps, 0, stream>>>(p, logprob);
    return cudaGetLastError();
}

}  // namespace gptq
