// Causal attention of new query rows over a sequence's cached prefix, read in place from the decode engine's static KV cache: the extend
// path of the engine (a second turn appended to a cached conversation is computed without re-running the conversation).
//
// A span (sequence b, start s, rows n) brings n query rows at positions s .. s + n - 1; its row i attends to keys 0 .. s + i of sequence b,
// whose cache rows s .. s + n - 1 the caller has written (keys after RoPE) before the call.  Only `out` is written.
//
//   CTA = 2 consumer warpgroups (64 query rows each) on one (span, head, 128-query-row tile); thread 0 issues the TMA loads
//   Q, K, V          : all K-major for TMA (head_dim contiguous), box 64 (dims) x 128 rows, SWIZZLE_128B: Q through a map over the q columns
//                      (column h * 128 + {0, 64}), K and V through maps over the layer's cache viewed as [batch * heads * max_seq, 128]
//                      (row (b * heads + h) * max_seq + key0).  Q is loaded once (32 KB); K | V tiles of 128 keys (64 KB) go through a
//                      2-stage ring behind mbarriers: 1 KB alignment + 32 KB + 2 x 64 KB = 161 KB of shared memory
//   S = Q K^T        : wgmma m64n128k16, both operands K-major from shared memory (8 k-steps over head_dim)
//   O += P V         : wgmma m64n128k16 with P from registers (the S accumulator fragment is the A-register layout) and V read MN-major
//                      (transpose-B), 8 k-steps over the 128 keys of the tile
//   masking          : key tiles entirely below the diagonal of every row of the CTA are not masked; the others (the diagonal and the span's
//                      end) are masked element by element with a select, so a NaN score of a masked key becomes -inf, and p = 0.
//                      Cache rows at or past s + n may hold anything (stale rows of an earlier conversation, NaN): P = 0 does not protect
//                      the P.V product against NaN in V (0 * NaN = NaN inside the MMA), so the key tile that reaches past s + n has its
//                      V rows >= s + n zeroed in shared memory before the MMA reads them
//   order            : a CTA walks its key tiles 0, 1, ... in order; no atomics, nothing shared between CTAs, so a span's output depends only
//                      on its own q rows and its sequence's cache, not on the other spans of the call or their order
//
// Numerics: scores are fp16 q . fp16 k with fp32 accumulation, multiplied in fp32 by log2(e) / sqrt(128) (one rounding; the softmax runs in
// base 2 with exp2f).  Online softmax in fp32 (running max and sum per row); P is rounded to fp16 for the P.V product, as flash-style SDPA
// does, while the row sum adds the fp32 p.  O accumulates in fp32, is divided by the fp32 row sum once at the end and rounded to fp16.
#include <cuda_fp16.h>

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

constexpr int kHeadDim = 128, BQ = 128, BKV = 128;
constexpr int kBoxBytes = 128 * kWgmmaBK * 2;  // 16 KB: 128 rows x 64 halves (one TMA box)
constexpr int kTileBytes = 2 * kBoxBytes;      // 32 KB: 128 rows x 128 halves = box of dims 0..63 | box of dims 64..127
constexpr int kStages = 2;
constexpr int kStageBytes = 2 * kTileBytes;  // K tile | V tile
constexpr int kThreads = 256;
constexpr size_t kSmemBytes = 1024 + kTileBytes + (size_t)kStages * kStageBytes;
constexpr float kScaleLog2 = 0.12751743082459868f;  // log2(e) / sqrt(128)

struct CachedAttnParams {
    int seq[kCachedAttnMaxSpans], start[kCachedAttnMaxSpans], rows[kCachedAttnMaxSpans];
    int row0[kCachedAttnMaxSpans];       // first q / out row of the span
    int tile0[kCachedAttnMaxSpans + 1];  // first 128-row query tile of the span; [n_spans] = all tiles
    int n_spans, n_heads, max_seq;
    int64_t ldo;
    __half* out;
};

__global__ void __launch_bounds__(kThreads, 1) cached_attention_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                                                                       const __grid_constant__ CUtensorMap tmV, const CachedAttnParams p) {
    extern __shared__ __align__(16) uint8_t smem_raw[];
    __shared__ __align__(8) unsigned long long bars[1 + kStages];  // [0]: Q landed; [1 + s]: K and V of stage s landed
    const int tid = threadIdx.x, wg = tid >> 7, warp = (tid & 127) >> 5, lane = tid & 31;
    const int h = blockIdx.y;
    // query tile of this CTA, the last tiles first (they have the most key tiles)
    const int t = p.tile0[p.n_spans] - 1 - (int)blockIdx.x;
    int sp = 0;
    while (t >= p.tile0[sp + 1]) ++sp;
    const int s0 = p.start[sp], n = p.rows[sp];
    const int r0 = (t - p.tile0[sp]) * BQ;           // first query row of the tile inside the span
    const int key_end = s0 + n;                      // keys at or past this are never read into the result
    const int nkt = (s0 + min(r0 + BQ, n) - 1) / BKV + 1;  // key tiles up to the last key a row of this tile sees
    const int kv_row0 = (p.seq[sp] * p.n_heads + h) * p.max_seq;  // < 2^31: checked by the host

    const uint32_t sbase = (smem_u32(smem_raw) + 1023u) & ~1023u;  // SWIZZLE_128B atoms need 1024 B alignment
    const uint32_t bar0 = smem_u32(&bars[0]);
    auto load_kv = [&](int kt) {
        const int s = kt % kStages;
        const uint32_t st = sbase + kTileBytes + s * kStageBytes, bar = bar0 + 8 * (1 + s);
        const int row = kv_row0 + kt * BKV;  // rows past this head's max_seq belong to the next head (or read as zeros): masked / zeroed
        mbar_expect_tx(bar, kStageBytes);
        tma_load_2d(st, &tmK, 0, row, bar);
        tma_load_2d(st + kBoxBytes, &tmK, 64, row, bar);
        tma_load_2d(st + kTileBytes, &tmV, 0, row, bar);
        tma_load_2d(st + kTileBytes + kBoxBytes, &tmV, 64, row, bar);
    };
    if (tid == 0) {
        for (int i = 0; i < 1 + kStages; ++i) mbar_init(bar0 + 8 * i, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        mbar_expect_tx(bar0, kTileBytes);
        tma_load_2d(sbase, &tmQ, h * kHeadDim, p.row0[sp] + r0, bar0);  // rows past the span are computed and dropped; past M: zeros
        tma_load_2d(sbase + kBoxBytes, &tmQ, h * kHeadDim + 64, p.row0[sp] + r0, bar0);
        for (int kt = 0; kt < kStages && kt < nkt; ++kt) load_kv(kt);
    }
    __syncthreads();  // the barriers are initialised before anybody waits on them

    // accumulator fragment: row 16 warp + lane / 4 (+ 8 for h2 = 1), column 8 j + 2 (lane % 4) + e at index 4 j + 2 h2 + e
    const int rt = 64 * wg + 16 * warp + (lane >> 2);
    int lim[2];  // the last key of each of the thread's two rows (rows past the span: the span's last key)
#pragma unroll
    for (int h2 = 0; h2 < 2; ++h2) lim[h2] = s0 + min(r0 + rt + 8 * h2, n - 1);
    float o[64], sc[64], m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
#pragma unroll
    for (int i = 0; i < 64; ++i) o[i] = 0.f;

    mbar_wait(bar0, 0);
#pragma unroll 1
    for (int kt = 0; kt < nkt; ++kt) {
        const int s = kt % kStages, k0 = kt * BKV;
        const uint32_t sK = sbase + kTileBytes + s * kStageBytes, sV = sK + kTileBytes;
        mbar_wait(bar0 + 8 * (1 + s), (kt / kStages) & 1u);
        if (k0 + BKV > key_end) {  // the tile reaches past the span's end: zero the V rows >= key_end (both boxes), 16 B per thread and step
            const int z0 = key_end - k0;
            for (int i = tid; i < (BKV - z0) * 16; i += kThreads) {
                const int row = z0 + (i >> 4), c = i & 15;
                asm volatile("st.shared.v4.u32 [%0], {%1, %1, %1, %1};" ::"r"(sV + (c >> 3) * kBoxBytes + row * 128 + (c & 7) * 16), "r"(0) : "memory");
            }
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // the generic stores become visible to the wgmma (async proxy)
            __syncthreads();
        }

        // ---- S = Q K^T for the warpgroup's 64 rows x 128 keys ----
#pragma unroll
        for (int i = 0; i < 64; ++i) sc[i] = 0.f;
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < kHeadDim / 16; ++kk) {
            const int box = kk >> 2;
            wgmma_m64n128k16(sc, smem_desc(sbase + box * kBoxBytes + wg * (kBoxBytes / 2)) + 2 * (kk & 3), smem_desc(sK + box * kBoxBytes) + 2 * (kk & 3));
        }
        wgmma_commit();
        pin(sc);
        wgmma_wait<0>();
        pin(sc);

        // ---- online softmax in base 2 ----
        const bool masked = k0 + BKV - 1 > s0 + r0;  // some row of the CTA does not see every key of the tile
        float mx[2] = {m[0], m[1]};
#pragma unroll
        for (int j = 0; j < BKV / 8; ++j)
#pragma unroll
            for (int h2 = 0; h2 < 2; ++h2)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int i = 4 * j + 2 * h2 + e, key = k0 + 8 * j + 2 * (lane & 3) + e;
                    float v = sc[i] * kScaleLog2;
                    if (masked && key > lim[h2]) v = -INFINITY;
                    sc[i] = v;
                    mx[h2] = fmaxf(mx[h2], v);
                }
        float alpha[2];
#pragma unroll
        for (int h2 = 0; h2 < 2; ++h2) {
            mx[h2] = fmaxf(mx[h2], __shfl_xor_sync(0xffffffffu, mx[h2], 1));
            mx[h2] = fmaxf(mx[h2], __shfl_xor_sync(0xffffffffu, mx[h2], 2));
            // finite from the first tile on: key 0 is visible to every row
            alpha[h2] = exp2f(m[h2] - mx[h2]);
            m[h2] = mx[h2];
            l[h2] *= alpha[h2];
        }
        uint32_t pa[32];  // fp16 P as the A registers of the P.V product: k-step kk holds keys 16 kk .. 16 kk + 15
#pragma unroll
        for (int j = 0; j < BKV / 8; ++j)
#pragma unroll
            for (int h2 = 0; h2 < 2; ++h2) {
                const int i = 4 * j + 2 * h2;
                const float p0 = exp2f(sc[i] - m[h2]), p1 = exp2f(sc[i + 1] - m[h2]);
                l[h2] += p0 + p1;
                const __half2 ph = __floats2half2_rn(p0, p1);
                pa[2 * j + h2] = *reinterpret_cast<const uint32_t*>(&ph);
                o[i] *= alpha[h2];
                o[i + 1] *= alpha[h2];
            }

        // ---- O += P V ----
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < BKV / 16; ++kk) {
            const uint32_t a[4] = {pa[4 * kk], pa[4 * kk + 1], pa[4 * kk + 2], pa[4 * kk + 3]};
            wgmma_m64n128k16_rs_tn(o, a, smem_desc_mn(sV + kk * 16 * 128, kBoxBytes));  // keys 16 kk ..: 16 rows of 128 B further
        }
        wgmma_commit();
        pin(o);
        wgmma_wait<0>();
        pin(o);

        __syncthreads();  // both warpgroups retired the wgmmas that read stage s: the next load may rewrite it
        if (tid == 0 && kt + kStages < nkt) load_kv(kt + kStages);
    }

    // ---- epilogue: O / row sum, fp16 ----
#pragma unroll
    for (int h2 = 0; h2 < 2; ++h2) {
        l[h2] += __shfl_xor_sync(0xffffffffu, l[h2], 1);
        l[h2] += __shfl_xor_sync(0xffffffffu, l[h2], 2);
        const int r = r0 + rt + 8 * h2;
        if (r >= n) continue;
        __half* dst = p.out + (int64_t)(p.row0[sp] + r) * p.ldo + h * kHeadDim + 2 * (lane & 3);
#pragma unroll
        for (int j = 0; j < kHeadDim / 8; ++j)
            *reinterpret_cast<__half2*>(dst + 8 * j) = __floats2half2_rn(o[4 * j + 2 * h2] / l[h2], o[4 * j + 2 * h2 + 1] / l[h2]);
    }
}

}  // namespace

cudaError_t launch_cached_attention(const void* q, int64_t ldq, const void* k_cache, const void* v_cache, int batch, int n_heads, int max_seq, int n_spans,
                                    const int32_t* span_seq, const int32_t* span_start, const int32_t* span_rows, void* out, int64_t ldo,
                                    cudaStream_t stream) {
    CachedAttnParams p{};
    int M = 0, tiles = 0;
    for (int i = 0; i < n_spans; ++i) {
        p.seq[i] = span_seq[i], p.start[i] = span_start[i], p.rows[i] = span_rows[i];
        p.row0[i] = M, p.tile0[i] = tiles;
        M += span_rows[i];
        tiles += ceil_div(span_rows[i], BQ);
    }
    p.tile0[n_spans] = tiles;
    if (tiles == 0) return cudaSuccess;
    p.n_spans = n_spans, p.n_heads = n_heads, p.max_seq = max_seq, p.ldo = ldo;
    p.out = static_cast<__half*>(out);
    CUtensorMap tmQ, tmK, tmV;
    const int kv_rows = batch * n_heads * max_seq;
    if (!make_kmajor_tensor_map(&tmQ, q, M, n_heads * kHeadDim, ldq) || !make_kmajor_tensor_map(&tmK, k_cache, kv_rows, kHeadDim, kHeadDim) ||
        !make_kmajor_tensor_map(&tmV, v_cache, kv_rows, kHeadDim, kHeadDim))
        return cudaErrorNotSupported;
    return launch_kernel(cached_attention_kernel, dim3(tiles, n_heads), dim3(kThreads), kSmemBytes, stream, false, tmQ, tmK, tmV, p);
}

}  // namespace gptq
