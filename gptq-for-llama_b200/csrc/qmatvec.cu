// Skinny (decode) quantized matvec for int4, M <= 8: the batch-1 hot kernel.
//
// out[M,N] = x[M,K] . deq(W)   (matmul_248_kernel, quant/quant_linear.py:84-137 of the reference;
// optional fused SwiGLU over two weights = fusedmatmul_248_kernel, quant/fused_mlp.py:84-168)
//
// Design (HBM-bound: 0.53 B/weight, ~2.8 issue slots per weight at 100 % of HBM):
//  * Work = units of 4 packed rows (32 k) x 256 columns (4 KB of qweight, 1 KB contiguous per row).
//    Units are numbered slab-major (slab = 256 columns) and split evenly over min(2 x 132 SMs, units) CTAs
//    ("stream-K"): every SM streams the same number of bytes whatever the layer shape.
//  * Each of the 8 warps owns a 32-column stripe of the slab and walks the k-steps of its CTA's range.
//    Weights are staged global -> shared memory by 16-byte asynchronous copies (cp.async / LDGSTS, L1 bypass):
//    a lane keeps 16 of them in flight in a private shared-memory ring (2 CTAs/SM x 8 warps x 8 KB = 128 KB in
//    flight per SM) and later reads back exactly the 16 bytes it copied, so the streaming loop has no barriers
//    and no bank conflicts.  The ring runs ahead across slab boundaries and is primed BEFORE
//    griddepcontrol.wait: under programmatic dependent launch the weights of kernel n+1 stream while kernel n
//    reduces.  (A TMA-tiled variant was measured: 512-byte boxes gave the same bandwidth at +60 % instructions.)
//  * The loop is rolled and the kernel is ~10 KB of SASS: a 38 KB unrolled build spent as long fetching
//    instructions as weights (an SM streams only ~56 KB of weights per 4096x4096 layer).
//  * Dequant is exact w.r.t. the reference: nibble -> fp16 by the 0x6400 magic-number trick (LOP3),
//    (w - z) exactly in fp16 (HSUB2 / HFMA2), one HMUL2 by the fp16 scale (the reference's single fp16
//    rounding), then fp16 x fp16 -> fp32 accumulation on the tensor pipe with the roles swapped
//    (mma.m16n8k16: A = 16 output columns x 16 k of weights, B = 16 k x 8 batch rows of x).  This is the
//    same arithmetic as the reference's tl.dot (fp16 operands, fp32 accumulate) at 1/4 of the issue
//    slots a CUDA-core FMA loop needs; the k-order inside a run of 8 is permuted identically in x and W.
//  * Partials of CTAs that share a slab go through a workspace; the last arriver (atomic counter, which
//    it resets) reduces them in a fixed order and zeroes them -> deterministic results, no memset between
//    launches, and the workspace is left zeroed for any shape or kernel that uses it next.
//  * Optional RMSNorm prologue (the reference's rms_norm_fwd_fused, quant/triton_norm.py:21-39) and
//    residual epilogue so that a decoder layer needs 5 launches; PDL hooks (griddepcontrol) let the
//    weight prefetch of kernel n+1 overlap the tail of kernel n.
#include <cstdlib>

#include "common.cuh"
#include "int4_core.cuh"
#include "kernels.h"

namespace gptq {

namespace {

constexpr int kWarps = 8;
constexpr int kThreads = kWarps * 32;
constexpr int kSlabCols = 256;
constexpr int kRingBytesPerWarp = 8192;  // 16 stages x 512 B (8 stages x 1 KB for the dual kernel)

using namespace int4;

#ifdef GPTQ_TRACE
}  // namespace
__device__ unsigned long long* g_trace_buf = nullptr;
namespace {
__device__ __forceinline__ unsigned long long gtime() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
    return t;
}
#define TRACE(slot)                                                                                \
    do {                                                                                           \
        if (g_trace_buf != nullptr && threadIdx.x == 0) g_trace_buf[blockIdx.x * 8 + (slot)] = gtime(); \
    } while (0)
#else
#define TRACE(slot) \
    do {            \
    } while (0)
#endif

struct SkinnyParams {
    const __half* x;
    int64_t ldx;
    const uint32_t* qw[2];
    const __half* sc[2];
    const uint32_t* qz[2];
    const __half* bias;      // [N] or null
    const __half* residual;  // [M, ldr] or null: out = residual + fp16(acc)
    int64_t ldr;
    const __half* norm_w;  // [K] or null: x is RMS-normalised (weight norm_w, eps) before the product
    float eps;
    __half* out;
    int64_t ldo;
    int M, K, N, groupsize;
    int nk;           // k-steps (32 k) per slab
    int total_units;  // nslabs * nk
    int max_contrib;
    float* ws_partial;
    int* ws_counter;
    int xs_pitch;  // halves between x rows in shared memory
};

template <bool DUAL>
__device__ __forceinline__ __half epilogue(const SkinnyParams& p, float a, float b, int m, int n) {
    if constexpr (DUAL) {
        return __float2half_rn(swiglu(a, b));
    } else {
        __half o = __float2half_rn(a);
        if (p.bias != nullptr) o = __hadd(o, p.bias[n]);  // plain loads: __ldg may be speculated above the null check
        if (p.residual != nullptr) o = __hadd(p.residual[(size_t)m * p.ldr + n], o);
        return o;
    }
}

template <bool DUAL>
__global__ void __launch_bounds__(kThreads, 2) qmatvec_int4_kernel(const SkinnyParams p) {
    constexpr int NW = DUAL ? 2 : 1;
    constexpr int STAGE_BYTES = NW * 512;
    constexpr int NST = kRingBytesPerWarp / STAGE_BYTES;  // ring depth in k-steps: 16 (8 for the dual kernel)
    extern __shared__ __align__(16) uint8_t smem_raw[];
    __shared__ float red_s[kWarps];
    __shared__ float rstd_s[8];
    __shared__ int pend_slab_s[2], pend_nc_s[2], pend_last_s[2];

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int g = lane >> 2, t = lane & 3;
    const unsigned nb = gridDim.x;
    const unsigned U = (unsigned)p.total_units;  // U * (nb + 1) < 2^31 (checked on the host)
    const int u_begin = (int)((blockIdx.x * U) / nb);
    const int u_end = (int)(((blockIdx.x + 1) * U) / nb);
    const int nk = p.nk, N = p.N;

    // shared memory: [per-warp weight rings: kWarps x 8 KB][x staging]
    __half* xs = reinterpret_cast<__half*>(smem_raw + kWarps * kRingBytesPerWarp);
    const uint32_t ring_lo = smem_u32(smem_raw) + warp * kRingBytesPerWarp + lane * 16;  // this lane's slot of stage 0
    const uint32_t ring_hi = ring_lo + kRingBytesPerWarp;

    TRACE(0);
    // ---- producer cursor: this lane's next 16 B of weights (row t of the next k-step, columns 4g..4g+3 of its stripe) ----
    const int first_slab = u_begin / nk;
    const int first_ks = u_begin - first_slab * nk;
    const uint4* gp[NW];
    {
        const size_t off = (size_t)(first_ks * 4 + t) * N + first_slab * kSlabCols + warp * 32 + 4 * g;
#pragma unroll
        for (int w = 0; w < NW; ++w) gp[w] = reinterpret_cast<const uint4*>(p.qw[w] + off);
    }
    const long long wrap = (long long)(kSlabCols / 4) - (long long)nk * N;  // next slab, back to row 0 (in uint4 units)
    int p_left = u_end - u_begin;                                          // k-steps not yet requested
    int p_rows_left = nk - first_ks;                                       // ... of them in the current slab
    int p_colw = first_slab * kSlabCols + warp * 32;                       // first column of the warp's stripe
    uint32_t slot = ring_lo;                                               // ring cursor (shared by producer and consumer)
    auto produce = [&](uint32_t dst) {
        if (p_left > 0) {
            if (p_colw < N) {
#pragma unroll
                for (int w = 0; w < NW; ++w) cp_async16(dst + w * 512, gp[w]);
            }
#pragma unroll
            for (int w = 0; w < NW; ++w) gp[w] += N;  // 4 packed rows down
            --p_left;
            if (--p_rows_left == 0) {
#pragma unroll
                for (int w = 0; w < NW; ++w) gp[w] += wrap;
                p_rows_left = nk;
                p_colw += kSlabCols;
            }
        }
        cp_async_commit();  // always commit (possibly empty) so that wait_group counts stay aligned
    };
#pragma unroll 1
    for (int s = 0; s < NST; ++s) produce(ring_lo + s * STAGE_BYTES);  // prime the ring: independent of the previous kernel
    grid_launch_dependents();
    TRACE(1);

    // ---- everything below may depend on the previous kernel's output ---------------------------------
    grid_dependency_wait();
    if (p.norm_w != nullptr) {  // RMSNorm prologue: rstd per row from the full x rows
        for (int m = 0; m < p.M; ++m) {
            const uint4* xr = reinterpret_cast<const uint4*>(p.x + (size_t)m * p.ldx);
            float ss = 0.f;
            for (int i = tid; i < p.K / 8; i += kThreads) {
                const uint4 v = __ldg(xr + i);
                const uint32_t wv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const float2 f = __half22float2(u32_as_h2(wv[j]));
                    ss = fmaf(f.x, f.x, ss);
                    ss = fmaf(f.y, f.y, ss);
                }
            }
            ss = warp_sum(ss);
            if (lane == 0) red_s[warp] = ss;
            __syncthreads();
            float tot = 0.f;
#pragma unroll
            for (int wv = 0; wv < kWarps; ++wv) tot += red_s[wv];
            if (tid == 0) rstd_s[m] = rms_rstd(tot, p.K, p.eps);
            __syncthreads();
        }
    }

    int npend = 0;
    int u = u_begin;
#pragma unroll 1
    while (u < u_end) {
        const int slab = u / nk;
        const int ks0 = u - slab * nk;
        const int nsteps = min(nk - ks0, u_end - u);
        const int col0 = slab * kSlabCols;
        const int ncols = min(kSlabCols, N - col0);
        const bool active = warp * 32 < ncols;
        const int col = col0 + warp * 32 + 4 * g;  // lane's first column

        const int gs_steps = p.groupsize >> 5;  // k-steps per group
        const int zshift = (col & 4) * 4;
        GroupRaw raw[NW];
        GroupConst gc[NW];
        const __half* scp[NW];    // next group's scales / zeros for the lane's columns
        const uint32_t* qzp[NW];
        if (active) {
            const int grp0 = (ks0 * 32) / p.groupsize;
#pragma unroll
            for (int w = 0; w < NW; ++w) {
                scp[w] = p.sc[w] + (size_t)grp0 * N + col;
                qzp[w] = p.qz[w] + (size_t)grp0 * (N >> 3) + (col >> 3);
                raw[w] = load_group_raw(scp[w], qzp[w]);
                scp[w] += N;
                qzp[w] += N >> 3;
            }
        }

        // ---- stage x[k-range of this segment] into shared memory (normalised, k-permuted) -------
        __syncthreads();  // previous segment's readers are done with xs
        {
            const int kbeg = ks0 * 32;
            const int chunks = nsteps * 4;  // 8-half chunks per row
            for (int idx = tid; idx < p.M * chunks; idx += kThreads) {
                const int m = idx / chunks, c = idx - m * chunks;
                uint4 v = __ldg(reinterpret_cast<const uint4*>(p.x + (size_t)m * p.ldx + kbeg) + c);
                if (p.norm_w != nullptr) {
                    const uint4 nw = __ldg(reinterpret_cast<const uint4*>(p.norm_w + kbeg) + c);
                    uint32_t xv[4] = {v.x, v.y, v.z, v.w};
                    const uint32_t wv[4] = {nw.x, nw.y, nw.z, nw.w};
                    const float rs = rstd_s[m];
#pragma unroll
                    for (int j = 0; j < 4; ++j) xv[j] = h2_as_u32(rms_apply2(__half22float2(u32_as_h2(xv[j])), rs, __half22float2(u32_as_h2(wv[j]))));
                    v = make_uint4(xv[0], xv[1], xv[2], xv[3]);
                }
                uint4 o;  // (k0,k4) (k1,k5) (k2,k6) (k3,k7): the order dequant8 produces
                o.x = __byte_perm(v.x, v.z, 0x5410);
                o.y = __byte_perm(v.x, v.z, 0x7632);
                o.z = __byte_perm(v.y, v.w, 0x5410);
                o.w = __byte_perm(v.y, v.w, 0x7632);
                *reinterpret_cast<uint4*>(xs + (size_t)m * p.xs_pitch + c * 8) = o;
            }
        }
        __syncthreads();

        TRACE(2);
        float acc[NW][2][4];
#pragma unroll
        for (int w = 0; w < NW; ++w)
#pragma unroll
            for (int h = 0; h < 2; ++h)
#pragma unroll
                for (int i = 0; i < 4; ++i) acc[w][h][i] = 0.f;

        if (active) {
#pragma unroll
            for (int w = 0; w < NW; ++w) build_group_const(gc[w], raw[w], zshift);
            int steps_left_in_grp = gs_steps - (ks0 % gs_steps);
            if (steps_left_in_grp < nsteps) {
#pragma unroll
                for (int w = 0; w < NW; ++w) {
                    raw[w] = load_group_raw(scp[w], qzp[w]);
                    scp[w] += N;
                    qzp[w] += N >> 3;
                }
            }
            uint32_t xaddr = smem_u32(xs) + ((g < p.M ? g : 0) * p.xs_pitch + t * 8) * 2;

#pragma unroll 1
            for (int step = 0; step < nsteps; ++step) {
                if (steps_left_in_grp == 0) {  // warp-uniform: entered a new group
#pragma unroll
                    for (int w = 0; w < NW; ++w) build_group_const(gc[w], raw[w], zshift);
                    steps_left_in_grp = gs_steps;
                    if (step + gs_steps < nsteps) {
#pragma unroll
                        for (int w = 0; w < NW; ++w) {
                            raw[w] = load_group_raw(scp[w], qzp[w]);
                            scp[w] += N;
                            qzp[w] += N >> 3;
                        }
                    }
                }
                --steps_left_in_grp;
                const uint4 xf = lds128(xaddr);
                xaddr += 64;
                cp_async_wait<NST - 1>();  // this lane's oldest copy has landed (a lane only reads bytes it copied itself)
#pragma unroll
                for (int w = 0; w < NW; ++w) {
                    const uint4 q = lds128(slot + w * 512);
                    uint32_t wf[4][4];
                    dequant8<0>(q.x, gc[w].za01, gc[w].zb01, gc[w].s01, wf[0]);
                    dequant8<1>(q.y, gc[w].za01, gc[w].zb01, gc[w].s01, wf[1]);
                    dequant8<0>(q.z, gc[w].za23, gc[w].zb23, gc[w].s23, wf[2]);
                    dequant8<1>(q.w, gc[w].za23, gc[w].zb23, gc[w].s23, wf[3]);
                    // A rows g / g+8 = columns (col+0, col+1) then (col+2, col+3); two k16 halves each
                    mma_16816(acc[w][0], wf[0][0], wf[1][0], wf[0][1], wf[1][1], xf.x, xf.y);
                    mma_16816(acc[w][0], wf[0][2], wf[1][2], wf[0][3], wf[1][3], xf.z, xf.w);
                    mma_16816(acc[w][1], wf[2][0], wf[3][0], wf[2][1], wf[3][1], xf.x, xf.y);
                    mma_16816(acc[w][1], wf[2][2], wf[3][2], wf[2][3], wf[3][3], xf.z, xf.w);
                }
                produce(slot);  // the slot's registers have been consumed by the mma's above: refill it NST steps ahead
                slot += STAGE_BYTES;
                if (slot == ring_hi) slot = ring_lo;
            }
        } else {
            // this warp owns no columns in the (ragged) last slab: keep its cursors in step
#pragma unroll 1
            for (int step = 0; step < nsteps; ++step) {
                produce(slot);
                slot += STAGE_BYTES;
                if (slot == ring_hi) slot = ring_lo;
            }
        }

        TRACE(3);
        // ---- flush this slab segment ---------------------------------------------------------------
        // lane (g,t) holds batch rows m0 = 2t, m1 = 2t+1 of columns col..col+3:
        //   acc[.][0][0|1] -> col+0, acc[.][0][2|3] -> col+1, acc[.][1][0|1] -> col+2, acc[.][1][2|3] -> col+3
        const int first_cta = (int)(((unsigned)(slab * nk + 1) * nb - 1) / U);
        const int last_cta = (int)(((unsigned)(slab * nk + nk) * nb - 1) / U);
        const int ncontrib = last_cta - first_cta + 1;
        if (ncontrib == 1) {
            if (active) {
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int m = 2 * t + h;
                    if (m < p.M) {
                        __half o[4];
#pragma unroll
                        for (int j = 0; j < 4; ++j) {
                            const float a = acc[0][j >> 1][(j & 1) * 2 + h];
                            const float b = DUAL ? acc[NW - 1][j >> 1][(j & 1) * 2 + h] : 0.f;
                            o[j] = epilogue<DUAL>(p, a, b, m, col + j);
                        }
                        uint2 pk;
                        pk.x = h2_as_u32(__halves2half2(o[0], o[1]));
                        pk.y = h2_as_u32(__halves2half2(o[2], o[3]));
                        *reinterpret_cast<uint2*>(p.out + (size_t)m * p.ldo + col) = pk;
                    }
                }
            }
        } else {
            const int cidx = blockIdx.x - first_cta;
            float* part = p.ws_partial + (size_t)(slab * p.max_contrib + cidx) * (NW * p.M * kSlabCols);
            if (active) {
#pragma unroll
                for (int w = 0; w < NW; ++w)
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const int m = 2 * t + h;
                        if (m < p.M)
                            *reinterpret_cast<float4*>(part + (size_t)(w * p.M + m) * kSlabCols + warp * 32 + 4 * g) =
                                make_float4(acc[w][0][h], acc[w][0][2 + h], acc[w][1][h], acc[w][1][2 + h]);
                    }
            }
            // only the first and the last segment of a CTA can be shared with other CTAs: at most two pending slabs
            if (tid == 0) {
                pend_slab_s[npend] = slab;
                pend_nc_s[npend] = ncontrib;
            }
            ++npend;
        }
        u += nsteps;
    }

    // ---- one release / arrive / acquire round for all shared slabs of this CTA -------------------------
    if (npend > 0) {
        fence_acq_rel_gpu();  // release: this thread's partial stores
        __syncthreads();
        TRACE(4);
        if (tid < npend) {
            const int old = atomicAdd(p.ws_counter + pend_slab_s[tid], 1);
            const int last = (old == pend_nc_s[tid] - 1);
            if (last) p.ws_counter[pend_slab_s[tid]] = 0;  // leave the workspace ready for the next launch
            pend_last_s[tid] = last;
        }
        __syncthreads();
        TRACE(5);
        for (int i = 0; i < npend; ++i) {
            if (!pend_last_s[i]) continue;
            fence_acq_rel_gpu();  // acquire: the other CTAs' partials
            const int slab = pend_slab_s[i], ncontrib = pend_nc_s[i];
            const int col0 = slab * kSlabCols;
            const int ncols = min(kSlabCols, N - col0);
            float* sp = p.ws_partial + (size_t)slab * p.max_contrib * (NW * p.M * kSlabCols);
            if (tid < ncols) {
                for (int m = 0; m < p.M; ++m) {
                    float a = 0.f, b = 0.f;
                    // fixed summation order (deterministic); loads are issued in batches of 8 so that the L2 round trips overlap
#pragma unroll 1
                    for (int c0 = 0; c0 < ncontrib; c0 += 8) {
                        float va[8], vb[8];
#pragma unroll
                        for (int j = 0; j < 8; ++j) {
                            const int c = min(c0 + j, ncontrib - 1);
                            const float* pc = sp + (size_t)c * (NW * p.M * kSlabCols);
                            va[j] = ld_cg(pc + (size_t)m * kSlabCols + tid);
                            if constexpr (DUAL) vb[j] = ld_cg(pc + (size_t)(p.M + m) * kSlabCols + tid);
                        }
#pragma unroll
                        for (int j = 0; j < 8; ++j) {
                            if (c0 + j < ncontrib) {
                                a += va[j];
                                if constexpr (DUAL) b += vb[j];
                                // leave the workspace zeroed (gptq_b200.h): a later call with more slabs has its counters where these
                                // partials lie, and other kernels sharing the workspace accumulate into it
                                float* pc = sp + (size_t)(c0 + j) * (NW * p.M * kSlabCols);
                                pc[(size_t)m * kSlabCols + tid] = 0.f;
                                if constexpr (DUAL) pc[(size_t)(p.M + m) * kSlabCols + tid] = 0.f;
                            }
                        }
                    }
                    p.out[(size_t)m * p.ldo + col0 + tid] = epilogue<DUAL>(p, a, b, m, col0 + tid);
                }
            }
        }
    }
    TRACE(6);
}

}  // namespace

// ------------------------------------------------------------------------------------------------
SkinnyPlan plan_skinny(int M, int K, int N) {
    SkinnyPlan pl{};
    pl.nslabs = ceil_div(N, kSlabCols);
    pl.nk = K / 32;
    pl.total_units = (long long)pl.nslabs * pl.nk;
    pl.grid = (int)(pl.total_units < 2LL * kNumSMs ? pl.total_units : 2LL * kNumSMs);
    int maxc = 1;
    for (int s = 0; s < pl.nslabs; ++s) {
        const long long first = (((long long)s * pl.nk + 1) * pl.grid - 1) / pl.total_units;
        const long long last = (((long long)s * pl.nk + pl.nk) * pl.grid - 1) / pl.total_units;
        maxc = max(maxc, (int)(last - first + 1));
    }
    pl.max_contrib = maxc;
    pl.seg_steps = (int)min((long long)pl.nk, ceil_div((int)pl.total_units, pl.grid) + 0LL);
    return pl;
}

size_t skinny_workspace_bytes(int M, int K, int N, bool dual) {
    if (M < 1 || M > 8 || K % 32 || N % 32) return 0;
    const SkinnyPlan pl = plan_skinny(M, K, N);
    const size_t counters = align256((size_t)pl.nslabs * sizeof(int));
    const size_t partial = (size_t)pl.nslabs * pl.max_contrib * (dual ? 2 : 1) * M * kSlabCols * sizeof(float);
    return counters + partial;
}

bool skinny_supported(const QLinearArgs& a) {
    const gptq_qweight& w = a.w;
    if (w.bits != 4 || a.M < 1 || a.M > 8) return false;
    if (w.groupsize <= 0 || w.groupsize % 32 != 0) return false;
    if (!aligned(a.x, 16) || a.ldx % 8 != 0) return false;
    if (!aligned(w.qweight, 16) || !aligned(w.scales, 8)) return false;
    if (!aligned(a.out, 8) || a.ldo % 4 != 0) return false;
    if (a.dual && (!aligned(a.w2.qweight, 16) || !aligned(a.w2.scales, 8))) return false;
    if (a.norm_w != nullptr && !aligned(a.norm_w, 16)) return false;
    const SkinnyPlan pl = plan_skinny(a.M, w.K, w.N);
    if (pl.total_units * (2LL * kNumSMs + 1) >= (1LL << 31)) return false;  // 32-bit unit arithmetic in the kernel
    const size_t smem = (size_t)kWarps * kRingBytesPerWarp + (size_t)a.M * (pl.seg_steps * 32 + 32) * sizeof(__half);
    return smem <= 110 * 1024;  // two CTAs per SM
}

cudaError_t launch_qlinear_skinny(const QLinearArgs& a, bool pdl) {
    const gptq_qweight& w = a.w;
    const SkinnyPlan pl = plan_skinny(a.M, w.K, w.N);
    SkinnyParams p{};
    p.x = reinterpret_cast<const __half*>(a.x);
    p.ldx = a.ldx;
    p.qw[0] = reinterpret_cast<const uint32_t*>(w.qweight);
    p.sc[0] = reinterpret_cast<const __half*>(w.scales);
    p.qz[0] = reinterpret_cast<const uint32_t*>(w.qzeros);
    if (a.dual) {
        p.qw[1] = reinterpret_cast<const uint32_t*>(a.w2.qweight);
        p.sc[1] = reinterpret_cast<const __half*>(a.w2.scales);
        p.qz[1] = reinterpret_cast<const uint32_t*>(a.w2.qzeros);
    }
    p.bias = reinterpret_cast<const __half*>(a.bias);
    p.residual = reinterpret_cast<const __half*>(a.residual);
    p.ldr = a.ldr;
    p.norm_w = reinterpret_cast<const __half*>(a.norm_w);
    p.eps = a.eps;
    p.out = reinterpret_cast<__half*>(a.out);
    p.ldo = a.ldo;
    p.M = a.M; p.K = w.K; p.N = w.N; p.groupsize = w.groupsize;
    p.nk = pl.nk;
    p.total_units = (int)pl.total_units;
    p.max_contrib = pl.max_contrib;
    const size_t counters = align256((size_t)pl.nslabs * sizeof(int));
    p.ws_counter = reinterpret_cast<int*>(a.workspace);
    p.ws_partial = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(a.workspace) + counters);
    // pitch: 64 B-odd multiple so that up to 8 x-rows map to distinct bank groups
    int pitch = pl.seg_steps * 32;
    if ((pitch / 32) % 2 == 0) pitch += 32;
    p.xs_pitch = pitch;
    const size_t smem = (size_t)kWarps * kRingBytesPerWarp + (size_t)a.M * pitch * sizeof(__half);

    return launch_kernel(a.dual ? qmatvec_int4_kernel<true> : qmatvec_int4_kernel<false>, dim3(pl.grid), dim3(kThreads), smem, a.stream, pdl, p);
}

}  // namespace gptq

#ifdef GPTQ_TRACE
extern "C" int gptq_debug_set_trace(void* buf) {
    unsigned long long* b = reinterpret_cast<unsigned long long*>(buf);
    return (int)cudaMemcpyToSymbol(gptq::g_trace_buf, &b, sizeof(b));
}
#endif
