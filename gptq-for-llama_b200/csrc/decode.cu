// Decode engine: one token step of a GPTQ LLaMA on a static KV cache (see include/gptq_b200.h).
//
// What it replaces in the reference: the body of the per-token loop of llama.py:419-433, i.e. HF's
// LlamaDecoderLayer over TritonLlamaRMSNorm (quant/triton_norm.py), QuantLlamaAttention.forward
// (quant/fused_attn.py:117-161) and QuantLlamaMLP.forward (quant/fused_mlp.py:203-218).  The reference
// re-copies the whole KV cache every token (torch.cat, fused_attn.py:142-143) and issues ~15 Python-
// dispatched launches per layer; here the cache is static, RoPE + KV append + attention are one kernel,
// the two RMSNorms and the two residual adds are fused into the matvecs, and nothing touches the host.
#include <cstdlib>

#include "common.cuh"
#include "kernels.h"

namespace gptq {
namespace {

constexpr int kAttnChunk = 256;    // keys per attention CTA
constexpr int kAttnThreads = 128;  // 16 groups of 8 lanes; a group owns one key at a time
constexpr int kHeadDim = 128;

// Every kernel of the chain is launched with programmatic dependent launch (launch_kernel's pdl).

__global__ void embed_kernel(const __half* __restrict__ embed, const int32_t* __restrict__ tokens, __half* __restrict__ x, int hidden, int vocab) {
    const int b = blockIdx.x;
    grid_launch_dependents();
    grid_dependency_wait();
    const uint4* src = reinterpret_cast<const uint4*>(embed + (size_t)min(max(tokens[b], 0), vocab - 1) * hidden);
    uint4* dst = reinterpret_cast<uint4*>(x + (size_t)b * hidden);
    for (int i = threadIdx.x; i < hidden / 8; i += blockDim.x) dst[i] = __ldg(src + i);
}

__global__ void residual_add_kernel(__half* __restrict__ x, const __half* __restrict__ y, int n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    grid_launch_dependents();
    grid_dependency_wait();
    if (i < n) x[i] = __hadd(x[i], y[i]);
}

// dims [16 j, 16 j + 16) of row t of a head's K or V: row pos from this CTA's own copy in shared memory, the others from the cache
__device__ __forceinline__ void load_key_dims(const __half* cache, const __half* fresh, int t, int pos, int j, uint4& a, uint4& b) {
    if (t == pos) {
        a = reinterpret_cast<const uint4*>(fresh)[2 * j];
        b = reinterpret_cast<const uint4*>(fresh)[2 * j + 1];
    } else {
        const uint4* src = reinterpret_cast<const uint4*>(cache + (size_t)t * kHeadDim) + 2 * j;
        a = src[0];
        b = src[1];
    }
}

// RoPE(q, k) + KV append + attention over keys [split*256, min(split*256+256, pos+1)).
//   rotation: rotate_half_kernel (quant/fused_attn.py:23-58): angle_i = rope_inv_freq(i) * pos (common.cuh), fp32, results rounded to fp16
//   scores:   fp16 q.k with fp32 accumulation, * head_dim^-0.5, softmax in fp32, fp32 P.V  (SDPA, fused_attn.py:154-155)
// grid (heads, nsplit, batch).  Partial (m, l, o[128]) per (batch, head, split) goes to `part`.
// Grouped-query attention: qkv rows are [hidden q | n_kv_heads * 128 k | n_kv_heads * 128 v] and query head h reads K/V head h / g
// (g = n_heads / n_kv_heads).  The g CTAs of a group that own the new key all rotate it, and each reads its own copy of the new row from shared
// memory, never from the cache (a sibling's store may not have landed); only the group's first head stores it.
__global__ void __launch_bounds__(kAttnThreads) attn_decode_kernel(const __half* __restrict__ qkv, int hidden, int n_kv_heads, __half* __restrict__ k_cache,
                                                                   __half* __restrict__ v_cache, const int32_t* __restrict__ positions, int n_heads, int max_seq,
                                                                   int batch, const RopeFreqs rope, float scale, float* __restrict__ part, int nsplit) {
    const int head = blockIdx.x, split = blockIdx.y, b = blockIdx.z;
    grid_launch_dependents();
    grid_dependency_wait();
    const int pos = min(max(positions[b], 0), max_seq - 1);  // the host rejects positions outside the cache; never write past it
    const int T = pos + 1;
    const int c0 = split * kAttnChunk;
    if (c0 >= T) return;
    const int c1 = min(c0 + kAttnChunk, T);
    const int tid = threadIdx.x;

    __shared__ float q_s[kHeadDim];
    __shared__ float cs_s[kHeadDim];  // cos[0..63], sin[0..63]
    __shared__ __align__(16) __half knew_s[kHeadDim], vnew_s[kHeadDim];  // row pos of K and V (if this CTA owns it)
    __shared__ float red_m[16], red_l[16];
    __shared__ float red_o[16][kHeadDim + 4];

    const int group = n_heads / n_kv_heads, kv_head = head / group;
    const int Hkv = n_kv_heads * kHeadDim;
    const __half* row = qkv + (size_t)b * (hidden + 2 * Hkv);
    const __half* q = row + head * kHeadDim;
    const __half* k = row + hidden + kv_head * kHeadDim;
    const __half* v = k + Hkv;
    __half* kc = k_cache + ((size_t)(b * n_kv_heads + kv_head) * max_seq) * kHeadDim;
    __half* vc = v_cache + ((size_t)(b * n_kv_heads + kv_head) * max_seq) * kHeadDim;

    if (tid < 64) {
        const float f = rope_inv_freq(tid, rope) * (float)pos;
        cs_s[tid] = cosf(f);
        cs_s[64 + tid] = sinf(f);
    }
    __syncthreads();
    {
        const int i = tid & 63;
        const float c = cs_s[i], s = cs_s[64 + i];
        const bool hi = tid >= 64;  // element i (x part) or i + 64 (y part)
        const float qx = __half2float(q[i]), qy = __half2float(q[i + 64]);
        const float qr = hi ? rope_y(qx, qy, c, s) : rope_x(qx, qy, c, s);
        q_s[tid] = __half2float(__float2half_rn(qr));  // the reference stores the rotated q as fp16
        if (pos >= c0 && pos < c1) {                   // this CTA owns the new key/value: append them
            const float kx = __half2float(k[i]), ky = __half2float(k[i + 64]);
            const float kr = hi ? rope_y(kx, ky, c, s) : rope_x(kx, ky, c, s);
            knew_s[tid] = __float2half_rn(kr);
            vnew_s[tid] = v[tid];
            if (head == kv_head * group) {
                kc[(size_t)pos * kHeadDim + tid] = knew_s[tid];
                vc[(size_t)pos * kHeadDim + tid] = vnew_s[tid];
            }
        }
    }
    __syncthreads();

    const int grp = tid >> 3, j = tid & 7;  // group of 8 lanes; lane j owns dims [16j, 16j+16)
    float qr[16];
#pragma unroll
    for (int d = 0; d < 16; ++d) qr[d] = q_s[16 * j + d];

    constexpr int ITER = kAttnChunk / 16;
    float sc[ITER];
    float mloc = -INFINITY;
#pragma unroll
    for (int it = 0; it < ITER; ++it) {
        const int t = c0 + grp + it * 16;
        float s = 0.f;
        if (t < c1) {
            uint4 a, bq;
            load_key_dims(kc, knew_s, t, pos, j, a, bq);
            const uint32_t w[8] = {a.x, a.y, a.z, a.w, bq.x, bq.y, bq.z, bq.w};
#pragma unroll
            for (int e = 0; e < 8; ++e) {
                const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&w[e]));
                s = fmaf(qr[2 * e], f.x, s);
                s = fmaf(qr[2 * e + 1], f.y, s);
            }
        }
        s += __shfl_xor_sync(0xffffffffu, s, 1);
        s += __shfl_xor_sync(0xffffffffu, s, 2);
        s += __shfl_xor_sync(0xffffffffu, s, 4);
        s = (t < c1) ? s * scale : -INFINITY;
        sc[it] = s;
        mloc = fmaxf(mloc, s);
    }
    float lloc = 0.f;
    float o[16];
#pragma unroll
    for (int d = 0; d < 16; ++d) o[d] = 0.f;
#pragma unroll
    for (int it = 0; it < ITER; ++it) {
        const int t = c0 + grp + it * 16;
        if (t < c1) {
            const float p = expf(sc[it] - mloc);
            lloc += p;
            uint4 a, bq;
            load_key_dims(vc, vnew_s, t, pos, j, a, bq);
            const uint32_t w[8] = {a.x, a.y, a.z, a.w, bq.x, bq.y, bq.z, bq.w};
#pragma unroll
            for (int e = 0; e < 8; ++e) {
                const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&w[e]));
                o[2 * e] = fmaf(p, f.x, o[2 * e]);
                o[2 * e + 1] = fmaf(p, f.y, o[2 * e + 1]);
            }
        }
    }
    if (j == 0) {
        red_m[grp] = mloc;
        red_l[grp] = lloc;
    }
#pragma unroll
    for (int d = 0; d < 16; ++d) red_o[grp][16 * j + d] = o[d];
    __syncthreads();
    // combine the 16 groups; thread tid owns output dim tid
    float M = -INFINITY;
#pragma unroll
    for (int gI = 0; gI < 16; ++gI) M = fmaxf(M, red_m[gI]);
    float L = 0.f, O = 0.f;
#pragma unroll
    for (int gI = 0; gI < 16; ++gI) {
        const float w = (red_m[gI] == -INFINITY) ? 0.f : expf(red_m[gI] - M);
        L = fmaf(red_l[gI], w, L);
        O = fmaf(red_o[gI][tid], w, O);
    }
    float* dst = part + ((size_t)(b * n_heads + head) * nsplit + split) * (kHeadDim + 2);
    dst[2 + tid] = O;
    if (tid == 0) {
        dst[0] = M;
        dst[1] = L;
    }
}

// attn_out[b, head*128 + d] = fp16( sum_s o_s[d] e^{m_s - M} / sum_s l_s e^{m_s - M} ); grid (heads, batch)
__global__ void __launch_bounds__(kHeadDim) attn_combine_kernel(const float* __restrict__ part, const int32_t* __restrict__ positions, __half* __restrict__ out,
                                                                int hidden, int n_heads, int nsplit) {
    const int head = blockIdx.x, b = blockIdx.y, d = threadIdx.x;
    grid_launch_dependents();
    grid_dependency_wait();
    const int nvalid = min(nsplit, max(positions[b], 0) / kAttnChunk + 1);
    const float* src = part + ((size_t)(b * n_heads + head) * nsplit) * (kHeadDim + 2);
    float M = -INFINITY;
    for (int s = 0; s < nvalid; ++s) M = fmaxf(M, src[(size_t)s * (kHeadDim + 2)]);
    float L = 0.f, O = 0.f;
    for (int s = 0; s < nvalid; ++s) {
        const float* ps = src + (size_t)s * (kHeadDim + 2);
        const float w = expf(ps[0] - M);
        L = fmaf(ps[1], w, L);
        O = fmaf(ps[2 + d], w, O);
    }
    out[(size_t)b * hidden + head * kHeadDim + d] = __float2half_rn(O / L);
}

// logits[b, v] = fp16( sum_h rmsnorm(x)[b,h] * W[v,h] ), fp16 W row-major [vocab, hidden] (nn.Linear lm_head);
// the final RMSNorm (quant/triton_norm.py numerics) is recomputed per CTA.  One warp per vocab row.
template <int MAXB>
__global__ void __launch_bounds__(256) lm_head_kernel(const __half* __restrict__ x, const __half* __restrict__ norm_w, float eps, const __half* __restrict__ W,
                                                      __half* __restrict__ logits, int hidden, int vocab, int batch) {
    extern __shared__ __align__(16) uint8_t smem_raw[];
    __half* xs = reinterpret_cast<__half*>(smem_raw);  // [batch][hidden] normalised
    __shared__ float red[8];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    grid_launch_dependents();
    grid_dependency_wait();
    for (int b = 0; b < batch; ++b) {
        const __half2* xr = reinterpret_cast<const __half2*>(x + (size_t)b * hidden);
        float ss = 0.f;
        for (int i = tid; i < hidden / 2; i += 256) {
            const float2 f = __half22float2(xr[i]);
            ss = fmaf(f.x, f.x, ss);
            ss = fmaf(f.y, f.y, ss);
        }
        ss = warp_sum(ss);
        if (lane == 0) red[warp] = ss;
        __syncthreads();
        float tot = 0.f;
#pragma unroll
        for (int w = 0; w < 8; ++w) tot += red[w];
        const float rstd = rms_rstd(tot, hidden, eps);
        for (int i = tid; i < hidden / 2; i += 256) {
            reinterpret_cast<__half2*>(xs + (size_t)b * hidden)[i] =
                rms_apply2(__half22float2(xr[i]), rstd, __half22float2(reinterpret_cast<const __half2*>(norm_w)[i]));
        }
        __syncthreads();
    }
    const int chunks = hidden / 8;
    for (int row = blockIdx.x * 8 + warp; row < vocab; row += gridDim.x * 8) {
        const uint4* wr = reinterpret_cast<const uint4*>(W + (size_t)row * hidden);
        float acc[MAXB];
#pragma unroll
        for (int b = 0; b < MAXB; ++b) acc[b] = 0.f;
        for (int c = lane; c < chunks; c += 32) {
            uint4 wv;
            asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(wv.x), "=r"(wv.y), "=r"(wv.z), "=r"(wv.w) : "l"(wr + c));
            const uint32_t ww[4] = {wv.x, wv.y, wv.z, wv.w};
#pragma unroll
            for (int b = 0; b < MAXB; ++b) {
                if (b < batch) {
                    const uint4 xv = *reinterpret_cast<const uint4*>(xs + (size_t)b * hidden + c * 8);
                    const uint32_t xw[4] = {xv.x, xv.y, xv.z, xv.w};
#pragma unroll
                    for (int e = 0; e < 4; ++e) {
                        const float2 wf = __half22float2(*reinterpret_cast<const __half2*>(&ww[e]));
                        const float2 xf = __half22float2(*reinterpret_cast<const __half2*>(&xw[e]));
                        acc[b] = fmaf(wf.x, xf.x, acc[b]);
                        acc[b] = fmaf(wf.y, xf.y, acc[b]);
                    }
                }
            }
        }
#pragma unroll
        for (int b = 0; b < MAXB; ++b) {
            if (b < batch) {
                const float s = warp_sum(acc[b]);
                if (lane == 0) logits[(size_t)b * vocab + row] = __float2half_rn(s);
            }
        }
    }
}

__global__ void __launch_bounds__(1024) argmax_kernel(const __half* __restrict__ logits, int vocab, int32_t* __restrict__ out) {
    const int b = blockIdx.x;
    grid_launch_dependents();
    grid_dependency_wait();
    const __half* row = logits + (size_t)b * vocab;
    float best = -INFINITY;
    int idx = 0x7fffffff;
    for (int i = threadIdx.x; i < vocab; i += 1024) {
        const float v = __half2float(row[i]);
        if (GPTQ_ARGMAX_BEATS(v, i, best, idx)) {
            best = v;
            idx = i;
        }
    }
    __shared__ float sv[32];
    __shared__ int si[32];
    GPTQ_WARP_ARGMAX(best, idx);
    if ((threadIdx.x & 31) == 0) {
        sv[threadIdx.x >> 5] = best;
        si[threadIdx.x >> 5] = idx;
    }
    __syncthreads();
    if (threadIdx.x < 32) {
        best = sv[threadIdx.x];
        idx = si[threadIdx.x];
        GPTQ_WARP_ARGMAX(best, idx);
        if (threadIdx.x == 0) out[b] = idx;
    }
}

struct ScratchLayout {
    size_t x, qkv, attn, h, xn, tmp, part, ws, mega, total;
    size_t ws_bytes;
    int nsplit;
};

ScratchLayout scratch_layout(const gptq_llama_model& m, int batch, int max_seq) {
    ScratchLayout L{};
    const size_t wide = (size_t)max(m.intermediate, 3 * m.hidden);
    L.nsplit = ceil_div(max_seq, kAttnChunk);
    L.x = carve(L.total, (size_t)batch * m.hidden * 2);
    L.qkv = carve(L.total, (size_t)batch * 3 * m.hidden * 2);
    L.attn = carve(L.total, (size_t)batch * m.hidden * 2);
    L.h = carve(L.total, (size_t)batch * m.intermediate * 2);
    L.xn = carve(L.total, (size_t)batch * wide * 2);
    L.tmp = carve(L.total, (size_t)batch * wide * 2);
    L.part = carve(L.total, (size_t)batch * m.n_heads * L.nsplit * (kHeadDim + 2) * sizeof(float));
    size_t ws = 0;
    ws = max(ws, skinny_workspace_bytes(batch, m.hidden, 3 * m.hidden, false));
    ws = max(ws, skinny_workspace_bytes(batch, m.hidden, m.hidden, false));
    ws = max(ws, skinny_workspace_bytes(batch, m.hidden, m.intermediate, true));
    ws = max(ws, skinny_workspace_bytes(batch, m.intermediate, m.hidden, false));
    L.ws_bytes = ws;
    L.ws = carve(L.total, ws);
    L.mega = carve(L.total, mega_scratch_bytes(m, batch));
    return L;
}

// One quantized linear of the kernel chain with its fused RMSNorm prologue (norm_w) or residual epilogue (residual), and whether the
// tuned int4 matvec serves it whole; otherwise the norm, the generic product and the residual add run as separate kernels.
struct ChainLinear {
    QLinearArgs a;
    bool skinny;
    int launches() const { return skinny ? 1 : 1 + (a.norm_w != nullptr) + (a.residual != nullptr); }
};

// The four quantized linears of layer ly in launch order: qkv (input norm), o_proj (x +=), gate|up (post norm), down_proj (x +=).
void chain_linears(const gptq_llama_model& m, const gptq_llama_layer& ly, const gptq_llama_state& st, const ScratchLayout& L, cudaStream_t stream,
                   ChainLinear (&out)[4]) {
    uint8_t* sc = reinterpret_cast<uint8_t*>(st.scratch);
    uint8_t* x = sc + L.x;
    const int H = m.hidden, I = m.intermediate;
    auto make = [&](const gptq_qweight& w, const gptq_qweight* w2, const void* in, int64_t ldx, const void* norm_w, const void* residual, void* o, int64_t ldo) {
        ChainLinear c{};
        QLinearArgs& a = c.a;
        a.x = in; a.ldx = ldx; a.w = w; a.dual = (w2 != nullptr);
        if (w2) a.w2 = *w2;
        a.norm_w = norm_w; a.eps = norm_w != nullptr ? m.rms_eps : 0.f; a.residual = residual; a.ldr = ldo; a.out = o; a.ldo = ldo; a.M = st.batch;
        a.workspace = sc + L.ws; a.ws_bytes = L.ws_bytes; a.stream = stream;
        c.skinny = skinny_supported(a);
        return c;
    };
    out[0] = make(ly.qkv, nullptr, x, H, ly.input_norm, nullptr, sc + L.qkv, ly.qkv.N);  // q | k | v rows of (n_heads + 2 n_kv_heads) heads
    out[1] = make(ly.o, nullptr, sc + L.attn, H, nullptr, x, x, H);
    out[2] = make(ly.gate, &ly.up, x, H, ly.post_norm, nullptr, sc + L.h, I);
    out[3] = make(ly.down, nullptr, sc + L.h, I, nullptr, x, x, H);
}

cudaError_t engine_linear(const ChainLinear& c, uint8_t* scratch, const ScratchLayout& L) {
    const QLinearArgs& a = c.a;
    if (c.skinny) return launch_qlinear_skinny(a, true);
    QLinearArgs g = a;
    g.norm_w = nullptr;
    g.residual = nullptr;
    if (a.norm_w != nullptr) {
        cudaError_t e = launch_rmsnorm(a.x, a.ldx, a.norm_w, scratch + L.xn, a.w.K, a.M, a.w.K, a.eps, a.stream);
        if (e != cudaSuccess) return e;
        g.x = scratch + L.xn;
        g.ldx = a.w.K;
    }
    if (a.residual != nullptr) {
        g.out = scratch + L.tmp;
        g.ldo = a.w.N;
    }
    cudaError_t e = launch_qlinear_generic(g);
    if (e != cudaSuccess) return e;
    if (a.residual != nullptr) {
        // residual and out are the same buffer in the engine (in-place x += f(x))
        const int n = a.M * a.w.N;
        return launch_kernel(residual_add_kernel, dim3(ceil_div(n, 256)), dim3(256), 0, a.stream, true, reinterpret_cast<__half*>(a.out),
                             reinterpret_cast<const __half*>(scratch + L.tmp), n);
    }
    return cudaSuccess;
}

}  // namespace
}  // namespace gptq

using namespace gptq;

extern "C" size_t gptq_llama_scratch_bytes(const gptq_llama_model* model, int batch, int max_seq) {
    if (model == nullptr || batch < 1 || batch > 8 || max_seq < 1) return 0;
    return scratch_layout(*model, batch, max_seq).total;
}

extern "C" size_t gptq_llama_persistent_scratch_offset(const gptq_llama_model* model, int batch, int max_seq) {
    if (model == nullptr || batch < 1 || batch > 8 || max_seq < 1) return 0;
    return scratch_layout(*model, batch, max_seq).mega;  // (0 for a tensor-parallel state)
}

extern "C" int gptq_llama_decode_launches(const gptq_llama_model* model, const gptq_llama_state* st) {
    if (model == nullptr || st == nullptr || model->layers == nullptr) return GPTQ_ERR_NULL;
    if (mega_supported(*model, *st)) return 1;
    if (has_input_perm(*model)) return GPTQ_ERR_UNSUPPORTED;  // regrouped act-order layers need the persistent kernel's gathers
    const ScratchLayout L = scratch_layout(*model, st->batch, st->max_seq);
    int n = 1 + 1 + (st->next_tokens != nullptr ? 1 : 0);  // embed + lm_head (+ argmax)
    for (int l = 0; l < model->n_layers; ++l) {
        ChainLinear c[4];
        chain_linears(*model, model->layers[l], *st, L, nullptr, c);
        n += 2;  // attention + combine
        for (const ChainLinear& lin : c) n += lin.launches();
    }
    return n;
}

extern "C" int gptq_llama_decode_step(const gptq_llama_model* model, const gptq_llama_state* st, gptq_stream_t stream) {
    return gptq_llama_decode_step_rope(model, st, nullptr, stream);
}

extern "C" int gptq_llama_decode_step_rope(const gptq_llama_model* model, const gptq_llama_state* st, const float* inv_freq, gptq_stream_t stream_) {
    if (model == nullptr || st == nullptr) return GPTQ_ERR_NULL;
    const gptq_llama_model& m = *model;
    if (m.layers == nullptr || m.embed == nullptr || m.final_norm == nullptr || m.lm_head == nullptr) return GPTQ_ERR_NULL;
    if (st->k_cache == nullptr || st->v_cache == nullptr || st->tokens == nullptr || st->positions == nullptr || st->logits == nullptr || st->scratch == nullptr)
        return GPTQ_ERR_NULL;
    if (m.head_dim != kHeadDim) return GPTQ_ERR_UNSUPPORTED;  // LLaMA-7B/13B/33B/65B all use head_dim 128
    if (inv_freq != nullptr && !rope_table_ok(inv_freq, kHeadDim / 2)) return GPTQ_ERR_SHAPE;
    const int Hq = m.n_heads * m.head_dim;  // = hidden, or this rank's share of it under tensor parallelism
    if ((st->tp == nullptr && Hq != m.hidden) || Hq < 1 || Hq > m.hidden || m.hidden % 32 != 0 || m.intermediate % 32 != 0 || m.n_layers < 1 || m.vocab < 1) return GPTQ_ERR_SHAPE;
    if (st->batch < 1 || st->batch > 8 || st->max_seq < 1) return GPTQ_ERR_SHAPE;
    const int n_kv = llama_kv_heads(m);
    if (n_kv < 1) return GPTQ_ERR_SHAPE;
    if (st->tp != nullptr && n_kv != m.n_heads) return GPTQ_ERR_UNSUPPORTED;  // tensor-parallel shards are dealt by whole query heads
    const ScratchLayout L = scratch_layout(m, st->batch, st->max_seq);
    if (st->scratch_bytes < L.total) return GPTQ_ERR_WORKSPACE;
    if (!aligned(st->scratch, 256)) return GPTQ_ERR_ALIGN;
    for (int l = 0; l < m.n_layers; ++l) {
        const gptq_llama_layer& ly = m.layers[l];
        if (ly.qkv.K != m.hidden || ly.qkv.N != Hq + 2 * n_kv * m.head_dim || ly.o.K != Hq || ly.o.N != m.hidden || ly.gate.K != m.hidden ||
            ly.gate.N != m.intermediate || ly.up.K != m.hidden || ly.up.N != m.intermediate || ly.down.K != m.intermediate || ly.down.N != m.hidden)
            return GPTQ_ERR_SHAPE;
        if (ly.input_norm == nullptr || ly.post_norm == nullptr) return GPTQ_ERR_NULL;
    }

    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    uint8_t* sc = reinterpret_cast<uint8_t*>(st->scratch);
    // tensor-parallel ranks keep the persistent kernel's region at the START of the scratch area (peers address it by offset)
    const cudaError_t mega = launch_decode_mega(m, *st, st->tp != nullptr ? sc : sc + L.mega, inv_freq, stream);
    if (mega == cudaSuccess) return GPTQ_OK;
    if (mega != cudaErrorCooperativeLaunchTooLarge && mega != cudaErrorInvalidConfiguration) return GPTQ_ERR_CUDA;
    // the step does not fit the persistent kernel, or the device cannot co-schedule its grid: per-op kernel chain below
    if (has_input_perm(m) || st->tp != nullptr) return GPTQ_ERR_UNSUPPORTED;  // only the persistent kernel implements these
    __half* x = reinterpret_cast<__half*>(sc + L.x);
    __half* qkv = reinterpret_cast<__half*>(sc + L.qkv);
    __half* attn = reinterpret_cast<__half*>(sc + L.attn);
    float* part = reinterpret_cast<float*>(sc + L.part);
    const int B = st->batch, H = m.hidden;
    const RopeFreqs rope = rope_freqs(m.rope_base, m.head_dim, inv_freq);
    const float scale = attn_scale(m.head_dim);
    const size_t layer_stride = (size_t)B * n_kv * st->max_seq * m.head_dim;

#define GPTQ_TRY(expr)                                   \
    do {                                                 \
        if ((expr) != cudaSuccess) return GPTQ_ERR_CUDA; \
    } while (0)

    GPTQ_TRY(launch_kernel(embed_kernel, dim3(B), dim3(256), 0, stream, true, reinterpret_cast<const __half*>(m.embed), st->tokens, x, H, m.vocab));
    for (int l = 0; l < m.n_layers; ++l) {
        ChainLinear c[4];
        chain_linears(m, m.layers[l], *st, L, stream, c);
        GPTQ_TRY(engine_linear(c[0], sc, L));
        GPTQ_TRY(launch_kernel(attn_decode_kernel, dim3(m.n_heads, L.nsplit, B), dim3(kAttnThreads), 0, stream, true, qkv, H, n_kv,
                               reinterpret_cast<__half*>(st->k_cache) + l * layer_stride, reinterpret_cast<__half*>(st->v_cache) + l * layer_stride,
                               st->positions, m.n_heads, st->max_seq, B, rope, scale, part, L.nsplit));
        GPTQ_TRY(launch_kernel(attn_combine_kernel, dim3(m.n_heads, B), dim3(kHeadDim), 0, stream, true, part, st->positions, attn, H, m.n_heads, L.nsplit));
        for (int i = 1; i < 4; ++i) GPTQ_TRY(engine_linear(c[i], sc, L));
    }
    GPTQ_TRY(launch_kernel(B == 1 ? lm_head_kernel<1> : lm_head_kernel<8>, dim3(min(ceil_div(m.vocab, 8), kNumSMs * 8)), dim3(256),
                           (size_t)B * H * sizeof(__half), stream, true, (const __half*)x, reinterpret_cast<const __half*>(m.final_norm), m.rms_eps,
                           reinterpret_cast<const __half*>(m.lm_head), reinterpret_cast<__half*>(st->logits), H, m.vocab, B));
    if (st->next_tokens != nullptr) {
        GPTQ_TRY(launch_kernel(argmax_kernel, dim3(B), dim3(1024), 0, stream, true, reinterpret_cast<const __half*>(st->logits), m.vocab, st->next_tokens));
    }
#undef GPTQ_TRY
    return GPTQ_OK;
}
