// extern "C" surface of libgptq_b200.so: argument validation, error codes, kernel dispatch.
// No torch types, no allocation, no synchronisation, no global mutable state.
#include <cstring>

#include "common.cuh"
#include "kernels.h"

using namespace gptq;

namespace {

inline bool bits_ok(int bits) { return bits == 2 || bits == 3 || bits == 4 || bits == 8; }

int check_weight(const gptq_qweight* w) {
    if (w == nullptr) return GPTQ_ERR_NULL;
    if (!bits_ok(w->bits)) return GPTQ_ERR_BITS;
    if (w->qweight == nullptr || w->scales == nullptr || w->qzeros == nullptr) return GPTQ_ERR_NULL;
    if (w->K <= 0 || w->N <= 0 || w->G <= 0) return GPTQ_ERR_SHAPE;
    if (w->K % 32 != 0 || w->N % 32 != 0) return GPTQ_ERR_SHAPE;  // whole runs only (quant_linear.py:316-317)
    if (w->groupsize > 0) {
        if ((w->K + w->groupsize - 1) / w->groupsize != w->G) return GPTQ_ERR_SHAPE;
    } else if (w->g_idx == nullptr) {
        return GPTQ_ERR_NULL;
    }
    if (!aligned(w->qweight, 4) || !aligned(w->qzeros, 4) || !aligned(w->scales, 2)) return GPTQ_ERR_ALIGN;
    return GPTQ_OK;
}

inline int cuda_status(cudaError_t e) { return e == cudaSuccess ? GPTQ_OK : GPTQ_ERR_CUDA; }

}  // namespace

extern "C" {

int gptq_abi_version(void) { return GPTQ_B200_ABI_VERSION; }

const char* gptq_strerror(int status) {
    switch (status) {
        case GPTQ_OK: return "ok";
        case GPTQ_ERR_BITS: return "Only 2,3,4,8 bits are supported.";
        case GPTQ_ERR_SHAPE: return "invalid shape: infeatures/outfeatures must be positive multiples of 32 and G must match groupsize";
        case GPTQ_ERR_NULL: return "required pointer is NULL";
        case GPTQ_ERR_ALIGN: return "pointer or leading dimension is misaligned";
        case GPTQ_ERR_WORKSPACE: return "workspace too small (see gptq_qlinear_workspace_bytes)";
        case GPTQ_ERR_CUDA: return "CUDA runtime error (launch failed; is this an sm_90a device?)";
        case GPTQ_ERR_UNSUPPORTED: return "request not supported by this build";
    }
    return "unknown gptq status";
}

size_t gptq_qlinear_workspace_bytes(int M, int K, int N, int bits) {
    if (bits != 4 || M <= 0 || K <= 0 || N <= 0) return 0;
    return skinny_workspace_bytes(M, K, N, false);
}

size_t gptq_fused_mlp_workspace_bytes(int M, int K, int N, int bits) {
    if (bits != 4 || M <= 0 || K <= 0 || N <= 0) return 0;
    return skinny_workspace_bytes(M, K, N, true);
}

static int run_qlinear(const QLinearArgs& a) {
    if (skinny_supported(a)) {
        const size_t need = skinny_workspace_bytes(a.M, a.w.K, a.w.N, a.dual);
        if (a.workspace == nullptr || a.ws_bytes < need) return GPTQ_ERR_WORKSPACE;
        if (!aligned(a.workspace, 256)) return GPTQ_ERR_ALIGN;
        return cuda_status(launch_qlinear_skinny(a, false));
    }
    if (gemm_tc_supported(a)) return cuda_status(launch_qlinear_gemm_tc(a));
    return cuda_status(launch_qlinear_generic(a));
}

int gptq_qlinear_fwd(const void* x, int64_t ldx, const gptq_qweight* w, const void* bias, void* out, int64_t ldo, int M, void* workspace, size_t ws_bytes,
                     gptq_stream_t stream) {
    if (int st = check_weight(w)) return st;
    if (x == nullptr || out == nullptr) return GPTQ_ERR_NULL;
    if (M < 0 || ldx < w->K || ldo < w->N) return GPTQ_ERR_SHAPE;
    if (!aligned(x, 2) || !aligned(out, 2) || (bias && !aligned(bias, 2))) return GPTQ_ERR_ALIGN;
    if (M == 0) return GPTQ_OK;
    QLinearArgs a{};
    a.x = x; a.ldx = ldx; a.w = *w; a.dual = false; a.bias = bias; a.out = out; a.ldo = ldo; a.M = M;
    a.workspace = workspace; a.ws_bytes = ws_bytes; a.stream = static_cast<cudaStream_t>(stream);
    return run_qlinear(a);
}

int gptq_fused_mlp_fwd(const void* x, int64_t ldx, const gptq_qweight* gate, const gptq_qweight* up, void* out, int64_t ldo, int M, void* workspace,
                       size_t ws_bytes, gptq_stream_t stream) {
    if (int st = check_weight(gate)) return st;
    if (int st = check_weight(up)) return st;
    if (gate->K != up->K || gate->N != up->N || gate->G != up->G || gate->bits != up->bits || (gate->groupsize > 0) != (up->groupsize > 0) ||
        (gate->groupsize > 0 && gate->groupsize != up->groupsize))
        return GPTQ_ERR_SHAPE;
    if (x == nullptr || out == nullptr) return GPTQ_ERR_NULL;
    if (M < 0 || ldx < gate->K || ldo < gate->N) return GPTQ_ERR_SHAPE;
    if (!aligned(x, 2) || !aligned(out, 2)) return GPTQ_ERR_ALIGN;
    if (M == 0) return GPTQ_OK;
    QLinearArgs a{};
    a.x = x; a.ldx = ldx; a.w = *gate; a.w2 = *up; a.dual = true; a.bias = nullptr; a.out = out; a.ldo = ldo; a.M = M;
    a.workspace = workspace; a.ws_bytes = ws_bytes; a.stream = static_cast<cudaStream_t>(stream);
    return run_qlinear(a);
}

int gptq_qlinear_transpose_fwd(const void* g, int64_t ldg, const gptq_qweight* w, void* out, int64_t ldo, int M, gptq_stream_t stream) {
    if (int st = check_weight(w)) return st;
    if (g == nullptr || out == nullptr) return GPTQ_ERR_NULL;
    if (M < 0 || ldg < w->N || ldo < w->K) return GPTQ_ERR_SHAPE;
    if (M == 0) return GPTQ_OK;
    if (gemm_t_tc_supported(g, ldg, *w, out, ldo, M))
        return cuda_status(launch_qlinear_transpose_tc(g, ldg, *w, out, ldo, M, static_cast<cudaStream_t>(stream)));
    return cuda_status(launch_qlinear_transpose_generic(g, ldg, *w, out, ldo, M, static_cast<cudaStream_t>(stream)));
}

int gptq_rope_inplace(void* qk, int64_t token_stride, const int64_t* position_ids, int64_t pos_batch_stride, int bsz, int seq, int rows, int head_dim,
                      float base, gptq_stream_t stream) {
    if (qk == nullptr || position_ids == nullptr) return GPTQ_ERR_NULL;
    if (bsz < 0 || seq < 0 || rows <= 0 || head_dim <= 0 || head_dim % 4 != 0 || !(base > 0.f)) return GPTQ_ERR_SHAPE;
    if (token_stride < (int64_t)rows * head_dim || pos_batch_stride < seq) return GPTQ_ERR_SHAPE;
    if (!aligned(qk, 4) || token_stride % 2 != 0 || !aligned(position_ids, 8)) return GPTQ_ERR_ALIGN;
    if ((int64_t)bsz * seq == 0) return GPTQ_OK;
    if ((int64_t)bsz * seq > 0x7fffffffLL) return GPTQ_ERR_SHAPE;
    return cuda_status(launch_rope(qk, token_stride, position_ids, pos_batch_stride, bsz, seq, rows, head_dim, base, nullptr, static_cast<cudaStream_t>(stream)));
}

int gptq_rope_inplace_freq(void* qk, int64_t token_stride, const int64_t* position_ids, int64_t pos_batch_stride, int bsz, int seq, int rows, int head_dim,
                           const float* inv_freq, gptq_stream_t stream) {
    if (qk == nullptr || position_ids == nullptr || inv_freq == nullptr) return GPTQ_ERR_NULL;
    if (bsz < 0 || seq < 0 || rows <= 0 || head_dim <= 0 || head_dim % 4 != 0) return GPTQ_ERR_SHAPE;
    if (head_dim > 2 * kRopeMaxPairs) return GPTQ_ERR_UNSUPPORTED;  // the table travels in the launch parameters
    if (!rope_table_ok(inv_freq, head_dim / 2)) return GPTQ_ERR_SHAPE;
    if (token_stride < (int64_t)rows * head_dim || pos_batch_stride < seq) return GPTQ_ERR_SHAPE;
    if (!aligned(qk, 4) || token_stride % 2 != 0 || !aligned(position_ids, 8)) return GPTQ_ERR_ALIGN;
    if ((int64_t)bsz * seq == 0) return GPTQ_OK;
    if ((int64_t)bsz * seq > 0x7fffffffLL) return GPTQ_ERR_SHAPE;
    return cuda_status(launch_rope(qk, token_stride, position_ids, pos_batch_stride, bsz, seq, rows, head_dim, 1.f, inv_freq, static_cast<cudaStream_t>(stream)));
}

int gptq_rmsnorm_fwd(const void* x, int64_t ldx, const void* weight, void* y, int64_t ldy, int M, int N, float eps, gptq_stream_t stream) {
    if (x == nullptr || weight == nullptr || y == nullptr) return GPTQ_ERR_NULL;
    if (M < 0 || N <= 0 || N % 2 != 0 || ldx < N || ldy < N) return GPTQ_ERR_SHAPE;
    if (N > 65536 / 2) return GPTQ_ERR_UNSUPPORTED;  // "This layer norm doesn't support feature dim >= 64KB." (triton_norm.py:56-60)
    if (!aligned(x, 4) || !aligned(y, 4) || !aligned(weight, 4) || ldx % 2 != 0 || ldy % 2 != 0) return GPTQ_ERR_ALIGN;
    if (M == 0) return GPTQ_OK;
    return cuda_status(launch_rmsnorm(x, ldx, weight, y, ldy, M, N, eps, static_cast<cudaStream_t>(stream)));
}

static int pack_common(const int32_t* src, int32_t* dst, int R, int C, int bits, bool along_cols, bool pack, gptq_stream_t stream) {
    if (!bits_ok(bits)) return GPTQ_ERR_BITS;
    if (src == nullptr || dst == nullptr) return GPTQ_ERR_NULL;
    if (R <= 0 || C <= 0 || R % 32 != 0) return GPTQ_ERR_SHAPE;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    return cuda_status(pack ? launch_pack_rows(src, dst, R, C, bits, along_cols, s) : launch_unpack_rows(src, dst, R, C, bits, along_cols, s));
}

int gptq_pack_qweight(const int32_t* intweight, int32_t* qweight, int K, int N, int bits, gptq_stream_t stream) {
    return pack_common(intweight, qweight, K, N, bits, false, true, stream);
}
int gptq_pack_qzeros(const int32_t* zeros_m1, int32_t* qzeros, int G, int N, int bits, gptq_stream_t stream) {
    return pack_common(zeros_m1, qzeros, N, G, bits, true, true, stream);
}
int gptq_unpack_qweight(const int32_t* qweight, int32_t* intweight, int K, int N, int bits, gptq_stream_t stream) {
    return pack_common(qweight, intweight, K, N, bits, false, false, stream);
}
int gptq_unpack_qzeros(const int32_t* qzeros, int32_t* zeros_m1, int G, int N, int bits, gptq_stream_t stream) {
    return pack_common(qzeros, zeros_m1, N, G, bits, true, false, stream);
}

size_t gptq_lm_head_logprob_workspace_bytes(int M, int V) { return lm_head_logprob_workspace_bytes(M, V); }

int gptq_lm_head_logprob(const void* x, int64_t ldx, const void* w, int64_t ldw, int M, int K, int V, const int32_t* targets, float* logprob,
                         void* workspace, size_t ws_bytes, gptq_stream_t stream) {
    if (x == nullptr || w == nullptr || targets == nullptr || logprob == nullptr) return GPTQ_ERR_NULL;
    if (K <= 0 || K % 64 != 0 || V <= 0 || M < 0 || ldx < K || ldw < K) return GPTQ_ERR_SHAPE;
    if ((int64_t)ceil_div(M, 256) * ceil_div(V, 128) > 0x7fffffffLL) return GPTQ_ERR_SHAPE;  // one CTA per 256 x 128 tile, 1-D grid
    if (!aligned(x, 16) || !aligned(w, 16) || ldx % 8 != 0 || ldw % 8 != 0) return GPTQ_ERR_ALIGN;  // TMA: 16-byte base and row pitch
    if (M == 0) return GPTQ_OK;
    if (workspace == nullptr || !aligned(workspace, 256) || ws_bytes < lm_head_logprob_workspace_bytes(M, V)) return GPTQ_ERR_WORKSPACE;
    return cuda_status(launch_lm_head_logprob(x, ldx, w, ldw, M, K, V, targets, logprob, workspace, static_cast<cudaStream_t>(stream)));
}

int gptq_cached_attention(const void* q, int64_t ldq, const void* k_cache, const void* v_cache, int batch, int n_heads, int head_dim, int max_seq,
                          int n_spans, const int32_t* span_seq, const int32_t* span_start, const int32_t* span_rows, void* out, int64_t ldo,
                          gptq_stream_t stream) {
    return gptq_cached_attention_gqa(q, ldq, k_cache, v_cache, batch, n_heads, n_heads, head_dim, max_seq, n_spans, span_seq, span_start, span_rows, out,
                                     ldo, stream);
}

int gptq_cached_attention_gqa(const void* q, int64_t ldq, const void* k_cache, const void* v_cache, int batch, int n_heads, int n_kv_heads, int head_dim,
                              int max_seq, int n_spans, const int32_t* span_seq, const int32_t* span_start, const int32_t* span_rows, void* out, int64_t ldo,
                              gptq_stream_t stream) {
    if (q == nullptr || k_cache == nullptr || v_cache == nullptr || out == nullptr) return GPTQ_ERR_NULL;
    if (n_spans > 0 && (span_seq == nullptr || span_start == nullptr || span_rows == nullptr)) return GPTQ_ERR_NULL;
    if (batch <= 0 || n_heads <= 0 || n_kv_heads <= 0 || head_dim <= 0 || max_seq <= 0) return GPTQ_ERR_SHAPE;
    if (n_heads % n_kv_heads != 0) return GPTQ_ERR_SHAPE;  // query head h reads K/V head h / (n_heads / n_kv_heads)
    if (head_dim != 128) return GPTQ_ERR_UNSUPPORTED;  // the head size of both decode engines
    if (n_spans < 0 || n_spans > kCachedAttnMaxSpans) return GPTQ_ERR_SHAPE;
    if ((int64_t)batch * n_kv_heads * max_seq > 0x7fffffffLL) return GPTQ_ERR_SHAPE;  // TMA row coordinates are 32-bit
    const int64_t width = (int64_t)n_heads * head_dim;
    if (ldq < width || ldo < width || ldq % 8 != 0 || ldo % 8 != 0) return GPTQ_ERR_SHAPE;  // TMA: 16-byte row pitch
    for (int i = 0; i < n_spans; ++i) {
        if (span_seq[i] < 0 || span_seq[i] >= batch || span_start[i] < 0 || span_rows[i] < 0) return GPTQ_ERR_SHAPE;
        if ((int64_t)span_start[i] + span_rows[i] > max_seq) return GPTQ_ERR_SHAPE;
        for (int j = 0; j < i; ++j)
            if (span_seq[j] == span_seq[i]) return GPTQ_ERR_SHAPE;
    }
    if (!aligned(q, 16) || !aligned(k_cache, 16) || !aligned(v_cache, 16) || !aligned(out, 16)) return GPTQ_ERR_ALIGN;
    return cuda_status(launch_cached_attention(q, ldq, k_cache, v_cache, batch, n_heads, n_kv_heads, max_seq, n_spans, span_seq, span_start, span_rows, out,
                                               ldo, static_cast<cudaStream_t>(stream)));
}

int gptq_sample_tokens(const void* logits, int64_t ld, int batch, int vocab, const int32_t* positions, const gptq_sampling* params,
                       int32_t* next_tokens, gptq_stream_t stream) {
    if (logits == nullptr || positions == nullptr || params == nullptr || next_tokens == nullptr) return GPTQ_ERR_NULL;
    if (params->temperature == nullptr || params->top_k == nullptr || params->top_p == nullptr || params->seed == nullptr ||
        params->eos_token == nullptr || params->min_length == nullptr)
        return GPTQ_ERR_NULL;
    if (batch < 1 || batch > kSampleMaxBatch || vocab < 1 || ld < vocab) return GPTQ_ERR_SHAPE;
    if (vocab > kSampleMaxVocab) return GPTQ_ERR_UNSUPPORTED;
    if (!aligned(logits, 2) || !aligned(positions, 4) || !aligned(next_tokens, 4) || !aligned(params->temperature, 4) || !aligned(params->top_k, 4) ||
        !aligned(params->top_p, 4) || !aligned(params->seed, 8) || !aligned(params->eos_token, 4) || !aligned(params->min_length, 4))
        return GPTQ_ERR_ALIGN;
    return cuda_status(launch_sample_tokens(logits, ld, batch, vocab, positions, *params, next_tokens, static_cast<cudaStream_t>(stream)));
}

int gptq_ipc_alloc(size_t bytes, void** ptr, unsigned char handle[64]) {
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "handle size");
    if (ptr == nullptr || handle == nullptr || bytes == 0) return GPTQ_ERR_NULL;
    void* d = nullptr;
    if (cudaMalloc(&d, bytes) != cudaSuccess) return GPTQ_ERR_CUDA;
    cudaIpcMemHandle_t h;
    if (cudaMemset(d, 0, bytes) != cudaSuccess || cudaDeviceSynchronize() != cudaSuccess || cudaIpcGetMemHandle(&h, d) != cudaSuccess) {
        cudaFree(d);
        return GPTQ_ERR_CUDA;
    }
    memcpy(handle, &h, 64);
    *ptr = d;
    return GPTQ_OK;
}
int gptq_ipc_open(const unsigned char handle[64], void** ptr) {
    if (ptr == nullptr || handle == nullptr) return GPTQ_ERR_NULL;
    cudaIpcMemHandle_t h;
    memcpy(&h, handle, 64);
    return cuda_status(cudaIpcOpenMemHandle(ptr, h, cudaIpcMemLazyEnablePeerAccess));
}
int gptq_ipc_close(void* ptr) { return ptr == nullptr ? GPTQ_ERR_NULL : cuda_status(cudaIpcCloseMemHandle(ptr)); }
int gptq_ipc_free(void* ptr) { return ptr == nullptr ? GPTQ_ERR_NULL : cuda_status(cudaFree(ptr)); }

int gptq_dequant(const gptq_qweight* w, void* out, int64_t ldo, gptq_stream_t stream) {
    if (int st = check_weight(w)) return st;
    if (out == nullptr) return GPTQ_ERR_NULL;
    if (ldo < w->N) return GPTQ_ERR_SHAPE;
    return cuda_status(launch_dequant(*w, out, ldo, static_cast<cudaStream_t>(stream)));
}

}  // extern "C"
