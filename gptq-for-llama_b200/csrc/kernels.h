// Internal launch interface between capi.cu (validation + dispatch) and the kernel files.
#pragma once
#include <cuda_runtime.h>

#include "gptq_b200.h"

namespace gptq {

// Does any layer carry an act-order input gather (gptq_llama_layer)?  Only the persistent kernel implements them.
inline bool has_input_perm(const gptq_llama_model& m) {
    for (int l = 0; l < m.n_layers; ++l)
        if (m.layers[l].qkv_perm != nullptr || m.layers[l].o_perm != nullptr || m.layers[l].mlp_perm != nullptr) return true;
    return false;
}

// K/V heads of a decode model, carried by the width of its fused q|k|v weight (gptq_llama_layer.qkv):
// n_kv_heads = (qkv.N / head_dim - n_heads) / 2.  -1 unless it is a positive divisor of n_heads and every layer has the same width.
inline int llama_kv_heads(const gptq_llama_model& m) {
    if (m.layers == nullptr || m.n_layers < 1 || m.n_heads < 1 || m.head_dim < 1) return -1;
    const int N = m.layers[0].qkv.N;
    for (int l = 1; l < m.n_layers; ++l)
        if (m.layers[l].qkv.N != N) return -1;
    if (N % m.head_dim != 0) return -1;
    const int rest = N / m.head_dim - m.n_heads;  // 2 * n_kv_heads
    if (rest <= 0 || rest % 2 != 0 || m.n_heads % (rest / 2) != 0) return -1;
    return rest / 2;
}

struct QLinearArgs {
    const void* x;
    int64_t ldx;
    gptq_qweight w;   // gate for the fused MLP
    gptq_qweight w2;  // up for the fused MLP (unused otherwise)
    bool dual;        // fused SwiGLU MLP
    const void* bias;      // fp16 [N] or null
    const void* residual;  // fp16 [M, ldr] or null: out = residual + fp16(acc)   (decode engine)
    int64_t ldr;
    const void* norm_w;    // fp16 [K] or null: RMSNorm(x; norm_w, eps) fused in front of the product
    float eps;
    void* out;
    int64_t ldo;
    int M;
    void* workspace;
    size_t ws_bytes;
    cudaStream_t stream;
};

// generic.cu -- CUDA-core kernels, any bits in {2,3,4,8}, any g_idx, any M.
cudaError_t launch_qlinear_generic(const QLinearArgs& a);
cudaError_t launch_qlinear_transpose_generic(const void* g, int64_t ldg, const gptq_qweight& w, void* out, int64_t ldo, int M, cudaStream_t stream);
cudaError_t launch_dequant(const gptq_qweight& w, void* out, int64_t ldo, cudaStream_t stream);

// qmatvec.cu -- tuned int4 decode kernel (M <= 8, no act-order): stream-K over 2 CTAs/SM.
struct SkinnyPlan {
    int nslabs, nk, grid, max_contrib, seg_steps;
    long long total_units;
};
SkinnyPlan plan_skinny(int M, int K, int N);
size_t skinny_workspace_bytes(int M, int K, int N, bool dual);
bool skinny_supported(const QLinearArgs& a);
cudaError_t launch_qlinear_skinny(const QLinearArgs& a, bool pdl);

// qgemm_wgmma.cu -- batched (prefill) int4 GEMM on wgmma tensor cores, M > 8
bool gemm_tc_supported(const QLinearArgs& a);
cudaError_t launch_qlinear_gemm_tc(const QLinearArgs& a);

// qgemm_wgmma_t.cu -- transposed int4 GEMM on wgmma (the gradient w.r.t. a quantized linear's input), M > 8
bool gemm_t_tc_supported(const void* g, int64_t ldg, const gptq_qweight& w, const void* out, int64_t ldo, int M);
cudaError_t launch_qlinear_transpose_tc(const void* g, int64_t ldg, const gptq_qweight& w, void* out, int64_t ldo, int M, cudaStream_t stream);

// lm_head_logprob.cu -- per-row log-probability of a target through the fp16 lm_head (wgmma + fused log-softmax), and its combine pass
size_t lm_head_logprob_workspace_bytes(int M, int V);
cudaError_t launch_lm_head_logprob(const void* x, int64_t ldx, const void* w, int64_t ldw, int M, int K, int V, const int32_t* targets, float* logprob,
                                   void* workspace, cudaStream_t stream);

// cached_attention.cu -- causal attention of new rows over a sequence's cached prefix (wgmma, read in place from the KV cache), head_dim 128
constexpr int kCachedAttnMaxSpans = 64;
cudaError_t launch_cached_attention(const void* q, int64_t ldq, const void* k_cache, const void* v_cache, int batch, int n_heads, int n_kv_heads, int max_seq,
                                    int n_spans, const int32_t* span_seq, const int32_t* span_start, const int32_t* span_rows, void* out, int64_t ldo,
                                    cudaStream_t stream);

// sample.cu -- one token per row of decode-step logits: temperature / top-k / top-p / Philox draw, or the argmax (gptq_sample_tokens)
constexpr int kSampleMaxBatch = 8, kSampleMaxVocab = 131072;
cudaError_t launch_sample_tokens(const void* logits, int64_t ld, int batch, int vocab, const int32_t* positions, const gptq_sampling& params,
                                 int32_t* next_tokens, cudaStream_t stream);

// decode_mega.cu -- persistent single-kernel decode step (batch 1 to 8, int4 kernel-form layers); inv_freq as for launch_rope
bool mega_supported(const gptq_llama_model& m, const gptq_llama_state& st);
size_t mega_scratch_bytes(const gptq_llama_model& m, int batch);
cudaError_t launch_decode_mega(const gptq_llama_model& m, const gptq_llama_state& st, uint8_t* scratch, const float* inv_freq, cudaStream_t stream);

// elementwise.cu -- inv_freq: a HOST table of head_dim / 2 frequencies (head_dim <= 128), or nullptr for the unscaled rule at `base` (common.cuh)
cudaError_t launch_rope(void* qk, int64_t token_stride, const int64_t* position_ids, int64_t pos_batch_stride, int bsz, int seq, int rows, int head_dim,
                        float base, const float* inv_freq, cudaStream_t stream);
cudaError_t launch_rmsnorm(const void* x, int64_t ldx, const void* weight, void* y, int64_t ldy, int M, int N, float eps, cudaStream_t stream);

// pack.cu
cudaError_t launch_pack_rows(const int32_t* vals, int32_t* packed, int R, int C, int bits, bool along_cols, cudaStream_t stream);
cudaError_t launch_unpack_rows(const int32_t* packed, int32_t* vals, int R, int C, int bits, bool along_cols, cudaStream_t stream);

}  // namespace gptq
