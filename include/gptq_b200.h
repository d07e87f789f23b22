/*
 * gptq_b200.h -- C ABI of libgptq_b200.so: the H100 (sm_90a) implementation of the
 * GPTQ-for-LLaMa quantized-linear inference hot path.
 *
 * The reference (qwopqwop200/GPTQ-for-LLaMa, triton branch) has no FFI layer: its boundary is
 * the Python module surface of quant/ plus the packed tensor layouts.  Each entry point below
 * replaces one Triton launch site of the reference; the citation names it (paths relative to
 * the reference root).  The host mirror (gptq-for-llama_b200/quant, a drop-in for the
 * reference's quant package) binds these symbols with ctypes; INTEGRATION.md shows the stub a
 * reference maintainer would add.
 *
 * Conventions
 *  - plain pointers and sizes only; all pointers are DEVICE pointers unless stated otherwise;
 *    "half" buffers are IEEE fp16 (passed as void*).
 *  - the caller owns every buffer; nothing is allocated, nothing is synchronised, no global
 *    mutable state: every call is asynchronous on `stream` (a cudaStream_t) and is CUDA-graph
 *    capturable.  Workspaces must be zero-filled once by the caller before first use; every
 *    call leaves them zeroed again, so they are reusable by stream-ordered calls.
 *  - return value: 0 on success, a negative gptq_status otherwise; never throws.
 *
 * Packed layout (quant/quant_linear.py:316-319), K = infeatures, N = outfeatures,
 * G = ceil(K / groupsize):
 *    qweight int32 [K/32*bits, N]   k packed along rows, value j of a run at bit bits*j (LSB first);
 *                                   3-bit: 32 values = one 96-bit little-endian stream over 3 rows
 *    qzeros  int32 [G, N/32*bits]   n packed along columns, stored MINUS ONE (:356)
 *    scales  fp16  [G, N]
 *    g_idx   int32 [K]              k -> group (act-order: arbitrary map, gptq.py:210-216)
 *    bias    fp16  [N] or NULL
 */
#ifndef GPTQ_B200_H
#define GPTQ_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GPTQ_B200_ABI_VERSION 6 /* 2: act-order input gathers; 3: gptq_llama_persistent_scratch_offset; 4: tensor parallelism (gptq_llama_tp, gptq_ipc_*);
                                   5: persistent path at batch 2..8 ([batch][hidden] residual rows in the persistent region);
                                   6: gptq_lm_head_logprob (scoring); gptq_cached_attention, gptq_sample_tokens, gptq_cached_attention_gqa,
                                   gptq_rope_inplace_freq and gptq_llama_decode_step_rope added later without a change to any existing struct
                                   or signature */

typedef void* gptq_stream_t; /* cudaStream_t */

typedef enum gptq_status {
    GPTQ_OK = 0,
    GPTQ_ERR_BITS = -1,        /* bits not in {2,3,4,8}  (reference: NotImplementedError, quant_linear.py:308-309) */
    GPTQ_ERR_SHAPE = -2,       /* K or N not a multiple of 32, non-positive sizes, bad strides */
    GPTQ_ERR_NULL = -3,        /* required pointer is NULL */
    GPTQ_ERR_ALIGN = -4,       /* pointer / leading dimension not aligned as required */
    GPTQ_ERR_WORKSPACE = -5,   /* workspace too small: see gptq_*_workspace_bytes */
    GPTQ_ERR_CUDA = -6,        /* a CUDA runtime call failed (launch error, wrong device arch) */
    GPTQ_ERR_UNSUPPORTED = -7, /* valid request this build cannot serve (e.g. norm width > 64 KB, triton_norm.py:59-60) */
} gptq_status;

/* One packed weight matrix, as stored in a GPTQ checkpoint. */
typedef struct gptq_qweight {
    const int32_t* qweight; /* [K/32*bits, N] */
    const void* scales;     /* fp16 [G, N] */
    const int32_t* qzeros;  /* [G, N/32*bits] */
    const int32_t* g_idx;   /* [K]; may be NULL iff groupsize > 0 */
    int K, N, G, bits;
    int groupsize;          /* > 0: caller guarantees g_idx[k] == k / groupsize (no act-order);
                               <= 0: general k -> group map, g_idx is gathered per row */
} gptq_qweight;

int gptq_abi_version(void);
const char* gptq_strerror(int status);

/* Bytes of zero-initialised device workspace the M-row forward of a [K,N] layer may need
 * (split-K partials + arrival counters).  0 means no workspace is needed.  The workspace must be
 * 256-byte aligned. */
size_t gptq_qlinear_workspace_bytes(int M, int K, int N, int bits);
size_t gptq_fused_mlp_workspace_bytes(int M, int K, int N, int bits);

/* out[M,N] = x[M,K] . deq(W) (+ bias), fp16 in / fp32 accumulate / fp16 out.
 * Replaces matmul248 + matmul_248_kernel (quant/quant_linear.py:263-269, :72-137) and the
 * bias add of QuantLinear.forward (:376).  ldx / ldo: row strides of x / out in elements. */
int gptq_qlinear_fwd(const void* x, int64_t ldx, const gptq_qweight* w, const void* bias, void* out, int64_t ldo, int M, void* workspace, size_t ws_bytes,
                     gptq_stream_t stream);

/* out[M,N] = silu(x . deq(Wgate)) * (x . deq(Wup)); SwiGLU on the fp32 accumulators.
 * Replaces QuantLlamaMLP.triton_llama_mlp + fusedmatmul_248_kernel (quant/fused_mlp.py:206-218, :84-168).
 * gate and up must have identical K, N, G, bits. */
int gptq_fused_mlp_fwd(const void* x, int64_t ldx, const gptq_qweight* gate, const gptq_qweight* up, void* out, int64_t ldo, int M, void* workspace,
                       size_t ws_bytes, gptq_stream_t stream);

/* grad_in[M,K] = g[M,N] . deq(W)^T.  Replaces transpose_matmul248 (quant/quant_linear.py:272-279, :191-258).
 * Arithmetic on every route: each weight is dequantised as in the forward, fp16((q - z) * s); products accumulate in fp32; one fp16
 * rounding at the store.  No atomics and no workspace: a row of the result depends on its own row of g only and repeats bit for bit.
 * Routing: the wgmma kernel (tensor cores) serves bits == 4 with groupsize > 0 and a multiple of 32, M > 8, K % 128 == 0, N % 64 == 0,
 * g and out 16-byte aligned with ldg % 8 == 0 and ldo % 8 == 0; every other request goes to the generic CUDA-core kernel (any bits,
 * any g_idx, any M).  Act-order and 2/3-bit layers reach the wgmma kernel through their kernel form (regrouped rows, widened fields). */
int gptq_qlinear_transpose_fwd(const void* g, int64_t ldg, const gptq_qweight* w, void* out, int64_t ldo, int M, gptq_stream_t stream);

/* In-place rotary embedding on q and k.  Replaces triton_rotate_half_ / rotate_half_kernel
 * (quant/fused_attn.py:61-93, :8-58).  qk is viewed as [tokens, rows, head_dim] fp16 with
 * `token_stride` elements between tokens (3*hidden for the fused qkv output) and rows = 2*heads
 * contiguous rows of head_dim; position_ids int64 [bsz, seq] with `pos_batch_stride` elements
 * between batches; tokens = bsz*seq. */
int gptq_rope_inplace(void* qk, int64_t token_stride, const int64_t* position_ids, int64_t pos_batch_stride, int bsz, int seq, int rows, int head_dim,
                      float base, gptq_stream_t stream);
/* The same rotation with the frequencies of a scaled RoPE (LLaMA-3.1 / 3.2 / 3.3's llama3 rule, or any other table): pair i of a row at
 * position p turns by the angle fp32(inv_freq[i] * (float)p), rounded once, through cosf / sinf, which is the angle HF computes from the same
 * fp32 table.  inv_freq is a HOST array of head_dim / 2 floats, read during the call and copied into the launch parameters (a captured graph
 * replays it; the array may be freed once the call returns).  It is required (GPTQ_ERR_NULL), each entry must be finite and > 0
 * (GPTQ_ERR_SHAPE, checked before any CUDA call), and head_dim must be at most 128 (GPTQ_ERR_UNSUPPORTED).  Everything else as
 * gptq_rope_inplace, whose unscaled rule is exp(i * -2 ln(base) / head_dim) in fp32. */
int gptq_rope_inplace_freq(void* qk, int64_t token_stride, const int64_t* position_ids, int64_t pos_batch_stride, int bsz, int seq, int rows, int head_dim,
                           const float* inv_freq, gptq_stream_t stream);

/* y[M,N] = x * rsqrt(mean(x^2) + eps) * weight, fp32 math, fp16 store.
 * Replaces TritonLlamaRMSNorm.forward / rms_norm_fwd_fused (quant/triton_norm.py:50-67, :7-39). */
int gptq_rmsnorm_fwd(const void* x, int64_t ldx, const void* weight, void* y, int64_t ldy, int M, int N, float eps, gptq_stream_t stream);

/* Device-side integer packing (the reference's "TODO: perform packing on GPU", llama.py:264):
 * the numpy shift-OR loops of QuantLinear.pack (quant/quant_linear.py:341-369).
 * intweight int32 [K,N] in [0,2^bits) -> qweight [K/32*bits, N];  zeros int32 [G,N] (already minus one)
 * -> qzeros [G, N/32*bits].  gptq_unpack_* are the inverses (used by tests and by load-time checks). */
int gptq_pack_qweight(const int32_t* intweight, int32_t* qweight, int K, int N, int bits, gptq_stream_t stream);
int gptq_pack_qzeros(const int32_t* zeros_m1, int32_t* qzeros, int G, int N, int bits, gptq_stream_t stream);
int gptq_unpack_qweight(const int32_t* qweight, int32_t* intweight, int K, int N, int bits, gptq_stream_t stream);
int gptq_unpack_qzeros(const int32_t* qzeros, int32_t* zeros_m1, int G, int N, int bits, gptq_stream_t stream);

/* fp16 [K,N] weight exactly as the reference kernel materialises it before the dot
 * (quant/quant_linear.py:114-128).  Used by tests and by load-time validation. */
int gptq_dequant(const gptq_qweight* w, void* out, int64_t ldo, gptq_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Decode engine (SURVEY.md 8(f) rank 1): one token step of a GPTQ LLaMA on a static KV cache, i.e. the
 * body of the reference's per-token benchmark loop (llama.py:419-433) -- LlamaDecoderLayer.forward over
 * TritonLlamaRMSNorm, QuantLlamaAttention.forward (quant/fused_attn.py:117-161: fused qkv, in-place RoPE,
 * KV append, SDPA, o_proj) and QuantLlamaMLP.forward (quant/fused_mlp.py:203-218) -- as a fixed sequence of
 * kernel launches on `stream`: no allocation, no host sync, position and token ids are read from device
 * memory, so the whole step can be captured once in a CUDA graph and replayed per token.
 * Per layer: [RMSNorm + qkv matvec] -> [RoPE + KV append + split-KV attention] -> [combine] ->
 * [o_proj + residual] -> [RMSNorm + gate/up matvec + SwiGLU] -> [down_proj + residual].
 */
typedef struct gptq_llama_layer {
    /* fused q|k|v (quant/fused_attn.py:177-181): n_heads query heads, then n_kv_heads key heads, then n_kv_heads value heads of head_dim
     * columns each, N = (n_heads + 2 * n_kv_heads) * head_dim.  The K/V head count is not a field: it is read from this width,
     * n_kv_heads = (N / head_dim - n_heads) / 2, and must be a positive divisor of n_heads, the same in every layer (else GPTQ_ERR_SHAPE).
     * N = 3 * n_heads * head_dim is multi-head attention (LLaMA-1); fewer K/V heads is grouped-query attention (LLaMA-2-70B, CodeLlama-34B,
     * LLaMA-3): query head h reads K/V head h / (n_heads / n_kv_heads).  Tensor parallelism requires n_kv_heads == n_heads
     * (GPTQ_ERR_UNSUPPORTED otherwise). */
    gptq_qweight qkv;
    gptq_qweight o, gate, up, down;
    const void* input_norm;  /* fp16 [hidden] */
    const void* post_norm;   /* fp16 [hidden] */
    /* Optional input gathers (device int32, NULL = identity) for act-order layers whose packed rows the host has
     * regrouped at load time so that every quantisation group is contiguous (g_idx then is the trivial k / groupsize
     * map): the matvec reads x'[k'] = x[perm[k']].  q|k|v share one map, gate|up share one map (same input, hence same
     * act-order, quant/fused_attn.py:180); down_proj's map is folded into the column order of gate|up by the host.
     * With qkv_perm set, input_norm is given in the same regrouped order (input_norm'[k'] = input_norm[perm[k']]);
     * likewise post_norm with mlp_perm.
     * Only the persistent single-kernel path implements the gathers; otherwise GPTQ_ERR_UNSUPPORTED is returned. */
    const int32_t* qkv_perm; /* [hidden] */
    const int32_t* o_perm;   /* [hidden] */
    const int32_t* mlp_perm; /* [hidden] */
} gptq_llama_layer;

typedef struct gptq_llama_model {
    int n_layers, hidden, n_heads, head_dim, intermediate, vocab;
    float rms_eps, rope_base;
    const gptq_llama_layer* layers; /* HOST array of n_layers entries (device pointers inside) */
    const void* embed;      /* fp16 [vocab, hidden] */
    const void* final_norm; /* fp16 [hidden] */
    const void* lm_head;    /* fp16 [vocab, hidden] (never quantized, llama_inference.py:46-48) */
} gptq_llama_model;

#define GPTQ_MAX_TP 8

/* Tensor-parallel decode (BASELINE config 5: LLaMA-65B across 8 GPUs; the reference has no equivalent, its multi-GPU mode is layer
 * placement, llama.py:328-382).  One process per GPU; every rank passes ITS shard of every layer in gptq_llama_model:
 *   qkv   columns of this rank's heads (q | k | v of those heads, N = 3 * n_heads * head_dim), o rows of the same heads (K = n_heads * head_dim),
 *   gate/up column slices (N = intermediate), down the matching row slice (K = intermediate), with model->n_heads / ->intermediate the LOCAL
 *   counts and model->hidden / ->vocab the full ones; lm_head points to this rank's rows [vocab_begin, vocab_end).
 * The persistent kernel adds the o_proj / down_proj partial sums into every rank's accumulators over NVLink (peer stores), so there is no
 * separate all-reduce; peer_scratch / peer_logits are the scratch and logits buffers of ALL ranks mapped into this process (gptq_ipc_*),
 * [rank] being the own ones.  Every rank must call gptq_llama_decode_step for the same step; the call still returns asynchronously. */
typedef struct gptq_llama_tp {
    int size, rank;
    int vocab_begin, vocab_end;
    int reduce_mode; /* 0: automatic; 1: every team RED-adds its partial sums into every rank; 2: local reduction, then every CTA hands a slice to the ranks */
    void* peer_scratch[GPTQ_MAX_TP];
    void* peer_logits[GPTQ_MAX_TP];
} gptq_llama_tp;

typedef struct gptq_llama_state {
    int batch;   /* sequences decoded in lock-step, 1..8 */
    int max_seq; /* KV-cache capacity in tokens */
    void* k_cache; /* fp16 [n_layers, batch, n_kv_heads, max_seq, head_dim] (n_kv_heads: gptq_llama_layer.qkv), keys stored after RoPE */
    void* v_cache; /* fp16, same shape */
    const int32_t* tokens;    /* device int32 [batch]: token ids of this step */
    const int32_t* positions; /* device int32 [batch]: position of this step's token (= tokens already cached) */
    void* logits;             /* fp16 [batch, vocab] out */
    int32_t* next_tokens;     /* device int32 [batch] out: argmax of logits, or NULL to skip */
    void* scratch;            /* device, gptq_llama_scratch_bytes() bytes, zero-filled once */
    size_t scratch_bytes;
    const gptq_llama_tp* tp;  /* NULL: single GPU */
} gptq_llama_state;

size_t gptq_llama_scratch_bytes(const gptq_llama_model* model, int batch, int max_seq);
int gptq_llama_decode_step(const gptq_llama_model* model, const gptq_llama_state* state, gptq_stream_t stream);
/* The decode step with a scaled RoPE: both engines rotate q and the appended k with the frequencies inv_freq, a HOST array of head_dim / 2
 * (= 64) floats, under gptq_rope_inplace_freq's angle rule, so the step appends exactly the cache rows gptq_rope_inplace_freq writes at the
 * same position.  model->rope_base is then unused.  NULL: model->rope_base's unscaled rule (gptq_llama_decode_step is this call with NULL).
 * A table entry that is not finite and > 0 gives GPTQ_ERR_SHAPE before any CUDA call.  The table is copied into the launch parameters, so a
 * captured step replays it.  gptq_llama_decode_launches does not depend on the rotation. */
int gptq_llama_decode_step_rope(const gptq_llama_model* model, const gptq_llama_state* state, const float* inv_freq, gptq_stream_t stream);
/* Number of kernels one gptq_llama_decode_step launches for this model/state: 1 when the persistent single-kernel
 * path applies (batch 1 to 8, every layer int4 in kernel form -- act-order layers with input gathers included -- and a shape
 * whose staging buffers fit the device's shared memory at this batch; tensor parallelism at batch 1 only), else the
 * per-operation kernel chain.  Each sequence b is stepped at its own positions[b]. */
int gptq_llama_decode_launches(const gptq_llama_model* model, const gptq_llama_state* state);
/* Diagnostics / tests: byte offset, inside the scratch area, of the persistent kernel's region.  It begins with the residual
 * stream ping-pong: two fp16 [batch, hidden] arrays (row b = sequence b), each padded to 256 bytes (after a step: [0] = the
 * residual entering the last layer, [1] = the residual after the last layer's attention block). */
size_t gptq_llama_persistent_scratch_offset(const gptq_llama_model* model, int batch, int max_seq);

/* ------------------------------------------------------------------------------------------------
 * Scoring (the perplexity evaluation of llama.py:246-259): per-row log-likelihood of a target token through the fp16 lm_head,
 *   logprob[m] = l[m, t_m] - logsumexp_v l[m, v],   l = fp16(x[m] . w[v]) (fp32 accumulation, one fp16 rounding),
 * with the log-softmax in fp32 on the fp16 logits and the [M, V] logits never written to memory.
 * x fp16 [M, K] (ldx elements between rows), w fp16 [V, K] as nn.Linear stores the lm_head (ldw), targets int32 [M] in [0, V)
 * (the caller validates them; a row whose target is outside that range gets NaN), logprob fp32 [M] out.
 * K must be a positive multiple of 64; x and w 16-byte aligned, ldx and ldw multiples of 8.  The workspace (256-byte aligned,
 * gptq_lm_head_logprob_workspace_bytes) follows the workspace rule above.  A row's result is bit-for-bit the same whatever M
 * is and whatever the other rows hold. */
size_t gptq_lm_head_logprob_workspace_bytes(int M, int V);
int gptq_lm_head_logprob(const void* x, int64_t ldx, const void* w, int64_t ldw, int M, int K, int V, const int32_t* targets, float* logprob,
                         void* workspace, size_t ws_bytes, gptq_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Extending cached sequences (LlamaDecoder.extend, generate(..., reuse_cache=True)).
 * Causal attention of new rows over a sequence's cached prefix, read in place from the decode engine's KV cache (one layer's slice:
 * fp16 [batch, n_heads, max_seq, head_dim], keys after RoPE).  Span i = (seq[i], start[i], rows[i]): its query rows are the next rows[i]
 * rows of q (spans in order, no gaps), at positions start[i] .. start[i] + rows[i] - 1; row j attends to keys 0 .. start[i] + j of
 * sequence seq[i], whose rows start[i] .. start[i] + rows[i] - 1 the caller has already written.  Cache rows at or past
 * start[i] + rows[i] are never read into the result (they may hold anything).  span_* are HOST arrays; sequences are distinct.
 * q / out: fp16 rows of n_heads * head_dim (ldq / ldo elements apart; q may be the q part of the fused qkv output).
 * head_dim must be 128 (GPTQ_ERR_UNSUPPORTED otherwise); 0 <= n_spans <= 64; ldq, ldo multiples of 8 (GPTQ_ERR_SHAPE otherwise); q, the
 * caches and out 16-byte aligned.  Zero rows in total launch nothing.  Arithmetic: fp32 scores and online softmax, P rounded to fp16 for
 * the P.V product, fp32 accumulation, one fp16 rounding of the output.  A span's result is bit-for-bit the same whatever the other spans
 * of the call are and in whatever order they come. */
int gptq_cached_attention(const void* q, int64_t ldq, const void* k_cache, const void* v_cache, int batch, int n_heads, int head_dim, int max_seq,
                          int n_spans, const int32_t* span_seq, const int32_t* span_start, const int32_t* span_rows, void* out, int64_t ldo,
                          gptq_stream_t stream);
/* The same over a grouped-query cache: the caches hold n_kv_heads heads (fp16 [batch, n_kv_heads, max_seq, head_dim]) and query head h reads
 * K/V head h / (n_heads / n_kv_heads).  n_kv_heads must be a positive divisor of n_heads (GPTQ_ERR_SHAPE otherwise).  gptq_cached_attention is
 * this call with n_kv_heads = n_heads. */
int gptq_cached_attention_gqa(const void* q, int64_t ldq, const void* k_cache, const void* v_cache, int batch, int n_heads, int n_kv_heads, int head_dim,
                              int max_seq, int n_spans, const int32_t* span_seq, const int32_t* span_start, const int32_t* span_rows, void* out, int64_t ldo,
                              gptq_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Sampling (model.generate(do_sample=True, ...) of llama_inference.py:119-127, with HF's warpers in HF's order): one token per row of the
 * fp16 logits a decode step leaves in gptq_llama_state.logits, written to next_tokens[b].  A launch of its own after the step, so one kernel
 * serves both decode engines.  Every gptq_sampling field is a DEVICE array of `batch` entries (read when the kernel runs, so a CUDA graph
 * can replay the call with new values).  For row b, with l the fp16 logits, p = positions[b] (the step's position):
 *   1. eos: if 0 <= eos_token[b] < vocab and p + 1 < min_length[b] (HF MinLengthLogitsProcessor: cur_len = p + 1), l[eos] = -inf.
 *      NaN counts as -inf.
 *   2. temperature[b] <= 0 (or NaN): the argmax, lowest id on ties (the decode step's next_tokens, with eos excluded while suppressed).
 *      Otherwise z_v = fp32(float(l_v) / T), the correctly rounded fp32 division (HF TemperatureLogitsWarper on logits.float()).
 *   3. top-k (0 < top_k[b] < vocab, else off): keep v iff z_v >= z_(k), the k-th largest z counted with multiplicity (HF TopKLogitsWarper).
 *   4. weights over the top-k set: w_v = exp((double)z_v - (double)z_max) in fp64; if some z is +inf, those entries weigh 1 and all others 0.
 *   5. top-p (top_p[b] < 1, else off): keep v iff (weight of top-k tokens with z_u > z_v) / (top-k weight) < top_p.  For distinct values this
 *      is HF's TopPLogitsWarper (cumsum <= 1 - top_p removed); a tie group straddling the boundary is kept whole, where HF keeps the part
 *      torch.sort happens to put first.  The largest z is always kept.
 *   6. draw: (x0, x1, x2, x3) = Philox4x32-10(counter (p, 0, 0, 0), key (seed lo 32 bits, seed hi 32 bits)),
 *      u = ((x0 >> 5) * 2^26 + (x1 >> 6)) * 2^-53; the token is the first kept id, ascending, whose inclusive fp64 running weight exceeds
 *      u * W (W: the kept weight); if rounding leaves none, the last kept id.
 *   7. a row with nothing above -inf gives 0.
 * The token depends only on the row's logits, its parameters and its position: no float atomics, every float sum in a fixed order.  The
 * counter is the position, so a re-run or resumed sequence draws the same u at the same position.  Running weights are summed per block of
 * ids and then over the blocks, so they can differ from a sequential sum in the last bits: a draw whose u * W lies that close to a
 * cumulative boundary may take the neighbouring token.
 * batch 1..8, vocab >= 1, ld >= vocab (GPTQ_ERR_SHAPE); vocab > 131072 gives GPTQ_ERR_UNSUPPORTED; logits 2-byte, seed 8-byte and the other
 * arrays 4-byte aligned.  No workspace. */
typedef struct gptq_sampling {
    const float* temperature;
    const int32_t* top_k;
    const float* top_p;
    const uint64_t* seed;
    const int32_t* eos_token;  /* < 0: none */
    const int32_t* min_length;
} gptq_sampling;
int gptq_sample_tokens(const void* logits, int64_t ld, int batch, int vocab, const int32_t* positions, const gptq_sampling* params,
                       int32_t* next_tokens, gptq_stream_t stream);

/* Device memory that other processes of the node can map (CUDA IPC), for the tensor-parallel scratch / logits buffers:
 * alloc returns a zero-filled device buffer and its 64-byte handle (to be sent to the peers, e.g. with torch.distributed);
 * open maps a peer's buffer into this process.  close / free release them. */
int gptq_ipc_alloc(size_t bytes, void** ptr, unsigned char handle[64]);
int gptq_ipc_open(const unsigned char handle[64], void** ptr);
int gptq_ipc_close(void* ptr);
int gptq_ipc_free(void* ptr);

#ifdef __cplusplus
}
#endif
#endif /* GPTQ_B200_H */
