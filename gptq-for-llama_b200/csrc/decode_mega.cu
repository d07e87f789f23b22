// Persistent decode step: ONE cooperative kernel per token (batch 1 to 8, int4 kernel-form layers; at batch 1 optionally one tensor-parallel shard).
//
// One CTA per SM (132 on H100 SXM), each with two consumer TEAMS of 8 warps and one producer warp per team.
// Everything a token reads from HBM -- packed weights with their scales/zeros, the KV cache, the fp16 lm_head --
// is streamed by the producer warps through the TMA unit (cp.async.bulk.tensor / cp.async.bulk) into a per-team ring of 17 KB stages in
// shared memory, in one fixed order per team for the whole token, so the producers run ahead across operations
// and across grid barriers: while the consumers synchronise, the next operation's bytes are already landing.
//
//   per layer:  Q  qkv matvec      x = rmsnorm(resid [+ fp16(acc_down)])           -> RED acc_qkv
//               A  attention       q,k,v = fp16(acc_qkv); RoPE; KV append; a head's 32-key units dealt to its teams -> part
//               O  o_proj matvec   x = combine(part)                                -> RED acc_o
//               G  gate|up matvec  x = rmsnorm(resid + fp16(acc_o))                 -> RED acc_gate, acc_up
//               D  down matvec     x = fp16(silu(acc_gate) * acc_up)                -> RED acc_down
//   then        L  lm_head         x = rmsnorm(resid + fp16(acc_down)), fp16 rows   -> logits;   argmax
//
// Matvec stage = up to 4 k-steps (16 packed rows = 128 k) x 256 columns of ONE quantisation group, plus that
// group's 256 scales and 256 zeros.  The weights of a stage arrive as ONE cp.async.bulk.tensor request (3-D view of the
// packed matrix: 128-byte column chunk x packed row x chunk index, box 32 x 16 x 8, SWIZZLE_128B so that the four rows a
// quarter-warp reads land on distinct banks); one tensor map per row stride serves every layer (the matrices of a
// class are addressed through the chunk coordinate).  Arithmetic (quant/quant_linear.py:113-133 regrouped): inside a group
//      sum_k x_k (w_k - z) s  =  s * ( sum_k x_k w_k  -  z * sum_k x_k )
// so the consumers feed the RAW nibbles to the tensor pipe (mma.sync m16n8k16, operands swapped: A = 16 output
// columns x 16 k of weights, B = x): a nibble masked in place IS an fp16 subnormal (n * 2^-24, or 16 n * 2^-24 for
// the odd nibbles, whose x carries a further 2^-4), products are exact and accumulate in fp32, and scale / zero are
// applied ONCE per group on the fp32 accumulator together with the group's sum of x (computed when x is staged).
// The staged x is scaled by a power of two per staged range (XScale) so that even the odd nibbles' copy of a small
// input stays an fp16 normal; the column totals are scaled back once.  5 integer instructions + 1 HMMA per packed
// word; the result differs from the reference only by NOT rounding every dequantised weight to fp16 (it is closer to
// the exact product); tests/test_gpu_decode_input_ranges.py holds it to the float64 product from tiny to massive inputs.
//
// Split-K partial sums are accumulated with red.global.add.f32 into fp32 vectors that the NEXT operation
// rounds to fp16 exactly where the reference rounds (a QuantLinear output is fp16); each vector is re-zeroed
// one operation after its last reader.  Only the fp32 summation order of those partials is unordered.
// Tensor parallelism (gptq_llama_tp): the o_proj / down_proj sums also go to the peer GPUs' accumulators (NVLink, see MegaParams).
//
// Batch B = 2..8 (the BATCH instantiation): the eight columns of the B operand carry up to eight DIFFERENT sequences (lane group g
// reads sequence min(g, B - 1)), so one weight stream, one dequantisation and one HMMA per packed word serve the whole batch.  Every
// per-sequence vector (residual stream, accumulators, staged x and its step sums, RoPE angles, logits) gets a [B] dimension; the
// attention teams are dealt to (sequence, head) pairs in proportion to each sequence's context (seq_teams).  Batch 1 is the
// !BATCH instantiation: its loops over the sequences have the compile-time count 1.
#include "common.cuh"
#include "int4_core.cuh"
#include "kernels.h"
#include "wgmma.cuh"

namespace gptq {
namespace {

using namespace int4;

constexpr int kTeams = 2;                             // consumer teams per CTA
constexpr int kTeamWarps = 8;
constexpr int kTeamThreads = kTeamWarps * 32;         // 256
constexpr int kConsumers = kTeams * kTeamThreads;     // 512
constexpr int kConsumerWarps = kTeams * kTeamWarps;   // 16
constexpr int kBlock = kConsumers + 32 * kTeams;      // + one producer warp per team
constexpr int kSlabCols = 256;
constexpr int kStageSteps = 4;         // k-steps (of 32 k = 4 packed rows) per stage
constexpr int kStepBytes = 4096;       // 4 packed rows x 256 columns
constexpr int kScaleOff = kStageSteps * kStepBytes;     // 16384: 256 fp16 scales of the stage's group
constexpr int kZeroOff = kScaleOff + 512;               // 16896: 32 qzeros words (256 nibbles)
constexpr int kStageBytes = 17 * 1024;                  // 17408: stages are 1 KB aligned (128-byte swizzle atoms of the TMA boxes)
constexpr int kHD = 128;
constexpr int kKeysPerUnit = 32;       // attention work unit: 32 keys of one head = 8 KB of K + 8 KB of V = one stage
constexpr int kVOff = 8192 + 256;      // V rows of a KV stage (K rows at offset 0)
constexpr int kRec = kHD + 4;          // floats per attention partial record: m, l, 2 pad, o[128]
constexpr int kMaxLayers = 80;
constexpr int kMaxStages = 8;
constexpr int kTeamScratch = 4224;     // per-team scratch (attention merge buffers / lm_head partials)
constexpr int kLmStageBytes = 16384;   // lm_head bytes per stage (whole rows)
constexpr int kMaxBatch = 8;           // sequences of one step (the columns of the mma B operand)
constexpr int kMaxTeams = 1024;        // >= kTeams * SM count of any device this library runs on (attention records in the scratch region)

#ifdef GPTQ_TRACE
}  // namespace
__device__ unsigned long long* g_mega_trace = nullptr;
namespace {

#define MTRACE(id)                                                                                                       \
    do {                                                                                                                 \
        if (g_mega_trace != nullptr && threadIdx.x == 0 && (id) < 36) {                                                   \
            unsigned long long t_;                                                                                       \
            asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t_));                                                        \
            g_mega_trace[blockIdx.x * 64 + (id)] = t_;                                                                   \
        }                                                                                                                \
    } while (0)
#else
#define MTRACE(id) \
    do {           \
    } while (0)
#endif

#ifdef GPTQ_TRACE
// per-op counters of layer 2, team 0 of every CTA: ids 48 + 3 * op + {0: cycles in the op, 1: of which waiting for stages, 2: stages}
#define OPTRACE_BEGIN(ring)                       \
    const long long optr_t0 = clock64();          \
    const long long optr_w0 = (ring).waited;      \
    const int optr_s0 = (ring).stages
#define OPTRACE_END(ring, layer, op)                                                                                   \
    do {                                                                                                               \
        if (g_mega_trace != nullptr && threadIdx.x == 0 && (layer) == 2) {                                              \
            g_mega_trace[blockIdx.x * 64 + 48 + 3 * (op)] = (unsigned long long)(clock64() - optr_t0);                  \
            g_mega_trace[blockIdx.x * 64 + 48 + 3 * (op) + 1] = (unsigned long long)((ring).waited - optr_w0);          \
            g_mega_trace[blockIdx.x * 64 + 48 + 3 * (op) + 2] = (unsigned long long)((ring).stages - optr_s0);          \
        }                                                                                                              \
    } while (0)
#else
#define OPTRACE_BEGIN(ring) \
    do {                    \
    } while (0)
#define OPTRACE_END(ring, layer, op) \
    do {                             \
    } while (0)
#endif

struct MatDesc {
    const __half* sc;
    const uint32_t* qz;
    int gs_steps;  // k-steps per quantisation group (groupsize / 32)
    int tmap;      // tensor-map class of qweight (0: N = 3H, 1: N = H, 2: N = I)
    int chunk0;    // chunk coordinate of the matrix: (qweight - class base) / 128 bytes
};
struct LayerDesc {
    MatDesc qkv, o, gate, up, down;
    const __half* input_norm;
    const __half* post_norm;
    const int32_t* qkv_perm;  // act-order input gathers (gptq_llama_layer), nullptr = identity
    const int32_t* o_perm;
    const int32_t* mlp_perm;
};
constexpr int kMaxTP = 8;
struct MegaParams {
    // H: hidden size (the residual stream, replicated under tensor parallelism); n_heads, Hq = 128 * n_heads, I: this rank's attention heads
    // / attention width / MLP width (the full ones on a single GPU); V: vocabulary, [v0, v1): the lm_head rows of this rank
    int n_layers, H, Hq, I, V, v0, v1, n_heads, max_seq, n_stages, lm_rows;
    int tp_size, tp_rank, tp_exchange;  // tp_exchange: reduce locally first, then hand slices to the ranks (else: every team REDs into every rank)
    float eps, inv_base, scale;
    const __half* embed;
    const __half* final_norm;
    const __half* lm_head;
    const int32_t* tokens;
    const int32_t* positions;
    __half* k_cache;
    __half* v_cache;
    size_t layer_stride;  // halves per layer in the caches
    __half* logits;
    int32_t* next_token;
    // scratch (device)
    __half* resid[2];  // residual stream ping-pong, fp16 [H]
    float* acc_qkv;    // [3H]
    float* acc_o;      // [H]
    float* acc_g;      // [I]
    float* acc_u;      // [I]
    float* acc_d;      // [H]
    float* part;       // [teams][kRec]  attention partial records (m, l, pad, pad, o[128]), one per team and layer
    float* rope_cs;    // [128]: cos[64], sin[64] of this step's position
    unsigned long long* bar;  // [0]: monotonic arrival counter of the grid barrier, [1]: its value when the previous launch ended
    // tensor parallelism (tp_size > 1): a rank first reduces its o_proj / down_proj partial sums locally (acc_*_loc), then every CTA adds its
    // slice of that vector into EVERY rank's accumulator over NVLink (peer pointers, red.sys: 4 bytes x H x ranks per hand-off instead of
    // every team's partials); the lm_head slices are stored into every rank's logits; the hand-offs that follow use a cross-GPU barrier:
    // xbar = this rank's arrival counters, one 256-byte line per source rank, line kMaxTP = value at launch end
    float* acc_o_loc;  // [H] this rank's partial sums of o_proj / down_proj before they are handed to the ranks (tp_size > 1)
    float* acc_d_loc;
    float* acc_o_peer[kMaxTP];
    float* acc_d_peer[kMaxTP];
    __half* logits_peer[kMaxTP];
    unsigned long long* xbar_peer[kMaxTP];
    LayerDesc layers[kMaxLayers];
    CUtensorMap tmaps[6];  // [class]: 16-row boxes (a full stage), [3 + class]: 4-row boxes (one k-step)
    // BATCH instantiation only: sequences of the step, and halves between the sequences' rows of the staged x (H + 32: a stride of
    // 64 mod 128 bytes puts the two lane groups of a quarter-warp on different banks).  Per-sequence vectors are [batch][n] with
    // n = H, 3 Hq, I, V or 128 (rope_cs); resid, acc_* and rope_cs are sized for the batch.
    int batch, xs_stride;
};

// ---- work split ------------------------------------------------------------------------------------------------
// U units of an operation are dealt to the nb teams as contiguous ranges [T*U/nb, (T+1)*U/nb).
__device__ __forceinline__ void team_range(unsigned T, unsigned U, unsigned nb, int& a, int& b) {
    a = (int)((T * U) / nb);  // T * U < 2^32 (checked by mega_plan)
    b = (int)(((T + 1) * U) / nb);
}
// Attention: the teams are dealt to the heads (nb / n_heads or one more each), a head's 32-key units to its teams: no team meets two
// heads, so every team writes exactly one partial record per layer (a neutral one if it has no unit).
struct HeadTeams {
    int first, count;  // teams [first, first + count) serve the head
};
__device__ __forceinline__ HeadTeams head_teams(int head, int n_heads, unsigned nb) {
    const int base = (int)nb / n_heads, rem = (int)nb % n_heads;
    HeadTeams h;
    h.first = head * base + min(head, rem);
    h.count = base + (head < rem ? 1 : 0);
    return h;
}
// (head, unit range [b0, b1) inside the head) of team T for a context of upb units per head
__device__ __forceinline__ void attn_range(unsigned T, int n_heads, unsigned nb, int upb, int& head, int& b0, int& b1) {
    const int base = (int)nb / n_heads, rem = (int)nb % n_heads;
    const int split = rem * (base + 1);
    int idx, cnt;
    if ((int)T < split) {
        head = (int)T / (base + 1);
        idx = (int)T - head * (base + 1);
        cnt = base + 1;
    } else {
        head = rem + ((int)T - split) / base;
        idx = ((int)T - split) % base;
        cnt = base;
    }
    b0 = idx * upb / cnt;
    b1 = (idx + 1) * upb / cnt;
}

// k-steps of the stage that starts `gpos` steps into its quantisation group, in a segment with `left` steps to go
__device__ __forceinline__ int stage_steps(int gpos, int gs_steps, int left) { return min(min(kStageSteps, gs_steps - gpos), left); }

// position of sequence s in this step, clamped to the cache (the host rejects pos >= max_seq; the kernel must not write outside)
__device__ __forceinline__ int step_pos(const MegaParams& p, int s) { return min(max(p.positions[s], 0), p.max_seq - 1); }

// Batched attention: sequence s is served by teams [first, first + count): n_heads teams plus a share of the other nb - batch * n_heads
// teams in proportion to its 32-key units (cumulative rounding: the shares add up to nb exactly).  Inside a sequence the teams are
// dealt to its heads as in batch 1 (attn_range / head_teams with count teams).  mega_plan guarantees batch * n_heads <= nb.
__device__ __forceinline__ HeadTeams seq_teams(const MegaParams& p, int s, unsigned nb) {
    int before = 0, mine = 0, tot = 0;
#pragma unroll 1
    for (int i = 0; i < p.batch; ++i) {
        const int units = step_pos(p, i) / kKeysPerUnit + 1;
        before += i < s ? units : 0;
        mine = i == s ? units : mine;
        tot += units;
    }
    const long long extra = (long long)nb - (long long)p.batch * p.n_heads;
    HeadTeams h;
    h.first = s * p.n_heads + (int)(extra * before / tot);
    h.count = (s + 1) * p.n_heads + (int)(extra * (before + mine) / tot) - h.first;
    return h;
}
// sequence of team T and that sequence's teams
__device__ __forceinline__ int team_seq(const MegaParams& p, unsigned T, unsigned nb, HeadTeams& st) {
    int s = 0;
#pragma unroll 1
    for (;; ++s) {
        st = seq_teams(p, s, nb);
        if ((int)T < st.first + st.count || s == p.batch - 1) return s;
    }
}
// (sequence, head, unit range [b0, b1)) of team T; pos = that sequence's position, Tlen = pos + 1 keys
template <bool BATCH>
__device__ __forceinline__ int attn_work(const MegaParams& p, unsigned T, unsigned nb, int& pos, int& Tlen, int& head, int& b0, int& b1) {
    int s = 0;
    HeadTeams st{0, (int)nb};
    if constexpr (BATCH) s = team_seq(p, T, nb, st);
    pos = step_pos(p, s);
    Tlen = pos + 1;
    const int upb = (Tlen + kKeysPerUnit - 1) / kKeysPerUnit;
    attn_range(T - st.first, p.n_heads, st.count, upb, head, b0, b1);
    return s;
}

// ---- team / CTA synchronisation ------------------------------------------------------------------------------------
__device__ __forceinline__ void team_sync(int team) { asm volatile("bar.sync %0, 256;" ::"r"(team + 1) : "memory"); }
__device__ __forceinline__ void cta_sync() { asm volatile("bar.sync 3, 512;" ::: "memory"); }  // all consumer warps (not the producers)

// ---- producer ------------------------------------------------------------------------------------------------------
struct ProdRing {
    uint32_t ring, full, empty;
    int stage, use, nstages;
#ifdef GPTQ_TRACE
    long long blocked;  // cycles spent waiting for a free stage
#endif
};
__device__ __forceinline__ uint32_t prod_acquire(ProdRing& r, uint32_t& bar) {
#ifdef GPTQ_TRACE
    const long long t0 = clock64();
#endif
    if (r.use > 0) mbar_wait_backoff(r.empty + r.stage * 8, (r.use - 1) & 1u);  // the consumers released the previous use of this stage
#ifdef GPTQ_TRACE
    r.blocked += clock64() - t0;
#endif
    bar = r.full + r.stage * 8;
    return r.ring + r.stage * kStageBytes;
}
__device__ __forceinline__ void prod_advance(ProdRing& r) {
    if (++r.stage == r.nstages) {
        r.stage = 0;
        ++r.use;
    }
}

__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap* tm, int c0, int c1, int c2, uint32_t bar, uint64_t policy) {
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1, {%2, %3, %4}], [%5], %6;" ::"r"(dst),
                 "l"(tm), "r"(c0), "r"(c1), "r"(c2), "r"(bar), "l"(policy)
                 : "memory");
}

// What one ring stage holds: a weight stage is n k-steps of packed rows from a tensor map (a 16-row box when n == kStageSteps, else n
// 4-row boxes) plus the group's scales (a) and qzeros (b); a KV stage is the K (a) and V (b) rows of one 32-key unit; an lm_head stage
// is whole fp16 rows (a).
struct StageLoad {
    const CUtensorMap* tm;  // weight stage: the map of its boxes, else nullptr
    int row, chunk, n;      // first packed row, chunk coordinate, k-steps
    const void* a;
    const void* b;          // nullptr: none
    uint32_t a_off, b_off, a_bytes, b_bytes;
};

// The order in which a team's producer fills its ring over the whole token: per layer the stages of Q (qkv), A (K/V units), O, G
// (gate|up) and D, then L (lm_head) -- the order in which the team's consumers take them (run_matvec, run_attention, run_lm_head).
// One flat walk rather than a loop nest per operation: measured 3 % faster at 7B (DESIGN.md 4.1).
template <bool BATCH>
struct StageWalk {
    enum { kQ, kA, kO, kG, kD, kL, kEnd };
    int l = 0, op = -1, u = 0, u1 = 0;  // layer, operation, next unit of the team's range [u, u1) of that operation
    int Tlen = 0;                       // A: the sequence's key count
    size_t kv = 0;                      // A: offset of the team's head (row 0) in the layer's K / V cache, in halves

    // the descriptor of the next stage; false once the token's last stage has been taken
    __device__ __forceinline__ bool next(const MegaParams& p, unsigned T, unsigned nb, StageLoad& s) {
        while (u >= u1) {
            if (op == kEnd) return false;
            if (++op == kL && l + 1 < p.n_layers) {
                ++l;
                op = kQ;
            }
            if (op == kA) {
                int pos, head;
                const int seq = attn_work<BATCH>(p, T, nb, pos, Tlen, head, u, u1);
                kv = (size_t)l * p.layer_stride + (size_t)(seq * p.n_heads + head) * p.max_seq * kHD;
            } else if (op == kL) {
                team_range(T, (unsigned)((p.v1 - p.v0 + p.lm_rows - 1) / p.lm_rows), nb, u, u1);
            } else if (op != kEnd) {
                int K, N, nm;
                matvec_shape(p, K, N, nm);
                team_range(T, (unsigned)(nm * (N / kSlabCols)) * (K / 32), nb, u, u1);
            }
        }
        s.tm = nullptr;
        s.b = nullptr;
        s.b_bytes = 0;
        if (op == kA) {
            const int nrows = min(kKeysPerUnit, Tlen - u * kKeysPerUnit);
            const size_t off = kv + (size_t)u * kKeysPerUnit * kHD;
            s.a = p.k_cache + off;
            s.b = p.v_cache + off;
            s.a_off = 0;
            s.b_off = kVOff;
            s.a_bytes = s.b_bytes = nrows * 256;
            ++u;
        } else if (op == kL) {
            const int R = p.lm_rows, nrows = min(R, p.v1 - p.v0 - u * R);
            s.a = p.lm_head + (size_t)u * R * p.H;
            s.a_off = 0;
            s.a_bytes = (uint32_t)nrows * p.H * 2;
            ++u;
        } else {
            // units of 32 k x 256 columns, slab-major (gate|up: one virtual matrix of 2 N/256 slabs); a stage stays inside one slab's
            // k-range and one quantisation group (run_matvec takes the same steps)
            int K, N, nm;
            matvec_shape(p, K, N, nm);
            const int nk = K / 32, nslab = N / kSlabCols;
            const int slab_v = u / nk, ks = u - slab_v * nk;
            const int mi = slab_v >= nslab ? 1 : 0, slab = slab_v - mi * nslab;
            const LayerDesc& L = p.layers[l];
            const MatDesc& m = op == kQ ? L.qkv : op == kO ? L.o : op == kD ? L.down : mi ? L.up : L.gate;
            const int g = ks / m.gs_steps;
            s.n = stage_steps(ks - g * m.gs_steps, m.gs_steps, min(nk - ks, u1 - u));
            s.tm = &p.tmaps[(s.n == kStageSteps ? 0 : 3) + m.tmap];
            s.row = ks * 4;
            s.chunk = m.chunk0 + slab * (kSlabCols / 32);
            s.a = m.sc + (size_t)g * N + slab * kSlabCols;
            s.b = m.qz + (size_t)g * (N >> 3) + slab * (kSlabCols / 8);
            s.a_off = kScaleOff;
            s.b_off = kZeroOff;
            s.a_bytes = 512;
            s.b_bytes = 128;
            u += s.n;
        }
        return true;
    }

    // K x N of the current matvec; nm = 2: gate|up side by side
    __device__ __forceinline__ void matvec_shape(const MegaParams& p, int& K, int& N, int& nm) const {
        K = op == kO ? p.Hq : op == kD ? p.I : p.H;
        N = op == kQ ? 3 * p.Hq : op == kG ? p.I : p.H;
        nm = op == kG ? 2 : 1;
    }
};

// Every byte a stage brings is read once per token, and the token streams far more than L2 holds, so the loads ask L2 to evict their lines
// first: the lines the hand-offs use (accumulators, attention records, residual rows, the barrier counter) stay resident instead of being
// pushed out by the stream.
template <bool BATCH>
__device__ void producer_loop(const MegaParams& p, ProdRing r, unsigned T, unsigned nb) {
    uint64_t policy;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(policy));
    StageWalk<BATCH> walk;
    StageLoad s;
#pragma unroll 1
    while (walk.next(p, T, nb, s)) {
        uint32_t bar;
        const uint32_t dst = prod_acquire(r, bar);
        mbar_expect_tx(bar, (s.tm != nullptr ? s.n * kStepBytes : 0) + s.a_bytes + s.b_bytes);
        if (s.tm != nullptr) {
            if (s.n == kStageSteps) {
                tma_load_3d(dst, s.tm, 0, s.row, s.chunk, bar, policy);
            } else {
                for (int j = 0; j < s.n; ++j) tma_load_3d(dst + j * kStepBytes, s.tm, 0, s.row + 4 * j, s.chunk, bar, policy);
            }
        }
        bulk_copy_g2s(dst + s.a_off, s.a, s.a_bytes, bar, policy);
        if (s.b != nullptr) bulk_copy_g2s(dst + s.b_off, s.b, s.b_bytes, bar, policy);
        prod_advance(r);
    }
#ifdef GPTQ_TRACE
    if (g_mega_trace != nullptr && (T & 1) == 0) g_mega_trace[(T / kTeams) * 64 + 63] = (unsigned long long)r.blocked;
#endif
}

// ---- consumer side of the ring -----------------------------------------------------------------------------------------
struct ConsRing {
    uint32_t ring, full;  // stage 0 / full[0]; empty[s] sits kMaxStages * 8 bytes after full[s]
    uint32_t tile, bar;   // current stage
    uint32_t parity;
    int left, nstages;
#ifdef GPTQ_TRACE
    long long waited;  // cycles spent waiting for stages to land
    int stages;
#endif
};
__device__ __forceinline__ uint32_t cons_wait(ConsRing& c) {
#ifdef GPTQ_TRACE
    const long long t0 = clock64();
#endif
    mbar_wait(c.bar, c.parity);
#ifdef GPTQ_TRACE
    c.waited += clock64() - t0;
    ++c.stages;
#endif
    return c.tile;
}
// every lane of the warp has finished reading the stage
__device__ __forceinline__ void cons_release(ConsRing& c, int lane) {
    __syncwarp();
    if (lane == 0) mbar_arrive(c.bar + kMaxStages * 8);
    c.tile += kStageBytes;
    c.bar += 8;
    if (--c.left == 0) {
        c.left = c.nstages;
        c.tile = c.ring;
        c.bar = c.full;
        c.parity ^= 1u;
    }
}

// ---- grid barrier: one monotonic 64-bit arrival counter ----------------------------------------------------------------
// arrive = red.release (fire and forget), wait = poll the same word with ld.acquire until it reaches this barrier's
// target.  `target` lives in thread 0 of each CTA.
__device__ __forceinline__ void grid_barrier(unsigned long long* bar, unsigned long long& target) {
    cta_sync();
    if (threadIdx.x == 0) {
        target += gridDim.x;
        asm volatile("red.release.gpu.global.add.u64 [%0], 1;" ::"l"(bar) : "memory");
        unsigned long long v;
        do {
            asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(bar) : "memory");
        } while (v < target);
    }
    cta_sync();
}

// Cross-GPU barrier of all CTAs of all tensor-parallel ranks: every CTA adds 1 to ITS source line of every rank's counter block and polls its
// own rank's lines.  ONE system-scope fence per CTA makes its remote REDs (partial sums in the peers' accumulators) visible before its
// arrivals; the arrivals themselves and the polls are relaxed (the counters and the data they guard live in the polling GPU's own L2, and
// everything that is read afterwards bypasses L1).
__device__ __forceinline__ void tp_barrier(const MegaParams& p, unsigned long long& target) {
    cta_sync();
    if (threadIdx.x == 0) {
        target += gridDim.x;
        asm volatile("fence.acq_rel.sys;" ::: "memory");
        for (int q = 0; q < p.tp_size; ++q)
            asm volatile("red.relaxed.sys.global.add.u64 [%0], 1;" ::"l"(p.xbar_peer[q] + 32 * p.tp_rank) : "memory");
        const unsigned long long* mine = p.xbar_peer[p.tp_rank];
        for (int q = 0; q < p.tp_size; ++q) {
            unsigned long long v;
            do {
                asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(mine + 32 * q) : "memory");
            } while (v < target);
        }
        asm volatile("fence.acq_rel.gpu;" ::: "memory");
    }
    cta_sync();
}

// This rank's locally reduced vector (n floats, complete after a grid barrier) is added into every rank's accumulator and cleared for its next use.
__device__ __forceinline__ void tp_exchange(const MegaParams& p, float* loc, float* const* peers, int n) {
    const int per = (n + gridDim.x - 1) / gridDim.x;
    const int lo = blockIdx.x * per, hi = min(n, lo + per);
    for (int j = lo + threadIdx.x; j < hi; j += kConsumers) {
        const float v = ld_cg(loc + j);
        loc[j] = 0.f;
        for (int q = 0; q < p.tp_size; ++q) asm volatile("red.relaxed.sys.global.add.f32 [%0], %1;" ::"l"(peers[q] + j), "f"(v) : "memory");
    }
}

__device__ __forceinline__ void zero_slice(float* buf, int n) {
    // this CTA's share of a distributed memset (n is a multiple of 4)
    const int per = ((n / 4 + gridDim.x - 1) / gridDim.x);
    const int lo = blockIdx.x * per, hi = min(n / 4, lo + per);
    for (int i = lo + threadIdx.x; i < hi; i += kConsumers) reinterpret_cast<float4*>(buf)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
}

// sum of v and the maxima of the two 16-bit lanes of m over the consumer threads (red_s: 2 * kConsumerWarps words)
__device__ __forceinline__ float block_sum(float v, uint32_t& m, float* red_s) {
    v = warp_sum(v);
    const uint32_t mx = __reduce_max_sync(0xffffffffu, m & 0xffffu), my = __reduce_max_sync(0xffffffffu, m >> 16);
    cta_sync();
    if ((threadIdx.x & 31) == 0) {
        red_s[threadIdx.x >> 5] = v;
        reinterpret_cast<uint32_t*>(red_s)[kConsumerWarps + (threadIdx.x >> 5)] = mx | (my << 16);
    }
    cta_sync();
    float t = 0.f;
    m = 0;
#pragma unroll
    for (int w = 0; w < kConsumerWarps; ++w) {
        t += red_s[w];
        m = __vmaxu2(m, reinterpret_cast<const uint32_t*>(red_s)[kConsumerWarps + w]);
    }
    return t;
}

// ---- x staging ----------------------------------------------------------------------------------------------------------
// Matvec input layout: 8 consecutive k (natural order, 4 half2 words w0..w3) are stored k-permuted as
// (k0,k4)(k1,k5)(k2,k6)(k3,k7): the B fragments of the two MMAs of a packed word.
__device__ __forceinline__ uint4 perm8(uint32_t w0, uint32_t w1, uint32_t w2, uint32_t w3) {
    return make_uint4(__byte_perm(w0, w2, 0x5410), __byte_perm(w0, w2, 0x7632), __byte_perm(w1, w3, 0x5410), __byte_perm(w1, w3, 0x7632));
}
// position of natural index j (0..7) inside the permuted run of 8
__device__ __forceinline__ int perm_pos(int j) { return ((j & 3) << 1) + (j >> 2); }

// A staged range (the whole row of Q / G, a team's k-range of O / D; per sequence) is scaled by a power of two 2^e chosen from its largest
// |x|, and the pairs that meet the ODD nibbles (k1,k5 / k3,k7; mask 0x00f000f0 = 16 n) by 2^(e - 4) more: the largest |x| lands in
// [2^14, 2^15) (its odd-nibble copy in [2^10, 2^11)), so every staged value is an fp16 normal unless it lies 2^-29 below that maximum, and
// the scaling is exact.  The step sums of x and the group epilogue's fp32 arithmetic scale with it (exactly: powers of two), and the
// column totals are multiplied by 2^-e once before they leave.
struct XScale {
    float even, odd, inv;  // 2^e, 2^(e - 4), 2^-e
};
// from an upper bound m of the range's largest |x| (a tighter bound keeps more of the range exact; the staged values cannot overflow, as
// e >= -1 and every |x| <= 65504)
__device__ __forceinline__ XScale x_scale(float m) {
    const int e = min(max(14 - ((int)((__float_as_uint(m) >> 23) & 255u) - 127), -1), 38);  // m = 0: any e (38)
    return XScale{__int_as_float((127 + e) << 23), __int_as_float((123 + e) << 23), __int_as_float((127 - e) << 23)};
}
// running max of the fp16 magnitudes of the four half2 words of v (per 16-bit lane)
__device__ __forceinline__ uint32_t max_abs8(uint32_t m, uint4 v) {
    m = __vmaxu2(m, v.x & 0x7fff7fffu);
    m = __vmaxu2(m, v.y & 0x7fff7fffu);
    m = __vmaxu2(m, v.z & 0x7fff7fffu);
    return __vmaxu2(m, v.w & 0x7fff7fffu);
}
__device__ __forceinline__ uint32_t scale_h2(uint32_t w, float f) {
    const float2 v = __half22float2(u32_as_h2(w));
    return h2_as_u32(__floats2half2_rn(v.x * f, v.y * f));
}
// one permuted run of 8 scaled for the tensor pipe
__device__ __forceinline__ uint4 scale_run(uint4 v, const XScale& sc) {
    return make_uint4(scale_h2(v.x, sc.even), scale_h2(v.y, sc.odd), scale_h2(v.z, sc.even), scale_h2(v.w, sc.odd));
}

// sum of the EFFECTIVE x of one staged run of 8 (what the tensor pipe will multiply the nibbles with)
__device__ __forceinline__ float run_sum(uint4 v) {
    const float2 a = __half22float2(u32_as_h2(v.x)), b = __half22float2(u32_as_h2(v.y)), c = __half22float2(u32_as_h2(v.z)), d = __half22float2(u32_as_h2(v.w));
    const float even = (a.x + a.y) + (c.x + c.y), odd = (b.x + b.y) + (d.x + d.y);
    return fmaf(odd, 16.0f, even);
}
// scales the nsteps k-steps staged at xs in place and sets xsum[s] = the sum over the 32 k of step s of the scaled x (4 runs of 8)
__device__ __forceinline__ void scale_and_sum(__half* xs, int nsteps, float* xsum, const XScale& sc, int tid, int nthreads) {
    const int n4 = nsteps * 4;
    for (int base = 0; base < n4; base += nthreads) {
        const int idx = base + tid;
        float v = 0.f;
        if (idx < n4) {
            uint4* run = reinterpret_cast<uint4*>(xs + idx * 8);
            const uint4 r = scale_run(*run, sc);
            *run = r;
            v = run_sum(r);
        }
        v += __shfl_xor_sync(0xffffffffu, v, 1);
        v += __shfl_xor_sync(0xffffffffu, v, 2);
        if (idx < n4 && (idx & 3) == 0) xsum[idx >> 2] = v;
    }
}

// x = rmsnorm(src [+ fp16(acc)]) for the whole row (K = H), staged in xs (matvec layout and scaled, *xinv = 2^-e, or natural order if
// PLAIN) with its per-step sums in xsum; the updated residual stream (src + fp16(acc)) is written to resid_out by slices.
// All 512 consumer threads.  ACT: the matvec's packed rows were regrouped by the host: position k' holds feature perm[k'].
// The staging scale comes from max|x| rstd max|w| >= max|x w rstd|, reduced with the sum of squares (no extra barrier).
template <bool ACT, bool PLAIN>
__device__ void stage_norm(const MegaParams& p, const __half* src, const float* acc, const __half* norm_w, __half* resid_out, __half* xs, float* xsum,
                           float* xinv, __half* tmp, float* red_s, const int32_t* perm) {
    const int H = p.H, tid = threadIdx.x, nch = H / 8;
    float ss = 0.f;
    uint32_t xm = 0, wm = 0;  // largest fp16 magnitudes of x and of the norm weights (two 16-bit lanes each)
    uint4 nwv[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        const int c = tid + i * kConsumers;
        nwv[i] = make_uint4(0, 0, 0, 0);
        if (c < nch) {
            nwv[i] = *reinterpret_cast<const uint4*>(norm_w + c * 8);  // same round trip as src / acc
            const uint4 v = ld_cg_u4(src + c * 8);  // written by other CTAs (residual slices): L2, not this SM's L1
            uint32_t xv[4] = {v.x, v.y, v.z, v.w};
            if (acc != nullptr) {
                const float4 a0 = ld_cg4(acc + c * 8), a1 = ld_cg4(acc + c * 8 + 4);
                const float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
#pragma unroll
                for (int j = 0; j < 4; ++j)  // residual + fp16(linear output): an fp16 add, as in HF's decoder layer
                    xv[j] = h2_as_u32(__hadd2(u32_as_h2(xv[j]), __floats2half2_rn(av[2 * j], av[2 * j + 1])));
            }
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const float2 f = __half22float2(u32_as_h2(xv[j]));
                ss = fmaf(f.x, f.x, ss);
                ss = fmaf(f.y, f.y, ss);
            }
            const uint4 xq = make_uint4(xv[0], xv[1], xv[2], xv[3]);
            *reinterpret_cast<uint4*>(tmp + c * 8) = xq;
            xm = max_abs8(xm, xq);
            wm = max_abs8(wm, nwv[i]);
        }
    }
    uint32_t m = max(xm & 0xffffu, xm >> 16) | (max(wm & 0xffffu, wm >> 16) << 16);
    const float tot = block_sum(ss, m, red_s);  // its barriers also publish tmp
    const float rstd = rms_rstd(tot, H, p.eps);
    XScale sc{1.f, 1.f, 1.f};
    if constexpr (!PLAIN) {
        sc = x_scale(__half2float(__ushort_as_half((unsigned short)(m & 0xffffu))) * rstd * __half2float(__ushort_as_half((unsigned short)(m >> 16))) * 1.001f);
        if (tid == 0) *xinv = sc.inv;
    }
    if (resid_out != nullptr) {
        const int per = (nch + gridDim.x - 1) / gridDim.x;
        const int c = blockIdx.x * per + tid;
        if (tid < per && c < nch) *reinterpret_cast<uint4*>(resid_out + c * 8) = *reinterpret_cast<const uint4*>(tmp + c * 8);
    }
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        const int c = tid + i * kConsumers;
        if (c < nch) {
            float xf[8];
            bool gathered = false;
            if constexpr (ACT) {
                if (perm != nullptr) {  // norm_w is given in regrouped order (gptq_b200.h); the gather itself reads shared memory
                    const ::int4 p0 = *reinterpret_cast<const ::int4*>(perm + c * 8), p1 = *reinterpret_cast<const ::int4*>(perm + c * 8 + 4);
                    const int k[8] = {p0.x, p0.y, p0.z, p0.w, p1.x, p1.y, p1.z, p1.w};
#pragma unroll
                    for (int j = 0; j < 8; ++j) xf[j] = __half2float(tmp[k[j]]);
                    gathered = true;
                }
            }
            if (!gathered) {
                const uint4 v = *reinterpret_cast<const uint4*>(tmp + c * 8);
                const uint32_t xv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const float2 f = __half22float2(u32_as_h2(xv[j]));
                    xf[2 * j] = f.x;
                    xf[2 * j + 1] = f.y;
                }
            }
            const uint32_t wv[4] = {nwv[i].x, nwv[i].y, nwv[i].z, nwv[i].w};
            uint32_t o[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const float2 wf = __half22float2(u32_as_h2(wv[j]));
                o[j] = h2_as_u32(rms_apply2(make_float2(xf[2 * j], xf[2 * j + 1]), rstd, wf));
            }
            if constexpr (PLAIN) {
                *reinterpret_cast<uint4*>(xs + c * 8) = make_uint4(o[0], o[1], o[2], o[3]);
            } else {
                const uint4 pv = scale_run(perm8(o[0], o[1], o[2], o[3]), sc);
                *reinterpret_cast<uint4*>(xs + c * 8) = pv;
                // per-step sums of the staged x: the 4 runs of a k-step sit in 4 consecutive lanes (c < nch is uniform per warp)
                float v = run_sum(pv);
                v += __shfl_xor_sync(0xffffffffu, v, 1);
                v += __shfl_xor_sync(0xffffffffu, v, 2);
                if ((c & 3) == 0) xsum[c >> 2] = v;
            }
        }
    }
    cta_sync();
}

// ---- matvec consumer ---------------------------------------------------------------------------------------------------
__device__ __forceinline__ void mma_16816_z(float (&d)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%10,%10,%10,%10};"
                 : "=f"(d[0]), "=f"(d[1]), "=f"(d[2]), "=f"(d[3])
                 : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1), "f"(0.f));
}

// the four A registers (k-pairs (0,4), (1,5), (2,6), (3,7)) of one packed word, masked in place: fp16 subnormals n * 2^-24 and 16 n * 2^-24
__device__ __forceinline__ void nibble_regs(uint32_t q, uint32_t (&a)[4]) {
    const uint32_t q8 = q >> 8;  // (as IMAD.HI on the FMA pipe it is far slower: tools/ubench/loop.cu, 1102 vs 817 cycles per stage)
    a[0] = q & 0x000f000fu;
    a[1] = q & 0x00f000f0u;
    a[2] = q8 & 0x000f000fu;
    a[3] = q8 & 0x00f000f0u;
}

// one k-step (4 packed words of this lane = columns 4g..4g+3 x 8 k) into the two accumulators
template <bool FIRST>
__device__ __forceinline__ void step_mma(const uint4& q, const uint4& xf, float (&acc0)[4], float (&acc1)[4]) {
    uint32_t c0[4], c1[4], c2[4], c3[4];
    nibble_regs(q.x, c0);
    nibble_regs(q.y, c1);
    nibble_regs(q.z, c2);
    nibble_regs(q.w, c3);
    if (FIRST) {
        mma_16816_z(acc0, c0[0], c1[0], c0[1], c1[1], xf.x, xf.y);
        mma_16816_z(acc1, c2[0], c3[0], c2[1], c3[1], xf.x, xf.y);
    } else {
        mma_16816(acc0, c0[0], c1[0], c0[1], c1[1], xf.x, xf.y);
        mma_16816(acc1, c2[0], c3[0], c2[1], c3[1], xf.x, xf.y);
    }
    mma_16816(acc0, c0[2], c1[2], c0[3], c1[3], xf.z, xf.w);
    mma_16816(acc1, c2[2], c3[2], c2[3], c3[3], xf.z, xf.w);
}

enum XMode { X_FULL = 0, X_ATTN = 1, X_SWIGLU = 2 };

struct TeamCtx {
    int team, wt, lane, ttid;  // team, warp in team, lane, thread in team
    unsigned T, nb;            // global team index / number of teams
    __half* xseg;              // this team's half of the xs buffer (per-segment inputs of O and D)
    float* xsum_seg;
    float* xinv_seg;           // [batch]: 2^-e of the staged segment (XScale)
    uint32_t* xmax;            // [batch]: largest fp16 magnitude of the staged segment
    uint8_t* scratch;          // kTeamScratch bytes
};

// softmax merge of dimension d of the partial records of teams [ht.first, ht.first + ht.count), NB records per round trip
template <int NB>
__device__ __forceinline__ float merge_records(const MegaParams& p, const HeadTeams& ht, int d) {
    float M = -INFINITY, Ls = 0.f, O = 0.f;
#pragma unroll 1
    for (int ib = 0; ib < ht.count; ib += NB) {
        float mv[NB], lv[NB], ov[NB];
#pragma unroll
        for (int i = 0; i < NB; ++i) {  // all loads of the batch are in flight together
            const bool on = ib + i < ht.count;
            const float* rc = p.part + (size_t)(ht.first + (on ? ib + i : 0)) * kRec;
            const float m = ld_cg(rc), l = ld_cg(rc + 1), o = ld_cg(rc + 4 + d);
            mv[i] = on ? m : -INFINITY;
            lv[i] = on ? l : 0.f;
            ov[i] = on ? o : 0.f;
        }
        float Mb = M;
#pragma unroll
        for (int i = 0; i < NB; ++i) Mb = fmaxf(Mb, mv[i]);
        const float w0 = (M == -INFINITY) ? 0.f : expf(M - Mb);
        Ls *= w0;
        O *= w0;
#pragma unroll
        for (int i = 0; i < NB; ++i) {
            const float w = (mv[i] == -INFINITY) ? 0.f : expf(mv[i] - Mb);
            Ls = fmaf(lv[i], w, Ls);
            O = fmaf(ov[i], w, O);
        }
        M = Mb;
    }
    return O / Ls;
}

// Input of o_proj (XMODE == X_ATTN) / down_proj (X_SWIGLU) for the team's WHOLE unit range [u0, u1) (units = k-steps of 32, numbered
// slab-major; the range wraps at most once from the end of one slab's k-range to the start of the next): staged once, in unit order,
// into the team's half of the xs buffer, then scaled (XScale, per sequence) with its per-step sums.  One L2 round trip for the common shapes.
// BATCH: sequence s of the range goes to xseg + s * xs_stride, its step sums to xsum_seg + s * H / 32.
template <int XMODE, bool ACT, bool BATCH>
__device__ void stage_range(const MegaParams& p, const TeamCtx& tc, int nk, int u0, int u1, const int32_t* perm) {
    const int nun = u1 - u0, nfeat = nun * 32;
    const int nbat = BATCH ? p.batch : 1;
    const int ksb = u0 % nk;  // k-step of the first unit
    auto k_of = [&](int e) {  // feature e of the range -> input index k
        int ks = ksb + (e >> 5);
        if (ks >= nk) ks -= nk;
        return ks * 32 + (e & 31);
    };
    if (tc.ttid < nbat) tc.xmax[tc.ttid] = 0;
    team_sync(tc.team);  // previous readers of xseg (and of xmax) are done
    if constexpr (XMODE == X_SWIGLU) {  // h = fp16(silu(acc_gate) * acc_up)  (quant/fused_mlp.py:163-165)
        for (int c = tc.ttid; c < nun * 4 * nbat; c += kTeamThreads) {
            int s = 0, cs = c;  // sequence, 8-feature chunk of the range
            if constexpr (BATCH) {
                s = c / (nun * 4);
                cs = c - s * (nun * 4);
            }
            const int k = k_of(cs * 8);
            const float* ag = p.acc_g + (size_t)s * p.I + k;
            const float* au = p.acc_u + (size_t)s * p.I + k;
            const float4 g0 = ld_cg4(ag), g1 = ld_cg4(ag + 4);
            const float4 a0 = ld_cg4(au), a1 = ld_cg4(au + 4);
            const uint32_t o0 = h2_as_u32(__floats2half2_rn(swiglu(g0.x, a0.x), swiglu(g0.y, a0.y)));
            const uint32_t o1 = h2_as_u32(__floats2half2_rn(swiglu(g0.z, a0.z), swiglu(g0.w, a0.w)));
            const uint32_t o2 = h2_as_u32(__floats2half2_rn(swiglu(g1.x, a1.x), swiglu(g1.y, a1.y)));
            const uint32_t o3 = h2_as_u32(__floats2half2_rn(swiglu(g1.z, a1.z), swiglu(g1.w, a1.w)));
            const uint4 pv = perm8(o0, o1, o2, o3);
            *reinterpret_cast<uint4*>(tc.xseg + (size_t)s * p.xs_stride + cs * 8) = pv;
            const uint32_t m = max_abs8(0, pv);
            atomicMax(tc.xmax + s, max(m & 0xffffu, m >> 16));
        }
    } else {
        // attention output: softmax-merge of the partial records (m, l, o[128]) of the head's teams (head_teams: contiguous, one
        // record each; BATCH: the head's teams inside the sequence's teams, seq_teams).
        constexpr int kBatch = 12;  // records fetched per round trip (a 7B head has 9 or 10 teams)
        uint32_t vmax = 0;  // largest fp16 magnitude this thread put (per sequence: flushed into xmax)
        auto put = [&](__half* xseg, int e, float v) {
            const __half hv = __float2half_rn(v);
            xseg[(e & ~7) + perm_pos(e & 7)] = hv;
            vmax = max(vmax, (uint32_t)(__half_as_ushort(hv) & 0x7fffu));
        };
        bool fast = false;
        if constexpr (!BATCH) {
            // heads of the range: [hA0, hA1] before the wrap, [0, hB1] after it
            const int nA = min(nun, nk - ksb);
            const int hA0 = (ksb * 32) / kHD, hA1 = ((ksb + nA) * 32 - 1) / kHD;
            const int nslotA = hA1 - hA0 + 1, nslotB = (nun > nA) ? ((nun - nA) * 32 - 1) / kHD + 1 : 0;
            fast = (nslotA + nslotB <= kTeamWarps) && (nun <= nk) && ((int)tc.nb / p.n_heads + 1 <= kBatch);
            if constexpr (ACT) fast = fast && (perm == nullptr);
            if (fast) {
                // ONE round trip (per 256 features): every thread fetches the o values of its feature from all records of its head while
                // warp w fetches (m, l) of the w-th head of the range and turns them into merge weights exp(m - M) / L.
                float* wts = reinterpret_cast<float*>(tc.scratch);  // [kTeamWarps][kBatch]
                float ov[kBatch];
                int slot = 0;
                auto fetch = [&](int e) {
                    const bool active = e < nfeat;
                    const int k = k_of(active ? e : 0);
                    const int head = k / kHD, d = k - head * kHD;
                    slot = ((e >> 5) < nA) ? head - hA0 : nslotA + head;
                    const HeadTeams ht = head_teams(head, p.n_heads, tc.nb);
#pragma unroll
                    for (int i = 0; i < kBatch; ++i) ov[i] = (active && i < ht.count) ? ld_cg(p.part + (size_t)(ht.first + i) * kRec + 4 + d) : 0.f;
                };
                auto emit = [&](int e) {
                    if (e < nfeat) {
                        float O = 0.f;
#pragma unroll
                        for (int i = 0; i < kBatch; ++i) O = fmaf(wts[slot * kBatch + i], ov[i], O);
                        put(tc.xseg, e, O);
                    }
                };
                fetch(tc.ttid);
                if (tc.wt < nslotA + nslotB) {
                    const int lane = tc.lane;
                    const int head = tc.wt < nslotA ? hA0 + tc.wt : tc.wt - nslotA;
                    const HeadTeams ht = head_teams(head, p.n_heads, tc.nb);
                    float m = -INFINITY, l = 0.f;
                    if (lane < ht.count) {
                        m = ld_cg(p.part + (size_t)(ht.first + lane) * kRec);
                        l = ld_cg(p.part + (size_t)(ht.first + lane) * kRec + 1);
                    }
                    float M = m;
#pragma unroll
                    for (int o = 8; o > 0; o >>= 1) M = fmaxf(M, __shfl_xor_sync(0xffffffffu, M, o));  // lanes 0..15 hold the batch
                    M = __shfl_sync(0xffffffffu, M, 0);
                    const float w = (m == -INFINITY) ? 0.f : expf(m - M);
                    float L = l * w;
#pragma unroll
                    for (int o = 8; o > 0; o >>= 1) L += __shfl_xor_sync(0xffffffffu, L, o);
                    L = __shfl_sync(0xffffffffu, L, 0);
                    if (lane < kBatch) wts[tc.wt * kBatch + lane] = w / L;
                }
                team_sync(tc.team);
                emit(tc.ttid);
                for (int e = tc.ttid + kTeamThreads; e - tc.ttid < nfeat; e += kTeamThreads) {  // wider ranges (13B, 65B): further round trips
                    fetch(e);
                    emit(e);
                }
                atomicMax(tc.xmax, vmax);
            }
        }
        if (!fast) {
            for (int s = 0; s < nbat; ++s) {
                HeadTeams st{0, (int)tc.nb};
                if constexpr (BATCH) st = seq_teams(p, s, tc.nb);
                for (int e = tc.ttid; e < nfeat; e += kTeamThreads) {
                    int k = k_of(e);
                    if constexpr (ACT) {
                        if (perm != nullptr) k = perm[k];  // regrouped rows: position k' of the matvec input is attention feature perm[k']
                    }
                    const int head = k / kHD, d = k - head * kHD;
                    HeadTeams ht = head_teams(head, p.n_heads, st.count);
                    ht.first += st.first;
                    put(tc.xseg + (size_t)s * p.xs_stride, e, merge_records<kBatch>(p, ht, d));
                }
                atomicMax(tc.xmax + s, vmax);
                vmax = 0;
            }
        }
    }
    team_sync(tc.team);
    for (int s = 0; s < nbat; ++s) {
        const XScale sc = x_scale(__half2float(__ushort_as_half((unsigned short)tc.xmax[s])));
        if (tc.ttid == 0) tc.xinv_seg[s] = sc.inv;
        scale_and_sum(tc.xseg + (size_t)s * p.xs_stride, nun, tc.xsum_seg + s * (p.H / 32), sc, tc.ttid, kTeamThreads);
    }
    team_sync(tc.team);
}

// One matvec op for this team: consume the stages of its unit range from the ring, RED the results.
// NM = 2: gate|up as one virtual matrix (out0 = gate accumulators, out1 = up accumulators).
// BATCH: B operand column g is sequence min(g, B - 1); lane (g, t) finishes columns 4 cg .. 4 cg + 3 of sequences 2t and 2t + 1 (the C
// fragment columns), and out0 / out1 are [B][N].
template <int NM, int XMODE, bool ACT = false, bool BATCH = false>
__device__ void run_matvec(const MegaParams& p, ConsRing& ring, const TeamCtx& tc, int gs_steps, int K, int N, float* out0, float* out1, const __half* xs_full,
                           const float* xsum_full, const float* xinv_full, const int32_t* perm = nullptr, float* const* peers = nullptr) {
    const int lane = tc.lane, g = lane >> 2, t = lane & 3;
    const int nk = K / 32, nslab = N / kSlabCols;
    int u, u_end;
    team_range(tc.T, (unsigned)(NM * nslab) * nk, tc.nb, u, u_end);
    // MMA row g of this lane carries the 4 columns of 16-byte unit cg of the warp's 128-byte chunk; cg is chosen so that the
    // swizzled units (unit ^ row) of a quarter-warp (g in {2q, 2q+1}, t = 0..3) are 8 distinct bank groups
    const int cg = (g >> 1) | ((g & 1) << 2);
    const int col_l = 4 * cg + t;  // the column (of the warp's 32) this lane finishes in the epilogue
    // 16-row box [chunk][row][128 B]: row 4j + t of chunk wt, unit cg ^ ((4j + t) & 7)
    const uint32_t lane_a0 = (uint32_t)((tc.wt * 16 + t) * 128 + ((cg ^ t) * 16));       // even k-steps of the stage
    const uint32_t lane_a1 = (uint32_t)((tc.wt * 16 + t) * 128 + ((cg ^ t ^ 4) * 16));   // odd k-steps
    // 4-row boxes (one per k-step, 4 KB apart) [chunk][row][128 B]: line wt * 4 + t
    const uint32_t lane_b = (uint32_t)((tc.wt * 4 + t) * 128 + ((cg ^ (4 * (tc.wt & 1) + t)) * 16));
    const uint32_t lane_s = (uint32_t)(kScaleOff + (tc.wt * 32 + col_l) * 2);      // scale of its column
    const uint32_t lane_z = (uint32_t)(kZeroOff + (tc.wt * 4 + (cg >> 1)) * 4);    // the qzeros word holding its zero
    const int zshift = (cg & 1) * 16 + t * 4;
    const float unit = 16777216.0f;  // the accumulators are in units of 2^-24
    // BATCH: lane group g feeds sequence min(g, B - 1) to the tensor pipe and the lane finishes sequences 2t and 2t + 1 (clamped: lanes
    // past the batch read sequence B - 1 and drop their results); xsum_hi = offset of the step sums of sequence 2t + 1 from those of 2t
    const int B = p.batch;
    const int xsum_hi = BATCH ? (min(2 * t + 1, B - 1) - min(2 * t, B - 1)) * (p.H / 32) : 0;
    const int u_begin = u;
    if constexpr (XMODE != X_FULL) {
        if (u < u_end) {
#ifdef GPTQ_TRACE
            const long long stg0 = clock64();
#endif
            stage_range<XMODE, ACT, BATCH>(p, tc, nk, u, u_end, perm);
#ifdef GPTQ_TRACE
            if (g_mega_trace != nullptr && threadIdx.x == 0) g_mega_trace[blockIdx.x * 64 + 36 + XMODE] += (unsigned long long)(clock64() - stg0);
#endif
        }
    }

#pragma unroll 1
    while (u < u_end) {
        const int slab_v = u / nk;
        const int ks0 = u - slab_v * nk;
        const int nseg = min(nk - ks0, u_end - u);
        const int mi = (NM > 1 && slab_v >= nslab) ? 1 : 0;
        float* outp = (mi ? out1 : out0) + (slab_v - mi * nslab) * kSlabCols + tc.wt * 32 + col_l;

        uint32_t xaddr;
        const float* xsum;
        if constexpr (XMODE == X_FULL) {
            xaddr = smem_u32(xs_full) + (ks0 * 32 + t * 8) * 2;
            xsum = xsum_full + ks0;
        } else {
            xaddr = smem_u32(tc.xseg) + ((u - u_begin) * 32 + t * 8) * 2;
            xsum = tc.xsum_seg + (u - u_begin);
        }
        float totb[4][2];  // BATCH: [column 4 cg + i][sequence 2t, 2t + 1]
        if constexpr (BATCH) {
            xaddr += (uint32_t)(min(g, B - 1) * p.xs_stride * 2);
            xsum += min(2 * t, B - 1) * (p.H / 32);
#pragma unroll
            for (int i = 0; i < 4; ++i) totb[i][0] = totb[i][1] = 0.f;
        }

        float tot = 0.f;  // lane (g, t) finishes column 4g + t of the warp's stripe
        int left = nseg, gpos = ks0 % gs_steps;
#pragma unroll 1
        while (left > 0) {
            const int n = stage_steps(gpos, gs_steps, left);
            const uint32_t st = cons_wait(ring);
            float acc0[4], acc1[4];
            float xs4, xs4b;  // xs4b: sum of x of sequence 2t + 1 (BATCH)
            if (n == kStageSteps) {
                uint4 q[4], xf[4];
#pragma unroll
                for (int j = 0; j < 4; ++j) q[j] = lds128(st + j * 512 + ((j & 1) ? lane_a1 : lane_a0));
#pragma unroll
                for (int j = 0; j < 4; ++j) xf[j] = lds128(xaddr + j * 64);
                step_mma<true>(q[0], xf[0], acc0, acc1);
                step_mma<false>(q[1], xf[1], acc0, acc1);
                step_mma<false>(q[2], xf[2], acc0, acc1);
                step_mma<false>(q[3], xf[3], acc0, acc1);
                xs4 = (xsum[0] + xsum[1]) + (xsum[2] + xsum[3]);
                if constexpr (BATCH) xs4b = (xsum[xsum_hi] + xsum[xsum_hi + 1]) + (xsum[xsum_hi + 2] + xsum[xsum_hi + 3]);
            } else {
                {
                    const uint4 q = lds128(st + lane_b), xf = lds128(xaddr);
                    step_mma<true>(q, xf, acc0, acc1);
                    xs4 = xsum[0];
                    if constexpr (BATCH) xs4b = xsum[xsum_hi];
                }
#pragma unroll 1
                for (int j = 1; j < n; ++j) {
                    const uint4 q = lds128(st + lane_b + j * kStepBytes), xf = lds128(xaddr + j * 64);
                    step_mma<false>(q, xf, acc0, acc1);
                    xs4 += xsum[j];
                    if constexpr (BATCH) xs4b += xsum[xsum_hi + j];
                }
            }
            // group epilogue: tot += s * (acc * unit - z * sum(x))   (z = stored zero + 1, quant/quant_linear.py:120-121).
            if constexpr (BATCH) {
                // acc0[0..1] / acc0[2..3] / acc1[0..1] / acc1[2..3]: columns 4 cg + 0 / 1 / 2 / 3 of sequences 2t, 2t + 1
                uint32_t s01, s23, zw;
                asm volatile("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(s01), "=r"(s23) : "r"(st + (uint32_t)(kScaleOff + (tc.wt * 32 + 4 * cg) * 2)));
                asm volatile("ld.shared.u32 %0, [%1];" : "=r"(zw) : "r"(st + lane_z));
                const float2 sa = __half22float2(u32_as_h2(s01)), sb = __half22float2(u32_as_h2(s23));
                const float sc[4] = {sa.x, sa.y, sb.x, sb.y};
                const float av[4][2] = {{acc0[0], acc0[1]}, {acc0[2], acc0[3]}, {acc1[0], acc1[1]}, {acc1[2], acc1[3]}};
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const float z = (float)(((zw >> ((cg & 1) * 16 + 4 * i)) & 15u) + 1u);
                    totb[i][0] = fmaf(sc[i], fmaf(av[i][0], unit, -z * xs4), totb[i][0]);
                    totb[i][1] = fmaf(sc[i], fmaf(av[i][1], unit, -z * xs4b), totb[i][1]);
                }
            } else {
                // All four t lanes hold the same four column sums (the batch columns of B are copies): lane t finishes column 4g + t.
                uint32_t sh, zw;
                asm volatile("ld.shared.u16 %0, [%1];" : "=r"(sh) : "r"(st + lane_s));
                asm volatile("ld.shared.u32 %0, [%1];" : "=r"(zw) : "r"(st + lane_z));
                const float a = (t & 2) ? ((t & 1) ? acc1[2] : acc1[0]) : ((t & 1) ? acc0[2] : acc0[0]);
                const float z = (float)(((zw >> zshift) & 15u) + 1u);
                tot = fmaf(__half2float(__ushort_as_half((unsigned short)sh)), fmaf(a, unit, -z * xs4), tot);
            }
            cons_release(ring, lane);
            xaddr += n * 64;
            xsum += n;
            left -= n;
            gpos += n;
            if (gpos == gs_steps) gpos = 0;
        }
        // the totals are in units of the staged x: times 2^-e (exact)
        const float* xinv = XMODE == X_FULL ? xinv_full : tc.xinv_seg;  // [sequence]
        if constexpr (BATCH) {  // the four columns of each of the lane's sequences: one 16-byte vector RED
            float* outq = (mi ? out1 : out0) + (slab_v - mi * nslab) * kSlabCols + tc.wt * 32 + 4 * cg;
#pragma unroll
            for (int j = 0; j < 2; ++j) {
                const float inv = xinv[min(2 * t + j, B - 1)];
                if (2 * t + j < B)
                    asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(outq + (size_t)(2 * t + j) * N), "f"(totb[0][j] * inv), "f"(totb[1][j] * inv),
                                 "f"(totb[2][j] * inv), "f"(totb[3][j] * inv)
                                 : "memory");
            }
        } else {
            tot *= xinv[0];
            if (peers == nullptr) {
                asm volatile("red.global.add.f32 [%0], %1;" ::"l"(outp), "f"(tot) : "memory");  // the warp's 32 columns: one 128-byte line
            } else {  // tensor parallelism, direct mode: the partial sum goes into out0's counterpart on every rank
                const size_t off = (size_t)(outp - out0);
                for (int q = 0; q < p.tp_size; ++q) asm volatile("red.relaxed.sys.global.add.f32 [%0], %1;" ::"l"(peers[q] + off), "f"(tot) : "memory");
            }
        }
        u += nseg;
    }
}

// ---- attention ----------------------------------------------------------------------------------------------------------
// Work units (head, 32 keys); a team serves one head (attn_range); one unit = one ring stage (K rows, V rows).  The team writes
// one partial record (m, l, o[128]) to p.part[T].
// BATCH: the team serves one (sequence, head) pair (attn_work), at that sequence's position, in that sequence's cache slot.
template <bool BATCH>
__device__ void run_attention(const MegaParams& p, ConsRing& ring, const TeamCtx& tc, int layer) {
    int pos, Tlen, head, b0, b_end;
    const int seq = attn_work<BATCH>(p, tc.T, tc.nb, pos, Tlen, head, b0, b_end);
    float* red_o = reinterpret_cast<float*>(tc.scratch);                 // [8][128]  end of a segment
    float* red_ml = reinterpret_cast<float*>(tc.scratch + 4096);         // [8][2]
    float* q_s = reinterpret_cast<float*>(tc.scratch);                   // [128]     start of a segment (aliases red_o)
    __half* knew = reinterpret_cast<__half*>(tc.scratch + 512);          // [128]
    __half* vnew = knew + kHD;                                          // [128]
    const int ttid = tc.ttid, lane = tc.lane, grp = ttid >> 3, j = ttid & 7;  // 32 groups of 8 lanes: group = key, lane j owns dims 8j..8j+7 and 64+8j..64+8j+7
    const int ub_new = pos / kKeysPerUnit;  // the unit that holds this step's key
    __half* kc_l = p.k_cache + layer * p.layer_stride;
    __half* vc_l = p.v_cache + layer * p.layer_stride;
    float* rec = p.part + (size_t)tc.T * kRec;
    if (b0 >= b_end) {  // no unit for this team (short context): a neutral record keeps the merge uniform
        if (ttid < kHD) rec[4 + ttid] = 0.f;
        if (ttid == 0) {
            rec[0] = -INFINITY;
            rec[1] = 0.f;
        }
        return;
    }
    {
        const int nseg = b_end - b0;
        const bool owns_new = (ub_new >= b0 && ub_new < b_end);
        team_sync(tc.team);  // scratch reuse
        if (ttid < kHD) {
            const int i = ttid & 63;
            const bool hi = ttid >= 64;
            const float c = ld_cg(p.rope_cs + seq * kHD + i), s = ld_cg(p.rope_cs + seq * kHD + 64 + i);
            const float* aq = p.acc_qkv + (size_t)seq * 3 * p.Hq + head * kHD;
            const float qx = __half2float(__float2half_rn(ld_cg(aq + i))), qy = __half2float(__float2half_rn(ld_cg(aq + i + 64)));  // the qkv projection output is fp16
            const float qr = hi ? rope_y(qx, qy, c, s) : rope_x(qx, qy, c, s);
            q_s[ttid] = __half2float(__float2half_rn(qr));
            if (owns_new) {  // this segment owns the new key/value: RoPE(k), append both to the cache
                const float* ak = aq + p.Hq;
                const float* av = aq + 2 * p.Hq;
                const float kx = __half2float(__float2half_rn(ld_cg(ak + i))), ky = __half2float(__float2half_rn(ld_cg(ak + i + 64)));
                const float kr = hi ? rope_y(kx, ky, c, s) : rope_x(kx, ky, c, s);
                const __half kh = __float2half_rn(kr), vh = __float2half_rn(ld_cg(av + ttid));
                knew[ttid] = kh;
                vnew[ttid] = vh;
                const size_t off = ((size_t)(seq * p.n_heads + head) * p.max_seq + pos) * kHD + ttid;
                kc_l[off] = kh;
                vc_l[off] = vh;
            }
        }
        team_sync(tc.team);
        float qr[16];
#pragma unroll
        for (int d = 0; d < 8; ++d) {
            qr[d] = q_s[8 * j + d];
            qr[8 + d] = q_s[64 + 8 * j + d];
        }
        float mloc = -INFINITY, lloc = 0.f, o[16];
#pragma unroll
        for (int d = 0; d < 16; ++d) o[d] = 0.f;
#pragma unroll 1
        for (int b = b0; b < b0 + nseg; ++b) {
            const uint32_t st = cons_wait(ring);
            if (b == ub_new) {
                // the stage was fetched before this step's key/value existed: patch its row from the fresh values
                team_sync(tc.team);  // (uniform per team) every warp has seen the stage land
                const int row = pos - b * kKeysPerUnit;
                if (ttid < 16) {
                    sts128(st + row * 256 + ttid * 16, reinterpret_cast<const uint4*>(knew)[ttid]);
                    fence_proxy_async_smem();  // generic-proxy writes into a stage the TMA unit will overwrite later
                } else if (ttid < 32) {
                    sts128(st + kVOff + row * 256 + (ttid - 16) * 16, reinterpret_cast<const uint4*>(vnew)[ttid - 16]);
                    fence_proxy_async_smem();
                }
                team_sync(tc.team);
            }
            const int key = b * kKeysPerUnit + grp;
            const bool valid = key < Tlen;
            float s = 0.f;
            if (valid) {
                const uint4 k0 = lds128(st + grp * 256 + j * 16), k1 = lds128(st + grp * 256 + 128 + j * 16);
                const uint32_t w[8] = {k0.x, k0.y, k0.z, k0.w, k1.x, k1.y, k1.z, k1.w};
#pragma unroll
                for (int e = 0; e < 8; ++e) {
                    const float2 f = __half22float2(u32_as_h2(w[e]));
                    s = fmaf(qr[2 * e], f.x, s);
                    s = fmaf(qr[2 * e + 1], f.y, s);
                }
            }
            s += __shfl_xor_sync(0xffffffffu, s, 1);
            s += __shfl_xor_sync(0xffffffffu, s, 2);
            s += __shfl_xor_sync(0xffffffffu, s, 4);
            if (valid) {
                s *= p.scale;
                const float mnew = fmaxf(mloc, s);
                const float alpha = (mloc == -INFINITY) ? 0.f : expf(mloc - mnew);
                const float pw = expf(s - mnew);
                lloc = fmaf(lloc, alpha, pw);
                const uint4 v0 = lds128(st + kVOff + grp * 256 + j * 16), v1 = lds128(st + kVOff + grp * 256 + 128 + j * 16);
                const uint32_t w[8] = {v0.x, v0.y, v0.z, v0.w, v1.x, v1.y, v1.z, v1.w};
#pragma unroll
                for (int e = 0; e < 8; ++e) {
                    const float2 f = __half22float2(u32_as_h2(w[e]));
                    o[2 * e] = fmaf(o[2 * e], alpha, pw * f.x);
                    o[2 * e + 1] = fmaf(o[2 * e + 1], alpha, pw * f.y);
                }
                mloc = mnew;
            }
            cons_release(ring, lane);
        }
        team_sync(tc.team);  // every warp has read q_s and passed the patch: the merge buffers (which alias q_s / knew / vnew) may be written
        // merge the 4 key groups of the warp (lanes xor 8, 16), then the 8 warps through shared memory
#pragma unroll
        for (int sh = 8; sh <= 16; sh <<= 1) {
            const float mo = __shfl_xor_sync(0xffffffffu, mloc, sh), lo = __shfl_xor_sync(0xffffffffu, lloc, sh);
            const float mn = fmaxf(mloc, mo);
            const float wa = (mloc == -INFINITY) ? 0.f : expf(mloc - mn), wb = (mo == -INFINITY) ? 0.f : expf(mo - mn);
            lloc = lloc * wa + lo * wb;
#pragma unroll
            for (int d = 0; d < 16; ++d) {
                const float oo = __shfl_xor_sync(0xffffffffu, o[d], sh);
                o[d] = o[d] * wa + oo * wb;
            }
            mloc = mn;
        }
        if (lane < 8) {
            if (lane == 0) {
                red_ml[tc.wt * 2] = mloc;
                red_ml[tc.wt * 2 + 1] = lloc;
            }
#pragma unroll
            for (int d = 0; d < 8; ++d) {
                red_o[tc.wt * kHD + 8 * lane + d] = o[d];
                red_o[tc.wt * kHD + 64 + 8 * lane + d] = o[8 + d];
            }
        }
        team_sync(tc.team);
        if (ttid < kHD) {
            float M = -INFINITY;
#pragma unroll
            for (int w = 0; w < kTeamWarps; ++w) M = fmaxf(M, red_ml[w * 2]);
            float L = 0.f, O = 0.f;
#pragma unroll
            for (int w = 0; w < kTeamWarps; ++w) {
                const float mw = red_ml[w * 2];
                const float wgt = (mw == -INFINITY) ? 0.f : expf(mw - M);
                L = fmaf(red_ml[w * 2 + 1], wgt, L);
                O = fmaf(red_o[w * kHD + ttid], wgt, O);
            }
            rec[4 + ttid] = O;
            if (ttid == 0) {
                rec[0] = M;
                rec[1] = L;
            }
        }
    }
}

// ---- lm_head: fp16 [V, H] rows through the ring, lm_rows whole rows per stage -------------------------------------------------
__device__ void run_lm_head(const MegaParams& p, ConsRing& ring, const TeamCtx& tc, const __half* xs_plain) {
    const int R = p.lm_rows, H = p.H, nch = H / 8;
    int u, u_end;
    const int nloc = p.v1 - p.v0;
    team_range(tc.T, (unsigned)((nloc + R - 1) / R), tc.nb, u, u_end);
    float* part_s = reinterpret_cast<float*>(tc.scratch);  // [2][R][8]
    // this thread's chunks of x (k = 8 * (ttid + 256 i)) stay in registers for the whole op
    float xr[4][8];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int c = tc.ttid + i * kTeamThreads;
        if (c < nch) {
            const uint4 v = *reinterpret_cast<const uint4*>(xs_plain + c * 8);
            const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const float2 f = __half22float2(u32_as_h2(w[e]));
                xr[i][2 * e] = f.x;
                xr[i][2 * e + 1] = f.y;
            }
        } else {
#pragma unroll
            for (int e = 0; e < 8; ++e) xr[i][e] = 0.f;
        }
    }
    int buf = 0;
#pragma unroll 1
    for (; u < u_end; ++u) {
        const int nrows = min(R, nloc - u * R);
        const uint32_t st = cons_wait(ring);
        float* ps = part_s + buf * (R * kTeamWarps);
#pragma unroll 1
        for (int r = 0; r < nrows; ++r) {
            float a = 0.f;
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int c = tc.ttid + i * kTeamThreads;
                if (c < nch) {
                    const uint4 wv = lds128(st + (uint32_t)(r * H * 2 + c * 16));
                    const uint32_t w[4] = {wv.x, wv.y, wv.z, wv.w};
#pragma unroll
                    for (int e = 0; e < 4; ++e) {
                        const float2 f = __half22float2(u32_as_h2(w[e]));
                        a = fmaf(f.x, xr[i][2 * e], a);
                        a = fmaf(f.y, xr[i][2 * e + 1], a);
                    }
                }
            }
            a = warp_sum(a);
            if (tc.lane == 0) ps[r * kTeamWarps + tc.wt] = a;
        }
        cons_release(ring, tc.lane);
        team_sync(tc.team);  // partials of this stage are visible; the other buffer is free again
        if (tc.ttid < nrows) {
            float a = 0.f;
#pragma unroll
            for (int w = 0; w < kTeamWarps; ++w) a += ps[tc.ttid * kTeamWarps + w];
            const __half lg = __float2half_rn(a);
            for (int q = 0; q < p.tp_size; ++q) p.logits_peer[q][(size_t)p.v0 + (size_t)u * R + tc.ttid] = lg;  // every rank holds all logits
        }
        buf ^= 1;
    }
}

// The same for a batch: x of sequence s is read from shared memory (xs + s * xs_stride, natural order) for every row, because the 32
// registers per sequence that batch 1 spends on it would not fit eight sequences; each weight chunk is loaded once for all of them.
// mega_plan keeps 2 * lm_rows * batch * kTeamWarps floats within the team scratch.
__device__ void run_lm_head_batch(const MegaParams& p, ConsRing& ring, const TeamCtx& tc, const __half* xs_plain) {
    const int R = p.lm_rows, H = p.H, nch = H / 8, B = p.batch;
    int u, u_end;
    team_range(tc.T, (unsigned)((p.V + R - 1) / R), tc.nb, u, u_end);
    float* part_s = reinterpret_cast<float*>(tc.scratch);  // [2][R][B][8]
    const uint32_t xbase = smem_u32(xs_plain);
    int buf = 0;
#pragma unroll 1
    for (; u < u_end; ++u) {
        const int nrows = min(R, p.V - u * R);
        const uint32_t st = cons_wait(ring);
        float* ps = part_s + buf * (R * B * kTeamWarps);
#pragma unroll 1
        for (int r = 0; r < nrows; ++r) {
            float a[kMaxBatch];
#pragma unroll
            for (int s = 0; s < kMaxBatch; ++s) a[s] = 0.f;
#pragma unroll 1
            for (int c = tc.ttid; c < nch; c += kTeamThreads) {
                const uint4 wv = lds128(st + (uint32_t)(r * H * 2 + c * 16));
                const uint32_t w[4] = {wv.x, wv.y, wv.z, wv.w};
#pragma unroll
                for (int s = 0; s < kMaxBatch; ++s) {
                    if (s < B) {
                        const uint4 xv = lds128(xbase + (uint32_t)((s * p.xs_stride + c * 8) * 2));
                        const uint32_t x[4] = {xv.x, xv.y, xv.z, xv.w};
#pragma unroll
                        for (int e = 0; e < 4; ++e) {
                            const float2 f = __half22float2(u32_as_h2(w[e])), xf = __half22float2(u32_as_h2(x[e]));
                            a[s] = fmaf(f.x, xf.x, a[s]);
                            a[s] = fmaf(f.y, xf.y, a[s]);
                        }
                    }
                }
            }
#pragma unroll
            for (int s = 0; s < kMaxBatch; ++s) {
                if (s < B) {
                    const float v = warp_sum(a[s]);
                    if (tc.lane == 0) ps[(r * B + s) * kTeamWarps + tc.wt] = v;
                }
            }
        }
        cons_release(ring, tc.lane);
        team_sync(tc.team);  // partials of this stage are visible; the other buffer is free again
        if (tc.ttid < nrows * B) {
            const int r = tc.ttid / B, s = tc.ttid - r * B;
            float a = 0.f;
#pragma unroll
            for (int w = 0; w < kTeamWarps; ++w) a += ps[tc.ttid * kTeamWarps + w];
            p.logits[(size_t)s * p.V + (size_t)u * R + r] = __float2half_rn(a);
        }
        buf ^= 1;
    }
}

// greedy argmax of one row of logits written by other CTAs (lowest index wins ties); all consumer threads, thread 0 stores
__device__ __forceinline__ void argmax_row(const __half* row, int V, int32_t* out) {
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    float best = -INFINITY;
    int idx = 0x7fffffff;
    for (int i = tid; i < V; i += kConsumers) {
        const float v = __half2float(ld_cg_h(row + i));  // written by other CTAs
        if (GPTQ_ARGMAX_BEATS(v, i, best, idx)) {
            best = v;
            idx = i;
        }
    }
    __shared__ float sv[kConsumerWarps];
    __shared__ int si[kConsumerWarps];
    GPTQ_WARP_ARGMAX(best, idx);
    if (lane == 0) {
        sv[warp] = best;
        si[warp] = idx;
    }
    cta_sync();
    if (tid == 0) {
        for (int w = 1; w < kConsumerWarps; ++w)
            if (GPTQ_ARGMAX_BEATS(sv[w], si[w], best, idx)) {
                best = sv[w];
                idx = si[w];
            }
        out[0] = idx;
    }
}

template <bool ACT, bool BATCH>
__global__ void __launch_bounds__(kBlock, 1) llama_decode_mega_kernel(const __grid_constant__ MegaParams p) {
    extern __shared__ __align__(16) uint8_t smem_dyn[];
    uint8_t* smem_raw = smem_dyn + ((1024u - (smem_u32(smem_dyn) & 1023u)) & 1023u);  // TMA swizzle atoms: 1 KB aligned stages (1 KB of slack is allocated)
    __shared__ float red_s[2 * kConsumerWarps];
    __shared__ uint32_t xmax_s[kTeams][kMaxBatch];               // largest |x| of a team's staged O / D range (fp16 magnitude bits)
    __shared__ float xinv_s[1 + kTeams][kMaxBatch];              // 2^-e of the staged x (XScale): [0] the rows of Q / G, [1 + team] the team's O / D range
    __shared__ __align__(8) unsigned long long bars_s[kTeams][2 * kMaxStages];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    // smem (1 KB aligned): [team 0 ring][team 1 ring][xs: H halves][xsum: H/32 floats][tmp / team scratch]
    // (BATCH: xs = batch rows of xs_stride halves, xsum = batch rows of H/32 floats)
    const uint32_t ring_bytes = (uint32_t)p.n_stages * kStageBytes;
    const int nbat = BATCH ? p.batch : 1;
    __half* xs = reinterpret_cast<__half*>(smem_raw + kTeams * ring_bytes);
    float* xsum = reinterpret_cast<float*>(xs + (BATCH ? nbat * p.xs_stride : p.H));
    uint8_t* tmp_raw = reinterpret_cast<uint8_t*>(xsum + nbat * (p.H / 32));
    tmp_raw += (16 - (reinterpret_cast<uintptr_t>(tmp_raw) & 15)) & 15;
    __half* tmp = reinterpret_cast<__half*>(tmp_raw);

    if (tid == 0) {
        for (int tm = 0; tm < kTeams; ++tm)
            for (int s = 0; s < p.n_stages; ++s) {
                mbar_init(smem_u32(&bars_s[tm][s]), 1);
                mbar_init(smem_u32(&bars_s[tm][kMaxStages + s]), kTeamWarps);
            }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    }
    __syncthreads();  // the only block-wide barrier: after it the producer warps and the consumers never meet again
    const unsigned nb = gridDim.x * kTeams;
    if (warp >= kConsumerWarps) {
        if (lane == 0) {
            const int tm = warp - kConsumerWarps;
            ProdRing r;
            r.ring = smem_u32(smem_raw) + tm * ring_bytes;
            r.full = smem_u32(&bars_s[tm][0]);
            r.empty = smem_u32(&bars_s[tm][kMaxStages]);
            r.stage = 0;
            r.use = 0;
            r.nstages = p.n_stages;
#ifdef GPTQ_TRACE
            r.blocked = 0;
#endif
            producer_loop<BATCH>(p, r, blockIdx.x * kTeams + tm, nb);
        }
        return;
    }
    TeamCtx tc;
    tc.team = warp / kTeamWarps;
    tc.wt = warp % kTeamWarps;
    tc.lane = lane;
    tc.ttid = tid - tc.team * kTeamThreads;
    tc.T = blockIdx.x * kTeams + tc.team;
    tc.nb = nb;
    tc.xseg = xs + tc.team * (p.H / 2);
    tc.xsum_seg = xsum + tc.team * (p.H / 64);
    tc.xinv_seg = xinv_s[1 + tc.team];
    tc.xmax = xmax_s[tc.team];
    tc.scratch = tmp_raw + tc.team * kTeamScratch;
    ConsRing ring;
    ring.ring = smem_u32(smem_raw) + tc.team * ring_bytes;
    ring.full = smem_u32(&bars_s[tc.team][0]);
    ring.tile = ring.ring;
    ring.bar = ring.full;
    ring.parity = 0;
    ring.left = p.n_stages;
    ring.nstages = p.n_stages;
#ifdef GPTQ_TRACE
    ring.waited = 0;
    ring.stages = 0;
#endif

    unsigned long long gen;  // barrier target (meaningful in thread 0): the counter value when this launch began
    {
        // bar[1] = counter value at the end of the previous launch (written by CTA 0 after its last barrier): CTAs that
        // start late may already see arrivals of this launch in bar[0], never in bar[1]
        unsigned long long v;
        asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p.bar + 1) : "memory");
        gen = v;
    }
    unsigned long long xgen = 0;  // the same for the cross-GPU barrier (tensor parallelism)
    if (p.tp_size > 1) asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(xgen) : "l"(p.xbar_peer[p.tp_rank] + 32 * kMaxTP) : "memory");
    // after the o_proj, down_proj and lm_head operations every rank needs every rank's contributions
    auto sync_all_ranks = [&](float* loc, float* const* peers) {
        if (p.tp_size == 1) {
            grid_barrier(p.bar, gen);
        } else {
            if (p.tp_exchange && loc != nullptr) {
                grid_barrier(p.bar, gen);
                tp_exchange(p, loc, peers, p.H);
            }
            tp_barrier(p, xgen);
        }
    };

    // this step's RoPE angles, one row per sequence (quant/fused_attn.py:43,91): freq_i = exp(i * inv_base) * pos
    if (blockIdx.x == 0 && tid < 64 * nbat) {
        const int s = tid >> 6, i = tid & 63;
        const float f = rope_inv_freq(i, p.inv_base) * (float)step_pos(p, s);
        p.rope_cs[s * kHD + i] = cosf(f);
        p.rope_cs[s * kHD + 64 + i] = sinf(f);
    }

    // residual stream: every stage_norm reads buffer `cur` (or, before the first layer, the embedding rows) and writes the other one
    const __half* resid_src = nullptr;
    const float* resid_acc = nullptr;
    int cur = 1;
    // stage_norm for every sequence in turn (its tmp row and red_s are reused); sequence s reads row s of src / acc (or its own
    // embedding row while acc is nullptr) and writes row s of resid_out, xs and xsum
    auto stage_norms = [&](bool plain, const __half* src, const float* acc, const __half* norm_w, __half* resid_out, const int32_t* perm) {
#pragma unroll 1
        for (int s = 0; s < nbat; ++s) {
            const __half* src_s = acc != nullptr ? src + (size_t)s * p.H : p.embed + (size_t)min(max(p.tokens[s], 0), p.V - 1) * p.H;
            const float* acc_s = acc != nullptr ? acc + (size_t)s * p.H : nullptr;
            __half* out_s = resid_out != nullptr ? resid_out + (size_t)s * p.H : nullptr;
            if (plain)
                stage_norm<false, true>(p, src_s, acc_s, norm_w, out_s, xs + (size_t)s * p.xs_stride, xsum + s * (p.H / 32), nullptr, tmp, red_s, nullptr);
            else
                stage_norm<ACT, false>(p, src_s, acc_s, norm_w, out_s, xs + (size_t)s * p.xs_stride, xsum + s * (p.H / 32), xinv_s[0] + s, tmp, red_s, perm);
        }
    };
#pragma unroll 1
    for (int l = 0; l < p.n_layers; ++l) {
        const LayerDesc& L = p.layers[l];
        // ---- Q ----
        MTRACE(l * 12 + 0);
        stage_norms(false, resid_src, resid_acc, L.input_norm, p.resid[cur ^ 1], L.qkv_perm);
        MTRACE(l * 12 + 1);
        cur ^= 1;
        zero_slice(p.acc_g, nbat * p.I);  // last read by the previous layer's D
        zero_slice(p.acc_u, nbat * p.I);
        {
            OPTRACE_BEGIN(ring);
            run_matvec<1, X_FULL, false, BATCH>(p, ring, tc, L.qkv.gs_steps, p.H, 3 * p.Hq, p.acc_qkv, nullptr, xs, xsum, xinv_s[0]);
            OPTRACE_END(ring, l, 0);
        }
        MTRACE(l * 12 + 2);
        grid_barrier(p.bar, gen);
        MTRACE(l * 12 + 3);
        // ---- A ----
        zero_slice(p.acc_d, nbat * p.H);  // last read by this layer's Q
        {
            OPTRACE_BEGIN(ring);
            run_attention<BATCH>(p, ring, tc, l);
            OPTRACE_END(ring, l, 1);
        }
        MTRACE(l * 12 + 4);
        grid_barrier(p.bar, gen);
        MTRACE(l * 12 + 5);
        // ---- O ----
        zero_slice(p.acc_qkv, nbat * 3 * p.Hq);
        {
            OPTRACE_BEGIN(ring);
            if constexpr (BATCH)
                run_matvec<1, X_ATTN, ACT, true>(p, ring, tc, L.o.gs_steps, p.Hq, p.H, p.acc_o, nullptr, xs, xsum, nullptr, L.o_perm);
            else
                run_matvec<1, X_ATTN, ACT>(p, ring, tc, L.o.gs_steps, p.Hq, p.H, p.tp_exchange ? p.acc_o_loc : p.acc_o, nullptr, xs, xsum, nullptr, L.o_perm, (p.tp_size > 1 && !p.tp_exchange) ? p.acc_o_peer : nullptr);
            OPTRACE_END(ring, l, 2);
        }
        MTRACE(l * 12 + 6);
        sync_all_ranks(p.acc_o_loc, p.acc_o_peer);
        MTRACE(l * 12 + 7);
        // ---- G ----
        stage_norms(false, p.resid[cur], p.acc_o, L.post_norm, p.resid[cur ^ 1], L.mlp_perm);
        cur ^= 1;
        MTRACE(l * 12 + 8);
        {
            OPTRACE_BEGIN(ring);
            run_matvec<2, X_FULL, false, BATCH>(p, ring, tc, L.gate.gs_steps, p.H, p.I, p.acc_g, p.acc_u, xs, xsum, xinv_s[0]);
            OPTRACE_END(ring, l, 3);
        }
        MTRACE(l * 12 + 9);
        grid_barrier(p.bar, gen);
        // ---- D ----
        zero_slice(p.acc_o, nbat * p.H);
        MTRACE(l * 12 + 10);
        {
            OPTRACE_BEGIN(ring);
            if constexpr (BATCH)
                run_matvec<1, X_SWIGLU, false, true>(p, ring, tc, L.down.gs_steps, p.I, p.H, p.acc_d, nullptr, xs, xsum, nullptr);
            else
                run_matvec<1, X_SWIGLU>(p, ring, tc, L.down.gs_steps, p.I, p.H, p.tp_exchange ? p.acc_d_loc : p.acc_d, nullptr, xs, xsum, nullptr, nullptr, (p.tp_size > 1 && !p.tp_exchange) ? p.acc_d_peer : nullptr);
            OPTRACE_END(ring, l, 4);
        }
        MTRACE(l * 12 + 11);
        sync_all_ranks(p.acc_d_loc, p.acc_d_peer);
        resid_src = p.resid[cur];
        resid_acc = p.acc_d;
    }
    // ---- L: final norm + lm_head ----
    stage_norms(true, resid_src, resid_acc, p.final_norm, nullptr, nullptr);
    zero_slice(p.acc_g, nbat * p.I);
    zero_slice(p.acc_u, nbat * p.I);
    if constexpr (BATCH)
        run_lm_head_batch(p, ring, tc, xs);
    else
        run_lm_head(p, ring, tc, xs);
    sync_all_ranks(nullptr, nullptr);
    zero_slice(p.acc_d, nbat * p.H);
    if (blockIdx.x == 0 && tid == 0) {  // every CTA has arrived at the last barrier: the counters rest at these values until the next launch
        p.bar[1] = gen;
        if (p.tp_size > 1) p.xbar_peer[p.tp_rank][32 * kMaxTP] = xgen;
    }
    if ((int)blockIdx.x < nbat && p.next_token != nullptr) argmax_row(p.logits + (size_t)blockIdx.x * p.V, p.V, p.next_token + blockIdx.x);  // CTA s: sequence s
}

// 3-D view of packed matrices with row stride N * 4 bytes: {32 words (128 B), packed rows, 128-byte chunks}, box 32 x box_rows x 8
// (= box_rows rows of a 256-column slab), 128-byte swizzle
bool encode_weight_map(CUtensorMap* tm, const void* base, int rows, uint64_t chunks, int N, int box_rows) {
    const cuuint64_t dims[3] = {32, (cuuint64_t)rows, (cuuint64_t)chunks};  // innermost first
    const cuuint64_t strides[2] = {(cuuint64_t)N * 4, 128};                 // bytes: packed row, chunk
    const cuuint32_t box[3] = {32, (cuuint32_t)box_rows, (cuuint32_t)(kSlabCols / 32)};
    return encode_tensor_map(tm, CU_TENSOR_MAP_DATA_TYPE_UINT32, 3, base, dims, strides, box);
}

// device properties that shape the launch (queried per call: no cached global state)
struct MegaPlan {
    int grid, n_stages, lm_rows;
    size_t smem;
};

// halves between the sequences' rows of the staged x at batch > 1 (see MegaParams::xs_stride)
inline int xs_stride(int H) { return H + 32; }

// Shared-memory plan for this model at `batch` sequences on a device with `sms` SMs and `smem_max` bytes of opt-in shared memory per block;
// returns false if the shape does not fit the kernel's staging buffers.  At batch B > 1 the staged x is B rows of xs_stride halves and its
// step sums B rows of H/32 floats, which leaves fewer ring stages; the attention needs B * n_heads <= teams (one team per (sequence, head)
// pair at least) and the lm_head partials of 2 * lm_rows * B rows x 8 warps must fit the team scratch.
bool mega_plan(const gptq_llama_model& m, int batch, int sms, size_t smem_max, size_t smem_static, MegaPlan& pl) {
    const int H = m.hidden, I = m.intermediate;
    const size_t xs_bytes = batch > 1 ? (size_t)batch * xs_stride(H) * 2 : (size_t)H * 2;
    const size_t fixed = xs_bytes + (size_t)batch * (H / 32) * 4 + 16 + max((size_t)H * 2, (size_t)kTeams * kTeamScratch);
    const size_t other = fixed + smem_static + 1024;  // + the kernel's static shared memory + 1 KB alignment slack of the rings
    if (smem_max < other) return false;
    int st = (int)((smem_max - other) / ((size_t)kTeams * kStageBytes));
    st = min(st, kMaxStages);
    if (st < 2) return false;
    pl.grid = sms;
    pl.n_stages = st;
    pl.smem = fixed + 1024 + (size_t)kTeams * st * kStageBytes;
    pl.lm_rows = max(1, kLmStageBytes / (H * 2));
    if (batch > 1) pl.lm_rows = max(1, min(pl.lm_rows, kTeamScratch / (2 * batch * kTeamWarps * 4)));
    if ((size_t)pl.lm_rows * H * 2 > (size_t)kStageBytes) return false;
    if ((size_t)2 * pl.lm_rows * batch * kTeamWarps * 4 > (size_t)kTeamScratch) return false;
    // per-team k-segments of o_proj / down_proj are staged in half of the xs buffer, their step sums in half of xsum
    const long long nteams = (long long)sms * kTeams;
    const int Hq = m.n_heads * m.head_dim;  // attention width of this rank (= H on a single GPU)
    const long long seg_o = ((long long)(H / kSlabCols) * (Hq / 32) + nteams - 1) / nteams + 1;
    const long long seg_d = ((long long)(H / kSlabCols) * (I / 32) + nteams - 1) / nteams + 1;
    const long long seg = max(seg_o, seg_d);
    if (seg * 32 > H / 2 || seg > H / 64) return false;
    if ((long long)batch * m.n_heads > nteams) return false;  // a team's attention range must meet at most two heads (one (sequence, head) pair at batch > 1)
    // 32-bit range arithmetic of team_range: (T + 1) * U must stay below 2^32 for every operation's unit count U
    const long long umax = max(max((long long)2 * (I / kSlabCols) * (H / 32), (long long)(H / kSlabCols) * (I / 32)),
                               max((long long)m.vocab, (long long)m.n_heads * 4096));
    if (umax * (nteams + 1) >= (1ll << 32)) return false;
    return true;
}


// Byte offsets of the persistent kernel's buffers in its scratch region.  The head (resid, acc_o, acc_d, xbar) depends on the hidden size
// and the batch only, so it has the same layout on every tensor-parallel rank: peers address acc_o / acc_d / xbar of this rank through its
// scratch base.  Every per-sequence buffer is [B][n] (gptq_b200.h); acc_qkv has room for 3 H (a tensor-parallel rank uses 3 Hq of it).
struct MegaScratch {
    size_t resid[2], acc_o, acc_d, xbar, acc_o_loc, acc_d_loc, acc_qkv, acc_g, acc_u, part, rope_cs, bar, total;
};
MegaScratch mega_scratch(const gptq_llama_model& m, int batch) {
    const size_t B = (size_t)batch, H = (size_t)m.hidden, I = (size_t)m.intermediate;
    MegaScratch s{};
    s.resid[0] = carve(s.total, B * H * 2);
    s.resid[1] = carve(s.total, B * H * 2);
    s.acc_o = carve(s.total, B * H * 4);
    s.acc_d = carve(s.total, B * H * 4);
    s.xbar = carve(s.total, (kMaxTP + 1) * 256);
    s.acc_o_loc = carve(s.total, H * 4);
    s.acc_d_loc = carve(s.total, H * 4);
    s.acc_qkv = carve(s.total, B * 3 * H * 4);
    s.acc_g = carve(s.total, B * I * 4);
    s.acc_u = carve(s.total, B * I * 4);
    s.part = carve(s.total, (size_t)kMaxTeams * kRec * 4);
    s.rope_cs = carve(s.total, B * 128 * 4);
    s.bar = carve(s.total, 256);
    return s;
}

// the instantiation for this model and batch: ACT if any layer carries an input gather, BATCH at batch > 1
using MegaKernel = void (*)(MegaParams);
MegaKernel mega_kernel(const gptq_llama_model& m, int batch) {
    const bool act = has_input_perm(m);
    return batch > 1 ? (act ? llama_decode_mega_kernel<true, true> : llama_decode_mega_kernel<false, true>)
                     : (act ? llama_decode_mega_kernel<true, false> : llama_decode_mega_kernel<false, false>);
}

// Launch plan of the persistent kernel for this step.  cudaErrorInvalidConfiguration: the step does not fit the kernel (the kernel chain
// runs it).  Any other error: the device could not be queried, and only the shapes were checked.
cudaError_t mega_step_plan(const gptq_llama_model& m, const gptq_llama_state& st, MegaPlan& pl) {
    constexpr cudaError_t kNo = cudaErrorInvalidConfiguration;
    if (st.batch < 1 || st.batch > kMaxBatch || m.n_layers > kMaxLayers || m.head_dim != kHD) return kNo;
    if (st.batch > 1 && st.tp != nullptr) return kNo;  // tensor parallelism: batch 1 only
    if (m.hidden % kSlabCols || m.intermediate % kSlabCols || m.hidden > 8192 || m.intermediate > 32768 || m.hidden % 64) return kNo;
    if ((3 * m.n_heads * m.head_dim) % kSlabCols) return kNo;  // the (local) fused qkv width is dealt in 256-column slabs
    if (st.tp != nullptr) {
        const gptq_llama_tp& tp = *st.tp;
        if (tp.size < 1 || tp.size > kMaxTP || tp.rank < 0 || tp.rank >= tp.size) return kNo;
        if (tp.vocab_begin < 0 || tp.vocab_end > m.vocab || tp.vocab_begin >= tp.vocab_end) return kNo;
        for (int q = 0; q < tp.size; ++q)
            if (q != tp.rank && (tp.peer_scratch[q] == nullptr || tp.peer_logits[q] == nullptr)) return kNo;
    } else if (m.n_heads * m.head_dim != m.hidden) {
        return kNo;
    }
    for (int l = 0; l < m.n_layers; ++l) {
        const gptq_llama_layer& ly = m.layers[l];
        const gptq_qweight* ws[5] = {&ly.qkv, &ly.o, &ly.gate, &ly.up, &ly.down};
        for (const gptq_qweight* w : ws) {
            if (w->bits != 4 || w->groupsize <= 0 || w->groupsize % 32) return kNo;
            if (!aligned(w->qweight, 16) || !aligned(w->scales, 16) || !aligned(w->qzeros, 16)) return kNo;
        }
        if (ly.gate.groupsize != ly.up.groupsize) return kNo;
    }
    if (!aligned(m.lm_head, 16) || !aligned(st.k_cache, 16) || !aligned(st.v_cache, 16)) return kNo;
    // the staging buffers of this batch must fit the current device
    int dev = 0, sms = 0, smem_optin = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess ||
        cudaDeviceGetAttribute(&smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev) != cudaSuccess)
        return cudaErrorInvalidDevice;
    cudaFuncAttributes fa;
    if (cudaFuncGetAttributes(&fa, mega_kernel(m, st.batch)) != cudaSuccess) return cudaErrorInvalidDeviceFunction;
    if (sms * kTeams > kMaxTeams || !mega_plan(m, st.batch, sms, (size_t)smem_optin, fa.sharedSizeBytes, pl)) return kNo;
    return cudaSuccess;
}

}  // namespace

// ---------------------------------------------------------------------------------------------------
bool mega_supported(const gptq_llama_model& m, const gptq_llama_state& st) {
    MegaPlan pl;
    return mega_step_plan(m, st, pl) != cudaErrorInvalidConfiguration;
}

size_t mega_scratch_bytes(const gptq_llama_model& m, int batch) { return mega_scratch(m, batch).total; }

cudaError_t launch_decode_mega(const gptq_llama_model& m, const gptq_llama_state& st, uint8_t* scratch, cudaStream_t stream) {
    static_assert(sizeof(MegaParams) < 32000, "kernel parameter space");
    MegaPlan pl;
    cudaError_t e = mega_step_plan(m, st, pl);
    if (e != cudaSuccess) return e;
    const int B = st.batch;
    const MegaKernel kernel = mega_kernel(m, B);

    MegaParams p{};
    p.n_layers = m.n_layers; p.H = m.hidden; p.Hq = m.n_heads * m.head_dim; p.I = m.intermediate; p.V = m.vocab; p.n_heads = m.n_heads;
    p.v0 = st.tp != nullptr ? st.tp->vocab_begin : 0;
    p.v1 = st.tp != nullptr ? st.tp->vocab_end : m.vocab;
    p.max_seq = st.max_seq;
    p.n_stages = pl.n_stages;
    p.lm_rows = pl.lm_rows;
    p.eps = m.rms_eps;
    p.inv_base = rope_inv_base(m.rope_base, m.head_dim);
    p.scale = attn_scale(m.head_dim);
    p.embed = reinterpret_cast<const __half*>(m.embed);
    p.final_norm = reinterpret_cast<const __half*>(m.final_norm);
    p.lm_head = reinterpret_cast<const __half*>(m.lm_head);
    p.tokens = st.tokens;
    p.positions = st.positions;
    p.k_cache = reinterpret_cast<__half*>(st.k_cache);
    p.v_cache = reinterpret_cast<__half*>(st.v_cache);
    p.layer_stride = (size_t)B * m.n_heads * st.max_seq * m.head_dim;
    p.logits = reinterpret_cast<__half*>(st.logits);
    p.next_token = st.next_tokens;
    p.batch = B;
    p.xs_stride = xs_stride(m.hidden);
    const MegaScratch ms = mega_scratch(m, B);
    p.resid[0] = reinterpret_cast<__half*>(scratch + ms.resid[0]);
    p.resid[1] = reinterpret_cast<__half*>(scratch + ms.resid[1]);
    p.acc_o = reinterpret_cast<float*>(scratch + ms.acc_o);
    p.acc_d = reinterpret_cast<float*>(scratch + ms.acc_d);
    const gptq_llama_tp* tp = st.tp;
    p.tp_size = tp != nullptr ? tp->size : 1;
    p.tp_rank = tp != nullptr ? tp->rank : 0;
    // measured on 65B (DESIGN.md section 6): direct peer REDs win up to 4 ranks, the local reduction + slice exchange at 8
    p.tp_exchange = (tp != nullptr && tp->size > 1) ? (tp->reduce_mode == 0 ? (tp->size > 4) : (tp->reduce_mode == 2)) : 0;
    for (int q = 0; q < p.tp_size; ++q) {
        uint8_t* base = (tp != nullptr && q != tp->rank) ? reinterpret_cast<uint8_t*>(tp->peer_scratch[q]) : scratch;
        p.acc_o_peer[q] = reinterpret_cast<float*>(base + ms.acc_o);
        p.acc_d_peer[q] = reinterpret_cast<float*>(base + ms.acc_d);
        p.xbar_peer[q] = reinterpret_cast<unsigned long long*>(base + ms.xbar);
        p.logits_peer[q] = reinterpret_cast<__half*>((tp != nullptr && q != tp->rank) ? tp->peer_logits[q] : st.logits);
    }
    p.acc_o_loc = reinterpret_cast<float*>(scratch + ms.acc_o_loc);
    p.acc_d_loc = reinterpret_cast<float*>(scratch + ms.acc_d_loc);
    p.acc_qkv = reinterpret_cast<float*>(scratch + ms.acc_qkv);
    p.acc_g = reinterpret_cast<float*>(scratch + ms.acc_g);
    p.acc_u = reinterpret_cast<float*>(scratch + ms.acc_u);
    p.part = reinterpret_cast<float*>(scratch + ms.part);
    p.rope_cs = reinterpret_cast<float*>(scratch + ms.rope_cs);
    p.bar = reinterpret_cast<unsigned long long*>(scratch + ms.bar);
    // One tensor map per row stride serves every layer: class 0 = qkv (N = 3H), 1 = o and down (N = H), 2 = gate and up (N = I).
    // Its base is the lowest qweight address of the class; a matrix is addressed through the chunk coordinate (128-byte units).
    const int classN[3] = {3 * m.n_heads * m.head_dim, m.hidden, m.intermediate};
    uintptr_t base[3] = {UINTPTR_MAX, UINTPTR_MAX, UINTPTR_MAX}, top[3] = {0, 0, 0};
    int rows_max[3] = {0, 0, 0};
    auto visit = [&](const gptq_qweight& w, int c) {
        const uintptr_t a = reinterpret_cast<uintptr_t>(w.qweight);
        base[c] = a < base[c] ? a : base[c];
        top[c] = a > top[c] ? a : top[c];
        rows_max[c] = max(rows_max[c], w.K / 8);
    };
    for (int l = 0; l < m.n_layers; ++l) {
        const gptq_llama_layer& ly = m.layers[l];
        visit(ly.qkv, 0); visit(ly.o, 1); visit(ly.down, 1); visit(ly.gate, 2); visit(ly.up, 2);
    }
    for (int c = 0; c < 3; ++c) {
        if (!aligned(reinterpret_cast<const void*>(base[c]), 128)) return cudaErrorInvalidConfiguration;
        const uint64_t chunks = (uint64_t)(top[c] - base[c]) / 128 + (uint64_t)classN[c] / 32;
        if (chunks >= (1ull << 31)) return cudaErrorInvalidConfiguration;
        for (int v = 0; v < 2; ++v)
            if (!encode_weight_map(&p.tmaps[3 * v + c], reinterpret_cast<const void*>(base[c]), rows_max[c], chunks, classN[c], v == 0 ? 4 * kStageSteps : 4))
                return cudaErrorNotSupported;
    }
    for (int l = 0; l < m.n_layers; ++l) {
        const gptq_llama_layer& ly = m.layers[l];
        bool whole_chunks = true;
        auto md = [&](const gptq_qweight& w, int c) {
            MatDesc d;
            d.sc = reinterpret_cast<const __half*>(w.scales);
            d.qz = reinterpret_cast<const uint32_t*>(w.qzeros);
            d.gs_steps = w.groupsize / 32;
            d.tmap = c;
            const uintptr_t delta = reinterpret_cast<uintptr_t>(w.qweight) - base[c];
            whole_chunks = whole_chunks && (delta % 128 == 0);
            d.chunk0 = (int)(delta / 128);
            return d;
        };
        p.layers[l].qkv = md(ly.qkv, 0);
        p.layers[l].o = md(ly.o, 1);
        p.layers[l].gate = md(ly.gate, 2);
        p.layers[l].up = md(ly.up, 2);
        p.layers[l].down = md(ly.down, 1);
        if (!whole_chunks) return cudaErrorInvalidConfiguration;
        p.layers[l].input_norm = reinterpret_cast<const __half*>(ly.input_norm);
        p.layers[l].post_norm = reinterpret_cast<const __half*>(ly.post_norm);
        p.layers[l].qkv_perm = ly.qkv_perm;
        p.layers[l].o_perm = ly.o_perm;
        p.layers[l].mlp_perm = ly.mlp_perm;
    }
    e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pl.smem);
    if (e != cudaSuccess) return e;
    int occ = 0;
    // cooperative launch: every CTA must be co-resident (one per SM); if the device cannot host them, the caller falls back to
    // the kernel-chain engine instead of risking a barrier deadlock
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kernel, kBlock, pl.smem) != cudaSuccess || occ < 1) return cudaErrorCooperativeLaunchTooLarge;
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(pl.grid);
    cfg.blockDim = dim3(kBlock);
    cfg.dynamicSmemBytes = pl.smem;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeCooperative;  // all CTAs co-resident: the grid barrier cannot deadlock
    attr[0].val.cooperative = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, kernel, p);
}

}  // namespace gptq

#ifdef GPTQ_TRACE
extern "C" int gptq_debug_set_mega_trace(void* buf) {
    unsigned long long* b = reinterpret_cast<unsigned long long*>(buf);
    return (int)cudaMemcpyToSymbol(gptq::g_mega_trace, &b, sizeof(b));
}
#endif
