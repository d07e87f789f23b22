"""Decode engine host side: a GPTQ LLaMA decoded token by token on a static KV cache, the whole step
captured once in a CUDA graph (gptq_llama_decode_step in include/gptq_b200.h).

This is the H100-native replacement for the reference's per-token loop (llama.py:419-433 /
model.generate in llama_inference.py:120): ~480 Python-dispatched launches and an O(n) torch.cat of
the KV cache per token become one graph replay.  torch is used for device memory, streams and graph
capture only.
"""
import ctypes
import math

import torch

from . import ops
from ._lib import LlamaLayer, LlamaModel, LlamaState, LlamaTP, Sampling, check, lib
from .ops import QLayerWeights

c_void_p, c_int, c_float, c_size_t = ctypes.c_void_p, ctypes.c_int, ctypes.c_float, ctypes.c_size_t


LLAMA_SHAPES = {  # hidden, intermediate, layers, heads (SURVEY.md section 8)
    '7b': (4096, 11008, 32, 32),
    '13b': (5120, 13824, 40, 40),
    '33b': (6656, 17920, 60, 52),
    '65b': (8192, 22016, 80, 64),
    'tiny': (256, 704, 2, 2),    # intermediate not a multiple of 256: exercises the kernel-chain engine
    'tiny256': (256, 768, 2, 2),  # eligible for the persistent single-kernel path
    'tiny512': (512, 1024, 2, 4),  # shardable over 2 tensor-parallel ranks (2 heads and 2 slabs of 256 MLP columns each)
    # grouped-query attention: their K/V head counts are in KV_HEADS
    '70b': (8192, 28672, 80, 64),        # LLaMA-2-70B
    '34b': (8192, 22016, 48, 64),        # CodeLlama-34B (RoPE base 1e6)
    'llama3-8b': (4096, 14336, 32, 32),  # LLaMA-3-8B (RoPE base 5e5, vocabulary 128256)
    'tiny-gqa2': (512, 1024, 2, 4),      # persistent single-kernel path, 2 query heads per K/V head
    'tiny-gqa1': (512, 1024, 2, 4),      # persistent, one K/V head for all 4 query heads
    'tiny-gqa2-chain': (512, 704, 2, 4),  # intermediate not a multiple of 256: the kernel-chain engine
    'tiny-gqa1-chain': (512, 704, 2, 4),
}
KV_HEADS = {'70b': 8, '34b': 8, 'llama3-8b': 8, 'tiny-gqa2': 2, 'tiny-gqa1': 1, 'tiny-gqa2-chain': 2, 'tiny-gqa1-chain': 1}  # other shapes: one per head


def kv_heads(size):
    """K/V heads of a named shape (LLAMA_SHAPES): KV_HEADS, else one per query head (multi-head attention)."""
    return KV_HEADS.get(size, LLAMA_SHAPES[size][3])


def random_qlayer(K, N, bits, groupsize, device, gen, act_order=False):
    """Synthetic packed layer (SURVEY.md 8(d) perf fixture): uniform random fields, scales ~ U(1e-3, 1.1e-2)."""
    G = math.ceil(K / groupsize)
    half = 1 << (bits - 1)
    if bits == 3:
        qw = ops.pack_qweight(torch.randint(0, 8, (K, N), device=device, generator=gen, dtype=torch.int32), 3)
    else:
        qw = torch.randint(-2**31, 2**31 - 1, (K // 32 * bits, N), device=device, generator=gen, dtype=torch.int32)
    # zero points centred on the weight grid like a real asymmetric GPTQ checkpoint (stored minus one: z = stored + 1 has the mean
    # of the uniform fields, 2^(bits-1) - 1/2).  Fully random zeros give every weight the same mean offset, and a 32-layer stack of
    # such matrices amplifies the common mode of the activations until fp16 overflows.
    lo, hi = (half - 3, half + 1) if bits >= 4 else (half - 2, half)
    qz = ops.pack_qzeros(torch.randint(lo, hi, (G, N), device=device, generator=gen, dtype=torch.int32), bits)
    s = (torch.rand(G, N, device=device, generator=gen) * 1e-2 + 1e-3).half()
    g = (torch.arange(K, device=device) // groupsize).to(torch.int32)
    if act_order:
        perm = torch.randperm(K, device=device, generator=gen)
        g = g[torch.argsort(perm)].contiguous()
    return QLayerWeights(qw, s, qz, g, bits, groupsize)


def kernel_layers(layers, allow_perm=True):
    """Load-time preparation of a layer stack for the decode kernels (the stored tensors stay as they are):
    2/3-bit fields widened to nibbles and act-order rows regrouped (QLayerWeights.kernel_form).  The input gathers this needs are
    returned per layer for the kernel (qkv, o, gate|up); down_proj's gather costs nothing at run time: it is folded into
    the column order of gate|up, whose SwiGLU output then comes out in down_proj's regrouped order.
    Returns (prepared layers, perms) or None when gate and up do not share their act-order map."""
    out, perms = [], []
    for ly in layers:
        mlp = ops.mlp_kernel_form(ly['gate'], ly['up'], allow_perm)
        if mlp is None:
            return None
        k = dict(zip(('gate', 'up'), mlp), **{name: ly[name].kernel_form(allow_perm) for name in ('qkv', 'o', 'down')})
        pm = {name: k[name].perm for name in ('qkv', 'o', 'gate', 'down')}
        if pm['down'] is not None:
            k['gate'], k['up'] = k['gate'].permute_columns(pm['down']), k['up'].permute_columns(pm['down'])
        # per-input-feature vectors of a regrouped matvec are handed over in regrouped order
        k['input_norm'] = ly['input_norm'] if pm['qkv'] is None else ly['input_norm'].index_select(0, pm['qkv']).contiguous()
        k['post_norm'] = ly['post_norm'] if pm['gate'] is None else ly['post_norm'].index_select(0, pm['gate']).contiguous()
        out.append(k)
        perms.append({n: (pm[n].to(torch.int32).contiguous() if pm[n] is not None else None) for n in ('qkv', 'o', 'gate')})
    return out, perms


SCORE_ROWS = 16384  # rows per scoring pass (LlamaDecoder.score): bounds the activations (at LLaMA-7B the fp16 MLP intermediate of a pass is 361 MB)


class LlamaDecoder:
    """Owns the weights, the KV cache and the captured graph; `step()` decodes one token per sequence."""

    def __init__(self, layers, embed, final_norm, lm_head, n_heads, rms_eps=1e-6, rope_base=10000.0, batch=1, max_seq=2048, use_graph=True, head_dim=None,
                 tp=None, n_kv_heads=None):
        """tp = (rank, size, vocab_begin, vocab_end[, reduce_mode]): this process holds one tensor-parallel shard (see shard_for_rank / gptq_llama_tp): `layers`,
        `lm_head` and `n_heads` are the LOCAL ones, head_dim must be given, and torch.distributed must be initialised (the scratch and logits
        buffers of the ranks are exchanged as CUDA IPC handles).
        n_kv_heads: K/V heads of grouped-query attention (None: n_heads, multi-head attention).  It must divide n_heads, and every layer's fused
        qkv must be (n_heads + 2 n_kv_heads) * head_dim wide (q, then k, then v heads; the width is how the kernels learn the count).
        The KV cache holds n_kv_heads heads.  Tensor parallelism needs n_kv_heads == n_heads."""
        self.dev = embed.device
        self.tp = tp
        self.head_dim = head_dim or embed.shape[1] // n_heads
        self.layers = layers  # list of dicts: qkv, o, gate, up, down (QLayerWeights), input_norm, post_norm (fp16 tensors)
        self.n_kv_heads = n_heads if n_kv_heads is None else int(n_kv_heads)
        if self.n_kv_heads < 1 or n_heads % self.n_kv_heads != 0:
            raise ValueError(f'n_kv_heads ({n_kv_heads}) must be a positive divisor of n_heads ({n_heads})')
        if tp is not None:
            _refuse_gqa_tp(n_heads, self.n_kv_heads)
        qkv_width = (n_heads + 2 * self.n_kv_heads) * self.head_dim
        for i, ly in enumerate(layers):
            if ly['qkv'].qweight.shape[1] != qkv_width:
                raise ValueError(f'layer {i}: fused qkv has {ly["qkv"].qweight.shape[1]} columns, {n_heads} query and {self.n_kv_heads} K/V heads of '
                                 f'{self.head_dim} need {qkv_width}')
        self.embed, self.final_norm, self.lm_head = embed.contiguous(), final_norm.contiguous(), lm_head.contiguous()
        self.hidden = embed.shape[1]
        self.vocab = embed.shape[0]
        self.n_heads = n_heads
        self.intermediate = layers[0]['gate'].qweight.shape[1]
        self.batch, self.max_seq = batch, max_seq
        with torch.cuda.device(self.dev):
            self._layer_arr = (LlamaLayer * len(layers))()  # filled below, once the kernel form of the layers is chosen
            m = LlamaModel()
            m.n_layers, m.hidden, m.n_heads, m.head_dim = len(layers), self.hidden, n_heads, self.head_dim
            m.intermediate, m.vocab, m.rms_eps, m.rope_base = self.intermediate, self.vocab, rms_eps, rope_base
            m.layers = ctypes.cast(self._layer_arr, ctypes.POINTER(LlamaLayer))
            m.embed, m.final_norm, m.lm_head = self.embed.data_ptr(), self.final_norm.data_ptr(), self.lm_head.data_ptr()
            self.model = m
            cache_shape = (len(layers), batch, self.n_kv_heads, max_seq, self.head_dim)
            self.k_cache = torch.zeros(cache_shape, dtype=torch.float16, device=self.dev)
            self.v_cache = torch.zeros(cache_shape, dtype=torch.float16, device=self.dev)
            self.tokens = torch.zeros(batch, dtype=torch.int32, device=self.dev)
            self.positions = torch.zeros(batch, dtype=torch.int32, device=self.dev)
            self.next_tokens = torch.zeros(batch, dtype=torch.int32, device=self.dev)
            nbytes = lib.gptq_llama_scratch_bytes(ctypes.byref(m), batch, max_seq)
            if nbytes == 0:
                raise ValueError('unsupported decode configuration (batch must be 1..8)')
            self._tp_struct = None
            if tp is None:
                self.logits = torch.zeros(batch, self.vocab, dtype=torch.float16, device=self.dev)
                self.scratch = torch.zeros(nbytes, dtype=torch.uint8, device=self.dev)
            else:
                self._setup_tp(nbytes)
            st = LlamaState()
            st.batch, st.max_seq = batch, max_seq
            st.k_cache, st.v_cache = self.k_cache.data_ptr(), self.v_cache.data_ptr()
            st.tokens, st.positions = self.tokens.data_ptr(), self.positions.data_ptr()
            st.logits, st.next_tokens = self.logits.data_ptr(), self.next_tokens.data_ptr()
            st.scratch, st.scratch_bytes = self.scratch.data_ptr(), nbytes
            if self._tp_struct is not None:
                st.tp = ctypes.pointer(self._tp_struct)
            self.state = st
            # kernel-side view of the weights: nibble-widened 2/3-bit fields, regrouped act-order rows (+ input gathers).  The gathers exist
            # only in the persistent kernel: when gate and up cannot share one, or the step would not take that kernel, act-order layers
            # keep their stored form.
            for allow_perm in (True, False):
                prepared = kernel_layers(layers, allow_perm)
                if prepared is not None:
                    self.klayers, self.perms = prepared
                    self._fill_layer_structs()
                    if all(p is None for pm in self.perms for p in pm.values()) or self.launches_per_step() == 1:
                        break
        # host-side record of the KV cache: lengths[b] positions of sequence b are cached, cached_tokens[b] are the token ids of its first
        # positions as far as they are known (reset, prefill_batch, set_input and extend keep both; raw writes to self.positions do not)
        self.lengths = [0] * batch
        self.cached_tokens = [[] for _ in range(batch)]
        self.n_launches = None
        self.graph = None
        self._sampling = None  # the gptq_sampling struct while set_sampling is in force
        self._sampling_arrays = self._sampling_struct = None  # its device arrays: allocated once, the sampled graph reads them in place
        self.sample_graph = None  # the decode step followed by gptq_sample_tokens, captured on first sampled use
        self._stream = torch.cuda.Stream(self.dev)
        if use_graph:
            self.graph = self._capture(self._enqueue, self._enqueue)

    def _setup_tp(self, scratch_bytes):
        """Scratch and logits in IPC-shareable device memory; every rank maps every other rank's buffers (gptq_llama_tp)."""
        import torch.distributed as dist
        rank, size, v0, v1 = self.tp[:4]
        assert self.batch == 1 and dist.is_initialized() and dist.get_world_size() == size

        def ipc_buffer(nbytes, dtype):
            ptr, handle = ctypes.c_void_p(), ctypes.create_string_buffer(64)
            check(lib.gptq_ipc_alloc(nbytes, ctypes.byref(ptr), handle))

            class _Raw:  # zero-copy torch view of the raw allocation
                __cuda_array_interface__ = {'shape': (nbytes, ), 'typestr': '|u1', 'data': (ptr.value, False), 'version': 2}

            t = torch.as_tensor(_Raw(), device=self.dev)
            return ptr.value, handle.raw, t.view(dtype)

        self._scratch_ptr, h_scr, self.scratch = ipc_buffer(scratch_bytes, torch.uint8)
        self._logits_ptr, h_log, logits = ipc_buffer(self.batch * self.vocab * 2, torch.float16)
        self.logits = logits.view(self.batch, self.vocab)
        handles = [None] * size
        dist.all_gather_object(handles, (h_scr, h_log))
        t = LlamaTP()
        t.size, t.rank, t.vocab_begin, t.vocab_end = size, rank, v0, v1
        t.reduce_mode = self.tp[4] if len(self.tp) > 4 else 0
        self._peer_maps = []
        for q, (hs, hl) in enumerate(handles):
            if q == rank:
                t.peer_scratch[q], t.peer_logits[q] = self._scratch_ptr, self._logits_ptr
                continue
            for field, h in ((t.peer_scratch, hs), (t.peer_logits, hl)):
                ptr = ctypes.c_void_p()
                check(lib.gptq_ipc_open(h, ctypes.byref(ptr)))
                field[q] = ptr.value
                self._peer_maps.append(ptr.value)
        self._tp_struct = t
        dist.barrier()  # every rank has mapped every buffer before anybody launches

    def _fill_layer_structs(self):
        for i, ly in enumerate(self.klayers):
            for name in ('qkv', 'o', 'gate', 'up', 'down'):
                setattr(self._layer_arr[i], name, ly[name].struct())
            self._layer_arr[i].input_norm = ly['input_norm'].data_ptr()
            self._layer_arr[i].post_norm = ly['post_norm'].data_ptr()
            pm = self.perms[i]
            self._layer_arr[i].qkv_perm = pm['qkv'].data_ptr() if pm['qkv'] is not None else None
            self._layer_arr[i].o_perm = pm['o'].data_ptr() if pm['o'] is not None else None
            self._layer_arr[i].mlp_perm = pm['gate'].data_ptr() if pm['gate'] is not None else None

    # ------------------------------------------------------------------------------------------
    def _enqueue(self, stream, sample=False):
        """One decode step on `stream`; with `sample`, followed by gptq_sample_tokens under set_sampling's parameters."""
        check(lib.gptq_llama_decode_step(ctypes.byref(self.model), ctypes.byref(self.state), ctypes.c_void_p(stream.cuda_stream)))
        if sample:
            self._enqueue_sample(stream)

    def _enqueue_sample(self, stream):
        check(lib.gptq_sample_tokens(self.logits.data_ptr(), self.vocab, self.batch, self.vocab, self.positions.data_ptr(), ctypes.byref(self._sampling),
                                     self.next_tokens.data_ptr(), ctypes.c_void_p(stream.cuda_stream)))

    def _capture(self, enqueue, warm_up):
        """A CUDA graph of enqueue(stream), captured on the decoder's stream after warm_up(stream) has run once outside the capture (lazy module
        loading, func attributes)."""
        with torch.cuda.device(self.dev):
            torch.cuda.synchronize()
            with torch.cuda.stream(self._stream):
                warm_up(self._stream)
                self._stream.synchronize()
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g, stream=self._stream):
                    enqueue(self._stream)
            torch.cuda.synchronize()
        return g

    def launches_per_step(self) -> int:
        """Kernels of ours launched per decoded token (1 on the persistent single-kernel path)."""
        return int(lib.gptq_llama_decode_launches(ctypes.byref(self.model), ctypes.byref(self.state)))

    def mega_scratch_offset(self) -> int:
        """Byte offset of the persistent kernel's region in self.scratch (diagnostics; see gptq_llama_persistent_scratch_offset)."""
        return int(lib.gptq_llama_persistent_scratch_offset(ctypes.byref(self.model), self.batch, self.max_seq))

    def step(self, stream=None):
        """Run one decode step on the tokens/positions currently in device memory.  With set_sampling in force, next_tokens is then drawn
        from the step's logits by gptq_sample_tokens (one more launch, in a second captured graph)."""
        sample = self._sampling is not None
        if self.graph is None:
            self._enqueue(stream or torch.cuda.current_stream(self.dev), sample)
        elif not sample:
            self.graph.replay()
        else:
            if self.sample_graph is None:  # warm-up: the sampling kernel alone, which reads the current logits and writes next_tokens only
                self.sample_graph = self._capture(lambda s: self._enqueue(s, sample=True), self._enqueue_sample)
            self.sample_graph.replay()

    def _refuse_tp(self, feature):
        """The ranks of a tensor-parallel decoder run the decode step only: anything else is refused before it touches the device."""
        if self.tp is not None:
            raise ValueError(f'{feature}: not supported under tensor parallelism')

    def _sampling_args(self, temperature, top_k, top_p, seed, eos_token_id, min_length):
        """set_sampling's arguments checked and as host tensors of one value per sequence, named after the gptq_sampling fields."""
        self._refuse_tp('sampling and eos stopping')
        t, k, p = sampling_lists(self.batch, temperature, top_k, top_p)
        eos = [-1 if v is None else int(v) for v in _per_seq(self.batch, eos_token_id, 'eos_token_id')]
        if any(not -1 <= e < self.vocab for e in eos):
            raise ValueError(f'eos_token_id outside the vocabulary (0..{self.vocab - 1})')
        return dict(temperature=torch.tensor(t, dtype=torch.float32), top_k=torch.tensor(k, dtype=torch.int32), top_p=torch.tensor(p, dtype=torch.float32),
                    seed=torch.tensor([(int(v) + 2**63) % 2**64 - 2**63 for v in _per_seq(self.batch, seed, 'seed')]),  # the uint64 seed's bits as int64
                    eos_token=torch.tensor(eos, dtype=torch.int32),
                    min_length=torch.tensor([int(v) for v in _per_seq(self.batch, min_length, 'min_length')], dtype=torch.int32))

    def set_sampling(self, temperature, top_k, top_p, seed, eos_token_id=None, min_length=0):
        """Draw next_tokens from each step's logits from now on (gptq_sample_tokens; clear_sampling ends it).  Every argument is one value for
        all sequences or a list of `batch`: temperature (0: greedy), top_k (0: off), top_p (1: off), seed (64-bit), eos_token_id (None: no eos)
        and min_length (eos is suppressed while position + 1 < min_length)."""
        args = self._sampling_args(temperature, top_k, top_p, seed, eos_token_id, min_length)
        if self._sampling_arrays is None:  # allocated once: the sampled graph reads them in place
            with torch.cuda.device(self.dev):
                self._sampling_arrays = {f: torch.zeros_like(v, device=self.dev) for f, v in args.items()}
            self._sampling_struct = Sampling(**{f: a.data_ptr() for f, a in self._sampling_arrays.items()})
        for f, v in args.items():
            self._sampling_arrays[f].copy_(v)
        self._sampling = self._sampling_struct

    def clear_sampling(self):
        """step() takes the argmax again (the decode step's own next_tokens)."""
        self._sampling = None

    def reset(self):
        self.positions.zero_()
        self.lengths = [0] * self.batch
        self.cached_tokens = [[] for _ in range(self.batch)]

    def _record(self, b, pos, toks):
        """Sequence b's cache rows pos .. pos + len(toks) - 1 now hold `toks` and nothing past them is cached.  The known token prefix grows only
        when it reaches pos (otherwise the rows in between are of unknown origin and the prefix stays as it was)."""
        self.lengths[b] = pos + len(toks)
        known = self.cached_tokens[b]
        self.cached_tokens[b] = known[:pos] + list(toks) if len(known) >= pos else known

    def _token_ids(self, tokens, what='token id', check=True):
        """Token ids given as a tensor (of any shape) or a sequence, as a list, each checked against the vocabulary (ValueError) unless `check`
        is False."""
        ids = tokens.reshape(-1).tolist() if isinstance(tokens, torch.Tensor) else [int(t) for t in tokens]
        if check and any(not 0 <= t < self.vocab for t in ids):
            raise ValueError(f'{what} outside the vocabulary (0..{self.vocab - 1})')
        return ids

    def set_input(self, tokens, positions):
        """Token ids (int or sequence of `batch` ints) and the cache position of this step (int: every sequence, or sequence of `batch` ints: one
        per sequence); validated on the host: the kernels only clamp (a position beyond the cache or a token outside the vocabulary must never
        reach them).  The step that follows caches row p of each sequence, so `lengths` becomes p + 1 (writing self.positions directly bypasses
        this record, and generate(..., reuse_cache=True) then reuses less or nothing)."""
        toks = self._token_ids([tokens] * self.batch if isinstance(tokens, int) else tokens)
        if len(toks) != self.batch:
            raise ValueError(f'expected {self.batch} token ids, got {len(toks)}')
        pos = [int(positions)] * self.batch if isinstance(positions, int) else [int(p) for p in positions]
        if len(pos) != self.batch:
            raise ValueError(f'expected {self.batch} positions, got {len(pos)}')
        if any(not 0 <= p < self.max_seq for p in pos):
            raise ValueError(f'position {positions} outside the KV cache (max_seq = {self.max_seq})')
        self.tokens.copy_(torch.tensor(toks, dtype=torch.int32))
        self.positions.copy_(torch.tensor(pos, dtype=torch.int32))
        for b, (t, p) in enumerate(zip(toks, pos)):
            self._record(b, p, [t])

    @torch.no_grad()
    def prefill(self, prompt_ids):
        """prefill_batch of one prompt (batch 1).  Returns the number of cached positions."""
        assert self.batch == 1
        return self.prefill_batch([prompt_ids])[0]

    def _forward_rows(self, seqs, cache=False, starts=None):
        """The ragged pass shared by prefill, scoring and extend: the token lists `seqs` are concatenated into one M-row pass (M = the sum of
        their lengths) through the quantized linears on the wgmma GEMM path (gptq_qlinear_fwd / gptq_fused_mlp_fwd), the RMSNorm kernel and the
        RoPE kernel (per-token positions).
        starts=None: every list from position 0; the causal attention runs per list in torch SDPA (as the reference's QuantLlamaAttention does,
        quant/fused_attn.py:154-155).  With `cache`, every layer's keys (after RoPE) and values of list b are written to rows 0..len - 1 of
        sequence b's KV cache; without, nothing but the returned tensor is written.
        starts[b] = p: list b continues sequence b from position p (its cache holds positions 0..p - 1; requires `cache`): its keys and values
        are written to rows p..p + len - 1, and the attention of all lists runs in one gptq_cached_attention call per layer, over each
        sequence's cached prefix and its new rows, read in place from the cache.
        Returns the residual stream after the last layer, fp16 [M, hidden] (final norm not applied)."""
        ns = [len(s) for s in seqs]
        total = sum(ns)
        H, nh, nkv, hd = self.hidden, self.n_heads, self.n_kv_heads, self.head_dim
        ids = [int(t) for s in seqs for t in s]
        x = self.embed[torch.tensor(ids, device=self.dev)]  # [total, H]
        if starts is None:
            pos = torch.cat([torch.arange(n, dtype=torch.int64) for n in ns]).to(self.dev)[None, :]
        else:
            assert cache
            pos = torch.cat([torch.arange(p, p + n, dtype=torch.int64) for p, n in zip(starts, ns)]).to(self.dev)[None, :]
        spans = [(b, sum(ns[:b]), n) for b, n in enumerate(ns) if n > 0]  # (list, first row, rows)
        sdpa = dict(enable_gqa=True) if nkv != nh else {}
        for li, ly in enumerate(self.layers):
            qkv = ops.matmul248(ops.rmsnorm(x, ly['input_norm'], self.model.rms_eps), *ly['qkv'].parts(), ly['qkv'].bits,
                                groupsize=ly['qkv'].hint).view(1, total, nh + 2 * nkv, hd)  # q | k | v heads
            # q and k are the first nh + nkv rows of head_dim of every token: one RoPE call rotates both
            ops.rotate_half_(qkv[:, :, :nh + nkv].unsqueeze(2), pos, base=self.model.rope_base)
            q_rows, k_rows, v_rows = qkv[0].split([nh, nkv, nkv], dim=1)  # [total, heads, hd]
            if starts is None:
                atts = []
                for b, r0, n in spans:
                    q, k, v = (t[r0:r0 + n].transpose(0, 1) for t in (q_rows, k_rows, v_rows))  # [heads, n, hd]
                    if cache:
                        self.k_cache[li, b, :, :n] = k
                        self.v_cache[li, b, :, :n] = v
                    atts.append(torch.nn.functional.scaled_dot_product_attention(q[None], k[None], v[None], is_causal=True, **sdpa)[0].transpose(0, 1).reshape(n, H))
                att = atts[0] if len(atts) == 1 else torch.cat(atts)
            else:
                for b, r0, n in spans:
                    p = starts[b]
                    self.k_cache[li, b, :, p:p + n] = k_rows[r0:r0 + n].transpose(0, 1)
                    self.v_cache[li, b, :, p:p + n] = v_rows[r0:r0 + n].transpose(0, 1)
                att = ops.cached_attention(qkv.view(total, -1)[:, :H], self.k_cache[li], self.v_cache[li], [(b, starts[b], n) for b, _, n in spans])
            x = x + ops.matmul248(att, *ly['o'].parts(), ly['o'].bits, groupsize=ly['o'].hint)
            h = ops.fused_mlp(ops.rmsnorm(x, ly['post_norm'], self.model.rms_eps), ly['gate'].parts(), ly['up'].parts(), ly['gate'].bits, ly['gate'].hint)
            x = x + ops.matmul248(h, *ly['down'].parts(), ly['down'].bits, groupsize=ly['down'].hint)
        return x

    @torch.no_grad()
    def prefill_batch(self, prompts):
        """Ragged pass (_forward_rows) over the first len(prompt) - 1 tokens of each of the `batch` prompts that fills sequence b's slot of the
        static KV cache.  The LAST token of each prompt then goes through the decode step like every generated one (it produces the first
        logits).  Returns the number of cached positions per prompt (0 for a prompt of length 1)."""
        self._refuse_tp('prefill_batch()')
        if len(prompts) != self.batch:
            raise ValueError(f'expected {self.batch} prompts, got {len(prompts)}')
        ns = [max(len(p) - 1, 0) for p in prompts]
        if any(n > self.max_seq for n in ns):
            raise ValueError(f'prompt does not fit the KV cache (max_seq = {self.max_seq})')
        if sum(ns) > 0:
            self._forward_rows([p[:n] for p, n in zip(prompts, ns)], cache=True)
        for b, (p, n) in enumerate(zip(prompts, ns)):
            self.cached_tokens[b] = []
            self._record(b, 0, [int(t) for t in p[:n]])
        return ns

    @torch.no_grad()
    def extend(self, chunks):
        """Append chunks[b] (a list of token ids, possibly empty) to sequence b, after the lengths[b] positions its KV cache already holds, in one
        ragged pass (_forward_rows with starts = lengths): the new rows attend to the cached prefix and to each other through
        gptq_cached_attention, and their keys and values are written to cache rows lengths[b] .. lengths[b] + len - 1.  An empty chunk leaves its
        sequence untouched.  The decode buffers and the captured graph are not touched; the next step(s) continue at the new lengths.
        Everything is validated before anything is written.  Returns the new lengths."""
        self._refuse_tp('extend()')
        if len(chunks) != self.batch:
            raise ValueError(f'expected {self.batch} chunks, got {len(chunks)}')
        seqs = [self._token_ids(c) for c in chunks]
        for b, s in enumerate(seqs):
            if self.lengths[b] + len(s) > self.max_seq:
                raise ValueError(f'sequence {b}: {self.lengths[b]} cached + {len(s)} new positions do not fit the KV cache (max_seq = {self.max_seq})')
        if any(seqs):
            self._forward_rows(seqs, cache=True, starts=list(self.lengths))
        for b, s in enumerate(seqs):
            if s:
                self._record(b, self.lengths[b], s)
        return list(self.lengths)

    @torch.no_grad()
    def score(self, sequences):
        """Per-token log-likelihood: for each token list t of length n >= 2, the n - 1 fp32 values log p(t_i | t_<i), i = 1..n-1 (one tensor per
        list).  Each list is scored from position 0 by the ragged pass (_forward_rows, no KV cache), the final RMSNorm and the fused
        lm_head + log-softmax kernel (gptq_lm_head_logprob).  Lists are grouped into passes of at most SCORE_ROWS rows (a longer list is scored
        alone), so activation memory stays bounded.  Independent of `batch` and `max_seq`; the KV cache, the decode buffers and the captured
        graph are not touched."""
        self._refuse_tp('score()')
        seqs = [self._token_ids(s) for s in sequences]
        if any(len(s) < 2 for s in seqs):
            raise ValueError('every scored sequence needs at least 2 tokens')
        out = []
        i = 0
        while i < len(seqs):
            j, rows = i + 1, len(seqs[i])
            while j < len(seqs) and rows + len(seqs[j]) <= SCORE_ROWS:
                rows += len(seqs[j])
                j += 1
            group = seqs[i:j]
            x = self._forward_rows(group)
            # row r of a list predicts its token r + 1: every row but the list's last
            keep, r0 = [], 0
            for s in group:
                keep.append(torch.arange(r0, r0 + len(s) - 1))
                r0 += len(s)
            xn = ops.rmsnorm(x.index_select(0, torch.cat(keep).to(self.dev)), self.final_norm, self.model.rms_eps)
            targets = torch.tensor([t for s in group for t in s[1:]], dtype=torch.int32, device=self.dev)
            out.extend(ops.lm_head_logprob(xn, self.lm_head, targets).split([len(s) - 1 for s in group]))
            i = j
        return out

    @torch.no_grad()
    def perplexity(self, token_ids, seqlen=2048):
        """Perplexity of a token stream as the reference's llama_eval computes it (llama.py:174-259): nsamples = len // seqlen chunks (the tail is
        dropped), each scored from position 0, ppl = exp(sum of the chunks' NLL / (nsamples * (seqlen - 1))), the NLL summed in fp64."""
        ids = self._token_ids(token_ids, check=False)  # score() checks the chunks; the dropped tail is never read
        if seqlen < 2:
            raise ValueError('seqlen must be at least 2')
        nsamples = len(ids) // seqlen
        if nsamples == 0:
            raise ValueError(f'{len(ids)} tokens do not fill one chunk of seqlen {seqlen}')
        lps = self.score([ids[i * seqlen:(i + 1) * seqlen] for i in range(nsamples)])
        nll = -float(torch.cat(lps).double().sum())
        return math.exp(nll / (nsamples * (seqlen - 1)))

    def _decode(self, prompts, max_new_tokens, starts, eos=None):
        """Lock-step decode: sequence b is stepped from position starts[b] (its cache holds the positions before it) until it has
        max_new_tokens new tokens or has emitted eos[b] (None: no eos); the prompts' remaining tokens are fed first.  The steps end when every
        sequence is done; a finished sequence is stepped along meanwhile, and the cache rows it writes then are dropped from its record."""
        out = [list(p) for p in prompts]
        steps = len(prompts[0]) + max_new_tokens - 1 - starts[0]
        assert all(len(p) + max_new_tokens - 1 - s == steps for p, s in zip(prompts, starts))
        stopped = [False] * len(prompts)
        for k in range(steps):
            pos = [s + k for s in starts]
            self.set_input([p[i] if i < len(p) else o[-1] for p, o, i in zip(prompts, out, pos)], pos)
            self.step()
            nxt = self.next_tokens.tolist()
            for b, (p, i) in enumerate(zip(prompts, pos)):
                if i >= len(p) - 1 and not stopped[b]:
                    out[b].append(nxt[b])
                    stopped[b] = eos is not None and nxt[b] == eos[b]
            if all(stopped):
                break
        for b, o in enumerate(out):
            if stopped[b]:  # the record covers the returned tokens but the last, as for a sequence that ran to max_new_tokens
                self.lengths[b] = len(o) - 1
                self.cached_tokens[b] = self.cached_tokens[b][:len(o) - 1]
        return out

    def _reuse(self, prompts, extend=True):
        """Keep what each sequence's cache shares with its prompt (reusable_prefix) and drop the rest of the record; with `extend`, append the
        uncached prompt tokens but the last in one extend() pass.  Returns the positions the decode steps start from."""
        keep = [reusable_prefix(p, self.cached_tokens[b][:self.lengths[b]]) for b, p in enumerate(prompts)]
        for b, c in enumerate(keep):
            self.lengths[b] = c
            self.cached_tokens[b] = self.cached_tokens[b][:c]
        if not extend:
            return keep
        self.extend([p[c:len(p) - 1] for p, c in zip(prompts, keep)])
        return [len(p) - 1 for p in prompts]

    def _generate(self, prompts, max_new_tokens, prefill, reuse_cache, do_sample, temperature, top_k, top_p, seed, eos_token_id, min_new_tokens):
        """generate and generate_batch.  Every argument is checked before the cache or its record is touched.  When sampling or an eos token is
        asked for, gptq_sample_tokens runs after every step (else exactly the greedy decode): sequence b draws with seed + b (seed None: a random
        64-bit seed from torch's host RNG) and cannot emit eos before min_new_tokens new tokens (min_length = len(prompt) + min_new_tokens)."""
        if len(prompts) != self.batch:
            raise ValueError(f'expected {self.batch} prompts, got {len(prompts)}')
        prompts = [self._token_ids(p, 'prompt token id') for p in prompts]
        for p in prompts:
            if len(p) < 1 or len(p) + max_new_tokens > self.max_seq + 1:
                raise ValueError(f'prompt ({len(p)}) + max_new_tokens ({max_new_tokens}) does not fit the KV cache (max_seq = {self.max_seq})')
        sampling = None
        if do_sample or eos_token_id is not None:
            eos = [None if v is None else int(v) for v in _per_seq(self.batch, eos_token_id, 'eos_token_id')]
            sampling = dict(temperature=temperature if do_sample else 0.0, top_k=top_k if do_sample else 0, top_p=top_p if do_sample else 1.0,
                            eos_token_id=eos, min_length=[len(p) + int(min_new_tokens) for p in prompts])
            self._sampling_args(seed=0, **sampling)  # the seed is drawn once everything has passed
            self._token_ids([e for e in eos if e is not None], 'eos_token_id')  # None is "no eos" here: unlike set_sampling, -1 is refused
        if int(min_new_tokens) < 0:
            raise ValueError('min_new_tokens must be >= 0')
        if reuse_cache or prefill:
            self._refuse_tp('reuse_cache' if reuse_cache else 'prefill')
        if reuse_cache:
            starts = self._reuse(prompts, extend=prefill)
        else:
            self.reset()
            starts = self.prefill_batch(prompts) if prefill else [0] * self.batch
        if sampling is None:
            return self._decode(prompts, max_new_tokens, starts)
        if seed is None:
            seed = int(torch.randint(-2**63, 2**63 - 1, (1, ), dtype=torch.int64)) % 2**64
        self.set_sampling(seed=[int(seed) + b for b in range(self.batch)], **sampling)
        try:
            return self._decode(prompts, max_new_tokens, starts, eos)
        finally:
            self.clear_sampling()

    @torch.no_grad()
    def generate(self, prompt_ids, max_new_tokens, prefill=True, reuse_cache=False, do_sample=False, temperature=1.0, top_k=50, top_p=1.0, seed=None,
                 eos_token_id=None, min_new_tokens=0):
        """Greedy decode (batch 1), or with do_sample=True sampled as HF's model.generate samples (llama_inference.py:119-127): temperature,
        top-k, top-p and one draw per token on the device (gptq_sample_tokens; the defaults are HF's).  seed None draws a random one; the same
        seed gives the same tokens.  With eos_token_id, generation stops after that token (greedy or sampled; it ends the returned list), but
        not before min_new_tokens new tokens.  One engine, two phases: the prompt is prefilled in one batched pass (wgmma GEMM path) into the static KV
        cache, then the persistent decode kernel takes over token by token; prefill=False, and tensor parallelism, feed the prompt through the
        decode step instead.  reuse_cache=True keeps the cached positions the prompt starts with (e.g. the conversation so far, when the prompt is
        that conversation plus a new turn) and computes only the rest (with extend(), or through the decode step with prefill=False)."""
        assert self.batch == 1
        return self._generate([prompt_ids], max_new_tokens, prefill and self.tp is None, reuse_cache, do_sample, temperature, top_k, top_p, seed,
                              eos_token_id, min_new_tokens)[0]

    @torch.no_grad()
    def generate_batch(self, prompts, max_new_tokens, reuse_cache=False, do_sample=False, temperature=1.0, top_k=50, top_p=1.0, seed=None,
                       eos_token_id=None, min_new_tokens=0):
        """Greedy decode of `batch` prompts of different lengths: one ragged prefill (prefill_batch), then every sequence is stepped in
        lock-step at its own position by the decode step (the persistent kernel decodes them all in one launch).  Returns one token list per
        prompt: the prompt followed by its max_new_tokens generated tokens.
        reuse_cache=True: sequence b keeps the longest prefix its cache shares with prompt b (at most len(prompt) - 1 positions) and only the
        rest of the prompt but its last token goes through one ragged extend() pass, so a second turn -- the previous output plus the new
        turn -- costs the new turn only.  The result is that of reuse_cache=False up to fp rounding.
        do_sample, temperature, top_k, top_p, seed, eos_token_id, min_new_tokens: as in generate; the sampling parameters may be lists of one
        value per sequence, and sequence b draws with seed + b, so row b is comparable with a batch-1 run seeded seed + b.  A sequence that
        emits eos stops (its list ends with it) while the others go on; afterwards each sequence's record (lengths, cached_tokens) covers its
        returned tokens but the last, so a following reuse_cache=True turn extends from there."""
        return self._generate(prompts, max_new_tokens, True, reuse_cache, do_sample, temperature, top_k, top_p, seed, eos_token_id, min_new_tokens)


def _per_seq(batch, v, name):
    """One value per sequence: a list of `batch` values, or one value for all."""
    vals = list(v) if isinstance(v, (list, tuple)) else [v] * batch
    if len(vals) != batch:
        raise ValueError(f'{name}: expected one value or {batch}, got {len(vals)}')
    return vals


def sampling_lists(batch, temperature, top_k, top_p):
    """Per-sequence temperature, top_k and top_p, checked as HF checks its warpers: temperature >= 0 (0: greedy), top_k >= 0 (0: off),
    0 < top_p <= 1 (1: off)."""
    t = [float(v) for v in _per_seq(batch, temperature, 'temperature')]
    k = [int(v) for v in _per_seq(batch, top_k, 'top_k')]
    p = [float(v) for v in _per_seq(batch, top_p, 'top_p')]
    if any(not (v >= 0 and math.isfinite(v)) for v in t):
        raise ValueError(f'temperature must be a finite value >= 0 (0: greedy), got {temperature}')
    if any(v < 0 for v in k):
        raise ValueError(f'top_k must be >= 0 (0: off), got {top_k}')
    if any(not 0 < v <= 1 for v in p):
        raise ValueError(f'top_p must be in (0, 1], got {top_p}')
    return t, k, p


def reusable_prefix(prompt, cached):
    """How many leading positions of a cache holding the token ids `cached` a new `prompt` can keep: the length of their common prefix, at most
    len(prompt) - 1, because the prompt's last token must still go through the decode step (it produces the first logits)."""
    n = min(len(prompt) - 1, len(cached))
    c = 0
    while c < n and int(prompt[c]) == int(cached[c]):
        c += 1
    return c


def _synthetic_draws(size, bits, groupsize, act_order, vocab, device, seed, n_layers):
    """The weights of the random-init model, drawn one at a time from one generator seeded with `seed`: each layer's dict, then the
    embedding, the lm_head and the final norm.  synthetic_llama and synthetic_llama_tp both build their model from these draws, so a
    tensor-parallel rank holds a shard of the very model synthetic_llama builds from the same seed.  groupsize -1: one group per linear (the
    reference's --groupsize -1, where QuantLinear takes groupsize = infeatures): hidden for qkv / o / gate / up, intermediate for down."""
    hidden, inter, layers, heads = LLAMA_SHAPES[size]
    qkv_cols = hidden + 2 * kv_heads(size) * (hidden // heads)  # q | k | v
    gs_h, gs_i = (hidden, inter) if groupsize == -1 else (groupsize, groupsize)
    dev = torch.device(device)
    gen = torch.Generator(device=dev).manual_seed(seed)
    qlayer = lambda K, N, gs: random_qlayer(K, N, bits, gs, dev, gen, act_order)
    norm = lambda: (torch.rand(hidden, device=dev, generator=gen) * 0.2 + 0.9).half()
    for _ in range(n_layers or layers):
        gate, up = qlayer(hidden, inter, gs_h), qlayer(hidden, inter, gs_h)
        if act_order:  # gate and up see the same input, hence the same Hessian diagonal and the same act-order map (gptq.py:210-216)
            up = QLayerWeights(up.qweight, up.scales, up.qzeros, gate.g_idx.clone(), bits, gs_h)
        # q/k/v share their input, hence their act-order map (quant/fused_attn.py:180): nothing to do, qkv is one layer here
        yield dict(qkv=qlayer(hidden, qkv_cols, gs_h), o=qlayer(hidden, hidden, gs_h), gate=gate, up=up, down=qlayer(inter, hidden, gs_i),
                   input_norm=norm(), post_norm=norm())
    yield (torch.randn(vocab, hidden, device=dev, generator=gen) * 0.5).half()
    yield (torch.randn(vocab, hidden, device=dev, generator=gen) * 0.02).half()
    yield norm()


def synthetic_llama(size='7b', bits=4, groupsize=128, act_order=False, vocab=32000, device='cuda:0', seed=0, n_layers=None, **kw):
    """Random-init GPTQ LLaMA of the named size (no checkpoints are reachable offline): every layer has its
    own distinct packed tensors so that a decode step streams the full model from HBM.  groupsize -1 as in _synthetic_draws."""
    *L, embed, lm_head, final_norm = _synthetic_draws(size, bits, groupsize, act_order, vocab, device, seed, n_layers)
    return LlamaDecoder(L, embed, final_norm, lm_head, LLAMA_SHAPES[size][3], n_kv_heads=kv_heads(size), **kw)


def _refuse_gqa_tp(n_heads, n_kv_heads):
    if n_kv_heads != n_heads:
        raise ValueError(f'tensor parallelism needs one K/V head per query head; this model has {n_heads} query and {n_kv_heads} K/V heads')


def shard_for_rank(layers, lm_head, n_heads, head_dim, rank, size):
    """Tensor-parallel shard of a layer stack (BASELINE config 5; DESIGN.md section 6): qkv columns of this rank's heads (q | k | v), o_proj rows
    of the same heads, gate/up column slabs of 256 with the matching down_proj rows, lm_head rows.  Plain g_idx only (row shards keep whole groups).
    Multi-head attention only: a grouped-query stack (qkv narrower than 3 * n_heads * head_dim) raises ValueError.
    Returns (local layers, local lm_head, local heads, (vocab_begin, vocab_end))."""
    H = n_heads * head_dim
    for ly in layers:
        _refuse_gqa_tp(n_heads, (ly['qkv'].qweight.shape[1] // head_dim - n_heads) / 2)
    assert n_heads % size == 0, 'heads must divide over the ranks'
    hl = n_heads // size
    dev = lm_head.device
    hcols = torch.arange(rank * hl * head_dim, (rank + 1) * hl * head_dim, device=dev)
    out = []
    for ly in layers:
        inter = ly['gate'].qweight.shape[1]
        nslab = inter // 256
        c0, c1 = rank * nslab // size * 256, (rank + 1) * nslab // size * 256
        mcols = torch.arange(c0, c1, device=dev)
        out.append(dict(qkv=ly['qkv'].column_slice(torch.cat([hcols, H + hcols, 2 * H + hcols])), o=ly['o'].row_slice(int(hcols[0]), int(hcols[-1]) + 1),
                        gate=ly['gate'].column_slice(mcols), up=ly['up'].column_slice(mcols), down=ly['down'].row_slice(c0, c1), input_norm=ly['input_norm'],
                        post_norm=ly['post_norm']))
    V = lm_head.shape[0]
    v0, v1 = rank * V // size, (rank + 1) * V // size
    return out, lm_head[v0:v1].contiguous(), hl, (v0, v1)


def synthetic_llama_tp(size_name, rank, world, bits=4, groupsize=128, vocab=32000, device='cuda:0', seed=0, n_layers=None, full=None, reduce_mode=0, **kw):
    """One tensor-parallel rank of the random-init model `synthetic_llama(size_name, seed=seed)` (every rank draws the same full model from the same
    seed layer by layer and keeps its shard), or of the given `full` decoder's weights.  groupsize -1 as in synthetic_llama."""
    hidden, _, _, heads = LLAMA_SHAPES[size_name]
    hd = hidden // heads
    _refuse_gqa_tp(heads, full.n_kv_heads if full is not None else kv_heads(size_name))
    if full is not None:
        L, lm_head, hl, (v0, v1) = shard_for_rank(full.layers, full.lm_head, heads, hd, rank, world)
        return LlamaDecoder(L, full.embed, full.final_norm, lm_head, hl, head_dim=hd, tp=(rank, world, v0, v1, reduce_mode), **kw)
    fake_head = torch.empty(0, hidden, device=device)
    shard = lambda w: shard_for_rank([w], fake_head, heads, hd, rank, world)[0][0] if isinstance(w, dict) else w
    # each layer is sharded as soon as it is drawn: a 65B model never exists whole on one GPU
    *L, embed, lm_head, final_norm = map(shard, _synthetic_draws(size_name, bits, groupsize, False, vocab, device, seed, n_layers))
    v0, v1 = rank * vocab // world, (rank + 1) * vocab // world
    return LlamaDecoder(L, embed, final_norm, lm_head[v0:v1].contiguous(), heads // world, head_dim=hd, tp=(rank, world, v0, v1, reduce_mode), **kw)


def from_hf_quant_model(model, batch=1, max_seq=2048, **kw):
    """Build a decoder from an HF LlamaForCausalLM that went through the reference's load_quant recipe with this
    repo's quant package (make_quant_linear -> load_state_dict -> make_quant_attn / make_quant_norm / make_fused_mlp)."""
    import quant
    L = []
    rope_bases = {layer.self_attn.rope_base for layer in model.model.layers if isinstance(layer.self_attn, quant.QuantLlamaAttention)}
    if len(rope_bases) > 1:
        raise ValueError(f'the attention layers disagree on the RoPE base: {sorted(rope_bases)}')
    for layer in model.model.layers:
        attn, mlp = layer.self_attn, layer.mlp
        if not isinstance(attn, quant.QuantLlamaAttention):
            raise ValueError('call quant.make_quant_attn(model) first')
        gate, up = mlp.weights() if isinstance(mlp, quant.QuantLlamaMLP) else (mlp.gate_proj.weights(), mlp.up_proj.weights())
        L.append(
            dict(qkv=attn.qkv_proj.weights(), o=attn.o_proj.weights(), gate=gate, up=up, down=mlp.down_proj.weights(),
                 input_norm=layer.input_layernorm.weight.data.half().contiguous(), post_norm=layer.post_attention_layernorm.weight.data.half().contiguous()))
    cfg = model.config
    return LlamaDecoder(L, model.model.embed_tokens.weight.data.half(), model.model.norm.weight.data.half().contiguous(), model.lm_head.weight.data.half(),
                        cfg.num_attention_heads, rms_eps=cfg.rms_norm_eps, rope_base=rope_bases.pop(), batch=batch, max_seq=max_seq,
                        n_kv_heads=model.model.layers[0].self_attn.num_key_value_heads, **kw)  # (make_quant_attn read it from the config)
