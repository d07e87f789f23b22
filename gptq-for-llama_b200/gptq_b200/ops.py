"""Tensor-level wrappers over the C ABI: the op-level signatures of the reference's quant package.

matmul248 / transpose_matmul248  <- quant/quant_linear.py:263-279
fused_mlp                        <- QuantLlamaMLP.triton_llama_mlp, quant/fused_mlp.py:206-218
rotate_half_                     <- triton_rotate_half_, quant/fused_attn.py:61-93
rmsnorm                          <- TritonLlamaRMSNorm.forward, quant/triton_norm.py:50-67
lm_head_logprob                  <- lm_head + shifted CrossEntropyLoss of llama_eval, llama.py:246-256 (per-token, fp32)
cached_attention                 <- causal SDPA of new rows over a sequence's cached prefix (the engine's extend path; no reference counterpart)
sample_tokens                    <- HF's temperature / top-k / top-p warpers + torch.multinomial of model.generate(do_sample=True), llama_inference.py:119-127

torch is plumbing here (device memory, current stream); all arithmetic happens in libgptq_b200.so.
"""
import ctypes
import functools
import math

import torch

from . import _lib
from ._lib import QWeight, check, lib

SUPPORTED_BITS = (2, 3, 4, 8)


def _require_cuda(*tensors):
    for t in tensors:
        if t is not None and not t.is_cuda:
            raise ValueError('Expected a cuda device: the quantized-linear path has no CPU implementation '
                             '(the reference raises the same from Triton)')


def _stream(t: torch.Tensor):
    return ctypes.c_void_p(torch.cuda.current_stream(t.device).cuda_stream)


def _rows(t: torch.Tensor):
    """A 2-D operand as the kernels take it: (t with a unit stride along its last dimension, copied only when it has none, and its leading
    dimension).  The leading dimension is the row stride, or the row width for a single row, whose row stride may be anything."""
    if t.stride(1) != 1:
        t = t.contiguous()
    return t, t.stride(0) if t.shape[0] > 1 else t.shape[1]


_workspaces = {}


def _workspace(dev: torch.device, nbytes: int):
    """Zero-initialised scratch, one per (device, stream); kernels leave it zeroed (include/gptq_b200.h)."""
    if nbytes == 0:
        return None, 0
    key = (dev.index, torch.cuda.current_stream(dev).cuda_stream)
    ws = _workspaces.get(key)
    if ws is None or ws.numel() < nbytes:
        ws = torch.zeros(max(nbytes, 1 << 20), dtype=torch.uint8, device=dev)
        _workspaces[key] = ws
    return ws, ws.numel()


def is_trivial_g_idx(g_idx: torch.Tensor, groupsize: int) -> bool:
    """True iff g_idx[k] == k // groupsize (no act-order).  One device->host sync; call at load time."""
    K = g_idx.numel()
    ref = torch.arange(K, device=g_idx.device, dtype=torch.int64) // groupsize
    return bool(torch.equal(g_idx[:K].to(torch.int64), ref))


def make_qweight(qweight, scales, qzeros, g_idx, bits: int, groupsize: int = 0) -> QWeight:
    """Build a gptq_qweight.  groupsize > 0 asserts g_idx is the trivial k // groupsize map."""
    if bits not in SUPPORTED_BITS:
        raise NotImplementedError('Only 2,3,4,8 bits are supported.')
    _require_cuda(qweight, scales, qzeros, g_idx)
    if qweight.dtype != torch.int32 or qzeros.dtype != torch.int32 or scales.dtype != torch.float16:
        raise ValueError('qweight/qzeros must be int32 and scales float16')
    if not (qweight.is_contiguous() and scales.is_contiguous() and qzeros.is_contiguous()):
        raise ValueError('packed tensors must be contiguous')
    K = qweight.shape[0] * 32 // bits
    N = qweight.shape[1]
    G = scales.shape[0]
    if g_idx is not None:
        if g_idx.dtype != torch.int32 or not g_idx.is_contiguous():
            raise ValueError('g_idx must be contiguous int32')
        if g_idx.numel() < K:  # the fused qkv g_idx is 3K long, only the first K entries are read (fused_attn.py:180)
            raise ValueError('g_idx shorter than infeatures')
    w = QWeight()
    w.qweight, w.scales, w.qzeros = qweight.data_ptr(), scales.data_ptr(), qzeros.data_ptr()
    w.g_idx = g_idx.data_ptr() if g_idx is not None else None
    w.K, w.N, w.G, w.bits, w.groupsize = K, N, G, bits, int(groupsize)
    return w


def matmul248(input, qweight, scales, qzeros, g_idx, bits, maxq=None, bias=None, groupsize: int = 0):
    """fp16 [M, N] = input[M, K] . deq(qweight) (+ bias).  `maxq` is accepted for signature parity and ignored."""
    _require_cuda(input, bias)
    if input.dim() != 2:
        raise ValueError('matmul248 expects a 2-D input')
    if input.dtype != torch.float16:
        input = input.half()
    input, ld = _rows(input)
    w = make_qweight(qweight, scales, qzeros, g_idx, bits, groupsize)
    if input.shape[1] != w.K:
        raise ValueError(f'input has {input.shape[1]} features, weight expects {w.K}')
    M = input.shape[0]
    if M == 0:
        return torch.empty((0, w.N), device=input.device, dtype=torch.float16)
    with torch.cuda.device(input.device):
        out = torch.empty((M, w.N), device=input.device, dtype=torch.float16)
        ws, ws_bytes = _workspace(input.device, lib.gptq_qlinear_workspace_bytes(M, w.K, w.N, bits))
        check(
            lib.gptq_qlinear_fwd(input.data_ptr(), ld, ctypes.byref(w), bias.data_ptr() if bias is not None else None, out.data_ptr(), w.N, M,
                                 ws.data_ptr() if ws is not None else None, ws_bytes, _stream(input)))
    return out


def transpose_matmul248(input, qweight, scales, qzeros, g_idx, bits, maxq=None, groupsize: int = 0):
    """fp16 [M, K] = input[M, N] . deq(qweight)^T  (gradient w.r.t. the layer input)."""
    _require_cuda(input)
    if input.dtype != torch.float16:
        input = input.half()
    input, ld = _rows(input)
    w = make_qweight(qweight, scales, qzeros, g_idx, bits, groupsize)
    M = input.shape[0]
    if M == 0:
        return torch.empty((0, w.K), device=input.device, dtype=torch.float16)
    with torch.cuda.device(input.device):
        out = torch.empty((M, w.K), device=input.device, dtype=torch.float16)
        check(lib.gptq_qlinear_transpose_fwd(input.data_ptr(), ld, ctypes.byref(w), out.data_ptr(), w.K, M, _stream(input)))
    return out


def fused_mlp(x, gate, up, bits, groupsize: int = 0):
    """silu(x . deq(gate)) * (x . deq(up)); gate / up = (qweight, scales, qzeros, g_idx)."""
    _require_cuda(x)
    if x.dtype != torch.float16:
        x = x.half()
    x, ld = _rows(x)
    wg = make_qweight(*gate, bits, groupsize)
    wu = make_qweight(*up, bits, groupsize)
    M = x.shape[0]
    if M == 0:
        return torch.empty((0, wg.N), device=x.device, dtype=torch.float16)
    with torch.cuda.device(x.device):
        out = torch.empty((M, wg.N), device=x.device, dtype=torch.float16)
        ws, ws_bytes = _workspace(x.device, lib.gptq_fused_mlp_workspace_bytes(M, wg.K, wg.N, bits))
        check(
            lib.gptq_fused_mlp_fwd(x.data_ptr(), ld, ctypes.byref(wg), ctypes.byref(wu), out.data_ptr(), wg.N, M, ws.data_ptr() if ws is not None else None,
                                   ws_bytes, _stream(x)))
    return out


LLAMA3_KEYS = ('factor', 'low_freq_factor', 'high_freq_factor', 'original_max_position_embeddings')


def rope_inv_freq(base: float, head_dim: int, rope_scaling):
    """The fp32 frequencies [head_dim / 2] of a scaled rotation, bit for bit the tensor HF builds for the same config
    (transformers.modeling_rope_utils._compute_llama3_parameters, the same fp32 operations in the same order), or None for an unscaled one
    (rope_scaling None, or its rope type 'default': the kernels then compute exp(i * -2 ln(base) / head_dim) themselves).

    The llama3 rule (LLaMA-3.1 / 3.2 / 3.3): with inv_freq = 1 / base^(2i / head_dim) and wavelength 2 pi / inv_freq, a frequency whose
    wavelength is below original_max_position_embeddings / high_freq_factor is kept, one above original_max_position_embeddings /
    low_freq_factor is divided by factor, and one in between is blended: (1 - s) inv_freq / factor + s inv_freq with
    s = (original_max_position_embeddings / wavelength - low_freq_factor) / (high_freq_factor - low_freq_factor).
    rope_scaling must carry every key of LLAMA3_KEYS with factor > 0, 0 < low_freq_factor < high_freq_factor and
    original_max_position_embeddings > 0; any other rope type, or a dict without those, raises ValueError."""
    if rope_scaling is None:
        return None
    rope_type = rope_scaling.get('rope_type', rope_scaling.get('type', 'default'))
    if rope_type == 'default':
        return None
    if rope_type != 'llama3':
        raise ValueError(f"RoPE type {rope_type!r} is not supported: only 'default' and 'llama3' rotary embeddings are computed")
    missing = [k for k in LLAMA3_KEYS if rope_scaling.get(k) is None]
    if missing:
        raise ValueError(f'llama3 RoPE scaling needs {", ".join(missing)}')
    if not all(isinstance(rope_scaling[k], (int, float)) and not isinstance(rope_scaling[k], bool) for k in LLAMA3_KEYS):
        raise ValueError(f'llama3 RoPE scaling: {", ".join(LLAMA3_KEYS)} must be numbers, got {rope_scaling}')
    factor, low, high, old_context = (float(rope_scaling[k]) for k in LLAMA3_KEYS)
    if not all(math.isfinite(v) for v in (factor, low, high, old_context, float(base))):
        raise ValueError(f'llama3 RoPE scaling: every value must be finite, got {rope_scaling} at base {base}')
    if not (factor > 0 and 0 < low < high and old_context > 0 and base > 0):
        raise ValueError(f'llama3 RoPE scaling needs factor > 0, 0 < low_freq_factor < high_freq_factor and original_max_position_embeddings > 0 '
                         f'(and base > 0), got {rope_scaling} at base {base}')
    if head_dim % 2 or head_dim < 2:
        raise ValueError(f'head_dim must be a positive even number, got {head_dim}')
    # HF keeps original_max_position_embeddings as the config holds it (an int in every published config); its operands are restated as such
    old_context = rope_scaling['original_max_position_embeddings']
    inv_freq = 1.0 / (float(base)**(torch.arange(0, head_dim, 2, dtype=torch.int64).to(dtype=torch.float) / head_dim))
    wavelen = 2 * math.pi / inv_freq
    scaled = torch.where(wavelen > old_context / rope_scaling['low_freq_factor'], inv_freq / rope_scaling['factor'], inv_freq)
    smooth = (old_context / wavelen - rope_scaling['low_freq_factor']) / (rope_scaling['high_freq_factor'] - rope_scaling['low_freq_factor'])
    smoothed = (1 - smooth) * scaled / rope_scaling['factor'] + smooth * scaled
    medium = ~(wavelen < old_context / rope_scaling['high_freq_factor']) * ~(wavelen > old_context / rope_scaling['low_freq_factor'])
    return torch.where(medium, smoothed, scaled).contiguous()


def _host_table(inv_freq):
    """A frequency table (tensor or sequence, [head_dim / 2]) as the C array the ABI reads on the host."""
    vals = inv_freq.detach().to('cpu', torch.float32).reshape(-1).tolist() if isinstance(inv_freq, torch.Tensor) else [float(v) for v in inv_freq]
    return (ctypes.c_float * len(vals))(*vals)


def rotate_half_(qk, position_ids, config=None, base: float = 10000.0, inv_freq=None):
    """In-place RoPE on qk[bsz, seq, 2, heads, head_dim] (may be a strided view of the qkv output).  inv_freq: the fp32 frequencies
    [head_dim / 2] of a scaled rotation (rope_inv_freq; gptq_rope_inplace_freq), which replace the unscaled rule at `base`."""
    _require_cuda(qk, position_ids)
    batch_size, seq_len, qandk, num_heads, head_dim = qk.shape
    # same argument checks as the reference (quant/fused_attn.py:69-74)
    assert qk.stride(3) == head_dim
    assert qk.stride(4) == 1
    assert position_ids.shape == (batch_size, seq_len)
    assert position_ids.stride(1) == 1, 'position_ids must be contiguous in the last dimension'
    assert qk.stride(2) == num_heads * head_dim and (batch_size == 1 or qk.stride(0) == seq_len * qk.stride(1)), 'q and k rows must be adjacent per token'
    if qk.dtype != torch.float16:
        raise ValueError('qk must be float16')
    if position_ids.dtype != torch.int64:
        position_ids = position_ids.long()
    if inv_freq is not None and len(inv_freq) != head_dim // 2:
        raise ValueError(f'inv_freq has {len(inv_freq)} entries, head_dim {head_dim} needs {head_dim // 2}')
    with torch.cuda.device(qk.device):
        if inv_freq is None:
            check(
                lib.gptq_rope_inplace(qk.data_ptr(), qk.stride(1), position_ids.data_ptr(), position_ids.stride(0), batch_size, seq_len, qandk * num_heads,
                                      head_dim, float(base), _stream(qk)))
        else:
            check(
                lib.gptq_rope_inplace_freq(qk.data_ptr(), qk.stride(1), position_ids.data_ptr(), position_ids.stride(0), batch_size, seq_len,
                                           qandk * num_heads, head_dim, _host_table(inv_freq), _stream(qk)))


def rmsnorm(x, weight, eps: float):
    _require_cuda(x, weight)
    x_arg, ld = _rows(x.reshape(-1, x.shape[-1]))
    if x_arg.dtype != torch.float16 or weight.dtype != torch.float16:
        raise ValueError('rmsnorm expects float16 activations and weight')
    M, N = x_arg.shape
    with torch.cuda.device(x.device):
        y = torch.empty((M, N), device=x.device, dtype=torch.float16)
        check(lib.gptq_rmsnorm_fwd(x_arg.data_ptr(), ld, weight.data_ptr(), y.data_ptr(), N, M, N, float(eps), _stream(x)))
    return y.reshape(x.shape)


def lm_head_logprob(x, weight, targets):
    """fp32 [M]: log-softmax of the fp16 logits fp16(x . weight^T) at column targets[m], for x fp16 [M, K] and the lm_head weight fp16 [V, K]
    (as nn.Linear stores it); the [M, V] logits are never materialised.  Targets are checked against [0, V) here (one device->host sync)."""
    _require_cuda(x, weight, targets)
    if x.dim() != 2 or weight.dim() != 2 or x.shape[1] != weight.shape[1]:
        raise ValueError(f'expected x [M, K] and weight [V, K], got {tuple(x.shape)} and {tuple(weight.shape)}')
    if x.dtype != torch.float16 or weight.dtype != torch.float16:
        raise ValueError('lm_head_logprob expects float16 activations and weight')
    M, K = x.shape
    V = weight.shape[0]
    targets = targets.reshape(-1)
    if targets.numel() != M:
        raise ValueError(f'expected {M} targets, got {targets.numel()}')
    if M == 0:
        return torch.empty(0, device=x.device, dtype=torch.float32)
    if int(targets.min()) < 0 or int(targets.max()) >= V:
        raise ValueError(f'target id outside the vocabulary (0..{V - 1})')
    targets = targets.to(torch.int32).contiguous()
    x, ldx = _rows(x)
    weight, ldw = _rows(weight)
    with torch.cuda.device(x.device):
        out = torch.empty(M, device=x.device, dtype=torch.float32)
        ws, ws_bytes = _workspace(x.device, lib.gptq_lm_head_logprob_workspace_bytes(M, V))
        check(
            lib.gptq_lm_head_logprob(x.data_ptr(), ldx, weight.data_ptr(), ldw, M, K, V, targets.data_ptr(), out.data_ptr(), ws.data_ptr(), ws_bytes,
                                     _stream(x)))
    return out


def cached_attention(q, k_cache, v_cache, spans):
    """fp16 [M, n_heads * head_dim]: causal attention of new query rows over their sequences' cached prefixes, read in place from one layer's
    slice of the KV cache (k_cache / v_cache fp16 [batch, n_kv_heads, max_seq, head_dim], keys after RoPE; see gptq_cached_attention_gqa).
    `spans` lists (seq, start, rows): the next `rows` rows of q (fp16 [M, n_heads * head_dim], rows may be strided, e.g. the q part of the
    fused qkv output) are sequence seq's positions start .. start + rows - 1, whose K and V rows the caller has already written.
    n_heads is q's width over head_dim and n_kv_heads the caches' head count (grouped-query attention: query head h reads K/V head
    h / (n_heads / n_kv_heads); n_kv_heads = n_heads is multi-head attention)."""
    _require_cuda(q, k_cache, v_cache)
    if q.dim() != 2 or k_cache.dim() != 4 or k_cache.shape != v_cache.shape:
        raise ValueError(f'expected q [M, heads * head_dim] and caches [batch, heads, max_seq, head_dim], got {tuple(q.shape)}, {tuple(k_cache.shape)}, '
                         f'{tuple(v_cache.shape)}')
    if q.dtype != torch.float16 or k_cache.dtype != torch.float16 or v_cache.dtype != torch.float16:
        raise ValueError('cached_attention expects float16 q and caches')
    if not (k_cache.is_contiguous() and v_cache.is_contiguous()):
        raise ValueError('the KV cache slices must be contiguous')
    B, nkv, S, hd = k_cache.shape
    spans = [(int(b), int(s), int(n)) for b, s, n in spans]
    M = sum(n for _, _, n in spans)
    nh = q.shape[1] // hd
    if q.shape[0] != M or q.shape[1] != nh * hd or nh % nkv != 0:
        raise ValueError(f'q has shape {tuple(q.shape)}, the spans need [{M}, n_heads * {hd}] with n_heads a multiple of the cache\'s {nkv} heads')
    out = torch.empty((M, nh * hd), device=q.device, dtype=torch.float16)
    if M == 0:
        return out
    q, ld = _rows(q)
    arr = lambda i: (ctypes.c_int32 * len(spans))(*[sp[i] for sp in spans])
    with torch.cuda.device(q.device):
        check(
            lib.gptq_cached_attention_gqa(q.data_ptr(), ld, k_cache.data_ptr(), v_cache.data_ptr(), B, nh, nkv, hd, S, len(spans), arr(0), arr(1), arr(2),
                                          out.data_ptr(), nh * hd, _stream(q)))
    return out


def sample_tokens(logits, positions, temperature, top_k, top_p, seed, eos_token=None, min_length=None, out=None):
    """int32 [B]: one token per row of the fp16 logits [B, V] (gptq_sample_tokens, the rule in include/gptq_b200.h).  positions int32 [B] are
    the rows' decode positions (the draw's counter); the parameters are device tensors of B entries -- temperature / top_p float32, top_k /
    eos_token / min_length int32, seed int64 (read as uint64) -- eos_token None: no eos."""
    _require_cuda(logits, positions, temperature, top_k, top_p, seed, eos_token, min_length, out)
    if logits.dim() != 2 or logits.dtype != torch.float16 or logits.stride(1) != 1:
        raise ValueError('sample_tokens expects fp16 logits [B, V] with unit column stride')
    B, V = logits.shape
    dev = logits.device
    if eos_token is None:
        eos_token = torch.full((B, ), -1, dtype=torch.int32, device=dev)
    if min_length is None:
        min_length = torch.zeros(B, dtype=torch.int32, device=dev)
    want = dict(positions=(positions, torch.int32), temperature=(temperature, torch.float32), top_k=(top_k, torch.int32), top_p=(top_p, torch.float32),
                seed=(seed, torch.int64), eos_token=(eos_token, torch.int32), min_length=(min_length, torch.int32))
    for name, (t, dt) in want.items():
        if t.dtype != dt or t.numel() != B or not t.is_contiguous():
            raise ValueError(f'{name}: expected a contiguous {dt} tensor of {B} entries')
    out = torch.empty(B, dtype=torch.int32, device=dev) if out is None else out
    prm = _lib.Sampling(temperature=temperature.data_ptr(), top_k=top_k.data_ptr(), top_p=top_p.data_ptr(), seed=seed.data_ptr(),
                        eos_token=eos_token.data_ptr(), min_length=min_length.data_ptr())
    with torch.cuda.device(dev):
        check(lib.gptq_sample_tokens(logits.data_ptr(), _rows(logits)[1], B, V, positions.data_ptr(), ctypes.byref(prm), out.data_ptr(), _stream(logits)))
    return out


def dequant(qweight, scales, qzeros, g_idx, bits, groupsize: int = 0):
    """fp16 [K, N] weight as the kernels see it (for tests / load-time validation)."""
    w = make_qweight(qweight, scales, qzeros, g_idx, bits, groupsize)
    with torch.cuda.device(qweight.device):
        out = torch.empty((w.K, w.N), device=qweight.device, dtype=torch.float16)
        check(lib.gptq_dequant(ctypes.byref(w), out.data_ptr(), w.N, _stream(qweight)))
    return out


def _pack_call(fn, src, bits, fields, out_shape):
    """int32 out_shape = fn(src) for one of the pack / unpack kernels (csrc/pack.cu), which take the [rows, cols] shape `fields` of the
    unpacked side."""
    _require_cuda(src)
    if bits not in SUPPORTED_BITS:
        raise NotImplementedError('Only 2,3,4,8 bits are supported.')
    src = src.to(torch.int32).contiguous()
    with torch.cuda.device(src.device):
        out = torch.empty(out_shape, device=src.device, dtype=torch.int32)
        check(fn(src.data_ptr(), out.data_ptr(), *fields, bits, _stream(src)))
    return out


def pack_qweight(intweight, bits):
    """int32 [K, N] in [0, 2^bits) -> qweight int32 [K/32*bits, N], on the device."""
    K, N = intweight.shape
    return _pack_call(lib.gptq_pack_qweight, intweight, bits, (K, N), (K // 32 * bits, N))


def pack_qzeros(zeros_m1, bits):
    """int32 [G, N] (already minus one) -> qzeros int32 [G, N/32*bits]."""
    G, N = zeros_m1.shape
    return _pack_call(lib.gptq_pack_qzeros, zeros_m1, bits, (G, N), (G, N // 32 * bits))


def unpack_qweight(qweight, bits):
    K, N = qweight.shape[0] * 32 // bits, qweight.shape[1]
    return _pack_call(lib.gptq_unpack_qweight, qweight, bits, (K, N), (K, N))


def unpack_qzeros(qzeros, bits):
    G, N = qzeros.shape[0], qzeros.shape[1] * 32 // bits
    return _pack_call(lib.gptq_unpack_qzeros, qzeros, bits, (G, N), (G, N))


class QLayerWeights:
    """One packed GPTQ layer: (qweight, scales, qzeros, g_idx) with its bit width and groupsize, and `perm`, the input gather
    x'[k'] = x[perm[k']] it expects (None for a stored layer; set on a kernel form with regrouped rows).  The one host object that
    knows the packed layout: the groupsize hint, the kernel form of act-order and 2/3-bit layers, and column / row slices."""

    def __init__(self, qweight, scales, qzeros, g_idx, bits, groupsize, perm=None):
        K = qweight.shape[0] * 32 // bits
        self.qweight, self.scales, self.qzeros = qweight.contiguous(), scales.contiguous(), qzeros.contiguous()
        self.g_idx = g_idx[:K].contiguous()  # the fused qkv g_idx of the reference is 3K long; only the first K entries are read
        self.bits, self.groupsize, self.perm = bits, groupsize, perm

    @functools.cached_property
    def hint(self) -> int:
        """groupsize when g_idx is the trivial k // groupsize map (the kernels then skip the gather), else 0.  One device->host sync, once."""
        return self.groupsize if is_trivial_g_idx(self.g_idx, self.groupsize) else 0

    def parts(self):
        """(qweight, scales, qzeros, g_idx): the layer as matmul248 and fused_mlp take it."""
        return self.qweight, self.scales, self.qzeros, self.g_idx

    def struct(self) -> QWeight:
        return make_qweight(*self.parts(), self.bits, self.hint)

    def kernel_form(self, allow_perm=True):
        """The layer in the layout the tuned int4 kernels (matvec, wgmma GEMM, persistent decode kernel) take, derived at load time for a
        layer they would otherwise leave to the generic kernel.  The stored tensors are not touched.

        * act-order (arbitrary g_idx, gptq.py:210-216) with equal-sized groups, if allow_perm: the packed rows are regrouped so that every
          group is contiguous (k' = rank of k in a stable sort by group); the caller feeds x'[k'] = x[perm[k']] (`.perm`, int64).  Every
          weight keeps its own scale/zero, so the products are the same numbers; only the fp32 summation order changes.
        * bits 2 or 3: every field is widened to a nibble (same integers, same stored-minus-one zeros), i.e. the layer is
          re-expressed in the int4 layout.  This trades 33 % (int3) / 100 % (int2) more weight bytes for the tuned kernels;
          a native 3-bit streaming kernel is the follow-up.

        Returns self when neither applies."""
        _require_cuda(self.qweight)
        K, G, gs = self.g_idx.numel(), self.scales.shape[0], self.groupsize
        perm, rows = None, None
        if not self.hint:
            g = self.g_idx.long()
            if not allow_perm or K % gs or G * gs != K or not bool((torch.bincount(g, minlength=G) == gs).all()):
                return self
            perm = torch.argsort(g, stable=True)
            rows = unpack_qweight(self.qweight, self.bits).index_select(0, perm)
        widen = self.bits in (2, 3)
        if perm is None and not widen:
            return self
        if rows is None:
            rows = unpack_qweight(self.qweight, self.bits)
        bits = 4 if widen else self.bits
        qzeros = pack_qzeros(unpack_qzeros(self.qzeros, self.bits), 4) if widen else self.qzeros
        g_triv = (torch.arange(K, device=self.qweight.device) // gs).to(torch.int32)
        out = QLayerWeights(pack_qweight(rows, bits), self.scales, qzeros, g_triv, bits, gs, perm)
        out.hint = gs  # trivial by construction: no probe
        return out

    def permute_columns(self, perm):
        """The same layer with output columns reordered: out'[:, j] = out[:, perm[j]] (folds the NEXT layer's input gather)."""
        zeros = unpack_qzeros(self.qzeros, self.bits).index_select(1, perm)
        return QLayerWeights(self.qweight.index_select(1, perm), self.scales.index_select(1, perm), pack_qzeros(zeros, self.bits), self.g_idx, self.bits,
                             self.groupsize, self.perm)

    def column_slice(self, cols):
        """The layer restricted to output columns `cols`: out[:, j] = full[:, cols[j]].  `cols` (a LongTensor) is made of whole runs of 32
        consecutive columns starting at multiples of 32, so that every packed zero word is kept whole (bits of them per run)."""
        runs = cols.view(-1, 32) if cols.numel() % 32 == 0 else None
        if runs is None or not bool(((runs[:, :1] % 32 == 0) & (runs - runs[:, :1] == torch.arange(32, device=cols.device))).all()):
            raise ValueError('column shards must be whole runs of 32 columns starting at multiples of 32')
        zcols = (runs[:, :1] // 32 * self.bits + torch.arange(self.bits, device=cols.device)).reshape(-1)
        return QLayerWeights(self.qweight.index_select(1, cols), self.scales.index_select(1, cols), self.qzeros.index_select(1, zcols), self.g_idx, self.bits,
                             self.groupsize, self.perm)

    def row_slice(self, k0, k1):
        """The layer restricted to input features [k0, k1): a K-shard whose partial outputs add up.  Needs the trivial g_idx and
        boundaries on whole quantisation groups and whole packed words."""
        gs, bits = self.groupsize, self.bits
        if not self.hint:
            raise ValueError('row sharding of act-order layers is not supported (scales/zeros would have to be replicated)')
        if k0 % gs or k1 % gs or k0 * bits % 32 or k1 * bits % 32:
            raise ValueError(f'row shard [{k0}, {k1}) does not keep whole groups of {gs} and whole packed words')
        g = (torch.arange(k1 - k0, device=self.g_idx.device) // gs).to(torch.int32)
        return QLayerWeights(self.qweight[k0 * bits // 32:k1 * bits // 32], self.scales[k0 // gs:k1 // gs], self.qzeros[k0 // gs:k1 // gs], g, bits, gs)


def mlp_kernel_form(gate, up, allow_perm=True):
    """Kernel forms (gate', up') of gate_proj and up_proj (QLayerWeights.kernel_form).  The two see the same input, so they must share
    one input gather: None when their act-order maps differ."""
    kg, ku = gate.kernel_form(allow_perm), up.kernel_form(allow_perm)
    if (kg.perm is None) != (ku.perm is None) or (kg.perm is not None and not torch.equal(kg.perm, ku.perm)):
        return None
    return kg, ku
