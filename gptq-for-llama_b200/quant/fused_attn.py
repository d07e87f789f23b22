"""Fused-QKV attention block: one packed QKV projection, in-place RoPE kernel, KV cache, SDPA, o_proj.

Mirrors quant/fused_attn.py of the reference (triton_rotate_half_ :61-93, QuantLlamaAttention
:96-161, make_quant_attn :164-204).  The reference was written against transformers ~4.28; the
module below accepts that calling convention (tuple ``past_key_value``, 3-tuple return) AND the
convention of current transformers (``past_key_values`` Cache object, 2-tuple return), because
the decoder layer that calls it is third-party code.
"""
import torch
from torch import nn
from torch.nn import functional as F

from gptq_b200 import ops
from .quant_linear import QuantLinear

try:
    from transformers.models.llama.modeling_llama import LlamaAttention
except Exception:  # pragma: no cover
    LlamaAttention = ()


def triton_rotate_half_(qk, position_ids, config=None):
    """In-place rotary embedding on qk[bsz, seq, 2, heads, head_dim] (reference name, :61; CUDA kernel
    gptq_rope_inplace).  `config` (Triton block sizes) is accepted and ignored."""
    ops.rotate_half_(qk, position_ids)


def rope_base_from_config(config):
    """The RoPE base (theta) an HF LLaMA config asks for: rope_parameters['rope_theta'] (transformers >= 5), else rope_theta
    (transformers 4.31 - 4.x), else 10000.  The kernels rotate by theta^(-2i/d) * pos on integer positions only, so a config
    whose rope type is anything but 'default' (linear, dynamic, yarn, llama3, ...) raises ValueError instead of decoding
    as if it were unscaled."""
    params = getattr(config, 'rope_parameters', None)
    if params is None:  # transformers 4.x: rope_theta beside an optional rope_scaling dict ('type' before 4.45, 'rope_type' after)
        scaling = getattr(config, 'rope_scaling', None) or {}
        params = {'rope_theta': getattr(config, 'rope_theta', None), 'rope_type': scaling.get('rope_type', scaling.get('type', 'default'))}
    rope_type = params.get('rope_type', 'default')
    if rope_type != 'default':
        raise ValueError(f"RoPE type {rope_type!r} is not supported: only 'default' (unscaled) rotary embeddings are computed")
    base = params.get('rope_theta')
    return 10000.0 if base is None else float(base)


def kv_heads_from_config(config):
    """K/V heads an HF LLaMA config asks for: num_key_value_heads (transformers >= 4.31, and 5.x), else -- older configs, which predate
    grouped-query attention -- one per attention head."""
    return getattr(config, 'num_key_value_heads', None) or config.num_attention_heads


class QuantLlamaAttention(nn.Module):
    """Multi-headed attention from 'Attention Is All You Need' paper, and grouped-query attention (num_key_value_heads < num_heads: query head h
    reads K/V head h / (num_heads / num_key_value_heads)).  qkv_proj is the fused q | k | v projection of num_heads + 2 num_key_value_heads
    heads; the cache holds num_key_value_heads heads."""

    def __init__(self, hidden_size, num_heads, qkv_proj, o_proj, layer_idx=None, rope_base=10000.0, num_key_value_heads=None):
        super().__init__()
        self.hidden_size = hidden_size
        self.num_heads = num_heads
        self.num_key_value_heads = num_heads if num_key_value_heads is None else num_key_value_heads
        self.head_dim = hidden_size // num_heads
        self.layer_idx = layer_idx
        self.rope_base = float(rope_base)
        if (self.head_dim * num_heads) != self.hidden_size:
            raise ValueError(f"hidden_size must be divisible by num_heads (got `hidden_size`: {self.hidden_size}"
                             f" and `num_heads`: {num_heads}).")
        if self.num_key_value_heads < 1 or num_heads % self.num_key_value_heads != 0:
            raise ValueError(f'num_key_value_heads ({self.num_key_value_heads}) must divide num_heads ({num_heads})')
        self.qkv_proj = qkv_proj
        self.o_proj = o_proj

    def forward(self, hidden_states, past_key_value=None, attention_mask=None, position_ids=None, output_attentions=False, use_cache=False,
                past_key_values=None, position_embeddings=None, **kwargs):
        """Input shape: Batch x Time x Channel.  Like the reference, `attention_mask` is ignored (:154-155)."""
        bsz, q_len, _ = hidden_states.size()
        modern = past_key_values is not None and hasattr(past_key_values, 'update')  # transformers Cache object
        if past_key_values is not None and not modern:
            past_key_value = past_key_values

        past_len = 0
        if modern:
            past_len = int(past_key_values.get_seq_length(self.layer_idx))
        elif past_key_value is not None:
            past_len = past_key_value[0].shape[-2]
        if position_ids is None:
            position_ids = torch.arange(past_len, past_len + q_len, device=hidden_states.device, dtype=torch.long).unsqueeze(0).expand(bsz, -1).contiguous()

        nh, nkv = self.num_heads, self.num_key_value_heads
        qkv_states = self.qkv_proj(hidden_states)
        qkv_states = qkv_states.view(bsz, q_len, nh + 2 * nkv, self.head_dim)  # q | k | v heads
        ops.rotate_half_(qkv_states[:, :, :nh + nkv].unsqueeze(2), position_ids, base=self.rope_base)  # q and k rotated in place (:126)

        query_states, key_states, value_states = (t.transpose(1, 2) for t in torch.split(qkv_states, [nh, nkv, nkv], dim=2))
        del qkv_states
        sdpa = dict(enable_gqa=True) if nkv != nh else {}

        if modern:
            key_states, value_states = past_key_values.update(key_states, value_states, self.layer_idx)
        elif past_key_value is not None:
            key_states = torch.cat([past_key_value[0], key_states], dim=2)
            value_states = torch.cat([past_key_value[1], value_states], dim=2)
        if use_cache and not modern:
            key_states, value_states, query_states = key_states.contiguous(), value_states.contiguous(), query_states.contiguous()
        present = (key_states, value_states) if (use_cache and not modern) else None

        kv_len = key_states.shape[-2]
        if kv_len == q_len:
            attn_output = F.scaled_dot_product_attention(query_states, key_states, value_states, is_causal=q_len > 1, **sdpa)
        elif q_len == 1:
            attn_output = F.scaled_dot_product_attention(query_states, key_states, value_states, is_causal=False, **sdpa)
        else:  # chunked prefill on top of a cache: bottom-right aligned causal mask
            mask = torch.ones(q_len, kv_len, dtype=torch.bool, device=hidden_states.device).tril(diagonal=kv_len - q_len)
            attn_output = F.scaled_dot_product_attention(query_states, key_states, value_states, attn_mask=mask, **sdpa)
        del query_states, key_states, value_states

        attn_output = attn_output.transpose(1, 2).reshape(bsz, q_len, self.hidden_size)
        attn_output = self.o_proj(attn_output)
        if modern or position_embeddings is not None:
            return attn_output, None
        return attn_output, None, present


def fuse_qkv(q_proj, k_proj, v_proj):
    """Concatenate three QuantLinear layers that share their input into one (reference :177-188).

    qweight/qzeros/scales are concatenated along N.  g_idx: q, k and v see the same input, hence the
    same act-order; the reference concatenates the three g_idx vectors and its kernel reads only the
    first K entries (:180) -- we keep the first K entries and verify the three maps are equal.
    """
    if not (q_proj.bits == k_proj.bits == v_proj.bits and q_proj.groupsize == k_proj.groupsize == v_proj.groupsize
            and q_proj.infeatures == k_proj.infeatures == v_proj.infeatures):
        raise ValueError('q/k/v projections must share bits, groupsize and infeatures')
    if not (torch.equal(q_proj.g_idx, k_proj.g_idx) and torch.equal(q_proj.g_idx, v_proj.g_idx)):
        raise ValueError('q/k/v projections have different g_idx; they cannot be fused')
    has_bias = q_proj.bias is not None
    qkv = QuantLinear(q_proj.bits, q_proj.groupsize, q_proj.infeatures, q_proj.outfeatures + k_proj.outfeatures + v_proj.outfeatures, has_bias)
    qkv.qweight = torch.cat([q_proj.qweight, k_proj.qweight, v_proj.qweight], dim=1)
    qkv.qzeros = torch.cat([q_proj.qzeros, k_proj.qzeros, v_proj.qzeros], dim=1)
    qkv.scales = torch.cat([q_proj.scales, k_proj.scales, v_proj.scales], dim=1)
    qkv.g_idx = q_proj.g_idx.clone()
    if has_bias:
        qkv.bias = torch.cat([q_proj.bias, k_proj.bias, v_proj.bias], dim=0)
    return qkv


def make_quant_attn(model):
    """Replace all LlamaAttention modules with QuantLlamaAttention modules, fusing the q, k, v projections (k and v are narrower than q under
    grouped-query attention).  Only the 'default' RoPE type is accepted (rope_base_from_config)."""
    if not LlamaAttention:
        return
    targets = [name for name, m in model.named_modules() if isinstance(m, LlamaAttention)]
    for name in targets:
        m = model.get_submodule(name)
        if not all(isinstance(p, QuantLinear) for p in (m.q_proj, m.k_proj, m.v_proj)):
            continue
        cfg = getattr(m, 'config', None)
        hidden_size = getattr(m, 'hidden_size', None) or cfg.hidden_size
        num_heads = getattr(m, 'num_heads', None) or cfg.num_attention_heads
        kv_heads = getattr(m, 'num_key_value_heads', None) or kv_heads_from_config(cfg if cfg is not None else model.config)
        rope_base = rope_base_from_config(cfg if cfg is not None else model.config)
        qkv_layer = fuse_qkv(m.q_proj, m.k_proj, m.v_proj)
        # the rotary embedding module is dropped: RoPE is computed in the kernel from position_ids and the config's base
        attn = QuantLlamaAttention(hidden_size, num_heads, qkv_layer, m.o_proj, layer_idx=getattr(m, 'layer_idx', None), rope_base=rope_base,
                                   num_key_value_heads=kv_heads)
        parent_name, _, child_name = name.rpartition('.')
        parent = model.get_submodule(parent_name) if parent_name else model
        setattr(parent, child_name, attn)
