"""CPU: grouped-query attention on the host -- the K/V head count read from HF configs, the quant-module surgery of a GQA model, the C ABI's
rule that derives the count from the fused qkv width (rejections return before any CUDA call), and the refusal of tensor parallelism for
GQA models before any device work."""
import ctypes
import types

import pytest
import torch

P = 0x100000  # a fake, 256-byte aligned device pointer: every call below is rejected during validation


def _gqa_config(heads=4, kv=2, **kw):
    from transformers import LlamaConfig
    return LlamaConfig(hidden_size=64 * heads, intermediate_size=256, num_hidden_layers=2, num_attention_heads=heads, num_key_value_heads=kv,
                       vocab_size=128, max_position_embeddings=64, **kw)


def test_kv_heads_from_config():
    from quant.fused_attn import kv_heads_from_config
    assert kv_heads_from_config(_gqa_config(8, 2)) == 2
    assert kv_heads_from_config(_gqa_config(8, 8)) == 8
    # a config written before grouped-query attention (transformers < 4.31) has no num_key_value_heads: one K/V head per head
    assert kv_heads_from_config(types.SimpleNamespace(num_attention_heads=32)) == 32
    assert kv_heads_from_config(types.SimpleNamespace(num_attention_heads=32, num_key_value_heads=None)) == 32
    # the LLaMA-3.1 rope type stays refused, grouped-query or not
    from quant.fused_attn import rope_base_from_config
    cfg = types.SimpleNamespace(rope_theta=5e5, rope_scaling={'rope_type': 'llama3', 'factor': 8.0})
    with pytest.raises(ValueError):
        rope_base_from_config(cfg)


def test_make_quant_attn_on_a_gqa_model():
    """4 query heads, 2 K/V heads: the surgery fuses q (256 columns) with the narrower k and v (128 each) and keeps the head counts."""
    import quant
    import utils
    from transformers import LlamaForCausalLM
    torch.manual_seed(0)
    model = LlamaForCausalLM(_gqa_config(4, 2)).half().eval()
    layers = utils.find_layers(model)
    layers.pop('lm_head')
    quant.make_quant_linear(model, layers, 4, 32)
    quant.make_quant_attn(model)
    for layer in model.model.layers:
        attn = layer.self_attn
        assert isinstance(attn, quant.QuantLlamaAttention)
        assert (attn.num_heads, attn.num_key_value_heads, attn.head_dim) == (4, 2, 64)
        assert attn.qkv_proj.outfeatures == (4 + 2 * 2) * 64
        assert attn.qkv_proj.qweight.shape[1] == 512 and attn.qkv_proj.scales.shape[1] == 512
    with pytest.raises(ValueError):
        quant.QuantLlamaAttention(256, 4, None, None, num_key_value_heads=3)


def _model(heads, widths, tp=None):
    """gptq_llama_model / gptq_llama_state with fake pointers, head_dim 128 and one layer per entry of `widths` (the qkv N)."""
    from gptq_b200 import _lib
    H, I = heads * 128, 512
    layers = (_lib.LlamaLayer * len(widths))()
    for ly, n in zip(layers, widths):
        for name, K, N in (('qkv', H, n), ('o', H, H), ('gate', H, I), ('up', H, I), ('down', I, H)):
            w = getattr(ly, name)
            w.qweight = w.scales = w.qzeros = w.g_idx = P
            w.K, w.N, w.G, w.bits, w.groupsize = K, N, K // 128, 4, 128
        ly.input_norm = ly.post_norm = P
    m = _lib.LlamaModel()
    m.n_layers, m.hidden, m.n_heads, m.head_dim, m.intermediate, m.vocab, m.rms_eps, m.rope_base = len(widths), H, heads, 128, I, 256, 1e-6, 1e4
    m.layers = ctypes.cast(layers, ctypes.POINTER(_lib.LlamaLayer))
    m.embed = m.final_norm = m.lm_head = P
    st = _lib.LlamaState()
    st.batch, st.max_seq = 1, 64
    st.k_cache = st.v_cache = st.tokens = st.positions = st.logits = st.scratch = P
    st.scratch_bytes = _lib.lib.gptq_llama_scratch_bytes(ctypes.byref(m), 1, 64)
    assert st.scratch_bytes > 0
    if tp is not None:
        st.tp = ctypes.pointer(tp)
    return m, st, layers


@pytest.mark.parametrize('widths', [
    [5 * 128],              # 4 heads + 2 * 0.5: odd remainder
    [4 * 128],              # no K/V heads
    [(4 + 2 * 3) * 128],    # 3 K/V heads do not divide 4 query heads
    [8 * 128 + 64],         # not a whole number of heads
    [8 * 128, 6 * 128],     # the layers disagree (2 and 1 K/V heads)
    [6 * 128, 12 * 128],
], ids=['odd', 'zero', 'non-divisor', 'partial-head', 'layers-disagree', 'layers-disagree-mha'])
def test_decode_step_rejects_qkv_widths_without_a_valid_kv_head_count(widths):
    from gptq_b200 import _lib
    m, st, _keep = _model(4, widths)
    assert _lib.lib.gptq_llama_decode_step(ctypes.byref(m), ctypes.byref(st), None) == _lib.ERR_SHAPE


def test_scratch_size_does_not_depend_on_the_kv_head_count():
    """The qkv scratch is sized for 3 * hidden, an upper bound of every valid width, without reading the layers."""
    from gptq_b200 import _lib
    sizes = {_lib.lib.gptq_llama_scratch_bytes(ctypes.byref(_model(8, [n])[0]), 2, 128) for n in ((8 + 2 * kv) * 128 for kv in (1, 2, 4, 8))}
    assert len(sizes) == 1


def test_tensor_parallel_gqa_is_refused():
    from gptq_b200 import _lib, engine
    from gptq_b200.ops import QLayerWeights
    # C ABI: a GQA shard under tensor parallelism is refused before any CUDA call
    tp = _lib.LlamaTP()
    tp.size, tp.rank, tp.vocab_begin, tp.vocab_end = 2, 0, 0, 128
    m, st, _keep = _model(4, [8 * 128], tp=tp)
    assert _lib.lib.gptq_llama_decode_step(ctypes.byref(m), ctypes.byref(st), None) == _lib.ERR_UNSUPPORTED
    # host: shard_for_rank, LlamaDecoder(tp=...) and synthetic_llama_tp raise ValueError before touching a device (CPU tensors / no draw)
    H, hd, nh, nkv = 512, 128, 4, 2
    q = lambda N: QLayerWeights(torch.zeros(H // 8, N, dtype=torch.int32), torch.zeros(H // 128, N, dtype=torch.float16),
                                torch.zeros(H // 128, N // 8, dtype=torch.int32), torch.zeros(H, dtype=torch.int32), 4, 128)
    layer = dict(qkv=q((nh + 2 * nkv) * hd), o=q(H), gate=q(1024), up=q(1024), down=q(H), input_norm=torch.ones(H).half(), post_norm=torch.ones(H).half())
    lm_head = torch.zeros(256, H, dtype=torch.float16)
    with pytest.raises(ValueError, match='tensor parallelism'):
        engine.shard_for_rank([layer], lm_head, nh, hd, 0, 2)
    with pytest.raises(ValueError, match='tensor parallelism'):
        engine.LlamaDecoder([layer], lm_head, torch.ones(H).half(), lm_head, nh, head_dim=hd, tp=(0, 2, 0, 128), n_kv_heads=nkv)
    with pytest.raises(ValueError, match='tensor parallelism'):
        engine.synthetic_llama_tp('70b', 0, 2, device='cpu')


def test_decoder_checks_the_kv_head_count_against_the_qkv_width():
    from gptq_b200 import engine
    from gptq_b200.ops import QLayerWeights
    H, nh = 512, 4
    q = lambda N: QLayerWeights(torch.zeros(H // 8, N, dtype=torch.int32), torch.zeros(H // 128, N, dtype=torch.float16),
                                torch.zeros(H // 128, N // 8, dtype=torch.int32), torch.zeros(H, dtype=torch.int32), 4, 128)
    layer = dict(qkv=q(8 * 128), o=q(H), gate=q(1024), up=q(1024), down=q(H), input_norm=torch.ones(H).half(), post_norm=torch.ones(H).half())
    embed = torch.zeros(256, H, dtype=torch.float16)
    for kv in (None, 1, 4):  # the width says 2 K/V heads
        with pytest.raises(ValueError, match='fused qkv'):
            engine.LlamaDecoder([layer], embed, torch.ones(H).half(), embed, nh, n_kv_heads=kv)
    with pytest.raises(ValueError, match='divisor'):
        engine.LlamaDecoder([layer], embed, torch.ones(H).half(), embed, nh, n_kv_heads=3)


def test_named_shapes():
    from gptq_b200 import engine
    assert all(len(v) == 4 for v in engine.LLAMA_SHAPES.values())
    assert set(engine.KV_HEADS) <= set(engine.LLAMA_SHAPES)
    for size, nkv in engine.KV_HEADS.items():
        H, I, L, nh = engine.LLAMA_SHAPES[size]
        assert nh % nkv == 0 and H // nh == 128 and L <= 80 and H <= 8192 and I <= 32768
    assert engine.kv_heads('7b') == 32 and engine.kv_heads('70b') == 8
    # the shapes the persistent kernel serves: qkv width and MLP width in whole 256-column slabs
    for size in ('70b', '34b', 'llama3-8b', 'tiny-gqa2', 'tiny-gqa1'):
        H, I, _, nh = engine.LLAMA_SHAPES[size]
        assert (nh + 2 * engine.kv_heads(size)) * 128 % 256 == 0 and I % 256 == 0
    assert all(engine.LLAMA_SHAPES[s][1] % 256 != 0 for s in ('tiny-gqa2-chain', 'tiny-gqa1-chain'))


def test_quant_attention_equals_hf_attention_with_repeat_kv(monkeypatch):
    """QuantLlamaAttention (fused q | k | v of 4 query and 2 K/V heads, SDPA with enable_gqa) against HF's LlamaAttention (separate
    projections, repeat_kv) on the same fp32 weights, for a prefill and then a step on the cache.  The RoPE op is replaced by an fp32
    restatement of it, because the kernel stores the rotated q and k in fp16, which HF's fp32 attention does not: with that rounding taken
    out, the two must agree to fp32 rounding."""
    import copy
    import math

    import quant.fused_attn as FA
    from transformers import LlamaForCausalLM

    def rope_fp32(qk, position_ids, base=10000.0):
        half = qk.shape[-1] // 2
        f = position_ids[:, :, None].double() * torch.exp(torch.arange(half, dtype=torch.float64) * (-2 * math.log(base) / qk.shape[-1]))
        c, s = torch.cos(f)[:, :, None, None].float(), torch.sin(f)[:, :, None, None].float()
        x, y = qk[..., :half].clone(), qk[..., half:].clone()
        qk[..., :half] = x * c - y * s
        qk[..., half:] = x * s + y * c

    monkeypatch.setattr(FA.ops, 'rotate_half_', rope_fp32)
    torch.manual_seed(0)
    cfg = _gqa_config(4, 2)
    cfg.hidden_size, cfg.head_dim = 512, 128
    hf = LlamaForCausalLM(cfg).float().eval()
    fused = copy.deepcopy(hf)
    for layer in fused.model.layers:
        a = layer.self_attn
        qkv = torch.nn.Linear(512, (4 + 2 * 2) * 128, bias=False)
        qkv.weight.data = torch.cat([a.q_proj.weight, a.k_proj.weight, a.v_proj.weight], 0)
        layer.self_attn = FA.QuantLlamaAttention(512, 4, qkv, a.o_proj, layer_idx=a.layer_idx, rope_base=FA.rope_base_from_config(cfg),
                                                 num_key_value_heads=FA.kv_heads_from_config(cfg))
    ids = torch.randint(0, cfg.vocab_size, (2, 9), generator=torch.Generator().manual_seed(1))
    with torch.no_grad():
        ref = hf(ids).logits
        out = fused(ids[:, :8], use_cache=True)
        step = fused(ids[:, 8:], past_key_values=out.past_key_values, use_cache=True)
    assert out.past_key_values.layers[0].keys.shape == (2, 2, 9, 128), 'the cache holds the 2 K/V heads of the 9 positions'
    torch.testing.assert_close(out.logits, ref[:, :8], rtol=1e-4, atol=1e-5)
    torch.testing.assert_close(step.logits[:, 0], ref[:, 8], rtol=1e-4, atol=1e-5)
