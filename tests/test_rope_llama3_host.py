"""CPU: the llama3 RoPE frequency scaling of LLaMA-3.1 / 3.2 / 3.3 on the host -- the frequency table against HF's, bit for bit, its
validation, the three config conventions, the quant-module surgery, the decoder's refusal of layers whose tables disagree, and the C ABI's
rejection of bad tables (every call below returns during validation, before any CUDA call)."""
import ctypes
import math
import types

import pytest
import torch

P = 0x100000  # a fake, 256-byte aligned device pointer

LLAMA3_1 = {'rope_type': 'llama3', 'factor': 8.0, 'low_freq_factor': 1.0, 'high_freq_factor': 4.0, 'original_max_position_embeddings': 8192}
LLAMA3_2 = dict(LLAMA3_1, factor=32.0)


def hf_table(base, head_dim, scaling):
    """HF's own llama3 inv_freq (ROPE_INIT_FUNCTIONS['llama3']) for a config with this base, head_dim and scaling dict."""
    from transformers import LlamaConfig
    from transformers.modeling_rope_utils import ROPE_INIT_FUNCTIONS
    old = scaling['original_max_position_embeddings']
    cfg = LlamaConfig(hidden_size=head_dim * 2, num_attention_heads=2, head_dim=head_dim, max_position_embeddings=math.ceil(2 * old) + 64,
                      rope_parameters=dict(scaling, rope_theta=base))
    return ROPE_INIT_FUNCTIONS['llama3'](cfg, 'cpu')[0]


def _edge_scaling(base, head_dim, i, edge):
    """A scaling dict whose low (edge='low') or high (edge='high') wavelength bound equals the wavelength of frequency i exactly, as HF
    compares them: 2 pi / fp32 inv_freq[i] (a float64 scalar over an fp32 tensor, rounded to fp32) against old_context / factor."""
    inv = 1.0 / (base**(torch.arange(0, head_dim, 2, dtype=torch.int64).float() / head_dim))
    wl = float((2 * math.pi / inv)[i])
    if edge == 'low':
        return {'rope_type': 'llama3', 'factor': 8.0, 'low_freq_factor': 1.0, 'high_freq_factor': 4.0, 'original_max_position_embeddings': wl}
    return {'rope_type': 'llama3', 'factor': 8.0, 'low_freq_factor': 0.25, 'high_freq_factor': 1.0, 'original_max_position_embeddings': wl}


@pytest.mark.parametrize('base', [5e5, 1e4])
@pytest.mark.parametrize('name,scaling', [('3.1', LLAMA3_1), ('3.2', LLAMA3_2), ('small-context', dict(LLAMA3_1, original_max_position_embeddings=64))])
def test_table_equals_hf_bit_for_bit(base, name, scaling):
    from gptq_b200 import ops
    got, ref = ops.rope_inv_freq(base, 128, scaling), hf_table(base, 128, scaling)
    assert got.dtype == torch.float32 and got.shape == (64, )
    assert torch.equal(got.view(torch.int32), ref.view(torch.int32)), f'{name} base {base}'


def test_small_context_puts_many_frequencies_in_the_blended_band():
    from gptq_b200 import ops
    t = ops.rope_inv_freq(1e4, 128, dict(LLAMA3_1, original_max_position_embeddings=64))
    plain = 1.0 / (1e4**(torch.arange(0, 128, 2).float() / 128))
    blended = ((t != plain) & (t != plain / 8)).sum().item()
    assert blended >= 8, blended


@pytest.mark.parametrize('edge', ['low', 'high'])
@pytest.mark.parametrize('i', [10, 40])
def test_table_at_a_band_edge(edge, i):
    """A frequency exactly on a band edge (HF's comparisons are strict): still HF's value, bit for bit."""
    from gptq_b200 import ops
    scaling = _edge_scaling(1e4, 128, i, edge)
    got, ref = ops.rope_inv_freq(1e4, 128, scaling), hf_table(1e4, 128, scaling)
    assert torch.equal(got.view(torch.int32), ref.view(torch.int32))


@pytest.mark.parametrize('bad', [
    dict(LLAMA3_1, factor=0.0), dict(LLAMA3_1, factor=-8.0), dict(LLAMA3_1, low_freq_factor=4.0), dict(LLAMA3_1, low_freq_factor=5.0),
    dict(LLAMA3_1, low_freq_factor=0.0), dict(LLAMA3_1, original_max_position_embeddings=0), dict(LLAMA3_1, original_max_position_embeddings=-1),
    dict(LLAMA3_1, factor=float('nan')), dict(LLAMA3_1, high_freq_factor=float('inf')), dict(LLAMA3_1, factor='8'), {'rope_type': 'llama3'},
    {k: v for k, v in LLAMA3_1.items() if k != 'high_freq_factor'}, dict(LLAMA3_1, low_freq_factor=None), dict(LLAMA3_1, rope_type='yarn'),
    {'type': 'linear', 'factor': 2.0}
], ids=lambda d: ','.join(f'{k}={v}' for k, v in d.items() if k != 'rope_type') or 'empty')
def test_invalid_scaling_raises(bad):
    from gptq_b200 import ops
    with pytest.raises(ValueError):
        ops.rope_inv_freq(5e5, 128, bad)


def test_unscaled_gives_no_table():
    from gptq_b200 import ops
    assert ops.rope_inv_freq(1e4, 128, None) is None and ops.rope_inv_freq(1e4, 128, {'rope_type': 'default'}) is None


def test_llama3_table_differs_from_the_default_in_the_low_and_blended_bands_only():
    """Tooth: the scaling keeps every frequency whose wavelength is below 8192 / 4 = 2048 positions and changes all the others."""
    from gptq_b200 import ops
    t = ops.rope_inv_freq(5e5, 128, LLAMA3_1)
    plain = 1.0 / (5e5**(torch.arange(0, 128, 2).float() / 128))
    wl = 2 * math.pi / plain
    high, low = wl < 2048, wl > 8192
    assert high.any() and low.any() and (~high & ~low).any()
    assert torch.equal(t[high], plain[high])
    assert torch.equal(t[low], plain[low] / 8)
    assert (t[~high] != plain[~high]).all() and (t[~high] < plain[~high]).all()


# ----------------------------------------------------------------------------------------------- config conventions and the quant modules
def test_rope_from_config_under_every_convention():
    from transformers import LlamaConfig
    from quant.fused_attn import rope_from_config
    from gptq_b200 import ops
    ref = ops.rope_inv_freq(5e5, 128, LLAMA3_1)
    hf5 = LlamaConfig(hidden_size=4096, num_attention_heads=32, max_position_embeddings=131072, rope_parameters=dict(LLAMA3_1, rope_theta=5e5))
    by_rope_type = types.SimpleNamespace(hidden_size=4096, num_attention_heads=32, rope_theta=5e5, rope_scaling=dict(LLAMA3_1))
    by_type = types.SimpleNamespace(hidden_size=4096, num_attention_heads=32, rope_theta=5e5,
                                    rope_scaling={('type' if k == 'rope_type' else k): v for k, v in LLAMA3_1.items()})
    for cfg in (hf5, by_rope_type, by_type):
        base, table = rope_from_config(cfg)
        assert base == 5e5 and torch.equal(table, ref)
    head_dim = types.SimpleNamespace(hidden_size=3072, num_attention_heads=24, head_dim=128, rope_theta=5e5, rope_scaling=dict(LLAMA3_2))
    assert torch.equal(rope_from_config(head_dim)[1], ops.rope_inv_freq(5e5, 128, LLAMA3_2))
    assert rope_from_config(LlamaConfig(rope_theta=1e6)) == (1e6, None)
    assert rope_from_config(types.SimpleNamespace()) == (10000.0, None)
    for rope_type in ('linear', 'dynamic', 'yarn'):
        for cfg in (types.SimpleNamespace(rope_theta=1e4, rope_scaling={'type': rope_type, 'factor': 2.0}),
                    types.SimpleNamespace(rope_theta=1e4, rope_scaling={'rope_type': rope_type, 'factor': 2.0}),
                    types.SimpleNamespace(rope_parameters={'rope_type': rope_type, 'factor': 2.0, 'rope_theta': 1e4})):
            with pytest.raises(ValueError, match=rope_type):
                rope_from_config(cfg)


def _tiny_llama3(**kw):
    from transformers import LlamaConfig, LlamaForCausalLM
    cfg = LlamaConfig(hidden_size=256, intermediate_size=256, num_hidden_layers=2, num_attention_heads=2, num_key_value_heads=1, vocab_size=128,
                      max_position_embeddings=512, rope_parameters=dict(LLAMA3_1, original_max_position_embeddings=64, rope_theta=5e5), **kw)
    torch.manual_seed(0)
    return LlamaForCausalLM(cfg).half().eval()


def _surgery(model):
    import quant
    import utils
    layers = utils.find_layers(model)
    layers.pop('lm_head')
    quant.make_quant_linear(model, layers, 4, 32)
    quant.make_quant_attn(model)
    return model


def test_make_quant_attn_sets_each_layers_table():
    from gptq_b200 import ops
    model = _surgery(_tiny_llama3())
    ref = ops.rope_inv_freq(5e5, 128, dict(LLAMA3_1, original_max_position_embeddings=64))
    for layer in model.model.layers:
        attn = layer.self_attn
        assert attn.rope_base == 5e5 and torch.equal(attn.rope_inv_freq, ref)
        assert attn.rope_inv_freq.dtype == torch.float32 and attn.rope_inv_freq.device.type == 'cpu'
    model.half()
    assert model.model.layers[0].self_attn.rope_inv_freq.dtype == torch.float32, 'casting the model must not round the table'


def test_decoder_refuses_layers_whose_tables_disagree():
    from gptq_b200 import engine
    model = _surgery(_tiny_llama3())
    model.model.layers[1].self_attn.rope_inv_freq[5] *= 2
    with pytest.raises(ValueError, match='disagree'):
        engine.from_hf_quant_model(model)
    model.model.layers[1].self_attn.rope_inv_freq = None
    with pytest.raises(ValueError, match='disagree'):
        engine.from_hf_quant_model(model)


def test_named_llama3_shapes_and_scalings():
    from gptq_b200 import engine
    assert engine.LLAMA_SHAPES['llama3.2-3b'] == (3072, 8192, 28, 24) and engine.kv_heads('llama3.2-3b') == 8
    assert engine.LLAMA3_1_ROPE_SCALING == LLAMA3_1 and engine.LLAMA3_3_ROPE_SCALING == LLAMA3_1 and engine.LLAMA3_2_ROPE_SCALING == LLAMA3_2
    assert engine.LLAMA3_ROPE_BASE == 5e5


def test_decoder_refuses_a_bad_table_before_device_work():
    from gptq_b200 import engine
    from gptq_b200.ops import QLayerWeights
    H, nh = 512, 4
    q = lambda N: QLayerWeights(torch.zeros(H // 8, N, dtype=torch.int32), torch.zeros(H // 128, N, dtype=torch.float16),
                                torch.zeros(H // 128, N // 8, dtype=torch.int32), torch.zeros(H, dtype=torch.int32), 4, 128)
    layer = dict(qkv=q(8 * 128), o=q(H), gate=q(1024), up=q(1024), down=q(H), input_norm=torch.ones(H).half(), post_norm=torch.ones(H).half())
    embed = torch.zeros(256, H, dtype=torch.float16)
    for table in (torch.ones(63), torch.zeros(64), torch.full((64, ), float('nan'))):
        with pytest.raises(ValueError, match='frequency table'):
            engine.LlamaDecoder([layer], embed, torch.ones(H).half(), embed, nh, n_kv_heads=2, rope_scaling=table)
    with pytest.raises(ValueError, match='yarn'):
        engine.LlamaDecoder([layer], embed, torch.ones(H).half(), embed, nh, n_kv_heads=2, rope_scaling={'rope_type': 'yarn', 'factor': 4.0})


# ----------------------------------------------------------------------------------------------- C ABI validation
def _table(values):
    return (ctypes.c_float * len(values))(*values)


BAD_TABLES = {'zero': 0.0, 'negative': -1e-3, 'nan': float('nan'), 'inf': float('inf')}


@pytest.mark.parametrize('bad', list(BAD_TABLES), ids=list(BAD_TABLES))
def test_rope_inplace_freq_rejects_bad_tables(bad):
    from gptq_b200 import _lib
    lib = _lib.lib
    good = [1.0 / (i + 1) for i in range(64)]
    for i in (0, 37, 63):
        t = list(good)
        t[i] = BAD_TABLES[bad]
        assert lib.gptq_rope_inplace_freq(P, 2 * 4 * 128, P, 1, 1, 1, 8, 128, _table(t), None) == _lib.ERR_SHAPE


def test_rope_inplace_freq_validation():
    from gptq_b200 import _lib
    lib = _lib.lib
    good = _table([1.0 / (i + 1) for i in range(64)])
    assert lib.gptq_rope_inplace_freq(P, 1024, P, 1, 1, 1, 8, 128, None, None) == _lib.ERR_NULL  # the table is required
    assert lib.gptq_rope_inplace_freq(None, 1024, P, 1, 1, 1, 8, 128, good, None) == _lib.ERR_NULL
    assert lib.gptq_rope_inplace_freq(P, 1024, None, 1, 1, 1, 8, 128, good, None) == _lib.ERR_NULL
    assert lib.gptq_rope_inplace_freq(P, 10, P, 1, 1, 1, 8, 128, good, None) == _lib.ERR_SHAPE  # token stride < rows * head_dim
    assert lib.gptq_rope_inplace_freq(P, 4096, P, 1, 1, 1, 8, 256, _table([1.0] * 128), None) == _lib.ERR_UNSUPPORTED  # head_dim > 128
    assert lib.gptq_rope_inplace_freq(P, 1024, P, 1, 0, 1, 8, 128, good, None) == _lib.OK  # no tokens: nothing to do
    # a 32-wide head reads only its 16 entries
    assert lib.gptq_rope_inplace_freq(P, 256, P, 1, 0, 1, 8, 32, _table([1.0] * 16 + [float('nan')] * 48), None) == _lib.OK


def _model():
    """gptq_llama_model / gptq_llama_state with fake pointers (one multi-head layer, head_dim 128): valid up to the first CUDA call."""
    from gptq_b200 import _lib
    H, I = 4 * 128, 512
    layers = (_lib.LlamaLayer * 1)()
    for name, K, N in (('qkv', H, 3 * H), ('o', H, H), ('gate', H, I), ('up', H, I), ('down', I, H)):
        w = getattr(layers[0], name)
        w.qweight = w.scales = w.qzeros = w.g_idx = P
        w.K, w.N, w.G, w.bits, w.groupsize = K, N, K // 128, 4, 128
    layers[0].input_norm = layers[0].post_norm = P
    m = _lib.LlamaModel()
    m.n_layers, m.hidden, m.n_heads, m.head_dim, m.intermediate, m.vocab, m.rms_eps, m.rope_base = 1, H, 4, 128, I, 256, 1e-6, 1e4
    m.layers = ctypes.cast(layers, ctypes.POINTER(_lib.LlamaLayer))
    m.embed = m.final_norm = m.lm_head = P
    st = _lib.LlamaState()
    st.batch, st.max_seq = 1, 64
    st.k_cache = st.v_cache = st.tokens = st.positions = st.logits = st.scratch = P
    st.scratch_bytes = _lib.lib.gptq_llama_scratch_bytes(ctypes.byref(m), 1, 64)
    return m, st, layers


@pytest.mark.parametrize('bad', list(BAD_TABLES), ids=list(BAD_TABLES))
def test_decode_step_rope_rejects_bad_tables(bad):
    from gptq_b200 import _lib
    m, st, _keep = _model()
    t = [1.0 / (i + 1) for i in range(64)]
    t[63] = BAD_TABLES[bad]
    assert _lib.lib.gptq_llama_decode_step_rope(ctypes.byref(m), ctypes.byref(st), _table(t), None) == _lib.ERR_SHAPE


def test_decode_step_rope_null_checks_come_first():
    from gptq_b200 import _lib
    lib = _lib.lib
    m, st, _keep = _model()
    good = _table([1.0 / (i + 1) for i in range(64)])
    assert lib.gptq_llama_decode_step_rope(None, ctypes.byref(st), good, None) == _lib.ERR_NULL
    assert lib.gptq_llama_decode_step_rope(ctypes.byref(m), None, good, None) == _lib.ERR_NULL
    st.logits = None
    assert lib.gptq_llama_decode_step_rope(ctypes.byref(m), ctypes.byref(st), good, None) == _lib.ERR_NULL
    assert lib.gptq_llama_decode_step(ctypes.byref(m), ctypes.byref(st), None) == _lib.ERR_NULL
