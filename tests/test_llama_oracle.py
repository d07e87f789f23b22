"""CPU: the reference decoder of llama_oracle.py and the rotation of O.rope_inplace -- grouped-query attention as multi-head attention over
repeated K/V heads, the frequency-table rotation against the base rule and against fp64."""
import math
import types

import numpy as np
import pytest
import torch

import attn_probe as P
from llama_oracle import LINEARS, LlamaOracle
from oracle import gptq_oracle as O

HD = 128


def _model(H, I, nh, nkv, vocab=256, seed=0):
    """One int4 g128 layer from O.random_packed (qkv of nh + 2 nkv heads), the norms, embedding and lm_head."""
    N = dict(qkv=(nh + 2 * nkv) * HD, o=H, gate=I, up=I, down=H)
    K = dict(qkv=H, o=H, gate=H, up=H, down=I)
    layer = {}
    for j, name in enumerate(LINEARS):
        qweight, scales, qzeros, g_idx, _ = O.random_packed(K[name], N[name], 4, 128, seed=10 * seed + j)
        layer[name] = types.SimpleNamespace(qweight=qweight, scales=scales, qzeros=qzeros, g_idx=g_idx, bits=4)
    gen = torch.Generator().manual_seed(seed)
    layer['input_norm'], layer['post_norm'] = (torch.rand(2, H, generator=gen) + 0.5).half()
    embed = torch.randn(vocab, H, generator=gen).half()
    return [layer], embed, (torch.rand(H, generator=gen) + 0.5).half(), (torch.randn(vocab, H, generator=gen) * 0.05).half()


def _repeat_kv_columns(layer, nh, nkv):
    """The layer with every K/V head's qkv columns repeated g = nh / nkv times (qweight, scales and the packed qzeros): the multi-head layer
    in which query head h reads a copy of K/V head h // g."""
    H, g = nh * HD, nh // nkv
    head = torch.arange(nh) // g
    kv = (head[:, None] * HD + torch.arange(HD)).reshape(-1)
    cols = torch.cat([torch.arange(H), H + kv, H + nkv * HD + kv])
    qkv = layer['qkv']
    words = cols.view(-1, 8)[:, 0] // 8  # int4: 8 columns per qzeros word, and a head's 128 columns are whole words
    rep = types.SimpleNamespace(qweight=qkv.qweight[:, cols], scales=qkv.scales[:, cols], qzeros=qkv.qzeros[:, words], g_idx=qkv.g_idx, bits=4)
    return dict(layer, qkv=rep)


@pytest.mark.parametrize('nkv', [2, 1])
def test_grouped_query_oracle_is_the_multi_head_oracle_over_repeated_kv_heads(nkv):
    """H 512, 4 query heads on nkv K/V heads: logits and attention() (with and without exact, from position 0 and on a cache prefix) equal
    those of the multi-head oracle whose K/V heads are the repeated ones, bit for bit."""
    nh, g = 4, 4 // nkv
    layers, embed, norm, lm_head = _model(512, 1024, nh, nkv)
    gqa = LlamaOracle(layers, embed, norm, lm_head, nh, eps=1e-6, base=10000.0, n_kv_heads=nkv)
    mha = LlamaOracle([_repeat_kv_columns(layers[0], nh, nkv)], embed, norm, lm_head, nh, eps=1e-6, base=10000.0)
    toks = [3, 200, 7, 7, 255, 0]
    ref = gqa.logits(toks)
    assert torch.equal(ref, mha.logits(toks)) and bool(torch.isfinite(ref).all())
    gen = torch.Generator().manual_seed(1)
    kp, vp = (torch.randn(2, nkv, 37, HD, generator=gen) * 0.5).half()
    x = embed[toks[:2]]
    for pos in (0, 37 - 2):
        for exact in (False, True):
            xg, kg, vg = gqa.attention(0, x, pos, kp, vp, exact=exact)
            xm, km, vm = mha.attention(0, x, pos, kp.repeat_interleave(g, 0), vp.repeat_interleave(g, 0), exact=exact)
            assert torch.equal(xg, xm) and bool(torch.isfinite(xg).all()), f'pos {pos} exact={exact}'
            assert torch.equal(kg.repeat_interleave(g, 0), km) and torch.equal(vg.repeat_interleave(g, 0), vm), f'pos {pos} exact={exact}'


def _positions():
    return torch.tensor([[0, 1, 31, 2047, 8191, 8192], [16383, 32767, 65535, 100000, 131070, 131071]])


@pytest.mark.parametrize('base', [1e4, 5e5, 1e6])
def test_rope_table_of_the_base_rule_is_the_base_rotation(base):
    """O.rope_inplace with the table exp(i * fp32(-2 ln(base) / 128)) in fp32 rotates bit for bit as it does at `base`."""
    qk = torch.randn(2, 6, 2, 3, HD, generator=torch.Generator().manual_seed(2)).half()
    table = torch.exp(torch.arange(HD // 2, dtype=torch.float32) * np.float32(-2.0 * math.log(base) / HD))
    a, b = qk.clone(), qk.clone()
    O.rope_inplace(a, _positions(), base=base)
    O.rope_inplace(b, _positions(), inv_freq=table)
    assert torch.equal(a, b) and not torch.equal(a, qk)


@pytest.mark.parametrize('scaling', ['LLAMA3_1_ROPE_SCALING', 'LLAMA3_2_ROPE_SCALING'])
def test_llama3_rotation_is_within_the_rope_row_bound(scaling):
    """O.rope_inplace with a llama3 table against fp64 RoPE of the same fp32 angles, within attn_probe.check_rope_row's bound, up to
    position 131071."""
    from gptq_b200 import engine, ops
    table = ops.rope_inv_freq(engine.LLAMA3_ROPE_BASE, HD, getattr(engine, scaling))
    qk = torch.randn(2, 6, 2, 4, HD, generator=torch.Generator().manual_seed(3)).half()
    out = qk.clone()
    O.rope_inplace(out, _positions(), inv_freq=table)
    pos = _positions()
    worst = max(P.check_rope_row(out[b, t].reshape(-1, HD), qk[b, t].reshape(-1), int(pos[b, t]), inv_freq=table) for b in range(2) for t in range(6))
    assert worst <= 1, worst
