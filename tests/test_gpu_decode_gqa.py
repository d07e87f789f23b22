"""GPU: grouped-query attention (n_kv_heads < n_heads; query head h reads K/V head h / g, g = n_heads / n_kv_heads) in both decode engines,
the prefill / extend / scoring pass, gptq_cached_attention_gqa and the quant modules.

  * both engines against the CPU reference decoder at g = 2 and with one K/V head (g = 4), int4, act-order and 3-bit, batch 1 and batch 4 at
    ragged positions;
  * LLaMA-2-70B (g = 8), CodeLlama-34B (RoPE base 1e6, context 16384) and LLaMA-3-8B (base 5e5, vocabulary 128256) layers, two of them, on
    the persistent kernel, block by block against the reference (llama_oracle.check_last_layer_blocks) on a random cache;
  * the shared new row: the g query heads of a group all use row pos, one of them stores it; every K/V head's row pos is the reference's
    rotated k, no other cache row changes, and prefill, extend and token-by-token decode write the same rows;
  * gptq_cached_attention_gqa against the float64 reference with the K/V heads repeated, and the MHA symbol unchanged;
  * the HF route: make_quant_attn and the engine built from the HF model against HF's decoder running QuantLlamaAttention.

The file sorts ahead of tests/test_gpu_exact.py, the first file that traces in the pytest process, and that is deliberate: its two minutes
of sustained GPU work would leave every later in-process profiler session without kernel records (module docstring of
tests/test_gpu_cuda_core_kernels.py), and the routing assertions of the files after it would skip.
"""
import ctypes

import pytest
import torch

from gpu_util import assert_rel_close, check_cached_attention, fill_quant_linear, make_kv_cache
from llama_oracle import CODELLAMA, KV_ROW_TOL, LlamaOracle, assert_no_failures, check, check_extend_against_stepping, check_last_layer_blocks, check_scores, \
    step_all
from oracle import gptq_oracle as O

pytestmark = pytest.mark.gpu

LLAMA2_70B = (10000.0, 1e-5)
LLAMA3 = (5e5, 1e-5)


class GqaOracle(LlamaOracle):
    """LlamaOracle with n_kv_heads K/V heads: the fused qkv output is q | k | v of nh | nkv | nkv heads, RoPE rotates the first nh + nkv
    heads, query head h attends with K/V head h // (nh // nkv).  attention() returns the new K / V rows of the nkv heads."""

    def __init__(self, *a, n_kv_heads, **kw):
        super().__init__(*a, **kw)
        self.n_kv_heads = n_kv_heads

    @classmethod
    def from_decoder(cls, dec, *, eps, base):
        return cls(dec.layers, dec.embed, dec.final_norm, dec.lm_head, dec.n_heads, eps=eps, base=base, n_kv_heads=dec.n_kv_heads)

    def attention(self, li, x, pos, k_prefix=None, v_prefix=None, exact=False):
        n, nh, nkv, hd = x.shape[0], self.n_heads, self.n_kv_heads, self.head_dim
        g = nh // nkv
        qkv = self._linear(li, 'qkv', O.rmsnorm_fwd(x, self._layer(li)['input_norm'], self.eps), exact).view(1, n, nh + 2 * nkv, hd).clone()
        O.rope_inplace(qkv[:, :, None, :nh + nkv], torch.arange(pos, pos + n)[None, :], base=self.base)
        q, k, v = (t.transpose(0, 1) for t in qkv[0].split([nh, nkv, nkv], 1))  # [heads, n, hd]
        K = torch.cat([k_prefix[:, :pos], k], 1) if pos else k
        V = torch.cat([v_prefix[:, :pos], v], 1) if pos else v
        qg = q.float().reshape(nkv, g, n, hd)  # query head kvh * g + j
        s = (qg @ K.float()[:, None].transpose(-1, -2)) * hd**-0.5  # [nkv, g, n, pos + n]
        s = s.masked_fill(torch.ones(n, pos + n, dtype=torch.bool).triu(pos + 1), float('-inf'))
        att = (torch.softmax(s, -1) @ V.float()[:, None]).reshape(nh, n, hd).half().transpose(0, 1).reshape(n, self.hidden)
        return x + self._linear(li, 'o', att, exact), k, v


def _decoder(size, **kw):
    from gptq_b200 import engine
    dec = engine.synthetic_llama(size, **kw)
    assert dec.n_kv_heads == engine.KV_HEADS[size] and dec.k_cache.shape[2] == dec.n_kv_heads
    persistent = not size.endswith('-chain')
    assert (dec.launches_per_step() == 1) == persistent, f'{size}: wrong engine'
    return dec


SIZES = ['tiny-gqa2', 'tiny-gqa1', 'tiny-gqa2-chain', 'tiny-gqa1-chain']


@pytest.mark.parametrize('bits,act', [(4, False), (4, True), (3, True)], ids=['int4', 'int4-act', 'int3-act'])
@pytest.mark.parametrize('size', SIZES)
def test_decode_steps_match_oracle(size, bits, act):
    """Six decode steps against the reference decoder (bound of test_gpu_engine.py::test_decode_steps_match_oracle)."""
    dec = _decoder(size, bits=bits, groupsize=64, act_order=act, vocab=512, seed=bits, max_seq=64)
    toks = torch.randint(0, 512, (6, ), generator=torch.Generator().manual_seed(0)).tolist()
    ref = GqaOracle.from_decoder(dec, eps=1e-6, base=10000.0).logits(toks)
    for pos, tok in enumerate(toks):
        dec.set_input(tok, pos)
        dec.step()
        torch.cuda.synchronize()
        assert_rel_close(dec.logits[0], ref[pos], rel=2e-2, what=f'{size} bits={bits} act={act} pos={pos}')
        assert int(dec.next_tokens[0]) == int(dec.logits[0].float().argmax())


@pytest.mark.parametrize('size', SIZES)
def test_batch4_ragged_positions(size):
    """Four sequences of different lengths stepped in lock-step, each at its own position (a finished sequence re-steps its last token at its
    last position, which rewrites the same row): every step's logits of every sequence against the reference of that sequence alone."""
    dec = _decoder(size, bits=4, groupsize=64, vocab=300, seed=7, max_seq=96, batch=4)
    lens = [5, 40, 2, 33]
    gen = torch.Generator().manual_seed(3)
    seqs = [torch.randint(0, 300, (n, ), generator=gen).tolist() for n in lens]
    oracle = GqaOracle.from_decoder(dec, eps=1e-6, base=10000.0)
    refs = [oracle.logits(s) for s in seqs]
    for k in range(max(lens)):
        pos = [min(k, n - 1) for n in lens]
        dec.set_input([s[p] for s, p in zip(seqs, pos)], pos)
        dec.step()
        torch.cuda.synchronize()
        for b in range(4):
            assert_rel_close(dec.logits[b], refs[b][pos[b]], rel=2e-2, what=f'{size} step {k} sequence {b} pos {pos[b]}')


def _real_shape_blocks(size, positions, max_seq, rope, vocab=32000):
    """Two layers of a real GQA shape on the persistent kernel, a random cache, one step at each position, block by block against the
    reference (the appended K rows against the exact linears, as test_gpu_engine_fullsize.py does where one-ulp roundings matter)."""
    from gptq_b200 import engine
    base, eps = rope
    dec2 = _decoder(size, bits=4, groupsize=128, vocab=vocab, seed=11, max_seq=max_seq, n_layers=2, rms_eps=eps, rope_base=base)
    dec1 = engine.LlamaDecoder(dec2.layers[:1], dec2.embed, dec2.final_norm, dec2.lm_head, dec2.n_heads, max_seq=max_seq, rms_eps=eps, rope_base=base,
                               n_kv_heads=dec2.n_kv_heads)
    assert dec1.launches_per_step() == 1
    gen = torch.Generator(device=dec2.dev).manual_seed(111)
    dec2.k_cache.copy_((torch.randn(dec2.k_cache.shape, device=dec2.dev, generator=gen) * 0.5).half())
    dec2.v_cache.copy_((torch.randn(dec2.v_cache.shape, device=dec2.dev, generator=gen) * 0.5).half())
    k0, v0 = dec2.k_cache.clone(), dec2.v_cache.clone()
    kc, vc = k0.cpu(), v0.cpu()
    oracle = GqaOracle.from_decoder(dec2, eps=eps, base=base)
    for i, pos in enumerate(positions):
        tok = (17 * i + 3) % vocab
        what = f'{size} base={base:g} pos={pos}'
        # every position starts from the same cache: a step rewrites row pos, which a later, short context would read
        for dec in (dec1, dec2):
            dec.k_cache.copy_(k0[:len(dec.layers)])
            dec.v_cache.copy_(v0[:len(dec.layers)])
        check_last_layer_blocks(dec1, oracle, tok, pos, kc, vc, what + ' (1 layer)', False)
        check_last_layer_blocks(dec2, oracle, tok, pos, kc, vc, what + ' (2 layers)', False)
        assert_no_failures()
    return dec2, oracle


def test_llama2_70b_layers():
    _real_shape_blocks('70b', [0, 31, 32, 2047, 4095], 4096, LLAMA2_70B)


def test_codellama_34b_layers_at_16k():
    _real_shape_blocks('34b', [16383], 16384, CODELLAMA)


def test_llama3_8b_layers_greedy_sampled_and_scored():
    dec, oracle = _real_shape_blocks('llama3-8b', [0, 2047], 2048, LLAMA3, vocab=128256)
    assert dec.vocab == 128256
    # greedy and sampled generation over the whole vocabulary (sampling takes up to 131072 ids)
    prompt = [5, 128255, 77, 1000]
    greedy = dec.generate(prompt, 6, prefill=True)
    assert greedy[:4] == prompt and len(greedy) == 10 and all(0 <= t < 128256 for t in greedy)
    sampled = dec.generate(prompt, 6, do_sample=True, temperature=0.8, top_k=0, top_p=0.95, seed=5)
    assert sampled[:4] == prompt and len(sampled) == 10 and all(0 <= t < 128256 for t in sampled)
    # the draw depends only on the logits, the parameters and the position (the step's logits themselves vary in their last bits from run to
    # run: unordered fp32 reductions), so the same logits and seed give the same token, over the whole vocabulary
    from gptq_b200 import ops
    logits = dec.logits.clone()
    dev = logits.device
    args = lambda seed: (torch.tensor([7], dtype=torch.int32, device=dev), torch.tensor([1.0], device=dev), torch.tensor([0], dtype=torch.int32, device=dev),
                         torch.tensor([1.0], device=dev), torch.tensor([seed], dtype=torch.int64, device=dev))
    draws = [int(ops.sample_tokens(logits, *args(seed))[0]) for seed in range(16)]
    assert draws == [int(ops.sample_tokens(logits, *args(seed))[0]) for seed in range(16)] and all(0 <= t < 128256 for t in draws)
    # score() through the ragged pass (SDPA with the K/V heads shared) against the reference's log-softmax
    seqs = [[3, 128255, 9, 4000, 17, 2], [8, 1, 64000]]
    assert check_scores(dec.score(seqs), seqs, oracle, 'llama3-8b score') <= 1


@pytest.mark.parametrize('size', ['tiny-gqa1', 'tiny-gqa2-chain'])
def test_shared_new_row(size):
    """After a step at pos (batch 2, positions 37 and 5): row pos of every K/V head of layer 0 is the reference's rotated k and v (the layer's
    input is the embedding row), the rows before pos are what they were and the NaN-poisoned rows after pos are untouched."""
    dec = _decoder(size, bits=4, groupsize=64, vocab=300, seed=9, max_seq=64, batch=2)
    oracle = GqaOracle.from_decoder(dec, eps=1e-6, base=10000.0)
    gen = torch.Generator(device=dec.dev).manual_seed(5)
    dec.k_cache.copy_((torch.randn(dec.k_cache.shape, device=dec.dev, generator=gen) * 0.5).half())
    dec.v_cache.copy_((torch.randn(dec.v_cache.shape, device=dec.dev, generator=gen) * 0.5).half())
    pos, toks = [37, 5], [11, 250]
    for b, p in enumerate(pos):
        dec.k_cache[:, b, :, p:] = float('nan')
        dec.v_cache[:, b, :, p:] = float('nan')
    before_k, before_v = dec.k_cache.clone(), dec.v_cache.clone()
    dec.set_input(toks, pos)
    dec.step()
    torch.cuda.synchronize()
    assert torch.isfinite(dec.logits).all()
    for b, (p, t) in enumerate(zip(pos, toks)):
        for c, c0 in ((dec.k_cache, before_k), (dec.v_cache, before_v)):
            assert torch.equal(c[:, b, :, :p], c0[:, b, :, :p]), f'sequence {b}: a row before pos changed'
            assert torch.isnan(c[:, b, :, p + 1:]).all(), f'sequence {b}: a row after pos was written'
            assert torch.isfinite(c[:, b, :, p]).all(), f'sequence {b}: row pos of some K/V head was not written'
        _, k_ex, v_ex = oracle.attention(0, dec.embed[t].cpu()[None, :], p, before_k[0, b].cpu(), before_v[0, b].cpu(), exact=True)
        check(dec.k_cache[0, b, :, p], k_ex[:, 0], rel=KV_ROW_TOL, what=f'{size} sequence {b}: K row pos vs Exact')
        check(dec.v_cache[0, b, :, p], v_ex[:, 0], rel=KV_ROW_TOL, what=f'{size} sequence {b}: V row pos vs Exact')
    assert_no_failures()


@pytest.mark.parametrize('size', ['tiny-gqa2', 'tiny-gqa1-chain'])
def test_prefill_extend_and_decode_write_the_same_rows(size):
    dec = _decoder(size, bits=4, groupsize=64, vocab=300, seed=5, max_seq=96)
    prompt = torch.randint(0, 300, (40, ), generator=torch.Generator().manual_seed(2)).tolist()
    step_all(dec, prompt, 0)
    ref_logits, ref_k, ref_v = dec.logits[0].float().clone(), dec.k_cache[:, 0, :, :40].float().clone(), dec.v_cache[:, 0, :, :40].float().clone()
    dec.k_cache.zero_()
    dec.v_cache.zero_()
    dec.reset()
    assert dec.prefill(prompt) == 39
    assert_rel_close(dec.k_cache[:, 0, :, :39], ref_k[:, :, :39], rel=1e-2, what=f'{size}: prefilled K rows')
    assert_rel_close(dec.v_cache[:, 0, :, :39], ref_v[:, :, :39], rel=1e-2, what=f'{size}: prefilled V rows')
    dec.set_input(prompt[-1], 39)
    dec.step()
    torch.cuda.synchronize()
    assert_rel_close(dec.logits[0], ref_logits, rel=2e-2, what=f'{size}: logits after prefill + 1 decode step')
    dec.reset()
    check_extend_against_stepping(dec, prompt, 17, f'{size} extend')


@pytest.mark.parametrize('nh,g', [(32, 4), (32, 8), (64, 8)], ids=['7b-heads-g4', '7b-heads-g8', '70b-heads-g8'])
def test_cached_attention_gqa(nh, g):
    """gptq_cached_attention_gqa against the float64 reference (gpu_util.cached_attention_reference) over the K/V heads repeated g times, with
    spans from position 0 and from start > 0, NaN in every cache row the kernel must not read."""
    from gptq_b200 import ops
    nkv = nh // g
    spans = [(0, 0, 130), (2, 1000, 77), (3, 127, 1)]
    q, _, _ = make_kv_cache(4, nh, 1280, spans, seed=3, layers=1, layer=0)  # q rows of nh heads (the same heavy-key direction u as below)
    _, kc, vc = make_kv_cache(4, nkv, 1280, spans, seed=3, layers=2, layer=1)
    out = ops.cached_attention(q, kc[1], vc[1], spans)
    torch.cuda.synchronize()
    worst = check_cached_attention(out, q, kc[1].repeat_interleave(g, 1), vc[1].repeat_interleave(g, 1), spans, f'{nh} heads / {nkv} K/V heads')
    print(f'  cached attention {nh}/{nkv}: worst |err| / bound = {worst:.3g}')


def test_cached_attention_mha_symbol_unchanged():
    """gptq_cached_attention (MHA) and gptq_cached_attention_gqa with n_kv_heads = n_heads are one implementation: identical bits."""
    from gptq_b200._lib import lib, check as ck
    spans = [(0, 0, 200), (1, 300, 64)]
    q, kc, vc = make_kv_cache(2, 32, 512, spans, seed=4, layers=1, layer=0)
    B, nh, S, hd = kc[0].shape
    outs = []
    for fn, extra in ((lib.gptq_cached_attention, ()), (lib.gptq_cached_attention_gqa, (nh, ))):
        out = torch.empty(q.shape, dtype=torch.float16, device='cuda')
        arr = lambda i: (ctypes.c_int32 * len(spans))(*[sp[i] for sp in spans])
        ck(fn(q.data_ptr(), q.shape[1], kc.data_ptr(), vc.data_ptr(), B, nh, *extra, hd, S, len(spans), arr(0), arr(1), arr(2), out.data_ptr(), q.shape[1],
              None))
        torch.cuda.synchronize()
        outs.append(out)
    assert torch.equal(outs[0], outs[1])
    check_cached_attention(outs[0], q, kc[0], vc[0], spans, 'MHA')


def _tiny_gqa_hf(heads=4, kv=2, seed=0):
    """A two-layer HF LLaMA (head_dim 128) with 4 query and 2 K/V heads, every linear but lm_head a randomly filled QuantLinear
    (quant.make_quant_linear only: HF's own attention, repeat_kv included, runs on them)."""
    import quant
    import utils
    from transformers import LlamaConfig, LlamaForCausalLM
    cfg = LlamaConfig(hidden_size=128 * heads, intermediate_size=1024, num_hidden_layers=2, num_attention_heads=heads, num_key_value_heads=kv,
                      vocab_size=256, max_position_embeddings=128)
    torch.manual_seed(seed)
    model = LlamaForCausalLM(cfg).half().eval()
    layers = utils.find_layers(model)
    layers.pop('lm_head')
    quant.make_quant_linear(model, layers, 4, 128)
    for i, m in enumerate(m for m in model.modules() if isinstance(m, quant.QuantLinear)):
        fill_quant_linear(m, 4, i + 1)
    return model


def test_hf_route():
    """The route a GQA checkpoint takes: make_quant_linear (QuantLinear projections) -> make_quant_attn -> engine.from_hf_quant_model (persistent
    kernel).  HF's decoder with QuantLlamaAttention is the reference here: it equals HF's own LlamaAttention (repeat_kv) up to the fp16 rounding
    of the rotated q and k, which the fused route shares with the reference's rotate_half kernel (tests/test_gqa_host.py holds it to HF's
    attention exactly with that rounding taken out).  Its prefill and a step on its cache against its full forward, and six decode steps of the
    engine against that forward and against the reference decoder, within rel=2e-2."""
    import quant
    from gptq_b200 import engine
    model = _tiny_gqa_hf()
    quant.make_quant_attn(model)
    assert all(isinstance(l.self_attn, quant.QuantLlamaAttention) and l.self_attn.num_key_value_heads == 2 for l in model.model.layers)
    model = model.cuda()
    ids = torch.randint(0, 256, (1, 9), generator=torch.Generator().manual_seed(1))
    with torch.no_grad():
        ref = model(ids.cuda()).logits[0].float()  # causal: row i is the prediction after token i
        out = model(ids[:, :8].cuda(), use_cache=True)
        assert_rel_close(out.logits[0], ref[:8], rel=2e-2, what='QuantLlamaAttention prefill')
        step = model(ids[:, 8:9].cuda(), past_key_values=out.past_key_values, use_cache=True)
        assert out.past_key_values.layers[0].keys.shape[1] == 2, 'the cache holds the K/V heads'
        assert_rel_close(step.logits[0, 0], ref[8], rel=2e-2, what='QuantLlamaAttention step on the cache')
    dec = engine.from_hf_quant_model(model, max_seq=16)
    assert dec.n_kv_heads == 2 and dec.launches_per_step() == 1
    oracle = GqaOracle.from_decoder(dec, eps=model.config.rms_norm_eps, base=10000.0).logits(ids[0, :6].tolist())
    for pos in range(6):
        dec.set_input(int(ids[0, pos]), pos)
        dec.step()
        torch.cuda.synchronize()
        assert_rel_close(dec.logits[0], oracle[pos], rel=2e-2, what=f'engine from the HF model vs the reference decoder, pos={pos}')
        assert_rel_close(dec.logits[0], ref[pos], rel=2e-2, what=f'engine from the HF model vs its QuantLlamaAttention forward, pos={pos}')
