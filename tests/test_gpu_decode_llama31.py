"""GPU: LLaMA-3.1 / 3.2 / 3.3 decoding -- the llama3 RoPE frequency scaling in every kernel that rotates, at positions up to 131071.

  * gptq_rope_inplace_freq against fp64 cos / sin of the same fp32 angles (attn_probe.check_rope_row with the table), at the band and context
    edges up to the last row of a 131072-row cache;
  * both decode engines on the attention probe's planted caches (attn_probe.Probe with rope_scaling) at long positions, batch 1 and 8, each
    sequence at its own position: the appended K row bit for bit what gptq_rope_inplace_freq (the prefill's rotation) writes, and against fp64
    RoPE; the output against an fp64 softmax within attn_probe.x_bound, and the bit-exact anchors (attn_probe.run_sweeps);
  * LLaMA-3.1-8B, 3.1-70B and 3.2-3B (tied lm_head) layers against the reference decoder with the table
    (llama_oracle.check_blocks_on_random_cache), and sampled generation at 128256 ids;
  * prefill and extend across the 8192 boundary and up to the last row of a 131072 cache, against stepping
    (llama_oracle.check_extend_against_stepping);
  * a tiny HF LLaMA with rope_scaling llama3 (original context 64, so all three bands act within 512 tokens): QuantLlamaAttention against HF's
    attention, the engine's score() and decode steps against HF's forward, and the unscaled rotation missing HF by more than 10x the bound.

The file sorts ahead of tests/test_gpu_exact.py for the reason tests/test_gpu_decode_gqa.py gives.
"""
import pytest
import torch

import attn_probe as P
from exact_fixtures import matvec_takes
from gpu_util import assert_rel_close, report
from llama_oracle import LlamaOracle, check_blocks_on_random_cache, check_extend_against_stepping
from oracle import gptq_oracle as O

pytestmark = pytest.mark.gpu

LONG = [0, 1, 8191, 8192, 8193, 32767, 65535, 131070, 131071]
LLAMA3_EPS = 1e-5


def _engine():
    from gptq_b200 import engine
    return engine


def _table(scaling):
    from gptq_b200 import ops
    return ops.rope_inv_freq(_engine().LLAMA3_ROPE_BASE, 128, scaling)


# ----------------------------------------------------------------------------- the rope kernel
def test_rope_kernel_against_fp64():
    from gptq_b200 import ops
    engine = _engine()
    gen = torch.Generator().manual_seed(31)
    positions = LONG + sorted(torch.randint(0, 131072, (23, ), generator=gen).tolist())
    x = (torch.randn(1, len(positions), 2, 8, 128, generator=gen)).half()
    pos = torch.tensor([positions])
    for name, scaling in (('3.1', engine.LLAMA3_1_ROPE_SCALING), ('3.2', engine.LLAMA3_2_ROPE_SCALING)):
        table = _table(scaling)
        dq = x.cuda()
        ops.rotate_half_(dq[:, :, :2], pos.cuda(), inv_freq=table)
        out = dq.cpu()
        worst = max(P.check_rope_row(out[0, t, :2].reshape(16, 128), x[0, t, :2].reshape(-1), p, inv_freq=table) for t, p in enumerate(positions))
        report(worst, f'gptq_rope_inplace_freq LLaMA-{name} vs fp64 RoPE')
        plain = x.cuda()
        ops.rotate_half_(plain[:, :, :2], pos.cuda(), base=engine.LLAMA3_ROPE_BASE)
        assert not torch.equal(plain.cpu()[0, 2:], out[0, 2:]), 'the table changed nothing'


# ----------------------------------------------------------------------------- planted caches at long positions, both engines
BATCH8 = [[131071, 131070, 65535, 32767, 8193, 8192, 8191, 1], [0, 100000, 131071, 12345, 8192, 77777, 50000, 131000]]


@pytest.mark.parametrize('size,batch', [('llama3-8b', 1), ('llama3-8b', 8), ('tiny-gqa2-chain', 1), ('tiny-gqa2-chain', 8)])
def test_long_positions_planted(size, batch):
    engine = _engine()
    probe = P.Probe(size, batch=batch, max_seq=131072, rope_base=engine.LLAMA3_ROPE_BASE, rope_scaling=engine.LLAMA3_1_ROPE_SCALING)
    assert probe.persistent == (size == 'llama3-8b') == (probe.dec.launches_per_step() == 1)
    sets = [[p] for p in LONG] if batch == 1 else BATCH8
    P.run_sweeps(probe, f'{size} batch {batch} llama3 (max_seq 131072)', sets, profiles=('heavy', 'late', 'uniform'), seed=4321,
                 toks=lambda i, b: 11 * i + 5 * b + 1, rotate_heavy=True)


# ----------------------------------------------------------------------------- real LLaMA-3.x layers against the reference decoder
def _llama3_decoder(size, scaling, max_seq, seed, tied=False, batch=1):
    """`size`'s shape, two int4 g128 layers, vocabulary 128256, LLaMA-3's epsilon and base with the table of `scaling`; tied: LLaMA-3.2's
    lm_head, which is the embedding."""
    engine = _engine()
    kw = dict(rms_eps=LLAMA3_EPS, rope_base=engine.LLAMA3_ROPE_BASE, rope_scaling=scaling, max_seq=max_seq)
    dec = engine.synthetic_llama(size, bits=4, groupsize=128, vocab=128256, seed=seed, n_layers=2, batch=batch, **kw)
    if tied:
        dec = engine.LlamaDecoder(dec.layers, dec.embed, dec.final_norm, dec.embed, dec.n_heads, n_kv_heads=dec.n_kv_heads, batch=batch, **kw)
        assert dec.lm_head.data_ptr() == dec.embed.data_ptr()
    assert torch.equal(dec.rope_inv_freq, _table(scaling))
    return dec


def _check_llama3_blocks(dec, size, scaling, positions):
    """The two layers of dec on the persistent kernel, block by block against the reference with LLaMA-3's epsilon, base and the table."""
    return check_blocks_on_random_cache(dec, positions, f'{size} llama3', eps=LLAMA3_EPS, base=_engine().LLAMA3_ROPE_BASE, inv_freq=_table(scaling),
                                        cache_seed=111, k_row_vs_reference=False)


def _batch_steps(dec, oracle, n_steps, vocab, what):
    """n_steps greedy-fed steps of `batch` sequences from position 0 (sequence b starts at token 1000 b + 7), every step's logits against the
    reference of that sequence alone (the bound of test_gpu_decode_gqa.test_batch4_ragged_positions) and next_tokens the argmax."""
    dec.reset()
    seqs = [[(1000 * b + 7) % vocab] for b in range(dec.batch)]
    for pos in range(n_steps):
        dec.set_input([s[-1] for s in seqs], pos)
        dec.step()
        torch.cuda.synchronize()
        nxt = dec.next_tokens.tolist()
        for b in range(dec.batch):
            assert nxt[b] == int(dec.logits[b].float().argmax())
            seqs[b].append(nxt[b])
    for b, s in enumerate(seqs):
        ref = oracle.logits(s[:n_steps])
        assert_rel_close(dec.logits[b], ref[n_steps - 1], rel=2e-2, what=f'{what} sequence {b} at pos {n_steps - 1}')


def test_llama31_8b():
    engine = _engine()
    dec = _llama3_decoder('llama3-8b', engine.LLAMA3_1_ROPE_SCALING, 12288, seed=21)
    _check_llama3_blocks(dec, 'llama3-8b', engine.LLAMA3_1_ROPE_SCALING, [0, 2047, 8191, 8192, 12000])
    # sampled generation over the whole 128256-id vocabulary on the scaled model
    prompt = [5, 128255, 77, 1000]
    sampled = dec.generate(prompt, 6, do_sample=True, temperature=0.8, top_k=0, top_p=0.95, seed=5)
    assert sampled[:4] == prompt and len(sampled) == 10 and all(0 <= t < 128256 for t in sampled)


def test_llama31_70b():
    """LLaMA-3.1-70B (and 3.3-70B, the same shape and scaling): batch 1 on the persistent kernel block by block, batch 8 on the kernel chain,
    whose launch count follows the matvec route rule (exact_fixtures.matvec_takes)."""
    engine = _engine()
    dec = _llama3_decoder('70b', engine.LLAMA3_3_ROPE_SCALING, 8448, seed=22)
    oracle = _check_llama3_blocks(dec, '70b', engine.LLAMA3_3_ROPE_SCALING, [0, 8192])
    d8 = engine.LlamaDecoder(dec.layers, dec.embed, dec.final_norm, dec.lm_head, dec.n_heads, n_kv_heads=8, batch=8, max_seq=64, rms_eps=LLAMA3_EPS,
                             rope_base=engine.LLAMA3_ROPE_BASE, rope_scaling=engine.LLAMA3_1_ROPE_SCALING)
    H, I, Hkv = dec.hidden, dec.intermediate, 8 * 128
    per_layer = 2 + sum(1 if matvec_takes(8, K, N) else 2 for K, N in ((H, H + 2 * Hkv), (H, H), (H, I), (I, H)))
    assert d8.launches_per_step() == 3 + 2 * per_layer, d8.launches_per_step()
    _batch_steps(d8, oracle, 4, 128256, '70b batch 8 chain')


@pytest.mark.parametrize('batch', [1, 8])
def test_llama32_3b_tied(batch):
    engine = _engine()
    scaling = engine.LLAMA3_2_ROPE_SCALING
    if batch == 1:
        _check_llama3_blocks(_llama3_decoder('llama3.2-3b', scaling, 32768, seed=23, tied=True), 'llama3.2-3b', scaling, [0, 8192, 30000])
        return
    dec = _llama3_decoder('llama3.2-3b', scaling, 16, seed=23, tied=True, batch=8)
    assert dec.n_kv_heads == 8 and dec.launches_per_step() == 1
    _batch_steps(dec, LlamaOracle.from_decoder(dec, eps=LLAMA3_EPS, base=engine.LLAMA3_ROPE_BASE, inv_freq=_table(scaling)), 5, 128256, '3.2-3b batch 8')


# ----------------------------------------------------------------------------- long prompts: prefill and extend against stepping
def test_long_prompts_prefill_and_extend():
    engine = _engine()
    dec = engine.synthetic_llama('llama3-8b', bits=4, groupsize=128, vocab=128256, seed=24, n_layers=2, max_seq=131072, rms_eps=LLAMA3_EPS,
                                 rope_base=engine.LLAMA3_ROPE_BASE, rope_scaling=engine.LLAMA3_1_ROPE_SCALING)
    assert dec.launches_per_step() == 1
    toks = torch.randint(0, 128256, (131072, ), generator=torch.Generator().manual_seed(8)).tolist()
    check_extend_against_stepping(dec, toks[:8400], 8100, 'llama3.1-8b across 8192', prefilled=8000)
    # (the first 130800 rows through extend(): its attention is the cache kernel, where the prefill's SDPA would hold 130800 rows at once)
    check_extend_against_stepping(dec, toks, 130816, 'llama3.1-8b to the last row of 131072', prefilled=130800, fill='extend')


# ----------------------------------------------------------------------------- HF parity
def _tiny_llama3_hf(seed=0):
    """(the quantized model: fp16, every linear but lm_head a QuantLinear with the synthetic models' fields (engine.random_qlayer: zero points
    centred on the weight grid, so that the residual stream stays well scaled over 512 positions); HF's fp32 LlamaForCausalLM on the same weights,
    each QuantLinear dequantised as the reference's kernel materialises it (O.dequant); the scaling dict).  HF's fp32 model is the reference:
    it rotates with HF's own fp32 llama3 table (an fp16 HF model would round that table and its cos / sin to fp16)."""
    import quant
    import utils
    from transformers import LlamaConfig, LlamaForCausalLM
    scaling = dict(_engine().LLAMA3_1_ROPE_SCALING, original_max_position_embeddings=64)
    cfg = LlamaConfig(hidden_size=512, intermediate_size=1024, num_hidden_layers=2, num_attention_heads=4, num_key_value_heads=2, vocab_size=256,
                      max_position_embeddings=512, rms_norm_eps=1e-5, rope_parameters=dict(scaling, rope_theta=5e5))
    torch.manual_seed(seed)
    hf = LlamaForCausalLM(cfg).float().eval()
    model = LlamaForCausalLM(cfg).eval()
    model.load_state_dict(hf.state_dict())
    model.half()
    layers = utils.find_layers(model)
    layers.pop('lm_head')
    quant.make_quant_linear(model, layers, 4, 128)
    gen = torch.Generator(device='cuda').manual_seed(seed + 7)
    for name, m in ((n, m) for n, m in model.named_modules() if isinstance(m, quant.QuantLinear)):
        q = _engine().random_qlayer(m.infeatures, m.outfeatures, 4, 128, 'cuda', gen)
        m.qweight, m.scales, m.qzeros, m.g_idx = (t.cpu() for t in (q.qweight, q.scales, q.qzeros, q.g_idx))
        hf.get_submodule(name).weight.data = O.dequant(m.qweight, m.scales, m.qzeros, m.g_idx, 4).t().float().contiguous()
    hf.model.embed_tokens.weight.data = model.model.embed_tokens.weight.data.float()
    hf.lm_head.weight.data = model.lm_head.weight.data.float()
    return model.cuda(), hf.cuda(), scaling


def _ratio(out, ref, rel):
    out, ref = out.float().cpu(), ref.float().cpu()
    rms = ref.pow(2).mean().sqrt()
    return ((out - ref).abs() / (rel * torch.maximum(ref.abs(), rms) + 1e-7)).max().item()


def _score_ratio(lps, ids, ref_logits):
    logits = ref_logits[:-1].double().cpu()
    ref = torch.log_softmax(logits, -1).gather(1, torch.tensor(ids[1:])[:, None])[:, 0]
    return ((lps.cpu().double() - ref).abs() / (2 * 2e-2 * logits.abs().amax(-1))).max().item()


def test_hf_parity():
    import quant
    engine = _engine()
    model, hf, scaling = _tiny_llama3_hf()
    assert torch.equal(hf.model.rotary_emb.inv_freq.cpu(), _table(scaling)), 'HF builds the table the engine takes'
    ids = torch.randint(0, 256, (1, 512), generator=torch.Generator().manual_seed(1))
    with torch.no_grad():
        ref = hf(ids.cuda()).logits[0].float()  # HF's LlamaAttention with its llama3 rotary embedding, fp32, on the dequantised weights
        quant.make_quant_attn(model)
        assert all(torch.equal(l.self_attn.rope_inv_freq, _table(scaling)) for l in model.model.layers)
        fused = model(ids.cuda()).logits[0].float()
    report(_ratio(fused, ref, 2e-2), 'QuantLlamaAttention vs HF LlamaAttention, 512 tokens, llama3 rope')
    dec = engine.from_hf_quant_model(model, max_seq=512)
    assert dec.n_kv_heads == 2 and dec.launches_per_step() == 1 and torch.equal(dec.rope_inv_freq, _table(scaling))
    toks = ids[0].tolist()
    report(_score_ratio(dec.score([toks])[0], toks, ref), 'engine score() vs HF, llama3 rope')
    assert dec.prefill(toks[:497]) == 496
    for pos in range(496, 512):
        dec.set_input(toks[pos], pos)
        dec.step()
        torch.cuda.synchronize()
        assert_rel_close(dec.logits[0], ref[pos], rel=2e-2, what=f'engine step vs HF, pos {pos}')
        tok = int(dec.next_tokens[0])
        assert tok == int(dec.logits[0].float().argmax())
        assert ref[pos].max() - ref[pos][tok] <= 4e-2 * ref[pos].abs().max(), f'pos {pos}: greedy token {tok} is not HF\'s (up to a near tie)'
    # the same model decoded with the unscaled rotation at the same base misses HF's logits by far more than their bound: the tests see the
    # scaling
    plain = engine.LlamaDecoder(dec.layers, dec.embed, dec.final_norm, dec.lm_head, 4, n_kv_heads=2, max_seq=512, rms_eps=1e-5, rope_base=5e5)
    assert plain.rope_inv_freq is None and plain.prefill(toks[:497]) == 496
    miss = 0.0
    for pos in range(496, 512):
        plain.set_input(toks[pos], pos)
        plain.step()
        torch.cuda.synchronize()
        miss = max(miss, _ratio(plain.logits[0], ref[pos], 2e-2))
    print(f'  engine with the unscaled rotation vs HF: worst |err| / bound = {miss:.3g}')
    assert miss >= 10, miss
