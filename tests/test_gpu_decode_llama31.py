"""GPU: LLaMA-3.1 / 3.2 / 3.3 decoding -- the llama3 RoPE frequency scaling in every kernel that rotates, at positions up to 131071.

  * gptq_rope_inplace_freq against fp64 cos / sin of the same fp32 angles (check_rope_row_table: attn_probe.check_rope_row's bound with the
    table's angles), at the band and context edges up to the last row of a 131072-row cache;
  * both decode engines on the attention probe's planted caches (ScaledProbe: attn_probe.Probe's model with the table) at long positions,
    batch 1 and 8, each
    sequence at its own position: the appended K row bit for bit what gptq_rope_inplace_freq (the prefill's rotation) writes, and against fp64
    RoPE; the output against an fp64 softmax within attn_probe.x_bound, and the bit-exact anchors;
  * LLaMA-3.1-8B, 3.1-70B and 3.2-3B (tied lm_head) layers against the reference decoder with the table, and sampled generation at 128256 ids;
  * prefill and extend across the 8192 boundary and up to the last row of a 131072 cache, against stepping;
  * a tiny HF LLaMA with rope_scaling llama3 (original context 64, so all three bands act within 512 tokens): QuantLlamaAttention against HF's
    attention, the engine's score() and decode steps against HF's forward, and the unscaled rotation missing HF by more than 10x the bound.

The file sorts ahead of tests/test_gpu_exact.py for the reason tests/test_gpu_decode_gqa.py gives.
"""
import numpy as np
import pytest
import torch

import attn_probe as P
from exact_fixtures import matvec_takes
from gpu_util import assert_rel_close, report, ulp16
from llama_oracle import LlamaOracle, assert_no_failures, check_last_layer_blocks, step_all
from oracle import gptq_oracle as O
from test_gpu_decode_attention import Worst, anchors, bounded, heavy_passes

pytestmark = pytest.mark.gpu

LONG = [0, 1, 8191, 8192, 8193, 32767, 65535, 131070, 131071]
LLAMA3_EPS = 1e-5


def _engine():
    from gptq_b200 import engine
    return engine


def _table(scaling):
    from gptq_b200 import ops
    return ops.rope_inv_freq(_engine().LLAMA3_ROPE_BASE, 128, scaling)


def rope_table_inplace(qk, position_ids, inv_freq):
    """O.rope_inplace with the frequencies of a scaled rotation: qk fp16 [bsz, seq, 2, heads, head_dim] in place, angle_i = fp32(inv_freq[i] *
    pos), fp32 cos / sin, x' = x cos - y sin, y' = x sin + y cos with y at +head_dim / 2, fp16 store."""
    half = qk.shape[-1] // 2
    freq = torch.as_tensor(inv_freq, dtype=torch.float32).cpu()[None, None, :] * position_ids[:, :, None].float()
    cos, sin = torch.cos(freq)[:, :, None, None, :], torch.sin(freq)[:, :, None, None, :]
    x, y = qk[..., :half].float(), qk[..., half:].float()
    qk[..., :half] = (x * cos - y * sin).half()
    qk[..., half:] = (x * sin + y * cos).half()


def check_rope_row_table(k_row, k_exact, pos, inv_freq):
    """attn_probe.check_rope_row with the angles of a scaled rotation, fp32(inv_freq[i] * pos): the rotated rows [rows, 128] (fp16) against
    fp64 RoPE of the exact rows [rows * 128], within 1 ulp16 plus a 4-ulp difference in the fp32 angle and in cos / sin.  Returns the worst
    |err| / bound."""
    f = np.float32
    th = (np.asarray(inv_freq, dtype=f) * f(pos)).astype(np.float64)
    x = k_exact.view(-1, P.HD)[:, :64].numpy()
    y = k_exact.view(-1, P.HD)[:, 64:].numpy()
    c, s = np.cos(th), np.sin(th)
    ref = torch.from_numpy(np.concatenate([x * c - y * s, x * s + y * c], 1))
    dth = 4 * np.spacing(th.astype(f)).astype(np.float64) + 4 * P.U24
    slack = torch.from_numpy(np.tile((np.abs(x) + np.abs(y)) * dth, 2))
    return ((k_row.double().cpu() - ref).abs() / (ulp16(ref) + slack)).max().item()


class ScaledProbe(P.Probe):
    """attn_probe.Probe whose decoder rotates with the frequency table of `rope_scaling`: the same layer, embedding and lm_head in a decoder
    built with the table (the probe's own decoder is dropped)."""

    def __init__(self, size, rope_scaling, **kw):
        super().__init__(size, **kw)
        d = self.dec
        self.dec = _engine().LlamaDecoder(d.layers, d.embed, d.final_norm, d.lm_head, d.n_heads, rms_eps=d.model.rms_eps, batch=d.batch,
                                          max_seq=d.max_seq, rope_base=d.model.rope_base, n_kv_heads=d.n_kv_heads, rope_scaling=rope_scaling)
        del d
        torch.cuda.empty_cache()
        assert self.persistent == (self.dec.launches_per_step() == 1)


class ScaledOracle(LlamaOracle):
    """The reference decoder with n_kv_heads K/V heads (query head h reads K/V head h // g) and the rotation of the caller's table; the fp32
    lm_head is kept once (a 128256-row head is 4 GB in fp32)."""

    def __init__(self, dec, *, eps, inv_freq):
        super().__init__(dec.layers, dec.embed, dec.final_norm, dec.lm_head, dec.n_heads, eps=eps, base=None)
        self.n_kv_heads, self.inv_freq = dec.n_kv_heads, inv_freq
        self._head = self.lm_head.float().t().contiguous()

    def attention(self, li, x, pos, k_prefix=None, v_prefix=None, exact=False):
        n, nh, nkv, hd = x.shape[0], self.n_heads, self.n_kv_heads, self.head_dim
        qkv = self._linear(li, 'qkv', O.rmsnorm_fwd(x, self._layer(li)['input_norm'], self.eps), exact).view(1, n, nh + 2 * nkv, hd).clone()
        rope_table_inplace(qkv[:, :, None, :nh + nkv], torch.arange(pos, pos + n)[None, :], self.inv_freq)
        q, k, v = (t.transpose(0, 1) for t in qkv[0].split([nh, nkv, nkv], 1))
        K = torch.cat([k_prefix[:, :pos], k], 1) if pos else k
        V = torch.cat([v_prefix[:, :pos], v], 1) if pos else v
        s = (q.float().reshape(nkv, nh // nkv, n, hd) @ K.float()[:, None].transpose(-1, -2)) * hd**-0.5
        s = s.masked_fill(torch.ones(n, pos + n, dtype=torch.bool).triu(pos + 1), float('-inf'))
        att = (torch.softmax(s, -1) @ V.float()[:, None]).reshape(nh, n, hd).half().transpose(0, 1).reshape(n, self.hidden)
        return x + self._linear(li, 'o', att, exact), k, v

    def head(self, x):
        return (O.rmsnorm_fwd(x, self.final_norm, self.eps).float() @ self._head).half()


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
        worst = max(check_rope_row_table(out[0, t, :2].reshape(16, 128), x[0, t, :2].reshape(-1), p, table) for t, p in enumerate(positions))
        report(worst, f'gptq_rope_inplace_freq LLaMA-{name} vs fp64 RoPE')
        plain = x.cuda()
        ops.rotate_half_(plain[:, :, :2], pos.cuda(), base=engine.LLAMA3_ROPE_BASE)
        assert not torch.equal(plain.cpu()[0, 2:], out[0, 2:]), 'the table changed nothing'


# ----------------------------------------------------------------------------- planted caches at long positions, both engines
def _prefill_row(probe, tok, pos):
    """The K rows of position pos as the prefill writes them: the exact k of the probe (exact_qv) rotated by gptq_rope_inplace_freq."""
    from gptq_b200 import ops
    k = P.exact_qv(probe.w, probe.dec.embed[tok])[1].half().view(1, 1, 1, probe.nkv, 128).cuda()
    ops.rotate_half_(k, torch.tensor([[pos]], device='cuda'), inv_freq=probe.dec.rope_inv_freq)
    return k.view(probe.nkv, 128)


def long_sweep(probe, position_sets, name):
    gen = torch.Generator(device='cuda:0').manual_seed(4321)
    worst = {k: Worst(f'{name} {k}') for k in ('heavy', 'late', 'uniform')}
    rope = Worst(f'{name} appended K row vs fp64 RoPE')
    table = probe.dec.rope_inv_freq
    for i, positions in enumerate(position_sets):
        toks = [(11 * i + 5 * b + 1) % probe.dec.vocab for b in range(probe.B)]
        what = f'toks {toks} positions {positions}'
        probe.learn(toks, positions)
        for b, p in enumerate(positions):
            k_exact = P.exact_qv(probe.w, probe.dec.embed[toks[b]])[1]
            rope.update(check_rope_row_table(probe.k_new[b], k_exact, p, table), f'{what} seq {b}')
            assert torch.equal(probe.k_new[b], _prefill_row(probe, toks[b], p)), f'{what} seq {b}: the step and the prefill rotate differently'
        anchors(probe, toks, positions, gen, what)
        for heavy in heavy_passes(probe, positions, rotate=i * 8 * probe.nh):
            plants = [P.profile('heavy', q, p, gen, heavy=hv, g=probe.g) for q, p, hv in zip(probe.q_rot, positions, heavy)]
            bounded(probe, toks, positions, plants, worst['heavy'], what + ' heavy')
        for kind in ('late', 'uniform'):
            plants = [P.profile(kind, q, p, gen, g=probe.g) for q, p in zip(probe.q_rot, positions)]
            bounded(probe, toks, positions, plants, worst[kind], f'{what} {kind}')
    for w in list(worst.values()) + [rope]:
        w.done()


BATCH8 = [[131071, 131070, 65535, 32767, 8193, 8192, 8191, 1], [0, 100000, 131071, 12345, 8192, 77777, 50000, 131000]]


@pytest.mark.parametrize('size,batch', [('llama3-8b', 1), ('llama3-8b', 8), ('tiny-gqa2-chain', 1), ('tiny-gqa2-chain', 8)])
def test_long_positions_planted(size, batch):
    engine = _engine()
    probe = ScaledProbe(size, engine.LLAMA3_1_ROPE_SCALING, batch=batch, max_seq=131072, rope_base=engine.LLAMA3_ROPE_BASE)
    assert probe.persistent == (size == 'llama3-8b')
    sets = [[p] for p in LONG] if batch == 1 else BATCH8
    long_sweep(probe, sets, f'{size} batch {batch} llama3 (max_seq 131072)')


# ----------------------------------------------------------------------------- real LLaMA-3.x layers against the reference decoder
def _scaled_blocks(size, scaling, positions, max_seq, vocab=128256, tied=False, seed=21):
    """Two layers of a real shape on the persistent kernel with the table, a random cache, one step at each position, block by block against
    the reference with the same table (llama_oracle.check_last_layer_blocks)."""
    engine = _engine()
    kw = dict(rms_eps=LLAMA3_EPS, rope_base=engine.LLAMA3_ROPE_BASE, rope_scaling=scaling, max_seq=max_seq)
    dec2 = engine.synthetic_llama(size, bits=4, groupsize=128, vocab=vocab, seed=seed, n_layers=2, **kw)
    if tied:  # LLaMA-3.2-3B: the lm_head is the embedding
        dec2 = engine.LlamaDecoder(dec2.layers, dec2.embed, dec2.final_norm, dec2.embed, dec2.n_heads, n_kv_heads=dec2.n_kv_heads, **kw)
        assert dec2.lm_head.data_ptr() == dec2.embed.data_ptr()
    dec1 = engine.LlamaDecoder(dec2.layers[:1], dec2.embed, dec2.final_norm, dec2.lm_head, dec2.n_heads, n_kv_heads=dec2.n_kv_heads, **kw)
    assert dec1.launches_per_step() == 1 and dec2.launches_per_step() == 1
    assert torch.equal(dec2.rope_inv_freq, _table(scaling))
    gen = torch.Generator(device=dec2.dev).manual_seed(111)
    dec2.k_cache.copy_((torch.randn(dec2.k_cache.shape, device=dec2.dev, generator=gen) * 0.5).half())
    dec2.v_cache.copy_((torch.randn(dec2.v_cache.shape, device=dec2.dev, generator=gen) * 0.5).half())
    k0, v0 = dec2.k_cache.clone(), dec2.v_cache.clone()
    kc, vc = k0.cpu(), v0.cpu()
    oracle = ScaledOracle(dec2, eps=LLAMA3_EPS, inv_freq=_table(scaling))
    for i, pos in enumerate(positions):
        tok = (17 * i + 3) % vocab
        what = f'{size} llama3 pos={pos}'
        for dec in (dec1, dec2):
            dec.k_cache.copy_(k0[:len(dec.layers)])
            dec.v_cache.copy_(v0[:len(dec.layers)])
        check_last_layer_blocks(dec1, oracle, tok, pos, kc, vc, what + ' (1 layer)', False)
        check_last_layer_blocks(dec2, oracle, tok, pos, kc, vc, what + ' (2 layers)', False)
        assert_no_failures()
    return dec2, oracle


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
    dec, oracle = _scaled_blocks('llama3-8b', engine.LLAMA3_1_ROPE_SCALING, [0, 2047, 8191, 8192, 12000], 12288)
    # sampled generation over the whole 128256-id vocabulary on the scaled model
    prompt = [5, 128255, 77, 1000]
    sampled = dec.generate(prompt, 6, do_sample=True, temperature=0.8, top_k=0, top_p=0.95, seed=5)
    assert sampled[:4] == prompt and len(sampled) == 10 and all(0 <= t < 128256 for t in sampled)


def test_llama31_70b():
    """LLaMA-3.1-70B (and 3.3-70B, the same shape and scaling): batch 1 on the persistent kernel block by block, batch 8 on the kernel chain,
    whose launch count follows the matvec route rule (exact_fixtures.matvec_takes)."""
    engine = _engine()
    dec, oracle = _scaled_blocks('70b', engine.LLAMA3_3_ROPE_SCALING, [0, 8192], 8448, seed=22)
    d8 = engine.LlamaDecoder(dec.layers, dec.embed, dec.final_norm, dec.lm_head, dec.n_heads, n_kv_heads=8, batch=8, max_seq=64, rms_eps=LLAMA3_EPS,
                             rope_base=engine.LLAMA3_ROPE_BASE, rope_scaling=engine.LLAMA3_1_ROPE_SCALING)
    H, I, Hkv = dec.hidden, dec.intermediate, 8 * 128
    per_layer = 2 + sum(1 if matvec_takes(8, K, N) else 2 for K, N in ((H, H + 2 * Hkv), (H, H), (H, I), (I, H)))
    assert d8.launches_per_step() == 3 + 2 * per_layer, d8.launches_per_step()
    _batch_steps(d8, oracle, 4, 128256, '70b batch 8 chain')


@pytest.mark.parametrize('batch', [1, 8])
def test_llama32_3b_tied(batch):
    engine = _engine()
    if batch == 1:
        _scaled_blocks('llama3.2-3b', engine.LLAMA3_2_ROPE_SCALING, [0, 8192, 30000], 32768, tied=True, seed=23)
        return
    base = engine.synthetic_llama('llama3.2-3b', bits=4, groupsize=128, vocab=128256, seed=23, n_layers=2, max_seq=16)
    dec = engine.LlamaDecoder(base.layers, base.embed, base.final_norm, base.embed, base.n_heads, n_kv_heads=8, batch=8, max_seq=16, rms_eps=LLAMA3_EPS,
                              rope_base=engine.LLAMA3_ROPE_BASE, rope_scaling=engine.LLAMA3_2_ROPE_SCALING)
    assert dec.lm_head.data_ptr() == dec.embed.data_ptr() and dec.launches_per_step() == 1
    _batch_steps(dec, ScaledOracle(dec, eps=LLAMA3_EPS, inv_freq=_table(engine.LLAMA3_2_ROPE_SCALING)), 5, 128256, '3.2-3b batch 8')


# ----------------------------------------------------------------------------- long prompts: prefill and extend against stepping
def _extend_vs_steps(dec, toks, prefilled, cached, what, fill='prefill'):
    """Fill toks[:prefilled] (by prefill, or by extend() from an empty cache), step to `cached`, extend() to the last token and step it; against
    the same fill and stepping every later token.  The bound of llama_oracle.check_extend_against_stepping (the run-to-run spread of DESIGN.md
    section 2)."""
    n = len(toks)
    runs = []
    for extend in (True, False):
        dec.reset()
        dec.k_cache.zero_()
        dec.v_cache.zero_()
        if fill == 'prefill':
            assert dec.prefill(toks[:prefilled + 1]) == prefilled
        else:
            assert dec.extend([toks[:prefilled]]) == [prefilled]
        step_all(dec, toks[prefilled:cached], prefilled)
        if extend:
            assert dec.extend([toks[cached:n - 1]]) == [n - 1]
            step_all(dec, toks[n - 1:], n - 1)
        else:
            step_all(dec, toks[cached:], cached)
        runs.append([dec.logits[0].float().clone(), dec.k_cache[:, 0, :, prefilled:n].float().clone(), dec.v_cache[:, 0, :, prefilled:n].float().clone()])
    for name, g, r in zip(('logits', 'K rows', 'V rows'), *runs):
        rms = r.pow(2).mean().sqrt().item()
        d = (g - r).abs()
        print(f'  {what} {name}: max |diff| / rms = {d.max().item() / rms:.3g}, rms diff / rms = {d.pow(2).mean().sqrt().item() / rms:.3g}')
        assert d.max().item() <= 1.5e-2 * rms and d.pow(2).mean().sqrt().item() <= 3e-3 * rms, f'{what}: {name}'


def test_long_prompts_prefill_and_extend():
    engine = _engine()
    dec = engine.synthetic_llama('llama3-8b', bits=4, groupsize=128, vocab=128256, seed=24, n_layers=2, max_seq=131072, rms_eps=LLAMA3_EPS,
                                 rope_base=engine.LLAMA3_ROPE_BASE, rope_scaling=engine.LLAMA3_1_ROPE_SCALING)
    assert dec.launches_per_step() == 1
    toks = torch.randint(0, 128256, (131072, ), generator=torch.Generator().manual_seed(8)).tolist()
    _extend_vs_steps(dec, toks[:8400], 8000, 8100, 'llama3.1-8b across 8192')
    # (the first 130800 rows through extend(): its attention is the cache kernel, where the prefill's SDPA would hold 130800 rows at once)
    _extend_vs_steps(dec, toks, 130800, 130816, 'llama3.1-8b to the last row of 131072', fill='extend')


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
