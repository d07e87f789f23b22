"""GPU: extending cached sequences -- LlamaDecoder.extend (the ragged pass with gptq_cached_attention over the KV cache) against the decode step
and the prefill, on both engines (tiny: kernel chain, tiny256: persistent kernel) and an int3 act-order model; the host-side record
(lengths, cached tokens); generate / generate_batch with reuse_cache=True over several turns; errors; LLaMA-7B shapes."""
import pytest
import torch

from gpu_util import assert_rel_close, run_kernel
from llama_oracle import check_extend_against_stepping, step_all

pytestmark = pytest.mark.gpu

MODELS = [('tiny', 4, False), ('tiny256', 4, False), ('tiny256', 3, True)]


def _model(size, bits, act, seed, gs=64, **kw):
    from gptq_b200 import engine
    return engine.synthetic_llama(size, bits=bits, groupsize=gs, act_order=act, vocab=300, seed=seed, **kw)


def _ids(n, seed):
    return torch.randint(0, 300, (n, ), generator=torch.Generator().manual_seed(seed)).tolist()


@pytest.mark.parametrize('size, bits, act, rope_base, cached', [pytest.param(*m, 10000.0, 10, id='-'.join(map(str, m))) for m in MODELS] +
                         [pytest.param(size, 4, False, 1e6, 2060, id=f'{size}-4-False-base1e6-cached2060') for size in ('tiny', 'tiny256')])
def test_extend_after_decode_matches_stepping(size, bits, act, rope_base, cached):
    """`cached` decode steps, then extend() with the next 29 tokens: the same cache rows as stepping them (1e-2) and the same logits at the
    next step (2e-2), the bounds of test_prefill_then_decode_matches_token_by_token.  At RoPE base 1e6 with 2060 cached positions the
    extend pass rotates with the RoPE kernel and the stepping with the decode kernel, at positions past 2048."""
    _extend_after_decode(_model(size, bits, act, seed=5, max_seq=cached + 86, rope_base=rope_base), what=f'{size} base={rope_base:g} cached={cached}',
                         cached=cached)


@pytest.mark.parametrize('gs, kernel', [(32, 'qlinear_generic_kernel'), (-1, 'qgemm_wgmma_kernel')])
def test_extend_after_decode_at_groupsizes(gs, kernel):
    """The same on the persistent-kernel model at groupsize 32 and -1 (one group per linear: 256, and 768 on down_proj).  The 29-row pass
    asserts its kernels: the wgmma GEMM needs groupsize % 64 == 0, so at 32 every quantized linear of it runs on the generic kernel."""
    dec = _model('tiny256', 4, False, seed=5, gs=gs, max_seq=96)
    assert dec.launches_per_step() == 1
    _extend_after_decode(dec, kernel, f'gs={gs}')


def _extend_after_decode(dec, kernel=None, what='', cached=10):
    c, e = cached, cached + 29
    prompt = _ids(e + 1, 2)
    step_all(dec, prompt, 0)
    ref_logits, ref_k, ref_v = dec.logits[0].float().clone(), dec.k_cache[:, 0, :, :e + 1].float().clone(), dec.v_cache[:, 0, :, :e + 1].float().clone()
    dec.reset()
    dec.k_cache.zero_()
    dec.v_cache.zero_()
    step_all(dec, prompt[:c], 0)
    assert dec.lengths == [c] and dec.cached_tokens == [prompt[:c]]

    def extend():  # repeatable (run_kernel may trace it again): from the c cached positions each time
        dec.lengths, dec.cached_tokens = [c], [prompt[:c]]
        return dec.extend([prompt[c:e]])

    assert (extend() if kernel is None else run_kernel(extend, kernel, f'extend of 29 rows {what}')) == [e]
    assert dec.lengths == [e] and dec.cached_tokens == [prompt[:e]]
    assert_rel_close(dec.k_cache[:, 0, :, c:e], ref_k[:, :, c:e], rel=1e-2, what=f'extended K rows {what}')
    assert_rel_close(dec.v_cache[:, 0, :, c:e], ref_v[:, :, c:e], rel=1e-2, what=f'extended V rows {what}')
    dec.set_input(prompt[e], e)
    dec.step()
    torch.cuda.synchronize()
    assert_rel_close(dec.logits[0], ref_logits, rel=2e-2, what=f'logits after extend + 1 decode step {what}')


@pytest.mark.parametrize('size, bits, act', MODELS)
def test_extend_from_an_empty_cache_matches_prefill(size, bits, act):
    dec = _model(size, bits, act, seed=6, max_seq=200)
    prompt = _ids(150, 3)
    assert dec.prefill_batch([prompt]) == [149]
    ref_k, ref_v = dec.k_cache[:, 0, :, :149].float().clone(), dec.v_cache[:, 0, :, :149].float().clone()
    dec.reset()
    dec.k_cache.zero_()
    dec.v_cache.zero_()
    assert dec.extend([prompt[:149]]) == [149]
    assert_rel_close(dec.k_cache[:, 0, :, :149], ref_k, rel=1e-2, what='K rows: extend from 0 against prefill')
    assert_rel_close(dec.v_cache[:, 0, :, :149], ref_v, rel=1e-2, what='V rows: extend from 0 against prefill')


@pytest.mark.parametrize('size', ['tiny', 'tiny256'])
def test_ragged_batch_extend(size):
    """Chunks of 0, 1, 17 and 40 tokens on sequences with 4, 0, 29 and 11 cached positions: the right lengths; the sequence with the empty
    chunk, every cached row before the chunks and every row past the new lengths stay bit-identical; each sequence's new rows match a batch-1
    extend of the same sequence (1e-2)."""
    from gptq_b200 import engine
    dec = _model(size, 4, False, seed=7, max_seq=64, batch=4)
    prompts = [_ids(n, 10 + n) for n in (5, 1, 30, 12)]
    assert dec.prefill_batch(prompts) == [4, 0, 29, 11]
    chunks = [[], _ids(1, 20), _ids(17, 21), _ids(40, 22)]
    k0, v0 = dec.k_cache.clone(), dec.v_cache.clone()
    assert dec.extend(chunks) == [4, 1, 46, 51] == dec.lengths
    for b, (old, new) in enumerate(zip([4, 0, 29, 11], dec.lengths)):
        assert dec.cached_tokens[b] == prompts[b][:old] + chunks[b]
        for c, c0 in ((dec.k_cache, k0), (dec.v_cache, v0)):
            assert torch.equal(c[:, b, :, :old], c0[:, b, :, :old]), f'sequence {b}: cached rows changed'
            assert torch.equal(c[:, b, :, new:], c0[:, b, :, new:]), f'sequence {b}: rows past the new length changed'
    one = engine.LlamaDecoder(dec.layers, dec.embed, dec.final_norm, dec.lm_head, dec.n_heads, max_seq=64, use_graph=False)
    for b in (1, 2, 3):
        one.reset()
        one.prefill_batch([prompts[b]])
        one.extend([chunks[b]])
        old, new = len(prompts[b]) - 1, dec.lengths[b]
        assert_rel_close(dec.k_cache[:, b, :, old:new], one.k_cache[:, 0, :, old:new], rel=1e-2, what=f'sequence {b}: K rows against batch 1')
        assert_rel_close(dec.v_cache[:, b, :, old:new], one.v_cache[:, 0, :, old:new], rel=1e-2, what=f'sequence {b}: V rows against batch 1')


@pytest.mark.parametrize('size, bits, act', MODELS)
def test_multi_turn_generate_batch_reuses_the_conversation(size, bits, act):
    """Turn 1: generate_batch(p1).  Turn 2: the outputs plus a new turn each, with reuse_cache=True: the same tokens as a fresh generate_batch of
    the same prompts (at most 2 greedy flips per sequence, the near-tie rule), and the reused rows are left bit-identical (only the new turn
    is computed).  Turn 3 repeats it on top of turn 2."""
    dec = _model(size, bits, act, seed=8, max_seq=96, batch=4)
    p = [_ids(n, 30 + n) for n in (3, 8, 20, 1)]
    out = dec.generate_batch(p, 10)
    for turn, lens in enumerate(((5, 1, 12, 7), (2, 9, 1, 4))):
        cached = list(dec.lengths)
        assert cached == [len(o) - 1 for o in out]
        k0, v0 = dec.k_cache.clone(), dec.v_cache.clone()
        p = [o + _ids(n, 50 + 10 * turn + n) for o, n in zip(out, lens)]
        out = dec.generate_batch(p, 10, reuse_cache=True)
        for b, c in enumerate(cached):
            assert torch.equal(dec.k_cache[:, b, :, :c], k0[:, b, :, :c]) and torch.equal(dec.v_cache[:, b, :, :c], v0[:, b, :, :c]), \
                f'turn {turn + 2}, sequence {b}: reused rows were rewritten'
        lengths, tokens = list(dec.lengths), [list(t) for t in dec.cached_tokens]
        k1, v1 = dec.k_cache.clone(), dec.v_cache.clone()
        fresh = dec.generate_batch(p, 10)
        for b, (o, f) in enumerate(zip(out, fresh)):
            assert len(o) == len(p[b]) + 10 and o[:len(p[b])] == p[b]
            assert sum(x != y for x, y in zip(o, f)) <= 2, f'turn {turn + 2}, sequence {b}: {o[len(p[b]):]} vs {f[len(p[b]):]}'
        dec.k_cache.copy_(k1)  # continue from the reused conversation, not the fresh one
        dec.v_cache.copy_(v1)
        dec.lengths, dec.cached_tokens = lengths, tokens


@pytest.mark.parametrize('size', ['tiny', 'tiny256'])
def test_prefix_edge_cases(size):
    """An edited middle turn reuses only the common prefix (and matches a fresh run); an identical repeated prompt re-steps only its last token
    (no ragged pass at all); a shorter prompt keeps only its own prefix."""
    dec = _model(size, 4, False, seed=9, max_seq=96)
    prompt = _ids(30, 4)
    a = dec.generate(prompt, 8)
    passes = []
    forward = dec._forward_rows
    dec._forward_rows = lambda seqs, **kw: passes.append([len(s) for s in seqs]) or forward(seqs, **kw)
    try:
        again = dec.generate(prompt, 8, reuse_cache=True)
        assert passes == []  # only the last prompt token went through the decode step
        assert again[:30] == prompt and sum(x != y for x, y in zip(again, a)) <= 2
        assert dec.lengths == [len(a) - 1]
        edited = list(a)
        edited[12] = (edited[12] + 1) % 300
        k0 = dec.k_cache.clone()
        b = dec.generate(edited, 5, reuse_cache=True)
        assert passes == [[len(edited) - 1 - 12]]  # positions 12 .. len - 2 recomputed
        assert torch.equal(dec.k_cache[:, 0, :, :12], k0[:, 0, :, :12])
        assert dec.cached_tokens[0][:len(edited)] == edited
        short = dec.generate(prompt[:7], 3, reuse_cache=True)
        assert len(passes) == 1  # 6 positions kept: nothing to extend
        assert dec.lengths == [7 + 3 - 1]
    finally:
        dec._forward_rows = forward
    fresh_b, fresh_short = dec.generate(edited, 5), dec.generate(prompt[:7], 3)
    assert sum(x != y for x, y in zip(b, fresh_b)) <= 2 and sum(x != y for x, y in zip(short, fresh_short)) <= 2


@pytest.mark.parametrize('size', ['tiny', 'tiny256'])
def test_errors_leave_the_state_untouched(size):
    dec = _model(size, 4, False, seed=10, max_seq=32, batch=2)
    dec.prefill_batch([_ids(20, 1), _ids(3, 2)])
    k0, lengths = dec.k_cache.clone(), list(dec.lengths)
    for bad in ([_ids(14, 3), []],  # 19 + 14 > 32
                [[], [0, 300]],  # outside the vocabulary
                [[], [-1]],
                [[1, 2]]):  # one chunk per sequence
        with pytest.raises(ValueError):
            dec.extend(bad)
        assert dec.lengths == lengths and torch.equal(dec.k_cache, k0)
    with pytest.raises(ValueError):
        dec.generate_batch([_ids(30, 4), _ids(2, 5)], 4, reuse_cache=True)  # 30 + 4 > max_seq + 1
    assert dec.extend([_ids(13, 3), []]) == [32, 2]  # exactly full
    # tensor parallelism: extend and reuse_cache are refused before anything runs (the check reads only the decoder's tp setting)
    dec.tp = (0, 2, 0, 150)
    try:
        with pytest.raises(ValueError):
            dec.extend([[], [1]])
        with pytest.raises(ValueError):
            dec.generate_batch([[1, 2], [3]], 2, reuse_cache=True)
    finally:
        dec.tp = None


def test_llama_7b_shapes_extend_256_at_1791():
    """LLaMA-7B shapes (int4 g128, 2 layers, persistent kernel): 1791 positions stepped, then 256 more through extend(), then one step; against
    stepping all of them.  Cache rows and logits within the run-to-run spread of DESIGN.md section 2 (max 1.5e-2, rms 3e-3 of the rms)."""
    from gptq_b200 import engine
    dec = engine.synthetic_llama('7b', bits=4, groupsize=128, vocab=32000, seed=15, max_seq=2048, n_layers=2)
    assert dec.launches_per_step() == 1
    toks = torch.randint(0, 32000, (2048, ), generator=torch.Generator().manual_seed(5)).tolist()
    check_extend_against_stepping(dec, toks, 1791, '7b extend')
