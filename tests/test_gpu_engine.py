"""GPU: the decode engine (gptq_llama_decode_step through the C ABI, CUDA-graph replayed) against the CPU reference decoder
(tests/llama_oracle.py)."""
import pytest
import torch

from gpu_util import assert_rel_close, tiny_quant_llama
from llama_oracle import CODELLAMA, LLAMA1, LlamaOracle, check_steps, scale_down_embedding_row

pytestmark = pytest.mark.gpu


DECODE_CASES = [('tiny', 4, False, True), ('tiny', 4, False, False), ('tiny', 4, True, True), ('tiny', 8, False, True), ('tiny', 3, True, True),
                ('tiny256', 4, False, True), ('tiny256', 4, False, False), ('tiny256', 4, True, True), ('tiny256', 3, True, True), ('tiny256', 3, False, True),
                ('tiny256', 2, True, False)]


@pytest.mark.parametrize('size,bits,act,use_graph,rope', [pytest.param(*c, LLAMA1, id='-'.join(map(str, c))) for c in DECODE_CASES] +
                         [pytest.param(size, 4, False, True, CODELLAMA, id=f'{size}-4-False-True-codellama') for size in ('tiny', 'tiny256')])
def test_decode_steps_match_oracle(size, bits, act, use_graph, rope):
    """Six decode steps against the oracle, on the kernel chain (tiny) and the persistent kernel (tiny256).  At the CodeLlama settings (RoPE
    base 1e6, RMSNorm epsilon 1e-5) the first token's embedding row is scaled to a mean square of about 4e-6, near the epsilon, so that the
    decoder's epsilon shows in the output."""
    from gptq_b200 import engine
    base, eps = rope
    dec = engine.synthetic_llama(size, bits=bits, groupsize=64, act_order=act, vocab=512, seed=bits, max_seq=600, use_graph=use_graph, rope_base=base,
                                 rms_eps=eps)
    if size == 'tiny256':
        # persistent single-kernel path, also for act-order (regrouped rows + input gathers) and 2/3-bit (nibble-widened) layers
        assert dec.launches_per_step() == 1
        assert all(k['qkv'].bits == 4 and k['qkv'].hint == 64 for k in dec.klayers)
        assert (dec.perms[0]['qkv'] is not None) == act
    else:
        assert dec.launches_per_step() > 1 and all(pm['qkv'] is None for pm in dec.perms)
    gen = torch.Generator().manual_seed(0)
    toks = torch.randint(0, 512, (6, ), generator=gen).tolist()
    if rope != LLAMA1:
        scale_down_embedding_row(dec.embed, toks[0], 8)
    check_steps(dec, LlamaOracle.from_decoder(dec, eps=eps, base=base), [toks], lambda k, b, pos: f'{size} bits={bits} act={act} base={base:g} eps={eps:g} pos={pos}')


@pytest.mark.parametrize('gs,rope', [pytest.param(-1, LLAMA1, id='-1'), pytest.param(32, LLAMA1, id='32'), pytest.param(32, CODELLAMA, id='32-codellama')])
def test_hf_checkpoint_groupsizes_decode_on_the_persistent_kernel(gs, rope):
    """The route a real checkpoint takes (the reference's load_quant recipe on the quant modules -> engine.from_hf_quant_model) at
    --groupsize -1 (QuantLinear takes groupsize = infeatures: 256 for qkv / o / gate / up, 768 for down) and 32: the persistent kernel
    serves it with every groupsize hint intact, and six decode steps match the oracle at the bound of test_decode_steps_match_oracle.  At the
    CodeLlama settings (config rope_theta 1e6, rms_norm_eps 1e-5) the decoder must take both from the checkpoint's config; the first token's
    embedding row is scaled to a mean square of about 1.6e-6 (HF's init has std 0.02) so that the epsilon shows in the output."""
    import quant
    from gptq_b200 import engine
    base, eps = rope
    model = tiny_quant_llama(gs=gs, hidden=256, intermediate=768, heads=2, rope_theta=base, rms_norm_eps=eps)
    toks = torch.randint(0, model.config.vocab_size, (6, ), generator=torch.Generator().manual_seed(gs + 2)).tolist()
    if rope != LLAMA1:
        scale_down_embedding_row(model.model.embed_tokens.weight, toks[0], 4)
    quant.make_quant_attn(model)
    quant.make_quant_norm(model)
    quant.make_fused_mlp(model)
    dec = engine.from_hf_quant_model(model.cuda(), max_seq=16)
    assert dec.launches_per_step() == 1
    assert (dec.model.rope_base, dec.model.rms_eps) == (base, pytest.approx(eps, rel=1e-7))
    for kl in dec.klayers:
        for name in ('qkv', 'o', 'gate', 'up', 'down'):
            K = kl[name].g_idx.numel()
            assert kl[name].hint == (K if gs == -1 else gs), f'{name}: groupsize hint {kl[name].hint}'
    check_steps(dec, LlamaOracle.from_decoder(dec, eps=eps, base=base), [toks], lambda k, b, pos: f'gs={gs} base={base:g} eps={eps:g} pos={pos}')


@pytest.mark.parametrize('size', ['tiny', 'tiny256'])
def test_long_context_attention_splits(size):
    """Positions beyond one attention chunk: split-KV partials + combine against the oracle (both engines)."""
    from gptq_b200 import engine
    dec = engine.synthetic_llama(size, bits=4, groupsize=128, vocab=256, seed=1, max_seq=640)
    toks = torch.randint(0, 256, (530, ), generator=torch.Generator().manual_seed(1)).tolist()
    check_steps(dec, LlamaOracle.from_decoder(dec, eps=1e-6, base=10000.0), [toks], lambda k, b, pos: f'pos={pos}', rel=3e-2,
                checked=(0, 255, 256, 257, 511, 512, 529))


def test_generate_is_deterministic_and_matches_stepwise():
    from gptq_b200 import engine
    dec = engine.synthetic_llama('tiny', bits=4, groupsize=64, vocab=300, seed=2, max_seq=64)
    a = dec.generate([5, 7, 11], 8)
    b = dec.generate([5, 7, 11], 8)
    assert a == b and len(a) == 11 and a[:3] == [5, 7, 11]


def test_batched_decode_matches_single():
    from gptq_b200 import engine
    d1 = engine.synthetic_llama('tiny', bits=4, groupsize=64, vocab=300, seed=3, max_seq=32, batch=1)
    d4 = engine.synthetic_llama('tiny', bits=4, groupsize=64, vocab=300, seed=3, max_seq=32, batch=4)
    seqs = torch.randint(0, 300, (4, 5), generator=torch.Generator().manual_seed(0))
    for pos in range(5):
        d4.tokens.copy_(seqs[:, pos].int())
        d4.positions.fill_(pos)
        d4.step()
    torch.cuda.synchronize()
    batched = d4.logits.clone()
    for b in range(4):
        for pos in range(5):
            d1.tokens.fill_(int(seqs[b, pos]))
            d1.positions.fill_(pos)
            d1.step()
        torch.cuda.synchronize()
        assert_rel_close(batched[b], d1.logits[0], rel=1e-2, what=f'batch row {b}')


def test_host_rejects_positions_and_tokens_outside_the_cache_and_vocabulary():
    """The kernels index the KV cache with the step's position and the embedding with the token id: the host API validates both
    (ADVICE r1), the kernels clamp as a last line of defence."""
    from gptq_b200 import engine
    dec = engine.synthetic_llama('tiny256', bits=4, groupsize=64, vocab=300, seed=4, max_seq=16)
    with pytest.raises(ValueError):
        dec.generate([1, 2, 3], 15)  # 3 + 15 - 1 positions > max_seq
    with pytest.raises(ValueError):
        dec.generate([1, 300], 2)
    with pytest.raises(ValueError):
        dec.set_input(5, 16)
    with pytest.raises(ValueError):
        dec.set_input(-1, 0)
    out = dec.generate([1, 2, 3], 14)  # exactly fills the cache
    assert len(out) == 17
    # a raw out-of-range position is clamped by the kernel instead of writing past the cache
    guard = dec.k_cache.clone()
    dec.tokens.fill_(7)
    dec.positions.fill_(10_000)
    dec.step()
    torch.cuda.synchronize()
    assert torch.isfinite(dec.logits).all()
    assert torch.equal(dec.k_cache[:, :, :, :15], guard[:, :, :, :15])  # only the last row may have been rewritten


@pytest.mark.parametrize('size', ['tiny', 'tiny256'])
def test_prefill_then_decode_matches_token_by_token(size):
    """One engine, two phases: the batched prefill (wgmma GEMM path + SDPA, filling the static KV cache) followed by the decode kernel gives the
    same cache rows and the same next-token logits as feeding the prompt token by token through the decode step."""
    from gptq_b200 import engine
    dec = engine.synthetic_llama(size, bits=4, groupsize=64, vocab=300, seed=5, max_seq=96)
    prompt = torch.randint(0, 300, (40, ), generator=torch.Generator().manual_seed(2)).tolist()
    for pos, tok in enumerate(prompt):
        dec.set_input(tok, pos)
        dec.step()
    torch.cuda.synchronize()
    ref_logits, ref_k, ref_v = dec.logits[0].float().clone(), dec.k_cache[:, 0, :, :40].float().clone(), dec.v_cache[:, 0, :, :40].float().clone()
    dec.k_cache.zero_()
    dec.v_cache.zero_()
    assert dec.prefill(prompt) == 39
    assert_rel_close(dec.k_cache[:, 0, :, :39], ref_k[:, :, :39], rel=1e-2, what='prefilled K rows')
    assert_rel_close(dec.v_cache[:, 0, :, :39], ref_v[:, :, :39], rel=1e-2, what='prefilled V rows')
    dec.set_input(prompt[-1], 39)
    dec.step()
    torch.cuda.synchronize()
    assert_rel_close(dec.logits[0], ref_logits, rel=2e-2, what='logits after prefill + 1 decode step')
    a, b = dec.generate(prompt[:12], 10, prefill=True), dec.generate(prompt[:12], 10, prefill=False)
    assert len(a) == 22 and a[:12] == prompt[:12] and sum(x != y for x, y in zip(a, b)) <= 2  # greedy picks may flip on near-ties
