"""GPU: the persistent decode kernel at batch 2..8 (one launch steps every sequence, each at its own position) and the batched host
interface (set_input with per-sequence positions, prefill_batch, generate_batch)."""
import pytest
import torch

from gpu_util import assert_rel_close
from llama_oracle import LlamaOracle, check_steps

pytestmark = pytest.mark.gpu

# A batched step and a batch-1 step of the same sequence differ only in the fp32 summation order of the split-K partial sums and of the
# lm_head: the bound of the measured run-to-run spread of one kernel (test_gpu_engine_fullsize.test_mega_kernel_run_to_run_spread_7b).
SPREAD_MAX, SPREAD_RMS = 1.5e-2, 3e-3


def _check_rows(batched, singles, what):
    """Row b of the batched logits against the batch-1 step of sequence b; the greedy tokens must agree where the margin is clear."""
    for b, ref in enumerate(singles):
        out, ref = batched[b].float(), ref.float()
        rms = ref.pow(2).mean().sqrt().item()
        err = (out - ref).abs()
        assert err.max().item() <= SPREAD_MAX * rms, f'{what} row {b}: max err {err.max().item():.3e} vs rms {rms:.3e}'
        assert err.pow(2).mean().sqrt().item() <= SPREAD_RMS * rms, f'{what} row {b}: rms err {err.pow(2).mean().sqrt().item():.3e} vs rms {rms:.3e}'
        top2 = ref.topk(2).values
        if (top2[0] - top2[1]).item() > SPREAD_MAX * rms:
            assert int(out.argmax()) == int(ref.argmax()), f'{what} row {b}: greedy token differs'


def _single_twin(dec):
    """A batch-1 decoder on the same weights."""
    from gptq_b200 import engine
    return engine.LlamaDecoder(dec.layers, dec.embed, dec.final_norm, dec.lm_head, dec.n_heads, max_seq=dec.max_seq)


def _singles(dec1, decb, toks, positions):
    """Logits of the batch-1 step of every sequence of decb, from that sequence's cache slot."""
    out = []
    for b, (tok, pos) in enumerate(zip(toks, positions)):
        dec1.k_cache.copy_(decb.k_cache[:, b:b + 1])
        dec1.v_cache.copy_(decb.v_cache[:, b:b + 1])
        dec1.set_input(tok, pos)
        dec1.step()
        torch.cuda.synchronize()
        out.append(dec1.logits[0].clone())
    return out


@pytest.mark.parametrize('batch', [2, 3, 8])
@pytest.mark.parametrize('size,bits,act', [('tiny256', 4, False), ('tiny256', 4, True), ('tiny256', 3, True), ('tiny512', 4, False), ('tiny512', 4, True),
                                           ('tiny512', 3, True)])
def test_batch_columns_match_oracle(size, bits, act, batch):
    """Distinct token streams in the batch columns, stepped at positions 0..5, against the oracle row by row (the bound of
    test_gpu_engine.test_decode_steps_match_oracle).  Batch 3 leaves lanes past the batch in the mma B operand."""
    from gptq_b200 import engine
    dec = engine.synthetic_llama(size, bits=bits, groupsize=64, act_order=act, vocab=512, seed=bits + batch, max_seq=64, batch=batch)
    assert dec.launches_per_step() == 1
    assert (dec.perms[0]['qkv'] is not None) == act
    toks = torch.randint(0, 512, (batch, 6), generator=torch.Generator().manual_seed(batch)).tolist()
    check_steps(dec, LlamaOracle.from_decoder(dec, eps=1e-6, base=10000.0), toks, lambda k, b, pos: f'{size} bits={bits} act={act} B={batch} seq={b} pos={pos}')


@pytest.mark.parametrize('size,bits,act,positions', [('7b', 4, False, [0, 31, 32, 255, 256, 1023, 2046, 2047]), ('13b', 3, True, [0, 255, 1023, 2047])])
def test_ragged_positions_match_single_sequence_steps(size, bits, act, positions):
    """At the shapes bench.py measures (2 layers): every sequence at a different position, one batched step against the batch-1
    persistent step of each sequence from the same cache slot."""
    from gptq_b200 import engine
    B = len(positions)
    dec = engine.synthetic_llama(size, bits=bits, groupsize=128, act_order=act, vocab=8192, seed=21, max_seq=2048, n_layers=2, batch=B)
    assert dec.launches_per_step() == 1
    dec1 = _single_twin(dec)
    assert dec1.launches_per_step() == 1
    gen = torch.Generator(device=dec.dev).manual_seed(22)
    dec.k_cache.normal_(0, 0.5, generator=gen)
    dec.v_cache.normal_(0, 0.5, generator=gen)
    toks = [(37 * b + 5) % 8192 for b in range(B)]
    singles = _singles(dec1, dec, toks, positions)
    dec.set_input(toks, positions)
    dec.step()
    torch.cuda.synchronize()
    _check_rows(dec.logits, singles, f'{size} int{bits} act={act}')


def test_ragged_positions_match_single_sequence_steps_65b():
    """The same at bench.py's 65B shapes (int4 g128, 2 layers) and the largest batch the persistent plan takes there (64 heads: 4 sequences on
    132 SMs)."""
    from gptq_b200 import engine
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    B = min(8, 2 * sms // 64)
    positions = [0, 2047, 256, 1023, 31, 32, 255, 2046][:B]
    dec = engine.synthetic_llama('65b', bits=4, groupsize=128, vocab=8192, seed=23, max_seq=2048, n_layers=2, batch=B)
    assert dec.launches_per_step() == 1, f'batch {B}: {dec.launches_per_step()} launches'
    dec1 = _single_twin(dec)
    assert dec1.launches_per_step() == 1
    gen = torch.Generator(device=dec.dev).manual_seed(24)
    dec.k_cache.normal_(0, 0.5, generator=gen)
    dec.v_cache.normal_(0, 0.5, generator=gen)
    toks = [(37 * b + 5) % 8192 for b in range(B)]
    singles = _singles(dec1, dec, toks, positions)
    dec.set_input(toks, positions)
    dec.step()
    torch.cuda.synchronize()
    _check_rows(dec.logits, singles, f'65b batch {B}')


def test_batched_step_writes_only_its_own_cache_rows():
    """A batched step rewrites one K row and one V row per sequence and layer, at that sequence's position; a position outside the cache
    is clamped for its own sequence only."""
    from gptq_b200 import engine
    dec = engine.synthetic_llama('tiny256', bits=4, groupsize=64, vocab=300, seed=6, max_seq=32, batch=3)
    assert dec.launches_per_step() == 1
    dec.k_cache.normal_(0, 0.5)
    dec.v_cache.normal_(0, 0.5)

    def step(positions, written):
        k0, v0 = dec.k_cache.clone(), dec.v_cache.clone()
        dec.tokens.copy_(torch.tensor([7, 8, 9], dtype=torch.int32))
        dec.positions.copy_(torch.tensor(positions, dtype=torch.int32))  # raw: set_input would reject 10_000
        dec.step()
        torch.cuda.synchronize()
        keep = torch.ones(dec.k_cache.shape[:4], dtype=torch.bool, device=dec.dev)
        for b, p in enumerate(written):
            keep[:, b, :, p] = False
        assert torch.equal(dec.k_cache[keep], k0[keep]) and torch.equal(dec.v_cache[keep], v0[keep]), f'rows outside {written} changed'
        assert not torch.equal(dec.k_cache[~keep], k0[~keep])
        assert torch.isfinite(dec.logits).all()
        return dec.logits.clone()

    kc, vc = dec.k_cache.clone(), dec.v_cache.clone()
    clamped = step([3, 10_000, 7], [3, 31, 7])
    dec.k_cache.copy_(kc)
    dec.v_cache.copy_(vc)
    inside = step([3, 31, 7], [3, 31, 7])
    _check_rows(clamped, list(inside), 'clamped position')


def test_generate_batch_matches_single_sequence_generate():
    """Ragged prompts: prefill_batch writes the same cache rows as token-by-token steps, and generate_batch gives every prompt what
    batch-1 generate gives it (greedy picks may flip on near-ties, as in test_gpu_engine.test_prefill_then_decode_matches_token_by_token)."""
    from gptq_b200 import engine
    dec = engine.synthetic_llama('tiny256', bits=4, groupsize=64, vocab=300, seed=7, max_seq=64, batch=4)
    dec1 = _single_twin(dec)
    gen = torch.Generator().manual_seed(3)
    prompts = [torch.randint(0, 300, (n, ), generator=gen).tolist() for n in (1, 5, 17, 40)]
    assert dec.prefill_batch(prompts) == [0, 4, 16, 39]
    for b, pr in enumerate(prompts):
        n = len(pr) - 1
        if n == 0:
            continue
        dec1.reset()
        for pos, tok in enumerate(pr[:n]):
            dec1.set_input(tok, pos)
            dec1.step()
        torch.cuda.synchronize()
        assert_rel_close(dec.k_cache[:, b, :, :n], dec1.k_cache[:, 0, :, :n], rel=1e-2, what=f'prefilled K rows of prompt {b}')
        assert_rel_close(dec.v_cache[:, b, :, :n], dec1.v_cache[:, 0, :, :n], rel=1e-2, what=f'prefilled V rows of prompt {b}')
    outs = dec.generate_batch(prompts, 10)
    for pr, out in zip(prompts, outs):
        ref = dec1.generate(pr, 10)
        assert len(out) == len(pr) + 10 and out[:len(pr)] == pr
        assert sum(x != y for x, y in zip(out, ref)) <= 2
    with pytest.raises(ValueError):
        dec.generate_batch(prompts[:3], 4)  # one prompt per sequence
    with pytest.raises(ValueError):
        dec.generate_batch(prompts, 26)  # 40 + 26 > max_seq + 1
    with pytest.raises(ValueError):
        dec.generate_batch([[1], [2], [3], [4, 300]], 2)
    with pytest.raises(ValueError):
        dec.set_input([1, 2, 3, 4], [0, 1, 64, 2])


def test_fallback_boundary_13b():
    """The plan needs one attention team per (sequence, head) pair: 13B (40 heads) fits floor(2 * SMs / 40) sequences (6 on 132 SMs).
    One sequence more takes the kernel chain, whose rows still match the batch-1 persistent steps."""
    from gptq_b200 import engine
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    b_in = min(8, 2 * sms // 40)
    assert b_in < 8
    positions = [0, 100, 200, 255, 256, 300, 400, 511]
    dec1 = None
    for B in (b_in, b_in + 1):
        dec = engine.synthetic_llama('13b', bits=4, groupsize=128, vocab=4096, seed=31, max_seq=512, n_layers=2, batch=B)
        assert (dec.launches_per_step() == 1) == (B == b_in), f'batch {B}: {dec.launches_per_step()} launches'
        dec1 = dec1 or _single_twin(dec)
        gen = torch.Generator(device=dec.dev).manual_seed(32)
        dec.k_cache.normal_(0, 0.5, generator=gen)
        dec.v_cache.normal_(0, 0.5, generator=gen)
        toks = [(11 * b + 1) % 4096 for b in range(B)]
        singles = _singles(dec1, dec, toks, positions[:B])
        dec.set_input(toks, positions[:B])
        dec.step()
        torch.cuda.synchronize()
        _check_rows(dec.logits, singles, f'13b batch {B}')
        del dec


@pytest.mark.parametrize('size', ['65b', '33b'])
def test_fallback_boundary_large(size):
    """The same boundary at 65B (64 heads: 4 sequences persistent on 132 SMs, 5 on the kernel chain) and 33B (52 heads: 5, then 6), on one
    layer: the chain and the batch-1 persistent step differ in fp32 summation order, and behind a second layer that difference re-rolled to
    3.0e-3 of the rms at 33B in one of two runs, the spread bound itself."""
    from gptq_b200 import engine
    nh = engine.LLAMA_SHAPES[size][3]
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    b_in = min(8, 2 * sms // nh)
    assert b_in < 8
    positions = [0, 100, 200, 255, 256, 300, 400, 511]
    dec1 = None
    for B in (b_in, b_in + 1):
        dec = engine.synthetic_llama(size, bits=4, groupsize=128, vocab=4096, seed=33, max_seq=512, n_layers=1, batch=B)
        assert (dec.launches_per_step() == 1) == (B == b_in), f'{size} batch {B}: {dec.launches_per_step()} launches'
        dec1 = dec1 or _single_twin(dec)
        gen = torch.Generator(device=dec.dev).manual_seed(34)
        dec.k_cache.normal_(0, 0.5, generator=gen)
        dec.v_cache.normal_(0, 0.5, generator=gen)
        toks = [(11 * b + 1) % 4096 for b in range(B)]
        singles = _singles(dec1, dec, toks, positions[:B])
        dec.set_input(toks, positions[:B])
        dec.step()
        torch.cuda.synchronize()
        _check_rows(dec.logits, singles, f'{size} batch {B}')
        del dec
