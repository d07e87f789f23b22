"""GPU: the persistent decode kernel hands attention to o_proj through epoch-tagged records instead of a grid barrier.

Each team's partial record (m, l, o[128]) is 130 64-bit words: the float's bits in the low half, the epoch of the (launch, layer) that
wrote it in the high half; o_proj's staging uses a word once it carries the current epoch.  These tests read the records and the
grid-barrier counter (u64 [0] arrivals, [1] the value at the end of the last step) in the kernel's scratch region, which starts at
gptq_llama_persistent_scratch_offset(); _mega_layout follows mega_scratch in csrc/decode_mega.cu and checks itself against the scratch size."""
import pytest
import torch

from llama_oracle import LlamaOracle, check_steps

pytestmark = pytest.mark.gpu

MAX_TEAMS, REC_WORDS, REGION_BYTES, TEAMS_PER_CTA = 512, 130, 528 * 1024, 2
# two runs of one step differ only in the fp32 summation order of the split-K partial sums (test_gpu_batch_decode.py)
SPREAD_MAX = 1.5e-2


def _align256(n):
    return (n + 255) // 256 * 256


def _mega_layout(dec):
    """byte offsets in dec.scratch of the records and of the barrier counter: the buffers of mega_scratch (csrc/decode_mega.cu), in its
    order, each padded to 256 bytes, from the region's exported start; the region is the last one of the scratch"""
    H, I, B, MAX_TP = dec.embed.shape[1], dec.intermediate, dec.batch, 8
    sizes = [('resid0', B * H * 2), ('resid1', B * H * 2), ('acc_o', B * H * 4), ('acc_d', B * H * 4), ('xbar', (MAX_TP + 1) * 256),
             ('acc_o_loc', H * 4), ('acc_d_loc', H * 4), ('acc_qkv', B * 3 * H * 4), ('acc_g', B * I * 4), ('acc_u', B * I * 4),
             ('part', REGION_BYTES), ('rope_cs', B * 128 * 4), ('bar', 256)]
    off, at = {}, dec.mega_scratch_offset()
    for name, n in sizes:
        off[name] = at
        at += _align256(n)
    assert at == dec.scratch.numel(), f'the scratch layout no longer matches mega_scratch: region ends at {at}, scratch is {dec.scratch.numel()} B'
    return off


def _counter(dec):
    """the grid-barrier counter: (arrivals, value at the end of the last step)"""
    at = _mega_layout(dec)['bar']
    c = dec.scratch[at:at + 16].view(torch.int64)
    return int(c[0]), int(c[1])


def _records(dec):
    """the record region as int64 [MAX_TEAMS, REC_WORDS] (a view into the scratch)"""
    at = _mega_layout(dec)['part']
    return dec.scratch[at:at + MAX_TEAMS * REC_WORDS * 8].view(torch.int64).view(MAX_TEAMS, REC_WORDS)


def _epoch(base, layer):
    """record_epoch in csrc/decode_mega.cu"""
    return (base + layer) % 0xffffffff + 1


def _grid():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _decoder(size, bits, act, batch, seed=7):
    from gptq_b200 import engine
    dec = engine.synthetic_llama(size, bits=bits, groupsize=128, act_order=act, vocab=4096, seed=seed, max_seq=2048, n_layers=2, batch=batch,
                                 use_graph=False)
    assert dec.launches_per_step() == 1
    gen = torch.Generator(device=dec.dev).manual_seed(seed + 1)
    for c in (dec.k_cache, dec.v_cache):
        c.copy_(torch.randn(c.shape, generator=gen, device=dec.dev) * 0.5)
    return dec


def _step(dec, positions):
    dec.set_input([1 + 7 * b for b in range(dec.batch)], positions)
    dec.step()
    torch.cuda.synchronize()


CASES = [('7b', 4, False, 1), ('7b', 4, False, 8), ('13b', 3, True, 1)]


@pytest.mark.parametrize('size,bits,act,batch', CASES)
def test_four_grid_barriers_per_layer(size, bits, act, batch):
    """One step passes 4 grid barriers per layer plus the lm_head's (Q->A, O->G, G->D, D->next), and leaves every team's record tagged with
    the last layer's epoch."""
    dec = _decoder(size, bits, act, batch)
    grid, n_layers = _grid(), len(dec.layers)
    for positions in ([100 + 250 * b for b in range(batch)], [1500 - 150 * b for b in range(batch)]):
        before, rest = _counter(dec)
        assert before == rest
        _step(dec, positions)
        after, rest = _counter(dec)
        assert after - before == grid * (4 * n_layers + 1), (after - before, grid, n_layers)
        assert rest == after
        tags = (_records(dec)[:grid * TEAMS_PER_CTA] >> 32) & 0xffffffff
        assert bool((tags == _epoch(before, n_layers - 1)).all())


@pytest.mark.parametrize('size,bits,act,batch', CASES)
def test_stale_records_are_not_read(size, bits, act, batch):
    """Between two steps at different positions, every record word is replaced by NaN tagged with one of the previous step's epochs (as if
    the writers of the next step had not stored yet): the next step must wait for the fresh words and compute what an untouched twin does."""
    poisoned, twin = _decoder(size, bits, act, batch), _decoder(size, bits, act, batch)
    n_layers = len(poisoned.layers)
    p0 = [40 + 5 * b for b in range(batch)]
    p1 = [1800 - 100 * b for b in range(batch)]
    base, _ = _counter(poisoned)
    for dec in (poisoned, twin):
        _step(dec, p0)
    stale = torch.tensor([_epoch(base, l) for l in range(n_layers)], dtype=torch.int64, device=poisoned.dev)
    pick = torch.randint(0, n_layers, (MAX_TEAMS, REC_WORDS), generator=torch.Generator(device=poisoned.dev).manual_seed(3), device=poisoned.dev)
    nan_bits = torch.tensor([float('nan')], dtype=torch.float32).view(torch.int32).item() & 0xffffffff
    _records(poisoned).copy_((stale[pick] << 32) | nan_bits)
    for dec in (poisoned, twin):
        _step(dec, p1)
    for b in range(batch):
        out, ref = poisoned.logits[b].float(), twin.logits[b].float()
        assert bool(torch.isfinite(out).all()), f'sequence {b}: a stale record was used'
        rms = ref.pow(2).mean().sqrt().item()
        assert (out - ref).abs().max().item() <= SPREAD_MAX * rms, f'sequence {b}'


def test_fresh_engine_first_step_matches_oracle():
    """A fresh engine's scratch is zeroed (every word tagged 0, which no epoch uses): its first step is right."""
    from gptq_b200 import engine
    dec = engine.synthetic_llama('tiny256', bits=4, groupsize=64, vocab=512, seed=5, max_seq=64, use_graph=False)
    assert dec.launches_per_step() == 1 and _counter(dec) == (0, 0)
    toks = [3, 9, 27]
    check_steps(dec, LlamaOracle.from_decoder(dec, eps=1e-6, base=10000.0), [toks], lambda k, b, pos: f'pos {pos}')
