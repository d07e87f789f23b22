"""GPU: decode attention of both engines against a float64 softmax, element by element, on the probe model of attn_probe.py (exact q, k,
v, identity o_proj, zero MLP: the residual after a step is fp16(x_in + fp16(att))).

* Bit-exact anchors (torch.equal): at pos 0 the softmax over one key is 1, so x_out == fp16(x_in + v_new); with every planted key equal to
  the new one and V rows (multiples of 2^-4, 0.5 <= |v| <= 2) that sum to 0 with v_new, every weight is exactly 1 and x_out == x_in at any
  position, split and team partition.  A key dropped, counted twice, read from the wrong head or sequence, or left unpatched moves the output
  by V_t / T >= 2^-12: four ulps of x_in = +-2^-4.
* Bounded profiles (attn_probe.PROFILES): x_out against x_in + att of a float64 softmax over the kernel's own q_rot, K and V rows, per
  element within attn_probe.x_bound.  Heavy keys are put at 0, at the last planted key, on both sides of every unit and split edge and at
  both ends of every team range; at the longest 7B context the heavy sets rotate until every key has been heavy in some head.
* The appended K row of every step against fp64 RoPE (attn_probe.check_rope_row) and bit for bit against the prefill's rotation of the
  same exact k (attn_probe.prefill_row).
* The cache rows at and after each position hold NaN before the step: the kernel must write the new row and never read a later one.  After
  the step the planted rows are bitwise unchanged and the later rows still NaN: exactly row pos of every K/V head was written.
* Grouped-query shapes (tiny-gqa*, LLaMA-3-8B, LLaMA-2-70B, CodeLlama-34B, and one K/V head at 7B and tiny): the query heads of a group
  have disjoint q supports, so each scores only the part of the shared K rows planted for it; a key read from another group, dropped at a
  team edge or left unpatched in one team's stage moves that head's output as in the multi-head case.

The worst |err| / bound of every sweep is printed (pytest -s)."""
import numpy as np
import pytest
import torch

import attn_probe as P
from attn_probe import run_sweeps
from gpu_util import check_fp64_bound

pytestmark = pytest.mark.gpu


def label(probe, size):
    """The shape's name in the printed sweeps, with its query and K/V head counts when they differ."""
    return size if probe.nkv == probe.nh else f'{size} ({probe.nh} / {probe.nkv} K/V heads)'


# ----------------------------------------------------------------------------- batch 1, every position of a 600-key cache
def every_position(probe, name, seed):
    """Every position 0..599 at batch 1: heavy keys at every position (rotating over the edges), one more profile in turn."""
    gen = torch.Generator(device='cuda:0').manual_seed(seed)
    worst = {k: P.Worst(f'{name} {k}') for k in P.PROFILES}
    rope = P.Worst(f'{name} appended K row vs fp64 RoPE')
    for i in range(600):
        P.sweep(probe, [[i]], ('heavy', P.PROFILES[1 + i % 6]), gen, worst, rope, toks=lambda j, b: i + 7 * j + 3 * b, rotate_heavy=True)
    for w in list(worst.values()) + [rope]:
        w.done()


def test_chain_tiny_every_position():
    """Kernel chain (tiny: intermediate 704 keeps it off the persistent path): 256-key splits and the combine, every position 0..599."""
    probe = P.Probe('tiny', max_seq=600)
    assert not probe.persistent and probe.dec.launches_per_step() > 1
    every_position(probe, 'chain tiny', 7)


def test_chain_tiny_gqa1_every_position():
    """The kernel chain with one K/V head for 4 query heads (tiny-gqa1-chain): the 4 CTAs of every 256-key split read the same K/V head and
    the first of them stores the new row, every position 0..599."""
    probe = P.Probe('tiny-gqa1-chain', max_seq=600)
    assert not probe.persistent and probe.dec.launches_per_step() > 1 and probe.nkv == 1
    every_position(probe, f'chain {label(probe, "tiny-gqa1-chain")}', 17)


def test_persistent_tiny256_every_position():
    """Persistent kernel at tiny256 (2 heads, 132 teams per head on 132 SMs): the general record merge, every position 0..599."""
    probe = P.Probe('tiny256', max_seq=600)
    assert probe.persistent
    assert probe.nb // probe.nh + 1 > 12, 'the fast merge would serve this shape'
    every_position(probe, 'persistent tiny256', 8)


def test_persistent_tiny_gqa2_every_position():
    """Persistent kernel at tiny-gqa2 (4 query heads on 2 K/V heads, 66 teams per query head): the general record merge over teams that
    share a K/V head, every team owning the new key's unit patching its own stage, every position 0..599."""
    probe = P.Probe('tiny-gqa2', max_seq=600)
    assert probe.persistent and probe.nkv == 2
    assert probe.nb // probe.nh + 1 > 12, 'the fast merge would serve this shape'
    every_position(probe, f'persistent {label(probe, "tiny-gqa2")}', 18)


# ----------------------------------------------------------------------------- batch 1 at the 7B and 13B shapes
POS_7B = [0, 1, 31, 32, 33, 255, 256, 257, 511, 512, 1023, 1024, 2015, 2016, 2046, 2047]
LLAMA2_EDGES = [0, 1, 31, 32, 33, 255, 256, 257, 1023, 1024, 2047, 2048, 2049, 4063, 4064, 4094, 4095]  # max_seq 4096


def test_persistent_7b_positions():
    """LLaMA-7B shapes (32 heads, 8 or 9 teams per head: the fast merge), at unit, split and team edges; at 2047 every key is heavy once."""
    probe = P.Probe('7b', max_seq=2048)
    assert probe.persistent
    assert probe.nb // probe.nh + 1 <= 12, 'the general merge would serve this shape'
    positions = sorted(set(POS_7B) | set(P.team_edge_positions(probe.nh, probe.nb)))
    run_sweeps(probe, '7b', [[p] for p in positions], full_rotation=(2047, ))


def test_persistent_7b_llama2_context():
    """LLaMA-2-7B context (max_seq 4096): the unit, split and team edges, both sides of 2048 and the last position 4095."""
    probe = P.Probe('7b', max_seq=4096)
    assert probe.persistent
    positions = sorted(set(LLAMA2_EDGES) | set(P.team_edge_positions(probe.nh, probe.nb)))
    run_sweeps(probe, '7b max_seq 4096', [[p] for p in positions])


def test_persistent_7b_codellama_context():
    """CodeLlama-7B context (max_seq 16384, RoPE base 1e6): the team edges, both sides of 8192 and the last position 16383, where the 512
    units of a head are split over 8 or 9 teams and every key is heavy once; the appended K row against fp64 RoPE at base 1e6."""
    probe = P.Probe('7b', max_seq=16384, rope_base=1e6)
    assert probe.persistent
    positions = sorted({0, 1, 8191, 8192, 16383} | set(P.team_edge_positions(probe.nh, probe.nb)))
    run_sweeps(probe, '7b max_seq 16384 base 1e6', [[p] for p in positions], full_rotation=(16383, ))


def test_persistent_7b_last_unit_past_the_slot():
    """max_seq 2000: the last 32-key unit of a head at pos 1999 reaches past the end of the head's slot (only 16 rows are fetched)."""
    probe = P.Probe('7b', max_seq=2000)
    assert probe.persistent
    run_sweeps(probe, '7b max_seq 2000', [[1999], [1998], [1984]])


def test_persistent_llama3_8b_positions():
    """LLaMA-3-8B (32 query heads on 8 K/V heads, RoPE base 5e5; 8 or 9 teams per query head: the fast merge): the edges of
    test_persistent_7b_positions, each K/V head streamed by the teams of its 4 query heads; at 2047 every key is heavy once."""
    probe = P.Probe('llama3-8b', max_seq=2048, rope_base=5e5)
    assert probe.persistent and probe.nkv == 8
    assert probe.nb // probe.nh + 1 <= 12, 'the general merge would serve this shape'
    positions = sorted(set(POS_7B) | set(P.team_edge_positions(probe.nh, probe.nb)))
    run_sweeps(probe, f'{label(probe, "llama3-8b")} base 5e5', [[p] for p in positions], full_rotation=(2047, ))


def test_persistent_llama3_8b_last_unit_past_the_slot():
    """LLaMA-3-8B at max_seq 2000: the last 32-key unit at pos 1999 reaches past the end of its K/V head's slot (16 rows are fetched), next to
    the rows of the following K/V head, which must not enter the softmax."""
    probe = P.Probe('llama3-8b', max_seq=2000, rope_base=5e5)
    assert probe.persistent and probe.nkv == 8
    run_sweeps(probe, f'{label(probe, "llama3-8b")} max_seq 2000', [[1999], [1998], [1984]])


def test_persistent_13b_act_order():
    """LLaMA-13B shapes with act-order layers: the qkv input gather (qkv_perm) and o_perm, whose staging takes the general merge path."""
    probe = P.Probe('13b', max_seq=2048, act_order=True)
    assert probe.persistent
    assert probe.dec.perms[0]['qkv'] is not None and probe.dec.perms[0]['o'] is not None
    run_sweeps(probe, '13b act-order', [[0], [1], [32], [257], [1023], [2047]])


def test_persistent_70b_act_order():
    """LLaMA-2-70B shapes with act-order layers: the qkv input gather (qkv_perm) at the grouped-query width (64 + 2 x 8 heads of 128)."""
    probe = P.Probe('70b', max_seq=2048, act_order=True)
    assert probe.persistent and probe.nkv == 8
    assert probe.dec.perms[0]['qkv'] is not None and probe.dec.perms[0]['o'] is not None
    run_sweeps(probe, f'{label(probe, "70b")} act-order', [[0], [1], [32], [257], [1023], [2047]])


# ----------------------------------------------------------------------------- batches
@pytest.mark.parametrize('batch,position_sets,max_seq', [
    pytest.param(2, [[2047, 1], [0, 0], [300, 2000]], 2048, id='2-position_sets0'),
    pytest.param(3, [[2047, 3, 500], [0, 0, 0], [31, 32, 33]], 2048, id='3-position_sets1'),
    pytest.param(8, [[0, 31, 32, 255, 256, 1023, 2046, 2047], [0] * 8, [2047, 0, 0, 0, 0, 0, 0, 5]], 2048, id='8-position_sets2'),
    pytest.param(8, [[4095, 0, 2047, 2048, 31, 32, 1024, 4094], [0] * 8, [4095, 0, 0, 0, 0, 0, 0, 2048]], 4096, id='8-max_seq4096'),
])
def test_persistent_7b_batched(batch, position_sets, max_seq):
    """Batched persistent kernel at 7B: ragged positions (seq_teams gives each sequence a share of the teams in proportion to its
    context), one long and one short sequence, everything at pos 0; stage_range_batch merges the records.  Also at the LLaMA-2 context."""
    probe = P.Probe('7b', batch=batch, max_seq=max_seq)
    assert probe.persistent
    run_sweeps(probe, f'7b batch {batch} max_seq {max_seq}', position_sets)


TINY_BATCHES = [(2, [[599, 0], [300, 301], [37, 599], [0, 0]]), (3, [[599, 1, 256], [0, 0, 0]])]


@pytest.mark.parametrize('size,batch,position_sets', [pytest.param('tiny256', *TINY_BATCHES[0], id='2-position_sets0'),
                                                      pytest.param('tiny256', *TINY_BATCHES[1], id='3-position_sets1'),
                                                      pytest.param('tiny-gqa2', *TINY_BATCHES[0], id='tiny-gqa2-2'),
                                                      pytest.param('tiny-gqa2', *TINY_BATCHES[1], id='tiny-gqa2-3')])
def test_persistent_tiny256_batched(size, batch, position_sets):
    """tiny256 batches, and the same at tiny-gqa2 (4 query heads on 2 K/V heads): tens of teams per (sequence, head), so merge_records takes
    several rounds of 12 records (the w0 rescale)."""
    probe = P.Probe(size, batch=batch, max_seq=600)
    assert probe.persistent
    assert max(P.seq_teams(position_sets[0], probe.nh, probe.nb, s)[1] for s in range(batch)) // probe.nh > 12
    run_sweeps(probe, f'{label(probe, size)} batch {batch}', position_sets)


def test_persistent_13b_batch6():
    probe = P.Probe('13b', batch=6, max_seq=2048)
    assert probe.persistent
    run_sweeps(probe, '13b batch 6', [[0, 255, 256, 1023, 1500, 2047], [5, 4, 3, 2, 1, 0]])


def test_chain_13b_batch7():
    """One sequence beyond the 13B plan: the kernel chain serves the batch."""
    probe = P.Probe('13b', batch=7, max_seq=1024)
    assert not probe.persistent and probe.dec.launches_per_step() > 1
    run_sweeps(probe, 'chain 13b batch 7', [[0, 1, 255, 256, 511, 800, 1023], [1023, 0, 1, 2, 3, 4, 256]])


def test_chain_13b_batch7_llama2_context():
    """The kernel chain at LLaMA-2-13B's context (max_seq 4096: 16 splits of 256 keys per head)."""
    probe = P.Probe('13b', batch=7, max_seq=4096)
    assert not probe.persistent and probe.dec.launches_per_step() > 1
    run_sweeps(probe, 'chain 13b batch 7 max_seq 4096', [[4095, 0, 1, 2047, 2048, 3839, 3840], [0, 4095, 256, 4094, 1, 2, 3]])


def test_chain_tiny_codellama_context():
    """The kernel chain at CodeLlama's context and RoPE base (max_seq 16384, base 1e6): 64 splits, so the combine reads 64 partials."""
    probe = P.Probe('tiny', max_seq=16384, rope_base=1e6)
    assert not probe.persistent and probe.dec.launches_per_step() > 1
    run_sweeps(probe, 'chain tiny max_seq 16384 base 1e6', [[p] for p in (0, 1, 255, 256, 4095, 8191, 8192, 16127, 16128, 16382, 16383)],
               full_rotation=(16383, ))


# ----------------------------------------------------------------------------- the 65B and 33B shapes
def max_persistent_batch(size):
    """The largest batch the persistent plan takes at `size`: one attention team per (sequence, head) pair, 2 teams per SM, at most 8."""
    from gptq_b200 import engine
    nh = engine.LLAMA_SHAPES[size][3]
    return min(8, 2 * torch.cuda.get_device_properties(0).multi_processor_count // nh)


LARGE_CONTEXTS = {  # max_seq, RoPE base, positions (besides the team edges), the position at which every key is heavy once
    '65b': (2048, 10000.0, POS_7B, 2047),
    '33b': (2048, 10000.0, POS_7B, None),
    '70b': (4096, 10000.0, LLAMA2_EDGES, 4095),
    '34b': (16384, 1e6, [0, 1, 8191, 8192, 16383], 16383),
}


@pytest.mark.parametrize('size', ['65b', '33b', '70b', '34b'])
def test_persistent_large_positions(size):
    """LLaMA-65B (64 heads, 4 or 5 teams per head on 132 SMs) and LLaMA-33B (52 heads, 5 or 6) at batch 1: the unit, split and team edges
    of POS_7B and of this shape's team partition; at 65B every key of the 2047-key context is heavy once.  LLaMA-2-70B (64 query heads on 8
    K/V heads) at its 4096 context and CodeLlama-34B (the same heads, RoPE base 1e6) at 16384: the 8 query heads of a group read one K/V
    head through 4 or 5 teams each; every key of the longest context is heavy once."""
    max_seq, base, edges, rotation = LARGE_CONTEXTS[size]
    probe = P.Probe(size, max_seq=max_seq, rope_base=base)
    assert probe.persistent and probe.dec.launches_per_step() == 1
    assert probe.nb // probe.nh + 1 <= 12, 'the general merge would serve this shape'
    positions = sorted(set(edges) | set(P.team_edge_positions(probe.nh, probe.nb)))
    name = label(probe, size) if max_seq == 2048 else f'{label(probe, size)} max_seq {max_seq} base {base:g}'
    run_sweeps(probe, name, [[p] for p in positions], full_rotation=(rotation, ) if rotation else ())


def _ragged(B):
    return [[2047, 0, 255, 256, 1023, 31, 32, 1500][:B], [0] * B]


@pytest.mark.parametrize('size', ['65b', '33b', '70b', 'llama3-8b'])
def test_persistent_large_largest_batch(size):
    """The largest batch the persistent plan takes at 65B / 33B / 70B / LLaMA-3-8B (4 / 5 / 4 / 8 sequences on 132 SMs): every team serves one
    (sequence, query head) pair or a share of one (256 of the 264 teams at LLaMA-3-8B); ragged positions and every sequence at position 0."""
    B = max_persistent_batch(size)
    probe = P.Probe(size, batch=B, max_seq=2048)
    assert probe.persistent and probe.dec.launches_per_step() == 1, f'{size} batch {B}'
    run_sweeps(probe, f'{label(probe, size)} batch {B}', _ragged(B))


@pytest.mark.parametrize('size', ['65b', '33b', '70b'])
def test_chain_large_above_the_plan(size):
    """One sequence more than the persistent plan takes at 65B / 33B / 70B: the kernel chain serves the batch."""
    B = max_persistent_batch(size) + 1
    assert B <= 8
    probe = P.Probe(size, batch=B, max_seq=1024)
    assert not probe.persistent and probe.dec.launches_per_step() > 1, f'{size} batch {B}'
    run_sweeps(probe, f'chain {label(probe, size)} batch {B}', [[1023, 0, 1, 255, 256, 511, 800, 31][:B], [0] * B])


def test_chain_70b_batch8_llama2_context():
    """LLaMA-2-70B at batch 8 on the kernel chain, the engine that serves it (8 x 64 (sequence, query head) pairs exceed the persistent
    kernel's teams), at its 4096 context: 16 splits of 256 keys per query head, the 8 query heads of a group on one K/V head."""
    probe = P.Probe('70b', batch=8, max_seq=4096)
    assert not probe.persistent and probe.dec.launches_per_step() > 1 and probe.nkv == 8
    run_sweeps(probe, f'chain {label(probe, "70b")} batch 8 max_seq 4096', [[4095, 0, 1, 2047, 2048, 3839, 3840, 255], [0] * 8])


@pytest.mark.parametrize('size,batch', [('7b', 1), ('7b', 8), ('tiny', 1), ('tiny', 8)])
def test_one_kv_head(size, batch):
    """One K/V head for every query head: at 7B (g = 32, each q on 2 of the 64 pairs) every team of the persistent kernel streams the same
    K/V head; tiny (g = 2) runs on the kernel chain."""
    probe = P.Probe(size, batch=batch, max_seq=2048, n_kv_heads=1)
    assert probe.persistent == (size == '7b') and (probe.dec.launches_per_step() == 1) == probe.persistent
    sets = [[p] for p in (0, 1, 31, 32, 255, 256, 1024, 2016, 2047)] if batch == 1 else [[0, 31, 32, 255, 256, 1023, 2046, 2047], [0] * 8]
    run_sweeps(probe, f'{"persistent" if probe.persistent else "chain"} {label(probe, size)} batch {batch}', sets)


# ----------------------------------------------------------------------------- lm_head and greedy token
@pytest.mark.parametrize('size,batch,vocab,dups,persistent', [
    ('7b', 1, 32001, [1001, 1002, 32000], True),
    ('7b', 8, 32001, [1001, 1002, 32000], True),
    ('tiny', 1, 600, [7, 8, 599], False),
    ('tiny', 3, 600, [7, 8, 599], False),
    ('llama3-8b', 1, 128256, [1001, 1002, 128255], True),
    ('llama3-8b', 8, 128256, [1001, 1002, 128255], True),
])
def test_lm_head_and_greedy_token(size, batch, vocab, dups, persistent):
    lm_head_and_greedy_token(size, batch, vocab, dups, persistent)


@pytest.mark.parametrize('size,batch,persistent', [('65b', 1, True), ('65b', 'max', True), ('65b', 'max+1', False), ('33b', 1, True),
                                                   ('33b', 'max', True)])
def test_lm_head_and_greedy_token_large(size, batch, persistent):
    """The same at 65B (one 16384-byte lm_head row fills a stage: every row is a stage of its own) and 33B (13312-byte rows), at batch 1,
    the largest persistent batch and, at 65B, one sequence more (the kernel chain); vocab 32001."""
    if batch != 1:
        batch = max_persistent_batch(size) + (batch == 'max+1')
    lm_head_and_greedy_token(size, batch, 32001, [1001, 1002, 32000], persistent)


def lm_head_and_greedy_token(size, batch, vocab, dups, persistent):
    """A pos-0 step, where the head's input x = fp16(x_in + v_new) is known exactly (and its sum of squares is exact, so the final RMSNorm is
    reproduced bit for bit in float32): the logits within check_fp64_bound, and duplicate maximal rows on both sides of an lm_head stage
    boundary (the persistent kernel stages 2 rows at 7B; vocab 32001 leaves row 32000 alone in a partial last stage) give bitwise equal
    logits -- each row goes through the same per-row arithmetic -- and next_tokens is the lowest index of the maximum."""
    from gptq_b200 import engine
    H = engine.LLAMA_SHAPES[size][0]
    lm =(torch.randn(vocab, H, generator=torch.Generator().manual_seed(5)) * 0.02).half()
    lm[dups] = 2.0**-6
    probe = P.Probe(size, batch=batch, max_seq=64, vocab=vocab, lm_head=lm)
    assert probe.persistent == persistent and (probe.dec.launches_per_step() == 1) == persistent
    toks = [(977 * b + 5) % vocab for b in range(batch)]
    positions = [0] * batch
    probe.learn(toks, positions)
    empty = torch.zeros(probe.nkv, 0, P.HD, dtype=torch.float16, device='cuda:0')
    x_in, x_out = probe.run(toks, positions, [(empty, empty)] * batch)
    want = (x_in.double() + torch.stack([v.repeat_interleave(probe.g, 0).reshape(-1) for v in probe.v_new]).double()).half()
    assert torch.equal(x_out, want)
    f = np.float32
    x = x_out.float().cpu().numpy()
    ss = (x.astype(np.float64)**2).sum(1)
    assert np.array_equal(ss.astype(f).astype(np.float64), ss), 'sum of squares not exact in fp32'
    rstd = f(1) / np.sqrt(ss.astype(f) / f(H))
    xn = torch.from_numpy(((x * rstd[:, None]).astype(f) * f(1)).astype(np.float16))
    logits = probe.dec.logits
    check_fp64_bound(logits, xn, lm.t().contiguous(), what=f'{size} batch {batch} logits')
    for b in range(batch):
        row = logits[b]
        assert torch.equal(row[dups], row[dups[:1]].expand(len(dups))), f'seq {b}: duplicate rows {dups} give {row[dups].tolist()}'
        assert row[dups[0]] == row.max() and int((row == row.max()).sum()) == len(dups)
        assert int(probe.dec.next_tokens[b]) == dups[0], f'seq {b}: next token {int(probe.dec.next_tokens[b])}, lowest maximum {dups[0]}'
