"""GPU: gptq_sample_tokens token for token against the numpy restatement (oracle/sampling.py) over a grid of vocabulary sizes, temperatures,
top-k, top-p, seeds, positions and crafted rows; greedy equivalence with the decode step; determinism and independence of the batch slot;
the distribution of 2^16 draws; the engine's sampled generate / generate_batch on both decode engines and int3 act-order; eos stopping."""
import numpy as np
import pytest
import torch

from oracle import sampling as S

pytestmark = pytest.mark.gpu

VOCABS = [1, 2, 33, 32000, 32001, 131072]
GRID = [(t, k, p) for t in (0.0, 0.1, 0.8, 1.0, 2.5) for k in ('0', '1', '50', 'V') for p in (0.05, 0.95, 1.0)]
KINDS = ['random', 'equal', 'outlier', 'ties at k', 'top-p boundary', '+inf', '-inf and NaN', 'all -inf']


def _row(kind, V, rng):
    if kind == 'random':
        return (rng.standard_normal(V) * 3).astype(np.float16)
    if kind == 'equal':
        return np.full(V, 0.75, dtype=np.float16)
    if kind == 'outlier':
        r = (rng.standard_normal(V) * 0.1).astype(np.float16)
        r[rng.integers(V)] = 8
        return r
    if kind == 'ties at k':
        r = (rng.standard_normal(V) * 2).astype(np.float16)
        order = np.argsort(-r.astype(np.float32), kind='stable')
        r[order[max(0, min(V, 50) - 8):min(V, 58)]] = r[order[min(V, 50) - 1]]
        return r
    if kind == 'top-p boundary':
        r = np.full(V, -9, dtype=np.float16)
        lv = np.array([4, 3, 3, 2, 2, 2, 2, 1, 1, 0, 0, 0], dtype=np.float16)[:V]
        r[rng.permutation(V)[:lv.size]] = lv
        return r
    if kind == '+inf':
        r = (rng.standard_normal(V) * 3).astype(np.float16)
        r[rng.integers(V, size=min(V, 3))] = np.inf
        return r
    if kind == '-inf and NaN':
        r = (rng.standard_normal(V) * 3).astype(np.float16)
        idx = rng.permutation(V)
        r[idx[:V // 3]] = -np.inf
        r[idx[V // 3:V // 2]] = np.nan
        return r
    r = np.full(V, -np.inf, dtype=np.float16)
    r[rng.integers(V)] = np.nan
    return r


def _launch(rows, positions, temps, ks, ps, seeds, eos, min_len):
    from gptq_b200 import ops
    d = lambda v, dt: torch.tensor(v, dtype=dt, device='cuda')
    logits = torch.from_numpy(np.stack(rows)).cuda()
    seeds64 = [s - 2**64 if s >= 2**63 else s for s in seeds]
    out = ops.sample_tokens(logits, d(positions, torch.int32), d(temps, torch.float32), d(ks, torch.int32), d(ps, torch.float32), d(seeds64, torch.int64),
                            d(eos, torch.int32), d(min_len, torch.int32))
    return out.tolist()


@pytest.mark.parametrize('V', VOCABS)
def test_tokens_match_the_restatement(V):
    """Every grid point (T, top_k, top_p) in one launch of B in {1, 3, 8} rows, each row a crafted kind with its own seed, position and eos
    state.  The only allowed difference: u * W within 2^-40 W of a cumulative boundary, where the token must be a neighbour (expected: none)."""
    rng = np.random.default_rng(V)
    near, checked = 0, 0
    for gi, (T, kname, p) in enumerate(GRID):
        B = (1, 3, 8)[gi % 3]
        k = {'0': 0, '1': 1, '50': 50, 'V': V}[kname]
        rows, pos, seeds, eos, ml = [], [], [], [], []
        for b in range(B):
            kind = KINDS[(gi * 3 + b) % len(KINDS)]
            rows.append(_row(kind, V, rng))
            pos.append(int(rng.integers(0, 1 << 20)))
            seeds.append(int(rng.integers(0, 2**63)) * 2 + int(rng.integers(2)))
            top = int(np.argmax(np.nan_to_num(rows[-1].astype(np.float32), nan=-np.inf)))
            eos.append(top if b % 2 == 0 else -1)
            ml.append(pos[-1] + 1 + (b % 4 == 0))  # suppressed on rows 0, 4; eos active but allowed on rows 2, 6
        got = _launch(rows, pos, [T] * B, [k] * B, [p] * B, seeds, eos, ml)
        for b in range(B):
            want, info = S.sample_row(rows[b], T, k, p, seeds[b], eos[b], ml[b], pos[b], details=True)
            checked += 1
            if got[b] == want:
                continue
            ok = info is not None and S.near_boundary(info, want, got[b])
            assert ok, f'V={V} T={T} top_k={k} top_p={p} row {b} ({KINDS[(gi * 3 + b) % len(KINDS)]}): kernel {got[b]}, restatement {want}'
            near += 1
    print(f'  V={V}: {checked} rows, {near} draws within 2^-40 W of a boundary')


def test_greedy_equals_the_decode_step():
    """T = 0 gives the decode step's next_tokens bit for bit, on both engines, at batch 1 and 3."""
    from gptq_b200 import engine, ops
    for size, batch in (('tiny256', 1), ('tiny256', 3), ('tiny', 3)):
        dec = engine.synthetic_llama(size, bits=4, groupsize=64, vocab=32000, seed=3, max_seq=64, batch=batch)
        z = lambda dt, v=0: torch.full((batch, ), v, dtype=dt, device='cuda')
        toks = torch.randint(0, 32000, (20, batch), generator=torch.Generator().manual_seed(1)).tolist()
        for i, t in enumerate(toks):
            dec.set_input(t, i)
            dec.step()
            got = ops.sample_tokens(dec.logits, dec.positions, z(torch.float32), z(torch.int32, 50), z(torch.float32, 0.5), z(torch.int64))
            assert torch.equal(got, dec.next_tokens), f'{size} batch {batch} step {i}'


def test_same_row_same_token_in_every_slot():
    """A row's token depends only on its logits, parameters and position: in every slot of a batch of 8, next to random rows, on every repeat."""
    rng = np.random.default_rng(5)
    V = 32000
    row = _row('random', V, rng)
    for T, k, p in ((0.8, 50, 0.95), (1.0, 0, 0.95), (2.5, 0, 1.0)):
        ref = S.sample_row(row, T, k, p, 77, -1, 0, 1234)
        for slot in range(8):
            for rep in range(3):
                rows = [_row('random', V, rng) for _ in range(8)]
                rows[slot] = row
                got = _launch(rows, [int(rng.integers(4096)) if b != slot else 1234 for b in range(8)], [T] * 8, [k] * 8, [p] * 8,
                              [int(rng.integers(2**62)) if b != slot else 77 for b in range(8)], [-1] * 8, [0] * 8)
                assert got[slot] == ref, (T, k, p, slot, rep)
        assert _launch([row], [1234], [T], [k], [p], [77], [-1], [0])[0] == ref


def test_distribution_of_draws():
    """2^16 draws (positions 0..65535, one seed) from a row with 50 kept tokens: chi-square against the fp64 target (fixed seeds: a fixed
    outcome) and nothing outside the kept set."""
    from scipy.stats import chisquare
    rng = np.random.default_rng(11)
    V = 32000
    row = (rng.standard_normal(V) - 6).astype(np.float16)
    top = rng.permutation(V)[:60]
    row[top] = np.linspace(0, 2.5, 60).astype(np.float16)
    T, k, p = 0.8, 50, 1.0
    z, w, keep = S.kept_weights(row, T, k, p)
    assert keep.sum() == 50
    from gptq_b200 import ops
    logits = torch.from_numpy(np.stack([row] * 8)).cuda()
    pos = torch.arange(65536, dtype=torch.int32, device='cuda').view(-1, 8)
    full = lambda v, dt: torch.full((8, ), v, dtype=dt, device='cuda')
    prm = (full(T, torch.float32), full(k, torch.int32), full(p, torch.float32), full(2024, torch.int64))
    drawn = torch.cat([ops.sample_tokens(logits, pos[i], *prm) for i in range(pos.shape[0])])
    counts = np.bincount(drawn.cpu().numpy(), minlength=V)
    assert counts[~keep].sum() == 0
    expected = w[keep] / w.sum() * 65536
    stat, pval = chisquare(counts[keep], expected)
    print(f'  chi-square {stat:.1f} over 49 degrees of freedom, p = {pval:.3g}')
    assert pval > 1e-4


# ----------------------------------------------------------------------------- engine
MODELS = [('tiny', 4, False), ('tiny256', 4, False), ('tiny256', 3, True)]


def _model(size, bits, act, seed=0, batch=1, vocab=300):
    from gptq_b200 import engine
    return engine.synthetic_llama(size, bits=bits, groupsize=64, act_order=act, vocab=vocab, seed=seed, max_seq=96, batch=batch)


def _ids(n, seed, vocab=300):
    return torch.randint(0, vocab, (n, ), generator=torch.Generator().manual_seed(seed)).tolist()


def _recording(dec):
    """Wrap dec.step so that every step's logits, positions and drawn tokens are kept."""
    log, step = [], dec.step

    def rec(*a, **kw):
        step(*a, **kw)
        torch.cuda.synchronize()
        log.append((dec.logits.cpu().numpy().copy(), dec.positions.tolist(), dec.next_tokens.tolist()))
    dec.step = rec
    return log


@pytest.mark.parametrize('size, bits, act', MODELS)
def test_engine_draws_what_the_restatement_draws(size, bits, act):
    """generate_batch(do_sample=True) with per-sequence parameters: at every step, inside the captured graph, each sequence's token is the
    restatement's on that step's logits row."""
    dec = _model(size, bits, act, seed=2, batch=3)
    if size == 'tiny256':
        assert dec.launches_per_step() == 1
    temps, ks, ps = [0.8, 1.3, 0.5], [50, 0, 7], [0.95, 0.9, 1.0]
    log = _recording(dec)
    out = dec.generate_batch([_ids(n, n) for n in (4, 9, 1)], 12, do_sample=True, temperature=temps, top_k=ks, top_p=ps, seed=99)
    assert all(len(o) == n + 12 for o, n in zip(out, (4, 9, 1)))
    near = 0
    for logits, pos, toks in log:
        for b in range(3):
            want, info = S.sample_row(logits[b], temps[b], ks[b], ps[b], 99 + b, -1, 0, pos[b], details=True)
            if toks[b] != want:
                assert S.near_boundary(info, want, toks[b]), (pos, b, toks[b], want)
                near += 1
    print(f'  {len(log)} steps, {near} near-boundary draws')
    assert dec.sample_graph is not None


@pytest.mark.parametrize('size, bits, act', MODELS)
def test_engine_greedy_seed_and_batch_rows(size, bits, act):
    """do_sample with temperature 0 is greedy generate; one seed gives one output; row b of generate_batch against a batch-1 run seeded
    seed + b: equal up to the first step whose two logits rows restate to different tokens."""
    dec = _model(size, bits, act, seed=4)
    prompt = _ids(6, 3)
    greedy = dec.generate(prompt, 16)
    assert dec.generate(prompt, 16, do_sample=True, temperature=0.0) == greedy
    assert dec.generate(prompt, 16) == greedy  # sampling is cleared afterwards: the greedy graph again
    a = dec.generate(prompt, 16, do_sample=True, temperature=1.0, top_k=0, seed=5)
    assert dec.generate(prompt, 16, do_sample=True, temperature=1.0, top_k=0, seed=5) == a
    assert a != greedy or dec.generate(prompt, 16, do_sample=True, temperature=1.0, top_k=0, seed=6) != a

    prompts = [_ids(n, 10 + n) for n in (5, 2, 8)]
    batch = _model(size, bits, act, seed=4, batch=3)
    blog = _recording(batch)
    rows = batch.generate_batch(prompts, 14, do_sample=True, temperature=0.9, top_p=0.95, seed=1000)
    for b, p in enumerate(prompts):
        slog = _recording(dec)
        one = dec.generate(p, 14, do_sample=True, temperature=0.9, top_p=0.95, seed=1000 + b)
        del dec.step
        j = next((i for i, (x, y) in enumerate(zip(rows[b], one)) if x != y), None)
        if j is None:
            continue
        step = j - len(p)  # generated token j came from step len(p) - 1 + step of this sequence (no prefill steps for batch 1 with prefill)
        lb = [e for e in blog if e[1][b] == j - 1][0]
        ls = [e for e in slog if e[1][0] == j - 1][0]
        tb = S.sample_row(lb[0][b], 0.9, 50, 0.95, 1000 + b, -1, 0, j - 1)
        ts = S.sample_row(ls[0][0], 0.9, 50, 0.95, 1000 + b, -1, 0, j - 1)
        assert tb != ts, f'sequence {b}: batch and batch-1 diverge at token {j} (step {step}) although both logits restate to {tb}'


@pytest.mark.parametrize('size, bits, act', MODELS)
def test_eos_stops_generation(size, bits, act):
    """eos at a token greedy emits at step j ends the output there; min_new_tokens > j keeps it out of the first min_new_tokens tokens."""
    dec = _model(size, bits, act, seed=6)
    prompt = _ids(5, 7)
    gen = dec.generate(prompt, 20)[5:]
    j = 6
    eos = gen[j]
    first = gen.index(eos)
    out = dec.generate(prompt, 20, eos_token_id=eos)
    assert out == prompt + gen[:first + 1]
    assert dec.lengths == [len(out) - 1] and dec.cached_tokens[0] == out[:-1]
    late = dec.generate(prompt, 20, eos_token_id=eos, min_new_tokens=j + 1)[5:]
    assert eos not in late[:j + 1]
    assert late[-1] == eos or len(late) == 20
    s = dec.generate(prompt, 20, do_sample=True, seed=3, eos_token_id=eos, min_new_tokens=3)[5:]
    assert eos not in s[:3] and (eos not in s or s.index(eos) == len(s) - 1)


@pytest.mark.parametrize('size, bits, act', MODELS)
def test_ragged_eos_record_and_second_turn(size, bits, act):
    """Sequences stopping at different steps: each record equals the returned tokens but the last, and a reuse_cache=True turn on top of it
    computes what a fresh generate_batch of the same prompts computes (the near-tie allowance of the multi-turn extend test)."""
    dec = _model(size, bits, act, seed=8, batch=3)
    prompts = [_ids(n, 30 + n) for n in (3, 8, 1)]
    greedy = dec.generate_batch(prompts, 16)
    eos = greedy[0][len(prompts[0]) + 4]
    out = dec.generate_batch(prompts, 16, eos_token_id=eos)
    stops = []
    for b, (o, g, p) in enumerate(zip(out, greedy, prompts)):
        gen = g[len(p):]
        n = gen.index(eos) + 1 if eos in gen else 16
        assert o == g[:len(p) + n], f'sequence {b}'
        assert dec.lengths[b] == len(o) - 1 and dec.cached_tokens[b] == o[:-1], f'sequence {b}: record'
        stops.append(n)
    assert stops[0] == 5
    turn2 = [o + _ids(4, 60 + b) for b, o in enumerate(out)]
    again = dec.generate_batch(turn2, 8, reuse_cache=True)
    fresh = dec.generate_batch(turn2, 8)
    for b in range(3):
        assert again[b][:len(turn2[b])] == turn2[b]
        assert sum(x != y for x, y in zip(again[b], fresh[b])) <= 2, f'sequence {b}: second turn'


def test_engine_argument_errors():
    dec = _model('tiny256', 4, False, batch=2)
    with pytest.raises(ValueError):
        dec.generate_batch([[1], [2]], 4, do_sample=True, temperature=[1.0, 1.0, 1.0])
    with pytest.raises(ValueError):
        dec.generate_batch([[1], [2]], 4, eos_token_id=300)
    with pytest.raises(ValueError):
        dec.generate_batch([[1], [2]], 4, do_sample=True, top_p=0)
