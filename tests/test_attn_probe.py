"""CPU: the constructions of attn_probe.py -- exact qkv products, zero-sum values, a bound that holds for a float32 emulation of the
persistent kernel's chunked online softmax and catches one dropped heavy key, and the float64 reference against torch SDPA."""
import numpy as np
import pytest
import torch

import attn_probe as P
from gpu_util import ulp16
from oracle import gptq_oracle as O


def _probe_qkv(H, act, nkv=None):
    w = P.probe_weights(H, 2 * H, act_order=act, seed=3, n_kv_heads=nkv)
    qw, sc, qz, g, _ = w['qkv']
    return w, O.dequant(qw, sc, qz, g, 4)


@pytest.mark.parametrize('H,act,nkv', [pytest.param(256, False, None, id='256-False'), pytest.param(256, True, None, id='256-True'),
                                       pytest.param(512, False, None, id='512-False')] +
                         [(H, act, nkv) for H, nkv in ((256, 1), (512, 2), (512, 1), (4096, 8), (4096, 1)) for act in (False, True)])
def test_qkv_products_are_exact_in_any_order(H, act, nkv):
    """q, k, v of every probe token are exact in float32 summed sequentially and pairwise and equal the one-tap values.  With nkv K/V heads
    (nh = H / 128, g = nh / nkv): the pair sets of a group cover the 64 RoPE pairs exactly once, q of head h is 0 off its pairs, and the K row
    of head h / g masked to them is q of head h (at g = 1: k == q)."""
    w, W = _probe_qkv(H, act, nkv)
    nh = H // P.HD
    nkv = nkv or nh
    g, Hkv = nh // nkv, nkv * P.HD
    assert W.shape == (H, H + 2 * Hkv)
    assert bool((w['support'].view(nkv, g, 64).sum(1) == 1).all()), 'the sets of a group must cover every pair exactly once'
    mask = P.pair_mask(w['support'])
    n = 16 if H <= 512 else 2
    emb = P.probe_embed(n, H, seed=3)
    x = emb.double() * 16
    assert torch.equal(x.abs(), torch.ones_like(x)), 'RMSNorm input must normalise to +-1'
    exact = x @ W.double()
    seq = np.cumsum((x.float()[:, :, None] * W.float()[None]).numpy(), axis=1, dtype=np.float32)[:, -1]
    pair = (x.float()[:, :, None] * W.float()[None]).numpy().sum(1, dtype=np.float32)
    assert np.array_equal(seq.astype(np.float64), exact.numpy()) and np.array_equal(pair.astype(np.float64), exact.numpy())
    for t in range(n):
        q, k, v = P.exact_qv(w, emb[t])
        assert torch.equal(exact[t, :H], q) and torch.equal(exact[t, H:H + Hkv], k) and torch.equal(exact[t, H + Hkv:], v)
        qh = q.view(nh, P.HD)
        assert not qh[~mask].any(), 'q is not 0 off its pairs'
        assert bool((qh[mask] != 0).all())
        assert torch.equal(k.view(nkv, P.HD).repeat_interleave(g, 0).masked_fill(~mask, 0), qh)
    v = exact[:, H + Hkv:]
    assert bool((v >= 0.5).all() and (v <= 0.875).all() and (v * 16 == (v * 16).round()).all())


def _rope32(x, pos, base):
    """float32 RoPE of rows x [n, 128] rounded to fp16, in the kernels' operation order (x c - y s, x s + y c, two roundings per term) and
    with the angle of check_rope_row (rope_angles32)."""
    f = np.float32
    th = P.rope_angles32(pos, base)
    c, s = np.cos(th).astype(f), np.sin(th).astype(f)
    a, b = x[:, :64].numpy().astype(f), x[:, 64:].numpy().astype(f)
    return torch.from_numpy(np.concatenate([a * c - b * s, a * s + b * c], 1).astype(np.float16))


@pytest.mark.parametrize('H,nkv', [(512, 2), (4096, 8), (4096, 1)])
@pytest.mark.parametrize('base', [1e4, 5e5, 1e6])
def test_rotated_q_is_the_masked_rotated_k(H, nkv, base):
    """RoPE works pair by pair, so the rotated q of head h is the rotated K row of its K/V head masked to h's pairs, bit for bit."""
    w, _ = _probe_qkv(H, False, nkv)
    nh, g = H // P.HD, H // P.HD // nkv
    mask = P.pair_mask(w['support'])
    emb = P.probe_embed(4, H, seed=3)
    for t in range(4):
        q, k, _ = P.exact_qv(w, emb[t])
        for pos in (0, 1, 2047, 16383):
            q_rot = _rope32(q.view(nh, P.HD), pos, base)
            k_rot = _rope32(k.view(nkv, P.HD), pos, base).repeat_interleave(g, 0).masked_fill(~mask, 0)
            assert torch.equal(q_rot, k_rot), f'token {t} pos {pos}'
            assert not q_rot[~mask].any()


def test_identity_o_proj_and_zero_mlp():
    w = P.probe_weights(256, 512, act_order=True, seed=4)
    assert torch.equal(O.dequant(*w['o'][:4], 4).double(), torch.eye(256, dtype=torch.float64))
    for name in ('gate', 'up', 'down'):
        assert torch.equal(O.dequant(*w[name][:4], 4).double().abs().sum(), torch.tensor(0.0, dtype=torch.float64))


@pytest.mark.parametrize('n', [0, 1, 2, 3, 31, 600, 2047])
def test_zero_sum_values_sum_to_exactly_zero(n):
    gen = torch.Generator().manual_seed(n)
    v_new = (torch.randint(8, 15, (4, P.HD), generator=gen) / 16.0).half()
    V = P.zero_sum_values(v_new, n, gen)
    assert V.shape == (4, n, P.HD)
    if n == 0:  # pos 0: no planted row (the anchor there is fp16(x_in + v_new))
        return
    assert bool((V.double().abs() >= 0.5).all() and (V.double().abs() <= 2).all())
    allv = torch.cat([V, v_new[:, None]], 1).float().numpy()
    assert bool((allv * 16 == np.round(allv * 16)).all())
    assert not np.cumsum(allv, axis=1, dtype=np.float32)[:, -1].any()
    assert not allv.sum(1, dtype=np.float32).any()


def _case(kind, T, seed, heavy=None, nh=1, nkv=1):
    """q_rot [nh, 128] of probe-like query heads (one-tap magnitudes, each head on its own pairs of its group: pair_split) and K, V
    [nkv, T, 128]: a planted profile followed by the new K row of each K/V head (the sum of its heads' q) and a new V row."""
    gen = torch.Generator().manual_seed(seed)
    q = (torch.randint(4, 8, (nh, P.HD), generator=gen) * (1 - 2 * torch.randint(0, 2, (nh, P.HD), generator=gen)) / 16.0).half()
    v_new = (torch.randint(8, 15, (nkv, P.HD), generator=gen) / 16.0).half()
    q = q.masked_fill(~P.pair_mask(P.pair_split(nh, nkv, gen)), 0)
    k_new = q.view(nkv, nh // nkv, P.HD).sum(1)  # disjoint supports: exact
    K, V = P.profile(kind, q, T - 1, gen, heavy=heavy, g=nh // nkv)
    return q, torch.cat([K, k_new[:, None]], 1), torch.cat([V, v_new[:, None]], 1)


def _ranges(T, nb=264, n_heads=32, head=0):
    return P.team_ranges([T - 1], n_heads, nb)[(0, head)]


def _ratio(att, E, out):
    """Worst |x_out - x_ref| / x_bound of one head's emulated att `out` [128] against the float64 att [1, 128], at x_in = 2^-4."""
    x_in = torch.full(att.shape, 2.0**-4, dtype=torch.float64)
    x_ref = x_in + att
    return (((x_in + out[None]).half().double() - x_ref).abs() / P.x_bound(att, x_ref, E)).max().item()


GQA = [(4, 2), (8, 1), (32, 8)]  # (query heads, K/V heads)


def _gqa_heavy(T, nh, nb=264):
    """Heavy keys of every query head: the edges of the team ranges of all heads, dealt so that the heads of a group take different keys."""
    edges = sorted(set().union(*[P.edge_keys(T - 1, _ranges(T, nb, nh, h)) for h in range(nh)]))
    return P.deal_heavy(edges, nh)[0]


@pytest.mark.parametrize('kind', P.PROFILES)
@pytest.mark.parametrize('T', [1, 2, 33, 257, 600, 2048])
def test_float32_emulation_is_within_the_bound(kind, T):
    """The bound of attn_probe.x_bound holds for a float32 restatement of the persistent kernel's algorithm (teams of a 7B head)."""
    heavy = [P.edge_keys(T - 1, _ranges(T))[:8]]
    q, K, V = _case(kind, T, T, heavy)
    att, E = P.softmax_ref(q, K, V)
    for nb in (264, 2 * 132 * 16):  # 8 or 9 teams per head, and more teams than units
        out = P.emulate_persistent(q[0], K[0], V[0], _ranges(T, nb)).double()
        x_in = torch.full((1, P.HD), 2.0**-4, dtype=torch.float64)
        x_ref = x_in + att
        x_out = (x_in + out[None]).half().double()
        assert ((x_out - x_ref).abs() / P.x_bound(att, x_ref, E)).max().item() <= 1


@pytest.mark.parametrize('kind', P.PROFILES)
@pytest.mark.parametrize('nh,nkv', GQA)
@pytest.mark.parametrize('T', [2, 257, 600])
def test_float32_emulation_with_shared_kv_heads_is_within_the_bound(kind, nh, nkv, T):
    """The same with g = nh / nkv query heads per K/V head: each query head's teams (team_ranges of nh heads) over K/V head h / g."""
    g = nh // nkv
    q, K, V = _case(kind, T, 7 * T + nh, _gqa_heavy(T, nh), nh, nkv)
    att, E = P.softmax_ref(q, K.repeat_interleave(g, 0), V.repeat_interleave(g, 0))
    for h in range(nh):
        out = P.emulate_persistent(q[h], K[h // g], V[h // g], _ranges(T, 264, nh, h)).double()
        assert _ratio(att[h:h + 1], E[h:h + 1], out) <= 1, f'{kind} head {h}'


@pytest.mark.parametrize('nh,nkv', [(8, 2), (32, 8)])
@pytest.mark.parametrize('T', [33, 600])
def test_reading_another_groups_kv_head_exceeds_the_bound_tenfold(nh, nkv, T):
    """The emulation reading K/V head h % nkv, or the next group's, instead of h / g is 10 times over the bound on the heavy profile."""
    g = nh // nkv
    q, K, V = _case('heavy', T, 11 * T + nh, _gqa_heavy(T, nh), nh, nkv)
    att, E = P.softmax_ref(q, K.repeat_interleave(g, 0), V.repeat_interleave(g, 0))
    checked = 0
    for h in range(nh):
        for c in {h % nkv, (h // g + 1) % nkv} - {h // g}:
            out = P.emulate_persistent(q[h], K[c], V[c], _ranges(T, 264, nh, h)).double()
            ratio = _ratio(att[h:h + 1], E[h:h + 1], out)
            assert ratio >= 10, f'head {h} reading K/V head {c}: worst ratio {ratio:.3g}'
            checked += 1
    assert checked >= nh


@pytest.mark.parametrize('T,nh,nkv', [pytest.param(33, 1, 1, id='33'), pytest.param(600, 1, 1, id='600'), pytest.param(2048, 1, 1, id='2048'),
                                      (33, 8, 2), (600, 8, 2), (600, 32, 8)])
def test_one_dropped_heavy_key_exceeds_the_bound_tenfold(T, nh, nkv):
    """Dropping one heavy key moves the output 10 times over the bound; with grouped-query attention the key is dropped from the shared K/V
    head and the query head it is heavy for (the first and the last head) is checked."""
    g = nh // nkv
    team_heads = nh if nh > 1 else 32  # multi-head: the teams of one 7B head

    def four(h):
        keys = P.edge_keys(T - 1, _ranges(T, 264, team_heads, h))
        return [keys[0], keys[len(keys) // 3], keys[len(keys) // 2], keys[-1]]

    heavy = [four(h) if h in (0, nh - 1) else [] for h in range(nh)]
    q, K, V = _case('heavy', T, 100 + T, heavy, nh, nkv)
    att, E = P.softmax_ref(q, K.repeat_interleave(g, 0), V.repeat_interleave(g, 0))
    for h, keys in enumerate(heavy):
        for t in keys:
            keep = [i for i in range(T) if i != t]
            out = P.emulate_persistent(q[h], K[h // g, keep], V[h // g, keep], _ranges(T - 1, 264, team_heads, h)).double()
            ratio = _ratio(att[h:h + 1], E[h:h + 1], out)
            assert ratio >= 10, f'dropping heavy key {t} of {T} (head {h}): worst ratio {ratio:.3g}'


@pytest.mark.parametrize('g', [1, 2, 8, 32])
def test_keys_for_scores_at_every_group_size(g):
    """With g query heads per K/V head (at g = 32 each q has 2 of the 64 pairs, so u is 4 times longer): the float64 score of every query
    head against the shared K rows is its own alpha within 6 sigma of the noise plus the fp16 rounding of K, and every profile's K stays
    finite in fp16."""
    nh, T = 32, 600
    w = P.probe_weights(4096, 8192, seed=5, n_kv_heads=nh // g)
    q = P.exact_qv(w, P.probe_embed(8, 4096, seed=5)[3])[0].view(nh, P.HD).half()
    gen = torch.Generator().manual_seed(g)
    alpha = torch.cat([torch.randn(nh, T - 3, generator=gen, dtype=torch.float64) * 20, torch.tensor([[95.0, -30.0, 10.5]], dtype=torch.float64).expand(nh, 3)], 1)
    K = P.keys_for_scores(q, alpha, gen, g=g)
    assert K.shape == (nh // g, T, P.HD)
    qd, Kd = q.double(), K.double().repeat_interleave(g, 0)
    s = P.SCALE * torch.einsum('hd,htd->ht', qd, Kd)
    tol = 6 * P.SCALE * 0.02 * qd.norm(dim=-1, keepdim=True) + P.SCALE * torch.einsum('hd,htd->ht', qd.abs(), 0.5 * ulp16(Kd))
    assert bool(((s - alpha).abs() <= tol).all()), f'worst |s - alpha| / tol {((s - alpha).abs() / tol).max().item():.3g}'
    for kind in P.PROFILES:
        Kp, Vp = P.profile(kind, q, T, gen, heavy=[[0, T - 1]] * nh, g=g)
        assert Kp.shape == Vp.shape == (nh // g, T, P.HD) and bool(torch.isfinite(Kp).all()), kind


@pytest.mark.parametrize('kind', ['heavy', 'offset', 'uniform'])
def test_reference_matches_sdpa_in_float64(kind):
    q, K, V = _case(kind, 300, 9, [[0, 31, 32, 298]])
    att, _ = P.softmax_ref(q, K, V)
    ref = torch.nn.functional.scaled_dot_product_attention(q.double()[:, None, :], K.double(), V.double())[:, 0]
    assert torch.allclose(att, ref, rtol=1e-12, atol=1e-12)


def test_partition_restatement():
    """team_ranges cover every unit of every (sequence, head) exactly once, contiguously; the batched shares add up to all teams."""
    for positions, nb, nh in (([2047], 264, 32), ([599], 264, 2), ([0, 31, 32, 255, 256, 1023, 2046, 2047], 264, 32), ([0, 255, 2047, 1, 5, 9], 264, 40)):
        ranges = P.team_ranges(positions, nh, nb)
        for s, p in enumerate(positions):
            for h in range(nh):
                rs = sorted(r for r in ranges[(s, h)] if r[0] < r[1])
                units = [u for b0, b1 in rs for u in range(b0, b1)]
                assert units == list(range(p // P.UNIT + 1))
        if len(positions) > 1:
            shares = [P.seq_teams(positions, nh, nb, s) for s in range(len(positions))]
            assert shares[0][0] == 0 and sum(c for _, c in shares) == nb
            assert all(a[0] + a[1] == b[0] for a, b in zip(shares, shares[1:]))


def test_edge_keys_and_rotation_cover_the_context():
    keys = P.edge_keys(600, _ranges(601))
    assert {0, 599, 31, 32, 255, 256, 511, 512} <= set(keys) and max(keys) < 600
    deal = P.deal_heavy(keys, 2)
    assert sorted(k for ps in deal for h in ps for k in h) == keys and all(len(h) <= 8 for ps in deal for h in ps)
