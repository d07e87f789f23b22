"""CPU: the constructions of attn_probe.py -- exact qkv products, zero-sum values, a bound that holds for a float32 emulation of the
persistent kernel's chunked online softmax and catches one dropped heavy key, and the float64 reference against torch SDPA."""
import numpy as np
import pytest
import torch

import attn_probe as P
from oracle import gptq_oracle as O


def _probe_qkv(H, act):
    w = P.probe_weights(H, 2 * H, act_order=act, seed=3)
    qw, sc, qz, g, _ = w['qkv']
    return w, O.dequant(qw, sc, qz, g, 4)


@pytest.mark.parametrize('H,act', [(256, False), (256, True), (512, False)])
def test_qkv_products_are_exact_in_any_order(H, act):
    """q, k, v of every probe token are exact in float32 summed sequentially and pairwise, equal the one-tap values, and k == q."""
    w, W = _probe_qkv(H, act)
    emb = P.probe_embed(16, H, seed=3)
    x = emb.double() * 16
    assert torch.equal(x.abs(), torch.ones_like(x)), 'RMSNorm input must normalise to +-1'
    exact = x @ W.double()
    seq = np.cumsum((x.float()[:, :, None] * W.float()[None]).numpy(), axis=1, dtype=np.float32)[:, -1]
    pair = (x.float()[:, :, None] * W.float()[None]).numpy().sum(1, dtype=np.float32)
    assert np.array_equal(seq.astype(np.float64), exact.numpy()) and np.array_equal(pair.astype(np.float64), exact.numpy())
    for t in range(16):
        q, v = P.exact_qv(w, emb[t])
        assert torch.equal(exact[t, :H], q) and torch.equal(exact[t, H:2 * H], q) and torch.equal(exact[t, 2 * H:], v)
    v = exact[:, 2 * H:]
    assert bool((v >= 0.5).all() and (v <= 0.875).all() and (v * 16 == (v * 16).round()).all())


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


def _case(kind, T, seed, heavy=None):
    gen = torch.Generator().manual_seed(seed)
    q = (torch.randint(4, 8, (1, P.HD), generator=gen) * (1 - 2 * torch.randint(0, 2, (1, P.HD), generator=gen)) / 16.0).half()
    v_new = (torch.randint(8, 15, (1, P.HD), generator=gen) / 16.0).half()
    K, V = P.profile(kind, q, T - 1, gen, heavy=heavy)
    return q, torch.cat([K, q[:, None]], 1), torch.cat([V, v_new[:, None]], 1)


def _ranges(T, nb=264, n_heads=32):
    return P.team_ranges([T - 1], n_heads, nb)[(0, 0)]


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


@pytest.mark.parametrize('T', [33, 600, 2048])
def test_one_dropped_heavy_key_exceeds_the_bound_tenfold(T):
    keys = P.edge_keys(T - 1, _ranges(T))
    heavy = [[keys[0], keys[len(keys) // 3], keys[len(keys) // 2], keys[-1]]]
    q, K, V = _case('heavy', T, 100 + T, heavy)
    att, E = P.softmax_ref(q, K, V)
    x_in = torch.full((1, P.HD), 2.0**-4, dtype=torch.float64)
    x_ref = x_in + att
    bound = P.x_bound(att, x_ref, E)
    for t in heavy[0]:
        keep = [i for i in range(T) if i != t]
        out = P.emulate_persistent(q[0], K[0, keep], V[0, keep], _ranges(T - 1)).double()
        ratio = (((x_in + out[None]).half().double() - x_ref).abs() / bound).max().item()
        assert ratio >= 10, f'dropping heavy key {t} of {T}: worst ratio {ratio:.3g}'


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
