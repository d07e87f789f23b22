"""A one-layer probe model that makes decode attention observable exactly, in both engines (kernel chain and persistent kernel).

* Inputs.  rms_eps = 0, input_norm = 1, embedding rows of +-2^-4 (+2^-4 on the first V_TAPS features of every row): RMSNorm yields
  exactly +-1 in both engines (the sum of squares is H * 2^-8, so every sqrtf and division is exact).
* qkv.  int4 with scale 2^-4, every weight equal to its column's zero point except one tap per column (exact_fixtures.pow2_packed taken to
  a single term): q_n = x_k * d * 2^-4 with |d| in [4, 7] on a feature k >= V_TAPS, v_n = d * 2^-4 with d in [8, 14] on a feature
  k < V_TAPS (so v > 0).  Every sum is exact in any order.  With n_kv_heads K/V heads (g = nh / nkv query heads per K/V head) the 64 RoPE
  pairs (i, i + 64) of each K/V group are split into g disjoint sets, one per query head (pair_split): query head h taps only the pairs of
  its set, its other q columns stay at the zero point and are exactly 0, and on pair i the k columns of K/V head h / g copy the taps of the
  query head that owns i.  RoPE works pair by pair (a zero pair rotates to zeros), and both engines rotate q and k with the same
  expression (decode.cu attn_decode_kernel, decode_mega.cu run_attention), so the kernel's rotated q of head h IS the appended K row of its
  K/V head masked to h's pairs, bit for bit: the reference reads it back from a first pass instead of re-deriving the fp32 RoPE (which
  check_rope_row holds to fp64 separately).  At g = 1 the set is every pair and the k columns are a copy of the q columns.
* o_proj.  int4 identity (q - z = delta, z = 1, scale 1); with act_order a random g_idx, which kernel_form regroups (o_perm).
* MLP.  gate, up and down have scale 0: the MLP adds exactly 0, so the residual after the step is the residual after attention,
  x_out = fp16(x_in + fp16(att)).

Where the result is read: the persistent kernel's residual ping-pong (resid_buffers: [0] = x entering the layer, [1] = x after attention),
the kernel chain's first scratch region (ScratchLayout.x, offset 0: x after the whole step).

Also: a float64 softmax reference with an element-wise error bound, the key profiles the GPU tests plant in the cache, a float32 emulation of
the persistent kernel's chunked online softmax (CPU tests), and the persistent kernel's attention partition (attn_range / seq_teams of
decode_mega.cu), restated to place keys on team edges.
"""
import math

import numpy as np
import torch

from gpu_util import fp16_ulp_distance, report, ulp16

HD = 128      # head dim
UNIT = 32     # keys per work unit of the persistent kernel (kKeysPerUnit)
SPLIT = 256   # keys per attention CTA of the kernel chain (kAttnChunk)
V_TAPS = 64   # the v taps read features [0, V_TAPS), where every probe embedding row is +2^-4
SCALE = HD**-0.5
U24 = 2.0**-24


# ----------------------------------------------------------------------------- the probe model
def _word(nib: int) -> int:
    return sum(nib << (4 * i) for i in range(8))


def _as_int32(t: torch.Tensor) -> torch.Tensor:
    return torch.where(t >= 2**31, t - 2**32, t).to(torch.int32)


def _pack_taps(K, base, taps_k, taps_val, device):
    """int4 qweight [K/8, N]: every nibble of column n is base[n], except nibble (taps_k[n], n) = taps_val[n]."""
    N = base.numel()
    qw = (base.to(torch.int64) * _word(1))[None, :].repeat(K // 8, 1).to(device)
    n = torch.arange(N, device=device)
    tk = taps_k.to(device)
    qw[tk // 8, n] += (taps_val - base).to(device).to(torch.int64) << (4 * (tk % 8))
    return _as_int32(qw)


def _g_idx(K, gs, act_order, gen):
    g = torch.arange(K) // gs
    if act_order:
        g = g[torch.argsort(torch.randperm(K, generator=gen))]
    return g.to(torch.int32)


def pair_split(nh, nkv, gen):
    """support [nh, 64] bool: the RoPE pairs (i, i + 64) on which query head h has q taps.  Within each K/V group the g = nh / nkv query
    heads get disjoint sets that together cover the 64 pairs exactly once, split at random (drawn from gen); at g = 1 the single set is every
    pair and nothing is drawn."""
    g = nh // nkv
    assert nh % nkv == 0 and g <= 64, (nh, nkv)
    if g == 1:
        return torch.ones(nh, 64, dtype=torch.bool)
    sup = torch.zeros(nh, 64, dtype=torch.bool)
    for c in range(nkv):
        perm = torch.randperm(64, generator=gen)
        for j in range(g):
            sup[c * g + j, perm[j * 64 // g:(j + 1) * 64 // g]] = True
    return sup


def probe_weights(H, I, act_order=False, seed=0, gs=128, n_kv_heads=None):
    """CPU tensors of the probe layer: dict of (qweight, scales, qzeros, g_idx, groupsize) per linear, the qkv taps
    (tq, dq, tk, dk, tv, dv) and the pair support of every query head (pair_split).  n_kv_heads: K/V heads (None: H / 128, multi-head).
    The qkv is (nh + 2 nkv) * 128 wide; query head h taps only the pairs of its set (its other columns are exactly 0), and on pair i of K/V
    head c the k columns copy the taps of the query head whose set holds i."""
    nh = H // HD
    nkv = nh if n_kv_heads is None else n_kv_heads
    Hkv = nkv * HD
    gen = torch.Generator().manual_seed(seed)
    tq = torch.randint(V_TAPS, H, (H, ), generator=gen)
    dq = torch.randint(4, 8, (H, ), generator=gen) * (1 - 2 * torch.randint(0, 2, (H, ), generator=gen))
    tv = torch.randint(0, V_TAPS, (Hkv, ), generator=gen)
    dv = torch.randint(8, 15, (Hkv, ), generator=gen)
    sup = pair_split(nh, nkv, gen)
    dq = dq * pair_mask(sup).reshape(-1)  # off the head's pairs the tap is the zero point: q = 0
    owner = torch.arange(nkv)[:, None] * (nh // nkv) + sup.view(nkv, nh // nkv, 64).to(torch.int64).argmax(1)  # [nkv, 64]: query head of pair i
    src = ((owner * HD).repeat(1, 2) + torch.arange(HD)).reshape(-1)  # the q column each k column copies
    tk, dk = tq[src], dq[src]
    G = H // gs
    base = torch.cat([torch.full((H + Hkv, ), 8), torch.full((Hkv, ), 1)])  # nibble of the zero point: z = stored zero + 1
    qkv = (_pack_taps(H, base, torch.cat([tq, tk, tv]), torch.cat([8 + dq, 8 + dk, 1 + dv]), 'cpu'), torch.full((G, H + 2 * Hkv), 2.0**-4).half(),
           _as_int32(torch.cat([torch.full((G, (H + Hkv) // 8), _word(7)), torch.zeros(G, Hkv // 8, dtype=torch.int64)], 1)), _g_idx(H, gs, act_order, gen), gs)
    eye = _pack_taps(H, torch.ones(H, dtype=torch.int64), torch.arange(H), torch.full((H, ), 2), 'cpu')
    o = (eye, torch.ones(G, H).half(), torch.zeros(G, H // 8, dtype=torch.int32), _g_idx(H, gs, act_order, gen), gs)
    gm = 128 if I % 128 == 0 else 64
    g_mlp = _g_idx(H, gm, act_order, gen)

    def zero_layer(K, N, g):
        return (_as_int32(torch.full((K // 8, N), _word(8))), torch.zeros(K // gm, N).half(), torch.zeros(K // gm, N // 8, dtype=torch.int32), g, gm)

    return dict(qkv=qkv, o=o, gate=zero_layer(H, I, g_mlp), up=zero_layer(H, I, g_mlp.clone()), down=zero_layer(I, H, _g_idx(I, gm, act_order, gen)),
                taps=(tq, dq, tk, dk, tv, dv), support=sup)


def probe_embed(vocab, H, seed=0):
    gen = torch.Generator().manual_seed(seed + 1)
    sign = 1 - 2 * torch.randint(0, 2, (vocab, H), generator=gen)
    sign[:, :V_TAPS] = 1
    return (sign * 2.0**-4).half()


def exact_qv(w, embed_row):
    """float64 q (before RoPE) [H], k (before RoPE) and v [nkv * 128] of the probe for one embedding row: one tap per column, x = embed * 16
    = +-1."""
    tq, dq, tk, dk, tv, dv = w['taps']
    x = embed_row.double().cpu() * 16
    return x[tq] * dq * 2.0**-4, x[tk] * dk * 2.0**-4, x[tv] * dv * 2.0**-4


def pair_mask(support):
    """[nh, 128] bool: the columns of each query head's pairs (i and i + 64 for every pair i of its set)."""
    return support.repeat(1, 2)


def align256(v):
    return (v + 255) // 256 * 256


def resid_buffers(dec):
    """The persistent kernel's residual ping-pong (fp16 [B, H] x 2 at the head of its scratch area, gptq_llama_persistent_scratch_offset):
    after a step [0] = x entering the last layer, [1] = x after the last layer's attention block."""
    B, H = dec.batch, dec.hidden
    step, base = align256(B * H * 2), dec.mega_scratch_offset()
    return [dec.scratch[base + i * step:base + i * step + B * H * 2].view(torch.float16).view(B, H).clone() for i in range(2)]


class Probe:
    """The probe model on a LlamaDecoder (1 layer, n_kv_heads K/V heads: default engine.kv_heads(size); RoPE at rope_base, or with the
    frequency table of rope_scaling, LlamaDecoder's argument).  learn() is pass 1 of a (tokens,
    positions) step: it reads the appended K and V rows of every K/V head (k_new, v_new) and from them each query head's rotated q (q_rot:
    the K row of its K/V head masked to its pairs); run() is pass 2: it plants the cache, poisons the rows at and after each position with
    NaN, steps, checks that exactly row pos of every K/V head was written, bit-identical to pass 1, and returns (x_in, x_out) [B, H] fp16."""

    def __init__(self, size, batch=1, max_seq=2048, act_order=False, vocab=64, seed=0, lm_head=None, rope_base=10000.0, n_kv_heads=None,
                 rope_scaling=None):
        from gptq_b200 import engine
        H, I, _, nh = engine.LLAMA_SHAPES[size]
        nkv = engine.kv_heads(size) if n_kv_heads is None else n_kv_heads
        dev = torch.device('cuda:0')
        self.w = probe_weights(H, I, act_order, seed, n_kv_heads=nkv)
        L = {}
        for name in ('qkv', 'o', 'gate', 'up', 'down'):
            qw, sc, qz, g, gs = self.w[name]
            L[name] = engine.QLayerWeights(qw.to(dev), sc.to(dev), qz.to(dev), g.to(dev), 4, gs)
        L['input_norm'] = torch.ones(H, dtype=torch.float16, device=dev)
        L['post_norm'] = torch.ones(H, dtype=torch.float16, device=dev)
        embed = probe_embed(vocab, H, seed).to(dev)
        if lm_head is None:
            lm_head = (torch.randn(vocab, H, generator=torch.Generator().manual_seed(seed + 2)) * 0.02).half()
        self.dec = engine.LlamaDecoder([L], embed, torch.ones(H, dtype=torch.float16, device=dev), lm_head.to(dev), nh, rms_eps=0.0, batch=batch,
                                       max_seq=max_seq, rope_base=rope_base, n_kv_heads=nkv, rope_scaling=rope_scaling)
        self.H, self.nh, self.nkv, self.g, self.B, self.max_seq = H, nh, nkv, nh // nkv, batch, max_seq
        self.rope = dict(base=rope_base, inv_freq=self.dec.rope_inv_freq)  # the rotation: O.rope_inplace, ops.rotate_half_, check_rope_row
        self.mask = pair_mask(self.w['support']).to(dev)
        self.persistent = self.dec.launches_per_step() == 1
        self.nb = 2 * torch.cuda.get_device_properties(dev).multi_processor_count
        self.q_rot = self.k_new = self.v_new = None

    def _step(self, toks, positions):
        self.dec.set_input(toks, positions)
        self.dec.step()
        torch.cuda.synchronize()

    def appended(self, positions):
        kc, vc = self.dec.k_cache, self.dec.v_cache
        return [kc[0, b, :, p].clone() for b, p in enumerate(positions)], [vc[0, b, :, p].clone() for b, p in enumerate(positions)]

    def learn(self, toks, positions):
        self.dec.k_cache.zero_()
        self.dec.v_cache.zero_()
        self._step(toks, positions)
        self.k_new, self.v_new = self.appended(positions)
        self.q_rot = [k.repeat_interleave(self.g, 0).masked_fill(~self.mask, 0) for k in self.k_new]
        return self.q_rot, self.v_new

    def run(self, toks, positions, plants):
        """plants[b] = (K, V) fp16 [nkv, positions[b], 128]: the cache rows before sequence b's position."""
        kc, vc = self.dec.k_cache, self.dec.v_cache
        for b, (p, (K, V)) in enumerate(zip(positions, plants)):
            kc[0, b, :, :p] = K
            vc[0, b, :, :p] = V
            kc[0, b, :, p:] = float('nan')
            vc[0, b, :, p:] = float('nan')
        self._step(toks, positions)
        k2, v2 = self.appended(positions)
        for b, (p, (K, V)) in enumerate(zip(positions, plants)):
            assert torch.equal(k2[b], self.k_new[b]) and torch.equal(v2[b], self.v_new[b]), f'sequence {b}: pass 2 appended other K / V rows'
            assert torch.equal(kc[0, b, :, :p], K) and torch.equal(vc[0, b, :, :p], V), f'sequence {b}: a planted row before pos {p} changed'
            assert bool(kc[0, b, :, p + 1:].isnan().all() and vc[0, b, :, p + 1:].isnan().all()), f'sequence {b}: a row after pos {p} was written'
        if self.persistent:
            x_in, x_out = resid_buffers(self.dec)
            assert torch.equal(x_in, self.dec.embed[torch.tensor(toks, device=x_in.device)]), 'residual entering the layer is not the embedding row'
        else:
            B, H = self.B, self.H
            x_in = self.dec.embed[torch.tensor(toks, device=self.dec.dev)]
            x_out = self.dec.scratch[:B * H * 2].view(torch.float16).view(B, H).clone()
        return x_in, x_out


# ----------------------------------------------------------------------------- float64 reference and bound
def softmax_ref(q, K, V):
    """float64 softmax attention of one sequence: q [nh, 128], K / V [nh, T, 128] (every key, the new one included) ->
    (att [nh, 128], E [nh, 128]): E bounds the error of an fp32 kernel before its fp16 store:
      * fp32 scores: |ds_t| <= (128 + 8) 2^-24 scale sum_i |q_i K_ti|, carried through the softmax as 2 max|ds| sum_t p_t |V_t - att|;
      * fp32 accumulation, expf and the rescales: 4 (T + 64) 2^-24 sum_t p_t |V_t|."""
    q64, K64, V64 = q.double(), K.double(), V.double()
    T = K.shape[1]
    s = torch.einsum('hd,htd->ht', q64, K64) * SCALE
    p = torch.softmax(s, -1)
    att = torch.einsum('ht,htd->hd', p, V64)
    ds = (HD + 8) * U24 * SCALE * torch.einsum('hd,htd->ht', q64.abs(), K64.abs())
    E = 2 * ds.max(-1).values[:, None] * torch.einsum('ht,htd->hd', p, (V64 - att[:, None, :]).abs())
    E = E + 4 * (T + 64) * U24 * torch.einsum('ht,htd->hd', p, V64.abs())
    return att, E


def x_bound(att, x_ref, E):
    """Bound of |x_out - x_ref| per element: the fp16 stores of att and of the residual add (1.5 ulp16 of the larger magnitude), the
    softmax error E, and the identity o_proj's zero-point term (s (sum x w - z sum x) over a group: 16 2^-24 sum_head |att|)."""
    return 1.5 * ulp16(torch.maximum(att.abs(), x_ref.abs())) + E + 16 * U24 * att.abs().sum(-1, keepdim=True)


# ----------------------------------------------------------------------------- planted keys
def keys_for_scores(q, alpha, gen, noise=0.02, g=1):
    """K [nh / g, T, 128] fp16 whose scores scale * q_h.K_t are about alpha [nh, T] for every query head h: K/V head c holds
    sum_j alpha_{cg+j} u_{cg+j} plus small noise, u_h = q_h / (scale |q_h|^2).  The query heads of a group have disjoint supports
    (pair_split), so q_h.u_h' = 0 for h' != h and each head scores against its own alpha."""
    qd = q.double()
    u = qd / (SCALE * (qd * qd).sum(-1, keepdim=True))
    nh, T = alpha.shape
    eta = torch.randn((nh // g, T, HD), generator=gen, device=q.device, dtype=torch.float64) * noise
    return ((alpha[..., None] * u[:, None, :]).view(nh // g, g, T, HD).sum(1) + eta).half()


def new_key_score(q):
    qd = q.double()
    return SCALE * (qd * qd).sum(-1)  # [nh]


def zero_sum_values(v_new, n, gen):
    """V [nh, n, 128] fp16, multiples of 2^-4 with 0.5 <= |v| <= 2, such that sum(V) + v_new = 0 exactly in every dimension (v_new: a
    multiple of 2^-4, |v_new| <= 1).  Greedy rows of magnitude [0.5, 1] towards zero keep |running sum| <= 1; the last two rows close it."""
    S = v_new.double().cpu().numpy().copy()
    rng = np.random.default_rng(int(torch.randint(0, 2**31, (1, ), generator=gen, device=gen.device).item()))
    rows = np.zeros((n, ) + S.shape)
    sgn = lambda a: np.where(a < 0, 1.0, -1.0)  # the sign that moves a towards 0 (or -1 at 0)
    for i in range(max(n - 2, 0)):
        rows[i] = sgn(S) * (0.5 + 0.0625 * rng.integers(0, 9, S.shape))
        S += rows[i]
    if n == 1:
        rows[0] = -S
    elif n >= 2:
        a = sgn(S) * np.where(np.abs(S) < 0.5, 1.0, 1.5)
        rows[n - 2], rows[n - 1] = a, -S - a
    rows = rows[rng.permutation(n)]
    return torch.from_numpy(np.ascontiguousarray(rows.transpose(1, 0, 2))).half().to(v_new.device)


def random_values(nh, n, gen, device):
    """V rows in [0.5, 2]: positive, so that att lies in [0.5, 2] too and the identity o_proj sums it exactly."""
    return (torch.rand(nh, n, HD, generator=gen, device=device, dtype=torch.float64) * 1.5 + 0.5).half()


PROFILES = ('heavy', 'ramp', 'late', 'new_max', 'offset', 'wide', 'uniform')


def profile(kind, q, n, gen, heavy=None, g=1):
    """(K, V) [nh / g, n, 128] fp16 planted before a new key whose score is new_key_score(q), per query head h of q [nh, 128]:
      heavy    background N(0, 1), the keys heavy[h] of head h about 10 above it (distinct random V rows)
      ramp     the scores climb with t: the running max moves in every unit and split (the alpha / w0 rescale)
      late     background N(0, 1), the max (+12) in the last unit and at the first key of the last split
      new_max  every planted key 10 below the new key
      offset   scores about +90 (fp32 exp overflows without the max subtraction); the new key ends up with weight 0
      wide     scores spread over 60: most of the background underflows next to the max
      uniform  near-equal scores: a missing unit of 32 keys shifts att by 32 / T of |V - att|
    g query heads share each K/V head (keys_for_scores)."""
    nh, dev = q.shape[0], q.device
    rnd = lambda *s: torch.randn(*s, generator=gen, device=dev, dtype=torch.float64)
    t = torch.arange(n, device=dev, dtype=torch.float64)
    if kind == 'heavy':
        alpha = rnd(nh, n)
        for h, keys in enumerate(heavy or []):
            if keys:
                alpha[h, list(keys)] = 10 + 0.5 * torch.rand(len(keys), generator=gen, device=dev, dtype=torch.float64)
    elif kind == 'ramp':
        alpha = 8 * t / max(n, 1) + 0.3 * rnd(nh, n)
    elif kind == 'late':
        alpha = rnd(nh, n)
        if n:
            alpha[:, n - 1] = 12
            alpha[:, (n - 1) // SPLIT * SPLIT] = 12
    elif kind == 'new_max':
        alpha = new_key_score(q)[:, None] - 10 + rnd(nh, n)
    elif kind == 'offset':
        alpha = 90 + rnd(nh, n)
    elif kind == 'wide':
        alpha = 30 - 60 * torch.rand(nh, n, generator=gen, device=dev, dtype=torch.float64)
    elif kind == 'uniform':
        alpha = 0.05 * rnd(nh, n)
    else:
        raise ValueError(kind)
    return keys_for_scores(q, alpha, gen, g=g), random_values(nh // g, n, gen, dev)


# ----------------------------------------------------------------------------- the persistent kernel's attention partition
def attn_range(T, n_heads, nb, upb):
    """decode_mega.cu attn_range: (head, b0, b1) of team T of nb for upb units per head."""
    base, rem = nb // n_heads, nb % n_heads
    split = rem * (base + 1)
    if T < split:
        head, idx, cnt = T // (base + 1), T % (base + 1), base + 1
    else:
        head, idx, cnt = rem + (T - split) // base, (T - split) % base, base
    return head, idx * upb // cnt, (idx + 1) * upb // cnt


def seq_teams(positions, n_heads, nb, s):
    """decode_mega.cu seq_teams: (first, count) of the teams of sequence s."""
    units = [p // UNIT + 1 for p in positions]
    extra = nb - len(positions) * n_heads
    before, tot = sum(units[:s]), sum(units)
    first = s * n_heads + extra * before // tot
    return first, (s + 1) * n_heads + extra * (before + units[s]) // tot - first


def team_ranges(positions, n_heads, nb):
    """{(sequence, head): [(b0, b1), ...]}: the unit ranges of the teams that serve each (sequence, head) pair."""
    out = {}
    for s, p in enumerate(positions):
        first, count = seq_teams(positions, n_heads, nb, s) if len(positions) > 1 else (0, nb)
        upb = (p + 1 + UNIT - 1) // UNIT
        for T in range(count):
            h, b0, b1 = attn_range(T, n_heads, count, upb)
            out.setdefault((s, h), []).append((b0, b1))
    return out


def edge_keys(pos, ranges=()):
    """Planted keys (< pos) where a partition can slip: 0, pos - 1, both sides of every unit and split edge, and the first and last unit of
    every team range (both ends of each)."""
    ks = {0, pos - 1}
    for e in range(UNIT, pos, UNIT):
        ks |= {e - 1, e}
    for b0, b1 in ranges:
        if b0 < b1:
            ks |= {UNIT * b0, UNIT * b0 + UNIT - 1, UNIT * (b1 - 1), UNIT * b1 - 1}
    return sorted(k for k in ks if 0 <= k < pos)


def team_edge_positions(n_heads, nb):
    """Positions where the number of units per head crosses the number of teams per head (empty teams appear or disappear)."""
    out = set()
    for cnt in {nb // n_heads, nb // n_heads + 1}:
        for u in (cnt - 1, cnt, cnt + 1):
            out |= {UNIT * u - 1, UNIT * u}
    return sorted(out)


def deal_heavy(edges, nh, per=8, offset=0):
    """Heavy key sets [nh][<= per] that cover `edges` over ceil(len / (nh * per)) passes; offset rotates the deal (one pass per position)."""
    n = len(edges)
    if n == 0:
        return [[[] for _ in range(nh)]]
    passes = max(1, -(-n // (nh * per)))
    rot = edges[offset % n:] + edges[:offset % n]
    return [[sorted(set(rot[(j * nh + h) * per:(j * nh + h + 1) * per])) for h in range(nh)] for j in range(passes)]


# ----------------------------------------------------------------------------- float32 emulation (CPU tests)
def emulate_persistent(q, K, V, ranges):
    """float32 emulation of run_attention + the record merge for one head: each team walks its units; key group g (of 32) keeps an online
    softmax over key g of every unit, the groups are merged, then the team records.  q [128], K / V [T, 128] -> att [128] (fp16)."""
    q32 = q.float().numpy()
    K32, V32 = K.float().numpy(), V.float().numpy()
    T = K.shape[0]
    f = np.float32
    recs = []
    for b0, b1 in ranges:
        if b0 >= b1:
            recs.append((f(-np.inf), f(0), np.zeros(HD, f)))
            continue
        m = np.full(UNIT, -np.inf, f)
        l = np.zeros(UNIT, f)
        o = np.zeros((UNIT, HD), f)
        for b in range(b0, b1):
            keys = b * UNIT + np.arange(UNIT)
            ok = keys < T
            kk = np.where(ok, keys, 0)
            s = (K32[kk] * q32).sum(-1, dtype=f) * f(SCALE)
            mn = np.where(ok, np.maximum(m, s), m)
            with np.errstate(invalid='ignore', over='ignore'):
                alpha = np.where(m == -np.inf, f(0), np.exp(m - mn)).astype(f)
                pw = np.exp(s - mn).astype(f)
            l = np.where(ok, l * alpha + pw, l).astype(f)
            o = np.where(ok[:, None], o * alpha[:, None] + pw[:, None] * V32[kk], o).astype(f)
            m = mn
        M = m.max()
        w = np.where(m == -np.inf, f(0), np.exp(m - M)).astype(f)
        recs.append((M, (l * w).sum(dtype=f), (o * w[:, None]).sum(0, dtype=f)))
    M = max(r[0] for r in recs)
    L, O = f(0), np.zeros(HD, f)
    for m, l, o in recs:
        w = f(0) if m == -np.inf else np.exp(f(m - M))
        L, O = f(L + l * w), (O + o * w).astype(f)
    return torch.from_numpy((O / L).astype(np.float16))


# ----------------------------------------------------------------------------- RoPE of the appended K row
def rope_angles32(pos, base=10000.0, inv_freq=None):
    """The fp32 RoPE angles [64] at pos, as the kernels and O.rope_inplace compute them: fp32(f_i * pos), where f_i is the table's
    inv_freq[i], else fp32 exp(i * fp32(-2 ln(base) / 128)) (quant/fused_attn.py:43)."""
    f = np.float32
    freq = np.exp(np.arange(64, dtype=f) * f(-2.0 * math.log(base) / HD)).astype(f) if inv_freq is None else np.asarray(inv_freq, dtype=f)
    return (freq * f(pos)).astype(f)


def check_rope_row(k_row, k_exact, pos, base=10000.0, inv_freq=None):
    """The rotated rows [rows, 128] (fp16; the appended K rows [nkv, 128]) against fp64 RoPE of the exact rows [rows * 128] (exact_qv) at
    the fp32 angles of rope_angles32 (the rotation at `base`, or the table's): within 1 ulp16, plus a 4-ulp difference in the fp32 angle and
    in cos / sin.  Returns the worst |err| / bound."""
    th = rope_angles32(pos, base, inv_freq).astype(np.float64)
    x = k_exact.view(-1, HD)[:, :64].numpy()
    y = k_exact.view(-1, HD)[:, 64:].numpy()
    c, s = np.cos(th), np.sin(th)
    ref = torch.from_numpy(np.concatenate([x * c - y * s, x * s + y * c], 1))
    dth = 4 * np.spacing(th.astype(np.float32)).astype(np.float64) + 4 * U24
    slack = torch.from_numpy(np.tile((np.abs(x) + np.abs(y)) * dth, 2))
    bound = ulp16(ref) + slack
    return ((k_row.double().cpu() - ref).abs() / bound).max().item()


def prefill_row(probe, tok, pos):
    """The K rows [nkv, 128] of position pos as the prefill writes them: the exact k of the probe (exact_qv) rotated by ops.rotate_half_
    with the probe's rotation."""
    from gptq_b200 import ops
    k = exact_qv(probe.w, probe.dec.embed[tok])[1].half().view(1, 1, 1, probe.nkv, HD).cuda()
    ops.rotate_half_(k, torch.tensor([[pos]], device='cuda'), **probe.rope)
    return k.view(probe.nkv, HD)


# ----------------------------------------------------------------------------- GPU sweeps of the probe
class Worst:
    def __init__(self, what):
        self.what, self.ratio, self.where = what, 0.0, ''

    def update(self, ratio_t, where):
        r = ratio_t.max().item() if torch.is_tensor(ratio_t) else float(ratio_t)
        if torch.is_tensor(ratio_t) and not r <= 1:
            idx = [int(i) for i in torch.nonzero(~(ratio_t <= 1))[0]]
            where = f'{where} head {idx[0]} dim {idx[1]}'
        if not r <= self.ratio:
            self.ratio, self.where = r, where

    def done(self):
        report(self.ratio, f'{self.what} (worst at {self.where})' if self.ratio > 1 else self.what)


def anchors(probe, toks, positions, gen, what):
    """Equal scores and zero-sum values (pos 0: the lone new key): x_out must be x_in (fp16(x_in + v_new) at pos 0) bit for bit."""
    plants = [(k[:, None, :].expand(-1, p, -1).contiguous(), zero_sum_values(v, p, gen)) for k, v, p in zip(probe.k_new, probe.v_new, positions)]
    x_in, x_out = probe.run(toks, positions, plants)
    for b, p in enumerate(positions):
        want = x_in[b] if p > 0 else (x_in[b].double() + probe.v_new[b].repeat_interleave(probe.g, 0).reshape(-1).double()).half()
        if not torch.equal(x_out[b], want):
            d = fp16_ulp_distance(x_out[b], want)
            i = int(torch.nonzero(d)[0])
            raise AssertionError(f'{what} seq {b} pos {p}: {int((d > 0).sum())} elements off, up to {int(d.max())} ulp; first at head {i // HD} '
                                 f'dim {i % HD}: {x_out[b, i].item()} vs {want[i].item()}')


def bounded(probe, toks, positions, plants, worst, what):
    x_in, x_out = probe.run(toks, positions, plants)
    for b, p in enumerate(positions):
        K = torch.cat([plants[b][0], probe.k_new[b][:, None, :]], 1).repeat_interleave(probe.g, 0)
        V = torch.cat([plants[b][1], probe.v_new[b][:, None, :]], 1).repeat_interleave(probe.g, 0)
        att, E = softmax_ref(probe.q_rot[b], K, V)
        x_ref = x_in[b].double().view(-1, HD) + att
        out = x_out[b].double().view(-1, HD)
        assert torch.isfinite(out).all(), f'{what} seq {b} pos {p}: non-finite output'
        worst.update((out - x_ref).abs() / x_bound(att, x_ref, E), f'{what} seq {b} pos {p}')


def heavy_passes(probe, positions, rotate=None):
    """Heavy key sets per pass: [pass][sequence][head] -> keys.  rotate = offset: one pass, the edges dealt from that offset."""
    ranges = team_ranges(positions, probe.nh, probe.nb) if probe.persistent else {}
    per_seq = []
    for b, p in enumerate(positions):
        edges = sorted(set().union(*[edge_keys(p, ranges.get((b, h), ())) for h in range(probe.nh)]))
        deal = deal_heavy(edges, probe.nh, offset=rotate or 0)
        per_seq.append(deal[:1] if rotate is not None else deal)
    n = max(len(d) for d in per_seq)
    return [[d[j % len(d)] for d in per_seq] for j in range(n)]


def rotation_passes(nh, T):
    """8 passes of nh heads x 8 keys in which every key t < T is heavy once: pass t % 8, head (t // 8) % nh."""
    out = [[[] for _ in range(nh)] for _ in range(8)]
    for t in range(T):
        out[t % 8][(t // 8) % nh].append(t)
    return out


def sweep(probe, position_sets, profiles, gen, worst, rope, toks=lambda i, b: 7 * i + 3 * b, rotate_heavy=False, full_rotation=()):
    """Position set i of `position_sets` with the tokens toks(i, b) % vocab: pass 1 (probe.learn), the appended K rows against fp64 RoPE
    (check_rope_row) and bit for bit against the prefill's rotation (prefill_row), the bit-exact anchors, then each profile, bounded."""
    vocab = probe.dec.vocab
    for i, positions in enumerate(position_sets):
        tk = [toks(i, b) % vocab for b in range(probe.B)]
        what = f'toks {tk} positions {positions}'
        probe.learn(tk, positions)
        for b, p in enumerate(positions):  # the appended K rows (q_rot, masked) against fp64 RoPE of the exact k and the prefill's rotation
            k_exact = exact_qv(probe.w, probe.dec.embed[tk[b]])[1]
            rope.update(check_rope_row(probe.k_new[b], k_exact, p, **probe.rope), f'{what} seq {b}')
            assert torch.equal(probe.k_new[b], prefill_row(probe, tk[b], p)), f'{what} seq {b}: the step and the prefill rotate differently'
        anchors(probe, tk, positions, gen, what)
        for kind in profiles:
            if kind == 'heavy':
                passes = heavy_passes(probe, positions, rotate=(i * 8 * probe.nh) if rotate_heavy else None)
                if len(positions) == 1 and positions[0] in full_rotation:
                    passes += [[r] for r in rotation_passes(probe.nh, positions[0])]
                for heavy in passes:
                    plants = [profile('heavy', q, p, gen, heavy=hv, g=probe.g) for q, p, hv in zip(probe.q_rot, positions, heavy)]
                    bounded(probe, tk, positions, plants, worst[kind], what + ' heavy')
            else:
                plants = [profile(kind, q, p, gen, g=probe.g) for q, p in zip(probe.q_rot, positions)]
                bounded(probe, tk, positions, plants, worst[kind], f'{what} {kind}')


def run_sweeps(probe, name, position_sets, profiles=PROFILES, seed=1234, **kw):
    """sweep over every position set, with the worst |err| / bound of each profile and of the RoPE rows printed (pytest -s)."""
    gen = torch.Generator(device='cuda:0').manual_seed(seed)
    worst = {k: Worst(f'{name} {k}') for k in profiles}
    rope = Worst(f'{name} appended K row vs fp64 RoPE')
    sweep(probe, position_sets, profiles, gen, worst, rope, **kw)
    for w in list(worst.values()) + [rope]:
        w.done()
