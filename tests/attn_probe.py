"""A one-layer probe model that makes decode attention observable exactly, in both engines (kernel chain and persistent kernel).

* Inputs.  rms_eps = 0, input_norm = 1, embedding rows of +-2^-4 (+2^-4 on the first V_TAPS features of every row): RMSNorm yields
  exactly +-1 in both engines (the sum of squares is H * 2^-8, so every sqrtf and division is exact).
* qkv.  int4 with scale 2^-4, every weight equal to its column's zero point except one tap per column (exact_fixtures.pow2_packed taken to
  a single term): q_n = x_k * d * 2^-4 with |d| in [4, 7] on a feature k >= V_TAPS, v_n = d * 2^-4 with d in [8, 14] on a feature
  k < V_TAPS (so v > 0).  Every sum is exact in any order.  The k columns are a copy of the q columns, and both engines rotate q and k with
  the same expression (decode.cu attn_decode_kernel, decode_mega.cu run_attention), so the appended K row IS the kernel's rotated q, bit for
  bit: the reference reads it back from a first pass instead of re-deriving the fp32 RoPE (which check_rope_row holds to fp64 separately).
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

from gpu_util import ulp16

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


def probe_weights(H, I, act_order=False, seed=0, gs=128):
    """CPU tensors of the probe layer: dict of (qweight, scales, qzeros, g_idx, groupsize) per linear, plus the qkv taps."""
    gen = torch.Generator().manual_seed(seed)
    tq = torch.randint(V_TAPS, H, (H, ), generator=gen)
    dq = torch.randint(4, 8, (H, ), generator=gen) * (1 - 2 * torch.randint(0, 2, (H, ), generator=gen))
    tv = torch.randint(0, V_TAPS, (H, ), generator=gen)
    dv = torch.randint(8, 15, (H, ), generator=gen)
    G = H // gs
    base = torch.cat([torch.full((2 * H, ), 8), torch.full((H, ), 1)])  # nibble of the zero point: z = stored zero + 1
    qkv = (_pack_taps(H, base, torch.cat([tq, tq, tv]), torch.cat([8 + dq, 8 + dq, 1 + dv]), 'cpu'), torch.full((G, 3 * H), 2.0**-4).half(),
           _as_int32(torch.cat([torch.full((G, 2 * H // 8), _word(7)), torch.zeros(G, H // 8, dtype=torch.int64)], 1)), _g_idx(H, gs, act_order, gen), gs)
    eye = _pack_taps(H, torch.ones(H, dtype=torch.int64), torch.arange(H), torch.full((H, ), 2), 'cpu')
    o = (eye, torch.ones(G, H).half(), torch.zeros(G, H // 8, dtype=torch.int32), _g_idx(H, gs, act_order, gen), gs)
    gm = 128 if I % 128 == 0 else 64
    g_mlp = _g_idx(H, gm, act_order, gen)

    def zero_layer(K, N, g):
        return (_as_int32(torch.full((K // 8, N), _word(8))), torch.zeros(K // gm, N).half(), torch.zeros(K // gm, N // 8, dtype=torch.int32), g, gm)

    return dict(qkv=qkv, o=o, gate=zero_layer(H, I, g_mlp), up=zero_layer(H, I, g_mlp.clone()), down=zero_layer(I, H, _g_idx(I, gm, act_order, gen)),
                taps=(tq, dq, tv, dv))


def probe_embed(vocab, H, seed=0):
    gen = torch.Generator().manual_seed(seed + 1)
    sign = 1 - 2 * torch.randint(0, 2, (vocab, H), generator=gen)
    sign[:, :V_TAPS] = 1
    return (sign * 2.0**-4).half()


def exact_qv(w, embed_row):
    """float64 q (before RoPE) and v [H] of the probe for one embedding row: one tap per column, x = embed * 16 = +-1."""
    tq, dq, tv, dv = w['taps']
    x = embed_row.double().cpu() * 16
    return x[tq] * dq * 2.0**-4, x[tv] * dv * 2.0**-4


def align256(v):
    return (v + 255) // 256 * 256


def resid_buffers(dec):
    """The persistent kernel's residual ping-pong (fp16 [B, H] x 2 at the head of its scratch area, gptq_llama_persistent_scratch_offset):
    after a step [0] = x entering the last layer, [1] = x after the last layer's attention block."""
    B, H = dec.batch, dec.hidden
    step, base = align256(B * H * 2), dec.mega_scratch_offset()
    return [dec.scratch[base + i * step:base + i * step + B * H * 2].view(torch.float16).view(B, H).clone() for i in range(2)]


class Probe:
    """The probe model on a LlamaDecoder (1 layer).  learn() is pass 1 of a (tokens, positions) step: it reads the appended K rows (= the
    kernel's rotated q) and V rows; run() is pass 2: it plants the cache, poisons the rows at and after each position with NaN, steps, checks
    that the appended rows are bit-identical to pass 1 and returns (x_in, x_out) [B, H] fp16."""

    def __init__(self, size, batch=1, max_seq=2048, act_order=False, vocab=64, seed=0, lm_head=None, rope_base=10000.0):
        from gptq_b200 import engine
        H, I, _, nh = engine.LLAMA_SHAPES[size]
        dev = torch.device('cuda:0')
        self.w = probe_weights(H, I, act_order, seed)
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
                                       max_seq=max_seq, rope_base=rope_base)
        self.H, self.nh, self.B, self.max_seq, self.rope_base = H, nh, batch, max_seq, rope_base
        self.persistent = self.dec.launches_per_step() == 1
        self.nb = 2 * torch.cuda.get_device_properties(dev).multi_processor_count
        self.q_rot = self.v_new = None

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
        self.q_rot, self.v_new = self.appended(positions)
        return self.q_rot, self.v_new

    def run(self, toks, positions, plants):
        """plants[b] = (K, V) fp16 [nh, positions[b], 128]: the cache rows before sequence b's position."""
        kc, vc = self.dec.k_cache, self.dec.v_cache
        for b, (p, (K, V)) in enumerate(zip(positions, plants)):
            kc[0, b, :, :p] = K
            vc[0, b, :, :p] = V
            kc[0, b, :, p:] = float('nan')
            vc[0, b, :, p:] = float('nan')
        self._step(toks, positions)
        k2, v2 = self.appended(positions)
        for b in range(self.B):
            assert torch.equal(k2[b], self.q_rot[b]) and torch.equal(v2[b], self.v_new[b]), f'sequence {b}: pass 2 appended other K / V rows'
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
def keys_for_scores(q, alpha, gen, noise=0.02):
    """K [nh, T, 128] fp16 whose scores scale * q.K_t are about alpha [nh, T]: alpha_t times q / (scale |q|^2), plus small noise."""
    qd = q.double()
    u = qd / (SCALE * (qd * qd).sum(-1, keepdim=True))
    eta = torch.randn(alpha.shape + (HD, ), generator=gen, device=q.device, dtype=torch.float64) * noise
    return (alpha[..., None] * u[:, None, :] + eta).half()


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


def profile(kind, q, n, gen, heavy=None):
    """(K, V) [nh, n, 128] fp16 planted before a new key whose score is new_key_score(q):
      heavy    background N(0, 1), the keys heavy[h] of head h about 10 above it (distinct random V rows)
      ramp     the scores climb with t: the running max moves in every unit and split (the alpha / w0 rescale)
      late     background N(0, 1), the max (+12) in the last unit and at the first key of the last split
      new_max  every planted key 10 below the new key
      offset   scores about +90 (fp32 exp overflows without the max subtraction); the new key ends up with weight 0
      wide     scores spread over 60: most of the background underflows next to the max
      uniform  near-equal scores: a missing unit of 32 keys shifts att by 32 / T of |V - att|"""
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
    return keys_for_scores(q, alpha, gen), random_values(nh, n, gen, dev)


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
def check_rope_row(k_row, q_exact, pos, rope_base):
    """The appended K row [nh, 128] (fp16) against fp64 RoPE of the exact q / k [H] at base rope_base, the angle computed in fp32 as the
    reference formula does (quant/fused_attn.py:43): within 1 ulp16, plus a 4-ulp difference in the fp32 angle and in cos / sin.  Returns the
    worst |err| / bound."""
    f = np.float32
    inv_base = f(-2.0 * math.log(rope_base) / HD)
    th = (np.exp(np.arange(64, dtype=f) * inv_base).astype(f) * f(pos)).astype(np.float64)
    x = q_exact.view(-1, HD)[:, :64].numpy()
    y = q_exact.view(-1, HD)[:, 64:].numpy()
    c, s = np.cos(th), np.sin(th)
    ref = torch.from_numpy(np.concatenate([x * c - y * s, x * s + y * c], 1))
    dth = 4 * np.spacing(th.astype(f)).astype(np.float64) + 4 * U24
    slack = torch.from_numpy(np.tile((np.abs(x) + np.abs(y)) * dth, 2))
    bound = ulp16(ref) + slack
    return ((k_row.double().cpu() - ref).abs() / bound).max().item()
