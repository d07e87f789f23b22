"""A one-layer probe model whose every quantized linear of the decode step has an output known bit for bit, at any groupsize, in both
engines (persistent kernel and kernel chain).  CPU-only: the GPU tests pack the fields with ops.pack_qweight / pack_qzeros.

* Inputs.  Embedding rows of +-2^-4 (+2^-4 on features [0, POS_FEATS)), rms_eps = 0, unit norm weights: both RMSNorms give exactly +-1.
* Fields.  Every (group, column) has its own zero z in [1, 2^bits - 2] and power-of-two scale 2^-j, and adjacent groups differ in both.
  A weight either sits at its own group's zero (it adds exactly 0 -- with the right group only) or is a tap, q != z.
    qkv   q and k columns dense (every weight a tap), j in [6, 10]; v columns one tap each, j in [5, 7] (|v| <= 15/32, a multiple of 2^-7)
    o     dense, j in [6, 8]
    gate  one tap per column on a feature k < POS_FEATS (x_k = +1), q = 2^bits - 1 and the tap group's scale 2^e chosen so that
          a = (q - z) 2^e lies in [20, 40)
    up    one tap per column, j in [5, 7] (|b| <= 15/32, a multiple of 2^-7)
    down  taps with density 1/16, j in [7, 8]
* SwiGLU made exact.  The kernels compute h = fp16((a * (1 / (1 + expf(-a)))) * b) (common.cuh swiglu).  At a >= 20, expf(-a) < 2.1e-9 is
  below half an ulp of 1 in fp32 (2^-24 = 6e-8), so the sigmoid is exactly 1 and h = fp16(a * b), a * b being exact in fp32 (an even
  integer below 2^6 times a multiple of 2^-7 below 1).
* Every sum is exact in fp32 (check_exact): with the input on a grid gx and scales >= s_min, each partial sum a kernel can form -- a
  stage's raw accumulator sum x_k q_k (<= 128 k, the units of 2^-24 and the 1/16 pre-scaling of the odd nibbles' x only shift the grid),
  the group sum of x, s (acc - z sum x) and any subset of those over the stages and split-K partials -- is a multiple of gx * s_min
  (gx for the raw sums) of magnitude below 2^24 of those units.  So out = fp16(exact float64 sum), in any summation order.

Where each linear is read after one step at position 0 (RoPE is the identity there and attention over the one key returns v_new):
    qkv              the appended K and V rows of the cache (exact(...).k / .v)
    o_proj           x after attention = fp16(x_in + fp16(o(v_new))), with gate/up/down scales 0 (the MLP adds exactly 0)
    gate/up -> down  x after the layer = fp16(x_in + fp16(down(h))), with o_proj scales 0 (x after attention is x_in)
"""
import math

import torch

from gpu_util import fp16_from_fp64
from oracle import gptq_oracle as O

# hidden, intermediate, heads (engine.LLAMA_SHAPES)
SHAPES = {'7b': (4096, 11008, 32), '13b': (5120, 13824, 40), '33b': (6656, 17920, 52), '65b': (8192, 22016, 64)}
POS_FEATS = 64  # every embedding row is +2^-4 on these features: the gate taps read x = +1
STAGE_K = 128   # k per stage of the persistent kernel (4 k-steps of 32), inside one group
STEP_K = 32
UNITS = 2**24   # fp32 holds every integer below this exactly


def _distinct_adjacent(v, lo, hi):
    """v [G, N] in [lo, hi] (hi > lo): entries equal to the previous group's are moved up by one (wrapping), so adjacent groups differ."""
    for g in range(1, v.shape[0]):
        row, same = v[g], v[g] == v[g - 1]
        row[same] = torch.where(row[same] == hi, torch.full_like(row[same], lo), row[same] + 1)
    return v


class Linear:
    """Fields of one probe linear: nibbles q [K, N], zeros z [G, N] (the real zero, stored zero + 1), scale exponents j [G, N]
    (scale 2^-j), g_idx [K] (int64) and the groupsize."""

    def __init__(self, q, z, j, g_idx, gs, bits):
        self.q, self.z, self.j, self.g_idx, self.gs, self.bits = q, z, j, g_idx, gs, bits
        self.K, self.N = q.shape

    @staticmethod
    def random(K, N, gs, bits, gen, jlo, jhi, g_idx, density=1.0, tap_ks=None):
        """Every weight at its group's zero except the taps: a random fraction `density`, or one per column at k = tap_ks[n]."""
        G = -(-K // gs)
        top = (1 << bits) - 1
        z = _distinct_adjacent(torch.randint(1, top, (G, N), generator=gen, dtype=torch.int16), 1, top - 1)
        j = _distinct_adjacent(torch.randint(jlo, jhi + 1, (G, N), generator=gen, dtype=torch.int16), jlo, jhi)
        own = z[g_idx]
        if tap_ks is None:
            tap = torch.rand(K, N, generator=gen) < density
        else:
            tap = torch.zeros(K, N, dtype=torch.bool)
            tap[tap_ks, torch.arange(N)] = True
        off = torch.randint(1, top + 1, (K, N), generator=gen, dtype=torch.int16)
        q = torch.where(tap, (own + off) % (top + 1), own)
        return Linear(q, z, j, g_idx, gs, bits)

    @staticmethod
    def cat(parts):
        """Column-wise concatenation of linears over the same g_idx."""
        p0 = parts[0]
        return Linear(torch.cat([p.q for p in parts], 1), torch.cat([p.z for p in parts], 1), torch.cat([p.j for p in parts], 1), p0.g_idx, p0.gs, p0.bits)

    def scales(self):
        return torch.pow(2.0, -self.j.double())

    def weight(self, cols=slice(None), device='cpu'):
        """float64 [K, n] (q - z) 2^-j of the columns `cols`."""
        g = self.g_idx.to(device)
        q = self.q[:, cols].to(device).double()
        z, s = self.z[:, cols].to(device).double(), self.scales()[:, cols].to(device)
        return (q - z[g]) * s[g]

    def taps_abs(self, device='cpu'):
        """float64 [K, N] |q - z| 2^-j: the magnitudes the exactness bounds sum."""
        return self.weight(device=device).abs()

    def stage_rows(self, g, n=STAGE_K):
        """The input rows of the first stage of group g in the kernels' (regrouped) order: its first min(n, group size) rows."""
        return torch.nonzero(self.g_idx == g).flatten()[:n]

    def packed(self, device):
        """(qweight, scales fp16, qzeros, g_idx int32) on `device`, packed by the project's own device packers."""
        from gptq_b200 import ops
        qw = ops.pack_qweight(self.q.to(device, torch.int32), self.bits)
        qz = ops.pack_qzeros((self.z - 1).to(device, torch.int32), self.bits)
        return qw, self.scales().half().to(device), qz, self.g_idx.to(device, torch.int32)


def group_size(gs, K):
    return K if gs == 'full' else gs


class ProbeLayer:
    """The probe's fields for one model size and groupsize (gs: an int or 'full' = each linear's K, the reference's --groupsize -1)."""

    def __init__(self, size, gs, bits=4, act_order=False, seed=0):
        H, I, nh = SHAPES[size]
        self.size, self.H, self.I, self.nh, self.bits, self.act_order = size, H, I, nh, bits, act_order
        self.gs = gs
        gen = torch.Generator().manual_seed(seed)
        gh, gi = group_size(gs, H), group_size(gs, I)
        g_h = O.make_g_idx(H, gh, act_order, gen).long()
        self.qkv = Linear.cat([Linear.random(H, 2 * H, gh, bits, gen, 6, 10, g_h),
                               Linear.random(H, H, gh, bits, gen, 5, 7, g_h, tap_ks=torch.randint(0, H, (H, ), generator=gen))])
        self.o = Linear.random(H, H, gh, bits, gen, 6, 8, O.make_g_idx(H, gh, act_order, gen).long())
        g_mlp = O.make_g_idx(H, gh, act_order, gen).long()  # gate and up share their input, hence their act-order map
        self.gate = Linear.random(H, I, gh, bits, gen, 5, 7, g_mlp, tap_ks=torch.randint(0, POS_FEATS, (I, ), generator=gen))
        top = (1 << bits) - 1
        ks = torch.nonzero(self.gate.q != self.gate.z[g_mlp]).t()  # the single tap of every column: (k, n), n ascending
        ks = ks[:, torch.argsort(ks[1])]
        self.gate.q[ks[0], ks[1]] = top
        d = (top - self.gate.z[g_mlp[ks[0]], ks[1]]).double()
        self.gate.j[g_mlp[ks[0]], ks[1]] = (-torch.ceil(torch.log2(20.0 / d))).to(torch.int16)
        self.up = Linear.random(H, I, gh, bits, gen, 5, 7, g_mlp.clone(), tap_ks=torch.randint(0, H, (I, ), generator=gen))
        self.down = Linear.random(I, H, gi, bits, gen, 7, 8, O.make_g_idx(I, gi, act_order, gen).long(), density=1 / 16)

    def linears(self):
        return dict(qkv=self.qkv, o=self.o, gate=self.gate, up=self.up, down=self.down)


def embed_rows(vocab, H, seed=0):
    """fp16 [vocab, H] of +-2^-4, +2^-4 on the first POS_FEATS features."""
    sign = 1 - 2 * torch.randint(0, 2, (vocab, H), generator=torch.Generator().manual_seed(seed + 1))
    sign[:, :POS_FEATS] = 1
    return (sign * 2.0**-4).half()


def fp16(v):
    """gpu_util.fp16_from_fp64 (float64 -> fp16 rounded once), kept on v's device."""
    return fp16_from_fp64(v).to(v.device)


def product(x, lin, device, cols=4096):
    """float64 x [B, K] @ lin.weight(), built column block by column block (a 65B qkv weight is 1.6 GB in float64)."""
    return torch.cat([x @ lin.weight(slice(c, c + cols), device=device) for c in range(0, lin.N, cols)], 1)


class Expect:
    """The exact outputs of one step at position 0 for input rows x_in [B, H] (fp16 embedding rows), all float64 / fp16 on `device`."""

    def __init__(self, layer, x_in, device='cpu'):
        L = layer
        self.x_in = x_in.to(device)
        self.x = self.x_in.double() * 16  # RMSNorm output, exactly +-1
        H = L.H
        self.qkv64 = product(self.x, L.qkv, device)
        self.k, self.v = fp16(self.qkv64[:, H:2 * H]), fp16(self.qkv64[:, 2 * H:])
        self.o64 = product(self.v.double(), L.o, device)
        self.x_attn = fp16(self.x_in.double() + fp16(self.o64).double())  # o-probe: MLP scales 0
        self.a = product(self.x, L.gate, device)
        self.b = product(self.x, L.up, device)
        self.h = fp16(self.a * self.b)  # sigmoid(a) == 1 in fp32 (module docstring)
        self.d64 = product(self.h.double(), L.down, device)
        self.x_mlp = fp16(self.x_in.double() + fp16(self.d64).double())  # mlp-probe: o_proj scales 0


# ----------------------------------------------------------------------------- exactness under the kernels' arithmetic
def input_bounds(L):
    """{linear: (xmax [K] float64, grid gx)}: the largest |input| per feature over every token and the grid the inputs lie on."""
    H = L.H
    one = torch.ones(H, dtype=torch.float64)
    vtap = L.qkv.taps_abs()[:, 2 * H:].max(0).values  # |v_n| <= its single tap's |q - z| 2^-j, on the grid 2^-7
    gate_a = L.gate.weight().max(0).values  # the gate's one tap: a_n for x = +1
    up_b = L.up.taps_abs().max(0).values
    # h = fp16(a b): a is even, b a multiple of 2^-7, and the fp16 rounding moves |h| up by at most 2^-11 relative
    return dict(qkv=(one, 1.0), o=(vtap, 2.0**-7), gate=(one, 1.0), up=(one, 1.0), down=(gate_a * up_b * (1 + 2.0**-11), 2.0 * 2.0**-7))


def check_exact(L):
    """For every linear: (worst total ratio, worst stage ratio) -- the largest partial sum in units of its grid, over 2^24.
    total = max_n sum_k xmax_k |q - z| s / (gx s_min): bounds the group epilogue, tot, and every split-K partial and their sum;
    stage = STAGE_K max(xmax) (2^bits - 1) / gx: bounds a stage's raw accumulator sum x_k q_k and z sum x_k."""
    out = {}
    bounds = input_bounds(L)
    for name, lin in L.linears().items():
        xmax, gx = bounds[name]
        assert gx / 16 >= 2.0**-24, f'{name}: the odd nibbles\' x / 16 falls below fp16 subnormals'
        smin = lin.scales().min().item()
        total = (xmax @ lin.taps_abs()).max().item() / (gx * smin) / UNITS
        stage = STAGE_K * xmax.max().item() * ((1 << lin.bits) - 1) / gx / UNITS
        out[name] = (total, stage)
    return out


# ----------------------------------------------------------------------------- what a wrong kernel would produce
def corruptions(lin, X, B_other=True):
    """{name: out'} float64 [B, N] for the input X [B, K] float64: the product the kernel would produce with one stage (in group
    min(8, G - 1), or in the last group when that one is partial) reading the neighbouring group's scale / zero, sequence 1 using sequence
    0's sum of x in that stage (B >= 2), or the first k-step of that stage dropped / repeated."""
    W = lin.weight()
    out = X @ W
    G = lin.z.shape[0]
    res = {}
    g = G - 1 if lin.K % lin.gs else min(8, G - 1)
    S = lin.stage_rows(g, n=lin.gs)
    S = S[256:256 + STAGE_K] if S.numel() >= 256 + STAGE_K else S[:STAGE_K]  # past the features every embedding row shares
    T = S[:STEP_K]
    q, z, s = lin.q.double(), lin.z.double(), lin.scales()
    if G > 1:
        gn = g - 1
        res['neighbour scale'] = out + X[:, S] @ ((q[S] - z[g]) * (s[gn] - s[g]))
        res['neighbour zero'] = out + X[:, S].sum(1, keepdim=True) * ((z[g] - z[gn]) * s[g])[None, :]
    if B_other and X.shape[0] > 1:
        o2 = out.clone()
        o2[1] -= (X[0, S].sum() - X[1, S].sum()) * z[g] * s[g]
        res['other sequence sum of x'] = o2
    res['dropped k-step'] = out - X[:, T] @ W[T]
    res['repeated k-step'] = out + X[:, T] @ W[T]
    return out, res


def teeth(L, x_in, cols=1024):
    """{(linear, corruption): (elements that differ, elements observed)} where each linear is observed (module docstring), over its
    first `cols` output columns (the K rows of qkv)."""
    H = L.H
    E = Expect(L, x_in)
    X1 = E.x
    res = {}
    # K row of qkv: fp16 of the k columns
    kl = Linear(L.qkv.q[:, H:H + cols], L.qkv.z[:, H:H + cols], L.qkv.j[:, H:H + cols], L.qkv.g_idx, L.qkv.gs, L.bits)
    out, bad = corruptions(kl, X1)
    for name, o2 in bad.items():
        res[('qkv', name)] = (int((fp16(o2) != fp16(out)).sum()), out.numel())
    # o_proj: through the residual add
    ol = Linear(L.o.q[:, :cols], L.o.z[:, :cols], L.o.j[:, :cols], L.o.g_idx, L.o.gs, L.bits)
    xin = E.x_in.double()[:, :cols]
    obs = lambda o: fp16(xin + fp16(o).double())
    out, bad = corruptions(ol, E.v.double())
    for name, o2 in bad.items():
        res[('o', name)] = (int((obs(o2) != obs(out)).sum()), out.numel())
    dl = Linear(L.down.q[:, :cols], L.down.z[:, :cols], L.down.j[:, :cols], L.down.g_idx, L.down.gs, L.bits)
    out, bad = corruptions(dl, E.h.double())
    for name, o2 in bad.items():
        res[('down', name)] = (int((obs(o2) != obs(out)).sum()), out.numel())
    return res


# (size, gs, bits, act_order, batch, engine): the GPU cases of tests/test_gpu_decode_groupsize.py.  batch 'max' is the largest batch the
# persistent plan takes at that shape, 'max+1' one sequence more (the kernel chain); both depend on the device (max_persistent_batch).
CASES = [('7b', gs, 4, False, B, 'persistent') for gs in (32, 64, 128, 1024, 'full') for B in (1, 8)]
CASES += [('13b', 32, 3, True, 1, 'persistent'), ('13b', 32, 4, False, 7, 'chain'), ('13b', 'full', 4, False, 7, 'chain')]
# 65B: hidden 8192 (the persistent kernel's limit), one lm_head row per stage; gs 1024 ends down_proj (K = 22016) in a partial group of 512.
# 33B at gs 1024: every linear ends in a partial group of 512 (6656 = 6 x 1024 + 512, 17920 = 17 x 1024 + 512).
CASES += [('65b', 128, 4, False, 1, 'persistent'), ('65b', 128, 4, False, 'max', 'persistent'), ('65b', 128, 4, False, 'max+1', 'chain'),
          ('65b', 1024, 4, False, 1, 'persistent'), ('65b', 128, 4, True, 1, 'persistent'),
          ('33b', 1024, 4, False, 1, 'persistent'), ('33b', 1024, 4, False, 'max', 'persistent'), ('33b', 'full', 4, False, 'max+1', 'chain')]
VOCAB = 64


def max_persistent_batch(n_heads, sms):
    """The largest batch the persistent plan takes: one attention team per (sequence, head) pair, 2 teams per SM (mega_plan), at most 8."""
    return min(8, 2 * sms // n_heads)


def resolve_batch(B, n_heads, sms):
    """A case's batch on a device with `sms` SMs (CASES)."""
    if B == 'max':
        return max_persistent_batch(n_heads, sms)
    if B == 'max+1':
        b = max_persistent_batch(n_heads, sms)
        assert b < 8, f'{n_heads} heads: every batch fits the persistent plan on {sms} SMs'
        return b + 1
    return B


def tokens(B):
    return [(7 * b + 3) % VOCAB for b in range(B)]


def layer_for(size, gs, bits, act_order):
    """The probe layer of a case (a fixed seed per configuration, so the CPU and GPU tests see the same fields)."""
    seed = {'7b': 1, '13b': 2, '33b': 3, '65b': 4}[size] * 100000 + (0 if gs == 'full' else gs) * 10 + bits + 5 * int(act_order)
    return ProbeLayer(size, gs, bits, act_order, seed)
