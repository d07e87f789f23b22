"""GPU: the persistent decode kernel's quantized linears (qkv, o_proj, down_proj) at the input ranges real LLaMA layers produce, element by
element against the float64 product, with no rms floor.

The persistent kernel does not dequantise each weight to fp16: it feeds the raw nibbles to the tensor pipe as fp16 subnormals (n 2^-24, or
16 n 2^-24 for the odd nibbles of a packed word) and applies scale and zero once per group, s (sum x q - z sum x).  The staged x of the odd
nibbles is scaled down by 16 to match; this must not push small inputs into fp16 subnormals, where they would lose mantissa bits.  The
inputs of o_proj (attention outputs) and down_proj (SwiGLU outputs) are not RMSNorm outputs: they can sit far below 2^-10.  At the other end
a few residual features reach thousands ("massive activations") and down_proj inputs reach the hundreds.

Models.  LlamaDecoder built from packed fields (ops.pack_qweight / pack_qzeros) at LLaMA-7B int4 g128 (batch 1 and 8) and LLaMA-13B int3 g128
act-order (batch 1): the plain, batched and act-order instantiations, each asserted to run as one launch per step.  One step at position 0:
RoPE is the identity and attention over the one key returns v_new exactly, so
    qkv       the appended K and V rows are fp16 of the qkv output;
    o_proj    o-probe (gate / up / down scales 0, one layer): x after attention = fp16(x_in + fp16(o));
    down_proj MLP probe (o_proj scales 0, two layers): x leaving layer 0 = fp16(x_in + fp16(down(h))).
The embedding rows are 0 on the observation features (every fourth), so there x = fp16(out) exactly: large x_in features cannot mask an error.

Bound, per element:  |out - ref| <= ulp16(ref) + depth 2^-24 |x| . A + delta . |W|
    ref    float64 product of the operation's input and the exactly dequantised weight W = (q - z) s;
    A      (q + z) s: the kernel accumulates sum x q and z sum x separately in fp32, each rounding relative to its own magnitude (for the
           kernels that dequantise per weight |W| <= A, so the controls meet the same bound);
    depth  gpu_util.default_depth(K);
    delta  the error of an internal input: one fp16 ulp of the RMSNorm output (fp32 normalisation, one rounding); for h = silu(a) b the
           rounding of h plus the accumulation errors Ea, Eb of a and b (and their inputs' delta) carried through silu(a) b as in
           gpu_util.check_swiglu_fp64_bound.
Regimes: O(1) control, small attention outputs, small and tiny SwiGLU outputs, massive residual features, heavy tails with dead features,
all-positive o_proj inputs against zero points of 2^bits, quantizer extremes (zero fields 0 and 2^bits - 1, fp16-subnormal scales next to
scales near 1, whole groups at their zero).  Each regime asserts that it reaches the inputs it names.

Controls: the same fp16 inputs through ops.matmul248 on the int4 split-K matvec (which dequantises every weight to fp16, as the reference
does) meet the same bound, taken over its fp16-rounded weights.

down_proj's bound is loose (hundreds of ulps): its input h is internal, and the worst-case fp32 errors of gate and up carried through
silu(a) b dominate.  The bit-exact anchor is what pins down_proj at small inputs; qkv and o_proj are held within a few ulps.

Anchor: a single tap on an odd-nibble k whose input x = (1 + 2^-10) 2^-11 lies below 2^-10 and uses its last mantissa bit; every other input
of its group is 0 and every other weight sits at its zero.  qkv, o_proj and down_proj must each return fp16(x w) exactly.
"""
from functools import lru_cache

import pytest
import torch

from attn_probe import resid_buffers
from gpu_util import default_depth, report, ulp16

pytestmark = pytest.mark.gpu

GS = 128
VOCAB = 8
EPS = 1e-5
U24 = 2.0**-24
SHAPES = {'7b': (4096, 11008, 32), '13b': (5120, 13824, 40)}  # hidden, intermediate, heads
CONFIGS = [('7b', 4, False, 1), ('7b', 4, False, 8), ('13b', 3, True, 1)]  # (size, bits, act_order, batch)
REGIMES = ['control', 'small_attn', 'small_swiglu', 'tiny_swiglu', 'massive', 'heavy_tail', 'positive', 'extremes']
DEV = 'cuda:0'


def obs_mask(H):
    return torch.arange(H, device=DEV) % 4 == 3


class Lin:
    """Fields of one linear on the device: nibbles q [K, N], stored zeros zs [G, N] (the real zero is zs + 1), fp16 scales s [G, N], g_idx."""

    def __init__(self, q, zs, s, g_idx, bits):
        self.q, self.zs, self.s, self.g_idx, self.bits = q, zs, s, g_idx, bits

    @staticmethod
    def group_map(K, act_order, gen):
        g_idx = torch.arange(K, device=DEV) // GS
        return g_idx[torch.randperm(K, generator=gen, device=DEV)] if act_order else g_idx

    @staticmethod
    def random(K, N, bits, gen, g_idx, scale=(1e-3, 1.1e-2), zeros='rand', q_lo=0, extremes=False):
        top = (1 << bits) - 1
        G = K // GS
        q = torch.randint(q_lo, top + 1, (K, N), generator=gen, device=DEV, dtype=torch.int32)
        if zeros == 'rand':
            zs = torch.randint(0, top + 1, (G, N), generator=gen, device=DEV, dtype=torch.int32)
        else:
            zs = torch.full((G, N), zeros, device=DEV, dtype=torch.int32)
        s = torch.rand(G, N, generator=gen, device=DEV, dtype=torch.float64) * (scale[1] - scale[0]) + scale[0]
        if extremes:
            # zero fields 0 and 2^bits - 1 in alternate groups, scales fp16-subnormal (< 6.1e-5) or near 1 per (group, column), and a
            # quarter of the (group, column) blocks with zero field 0 entirely at their zero (q = 1)
            zs = torch.where(torch.arange(G, device=DEV)[:, None] % 2 == 0, 0, top).expand(G, N).to(torch.int32).contiguous()
            sub = torch.rand(G, N, generator=gen, device=DEV) < 0.5
            s = torch.where(sub, torch.rand(G, N, generator=gen, device=DEV, dtype=torch.float64) * 6e-5 + 1e-7,
                            torch.rand(G, N, generator=gen, device=DEV, dtype=torch.float64) * 0.5 + 0.5)
            dead = (torch.rand(G, N, generator=gen, device=DEV) < 0.25) & (zs == 0)
            q = torch.where(dead[g_idx], torch.ones_like(q), q)
        return Lin(q, zs, s.half(), g_idx, bits)

    @staticmethod
    def cat(parts):
        p0 = parts[0]
        return Lin(torch.cat([p.q for p in parts], 1), torch.cat([p.zs for p in parts], 1), torch.cat([p.s for p in parts], 1), p0.g_idx, p0.bits)

    def W(self):
        """float64 [K, N]: the exactly dequantised weight (q - z) s."""
        g = self.g_idx
        return (self.q.double() - (self.zs.double() + 1)[g]) * self.s.double()[g]

    def A(self):
        """float64 [K, N]: (q + z) s, the magnitudes the regrouped fp32 sums round relative to."""
        g = self.g_idx
        return (self.q.double() + (self.zs.double() + 1)[g]) * self.s.double()[g]

    def weights(self, zero_scales=False):
        from gptq_b200 import engine, ops
        qw = ops.pack_qweight(self.q, self.bits)
        qz = ops.pack_qzeros(self.zs, self.bits)
        s = torch.zeros_like(self.s) if zero_scales else self.s
        return engine.QLayerWeights(qw, s, qz, self.g_idx.to(torch.int32), self.bits, GS)


def uniform(gen, n, lo, hi):
    return torch.rand(n, generator=gen, device=DEV, dtype=torch.float64) * (hi - lo) + lo


def regime(name, size, bits, act, B, seed):
    """(x_in fp16 [B, H], input_norm, post_norm fp16 [H], {linear: Lin}) of a regime."""
    H, I, _ = SHAPES[size]
    gen = torch.Generator(device=DEV).manual_seed(seed)
    rnd = lambda *s: torch.randn(*s, generator=gen, device=DEV, dtype=torch.float64)
    x = rnd(B, H)
    in_norm, post_norm = uniform(gen, H, 0.9, 1.1), uniform(gen, H, 0.9, 1.1)
    sc = dict(qk=(1e-3, 1.1e-2), v=(1e-3, 1.1e-2), o=(1e-3, 1.1e-2), gate=(1e-3, 1.1e-2), up=(1e-3, 1.1e-2), down=(1e-3, 1.1e-2))
    kw = {k: {} for k in sc}
    if name == 'small_attn':  # v ~ 3e-4: small input norm weights and small v scales
        in_norm = uniform(gen, H, 0.009, 0.011)
        sc['v'] = (3e-5, 1e-4)
    elif name == 'small_swiglu':  # a, b ~ 0.02: median |h| ~ 1e-4
        post_norm = uniform(gen, H, 0.009, 0.011)
        sc['gate'] = sc['up'] = (2e-3, 6e-3)
    elif name == 'tiny_swiglu':  # a, b ~ 3e-3: median |h| ~ 3e-6
        post_norm = uniform(gen, H, 0.009, 0.011)
        sc['gate'] = sc['up'] = (4e-4, 1e-3)
    elif name == 'massive':  # four residual features at +-1e3 ... 4e3 with norm weights ~1e-3; gate / up large enough for h in the hundreds
        feats = torch.tensor([5, 1234, 2050, H - 7], device=DEV)  # not observation features (k % 4 != 3)
        x[:, feats] = torch.tensor([1e3, -2e3, 3e3, -4e3], device=DEV, dtype=torch.float64)
        in_norm[feats] = 1e-3
        post_norm[feats] = 1e-3
        sc['gate'] = sc['up'] = (2.0, 4.0)
    elif name == 'heavy_tail':
        x = x * torch.exp(2 * rnd(B, H))
        x[:, ::7] = 0
    elif name == 'positive':  # x_in, norm weights and v weights >= 0: all-positive o_proj inputs; o_proj zero fields 2^bits - 1
        x = x.abs()
        sc['v'] = (1e-4, 1.1e-3)
        kw['v'] = dict(zeros=0, q_lo=1)
        kw['o'] = dict(zeros=(1 << bits) - 1)
    elif name == 'extremes':
        in_norm = uniform(gen, H, 0.018, 0.022)
        for k in ('qk', 'v', 'o', 'down'):
            kw[k] = dict(extremes=True)
    x[:, obs_mask(H)] = 0
    x_in = x.half()
    assert torch.isfinite(x_in).all()
    g_qkv, g_o, g_mlp, g_down = (Lin.group_map(K, act, gen) for K in (H, H, H, I))  # gate and up share their input, hence their map
    lin = lambda K, N, key, g: Lin.random(K, N, bits, gen, g, scale=sc[key], **kw[key])
    L = dict(qkv=Lin.cat([lin(H, 2 * H, 'qk', g_qkv), lin(H, H, 'v', g_qkv)]), o=lin(H, H, 'o', g_o), gate=lin(H, I, 'gate', g_mlp),
             up=lin(H, I, 'up', g_mlp), down=lin(I, H, 'down', g_down))
    return x_in, in_norm.half(), post_norm.half(), L


def build(size, B, L, in_norm, post_norm, x_in, mode):
    """mode 'o': gate / up / down scales 0, one layer; 'mlp': o_proj scales 0, two layers.  Embedding row b = x_in[b]."""
    from gptq_b200 import engine
    H, I, nh = SHAPES[size]
    ly = {k: lin.weights(zero_scales=(mode == 'o' and k in ('gate', 'up', 'down')) or (mode == 'mlp' and k == 'o')) for k, lin in L.items()}
    ly['input_norm'], ly['post_norm'] = in_norm, post_norm
    embed = torch.zeros(VOCAB, H, dtype=torch.float16, device=DEV)
    embed[:B] = x_in
    lm_head = (torch.randn(VOCAB, H, generator=torch.Generator().manual_seed(5)) * 0.02).half().to(DEV)
    dec = engine.LlamaDecoder([ly] * (1 if mode == 'o' else 2), embed, torch.ones(H, dtype=torch.float16, device=DEV), lm_head, nh, rms_eps=EPS,
                              batch=B, max_seq=32)
    assert dec.launches_per_step() == 1, f'{size} batch {B}: {dec.launches_per_step()} launches per step (not the persistent kernel)'
    dec.set_input(list(range(B)), [0] * B)
    dec.step()
    torch.cuda.synchronize()
    return dec


def rmsnorm64(x, w):
    x = x.double()
    return x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + EPS) * w.double()


def ratio(out, ref, bound, cols=None):
    r = (out.double() - ref).abs() / bound
    return (r if cols is None else r[:, cols]).max().item()


def rounded(v, err):
    """The fp16 input a kernel forms from a value within err of v (float64), one rounding: (fp16(v) as float64, delta) with delta = 0
    where every value of [v - err, v + err] rounds to fp16(v), else ulp16(v) + err (the kernel may take the neighbouring fp16 value)."""
    v16 = fp16_of(v).double()
    straddle = fp16_of(v - err) != fp16_of(v + err)
    return v16, torch.where(straddle, ulp16(v) + err, torch.zeros_like(v))


NORM_ERR = 64 * U24  # relative error of the kernels' fp32 RMSNorm before its rounding: the sum of squares (a depth-37 fp32 sum), mean, sqrt,
                     # reciprocal and the two multiplies, with room to spare


class Reference:
    """float64 products, bounds and the inputs of each observed linear.  An internal input enters as its fp16 rounding plus delta
    (rounded()): one ulp plus the pre-rounding error where that error could move the rounding, 0 elsewhere."""

    def __init__(self, x_in, in_norm, post_norm, L):
        self.L = L
        xq64 = rmsnorm64(x_in, in_norm)
        self.xq, self.dq = rounded(xq64, NORM_ERR * xq64.abs())
        self.qkv, self.qkv_b = self.product(self.xq, L['qkv'], self.dq)
        xg64 = rmsnorm64(x_in, post_norm)  # MLP probe: x after attention is x_in (o_proj adds exactly 0)
        xg, dg = rounded(xg64, NORM_ERR * xg64.abs())
        a, Ea = self.product(xg, L['gate'], dg, err_only=True)
        b, Eb = self.product(xg, L['up'], dg, err_only=True)
        sa = a * torch.sigmoid(a)
        h64 = sa * b
        # before its rounding the kernels' h is within this of h64 (gpu_util.check_swiglu_fp64_bound: |silu'| <= 1.1, 8 fp32 roundings)
        self.h, self.dh = rounded(h64, 1.1 * Ea * (b.abs() + Eb) + sa.abs() * Eb + 8 * U24 * h64.abs())
        self.down, self.down_b = self.product(self.h, L['down'], self.dh)

    @staticmethod
    def product(x, lin, delta=None, err_only=False, per_weight=False):
        """(x . W, bound): ulp16(ref) + depth 2^-24 |x| . A + delta . |W| (err_only: without the fp16 rounding of the output).
        per_weight: W rounded to fp16 weight by weight and A = |W|, the arithmetic of the kernels that dequantise like the reference."""
        W = lin.W()
        if per_weight:
            W = fp16_of(W).double()
        ref = x @ W
        xa = x.abs() + (0 if delta is None else delta)
        err = default_depth(W.shape[0]) * U24 * (xa @ (W.abs() if per_weight else lin.A()))
        if delta is not None:
            err = err + delta @ W.abs()
        del W
        return ref, err if err_only else ulp16(ref) + err


@lru_cache(maxsize=1)
def case(size, bits, act, B, name):
    seed = 1000 * REGIMES.index(name) + 10 * B + bits + 100000 * int(size == '13b')
    x_in, in_norm, post_norm, L = regime(name, size, bits, act, B, seed)
    H = x_in.shape[1]
    R = Reference(x_in, in_norm, post_norm, L)
    dec = build(size, B, L, in_norm, post_norm, x_in, 'o')
    k = dec.k_cache[0, :B, :, 0].reshape(B, H)
    v = dec.v_cache[0, :B, :, 0].reshape(B, H)
    x_attn = resid_buffers(dec)[1]
    del dec
    dec = build(size, B, L, in_norm, post_norm, x_in, 'mlp')
    x_mlp = resid_buffers(dec)[0]
    del dec
    torch.cuda.empty_cache()
    return x_in, L, R, k, v, x_attn, x_mlp


def share_below(x, t=2.0**-10):
    x = x.double().abs()
    return float(((x < t) & (x > 0)).double().sum() / (x > 0).double().sum())


@pytest.mark.parametrize('name', REGIMES)
@pytest.mark.parametrize('size,bits,act,B', CONFIGS, ids=lambda v: str(v))
def test_linears_within_fp64_bound(size, bits, act, B, name):
    from gptq_b200 import ops
    x_in, L, R, k, v, x_attn, x_mlp = case(size, bits, act, B, name)
    H = x_in.shape[1]
    what = f'{size} int{bits} act={act} batch {B} [{name}]'
    obs = obs_mask(H)
    # the regime reaches the inputs it names
    sv, sh = share_below(v), share_below(R.h)
    med_v, med_h = v.double().abs().median().item(), R.h.abs().median().item()
    print(f'  {what}: median |v| {med_v:.3g} (share below 2^-10 {sv:.2f}), median |h| {med_h:.3g} (share {sh:.2f}), max |h| {R.h.abs().max().item():.3g}')
    if name == 'small_attn':
        assert sv > 0.9 and 1e-4 < med_v < 1e-3, (sv, med_v)
    if name in ('small_swiglu', 'tiny_swiglu'):
        lo, hi = (1e-5, 3e-4) if name == 'small_swiglu' else (2e-7, 1e-5)  # int3 weights (|q - z| <= 8) give the smaller h
        assert sh > 0.9 and lo < med_h < hi, (sh, med_h)
    if name == 'massive':
        assert x_in.double().abs().max().item() >= 4e3 - 2 and R.h.abs().max().item() > 100
    if name == 'positive':
        assert bool((v >= 0).all()) and bool((R.h.abs() > 0).any())
    worst = {}
    worst['qkv K'] = ratio(k, R.qkv[:, H:2 * H], R.qkv_b[:, H:2 * H])
    worst['qkv V'] = ratio(v, R.qkv[:, 2 * H:], R.qkv_b[:, 2 * H:])
    o64, o_b = R.product(v.double(), L['o'])
    worst['o_proj'] = ratio(x_attn, o64, o_b, obs)
    worst['down_proj'] = ratio(x_mlp, R.down, R.down_b, obs)
    # controls: the same fp16 inputs through ops.matmul248 on the int4 split-K matvec, which dequantises every weight to fp16 as the
    # reference does, held to the same bound over its own (fp16-rounded) weights: qkv from fp16 of the float64 RMSNorm output, o_proj
    # from the persistent kernel's own V rows, down_proj from fp16 of the float64 SwiGLU output
    for op, xc, lin in (('qkv', R.xq.half(), L['qkv']), ('o_proj', v.contiguous(), L['o']), ('down_proj', R.h.half(), L['down'])):
        if bits != 4 or act:
            break
        w = lin.weights()
        out = ops.matmul248(xc, w.qweight, w.scales, w.qzeros, w.g_idx, bits, groupsize=GS)
        ref, b = R.product(xc.double(), lin, per_weight=True)
        worst[f'{op} (matmul248 control)'] = ratio(out, ref, b)
    for op, r in worst.items():
        report(r, f'{what} {op}')


# ----------------------------------------------------------------------------- bit-exact anchor
X0 = (1 + 2.0**-10) * 2.0**-11  # below 2^-10, last mantissa bit set: x / 16 is an fp16 subnormal that cannot hold it


@pytest.mark.parametrize('B', [1, 8])
def test_odd_nibble_anchor_is_bit_exact(B):
    """Embedding rows +-2^-4 on a quarter of the features (the live ones), 0 elsewhere, rms_eps 0: RMSNorm gives exactly +-2 there.
    qkv: input norm weight X0 / 2 on feature KA (odd nibble; every row +2^-4 there) and 0 on the rest of its group, so x_KA = X0; every
    q / k column has one tap at KA with (q - z) 2^-j, j in [0, 4] -> K rows fp16(X0 (q - z) 2^-j); of the v columns only KO (odd) taps KA,
    with w = 1 -> v_KO = X0, every other v is 0.
    o_proj: every column one tap at KO (all other inputs of its group are 0).  MLP: gate column KD (odd) = 2 * 1 * 16 + 2 * 1 * 2^-6
    (two taps in two groups: a = 32 (1 + 2^-10), sigmoid exactly 1), up column KD = 2 * 1 * 2^-17 (a subnormal fp16 scale): h_KD =
    X0, every other gate / up column 0; down_proj: every column one tap at KD.  Observed on the non-live features."""
    from gptq_b200 import engine, ops
    H, I, nh = SHAPES['7b']
    KA, KO, KD, KG1, KG2, KU = 1001, 2049, 4097, 8, 264, 520  # KA, KO, KD odd; KG1, KG2, KU live features of different groups than KA
    gen = torch.Generator(device=DEV).manual_seed(11)
    live = torch.arange(H, device=DEV) % 4 == 0
    live[KA] = True
    live[KA - 1] = False  # keep the live count at H / 4
    assert int(live.sum()) == H // 4
    sign = torch.where(torch.rand(B, H, generator=gen, device=DEV) < 0.5, -1.0, 1.0)
    sign[:, [KA, KG1, KG2, KU]] = 1
    x_in = (sign * live * 2.0**-4).half()
    in_norm = torch.ones(H, device=DEV, dtype=torch.float64)
    grp = torch.arange(H, device=DEV) // GS
    in_norm[grp == KA // GS] = 0
    in_norm[KA] = X0 / 2

    def taps(K, N, k_of_n, d, j, zeros=7):
        """Lin with every weight at its zero (stored 7, z = 8) except (k_of_n[n], n): q - z = d[n], scale 2^-j[n] in the tap's group."""
        G = K // GS
        q = torch.full((K, N), zeros + 1, dtype=torch.int32, device=DEV)
        n = torch.arange(N, device=DEV)
        q[k_of_n, n] = (zeros + 1 + d).to(torch.int32)
        s = torch.ones(G, N, dtype=torch.float64, device=DEV)
        s[k_of_n // GS, n] = torch.pow(2.0, -j.double())
        return Lin(q, torch.full((G, N), zeros, dtype=torch.int32, device=DEV), s.half(), torch.arange(K, device=DEV) // GS, 4)

    def rand_d(N):
        d = torch.randint(1, 8, (N, ), generator=gen, device=DEV) * torch.where(torch.rand(N, generator=gen, device=DEV) < 0.5, -1, 1)
        return d, torch.randint(0, 5, (N, ), generator=gen, device=DEV)

    d, j = rand_d(3 * H)
    d[2 * H:], j[2 * H:] = 0, 0  # v: one column, KO, with w = 1: v_KO = X0 and 0 elsewhere
    d[2 * H + KO] = 1
    qkv = taps(H, 3 * H, torch.full((3 * H, ), KA, device=DEV), d, j)
    do, jo = rand_d(H)
    o = taps(H, H, torch.full((H, ), KO, device=DEV), do, jo)
    dd, jd = rand_d(H)
    down = taps(I, H, torch.full((H, ), KD, device=DEV), dd, jd)
    zero_col = lambda K, N: taps(K, N, torch.zeros(N, dtype=torch.long, device=DEV), torch.zeros(N, dtype=torch.long, device=DEV),
                                 torch.zeros(N, dtype=torch.long, device=DEV))
    gate, up = zero_col(H, I), zero_col(H, I)
    # gate column KD: taps 8 * 2 at KG1 (scale 2) and 1 * 2^-6 at KG2; up column KD: 1 * 2^-17 at KU
    gate.q[KG1, KD], gate.q[KG2, KD], up.q[KU, KD] = 9, 9, 9  # q - z = 1
    gate.s[KG1 // GS, KD], gate.s[KG2 // GS, KD], up.s[KU // GS, KD] = 16.0, 2.0**-6, 2.0**-17
    assert up.s[KU // GS, KD].double().item() == 2.0**-17
    L = dict(qkv=qkv, o=o, gate=gate, up=up, down=down)

    xq = torch.zeros(H, dtype=torch.float64, device=DEV)
    xq[KA] = X0
    want_kv = fp16_of((xq @ qkv.W())[None].expand(B, -1))
    want_o = fp16_of(X0 * o.W()[KO][None].expand(B, -1))
    want_d = fp16_of(X0 * down.W()[KD][None].expand(B, -1))
    nonlive = ~live
    bad = []
    for mode in ('o', 'mlp'):
        ly = {k: lin.weights(zero_scales=(mode == 'o' and k in ('gate', 'up', 'down')) or (mode == 'mlp' and k == 'o')) for k, lin in L.items()}
        ly['input_norm'], ly['post_norm'] = in_norm.half(), torch.ones(H, dtype=torch.float16, device=DEV)
        embed = torch.zeros(VOCAB, H, dtype=torch.float16, device=DEV)
        embed[:B] = x_in
        dec = engine.LlamaDecoder([ly] * (1 if mode == 'o' else 2), embed, torch.ones(H, dtype=torch.float16, device=DEV),
                                  torch.zeros(VOCAB, H, dtype=torch.float16, device=DEV), nh, rms_eps=0.0, batch=B, max_seq=32)
        assert dec.launches_per_step() == 1
        dec.set_input(list(range(B)), [0] * B)
        dec.step()
        torch.cuda.synchronize()
        if mode == 'o':
            got = {'K row': dec.k_cache[0, :B, :, 0].reshape(B, H), 'V row': dec.v_cache[0, :B, :, 0].reshape(B, H)}
            want = {'K row': want_kv[:, H:2 * H], 'V row': want_kv[:, 2 * H:]}
            got['o_proj'], want['o_proj'] = resid_buffers(dec)[1][:, nonlive], want_o[:, nonlive]
        else:
            got, want = {'down_proj': resid_buffers(dec)[0][:, nonlive]}, {'down_proj': want_d[:, nonlive]}
        for op in got:
            n_off = int((got[op].double() != want[op].double()).sum())
            print(f'  batch {B} {op}: {n_off} / {got[op].numel()} elements off the anchor')
            if n_off:
                i = int(torch.nonzero((got[op].double() != want[op].double()).reshape(-1))[0])
                bad.append(f'batch {B} {op}: {n_off} elements off; first {got[op].reshape(-1)[i].item()!r} vs {want[op].reshape(-1)[i].item()!r}')
        del dec
    assert not bad, '\n'.join(bad)


def fp16_of(v):
    """float64 -> fp16 rounded once, on the device."""
    from gpu_util import fp16_from_fp64
    return fp16_from_fp64(v).to(v.device)
