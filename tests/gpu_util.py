"""Helpers shared by the GPU tests."""
import math
import time

import numpy as np
import pytest
import torch

from oracle import gptq_oracle as O

REL_TOL = 1e-3  # north_star: outputs within 1e-3 relative of the reference's dequant->fp16 matmul


def assert_rel_close(out: torch.Tensor, ref: torch.Tensor, rel: float = REL_TOL, what: str = ''):
    """|out - ref| <= rel * max(|ref|, rms(ref)) element-wise; prints the worst |err| / bound (visible under -s).

    fp16 results that differ only by the fp32 summation order sit within one fp16 ulp (<= 9.8e-4 relative);
    the rms floor covers outputs that cancel to ~0, where a relative bound is meaningless."""
    out32, ref32 = out.detach().float().cpu(), ref.detach().float().cpu()
    assert out32.shape == ref32.shape, (out32.shape, ref32.shape)
    assert torch.isfinite(out32).all(), f'{what}: non-finite output'
    rms = ref32.pow(2).mean().sqrt().item()
    bound = rel * torch.maximum(ref32.abs(), torch.full_like(ref32, rms)) + 1e-7
    err = (out32 - ref32).abs()
    print(f'  {what}: worst |err| / bound = {(err / bound).max().item():.3g} (bound {rel:g})')
    bad = err > bound
    assert not bad.any(), f'{what}: {int(bad.sum())} / {bad.numel()} elements off; max err {err.max().item():.3e}, rms(ref) {rms:.3e}'


def cuda(*ts):
    return tuple(t.cuda() if t is not None else None for t in ts)


@pytest.fixture(scope='module')
def ops():
    from gptq_b200 import ops as _ops  # raises if libgptq_b200.so is missing: no fallback
    return _ops


# ----------------------------------------------------------------------------- which kernel ran
MATVEC, MATVEC_DUAL = 'qmatvec_int4_kernel<false>', 'qmatvec_int4_kernel<true>'
GEMM_1, GEMM_2, GEMM_DUAL = 'qgemm_wgmma_kernel<false, 1, 6>', 'qgemm_wgmma_kernel<false, 2, 4>', 'qgemm_wgmma_kernel<true, 1, 4>'
GENERIC_4 = 'qlinear_generic_kernel<4, 4, false>'


def generic(bits, M, dual=False):
    return f'qlinear_generic_kernel<{bits}, {M if M <= 2 else 4}, {str(dual).lower()}>'


def generic_t(bits):
    return f'qlinear_transpose_generic_kernel<{bits}, 2>'


def launched_kernels(fn):
    """Run fn() under torch.profiler (launch and kernel activity records, no hardware counters) -> (fn's result, set of names
    of the device-side events).

    Names are the demangled ones, e.g. 'void gptq::(anonymous namespace)::qmatvec_int4_kernel<false>(...)'.  The traced window
    is padded by a few milliseconds on both sides, so that device activity at either end of it is not cut off."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        time.sleep(0.003)
        res = fn()
        torch.cuda.synchronize()
        time.sleep(0.003)
    events = prof.events()
    return res, {e.name for e in events if e.device_type == torch.autograd.DeviceType.CUDA}


def run_kernel(fn, kernel: str, what: str = ''):
    """fn() must launch `kernel` (a demangled name with its template arguments, e.g. 'qgemm_wgmma_kernel<false, 2, 4>') and no
    other quantized-linear kernel.  Returns fn's result.

    fn must be repeatable: a trace without any kernel record (the launch call was traced, the kernel was not; seen on an H100
    about once in 200 sessions) is taken again, up to three times.  A machine whose activity tracing returns no CUDA events at
    all skips the test: a routing assertion that cannot see kernels must not pass."""
    strip = lambda s: s.replace(' ', '')
    families = ('qmatvec_int4_kernel', 'qgemm_wgmma_kernel', 'qlinear_generic_kernel', 'qlinear_transpose_generic_kernel')
    for _ in range(3):
        res, names = launched_kernels(fn)
        if names:
            break
    if not names:
        pytest.skip(f'{what}: CUDA activity tracing returned no kernel events on this machine')
    qk = sorted(n for n in names if any(f + '<' in n for f in families))
    hit = [n for n in qk if strip(kernel) in strip(n)]
    assert hit and len(hit) == len(qk), f'{what}: expected {kernel}, launched {sorted(names)}'
    return res


# ----------------------------------------------------------------------------- fp64 reference with an element-wise bound
def ulp16(v: torch.Tensor) -> torch.Tensor:
    """Spacing of fp16 numbers at |v| (2^-24 in the subnormal range); v in float64."""
    e = torch.floor(torch.log2(v.abs().clamp_min(2.0**-14)))
    return torch.pow(2.0, e - 10)


def fp32_sum_bound(A: torch.Tensor, depth: float) -> torch.Tensor:
    """Worst-case error of an fp32 sum of exact products whose absolute values sum to A, accumulated `depth` additions deep
    (round to nearest, 2^-24 relative per addition)."""
    return depth * 2.0**-24 * A


def default_depth(K: int) -> float:
    """Accumulation depth of the tensor-core kernels: K/16 sequential k16 mma / wgmma steps, plus 64 for the inside of an mma
    and the split-K partial reduction of the matvec."""
    return K / 16 + 64


def report(ratio: float, what: str, limit: float = 1.0):
    """Print the worst |err| / bound (visible under -s) and fail above `limit`."""
    print(f'  {what}: worst |err| / bound = {ratio:.3g}')
    assert ratio <= limit, f'{what}: worst |err| / bound = {ratio:.3g}'


def _where(bad: torch.Tensor, locate) -> str:
    idx = [int(i) for i in torch.nonzero(bad)[0]]
    return locate(*idx) if locate is not None else f'first bad index {tuple(idx)}'


def check_fp64_bound(out, x, W, bias=None, what='', depth=None, locate=None) -> float:
    """out[M, N] (fp16, device) against the fp64 product of the fp16 x [M, K] and the oracle's fp16 weight W [K, N] (+ bias):

        |out - ref| <= ulp16(max(|x.W|, |ref|)) + depth * 2^-24 * (|x| . |W|)

    The first term covers the fp16 store of the accumulator and the fp16 bias add after it (hence the larger of the two
    magnitudes: a bias can cancel the product); the second bounds the fp32 accumulation (default_depth).  Returns the worst
    |err| / bound and fails, naming the first offending element (locate(m, n) -> str), if it exceeds 1."""
    x64, W64 = x.to('cuda', torch.float64), W.to('cuda', torch.float64)
    acc = x64 @ W64
    A = x64.abs() @ W64.abs()
    ref = acc if bias is None else acc + bias.to('cuda', torch.float64)
    bound = ulp16(torch.maximum(acc.abs(), ref.abs())) + fp32_sum_bound(A, default_depth(W.shape[0]) if depth is None else depth)
    out64 = out.to(torch.float64)
    assert torch.isfinite(out64).all(), f'{what}: non-finite output'
    ratio_t = (out64 - ref).abs() / bound
    ratio = ratio_t.max().item()
    if ratio > 1:
        what = f'{what}: {_where(ratio_t > 1, locate)}'
    report(ratio, what)
    return ratio


def check_swiglu_fp64_bound(out, x, Wg, Wu, what='', depth=None, locate=None) -> float:
    """out = fp16(silu(x.Wg) * (x.Wu)) against fp64: the accumulation bounds Ea, Eb of both products (check_fp64_bound) carried
    through silu(a) * b (|silu'| <= 1.1), plus 8 fp32 roundings of the epilogue and the fp16 store."""
    x64 = x.to('cuda', torch.float64)
    Wg64, Wu64 = Wg.to('cuda', torch.float64), Wu.to('cuda', torch.float64)
    a, b = x64 @ Wg64, x64 @ Wu64
    d = default_depth(Wg.shape[0]) if depth is None else depth
    Ea, Eb = fp32_sum_bound(x64.abs() @ Wg64.abs(), d), fp32_sum_bound(x64.abs() @ Wu64.abs(), d)
    sa = a * torch.sigmoid(a)
    ref = sa * b
    bound = ulp16(ref) + 1.1 * Ea * (b.abs() + Eb) + sa.abs() * Eb + 8 * 2.0**-24 * ref.abs()
    out64 = out.to(torch.float64)
    assert torch.isfinite(out64).all(), f'{what}: non-finite output'
    ratio_t = (out64 - ref).abs() / bound
    ratio = ratio_t.max().item()
    if ratio > 1:
        what = f'{what}: {_where(ratio_t > 1, locate)}'
    report(ratio, what)
    return ratio


# ----------------------------------------------------------------------------- bit-level comparisons
def fp16_ulp_distance(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """Number of fp16 values between a and b (both fp16; +0 and -0 are the same point)."""
    def ordered(t):
        u = t.contiguous().view(torch.int16).to(torch.int32) & 0xFFFF
        return torch.where(u >= 0x8000, 0x8000 - u, u)
    return (ordered(a) - ordered(b)).abs()


def fp16_from_fp64(v: torch.Tensor) -> torch.Tensor:
    """float64 -> fp16 rounded once (numpy converts directly; a float64 -> float32 -> fp16 cast can round twice)."""
    return torch.from_numpy(v.detach().cpu().numpy().astype(np.float16))


def assert_equal(out, exp, what, locate):
    """torch.equal, naming the first mismatching element through locate(row, col)."""
    assert out.shape == exp.shape, (what, out.shape, exp.shape)
    if torch.equal(out, exp):
        return
    bad = out != exp
    r, c = (int(i) for i in torch.nonzero(bad)[0])
    raise AssertionError(f'{what}: {int(bad.sum())} / {bad.numel()} outputs differ; first at {locate(r, c)}: got {out[r, c].item()!r}, '
                         f'want {exp[r, c].item()!r}')


class WorstRatios(dict):
    """sweep -> worst |err| / bound of a test module; a module-scoped fixture prints summary() at its end (pytest -s)."""

    def note(self, sweep, ratio):
        self[sweep] = max(self.get(sweep, 0.0), ratio)
        return ratio

    def summary(self):
        for sweep, r in self.items():
            print(f'worst |err| / bound, {sweep}: {r:.3g}')


# ----------------------------------------------------------------------------- layers and inputs
class Layer:
    """A packed layer on the CPU and on the device, the oracle's fp16 weight W [K, N] (O.dequant, built on the CPU) on the device, the
    bias on the device, and the groupsize hint the kernels get: gs for a trivial g_idx, 0 (the g_idx gather) for act-order."""

    def __init__(self, packed, bits, gs=None, act=False, bias=None):
        self.cpu = tuple(packed)
        self.dev = tuple(t.cuda() for t in packed)
        self.bits, self.gs, self.act = bits, gs, act
        self.hint = 0 if act else gs
        self.W = O.dequant(*packed, bits).cuda()
        self.bias = bias.cuda() if bias is not None else None

    @property
    def K(self):
        return self.W.shape[0]

    @classmethod
    def random(cls, K, N, bits, gs, act=False, bias=False, seed=0):
        qw, s, qz, g, b = O.random_packed(K, N, bits, gs, act_order=act, seed=seed, bias=bias)
        return cls((qw, s, qz, g), bits, gs, act, b)


def cyclic(ks, M):
    """ks padded (cyclically) to a multiple of M."""
    ks = list(ks)
    return ks + ks[:(-len(ks)) % M]


def randn_x(M, K, seed, ld=None):
    """fp16 [M, K] ~ N(0, 1) on the device; with ld, a column slice of an [M, ld] buffer (row stride ld)."""
    buf = torch.randn(M, ld or K, generator=torch.Generator().manual_seed(seed)).half().cuda()
    return buf[:, :K]


class recorded_transposes:
    """Records every ops.transpose_matmul248 request made inside the block (QuantLinearFunction.backward issues them from the autograd
    worker thread); check() holds each to the form the wgmma kernel takes: int4 with a positive groupsize hint, more than 8 rows."""

    def __enter__(self):
        from gptq_b200 import ops as _ops
        self.ops, self.shipped, self.calls = _ops, _ops.transpose_matmul248, []

        def record(*args, **kw):
            self.calls.append((args, kw))
            return self.shipped(*args, **kw)

        _ops.transpose_matmul248 = record
        return self

    def __exit__(self, *exc):
        self.ops.transpose_matmul248 = self.shipped

    def check(self, what, at_least=1):
        assert len(self.calls) >= at_least, f'{what}: {len(self.calls)} transposed requests, expected at least {at_least}'
        for args, kw in self.calls:
            assert args[5] == 4 and kw.get('groupsize', 0) % 32 == 0 and kw.get('groupsize', 0) > 0 and args[0].shape[0] > 8, \
                f'{what}: backward request with bits={args[5]}, hint={kw.get("groupsize")}, M={args[0].shape[0]}'


# ----------------------------------------------------------------------------- quantized HF modules
def fill_quant_linear(ql, bits, seed, act=False):
    """Random packed fields (O.random_packed) into a QuantLinear, and a random bias where it has one."""
    qw, s, qz, g, b = O.random_packed(ql.infeatures, ql.outfeatures, bits, ql.groupsize, act_order=act, seed=seed, bias=ql.bias is not None)
    ql.qweight, ql.scales, ql.qzeros, ql.g_idx = qw, s, qz, g
    if b is not None:
        ql.bias = b


def tiny_quant_llama(bits=4, gs=32, act=False, hidden=128, intermediate=352, heads=4, rope_theta=10000.0, rms_norm_eps=1e-6):
    """A two-layer HF LLaMA with every linear but lm_head replaced by a randomly filled QuantLinear (quant.make_quant_linear)."""
    import quant
    import utils
    from transformers import LlamaConfig, LlamaForCausalLM
    cfg = LlamaConfig(hidden_size=hidden, intermediate_size=intermediate, num_hidden_layers=2, num_attention_heads=heads, num_key_value_heads=heads,
                      vocab_size=256, max_position_embeddings=128, rope_theta=rope_theta, rms_norm_eps=rms_norm_eps)
    torch.manual_seed(0)
    model = LlamaForCausalLM(cfg).half().eval()
    layers = utils.find_layers(model)
    layers.pop('lm_head')
    quant.make_quant_linear(model, layers, bits, gs)
    seed = 0
    for name, m in model.named_modules():
        if isinstance(m, quant.QuantLinear):
            seed += 1
            # q/k/v of one block share their input, hence their act-order
            fill_quant_linear(m, bits, seed, act=False)
            if act:
                blk = name.split('.')[2]
                m.g_idx = O.make_g_idx(m.infeatures, gs, True, torch.Generator().manual_seed(int(blk) + m.infeatures))
    return model


# ----------------------------------------------------------------------------- lm_head + log-softmax (gptq_lm_head_logprob)
U = 2.0**-24
# fp32 part of the bound (everything after the fp16 logits).  The row's sum s = sum exp(l - max) is formed by 31 sequential adds per
# thread, 2 quad shuffles, ceil(ntiles / 32) per-lane merges of the ntiles = ceil(V / 128) vocabulary tiles and 5 butterfly merges, each
# merge 2 expf (2 ulp), 2 multiplies and 1 add; with 2 ulp for the terms' expf that is 31 + 2 + (merges + 5) * 6 + 2 roundings of relative
# size 2^-24: 113 at V = 32000 (8 merges), 257 at LLaMA-3's 128256 (1002 tiles, 32 merges), so |log s' - log s| <= max(128, that) 2^-24.
# The exp arguments l - max are rounded relative to their size; weighted by exp(-a) that adds at most (log V + 1) 2^-24, and logf,
# max + log s and l_t - (...) round relative to their magnitudes: 2^-23 (|max l| + log V + |logprob|).
LSE_EPS = 128 * U


def lse_roundings(V):
    """Roundings of relative size 2^-24 in a row's sum of exponentials (above)."""
    merges = -(-(-(-V // 128)) // 32)
    return 31 + 2 + (merges + 5) * 6 + 2


def lse_tol(lmax, V, ref):
    return max(LSE_EPS, lse_roundings(V) * U) + 2 * U * (lmax + math.log(V) + ref.abs())


def ref_logprob(x, W, targets, rows=2048):
    """float64 log-softmax of the fp16 logits fp16(x . W^T), on the GPU, `rows` rows at a time (an 8191 x 128256 float64 logit matrix
    alone is 8.4 GB).  (CUDA's float64 -> fp16 cast goes through fp32, which can move a logit by one fp16 ulp at a tie: the per-logit ulp
    terms of the bound cover it; on the integer grid every logit is exact.)"""
    W64 = W.double().t()
    out = []
    for r in range(0, x.shape[0], rows):
        l = (x[r:r + rows].double() @ W64).half().double()
        lt = l.gather(1, targets[r:r + rows].long()[:, None])[:, 0]
        out.append((lt - torch.logsumexp(l, -1), lt, l.abs().amax(-1)))
        del l
    return tuple(torch.cat(t) for t in zip(*out))


def check_logprob(lp, x, W, targets, what, exact=False):
    """|logprob - ref| <= ulp16(|l_t|) + ulp16(max |l|) + lse_tol: logsumexp is 1-Lipschitz in the max-norm, so a one-ulp flip of any fp16
    logit (fp32 summation order) moves the result by at most ulp16(max |l|), and the target's own flip by ulp16(|l_t|).  exact: the logits
    are exact, only the fp32 log-softmax part remains."""
    ref, lt, lmax = ref_logprob(x, W, targets)
    tol = lse_tol(lmax, W.shape[0], ref)
    if not exact:
        tol = tol + ulp16(lt) + ulp16(lmax)
    assert torch.isfinite(lp).all(), f'{what}: non-finite output'
    ratio_t = (lp.double() - ref).abs() / tol
    ratio = ratio_t.max().item()
    if ratio > 1:
        what = f'{what}: first bad row {int(torch.nonzero(ratio_t > 1)[0])}'
    report(ratio, what)
    return ref


def random_logprob_inputs(M, V, K, ldx=None, ldw=None, seed=0):
    g = torch.Generator(device='cuda').manual_seed(seed)
    x = torch.randn(M, ldx or K, device='cuda', generator=g).half()[:, :K]
    W = (torch.randn(V, ldw or K, device='cuda', generator=g) * (2.5 / math.sqrt(K))).half()[:, :K]  # logits of std ~2.5
    t = torch.randint(0, V, (M, ), device='cuda', generator=g, dtype=torch.int32)
    t[:4] = torch.tensor([0, V - 1, min(127, V - 1), min(128, V - 1)], dtype=torch.int32)[:M]
    return x, W, t


# ----------------------------------------------------------------------------- attention over the KV cache (gptq_cached_attention)
HD = 128


def make_kv_cache(B, nh, S, spans, seed=0, layers=3, layer=1, poison=True):
    """q rows for `spans` and a [layers, B, nh, S, 128] cache whose slice `layer` holds random keys / values in every row a span may read
    (rows 0 .. start + rows - 1 of its sequence), with heavy keys (scores a few units above the rest) on both sides of every 128-key tile edge
    and on the diagonal of every span.  Every other cache row -- past a span's end, sequences without a span, the other layers -- is NaN
    (poison) or random."""
    g = torch.Generator(device='cuda').manual_seed(seed)
    M = sum(n for _, _, n in spans)
    u = torch.randn(HD, device='cuda', generator=g, dtype=torch.float64)
    u = u / u.norm()
    q = (torch.randn(M, nh, HD, device='cuda', generator=g, dtype=torch.float64) + 8 * u).half().view(M, nh * HD)
    shape = (layers, B, nh, S, HD)
    fill = float('nan') if poison else 0.0
    kc = torch.full(shape, fill, device='cuda', dtype=torch.float16)
    vc = torch.full(shape, fill, device='cuda', dtype=torch.float16)
    if not poison:
        kc.normal_(generator=g)
        vc.normal_(generator=g)
    for b, s, n in spans:
        L = s + n
        k = torch.randn(nh, L, HD, device='cuda', generator=g, dtype=torch.float64) * 0.5
        heavy = [j for e in range(128, L + 128, 128) for j in (e - 2, e - 1, e, e + 1) if 0 <= j < L] + list(range(s, L, 7))
        k[:, heavy] += 4 * u
        kc[layer, b, :, :L] = k.half()
        vc[layer, b, :, :L] = torch.randn(nh, L, HD, device='cuda', generator=g).half()
    return q, kc, vc


def make_gqa_kv_cache(B, nh, nkv, S, spans, seed=0, layers=3, layer=1):
    """make_kv_cache with q rows of nh query heads over a cache of nkv K/V heads: q is drawn right after the heavy-key direction u, before
    the cache, so both draws of one seed share u.  Compare against the reference with each K/V head repeated nh / nkv times."""
    if nkv == nh:
        return make_kv_cache(B, nh, S, spans, seed=seed, layers=layers, layer=layer)
    q = make_kv_cache(B, nh, S, spans, seed=seed, layers=1, layer=0)[0]
    torch.cuda.empty_cache()
    _, kc, vc = make_kv_cache(B, nkv, S, spans, seed=seed, layers=layers, layer=layer)
    return q, kc, vc


def cached_attention_reference(q, kc, vc, spans):
    """float64 attention of each span and the per-element bound of the kernel's arithmetic (module docstring of csrc/cached_attention.cu):
      scores      fp32 accumulation of 128 products, default depth 128 / 16 + 64 = 72 roundings, then * log2(e)/sqrt(128) in fp32 (the constant's
                  rounding, the multiply, and the subtraction of the running max: <= 6 u |t|):  eps = max_j (72 u (|q|.|k_j|) / sqrt(128) + 6 u |t_j|)
                  moves every normalised weight by a factor within exp(+-2 eps)
      exp2f       2 ulp = 2^-22 relative, numerator and denominator
      fp16(P)     numerator only: 2^-11 relative, or 2^-25 absolute (subnormal fp16, p <= 1 and the final row sum >= 1)
      sums        P.V in fp32: 8 k-steps per key tile (+ 64 inside the MMA) and one rescale per tile; the row sum: 32 adds per tile per thread,
                  a rescale per tile and 2 shuffles; the division: 1 rounding;  all relative to A = sum_j p_j |v_j|
      output      one fp16 rounding: ulp16
    Returns per span (ref [n, nh, 128], bound [n, nh, 128])."""
    out, r0 = [], 0
    nh = kc.shape[1]
    for b, s, n in spans:
        L = s + n
        Q = q[r0:r0 + n].view(n, nh, HD).transpose(0, 1).double()  # [nh, n, 128]
        K, V = kc[b, :, :L].double(), vc[b, :, :L].double()          # [nh, L, 128]
        T = Q @ K.transpose(1, 2) / math.sqrt(HD)
        Aqk = Q.abs() @ K.abs().transpose(1, 2) / math.sqrt(HD)
        vis = torch.arange(L, device='cuda')[None, :] <= (s + torch.arange(n, device='cuda'))[:, None]  # [n, L]
        T = T.masked_fill(~vis, -math.inf)
        P = torch.softmax(T, -1)
        ref = P @ V
        A = P @ V.abs()
        nkt = (L - 1) // 128 + 1
        eps = (72 * U * Aqk + 6 * U * T.abs()).masked_fill(~vis, 0).amax(-1, keepdim=True)
        Vsum = vis.double() @ V.abs()  # sum over the visible keys of |v_j|
        rel = (torch.exp(2 * eps) - 1) + 2.0**-11 + 2 * 2.0**-22 + (8 * nkt + 64 + 2 * nkt + 32 * nkt + nkt + 2 + 2) * U
        E = rel * A + 2.0**-25 * Vsum
        bound = ulp16(ref.abs() + E) + E
        out.append((ref.transpose(0, 1), bound.transpose(0, 1)))
        r0 += n
    return out


def check_cached_attention(out, q, kc, vc, spans, what):
    worst, r0 = 0.0, 0
    nh = kc.shape[1]
    assert torch.isfinite(out).all(), f'{what}: non-finite output'
    for (b, s, n), (ref, bound) in zip(spans, cached_attention_reference(q, kc, vc, spans)):
        got = out[r0:r0 + n].view(n, nh, HD).double()
        ratio_t = (got - ref).abs() / bound
        ratio = ratio_t.max().item()
        assert ratio <= 1, f'{what}: span (seq {b}, start {s}, rows {n}): first bad (row, head, dim) {tuple(int(i) for i in torch.nonzero(ratio_t > 1)[0])}'
        worst = max(worst, ratio)
        r0 += n
    return worst


def run_cached_attention(q, kc, vc, spans, layer=1):
    from gptq_b200 import ops
    out = ops.cached_attention(q, kc[layer], vc[layer], spans)
    torch.cuda.synchronize()
    return out
