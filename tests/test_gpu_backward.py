"""GPU: the transposed int4 GEMM on wgmma (csrc/qgemm_wgmma_t.cu), out[M, K] = g[M, N] . deq(W)^T, and the backward pass it serves.

  * routing: which requests take the wgmma kernel and which stay on the generic CUDA-core kernel;
  * bit-exact anchors (tests/exact_fixtures.py): one-hot gradient rows return columns of W, integer-grid inputs return fp16(exact sum);
  * an element-wise bound against the fp64 product, at the tile edges and at the LLaMA-7B / 65B linears;
  * row independence, determinism, and nothing read past row M of g;
  * QuantLinear backward for act-order / 2-bit / 3-bit layers through their kernel form, and a LoRA training step against a dense twin.

The kernel tiles 128 (M <= 128) or 256 rows x 128 output features k and reduces over N in steps of 64 columns; a thread dequantises
32 consecutive k of one column n per step."""
import copy
import json
import os
import subprocess
import sys
from functools import lru_cache

import pytest
import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, 'gptq-for-llama_b200')):  # as tests/conftest.py does; needed when this file runs as the routing probe
    if _p not in sys.path:
        sys.path.insert(0, _p)

import exact_fixtures as X  # noqa: E402
from gpu_util import assert_equal, check_fp64_bound, fill_quant_linear, fp16_from_fp64, generic_t, launched_kernels, ops, recorded_transposes, \
    report  # noqa: E402
from oracle import gptq_oracle as O  # noqa: E402

pytestmark = pytest.mark.gpu

TC_1, TC_2 = 'qgemm_wgmma_t_kernel<1, 6>', 'qgemm_wgmma_t_kernel<2, 4>'
TILE_EDGE_M = [9, 63, 64, 65, 127, 128, 129, 255, 256, 257, 300]


def tc_kernel(M):
    return TC_2 if M > 128 else TC_1


FAMILIES = ('qgemm_wgmma_t_kernel', 'qlinear_transpose_generic_kernel')
FULL_K, FULL_N, FULL_GS = 4096, 4096, 128
KERNEL_FORMS = [(4, True), (3, True), (2, False)]


def _kernel_form_layer(bits, act, K=1024, N=512, gs=128):
    import quant
    ql = quant.QuantLinear(bits, gs, K, N, False)
    fill_quant_linear(ql, bits, seed=30 + bits, act=act)
    return ql.cuda()


def probe_routes():
    """Runs in a process of its own (python tests/test_gpu_backward.py): every routing case once under the activity trace, printed as one
    JSON line {label: {'transposed': [names of the transposed quantized-linear kernels launched], 'any': trace had kernel records}}.
    The trace is kept out of the pytest process: once a process has attached the activity tracer, the CUDA-graph and cooperative-launch
    tests that run later in the same process leave it dropping kernel records, and the routing assertions of the files after them skip."""
    from gptq_b200 import ops
    out = {}
    plans = {(bits, act): _kernel_form_layer(bits, act).kernel_plan() for bits, act in KERNEL_FORMS}  # derived before the first trace

    def trace(label, fn):
        fn()  # first launch (module load, shared-memory attribute) outside the trace
        for _ in range(3):  # a trace that lacks the kernel's record (the launch was traced, the kernel was not) is taken again
            _, names = launched_kernels(fn)
            qk = sorted(n for n in names if any(f + '<' in n for f in FAMILIES))
            if qk:
                break
        out[label] = {'transposed': qk, 'any': bool(names)}

    K, N, gs = 256, 128, 64
    L = random_layer(K, N, 4, gs, seed=1)
    g = gradients('random', 300, N, 0)
    for M in (8, 9, 128, 129, 300):
        trace(f'int4 hint M={M}', lambda: ops.transpose_matmul248(g[:M], *L.dev, 4, 15, groupsize=gs))
    trace('8-bit', lambda: ops.transpose_matmul248(g, *random_layer(K, N, 8, gs, seed=2).dev, 8, 255, groupsize=gs))
    trace('stored act-order form', lambda: ops.transpose_matmul248(g, *random_layer(K, N, 4, gs, act=True, seed=3).dev, 4, 15, groupsize=0))
    trace('groupsize 16', lambda: ops.transpose_matmul248(g, *random_layer(K, N, 4, 16, seed=5).dev, 4, 15, groupsize=16))
    trace('N=96', lambda: ops.transpose_matmul248(g[:, :96].contiguous(), *random_layer(K, 96, 4, gs, seed=4).dev, 4, 15, groupsize=gs))
    trace('misaligned ldg', lambda: ops.transpose_matmul248(misaligned(g), *L.dev, 4, 15, groupsize=gs))
    dev, _ = device_layer(FULL_K, FULL_N, FULL_GS, seed=1)
    for M in (300, 2048):
        gf = gradients('random', M, FULL_N, M)
        trace(f'full size M={M}', lambda: ops.transpose_matmul248(gf, *dev, 4, 15, groupsize=FULL_GS))
    trace('full size without the hint', lambda: ops.transpose_matmul248(gf, *dev, 4, 15, groupsize=0))
    for bits, act in KERNEL_FORMS:
        plan = plans[bits, act]
        for M in (40, 300):
            go = gradients('random', M, 512, 2)
            trace(f'kernel form bits={bits} act={act} M={M}', lambda: ops.transpose_matmul248(go, *plan.parts(), plan.bits, 15, groupsize=plan.hint))
    print('ROUTES ' + json.dumps(out))


def misaligned(g):
    """The same values behind a row stride that is not a multiple of 8 elements."""
    wide = torch.zeros(g.shape[0], g.shape[1] + 4, dtype=torch.float16, device='cuda')
    wide[:, :g.shape[1]] = g
    view = wide[:, :g.shape[1]]
    assert view.stride(0) % 8 != 0
    return view


@pytest.fixture(scope='module')
def routes():
    res = subprocess.run([sys.executable, os.path.abspath(__file__)], capture_output=True, text=True, timeout=900)
    assert res.returncode == 0, f'the routing probe failed:\n{res.stdout[-2000:]}\n{res.stderr[-4000:]}'
    table = json.loads([line for line in res.stdout.splitlines() if line.startswith('ROUTES ')][-1][7:])
    if not any(v['any'] for v in table.values()):  # a routing assertion that cannot see kernels must not pass
        pytest.skip('CUDA activity tracing returned no kernel events on this machine')
    return table


def assert_route(routes, label, kernel):
    """The request `label` launched `kernel` (demangled name with its template arguments) and no other transposed quantized-linear kernel."""
    strip = lambda t: t.replace(' ', '')
    qk = routes[label]['transposed']
    assert qk and all(strip(kernel) in strip(n) for n in qk), f'{label}: expected {kernel}, launched {qk}'


@pytest.fixture(scope='module', autouse=True)
def release_device_memory():
    """The full-size layers and their fp64 references are cached for the module; hand the memory back when it is done."""
    yield
    random_layer.cache_clear()
    device_layer.cache_clear()
    torch.cuda.empty_cache()


class Layer:
    """A packed layer on the device with the oracle's fp16 weight (built on the CPU) transposed to [N, K]."""

    def __init__(self, packed, bits):
        self.cpu = tuple(packed)
        self.dev = tuple(t.cuda() for t in packed)
        self.Wt = O.dequant(*packed, bits).cuda().t().contiguous()


@lru_cache(maxsize=None)
def random_layer(K, N, bits, gs, act=False, seed=0):
    return Layer(O.random_packed(K, N, bits, gs, act_order=act, seed=seed)[:4], bits)


@lru_cache(maxsize=2)
def device_layer(K, N, gs, seed=0):
    """A random int4 layer generated on the device (full-size shapes), with the fp16 weight the kernels see, transposed: [N, K].
    The dequantisation kernel behind ops.dequant is pinned bit for bit to the oracle elsewhere in the suite."""
    from gptq_b200 import ops as _ops
    gen = torch.Generator(device='cuda').manual_seed(seed)
    G = -(-K // gs)
    rnd = lambda *shape: torch.randint(-2**31, 2**31, shape, generator=gen, device='cuda', dtype=torch.int64).to(torch.int32)
    qw, qz = rnd(K // 8, N), rnd(G, N // 8)
    s = (torch.rand(G, N, generator=gen, device='cuda') * 1e-2 + 1e-3).half()
    gi = (torch.arange(K, device='cuda') // gs).to(torch.int32)
    return (qw, s, qz, gi), _ops.dequant(qw, s, qz, gi, 4, gs).t().contiguous()


def gradients(kind, M, N, seed):
    gen = torch.Generator(device='cuda').manual_seed(seed)
    g = torch.randn(M, N, generator=gen, device='cuda')
    if kind == 'heavy':  # a few entries carry most of the mass (log-normal magnitudes, kept inside fp16)
        g = (g * torch.exp(2.0 * torch.randn(M, N, generator=gen, device='cuda'))).clamp(-3e4, 3e4)
    elif kind == 'sparse':
        g = g * (torch.rand(M, N, generator=gen, device='cuda') < 0.02)
    return g.half()


def where(M, N, m, k, n=None):
    wt = 2 if M > 128 else 1
    s = f'm={m} k={k} tile (row {m // (128 * wt)}, feature {k // 128}) WT={wt} warpgroup {(m % (128 * wt)) // (64 * wt)}'
    return s if n is None else s + f' n={n} (step {n // 64}, n%64={n % 64})'


# ============================================================================= routing
def test_routing(ops, routes):
    for M in (9, 128, 129, 300):
        assert_route(routes, f'int4 hint M={M}', tc_kernel(M))
    assert_route(routes, 'int4 hint M=8', generic_t(4))
    assert_route(routes, '8-bit', generic_t(8))
    for label in ('stored act-order form', 'groupsize 16', 'N=96', 'misaligned ldg', 'full size without the hint'):
        assert_route(routes, label, generic_t(4))
    for M in (300, 2048):
        assert_route(routes, f'full size M={M}', TC_2)
    # Kernel-form requests: the trace of these calls has been seen to come back without the kernel's record; the request itself is pinned
    # by test_kernel_form_layers_backpropagate_on_the_wgmma_kernel (int4, hint, M > 8: the predicate's inputs), so only a record that is
    # present is held to the wgmma kernel here.
    for bits, act in KERNEL_FORMS:
        for M in (40, 300):
            label = f'kernel form bits={bits} act={act} M={M}'
            if routes[label]['transposed']:
                assert_route(routes, label, tc_kernel(M))
            else:
                print(f'  {label}: no kernel record in the trace')
    # the generic route on the request the wgmma kernel rejects for its stride computes the same product
    K, N, gs = 256, 128, 64
    L = random_layer(K, N, 4, gs, seed=1)
    g = gradients('random', 300, N, 0)
    out = ops.transpose_matmul248(misaligned(g), *L.dev, 4, 15, groupsize=gs)
    check_fp64_bound(out, g, L.Wt, what='misaligned ldg (generic)', depth=N / 16 + 64)


# ============================================================================= bit-exact anchors
GROUPS = [(256, 32), (256, 64), (256, 128), (256, 256), (384, 256)]  # (K, groupsize); the last: a partial last group of 128


@pytest.mark.parametrize('K,gs', GROUPS)
@pytest.mark.parametrize('M', TILE_EDGE_M)
def test_onehot_rows_return_columns(ops, K, gs, M):
    """g[r] = sign * 2^e * e_n for every n of three 64-column steps: out[r] is column n of W, at every k of two or three 128-feature
    tiles, so every dequantised weight, its place in the MN-major tile and the reduction order of the staging are pinned."""
    N = 192
    L = random_layer(K, N, 4, gs, seed=K + gs)
    assert L.cpu[1].shape[0] == -(-K // gs)
    ns = list(range(N))
    ns = ns + ns[:(-len(ns)) % M]
    gin, mult = X.onehot_rows(ns, N, salt=M)
    gin = gin.cuda()
    what = f'transposed one-hot K={K} gs={gs} M={M}'
    outs = [ops.transpose_matmul248(gin[c * M:(c + 1) * M], *L.dev, 4, 15, groupsize=gs) for c in range(len(ns) // M)]
    assert_equal(torch.cat(outs), X.onehot_expect(L.Wt, ns, mult), what, lambda r, k: where(M, N, r % M, k, ns[r]) + f', call {r // M}')


@pytest.mark.parametrize('K,N,gs,M', [(4096, 4096, 128, 300), (4096, 11008, 128, 129), (11008, 4096, 1024, 257), (512, 16384, 32, 9)])
def test_integer_grid_sums_are_exact(ops, K, N, gs, M):
    """g integer in [-2, 2] and power-of-two scales: every partial sum over N <= 16384 is exact in fp32, so out == fp16(exact)."""
    packed = X.pow2_packed(K, N, gs, seed=K + N)
    dev = tuple(t.cuda() for t in packed)
    Wt = O.dequant(*packed, 4).cuda().t().contiguous()
    g = X.int_x(M, N, -2, 2, seed=M).cuda()
    what = f'transposed integer grid M={M} K={K} N={N} gs={gs}'
    out = ops.transpose_matmul248(g, *dev, 4, 15, groupsize=gs)
    exp = fp16_from_fp64(X.exact_product(g, Wt)).cuda()
    assert_equal(out, exp, what, lambda m, k: where(M, N, m, k))


# ============================================================================= fp64 bound
KINDS = ('random', 'heavy', 'sparse')


@pytest.mark.parametrize('K,gs', GROUPS)
def test_fp64_bound_at_tile_edges(ops, K, gs):
    N = 192
    L = random_layer(K, N, 4, gs, seed=K + gs)
    worst = 0.0
    for M in TILE_EDGE_M:
        for i, kind in enumerate(KINDS):
            g = gradients(kind, M, N, seed=M + i)
            what = f'transposed {kind} K={K} gs={gs} M={M}'
            out = ops.transpose_matmul248(g, *L.dev, 4, 15, groupsize=gs)
            worst = max(worst, check_fp64_bound(out, g, L.Wt, what=what, depth=N / 16 + 64, locate=lambda m, k: where(M, N, m, k)))
    report(worst, f'transposed tile edges K={K} gs={gs}: all M, all inputs')


# 7B linears, 65B extremes; LLaMA-2-70B qkv, gate|up and down_proj; LLaMA-3-8B gate|up
FULL_SHAPES = [(4096, 12288), (4096, 4096), (4096, 11008), (11008, 4096), (8192, 24576), (22016, 8192), (8192, 10240), (8192, 28672), (28672, 8192),
               (4096, 14336)]


@pytest.mark.parametrize('K,N', FULL_SHAPES)
@pytest.mark.parametrize('gs', [128, 1024])
def test_fp64_bound_and_generic_parity_at_llama_shapes(ops, K, N, gs):
    """M = 300 and 2048 on random, heavy-tailed and sparse gradients.  At M = 300 the generic kernel runs on the same inputs (taken
    without the hint): the same dequantised operands in another summation order, so both sit inside the bound of the same fp64 value."""
    dev, Wt = device_layer(K, N, gs, seed=K + N + gs)
    for M in (300, 2048):
        for i, kind in enumerate(KINDS):
            g = gradients(kind, M, N, seed=M + i)
            what = f'transposed {kind} M={M} K={K} N={N} gs={gs}'
            out = ops.transpose_matmul248(g, *dev, 4, 15, groupsize=gs)
            check_fp64_bound(out, g, Wt, what=what, depth=N / 16 + 64, locate=lambda m, k: where(M, N, m, k))
            if M == 300 and kind == 'random' and K * N <= 4096 * 12288:
                gen = ops.transpose_matmul248(g, *dev, 4, 15, groupsize=0)
                check_fp64_bound(gen, g, Wt, what=what + ' (generic)', depth=N / 16 + 64)
                d = (out.double() - gen.double()).abs().max().item()
                print(f'  {what}: max |wgmma - generic| = {d:.3g}')


# ============================================================================= independence, determinism
def test_rows_are_independent_and_runs_repeat(ops):
    K, N, gs = 512, 1024, 128
    L = random_layer(K, N, 4, gs, seed=7)
    fn = lambda x: ops.transpose_matmul248(x, *L.dev, 4, 15, groupsize=gs)
    g = gradients('random', 300, N, 5)
    ref = fn(g)
    assert torch.equal(fn(g), ref), 'two runs differ'
    for r in (0, 63, 64, 127, 128, 255, 256, 299):
        poisoned = torch.full_like(g, float('nan'))
        poisoned[r] = g[r]
        assert torch.equal(fn(poisoned)[r], ref[r]), f'row {r} of M=300 depends on the other rows'
        small = torch.full((9, N), float('nan'), dtype=torch.float16, device='cuda')
        small[r % 9] = g[r]
        assert torch.equal(fn(small)[r % 9], ref[r]), f'row {r}: M=9 and M=300 disagree'


@pytest.mark.parametrize('M', [9, 100, 129, 300])
def test_nothing_past_row_M_is_read_into_the_result(ops, M):
    K, N, gs = 256, 256, 64
    L = random_layer(K, N, 4, gs, seed=8)
    buf = torch.full((512, N), float('nan'), dtype=torch.float16, device='cuda')
    g = gradients('random', M, N, M)
    buf[:M] = g
    out = ops.transpose_matmul248(buf[:M], *L.dev, 4, 15, groupsize=gs)
    assert torch.isfinite(out).all()
    assert torch.equal(out, ops.transpose_matmul248(g, *L.dev, 4, 15, groupsize=gs))


# ============================================================================= modules: kernel-form layers
@pytest.mark.parametrize('bits,act', KERNEL_FORMS)
@pytest.mark.parametrize('M', [40, 300])
def test_kernel_form_layers_backpropagate_on_the_wgmma_kernel(ops, bits, act, M):
    """Act-order and 2/3-bit layers: QuantLinear hands its kernel form (rows regrouped, fields widened to int4) to the autograd function
    and gathers x; the gradient comes back through that gather.  x.grad equals go . W^T of the STORED tensors within the bound."""
    K, N = 1024, 512
    ql = _kernel_form_layer(bits, act)
    assert ql.kernel_plan() is not None and ql.kernel_plan().bits == 4 and (ql.kernel_plan().perm is not None) == act
    Wt = ops.dequant(ql.qweight, ql.scales, ql.qzeros, ql.g_idx, bits, 0).t().contiguous()
    x = gradients('random', M, K, 1).requires_grad_(True)
    go = gradients('random', M, N, 2)
    out = ql(x)
    what = f'kernel-form backward bits={bits} act={act} M={M}'
    with recorded_transposes() as rec:
        out.backward(go)
    assert x.grad.dtype == torch.float16 and x.grad.shape == x.shape
    check_fp64_bound(x.grad, go, Wt, what=what, depth=N / 16 + 64)
    assert len(rec.calls) == 1 and rec.calls[0][0][1].data_ptr() == ql.kernel_plan().qweight.data_ptr(), 'the backward did not receive the kernel form'
    rec.check(what)  # test_routing asserts the kernel this request launches


def test_backward_under_autocast_returns_the_inputs_dtype():
    """custom_fwd(cast_inputs=float16) semantics: an fp32 input under autocast gets an fp32 gradient (autograd casts it back)."""
    import quant
    ql = quant.QuantLinear(4, 128, 256, 128, False)
    fill_quant_linear(ql, 4, seed=40)
    ql = ql.cuda()
    x = torch.randn(16, 256, device='cuda', requires_grad=True)
    with torch.autocast('cuda', dtype=torch.float16):
        out = ql(x)
    out.float().sum().backward()
    assert out.dtype == torch.float16 and x.grad.dtype == torch.float32 and torch.isfinite(x.grad).all()


# ============================================================================= a training step
class LoRA(nn.Module):
    """base(x) + (x A^T) B^T with fp32 master adapters applied in the activation dtype."""

    def __init__(self, base, fin, fout, r=8, seed=0):
        super().__init__()
        gen = torch.Generator().manual_seed(seed)
        self.base = base
        self.A = nn.Parameter(torch.randn(r, fin, generator=gen) * 0.05)
        self.B = nn.Parameter(torch.randn(fout, r, generator=gen) * 0.05)

    def forward(self, x):
        return self.base(x) + (x @ self.A.t().to(x.dtype)) @ self.B.t().to(x.dtype)


def rel_err(out, ref):
    """max |out - ref| / max(|ref|, rms(ref)): relative to the element where it is large, to the tensor's scale where it cancels."""
    out, ref = out.detach().double(), ref.detach().double()
    return ((out - ref).abs() / torch.maximum(ref.abs(), ref.pow(2).mean().sqrt())).max().item()


def test_lora_step_on_one_layer_matches_the_dense_twin(ops):
    """Forward in fp16 on the quantized layer, backward through the wgmma kernel: x.grad and the adapter gradients against an fp32 twin
    whose base weight is ops.dequant of the same tensors.  Bound 4e-3: each of the fp16 roundings on the way (the two products, their
    sum, the adapter's intermediate) is worth 2^-11 ~ 4.9e-4 relative to its own value."""
    import quant
    K, N, M, gs = 512, 256, 64, 128
    ql = quant.QuantLinear(4, gs, K, N, False)
    fill_quant_linear(ql, 4, seed=50)
    ql = ql.cuda()
    W = ops.dequant(ql.qweight, ql.scales, ql.qzeros, ql.g_idx, 4, gs).float()
    dense = nn.Linear(K, N, bias=False).cuda()
    dense.weight.data = W.t().contiguous()
    dense.weight.requires_grad_(False)
    q, d = LoRA(ql, K, N).cuda(), LoRA(dense, K, N).cuda()
    xq = gradients('random', M, K, 3).requires_grad_(True)
    xd = xq.detach().float().requires_grad_(True)
    t = torch.randn(M, N, device='cuda', generator=torch.Generator(device='cuda').manual_seed(4))
    out = q(xq)
    loss_q = (out.float() * t).sum() / M
    with recorded_transposes() as rec:
        loss_q.backward()
    rec.check('lora step backward')
    ((d(xd) * t).sum() / M).backward()
    for name, a, b in (('x.grad', xq.grad, xd.grad), ('A.grad', q.A.grad, d.A.grad), ('B.grad', q.B.grad, d.B.grad)):
        report(rel_err(a, b), f'lora step {name} vs dense twin (relative)', limit=4e-3)


def test_lora_finetuning_of_a_tiny_llama_matches_the_dense_twin(ops):
    """A random HF LLaMA after make_quant_linear only (the training recipe: the fused attention / MLP / norm modules have no backward),
    LoRA adapters on q_proj and v_proj, two SGD steps on a fixed batch.  The twin is the same model in fp32 with every quantized linear
    replaced by its dequantised weight.  fp16 activations, softmax and norms through two decoder layers against fp32 ones: the adapter
    gradients stay within 0.1 of the twin's (relative to max(|ref|, rms); about 0.02 at the first step), the losses within 5e-3; the
    packed buffers are untouched and the loss goes down."""
    import quant
    import utils
    from transformers import LlamaConfig, LlamaForCausalLM
    cfg = LlamaConfig(hidden_size=128, intermediate_size=384, num_hidden_layers=2, num_attention_heads=2, num_key_value_heads=2, vocab_size=256,
                      max_position_embeddings=64)
    torch.manual_seed(0)
    model = LlamaForCausalLM(cfg).half().eval()
    twin = copy.deepcopy(model).float().cuda()
    layers = utils.find_layers(model)
    layers.pop('lm_head')
    quant.make_quant_linear(model, layers, 4, 32)
    seed = 0
    for name, m in model.named_modules():
        if isinstance(m, quant.QuantLinear):
            seed += 1
            fill_quant_linear(m, 4, seed=60 + seed)
    model = model.cuda()
    for name, m in list(model.named_modules()):
        if isinstance(m, quant.QuantLinear):
            lin = twin.get_submodule(name)
            lin.weight.data = ops.dequant(m.qweight, m.scales, m.qzeros, m.g_idx, 4, 32).float().t().contiguous()
    for mdl in (model, twin):
        for p in mdl.parameters():
            p.requires_grad_(False)
        for li, layer in enumerate(mdl.model.layers):
            for j, pname in enumerate(('q_proj', 'v_proj')):
                setattr(layer.self_attn, pname, LoRA(getattr(layer.self_attn, pname), 128, 128, seed=10 * li + j).cuda())
    adapters = lambda mdl: [p for p in mdl.parameters() if p.requires_grad]
    assert len(adapters(model)) == 8
    before = {k: v.clone() for k, v in model.state_dict().items() if k.rsplit('.', 1)[-1] in ('qweight', 'qzeros', 'scales', 'g_idx')}
    assert len(before) == 4 * 7 * 2
    ids = torch.randint(0, 256, (2, 24), generator=torch.Generator().manual_seed(1)).cuda()
    lr, losses = 0.5, {id(model): [], id(twin): []}
    for step in range(3):
        for mdl in (model, twin):
            for p in adapters(mdl):
                p.grad = None
            fn = lambda: mdl(ids, labels=ids, use_cache=False).loss
            loss = fn()
            losses[id(mdl)].append(loss.item())
            if step == 2:
                continue
            if mdl is model and step == 0:
                with recorded_transposes() as rec:
                    loss.backward()
                rec.check('tiny llama backward', at_least=11)  # every quantized linear whose input depends on an adapter
            else:
                loss.backward()
        if step == 2:
            break
        worst = max(rel_err(a.grad, b.grad) for a, b in zip(adapters(model), adapters(twin)))
        report(worst, f'tiny llama step {step}: adapter gradients vs dense twin (relative)', limit=0.1)
        with torch.no_grad():
            for mdl in (model, twin):
                for p in adapters(mdl):
                    p -= lr * p.grad
    lq, lt = losses[id(model)], losses[id(twin)]
    print(f'  tiny llama losses: quantized {lq}, dense twin {lt}')
    assert all(abs(a - b) <= 5e-3 * abs(b) for a, b in zip(lq, lt))
    assert lq[2] < lq[1] < lq[0] and lt[2] < lt[1] < lt[0]
    after = model.state_dict()
    assert all(torch.equal(after[k], v) for k, v in before.items()), 'a packed buffer changed during training'


if __name__ == '__main__':
    probe_routes()
