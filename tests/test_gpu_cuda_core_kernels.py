"""GPU: the generic CUDA-core kernels (csrc/generic.cu) at LLaMA shapes, and the engine paths that run on them.

The generic kernels are the only path for every 8-bit layer (the int4 matvec, the wgmma GEMMs and the persistent decode kernel take
bits 4 only) and for act-order layers whose groups are not all the same size (act-order at groupsize 1024 on down_proj: 11008 =
10 x 1024 + 768, 13824 = 13.5 x 1024), which QLayerWeights.kernel_form leaves in their stored form.  Here they are held to:
  * ops.dequant == the oracle's dequantisation (O.dequant, CPU), bit for bit, at the 7B / 13B / 65B linears: the reference that
    tests/test_gpu_backward.py and tests/test_gpu_modules.py compare against is itself pinned;
  * forward (qlinear_generic_kernel): one-hot rows bit for bit at every k of the first and last run of each warp's k-stride, both sides
    of every group boundary, and k whose neighbour k ^ 1 has another g_idx; integer-grid inputs give fp16 of the exact sum; random,
    heavy-tailed and SwiGLU-sized inputs stay within the fp64 bound of depth K / 8 + 8 (one warp's fmaf chain over K / 8 products, then
    8 warp partials); the fused SwiGLU (DUAL) instance at 4096 -> 11008;
  * transposed (qlinear_transpose_generic_kernel): one-hot gradient rows return whole columns of W; random gradients within the bound
    of depth N / 256 + 13 (derived in transpose_depth);
  * the gridDim.y chunk loops of both launchers, rows written exactly once and nothing past row M;
  * the engine on these kernels: 7B int8 g128, 7B int4 act-order gs 1024 and 13B int3 act-order gs 1024 decode on the kernel chain
    (asserted from an activity trace taken in a child process), with bit-exact V rows, K rows and logits against the oracle; extend and
    score of the 7B int8 model; an 8-bit QuantLinear backward at the down_proj shape.
Which kernel serves each class of request is read from activity traces taken once, in a child process (probe_routes).

The file sorts ahead of tests/test_gpu_exact.py, the first file that traces in the pytest process, and that is deliberate.  Once torch.profiler
has run in a process, sustained untraced GPU work in that process, or a profiler session in a child process, leaves its later sessions without
kernel records (on an H100: 45 s of back-to-back matmuls did it, as did one child that profiled; 45 s of sleep and a child that only used
CUDA did not), and gpu_util.run_kernel then skips.  This file launches tens of thousands of kernels and runs a profiling child, so like
test_gpu_backward.py and test_gpu_cached_attention.py it runs before any in-process trace is taken.

One-hot rows carry the multiplier sign * 3 * 2^e rather than a power of two: 3 * W is exact in fp32 but not in fp16, so the output is the
single fp16 rounding of 3 * 2^e * W16, and a kernel that fed an unrounded (w - z) * s into the product would round twice and differ.
The worst |err| / bound per sweep is printed at the end of the module (pytest -s)."""
import ctypes
import json
import math
import os
import subprocess
import sys
from functools import lru_cache

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, 'gptq-for-llama_b200')):  # as tests/conftest.py does; needed when this file runs as the routing probe
    if _p not in sys.path:
        sys.path.insert(0, _p)

import pytest  # noqa: E402
import torch  # noqa: E402

import exact_fixtures as X  # noqa: E402
from gpu_util import Layer, WorstRatios, assert_equal, check_fp64_bound, check_swiglu_fp64_bound, cyclic, fp16_from_fp64, fp16_ulp_distance, \
    generic, generic_t, launched_kernels, ops, recorded_transposes  # noqa: E402
from llama_oracle import END_TO_END_TOL, KV_ROW_TOL, MLP_HEAD_TOL, LlamaOracle, assert_no_failures, check, check_extend_against_stepping, \
    check_scores  # noqa: E402
from oracle import gptq_oracle as O  # noqa: E402

pytestmark = pytest.mark.gpu

WORST = WorstRatios()
note = WORST.note


@pytest.fixture(scope='module', autouse=True)
def worst_ratio_summary():
    yield
    layer.cache_clear()
    torch.cuda.empty_cache()
    WORST.summary()


# ----------------------------------------------------------------------------- layers and inputs
@lru_cache(maxsize=1)
def layer(K, N, bits, gs, act, seed=0):
    return Layer.random(K, N, bits, gs, act, seed=seed)


def pow2_layer(K, N, bits, gs, act, seed=0):
    """Random fields and zeros of any bit width, scales 2^-j with j in [bits, bits + 2] per (group, column): every weight is a multiple of
    2^-(bits+2) with |W| <= 1, so with x in {-1, 0, 1} every partial sum is a multiple of 2^-(bits+2) below K: under 2^24 units for
    K <= 16384, exact in fp32 in any order."""
    assert K * 2**(bits + 2) <= 2**24
    gen = torch.Generator().manual_seed(seed)
    G = -(-K // gs)
    q = torch.randint(0, 2**bits, (K, N), generator=gen).numpy()
    z = torch.randint(0, 2**bits, (G, N), generator=gen).numpy()
    s = torch.pow(2.0, -torch.randint(bits, bits + 3, (G, N), generator=gen).double()).half()
    g = O.make_g_idx(K, gs, act, gen)
    return Layer((torch.from_numpy(O.pack_rows(q, bits)), s, torch.from_numpy(O.pack_cols(z, bits)), g), bits, gs, act)


def onehot3(ks, K, salt=0):
    """Row r = sign_r * 3 * 2^e_r * e_{ks[r]}, e in [-2, 1].  Returns (x fp16 [R, K], mult float64 [R])."""
    x, mult = X.onehot_rows(ks, K, salt)
    mult = mult * 3 / torch.where(mult.abs() > 2, 2.0, 1.0).double()  # e in [-2, 1]: |3 * 2^e * W| stays far inside fp16
    x.zero_()
    x[torch.arange(len(ks)), torch.as_tensor(ks)] = mult.half()
    assert torch.equal(x.double().sum(1), mult)
    return x, mult


def onehot3_expect(W, ks, mult):
    """fp16 [R, N]: 3 * 2^e * W[ks[r]] rounded once (the product is exact in fp32 and float64)."""
    rows = W.index_select(0, torch.as_tensor(ks, device=W.device)).double() * mult.to(W.device)[:, None]
    return fp16_from_fp64(rows).to(W.device)


def generic_ks(L, extra=64, seed=0):
    """k of a one-hot sweep of the forward kernel: all 32 positions of the first and the last run of each of the 8 warps' k-strides (run r
    goes to warp r % 8; 3-bit fields straddle two words at positions 10 and 21), both sides of every group boundary, and for act-order
    layers k and k ^ 1 where the two have different g_idx (WeightCursor::set_group keeps the last group it loaded), plus random k."""
    K, runs = L.K, L.K // 32
    ks = set()
    for w in range(8):
        rs = list(range(w, runs, 8))
        for r in (rs[0], rs[-1]):
            ks |= set(range(32 * r, 32 * r + 32))
    ks |= {k for b in range(L.gs, K, L.gs) for k in (b - 1, b)}
    gen = torch.Generator().manual_seed(seed)
    ks |= set(torch.randint(0, K, (extra, ), generator=gen).tolist())
    if L.act:
        g = L.cpu[3].long()
        diff = torch.nonzero(g != g[torch.arange(K) ^ 1])[:, 0]
        ks |= {int(k) ^ b for k in diff[torch.randperm(diff.numel(), generator=gen)[:extra]] for b in (0, 1)}
    return sorted(ks)


def inputs(kind, M, K, seed):
    """fp16 [M, K] on the device: 'randn' N(0, 1); 'heavy' log-normal magnitudes (a few entries carry most of the mass); 'swiglu'
    silu(a) * b with a, b ~ N(0, 0.02), median |x| about 7e-5, nearly half of them fp16 subnormals, like the down_proj input of a real layer."""
    gen = torch.Generator(device='cuda').manual_seed(seed)
    x = torch.randn(M, K, generator=gen, device='cuda')
    if kind == 'heavy':
        x = (x * torch.exp(2.0 * torch.randn(M, K, generator=gen, device='cuda'))).clamp(-1e3, 1e3)  # an 8-bit weight reaches 2.8: no fp16 overflow
    elif kind == 'swiglu':
        a, b = x * 0.02, torch.randn(M, K, generator=gen, device='cuda') * 0.02
        x = torch.nn.functional.silu(a) * b
    return x.half()


def check_sliced(out, x, W, depth, what, cols=4096):
    """check_fp64_bound over slices of `cols` output columns (the fp64 copies of a 65B weight stay small)."""
    worst = 0.0
    for c0 in range(0, W.shape[1], cols):
        c1 = min(c0 + cols, W.shape[1])
        worst = max(worst, check_fp64_bound(out[:, c0:c1], x, W[:, c0:c1], what=f'{what} cols {c0}:{c1}', depth=depth,
                                            locate=lambda m, n, c0=c0: f'm={m} n={c0 + n}'))
    return worst


def forward_depth(K):
    """qlinear_generic_kernel: lane n of warp w accumulates run r = w, w + 8, ... (K / 256 runs of 32 k: K / 8 fmaf in one chain); warp 0
    then adds the 8 warp partials one after another."""
    return K / 8 + 8


def transpose_depth(N):
    """qlinear_transpose_generic_kernel: lane l of warp w accumulates n = 32 w + l + 256 i (ceil(N / 256) fmaf in one chain per k); warp_sum
    then adds the 32 lanes in a 5-level butterfly, and warp 0 adds the 8 warp partials one after another: N / 256 + 5 + 8."""
    return math.ceil(N / 256) + 5 + 8



# ============================================================================= 1. ops.dequant, bit for bit
# (bits, K, N, gs, act): every bit width; the hint and the act-order gather; gs 32 / 128 / 1024 (a partial last group on K = 11008 and
# 22016) / full K; the 7B linears, 13B down_proj and 65B down_proj.
DEQUANT_CASES = [
    (2, 4096, 12288, 32, False), (2, 11008, 4096, 1024, True), (2, 4096, 11008, 4096, False),
    (3, 4096, 12288, 128, True), (3, 11008, 4096, 1024, False), (3, 4096, 4096, 4096, True),
    (4, 4096, 11008, 32, True), (4, 11008, 4096, 11008, False), (4, 13824, 5120, 1024, True),
    (8, 4096, 12288, 128, False), (8, 4096, 4096, 32, True), (8, 11008, 4096, 1024, True), (8, 4096, 11008, 4096, False),
    (4, 22016, 8192, 1024, False), (8, 22016, 8192, 128, True),
]


def test_dequant_cases_cover_the_table():
    assert {c[0] for c in DEQUANT_CASES} == {2, 3, 4, 8}
    for bits in (2, 3, 4, 8):
        assert {c[4] for c in DEQUANT_CASES if c[0] == bits} == {True, False}
    assert {c[3] for c in DEQUANT_CASES} >= {32, 128, 1024} and any(c[3] == c[1] for c in DEQUANT_CASES)
    assert any(c[1] % c[3] for c in DEQUANT_CASES)
    assert {(c[1], c[2]) for c in DEQUANT_CASES} >= {(4096, 12288), (4096, 4096), (4096, 11008), (11008, 4096), (13824, 5120), (22016, 8192)}


@pytest.mark.parametrize('bits,K,N,gs,act', DEQUANT_CASES)
def test_dequant_matches_the_oracle_bit_for_bit(ops, bits, K, N, gs, act):
    packed = O.random_packed(K, N, bits, gs, act_order=act, seed=bits + K + N + gs)[:4]
    W = O.dequant(*packed, bits)
    dev = tuple(t.cuda() for t in packed)
    out = ops.dequant(*dev, bits, 0 if act else gs)
    torch.cuda.synchronize()
    what = f'dequant bits={bits} K={K} N={N} gs={gs} act={act}'
    got, want = out.cpu().view(torch.int16), W.view(torch.int16)
    if not torch.equal(got, want):
        bad = got != want
        k, n = (int(i) for i in torch.nonzero(bad)[0])
        raise AssertionError(f'{what}: {int(bad.sum())} / {bad.numel()} weights differ; first at k={k} (g_idx {int(packed[3][k])}) n={n}: '
                             f'got {out[k, n].item()!r}, want {W[k, n].item()!r}')


# ============================================================================= 2. forward generic kernel at LLaMA linears
SHAPES_7B = {'qkv': (4096, 12288), 'o': (4096, 4096), 'gate': (4096, 11008), 'down': (11008, 4096)}
# (bits, act, gs, K, N)
FORWARD_CASES = [(8, False, 128, *SHAPES_7B[s]) for s in ('qkv', 'o', 'gate', 'down')]
FORWARD_CASES += [(3, False, 1024, *SHAPES_7B[s]) for s in ('qkv', 'down')]
FORWARD_CASES += [(8, True, 128, *SHAPES_7B[s]) for s in ('o', 'down')]
FORWARD_CASES += [(4, True, 1024, *SHAPES_7B[s]) for s in ('gate', 'down')]
FORWARD_CASES += [(3, True, 128, *SHAPES_7B[s]) for s in ('qkv', 'o')]
FORWARD_CASES += [(3, True, 1024, 13824, 5120), (8, False, 128, 22016, 8192)]  # 13B and 65B down_proj
SMALL_M = (1, 2, 3, 5, 8)
BATCHED_M = 300


def _forward(ops, L, x):
    return ops.matmul248(x, *L.dev, L.bits, None, groupsize=L.hint)


@pytest.mark.parametrize('bits,act,gs,K,N', FORWARD_CASES)
def test_forward_at_llama_linears(ops, routes, bits, act, gs, K, N):
    """M = 1, 2, 3, 5, 8 (the MB = 1, 2 and 4 instantiations, the last with a clamped row block) and 300.  One-hot rows: out[r] =
    fp16(3 * 2^e * W[k_r]) bit for bit.  Random and heavy-tailed inputs (and SwiGLU-sized ones on the down_proj shapes) within the fp64
    bound of depth forward_depth(K)."""
    for M in SMALL_M + (BATCHED_M, ):
        assert_route(routes, f'forward {bits} {act} {gs} M={M}', generic(bits, M))
    L = layer(K, N, bits, gs, act, seed=K + N + bits + act)
    ks0 = generic_ks(L, seed=K + bits)
    g = L.cpu[3]
    kinds = ('randn', 'heavy', 'swiglu') if K > 4096 else ('randn', 'heavy')
    for M in SMALL_M + (BATCHED_M, ):
        ks = cyclic(ks0, M)
        x, mult = onehot3(ks, K, salt=M)
        x = x.cuda()
        what = f'one-hot bits={bits} act={act} gs={gs} K={K} N={N} M={M}'
        out = torch.cat([_forward(ops, L, x[c * M:(c + 1) * M]) for c in range(len(ks) // M)])
        assert_equal(out, onehot3_expect(L.W, ks, mult), what,
                     lambda r, n: f'm={r % M} k={ks[r]} (run {ks[r] // 32}, warp {ks[r] // 32 % 8}, j={ks[r] % 32}, g_idx={int(g[ks[r]])}, '
                     f'g_idx[k^1]={int(g[ks[r] ^ 1])}) n={n}, call {r // M}')
        for i, kind in enumerate(kinds):
            x = inputs(kind, M, K, seed=M + 10 * i)
            what = f'forward {kind} bits={bits} act={act} gs={gs} K={K} N={N} M={M}'
            note(f'forward {kind}', check_sliced(_forward(ops, L, x), x, L.W, forward_depth(K), what))


# (bits, act, gs, K, N): each bit width and both g_idx forms at 7B shapes and 13B down_proj; x in {-1, 0, 1}
INTEGER_CASES = [(8, False, 128, 4096, 12288), (8, True, 128, 11008, 4096), (3, False, 1024, 11008, 4096), (3, True, 1024, 4096, 11008),
                 (4, True, 1024, 13824, 5120)]


@pytest.mark.parametrize('bits,act,gs,K,N', INTEGER_CASES)
def test_forward_integer_grid_is_exact(ops, routes, bits, act, gs, K, N):
    L = pow2_layer(K, N, bits, gs, act, seed=K + bits)
    for M in (1, 3, 8, BATCHED_M):
        assert_route(routes, f'forward {bits} {act} {gs} M={M}', generic(bits, M))
        x = X.int_x(M, K, -1, 1, seed=M).cuda()
        what = f'integer grid bits={bits} act={act} gs={gs} K={K} N={N} M={M}'
        out = _forward(ops, L, x)
        assert_equal(out, fp16_from_fp64(X.exact_product(x, L.W)).cuda(), what, lambda m, n: f'm={m} n={n}')


DUAL_CASES, DUAL_M = [(8, False), (3, True)], (1, 3, 5, 8, BATCHED_M)


@pytest.mark.parametrize('bits,act', DUAL_CASES)
def test_fused_mlp_at_7b_gate_up(ops, routes, bits, act):
    """The DUAL instance at 4096 -> 11008, gate and up sharing their act-order map (as they do in a checkpoint): one-hot rows within one
    fp16 ulp of fp16(silu(a) * b) evaluated in fp64 (the epilogue runs in fp32), random inputs within check_swiglu_fp64_bound."""
    K, N, gs = 4096, 11008, 128
    for M in DUAL_M:
        assert_route(routes, f'dual {bits} {act} M={M}', generic(bits, M, True))
    G = Layer(O.random_packed(K, N, bits, gs, act_order=act, seed=1)[:4], bits, gs, act)
    qw, s, qz, _, _ = O.random_packed(K, N, bits, gs, act_order=act, seed=2)
    U = Layer((qw, s, qz, G.cpu[3]), bits, gs, act)
    fn = lambda x: ops.fused_mlp(x, G.dev, U.dev, bits, G.hint)
    ks0 = generic_ks(G, seed=3)
    for M in (1, 3, 8):
        ks = cyclic(ks0, M)
        x, mult = onehot3(ks, K, salt=M)
        x = x.cuda()
        what = f'fused mlp one-hot bits={bits} act={act} M={M}'
        out = torch.cat([fn(x[c * M:(c + 1) * M]) for c in range(len(ks) // M)])
        kt = torch.as_tensor(ks, device='cuda')
        a = G.W.index_select(0, kt).double() * mult.cuda()[:, None]
        b = U.W.index_select(0, kt).double() * mult.cuda()[:, None]
        d = fp16_ulp_distance(out.cpu(), fp16_from_fp64(a * torch.sigmoid(a) * b))
        assert int(d.max()) <= 1, f'{what}: {int((d > 1).sum())} outputs more than 1 ulp off, first at row {int(torch.nonzero(d > 1)[0, 0])}'
    for M in (1, 5, BATCHED_M):
        x = inputs('randn', M, K, seed=M)
        what = f'fused mlp bits={bits} act={act} M={M}'
        out = fn(x)
        note('fused mlp', check_swiglu_fp64_bound(out, x, G.W, U.W, what, depth=forward_depth(K)))


# ============================================================================= 3. transposed generic kernel
# (bits, act, gs, K, N): 8-bit at the 7B linears (one act-order), stored 3-bit and act-order 2-bit (the forms QuantLinear keeps when it
# has no kernel form: gs 1024 on K = 11008 has unequal groups)
TRANSPOSE_CASES = [(8, False, 128, 4096, 12288), (8, False, 128, 11008, 4096), (8, True, 128, 4096, 11008), (3, False, 1024, 4096, 4096),
                   (2, True, 1024, 11008, 4096)]
TRANSPOSE_M = (9, 100, 300)


@pytest.mark.parametrize('bits,act,gs,K,N', TRANSPOSE_CASES)
def test_transpose_at_llama_shapes(ops, routes, bits, act, gs, K, N):
    """One-hot gradient rows g[r] = 3 * 2^e * e_n return column n of W, rounded once, at every n of the first two 256-column rounds of
    the lanes and warps, the last round and random n; random and heavy-tailed gradients within the bound of depth transpose_depth(N)."""
    for M in TRANSPOSE_M:
        assert_route(routes, f'transpose {bits} {act} {gs} M={M}', generic_t(bits))
    L = layer(K, N, bits, gs, act, seed=K + N + bits + act)
    Wt = L.W.t().contiguous()
    fn = lambda gin: ops.transpose_matmul248(gin, *L.dev, bits, None, groupsize=L.hint)
    ns0 = sorted(set(range(512)) | set(range(N - 256, N)) | set(torch.randint(0, N, (64, ), generator=torch.Generator().manual_seed(N)).tolist()))
    for M in TRANSPOSE_M:
        ns = cyclic(ns0, M)
        gin, mult = onehot3(ns, N, salt=M)
        gin = gin.cuda()
        what = f'transpose one-hot bits={bits} act={act} gs={gs} K={K} N={N} M={M}'
        out = torch.cat([fn(gin[c * M:(c + 1) * M]) for c in range(len(ns) // M)])
        assert_equal(out, onehot3_expect(Wt, ns, mult), what, lambda r, k: f'row {r} n={ns[r]} k={k} (g_idx {int(L.cpu[3][k])})')
        for i, kind in enumerate(('randn', 'heavy')):
            gr = inputs(kind, M, N, seed=M + i)
            what = f'transpose {kind} bits={bits} act={act} gs={gs} K={K} N={N} M={M}'
            note('transpose', check_sliced(fn(gr), gr, Wt, transpose_depth(N), what))


# ============================================================================= 4. the gridDim.y chunk loops
CHUNK_K, CHUNK_N = 256, 64
FWD_CHUNK = 65535 * 4  # rows per launch of the MB = 4 instantiation
T_CHUNK = 65535 * 2    # rows per launch of the transposed kernel
SENTINEL = 0x7E5A      # a NaN bit pattern in the rows past M


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _sentinel_buffer(rows, cols):
    return torch.full((rows, cols), SENTINEL, dtype=torch.int16, device='cuda').view(torch.float16)


def _place_onehots(x, rows, salt):
    """Overwrite rows `rows` of x with distinct one-hot rows; returns (ks, mult)."""
    ks = [(37 * i + salt) % x.shape[1] for i in range(len(rows))]
    oh, mult = onehot3(ks, x.shape[1], salt=salt)
    x[torch.as_tensor(rows, device=x.device)] = oh.cuda()
    return ks, mult


def _check_chunked(out, x, W, M, rows, ks, mult, depth, what):
    """rows (one-hot) exactly; every row < M within the fp64 bound, in slices of rows; every row >= M still the sentinel."""
    assert_equal(out[torch.as_tensor(rows, device='cuda')], onehot3_expect(W, ks, mult), what, lambda i, n: f'row {rows[i]} n={n}')
    worst = 0.0
    for r0 in range(0, M, 65536):
        r1 = min(r0 + 65536, M)
        worst = max(worst, check_fp64_bound(out[r0:r1], x[r0:r1], W, what=f'{what} rows {r0}:{r1}', depth=depth,
                                            locate=lambda m, n, r0=r0: f'row {r0 + m} n={n}'))
    tail = out[M:].view(torch.int16)
    assert bool((tail == SENTINEL).all()), f'{what}: rows past M were written'
    return worst


CHUNK_CASES = [(8, False), (3, True)]


@pytest.mark.parametrize('bits,act', CHUNK_CASES)
@pytest.mark.parametrize('M', [FWD_CHUNK, FWD_CHUNK + 1, FWD_CHUNK + 4])
def test_forward_chunk_loop(ops, routes, bits, act, M):
    """gptq_qlinear_fwd into an [M + 8, N] buffer whose every element starts as a NaN sentinel: M = 262140 (one full launch), 262141 (a
    second launch of one row), 262144 (of one row block)."""
    from gptq_b200._lib import check, lib
    L = layer(CHUNK_K, CHUNK_N, bits, 64, act, seed=bits)
    x = inputs('randn', M, CHUNK_K, seed=M)
    rows = sorted({0, 1, 2, 3, 4, 65535, 131071, FWD_CHUNK - 4, FWD_CHUNK - 1} | {r for r in (FWD_CHUNK, FWD_CHUNK + 1, M - 2, M - 1) if r < M})
    ks, mult = _place_onehots(x, rows, salt=M)
    out = _sentinel_buffer(M + 8, CHUNK_N)
    w = ops.make_qweight(*L.dev, bits, L.hint)
    call = lambda: check(lib.gptq_qlinear_fwd(x.data_ptr(), CHUNK_K, ctypes.byref(w), None, out.data_ptr(), CHUNK_N, M, None, 0, _stream()))
    what = f'forward chunk loop bits={bits} act={act} M={M}'
    assert_route(routes, f'forward chunk {bits} {act}', generic(bits, M))
    call()
    note('forward chunk loop', _check_chunked(out, x, L.W, M, rows, ks, mult, forward_depth(CHUNK_K), what))


@pytest.mark.parametrize('M', [T_CHUNK, T_CHUNK + 1, T_CHUNK + 2])
def test_transpose_chunk_loop(ops, routes, M):
    """gptq_qlinear_transpose_fwd, 8-bit, into an [M + 8, K] sentinel buffer: M = 131070 (one full launch), 131071 and 131072 (one
    gradient row of 64 x 2048 tokens per row: a fine-tuning batch)."""
    from gptq_b200._lib import check, lib
    L = layer(CHUNK_K, CHUNK_N, 8, 64, False, seed=8)
    Wt = L.W.t().contiguous()
    g = inputs('randn', M, CHUNK_N, seed=M)
    rows = sorted({0, 1, 2, 32767, 32768, 65535, T_CHUNK - 2, T_CHUNK - 1} | {r for r in (T_CHUNK, M - 1) if r < M})
    ns, mult = _place_onehots(g, rows, salt=M)
    out = _sentinel_buffer(M + 8, CHUNK_K)
    w = ops.make_qweight(*L.dev, 8, L.hint)
    call = lambda: check(lib.gptq_qlinear_transpose_fwd(g.data_ptr(), CHUNK_N, ctypes.byref(w), out.data_ptr(), CHUNK_K, M, _stream()))
    what = f'transpose chunk loop M={M}'
    assert_route(routes, 'transpose chunk', generic_t(8))
    call()
    note('transpose chunk loop', _check_chunked(out, g, Wt, M, rows, ns, mult, transpose_depth(CHUNK_N), what))


# ============================================================================= 5. the engine on the generic kernels
# name -> (size, bits, act, gs): every linear of these models reaches the generic kernel (8-bit; act-order at gs 1024, where down_proj's
# groups are unequal and the whole model keeps its stored form)
ENGINE_MODELS = {'7b-int8-g128': ('7b', 8, False, 128), '7b-int4-act-g1024': ('7b', 4, True, 1024), '13b-int3-act-g1024': ('13b', 3, True, 1024)}
VOCAB = 32000
MAX_SEQ = 2048


def _model(name, n_layers=2, max_seq=MAX_SEQ, **kw):
    from gptq_b200 import engine
    size, bits, act, gs = ENGINE_MODELS[name]
    dec = engine.synthetic_llama(size, bits=bits, groupsize=gs, act_order=act, vocab=VOCAB, seed=bits + 10 * act, max_seq=max_seq, n_layers=n_layers,
                                 use_graph=False, **kw)
    if bits == 8:
        # synthetic_llama draws the scales of an int4 layer (U(1e-3, 1.1e-2)); |w - z| of an 8-bit layer spans 16 times the integer range, so
        # a real 8-bit layer of the same weight magnitudes has 16 times smaller scales.  Unscaled, the 7B activations overflow fp16 in
        # the first MLP.  The multiply is exact (every scale stays above 2^-14) and in place: the engine reads these very tensors.
        for ly in dec.layers:
            for k in ('qkv', 'o', 'gate', 'up', 'down'):
                ly[k].scales.mul_(2.0**-4)
    return dec


def probe_routes():
    """Runs in a process of its own (python tests/test_gpu_cuda_core_kernels.py), so that the activity tracer is never attached to the pytest
    process (once it has been, the CUDA-graph and cooperative-launch tests that run later in that process leave it dropping kernel records).
    Prints one JSON line: 'kernels': {request label: [kernel names]} for every request class of the kernel tests above (bits, g_idx form,
    groupsize, M; at the 7B o_proj shape, and the chunk-loop sizes at K = 256, N = 64) and the int8 down_proj backward; and per engine
    model {'launches', 'perms_none', 'step': one decode step, and for the 7B int8 model 'extend' / 'score': a 29-row extend and a 23-token
    score}."""
    from gptq_b200 import ops
    out = {'kernels': {}}

    def trace(fn):
        fn()  # first launch (module load) outside the trace
        for _ in range(3):  # a trace without any kernel record is taken again, as in gpu_util.run_kernel
            _, names = launched_kernels(fn)
            names = sorted(n for n in names if not n.startswith(('Memcpy', 'Memset')))
            if names:
                return names
        return []

    def packed(K, N, bits, gs, act, seed=0):
        return tuple(t.cuda() for t in O.random_packed(K, N, bits, gs, act_order=act, seed=seed)[:4])

    kern = out['kernels']
    for bits, act, gs in sorted({c[:3] for c in FORWARD_CASES + INTEGER_CASES}):
        w = packed(4096, 4096, bits, gs, act)
        for M in SMALL_M + (BATCHED_M, ):
            x = inputs('randn', M, 4096, seed=M)
            kern[f'forward {bits} {act} {gs} M={M}'] = trace(lambda: ops.matmul248(x, *w, bits, None, groupsize=0 if act else gs))
    for bits, act in DUAL_CASES:
        gw, uw = packed(4096, 4096, bits, 128, act, seed=1), packed(4096, 4096, bits, 128, act, seed=2)
        uw = uw[:3] + gw[3:]
        for M in DUAL_M:
            x = inputs('randn', M, 4096, seed=M)
            kern[f'dual {bits} {act} M={M}'] = trace(lambda: ops.fused_mlp(x, gw, uw, bits, 0 if act else 128))
    for bits, act, gs in sorted({c[:3] for c in TRANSPOSE_CASES}):
        w = packed(4096, 4096, bits, gs, act)
        for M in TRANSPOSE_M:
            gr = inputs('randn', M, 4096, seed=M)
            kern[f'transpose {bits} {act} {gs} M={M}'] = trace(lambda: ops.transpose_matmul248(gr, *w, bits, None, groupsize=0 if act else gs))
    for bits, act in CHUNK_CASES:
        w = packed(CHUNK_K, CHUNK_N, bits, 64, act)
        x = inputs('randn', FWD_CHUNK + 1, CHUNK_K, seed=1)
        kern[f'forward chunk {bits} {act}'] = trace(lambda: ops.matmul248(x, *w, bits, None, groupsize=0 if act else 64))
    w = packed(CHUNK_K, CHUNK_N, 8, 64, False)
    gr = inputs('randn', T_CHUNK + 1, CHUNK_N, seed=1)
    kern['transpose chunk'] = trace(lambda: ops.transpose_matmul248(gr, *w, 8, None, groupsize=64))
    del x, gr, w

    ql, _, go = _int8_down_proj()
    w = ql.weights()  # the request QuantLinearFunction.backward makes (test_int8_quant_linear_backward_at_down_proj checks it does)
    kern['int8 backward'] = trace(lambda: ops.transpose_matmul248(go, *w.parts(), w.bits, None, groupsize=w.hint))
    del ql, go, w
    for name in ENGINE_MODELS:
        dec = _model(name, max_seq=64)
        rec = {'launches': dec.launches_per_step(), 'perms_none': all(p is None for pm in dec.perms for p in pm.values())}
        dec.tokens.fill_(7)
        dec.positions.fill_(3)
        rec['step'] = trace(dec.step)
        if name == '7b-int8-g128':
            ids = list(range(100, 129))

            def extend():
                dec.reset()
                return dec.extend([ids])

            rec['extend'] = trace(extend)
            rec['score'] = trace(lambda: dec.score([ids[:23]]))
        out[name] = rec
        del dec
        torch.cuda.empty_cache()
    print('ROUTES ' + json.dumps(out))


@pytest.fixture(scope='module')
def routes():
    res = subprocess.run([sys.executable, os.path.abspath(__file__)], capture_output=True, text=True, timeout=900)
    assert res.returncode == 0, f'the routing probe failed:\n{res.stdout[-2000:]}\n{res.stderr[-4000:]}'
    return json.loads([line for line in res.stdout.splitlines() if line.startswith('ROUTES ')][-1][7:])


def assert_route(routes, label, kernel):
    """The request class `label` launched `kernel` (a demangled name with its template arguments) and no other quantized-linear kernel.  A trace
    without the kernel's record is reported, not failed: the numeric checks of the test still run."""
    q = _quantized(routes['kernels'][label])
    if not q:
        print(f'  {label}: no kernel record in the trace')
        return
    assert all(kernel.replace(' ', '') in n.replace(' ', '') for n in q), f'{label}: expected {kernel}, launched {q}'


def _quantized(names):
    fam = ('qmatvec_int4_kernel', 'qgemm_wgmma_kernel', 'qgemm_wgmma_t_kernel', 'qlinear_generic_kernel', 'qlinear_transpose_generic_kernel')
    return [n for n in names if any(f + '<' in n for f in fam)]


@pytest.mark.parametrize('name', list(ENGINE_MODELS))
def test_engine_route(routes, name):
    """Every model decodes on the kernel chain, act-order layers in their stored form (the gs-1024 fallback: kernel_form refuses down_proj's
    unequal groups, the persistent kernel cannot take the stored act-order layer, and LlamaDecoder drops the regrouping of the others), and
    every quantized linear of the step runs on the generic kernel of the model's bit width."""
    bits = ENGINE_MODELS[name][1]
    r = routes[name]
    assert r['launches'] > 1 and r['perms_none'], r
    step = r['step']
    if not step:
        pytest.skip(f'{name}: the trace of the decode step had no kernel records')
    assert not any('qmatvec_int4_kernel' in n or 'llama_decode_mega_kernel' in n for n in step), step
    q = _quantized(step)
    strip = lambda s: s.replace(' ', '')
    assert q and all(strip(f'qlinear_generic_kernel<{bits},1,') in strip(n) for n in q), q
    assert any(strip(generic(bits, 1, True)) in strip(n) for n in q) and any(strip(generic(bits, 1)) in strip(n) for n in q), q


def test_batched_passes_of_the_int8_model_run_on_the_generic_kernel(routes):
    strip = lambda s: s.replace(' ', '')
    for what in ('extend', 'score'):
        q = _quantized(routes['7b-int8-g128'][what])
        if not q:
            pytest.skip(f'{what}: the trace had no kernel records')
        assert {strip(n[n.index('qlinear'):n.index('>') + 1]) for n in q} == {strip(generic(8, 29 if what == 'extend' else 23)),
                                                                                strip(generic(8, 29, True))}, (what, q)


def _rope64(k, pos, base=10000.0):
    """k fp16 [heads, 128] rotated in float64 (rotate_half: x' = x cos - y sin, y' = x sin + y cos, y at +64)."""
    k = k.double()
    half = k.shape[-1] // 2
    f = pos * torch.pow(torch.tensor(base, dtype=torch.float64), -2.0 * torch.arange(half, dtype=torch.float64, device=k.device) / k.shape[-1])
    c, s = torch.cos(f), torch.sin(f)
    x, y = k[..., :half], k[..., half:]
    return torch.cat([x * c - y * s, x * s + y * c], -1)


@pytest.mark.parametrize('name', list(ENGINE_MODELS))
def test_engine_decode_on_the_generic_kernels(ops, name):
    """Batch 1 at positions {0, 255, 256, 2047} and batch 8 at those positions, on a random KV cache.  The layer-0 V rows equal the V columns
    of ops.matmul248(ops.rmsnorm(embedding rows), qkv) bit for bit (the same generic kernel instance at the same M), the K rows are within
    KV_ROW_TOL of a float64 RoPE of that product; the logits of the 1-layer model (input: the embedding row, known exactly) and of the
    2-layer model are within the block and end-to-end bounds of tests/llama_oracle.py against the oracle; next_tokens is the
    argmax."""
    from gptq_b200 import engine
    base = _model(name)
    oracle = LlamaOracle.from_decoder(base, eps=1e-6, base=10000.0)
    eps = base.model.rms_eps
    H, nh, hd = base.hidden, base.n_heads, base.head_dim
    for B, positions in ((1, [0, 255, 256, 2047]), (8, [0, 255, 256, 2047, 2047, 256, 255, 0])):
        decs = {n: engine.LlamaDecoder(base.layers[:n], base.embed, base.final_norm, base.lm_head, nh, batch=B, max_seq=MAX_SEQ, use_graph=False)
                for n in (1, 2)}
        for n, dec in decs.items():
            assert dec.launches_per_step() > 1 and all(p is None for pm in dec.perms for p in pm.values()), f'{name}: not on the kernel chain'
        gen = torch.Generator(device='cuda').manual_seed(B)
        kc_dev = (torch.randn(decs[2].k_cache.shape, device='cuda', generator=gen) * 0.5).half()
        vc_dev = (torch.randn(decs[2].v_cache.shape, device='cuda', generator=gen) * 0.5).half()
        kc, vc = kc_dev.cpu(), vc_dev.cpu()
        q0 = decs[2].klayers[0]['qkv']
        steps = [[(b, p) for b, p in enumerate(positions)]] if B == 8 else [[(0, p)] for p in positions]
        for si, step in enumerate(steps):
            pos = [p for _, p in step]
            toks = [(101 * (si + b) + 3 * p + 7) % VOCAB for b, p in step]
            for n, dec in decs.items():
                dec.k_cache.copy_(kc_dev[:n])
                dec.v_cache.copy_(vc_dev[:n])
                dec.tokens.copy_(torch.tensor(toks, dtype=torch.int32))
                dec.positions.copy_(torch.tensor(pos, dtype=torch.int32))
                dec.step()
            torch.cuda.synchronize()
            what = f'{name} B={B} positions={pos}'
            qkv = ops.matmul248(ops.rmsnorm(base.embed[torch.tensor(toks, device='cuda')], decs[2].klayers[0]['input_norm'], eps), *q0.parts(), q0.bits,
                                groupsize=q0.hint)
            for b, p in step:
                v_row = decs[2].v_cache[0, b, :, p]
                v_want = qkv[b, 2 * H:].view(nh, hd)
                assert torch.equal(v_row.view(torch.int16), v_want.reshape(nh, hd).contiguous().view(torch.int16)), \
                    f'{what}: layer-0 V row of sequence {b} differs from the product in {int((v_row != v_want).sum())} elements'
                check(decs[2].k_cache[0, b, :, p], _rope64(qkv[b, H:2 * H].view(nh, hd), p), KV_ROW_TOL, f'{what}: layer-0 K row of sequence {b}')
                x = base.embed[toks[b]].cpu()[None, :].clone()
                refs = []
                for li in range(2):
                    x = oracle.mlp(li, oracle.attention(li, x, p, kc[li, b], vc[li, b])[0])
                    refs.append(oracle.head(x)[0])
                check(decs[1].logits[b], refs[0], MLP_HEAD_TOL, f'{what}: logits of sequence {b} after 1 layer')
                check(decs[2].logits[b], refs[1], END_TO_END_TOL, f'{what}: logits of sequence {b} after 2 layers, end to end')
                for n, dec in decs.items():
                    assert int(dec.next_tokens[b]) == int(dec.logits[b].float().argmax()), f'{what}: greedy token of sequence {b}, {n} layers'
        del decs
        torch.cuda.empty_cache()
    assert_no_failures()


def test_extend_of_the_int8_model_matches_stepping():
    """7B int8: 1791 chain steps, extend() of the next 256 tokens (the ragged pass on qlinear_generic_kernel<8, 4, ...>, see
    test_batched_passes_of_the_int8_model_run_on_the_generic_kernel), one step; against stepping all of them.  Cache rows and logits within
    the run-to-run spread bounds of tests/test_gpu_extend.py (max 1.5e-2, rms 3e-3 of the rms)."""
    dec = _model('7b-int8-g128')
    toks = torch.randint(0, VOCAB, (2048, ), generator=torch.Generator().manual_seed(3)).tolist()
    check_extend_against_stepping(dec, toks, 1791, '7b int8 extend vs stepping')


def test_score_of_the_int8_model_matches_the_oracle():
    """Three lists in one score() call against float64 log-softmaxes of the oracle's fp16 logits, at the bound of tests/test_gpu_score.py:
    2 x 2e-2 x max|ref logits| per element."""
    dec = _model('7b-int8-g128', max_seq=16)
    g = torch.Generator().manual_seed(8)
    seqs = [torch.randint(0, VOCAB, (n, ), generator=g).tolist() for n in (9, 2, 23)]
    out = dec.score(seqs)
    note('score 7b int8', check_scores(out, seqs, LlamaOracle.from_decoder(dec, eps=1e-6, base=10000.0), 'score 7b int8'))


def _int8_down_proj(M=300):
    """An 8-bit QuantLinear at down_proj's shape (11008 -> 4096) on the device, an input that requires grad and an output gradient."""
    import quant
    K, N, gs = 11008, 4096, 128
    ql = quant.QuantLinear(8, gs, K, N, False)
    ql.qweight, ql.scales, ql.qzeros, ql.g_idx = O.random_packed(K, N, 8, gs, seed=9)[:4]
    return ql.cuda(), inputs('randn', M, K, seed=1).requires_grad_(True), inputs('randn', M, N, seed=2)


def test_int8_quant_linear_backward_at_down_proj(ops, routes):
    """M = 300: the backward makes one 8-bit transposed request with the groupsize hint, which runs on qlinear_transpose_generic_kernel<8, 2>
    (routing probe), and x.grad is within the transposed bound of the fp64 product go . W^T, W = ops.dequant of the stored tensors (pinned
    to the oracle above)."""
    assert_route(routes, 'int8 backward', generic_t(8))
    ql, x, go = _int8_down_proj()
    N = ql.outfeatures
    Wt = ops.dequant(ql.qweight, ql.scales, ql.qzeros, ql.g_idx, 8, ql.groupsize).t().contiguous()
    out = ql(x)
    with recorded_transposes() as rec:
        grad = torch.autograd.grad(out, x, go)[0]
    assert len(rec.calls) == 1, rec.calls
    args, kw = rec.calls[0]
    assert args[0].shape == go.shape and args[5] == 8 and kw.get('groupsize') == ql.groupsize, (args[5], kw)
    assert grad.dtype == torch.float16 and grad.shape == x.shape
    note('int8 QuantLinear backward', check_sliced(grad, go, Wt, transpose_depth(N), 'int8 QuantLinear backward at down_proj'))


if __name__ == '__main__':
    probe_routes()
