"""GPU: bit-exact probes of every quantized-linear kernel (split-K matvec, wgmma GEMM, fused MLP, generic, transposed).

The inputs (tests/exact_fixtures.py) have answers that do not depend on the summation order, so the kernels are compared with
torch.equal against the oracle's fp16 weight (O.dequant, built on the CPU):
  * one-hot rows give out[r] = fp16(sign * 2^e * W[k_r]) (+ bias): every dequantised weight the kernel feeds its tensor cores
    is pinned to the reference's fp16(fp16(q - z) * s), at every k of a k-loop, and the k order of the staging is pinned to it;
  * integer-exact fixtures at LLaMA-7B shapes give out = fp16(exact sum): the split-K partials, the last-arriver reduction, the
    wgmma tiles and every epilogue mapping must round the one correct fp32 value.
The fused SwiGLU epilogue evaluates silu(a) * b in fp32 (expf), so it is held to 1 fp16 ulp of the fp64 value instead.
Every case asserts which kernel served it (gpu_util.run_kernel)."""
from functools import lru_cache

import pytest
import torch

import exact_fixtures as X
from gpu_util import GEMM_1, GEMM_2, GEMM_DUAL, MATVEC, MATVEC_DUAL, Layer, assert_equal, cyclic, fp16_from_fp64, fp16_ulp_distance, generic, ops, \
    run_kernel

pytestmark = pytest.mark.gpu

def gemm_kernel(M):
    return GEMM_2 if M > 128 else GEMM_1


@lru_cache(maxsize=None)
def random_layer(K, N, bits, gs, act=False, bias=False, seed=0):
    return Layer.random(K, N, bits, gs, act, bias, seed)


@lru_cache(maxsize=None)
def pow2_layer(K, N, gs, jmin=6, seed=0):
    return Layer(X.pow2_packed(K, N, gs, jmin=jmin, seed=seed), 4)


def assert_ulp1(out, ref_fp64, what, locate):
    """out (fp16) within one fp16 ulp of the fp64 value rounded once to fp16."""
    d = fp16_ulp_distance(out.cpu(), fp16_from_fp64(ref_fp64))
    if int(d.max()) <= 1:
        return
    r, n = (int(i) for i in torch.nonzero(d > 1)[0])
    raise AssertionError(f'{what}: {int((d > 1).sum())} outputs more than 1 ulp off (max {int(d.max())}); first at {locate(r, n)}: '
                         f'got {out[r, n].item()!r}, want {ref_fp64[r, n].item()!r}')


def batched_calls(fn, x, M, kernel, what):
    """fn(x[c*M:(c+1)*M]) for every chunk of M rows, concatenated; the first call asserts the kernel."""
    outs = []
    for c in range(x.shape[0] // M):
        xc = x[c * M:(c + 1) * M]
        outs.append(run_kernel(lambda: fn(xc), kernel, what) if c == 0 else fn(xc))
    return torch.cat(outs)


# ============================================================================= one-hot rows: every path
@pytest.mark.parametrize('K,N,bias', [(512, 4096, False), (512, 4096 + 96, True), (4096, 4096, True), (4096, 4096 + 96, False),
                                      (11008, 4096, False)])
def test_matvec_onehot_reproduces_every_weight(ops, K, N, bias):
    """M = 1..8: each row of a call probes a different k, so every epilogue row mapping (m = 2t + h), the x-row clamp for g >= M
    and the k-permuted x staging are pinned.  K = 512: every k.  7B shapes: every k % 8, both sides of each group boundary, and
    the first / last k of the CTA ranges (split K over two slabs per CTA, last-arriver reduction)."""
    gs = 128
    L = random_layer(K, N, 4, gs, bias=bias, seed=K + N)
    ks0 = range(K) if K <= 512 else X.sampled_ks(K, gs, X.matvec_cta_ks(K, N), seed=K)
    for M in range(1, 9):
        ks = cyclic(ks0, M)
        x, mult = X.onehot_rows(ks, K, salt=M)
        what = f'matvec one-hot K={K} N={N} M={M} bias={bias}'
        out = batched_calls(lambda xc: ops.matmul248(xc, *L.dev, 4, 15, bias=L.bias, groupsize=gs), x.cuda(), M, MATVEC, what)
        exp = X.onehot_expect(L.W, ks, mult, L.bias)
        assert_equal(out, exp, what, lambda r, n: X.matvec_where(K, N, gs, r % M, n, ks[r]) + f', call {r // M}')


@pytest.mark.parametrize('K,M,N,gs,bias', [(128, 128, 384, 64, True), (128, 129, 384, 64, False), (512, 512, 256, 128, False),
                                           (512, 513, 256, 128, True), (256, 256, 128, 256, False)])
def test_wgmma_onehot_reproduces_the_whole_weight(ops, K, M, N, gs, bias):
    """x = diag(sign * 2^e) (M = K; M = K + 1 repeats the last k in a ragged last tile): out is the whole dequantised weight,
    through the 128-byte swizzle of the B tile and the TMA-staged A tile."""
    L = random_layer(K, N, 4, gs, bias=bias, seed=M + N)
    ks = list(range(K)) + [K - 1] * (M - K)
    x, mult = X.onehot_rows(ks, K)
    what = f'wgmma one-hot M={M} K={K} N={N} gs={gs}'
    out = run_kernel(lambda: ops.matmul248(x.cuda(), *L.dev, 4, 15, bias=L.bias, groupsize=gs), gemm_kernel(M), what)
    assert_equal(out, X.onehot_expect(L.W, ks, mult, L.bias), what, lambda r, n: X.gemm_where(M, K, gs, r, n, ks[r]))


def _silu_mul_fp64(Wg, Wu, ks, mult):
    ks = torch.as_tensor(ks, device=Wg.device)
    a = Wg.index_select(0, ks).double() * mult.to(Wg.device)[:, None]
    b = Wu.index_select(0, ks).double() * mult.to(Wg.device)[:, None]
    return a * torch.sigmoid(a) * b


@pytest.mark.parametrize('K,N,M', [(512, 1024, 1), (512, 1024, 3), (512, 1024, 8), (256, 384, 256), (128, 256, 129)])
def test_fused_mlp_onehot(ops, K, N, M):
    """a and b are single exact weights, so fp16(silu(a) * b) is known to within the fp32 epilogue: <= 1 fp16 ulp of fp64."""
    gs = 64
    G, U = random_layer(K, N, 4, gs, seed=1), random_layer(K, N, 4, gs, seed=2)
    ks = cyclic(range(K), M)
    x, mult = X.onehot_rows(ks, K, salt=3)
    kernel = MATVEC_DUAL if M <= 8 else GEMM_DUAL
    what = f'fused mlp one-hot K={K} N={N} M={M}'
    out = batched_calls(lambda xc: ops.fused_mlp(xc, G.dev, U.dev, 4, gs), x.cuda(), M, kernel, what)
    where = (lambda r, n: X.matvec_where(K, N, gs, r % M, n, ks[r])) if M <= 8 else (lambda r, n: X.gemm_where(M, K, gs, r, n, ks[r], dual=True))
    assert_ulp1(out, _silu_mul_fp64(G.W, U.W, ks, mult), what, where)


@pytest.mark.parametrize('bits,act', [(2, False), (3, False), (8, False), (4, True), (3, True), (8, True)])
@pytest.mark.parametrize('M', [1, 2, 5, 17])
def test_generic_onehot(ops, bits, act, M):
    """The CUDA-core kernel for every bit width, with the groupsize hint or the act-order g_idx gather."""
    K, N, gs = 256, 96, 64
    L = random_layer(K, N, bits, gs, act=act, bias=True, seed=bits + 10 * act)
    ks = cyclic(range(K), M)
    x, mult = X.onehot_rows(ks, K, salt=bits)
    what = f'generic one-hot bits={bits} act={act} M={M}'
    out = batched_calls(lambda xc: ops.matmul248(xc, *L.dev, bits, None, bias=L.bias, groupsize=0 if act else gs), x.cuda(), M,
                        generic(bits, M), what)
    g = L.cpu[3]
    assert_equal(out, X.onehot_expect(L.W, ks, mult, L.bias), what,
                 lambda r, n: f'm={r % M} k={ks[r]} (k%8={ks[r] % 8}, g_idx={int(g[ks[r]])}) n={n}')


@pytest.mark.parametrize('bits', [2, 3, 4, 8])
def test_transpose_onehot_returns_columns(ops, bits):
    """g[r] = sign * 2^e * e_{n_r}: out[r] = the whole column n_r of W (act-order g_idx)."""
    K, N, gs = 256, 96, 64
    L = random_layer(K, N, bits, gs, act=True, seed=bits)
    ns = list(range(N)) + [N - 1]  # 97 rows: a ragged last row pair
    gin, mult = X.onehot_rows(ns, N, salt=bits)
    what = f'transpose one-hot bits={bits}'
    out = run_kernel(lambda: ops.transpose_matmul248(gin.cuda(), *L.dev, bits, None), f'qlinear_transpose_generic_kernel<{bits}, 2>', what)
    exp = X.onehot_expect(L.W.t().contiguous(), ns, mult)
    assert_equal(out, exp, what, lambda r, k: f'row {r} n={ns[r]} k={k} (k%8={k % 8}, g_idx={int(L.cpu[3][k])})')


@pytest.mark.parametrize('bits,act', [(4, True), (3, True), (3, False), (2, False)])
def test_qlayer_kernel_form_onehot(ops, bits, act):
    """Layers served through ops.QLayerWeights.kernel_form (act-order rows regrouped, 2/3-bit fields widened to int4): a one-hot at k' of the
    permuted basis must return the stored layer's row perm[k'], through the matvec (M = 8) and the wgmma GEMM (M = K)."""
    K, N, gs = 256, 256, 64
    L = random_layer(K, N, bits, gs, act=act, seed=20 + bits + act)
    qw, s, qz, g = L.dev
    stored = ops.QLayerWeights(qw, s, qz, g, bits, gs)
    kf = stored.kernel_form()
    assert kf is not stored and kf.bits == 4
    perm = kf.perm.cpu() if kf.perm is not None else torch.arange(K)
    assert not act or not torch.equal(perm, torch.arange(K))
    layer = (kf.qweight, s, kf.qzeros, kf.g_idx)
    for M, kernel in ((8, MATVEC), (K, gemm_kernel(K))):
        ks = cyclic(range(K), M)
        x, mult = X.onehot_rows(ks, K, salt=M)
        what = f'kernel_form one-hot bits={bits} act={act} M={M}'
        out = batched_calls(lambda xc: ops.matmul248(xc, *layer, 4, 15, groupsize=gs), x.cuda(), M, kernel, what)
        rows = perm[torch.tensor(ks)].tolist()
        assert_equal(out, X.onehot_expect(L.W, rows, mult), what, lambda r, n: f"m={r % M} k'={ks[r]} (stored row {rows[r]}) n={n}")


@pytest.mark.parametrize('M', [1, 5, 8, 129])
def test_onehot_partial_last_group(ops, M):
    """down_proj at gs 1024: K = 11008 = 10 x 1024 + 768, so the last of the 11 groups is partial.  One-hot rows at every k % 8, both
    sides of every group boundary (the last one at 10240 included), the first / last 64 k and the matvec's CTA-range edges, through the
    split-K matvec (M <= 8) and the wgmma GEMM (M = 129)."""
    K, N, gs = 11008, 4096, 1024
    L = random_layer(K, N, 4, gs, seed=K + gs)
    ks0 = X.sampled_ks(K, gs, X.matvec_cta_ks(K, N), seed=gs)
    assert {10239, 10240, K - 1} <= set(ks0)
    ks = cyclic(ks0, M)
    x, mult = X.onehot_rows(ks, K, salt=M)
    what = f'one-hot partial last group K={K} gs={gs} M={M}'
    fn = lambda xc: ops.matmul248(xc, *L.dev, 4, 15, groupsize=gs)
    if M <= 8:
        out = batched_calls(fn, x.cuda(), M, MATVEC, what)
        where = lambda r, n: X.matvec_where(K, N, gs, r % M, n, ks[r]) + f', call {r // M}'
    else:
        out = batched_calls(fn, x.cuda(), M, gemm_kernel(M), what)
        where = lambda r, n: X.gemm_where(M, K, gs, r % M, n, ks[r]) + f', call {r // M}'
    assert_equal(out, X.onehot_expect(L.W, ks, mult), what, where)


# ============================================================================= integer-exact sums at full size
SHAPES_7B = [(4096, 4096), (4096, 12288), (11008, 4096)]


@pytest.mark.parametrize('M', [1, 5, 8, 129, 512])
def test_integer_exact_partial_last_group(ops, M):
    """down_proj at gs 1024 (the last of 11 groups holds 768 k) and power-of-two scales per (group, column): out == fp16(exact) through
    the matvec (M <= 8) and the wgmma GEMM, so a scale or zero of the partial group read from the wrong row shows in every column."""
    K, N, gs = 11008, 4096, 1024
    L = pow2_layer(K, N, gs, seed=K + gs)
    assert L.cpu[1].shape[0] == 11
    x = X.int_x(M, K, -2, 2, seed=M).cuda()
    what = f'integer-exact partial last group K={K} gs={gs} M={M}'
    out = run_kernel(lambda: ops.matmul248(x, *L.dev, 4, 15, groupsize=gs), MATVEC if M <= 8 else gemm_kernel(M), what)
    exp = fp16_from_fp64(X.exact_product(x, L.W)).cuda()
    where = (lambda m, n: X.matvec_where(K, N, gs, m, n)) if M <= 8 else (lambda m, n: X.gemm_where(M, K, gs, m, n))
    assert_equal(out, exp, what, where)


@pytest.mark.parametrize('K,N', SHAPES_7B)
def test_matvec_integer_exact_full_size(ops, K, N):
    """M = 1..8 at the 7B shapes: every CTA spans two slabs, partials go through the workspace; out == fp16(exact) everywhere."""
    gs = 128
    L = pow2_layer(K, N, gs, seed=K + N)
    for M in range(1, 9):
        x = X.int_x(M, K, -2, 2, seed=M).cuda()
        what = f'matvec integer-exact K={K} N={N} M={M}'
        out = run_kernel(lambda: ops.matmul248(x, *L.dev, 4, 15, groupsize=gs), MATVEC, what)
        exp = fp16_from_fp64(X.exact_product(x, L.W)).cuda()
        assert_equal(out, exp, what, lambda m, n: X.matvec_where(K, N, gs, m, n))


@pytest.mark.parametrize('K,N', SHAPES_7B)
@pytest.mark.parametrize('M', [129, 512])
def test_wgmma_integer_exact_full_size(ops, K, N, M):
    gs = 128
    L = pow2_layer(K, N, gs, seed=K + N)
    x = X.int_x(M, K, -2, 2, seed=M).cuda()
    what = f'wgmma integer-exact M={M} K={K} N={N}'
    out = run_kernel(lambda: ops.matmul248(x, *L.dev, 4, 15, groupsize=gs), gemm_kernel(M), what)
    exp = fp16_from_fp64(X.exact_product(x, L.W)).cuda()
    assert_equal(out, exp, what, lambda m, n: X.gemm_where(M, K, gs, m, n))


@pytest.mark.parametrize('M', [1, 5, 8, 129, 300])
def test_fused_mlp_integer_exact_full_size(ops, M):
    """gate / up at (4096, 11008): x in {-1, 0, 1} and scales <= 2^-9 keep |a|, |b| <= 128 (no fp16 overflow of silu(a) * b);
    a and b are exact in fp32, so the output is within 1 fp16 ulp of fp16(silu(a) * b) evaluated in fp64."""
    K, N, gs = 4096, 11008, 128
    G, U = pow2_layer(K, N, gs, jmin=9, seed=1), pow2_layer(K, N, gs, jmin=9, seed=2)
    x = X.int_x(M, K, -1, 1, seed=M).cuda()
    what = f'fused mlp integer-exact M={M}'
    out = run_kernel(lambda: ops.fused_mlp(x, G.dev, U.dev, 4, gs), MATVEC_DUAL if M <= 8 else GEMM_DUAL, what)
    a, b = X.exact_product(x, G.W), X.exact_product(x, U.W)
    where = (lambda m, n: X.matvec_where(K, N, gs, m, n)) if M <= 8 else (lambda m, n: X.gemm_where(M, K, gs, m, n, dual=True))
    assert_ulp1(out, a * torch.sigmoid(a) * b, what, where)
