"""GPU: the tuned int4 kernels at their tile, ring and split edges, against an fp64 reference with an element-wise bound.

Random layers (O.random_packed) and randn activations; the reference is the fp64 product of the same fp16 inputs with the oracle's
fp16 weight, and every output must lie within ulp16 + depth * 2^-24 * (|x| . |W|) of it (gpu_util.check_fp64_bound), a bound that
a last-bit error per weight or a dropped / duplicated k-step cannot hide under, unlike a bound relative to rms(ref).  Every case
asserts which kernel served it: the tuned paths fall back to the generic kernel silently when an argument does not suit them.

  * wgmma GEMM: an explicit table over M (tile edges 128 / 256 / 384, ragged and fully out-of-bounds TMA boxes), K (1 and 3
    K steps, i.e. the prologue / tail guards of the TMA and register rings; 172 steps at 11008), N (1 .. 96 column tiles),
    groupsize (64, 128, K, and 1024 on K = 11008: a partial last group), bias and a strided activation, so that each instantiation
    meets every edge at least once;
  * split-K matvec: M = 1..8 at the 7B shapes (two slabs per CTA: workspace partials, last-arriver reduction), a ragged N and
    groupsizes 32 / 96 / 128 / K, and 1024 on K = 11008; after every call the workspace counters must be back to zero;
  * documented fallbacks (misaligned x, groupsize 32 or N = 96 at M > 8) must reach the generic kernel and still be right;
  * determinism: repeated calls, and a call between two shapes that share the workspace, give bit-identical results.
"""
from functools import lru_cache

import pytest
import torch

import exact_fixtures as X
from gpu_util import GEMM_1, GEMM_2, GEMM_DUAL, GENERIC_4, MATVEC, MATVEC_DUAL, Layer, WorstRatios, check_fp64_bound, check_swiglu_fp64_bound, ops, randn_x, \
    run_kernel

pytestmark = pytest.mark.gpu

WORST = WorstRatios()
note = WORST.note


@pytest.fixture(scope='module', autouse=True)
def worst_ratio_summary():
    yield
    WORST.summary()


@lru_cache(maxsize=None)
def layer(K, N, gs, bias=False, seed=0):
    return Layer.random(K, N, 4, gs, bias=bias, seed=seed)


def workspace_counters(ops, dev, N):
    """The slab counters at the head of the per-stream workspace (qmatvec.cu: rounded up to 256 B)."""
    ws = ops._workspaces[(dev.index, torch.cuda.current_stream(dev).cuda_stream)]
    nslabs = X.matvec_plan(32, N)[0]
    return ws[:(nslabs * 4 + 255) // 256 * 256]


# ============================================================================= wgmma GEMM
# (M, K, N, gs, bias, ldx): rows with M <= 128 run <false, 1, 6>, the others <false, 2, 4>.  Each instantiation meets every K, N, gs in
# {64, 128, K}, a partial last group (gs 1024 on K = 11008), bias on and off and a strided x at least once
# (test_wgmma_table_covers_every_edge_per_instantiation).
GEMM_TABLE = [
    (9, 64, 128, 64, True, None),         # 1 K step, gs = K, one column tile
    (64, 192, 384, 64, False, 192 + 64),  # 3 K steps (fewer than the B register ring and the TMA lookahead), strided x
    (127, 128, 4096, 128, True, None),    # gs = K = 128
    (128, 4096, 12288, 128, False, None),  # tile edge; N = qkv of the prefill benchmark
    (128, 11008, 4096, 64, True, 11008 + 64),  # down_proj: 172 K steps, 172 groups, strided
    (64, 4096, 4096, 4096, False, None),  # one group
    (9, 192, 128, 192, False, None),      # gs = K = 192: 3 K steps in one group
    (129, 64, 384, 64, True, None),       # first WT = 2 size: one row in the tile, its second TMA box entirely out of bounds
    (255, 192, 128, 64, False, 192 + 64),  # strided
    (256, 128, 4096, 128, False, None),   # exactly one 256-row tile, gs = K
    (257, 4096, 12288, 64, True, None),   # one row in the second tile; gs = 64 on WT = 2
    (384, 11008, 4096, 128, False, 11008 + 64),  # 1.5 tiles: the last tile's second box out of bounds; strided
    (1000, 4096, 4096, 4096, True, None),  # one group, ragged last tile
    (384, 192, 384, 192, True, None),     # gs = K = 192
    # down_proj at the groupsizes of published checkpoints: 1024 (11008 = 10 x 1024 + 768: a partial last group) and full (gs = K)
    (9, 11008, 4096, 1024, False, None),
    (128, 11008, 4096, 11008, True, None),
    (257, 11008, 4096, 1024, True, 11008 + 64),
    (1000, 11008, 4096, 11008, False, None),
]


@pytest.mark.parametrize('M,K,N,gs,bias,ldx', GEMM_TABLE)
def test_wgmma_gemm_edges(ops, M, K, N, gs, bias, ldx):
    L = layer(K, N, gs, bias, seed=K + N + gs)
    x = randn_x(M, K, seed=M, ld=ldx)
    assert ldx is None or (x.stride(0) == ldx and x.data_ptr() % 16 == 0)
    what = f'wgmma M={M} K={K} N={N} gs={gs} bias={bias} ldx={ldx or K}'
    kernel = GEMM_2 if M > 128 else GEMM_1
    out = run_kernel(lambda: ops.matmul248(x, *L.dev, 4, 15, bias=L.bias, groupsize=gs), kernel, what)
    ratio = check_fp64_bound(out, x, L.W, L.bias, what, locate=lambda m, n: X.gemm_where(M, K, gs, m, n))
    note(f'wgmma {kernel}', ratio)
    if gs in (1024, 11008):
        note('wgmma, K = 11008 at gs 1024 / 11008', ratio)


def test_wgmma_table_covers_every_edge_per_instantiation():
    for small in (True, False):
        rows = [r for r in GEMM_TABLE if (r[0] <= 128) == small]
        assert {r[1] for r in rows} == {64, 128, 192, 4096, 11008}
        assert {r[2] for r in rows} == {128, 384, 4096, 12288}
        assert {64, 128} <= {r[3] for r in rows} and any(r[3] == r[1] for r in rows)
        assert any(r[1] % r[3] for r in rows) and any(r[1] == r[3] == 11008 for r in rows)  # a partial last group; down_proj at gs = K
        assert {r[4] for r in rows} == {True, False} and any(r[5] for r in rows)
    assert {r[0] for r in GEMM_TABLE} == {9, 64, 127, 128, 129, 255, 256, 257, 384, 1000}


@pytest.mark.parametrize('M,K,gs', [(9, 64, 64), (9, 4096, 128), (128, 4096, 128), (129, 4096, 64), (300, 64, 64), (300, 4096, 128)])
def test_wgmma_fused_mlp_edges(ops, M, K, gs):
    N = 384 if K == 64 else 1024
    G, U = layer(K, N, gs, seed=1), layer(K, N, gs, seed=2)
    x = randn_x(M, K, seed=M)
    what = f'wgmma fused mlp M={M} K={K} N={N} gs={gs}'
    out = run_kernel(lambda: ops.fused_mlp(x, G.dev, U.dev, 4, gs), GEMM_DUAL, what)
    note('wgmma fused mlp', check_swiglu_fp64_bound(out, x, G.W, U.W, what, locate=lambda m, n: X.gemm_where(M, K, gs, m, n, dual=True)))


# ============================================================================= split-K matvec
MATVEC_SHAPES = [(4096, 4096), (4096, 12288), (11008, 4096), (4096, 4096 + 96), (256, 96)]
MATVEC_CASES = [(M, K, N, 128) for K, N in MATVEC_SHAPES for M in range(1, 9)]
MATVEC_CASES += [(M, K, N, gs) for K, N in MATVEC_SHAPES for gs in (32, 96, K) for M in (2, 5, 8)]
MATVEC_CASES += [(M, 11008, 4096, 1024) for M in (1, 2, 5, 8)]  # partial last group: 11008 = 10 x 1024 + 768


@pytest.mark.parametrize('M,K,N,gs', MATVEC_CASES)
def test_matvec_edges(ops, M, K, N, gs):
    bias = M % 2 == 0
    L = layer(K, N, gs, bias, seed=K + N + gs)
    x = randn_x(M, K, seed=M)
    what = f'matvec M={M} K={K} N={N} gs={gs} bias={bias}'
    out = run_kernel(lambda: ops.matmul248(x, *L.dev, 4, 15, bias=L.bias, groupsize=gs), MATVEC, what)
    torch.cuda.synchronize()
    ctr = workspace_counters(ops, x.device, N)
    assert int(ctr.count_nonzero()) == 0, f'{what}: workspace counters left non-zero'
    ratio = check_fp64_bound(out, x, L.W, L.bias, what, locate=lambda m, n: X.matvec_where(K, N, gs, m, n))
    note('matvec', ratio)
    if gs in (1024, 11008):
        note('matvec, K = 11008 at gs 1024 / 11008', ratio)


@pytest.mark.parametrize('M', range(1, 9))
def test_matvec_fused_mlp_7b(ops, M):
    K, N, gs = 4096, 11008, 128
    G, U = layer(K, N, gs, seed=1), layer(K, N, gs, seed=2)
    x = randn_x(M, K, seed=M)
    what = f'matvec fused mlp M={M} K={K} N={N}'
    out = run_kernel(lambda: ops.fused_mlp(x, G.dev, U.dev, 4, gs), MATVEC_DUAL, what)
    torch.cuda.synchronize()
    assert int(workspace_counters(ops, x.device, N).count_nonzero()) == 0, f'{what}: workspace counters left non-zero'
    note('matvec fused mlp', check_swiglu_fp64_bound(out, x, G.W, U.W, what, locate=lambda m, n: X.matvec_where(K, N, gs, m, n)))


# ============================================================================= documented fallbacks to the generic kernel
def _misaligned(M, K, seed):
    buf = randn_x(M, K + 8, seed)
    x = buf[:, 1:K + 1]  # 2 bytes past a 16-byte boundary; row stride K + 8 stays a multiple of 8
    assert x.data_ptr() % 16 == 2
    return x


@pytest.mark.parametrize('case,M,K,N,gs', [('misaligned x', 4, 4096, 1024, 128), ('misaligned x', 40, 4096, 1024, 128),
                                           ('groupsize 32', 40, 1024, 512, 32), ('N = 96', 40, 1024, 96, 128)])
def test_fallback_to_generic(ops, case, M, K, N, gs):
    L = layer(K, N, gs, True, seed=K + N + gs)
    x = _misaligned(M, K, seed=M) if case == 'misaligned x' else randn_x(M, K, seed=M)
    what = f'fallback ({case}) M={M} K={K} N={N} gs={gs}'
    out = run_kernel(lambda: ops.matmul248(x, *L.dev, 4, 15, bias=L.bias, groupsize=gs), GENERIC_4, what)
    # the generic kernel accumulates K / 8 products per warp with fmaf, then adds 8 warp partials
    note('generic fallback', check_fp64_bound(out, x, L.W, L.bias, what, depth=K / 8 + 8))


# ============================================================================= workspace reuse and determinism
def test_matvec_workspace_shared_across_shapes(ops):
    """Shape A, then B (three times the slabs: more counters, more partials in the same workspace), then A again: bit-identical."""
    M, gs = 4, 128
    A, B = layer(4096, 4096, gs, seed=7), layer(4096, 12288, gs, seed=8)
    x = randn_x(M, 4096, seed=9)
    a1 = run_kernel(lambda: ops.matmul248(x, *A.dev, 4, 15, groupsize=gs), MATVEC, 'shape A')
    run_kernel(lambda: ops.matmul248(x, *B.dev, 4, 15, groupsize=gs), MATVEC, 'shape B')
    torch.cuda.synchronize()
    assert int(workspace_counters(ops, x.device, 12288).count_nonzero()) == 0
    a2 = ops.matmul248(x, *A.dev, 4, 15, groupsize=gs)
    assert torch.equal(a1, a2)


@pytest.mark.parametrize('kind,M', [('matvec', 8), ('matvec', 3), ('fused matvec', 5), ('wgmma', 512), ('wgmma', 100), ('fused wgmma', 200)])
def test_repeated_calls_are_bit_identical(ops, kind, M):
    gs = 128
    if kind.startswith('fused'):
        G, U = layer(4096, 11008, gs, seed=1), layer(4096, 11008, gs, seed=2)
        x = randn_x(M, 4096, seed=M)
        fn = lambda: ops.fused_mlp(x, G.dev, U.dev, 4, gs)
        kernel = MATVEC_DUAL if M <= 8 else GEMM_DUAL
    else:
        L = layer(4096, 4096, gs, seed=3)
        x = randn_x(M, 4096, seed=M)
        fn = lambda: ops.matmul248(x, *L.dev, 4, 15, groupsize=gs)
        kernel = MATVEC if M <= 8 else (GEMM_2 if M > 128 else GEMM_1)
    outs = [run_kernel(fn, kernel, kind)] + [fn() for _ in range(2)]
    assert torch.equal(outs[0], outs[1]) and torch.equal(outs[0], outs[2])
