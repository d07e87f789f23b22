"""GPU: the kernels of the batched passes (prefill, extend, score) and of the kernel chain at the LLaMA-65B and LLaMA-33B shapes, which the
7B / 13B tables of test_gpu_kernel_edges.py and the other kernel tests do not reach:

  * wgmma GEMM at K = 8192 / 22016 / 6656 / 17920 / 28672 / 14336 / 4096 and N up to 24576 (65B qkv), gs 128 and 1024 (a partial last
    group of 512 wherever K is not a multiple of 1024), M in {9, 257, 2048}, and the fused MLP at (8192, 22016), (6656, 17920),
    (8192, 28672) and (4096, 14336): within check_fp64_bound;
  * split-K matvec at the same shapes, M = 1..8, single and dual, with the whole workspace back at zero after every call (the partials
    of one call used to stay behind, where a later call with more column slabs keeps its arrival counters);
  * lm_head_logprob at K = 8192 and 6656, V = 32000, M = 2048 (the bound of test_gpu_score.py);
  * cached_attention at 64 and 52 heads (the bound of test_gpu_cached_attention.py, NaN in every row the kernel must not read), and with
    grouped K/V heads at 64 / 8 over 4096 rows (LLaMA-2-70B) and 32 / 8 over 8192 (LLaMA-3-8B);
  * LlamaDecoder.extend against stepping and score against the oracle on a two-layer 65B model, and extend at the last cache row of
    two-layer LLaMA-2-70B and LLaMA-3-8B models.
The grouped-query linears join the tables: 70B / 34B qkv (8192 -> 10240), 70B down_proj (28672 -> 8192), 70B gate|up (8192 -> 28672),
LLaMA-3-8B qkv (4096 -> 6144), gate|up (4096 -> 14336) and down_proj (14336 -> 4096).  The matvec cases take their expected kernel from
exact_fixtures.matvec_takes: at 70B gate|up and down_proj, M = 7 and 8, the generic kernel serves the call.

The layers are drawn on the device: uniform nibbles and zeros packed by ops.pack_qweight / pack_qzeros, scales ~ U(1e-3, 1.1e-2), and the
reference weight is formed from the same integers in torch as the reference's matmul248 forms it (oracle.gptq_oracle.dequant: (w - z) to
fp16, times the fp16 scale, one rounding).  Every kernel case asserts which kernel served it.  The two engine cases take no trace: a
torch.profiler session around a 65B extend or score left later sessions of the test process with kernel records missing
(tests/test_gpu_launches.py); the kernel cases above cover their batched linears at the same shapes."""
from functools import lru_cache

import pytest
import torch

from exact_fixtures import matvec_takes
from gpu_util import GEMM_1, GEMM_2, GEMM_DUAL, GENERIC_4, MATVEC, MATVEC_DUAL, WorstRatios, check_cached_attention, check_fp64_bound, check_logprob, \
    check_swiglu_fp64_bound, generic, make_gqa_kv_cache, random_logprob_inputs, randn_x, report, run_cached_attention, run_kernel
from llama_oracle import LlamaOracle, check_extend_against_stepping, check_scores

pytestmark = pytest.mark.gpu

WORST = WorstRatios()
note = WORST.note


@pytest.fixture(scope='module', autouse=True)
def worst_ratio_summary():
    yield
    WORST.summary()


class Layer:
    """A random int4 layer on the device: the packed fields, and the reference's fp16 weight W [K, N] formed from the same integers."""

    def __init__(self, K, N, gs, seed):
        from gptq_b200 import ops
        dev = torch.device('cuda:0')
        gen = torch.Generator(device=dev).manual_seed(seed)
        G = -(-K // gs)
        w = torch.randint(0, 16, (K, N), device=dev, generator=gen, dtype=torch.int32)
        z = torch.randint(0, 16, (G, N), device=dev, generator=gen, dtype=torch.int32)  # stored zero; the real zero is z + 1
        s = (torch.rand(G, N, device=dev, generator=gen) * 1e-2 + 1e-3).half()
        g = (torch.arange(K, device=dev) // gs).to(torch.int32)
        self.dev = (ops.pack_qweight(w, 4), s, ops.pack_qzeros(z, 4), g)
        gl = g.long()
        self.W = (w - (z + 1)[gl]).half() * s[gl]
        del w


@lru_cache(maxsize=2)
def layer(K, N, gs, seed=0):
    return Layer(K, N, gs, seed)


# (K, N): 65B qkv / o_proj / down_proj, 33B gate|up / down_proj, 70B and 34B qkv (64 / 8 heads), 70B down_proj, LLaMA-3-8B qkv (32 / 8
# heads) and down_proj
SHAPES = [(8192, 24576), (8192, 8192), (22016, 8192), (6656, 19968), (17920, 6656), (8192, 10240), (28672, 8192), (4096, 6144), (14336, 4096)]
# (K, N) of gate and of up: 65B and 34B, 33B, 70B, LLaMA-3-8B
MLP_SHAPES = [(8192, 22016), (6656, 17920), (8192, 28672), (4096, 14336)]
GS = (128, 1024)


# ============================================================================= wgmma GEMM
@pytest.mark.parametrize('M', [9, 257, 2048])
@pytest.mark.parametrize('gs', GS)
@pytest.mark.parametrize('K,N', SHAPES)
def test_wgmma_gemm(K, N, gs, M):
    from gptq_b200 import ops
    L = layer(K, N, gs, seed=K + N + gs)
    x = randn_x(M, K, seed=M)
    what = f'wgmma M={M} K={K} N={N} gs={gs}'
    kernel = GEMM_2 if M > 128 else GEMM_1
    out = run_kernel(lambda: ops.matmul248(x, *L.dev, 4, 15, groupsize=gs), kernel, what)
    note(f'wgmma {kernel}', check_fp64_bound(out, x, L.W, what=what))


@pytest.mark.parametrize('M', [9, 257, 2048])
@pytest.mark.parametrize('K,N', MLP_SHAPES)
def test_wgmma_fused_mlp(K, N, M):
    from gptq_b200 import ops
    gs = 128
    G, U = layer(K, N, gs, seed=1), layer(K, N, gs, seed=2)
    x = randn_x(M, K, seed=M)
    what = f'wgmma fused mlp M={M} K={K} N={N} gs={gs}'
    out = run_kernel(lambda: ops.fused_mlp(x, G.dev, U.dev, 4, gs), GEMM_DUAL, what)
    note('wgmma fused mlp', check_swiglu_fp64_bound(out, x, G.W, U.W, what))


# ============================================================================= split-K matvec
# Where the x segment of a CTA and the weight rings need more than the 110 KB of shared memory that two CTAs per SM leave (qmatvec.cu
# skinny_supported, restated by exact_fixtures.matvec_takes), the generic kernel serves the call: the 65B qkv at M = 8 (94 k-steps of 8
# rows), and 70B gate|up and down_proj at M = 7 and 8 (109 k-steps).


def workspace_is_zero(ops, dev):
    """The whole per-stream workspace, counters and partials, is zero again after a call (include/gptq_b200.h)."""
    ws = ops._workspaces[(dev.index, torch.cuda.current_stream(dev).cuda_stream)]
    return int(ws.count_nonzero()) == 0


@pytest.mark.parametrize('M', range(1, 9))
@pytest.mark.parametrize('gs', GS)
@pytest.mark.parametrize('K,N', SHAPES)
def test_matvec(K, N, gs, M):
    from gptq_b200 import ops
    L = layer(K, N, gs, seed=K + N + gs)
    x = randn_x(M, K, seed=M)
    what = f'matvec M={M} K={K} N={N} gs={gs}'
    generic = not matvec_takes(M, K, N)  # (only at M >= 7, where the generic kernel runs 4 rows per block)
    out = run_kernel(lambda: ops.matmul248(x, *L.dev, 4, 15, groupsize=gs), GENERIC_4 if generic else MATVEC, what)
    torch.cuda.synchronize()
    assert workspace_is_zero(ops, x.device), f'{what}: workspace left non-zero'
    # the generic kernel accumulates K / 8 products per warp with fmaf, then adds 8 warp partials (test_gpu_kernel_edges)
    print(f'  {what}: {GENERIC_4 if generic else MATVEC}')
    note('generic (matvec over its shared memory)' if generic else 'matvec', check_fp64_bound(out, x, L.W, what=what, depth=K / 8 + 8 if generic else None))


@pytest.mark.parametrize('M', range(1, 9))
@pytest.mark.parametrize('K,N', MLP_SHAPES)
def test_matvec_fused_mlp(K, N, M):
    """At 70B (8192 -> 28672) and M = 7, 8 the generic dual kernel serves the call, as it serves the kernel chain's gate|up."""
    from gptq_b200 import ops
    gs = 128
    G, U = layer(K, N, gs, seed=1), layer(K, N, gs, seed=2)
    x = randn_x(M, K, seed=M)
    what = f'matvec fused mlp M={M} K={K} N={N}'
    on_generic = not matvec_takes(M, K, N)
    kernel = generic(4, M, dual=True) if on_generic else MATVEC_DUAL
    out = run_kernel(lambda: ops.fused_mlp(x, G.dev, U.dev, 4, gs), kernel, what)
    torch.cuda.synchronize()
    assert workspace_is_zero(ops, x.device), f'{what}: workspace left non-zero'
    print(f'  {what}: {kernel}')
    note('generic fused mlp (matvec over its shared memory)' if on_generic else 'matvec fused mlp',
         check_swiglu_fp64_bound(out, x, G.W, U.W, what, depth=K / 8 + 8 if on_generic else None))


def test_matvec_partials_do_not_leak_into_the_next_call():
    """A matvec with 32 slabs of 256 columns (N 8192) and then one with 96 (N 24576), as the 65B kernel chain calls o_proj and then the next
    layer's qkv on one workspace: the first call's split-K partials lie where the second call keeps its arrival counters for slabs 64..95, so
    they must be gone.  Then lm_head_logprob, which accumulates into the same workspace."""
    from gptq_b200 import ops
    small, big = layer(8192, 8192, 128, seed=8192 + 8192 + 128), layer(8192, 24576, 128, seed=8192 + 24576 + 128)
    x = randn_x(4, 8192, seed=4)
    for L, N in ((small, 8192), (big, 24576), (small, 8192), (big, 24576)):
        what = f'matvec M=4 K=8192 N={N} after the other shape'
        out = run_kernel(lambda: ops.matmul248(x, *L.dev, 4, 15, groupsize=128), MATVEC, what)
        torch.cuda.synchronize()
        assert workspace_is_zero(ops, x.device), f'{what}: workspace left non-zero'
        note('matvec', check_fp64_bound(out, x, L.W, what=what))
    xl, W, t = random_logprob_inputs(300, 1000, 8192, seed=3)
    check_logprob(ops.lm_head_logprob(xl, W, t), xl, W, t, 'lm_head_logprob after the matvecs')


# ============================================================================= lm_head + log-softmax
@pytest.mark.parametrize('K', [8192, 6656])
def test_lm_head_logprob(K):
    from gptq_b200 import ops
    x, W, t = random_logprob_inputs(2048, 32000, K, seed=K)
    lp = ops.lm_head_logprob(x, W, t)
    check_logprob(lp, x, W, t, f'lm_head_logprob M=2048 V=32000 K={K}')


# ============================================================================= attention over the KV cache
# (query heads, K/V heads, cache rows): 65B, 33B, LLaMA-2-70B at its 4096 context, LLaMA-3-8B at its 8192 context
ATTN_SHAPES = [(64, 64, 2048), (52, 52, 2048), (64, 8, 4096), (32, 8, 8192)]


@pytest.mark.parametrize('nh,nkv,S', ATTN_SHAPES, ids=[str(nh) if nh == nkv else f'{nh}-{nkv}-{S}' for nh, nkv, S in ATTN_SHAPES])
def test_cached_attention(nh, nkv, S):
    """128 rows ending at the last cache row next to a ragged second sequence, then a ragged call of four spans.  With K/V heads shared
    by nh / nkv query heads, against the reference over the K/V heads repeated."""
    g = nh // nkv
    sweep = f'cached attention, {nh} heads' + ('' if g == 1 else f' / {nkv} K/V heads')
    for spans in ([(0, S - 128, 128), (1, 700, 77)], [(0, 0, 300), (1, 1000, 129), (2, 63, 1), (3, S - 129, 129)]):
        q, kc, vc = make_gqa_kv_cache(len(spans), nh, nkv, S, spans, seed=nh + len(spans), layers=2, layer=1)
        out = run_cached_attention(q, kc, vc, spans)
        note(sweep, check_cached_attention(out, q, kc[1].repeat_interleave(g, 1), vc[1].repeat_interleave(g, 1), spans, f'{sweep} {spans}'))
        del q, kc, vc
    report(WORST[sweep], sweep)


# ============================================================================= the engine on a two-layer 65B model
def test_extend_65b_against_stepping():
    """LLaMA-65B shapes (int4 g128, 2 layers, persistent kernel): 1791 positions stepped, then 256 more through extend(), then one step,
    against stepping all of them, within the run-to-run spread of DESIGN.md section 2 (max 1.5e-2, rms 3e-3 of the rms)."""
    from gptq_b200 import engine
    dec = engine.synthetic_llama('65b', bits=4, groupsize=128, vocab=32000, seed=15, max_seq=2048, n_layers=2)
    assert dec.launches_per_step() == 1
    toks = torch.randint(0, 32000, (2048, ), generator=torch.Generator().manual_seed(5)).tolist()
    check_extend_against_stepping(dec, toks, 1791, '65b extend')


def test_extend_70b_against_stepping():
    """LLaMA-2-70B shapes (64 query / 8 K/V heads, int4 g128, 2 layers, persistent kernel) at its 4096 context: 3839 positions stepped,
    then 256 through extend(), so that the span ends at the last cache row, against stepping them (the bound of the 65B case)."""
    from gptq_b200 import engine
    dec = engine.synthetic_llama('70b', bits=4, groupsize=128, vocab=32000, seed=16, max_seq=4096, n_layers=2)
    assert dec.launches_per_step() == 1 and dec.n_kv_heads == 8
    toks = torch.randint(0, 32000, (4096, ), generator=torch.Generator().manual_seed(6)).tolist()
    check_extend_against_stepping(dec, toks, 3839, '70b extend')


def test_extend_llama3_8b_against_stepping():
    """LLaMA-3-8B shapes (32 query / 8 K/V heads, RoPE base 5e5, vocabulary 128256, 2 layers) at its 8192 context: 7935 positions stepped,
    then 256 through extend() up to the last cache row, against stepping them."""
    from gptq_b200 import engine
    dec = engine.synthetic_llama('llama3-8b', bits=4, groupsize=128, vocab=128256, seed=17, max_seq=8192, n_layers=2, rope_base=500000.0)
    assert dec.launches_per_step() == 1 and dec.n_kv_heads == 8
    toks = torch.randint(0, 128256, (8192, ), generator=torch.Generator().manual_seed(7)).tolist()
    check_extend_against_stepping(dec, toks, 7935, 'llama3-8b extend')


def test_score_65b_against_the_oracle():
    """score() on a two-layer 65B model (one 34-row batched pass) against float64 log-softmaxes of the oracle's fp16 logits, within
    the bound of test_gpu_score.test_score_matches_the_oracle (2 x 2e-2 x max|ref logits| per element)."""
    from gptq_b200 import engine
    dec = engine.synthetic_llama('65b', bits=4, groupsize=128, vocab=300, seed=9, max_seq=16, use_graph=False, n_layers=2)
    g = torch.Generator().manual_seed(4)
    seqs = [torch.randint(0, 300, (n, ), generator=g).tolist() for n in (9, 2, 23)]
    out = dec.score(seqs)
    assert [o.shape[0] for o in out] == [8, 1, 22]
    check_scores(out, seqs, LlamaOracle.from_decoder(dec, eps=1e-6, base=10000.0), '65b score')
