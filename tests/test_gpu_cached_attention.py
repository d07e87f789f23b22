"""GPU: causal attention over the KV cache (gptq_cached_attention, csrc/cached_attention.cu) -- against a float64 softmax with a per-element
bound derived from the kernel's arithmetic, at every query-tile and key-tile edge; bit-exact anchors; NaN in every cache row the result must
not read; determinism and independence of the spans; which kernels run."""
import json
import os
import subprocess
import sys

import pytest
import torch

from gpu_util import HD, check_cached_attention, make_gqa_kv_cache, make_kv_cache, report, run_cached_attention

pytestmark = pytest.mark.gpu

STARTS = (0, 1, 63, 64, 65, 127, 128, 129, 1000, 2047, 2048, 4095, None)  # None: max_seq - rows
ROWS = (1, 2, 63, 64, 65, 127, 128, 129, 300)


# (query heads, K/V heads): multi-head, one K/V head for 8 query heads, and 16 / 2 (g = 8 over two K/V heads, as LLaMA-2-70B and
# LLaMA-3-8B group them).  The multi-head cases keep their ids.
EDGE_CASES = [(nh, nkv, rows) for nh, nkv in ((2, 2), (8, 1), (16, 2)) for rows in ROWS]


@pytest.mark.parametrize('nh,nkv,rows', EDGE_CASES, ids=[str(r) if nh == nkv else f'{nh}-{nkv}-{r}' for nh, nkv, r in EDGE_CASES])
def test_against_fp64_softmax_at_every_edge(nh, nkv, rows):
    """Every start of STARTS with `rows` query rows, one span per sequence (8 per call, the last call partly filled), on a cache of CodeLlama's
    16384 positions; every cache row outside the spans' reach is NaN.  With nkv < nh each K/V head serves nh / nkv query heads, and the
    reference repeats it that many times."""
    S, g = 16384, nh // nkv
    starts = [S - rows if s is None else s for s in STARTS]
    worst = 0.0
    for c in range(0, len(starts), 8):
        spans = [(b, s, rows) for b, s in enumerate(starts[c:c + 8])]
        q, kc, vc = make_gqa_kv_cache(8, nh, nkv, S, spans, seed=rows * 100 + c)
        out = run_cached_attention(q, kc, vc, spans)
        worst = max(worst, check_cached_attention(out, q, kc[1].repeat_interleave(g, 1), vc[1].repeat_interleave(g, 1), spans, f'{nh} / {nkv} heads, rows {rows}'))
        del q, kc, vc, out
    report(worst, f'{nh} / {nkv} heads, {rows} rows at starts {starts}')


def test_llama_7b_shape():
    """32 heads, max_seq 2048: 128 rows at start 1920 (the span ends at the last cache row), next to a ragged second sequence."""
    spans = [(0, 1920, 128), (1, 700, 77)]
    q, kc, vc = make_kv_cache(2, 32, 2048, spans, seed=7, layers=2, layer=1)
    report(check_cached_attention(run_cached_attention(q, kc, vc, spans), q, kc[1], vc[1], spans, '7B shape'), '32 heads, start 1920, 128 rows')


def test_strided_q_from_the_fused_qkv_output():
    """q read in place from the q columns of a [M, 3 * H] qkv tensor (row pitch 3 H), as the engine passes it."""
    from gptq_b200 import ops
    spans = [(0, 5, 40), (1, 0, 130)]
    q, kc, vc = make_kv_cache(2, 2, 256, spans, seed=8)
    qkv = torch.randn(q.shape[0], 3 * q.shape[1], device='cuda').half()
    qkv[:, :q.shape[1]] = q
    out = ops.cached_attention(qkv[:, :q.shape[1]], kc[1], vc[1], spans)
    assert torch.equal(out, run_cached_attention(q, kc, vc, spans))


# ----------------------------------------------------------------------------- bit-exact anchors
def test_position_zero_returns_its_own_value_row():
    spans = [(0, 0, 200), (1, 0, 1), (2, 0, 129)]
    q, kc, vc = make_kv_cache(3, 2, 512, spans, seed=9)
    out = run_cached_attention(q, kc, vc, spans)
    r0 = 0
    for b, _, n in spans:
        assert torch.equal(out[r0].view(2, HD), vc[1, b, :, 0]), f'sequence {b}: position 0'
        r0 += n


def test_equal_keys_and_alternating_values_cancel_exactly():
    """All keys of a head equal (entries in {-1/4, 0, 1/4}: every score is exact and the same, so every p is exactly 1), values +w, -w, +w, ...
    (multiples of 2^-4): a row whose prefix has even length sums to exactly 0.  A key missed, counted twice or read past the causal limit
    leaves a nonzero output."""
    S, nh = 1300, 2
    spans = [(0, 0, 300), (1, 1, 129), (2, 127, 130), (3, 1000, 300), (4, 64, 1), (5, 65, 2)]
    q, kc, vc = make_kv_cache(6, nh, S, spans, seed=10)
    g = torch.Generator(device='cuda').manual_seed(11)
    M = q.shape[0]
    q.copy_((torch.randint(-1, 2, (M, nh * HD), device='cuda', generator=g) * 0.25).half())
    for b, s, n in spans:
        L = s + n
        kc[1, b, :, :L] = (torch.randint(-1, 2, (nh, 1, HD), device='cuda', generator=g) * 0.25).half()
        w = (torch.randint(-32, 33, (nh, 1, HD), device='cuda', generator=g) / 16).half()
        sign = 1 - 2 * (torch.arange(L, device='cuda') % 2).half()
        vc[1, b, :, :L] = w * sign[None, :, None]
    out = run_cached_attention(q, kc, vc, spans)
    r0, checked = 0, 0
    for b, s, n in spans:
        for i in range(n):
            if (s + i + 1) % 2 == 0:
                assert torch.equal(out[r0 + i], torch.zeros_like(out[r0 + i])), f'sequence {b}, position {s + i}: {out[r0 + i].abs().max().item()}'
                checked += 1
        r0 += n
    assert checked > 400


# ----------------------------------------------------------------------------- NaN isolation, determinism, independence
def test_nan_in_unread_rows_does_not_reach_the_result():
    """The same spans on a cache whose unread rows are NaN and on one where they are random: every output finite and bit-identical."""
    spans = [(0, 0, 1), (2, 127, 130), (3, 200, 57), (1, 1000, 300)]
    q, kc, vc = make_kv_cache(5, 2, 1400, spans, seed=12, poison=True)
    _, kc2, vc2 = make_kv_cache(5, 2, 1400, spans, seed=12, poison=False)
    for b, s, n in spans:  # the same rows that are read
        kc2[1, b, :, :s + n] = kc[1, b, :, :s + n]
        vc2[1, b, :, :s + n] = vc[1, b, :, :s + n]
    a, c = run_cached_attention(q, kc, vc, spans), run_cached_attention(q, kc2, vc2, spans)
    assert torch.isfinite(a).all() and torch.equal(a, c)


def test_determinism_and_span_independence():
    from gptq_b200 import ops
    spans = [(0, 3, 200), (1, 500, 64), (2, 0, 1), (3, 127, 129)]
    q, kc, vc = make_kv_cache(4, 2, 1024, spans, seed=13)
    a = run_cached_attention(q, kc, vc, spans)
    assert torch.equal(a, run_cached_attention(q, kc, vc, spans)), 'two runs differ'
    rows = [n for _, _, n in spans]
    parts = a.split(rows)
    qs = q.split(rows)
    for i, sp in enumerate(spans):
        alone = ops.cached_attention(qs[i].contiguous(), kc[1], vc[1], [sp])
        assert torch.equal(alone, parts[i]), f'span {sp} alone'
    order = [3, 1, 0, 2]
    perm = ops.cached_attention(torch.cat([qs[i] for i in order]), kc[1], vc[1], [spans[i] for i in order])
    assert torch.equal(perm, torch.cat([parts[i] for i in order])), 'spans reordered'


TESTS = os.path.dirname(os.path.abspath(__file__))
_ROUTING_CHILD = """
import json, sys
sys.path[:0] = {paths!r}
import torch
from gpu_util import launched_kernels
from gptq_b200 import ops
g = torch.Generator(device='cuda').manual_seed(14)
kc, vc = (torch.randn(2, 2, 256, 128, device='cuda', generator=g).half() for _ in range(2))
q = torch.randn(50, 256, device='cuda', generator=g).half()
fn = lambda: ops.cached_attention(q, kc, vc, [(0, 10, 50), (1, 0, 0)])
fn()  # warm-up: module loading and function attributes
for _ in range(3):  # a trace without any kernel record is taken again, as in gpu_util.run_kernel
    names = launched_kernels(fn)[1]
    if names:
        break
print(json.dumps(sorted(names)))
"""


def test_empty_call():
    from gptq_b200 import ops
    q, kc, vc = make_kv_cache(2, 2, 256, [(0, 10, 50)], seed=14)
    assert ops.cached_attention(q[:0], kc[1], vc[1], [(1, 0, 0)]).shape == (0, 2 * HD)


def test_routing():
    """A call launches the cached-attention kernel and no SDPA / flash kernel.  The trace is taken in a child process: a torch.profiler
    session opened in the test process ahead of the engine tests left later sessions of that process with kernel records missing (partial
    or empty traces in tests/test_gpu_launches.py, tests/test_gpu_exact.py, tests/test_gpu_kernel_edges.py)."""
    root = os.path.dirname(TESTS)
    code = _ROUTING_CHILD.format(paths=[root, os.path.join(root, 'gptq-for-llama_b200'), TESTS])
    flags = ['-s'] if sys.flags.no_user_site else []
    res = subprocess.run([sys.executable, *flags, '-c', code], capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, res.stderr[-4000:]
    names = json.loads(res.stdout.strip().splitlines()[-1])
    if not names:
        pytest.skip('CUDA activity tracing returned no kernel events on this machine')
    assert any('cached_attention_kernel' in n for n in names), sorted(names)
    assert not any(k in n.lower() for n in names for k in ('flash', 'fmha', 'sdpa', 'efficient_attention', 'softmax')), sorted(names)
