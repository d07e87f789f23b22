"""CPU: argument validation of gptq_cached_attention (it runs before any CUDA call, so no GPU is needed), the ops wrapper's device check, and
the host-side prefix matching behind generate(..., reuse_cache=True)."""
import ctypes

import pytest

P = 0x1000  # a 16-byte aligned fake device pointer: every call below returns before anything is dereferenced


def _spans(seq, start, rows):
    arr = lambda v: (ctypes.c_int32 * max(len(v), 1))(*v)
    return len(seq), arr(seq), arr(start), arr(rows)


def _call(q=P, ldq=256, k=P, v=P, batch=4, n_heads=2, head_dim=128, max_seq=512, spans=((0, 0, 3), (2, 100, 40)), out=P, ldo=256, arrays=True):
    from gptq_b200._lib import lib
    n, seq, start, rows = _spans([s[0] for s in spans], [s[1] for s in spans], [s[2] for s in spans])
    if not arrays:
        seq = start = rows = None
    return lib.gptq_cached_attention(q, ldq, k, v, batch, n_heads, head_dim, max_seq, n, seq, start, rows, out, ldo, None)


@pytest.mark.parametrize('field', ['q', 'k', 'v', 'out'])
def test_null_pointers(field):
    from gptq_b200 import _lib
    assert _call(**{field: None}) == _lib.ERR_NULL


def test_null_span_arrays():
    from gptq_b200 import _lib
    assert _call(arrays=False) == _lib.ERR_NULL
    assert _call(arrays=False, spans=()) == _lib.OK  # no spans: nothing is read


@pytest.mark.parametrize('head_dim', [64, 96, 256])
def test_head_dim_other_than_128_is_unsupported(head_dim):
    from gptq_b200 import _lib
    assert _call(head_dim=head_dim, ldq=2 * head_dim, ldo=2 * head_dim) == _lib.ERR_UNSUPPORTED


@pytest.mark.parametrize('kw', [
    dict(batch=0), dict(batch=-1), dict(n_heads=0), dict(head_dim=0), dict(max_seq=0), dict(max_seq=-5),
    dict(spans=[(i, 0, 1) for i in range(65)], batch=65),  # more than 64 spans
    dict(spans=((4, 0, 1), )), dict(spans=((-1, 0, 1), )),  # sequence out of range
    dict(spans=((1, 0, 1), (1, 5, 2))),  # a sequence twice
    dict(spans=((0, -1, 1), )), dict(spans=((0, 0, -1), )),  # negative start / rows
    dict(spans=((0, 500, 13), )), dict(spans=((0, 512, 1), )),  # past max_seq
    dict(ldq=255 - 7), dict(ldo=128), dict(ldq=260), dict(ldo=252 + 10),  # below n_heads * 128 or not a multiple of 8
    dict(batch=8, n_heads=64, max_seq=1 << 23),  # 2^32 cache rows: beyond 32-bit TMA coordinates
])
def test_shape_errors(kw):
    from gptq_b200 import _lib
    assert _call(**kw) == _lib.ERR_SHAPE


def test_span_counts_at_the_limits_pass_validation():
    from gptq_b200 import _lib
    assert _call(spans=[(i, 0, 0) for i in range(64)], batch=64) == _lib.OK  # 64 spans, zero rows: nothing to launch
    assert _call(spans=((0, 512, 0), (1, 0, 0))) == _lib.OK  # start == max_seq with no rows is valid


@pytest.mark.parametrize('kw', [dict(q=P + 8), dict(k=P + 2), dict(v=P + 4), dict(out=P + 8)])
def test_alignment_errors(kw):
    from gptq_b200 import _lib
    assert _call(**kw) == _lib.ERR_ALIGN


def test_zero_rows_is_ok():
    from gptq_b200 import _lib
    assert _call(spans=()) == _lib.OK
    assert _call(spans=((0, 10, 0), (3, 511, 0))) == _lib.OK


def test_ops_wrapper_rejects_cpu_tensors():
    import torch
    from gptq_b200 import ops
    kc = torch.zeros(1, 2, 16, 128, dtype=torch.float16)
    with pytest.raises(ValueError):
        ops.cached_attention(torch.zeros(3, 256, dtype=torch.float16), kc, kc.clone(), [(0, 0, 3)])


@pytest.mark.parametrize('prompt, cached, expected', [
    ([5, 6, 7], [], 0),  # empty cache
    ([5, 6, 7], [5, 6, 7], 2),  # full match: capped at len - 1, the last token goes through the decode step
    ([5, 6, 7, 8], [5, 6, 7, 8, 9, 10], 3),  # the cache is longer than the prompt
    ([5, 6, 7, 8, 9], [5, 6, 1, 8, 9], 2),  # divergence in the middle (an edited turn)
    ([5, 6], [5, 6, 7, 8], 1),  # a prompt shorter than the cache
    ([4, 6, 7], [5, 6, 7], 0),  # diverges at once
    ([5, 6, 7, 8, 9], [5, 6], 2),  # the cache is a prefix of the prompt (a second turn)
    ([5], [5, 6], 0),  # a one-token prompt keeps nothing
])
def test_reusable_prefix(prompt, cached, expected):
    from gptq_b200.engine import reusable_prefix
    assert reusable_prefix(prompt, cached) == expected
