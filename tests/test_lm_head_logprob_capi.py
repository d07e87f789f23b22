"""CPU: argument validation of gptq_lm_head_logprob (it runs before any CUDA call, so no GPU is needed) and its workspace size."""
import ctypes

import pytest

P = 0x1000  # a 256-byte aligned fake device pointer: every call below returns before anything is dereferenced


def _call(x=P, ldx=128, w=P, ldw=128, M=4, K=128, V=300, targets=P, logprob=P, ws=P, ws_bytes=None):
    from gptq_b200._lib import lib
    if ws_bytes is None:
        ws_bytes = lib.gptq_lm_head_logprob_workspace_bytes(M, V)
    return lib.gptq_lm_head_logprob(x, ldx, w, ldw, M, K, V, targets, logprob, ws, ws_bytes, None)


@pytest.mark.parametrize('field', ['x', 'w', 'targets', 'logprob'])
def test_null_pointers(field):
    from gptq_b200 import _lib
    assert _call(**{field: None}) == _lib.ERR_NULL


@pytest.mark.parametrize('kw', [dict(K=0, ldx=0, ldw=0), dict(K=-64), dict(K=96), dict(K=100, ldx=128, ldw=128), dict(V=0), dict(V=-1), dict(M=-1),
                                dict(ldx=120), dict(ldw=64)])
def test_shape_errors(kw):
    from gptq_b200 import _lib
    assert _call(**kw) == _lib.ERR_SHAPE


@pytest.mark.parametrize('kw', [dict(x=P + 8), dict(w=P + 2), dict(ldx=132), dict(ldw=140)])
def test_alignment_errors(kw):
    from gptq_b200 import _lib
    assert _call(**kw) == _lib.ERR_ALIGN


def test_workspace_errors():
    from gptq_b200 import _lib
    need = _lib.lib.gptq_lm_head_logprob_workspace_bytes(4, 300)
    assert _call(ws=None) == _lib.ERR_WORKSPACE
    assert _call(ws_bytes=need - 1) == _lib.ERR_WORKSPACE
    assert _call(ws=P + 16) == _lib.ERR_WORKSPACE  # the workspace must be 256-byte aligned


def test_empty_batch_is_ok():
    from gptq_b200 import _lib
    assert _call(M=0, ws=None, ws_bytes=0) == _lib.OK
    assert _lib.lib.gptq_lm_head_logprob_workspace_bytes(0, 32000) == 0


def test_workspace_grows_with_rows_and_vocabulary():
    from gptq_b200._lib import lib
    size = lib.gptq_lm_head_logprob_workspace_bytes
    for M, V in ((1, 1), (1, 300), (4099, 32001), (16384, 32000)):
        assert size(M, V) % 256 == 0
        # one (max, sum) float2 per row and 128-column vocabulary tile, plus the target logit of every row
        assert size(M, V) >= M * (-(-V // 128)) * 8 + M * 4
    assert size(64, 300) > size(1, 300) and size(2048, 32000) > size(1024, 32000)
    assert size(1, 32000) > size(1, 300) and size(64, 32001) > size(64, 32000)


def test_ops_wrapper_rejects_cpu_tensors():
    import torch
    from gptq_b200 import ops
    with pytest.raises(ValueError):
        ops.lm_head_logprob(torch.zeros(2, 64, dtype=torch.float16), torch.zeros(300, 64, dtype=torch.float16), torch.zeros(2, dtype=torch.int32))


def test_abi_version_is_6():
    from gptq_b200._lib import ABI_VERSION, lib
    assert ABI_VERSION == lib.gptq_abi_version() == 6
    assert ctypes.c_size_t(lib.gptq_lm_head_logprob_workspace_bytes(1, 128)).value > 0
