"""The forward arithmetic against OUTPUTS OF THE REFERENCE'S OWN TRITON KERNELS (tests/golden/fwd_ref_triton.npz, generated on a
GPU from the unmodified reference by tests/golden/make_fwd_golden.py): matmul248 (+bias), the fused SwiGLU MLP kernel,
triton_rotate_half_ and TritonLlamaRMSNorm.

  * CPU: the oracle (oracle/gptq_oracle.py, and its C restatement) reproduces the reference outputs within 1e-3 -- this is what
    pins the forward oracle to the reference's execution (SURVEY.md 8(c)(iii)), not only to its source.
  * GPU: this repo's CUDA path reproduces the same reference outputs through the C ABI.
"""
import importlib.util
import os

import numpy as np
import pytest
import torch

from oracle import cref
from oracle import gptq_oracle as O
from gpu_util import assert_rel_close

HERE = os.path.dirname(os.path.abspath(__file__))
spec = importlib.util.spec_from_file_location('make_fwd_golden', os.path.join(HERE, 'golden', 'make_fwd_golden.py'))
G = importlib.util.module_from_spec(spec)
spec.loader.exec_module(G)  # case list and input generators shared with the generator script

REF = dict(np.load(os.path.join(HERE, 'golden', 'fwd_ref_triton.npz')))


def ref(key):
    return torch.from_numpy(REF[key])


def pack_cases():
    for name, fx in G.pack_fixtures().items():
        for M in G.PACK_M:
            yield name, fx, M


def _fixture_tensors(fx):
    qw, qz, sc, gi = (torch.from_numpy(fx[k]) for k in ('qweight', 'qzeros', 'scales_h', 'g_idx'))
    bias = torch.from_numpy(fx['bias_h']) if 'bias_h' in fx else None
    return qw, sc, qz, gi, bias


# ------------------------------------------------------------------------------------------------- CPU: oracle vs reference
@pytest.mark.parametrize('impl', ['numpy', 'c'])
def test_oracle_matmul248_matches_reference_triton(impl):
    if impl == 'c' and not cref.available():
        pytest.skip('oracle/libgptq_oracle.so not built')
    Q = cref if impl == 'c' else O
    n = 0
    for name, fx, M in pack_cases():
        qw, sc, qz, gi, bias = _fixture_tensors(fx)
        x = G.x_for(G.name_seed(name), M, int(fx['K']))
        assert_rel_close(Q.qlinear_fwd(x, qw, sc, qz, gi, int(fx['bits']), bias), ref(f'pack/{name}/M{M}'), what=f'pack/{name}/M{M}')
        n += 1
    for name, K, N, bits, gs, act, seed, Ms in G.RANDOM_CASES:
        qw, sc, qz, gi, _ = O.random_packed(K, N, bits, gs, seed=seed, act_order=act)
        for M in Ms:
            assert_rel_close(Q.qlinear_fwd(G.x_for(seed, M, K), qw, sc, qz, gi, bits), ref(f'random/{name}/M{M}'), what=f'random/{name}/M{M}')
            n += 1
    assert n == 43


def test_oracle_fused_mlp_rope_rmsnorm_match_reference_triton():
    for name, K, N, bits, gs, seed, Ms in G.MLP_CASES:
        gate, up = O.random_packed(K, N, bits, gs, seed=seed)[:4], O.random_packed(K, N, bits, gs, seed=seed + 100)[:4]
        for M in Ms:
            assert_rel_close(O.fused_mlp_fwd(G.x_for(seed, M, K), gate, up, bits), ref(f'mlp/{name}/M{M}'), what=f'mlp/{name}/M{M}')
    qk, pos = G.rope_input()
    O.rope_inplace(qk[:, :, :2], pos)
    assert_rel_close(qk, ref('rope/out'), what='rotate_half')
    for name, M, N, seed in G.NORM_CASES:
        x, w = G.norm_input(M, N, seed)
        assert_rel_close(O.rmsnorm_fwd(x, w, 1e-6), ref(f'norm/{name}'), what=name)


# ------------------------------------------------------------------------------------------------- GPU: CUDA path vs reference
@pytest.mark.gpu
def test_cuda_matmul248_matches_reference_triton():
    from gptq_b200 import ops
    dev = torch.device('cuda:0')
    for name, fx, M in pack_cases():
        qw, sc, qz, gi, bias = _fixture_tensors(fx)
        x = G.x_for(G.name_seed(name), M, int(fx['K']))
        out = ops.matmul248(x.to(dev), qw.to(dev), sc.to(dev), qz.to(dev), gi.to(dev), int(fx['bits']), bias=bias.to(dev) if bias is not None else None)
        assert_rel_close(out, ref(f'pack/{name}/M{M}'), rel=1e-3 if M <= 8 else 2e-3, what=f'pack/{name}/M{M}')  # M > 8: tensor-core accumulation is not IEEE per add
    for name, K, N, bits, gs, act, seed, Ms in G.RANDOM_CASES:
        qw, sc, qz, gi, _ = O.random_packed(K, N, bits, gs, seed=seed, act_order=act)
        for M in Ms:
            out = ops.matmul248(G.x_for(seed, M, K).to(dev), qw.to(dev), sc.to(dev), qz.to(dev), gi.to(dev), bits, groupsize=0 if act else gs)
            assert_rel_close(out, ref(f'random/{name}/M{M}'), rel=1e-3 if M <= 8 else 2e-3, what=f'random/{name}/M{M}')


@pytest.mark.gpu
def test_cuda_fused_mlp_rope_rmsnorm_match_reference_triton():
    from gptq_b200 import ops
    dev = torch.device('cuda:0')
    for name, K, N, bits, gs, seed, Ms in G.MLP_CASES:
        gate, up = O.random_packed(K, N, bits, gs, seed=seed)[:4], O.random_packed(K, N, bits, gs, seed=seed + 100)[:4]
        for M in Ms:
            out = ops.fused_mlp(G.x_for(seed, M, K).to(dev), tuple(t.to(dev) for t in gate), tuple(t.to(dev) for t in up), bits, gs)
            assert_rel_close(out, ref(f'mlp/{name}/M{M}'), rel=1e-3 if M <= 8 else 2e-3, what=f'mlp/{name}/M{M}')
    qk, pos = G.rope_input()
    dq = qk.to(dev)
    ops.rotate_half_(dq[:, :, :2], pos.to(dev))
    assert_rel_close(dq, ref('rope/out'), what='rotate_half')
    for name, M, N, seed in G.NORM_CASES:
        x, w = G.norm_input(M, N, seed)
        assert_rel_close(ops.rmsnorm(x.to(dev), w.to(dev), 1e-6), ref(f'norm/{name}'), what=name)
