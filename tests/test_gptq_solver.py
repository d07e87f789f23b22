"""SURVEY.md 8(f) rank 4: the GPTQ solver (`gptq.GPTQ`, drop-in for the reference module) against what the reference's own `gptq.py`
computes on the same layers and calibration batches (stored in tests/golden/solver_ref.npz by tests/golden/make_solver_golden.py):
scales, zeros, g_idx and the on-grid weights must agree."""
import importlib.util
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn as nn

HERE = os.path.dirname(os.path.abspath(__file__))
spec = importlib.util.spec_from_file_location('make_solver_golden', os.path.join(HERE, 'golden', 'make_solver_golden.py'))
G = importlib.util.module_from_spec(spec)
spec.loader.exec_module(G)
REF = dict(np.load(G.OUT))


@pytest.mark.parametrize('K,N,bits,groupsize,actorder', G.CASES)
def test_solver_matches_reference_gptq(K, N, bits, groupsize, actorder):
    import gptq as ours_mod
    assert 'gptq-for-llama_b200' in ours_mod.__file__
    n = G.case_name(K, N, bits, groupsize, actorder)
    ga, sa, za, ea = (torch.from_numpy(REF[f'{n}/{k}']) for k in ('g_idx', 'scale', 'zero', 'err'))
    ea = float(ea)
    Wa = sa[:, ga.long()] * (torch.from_numpy(REF[f'{n}/codes']).float() - za[:, ga.long()])  # the reference's on-grid weights, exactly
    sync = torch.cuda.synchronize
    torch.cuda.synchronize = lambda *a, **k: None  # the solver mirrors the reference's unconditional synchronise (gptq.py:205); there may be no GPU
    try:
        weight, batches = G.make_inputs(K, N, bits)
        lin_b = nn.Linear(K, N, bias=True)
        lin_b.weight.data = weight.clone()
        b = ours_mod.GPTQ(lin_b)
        b.quantizer.configure(bits, perchannel=True, sym=False, mse=False)
        for x in batches:
            b.add_batch(x, None)
        r, c = G.h_sample(K)
        assert torch.allclose(torch.diagonal(b.H), torch.from_numpy(REF[f'{n}/H_diag']), rtol=1e-5, atol=1e-6)
        assert torch.allclose(b.H[r, c], torch.from_numpy(REF[f'{n}/H_sample']), rtol=1e-5, atol=1e-6)
        sb, zb, gb, eb = b.fasterquant(blocksize=128, percdamp=.01, groupsize=groupsize, actorder=actorder, name='t')
    finally:
        torch.cuda.synchronize = sync
    assert torch.equal(ga, gb.cpu().to(ga.dtype)) and sa.shape == sb.shape and za.shape == zb.shape
    if actorder:
        assert not torch.equal(gb.cpu(), (torch.arange(K) // (groupsize if groupsize != -1 else K)).int())  # the fixture really exercises the permutation
    # the same algorithm in fp32 with a different operation order: scales / zeros agree closely, a handful of weights may land on a neighbouring grid point
    sb, zb = sb.cpu(), zb.cpu()
    assert torch.allclose(sa, sb, rtol=1e-4, atol=1e-7)
    assert (za != zb).float().mean().item() < 0.01
    Wb = lin_b.weight.data
    step = sb.mean().item()
    differing = ((Wa - Wb).abs() > 0.5 * step).float().mean().item()
    assert differing < 0.01, f'{differing:.2%} of the quantised weights differ'
    assert abs(ea - eb) <= 0.02 * abs(ea) + 1e-9
    # and the point of the exercise: the layer output error stays small and comparable
    x = batches[0].reshape(-1, K)
    assert torch.allclose(x @ Wa.t(), x @ Wb.t(), rtol=0, atol=0.05 * (x @ Wa.t()).abs().mean().item() + 1e-6)
    sys.modules.pop('gptq', None)


def test_quantize_linears_drives_a_block_with_bias_layers():
    """OPT / GPT-NeoX wiring (opt.py:249-285, neox.py:234-273): their blocks are nn.Linear WITH bias; the generic sequential recipe quantises them
    through forward hooks and leaves on-grid weights behind for QuantLinear.pack."""
    import gptq as ours_mod
    torch.manual_seed(0)

    class Block(nn.Module):
        def __init__(self):
            super().__init__()
            self.fc1, self.fc2 = nn.Linear(64, 128, bias=True), nn.Linear(128, 64, bias=True)

        def forward(self, x):
            return self.fc2(torch.relu(self.fc1(x)))

    blk = Block()
    before = {n: p.detach().clone() for n, p in blk.named_parameters()}
    res = ours_mod.quantize_linears(blk, [torch.randn(4, 16, 64) for _ in range(2)], wbits=4, groupsize=32, act_order=False)
    assert set(res) == {'fc1', 'fc2'}
    for n, (scale, zero, g_idx, err) in res.items():
        lin = getattr(blk, n)
        K = lin.in_features
        assert scale.shape == (lin.out_features, K // 32) and zero.shape == scale.shape and g_idx.shape == (K, ) and err >= 0
        assert torch.equal(before[n + '.bias'], lin.bias.detach())  # biases are untouched (they travel as fp16 buffers of QuantLinear)
        # every weight sits on its group's grid: w = scale * (q - zero), q integer in [0, 15]
        q = lin.weight.data / scale.repeat_interleave(32, dim=1) + zero.repeat_interleave(32, dim=1)
        assert torch.allclose(q, q.round(), atol=1e-3) and q.min() >= -1e-3 and q.max() <= 15 + 1e-3
        assert (lin.weight.data - before[n + '.weight']).abs().mean() < scale.mean()  # moved by quantisation + error compensation, not destroyed
    sys.modules.pop('gptq', None)
