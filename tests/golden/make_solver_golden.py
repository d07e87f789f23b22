"""Generate tests/golden/solver_ref.npz: what the reference's own GPTQ solver (gptq.py, imported unmodified) computes on the
layers and calibration batches of tests/test_gptq_solver.py.

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_solver_golden.py REFERENCE_CHECKOUT

Its table-printing dependency `texttable` and the SNR helper it pulls from `utils` are stubbed: neither touches the result.
Stored per case: g_idx, scales, zeros, the reported error, the on-grid weights as integer codes (the weight is
scale * (code - zero), exactly the reference's Quantizer arithmetic) and a fixed sample of the Hessian.
"""
import importlib
import os
import sys
import types

import numpy as np
import torch
import torch.nn as nn

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, 'solver_ref.npz')

CASES = [(256, 96, 4, 64, False), (256, 96, 4, 128, True), (192, 64, 3, -1, False), (256, 64, 8, 128, False), (256, 96, 2, 32, True)]  # K, N, bits, groupsize, actorder
H_SAMPLES = 512


def case_name(K, N, bits, groupsize, actorder):
    return f'K{K}_N{N}_b{bits}_g{groupsize}' + ('_act' if actorder else '')


def make_inputs(K, N, bits):
    """The layer weight and the calibration batches: correlated inputs with a few dominant (and one dead) features, so that
    act-order actually reorders."""
    g = torch.Generator().manual_seed(K + N + bits)
    weight = torch.randn(N, K, generator=g) * 0.05
    mix = torch.randn(K, K, generator=g) * 0.2 + torch.eye(K)
    gain = torch.rand(K, generator=g) * 3 + 0.1
    gain[5] = 0.0
    batches = [(torch.randn(2, 24, K, generator=g) @ mix) * gain for _ in range(3)]
    return weight, batches


def h_sample(K):
    """Fixed entries of the K x K Hessian compared with the stored sample (the diagonal is stored whole)."""
    g = torch.Generator().manual_seed(K)
    return torch.randint(0, K, (H_SAMPLES, ), generator=g), torch.randint(0, K, (H_SAMPLES, ), generator=g)


def codes(W, scale, zero, g_idx, bits):
    """Integer grid codes of on-grid weights W = scale * (code - zero) (per output row, per group g_idx[k])."""
    s, z = scale[:, g_idx.long()], zero[:, g_idx.long()]
    return torch.clamp(torch.round(W / s + z), 0, 2**bits - 1).to(torch.uint8)


def solve(module, K, N, bits, groupsize, actorder):
    weight, batches = make_inputs(K, N, bits)
    lin = nn.Linear(K, N, bias=True)
    lin.weight.data = weight.clone()
    s = module.GPTQ(lin)
    s.quantizer.configure(bits, perchannel=True, sym=False, mse=False)
    for x in batches:
        s.add_batch(x, None)
    H = s.H.clone()
    scale, zero, g_idx, err = s.fasterquant(blocksize=128, percdamp=.01, groupsize=groupsize, actorder=actorder, name='t')
    return H, scale.cpu(), zero.cpu(), g_idx.cpu(), float(err), lin.weight.data.clone()


def _reference_gptq(ref_dir):
    sys.path.insert(0, os.path.join(os.path.dirname(HERE), '..', 'gptq-for-llama_b200'))
    import utils as ours
    tt = types.ModuleType('texttable')

    class Texttable:  # only used to print one line per layer
        def header(self, *a): pass
        def set_cols_dtype(self, *a): pass
        def add_row(self, *a): pass
        def draw(self): return 'a\nb\nc'
    tt.Texttable = Texttable
    shim = types.ModuleType('utils')
    shim.find_layers, shim.DEV = ours.find_layers, ours.DEV
    shim.torch_snr_error = lambda a, b, reduction='mean': ((a - b)**2 / (b**2 + 1e-12)).mean()
    sys.modules.update(texttable=tt, utils=shim)
    sys.modules.pop('gptq', None)
    sys.path.insert(0, ref_dir)
    ref = importlib.import_module('gptq')
    assert os.path.abspath(ref.__file__).startswith(os.path.abspath(ref_dir))
    torch.cuda.synchronize = lambda *a, **k: None  # the reference synchronises unconditionally (gptq.py:205)
    return ref


def main(ref_dir):
    sys.dont_write_bytecode = True
    ref = _reference_gptq(ref_dir)
    out = {}
    for case in CASES:
        K, N, bits, groupsize, actorder = case
        H, scale, zero, g_idx, err, W = solve(ref, *case)
        r, c = h_sample(K)
        n = case_name(*case)
        q = codes(W, scale, zero, g_idx, bits)
        assert torch.equal(scale[:, g_idx.long()] * (q.float() - zero[:, g_idx.long()]), W), n  # the codes reproduce the weights exactly
        out.update({f'{n}/g_idx': g_idx.numpy().astype(np.int32), f'{n}/scale': scale.numpy(), f'{n}/zero': zero.numpy(), f'{n}/err': np.float64(err),
                    f'{n}/codes': q.numpy(), f'{n}/H_diag': torch.diagonal(H).numpy(), f'{n}/H_sample': H[r, c].numpy()})
    np.savez_compressed(OUT, **out)
    print(f'wrote {len(out)} arrays to {OUT} ({os.path.getsize(OUT)} bytes)')


if __name__ == '__main__':
    main(sys.argv[1])
