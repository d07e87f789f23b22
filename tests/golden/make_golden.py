"""Generate the golden pack() fixtures by running the UNMODIFIED reference.

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden.py REFERENCE_CHECKOUT

Imports ``quant`` from a checkout of the reference (the tests do not need it: the outputs are
committed as small .npz files next to this script).  For every case:
random fp weights -> per-group ``Quantizer`` (quant/quantizer.py, configured as in
gptq.py:185-194) -> on-grid weights Q -> the reference's own ``QuantLinear.pack``
(quant/quant_linear.py:325-371).  Stored: the inputs and the packed tensors the
reference produced, which pin the oracle's integer layout bit-exactly.
"""
import os
import sys

import numpy as np
import torch

sys.dont_write_bytecode = True
sys.path.insert(0, sys.argv[1])
import quant as refquant  # noqa: E402  (the reference package)
import torch.nn as nn  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))

CASES = [
    # name, bits, groupsize, K, N, act_order, bias
    ('b4_g128', 4, 128, 256, 64, False, False),
    ('b4_g128_act', 4, 128, 256, 64, True, False),
    ('b4_g32_bias', 4, 32, 128, 96, False, True),
    ('b4_gfull', 4, -1, 128, 64, False, False),
    ('b2_g64', 2, 64, 128, 64, False, False),
    ('b2_g64_act', 2, 64, 128, 64, True, False),
    ('b8_g128', 8, 128, 256, 32, False, False),
    ('b8_g128_act', 8, 128, 256, 32, True, True),
]


def make_case(name, bits, groupsize, K, N, act_order, bias, seed):
    gen = torch.Generator().manual_seed(seed)
    W = torch.randn(N, K, generator=gen) * 0.02
    gs = K if groupsize == -1 else groupsize
    G = K // gs
    g_idx = torch.arange(K) // gs
    if act_order:  # gptq.py:150-153 permutes columns, :213-216 maps g_idx back through invperm
        perm = torch.randperm(K, generator=gen)
        invperm = torch.argsort(perm)
        g_idx = g_idx[invperm]
    # per-group quantizer (gptq.py:185-194): columns of one group share scale/zero per output row
    scale = torch.zeros(N, G)
    zero = torch.zeros(N, G)
    Q = torch.zeros_like(W)
    for g in range(G):
        cols = (g_idx == g).nonzero().flatten()
        q = refquant.Quantizer()
        q.configure(bits, perchannel=True, sym=False, mse=False)
        q.find_params(W[:, cols], weight=True)
        Q[:, cols] = q.quantize(W[:, cols])
        scale[:, g] = q.scale.flatten()
        zero[:, g] = q.zero.flatten()
    lin = nn.Linear(K, N, bias=bias)
    lin.weight.data = Q.clone()
    if bias:
        lin.bias.data = torch.randn(N, generator=gen) * 0.1
    ql = refquant.QuantLinear(bits, groupsize, K, N, bias)
    ql.pack(lin, scale.clone(), zero.clone(), g_idx.to(torch.int32))
    out = dict(bits=bits, groupsize=groupsize, K=K, N=N, W=W.numpy(), Q=Q.numpy(), scale=scale.numpy(), zero=zero.numpy(), g_idx=ql.g_idx.numpy().astype(np.int32),
               qweight=ql.qweight.numpy(), qzeros=ql.qzeros.numpy(), scales_h=ql.scales.numpy())
    if bias:
        out['bias_h'] = ql.bias.detach().numpy()
    np.savez_compressed(os.path.join(HERE, f'pack_{name}.npz'), **out)
    print(name, 'qweight', ql.qweight.shape, 'qzeros', ql.qzeros.shape)


if __name__ == '__main__':
    for i, c in enumerate(CASES):
        make_case(*c, seed=100 + i)
