"""CPU: the algebra behind gptq_b200.ops.QLayerWeights.kernel_form (load-time derived buffers), restated with the oracle's pack/unpack.

Regrouping act-order rows by a stable sort on the group and widening 2/3-bit fields to nibbles must leave every
dequantised weight bit-identical (rows permuted), so the only difference between the derived form and the stored
form is the fp32 summation order.  The CUDA implementation is checked against the oracle in tests/test_gpu_modules.py;
this file pins the identity itself without a GPU."""
import numpy as np
import pytest
import torch

from oracle import gptq_oracle as O


def _kernel_form_oracle(qw, s, qz, g, bits, gs):
    K = qw.shape[0] * 32 // bits
    rows = O.unpack_rows(qw.numpy(), bits)
    perm = torch.argsort(g[:K].long(), stable=True)
    rows = rows[perm.numpy()]
    new_bits = 4 if bits in (2, 3) else bits
    zeros = O.unpack_cols(qz.numpy(), bits)
    qw2 = torch.from_numpy(O.pack_rows(rows, new_bits))
    qz2 = torch.from_numpy(O.pack_cols(zeros, new_bits))
    g2 = (torch.arange(K) // gs).to(torch.int32)
    return qw2, qz2, g2, new_bits, perm


@pytest.mark.parametrize('bits', [2, 3, 4, 8])
@pytest.mark.parametrize('act', [False, True])
def test_regrouped_and_widened_layer_has_the_same_weights(bits, act):
    K, N, gs = 256, 64, 64
    qw, s, qz, g, _ = O.random_packed(K, N, bits, gs, act_order=act, seed=10 * bits + act)
    qw2, qz2, g2, nb, perm = _kernel_form_oracle(qw, s, qz, g, bits, gs)
    W = O.dequant(qw, s, qz, g, bits)
    W2 = O.dequant(qw2, s, qz2, g2, nb)
    assert torch.equal(W2, W.index_select(0, perm))
    if not act:
        assert torch.equal(perm, torch.arange(K))
    # groups are contiguous after the regrouping, every row kept its own group
    assert torch.equal(g[perm].long(), g2.long())
    x = torch.randn(3, K, generator=torch.Generator().manual_seed(1)).half()
    ref = O.qlinear_fwd(x, qw, s, qz, g, bits).float()
    out = O.qlinear_fwd(x.index_select(1, perm), qw2, s, qz2, g2, nb).float()
    assert float((out - ref).abs().max()) <= 1e-3 * float(ref.pow(2).mean().sqrt()) + 1e-6


def test_column_permutation_folds_the_next_layers_gather():
    """down(h[perm]) with regrouped rows == down(h): permuting the OUTPUT columns of gate|up by down's map makes the
    fused SwiGLU output come out in down's regrouped order (engine.kernel_layers)."""
    H, I, gs, bits = 128, 256, 64, 4
    gate = O.random_packed(H, I, bits, gs, seed=1)[:4]
    up = O.random_packed(H, I, bits, gs, seed=2)[:4]
    dqw, ds, dqz, dg, _ = O.random_packed(I, H, bits, gs, act_order=True, seed=3)
    dqw2, dqz2, dg2, _, perm = _kernel_form_oracle(dqw, ds, dqz, dg, bits, gs)

    def permute_cols(w):
        qw, s, qz, g = w
        zeros = O.unpack_cols(qz.numpy(), bits)[:, perm.numpy()]
        return qw[:, perm].contiguous(), s[:, perm].contiguous(), torch.from_numpy(O.pack_cols(np.ascontiguousarray(zeros), bits)), g

    x = torch.randn(2, H, generator=torch.Generator().manual_seed(0)).half()
    h = O.fused_mlp_fwd(x, gate, up, bits)
    h_folded = O.fused_mlp_fwd(x, permute_cols(gate), permute_cols(up), bits)
    assert torch.equal(h_folded, h.index_select(1, perm))  # column-wise independent: bit-identical
    ref = O.qlinear_fwd(h, dqw, ds, dqz, dg, bits).float()
    out = O.qlinear_fwd(h_folded, dqw2, ds, dqz2, dg2, bits).float()
    assert float((out - ref).abs().max()) <= 1e-3 * float(ref.pow(2).mean().sqrt()) + 1e-6
