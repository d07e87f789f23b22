"""CPU: the fixtures of tests/test_gpu_exact.py really have order-independent exact answers.

The GPU tests compare kernels bit for bit against these expectations, so the expectations themselves are pinned here: the
integer-exact sums come out the same in fp32 summed sequentially, in fp32 summed pairwise and in fp64, and the one-hot
expectation equals the oracle's forward (O.qlinear_fwd) on the one-hot input."""
import numpy as np
import pytest
import torch

import exact_fixtures as X
from oracle import gptq_oracle as O


def _pairwise_fp32(p: np.ndarray) -> np.ndarray:
    """Tree sum over axis 0 in fp32 (zero-padded to a power of two)."""
    n = 1 << (p.shape[0] - 1).bit_length()
    t = np.zeros((n, ) + p.shape[1:], dtype=np.float32)
    t[:p.shape[0]] = p
    while t.shape[0] > 1:
        t = t[0::2] + t[1::2]
    return t[0]


@pytest.mark.parametrize('K,gs,lo,hi,jmin', [(11008, 128, -2, 2, 6), (4096, 128, -1, 1, 9), (4096, 64, -2, 2, 6)])
def test_integer_fixture_sums_are_exact_in_fp32(K, gs, lo, hi, jmin):
    N, M = 64, 3
    qw, s, qz, g = X.pow2_packed(K, N, gs, jmin=jmin, seed=K + jmin)
    W = O.dequant(qw, s, qz, g, 4)
    # every weight is exact in fp16: (q - z) * 2^-j
    q = torch.from_numpy(O.unpack_rows(qw.numpy(), 4)).double()
    z = torch.from_numpy(O.unpack_cols(qz.numpy(), 4)).double() + 1
    assert torch.equal(W.double(), (q - z[g.long()]) * s[g.long()].double())
    assert set(torch.unique(s).double().log2().tolist()) <= set(float(-j) for j in range(jmin, 11))
    x = X.int_x(M, K, lo, hi, seed=K)
    assert x.min() >= lo and x.max() <= hi
    exact = X.exact_product(x, W).numpy()
    Wn = W.double().numpy()
    for m in range(M):
        prod = x[m].double().numpy()[:, None] * Wn  # [K, N], exact
        assert np.all(prod * 1024 == np.round(prod * 1024)), 'products must be multiples of 2^-10'
        seq32 = np.cumsum(prod.astype(np.float32), axis=0, dtype=np.float32)  # every sequential partial sum
        seq64 = np.cumsum(prod, axis=0)
        assert np.array_equal(seq32.astype(np.float64), seq64), 'a sequential fp32 partial sum rounded'
        assert np.abs(seq64).max() < 2**13
        assert np.array_equal(seq64[-1], exact[m])
        assert np.array_equal(_pairwise_fp32(prod.astype(np.float32)).astype(np.float64), exact[m]), 'a pairwise fp32 sum rounded'
        # reversed order too (the k loop of another CTA split)
        assert np.array_equal(np.cumsum(prod[::-1].astype(np.float32), axis=0, dtype=np.float32)[-1].astype(np.float64), exact[m])


def test_mlp_fixture_cannot_overflow_fp16():
    """x in {-1, 0, 1} and scales <= 2^-9 at K = 4096: |a|, |b| <= 4096 * 16 * 2^-9 = 128, so |silu(a) * b| < 2^14."""
    K, N, gs = 4096, 64, 128
    Wg = O.dequant(*X.pow2_packed(K, N, gs, jmin=9, seed=1), 4).double()
    Wu = O.dequant(*X.pow2_packed(K, N, gs, jmin=9, seed=2), 4).double()
    x = X.int_x(4, K, -1, 1, seed=3).double()
    bound = x.abs() @ torch.ones(K, N, dtype=torch.float64) * 16 * 2.0**-9
    assert (bound <= 128).all()
    a, b = x @ Wg, x @ Wu
    assert ((a * torch.sigmoid(a) * b).abs() < 65504).all()


@pytest.mark.parametrize('bits,act,bias', [(4, False, True), (3, True, False), (8, True, True), (2, False, False)])
def test_onehot_expectation_matches_oracle_forward(bits, act, bias):
    K, N, gs = 256, 96, 64
    qw, s, qz, g, b = O.random_packed(K, N, bits, gs, act_order=act, seed=bits, bias=bias)
    W = O.dequant(qw, s, qz, g, bits)
    ks = list(range(K)) + [0, K - 1, 17]
    x, mult = X.onehot_rows(ks, K, salt=bits)
    assert set(mult.abs().log2().tolist()) == {-2.0, -1.0, 0.0, 1.0, 2.0} and (mult < 0).any()
    exp = X.onehot_expect(W, ks, mult, b)
    assert torch.equal(exp, O.qlinear_fwd(x, qw, s, qz, g, bits, b))


def test_sampled_ks_cover_the_k_loop_edges():
    K, gs, N = 11008, 128, 4096
    cta = X.matvec_cta_ks(K, N)
    ks = X.sampled_ks(K, gs, cta)
    assert set(k % 8 for k in ks) == set(range(8))
    assert all(b - 1 in ks and b in ks for b in range(gs, K, gs))
    assert cta - {-1} <= set(ks) and len(cta) > 30
    assert 0 in ks and K - 1 in ks


def test_matvec_plan_matches_the_kernel_at_7b_shapes():
    """Two column slabs per CTA at every 7B shape (so partials go through the workspace), and the CTA ranges tile the units."""
    for K, N in [(4096, 4096), (4096, 12288), (11008, 4096), (4096, 11008)]:
        nslabs, nk, U, nb = X.matvec_plan(K, N)
        assert nb == 264 and U > nb
        owners = [X.matvec_cta(K, N, k, n)[0] for n in range(0, N, 256) for k in range(0, K, 32)]
        assert owners == sorted(owners) and owners[0] == 0 and owners[-1] == nb - 1
        assert set(np.bincount(owners)) <= {U // nb, U // nb + 1}
        assert len({X.matvec_cta(K, N, 0, n)[0] for n in range(0, N, 256)}) == nslabs  # every slab starts in its own CTA
        assert nk == K // 32


# (K, N) of every quantized linear of the LLaMA-65B, LLaMA-2-70B, CodeLlama-34B and LLaMA-3-8B decode step (qkv, o_proj, gate|up, down_proj)
ROUTE_SHAPES = [(8192, 24576), (8192, 8192), (8192, 22016), (22016, 8192), (8192, 10240), (8192, 28672), (28672, 8192), (4096, 6144),
                (4096, 4096), (4096, 14336), (14336, 4096)]


def test_matvec_route_rule():
    """skinny_supported's shared-memory rule, worked by hand: the x segment of a CTA is ceil(U / 264) k-steps of 32 per row.  65B qkv at
    M = 8: 94 steps, 64 KB + 8 x 3040 x 2 B = 114176 B > 110 KB.  70B gate|up and down_proj: U = 28672, 109 steps, 64 KB + M x 7040 B:
    107776 B at M = 6, 114816 B at M = 7.  Every other (shape, M) of the table fits."""
    generic = {(8192, 24576, 8), (8192, 28672, 7), (8192, 28672, 8), (28672, 8192, 7), (28672, 8192, 8)}
    assert X.matvec_smem_bytes(8, 8192, 24576) == 114176
    assert X.matvec_smem_bytes(6, 8192, 28672) == X.matvec_smem_bytes(6, 28672, 8192) == 107776
    assert X.matvec_smem_bytes(7, 8192, 28672) == X.matvec_smem_bytes(7, 28672, 8192) == 114816
    for K, N in ROUTE_SHAPES:
        for M in range(1, 9):
            assert X.matvec_takes(M, K, N) == ((K, N, M) not in generic), f'M={M} K={K} N={N}: {X.matvec_smem_bytes(M, K, N)} B'
    assert not X.matvec_takes(9, 4096, 4096) and not X.matvec_takes(0, 4096, 4096)
