"""CPU: the oracle's transposed product, which the GPU backward tests lean on, held to float64 at a LLaMA-7B shape."""
import torch

from oracle import gptq_oracle as O


def test_oracle_transpose_matches_float64_at_a_llama_7b_shape():
    """o_proj of LLaMA-7B (4096 x 4096, int4, groupsize 128): O.qlinear_transpose_fwd(g) == g . W^T of the oracle's own fp16 weight
    evaluated in float64, within one fp16 spacing of the result plus the fp32 accumulation of 4096 products (any summation order)."""
    K, N, gs, M = 4096, 4096, 128, 5
    qw, s, qz, gi, _ = O.random_packed(K, N, 4, gs, seed=3)
    g = torch.randn(M, N, generator=torch.Generator().manual_seed(1)).half()
    out = O.qlinear_transpose_fwd(g, qw, s, qz, gi, 4)
    assert out.shape == (M, K) and out.dtype == torch.float16
    W = O.dequant(qw, s, qz, gi, 4).double()
    ref = g.double() @ W.t()
    ulp = torch.pow(2.0, torch.floor(torch.log2(ref.abs().clamp_min(2.0**-14))) - 10)
    bound = ulp + N * 2.0**-24 * (g.double().abs() @ W.abs().t())
    ratio = ((out.double() - ref).abs() / bound).max().item()
    assert ratio <= 1, f'worst |err| / bound = {ratio:.3g}'
    # a one-hot gradient row returns a column of W^T, i.e. row n of the weight's transpose, exactly
    e = torch.zeros(1, N, dtype=torch.float16)
    e[0, 1234] = 2.0
    assert torch.equal(O.qlinear_transpose_fwd(e, qw, s, qz, gi, 4)[0].double(), 2.0 * W[:, 1234])
