"""CPU model of the decode kernels' group arithmetic (csrc/decode_mega.cu: raw nibbles on the tensor pipe, the staged x scaled by a power
of two per staged range -- the odd nibbles' copy by 2^-4 more -- so that it stays an fp16 normal, scale and zero applied once per group on the
fp32 accumulator) against the float64 product and the oracle (the reference's per-weight fp16 rounding), over activation ranges a real model
can produce: O(1) RMSNorm outputs, tiny, large, heavy-tailed, dead features, small attention outputs (o_proj), small SwiGLU outputs
(down_proj, most of their mass far below 2^-10), a few massive residual features among O(1) ones, and all-positive inputs against zero
points of 16.  Every kind is held to the same bound.  The kernels themselves are checked on the GPU (tests/test_gpu_decode_input_ranges.py)."""
import numpy as np
import pytest
import torch

from oracle import gptq_oracle as O
from gpu_util import REL_TOL, assert_rel_close


def staging_exponent(xh):
    """decode_mega.cu x_scale: e such that the largest |x| of the staged range, times 2^e, lies in [2^14, 2^15) (clamped to [-1, 38]).
    The model stages the whole row as one range; the kernel's ranges of o_proj / down_proj are the teams' k-ranges (a smaller maximum
    only moves e up)."""
    m = float(np.abs(xh.astype(np.float32)).max())
    return 38 if m == 0 else min(max(14 - int(np.floor(np.log2(m))), -1), 38)


def kernel_model(x, qweight, scales, qzeros, bits=4, gs=128):
    """out[n] = fp16( sum_g s[g,n] * ( sum_{k in g} xe[k] * w[k,n]  -  z[g,n] * sum_{k in g} xe[k] ) ), products exact, fp32 accumulation per group."""
    K = x.shape[1]
    w = O.unpack_rows(qweight.numpy(), bits).astype(np.float64)            # [K, N] raw fields
    z = (O.unpack_cols(qzeros.numpy(), bits) + 1).astype(np.float64)       # [G, N], stored minus one
    s = scales.numpy().astype(np.float64)
    xh = x[0].numpy().astype(np.float16)
    odd = (np.arange(K) % 2) == 1                                          # nibbles 1, 3, 5, 7 of every packed word
    e = staging_exponent(xh)
    xe = (xh.astype(np.float32) * np.float32(2.0**e)).astype(np.float16).astype(np.float64) * 2.0**-e
    xe[odd] = (xh[odd].astype(np.float32) * np.float32(2.0**(e - 4))).astype(np.float16).astype(np.float64) * 2.0**(4 - e)  # what the tensor pipe effectively multiplies with
    out = np.zeros(w.shape[1], dtype=np.float64)
    for g in range(K // gs):
        sl = slice(g * gs, (g + 1) * gs)
        acc = np.float32((xe[sl, None] * w[sl]).sum(0))                    # exact products, fp32 accumulator
        xsum = np.float32(xe[sl].sum())
        out = np.float32(out + np.float32(s[g]) * (acc - np.float32(z[g]) * xsum))
    return torch.from_numpy(out.astype(np.float16))[None, :]


def exact(x, qweight, scales, qzeros, g_idx, bits=4):
    """The product in float64 from the stored fields: no per-weight rounding, no accumulation error."""
    w = O.unpack_rows(qweight.numpy(), bits).astype(np.float64)
    z = (O.unpack_cols(qzeros.numpy(), bits) + 1).astype(np.float64)
    g = g_idx.numpy()
    W = (w - z[g]) * scales.numpy().astype(np.float64)[g]
    return torch.from_numpy(x[0].numpy().astype(np.float64) @ W)[None, :]


def activations(kind, K):
    gen = torch.Generator().manual_seed(7)
    x = torch.randn(1, K, generator=gen)
    if kind == 'tiny':
        x = x * 3e-3
    elif kind == 'large':
        x = x * 300.0
    elif kind == 'heavy_tail':
        x = x * torch.exp(torch.randn(1, K, generator=gen) * 2.0)
    elif kind == 'dead_and_outliers':
        x[:, ::7] = 0.0
        x[:, 5::97] *= 500.0
    elif kind == 'near_subnormal':
        x = x * 2e-4  # many values below 2^-10
    elif kind.startswith('swiglu_'):  # down_proj input h = silu(4 sigma e) sigma e' (fp16), sigma from the kind's name
        sigma = float(kind.split('_')[1])
        a = 4 * sigma * x
        x = a * torch.sigmoid(a) * sigma * torch.randn(1, K, generator=gen)
    elif kind.startswith('attn_'):  # o_proj input: attention outputs N(0, sigma^2)
        x = x * float(kind.split('_')[1])
    elif kind == 'massive':  # residual row with a few massive features (+-1e3 ... 4e3) among O(1) ones
        idx = torch.randperm(K, generator=gen)[:4]
        x[0, idx] = torch.tensor([1e3, -2e3, 3e3, -4e3])
    elif kind == 'positive':  # all-positive inputs (paired with zero points of 16 below)
        x = x.abs() * 1e-2
    x = x.half()
    assert torch.isfinite(x).all()
    return x


KINDS = ['normal', 'tiny', 'large', 'heavy_tail', 'dead_and_outliers', 'near_subnormal', 'massive', 'positive']
KINDS += [f'swiglu_{s}' for s in ('0.05', '0.02', '0.01', '0.005', '0.002')] + [f'attn_{s}' for s in ('0.01', '0.001', '0.0003')]


def shape(kind):
    """(K, N) of the linear the kind feeds: down_proj at LLaMA-7B for SwiGLU outputs, o_proj (K = 4096) for attention outputs."""
    return (11008, 256) if kind.startswith('swiglu_') else (4096, 256) if kind.startswith('attn_') else (1024, 256)


def fields(kind):
    K, N = shape(kind)
    qw, s, qz, g, _ = O.random_packed(K, N, 4, 128, seed=3)
    if kind == 'positive':
        qz = torch.full_like(qz, -1)  # every stored zero 15: z = 16, every weight (q - 16) s < 0
    return qw, s, qz, g


@pytest.mark.parametrize('kind', KINDS)
def test_regrouped_arithmetic_is_within_tolerance_of_exact(kind):
    """Against the float64 product the model is off by the final fp16 rounding (half an ulp, <= 4.9e-4 relative) plus fp32 accumulation
    noise: inside the 1e-3 of the north star for every activation range, where the reference's own per-weight fp16 rounding is not always
    (heavy tails: a few large x_k carry the weight-rounding error of their column straight into the output).  With the staged x kept in
    fp16 normals this holds for inputs far below 2^-10 too (SwiGLU and attention outputs); the parent's fixed 1/16 pre-scaling of the
    odd nibbles' x lost up to 4 bits of each of them there (3e-3 to 9e-2 off)."""
    qw, s, qz, g = fields(kind)
    x = activations(kind, qw.shape[0] * 8)
    ex = exact(x, qw, s, qz, g)
    out = kernel_model(x, qw, s, qz)
    assert_rel_close(out, ex, rel=REL_TOL, what=kind)
    ref = O.qlinear_fwd(x, qw, s, qz, g, 4)
    err_model = (out.double() - ex).abs().max().item()
    err_ref = (ref.double() - ex).abs().max().item()
    assert err_model <= err_ref * 1.01 + 1e-12, (kind, err_model, err_ref)  # never further from exact than the reference is


def test_small_inputs_stay_exact_when_staged():
    """The staged x of the model is the fp16 input itself, scaled by powers of two: no input below 2^-10 loses a bit."""
    for kind in ('near_subnormal', 'swiglu_0.002', 'attn_0.0003'):
        xh = activations(kind, shape(kind)[0])[0].numpy()
        e = staging_exponent(xh)
        for f in (2.0**e, 2.0**(e - 4)):
            staged = (xh.astype(np.float32) * np.float32(f)).astype(np.float16)
            assert np.array_equal(staged.astype(np.float64) / f, xh.astype(np.float64)), kind


@pytest.mark.parametrize('kind', ['normal', 'tiny', 'dead_and_outliers'])
def test_regrouped_arithmetic_matches_the_reference(kind):
    """... and within 1e-3 of the reference itself on the activation ranges where the reference is within 1e-3 of exact."""
    K, N = 1024, 256
    qw, s, qz, g, _ = O.random_packed(K, N, 4, 128, seed=3)
    x = activations(kind, K)
    assert_rel_close(kernel_model(x, qw, s, qz), O.qlinear_fwd(x, qw, s, qz, g, 4), what=kind)
