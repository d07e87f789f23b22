"""GPU parity tests proper: the CUDA path, called through the C ABI (gptq_b200.ops -> libgptq_b200.so),
against the CPU oracle on the same seeded inputs and against the golden fixtures."""
import numpy as np
import pytest
import torch

from oracle import gptq_oracle as O
from gpu_util import assert_rel_close, cuda

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def ops():
    from gptq_b200 import ops as _ops  # raises if libgptq_b200.so is missing: no fallback
    return _ops


# ----------------------------------------------------------------------------- integer work: bit-exact
@pytest.mark.parametrize('bits', [2, 3, 4, 8])
def test_pack_unpack_bit_exact(ops, bits):
    rng = np.random.default_rng(bits)
    K, N, G = 256, 96, 4
    w = rng.integers(0, 2**bits, size=(K, N)).astype(np.int32)
    z = rng.integers(0, 2**bits, size=(G, N)).astype(np.int32)
    qw = ops.pack_qweight(torch.from_numpy(w).cuda(), bits)
    qz = ops.pack_qzeros(torch.from_numpy(z).cuda(), bits)
    assert np.array_equal(qw.cpu().numpy(), O.pack_rows(w, bits))
    assert np.array_equal(qz.cpu().numpy(), O.pack_cols(z, bits))
    assert np.array_equal(ops.unpack_qweight(qw, bits).cpu().numpy(), w)
    assert np.array_equal(ops.unpack_qzeros(qz, bits).cpu().numpy(), z)


def test_golden_unpack_and_dequant(ops, golden_cases):
    """Reference-packed tensors: device unpack == oracle unpack (bit-exact); device dequant == oracle dequant (bit-exact fp16)."""
    for name, d in golden_cases.items():
        bits = int(d['bits'])
        qw, qz, sc, gi = (torch.from_numpy(d[k]).cuda() for k in ('qweight', 'qzeros', 'scales_h', 'g_idx'))
        assert np.array_equal(ops.unpack_qweight(qw, bits).cpu().numpy(), O.unpack_rows(d['qweight'], bits)), name
        assert np.array_equal(ops.unpack_qzeros(qz, bits).cpu().numpy(), O.unpack_cols(d['qzeros'], bits)), name
        W = ops.dequant(qw, sc, qz, gi, bits)
        Wref = O.dequant(*(torch.from_numpy(d[k]) for k in ('qweight', 'scales_h', 'qzeros', 'g_idx')), bits)
        assert torch.equal(W.cpu(), Wref), name
        assert (W.float().t().cpu() - torch.from_numpy(d['Q'])).abs().max() < 1e-4


def test_quantlinear_pack_matches_reference_pack(golden_cases):
    """QuantLinear.pack (GPU) reproduces the reference's CPU pack() bit for bit."""
    import quant
    import torch.nn as nn
    for name, d in golden_cases.items():
        bits, gs, K, N = int(d['bits']), int(d['groupsize']), int(d['K']), int(d['N'])
        lin = nn.Linear(K, N, bias='bias_h' in d)
        lin.weight.data = torch.from_numpy(d['Q']).clone()
        if 'bias_h' in d:
            lin.bias.data = torch.from_numpy(d['bias_h']).float()
        ql = quant.QuantLinear(bits, gs, K, N, 'bias_h' in d)
        ql.pack(lin, torch.from_numpy(d['scale']).clone(), torch.from_numpy(d['zero']).clone(), torch.from_numpy(d['g_idx']))
        assert np.array_equal(ql.qweight.cpu().numpy(), d['qweight']), name
        assert np.array_equal(ql.qzeros.cpu().numpy(), d['qzeros']), name
        assert np.array_equal(ql.scales.cpu().numpy(), d['scales_h']), name
        assert np.array_equal(ql.g_idx.cpu().numpy(), d['g_idx']), name


# ----------------------------------------------------------------------------- qlinear forward
@pytest.mark.parametrize('bits', [2, 3, 4, 8])
@pytest.mark.parametrize('act', [False, True])
@pytest.mark.parametrize('M', [1, 2, 3, 8, 17])
def test_qlinear_vs_oracle(ops, bits, act, M):
    K, N, gs = 512, 256, 128
    qw, s, qz, g, b = O.random_packed(K, N, bits, gs, act_order=act, seed=10 * bits + M, bias=(M % 2 == 0))
    x = torch.randn(M, K, generator=torch.Generator().manual_seed(M)).half()
    ref = O.qlinear_fwd(x, qw, s, qz, g, bits, b)
    dqw, ds, dqz, dg, db, dx = cuda(qw, s, qz, g, b, x)
    out = ops.matmul248(dx, dqw, ds, dqz, dg, bits, 2**bits - 1, bias=db, groupsize=0)
    assert_rel_close(out, ref, what=f'gather bits={bits} act={act} M={M}')
    if not act:  # trivial g_idx: the groupsize hint must give the same answer
        out2 = ops.matmul248(dx, dqw, ds, dqz, dg, bits, 2**bits - 1, bias=db, groupsize=gs)
        assert_rel_close(out2, ref, what=f'hint bits={bits} M={M}')


@pytest.mark.parametrize('K,N,gs', [(128, 32, 32), (4096, 64, 128), (256, 4096, -1), (11008, 96, 128), (96, 160, 32)])
def test_qlinear_shapes(ops, K, N, gs):
    qw, s, qz, g, _ = O.random_packed(K, N, 4, gs, seed=K + N)
    x = torch.randn(2, K, generator=torch.Generator().manual_seed(0)).half()
    ref = O.qlinear_fwd(x, qw, s, qz, g, 4)
    out = ops.matmul248(x.cuda(), *cuda(qw, s, qz, g), 4, 15, groupsize=(K if gs == -1 else gs))
    assert_rel_close(out, ref, what=f'K={K} N={N} gs={gs}')


def test_qlinear_golden_fixture_with_bias(ops, golden_cases):
    for name, d in golden_cases.items():
        bits = int(d['bits'])
        t = {k: torch.from_numpy(d[k]) for k in ('qweight', 'scales_h', 'qzeros', 'g_idx')}
        b = torch.from_numpy(d['bias_h']) if 'bias_h' in d else None
        x = torch.randn(3, int(d['K']), generator=torch.Generator().manual_seed(7)).half()
        ref = O.qlinear_fwd(x, t['qweight'], t['scales_h'], t['qzeros'], t['g_idx'], bits, b)
        out = ops.matmul248(x.cuda(), t['qweight'].cuda(), t['scales_h'].cuda(), t['qzeros'].cuda(), t['g_idx'].cuda(), bits, None,
                            bias=b.cuda() if b is not None else None)
        assert_rel_close(out, ref, what=name)


def test_strided_input_and_empty_batch(ops):
    K, N = 256, 64
    qw, s, qz, g, _ = O.random_packed(K, N, 4, 128, seed=5)
    big = torch.randn(4, 2 * K, generator=torch.Generator().manual_seed(0)).half()
    x = big[:, :K]  # row stride 2K
    ref = O.qlinear_fwd(x, qw, s, qz, g, 4)
    out = ops.matmul248(x.cuda()[:, :], *cuda(qw, s, qz, g), 4, 15)
    assert_rel_close(out, ref)
    xs = big.cuda()[:, :K]
    assert xs.stride(0) == 2 * K
    assert_rel_close(ops.matmul248(xs, *cuda(qw, s, qz, g), 4, 15), ref, what='strided')
    empty = ops.matmul248(torch.empty(0, K, dtype=torch.float16, device='cuda'), *cuda(qw, s, qz, g), 4, 15)
    assert empty.shape == (0, N)


@pytest.mark.parametrize('bits', [2, 3, 4, 8])
def test_transpose_matmul_vs_oracle(ops, bits):
    K, N = 256, 128
    qw, s, qz, g, _ = O.random_packed(K, N, bits, 64, act_order=True, seed=bits)
    gr = torch.randn(3, N, generator=torch.Generator().manual_seed(1)).half()
    ref = O.qlinear_transpose_fwd(gr, qw, s, qz, g, bits)
    out = ops.transpose_matmul248(gr.cuda(), *cuda(qw, s, qz, g), bits, None)
    assert_rel_close(out, ref, what=f'transpose bits={bits}')


# ----------------------------------------------------------------------------- fused MLP / RoPE / RMSNorm
@pytest.mark.parametrize('bits', [2, 3, 4, 8])
@pytest.mark.parametrize('act', [False, True])
@pytest.mark.parametrize('M', [1, 5])
def test_fused_mlp_vs_oracle(ops, bits, act, M):
    K, N, gs = 256, 352, 64
    gate = O.random_packed(K, N, bits, gs, act_order=act, seed=1)[:4]
    up = O.random_packed(K, N, bits, gs, act_order=act, seed=2)[:4]
    x = (torch.randn(M, K, generator=torch.Generator().manual_seed(3)) * 2).half()
    ref = O.fused_mlp_fwd(x, gate, up, bits)
    out = ops.fused_mlp(x.cuda(), cuda(*gate), cuda(*up), bits, 0 if act else gs)
    assert_rel_close(out, ref, rel=2e-3, what=f'mlp bits={bits} act={act} M={M}')  # product of two rounded dots


@pytest.mark.parametrize('shape', [(1, 1, 32, 128), (2, 5, 4, 64), (1, 7, 2, 16)])
def test_rope_vs_oracle(ops, shape):
    bsz, seq, heads, hd = shape
    gen = torch.Generator().manual_seed(0)
    qkv = torch.randn(bsz, seq, 3, heads, hd, generator=gen).half()
    pos = torch.randint(0, 2048, (bsz, seq), generator=gen)
    ref = qkv.clone()
    O.rope_inplace(ref[:, :, :2], pos)
    dq = qkv.cuda()
    ops.rotate_half_(dq[:, :, :2], pos.cuda())
    assert torch.equal(dq[:, :, 2].cpu(), qkv[:, :, 2]), 'v must be untouched'
    # fp16 store of fp32 rotations computed with different sin/cos implementations: 1 ulp + tiny absolute slack at large angles
    assert torch.allclose(dq.float().cpu(), ref.float(), rtol=2e-3, atol=2e-3)
    assert (dq.float().cpu() - ref.float()).abs().mean() < 2e-4


@pytest.mark.parametrize('M,N', [(1, 4096), (3, 5120), (2, 64), (5, 8192)])
def test_rmsnorm_vs_oracle(ops, M, N):
    gen = torch.Generator().manual_seed(N)
    x = (torch.randn(M, N, generator=gen) * 3).half()
    w = (torch.rand(N, generator=gen) + 0.5).half()
    ref = O.rmsnorm_fwd(x, w, 1e-6)
    out = ops.rmsnorm(x.cuda(), w.cuda(), 1e-6)
    assert_rel_close(out, ref, what=f'rmsnorm {M}x{N}')


def test_error_mapping_on_device(ops):
    qw, s, qz, g, _ = O.random_packed(128, 32, 4, 128)
    with pytest.raises(NotImplementedError):
        ops.matmul248(torch.zeros(1, 128).half().cuda(), *cuda(qw, s, qz, g), 5, 31)
    with pytest.raises(ValueError):
        ops.matmul248(torch.zeros(1, 64).half().cuda(), *cuda(qw, s, qz, g), 4, 15)
    with pytest.raises(ValueError, match='cuda'):
        ops.matmul248(torch.zeros(1, 128).half(), qw, s, qz, g, 4, 15)


# ----------------------------------------------------------------------------- batched (prefill) path: wgmma GEMM
@pytest.mark.parametrize('M,K,N,gs', [(16, 512, 256, 128), (100, 1024, 384, 64), (128, 256, 128, 128), (300, 2048, 512, 128), (129, 128, 128, 64)])
def test_prefill_gemm_vs_oracle(ops, M, K, N, gs):
    """M > 8, int4, no act-order: wgmma GEMM (qgemm_wgmma.cu) against the CPU oracle."""
    qw, s, qz, g, b = O.random_packed(K, N, 4, gs, seed=M + K, bias=(M % 2 == 0))
    x = torch.randn(M, K, generator=torch.Generator().manual_seed(M)).half()
    ref = O.qlinear_fwd(x, qw, s, qz, g, 4, b)
    out = ops.matmul248(x.cuda(), *cuda(qw, s, qz, g), 4, 15, bias=b.cuda() if b is not None else None, groupsize=gs)
    # tensor-core fp32 accumulation is not IEEE round-to-nearest per add (the reference's tl.dot has the same property): allow 2 fp16 ulps
    assert_rel_close(out, ref, rel=2e-3, what=f'prefill M={M} K={K} N={N} gs={gs}')


def test_prefill_gemm_full_size_matches_dequant_matmul(ops):
    """LLaMA-7B layer size, M = 512: wgmma GEMM == fp32 matmul over the device-dequantised weight; exact homogeneity."""
    K, N, M = 4096, 4096, 512
    qw, s, qz, g, _ = cuda(*O.random_packed(K, N, 4, 128, seed=3))
    x = torch.randn(M, K, generator=torch.Generator().manual_seed(0)).half().cuda()
    W = ops.dequant(qw, s, qz, g, 4, 128)
    ref = (x.float() @ W.float()).half()
    out = ops.matmul248(x, qw, s, qz, g, 4, 15, groupsize=128)
    assert_rel_close(out, ref, rel=2e-3, what='prefill full size')
    out2 = ops.matmul248(x * 2, qw, s, qz, g, 4, 15, groupsize=128)
    normal = out.abs() > 1e-3  # fp16 subnormal results do not scale exactly
    assert torch.equal(out2[normal], (out * 2)[normal])
    assert torch.equal(ops.matmul248(x, qw, s, qz, g, 4, 15, groupsize=128), out)  # deterministic


@pytest.mark.parametrize('M', [24, 200])
def test_prefill_fused_mlp_vs_oracle(ops, M):
    """Fused SwiGLU MLP at M > 8: dual-accumulator wgmma GEMM, silu*mul on the fp32 accumulators in the epilogue."""
    K, N, gs = 512, 384, 128
    gate = O.random_packed(K, N, 4, gs, seed=1)[:4]
    up = O.random_packed(K, N, 4, gs, seed=2)[:4]
    x = (torch.randn(M, K, generator=torch.Generator().manual_seed(3)) * 2).half()
    ref = O.fused_mlp_fwd(x, gate, up, 4)
    out = ops.fused_mlp(x.cuda(), cuda(*gate), cuda(*up), 4, gs)
    assert_rel_close(out, ref, rel=3e-3, what=f'prefill fused mlp M={M}')
