"""Helpers shared by the GPU parity tests."""
import time

import numpy as np
import pytest
import torch

REL_TOL = 1e-3  # north_star: outputs within 1e-3 relative of the reference's dequant->fp16 matmul


def assert_rel_close(out: torch.Tensor, ref: torch.Tensor, rel: float = REL_TOL, what: str = ''):
    """|out - ref| <= rel * max(|ref|, rms(ref)) element-wise; prints the worst |err| / bound (visible under -s).

    fp16 results that differ only by the fp32 summation order sit within one fp16 ulp (<= 9.8e-4 relative);
    the rms floor covers outputs that cancel to ~0, where a relative bound is meaningless."""
    out32, ref32 = out.detach().float().cpu(), ref.detach().float().cpu()
    assert out32.shape == ref32.shape, (out32.shape, ref32.shape)
    assert torch.isfinite(out32).all(), f'{what}: non-finite output'
    rms = ref32.pow(2).mean().sqrt().item()
    bound = rel * torch.maximum(ref32.abs(), torch.full_like(ref32, rms)) + 1e-7
    err = (out32 - ref32).abs()
    print(f'  {what}: worst |err| / bound = {(err / bound).max().item():.3g} (bound {rel:g})')
    bad = err > bound
    assert not bad.any(), f'{what}: {int(bad.sum())} / {bad.numel()} elements off; max err {err.max().item():.3e}, rms(ref) {rms:.3e}'


def cuda(*ts):
    return tuple(t.cuda() if t is not None else None for t in ts)


# ----------------------------------------------------------------------------- which kernel ran
def launched_kernels(fn):
    """Run fn() under torch.profiler (launch and kernel activity records, no hardware counters) -> (fn's result, set of names
    of the device-side events).

    Names are the demangled ones, e.g. 'void gptq::(anonymous namespace)::qmatvec_int4_kernel<false>(...)'.  The traced window
    is padded by a few milliseconds on both sides, so that device activity at either end of it is not cut off."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        time.sleep(0.003)
        res = fn()
        torch.cuda.synchronize()
        time.sleep(0.003)
    events = prof.events()
    return res, {e.name for e in events if e.device_type == torch.autograd.DeviceType.CUDA}


def run_kernel(fn, kernel: str, what: str = ''):
    """fn() must launch `kernel` (a demangled name with its template arguments, e.g. 'qgemm_wgmma_kernel<false, 2, 4>') and no
    other quantized-linear kernel.  Returns fn's result.

    fn must be repeatable: a trace without any kernel record (the launch call was traced, the kernel was not; seen on an H100
    about once in 200 sessions) is taken again, up to three times.  A machine whose activity tracing returns no CUDA events at
    all skips the test: a routing assertion that cannot see kernels must not pass."""
    strip = lambda s: s.replace(' ', '')
    families = ('qmatvec_int4_kernel', 'qgemm_wgmma_kernel', 'qlinear_generic_kernel', 'qlinear_transpose_generic_kernel')
    for _ in range(3):
        res, names = launched_kernels(fn)
        if names:
            break
    if not names:
        pytest.skip(f'{what}: CUDA activity tracing returned no kernel events on this machine')
    qk = sorted(n for n in names if any(f + '<' in n for f in families))
    hit = [n for n in qk if strip(kernel) in strip(n)]
    assert hit and len(hit) == len(qk), f'{what}: expected {kernel}, launched {sorted(names)}'
    return res


# ----------------------------------------------------------------------------- fp64 reference with an element-wise bound
def ulp16(v: torch.Tensor) -> torch.Tensor:
    """Spacing of fp16 numbers at |v| (2^-24 in the subnormal range); v in float64."""
    e = torch.floor(torch.log2(v.abs().clamp_min(2.0**-14)))
    return torch.pow(2.0, e - 10)


def fp32_sum_bound(A: torch.Tensor, depth: float) -> torch.Tensor:
    """Worst-case error of an fp32 sum of exact products whose absolute values sum to A, accumulated `depth` additions deep
    (round to nearest, 2^-24 relative per addition)."""
    return depth * 2.0**-24 * A


def default_depth(K: int) -> float:
    """Accumulation depth of the tensor-core kernels: K/16 sequential k16 mma / wgmma steps, plus 64 for the inside of an mma
    and the split-K partial reduction of the matvec."""
    return K / 16 + 64


def report(ratio: float, what: str, limit: float = 1.0):
    """Print the worst |err| / bound (visible under -s) and fail above `limit`."""
    print(f'  {what}: worst |err| / bound = {ratio:.3g}')
    assert ratio <= limit, f'{what}: worst |err| / bound = {ratio:.3g}'


def _where(bad: torch.Tensor, locate) -> str:
    idx = [int(i) for i in torch.nonzero(bad)[0]]
    return locate(*idx) if locate is not None else f'first bad index {tuple(idx)}'


def check_fp64_bound(out, x, W, bias=None, what='', depth=None, locate=None) -> float:
    """out[M, N] (fp16, device) against the fp64 product of the fp16 x [M, K] and the oracle's fp16 weight W [K, N] (+ bias):

        |out - ref| <= ulp16(max(|x.W|, |ref|)) + depth * 2^-24 * (|x| . |W|)

    The first term covers the fp16 store of the accumulator and the fp16 bias add after it (hence the larger of the two
    magnitudes: a bias can cancel the product); the second bounds the fp32 accumulation (default_depth).  Returns the worst
    |err| / bound and fails, naming the first offending element (locate(m, n) -> str), if it exceeds 1."""
    x64, W64 = x.to('cuda', torch.float64), W.to('cuda', torch.float64)
    acc = x64 @ W64
    A = x64.abs() @ W64.abs()
    ref = acc if bias is None else acc + bias.to('cuda', torch.float64)
    bound = ulp16(torch.maximum(acc.abs(), ref.abs())) + fp32_sum_bound(A, default_depth(W.shape[0]) if depth is None else depth)
    out64 = out.to(torch.float64)
    assert torch.isfinite(out64).all(), f'{what}: non-finite output'
    ratio_t = (out64 - ref).abs() / bound
    ratio = ratio_t.max().item()
    if ratio > 1:
        what = f'{what}: {_where(ratio_t > 1, locate)}'
    report(ratio, what)
    return ratio


def check_swiglu_fp64_bound(out, x, Wg, Wu, what='', depth=None, locate=None) -> float:
    """out = fp16(silu(x.Wg) * (x.Wu)) against fp64: the accumulation bounds Ea, Eb of both products (check_fp64_bound) carried
    through silu(a) * b (|silu'| <= 1.1), plus 8 fp32 roundings of the epilogue and the fp16 store."""
    x64 = x.to('cuda', torch.float64)
    Wg64, Wu64 = Wg.to('cuda', torch.float64), Wu.to('cuda', torch.float64)
    a, b = x64 @ Wg64, x64 @ Wu64
    d = default_depth(Wg.shape[0]) if depth is None else depth
    Ea, Eb = fp32_sum_bound(x64.abs() @ Wg64.abs(), d), fp32_sum_bound(x64.abs() @ Wu64.abs(), d)
    sa = a * torch.sigmoid(a)
    ref = sa * b
    bound = ulp16(ref) + 1.1 * Ea * (b.abs() + Eb) + sa.abs() * Eb + 8 * 2.0**-24 * ref.abs()
    out64 = out.to(torch.float64)
    assert torch.isfinite(out64).all(), f'{what}: non-finite output'
    ratio_t = (out64 - ref).abs() / bound
    ratio = ratio_t.max().item()
    if ratio > 1:
        what = f'{what}: {_where(ratio_t > 1, locate)}'
    report(ratio, what)
    return ratio


# ----------------------------------------------------------------------------- bit-level comparisons
def fp16_ulp_distance(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """Number of fp16 values between a and b (both fp16; +0 and -0 are the same point)."""
    def ordered(t):
        u = t.contiguous().view(torch.int16).to(torch.int32) & 0xFFFF
        return torch.where(u >= 0x8000, 0x8000 - u, u)
    return (ordered(a) - ordered(b)).abs()


def fp16_from_fp64(v: torch.Tensor) -> torch.Tensor:
    """float64 -> fp16 rounded once (numpy converts directly; a float64 -> float32 -> fp16 cast can round twice)."""
    return torch.from_numpy(v.detach().cpu().numpy().astype(np.float16))
