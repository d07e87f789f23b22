"""CPU oracle for the GPTQ-for-LLaMa quantized-linear hot path.

THIS IS TEST INFRASTRUCTURE, NOT PRODUCT CODE.  Only ``tests/``,
``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline`` / ``--impl reference``
legs may import it.  The product path (``gptq-for-llama_b200/``) never does and has
no CPU fallback.

It is a plain numpy / torch-CPU restatement of the arithmetic of the reference's
Triton kernels (which cannot run without a GPU) and of its CPU ``pack()``.
Every function cites the reference lines (relative to the reference checkout) it follows.

Pinning status
--------------
* bits 2/4/8 pack layout: PINNED bit-exactly against the reference's own
  ``QuantLinear.pack`` (quant/quant_linear.py:325-371) through the committed
  fixtures ``tests/golden/pack_*.npz`` (generator: ``tests/golden/make_golden.py``,
  which imports the reference in the build container).
* dequant / matmul: pinned through the identity deq(pack(Q)) == Q on the same
  fixtures (the reference has no CPU forward and no tests; SURVEY.md section 4).
* bits 3: PARITY UNPINNED.  The reference at this commit raises
  NotImplementedError for 3 bits (quant/quant_linear.py:308-309).  The layout
  here is the 96-bit little-endian bit-stream of the upstream cuda branch
  (32 values in 3 consecutive int32 words); it is pinned only by its own
  pack<->unpack round trip.
* RoPE / RMSNorm / fused MLP: restated from the kernel source only; the
  reference holds no golden vectors for them ("parity unpinned" beyond the code).
"""
import math

import numpy as np
import torch

SUPPORTED_BITS = (2, 3, 4, 8)


# --------------------------------------------------------------------------
# integer layout
# --------------------------------------------------------------------------
def pack_rows(vals: np.ndarray, bits: int) -> np.ndarray:
    """Pack ``vals[R, C]`` (0 <= v < 2**bits) along axis 0 into ``[R//32*bits, C]`` int32.

    quant/quant_linear.py:341-352: value j of each run of ``32//bits`` rows is OR-ed
    in at bit ``bits*j`` (LSB first).  For 3 bits the 32 values of a run form one
    96-bit little-endian bit-stream over three words (upstream cuda-branch layout;
    unpinned, see module docstring).  Like the reference there is NO clamp: the
    caller must pass on-grid values; we assert instead of silently corrupting.
    """
    assert bits in SUPPORTED_BITS
    vals = np.asarray(vals)
    R, C = vals.shape
    assert R % 32 == 0, "rows must be a multiple of 32"
    assert vals.min() >= 0 and vals.max() < (1 << bits), "off-grid value"
    v = vals.astype(np.uint64)
    out = np.zeros((R // 32 * bits, C), dtype=np.uint32)
    if bits in (2, 4, 8):
        ipb = 32 // bits
        v = v.reshape(R // ipb, ipb, C)
        for j in range(ipb):
            out |= (v[:, j, :] << np.uint64(bits * j)).astype(np.uint32)
    else:
        v = v.reshape(R // 32, 32, C)
        o = out.reshape(R // 32, 3, C)
        for j in range(32):
            bit = 3 * j
            w, sh = bit // 32, bit % 32
            o[:, w, :] |= ((v[:, j, :] << np.uint64(sh)) & np.uint64(0xFFFFFFFF)).astype(np.uint32)
            if sh + 3 > 32:  # value straddles two words
                o[:, w + 1, :] |= (v[:, j, :] >> np.uint64(32 - sh)).astype(np.uint32)
        out = o.reshape(R // 32 * 3, C)
    return out.view(np.int32)


def unpack_rows(packed: np.ndarray, bits: int) -> np.ndarray:
    """Inverse of :func:`pack_rows`: ``[R//32*bits, C]`` int32 -> ``[R, C]`` int32 in [0, 2**bits).

    quant/quant_linear.py:103,124-127: ``(b >> ((k % ipb) * bits)) & maxq``.
    """
    assert bits in SUPPORTED_BITS
    p = np.ascontiguousarray(packed).view(np.uint32)
    PR, C = p.shape
    maxq = (1 << bits) - 1
    if bits in (2, 4, 8):
        ipb = 32 // bits
        shifts = (np.arange(ipb, dtype=np.uint32) * bits)[None, :, None]
        return ((p[:, None, :] >> shifts) & maxq).reshape(PR * ipb, C).astype(np.int32)
    assert PR % 3 == 0
    w = p.reshape(PR // 3, 3, C).astype(np.uint64)
    out = np.empty((PR // 3, 32, C), dtype=np.int32)
    for j in range(32):
        bit = 3 * j
        wi, sh = bit // 32, bit % 32
        val = w[:, wi, :] >> np.uint64(sh)
        if sh + 3 > 32:
            val = val | (w[:, wi + 1, :] << np.uint64(32 - sh))
        out[:, j, :] = (val & np.uint64(7)).astype(np.int32)
    return out.reshape(PR // 3 * 32, C)


def pack_cols(vals: np.ndarray, bits: int) -> np.ndarray:
    """Pack ``vals[R, C]`` along axis 1 (qzeros layout, quant/quant_linear.py:358-369)."""
    return np.ascontiguousarray(pack_rows(np.ascontiguousarray(np.asarray(vals).T), bits).T)


def unpack_cols(packed: np.ndarray, bits: int) -> np.ndarray:
    return np.ascontiguousarray(unpack_rows(np.ascontiguousarray(np.asarray(packed).T), bits).T)


def pack(weight: torch.Tensor, scales: torch.Tensor, zeros: torch.Tensor, g_idx: torch.Tensor, bits: int):
    """Restatement of ``QuantLinear.pack`` (quant/quant_linear.py:325-371).

    weight: fp ``[N, K]`` (already on the quantisation grid, gptq.py:108)
    scales, zeros: ``[N, G]`` (as produced by gptq.py:210-228); g_idx: int ``[K]``.
    Returns (qweight int32 [K//32*bits, N], qzeros int32 [G, N//32*bits], scales fp16 [G, N]).
    """
    scales_t = scales.t().contiguous()  # :328
    zeros_t = zeros.t().contiguous()  # :329
    scale_zeros = zeros_t * scales_t  # :330
    scales_h = scales_t.clone().half()  # :331
    g = g_idx.long()
    # :336-337 -- per column: round((W[:, k] + scale*zero[g]) / scale_fp16[g]); the division is
    # fp32 / fp16 -> fp32 (type promotion), rounding is round-half-even, cast to int32.
    intweight = torch.round((weight.t() + scale_zeros[g]) / scales_h[g]).to(torch.int)  # [K, N]
    qweight = pack_rows(intweight.numpy(), bits)
    zeros_m1 = (zeros_t - 1).numpy().astype(np.uint32)  # :356-357
    qzeros = pack_cols(zeros_m1.astype(np.int64), bits)
    return torch.from_numpy(qweight), torch.from_numpy(qzeros), scales_h


# --------------------------------------------------------------------------
# forward arithmetic
# --------------------------------------------------------------------------
def dequant(qweight, scales, qzeros, g_idx, bits: int) -> torch.Tensor:
    """fp16 ``[K, N]`` weight exactly as ``matmul_248_kernel`` materialises it.

    quant/quant_linear.py:114-128: gather scales/zeros by g_idx; zeros are
    ``((qz >> shift) & maxq) + 1`` with the +1 UNMASKED; ``(b - zeros) * scales`` is an
    int32 * fp16 product, i.e. (b - zeros) converted to fp16 (exact, |.| <= 256) and
    multiplied in fp16 with one rounding.
    """
    w = torch.from_numpy(unpack_rows(qweight.numpy(), bits))  # [K, N] int32
    z = torch.from_numpy(unpack_cols(qzeros.numpy(), bits)) + 1  # [G, N]
    g = g_idx.long()
    return (w - z[g]).to(torch.float16) * scales[g]


def qlinear_fwd(x, qweight, scales, qzeros, g_idx, bits: int, bias=None) -> torch.Tensor:
    """``QuantLinear.forward`` (quant/quant_linear.py:373-377) over ``matmul248`` (:263-269).

    fp16 x fp16 products accumulated in fp32 (:111,:130), stored as fp16 (:137, :265);
    bias added afterwards in fp16 (:376).
    """
    W = dequant(qweight, scales, qzeros, g_idx, bits)
    x2 = x.reshape(-1, x.shape[-1])
    out = (x2.float() @ W.float()).half()
    if bias is not None:
        out = out + bias
    return out.reshape(x.shape[:-1] + (W.shape[1], ))


def qlinear_transpose_fwd(g, qweight, scales, qzeros, g_idx, bits: int) -> torch.Tensor:
    """``transpose_matmul248`` (quant/quant_linear.py:272-279, kernel :191-258): g[M,N] . deq(W)^T -> [M,K]."""
    W = dequant(qweight, scales, qzeros, g_idx, bits)
    g2 = g.reshape(-1, g.shape[-1])
    return (g2.float() @ W.float().t()).half().reshape(g.shape[:-1] + (W.shape[0], ))


def fused_mlp_fwd(x, gate, up, bits: int) -> torch.Tensor:
    """``fusedmatmul_248_kernel`` (quant/fused_mlp.py:128-168).

    gate / up are ``(qweight, scales, qzeros, g_idx)``.  Two fp32 accumulators (:126-127);
    ``silu(acc1) * acc2`` in fp32 (:163-164, silu = x*sigmoid(x) :170-172), one cast to fp16 (:165).
    """
    x2 = x.reshape(-1, x.shape[-1]).float()
    a1 = x2 @ dequant(*gate, bits).float()
    a2 = x2 @ dequant(*up, bits).float()
    c = (a1 * torch.sigmoid(a1) * a2).half()
    return c.reshape(x.shape[:-1] + (c.shape[-1], ))


def rope_inplace(qk: torch.Tensor, position_ids: torch.Tensor, base: float = 10000.0) -> None:
    """``rotate_half_kernel`` / ``triton_rotate_half_`` (quant/fused_attn.py:8-93), in place.

    qk: fp16 ``[bsz, seq, 2, heads, head_dim]`` (a view is fine).  :43 ``freq_i =
    exp(i * INV_BASE) * pos`` with INV_BASE = -2 ln(base)/head_dim (:91), fp32 cos/sin (:44-45);
    x' = x cos - y sin, y' = x sin + y cos with y at +head_dim/2 (:52-57), fp16 store.
    """
    bsz, seq, two, heads, hd = qk.shape
    half = hd // 2
    inv_base = np.float32(-2.0 * math.log(base) / hd)
    freq = torch.exp(torch.arange(half, dtype=torch.float32) * inv_base)[None, None, :] * position_ids[:, :, None].float()
    cos = torch.cos(freq)[:, :, None, None, :]
    sin = torch.sin(freq)[:, :, None, None, :]
    x = qk[..., :half].float()
    y = qk[..., half:].float()
    qk[..., :half] = (x * cos - y * sin).half()
    qk[..., half:] = (x * sin + y * cos).half()


def rmsnorm_fwd(x: torch.Tensor, weight: torch.Tensor, eps: float) -> torch.Tensor:
    """``rms_norm_fwd_fused`` (quant/triton_norm.py:21-39): fp32 variance, ``x*rstd*w`` in fp32, fp16 store."""
    xf = x.float()
    var = (xf * xf).sum(-1, keepdim=True) / x.shape[-1]
    rstd = 1.0 / torch.sqrt(var + eps)
    return (xf * rstd * weight.float()).to(x.dtype)


# --------------------------------------------------------------------------
# synthetic fixtures (SURVEY.md section 8(d))
# --------------------------------------------------------------------------
def make_g_idx(K: int, groupsize: int, act_order: bool, gen: torch.Generator) -> torch.Tensor:
    """Trivial ``k // groupsize`` (quant/quant_linear.py:319) or an act-order map built like gptq.py:210-216."""
    g = torch.arange(K) // groupsize
    if act_order:
        perm = torch.randperm(K, generator=gen)
        invperm = torch.argsort(perm)
        g = g[invperm]
    return g.to(torch.int32)


def random_packed(K: int, N: int, bits: int, groupsize: int, act_order: bool = False, seed: int = 0, bias: bool = False):
    """Perf-style fixture: uniform random fields, scales ~ U(1e-3, 1.1e-2) fp16 (SURVEY.md 8(d))."""
    gen = torch.Generator().manual_seed(seed)
    gs = K if groupsize == -1 else groupsize
    G = math.ceil(K / gs)
    if bits == 3:
        w = torch.randint(0, 8, (K, N), generator=gen).numpy()
        z = torch.randint(0, 8, (G, N), generator=gen).numpy()
        qweight = torch.from_numpy(pack_rows(w, 3))
        qzeros = torch.from_numpy(pack_cols(z, 3))
    else:
        qweight = torch.randint(-2**31, 2**31, (K // 32 * bits, N), generator=gen, dtype=torch.int64).to(torch.int32)
        qzeros = torch.randint(-2**31, 2**31, (G, N // 32 * bits), generator=gen, dtype=torch.int64).to(torch.int32)
    scales = (torch.rand(G, N, generator=gen) * 1e-2 + 1e-3).half()
    g_idx = make_g_idx(K, gs, act_order, gen)
    b = (torch.randn(N, generator=gen) * 0.1).half() if bias else None
    return qweight, scales, qzeros, g_idx, b
