"""Inputs whose quantized-linear outputs are known exactly, whatever the kernel's summation order.

* One-hot rows: x[r] = sign * 2^e * e_k (e in [-2, 2]).  out[r, n] = fp16(sign * 2^e * W[k, n]) (+ fp16 bias) exactly: a single
  exact product plus zeros, so fp32 accumulation, split-K and the tensor-core k order cannot change it.  A last-bit error in
  one dequantised weight, or a k / column mix-up in the staging, shows up as a mismatch at that (k, n).
* Integer-exact sums: x integer in [-2, 2], scales powers of two in [2^-10, 2^-6], random nibbles and zeros.  Every weight is
  a multiple of 2^-10 of magnitude <= 16 * 2^-6, every product a multiple of 2^-10 of magnitude <= 0.5, so at K <= 16384
  every partial sum is a multiple of 2^-10 below 2^13: under 2^23 units, exact in fp32 in any order.  out = fp16(exact sum).

Also the stream-K plan of the split-K matvec (qmatvec.cu: plan_skinny and the CTA unit ranges), restated for error reports, and
which products the matvec takes at all (skinny_supported), restated for the tests' expected routes.
"""
import math

import numpy as np
import torch

from oracle import gptq_oracle as O


# ----------------------------------------------------------------------------- one-hot rows
def onehot_rows(ks, K: int, salt: int = 0):
    """Row r = sign_r * 2^e_r * e_{ks[r]}.  Returns (x fp16 [R, K], mult float64 [R])."""
    ks = torch.as_tensor(ks, dtype=torch.int64)
    r = torch.arange(ks.numel())
    e = (ks * 3 + r + salt) % 5 - 2
    sign = 1 - 2 * ((ks + r + salt) % 2)
    mult = sign.double() * torch.pow(2.0, e.double())
    x = torch.zeros(ks.numel(), K, dtype=torch.float16)
    x[r, ks] = mult.half()
    return x, mult


def onehot_expect(W: torch.Tensor, ks, mult: torch.Tensor, bias=None) -> torch.Tensor:
    """fp16 [R, N]: mult[r] * W[ks[r]] (exact: a power of two times an fp16 normal number), then + bias in fp16."""
    ks = torch.as_tensor(ks, dtype=torch.int64, device=W.device)
    out = (W.index_select(0, ks).double() * mult.to(W.device)[:, None]).half()
    assert torch.equal(out.double(), W.index_select(0, ks).double() * mult.to(W.device)[:, None]), 'one-hot product not exact in fp16'
    if bias is not None:
        out = out + bias.to(W.device)
    return out


def sampled_ks(K: int, gs: int, cta_ks=(), extra: int = 64, seed: int = 0):
    """k values that matter to a k-loop: the first and last 64 (every k % 8, the first and last k-steps), both sides of every
    group boundary, the given CTA-range boundaries, and `extra` random ones."""
    ks = set(range(min(64, K))) | set(range(max(0, K - 64), K))
    for b in range(gs, K, gs):
        ks |= {b - 1, b}
    ks |= {k for k in cta_ks if 0 <= k < K}
    ks |= set(torch.randint(0, K, (extra, ), generator=torch.Generator().manual_seed(seed)).tolist())
    return sorted(ks)


# ----------------------------------------------------------------------------- integer-exact fixtures
def pow2_packed(K: int, N: int, gs: int, jmin: int = 6, jmax: int = 10, seed: int = 0):
    """int4 layer with trivial g_idx: random nibbles and zeros, scales 2^-j with j drawn per (group, column) from [jmin, jmax].
    Returns (qweight, scales, qzeros, g_idx) like O.random_packed."""
    gen = torch.Generator().manual_seed(seed)
    G = math.ceil(K / gs)
    q = torch.randint(0, 16, (K, N), generator=gen).numpy()
    z = torch.randint(0, 16, (G, N), generator=gen).numpy()
    j = torch.randint(jmin, jmax + 1, (G, N), generator=gen)
    scales = torch.pow(2.0, -j.double()).half()
    return torch.from_numpy(O.pack_rows(q, 4)), scales, torch.from_numpy(O.pack_cols(z, 4)), O.make_g_idx(K, gs, False, gen)


def int_x(M: int, K: int, lo: int, hi: int, seed: int = 0) -> torch.Tensor:
    """fp16 [M, K] of integers drawn uniformly from [lo, hi]."""
    return torch.randint(lo, hi + 1, (M, K), generator=torch.Generator().manual_seed(seed)).half()


def exact_product(x: torch.Tensor, W: torch.Tensor) -> torch.Tensor:
    """x . W in float64 (exact for the integer-exact fixtures: every partial sum is an integer multiple of 2^-10 below 2^13)."""
    return x.double() @ W.double()


# ----------------------------------------------------------------------------- the split-K matvec's plan (qmatvec.cu)
SLAB = 256  # output columns per slab
STEP = 32   # k per unit
NUM_SMS = 132


def matvec_plan(K: int, N: int):
    """(nslabs, nk, total units U, grid): units are (slab, k-step) pairs numbered slab-major, split over min(2 x SMs, U) CTAs."""
    nslabs, nk = -(-N // SLAB), K // STEP
    U = nslabs * nk
    return nslabs, nk, U, min(U, 2 * NUM_SMS)


MATVEC_RING_BYTES = 8 * 8192  # 8 warps x an 8 KB weight ring each
MATVEC_SMEM_LIMIT = 110 * 1024  # two CTAs per SM


def matvec_smem_bytes(M: int, K: int, N: int) -> int:
    """The shared memory skinny_supported budgets: the weight rings plus M rows of the CTA's x segment, seg_steps = ceil(U / grid)
    k-steps of 32 (at most nk) and one step more for the bank-spreading pitch."""
    _, nk, U, nb = matvec_plan(K, N)
    seg_steps = min(nk, -(-U // nb))
    return MATVEC_RING_BYTES + M * (seg_steps * 32 + 32) * 2


def matvec_takes(M: int, K: int, N: int) -> bool:
    """Whether the split-K matvec serves an int4 product of M rows at (K, N), groupsize a multiple of 32 and aligned operands
    (qmatvec.cu skinny_supported); otherwise the generic kernel does, and the kernel chain runs the RMSNorm and the residual add as
    kernels of their own around it."""
    _, _, U, _ = matvec_plan(K, N)
    return 1 <= M <= 8 and K % 32 == 0 and U * (2 * NUM_SMS + 1) < 2**31 and matvec_smem_bytes(M, K, N) <= MATVEC_SMEM_LIMIT


def matvec_cta(K: int, N: int, k: int, n: int):
    """The CTA that owns weight (k, n) and its unit range [u_begin, u_end)."""
    _, nk, U, nb = matvec_plan(K, N)
    u = (n // SLAB) * nk + k // STEP
    b = -(-((u + 1) * nb) // U) - 1
    return b, b * U // nb, (b + 1) * U // nb


def matvec_cta_ks(K: int, N: int):
    """The first k of every CTA range and the last k before it (inside one slab), over all slabs."""
    _, nk, U, nb = matvec_plan(K, N)
    ks = set()
    for b in range(nb):
        k0 = (b * U // nb % nk) * STEP
        ks |= {k0, k0 - 1}
    return ks


def matvec_where(K: int, N: int, gs: int, m: int, n: int, k=None) -> str:
    """Error-report location of out[m, n] (and the contributing k, for one-hot inputs) in the matvec's decomposition."""
    slab = n // SLAB
    _, nk, U, nb = matvec_plan(K, N)
    first, last = matvec_cta(K, N, 0, n)[0], matvec_cta(K, N, K - 1, n)[0]
    s = f'm={m} n={n} slab={slab} CTAs {first}..{last} share the slab'
    if k is not None:
        b, ub, ue = matvec_cta(K, N, k, n)
        s = f'm={m} k={k} (k%8={k % 8}, k//gs={k // gs}) n={n} slab={slab} CTA {b} units [{ub}, {ue}) of {U}'
    return s


def gemm_where(M: int, K: int, gs: int, m: int, n: int, k=None, dual: bool = False) -> str:
    """Error-report location of out[m, n] in the wgmma GEMM's tiling (128 columns x 128 * WT rows, K step 64; WT = 2 for a
    single weight above 128 rows)."""
    wt = 2 if M > 128 and not dual else 1
    s = f'm={m} n={n} tile (row {m // (128 * wt)}, col {n // 128}) WT={wt} warpgroup {(m % (128 * wt)) // (64 * wt)}'
    if k is not None:
        s += f' k={k} (k%8={k % 8}, k//gs={k // gs}, K step {k // 64})'
    return s
