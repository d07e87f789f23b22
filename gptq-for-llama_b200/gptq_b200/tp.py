"""Tensor-parallel sharding of packed GPTQ layers (BASELINE.json config 5: LLaMA-65B over 8 GPUs).

The reference has no tensor parallelism (its "multi-GPU" is layer placement, llama.py:328-382); this is new
design on top of the packed layout, checked against the single-GPU result:

* column parallel (gate, up; q, k, v SEPARATELY): slice N.  qweight[:, n0:n1], scales[:, n0:n1], qzeros[:, n0*bits/32 : n1*bits/32];
  g_idx is replicated.  Shard boundaries are multiples of 32 columns.  No communication (attention is head-local).
  A FUSED qkv layer is [q | k | v] along N: a contiguous slice of it is not a set of heads; shard it per head with
  ``engine.shard_for_rank`` (what the tensor-parallel decode engine does), or shard q, k, v before fusing them.
* row parallel (o_proj, down_proj): slice K at GROUP boundaries so that every shard keeps the trivial
  ``k // groupsize`` map (and therefore the tuned kernels): 65B down_proj has K = 22016 = 172 groups, i.e. 21.5
  per rank, so shards are uneven by one group.  Each rank multiplies its slice of x; one all-reduce (sum) of the
  [M, N] partial outputs follows -- the only collective on the path.

Pure tensor slicing + ``torch.distributed``; works with the gloo backend on CPU for the host logic (tests) and NCCL
over NVLink on GPUs.
"""
import math

import torch
import torch.distributed as dist
import torch.nn as nn

from .ops import QLayerWeights


def column_partition(N: int, world: int, align: int = 32):
    """Boundaries [n_0 .. n_world] splitting N into `world` contiguous shards of multiples of `align` columns."""
    if N % align:
        raise ValueError(f'N={N} is not a multiple of {align}')
    units = N // align
    return [align * ((units * r) // world) for r in range(world + 1)]


def row_partition(K: int, groupsize: int, world: int):
    """Boundaries splitting K at group boundaries, as evenly as the group count allows."""
    if K % groupsize:
        raise ValueError('row sharding needs K to be a whole number of groups')
    groups = K // groupsize
    if groups < world:
        raise ValueError('fewer groups than ranks')
    return [groupsize * ((groups * r) // world) for r in range(world + 1)]


def shard_columns(qweight, scales, qzeros, g_idx, bits: int, rank: int, world: int, bias=None):
    """This rank's column shard of a packed layer: (qweight, scales, qzeros, g_idx, bias)."""
    b = column_partition(qweight.shape[1], world)
    n0, n1 = b[rank], b[rank + 1]
    # a column slice does not depend on the groupsize (0: no hint is ever asked of this layer)
    w = QLayerWeights(qweight, scales, qzeros, g_idx, bits, 0).column_slice(torch.arange(n0, n1, device=qweight.device))
    return w.qweight, w.scales, w.qzeros, w.g_idx.clone(), bias[n0:n1].contiguous() if bias is not None else None


def shard_rows(qweight, scales, qzeros, g_idx, bits: int, groupsize: int, rank: int, world: int):
    """This rank's row (K) shard: (qweight, scales, qzeros, g_idx_local, (k0, k1)).  Requires the trivial g_idx."""
    w = QLayerWeights(qweight, scales, qzeros, g_idx, bits, groupsize)
    b = row_partition(w.g_idx.numel(), groupsize, world)
    k0, k1 = b[rank], b[rank + 1]
    w = w.row_slice(k0, k1)
    return w.qweight, w.scales, w.qzeros, w.g_idx, (k0, k1)


class TPQuantLinear(nn.Module):
    """A QuantLinear sharded over a process group.

    mode='column': y_local = x . W[:, shard]            (optionally all-gathered along N)
    mode='row'   : y = all_reduce_sum( x[:, shard] . W[shard, :] ) (+ bias on every rank after the reduction)
    """

    def __init__(self, full, mode: str, group=None, gather_output: bool = False):
        super().__init__()
        from quant import QuantLinear
        self.mode, self.group, self.gather_output = mode, group, gather_output
        self.world = dist.get_world_size(group)
        self.rank = dist.get_rank(group)
        bits, gs = full.bits, full.groupsize
        self.outfeatures_full = full.outfeatures
        if mode == 'column':
            qw, sc, qz, gi, bias = shard_columns(full.qweight, full.scales, full.qzeros, full.g_idx, bits, self.rank, self.world, full.bias)
            self.local = QuantLinear(bits, gs, full.infeatures, qw.shape[1], bias is not None)
            self.k_range = (0, full.infeatures)
            self.bias_after = None
        elif mode == 'row':
            qw, sc, qz, gi, self.k_range = shard_rows(full.qweight, full.scales, full.qzeros, full.g_idx, bits, gs, self.rank, self.world)
            self.local = QuantLinear(bits, gs, self.k_range[1] - self.k_range[0], full.outfeatures, False)
            bias = None
            self.bias_after = full.bias.clone() if full.bias is not None else None
        else:
            raise ValueError("mode must be 'column' or 'row'")
        self.local.qweight, self.local.scales, self.local.qzeros, self.local.g_idx = qw, sc, qz, gi
        if bias is not None:
            self.local.bias = bias
        self.column_bounds = column_partition(full.outfeatures, self.world) if mode == 'column' else None

    def forward(self, x):
        if self.mode == 'column':
            y = self.local(x)
            if not self.gather_output:
                return y
            parts = [torch.empty(x.shape[:-1] + (self.column_bounds[r + 1] - self.column_bounds[r], ), dtype=y.dtype, device=y.device) for r in range(self.world)]
            dist.all_gather(parts, y.contiguous(), group=self.group)
            return torch.cat(parts, dim=-1)
        k0, k1 = self.k_range
        y = self.local(x[..., k0:k1].contiguous())
        y32 = y.float()  # reduce in fp32: the only extra rounding w.r.t. the single-GPU result is each rank's fp16 partial
        dist.all_reduce(y32, op=dist.ReduceOp.SUM, group=self.group)
        y = y32.to(torch.float16)
        if self.bias_after is not None:
            y = y + self.bias_after.to(y.device)
        return y


def per_rank_bytes(K: int, N: int, bits: int, groupsize: int, world: int, mode: str):
    """Algorithmic weight bytes each rank streams per forward (for the scaling table in DESIGN.md)."""
    out = []
    for r in range(world):
        if mode == 'column':
            b = column_partition(N, world)
            n = b[r + 1] - b[r]
            k = K
        else:
            b = row_partition(K, groupsize, world)
            k = b[r + 1] - b[r]
            n = N
        G = math.ceil(k / groupsize)
        out.append(k * n * bits // 8 + G * n * 2 + G * n * bits // 8)
    return out
