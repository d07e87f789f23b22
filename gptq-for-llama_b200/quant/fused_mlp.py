"""Fused SwiGLU MLP over two packed weights: ``down( silu(x.Wgate) * (x.Wup) )``.

Mirrors quant/fused_mlp.py of the reference (QuantLlamaMLP :177-238, make_fused_mlp :241-253,
autotune_warmup_fused :256-288); the gate/up contraction + SwiGLU epilogue is one CUDA kernel
(gptq_fused_mlp_fwd) instead of ``fusedmatmul_248_kernel`` (:84-168).
"""
import torch.nn as nn

from gptq_b200 import ops
from .quant_linear import QuantLinear, _PackedView

try:  # only needed by make_fused_mlp's isinstance test
    from transformers.models.llama.modeling_llama import LlamaMLP
except Exception:  # pragma: no cover - transformers is optional for the kernels themselves
    LlamaMLP = ()

_PARTS = ('qweight', 'scales', 'qzeros', 'g_idx')


class QuantLlamaMLP(_PackedView, nn.Module):

    def __init__(self, gate_proj, down_proj, up_proj):
        super().__init__()
        for part in _PARTS:  # same buffer names as the reference (:186-193); never stored in checkpoints
            self.register_buffer(f'gate_proj_{part}', getattr(gate_proj, part))
            self.register_buffer(f'up_proj_{part}', getattr(up_proj, part))
        if (gate_proj.infeatures, gate_proj.outfeatures, gate_proj.bits, gate_proj.groupsize) != (up_proj.infeatures, up_proj.outfeatures, up_proj.bits,
                                                                                                  up_proj.groupsize):
            raise ValueError('gate_proj and up_proj must have the same shape, bits and groupsize')
        self.infeatures = gate_proj.infeatures
        self.intermediate_size = gate_proj.outfeatures
        self.outfeatures = down_proj.outfeatures
        self.bits = gate_proj.bits
        self.maxq = gate_proj.maxq
        self.groupsize = gate_proj.groupsize
        self.down_proj = down_proj

    def _packed(self):
        return [getattr(self, f'{proj}_{part}') for proj in ('gate_proj', 'up_proj') for part in _PARTS]

    def weights(self):
        """(gate, up) as gptq_b200.ops.QLayerWeights (cached until a buffer is replaced or modified)."""
        def pair():
            bufs = self._packed()
            return ops.QLayerWeights(*bufs[:4], self.bits, self.groupsize), ops.QLayerWeights(*bufs[4:], self.bits, self.groupsize)
        return self._derived('weights', pair)

    def kernel_plan(self):
        """(gate, up) in the layout of the tuned int4 kernels (ops.mlp_kernel_form: act-order rows regrouped, 2/3-bit fields widened;
        their shared input gather in `perm`) when both need it and share their input gather; None otherwise."""
        def plan():
            gate, up = self.weights()
            plan = ops.mlp_kernel_form(gate, up)
            # the fused kernel takes one bit width: a pair with a layer left as stored runs as stored
            return None if plan is None or plan[0] is gate or plan[1] is up else plan
        return self._derived('plan', plan)

    def forward(self, x):
        return self.down_proj(self.triton_llama_mlp(x))

    def groupsize_hint(self):
        gate, up = self.weights()
        return min(gate.hint, up.hint)  # groupsize when both g_idx are trivial, else 0

    def triton_llama_mlp(self, x):
        """fp16 [..., intermediate] = silu(x.Wgate) * (x.Wup).  The name is the reference's (:206); no Triton is involved."""
        out_shape = x.shape[:-1] + (self.intermediate_size, )
        x2 = x.reshape(-1, x.shape[-1])
        gate, up = self.kernel_plan() or self.weights()
        if gate.perm is not None:  # regrouped rows: x is gathered to match
            x2 = x2.index_select(1, gate.perm)
        c = ops.fused_mlp(x2, gate.parts(), up.parts(), gate.bits, min(gate.hint, up.hint))
        return c.reshape(out_shape)

    fused_llama_mlp = triton_llama_mlp

    def _move(self, device):
        for proj in ('gate_proj', 'up_proj'):
            for part in _PARTS:
                name = f'{proj}_{part}'
                setattr(self, name, getattr(self, name).to(device))

    def fused2cuda(self):
        self._move('cuda')

    def fused2cpu(self):
        self._move('cpu')


def make_fused_mlp(m, parent_name=''):
    """Replace every LlamaMLP whose projections are QuantLinear by a QuantLlamaMLP (:241-253)."""
    if LlamaMLP and isinstance(m, LlamaMLP):
        if not all(isinstance(p, QuantLinear) for p in (m.gate_proj, m.down_proj, m.up_proj)):
            return m
        return QuantLlamaMLP(m.gate_proj, m.down_proj, m.up_proj)
    for name, child in list(m.named_children()):
        new = make_fused_mlp(child, parent_name=f'{parent_name}.{name}')
        if new is not child:
            setattr(m, name, new)
    return m


def autotune_warmup_fused(model):
    """API-compatibility shim (:256-288): nothing to tune; primes the act-order probes of fused MLPs on the GPU."""
    n = 0
    for _, m in model.named_modules():
        if isinstance(m, QuantLlamaMLP) and m.gate_proj_qweight.is_cuda:
            m.groupsize_hint()
            m.kernel_plan()
            n += 1
    return n
