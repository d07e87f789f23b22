"""QuantLinear: packed-weight linear layer on hand-written sm_90a CUDA.

Mirrors the module surface of the reference's quant/quant_linear.py (QuantLinear :304-377,
matmul248 :263-269, transpose_matmul248 :272-279, QuantLinearFunction :282-301,
make_quant_linear :380-390, autotune_warmup_linear :393-423): same constructor, buffer names,
shapes and dtypes (so existing .pt/.safetensors checkpoints load), same exceptions.
Differences, all additive: 3-bit is accepted (the reference commit raises for it), ``make_quant``
aliases ``make_quant_linear``, bias is fused into the kernel epilogue, and the autotune warm-up
is a cheap load-time preparation pass because dispatch is static (matvec vs wgmma GEMM by M).
"""
import math

import torch
import torch.nn as nn

from gptq_b200 import ops

_SUPPORTED_BITS = (2, 3, 4, 8)


def matmul248(input, qweight, scales, qzeros, g_idx, bits, maxq):
    """output[M, N] fp16 = input[M, K] . deq(qweight); reference signature (quant_linear.py:263)."""
    return ops.matmul248(input, qweight, scales, qzeros, g_idx, bits, maxq)


def transpose_matmul248(input, qweight, scales, qzeros, g_idx, bits, maxq):
    """output[M, K] fp16 = input[M, N] . deq(qweight)^T; reference signature (quant_linear.py:272)."""
    return ops.transpose_matmul248(input, qweight, scales, qzeros, g_idx, bits, maxq)


class QuantLinearFunction(torch.autograd.Function):
    """Frozen-weight autograd wrapper (quant_linear.py:282-301): grad flows to the input only."""

    @staticmethod
    def forward(ctx, input, qweight, scales, qzeros, g_idx, bits, maxq, bias=None, groupsize=0):
        if torch.is_autocast_enabled():  # custom_fwd(cast_inputs=torch.float16)
            input = input.half()
        output = ops.matmul248(input, qweight, scales, qzeros, g_idx, bits, maxq, bias=bias, groupsize=groupsize)
        ctx.save_for_backward(qweight, scales, qzeros, g_idx)
        ctx.bits, ctx.maxq, ctx.groupsize = bits, maxq, groupsize
        return output

    @staticmethod
    def backward(ctx, grad_output):
        qweight, scales, qzeros, g_idx = ctx.saved_tensors
        grad_input = None
        if ctx.needs_input_grad[0]:
            grad_input = ops.transpose_matmul248(grad_output, qweight, scales, qzeros, g_idx, ctx.bits, ctx.maxq, groupsize=ctx.groupsize)
        return grad_input, None, None, None, None, None, None, None, None


class _PackedView:
    """What a module over packed buffers (the tensors _packed() returns) derives from them -- weights() and kernel_plan() -- each computed
    once and kept until a buffer is replaced or modified: pack(), load_state_dict, .cuda() and fused2cuda / fused2cpu do."""
    _view = None  # {'key': the buffers' identity and versions, name: what _derived(name, ...) computed for them}

    def _derived(self, name, derive):
        key = [(t.device, t.data_ptr(), t._version) for t in self._packed()]
        if self._view is None or self._view['key'] != key:
            self._view = dict(key=key)
        if name not in self._view:
            self._view[name] = derive()
        return self._view[name]


class QuantLinear(_PackedView, nn.Module):

    def __init__(self, bits, groupsize, infeatures, outfeatures, bias):
        super().__init__()
        if bits not in _SUPPORTED_BITS:
            raise NotImplementedError("Only 2,3,4,8 bits are supported.")
        self.infeatures = infeatures
        self.outfeatures = outfeatures
        self.bits = bits
        self.maxq = 2**self.bits - 1
        self.groupsize = groupsize if groupsize != -1 else infeatures

        groups = math.ceil(infeatures / self.groupsize)
        self.register_buffer('qweight', torch.zeros((infeatures // 32 * self.bits, outfeatures), dtype=torch.int32))
        self.register_buffer('qzeros', torch.zeros((groups, outfeatures // 32 * self.bits), dtype=torch.int32))
        self.register_buffer('scales', torch.zeros((groups, outfeatures), dtype=torch.float16))
        self.register_buffer('g_idx', (torch.arange(infeatures, dtype=torch.int64) // self.groupsize).to(torch.int32))
        if bias:
            self.register_buffer('bias', torch.zeros((outfeatures), dtype=torch.float16))
        else:
            self.bias = None

    # ------------------------------------------------------------------ packing (offline)
    def pack(self, linear, scales, zeros, g_idx=None):
        """Quantise-and-pack on the GPU (the reference does this on the CPU with a Python loop over K,
        quant_linear.py:325-371, and carries a "TODO: perform packing on GPU", llama.py:264).

        linear.weight [N, K] must already lie on the quantisation grid (gptq.py:108); scales/zeros are
        [N, G].  Integer results are bit-identical to the reference's pack().
        """
        from gptq_b200.ops import pack_qweight, pack_qzeros
        if not torch.cuda.is_available():
            raise RuntimeError('QuantLinear.pack runs on the GPU; no CUDA device is available')
        home = self.qweight.device
        dev = linear.weight.device if linear.weight.is_cuda else torch.device('cuda', torch.cuda.current_device())
        self.g_idx = g_idx.clone().to(torch.int32) if g_idx is not None else self.g_idx
        gi = self.g_idx.to(dev).long()

        scales_t = scales.to(dev).t().contiguous()
        zeros_t = zeros.to(dev).t().contiguous()
        scale_zeros = zeros_t * scales_t
        scales_h = scales_t.clone().half()
        # round((W[:, k] + scale*zero[g]) / scale_fp16[g]) for every k at once; fp32 / fp16 promotes to fp32
        W = linear.weight.data.to(dev)
        intweight = torch.round((W.t() + scale_zeros[gi]) / scales_h[gi]).to(torch.int32)
        self.qweight = pack_qweight(intweight, self.bits).to(home)
        self.qzeros = pack_qzeros((zeros_t - 1).to(torch.int64).to(torch.int32), self.bits).to(home)
        self.scales = scales_h.to(home)
        if linear.bias is not None:
            self.bias = linear.bias.detach().clone().half().to(home)

    # ------------------------------------------------------------------ forward
    def _packed(self):
        return self.qweight, self.scales, self.qzeros, self.g_idx

    def weights(self):
        """The buffers as one gptq_b200.ops.QLayerWeights (cached until a buffer is replaced or modified)."""
        return self._derived('weights', lambda: ops.QLayerWeights(*self._packed(), self.bits, self.groupsize))

    def groupsize_hint(self):
        """groupsize if g_idx is the trivial k // groupsize map (lets the kernels skip the gather), else 0.
        The probe costs one device->host sync and is cached until a buffer is replaced."""
        return self.weights().hint

    def kernel_plan(self):
        """The derived layer (ops.QLayerWeights.kernel_form, with its input gather in `perm`) that routes an act-order and/or 2/3-bit layer to
        the tuned int4 kernels without touching the stored tensors; None when the layer needs none or does not qualify."""
        def plan():
            stored = self.weights()
            form = stored.kernel_form()
            return None if form is stored else form
        return self._derived('plan', plan)

    def forward(self, x):
        out_shape = x.shape[:-1] + (self.outfeatures, )
        x2 = x.reshape(-1, x.shape[-1])
        w = self.kernel_plan() or self.weights()
        if w.perm is not None:  # regrouped rows: x is gathered to match
            x2 = x2.index_select(1, w.perm)
        out = QuantLinearFunction.apply(x2, *w.parts(), w.bits, 2**w.bits - 1, self.bias, w.hint)
        return out.reshape(out_shape)


def make_quant_linear(module, names, bits, groupsize, name=''):
    """Swap every nn.Linear whose dotted name is in `names` for a QuantLinear (quant_linear.py:380-390)."""
    if isinstance(module, QuantLinear):
        return
    for child_name, child in list(module.named_children()):
        full = f'{name}.{child_name}' if name else child_name
        if full in names and not isinstance(child, QuantLinear):
            setattr(module, child_name, QuantLinear(bits, groupsize, child.in_features, child.out_features, child.bias is not None))
        else:
            make_quant_linear(child, names, bits, groupsize, full)


make_quant = make_quant_linear  # older / cuda-branch entry-point name


def autotune_warmup_linear(model, transpose=False):
    """Kept for API compatibility (quant_linear.py:393-423).  There is nothing to autotune: dispatch is
    static.  The pass only primes each layer's act-order probe and kernel form (act-order rows regrouped, 2- and 3-bit
    fields widened) so that the first forward (possibly under CUDA-graph capture) does no device->host sync."""
    n = 0
    for _, m in model.named_modules():
        if isinstance(m, QuantLinear) and m.qweight.is_cuda:
            m.groupsize_hint()
            m.kernel_plan()
            n += 1
    return n
