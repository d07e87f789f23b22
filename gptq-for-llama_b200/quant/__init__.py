"""Drop-in replacement for the reference's ``quant`` package (quant/__init__.py:1-5 of
qwopqwop200/GPTQ-for-LLaMa, triton branch), backed by hand-written sm_90a CUDA in
libgptq_b200.so instead of Triton.  Same public names; ``make_quant`` is the older alias of
``make_quant_linear``.
"""
import os as _os
import sys as _sys

_root = _os.path.dirname(_os.path.dirname(_os.path.abspath(__file__)))
if _root not in _sys.path:  # make the sibling host package `gptq_b200` importable
    _sys.path.insert(0, _root)

from .quantizer import Quantizer  # noqa: E402
from .fused_attn import QuantLlamaAttention, make_quant_attn  # noqa: E402
from .fused_mlp import QuantLlamaMLP, make_fused_mlp, autotune_warmup_fused  # noqa: E402
from .quant_linear import QuantLinear, make_quant_linear, make_quant, autotune_warmup_linear  # noqa: E402
from .triton_norm import TritonLlamaRMSNorm, make_quant_norm  # noqa: E402
