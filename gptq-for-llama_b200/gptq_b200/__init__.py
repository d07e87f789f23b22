"""Host side of the H100-native GPTQ quantized-linear path: ctypes binding of libgptq_b200.so
(`_lib`), tensor-level ops (`ops`).  The reference-facing module surface lives in the sibling
`quant` package."""
from . import _lib, ops, engine  # noqa: F401  (importing fails loudly if the CUDA library is missing)
