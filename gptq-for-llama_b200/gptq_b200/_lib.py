"""ctypes binding of libgptq_b200.so (the C ABI declared in include/gptq_b200.h).

There is NO fallback: if the shared library is missing or a symbol is absent, importing this
module raises.  The library has no torch dependency; torch only supplies device pointers and
the current stream.
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get('GPTQ_B200_LIB') or os.path.join(os.path.dirname(_HERE), 'libgptq_b200.so')  # env override: A/B builds during development

ABI_VERSION = 6

c_void_p, c_int, c_int64, c_size_t, c_float = ctypes.c_void_p, ctypes.c_int, ctypes.c_int64, ctypes.c_size_t, ctypes.c_float


class QWeight(ctypes.Structure):
    """struct gptq_qweight (include/gptq_b200.h)."""
    _fields_ = [
        ('qweight', c_void_p),
        ('scales', c_void_p),
        ('qzeros', c_void_p),
        ('g_idx', c_void_p),
        ('K', c_int),
        ('N', c_int),
        ('G', c_int),
        ('bits', c_int),
        ('groupsize', c_int),
    ]


_QW = ctypes.POINTER(QWeight)


class LlamaLayer(ctypes.Structure):
    """struct gptq_llama_layer."""
    _fields_ = [('qkv', QWeight), ('o', QWeight), ('gate', QWeight), ('up', QWeight), ('down', QWeight), ('input_norm', c_void_p), ('post_norm', c_void_p),
                ('qkv_perm', c_void_p), ('o_perm', c_void_p), ('mlp_perm', c_void_p)]


class LlamaModel(ctypes.Structure):
    """struct gptq_llama_model."""
    _fields_ = [('n_layers', c_int), ('hidden', c_int), ('n_heads', c_int), ('head_dim', c_int), ('intermediate', c_int), ('vocab', c_int), ('rms_eps', c_float),
                ('rope_base', c_float), ('layers', ctypes.POINTER(LlamaLayer)), ('embed', c_void_p), ('final_norm', c_void_p), ('lm_head', c_void_p)]


MAX_TP = 8


class LlamaTP(ctypes.Structure):
    """struct gptq_llama_tp."""
    _fields_ = [('size', c_int), ('rank', c_int), ('vocab_begin', c_int), ('vocab_end', c_int), ('reduce_mode', c_int), ('peer_scratch', c_void_p * MAX_TP),
                ('peer_logits', c_void_p * MAX_TP)]


class LlamaState(ctypes.Structure):
    """struct gptq_llama_state."""
    _fields_ = [('batch', c_int), ('max_seq', c_int), ('k_cache', c_void_p), ('v_cache', c_void_p), ('tokens', c_void_p), ('positions', c_void_p),
                ('logits', c_void_p), ('next_tokens', c_void_p), ('scratch', c_void_p), ('scratch_bytes', c_size_t), ('tp', ctypes.POINTER(LlamaTP))]


class Sampling(ctypes.Structure):
    """struct gptq_sampling (device arrays of `batch` entries)."""
    _fields_ = [('temperature', c_void_p), ('top_k', c_void_p), ('top_p', c_void_p), ('seed', c_void_p), ('eos_token', c_void_p), ('min_length', c_void_p)]


# name -> (restype, argtypes); must list every symbol include/gptq_b200.h declares
SIGNATURES = {
    'gptq_abi_version': (c_int, []),
    'gptq_strerror': (ctypes.c_char_p, [c_int]),
    'gptq_qlinear_workspace_bytes': (c_size_t, [c_int, c_int, c_int, c_int]),
    'gptq_fused_mlp_workspace_bytes': (c_size_t, [c_int, c_int, c_int, c_int]),
    'gptq_qlinear_fwd': (c_int, [c_void_p, c_int64, _QW, c_void_p, c_void_p, c_int64, c_int, c_void_p, c_size_t, c_void_p]),
    'gptq_fused_mlp_fwd': (c_int, [c_void_p, c_int64, _QW, _QW, c_void_p, c_int64, c_int, c_void_p, c_size_t, c_void_p]),
    'gptq_qlinear_transpose_fwd': (c_int, [c_void_p, c_int64, _QW, c_void_p, c_int64, c_int, c_void_p]),
    'gptq_rope_inplace': (c_int, [c_void_p, c_int64, c_void_p, c_int64, c_int, c_int, c_int, c_int, c_float, c_void_p]),
    'gptq_rmsnorm_fwd': (c_int, [c_void_p, c_int64, c_void_p, c_void_p, c_int64, c_int, c_int, c_float, c_void_p]),
    'gptq_pack_qweight': (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p]),
    'gptq_pack_qzeros': (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p]),
    'gptq_unpack_qweight': (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p]),
    'gptq_unpack_qzeros': (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p]),
    'gptq_dequant': (c_int, [_QW, c_void_p, c_int64, c_void_p]),
    'gptq_llama_scratch_bytes': (c_size_t, [ctypes.POINTER(LlamaModel), c_int, c_int]),
    'gptq_llama_decode_step': (c_int, [ctypes.POINTER(LlamaModel), ctypes.POINTER(LlamaState), c_void_p]),
    'gptq_llama_decode_launches': (c_int, [ctypes.POINTER(LlamaModel), ctypes.POINTER(LlamaState)]),
    'gptq_llama_persistent_scratch_offset': (c_size_t, [ctypes.POINTER(LlamaModel), c_int, c_int]),
    'gptq_lm_head_logprob_workspace_bytes': (c_size_t, [c_int, c_int]),
    'gptq_lm_head_logprob': (c_int, [c_void_p, c_int64, c_void_p, c_int64, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    'gptq_cached_attention': (c_int, [c_void_p, c_int64, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_int64,
                                      c_void_p]),
    'gptq_cached_attention_gqa': (c_int, [c_void_p, c_int64, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p,
                                          c_int64, c_void_p]),
    'gptq_sample_tokens': (c_int, [c_void_p, c_int64, c_int, c_int, c_void_p, ctypes.POINTER(Sampling), c_void_p, c_void_p]),
    'gptq_ipc_alloc':(c_int, [c_size_t, ctypes.POINTER(c_void_p), ctypes.c_char_p]),
    'gptq_ipc_open': (c_int, [ctypes.c_char_p, ctypes.POINTER(c_void_p)]),
    'gptq_ipc_close': (c_int, [c_void_p]),
    'gptq_ipc_free': (c_int, [c_void_p]),
}

# gptq_status (include/gptq_b200.h)
OK, ERR_BITS, ERR_SHAPE, ERR_NULL, ERR_ALIGN, ERR_WORKSPACE, ERR_CUDA, ERR_UNSUPPORTED = 0, -1, -2, -3, -4, -5, -6, -7


def _load():
    if not os.path.exists(LIB_PATH):
        raise ImportError(f'{LIB_PATH} not found: build it with `make -C gptq-for-llama_b200/csrc` (or __graft_entry__.build()). '
                          'There is no CPU / PyTorch fallback for the quantized-linear path.')
    lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the symbol is missing -> fail loudly
        fn.restype = res
        fn.argtypes = args
    if lib.gptq_abi_version() != ABI_VERSION:
        raise ImportError(f'libgptq_b200.so ABI {lib.gptq_abi_version()} != binding ABI {ABI_VERSION}: rebuild')
    return lib


lib = _load()


def check(status: int) -> None:
    """Map a gptq_status to the exception the reference raises at the same place."""
    if status == OK:
        return
    msg = lib.gptq_strerror(status).decode()
    if status == ERR_BITS:
        raise NotImplementedError(msg)  # quant/quant_linear.py:308-309
    if status in (ERR_SHAPE, ERR_ALIGN, ERR_NULL):
        raise ValueError(msg)
    raise RuntimeError(msg)  # incl. norm width > 64 KB (quant/triton_norm.py:59-60)
