"""CPU: the numpy restatement of the sampling rule (oracle/sampling.py) -- Philox4x32-10 against Random123's known-answer vectors, the kept set
against transformers' own warpers -- and the argument validation of gptq_sample_tokens, which runs before any CUDA call."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import sampling as S


@pytest.mark.parametrize('counter, key, expected', [
    ([0, 0, 0, 0], [0, 0], [0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8]),
    ([0xffffffff] * 4, [0xffffffff] * 2, [0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd]),
    ([0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344], [0xa4093822, 0x299f31d0], [0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1]),
])
def test_philox_known_answers(counter, key, expected):
    assert S.philox4x32_10(np.array(counter), np.array(key)).tolist() == expected


def test_uniform_uses_53_bits_of_the_first_two_words():
    x = S.philox4x32_10(np.array([7, 0, 0, 0]), np.array([0x89abcdef, 0x01234567]))
    u = ((int(x[0]) >> 5) * 2**26 + (int(x[1]) >> 6)) / 2.0**53
    assert S.uniform(7, 0x0123456789abcdef) == u
    us = S.uniform(np.arange(4096), 12345)
    assert us.min() >= 0 and us.max() < 1 and len(set(us.tolist())) == 4096


def _hf_kept(l16, temperature, top_k, top_p):
    """The tokens transformers' TemperatureLogitsWarper -> TopKLogitsWarper -> TopPLogitsWarper leave finite, on the fp16 logits as fp32."""
    from transformers.generation.logits_process import TemperatureLogitsWarper, TopKLogitsWarper, TopPLogitsWarper
    scores = torch.from_numpy(np.asarray(l16, dtype=np.float16)).float()[None]
    ids = torch.zeros(1, 1, dtype=torch.long)
    scores = TemperatureLogitsWarper(temperature)(ids, scores)
    if top_k:
        scores = TopKLogitsWarper(top_k)(ids, scores)
    if top_p < 1:
        scores = TopPLogitsWarper(top_p)(ids, scores)
    return torch.isfinite(scores[0]).numpy()


def _rows():
    rng = np.random.default_rng(0)
    rows = [('random', (rng.standard_normal(32000) * 3).astype(np.float16)) for _ in range(4)]
    rows.append(('random wide', (rng.standard_normal(4096) * 12).astype(np.float16)))
    tie = (rng.standard_normal(1000) * 2).astype(np.float16)
    tie[np.argsort(-tie.astype(np.float32))[45:60]] = np.sort(tie.astype(np.float32))[::-1][47]  # 15 equal values around the 50th
    rows.append(('ties at the k-th value', tie))
    b = np.full(200, -8, dtype=np.float16)
    b[:10] = [4, 3, 3, 2, 2, 2, 1, 1, 0, 0]  # distinct levels whose mass crosses top_p well away from it
    rows.append(('top-p boundary', b))
    return rows


@pytest.mark.parametrize('temperature', [0.8, 1.0, 2.5])
@pytest.mark.parametrize('top_k, top_p', [(50, 0.95), (0, 0.95), (50, 1.0), (0, 0.5), (5, 0.05), (1000, 0.9)])
def test_kept_set_matches_transformers(temperature, top_k, top_p):
    pytest.importorskip('transformers')
    for name, l16 in _rows():
        hf = _hf_kept(l16, temperature, top_k, top_p)
        z, w, keep = S.kept_weights(l16, temperature, top_k, top_p)
        diff = np.nonzero(hf != keep)[0]
        if diff.size == 0:
            continue
        # allowed: tokens in HF's set's tie groups (the restatement keeps a straddling tie group whole), and tokens whose mass above lies
        # within 1e-5 of top_p (HF sums fp32 probabilities, the restatement fp64 weights)
        kw = S.kept_weights(l16, temperature, top_k, 1.0)[1]
        W = kw.sum()
        for v in diff:
            above = kw[z > z[v]].sum() / W
            tie_superset = keep[v] and not hf[v] and np.any(hf & (z == z[v]))
            assert tie_superset or abs(above - top_p) <= 1e-5, f'{name}: token {v} kept by {"restatement" if keep[v] else "transformers"} only'


def test_tie_straddling_top_p_is_kept_whole():
    l16 = np.array([2, 2, 2, 2, -30, -30], dtype=np.float16)  # four equal tokens, top_p 0.5: transformers keeps two of them
    z, w, keep = S.kept_weights(l16, 1.0, 0, 0.5)
    assert keep.tolist() == [True] * 4 + [False] * 2
    assert _hf_kept(l16, 1.0, 0, 0.5).sum() in (2, 3)


def test_rule_edges():
    row = np.array([1, 5, 5, -2], dtype=np.float16)
    assert S.sample_row(row, 0.0) == 1  # argmax, lowest id on ties
    assert S.sample_row(row, 0.0, eos=1, min_length=10, position=3) == 2  # eos suppressed: p + 1 < min_length
    assert S.sample_row(row, 0.0, eos=1, min_length=4, position=3) == 1  # no longer suppressed
    assert S.sample_row(np.array([np.nan, -np.inf], dtype=np.float16), 1.0) == 0  # nothing above -inf
    inf = np.array([0, np.inf, 3, np.inf], dtype=np.float16)
    assert {S.sample_row(inf, 0.7, seed=s, position=p) for s in range(4) for p in range(16)} == {1, 3}  # +inf entries share the mass
    assert S.sample_row(np.array([np.nan, 1, np.nan], dtype=np.float16), 1.0, top_k=1) == 1  # NaN is -inf
    assert S.sample_row(np.array([-0.0, 0.0], dtype=np.float16), 0.0) == 0  # -0 == +0: lowest id


P = 0x1000  # an aligned fake device pointer: every call below returns during validation


def _params(**null):
    from gptq_b200._lib import Sampling
    s = Sampling()
    for f, _ in Sampling._fields_:
        setattr(s, f, None if f in null else P)
    return s


def _call(logits=P, ld=32000, batch=1, vocab=32000, positions=P, params=None, out=P):
    from gptq_b200._lib import lib
    prm = _params() if params is None else params
    return lib.gptq_sample_tokens(logits, ld, batch, vocab, positions, None if params is False else ctypes.byref(prm), out, None)


def test_validation_null():
    from gptq_b200 import _lib
    assert _call(logits=None) == _lib.ERR_NULL
    assert _call(positions=None) == _lib.ERR_NULL
    assert _call(out=None) == _lib.ERR_NULL
    assert _call(params=False) == _lib.ERR_NULL
    for f in ('temperature', 'top_k', 'top_p', 'seed', 'eos_token', 'min_length'):
        assert _call(params=_params(**{f: True})) == _lib.ERR_NULL, f


@pytest.mark.parametrize('kw', [dict(batch=0), dict(batch=9), dict(batch=-1), dict(vocab=0), dict(vocab=-3), dict(ld=31999)])
def test_validation_shape(kw):
    from gptq_b200 import _lib
    assert _call(**kw) == _lib.ERR_SHAPE


def test_validation_vocab_limit():
    from gptq_b200 import _lib
    assert _call(vocab=131073, ld=131073) == _lib.ERR_UNSUPPORTED
    assert _call(vocab=131072, ld=131072, logits=P + 1) == _lib.ERR_ALIGN  # 131072 itself is accepted


@pytest.mark.parametrize('field', ['logits', 'positions', 'out'])
def test_validation_alignment(field):
    from gptq_b200 import _lib
    assert _call(**{field: P + 1}) == _lib.ERR_ALIGN


@pytest.mark.parametrize('field', ['temperature', 'top_k', 'top_p', 'seed', 'eos_token', 'min_length'])
def test_validation_param_alignment(field):
    from gptq_b200 import _lib
    prm = _params()
    setattr(prm, field, P + (4 if field == 'seed' else 2))
    assert _call(params=prm) == _lib.ERR_ALIGN


def test_engine_rejects_sampling_arguments_before_any_device_work():
    from gptq_b200.engine import sampling_lists
    with pytest.raises(ValueError):
        sampling_lists(2, temperature=[1.0], top_k=50, top_p=1.0)  # one value per sequence or one for all
    with pytest.raises(ValueError):
        sampling_lists(1, temperature=1.0, top_k=50, top_p=1.5)
    with pytest.raises(ValueError):
        sampling_lists(1, temperature=1.0, top_k=50, top_p=0.0)
    with pytest.raises(ValueError):
        sampling_lists(1, temperature=-1.0, top_k=50, top_p=1.0)
    t, k, p = sampling_lists(3, temperature=[0.5, 1.0, 2.0], top_k=7, top_p=0.9)
    assert t == [0.5, 1.0, 2.0] and k == [7] * 3 and p == [0.9] * 3


def test_tensor_parallel_decoder_refuses_sampling_and_eos():
    """The guard runs before any device work, so a decoder shell with a tensor-parallel configuration is enough here."""
    from gptq_b200.engine import LlamaDecoder
    dec = LlamaDecoder.__new__(LlamaDecoder)
    dec.tp, dec.batch, dec.max_seq, dec.vocab = (0, 2, 0, 256), 1, 64, 512
    with pytest.raises(ValueError, match='tensor parallelism'):
        dec.generate([1, 2], 4, do_sample=True)
    with pytest.raises(ValueError, match='tensor parallelism'):
        dec.generate([1, 2], 4, eos_token_id=3)
    with pytest.raises(ValueError, match='tensor parallelism'):
        dec.set_sampling(1.0, 50, 1.0, 0)


TP = (0, 2, 0, 256)  # rank 0 of 2, holding vocabulary rows 0..255
OOV = 512  # the shell's vocabulary is 0..511


def _decoder_shell(tp, batch):
    """A decoder without weights, cache or device buffers: a call that got past its argument checks fails on a missing attribute instead."""
    from gptq_b200.engine import LlamaDecoder
    dec = LlamaDecoder.__new__(LlamaDecoder)
    dec.tp, dec.batch, dec.max_seq, dec.vocab = tp, batch, 64, 512
    dec.lengths, dec.cached_tokens = [0] * batch, [[] for _ in range(batch)]
    return dec


@pytest.mark.parametrize('tp, batch, call', [
    pytest.param(None, 1, lambda d: d.set_input(OOV, 0), id='set_input-oov'),
    pytest.param(None, 2, lambda d: d.set_input(torch.tensor([3, -1]), [0, 1]), id='set_input-negative-tensor'),
    pytest.param(None, 1, lambda d: d.extend([[1, OOV]]), id='extend-oov'),
    pytest.param(None, 2, lambda d: d.extend([[], torch.tensor([[3], [OOV]])]), id='extend-oov-tensor'),
    pytest.param(TP, 1, lambda d: d.extend([[1, 2]]), id='extend-tp'),
    pytest.param(None, 1, lambda d: d.score([[1, 2], [3, OOV]]), id='score-oov'),
    pytest.param(TP, 1, lambda d: d.score([[1, 2]]), id='score-tp'),
    pytest.param(None, 1, lambda d: d.perplexity(torch.tensor([[1, 2, OOV, 3]]), seqlen=2), id='perplexity-oov'),
    pytest.param(TP, 1, lambda d: d.perplexity([1, 2, 3, 4], seqlen=2), id='perplexity-tp'),
    pytest.param(None, 1, lambda d: d.generate([1, OOV], 4), id='generate-oov'),
    pytest.param(None, 1, lambda d: d.generate([1, 2], 4, eos_token_id=OOV), id='generate-eos-oov'),
    pytest.param(None, 1, lambda d: d.generate([1, 2], 4, eos_token_id=-1), id='generate-eos-negative'),
    pytest.param(TP, 1, lambda d: d.generate([1, 2], 4, do_sample=True), id='generate-tp-sample'),
    pytest.param(TP, 1, lambda d: d.generate([1, 2], 4, eos_token_id=3), id='generate-tp-eos'),
    pytest.param(TP, 1, lambda d: d.generate([1, 2], 4, reuse_cache=True), id='generate-tp-reuse'),
    pytest.param(None, 1, lambda d: d.generate([1, 2], 4, do_sample=True, top_p=1.5), id='generate-top_p'),
    pytest.param(None, 1, lambda d: d.generate([1, 2], 4, do_sample=True, temperature=-1.0), id='generate-temperature'),
    pytest.param(None, 1, lambda d: d.generate([1, 2], 4, min_new_tokens=-1), id='generate-min_new_tokens'),
    pytest.param(None, 2, lambda d: d.generate_batch([[1, 2], [3, OOV]], 4), id='generate_batch-oov'),
    pytest.param(None, 2, lambda d: d.generate_batch([[1, 2], [3]], 4, eos_token_id=[5, OOV]), id='generate_batch-eos-oov'),
    pytest.param(TP, 1, lambda d: d.generate_batch([[1, 2]], 4, reuse_cache=True), id='generate_batch-tp-reuse'),
    pytest.param(TP, 1, lambda d: d.generate_batch([[1, 2]], 4, do_sample=True), id='generate_batch-tp-sample'),
    pytest.param(None, 2, lambda d: d.generate_batch([[1, 2], [3]], 4, do_sample=True, temperature=[1.0]), id='generate_batch-temperature-list'),
    pytest.param(None, 2, lambda d: d.generate_batch([[1, 2], [3]], 4, do_sample=True, top_k=[5, -1]), id='generate_batch-top_k'),
    pytest.param(None, 1, lambda d: d.set_sampling(1.0, 50, 1.0, 0, eos_token_id=OOV), id='set_sampling-eos-oov'),
    pytest.param(TP, 1, lambda d: d.set_sampling(1.0, 50, 1.0, 0), id='set_sampling-tp'),
    pytest.param(None, 1, lambda d: d.set_sampling(1.0, 50, 0.0, 0), id='set_sampling-top_p'),
    pytest.param(None, 2, lambda d: d.set_sampling(1.0, 50, 1.0, 0, min_length=[1, 2, 3]), id='set_sampling-min_length-list'),
])
def test_decoder_entry_points_refuse_bad_arguments_before_any_device_work(tp, batch, call):
    """Out-of-vocabulary token ids, features a tensor-parallel rank does not run, and bad sampling arguments raise ValueError from every
    public entry point of the decoder while its checks run, before anything is written to the device, the cache or its record."""
    dec = _decoder_shell(tp, batch)
    with pytest.raises(ValueError, match='tensor parallelism' if tp else None):
        call(dec)
    assert dec.lengths == [0] * batch and dec.cached_tokens == [[]] * batch


def test_tensor_parallel_generate_batch_is_refused_before_the_cache_is_reset():
    """A tensor-parallel rank cannot prefill, so generate_batch refuses outright rather than feed the prompts through the decode step."""
    dec = _decoder_shell(TP, 1)
    with pytest.raises(ValueError, match='tensor parallelism'):
        dec.generate_batch([[1, 2, 3]], 4)
    with pytest.raises(ValueError, match='tensor parallelism'):
        dec.prefill_batch([[1, 2, 3]])
