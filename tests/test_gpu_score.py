"""GPU: scoring -- the fused lm_head + log-softmax kernel (gptq_lm_head_logprob) against a float64 log-softmax with a per-element bound,
bit-exact anchors on an integer grid, tile edges, determinism; LlamaDecoder.score / perplexity against the oracle and against the
reference's own perplexity formula on the HF module path; no side effects on the decode state; which kernels run."""
import math

import pytest
import torch

from gpu_util import check_logprob, launched_kernels, lse_tol, random_logprob_inputs, report, run_kernel, tiny_quant_llama
from llama_oracle import CODELLAMA, LLAMA1, LlamaOracle, check_scores, scale_down_embedding_row

pytestmark = pytest.mark.gpu

# ----------------------------------------------------------------------------- the kernel
def test_exact_anchors_on_an_integer_grid():
    """x = a 2^-4, W = b 2^-4 with small integers: every product and partial sum is a multiple of 2^-8 below 2^16 (exact in fp32) and every
    logit is a multiple of 2^-8 below 8, or 1000: exact in fp16.  Then only the fp32 log-softmax separates the kernel from float64."""
    check_integer_grid_anchors(32001)


def test_exact_anchors_on_an_integer_grid_at_the_llama3_vocabulary():
    """The same at LLaMA-3's vocabulary, 128256: the combine pass merges 1002 vocabulary tiles per row, 32 per lane."""
    check_integer_grid_anchors(128256)


def integer_grid_inputs(V, K=5120, P=4000, vstar=4242):
    """(x [19, K], W [V, K], targets) on the device, every value exact in fp16 (W is built in fp16: 1.3 GB at V = 128256)."""
    g = torch.Generator().manual_seed(0)
    W = torch.zeros(V, K, dtype=torch.float16)
    idx = torch.randint(0, K, (V, 64), generator=g)
    W.scatter_(1, idx, (torch.randint(1, 3, (V, 64), generator=g) * (2 * torch.randint(0, 2, (V, 64), generator=g) - 1)).half())  # <= 64 nonzeros in +-{1,2}
    W[vstar] = 0
    W[vstar, :P] = 8  # only the dominant row reaches this vocabulary row
    x = torch.zeros(19, K)
    x[:16, P:] = torch.randint(-3, 4, (16, K - P), generator=g).float()  # ordinary rows: |l| <= 64 * 3 * 2 * 2^-8 = 1.5
    # row 16: all zeros -> every logit 0 -> -log V; rows 17, 18: the dominant row, l[vstar] = 4000 * 64 * 2^-8 = 1000, every other |l| <= 4
    x[17:, :P] = 8
    targets = torch.tensor([0, 127, 128, V - 1, vstar] + torch.randint(0, V, (11, ), generator=g).tolist() + [5, vstar, 0], dtype=torch.int32)
    W = W.cuda()
    W /= 16  # exact: a power of two on small integers
    return (x / 16).half().cuda(), W, targets.cuda()


def check_integer_grid_anchors(V):
    from gptq_b200 import ops
    x, W, targets = integer_grid_inputs(V)
    lp = ops.lm_head_logprob(x, W, targets)
    ref = check_logprob(lp, x, W, targets, f'integer grid V={V}', exact=True)
    assert abs(ref[16].item() + math.log(V)) < 1e-12 and abs(lp[16].item() + math.log(V)) <= lse_tol(0.0, V, ref[16]).item()
    assert lp[17].item() == 0.0  # every other exp underflows: 1000 - (1000 + log 1)
    assert ref[18].item() < -990 and lp[18].item() == ref[18].item()  # l_0 - 1000 is exact


EDGES = ([(M, 32001, 256, None, None) for M in (1, 2, 127, 128, 129, 255, 256, 257, 4099)] + [(257, V, 64, None, None) for V in (300, 1000, 32000, 32001)] +
         [(129, 1000, K, None, None) for K in (64, 256, 4096, 5120)] + [(300, 32001, 4096, 4096 + 64, 4096 + 8), (129, 300, 64, 72, 128)] +
         [(M, 128256, 4096, None, None) for M in (1, 257, 4099, 8191)])  # LLaMA-3-8B: 1002 vocabulary tiles; a perplexity chunk of 8191 rows


@pytest.mark.parametrize('M,V,K,ldx,ldw', EDGES)
def test_tile_edges_against_fp64(M, V, K, ldx, ldw):
    from gptq_b200 import ops
    x, W, t = random_logprob_inputs(M, V, K, ldx, ldw, seed=M + V + K)
    assert (ldx is None or x.stride(0) == ldx) and (ldw is None or W.stride(0) == ldw)
    check_logprob(ops.lm_head_logprob(x, W, t), x, W, t, f'M={M} V={V} K={K} ldx={ldx} ldw={ldw}')


def test_deterministic_and_independent_of_the_other_rows():
    from gptq_b200 import ops
    x, W, t = random_logprob_inputs(4099, 32000, 4096, seed=7)
    a = ops.lm_head_logprob(x, W, t)
    b = ops.lm_head_logprob(x, W, t)
    assert torch.equal(a, b)
    alone = ops.lm_head_logprob(x[:100].contiguous(), W, t[:100].clone())
    assert torch.equal(alone, a[:100])


def test_workspace_is_left_zeroed_and_bad_targets_are_rejected():
    from gptq_b200 import ops
    x, W, t = random_logprob_inputs(300, 1000, 256, seed=3)
    ops.lm_head_logprob(x, W, t)
    torch.cuda.synchronize()
    for ws in ops._workspaces.values():
        assert int(ws.count_nonzero()) == 0
    for bad in (-1, 1000):
        tb = t.clone()
        tb[5] = bad
        with pytest.raises(ValueError):
            ops.lm_head_logprob(x, W, tb)


def test_measured_configuration_7b():
    """LLaMA-7B shapes (K 4096, V 32000), one 2048-row chunk of final-normed hidden rows of a 2-layer synthetic 7B engine, against float64;
    perplexity() of the same engine is finite and is the exponentiated mean NLL of score()."""
    from gptq_b200 import engine, ops
    dec = engine.synthetic_llama('7b', bits=4, groupsize=128, n_layers=2, vocab=32000, max_seq=16, use_graph=False, seed=0)
    ids = torch.randint(0, 32000, (2 * 2048 + 7, ), generator=torch.Generator().manual_seed(0)).tolist()
    with torch.no_grad():
        x = ops.rmsnorm(dec._forward_rows([ids[:2048]]), dec.final_norm, dec.model.rms_eps)
    t = torch.tensor(ids[1:2049], dtype=torch.int32, device='cuda')
    lp = ops.lm_head_logprob(x, dec.lm_head, t)
    check_logprob(lp, x, dec.lm_head, t, '7b chunk')
    assert torch.equal(dec.score([ids[:2048]])[0], lp[:2047])
    ppl = dec.perplexity(ids, seqlen=2048)
    lps = dec.score([ids[:2048], ids[2048:4096]])
    assert math.isfinite(ppl) and ppl > 1
    assert ppl == pytest.approx(math.exp(-float(torch.cat(lps).double().sum()) / (2 * 2047)), rel=1e-12)


# ----------------------------------------------------------------------------- the engine
ENGINES = [('tiny', 4, False), ('tiny', 4, True), ('tiny', 3, True), ('tiny', 8, False), ('tiny256', 4, False), ('tiny256', 4, True),
           ('tiny256', 3, True), ('tiny256', 8, False)]


@pytest.mark.parametrize('size,bits,act,rope', [pytest.param(*e, LLAMA1, id='-'.join(map(str, e))) for e in ENGINES] +
                         [pytest.param(size, 4, False, CODELLAMA, id=f'{size}-4-False-codellama') for size in ('tiny', 'tiny256')])
def test_score_matches_the_oracle(size, bits, act, rope):
    """Three sequences of different lengths in one call against float64 log-softmaxes of the oracle's fp16 per-position logits.  The prefill
    and decode tests hold the logits to 2e-2 * max|ref logits| of the oracle; logsumexp is 1-Lipschitz in the max-norm, so the target logit
    and the logsumexp move by at most that each: 2 x 2e-2 x max|ref logits| per element.  Also at the CodeLlama settings (RoPE base 1e6,
    RMSNorm epsilon 1e-5), with the first token's embedding row scaled near the epsilon."""
    from gptq_b200 import engine
    base, eps = rope
    dec = engine.synthetic_llama(size, bits=bits, groupsize=64, act_order=act, vocab=300, seed=bits + act, max_seq=16, use_graph=False, rope_base=base,
                                 rms_eps=eps)
    _score_against_oracle(dec, bits, f'{size} bits={bits} act={act} base={base:g} eps={eps:g}', rope=rope)


@pytest.mark.parametrize('gs, kernel', [(32, 'qlinear_generic_kernel'), (-1, 'qgemm_wgmma_kernel')])
def test_score_matches_the_oracle_at_groupsizes(gs, kernel):
    """The same at groupsize 32 and -1 (one group per linear: 256, and 768 on down_proj).  The 34-row pass asserts its kernels: the wgmma
    GEMM needs groupsize % 64 == 0, so at 32 every quantized linear of it runs on the generic kernel."""
    from gptq_b200 import engine
    dec = engine.synthetic_llama('tiny256', bits=4, groupsize=gs, vocab=300, seed=7, max_seq=16, use_graph=False)
    _score_against_oracle(dec, 4, f'tiny256 gs={gs}', kernel)


def _score_against_oracle(dec, seed, what, kernel=None, rope=LLAMA1):
    g = torch.Generator().manual_seed(seed)
    seqs = [torch.randint(0, 300, (n, ), generator=g).tolist() for n in (9, 2, 23)]
    base, eps = rope
    if rope != LLAMA1:
        scale_down_embedding_row(dec.embed, seqs[0][0], 8)
    out = dec.score(seqs) if kernel is None else run_kernel(lambda: dec.score(seqs), kernel, f'{what}: score')
    assert [o.shape[0] for o in out] == [8, 1, 22] and all(o.dtype == torch.float32 for o in out)
    check_scores(out, seqs, LlamaOracle.from_decoder(dec, eps=eps, base=base), what)


def test_perplexity_matches_the_reference_formula_on_the_hf_modules():
    """llama_eval's arithmetic on the HF module path (model(chunk).logits, shifted fp16 CrossEntropyLoss, loss.float() * seqlen,
    exp(sum / (nsamples * seqlen))) against LlamaDecoder.perplexity of the same quantized model, with a tail that is dropped.
    Bound: the HF modules and the engine are each within 2e-2 * max|logits| of the oracle (test_load_quant_pipeline_on_tiny_llama, the
    prefill tests), so a log-prob differs by at most 2 x 2 x 2e-2 x max|logits|; the reference's fp16 CrossEntropyLoss rounds the
    log-softmax outputs and the mean loss (|loss| < 8: half an ulp, 2^-9, each).  The mean NLL differs by at most the sum of the two."""
    import quant
    from gptq_b200 import engine
    model = tiny_quant_llama(hidden=256, intermediate=768, heads=2)
    quant.make_quant_attn(model)
    quant.make_quant_norm(model)
    quant.make_fused_mlp(model)
    model = model.cuda()
    seqlen, V = 64, model.config.vocab_size
    ids = torch.randint(0, V, (1, 3 * seqlen + 5), generator=torch.Generator().manual_seed(0)).cuda()
    nsamples = ids.numel() // seqlen
    nlls, maxabs = [], 0.0
    with torch.no_grad():
        for i in range(nsamples):
            batch = ids[:, i * seqlen:(i + 1) * seqlen]
            lm_logits = model(batch).logits
            maxabs = max(maxabs, lm_logits.abs().max().item())
            shift_logits = lm_logits[:, :-1, :].contiguous()
            loss = torch.nn.CrossEntropyLoss()(shift_logits.view(-1, shift_logits.size(-1)), batch[:, 1:].reshape(-1))
            nlls.append(loss.float() * seqlen)
    ref = torch.exp(torch.stack(nlls).sum() / (nsamples * seqlen)).item()
    ppl = engine.from_hf_quant_model(model, max_seq=16, use_graph=False).perplexity(ids[0], seqlen=seqlen)
    bound = math.expm1(2 * 2 * 2e-2 * maxabs + 2 * 2.0**-9)
    report(abs(ppl / ref - 1) / bound, f'perplexity {ppl:.6f} vs reference formula {ref:.6f}')


def test_score_has_no_side_effects_on_the_decode_state():
    from gptq_b200 import engine
    dec = engine.synthetic_llama('tiny256', bits=4, groupsize=64, vocab=300, seed=4, max_seq=32)
    prompt = [3, 1, 4, 1, 5, 9, 2, 6]
    before = dec.generate(prompt, 6)
    torch.cuda.synchronize()
    names = ('k_cache', 'v_cache', 'positions', 'tokens', 'logits', 'next_tokens')
    snap = {n: getattr(dec, n).clone() for n in names}
    dec.score([list(range(40)), [7, 8, 9]])  # longer than max_seq: scoring does not use the cache
    torch.cuda.synchronize()
    for n in names:
        assert torch.equal(getattr(dec, n), snap[n]), n
    assert dec.generate(prompt, 6) == before


def test_score_launches_the_fused_kernels_and_no_decode_kernel():
    from gptq_b200 import engine
    dec = engine.synthetic_llama('tiny256', bits=4, groupsize=64, vocab=300, seed=5, max_seq=16)
    _, names = launched_kernels(lambda: dec.score([[1, 2, 3, 4, 5], [6, 7, 8]]))
    if not names:
        pytest.skip('CUDA activity tracing returned no kernel events on this machine')
    assert any('lm_head_logprob_kernel' in n for n in names), sorted(names)
    assert any('lm_head_logprob_combine_kernel' in n for n in names), sorted(names)
    decode = ('llama_decode_mega_kernel', 'attn_decode_kernel', 'attn_combine_kernel', 'lm_head_kernel', 'argmax_kernel', 'embed_kernel')
    assert not [n for n in names if any(d + '(' in n or d + '<' in n for d in decode)], sorted(names)


def test_score_and_perplexity_validate_their_input():
    from gptq_b200 import engine
    dec = engine.synthetic_llama('tiny', bits=4, groupsize=64, vocab=300, seed=6, max_seq=16, use_graph=False)
    for bad in ([[1]], [[1, 300]], [[-1, 2]]):
        with pytest.raises(ValueError):
            dec.score(bad)
    with pytest.raises(ValueError):
        dec.perplexity(list(range(63)), seqlen=64)
