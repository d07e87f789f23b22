"""GPU: the persistent decode kernel (llama_decode_mega_kernel) at the shapes bench.py measures.

The small-model tests (test_gpu_engine.py) cannot reach the stream-K ranges, attention unit splits, ring wrap-arounds and
staging sizes of the 7B / 13B configurations, so here the kernel runs LLaMA-7B-shaped (int4 g128, BASELINE config 2) and
LLaMA-13B-shaped (int3 g128 act-order, config 4) layers -- two of them, which exercises every inter-layer hand-off -- on a
randomly filled KV cache at the context positions {0, 255, 256, 2046, 2047}, against the oracle (tests/llama_oracle.py); and 7B at
the groupsizes 32, 1024 and -1 (one group per linear) at the positions {0, 2047}.  LLaMA-65B-shaped layers (int4 g128, bench.py
--config 65b: hidden 8192, the kernel's limit) run at the same five positions, LLaMA-33B-shaped ones at gs 1024 (every linear ends in a
partial group of 512) at {0, 2047}.

Checked per BLOCK, each block's oracle fed with the kernel's own input to that block (read back from its scratch), so that a
1e-3-class bound stays meaningful: a decoder is a chain of fp16 rounding points, and a one-ulp difference early on (any other
fp32 summation order produces some) re-rolls every later rounding -- measured run to run on this kernel: up to 3e-3 of rms on
the logits after ONE layer -- which says nothing about any single operation.
  * attention block of the last layer: x entering the layer -> RMSNorm, qkv, RoPE, KV append, attention, o_proj, residual
  * MLP block of the last layer + head: x after attention -> RMSNorm, gate/up, SwiGLU, down, residual, final norm, lm_head
for the one-layer and the two-layer model (the second one's input has gone through a full layer of the kernel), plus a loose
end-to-end bound on the logits against the oracle run from the embedding.
"""
import pytest
import torch

from llama_oracle import END_TO_END_TOL, LlamaOracle, assert_no_failures, check, check_last_layer_blocks, scale_down_embedding_row

pytestmark = pytest.mark.gpu


def _run_case(size, bits, act, positions, vocab, seed, gs=128, max_seq=2048, rms_eps=1e-6, rope_base=10000.0, small_embedding=False,
              k_row_vs_reference=True):
    """Both decoders and every oracle call take max_seq, rms_eps and rope_base from the arguments.  small_embedding: the token of the first
    position has its embedding row scaled by 2^-8 (mean square about 4e-6, near the epsilon), so that the 1-layer checks see the epsilon.
    k_row_vs_reference=False holds the appended K rows to the exact linears only (see the comment in the loop)."""
    from gptq_b200 import engine
    dec2 = engine.synthetic_llama(size, bits=bits, groupsize=gs, act_order=act, vocab=vocab, seed=seed, max_seq=max_seq, n_layers=2, rms_eps=rms_eps,
                                  rope_base=rope_base)
    assert dec2.launches_per_step() == 1, 'the persistent kernel must be the path under test'
    for name, ly in dec2.klayers[0].items():
        if hasattr(ly, 'qweight'):
            assert ly.hint == (ly.g_idx.numel() if gs == -1 else gs), f'{name}: groupsize hint {ly.hint}'
    if small_embedding:
        scale_down_embedding_row(dec2.embed, 3, 8)  # the token of the first position (17 * 0 + 3)
    dec1 = engine.LlamaDecoder(dec2.layers[:1], dec2.embed, dec2.final_norm, dec2.lm_head, dec2.n_heads, max_seq=max_seq, rms_eps=rms_eps, rope_base=rope_base)
    assert dec1.launches_per_step() == 1
    gen = torch.Generator(device=dec2.dev).manual_seed(seed + 100)
    dec2.k_cache.copy_((torch.randn(dec2.k_cache.shape, device=dec2.dev, generator=gen) * 0.5).half())
    dec2.v_cache.copy_((torch.randn(dec2.v_cache.shape, device=dec2.dev, generator=gen) * 0.5).half())
    kc, vc = dec2.k_cache.cpu(), dec2.v_cache.cpu()
    oracle = LlamaOracle.from_decoder(dec2, eps=rms_eps, base=rope_base)
    for i, pos in enumerate(positions):
        tok = (17 * i + 3) % vocab
        what = f'{size} int{bits} g{gs} act={act} eps={rms_eps:g} base={rope_base:g} pos={pos}'
        dec1.k_cache.copy_(dec2.k_cache[:1])
        dec1.v_cache.copy_(dec2.v_cache[:1])
        # The K row is rotated after the fp16 rounding of k, so a one-ulp difference in k before RoPE can land on a small element of the
        # rotated row, whose bound is relative to the row's rms: whether the reference's per-weight fp16 rounding does that is a matter of
        # the random draw, not of the groupsize.  The draw of the gs -1 case does it: at context 2047, layer 1, one K-row element is
        # 1.15 of its bound from the reference rounding, while the kernel equals Exact there (measured: fp64 9.289385, kernel and Exact
        # 9.2890625, the nearest fp16; reference rounding 9.296875).  That case holds its K rows to Exact only, and so does the LLaMA-2-13B
        # case: at context 4095, layer 0, one K-row element is 1.05 of its bound from the reference rounding (|err| 2.93e-3, row rms 1.12)
        # while the whole row stays within 0.39 of its bound from Exact.
        k_row = k_row_vs_reference and gs != -1
        check_last_layer_blocks(dec1, oracle, tok, pos, kc, vc, what + ' (1 layer)', k_row)
        logits2 = check_last_layer_blocks(dec2, oracle, tok, pos, kc, vc, what + ' (2 layers)', k_row)
        # end to end from the embedding
        x = dec2.embed[tok].cpu()[None, :].clone()
        for li in range(2):
            x = oracle.mlp(li, oracle.attention(li, x, pos, kc[li, 0], vc[li, 0])[0])
        check(logits2, oracle.head(x)[0], rel=END_TO_END_TOL, what=what + ': logits after 2 layers, end to end')
        dec2.k_cache.copy_(kc)  # every position starts from the same cache
        dec2.v_cache.copy_(vc)
    assert_no_failures()


def test_mega_kernel_7b_int4_g128_matches_oracle():
    """BASELINE config 2 shapes (hidden 4096, intermediate 11008, 32 heads, vocab 32000), the configuration bench.py times."""
    _run_case('7b', 4, False, [0, 255, 256, 2046, 2047], 32000, seed=11)


@pytest.mark.parametrize('gs', [32, 1024, -1])
def test_mega_kernel_7b_int4_groupsizes_match_oracle(gs):
    """The same 7B check at the other groupsizes of published checkpoints: 32 (one k-step per stage), 1024 (down_proj's K = 11008 ends
    in a partial group of 768) and -1 (one group per linear: 4096, and 11008 on down_proj)."""
    _run_case('7b', 4, False, [0, 2047], 32000, seed=14, gs=gs)


def test_mega_kernel_llama2_7b_matches_oracle():
    """LLaMA-2-7B settings: RMSNorm epsilon 1e-5, 4096 context, at the first, middle and last position; the first token's embedding row is
    scaled near the epsilon."""
    _run_case('7b', 4, False, [0, 2048, 4095], 32000, seed=18, max_seq=4096, rms_eps=1e-5, small_embedding=True)


def test_mega_kernel_codellama_7b_matches_oracle():
    """CodeLlama-7B settings: RMSNorm epsilon 1e-5, RoPE base 1e6, vocab 32016 (not a multiple of 32), 16384 context."""
    _run_case('7b', 4, False, [0, 4096, 16383], 32016, seed=19, max_seq=16384, rms_eps=1e-5, rope_base=1e6, small_embedding=True)


def test_mega_kernel_13b_int3_actorder_matches_oracle():
    """BASELINE config 4 shapes (hidden 5120, intermediate 13824, 40 heads), int3 g128 with act-order g_idx."""
    _run_case('13b', 3, True, [0, 2047], 8192, seed=12)


def test_mega_kernel_llama2_13b_int3_actorder_matches_oracle():
    """The int3 act-order 13B shapes at LLaMA-2-13B settings: RMSNorm epsilon 1e-5, 4096 context."""
    _run_case('13b', 3, True, [0, 4095], 8192, seed=20, max_seq=4096, rms_eps=1e-5, small_embedding=True, k_row_vs_reference=False)


def test_mega_kernel_65b_int4_g128_matches_oracle():
    """bench.py --config 65b shapes (hidden 8192, intermediate 22016, 64 heads, vocab 32000) at two of its 80 layers."""
    _run_case('65b', 4, False, [0, 255, 256, 2046, 2047], 32000, seed=16)


def test_mega_kernel_33b_int4_g1024_matches_oracle():
    """LLaMA-33B shapes (hidden 6656, intermediate 17920, 52 heads) at gs 1024: 6656 = 6 x 1024 + 512 and 17920 = 17 x 1024 + 512, so
    every linear ends in a partial group."""
    _run_case('33b', 4, False, [0, 2047], 32000, seed=17, gs=1024)


def test_mega_kernel_run_to_run_spread_7b():
    """The split-K partials are accumulated with unordered fp32 atomics, so two runs can round an accumulator to neighbouring
    fp16 values; every later rounding point then re-rolls (module docstring).  Measured here at 7B size, 4 layers, context 2047:
    the spread of the logits stays at the level of the fp16 rounding noise of the pipeline itself (a few ulps), the greedy
    token is stable, and nothing worse (a race would show up as far larger, structured differences)."""
    from gptq_b200 import engine
    dec = engine.synthetic_llama('7b', bits=4, groupsize=128, vocab=32000, seed=13, max_seq=2048, n_layers=4)
    dec.k_cache.normal_(0, 0.5)
    dec.v_cache.normal_(0, 0.5)
    kc, vc = dec.k_cache.clone(), dec.v_cache.clone()
    outs = []
    for _ in range(8):
        dec.k_cache.copy_(kc)
        dec.v_cache.copy_(vc)
        dec.tokens.fill_(5)
        dec.positions.fill_(2047)
        dec.step()
        torch.cuda.synchronize()
        outs.append(dec.logits[0].float().clone())
    ref = outs[0]
    rms = ref.pow(2).mean().sqrt().item()
    spread = max((o - ref).abs().max().item() for o in outs[1:])
    rms_spread = max((o - ref).pow(2).mean().sqrt().item() for o in outs[1:])
    print(f'run-to-run spread of the logits: max {spread:.3e}, rms {rms_spread:.3e}, rms(logits) {rms:.3e}')
    assert spread <= 1.5e-2 * rms, f'run-to-run spread {spread:.3e} vs rms {rms:.3e}'
    assert rms_spread <= 3e-3 * rms, f'rms run-to-run difference {rms_spread:.3e} vs rms {rms:.3e}'
    assert all(int(o.argmax()) == int(ref.argmax()) for o in outs)
