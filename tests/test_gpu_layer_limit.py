"""GPU: the persistent decode kernel at its 80-layer limit (kMaxLayers, the depth of LLaMA-65B), and the kernel chain one layer beyond it.

A LLaMA-65B-shaped stack (hidden 8192, 64 heads) that needs the memory of about two layers:
  * layers 0 .. n-2 all alias the tensors of one 65B probe layer of gs_probe.py (int4 g128) whose o_proj and down_proj scales are 0: each of
    them adds exactly 0 to the residual, but still runs its RMSNorm, qkv, attention and KV append;
  * the last layer has its own random tensors (engine.synthetic_llama).
Inputs are the probe's embedding rows with rms_eps = 0 and unit norms, at position 0.  Then x entering the last layer is the embedding row
bit for bit, and every aliased layer appends the probe's exact K / V rows (gs_probe.Expect.k / .v) to its own cache slice: the probe's sums
are exact in fp32, so these rows do not depend on the order in which the split-K atomics add.  The last layer is checked block by block
(llama_oracle.check_last_layer_blocks) on the persistent kernel; on the chain, which keeps no x after attention, its logits are
held to the oracle run from the (exact) embedding row at the MLP block's bound."""
import pytest
import torch

import gs_probe as P
from attn_probe import resid_buffers
from llama_oracle import MLP_HEAD_TOL, LlamaOracle, assert_no_failures, check, check_last_layer_blocks

pytestmark = pytest.mark.gpu

MAX_LAYERS = 80  # kMaxLayers (decode_mega.cu)
TOK = 5


def _stack():
    """(probe layer fields, the probe's decoder layer with o_proj / down_proj scales 0, the random last layer, its final norm and lm_head)."""
    from gptq_b200 import engine
    dev = torch.device('cuda:0')
    L = P.layer_for('65b', 128, 4, False)
    ly = {}
    for name, lin in L.linears().items():
        qw, sc, qz, g = lin.packed(dev)
        ly[name] = engine.QLayerWeights(qw, torch.zeros_like(sc) if name in ('o', 'down') else sc, qz, g, L.bits, P.group_size(L.gs, lin.K))
    ly['input_norm'] = torch.ones(L.H, dtype=torch.float16, device=dev)
    ly['post_norm'] = torch.ones(L.H, dtype=torch.float16, device=dev)
    rnd = engine.synthetic_llama('65b', bits=4, groupsize=128, vocab=P.VOCAB, seed=41, max_seq=64, n_layers=1)
    last, final_norm, lm_head = rnd.layers[0], rnd.final_norm, rnd.lm_head
    del rnd
    return L, ly, last, final_norm, lm_head


def _decoder(ly, last, final_norm, lm_head, n_layers):
    from gptq_b200 import engine
    embed = P.embed_rows(P.VOCAB, ly['input_norm'].numel()).to(ly['input_norm'].device)
    return engine.LlamaDecoder([ly] * (n_layers - 1) + [last], embed, final_norm, lm_head, P.SHAPES['65b'][2], rms_eps=0.0, max_seq=64)


def _check_aliased_kv(dec, E, n_alias, what):
    bad = []
    for li in range(n_alias):
        for name, cache, want in (('K', dec.k_cache, E.k[0]), ('V', dec.v_cache, E.v[0])):
            got = cache[li, 0, :, 0].reshape(-1)
            if not torch.equal(got, want):
                bad.append(f'{what}: layer {li} {name} row: {int((got != want).sum())} / {got.numel()} elements off')
    print(f'  {what}: K / V rows of the {n_alias} aliased layers {"bit-exact" if not bad else f"{len(bad)} broken"}')
    assert not bad, '\n'.join(bad[:20])


def test_persistent_kernel_at_80_layers_and_chain_at_81():
    L, ly, last, final_norm, lm_head = _stack()
    dev = torch.device('cuda:0')
    E = P.Expect(L, P.embed_rows(P.VOCAB, L.H)[torch.tensor([TOK])], device=dev)

    dec = _decoder(ly, last, final_norm, lm_head, MAX_LAYERS)
    assert dec.launches_per_step() == 1, f'{MAX_LAYERS} layers: {dec.launches_per_step()} launches'
    oracle = LlamaOracle.from_decoder(dec, eps=0.0, base=10000.0)  # only the last layer's blocks run on it
    kc, vc = dec.k_cache.cpu(), dec.v_cache.cpu()
    check_last_layer_blocks(dec, oracle, TOK, 0, kc, vc, f'65b {MAX_LAYERS} layers')
    x_in = resid_buffers(dec)[0][0]
    assert torch.equal(x_in, dec.embed[TOK]), 'x entering layer 79 is not the embedding row'
    _check_aliased_kv(dec, E, MAX_LAYERS - 1, f'65b {MAX_LAYERS} layers (persistent)')
    del dec

    n = MAX_LAYERS + 1
    dec = _decoder(ly, last, final_norm, lm_head, n)
    assert dec.launches_per_step() == 3 + 6 * n, f'{n} layers: {dec.launches_per_step()} launches, expected the kernel chain'
    dec.set_input([TOK], [0])
    dec.step()
    torch.cuda.synchronize()
    _check_aliased_kv(dec, E, n - 1, f'65b {n} layers (kernel chain)')
    x = dec.embed[TOK].cpu()[None, :].clone()
    x_attn, _, _ = oracle.attention(MAX_LAYERS - 1, x, 0, exact=True)  # the last layer: the same tensors at 80 and 81 layers
    check(dec.logits[0], oracle.head(oracle.mlp(MAX_LAYERS - 1, x_attn))[0], rel=MLP_HEAD_TOL,
          what=f'65b {n} layers (kernel chain): last layer + lm_head from the embedding row')
    assert_no_failures()
