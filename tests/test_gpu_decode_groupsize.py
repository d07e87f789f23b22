"""GPU: every quantized linear of the decode step, bit for bit, at every groupsize real checkpoints use, in both engines.

The probe layer of gs_probe.py (exact fields, RMSNorm and attention at position 0) is stepped once per case and each linear is read where
the step leaves it; every anchor must hold exactly (torch.equal against fp16 of the float64 sum):
    qkv              the appended K and V rows
    o_proj           x after attention (persistent kernel: resid_buffers[1] of a one-layer model; kernel chain: scratch offset 0), MLP scales 0
    gate/up -> down  x leaving layer 0 (persistent: resid_buffers[0] of a two-layer model; chain: scratch offset 0), o_proj scales 0
The groupsizes: 32 (one k-step per stage of the persistent kernel, per-step boxes), 64, 128, 1024 (a group spans 8 stages; down_proj's K =
11008 ends in a partial group of 768) and full (each linear's K: 4096, and 11008 on down_proj -- the reference's --groupsize -1).  At batch
8 the eight sequences carry distinct tokens, so each lane group of the batched kernel feeds its own x and the epilogue its own sums of x.
At LLaMA-65B shapes (hidden 8192, the persistent kernel's limit) the cases are gs 128 at batch 1, at the largest persistent batch and one
sequence above it (the kernel chain), gs 1024 (down_proj, K = 22016, ends in a partial group of 512) and int4 act-order gs 128 (the
qkv_perm / mlp_perm gathers at H = 8192); at LLaMA-33B gs 1024, where every linear ends in a partial group of 512, at batch 1 and the
largest persistent batch, and gs full on the kernel chain.  The batch limits come from the device's SM count (gs_probe.resolve_batch).
At the grouped-query shapes (qkv H + 2 Hkv wide, o_proj reading each K/V head's V row once per query head of its group): LLaMA-2-70B gs
128 at batch 1, the largest persistent batch, one above it and batch 8, gs 1024 at batch 7, int4 act-order gs 128; CodeLlama-34B gs 1024
at batch 1 and 8; LLaMA-3-8B gs 128 at batch 1 and 8 and gs full.  At 70B batch 7 and 8 the kernel chain runs gate|up and down_proj on
the generic kernel (the split-K matvec's x segment exceeds its shared memory there), with the RMSNorm and the residual add as separate
launches: 11 per step instead of 9.
Each case asserts its path: the launch count (gs_probe.chain_launches on the kernel chain) and the groupsize hint of every kernel layer.  tests/test_decode_groupsize_fixtures.py shows
on the CPU that the fixtures are exact and that a group, sequence or k-step mix-up would break these anchors; the last test here shows it
on the device.
"""
from functools import lru_cache

import pytest
import torch

import gs_probe as P
from attn_probe import resid_buffers
from gpu_util import fp16_ulp_distance

pytestmark = pytest.mark.gpu

def build(L, mode, B, n_layers):
    """LlamaDecoder of the probe layer: mode 'o' (gate / up / down scales 0) or 'mlp' (o_proj scales 0)."""
    from gptq_b200 import engine
    dev = torch.device('cuda:0')
    ly = {}
    for name, lin in L.linears().items():
        qw, sc, qz, g = lin.packed(dev)
        zero = (mode == 'o' and name in ('gate', 'up', 'down')) or (mode == 'mlp' and name == 'o')
        ly[name] = engine.QLayerWeights(qw, torch.zeros_like(sc) if zero else sc, qz, g, L.bits, P.group_size(L.gs, lin.K))
    ly['input_norm'] = torch.ones(L.H, dtype=torch.float16, device=dev)
    ly['post_norm'] = torch.ones(L.H, dtype=torch.float16, device=dev)
    embed = P.embed_rows(P.VOCAB, L.H).to(dev)
    lm_head = (torch.randn(P.VOCAB, L.H, generator=torch.Generator().manual_seed(5)) * 0.02).half().to(dev)
    return engine.LlamaDecoder([ly] * n_layers, embed, torch.ones(L.H, dtype=torch.float16, device=dev), lm_head, L.nh, rms_eps=0.0, batch=B,
                               max_seq=32, n_kv_heads=L.nkv)


def step(dec, toks):
    dec.set_input(toks, [0] * len(toks))
    dec.step()
    torch.cuda.synchronize()


def mismatch(got, want):
    """None when bit-identical, else a description of the differences."""
    if torch.equal(got, want):
        return None
    d = fp16_ulp_distance(got.reshape(-1), want.reshape(-1))
    i = int(torch.nonzero(d)[0])
    return f'{int((d > 0).sum())} / {d.numel()} elements off, up to {int(d.max())} ulp; first at {i}: {got.reshape(-1)[i].item()} vs {want.reshape(-1)[i].item()}'


def check_path(dec, L, B, engine_name, what):
    """One launch on the persistent kernel; on the chain 9 when the split-K matvec serves every linear, 2 more per linear it does not
    take (gs_probe.chain_launches)."""
    n = dec.launches_per_step()
    assert n == (1 if engine_name == 'persistent' else P.chain_launches(L, B)), f'{what}: {n} launches per step'
    for kl in dec.klayers:
        for name in ('qkv', 'o', 'gate', 'up', 'down'):
            K = L.linears()[name].K
            assert kl[name].hint == P.group_size(L.gs, K), f'{what}: {name} hint {kl[name].hint}'
            assert (kl[name].perm is not None) == L.act_order, f'{what}: {name}: regrouped rows expected exactly for act-order'


def x_after(dec, engine_name, B, H, which):
    """which 1: x after attention (one layer); 0: x leaving layer 0 (persistent: two layers)."""
    if engine_name == 'persistent':
        return resid_buffers(dec)[which]
    return dec.scratch[:B * H * 2].view(torch.float16).view(B, H).clone()


@lru_cache(maxsize=1)
def probe_layer(size, gs, bits, act):
    """The cases of one configuration follow each other in P.CASES: a 65B layer takes tens of seconds to draw on the CPU."""
    return P.layer_for(size, gs, bits, act)


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def run_case(size, gs, bits, act, B, engine_name):
    L = probe_layer(size, gs, bits, act)
    B = P.resolve_batch(B, L.nh, sms())
    H, dev = L.H, torch.device('cuda:0')
    toks = P.tokens(B)
    x_in = P.embed_rows(P.VOCAB, H)[torch.tensor(toks)]
    E = P.Expect(L, x_in, device=dev)
    assert bool((E.a >= 20).all()), 'gate outputs below 20: the sigmoid is not exactly 1'
    route = '' if engine_name == 'persistent' else f', {P.chain_launches(L, B)} launches'
    what = f'{size} int{bits} act={act} gs={gs} batch {B} ({engine_name}{route})'
    bad = []
    for mode in ('o', 'mlp'):
        n_layers = 2 if (mode == 'mlp' and engine_name == 'persistent') else 1
        dec = build(L, mode, B, n_layers)
        check_path(dec, L, B, engine_name, what)
        step(dec, toks)
        for b in range(B):
            for name, got, want in (('K row', dec.k_cache[0, b, :, 0], E.k[b]), ('V row', dec.v_cache[0, b, :, 0], E.v[b])):
                m = mismatch(got.reshape(-1), want)
                if m:
                    bad.append(f'{what} [{mode} probe] seq {b} {name} (qkv): {m}')
        if mode == 'o':
            got, want, lin = x_after(dec, engine_name, B, H, 1), E.x_attn, 'x after attention (o_proj)'
        else:
            got, want, lin = x_after(dec, engine_name, B, H, 0), E.x_mlp, 'x leaving the layer (gate/up -> down)'
        for b in range(B):
            m = mismatch(got[b], want[b])
            if m:
                bad.append(f'{what} seq {b} {lin}: {m}')
        del dec
    torch.cuda.empty_cache()
    print(f'  {what}: {"every anchor bit-exact" if not bad else f"{len(bad)} anchors broken"}')
    assert not bad, '\n'.join(bad)


@pytest.mark.parametrize('size,gs,bits,act,B,engine_name', P.CASES, ids=lambda v: str(v))
def test_decode_linears_bit_exact(size, gs, bits, act, B, engine_name):
    run_case(size, gs, bits, act, B, engine_name)


def test_swapped_scale_rows_break_the_anchors():
    """Two adjacent groups' scale rows of qkv swapped in the device copy only (every column has different scales in the two, gs_probe):
    the K rows must then miss their anchor in most elements -- the anchors see a group mix-up in the kernel's indexing."""
    swapped_scale_rows(P.layer_for('7b', 128, 4, False))


def test_swapped_scale_rows_break_the_anchors_65b():
    """The same at LLaMA-65B shapes (hidden 8192): the anchors of the largest configuration see a group mix-up too."""
    swapped_scale_rows(probe_layer('65b', 128, 4, False))


def swapped_scale_rows(L):
    dev = torch.device('cuda:0')
    toks = P.tokens(1)
    E = P.Expect(L, P.embed_rows(P.VOCAB, L.H)[torch.tensor(toks)], device=dev)
    dec = build(L, 'o', 1, 1)
    assert dec.launches_per_step() == 1
    sc = dec.klayers[0]['qkv'].scales
    assert sc.data_ptr() == dec.layers[0]['qkv'].scales.data_ptr()  # int4, trivial g_idx: the kernel reads the stored tensor
    step(dec, toks)
    assert torch.equal(dec.k_cache[0, 0, :, 0].reshape(-1), E.k[0])
    sc[[3, 4]] = sc[[4, 3]].clone()
    step(dec, toks)
    got = dec.k_cache[0, 0, :, 0].reshape(-1)
    off = int((got != E.k[0]).sum())
    print(f'  {L.size}: qkv scale rows 3 and 4 swapped: {off} / {got.numel()} K-row elements miss the anchor')
    assert off >= got.numel() // 2, f'only {off} elements moved'
    sc[[3, 4]] = sc[[4, 3]].clone()
    step(dec, toks)
    assert torch.equal(dec.k_cache[0, 0, :, 0].reshape(-1), E.k[0])
