"""Extending cached sequences on one GPU, one JSON line:
  * the causal attention over the KV cache (gptq_cached_attention) alone at LLaMA-7B attention shapes (32 heads, head_dim 128, max_seq 2048):
    (a) batch 1, a 512-row chunk at start 1536; (b) batch 8, chunks of 256 rows at ragged starts.  CUDA-event time over >= 50 launches after
    warm-up, achieved TFLOP/s (4 * 128 * heads * sum over rows of the keys they see, start + i + 1) and its share of the 989 TFLOP/s dense fp16
    data-sheet rate; alternated with it in the same process, the torch restatement (per-span SDPA with an explicit offset-causal mask over the
    cache rows 0 .. start + rows - 1) on the same inputs, and the max difference between the two;
  * end to end on a synthetic LLaMA-7B int4 g128 (32 layers): the time to the first token of a second turn -- 1536 cached positions plus 512
    new prompt tokens -- with generate(..., reuse_cache=True), against re-prefilling all 2048 tokens (reuse_cache=False) and against feeding
    the 512 through the decode step (prefill=False, reuse_cache=True).
The card's name and power limit are read in the same run.  Nothing is written to disk."""
import json
import os
import statistics
import sys
import time

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'gptq-for-llama_b200'))
from gptq_b200 import engine, ops  # noqa: E402
from score_bench import PEAK_TFLOPS, gpu_identity, timed  # noqa: E402

HEADS, HD, MAX_SEQ = 32, 128, 2048


def kernel_vs_torch(name, starts, rows, launches=50, rounds=3):
    B = len(starts)
    g = torch.Generator(device='cuda').manual_seed(B)
    kc = torch.randn(B, HEADS, MAX_SEQ, HD, device='cuda', generator=g).half()
    vc = torch.randn(B, HEADS, MAX_SEQ, HD, device='cuda', generator=g).half()
    spans = [(b, s, rows) for b, s in enumerate(starts)]
    q = torch.randn(B * rows, HEADS * HD, device='cuda', generator=g).half()
    masks = [torch.arange(s + rows, device='cuda')[None, :] <= (s + torch.arange(rows, device='cuda'))[:, None] for s in starts]
    kernel = lambda: ops.cached_attention(q, kc, vc, spans)

    def restated():
        outs = []
        for (b, s, n), m in zip(spans, masks):
            qs = q[b * rows:(b + 1) * rows].view(n, HEADS, HD).transpose(0, 1)[None]
            o = F.scaled_dot_product_attention(qs, kc[b:b + 1, :, :s + n], vc[b:b + 1, :, :s + n], attn_mask=m)
            outs.append(o[0].transpose(0, 1).reshape(n, HEADS * HD))
        return torch.cat(outs)

    diff = (kernel().float() - restated().float()).abs().max().item()
    for _ in range(3):
        kernel()
        restated()
    kt, tt = [], []
    for _ in range(rounds):  # alternated, so that both see the same state of the shared machine
        kt.append(timed(kernel, launches)[0])
        tt.append(timed(restated, launches)[0])
    kms, tms = statistics.median(kt), statistics.median(tt)
    flop = 4 * HD * HEADS * sum(s * rows + rows * (rows + 1) // 2 for s in starts)
    tflops = flop / (kms * 1e-3) / 1e12
    return {'case': name, 'starts': starts, 'rows': rows, 'kernel_ms': round(kms, 4), 'kernel_ms_all': [round(v, 4) for v in kt],
            'kernel_tflops': round(tflops, 1), 'kernel_share_of_989': round(tflops / PEAK_TFLOPS, 3), 'torch_sdpa_ms': round(tms, 4),
            'torch_sdpa_ms_all': [round(v, 4) for v in tt], 'max_abs_diff_kernel_vs_torch': diff}


def second_turn(cached=1536, new=512, reps=3):
    dec = engine.synthetic_llama('7b', bits=4, groupsize=128, vocab=32000, max_seq=MAX_SEQ, seed=0)
    ids = torch.randint(0, 32000, (cached + new, ), generator=torch.Generator().manual_seed(0)).tolist()
    dec.generate(ids[:cached + 1], 1)  # turn 1: the first `cached` positions are in the cache

    def keep_first_turn():  # what the cache holds after turn 1 (the rows past it are stale and get rewritten)
        dec.lengths, dec.cached_tokens = [cached], [ids[:cached]]

    def run(**kw):
        keep_first_turn()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        tok = dec.generate(ids, 1, **kw)[-1]  # host list: ends in a device synchronise
        return time.perf_counter() - t0, tok

    legs = {'reuse_cache_extend': dict(reuse_cache=True), 'reprefill_all': dict(), 'reuse_cache_decode_steps': dict(prefill=False, reuse_cache=True)}
    for kw in legs.values():
        run(**kw)  # warm-up
    times, toks = {k: [] for k in legs}, {k: set() for k in legs}
    for _ in range(reps):
        for k, kw in legs.items():
            t, tok = run(**kw)
            times[k].append(t)
            toks[k].add(tok)
    res = {'config': f'LLaMA-7B int4 g128, 32 layers, {cached} cached + {new} new tokens, time to the first token'}
    for k in legs:
        res[k + '_ms'] = round(statistics.median(times[k]) * 1e3, 2)
        res[k + '_ms_all'] = [round(v * 1e3, 2) for v in times[k]]
        res[k + '_first_tokens'] = sorted(toks[k])
    return res


def main():
    assert torch.cuda.is_available(), 'extend_bench needs a CUDA device'
    torch.cuda.set_device(0)
    res = {'gpu': gpu_identity(),
           'kernel': [kernel_vs_torch('B=1, 512 rows at 1536', [1536], 512),
                      kernel_vs_torch('B=8, 256 rows at ragged starts', [0, 129, 384, 700, 1000, 1311, 1536, 1792], 256)]}
    torch.cuda.empty_cache()
    res['end_to_end'] = second_turn()
    print(json.dumps(res))


if __name__ == '__main__':
    main()
