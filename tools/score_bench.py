"""Scoring throughput on one GPU, one JSON line:
  * perplexity() of a synthetic LLaMA-7B int4 g128 (32 layers) over 8 chunks of 2048 tokens: scored tokens/s;
  * the fused lm_head + log-softmax kernel (gptq_lm_head_logprob) alone at M = 2048 and 16384 rows (K 4096, V 32000): CUDA-event time over
    >= 50 launches after warm-up, achieved TFLOP/s (2 M K V over that time) and its share of the 989 TFLOP/s dense fp16 data-sheet rate;
  * alternated with it in the same process, the torch restatement F.log_softmax((x @ W.T).float(), -1).gather(...) on the same inputs:
    its time and its peak of torch.cuda.max_memory_allocated above the inputs (the fused kernel's peak is measured the same way).
The card's name and power limit are read in the same run.  Nothing is written to disk."""
import json
import math
import os
import statistics
import subprocess
import sys
import time

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'gptq-for-llama_b200'))
from gptq_b200 import engine, ops  # noqa: E402

PEAK_TFLOPS = 989.0  # dense fp16, NVIDIA H100 SXM data sheet (700 W)
K, V = 4096, 32000


def gpu_identity():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i', '0'], capture_output=True, text=True,
                             timeout=30).stdout.strip()
        name, limit = [f.strip() for f in out.split(',')]
        return {'name': name, 'power_limit': limit}
    except (OSError, ValueError, subprocess.SubprocessError):
        return {'name': torch.cuda.get_device_name(0), 'power_limit': None}


def timed(fn, n):
    """Per-call milliseconds of n back-to-back calls (CUDA events), and the peak allocation above what was allocated before."""
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n, torch.cuda.max_memory_allocated() - base


def kernel_vs_torch(M, launches=50, rounds=3):
    g = torch.Generator(device='cuda').manual_seed(M)
    x = torch.randn(M, K, device='cuda', generator=g).half()
    W = (torch.randn(V, K, device='cuda', generator=g) * (2.5 / math.sqrt(K))).half()
    t = torch.randint(0, V, (M, ), device='cuda', generator=g, dtype=torch.int32)
    tl = t.long()[:, None]
    fused = lambda: ops.lm_head_logprob(x, W, t)
    restated = lambda: F.log_softmax((x @ W.T).float(), -1).gather(1, tl)[:, 0]
    diff = (fused() - restated()).abs().max().item()
    for _ in range(3):  # warm-up: module load, workspace, cuBLAS heuristics
        fused()
        restated()
    fk, tk, fmem, tmem = [], [], 0, 0
    for _ in range(rounds):  # alternated, so that both see the same state of the shared machine
        ms, mem = timed(fused, launches)
        fk.append(ms)
        fmem = max(fmem, mem)
        ms, mem = timed(restated, max(10, launches // 5))
        tk.append(ms)
        tmem = max(tmem, mem)
    fms, tms = statistics.median(fk), statistics.median(tk)
    tflops = 2 * M * K * V / (fms * 1e-3) / 1e12
    return {'M': M, 'fused_ms': round(fms, 4), 'fused_ms_all': [round(v, 4) for v in fk], 'fused_tflops': round(tflops, 1),
            'fused_share_of_989': round(tflops / PEAK_TFLOPS, 3), 'fused_peak_extra_bytes': fmem, 'torch_ms': round(tms, 4),
            'torch_ms_all': [round(v, 4) for v in tk], 'torch_peak_extra_bytes': tmem, 'max_abs_diff_fused_vs_torch': diff}


def perplexity_rate(seqlen=2048, nsamples=8, reps=3):
    dec = engine.synthetic_llama('7b', bits=4, groupsize=128, vocab=V, max_seq=16, use_graph=False, seed=0)
    ids = torch.randint(0, V, (seqlen * nsamples, ), generator=torch.Generator().manual_seed(0)).tolist()
    ppl = dec.perplexity(ids, seqlen)  # warm-up
    times, repeats = [], True
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        p = dec.perplexity(ids, seqlen)  # returns a host float: ends in a device synchronise
        times.append(time.perf_counter() - t0)
        repeats &= p == ppl
    s = statistics.median(times)
    scored = nsamples * (seqlen - 1)
    return {'config': f'LLaMA-7B int4 g128, 32 layers, {nsamples} x {seqlen} tokens', 'perplexity': ppl, 'seconds': round(s, 4),
            'seconds_all': [round(v, 4) for v in times], 'bit_identical_repeats': repeats, 'scored_tokens_per_s': round(scored / s, 1)}


def main():
    assert torch.cuda.is_available(), 'score_bench needs a CUDA device'
    torch.cuda.set_device(0)
    res = {'gpu': gpu_identity(), 'kernel': [kernel_vs_torch(2048), kernel_vs_torch(16384)]}
    torch.cuda.empty_cache()
    res['perplexity'] = perplexity_rate()
    print(json.dumps(res))


if __name__ == '__main__':
    main()
