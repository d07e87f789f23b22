"""On-device sampling on one GPU, one JSON line:
  * the sampling kernel (gptq_sample_tokens) alone at V = 32000, B in {1, 8}: llama_inference.py's settings (temperature 0.8, top_k 50,
    top_p 0.95) and top_k 0 with top_p 0.95 (the whole vocabulary a candidate).  CUDA-event time per launch over 50 launches after warm-up,
    median of three rounds alternated with a torch restatement on the same logits (HF's temperature / top-k / top-p warpers, softmax,
    torch.multinomial, all on the GPU);
  * end to end on a synthetic LLaMA-7B int4 g128 (32 layers): tokens/s of generate_batch sampled against greedy at B = 1 and 8, in the same
    process, alternated.
The card's name and power limit are read in the same run.  Nothing is written to disk."""
import json
import os
import statistics
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'gptq-for-llama_b200'))
from gptq_b200 import engine, ops  # noqa: E402
from score_bench import gpu_identity, timed  # noqa: E402

V = 32000


def torch_restated(logits, temperature, top_k, top_p):
    """HF's TemperatureLogitsWarper -> TopKLogitsWarper -> TopPLogitsWarper on logits.float(), then softmax and torch.multinomial."""
    s = logits.float() / temperature
    if top_k:
        s = s.masked_fill(s < torch.topk(s, top_k)[0][..., -1, None], -float('inf'))
    if top_p < 1:
        sl, si = torch.sort(s, descending=False)
        rm = sl.softmax(-1).cumsum(-1) <= 1 - top_p
        rm[..., -1:] = False
        s = s.masked_fill(rm.scatter(1, si, rm), -float('inf'))
    return torch.multinomial(s.softmax(-1), 1)[:, 0]


def kernel_vs_torch(B, temperature, top_k, top_p, launches=50, rounds=3):
    g = torch.Generator(device='cuda').manual_seed(B)
    logits = (torch.randn(B, V, device='cuda', generator=g) * 3).half()
    full = lambda v, dt: torch.full((B, ), v, dtype=dt, device='cuda')
    pos = torch.arange(B, dtype=torch.int32, device='cuda')
    prm = (full(temperature, torch.float32), full(top_k, torch.int32), full(top_p, torch.float32), full(7, torch.int64))
    out = torch.empty(B, dtype=torch.int32, device='cuda')
    kernel = lambda: ops.sample_tokens(logits, pos, *prm, out=out)
    restated = lambda: torch_restated(logits, temperature, top_k, top_p)
    for _ in range(3):
        kernel()
        restated()
    kt, tt = [], []
    for _ in range(rounds):
        kt.append(timed(kernel, launches)[0])
        tt.append(timed(restated, launches)[0])
    return {'B': B, 'temperature': temperature, 'top_k': top_k, 'top_p': top_p, 'kernel_us': round(statistics.median(kt) * 1e3, 2),
            'kernel_us_all': [round(v * 1e3, 2) for v in kt], 'torch_us': round(statistics.median(tt) * 1e3, 2), 'torch_us_all': [round(v * 1e3, 2) for v in tt]}


def end_to_end(B, new=128, reps=3):
    dec = engine.synthetic_llama('7b', bits=4, groupsize=128, vocab=V, max_seq=512, batch=B, seed=0)
    prompts = [torch.randint(0, V, (16 + 8 * b, ), generator=torch.Generator().manual_seed(b)).tolist() for b in range(B)]
    legs = {'greedy': dict(), 'sampled': dict(do_sample=True, temperature=0.8, top_k=50, top_p=0.95, seed=1)}

    def run(kw):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        dec.generate_batch(prompts, new, **kw)  # host lists: ends in a device synchronise
        return time.perf_counter() - t0

    for kw in legs.values():
        run(kw)  # warm-up (captures the sampled graph)
    times = {k: [] for k in legs}
    for _ in range(reps):
        for k, kw in legs.items():
            times[k].append(run(kw))
    res = {'config': f'LLaMA-7B int4 g128, 32 layers, B={B}, {new} new tokens per sequence (prefill included)', 'launches_per_step': dec.launches_per_step()}
    for k in legs:
        res[k + '_tok_s'] = round(B * new / statistics.median(times[k]), 1)
        res[k + '_s_all'] = [round(v, 4) for v in times[k]]
    res['sampled_over_greedy_time'] = round(statistics.median(times['sampled']) / statistics.median(times['greedy']), 4)
    del dec
    torch.cuda.empty_cache()
    return res


def main():
    assert torch.cuda.is_available(), 'sample_bench needs a CUDA device'
    torch.cuda.set_device(0)
    res = {'gpu': gpu_identity(), 'kernel': [kernel_vs_torch(B, *case) for case in ((0.8, 50, 0.95), (0.8, 0, 0.95)) for B in (1, 8)]}
    res['end_to_end'] = [end_to_end(1), end_to_end(8)]
    print(json.dumps(res))


if __name__ == '__main__':
    main()
