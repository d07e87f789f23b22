#!/usr/bin/env python
"""Decode throughput of grouped-query-attention models: synthetic LLaMA-2-70B (all 80 layers) and LLaMA-3-8B, int4 g128, at batch 1 and 8,
one JSON line per (model, batch).

    python tools/gqa_bench.py [--models 70b,llama3-8b] [--batch 1,8] [--context 2047] [--steps K] [--warmup W]

Each of the B sequences has its own seeded random KV cache holding `context` tokens, and the step decodes the next token of every sequence.
Reported per line:
  value           aggregate tokens/s = B x steps / device time (CUDA events around the graph replays)
  engine          the persistent single kernel, or the kernel chain when the step is outside its plan (at 64 query heads and batch 8 the
                  512 (sequence, head) pairs exceed the attention teams of one kernel)
  bytes_per_step  algorithmic bytes, each counted once: quantized weights, fp16 lm_head, and every sequence's K/V rows (n_kv_heads per layer and
                  position).  The kernels stream a K/V row once per query head of its group; the repeats are expected to come from L2 and are
                  not counted
  roofline        those bytes over the step time, against the H100 SXM data sheet's HBM bandwidth
  gpu             card name and power limit, read in the same run
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402  (its module level puts the package on sys.path and imports torch)
import torch  # noqa: E402

VOCAB = {'70b': 32000, 'llama3-8b': 128256, '34b': 32016}
TITLE = {'70b': 'LLaMA-2-70B', 'llama3-8b': 'LLaMA-3-8B', '34b': 'CodeLlama-34B'}


def run(args):
    from gptq_b200 import engine
    dev = torch.device('cuda', 0)
    torch.cuda.set_device(dev)
    gpu = bench.gpu_identity(0)
    peak, _, peak_src = bench.datasheet_peaks()
    pos = args.context
    max_seq = pos + 1
    steps, warm = max(1, args.steps), max(3, args.warmup)
    for size in args.models:
        base = engine.synthetic_llama(size, bits=4, groupsize=bench.GROUP, vocab=VOCAB[size], device=str(dev), seed=0, max_seq=max_seq, use_graph=False)
        H, I, V, L, nh, nkv, hd = base.hidden, base.intermediate, base.vocab, len(base.layers), base.n_heads, base.n_kv_heads, base.head_dim
        per_layer = bench.alg_bytes_qlinear(H, H + 2 * nkv * hd, 4) + bench.alg_bytes_qlinear(H, H, 4) + 2 * bench.alg_bytes_qlinear(H, I, 4) + \
            bench.alg_bytes_qlinear(I, H, 4)
        for B in args.batch:
            dec = engine.LlamaDecoder(base.layers, base.embed, base.final_norm, base.lm_head, nh, batch=B, max_seq=max_seq, n_kv_heads=nkv)
            gen = torch.Generator(device=dev).manual_seed(1000 + B)
            dec.k_cache.normal_(0, 0.5, generator=gen)
            dec.v_cache.normal_(0, 0.5, generator=gen)
            dec.positions.fill_(pos)
            dec.tokens.copy_(torch.arange(1, B + 1, dtype=torch.int32))
            for _ in range(warm):
                dec.step()
            torch.cuda.synchronize()
            assert bool(torch.isfinite(dec.logits).all()), 'non-finite logits'
            t_dev = bench.timed(dec.step, steps, False)
            kv = B * 2 * L * (pos + 1) * nkv * hd * 2
            step_bytes = L * per_layer + V * H * 2 + kv
            t_step = t_dev / steps
            launches = dec.launches_per_step()
            print(json.dumps({
                'model': size, 'batch': B, 'metric': f'aggregate tokens/sec, synthetic {TITLE[size]} int4 g128, batch={B}, context {pos}',
                'value': B * steps / t_dev, 'unit': 'tokens/s', 'steps': steps, 'warmup': warm, 'ms_per_step': t_step * 1e3,
                'engine': 'persistent' if launches == 1 else 'kernel chain', 'launches_per_step': launches,
                'config': {'layers': L, 'hidden': H, 'intermediate': I, 'heads': nh, 'kv_heads': nkv, 'vocab': V, 'weights_bytes': L * per_layer,
                           'lm_head_bytes': V * H * 2, 'kv_bytes': kv},
                'bytes_per_step': step_bytes,
                'roofline': {'bound': 'hbm', 'achieved': step_bytes / t_step / 1e9, 'peak': peak, 'unit': 'GB/s', 'frac': step_bytes / t_step / 1e9 / peak,
                             'peak_source': peak_src},
                'gpu': gpu,
            }), flush=True)
            del dec
            torch.cuda.empty_cache()
        del base
        torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--models', default='70b,llama3-8b', type=lambda s: s.split(','), help=f'comma-separated, of {sorted(VOCAB)}')
    ap.add_argument('--batch', default='1,8', type=lambda s: [int(b) for b in s.split(',')], help='comma-separated batch sizes (1..8)')
    ap.add_argument('--context', type=int, default=2047, help='cached tokens per sequence (the position of the decoded token)')
    ap.add_argument('--steps', type=int, default=30)
    ap.add_argument('--warmup', type=int, default=5)
    args = ap.parse_args()
    if any(m not in VOCAB for m in args.models):
        sys.exit(f'--models: choose from {sorted(VOCAB)}')
    if any(not 1 <= b <= 8 for b in args.batch):
        sys.exit('--batch: the decode engine steps 1..8 sequences')
    run(args)


if __name__ == '__main__':
    main()
