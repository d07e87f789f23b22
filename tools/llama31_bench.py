#!/usr/bin/env python
"""Decode throughput of LLaMA-3.1-8B (synthetic, all 32 layers, int4 g128, vocabulary 128256, RoPE base 5e5 with the llama3 frequency scaling)
at long contexts, one JSON line per (batch, context).

    python tools/llama31_bench.py [--configs 1:2047,1:8191,1:32767,1:131071,8:2047,8:32767] [--steps K] [--warmup W]

Each of the B sequences has its own seeded random KV cache holding `context` tokens, and the step decodes the next token of every sequence.
Batch 8 at 131071 is left out: its KV cache (8 x 17.2 GB) does not fit an 80 GB card.  Reported per line:
  value           aggregate tokens/s = B x steps / device time (CUDA events around the graph replays)
  bytes_per_step  algorithmic bytes, each counted once: quantized weights, fp16 lm_head, and every sequence's K/V rows (8 K/V heads per layer
                  and position).  The kernels stream a K/V row once per query head of its group (4 at LLaMA-3); how much of the repeats L2
                  serves is not measured here
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


def run(args):
    from gptq_b200 import engine
    dev = torch.device('cuda', 0)
    torch.cuda.set_device(dev)
    gpu = bench.gpu_identity(0)
    peak, _, peak_src = bench.datasheet_peaks()
    steps, warm = max(1, args.steps), max(3, args.warmup)
    base = engine.synthetic_llama('llama3-8b', bits=4, groupsize=bench.GROUP, vocab=128256, device=str(dev), seed=0, max_seq=16, use_graph=False)
    H, I, V, L, nh, nkv, hd = base.hidden, base.intermediate, base.vocab, len(base.layers), base.n_heads, base.n_kv_heads, base.head_dim
    per_layer = bench.alg_bytes_qlinear(H, H + 2 * nkv * hd, 4) + bench.alg_bytes_qlinear(H, H, 4) + 2 * bench.alg_bytes_qlinear(H, I, 4) + \
        bench.alg_bytes_qlinear(I, H, 4)
    for B, pos in args.configs:
        dec = engine.LlamaDecoder(base.layers, base.embed, base.final_norm, base.lm_head, nh, batch=B, max_seq=pos + 1, n_kv_heads=nkv, rms_eps=1e-5,
                                  rope_base=engine.LLAMA3_ROPE_BASE, rope_scaling=engine.LLAMA3_1_ROPE_SCALING)
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
            'model': 'llama3.1-8b', 'batch': B, 'context': pos,
            'metric': f'aggregate tokens/sec, synthetic LLaMA-3.1-8B int4 g128 (llama3 RoPE scaling), batch={B}, context {pos}',
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--configs', default='1:2047,1:8191,1:32767,1:131071,8:2047,8:32767',
                    type=lambda s: [tuple(int(v) for v in c.split(':')) for c in s.split(',')], help='comma-separated batch:context pairs')
    ap.add_argument('--steps', type=int, default=30)
    ap.add_argument('--warmup', type=int, default=5)
    args = ap.parse_args()
    if any(not 1 <= b <= 8 or not 0 <= p < 131072 for b, p in args.configs):
        sys.exit('--configs: batch 1..8, context 0..131071')
    run(args)


if __name__ == '__main__':
    main()
