#!/usr/bin/env python
"""Batched decode benchmark: aggregate tokens/s of the persistent decode kernel stepping B sequences per launch, one JSON line per batch size.

    python tools/batch_bench.py [--config 7b|13b-int3|65b] [--batch 1,2,4,8] [--context N] [--steps K] [--warmup W] [--dump-outputs DIR]

One random-init model (bench.py's synthetic weights) serves every batch size of the sweep.  Each of the B sequences has its own seeded random
KV cache holding `context` tokens, and the step decodes the next token of every sequence.  Reported per batch size:
  value         aggregate tokens/s = B x steps / device time (CUDA events around the graph replays)
  ms_per_step   device time of one step
  bytes_per_step  algorithmic bytes: quantized weights of the checkpoint + fp16 lm_head + B x KV cache at this context
  roofline      those bytes over the step time, against the H100 SXM data sheet's HBM bandwidth
  e2e           B tokens and positions in from pinned host memory, one step, [B, V] logits out, synchronised every step
A batch size outside the persistent kernel's plan (DESIGN.md section 4.1) is reported with the boundary it crosses and is not timed.
--dump-outputs DIR writes the last timed step's [B, V] logits and B tokens as DIR/b<B>_{logits,next_tokens}.npy.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402  (its module level puts the package on sys.path and imports torch)
import torch  # noqa: E402


def plan_boundary(dec, B):
    """Why this batch size does not take the persistent kernel."""
    teams = 2 * torch.cuda.get_device_properties(dec.dev).multi_processor_count
    if B * dec.n_heads > teams:
        return f'{B} x {dec.n_heads} (sequence, head) pairs exceed the {teams} attention teams'
    return f'the staged x of {B} sequences leaves fewer than 2 ring stages of shared memory'


def run(args):
    from gptq_b200 import engine
    dev = torch.device('cuda', 0)
    torch.cuda.set_device(dev)
    size, bits, act, title = bench.CONFIGS[args.config]
    pos = args.context
    max_seq = max(bench.SEQ, pos + 1)
    base = engine.synthetic_llama(size, bits=bits, groupsize=bench.GROUP, act_order=act, device=str(dev), seed=0, max_seq=max_seq, use_graph=False, batch=1)
    H, I, V, L = base.hidden, base.intermediate, base.vocab, len(base.layers)
    per_layer = bench.alg_bytes_qlinear(H, 3 * H, bits) + bench.alg_bytes_qlinear(H, H, bits) + 2 * bench.alg_bytes_qlinear(H, I, bits) + \
        bench.alg_bytes_qlinear(I, H, bits)
    peak, _, peak_src = bench.datasheet_peaks()
    gpu = bench.gpu_identity(0)
    steps, warm = max(1, args.steps), max(3, args.warmup)
    for B in args.batch:
        workload = f'{title.replace("batch=1", f"batch={B}")}, context {pos} (seq={max_seq}), {L} layers, random-init packed weights, B sequences with their own random caches'
        dec = engine.LlamaDecoder(base.layers, base.embed, base.final_norm, base.lm_head, base.n_heads, batch=B, max_seq=max_seq)
        if dec.launches_per_step() != 1:
            print(json.dumps({'batch': B, 'config': {'workload': workload}, 'value': None,
                              'outside_plan': f'{plan_boundary(dec, B)}: the step would take the kernel chain, which is not timed here'}))
            del dec
            continue
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
        if args.dump_outputs:
            bench.dump_outputs(args.dump_outputs, {f'b{B}_logits': dec.logits, f'b{B}_next_tokens': dec.next_tokens})

        tok_host = torch.arange(1, B + 1, dtype=torch.int32).pin_memory()
        pos_host = torch.full((B, ), pos, dtype=torch.int32).pin_memory()
        logits_host = torch.empty(B, V, dtype=torch.float16).pin_memory()

        def e2e_step():
            dec.tokens.copy_(tok_host, non_blocking=True)
            dec.positions.copy_(pos_host, non_blocking=True)
            dec.step()
            logits_host.copy_(dec.logits, non_blocking=True)
            torch.cuda.current_stream().synchronize()
            tok_host[0] = int(logits_host[0, :8].float().argmax())

        for _ in range(warm):
            e2e_step()
        t_e2e = bench.timed(e2e_step, steps, False)
        kv = B * 2 * L * (pos + 1) * H * 2
        step_bytes = L * per_layer + V * H * 2 + kv
        t_step = t_dev / steps
        print(json.dumps({
            'batch': B, 'metric': f'aggregate tokens/sec {title.replace("batch=1", f"batch={B}")}', 'value': B * steps / t_dev, 'unit': 'tokens/s',
            'steps': steps, 'warmup': warm, 'ms_per_step': t_step * 1e3, 'bytes_per_step': step_bytes,
            'config': {'workload': workload, 'weights_bytes': L * per_layer, 'lm_head_bytes': V * H * 2, 'kv_bytes': kv},
            'roofline': {'bound': 'hbm', 'kernel': 'llama_decode_mega_kernel', 'achieved': step_bytes / t_step / 1e9, 'peak': peak, 'unit': 'GB/s',
                         'frac': step_bytes / t_step / 1e9 / peak, 'peak_source': peak_src},
            'e2e': {'value': B * steps / t_e2e, 'unit': 'tokens/s', 'h2d_bytes_per_step': 8 * B, 'd2h_bytes_per_step': B * V * 2},
            'gpu_launches': dec.launches_per_step() * steps, 'gpu': gpu,
        }))
        del dec
        torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--config', default='7b', choices=[c for c in bench.CONFIGS if not c.endswith('-tp')])
    ap.add_argument('--batch', default='1,2,4,8', type=lambda s: [int(b) for b in s.split(',')], help='comma-separated batch sizes (1..8)')
    ap.add_argument('--context', type=int, default=bench.SEQ - 1, help='cached tokens per sequence (the position of the decoded token)')
    ap.add_argument('--steps', type=int, default=50)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--dump-outputs', metavar='DIR', default=None)
    args = ap.parse_args()
    if any(not 1 <= b <= 8 for b in args.batch):
        sys.exit('--batch: the persistent decode kernel serves 1..8 sequences per step')
    run(args)


if __name__ == '__main__':
    main()
