"""Kernel micro-benchmark: every LLaMA-7B QuantLinear shape at M=1 (rotating over distinct weight sets
totalling > L2 so reads are HBM-cold), CUDA-event timed.  Development tool; bench.py is the judged entry."""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'gptq-for-llama_b200'))
from gptq_b200 import ops  # noqa: E402


def alg_bytes(K, N, bits, gs, M):
    G = (K + gs - 1) // gs
    return K * N * bits // 8 + G * N * 2 + G * N * bits // 8 + 4 * K + 2 * M * K + 2 * M * N


def rand_layer(K, N, bits, gs, dev):
    G = (K + gs - 1) // gs
    qw = torch.randint(-2**31, 2**31 - 1, (K // 32 * bits, N), dtype=torch.int32, device=dev)
    qz = torch.randint(-2**31, 2**31 - 1, (G, N // 32 * bits), dtype=torch.int32, device=dev)
    s = (torch.rand(G, N, device=dev) * 1e-2 + 1e-3).half()
    g = (torch.arange(K, device=dev) // gs).int()
    return qw, s, qz, g


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--M', type=int, default=1)
    ap.add_argument('--bits', type=int, default=4)
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--hint', type=int, default=1)
    args = ap.parse_args()
    dev = torch.device('cuda:0')
    peak = 3350.0  # GB/s, H100 SXM data sheet
    gs = 128
    for (K, N, dual) in [(4096, 4096, False), (4096, 12288, False), (11008, 4096, False), (4096, 11008, True)]:
        per = alg_bytes(K, N, args.bits, gs, args.M) * (2 if dual else 1)
        nsets = max(2, int(400e6 // per) + 1)
        sets = [(rand_layer(K, N, args.bits, gs, dev), rand_layer(K, N, args.bits, gs, dev) if dual else None) for _ in range(nsets)]
        x = torch.randn(args.M, K, device=dev).half()
        hint = gs if args.hint else 0

        def run(i):
            a, b = sets[i % nsets]
            if dual:
                return ops.fused_mlp(x, a, b, args.bits, hint)
            return ops.matmul248(x, *a, args.bits, None, groupsize=hint)

        for i in range(nsets):
            run(i)
        torch.cuda.synchronize()
        # CUDA graph of one pass over all weight sets: removes the Python/ctypes launch overhead (~20 us/call)
        graph = torch.cuda.CUDAGraph()
        side = torch.cuda.Stream()
        with torch.cuda.stream(side):
            run(0)
            torch.cuda.synchronize()
            with torch.cuda.graph(graph, stream=side):
                for i in range(nsets):
                    run(i)
        torch.cuda.synchronize()
        graph.replay()
        torch.cuda.synchronize()
        ts = []
        for _ in range(args.iters):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            graph.replay()
            b.record()
            torch.cuda.synchronize()
            ts.append(a.elapsed_time(b) * 1e3 / nsets)
        ts.sort()
        med = ts[len(ts) // 2]
        b2b = ts[0]
        print(f'K={K} N={N} dual={dual} M={args.M} bits={args.bits}: graph-replay median {med:.2f} us/kernel ({per / med / 1e3:.0f} GB/s), best {b2b:.2f} us '
              f'({per / b2b / 1e3:.0f} GB/s = {per / b2b / 1e3 / peak:.2%} of measured {peak:.0f} GB/s); {nsets} weight sets')


if __name__ == '__main__':
    main()
